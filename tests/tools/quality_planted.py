"""TEST INFRASTRUCTURE (runs the compiled reference under oracle/_ref next to the product).
SURVEY Appendix B quality protocol at full size: planted-topic corpus (V=20000, 50 topics, 250k
sentences x 20 tokens), D=200 W=8 neg=24 bitlevel 1, 3 epochs.  Reference (16 CPU threads) vs the GPU
CLI at its default shard count and at chosen shard counts.  Prints epoch losses
and same-topic purity of the top-10 neighbours of the 3000 most frequent words."""
import os, re, subprocess, sys, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
from tests.util import planted_topic_corpus, topic_purity

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
tmp = tempfile.mkdtemp()
path = planted_topic_corpus(os.path.join(tmp, "topics.txt"), vocab=20000, topics=50, sentences=250000, length=20)
common = ["-train", path, "-size", "200", "-window", "8", "-negative", "24", "-bitlevel", "1", "-iter", "3",
          "-min-count", "5", "-binary", "1", "-debug", "0"]


def read_bin(fn):
    with open(fn, "rb") as f:
        V, D = [int(x) for x in f.readline().split()]
        words, vec = [], np.empty((V, D), np.float32)
        for i in range(V):
            w = b""
            while True:
                ch = f.read(1)
                if ch == b" ":
                    break
                if ch != b"\n":
                    w += ch
            words.append(w.decode())
            vec[i] = np.frombuffer(f.read(4 * D), np.float32)
    return words, vec


def run(name, exe, extra):
    out = os.path.join(tmp, name + ".bin")
    t0 = time.time()
    r = subprocess.run([exe] + common + ["-output", out] + extra, capture_output=True, text=True)
    dt = time.time() - t0
    losses = [float(x) for x in re.findall(r"Epoch Loss: (-?[0-9.]+)", r.stdout)]
    words, vec = read_bin(out)
    pur = topic_purity(words, vec, 50, top_words=3000)
    print("%-28s wall %6.1f s  epoch losses %s  purity@10 %.4f" % (name, dt, ["%.4g" % l for l in losses], pur), flush=True)


ref = os.path.join(ROOT, "oracle", "_ref", "word2bits")
ours = os.path.join(ROOT, "word2bits_b200", "word2bits")
# python tests/tools/quality_planted.py [shard counts; 0 = the CLI's default, "ref" = the reference at 16 threads]
which = sys.argv[1:] or ["ref", "0", "16", "132", "2640"]
for w in which:
    if w == "ref":
        if os.path.exists(ref):
            run("reference -threads 16", ref, ["-threads", "16"])
    elif w == "0":
        run("gpu default shards", ours, [])
    else:
        run("gpu -threads %s" % w, ours, ["-threads", w])
