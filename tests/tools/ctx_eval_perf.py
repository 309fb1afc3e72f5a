"""Evaluating a training context in place (Trainer.compute_accuracy) against the file round trip it replaces, on the GPU:
    python tests/tools/ctx_eval_perf.py [V] [D] [questions] [distinct words] [rounds]
Defaults are the Google-set shape: V = 400 000 (plus </s>), D = 800, 19 544 questions over about 900 distinct words,
made the way eval_packed_perf.py makes them.  For training bit levels 0, 1 and 2 a context is initialised (InitNet's
random u, then one short training step so that v is not zero) and, after a warm-up of each, the two ways alternate in
one process: (a) the context call; (b) export() + write_vectors (write_packed at 1 and 2 bits) + the file-based
call.  The reports must be equal.  Printed per call: the host clock around the whole call, gpu_ms (CUDA events) and
the peak device memory in use during the call above what was in use before it, sampled with cudaMemGetInfo every
millisecond from a second thread.  Needs a GPU; the card's name and power limit are read in the same run."""
import os
import subprocess
import sys
import tempfile
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import word2bits_b200 as w2b  # noqa: E402

V, D, NQ, NW, ROUNDS = (int(sys.argv[i]) if len(sys.argv) > i else d for i, d in enumerate((400000, 800, 19544, 900, 3), 1))
assert torch.cuda.is_available(), "this measurement needs a GPU"
print("GPU: " + subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip(), flush=True)
tmp = tempfile.mkdtemp()
rng = np.random.default_rng(0)
corpus_file = os.path.join(tmp, "corpus.txt")
with open(corpus_file, "w") as f:  # every word once: a vocabulary of V words (+ </s>) in a few MB
    f.write(" ".join("w%d" % i for i in range(V)) + "\n")
corpus = w2b.Corpus(corpus_file, 1)
qf = os.path.join(tmp, "q.txt")
qwords = rng.choice(min(V, 30000), NW, replace=False)
with open(qf, "w") as f:
    for s in range(14):
        f.write(": s%d\n" % s)
        for _ in range(NQ // 14):
            f.write(" ".join("w%d" % i for i in rng.choice(qwords, 4)) + "\n")


class PeakMemory:
    """Largest device memory in use (cudaMemGetInfo) while the block runs, above the use when it started."""

    def __enter__(self):
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()
        self.base, self.total, self.low, self.run = total - free, total, free, True
        self.t = threading.Thread(target=self._poll)
        self.t.start()
        return self

    def _poll(self):
        while self.run:
            self.low = min(self.low, torch.cuda.mem_get_info()[0])
            time.sleep(0.001)

    def __exit__(self, *a):
        self.run = False
        self.t.join()
        self.peak = self.total - self.low - self.base


def timed(fn):
    with PeakMemory() as m:
        t0 = time.time()
        rep, acc = fn()
        wall = time.time() - t0
    return rep, acc, wall, m.peak


for bits in (0, 1, 2):
    t = w2b.Trainer(corpus, size=D, bitlevel=bits, threads=64, iter=1)
    t.epoch_begin()
    t.train_step(200)  # v gets a few updates: quantize(u + v) is not quantize(u)
    path = os.path.join(tmp, "vec%d" % bits)

    def in_place():
        return t.compute_accuracy(qf)

    def round_trip():
        vec = t.export()
        if bits in (1, 2):
            corpus.write_packed(path, vec, bits)
            return w2b.compute_accuracy_packed(path, qf)
        corpus.write_vectors(path, vec, 1)
        return w2b.compute_accuracy(path, qf)

    rep_c, acc_c, _, _ = timed(in_place)  # warm-up
    rep_f, acc_f, _, _ = timed(round_trip)
    assert rep_c == rep_f, "the context's report differs from the file's"
    print("\ntraining bit level %d, V=%d D=%d, %d questions over %d distinct words: reports equal"
          % (bits, t.V, D, acc_c["questions_seen"], NW), flush=True)
    print("  " + rep_c.strip().splitlines()[-2].strip())
    for r in range(ROUNDS):
        for label, fn in (("context   ", in_place), ("round trip", round_trip)):
            rep, acc, wall, peak = timed(fn)
            assert rep == rep_c
            print("  round %d %s: whole call %6.3f s, kernels %7.1f ms, peak device memory +%7.1f MB"
                  % (r, label, wall, acc["gpu_ms"], peak / 1e6), flush=True)
    t.close()
    if os.path.exists(path):
        os.unlink(path)
