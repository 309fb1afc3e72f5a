"""Timing of the top-k lists (w2b_analogy_topk, w2b_nearest) on the GPU, next to the arg-max evaluator:
    python tests/tools/topk_perf.py [V] [D] [questions] [distinct words]
Defaults are the Google-set shape: V = 400 000, D = 800, 19 544 questions over 900 distinct words; random 1-bit and
2-bit levels, each written as a word2vec-binary file and as a packed file.  Per file: analogy lists at k = 1, 10, 100
and nearest neighbours of 900 and of 10 000 words at k = 40.  Checks: the k = 1 lists are w2b_analogy_answers' answers
for every question, and 64 sampled analogy queries at k = 100 equal the CPU restatement (tests/topk_oracle.py).
Times are CUDA events (gpu_ms: from the first kernel to the last, uploads outside) and the host clock around the whole
call (file read and H2D included); the peak device memory of a call is sampled with cudaMemGetInfo from a second
thread while it runs (every millisecond, above what was in use before); one torch.profiler pass per call, and one of
the arg-max evaluator, gives every kernel."""
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
from tests import packed_cases as pc  # noqa: E402
from tests import topk_oracle as to  # noqa: E402

V, D, NQ, NW = (int(sys.argv[i]) if len(sys.argv) > i else d for i, d in enumerate((400000, 800, 19544, 900), 1))
assert torch.cuda.is_available(), "this measurement needs a GPU"
print("GPU: " + subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip(), flush=True)
tmp = tempfile.mkdtemp()
rng = np.random.default_rng(0)
qf = os.path.join(tmp, "q.txt")
qwords = rng.choice(min(V, 30000), NW, replace=False)
with open(qf, "w") as f:
    for s in range(14):
        f.write(": s%d\n" % s)
        for _ in range(NQ // 14):
            f.write(" ".join("w%d" % i for i in rng.choice(qwords, 4)) + "\n")
near = {n: ["w%d" % i for i in rng.choice(V, n, replace=False)] for n in (900, 10000)}


def write_both(bits):
    vf, pf = os.path.join(tmp, "vec%d.bin" % bits), os.path.join(tmp, "vec%d.packed" % bits)
    levels = np.array([-1, 1], np.float32) / np.float32(3) if bits == 1 else np.array([-0.75, -0.25, 0.25, 0.75], np.float32)
    with open(vf, "wb") as fv, open(pf, "wb") as fp:
        fv.write(b"%d %d\n" % (V, D))
        fp.write(b"%d %d %d\n" % (V, D, bits))
        for a in range(0, V, 20000):
            x = levels[rng.integers(0, len(levels), (min(20000, V - a), D))]
            rows = pc.pack_rows(x, bits)
            for i in range(len(x)):
                name = b"w%d " % (a + i)
                fv.write(name + x[i].tobytes() + b"\n")
                fp.write(name + rows[i].tobytes() + b"\n")
    return vf, pf


def peak_bytes(fn):
    """(fn(), peak device bytes in use above the level before the call)"""
    base = torch.cuda.mem_get_info()
    peak, done = [0], threading.Event()

    def poll():
        while not done.is_set():
            free, total = torch.cuda.mem_get_info()
            peak[0] = max(peak[0], (base[0] - free))
            time.sleep(0.001)
    t = threading.Thread(target=poll)
    t.start()
    try:
        out = fn()
    finally:
        done.set()
        t.join()
    return out, peak[0]


def kernel_times(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if ("eval_" in e.key or "topk" in e.key) and t:
            key = e.key.split("(")[0].replace("void ", "")
            for ns in ("w2b::bits::", "w2b::tc::", "w2b::topk::", "(anonymous namespace)::"):
                key = key.replace(ns, "")
            out[key] = (t / 1e3, e.count)
    return out


for bits in (1, 2):
    vf, pf = write_both(bits)
    ans = w2b.analogy_answers(vf, qf, bitlevel=bits)
    t0 = time.time()
    _, acc = w2b.compute_accuracy(vf, qf, bitlevel=bits)
    print("\n%d-bit levels, V=%d D=%d, %d questions over %d words; arg-max evaluator (fp32 file): kernels %.1f ms, wall %.2f s"
          % (bits, V, D, len(ans), NW, acc["gpu_ms"], time.time() - t0))
    _, accp = w2b.compute_accuracy_packed(pf, qf)
    print("  arg-max evaluator (packed file): kernels %.1f ms" % accp["gpu_ms"])
    for label, fn in (("fp32", lambda: w2b.compute_accuracy(vf, qf, bitlevel=bits)), ("packed", lambda: w2b.compute_accuracy_packed(pf, qf))):
        print("  arg-max %s kernels (torch.profiler, ms x launches): " % label
              + ", ".join("%s %.2f x %d" % (k, t, n) for k, (t, n) in sorted(kernel_times(fn).items())), flush=True)
    names, M = None, None
    for label, f, kw in (("fp32  ", vf, dict(bitlevel=bits)), ("packed", pf, {})):
        runs = [("analogy k=%d" % k, lambda k=k: w2b.analogy_topk(f, qf, k, **kw)) for k in (1, 10, 100)]
        runs += [("nearest %d k=40" % n, lambda n=n: w2b.nearest(f, near[n], 40, **kw)) for n in (900, 10000)]
        for name, fn in runs:
            t0 = time.time()
            (ids, scores, st), dev = peak_bytes(fn)
            wall = time.time() - t0
            print("  %s %-16s kernels %8.1f ms, wall %6.2f s, %5.1f candidates and %5.1f re-scored per query, %d chunks, "
                  "simt %d, peak device memory %.0f MB" % (label, name, st["gpu_ms"], wall, st["candidates"] / st["queries"],
                                                          st["rescored"] / st["queries"], st["chunks"], st["simt"], dev / 1e6),
                  flush=True)
            if name == "analogy k=1":
                assert np.array_equal(ids[:, 0], ans), "k = 1 lists differ from the evaluator's answers"
            if name == "analogy k=100":
                if M is None:
                    names, M = to.load(vf, bits)
                    queries = to.analogy_queries(qf, names)
                    sample = rng.choice([i for i, q in enumerate(queries) if q is not None], 64, replace=False)
                    want = to.lists(M, [queries[i] for i in sample], k=100)
                assert np.array_equal(ids[sample], want[0]), "sampled lists differ from the oracle"
                assert np.array_equal(scores[sample].view(np.uint32), want[1].view(np.uint32))
        for name, fn in runs[1:2] + runs[3:4]:
            print("  %s %s kernels (torch.profiler, ms x launches): " % (label, name)
                  + ", ".join("%s %.2f x %d" % (k, t, n) for k, (t, n) in sorted(kernel_times(fn).items())), flush=True)
    print("  k = 1 lists equal the evaluator's answers for all %d questions; 64 sampled k = 100 lists equal the oracle's"
          % len(ans))
    os.unlink(vf)
    os.unlink(pf)
