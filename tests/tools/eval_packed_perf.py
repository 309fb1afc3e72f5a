"""Timing of the analogy evaluator on a packed vector file against the same vectors as word2vec-binary, on the GPU:
    python tests/tools/eval_packed_perf.py [V] [D] [questions] [distinct words] [rounds]
Defaults are the Google-set shape: V = 400 000, D = 800, 19 544 questions over about 900 distinct words.  For 1-bit
and 2-bit levels the two evaluators alternate in one process after a warm-up call each; the reports must be equal.
Needs a GPU; the byte counts are computed from the shapes, the times are CUDA events (gpu_ms), the host clock around
the whole call (file read and H2D included) and, per kernel, torch.profiler in a pass of its own."""
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import word2bits_b200 as w2b  # noqa: E402
from tests import packed_cases as pc  # noqa: E402

V, D, NQ, NW, ROUNDS = (int(sys.argv[i]) if len(sys.argv) > i else d for i, d in enumerate((400000, 800, 19544, 900, 3), 1))
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


def timed(fn):
    t0 = time.time()
    rep, acc = fn()
    return rep, acc, time.time() - t0


def kernel_times(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if "eval_" in e.key and t:
            out[e.key.split("(")[0].replace("void ", "").replace("w2b::bits::", "").replace("w2b::tc::", "")] = (t / 1e3, e.count)
    return out


for bits in (1, 2):
    vf, pf = write_both(bits)
    fp32 = lambda: w2b.compute_accuracy(vf, qf, bitlevel=bits)
    packed = lambda: w2b.compute_accuracy_packed(pf, qf)
    rep_f, acc_f, _ = timed(fp32)  # warm-up
    rep_p, acc_p, _ = timed(packed)
    assert rep_f == rep_p, "the packed evaluator's report differs from the fp32 evaluator's"
    ans_f, ans_p = w2b.analogy_answers(vf, qf, bitlevel=bits), w2b.analogy_answers_packed(pf, qf)
    assert np.array_equal(ans_f, ans_p), "%d of %d questions are answered differently" % ((ans_f != ans_p).sum(), len(ans_f))
    print("\nboth evaluators choose the same word for all %d questions (%d have an answer)" % (len(ans_f), (ans_f >= 0).sum()))
    nq, W = acc_p["questions_seen"], NW
    Dp, Wp, nbytes = (D + 31) // 32 * 32, ((D + 31) // 32 + 3) // 4 * 4, (D * bits + 7) // 8
    chunk = min((V + 1023) // 1024 * 1024, max(1024, (32 << 20) // 4 // W // 1024 * 1024))
    print("%d-bit levels, V=%d D=%d, %d questions over %d distinct words" % (bits, V, D, nq, W))
    print("  bytes read and copied to the device: fp32 %.1f MB, packed %.1f MB" % (V * D * 4 / 1e6, V * nbytes / 1e6))
    print("  device bytes allocated: fp32 path %.1f MB (table %.1f, queries %.1f, candidates %.1f), packed path %.1f MB "
          "(rows %.1f, planes %.1f, G chunk of %d words %.1f, candidates %.1f)"
          % ((V * Dp * 4 + nq * Dp * 4 + nq * 1024 * 12) / 1e6, V * Dp * 4 / 1e6, nq * Dp * 4 / 1e6, nq * 1024 * 12 / 1e6,
             (V * nbytes + V * Wp * 4 * bits + V * 12 + W * chunk * 4 + nq * 1024 * 12) / 1e6, V * nbytes / 1e6,
             V * Wp * 4 * bits / 1e6, chunk, W * chunk * 4 / 1e6, nq * 1024 * 12 / 1e6))
    print("  popcounts of the Gram kernel: %.2e (W x V x ceil(D/32) word pairs x %d); multiply-adds of the fp32 contraction: %.2e"
          % (W * V * ((D + 31) // 32) * (1 if bits == 1 else 5), 1 if bits == 1 else 5, nq * V * D))
    for r in range(ROUNDS):
        for label, fn in (("fp32  ", fp32), ("packed", packed)):
            rep, acc, wall = timed(fn)
            assert rep == rep_f
            print("  round %d %s: kernels %8.1f ms, wall %6.2f s, %.1f candidates and %.2f re-scored per question"
                  % (r, label, acc["gpu_ms"], wall, acc["candidates"] / nq, acc["rescored"] / nq), flush=True)
    for label, fn in (("fp32  ", fp32), ("packed", packed)):
        print("  kernels of one %s call (torch.profiler, ms x launches): " % label.strip()
              + ", ".join("%s %.2f x %d" % (k, t, n) for k, (t, n) in sorted(kernel_times(fn).items())), flush=True)
    os.unlink(vf)
    os.unlink(pf)
