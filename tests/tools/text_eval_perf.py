"""Cost of evaluating text vector files (-binary 0), parsed on the GPU (csrc/w2b_text.cu), at the shape of the
published vectors: V = 400 001, D = 800, text at bit levels 0 and 1.  Reports, with the card's name and power limit
read in the same run:
  * the parse kernel's time (torch.profiler, CUDA activities: every text_parse_kernel launch of one read) and the text
    bytes per second of kernel time, the host-to-device copies of the chunks, and the wall time of read_text_vectors;
  * the whole compute_accuracy call on the text file against the same call on the equivalent binary file (the values
    the text parses to), each in a fresh process, alternating, three times: wall time, peak host memory of the process
    (VmHWM) and peak device memory (cudaMemGetInfo sampled every 2 ms, less the process's context).
    python tests/tools/text_eval_perf.py [output.json]"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

V, D, NQ, REPS = 400001, 800, 19544, 3


def child(vf, qf):
    """One compute_accuracy call in this process: prints a JSON line."""
    import word2bits_b200 as w2b
    rt = C.CDLL("libcudart.so.12")
    free, total = C.c_size_t(), C.c_size_t()
    rt.cudaSetDevice(0)
    rt.cudaFree(None)
    rt.cudaMemGetInfo(C.byref(free), C.byref(total))
    base, peak, done = total.value - free.value, [0], []

    def sample():
        while not done:
            rt.cudaMemGetInfo(C.byref(free), C.byref(total))
            peak[0] = max(peak[0], total.value - free.value - base)
            time.sleep(0.002)
    th = threading.Thread(target=sample)
    th.start()
    t0 = time.perf_counter()
    rep, acc = w2b.compute_accuracy(vf, qf)
    wall = time.perf_counter() - t0
    done.append(1)
    th.join()
    print(json.dumps({"wall_s": wall, "gpu_ms": acc["gpu_ms"], "seen": acc["questions_seen"], "correct": acc["correct"],
                      "report": rep, "peak_device_bytes": peak[0],
                      "peak_host_bytes": peak_rss()}))


def peak_rss():
    """VmHWM of this process (ru_maxrss would include the parent's peak, inherited across fork and exec)."""
    with open("/proc/self/status") as f:
        return next(int(l.split()[1]) * 1024 for l in f if l.startswith("VmHWM:"))


def run_child(vf, qf):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", vf, qf], capture_output=True, text=True,
                       check=True)
    return json.loads(r.stdout.strip().splitlines()[-1])


def parse_profile(w2b, tf):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    w2b.read_text_vectors(tf)  # warm: module load, page cache
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        names, vec = w2b.read_text_vectors(tf)
        wall = time.perf_counter() - t0
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    parse = [e for e in kern if "text_parse_kernel" in e.name]
    copies = [e for e in kern if "HtoD" in e.name]
    us = lambda ev: sum(e.time_range.elapsed_us() for e in ev)
    return names, vec, {"parse_kernel_ms": us(parse) / 1e3, "parse_launches": len(parse),
                        "h2d_copy_ms": us(copies) / 1e3, "read_text_vectors_wall_s": wall}


def main():
    import word2bits_b200 as w2b
    from oracle import pyoracle as po
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"gpu": q, "V": V, "D": D, "questions": NQ, "runs": {}}
    print("card (name, power limit, max SM clock):", q, flush=True)
    tmp = tempfile.mkdtemp()
    corpus = os.path.join(tmp, "corpus.txt")
    with open(corpus, "w") as f:
        for a in range(0, V - 1, 1000):
            f.write(" ".join("w%d" % i for i in range(a, min(a + 1000, V - 1))) + "\n")
    c = w2b.Corpus(corpus, 1)
    assert c.vocab_size == V
    names = c.words()
    rng = np.random.default_rng(0)
    qf = os.path.join(tmp, "q.txt")
    with open(qf, "w") as f:
        for s in range(14):
            f.write(": s%d\n" % s)
            for _ in range(NQ // 14):
                f.write(" ".join(names[i] for i in rng.integers(1, 30000, 4)) + "\n")
    for bits in (0, 1):
        vec = rng.normal(size=(V, D)).astype(np.float32) * np.float32(0.3)
        if bits:
            vec = po.quantize(vec, bits)
        tf, bf = os.path.join(tmp, "vec.txt"), os.path.join(tmp, "vec.bin")
        c.write_vectors(tf, vec, 0)
        del vec
        _, parsed, prof = parse_profile(w2b, tf)
        c.write_vectors(bf, parsed, 1)
        del parsed
        r = dict(prof, text_bytes=os.path.getsize(tf), binary_bytes=os.path.getsize(bf))
        r["parse_text_GBps"] = r["text_bytes"] / (r["parse_kernel_ms"] * 1e6)
        calls = {"text": [], "binary": []}
        for _ in range(REPS):
            for kind, f in (("text", tf), ("binary", bf)):
                calls[kind].append(run_child(f, qf))
        assert calls["text"][0]["report"] == calls["binary"][0]["report"], "text and binary reports differ"
        for kind in calls:
            rs = calls[kind]
            r[kind] = {"wall_s": sorted(x["wall_s"] for x in rs), "gpu_ms": sorted(x["gpu_ms"] for x in rs),
                       "peak_host_MB": max(x["peak_host_bytes"] for x in rs) / 2 ** 20,
                       "peak_device_MB": max(x["peak_device_bytes"] for x in rs) / 2 ** 20}
        res["runs"]["bits%d" % bits] = r
        print("bit level %d: %.2f GB of text; parse kernel %.1f ms in %d launches = %.1f GB/s of text; H2D copies %.1f ms; "
              "read_text_vectors %.2f s" % (bits, r["text_bytes"] / 1e9, r["parse_kernel_ms"], r["parse_launches"],
                                              r["parse_text_GBps"], r["h2d_copy_ms"], r["read_text_vectors_wall_s"]))
        for kind in ("text", "binary"):
            k = r[kind]
            print("  compute_accuracy on the %s file: wall %s s, kernels %s ms, peak host %.0f MB, peak device %.0f MB"
                  % (kind, " / ".join("%.2f" % x for x in k["wall_s"]), " / ".join("%.1f" % x for x in k["gpu_ms"]),
                     k["peak_host_MB"], k["peak_device_MB"]), flush=True)
        os.remove(tf)
        os.remove(bf)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        child(sys.argv[2], sys.argv[3])
    else:
        main()
