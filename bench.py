#!/usr/bin/env python
"""bench.py — Word2Bits training path on H100: words/sec at bitlevel=1 size=800 negative=24.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--dump-outputs DIR]

One "step" = every corpus shard advances by --words-per-shard words (whole sentences) of a
synthetic Zipf(1.0) corpus, V=400k, window 10 — BASELINE.json configs[1].  N>1 is launched
under torchrun (one rank per GPU): every GPU trains its own shard range on a full replica of
u/v and the replicas are all-reduce-averaged over NCCL every --sync-every steps.
Prints ONE JSON line (rank 0).  See DESIGN.md "Measurement" for what each field means.

--dump-outputs DIR writes, after the timed steps (inputs depend only on the arguments):
  last_step.npy   float64: words, positions, context_rows, target_rows, shards_done, word_count_actual of the last
                  timed step — they depend only on the inputs, so they compare exactly;
  probe_step.npy  float64: loss, alpha, words, positions, context_rows, target_rows of one step of the same kernel
                  (same instantiation, same step size) over shard 0's tokens from the initial tables, run as ONE
                  shard, and probe_rows.npy / probe_u.npy / probe_v.npy: a fixed, seeded sample of 4096 rows (the
                  2048 most frequent words + 2048 seeded others) of u and v after that step, float32.  One shard
                  trains its positions strictly in order, so these repeat to rounding and carry the kernel's
                  arithmetic (gradient, expTable, quantize, scatter-add); compare them with an fp32 tolerance.
The tables, loss and alpha of the timed step itself are not dumped: its 1584 shards train lock-free (Hogwild, like
the reference's threads), so those values depend on how the shards interleave and differ from run to run.

--workload c3|c4|c5 runs the other BASELINE.json configurations through the same harness (they
are parity-test shapes, not the headline: the default is c2).
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "words/sec training throughput, bitlevel=1 size=800 neg=24; HBM GB/s vs peak"
V, D, WINDOW, NEG, BITS = 400_000, 800, 10, 24, 1
SAMPLE, ALPHA = 1e-3, 0.05
# BASELINE.json configs[1..4]: name -> (V, D, window, negative, bitlevel, workload text)
WORKLOADS = {
    "c2": (400_000, 800, 10, 24, 1, "synthetic Zipf corpus vocab=400k, bitlevel=1, size=800, window=10, negative=24"),
    "c3": (400_000, 400, 10, 12, 2, "synthetic Zipf corpus vocab=400k, bitlevel=2, size=400, window=10, negative=12"),
    "c4": (400_000, 400, 10, 24, 0, "synthetic Zipf corpus vocab=400k, bitlevel=0 (fp32), size=400, window=10, negative=24"),
    "c5": (3_700_000, 800, 10, 24, 1, "synthetic Zipf corpus vocab=3.7M, bitlevel=1, size=800, window=10, negative=24"),
}
WORKLOAD, WORKLOAD_TEXT = "c2", WORKLOADS["c2"][5]


def select_workload(name):
    global V, D, WINDOW, NEG, BITS, WORKLOAD, WORKLOAD_TEXT
    V, D, WINDOW, NEG, BITS, WORKLOAD_TEXT = WORKLOADS[name]
    WORKLOAD = name
FALLBACK_HBM_GBS = 3350.0  # H100 SXM data sheet (HBM3)
DUMP_FIELDS = ("words", "positions", "context_rows", "target_rows", "shards_done", "word_count_actual")
PROBE_FIELDS = ("loss", "alpha", "words", "positions", "context_rows", "target_rows")
PROBE_HOT_ROWS, PROBE_ROWS = 2048, 4096


def zipf_cdf(v):
    p = 1.0 / np.arange(1, v + 1, dtype=np.float64)
    return np.cumsum(p) / p.sum(), p / p.sum()


def synth_ids(n, seed, cdf):
    """n token ids in [1, V] (id = Zipf rank, so the vocabulary is already count-sorted).
    Deterministic: chunk c of 4 Mi tokens is drawn from default_rng([seed, c]); chunks are filled by a
    thread pool (numpy releases the GIL inside random() and searchsorted())."""
    from concurrent.futures import ThreadPoolExecutor
    out = np.empty(n, np.int32)
    step = 1 << 22
    vmax = len(cdf)

    def fill(c):
        a, b = c * step, min(n, (c + 1) * step)
        rng = np.random.default_rng([seed, c])
        out[a:b] = np.minimum(np.searchsorted(cdf, rng.random(b - a)) + 1, vmax)

    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as ex:
        list(ex.map(fill, range((n + step - 1) // step)))
    return out


def expected_counts(total_tokens, pmf):
    cn = np.maximum(np.rint(pmf * total_tokens), 1).astype(np.int64)
    return np.concatenate([[0], cn])  # </s> never occurs (text8-style corpus, no newlines)


class ClockSampler:
    """nvidia-smi clocks / throttle reasons / power limit during the timed region (read-only queries)."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap,power.limit")

    def __init__(self, index):
        self.rows, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), line.strip()))

    def stop(self, t0, t1):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, plim, reasons = [], None, None, set()
        for ts, line in self.rows:
            f = [x.strip() for x in line.split(",")]
            if len(f) < 8 or not (t0 - 0.05 <= ts <= t1 + 0.15):
                continue
            try:
                sm.append(float(f[0])); mx = float(f[1])
            except ValueError:
                continue
            try:
                plim = float(f[7])
            except ValueError:
                pass
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": mx, "power_limit_w": plim,
                "reasons": sorted(reasons), "samples": len(sm)}


def measured_peak():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return FALLBACK_HBM_GBS, "H100 SXM data sheet (not measured)"


def ncu_traffic_per_position():
    """DRAM bytes per trained position of the training kernel, when an ncu capture of this workload at the bench's
    own step size has been stored (profiles/traffic.json, written by tools/measure_traffic.sh and
    tools/make_traffic_json.py: dram__bytes_read.sum + dram__bytes_write.sum of one launch, divided by the positions
    that launch trained); None otherwise."""
    try:
        with open(os.path.join(ROOT, "profiles", "traffic.json")) as f:
            return float(json.load(f)[WORKLOAD]["dram_bytes_per_position"])
    except Exception:
        return None


# ------------------------------------------------------------------------------ reference arm
def _write_text(ids, path_prefix):
    words = np.array([("w%d" % i).encode() for i in range(V + 1)], dtype=object)
    tmp = tempfile.NamedTemporaryFile(prefix=path_prefix, suffix=".txt", delete=False)
    step = 1 << 20
    for a in range(0, len(ids), step):
        tmp.write(b" ".join(words[ids[a:a + step]]) + b" ")
    tmp.close()
    return tmp.name


def host_core_budget():
    """Cores this process may use: the affinity mask, capped by a cgroup CPU quota when one is set."""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    quota = None
    try:  # cgroup v2
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            quota = float(q) / float(per)
    except Exception:
        try:  # cgroup v1
            q = float(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / per
        except Exception:
            pass
    if quota:
        n = max(1, min(n, int(quota + 0.5)))
    return n, quota


def ref_flavour(po):
    """The reference's Makefile builds with -march=native (Makefile:2).  oracle/_ref holds such a build
    (libw2b_ref_native.so, made where the repo was built) beside the portable x86-64-v3 one; the native one is
    used when it runs on this host (probed in a child process: an illegal instruction must not take the bench down)."""
    if os.environ.get("W2B_REF_FLAVOUR"):
        return os.environ["W2B_REF_FLAVOUR"]
    if po.ref_available("native"):
        probe = ("import sys; sys.path.insert(0, %r); from oracle import pyoracle as po; r = po.Ref('native'); "
                 "import numpy as np; print(r.L.ref_quantize(0.3, 1))" % ROOT)
        try:
            r = subprocess.run([sys.executable, "-c", probe], capture_output=True, text=True, timeout=120)
            if r.returncode == 0:
                return "native"
        except Exception:
            pass
    return "o3" if po.ref_available("o3") else None


def _ref_runner(po, path, threads, iters, flavour):
    """(run_one_pass, words_per_pass, kind) for the reference on `path` with `threads` threads."""
    if flavour:
        ref = po.Ref(flavour)
        ref.configure(path, D, WINDOW, NEG, BITS, threads=threads, iters=iters, min_count=1, alpha=ALPHA, sample=SAMPLE)
        ref.learn_vocab(); ref.init_net(); ref.init_unigram()
        return ref.train_epoch, ref.train_words, "reference"
    corpus = po.Corpus(path, 1)
    model = po.OracleModel(corpus, D, WINDOW, NEG, BITS, shards=threads, iters=iters, alpha=ALPHA, sample=SAMPLE)
    return model.train_epoch_threads, corpus.train_words, "port"


def run_reference(args, rank, budget_s=100.0):
    """The reference's own CPU implementation of the path (oracle/_ref = the unmodified source compiled as a
    library, -march=native like its Makefile when that build runs here, else x86-64-v3; else the C port) on a
    bounded sample of the same workload; one step = one pass over the sample (the reference's per-epoch thread
    launch).  Threads: best of {all, 1/2, 1/4 of the cores this process may use} on a >= 2 M-token calibration pass
    (Hogwild on two sockets can get slower with more threads; a short pass would measure thread start-up instead);
    the sample is sized so that W+K passes fit the time budget."""
    if rank != 0:
        return None
    from oracle import pyoracle as po
    cores, quota = host_core_budget()
    flavour = ref_flavour(po)
    cdf, _ = zipf_cdf(V)
    ids = synth_ids(int(os.environ.get("W2B_REF_MAX_TOKENS", 16_000_000)), 4242, cdf)
    cands = [int(os.environ["W2B_REF_THREADS"])] if "W2B_REF_THREADS" in os.environ else \
        sorted({max(1, cores // k) for k in (1, 2, 4)}, reverse=True)
    cal_n = min(len(ids), int(os.environ.get("W2B_REF_CAL_TOKENS", 2_000_000)))  # (tests shrink it)
    cal = _write_text(ids[:cal_n], "w2b_cal_")
    best = (0.0, cands[-1])
    tried = []
    try:
        for th in cands:
            run, wpp, kind = _ref_runner(po, cal, th, 1, flavour)
            t0 = time.time()
            run()
            rate = wpp / (time.time() - t0)
            tried.append((th, round(rate)))
            if rate > best[0]:
                best = (rate, th)
    finally:
        os.unlink(cal)
    rate, threads = best
    passes = args.steps + args.warmup
    n = int(min(len(ids), max(int(os.environ.get("W2B_REF_MIN_TOKENS", 1_000_000)), rate * min(15.0, budget_s / passes))))
    path = _write_text(ids[:n], "w2b_ref_")
    distinct = int(len(np.unique(ids[:n])))
    try:
        run, words_per_pass, kind = _ref_runner(po, path, threads, passes, flavour)
        for _ in range(args.warmup):
            run()
        t0 = time.time()
        for _ in range(args.steps):
            run()
        dt = time.time() - t0
    finally:
        os.unlink(path)
    value = words_per_pass * args.steps / dt
    build = {"native": "oracle/_ref (unmodified reference, -O3 -march=native as its Makefile:2)",
             "o3": "oracle/_ref (unmodified reference, -O3 -march=x86-64-v3: the native build does not run on this host)",
             None: "oracle C port"}.get(flavour, "oracle/_ref (%s)" % flavour)
    sample = ("%d-token Zipf(1.0) V=%d text sample (%d distinct words occur, so fewer table rows than the GPU arm's %d: "
              "favours the CPU), %d timed passes, %s; threads chosen from %s (words/s on a %d-token calibration pass); "
              "cores usable by this process: %d%s" % (
                  n, V, distinct, V, args.steps, build, tried, cal_n, cores,
                  " (cgroup quota %.1f)" % quota if quota else ""))
    return {"metric": METRIC, "value": value, "unit": "words/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic", "impl": "reference",
            "config": {"workload": WORKLOAD_TEXT + " (CPU, bounded sample)",
                       "threads": threads, "host_threads": cores, "host_cpu_count": os.cpu_count(),
                       "distinct_words_in_sample": distinct, "sample_tokens": n},
            "cpu_baseline": {"value": value, "unit": "words/s", "cores": threads, "kind": kind, "sample": sample},
            "e2e": {"value": value, "unit": "words/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}


def cpu_baseline_leg():
    """Bounded (~10-30 s) run of the reference on this host's cores, for the cpu_baseline object."""
    class A:
        pass
    a = A()
    a.steps, a.warmup, a.gpus = 1, 0, 1
    out = run_reference(a, 0, budget_s=15.0)
    return out["cpu_baseline"]


# ------------------------------------------------------------------------------------ GPU arm
def dump_outputs(path, st, make_probe, B):
    """The run-independent counters the last timed step returned (DUMP_FIELDS, in that order), and one step of the
    same kernel as a single shard (PROBE_FIELDS and a seeded row sample of u and v): see the module docstring."""
    os.makedirs(path, exist_ok=True)
    np.save(os.path.join(path, "last_step.npy"), np.array([st[k] for k in DUMP_FIELDS], np.float64))
    t = make_probe()
    ps = t.train_step(B)
    u, v = t.download_raw()
    t.close()
    rest = np.random.default_rng(1234).choice(np.arange(PROBE_HOT_ROWS + 1, u.shape[0]), PROBE_ROWS - PROBE_HOT_ROWS,
                                              replace=False)
    rows = np.concatenate([np.arange(1, PROBE_HOT_ROWS + 1), np.sort(rest)])  # (row 0 is </s>, never trained here)
    np.save(os.path.join(path, "probe_step.npy"), np.array([ps[k] for k in PROBE_FIELDS], np.float64))
    np.save(os.path.join(path, "probe_rows.npy"), rows.astype(np.float64))
    np.save(os.path.join(path, "probe_u.npy"), np.ascontiguousarray(u[rows], np.float32))
    np.save(os.path.join(path, "probe_v.npy"), np.ascontiguousarray(v[rows], np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--words-per-shard", type=int, default=65536)
    ap.add_argument("--sync-every", type=int, default=0,
                    help="steps between two replica exchanges; 0 = 4, or more when the tables are large (one exchange per ~3.2 GB-steps: C2 4, C5 8)")
    ap.add_argument("--sync-mode", default="avg", choices=["avg", "sum"],
                    help="replica exchange: average (BASELINE.json's north_star) or sum of every rank's updates")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--workload", default="c2", choices=sorted(WORKLOADS))
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's counters and a single-shard probe of the same kernel to DIR/*.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    select_workload(args.workload)
    if args.sync_every <= 0:
        args.sync_every = max(4, int(round(2.0 * (V + 1) * D * 4 / 3.2e9)))
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))

    if args.impl == "reference":
        out = run_reference(args, rank)
        if out is not None:
            print(json.dumps(out), flush=True)
        return 0

    import torch
    import word2bits_b200 as w2b
    from word2bits_b200.parallel import DataParallel, exchange_unique_id
    if not torch.cuda.is_available() or w2b.device_count() == 0:
        raise SystemExit("bench.py: no CUDA device — the product path has no CPU fallback")
    dist = None
    if world > 1:
        os.environ.setdefault("NCCL_DEBUG", "WARN")  # keep stdout to the one JSON line
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    # ---- synthetic workload: every rank owns a contiguous 1/world of the corpus (weak scaling)
    cfg0 = dict(size=D, window=WINDOW, negative=NEG, bitlevel=BITS, alpha=ALPHA, sample=SAMPLE, iter=1, device=local)
    probe = w2b.Trainer(None, vocab_size=V + 1, threads=None, init=False, **cfg0)
    S_local = probe.threads
    probe.close()
    S = S_local * world
    B = args.words_per_shard
    total_steps = args.steps + args.warmup
    # keep the synthetic corpus of one rank under ~300 M tokens (1.2 GB of host ids): very long runs
    # get proportionally shorter steps instead of a bigger corpus
    while B > 8192 and (total_steps + 2) * (B + 1500) * 1.05 * S_local > 300e6:
        B //= 2
    per_shard = int((total_steps + 2) * (B + 1500) * 1.05) + 4096
    n_local = per_shard * S_local
    cdf, pmf = zipf_cdf(V)
    ids = synth_ids(n_local, 42 + rank, cdf)
    cn = expected_counts(n_local * world, pmf)
    train_words = int(n_local) * world
    # global shard table; this rank's shards index into its own token array
    start = np.zeros(S, np.int64)
    start[rank * S_local:(rank + 1) * S_local] = np.arange(S_local, dtype=np.int64) * per_shard
    first = np.full(S, -1, np.int32)

    def make(resident):
        t = w2b.Trainer(None, vocab_size=V + 1, threads=S, shard_range=(rank * S_local, (rank + 1) * S_local),
                        init=False, sync_mode=1 if args.sync_mode == "sum" else 0, **cfg0)
        t.set_vocab_counts(cn, train_words)
        t.set_corpus(ids, start, first, resident)
        t.init_tables()
        if world > 1:
            t.nccl_init(exchange_unique_id(dist, w2b.nccl_unique_id, device="cuda"), rank, world)
        return t

    def run(t, steps, warmup, sampler_index=None):
        dp = DataParallel(t, dist, args.sync_every, device="cuda")
        for i in range(warmup):
            dp.step(B)
        if world > 1:
            # the first collective of a communicator sets up its transports (hundreds of ms): keep that, like every
            # other one-time cost, out of the timed region; then restart the cadence so that the timed steps see
            # exactly steps // sync_every exchanges
            t.sync()
            dp.steps = dp.syncs = 0
            dp.sync_ms = 0.0
        torch.cuda.synchronize()
        if dist:
            dist.barrier()
        torch.cuda.synchronize()
        clocks = ClockSampler(sampler_index) if sampler_index is not None else None
        acc = dict(words=0, positions=0, rows=0, kernel_ms=0.0, launches=0, h2d=0, d2h=0, loss=0.0, sync_ms=0.0, syncs=0)
        sync_ms0, syncs0 = dp.sync_ms, dp.syncs
        t0 = time.time()
        for i in range(steps):
            st = dp.step(B)  # train_step + (every sync_every steps) the NCCL replica average (device-timed inside libw2b)
            acc["words"] += st["words"]; acc["positions"] += st["positions"]
            acc["rows"] += st["context_rows"] + st["target_rows"]
            acc["kernel_ms"] += st["kernel_ms"]; acc["launches"] += st["launches"]
            acc.setdefault("per_step", []).append((st["positions"], st["kernel_ms"], st["launches"]))
            acc["h2d"] += st["h2d_bytes"]; acc["d2h"] += st["d2h_bytes"]; acc["loss"] += st["loss"]
        torch.cuda.synchronize()
        if dist:
            dist.barrier()
        torch.cuda.synchronize()
        t1 = time.time()
        acc["sync_ms"], acc["syncs"] = dp.sync_ms - sync_ms0, dp.syncs - syncs0
        dp.finish()  # outside the timed region: leave the replicas averaged, then compare their fingerprints
        acc["replicas_identical"] = dp.replicas_identical()
        acc["wall_s"] = t1 - t0
        acc["alpha"] = st["alpha"]
        acc["last"] = st
        acc["clocks"] = clocks.stop(t0, t1) if clocks else None
        return acc

    def reduce_max(x):
        if not dist:
            return x
        tt = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        return float(tt.item())

    def reduce_sum(x):
        if not dist:
            return x
        tt = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(tt, op=dist.ReduceOp.SUM)
        return float(tt.item())

    # ---- device-resident run: `value`, roofline
    t = make(resident=True)
    a = run(t, args.steps, args.warmup, sampler_index=local if rank == 0 else None)
    t.close()
    if args.dump_outputs and rank == 0:
        def make_probe():  # shard 0's tokens, one shard, same configuration and kernel
            p = w2b.Trainer(None, vocab_size=V + 1, threads=1, init=False, **cfg0)
            p.set_vocab_counts(cn, train_words)
            p.set_corpus(ids[:per_shard], np.zeros(1, np.int64), np.full(1, -1, np.int32), True)
            p.init_tables()
            return p
        dump_outputs(args.dump_outputs, a["last"], make_probe, B)
    if os.environ.get("W2B_BENCH_STEP_LOG") and rank == 0:  # tools/measure_traffic.sh pairs this with ncu's launch list
        with open(os.environ["W2B_BENCH_STEP_LOG"], "w") as f:
            json.dump({"workload": WORKLOAD, "warmup": args.warmup, "per_step": a["per_step"]}, f)
    if os.environ.get("W2B_BENCH_RESIDENT_ONLY"):
        return 0
    # device time of the timed region = kernel events + sync; whole-job rate = all ranks' words / max time
    dev_s = reduce_max(a["kernel_ms"] / 1e3 + a["sync_ms"] / 1e3)
    wall_s = reduce_max(a["wall_s"])
    words = reduce_sum(a["words"])
    positions = reduce_sum(a["positions"])
    value = words / dev_s
    alg_bytes = 2.0 * 4.0 * D * a["rows"]
    kern_s = a["kernel_ms"] / 1e3
    achieved = alg_bytes / kern_s / 1e9
    peak, peak_src = measured_peak()
    tpp = ncu_traffic_per_position()
    roof = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
            "traffic": (tpp * a["positions"] / max(a["launches"], 1)) if tpp else None,
            "peak_source": peak_src,
            "kernel": "train_warp_kernel<%d,%d> (one launch per step, one 32-thread CTA per shard)" % (
                BITS if BITS in (0, 1, 2) else 9, (D // 4 + 31) // 32),
            "algorithmic_bytes_per_launch": alg_bytes / max(a["launches"], 1),
            "kernel_ms_per_launch": a["kernel_ms"] / max(a["launches"], 1),
            "bytes_per_position": alg_bytes / max(a["positions"], 1)}

    gpu_name = torch.cuda.get_device_name(local)

    # ---- end-to-end run: host token buffers, H2D slices + D2H shard state inside every step
    t = make(resident=False)
    e = run(t, args.steps, args.warmup)
    t.close()
    e_wall = reduce_max(e["wall_s"])
    e_words = reduce_sum(e["words"])
    e2e = {"value": e_words / e_wall, "unit": "words/s", "h2d_bytes_per_step": int(e["h2d"] / args.steps),
           "d2h_bytes_per_step": int(e["d2h"] / args.steps), "kernel_ms_per_step": e["kernel_ms"] / args.steps,
           "wall_ms_per_step": e_wall / args.steps * 1e3}

    out = {"metric": METRIC, "value": value, "unit": "words/s", "n_gpus": world, "steps": args.steps,
           "warmup": args.warmup, "ms_per_step": dev_s / args.steps * 1e3, "higher_is_better": True,
           "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
           "config": {"workload": WORKLOAD_TEXT + ", 1x%s" % gpu_name if world == 1 else
                      WORKLOAD_TEXT + ", %dx%s data-parallel (one corpus block per GPU)" % (world, gpu_name),
                      "vocab": V, "size": D, "window": WINDOW, "negative": NEG, "bitlevel": BITS, "sample": SAMPLE,
                      "shards_per_gpu": S_local, "words_per_shard_per_step": B,
                      "l2": "inputs larger than L2: 2 x %.2f GB embedding tables + 400 MB unigram table per GPU, rows drawn at random" % ((V + 1) * D * 4 / 1e9),
                      "parallelism": "dp%d, replica all-reduce-average of u and v every %d steps (NCCL)" % (world, args.sync_every) if world > 1 else "single GPU, %d concurrent shards (one warp each)" % S_local},
           "positions_per_s": positions / dev_s, "wall_ms_per_step": wall_s / args.steps * 1e3,
           "sync_ms_per_step": a["sync_ms"] / args.steps,
           "sync": None if world == 1 else {
               "every_steps": args.sync_every, "mode": args.sync_mode, "syncs_timed": a["syncs"],
               "ms_per_sync": a["sync_ms"] / max(a["syncs"], 1),
               "bytes_per_sync": 2 * (V + 1) * D * 4,
               "allreduce_bus_gbs": (2.0 * (world - 1) / world) * (2 * (V + 1) * D * 4) / 1e9 / max(a["sync_ms"] / max(a["syncs"], 1) / 1e3, 1e-9),
               "what": "one NCCL group: ncclAllReduce(%s) of u and of v in place + the exact global word counter, on the training stream (device time incl. waiting for the slowest rank)" % (
                   "sum of each rank's updates since the last exchange, added to the common base" if args.sync_mode == "sum" else "avg"),
               "sync_check": {"replicas_bit_identical_after_sync": bool(a["replicas_identical"])}},
           "roofline": roof, "e2e": e2e, "clocks": a["clocks"], "gpu_launches": int(a["launches"]),
           "mean_loss_per_position": a["loss"] / max(a["positions"], 1)}
    if rank == 0:
        if world == 1 and not args.no_cpu_baseline:
            try:
                out["cpu_baseline"] = cpu_baseline_leg()
            except Exception as ex:  # the baseline is reported, never required for the GPU number
                out["cpu_baseline"] = {"value": None, "unit": "words/s", "cores": os.cpu_count(), "kind": "reference",
                                       "sample": "failed: %r" % (ex,)}
        print(json.dumps(out), flush=True)
    if dist:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
