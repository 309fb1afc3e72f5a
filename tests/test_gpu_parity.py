"""GPU parity tests (need an H100): the CUDA path through the C ABI vs the CPU oracle and the reference.

Levels follow SURVEY §8(c): L0 bit-exact integer/functional pieces, L1 single step
(fp tolerance), L2 strict-mode trajectories (bit-exact against the sequential-IEEE
oracle), L3 statistical end-to-end for the production (fast, Hogwild) kernel."""
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.util import bits, reference_outputs, zipf_corpus

pytestmark = pytest.mark.gpu

w2b = pytest.importorskip("word2bits_b200")
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_CORPUS = os.path.join(G, "golden_corpus.txt")


@pytest.fixture(scope="module")
def small(tmp_path_factory):
    d = tmp_path_factory.mktemp("c")
    return zipf_corpus(str(d / "small.txt"), 12500, 30, seed=1, newline_every=15)


@pytest.fixture(scope="module")
def medium(tmp_path_factory):
    d = tmp_path_factory.mktemp("c")
    return zipf_corpus(str(d / "medium.txt"), 60000, 3000, seed=2)


@pytest.fixture(scope="module")
def large(tmp_path_factory):
    d = tmp_path_factory.mktemp("c")
    return zipf_corpus(str(d / "large.txt"), 400000, 5000, seed=3)


# ------------------------------------------------------------------------------------ L0
def test_quantize_bits(small):
    c = w2b.Corpus(small, 1)
    t = w2b.Trainer(c, size=8, window=3, negative=4, threads=1, init=False)
    xs = np.concatenate([
        np.array([0.0, -0.0, 1e-30, -1e-30, .25, .5, np.nextafter(np.float32(.5), np.float32(1)), .75, 1.0, -1.0,
                  3.7, -3.7, 1 / 32, .0624, .0625, .09375, .49999, -.5, -.50001, .124, .126], np.float32),
        np.random.default_rng(0).uniform(-1.5, 1.5, 4000).astype(np.float32)])
    for b in range(0, 9):
        got = t.quantize(xs, b)
        want = po.quantize(xs, b)
        assert np.array_equal(bits(got), bits(want)), b
    assert bits(t.quantize(np.array([0.7, -0.7, -0.0], np.float32), 1)).tolist() == [0x3EAAAAAB, 0xBEAAAAAB, 0x3EAAAAAB]


def test_tables_bit_exact(medium):
    c = w2b.Corpus(medium, 5)
    o = po.Corpus(medium, 5)
    assert c.words() == o.words() and np.array_equal(c.counts, o.counts)
    t = w2b.Trainer(c, size=20, window=5, negative=6, threads=3)
    u, v = t.download_raw()
    ou, ov = po.init_net(o.vocab_size, 20)
    assert np.array_equal(bits(u), bits(ou)) and np.array_equal(bits(v), bits(ov))
    assert np.array_equal(bits(t.download_exptable()), bits(po.exptable()))
    assert np.array_equal(t.download_table(), po.unigram_table(o.counts))


@pytest.mark.parametrize("cfg", [
    ("small", 1, 3, 4, 1e-3, 3), ("small", 1, 5, 6, 1e-2, 2), ("small", 1, 3, 4, 0.0, 1),
    ("medium", 5, 5, 6, 1e-3, 4), ("medium", 1, 8, 24, 1e-4, 7), ("medium", 5, 10, 40, 1e-3, 2),
])
@pytest.mark.parametrize("kernel", [0, 1])
def test_draw_trace_bit_exact(cfg, kernel, small, medium):
    """kernel=0: the production (warp-per-shard) kernel's sampling code (jump-ahead + prefetched table lookups);
    kernel=1: the register kernel's inline sampler.  Both must replay the oracle's draws exactly."""
    name, mc, W, neg, sample, shards = cfg
    path = {"small": small, "medium": medium}[name]
    c = w2b.Corpus(path, mc)
    o = po.Corpus(path, mc)
    t = w2b.Trainer(c, size=8, window=W, negative=neg, bitlevel=1, sample=sample, threads=shards, kernel=kernel)
    table = po.unigram_table(o.counts)
    for sid in range(shards):
        m = po.OracleModel(o, 8, W, neg, 1, shards=shards, sample=sample, table=table)
        _, want = m.train_shard(sid, trace_cap=200000)
        got = t.trace(sid, cap=200000)
        assert len(got) == len(want) and len(got) > 0
        for a, b in zip(got, want):
            assert a[:4] == b[:4], (sid, a, b)


# ------------------------------------------------------------------------------------ L1
@pytest.mark.parametrize("b,D,reg", [(1, 200, 0.0), (2, 400, 0.0), (0, 400, 0.0), (5, 100, 0.0), (1, 800, 0.0),
                                      (0, 800, 0.0), (2, 800, 0.0), (0, 200, 0.0), (2, 200, 0.0), (1, 400, 0.0),
                                      (1, 1024, 0.0), (1, 4, 0.0), (1, 50, 0.0), (2, 64, 0.01), (1, 1200, 0.0), (0, 2048, 0.0),
                                      (1, 150, 0.005)])
def test_single_step(b, D, reg, medium):
    """L1: one explicit position through the kernel that trains this configuration — w2b_apply_position launches the
    production (warp-per-shard) kernel itself for every D % 4 == 0, reg == 0 case (the BASELINE shapes D = 800 / 400 /
    200 at bitlevel 0 / 1 / 2 among them), the register kernel for D = 50 and reg != 0."""
    c = w2b.Corpus(medium, 5)
    o = po.Corpus(medium, 5)
    V = c.vocab_size
    rng = np.random.default_rng(7)
    t = w2b.Trainer(c, size=D, window=5, negative=24, bitlevel=b, reg=reg, threads=1)
    m = po.OracleModel(o, D, 5, 24, b, reg=reg, table=np.zeros(1, np.int32))
    for trial in range(4):
        cw = int(rng.integers(1, 11))
        ctx = rng.integers(1, V, cw).astype(np.int32)
        tg = rng.choice(np.arange(1, V), 25, replace=False).astype(np.int32)
        f_gpu = t.apply_position(ctx, tg)
        f_cpu, _ = m.apply_position(ctx, tg)
        # f within 1e-5 relative (reduction order only; twice that beyond 1024 terms per dot product)
        k = max(1, D // 1024)
        assert np.allclose(f_gpu, f_cpu, rtol=k * 1e-5, atol=k * 1e-6)
        u, v = t.download_raw()
        touched_v = np.zeros(V, bool); touched_v[tg] = True
        touched_u = np.zeros(V, bool); touched_u[ctx] = True
        assert np.array_equal(bits(u[~touched_u]), bits(m.u[~touched_u]))
        assert np.array_equal(bits(v[~touched_v]), bits(m.v[~touched_v]))
        # SURVEY L1 bar: 1e-6 abs / 1e-5 rel, or one expTable slot (0.0031*alpha) propagated
        slack = 0.0031 * 0.05 * 25
        assert np.max(np.abs(v - m.v)) <= 1e-6 + slack * 0.4
        assert np.max(np.abs(u - m.u)) <= 1e-6 + slack
        t.upload_raw(m.u, m.v)  # keep both sides on the same trajectory


# ------------------------------------------------------------------------------------ L2
STRICT_CASES = [
    ("small", 8, 3, 4, 1, 1, 1, 1e-3, 0.0, 1),
    ("small", 8, 3, 4, 2, 2, 1, 1e-3, 0.0, 1),
    ("small", 8, 3, 4, 0, 1, 1, 1e-3, 0.0, 2),
    ("small", 8, 3, 4, 5, 3, 2, 1e-2, 0.0, 1),
    ("small", 8, 3, 4, 3, 1, 1, 1e-3, 0.0, 1),
    ("small", 8, 3, 4, 1, 2, 1, 1e-3, 0.01, 1),
    ("small", 10, 3, 4, 1, 2, 1, 1e-3, 0.0, 1),   # D % 4 != 0 -> scalar-column kernel
    ("medium", 20, 5, 6, 1, 4, 5, 1e-3, 0.0, 2),
    ("medium", 200, 8, 24, 1, 2, 5, 1e-3, 0.0, 1),
    ("medium", 100, 5, 12, 2, 3, 5, 1e-4, 0.0, 1),
]


@pytest.mark.parametrize("case", STRICT_CASES)
def test_strict_trajectory_bit_exact(case, small, medium):
    name, D, W, neg, b, shards, mc, sample, reg, iters = case
    path = {"small": small, "medium": medium}[name]
    c = w2b.Corpus(path, mc)
    o = po.Corpus(path, mc)
    t = w2b.Trainer(c, size=D, window=W, negative=neg, bitlevel=b, sample=sample, reg=reg, iter=iters,
                    threads=shards, mode=w2b.MODE_STRICT)
    m = po.OracleModel(o, D, W, neg, b, shards=shards, iters=iters, sample=sample, reg=reg)
    for _ in range(iters):
        lo = sum(m.train_shard(s) for s in range(shards))
        lg, st = t.train_epoch()
        assert st["shards_done"] == shards
        assert abs(lg - lo) <= 1e-4 * abs(lo) + 1e-3, (lg, lo)
    u, v = t.download_raw()
    assert np.array_equal(bits(v), bits(m.v))
    assert np.array_equal(bits(u), bits(m.u))
    a, wca = t.get_state()
    assert bits(np.float32(a)) == bits(np.float32(m.alpha)) and wca == m.word_count_actual
    assert np.array_equal(bits(t.export()), bits(m.export()))


@pytest.mark.parametrize("k", range(6))
def test_strict_vs_reference_golden(k):
    """Straight against vectors produced by the unmodified reference (tests/golden)."""
    gold = np.load(os.path.join(G, "reference_strict.npz"))
    D, W, neg, b, shards, mc, iters = [int(x) for x in gold["case%d_cfg" % k]]
    sample, reg = [float(x) for x in gold["case%d_fcfg" % k]]
    c = w2b.Corpus(GOLDEN_CORPUS, mc)
    t = w2b.Trainer(c, size=D, window=W, negative=neg, bitlevel=b, sample=sample, reg=reg, iter=iters,
                    threads=shards, mode=w2b.MODE_STRICT)
    for _ in range(iters):
        t.train_epoch()
    u, v = t.download_raw()
    assert np.array_equal(bits(u), bits(gold["case%d_u" % k]))
    assert np.array_equal(bits(v), bits(gold["case%d_v" % k]))
    a, wca = t.get_state()
    assert bits(np.float32(a)) == bits(gold["case%d_alpha" % k]) and wca == int(gold["case%d_wca" % k])


def test_streaming_equals_resident(medium):
    c = w2b.Corpus(medium, 5)
    outs = []
    for resident in (True, False):
        t = w2b.Trainer(c, size=20, window=5, negative=6, bitlevel=1, threads=3, iter=1, mode=w2b.MODE_STRICT,
                        resident=resident)
        t.epoch_begin()
        steps = 0
        while True:
            st = t.train_step(3000)
            steps += 1
            if st["shards_done"] == 3:
                break
            assert steps < 1000
        outs.append(t.download_raw() + (t.get_state(),))
    assert np.array_equal(bits(outs[0][0]), bits(outs[1][0])) and np.array_equal(bits(outs[0][1]), bits(outs[1][1]))
    assert outs[0][2] == outs[1][2]


def test_stepwise_equals_epoch(medium):
    c = w2b.Corpus(medium, 5)
    # one shard: with several, stepping interleaves the shards (a different, equally valid order)
    t1 = w2b.Trainer(c, size=20, window=5, negative=6, bitlevel=2, threads=1, iter=1, mode=w2b.MODE_STRICT)
    l1, s1 = t1.train_epoch()
    t2 = w2b.Trainer(c, size=20, window=5, negative=6, bitlevel=2, threads=1, iter=1, mode=w2b.MODE_STRICT)
    t2.epoch_begin()
    words = pos = 0
    loss = 0.0
    while True:
        st = t2.train_step(2500)
        words += st["words"]; pos += st["positions"]; loss += st["loss"]
        if st["shards_done"] == 1:
            break
    assert words == s1["words"] and pos == s1["positions"] and abs(loss - l1) < 1e-6 * abs(l1)
    for a, b in zip(t1.download_raw(), t2.download_raw()):
        assert np.array_equal(bits(a), bits(b))


# ------------------------------------------------------------------------------------ L3
# kernel 0 = warp-per-shard kernel (production), 1 = register kernel; prefetch=1 = production kernel with rows
# fetched across position boundaries.  All run S shards concurrently (Hogwild), so the comparator is the
# oracle with S concurrent pthreads (the reference's own execution model), not sequential shards.
# Bars (SURVEY 8(c) L3): epoch loss within 1 % (2 % with prefetch at D=800 on this 5k-word vocabulary, where a
# stale context row weighs most); sign agreement at b=1 at least the reference's own run-to-run agreement minus
# 5 points (0.852 -> 0.80 at equal concurrency; 0.70 floor); master weights strongly correlated.
@pytest.mark.parametrize("b,D,neg,group,kernel,prefetch", [
    (1, 200, 24, 0, 0, 0), (2, 100, 12, 0, 0, 0), (0, 100, 24, 0, 0, 0), (1, 800, 24, 0, 0, 0), (5, 64, 5, 0, 0, 0),
    (1, 200, 24, 0, 0, 1), (0, 400, 24, 0, 0, 0), (2, 400, 12, 0, 0, 0), (1, 100, 5, 0, 0, 0), (1, 800, 24, 0, 0, 1),
    (1, 200, 24, 0, 1, 0), (0, 100, 24, 9, 1, 0), (1, 800, 24, 5, 1, 0), (2, 50, 12, 0, 0, 0)])
def test_fast_statistical(b, D, neg, group, kernel, prefetch, large):
    shards = 16
    c = w2b.Corpus(large, 5)
    o = po.Corpus(large, 5)
    t = w2b.Trainer(c, size=D, window=8, negative=neg, bitlevel=b, threads=shards, iter=2, group=group,
                    kernel=kernel, prefetch=prefetch)
    m = po.OracleModel(o, D, 8, neg, b, shards=shards, iters=2)
    words_total = 0
    for ep in range(2):
        lo = m.train_epoch_threads()
        lg, st = t.train_epoch()
        words_total += st["words"]
        assert st["shards_done"] == shards
        assert abs(lg - lo) <= (0.02 if (D >= 800 and prefetch) else 0.01) * abs(lo), (ep, lg, lo)
    a, wca = t.get_state()
    # the device counter is an atomic: exact.  The oracle's 16 threads race on word_count_actual
    # like the reference's do (:380,:415) and may lose increments, never gain any.
    assert wca == words_total and m.word_count_actual <= wca
    out = t.export()
    if b == 1:
        assert set(np.unique(bits(out)).tolist()) <= {0x3EAAAAAB, 0xBEAAAAAB}
    if b == 2:
        assert set(np.unique(np.abs(out)).tolist()) <= {0.25, 0.75}
    u, v = t.download_raw()
    cu = np.corrcoef(u.ravel(), m.u.ravel())[0, 1]
    cv = np.corrcoef(v.ravel(), m.v.ravel())[0, 1]
    agree = np.mean(bits(out) == bits(m.export())) if b == 1 else 1.0
    print("fast-vs-oracle b=%d D=%d kernel=%d prefetch=%d: corr(u)=%.4f corr(v)=%.4f sign agreement=%.4f loss %.1f vs %.1f"
          % (b, D, kernel, prefetch, cu, cv, agree, lg, lo))
    assert cu > 0.75 and cv > 0.90, (cu, cv)
    if b == 1:
        assert agree > 0.70, agree
    if b == 0 and kernel == 0:
        # fp32 tolerance (north_star: "within a stated fp tolerance for bitlevel=0"): relative L2 distance of the master
        # tables to the oracle's, in units of the oracle's own run-to-run distance at the same concurrency (two
        # runs of its 16 Hogwild threads) — the GPU may be at most 2.5 times as far from the oracle as the oracle
        # is from itself
        m2 = po.OracleModel(o, D, 8, neg, b, shards=shards, iters=2)
        for ep in range(2):
            m2.train_epoch_threads()
        rel = lambda x, y: float(np.linalg.norm(x - y) / np.linalg.norm(y))
        base_u, base_v = rel(m2.u, m.u), rel(m2.v, m.v)
        gu, gv = rel(u, m.u), rel(v, m.v)
        print("b=0 D=%d prefetch=%d rel-L2 vs oracle: u %.4f v %.4f; oracle vs oracle: u %.4f v %.4f" % (D, prefetch, gu, gv, base_u, base_v))
        # (+ 0.03 absolute: the oracle's own distance moves between 0.03 and 0.19 from run to run on this corpus)
        assert gu <= 2.5 * base_u + 0.03 and gv <= 2.5 * base_v + 0.03, (gu, gv, base_u, base_v)


@pytest.mark.parametrize("kernel", [0, 1])
def test_fast_counters_match_oracle(kernel, large):
    shards = 8
    c = w2b.Corpus(large, 5)
    o = po.Corpus(large, 5)
    t = w2b.Trainer(c, size=64, window=10, negative=24, bitlevel=1, threads=shards, iter=1, kernel=kernel)
    _, st = t.train_epoch()
    table = po.unigram_table(o.counts)
    pos = ctx = tgt = 0
    for s in range(shards):
        m = po.OracleModel(o, 4, 10, 24, 1, shards=shards, table=table)
        _, tr = m.train_shard(s, trace_cap=400000)
        for r in tr:
            if r[2] > 0:
                pos += 1; ctx += r[2]; tgt += len(r[3])
    assert (st["positions"], st["context_rows"], st["target_rows"]) == (pos, ctx, tgt)
    assert st["shards_done"] == shards


def test_fast_streaming_and_steps(large):
    """Production kernel driven step by step from host slices (the e2e path, double-buffered: the next
    step's slices are gathered and uploaded while the current one runs): every shard ends, counters equal the
    resident run's — also when the step size changes between calls (prefetched slices no longer fit)."""
    c = w2b.Corpus(large, 5)
    tot = []
    for resident in (True, False):
        t = w2b.Trainer(c, size=128, window=5, negative=12, bitlevel=1, threads=12, iter=1, resident=resident)
        t.epoch_begin()
        words = pos = 0
        for k in range(10000):
            st = t.train_step(5000 if k % 7 else 1200)
            words += st["words"]; pos += st["positions"]
            if st["shards_done"] == 12:
                break
        assert st["shards_done"] == 12
        tot.append((words, pos))
    assert tot[0] == tot[1]


def test_set_corpus_validates_and_can_be_repeated(medium):
    """The kernels use token ids as row indices and shard starts as stream offsets: w2b_set_corpus refuses ids outside
    the vocabulary and starts outside the stream (W2B_EINVAL, nothing uploaded).  Switching a context between
    resident and streaming corpora, and setting a streaming corpus twice, keeps working (the staging buffers of the
    previous stream are not reused blindly)."""
    c = w2b.Corpus(medium, 5)
    S = 4
    t = w2b.Trainer(c, size=32, window=5, negative=6, bitlevel=1, threads=S, iter=1)
    start, first = c.shards(S)
    bad = np.array(c.tokens, np.int32).copy()
    bad[len(bad) // 2] = c.vocab_size
    with pytest.raises(w2b.W2BError, match="token id"):
        t.set_corpus(bad, start, first, True)
    bad[len(bad) // 2] = -3
    with pytest.raises(w2b.W2BError, match="token id"):
        t.set_corpus(bad, start, first, False)
    s2 = np.array(start, np.int64).copy()
    s2[-1] = len(c.tokens) + 5
    with pytest.raises(w2b.W2BError, match="outside the stream"):
        t.set_corpus(c.tokens, s2, first, True)
    totals = []
    for resident in (False, False, True, False):
        t.set_corpus(c.tokens, start, first, resident)
        words = 0
        for _ in range(1000):
            st = t.train_step(3000)
            words += st["words"]
            if st["shards_done"] == S:
                break
        assert st["shards_done"] == S
        totals.append(words)
    assert len(set(totals)) == 1 and totals[0] > 0
    t.close()


@pytest.mark.parametrize("kernel,prefetch", [(1, 0), (0, 0), (0, 1)])
@pytest.mark.parametrize("b,D", [(0, 64), (0, 200), (2, 64), (0, 800), (0, 50)])
def test_fast_single_shard_tracks_oracle(kernel, prefetch, b, D, medium):
    """One shard, positions in order (register kernel; production kernel in its default mode): the
    production arithmetic (FMA, shuffle-tree dot, atomic-add scatter) must stay close to the
    sequential oracle over a whole epoch.  Calibration (SURVEY 8(c) L2): the reference's own
    -O3 vs strict-fp builds differ on this corpus by d0 = 8.7e-5 (D=64) / 3.5e-4 (D=200) at b=0
    and by 0.13 (sign flips) at b=2; the GPU kernels additionally read duplicate targets of one
    group before either update (a within-position Hogwild effect)."""
    c = w2b.Corpus(medium, 5)
    o = po.Corpus(medium, 5)
    t = w2b.Trainer(c, size=D, window=5, negative=6, bitlevel=b, threads=1, iter=1, kernel=kernel,
                    prefetch=prefetch)
    m = po.OracleModel(o, D, 5, 6, b, shards=1, iters=1)
    lo = m.train_shard(0)
    lg, st = t.train_epoch()
    u, v = t.download_raw()
    du, dv = np.max(np.abs(u - m.u)), np.max(np.abs(v - m.v))
    fu, fv = np.mean(np.abs(u - m.u) < 1e-3), np.mean(np.abs(v - m.v) < 1e-3)
    print("single-shard kernel=%d b=%d D=%d: max|du|=%.3g max|dv|=%.3g within1e-3: %.4f %.4f loss %.3f vs %.3f"
          % (kernel, b, D, du, dv, fu, fv, lg, lo))
    ordered = not prefetch  # prefetch on: context rows are read one update stale
    assert abs(lg - lo) <= (1e-3 if ordered else 5e-3) * abs(lo)
    if b == 0:
        lim = (5e-3 if D <= 200 else 2e-2) if ordered else 1e-1  # D=800: 4x the terms per dot product and update
        assert du < lim and dv < lim, (du, dv)
    else:  # b=2 is chaotic (level flips feed back): the reference's own two builds agree within
        # 1e-3 on only 26 % of the elements here, so hold the trajectories to correlation instead
        cu = np.corrcoef(u.ravel(), m.u.ravel())[0, 1]
        cv = np.corrcoef(v.ravel(), m.v.ravel())[0, 1]
        assert cu > 0.9 and cv > 0.9, (cu, cv)


def test_cli_end_to_end(tmp_path):
    """The drop-in binary: strict mode writes byte-for-byte the file the oracle writes (text and
    binary formats, :560-576); the production mode writes a well-formed 1-bit file."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cli = os.path.join(root, "word2bits_b200", "word2bits")
    o = po.Corpus(GOLDEN_CORPUS, 1)
    for binary in (0, 1):
        out = str(tmp_path / ("strict%d" % binary))
        r = subprocess.run([cli, "-train", GOLDEN_CORPUS, "-output", out, "-size", "16", "-window", "3", "-negative", "4",
                            "-bitlevel", "2", "-threads", "2", "-iter", "2", "-min-count", "1", "-binary", str(binary),
                            "-strict", "1", "-save-every-epoch", "1"], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "Starting epoch: 0" in r.stdout and "Starting epoch: 1" in r.stdout and "Epoch Loss:" in r.stdout
        m = po.OracleModel(o, 16, 3, 4, 2, shards=2, iters=2)
        for ep in range(2):
            for s in range(2):
                m.train_shard(s)
            want = str(tmp_path / "want")
            m.write_vectors(want, binary)
            assert open(out + "_epoch%d" % ep, "rb").read() == open(want, "rb").read()
        assert open(out, "rb").read() == open(want, "rb").read()
    out = str(tmp_path / "fast.bin")
    r = subprocess.run([cli, "-train", GOLDEN_CORPUS, "-output", out, "-size", "32", "-window", "3", "-negative", "4",
                        "-min-count", "1", "-binary", "1", "-iter", "1", "-debug", "0"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(out, "rb").read()
    assert raw.startswith(b"31 32\n</s> ")
    body = raw[len(b"31 32\n</s> "):][: 32 * 4]
    assert set(np.frombuffer(body, np.uint32).tolist()) <= {0x3EAAAAAB, 0xBEAAAAAB}  # README.md:124-131


def DEBUG2_ARGS(train):
    return ["-train", train, "-size", "40", "-window", "5", "-negative", "6", "-bitlevel", "1", "-threads", "4",
            "-iter", "2", "-min-count", "5", "-binary", "1", "-debug", "2"]


def debug2_skeleton(txt):
    """The lines of a `-debug 2` log with every progress line removed and every decimal number replaced by #."""
    import re
    prog = re.compile(r"\rAlpha: \d+\.\d{6}  Progress: \d+\.\d{2}%  Cost: -?\d+\.\d{6} Words/thread/sec: \d+\.\d{2}k  ")
    assert prog.search(txt), txt[:500]
    txt = prog.sub("", txt)
    return [re.sub(r"-?\d+\.\d+", "#", line) for line in txt.split("\n")]


def test_cli_debug2_lines_match_the_reference(tmp_path, medium):
    """A `-debug 2` training run prints what the reference prints (:295-298,:523,:533,:384-387,:539): the fixed lines
    are identical, the progress line has the reference's format and label — anything that parses the reference's
    log parses this one.  (Numbers differ: different machine, Hogwild.)  The reference's log of the same run is
    stored in tests/golden/reference_outputs.json."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([os.path.join(root, "word2bits_b200", "word2bits")] + DEBUG2_ARGS(medium) +
                       ["-output", str(tmp_path / "ours.bin")], capture_output=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    ours = r.stdout.decode("latin1")  # (bytes: the carriage returns must survive)
    want = [line.replace("{train}", medium) for line in reference_outputs("gpu_parity")["cli_debug2_skeleton"]]
    assert want == debug2_skeleton(ours), (want[:8], ours[:800])
    assert "Starting training using file" in ours and ours.count("Epoch Loss: ") == 2


def test_planted_topic_quality(tmp_path):
    """L3 statistical end-to-end (SURVEY Appendix B): on a corpus with planted topics the trained
    1-bit vectors must recover the topics as well as the reference's own (kNN purity within 0.04,
    final epoch loss within 1 %), for the production kernel in its default mode and with its prefetch on."""
    from tests.util import planted_topic_corpus, topic_purity
    topics = 25
    path = planted_topic_corpus(str(tmp_path / "topics.txt"), vocab=5000, topics=topics, sentences=60000, length=20)
    D, W, neg, iters, shards = 100, 5, 12, 2, 16
    c = w2b.Corpus(path, 5)
    o = po.Corpus(path, 5)
    words = c.words()
    # the unmodified reference, 16 concurrent threads (-O3), on the same corpus
    ref = reference_outputs("gpu_parity")["planted_topics"]
    res = {"reference": (ref["final_loss"], ref["purity"])}
    m = po.OracleModel(o, D, W, neg, 1, shards=shards, iters=iters)
    losses = [m.train_epoch_threads() for _ in range(iters)]
    res["oracle"] = (losses[-1], topic_purity(words, m.export(), topics))
    for name, kw in (("warp", dict(kernel=0)), ("warp_prefetch", dict(kernel=0, prefetch=1)), ("register", dict(kernel=1))):
        t = w2b.Trainer(c, size=D, window=W, negative=neg, bitlevel=1, threads=shards, iter=iters, **kw)
        losses = [t.train_epoch()[0] for _ in range(iters)]
        res[name] = (losses[-1], topic_purity(words, t.export(), topics))
        t.close()
    print("planted-topic quality (final-epoch loss, kNN purity):", {k: (round(v[0], 1), round(v[1], 4)) for k, v in res.items()})
    base = res["reference"]
    assert base[1] > 0.5, "corpus too weak to measure anything"
    for name in ("warp", "warp_prefetch", "register"):
        assert abs(res[name][1] - base[1]) <= 0.04, (name, res)   # reference vs oracle differ by 0.011 themselves
        assert abs(res[name][0] - base[0]) <= 0.01 * abs(base[0]), (name, res)


@pytest.mark.parametrize("D,W,neg,b", [(4, 1, 0, 1), (8, 2, 1, 2), (100, 5, 5, 1), (256, 20, 40, 0), (1024, 3, 7, 1),
                                         (300, 10, 63, 2), (800, 10, 24, 1), (64, 30, 12, 1), (12, 5, 3, 4), (800, 10, 63, 1),
                                         (100, 5, 63, 1), (132, 64, 63, 1), (50, 5, 6, 1), (150, 8, 12, 2), (6, 2, 3, 0),
                                         (250, 5, 24, 1), (3, 1, 1, 1), (1200, 5, 12, 1), (1530, 3, 4, 0), (2048, 2, 3, 2),
                                         (64, 200, 10, 1), (32, 512, 63, 1), (800, 300, 24, 1)])
def test_production_kernel_odd_shapes(D, W, neg, b, medium):
    """Production kernel on edge geometries (negative=0, window 1..512 — as wide as a sentence —, D 3..2048 incl. D % 4 != 0 — rows padded to whole
    float4s on the device — and the reference's published 1200 dimensions, > 32 negatives):
    terminates, trains every position the oracle's trace holds, loss within 2 % of the oracle."""
    shards = 6
    c = w2b.Corpus(medium, 5)
    o = po.Corpus(medium, 5)
    t = w2b.Trainer(c, size=D, window=W, negative=neg, bitlevel=b, threads=shards, iter=1)
    lg, st = t.train_epoch()
    assert st["shards_done"] == shards
    table = po.unigram_table(o.counts)
    pos = ctx = tgt = 0
    for s in range(shards):
        m0 = po.OracleModel(o, 4, W, neg, b, shards=shards, table=table)
        _, tr = m0.train_shard(s, trace_cap=200000)
        for r in tr:
            if r[2] > 0:
                pos += 1; ctx += r[2]; tgt += len(r[3])
    assert (st["positions"], st["context_rows"], st["target_rows"]) == (pos, ctx, tgt)
    m = po.OracleModel(o, D, W, neg, b, shards=shards, table=table)
    lo = m.train_epoch_threads()
    # loss: a sanity bar here (the statistical bars live in test_fast_statistical); wide 1-bit rows on
    # this 2k-word vocabulary make concurrent shards collide far more than any real configuration
    tol = 0.05 if D >= 512 else 0.02
    if W <= 64:
        assert abs(lg - lo) <= tol * abs(lo) + 1.0, (D, W, neg, b, lg, lo)
    else:
        # Windows wider than 64: when these cases were last run on a GPU the oracle port still kept a position's context
        # ids in a 130-entry buffer (fixed since; pinned at window 300 by tests/test_oracle_vs_ref.py), so its loss was
        # garbage there and only the counters were compared.  With the fixed oracle the kernel's own source matches
        # it to 1e-4 .. 4e-4 at windows 200 .. 512 on the emulator (tests/test_warp_emulation.py::
        # test_sentence_wide_windows_track_the_oracle) and the oracle's concurrent-vs-sequential spread is 0.4 - 0.7 %;
        # the gap is printed here, the bar stays on the counters until a GPU run has confirmed it.
        print("wide window D=%d W=%d neg=%d: GPU loss %.1f, oracle %.1f (rel. gap %.4f)" % (D, W, neg, lg, lo, abs(lg - lo) / abs(lo)))
    u, v = t.download_raw()
    assert np.isfinite(u).all() and np.isfinite(v).all()


def test_checkpoint_resume_is_exact(tmp_path, medium):
    """SURVEY 8(f).4: fp32 master tables + alpha + word counter on disk; a run resumed from the
    checkpoint after epoch 1 ends bit-identical to an uninterrupted run (strict mode)."""
    c = w2b.Corpus(medium, 5)
    kw = dict(size=22, window=5, negative=6, bitlevel=1, threads=2, iter=2, mode=w2b.MODE_STRICT)  # (22: padded rows)
    a = w2b.Trainer(c, **kw)
    a.train_epoch(); a.train_epoch()
    b = w2b.Trainer(c, **kw)
    b.train_epoch()
    ck = str(tmp_path / "ck.bin")
    b.checkpoint_save(ck, 1)
    b.close()
    r = w2b.Trainer(c, **kw)
    assert r.checkpoint_load(ck) == 1
    r.train_epoch()
    for x, y in zip(a.download_raw(), r.download_raw()):
        assert np.array_equal(bits(x), bits(y))
    assert a.get_state() == r.get_state()
    with pytest.raises(w2b.W2BError):
        w2b.Trainer(c, size=24, window=5, negative=6, threads=2, iter=2).checkpoint_load(ck)  # wrong shape
    for other in (dict(kw, bitlevel=2), dict(kw, iter=3)):  # another bit level / learning-rate schedule is refused
        with pytest.raises(w2b.W2BError, match="was written with"):
            w2b.Trainer(c, **other).checkpoint_load(ck)
    assert not os.path.exists(ck + ".tmp")  # written beside the target, then renamed over it
    open(ck + ".junk", "wb").write(open(ck, "rb").read()[:1000])
    with pytest.raises(w2b.W2BError):
        w2b.Trainer(c, **kw).checkpoint_load(ck + ".junk")  # truncated file


def _analogy_fixture(tmp_path, D=48, pairs=300, sections=8, per_section=120, bits=0, seed=5):
    """Vector file (word2vec binary) with planted a:b offsets + a question file with `sections`
    sections, OOV words, mixed case and a trailing EXIT-less EOF, like questions-words.txt."""
    rng = np.random.default_rng(seed)
    off = rng.normal(size=D).astype(np.float32) * 1.5
    a = rng.normal(size=(pairs, D)).astype(np.float32)
    b = a + off + 1.1 * rng.normal(size=(pairs, D)).astype(np.float32)
    words = ["</s>"] + ["Alpha%d" % i for i in range(pairs)] + ["beta%d" % i for i in range(pairs)] + ["noise%d" % i for i in range(400)]
    vec = np.concatenate([np.zeros((1, D), np.float32) + 0.01, a, b, rng.normal(size=(400, D)).astype(np.float32)])
    if bits:
        vec = po.quantize(vec * 0.3, bits)
    vf = str(tmp_path / "vec.bin")
    with open(vf, "wb") as f:
        f.write(b"%d %d\n" % (len(words), D))
        for w, row in zip(words, vec):
            f.write(w.encode() + b" " + row.astype(np.float32).tobytes() + b"\n")
    qf = str(tmp_path / "questions.txt")
    with open(qf, "w") as f:
        for s in range(sections):
            f.write(": section-%d\n" % s)
            for _ in range(per_section):
                i, j = rng.integers(0, pairs, 2)
                q = ["alpha%d" % i, "BETA%d" % i, "Alpha%d" % j, "beta%d" % j]
                if rng.random() < 0.05:
                    q[rng.integers(0, 4)] = "missingword"
                f.write(" ".join(q) + "\n")
    return vf, qf


@pytest.mark.parametrize("bits,threshold", [(0, 0), (0, 700), (2, 0), (1, 0)])
def test_gpu_analogy_evaluator_matches_reference(tmp_path, bits, threshold):
    """SURVEY 8(f).2: the GPU evaluator prints what src/compute-accuracy.c prints.  fp32 vectors:
    the report is identical text; 1-/2-bit vectors produce exact score ties whose winner depends on
    the summation order even inside the reference, so the counters are held to +-2 %."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    vf, qf = _analogy_fixture(tmp_path, bits=bits)
    want = reference_outputs("gpu_parity")["analogy_%d_%d" % (bits, threshold)]  # src/compute-accuracy.c's report
    got, acc = w2b.compute_accuracy(vf, qf, bitlevel=bits, threshold=threshold)
    cli = subprocess.run([os.path.join(root, "word2bits_b200", "compute_accuracy"), vf, str(bits), str(threshold)],
                         stdin=open(qf), capture_output=True, text=True).stdout
    assert cli == got
    assert acc["questions_total"] == 8 * 120 and acc["questions_seen"] > 0
    if bits == 0:
        assert got == want
        assert acc["correct"] > 0.3 * acc["questions_seen"]   # the planted offsets are recoverable
    else:
        import re
        def nums(txt):
            return [float(x) for x in re.findall(r"[-+]?\d+\.\d+|\d+", txt)]
        gw, gg = nums(want), nums(got)
        assert len(gw) == len(gg) and want.splitlines()[1] == got.splitlines()[1]
        assert want.splitlines()[-1] == got.splitlines()[-1]          # questions seen / total: exact
        total_w = [l for l in want.splitlines() if l.startswith("Total accuracy")][-1]
        total_g = [l for l in got.splitlines() if l.startswith("Total accuracy")][-1]
        assert abs(nums(total_w)[0] - nums(total_g)[0]) <= 2.0, (total_w, total_g)


@pytest.mark.parametrize("D,bits,vocab", [(200, 1, 30000), (72, 0, 9000), (800, 2, 6000), (130, 0, 700)])
def test_evaluator_tensor_core_filter_is_exact(tmp_path, D, bits, vocab):
    """The evaluator scores on the tensor cores (TF32 wgmma fed by TMA) only to FILTER: words whose approximate
    score lies within the proven error bound of the best are re-scored in fp32 in the reference's operation order.
    So its report must equal, character for character, the report of the same pipeline with every score computed
    in fp32 on the SIMT cores (W2B_EVAL_SIMT=1) — on many 256-word tiles, row pitches that need padding (D = 72,
    130), exact-tie-heavy 1-/2-bit vectors, and a vocabulary that is not a multiple of the tile."""
    import subprocess
    rng = np.random.default_rng(D + bits)
    pairs = min(1500, (vocab - 1) // 3)
    off = rng.normal(size=D).astype(np.float32) * 1.5
    a = rng.normal(size=(pairs, D)).astype(np.float32)
    b = a + off + 1.1 * rng.normal(size=(pairs, D)).astype(np.float32)
    noise = rng.normal(size=(vocab - 2 * pairs - 1, D)).astype(np.float32) if vocab > 2 * pairs + 1 else np.zeros((0, D), np.float32)
    vec = np.concatenate([np.zeros((1, D), np.float32) + 0.01, a, b, noise])[:vocab]
    words = (["</s>"] + ["alpha%d" % i for i in range(pairs)] + ["beta%d" % i for i in range(pairs)] +
             ["noise%d" % i for i in range(len(noise))])[:vocab]
    if bits:
        vec = po.quantize(vec * 0.3, bits)
    vf = str(tmp_path / "vec.bin")
    with open(vf, "wb") as f:
        f.write(b"%d %d\n" % (len(words), D))
        for w, row in zip(words, vec):
            f.write(w.encode() + b" " + row.astype(np.float32).tobytes() + b"\n")
    usable = pairs
    qf = str(tmp_path / "questions.txt")
    with open(qf, "w") as f:
        for sec in range(6):
            f.write(": section-%d\n" % sec)
            for _ in range(500):
                i, j = rng.integers(0, usable, 2)
                f.write("alpha%d beta%d alpha%d beta%d\n" % (i, i, j, j))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cli = os.path.join(root, "word2bits_b200", "compute_accuracy")
    out = {}
    for simt in ("0", "1"):
        out[simt] = subprocess.run([cli, vf, str(bits), "0"], stdin=open(qf), capture_output=True, text=True,
                                   env=dict(os.environ, W2B_EVAL_SIMT=simt), timeout=300).stdout
    assert "Questions seen / total: 3000 3000" in out["0"]
    assert out["0"] == out["1"]
    _, acc = w2b.compute_accuracy(vf, qf, bitlevel=bits)
    print("evaluator D=%d bits=%d vocab=%d: %.2f ms, filter let %.1f candidates per question through, %.1f re-scored in fp32"
          % (D, bits, vocab, acc["gpu_ms"], acc["candidates"] / 3000.0, acc["rescored"] / 3000.0))
    assert 3000 <= acc["rescored"] <= acc["candidates"] < 3000 * vocab // 10


def test_full_size_shape_properties(tmp_path):
    """BASELINE configs[1] shape (400k-word Zipf vocabulary, D=800, window 10, negative 24, 132 shards),
    checked through size-independent properties: vocabulary/table/InitNet equal the oracle's on the
    full arrays, the production sampler replays the oracle's draws on a 1e8-slot table over ~300k words,
    every shard ends, the word accounting adds up, and quantize is idempotent on the exported matrix."""
    import bench
    cdf, _ = bench.zipf_cdf(400000)
    ids = bench.synth_ids(FULL_SIZE_CORPUS[0], FULL_SIZE_CORPUS[1], cdf)
    path = bench._write_text(ids, str(tmp_path / "big_"))
    try:
        c = w2b.Corpus(path, 1)
        o = po.Corpus(path, 1)
        V, D, S = c.vocab_size, 800, 132
        assert V > 250000 and c.words() == o.words() and np.array_equal(c.counts, o.counts)
        assert np.array_equal(c.tokens, o.tokens)
        t = w2b.Trainer(c, size=D, window=10, negative=24, bitlevel=1, threads=S, iter=1)
        table = po.unigram_table(o.counts)
        assert np.array_equal(t.download_table(), table)
        u, v = t.download_raw()
        ou, ov = po.init_net(V, D)
        assert np.array_equal(bits(u), bits(ou)) and np.array_equal(bits(v), bits(ov))
        del ou, ov
        for sid in (0, 3, S - 1):                         # first, middle (mid-word seek), last shard
            got = t.trace(sid, max_iterations=1500, cap=2000)
            m = po.OracleModel(o, 4, 10, 24, 1, shards=S, table=table)
            _, want = m.train_shard(sid, max_positions=1500, trace_cap=2000)
            assert len(got) == len(want) == 1500
            assert all(a[:4] == b[:4] for a, b in zip(got, want)), sid
        loss, st = t.train_epoch()
        assert st["shards_done"] == S and np.isfinite(loss)
        # every shard stops after the first sentence that takes it past train_words/S (:414)
        assert st["words"] > c.train_words - S and st["words"] < c.train_words + S * 1300
        assert st["positions"] > 0.7 * st["words"] and st["target_rows"] > 24.9 * st["positions"]
        out = t.export()
        assert set(np.unique(bits(out)).tolist()) <= {0x3EAAAAAB, 0xBEAAAAAB}
        assert np.array_equal(bits(t.quantize(out, 1)), bits(out))       # idempotent
        u2, v2 = t.download_raw()
        assert np.isfinite(u2).all() and np.isfinite(v2).all() and not np.array_equal(bits(v2), bits(v))
    finally:
        os.unlink(path)


# (first epoch, second epoch) bars per shard count.  Stored reference losses: 16 shards = mean of three runs on a
# 16-core host (they agree to 0.1 %); the others one run each on an 8-core host.  Gaps measured on an H100: 16 shards
# 0.15 % / 0.71 %; 132 shards 0.6-0.7 % / 1.1-1.2 %; 148 shards 0.5-0.6 % / 0.7 %; 1584 shards 5.5-5.6 % /
# 0.3-1.3 %; 1776 shards 5.2 % / 1.2-1.4 %.  The GPU runs every shard truly concurrently; the reference's
# pthreads are time-sliced over the host's cores, so beyond the core count the two sides stop being at equal
# concurrency — and on this 3 M-token corpus 1584 shards are 1.6 sentences each, all of them started from the same
# initial weights at the same moment.  The 1 % bar of SURVEY 8(c) L3 is applied where the comparison is like for like
# (16 shards).
L3_BARS = {16: (0.01, 0.01), 132: (0.02, 0.02), 148: (0.02, 0.02), 1584: (0.08, 0.02), 1776: (0.08, 0.02)}
FULL_SIZE_CORPUS = (3_000_000, 99)  # tokens, seed of bench.synth_ids


@pytest.mark.parametrize("S", [16, 132, 148, 1584, 1776])
def test_full_size_shape_loss_tracks_the_reference(S, tmp_path):
    """L3 at the benchmarked shape (SURVEY 8(c)): a 400k-class Zipf vocabulary, D=800, window 10,
    negative 24, bitlevel 1, two epochs — with 16 shards, 132 shards (one per SM of an H100), the 1584 shards the
    bench runs there (132 SMs x 12 warps), and 148 / 1776 shards (the same for a 148-SM GPU).  Comparator: the epoch losses of the unmodified reference (oracle/_ref,
    -O3) with as many pthreads as there are shards on the same corpus (tests/golden/reference_outputs.json)."""
    import bench
    cdf, _ = bench.zipf_cdf(400000)
    ids = bench.synth_ids(FULL_SIZE_CORPUS[0], FULL_SIZE_CORPUS[1], cdf)
    path = bench._write_text(ids, str(tmp_path / "big_"))
    D, W, neg, b, iters = 800, 10, 24, 1, 2
    try:
        want = reference_outputs("full_size")[str(S)]
        lo, V = want["losses"], want["V"]
        c = w2b.Corpus(path, 1)
        assert c.vocab_size == V
        t = w2b.Trainer(c, size=D, window=W, negative=neg, bitlevel=b, threads=S, iter=iters)
        lg = []
        for _ in range(iters):
            loss, st = t.train_epoch()
            assert st["shards_done"] == S
            lg.append(loss)
        t.close()
        gaps = [abs(a - r) / abs(r) for a, r in zip(lg, lo)]
        print("full-size L3, %d shards: GPU epoch losses %s, reference %s, rel. gaps %s"
              % (S, ["%.0f" % x for x in lg], ["%.0f" % x for x in lo], ["%.4f" % g for g in gaps]))
        assert gaps[0] <= L3_BARS[S][0] and gaps[1] <= L3_BARS[S][1], (S, lg, lo)
    finally:
        os.unlink(path)
