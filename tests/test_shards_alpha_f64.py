"""Many-shard training steps in which the shared learning rate moves, element by element, against a float64 Hogwild
replay at the alphas the shards really trained with.

tests/test_shards_f64.py checks steps in which no shard crosses a 10 000-word period.  Here every shard crosses once,
in the middle of the checked sentence, and w2b_train_step_traced records, per shard, every window draw of the real
step with the alpha its position trained at.  Each case checks:
  * the draws (centre, b, cw, targets) of a seeded sample of shards equal the draws-only w2b_trace;
  * the alphas are admissible (tests/alpha_protocol.py): every value is the alpha before the step or f(a value the
    counter can have held); under the warp kernel a sentence trains at one alpha until the shard's own crossing and at
    f(its own counter value) after it, and the crossings took every counter slot exactly once; the counter after the
    step is the one before plus every crossing and end-of-shard add;
  * the tables and the loss lie inside the Hogwild replay at the recorded alphas (ManyShards), and leaving a shard out
    fails it;
  * controls that must fail: the replay at the alpha before the step, and one sentence's alpha moved by one counter
    slot, each for 8 shards.
On the CPU a seeded executor of the counter protocol passes the checker under both kernels' semantics and each wrong
version of the protocol fails it; the warp kernel's own source, emulated, trains several shards one after another and
its records equal the sequential protocol exactly."""
import time
from types import SimpleNamespace

import numpy as np
import pytest

from tests.alpha_protocol import Executor, Sentences, ShardClock, check_alphas, f_alpha, plan_step
from tests.f64_bounds import quantizer
from tests.test_shards_f64 import ManyShards, dense_inputs, seeded_rows
from tests.test_trajectory_f64 import check_step, model_for, sentence_positions, split_sentences

A0 = 0.05


# ------------------------------------------------------------------------------------------------ inputs
def crossing_inputs(S, V, F, L, nsent):
    """Shard s: F/2 one-word filler sentences (nothing trained), then `nsent` L-word sentences of its own ids."""
    filler = np.tile(np.array([1, 0], np.int32), F // 2)
    regions = []
    for s in range(S):
        ids = (2 + (s * nsent + np.arange(nsent))[:, None] * L + np.arange(L)[None, :]).astype(np.int32)
        own = np.concatenate([ids, np.zeros((nsent, 1), np.int32)], 1).ravel()
        regions.append(np.concatenate([filler, own]))
    start = np.cumsum([0] + [len(r) for r in regions[:-1]]).astype(np.int64)
    tail = np.tile(np.array([V - 1, 0], np.int32), 8)  # the last shard never meets the end of the corpus
    return np.concatenate(regions + [tail]), start, np.full(V, 1000, np.int64)


def advance(sents, clocks, budget, limit, lens=None):
    return [plan_step(sents, c, budget, limit, None if lens is None else lens[s]) for s, c in enumerate(clocks)]


# ------------------------------------------------------------------------------------------------ the CPU: checker
def cpu_plans(S=12, F=9998, L=3, nsent=4, to_end=False, seed=0):
    """The plans of one step of S shards of crossing_inputs after a warm-up of F words: one sentence each (every shard
    crosses mid-sentence), or with to_end the rest of the shard (a crossing, then an end-of-shard add)."""
    tokens, start, _ = crossing_inputs(S, 10 ** 6, F, L, nsent)
    limit = F + (L + 1) * (nsent - 1)
    clocks = [ShardClock(c) for c in start]
    sents = Sentences(tokens)
    warm = advance(sents, clocks, F, limit)
    assert not any(p["cross"] for p in warm)
    plans = advance(sents, clocks, 0 if to_end else L + 1, limit, [[L] * (nsent - 1 if to_end else 1)] * S)
    return plans, sum(d for p in plans for d, _, _ in p["cross"])


SCENARIOS = {"mid-sentence": {}, "to-the-end": dict(to_end=True)}


@pytest.mark.parametrize("scenario", list(SCENARIOS))
@pytest.mark.parametrize("kernel", ["warp", "register"])
def test_protocol_executor_passes_the_checker(scenario, kernel):
    plans, moved = cpu_plans(**SCENARIOS[scenario])
    assert all(len(p["cross"]) == 1 and p["cross"][0][2] == 1 for p in plans)
    denom = np.float32(moved / 0.3)
    ex = Executor(A0, denom, 0, A0)
    for seed in range(4):
        alphas, W1, g = ex.run(plans, kernel, seed)
        res = check_alphas(plans, alphas, A0, denom, 0, A0, W1, g, kernel)
        assert res["crossings"] == len(plans) and (kernel == "register" or res["slots"] == len(plans)), res
        assert res["ends"] == (len(plans) if scenario == "to-the-end" else 0)


FAULTS = [("pre_add", "warp"), ("twice", "warp"), ("lost", "warp"), ("late", "warp"),
          ("no_floor", "warp"), ("no_floor", "register"), ("no_end_add", "warp"), ("register_as_warp", "warp")]


@pytest.mark.parametrize("fault,kernel", FAULTS, ids=["%s-%s" % f for f in FAULTS])
def test_protocol_faults_fail_the_checker(fault, kernel):
    """Alpha from the counter before the add, a slot taken twice or lost, the own alpha one position late, the floor
    skipped, the end-of-shard add missing, register-kernel records judged as the warp kernel's: each fails."""
    plans, moved = cpu_plans(to_end=fault == "no_end_add")
    denom = np.float32(moved / 0.3)
    W0, alpha0 = 0, np.float32(A0)
    if fault == "no_floor":  # the counter starts near the end: every crossing drives f below the floor
        W0 = int(float(denom) * (1 - 1.5e-4))
        alpha0 = f_alpha(W0, A0, denom)
    ex = Executor(A0, denom, W0, alpha0)
    run_as = "register" if fault == "register_as_warp" else kernel
    for seed in range(3):
        alphas, W1, g = ex.run(plans, run_as, seed, fault=None if fault == "register_as_warp" else fault)
        with pytest.raises(AssertionError) as e:
            check_alphas(plans, alphas, A0, denom, W0, alpha0, W1, g, kernel)
        print(fault, kernel, seed, str(e.value)[:160])


def test_floor_is_compared_in_double():
    """Where the float32 alpha is below starting_alpha * 1e-4 only in double, the floor applies."""
    a0, denom = np.float32(0.05), np.float32(1e6)
    floor32 = np.float32(float(a0) * 1e-4)
    Ws = np.arange(999_800, 1_000_000, dtype=np.int64)
    got = f_alpha(Ws, a0, denom)
    raw = (a0 * (np.float32(1) - Ws.astype(np.float32) / denom)).astype(np.float32)
    want = np.where(raw.astype(np.float64) < float(a0) * 1e-4, floor32, raw)
    assert np.array_equal(got, want) and (got == floor32).any() and (got > floor32).any()
    # a float32 comparison against the rounded floor keeps the values between the two
    between = (raw.astype(np.float64) < float(a0) * 1e-4) & (raw >= floor32)
    assert not between.any() or (got[between] == floor32).all()


def test_emulated_shards_in_order_equal_the_sequential_protocol():
    """The warp kernel's source, emulated: three shards run one after another in one launch, tracing into their own
    regions while they train.  Shard k starts from the counter and alpha shard k - 1 left, so its records' alphas
    equal the protocol run in shard order exactly; the draws equal each shard's draws-only trace."""
    import word2bits_b200 as w2b
    from oracle import pyoracle as po
    from tests.emu import emu
    S, F, L, nsent, W = 3, 9998, 3, 4, 2
    V = 64
    tokens, start, counts = crossing_inputs(S, V, F, L, nsent)
    counts[:] = 1  # nothing is sub-sampled: every sentence keeps its words, so every crossing is inside one
    limit = F + (L + 1) * (nsent - 1)
    corpus = SimpleNamespace(vocab_size=V, counts=counts, train_words=limit * S + 1, tokens=tokens,
                             shards=lambda n: (start, np.full(n, -1, np.int32)))
    table = po.unigram_table(counts)
    rng = np.random.default_rng(4)
    u = rng.uniform(-0.5, 0.5, (V, 32)).astype(np.float32)
    v = rng.uniform(-0.5, 0.5, (V, 32)).astype(np.float32)
    kw = dict(size=32, window=W, negative=2, bitlevel=1, shards=S, iters=3)  # iter 3: the crossings stay above the floor
    out = emu.train_epoch_warp(corpus, table, u, v, trace_cap=8000, trace_train=True, **kw)
    recs = out["traces"]
    assert list(out["trace_n"]) == [len(r) for r in recs] and all(out["done"])
    clocks = [ShardClock(c) for c in start]
    plans = advance(Sentences(tokens), clocks, 0, limit, [[L for _, L, _ in split_sentences(r, W)] for r in recs])
    denom = np.float32(3 * corpus.train_words + 1)
    ex = Executor(A0, denom, 0, A0)
    order = np.concatenate([np.full(n, s) for s, n in enumerate(ex_lengths(ex, plans))])
    want, W1, g = ex.run(plans, "warp", 0, order=order)
    got = [np.array([r[4] for r in rs], np.float32) for rs in recs]
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert out["wca"] == W1 and np.float32(out["alpha"]) == g
    res = check_alphas(plans, got, A0, denom, 0, A0, out["wca"], out["alpha"], "warp")
    assert res["crossings"] == S and res["slots"] == S and res["ends"] == S, res
    for s in range(S):
        draws = emu.train_epoch_warp(corpus, table, u.copy(), v.copy(), trace_shard=s, trace_cap=8000, **kw)["trace"]
        assert [r[:4] for r in draws] == [r[:4] for r in recs[s]], s
    print("emulated: %d shards, alphas %s, counter %d" % (S, sorted({float(a) for x in got for a in x}), W1))


def ex_lengths(ex, plans):
    """Actions per shard of Executor.run (a crossing, a sentence start, a record or an end add each)."""
    return [p["n"] + len(p["starts"]) + len(p["cross"]) + (p["end"] is not None) for p in plans]


# ------------------------------------------------------------------------------------------------------ the GPU
F_SPARSE = 9998  # filler words: the checked 2-word sentence (3 words) takes a shard to 10 001 > 10 000

GPU_CASES = {
    "bench": dict(D=800, W=10, N=24, b=1, reg=0.0, expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=1584),
    "bench-streamed": dict(D=800, W=10, N=24, b=1, reg=0.0, resident=False,
                           expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=1584),
    "bench-reg": dict(D=800, W=10, N=24, b=1, reg=0.002, expect={"warp": 1, "nj": 7, "minb": 8, "reg": 1}),
    "register-tuned": dict(D=512, W=5, N=8, b=1, reg=0.0, kernel=1,
                           expect={"warp": 0, "wide": 0, "vec": 4, "group": 9}),
    "epoch-end": dict(D=128, W=5, N=8, b=1, reg=0.0, threads=264, kind="end", iter=2, expect={"warp": 1}),
    "floor": dict(D=256, W=5, N=8, b=1, reg=0.0, threads=264, kind="floor", expect={"warp": 1}),
    # bit level 1: without quantization the fixed point of the dense corpus does not settle (DESIGN.md, L1 many shards)
    "dense": dict(corpus="dense", D=400, W=10, N=24, b=1, reg=0.0, threads=132, iter=4, expect={"warp": 1}),
}


def positions_of(recs, W):
    """(ctx, targets, alpha) of every trained record, and the records of each sentence."""
    pos, lens = [], []
    for first, L, sen in split_sentences(recs, W):
        pos += sentence_positions(recs, first, L, sen, W)
        lens.append(L)
    assert sum(lens) == len(recs), "the step's trace ends inside a sentence"
    return pos, lens


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_CASES))
def test_crossing_step_within_hogwild_f64_bounds(name):
    w2b = pytest.importorskip("word2bits_b200")
    t_start = time.time()
    cfg = GPU_CASES[name]
    D, W, N, b, reg = cfg["D"], cfg["W"], cfg["N"], cfg["b"], cfg["reg"]
    iters = cfg.get("iter", 1)
    kind = cfg.get("kind", "cross")
    kw = dict(size=D, window=W, negative=N, bitlevel=b, reg=reg, iter=iters, kernel=cfg.get("kernel", 0))
    dense = cfg.get("corpus") == "dense"
    V = 5000 if dense else 2_000_001
    S = cfg.get("threads")
    if S is None:
        probe = w2b.Trainer(None, vocab_size=V, threads=None, init=False, **kw)
        S = probe.threads
        probe.close()
    if "shards" in cfg:
        assert S == cfg["shards"], (S, cfg["shards"])
    if dense:  # 769 sentences of 13 words = 9997 words, then the checked sentence crosses
        warm, step = 769 * 13, 13
        tokens, start, counts, dense_words = dense_inputs(S, 777)
        delta = warm + step
    else:
        L = 2
        warm, step = F_SPARSE, L + 1
        tokens, start, counts = crossing_inputs(S, V, F_SPARSE, L, 5)
        delta = warm + step
    if kind == "end":  # the first own sentence crosses in the warm-up; three more sentences, then the end
        warm = F_SPARSE + 3
        limit = F_SPARSE + 12
        train_words = limit * S + S // 2
    elif dense:  # sub-sampled as in tests/test_shards_f64.py (its fixed point settles there); iter 4: alpha moves 25 %
        train_words = dense_words
    else:  # the step moves alpha by about 30 %
        train_words = int(S * delta / 0.3 / iters)
    limit = train_words // S
    denom = np.float32(iters * train_words + 1)
    resident = cfg.get("resident", True)

    def make(res):
        t = w2b.Trainer(None, vocab_size=V, threads=S, init=False, **kw)
        t.set_vocab_counts(counts, train_words)
        t.set_corpus(tokens, start, np.full(S, -1, np.int32), res)
        return t

    rng = np.random.default_rng(17)
    sample = sorted(rng.choice(S, 8, replace=False).tolist())
    t = make(True)
    draws = {s: t.trace(s, cap=20000, max_iterations=20000) for s in sample}
    if not resident:
        t.close()
        t = make(False)
    info = t.kernel_info()
    got = dict(info, **{k: v for k, v in w2b.warp_plan(size=D, window=W, negative=N, bitlevel=b, reg=reg,
                                                        kernel=kw["kernel"]).items() if k == "sentence_in_smem"})
    assert all(got[k] == v for k, v in cfg["expect"].items()), (cfg["expect"], got)
    kernel = "warp" if info["warp"] else "register"
    t.init_tables()
    clocks = [ShardClock(c) for c in start]
    st, warm_recs, warm_n = t.train_step_traced(warm, 8)
    sents = Sentences(tokens)
    advance(sents, clocks, warm, limit)
    assert st["words"] == S * warm and st["shards_done"] == 0, st
    if kind == "floor":  # W0 near the end: f(W0) is 1.5 x the floor, every crossing drives it below
        W0 = int(float(denom) * (1 - 1.5e-4))
        t.set_state(float(f_alpha(W0, A0, denom)), W0)
    u0, v0 = t.download_raw()
    alpha_before, W0 = t.get_state()
    W0 = int(W0)

    # rows the step touches get seeded values, so that f covers the expTable range
    budget = 0 if kind == "end" else step
    if not dense:
        ids = np.concatenate([np.arange(2 + s * 10, 2 + s * 10 + 10) for s in range(S)])
        su, sv = seeded_rows(len(ids), D, 11, cw=1)
        u0[ids], v0[ids] = su, sv
        t.upload_raw(u0, v0)
    t0 = time.time()
    st, recs, ns = t.train_step_traced(budget, 64)
    t_gpu = time.time() - t0
    u1, v1 = t.download_raw()
    exptab = t.download_exptable()
    assert ns == [len(r) for r in recs], "a shard made more records than the cap"
    pos, lens = zip(*[positions_of(r, W) for r in recs])
    plans = advance(sents, clocks, budget, limit, lens)
    alphas = [np.array([r[4] for r in rs], np.float32) for rs in recs]
    res = check_alphas(plans, alphas, A0, denom, W0, alpha_before, st["word_count_actual"], st["alpha"], kernel)
    assert st["positions"] == sum(len(p) for p in pos) and st["words"] == sum(c.wc for c in clocks) - S * warm, st
    assert st["context_rows"] == sum(len(c) for p in pos for c, _, _ in p), st
    assert st["target_rows"] == sum(len(g) for p in pos for _, g, _ in p), st
    if kind == "end":
        assert st["shards_done"] == S and res["crossings"] == 0 and res["ends"] == S, (st, res)
        assert all(len(p) == 3 * 2 for p in pos), "the sentence read past the limit was trained"
    else:
        assert st["shards_done"] == 0 and res["crossings"] == S, (st, res)
        if kind == "floor":
            floor = np.float32(float(np.float32(A0)) * 1e-4)
            assert all((a[1:] == floor).all() for a in alphas), "a position after a crossing trained above the floor"
        elif kernel == "warp":  # every crossing inside a sentence gives its slot back
            mid = sum(m for p in plans for _, _, m in p["cross"])
            assert res["slots"] == mid and (dense or mid == S), res
    # draws of the sample equal the draws-only trace (the step's records follow the warm-up's)
    for s in sample:
        k0 = warm_n[s]
        assert [r[:4] for r in recs[s]] == [r[:4] for r in draws[s][k0:k0 + len(recs[s])]], s

    q = quantizer(b, info["warp"] == 1 and not reg and b in (1, 2) and info["bm"] != 9)
    args = (b, q, reg, exptab, model_for(info))
    chk = ManyShards(u0, v0, list(pos), *args)
    res_r = chk.check(u1, v1, st["loss"])
    assert res_r is not None, "unresolved"
    pick, passed = chk.leave_one_out(st["loss"])
    assert len(pick) >= 8 and not passed, ("shards whose removal passes", passed)

    # controls: the replay at the alpha before the step, and one sentence moved by one counter slot
    ctl = [s for s in chk.isolated if any(a != np.float32(alpha_before) for _, _, a in pos[s])]
    ctl = [int(x) for x in rng.choice(ctl, min(8, len(ctl)), replace=False)]
    slot = delta if kind != "end" else 12

    def shifted(p):
        out = []
        for c, g, a in p:
            w = np.int64(round((1 - float(a) / A0) * float(denom)))
            out.append((c, g, f_alpha(w + slot, A0, denom) if a != np.float32(alpha_before) else a))
        return out

    fails = {"pre-step": 0, "slot": 0}
    if not ctl and kind != "end":  # no isolated shard (dense): the whole step at the alpha before it
        ctl = [-1]
        try:
            ManyShards(u0, v0, [[(c, g, np.float32(alpha_before)) for c, g, _ in p] for p in pos], *args).check(
                u1, v1, st["loss"])
        except AssertionError:
            fails["pre-step"] = fails["slot"] = 1
    for s in ctl:
        for name_c, p in (("pre-step", [(c, g, np.float32(alpha_before)) for c, g, _ in pos[s]]),
                          ("slot", shifted(pos[s]))):
            try:
                check_step(u0, v0, u1, v1, None, p, *args)
            except AssertionError:
                fails[name_c] += 1
    elapsed = time.time() - t_start
    print("%s %s: %d shards, %d crossings, %d slots, %d floored, %d end adds; alpha %.6g .. %.6g (before %.6g); "
          "%d sentence starts read another shard's alpha; worst err/bound u %.3f v %.3f loss %.3f; median "
          "|update|/radius isolated %s, component %s; %d passes; %d/%d left out fail; controls failing: pre-step %d/%d, "
          "slot %d/%d; step %.2f s, case %.0f s" % (
              name, info, S, res["crossings"], res["slots"], res["floored"], res["ends"], res["alpha_min"],
              res["alpha_max"], alpha_before, res["foreign"], res_r["u"], res_r["v"], res_r["loss"],
              "%.3g" % res_r["median_iso"] if res_r["median_iso"] is not None else "-",
              "%.3g" % res_r["median_comp"] if res_r["median_comp"] is not None else "-", res_r["passes"],
              len(pick) - len(passed), len(pick), fails["pre-step"], len(ctl), fails["slot"], len(ctl), t_gpu,
              elapsed))
    if kind != "end":
        assert len(ctl) >= 8 or dense, ctl
        assert fails["pre-step"] == len(ctl), fails
        assert kind == "floor" or fails["slot"] == len(ctl), fails  # below the floor a slot changes nothing
    if kind not in ("floor",) and chk.isolated:
        assert res_r["median_iso"] >= 1e3, res_r
    if kind == "end":  # epoch 2 starts where epoch 1 started, at the carried alpha
        alpha_c, wca_c = t.get_state()
        t.epoch_begin()
        st2, recs2, _ = t.train_step_traced(6, 8)
        assert t.get_state()[1] == wca_c
        for s in range(S):
            assert [r[:4] for r in recs2[s]] == [r[:4] for r in warm_recs[s][:len(recs2[s])]], s
            assert all(r[4] == np.float32(alpha_c) for r in recs2[s]), s
        assert np.float32(alpha_c) != np.float32(A0)
    t.close()
    assert elapsed < 300
