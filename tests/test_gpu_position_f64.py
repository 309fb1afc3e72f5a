"""One training position, element by element, against a float64 restatement of :431-503.

Each case trains explicit positions (Trainer.apply_position) and checks every element the position writes against
float64 arithmetic on the same quantized inputs, with bounds from the standard rounding-error accounting: with
u = 2^-24 and gamma_n = n*u / (1 - n*u), a sum of n float32 terms in any order is off by at most gamma_n times the
sum of the terms' absolute values.  The bounds allow any summation order (warp butterflies, fused multiply-adds,
atomic scatters) but not a dropped, doubled or misplaced term: at the tested alpha = 0.05 an update is ~5e-3 and a
bound ~1e-8.  Every kernel that can train a position is covered: the production warp kernel at every column-group
count and occupancy tier, the register kernel (kernel=1, fast mode above 2048 columns, strict mode) at every width
the ABI accepts, bit levels 0 - 24, -reg, 1 - 1024 context rows and 1 - 64 targets, and tables holding
quantization thresholds, -0.0, denormals and rows that saturate f beyond +-6.

The checker itself is tested on the CPU: the sequential float32 oracle passes the same bounds at the same shapes,
and tampered copies of its output (a decay dropped, g from the neighbouring expTable slot, a target's error left
out, unquantized rows in the error, a column zeroed) fail them."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.f64_bounds import SUB, TINY, gamma, grad_scalar, quantizer, special_values
from tests.util import bits, zipf_corpus

def neighbour_slot(f):
    idx = int(np.float32(np.float32(np.float32(f) + np.float32(6)) * np.float32(83)))
    return 1 if idx < 996 else -1


class Check:
    """Float64 expectation and bounds of one position; r_* are |error| / bound (a pass is <= 1)."""

    def __init__(self, q, u0, v0, u1, v1, ctx, tg, f, alpha, reg, exptab, g=None):
        ctx, tg = np.asarray(ctx), np.asarray(tg)
        cw, nt, D = len(ctx), len(tg), u0.shape[1]
        qu = q(u0[ctx]).astype(np.float64)
        qv = q(v0[tg]).astype(np.float64)
        self.avg = qu.sum(0) / cw                                    # :449
        A = np.abs(qu).sum(0) / cw
        f_ref = qv @ self.avg                                        # :464-470
        self.bound_f = gamma(D + cw + 2) * (np.abs(qv) @ A) + (D + cw + 2) * SUB
        self.r_f = np.abs(np.asarray(f, np.float64) - f_ref) / self.bound_f
        self.old_bar = 1e-5 * np.abs(f_ref) + 1e-6                   # test_gpu_parity.py::test_single_step
        if g is None:
            g = [grad_scalar(f[t], int(t == 0), alpha, exptab) for t in range(nt)]
        self.g = np.asarray(g, np.float64)
        d = 2.0 * float(np.float32(alpha)) * float(np.float32(reg))
        v0t = v0[tg].astype(np.float64)
        v_ref = v0t + self.g[:, None] * self.avg[None, :] - d * v0t   # :490
        self.bound_v = (gamma(2) * np.abs(v0t) + gamma(cw + 4) * np.abs(self.g)[:, None] * A[None, :]
                        + gamma(5) * d * np.abs(v0t) + 4 * TINY + 8 * SUB)
        self.r_v_rows = (np.abs(v1[tg] - v_ref) / self.bound_v).max(1)
        ids, m = np.unique(ctx, return_counts=True)
        m = m[:, None].astype(np.float64)
        E = self.g @ qv                                              # :487, quantized old v
        Eabs = np.abs(self.g) @ np.abs(qv)
        u0c = u0[ids].astype(np.float64)
        u_ref = u0c + m * (E[None, :] - d * u0c)                     # :494-503, each occurrence of a context id
        bound_u = (gamma(m + 2) * (np.abs(u0c) + m * (Eabs[None, :] + d * np.abs(u0c))) + m * gamma(nt + 2) * Eabs[None, :]
                   + m * gamma(5) * d * np.abs(u0c) + (m + 3) * TINY + (nt + 8) * m * SUB)
        self.r_u = float((np.abs(u1[ids] - u_ref) / bound_u).max())
        self.r_v = float(self.r_v_rows.max())
        keep_u = np.ones(len(u0), bool); keep_u[ids] = False
        keep_v = np.ones(len(v0), bool); keep_v[tg] = False
        self.untouched = (np.array_equal(bits(u1[keep_u]), bits(u0[keep_u]))
                          and np.array_equal(bits(v1[keep_v]), bits(v0[keep_v])))

    @property
    def worst(self):
        return max(float(self.r_f.max()), self.r_v, self.r_u)

    def ok(self):
        return self.worst <= 1.0 and self.untouched


def fill_special(u, v, ctx, tg, b, rng):
    """Context rows near a common row r of magnitude 3 (f beyond +-6 against +-r) with special values sprinkled in;
    targets 0..2 = -r, +r, -r (saturated f with g = alpha, -alpha and 0), the others sprinkled."""
    D = u.shape[1]
    sv = special_values(b)
    r = (np.where(rng.random(D) < 0.5, -3.0, 3.0) * rng.uniform(0.9, 1.1, D)).astype(np.float32)
    for i in np.unique(ctx):
        row = r + rng.uniform(-0.05, 0.05, D).astype(np.float32)
        at = rng.random(D) < 0.25
        row[at] = rng.choice(sv, int(at.sum()))
        u[i] = row
    for k, i in enumerate(tg):
        if k < 3:
            v[i] = -r if k != 1 else r
        else:
            at = rng.random(D) < 0.5
            v[i, at] = rng.choice(sv, int(at.sum()))


# ------------------------------------------------------------------------------------------------------------- cases
WARP_D = [1, 3, 5, 127, 128, 129, 255, 260, 511, 516, 1021, 1024, 1028, 1200, 1536, 1537, 1540, 2044, 2045, 2048]
REGISTER_D = [673, 1023, 1024, 1408, 1412, 1536, 1920, 2048]   # kernel = 1
WIDE_D = [2052, 2560, 3072, 3588, 4096]                       # fast mode beyond the warp kernel: register kernel
STRICT_D = [1023, 3584, 3588, 4096]
BITS = [0, 1, 2, 3, 5, 8, 24]
REGS = [0.0, 0.05]
NT = [1, 25, 33, 64]
CW = [1, 2, 5, 9, 10]  # window 5


def _cases():
    out = []
    rot = [("warp", D) for D in WARP_D] + [("register", D) for D in REGISTER_D] + [("wide", D) for D in WIDE_D] + \
          [("strict", D) for D in STRICT_D]
    for j, (kind, D) in enumerate(rot):   # bit level and reg rotate along the list (7 x 2: every pair in 14 cases)
        b, reg = BITS[j % 7], REGS[j % 2]
        out.append((kind, D, b, reg, 5, j % 3 == 1, reg == 0.0 and j % 4 == 0))
    for kind, D in (("warp", 800), ("warp", 1200), ("warp", 2048), ("wide", 4096)):
        for b in BITS:
            for reg in REGS:
                out.append((kind, D, b, reg, 5, b in (1, 5), False))
    out.append(("warp", 260, 1, 0.0, 512, False, True))       # ~1000 context rows
    out.append(("register", 1024, 2, 0.05, 512, True, False))  # 1024 context rows
    return out


CASES = _cases()


def case_id(c):
    kind, D, b, reg, W, special, dup = c
    return "%s-D%d-b%d-reg%g%s%s%s" % (kind, D, b, reg, "-W%d" % W if W != 5 else "", "-special" if special else "",
                                      "-dupctx" if dup else "")


def positions(case, V, seed):
    """(context ids, target ids) of the positions of a case: targets distinct, context ids distinct unless `dup`."""
    kind, D, b, reg, W, special, dup = case
    rng = np.random.default_rng(seed)
    shapes = [(CW[(seed + k) % 5], NT[k]) for k in range(4)] if W == 5 else [(2 * W - 24 * (kind == "warp"), 64), (3, 33)]
    out = []
    for cw, nt in shapes:
        ctx = rng.choice(np.arange(1, V), cw, replace=bool(dup)).astype(np.int32)
        if dup and cw > 1:
            ctx[-1] = ctx[0]
        tg = rng.choice(np.arange(1, V), nt, replace=False).astype(np.int32)
        out.append((ctx, tg))
    return out


def minus_zero_takes_sign(kind, D, b, reg):
    nj = ((D + 3) // 4 + 31) // 32  # float4 column groups per lane: beyond 12 the warp kernel decides b at run time
    return kind == "warp" and reg == 0.0 and b in (1, 2) and nj <= 12


def run_case(side, case, V, alpha, exptab, q, seed, report, strict_oracle=None):
    """Trains the case's positions through `side` and checks each; returns the worst ratio per quantity."""
    kind, D, b, reg, W, special, dup = case
    pos = positions(case, V, seed)
    if special:
        u, v = side.tables()
        fill_special(u, v, pos[0][0], pos[0][1], b, np.random.default_rng(seed + 1))
        side.upload(u, v)
    worst = {"f": 0.0, "v": 0.0, "u": 0.0}
    n_slot_checks = 0
    for ctx, tg in pos:
        u0, v0 = side.tables()
        f = side.apply(ctx, tg)
        u1, v1 = side.tables()
        ch = Check(q, u0, v0, u1, v1, ctx, tg, f, alpha, reg, exptab)
        worst["f"] = max(worst["f"], float(ch.r_f.max()))
        worst["v"] = max(worst["v"], ch.r_v)
        worst["u"] = max(worst["u"], ch.r_u)
        assert ch.untouched, "%s: a row outside the position changed" % case_id(case)
        assert ch.ok(), (case_id(case), len(ctx), len(tg), ch.r_f.max(), ch.r_v, ch.r_u)
        # the returned f is the one that fed g: g of the neighbouring expTable slot fails wherever it would be visible
        g_alt = ch.g.copy()
        sat = np.abs(np.asarray(f, np.float32)) > 6
        for t in np.nonzero(~sat)[0]:
            g_alt[t] = grad_scalar(f[t], int(t == 0), alpha, exptab, neighbour_slot(f[t]))
        alt = Check(q, u0, v0, u1, v1, ctx, tg, f, alpha, reg, exptab, g=g_alt)
        visible = (np.abs(g_alt - ch.g)[:, None] * np.abs(ch.avg)[None, :] > 2 * ch.bound_v).any(1)
        assert (alt.r_v_rows[visible] > 1).all(), (case_id(case), alt.r_v_rows[visible])
        n_slot_checks += int(visible.sum())
        if strict_oracle is not None:
            m = strict_oracle
            m.u[...] = u0
            m.v[...] = v0
            fo, _ = m.apply_position(ctx, tg)
            assert np.array_equal(bits(f), bits(fo)) and np.array_equal(bits(u1), bits(m.u)) and \
                np.array_equal(bits(v1), bits(m.v)), "%s: strict mode differs from the oracle" % case_id(case)
    if b != 3 and not special:
        assert n_slot_checks > 0
    report("%s: max err/bound f %.3f v %.3f u %.3f; f bound / old 1e-5 bar %.1e; slot checks %d"
           % (case_id(case), worst["f"], worst["v"], worst["u"], float((ch.bound_f / ch.old_bar).max()), n_slot_checks))
    return worst


@pytest.fixture(scope="module")
def corpus_path(tmp_path_factory):
    d = tmp_path_factory.mktemp("c")
    return zipf_corpus(str(d / "zipf1k.txt"), 20000, 1100, seed=11, newline_every=20)


@pytest.fixture(scope="module")
def oracle_corpus(corpus_path):
    return po.Corpus(corpus_path, 1)


# ----------------------------------------------------------------------------------------------------- on the CPU
class OracleSide:
    def __init__(self, o, D, b, reg, W):
        self.m = po.OracleModel(o, D, W, 63, b, reg=reg, table=np.zeros(1, np.int32))

    def tables(self):
        return self.m.u.copy(), self.m.v.copy()

    def upload(self, u, v):
        self.m.u[...] = u
        self.m.v[...] = v

    def apply(self, ctx, tg):
        return self.m.apply_position(ctx, tg)[0]


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_oracle_within_f64_bounds(case, oracle_corpus):
    """The sequential float32 oracle meets the bounds the kernels are held to, at the same shapes."""
    kind, D, b, reg, W, special, dup = case
    side = OracleSide(oracle_corpus, D, b, reg, W)
    run_case(side, case, oracle_corpus.vocab_size, side.m.alpha, po.exptable(), quantizer(b, False),
             CASES.index(case), print)


TAMPER = ["decay_dropped", "neighbour_slot", "target_error_omitted", "unquantized_error", "last_float4_column_zeroed"]


@pytest.mark.parametrize("D", [5, 260, 1024])
@pytest.mark.parametrize("tamper", TAMPER)
def test_checker_catches_tampered_oracle(tamper, D, oracle_corpus):
    """Each tampered copy of the oracle's output fails the bounds the untampered output meets."""
    b, reg, W = 1, 0.05, 5
    V = oracle_corpus.vocab_size
    side = OracleSide(oracle_corpus, D, b, reg, W)
    ctx, tg = positions(("warp", D, b, reg, W, False, False), V, 3)[2]
    q = po.exptable()
    alpha = side.m.alpha
    u0, v0 = side.tables()
    if tamper == "neighbour_slot":  # the oracle run with expTable slot i holding slot i + 1
        ex = np.ascontiguousarray(np.roll(q, -1))
        f = np.zeros(len(tg), np.float32)
        po.lib().w2bo_apply_position(C.byref(side.m.m), ex, ctx, len(ctx), tg, len(tg), f, C.byref(C.c_double()))
    else:
        f = side.apply(ctx, tg)
    u1, v1 = side.tables()
    quant = quantizer(b, False)
    honest = Check(quant, u0, v0, u1, v1, ctx, tg, f, alpha, reg, q)
    if tamper == "neighbour_slot":
        assert not honest.ok()
        return
    assert honest.ok(), (honest.r_f.max(), honest.r_v, honest.r_u)
    d = np.float32(2 * alpha * reg)
    g = honest.g.astype(np.float32)
    if tamper == "decay_dropped":
        v1[tg[0]] = v1[tg[0]] + d * v0[tg[0]]
    elif tamper == "target_error_omitted":
        v_last = quant(v0[tg[-1]])
        for i in np.unique(ctx):
            u1[i] = u1[i] - g[-1] * v_last
    elif tamper == "unquantized_error":
        for i in np.unique(ctx):
            u1[i] = u1[i] + (g[:, None] * (v0[tg] - quant(v0[tg]))).sum(0)
    else:
        v1[tg[0], D - 1] = 0.0
    tampered = Check(quant, u0, v0, u1, v1, ctx, tg, f, alpha, reg, q)
    assert not tampered.ok(), (tamper, tampered.r_f.max(), tampered.r_v, tampered.r_u)


# ----------------------------------------------------------------------------------------------------- on the GPU
class TrainerSide:
    def __init__(self, t):
        self.t = t

    def tables(self):
        return self.t.download_raw()

    def upload(self, u, v):
        self.t.upload_raw(u, v)

    def apply(self, ctx, tg):
        return self.t.apply_position(ctx, tg)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_position_within_f64_bounds(case, corpus_path, oracle_corpus):
    w2b = pytest.importorskip("word2bits_b200")
    kind, D, b, reg, W, special, dup = case
    c = w2b.Corpus(corpus_path, 1)
    kw = dict(size=D, window=W, negative=63, bitlevel=b, reg=reg, threads=1, iter=1,
              kernel=1 if kind == "register" else 0, mode=w2b.MODE_STRICT if kind == "strict" else w2b.MODE_FAST)
    plan = w2b.warp_plan(vocab_size=c.vocab_size, **{k: kw[k] for k in ("size", "window", "negative", "bitlevel", "reg",
                                                                        "mode", "kernel")})
    assert plan["warp"] == (kind == "warp")  # the kernel the case is meant for is the one that runs
    t = w2b.Trainer(c, **kw)
    alpha, _ = t.get_state()
    oracle = None
    if kind == "strict":
        oracle = po.OracleModel(oracle_corpus, D, W, 63, b, reg=reg, table=np.zeros(1, np.int32))
        oracle.m.alpha = alpha
    run_case(TrainerSide(t), case, c.vocab_size, alpha, t.download_exptable(),
             quantizer(b, minus_zero_takes_sign(kind, D, b, reg)), CASES.index(case), print, strict_oracle=oracle)
    t.close()


@pytest.mark.gpu
def test_quantize_bits_beyond_8():
    """Bit levels 9..24 (validate() accepts up to 24) bit for bit against the oracle, on L0's inputs
    (test_gpu_parity.py::test_quantize_bits) plus each level's rounding thresholds and their neighbours."""
    w2b = pytest.importorskip("word2bits_b200")
    t = w2b.Trainer(None, vocab_size=4, size=8, window=3, negative=4, threads=1)
    xs = np.concatenate([
        np.array([0.0, -0.0, 1e-30, -1e-30, .25, .5, np.nextafter(np.float32(.5), np.float32(1)), .75, 1.0, -1.0,
                  3.7, -3.7, 1 / 32, .0624, .0625, .09375, .49999, -.5, -.50001, .124, .126], np.float32),
        np.random.default_rng(0).uniform(-1.5, 1.5, 4000).astype(np.float32)])
    for b in range(9, 25):
        x = np.concatenate([xs, special_values(b)])
        assert np.array_equal(bits(t.quantize(x, b)), bits(po.quantize(x, b))), b


@pytest.mark.gpu
def test_wide_rows_train_an_epoch(tmp_path):
    """Widths only the register kernel serves train a whole epoch: strict mode at D = 4096 and fast mode at D = 3000
    through the CLI, kernel = 1 at D = 1920 through the Python API."""
    import subprocess
    w2b = pytest.importorskip("word2bits_b200")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    golden = os.path.join(root, "tests", "golden", "golden_corpus.txt")
    for size, strict in ((4096, 1), (3000, 0)):
        out = str(tmp_path / ("v%d" % size))
        r = subprocess.run([os.path.join(root, "word2bits_b200", "word2bits"), "-train", golden, "-output", out,
                            "-size", str(size), "-window", "3", "-negative", "2", "-threads", "2", "-iter", "1",
                            "-min-count", "1", "-binary", "1", "-strict", str(strict)],
                           capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        assert "Epoch Loss:" in r.stdout and open(out, "rb").read().startswith(b"31 %d\n" % size)
    c = w2b.Corpus(golden, 1)
    t = w2b.Trainer(c, size=1920, window=3, negative=4, bitlevel=1, threads=4, iter=1, kernel=1)
    loss, st = t.train_epoch()
    assert st["shards_done"] == 4 and st["positions"] > 0 and np.isfinite(loss)
    u, v = t.download_raw()
    assert np.isfinite(u).all() and np.isfinite(v).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D", [("register", D) for D in REGISTER_D] + [("wide", D) for D in WIDE_D] +
                         [("strict", D) for D in STRICT_D], ids=lambda x: str(x))
def test_register_kernel_trains_at_every_width(kind, D, corpus_path):
    """The register kernel's training launches (not only the single-position hook above) at every width it serves, for
    each instantiation the dispatch can pick there: groups of 5 / 9 / 13 targets (negative 4 / 8 / 12), -reg, and the
    compile-time and run-time bit levels."""
    w2b = pytest.importorskip("word2bits_b200")
    c = w2b.Corpus(corpus_path, 1)
    configs = ((4, 1, 0.0), (8, 2, 0.0), (12, 0, 0.0), (12, 5, 0.05)) if kind != "strict" else ((4, 1, 0.0), (6, 5, 0.05))
    for neg, b, reg in configs:
        t = w2b.Trainer(c, size=D, window=5, negative=neg, bitlevel=b, reg=reg, threads=2, iter=1,
                        kernel=1 if kind == "register" else 0, mode=w2b.MODE_STRICT if kind == "strict" else w2b.MODE_FAST)
        st = t.train_step(400 if kind == "strict" else 1500)
        assert st["positions"] > 0 and np.isfinite(st["loss"]), (neg, b, reg, st)
        u, v = t.download_raw()
        assert np.isfinite(u).all() and np.isfinite(v).all()
        t.close()
