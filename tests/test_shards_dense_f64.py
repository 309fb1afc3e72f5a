"""Dense many-shard training steps at the planner's shard count, element by element, on tables whose quantized levels
no interleaving of the step can change.

tests/test_shards_f64.py checks the benchmarked shard count only on a sparse corpus, where shards share rows through
negative draws alone; on the dense corpus its Hogwild fixed point settles only at 132 shards.  Here the corpus is
bench.py's (ids = Zipf rank, bench's counts and sub-sampling), cut into short sentences, at the planner's shard count:
the v rows of the most frequent words take hundreds to thousands of concurrent scatters per step.

At bit levels 1 and 2 a training read sees a row only through quantize().  The tables are seeded so that every
element a step touches starts far enough inside its quantization level that no subset of the step's updates to it can
move it out.  Then every read of every interleaving quantizes to the seeded level, so ctx_avg, f, g, the loss and every
update are fixed by the draws alone, and the replay is one float64 pass (the Replay arithmetic and bounds of
tests/test_trajectory_f64.py) against the fixed levels; a -reg decay, which reads the row itself, takes the whole
level box.  The checker does not trust the seeding: from its own update intervals it verifies that x0 minus the sum
of every update's negative hull and x0 plus the sum of the positive hulls (plus the rounding of every add) stay
strictly inside the box it assumed for the reads, which lies inside the level; otherwise it refuses the tables.
On every touched element the final value must then lie in x0 + the sum of the update centres +- (the sum of their
radii + one float32 add's rounding per update, at the largest partial sum any order can reach, + the flushed-denormal
allowance): an accounting check that no order can change.

What this sees: every scatter, on every touched element, exactly once per update: a lost, doubled, misdirected or
partial-row scatter, or one landed twice after its ring slot was reused; a read of the wrong row or of garbage (it
changes f and g).  What it cannot see: a stale or torn read of the right row, which gives the same level (Hogwild
admits such reads anyway).  Bit level 0 has no level to hold; its dense check stays the 132-shard case of
tests/test_shards_f64.py.

On the CPU the Hogwild executor of tests/test_shards_f64.py (random interleavings, late landings, element-wise
prefixes) runs on margin-seeded tables: no read sees another level, and the result passes; its dropped, doubled and
race-overwritten updates, shards trained on their neighbour's sentence and a lost shard loss fail; InitNet tables
are refused."""
import multiprocessing as mp
import os
import time
from contextlib import nullcontext

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.f64_bounds import TINY, U, quantizer
from tests.test_shards_f64 import HogwildExecutor, changed_rows, synthetic_positions, traces
from tests.test_trajectory_f64 import Model, Replay, Trajectory, model_for
from tests.util import bits, zipf_corpus

SHRINK = 1 - 2.0 ** -10  # the read box keeps this hair inside its level
SLACK = 1.5              # seeding: the box's half-width over the larger of an element's update hulls


class Refused(AssertionError):
    """The tables do not hold every touched element inside its quantization level for the step checked."""


def level_box(x0, b):
    """Half-width h of the interval x0 +- h (float64) that a read of the element is assumed to see: the largest one
    around x0 inside x0's quantization level, shrunk by a hair.  0 on a level boundary (0; |x| = 0.5 at bit level 2)."""
    a = np.abs(x0)
    if b == 1:  # x < 0 -> -1/3, else 1/3
        h = a
    else:       # b = 2: |x| <= 0.5 -> 0.25, else 0.75
        h = np.where(a <= 0.5, np.minimum(a, 0.5 - a), a - 0.5)
    return h * SHRINK


def rounding(n, x0, P, N):
    """n float32 adds' rounding, each at the largest partial sum any order can reach, and their flushed denormals."""
    return n * (1.01 * U * (np.abs(x0) + P + N) + 2 * TINY)


class LevelReplay(Replay):
    """The replay against fixed levels.  A read of row i sees x0 +- level_box(x0): quantized it is x0's level with
    radius 0, and a -reg decay takes the box.  add_to leaves the row as it is and adds the update's interval to the
    element's account [sum of centres, sum of radii, sum of positive hulls, sum of negative hulls, adds].  Nothing of
    this holds until LevelStep.check has verified the margins from the accounts."""

    def __init__(self, u0, v0, b, q, reg, exptab, model, watch=()):
        assert b in (1, 2)
        super().__init__(u0, v0, b, q, reg, exptab, model)
        self.hull = True  # a repeated target reads before or after the earlier update: the same level either way
        self.acc, self.box = {}, {}
        self.watch, self.log = set(watch), {}

    def key(self, T, i):
        return ("u" if T is self.U else "v", i)

    def read(self, T, src, i):
        k = self.key(T, i)
        if k not in self.box:
            x0 = src[i].astype(np.float64)
            self.box[k] = (x0, level_box(x0, self.b))
        x0, h = self.box[k]
        return [x0.copy(), h.copy()]

    def quant(self, c, r):
        # c is x0 or x0 + half an earlier update of the same position: inside the box once the margins are verified.
        # quantize() of a nonzero float32 at bit level 1 or 2 (w2b_quant.cuh), the level as float32
        lv = np.float32(1 / 3) if self.b == 1 else np.where(np.abs(c) <= 0.5, np.float32(0.25), np.float32(0.75))
        return np.where(c < 0, -lv, lv).astype(np.float64), np.zeros(self.D)

    def add_to(self, T, i, dc, dr):
        k = self.key(T, i)
        a = self.acc.get(k)
        if a is None:
            z = np.zeros(self.D)
            a = self.acc[k] = [z, z, z, z, 0]
        a[0], a[1] = a[0] + dc, a[1] + dr
        a[2], a[3] = a[2] + np.maximum(dc + dr, 0), a[3] + np.maximum(dr - dc, 0)
        a[4] += 1
        if k in self.watch:
            self.log.setdefault(k, []).append((dc, dr))


_WORKER = None  # (LevelStep, u0, v0, watch): read by the forked workers of LevelStep.accounts


def _replay_chunk(shards):
    m, u0, v0, watch = _WORKER
    r = LevelReplay(u0, v0, *m.args, watch=watch)
    loss = []
    for s in shards:
        c0, r0 = r.loss_c, r.loss_r
        for ctx, tg, a in m.pos[s]:
            r.position(ctx, tg, a)
        loss.append((s, r.loss_c - c0, r.loss_r - r0))
    out = {}
    for name in "uv":
        keys = sorted(k[1] for k in r.acc if k[0] == name)
        A = np.stack([np.stack(r.acc[(name, i)][:4]) for i in keys]) if keys else np.zeros((0, 4, r.D))
        out[name] = (np.array(keys, np.int64), A, np.array([r.acc[(name, i)][4] for i in keys], np.int64))
    return out, loss, r.log


class LevelStep:
    """One many-shard step, `positions[s]` = shard s's positions (ctx, targets, alpha), checked against fixed levels."""

    def __init__(self, positions, b, q, reg, exptab, model):
        self.pos, self.b, self.args = positions, b, (b, q, reg, exptab, model)
        self.users = {"u": {}, "v": {}}  # row -> shards touching it
        self.occ = {"u": {}, "v": {}}    # row -> occurrences in the step's positions
        for s, ps in enumerate(positions):
            for ctx, tg, _ in ps:
                for name, ids in (("u", ctx), ("v", tg)):
                    for i in ids.tolist():
                        self.users[name].setdefault(i, set()).add(s)
                        self.occ[name][i] = self.occ[name].get(i, 0) + 1
        self.rows = {k: np.array(sorted(self.users[k]), np.int64) for k in "uv"}
        self.hot = {k: max(self.occ[k], key=lambda i: (self.occ[k][i], -i)) for k in "uv"}

    # ---------------------------------------------------------------------------------------------- the pass
    def accounts(self, u0, v0, watch=()):
        """Every shard's positions replayed once: {table: (update sums [rows, 4, D], adds [rows])} aligned with
        self.rows, the loss interval of each shard, and every update of the watched rows."""
        global _WORKER
        A = {k: np.zeros((len(self.rows[k]), 4, u0.shape[1])) for k in "uv"}
        n = {k: np.zeros(len(self.rows[k]), np.int64) for k in "uv"}
        loss = np.zeros((len(self.pos), 2))
        log = {}
        procs = min(32, len(os.sched_getaffinity(0)))
        chunks = [list(range(a, len(self.pos), procs)) for a in range(min(procs, len(self.pos)))]
        _WORKER = (self, u0, v0, tuple(watch))
        try:
            with mp.get_context("fork").Pool(procs) if procs > 1 else nullcontext() as pool:
                it = pool.imap_unordered(_replay_chunk, chunks) if pool else map(_replay_chunk, chunks)
                for out, ls, lg in it:
                    for k in "uv":
                        rows, a, c = out[k]
                        idx = np.searchsorted(self.rows[k], rows)
                        A[k][idx] += a
                        n[k][idx] += c
                    for s, c, r in ls:
                        loss[s] = (c, r)
                    for key, ups in lg.items():
                        log.setdefault(key, []).extend(ups)
        finally:
            _WORKER = None
        return A, n, loss, log

    def shard_accounts(self, u0, v0, positions):
        """The accounts of one shard's positions alone (the controls): {table: {row: (update sums, adds)}}, loss."""
        r = LevelReplay(u0, v0, *self.args)
        for ctx, tg, a in positions:
            r.position(ctx, tg, a)
        out = {"u": {}, "v": {}}
        for (name, i), a in r.acc.items():
            out[name][i] = (np.stack(a[:4]), a[4])
        return out, (r.loss_c, r.loss_r)

    # ------------------------------------------------------------------------------------------ the margins
    def margins(self, u0, v0, A, n, chunk=4096):
        """Raises Refused unless every touched element's reachable values (x0 - its negative hulls .. x0 + its
        positive hulls, with every add's rounding) lie strictly inside the box its reads were replayed with.
        Returns the smallest box / reach ratio."""
        worst = np.inf
        for name, T in (("u", u0), ("v", v0)):
            rows = self.rows[name]
            for a in range(0, len(rows), chunk):
                x0 = T[rows[a:a + chunk]].astype(np.float64)
                C, R, P, N = np.moveaxis(A[name][a:a + chunk], 1, 0)
                reach = np.maximum(P, N) + rounding(n[name][a:a + chunk, None], x0, P, N)
                h = level_box(x0, self.b)
                bad = ~(reach < h)
                if bad.any():
                    k, col = np.unravel_index(int(np.argmax(bad)), bad.shape)
                    raise Refused("%s row %d column %d: x0 %r, box +-%.3g inside its level, but its updates reach "
                                  "+%.3g / -%.3g (%d adds); %d elements of the step outside their level box" % (
                                      name, rows[a + k], col, x0[k, col], h[k, col], P[k, col], N[k, col],
                                      n[name][a + k], int(bad.sum())))
                worst = min(worst, float((h / reach).min()))
        return worst

    # -------------------------------------------------------------------------------------------- the check
    def check(self, u0, v0, u1, v1, loss, watch=()):
        """Verifies the margins, then every touched element, the untouched rows and the loss.  Raises Refused or
        AssertionError; returns the summary."""
        A, n, lossiv, log = self.accounts(u0, v0, watch)
        self.A, self.n, self.loss_sh, self.log = A, n, lossiv, log
        out = dict(margin=self.margins(u0, v0, A, n))
        self.before, self.after = {"u": u0, "v": v0}, {"u": u1, "v": v1}
        shared_ratio = []
        for name in "uv":
            rows = self.rows[name]
            shared = np.array([len(self.users[name][i]) > 1 for i in rows.tolist()], bool)
            worst = 0.0
            for a in range(0, len(rows), 4096):
                ids = rows[a:a + 4096]
                x0, x1 = self.before[name][ids].astype(np.float64), self.after[name][ids].astype(np.float64)
                C, R, P, N = np.moveaxis(A[name][a:a + 4096], 1, 0)
                rad = R + rounding(n[name][a:a + 4096, None], x0, P, N)
                ratio = np.abs(x1 - x0 - C) / rad
                worst = max(worst, float(ratio.max()))
                if ratio.max() > 1:
                    k, col = np.unravel_index(int(ratio.argmax()), ratio.shape)
                    i = int(ids[k])
                    raise AssertionError("%s row %d column %d (%d adds from %d shards): %r, replay %r +- %.3g" % (
                        name, i, col, n[name][a + k], len(self.users[name][i]), x1[k, col], x0[k, col] + C[k, col],
                        rad[k, col]))
                sh = shared[a:a + 4096]
                shared_ratio.append((np.abs(x1 - x0)[sh] / rad[sh]).ravel())
            out[name] = worst
            bad = sorted(set(changed_rows(self.after[name], self.before[name]).tolist()) - set(rows.tolist()))
            assert not bad, "%s row %d changed, and no shard touched it" % (name, bad[0])
        lr = lossiv[:, 1] + 1e-9 * np.abs(lossiv[:, 0])
        self.loss_lo, self.loss_hi = float((lossiv[:, 0] - lr).sum()), float((lossiv[:, 0] + lr).sum())
        mid, half = (self.loss_lo + self.loss_hi) / 2, (self.loss_hi - self.loss_lo) / 2
        out["loss"] = abs(loss - mid) / half
        assert out["loss"] <= 1, "loss %r outside the shards' sum %r +- %.3g" % (loss, mid, half)
        self.loss = loss
        sr = np.concatenate(shared_ratio) if shared_ratio else np.zeros(0)
        out["median_shared"] = float(np.median(sr)) if len(sr) else None
        return out

    def index(self, name, i):
        return int(np.searchsorted(self.rows[name], i))

    def row_fails(self, name, i, dA, dn):
        """True when row i, its accounts changed by dA / dn, is outside its interval (or, left with no update,
        changed)."""
        k = self.index(name, i)
        x0, x1 = self.before[name][i].astype(np.float64), self.after[name][i].astype(np.float64)
        C, R, P, N = self.A[name][k] + dA
        n = self.n[name][k] + dn
        if n == 0:
            return not np.array_equal(bits(self.after[name][i]), bits(self.before[name][i]))
        P, N = np.maximum(P, self.A[name][k][2]), np.maximum(N, self.A[name][k][3])  # the larger rounding
        return bool((np.abs(x1 - x0 - C) > R + rounding(n, x0, P, N)).any())

    # ------------------------------------------------------------------------------------------ the controls
    def fails_with(self, s, replacement=None, rows=None):
        """True when the step fails with shard s's positions left out (replacement None) or replaced: some row's
        element outside its changed interval, a row left with no update found changed, a row no shard touched
        found updated, or the loss outside the changed sum.  `rows` restricts the rows looked at, and leaves the
        loss out of it."""
        u0, v0 = self.before["u"], self.before["v"]
        mine, (lc, lr) = self.shard_accounts(u0, v0, self.pos[s])
        alt, (ac, ar) = self.shard_accounts(u0, v0, replacement) if replacement is not None else ({"u": {}, "v": {}},
                                                                                              (0.0, 0.0))
        for name in "uv":
            for i in set(mine[name]) | set(alt[name]):
                if rows is not None and (name, i) not in rows:
                    continue
                a0, n0 = mine[name].get(i, (0.0, 0))
                a1, n1 = alt[name].get(i, (0.0, 0))
                if i not in self.users[name]:  # a row only the replacement touches: updated where nothing changed
                    x1 = self.after[name][i].astype(np.float64) - self.before[name][i]
                    C, R, P, N = a1
                    if (np.abs(x1 - C) > R + rounding(n1, self.before[name][i], P, N)).any():
                        return True
                    continue
                if self.row_fails(name, i, a1 - a0, n1 - n0):
                    return True
        if rows is not None:
            return False
        l0 = (lc - (lr + 1e-9 * abs(lc)), lc + (lr + 1e-9 * abs(lc)))
        l1 = (ac - (ar + 1e-9 * abs(ac)), ac + (ar + 1e-9 * abs(ac))) if replacement is not None else (0.0, 0.0)
        return not (self.loss_lo - l0[0] + l1[0] <= self.loss <= self.loss_hi - l0[1] + l1[1])

    def resolvable(self, key):
        """Largest single update of the watched row `key` over the row's largest radius."""
        name, i = key
        k = self.index(name, i)
        C, R, P, N = self.A[name][k]
        rad = R + rounding(self.n[name][k], self.before[name][i].astype(np.float64), P, N)
        return max(float(np.abs(dc).max()) for dc, _ in self.log[key]) / float(rad.max())

    def update_fails(self, key, times):
        """True when the largest update of the watched row `key` counted `times` times (0: dropped, 2: doubled)
        fails the row."""
        dc, dr = max(self.log[key], key=lambda u: float(np.abs(u[0]).max()))
        d = times - 1
        z = np.zeros_like(dc)
        return self.row_fails(key[0], key[1], np.stack([d * dc, d * dr, z, z]), d)

    # -------------------------------------------------------------------------------------------- the seeding
    def seed(self, u0, v0, rng, cold_adds=2, rounds=6):
        """Tables in which every touched element's level is drawn with `rng` and its magnitude set SLACK times
        outside its update hulls: at bit level 2 the elements of v rows with at most `cold_adds` occurrences take
        0.25 or 0.75 at random (one such update moves an element by at most alpha * 0.75, so 0.25 fits), every other
        element 0.75.  Untouched rows stay as they are.  The accounts depend on the levels, and under -reg on the
        magnitudes, so the pass is repeated until the margins hold (check() verifies them again from its own pass)."""
        u0, v0 = u0.copy(), v0.copy()
        T = {"u": u0, "v": v0}
        D = u0.shape[1]
        sign, outer = {}, {}
        for name in "uv":
            rows = self.rows[name]
            sign[name] = np.where(rng.random((len(rows), D)) < 0.5, -1.0, 1.0)
            adds = np.array([self.occ[name][i] for i in rows.tolist()])
            outer[name] = (rng.random((len(rows), D)) < 0.5) | (adds[:, None] > cold_adds) | (name == "u")
            T[name][rows] = sign[name] * np.where(outer[name], 1.0, 0.25) if self.b == 2 else sign[name] * 0.5
        A, n, _, _ = self.accounts(u0, v0)
        for _ in range(rounds):
            moved = False  # an element changed level: every update of its rows' positions changes
            for name in "uv":
                rows = self.rows[name]
                C, R, P, N = np.moveaxis(A[name], 1, 0)
                m = SLACK * (np.maximum(P, N) + rounding(n[name][:, None], 2.0, P, N)) + 1e-5
                if self.b == 1:
                    mag = m * (1 + 0.5 * rng.random(m.shape))
                else:  # (0, 0.5] only for hulls well inside it: the accounts change with every level moved
                    moved = moved or bool((~outer[name] & (m >= 0.2)).any())
                    outer[name] |= m >= 0.2
                    inner = 0.25 + (rng.random(m.shape) - 0.5) * (0.5 - 2 * m)
                    mag = np.where(outer[name], 0.5 + m * (1 + 0.5 * rng.random(m.shape)), inner)
                T[name][rows] = (sign[name] * mag).astype(np.float32)
            if self.args[2] or moved:  # without -reg or a level moved, the updates do not depend on the magnitudes
                A, n, _, _ = self.accounts(u0, v0)
            if moved:
                continue
            try:
                self.margins(u0, v0, A, n)
                return u0, v0
            except Refused:
                continue
        return u0, v0


# ----------------------------------------------------------------------------------------- the CPU: an executor
class LevelExecutor(HogwildExecutor):
    """The Hogwild executor, counting reads whose quantized value is not the row's level before the step."""

    def __init__(self, *a, b):
        super().__init__(*a)
        self.b, self.reads, self.off = b, 0, 0

    def view(self, key, s, landed, rng):
        x = super().view(key, s, landed, rng)
        x0 = (self.u0 if key[0] == "u" else self.v0)[key[1]]
        self.reads += x.size
        self.off += int((po.quantize(x, self.b) != po.quantize(x0, self.b)).sum())
        return x


@pytest.fixture(scope="module")
def dense_corpus(tmp_path_factory):
    path = zipf_corpus(str(tmp_path_factory.mktemp("dense") / "z.txt"), 20000, 5000, seed=43, newline_every=12)
    return po.Corpus(path, 1)


EXECUTOR_SHAPES = [  # D, window, negative, bit level, reg, model
    (64, 5, 12, 1, 0.0, "warp"), (64, 5, 12, 1, 0.002, "warp"), (48, 5, 6, 2, 0.0, "warp"),
    (48, 5, 6, 2, 0.002, "seq"), (32, 5, 8, 1, 0.002, "register-g9"), (32, 5, 8, 2, 0.0, "register-g9"),
]


def executor_case(corpus, shape, shards=12, per_shard=4, seed=0):
    """Shards of synthetic positions whose negatives come from 40 ids and a third of whose positions share a
    context row: every shared row is shared by most shards.  InitNet tables, touched rows margin-seeded."""
    D, W, N, b, reg, kind = shape
    V = corpus.vocab_size
    pos = synthetic_positions(shards, per_shard, N, V, seed, pool=40, shared_ctx=0.3)
    model = Model("warp", nj=1) if kind == "warp" else Model("seq")
    if kind == "register-g9":  # the oracle reads a group's rows before its updates when no group repeats a target
        model = Model("register", G=9, vec=1, threads=32)
        pos = [[p for p in ps if len(np.unique(p[1][:9])) == len(p[1][:9])] for ps in pos]
    ex_tab = po.exptable()
    chk = LevelStep(pos, b, quantizer(b, False), reg, ex_tab, model)
    u0, v0 = chk.seed(*po.init_net(V, D), np.random.default_rng(seed + 1))
    return LevelExecutor(corpus, D, W, N, b, reg, u0, v0, b=b), pos, chk, u0, v0


@pytest.mark.parametrize("shape", EXECUTOR_SHAPES, ids=lambda s: "D%d-W%d-N%d-b%d-reg%g-%s" % s)
def test_level_tables_hold_under_the_hogwild_executor(shape, dense_corpus):
    """Random interleavings, late landings and element-wise prefixes on margin-seeded tables: every read quantizes
    to the seeded level, and the result passes the one-pass check."""
    ex, pos, chk, u0, v0 = executor_case(dense_corpus, shape)
    hot = max(len(s) for s in chk.users["v"].values())
    assert hot >= len(pos) // 2, hot  # the hottest v row is shared by most shards
    if shape[3] == 2:
        lv = np.abs(po.quantize(v0[chk.rows["v"]], 2))
        assert (lv == np.float32(0.25)).any() and (lv == np.float32(0.75)).any()
    for seed in range(3):
        u1, v1, losses = ex.run(pos, seed)
        res = chk.check(u0, v0, u1, v1, float(losses.sum()))
        print(shape, "seed", seed, "%d reads, %d off level; worst err/bound u %.3f v %.3f loss %.3f; margin x%.3g; "
              "median |update|/radius shared %.3g" % (ex.reads, ex.off, res["u"], res["v"], res["loss"],
                                                      res["margin"], res["median_shared"]))
        assert ex.reads > 0 and ex.off == 0
        assert res["median_shared"] > 10


CORRUPTIONS = ["drop", "twice", "overwrite", "neighbour_positions", "loss_left_out"]


@pytest.mark.parametrize("kind", CORRUPTIONS)
def test_executor_corruptions_fail_the_level_check(kind, dense_corpus):
    """The update of a shared row largest against its row's radius dropped, applied twice, or lost to a
    load/add/store race; shards trained on their neighbour's sentence with their own draws; a lost shard loss: each
    fails the check (and not by refusing the tables)."""
    ex, pos, chk, u0, v0 = executor_case(dense_corpus, EXECUTOR_SHAPES[0])
    log = []
    u1, v1, losses = ex.run(pos, 7, log=log)
    chk.check(u0, v0, u1, v1, float(losses.sum()))
    if kind in ("drop", "twice", "overwrite"):
        shared = lambda k: len(chk.users[k[0]].get(k[1], ())) > 1
        cand = [(pm if kind == "overwrite" else m, j) for j, (k, s, m, prev, pm) in enumerate(log)
                if shared(k) and (kind != "overwrite" or (prev is not None and prev != s))]
        u1, v1, losses = ex.run(pos, 7, corrupt=(kind, max(cand)[1]))
    elif kind == "neighbour_positions":
        shifted = [[(c1, np.concatenate([t1[:1], t0[1:]]), a) for (_, t0, a), (c1, t1, _) in
                    zip(pos[s], pos[(s + 1) % len(pos)])] for s in range(len(pos))]
        u1, v1, losses = ex.run(shifted, 7)
    else:
        losses[2] = 0.0
    with pytest.raises(AssertionError) as e:
        chk.check(u0, v0, u1, v1, float(losses.sum()))
    assert not isinstance(e.value, Refused), e.value
    print(kind, str(e.value)[:200])


def test_margin_check_refuses_tables_without_margins(dense_corpus):
    """InitNet tables (v = 0: every element on a level boundary) are refused; so are seeded tables in which one
    element of the hottest v row is moved inside its negative hull."""
    ex, pos, chk, u0, v0 = executor_case(dense_corpus, EXECUTOR_SHAPES[0])
    ui, vi = po.init_net(dense_corpus.vocab_size, 64)
    u1, v1, losses = ex.run(pos, 0)
    with pytest.raises(Refused):
        chk.check(ui, vi, u1, v1, float(losses.sum()))
    chk.check(u0, v0, u1, v1, float(losses.sum()))
    i = chk.hot["v"]
    k = chk.index("v", i)
    C, R, P, N = chk.A["v"][k]
    col = int(np.argmax(N * (v0[i] > 0)))
    bad = v0.copy()
    bad[i, col] = np.float32(N[col] / 2)
    with pytest.raises(Refused) as e:
        chk.check(u0, bad, u1, v1, float(losses.sum()))
    print(str(e.value)[:200])


def test_level_box():
    x = np.array([0.0, -0.0, 1e-30, -0.3, 0.5, 0.6, -2.0], np.float32).astype(np.float64)
    assert np.array_equal(level_box(x, 1), np.abs(x) * SHRINK)
    h2 = level_box(x, 2)
    assert h2[0] == h2[1] == h2[4] == 0 and h2[2] > 0
    assert np.isclose(h2[3], 0.2 * SHRINK) and np.isclose(h2[5], 0.1 * SHRINK) and np.isclose(h2[6], 1.5 * SHRINK)
    for b in (1, 2):  # the box's float32 ends quantize to x0's level
        y = x[np.abs(x) > 1e-20]
        h = level_box(y, b)
        for e in (y - h, y + h):
            e32 = e.astype(np.float32)
            assert np.array_equal(po.quantize(e32, b), po.quantize(y.astype(np.float32), b))


# ------------------------------------------------------------------------------------------------------ the GPU
NOMINAL_WORDS = 300_000_000  # bench.py caps one rank's corpus near this: its counts and sub-sampling at that size
KEEP_RANK = 100               # sub-sampling keeps every word of Zipf rank >= 100 (ran >= 1) at V = 5 000 and 400 001


def bench_inputs(S, V, L=4, per_shard=3, seed=43):
    """bench.py's corpus over V - 1 words (ids = Zipf rank, its expected counts), cut into L-word sentences: shard s
    owns `per_shard` of them.  Each sentence holds at least 2 words sub-sampling always keeps, so every shard trains
    at least 2 positions; about one in three repeats a word two slots later, a repeated context id."""
    import bench
    cdf, pmf = bench.zipf_cdf(V - 1)
    n = S * per_shard
    ids = bench.synth_ids(8 * n * L, seed, cdf).reshape(-1, L)
    ids[::3, L - 1] = ids[::3, L - 3]
    ids = ids[(ids >= KEEP_RANK).sum(1) >= 2][:n].copy()
    assert len(ids) == n
    tokens = np.concatenate([ids, np.zeros((n, 1), np.int32)], 1).ravel().astype(np.int32)
    start = np.arange(S, dtype=np.int64) * per_shard * (L + 1)
    return tokens, start, bench.expected_counts(NOMINAL_WORDS, pmf), NOMINAL_WORDS


GPU_CASES = {  # name -> configuration; "expect" is the instantiation and geometry the case is written for
    "c2": dict(D=800, W=10, N=24, b=1, reg=0.0, expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=1584),
    "c2-streamed": dict(D=800, W=10, N=24, b=1, reg=0.0, resident=False,
                        expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=1584),
    "c2-two-waves": dict(D=800, W=10, N=24, b=1, reg=0.0, waves=2,
                         expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=3168),
    "c3": dict(D=400, W=10, N=12, b=2, reg=0.0, expect={"warp": 1, "bm": 2}),
    "reg": dict(D=800, W=10, N=5, b=1, reg=0.002, expect={"warp": 1, "nj": 7, "minb": 8, "reg": 1}),
    "register-tuned": dict(D=512, W=5, N=8, b=1, reg=0.0, kernel=1, expect={"warp": 0, "wide": 0, "vec": 4, "group": 9}),
    "small-vocab": dict(D=800, W=10, N=24, b=1, reg=0.0, V=5000, expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}),
}


def take(tj, words):
    pos, w = [], 0
    while w < words:
        pos += tj.next_positions()
        w += tj.advance()
    return pos, w


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_CASES))
def test_dense_many_shard_step_on_level_tables(name):
    w2b = pytest.importorskip("word2bits_b200")
    t_start = time.time()
    cfg = GPU_CASES[name]
    D, W, N, b, reg = cfg["D"], cfg["W"], cfg["N"], cfg["b"], cfg["reg"]
    V = cfg.get("V", 400_001)
    kw = dict(size=D, window=W, negative=N, bitlevel=b, reg=reg, iter=1, kernel=cfg.get("kernel", 0))
    probe = w2b.Trainer(None, vocab_size=V, threads=None, init=False, **kw)
    planned = probe.threads
    probe.close()
    S = planned * cfg.get("waves", 1)
    assert S in (planned, 2 * planned)
    if "shards" in cfg:
        assert S == cfg["shards"], (S, cfg["shards"])
    tokens, start, counts, train_words = bench_inputs(S, V)
    first = np.full(S, -1, np.int32)
    resident = cfg.get("resident", True)

    def make(res):
        t = w2b.Trainer(None, vocab_size=V, threads=S, init=False, **kw)
        t.set_vocab_counts(counts, train_words)
        t.set_corpus(tokens, start, first, res)
        return t

    t = make(True)
    recs = traces(t, S, 64)
    if not resident:
        t.close()
        t = make(False)
    info = t.kernel_info()
    got = dict(info, **{k: v for k, v in w2b.warp_plan(size=D, window=W, negative=N, bitlevel=b, reg=reg,
                                                        kernel=kw["kernel"]).items() if k == "sentence_in_smem"})
    assert all(got[k] == v for k, v in cfg["expect"].items()), (cfg["expect"], got)
    t.init_tables()
    trajs = []
    for s in range(S):
        tj = Trajectory(None, recs[s], tokens, W, 0.05, train_words)
        tj.cursor = int(start[s])
        trajs.append(tj)
    steps = [take(tj, 1) for tj in trajs]
    assert all(tj.counter.wca == 0 for tj in trajs), "a shard crosses a learning-rate period inside the step"
    alpha, wca = t.get_state()
    positions = [[(c, g, np.float32(alpha)) for c, g, _ in ps] for ps, _ in steps]
    assert min(len(p) for p in positions) >= 2
    rep_ctx = sum(len(np.unique(c)) < len(c) for p in positions for c, _, _ in p)
    rep_tg = sum(len(np.unique(g)) < len(g) for p in positions for _, g, _ in p)
    assert rep_ctx > 0 and rep_tg > 0, (rep_ctx, rep_tg)
    exptab = t.download_exptable()
    q = quantizer(b, info["warp"] == 1 and not reg and b in (1, 2) and info["bm"] != 9)
    chk = LevelStep(positions, b, q, reg, exptab, model_for(info))
    init_u, init_v = t.download_raw()
    u0, v0 = chk.seed(init_u, init_v, np.random.default_rng(5))
    del init_u, init_v
    t.upload_raw(u0, v0)
    t_seeded = time.time()
    st = t.train_step(1)
    u1, v1 = t.download_raw()
    assert t.get_state() == (alpha, wca)
    t.close()
    assert st["positions"] == sum(len(p) for p in positions), st
    assert st["context_rows"] == sum(len(c) for p in positions for c, _, _ in p), st
    assert st["target_rows"] == sum(len(g) for p in positions for _, g, _ in p), st
    assert st["words"] == sum(w for _, w in steps) and st["shards_done"] == 0, st
    assert np.float32(st["alpha"]) == np.float32(alpha) and st["word_count_actual"] == wca, st
    watch = []  # the hottest rows; under -reg also the hottest with at most 64 and 16 occurrences
    for k in "uv":
        watch.append((k, chk.hot[k]))
        for cap in (64, 16) if reg else ():
            c = [i for i, o in chk.occ[k].items() if o <= cap]
            watch.append((k, max(c, key=lambda i: (chk.occ[k][i], -i))))
    res = chk.check(u0, v0, u1, v1, st["loss"], watch=watch)
    if b == 2:
        lv = np.abs(q(v0[chk.rows["v"]]))
        assert (lv == np.float32(0.25)).any() and (lv == np.float32(0.75)).any()
        assert (lv[chk.index("v", chk.hot["v"])] == np.float32(0.75)).all()

    # controls, against the same result
    rng = np.random.default_rng(17)
    hottest = sorted(((name_, i) for name_ in "uv" for i in chk.rows[name_].tolist()),
                     key=lambda k: -chk.n[k[0]][chk.index(*k)])[:100]
    top = set(hottest)
    onhot = [s for s in range(S) if any(k in top for k in [("v", int(i)) for p in positions[s] for i in p[1]])]
    pick_hot = [int(x) for x in rng.choice(onhot, 4, replace=False)]
    pick_any = [int(x) for x in rng.choice([s for s in range(S) if s not in pick_hot], 4, replace=False)]
    # under -reg a hot row's decays read the row itself: its interval grows with (adds)^2 * reg, past one update
    left_out = [s for s in pick_hot if not chk.fails_with(s, rows=None if reg else top)] + \
               [s for s in pick_any if not chk.fails_with(s)]
    ctl = [next(w for w in watch if w[0] == k and (not reg or chk.resolvable(w) > 1)) for k in "uv"]
    updates = {"%s row %d (%d adds, update/radius %.3g) %s" % (
        k[0], k[1], chk.n[k[0]][chk.index(*k)], chk.resolvable(k), how): chk.update_fails(k, times)
        for k in ctl for how, times in (("dropped", 0), ("doubled", 2))}
    print("hottest rows' largest update / radius: u %.3g, v %.3g" % (chk.resolvable(watch[0]),
                                                                      chk.resolvable(next(w for w in watch if w[0] == "v"))))
    s_n = int(rng.choice([s for s in range(S) if len(positions[s]) >= 2]))
    nb = positions[(s_n + 1) % S]
    neighbour = chk.fails_with(s_n, [(c, g1, a) for (c, _, a), (_, g1, _) in zip(positions[s_n], nb)])
    elapsed = time.time() - t_start
    counts_of = {k: (int(chk.n[k][chk.index(k, chk.hot[k])]), len(chk.users[k][chk.hot[k]])) for k in "uv"}
    print("%s %s: %d shards (planner %d), %d positions (%d with a repeated context id, %d with a repeated target); "
          "hottest u row %d: %d adds from %d shards; hottest v row %d: %d adds from %d shards; worst err/bound u %.3f "
          "v %.3f loss %.3f; margin x%.3g; median |update|/radius on shared elements %.3g; controls failing: "
          "left out %d/8 (4 judged on the 100 hottest rows alone, except under -reg), %s, neighbour's targets %s; seeding %.0f s, case %.0f s" % (
              name, info, S, planned, st["positions"], rep_ctx, rep_tg, chk.hot["u"], *counts_of["u"], chk.hot["v"],
              *counts_of["v"], res["u"], res["v"], res["loss"], res["margin"], res["median_shared"],
              8 - len(left_out), ", ".join("%s %s" % (k, v) for k, v in updates.items()), neighbour,
              t_seeded - t_start, elapsed))
    assert not left_out, ("shards whose removal passes", left_out)
    assert all(updates.values()), updates
    assert neighbour
