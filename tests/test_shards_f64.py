"""One real many-shard training launch, element by element, against a float64 Hogwild replay of every shard's positions.

tests/test_trajectory_f64.py checks one shard per launch.  Here one train_step of many shards at once (the launch
bench.py times: 1584 shards at D = 800 on an H100 SXM) is replayed from the draw traces of every shard:
  * shards are grouped into components, linked by a shared u row (context) or a shared v row (targets);
  * a shard with no link is isolated and is checked exactly as the trajectory test checks one shard: the kernel's
    ordering model, expTable branches and quantization hulls, on its own rows;
  * the shards of a component are replayed under a Hogwild model.  A read of a row other shards also update may
    see, element by element, any prefix of each of their updates to it: the row's interval widens by the hull of
    their running update (its largest positive and negative prefix).  Those hulls come from a fixed point: a pass
    without widening, then passes that widen by the previous pass's hulls, inflated, until every new hull lies inside
    the inflated previous one (else the step is unresolved).  Inside a component g and the warp kernel's
    before/after reads of a repeated target take their hull instead of branching;
  * a shared row's final value must lie in x0 + the sum over its shards of their own update intervals, plus one
    float32 add's rounding per update: every update lands exactly once;
  * rows no shard touched are bit-identical, the loss lies within the sum of the shards' loss intervals, and the
    counters equal the sums over the traces.
No shard crosses a 10 000-word learning-rate period inside a checked step here (asserted from the traces), so every
position trains at the alpha get_state() reports before the step; tests/test_shards_alpha_f64.py checks steps in which
every shard crosses one, or reaches its end, at the alphas w2b_train_step_traced records.

On the CPU a Hogwild executor built on the oracle's single-position step interleaves shards in random order, lands
each update late and shows every read a random element-wise prefix of the other shards' landed updates; it passes the
model, and dropped, doubled and overwritten updates, a shard trained on its neighbour's positions and a lost shard
loss all fail it."""
import ctypes as C
import multiprocessing as mp
import os
from contextlib import nullcontext
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.f64_bounds import TINY, U, quantizer
from tests.test_trajectory_f64 import LOOSE_MAX, Model, Replay, Trajectory, check_step, model_for
from tests.util import bits, zipf_corpus

MAX_PASSES = 10


def inflate(h):
    """The fixed point's inflation of a hull of the previous pass: by a quarter, and by a tenth of the row's largest
    element (an element that hardly moved in one pass may move with the wider reads of the next)."""
    return 1.25 * h + 0.1 * h.max()


# ------------------------------------------------------------------------------------------------ components
def components(rows_u, rows_v):
    """Shards linked by a shared u row or a shared v row: lists of shard indices, the largest first.  A shard that
    shares no row is a list of its own."""
    parent = list(range(len(rows_u)))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    for rows in (rows_u, rows_v):
        owner = {}
        for s, rs in enumerate(rows):
            for i in rs:
                t = owner.setdefault(i, s)
                if t != s:
                    parent[find(s)] = find(t)
    groups = {}
    for s in range(len(rows_u)):
        groups.setdefault(find(s), []).append(s)
    return sorted(groups.values(), key=lambda g: (-len(g), g[0]))


class SharedReplay(Replay):
    """One shard of a component.  `wid[(table, row)]` = (positive, negative) widening of a row other shards update;
    the shard's own updates are kept apart in `own[(table, row)]` = [sum of centres, sum of radii, largest positive
    prefix, largest negative prefix, adds]."""

    def __init__(self, u0, v0, b, q, reg, exptab, model, wid):
        super().__init__(u0, v0, b, q, reg, exptab, model)
        self.hull = True
        self.wid, self.own = wid, {}

    def key(self, T, i):
        return ("u" if T is self.U else "v", i)

    def read(self, T, src, i):
        c, r = super().read(T, src, i)
        w = self.wid.get(self.key(T, i))
        if w is None:
            return [c, r]
        return [c + (w[0] - w[1]) / 2, r + (w[0] + w[1]) / 2]

    def add_to(self, T, i, dc, dr):
        k = self.key(T, i)
        w = self.wid.get(k)
        row = T[i]
        row[0] = row[0] + dc  # the shard's own view: x0 + its own updates; the add rounds the value others widen
        row[1] = row[1] + dr + U * (np.abs(row[0]) + row[1] + (0 if w is None else w[0] + w[1])) + 2 * TINY
        o = self.own.get(k)
        if o is None:
            z = np.zeros(self.D)
            o = self.own[k] = [z, z, z, z, 0]
        o[0], o[1] = o[0] + dc, o[1] + dr
        o[2], o[3] = np.maximum(o[2], o[0] + o[1]), np.maximum(o[3], o[1] - o[0])
        o[4] += 1


class ManyShards:
    """The replay of one many-shard step: `positions[s]` = shard s's positions in order, (ctx, targets, alpha)."""

    def __init__(self, u0, v0, positions, b, q, reg, exptab, model):
        self.u0, self.v0, self.pos = u0, v0, positions
        self.args = (b, q, reg, exptab, model)
        self.rows_u = [set(int(i) for p in ps for i in p[0]) for ps in positions]
        self.rows_v = [set(int(i) for p in ps for i in p[1]) for ps in positions]
        groups = components(self.rows_u, self.rows_v)
        self.isolated = [g[0] for g in groups if len(g) == 1 and positions[g[0]]]
        self.comps = [g for g in groups if len(g) > 1]
        self.table = {"u": u0, "v": v0}
        self.hulls = {}  # shard -> (table, row) -> the inflated hulls its accepted fixed point assumed

    def check(self, u1, v1, loss):
        """Raises AssertionError at the first element outside the replay; returns the summary, or None when a
        component's fixed point or an isolated shard's branches do not resolve."""
        self.after = {"u": u1, "v": v1}
        global _WORKER
        _WORKER = self
        procs = min(32, len(os.sched_getaffinity(0)))
        with mp.get_context("fork").Pool(procs) if procs > 1 else nullcontext() as pool:
            self.map = (lambda f, xs: pool.map(f, xs, chunksize=8)) if pool else (lambda f, xs: list(map(f, xs)))
            try:
                return self._check(u1, v1, loss)
            finally:
                _WORKER = None
                self.map = None

    def _check(self, u1, v1, loss):
        out = dict(u=0.0, v=0.0, upd_iso=[], upd_comp=[], moved=0, loose=0, passes=0)
        lo = hi = 0.0
        self.iso_loss = {}
        for s, res in zip(self.isolated, self.map(_isolated_check, self.isolated)):
            if isinstance(res, str):
                raise AssertionError("isolated shard %d: %s" % (s, res))
            if res is None:
                return None
            out["u"], out["v"] = max(out["u"], res["u"]), max(out["v"], res["v"])
            out["upd_iso"] += res["upd"]
            out["moved"] += res["moved"]
            out["loose"] += res["loose"]
            self.iso_loss[s] = (res["loss_lo"], res["loss_hi"])
            lo, hi = lo + res["loss_lo"], hi + res["loss_hi"]
        self.reps, self.shared = {}, {}
        for g in self.comps:
            fp = self.fixed_point(g)
            if fp is None:
                return None
            reps, shared, passes = fp
            self.reps.update(reps)
            self.shared.update(shared)
            out["passes"] = max(out["passes"], passes)
        for s, r in self.reps.items():
            lr = r.loss_r + 1e-9 * abs(r.loss_c)
            lo, hi = lo + r.loss_c - lr, hi + r.loss_c + lr
        for key, (c, r, before) in self.final_intervals().items():
            after = self.after[key[0]][key[1]].astype(np.float64)
            ratio = np.abs(after - c) / r
            out[key[0]] = max(out[key[0]], float(ratio.max()))
            out["upd_comp"].append(np.abs(after - before) / r)
            if ratio.max() > 1:
                col = int(np.argmax(ratio))
                raise AssertionError("%s row %d column %d (%s): %r, replay %r +- %.3g" % (
                    key[0], key[1], col, "shared by %d shards" % len(self.shared[key]) if key in self.shared else
                    "one shard of a component", after[col], c[col], r[col]))
        touched_u = set().union(*self.rows_u)
        touched_v = set().union(*self.rows_v)
        for name, touched in (("u", touched_u), ("v", touched_v)):
            bad = sorted(set(changed_rows(self.after[name], self.table[name]).tolist()) - touched)
            assert not bad, "%s row %d changed, and no shard touched it" % (name, bad[0])
        mid, half = (lo + hi) / 2, (hi - lo) / 2
        out["loss"] = abs(loss - mid) / half
        assert out["loss"] <= 1, "loss %r outside the shards' sum %r +- %.3g" % (loss, mid, half)
        self.loss_iv = (lo, hi)
        out["median_iso"] = float(np.median(np.concatenate(out["upd_iso"]))) if out["upd_iso"] else None
        out["median_comp"] = float(np.median(np.concatenate(out["upd_comp"]))) if out["upd_comp"] else None
        out["loose_frac"] = out["loose"] / max(out["moved"], 1)
        return out

    def fixed_point(self, shards):
        users = {}
        for s in shards:
            for name, rows in (("u", self.rows_u[s]), ("v", self.rows_v[s])):
                for i in rows:
                    users.setdefault((name, i), []).append(s)
        shared = {k: ss for k, ss in users.items() if len(ss) > 1}
        wid = {s: {} for s in shards}
        prev = None
        for it in range(MAX_PASSES):
            reps = dict(zip(shards, self.map(_shared_replay, [(s, wid[s]) for s in shards])))
            if prev is not None and all(np.all(reps[s].own[k][2] <= prev[s][k][0]) and
                                        np.all(reps[s].own[k][3] <= prev[s][k][1])
                                        for s in shards for k in prev[s]):
                self.hulls.update(prev)
                return reps, shared, it + 1
            # the next pass widens by this pass's hulls, inflated, and by the rounding of the other shards' adds
            prev = {s: {k: (inflate(o[2]), inflate(o[3]), o[4]) for k, o in reps[s].own.items() if k in shared}
                    for s in shards}
            for k, ss in shared.items():
                P = sum(prev[s][k][0] for s in ss)
                N = sum(prev[s][k][1] for s in ss)
                A = sum(prev[s][k][2] for s in ss)
                M = np.abs(self.table[k[0]][k[1]].astype(np.float64)) + P + N
                for s in ss:
                    rnd = (A - prev[s][k][2]) * (1.01 * U * M + 2 * TINY)
                    wid[s][k] = (np.maximum(P - prev[s][k][0], 0) * (1 + 1e-12) + rnd,
                                 np.maximum(N - prev[s][k][1], 0) * (1 + 1e-12) + rnd)
        return None

    def final_intervals(self, without=None):
        """(table, row) -> (centre, radius, value before) of every component row, leaving shard `without` out."""
        out = {}
        for s, r in self.reps.items():
            for name, T in (("u", r.U), ("v", r.V)):
                for i, (c, rad) in T.items():
                    k = (name, i)
                    if k in self.shared or s == without:
                        continue
                    out[k] = (c, rad, self.table[name][i].astype(np.float64))
        for k, ss in self.shared.items():
            x0 = self.table[k[0]][k[1]].astype(np.float64)
            keep = [s for s in ss if s != without]
            c = x0 + sum(self.reps[s].own[k][0] for s in keep)
            r = sum(self.reps[s].own[k][1] for s in keep)
            M = np.abs(x0) + sum(self.hulls[s][k][0] + self.hulls[s][k][1] for s in ss)
            A = sum(self.reps[s].own[k][4] for s in keep)
            out[k] = (c, r + A * (1.01 * U * M + 2 * TINY), x0)
        return out

    def fails_without(self, s, loss):
        """True when the step, replayed without shard s's positions, fails: a row s alone touched changed, a shared
        row is outside the other shards' sum, or the loss is outside the other shards' intervals."""
        mine = [("u", i) for i in self.rows_u[s]] + [("v", i) for i in self.rows_v[s]]
        iv = self.final_intervals(without=s) if s in self.reps else {}
        for k in mine:
            after = self.after[k[0]][k[1]]
            if k in iv:
                c, r, _ = iv[k]
                if np.any(np.abs(after.astype(np.float64) - c) > r):
                    return True
            elif not np.array_equal(bits(after), bits(self.table[k[0]][k[1]])):
                return True
        if s in self.reps:
            r = self.reps[s]
            lr = r.loss_r + 1e-9 * abs(r.loss_c)
            slo, shi = r.loss_c - lr, r.loss_c + lr
        else:
            slo, shi = self.iso_loss[s]
        return not (self.loss_iv[0] - slo <= loss <= self.loss_iv[1] - shi)

    def leave_one_out(self, loss, n=8, from_largest=4, seed=0):
        rng = np.random.default_rng(seed)
        big = list(self.comps[0]) if self.comps else []
        pick = [int(x) for x in rng.choice(big, min(from_largest, len(big)), replace=False)] if big else []
        rest = [s for s in self.isolated + [x for g in self.comps for x in g] if s not in pick]
        pick += [int(x) for x in rng.choice(rest, min(n - len(pick), len(rest)), replace=False)]
        return pick, [s for s in pick if not self.fails_without(s, loss)]


# The shards of one pass, and the isolated shards, are replayed in forked worker processes that read the tables of
# the ManyShards being checked from _WORKER; they return only what the check uses, never the tables.
_WORKER = None


def _isolated_check(s):
    m = _WORKER
    try:
        return check_step(m.u0, m.v0, m.after["u"], m.after["v"], None, m.pos[s], *m.args)
    except AssertionError as e:
        return str(e)


def _shared_replay(job):
    s, wid = job
    m = _WORKER
    r = SharedReplay(m.u0, m.v0, *m.args, wid=wid)
    for ctx, tg, a in m.pos[s]:
        r.position(ctx, tg, a)
    return SimpleNamespace(own=r.own, U=r.U, V=r.V, loss_c=r.loss_c, loss_r=r.loss_r)


def changed_rows(after, before, chunk=1 << 16):
    out = []
    for a in range(0, len(after), chunk):
        ne = (bits(after[a:a + chunk]) != bits(before[a:a + chunk])).any(1)
        out.append(np.flatnonzero(ne) + a)
    return np.concatenate(out) if out else np.zeros(0, np.int64)


# ----------------------------------------------------------------------------------------- the CPU: an executor
class HogwildExecutor:
    """Shards' positions run through the oracle's single-position step (w2bo_apply_position) in a seeded random
    interleaving.  Each position's update of a row lands in the shared table later, at a random time; a shard's own
    updates land before its next position reads.  Every read of a row sees, element by element, a random prefix of
    each other shard's landed updates to it."""

    def __init__(self, o, D, W, N, b, reg, u0, v0):
        self.m = po.OracleModel(o, D, W, N, b, reg=reg, table=np.zeros(1, np.int32))
        self.ex = po.exptable()
        self.u0, self.v0 = u0, v0

    def run(self, positions, seed, corrupt=None, log=None):
        """Returns (u, v, loss per shard).  corrupt = (kind, landing index): "drop" skips that landing, "twice"
        applies it twice, "overwrite" stores it on the value before the previous landing (a plain load/add/store
        race losing the other shard's update).  `log` collects (row key, shard, max |update|, previous shard)."""
        rng = np.random.default_rng(seed)
        T = {"u": self.u0.copy(), "v": self.v0.copy()}
        landed = {}   # key -> [(shard, update)] in landing order
        before_last = {}
        pending = []  # (time, sequence, shard, key, update)
        order = rng.permutation(np.repeat(np.arange(len(positions)), [len(p) for p in positions]))
        nxt = [0] * len(positions)
        losses = np.zeros(len(positions))
        n_landed = [0]

        def land(p):
            _, _, s, key, d = p
            j = n_landed[0]
            n_landed[0] += 1
            prev, prev_d = landed.get(key, [(None, np.zeros(1))])[-1]
            if log is not None:
                log.append((key, s, float(np.abs(d).max()), prev, float(np.abs(prev_d).max())))
            row = T[key[0]][key[1]]
            kind = corrupt[0] if corrupt and corrupt[1] == j else None
            if kind == "drop":
                return
            old = row.copy()
            if kind == "overwrite":
                row[...] = before_last[key] + d
            else:
                row[...] = row + d
                if kind == "twice":
                    row[...] = row + d
            before_last[key] = old
            landed.setdefault(key, []).append((s, d))

        for tick, s in enumerate(order.tolist()):
            due = sorted((p for p in pending if p[0] <= tick or p[2] == s), key=lambda p: (p[0], p[1]))
            for p in due:
                land(p)
            pending = [p for p in pending if not (p[0] <= tick or p[2] == s)]
            ctx, tg, a = positions[s][nxt[s]]
            nxt[s] += 1
            views = {}
            for name, ids in (("u", ctx), ("v", tg)):
                for i in set(int(x) for x in ids):
                    views[(name, i)] = self.view((name, i), s, landed, rng)
                    getattr(self.m, name)[i] = views[(name, i)]
            self.m.m.alpha = a
            f = np.zeros(max(len(tg), 1), np.float32)
            loss = C.c_double()
            po.lib().w2bo_apply_position(C.byref(self.m.m), self.ex, ctx, len(ctx), tg, len(tg), f, C.byref(loss))
            losses[s] += loss.value
            for key, x in views.items():
                d = getattr(self.m, key[0])[key[1]] - x  # float32: the row's update as the position stores it
                pending.append((tick + int(rng.integers(1, 12)), len(pending) + tick * 4096, s, key, d))
        for p in sorted(pending, key=lambda p: (p[0], p[1])):
            land(p)
        return T["u"], T["v"], losses

    def view(self, key, s, landed, rng):
        x = (self.u0 if key[0] == "u" else self.v0)[key[1]].copy()
        seen = {}
        for t, d in landed.get(key, []):
            seen[t] = seen.get(t, 0) + 1
        cut = {t: rng.integers(0, n + 1, x.shape) for t, n in seen.items() if t != s}
        k = {}
        for t, d in landed.get(key, []):
            j = k.get(t, 0)
            k[t] = j + 1
            x = x + d if t == s else np.where(j < cut[t], x + d, x).astype(np.float32)
        return x


@pytest.fixture(scope="module")
def shard_corpus(tmp_path_factory):
    path = zipf_corpus(str(tmp_path_factory.mktemp("shards") / "z.txt"), 20000, 5000, seed=41, newline_every=12)
    return po.Corpus(path, 1)


def synthetic_positions(shards, per_shard, N, V, seed, pool=400, shared_ctx=0.3):
    """Positions of `shards` shards shaped like the sparse GPU corpus: context rows (repeats included) and centres
    from each shard's own block of ids, with probability `shared_ctx` one of 8 context rows a few shards share, and
    negatives drawn from the last `pool` ids, so that rows are shared by a few shards, not by all."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(shards):
        own = 1 + 16 * s + np.arange(16)
        ps = []
        for p in range(per_shard):
            ctx = rng.choice(own[:8], int(rng.integers(1, 9)))
            if rng.random() < shared_ctx:
                ctx[-1] = V - pool - 1 - rng.integers(0, 8)
            tg = np.concatenate([[own[8 + p % 8]], rng.integers(V - pool, V, N)])
            ps.append((ctx.astype(np.int32), tg.astype(np.int32), np.float32(0.05)))
        out.append(ps)
    return out


def seeded_rows(V, D, seed, cw=10):
    """Random tables whose f covers the expTable range with about `cw` context rows (tests/test_trajectory_f64.py
    seeded_tables at cw = 10)."""
    s = float(np.clip(np.sqrt(9 * np.sqrt(cw) / np.sqrt(D)), 0.3, 5.0))
    rng = np.random.default_rng(seed)
    return rng.uniform(-s, s, (V, D)).astype(np.float32), rng.uniform(-s, s, (V, D)).astype(np.float32)


EXECUTOR_SHAPES = [  # D, window, negative, bit level, reg, model
    (64, 5, 12, 0, 0.0, "seq"), (64, 5, 12, 1, 0.002, "seq"), (48, 5, 6, 2, 0.0, "seq"),
    (32, 5, 8, 0, 0.002, "register-g9"),
]


def executor_case(shard_corpus, shape, shards=10, per_shard=4):
    D, W, N, b, reg, kind = shape
    pos = synthetic_positions(shards, per_shard, N, shard_corpus.vocab_size, 0, pool=3000, shared_ctx=0.0)
    model = Model("seq")
    if kind == "register-g9":  # the register kernel reads a group's rows before its updates: the oracle does so
        model = Model("register", G=9, vec=1, threads=32)  # when no group repeats a target
        pos = [[p for p in ps if len(np.unique(p[1][:9])) == len(p[1][:9])] for ps in pos]
    u0, v0 = seeded_rows(shard_corpus.vocab_size, D, 5)
    ex = HogwildExecutor(shard_corpus, D, W, N, b, reg, u0, v0)
    return ex, pos, ManyShards(u0, v0, pos, b, quantizer(b, False), reg, ex.ex, model)


@pytest.mark.parametrize("shape", EXECUTOR_SHAPES, ids=lambda s: "D%d-W%d-N%d-b%d-reg%g-%s" % s)
def test_hogwild_executor_within_the_model(shape, shard_corpus):
    """The executor's interleavings, late landings and partial reads stay inside the Hogwild replay."""
    ex, pos, chk = executor_case(shard_corpus, shape)
    assert chk.comps and len(chk.comps[0]) >= 3
    for seed in range(3):
        u1, v1, losses = ex.run(pos, seed)
        res = chk.check(u1, v1, float(losses.sum()))
        assert res is not None, "unresolved"
        print(shape, "seed", seed, "worst u %.3f v %.3f loss %.3f; median |update|/radius %.3g; %d passes" % (
            res["u"], res["v"], res["loss"], res["median_comp"], res["passes"]))
        assert len(chk.shared) >= 10
        pick, passed = chk.leave_one_out(float(losses.sum()), n=4, from_largest=4)
        assert not passed, passed


CORRUPTIONS = ["drop", "twice", "overwrite", "neighbour_positions", "loss_left_out"]


@pytest.mark.parametrize("kind", CORRUPTIONS)
def test_hogwild_corruptions_fail(kind, shard_corpus):
    """One update of a shared row dropped, applied twice or lost to a load/add/store race; a shard trained on its
    neighbour's positions; one shard's loss left out: each fails the replay."""
    ex, pos, chk = executor_case(shard_corpus, EXECUTOR_SHAPES[0])
    log = []
    u1, v1, losses = ex.run(pos, 7, log=log)
    assert chk.check(u1, v1, float(losses.sum())) is not None
    if kind in ("drop", "twice", "overwrite"):
        # the update of a shared row largest against the row's radius; for the race, the other shard's update that
        # the store right after it loses
        iv = chk.final_intervals()
        cand = [((pm if kind == "overwrite" else m) / iv[k][1].max(), j) for j, (k, s, m, prev, pm) in enumerate(log)
                if k in chk.shared and (kind != "overwrite" or (prev is not None and prev != s))]
        j = max(cand)[1]
        u1, v1, losses = ex.run(pos, 7, corrupt=(kind, j))
    elif kind == "neighbour_positions":
        # shard s trains shard s + 1's sentence (context rows and centre) with its own negative draws: its random
        # state is its own.  (Rotating whole positions would only hand the same updates to other shards.)
        shifted = [[(c1, np.concatenate([t1[:1], t0[1:]]), a) for (_, t0, a), (c1, t1, _) in
                    zip(pos[s], pos[(s + 1) % len(pos)])] for s in range(len(pos))]
        u1, v1, losses = ex.run(shifted, 7)
    else:
        losses[2] = 0.0
    with pytest.raises(AssertionError) as e:
        chk.check(u1, v1, float(losses.sum()))
    print(kind, str(e.value)[:200])


def test_components():
    """Shards linked through a chain of shared rows form one component, whichever table links them."""
    rows_u = [{1, 2}, {3}, {2}, {7}, set(), {9}]
    rows_v = [{10}, {11, 12}, {13}, {12}, {14}, {15, 10}]
    assert components(rows_u, rows_v) == [[0, 2, 5], [1, 3], [4]]
    assert components([{1}, {2}], [{3}, {4}]) == [[0], [1]]


# ------------------------------------------------------------------------------------------------------ the GPU
def sparse_inputs(shards, L, V):
    """V words with equal counts; shard s starts with one L-word sentence of its own ids 1 + s*L .. (s+1)*L."""
    ids = np.arange(1, shards * L + 1, dtype=np.int32).reshape(shards, L)
    tokens = np.concatenate([ids, np.zeros((shards, 1), np.int32)], 1).ravel()
    tail = np.tile(np.concatenate([np.arange(V - L, V, dtype=np.int32), [0]]), 4)
    tokens = np.concatenate([tokens, tail])
    start = np.arange(shards, dtype=np.int64) * (L + 1)
    counts = np.full(V, 1000, np.int64)
    return tokens, start, counts, int(counts.sum())


def dense_inputs(shards, sentences, V=5000, L=12, seed=3):
    """Zipf(1) words over V - 1 ids, L-word sentences; shard s owns `sentences` sentences."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, V)
    ids = rng.choice(V - 1, size=(shards * sentences, L), p=p / p.sum()).astype(np.int32) + 1
    tokens = np.concatenate([ids, np.zeros((len(ids), 1), np.int32)], 1).ravel()
    start = np.arange(shards, dtype=np.int64) * sentences * (L + 1)
    counts = np.bincount(tokens, minlength=V).astype(np.int64)
    return tokens, start, counts, int(counts.sum())


GPU_CASES = {  # name -> configuration; "expect" is the instantiation and geometry the case is written for
    "bench": dict(corpus="sparse", D=800, W=10, N=24, b=1, reg=0.0, L=2,
                  expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=1584),
    "bench-streamed": dict(corpus="sparse", D=800, W=10, N=24, b=1, reg=0.0, L=2, resident=False,
                           expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=1584),
    "bench-two-waves": dict(corpus="sparse", D=800, W=10, N=24, b=1, reg=0.0, L=2, waves=2,
                            expect={"warp": 1, "nj": 7, "minb": 12, "bm": 1}, shards=3168),
    "bench-reg": dict(corpus="sparse", D=800, W=10, N=24, b=1, reg=0.002, L=2,
                      expect={"warp": 1, "nj": 7, "minb": 8, "reg": 1}),
    "window200": dict(corpus="sparse", D=256, W=200, N=2, b=1, reg=0.0, L=12,
                      expect={"warp": 1, "sentence_in_smem": 0}),
    "register-tuned": dict(corpus="sparse", D=512, W=5, N=8, b=1, reg=0.0, L=2, kernel=1,
                           expect={"warp": 0, "wide": 0, "vec": 4, "group": 9}),
    "register-wide": dict(corpus="sparse", D=4096, W=5, N=12, b=1, reg=0.0, L=2, V=200_001,
                          expect={"warp": 0, "wide": 1, "vec": 4}),
    "dense-period": dict(corpus="dense", D=400, W=10, N=24, b=0, reg=0.0, threads=132, warmup=10001,
                         expect={"warp": 1, "minb": 16}),
}


def traces(t, shards, iters):
    return [t.trace(s, max_iterations=iters, cap=iters) for s in range(shards)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_CASES))
def test_many_shard_step_within_hogwild_f64_bounds(name):
    w2b = pytest.importorskip("word2bits_b200")
    cfg = GPU_CASES[name]
    D, W, N, b, reg = cfg["D"], cfg["W"], cfg["N"], cfg["b"], cfg["reg"]
    kw = dict(size=D, window=W, negative=N, bitlevel=b, reg=reg, iter=1, kernel=cfg.get("kernel", 0))
    V = cfg.get("V", 2_000_001) if cfg["corpus"] == "sparse" else 5000
    S = cfg.get("threads")
    if S is None:
        probe = w2b.Trainer(None, vocab_size=V, threads=None, init=False, **kw)
        S = probe.threads * cfg.get("waves", 1)
        probe.close()
    if "shards" in cfg:
        assert S == cfg["shards"], (S, cfg["shards"])
    warmup = cfg.get("warmup", 0)
    if cfg["corpus"] == "sparse":
        tokens, start, counts, train_words = sparse_inputs(S, cfg["L"], V)
    else:
        tokens, start, counts, train_words = dense_inputs(S, (warmup + 60) // 13 + 4)
    first = np.full(S, -1, np.int32)
    resident = cfg.get("resident", True)

    def make(res):
        t = w2b.Trainer(None, vocab_size=V, threads=S, init=False, **kw)
        t.set_vocab_counts(counts, train_words)
        t.set_corpus(tokens, start, first, res)
        return t

    iters = warmup + 64 + 2 * cfg.get("L", 12)
    if resident:
        t = make(True)
        recs = traces(t, S, iters)
    else:
        tr = make(True)
        recs = traces(tr, S, iters)
        tr.close()
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

    def take(tj, words):
        pos, w = [], 0
        while w < words:
            pos += tj.next_positions()
            w += tj.advance()
        return pos, w

    if warmup:  # every shard crosses the 10 000-word period once; word_count_actual is the sum of the crossings
        for tj in trajs:
            take(tj, warmup)
            assert tj.counter.wca > 0
        st = t.train_step(warmup)
        assert st["word_count_actual"] == sum(tj.counter.wca for tj in trajs) and st["shards_done"] == 0, st
    u0, v0 = t.download_raw()
    wca0 = [tj.counter.wca for tj in trajs]
    steps = [take(tj, 1) for tj in trajs]
    assert [tj.counter.wca for tj in trajs] == wca0, "a shard crosses a learning-rate period inside the step"
    if cfg["corpus"] == "sparse":  # seeded values on every row a shard touches, so that f covers the expTable
        ru = np.array(sorted({int(i) for ps, _ in steps for p in ps for i in p[0]}))
        rv = np.array(sorted({int(i) for ps, _ in steps for p in ps for i in p[1]}))
        su, sv = seeded_rows(max(len(ru), len(rv)), D, 11, cw=cfg["L"] - 1)
        u0[ru], v0[rv] = su[:len(ru)], sv[:len(rv)]
        t.upload_raw(u0, v0)
    alpha, wca = t.get_state()
    positions = [[(c, g, np.float32(alpha)) for c, g, _ in ps] for ps, _ in steps]
    st = t.train_step(1)
    u1, v1 = t.download_raw()
    assert t.get_state() == (alpha, wca)
    exptab = t.download_exptable()
    t.close()
    assert st["positions"] == sum(len(p) for p in positions), st
    assert st["context_rows"] == sum(len(c) for p in positions for c, _, _ in p), st
    assert st["target_rows"] == sum(len(g) for p in positions for _, g, _ in p), st
    assert st["words"] == sum(w for _, w in steps) and st["shards_done"] == 0, st
    assert np.float32(st["alpha"]) == np.float32(alpha) and st["word_count_actual"] == wca, st
    q = quantizer(b, info["warp"] == 1 and not reg and b in (1, 2) and info["bm"] != 9)
    chk = ManyShards(u0, v0, positions, b, q, reg, exptab, model_for(info))
    res = chk.check(u1, v1, st["loss"])
    assert res is not None, "unresolved"
    pick, passed = chk.leave_one_out(st["loss"])
    biggest = len(chk.comps[0]) if chk.comps else 0
    print("%s %s: %d shards, %d isolated, largest component %d (%d components); worst err/bound u %.3f v %.3f "
          "loss %.3f; median |update|/radius isolated %s, component %s; radius above the update at %.2g of the "
          "isolated shards' moved elements; fixed point in %d passes; %d/%d shards left out fail" % (
              name, info, S, len(chk.isolated), biggest, len(chk.comps), res["u"], res["v"], res["loss"],
              "%.3g" % res["median_iso"] if res["median_iso"] is not None else "-",
              "%.3g" % res["median_comp"] if res["median_comp"] is not None else "-", res["loose_frac"],
              res["passes"], len(pick) - len(passed), len(pick)))
    assert len(pick) >= 8 and not passed, ("shards whose removal passes", passed)
    if chk.isolated:
        assert res["median_iso"] >= 1e3 and res["loose_frac"] <= LOOSE_MAX, res
