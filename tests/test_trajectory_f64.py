"""Whole training steps, element by element, against a float64 replay of the step's positions.

A single shard (threads=1, prefetch=0) trains one sentence per train_step(1).  After each step every element of u and
v, the step's loss and its counters are checked against a float64 replay that starts from the tables as they were
before the step and walks the step's positions (taken from the draw trace, which test_draw_trace_bit_exact pins to
the oracle's).  Each element of the replay carries an error radius: every float32 operation adds the gamma_h bound of
tests/f64_bounds.py (h = the depth of the kernel's own summation tree), errors carried in from earlier positions of
the step propagate to first order, and flushed denormals add their allowance.  Where the radius of a row that is
read again straddles a quantization level, the quantized value takes the hull of the two levels (with rigorous bounds
most steps at D = 800 hold such a read, so leaving those steps unchecked would check few).  Where f's interval
straddles an expTable slot or a saturation branch, every value of g is followed as a branch; a branch dies as soon as
a row whose last update in the step is done leaves its interval, which is normally its own target row.  A step is
unresolved (only its counters are checked) when more than 16 branches are alive at once.

What each kernel may do inside a position is modelled exactly and no more:
  * oracle and strict mode: the reference order (:431-503);
  * register kernel, fast mode: targets in groups of G; every row of a group is read before any of its updates,
    later groups see earlier groups' updates; a repeated context row is updated occurrence after occurrence, each
    -reg decay from the row as that occurrence reads it;
  * warp kernel, serial: a target id that occurs again in the same position may read its row before or after each
    earlier occurrence's update (both are followed, and one must hold every element); with -reg a repeated context row's later reads may or may not see the earlier occurrences' decay (an
    interval, not a branch); everything of position p has landed before p+1 is read.

The checker is shown not to be vacuous on the CPU: the oracle passes it under the sequential model; the warp kernel's
own source, emulated with late and shuffled completion of its bulk copies, passes the warp model with repeated targets
seen reading both before and after an earlier update, and fails it when the ring prefetches across positions;
corrupted oracle trajectories fail it."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.f64_bounds import SUB, TINY, U, gamma, grad_scalar, quantizer
from tests.util import bits, zipf_corpus

MAX_BRANCHES = 16
# At most this fraction of the elements a step moves may have a radius above their update.  Measured on an H100: up
# to 0.15 (warp kernel, D = 2048, b = 1: the most quantized reads straddling a level), 0.06 with b = 0.
LOOSE_MAX = 0.2
LOG_1E9 = float(np.log(np.float32(1e-9)))


# ------------------------------------------------------------------------------------------------ trace -> steps
def split_sentences(recs, W):
    """The draw trace cut into sentences: [(first record, number of records, kept-word ids)].  A sentence of L kept
    words has L records (one with center -1 when L = 0); its last record is the first whose cw has no right
    neighbour (a = W + 1 is always inside the shrunk window because b < W).  A sentence the end of the trace cuts
    off is left out."""
    out, i = [], 0
    while i < len(recs):
        if recs[i][0] < 0:
            out.append((i, 1, []))
            i += 1
            continue
        L = 1
        while True:
            if i + L > len(recs):
                return out
            b, cw = recs[i + L - 1][1], recs[i + L - 1][2]
            if cw == len([a for a in range(b, 2 * W + 1 - b) if a < W and L - 1 - W + a >= 0]):
                break
            L += 1
        out.append((i, L, [r[0] for r in recs[i:i + L]]))
        i += L
    return out


def sentence_positions(recs, first, L, sen, W):
    """(context ids in the kernels' order, targets, alpha) of the trained records (cw > 0) of one sentence."""
    pos = []
    for sp in range(L):
        center, b, cw, tg, alpha = recs[first + sp]
        ctx = [sen[sp - W + a] for a in range(b, 2 * W + 1 - b) if a != W and 0 <= sp - W + a < L]
        assert len(ctx) == cw and (cw == 0 or tg[0] == center), (first, sp)
        if cw:
            pos.append((np.array(ctx, np.int32), np.array(tg, np.int32), alpha))
    return pos


def sentence_words(tokens, cursor):
    """Words a sentence read from `cursor` consumes: up to and including the next </s> (:394-413)."""
    z = np.flatnonzero(tokens[cursor:] == 0)
    return int(z[0]) + 1 if len(z) else len(tokens) - cursor


class Counter:
    """word_count_actual and alpha of one shard, updated where the kernels update them (:379-393)."""

    def __init__(self, alpha0, train_words, iters=1):
        self.a0, self.denom = np.float32(alpha0), np.float32(iters * train_words + 1)
        self.wc = self.last = self.wca = 0
        self.alpha = self.a0

    def sentence(self, words):
        self.wc += words
        if self.wc - self.last > 10000:
            self.wca += self.wc - self.last
            self.last = self.wc
            a = np.float32(self.a0 * np.float32(np.float32(1) - np.float32(np.float32(self.wca) / self.denom)))
            self.alpha = max(a, np.float32(float(self.a0) * 1e-4))


# ------------------------------------------------------------------------------------------------- the model
class Model:
    """Ordering model of a kernel: kind "seq" (oracle, strict), "register" (group G, `threads` threads of `vec`
    columns) or "warp" (`nj` float4 column groups per lane)."""

    def __init__(self, kind, G=1, vec=1, threads=32, nj=1):
        self.kind, self.G, self.vec, self.threads, self.nj = kind, G, vec, threads, nj

    def f_rounding(self, avg, qc, A, Q):
        """Bound on the rounding error of f = sum(avg * q) in the kernel's own summation tree: the running error bound
        u * (sum of |every intermediate sum|) (a fused multiply-add rounds once), with the inputs' radii added to
        every magnitude.  seq: column order (:464-470).  register: each thread's vec columns by fma, a 32-lane
        butterfly, the warps' partial sums in order.  warp: per lane four fma chains (float4 components) over the nj
        column groups, (x + y) + (z + w), a 32-lane butterfly."""
        p = avg * qc
        pr = A * Q - np.abs(p)
        mag = np.abs(p) + pr
        if self.kind == "seq":
            nodes = [mag, np.abs(np.cumsum(p)) + np.cumsum(pr)]
        else:
            lanes = self.threads if self.kind == "register" else 32
            per = self.vec if self.kind == "register" else 4 * self.nj
            n = lanes * per
            P, M = np.zeros(n), np.zeros(n)
            P[:len(p)], M[:len(p)] = p, mag
            if self.kind == "register":  # [warp, lane, column of the thread]
                P, M = P.reshape(lanes // 32, 32, per), M.reshape(lanes // 32, 32, per)
                chain_p, chain_m = np.cumsum(P, 2), np.cumsum(M, 2)
                nodes = [np.abs(chain_p) + chain_m]
                xp, xm = chain_p[:, :, -1], chain_m[:, :, -1]
            else:  # [column group, lane, component]
                P, M = P.reshape(self.nj, 32, 4), M.reshape(self.nj, 32, 4)
                chain_p, chain_m = np.cumsum(P, 0), np.cumsum(M, 0)
                nodes = [np.abs(chain_p) + chain_m]
                cp, cm = chain_p[-1], chain_m[-1]
                s01, s23 = cp[:, 0] + cp[:, 1], cp[:, 2] + cp[:, 3]
                m01, m23 = cm[:, 0] + cm[:, 1], cm[:, 2] + cm[:, 3]
                nodes += [np.abs(s01) + m01, np.abs(s23) + m23]
                xp, xm = (s01 + s23)[None, :], (m01 + m23)[None, :]
                nodes.append(np.abs(xp) + xm)
            for o in (16, 8, 4, 2, 1):  # butterfly: after the step of stride o, lanes 0 .. o-1 hold the distinct sums
                perm = np.arange(32) ^ o
                xp, xm = xp + xp[:, perm], xm + xm[:, perm]
                nodes.append(np.abs(xp[:, :o]) + xm[:, :o])
            if self.kind == "register":  # the warps' partials, in order
                nodes.append(np.abs(np.cumsum(xp[:, 0])) + np.cumsum(xm[:, 0]))
        return 1.01 * U * float(sum(x.sum() for x in nodes)) + 64 * len(p) * SUB


def model_for(info):
    if info["warp"]:
        return Model("warp", nj=info["nj"])
    return Model("register", G=info["group"], vec=info["vec"], threads=info["threads"])


def qinterval(q, c, r):
    """Quantized values at the float32 ends of [c - r, c + r] (float64 arrays).  quantize is monotone, so where they
    are equal that level holds everywhere inside, and otherwise every value inside lies between them."""
    if not r.any():
        ql = q(c.astype(np.float32))
        return ql, ql
    exact = r == 0
    lo = np.where(exact, c, np.nextafter((c - r).astype(np.float32), np.float32(-np.inf))).astype(np.float32)
    hi = np.where(exact, c, np.nextafter((c + r).astype(np.float32), np.float32(np.inf))).astype(np.float32)
    ql, qh = q(lo), q(hi)
    return ql, qh


class NeedChoice(Exception):
    def __init__(self, n):
        self.n = n


def g_candidates(fc, fr, label, alpha, exptab):
    """The values g (:473-475) takes for the float32 f in fc +- fr: one per expTable slot and saturation branch."""
    lo = np.nextafter(np.float32(fc - fr), np.float32(-np.inf))
    hi = np.nextafter(np.float32(fc + fr), np.float32(np.inf))
    vals = {float(grad_scalar(lo, label, alpha, exptab)), float(grad_scalar(hi, label, alpha, exptab))}
    a, b = max(lo, np.float32(-6)), min(hi, np.float32(6))
    if a <= b:
        slot = lambda f: int(np.float32(np.float32(f + np.float32(6)) * np.float32(83)))
        for k in range(slot(a), min(slot(b), slot(a) + 8) + 1):
            vals.add(float(np.float32(np.float32(np.float32(label) - exptab[k]) * np.float32(alpha))))
    return sorted(vals)


class Replay:
    """Float64 centres and radii of every row a step touches, from the tables before the step.  Where the kernel's
    outcome has more than one admissible value (g of an f that straddles a slot, a warp-kernel target that may or may
    not see an earlier occurrence's update) the replay asks for a choice (NeedChoice) and check_step follows each."""

    def __init__(self, u0, v0, b, q, reg, exptab, model):
        self.u0, self.v0, self.b, self.q, self.reg, self.ex, self.m = u0, v0, b, q, np.float32(reg), exptab, model
        self.U, self.V = {}, {}
        self.loss_c = self.loss_r = 0.0
        self.straddles = 0  # quantized reads whose interval held two levels
        self.choices, self.k, self.g_choices = [], 0, 0
        self.dup_taken = []  # warp kernel: 1 = a repeated target read its row after an earlier occurrence's update
        self.moved = True  # the last position changed something
        self.D = u0.shape[1]
        self.hull = False  # take the hull of every admissible outcome instead of asking for a choice

    def copy(self, choices):
        c = object.__new__(Replay)
        c.__dict__.update(self.__dict__)
        c.U = {i: list(x) for i, x in self.U.items()}  # rows are replaced, never modified in place
        c.V = {i: list(x) for i, x in self.V.items()}
        c.choices, c.k, c.g_choices = choices, 0, 0
        c.dup_taken = list(self.dup_taken)
        return c

    def choose(self, n):
        if self.k < len(self.choices):
            self.k += 1
            return self.choices[self.k - 1]
        raise NeedChoice(n)

    def row(self, T, src, i):
        if i not in T:
            T[i] = [src[i].astype(np.float64), np.zeros(self.D)]
        return T[i]

    def read(self, T, src, i):
        """Row i as a position reads it: [centre, radius] copies."""
        return [x.copy() for x in self.row(T, src, i)]

    def quant(self, c, r):
        """Quantized values of the interval c +- r: the level, or where the interval holds two levels their hull."""
        if self.b == 0:
            return c, r
        ql, qh = qinterval(self.q, c, r)
        ql, qh = ql.astype(np.float64), qh.astype(np.float64)
        self.straddles += int((ql != qh).sum())
        return (ql + qh) / 2, np.abs(qh - ql) / 2

    def add_to(self, T, i, dc, dr):
        """Row i of T += d as one rounded add (flushing denormal inputs and results)."""
        row = T[i]
        row[0] = row[0] + dc
        row[1] = row[1] + dr + U * (np.abs(row[0]) + row[1]) + 2 * TINY

    def position(self, ctx, tg, alpha):
        m, D = self.m, self.D
        alpha = np.float32(alpha)
        d = float(np.float32(np.float32(2 * alpha) * self.reg))
        cw, nt = len(ctx), len(tg)
        # ---- context rows (:431-449)
        pre = {i: self.read(self.U, self.u0, i) for i in set(ctx.tolist())}
        seen = {}
        qs_c, qs_r = np.zeros(D), np.zeros(D)
        s32, exact = np.zeros(D, np.float32), True  # every kernel sums the context rows in order, in float32
        partial = np.zeros(D)  # sum over the context rows of |running sum| (+ radii): the sum's running error bound
        for i in ctx.tolist():
            c, r = pre[i]
            j = seen.get(i, 0)
            if m.kind == "warp" and d:  # earlier occurrences' decays may or may not have landed
                r = r + j * (d * (np.abs(c) + r) + gamma(2) * np.abs(c))
            seen[i] = j + 1
            qc, qr = self.quant(c, r)
            exact = exact and not qr.any()
            s32 = s32 + qc.astype(np.float32)
            qs_c += qc
            qs_r += qr
            partial += np.abs(qs_c) + qs_r
            if self.reg:
                sq = qc * qc
                self.loss_c -= float(self.reg) * sq.sum()
                self.loss_r += float(self.reg) * ((2 * np.abs(qc) * qr + qr * qr).sum() + gamma(D + 8) * (sq + 2 * np.abs(qc) * qr + qr * qr).sum())
            if m.kind == "warp" and d:  # the decay is scattered when the row is read
                self.add_to(self.U, i, -d * c, d * r + gamma(2) * d * (np.abs(c) + r))
        if exact:  # exact inputs: the float32 average itself (:449, IEEE division in every kernel)
            avg, r_avg = (s32 / np.float32(cw)).astype(np.float64), np.zeros(D)
        else:
            avg = qs_c / cw
            r_avg = qs_r / cw + 1.01 * U * (partial / cw + np.abs(avg) + qs_r / cw) + 2 * SUB
        A = np.abs(avg) + r_avg
        # ---- targets (:450-492)
        moved = d != 0
        e_c, e_r, e_abs = np.zeros(D), np.zeros(D), np.zeros(D)
        snap = None
        deltas = {}  # warp: target id -> [(occurrence index, centre, radius) of its updates in this position]
        vpre = {}
        for t in range(nt):
            i = int(tg[t])
            if m.kind == "register" and t % m.G == 0:
                snap = {int(k): self.read(self.V, self.v0, int(k)) for k in tg[t:t + m.G]}
            if m.kind == "register":
                xc, xr = snap[i]
            elif m.kind == "warp":
                if i not in vpre:
                    vpre[i] = self.read(self.V, self.v0, i)
                xc, xr = vpre[i][0].copy(), vpre[i][1].copy()
                for (_, dc, dr) in deltas.get(i, []):
                    if self.hull:  # before or after the earlier occurrence's update
                        xc, xr = xc + dc / 2, xr + np.abs(dc) / 2 + dr
                        continue
                    self.dup_taken.append(self.choose(2))
                    if self.dup_taken[-1]:
                        xc += dc
                        xr = xr + dr
            else:
                xc, xr = self.read(self.V, self.v0, i)
            qc, qr = self.quant(xc, xr)
            Q = np.abs(qc) + qr
            fc = float(avg @ qc)
            fr = float(np.abs(qc) @ r_avg + np.abs(avg) @ qr + r_avg @ qr) + m.f_rounding(avg, qc, A, Q)
            label = int(t == 0)
            gs = g_candidates(fc, fr, label, alpha, self.ex)
            if len(gs) == 1:
                gc, gr = gs[0], 0.0
            elif not self.hull and len(gs) <= 3 and self.g_choices < 3:
                self.g_choices += 1
                gc, gr = gs[self.choose(len(gs))], 0.0
            else:  # f too uncertain, or too many such targets in the position to follow each: the hull of the values
                gc, gr = (gs[0] + gs[-1]) / 2, (gs[-1] - gs[0]) / 2
            moved = moved or gc != 0 or gr != 0
            G_ = abs(gc) + gr
            # reported loss (:480-483)
            dlo, dhi = (fc - fr, fc + fr) if label else (-fc - fr, -fc + fr)
            l_lo, l_hi = logsig(dlo), logsig(dhi)
            self.loss_c += (l_lo + l_hi) / 2
            self.loss_r += (l_hi - l_lo) / 2 + 8 * U * (1 + abs(l_lo) + abs(l_hi))
            if self.reg:
                sq = qc * qc
                self.loss_c -= float(self.reg) * sq.sum()
                self.loss_r += float(self.reg) * ((2 * np.abs(qc) * qr + qr * qr).sum() + gamma(D + 8) * (Q * Q).sum())
            # error (:487, quantized old v) and the row's update (:490)
            e_c += gc * qc
            e_r += abs(gc) * qr + gr * Q
            e_abs += G_ * Q
            X = np.abs(xc) + xr
            dc = gc * avg - d * xc
            dr = abs(gc) * r_avg + gr * A + d * xr + gamma(3) * (G_ * A + d * X) + 3 * SUB
            if m.kind == "warp":
                deltas.setdefault(i, []).append((t, dc, dr))
            self.add_to(self.V, i, dc, dr)
        e_r = e_r + gamma(nt + 1) * e_abs + nt * SUB
        # ---- the error to every context occurrence (:494-503)
        E = np.abs(e_c) + e_r
        for i in ctx.tolist():
            if d and m.kind != "warp":  # decay of the row as this occurrence reads it
                xc, xr = self.read(self.U, self.u0, i)
                self.add_to(self.U, i, e_c - d * xc, e_r + d * xr + gamma(3) * (E + d * (np.abs(xc) + xr)) + 3 * SUB)
            else:
                self.add_to(self.U, i, e_c, e_r)
        self.moved = moved

    def final_rows_off(self, ids_u, ids_v, u1, v1):
        """The first of the given rows (whose last update in the step is done) that is outside its interval."""
        for name, T, after, ids in (("u", self.U, u1, ids_u), ("v", self.V, v1, ids_v)):
            for i in ids:
                c, r = T[i]
                bad = np.abs(after[i].astype(np.float64) - c) > r
                if bad.any():
                    col = int(np.argmax(bad))
                    return "%s row %d column %d: %r, replay %r +- %.3g" % (name, i, col, after[i, col], c[col], r[col])
        return None


def logsig(x):
    """log(sigmoid(x)) of the reported loss (:67-71, :481), monotone in x."""
    if x > 6:
        return 0.0
    if x < -6:
        return LOG_1E9
    return -float(np.log1p(np.exp(-x)))


def check_step(u0, v0, u1, v1, loss, positions, b, q, reg, exptab, model):
    """Checks one step.  Returns None when unresolved (more than MAX_BRANCHES admissible outcomes alive at once),
    else a dict of worst ratios (error / radius) of a branch that holds every element, or raises AssertionError naming
    the first failing element.  A branch is dropped as soon as a row whose last update in the step is done leaves its
    interval, so a wrong expTable slot or a wrong before/after choice dies with its own target row.  With loss None
    only the rows the positions touch are compared, and the result carries the hull [loss_lo, loss_hi] of the
    surviving branches' loss intervals."""
    last_u, last_v = {}, {}
    for p, (ctx, tg, _) in enumerate(positions):
        last_u.update((int(i), p) for i in ctx)
        last_v.update((int(i), p) for i in tg)
    done_u = [[i for i in set(ctx.tolist()) if last_u[i] == p] for p, (ctx, _, _) in enumerate(positions)]
    done_v = [[i for i in set(tg.tolist()) if last_v[i] == p] for p, (_, tg, _) in enumerate(positions)]
    states, why = [Replay(u0, v0, b, q, reg, exptab, model)], None
    for p, (ctx, tg, alpha) in enumerate(positions):
        new = []
        for st in states:
            todo = [[]]
            while todo:
                r = st.copy(todo.pop())
                try:
                    r.position(ctx, tg, alpha)
                except NeedChoice as e:
                    todo.extend(r.choices + [j] for j in range(e.n))
                    continue
                off = r.final_rows_off(done_u[p], done_v[p], u1, v1)
                if off is None:
                    new.append(r)
                else:
                    why = "position %d: %s" % (p, off)
                if len(new) > MAX_BRANCHES:
                    return None
        states = new
        if not states:
            raise AssertionError(why)
    results = []
    for rp in states:
        res = compare(rp, u1, v1, loss)
        res["straddles"], res["last_moved"] = rp.straddles, rp.moved
        results.append((res, rp.dup_taken))
    ok = [(r, d) for r, d in results if r["ok"]]
    if not ok:
        raise AssertionError(min((r for r, _ in results), key=lambda r: r["worst"])["first"])
    res = ok[0][0]
    res["loss_lo"], res["loss_hi"] = min(r["loss_lo"] for r, _ in ok), max(r["loss_hi"] for r, _ in ok)
    # the before (0) / after (1) reads every surviving branch agrees on: both were followed, so the other was rejected
    res["dups_forced"] = [x for x, *others in zip(*(d for _, d in ok)) if all(o == x for o in others)]
    return res


def compare(rp, u1, v1, loss):
    out = {"ok": True, "first": None, "u": 0.0, "v": 0.0, "loss": 0.0, "upd": [], "moved": 0, "loose": 0}
    for name, T, after, before in (("u", rp.U, u1, rp.u0), ("v", rp.V, v1, rp.v0)):
        if not T:
            continue
        ids = np.fromiter(T, np.int64)
        c = np.stack([T[i][0] for i in ids])
        r = np.stack([T[i][1] for i in ids])
        err = np.abs(after[ids].astype(np.float64) - c)
        ratio = err / r
        out[name] = float(ratio.max())
        out["upd"].append((np.abs(after[ids].astype(np.float64) - before[ids]) / r).ravel())
        step = np.abs(c - before[ids])  # the replay's own update: elements it moves, and those whose radius exceeds it
        out["moved"] += int((step > 0).sum())
        out["loose"] += int(((step > 0) & (r > step)).sum())
        if out[name] > 1 and out["ok"]:
            k, col = np.unravel_index(int(ratio.argmax()), ratio.shape)
            out["ok"] = False
            out["first"] = "%s row %d column %d: %r, replay %r +- %.3g" % (name, ids[k], col, after[ids[k], col],
                                                                        c[k, col], r[k, col])
        if loss is None:
            continue
        keep = np.ones(len(after), bool)
        keep[ids] = False
        if not np.array_equal(bits(after[keep]), bits(before[keep])):
            out["ok"] = False
            out["first"] = out["first"] or "%s: a row the step did not touch changed" % name
    lr = rp.loss_r + 1e-9 * abs(rp.loss_c)
    out["loss_lo"], out["loss_hi"] = rp.loss_c - lr, rp.loss_c + lr
    if loss is None:  # the replay's rows only; the caller checks the other rows and the loss
        out["worst"] = max(out["u"], out["v"])
        return out
    out["loss"] = abs(loss - rp.loss_c) / lr
    if out["loss"] > 1 and out["ok"]:
        out["ok"] = False
        out["first"] = "loss %r, replay %r +- %.3g" % (loss, rp.loss_c, lr)
    out["worst"] = max(out["u"], out["v"], out["loss"])
    return out


# ------------------------------------------------------------------------------------------------ trajectories
def seeded_tables(V, D, seed):
    """Random tables whose f covers the expTable range and both saturated ends (f has a standard deviation of about 3
    with 10 context rows at bit level 0)."""
    s = float(np.clip(np.sqrt(9 * np.sqrt(10) / np.sqrt(D)), 0.3, 5.0))
    rng = np.random.default_rng(seed)
    return (rng.uniform(-s, s, (V, D)).astype(np.float32), rng.uniform(-s, s, (V, D)).astype(np.float32))


class Trajectory:
    """Steps of one shard: `tables()`, `step()` -> (loss, counters), `state()` -> (alpha, wca)."""

    def __init__(self, side, recs, tokens, W, alpha0, train_words):
        self.side, self.recs, self.tokens, self.W = side, recs, tokens, W
        self.sentences = split_sentences(recs, W)
        self.k = 0
        self.cursor = 0
        self.counter = Counter(alpha0, train_words)

    def skip(self, words):
        """Trains whole sentences until `words` words are read (one train_step(words) / oracle steps)."""
        n = w = 0
        while w < words:
            w += self.advance()
            n += 1
        return n

    def advance(self):
        words = sentence_words(self.tokens, self.cursor)
        self.cursor += words
        self.counter.sentence(words)
        self.k += 1
        return words

    def next_positions(self):
        first, L, sen = self.sentences[self.k]
        return sentence_positions(self.recs, first, L, sen, self.W)


def run_trajectory(traj, steps, b, q, reg, exptab, model, report, name, tamper=None):
    """Checks `steps` consecutive one-sentence steps; returns the summary.  `tamper(k, positions)` may corrupt the
    side's output of step k (the controls)."""
    resolved, worst, upd, left_out, straddles, moved, loose = 0, {"u": 0.0, "v": 0.0, "loss": 0.0}, [], 0, 0, 0, 0
    checked = 0
    u1, v1 = traj.side.tables()
    for k in range(steps):
        positions = traj.next_positions()
        u0, v0 = u1, v1
        loss, st = traj.side.step(positions, k, tamper)
        traj.advance()
        u1, v1 = traj.side.tables()
        assert st["positions"] == len(positions), (name, k, st)
        assert st["context_rows"] == sum(len(p[0]) for p in positions), (name, k)
        assert st["target_rows"] == sum(len(p[1]) for p in positions), (name, k)
        a, wca = traj.side.state()
        assert (np.float32(a), wca) == (traj.counter.alpha, traj.counter.wca), (name, k, a, wca, traj.counter.alpha)
        if not positions:
            assert np.array_equal(bits(u1), bits(u0)) and np.array_equal(bits(v1), bits(v0))
            continue
        checked += 1
        try:
            res = check_step(u0, v0, u1, v1, loss, positions, b, q, reg, exptab, model)
        except AssertionError as e:
            raise AssertionError("%s: step %d (%d positions): %s" % (name, k, len(positions), e)) from None
        if res is None:
            continue
        resolved += 1
        straddles += res["straddles"]
        moved += res["moved"]
        loose += res["loose"]
        for key in worst:
            worst[key] = max(worst[key], res[key])
        upd.append(np.concatenate(res["upd"]))
        # the step without its last position must fail
        if res["last_moved"]:  # (a saturated f with g = 0 and no -reg changes nothing)
            try:
                short = check_step(u0, v0, u1, v1, loss, positions[:-1], b, q, reg, exptab, model)
            except AssertionError:
                short = "fails"
            assert short == "fails", "%s: step %d without its last position: %r" % (name, k, short)
            left_out += 1
    med = float(np.median(np.concatenate(upd))) if upd else 0.0
    loose_frac = loose / max(moved, 1)
    report("%s: %d/%d steps resolved (%d fail without their last position); worst err/bound u %.3f v %.3f loss %.3f; "
           "median |update|/radius %.3g; radius above the update at %.2g of the moved elements; %d quantized reads "
           "straddled a level" % (name, resolved, checked, left_out, worst["u"], worst["v"], worst["loss"], med,
                                  loose_frac, straddles))
    return dict(resolved=resolved, checked=checked, worst=worst, median=med, left_out=left_out, loose=loose_frac,
                straddles=straddles)


# ----------------------------------------------------------------------------------------------------- the CPU
class OracleSide:
    """The oracle stepped position by position with the trace's alpha (w2bo_apply_position)."""

    def __init__(self, o, D, W, N, b, reg, seed):
        self.m = po.OracleModel(o, D, W, N, b, reg=reg, table=np.zeros(1, np.int32))
        self.m.u[...], self.m.v[...] = seeded_tables(o.vocab_size, D, seed)
        self.ex = po.exptable()

    def tables(self):
        return self.m.u.copy(), self.m.v.copy()

    def apply(self, ctx, tg, alpha):
        self.m.m.alpha = alpha
        f = np.zeros(max(len(tg), 1), np.float32)
        loss = C.c_double()
        po.lib().w2bo_apply_position(C.byref(self.m.m), self.ex, ctx, len(ctx), tg, len(tg), f, C.byref(loss))
        return loss.value

    def step(self, positions, k, tamper=None):
        if tamper:
            return tamper(self, k, positions)
        loss = sum(self.apply(ctx, tg, a) for ctx, tg, a in positions)
        return loss, counters(positions)

    def quiet_step(self, positions):
        for ctx, tg, a in positions:
            self.apply(ctx, tg, a)


def oracle_trajectory(o, D, W, N, b, reg, seed=5):
    """An oracle Trajectory: the draw trace of shard 0 (from a 1-column model: the draws do not depend on D)."""
    t = po.OracleModel(o, 1, W, N, b, reg=reg)
    _, recs = t.train_shard(0, trace_cap=200000)
    side = OracleSide(o, D, W, N, b, reg, seed)
    traj = Trajectory(side, recs, o.tokens, W, 0.05, o.train_words)
    # the oracle's learning rate is the trace's, set per position: its state is the counter's by construction
    side.state = lambda: (traj.counter.alpha, traj.counter.wca)
    return traj, side


def counters(positions):
    return dict(positions=len(positions), context_rows=sum(len(p[0]) for p in positions),
                target_rows=sum(len(p[1]) for p in positions))


@pytest.fixture(scope="module")
def cpu_corpus(tmp_path_factory):
    d = tmp_path_factory.mktemp("traj")
    path = zipf_corpus(str(d / "z.txt"), 30000, 1100, seed=21, newline_every=12)
    return po.Corpus(path, 1)


def oracle_prefix(traj, words):
    """Trains the oracle through the sentences of the first `words` words (unchecked)."""
    w = 0
    while w < words:
        traj.side.quiet_step(traj.next_positions())
        w += traj.advance()


CPU_CASES = [  # D, window, negative, bit level, reg
    (5, 5, 5, 0, 0.0), (128, 5, 24, 1, 0.002), (200, 10, 24, 2, 0.0), (800, 10, 24, 1, 0.0),
    (260, 1, 40, 5, 0.002), (1024, 5, 5, 8, 0.0), (96, 64, 0, 0, 0.002), (33, 5, 24, 3, 0.0),
]


@pytest.mark.parametrize("case", CPU_CASES, ids=lambda c: "D%d-W%d-N%d-b%d-reg%g" % c)
def test_oracle_trajectory_within_f64_bounds(case, cpu_corpus):
    """The sequential float32 oracle, stepped with the trace's positions and alpha, meets the replay's bounds, with
    the 10 000-word learning-rate period crossed inside the checked steps."""
    D, W, N, b, reg = case
    traj, side = oracle_trajectory(cpu_corpus, D, W, N, b, reg)
    oracle_prefix(traj, 9600)
    res = run_trajectory(traj, 40, b, quantizer(b, False), reg, side.ex, Model("seq"), print, "oracle")
    assert res["resolved"] >= 0.95 * res["checked"] and res["checked"] >= 30
    assert res["median"] >= 1e3 or b == 3  # bit level 3 quantizes every value to +-0: nothing moves
    assert res["loose"] <= LOOSE_MAX or b == 3


def test_oracle_stepping_equals_train_shard(cpu_corpus):
    """Stepping the oracle position by position through the trace is train_shard itself, bit for bit."""
    D, W, N, b, reg = 16, 5, 6, 1, 0.002
    traj, side = oracle_trajectory(cpu_corpus, D, W, N, b, reg)
    m = po.OracleModel(cpu_corpus, D, W, N, b, reg=reg)
    m.u[...], m.v[...] = side.m.u, side.m.v
    loss_ref = m.train_shard(0)
    loss = 0.0
    for first, L, sen in traj.sentences:
        for ctx, tg, a in sentence_positions(traj.recs, first, L, sen, W):
            loss += side.apply(ctx, tg, a)
    assert np.array_equal(bits(side.m.u), bits(m.u)) and np.array_equal(bits(side.m.v), bits(m.v))
    assert loss == pytest.approx(loss_ref, rel=1e-12)


CONTROLS = ["v_update_dropped", "u_scatter_twice", "alpha_early", "register_g13", "loss_omitted"]


@pytest.mark.parametrize("control", CONTROLS)
def test_checker_fails_corrupted_trajectories(control, cpu_corpus):
    """Each corruption of the oracle's trajectory fails the replay at the step it corrupts, and the steps before it
    pass.  register_g13 is the uncorrupted oracle held to the register kernel's model with groups of 13 targets: it
    fails at the first step with a repeated target inside one group."""
    D, W, N, b = 64, 5, 24, 0
    traj, side = oracle_trajectory(cpu_corpus, D, W, N, b, 0.0)
    if control == "alpha_early":
        oracle_prefix(traj, 9600)
    model = Model("register", G=13, vec=1, threads=64) if control == "register_g13" else Model("seq")
    hit = []

    def tamper(s, k, positions):
        loss = 0.0
        j = len(positions) // 2
        a_next = None
        if control == "alpha_early" and traj.k + 1 < len(traj.sentences):
            a_next = traj.recs[traj.sentences[traj.k + 1][0]][4]
        for n, (ctx, tg, a) in enumerate(positions):
            u0, v0 = s.tables()
            if a_next is not None and a_next != a:
                a = a_next  # the next period's learning rate one sentence early
                hit.append(traj.k)
            lp = s.apply(ctx, tg, a)
            if n == j and not hit:
                if control == "v_update_dropped":
                    s.m.v[tg] = v0[tg]
                    hit.append(traj.k)
                elif control == "u_scatter_twice" and len(np.unique(ctx)) == len(ctx):
                    s.m.u[ctx[0]] = s.m.u[ctx[0]] + (s.m.u[ctx[0]] - u0[ctx[0]])
                    hit.append(traj.k)
                elif control == "loss_omitted":
                    lp = 0.0
                    hit.append(traj.k)
            if control == "register_g13" and any(len(np.unique(tg[g:g + 13])) < len(tg[g:g + 13])
                                                 for g in range(0, len(tg), 13)):
                hit.append(traj.k)
            loss += lp
        return loss, counters(positions)

    failed = None
    for k in range(200):
        try:
            run_trajectory(traj, 1, b, quantizer(b, False), 0.0, side.ex, model, print, control, tamper)
        except AssertionError as e:
            failed = (traj.k - 1, str(e))
            break
        # a repeated target whose first update is tiny (saturated f) can leave a step indistinguishable
        assert not hit or control == "register_g13", "%s: the corrupted step passed" % control
    assert failed is not None and hit and hit[-1] == failed[0], (control, hit, failed)
    print(control, failed[1][:300])


# ------------------------------------------------------------------------ the warp kernel's own source, emulated
@pytest.fixture(scope="module")
def emu_corpus(tmp_path_factory):
    import word2bits_b200 as w2b
    path = zipf_corpus(str(tmp_path_factory.mktemp("traj_emu") / "e.txt"), 1600, 1500, seed=31, newline_every=10,
                       exponent=0.5)
    o = po.Corpus(path, 1)
    return w2b.Corpus(path, 1), o, po.unigram_table(o.counts)


def emulated_shard_steps(emu_corpus, D, W, N, b, reg, serial, shards=12):
    """Each shard of a short corpus, trained by the warp kernel's source under the emulator (tests/emu: adversarially
    late completion of loads and reduces, shuffled scheduling), as one step: (u0, v0, u1, v1, loss, positions).
    The ring has 3 slots (one load in flight), so a repeated target's later load is issued after the earlier
    occurrence's reduce, which may or may not have landed; with 16 slots every load of a position is issued first."""
    from tests.emu import emu
    c, o, table = emu_corpus
    u, v = seeded_tables(c.vocab_size, D, 3)
    kw = dict(size=D, window=W, negative=N, bitlevel=b, shards=shards, reg=reg, slots=3)
    for s in range(shards):
        tr = emu.train_epoch_warp(c, table, u.copy(), v.copy(), trace_shard=s, trace_cap=100000, **kw)
        positions = [p for first, L, sen in split_sentences(tr["trace"], W)
                     for p in sentence_positions(tr["trace"], first, L, sen, W)]
        u0, v0 = u.copy(), v.copy()
        out = emu.train_epoch_warp(c, table, u, v, trace_shard=s, serial=serial, async_mode=2, seed=s + 1, **kw)
        assert out["n_pos"][s] == len(positions) and out["done"][s] == 1
        yield u0, v0, u.copy(), v.copy(), float(out["loss"][s]), positions


@pytest.mark.parametrize("reg", [0.0, 0.002])
def test_emulated_warp_kernel_within_the_warp_model(reg, emu_corpus):
    """The warp kernel's source, with serial = 1 and late, shuffled completion of its bulk copies, passes the warp
    model over whole short shards; repeated targets are seen to read their rows both before and after an earlier
    occurrence's update (each read being the only one that holds, the other branch rejected)."""
    D, W, N, b = 64, 5, 12, 0
    forced, resolved, n = [], 0, 0
    for u0, v0, u1, v1, loss, positions in emulated_shard_steps(emu_corpus, D, W, N, b, reg, serial=1):
        n += 1
        res = check_step(u0, v0, u1, v1, loss, positions, b, quantizer(b, False), reg, po.exptable(),
                         Model("warp", nj=1))
        if res is not None:
            resolved += 1
            forced += res["dups_forced"]
    print("emulated warp kernel, reg %g: %d/%d shards resolved; repeated targets read before %d and after %d times"
          % (reg, resolved, n, forced.count(0), forced.count(1)))
    assert resolved >= 0.6 * n  # a step here is a whole shard (~130 positions): more live branches than one sentence
    assert forced.count(0) > 0 and forced.count(1) > 0


def test_emulated_prefetch_fails_the_warp_model(emu_corpus):
    """serial = 0 lets the ring fetch position p+1's rows before p's updates land (a context row shared by neighbours
    is read stale): the replay rejects it."""
    D, W, N, b = 64, 5, 12, 0
    failed, n = 0, 0
    for u0, v0, u1, v1, loss, positions in emulated_shard_steps(emu_corpus, D, W, N, b, 0.0, serial=0):
        n += 1
        try:
            check_step(u0, v0, u1, v1, loss, positions, b, quantizer(b, False), 0.0, po.exptable(), Model("warp", nj=1))
        except AssertionError as e:
            failed += 1
            first = str(e)
    print("emulated prefetch: %d/%d shards fail; %s" % (failed, n, first if failed else ""))
    assert failed >= n // 2


# ----------------------------------------------------------------------------------------------------- the GPU
class TrainerSide:
    def __init__(self, t):
        self.t = t

    def tables(self):
        return self.t.download_raw()

    def step(self, positions, k, tamper=None):
        st = self.t.train_step(1)
        return st["loss"], st

    def state(self):
        return self.t.get_state()


GPU_CASES = [  # family, D, window, negative, bit level, reg, kernel, resident, what the case asserts it runs
    ("warp", 5, 5, 5, 0, 0.0, 0, True, {"minb": 24, "bm": 0}),
    ("warp", 128, 5, 24, 8, 0.002, 0, True, {"minb": 20, "reg": 1}),
    ("warp", 200, 10, 24, 2, 0.0, 0, True, {"minb": 20, "bm": 2}),
    ("warp", 200, 5, 5, 0, 0.002, 0, True, {"minb": 16, "reg": 1}),
    ("warp", 384, 5, 5, 0, 0.0, 0, True, {"minb": 16}),
    ("warp", 384, 5, 12, 1, 0.002, 0, True, {"minb": 12, "reg": 1}),
    ("warp", 800, 10, 24, 1, 0.0, 0, True, {"minb": 12, "bm": 1}),     # the benchmarked shape
    ("warp", 800, 10, 24, 1, 0.0, 0, False, {"minb": 12}),             # streamed slices
    ("warp", 1024, 1, 40, 5, 0.002, 0, True, {"minb": 8, "reg": 1}),
    ("warp", 1200, 5, 0, 0, 0.0, 0, True, {"minb": 8}),
    ("warp", 1536, 64, 5, 3, 0.002, 0, True, {"minb": 4, "reg": 1}),
    ("warp", 2048, 5, 24, 1, 0.0, 0, True, {"minb": 4, "bm": 9}),
    ("warp", 256, 200, 5, 0, 0.0, 0, True, {"sentence_in_smem": 0}),  # sentence buffer in global memory
    ("register", 512, 5, 4, 1, 0.0, 1, True, {"wide": 0, "vec": 4, "group": 5}),
    ("register", 512, 5, 8, 0, 0.0, 1, True, {"wide": 0, "vec": 4, "group": 9}),
    ("register", 512, 5, 12, 2, 0.0, 1, True, {"wide": 0, "vec": 4, "group": 13}),
    ("register", 640, 5, 12, 5, 0.002, 1, True, {"wide": 0, "vec": 4, "group": 9, "reg": 1}),
    ("register", 101, 5, 12, 1, 0.0, 1, True, {"wide": 0, "vec": 1, "group": 9}),
    ("register", 101, 5, 6, 0, 0.002, 1, True, {"wide": 0, "vec": 1, "group": 9, "reg": 1}),
    ("register", 1023, 5, 12, 0, 0.0, 1, True, {"wide": 1, "vec": 1, "threads": 1024}),
    ("register", 1021, 5, 6, 1, 0.002, 1, True, {"wide": 1, "vec": 1, "reg": 1}),
    ("register", 2048, 5, 6, 1, 0.0, 1, True, {"wide": 1, "vec": 4}),  # kernel = 1 where the tuned copy cannot
    ("wide", 2052, 5, 24, 0, 0.0, 0, True, {"wide": 1, "vec": 4, "group": 5}),
    ("wide", 3072, 5, 24, 1, 0.002, 0, True, {"wide": 1, "vec": 4, "group": 5, "reg": 1}),
    ("wide", 4096, 5, 12, 5, 0.0, 0, True, {"wide": 1, "vec": 4, "group": 5}),
    ("wide", 4096, 5, 12, 0, 0.002, 0, True, {"wide": 1, "vec": 4, "group": 5, "reg": 1}),
]


def gpu_case_id(c):
    return "%s-D%d-W%d-N%d-b%d-reg%g%s" % (c[0], c[1], c[2], c[3], c[4], c[5], "" if c[7] else "-streamed")


@pytest.fixture(scope="module")
def gpu_corpus_path(tmp_path_factory):
    d = tmp_path_factory.mktemp("traj_gpu")
    return zipf_corpus(str(d / "flat.txt"), 14000, 5000, seed=23, newline_every=12, exponent=0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=gpu_case_id)
def test_training_steps_within_f64_bounds(case, gpu_corpus_path):
    w2b = pytest.importorskip("word2bits_b200")
    kind, D, W, N, b, reg, kernel, resident, expect = case
    c = w2b.Corpus(gpu_corpus_path, 1)
    t = w2b.Trainer(c, size=D, window=W, negative=N, bitlevel=b, reg=reg, threads=1, iter=1, kernel=kernel,
                    resident=resident)
    info = t.kernel_info()
    # the instantiation (and geometry) the case is written for is the one that runs
    got = dict(info, **{k: v for k, v in warp_plan_of(w2b, case).items() if k == "sentence_in_smem"})
    assert info["warp"] == (kind == "warp") and all(got[k] == v for k, v in expect.items()), (expect, got)
    t.upload_raw(*seeded_tables(c.vocab_size, D, 7))
    t.epoch_begin()
    recs = t.trace(0, cap=200000) if resident else w2b_trace_resident(w2b, c, case)
    traj = Trajectory(TrainerSide(t), recs, c.tokens, W, 0.05, c.train_words)
    st = t.train_step(9400)
    n = traj.skip(9400)
    assert st["words"] == traj.cursor, (st["words"], traj.cursor, n)
    q = quantizer(b, info["warp"] == 1 and not reg and b in (1, 2) and info["bm"] != 9)
    res = run_trajectory(traj, 24, b, q, reg, t.download_exptable(), model_for(info), print,
                         "%s %s" % (gpu_case_id(case), info))
    assert res["checked"] >= 18 and res["resolved"] >= 0.95 * res["checked"], res
    assert res["median"] >= 1e3 or b == 3, res
    assert res["loose"] <= LOOSE_MAX or b == 3, res
    t.close()


def warp_plan_of(w2b, case):
    kind, D, W, N, b, reg, kernel, resident, expect = case
    return w2b.warp_plan(size=D, window=W, negative=N, bitlevel=b, reg=reg, kernel=kernel)


def w2b_trace_resident(w2b, c, case):
    """The draw trace of a streamed case, from a resident context of the same configuration (the draws are the same)."""
    kind, D, W, N, b, reg, kernel, resident, expect = case
    t = w2b.Trainer(c, size=D, window=W, negative=N, bitlevel=b, reg=reg, threads=1, iter=1, kernel=kernel)
    recs = t.trace(0, cap=200000)
    t.close()
    return recs


STRICT_EPOCH_D = [1023, 3588, 4096]


@pytest.mark.gpu
@pytest.mark.parametrize("D", STRICT_EPOCH_D)
def test_strict_wide_epoch_equals_oracle(D, gpu_corpus_path):
    """Strict mode through the wide instantiations, a whole short epoch: u, v, alpha and wca bit for bit against the
    oracle, the loss to 1e-4 (L2)."""
    w2b = pytest.importorskip("word2bits_b200")
    with tempfile.TemporaryDirectory() as d:
        path = zipf_corpus(os.path.join(d, "s.txt"), 1500, 300, seed=29, newline_every=12)
        c = w2b.Corpus(path, 1)
        o = po.Corpus(path, 1)
    t = w2b.Trainer(c, size=D, window=5, negative=6, bitlevel=1, reg=0.002, threads=1, iter=1, mode=w2b.MODE_STRICT)
    info = t.kernel_info()
    assert info["warp"] == 0 and info["wide"] == 1 and info["group"] == 1
    m = po.OracleModel(o, D, 5, 6, 1, reg=0.002)
    t.upload_raw(m.u, m.v)
    loss, st = t.train_epoch()
    lo = m.train_shard(0)
    u, v = t.download_raw()
    a, wca = t.get_state()
    assert np.array_equal(bits(u), bits(m.u)) and np.array_equal(bits(v), bits(m.v))
    assert (np.float32(a), wca) == (np.float32(m.alpha), m.word_count_actual)
    assert abs(loss - lo) <= 1e-4 * abs(lo)
    t.close()


def family(info, strict=False):
    """The instantiation family of a kernel_info(): warp kernel by occupancy tier and -reg, and by compiled bit level;
    register kernel by copy (tuned / wide), VEC, group and -reg; strict mode by VEC."""
    if info["warp"]:
        return {("warp", info["minb"], info["reg"]), ("warp-bm", info["bm"])}
    if strict:
        return {("strict", info["vec"])}
    return {("register", "wide" if info["wide"] else "tuned", info["vec"], info["group"], info["reg"])}


def families_of(w2b, configs):
    fam = set()
    for kw, strict in configs:
        try:
            t = w2b.Trainer(None, vocab_size=64, threads=1, init=False, mode=w2b.MODE_STRICT if strict else w2b.MODE_FAST,
                            **kw)
        except w2b.W2BError as e:
            assert e.code == 1, e  # a width the configuration refuses
            continue
        fam |= family(t.kernel_info(), strict)
        t.close()
    return fam


@pytest.mark.gpu
def test_every_training_instantiation_family_was_checked():
    """Every family of training instantiation the dispatch can launch — found by sweeping widths, bit levels, -reg,
    group sizes, kernel choice and mode through kernel_info() — is run by one of the cases above."""
    w2b = pytest.importorskip("word2bits_b200")
    sweep = [(dict(size=128 * nj - 3, bitlevel=b, reg=reg, negative=5), False)
             for nj in range(1, 17) for b in (0, 1, 2, 5) for reg in (0.0, 0.002)]
    sweep += [(dict(size=D, bitlevel=1, reg=reg, negative=N, kernel=k), False)
              for D in (101, 512, 673, 1021, 1023, 1024, 1412, 2048, 2052, 3000, 4096) for k in (0, 1)
              for reg in (0.0, 0.002) for N in (4, 8, 12)]
    sweep += [(dict(size=D, bitlevel=1, reg=reg, negative=6), True) for D in (101, 1023, 1024, 4096)
              for reg in (0.0, 0.002)]
    reachable = families_of(w2b, sweep)
    cases = [(dict(size=c[1], window=c[2], negative=c[3], bitlevel=c[4], reg=c[5], kernel=c[6]), False)
             for c in GPU_CASES]
    cases += [(dict(size=D, window=5, negative=6, bitlevel=1, reg=0.002), True) for D in STRICT_EPOCH_D]
    checked = families_of(w2b, cases)
    print("%d families reachable, %d checked" % (len(reachable), len(checked)))
    assert reachable <= checked, sorted(reachable - checked, key=str)
