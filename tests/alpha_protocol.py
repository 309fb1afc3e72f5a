"""The shared learning rate of a many-shard training step (:379-393), in plain Python: which alphas a shard's positions
may have trained with, given the corpus, every shard's counters before the step and the kernel.

Both kernels check for a crossing at the top of their loop, before each window draw and before each sentence is
read: when wc - last > 10000 the shard adds delta = wc - last to the global counter and stores f(the counter after its
add) as the global alpha.  A shard that reaches its end (wc past train_words / shards) adds wc - last as well and
stores nothing.
  * warp kernel: the crossing shard trains with its own f(W_own) from the next position on; every sentence start
    re-reads the global alpha (a value any shard may have stored, or the value before the step);
  * register kernel: every position re-reads the global alpha.
`plan_step` derives each shard's crossings, their deltas and its end-of-shard add from the corpus; `check_alphas`
judges recorded alphas against them; `Executor` runs the protocol for many shards in a seeded interleaving (and with
injected faults) on the CPU."""
import numpy as np

PERIOD = 10000


class Sentences:
    """Where each sentence of a token stream ends: words(cursor) = the words a sentence read from `cursor` consumes,
    up to and including the next </s> (:394-413), without scanning the stream."""

    def __init__(self, tokens):
        self.ends = np.flatnonzero(np.asarray(tokens) == 0)
        self.n = len(tokens)

    def words(self, cursor, at_least=1):
        """Words of the sentences from `cursor` up to the first whose end makes at least `at_least` words."""
        i = int(np.searchsorted(self.ends, cursor + at_least - 1))
        return (int(self.ends[i]) + 1 if i < len(self.ends) else self.n) - cursor


def f_alpha(W, a0, denom):
    """alpha after the counter reads W (int or int64 array), as the kernels compute it: float32 arithmetic, the floor
    compared in double."""
    a0, denom = np.float32(a0), np.float32(denom)
    w = np.asarray(W, np.float64).astype(np.float32)  # exact in double, one rounding to float32 like (float)wca
    a = (a0 * (np.float32(1) - w / denom)).astype(np.float32)
    floor = float(a0) * 1e-4
    return np.where(a.astype(np.float64) < floor, np.float32(floor), a).astype(np.float32)


class ShardClock:
    """A shard's counters as the kernel keeps them: cursor, word_count, last_word_count, done."""

    def __init__(self, cursor, wc=0, last=0):
        self.cursor, self.wc, self.last, self.done = int(cursor), int(wc), int(last), False


def plan_step(sents, clock, budget, limit, lens):
    """The events of one shard's step, from the corpus (`sents`, a Sentences) and the shard's counters before the step
    (`clock`, advanced in place).  `lens` = records of each sentence of the step (split_sentences of its trace), or None for a step whose
    records are not counted; budget <= 0: to the end.
    Returns dict(cross=[(delta, index of the record it precedes, 1 inside a sentence (that record on trains at the
    shard's own alpha) / 0 at a sentence boundary)], end=delta or None, starts=[first record of each sentence],
    n=records)."""
    out = dict(cross=[], end=None, starts=[], n=0)
    wc0, rec, k = clock.wc, 0, 0

    def top(mid):
        if clock.wc - clock.last > PERIOD:
            out["cross"].append((clock.wc - clock.last, rec, mid))
            clock.last = clock.wc

    while True:
        top(0)
        if budget > 0 and clock.wc - wc0 >= budget:
            break
        if lens is None:  # records not counted: read up to the next sentence that crosses, ends or fills the budget
            need = min(clock.last + PERIOD + 1, limit + 1, wc0 + budget if budget > 0 else limit + 1) - clock.wc
            words = sents.words(clock.cursor, max(need, 1))
        else:
            words = sents.words(clock.cursor)
        clock.cursor += words
        clock.wc += words
        if clock.wc > limit:  # :414-423: the sentence read past the limit is not trained
            out["end"] = clock.wc - clock.last
            clock.last = clock.wc
            clock.done = True
            break
        assert lens is None or k < len(lens), "the trace ends before the step does"
        out["starts"].append(rec)
        for j in range(1 if lens is None else lens[k]):
            if j:
                top(1)
            rec += 1
        k += 1
    assert lens is None or k == len(lens), "the trace holds more sentences than the step reads"
    out["n"] = rec
    return out


def subset_sums(deltas):
    """Every sum of a sub-multiset of `deltas` (sorted int64 array), grouped by value so that equal deltas stay cheap."""
    sums = np.zeros(1, np.int64)
    vals, counts = np.unique(np.asarray(deltas, np.int64), return_counts=True)
    for d, c in zip(vals.tolist(), counts.tolist()):
        sums = np.unique((sums[None, :] + d * np.arange(c + 1, dtype=np.int64)[:, None]).ravel())
    return sums


def check_alphas(plans, alphas, a0, denom, W0, alpha_before, W1, stats_alpha, kernel):
    """Raises AssertionError unless the recorded alphas (alphas[s] = float32 per record of shard s, plans[s] from
    plan_step) are admissible for `kernel` ("warp" or "register"), and the counter moved from W0 to W1 by exactly the
    step's crossings and end-of-shard adds.  Returns a summary: crossings, slots recovered, the alpha range, and how
    many sentence starts read an alpha another shard stored."""
    cross = [(s, d) for s, p in enumerate(plans) for d, _, _ in p["cross"]]
    ends = [p["end"] for p in plans if p["end"] is not None]
    total = sum(d for _, d in cross) + sum(ends)
    assert W1 == W0 + total, "counter %d, want %d + %d crossings + %d end adds = %d" % (
        W1, W0, len(cross), len(ends), W0 + total)
    sums = subset_sums([d for _, d in cross] + ends)
    cand = W0 + sums[sums > 0]
    fc = f_alpha(cand, a0, denom)
    stored = set(fc.tolist()) if cross else set()
    admissible = stored | {float(np.float32(alpha_before))}
    inverse = {}
    for w, a in zip(cand.tolist(), fc.tolist()):
        inverse.setdefault(a, []).append(w)
    own, foreign, floored = [], 0, 0
    floor = float(np.float32(float(np.float32(a0)) * 1e-4))
    for s, (p, al) in enumerate(zip(plans, alphas)):
        al = np.asarray(al, np.float32)
        assert len(al) == p["n"], "shard %d: %d records, the corpus gives %d" % (s, len(al), p["n"])
        bad = [i for i, a in enumerate(al.tolist()) if a not in admissible]
        assert not bad, "shard %d record %d: alpha %r is no value the counter can have given" % (s, bad[0], al[bad[0]])
        if kernel == "register":
            continue
        mine = {at: d for d, at, mid in p["cross"] if mid}
        ends_at = p["starts"][1:] + [p["n"]]
        for i0, i1 in zip(p["starts"], ends_at):
            a = float(al[i0])
            if a != float(np.float32(alpha_before)) and not any(o[0] == s and o[2] == a for o in own):
                foreign += 1
            for i in range(i0 + 1, i1):
                if i in mine:
                    a = float(al[i])
                    if a == floor:  # every counter value past the floor gives it: no slot to recover
                        floored += 1
                        continue
                    ws = [w for w in inverse.get(a, []) if w - W0 >= mine[i]]
                    assert len(ws) == 1, "shard %d record %d: own alpha %r from %s counter values" % (
                        s, i, a, len(ws) or "no")
                    own.append((s, ws[0], a, mine[i]))
                assert float(al[i]) == a, "shard %d record %d: alpha %r inside a sentence that trains at %r" % (
                    s, i, al[i], a)
    out = dict(crossings=len(cross), ends=len(ends), slots=len(own), floored=floored, foreign=foreign,
               alpha_min=float(min((min(a) for a in alphas if len(a)), default=np.nan)),
               alpha_max=float(max((max(a) for a in alphas if len(a)), default=np.nan)))
    if kernel == "warp" and own:
        own.sort(key=lambda o: o[1])
        ws = np.array([o[1] for o in own], np.int64)
        assert len(set(ws.tolist())) == len(ws), "two crossings were given the same counter value"
        if len(own) == len(cross) and not ends:  # every slot W0 + delta_1 + ... + delta_k exactly once
            want = W0 + np.cumsum([o[3] for o in own])
            bad = np.flatnonzero(ws != want)
            assert not len(bad), "crossing %d of the step read counter %d, want %d" % (bad[0], ws[bad[0]], want[bad[0]])
        else:
            gaps = np.diff(np.concatenate([[W0], ws])) - np.array([o[3] for o in own])
            assert (gaps >= 0).all() and ws[-1] <= W1, "crossings overlap on the counter"
    if cross:
        pool = {o[2] for o in own} if kernel == "warp" and len(own) == len(cross) else stored
        assert float(np.float32(stats_alpha)) in pool, "alpha after the step %r is no crossing's" % stats_alpha
    else:
        assert float(np.float32(stats_alpha)) == float(np.float32(alpha_before)), stats_alpha
    return out


class Executor:
    """Many shards' plans run through the counter protocol in a seeded random interleaving (one action of one shard at
    a time: a crossing, a sentence start, a record, an end-of-shard add).  Returns the records' alphas per shard, the
    final counter and the final global alpha.  `fault` injects one of the wrong versions the checker must refuse:
    "pre_add" (alpha from the counter before the add), "twice" (one crossing added twice), "lost" (one crossing never
    added), "late" (the own alpha from one position later), "no_floor", "no_end_add"."""

    def __init__(self, a0, denom, W0, alpha0):
        self.a0, self.denom, self.W0, self.alpha0 = a0, denom, W0, np.float32(alpha0)

    def f(self, W, floor=True):
        if floor:
            return np.float32(f_alpha(W, self.a0, self.denom))
        a0, denom = np.float32(self.a0), np.float32(self.denom)
        return np.float32(a0 * (np.float32(1) - np.float32(np.float32(float(W)) / denom)))

    def run(self, plans, kernel, seed, fault=None, order=None):
        rng = np.random.default_rng(seed)
        acts = []
        for p in plans:
            cross_at = {}
            for d, at, _ in p["cross"]:
                cross_at.setdefault(at, []).append(d)
            a, starts = [], set(p["starts"])
            for i in range(p["n"] + 1):
                for d in cross_at.get(i, []):
                    a.append(("cross", d))
                if i == p["n"]:
                    break
                if i in starts:
                    a.append(("start",))
                a.append(("rec", i))
            if p["end"] is not None:
                a.append(("end", p["end"]))
            acts.append(a)
        counter, g = self.W0, self.alpha0
        own = [self.alpha0] * len(plans)
        out = [np.zeros(p["n"], np.float32) for p in plans]
        nxt = [0] * len(plans)
        seq = order if order is not None else rng.permutation(np.repeat(np.arange(len(plans)), [len(x) for x in acts]))
        victim = int(rng.integers(0, len(plans)))
        late = [False] * len(plans)
        for s in seq.tolist():
            act = acts[s][nxt[s]]
            nxt[s] += 1
            if act[0] == "cross":
                faulty = fault in ("twice", "lost") and s == victim and act[1] == plans[s]["cross"][0][0]
                if faulty and fault == "lost":
                    continue
                counter += act[1] * (2 if faulty else 1)
                w = counter - act[1] if fault == "pre_add" else counter
                a = self.f(w, floor=fault != "no_floor")
                g = a
                if fault == "late" and s == victim:
                    late[s] = a  # the shard keeps its old alpha for one more position
                else:
                    own[s] = a
            elif act[0] == "start":
                own[s] = g
            elif act[0] == "rec":
                out[s][act[1]] = g if kernel == "register" else own[s]
                if late[s] is not False:
                    own[s], late[s] = late[s], False
            elif fault != "no_end_add":
                counter += act[1]
        return out, counter, g
