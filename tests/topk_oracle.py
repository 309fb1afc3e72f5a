"""CPU restatement of the evaluator's top-k lists (w2b_analogy_topk, w2b_nearest): the reference's top-N list of
src/compute-accuracy.c (:166-175) at N = k.  Rows are normalised by the oracle's w2bo_analogy_normalize (the
reference's build order), vec = (M[b2] - M[b1]) + M[b3], every word scored in fp32 with each product rounded and
then added in index order, and a list holds the k largest scores > 0 of the words not in the query, best first; the
reference's strict `>` insertion puts the smaller index first on equal scores.  At k = 1 this is w2bo_analogy's
answer, and its ranks 1 and 2 of every nearest-neighbour list are what the unmodified reference gives
(tests/golden/reference_nearest.json; tests/test_oracle_topk.py holds both).

flags: po.AN_LANE_NORM normalises in another order (the oracle's negative control), to show the pins notice it."""
import numpy as np

from oracle import pyoracle as po
from tests import analogy_cases as ac
from tests import packed_cases as pc

KMAX = 1024


def load(vf, bitlevel=0, threshold=0, flags=0):
    """(upper-cased names, normalised rows) of the first `threshold` words of a word2vec-binary file."""
    names, vec = pc.read_vectors(vf)
    if threshold and len(names) > threshold:
        names, vec = names[:threshold], vec[:threshold]
    return [n.upper() for n in names], po.analogy_normalize(vec, bitlevel, flags & po.AN_LANE_NORM)


def _first(names):
    first = {}
    for i, n in enumerate(names):
        first.setdefault(n, i)
    return first


def analogy_queries(qf, names):
    """Per question of qf in file order: (b1, b2, b3), or None when one of its four words is not in the vocabulary."""
    first = _first(names)
    out = []
    for q in ac.read_questions(qf):
        ids = [first.get(w.upper()) for w in q[:4]]
        out.append(None if any(i is None for i in ids) else tuple(ids[:3]))
    return out


def nearest_queries(words, names):
    """Per word: (w, w, w), or None when it is not in the vocabulary."""
    first = _first(names)
    return [(first[w.upper()],) * 3 if w.upper() in first else None for w in words]


def lists(M, queries, k=KMAX, block=256):
    """(ids [n, k], scores [n, k]) of every query (None: an all -1 row)."""
    n, V, D = len(queries), M.shape[0], M.shape[1]
    ids = np.full((n, k), -1, np.int32)
    scores = np.zeros((n, k), np.float32)
    live = [i for i, q in enumerate(queries) if q is not None]
    for s0 in range(0, len(live), block):
        rows = live[s0:s0 + block]
        b = np.array([queries[i] for i in rows], np.int64)
        vec = ((M[b[:, 1]] - M[b[:, 0]]) + M[b[:, 2]]).astype(np.float32)
        S = np.zeros((len(rows), V), np.float32)
        for a in range(D):  # each product rounded, then added, in index order
            S = S + np.outer(vec[:, a], M[:, a])
        for j, r in enumerate(rows):
            s = S[j].copy()
            s[list(b[j])] = np.nan  # the query's own words are never in its list
            cand = np.nonzero(s > 0)[0]  # NaN (a zero row) is not > 0
            order = cand[np.lexsort((cand, -s[cand]))][:k]
            ids[r, : len(order)] = order
            scores[r, : len(order)] = s[order]
    return ids, scores
