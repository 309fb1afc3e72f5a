"""Generates tests/golden/reference_nearest.json: ranks 1 and 2 of every nearest-neighbour list of
tests/nearest_cases.py, as the UNMODIFIED reference compute_accuracy (oracle/_ref, built by oracle/Makefile) gives them.
The reference returns only its best word, so each rank is read off a question of its own, in a section of its own:
    w w w t1      vec = (M[w] - M[w]) + M[w] = M[w] exactly and only w is skipped: correct iff rank 1 is t1;
    t1 t1 w t2    vec = M[w] exactly again, {t1, w} skipped: correct iff rank 2 (after t1) is t2.
t1 and t2 are the CPU restatement's ranks (tests/topk_oracle.py); every such question must be counted correct, and the
digest of the restatement's ranks 1-2 is stored.  A rank whose word shares its name with an earlier word cannot be named
in a question (the reference resolves a name to its first row) and is left out of the pin; the count is stored.
Ranks >= 3 rest on the restatement; at k = 1 analogy lists are w2bo_analogy's answers, pinned in
reference_outputs.json / reference_packed.json.

    python tests/golden/make_reference_nearest.py"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests import analogy_cases as ac  # noqa: E402
from tests import nearest_cases as nc  # noqa: E402
from tests import topk_oracle as to  # noqa: E402
from tests.util import digest  # noqa: E402

OUT = os.path.join(HERE, "reference_nearest.json")
REFACC = os.path.join(ROOT, "oracle", "_ref", "compute_accuracy")


def rank_questions(words, names, queries, ids, path):
    """The per-rank question file; returns {section: 1} for every question written."""
    first = to._first(names)
    want = {}
    with open(path, "w") as f:
        for i, (w, q) in enumerate(zip(words, queries)):
            t1, t2 = ids[i, 0], ids[i, 1]
            if q is None or t1 < 0 or first[names[t1]] != t1:
                continue
            f.write(": a%d\n%s %s %s %s\n" % (i, w, w, w, names[t1]))
            want["a%d" % i] = 1
            if t2 >= 0 and first[names[t2]] == t2:
                f.write(": b%d\n%s %s %s %s\n" % (i, names[t1], names[t1], w, names[t2]))
                want["b%d" % i] = 1
    return want


def main():
    assert os.path.exists(REFACC), "build oracle/_ref first"
    out = {}
    for name in nc.CASES:
        with tempfile.TemporaryDirectory() as d:
            _, vf, _, words, b, th = nc.build(name, d)
            names, M = to.load(vf, b, th)
            queries = to.nearest_queries(words, names)
            ids, _ = to.lists(M, queries, k=2)
            pq = os.path.join(d, "ranks.txt")
            want = rank_questions(words, names, queries, ids, pq)
            rep = subprocess.run([REFACC, vf, str(b), str(th)], stdin=open(pq), capture_output=True, text=True).stdout
            got = ac.per_question_counts(rep)
            assert got == want, (name, sorted(k for k in want if got.get(k) != 1)[:10])
            n1 = sum(k[0] == "a" for k in want)
            out[name] = {"ranks12": digest(ids), "rank1_pinned": n1, "rank2_pinned": len(want) - n1}
            print(name, "ok", out[name], flush=True)
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
