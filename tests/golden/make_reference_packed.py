"""Generates tests/golden/reference_packed.json: what the UNMODIFIED reference compute_accuracy (oracle/_ref, built
by oracle/Makefile) answers on the unpacked file of every case of tests/packed_cases.py, the pin of the packed
evaluator.  As make_reference_outputs.py::analogy does, the choices are read off the reference itself: its report
must equal the oracle's, and every question, run again as a section of its own with the oracle's choice as fourth
word, must be counted correct.

    python tests/golden/make_reference_packed.py"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import pyoracle as po  # noqa: E402
from tests import analogy_cases as ac  # noqa: E402
from tests import packed_cases as pc  # noqa: E402
from tests.util import digest  # noqa: E402

OUT = os.path.join(HERE, "reference_packed.json")
REFACC = os.path.join(ROOT, "oracle", "_ref", "compute_accuracy")


def main():
    assert os.path.exists(REFACC), "build oracle/_ref first"
    out = {}
    for name in pc.CASES:
        with tempfile.TemporaryDirectory() as d:
            _, vf, qf, b, th = pc.build(name, d)
            run = lambda q: subprocess.run([REFACC, vf, str(b), str(th)], stdin=open(q), capture_output=True, text=True).stdout
            report = run(qf)
            rep, ans = po.analogy(vf, qf, b, th)
            assert rep == report, name
            pq = os.path.join(d, "per_question.txt")
            want = ac.per_question_file(qf, ans, ac.vocab_names(vf, th), pq)
            assert ac.per_question_counts(run(pq)) == want, name
            out[name] = {"report": report, "answers": digest(ans)}
            print(name, "ok", flush=True)
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
