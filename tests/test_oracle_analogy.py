"""The CPU restatement of src/compute-accuracy.c (oracle/w2b_oracle.c, w2bo_analogy) against the reference.

On every input of tests/analogy_cases.py the oracle prints the reference's report character for character and
chooses the word the reference chose for every question.  The reference's choices are stored as digests in
tests/golden/reference_outputs.json ("analogy"), read off the reference by make_reference_outputs.py; where
oracle/_ref is built the same checks also run live: each question becomes a section of its own whose fourth word is
the oracle's choice, and the reference must count it correct.  Two plausible other orders of the same arithmetic
(fused scoring; the 32-lane normalisation the GPU used before) must be told apart from it."""
import os
import subprocess

import pytest

from oracle import pyoracle as po
from tests import analogy_cases as ac
from tests.util import digest, reference_outputs

REFACC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "compute_accuracy")
STORED = reference_outputs("analogy")


def test_every_case_is_stored():
    assert set(STORED) == set(ac.CASES)


@pytest.mark.parametrize("name", sorted(ac.CASES))
def test_oracle_answers_like_the_reference(tmp_path, name):
    vf, qf, b, th = ac.build(name, str(tmp_path))
    report, ans = po.analogy(vf, qf, b, th)
    assert report == STORED[name]["report"]
    assert digest(ans) == STORED[name]["answers"]
    assert len(ans) == len(ac.read_questions(qf))
    if name == "small_positive":
        assert ans[0] == 2  # the one word scoring above 0, if only just
    if name == "all_equal":
        q = [[int(w[1:]) for w in qq[:3]] for qq in ac.read_questions(qf)]
        assert list(ans) == [min(set(range(10)) - set(x)) for x in q]  # every score ties: the first free index


@pytest.mark.ref
@pytest.mark.skipif(not os.path.exists(REFACC), reason="oracle/_ref not built (the stored answers are checked above)")
@pytest.mark.parametrize("name", sorted(ac.CASES))
def test_oracle_against_the_reference_binary(tmp_path, name):
    vf, qf, b, th = ac.build(name, str(tmp_path))
    run = lambda q: subprocess.run([REFACC, vf, str(b), str(th)], stdin=open(q), capture_output=True, text=True,
                                   timeout=120).stdout
    report, ans = po.analogy(vf, qf, b, th)
    assert report == run(qf)
    pq = str(tmp_path / "per_question.txt")
    want = ac.per_question_file(qf, ans, ac.vocab_names(vf, th), pq)
    assert want and ac.per_question_counts(run(pq)) == want


@pytest.mark.parametrize("flags", [po.AN_FUSED, po.AN_LANE_NORM], ids=["fused_scoring", "lane_order_normalisation"])
def test_other_arithmetic_orders_are_noticed(tmp_path, flags):
    """The pin is tight enough to see the difference between two orders of fp32 arithmetic on 1-bit vectors."""
    vf, qf, b, th = ac.build("nq3000_b1", str(tmp_path))
    _, ans = po.analogy(vf, qf, b, th, flags=flags)
    assert digest(ans) != STORED["nq3000_b1"]["answers"]
    if os.path.exists(REFACC):
        pq = str(tmp_path / "per_question.txt")
        want = ac.per_question_file(qf, ans, ac.vocab_names(vf, th), pq)
        got = ac.per_question_counts(subprocess.run([REFACC, vf, str(b), str(th)], stdin=open(pq), capture_output=True,
                                                    text=True, timeout=120).stdout)
        assert got != want
