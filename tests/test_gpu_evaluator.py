"""The GPU analogy evaluator (csrc/w2b_eval.cu, csrc/w2b_eval_tc.cuh) against the reference, question by question.

For every input of tests/analogy_cases.py the word the GPU chooses for each question must be the one
src/compute-accuracy.c chooses: the CPU restatement (oracle w2bo_analogy) computes them, and its digest must equal
the reference's stored one.  Both pipelines run: the tensor-core filter + fp32 re-score, and W2B_EVAL_SIMT=1 (every
score on the SIMT cores).  A second test holds the filter's TF32 scores to its error bound eps at every D."""
import os

import numpy as np
import pytest

import word2bits_b200 as w2b
from oracle import pyoracle as po
from tests import analogy_cases as ac
from tests.util import digest, reference_outputs

pytestmark = pytest.mark.gpu
STORED = reference_outputs("analogy")


def _gpu_answers(vf, qf, b, th, simt):
    old = os.environ.get("W2B_EVAL_SIMT")
    os.environ["W2B_EVAL_SIMT"] = "1" if simt else "0"
    try:
        return w2b.analogy_answers(vf, qf, bitlevel=b, threshold=th)
    finally:
        if old is None:
            del os.environ["W2B_EVAL_SIMT"]
        else:
            os.environ["W2B_EVAL_SIMT"] = old


@pytest.mark.parametrize("name", sorted(ac.CASES))
def test_gpu_answers_every_question_like_the_reference(tmp_path, name):
    vf, qf, b, th = ac.build(name, str(tmp_path))
    report, want = po.analogy(vf, qf, b, th)
    assert digest(want) == STORED[name]["answers"] and report == STORED[name]["report"]
    for simt in (False, True):
        got = _gpu_answers(vf, qf, b, th, simt)
        bad = np.nonzero(got != want)[0]
        assert len(got) == len(want) and not len(bad), (
            "simt=%d: %d of %d questions differ, first %s: gpu %s, reference %s"
            % (simt, len(bad), len(want), bad[:5], got[bad[:5]], want[bad[:5]]))
    text, acc = w2b.compute_accuracy(vf, qf, bitlevel=b, threshold=th)
    assert text == report
    if name == "all_equal":  # every score ties: the candidate list overflows and the SIMT scorer takes over
        assert acc["candidates"] > 1024 * acc["questions_seen"]
    if name == "small_positive":
        assert want[0] == 2


def _unit_rows(rng, n, D):
    x = rng.normal(size=(n, D))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _worst_rows(rng, n, D):
    """Positive rows of length <= 1 whose values all sit just below a power of two times (1 + 2^-10): TF32 drops
    nearly 2^-10 of each, so all products lose nearly 2^-9 in the same direction."""
    k = int(np.ceil(np.log2(np.sqrt(D))))
    e = np.full((n, D), -k)
    target = 1.0 / (1 + 2.0 ** -10) ** 2
    for i in range(n):
        order = rng.permutation(D)
        s = D * 4.0 ** -k
        for j in order:  # raise single entries by one binade while the length stays <= 1
            if s + 3 * 4.0 ** -k <= target:
                e[i, j] += 1
                s += 3 * 4.0 ** -k
    m = np.float32(1 + 2.0 ** -10 - 2.0 ** -23)
    return (np.ldexp(1.0, e) * m).astype(np.float32)


@pytest.mark.parametrize("D", [1, 3, 7, 8, 12, 31, 32, 33, 72, 130, 200, 800, 1200, 2000])
def test_tensor_core_filter_error_is_within_eps(D):
    """|approx - exact| <= eps for every (question, word) pair, where exact is the float64 product and also the
    reference's fp32 order (the filter is only correct if both hold).  Random unit rows, queries built like the
    evaluator's (b - a) + c, and rows built to make TF32 drop the most."""
    rng = np.random.default_rng(D)
    M = np.concatenate([_unit_rows(rng, 700, D), _worst_rows(rng, 100, D)])
    t = rng.integers(0, 700, (150, 3))
    Q = np.concatenate([(M[t[:, 1]] - M[t[:, 0]]) + M[t[:, 2]], _worst_rows(rng, 40, D)]).astype(np.float32)
    approx, eps = w2b.eval_filter_scores(Q, M)
    exact = Q.astype(np.float64) @ M.astype(np.float64).T
    ref = np.zeros(approx.shape, np.float32)
    for a in range(D):  # sequential, each product rounded then added, as the reference's build does
        ref = ref + np.outer(Q[:, a], M[:, a])
    norm = np.linalg.norm(Q.astype(np.float64), axis=1)
    assert np.all(eps >= 2.0 ** -9 * norm) and np.all(eps <= (2.0 ** -9 + 5 * D * 2.0 ** -24 + 1e-6) * 1.06 * norm)
    r64 = np.abs(approx - exact) / eps[:, None]
    r32 = np.abs(approx.astype(np.float64) - ref) / eps[:, None]
    print("D=%d: worst |approx - exact|/eps %.3f (worst-case rows %.3f), |approx - fp32 reference|/eps %.3f"
          % (D, r64.max(), r64[150:, 700:].max(), r32.max()))
    assert r64.max() <= 1.0 and r32.max() <= 1.0
