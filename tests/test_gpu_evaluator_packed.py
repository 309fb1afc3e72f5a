"""The evaluator on packed vector files (csrc/w2b_eval_bits.cuh) against the reference, question by question.

For every case of tests/packed_cases.py the word chosen for each question of the PACKED file must be the one
src/compute-accuracy.c chooses on the unpacked file: the CPU restatement computes them and its digest must equal the
reference's stored one (tests/golden/reference_packed.json).  Both pipelines run: bit-domain Gram + filter + fp32
re-score, and W2B_EVAL_SIMT=1 (planes decoded to fp32, every score on the SIMT scorer).  The second half holds the
Gram kernel to the integer dot product exactly and the filter to its error bound, at every D."""
import os
import subprocess

import numpy as np
import pytest

import word2bits_b200 as w2b
from oracle import pyoracle as po
from tests import packed_cases as pc
from tests.util import digest

pytestmark = pytest.mark.gpu
STORED = pc.reference_answers()
CLI = os.path.join(os.path.dirname(os.path.abspath(w2b.__file__)), "compute_accuracy")


class _simt:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = os.environ.get("W2B_EVAL_SIMT")
        os.environ["W2B_EVAL_SIMT"] = "1" if self.on else "0"

    def __exit__(self, *a):
        if self.old is None:
            del os.environ["W2B_EVAL_SIMT"]
        else:
            os.environ["W2B_EVAL_SIMT"] = self.old


@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_packed_file_answers_every_question_like_the_reference(tmp_path, name):
    pf, vf, qf, b, th = pc.build(name, str(tmp_path))
    report, want = po.analogy(vf, qf, b, th)
    assert digest(want) == STORED[name]["answers"] and report == STORED[name]["report"]
    for simt in (False, True):
        with _simt(simt):
            got = w2b.analogy_answers_packed(pf, qf, threshold=th)
        bad = np.nonzero(got != want)[0]
        assert len(got) == len(want) and not len(bad), (
            "simt=%d: %d of %d questions differ, first %s: gpu %s, reference %s"
            % (simt, len(bad), len(want), bad[:5], got[bad[:5]], want[bad[:5]]))
    with _simt(False):
        text, acc = w2b.compute_accuracy_packed(pf, qf, threshold=th)
    assert text == report
    assert acc["vocab"] == (th or len(pc.read_vectors(vf)[0])) and acc["size"] == pc.CASES[name][1].get("D", 32)
    print("%s: %.1f candidates and %.1f re-scored per question"
          % (name, acc["candidates"] / max(acc["questions_seen"], 1), acc["rescored"] / max(acc["questions_seen"], 1)))
    if name == "all_equal_b1":  # every score ties: the candidate list overflows and the SIMT scorer takes over
        assert acc["candidates"] > 1024 * acc["questions_seen"]
    elif not name.startswith("ties"):
        assert acc["rescored"] >= acc["questions_seen"] - 20  # the bit path answered, not the fallback


@pytest.mark.parametrize("name", ["D33_b2", "D800_b1", "V2000_threshold700_b2", "edges_b1"])
def test_cli_prints_on_the_packed_file_what_it_prints_on_the_unpacked_file(tmp_path, name):
    pf, vf, qf, b, th = pc.build(name, str(tmp_path))
    run = lambda *a: subprocess.run([CLI, *a], stdin=open(qf), capture_output=True, text=True, timeout=300)
    want = run(vf, str(b), str(th))
    assert want.returncode == 0 and want.stdout == STORED[name]["report"]
    for args in ((pf, str(b), str(th)), (pf, "0", str(th))) + (((pf,),) if not th else ()):
        got = run(*args)
        assert got.returncode == 0 and got.stdout == want.stdout, args
    other = run(pf, str(3 - b), str(th))  # re-quantising a packed file is not offered
    assert other.returncode != 0 and "<bitlevel>" in other.stdout


def _adversarial(D, bits):
    big = 0.75 if bits == 2 else 1.0 / 3
    alt = np.where(np.arange(D) % 2 == 0, big, -big)
    rows = [np.full(D, big), np.full(D, -big), alt, -alt]
    if bits == 2:
        rows += [np.full(D, 0.25), np.full(D, -0.25), np.where(np.arange(D) % 2 == 0, 0.25, -0.75),
                 np.where(np.arange(D) % 3 == 0, 0.75, 0.25)]
    return np.array(rows, np.float32)


@pytest.mark.parametrize("bits", [1, 2])
@pytest.mark.parametrize("D", [1, 3, 7, 8, 31, 32, 33, 63, 64, 65, 127, 128, 130, 200, 800, 1200, 2000])
def test_gram_is_exact_and_filter_error_is_within_eps(D, bits):
    """gram == the integer dot product; |approx - ref| <= eps for every (question, word) pair, ref the reference's
    fp32 order (normalised rows, vec = (m2 - m1) + m3, products rounded then added in index order) and also float64;
    eps <= (2 D + 32) 2^-24 1.1 max(|vec|, 1), so a loose bound cannot pass (1e-4 |vec| at D = 800, where the TF32
    filter's is 2e-3 |vec|).  The max: the roundings of the three unit-length rows that make up vec do not shrink
    when the rows nearly cancel (|vec| = 0.04 occurs at D = 3)."""
    rng = np.random.default_rng(10 * D + bits)
    adv = _adversarial(D, bits)
    vec = np.concatenate([adv, po.quantize((rng.normal(size=(700, D)) * 0.5).astype(np.float32), bits)])
    V, nadv = len(vec), len(adv)
    qid = np.concatenate([np.arange(nadv), rng.choice(np.arange(nadv, V), 90, replace=False)]).astype(np.int32)
    q3 = np.concatenate([rng.integers(0, len(qid), (150, 3)), rng.integers(0, nadv, (40, 3))]).astype(np.int32)
    gram, approx, eps = w2b.eval_packed_scores(pc.pack_rows(vec, bits), D, bits, qid, q3)
    L = pc.integer_levels(vec, bits)
    assert np.array_equal(gram, L[qid] @ L.T)

    M = po.analogy_normalize(vec, bits)
    b = qid[q3]
    Q = ((M[b[:, 1]] - M[b[:, 0]]) + M[b[:, 2]]).astype(np.float32)
    ref = np.zeros(approx.shape, np.float32)
    for a in range(D):  # sequential, each product rounded then added, as the reference's build does
        ref = ref + np.outer(Q[:, a], M[:, a])
    exact = Q.astype(np.float64) @ M.astype(np.float64).T
    norm = np.linalg.norm(Q.astype(np.float64), axis=1)
    assert np.all(eps > 0) and np.all(eps <= (2 * D + 32) * 2.0 ** -24 * 1.1 * np.maximum(norm, 1.0))
    r32 = np.abs(approx.astype(np.float64) - ref) / eps[:, None]
    r64 = np.abs(approx - exact) / eps[:, None]
    print("D=%d, %d bit: worst |approx - fp32 reference|/eps %.3f, |approx - float64|/eps %.3f, eps/|vec| %.2e .. %.2e"
          % (D, bits, r32.max(), r64.max(), (eps / norm).min(), (eps / norm).max()))
    assert r32.max() <= 1.0 and r64.max() <= 1.0
