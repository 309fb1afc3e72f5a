"""The pin of the packed evaluator: on the unpacked file of every case of tests/packed_cases.py the CPU restatement
of src/compute-accuracy.c (oracle w2bo_analogy) reproduces what the reference itself answered
(tests/golden/reference_packed.json, written by tests/golden/make_reference_packed.py), and the packed file of the
case holds exactly those vectors.  Controls: the Gram kernel's popcount formulas, restated in numpy, equal the integer
dot product, and stop doing so when a padding bit is set, the magnitude plane is dropped or the planes are swapped —
so the GPU equality test of tests/test_gpu_evaluator_packed.py can fail."""
import numpy as np
import pytest

import word2bits_b200 as w2b
from oracle import pyoracle as po
from tests import packed_cases as pc
from tests.util import digest

STORED = pc.reference_answers()


def test_every_case_is_stored():
    assert set(STORED) == set(pc.CASES)


@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_oracle_answers_like_the_reference_on_the_unpacked_file(tmp_path, name):
    pf, vf, qf, b, th = pc.build(name, str(tmp_path))
    report, ans = po.analogy(vf, qf, b, th)
    assert report == STORED[name]["report"]
    assert digest(ans) == STORED[name]["answers"]
    names, vec = pc.read_vectors(vf)
    words, back, bits = w2b.read_packed(pf)  # the library's own reader sees the same table
    assert bits == b and words == names and np.array_equal(back.view(np.uint32), vec.view(np.uint32))


@pytest.mark.parametrize("bits", [1, 2])
@pytest.mark.parametrize("D", [1, 31, 32, 33, 64, 130, 800])
def test_popcount_formulas_equal_the_integer_dot_product(D, bits):
    rng = np.random.default_rng(D + bits)
    vec = po.quantize((rng.normal(size=(40, D)) * 0.5).astype(np.float32), bits)
    L = pc.integer_levels(vec, bits)
    exact = L[:7] @ L.T
    n, h = pc.planes(vec, bits)
    assert np.array_equal(pc.gram_from_planes(n[:7], h[:7], n, h, D, bits), exact)
    if D % 32:  # a set padding bit is counted as a sign difference
        bad = n.copy()
        bad[:, -1] |= np.uint32(1 << 31)
        assert not np.array_equal(pc.gram_from_planes(n[:7], h[:7], bad, h, D, bits), exact)
    if bits == 2:
        assert not np.array_equal(pc.gram_from_planes(n[:7], h[:7], n, np.zeros_like(h), D, bits), exact)
        assert not np.array_equal(pc.gram_from_planes(h[:7], n[:7], h, n, D, bits), exact)
