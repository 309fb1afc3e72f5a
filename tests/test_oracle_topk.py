"""The CPU restatement of the top-k lists (tests/topk_oracle.py) and the argument checks of the top-k ABI, without a
GPU: at k = 1 the lists are w2bo_analogy's answers (the arg-max pinned against the reference), the order of the scoring
arithmetic shows in the lists, and bad arguments are refused before any device is touched."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import word2bits_b200 as w2b
from oracle import pyoracle as po
from tests import analogy_cases as ac
from tests import nearest_cases as nc
from tests import packed_cases as pc
from tests import topk_oracle as to
from tests.util import digest
from word2bits_b200 import _lib


@pytest.mark.parametrize("name", sorted(ac.CASES))
def test_lists_at_k1_are_the_oracles_answers(tmp_path, name):
    vf, qf, b, th = ac.build(name, str(tmp_path))
    _, want = po.analogy(vf, qf, b, th)
    names, M = to.load(vf, b, th)
    ids, scores = to.lists(M, to.analogy_queries(qf, names), k=3)
    assert np.array_equal(ids[:, 0], want)
    assert np.all(scores[ids >= 0] > 0) and np.all(scores[ids < 0] == 0)
    assert np.all(np.diff(scores, axis=1)[(ids[:, 1:] >= 0)] <= 0)  # best first


@pytest.mark.parametrize("name", sorted(nc.CASES))
def test_nearest_lists_skip_only_the_word_and_are_ordered(tmp_path, name):
    gf, vf, wf, words, b, th = nc.build(name, str(tmp_path))
    names, M = to.load(vf, b, th)
    queries = to.nearest_queries(words, names)
    ids, scores = to.lists(M, queries, k=10)
    assert queries[len(words) - 4] is None and np.all(ids[len(words) - 4] == -1)  # "missingword"
    for q, row, sc in zip(queries, ids, scores):
        if q is None:
            continue
        assert q[0] not in row
        live = row[row >= 0]
        key = [(-s, i) for s, i in zip(sc[: len(live)], live)]
        assert key == sorted(key)  # descending scores, the smaller index first on ties


STORED = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_nearest.json")))


@pytest.mark.parametrize("name", sorted(nc.CASES))
def test_nearest_ranks_1_2_are_the_references(tmp_path, name):
    """Ranks 1 and 2 of every nearest-neighbour list equal what the unmodified reference compute_accuracy gives, one
    question per rank (tests/golden/make_reference_nearest.py): this pins the tie order of the lists, not only their
    best word."""
    _, vf, _, words, b, th = nc.build(name, str(tmp_path))
    names, M = to.load(vf, b, th)
    ids, _ = to.lists(M, to.nearest_queries(words, names), k=2)
    assert digest(ids) == STORED[name]["ranks12"]
    assert STORED[name]["rank1_pinned"] > 0


def test_the_pins_notice_the_order_of_the_arithmetic(tmp_path):
    """The oracle's negative controls change what the pins hold: on the tie-heavy inputs the fused-scoring oracle
    (W2BO_AN_FUSED) chooses other words than the lists' rank 1, and lane-order normalisation (W2BO_AN_LANE_NORM)
    changes some ranks 1-2 of the nearest-neighbour lists pinned to the reference."""
    fused = {}
    for name in ("ties_D8_b1", "D7_b1", "edges_b1"):
        _, vf, qf, b, th = pc.build(name, str(tmp_path / name))
        names, M = to.load(vf, b, th)
        ids, _ = to.lists(M, to.analogy_queries(qf, names), k=1)
        _, plain = po.analogy(vf, qf, b, th)
        _, fus = po.analogy(vf, qf, b, th, flags=po.AN_FUSED)
        assert np.array_equal(ids[:, 0], plain)
        fused[name] = int(np.sum(ids[:, 0] != fus))
    lane = {}
    for name in ("packed_ties_D8_b1", "edges_b1", "V255_b1"):
        _, vf, _, words, b, th = nc.build(name, str(tmp_path / ("n" + name)))
        names, M = to.load(vf, b, th, flags=po.AN_LANE_NORM)
        ids, _ = to.lists(M, to.nearest_queries(words, names), k=2)
        lane[name] = digest(ids) != STORED[name]["ranks12"]
    print("questions answered otherwise with fused scoring:", fused, "ranks 1-2 moved by lane-order norms:", lane)
    assert any(fused.values()) and any(lane.values())


def test_counting_the_queries_needs_no_vectors_and_no_gpu(tmp_path):
    _, _, wf, words, _, _ = nc.build("V4_b1", str(tmp_path))
    qf = ac.build("V5_b1", str(tmp_path / "q"))[1]
    for fn, inp, want in ((_lib.lib.w2b_nearest, wf, len(words)), (_lib.lib.w2b_analogy_topk, qf, len(ac.read_questions(qf)))):
        n = C.c_int64(-1)
        assert fn(str(tmp_path / "none.bin").encode(), 0, 0, inp.encode(), 10, 0, None, None, 0, C.byref(n), None) == 0
        assert n.value == want


def _call(fn, vf=b"x", k=10, ids=True, scores=True, cap=1):
    a = np.zeros(16 * 1025, np.int32)
    s = np.zeros(16 * 1025, np.float32)
    n = C.c_int64(-7)
    return fn(vf, 0, 0, None, k, 0, _lib.ptr(a) if ids else None, _lib.ptr(s) if scores else None, cap, C.byref(n),
              None), n.value


@pytest.mark.parametrize("fn", ["w2b_analogy_topk", "w2b_nearest"])
def test_abi_refuses_bad_arguments_without_a_gpu(fn):
    f = getattr(_lib.lib, fn)
    for kw in (dict(k=0), dict(k=1025), dict(k=-1), dict(vf=None), dict(ids=False), dict(scores=False), dict(cap=-1)):
        rc, n = _call(f, **kw)
        assert rc == _lib.EINVAL and n == -7, kw
    with pytest.raises(w2b.W2BError) as e:
        w2b.nearest("/nonexistent", ["a"], 0)
    assert e.value.code == _lib.EINVAL


def test_packed_file_refuses_another_bitlevel(tmp_path):
    pf, vf, qf, b, th = pc.build("D8_b1", str(tmp_path))
    for fn, inp in ((w2b.analogy_topk, qf), (w2b.nearest, ["w0"])):
        with pytest.raises(w2b.W2BError) as e:
            fn(pf, inp, 5, bitlevel=2)
        assert e.value.code == _lib.EINVAL and "1-bit" in str(e.value)


def test_missing_vector_file_is_reported(tmp_path):
    with pytest.raises(w2b.W2BError) as e:
        w2b.nearest(str(tmp_path / "none.bin"), ["a"], 5)
    assert e.value.code == _lib.EIO and "Input file not found" in str(e.value)
