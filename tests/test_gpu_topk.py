"""Top-k lists on the GPU (w2b_analogy_topk, w2b_nearest; csrc/w2b_eval_topk.cuh) against the CPU restatement
(tests/topk_oracle.py), query by query: identical ids and bit-identical scores at every k, on the filter path (TF32 or
bit-domain scores, then exact re-scores) and on the exact SIMT path (W2B_EVAL_SIMT=1).  At k = 1 the lists are the
evaluator's answers.  Each run states which path it took: the all-equal inputs overflow the candidate lists into the
SIMT fall-back, the 40 000-word inputs cross several vocabulary chunks, the others stay on the filter."""
import os
import subprocess

import numpy as np
import pytest

import word2bits_b200 as w2b
from tests import analogy_cases as ac
from tests import nearest_cases as nc
from tests import packed_cases as pc
from tests import topk_oracle as to

pytestmark = pytest.mark.gpu
KS = (1, 10, 100, 1024)
CLI = os.path.join(os.path.dirname(os.path.abspath(w2b.__file__)), "nearest")


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


def _path(name, k):
    """The path a filter run must take: 1 = SIMT fall-back (overflow), 0 = filter, None = either (1-bit ties at D = 8
    fill a list or not depending on k)."""
    if "all_equal" in name:
        return 1 if k <= 10 else 0  # 1500 equal words: more than 8k + 1024 candidates while k <= 10
    return None if "ties" in name else 0


def _compare(run, want_ids, want_scores, name, packed, answers=None):
    for simt in (False, True):
        for k in KS:
            with _simt(simt):
                ids, scores, st = run(k)
            tag = "%s simt=%d k=%d" % (name, simt, k)
            assert ids.shape == (len(want_ids), k), tag
            bad = np.nonzero(np.any(ids != want_ids[:, :k], axis=1))[0]
            assert not len(bad), "%s: %d lists differ, first %s: gpu %s, oracle %s" % (
                tag, len(bad), bad[:3], ids[bad[0]][:8], want_ids[bad[0]][:8])
            assert np.array_equal(scores.view(np.uint32), want_scores[:, :k].view(np.uint32)), tag
            assert st["queries"] == len(want_ids) and st["packed"] == packed, (tag, st)
            if simt:
                assert st["simt"] == 1, (tag, st)
            elif _path(name, k) is not None:
                assert st["simt"] == _path(name, k), (tag, st)
            if "V40000" in name and not simt:
                assert st["chunks"] >= 3, (tag, st)
            if k == 1 and answers is not None:
                assert np.array_equal(ids[:, 0], answers), tag
            print("%s: %d chunks, %.1f candidates and %.1f re-scored per query, simt %d, %.2f ms"
                  % (tag, st["chunks"], st["candidates"] / max(st["queries"], 1), st["rescored"] / max(st["queries"], 1),
                     st["simt"], st["gpu_ms"]))


@pytest.mark.parametrize("name", sorted(ac.CASES))
def test_analogy_lists_equal_the_oracle(tmp_path, name):
    vf, qf, b, th = ac.build(name, str(tmp_path))
    names, M = to.load(vf, b, th)
    want = to.lists(M, to.analogy_queries(qf, names))
    with _simt(False):
        answers = w2b.analogy_answers(vf, qf, bitlevel=b, threshold=th)
    _compare(lambda k: w2b.analogy_topk(vf, qf, k, bitlevel=b, threshold=th), *want, name, 0, answers)


@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_packed_analogy_lists_equal_the_oracle(tmp_path, name):
    pf, vf, qf, b, th = pc.build(name, str(tmp_path))
    names, M = to.load(vf, b, th)
    want = to.lists(M, to.analogy_queries(qf, names))
    with _simt(False):
        answers = w2b.analogy_answers_packed(pf, qf, threshold=th)
        fp32 = w2b.analogy_topk(vf, qf, 10, bitlevel=b, threshold=th)
        packed = w2b.analogy_topk(pf, qf, 10, threshold=th)
    assert np.array_equal(fp32[0], packed[0]) and np.array_equal(fp32[1].view(np.uint32), packed[1].view(np.uint32))
    _compare(lambda k: w2b.analogy_topk(pf, qf, k, threshold=th), *want, name, 1, answers)


@pytest.mark.parametrize("name", sorted(nc.CASES))
def test_nearest_lists_equal_the_oracle(tmp_path, name):
    gf, vf, wf, words, b, th = nc.build(name, str(tmp_path))
    names, M = to.load(vf, b, th)
    want = to.lists(M, to.nearest_queries(words, names))
    packed = int(gf != vf)
    _compare(lambda k: w2b.nearest(gf, wf, k, bitlevel=0 if packed else b, threshold=th), *want, name, packed)
    ids, scores, st = w2b.nearest(gf, words[:50], 7, bitlevel=0 if packed else b, threshold=th)  # a list of words
    assert np.array_equal(ids, want[0][:50, :7])


def test_cli_prints_the_lists(tmp_path):
    gf, vf, wf, words, b, th = nc.build("edges_b1", str(tmp_path))
    ids, scores, _ = w2b.nearest(gf, wf, 5, bitlevel=b)
    names = [n.upper() for n in pc.read_vectors(vf)[0]]
    want = []
    for w, row, sc in zip(words, ids, scores):
        if row[0] < 0 and w.upper() not in names:
            want.append("%s: not in vocabulary" % w.upper())
            continue
        want.append("%s:" % w.upper())
        want += ["%d\t%s\t%f" % (j + 1, names[c], s) for j, (c, s) in enumerate(zip(row, sc)) if c >= 0]
    got = subprocess.run([CLI, gf, "5", str(b)], stdin=open(wf), capture_output=True, text=True, timeout=300)
    assert got.returncode == 0 and got.stdout == "\n".join(want) + "\n"
    missing = subprocess.run([CLI, str(tmp_path / "none.bin")], stdin=open(wf), capture_output=True, text=True)
    assert missing.returncode != 0 and missing.stdout == "Input file not found\n"
