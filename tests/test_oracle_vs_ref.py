"""Pins the CPU oracle (oracle/w2b_oracle.c) against the UNMODIFIED reference compiled as a
library (oracle/_ref/libw2b_ref_strict.so = -O2 -ffp-contract=off -fno-tree-vectorize), through what
that library computed on the same seeded inputs (tests/golden/reference_outputs.json, written by
tests/golden/make_reference_outputs.py).  Bit-exact on: quantize, expTable, vocab order/counts, InitNet,
the unigram table, and the trained u / v / alpha / word_count_actual / loss after running shards
sequentially."""
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.util import bits, digest, reference_outputs, zipf_corpus

QUANTIZE_XS = [0.0, -0.0, 1e-30, -1e-30, .25, .5, float(np.nextafter(np.float32(.5), np.float32(1))), .75, 1.0, -1.0,
               3.7, -3.7, 1 / 32, .0624, .0625, .09375, 0.49999, -0.5, -0.50001, 0.124, 0.126]
QUANTIZE_XS += [float(x) for x in np.random.default_rng(0).uniform(-1.5, 1.5, 500).astype(np.float32)]


@pytest.fixture(scope="module")
def want():
    return reference_outputs("oracle_vs_ref")


def test_quantize_bits(want):
    for b in range(0, 9):
        got = np.array([bits(np.float32(po.lib().w2bo_quantize(float(np.float32(x)), b))) for x in QUANTIZE_XS],
                       np.uint32)
        assert digest(got) == want["quantize"][b], b
    # README.md:12-17,124-131 known answers
    assert [int(np.float32(po.lib().w2bo_quantize(x, 1)).view(np.uint32)) for x in (0.7, -0.7, -0.0)] == \
        [0x3EAAAAAB, 0xBEAAAAAB, 0x3EAAAAAB]


@pytest.fixture(scope="module")
def small(tmp_path_factory):
    d = tmp_path_factory.mktemp("c")
    return zipf_corpus(str(d / "small.txt"), 12500, 30, seed=1, newline_every=15)


@pytest.fixture(scope="module")
def medium(tmp_path_factory):
    d = tmp_path_factory.mktemp("c")
    return zipf_corpus(str(d / "medium.txt"), 60000, 3000, seed=2)


def test_exptable():
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_strict.npz"))
    assert np.array_equal(bits(gold["exptable"]), bits(po.exptable()))


@pytest.mark.parametrize("min_count", [1, 5])
def test_vocab_and_init(small, medium, min_count, want):
    for name, path in (("small", small), ("medium", medium)):
        w = want["vocab_%s_mc%d" % (name, min_count)]
        c = po.Corpus(path, min_count)
        assert c.vocab_size == w["V"] and c.train_words == w["train_words"] and c.file_size == w["file_size"]
        assert digest(c.words()) == w["words"]
        assert digest(c.counts) == w["counts"]
        u, v = po.init_net(c.vocab_size, 8)
        assert digest(bits(u)) == w["u"] and digest(bits(v)) == w["v"]


def test_unigram_table(medium, want):
    c = po.Corpus(medium, 1)
    t = po.unigram_table(c.counts)
    assert digest(t) == want["unigram_table_medium"]
    s = po.unigram_bounds(c.counts)
    # boundary form reproduces the table
    idx = np.searchsorted(s, np.arange(0, po.TABLE_SIZE, 9973), side="right") - 1
    assert np.array_equal(idx, t[::9973])
    assert s[0] == 0 and s[-1] == po.TABLE_SIZE and np.all(np.diff(s) >= 0)


CASES = [
    # path, D, W, neg, bits, shards, min_count, sample, reg, iters
    ("small", 8, 3, 4, 1, 1, 1, 1e-3, 0.0, 1),
    ("small", 8, 3, 4, 2, 1, 1, 1e-3, 0.0, 1),
    ("small", 8, 3, 4, 0, 1, 1, 1e-3, 0.0, 1),
    ("small", 8, 3, 4, 5, 1, 1, 1e-3, 0.0, 1),
    ("small", 8, 3, 4, 3, 1, 1, 1e-3, 0.0, 1),
    ("small", 12, 5, 6, 1, 3, 1, 1e-2, 0.0, 2),
    ("small", 8, 3, 4, 1, 1, 1, 0.0, 0.0, 1),
    ("small", 8, 3, 4, 2, 2, 5, 1e-3, 0.01, 1),
    ("medium", 20, 5, 6, 1, 4, 5, 1e-3, 0.0, 2),
    ("medium", 16, 4, 5, 0, 3, 1, 1e-4, 0.0, 1),
    # windows wider than 64 and more than 63 negatives (the reference has no bound on either; until round 2 the port
    # kept a position's context ids in a 130-entry buffer — found when the product's window limit went to 512)
    ("medium", 8, 300, 4, 1, 2, 1, 1e-3, 0.0, 1),
    ("small", 8, 100, 70, 0, 1, 1, 1e-3, 0.0, 1),
]


@pytest.mark.parametrize("case", CASES)
def test_trajectory_bit_exact(case, small, medium, want):
    name, D, W, neg, b, shards, mc, sample, reg, iters = case
    w = want["trajectories"][CASES.index(case)]
    path = {"small": small, "medium": medium}[name]
    c = po.Corpus(path, mc)
    m = po.OracleModel(c, D, W, neg, b, shards=shards, iters=iters, sample=sample, reg=reg)
    k = 0
    for _ in range(iters):
        for sid in range(shards):
            lo = m.train_shard(sid)
            assert lo == w["loss"][k], (sid, lo, w["loss"][k])
            assert int(np.float32(m.alpha).view(np.uint32)) == w["alpha"][k]
            assert m.word_count_actual == w["wca"][k]
            k += 1
    assert digest(bits(m.u)) == w["u"]
    assert digest(bits(m.v)) == w["v"]
    # the run must actually have trained something
    u0, v0 = po.init_net(c.vocab_size, D)
    if b != 3:  # bitlevel 3 quantizes everything to +-0 (:73-108 quirk): nothing moves
        assert not np.array_equal(bits(m.u), bits(u0))
