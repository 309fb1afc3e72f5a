"""Text vector files (-binary 0) without a GPU: the decimal-to-float routine the GPU text reader runs
(w2b_host_parse_floats, csrc/w2b_text.cuh) against glibc strtof bit for bit, its grammar, and the one rule that tells
binary, text and packed vector files apart (w2b_vector_file_info) with the names it reads (w2b_vector_names)."""
import ctypes as C
import os

import numpy as np
import pytest

import word2bits_b200 as w2b
from oracle import pyoracle as po
from tests import analogy_cases as ac
from tests import nearest_cases as nc
from tests import packed_cases as pc
from tests import text_cases as tc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REF_TEXT = ("reference_text_b0.txt", "reference_text_b1.txt")


def _check(tokens):
    got = w2b.host_parse_floats(" ".join(tokens)).view(np.uint32)
    want = tc.strtof_bits(tokens)
    assert len(got) == len(tokens)
    bad = np.nonzero(got != want)[0]
    assert not len(bad), "%d of %d differ, first %s: %08x, strtof %08x" % (
        len(bad), len(tokens), tokens[bad[0]], got[bad[0]], want[bad[0]])


def test_lf_of_random_float_bits_equals_strtof():
    rng = np.random.default_rng(1)
    x = rng.integers(0, 2 ** 32, 1_000_000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    tokens = [tc.lf(v) for v in x]
    _check(tokens)
    assert np.array_equal(tc.strtof_fast(tokens[:200000]), tc.strtof_bits(tokens[:200000]))  # the GPU tests' shortcut


def test_lf_of_every_quantize_level_equals_strtof():
    grid = np.linspace(-1.5, 1.5, 300001, dtype=np.float32)
    for b in range(1, 9):
        levels = np.unique(po.quantize(grid, b))
        _check([tc.lf(v) for v in levels])


@pytest.mark.parametrize("where", ["normal", "subnormal", "near_max"])
def test_midpoints_and_their_neighbours_equal_strtof(where):
    rng = np.random.default_rng({"normal": 2, "subnormal": 3, "near_max": 4}[where])
    lo, hi = {"normal": (0x00800000, 0x7F7FFFFF), "subnormal": (0, 0x00800000), "near_max": (0x7F700000, 0x7F800000)}[where]
    bits = rng.integers(lo, hi, 34000).tolist()
    bits += [lo, hi - 1]  # the ends: the smallest subnormal, FLT_MAX (its midpoint rounds to inf)
    tokens = tc.midpoint_tokens(bits)
    _check(tokens)
    _check(["-" + t for t in tokens[:20000]])


def test_exponents_leading_zeros_and_specials():
    tokens = ["0", "-0", "+0", "0.000000", "-0.000000", "00000.000100", "000123.4500e+3", ".5", "5.", "-.5e-1", "1e0",
              "1E+10", "1e-10", "1e38", "3.4028235e38", "3.40282357e38", "3.4028236e38", "1e39", "1e-45", "1.4e-45",
              "7e-46", "7.1e-46", "1e-46", "1e400", "-1e400", "1e-400", "1e999999999999999999999", "1e-99999999999999999",
              "0e999999999", "0.0000000000000000000000000000000000000000000000000000001e60", "16777217", "16777216.5",
              "16777217.000000000000000000001", "9007199254740993", "123456789012345678901234567890",
              "0.1", "0.2", "0.3", "2.5", "1.00000005960464477539062500000000001", "1.000000059604644775390625",
              "nan", "-nan", "NaN", "+NAN", "inf", "-inf", "INF", "Infinity", "-INFINITY", "+infinity", "iNfInItY",
              "0.333333", "-0.333333", "0.250000", "0.750000", "1" + "0" * 60, "0." + "0" * 60 + "1"]
    _check(tokens)
    assert np.signbit(w2b.host_parse_floats("-0.000000")[0])


@pytest.mark.parametrize("token", ["", "-", "+", ".", "-.", "e5", "1e", "1e+", "1e-", "1.2.3", "0x1p3", "0x10", "12a",
                                   "1,5", "nana", "infinit", "infinityy", "in", "n", "--1", "+-1", "1e5.0", "1d5", "\x00",
                                   "nan(1)", "1_000"])
def test_tokens_outside_the_grammar_are_refused(token):
    with pytest.raises(w2b.W2BError) as e:
        w2b.host_parse_floats("1.0 " + token + " 2.0") if token else w2b.host_parse_floats("1.0 - 2.0")
    assert e.value.code == w2b._lib.EIO and "token 1" in str(e.value)


def test_separators():
    assert w2b.host_parse_floats("  1.5\t-2\r\n3e1 \n").tolist() == [1.5, -2.0, 30.0]
    assert len(w2b.host_parse_floats("")) == 0 and len(w2b.host_parse_floats(" \n ")) == 0


# ---- the format rule
def test_golden_files_keep_their_kind():
    for name in sorted(os.listdir(GOLDEN)):
        kind = w2b.vector_file_info(os.path.join(GOLDEN, name))[0]
        assert kind == ("text" if name in REF_TEXT else "binary"), name
    for name, D in zip(REF_TEXT, (12, 8)):
        kind, V, d, bits = w2b.vector_file_info(os.path.join(GOLDEN, name))
        assert (kind, d, bits) == ("text", D, 0) and V > 10
        assert w2b.vector_file_info(os.path.join(GOLDEN, name), threshold=5)[1] == 5


@pytest.mark.parametrize("gen", ["analogy", "packed", "nearest"])
def test_generated_files_keep_their_kind(tmp_path, gen):
    cases = {"analogy": ac.CASES, "packed": pc.CASES, "nearest": nc.CASES}[gen]
    for name in sorted(cases):
        d = str(tmp_path / name)
        if gen == "analogy":
            files = {ac.build(name, d)[0]: "binary"}
        elif gen == "packed":
            pf, vf = pc.build(name, d)[:2]
            files = {pf: "packed", vf: "binary"}
        else:
            gf, vf = nc.build(name, d)[:2]
            files = {gf: "packed" if gf != vf else "binary", vf: "binary"}
        for f, kind in files.items():
            assert w2b.vector_file_info(f)[0] == kind, (name, f)


def test_corpus_writer_files(tmp_path):
    c = w2b.Corpus(os.path.join(GOLDEN, "golden_corpus.txt"), 1)
    rng = np.random.default_rng(5)
    for b in (0, 1, 2, 8):
        vec = po.quantize(rng.normal(size=(c.vocab_size, 24)).astype(np.float32) * 0.4, b)
        for binary, kind in ((0, "text"), (1, "binary")):
            f = str(tmp_path / ("v%d_%d" % (b, binary)))
            c.write_vectors(f, vec, binary)
            assert w2b.vector_file_info(f) == (kind, c.vocab_size, 24, 0)
        names, rows = tc.read_tokens(str(tmp_path / ("v%d_0" % b)))
        assert names == c.words() and all(len(r) == 24 for r in rows)
    c.close()


def test_binary_rows_of_ascii_digits_stay_binary(tmp_path):
    f = str(tmp_path / "d1.bin")
    with open(f, "wb") as o:  # D = 1: each value's 4 bytes are ASCII digits, which also read as one token
        o.write(b"3 1\nw1 1234\nw2 5678\nw3 0.25\n")
    assert w2b.vector_file_info(f) == ("binary", 3, 1, 0)
    with open(f, "wb") as o:  # D = 2: "0.5 0.25" is 8 bytes, two tokens
        o.write(b"1 2\nw 0.5 0.25\n")
    assert w2b.vector_file_info(f)[0] == "binary"
    with open(f, "wb") as o:  # the same bytes with one more space: not '\n' after 4 D bytes, two tokens: text
        o.write(b"1 2\nw 0.5  0.25\n")
    assert w2b.vector_file_info(f)[0] == "text"


def test_first_row_must_hold_d_tokens(tmp_path):
    f = str(tmp_path / "t.txt")
    for row, kind in ((b"0.100000 0.200000 0.300000 ", "text"), (b"0.100000 0.200000 ", "binary"),
                      (b"0.100000 0.200000 0.300000 0.400000 ", "binary"), (b"0.100000 0.200000 x.000000 ", "binary"),
                      (b"0.100000 0.200000 0x300000 ", "binary"), (b"0.100000 nan -inf", "text"),
                      (b"0.1 0.2 0.3 ", "binary")):  # 12 bytes = 4 D, then '\n': a binary row (no "%lf" row is)
        with open(f, "wb") as o:
            o.write(b"2 3\nw " + row + b"\nv 1 2 3 \n")
        assert w2b.vector_file_info(f)[0] == kind, row
    with open(f, "wb") as o:
        o.write(b"1 2 1\nw \x01\n")
    assert w2b.vector_file_info(f) == ("packed", 1, 2, 1)
    with pytest.raises(w2b.W2BError):
        w2b.vector_file_info(str(tmp_path / "missing"))


def test_names_of_every_kind(tmp_path):
    vf, _, _, _ = ac.build("edges_b1", str(tmp_path))
    want = ac.vocab_names(vf)
    tf, _ = tc.twin(vf, str(tmp_path))
    pf = pc.build("edges_b1", str(tmp_path / "p"))[0]
    for f, names in ((vf, want), (tf, want), (pf, ac.vocab_names(pc.build("edges_b1", str(tmp_path / "p"))[1]))):
        for th in (0, 7):
            V = w2b.vector_file_info(f, th)[1]
            buf = np.zeros((V, 51), np.uint8)
            n = C.c_int64()
            w2b._lib.check(w2b._lib.lib.w2b_vector_names(f.encode(), th, w2b._lib.ptr(buf), 51, C.byref(n)))
            got = [bytes(r[: list(r).index(0)]).decode("latin1") for r in buf]
            assert n.value == V and got == names[:V], f
