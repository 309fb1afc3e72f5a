"""Text vector files (-binary 0) parsed on the GPU (csrc/w2b_text.cu): every value equals glibc strtof of its token,
bit for bit, on files the reference wrote, on files this project writes at bit levels 0, 1, 2 and 8, on long and
exponent tokens and on files whose rows cross many chunk boundaries; malformed rows name their row and token; and the
evaluator gives on a text file exactly what it gives on the binary file holding the strtof values of its tokens (that
route is pinned to the reference): reports, answers, top-k ids and score bits, nearest lists and CLI output."""
import os
import subprocess

import numpy as np
import pytest

import word2bits_b200 as w2b
from oracle import pyoracle as po
from tests import analogy_cases as ac
from tests import nearest_cases as nc
from tests import text_cases as tc

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HERE = os.path.dirname(os.path.abspath(w2b.__file__))


def _same_as_strtof(path):
    names, vec = w2b.read_text_vectors(path)
    want_names, rows = tc.read_tokens(path)
    want = tc.strtof_bits([t for r in rows for t in r]).reshape(len(rows), -1)
    assert names == want_names
    bad = np.argwhere(vec.view(np.uint32) != want)
    assert not len(bad), "%d values differ, first at %s: %08x, strtof %08x" % (
        len(bad), bad[0], vec.view(np.uint32)[tuple(bad[0])], want[tuple(bad[0])])
    return vec


@pytest.mark.parametrize("name", ["reference_text_b0.txt", "reference_text_b1.txt"])
def test_reference_written_files(name):
    vec = _same_as_strtof(os.path.join(GOLDEN, name))
    if name.endswith("b1.txt"):
        assert set(np.abs(vec).ravel().tolist()) == {np.float32(0.333333)}


@pytest.mark.parametrize("bits", [0, 1, 2, 8])
def test_corpus_writer_files(tmp_path, bits):
    c = w2b.Corpus(os.path.join(GOLDEN, "golden_corpus.txt"), 1)
    vec = po.quantize(np.random.default_rng(bits).normal(size=(c.vocab_size, 50)).astype(np.float32) * 0.4, bits)
    f = str(tmp_path / "v.txt")
    c.write_vectors(f, vec, 0)
    _same_as_strtof(f)
    c.close()


def test_long_and_exponent_tokens(tmp_path):
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 0x7F800000, 3000).tolist() + [0, 1, 0x7FFFFF, 0x800000, 0x7F7FFFFE]
    toks = tc.midpoint_tokens(bits)
    toks += ["-" + t for t in toks[:500]] + ["nan", "-nan", "INF", "-Infinity", "1e-400", "-1e400", ".5", "5.", "+3E+2"]
    toks += ["%.9e" % x for x in rng.normal(size=500)] + ["0" * 70 + "1." + "0" * 30 + "e-5"]
    D = 37
    toks += ["0"] * (-len(toks) % D)
    rows = [toks[i:i + D] for i in range(0, len(toks), D)]
    f = str(tmp_path / "long.txt")
    with open(f, "w") as o:
        o.write("%d %d\n" % (len(rows), D))
        for k, r in enumerate(rows):  # tabs, several spaces, no trailing space, CRLF
            sep = ("  ", "\t", " ")[k % 3]
            o.write("w%d %s%s\n" % (k, sep.join(r), "\r" if k % 5 == 0 else ""))
    assert w2b.vector_file_info(f)[0] == "text"
    _same_as_strtof(f)


class _chunk:
    def __init__(self, n):
        self.n = n

    def __enter__(self):
        os.environ["W2B_TEXT_CHUNK_BYTES"] = str(self.n)

    def __exit__(self, *a):
        del os.environ["W2B_TEXT_CHUNK_BYTES"]


@pytest.mark.parametrize("chunk", [1 << 20, 10007, 3000, 64])  # 64: every row is longer than a chunk
def test_rows_across_chunk_boundaries(tmp_path, chunk):
    rng = np.random.default_rng(11)
    V, D = 5000, 90
    names = ["w%d" % i for i in range(V)]
    vec = (rng.normal(size=(V, D)) * np.exp(rng.uniform(-8, 8, (V, 1)))).astype(np.float32)
    f = str(tmp_path / "big.txt")
    tc.write_text(f, names, vec)
    assert os.path.getsize(f) > 20 * 3000
    with _chunk(chunk):
        _same_as_strtof(f)
        got = w2b.read_text_vectors(f)[1]
    assert np.array_equal(got.view(np.uint32), w2b.read_text_vectors(f)[1].view(np.uint32))


def test_malformed_rows_name_row_and_token(tmp_path):
    f = str(tmp_path / "bad.txt")
    good = " ".join(["0.500000"] * 4)
    for row, msg in (("0.500000 0.500000 0.500000", "row 3 (w3) has fewer than 4 values"),
                     (good + " 0.1", "row 3 (w3) has more than 4 values"),
                     ("0.500000 0.5x0000 0.500000 0.500000", "row 3 (w3), value 1: '0.5x0000' is not a number"),
                     ("0.500000 0.500000 0.500000 0x1p3", "row 3 (w3), value 3: '0x1p3' is not a number")):
        lines = ["w%d %s \n" % (k, good) for k in range(6)]
        lines[3] = "w3 %s \n" % row
        lines[5] = "w5 0.1 \n"  # a later row that is also wrong: the first one is reported
        with open(f, "w") as o:
            o.write("6 4\n" + "".join(lines))
        with _chunk(40):  # the bad row's chunk is parsed after others
            with pytest.raises(w2b.W2BError) as e:
                w2b.read_text_vectors(f)
        assert e.value.code == w2b._lib.EIO and msg in str(e.value), str(e.value)
    with open(f, "w") as o:
        o.write("6 4\n" + "".join("w%d %s \n" % (k, good) for k in range(4)))
    with pytest.raises(w2b.W2BError, match="truncated at word 4"):
        w2b.read_text_vectors(f)
    qf = str(tmp_path / "q.txt")
    open(qf, "w").write(": s\nw0 w1 w2 w3\n")
    with pytest.raises(w2b.W2BError, match="truncated at word 4"):
        w2b.compute_accuracy(f, qf)
    rep, _ = w2b.compute_accuracy(f, qf, threshold=4)  # the first 4 rows are whole
    assert "Questions seen / total: 1 1" in rep


def _same_lists(a, b, tag):
    assert np.array_equal(a[0], b[0]), tag
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)), tag
    assert a[2]["packed"] == 0 and b[2]["packed"] == 0 and a[2]["queries"] == b[2]["queries"], tag


@pytest.mark.parametrize("name", sorted(ac.CASES))
def test_analogy_cases_text_equals_binary(tmp_path, name):
    vf, qf, b, th = ac.build(name, str(tmp_path))
    tf, bf = tc.twin(vf, str(tmp_path))
    assert w2b.vector_file_info(tf)[0] == "text"
    rt, at = w2b.compute_accuracy(tf, qf, bitlevel=b, threshold=th)
    rb, ab = w2b.compute_accuracy(bf, qf, bitlevel=b, threshold=th)
    assert rt == rb
    for k in ("questions_seen", "correct", "rescored", "vocab", "size"):  # (candidates depends on CTA order)
        assert at[k] == ab[k], k
    assert np.array_equal(w2b.analogy_answers(tf, qf, bitlevel=b, threshold=th),
                          w2b.analogy_answers(bf, qf, bitlevel=b, threshold=th))
    for k in (1, 10):
        _same_lists(w2b.analogy_topk(tf, qf, k, bitlevel=b, threshold=th),
                    w2b.analogy_topk(bf, qf, k, bitlevel=b, threshold=th), "%s k=%d" % (name, k))
    if name in ("edges_b1", "V2000_threshold700_b1", "bits1_quantized"):
        cli = os.path.join(HERE, "compute_accuracy")
        out = [subprocess.run([cli, f, str(b), str(th)], stdin=open(qf), capture_output=True, text=True, timeout=300)
               for f in (tf, bf)]
        assert out[0].returncode == 0 and out[0].stdout == out[1].stdout


@pytest.mark.parametrize("name", sorted(nc.CASES))
def test_nearest_cases_text_equals_binary(tmp_path, name):
    gf, vf, wf, words, b, th = nc.build(name, str(tmp_path))
    tf, bf = tc.twin(vf, str(tmp_path))
    for k in (1, 10, 100):
        _same_lists(w2b.nearest(tf, wf, k, bitlevel=b, threshold=th), w2b.nearest(bf, wf, k, bitlevel=b, threshold=th),
                    "%s k=%d" % (name, k))
    if name in ("edges_b1", "V2000_threshold700_b1", "packed_edges_b2"):
        cli = os.path.join(HERE, "nearest")
        out = [subprocess.run([cli, f, "5", str(b), str(th)], stdin=open(wf), capture_output=True, text=True, timeout=300)
               for f in (tf, bf)]
        assert out[0].returncode == 0 and out[0].stdout == out[1].stdout and out[0].stdout.count("\n") > len(words)
