"""The C ABI of the packed evaluator rejects bad input with an error code: no crash, and no device needed."""
import ctypes as C

import numpy as np

from word2bits_b200._lib import EINVAL, EIO, lib
from tests import analogy_cases as ac
from tests import packed_cases as pc


def _files(tmp_path, D=40, V=30, bits=2):
    rng = np.random.default_rng(0)
    vec = np.where(rng.random((V, D)) < 0.5, -0.25, 0.75).astype(np.float32)
    names = ["w%d" % i for i in range(V)]
    pf, vf, qf = (str(tmp_path / n) for n in ("vec.packed", "vec.bin", "q.txt"))
    pc.write_packed(pf, names, pc.pack_rows(vec, bits), D, bits)
    ac.write_vectors(vf, names, vec)
    ac.write_questions(qf, [["w1", "w2", "w3", "w4"]])
    return pf, vf, qf


def _both(path, qf):
    n, ans = C.c_int64(), np.zeros(8, np.int32)
    return (lib.w2b_compute_accuracy_packed(path, 0, qf, 0, None, None, 0),
            lib.w2b_analogy_answers_packed(path, 0, qf, 0, ans.ctypes.data_as(C.c_void_p), len(ans), C.byref(n)))


def test_null_pointers_are_invalid_arguments():
    assert lib.w2b_compute_accuracy_packed(None, 0, None, 0, None, None, 0) == EINVAL
    assert lib.w2b_analogy_answers_packed(None, 0, None, 0, None, 0, None) == EINVAL
    assert lib.w2b_analogy_answers_packed(b"x", 0, b"y", 0, None, 4, None) == EINVAL
    assert lib.w2b_eval_packed_scores(None, 1, 1, 1, None, 1, None, 0, 0, None, None, None) == EINVAL
    rows, qid, gram = np.zeros((2, 1), np.uint8), np.zeros(1, np.int32), np.zeros(2, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.w2b_eval_packed_scores(p(rows), 2, 8, 3, p(qid), 1, None, 0, 0, p(gram), None, None) == EINVAL  # bit level
    qid[0] = 2
    assert lib.w2b_eval_packed_scores(p(rows), 2, 8, 1, p(qid), 1, None, 0, 0, p(gram), None, None) == EINVAL  # word id
    qid[0] = 0
    assert lib.w2b_eval_packed_scores(p(rows), 2, 8, 1, p(qid), 1, None, 1, 0, p(gram), None, None) == EINVAL  # no q3


def test_missing_and_foreign_files_are_io_errors(tmp_path):
    pf, vf, qf = _files(tmp_path)
    assert _both(str(tmp_path / "nothing").encode(), qf.encode()) == (EIO, EIO)
    assert _both(vf.encode(), qf.encode()) == (EIO, EIO)  # a word2vec-binary file: two header fields
    assert b"not a packed vector file" in lib.w2b_last_error()


def test_truncated_file_is_an_io_error(tmp_path):
    pf, vf, qf = _files(tmp_path)
    data = open(pf, "rb").read()
    for cut in (len(data) - 3, len(data) // 2, data.index(b"\n") + 1):
        short = str(tmp_path / "short.packed")
        open(short, "wb").write(data[:cut])
        assert _both(short.encode(), qf.encode()) == (EIO, EIO), cut


def test_bad_headers_are_io_errors(tmp_path):
    pf, vf, qf = _files(tmp_path)
    body = open(pf, "rb").read().split(b"\n", 1)[1]
    for header in (b"30 40 3", b"30 40 0", b"30 0 2", b"0 40 2", b"-5 40 2", b"30 40 2 7", b"30 99999999999 2",
                   b"99999999999 40 2", b"30 40 x"):
        bad = str(tmp_path / "bad.packed")
        open(bad, "wb").write(header + b"\n" + body)
        assert _both(bad.encode(), qf.encode()) == (EIO, EIO), header
