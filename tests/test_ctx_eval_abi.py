"""The evaluator on a context's own tables (w2b_ctx_*), the parts that need no device: the C ABI rejects null
arguments and a bad k with W2B_EINVAL, and the CLI refuses a missing -eval questions file before it reads the
corpus."""
import ctypes as C
import os
import subprocess

import numpy as np

from word2bits_b200._lib import EINVAL, TopkStats, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "word2bits_b200", "word2bits")


def test_null_arguments_are_invalid():
    names = (C.c_char_p * 2)(b"a", b"b")
    n = C.c_int64()
    ids, scores = np.zeros(4, np.int32), np.zeros(4, np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    st = TopkStats()
    for ctx, words in ((None, names), (None, None), (C.c_void_p(8), None)):
        assert lib.w2b_ctx_compute_accuracy(ctx, words, 0, 0, b"q", None, None, 0) == EINVAL
        assert lib.w2b_ctx_analogy_answers(ctx, words, 0, 0, b"q", p(ids), 4, C.byref(n)) == EINVAL
        assert lib.w2b_ctx_analogy_topk(ctx, words, 0, 0, b"q", 1, p(ids), p(scores), 4, C.byref(n), C.byref(st)) == EINVAL
        assert lib.w2b_ctx_nearest(ctx, words, 0, 0, b"q", 1, p(ids), p(scores), 4, C.byref(n), C.byref(st)) == EINVAL
    assert "null words" in lib.w2b_last_error().decode()
    assert lib.w2b_ctx_compute_accuracy(None, names, 0, 0, b"q", None, None, 0) == EINVAL
    assert "null ctx" in lib.w2b_last_error().decode()
    assert lib.w2b_ctx_analogy_answers(None, names, 0, 0, b"q", None, 4, C.byref(n)) == EINVAL  # rows without a buffer
    for k in (0, -1, 1025):
        assert lib.w2b_ctx_analogy_topk(None, names, 0, 0, b"q", k, p(ids), p(scores), 4, None, None) == EINVAL
        assert lib.w2b_ctx_nearest(None, names, 0, 0, b"q", k, p(ids), p(scores), 4, None, None) == EINVAL
    assert lib.w2b_ctx_nearest(None, names, 0, 0, b"q", 1, None, None, 4, None, None) == EINVAL  # rows without buffers


def test_missing_eval_file_stops_before_the_corpus_is_read(tmp_path):
    corpus = os.path.join(ROOT, "tests", "golden", "golden_corpus.txt")
    missing = str(tmp_path / "no-questions.txt")
    got = subprocess.run([CLI, "-train", corpus, "-output", str(tmp_path / "vec.bin"), "-eval", missing],
                         capture_output=True, text=True, timeout=60)
    assert got.returncode == 1
    assert got.stdout == "ERROR: questions file %s not found!\n" % missing
    assert not os.path.exists(tmp_path / "vec.bin")
