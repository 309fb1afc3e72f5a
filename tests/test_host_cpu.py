"""CPU-only tests of the product's host side: the C-ABI library loads without a GPU and exports
every symbol include/w2b.h declares; the corpus/vocabulary glue equals the oracle (and through
it the reference); the CLI reproduces the reference's messages and exit codes; compute entry
points fail loudly (no CPU fallback)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from tests.util import digest, reference_outputs, zipf_corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "word2bits_b200", "libw2b.so")
CLI = os.path.join(ROOT, "word2bits_b200", "word2bits")


def _has_gpu():
    import word2bits_b200 as w2b
    return w2b.device_count() > 0


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "w2b.h")).read()
    names = set(re.findall(r"\b(w2b_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 35
    lib = ctypes.CDLL(LIB)
    for n in sorted(names):
        assert hasattr(lib, n), n


def test_no_cpu_fallback():
    import word2bits_b200 as w2b
    if _has_gpu():
        pytest.skip("GPU present")
    with pytest.raises(w2b.W2BError) as e:
        w2b.Trainer(None, vocab_size=100, size=8, threads=2)
    assert e.value.code == 2  # W2B_ECUDA


def test_product_does_not_import_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "word2bits_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert "pyoracle" not in src and "liboracle" not in src and "w2b_oracle" not in src, f
                # the emulator (tests/emu) is reachable only through the W2B_EMULATE seam of w2b_ptx.cuh,
                # a macro no product build defines
                if "w2b_emu" in src or "libw2bemu" in src:
                    assert f == "w2b_ptx.cuh" and src.count('#include "w2b_emu_ptx.h"') == 1 and "#ifdef W2B_EMULATE" in src, f


@pytest.mark.parametrize("newline_every,min_count,vocab", [(0, 5, 3000), (15, 1, 30), (7, 2, 200)])
def test_corpus_matches_oracle(tmp_path, newline_every, min_count, vocab):
    import word2bits_b200 as w2b
    path = zipf_corpus(str(tmp_path / "c.txt"), 50000, vocab, seed=11, newline_every=newline_every)
    c = w2b.Corpus(path, min_count)
    o = po.Corpus(path, min_count)
    assert (c.vocab_size, c.train_words, c.file_size, c.num_tokens) == (o.vocab_size, o.train_words, o.file_size, o.num_tokens)
    assert c.words() == o.words()
    assert np.array_equal(c.counts, o.counts) and np.array_equal(c.tokens, o.tokens)
    for n in (1, 2, 3, 7, 16, 61, 148):
        s, f = c.shards(n)
        want = [o.shard_start(i, n) for i in range(n)]
        assert [w[0] for w in want] == list(s) and [w[1] for w in want] == list(f), n


def test_corpus_edge_cases(tmp_path):
    import word2bits_b200 as w2b
    cases = {
        "empty.txt": b"",
        "one.txt": b"hello",                      # last token without trailing whitespace is never seen
        "nl.txt": b"\n\n\n",
        "crlf.txt": b"a b\r\nc\td  e\r\n\r\nf" + b" g" * 10,
        "long.txt": b"x" * 5000 + b" y y y\n",    # token longer than MAX_STRING is truncated
        "tie.txt": b"b a c a b c d d e\n" * 3,    # equal counts keep first-appearance order
    }
    for name, data in cases.items():
        p = tmp_path / name
        p.write_bytes(data)
        c = w2b.Corpus(str(p), 1)
        o = po.Corpus(str(p), 1)
        assert c.words() == o.words(), name
        assert np.array_equal(c.counts, o.counts) and np.array_equal(c.tokens, o.tokens), name
        assert (c.train_words, c.file_size) == (o.train_words, o.file_size), name
        for n in (1, 2, 5):
            s, f = c.shards(n)
            assert [o.shard_start(i, n) for i in range(n)] == list(zip(s.tolist(), f.tolist())), (name, n)


def test_corpus_matches_reference(tmp_path):
    """Vocabulary, counts and sizes equal what the unmodified reference's LearnVocabFromTrainFile computed on the
    same corpus (tests/golden/reference_outputs.json)."""
    import word2bits_b200 as w2b
    path = zipf_corpus(str(tmp_path / "c.txt"), 80000, 5000, seed=5)
    for mc in (1, 5):
        want = reference_outputs("host_cpu")["corpus_seed5_mc%d" % mc]
        c = w2b.Corpus(path, mc)
        assert digest(c.words()) == want["words"] and digest(c.counts) == want["counts"]
        assert (c.vocab_size, c.train_words, c.file_size) == (want["V"], want["train_words"], want["file_size"])


def test_vector_writer_matches_oracle(tmp_path):
    import word2bits_b200 as w2b
    path = os.path.join(ROOT, "tests", "golden", "golden_corpus.txt")
    c = w2b.Corpus(path, 1)
    o = po.Corpus(path, 1)
    m = po.OracleModel(o, 8, 3, 4, 2)
    vec = m.export()
    for binary in (0, 1):
        a, b = str(tmp_path / ("a%d" % binary)), str(tmp_path / ("b%d" % binary))
        c.write_vectors(a, vec, binary)
        m.write_vectors(b, binary)
        assert open(a, "rb").read() == open(b, "rb").read()
    # README.md:124-131 framing: header, "</s> " first, rows end with "\n"
    raw = open(a, "rb").read()
    assert raw.startswith(b"31 8\n</s> ") and raw.endswith(b"\n")


def test_cli_messages_and_exit_codes(tmp_path):
    def run(exe, *args):
        r = subprocess.run([exe, *args], capture_output=True, text=True)
        return r.returncode, r.stdout
    golden = os.path.join(ROOT, "tests", "golden", "golden_corpus.txt")
    ours = [run(CLI, "-train", "/nonexistent", "-output", "x"), run(CLI, "-train"),
            run(CLI, "-train", golden, "-min-count", "1"), run(CLI, "-train", golden, "-min-count", "5", "-debug", "0")]
    assert ours[0] == (1, "Starting training using file /nonexistent\nERROR: training data file not found!\n")
    assert ours[1] == (1, "Argument missing for -train\n")
    assert ours[2] == (0, "Starting training using file %s\nVocab size: 31\nWords in train file: 13533\n" % golden)
    # the reference's own binary, same four calls
    theirs = [(rc, out.replace("{golden}", golden)) for rc, out in reference_outputs("host_cpu")["cli_messages"]]
    assert ours == theirs


def test_parallel_tokenizer_equals_sequential(tmp_path, monkeypatch):
    """The corpus reader cuts the file into chunks for several threads; word order, counts, the
    token stream and every shard start must not depend on the number of chunks."""
    import word2bits_b200 as w2b
    path = zipf_corpus(str(tmp_path / "c.txt"), 300000, 8000, seed=21, newline_every=23)
    monkeypatch.setenv("W2B_TOKENIZER_MIN_CHUNK", "50000")
    res = []
    for threads in ("1", "2", "5", "16"):
        monkeypatch.setenv("W2B_TOKENIZER_THREADS", threads)
        c = w2b.Corpus(path, 3)
        s, f = c.shards(37)
        res.append((c.words(), c.counts.copy(), c.tokens.copy(), c.train_words, s.copy(), f.copy()))
    o = po.Corpus(path, 3)
    assert res[0][0] == o.words() and np.array_equal(res[0][2], o.tokens)
    for r in res[1:]:
        assert r[0] == res[0][0] and np.array_equal(r[1], res[0][1]) and np.array_equal(r[2], res[0][2])
        assert r[3] == res[0][3] and np.array_equal(r[4], res[0][4]) and np.array_equal(r[5], res[0][5])


@pytest.mark.parametrize("bits", [1, 2])
def test_packed_vector_file_round_trip(tmp_path, bits):
    """SURVEY 8(f).3: bitlevel bits per value on disk; unpack restores the exact float levels."""
    import word2bits_b200 as w2b
    path = os.path.join(ROOT, "tests", "golden", "golden_corpus.txt")
    c = w2b.Corpus(path, 1)
    o = po.Corpus(path, 1)
    m = po.OracleModel(o, 20, 3, 4, bits)
    vec = m.export()                       # quantize(u+v): on the level set
    out = str(tmp_path / "packed.bin")
    c.write_packed(out, vec, bits)
    words, back, b = w2b.read_packed(out)
    assert b == bits and words == c.words()
    assert np.array_equal(back.view(np.uint32), vec.view(np.uint32))
    full = str(tmp_path / "full.bin")
    c.write_vectors(full, vec, 1)
    ratio = os.path.getsize(full) / os.path.getsize(out)
    assert ratio > 5                       # 20 dims only: the word names dominate, still >> 1
    with pytest.raises(w2b.W2BError):
        c.write_packed(out, vec, 4)


# ---------------------------------------------------------------- host arithmetic the device path uploads
def test_host_unigram_bounds_match_oracle():
    """InitUnigramTable (:112-128) in boundary form, same libm pow(): the boundaries libw2b uploads equal the
    oracle's (which tests/test_oracle_vs_ref.py pins to the reference's full 1e8-entry table)."""
    import word2bits_b200 as w2b
    rng = np.random.default_rng(3)
    cases = [
        np.array([0, 5, 5, 5], np.int64),                                  # </s> never seen
        np.array([7, 1], np.int64),
        np.concatenate([[1000], np.sort(rng.integers(1, 10**6, 5000))[::-1]]).astype(np.int64),
        np.maximum(1, (3e8 / np.arange(1, 400_001)).astype(np.int64)),    # C2-sized Zipf vocabulary
        np.concatenate([[0], np.full(3_000_000, 1)]).astype(np.int64),    # more words than some slices are wide
    ]
    for cn in cases:
        got = w2b.host_unigram_bounds(cn)
        want = po.unigram_bounds(cn)
        assert got.dtype == np.int32 and np.array_equal(got.astype(np.int64), want), len(cn)
        assert got[0] == 0 and got[-1] == w2b._lib.TABLE_SIZE and np.all(np.diff(got.astype(np.int64)) >= 0)


def test_host_exptable_and_keep_thresholds():
    import word2bits_b200 as w2b
    assert np.array_equal(w2b.host_exptable().view(np.uint32), po.exptable().view(np.uint32))
    # `ran` (:403-404) in float32, operation by operation
    rng = np.random.default_rng(5)
    cn = np.concatenate([[0], rng.integers(1, 10**7, 2000)]).astype(np.int64)
    for train_words, sample in ((int(cn.sum()), 1e-3), (17_000_000, 1e-4), (123, 1e-3)):
        got = w2b.host_keep_thresholds(cn, train_words, sample)
        S = np.float32(sample) * np.float32(train_words)
        with np.errstate(divide="ignore", invalid="ignore"):
            c = cn.astype(np.float32)
            want = (np.sqrt(c / S, dtype=np.float32) + np.float32(1)) * S / c
        assert np.array_equal(got[1:].view(np.uint32), want[1:].astype(np.float32).view(np.uint32))


def test_host_lcg_jump_tables():
    """r_k = r*ja[k] + jc[k] is k steps of the reference's LCG (:352,:405,:428,:455); pa/pc are the 2^j-step
    constants InitNet's jump-ahead uses."""
    import word2bits_b200 as w2b
    ja, jc, pa, pc = w2b.host_lcg_tables()
    M = (1 << 64) - 1
    L = po.lib()
    for r0 in (0, 1, 11, 147, 2**63 + 12345, M):
        r = r0
        for k in range(65):
            assert (r0 * int(ja[k]) + int(jc[k])) & M == r, (r0, k)
            r = L.w2bo_lcg(r)
    r = 1
    steps = 0
    for j in range(20):  # 2^j steps by repeated single steps, j < 20
        while steps < (1 << j):
            r = L.w2bo_lcg(r)
            steps += 1
        assert (1 * int(pa[j]) + int(pc[j])) & M == r, j
    for j in range(1, 64):  # squaring rule for the rest
        assert int(pa[j]) == (int(pa[j - 1]) ** 2) & M
        assert int(pc[j]) == (int(pa[j - 1]) * int(pc[j - 1]) + int(pc[j - 1])) & M


def test_null_arguments_are_errors_not_crashes():
    import ctypes as C
    import word2bits_b200 as w2b
    from word2bits_b200._lib import lib, EINVAL
    assert lib.w2b_train_step(None, 10, None) == EINVAL and b"null" in lib.w2b_last_error()
    for fn in ("w2b_init_tables", "w2b_epoch_begin", "w2b_sync"):
        assert getattr(lib, fn)(None) == EINVAL
    assert lib.w2b_export(None, None) == EINVAL
    assert lib.w2b_create(None, C.byref(C.c_void_p())) == EINVAL
    assert lib.w2b_warp_plan_query(None, None) == EINVAL
    assert lib.w2b_corpus_shards(None, 2, None, None) == EINVAL
    assert lib.w2b_host_unigram_bounds(None, 5, None) == EINVAL
    assert lib.w2b_destroy(None) == 0  # like free(NULL)
    assert lib.w2b_read_packed_header(None, None, None, None) == EINVAL
    assert lib.w2b_read_packed(None, None, None, 0) == EINVAL
    with pytest.raises(w2b.W2BError) as e:
        w2b.Corpus(os.path.join(ROOT, "tests"), 1)  # a directory is not a training file
    assert e.value.code == 3


@pytest.mark.parametrize("nthreads", [1, 2, 3, 8, 0])
def test_streaming_slice_gather(nthreads):
    """The host half of a streaming step (w2b_train_step with host token buffers): every unfinished shard's next L
    tokens land in its slice of the staging buffer whatever the number of host threads; finished shards are skipped;
    a pending override token (cursor -1) starts the slice at 0; the last slice is clipped at the end of the stream."""
    import ctypes as C
    from word2bits_b200._lib import lib, ptr
    rng = np.random.default_rng(9)
    n, S, L = 3_000_000, 37, 70_000
    ids = rng.integers(0, 1 << 20, n).astype(np.int32)
    cursor = np.sort(rng.integers(0, n, S)).astype(np.int64)
    cursor[0] = -1
    cursor[-1] = n - 1234          # clipped at EOF
    cursor[-2] = n                 # nothing left to read
    done = np.zeros(S, np.int32)
    done[5] = done[20] = 1
    stage = np.full(S * L, -7, np.int32)
    xl = np.full(S, -99, np.int64); lim = np.full(S, -99, np.int64); eof = np.full(S, -99, np.int32)
    assert lib.w2b_host_gather_slices(ptr(ids), n, L, S, ptr(cursor), ptr(done), ptr(stage), ptr(xl), ptr(lim), ptr(eof),
                                      nthreads) == 0
    for i in range(S):
        sl = stage[i * L:(i + 1) * L]
        if done[i]:
            assert (sl == -7).all() and (xl[i], lim[i], eof[i]) == (-99, -99, -99)
            continue
        b = max(int(cursor[i]), 0)
        e = min(b + L, n)
        assert np.array_equal(sl[:e - b], ids[b:e]) and (sl[e - b:] == -7).all()
        assert (xl[i], lim[i], eof[i]) == (b - i * L, e, int(e == n))
        # the kernel reads token g at staging index g - xlate
        if e > b:
            assert stage[b - xl[i]] == ids[b]
    assert lib.w2b_host_gather_slices(None, n, L, S, ptr(cursor), ptr(done), ptr(stage), ptr(xl), ptr(lim), ptr(eof), 1) != 0


def fuzz_corpus(path, seed):
    rng = np.random.default_rng(100 + seed)
    alphabet = np.frombuffer(b"abcde" * 6 + b"  \t\n\n\r\x00\x01\xff\xc3\xa9", np.uint8)
    body = alphabet[rng.integers(0, len(alphabet), 400_000)].tobytes()
    long_words = b" " + b"x" * 4094 + b" " + b"y" * 4095 + b" " + b"z" * 4096 + b"q " + b"k" * 9000 + b"\n"
    data = body[:150_000] + long_words + body[150_000:] + (b"" if seed == 0 else b" tail" if seed == 1 else b"\r")
    with open(path, "wb") as f:
        f.write(data)
    return path


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_tokenizer_fuzz_against_oracle(tmp_path, monkeypatch, seed):
    """Random bytes from a hostile alphabet (CR and NUL inside words, control characters, high bytes, runs of
    newlines, words longer than MAX_STRING, no trailing whitespace), cut into many chunks: the fast path (words
    hashed straight from the mapping) and the byte-by-byte slow path must reproduce the reference's reader for
    every thread count — words, counts, token stream and shard starts."""
    import word2bits_b200 as w2b
    p = fuzz_corpus(str(tmp_path / "fuzz.txt"), seed)
    o = po.Corpus(str(p), 2)
    monkeypatch.setenv("W2B_TOKENIZER_MIN_CHUNK", "20000")
    for threads in ("1", "3", "16"):
        monkeypatch.setenv("W2B_TOKENIZER_THREADS", threads)
        c = w2b.Corpus(str(p), 2)
        assert c.words() == o.words(), threads
        assert np.array_equal(c.counts, o.counts) and np.array_equal(c.tokens, o.tokens), threads
        assert (c.train_words, c.file_size, c.num_tokens) == (o.train_words, o.file_size, o.num_tokens)
        for n in (1, 7, 64):
            s, f = c.shards(n)
            assert [o.shard_start(i, n) for i in range(n)] == list(zip(s.tolist(), f.tolist())), (threads, n)
    want = reference_outputs("host_cpu")["tokenizer_fuzz%d" % seed]  # the unmodified reference's reader
    assert digest(c.words()) == want["words"] and digest(c.counts) == want["counts"]
    assert c.train_words == want["train_words"]


def test_text_writer_parallel_and_cached_formatting(tmp_path, monkeypatch):
    """The text writer formats blocks of rows on several threads through a per-thread value cache: the bytes
    must not depend on the thread count and must equal "%lf " of every value (checked with Python's own
    correctly-rounded formatting for finite floats; NaN / inf / -0.0 only for thread-independence)."""
    import word2bits_b200 as w2b
    path = zipf_corpus(str(tmp_path / "c.txt"), 30000, 3000, seed=4)
    c = w2b.Corpus(path, 1)
    V, D = c.vocab_size, 37
    rng = np.random.default_rng(8)
    vec = (rng.standard_normal((V, D)) * np.exp(rng.uniform(-20, 20, (V, D)))).astype(np.float32)
    vec[rng.random((V, D)) < 0.5] = np.float32(1 / 3)             # cache hits, like trained 1-bit vectors
    vec[5, :6] = [np.nan, -np.nan, np.inf, -np.inf, -0.0, np.float32(3.4e38)]
    outs = []
    for threads in ("1", "4", "32"):
        monkeypatch.setenv("W2B_WRITER_THREADS", threads)
        out = str(tmp_path / ("v%s.txt" % threads))
        c.write_vectors(out, vec, 0)
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1] == outs[2]
    lines = outs[0].split(b"\n")
    assert lines[0] == b"%d %d" % (V, D) and lines[-1] == b"" and len(lines) == V + 2
    words = c.words()
    for a in (0, 1, 2, 77, V - 1):
        want = words[a].encode("latin1") + b" " + b"".join(b"%f " % float(x) for x in vec[a])
        assert lines[1 + a] == want, a


def _vector_file(path, words, D, seed=0):
    rng = np.random.default_rng(seed)
    with open(path, "wb") as f:
        f.write(b"%d %d\n" % (len(words), D))
        for w in words:
            f.write(w.encode() + b" " + rng.standard_normal(D).astype(np.float32).tobytes() + b"\n")


EMPTY_REPORT_QUESTIONS = ": capital-common-countries\nathens greece baghdad iraq\nzzz yyy xxx www\n: family\nboy girl zzz sister\n"


def test_evaluator_host_side_errors_and_empty_report(tmp_path):
    """w2b_compute_accuracy (SURVEY 8(f).2) before any GPU work: bad arguments and unreadable / hostile vector files
    are error codes, never crashes or exceptions across the C ABI; a question stream in which no question can be
    answered (every line has an out-of-vocabulary word) needs no device and prints what src/compute-accuracy.c prints."""
    import ctypes as C
    import word2bits_b200 as w2b
    from word2bits_b200._lib import lib, EINVAL
    acc = w2b._lib.Accuracy()
    buf = C.create_string_buffer(4096)
    qf = tmp_path / "q.txt"
    qf.write_text(EMPTY_REPORT_QUESTIONS)
    call = lambda vf: lib.w2b_compute_accuracy(vf, 0, 0, str(qf).encode(), 0, C.byref(acc), buf, len(buf))
    assert call(None) == EINVAL
    assert call(str(tmp_path / "missing.bin").encode()) == 3 and b"not found" in lib.w2b_last_error()
    for name, content in (("text.bin", b"hello world\n"), ("neg.bin", b"-5 10\n"), ("zero.bin", b"10 0\n"),
                          ("huge.bin", b"999999999999 999999\n"), ("big.bin", b"2000000000 1000000\n"),
                          ("short.bin", b"3 8\nathens " + b"\0" * 32 + b"\ngreece " + b"\0" * 7)):
        p = tmp_path / name
        p.write_bytes(content)
        assert call(str(p).encode()) == 3, name  # W2B_EIO
    vf = str(tmp_path / "vec.bin")
    _vector_file(vf, ["athens", "greece", "baghdad", "boy", "girl", "sister"], 8)
    got, counters = w2b.compute_accuracy(vf, str(qf))
    assert counters["questions_total"] == 3 and counters["questions_seen"] == 0 and counters["gpu_ms"] == 0.0
    assert got == reference_outputs("host_cpu")["evaluator_empty_report"]  # src/compute-accuracy.c's report


def test_corpus_above_the_reduce_vocab_threshold_is_refused(tmp_path, monkeypatch):
    """Above 0.7 * 30 M distinct words the reference prunes its vocabulary in the middle of the scan (ReduceVocab,
    :245-263, called from :292) — an order-dependent cut the one-pass reader does not reproduce, so such a corpus
    is an error, not a silently different vocabulary.  (The threshold is lowered through the test hook.)"""
    import word2bits_b200 as w2b
    p = tmp_path / "c.txt"
    p.write_text(" ".join("w%d" % (i % 12) for i in range(200)) + "\n")  # 12 words + </s> = 13 vocabulary entries
    monkeypatch.setenv("W2B_TOKENIZER_MAX_DISTINCT", "13")
    c = w2b.Corpus(str(p), 1)
    assert c.vocab_size == 13
    c.close()
    monkeypatch.setenv("W2B_TOKENIZER_MAX_DISTINCT", "12")
    with pytest.raises(w2b.W2BError, match="ReduceVocab") as e:
        w2b.Corpus(str(p), 1)
    assert e.value.code == 1


def test_default_geometry_is_the_measured_one():
    """The launch geometries of the production kernel the benchmark runs: one 32-thread CTA per shard, `warps_per_sm`
    of them resident per SM.  Pinned so that a planner change cannot move the benchmarked configuration silently."""
    import word2bits_b200 as w2b
    want = {  # (D, window, negative, bitlevel): (slots, queue_entries, warps_per_sm, smem_bytes)
        (800, 10, 24, 1): (4, 128, 12, 17440),   # BASELINE configs[1]
        (400, 10, 12, 2): (5, 128, 16, 12656),   # configs[2]
        (400, 10, 24, 0): (5, 128, 16, 12656),   # configs[3]
        (200, 8, 24, 1): (7, 128, 20, 10272),    # configs[0] shape
    }
    for (D, W, neg, b), geo in want.items():
        p = w2b.warp_plan(size=D, window=W, negative=neg, bitlevel=b, vocab_size=400001)
        assert p["warp"] == 1
        assert (p["slots"], p["queue_entries"], p["warps_per_sm"], p["smem_bytes"]) == geo, (D, p)


def test_wide_register_kernels_fit_1024_threads():
    """The register kernel runs one thread per column group, up to 1024 per CTA (D = 4096).  The instantiations the
    dispatch launches at that width (strict mode always; fast mode when the speed-tuned ones cannot take a row's
    threads) must hold at most 64 registers per thread: 1024 x 64 is the register file of an SM."""
    import shutil
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, check=True).stdout
    regs = {m.group(1): int(m.group(2)) for m in re.finditer(r"Function (\S+):\s+REG:(\d+)", out)}
    wide = {k: r for k, r in regs.items() if "train_shards_wide_kernel" in k or "apply_position_wide_kernel" in k}
    assert len(wide) == 12, sorted(wide)  # {train, apply} x {VEC 4, VEC 1} x {fast, fast -reg, strict}
    assert all(r <= 64 for r in wide.values()), wide
