"""word2bits_b200 — H100-native Word2Bits training path.

Python mirror of the C ABI (include/w2b.h); the compute lives in libw2b.so (hand-written
sm_90a CUDA) and is driven the same way the C++ CLI (csrc/main.cpp) drives it.
Mirrors the reference's surface: the constructor arguments are its command-line flags
(src/word2bits.cpp:596-611, same names and defaults)."""
import ctypes as C
import os

import numpy as np

from . import _lib
from ._lib import MODE_FAST, MODE_STRICT, TABLE_SIZE, W2BError, check, lib, ptr

__all__ = ["Corpus", "Trainer", "W2BError", "MODE_FAST", "MODE_STRICT", "device_count", "read_packed", "nccl_unique_id",
           "compute_accuracy", "analogy_answers", "eval_filter_scores", "compute_accuracy_packed", "analogy_answers_packed",
           "eval_packed_scores", "host_unigram_bounds", "host_exptable", "host_keep_thresholds", "host_lcg_tables", "warp_plan",
           "analogy_topk", "nearest", "host_parse_floats", "vector_file_info", "read_text_vectors"]


def device_count():
    n = C.c_int(0)
    rc = lib.w2b_device_count(C.byref(n))
    return n.value if rc == 0 else 0


# -- host-side arithmetic of the path (no GPU needed): exactly what the device path uploads
def host_unigram_bounds(counts):
    """InitUnigramTable (:112-128) in boundary form: start[i] = first table slot of word i, start[V] = 1e8."""
    cn = np.ascontiguousarray(counts, np.int64)
    start = np.empty(len(cn) + 1, np.int32)
    check(lib.w2b_host_unigram_bounds(ptr(cn), len(cn), ptr(start)))
    return start


def host_exptable():
    t = np.empty(1000, np.float32)
    check(lib.w2b_host_exptable(ptr(t)))
    return t


def host_keep_thresholds(counts, train_words, sample):
    """Sub-sampling thresholds `ran` (:403-404), float32."""
    cn = np.ascontiguousarray(counts, np.int64)
    out = np.empty(len(cn), np.float32)
    check(lib.w2b_host_keep_thresholds(ptr(cn), len(cn), int(train_words), float(sample), ptr(out)))
    return out


def host_lcg_tables():
    """(ja, jc, pa, pc): k-step (k = 0..64) and 2^j-step (j = 0..63) jump constants of the LCG."""
    ja, jc = np.empty(65, np.uint64), np.empty(65, np.uint64)
    pa, pc = np.empty(64, np.uint64), np.empty(64, np.uint64)
    check(lib.w2b_host_lcg_tables(ptr(ja), ptr(jc), ptr(pa), ptr(pc)))
    return ja, jc, pa, pc


def warp_plan(*, size, window, negative, bitlevel=1, reg=0.0, vocab_size=1000, mode=MODE_FAST, kernel=0, slots=0):
    """Geometry of the production (warp-per-shard) kernel for a configuration (pure host arithmetic)."""
    cfg = _lib.Config(vocab_size=vocab_size, layer1_size=size, window=window, negative=negative, bitlevel=bitlevel,
                      alpha=0.05, sample=1e-3, reg=reg, iter=1, num_shards=1, shard_begin=0, shard_end=0, device=0,
                      mode=mode, group=0, plain_store=0, kernel=kernel, slots=slots, prefetch=0, sync_mode=0)
    out = _lib.WarpPlan()
    check(lib.w2b_warp_plan_query(C.byref(cfg), C.byref(out)))
    return out.as_dict()


class Corpus:
    """Tokenised training file + vocabulary (LearnVocabFromTrainFile, :265-301)."""

    def __init__(self, train, min_count=5):
        h = C.c_void_p()
        check(lib.w2b_corpus_load(train.encode(), int(min_count), C.byref(h)))
        self.h = h
        self.vocab_size = lib.w2b_corpus_vocab_size(h)
        self.train_words = lib.w2b_corpus_train_words(h)
        self.file_size = lib.w2b_corpus_file_size(h)
        self.num_tokens = lib.w2b_corpus_num_tokens(h)

    @property
    def counts(self):
        return np.ctypeslib.as_array(lib.w2b_corpus_counts(self.h), (self.vocab_size,))

    @property
    def tokens(self):
        if self.num_tokens == 0:
            return np.zeros(0, np.int32)
        return np.ctypeslib.as_array(lib.w2b_corpus_tokens(self.h), (self.num_tokens,))

    def words(self):
        return [lib.w2b_corpus_word(self.h, i).decode("latin1") for i in range(self.vocab_size)]

    def shards(self, n):
        start = np.empty(n, np.int64)
        first = np.empty(n, np.int32)
        check(lib.w2b_corpus_shards(self.h, n, ptr(start), ptr(first)))
        return start, first

    def write_vectors(self, path, vectors, binary):
        vectors = np.ascontiguousarray(vectors, np.float32)
        V, D = vectors.shape
        check(lib.w2b_write_vectors(path.encode(), self.h, ptr(vectors), V, D, int(binary)))

    def write_packed(self, path, vectors, bitlevel):
        vectors = np.ascontiguousarray(vectors, np.float32)
        V, D = vectors.shape
        check(lib.w2b_write_packed(path.encode(), self.h, ptr(vectors), V, D, int(bitlevel)))

    def close(self):
        if self.h:
            lib.w2b_corpus_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Trainer:
    """One device context = the reference's globals u, v, table, expTable, alpha, ... (:45-61).

    size/window/negative/bitlevel/alpha/sample/reg/iter/threads are the reference's flags;
    `threads` is the total number of corpus shards (None = enough to fill the GPU)."""

    def __init__(self, corpus=None, *, size=100, window=5, negative=5, bitlevel=1, alpha=0.05, sample=1e-3,
                 reg=0.0, iter=5, threads=None, device=0, mode=MODE_FAST, shard_range=None, group=0,
                 plain_store=0, resident=True, vocab_size=None, init=True, kernel=0, slots=0, prefetch=0, sync_mode=0):
        V = corpus.vocab_size if corpus is not None else vocab_size
        cfg = _lib.Config(vocab_size=V, layer1_size=size, window=window, negative=negative, bitlevel=bitlevel,
                          alpha=alpha, sample=sample, reg=reg, iter=iter, num_shards=threads or 1,
                          shard_begin=0, shard_end=0, device=device, mode=mode, group=group,
                          plain_store=plain_store, kernel=kernel, slots=slots, prefetch=prefetch, sync_mode=sync_mode)
        if threads is None:
            n = C.c_int(0)
            check(lib.w2b_suggest_shards(C.byref(cfg), C.byref(n)))
            threads = n.value
            cfg.num_shards = threads
        if shard_range is not None:
            cfg.shard_begin, cfg.shard_end = shard_range
        self.cfg = cfg
        self.V, self.D, self.threads = V, size, threads
        self.corpus = corpus
        h = C.c_void_p()
        check(lib.w2b_create(C.byref(cfg), C.byref(h)))
        self.h = h
        if corpus is not None:
            self.set_vocab_counts(corpus.counts, corpus.train_words)
            start, first = corpus.shards(threads)
            self.set_corpus(corpus.tokens, start, first, resident)
        if init:
            self.init_tables()

    # -- setup
    def set_vocab_counts(self, counts, train_words):
        counts = np.ascontiguousarray(counts, np.int64)
        check(lib.w2b_set_vocab_counts(self.h, ptr(counts), len(counts), int(train_words)))

    def set_corpus(self, tokens, shard_start, shard_first, resident=True):
        self._tokens = np.ascontiguousarray(tokens, np.int32)  # kept alive for streaming mode
        s = np.ascontiguousarray(shard_start, np.int64)
        f = np.ascontiguousarray(shard_first, np.int32)
        check(lib.w2b_set_corpus(self.h, ptr(self._tokens), len(self._tokens), ptr(s), ptr(f), int(resident)))

    def init_tables(self):
        check(lib.w2b_init_tables(self.h))

    # -- training
    def epoch_begin(self):
        check(lib.w2b_epoch_begin(self.h))

    def train_step(self, words_per_shard=0):
        st = _lib.StepStats()
        check(lib.w2b_train_step(self.h, int(words_per_shard), C.byref(st)))
        return st.as_dict()

    def train_epoch(self):
        st = _lib.StepStats()
        loss = C.c_double()
        check(lib.w2b_train_epoch(self.h, C.byref(loss), C.byref(st)))
        return loss.value, st.as_dict()

    def kernel_info(self):
        """The instantiations this context launches: {"warp": 1, "nj", "minb", "bm", "reg"} for the warp kernel; for the
        register kernel vec, threads, bm, reg, and wide / group of the training launch and apply_* of the
        single-position hook (w2b.h w2b_kernel_info)."""
        out = _lib.KernelInfo()
        check(lib.w2b_kernel_query(self.h, C.byref(out)))
        return out.as_dict()

    # -- parity hooks
    def trace(self, shard, max_iterations=-1, cap=100000):
        recs = (_lib.TraceRec * cap)()
        n = C.c_int64()
        check(lib.w2b_trace(self.h, shard, max_iterations, C.cast(recs, C.c_void_p), cap, C.byref(n)))
        return [(r.center, r.b, r.cw, list(r.targets[: r.ntargets]), r.alpha) for r in recs[: n.value]]

    def train_step_traced(self, words_per_shard, cap):
        """train_step, and every local shard's draw records of the step (at most `cap` each) in the format of trace();
        a record's alpha is the learning rate its position trained with.  Returns (stats, [records of shard i],
        [records shard i made, capped or not])."""
        st = _lib.StepStats()
        nloc = (self.cfg.shard_end or self.threads) - self.cfg.shard_begin
        recs = (_lib.TraceRec * max(cap * nloc, 1))()
        n = np.zeros(nloc, np.int64)
        check(lib.w2b_train_step_traced(self.h, int(words_per_shard), C.byref(st), C.cast(recs, C.c_void_p), int(cap),
                                        ptr(n)))
        out = [[(r.center, r.b, r.cw, list(r.targets[: r.ntargets]), r.alpha)
                for r in recs[i * cap: i * cap + min(int(n[i]), cap)]] for i in range(nloc)]
        return st.as_dict(), out, n.tolist()

    def strict_prefix(self, shard, max_iterations):
        loss = C.c_double()
        check(lib.w2b_strict_prefix(self.h, shard, max_iterations, C.byref(loss)))
        return loss.value

    def apply_position(self, ctx, targets):
        ctx = np.ascontiguousarray(ctx, np.int32)
        targets = np.ascontiguousarray(targets, np.int32)
        f = np.zeros(max(len(targets), 1), np.float32)
        check(lib.w2b_apply_position(self.h, ptr(ctx), len(ctx), ptr(targets), len(targets), ptr(f)))
        return f[: len(targets)]

    def get_state(self):
        a, w = C.c_float(), C.c_int64()
        check(lib.w2b_get_state(self.h, C.byref(a), C.byref(w)))
        return a.value, w.value

    def set_state(self, alpha, wca):
        check(lib.w2b_set_state(self.h, alpha, wca))

    def download_raw(self):
        u = np.empty((self.V, self.D), np.float32)
        v = np.empty((self.V, self.D), np.float32)
        check(lib.w2b_download_raw(self.h, ptr(u), ptr(v)))
        return u, v

    def upload_raw(self, u=None, v=None):
        u = None if u is None else np.ascontiguousarray(u, np.float32)
        v = None if v is None else np.ascontiguousarray(v, np.float32)
        check(lib.w2b_upload_raw(self.h, ptr(u), ptr(v)))

    def download_table(self):
        t = np.empty(TABLE_SIZE, np.int32)
        check(lib.w2b_download_table(self.h, ptr(t)))
        return t

    def download_exptable(self):
        t = np.empty(1000, np.float32)
        check(lib.w2b_download_exptable(self.h, ptr(t)))
        return t

    def export(self):
        out = np.empty((self.V, self.D), np.float32)
        check(lib.w2b_export(self.h, ptr(out)))
        return out

    def quantize(self, x, bitlevel):
        x = np.ascontiguousarray(x, np.float32)
        out = np.empty_like(x)
        check(lib.w2b_quantize(self.h, ptr(x), ptr(out), x.size, bitlevel))
        return out

    def checkpoint_save(self, path, epochs_done=0):
        check(lib.w2b_checkpoint_save(self.h, path.encode(), int(epochs_done)))

    def checkpoint_load(self, path):
        n = C.c_int64()
        check(lib.w2b_checkpoint_load(self.h, path.encode(), C.byref(n)))
        return n.value

    # -- evaluation of the tables as they stand (quantize(u + v), what export() returns), no file in between
    def _names(self, names):
        """The row names as a C array (kept alive with the returned object)."""
        if names is None:
            if self.corpus is None:
                raise ValueError("a Trainer built without a corpus needs the row names")
            names = self.corpus.words()
        enc = [n if isinstance(n, bytes) else n.encode("latin1") for n in names]
        if len(enc) != self.V:
            raise ValueError("%d names for %d rows" % (len(enc), self.V))
        return (C.c_char_p * len(enc))(*enc)

    def compute_accuracy(self, questions_file, names=None, bitlevel=0, threshold=0):
        """compute_accuracy on this context's tables: (report text, dict of counters), exactly what the module-level
        compute_accuracy returns on the file export() would be written to (-binary 1), names = the row names."""
        words = self._names(names)
        acc = _lib.Accuracy()
        buf = C.create_string_buffer(1 << 20)
        check(lib.w2b_ctx_compute_accuracy(self.h, words, int(bitlevel), int(threshold), questions_file.encode(),
                                           C.byref(acc), buf, len(buf)))
        return buf.value.decode("latin1"), {k: getattr(acc, k) for k, _ in acc._fields_}

    def analogy_answers(self, questions_file, names=None, bitlevel=0, threshold=0):
        """analogy_answers on this context's tables (int32 numpy array, one entry per question)."""
        words = self._names(names)
        ans = np.empty(os.path.getsize(questions_file) // 4 + 1, np.int32)
        n = C.c_int64()
        check(lib.w2b_ctx_analogy_answers(self.h, words, int(bitlevel), int(threshold), questions_file.encode(),
                                          ptr(ans), len(ans), C.byref(n)))
        return ans[: n.value].copy()

    def _topk(self, fn, input_file, k, names, bitlevel, threshold):
        words = self._names(names)
        args = (self.h, words, int(bitlevel), int(threshold), input_file.encode() if input_file else None, int(k))
        n = C.c_int64()
        check(fn(*args, None, None, 0, C.byref(n), None))
        ids = np.empty((max(n.value, 1), max(int(k), 1)), np.int32)
        scores = np.empty(ids.shape, np.float32)
        st = _lib.TopkStats()
        check(fn(*args, ptr(ids), ptr(scores), max(n.value, 1), C.byref(n), C.byref(st)))
        return ids[: n.value].copy(), scores[: n.value].copy(), st.as_dict()

    def analogy_topk(self, questions_file, k, names=None, bitlevel=0, threshold=0):
        """analogy_topk on this context's tables: (ids int32 [n, k], scores float32 [n, k], stats)."""
        return self._topk(lib.w2b_ctx_analogy_topk, questions_file, k, names, bitlevel, threshold)

    def nearest(self, query_words_or_file, k, names=None, bitlevel=0, threshold=0):
        """nearest on this context's tables: query_words_or_file is a list of words or the path of a file of
        whitespace-separated words.  Returns (ids int32 [n, k], scores float32 [n, k], stats)."""
        if isinstance(query_words_or_file, (list, tuple)):
            import tempfile
            with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
                f.write("\n".join(query_words_or_file) + "\n")
            try:
                return self._topk(lib.w2b_ctx_nearest, f.name, k, names, bitlevel, threshold)
            finally:
                os.unlink(f.name)
        return self._topk(lib.w2b_ctx_nearest, query_words_or_file, k, names, bitlevel, threshold)

    # -- multi-GPU
    def device_ptrs(self):
        u, v, n = C.c_void_p(), C.c_void_p(), C.c_int64()
        check(lib.w2b_device_ptrs(self.h, C.byref(u), C.byref(v), C.byref(n)))
        return u.value, v.value, n.value

    def nccl_init(self, uid, rank, nranks):
        buf = (C.c_char * 128).from_buffer_copy(uid)
        check(lib.w2b_nccl_init(self.h, C.cast(buf, C.c_void_p), rank, nranks))

    def sync(self):
        """Replica average + exact global word counter; returns the device time of the exchange in ms."""
        ms = C.c_float(0)
        check(lib.w2b_sync_timed(self.h, C.byref(ms)))
        return ms.value

    def table_checksum(self):
        """(sum of u's bit patterns, sum of v's) mod 2^64: equal on every rank right after sync()."""
        a, b = C.c_uint64(0), C.c_uint64(0)
        check(lib.w2b_table_checksum(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def close(self):
        if getattr(self, "h", None):
            lib.w2b_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def nccl_unique_id():
    buf = (C.c_char * 128)()
    check(lib.w2b_nccl_unique_id(C.cast(buf, C.c_void_p)))
    return bytes(buf)


def read_packed(path, max_word=64):
    """(words, vectors, bitlevel) of a packed vector file written by Corpus.write_packed / -binary 2."""
    V, D, b = C.c_int64(), C.c_int64(), C.c_int()
    check(lib.w2b_read_packed_header(path.encode(), C.byref(V), C.byref(D), C.byref(b)))
    vec = np.empty((V.value, D.value), np.float32)
    names = np.zeros((V.value, max_word), np.uint8)
    check(lib.w2b_read_packed(path.encode(), ptr(vec), ptr(names), max_word))
    words = [bytes(r[: list(r).index(0)] if 0 in r else r).decode("latin1") for r in names]
    return words, vec, b.value


def host_parse_floats(text):
    """The float32 values of the white-space separated tokens of `text` (bytes or str), each exactly what glibc strtof
    returns for it, converted on the host by the routine the GPU text reader runs.  A token outside the grammar
    [+-]?(d+[.d*]|.d+)([eE][+-]?d+)? (or nan, inf, infinity, signed or not, in any case) raises W2BError."""
    if isinstance(text, str):
        text = text.encode("latin1")
    out = np.empty(max(len(text) // 2 + 1, 1), np.float32)  # a token and its separator take at least 2 bytes
    n = C.c_int64()
    check(lib.w2b_host_parse_floats(text, len(text), ptr(out), len(out), C.byref(n)))
    return out[: n.value].copy()


def vector_file_info(path, threshold=0):
    """(kind, V, D, bits) of a vector file: kind "binary" (word2vec binary), "text" (-binary 0) or "packed"
    (-binary 2), V its words (at most threshold when threshold > 0), D their size, bits a packed file's bit level."""
    kind, V, D, bits = C.c_int(), C.c_int64(), C.c_int64(), C.c_int()
    check(lib.w2b_vector_file_info(path.encode(), int(threshold), C.byref(kind), C.byref(V), C.byref(D), C.byref(bits)))
    return ("binary", "text", "packed")[kind.value], V.value, D.value, bits.value


def read_text_vectors(path, device=0, max_word=64):
    """(words, vectors) of a text vector file (-binary 0, Corpus.write_vectors(binary=0)), parsed on the GPU: vectors
    is V x D float32, each value what strtof returns for its token; words as written (cut to max_word - 1 bytes)."""
    kind, V, D, _ = vector_file_info(path)
    if kind != "text":
        raise W2BError(_lib.EIO, "%s is not a text vector file" % path)
    vec = np.empty((V, D), np.float32)
    names = np.zeros((max(V, 1), max_word), np.uint8)
    check(lib.w2b_read_text_vectors(path.encode(), int(device), ptr(vec), ptr(names), max_word))
    words = [bytes(r[: list(r).index(0)] if 0 in r else r).decode("latin1") for r in names[:V]]
    return words, vec


def compute_accuracy(vectors_file, questions_file, bitlevel=0, threshold=0, device=0):
    """GPU port of the reference's compute_accuracy: returns (report text, dict of counters).  A word2vec-binary or
    text (-binary 0, parsed on the GPU) vector file."""
    acc = _lib.Accuracy()
    buf = C.create_string_buffer(1 << 20)
    check(lib.w2b_compute_accuracy(vectors_file.encode(), int(bitlevel), int(threshold), questions_file.encode(),
                                   int(device), C.byref(acc), buf, len(buf)))
    return buf.value.decode("latin1"), {k: getattr(acc, k) for k, _ in acc._fields_}


def analogy_answers(vectors_file, questions_file, bitlevel=0, threshold=0, device=0):
    """Per question of questions_file, in file order: the index of the word compute_accuracy chooses, or -1 (the
    question is skipped, or no word scores above 0).  int32 numpy array."""
    ans = np.empty(os.path.getsize(questions_file) // 4 + 1, np.int32)  # a question takes at least 4 bytes
    n = C.c_int64()
    check(lib.w2b_analogy_answers(vectors_file.encode(), int(bitlevel), int(threshold), questions_file.encode(),
                                  int(device), ptr(ans), len(ans), C.byref(n)))
    return ans[: n.value].copy()


def eval_filter_scores(Q, M, device=0):
    """Test hook: (approx, eps) of the evaluator's tensor-core filter for float32 rows Q (nq x D) and M (words x D):
    approx[q, c] its TF32 score, eps[q] the error bound it assumes for question q (rows of M of length <= 1)."""
    Q = np.ascontiguousarray(Q, np.float32)
    M = np.ascontiguousarray(M, np.float32)
    approx = np.empty((Q.shape[0], M.shape[0]), np.float32)
    eps = np.empty(Q.shape[0], np.float32)
    check(lib.w2b_eval_filter_scores(ptr(Q), Q.shape[0], ptr(M), M.shape[0], Q.shape[1], int(device), ptr(approx), ptr(eps)))
    return approx, eps


def compute_accuracy_packed(packed_file, questions_file, threshold=0, device=0):
    """compute_accuracy on a packed vector file (Corpus.write_packed / -binary 2), scored in the bit domain: returns
    what compute_accuracy returns on the unpacked file with bitlevel = the file's bit level."""
    acc = _lib.Accuracy()
    buf = C.create_string_buffer(1 << 20)
    check(lib.w2b_compute_accuracy_packed(packed_file.encode(), int(threshold), questions_file.encode(), int(device),
                                          C.byref(acc), buf, len(buf)))
    return buf.value.decode("latin1"), {k: getattr(acc, k) for k, _ in acc._fields_}


def analogy_answers_packed(packed_file, questions_file, threshold=0, device=0):
    """analogy_answers on a packed vector file."""
    ans = np.empty(os.path.getsize(questions_file) // 4 + 1, np.int32)
    n = C.c_int64()
    check(lib.w2b_analogy_answers_packed(packed_file.encode(), int(threshold), questions_file.encode(), int(device),
                                         ptr(ans), len(ans), C.byref(n)))
    return ans[: n.value].copy()


def eval_packed_scores(rows, D, bitlevel, qid, q3, device=0):
    """Test hook of the packed evaluator: rows (V x ceil(D*bitlevel/8) uint8, packed as in the file), qid (W word
    ids), q3 (nq x 3 indices into qid) -> (gram, approx, eps): gram[w, c] the exact integer dot product of rows qid[w]
    and c in level units, approx[q, c] the filter's score, eps[q] its bound on |approx - the reference's score|."""
    rows = np.ascontiguousarray(rows, np.uint8)
    qid = np.ascontiguousarray(qid, np.int32)
    q3 = np.ascontiguousarray(q3, np.int32).reshape(-1, 3)
    V, W, nq = rows.shape[0], len(qid), len(q3)
    if rows.shape[1] != (D * bitlevel + 7) // 8:
        raise ValueError("rows must be ceil(D * bitlevel / 8) bytes wide")
    gram = np.empty((W, V), np.int32)
    approx = np.empty((nq, V), np.float32)
    eps = np.empty(nq, np.float32)
    check(lib.w2b_eval_packed_scores(ptr(rows), V, int(D), int(bitlevel), ptr(qid), W, ptr(q3), nq, int(device),
                                     ptr(gram), ptr(approx), ptr(eps)))
    return gram, approx, eps


def _topk(fn, vectors_file, input_file, k, bitlevel, threshold, device):
    args = (vectors_file.encode(), int(bitlevel), int(threshold), input_file.encode() if input_file else None, int(k),
            int(device))
    n = C.c_int64()
    check(fn(*args, None, None, 0, C.byref(n), None))  # counts the queries: the rows are sized exactly
    ids = np.empty((max(n.value, 1), max(int(k), 1)), np.int32)
    scores = np.empty(ids.shape, np.float32)
    st = _lib.TopkStats()
    check(fn(*args, ptr(ids), ptr(scores), max(n.value, 1), C.byref(n), C.byref(st)))
    return ids[: n.value].copy(), scores[: n.value].copy(), st.as_dict()


def analogy_topk(vectors_file, questions_file, k, bitlevel=0, threshold=0, device=0):
    """The reference's top-N list at N = k for every question of questions_file, in file order: (ids int32 [n, k],
    scores float32 [n, k], stats).  Row i holds the k words of largest fp32 score > 0 (not the question's own words),
    best first, the smaller index first on equal scores; -1 (score 0) pads a short list and fills the row of a question
    with a word not in the vocabulary.  Word2vec-binary, text or packed vector file (bitlevel then 0 or the file's)."""
    return _topk(lib.w2b_analogy_topk, vectors_file, questions_file, k, bitlevel, threshold, device)


def nearest(vectors_file, words, k, bitlevel=0, threshold=0, device=0):
    """Nearest neighbours: the list of analogy_topk for the question (w, w, w) of every word w of `words` (a list of
    words, or the path of a file of whitespace-separated words): the k words whose vectors have the largest cosine
    with w's, w itself excluded.  Returns (ids int32 [n, k], scores float32 [n, k], stats)."""
    if isinstance(words, (list, tuple)):
        import tempfile
        with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
            f.write("\n".join(words) + "\n")
        try:
            return _topk(lib.w2b_nearest, vectors_file, f.name, k, bitlevel, threshold, device)
        finally:
            os.unlink(f.name)
    return _topk(lib.w2b_nearest, vectors_file, words, k, bitlevel, threshold, device)
