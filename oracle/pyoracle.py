"""TEST INFRASTRUCTURE — ctypes bindings for the CPU oracle (liboracle.so) and for the
unmodified reference compiled as a library (oracle/_ref/libw2b_ref*.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this module.  The product package word2bits_b200 never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
TABLE_SIZE = 100_000_000

_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")


def build(ref: bool = True) -> None:
    """Compile liboracle.so and, when /root/reference is present, oracle/_ref/."""
    subprocess.check_call(["make", "-s", "-C", HERE, "oracle"])
    if ref and os.path.exists("/root/reference/src/word2bits.cpp"):
        subprocess.check_call(["make", "-s", "-C", HERE, "ref"], stderr=subprocess.DEVNULL)


# ------------------------------------------------------------------------------ oracle
class TraceRec(C.Structure):
    _fields_ = [("center", C.c_int32), ("b", C.c_int32), ("cw", C.c_int32), ("ntargets", C.c_int32),
                ("targets", C.c_int32 * 64), ("alpha", C.c_float)]


class Trace(C.Structure):
    _fields_ = [("rec", C.POINTER(TraceRec)), ("cap", C.c_int64), ("n", C.c_int64)]


class Model(C.Structure):
    _fields_ = [("V", C.c_int64), ("D", C.c_int64),
                ("window", C.c_int), ("negative", C.c_int), ("bitlevel", C.c_int),
                ("sample", C.c_float), ("reg", C.c_float), ("starting_alpha", C.c_float),
                ("iter", C.c_int64), ("train_words", C.c_int64),
                ("num_shards", C.c_int),
                ("u", C.c_void_p), ("v", C.c_void_p), ("table", C.c_void_p), ("cn", C.c_void_p),
                ("alpha", C.c_float), ("word_count_actual", C.c_int64)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(HERE, "liboracle.so")
        if not os.path.exists(path):
            build(ref=False)
        L = C.CDLL(path)
        L.w2bo_quantize.restype = C.c_float
        L.w2bo_quantize.argtypes = [C.c_float, C.c_int]
        L.w2bo_quantize_n.argtypes = [_f32p, _f32p, C.c_int64, C.c_int]
        L.w2bo_sigmoid.restype = C.c_float
        L.w2bo_sigmoid.argtypes = [C.c_float]
        L.w2bo_lcg.restype = C.c_uint64
        L.w2bo_lcg.argtypes = [C.c_uint64]
        L.w2bo_exptable.argtypes = [_f32p]
        L.w2bo_init_net.argtypes = [C.c_int64, C.c_int64, _f32p, _f32p]
        L.w2bo_unigram_table.argtypes = [_i64p, C.c_int64, _i32p]
        L.w2bo_unigram_bounds.argtypes = [_i64p, C.c_int64, _i64p]
        L.w2bo_corpus_load.restype = C.c_void_p
        L.w2bo_corpus_load.argtypes = [C.c_char_p, C.c_int]
        L.w2bo_corpus_free.argtypes = [C.c_void_p]
        for name in ("vocab_size", "train_words", "file_size", "num_tokens"):
            fn = getattr(L, "w2bo_" + name)
            fn.restype = C.c_int64
            fn.argtypes = [C.c_void_p]
        L.w2bo_word.restype = C.c_char_p
        L.w2bo_word.argtypes = [C.c_void_p, C.c_int64]
        L.w2bo_counts.restype = C.POINTER(C.c_int64)
        L.w2bo_counts.argtypes = [C.c_void_p]
        L.w2bo_tokens.restype = C.POINTER(C.c_int32)
        L.w2bo_tokens.argtypes = [C.c_void_p]
        L.w2bo_shard_start.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int32)]
        L.w2bo_train_shard.restype = C.c_double
        L.w2bo_train_shard.argtypes = [C.POINTER(Model), C.c_void_p, C.c_int, C.c_int64, C.POINTER(Trace)]
        L.w2bo_train_epoch_threads.restype = C.c_double
        L.w2bo_train_epoch_threads.argtypes = [C.POINTER(Model), C.c_void_p]
        L.w2bo_apply_position.argtypes = [C.POINTER(Model), _f32p, _i32p, C.c_int, _i32p, C.c_int, _f32p,
                                          C.POINTER(C.c_double)]
        L.w2bo_export.argtypes = [C.POINTER(Model), _f32p]
        L.w2bo_write_vectors.restype = C.c_int
        L.w2bo_write_vectors.argtypes = [C.POINTER(Model), C.c_void_p, C.c_char_p, C.c_int]
        L.w2bo_analogy_normalize.argtypes = [_f32p, C.c_int64, C.c_int64, C.c_int, C.c_int]
        L.w2bo_analogy.restype = C.c_int
        L.w2bo_analogy.argtypes = [C.c_char_p, C.c_int, C.c_int64, C.c_char_p, C.c_int, C.c_int, C.c_char_p,
                                   C.c_int64, _i32p, C.c_int64, C.POINTER(C.c_int64)]
        _lib = L
    return _lib


def quantize(x, b):
    x = np.asarray(x, dtype=np.float32)
    flat = np.ascontiguousarray(x.ravel())
    out = np.empty_like(flat)
    lib().w2bo_quantize_n(flat, out, flat.size, int(b))
    return out.reshape(x.shape)


AN_FUSED, AN_LANE_NORM = 1, 2  # negative controls of the analogy evaluator (w2b_oracle.h)


def analogy_normalize(M, bits, flags=0):
    """compute-accuracy.c :106-110 on a copy of M (words x D): quantize, then divide by the row's length."""
    M = np.array(M, np.float32, order="C", copy=True)
    lib().w2bo_analogy_normalize(M.reshape(-1), M.shape[0], M.shape[1], int(bits), int(flags))
    return M


def analogy(vectors_file, questions_file, bitlevel=0, threshold=0, flags=0, threads=None):
    """src/compute-accuracy.c on the CPU: (report text, int32 array of the chosen word per question in file order,
    -1 where the question is skipped or no word scores above 0)."""
    threads = threads or min(32, os.cpu_count() or 1)
    buf = C.create_string_buffer(1 << 22)
    ans = np.empty(os.path.getsize(questions_file) // 4 + 1, np.int32)  # a question takes at least 4 bytes
    n = C.c_int64()
    rc = lib().w2bo_analogy(vectors_file.encode(), int(bitlevel), int(threshold), questions_file.encode(),
                            int(flags), int(threads), buf, len(buf), ans, len(ans), C.byref(n))
    if rc:
        raise OSError("w2bo_analogy failed (%d) on %s / %s" % (rc, vectors_file, questions_file))
    return buf.value.decode("latin1"), ans[: n.value].copy()


def exptable():
    t = np.empty(1000, np.float32)
    lib().w2bo_exptable(t)
    return t


def init_net(V, D):
    u = np.empty(V * D, np.float32)
    v = np.empty(V * D, np.float32)
    lib().w2bo_init_net(V, D, u, v)
    return u.reshape(V, D), v.reshape(V, D)


def unigram_table(cn):
    cn = np.ascontiguousarray(cn, np.int64)
    t = np.empty(TABLE_SIZE, np.int32)
    lib().w2bo_unigram_table(cn, len(cn), t)
    return t


def unigram_bounds(cn):
    cn = np.ascontiguousarray(cn, np.int64)
    s = np.empty(len(cn) + 1, np.int64)
    lib().w2bo_unigram_bounds(cn, len(cn), s)
    return s


class Corpus:
    def __init__(self, path, min_count=5):
        self.L = lib()
        self.h = self.L.w2bo_corpus_load(path.encode(), min_count)
        if not self.h:
            raise FileNotFoundError(path)
        self.path = path
        self.vocab_size = self.L.w2bo_vocab_size(self.h)
        self.train_words = self.L.w2bo_train_words(self.h)
        self.file_size = self.L.w2bo_file_size(self.h)
        self.num_tokens = self.L.w2bo_num_tokens(self.h)
        self.counts = np.ctypeslib.as_array(self.L.w2bo_counts(self.h), (self.vocab_size,)).copy()
        self.tokens = (np.ctypeslib.as_array(self.L.w2bo_tokens(self.h), (self.num_tokens,)).copy()
                       if self.num_tokens else np.zeros(0, np.int32))

    def words(self):
        return [self.L.w2bo_word(self.h, i).decode("latin1") for i in range(self.vocab_size)]

    def shard_start(self, sid, n):
        s, f = C.c_int64(), C.c_int32()
        self.L.w2bo_shard_start(self.h, sid, n, C.byref(s), C.byref(f))
        return s.value, f.value

    def __del__(self):
        try:
            self.L.w2bo_corpus_free(self.h)
        except Exception:
            pass


class OracleModel:
    """u, v, table and the shared scalars of one training run on the oracle."""

    def __init__(self, corpus, size, window, negative, bitlevel, shards=1, iters=1, alpha=0.05,
                 sample=1e-3, reg=0.0, table=None):
        self.corpus = corpus
        V = corpus.vocab_size
        self.u, self.v = init_net(V, size)
        self.table = table if table is not None else unigram_table(corpus.counts)
        self.cn = np.ascontiguousarray(corpus.counts, np.int64)
        self.m = Model(V=V, D=size, window=window, negative=negative, bitlevel=bitlevel,
                       sample=sample, reg=reg, starting_alpha=alpha, iter=iters,
                       train_words=corpus.train_words, num_shards=shards,
                       u=self.u.ctypes.data, v=self.v.ctypes.data, table=self.table.ctypes.data,
                       cn=self.cn.ctypes.data, alpha=alpha, word_count_actual=0)

    def train_shard(self, sid, max_positions=-1, trace_cap=0):
        tr = None
        recs = None
        if trace_cap:
            recs = (TraceRec * trace_cap)()
            tr = Trace(rec=recs, cap=trace_cap, n=0)
        loss = lib().w2bo_train_shard(C.byref(self.m), self.corpus.h, sid, max_positions,
                                      C.byref(tr) if tr is not None else None)
        if tr is None:
            return loss
        out = []
        for i in range(tr.n):
            r = recs[i]
            out.append((r.center, r.b, r.cw, list(r.targets[: r.ntargets]), r.alpha))
        return loss, out

    def train_epoch_threads(self):
        return lib().w2bo_train_epoch_threads(C.byref(self.m), self.corpus.h)

    def apply_position(self, ctx, targets):
        ctx = np.ascontiguousarray(ctx, np.int32)
        targets = np.ascontiguousarray(targets, np.int32)
        f = np.zeros(max(len(targets), 1), np.float32)
        loss = C.c_double()
        lib().w2bo_apply_position(C.byref(self.m), exptable(), ctx, len(ctx), targets, len(targets), f,
                                  C.byref(loss))
        return f[: len(targets)], loss.value

    def export(self):
        out = np.empty(self.m.V * self.m.D, np.float32)
        lib().w2bo_export(C.byref(self.m), out)
        return out.reshape(self.m.V, self.m.D)

    def write_vectors(self, path, binary):
        return lib().w2bo_write_vectors(C.byref(self.m), self.corpus.h, path.encode(), int(binary))

    @property
    def alpha(self):
        return self.m.alpha

    @property
    def word_count_actual(self):
        return self.m.word_count_actual


# --------------------------------------------------------------------------- reference
def ref_available(flavour="strict"):
    return os.path.exists(os.path.join(REF_DIR, _ref_name(flavour)))


def _ref_name(flavour):
    return {"strict": "libw2b_ref_strict.so", "o3": "libw2b_ref.so", "native": "libw2b_ref_native.so"}[flavour]


class Ref:
    """The unmodified reference as a library.  One instance per flavour per process
    (the reference keeps its state in file-scope globals)."""

    _cache = {}

    def __new__(cls, flavour="strict"):
        if flavour in cls._cache:
            return cls._cache[flavour]
        self = super().__new__(cls)
        L = C.CDLL(os.path.join(REF_DIR, _ref_name(flavour)))
        L.ref_configure.argtypes = [C.c_char_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong,
                                    C.c_int, C.c_float, C.c_float, C.c_float]
        for n in ("vocab_size", "train_words", "file_size", "word_count_actual"):
            getattr(L, "ref_" + n).restype = C.c_longlong
        L.ref_set_word_count_actual.argtypes = [C.c_longlong]
        L.ref_vocab_word.restype = C.c_char_p
        L.ref_vocab_word.argtypes = [C.c_longlong]
        L.ref_vocab_cn.restype = C.c_longlong
        L.ref_vocab_cn.argtypes = [C.c_longlong]
        L.ref_u.restype = C.POINTER(C.c_float)
        L.ref_v.restype = C.POINTER(C.c_float)
        L.ref_table.restype = C.POINTER(C.c_int)
        L.ref_exptable.restype = C.POINTER(C.c_float)
        L.ref_get_alpha.restype = C.c_float
        L.ref_set_alpha.argtypes = [C.c_float]
        L.ref_quantize.restype = C.c_float
        L.ref_quantize.argtypes = [C.c_float, C.c_int]
        L.ref_sigmoid.restype = C.c_float
        L.ref_sigmoid.argtypes = [C.c_float]
        L.ref_thread_loss.restype = C.c_double
        L.ref_thread_loss.argtypes = [C.c_int]
        L.ref_train_thread.argtypes = [C.c_longlong]
        L.ref_train_epoch.restype = C.c_double
        self.L = L
        cls._cache[flavour] = self
        return self

    def configure(self, train, size, window, negative, bitlevel, threads=1, iters=1, min_count=5,
                  alpha=0.05, sample=1e-3, reg=0.0):
        self.size = size
        self.L.ref_configure(train.encode(), size, window, negative, bitlevel, threads, iters, min_count,
                             alpha, sample, reg)

    def learn_vocab(self):
        self.L.ref_learn_vocab()
        self.V = self.L.ref_vocab_size()
        return self.V

    def words(self):
        return [self.L.ref_vocab_word(i).decode("latin1") for i in range(self.V)]

    def counts(self):
        return np.array([self.L.ref_vocab_cn(i) for i in range(self.V)], np.int64)

    def init_net(self):
        self.L.ref_init_net()

    def init_unigram(self):
        self.L.ref_init_unigram()

    def u(self):
        return np.ctypeslib.as_array(self.L.ref_u(), (self.V, self.size))

    def v(self):
        return np.ctypeslib.as_array(self.L.ref_v(), (self.V, self.size))

    def table(self):
        return np.ctypeslib.as_array(self.L.ref_table(), (TABLE_SIZE,))

    def exptable(self):
        return np.ctypeslib.as_array(self.L.ref_exptable(), (1000,)).copy()

    def quantize(self, x, b):
        return np.float32(self.L.ref_quantize(float(np.float32(x)), b))

    def train_thread(self, tid):
        self.L.ref_train_thread(tid)
        return self.L.ref_thread_loss(tid)

    def train_epoch(self):
        return self.L.ref_train_epoch()

    @property
    def alpha(self):
        return self.L.ref_get_alpha()

    @property
    def train_words(self):
        return self.L.ref_train_words()

    @property
    def file_size(self):
        return self.L.ref_file_size()

    @property
    def word_count_actual(self):
        return self.L.ref_word_count_actual()
