"""ctypes binding of libw2b.so (C ABI in include/w2b.h).  No torch types cross this
boundary; numpy arrays are passed as plain pointers.  There is no fallback: if the
shared library is missing this module raises at import time."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libw2b.so")

OK, EINVAL, ECUDA, EIO, ESTATE, ENCCL, ENOMEM = range(7)
VECTORS_BINARY, VECTORS_TEXT, VECTORS_PACKED = range(3)
TABLE_SIZE = 100_000_000
MODE_FAST, MODE_STRICT = 0, 1


class W2BError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libw2b error %d: %s" % (code, msg))
        self.code = code


class Config(C.Structure):
    _fields_ = [("vocab_size", C.c_int64), ("layer1_size", C.c_int64),
                ("window", C.c_int32), ("negative", C.c_int32), ("bitlevel", C.c_int32),
                ("alpha", C.c_float), ("sample", C.c_float), ("reg", C.c_float),
                ("iter", C.c_int64),
                ("num_shards", C.c_int32), ("shard_begin", C.c_int32), ("shard_end", C.c_int32),
                ("device", C.c_int32), ("mode", C.c_int32), ("group", C.c_int32), ("plain_store", C.c_int32),
                ("kernel", C.c_int32), ("slots", C.c_int32), ("prefetch", C.c_int32), ("sync_mode", C.c_int32)]


class StepStats(C.Structure):
    _fields_ = [("loss", C.c_double), ("words", C.c_int64), ("positions", C.c_int64),
                ("context_rows", C.c_int64), ("target_rows", C.c_int64), ("shards_done", C.c_int64),
                ("alpha", C.c_float), ("word_count_actual", C.c_int64), ("kernel_ms", C.c_float),
                ("launches", C.c_int32), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Accuracy(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("questions_total", "questions_seen", "correct", "semantic_correct",
                                         "semantic_seen", "syntactic_correct", "syntactic_seen", "vocab", "size")] + \
               [("gpu_ms", C.c_float), ("candidates", C.c_int64), ("rescored", C.c_int64)]


class TopkStats(C.Structure):
    _fields_ = [("gpu_ms", C.c_float), ("queries", C.c_int64), ("skipped", C.c_int64), ("chunks", C.c_int64),
                ("candidates", C.c_int64), ("rescored", C.c_int64), ("simt", C.c_int32), ("packed", C.c_int32)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


MAX_TOPK = 1024


class WarpPlan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("warp", "slots", "queue_entries", "warps_per_sm", "sentence_in_smem", "reserved")] + \
               [("smem_bytes", C.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class KernelInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("warp", "nj", "minb", "bm", "reg", "vec", "threads", "wide", "group",
                                         "apply_wide", "apply_bm", "apply_group")]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class TraceRec(C.Structure):
    _fields_ = [("center", C.c_int32), ("b", C.c_int32), ("cw", C.c_int32), ("ntargets", C.c_int32),
                ("targets", C.c_int32 * 64), ("alpha", C.c_float)]


EXPORTS = [
    "w2b_corpus_load", "w2b_corpus_free", "w2b_corpus_vocab_size", "w2b_corpus_train_words",
    "w2b_corpus_file_size", "w2b_corpus_word", "w2b_corpus_counts", "w2b_corpus_num_tokens",
    "w2b_corpus_tokens", "w2b_corpus_shards", "w2b_write_vectors", "w2b_last_error", "w2b_device_count",
    "w2b_suggest_shards", "w2b_create", "w2b_destroy", "w2b_set_vocab_counts", "w2b_set_corpus",
    "w2b_init_tables", "w2b_epoch_begin", "w2b_train_step", "w2b_train_epoch", "w2b_trace",
    "w2b_train_step_traced", "w2b_strict_prefix", "w2b_apply_position", "w2b_get_state", "w2b_set_state", "w2b_download_raw",
    "w2b_upload_raw", "w2b_download_table", "w2b_download_exptable", "w2b_export", "w2b_quantize",
    "w2b_device_ptrs", "w2b_nccl_unique_id", "w2b_nccl_init", "w2b_sync", "w2b_sync_timed", "w2b_table_checksum", "w2b_scale_tables",
    "w2b_write_packed", "w2b_read_packed_header", "w2b_read_packed", "w2b_checkpoint_save", "w2b_checkpoint_load", "w2b_compute_accuracy",
    "w2b_analogy_answers", "w2b_eval_filter_scores",
    "w2b_compute_accuracy_packed", "w2b_analogy_answers_packed", "w2b_eval_packed_scores",
    "w2b_analogy_topk", "w2b_nearest",
    "w2b_ctx_compute_accuracy", "w2b_ctx_analogy_answers", "w2b_ctx_analogy_topk", "w2b_ctx_nearest",
    "w2b_host_unigram_bounds", "w2b_host_exptable", "w2b_host_keep_thresholds", "w2b_host_lcg_tables", "w2b_warp_plan_query", "w2b_host_gather_slices",
    "w2b_kernel_query", "w2b_host_parse_floats", "w2b_vector_file_info", "w2b_vector_names", "w2b_read_text_vectors",
]

if not os.path.exists(LIB_PATH):
    raise ImportError("libw2b.so is not built (run __graft_entry__.build() or make -C word2bits_b200/csrc); "
                      "word2bits_b200 has no CPU fallback")

lib = C.CDLL(LIB_PATH)
_vp, _i64, _i32, _f = C.c_void_p, C.c_int64, C.c_int32, C.c_float
_P = C.POINTER

lib.w2b_last_error.restype = C.c_char_p
lib.w2b_corpus_load.argtypes = [C.c_char_p, C.c_int, _P(_vp)]
lib.w2b_corpus_free.argtypes = [_vp]
lib.w2b_corpus_free.restype = None
for _n in ("vocab_size", "train_words", "file_size", "num_tokens"):
    _fn = getattr(lib, "w2b_corpus_" + _n)
    _fn.restype = _i64
    _fn.argtypes = [_vp]
lib.w2b_corpus_word.restype = C.c_char_p
lib.w2b_corpus_word.argtypes = [_vp, _i64]
lib.w2b_corpus_counts.restype = _P(_i64)
lib.w2b_corpus_counts.argtypes = [_vp]
lib.w2b_corpus_tokens.restype = _P(_i32)
lib.w2b_corpus_tokens.argtypes = [_vp]
lib.w2b_corpus_shards.argtypes = [_vp, C.c_int, _vp, _vp]
lib.w2b_write_vectors.argtypes = [C.c_char_p, _vp, _vp, _i64, _i64, C.c_int]
lib.w2b_write_packed.argtypes = [C.c_char_p, _vp, _vp, _i64, _i64, C.c_int]
lib.w2b_read_packed_header.argtypes = [C.c_char_p, _P(_i64), _P(_i64), _P(C.c_int)]
lib.w2b_read_packed.argtypes = [C.c_char_p, _vp, _vp, C.c_int]
lib.w2b_host_parse_floats.argtypes = [C.c_char_p, _i64, _vp, _i64, _P(_i64)]
lib.w2b_vector_file_info.argtypes = [C.c_char_p, _i64, _P(C.c_int), _P(_i64), _P(_i64), _P(C.c_int)]
lib.w2b_vector_names.argtypes = [C.c_char_p, _i64, _vp, C.c_int, _P(_i64)]
lib.w2b_read_text_vectors.argtypes = [C.c_char_p, C.c_int, _vp, _vp, C.c_int]
lib.w2b_checkpoint_save.argtypes = [_vp, C.c_char_p, _i64]
lib.w2b_checkpoint_load.argtypes = [_vp, C.c_char_p, _P(_i64)]
lib.w2b_compute_accuracy.argtypes = [C.c_char_p, C.c_int, _i64, C.c_char_p, C.c_int, _P(Accuracy), C.c_char_p, _i64]
lib.w2b_analogy_answers.argtypes = [C.c_char_p, C.c_int, _i64, C.c_char_p, C.c_int, _vp, _i64, _P(_i64)]
lib.w2b_eval_filter_scores.argtypes = [_vp, _i64, _vp, _i64, _i64, C.c_int, _vp, _vp]
lib.w2b_compute_accuracy_packed.argtypes = [C.c_char_p, _i64, C.c_char_p, C.c_int, _P(Accuracy), C.c_char_p, _i64]
lib.w2b_analogy_answers_packed.argtypes = [C.c_char_p, _i64, C.c_char_p, C.c_int, _vp, _i64, _P(_i64)]
lib.w2b_eval_packed_scores.argtypes = [_vp, _i64, _i64, C.c_int, _vp, _i64, _vp, _i64, C.c_int, _vp, _vp, _vp]
lib.w2b_analogy_topk.argtypes = [C.c_char_p, C.c_int, _i64, C.c_char_p, C.c_int, C.c_int, _vp, _vp, _i64, _P(_i64),
                                 _P(TopkStats)]
lib.w2b_nearest.argtypes = [C.c_char_p, C.c_int, _i64, C.c_char_p, C.c_int, C.c_int, _vp, _vp, _i64, _P(_i64),
                            _P(TopkStats)]
lib.w2b_ctx_compute_accuracy.argtypes = [_vp, _vp, C.c_int, _i64, C.c_char_p, _P(Accuracy), C.c_char_p, _i64]
lib.w2b_ctx_analogy_answers.argtypes = [_vp, _vp, C.c_int, _i64, C.c_char_p, _vp, _i64, _P(_i64)]
lib.w2b_ctx_analogy_topk.argtypes = [_vp, _vp, C.c_int, _i64, C.c_char_p, C.c_int, _vp, _vp, _i64, _P(_i64), _P(TopkStats)]
lib.w2b_ctx_nearest.argtypes = [_vp, _vp, C.c_int, _i64, C.c_char_p, C.c_int, _vp, _vp, _i64, _P(_i64), _P(TopkStats)]
lib.w2b_host_unigram_bounds.argtypes = [_vp, _i64, _vp]
lib.w2b_host_exptable.argtypes = [_vp]
lib.w2b_host_keep_thresholds.argtypes = [_vp, _i64, _i64, _f, _vp]
lib.w2b_host_lcg_tables.argtypes = [_vp, _vp, _vp, _vp]
lib.w2b_warp_plan_query.argtypes = [_P(Config), _P(WarpPlan)]
lib.w2b_host_gather_slices.argtypes = [_vp, _i64, _i64, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int]
lib.w2b_device_count.argtypes = [_P(C.c_int)]
lib.w2b_suggest_shards.argtypes = [_P(Config), _P(C.c_int)]
lib.w2b_create.argtypes = [_P(Config), _P(_vp)]
lib.w2b_destroy.argtypes = [_vp]
lib.w2b_kernel_query.argtypes = [_vp, _P(KernelInfo)]
lib.w2b_set_vocab_counts.argtypes = [_vp, _vp, _i64, _i64]
lib.w2b_set_corpus.argtypes = [_vp, _vp, _i64, _vp, _vp, C.c_int]
lib.w2b_init_tables.argtypes = [_vp]
lib.w2b_epoch_begin.argtypes = [_vp]
lib.w2b_train_step.argtypes = [_vp, _i64, _P(StepStats)]
lib.w2b_train_epoch.argtypes = [_vp, _P(C.c_double), _P(StepStats)]
lib.w2b_trace.argtypes = [_vp, C.c_int, _i64, _vp, _i64, _P(_i64)]
lib.w2b_train_step_traced.argtypes = [_vp, _i64, _P(StepStats), _vp, _i64, _vp]
lib.w2b_strict_prefix.argtypes = [_vp, C.c_int, _i64, _P(C.c_double)]
lib.w2b_apply_position.argtypes = [_vp, _vp, C.c_int, _vp, C.c_int, _vp]
lib.w2b_get_state.argtypes = [_vp, _P(_f), _P(_i64)]
lib.w2b_set_state.argtypes = [_vp, _f, _i64]
lib.w2b_download_raw.argtypes = [_vp, _vp, _vp]
lib.w2b_upload_raw.argtypes = [_vp, _vp, _vp]
lib.w2b_download_table.argtypes = [_vp, _vp]
lib.w2b_download_exptable.argtypes = [_vp, _vp]
lib.w2b_export.argtypes = [_vp, _vp]
lib.w2b_quantize.argtypes = [_vp, _vp, _vp, _i64, C.c_int]
lib.w2b_device_ptrs.argtypes = [_vp, _P(_vp), _P(_vp), _P(_i64)]
lib.w2b_nccl_unique_id.argtypes = [_vp]
lib.w2b_nccl_init.argtypes = [_vp, _vp, C.c_int, C.c_int]
lib.w2b_sync.argtypes = [_vp]
lib.w2b_sync_timed.argtypes = [_vp, _P(_f)]
lib.w2b_table_checksum.argtypes = [_vp, _P(C.c_uint64), _P(C.c_uint64)]
lib.w2b_scale_tables.argtypes = [_vp, _f]


def check(rc):
    if rc != OK:
        raise W2BError(rc, lib.w2b_last_error().decode("utf-8", "replace"))


def ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None
