"""TEST INFRASTRUCTURE — ctypes front end of tests/emu/libw2bemu.so: the production kernel's source compiled for
the host and run on fibers (tests/emu/emu_main.cpp).  Used by tests/test_warp_emulation.py to check the kernel
functionally when no GPU is at hand."""
import ctypes as C
import os
import subprocess

import numpy as np

import word2bits_b200 as w2b
from word2bits_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
_emu = None


class EmuRun(C.Structure):
    _fields_ = [("V", C.c_int64), ("D", C.c_int64), ("window", C.c_int32), ("negative", C.c_int32), ("bitlevel", C.c_int32),
                ("sample", C.c_float), ("alpha0", C.c_float), ("iter", C.c_int64), ("train_words", C.c_int64),
                ("num_shards", C.c_int32),
                ("opt", C.c_int32), ("lpr", C.c_int32), ("xw", C.c_int32), ("nu", C.c_int32), ("nv", C.c_int32),
                ("G", C.c_int32), ("threads", C.c_int32), ("serial", C.c_int32),
                ("u", C.c_void_p), ("v", C.c_void_p), ("table", C.c_void_p), ("keep", C.c_void_p), ("exptab", C.c_void_p),
                ("tokens", C.c_void_p), ("n_tokens", C.c_int64), ("shard_start", C.c_void_p), ("shard_first", C.c_void_p),
                ("alpha", C.c_void_p), ("wca", C.c_void_p), ("word_budget", C.c_int64), ("max_iters", C.c_int64),
                ("seed", C.c_uint64), ("async_mode", C.c_int32), ("train", C.c_int32),
                ("loss", C.c_void_p), ("words", C.c_void_p), ("n_pos", C.c_void_p), ("n_ctx", C.c_void_p),
                ("n_tgt", C.c_void_p), ("done", C.c_void_p),
                ("trace", C.c_void_p), ("trace_cap", C.c_int64), ("trace_n", C.c_void_p), ("only_shard", C.c_int32),
                ("fault", C.c_int32), ("reg", C.c_float)]


def lib():
    global _emu
    if _emu is None:
        subprocess.check_call(["make", "-s", "-C", HERE], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        _emu = C.CDLL(os.path.join(HERE, "libw2bemu.so"))
        _emu.emu_last_error.restype = C.c_char_p
        _emu.emu_run_warp.argtypes = [C.POINTER(EmuRun)]
    return _emu


class EmuError(RuntimeError):
    pass


def train_epoch_warp(corpus, table, u, v, *, size, window, negative, bitlevel, shards, serial=0, alpha=0.05,
                     sample=1e-3, iters=1, async_mode=1, seed=1, state=None, trace_shard=None, trace_cap=0, max_iters=-1,
                     slots=0, fault=0, reg=0.0, trace_train=False):
    """One pass of every shard (one 32-thread CTA after another) through the emulated warp-per-shard kernel
    (csrc/w2b_warp.cuh).  u, v are updated in place.  Returns a dict of per-shard statistics; `state` carries
    (alpha, word_count_actual) across epochs.  With trace_cap the kernel records every shard's draws in its own
    region (the layout of w2b_train_step_traced): out["traces"][i] is shard i's, out["trace"] that of `trace_shard`.
    Tracing runs draws only (trace_shard alone), unless trace_train: then every shard trains as well."""
    plan = w2b.warp_plan(size=size, window=window, negative=negative, bitlevel=bitlevel, vocab_size=corpus.vocab_size,
                         slots=slots, reg=reg)
    if not plan["warp"]:
        raise EmuError("the warp kernel does not apply to this shape")
    start, first = corpus.shards(shards)
    keep = w2b.host_keep_thresholds(corpus.counts, corpus.train_words, sample)
    exptab = w2b.host_exptable()
    tokens = np.ascontiguousarray(corpus.tokens, np.int32)
    a = np.array([alpha if state is None else state[0]], np.float32)
    wca = np.array([0 if state is None else state[1]], np.uint64)
    out = dict(loss=np.zeros(shards), words=np.zeros(shards, np.int64), n_pos=np.zeros(shards, np.int64),
               n_ctx=np.zeros(shards, np.int64), n_tgt=np.zeros(shards, np.int64), done=np.zeros(shards, np.int32))
    trace = (_lib.TraceRec * max(trace_cap * shards, 1))()
    trace_n = np.zeros(shards, np.uint64)
    p = _lib.ptr
    pitch = (size + 3) // 4 * 4  # the device layout: rows padded to whole float4s, padding zero
    u_in, v_in = u, v
    if pitch != size:
        u = np.zeros((u_in.shape[0], pitch), np.float32); u[:, :size] = u_in
        v = np.zeros((v_in.shape[0], pitch), np.float32); v[:, :size] = v_in
    r = EmuRun(V=corpus.vocab_size, D=size, window=window, negative=negative, bitlevel=bitlevel, sample=sample,
               alpha0=alpha, iter=iters, train_words=corpus.train_words, num_shards=shards,
               opt=0, lpr=32 if plan["sentence_in_smem"] else 0, xw=0, nu=plan["queue_entries"], nv=plan["slots"], G=0, threads=32,
               serial=serial,
               u=p(u), v=p(v), table=p(table), keep=p(keep), exptab=p(exptab), tokens=p(tokens), n_tokens=len(tokens),
               shard_start=p(start), shard_first=p(first), alpha=p(a), wca=p(wca), word_budget=0, max_iters=max_iters,
               seed=seed, async_mode=async_mode, train=0 if trace_cap and not trace_train else 1,
               loss=p(out["loss"]), words=p(out["words"]), n_pos=p(out["n_pos"]), n_ctx=p(out["n_ctx"]),
               n_tgt=p(out["n_tgt"]), done=p(out["done"]),
               trace=C.cast(trace, C.c_void_p) if trace_cap else None, trace_cap=trace_cap,
               trace_n=p(trace_n) if trace_cap else None, only_shard=-1 if trace_shard is None else trace_shard,
               fault=fault, reg=reg)
    rc = lib().emu_run_warp(C.byref(r))
    if rc:
        raise EmuError(lib().emu_last_error().decode())
    if pitch != size:
        assert not v[:, size:].any()  # the padding of v never moves
        u_in[:] = u[:, :size]
        v_in[:] = v[:, :size]
    out["alpha"], out["wca"] = float(a[0]), int(wca[0])
    out["plan"] = plan
    if trace_cap:
        out["traces"] = [[(t.center, t.b, t.cw, list(t.targets[: t.ntargets]), t.alpha)
                          for t in trace[i * trace_cap: i * trace_cap + min(int(trace_n[i]), trace_cap)]]
                         for i in range(shards)]
        out["trace_n"] = trace_n.astype(np.int64)
        if trace_shard is not None:
            out["trace"] = out["traces"][trace_shard]
    return out
