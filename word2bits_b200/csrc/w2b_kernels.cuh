// Device code of the Word2Bits training path for sm_90a.
//
// One CTA walks one corpus shard exactly like one reference thread does
// (TrainModelThread, src/word2bits.cpp:363-516): sentence builder + sub-sampling,
// window draw, negative draws from the unigram table, then the arithmetic of one
// position.  Thread t of the CTA owns embedding columns [t*VEC, t*VEC+VEC) of every
// row the position touches, so the context average, the error accumulator and both
// scatter updates are private per thread; only the dim-D dot product is reduced across
// the CTA (warp shuffles, then one shared-memory hop).
//
// HBM layout: u, v = fp32 [V][D] row-major (rows 16-byte aligned when D%4==0);
// table = int32[1e8]; keep_thr = fp32[V]; tokens = int32 stream.  Rows are read with
// ld.global.cg (L2-coherent: other CTAs update them concurrently) and updated with
// red.global.add.v4.f32 (no lost updates) or, in strict mode, load/add/store.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "w2b.h"
#include "w2b_quant.cuh"

namespace w2b {

constexpr unsigned long long kLcgA = 25214903917ULL;
constexpr unsigned long long kLcgC = 11ULL;
constexpr int kMaxS = W2B_MAX_SENTENCE;
constexpr int kExpN = 1000;

// k-step jump constants of the LCG, k = 0..64, and 2^j-step constants, j = 0..63.
__constant__ unsigned long long c_JA[65];
__constant__ unsigned long long c_JC[65];
__constant__ unsigned long long c_PA[64];
__constant__ unsigned long long c_PC[64];

struct ShardState {
  unsigned long long rng;  // LCG state at the next sentence build (:368 seed = shard id)
  long long cursor;        // next token index (global index space)
  long long limit;         // tokens [.., limit) are readable in this launch
  long long xlate;         // device index = global index - xlate (slice staging)
  long long word_count;    // :399
  long long last_word_count;
  long long ovr_idx;       // index whose token is replaced by ovr_tok (mid-word seek, :377)
  int ovr_tok;
  int done;
  int limit_is_eof;
  int pad;
  double loss;             // thread_losses[id], :511
  unsigned long long n_iter, n_pos, n_ctx, n_tgt;
};

struct PosDesc {
  int center, b, cw, nt;
  float alpha;
  int ctx[2 * W2B_MAX_WINDOW];
  int tg[W2B_MAX_NEGATIVE + 1];
};

struct TrainParams {
  float *u, *v;
  const int *table;
  const float *keep_thr;
  const float *exptab;
  const int *tokens;
  ShardState *shards;
  float *alpha;                 // shared learning rate (:53), racy like the reference
  unsigned long long *wca;      // word_count_actual (:51)
  long long D, V;
  long long pitch;              // floats between two rows of u / v: D, rounded up to a multiple of 4 (16-byte rows)
  int ncol;                     // register kernel: threads that own columns = ceil(D / VEC)
  int window, negative, bitlevel;
  float sample, reg, starting_alpha, alpha_denom;  // alpha_denom = (float)(iter*train_words+1)
  long long shard_word_limit;   // train_words / num_shards (:414)
  long long word_budget;        // <=0: run shards to their end
  long long max_iters;          // test hook: stop after this many window draws (<0: none)
  int shard_base;               // first local shard handled by blockIdx 0
  int train;                    // 0: draws only (trace)
  int serial;                   // warp kernel: 1 = position p+1 is fetched after every update of p completed
  int wca_scale;                // multi-GPU: local words stand for wca_scale x as many globally
  int *sen;                     // warp kernel: global sentence buffers (kMaxS ints per local shard + 1) when they do not fit shared memory
  w2b_trace_rec *trace;         // parity hooks (nullptr in production): draw records, at most trace_cap per region,
  long long trace_cap;          // and their count (which may exceed the cap)
  unsigned long long *trace_n;
  int trace_per_shard;          // 1: local shard i's region is trace[i * trace_cap ..), its count trace_n[i]
                                // (w2b_train_step_traced); 0: every CTA uses region 0 (w2b_trace: one CTA)
};

// ------------------------------------------------------------------------- scalar bits
__device__ __forceinline__ unsigned long long lcg(unsigned long long r) { return r * kLcgA + kLcgC; }
__device__ __forceinline__ unsigned long long lcg_jump(unsigned long long r, int k) {
  return r * c_JA[k] + c_JC[k];
}
__device__ inline unsigned long long lcg_jump_big(unsigned long long r, unsigned long long k) {
  for (int j = 0; k; ++j, k >>= 1)
    if (k & 1) r = r * c_PA[j] + c_PC[j];
  return r;
}

// r mod w for 1 <= w <= 64 with 32-bit arithmetic (the window draw, :429).
__device__ __forceinline__ int mod_small(unsigned long long r, unsigned w) {
  const unsigned hi = (unsigned)(r >> 32), lo = (unsigned)r;
  const unsigned two32 = (0xffffffffu % w + 1u) % w;  // 2^32 mod w
  return (int)(((hi % w) * two32 + lo % w) % w);
}

// :67-71 — reporting only.
__device__ __forceinline__ float sigmoid_report(float x) {
  if (x > 6.f) return 1.f;
  if (x < -6.f) return 1e-9f;
  return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
}

// gradient scalar, :473-475.  (EXP_TABLE_SIZE / MAX_EXP / 2) is integer arithmetic = 83.
__device__ __forceinline__ float grad_scalar(float f, int label, float alpha, const float *exptab) {
  if (f > 6.f) return __fmul_rn((float)(label - 1), alpha);
  if (f < -6.f) return __fmul_rn((float)label, alpha);
  int idx = __float2int_rz(__fmul_rn(__fadd_rn(f, 6.f), 83.f));
  return __fmul_rn(__fsub_rn((float)label, exptab[idx]), alpha);
}

// ---------------------------------------------------------------- vector row accessors
template <int VEC>
struct Vec;
template <>
struct Vec<4> {
  float a[4];
  __device__ __forceinline__ void load(const float *p) {
    float4 t = __ldcg(reinterpret_cast<const float4 *>(p));
    a[0] = t.x; a[1] = t.y; a[2] = t.z; a[3] = t.w;
  }
  __device__ __forceinline__ void store(float *p) const {
    __stcg(reinterpret_cast<float4 *>(p), make_float4(a[0], a[1], a[2], a[3]));
  }
  __device__ __forceinline__ void red_add(float *p) const {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a[0]), "f"(a[1]),
                 "f"(a[2]), "f"(a[3])
                 : "memory");
  }
};
template <>
struct Vec<1> {
  float a[1];
  __device__ __forceinline__ void load(const float *p) { a[0] = __ldcg(p); }
  __device__ __forceinline__ void store(float *p) const { __stcg(p, a[0]); }
  __device__ __forceinline__ void red_add(float *p) const {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(a[0]) : "memory");
  }
};

// -------------------------------------------------------------------- sampler (warp 0)
// Sentence builder + sub-sampling, :394-413, 32 tokens per round.  Lane i tests token i
// with the state i+1 draws ahead (every in-vocab non-</s> word read consumes one draw).
// status: 0 = sentence complete (possibly empty), 1 = EOF (:397), 2 = slice exhausted
// before the sentence ended (streaming: the caller retries with the next slice).
__device__ inline int build_sentence(const TrainParams &p, const ShardState &sh, int lane, int *sen,
                                     unsigned long long &r, long long &cursor, long long &wc,
                                     int &len_out) {
  int len = 0;
  int status = 0;
  for (;;) {
    long long avail = sh.limit - cursor;
    if (avail <= 0) {
      status = sh.limit_is_eof ? 1 : 2;
      break;
    }
    int n = avail < 32 ? (int)avail : 32;
    int tok = -1;
    if (lane < n) {
      long long i = cursor + lane;
      tok = (i == sh.ovr_idx) ? sh.ovr_tok : p.tokens[i - sh.xlate];
    }
    unsigned eos = __ballot_sync(kFull, tok == 0);
    int first_eos = eos ? (__ffs(eos) - 1) : 32;
    int nw = n < first_eos ? n : first_eos;
    bool keep = lane < nw;
    unsigned long long rl = r;
    if (p.sample > 0.f) {
      rl = lcg_jump(r, lane + 1);
      if (keep) {
        float thr = p.keep_thr[tok];                       // `ran`, :403-404
        float draw = (float)(rl & 0xFFFFull) / 65536.0f;  // :406
        if (thr < draw) keep = false;
      }
    }
    unsigned km = __ballot_sync(kFull, keep);
    int need = kMaxS - len;
    int pc = __popc(km & (0xffffffffu >> (31 - lane)));  // inclusive prefix count
    int consumed, draws;
    bool finished;
    if (__popc(km) >= need) {  // the sentence reaches MAX_SENTENCE_LENGTH inside this round (:410)
      unsigned jm = __ballot_sync(kFull, keep && pc == need);
      int j = __ffs(jm) - 1;
      if (keep && lane <= j) sen[len + pc - 1] = tok;
      len = kMaxS;
      consumed = j + 1;
      draws = j + 1;
      finished = true;
    } else {
      if (keep) sen[len + pc - 1] = tok;
      len += __popc(km);
      if (first_eos < n) {  // </s> ends the sentence and is counted (:399-400)
        consumed = nw + 1;
        draws = nw;
        finished = true;
      } else {
        consumed = n;
        draws = n;
        finished = false;
      }
    }
    wc += consumed;
    cursor += consumed;
    if (p.sample > 0.f && draws > 0) r = __shfl_sync(kFull, rl, draws - 1);
    if (finished) break;
  }
  len_out = len;
  return status;
}

// Window draw, context slots and the 1+negative targets of one position (:428-460).
// Writes the descriptor; returns the RNG state after the position's draws.
template <class Desc>
__device__ inline unsigned long long make_position(const TrainParams &p, int lane, const int *sen, int len,
                                                   int sp, unsigned long long r, Desc *d) {
  r = lcg(r);
  const int W = p.window;
  int b = (int)(r % (unsigned long long)W);
  int center = len ? sen[sp] : -1;
  int cw = 0;
  if (len) {
    for (int a0 = b; a0 < 2 * W + 1 - b; a0 += 32) {
      int a = a0 + lane;
      int q = sp - W + a;
      bool ok = (a < 2 * W + 1 - b) && (a != W) && q >= 0 && q < len;
      unsigned m = __ballot_sync(kFull, ok);
      if (ok) d->ctx[cw + __popc(m & ((1u << lane) - 1))] = sen[q];
      cw += __popc(m);
    }
  }
  int nt = 0;
  if (cw) {
    if (lane == 0) d->tg[0] = center;
    nt = 1;
    for (int d0 = 1; d0 <= p.negative; d0 += 32) {
      int k = d0 + lane;
      bool ok = k <= p.negative;
      int t = 0;
      if (ok) {
        unsigned long long rd = lcg_jump(r, k);
        t = p.table[(rd >> 16) % (unsigned long long)W2B_TABLE_SIZE];                 // :456
        if (t == 0) t = (int)(rd % (unsigned long long)(p.V - 1)) + 1;                // :457
        ok = (t != center);                                                           // :458
      }
      unsigned m = __ballot_sync(kFull, ok);
      if (ok) d->tg[nt + __popc(m & ((1u << lane) - 1))] = t;
      nt += __popc(m);
    }
    r = lcg_jump(r, p.negative);
  }
  if (lane == 0) {
    d->center = center;
    d->b = b;
    d->cw = cw;
    d->nt = nt;
  }
  return r;
}

// ------------------------------------------------------------------- position arithmetic
struct BlockScratch {
  float red[2][2][16][32];  // [buffer][dot|qq][target in group][warp]
  float f, qq;              // strict-mode broadcast
};

template <bool STRICT>
__device__ __forceinline__ float mad(float a, float b, float c) {
  return STRICT ? __fadd_rn(__fmul_rn(a, b), c) : fmaf(a, b, c);
}

// Block-wide sequential sum over the D per-column values staged in `buf` (strict mode):
// the reference adds columns in ascending order (:464-470).
__device__ inline float strict_sum(float *buf, long long D, float *slot) {
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (long long c = 0; c < D; ++c) s = __fadd_rn(s, buf[c]);
    *slot = s;
  }
  __syncthreads();
  float s = *slot;
  __syncthreads();
  return s;
}

// Steps 5-7 of SURVEY Appendix A (= :431-503) for the position described by `d`.
// first_positive: target 0 carries label 1 (d == 0, :451-453).
template <int VEC, int BM, bool HAS_REG, bool STRICT, int G>
__device__ __forceinline__ void process_position(const TrainParams &p, const PosDesc *d, const QParams &qp,
                                                 const float *s_exptab, BlockScratch *bs, float *dyn,
                                                 int &redbuf, double &loss, float *f_out) {
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const bool active = tid < p.ncol;
  const long long col = (long long)tid * VEC;
  const long long D = p.D;
  const int cw = d->cw, nt = d->nt;
  const float alpha = d->alpha;
  constexpr int GG = STRICT ? 1 : G;

  // ---- context gather + quantize + average (:431-449)
  float avg[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) avg[i] = 0.f;
  float ctx_qq = 0.f;
  constexpr int CB = STRICT ? 1 : 8;
  for (int k0 = 0; k0 < cw; k0 += CB) {
    Vec<VEC> x[CB];
#pragma unroll
    for (int k = 0; k < CB; ++k)
      if (k0 + k < cw && active) x[k].load(p.u + (long long)d->ctx[k0 + k] * p.pitch + col);
#pragma unroll
    for (int k = 0; k < CB; ++k) {
      if (k0 + k < cw) {
        float rowqq[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          float q = active ? quant<BM>(x[k].a[i], qp) : 0.f;
          avg[i] = __fadd_rn(avg[i], q);
          rowqq[i] = __fmul_rn(q, q);
          if (!STRICT && HAS_REG) ctx_qq += rowqq[i];
        }
        if (STRICT) {  // per-row regularisation loss in column order (:441-445)
          if (active)
            for (int i = 0; i < VEC; ++i) dyn[col + i] = rowqq[i];
          float s = strict_sum(dyn, D, &bs->qq);
          if (tid == 0) loss += (double)(-__fmul_rn(p.reg, s));
        }
      }
    }
  }
  if (cw == 0) return;
#pragma unroll
  for (int i = 0; i < VEC; ++i) avg[i] = __fdiv_rn(avg[i], (float)cw);

  // ---- targets (:450-492)
  float err[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) err[i] = 0.f;

  for (int g0 = 0; g0 < nt; g0 += GG) {
    const int ng = (nt - g0) < GG ? (nt - g0) : GG;
    Vec<VEC> x[GG];
#pragma unroll
    for (int k = 0; k < GG; ++k)
      if (k < ng && active) x[k].load(p.v + (long long)d->tg[g0 + k] * p.pitch + col);
    float fs = 0.f, qs = 0.f;  // strict mode: the single target's sums
    if (STRICT) {
      if (active)
        for (int i = 0; i < VEC; ++i) dyn[col + i] = __fmul_rn(avg[i], quant<BM>(x[0].a[i], qp));
      fs = strict_sum(dyn, D, &bs->f);
      if (active)
        for (int i = 0; i < VEC; ++i) {
          float q = quant<BM>(x[0].a[i], qp);
          dyn[col + i] = __fmul_rn(q, q);
        }
      qs = strict_sum(dyn, D, &bs->qq);
    } else {
#pragma unroll
      for (int k = 0; k < GG; ++k) {
        float pd = 0.f, pq = 0.f;
        if (k < ng && active) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) {
            float q = quant<BM>(x[k].a[i], qp);
            pd = fmaf(avg[i], q, pd);
            if (HAS_REG) pq = fmaf(q, q, pq);
          }
        }
        if (k < ng) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            pd += __shfl_xor_sync(kFull, pd, o);
            if (HAS_REG) pq += __shfl_xor_sync(kFull, pq, o);
          }
          if (lane == 0) {
            bs->red[redbuf][0][k][warp] = pd;
            if (HAS_REG) bs->red[redbuf][1][k][warp] = pq;
          }
        }
      }
      if (HAS_REG && g0 == 0) {  // context-row regularisation loss rides on the first reduction
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ctx_qq += __shfl_xor_sync(kFull, ctx_qq, o);
        if (lane == 0) bs->red[redbuf][1][15][warp] = ctx_qq;
      }
      __syncthreads();
      if (HAS_REG && g0 == 0 && tid == 0) {
        float s = 0.f;
        for (int w = 0; w < nwarps; ++w) s += bs->red[redbuf][1][15][w];
        loss += (double)(-__fmul_rn(p.reg, s));
      }
    }
    const int rb = redbuf;
    if (!STRICT) {
      redbuf ^= 1;
      // reported loss (:480-483): lane k of warp 0 handles target k of the group; the
      // per-lane partial sums are combined when the shard state is written back
      if (warp == 0 && lane < ng) {
        float f = 0.f, fq = 0.f;
        for (int w = 0; w < nwarps; ++w) {
          f += bs->red[rb][0][lane][w];
          if (HAS_REG) fq += bs->red[rb][1][lane][w];
        }
        float dp = (g0 + lane == 0) ? f : -f;
        float ll = logf(sigmoid_report(dp));
        float rl = HAS_REG ? __fmul_rn(p.reg, fq) : 0.f;
        loss += (double)__fsub_rn(ll, rl);
        if (f_out) f_out[g0 + lane] = f;
      }
    }
#pragma unroll
    for (int k = 0; k < GG; ++k) {
      if (k < ng) {
        const int label = (g0 + k == 0) ? 1 : 0;
        float f = fs, fq = qs;
        if (!STRICT) {  // fixed-order sum of the per-warp partials
          f = 0.f;
          fq = 0.f;
          for (int w = 0; w < nwarps; ++w) {
            f += bs->red[rb][0][k][w];
            if (HAS_REG) fq += bs->red[rb][1][k][w];
          }
        }
        const float g = grad_scalar(f, label, alpha, s_exptab);
        if (STRICT && tid == 0) {
          float dp = label ? f : -f;                                   // :480
          float ll = logf(sigmoid_report(dp));                         // :481
          float rl = (HAS_REG || STRICT) ? __fmul_rn(p.reg, fq) : 0.f;
          loss += (double)__fsub_rn(ll, rl);                           // :482-483
          if (f_out) f_out[g0 + k] = f;
        }
        if (active) {
          Vec<VEC> upd;
#pragma unroll
          for (int i = 0; i < VEC; ++i) {
            float q = quant<BM>(x[k].a[i], qp);
            err[i] = mad<STRICT>(g, q, err[i]);                        // :487 (old v)
            float dv;
            if (STRICT || HAS_REG) {                                    // :490
              float t2 = __fmul_rn(__fmul_rn(__fmul_rn(2.f, alpha), p.reg), x[k].a[i]);
              dv = __fsub_rn(__fmul_rn(g, avg[i]), t2);
            } else {
              dv = g * avg[i];
            }
            upd.a[i] = STRICT ? __fadd_rn(x[k].a[i], dv) : dv;
          }
          float *row = p.v + (long long)d->tg[g0 + k] * p.pitch + col;
          if (STRICT) upd.store(row);
          else upd.red_add(row);
        }
      }
    }
  }

  // ---- scatter the accumulated error to every context row (:494-503)
  if (active) {
    for (int k = 0; k < cw; ++k) {
      float *row = p.u + (long long)d->ctx[k] * p.pitch + col;
      if (STRICT || HAS_REG) {
        Vec<VEC> x;
        x.load(row);
        Vec<VEC> upd;
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          float t2 = (STRICT || HAS_REG) ? __fmul_rn(__fmul_rn(__fmul_rn(2.f, alpha), p.reg), x.a[i]) : 0.f;
          float du = (STRICT || HAS_REG) ? __fsub_rn(err[i], t2) : err[i];
          upd.a[i] = STRICT ? __fadd_rn(x.a[i], du) : du;
        }
        if (STRICT) upd.store(row);
        else upd.red_add(row);
      } else {
        Vec<VEC> upd;
#pragma unroll
        for (int i = 0; i < VEC; ++i) upd.a[i] = err[i];
        upd.red_add(row);
      }
    }
  }
}

// ----------------------------------------------------------------------- shard kernel
template <int VEC, int BM, bool HAS_REG, bool STRICT, int G>
__device__ __forceinline__ void train_shards(TrainParams p) {
  extern __shared__ float dyn[];  // strict mode: D floats
  __shared__ int s_sen[kMaxS];
  __shared__ PosDesc s_desc[2];
  __shared__ BlockScratch s_bs;
  __shared__ float s_exptab[kExpN];
  __shared__ int s_len, s_status;
  __shared__ long long s_wc;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ShardState *shp = p.shards + p.shard_base + blockIdx.x;
  const ShardState sh = *shp;
  if (sh.done) return;
  for (int i = tid; i < kExpN; i += blockDim.x) s_exptab[i] = p.exptab[i];
  QParams qp;
  qp.bits = p.bitlevel;
  qp.seg = (p.bitlevel >= 4) ? exp2f((float)(p.bitlevel - 1)) : 1.f;

  // sampler state lives in warp 0's registers (uniform across its lanes)
  unsigned long long r = sh.rng;
  long long cursor = sh.cursor;
  long long wc = sh.word_count, last = sh.last_word_count;
  const long long wc0 = wc;
  int len = 0, sp = 0, status = 0, par = 0, redbuf = 0, done = 0;
  long long iters = 0;
  double loss = 0.0;
  unsigned long long n_pos = 0, n_ctx = 0, n_tgt = 0;
  __syncthreads();

  for (;;) {
    if (wc - last > 10000) {  // :379-393
      if (tid == 0) {
        unsigned long long delta = (unsigned long long)(wc - last) * (unsigned long long)p.wca_scale;
        long long wca = (long long)(atomicAdd(p.wca, delta) + delta);
        float a = __fmul_rn(p.starting_alpha, __fsub_rn(1.f, __fdiv_rn((float)wca, p.alpha_denom)));
        if ((double)a < (double)p.starting_alpha * 0.0001) a = (float)((double)p.starting_alpha * 0.0001);
        *(volatile float *)p.alpha = a;
      }
      last = wc;
    }
    if (len == 0) {
      if (p.word_budget > 0 && wc - wc0 >= p.word_budget) break;
      if (warp == 0) {
        unsigned long long r2 = r;
        long long c2 = cursor, w2 = wc;
        int l2 = 0;
        int st = build_sentence(p, sh, lane, s_sen, r2, c2, w2, l2);
        if (st != 2) {
          r = r2;
          cursor = c2;
        } else {
          w2 = wc;  // roll back: nothing of the partial sentence is committed
        }
        if (lane == 0) {
          s_len = l2;
          s_status = st;
          s_wc = w2;
        }
      }
      __syncthreads();
      len = s_len;
      status = s_status;
      wc = s_wc;
      sp = 0;
      if (status == 2) break;
    }
    if (status == 1 || wc > p.shard_word_limit) {  // :414-423 (a partial sentence is dropped)
      if (tid == 0) atomicAdd(p.wca, (unsigned long long)(wc - last) * (unsigned long long)p.wca_scale);
      last = wc;
      done = 1;
      break;
    }
    if (p.max_iters >= 0 && iters >= p.max_iters) break;
    ++iters;

    PosDesc *d = &s_desc[par];
    if (warp == 0) {
      r = make_position(p, lane, s_sen, len, sp, r, d);
      if (lane == 0) d->alpha = *(volatile float *)p.alpha;
    }
    __syncthreads();
    if (tid == 0 && p.trace) {  // parity hook: one record per window draw
      const long long shard = (long long)(p.shard_base + (int)blockIdx.x) * p.trace_per_shard;  // its region
      unsigned long long slot = p.trace_n[shard]++;
      if ((long long)slot < p.trace_cap) {
        w2b_trace_rec *t = p.trace + shard * p.trace_cap + slot;
        t->center = d->center; t->b = d->b; t->cw = d->cw; t->ntargets = d->nt; t->alpha = d->alpha;
        for (int k = 0; k < d->nt; ++k) t->targets[k] = d->tg[k];
      }
    }
    if (d->cw > 0) {
      n_pos += 1; n_ctx += d->cw; n_tgt += d->nt;
      if (p.train)
        process_position<VEC, BM, HAS_REG, STRICT, G>(p, d, qp, s_exptab, &s_bs, dyn, redbuf, loss, nullptr);
    }
    par ^= 1;
    ++sp;
    if (sp >= len) len = 0;  // :505-509
  }

  if (!STRICT && warp == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(kFull, loss, o);
  }
  if (tid == 0) {
    shp->rng = r;
    shp->cursor = cursor;
    shp->word_count = wc;
    shp->last_word_count = last;
    shp->done = done;
    shp->loss = sh.loss + loss;
    shp->n_iter = sh.n_iter + (unsigned long long)iters;
    shp->n_pos = sh.n_pos + n_pos;
    shp->n_ctx = sh.n_ctx + n_ctx;
    shp->n_tgt = sh.n_tgt + n_tgt;
  }
}

// A CTA has one thread per column group (ceil(D / VEC) of them, up to 1024).  train_shards_kernel is compiled for
// speed and holds more registers than 1024 threads may have (up to 182 per thread: 352 threads); the wide copy is
// held to 64 registers so that every width the ABI accepts launches.  Strict mode always runs the wide copy.
template <int VEC, int BM, bool HAS_REG, bool STRICT, int G>
__global__ void train_shards_kernel(TrainParams p) { train_shards<VEC, BM, HAS_REG, STRICT, G>(p); }
template <int VEC, int BM, bool HAS_REG, bool STRICT, int G>
__global__ void __launch_bounds__(1024, 1) train_shards_wide_kernel(TrainParams p) {
  train_shards<VEC, BM, HAS_REG, STRICT, G>(p);
}

// One explicit position (L1 single-step parity hook).
template <int VEC, int BM, bool HAS_REG, bool STRICT, int G>
__device__ __forceinline__ void apply_position(TrainParams p, const int *ctx, int cw, const int *tg, int nt,
                                               float *f_out, double *loss_out) {
  extern __shared__ float dyn[];
  __shared__ PosDesc s_desc;
  __shared__ BlockScratch s_bs;
  __shared__ float s_exptab[kExpN];
  for (int i = threadIdx.x; i < kExpN; i += blockDim.x) s_exptab[i] = p.exptab[i];
  if (threadIdx.x == 0) {
    s_desc.center = nt ? tg[0] : -1;
    s_desc.b = 0;
    s_desc.cw = cw;
    s_desc.nt = nt;
    s_desc.alpha = *p.alpha;
    for (int k = 0; k < cw; ++k) s_desc.ctx[k] = ctx[k];
    for (int k = 0; k < nt; ++k) s_desc.tg[k] = tg[k];
  }
  __syncthreads();
  QParams qp;
  qp.bits = p.bitlevel;
  qp.seg = (p.bitlevel >= 4) ? exp2f((float)(p.bitlevel - 1)) : 1.f;
  int redbuf = 0;
  double loss = 0.0;
  process_position<VEC, BM, HAS_REG, STRICT, G>(p, &s_desc, qp, s_exptab, &s_bs, dyn, redbuf, loss, f_out);
  if (!STRICT && threadIdx.x < 32) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(kFull, loss, o);
  }
  if (threadIdx.x == 0 && loss_out) *loss_out = loss;
}
template <int VEC, int BM, bool HAS_REG, bool STRICT, int G>
__global__ void apply_position_kernel(TrainParams p, const int *ctx, int cw, const int *tg, int nt, float *f_out,
                                      double *loss_out) {
  apply_position<VEC, BM, HAS_REG, STRICT, G>(p, ctx, cw, tg, nt, f_out, loss_out);
}
template <int VEC, int BM, bool HAS_REG, bool STRICT, int G>
__global__ void __launch_bounds__(1024, 1) apply_position_wide_kernel(TrainParams p, const int *ctx, int cw,
                                                                      const int *tg, int nt, float *f_out,
                                                                      double *loss_out) {
  apply_position<VEC, BM, HAS_REG, STRICT, G>(p, ctx, cw, tg, nt, f_out, loss_out);
}

// ------------------------------------------------------------------- auxiliary kernels
// InitNet (:343-361): element e (v first, then u) takes draw e+1 of the LCG seeded with 1.  n = V*D elements per table;
// element (row, col) is stored at row*pitch + col (padding columns, if any, stay zero).
__global__ void init_net_kernel(float *v, float *u, long long n, long long D, long long pitch) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long e0 = t * 4;
  if (e0 >= 2 * n) return;
  unsigned long long r = lcg_jump_big(1ULL, (unsigned long long)e0);
  for (int i = 0; i < 4; ++i) {
    long long e = e0 + i;
    if (e >= 2 * n) break;
    r = lcg(r);
    float val = __fsub_rn((float)(r & 0xFFFFull) / 65536.0f, 0.5f);
    const long long x = e < n ? e : e - n;
    const long long at = pitch == D ? x : (x / D) * pitch + x % D;
    if (e < n) v[at] = val;
    else u[at] = val;
  }
}

// InitUnigramTable (:112-128) from host-computed boundaries: table[a] = max{i: start[i] <= a}.
__global__ void fill_table_kernel(int *table, const int *start, int V) {
  long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= W2B_TABLE_SIZE) return;
  int lo = 0, hi = V;  // invariant: start[lo] <= a < start[hi] (start[V] = 1e8)
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (start[mid] <= (int)a) lo = mid; else hi = mid;
  }
  table[a] = lo;
}

// quantize(u+v), :568-569; out is V x D contiguous, u and v have rows of `pitch` floats
__global__ void export_kernel(const float *u, const float *v, float *out, long long n, long long D, long long pitch, int bits) {
  QParams qp;
  qp.bits = bits;
  qp.seg = (bits >= 4) ? exp2f((float)(bits - 1)) : 1.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long at = pitch == D ? i : (i / D) * pitch + i % D;
    out[i] = quant<9>(__fadd_rn(u[at], v[at]), qp);
  }
}

__global__ void quantize_kernel(const float *in, float *out, long long n, int bits) {
  QParams qp;
  qp.bits = bits;
  qp.seg = (bits >= 4) ? exp2f((float)(bits - 1)) : 1.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = quant<9>(in[i], qp);
}

__global__ void scale_kernel(float *x, long long n, float s) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[i] *= s;
}

}  // namespace w2b
