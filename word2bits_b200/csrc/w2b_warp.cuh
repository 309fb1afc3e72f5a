// Production kernel of the Word2Bits training path for sm_90a: one WARP per corpus shard.
//
// A shard is what one reference thread walks (TrainModelThread, src/word2bits.cpp:363-516).  Here it is one
// warp in a CTA of its own (32 threads, grid = shards), so an H100 runs 132 x 4..24 shards side by side and
// hides HBM latency with shards, not with a deep pipeline inside a shard.  The warp does everything the
// reference thread does, in the reference's order:
//   * sampling (:379-460): learning-rate schedule, sentence builder + sub-sampling, shard termination, window
//     draw, negative draws — 32 draws at a time by LCG jump-ahead; the unigram-table lookups of position p+1
//     are in flight while position p is trained;
//   * every embedding row a position touches streams through a small ring of K shared-memory slots as a JOB:
//     cw context rows of u, then 1+negative target rows of v, then one staging job.  Lane 0 moves rows with
//     the bulk-copy engine (cp.async.bulk global -> shared, completion on an mbarrier per slot) and keeps
//     K-2 loads in flight while the warp works on a landed row;
//   * context job (:431-449): lane l owns float4 columns l, l+32, ...; quantize and accumulate in registers;
//   * target job (:450-492): quantize, dot against the context average (registers), 5-step butterfly, g from
//     the expTable (constant memory, warp-uniform index), error accumulated in registers (:487), the row is
//     overwritten in place with g*context_avg (:490) and handed back with ONE cp.reduce.async.bulk.add.f32
//     (an atomic-add scatter of the whole row in L2);
//   * staging job (:494-503): the error registers are written to the slot and bulk-reduced into every
//     context row of u.
// Flow control is private to the warp: job j lives in slot j mod K; every job commits exactly one bulk
// async-group (empty for a context job), so after `wait_group.read 1` the slot of the job before the one just
// finished is free and the next load is issued into it.  No CTA barrier, no inter-warp traffic, context_avg
// and the error never leave registers.
//
// Ordering semantics: TrainParams::serial = 1 fetches the rows of position p+1 only after every update of
// position p has completed (sequential semantics inside a shard, like one reference thread; the only
// staleness left is Hogwild between shards, which the reference's threads have too).  serial = 0 lets the ring
// run ahead across positions: a context row shared by neighbouring positions is then read one update stale
// (no update is ever lost: all scatters are atomic adds).  Duplicate targets inside one position read the same
// old row in both modes.
#pragma once
#include "w2b_kernels.cuh"
#include "w2b_ptx.cuh"

namespace w2b {

__constant__ float c_exptab[kExpN];  // expTable (:614-618), uploaded by w2b_create

constexpr int kJobTarget = 0x40000000;  // job queue entry: row id | kJobTarget = row of v; -1 = staging job
constexpr int kJobIdMask = 0x3fffffff;

// Shared-memory carve-up of one warp (host and device agree through this helper).
// Sampler state of a shard: warp-uniform, kept in shared memory between positions (the arithmetic needs the
// registers; every lane stores the same values).
struct WarpSampler {
  unsigned long long r;
  long long cursor, wc, last, wc0, iters;
  unsigned long long r1_pre;
  int len, sp, status, done;
  int have_pre;
  float alpha_c;
  unsigned n_pos, n_ctx, n_tgt;  // per launch (a launch is bounded to 4 M words per shard)
};

struct WarpLayout {
  int rowb, K, qcap;
  size_t off_ring, off_sen, off_jobq, off_samp, off_bar, total;
};
// sen_smem: the shard's current sentence (4000 B) lives in shared memory; 0: in a global scratch buffer
// (TrainParams::sen) — wide rows at 16 warps per SM leave no room for it.
__host__ __device__ inline WarpLayout warp_layout(long long D, int K, int qcap, int sen_smem) {
  WarpLayout L;
  L.rowb = (int)(D * 4);
  L.K = K;
  L.qcap = qcap;
  size_t o = 0;
  L.off_ring = o; o += (size_t)K * L.rowb;
  L.off_sen = o;  o += sen_smem ? sizeof(int) * (size_t)kMaxS : 0;  // the shard's current sentence (:394-413)
  L.off_jobq = o; o += sizeof(int) * (size_t)qcap;
  o = (o + 7) & ~(size_t)7;
  L.off_samp = o; o += sizeof(WarpSampler);
  o = (o + 7) & ~(size_t)7;
  L.off_bar = o;  o += 8 * (size_t)K;
  L.total = (o + 15) & ~(size_t)15;
  return L;
}
// job queue capacity: two positions (the one being trained and the one sampled ahead), power of two
__host__ __device__ inline int warp_queue_capacity(int window, int negative) {
  const int need = 2 * (2 * window + negative + 2);
  int q = 32;
  while (q < need) q <<= 1;
  return q;
}

// ---------------------------------------------------------------------------- fp32 pairs
// (sm_90 has no packed fp32 arithmetic: a pair is two scalar round-to-nearest operations)
struct F2 { float x, y; };
__device__ __forceinline__ F2 fma2(F2 a, F2 b, F2 c) { return F2{fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)}; }
__device__ __forceinline__ F2 mul2(F2 a, F2 b) { return F2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 add2(F2 a, F2 b) { return F2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
#ifdef W2B_EMULATE
__device__ __forceinline__ float sign_level(float x, float level) {  // (x & 0x80000000) | level
  unsigned xi, li;
  memcpy(&xi, &x, 4); memcpy(&li, &level, 4);
  xi = (xi & 0x80000000u) | li;
  float r; memcpy(&r, &xi, 4);
  return r;
}
__device__ __forceinline__ float ldc_exptab(int i) { return c_exptab[i]; }
#else
__device__ __forceinline__ float sign_level(float x, float level) {  // (x & 0x80000000) | level: one LOP3
  unsigned r;
  asm("lop3.b32 %0, %1, 0x80000000, %2, 0xEA;" : "=r"(r) : "r"(__float_as_uint(x)), "r"(__float_as_uint(level)));
  return __uint_as_float(r);
}
__device__ __forceinline__ float ldc_exptab(int i) { return c_exptab[i]; }
#endif

// a / fcw for a small integer fcw with rc = RN(1 / fcw), correctly rounded without the division subroutine (which
// takes its slow path for every exactly-zero numerator — and sums of +-1/3 are often exactly zero): q = a*rc, then
// one Newton step on the exact remainder.  Equals IEEE division for every fcw <= 128 and every numerator in range
// (tests/test_warp_emulation.py::test_division_free_average_is_ieee_division runs this very function on the host).
__device__ __forceinline__ F2 div_by_count(F2 a, float fcw, float rc) {
  const F2 r2 = F2{rc, rc}, nc2 = F2{-fcw, -fcw};
  const F2 q0 = mul2(a, r2);
  const F2 rem = fma2(q0, nc2, a);
  return fma2(rem, r2, q0);
}

// quantize() (:73-108) as the training loop uses it.  bitlevel 1 and 2 copy the SIGN BIT onto the level instead
// of testing x < 0: identical for every value except -0.0 (and NaNs with the sign bit set), which the reference
// maps to the positive level; a master weight can only become -0.0 through a flushed negative denormal sum.
// The exported vectors (export_kernel) and the strict kernel use the exact form (w2b_quant.cuh).
template <int BM>
__device__ __forceinline__ float quant_fast(float x, const QParams &q) {
  if (BM == 0) return x;
  if (BM == 1) return sign_level(x, 0.33333334f);
  if (BM == 2) return sign_level(x, fabsf(x) <= 0.5f ? 0.25f : 0.75f);
  return quant<9>(x, q);
}

// gradient scalar (:473-475) with the expTable in constant memory (f is warp-uniform after the butterfly).
__device__ __forceinline__ float grad_scalar_c(float f, int label, float alpha) {
  if (f > 6.f) return __fmul_rn((float)(label - 1), alpha);
  if (f < -6.f) return __fmul_rn((float)label, alpha);
  const int idx = __float2int_rz(__fmul_rn(__fadd_rn(f, 6.f), 83.f));
  return __fmul_rn(__fsub_rn((float)label, ldc_exptab(idx)), alpha);
}

// Explicit single position (L1 parity hook, w2b_apply_position): ids instead of draws.
struct ApplyArgs {
  const int *ctx, *tg;
  int cw, nt;
  float *f_out;
};

// Samples forward to the next trained position (cw > 0) of the shard and appends its jobs — cw context ids, nt
// target ids | kJobTarget, -1 — to the job queue at index qtail.  Returns 1 with cw / nt / alpha of the position,
// or 0 when the launch is over for this shard (word budget, shard end, slice exhausted, max_iters).
// Control flow and draw order of :379-460.  While a position is trained, the unigram-table lookups of the next
// position of the same sentence (whose draws are already determined) are in flight in `t_pre` / S.r1_pre.
__device__ inline int warp_next_position(const TrainParams &p, const ShardState &sh, WarpSampler &Ssm, int lane, int *sen,
                                         int *jobq, int qmask, unsigned qtail, int &t_pre, int &cw_out, int &nt_out,
                                         float &alpha_out) {
  const int W = p.window, neg = p.negative;
  const unsigned long long JA1 = c_JA[lane + 1], JC1 = c_JC[lane + 1];  // lane's own jump constants
  // every lane works on its own (identical) copy; lane 0 writes it back on the way out.  Updating the shared copy
  // in place would be a race: lanes of a warp are not guaranteed to take the read-modify-writes in lockstep.
  WarpSampler S = Ssm;
  auto leave = [&](int rc) {
    __syncwarp();
    if (lane == 0) Ssm = S;
    __syncwarp();
    return rc;
  };
  const int negl = neg < 32 ? neg : 32;
  const unsigned long long JAn = c_JA[neg], JCn = c_JC[neg];
  for (;;) {
    if (S.wc - S.last > 10000) {  // :379-393
      const unsigned long long delta = (unsigned long long)(S.wc - S.last) * (unsigned long long)p.wca_scale;
      long long wca = 0;
      if (lane == 0) wca = (long long)(atomicAdd(p.wca, delta) + delta);
      wca = __shfl_sync(kFull, wca, 0);
      float a = __fmul_rn(p.starting_alpha, __fsub_rn(1.f, __fdiv_rn((float)wca, p.alpha_denom)));
      if ((double)a < (double)p.starting_alpha * 0.0001) a = (float)((double)p.starting_alpha * 0.0001);
      if (lane == 0) *(volatile float *)p.alpha = a;
      S.alpha_c = a;
      S.last = S.wc;
    }
    if (S.len == 0) {
      if (p.word_budget > 0 && S.wc - S.wc0 >= p.word_budget) return leave(0);
      unsigned long long r2 = S.r;
      long long c2 = S.cursor, w2 = S.wc;
      int l2 = 0;
      S.status = build_sentence(p, sh, lane, sen, r2, c2, w2, l2);
      __syncwarp();
      if (S.status == 2) return leave(0);  // slice exhausted mid-sentence: nothing committed
      S.r = r2; S.cursor = c2; S.wc = w2; S.len = l2; S.sp = 0;
      S.have_pre = 0;
      // the shared learning rate (:53) is re-read once per sentence: other shards move it every 10k words each
      S.alpha_c = *(volatile float *)p.alpha;
    }
    if (S.status == 1 || S.wc > p.shard_word_limit) {  // :414-423
      if (lane == 0) atomicAdd(p.wca, (unsigned long long)(S.wc - S.last) * (unsigned long long)p.wca_scale);
      S.last = S.wc;
      S.done = 1;
      return leave(0);
    }
    ++S.iters;
    // ---- draws of this position (:428-460)
    unsigned long long r1, rd;
    int t = 0;
    if (S.have_pre) {
      r1 = S.r1_pre; rd = r1 * JA1 + JC1; t = t_pre;
    } else {
      r1 = lcg(S.r);
      rd = r1 * JA1 + JC1;
      if (lane < negl) t = p.table[(rd >> 16) % (unsigned long long)W2B_TABLE_SIZE];
    }
    S.have_pre = 0;
    const int b = mod_small(r1, (unsigned)W);
    const int len = S.len, sp = S.sp;
    const int center = len ? sen[sp] : -1;
    int cw = 0;
    if (len) {
      for (int a0 = b; a0 < 2 * W + 1 - b; a0 += 32) {
        const int a = a0 + lane;
        const int qq = sp - W + a;
        const bool ok = (a < 2 * W + 1 - b) && (a != W) && qq >= 0 && qq < len;
        const unsigned m = __ballot_sync(kFull, ok);
        if (ok) jobq[(qtail + cw + __popc(m & ((1u << lane) - 1))) & qmask] = sen[qq];
        cw += __popc(m);
      }
    }
    int nt = 0;
    if (cw) {
      const unsigned long long r_after = r1 * JAn + JCn;
      if (sp + 1 < len) {  // next position of the sentence: its draws are already determined
        const unsigned long long r1n = lcg(r_after);
        const unsigned long long rdn = r1n * JA1 + JC1;
        S.r1_pre = r1n;
        t_pre = 0;
        if (lane < negl) t_pre = p.table[(rdn >> 16) % (unsigned long long)W2B_TABLE_SIZE];
        S.have_pre = 1;
      }
      const unsigned tq = qtail + cw;
      if (lane == 0) jobq[tq & qmask] = center | kJobTarget;
      nt = 1;
      {
        bool ok = lane < negl;
        int tt = t;
        if (ok && tt == 0) tt = (int)(rd % (unsigned long long)(p.V - 1)) + 1;  // :457
        ok = ok && (tt != center);                                                 // :458
        const unsigned m = __ballot_sync(kFull, ok);
        if (ok) jobq[(tq + nt + __popc(m & ((1u << lane) - 1))) & qmask] = tt | kJobTarget;
        nt += __popc(m);
      }
      for (int d0 = 33; d0 <= neg; d0 += 32) {  // negative > 32: remaining draws, not prefetched
        const int k = d0 + lane;
        bool ok = k <= neg;
        int tt = 0;
        if (ok) {
          const unsigned long long rd2 = lcg_jump(r1, k);
          tt = p.table[(rd2 >> 16) % (unsigned long long)W2B_TABLE_SIZE];
          if (tt == 0) tt = (int)(rd2 % (unsigned long long)(p.V - 1)) + 1;
          ok = (tt != center);
        }
        const unsigned m = __ballot_sync(kFull, ok);
        if (ok) jobq[(tq + nt + __popc(m & ((1u << lane) - 1))) & qmask] = tt | kJobTarget;
        nt += __popc(m);
      }
      if (lane == 0) jobq[(tq + nt) & qmask] = -1;  // staging job (:494-503)
      S.r = r_after;
    } else {
      S.r = r1;
    }
    ++S.sp;
    if (S.sp >= S.len) S.len = 0;  // :505-509
    __syncwarp();                  // the queue entries are visible to every lane
    if (p.trace) {  // parity hook: one record per window draw, exactly what the oracle's trace holds
      if (lane == 0) {
        const long long shard = (long long)(p.shard_base + (int)blockIdx.x) * p.trace_per_shard;  // its region
        const unsigned long long k = p.trace_n[shard]++;
        if ((long long)k < p.trace_cap) {
          w2b_trace_rec *tr = p.trace + shard * p.trace_cap + k;
          tr->center = center; tr->b = b; tr->cw = cw; tr->ntargets = nt; tr->alpha = S.alpha_c;
          for (int i = 0; i < nt; ++i) tr->targets[i] = jobq[(qtail + cw + i) & qmask] & kJobIdMask;
        }
      }
      __syncwarp();
    }
    if (p.max_iters >= 0 && S.iters >= p.max_iters) {
      if (cw) { S.n_pos += 1; S.n_ctx += cw; S.n_tgt += nt; }
      return leave(0);
    }
    if (cw == 0) continue;  // single-word or empty sentence: one window draw, nothing trained
    S.n_pos += 1; S.n_ctx += cw; S.n_tgt += nt;
    if (!p.train) continue;  // draws only
    cw_out = cw; nt_out = nt; alpha_out = S.alpha_c;
    return leave(1);
  }
}

// BM: compile-time bitlevel 0/1/2, 9 = run time.  NJ = float4 columns per lane = ceil(D / 128).  MINB = CTAs (warps)
// per SM the register allocation is sized for.
// REG = 1: -reg != 0 (:443-445,:471,:490,:501).  Every row then also decays by 2*alpha*reg times its own (raw) value:
// a target row in the same scatter as its update (g*context_avg - 2*alpha*reg*v), a context row by a scatter of its
// own when it is read (the reference subtracts at the end of the position from a value this thread has not changed
// in between — same sum, other order); the regularisation terms of the reported loss are accumulated per lane.
template <int BM, int NJ, int MINB, int REG = 0>
__global__ void __launch_bounds__(32, MINB) train_warp_kernel(TrainParams p, int K, int qcap_sen, ApplyArgs ap) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int lane = threadIdx.x;
  const int qcap = qcap_sen & 0x7fffffff, sen_smem = (qcap_sen >> 31) & 1;  // top bit: sentence in shared memory
  const WarpLayout L = warp_layout(p.pitch, K, qcap, sen_smem);
  const unsigned s_base = smem_u32(smem);
  const unsigned ring = s_base + (unsigned)L.off_ring;
  const unsigned bars = s_base + (unsigned)L.off_bar;
  int *jobq = reinterpret_cast<int *>(smem + L.off_jobq);
  const int qmask = qcap - 1;
  const unsigned rowb = (unsigned)L.rowb;
  const int D4 = (int)(p.pitch >> 2);  // float4 columns of a row
  const int shard = p.shard_base + blockIdx.x;
  ShardState *shp = p.shards + shard;
  if (!ap.ctx && shp->done) return;
  int *sen = sen_smem ? reinterpret_cast<int *>(smem + L.off_sen) : p.sen + (size_t)shard * kMaxS;

  if (lane == 0) {
    for (int i = 0; i < K; ++i) mbar_init(reinterpret_cast<unsigned long long *>(smem + L.off_bar) + i, 1);
#ifndef W2B_EMULATE
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  }
  __syncwarp();

  QParams qp;
  qp.bits = p.bitlevel;
  qp.seg = (p.bitlevel >= 4) ? exp2f((float)(p.bitlevel - 1)) : 1.f;

  // lane's float4 columns j*32+lane; every column group but the last is full (NJ == ceil(D4 / 32)); columns past
  // the row end are clamped for loads and masked for stores (their context_avg is zero, so they add nothing)
  const unsigned lane16 = (unsigned)lane * 16u;
  const bool on_last = (NJ - 1) * 32 + lane < D4;
  const unsigned coff_last = (unsigned)(on_last ? (NJ - 1) * 32 + lane : D4 - 1) * 16u;
  // D % 4 != 0: rows are padded to whole float4s; the lane that holds the last float4 keeps only its first `tail`
  // components of context_avg (the padding must not enter a dot product: quantize(0) is a level, not zero)
  const int tail = ((NJ - 1) * 32 + lane == D4 - 1) ? (int)(p.D & 3) : 0;
#define W2B_COFF(j) ((j) < NJ - 1 ? lane16 + (unsigned)(j) * 512u : coff_last)

  const ShardState &sh = *shp;
  WarpSampler &S = *reinterpret_cast<WarpSampler *>(smem + L.off_samp);
  S.r = sh.rng; S.cursor = sh.cursor; S.wc = sh.word_count; S.last = sh.last_word_count; S.wc0 = S.wc;
  S.iters = 0; S.len = 0; S.sp = 0; S.status = 0; S.done = 0; S.have_pre = 0;
  S.r1_pre = 0; S.n_pos = S.n_ctx = S.n_tgt = 0;
  S.alpha_c = *(volatile float *)p.alpha;
  int t_pre = 0;  // per lane: the next position's unigram-table lookup, in flight while this one is trained
  __syncwarp();

  // ---- job bookkeeping (all warp-uniform).  Job j lives in slot j mod K; the issue side and the arithmetic each
  // keep their slot's shared-memory address and mbarrier incrementally.  Every job arms its slot's mbarrier exactly
  // once (a staging job with 0 bytes), so all slots advance one phase per trip round the ring and one parity bit,
  // flipped at the wrap, serves every wait.
  unsigned q_tail = 0;   // jobs appended to the queue
  unsigned q_issue = 0;  // jobs whose load has been issued (staging jobs: barrier armed)
  unsigned q_cons = 0;   // jobs consumed
  unsigned q_limit = 0;  // jobs the issue side may look at (serial: end of the current position)
  const unsigned ring_end = ring + (unsigned)K * rowb;
  unsigned i_row = ring, i_bar = bars;  // issue slot
  unsigned c_row = ring, c_bar = bars;  // slot of the job being worked on
  unsigned c_par = 0;
  double loss = 0.0;     // per lane: reported loss of the targets this lane looked after
  // a job may be issued once the job K before it has left its slot, which is known after the `wait_group.read 1`
  // that follows the NEXT job: K - 2 loads in flight behind the row being worked on
  const unsigned ahead = (unsigned)K - 2u;

  auto issue_one = [&]() {  // all lanes; lane 0 acts.  Precondition: q_issue < q_limit, slot free.
    const int e = jobq[q_issue & qmask];
    if (lane == 0) {
      if (e >= 0) {
        const float *src = (e & kJobTarget) ? p.v + (long long)(e & kJobIdMask) * p.pitch : p.u + (long long)e * p.pitch;
        mbar_expect_tx(i_bar, rowb);
        bulk_load(i_row, src, rowb, i_bar);
      } else {
        mbar_expect_tx(i_bar, 0);
      }
    }
    ++q_issue;
    i_row += rowb; i_bar += 8u;
    if (i_row == ring_end) { i_row = ring; i_bar = bars; }
  };
  auto pump = [&]() {
    while (q_issue < q_limit && q_issue <= q_cons + ahead) issue_one();
  };
  // End of a job, after every lane is done with the slot (__syncwarp by the caller): lane 0 hands the slot's row to
  // the bulk-copy engine as an atomic-add scatter — to `dst` (target job), or to the position's n_dst context rows
  // of u (staging job; none for a context job) — confirms the previous job's slot and refills it: one divergent
  // region per job.
  auto finish_job = [&](float *dst, int n_dst, unsigned q0) {
    ++q_cons;
    const bool can = q_issue < q_limit && q_issue <= q_cons + ahead;
    const int e = can ? jobq[q_issue & qmask] : -1;
    if (lane == 0) {
      if (dst) bulk_reduce_add(dst, c_row, rowb);
      else for (int k = 0; k < n_dst; ++k) bulk_reduce_add(p.u + (long long)jobq[(q0 + k) & qmask] * p.pitch, c_row, rowb);
      bulk_commit();
      bulk_wait_read<1>();
      if (can) {
        if (e >= 0) {
          const float *src = (e & kJobTarget) ? p.v + (long long)(e & kJobIdMask) * p.pitch : p.u + (long long)e * p.pitch;
          mbar_expect_tx(i_bar, rowb);
          bulk_load(i_row, src, rowb, i_bar);
        } else {
          mbar_expect_tx(i_bar, 0);
        }
      }
    }
    if (can) {
      ++q_issue;
      i_row += rowb; i_bar += 8u;
      if (i_row == ring_end) { i_row = ring; i_bar = bars; }
    }
    c_row += rowb; c_bar += 8u;
    if (c_row == ring_end) { c_row = ring; c_bar = bars; c_par ^= 1u; }
  };

  int n_cw = 0, n_nt = 0;
  float n_alpha = 0.f;
  int have_next;
  if (ap.ctx) {  // one explicit position
    for (int k = lane; k < ap.cw; k += 32) jobq[k & qmask] = ap.ctx[k];
    for (int k = lane; k < ap.nt; k += 32) jobq[(ap.cw + k) & qmask] = ap.tg[k] | kJobTarget;
    if (lane == 0) jobq[(ap.cw + ap.nt) & qmask] = -1;
    __syncwarp();
    n_cw = ap.cw; n_nt = ap.nt; n_alpha = S.alpha_c;
    have_next = ap.cw > 0;
  } else {
    have_next = warp_next_position(p, sh, S, lane, sen, jobq, qmask, q_tail, t_pre, n_cw, n_nt, n_alpha);
  }
  if (have_next) q_tail += (unsigned)(n_cw + n_nt + 1);

  while (have_next) {
    const int cw = n_cw, nt = n_nt;
    const float alpha = n_alpha;
    const unsigned q0 = q_cons;  // first job of this position
    q_limit = q0 + (unsigned)(cw + nt + 1);
    pump();
    // sample one position ahead: its jobs extend the queue (and, without serial, what the ring may prefetch)
    have_next = ap.ctx ? 0 : warp_next_position(p, sh, S, lane, sen, jobq, qmask, q_tail, t_pre, n_cw, n_nt, n_alpha);
    if (have_next) q_tail += (unsigned)(n_cw + n_nt + 1);
    if (!p.serial) { q_limit = q_tail; pump(); }

    // ---- context jobs: gather + quantize + average (:431-449)
    F2 a[NJ][2];
#pragma unroll
    for (int j = 0; j < NJ; ++j) a[j][0] = a[j][1] = F2{0.f, 0.f};
    float regsum = 0.f;                                    // REG: sum of squared quantized values this lane saw
    const float decay = REG ? -2.f * alpha * p.reg : 0.f;  // REG: row += decay * row
    for (int k = 0; k < cw; ++k) {
      float *urow = REG ? p.u + (long long)jobq[q_cons & qmask] * p.pitch : nullptr;
      mbar_wait(c_bar, c_par);
      float4 x[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) x[j] = lds128(c_row + W2B_COFF(j));
      if constexpr (REG) {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const float4 xq = make_float4(quant_fast<BM>(x[j].x, qp), quant_fast<BM>(x[j].y, qp), quant_fast<BM>(x[j].z, qp),
                                        quant_fast<BM>(x[j].w, qp));
          a[j][0] = add2(a[j][0], F2{xq.x, xq.y});
          a[j][1] = add2(a[j][1], F2{xq.z, xq.w});
          if ((j < NJ - 1) || on_last) {
            const bool tl = tail && j == NJ - 1;  // padding components do not count
            regsum += (xq.x * xq.x + ((tl && tail < 2) ? 0.f : xq.y * xq.y)) +
                      (((tl && tail < 3) ? 0.f : xq.z * xq.z) + (tl ? 0.f : xq.w * xq.w));
            sts128(c_row + W2B_COFF(j), make_float4(decay * x[j].x, decay * x[j].y, decay * x[j].z, decay * x[j].w));
          }
        }
        fence_async_smem();
        __syncwarp();
        finish_job(urow, 0, q0);
      } else {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          a[j][0] = add2(a[j][0], F2{quant_fast<BM>(x[j].x, qp), quant_fast<BM>(x[j].y, qp)});
          a[j][1] = add2(a[j][1], F2{quant_fast<BM>(x[j].z, qp), quant_fast<BM>(x[j].w, qp)});
        }
        __syncwarp();
        finish_job(nullptr, 0, q0);
      }
    }
    {  // context_avg = sum / cw (:449)
      const float fcw = (float)cw;
      const float rc = __frcp_rn(fcw);
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const bool on = (j < NJ - 1) || on_last;
#pragma unroll
        for (int h = 0; h < 2; ++h) a[j][h] = on ? div_by_count(a[j][h], fcw, rc) : F2{0.f, 0.f};
      }
      if (tail) {  // (tail lanes are in the last column group)
        if (tail < 2) a[NJ - 1][0].y = 0.f;
        if (tail < 3) a[NJ - 1][1].x = 0.f;
        a[NJ - 1][1].y = 0.f;
      }
    }

    // ---- target jobs (:450-492)
    F2 e[NJ][2];
#pragma unroll
    for (int j = 0; j < NJ; ++j) e[j][0] = e[j][1] = F2{0.f, 0.f};
    float myf0 = 0.f, myf1 = 0.f;  // lane i keeps +-f of targets i and 32+i for the reported loss (:480-483)
    for (int i = 0; i < nt; ++i) {
      float *dst = p.v + (long long)(jobq[q_cons & qmask] & kJobIdMask) * p.pitch;
      mbar_wait(c_bar, c_par);
      float4 x[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) x[j] = lds128(c_row + W2B_COFF(j));
      F2 d0 = F2{0.f, 0.f}, d1 = F2{0.f, 0.f};
      float4 raw[REG ? NJ : 1];  // REG: the decay needs the row as it was loaded
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        if (REG) raw[j] = x[j];
        x[j] = make_float4(quant_fast<BM>(x[j].x, qp), quant_fast<BM>(x[j].y, qp), quant_fast<BM>(x[j].z, qp),
                           quant_fast<BM>(x[j].w, qp));
        d0 = fma2(a[j][0], F2{x[j].x, x[j].y}, d0);
        d1 = fma2(a[j][1], F2{x[j].z, x[j].w}, d1);
        if (REG && ((j < NJ - 1) || on_last)) {
          const bool tl = tail && j == NJ - 1;
          regsum += (x[j].x * x[j].x + ((tl && tail < 2) ? 0.f : x[j].y * x[j].y)) +
                    (((tl && tail < 3) ? 0.f : x[j].z * x[j].z) + (tl ? 0.f : x[j].w * x[j].w));
        }
      }
      float f = (d0.x + d0.y) + (d1.x + d1.y);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) f += __shfl_xor_sync(kFull, f, o);
      const float g = grad_scalar_c(f, i == 0 ? 1 : 0, alpha);
      {
        const float sf = (i == 0) ? f : -f;
        if (i < 32) { if (lane == i) myf0 = sf; }
        else if (lane == i - 32) myf1 = sf;
      }
      const F2 g2 = F2{g, g};
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        e[j][0] = fma2(g2, F2{x[j].x, x[j].y}, e[j][0]);  // :487, quantized OLD v
        e[j][1] = fma2(g2, F2{x[j].z, x[j].w}, e[j][1]);
        F2 u0 = mul2(g2, a[j][0]), u1 = mul2(g2, a[j][1]);  // :490: g*context_avg replaces the row in its slot
        if (REG) {
          u0 = F2{fmaf(decay, raw[j].x, u0.x), fmaf(decay, raw[j].y, u0.y)};
          u1 = F2{fmaf(decay, raw[j].z, u1.x), fmaf(decay, raw[j].w, u1.y)};
        }
        if ((j < NJ - 1) || on_last) sts128(c_row + W2B_COFF(j), make_float4(u0.x, u0.y, u1.x, u1.y));
      }
      fence_async_smem();
      __syncwarp();
      finish_job(dst, 1, q0);
    }

    // ---- staging job: the error goes to every context row of u (:494-503)
    {
      mbar_wait(c_bar, c_par);  // armed with 0 bytes, long complete: every job observes its slot's phase (synccheck-clean)
#pragma unroll
      for (int j = 0; j < NJ; ++j)
        if ((j < NJ - 1) || on_last) sts128(c_row + W2B_COFF(j), make_float4(e[j][0].x, e[j][0].y, e[j][1].x, e[j][1].y));
      fence_async_smem();
      __syncwarp();
      if (lane < nt) loss += (double)logf(sigmoid_report(myf0));
      if (lane + 32 < nt) loss += (double)logf(sigmoid_report(myf1));
      if (REG) loss -= (double)(p.reg * regsum);  // :443-445 and :471, summed over the position's rows
      if (ap.f_out) {
        if (lane < nt) ap.f_out[lane] = lane == 0 ? myf0 : -myf0;
        if (lane + 32 < nt) ap.f_out[lane + 32] = -myf1;
      }
      finish_job(nullptr, cw, q0);
      if (p.serial) {  // every update of this position has completed before the next position's rows are fetched
        if (lane == 0) bulk_wait_all();
        __syncwarp();
      }
    }
  }
#undef W2B_COFF
  if (lane == 0) bulk_wait_all();
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(kFull, loss, o);
  if (lane == 0 && !ap.ctx) {
    shp->rng = S.r;
    shp->cursor = S.cursor;
    shp->word_count = S.wc;
    shp->last_word_count = S.last;
    shp->done = S.done;
    shp->loss = sh.loss + loss;
    shp->n_iter = sh.n_iter + (unsigned long long)S.iters;
    shp->n_pos = sh.n_pos + S.n_pos;
    shp->n_ctx = sh.n_ctx + S.n_ctx;
    shp->n_tgt = sh.n_tgt + S.n_tgt;
  }
}

}  // namespace w2b
