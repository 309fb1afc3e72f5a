// Bit-domain scoring of the analogy evaluator on packed 1-bit and 2-bit vector files (w2b_write_packed) for sm_90a.
//
// A packed row holds one or two bits per value: the sign and, at 2 bits, which of the two magnitudes.  The dot
// product of two such rows is an exact integer in units of the squared level step (1 bit: levels +-L, L = fp32 1/3,
// unit L^2; 2 bits: levels +-.25, +-.75, unit 1/16), computed with xor / and / popc on the SIMT pipe.  The pipeline
// (driven from w2b_eval.cu):
//   planes   eval_bits_planes_kernel: the file's rows -> a sign plane and a magnitude plane of uint32 words on a
//            16-byte row pitch (padding bits 0), popc of the magnitude plane, and the row's fp32 length summed in
//            the order eval_normalize_kernel uses (the reference's build order); eval_ctx_planes_kernel builds the
//            same planes from a training context's u + v (the evaluator on a context's own tables);
//   Gram     eval_bits_gram_kernel: G[w][c] = integer dot of distinct query word w and vocabulary word c, a chunk of
//            the vocabulary at a time;
//   combine  eval_bits_combine_kernel: approx(q, c) = (G[w2][c]/len2 - G[w1][c]/len1 + G[w3][c]/len3) unit / len_c, the
//            FILTER: running best per question and a candidate list, the scheme of eval_tc_kernel's epilogue;
//   re-score eval_bits_rescore_kernel: candidates within 2 eps of the final best in fp32 in the reference's order,
//            rows decoded from the planes on the fly.
// eps (eval_bits_qeps_kernel) only has to cover fp32 rounding: the integers are exact.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "w2b_eval_tc.cuh"
#include "w2b_quant.cuh"

namespace w2b {
namespace bits {

// the float32 levels w2b_read_packed restores: sign bit n, magnitude bit h
template <int BITS> __device__ __forceinline__ float level(unsigned n, unsigned h) {
  const float m = (BITS == 1) ? 0.33333334f : (h ? 0.75f : 0.25f);
  return n ? -m : m;
}
// G counts in units of unit<BITS>() (a real number; 1 bit: the square of the fp32 level, not 1/9)
template <int BITS> __host__ __device__ __forceinline__ double unit() {
  return BITS == 1 ? (double)0.33333334f * (double)0.33333334f : 0.0625;
}
// bits 0, 2, 4, ..., 62 of x, compacted into 32 bits
__device__ __forceinline__ unsigned even_bits(unsigned long long x) {
  x &= 0x5555555555555555ull;
  x = (x | (x >> 1)) & 0x3333333333333333ull;
  x = (x | (x >> 2)) & 0x0f0f0f0f0f0f0f0full;
  x = (x | (x >> 4)) & 0x00ff00ff00ff00ffull;
  x = (x | (x >> 8)) & 0x0000ffff0000ffffull;
  x = (x | (x >> 16)) & 0x00000000ffffffffull;
  return (unsigned)x;
}

// What both plane kernels derive from a row's plane words, which they feed in order k = 0, 1, ...: popc of the
// magnitude plane and the row's fp32 length, every value's square added in index order as every lane of
// eval_normalize_kernel does (the squares of the first 4*floor(D/4) values rounded on their own and added one at a
// time, the last D mod 4 fused).  The two kernels differ only in where the bits come from.
template <int BITS> struct RowLength {
  float s = 0.f;
  int ph = 0;
  __device__ __forceinline__ void add(unsigned n, unsigned h, int k, int D) {
    const int valid = min(32, max(0, D - 32 * k)), D4 = D & ~3;
    ph += __popc(h);
    for (int j = 0; j < valid; ++j) {
      const float q = level<BITS>((n >> j) & 1u, (h >> j) & 1u);
      s = (32 * k + j < D4) ? __fadd_rn(s, __fmul_rn(q, q)) : __fmaf_rn(q, q, s);
    }
  }
  __device__ __forceinline__ void store(long long row, float *len, float *ilen, int *hpop) const {
    const float l = __fsqrt_rn(s);
    len[row] = l;
    ilen[row] = (float)(1.0 / (double)l);  // one rounding of the exact reciprocal
    hpop[row] = ph;
  }
};

// One warp per row.  Every lane assembles plane word k from the row's bytes (the same addresses in all lanes: one
// broadcast load each) and adds the 32 squares in index order (RowLength).
// rows are nbytes apart (the file's row, no alignment); Wp = plane words per row, a multiple of 4.
template <int BITS>
__global__ void eval_bits_planes_kernel(const uint8_t *rows, long long V, int D, long long nbytes, int Wp, unsigned *sign,
                                        unsigned *mag, float *len, float *ilen, int *hpop) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= V) return;
  const uint8_t *r = rows + row * nbytes;
  RowLength<BITS> rl;
  for (int k = 0; k < Wp; ++k) {
    unsigned long long raw = 0;
    const long long b0 = (long long)k * 4 * BITS;
#pragma unroll
    for (int i = 0; i < 4 * BITS; ++i)
      if (b0 + i < nbytes) raw |= (unsigned long long)r[b0 + i] << (8 * i);
    const int valid = min(32, max(0, D - 32 * k));
    const unsigned mask = valid == 32 ? 0xffffffffu : ((1u << valid) - 1u);
    const unsigned n = (BITS == 1 ? (unsigned)raw : even_bits(raw)) & mask;
    const unsigned h = (BITS == 1) ? 0u : (even_bits(raw >> 1) & mask);
    if (lane == 0) {
      sign[row * Wp + k] = n;
      if (BITS == 2) mag[row * Wp + k] = h;
    }
    rl.add(n, h, k, D);
  }
  if (lane == 0) rl.store(row, len, ilen, hpop);
}

// The same planes straight from a training context's tables: value a of row `row` is quantize(u + v) exactly as
// export_kernel forms it (the row w2b_export returns), and its codes are the ones w2b_write_packed writes for that
// value (sign: < 0; magnitude: |x| > 0.5).  Lane l reads column 32 k + l of u and v (rows `pitch` floats apart,
// padding columns not read) and the warp's ballots are plane word k, padding bits 0: bit for bit what
// eval_bits_planes_kernel derives from the packed file of w2b_export's output.
template <int BITS>
__global__ void eval_ctx_planes_kernel(const float *u, const float *v, long long pitch, long long V, int D, int Wp,
                                       unsigned *sign, unsigned *mag, float *len, float *ilen, int *hpop) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= V) return;  // (the whole warp: the ballots below see every lane)
  QParams qp;
  qp.bits = BITS;
  qp.seg = 1.f;
  const float *ur = u + row * pitch, *vr = v + row * pitch;
  RowLength<BITS> rl;
  for (int k = 0; k < Wp; ++k) {
    const int a = 32 * k + lane;
    bool neg = false, big = false;
    if (a < D) {
      const float x = quant<9>(__fadd_rn(ur[a], vr[a]), qp);
      neg = x < 0.f;
      big = fabsf(x) > 0.5f;
    }
    const unsigned n = __ballot_sync(kFull, neg);
    const unsigned h = (BITS == 2) ? __ballot_sync(kFull, big) : 0u;
    if (lane == 0) {
      sign[row * Wp + k] = n;
      if (BITS == 2) mag[row * Wp + k] = h;
    }
    rl.add(n, h, k, D);
  }
  if (lane == 0) rl.store(row, len, ilen, hpop);
}

// G[w * ldg + (c - c0)] for w in [0, W), c in [c0, c0 + nc): the exact integer dot of rows qid[w] and c.
//   1 bit: D - 2 popc(x), x = n_w ^ n_c (positions whose signs differ)
//   2 bits: every position weighs (1 + 2 h_w)(1 + 2 h_c) = 1 + 2 h_w + 2 h_c + 4 h_w h_c and counts + where the signs
//           agree: A - 2B, A = D + 2 popc(h_w) + 2 popc(h_c) + 4 popc(h_w & h_c),
//           B = popc(x) + 2 popc(x & h_w) + 2 popc(x & h_c) + 4 popc(x & h_w & h_c).
// Tiled like a GEMM: 64 query rows x 64 vocabulary rows per CTA, 8 plane words (256 values) per stage read with
// 16-byte loads into shared memory (word-major, so the 4 rows a thread needs are one 16-byte read), 4 x 4 integer
// accumulators per thread.  Padding words are 0 in every plane and add nothing.
constexpr int GT = 64, GK = 8;
template <int BITS>
__global__ void __launch_bounds__(256) eval_bits_gram_kernel(const unsigned *sign, const unsigned *mag, const int *hpop,
                                                             const int *qid, int W, long long c0, int nc, int D, int Wp,
                                                             int *G, long long ldg) {
  __shared__ __align__(16) unsigned sP[2 * BITS][GK][GT];  // [operand]: sign planes, [2 + operand]: magnitude planes
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int w0 = blockIdx.y * GT, t0 = blockIdx.x * GT;
  // loader role: operand (0 = query rows, 1 = vocabulary rows), row of the tile, which 4 of the stage's 8 words
  const int op = tid >> 7, lr = (tid & 127) >> 1, half = tid & 1;
  long long src = -1;
  if (op == 0 && w0 + lr < W) src = qid[w0 + lr];
  if (op == 1 && t0 + lr < nc) src = c0 + t0 + lr;
  int acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0;
  for (int k0 = 0; k0 < Wp; k0 += GK) {
    const int kw = k0 + 4 * half;
    uint4 vn = make_uint4(0, 0, 0, 0), vh = vn;
    if (src >= 0 && kw < Wp) {
      vn = *reinterpret_cast<const uint4 *>(sign + src * Wp + kw);
      if constexpr (BITS == 2) vh = *reinterpret_cast<const uint4 *>(mag + src * Wp + kw);
    }
    sP[op][4 * half + 0][lr] = vn.x; sP[op][4 * half + 1][lr] = vn.y;
    sP[op][4 * half + 2][lr] = vn.z; sP[op][4 * half + 3][lr] = vn.w;
    if constexpr (BITS == 2) {
      sP[2 + op][4 * half + 0][lr] = vh.x; sP[2 + op][4 * half + 1][lr] = vh.y;
      sP[2 + op][4 * half + 2][lr] = vh.z; sP[2 + op][4 * half + 3][lr] = vh.w;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GK; ++k) {
      const uint4 a4 = *reinterpret_cast<const uint4 *>(&sP[0][k][ty * 4]);
      const uint4 b4 = *reinterpret_cast<const uint4 *>(&sP[1][k][tx * 4]);
      const unsigned a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
      if constexpr (BITS == 1) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] += __popc(a[i] ^ b[j]);
      } else {
        const uint4 g4 = *reinterpret_cast<const uint4 *>(&sP[2][k][ty * 4]);
        const uint4 h4 = *reinterpret_cast<const uint4 *>(&sP[3][k][tx * 4]);
        const unsigned ah[4] = {g4.x, g4.y, g4.z, g4.w}, bh[4] = {h4.x, h4.y, h4.z, h4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const unsigned x = a[i] ^ b[j], hh = ah[i] & bh[j];
            // 4 popc(h_w & h_c) - 2 B of this word
            acc[i][j] += 4 * __popc(hh) - 2 * (__popc(x) + 2 * (__popc(x & ah[i]) + __popc(x & bh[j])) + 4 * __popc(x & hh));
          }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int w = w0 + ty * 4 + i;
    if (w >= W) continue;
    const int hw = (BITS == 2) ? hpop[qid[w]] : 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int t = t0 + tx * 4 + j;
      if (t >= nc) continue;
      G[w * ldg + t] = (BITS == 1) ? D - 2 * acc[i][j] : D + 2 * hw + 2 * hpop[c0 + t] + acc[i][j];
    }
  }
}

// Per question: qk[3q + i] = unit / len of its i-th query word (one rounding of the real quotient) and qeps[q], a
// bound on |approx - ref|: ref the score src/compute-accuracy.c computes in fp32 (m = level / len rounded,
// vec = (m2 - m1) + m3 rounded twice, D rounded products added one at a time), approx what eval_bits_combine_kernel
// computes.  Both approximate E = sum_a vec[a] m_c[a] taken in real arithmetic on the fp32 lengths, which is
// (G2 / len2 - G1 / len1 + G3 / len3) unit / len_c exactly.  With u = 2^-24, |m_i| = 1 up to (D + 2) u / 2 and
// sum_a |x[a] m_c[a]| <= |x| |m_c| (Cauchy-Schwarz), to first order in u:
//   ref:     the three m_i[a], the subtraction and the addition put u (|vec[a]| + 2 |m1[a]| + 2 |m2[a]| + |m3[a]|) on
//            vec[a]; m_c[a] and the product add 2 u |vec[a] m_c[a]|; the D - 1 rounded adds (D - 1) u sum |vec m_c|:
//                                                                           <= u ((D + 2) |vec| + 5)
//   approx:  the G are exact integers below 2^24 (9 D, D <= 2^17).  t1 = fl(G1 k1); s1 = fma(G2, k2, -t1);
//            s = fma(G3, k3, s1); approx = fl(s ilen_c): k_i, ilen_c one rounding each.  With e_i = m_i . m_c,
//            |e_i| <= 1: u (3 |e1| + 2 |e2| + |e3|) + 3 u |E|                   <= u (3 |vec| + 6)
//   eps = 1.05 u ((D + 5) |vec| + 11); the 5 % slack covers |vec| being computed here in fp32 and the
//   (1 + O(D u)) factors, D u < 1/100.  At D = 800, |vec| = 1.7: 8.6e-5.
// One warp per question; vec is built from the planes exactly as the reference builds it.
constexpr float kSlack = 1.05f;
template <int BITS>
__global__ void eval_bits_qeps_kernel(const unsigned *sign, const unsigned *mag, const float *len, const int *qid,
                                      const int *q3w, float *qk, float *qeps, long long nq, int D, int Wp) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  long long r[3];
  float l[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    r[i] = qid[q3w[q * 3 + i]];
    l[i] = len[r[i]];
  }
  double n2 = 0.0;
  for (int a = lane; a < D; a += 32) {
    float m[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const unsigned n = (sign[r[i] * Wp + (a >> 5)] >> (a & 31)) & 1u;
      const unsigned h = (BITS == 2) ? (mag[r[i] * Wp + (a >> 5)] >> (a & 31)) & 1u : 0u;
      m[i] = __fdiv_rn(level<BITS>(n, h), l[i]);
    }
    const float v = __fadd_rn(__fsub_rn(m[1], m[0]), m[2]);
    n2 += (double)v * (double)v;
  }
  for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(kFull, n2, o);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    if (lane == i) qk[q * 3 + i] = (float)(unit<BITS>() / (double)l[i]);
  if (lane == 0) qeps[q] = kSlack * 0x1p-24f * (((float)D + 5.f) * (float)sqrt(n2) + 11.f);
}

// The filter.  A warp takes one question and CT consecutive words of the chunk: 32 scores per lane from three rows
// of G (coalesced; the chunk of G was just written and is sized to stay in L2).  The best of the tile joins the
// question's running best before anything is appended, so a tile adds only what lies within 2 eps of its own best
// and of every tile seen before; the rule is eval_tc_kernel's: keep s > -2 eps (a word whose fp32 score is a little
// above 0 can have an approximate score <= 0) and s >= running best - 2 eps.  q3 = the question's three vocabulary
// ids (skipped as answers; -1 = none), q3w = their rows of G.
constexpr int CT = 1024, CPL = CT / 32;
__device__ __forceinline__ float combine(int g1, int g2, int g3, float k1, float k2, float k3, float ilen) {
  const float t1 = __fmul_rn((float)g1, k1);
  return __fmul_rn(__fmaf_rn((float)g3, k3, __fmaf_rn((float)g2, k2, -t1)), ilen);
}
__global__ void __launch_bounds__(256) eval_bits_combine_kernel(const int *G, long long ldg, long long c0, int nc,
                                                                const float *ilen, const int *q3, const int *q3w,
                                                                const float *qk, const float *qeps, unsigned *gmax,
                                                                tc::Candidate *cand, unsigned long long *n_cand,
                                                                unsigned long long cand_cap, int nq) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  const int t0 = blockIdx.y * CT;
  const int b1 = q3[q * 3], b2 = q3[q * 3 + 1], b3 = q3[q * 3 + 2];
  const int *g1 = G + q3w[q * 3] * ldg, *g2 = G + q3w[q * 3 + 1] * ldg, *g3 = G + q3w[q * 3 + 2] * ldg;
  const float k1 = qk[q * 3], k2 = qk[q * 3 + 1], k3 = qk[q * 3 + 2];
  const float eps2 = 2.f * qeps[q];
  float s[CPL];
  float best = 0.f;
#pragma unroll
  for (int i = 0; i < CPL; ++i) {
    const int t = t0 + 32 * i + lane;
    const long long c = c0 + t;
    s[i] = -INFINITY;  // not a competitor
    if (t < nc && c != b1 && c != b2 && c != b3) {
      s[i] = combine(g1[t], g2[t], g3[t], k1, k2, k3, ilen[c]);
      best = fmaxf(best, s[i]);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(kFull, best, o));
  const unsigned g = *(volatile unsigned *)(gmax + q);
  const float thr = fmaxf(g ? __uint_as_float(g & 0x7fffffffu) : 0.f, best) - eps2;
  if (lane == 0 && best > 0.f) atomicMax(gmax + q, tc::ordered(best));
#pragma unroll
  for (int i = 0; i < CPL; ++i)
    if (s[i] > -eps2 && s[i] >= thr) {
      const unsigned long long at = atomicAdd(n_cand, 1ull);
      if (at < cand_cap) cand[at] = tc::Candidate{q, (int)(c0 + t0 + 32 * i + lane), s[i]};
    }
}

// The same scores stored densely, for the top-k selection (w2b_eval_topk.cuh): S[q * ldS + t] = the filter's score
// of question q against word c0 + t, t < nc, every word (the selection skips the query words).
__global__ void __launch_bounds__(256) eval_bits_combine_store_kernel(const int *G, long long ldg, long long c0, int nc,
                                                                      const float *ilen, const int *q3w, const float *qk,
                                                                      float *S, long long ldS) {
  const int q = blockIdx.y, t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nc) return;
  const int w1 = q3w[q * 3], w2 = q3w[q * 3 + 1], w3 = q3w[q * 3 + 2];
  S[(long long)q * ldS + t] = combine(G[w1 * ldg + t], G[w2 * ldg + t], G[w3 * ldg + t], qk[q * 3], qk[q * 3 + 1],
                                      qk[q * 3 + 2], ilen[c0 + t]);
}

// dist of one packed candidate: r = its question's three rows and the candidate's row (see eval_bits_rescore_kernel)
template <int BITS>
__device__ __forceinline__ float exact_score(const unsigned *sign, const unsigned *mag, const float *len,
                                             const long long (&r)[4], int D, int Wp) {
  float lo[4], hi[4];  // the row's quotients for the small (or only) and the large magnitude
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float l = len[r[j]];
    lo[j] = __fdiv_rn(level<BITS>(0, 0), l);
    hi[j] = __fdiv_rn(level<BITS>(0, 1), l);
  }
  float acc = 0.f;
  for (int k = 0; k < Wp; ++k) {
    unsigned n[4], h[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      n[j] = sign[r[j] * Wp + k];
      h[j] = (BITS == 2) ? mag[r[j] * Wp + k] : 0u;
    }
    const int valid = min(32, D - 32 * k);
    for (int a = 0; a < valid; ++a) {
      float m[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = ((h[j] >> a) & 1u) ? hi[j] : lo[j];
        m[j] = ((n[j] >> a) & 1u) ? -v : v;
      }
      acc = __fadd_rn(acc, __fmul_rn(__fadd_rn(__fsub_rn(m[1], m[0]), m[2]), m[3]));
    }
  }
  return acc;
}

// Exact scores of the surviving candidates, the packed counterpart of eval_rescore_kernel: a candidate still within
// 2 eps of the question's final best is scored as src/compute-accuracy.c:155-165 does on the unpacked file,
// m = level / len (a row has one or two magnitudes: the quotients are taken once per row, the sign is exact),
// vec[a] = (m2[a] - m1[a]) + m3[a], dist += vec[a] * m_c[a] with the product rounded, then added, a ascending; and
// competes under the reference's rule: strictly positive, larger score wins, smaller index on ties.
template <int BITS>
__global__ void eval_bits_rescore_kernel(const unsigned *sign, const unsigned *mag, const float *len, const int *q3,
                                         const tc::Candidate *cand, unsigned long long n_cand, const float *qeps,
                                         const unsigned *gmax, unsigned long long *best, unsigned long long *n_rescored,
                                         int D, int Wp) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_cand) return;
  const tc::Candidate cd = cand[i];
  const unsigned g = gmax[cd.q];
  if (!(cd.s >= __uint_as_float(g & 0x7fffffffu) - 2.f * qeps[cd.q])) return;
  const long long r[4] = {q3[cd.q * 3], q3[cd.q * 3 + 1], q3[cd.q * 3 + 2], cd.c};
  const float acc = exact_score<BITS>(sign, mag, len, r, D, Wp);
  atomicAdd(n_rescored, 1ull);
  if (acc > 0.f)
    atomicMax(best + cd.q, ((unsigned long long)__float_as_uint(acc) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)cd.c));
}

// The planes back to the fp32 levels of the unpacked file, rows Dp floats apart (padding left as it is): the input of
// eval_normalize_kernel when every score is taken on the fp32 SIMT scorer.
template <int BITS>
__global__ void eval_bits_decode_kernel(const unsigned *sign, const unsigned *mag, float *M, long long V, int D, int Wp,
                                        long long Dp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V * D) return;
  const long long row = i / D;
  const int a = (int)(i % D);
  const unsigned n = (sign[row * Wp + (a >> 5)] >> (a & 31)) & 1u;
  const unsigned h = (BITS == 2) ? (mag[row * Wp + (a >> 5)] >> (a & 31)) & 1u : 0u;
  M[row * Dp + a] = level<BITS>(n, h);
}

}  // namespace bits
}  // namespace w2b
