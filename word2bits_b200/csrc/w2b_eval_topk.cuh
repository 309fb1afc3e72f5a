// Exact top-k lists of the analogy evaluator (w2b_analogy_topk, w2b_nearest) for sm_90a.
//
// The list of a query is the reference's top-N list at N = k (src/compute-accuracy.c:166-175): the k largest fp32
// scores that are > 0 over the words that are not query words, in descending order, the smaller index first on equal
// scores.  The pipeline (driven from w2b_eval.cu) runs over the vocabulary a chunk at a time:
//   producer  a dense chunk of scores, queries x chunk words: TF32 tensor-core scores (eval_tc_kernel<true>), bit-domain
//             scores of a packed file (eval_bits_combine_store_kernel), or exact fp32 scores (eval_score_kernel<true>);
//   select    topk_select_kernel: every query keeps the k largest keys it has seen (its kept set) and, from approximate
//             scores, appends the candidates of the chunk to its own slice of the candidate list;
//   re-score  topk_rescore_kernel / topk_bits_rescore_kernel: the candidates within 2 eps of the query's final k-th
//             best, scored in the reference's fp32 order;
//   order     topk_final_kernel: the k largest exact keys of each query, sorted, as ids and scores.
// Keys: approximate scores are ordered as floats (32-bit, tc::ordered); exact ones as (ordered score << 32 | ~index),
// so that a larger key is a larger score or, on equal scores, the smaller index.  0 is no key.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <type_traits>

#include "w2b_eval_bits.cuh"
#include "w2b_eval_tc.cuh"
#include "w2b_quant.cuh"

namespace w2b {

// dist of src/compute-accuracy.c:162-165 as the reference's build computes it: each product rounded, then added, in
// index order (vmulss, vaddss: never fused).
__device__ __forceinline__ float fp32_score(const float *v, const float *m, int D) {
  float acc = 0.f;
  for (int a = 0; a < D; ++a) acc = __fadd_rn(acc, __fmul_rn(v[a], m[a]));
  return acc;
}

namespace topk {

constexpr int KMAX = 1024;   // W2B_MAX_TOPK
constexpr int PEND = 2048;   // keys a block takes in before it merges them into its kept set
constexpr int THREADS = 256;

struct Cand { int c; float s; };  // slot of a query's candidate list: word and approximate score

__device__ __forceinline__ float unordered(unsigned u) {  // inverse of tc::ordered
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
__device__ __forceinline__ unsigned long long exact_key(float s, long long c) {
  return ((unsigned long long)tc::ordered(s) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)c);
}

template <class K> struct Smem {
  K buf[KMAX + PEND];  // [0, k): the kept set (0 = empty slot); [k, k + m): keys taken in since the last merge
  K nk[KMAX];          // the part of the new kept set above its k-th key, while it is assembled
  int hist[256];
  int cnt, digit, above, changed;
  K kth;               // the k-th largest key of the kept set (0 while it holds fewer than k keys)
};

// buf[0, n) (n >= k) -> its k largest keys in buf[0, k) as a multiset, and sm.kth = the k-th largest.  Radix select,
// 8 bits a pass from the top: the digit of the k-th largest is where the count of keys from the top reaches k.
template <class K> __device__ void merge(Smem<K> &sm, int k, int n) {
  const int tid = threadIdx.x;
  K prefix = 0, mask = 0;
  int r = k;  // rank, from the top, of the k-th largest among the keys that match prefix under mask
  for (int shift = 8 * (int)sizeof(K) - 8; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += THREADS) sm.hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < n; i += THREADS) {
      const K x = sm.buf[i];
      if ((x & mask) == prefix) atomicAdd(&sm.hist[(int)((x >> shift) & 255)], 1);
    }
    __syncthreads();
    if (tid < 32) {  // lane l holds digits 255 - 8l down to 248 - 8l
      int h[8], s = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        h[j] = sm.hist[255 - 8 * tid - j];
        s += h[j];
      }
      int inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(kFull, inc, o);
        if (tid >= o) inc += v;
      }
      int acc = inc - s;
      if (acc < r && r <= inc) {  // the one lane whose digits reach rank r
        for (int j = 0; j < 8; ++j) {
          if (acc + h[j] >= r) {
            sm.digit = 255 - 8 * tid - j;
            sm.above = acc;
            break;
          }
          acc += h[j];
        }
      }
    }
    __syncthreads();
    prefix |= (K)sm.digit << shift;
    mask |= (K)255 << shift;
    r -= sm.above;
    __syncthreads();
  }
  const K T = prefix;
  if (tid == 0) sm.cnt = 0;
  __syncthreads();
  for (int i = tid; i < n; i += THREADS) {
    const K x = sm.buf[i];
    if (x > T) sm.nk[atomicAdd(&sm.cnt, 1)] = x;  // fewer than k keys lie above the k-th largest
  }
  __syncthreads();
  const int g = sm.cnt;
  for (int i = tid; i < k; i += THREADS) sm.buf[i] = i < g ? sm.nk[i] : T;
  if (tid == 0) {
    sm.kth = T;
    sm.changed = 1;
  }
  __syncthreads();
}

// Takes the keys row(0), ..., row(n - 1) into the kept set: only keys above its k-th largest can enter it; they are
// gathered PEND at a time and merged.  Afterwards buf[0, k) is the k largest of the old set and the row.
template <class K, class Row> __device__ void absorb(Smem<K> &sm, int k, int n, Row row) {
  for (int base = 0; base < n; base += PEND) {
    if (threadIdx.x == 0) sm.cnt = 0;
    __syncthreads();
    const K kth = sm.kth;
    const int end = min(n, base + PEND);
    for (int i = base + threadIdx.x; i < end; i += THREADS) {
      const K x = row(i);
      if (x > kth) sm.buf[k + atomicAdd(&sm.cnt, 1)] = x;
    }
    __syncthreads();
    const int m = sm.cnt;
    if (m) merge(sm, k, k + m);
    __syncthreads();
  }
}

// The candidate selection, one block per query of a block of queries, one chunk of the vocabulary per launch:
// S[q * ldS + i] is the score of word c0 + i (i < nc), q3 the query's three words (not answers), kept[q * k ...] and
// kth[q] its kept set, carried from chunk to chunk.
// EXACT = false: S holds approximate scores A with |A - E| <= eps_q for the exact fp32 score E of every word (the
//   bound of eval_qeps_kernel / eval_bits_qeps_kernel).  The kept set holds the k largest A seen so far (32-bit keys),
//   so its k-th largest t_q is the running k-th best; it only rises.  Every word with A >= t_q - 2 eps_q and
//   A > -2 eps_q is appended to the query's candidate list (cand[q * cap ...], n_cand[q] counts on past cap: the
//   caller checks for overflow).  The candidates are a superset of the exact top-k: let a_k, e_k be the k-th largest
//   A and E over all eligible words.  |A - E| <= eps moves an order statistic by at most eps, so a_k <= e_k + eps;
//   a member w of the exact top-k has E_w >= e_k, hence A_w >= E_w - eps >= e_k - eps >= a_k - 2 eps; and a running
//   threshold is <= the final a_k, so A_w >= t_q - 2 eps held when w's chunk was read.  A member also has E_w > 0,
//   so A_w > -eps.  With fewer than k eligible words a_k does not exist and t_q stays -inf.
// EXACT = true: S holds exact fp32 scores, eps = 0, the keys are 64-bit (score, ~index) and only scores > 0 count:
//   after the last chunk the kept set is the exact top-k.  No candidates are appended.
template <bool EXACT>
__global__ void __launch_bounds__(THREADS)
topk_select_kernel(const float *S, long long ldS, long long c0, int nc, const int *q3, const float *qeps,
                   typename std::conditional<EXACT, unsigned long long, unsigned>::type *kept,
                   typename std::conditional<EXACT, unsigned long long, unsigned>::type *kth, Cand *cand, int *n_cand,
                   int cap, int k) {
  using K = typename std::conditional<EXACT, unsigned long long, unsigned>::type;
  __shared__ Smem<K> sm;
  const int q = blockIdx.x, tid = threadIdx.x;
  const float *srow = S + (long long)q * ldS;
  const long long b1 = q3[q * 3], b2 = q3[q * 3 + 1], b3 = q3[q * 3 + 2];
  K *kq = kept + (long long)q * k;
  for (int i = tid; i < k; i += THREADS) sm.buf[i] = kq[i];
  if (tid == 0) {
    sm.kth = kth[q];
    sm.changed = 0;
  }
  __syncthreads();
  absorb(sm, k, nc, [&](int i) -> K {
    const long long c = c0 + i;
    const float s = srow[i];
    if (c == b1 || c == b2 || c == b3 || !(s == s)) return 0;  // a zero row normalises to NaN: never an answer
    if constexpr (EXACT) return s > 0.f ? exact_key(s, c) : 0ull;
    else return tc::ordered(s);
  });
  if (sm.changed) {
    for (int i = tid; i < k; i += THREADS) kq[i] = sm.buf[i];
    if (tid == 0) kth[q] = sm.kth;
  }
  if constexpr (!EXACT) {
    const float eps2 = 2.f * qeps[q];
    const float t = sm.kth ? unordered(sm.kth) : -INFINITY;
    for (int i = tid; i < nc; i += THREADS) {
      const long long c = c0 + i;
      const float s = srow[i];
      if (c != b1 && c != b2 && c != b3 && s > -eps2 && s >= t - eps2) {
        const int at = atomicAdd(n_cand + q, 1);
        if (at < cap) cand[(long long)q * cap + at] = Cand{(int)c, s};
      }
    }
  }
}

// Which candidates are re-scored: those still within 2 eps of the query's final k-th best approximate score.
__device__ __forceinline__ bool survives(const Cand &cd, unsigned kth, float eps) {
  return cd.s >= (kth ? unordered(kth) : -INFINITY) - 2.f * eps;
}

// Exact scores of the surviving candidates (thread per slot of the candidate lists, cap slots a query): the
// arithmetic of eval_rescore_kernel, written as a key (0: not re-scored, or not > 0) instead of taking a maximum.
__global__ void topk_rescore_kernel(const float *Q, const float *M, const Cand *cand, const int *n_cand, int cap,
                                    const unsigned *kth, const float *qeps, unsigned long long *keys,
                                    unsigned long long *n_rescored, long long nq, int D, long long Dp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long q = i / cap;
  if (q >= nq || i % cap >= min(n_cand[q], cap)) return;
  const Cand cd = cand[i];
  unsigned long long key = 0;
  if (survives(cd, kth[q], qeps[q])) {
    const float acc = fp32_score(Q + q * Dp, M + (long long)cd.c * Dp, D);
    atomicAdd(n_rescored, 1ull);
    if (acc > 0.f) key = exact_key(acc, cd.c);
  }
  keys[i] = key;
}

// The packed counterpart: the arithmetic of eval_bits_rescore_kernel (rows decoded from the planes on the fly).
template <int BITS>
__global__ void topk_bits_rescore_kernel(const unsigned *sign, const unsigned *mag, const float *len, const int *q3,
                                         const Cand *cand, const int *n_cand, int cap, const unsigned *kth,
                                         const float *qeps, unsigned long long *keys, unsigned long long *n_rescored,
                                         long long nq, int D, int Wp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long q = i / cap;
  if (q >= nq || i % cap >= min(n_cand[q], cap)) return;
  const Cand cd = cand[i];
  unsigned long long key = 0;
  if (survives(cd, kth[q], qeps[q])) {
    const long long r[4] = {q3[q * 3], q3[q * 3 + 1], q3[q * 3 + 2], cd.c};
    const float acc = bits::exact_score<BITS>(sign, mag, len, r, D, Wp);
    atomicAdd(n_rescored, 1ull);
    if (acc > 0.f) key = exact_key(acc, cd.c);
  }
  keys[i] = key;
}

// One block per query: the k largest of its exact keys keys[q * ld + i], i < n_keys[q] (all ld when n_keys is NULL),
// sorted descending (bitonic sort in shared memory) -> ids[q * k + j] (-1 past the end of the list), scores.
__global__ void __launch_bounds__(THREADS)
topk_final_kernel(const unsigned long long *keys, const int *n_keys, long long ld, int k, int *ids, float *scores) {
  __shared__ Smem<unsigned long long> sm;
  const int q = blockIdx.x, tid = threadIdx.x;
  int N = 1;
  while (N < k) N <<= 1;
  for (int i = tid; i < N; i += THREADS) sm.buf[i] = 0;
  if (tid == 0) sm.kth = 0;
  __syncthreads();
  const unsigned long long *row = keys + q * ld;
  const int n = n_keys ? (int)min((long long)n_keys[q], ld) : (int)ld;
  absorb(sm, k, n, [&](int i) { return row[i]; });
  for (int i = k + tid; i < N; i += THREADS) sm.buf[i] = 0;
  __syncthreads();
  for (int size = 2; size <= N; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < N; i += THREADS) {
        const int j = i ^ stride;
        if (j > i) {
          const unsigned long long a = sm.buf[i], b = sm.buf[j];
          if (((i & size) == 0) ? a < b : a > b) {
            sm.buf[i] = b;
            sm.buf[j] = a;
          }
        }
      }
      __syncthreads();
    }
  for (int j = tid; j < k; j += THREADS) {
    const unsigned long long x = sm.buf[j];
    ids[(long long)q * k + j] = x ? (int)(0xFFFFFFFFu - (unsigned)(x & 0xFFFFFFFFull)) : -1;
    scores[(long long)q * k + j] = x ? unordered((unsigned)(x >> 32)) : 0.f;
  }
}

}  // namespace topk
}  // namespace w2b
