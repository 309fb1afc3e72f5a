// Analogy evaluator on the GPU (SURVEY section 8(f).2) — the "next" row after the training path.
// Replaces src/compute-accuracy.c:63-189: load word2vec-binary vectors, optional re-quantize,
// L2-normalise (:96-111), and for every question a:b :: c:? take vec = (M[b] - M[a]) + M[c]
// (:155) and the arg-max cosine over the whole vocabulary except the three query words
// (:158-177), first index winning ties and only strictly positive scores counting (bestd
// starts at 0, :150).  Here all questions are scored together as one Q x V x D contraction
// on the tensor cores (w2b_eval_tc.cuh: TF32 wgmma fed by TMA, accumulators in registers) used as a FILTER
// with a proven error bound, followed by an fp32 re-score of the surviving candidates in the operation order of the
// reference's build (gcc -O3 -march=x86-64-v3, oracle/Makefile) — so the arg-max is the reference's arg-max; the
// report text is the reference's, line for line.
#include <cuda_runtime.h>
#include <ctype.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <unordered_map>
#include <vector>

#include "w2b.h"
#include "w2b_internal.h"
#include "w2b_quant.cuh"
#include "w2b_eval_tc.cuh"

using namespace w2b;

#define CKE(call)                                                                         \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      w2b_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return W2B_ECUDA;                                                                   \
    }                                                                                     \
  } while (0)

namespace {

// device buffers / events released on every return path
struct DevBuf {
  void *p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
  template <class T> T *as() const { return static_cast<T *>(p); }
};
struct DevEvent {
  cudaEvent_t e = nullptr;
  ~DevEvent() { if (e) cudaEventDestroy(e); }
};
struct FileCloser {
  FILE *f;
  ~FileCloser() { if (f && f != stdin) fclose(f); }
};

// quantize (:106) + L2 normalise (:107-110): one warp per row.  len is summed in the order of the reference's build:
// the squares of the first 4*floor(D/4) values are rounded on their own (vmulps) and added one at a time in index
// order (vaddss); the last D mod 4 terms are fused (vfmadd231ss).  The lanes quantize and square 32 values at once;
// every lane then adds the 32 in order (the same value in every lane, no reduction tree).
__global__ void eval_normalize_kernel(float *M, long long words, long long D, long long Dp, int bits) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= words) return;
  QParams qp;
  qp.bits = bits;
  qp.seg = (bits >= 4) ? exp2f((float)(bits - 1)) : 1.f;
  float *r = M + row * Dp;  // rows are padded to Dp floats (zeros) for the tensor-core pass
  const long long D4 = D & ~3LL;
  float s = 0.f;
  for (long long a0 = 0; a0 < D; a0 += 32) {
    const long long a = a0 + lane;
    float q = 0.f;
    if (a < D) {
      q = quant<9>(r[a], qp);
      r[a] = q;
    }
    const float p = __fmul_rn(q, q);
    const int n = (int)min(32LL, D - a0);
    for (int j = 0; j < n; ++j) {
      const float pj = __shfl_sync(kFull, p, j), qj = __shfl_sync(kFull, q, j);
      s = (a0 + j < D4) ? __fadd_rn(s, pj) : __fmaf_rn(qj, qj, s);
    }
  }
  const float len = __fsqrt_rn(s);
  for (long long a = lane; a < D; a += 32) r[a] = __fdiv_rn(r[a], len);
}

// vec = (M[b2] - M[b1]) + M[b3] (:155), rows padded to a multiple of 64 with zeros.
__global__ void eval_query_kernel(const float *M, const int *q3, float *Q, long long nq, long long D, long long Dp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq * D) return;
  const long long q = i / D, a = i % D;
  const long long b1 = q3[q * 3], b2 = q3[q * 3 + 1], b3 = q3[q * 3 + 2];
  Q[q * Dp + a] = __fadd_rn(__fsub_rn(M[b2 * Dp + a], M[b1 * Dp + a]), M[b3 * Dp + a]);
}

// eps of the tensor-core filter per question, a bound on |approx - ref| where ref is the score in the reference's fp32
// order and approx the tensor core's.  With u = 2^-24 and sum|v_a m_a| <= |vec| |m| (Cauchy-Schwarz), |m| = 1:
//   operands: TF32 keeps 10 explicit mantissa bits of each (the rest is dropped), so a product is off by at most
//             (1 + 2^-10)^2 - 1 < 2^-9 (1 + 2^-11) relative:                    <= 2^-9 (1 + 2^-11) |vec|
//   tensor-core sum of Dp products: its fp32 accumulation is not specified; taken as truncating (unit 2u), Dp adds:
//                                                                               <= 2 Dp u |vec| (1 + O(Dp u))
//   reference sum: each product rounded once, then D rounded adds:              <= (D + 1) u |vec| (1 + O(D u))
//   |m| and the |vec| computed here in fp32 are each within (D + 2) u of the true lengths; covered by one more
//   Dp u term, and the (1 + O(Dp u)) factors by the 5 % slack for Dp u < 1/100 (Dp < 1.6e5; the reference's own
//   limit is D <= 2000):
//   eps = 1.05 |vec| (2^-9 (1 + 2^-11) + (4 Dp + 1) u).  At D = 800 the sum terms are 1.7e-4, at D = 2000 4.9e-4.
__global__ void eval_qeps_kernel(const float *Q, float *qeps, long long nq, long long Dp) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= nq) return;
  float n2 = 0.f;
  for (long long a = lane; a < Dp; a += 32) {
    const float x = Q[q * Dp + a];
    n2 = fmaf(x, x, n2);
  }
  for (int o = 16; o > 0; o >>= 1) n2 += __shfl_xor_sync(kFull, n2, o);
  if (lane == 0) qeps[q] = (0.001953125f * (1.f + 0x1p-11f) + (4.f * (float)Dp + 1.f) * 0x1p-24f) * 1.05f * sqrtf(n2);
}

// Pass 2: exact scores of the surviving candidates.  Thread per candidate: one whose approximate score is still
// within 2*eps of the question's FINAL best is scored in fp32 exactly like the reference's build runs :162-165 —
// dist = sum over a ascending of vec[a] * M[a + c*size], each product rounded, then added (vmulss, vaddss: never
// fused), the order the fp32 SIMT scorer uses — and competes for best[q] with the reference's rule: strictly positive, larger score wins, smaller index on ties.
__global__ void eval_rescore_kernel(const float *Q, const float *M, const tc::Candidate *cand, unsigned long long n_cand,
                                    const float *qeps, const unsigned *gmax, unsigned long long *best,
                                    unsigned long long *n_rescored, int D, long long Dp) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_cand) return;
  const tc::Candidate cd = cand[i];
  const unsigned g = gmax[cd.q];
  if (!(cd.s >= __uint_as_float(g & 0x7fffffffu) - 2.f * qeps[cd.q])) return;
  const float *v = Q + (size_t)cd.q * Dp, *m = M + (size_t)cd.c * Dp;
  float acc = 0.f;
  for (int a = 0; a < D; ++a) acc = __fadd_rn(acc, __fmul_rn(v[a], m[a]));
  atomicAdd(n_rescored, 1ull);
  if (acc > 0.f)
    atomicMax(best + cd.q, ((unsigned long long)__float_as_uint(acc) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)cd.c));
}

// Parity hook (W2B_EVAL_SIMT=1) and fall-back for pathological inputs: every score in fp32 on the SIMT cores, same
// operation order per (question, word) as the re-score pass — tests hold the tensor-core pipeline to an identical
// report against it.  scores = Q (nq x D) . M^T (D x words), 64 x 64 tile per CTA, 4 x 4 per thread, fused arg-max:
// best[q] = max over c not in {b1,b2,b3} with score > 0 of (score, smallest c).
constexpr int TM = 64, TN = 64, TK = 16;
__global__ void __launch_bounds__(256) eval_score_kernel(const float *Q, const float *M, const int *q3,
                                                         unsigned long long *best, long long nq, long long words,
                                                         long long D, long long Dp) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Bs[TK][TN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 threads, each 4 x 4 outputs
  const long long q0 = (long long)blockIdx.y * TM, c0 = (long long)blockIdx.x * TN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long long k0 = 0; k0 < D; k0 += TK) {
    // 64 rows x 16 k per operand = 1024 floats, 4 per thread
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const int e = tid + l * 256;
      const int r = e >> 4, k = e & 15;
      const long long qa = q0 + r, ca = c0 + r, ka = k0 + k;
      As[k][r] = (qa < nq && ka < D) ? Q[qa * Dp + ka] : 0.f;
      Bs[k][r] = (ca < words && ka < D) ? M[ca * Dp + ka] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = __fadd_rn(acc[i][j], __fmul_rn(a[i], b[j]));
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long q = q0 + ty * 4 + i;
    const bool qok = q < nq;  // no early exit: the shuffles below need the whole warp
    const int b1 = qok ? q3[q * 3] : -1, b2 = qok ? q3[q * 3 + 1] : -1, b3 = qok ? q3[q * 3 + 2] : -1;
    unsigned long long key = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long c = c0 + tx * 4 + j;
      const float s = acc[i][j];
      if (qok && c < words && c != b1 && c != b2 && c != b3 && s > 0.f) {
        const unsigned long long k2 =
            ((unsigned long long)__float_as_uint(s) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)c);
        key = k2 > key ? k2 : key;
      }
    }
    // combine the 16 threads of this row (same ty): lanes tx = 0..15 are contiguous in a half warp
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(kFull, key, o);
      key = other > key ? other : key;
    }
    if (tx == 0 && key && qok) atomicMax(best + q, key);
  }
}

std::string upper(std::string s) {
  for (auto &ch : s) ch = (char)toupper((unsigned char)ch);
  return s;
}

}  // namespace

// Reads the word2vec-binary file exactly like :85-111 (names up to the first ' ', '\n' skipped,
// upper-cased; D raw float32 per word).
static int read_vectors(const char *path, long long threshold, std::vector<std::string> &names,
                        std::vector<float> &M, long long &words, long long &size) {
  FILE *f = fopen(path, "rb");
  if (!f) {
    w2b_set_error("Input file not found");
    return W2B_EIO;
  }
  FileCloser closer{f};
  if (fscanf(f, "%lld", &words) != 1) { w2b_set_error("bad header"); return W2B_EIO; }
  if (threshold > 0 && words > threshold) words = threshold;
  if (fscanf(f, "%lld", &size) != 1) { w2b_set_error("bad header"); return W2B_EIO; }
  // (the reference mallocs words * size floats unchecked; a header this library cannot hold is an error, not a crash)
  if (words < 1 || size < 1 || words > 0x7fffffffLL || size > (1LL << 20) || words > (1LL << 40) / size) {
    w2b_set_error("bad header: %lld words of size %lld", words, size);
    return W2B_EIO;
  }
  names.resize(words);
  M.resize((size_t)words * size);
  for (long long b = 0; b < words; ++b) {
    std::string w;
    for (;;) {
      const int ch = fgetc(f);
      if (ch == EOF || ch == ' ') break;
      if (ch != '\n' && w.size() < 50) w.push_back((char)ch);
    }
    names[b] = upper(w);
    if (fread(&M[(size_t)b * size], sizeof(float), size, f) != (size_t)size) {
      w2b_set_error("vector file truncated at word %lld", b);
      return W2B_EIO;
    }
  }
  return W2B_OK;
}

static int compute_accuracy_impl(const char *vectors_file, int bitlevel, int64_t threshold,
                                 const char *questions_file, int device, w2b_accuracy *acc, char *report,
                                 int64_t report_cap, int32_t *answers, int64_t answers_cap, int64_t *n_questions);
// nothing is thrown across the C ABI (std::bad_alloc on a huge vocabulary, ...)
template <class F> static int no_throw(const char *who, F &&f) {
  try {
    return f();
  } catch (const std::exception &ex) {
    w2b_set_error("%s: %s", who, ex.what());
    return W2B_EINVAL;
  } catch (...) {
    w2b_set_error("%s: unexpected exception", who);
    return W2B_EINVAL;
  }
}
extern "C" int w2b_compute_accuracy(const char *vectors_file, int bitlevel, int64_t threshold,
                                    const char *questions_file, int device, w2b_accuracy *acc, char *report,
                                    int64_t report_cap) {
  if (!vectors_file) { w2b_set_error("w2b_compute_accuracy: null vectors_file"); return W2B_EINVAL; }
  if (report && report_cap > 0) report[0] = 0;
  return no_throw("w2b_compute_accuracy", [&] {
    return compute_accuracy_impl(vectors_file, bitlevel, threshold, questions_file, device, acc, report, report_cap,
                                 nullptr, 0, nullptr);
  });
}
extern "C" int w2b_analogy_answers(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file,
                                   int device, int32_t *answers, int64_t answers_cap, int64_t *n_questions) {
  if (!vectors_file) { w2b_set_error("w2b_analogy_answers: null vectors_file"); return W2B_EINVAL; }
  return no_throw("w2b_analogy_answers", [&] {
    return compute_accuracy_impl(vectors_file, bitlevel, threshold, questions_file, device, nullptr, nullptr, 0, answers,
                                 answers_cap, n_questions);
  });
}

static int compute_accuracy_impl(const char *vectors_file, int bitlevel, int64_t threshold,
                                 const char *questions_file, int device, w2b_accuracy *acc, char *report,
                                 int64_t report_cap, int32_t *answers, int64_t answers_cap, int64_t *n_questions) {
  std::vector<std::string> names;
  std::vector<float> M;
  long long words = 0, size = 0;
  int rc = read_vectors(vectors_file, threshold, names, M, words, size);
  if (rc) return rc;
  std::unordered_map<std::string, int> first;  // the reference's linear strcmp scan = first match (:140-145)
  for (long long b = words - 1; b >= 0; --b) first[names[b]] = (int)b;
  auto find = [&](const std::string &s) -> long long {
    auto it = first.find(s);
    return it == first.end() ? words : it->second;
  };

  // ---- parse the question stream the way the scanf loop does (:113-147), resolving ids
  FILE *qf = questions_file ? fopen(questions_file, "rb") : stdin;
  if (!qf) { w2b_set_error("questions file not found"); return W2B_EIO; }
  std::vector<std::string> tok;
  {
    FileCloser closer{qf};
    char buf[2048];
    while (fscanf(qf, "%2000s", buf) == 1) tok.push_back(buf);
  }
  struct Ev { int kind; std::string name; long long b1, b2, b3; std::string st4; int qidx; };  // 0 = section, 1 = question
  std::vector<Ev> events;
  std::vector<int> q3;
  size_t t = 0;
  std::string st1;
  for (;;) {
    const bool eof = t >= tok.size();
    if (!eof) st1 = upper(tok[t++]);
    if (st1 == ":" || st1 == "EXIT" || eof) {
      Ev e{0, "", 0, 0, 0, "", -1};
      const bool eof2 = t >= tok.size();
      if (!eof2) e.name = tok[t++];
      e.b1 = eof2 ? 1 : 0;  // b1 = "stream ended here"
      events.push_back(e);
      if (eof2) break;
      continue;
    }
    std::string st2 = t < tok.size() ? upper(tok[t++]) : st1;
    std::string st3 = t < tok.size() ? upper(tok[t++]) : st2;
    std::string st4 = t < tok.size() ? upper(tok[t++]) : st3;
    Ev e{1, "", find(st1), find(st2), find(st3), st4, -1};
    if (e.b1 != words && e.b2 != words && e.b3 != words && find(st4) != words) {
      e.qidx = (int)(q3.size() / 3);
      q3.push_back((int)e.b1); q3.push_back((int)e.b2); q3.push_back((int)e.b3);
    }
    events.push_back(e);
  }
  const long long nq = (long long)q3.size() / 3;

  // ---- GPU: normalise, build queries, tensor-core candidate pass, exact re-score of the candidate tiles
  std::vector<unsigned long long> best(nq > 0 ? nq : 1, 0);
  float ms = 0.f;
  if (nq > 0) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device >= ndev) {
      w2b_set_error("no CUDA device %d: the evaluator has no CPU fallback", device);
      return W2B_ECUDA;
    }
    CKE(cudaSetDevice(device));
    const long long Dp = (size + tc::BK - 1) / tc::BK * tc::BK;  // row pitch: whole 128-byte k-blocks, zero padded
    const int ntiles = (int)((words + tc::BN - 1) / tc::BN);
    if (acc) acc->candidates = acc->rescored = 0;
    const char *dbg = getenv("W2B_EVAL_SIMT");  // parity hook: score everything with the fp32 SIMT kernel instead
    const bool simt = dbg && atoi(dbg) != 0;
    DevBuf bM, bQ, bq3, bbest, bgmax, bcand, bqeps, bcnt;
    const unsigned long long cand_cap = (unsigned long long)nq * 1024ull;  // measured: tens to hundreds per question
    CKE(bM.alloc((size_t)words * Dp * sizeof(float)));
    CKE(bQ.alloc((size_t)nq * Dp * sizeof(float)));
    CKE(bq3.alloc(q3.size() * sizeof(int)));
    CKE(bbest.alloc(nq * sizeof(unsigned long long)));
    CKE(bgmax.alloc(nq * sizeof(unsigned)));
    CKE(bqeps.alloc(nq * sizeof(float)));
    CKE(bcnt.alloc(2 * sizeof(unsigned long long)));
    if (!simt) CKE(bcand.alloc(cand_cap * sizeof(tc::Candidate)));
    float *dM = bM.as<float>(), *dQ = bQ.as<float>();
    int *dq3 = bq3.as<int>();
    unsigned long long *dbest = bbest.as<unsigned long long>(), *dcnt = bcnt.as<unsigned long long>();
    CKE(cudaMemset(dM, 0, (size_t)words * Dp * sizeof(float)));
    CKE(cudaMemset(dQ, 0, (size_t)nq * Dp * sizeof(float)));
    CKE(cudaMemcpy2D(dM, Dp * sizeof(float), M.data(), size * sizeof(float), size * sizeof(float), words, cudaMemcpyHostToDevice));
    CKE(cudaMemcpy(dq3, q3.data(), q3.size() * sizeof(int), cudaMemcpyHostToDevice));
    CKE(cudaMemset(dbest, 0, nq * sizeof(unsigned long long)));
    CKE(cudaMemset(bgmax.p, 0, nq * sizeof(unsigned)));
    CKE(cudaMemset(dcnt, 0, 2 * sizeof(unsigned long long)));
    DevEvent e0, e1;
    CKE(cudaEventCreate(&e0.e));
    CKE(cudaEventCreate(&e1.e));
    CKE(cudaEventRecord(e0.e));
    eval_normalize_kernel<<<(unsigned)((words + 7) / 8), 256>>>(dM, words, size, Dp, bitlevel);
    eval_query_kernel<<<(unsigned)((nq * size + 255) / 256), 256>>>(dM, dq3, dQ, nq, size, Dp);
    bool need_simt = simt;
    unsigned long long h_cnt[2] = {0, 0};
    if (!simt) {
      CUtensorMap mapQ, mapM;
      if (!tc::make_map(&mapQ, dQ, nq, Dp, tc::BM) || !tc::make_map(&mapM, dM, words, Dp, tc::BN)) {
        w2b_set_error("cuTensorMapEncodeTiled failed (driver too old for TMA?)");
        return W2B_ECUDA;
      }
      eval_qeps_kernel<<<(unsigned)((nq + 7) / 8), 256>>>(dQ, bqeps.as<float>(), nq, Dp);
      CKE(cudaFuncSetAttribute(tc::eval_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES));
      // x = question tile (fastest): the CTAs that share a 256-word tile of M run together, M streams from HBM once
      dim3 grid((unsigned)((nq + tc::BM - 1) / tc::BM), (unsigned)ntiles);
      tc::eval_tc_kernel<<<grid, tc::THREADS, tc::SMEM_BYTES>>>(mapQ, mapM, dq3, bqeps.as<float>(), bgmax.as<unsigned>(),
                                                               bcand.as<tc::Candidate>(), dcnt, cand_cap, (int)nq, (int)words,
                                                               (int)Dp);
      CKE(cudaGetLastError());
      CKE(cudaMemcpy(h_cnt, dcnt, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      if (h_cnt[0] > cand_cap) {
        need_simt = true;  // pathological input (e.g. all vectors equal): score everything in fp32 instead
      } else if (h_cnt[0]) {
        eval_rescore_kernel<<<(unsigned)((h_cnt[0] + 127) / 128), 128>>>(dQ, dM, bcand.as<tc::Candidate>(), h_cnt[0],
                                                                       bqeps.as<float>(), bgmax.as<unsigned>(), dbest, dcnt + 1,
                                                                       (int)size, Dp);
      }
    }
    if (need_simt) {
      CKE(cudaMemset(dbest, 0, nq * sizeof(unsigned long long)));
      dim3 grid((unsigned)((words + TN - 1) / TN), (unsigned)((nq + TM - 1) / TM));
      eval_score_kernel<<<grid, 256>>>(dQ, dM, dq3, dbest, nq, words, size, Dp);
    }
    CKE(cudaGetLastError());
    CKE(cudaEventRecord(e1.e));
    CKE(cudaMemcpy(best.data(), dbest, nq * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    CKE(cudaEventElapsedTime(&ms, e0.e, e1.e));
    if (acc && !simt) {
      CKE(cudaMemcpy(h_cnt, dcnt, sizeof h_cnt, cudaMemcpyDeviceToHost));
      acc->candidates = (int64_t)h_cnt[0];
      acc->rescored = (int64_t)h_cnt[1];
    }
  }

  // ---- replay the control flow of :113-187 to produce the same report
  std::string out = "Starting eval...\n";
  char line[512];
  int TCN = 0, CCN = 0, TACN = 0, CACN = 0, SECN = 0, SYCN = 0, SEAC = 0, SYAC = 0, QID = 0, TQ = 0, TQS = 0;
  for (const Ev &e : events) {
    if (e.kind == 0) {
      if (TCN == 0) TCN = 1;
      if (QID != 0) {
        snprintf(line, sizeof line, "ACCURACY TOP1: %.2f %%  (%d / %d)\n", CCN / (float)TCN * 100, CCN, TCN);
        out += line;
        snprintf(line, sizeof line,
                 "Total accuracy: %.2f %%   Semantic accuracy: %.2f %%   Syntactic accuracy: %.2f %% \n",
                 CACN / (float)TACN * 100, SEAC / (float)SECN * 100, SYAC / (float)SYCN * 100);
        out += line;
      }
      QID++;
      if (e.b1) break;  // stream ended
      out += e.name + ":\n";
      TCN = 0;
      CCN = 0;
      continue;
    }
    TQ++;
    const unsigned long long key = e.qidx >= 0 ? best[e.qidx] : 0;
    if (answers && TQ <= answers_cap) answers[TQ - 1] = key ? (int32_t)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull)) : -1;
    if (e.qidx < 0) continue;
    TQS++;
    std::string bestw;
    if (key) bestw = names[0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull)];
    if (e.st4 == bestw) {
      CCN++; CACN++;
      if (QID <= 5) SEAC++; else SYAC++;
    }
    if (QID <= 5) SECN++; else SYCN++;
    TCN++;
    TACN++;
  }
  snprintf(line, sizeof line, "Questions seen / total: %d %d   %.2f %% \n", TQS, TQ, TQS / (float)TQ * 100);
  out += line;
  if (n_questions) *n_questions = TQ;
  if (acc) {
    acc->questions_total = TQ; acc->questions_seen = TQS; acc->correct = CACN;
    acc->semantic_correct = SEAC; acc->semantic_seen = SECN; acc->syntactic_correct = SYAC; acc->syntactic_seen = SYCN;
    acc->gpu_ms = ms; acc->vocab = words; acc->size = size;
  }
  if (report && report_cap > 0) {
    strncpy(report, out.c_str(), (size_t)report_cap - 1);
    report[report_cap - 1] = 0;
  }
  return W2B_OK;
}

// Test hook: the tensor-core filter's approximate score of every (question, word) pair and its eps per question.
// Q (nq x D) and M (words x D) are used as given (no quantize, no normalisation: rows of M should have length <= 1
// for eps to bound the error).  eval_tc_kernel runs unchanged, with eps = +inf (so every pair is a candidate), no
// query words to skip and room for nq * words candidates; eps itself comes from eval_qeps_kernel.
extern "C" int w2b_eval_filter_scores(const float *Q, int64_t nq, const float *M, int64_t words, int64_t D, int device,
                                      float *approx, float *eps) {
  if (!Q || !M || !approx || nq < 1 || words < 1 || D < 1 || nq * words > (1LL << 31)) {
    w2b_set_error("w2b_eval_filter_scores: bad arguments");
    return W2B_EINVAL;
  }
  return no_throw("w2b_eval_filter_scores", [&]() -> int {
    CKE(cudaSetDevice(device));
    const long long Dp = (D + tc::BK - 1) / tc::BK * tc::BK;
    const unsigned long long cap = (unsigned long long)nq * (unsigned long long)words;
    DevBuf bM, bQ, bq3, bgmax, bcand, bqeps, binf, bcnt;
    CKE(bM.alloc((size_t)words * Dp * sizeof(float)));
    CKE(bQ.alloc((size_t)nq * Dp * sizeof(float)));
    CKE(bq3.alloc((size_t)nq * 3 * sizeof(int)));
    CKE(bgmax.alloc(nq * sizeof(unsigned)));
    CKE(bqeps.alloc(nq * sizeof(float)));
    CKE(binf.alloc(nq * sizeof(float)));
    CKE(bcnt.alloc(sizeof(unsigned long long)));
    CKE(bcand.alloc(cap * sizeof(tc::Candidate)));
    CKE(cudaMemset(bM.p, 0, (size_t)words * Dp * sizeof(float)));
    CKE(cudaMemset(bQ.p, 0, (size_t)nq * Dp * sizeof(float)));
    CKE(cudaMemcpy2D(bM.p, Dp * sizeof(float), M, D * sizeof(float), D * sizeof(float), words, cudaMemcpyHostToDevice));
    CKE(cudaMemcpy2D(bQ.p, Dp * sizeof(float), Q, D * sizeof(float), D * sizeof(float), nq, cudaMemcpyHostToDevice));
    CKE(cudaMemset(bq3.p, 0xff, (size_t)nq * 3 * sizeof(int)));  // -1: no query words
    CKE(cudaMemset(bgmax.p, 0, nq * sizeof(unsigned)));
    CKE(cudaMemset(bcnt.p, 0, sizeof(unsigned long long)));
    std::vector<float> inf((size_t)nq, INFINITY);
    CKE(cudaMemcpy(binf.p, inf.data(), nq * sizeof(float), cudaMemcpyHostToDevice));
    CUtensorMap mapQ, mapM;
    if (!tc::make_map(&mapQ, bQ.as<float>(), nq, Dp, tc::BM) || !tc::make_map(&mapM, bM.as<float>(), words, Dp, tc::BN)) {
      w2b_set_error("cuTensorMapEncodeTiled failed (driver too old for TMA?)");
      return W2B_ECUDA;
    }
    eval_qeps_kernel<<<(unsigned)((nq + 7) / 8), 256>>>(bQ.as<float>(), bqeps.as<float>(), nq, Dp);
    CKE(cudaFuncSetAttribute(tc::eval_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES));
    dim3 grid((unsigned)((nq + tc::BM - 1) / tc::BM), (unsigned)((words + tc::BN - 1) / tc::BN));
    tc::eval_tc_kernel<<<grid, tc::THREADS, tc::SMEM_BYTES>>>(mapQ, mapM, bq3.as<int>(), binf.as<float>(), bgmax.as<unsigned>(),
                                                             bcand.as<tc::Candidate>(), bcnt.as<unsigned long long>(), cap,
                                                             (int)nq, (int)words, (int)Dp);
    CKE(cudaGetLastError());
    unsigned long long n = 0;
    CKE(cudaMemcpy(&n, bcnt.p, sizeof n, cudaMemcpyDeviceToHost));
    if (n != cap) {
      w2b_set_error("w2b_eval_filter_scores: %llu of %llu pairs came through (NaN input?)", n, cap);
      return W2B_EINVAL;
    }
    std::vector<tc::Candidate> cand((size_t)n);
    CKE(cudaMemcpy(cand.data(), bcand.p, n * sizeof(tc::Candidate), cudaMemcpyDeviceToHost));
    for (const tc::Candidate &c : cand) approx[(size_t)c.q * words + c.c] = c.s;
    if (eps) CKE(cudaMemcpy(eps, bqeps.p, nq * sizeof(float), cudaMemcpyDeviceToHost));
    return W2B_OK;
  });
}
