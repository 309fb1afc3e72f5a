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
#include "w2b_eval_bits.cuh"
#include "w2b_eval_topk.cuh"

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
  ~DevBuf() { reset(); }
  void reset() {
    if (p) cudaFree(p);
    p = nullptr;
  }
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

// The fp32 table of a training context: row r of M (Dp floats apart, padding columns left as they are) =
// quantize(u + v) of row r with export_kernel's arithmetic, i.e. the row w2b_export returns and -binary 1 writes.
// One warp per row; u and v rows are `pitch` floats apart and their padding columns are not read.
__global__ void eval_ctx_table_kernel(const float *u, const float *v, long long pitch, float *M, long long words,
                                      long long D, long long Dp, int bits) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= words) return;
  QParams qp;
  qp.bits = bits;
  qp.seg = (bits >= 4) ? exp2f((float)(bits - 1)) : 1.f;
  for (long long a = lane; a < D; a += 32) M[row * Dp + a] = quant<9>(__fadd_rn(u[row * pitch + a], v[row * pitch + a]), qp);
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
  const float acc = fp32_score(Q + (size_t)cd.q * Dp, M + (size_t)cd.c * Dp, D);
  atomicAdd(n_rescored, 1ull);
  if (acc > 0.f)
    atomicMax(best + cd.q, ((unsigned long long)__float_as_uint(acc) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)cd.c));
}

// Parity hook (W2B_EVAL_SIMT=1) and fall-back for pathological inputs: every score in fp32 on the SIMT cores, same
// operation order per (question, word) as the re-score pass — tests hold the tensor-core pipeline to an identical
// report against it.  scores = Q (nq x D) . M^T (D x words), 64 x 64 tile per CTA, 4 x 4 per thread, fused arg-max:
// best[q] = max over c not in {b1,b2,b3} with score > 0 of (score, smallest c).
// STORE = true (the top-k lists' fall-back, w2b_eval_topk.cuh): every score is stored instead, S[q * ldS + c] for
// q < nq, c < words (Q and M then point at one block of queries and one chunk of the vocabulary); q3 and best unused.
constexpr int TM = 64, TN = 64, TK = 16;
template <bool STORE>
__global__ void __launch_bounds__(256) eval_score_kernel(const float *Q, const float *M, const int *q3,
                                                         unsigned long long *best, long long nq, long long words,
                                                         long long D, long long Dp, float *S, long long ldS) {
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
  if constexpr (STORE) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long q = q0 + ty * 4 + i;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long c = c0 + tx * 4 + j;
        if (q < nq && c < words) S[q * ldS + c] = acc[i][j];
      }
    }
  } else {
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
}

std::string upper(std::string s) {
  for (auto &ch : s) ch = (char)toupper((unsigned char)ch);
  return s;
}

// The table an evaluation reads, with the names of its rows: a binary or packed vector file read into host memory, a
// text vector file parsed on the device, or a training context's u and v, which stay on the device (the scoring behind
// it is the same for all).
struct Table {
  std::vector<std::string> names;
  long long words = 0, size = 0;
  std::vector<float> M;              // word2vec-binary file: words x size floats
  std::vector<uint8_t> rows;         // packed file: words packed rows
  DevBuf text;                       // text file: the fp32 table on the device (rows Dp floats apart, zero padded)
  int bits = 0;                      // 1 or 2: scored in the bit domain (a packed file, or the context's own levels)
  const w2b_ctx_tables *ctx = nullptr;
};

// The fp32 table on the device, rows Dp floats apart and zero padded: upload_fp32 before the timed kernels (a binary
// file's table is copied into bM; a text file's was parsed into place when the file was read), build_fp32 as the first
// of them (a context's table is formed from u and v).  *dM = the table.
int upload_fp32(const Table &t, DevBuf &bM, long long Dp, float **dM) {
  if (t.text.p) {
    *dM = t.text.as<float>();
    return W2B_OK;
  }
  CKE(bM.alloc((size_t)t.words * Dp * sizeof(float)));
  *dM = bM.as<float>();
  CKE(cudaMemset(*dM, 0, (size_t)t.words * Dp * sizeof(float)));
  if (!t.ctx)
    CKE(cudaMemcpy2D(*dM, Dp * sizeof(float), t.M.data(), t.size * sizeof(float), t.size * sizeof(float), t.words,
                     cudaMemcpyHostToDevice));
  return W2B_OK;
}
void build_fp32(const Table &t, float *dM, long long Dp) {
  if (t.ctx)
    eval_ctx_table_kernel<<<(unsigned)((t.words + 7) / 8), 256>>>(t.ctx->u, t.ctx->v, t.ctx->pitch, dM, t.words, t.size,
                                                                 Dp, t.ctx->bitlevel);
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

// The kind of a vector file (w2b_vector_file_info); a file that cannot be opened is left to its reader to report.
static int vector_kind(const char *path, int *bits) {
  int kind = W2B_VECTORS_BINARY;
  int64_t V, D;
  *bits = 0;
  if (w2b_vector_file_info(path, 0, &kind, &V, &D, bits)) kind = W2B_VECTORS_BINARY;
  return kind;
}

// A text vector file (w2b_text.cu): the first `threshold` rows (all when threshold <= 0) parsed on the device into
// t.text, names as read_vectors reads them.
static int read_text(const char *path, int64_t threshold, int device, Table &t) {
  int kind, bits;
  int64_t V, D;
  int rc = w2b_vector_file_info(path, threshold, &kind, &V, &D, &bits);
  if (rc) return rc;
  if (V < 1 || V > 0x7fffffffLL || D > (1LL << 20) || V > (1LL << 40) / D) {
    w2b_set_error("bad header: %lld words of size %lld", (long long)V, (long long)D);
    return W2B_EIO;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device < 0 || device >= ndev) {
    w2b_set_error("no CUDA device %d: the evaluator has no CPU fallback", device);
    return W2B_ECUDA;
  }
  CKE(cudaSetDevice(device));
  const long long Dp = (D + tc::BK - 1) / tc::BK * tc::BK;
  CKE(t.text.alloc((size_t)V * Dp * sizeof(float)));
  CKE(cudaMemset(t.text.p, 0, (size_t)V * Dp * sizeof(float)));
  std::vector<std::string> raw;
  if ((rc = w2b_text_parse(path, V, D, t.text.as<float>(), Dp, raw))) return rc;
  t.names.resize(V);
  for (int64_t b = 0; b < V; ++b) t.names[b] = upper(raw[b].substr(0, 50));
  t.words = V;
  t.size = D;
  return W2B_OK;
}

static int compute_accuracy_impl(const Table &t, int bitlevel, const char *questions_file, int device, w2b_accuracy *acc,
                                 char *report, int64_t report_cap, int32_t *answers, int64_t answers_cap,
                                 int64_t *n_questions);
// a word2vec-binary or text file's table, then the evaluation
static int compute_accuracy_file(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file,
                                 int device, w2b_accuracy *acc, char *report, int64_t report_cap, int32_t *answers,
                                 int64_t answers_cap, int64_t *n_questions) {
  Table t;
  int bits;
  const int rc = vector_kind(vectors_file, &bits) == W2B_VECTORS_TEXT
                     ? read_text(vectors_file, threshold, device, t)
                     : read_vectors(vectors_file, threshold, t.names, t.M, t.words, t.size);
  if (rc) return rc;
  return compute_accuracy_impl(t, bitlevel, questions_file, device, acc, report, report_cap, answers, answers_cap,
                               n_questions);
}
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
    return compute_accuracy_file(vectors_file, bitlevel, threshold, questions_file, device, acc, report, report_cap,
                                 nullptr, 0, nullptr);
  });
}
extern "C" int w2b_analogy_answers(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file,
                                   int device, int32_t *answers, int64_t answers_cap, int64_t *n_questions) {
  if (!vectors_file) { w2b_set_error("w2b_analogy_answers: null vectors_file"); return W2B_EINVAL; }
  return no_throw("w2b_analogy_answers", [&] {
    return compute_accuracy_file(vectors_file, bitlevel, threshold, questions_file, device, nullptr, nullptr, 0, answers,
                                 answers_cap, n_questions);
  });
}

// The question stream as the reference walks it: section headers and question lines in file order, and the three
// query word ids of every question all of whose four words are in the vocabulary.
struct Ev { int kind; std::string name; long long b1, b2, b3; std::string st4; int qidx; };  // 0 = section, 1 = question
struct Questions {
  std::vector<Ev> events;
  std::vector<int> q3;
};
static int parse_questions(const char *questions_file, const std::vector<std::string> &names, Questions &qs) {
  const long long words = (long long)names.size();
  std::vector<Ev> &events = qs.events;
  std::vector<int> &q3 = qs.q3;
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
  return W2B_OK;
}

// Replays the control flow of :113-187 over the chosen words (best[q] = score << 32 | ~index, 0 = none) to produce
// the reference's report, the per-question answers and the counters.
static void write_report(const Questions &qs, const std::vector<std::string> &names,
                         const std::vector<unsigned long long> &best, long long words, long long size, float ms,
                         w2b_accuracy *acc, char *report, int64_t report_cap, int32_t *answers, int64_t answers_cap,
                         int64_t *n_questions);

static int compute_accuracy_impl(const Table &t, int bitlevel, const char *questions_file, int device, w2b_accuracy *acc,
                                 char *report, int64_t report_cap, int32_t *answers, int64_t answers_cap,
                                 int64_t *n_questions) {
  const std::vector<std::string> &names = t.names;
  const long long words = t.words, size = t.size;
  Questions qs;
  int rc = parse_questions(questions_file, names, qs);
  if (rc) return rc;
  const std::vector<int> &q3 = qs.q3;
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
    CKE(bQ.alloc((size_t)nq * Dp * sizeof(float)));
    CKE(bq3.alloc(q3.size() * sizeof(int)));
    CKE(bbest.alloc(nq * sizeof(unsigned long long)));
    CKE(bgmax.alloc(nq * sizeof(unsigned)));
    CKE(bqeps.alloc(nq * sizeof(float)));
    CKE(bcnt.alloc(2 * sizeof(unsigned long long)));
    if (!simt) CKE(bcand.alloc(cand_cap * sizeof(tc::Candidate)));
    float *dM = nullptr, *dQ = bQ.as<float>();
    int *dq3 = bq3.as<int>();
    unsigned long long *dbest = bbest.as<unsigned long long>(), *dcnt = bcnt.as<unsigned long long>();
    if ((rc = upload_fp32(t, bM, Dp, &dM))) return rc;
    CKE(cudaMemset(dQ, 0, (size_t)nq * Dp * sizeof(float)));
    CKE(cudaMemcpy(dq3, q3.data(), q3.size() * sizeof(int), cudaMemcpyHostToDevice));
    CKE(cudaMemset(dbest, 0, nq * sizeof(unsigned long long)));
    CKE(cudaMemset(bgmax.p, 0, nq * sizeof(unsigned)));
    CKE(cudaMemset(dcnt, 0, 2 * sizeof(unsigned long long)));
    DevEvent e0, e1;
    CKE(cudaEventCreate(&e0.e));
    CKE(cudaEventCreate(&e1.e));
    CKE(cudaEventRecord(e0.e));
    build_fp32(t, dM, Dp);
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
      CKE(cudaFuncSetAttribute(tc::eval_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES));
      // x = question tile (fastest): the CTAs that share a 256-word tile of M run together, M streams from HBM once
      dim3 grid((unsigned)((nq + tc::BM - 1) / tc::BM), (unsigned)ntiles);
      tc::eval_tc_kernel<false><<<grid, tc::THREADS, tc::SMEM_BYTES>>>(mapQ, mapM, dq3, bqeps.as<float>(), bgmax.as<unsigned>(),
                                                               bcand.as<tc::Candidate>(), dcnt, cand_cap, (int)nq, (int)words,
                                                               (int)Dp, nullptr, 0);
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
      eval_score_kernel<false><<<grid, 256>>>(dQ, dM, dq3, dbest, nq, words, size, Dp, nullptr, 0);
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

  write_report(qs, names, best, words, size, ms, acc, report, report_cap, answers, answers_cap, n_questions);
  return W2B_OK;
}

static void write_report(const Questions &qs, const std::vector<std::string> &names,
                         const std::vector<unsigned long long> &best, long long words, long long size, float ms,
                         w2b_accuracy *acc, char *report, int64_t report_cap, int32_t *answers, int64_t answers_cap,
                         int64_t *n_questions) {
  std::string out = "Starting eval...\n";
  char line[512];
  int TCN = 0, CCN = 0, TACN = 0, CACN = 0, SECN = 0, SYCN = 0, SEAC = 0, SYAC = 0, QID = 0, TQ = 0, TQS = 0;
  for (const Ev &e : qs.events) {
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
    CKE(cudaFuncSetAttribute(tc::eval_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES));
    dim3 grid((unsigned)((nq + tc::BM - 1) / tc::BM), (unsigned)((words + tc::BN - 1) / tc::BN));
    tc::eval_tc_kernel<false><<<grid, tc::THREADS, tc::SMEM_BYTES>>>(mapQ, mapM, bq3.as<int>(), binf.as<float>(), bgmax.as<unsigned>(),
                                                             bcand.as<tc::Candidate>(), bcnt.as<unsigned long long>(), cap,
                                                             (int)nq, (int)words, (int)Dp, nullptr, 0);
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

// ------------------------------------------------------------------------------------------------------------------
// Packed vector files (w2b_write_packed / -binary 2): the table stays packed, scores are taken in the bit domain
// (w2b_eval_bits.cuh).  The file format chooses this path; W2B_EVAL_SIMT=1, and a candidate list that overflows
// (1-bit vectors at small D tie by the thousand), decode the planes to fp32 and run the fp32 SIMT scorer above.
namespace {

constexpr size_t kGramChunkBytes = 32u << 20;  // a chunk of G, written by the Gram kernel and read back by the filter

struct HostPin {  // page-locks a host range for the duration of its copy
  void *p = nullptr;
  ~HostPin() { if (p) cudaHostUnregister(p); }
};

struct BitsState {
  DevBuf rows, sign, mag, len, ilen, hpop, qid, q3, q3w, qk, qeps, gmax, cand, cnt, G;
  long long V = 0, nbytes = 0, nq = 0, chunk = 0;
  int D = 0, Wp = 0, W = 0;
  unsigned long long cand_cap = 0;
  const w2b_ctx_tables *ctx = nullptr;  // set: the planes come from the context's u + v (rows is then NULL)
};

// Device buffers of one run: rows = V packed rows nbytes apart (NULL: the planes come from st.ctx), qid = the W distinct
// query words, q3w = per question its three rows of G (indices into qid), q3 = per question the three vocabulary ids
// that cannot be its answer.
int bits_upload(BitsState &st, const uint8_t *rows, long long V, int D, int bits, const int *qid, int W, const int *q3w,
                const int *q3, long long nq, unsigned long long cand_cap) {
  st.V = V; st.D = D; st.W = W; st.nq = nq; st.cand_cap = cand_cap;
  st.nbytes = ((long long)D * bits + 7) / 8;
  st.Wp = ((D + 31) / 32 + 3) & ~3;
  const long long vround = (V + bits::CT - 1) / bits::CT * bits::CT;
  st.chunk = std::min<long long>(vround, std::max<long long>(bits::CT, (long long)(kGramChunkBytes / 4 / W) / bits::CT * bits::CT));
  if (rows) CKE(st.rows.alloc((size_t)V * st.nbytes));
  CKE(st.sign.alloc((size_t)V * st.Wp * 4));
  if (bits == 2) CKE(st.mag.alloc((size_t)V * st.Wp * 4));
  CKE(st.len.alloc(V * 4));
  CKE(st.ilen.alloc(V * 4));
  CKE(st.hpop.alloc(V * 4));
  CKE(st.qid.alloc((size_t)W * 4));
  CKE(st.q3.alloc((size_t)nq * 12));
  CKE(st.q3w.alloc((size_t)nq * 12));
  CKE(st.qk.alloc((size_t)nq * 12));
  CKE(st.qeps.alloc((size_t)nq * 4));
  CKE(st.gmax.alloc((size_t)nq * 4));
  CKE(st.cnt.alloc(2 * sizeof(unsigned long long)));
  CKE(st.cand.alloc(cand_cap * sizeof(tc::Candidate)));
  CKE(st.G.alloc((size_t)W * st.chunk * 4));
  if (rows) {
    HostPin pin;
    CKE(cudaHostRegister((void *)rows, (size_t)V * st.nbytes, cudaHostRegisterDefault));
    pin.p = (void *)rows;
    CKE(cudaMemcpy(st.rows.p, rows, (size_t)V * st.nbytes, cudaMemcpyHostToDevice));
  }
  CKE(cudaMemcpy(st.qid.p, qid, (size_t)W * 4, cudaMemcpyHostToDevice));
  CKE(cudaMemcpy(st.q3.p, q3, (size_t)nq * 12, cudaMemcpyHostToDevice));
  CKE(cudaMemcpy(st.q3w.p, q3w, (size_t)nq * 12, cudaMemcpyHostToDevice));
  CKE(cudaMemset(st.gmax.p, 0, (size_t)nq * 4));
  CKE(cudaMemset(st.cnt.p, 0, 2 * sizeof(unsigned long long)));
  return W2B_OK;
}

// planes + row lengths, then eps and the scale factors of every question
template <int BITS> int bits_planes(BitsState &st) {
  if (st.ctx)
    bits::eval_ctx_planes_kernel<BITS><<<(unsigned)((st.V + 7) / 8), 256>>>(
        st.ctx->u, st.ctx->v, st.ctx->pitch, st.V, st.D, st.Wp, st.sign.as<unsigned>(), st.mag.as<unsigned>(),
        st.len.as<float>(), st.ilen.as<float>(), st.hpop.as<int>());
  else
    bits::eval_bits_planes_kernel<BITS><<<(unsigned)((st.V + 7) / 8), 256>>>(
        st.rows.as<uint8_t>(), st.V, st.D, st.nbytes, st.Wp, st.sign.as<unsigned>(), st.mag.as<unsigned>(),
        st.len.as<float>(), st.ilen.as<float>(), st.hpop.as<int>());
  bits::eval_bits_qeps_kernel<BITS><<<(unsigned)((st.nq + 7) / 8), 256>>>(
      st.sign.as<unsigned>(), st.mag.as<unsigned>(), st.len.as<float>(), st.qid.as<int>(), st.q3w.as<int>(), st.qk.as<float>(),
      st.qeps.as<float>(), st.nq, st.D, st.Wp);
  CKE(cudaGetLastError());
  return W2B_OK;
}

// Gram + filter over the vocabulary, a chunk at a time; gram (host, W x V, may be NULL) receives every chunk of G.
template <int BITS> int bits_filter(BitsState &st, int32_t *gram) {
  for (long long c0 = 0; c0 < st.V; c0 += st.chunk) {
    const int nc = (int)std::min(st.chunk, st.V - c0);
    dim3 gg((unsigned)((nc + bits::GT - 1) / bits::GT), (unsigned)((st.W + bits::GT - 1) / bits::GT));
    bits::eval_bits_gram_kernel<BITS><<<gg, 256>>>(st.sign.as<unsigned>(), st.mag.as<unsigned>(), st.hpop.as<int>(),
                                                  st.qid.as<int>(), st.W, c0, nc, st.D, st.Wp, st.G.as<int>(), st.chunk);
    // x = questions (fastest): every question meets the chunk's first tile before any meets its second
    dim3 gc((unsigned)((st.nq + 7) / 8), (unsigned)((nc + bits::CT - 1) / bits::CT));
    bits::eval_bits_combine_kernel<<<gc, 256>>>(st.G.as<int>(), st.chunk, c0, nc, st.ilen.as<float>(), st.q3.as<int>(),
                                               st.q3w.as<int>(), st.qk.as<float>(), st.qeps.as<float>(), st.gmax.as<unsigned>(),
                                               st.cand.as<tc::Candidate>(), st.cnt.as<unsigned long long>(), st.cand_cap,
                                               (int)st.nq);
    CKE(cudaGetLastError());
    if (gram)
      CKE(cudaMemcpy2D(gram + c0, (size_t)st.V * 4, st.G.p, (size_t)st.chunk * 4, (size_t)nc * 4, st.W, cudaMemcpyDeviceToHost));
  }
  return W2B_OK;
}

// Every score on the fp32 SIMT scorer: the planes become the fp32 table of the unpacked file, and
// eval_normalize_kernel / eval_query_kernel / eval_score_kernel run as they do on a word2vec-binary file.
template <int BITS> int bits_fp32(BitsState &st, DevBuf &bM, DevBuf &bQ, long long Dp) {
  CKE(bM.alloc((size_t)st.V * Dp * sizeof(float)));
  CKE(bQ.alloc((size_t)st.nq * Dp * sizeof(float)));
  CKE(cudaMemset(bM.p, 0, (size_t)st.V * Dp * sizeof(float)));
  CKE(cudaMemset(bQ.p, 0, (size_t)st.nq * Dp * sizeof(float)));
  bits::eval_bits_decode_kernel<BITS><<<(unsigned)((st.V * st.D + 255) / 256), 256>>>(
      st.sign.as<unsigned>(), st.mag.as<unsigned>(), bM.as<float>(), st.V, st.D, st.Wp, Dp);
  eval_normalize_kernel<<<(unsigned)((st.V + 7) / 8), 256>>>(bM.as<float>(), st.V, st.D, Dp, BITS);
  eval_query_kernel<<<(unsigned)((st.nq * st.D + 255) / 256), 256>>>(bM.as<float>(), st.q3.as<int>(), bQ.as<float>(), st.nq, st.D, Dp);
  return W2B_OK;
}

template <int BITS> int bits_score_simt(BitsState &st, unsigned long long *dbest) {
  const long long Dp = (st.D + tc::BK - 1) / tc::BK * tc::BK;
  DevBuf bM, bQ;
  CKE(cudaMemset(dbest, 0, st.nq * sizeof(unsigned long long)));
  int rc = bits_fp32<BITS>(st, bM, bQ, Dp);
  if (rc) return rc;
  dim3 grid((unsigned)((st.V + TN - 1) / TN), (unsigned)((st.nq + TM - 1) / TM));
  eval_score_kernel<false><<<grid, 256>>>(bQ.as<float>(), bM.as<float>(), st.q3.as<int>(), dbest, st.nq, st.V, st.D, Dp, nullptr, 0);
  CKE(cudaGetLastError());
  CKE(cudaDeviceSynchronize());  // bM and bQ are freed on return
  return W2B_OK;
}

// best[q] of every question of a packed table; counts = {candidates, re-scored}
template <int BITS> int bits_answers(BitsState &st, bool simt, unsigned long long *dbest, unsigned long long counts[2]) {
  int rc = bits_planes<BITS>(st);
  if (rc) return rc;
  if (!simt) {
    rc = bits_filter<BITS>(st, nullptr);
    if (rc) return rc;
    CKE(cudaMemcpy(counts, st.cnt.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    if (counts[0] > st.cand_cap) {
      simt = true;
    } else if (counts[0]) {
      bits::eval_bits_rescore_kernel<BITS><<<(unsigned)((counts[0] + 127) / 128), 128>>>(
          st.sign.as<unsigned>(), st.mag.as<unsigned>(), st.len.as<float>(), st.q3.as<int>(), st.cand.as<tc::Candidate>(),
          counts[0], st.qeps.as<float>(), st.gmax.as<unsigned>(), dbest, st.cnt.as<unsigned long long>() + 1, st.D, st.Wp);
      CKE(cudaGetLastError());
    }
  }
  return simt ? bits_score_simt<BITS>(st, dbest) : W2B_OK;
}

// The rows and names of a packed file (the first `threshold` words when threshold > 0).
int read_packed(const char *packed_file, int64_t threshold, std::vector<std::string> &names, std::vector<uint8_t> &rows,
                long long &words, long long &size, int &bits) {
  w2b_packed_file pf;
  int rc = w2b_packed_open(packed_file, &pf);
  if (rc) return rc;
  words = pf.V;
  size = pf.D;
  bits = pf.bits;
  if (threshold > 0 && words > threshold) words = threshold;
  // D <= 2^17: the integer scores stay below 2^24 and eval_bits_qeps_kernel's slack holds
  if (words < 1 || words > 0x7fffffffLL || size > (1LL << 17) || words > (1LL << 40) / pf.nbytes) {
    w2b_set_error("bad header: %lld words of size %lld", words, size);
    return W2B_EIO;
  }
  names.resize(words);
  rows.resize((size_t)words * pf.nbytes);
  for (long long b = 0; b < words; ++b) {
    char raw[256];
    rc = w2b_packed_next(&pf, raw, sizeof raw, &rows[(size_t)b * pf.nbytes]);
    if (rc) return rc;
    std::string w;  // read_vectors' rule for a name
    for (const char *p = raw; *p; ++p)
      if (*p != '\n' && w.size() < 50) w.push_back(*p);
    names[b] = upper(w);
  }
  return W2B_OK;
}

// the distinct query words: the Gram kernel runs once per word, not once per question
void distinct_words(const std::vector<int> &q3, std::vector<int> &qid, std::vector<int> &q3w) {
  q3w.resize(q3.size());
  std::unordered_map<int, int> row_of;
  for (size_t i = 0; i < q3.size(); ++i) {
    auto it = row_of.emplace(q3[i], (int)qid.size());
    if (it.second) qid.push_back(q3[i]);
    q3w[i] = it.first->second;
  }
}

// a packed table (t.bits = 1 or 2: a packed file, or a context on the bit-domain route)
int compute_accuracy_packed_impl(const Table &t, const char *questions_file, int device, w2b_accuracy *acc, char *report,
                                 int64_t report_cap, int32_t *answers, int64_t answers_cap, int64_t *n_questions) {
  const std::vector<std::string> &names = t.names;
  const long long words = t.words, size = t.size;
  const int file_bits = t.bits;
  Questions qs;
  int rc = parse_questions(questions_file, names, qs);
  if (rc) return rc;
  const long long nq = (long long)qs.q3.size() / 3;
  std::vector<int> qid, q3w;
  distinct_words(qs.q3, qid, q3w);

  std::vector<unsigned long long> best(nq > 0 ? nq : 1, 0);
  float ms = 0.f;
  if (nq > 0) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device >= ndev) {
      w2b_set_error("no CUDA device %d: the evaluator has no CPU fallback", device);
      return W2B_ECUDA;
    }
    CKE(cudaSetDevice(device));
    if (acc) acc->candidates = acc->rescored = 0;
    const char *dbg = getenv("W2B_EVAL_SIMT");
    const bool simt = dbg && atoi(dbg) != 0;
    BitsState st;
    st.ctx = t.ctx;
    DevBuf bbest;
    rc = bits_upload(st, t.ctx ? nullptr : t.rows.data(), words, (int)size, file_bits, qid.data(), (int)qid.size(), q3w.data(), qs.q3.data(), nq,
                     (unsigned long long)nq * 1024ull);  // the cap of the tensor-core filter's list
    if (rc) return rc;
    CKE(bbest.alloc(nq * sizeof(unsigned long long)));
    CKE(cudaMemset(bbest.p, 0, nq * sizeof(unsigned long long)));
    DevEvent e0, e1;
    CKE(cudaEventCreate(&e0.e));
    CKE(cudaEventCreate(&e1.e));
    CKE(cudaEventRecord(e0.e));
    unsigned long long counts[2] = {0, 0};
    rc = file_bits == 1 ? bits_answers<1>(st, simt, bbest.as<unsigned long long>(), counts)
                      : bits_answers<2>(st, simt, bbest.as<unsigned long long>(), counts);
    if (rc) return rc;
    CKE(cudaEventRecord(e1.e));
    CKE(cudaMemcpy(best.data(), bbest.p, nq * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    CKE(cudaEventElapsedTime(&ms, e0.e, e1.e));
    if (acc && !simt) {
      CKE(cudaMemcpy(counts, st.cnt.p, sizeof(unsigned long long) * 2, cudaMemcpyDeviceToHost));
      acc->candidates = (int64_t)counts[0];
      acc->rescored = (int64_t)counts[1];
    }
  }
  write_report(qs, names, best, words, size, ms, acc, report, report_cap, answers, answers_cap, n_questions);
  return W2B_OK;
}

int compute_accuracy_packed_file(const char *packed_file, int64_t threshold, const char *questions_file, int device,
                                 w2b_accuracy *acc, char *report, int64_t report_cap, int32_t *answers,
                                 int64_t answers_cap, int64_t *n_questions) {
  Table t;
  const int rc = read_packed(packed_file, threshold, t.names, t.rows, t.words, t.size, t.bits);
  if (rc) return rc;
  return compute_accuracy_packed_impl(t, questions_file, device, acc, report, report_cap, answers, answers_cap,
                                      n_questions);
}

}  // namespace

extern "C" int w2b_compute_accuracy_packed(const char *packed_file, int64_t threshold, const char *questions_file,
                                           int device, w2b_accuracy *acc, char *report, int64_t report_cap) {
  if (!packed_file) { w2b_set_error("w2b_compute_accuracy_packed: null packed_file"); return W2B_EINVAL; }
  if (report && report_cap > 0) report[0] = 0;
  return no_throw("w2b_compute_accuracy_packed", [&] {
    return compute_accuracy_packed_file(packed_file, threshold, questions_file, device, acc, report, report_cap, nullptr,
                                        0, nullptr);
  });
}
extern "C" int w2b_analogy_answers_packed(const char *packed_file, int64_t threshold, const char *questions_file,
                                          int device, int32_t *answers, int64_t answers_cap, int64_t *n_questions) {
  if (!packed_file || (!answers && answers_cap > 0)) {
    w2b_set_error("w2b_analogy_answers_packed: null argument");
    return W2B_EINVAL;
  }
  return no_throw("w2b_analogy_answers_packed", [&] {
    return compute_accuracy_packed_file(packed_file, threshold, questions_file, device, nullptr, nullptr, 0, answers,
                                        answers_cap, n_questions);
  });
}

// Test hook of the bit path: the Gram kernel's integers for explicit packed rows and query words, and the filter's
// score of every (question, word) pair: eval_bits_combine_kernel runs unchanged with eps = +inf (every pair is a
// candidate), no words to skip and room for nq * V candidates; eps itself comes from eval_bits_qeps_kernel.
extern "C" int w2b_eval_packed_scores(const uint8_t *rows, int64_t V, int64_t D, int bitlevel, const int32_t *qid,
                                      int64_t W, const int32_t *q3, int64_t nq, int device, int32_t *gram, float *approx,
                                      float *eps) {
  if (!rows || !qid || !gram || V < 1 || D < 1 || D > (1LL << 17) || (bitlevel != 1 && bitlevel != 2) || W < 1 || nq < 0 ||
      (nq > 0 && !q3) || (approx && nq < 1) || W * V > (1LL << 31) || nq * V > (1LL << 31)) {
    w2b_set_error("w2b_eval_packed_scores: bad arguments");
    return W2B_EINVAL;
  }
  for (int64_t i = 0; i < W; ++i)
    if (qid[i] < 0 || qid[i] >= V) { w2b_set_error("w2b_eval_packed_scores: qid[%lld] out of range", (long long)i); return W2B_EINVAL; }
  for (int64_t i = 0; i < 3 * nq; ++i)
    if (q3[i] < 0 || q3[i] >= W) { w2b_set_error("w2b_eval_packed_scores: q3[%lld] out of range", (long long)i); return W2B_EINVAL; }
  return no_throw("w2b_eval_packed_scores", [&]() -> int {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device >= ndev) {
      w2b_set_error("no CUDA device %d: the evaluator has no CPU fallback", device);
      return W2B_ECUDA;
    }
    CKE(cudaSetDevice(device));
    const long long nqd = nq > 0 ? nq : 1;  // without questions: one that reads query word 0, its scores unused
    std::vector<int> none((size_t)nqd * 3, -1), q3w((size_t)nqd * 3, 0);
    if (nq > 0) q3w.assign(q3, q3 + 3 * nq);
    const unsigned long long cap = approx ? (unsigned long long)nq * (unsigned long long)V : 1ull;
    BitsState st;
    int rc = bits_upload(st, rows, V, (int)D, bitlevel, qid, (int)W, q3w.data(), none.data(), nqd, cap);
    if (rc) return rc;
    rc = bitlevel == 1 ? bits_planes<1>(st) : bits_planes<2>(st);
    if (rc) return rc;
    if (eps && nq > 0) CKE(cudaMemcpy(eps, st.qeps.p, nq * sizeof(float), cudaMemcpyDeviceToHost));
    std::vector<float> inf((size_t)nqd, INFINITY);
    CKE(cudaMemcpy(st.qeps.p, inf.data(), nqd * sizeof(float), cudaMemcpyHostToDevice));
    rc = bitlevel == 1 ? bits_filter<1>(st, gram) : bits_filter<2>(st, gram);
    if (rc) return rc;
    if (approx) {
      unsigned long long n = 0;
      CKE(cudaMemcpy(&n, st.cnt.p, sizeof n, cudaMemcpyDeviceToHost));
      if (n != cap) {
        w2b_set_error("w2b_eval_packed_scores: %llu of %llu pairs came through", n, cap);
        return W2B_EINVAL;
      }
      std::vector<tc::Candidate> cand((size_t)n);
      CKE(cudaMemcpy(cand.data(), st.cand.p, n * sizeof(tc::Candidate), cudaMemcpyDeviceToHost));
      for (const tc::Candidate &c : cand) approx[(size_t)c.q * V + c.c] = c.s;
    }
    return W2B_OK;
  });
}

// ------------------------------------------------------------------------------------------------------------------
// Top-k lists (w2b_analogy_topk, w2b_nearest; kernels in w2b_eval_topk.cuh).  A query is an analogy question or a
// nearest-neighbour word w taken as the question (w, w, w): vec = (M[w] - M[w]) + M[w] = M[w] exactly, and only w is
// skipped.  The vocabulary is walked a chunk at a time; a chunk of scores for a block of queries is written densely
// (kDenseFloats floats at most) and read by the selection kernel, which carries every query's kept set to the next
// chunk.  Approximate scores (TF32, or the bit domain of a packed file) leave a candidate list per query that is
// re-scored exactly; a list that overflows, and W2B_EVAL_SIMT=1, take exact fp32 scores from the SIMT scorer instead
// and select with 64-bit keys.
namespace {

constexpr long long kDenseFloats = 8ll << 20;  // a chunk of scores: 32 MB
constexpr long long kListBytes = 2ll << 30;     // candidate lists, keys, kept sets and lists of one batch of queries

struct TopkBufs {
  DevBuf kept, kth, cand, ncand, keys, ids, scores, cnt, S;
  long long nq = 0, nqb = 0, ch = 0, chunks = 0;
  int k = 0, cap = 0;
};

// queries per block and words per chunk of the dense score buffer
void dense_geometry(TopkBufs &b, long long words, long long max_ch) {
  b.nqb = std::min<long long>(b.nq, 1024);
  b.ch = std::max<long long>(256, kDenseFloats / b.nqb / 256 * 256);
  b.ch = std::min(b.ch, std::min(max_ch, (words + 255) / 256 * 256));
}

int topk_alloc(TopkBufs &b, long long nq, int k) {
  b.nq = nq;
  b.k = k;
  // candidates a query may have: its k and what ties within 2 eps of them, plus what each chunk adds above a
  // threshold that is still rising (about k ln(chunks) over a walk of the vocabulary, measured at 20 chunks)
  b.cap = 8 * k + 1024;
  CKE(b.kept.alloc((size_t)nq * k * 8));
  CKE(b.kth.alloc((size_t)nq * 8));
  CKE(b.cand.alloc((size_t)nq * b.cap * sizeof(topk::Cand)));
  CKE(b.ncand.alloc((size_t)nq * 4));
  CKE(b.keys.alloc((size_t)nq * b.cap * 8));
  CKE(b.ids.alloc((size_t)nq * k * 4));
  CKE(b.scores.alloc((size_t)nq * k * 4));
  CKE(b.cnt.alloc(8));
  CKE(cudaMemset(b.ncand.p, 0, (size_t)nq * 4));
  CKE(cudaMemset(b.cnt.p, 0, 8));
  return W2B_OK;
}

int topk_reset(TopkBufs &b) {  // empty kept sets
  CKE(cudaMemset(b.kept.p, 0, (size_t)b.nq * b.k * 8));
  CKE(cudaMemset(b.kth.p, 0, (size_t)b.nq * 8));
  b.chunks = 0;
  return W2B_OK;
}

template <bool EXACT> int topk_select(TopkBufs &b, long long qb, long long nqb, long long c0, int nc, const int *dq3,
                                      const float *dqeps) {
  using K = typename std::conditional<EXACT, unsigned long long, unsigned>::type;
  topk::topk_select_kernel<EXACT><<<(unsigned)nqb, topk::THREADS>>>(
      b.S.as<float>(), b.ch, c0, nc, dq3 + 3 * qb, EXACT ? nullptr : dqeps + qb, b.kept.as<K>() + qb * b.k,
      b.kth.as<K>() + qb, EXACT ? nullptr : b.cand.as<topk::Cand>() + qb * b.cap, EXACT ? nullptr : b.ncand.as<int>() + qb,
      b.cap, b.k);
  CKE(cudaGetLastError());
  return W2B_OK;
}

// exact lists from the SIMT scorer: Q (nq x Dp) against M (words x Dp), both normalised fp32
int topk_simt(TopkBufs &b, const float *dQ, const float *dM, const int *dq3, long long words, long long D, long long Dp) {
  int rc = topk_reset(b);
  if (rc) return rc;
  for (long long c0 = 0; c0 < words; c0 += b.ch, ++b.chunks) {
    const int nc = (int)std::min(b.ch, words - c0);
    for (long long qb = 0; qb < b.nq; qb += b.nqb) {
      const long long n = std::min(b.nqb, b.nq - qb);
      dim3 grid((unsigned)((nc + TN - 1) / TN), (unsigned)((n + TM - 1) / TM));
      eval_score_kernel<true><<<grid, 256>>>(dQ + qb * Dp, dM + c0 * Dp, nullptr, nullptr, n, nc, D, Dp, b.S.as<float>(), b.ch);
      if ((rc = topk_select<true>(b, qb, n, c0, nc, dq3, nullptr))) return rc;
    }
  }
  topk::topk_final_kernel<<<(unsigned)b.nq, topk::THREADS>>>(b.kept.as<unsigned long long>(), nullptr, b.k, b.k,
                                                             b.ids.as<int>(), b.scores.as<float>());
  CKE(cudaGetLastError());
  return W2B_OK;
}

// after a filter pass: true when some query's candidate list overflowed
int topk_overflowed(TopkBufs &b, bool &over, int64_t &candidates) {
  std::vector<int> n((size_t)b.nq);
  CKE(cudaMemcpy(n.data(), b.ncand.p, (size_t)b.nq * 4, cudaMemcpyDeviceToHost));
  over = false;
  for (int x : n) {
    over |= x > b.cap;
    candidates += x;
  }
  return W2B_OK;
}

int topk_final(TopkBufs &b) {
  topk::topk_final_kernel<<<(unsigned)b.nq, topk::THREADS>>>(b.keys.as<unsigned long long>(), b.ncand.as<int>(), b.cap,
                                                             b.k, b.ids.as<int>(), b.scores.as<float>());
  CKE(cudaGetLastError());
  return W2B_OK;
}

// fp32 file: the queries of one batch against the normalised table dM, TF32 filter + exact re-score (or the SIMT
// scorer).  *ms += the device time from the first kernel to the last (uploads and frees outside it).
int topk_fp32(const float *dM, long long words, long long size, const std::vector<int> &q3, bool simt, TopkBufs &b,
              w2b_topk_stats &s, float *ms) {
  const long long nq = b.nq, Dp = (size + tc::BK - 1) / tc::BK * tc::BK;
  DevBuf bQ, bq3, bqeps;
  DevEvent e0, e1;
  CKE(bQ.alloc((size_t)nq * Dp * sizeof(float)));
  CKE(bq3.alloc(q3.size() * sizeof(int)));
  CKE(bqeps.alloc(nq * sizeof(float)));
  float *dQ = bQ.as<float>();
  int *dq3 = bq3.as<int>();
  CKE(cudaMemset(dQ, 0, (size_t)nq * Dp * sizeof(float)));
  CKE(cudaMemcpy(dq3, q3.data(), q3.size() * sizeof(int), cudaMemcpyHostToDevice));
  dense_geometry(b, words, 1LL << 40);
  CKE(b.S.alloc((size_t)b.nqb * b.ch * sizeof(float)));
  CKE(cudaEventCreate(&e0.e));
  CKE(cudaEventCreate(&e1.e));
  CKE(cudaEventRecord(e0.e));
  eval_query_kernel<<<(unsigned)((nq * size + 255) / 256), 256>>>(dM, dq3, dQ, nq, size, Dp);
  int rc = W2B_OK;
  if (!simt) {
    if ((rc = topk_reset(b))) return rc;
    if (rc) return rc;
    eval_qeps_kernel<<<(unsigned)((nq + 7) / 8), 256>>>(dQ, bqeps.as<float>(), nq, Dp);
    CKE(cudaFuncSetAttribute(tc::eval_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES));
    std::vector<CUtensorMap> mapQ((size_t)((nq + b.nqb - 1) / b.nqb));  // one per block of queries
    for (size_t i = 0; i < mapQ.size(); ++i)
      if (!tc::make_map(&mapQ[i], dQ + (long long)i * b.nqb * Dp, std::min(b.nqb, nq - (long long)i * b.nqb), Dp, tc::BM)) {
        w2b_set_error("cuTensorMapEncodeTiled failed (driver too old for TMA?)");
        return W2B_ECUDA;
      }
    for (long long c0 = 0; c0 < words; c0 += b.ch, ++b.chunks) {
      const int nc = (int)std::min(b.ch, words - c0);
      CUtensorMap mapM;
      if (!tc::make_map(&mapM, dM + c0 * Dp, nc, Dp, tc::BN)) {
        w2b_set_error("cuTensorMapEncodeTiled failed (driver too old for TMA?)");
        return W2B_ECUDA;
      }
      for (long long qb = 0; qb < nq; qb += b.nqb) {
        const long long n = std::min(b.nqb, nq - qb);
        dim3 grid((unsigned)((n + tc::BM - 1) / tc::BM), (unsigned)((nc + tc::BN - 1) / tc::BN));
        tc::eval_tc_kernel<true><<<grid, tc::THREADS, tc::SMEM_BYTES>>>(mapQ[qb / b.nqb], mapM, nullptr, nullptr, nullptr, nullptr,
                                                                       nullptr, 0, (int)n, nc, (int)Dp, b.S.as<float>(), b.ch);
        if ((rc = topk_select<false>(b, qb, n, c0, nc, dq3, bqeps.as<float>()))) return rc;
      }
    }
    bool over = false;
    if ((rc = topk_overflowed(b, over, s.candidates))) return rc;
    if (over) {
      simt = true;  // ties by the thousand (e.g. all vectors equal): every score exactly instead
    } else {
      topk::topk_rescore_kernel<<<(unsigned)((nq * b.cap + 127) / 128), 128>>>(
          dQ, dM, b.cand.as<topk::Cand>(), b.ncand.as<int>(), b.cap, b.kth.as<unsigned>(), bqeps.as<float>(),
          b.keys.as<unsigned long long>(), b.cnt.as<unsigned long long>(), nq, (int)size, Dp);
      if ((rc = topk_final(b))) return rc;
    }
  }
  s.simt |= simt;
  if (simt && (rc = topk_simt(b, dQ, dM, dq3, words, size, Dp))) return rc;
  CKE(cudaEventRecord(e1.e));
  CKE(cudaEventSynchronize(e1.e));  // bQ, bq3 and bqeps are freed on return
  float t = 0.f;
  CKE(cudaEventElapsedTime(&t, e0.e, e1.e));
  *ms += t;
  return W2B_OK;
}

// packed file: planes, then per chunk the Gram kernel and the bit-domain scores of every block of queries
template <int BITS> int topk_packed_run(BitsState &st, bool simt, TopkBufs &b, w2b_topk_stats &s) {
  int rc = bits_planes<BITS>(st);
  if (rc) return rc;
  const long long nq = b.nq;
  if (!simt) {
    if ((rc = topk_reset(b))) return rc;
    b.nqb = std::max<long long>(1, std::min(nq, kDenseFloats / st.chunk));
    b.ch = st.chunk;
    CKE(b.S.alloc((size_t)b.nqb * b.ch * sizeof(float)));
    for (long long c0 = 0; c0 < st.V; c0 += st.chunk, ++b.chunks) {
      const int nc = (int)std::min(st.chunk, st.V - c0);
      dim3 gg((unsigned)((nc + bits::GT - 1) / bits::GT), (unsigned)((st.W + bits::GT - 1) / bits::GT));
      bits::eval_bits_gram_kernel<BITS><<<gg, 256>>>(st.sign.as<unsigned>(), st.mag.as<unsigned>(), st.hpop.as<int>(),
                                                    st.qid.as<int>(), st.W, c0, nc, st.D, st.Wp, st.G.as<int>(), st.chunk);
      for (long long qb = 0; qb < nq; qb += b.nqb) {
        const long long n = std::min(b.nqb, nq - qb);
        bits::eval_bits_combine_store_kernel<<<dim3((unsigned)((nc + 255) / 256), (unsigned)n), 256>>>(
            st.G.as<int>(), st.chunk, c0, nc, st.ilen.as<float>(), st.q3w.as<int>() + 3 * qb, st.qk.as<float>() + 3 * qb,
            b.S.as<float>(), b.ch);
        if ((rc = topk_select<false>(b, qb, n, c0, nc, st.q3.as<int>(), st.qeps.as<float>()))) return rc;
      }
    }
    bool over = false;
    if ((rc = topk_overflowed(b, over, s.candidates))) return rc;
    if (over) {
      simt = true;
    } else {
      topk::topk_bits_rescore_kernel<BITS><<<(unsigned)((nq * b.cap + 127) / 128), 128>>>(
          st.sign.as<unsigned>(), st.mag.as<unsigned>(), st.len.as<float>(), st.q3.as<int>(), b.cand.as<topk::Cand>(),
          b.ncand.as<int>(), b.cap, b.kth.as<unsigned>(), st.qeps.as<float>(), b.keys.as<unsigned long long>(),
          b.cnt.as<unsigned long long>(), nq, st.D, st.Wp);
      return topk_final(b);
    }
  }
  s.simt = 1;
  const long long Dp = (st.D + tc::BK - 1) / tc::BK * tc::BK;
  DevBuf bM, bQ;
  if ((rc = bits_fp32<BITS>(st, bM, bQ, Dp))) return rc;
  dense_geometry(b, st.V, 1LL << 40);
  b.S.reset();  // the filter's chunk had another shape
  CKE(b.S.alloc((size_t)b.nqb * b.ch * sizeof(float)));
  if ((rc = topk_simt(b, bQ.as<float>(), bM.as<float>(), st.q3.as<int>(), st.V, st.D, Dp))) return rc;
  CKE(cudaDeviceSynchronize());  // bM and bQ are freed on return
  return W2B_OK;
}

// the packed pipeline of one batch, timed from the plane kernel on (as the arg-max evaluator times it)
template <int BITS> int topk_packed(BitsState &st, bool simt, TopkBufs &b, w2b_topk_stats &s, float *ms) {
  DevEvent e0, e1;
  CKE(cudaEventCreate(&e0.e));
  CKE(cudaEventCreate(&e1.e));
  CKE(cudaEventRecord(e0.e));
  int rc = topk_packed_run<BITS>(st, simt, b, s);
  if (rc) return rc;
  CKE(cudaEventRecord(e1.e));
  CKE(cudaEventSynchronize(e1.e));
  float t = 0.f;
  CKE(cudaEventElapsedTime(&t, e0.e, e1.e));
  *ms += t;
  return W2B_OK;
}

// t: the table (names only matter when cap_queries > 0: counting the queries needs no vectors); packed = t.bits, the
// level of a packed file or of a context on the bit-domain route, 0 for an fp32 table.
int topk_impl(const Table &t, int packed, int bitlevel, bool nearest, const char *input, int k, int device, int32_t *ids,
              float *scores, int64_t cap_queries, int64_t *n_queries, w2b_topk_stats *stats) {
  w2b_topk_stats s;
  memset(&s, 0, sizeof s);
  const std::vector<std::string> &names = t.names;
  const long long words = t.words, size = t.size;
  const int file_bits = packed;
  int rc = W2B_OK;
  // per output row (file order): the query it is, or -1 (a word is not in the vocabulary)
  std::vector<int> q3, row_q;
  if (nearest) {
    std::unordered_map<std::string, int> first;  // first match, as parse_questions finds words
    for (long long w = words - 1; w >= 0; --w) first[names[w]] = (int)w;
    FILE *f = input ? fopen(input, "rb") : stdin;
    if (!f) { w2b_set_error("words file not found"); return W2B_EIO; }
    FileCloser closer{f};
    char buf[2048];
    while (fscanf(f, "%2000s", buf) == 1) {
      auto it = first.find(upper(buf));
      row_q.push_back(it == first.end() ? -1 : (int)(q3.size() / 3));
      if (it != first.end()) q3.insert(q3.end(), {it->second, it->second, it->second});
    }
  } else {
    Questions qs;
    if ((rc = parse_questions(input, names, qs))) return rc;
    for (const Ev &e : qs.events)
      if (e.kind == 1) row_q.push_back(e.qidx);
    q3 = qs.q3;
  }
  const long long nq = (long long)q3.size() / 3;
  s.queries = (int64_t)row_q.size();
  s.skipped = s.queries - nq;
  s.packed = packed != 0;
  std::vector<int32_t> hid((size_t)nq * k);
  std::vector<float> hsc((size_t)nq * k);
  if (nq > 0 && cap_queries > 0) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device >= ndev) {
      w2b_set_error("no CUDA device %d: the evaluator has no CPU fallback", device);
      return W2B_ECUDA;
    }
    CKE(cudaSetDevice(device));
    const char *dbg = getenv("W2B_EVAL_SIMT");
    const bool simt = dbg && atoi(dbg) != 0;
    // fp32 table: uploaded and normalised once for every batch
    DevBuf bM;
    float *dM = nullptr;
    const long long Dp = (size + tc::BK - 1) / tc::BK * tc::BK;
    if (!packed) {
      DevEvent e0, e1;
      if ((rc = upload_fp32(t, bM, Dp, &dM))) return rc;
      CKE(cudaEventCreate(&e0.e));
      CKE(cudaEventCreate(&e1.e));
      CKE(cudaEventRecord(e0.e));
      build_fp32(t, dM, Dp);
      eval_normalize_kernel<<<(unsigned)((words + 7) / 8), 256>>>(dM, words, size, Dp, bitlevel);
      CKE(cudaEventRecord(e1.e));
      CKE(cudaEventSynchronize(e1.e));
      CKE(cudaEventElapsedTime(&s.gpu_ms, e0.e, e1.e));
    }
    // queries in batches, so that candidate lists and kept sets stay within kListBytes
    const long long per_query = (8LL * k + 1024) * 16 + 16LL * k + 16;
    const long long batch = std::max<long long>(1024, kListBytes / per_query);
    for (long long q0 = 0; q0 < nq; q0 += batch) {
      const long long nb = std::min(batch, nq - q0);
      const std::vector<int> sub(q3.begin() + 3 * q0, q3.begin() + 3 * (q0 + nb));
      TopkBufs b;
      if ((rc = topk_alloc(b, nb, k))) return rc;
      if (!packed) {
        rc = topk_fp32(dM, words, size, sub, simt, b, s, &s.gpu_ms);
      } else {
        BitsState st;
        st.ctx = t.ctx;
        std::vector<int> qid, q3w;
        distinct_words(sub, qid, q3w);
        if ((rc = bits_upload(st, t.ctx ? nullptr : t.rows.data(), words, (int)size, file_bits, qid.data(), (int)qid.size(), q3w.data(),
                              sub.data(), nb, 1)))  // (its arg-max candidate list is not used)
          return rc;
        rc = file_bits == 1 ? topk_packed<1>(st, simt, b, s, &s.gpu_ms) : topk_packed<2>(st, simt, b, s, &s.gpu_ms);
      }
      if (rc) return rc;
      CKE(cudaMemcpy(hid.data() + q0 * k, b.ids.p, (size_t)nb * k * 4, cudaMemcpyDeviceToHost));
      CKE(cudaMemcpy(hsc.data() + q0 * k, b.scores.p, (size_t)nb * k * 4, cudaMemcpyDeviceToHost));
      unsigned long long n_rescored = 0;
      CKE(cudaMemcpy(&n_rescored, b.cnt.p, 8, cudaMemcpyDeviceToHost));
      s.rescored += (int64_t)n_rescored;
      s.chunks = std::max<int64_t>(s.chunks, b.chunks);
    }
  }
  for (size_t r = 0; r < row_q.size() && (int64_t)r < cap_queries; ++r)
    for (int j = 0; j < k; ++j) {
      const int q = row_q[r];
      ids[r * k + j] = q >= 0 ? hid[(size_t)q * k + j] : -1;
      scores[r * k + j] = q >= 0 ? hsc[(size_t)q * k + j] : 0.f;
    }
  if (n_queries) *n_queries = (int64_t)row_q.size();
  if (stats) *stats = s;
  return W2B_OK;
}

int topk_file(const char *vectors_file, int bitlevel, int64_t threshold, bool nearest, const char *input, int k,
              int device, int32_t *ids, float *scores, int64_t cap_queries, int64_t *n_queries, w2b_topk_stats *stats) {
  int bits;
  const int kind = vector_kind(vectors_file, &bits);
  const int packed = kind == W2B_VECTORS_PACKED ? bits : 0;
  if (packed && bitlevel != 0 && bitlevel != packed) {
    w2b_set_error("%s holds %d-bit vectors: bitlevel must be %d or 0", vectors_file, packed, packed);
    return W2B_EINVAL;
  }
  Table t;
  if (cap_queries > 0) {  // (counting the queries needs no vectors: no word is then in the vocabulary)
    const int rc = packed                        ? read_packed(vectors_file, threshold, t.names, t.rows, t.words, t.size, t.bits)
                   : kind == W2B_VECTORS_TEXT ? read_text(vectors_file, threshold, device, t)
                                              : read_vectors(vectors_file, threshold, t.names, t.M, t.words, t.size);
    if (rc) return rc;
  }
  return topk_impl(t, packed, bitlevel, nearest, input, k, device, ids, scores, cap_queries, n_queries, stats);
}

int topk_args(const char *who, const char *vectors_file, int k, const int32_t *ids, const float *scores,
              int64_t cap_queries) {
  if (!vectors_file || k < 1 || k > W2B_MAX_TOPK || cap_queries < 0 || (cap_queries > 0 && (!ids || !scores))) {
    w2b_set_error("%s: bad arguments (vectors_file %s, k = %d: 1 <= k <= %d, ids and scores for %lld rows)", who,
                  vectors_file ? "set" : "NULL", k, W2B_MAX_TOPK, (long long)cap_queries);
    return W2B_EINVAL;
  }
  return W2B_OK;
}

}  // namespace

extern "C" int w2b_analogy_topk(const char *vectors_file, int bitlevel, int64_t threshold, const char *questions_file,
                                int k, int device, int32_t *ids, float *scores, int64_t cap_queries, int64_t *n_queries,
                                w2b_topk_stats *st) {
  if (int rc = topk_args("w2b_analogy_topk", vectors_file, k, ids, scores, cap_queries)) return rc;
  return no_throw("w2b_analogy_topk", [&] {
    return topk_file(vectors_file, bitlevel, threshold, false, questions_file, k, device, ids, scores, cap_queries,
                     n_queries, st);
  });
}

extern "C" int w2b_nearest(const char *vectors_file, int bitlevel, int64_t threshold, const char *words_file, int k,
                           int device, int32_t *ids, float *scores, int64_t cap_queries, int64_t *n_queries,
                           w2b_topk_stats *st) {
  if (int rc = topk_args("w2b_nearest", vectors_file, k, ids, scores, cap_queries)) return rc;
  return no_throw("w2b_nearest", [&] {
    return topk_file(vectors_file, bitlevel, threshold, true, words_file, k, device, ids, scores, cap_queries, n_queries,
                     st);
  });
}

// ------------------------------------------------------------------------------------------------------------------
// The evaluator on a training context's own tables (w2b_ctx_*): the table is quantize(u + v), formed on the device from
// u and v, with words[i] the name of row i.  The route follows from what the context holds: a 1-bit or 2-bit context
// evaluated at its own level (bitlevel 0 or the same) is scored in the bit domain from planes built straight from u and
// v (eval_ctx_planes_kernel), as its packed file would be; every other case fills the fp32 table that -binary 1 would
// write (eval_ctx_table_kernel) and runs the fp32 pipeline.  Either way nothing is copied to the host and u, v, alpha,
// the word counter and the shard states are only read.
namespace {

// names as read_vectors reads them from the written file (at most 50 characters, upper-cased); the context's stream
// is drained first, since training may still be running on it
int ctx_table(const char *who, w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
              w2b_ctx_tables &ct, Table &t) {
  int rc = w2b_ctx_tables_of(ctx, &ct);
  if (rc) return rc;
  t.words = (threshold > 0 && ct.V > threshold) ? threshold : ct.V;
  t.size = ct.D;
  t.names.resize(t.words);
  for (long long b = 0; b < t.words; ++b) {
    const char *w = words[b];
    if (!w || strpbrk(w, " \n")) {  // a name the file round trip cannot carry
      w2b_set_error("%s: the name of row %lld %s", who, b, w ? "contains ' ' or '\\n'" : "is NULL");
      return W2B_EINVAL;
    }
    std::string n;
    for (const char *p = w; *p && n.size() < 50; ++p) n.push_back(*p);
    t.names[b] = upper(n);
  }
  t.ctx = &ct;
  t.bits = ((ct.bitlevel == 1 || ct.bitlevel == 2) && (bitlevel == 0 || bitlevel == ct.bitlevel)) ? ct.bitlevel : 0;
  CKE(cudaSetDevice(ct.device));
  CKE(cudaStreamSynchronize((cudaStream_t)ct.stream));
  return W2B_OK;
}

int ctx_topk_args(const char *who, int k, const int32_t *ids, const float *scores, int64_t cap_queries) {
  if (k < 1 || k > W2B_MAX_TOPK || cap_queries < 0 || (cap_queries > 0 && (!ids || !scores))) {
    w2b_set_error("%s: bad arguments (k = %d: 1 <= k <= %d, ids and scores for %lld rows)", who, k, W2B_MAX_TOPK,
                  (long long)cap_queries);
    return W2B_EINVAL;
  }
  return W2B_OK;
}

template <class F> int ctx_call(const char *who, w2b_ctx *ctx, const char *const *words, F &&f) {
  if (!ctx || !words) {
    w2b_set_error("%s: null %s", who, ctx ? "words" : "ctx");
    return W2B_EINVAL;
  }
  const int rc = no_throw(who, f);
  if (rc) (void)cudaGetLastError();  // e.g. a failed allocation: not reported again by the context's next call
  return rc;
}

int ctx_accuracy(const char *who, w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                 const char *questions_file, w2b_accuracy *acc, char *report, int64_t report_cap, int32_t *answers,
                 int64_t answers_cap, int64_t *n_questions) {
  w2b_ctx_tables ct;
  Table t;
  const int rc = ctx_table(who, ctx, words, bitlevel, threshold, ct, t);
  if (rc) return rc;
  return t.bits ? compute_accuracy_packed_impl(t, questions_file, ct.device, acc, report, report_cap, answers,
                                               answers_cap, n_questions)
                : compute_accuracy_impl(t, bitlevel, questions_file, ct.device, acc, report, report_cap, answers,
                                        answers_cap, n_questions);
}

int ctx_topk(const char *who, w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold, bool nearest,
             const char *input, int k, int32_t *ids, float *scores, int64_t cap_queries, int64_t *n_queries,
             w2b_topk_stats *st) {
  w2b_ctx_tables ct;
  Table t;
  const int rc = ctx_table(who, ctx, words, bitlevel, threshold, ct, t);
  if (rc) return rc;
  return topk_impl(t, t.bits, bitlevel, nearest, input, k, ct.device, ids, scores, cap_queries, n_queries, st);
}

}  // namespace

extern "C" int w2b_ctx_compute_accuracy(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                                        const char *questions_file, w2b_accuracy *acc, char *report, int64_t report_cap) {
  if (report && report_cap > 0) report[0] = 0;
  return ctx_call("w2b_ctx_compute_accuracy", ctx, words, [&] {
    return ctx_accuracy("w2b_ctx_compute_accuracy", ctx, words, bitlevel, threshold, questions_file, acc, report,
                        report_cap, nullptr, 0, nullptr);
  });
}

extern "C" int w2b_ctx_analogy_answers(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                                       const char *questions_file, int32_t *answers, int64_t answers_cap,
                                       int64_t *n_questions) {
  if (!answers && answers_cap > 0) {
    w2b_set_error("w2b_ctx_analogy_answers: null answers");
    return W2B_EINVAL;
  }
  return ctx_call("w2b_ctx_analogy_answers", ctx, words, [&] {
    return ctx_accuracy("w2b_ctx_analogy_answers", ctx, words, bitlevel, threshold, questions_file, nullptr, nullptr, 0,
                        answers, answers_cap, n_questions);
  });
}

extern "C" int w2b_ctx_analogy_topk(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                                    const char *questions_file, int k, int32_t *ids, float *scores, int64_t cap_queries,
                                    int64_t *n_queries, w2b_topk_stats *st) {
  if (int rc = ctx_topk_args("w2b_ctx_analogy_topk", k, ids, scores, cap_queries)) return rc;
  return ctx_call("w2b_ctx_analogy_topk", ctx, words, [&] {
    return ctx_topk("w2b_ctx_analogy_topk", ctx, words, bitlevel, threshold, false, questions_file, k, ids, scores,
                    cap_queries, n_queries, st);
  });
}

extern "C" int w2b_ctx_nearest(w2b_ctx *ctx, const char *const *words, int bitlevel, int64_t threshold,
                               const char *words_file, int k, int32_t *ids, float *scores, int64_t cap_queries,
                               int64_t *n_queries, w2b_topk_stats *st) {
  if (int rc = ctx_topk_args("w2b_ctx_nearest", k, ids, scores, cap_queries)) return rc;
  return ctx_call("w2b_ctx_nearest", ctx, words, [&] {
    return ctx_topk("w2b_ctx_nearest", ctx, words, bitlevel, threshold, true, words_file, k, ids, scores, cap_queries,
                    n_queries, st);
  });
}
