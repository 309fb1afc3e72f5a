// Text vector files (-binary 0: header "V D", then per word "<word> ", D values "%lf ", "\n") parsed on the GPU.
// The host reads the file in fixed-size chunks into two pinned buffers and, in one pass over the bytes, finds each
// row's name and the span of its values; a chunk's partial last row moves to the front of the next chunk.  Each chunk
// is uploaded on its own stream, so that one chunk's copy runs while the other's rows are parsed.  On the device one
// warp takes a row: ballots over 32 bytes at a time find where tokens start, each lane converts one token with the
// exact routine of w2b_text.cuh, and the value goes straight into the evaluator's fp32 table (rows Dp floats apart).
#include <cuda_runtime.h>
#include <ctype.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "w2b.h"
#include "w2b_internal.h"
#include "w2b_text.cuh"

#define CKT(call)                                                                         \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      w2b_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return W2B_ECUDA;                                                                   \
    }                                                                                     \
  } while (0)

namespace {

constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kParseWarps = 8;
constexpr long long kChunkBytes = 64ll << 20;  // text per chunk (a row longer than this grows its buffer)

// a problem found on the device: the smallest key over the file wins (row first, then token)
enum { kBadToken = 1, kTooFew = 2, kTooMany = 3 };
__device__ __forceinline__ unsigned long long err_key(long long row, long long tok, int kind) {
  return ((unsigned long long)row << 24) | ((unsigned long long)min(tok, (long long)0x3fffff) << 2) | (unsigned)kind;
}

// Row first_row + r of the table: its values are buf[rows[2r], rows[2r+1]).  One warp per row; token starts are
// queued in shared memory and converted 32 at a time (lane j takes the j-th queued token).
__global__ void __launch_bounds__(kParseWarps * 32) text_parse_kernel(const char *buf, const long long *rows, int nrows,
                                                                      long long first_row, float *M, long long D,
                                                                      long long Dp, unsigned long long *err) {
  __shared__ int queue[kParseWarps][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * kParseWarps + warp;
  if (r >= nrows) return;
  const long long s = rows[2 * r], e = rows[2 * r + 1], row = first_row + r;
  const char *end = buf + e;
  float *out = M + row * Dp;
  int *q = queue[warp];
  long long ntok = 0;
  int nq = 0;
  bool prev_space = true;  // the byte before the window
  unsigned long long bad = ~0ull;
  auto convert = [&](int n) {  // the first n queued tokens: tokens ntok .. ntok + n - 1 of the row
    if (lane < n) {
      const long long t = ntok + lane;
      const char *tok = buf + s + q[lane];
      float v;
      if (!w2b::text::parse_token(tok, w2b::text::token_end(tok, end), &v))
        bad = min(bad, err_key(row, t, kBadToken));
      else if (t < D)
        out[t] = v;
    }
  };
  for (long long base = s; base < e; base += 32) {
    const long long p = base + lane;
    const bool space = p >= e || w2b::text::is_space(buf[p]);
    const bool left = __shfl_up_sync(kFullMask, space, 1);
    const bool start = !space && (lane ? left : prev_space);
    const unsigned m = __ballot_sync(kFullMask, start);
    if (start) q[nq + __popc(m & ((1u << lane) - 1))] = (int)(p - s);
    nq += __popc(m);
    prev_space = __shfl_sync(kFullMask, space, 31);
    if (nq >= 32) {
      __syncwarp();
      convert(32);
      __syncwarp();
      if (lane < nq - 32) q[lane] = q[lane + 32];
      __syncwarp();
      nq -= 32;
      ntok += 32;
    }
  }
  __syncwarp();
  convert(nq);
  ntok += nq;
  if (lane == 0 && ntok != D) bad = min(bad, err_key(row, ntok < D ? ntok : D, ntok < D ? kTooFew : kTooMany));
  if (bad != ~0ull) atomicMin(err, bad);
}

// one of the two chunk buffers: pinned host bytes, their device copy, the row spans, the stream they go on
struct Chunk {
  char *h = nullptr, *d = nullptr;
  long long *hrows = nullptr, *drows = nullptr;
  long long cap = 0, rcap = 0;
  cudaStream_t st = nullptr;
  cudaEvent_t done = nullptr;  // the chunk's copies and kernel have finished: its host buffer may be refilled
  bool used = false;
  ~Chunk() { release(); if (done) cudaEventDestroy(done); if (st) cudaStreamDestroy(st); }
  void release() {
    if (h) cudaFreeHost(h);
    if (d) cudaFree(d);
    if (hrows) cudaFreeHost(hrows);
    if (drows) cudaFree(drows);
    h = d = nullptr;
    hrows = drows = nullptr;
  }
  // room for `bytes` bytes; the first `keep` bytes of the host buffer are kept
  int reserve(long long bytes, long long keep, long long D) {
    if (bytes <= cap) return W2B_OK;
    char *nh = nullptr;
    CKT(cudaHostAlloc((void **)&nh, (size_t)bytes, cudaHostAllocDefault));
    if (keep) memcpy(nh, h, (size_t)keep);
    release();
    h = nh;
    cap = bytes;
    rcap = cap / (2 * D + 1) + 1;  // a complete row takes at least 2 D + 1 bytes (' ', D tokens and spaces, '\n')
    CKT(cudaMalloc(&d, (size_t)cap));
    CKT(cudaHostAlloc((void **)&hrows, (size_t)rcap * 16, cudaHostAllocDefault));
    CKT(cudaMalloc(&drows, (size_t)rcap * 16));
    return W2B_OK;
  }
};

struct FileCloser {
  FILE *f;
  ~FileCloser() { if (f) fclose(f); }
};

// the rows of c.h[0, len): names and value spans, at most c.rcap rows and `want` rows.  *used = bytes consumed (the
// start of the first incomplete row).  eof: the data ends the file, so a last row without '\n' is complete.
int scan_rows(Chunk &c, long long len, bool eof, long long want, std::vector<std::string> &names, long long *used) {
  const char *h = c.h;
  long long pos = 0;
  int n = 0;
  std::string name;
  while (n < c.rcap && n < want) {
    long long p = pos;
    name.clear();
    while (p < len && h[p] != ' ') {
      if (h[p] != '\n') name.push_back(h[p]);
      ++p;
    }
    if (p == len) break;  // the name goes on in the next chunk (or the file ends: truncated)
    const long long vs = p + 1;
    const char *nl = (const char *)memchr(h + vs, '\n', (size_t)(len - vs));
    if (!nl && !eof) break;
    const long long ve = nl ? nl - h : len;
    c.hrows[2 * n] = vs;
    c.hrows[2 * n + 1] = ve;
    names.push_back(name);
    ++n;
    pos = nl ? ve + 1 : len;
  }
  *used = pos;
  return n;
}

int parse_error(const char *path, unsigned long long key, long long D) {
  const long long row = (long long)(key >> 24), tok = (long long)((key >> 2) & 0x3fffff);
  const int kind = (int)(key & 3);
  std::string name, values;
  w2b_text_row(path, row, name, values);
  if (kind != kBadToken) {
    w2b_set_error("%s: row %lld (%s) has %s %lld values", path, row, name.c_str(), kind == kTooFew ? "fewer than" : "more than", D);
    return W2B_EIO;
  }
  const char *p = values.data(), *end = p + values.size();
  for (long long k = 0;; ++k) {  // the token the device refused
    while (p < end && w2b::text::is_space(*p)) ++p;
    const char *e = w2b::text::token_end(p, end);
    if (k == tok || e == end) {
      w2b_set_error("%s: row %lld (%s), value %lld: '%.*s' is not a number", path, row, name.c_str(), tok,
                    (int)std::min<long long>(e - p, 64), p);
      return W2B_EIO;
    }
    p = e;
  }
}

}  // namespace

int w2b_text_parse(const char *path, int64_t V, int64_t D, float *M, int64_t Dp, std::vector<std::string> &names) {
  long long chunk_bytes = kChunkBytes;
  if (const char *t = getenv("W2B_TEXT_CHUNK_BYTES")) chunk_bytes = std::max(1LL, atoll(t));  // test hook
  FILE *f = fopen(path, "rb");
  if (!f) {
    w2b_set_error("Input file not found");
    return W2B_EIO;
  }
  FileCloser closer{f};
  long long v, d;
  if (fscanf(f, "%lld", &v) != 1 || fscanf(f, "%lld", &d) != 1) {
    w2b_set_error("bad header");
    return W2B_EIO;
  }
  names.clear();
  names.reserve((size_t)V);
  unsigned long long *derr = nullptr;
  CKT(cudaMalloc(&derr, sizeof *derr));
  struct ErrFree { unsigned long long *p; ~ErrFree() { cudaFree(p); } } err_free{derr};
  CKT(cudaMemset(derr, 0xff, sizeof *derr));
  Chunk c[2];
  for (Chunk &x : c) {
    CKT(cudaStreamCreateWithFlags(&x.st, cudaStreamNonBlocking));
    CKT(cudaEventCreateWithFlags(&x.done, cudaEventDisableTiming));
    if (int rc = x.reserve(chunk_bytes, 0, D)) return rc;
  }
  long long row = 0, carry = 0;
  const char *carry_from = nullptr;
  bool eof = false;
  for (int i = 0; row < V; i ^= 1) {
    Chunk &b = c[i];
    if (b.used) CKT(cudaEventSynchronize(b.done));
    if (int rc = b.reserve(std::max<long long>(b.cap, 2 * carry), 0, D)) return rc;
    if (carry) memmove(b.h, carry_from, (size_t)carry);
    long long len = carry, used = 0;
    int n = 0;
    for (;;) {
      if (!eof) {
        const size_t got = fread(b.h + len, 1, (size_t)(b.cap - len), f);
        len += (long long)got;
        eof = len < b.cap && (feof(f) || ferror(f));
      }
      n = scan_rows(b, len, eof, V - row, names, &used);
      if (n > 0 || eof) break;
      if (int rc = b.reserve(2 * b.cap, len, D)) return rc;  // one row longer than the buffer
    }
    if (n == 0) {
      for (Chunk &x : c) CKT(cudaStreamSynchronize(x.st));
      w2b_set_error("%s: vector file truncated at word %lld", path, row);
      return W2B_EIO;
    }
    const long long bytes = b.hrows[2 * n - 1];
    CKT(cudaMemcpyAsync(b.d, b.h, (size_t)bytes, cudaMemcpyHostToDevice, b.st));
    CKT(cudaMemcpyAsync(b.drows, b.hrows, (size_t)n * 16, cudaMemcpyHostToDevice, b.st));
    text_parse_kernel<<<(unsigned)((n + kParseWarps - 1) / kParseWarps), kParseWarps * 32, 0, b.st>>>(b.d, b.drows, n, row, M, D, Dp, derr);
    CKT(cudaGetLastError());
    CKT(cudaEventRecord(b.done, b.st));
    b.used = true;
    row += n;
    carry = len - used;
    carry_from = b.h + used;
  }
  for (Chunk &x : c) CKT(cudaStreamSynchronize(x.st));
  unsigned long long key = 0;
  CKT(cudaMemcpy(&key, derr, sizeof key, cudaMemcpyDeviceToHost));
  if (key != ~0ull) return parse_error(path, key, D);
  return W2B_OK;
}

extern "C" int w2b_read_text_vectors(const char *path, int device, float *vectors, char *words, int max_word) {
  if (!path || !vectors || (words && max_word < 1)) {
    w2b_set_error("w2b_read_text_vectors: bad argument");
    return W2B_EINVAL;
  }
  return w2b_guarded("w2b_read_text_vectors", [&]() -> int {
    int kind, bits;
    int64_t V, D;
    int rc = w2b_vector_file_info(path, 0, &kind, &V, &D, &bits);
    if (rc) return rc;
    if (kind != W2B_VECTORS_TEXT) {
      w2b_set_error("%s is not a text vector file", path);
      return W2B_EIO;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device < 0 || device >= ndev) {
      w2b_set_error("no CUDA device %d: the text reader has no CPU fallback", device);
      return W2B_ECUDA;
    }
    CKT(cudaSetDevice(device));
    if (V < 1) return W2B_OK;
    float *dM = nullptr;
    CKT(cudaMalloc(&dM, (size_t)V * D * sizeof(float)));
    struct Free { float *p; ~Free() { cudaFree(p); } } fr{dM};
    CKT(cudaMemset(dM, 0, (size_t)V * D * sizeof(float)));
    std::vector<std::string> names;
    if ((rc = w2b_text_parse(path, V, D, dM, D, names))) return rc;
    CKT(cudaMemcpy(vectors, dM, (size_t)V * D * sizeof(float), cudaMemcpyDeviceToHost));
    if (words)
      for (int64_t k = 0; k < V; ++k) {
        const size_t n = std::min(names[k].size(), (size_t)max_word - 1);
        memcpy(words + k * max_word, names[k].data(), n);
        words[k * max_word + n] = 0;
      }
    return W2B_OK;
  });
}
