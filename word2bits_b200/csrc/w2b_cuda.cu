// libw2b device side: context management, kernel dispatch, C ABI (include/w2b.h).
// The product path has no CPU fallback: every entry point that computes fails with
// W2B_ECUDA when no CUDA device is usable.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "w2b.h"
#include "w2b_internal.h"
#include "w2b_kernels.cuh"
#include "w2b_warp.cuh"

using namespace w2b;

// ------------------------------------------------------------------------------ errors
static thread_local std::string g_err;
void w2b_set_error(const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
}
extern "C" const char *w2b_last_error(void) { return g_err.c_str(); }

#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      w2b_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return W2B_ECUDA;                                                                   \
    }                                                                                     \
  } while (0)

#define NEED(ptr)                                                   \
  do {                                                              \
    if (!(ptr)) {                                                   \
      w2b_set_error("%s: null %s", __func__, #ptr);                 \
      return W2B_EINVAL;                                            \
    }                                                               \
  } while (0)

// Temporary device allocation that is released on every return path.
struct DevTmp {
  void *p = nullptr;
  ~DevTmp() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
  template <class T> T *as() const { return static_cast<T *>(p); }
};

// --------------------------------------------------------------------------- NCCL (dlopen)
// Loaded lazily so that single-GPU use never touches NCCL and the library has no link-time
// dependency on it (inside a torch process the already-loaded libnccl.so.2 is reused).
typedef struct { char internal[128]; } nccl_uid;
typedef void *nccl_comm;
struct NcclApi {
  void *h = nullptr;
  int (*GetUniqueId)(nccl_uid *) = nullptr;
  int (*CommInitRank)(nccl_comm *, int, nccl_uid, int) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, nccl_comm, cudaStream_t) = nullptr;
  int (*CommDestroy)(nccl_comm) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static int nccl_load() {
  if (g_nccl.h) return W2B_OK;
  const char *names[] = {"libnccl.so.2", "libnccl.so"};
  void *h = nullptr;
  for (const char *n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) {
    w2b_set_error("NCCL not loadable: %s", dlerror());
    return W2B_ENCCL;
  }
  g_nccl.GetUniqueId = (int (*)(nccl_uid *))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (int (*)(nccl_comm *, int, nccl_uid, int))dlsym(h, "ncclCommInitRank");
  g_nccl.AllReduce =
      (int (*)(const void *, void *, size_t, int, int, nccl_comm, cudaStream_t))dlsym(h, "ncclAllReduce");
  g_nccl.CommDestroy = (int (*)(nccl_comm))dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (const char *(*)(int))dlsym(h, "ncclGetErrorString");
  g_nccl.GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
  g_nccl.GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.GroupStart || !g_nccl.GroupEnd) {
    w2b_set_error("NCCL symbols missing");
    return W2B_ENCCL;
  }
  g_nccl.h = h;
  return W2B_OK;
}
enum { kNcclUint64 = 5, kNcclFloat32 = 7, kNcclSum = 0, kNcclAvg = 4 };

// ------------------------------------------------------------------------------ plan
typedef void (*train_fn)(TrainParams);
typedef void (*apply_fn)(TrainParams, const int *, int, const int *, int, float *, double *);
typedef void (*warp_fn)(TrainParams, int, int, ApplyArgs);

// Which register-kernel instantiation a train or apply pointer is (w2b_kernel_query).
struct RegDesc {
  int wide = 0;  // 1: the __launch_bounds__(1024, 1) copy
  int vec = 0, bm = 0, reg = 0, group = 0;
};
// Which train_warp_kernel<BM, NJ, MINB, REG> instantiation a warp pointer is (w2b_kernel_query).
struct WarpDesc {
  int nj = 0, minb = 0, bm = 0, reg = 0;
};

// Which kernel trains a configuration and with what launch geometry (plan_config).
struct Plan {
  int rc = W2B_OK;      // validate(): W2B_EINVAL (message set) leaves the rest unplanned
  long long pitch = 0;  // floats per row of u / v: layer1_size rounded up to a multiple of 4 (bulk copies move 16-byte units)
  int vec = 4, ncol = 0, threads = 0;  // register kernel: floats per thread, threads with columns, threads per CTA
  int group = 9;        // register kernel: target rows in flight per step (5, 9 or 13 are instantiated)
  bool warp = false;    // production warp-per-shard kernel (csrc/w2b_warp.cuh) usable for this configuration
  int warp_k = 0, warp_qcap = 0, warps_per_sm = 0;  // ring slots per warp, job queue entries, resident warps per SM
  int warp_sen_smem = 1;  // the sentence buffer fits shared memory (else w2b_ctx::d_sen)
  size_t warp_smem = 0;
  warp_fn warp_kernel = nullptr;
  WarpDesc warp_desc;
  train_fn train = nullptr;  // register kernel (configurations the warp kernel does not take)
  apply_fn apply = nullptr;
  RegDesc train_desc, apply_desc;
  size_t reg_smem = 0;       // register kernel's dynamic shared memory: strict mode keeps a row (D floats)
};

// ------------------------------------------------------------------------------ context
struct w2b_ctx {
  w2b_config cfg;
  int nlocal = 0;  // shards owned by this context
  Plan plan;
  int *d_sen = nullptr;    // global sentence buffers: kMaxS ints per local shard (+ 1 for the parity hooks)
  int sm_count = 0;
  long long train_words = 0;
  float *d_u = nullptr, *d_v = nullptr, *d_keep = nullptr, *d_exptab = nullptr, *d_alpha = nullptr;
  float *d_base_u = nullptr, *d_base_v = nullptr;  // sync_mode 1: the tables as they were after the last exchange
  int *d_table = nullptr, *d_tokens = nullptr;
  unsigned long long *d_wca = nullptr;
  ShardState *d_shards = nullptr;
  std::vector<ShardState> h_shards;
  std::vector<long long> shard_start;
  std::vector<int> shard_first;
  const int32_t *h_ids = nullptr;  // streaming mode: caller-owned
  long long n_tokens = 0;
  bool resident = true, have_counts = false, have_corpus = false, have_tables = false;
  // streaming mode: two staging buffers (pinned host + device).  While a launch reads one, the next launch's
  // slices are gathered and copied into the other on copy_stream (speculatively: a shard advances by at least
  // the word budget and at most budget + one sentence, so its next slice is known to within `stage_margin`).
  int *h_stage[2] = {nullptr, nullptr};
  int *d_stage[2] = {nullptr, nullptr};
  long long stage_cap[2] = {0, 0};
  long long stage_margin = 4096;
  int stage_cur = 0;  // buffer the next launch reads
  struct Prefetch {
    bool valid = false;
    int buf = 0;
    long long L = 0, chunk = 0;
    std::vector<long long> begin, limit;  // per local shard: global index of the slice's first token / its end
    std::vector<int> eof;
  } pf;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_copy = nullptr;
  unsigned long long *d_scratch = nullptr;  // 64 B: [0] own words since the last sync (all-reduced), [1] counter at the last sync
  cudaEvent_t ev_s0 = nullptr, ev_s1 = nullptr;
  float last_sync_ms = 0.f;
  nccl_comm comm = nullptr;
  int rank = 0, nranks = 1;
  long long wca_at_sync = 0;
};

static long long pitch_of(long long D) { return (D + 3) & ~3LL; }
static size_t table_elems(const w2b_ctx *c) { return (size_t)c->cfg.vocab_size * (size_t)c->plan.pitch; }

static void lcg_tables(unsigned long long *JA, unsigned long long *JC, unsigned long long *PA,
                       unsigned long long *PC) {
  JA[0] = 1;
  JC[0] = 0;
  for (int k = 1; k <= 64; ++k) {
    JA[k] = JA[k - 1] * kLcgA;
    JC[k] = JC[k - 1] * kLcgA + kLcgC;
  }
  PA[0] = kLcgA;
  PC[0] = kLcgC;
  for (int j = 1; j < 64; ++j) {
    PA[j] = PA[j - 1] * PA[j - 1];
    PC[j] = PA[j - 1] * PC[j - 1] + PC[j - 1];
  }
}

// ------------------------------------------------------------------------ kernel dispatch
static int bm_of(int bits) { return (bits == 0 || bits == 1 || bits == 2) ? bits : 9; }

// Strict mode, kernel = 1 and rows wider than 2048 floats run the register kernel; the warp kernel is not
// instantiated beyond 2048.  validate() refuses the widths the register kernel cannot take by this predicate;
// plan_config also sends a mode other than W2B_MODE_FAST (which validate() does not check) to the register kernel.
static bool needs_register_kernel(const w2b_config &cfg) {
  return cfg.mode == W2B_MODE_STRICT || cfg.kernel == 1 || cfg.layer1_size > 2048;
}

// ---- register kernel (csrc/w2b_kernels.cuh)
struct RegKernel {
  train_fn train;
  apply_fn apply;
  RegDesc t, a;
};
// Instantiations compiled for speed.  The apply hook runs G = 9 whatever the configuration's group.
template <int VEC, int BM, bool REG, int G>
static RegKernel reg_tuned() {
  return {train_shards_kernel<VEC, BM, REG, false, G>, apply_position_kernel<VEC, BM, REG, false, 9>,
          {0, VEC, BM, REG, G}, {0, VEC, BM, REG, 9}};
}
// __launch_bounds__(1024, 1) instantiations: bit level decided at run time, G = 5 (strict mode: 1).
template <int VEC, bool REG, bool STRICT>
static RegKernel reg_wide() {
  constexpr int G = STRICT ? 1 : 5;
  return {train_shards_wide_kernel<VEC, 9, REG, STRICT, G>, apply_position_wide_kernel<VEC, 9, REG, STRICT, G>,
          {1, VEC, 9, REG, G}, {1, VEC, 9, REG, G}};
}
template <int BM>
static RegKernel reg_tuned_vec4(bool reg, int group) {
  if (reg) return reg_tuned<4, BM, true, 9>();
  if (group == 5) return reg_tuned<4, BM, false, 5>();
  if (group == 13) return reg_tuned<4, BM, false, 13>();
  return reg_tuned<4, BM, false, 9>();
}
// Strict mode always runs the wide instantiations; fast mode runs them when `wide` (plan_register_kernel), else the
// speed-tuned ones, which compile the bit level in for VEC = 4 and run G = 9 with -reg or VEC = 1.
static RegKernel register_kernel(const w2b_config &cfg, int vec, int group, bool wide) {
  const bool reg = cfg.reg != 0.f;
  if (cfg.mode == W2B_MODE_STRICT) return vec == 4 ? reg_wide<4, true, true>() : reg_wide<1, true, true>();
  if (wide) {
    if (vec == 1) return reg ? reg_wide<1, true, false>() : reg_wide<1, false, false>();
    return reg ? reg_wide<4, true, false>() : reg_wide<4, false, false>();
  }
  if (vec == 1) return reg ? reg_tuned<1, 9, true, 9>() : reg_tuned<1, 9, false, 9>();
  switch (bm_of(cfg.bitlevel)) {
    case 0: return reg_tuned_vec4<0>(reg, group);
    case 1: return reg_tuned_vec4<1>(reg, group);
    case 2: return reg_tuned_vec4<2>(reg, group);
    default: return reg_tuned_vec4<9>(reg, group);
  }
}

// ---- warp-per-shard kernel (csrc/w2b_warp.cuh)
// Warps (= 1-warp CTAs) per SM that train_warp_kernel<BM, NJ, MINB, REG> is compiled for (MINB) and plan_warp sizes
// shared memory for.  Multiples of 4 because the register file is split over the four SM sub-partitions: 12 warps ->
// 168 registers per thread, 16 -> 128, 20 -> 96, 24 -> 80.  Rows wider than 1024 floats (the reference publishes
// 1200-dimensional vectors): 8 warps (216 registers) up to 1536 floats, 4 warps (248 registers) up to 2048.  -reg
// keeps the raw row live: one step lower occupancy, at least 4 warps.
static constexpr int warp_minb(int nj, bool reg) {
  const int minb = nj >= 13 ? 4 : (nj >= 9 ? 8 : (nj >= 5 ? 12 : (nj >= 3 ? 16 : (nj == 2 ? 20 : 24))));
  return reg ? std::max(4, minb - 4) : minb;
}
// Bit level compiled in (BM = 0, 1, 2) up to 1536 floats without -reg; decided at run time (BM = 9) beyond and with
// -reg, for fewer instantiations.
static constexpr int warp_bm(int bm, bool reg, int nj) { return reg || nj >= 13 ? 9 : bm; }
// One instantiation per row width of NJ = I + 1 = 1 ... 16 column groups (32 float4s each), with its descriptor.
template <int BM, bool REG, int... I>
static warp_fn warp_kernel_of(int nj, std::integer_sequence<int, I...>, WarpDesc *desc) {
  static const warp_fn by_nj[] = {train_warp_kernel<warp_bm(BM, REG, I + 1), I + 1, warp_minb(I + 1, REG), REG>...};
  static const WarpDesc descs[] = {{I + 1, warp_minb(I + 1, REG), warp_bm(BM, REG, I + 1), REG}...};
  *desc = descs[nj - 1];
  return by_nj[nj - 1];
}
static warp_fn warp_kernel(const w2b_config &cfg, int nj, WarpDesc *desc) {
  const auto widths = std::make_integer_sequence<int, 16>();
  if (cfg.reg != 0.f) return warp_kernel_of<9, true>(nj, widths, desc);
  switch (bm_of(cfg.bitlevel)) {
    case 0: return warp_kernel_of<0, false>(nj, widths, desc);
    case 1: return warp_kernel_of<1, false>(nj, widths, desc);
    case 2: return warp_kernel_of<2, false>(nj, widths, desc);
    default: return warp_kernel_of<9, false>(nj, widths, desc);
  }
}

// Geometry: as many ring slots as the warp's share of the SM's 228 KB holds (each resident CTA also costs 1 KB of
// reserved shared memory); at least 3 (one row being worked on, one draining, one in flight).
static void plan_warp(const w2b_config &cfg, Plan *pl) {
  const int nj = (int)((pl->pitch / 4 + 31) / 32);  // <= 16: D <= 2048
  const int qcap = warp_queue_capacity(cfg.window, cfg.negative);
  // the sentence buffer (4000 B) moves to global memory when keeping it in shared memory would cost ring slots
  // below 4 (wide rows); a job queue too large for the warp's share of shared memory (very wide windows) is paid
  // for with fewer resident warps (the kernel compiled for `minb` warps runs at any lower occupancy)
  int sen_smem = 1, K = 0, wps = warp_minb(nj, cfg.reg != 0.f);
  for (; wps >= 4; wps -= 4) {
    const size_t budget = (size_t)(228 * 1024) / wps - 1024;
    sen_smem = 1;
    K = cfg.slots > 0 ? std::min(cfg.slots, 32) : 16;
    while (K >= 3 && warp_layout(pl->pitch, K, qcap, sen_smem).total > budget) --K;
    if (K < 4) {
      int K2 = cfg.slots > 0 ? std::min(cfg.slots, 32) : 16;
      while (K2 >= 3 && warp_layout(pl->pitch, K2, qcap, 0).total > budget) --K2;
      if (K2 > K) { K = K2; sen_smem = 0; }
    }
    if (K >= 3) break;
  }
  if (wps < 4 || K < 3) return;
  pl->warp = true;
  pl->warp_k = K;
  pl->warp_qcap = qcap;
  pl->warps_per_sm = wps;
  pl->warp_sen_smem = sen_smem;
  pl->warp_smem = warp_layout(pl->pitch, K, qcap, sen_smem).total;
  pl->warp_kernel = warp_kernel(cfg, nj, &pl->warp_desc);
}

// Register kernel (configurations the warp kernel does not take): pl->threads threads per CTA.  The instantiations
// compiled for speed run when they can take that many threads; otherwise the wide ones (__launch_bounds__(1024)).
// A width that not even those can serve is refused here, at creation, instead of failing at its first launch.
static int plan_register_kernel(const w2b_config &cfg, Plan *pl) {
  const RegKernel wide = register_kernel(cfg, pl->vec, pl->group, true);
  cudaFuncAttributes fa;
  if (cfg.mode != W2B_MODE_STRICT) {
    CK(cudaFuncGetAttributes(&fa, (const void *)pl->train));
    if (pl->threads > fa.maxThreadsPerBlock) { pl->train = wide.train; pl->train_desc = wide.t; }
    CK(cudaFuncGetAttributes(&fa, (const void *)pl->apply));
    if (pl->threads > fa.maxThreadsPerBlock) { pl->apply = wide.apply; pl->apply_desc = wide.a; }
  }
  for (const void *fn : {(const void *)pl->train, (const void *)pl->apply}) {
    CK(cudaFuncGetAttributes(&fa, fn));
    if (pl->threads > fa.maxThreadsPerBlock) {
      w2b_set_error("layer1_size %lld needs %d threads per CTA; the register kernel takes at most %d for this "
                    "configuration", (long long)cfg.layer1_size, pl->threads, fa.maxThreadsPerBlock);
      return W2B_EINVAL;
    }
  }
  return W2B_OK;
}

static TrainParams base_params(const w2b_ctx *c) {
  TrainParams p;
  memset(&p, 0, sizeof p);
  p.u = c->d_u;
  p.v = c->d_v;
  p.table = c->d_table;
  p.keep_thr = c->d_keep;
  p.exptab = c->d_exptab;
  p.tokens = c->d_tokens;
  p.shards = c->d_shards;
  p.alpha = c->d_alpha;
  p.wca = c->d_wca;
  p.D = c->cfg.layer1_size;
  p.pitch = c->plan.pitch;
  p.V = c->cfg.vocab_size;
  p.ncol = c->plan.ncol;
  p.window = c->cfg.window;
  p.negative = c->cfg.negative;
  p.bitlevel = c->cfg.bitlevel;
  p.sample = c->cfg.sample;
  p.reg = c->cfg.reg;
  p.starting_alpha = c->cfg.alpha;
  p.alpha_denom = (float)(c->cfg.iter * c->train_words + 1);  // :391
  p.shard_word_limit = c->train_words / c->cfg.num_shards;    // :414
  p.word_budget = 0;
  p.max_iters = -1;
  p.shard_base = 0;
  p.train = 1;
  p.serial = c->cfg.prefetch ? 0 : 1;  // default: the positions of a shard strictly one after another
  p.wca_scale = c->nranks;
  p.sen = c->d_sen;
  return p;
}

// ---------------------------------------------------------------------------- lifecycle
extern "C" int w2b_device_count(int *n) {
  NEED(n);
  int k = 0;
  cudaError_t e = cudaGetDeviceCount(&k);
  if (e != cudaSuccess) {
    *n = 0;
    w2b_set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e));
    return W2B_ECUDA;
  }
  *n = k;
  return W2B_OK;
}

static int validate(const w2b_config *c) {
  if (c->vocab_size < 2) { w2b_set_error("vocab_size must be >= 2"); return W2B_EINVAL; }
  if (c->layer1_size < 1) { w2b_set_error("layer1_size must be >= 1"); return W2B_EINVAL; }
  if (c->window < 1 || c->window > W2B_MAX_WINDOW) { w2b_set_error("window must be in [1,%d]", W2B_MAX_WINDOW); return W2B_EINVAL; }
  if (c->negative < 0 || c->negative > W2B_MAX_NEGATIVE) { w2b_set_error("negative must be in [0,%d]", W2B_MAX_NEGATIVE); return W2B_EINVAL; }
  if (c->bitlevel > 24) { w2b_set_error("bitlevel must be <= 24"); return W2B_EINVAL; }
  if (c->num_shards < 1) { w2b_set_error("num_shards must be >= 1"); return W2B_EINVAL; }
  if (c->iter < 1) { w2b_set_error("iter must be >= 1"); return W2B_EINVAL; }
  if (c->plain_store != 0) { w2b_set_error("plain_store: the racy load/add/store variant was removed; must be 0"); return W2B_EINVAL; }
  const long long D = c->layer1_size;
  // production kernel: any D <= 2048 (rows padded to whole float4s); register kernel: D <= 4096 when divisible by 4
  // (a thread per float4), else D <= 1024 (a thread per float) — strict mode and kernel = 1 always run the latter.
  // Every width accepted here launches (the wide instantiations, plan_register_kernel).
  if (D > 4096 || (needs_register_kernel(*c) && D % 4 != 0 && D > 1024)) {
    w2b_set_error("layer1_size %lld unsupported (at most 4096; in strict mode, with kernel 1 and above 2048 it must "
                  "also be divisible by 4 when above 1024)", D);
    return W2B_EINVAL;
  }
  return W2B_OK;
}

// Everything the launches of a configuration depend on, without a CUDA call (w2b_warp_plan_query runs it on hosts
// without a GPU).  The register kernel's instantiations are the speed-tuned ones in fast mode until
// plan_register_kernel has checked them against the device.
static Plan plan_config(const w2b_config &cfg) {
  Plan pl;
  pl.rc = validate(&cfg);
  if (pl.rc) return pl;
  const long long D = cfg.layer1_size;
  pl.pitch = pitch_of(D);
  pl.vec = (D % 4 == 0) ? 4 : 1;
  pl.ncol = (int)((D + pl.vec - 1) / pl.vec);
  pl.threads = std::max(32, (pl.ncol + 31) / 32 * 32);
  pl.group = cfg.group ? cfg.group : (cfg.negative + 1 > 9 ? 13 : (cfg.negative + 1 > 5 ? 9 : 5));
  if (pl.group != 5 && pl.group != 9 && pl.group != 13) pl.group = 9;  // register kernel instantiations
  const RegKernel rk = register_kernel(cfg, pl.vec, pl.group, false);
  pl.train = rk.train;
  pl.apply = rk.apply;
  pl.train_desc = rk.t;
  pl.apply_desc = rk.a;
  pl.reg_smem = cfg.mode == W2B_MODE_STRICT ? (size_t)D * sizeof(float) : 0;
  if (cfg.mode == W2B_MODE_FAST && !needs_register_kernel(cfg)) plan_warp(cfg, &pl);
  return pl;
}

extern "C" int w2b_suggest_shards(const w2b_config *cfg, int *out) {
  NEED(cfg);
  NEED(out);
  Plan pl = plan_config(*cfg);
  if (pl.rc) return pl.rc;
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  int per_sm = 0;
  if (pl.warp) {
    CK(cudaFuncSetAttribute(pl.warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.warp_smem));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pl.warp_kernel, 32, pl.warp_smem));
  } else {
    const int rc = plan_register_kernel(*cfg, &pl);
    if (rc) return rc;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pl.train, pl.threads, pl.reg_smem));
  }
  *out = std::max(1, per_sm) * prop.multiProcessorCount;
  return W2B_OK;
}

// ---- host-only views of the path's host logic (no CUDA call: usable, and tested, without a GPU)
extern "C" int w2b_warp_plan_query(const w2b_config *cfg, w2b_warp_plan *out) {
  if (!cfg || !out) { w2b_set_error("null argument"); return W2B_EINVAL; }
  const Plan pl = plan_config(*cfg);
  if (pl.rc) return pl.rc;
  memset(out, 0, sizeof *out);
  out->warp = pl.warp ? 1 : 0;
  if (!pl.warp) return W2B_OK;
  out->slots = pl.warp_k;
  out->sentence_in_smem = pl.warp_sen_smem;
  out->queue_entries = pl.warp_qcap;
  out->warps_per_sm = pl.warps_per_sm;
  out->smem_bytes = (int64_t)pl.warp_smem;
  return W2B_OK;
}

extern "C" int w2b_kernel_query(w2b_ctx *c, w2b_kernel_info *out) {
  NEED(c);
  NEED(out);
  const Plan &pl = c->plan;
  memset(out, 0, sizeof *out);
  if (pl.warp) {
    out->warp = 1;
    out->nj = pl.warp_desc.nj;
    out->minb = pl.warp_desc.minb;
    out->bm = pl.warp_desc.bm;
    out->reg = pl.warp_desc.reg;
    return W2B_OK;
  }
  out->threads = pl.threads;
  out->vec = pl.train_desc.vec;
  out->bm = pl.train_desc.bm;
  out->reg = pl.train_desc.reg;
  out->wide = pl.train_desc.wide;
  out->group = pl.train_desc.group;
  out->apply_wide = pl.apply_desc.wide;
  out->apply_bm = pl.apply_desc.bm;
  out->apply_group = pl.apply_desc.group;
  return W2B_OK;
}

extern "C" int w2b_host_lcg_tables(uint64_t *ja, uint64_t *jc, uint64_t *pa, uint64_t *pc) {
  if (!ja || !jc || !pa || !pc) { w2b_set_error("null argument"); return W2B_EINVAL; }
  unsigned long long JA[65], JC[65], PA[64], PC[64];
  lcg_tables(JA, JC, PA, PC);
  for (int i = 0; i < 65; ++i) { ja[i] = JA[i]; jc[i] = JC[i]; }
  for (int i = 0; i < 64; ++i) { pa[i] = PA[i]; pc[i] = PC[i]; }
  return W2B_OK;
}

static int create_impl(const w2b_config *cfg, w2b_ctx **out);
extern "C" int w2b_create(const w2b_config *cfg, w2b_ctx **out) {
  NEED(out);
  *out = nullptr;
  NEED(cfg);
  w2b_ctx *c = nullptr;
  const int rc = w2b_guarded("w2b_create", [&] { return create_impl(cfg, &c); });
  if (rc) {
    const std::string keep = w2b_last_error();  // destroy must not clobber the message
    if (c) w2b_destroy(c);
    w2b_set_error("%s", keep.c_str());
    return rc;
  }
  *out = c;
  return W2B_OK;
}

static int create_impl(const w2b_config *cfg, w2b_ctx **out) {
  *out = nullptr;
  const Plan plan = plan_config(*cfg);
  if (plan.rc) return plan.rc;
  int ndev = 0;
  int rc = w2b_device_count(&ndev);
  if (rc) return rc;
  if (ndev == 0 || cfg->device < 0 || cfg->device >= ndev) {
    w2b_set_error("no CUDA device %d (found %d): this library has no CPU fallback", cfg->device, ndev);
    return W2B_ECUDA;
  }
  w2b_ctx *c = new w2b_ctx();
  *out = c;  // owned by the caller from here on (destroyed there if anything below fails)
  c->cfg = *cfg;
  if (c->cfg.shard_end <= c->cfg.shard_begin) {
    c->cfg.shard_begin = 0;
    c->cfg.shard_end = cfg->num_shards;
  }
  if (c->cfg.shard_end > cfg->num_shards) {
    w2b_set_error("shard range exceeds num_shards");
    return W2B_EINVAL;
  }
  c->nlocal = c->cfg.shard_end - c->cfg.shard_begin;
  c->plan = plan;
  CK(cudaSetDevice(cfg->device));
  if (!c->plan.warp) {
    rc = plan_register_kernel(*cfg, &c->plan);
    if (rc) return rc;
  }
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  c->sm_count = prop.multiProcessorCount;
  CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  CK(cudaEventCreate(&c->ev0));
  CK(cudaEventCreate(&c->ev1));
  CK(cudaEventCreateWithFlags(&c->ev_copy, cudaEventDisableTiming));
  unsigned long long JA[65], JC[65], PA[64], PC[64];
  lcg_tables(JA, JC, PA, PC);
  CK(cudaMemcpyToSymbol(c_JA, JA, sizeof JA));
  CK(cudaMemcpyToSymbol(c_JC, JC, sizeof JC));
  CK(cudaMemcpyToSymbol(c_PA, PA, sizeof PA));
  CK(cudaMemcpyToSymbol(c_PC, PC, sizeof PC));
  const size_t n = table_elems(c);
  CK(cudaMalloc(&c->d_u, n * sizeof(float)));
  CK(cudaMalloc(&c->d_v, n * sizeof(float)));
  if (c->plan.pitch != cfg->layer1_size) {  // padding columns start (and, in v, stay) at zero
    CK(cudaMemset(c->d_u, 0, n * sizeof(float)));
    CK(cudaMemset(c->d_v, 0, n * sizeof(float)));
  }
  CK(cudaMalloc(&c->d_keep, cfg->vocab_size * sizeof(float)));
  CK(cudaMalloc(&c->d_exptab, kExpN * sizeof(float)));
  CK(cudaMalloc(&c->d_alpha, sizeof(float)));
  CK(cudaMalloc(&c->d_wca, sizeof(unsigned long long)));
  CK(cudaMalloc(&c->d_table, (size_t)W2B_TABLE_SIZE * sizeof(int)));
  CK(cudaMalloc(&c->d_shards, sizeof(ShardState) * c->nlocal));
  CK(cudaMemset(c->d_wca, 0, sizeof(unsigned long long)));
  CK(cudaMemcpy(c->d_alpha, &cfg->alpha, sizeof(float), cudaMemcpyHostToDevice));
  c->h_shards.assign(c->nlocal, ShardState());
  {  // expTable (:614-618) does not depend on the corpus: ready as soon as the context exists
    float t[kExpN];
    w2b_exptable(t);
    CK(cudaMemcpy(c->d_exptab, t, sizeof t, cudaMemcpyHostToDevice));
    CK(cudaMemcpyToSymbol(c_exptab, t, sizeof t));
  }
  CK(cudaMalloc(&c->d_scratch, 64));
  CK(cudaMemset(c->d_scratch, 0, 64));
  if (c->plan.warp && !c->plan.warp_sen_smem) CK(cudaMalloc(&c->d_sen, sizeof(int) * (size_t)kMaxS * (c->nlocal + 1)));
  CK(cudaEventCreate(&c->ev_s0));
  CK(cudaEventCreate(&c->ev_s1));
  // the memsets above ran on the legacy stream, which the context's non-blocking streams do not wait for
  CK(cudaDeviceSynchronize());
  return W2B_OK;
}

extern "C" int w2b_destroy(w2b_ctx *c) {
  if (!c) return W2B_OK;
  cudaSetDevice(c->cfg.device);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  cudaFree(c->d_u); cudaFree(c->d_v); cudaFree(c->d_keep); cudaFree(c->d_exptab);
  cudaFree(c->d_base_u); cudaFree(c->d_base_v);
  cudaFree(c->d_alpha); cudaFree(c->d_wca); cudaFree(c->d_table); cudaFree(c->d_tokens);
  cudaFree(c->d_shards);
  cudaFree(c->d_scratch);
  cudaFree(c->d_sen);
  if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
  for (int b = 0; b < 2; ++b) {
    if (c->h_stage[b]) cudaFreeHost(c->h_stage[b]);
    cudaFree(c->d_stage[b]);
  }
  if (c->ev0) cudaEventDestroy(c->ev0);
  if (c->ev1) cudaEventDestroy(c->ev1);
  if (c->ev_copy) cudaEventDestroy(c->ev_copy);
  if (c->ev_s0) cudaEventDestroy(c->ev_s0);
  if (c->ev_s1) cudaEventDestroy(c->ev_s1);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  delete c;
  return W2B_OK;
}

// ------------------------------------------------------------------------------- tables
static int w2b_set_vocab_counts_impl(w2b_ctx *c, const int64_t *cn, int64_t V, int64_t train_words);
extern "C" int w2b_set_vocab_counts(w2b_ctx *c, const int64_t *cn, int64_t V, int64_t train_words) {
  return w2b_guarded("w2b_set_vocab_counts", [&] { return w2b_set_vocab_counts_impl(c, cn, V, train_words); });
}
static int w2b_set_vocab_counts_impl(w2b_ctx *c, const int64_t *cn, int64_t V, int64_t train_words) {
  NEED(c);
  NEED(cn);
  if (V != c->cfg.vocab_size) { w2b_set_error("V mismatch"); return W2B_EINVAL; }
  if (train_words < 1) { w2b_set_error("train_words must be >= 1"); return W2B_EINVAL; }
  CK(cudaSetDevice(c->cfg.device));
  c->train_words = train_words;
  // sub-sampling threshold `ran` (:403-404), float32 throughout
  std::vector<float> keep(V);
  w2b_keep_thresholds(cn, V, train_words, c->cfg.sample, keep.data());
  CK(cudaMemcpyAsync(c->d_keep, keep.data(), V * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  // unigram boundaries (:112-128) with the host libm pow(); the device expands them
  std::vector<int> start(V + 1);
  w2b_unigram_bounds(cn, V, start.data());
  DevTmp d_start;
  CK(d_start.alloc((V + 1) * sizeof(int)));
  CK(cudaMemcpyAsync(d_start.p, start.data(), (V + 1) * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  fill_table_kernel<<<(W2B_TABLE_SIZE + 255) / 256, 256, 0, c->stream>>>(c->d_table, d_start.as<int>(), (int)V);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  c->have_counts = true;
  return W2B_OK;
}

extern "C" int w2b_init_tables(w2b_ctx *c) {
  NEED(c);
  CK(cudaSetDevice(c->cfg.device));
  const long long n = c->cfg.vocab_size * c->cfg.layer1_size;
  const long long threads = (2 * n + 3) / 4;
  init_net_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, c->stream>>>(c->d_v, c->d_u, n, c->cfg.layer1_size, c->plan.pitch);
  CK(cudaGetLastError());
  float t[kExpN];
  w2b_exptable(t);
  CK(cudaMemcpyAsync(c->d_exptab, t, sizeof t, cudaMemcpyHostToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  c->have_tables = true;
  return W2B_OK;
}

static int w2b_set_corpus_impl(w2b_ctx *c, const int32_t *ids, int64_t n, const int64_t *shard_start,
                              const int32_t *shard_first, int resident);
extern "C" int w2b_set_corpus(w2b_ctx *c, const int32_t *ids, int64_t n, const int64_t *shard_start,
                              const int32_t *shard_first, int resident) {
  return w2b_guarded("w2b_set_corpus", [&] { return w2b_set_corpus_impl(c, ids, n, shard_start, shard_first, resident); });
}
static int w2b_set_corpus_impl(w2b_ctx *c, const int32_t *ids, int64_t n, const int64_t *shard_start,
                              const int32_t *shard_first, int resident) {
  NEED(c);
  NEED(shard_start);
  NEED(shard_first);
  if (n < 0 || (n > 0 && !ids)) { w2b_set_error("w2b_set_corpus: bad token stream"); return W2B_EINVAL; }
  // the kernels use token ids as row indices of u / v and shard starts as stream offsets: check them once
  for (int i = c->cfg.shard_begin; i < c->cfg.shard_end; ++i) {
    const int64_t lo = shard_first[i] >= 0 ? 1 : 0;
    if (shard_start[i] < lo || shard_start[i] > n || shard_first[i] >= c->cfg.vocab_size) {
      w2b_set_error("w2b_set_corpus: shard %d starts at %lld (first token %d) outside the stream of %lld tokens", i,
                    (long long)shard_start[i], (int)shard_first[i], (long long)n);
      return W2B_EINVAL;
    }
  }
  {
    const uint32_t V = (uint32_t)c->cfg.vocab_size;
    uint32_t bad = 0;
    for (int64_t i = 0; i < n; ++i) bad |= (uint32_t)((uint32_t)ids[i] >= V);
    if (bad) { w2b_set_error("w2b_set_corpus: token id outside [0, %u)", V); return W2B_EINVAL; }
  }
  CK(cudaSetDevice(c->cfg.device));
  c->n_tokens = n;
  c->resident = resident != 0;
  c->shard_start.assign(shard_start + c->cfg.shard_begin, shard_start + c->cfg.shard_end);
  c->shard_first.assign(shard_first + c->cfg.shard_begin, shard_first + c->cfg.shard_end);
  if (c->d_tokens) { cudaFree(c->d_tokens); c->d_tokens = nullptr; }
  if (c->copy_stream) CK(cudaStreamSynchronize(c->copy_stream));
  c->pf.valid = false;  // slices prefetched from the previous stream are void
  if (c->resident) {
    CK(cudaMalloc(&c->d_tokens, std::max<int64_t>(n, 1) * sizeof(int)));
    CK(cudaMemcpyAsync(c->d_tokens, ids, n * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    c->h_ids = nullptr;
  } else {
    c->h_ids = ids;
  }
  c->have_corpus = true;
  return w2b_epoch_begin(c);
}

// Local shard i's state at the start of an epoch.
static ShardState shard_epoch_start(const w2b_ctx *c, int i) {
  ShardState s;
  memset(&s, 0, sizeof s);
  s.rng = (unsigned long long)(long long)(c->cfg.shard_begin + i);  // :368
  const bool ovr = c->shard_first[i] >= 0;
  s.cursor = ovr ? c->shard_start[i] - 1 : c->shard_start[i];
  s.ovr_idx = ovr ? c->shard_start[i] - 1 : -2;
  s.ovr_tok = ovr ? c->shard_first[i] : -1;
  s.limit = c->n_tokens;
  s.limit_is_eof = 1;
  return s;
}

extern "C" int w2b_epoch_begin(w2b_ctx *c) {
  NEED(c);
  if (!c->have_corpus) { w2b_set_error("set_corpus first"); return W2B_ESTATE; }
  CK(cudaSetDevice(c->cfg.device));
  for (int i = 0; i < c->nlocal; ++i) c->h_shards[i] = shard_epoch_start(c, i);
  CK(cudaMemcpyAsync(c->d_shards, c->h_shards.data(), sizeof(ShardState) * c->nlocal, cudaMemcpyHostToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return W2B_OK;
}

// ------------------------------------------------------------------------------ training
static void sum_shards(const std::vector<ShardState> &s, w2b_step_stats *o) {
  memset(o, 0, sizeof *o);
  for (const ShardState &x : s) {
    o->loss += x.loss;
    o->words += x.word_count;
    o->positions += (int64_t)x.n_pos;
    o->context_rows += (int64_t)x.n_ctx;
    o->target_rows += (int64_t)x.n_tgt;
    o->shards_done += x.done;
  }
}

// ---- streaming mode (host token buffers)
static int stage_reserve(w2b_ctx *c, int b, long long need) {
  if (need <= c->stage_cap[b]) return W2B_OK;
  c->stage_cap[b] = 0;
  if (c->h_stage[b]) { cudaFreeHost(c->h_stage[b]); c->h_stage[b] = nullptr; }
  if (c->d_stage[b]) { cudaFree(c->d_stage[b]); c->d_stage[b] = nullptr; }
  CK(cudaMallocHost(&c->h_stage[b], need * sizeof(int)));
  CK(cudaMalloc(&c->d_stage[b], need * sizeof(int)));
  c->stage_cap[b] = need;
  return W2B_OK;
}

// Gathers, for every unfinished shard, the L tokens from `begin[i]` into staging buffer b (slice i at i*L) and
// starts the H2D copy on `stream`.  Host threads: w2b_gather_slices (tested on the CPU).
static int stage_gather(w2b_ctx *c, int b, long long L, const std::vector<long long> &begin, cudaStream_t stream,
                        std::vector<long long> &limit, std::vector<int> &eof, w2b_step_stats *acc) {
  const long long need = L * c->nlocal;
  int rc = stage_reserve(c, b, need);
  if (rc) return rc;
  std::vector<long long> xlate(c->nlocal);
  std::vector<int> done(c->nlocal);
  limit.assign(c->nlocal, 0);
  eof.assign(c->nlocal, 0);
  for (int i = 0; i < c->nlocal; ++i) done[i] = c->h_shards[i].done;
  w2b_gather_slices(c->h_ids, c->n_tokens, L, c->nlocal, begin.data(), done.data(), c->h_stage[b], xlate.data(),
                    limit.data(), eof.data(), 0);
  CK(cudaMemcpyAsync(c->d_stage[b], c->h_stage[b], need * sizeof(int), cudaMemcpyHostToDevice, stream));
  acc->h2d_bytes += need * (long long)sizeof(int);
  return W2B_OK;
}

// Points the shard states at the slices of this launch: the prefetched buffer when it covers every unfinished
// shard's next `chunk + margin` tokens, else a synchronous gather from the cursors.
static int stage_acquire(w2b_ctx *c, long long chunk, w2b_step_stats *acc) {
  w2b_ctx::Prefetch &pf = c->pf;
  bool use = pf.valid && pf.chunk == chunk;
  if (use)
    for (int i = 0; i < c->nlocal && use; ++i) {
      const ShardState &sh = c->h_shards[i];
      if (sh.done) continue;
      const long long cur = std::max<long long>(sh.cursor, 0);
      const long long want_end = std::min<long long>(cur + chunk + c->stage_margin, c->n_tokens);
      if (cur < pf.begin[i] || want_end > pf.limit[i]) use = false;
    }
  if (use) {
    CK(cudaStreamWaitEvent(c->stream, c->ev_copy, 0));
    c->stage_cur = pf.buf;
    for (int i = 0; i < c->nlocal; ++i) {
      ShardState &sh = c->h_shards[i];
      if (sh.done) continue;
      sh.xlate = pf.begin[i] - (long long)i * pf.L;
      sh.limit = pf.limit[i];
      sh.limit_is_eof = pf.eof[i];
    }
  } else {
    if (pf.valid) CK(cudaStreamSynchronize(c->copy_stream));  // its buffer may be the one re-used below
    const long long L = chunk + c->stage_margin;
    std::vector<long long> begin(c->nlocal), limit;
    std::vector<int> eof;
    for (int i = 0; i < c->nlocal; ++i) begin[i] = std::max<long long>(c->h_shards[i].cursor, 0);
    int rc = stage_gather(c, c->stage_cur, L, begin, c->stream, limit, eof, acc);
    if (rc) return rc;
    for (int i = 0; i < c->nlocal; ++i) {
      ShardState &sh = c->h_shards[i];
      if (sh.done) continue;
      sh.xlate = begin[i] - (long long)i * L;
      sh.limit = limit[i];
      sh.limit_is_eof = eof[i];
    }
  }
  pf.valid = false;
  CK(cudaMemcpyAsync(c->d_shards, c->h_shards.data(), sizeof(ShardState) * c->nlocal, cudaMemcpyHostToDevice,
                     c->stream));
  acc->h2d_bytes += (long long)sizeof(ShardState) * c->nlocal;
  return W2B_OK;
}

// While the launch that was just enqueued runs: gather and upload what the NEXT launch of the same budget will
// read.  A shard that starts at cursor c ends this launch in [c + chunk, c + chunk + one sentence], so the slice
// [c + chunk, c + 2*chunk + 2*margin) covers the next launch's cursor .. cursor + chunk + margin.
static int stage_prefetch(w2b_ctx *c, long long chunk, w2b_step_stats *acc) {
  w2b_ctx::Prefetch &pf = c->pf;
  pf.valid = false;
  pf.buf = c->stage_cur ^ 1;
  pf.chunk = chunk;
  pf.L = chunk + 2 * c->stage_margin;
  pf.begin.assign(c->nlocal, 0);
  for (int i = 0; i < c->nlocal; ++i) pf.begin[i] = std::max<long long>(c->h_shards[i].cursor, 0) + chunk;
  int rc = stage_gather(c, pf.buf, pf.L, pf.begin, c->copy_stream, pf.limit, pf.eof, acc);
  if (rc) return rc;
  CK(cudaEventRecord(c->ev_copy, c->copy_stream));
  pf.valid = true;
  return W2B_OK;
}

// Launches the warp kernel: one warp (a 32-thread CTA) per local shard, or for a parity hook a single one that uses
// the hooks' own sentence buffer, so that no shard's sentence is overwritten.
static int launch_warp(const w2b_ctx *c, TrainParams p, const ApplyArgs &ap, bool hook) {
  const Plan &pl = c->plan;
  const warp_fn fn = pl.warp_kernel;
  CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.warp_smem));
  if (hook && p.sen) p.sen += (size_t)kMaxS * c->nlocal;
  fn<<<hook ? 1 : c->nlocal, 32, pl.warp_smem, c->stream>>>(p, pl.warp_k, pl.warp_qcap | (pl.warp_sen_smem << 31), ap);
  return W2B_OK;
}

// Launches the register kernel's train or apply instantiation: `blocks` CTAs of plan.threads threads.
template <class Fn, class... Args>
static int launch_register(const w2b_ctx *c, Fn fn, int blocks, Args... args) {
  const size_t smem = c->plan.reg_smem;
  if (smem > 48 * 1024) CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  fn<<<blocks, c->plan.threads, smem, c->stream>>>(args...);
  return W2B_OK;
}

// Enqueues the training kernel(s) of one launch on the context's stream (between ev0 and ev1).
static int launch_enqueue(w2b_ctx *c, TrainParams p, w2b_step_stats *acc) {
  CK(cudaEventRecord(c->ev0, c->stream));
  int launches = 1, rc = W2B_OK;
  if (c->plan.warp) {  // production path
    rc = launch_warp(c, p, ApplyArgs{}, false);
  } else if (c->cfg.mode == W2B_MODE_STRICT) {
    launches = 0;
    for (int i = 0; i < c->nlocal && !rc; ++i) {  // shards one after another, like joined threads
      p.shard_base = i;
      rc = launch_register(c, c->plan.train, 1, p);
      ++launches;
    }
  } else {
    rc = launch_register(c, c->plan.train, c->nlocal, p);
  }
  if (rc) return rc;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->stream));
  acc->launches += launches;
  return W2B_OK;
}

// Waits for the launch and reads the shard states back.
static int launch_finish(w2b_ctx *c, w2b_step_stats *acc) {
  CK(cudaMemcpyAsync(c->h_shards.data(), c->d_shards, sizeof(ShardState) * c->nlocal, cudaMemcpyDeviceToHost,
                     c->stream));
  CK(cudaStreamSynchronize(c->stream));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  acc->kernel_ms += ms;
  acc->d2h_bytes += (long long)sizeof(ShardState) * c->nlocal;
  return W2B_OK;
}

static int launch_train(w2b_ctx *c, TrainParams p, w2b_step_stats *acc) {
  int rc = launch_enqueue(c, p, acc);
  if (rc) return rc;
  return launch_finish(c, acc);
}

// Per-shard draw records of a training step (w2b_train_step_traced): device buffers that live for every launch of the
// step, so that a shard's records continue across bounded launches and streamed slices.
struct StepTrace {
  w2b_trace_rec *recs;
  int64_t cap;
  int64_t *n;
};

static int w2b_train_step_impl(w2b_ctx *c, int64_t words_per_shard, w2b_step_stats *stats, const StepTrace *tr);
extern "C" int w2b_train_step(w2b_ctx *c, int64_t words_per_shard, w2b_step_stats *stats) {
  return w2b_guarded("w2b_train_step", [&] { return w2b_train_step_impl(c, words_per_shard, stats, nullptr); });
}
extern "C" int w2b_train_step_traced(w2b_ctx *c, int64_t words_per_shard, w2b_step_stats *stats,
                                     w2b_trace_rec *recs, int64_t cap_per_shard, int64_t *n_per_shard) {
  return w2b_guarded("w2b_train_step_traced", [&] {
    NEED(n_per_shard);
    if (cap_per_shard < 0) { w2b_set_error("w2b_train_step_traced: negative cap"); return W2B_EINVAL; }
    if (cap_per_shard > 0) NEED(recs);
    NEED(c);
    const StepTrace tr{recs, cap_per_shard, n_per_shard};
    return w2b_train_step_impl(c, words_per_shard, stats, &tr);
  });
}
static int w2b_train_step_impl(w2b_ctx *c, int64_t words_per_shard, w2b_step_stats *stats, const StepTrace *tr) {
  NEED(c);
  if (!c->have_corpus || !c->have_tables || !c->have_counts) {
    w2b_set_error("train_step before set_vocab_counts/set_corpus/init_tables");
    return W2B_ESTATE;
  }
  CK(cudaSetDevice(c->cfg.device));
  w2b_step_stats before, after, acc;
  memset(&acc, 0, sizeof acc);
  sum_shards(c->h_shards, &before);
  TrainParams p = base_params(c);
  DevTmp t_tr, t_cnt;
  if (tr) {
    if (tr->cap > ((int64_t)1 << 40) / (int64_t)sizeof(w2b_trace_rec) / std::max(c->nlocal, 1)) {
      w2b_set_error("w2b_train_step_traced: cap_per_shard %lld too large", (long long)tr->cap);
      return W2B_EINVAL;
    }
    CK(t_tr.alloc((size_t)std::max<int64_t>(tr->cap * c->nlocal, 1) * sizeof(w2b_trace_rec)));
    CK(t_cnt.alloc(sizeof(unsigned long long) * c->nlocal));
    CK(cudaMemsetAsync(t_cnt.p, 0, sizeof(unsigned long long) * c->nlocal, c->stream));
    p.trace = t_tr.as<w2b_trace_rec>();
    p.trace_cap = tr->cap;
    p.trace_n = t_cnt.as<unsigned long long>();
    p.trace_per_shard = 1;
  }
  // The production kernel keeps 32-bit job and row counters per launch and the streaming path stages one slice
  // per shard in pinned memory, so a step is cut into bounded launches: 4 M words per shard per launch
  // (resident) / 1 M words per slice (streaming).  Steps up to those sizes are exactly one launch.
  const long long kLaunchWords = 4 << 20, kSliceWords = 1 << 20;
  if (c->resident) {
    if (c->cfg.mode == W2B_MODE_STRICT) {
      p.word_budget = words_per_shard;  // <= 0: every shard to its end, one after another
      int rc = launch_train(c, p, &acc);
      if (rc) return rc;
    } else {
      long long left = words_per_shard;  // <= 0: to the end of every shard
      for (;;) {
        p.word_budget = words_per_shard > 0 ? std::min(left, kLaunchWords) : kLaunchWords;
        int rc = launch_train(c, p, &acc);
        if (rc) return rc;
        if (words_per_shard > 0 && (left -= p.word_budget) <= 0) break;
        w2b_step_stats now;
        sum_shards(c->h_shards, &now);
        if (now.shards_done == c->nlocal) break;
      }
    }
  } else {
    // streaming: slices of (budget + margin) tokens; run-to-end loops over slices.  The slices of the launch after
    // this one are gathered and uploaded while this one runs (stage_prefetch).
    long long left = words_per_shard;
    for (;;) {
      const long long chunk = words_per_shard > 0 ? std::min(left, kSliceWords) : 65536;
      int rc = stage_acquire(c, chunk, &acc);
      if (rc) return rc;
      p.tokens = c->d_stage[c->stage_cur];
      p.word_budget = chunk;
      std::vector<long long> wc_before(c->nlocal);
      for (int i = 0; i < c->nlocal; ++i) wc_before[i] = c->h_shards[i].word_count;
      rc = launch_enqueue(c, p, &acc);
      if (rc) return rc;
      rc = stage_prefetch(c, chunk, &acc);  // overlaps the kernel; cursors are still the pre-launch ones
      if (rc) return rc;
      rc = launch_finish(c, &acc);
      if (rc) return rc;
      w2b_step_stats a2;
      sum_shards(c->h_shards, &a2);
      bool stuck = false;  // a sentence longer than the slice: widen the margin and retry
      for (int i = 0; i < c->nlocal; ++i)
        if (!c->h_shards[i].done && !c->h_shards[i].limit_is_eof && c->h_shards[i].word_count == wc_before[i])
          stuck = true;
      if (stuck) c->stage_margin *= 2;
      else if (words_per_shard > 0 && (left -= chunk) <= 0) break;
      if (a2.shards_done == c->nlocal) break;
    }
  }
  sum_shards(c->h_shards, &after);
  if (stats) {
    stats->loss = after.loss - before.loss;
    stats->words = after.words - before.words;
    stats->positions = after.positions - before.positions;
    stats->context_rows = after.context_rows - before.context_rows;
    stats->target_rows = after.target_rows - before.target_rows;
    stats->shards_done = after.shards_done;
    stats->kernel_ms = acc.kernel_ms;
    stats->launches = acc.launches;
    stats->h2d_bytes = acc.h2d_bytes;
    stats->d2h_bytes = acc.d2h_bytes + (long long)(sizeof(float) + sizeof(unsigned long long));
    unsigned long long wca = 0;
    CK(cudaMemcpy(&stats->alpha, c->d_alpha, sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&wca, c->d_wca, sizeof wca, cudaMemcpyDeviceToHost));
    stats->word_count_actual = (int64_t)wca;
  }
  if (tr) {
    std::vector<unsigned long long> n(c->nlocal);
    CK(cudaMemcpy(n.data(), p.trace_n, sizeof(unsigned long long) * c->nlocal, cudaMemcpyDeviceToHost));
    for (int i = 0; i < c->nlocal; ++i) {
      tr->n[i] = (int64_t)n[i];
      const int64_t k = std::min<int64_t>((int64_t)n[i], tr->cap);
      if (k) CK(cudaMemcpy(tr->recs + i * tr->cap, p.trace + i * tr->cap, k * sizeof(w2b_trace_rec),
                           cudaMemcpyDeviceToHost));
    }
  }
  return W2B_OK;
}

extern "C" int w2b_train_epoch(w2b_ctx *c, double *loss, w2b_step_stats *stats) {
  NEED(c);
  int rc = w2b_epoch_begin(c);
  if (rc) return rc;
  w2b_step_stats st;
  rc = w2b_train_step(c, 0, &st);
  if (rc) return rc;
  if (loss) *loss = st.loss;
  if (stats) *stats = st;
  return W2B_OK;
}

// --------------------------------------------------------------------------- parity hooks
static int w2b_trace_impl(w2b_ctx *c, int shard, int64_t max_iterations, w2b_trace_rec *out, int64_t cap,
                         int64_t *n_out);
extern "C" int w2b_trace(w2b_ctx *c, int shard, int64_t max_iterations, w2b_trace_rec *out, int64_t cap,
                         int64_t *n_out) {
  return w2b_guarded("w2b_trace", [&] { return w2b_trace_impl(c, shard, max_iterations, out, cap, n_out); });
}
static int w2b_trace_impl(w2b_ctx *c, int shard, int64_t max_iterations, w2b_trace_rec *out, int64_t cap,
                         int64_t *n_out) {
  NEED(c);
  NEED(n_out);
  if (cap > 0) NEED(out);
  if (!c->have_corpus || !c->have_counts || !c->resident) {
    w2b_set_error("trace needs set_vocab_counts + a resident corpus");
    return W2B_ESTATE;
  }
  if (shard < c->cfg.shard_begin || shard >= c->cfg.shard_end) { w2b_set_error("shard not local"); return W2B_EINVAL; }
  CK(cudaSetDevice(c->cfg.device));
  // scratch copies: the draws must not disturb the training state
  const ShardState s = shard_epoch_start(c, shard - c->cfg.shard_begin);
  DevTmp t_s, t_alpha, t_cnt, t_tr;
  CK(t_s.alloc(sizeof s));
  CK(t_alpha.alloc(sizeof(float)));
  CK(t_cnt.alloc(2 * sizeof(unsigned long long)));
  CK(t_tr.alloc(std::max<int64_t>(cap, 1) * sizeof(w2b_trace_rec)));
  ShardState *d_s = t_s.as<ShardState>();
  float *d_alpha = t_alpha.as<float>();
  unsigned long long *d_cnt = t_cnt.as<unsigned long long>();
  w2b_trace_rec *d_tr = t_tr.as<w2b_trace_rec>();
  CK(cudaMemcpyAsync(d_s, &s, sizeof s, cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemcpyAsync(d_alpha, &c->cfg.alpha, sizeof(float), cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemsetAsync(d_cnt, 0, 2 * sizeof(unsigned long long), c->stream));
  TrainParams p = base_params(c);
  p.shards = d_s;
  p.alpha = d_alpha;
  p.wca = d_cnt;
  p.trace_n = d_cnt + 1;
  p.trace = d_tr;
  p.trace_cap = cap;
  p.train = 0;
  p.max_iters = max_iterations;
  p.wca_scale = 1;
  // with the warp kernel: the production kernel's own sampling code (prefetching draw path)
  const int rc = c->plan.warp ? launch_warp(c, p, ApplyArgs{}, true) : launch_register(c, c->plan.train, 1, p);
  if (rc) return rc;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  unsigned long long cnt[2];
  CK(cudaMemcpy(cnt, d_cnt, sizeof cnt, cudaMemcpyDeviceToHost));
  int64_t n = std::max<int64_t>(0, std::min<int64_t>((int64_t)cnt[1], cap));
  if (n) CK(cudaMemcpy(out, d_tr, n * sizeof(w2b_trace_rec), cudaMemcpyDeviceToHost));
  *n_out = n;
  return W2B_OK;
}

extern "C" int w2b_strict_prefix(w2b_ctx *c, int shard, int64_t max_iterations, double *loss) {
  NEED(c);
  if (c->cfg.mode != W2B_MODE_STRICT) { w2b_set_error("strict_prefix needs W2B_MODE_STRICT"); return W2B_ESTATE; }
  if (!c->have_corpus || !c->have_tables || !c->have_counts || !c->resident) {
    w2b_set_error("strict_prefix before setup");
    return W2B_ESTATE;
  }
  CK(cudaSetDevice(c->cfg.device));
  const int i = shard - c->cfg.shard_begin;
  if (i < 0 || i >= c->nlocal) { w2b_set_error("shard not local"); return W2B_EINVAL; }
  TrainParams p = base_params(c);
  p.shard_base = i;
  p.max_iters = max_iterations;
  const double before = c->h_shards[i].loss;
  const int rc = launch_register(c, c->plan.train, 1, p);
  if (rc) return rc;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(c->h_shards.data(), c->d_shards, sizeof(ShardState) * c->nlocal, cudaMemcpyDeviceToHost,
                     c->stream));
  CK(cudaStreamSynchronize(c->stream));
  if (loss) *loss = c->h_shards[i].loss - before;
  return W2B_OK;
}

extern "C" int w2b_apply_position(w2b_ctx *c, const int32_t *ctx_ids, int cw, const int32_t *targets, int nt,
                                  float *f_out) {
  NEED(c);
  if (!c->have_tables) { w2b_set_error("init_tables first"); return W2B_ESTATE; }
  if (cw < 0 || cw > 2 * W2B_MAX_WINDOW || nt < 0 || nt > W2B_MAX_NEGATIVE + 1) { w2b_set_error("cw/nt out of range"); return W2B_EINVAL; }
  if ((cw > 0 && !ctx_ids) || (nt > 0 && !targets)) { w2b_set_error("w2b_apply_position: null ids"); return W2B_EINVAL; }
  for (int k = 0; k < cw + nt; ++k) {
    const int id = k < cw ? ctx_ids[k] : targets[k - cw];
    if (id < 0 || id >= c->cfg.vocab_size) { w2b_set_error("w2b_apply_position: id %d out of range", id); return W2B_EINVAL; }
  }
  CK(cudaSetDevice(c->cfg.device));
  DevTmp t_ids, t_f;
  CK(t_ids.alloc((cw + nt + 1) * sizeof(int)));
  CK(t_f.alloc((nt + 1) * sizeof(float)));
  int *d_ids = t_ids.as<int>();
  float *d_f = t_f.as<float>();
  if (cw) CK(cudaMemcpyAsync(d_ids, ctx_ids, cw * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  if (nt) CK(cudaMemcpyAsync(d_ids + cw, targets, nt * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  TrainParams p = base_params(c);
  if (c->plan.warp) {  // L1 hook through the production kernel itself: one explicit position, one launch
    if (cw > 2 * c->cfg.window || nt > c->cfg.negative + 1) {
      w2b_set_error("w2b_apply_position: cw <= 2*window and ntargets <= negative+1 for this context");
      return W2B_EINVAL;
    }
    if (cw == 0) return W2B_OK;  // nothing is trained without context (:450)
    DevTmp t_s;
    CK(t_s.alloc(sizeof(ShardState)));
    CK(cudaMemsetAsync(t_s.p, 0, sizeof(ShardState), c->stream));
    p.shards = t_s.as<ShardState>();
    p.serial = 1;
    const int rc = launch_warp(c, p, ApplyArgs{d_ids, d_ids + cw, cw, nt, d_f}, true);
    if (rc) return rc;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(c->stream));
    if (f_out && nt) CK(cudaMemcpy(f_out, d_f, nt * sizeof(float), cudaMemcpyDeviceToHost));
    return W2B_OK;
  }
  const int rc = launch_register(c, c->plan.apply, 1, p, d_ids, cw, d_ids + cw, nt, d_f, nullptr);
  if (rc) return rc;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  if (f_out && nt) CK(cudaMemcpy(f_out, d_f, nt * sizeof(float), cudaMemcpyDeviceToHost));
  return W2B_OK;
}

extern "C" int w2b_get_state(w2b_ctx *c, float *alpha, int64_t *wca) {
  NEED(c);
  CK(cudaSetDevice(c->cfg.device));
  unsigned long long w = 0;
  if (alpha) CK(cudaMemcpy(alpha, c->d_alpha, sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&w, c->d_wca, sizeof w, cudaMemcpyDeviceToHost));
  if (wca) *wca = (int64_t)w;
  return W2B_OK;
}

extern "C" int w2b_set_state(w2b_ctx *c, float alpha, int64_t wca) {
  NEED(c);
  CK(cudaSetDevice(c->cfg.device));
  unsigned long long w = (unsigned long long)wca;
  CK(cudaMemcpyAsync(c->d_alpha, &alpha, sizeof(float), cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemcpyAsync(c->d_wca, &w, sizeof w, cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemcpyAsync(c->d_scratch + 1, &w, sizeof w, cudaMemcpyHostToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  c->wca_at_sync = wca;
  return W2B_OK;
}

extern "C" int w2b_download_raw(w2b_ctx *c, float *u, float *v) {
  NEED(c);
  CK(cudaSetDevice(c->cfg.device));
  const size_t row = (size_t)c->cfg.layer1_size * sizeof(float), dp = (size_t)c->plan.pitch * sizeof(float);
  if (u) CK(cudaMemcpy2D(u, row, c->d_u, dp, row, c->cfg.vocab_size, cudaMemcpyDeviceToHost));
  if (v) CK(cudaMemcpy2D(v, row, c->d_v, dp, row, c->cfg.vocab_size, cudaMemcpyDeviceToHost));
  return W2B_OK;
}

extern "C" int w2b_upload_raw(w2b_ctx *c, const float *u, const float *v) {
  NEED(c);
  CK(cudaSetDevice(c->cfg.device));
  const size_t row = (size_t)c->cfg.layer1_size * sizeof(float), dp = (size_t)c->plan.pitch * sizeof(float);
  if (u) CK(cudaMemcpy2DAsync(c->d_u, dp, u, row, row, c->cfg.vocab_size, cudaMemcpyHostToDevice, c->stream));
  if (v) CK(cudaMemcpy2DAsync(c->d_v, dp, v, row, row, c->cfg.vocab_size, cudaMemcpyHostToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return W2B_OK;
}

extern "C" int w2b_download_table(w2b_ctx *c, int32_t *table) {
  NEED(c);
  NEED(table);
  CK(cudaSetDevice(c->cfg.device));
  CK(cudaMemcpy(table, c->d_table, (size_t)W2B_TABLE_SIZE * sizeof(int), cudaMemcpyDeviceToHost));
  return W2B_OK;
}

extern "C" int w2b_download_exptable(w2b_ctx *c, float *t) {
  NEED(c);
  NEED(t);
  CK(cudaSetDevice(c->cfg.device));
  CK(cudaMemcpy(t, c->d_exptab, kExpN * sizeof(float), cudaMemcpyDeviceToHost));
  return W2B_OK;
}

// Resumable checkpoint: header + raw fp32 u, v (device -> host in 64 MB pieces).
struct CkptHeader {
  char magic[8];
  int64_t V, D, epochs_done, wca;
  float alpha;
  int32_t bitlevel;
  int64_t iter, train_words;  // what the learning-rate schedule (:391) is built from
};
static int w2b_checkpoint_save_impl(w2b_ctx *c, const char *path, int64_t epochs_done);
extern "C" int w2b_checkpoint_save(w2b_ctx *c, const char *path, int64_t epochs_done) {
  return w2b_guarded("w2b_checkpoint_save", [&] { return w2b_checkpoint_save_impl(c, path, epochs_done); });
}
static int w2b_checkpoint_save_impl(w2b_ctx *c, const char *path, int64_t epochs_done) {
  NEED(c);
  NEED(path);
  CK(cudaSetDevice(c->cfg.device));
  CkptHeader h;
  memset(&h, 0, sizeof h);
  memcpy(h.magic, "W2BCKPT2", 8);
  h.V = c->cfg.vocab_size; h.D = c->cfg.layer1_size; h.epochs_done = epochs_done;
  h.bitlevel = c->cfg.bitlevel; h.iter = c->cfg.iter; h.train_words = c->train_words;
  unsigned long long w = 0;
  CK(cudaMemcpy(&h.alpha, c->d_alpha, sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&w, c->d_wca, sizeof w, cudaMemcpyDeviceToHost));
  h.wca = (int64_t)w;
  // written beside the target and renamed over it: a crash or a full disk mid-write keeps the previous checkpoint
  const std::string tmp = std::string(path) + ".tmp";
  FILE *f = fopen(tmp.c_str(), "wb");
  if (!f) { w2b_set_error("cannot open %s for writing", tmp.c_str()); return W2B_EIO; }
  bool ok = fwrite(&h, sizeof h, 1, f) == 1;
  // the file holds V x D contiguous floats per table whatever the row pitch on the device: whole rows per piece
  const size_t D = (size_t)h.D, rows_per_piece = std::max<size_t>(1, (16u << 20) / D);
  std::vector<float> buf(std::min((size_t)h.V, rows_per_piece) * D);
  for (const float *src : {c->d_u, c->d_v})
    for (size_t r0 = 0; r0 < (size_t)h.V && ok; r0 += rows_per_piece) {
      const size_t nr = std::min(rows_per_piece, (size_t)h.V - r0);
      if (cudaMemcpy2D(buf.data(), D * sizeof(float), src + r0 * c->plan.pitch, (size_t)c->plan.pitch * sizeof(float),
                       D * sizeof(float), nr, cudaMemcpyDeviceToHost) != cudaSuccess) {
        fclose(f);
        remove(tmp.c_str());
        w2b_set_error("checkpoint download failed");
        return W2B_ECUDA;
      }
      ok = fwrite(buf.data(), sizeof(float), nr * D, f) == nr * D;
    }
  if (ok && fflush(f) != 0) ok = false;
  if (ok && fsync(fileno(f)) != 0) ok = false;
  if (fclose(f) != 0) ok = false;
  if (!ok) { remove(tmp.c_str()); w2b_set_error("short write to %s (disk full?)", tmp.c_str()); return W2B_EIO; }
  if (rename(tmp.c_str(), path) != 0) { remove(tmp.c_str()); w2b_set_error("cannot move %s to %s", tmp.c_str(), path); return W2B_EIO; }
  return W2B_OK;
}

static int w2b_checkpoint_load_impl(w2b_ctx *c, const char *path, int64_t *epochs_done);
extern "C" int w2b_checkpoint_load(w2b_ctx *c, const char *path, int64_t *epochs_done) {
  return w2b_guarded("w2b_checkpoint_load", [&] { return w2b_checkpoint_load_impl(c, path, epochs_done); });
}
static int w2b_checkpoint_load_impl(w2b_ctx *c, const char *path, int64_t *epochs_done) {
  NEED(c);
  NEED(path);
  CK(cudaSetDevice(c->cfg.device));
  FILE *f = fopen(path, "rb");
  if (!f) { w2b_set_error("cannot open %s", path); return W2B_EIO; }
  CkptHeader h;
  if (fread(&h, sizeof h, 1, f) != 1 || memcmp(h.magic, "W2BCKPT2", 8) != 0 || h.V != c->cfg.vocab_size ||
      h.D != c->cfg.layer1_size) {
    fclose(f);
    w2b_set_error("%s is not a checkpoint of a %lld x %lld model", path, (long long)c->cfg.vocab_size,
                  (long long)c->cfg.layer1_size);
    return W2B_EIO;
  }
  if (h.bitlevel != c->cfg.bitlevel || h.iter != c->cfg.iter || (c->have_counts && h.train_words != c->train_words)) {
    fclose(f);  // resuming under another schedule or bit level would silently train something else
    w2b_set_error("%s was written with -bitlevel %d -iter %lld on %lld training words; this run has -bitlevel %d -iter %lld on %lld",
                  path, (int)h.bitlevel, (long long)h.iter, (long long)h.train_words, (int)c->cfg.bitlevel,
                  (long long)c->cfg.iter, (long long)c->train_words);
    return W2B_EINVAL;
  }
  const size_t D = (size_t)h.D, rows_per_piece = std::max<size_t>(1, (16u << 20) / D);
  std::vector<float> buf(std::min((size_t)h.V, rows_per_piece) * D);
  for (float *dst : {c->d_u, c->d_v})
    for (size_t r0 = 0; r0 < (size_t)h.V; r0 += rows_per_piece) {
      const size_t nr = std::min(rows_per_piece, (size_t)h.V - r0);
      if (fread(buf.data(), sizeof(float), nr * D, f) != nr * D ||
          cudaMemcpy2D(dst + r0 * c->plan.pitch, (size_t)c->plan.pitch * sizeof(float), buf.data(), D * sizeof(float),
                       D * sizeof(float), nr, cudaMemcpyHostToDevice) != cudaSuccess) {
        fclose(f);
        w2b_set_error("checkpoint %s is truncated or the upload failed", path);
        return W2B_EIO;
      }
    }
  fclose(f);
  CK(cudaDeviceSynchronize());  // the uploads ran on the legacy stream
  if (epochs_done) *epochs_done = h.epochs_done;
  c->have_tables = true;  // u and v now hold trained values
  return w2b_set_state(c, h.alpha, h.wca);
}

extern "C" int w2b_export(w2b_ctx *c, float *out) {
  NEED(c);
  NEED(out);
  CK(cudaSetDevice(c->cfg.device));
  const long long n = c->cfg.vocab_size * c->cfg.layer1_size;
  DevTmp t_out;
  CK(t_out.alloc(n * sizeof(float)));
  float *d_out = t_out.as<float>();
  export_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->d_u, c->d_v, d_out, n, c->cfg.layer1_size, c->plan.pitch, c->cfg.bitlevel);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, d_out, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return W2B_OK;
}

int w2b_ctx_tables_of(w2b_ctx *c, w2b_ctx_tables *out) {
  NEED(c);
  if (!c->have_tables) { w2b_set_error("init_tables or checkpoint_load first"); return W2B_ESTATE; }
  out->u = c->d_u;
  out->v = c->d_v;
  out->V = c->cfg.vocab_size;
  out->D = c->cfg.layer1_size;
  out->pitch = c->plan.pitch;
  out->bitlevel = c->cfg.bitlevel;
  out->device = c->cfg.device;
  out->stream = c->stream;
  return W2B_OK;
}

extern "C" int w2b_quantize(w2b_ctx *c, const float *in, float *out, int64_t n, int bitlevel) {
  NEED(c);
  if (n <= 0) return W2B_OK;
  NEED(in);
  NEED(out);
  CK(cudaSetDevice(c->cfg.device));
  DevTmp t;
  CK(t.alloc(2 * n * sizeof(float)));
  float *d = t.as<float>();
  CK(cudaMemcpyAsync(d, in, n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  quantize_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(d, d + n, n, bitlevel);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, d + n, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return W2B_OK;
}

// ------------------------------------------------------------------------------ multi-GPU
extern "C" int w2b_device_ptrs(w2b_ctx *c, void **u, void **v, int64_t *elems) {
  NEED(c);
  if (u) *u = c->d_u;
  if (v) *v = c->d_v;
  if (elems) *elems = (int64_t)table_elems(c);  // rows of pitch = round_up(layer1_size, 4) floats
  return W2B_OK;
}

extern "C" int w2b_nccl_unique_id(void *id128) {
  NEED(id128);
  int rc = nccl_load();
  if (rc) return rc;
  nccl_uid id;
  int e = g_nccl.GetUniqueId(&id);
  if (e) { w2b_set_error("ncclGetUniqueId: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "?"); return W2B_ENCCL; }
  memcpy(id128, &id, sizeof id);
  return W2B_OK;
}

extern "C" int w2b_nccl_init(w2b_ctx *c, const void *id128, int rank, int nranks) {
  NEED(c);
  if (nranks <= 1) { c->rank = 0; c->nranks = 1; return W2B_OK; }
  NEED(id128);
  if (rank < 0 || rank >= nranks) { w2b_set_error("rank %d outside [0,%d)", rank, nranks); return W2B_EINVAL; }
  int rc = nccl_load();
  if (rc) return rc;
  CK(cudaSetDevice(c->cfg.device));
  nccl_uid id;
  memcpy(&id, id128, sizeof id);
  if (c->comm) {  // a second init replaces the communicator instead of leaking it
    if (g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
    c->comm = nullptr;
  }
  int e = g_nccl.CommInitRank(&c->comm, nranks, id, rank);
  if (e) { w2b_set_error("ncclCommInitRank: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "?"); return W2B_ENCCL; }
  c->rank = rank;
  c->nranks = nranks;
  if (c->cfg.sync_mode == 1) {  // sum of deltas: remember the common starting point (same InitNet / checkpoint on every rank)
    const size_t bytes = table_elems(c) * sizeof(float);
    if (!c->d_base_u) CK(cudaMalloc(&c->d_base_u, bytes));
    if (!c->d_base_v) CK(cudaMalloc(&c->d_base_v, bytes));
    CK(cudaMemcpyAsync(c->d_base_u, c->d_u, bytes, cudaMemcpyDeviceToDevice, c->stream));
    CK(cudaMemcpyAsync(c->d_base_v, c->d_v, bytes, cudaMemcpyDeviceToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
  }
  return W2B_OK;
}

extern "C" int w2b_scale_tables(w2b_ctx *c, float s) {
  NEED(c);
  CK(cudaSetDevice(c->cfg.device));
  const long long n = (long long)table_elems(c);
  scale_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->d_u, n, s);
  scale_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->d_v, n, s);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  return W2B_OK;
}

// word_count_actual across ranks, on the device: between two syncs every rank advances its counter by nranks x its
// own words (TrainParams::wca_scale), so that the learning-rate schedule runs on the global clock; at a sync the
// exact global count replaces the estimate.  scratch[1] = counter at the last sync.
__global__ void wca_own_kernel(const unsigned long long *wca, unsigned long long *scratch, int nranks) {
  scratch[0] = (*wca - scratch[1]) / (unsigned long long)nranks;
}
__global__ void wca_apply_kernel(unsigned long long *wca, unsigned long long *scratch) {
  scratch[1] += scratch[0];
  *wca = scratch[1];
}
// sync_mode 1 (sum of deltas): x <- x - base before the all-reduce(sum); x <- base + x, base <- x after it
__global__ void delta_kernel(float *x, const float *base, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[i] = __fsub_rn(x[i], base[i]);
}
__global__ void rebase_kernel(float *x, float *base, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float y = __fadd_rn(base[i], x[i]);
    x[i] = y;
    base[i] = y;
  }
}
// order-independent fingerprint of a table: sum of its 32-bit patterns (mod 2^64)
__global__ void checksum_kernel(const unsigned *x, long long n, unsigned long long *out) {
  unsigned long long acc = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) acc += x[i];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

// Replica exchange: u, v <- mean over ranks (ncclAvg, in place; cfg.sync_mode 0, what BASELINE.json's north_star
// names) or u, v <- common base + SUM over ranks of what each rank added since the last exchange (sync_mode 1: every
// rank's updates land in full, as the reference's threads' do in shared memory; averaging divides them by the number
// of ranks, which for rows only one rank touched is a G-fold smaller step), and word_count_actual <- exact global sum, as ONE
// NCCL group on this context's stream — no host round trip between the three reductions.  G=1: no-op, NCCL never
// touched.  *ms (optional) = device time of the exchange (CUDA events).
extern "C" int w2b_sync_timed(w2b_ctx *c, float *ms) {
  NEED(c);
  if (ms) *ms = 0.f;
  if (c->nranks <= 1) return W2B_OK;
  if (!c->comm) { w2b_set_error("w2b_nccl_init first"); return W2B_ESTATE; }
  CK(cudaSetDevice(c->cfg.device));
  const size_t n = table_elems(c);
  const bool sum = c->cfg.sync_mode == 1;
  if (sum && !c->d_base_u) {  // first exchange: every rank still holds the common starting point in `base`
    w2b_set_error("w2b_sync: sync_mode 1 needs w2b_nccl_init after the tables were initialised");
    return W2B_ESTATE;
  }
  CK(cudaEventRecord(c->ev_s0, c->stream));
  wca_own_kernel<<<1, 1, 0, c->stream>>>(c->d_wca, c->d_scratch, c->nranks);
  if (sum) {
    delta_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->d_u, c->d_base_u, (long long)n);
    delta_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->d_v, c->d_base_v, (long long)n);
  }
  CK(cudaGetLastError());
  const int op = sum ? kNcclSum : kNcclAvg;
  int e = g_nccl.GroupStart();
  if (!e) e = g_nccl.AllReduce(c->d_u, c->d_u, n, kNcclFloat32, op, c->comm, c->stream);
  if (!e) e = g_nccl.AllReduce(c->d_v, c->d_v, n, kNcclFloat32, op, c->comm, c->stream);
  if (!e) e = g_nccl.AllReduce(c->d_scratch, c->d_scratch, 1, kNcclUint64, kNcclSum, c->comm, c->stream);
  const int e2 = g_nccl.GroupEnd();
  if (!e) e = e2;
  if (e) { w2b_set_error("ncclAllReduce: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(e) : "?"); return W2B_ENCCL; }
  wca_apply_kernel<<<1, 1, 0, c->stream>>>(c->d_wca, c->d_scratch);
  if (sum) {
    rebase_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->d_u, c->d_base_u, (long long)n);
    rebase_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(c->d_v, c->d_base_v, (long long)n);
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev_s1, c->stream));
  unsigned long long at_sync = 0;
  CK(cudaMemcpyAsync(&at_sync, c->d_scratch + 1, sizeof at_sync, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  c->wca_at_sync = (long long)at_sync;
  CK(cudaEventElapsedTime(&c->last_sync_ms, c->ev_s0, c->ev_s1));
  if (ms) *ms = c->last_sync_ms;
  return W2B_OK;
}
extern "C" int w2b_sync(w2b_ctx *c) { return w2b_sync_timed(c, nullptr); }

// Fingerprints of u and v (sum of the 32-bit patterns): equal on every rank after w2b_sync.
extern "C" int w2b_table_checksum(w2b_ctx *c, uint64_t *u_sum, uint64_t *v_sum) {
  NEED(c);
  NEED(u_sum);
  NEED(v_sum);
  CK(cudaSetDevice(c->cfg.device));
  const long long n = (long long)table_elems(c);
  DevTmp t;
  CK(t.alloc(16));
  CK(cudaMemsetAsync(t.p, 0, 16, c->stream));
  checksum_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>((const unsigned *)c->d_u, n, t.as<unsigned long long>());
  checksum_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>((const unsigned *)c->d_v, n, t.as<unsigned long long>() + 1);
  CK(cudaGetLastError());
  unsigned long long h[2];
  CK(cudaMemcpyAsync(h, t.p, 16, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  *u_sum = h[0];
  *v_sum = h[1];
  return W2B_OK;
}
