// Micro-benchmark (not part of the product): how fast can an H100 stream embedding rows through shared memory with
// one WARP per stream — cp.async.bulk row in, (optional touch), cp.reduce.async.bulk.add.f32 row back — as a function
// of warps per SM, ring depth and row size, for Zipf(1.0) and uniform row ids?  This is the skeleton of the
// warp-per-shard training kernel without its arithmetic: the number it prints is the memory-system ceiling of that
// design (gather + scatter-add, "algorithmic" bytes = 2 x row bytes per row).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o membench membench.cu && ./membench
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <algorithm>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  asm volatile(
      "{\n.reg .pred P1;\nLAB_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n@P1 bra DONE;\nbra LAB_WAIT;\nDONE:\n}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_load(unsigned dst, const void *src, unsigned bytes, unsigned bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void bulk_reduce_add(void *dst, unsigned src, unsigned bytes) {
  asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }

// mode: 0 = load + bulk reduce, 1 = load only, 2 = load + LDS/STS touch + bulk reduce,
//       3 = load + LDS + red.global.add.v4.f32 from registers (the load/store unit carries the scatter-add)
__global__ void __launch_bounds__(32) stream_kernel(float *tab, float *tab2, const int *ids, long long per_warp, int rowb, int K, int mode,
                                                    unsigned long long *sink) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int lane = threadIdx.x;
  const unsigned ring = smem_u32(smem);
  const unsigned bars = ring + (unsigned)K * rowb;
  if (lane == 0) {
    for (int i = 0; i < K; ++i) mbar_init(bars + 8 * i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const int *my = ids + (long long)blockIdx.x * per_warp;
  const long long D = rowb / 4;
  // prime K-1 loads
  if (lane == 0)
    for (int j = 0; j < K - 1 && j < per_warp; ++j) {
      mbar_expect_tx(bars + 8 * j, rowb);
      bulk_load(ring + j * rowb, ((my[j] >> 30) ? tab2 : tab) + (long long)(my[j] & 0x3fffffff) * D, rowb, bars + 8 * j);
    }
  unsigned phase = 0;
  int slot = 0, islot = K - 1;
  float acc = 0.f;
  int id_cur = 0, id_nxt = my[lane];  // ids of the current / next block of 32 jobs, one per lane (per_warp % 32 == 0)
  for (long long j = 0; j < per_warp; ++j) {
    if ((j & 31) == 0) {
      id_cur = id_nxt;
      if (j + 32 < per_warp) id_nxt = my[j + 32 + lane];
    }
    const int id_j = __shfl_sync(0xffffffffu, id_cur, (int)(j & 31));
    const long long nj = j + K - 1;
    const int id_a = __shfl_sync(0xffffffffu, id_cur, (int)(nj & 31)), id_b = __shfl_sync(0xffffffffu, id_nxt, (int)(nj & 31));
    const int id_n = ((nj >> 5) == (j >> 5)) ? id_a : id_b;
    mbar_wait(bars + 8 * slot, (phase >> slot) & 1u);
    phase ^= 1u << slot;
    const unsigned row = ring + slot * rowb;
    if (mode == 2) {
      for (int c = lane * 16; c < rowb; c += 512) {
        float4 v;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(row + c) : "memory");
        acc += v.x + v.y + v.z + v.w;
        v.x *= 0.5f; v.y *= 0.5f; v.z *= 0.5f; v.w *= 0.5f;
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(row + c), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    if (mode == 3) {
      float *dst = ((id_j >> 30) ? tab2 : tab) + (long long)(id_j & 0x3fffffff) * D;
      for (int c = lane * 16; c < rowb; c += 512) {
        float4 v;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(row + c) : "memory");
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + c / 4), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
      }
    }
    __syncwarp();
    if (lane == 0) {
      if (mode != 1 && mode != 3) bulk_reduce_add(((id_j >> 30) ? tab2 : tab) + (long long)(id_j & 0x3fffffff) * D, row, rowb);
      bulk_commit();
      asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      if (nj < per_warp) {
        mbar_expect_tx(bars + 8 * islot, rowb);
        bulk_load(ring + islot * rowb, ((id_n >> 30) ? tab2 : tab) + (long long)(id_n & 0x3fffffff) * D, rowb, bars + 8 * islot);
      }
    }
    __syncwarp();
    if (++slot == K) slot = 0;
    if (++islot == K) islot = 0;
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  if (acc == 123.456f) *sink = 1;
}

int main(int argc, char **argv) {
  const int V = argc > 1 ? atoi(argv[1]) : 400000;
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const long long NIDS = 48ll << 20;
  std::vector<int> h(NIDS);
  std::vector<double> cdf(V);
  double s = 0;
  for (int i = 0; i < V; ++i) { s += 1.0 / (i + 1); cdf[i] = s; }
  unsigned long long r = 88172645463325252ull;
  auto rnd = [&]() { r ^= r << 13; r ^= r >> 7; r ^= r << 17; return (double)(r >> 11) / 9007199254740992.0; };
  int *d_zipf, *d_unif;
  for (long long i = 0; i < NIDS; ++i) h[i] = (int)(std::lower_bound(cdf.begin(), cdf.end(), rnd() * s) - cdf.begin());
  CK(cudaMalloc(&d_zipf, NIDS * 4));
  CK(cudaMemcpy(d_zipf, h.data(), NIDS * 4, cudaMemcpyHostToDevice));
  for (long long i = 0; i < NIDS; ++i) h[i] = (int)(rnd() * V);
  CK(cudaMalloc(&d_unif, NIDS * 4));
  CK(cudaMemcpy(d_unif, h.data(), NIDS * 4, cudaMemcpyHostToDevice));
  // training mix (C2 shape): per position 11 context rows of u drawn from the sub-sampled unigram distribution
  // (sample = 1e-3: keep = (sqrt(f/s)+1)*s/f), then in v the center (same distribution) and 24 negatives ~ f^0.75
  int *d_mix;
  {
    std::vector<double> csub(V), cneg(V);
    double ss = 0, sn = 0;
    for (int i = 0; i < V; ++i) {
      const double f = (1.0 / (i + 1)) / s;
      const double keep = std::min(1.0, (sqrt(f / 1e-3) + 1.0) * 1e-3 / f);
      ss += f * keep; csub[i] = ss;
      sn += pow(f, 0.75); cneg[i] = sn;
    }
    for (long long i = 0; i < NIDS; ++i) {
      const int k = (int)(i % 36);
      if (k < 12) h[i] = (int)(std::lower_bound(csub.begin(), csub.end(), rnd() * ss) - csub.begin()) | (k == 11 ? (1 << 30) : 0);
      else h[i] = (int)(std::lower_bound(cneg.begin(), cneg.end(), rnd() * sn) - cneg.begin()) | (1 << 30);
    }
    CK(cudaMalloc(&d_mix, NIDS * 4));
    CK(cudaMemcpy(d_mix, h.data(), NIDS * 4, cudaMemcpyHostToDevice));
  }
  unsigned long long *sink;
  CK(cudaMalloc(&sink, 8));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  printf("| D | ids | mode | warps/SM | ring K | rows in flight/SM | M rows/s | GB/s (2 x row bytes) |\n|---|---|---|---|---|---|---|---|\n");
  struct Cfg { int D, wps, K; };
  std::vector<Cfg> cfgs = {{800, 12, 4}, {800, 16, 4}, {800, 20, 3}, {400, 16, 5}, {400, 24, 5}, {200, 20, 7}, {200, 28, 8}, {100, 28, 8}};
  for (const Cfg &c : cfgs) {
    const int rowb = c.D * 4;
    float *tab, *tab2;
    CK(cudaMalloc(&tab, (size_t)V * rowb));
    CK(cudaMemset(tab, 0, (size_t)V * rowb));
    CK(cudaMalloc(&tab2, (size_t)V * rowb));
    CK(cudaMemset(tab2, 0, (size_t)V * rowb));
    const size_t smem = (size_t)c.K * rowb + 8 * c.K + 16;
    CK(cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, stream_kernel, 32, smem));
    if (per_sm < c.wps) { printf("| %d | - | - | %d | %d | does not fit (%d CTAs/SM) | | |\n", c.D, c.wps, c.K, per_sm); cudaFree(tab); continue; }
    const int grid = sms * c.wps;
    long long per_warp = std::min<long long>(NIDS / grid, (long long)(12.0e9 / rowb / grid)) / 32 * 32;
    for (int ids = 0; ids < 3; ++ids)
      for (int mode = 0; mode < 4; ++mode) {
        if (ids == 1 && mode == 2) continue;
        if (ids == 0 && mode != 0) continue;
        float best = 1e30f;
        for (int rep = 0; rep < 3; ++rep) {
          CK(cudaEventRecord(e0));
          stream_kernel<<<grid, 32, smem>>>(tab, tab2, ids == 2 ? d_mix : ids ? d_unif : d_zipf, per_warp, rowb, c.K, mode, sink);
          CK(cudaEventRecord(e1));
          CK(cudaEventSynchronize(e1));
          CK(cudaGetLastError());
          float ms;
          CK(cudaEventElapsedTime(&ms, e0, e1));
          if (rep) best = std::min(best, ms);
        }
        const double rows = (double)per_warp * grid;
        printf("| %d | %s | %s | %d | %d | %d | %.1f | %.0f |\n", c.D, ids == 2 ? "train-mix" : ids ? "uniform" : "zipf",
               mode == 0 ? "load+reduce" : mode == 1 ? "load only" : mode == 2 ? "load+touch+reduce" : "load+red.v4", c.wps, c.K, c.wps * (c.K - 2),
               rows / best / 1e3, rows * rowb * (mode == 1 ? 1 : 2) / best / 1e6);
        fflush(stdout);
      }
    cudaFree(tab);
    cudaFree(tab2);
  }
  return 0;
}
