// Tensor-core candidate pass of the analogy evaluator (src/compute-accuracy.c:150-177) for sm_90a.
//
// scores = Q (nq x D) . M^T (D x words) is the one dense contraction in this repository.  The reference's
// arg-max must be reproduced exactly (first index wins ties, only positive scores count, the three query
// words are skipped), so the tensor cores are used as a FILTER, not as the scorer:
//   pass 1 (this file): TF32 wgmma on the fp32 operands as they are (TMA -> 128B-swizzled shared memory,
//          4-stage mbarrier pipeline -> wgmma, accumulators in registers), 128 questions x 256 words per CTA;
//          the epilogue keeps the question's best approximate score so far (atomicMax) and appends every
//          (question, word) whose approximate score lies within 2*eps of the running best to a candidate list.  TF32 drops the low 13 mantissa bits of either operand, so
//          |approx - exact| <= 2^-9 * |vec| * |m| (+ the two fp32 accumulations, eval_qeps_kernel): a bound.
//          A question with no positive approximate score keeps every word above -2*eps: the reference answers
//          any word whose exact score is > 0.
//   pass 2 (w2b_eval.cu): candidates still within 2*eps of the FINAL best (of 0 if none was positive) are
//          re-scored in fp32 in the reference's operation order; the arg-max over them is the reference's arg-max.
// Layout: both operands K-major with a row pitch of Dp = D rounded up to 32 floats (zero padding), so a k-block
// is one 128-byte swizzle row; rows beyond nq / words are zero-filled by the TMA unit (OOB fill).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace w2b {
namespace tc {

constexpr int BM = 128;        // questions per CTA: two consumer warpgroups of 64 rows (wgmma M = 64)
constexpr int BN = 256;        // words per CTA (wgmma N)
constexpr int BK = 32;         // floats per k-block = one 128-byte swizzle row
constexpr int MMA_K = 8;       // tf32: 8 elements (32 bytes) per instruction
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK * 4, B_BYTES = BN * BK * 4;
constexpr int SMEM_BYTES = STAGES * (A_BYTES + B_BYTES) + 1024 /*alignment*/ + 256 /*barriers*/;
constexpr int THREADS = 288;   // warps 0-7: two consumer warpgroups (MMA + epilogue), warp 8: TMA producer

__device__ __forceinline__ unsigned s32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(unsigned bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(unsigned bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void bar_wait(unsigned bar, unsigned parity) {
  asm volatile(
      "{\n.reg .pred P1;\nTC_WAIT:\nmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n@P1 bra TC_DONE;\nbra TC_WAIT;\nTC_DONE:\n}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(unsigned dst, const CUtensorMap *map, int x, int y, unsigned bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(map), "r"(x), "r"(y), "r"(bar)
               : "memory");
}
// K-major operand tile in 128B-swizzled shared memory: rows of 128 bytes, groups of 8 rows 1024 bytes apart.
__device__ __forceinline__ unsigned long long gmma_desc(unsigned smem_addr) {
  unsigned long long d = 0;
  d |= (unsigned long long)((smem_addr & 0x3FFFF) >> 4);  // start address, 16-byte units, bits [0,14)
  d |= (unsigned long long)1 << 16;                        // leading byte offset (unused for swizzled K-major)
  d |= (unsigned long long)(1024 >> 4) << 32;              // stride byte offset: 8 rows x 128 bytes
  d |= (unsigned long long)1 << 62;                        // SWIZZLE_128B
  return d;
}
// D (64 x 256, f32, registers of the warpgroup) (+)= A (64 x 8 tf32, shared) . B^T (256 x 8 tf32, shared), both K-major
__device__ __forceinline__ void wgmma_tf32(float (&d)[128], unsigned long long a, unsigned long long b, unsigned accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all(float (&d)[128]) {
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
  for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");  // accumulators are final only from here
}
__device__ __forceinline__ unsigned ordered(float s) {  // monotone map float -> uint for atomicMax
  const unsigned b = __float_as_uint(s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

struct Candidate { int q, c; float s; };

// gmax[q] = ordered() of the best approximate score of question q over its valid, non-query words (0: none is
// positive).  cand[0 .. *n_cand) = every (q, c, approximate score) that was within 2*qeps[q] of the running best
// its thread had seen when the score was read (a superset of what is within 2*qeps[q] of the final best); entries
// beyond cand_cap are dropped and *n_cand keeps counting (the caller checks for overflow).
__global__ void __launch_bounds__(THREADS, 1)
eval_tc_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapM, const int *q3,
               const float *qeps, unsigned *gmax, Candidate *cand, unsigned long long *n_cand, unsigned long long cand_cap,
               int nq, int words, int Dp) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char *sA = smem, *sB = smem + STAGES * A_BYTES;
  unsigned long long *bars = (unsigned long long *)(smem + STAGES * (A_BYTES + B_BYTES));
  const unsigned full0 = s32(bars), empty0 = s32(bars + STAGES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int nk = Dp / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { bar_init(full0 + 8 * s, 1); bar_init(empty0 + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {  // ---- TMA producer
      for (int k = 0; k < nk; ++k) {
        const int s = k % STAGES;
        if (k >= STAGES) bar_wait(empty0 + 8 * s, ((k / STAGES) - 1) & 1);
        bar_expect_tx(full0 + 8 * s, A_BYTES + B_BYTES);
        tma_load_2d(s32(sA + s * A_BYTES), &mapQ, k * BK, m0, full0 + 8 * s);
        tma_load_2d(s32(sB + s * B_BYTES), &mapM, k * BK, n0, full0 + 8 * s);
      }
    }
    return;
  }
  // ---- consumer warpgroup wg: questions m0 + 64*wg .. +63 against the CTA's 256 words
  const int wg = warp >> 2, t = threadIdx.x & 127;
  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  for (int k = 0; k < nk; ++k) {
    const int s = k % STAGES;
    bar_wait(full0 + 8 * s, (k / STAGES) & 1);
    const unsigned long long da = gmma_desc(s32(sA + s * A_BYTES + wg * (64 * 128))), db = gmma_desc(s32(sB + s * B_BYTES));
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < BK / MMA_K; ++j)  // advance 32 bytes (2 x 16-byte units) inside the swizzle row
      wgmma_tf32(d, da + 2 * j, db + 2 * j, (k | j) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait_all(d);
    if (t == 0) bar_arrive(empty0 + 8 * s);  // this warpgroup has read the stage
  }

  // ---- epilogue.  Accumulator layout of m64nN: thread t holds rows 16*(t/32) + (t%32)/4 (+8) and, per 8-column
  // block j, columns 8j + 2*(t%4) (+1): d[4j + 2h + e] = (row + 8h, col + e).
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = wg * 64 + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h, q = m0 + row;
    const bool qok = q < nq;
    const int b1 = qok ? q3[q * 3] : -1, b2 = qok ? q3[q * 3 + 1] : -1, b3 = qok ? q3[q * 3 + 2] : -1;
    // lower bound for candidates: the question's best so far (any tile, any CTA) minus the error window
    float thr = 0.f, eps2 = 0.f;
    if (qok) {
      const unsigned g = *(volatile unsigned *)(gmax + q);
      eps2 = 2.f * qeps[q];
      thr = (g ? __uint_as_float(g & 0x7fffffffu) : 0.f) - eps2;
    }
    float best = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = n0 + 8 * j + 2 * (t & 3) + e;
        const float s = d[4 * j + 2 * h + e];
        // s > -eps2, not s > 0: a word whose exact score is a little above 0 can have an approximate score <= 0
        if (qok && c < words && c != b1 && c != b2 && c != b3 && s > -eps2 && s >= thr) {
          if (s > best) {
            best = s;
            thr = fmaxf(thr, s - eps2);  // (a superset is fine: thr only ever rises)
          }
          const unsigned long long at = atomicAdd(n_cand, 1ull);
          if (at < cand_cap) cand[at] = Candidate{q, c, s};
        }
      }
    }
    // the four threads of a row hold disjoint columns: one atomic per row
    best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, 1));
    best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, 2));
    if (qok && (t & 3) == 0 && best > 0.f) atomicMax(gmax + q, ordered(best));
  }
}

// ---- host: 2-D tensor maps over the padded row-major operands (rows x Dp floats), box = BK floats x box_rows
typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline bool make_map(CUtensorMap *map, const float *base, long long rows, long long Dp, int box_rows) {
  static encode_fn enc = nullptr;
  if (!enc) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) return false;
    enc = (encode_fn)fn;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)Dp, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)Dp * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace tc
}  // namespace w2b
