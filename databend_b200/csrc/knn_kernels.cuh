// knn_kernels.cuh — vector distance kernels for sm_90a.
//
//  (1) exact row-wise cosine / L2 in f32 with the reference's evaluation order
//      (src/common/vector/src/distance.rs:19-35,65-80; ndarray 0.15.6 unrolled_fold for the
//      cosine sums) — the ScalarFunction::eval replacement and the re-rank of kNN candidates;
//      templated on the element type: Vector(Float32) or Vector(Int8) widened to f32;
//  (2) the batched query x corpus similarity GEMM on the Hopper tensor cores:
//      TMA (cp.async.bulk.tensor, multicast across a cluster) -> 128B-swizzled shared memory ->
//      wgmma (bf16 in, f32 accumulators, for Float32 corpora; s8 in, exact s32 accumulators, for
//      Int8 corpora) -> epilogue on the accumulator fragment that turns dot products into
//      similarities and keeps only entries that beat the per-query boundary (the k'-th best so
//      far), i.e. the score matrix is never written to HBM.
#pragma once
#include <cuda_bf16.h>

#include <type_traits>

#include "common.cuh"

namespace dbx {

// ---------------------------------------------------------------- exact f32 distances
// ndarray's unrolled_fold: eight interleaved accumulators over full chunks of 8, combined as
// ((((0 + (p0+p4)) + (p1+p5)) + (p2+p6)) + (p3+p7)), then the < 8 tail sequentially.  Products
// are rounded to f32 before the add (`&a * &b` materialises an f32 array): no FMA contraction.
struct CosAcc {
  float aa[8], bb[8], ab[8];
};
__device__ __forceinline__ void cos_acc_init(CosAcc& c) {
#pragma unroll
  for (int j = 0; j < 8; ++j) c.aa[j] = c.bb[j] = c.ab[j] = 0.0f;
}
__device__ __forceinline__ float fold8(const float (&p)[8]) {
  float acc = 0.0f;
  acc = __fadd_rn(acc, __fadd_rn(p[0], p[4]));
  acc = __fadd_rn(acc, __fadd_rn(p[1], p[5]));
  acc = __fadd_rn(acc, __fadd_rn(p[2], p[6]));
  acc = __fadd_rn(acc, __fadd_rn(p[3], p[7]));
  return acc;
}
__device__ __forceinline__ float exact_cosine(const float* __restrict__ a, const float* __restrict__ b, int dim) {
  CosAcc c;
  cos_acc_init(c);
  int i = 0;
  const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
  for (; i + 8 <= dim; i += 8) {
    float x[8], y[8];
    if (vec) {
      float4 x0 = *reinterpret_cast<const float4*>(a + i), x1 = *reinterpret_cast<const float4*>(a + i + 4);
      float4 y0 = *reinterpret_cast<const float4*>(b + i), y1 = *reinterpret_cast<const float4*>(b + i + 4);
      x[0] = x0.x; x[1] = x0.y; x[2] = x0.z; x[3] = x0.w; x[4] = x1.x; x[5] = x1.y; x[6] = x1.z; x[7] = x1.w;
      y[0] = y0.x; y[1] = y0.y; y[2] = y0.z; y[3] = y0.w; y[4] = y1.x; y[5] = y1.y; y[6] = y1.z; y[7] = y1.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) { x[j] = a[i + j]; y[j] = b[i + j]; }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      c.aa[j] = __fadd_rn(c.aa[j], __fmul_rn(x[j], x[j]));
      c.bb[j] = __fadd_rn(c.bb[j], __fmul_rn(y[j], y[j]));
      c.ab[j] = __fadd_rn(c.ab[j], __fmul_rn(x[j], y[j]));
    }
  }
  float aa = fold8(c.aa), bb = fold8(c.bb), ab = fold8(c.ab);
  for (; i < dim; ++i) {
    aa = __fadd_rn(aa, __fmul_rn(a[i], a[i]));
    bb = __fadd_rn(bb, __fmul_rn(b[i], b[i]));
    ab = __fadd_rn(ab, __fmul_rn(a[i], b[i]));
  }
  // 1 - ab / (sqrt(aa) * sqrt(bb))
  return __fsub_rn(1.0f, __fdiv_rn(ab, __fmul_rn(__fsqrt_rn(aa), __fsqrt_rn(bb))));
}
// l2_distance: strictly sequential f32 fold of (a-b)^2, then sqrt
template <typename T>
__device__ __forceinline__ float exact_l2(const T* __restrict__ a, const T* __restrict__ b, int dim) {
  float acc = 0.0f;
  for (int i = 0; i < dim; ++i) {
    float d = __fsub_rn((float)a[i], (float)b[i]);
    acc = __fadd_rn(acc, __fmul_rn(d, d));
  }
  return __fsqrt_rn(acc);
}
__device__ __forceinline__ float exact_distance(int kind, const float* a, const float* b, int dim) {
  return kind == DBX_DIST_COSINE ? exact_cosine(a, b, dim) : exact_l2(a, b, dim);
}

// Vector(Int8) arguments (calculate_distance, scalars/vector.rs:515-524) are widened element by
// element (`*v as f32`) and then go through the same f32 functions.  The widening is exact (every
// value is an integer in [-128, 127]), so the int8 instantiations below compute literally the
// reference's f32 expression over the widened values, bit for bit, at every dim.  For int8 the
// f32 arithmetic is even exact in most cases: every product has magnitude <= 2^14 and every
// (a-b)^2 <= 65 025, so the sums stay exact while every partial sum is <= 2^24 — for cosine
// (the 8-way fold) for every input with dim <= 1024, for L2 (a sequential fold of non-negative
// terms) for every input with dim <= 258 and, beyond, for every pair with sum S <= 2^24 (once
// S > 2^24 the fold's result is >= 2^24).

// Coalesced form of exact_cosine: the 8 lanes of a group own the 8 interleaved accumulators of
// ONE row (lane j accumulates elements 8c+j, c ascending — the same chains in the same order),
// so a group reads one 32-byte sector per step; the fold and the tail are then done redundantly
// by every lane of the group.  All 32 lanes of the warp must call this together.
template <typename T>
__device__ __forceinline__ float exact_cosine_g8(const T* __restrict__ a, const T* __restrict__ b, int dim, int lane) {
  const int sub = lane & 7, gbase = lane & 24;
  float aa = 0.0f, bb = 0.0f, ab = 0.0f;
  const int n_chunks = dim >> 3;
  int c = 0;
  for (; c + 8 <= n_chunks; c += 8) {
    float x[8], y[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) { x[u] = (float)__ldg(a + (c + u) * 8 + sub); y[u] = (float)__ldg(b + (c + u) * 8 + sub); }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      aa = __fadd_rn(aa, __fmul_rn(x[u], x[u]));
      bb = __fadd_rn(bb, __fmul_rn(y[u], y[u]));
      ab = __fadd_rn(ab, __fmul_rn(x[u], y[u]));
    }
  }
  for (; c < n_chunks; ++c) {
    const float x = (float)__ldg(a + c * 8 + sub), y = (float)__ldg(b + c * 8 + sub);
    aa = __fadd_rn(aa, __fmul_rn(x, x));
    bb = __fadd_rn(bb, __fmul_rn(y, y));
    ab = __fadd_rn(ab, __fmul_rn(x, y));
  }
  float paa[8], pbb[8], pab[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    paa[j] = __shfl_sync(0xffffffffu, aa, gbase + j);
    pbb[j] = __shfl_sync(0xffffffffu, bb, gbase + j);
    pab[j] = __shfl_sync(0xffffffffu, ab, gbase + j);
  }
  float saa = fold8(paa), sbb = fold8(pbb), sab = fold8(pab);
  for (int i = n_chunks * 8; i < dim; ++i) {
    const float x = (float)__ldg(a + i), y = (float)__ldg(b + i);
    saa = __fadd_rn(saa, __fmul_rn(x, x));
    sbb = __fadd_rn(sbb, __fmul_rn(y, y));
    sab = __fadd_rn(sab, __fmul_rn(x, y));
  }
  return __fsub_rn(1.0f, __fdiv_rn(sab, __fmul_rn(__fsqrt_rn(saa), __fsqrt_rn(sbb))));
}

// calculate_distance (scalars/vector.rs:497-556), either side may be const; T = float or int8_t.
// cosine: 8 lanes per row (coalesced sectors); L2 (one strictly sequential chain): one thread per row.
template <typename T>
__global__ void distance_rows_kernel(int kind, const T* lhs, int lhs_const, const T* rhs, int rhs_const,
                                     int64_t rows, int dim, const uint8_t* lv, int64_t lv_off, const uint8_t* rv,
                                     int64_t rv_off, float* out, uint8_t* out_valid_bytes) {
  if (kind == DBX_DIST_COSINE) {
    const int lane = threadIdx.x & 31, g = lane >> 3;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t base = warp * 4; base < rows; base += n_warps * 4) {
      const int64_t r = base + g;
      const bool in = r < rows;
      const int64_t rr = in ? r : rows - 1;
      const float d = exact_cosine_g8(lhs + (lhs_const ? 0 : rr * dim), rhs + (rhs_const ? 0 : rr * dim), dim, lane);
      if (in && (lane & 7) == 0) {
        const bool ok = (!lv || bit_test(lv, lv_off + r)) && (!rv || bit_test(rv, rv_off + r));
        out[r] = ok ? d : 0.0f;
        if (out_valid_bytes) out_valid_bytes[r] = ok ? 1 : 0;
      }
    }
    return;
  }
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    bool ok = (!lv || bit_test(lv, lv_off + r)) && (!rv || bit_test(rv, rv_off + r));
    const T* a = lhs + (lhs_const ? 0 : r * dim);
    const T* b = rhs + (rhs_const ? 0 : r * dim);
    out[r] = ok ? exact_l2(a, b, dim) : 0.0f;
    if (out_valid_bytes) out_valid_bytes[r] = ok ? 1 : 0;
  }
}

// ---------------------------------------------------------------- corpus / query preparation
// f32 rows -> bf16 operand of the similarity GEMM (round to nearest even):
//   cosine: the row is normalised first (x / |x|), so the GEMM yields cosine similarities directly
//           and the epilogue is a bare compare; scale[r] = 1/|x| (kept for inspection);
//   L2:     the row is copied as is; scale[r] = |x|^2, combined in the epilogue.
// The sums here only steer candidate selection (returned distances are recomputed exactly).
// A zero vector becomes a NaN operand row: its similarities are NaN and never pass the filter.
// max_norm_bits (optional): bit pattern of the largest row norm (non-negative floats order like
// their bit patterns), the corpus-side constant of the L2 certificate.
//
// The certificate's error budget holds only for rows whose squared norm |x|^2 lies in
// [2^-100, 2^100] (cosine) or is at most 2^100 (L2): outside it the f32 sums underflow or
// overflow, and the bf16 operand can become inf / NaN or lose all precision while the exact
// distance stays finite.  Rows whose exact distance is NaN for every query are harmless (they rank
// last and the candidate pass never needs them): for cosine a row with a NaN / inf component or no
// non-zero component, for L2 a row with a NaN component.  unsafe_rows (optional) counts the other
// rows outside the range; a corpus with any of them gets no certificate.
constexpr float kCertNormLo = 7.8886091e-31f;  // 2^-100
constexpr float kCertNormHi = 1.2676506e30f;   // 2^100
__global__ void prep_rows_kernel(const float* src, int64_t rows, int dim, int dim_pad, __nv_bfloat16* dst, float* scale,
                                 int kind, unsigned int* max_norm_bits, unsigned int* unsafe_rows) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float wmax = 0.0f;
  unsigned int n_unsafe = 0;
  for (int64_t r = warp; r < rows; r += n_warps) {
    const float* a = src + r * dim;
    __nv_bfloat16* d = dst + r * dim_pad;
    float s = 0.0f;
    bool has_nan = false, has_inf = false, has_nonzero = false;
    for (int i = lane; i < dim; i += 32) {
      const float x = a[i];
      s += x * x;
      has_nan |= x != x;
      has_inf |= fabsf(x) == INFINITY;
      has_nonzero |= x != 0.0f;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mul = kind == DBX_DIST_COSINE ? rsqrtf(s) : 1.0f;
    for (int i = lane * 2; i < dim_pad; i += 64) {  // dim_pad is a multiple of 64
      const float x0 = i < dim ? a[i] * mul : 0.0f, x1 = i + 1 < dim ? a[i + 1] * mul : 0.0f;
      *reinterpret_cast<__nv_bfloat162*>(d + i) = __floats2bfloat162_rn(x0, x1);
    }
    if (unsafe_rows) {
      has_nan = __any_sync(0xffffffffu, has_nan);
      has_inf = __any_sync(0xffffffffu, has_inf);
      has_nonzero = __any_sync(0xffffffffu, has_nonzero);
      const bool harmless = kind == DBX_DIST_COSINE ? (has_nan || has_inf || !has_nonzero) : has_nan;
      const bool in_range = kind == DBX_DIST_COSINE ? (s >= kCertNormLo && s <= kCertNormHi) : s <= kCertNormHi;
      n_unsafe += (!harmless && !in_range) ? 1u : 0u;
    }
    if (lane == 0) scale[r] = kind == DBX_DIST_COSINE ? mul : s;
    if (s == s) wmax = fmaxf(wmax, sqrtf(s));
  }
  if (max_norm_bits && lane == 0 && wmax > 0.0f) atomicMax(max_norm_bits, __float_as_uint(wmax));
  if (unsafe_rows && lane == 0 && n_unsafe) atomicAdd(unsafe_rows, n_unsafe);
}

// i8 rows -> int8 operand of the similarity GEMM, zero-padded to dim_pad (a multiple of 128), plus
//   sq[r]    = sum of x^2, exact in int32 (<= 2^14 dim < 2^31 for dim < 131 072);
//   scale[r] = cosine: 1/|x| (f32 sqrt of the f32-rounded sum, then an f32 reciprocal; +inf for a
//              zero row, whose similarities are then NaN and never pass the filter — harmless, its
//              exact cosine distance is NaN for every query), L2: sum of x^2 rounded to f32 (the
//              certificate's |q|^2; the GEMM's epilogue uses the exact sq).
// max_norm_bits as for prep_rows_kernel.  int8 has no inf or NaN, so no row is outside the
// certificate's range.
__global__ void prep_rows_i8_kernel(const int8_t* src, int64_t rows, int dim, int dim_pad, int8_t* dst, int32_t* sq, float* scale,
                                    int kind, unsigned int* max_norm_bits) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float wmax = 0.0f;
  for (int64_t r = warp; r < rows; r += n_warps) {
    const int8_t* a = src + r * dim;
    int8_t* d = dst + r * dim_pad;
    int s = 0;
    for (int i = lane * 4; i < dim_pad; i += 128) {
      char4 v;
      v.x = i < dim ? a[i] : 0;
      v.y = i + 1 < dim ? a[i + 1] : 0;
      v.z = i + 2 < dim ? a[i + 2] : 0;
      v.w = i + 3 < dim ? a[i + 3] : 0;
      s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
      *reinterpret_cast<char4*>(d + i) = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float sf = __int2float_rn(s), nrm = __fsqrt_rn(sf);
    if (lane == 0) {
      sq[r] = s;
      scale[r] = kind == DBX_DIST_COSINE ? __fdiv_rn(1.0f, nrm) : sf;
    }
    wmax = fmaxf(wmax, nrm);
  }
  if (max_norm_bits && lane == 0 && wmax > 0.0f) atomicMax(max_norm_bits, __float_as_uint(wmax));
}

// ---------------------------------------------------------------- wgmma GEMM with fused filter
constexpr int kGemmBM = 128;      // queries per tile: two consumer warpgroups of 64 (wgmma M = 64)
constexpr int kGemmBN = 128;      // corpus rows per tile  (wgmma N)
constexpr int kGemmBK = 64;       // bf16 per k-block = 128 bytes = one swizzle row (int8: 128 per k-block)
constexpr int kGemmStages = 5;
constexpr int kGemmThreads = 384; // warpgroup 0: TMA (one thread), warpgroups 1-2: wgmma + epilogue
constexpr int kWgmmaK = 16;       // bf16 per wgmma k-step = 32 bytes (int8: 32 per k-step)
constexpr int kKBlockBytes = 128;
// elements of T per k-block: 64 bf16 or 128 int8, one 128-byte swizzle row either way
template <typename T>
constexpr int kBlockK = kKBlockBytes / (int)sizeof(T);
constexpr uint32_t kStageBytesA = kGemmBM * kGemmBK * 2;
constexpr uint32_t kStageBytesB = kGemmBN * kGemmBK * 2;
constexpr int kCandStage = 512;   // staged survivors per consumer warp

struct GemmSmem {
  alignas(1024) uint8_t a[kGemmStages][kStageBytesA];
  alignas(1024) uint8_t b[kGemmStages][kStageBytesB];
  alignas(8) uint64_t full_bar[kGemmStages];
  uint64_t empty_bar[kGemmStages];
  // per consumer warp: survivors are staged here and written out in coalesced bursts, one
  // reservation (atomic on the global candidate counter) per burst instead of one per survivor
  alignas(16) uint64_t stage_key[8][kCandStage];
  uint32_t stage_row[8][kCandStage];
};

struct KnnGemmParams {
  int32_t kind;
  int32_t nq;            // valid queries
  int32_t nq_pad;        // multiple of kGemmBM * cluster size
  int32_t dim_pad;       // multiple of kGemmBK
  int64_t n0;            // first corpus row of this pass
  int64_t n_rows;        // corpus rows in this pass
  const float* q_scale;  // bf16 L2: |q|^2; int8 cosine: 1/|q|   (bf16 cosine: unused, operands are pre-normalised)
  const float* c_scale;  // bf16 L2: |c|^2; int8 cosine: 1/|c|, by global row
  const float* bound;    // per query: only score >= bound can still reach the top k'
  uint64_t* cand_key;    // (query << 32) | ~ordered(score): ascending sort = best first
  uint32_t* cand_row;    // corpus row
  unsigned long long* cand_count;
  int64_t cand_cap;
  const int32_t* q_sq;   // int8 L2: exact |q|^2
  const int32_t* c_sq;   // int8 L2: exact |c|^2 by global row
};

// arrive on the barrier at this offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n"
      ".reg .b32 ra;\n"
      "mapa.shared::cluster.u32 ra, %0, %1;\n"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const void* tmap, uint64_t* bar, void* dst, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// Same box delivered to the same shared-memory offset of every CTA in `mask`; each destination
// CTA's mbarrier (same offset) receives the complete_tx for the bytes that landed in ITS smem.
__device__ __forceinline__ void tma_load_2d_multicast(const void* tmap, uint64_t* bar, void* dst, int32_t c0, int32_t c1,
                                                      uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
      "[%0], [%1, {%4, %5}], [%2], %3;" ::"r"(smem_u32(dst)),
      "l"(tmap), "r"(smem_u32(bar)), "h"(mask), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" "barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma: start>>4 | LBO(=1, ignored for
// swizzled K-major)<<16 | SBO(1024 B between 8-row groups)>>4 <<32 | layout SWIZZLE_128B(1) <<62.
// A k-step of 16 bf16 inside the 128-byte swizzle row advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, bf16 in, f32 accumulators in registers, both K-major
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 128] (+)= A[64 x 32] * B[128 x 32]^T, s8 in, s32 accumulators in registers, both K-major.
// Integer wgmma has no negate / transpose immediates.  The accumulators are exact while |sum ab| <
// 2^31, i.e. for dim < 131 072 (every product is <= 2^14 in magnitude).
__device__ __forceinline__ void wgmma_m64n128k32_s8(int32_t (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
        "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
        "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
        "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
        "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// Similarity of an int8 pair from the exact integer dot product ab (larger = closer):
//   cosine: ab / (|q| |c|) = (f32(ab) * (1/|q|)) * (1/|c|), a few f32 roundings of a value in [-1, 1];
//   L2:     -S with S = |q|^2 + |c|^2 - 2ab computed exactly in 64-bit integers, rounded once to f32.
__device__ __forceinline__ float i8_score(bool is_l2, int32_t ab, float q_inv, float c_inv, int32_t q_sq, int32_t c_sq) {
  if (is_l2) return __ll2float_rn(2LL * ab - (long long)q_sq - (long long)c_sq);
  return __fmul_rn(__fmul_rn(__int2float_rn(ab), q_inv), c_inv);
}
__device__ __forceinline__ uint32_t f32_to_ordered32(float f) {
  if (f != f) return 0u;  // NaN: worst similarity
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// One reservation + coalesced copy of a warp's staged survivors into the global candidate list.
__device__ __forceinline__ void flush_stage(const uint64_t* skey, const uint32_t* srow, int cnt, int lane, const KnnGemmParams& p) {
  if (cnt == 0) return;
  __syncwarp();
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(p.cand_count, (unsigned long long)cnt);
  base = __shfl_sync(0xffffffffu, base, 0);
  if ((int64_t)(base + cnt) <= p.cand_cap) {
    for (int i = lane; i < cnt; i += 32) {
      p.cand_key[base + i] = skey[i];
      p.cand_row[base + i] = srow[i];
    }
  }
  __syncwarp();
}

// Persistent, warp-specialised kernel.  A cluster of C CTAs works on C consecutive query blocks
// against the SAME 128-row corpus tile: every CTA streams its own query tile (A) and 1/C of the
// corpus tile (B), which TMA multicasts into the shared memory of all C CTAs — so per CTA the
// L2 -> SM traffic per k-block drops from 16+16 KB to 16+16/C KB.  Consecutive cluster tiles walk
// the query blocks first, so a corpus tile is fetched from HBM once and re-read from L2.
// Each consumer warpgroup multiplies 64 of the tile's 128 queries with wgmma and filters its
// accumulator fragment in registers, so the score matrix is never written anywhere.
// T = __nv_bfloat16 (Float32 corpora) or int8_t (Int8 corpora): a k-block is one 128-byte swizzle
// row of either, split into four 32-byte wgmma k-steps, so the producer, the barriers, the stages,
// the multicast and the candidate staging are the same bytes for both; only the MMA instruction,
// the accumulator type and the score differ.
template <int C, typename T>
__global__ void __launch_bounds__(kGemmThreads, 1)
knn_gemm_filter_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_c,
                       const __grid_constant__ KnnGemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  GemmSmem& sm = *reinterpret_cast<GemmSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t cta_rank = C > 1 ? cluster_ctarank() : 0u;
  const int64_t cluster_id = blockIdx.x / C, n_clusters = gridDim.x / C;
  const int n_mgrp = p.nq_pad / (kGemmBM * C);  // groups of C query blocks
  const int64_t n_nblk = (p.n_rows + kGemmBN - 1) / kGemmBN;
  const int64_t n_tiles = n_nblk * n_mgrp;      // cluster-level tiles
  constexpr bool kI8 = std::is_same<T, int8_t>::value;
  constexpr int kBK = kBlockK<T>;
  const int n_kblk = p.dim_pad / kBK;
  constexpr uint16_t kMask = (uint16_t)((1u << C) - 1u);
  constexpr int kSliceRows = kGemmBN / C;       // corpus rows this CTA fetches for the whole cluster

  if (threadIdx.x == 0) {
    // a slot is free once both consumer warpgroups of every CTA in the cluster have read it
    for (int s = 0; s < kGemmStages; ++s) { mbar_init(&sm.full_bar[s], 1); mbar_init(&sm.empty_bar[s], 2 * C); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_q) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_c) : "memory");
  }
  if (C > 1) cluster_sync_all(); else __syncthreads();  // peers' barriers are initialised before anyone signals them

  if (warp < 4) {
    // ===== TMA producer =====
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t t = cluster_id; t < n_tiles; t += n_clusters) {
        const int m_blk = (int)(t % n_mgrp) * C + (int)cta_rank;
        const int64_t n_blk = t / n_mgrp;
        const int32_t row_b = (int32_t)(p.n0 + n_blk * kGemmBN) + (int32_t)cta_rank * kSliceRows;
        for (int kb = 0; kb < n_kblk; ++kb) {
          mbar_wait(&sm.empty_bar[stage], phase ^ 1);  // all C CTAs have consumed this slot
          mbar_expect_tx(&sm.full_bar[stage], kStageBytesA + kStageBytesB);
          tma_load_2d(&tmap_q, &sm.full_bar[stage], sm.a[stage], kb * kBK, m_blk * kGemmBM);
          if (C > 1)
            tma_load_2d_multicast(&tmap_c, &sm.full_bar[stage], sm.b[stage] + cta_rank * (kSliceRows * kKBlockBytes), kb * kBK, row_b, kMask);
          else
            tma_load_2d(&tmap_c, &sm.full_bar[stage], sm.b[stage], kb * kBK, row_b);
          if (++stage == kGemmStages) { stage = 0; phase ^= 1; }
        }
      }
      if (C > 1) {  // tail: do not leave while peers may still signal this CTA's barriers
        for (int i = 0; i < kGemmStages; ++i) {
          mbar_wait(&sm.empty_bar[stage], phase ^ 1);
          if (++stage == kGemmStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===== consumers: wgmma into registers -> score -> boundary filter -> candidate list =====
    const int cw = warp - 4;            // consumer warp 0..7
    const int wg = cw >> 2;             // queries [64*wg, +64) of the tile
    const uint32_t tid_wg = threadIdx.x & 127;
    const bool is_l2 = p.kind != DBX_DIST_COSINE;
    // accumulator fragment of m64nNk16 (and m64nNk32): register 4j + 2h + e holds row
    // 16*(warp%4) + lane/4 + 8h, column 8j + 2*(lane%4) + e
    const int col_l = 2 * (lane & 3);
    int stage = 0;
    uint32_t phase = 0;
    int stage_cnt = 0;  // warp-uniform
    typename std::conditional<kI8, int32_t, float>::type acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0;
    auto release = [&](int s) {  // one arrival per consumer warpgroup on slot s of every CTA in the cluster
      if (tid_wg < (uint32_t)C) {
        if (C > 1) mbar_arrive_cluster(&sm.empty_bar[s], tid_wg); else mbar_arrive(&sm.empty_bar[s]);
      }
    };
    for (int64_t t = cluster_id; t < n_tiles; t += n_clusters) {
      const int m_blk = (int)(t % n_mgrp) * C + (int)cta_rank;
      const int64_t n_blk = t / n_mgrp;
      int prev = -1;
      for (int kb = 0; kb < n_kblk; ++kb) {
        mbar_wait(&sm.full_bar[stage], phase);
        wgmma_fence();
        const uint32_t a_addr = smem_u32(sm.a[stage]) + (uint32_t)wg * (64 * kKBlockBytes), b_addr = smem_u32(sm.b[stage]);
#pragma unroll
        for (int k = 0; k < kGemmBK / kWgmmaK; ++k) {  // four 32-byte k-steps
          if constexpr (kI8)
            wgmma_m64n128k32_s8(acc, make_smem_desc(a_addr + k * 32), make_smem_desc(b_addr + k * 32), (kb | k) != 0 ? 1u : 0u);
          else
            wgmma_m64n128k16_bf16(acc, make_smem_desc(a_addr + k * kWgmmaK * 2), make_smem_desc(b_addr + k * kWgmmaK * 2), (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        if (prev >= 0) { wgmma_wait<1>(); release(prev); }  // the previous k-block's MMAs are done with their slot
        prev = stage;
        if (++stage == kGemmStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      release(prev);

      const int q_a = m_blk * kGemmBM + wg * 64 + (cw & 3) * 16 + (lane >> 2);
      int qs[2];
      float qq[2], bnd[2];
      int32_t qsq[2] = {0, 0};  // int8 L2
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        qs[h] = q_a + 8 * h;
        const bool q_ok = qs[h] < p.nq;
        if constexpr (kI8) {
          qq[h] = (q_ok && !is_l2) ? p.q_scale[qs[h]] : 0.0f;
          qsq[h] = (q_ok && is_l2) ? p.q_sq[qs[h]] : 0;
        } else {
          qq[h] = (q_ok && is_l2) ? p.q_scale[qs[h]] : 0.0f;
        }
        bnd[h] = q_ok ? p.bound[qs[h]] : __int_as_float(0x7f800000);  // +inf: nothing passes
      }
      const int64_t row0 = p.n0 + n_blk * kGemmBN;
      const int64_t left = p.n0 + p.n_rows - row0;  // rows of this tile that exist
#pragma unroll
      for (int c = 0; c < kGemmBN / 32; ++c) {  // 32 columns per round: 16 scores per thread
        float sc[16];
        uint32_t pass = 0;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int col = (c * 4 + jj) * 8 + col_l;
          float cc[2] = {0.0f, 0.0f};
          int32_t csq[2] = {0, 0};  // int8 L2
          if constexpr (kI8) {
            if (is_l2) {
              if (col < left) csq[0] = __ldg(p.c_sq + row0 + col);
              if (col + 1 < left) csq[1] = __ldg(p.c_sq + row0 + col + 1);
            } else {
              if (col < left) cc[0] = __ldg(p.c_scale + row0 + col);
              if (col + 1 < left) cc[1] = __ldg(p.c_scale + row0 + col + 1);
            }
          } else if (is_l2) {
            if (col < left) cc[0] = __ldg(p.c_scale + row0 + col);
            if (col + 1 < left) cc[1] = __ldg(p.c_scale + row0 + col + 1);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int idx = jj * 4 + h * 2 + e;
              float s;
              if constexpr (kI8) {
                s = i8_score(is_l2, acc[(c * 4 + jj) * 4 + h * 2 + e], qq[h], cc[e], qsq[h], csq[e]);
              } else {
                s = acc[(c * 4 + jj) * 4 + h * 2 + e];
                // cosine: operands are pre-normalised, the accumulator IS the similarity;
                // L2: score = -(|q|^2 + |c|^2 - 2 q.c)   (larger = closer)
                if (is_l2) s = 2.0f * s - qq[h] - cc[e];
              }
              sc[idx] = s;
              pass |= (s >= bnd[h] && col + e < left) ? (1u << idx) : 0u;
            }
          }
        }
        if (__any_sync(0xffffffffu, pass != 0)) {
          const int n = __popc(pass);
          int incl = n;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
          }
          const int total = __shfl_sync(0xffffffffu, incl, 31);
          const int excl = incl - n;
          if (total > kCandStage / 2) {
            // dense round (loose boundary in the first passes): reserve once per warp, write direct
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(p.cand_count, (unsigned long long)total);
            base = __shfl_sync(0xffffffffu, base, 0);
            if ((int64_t)(base + total) <= p.cand_cap) {
              unsigned long long pos = base + excl;
#pragma unroll
              for (int idx = 0; idx < 16; ++idx) {
                if ((pass >> idx) & 1) {
                  p.cand_key[pos] = ((uint64_t)(uint32_t)qs[(idx >> 1) & 1] << 32) | (uint64_t)(~f32_to_ordered32(sc[idx]));
                  p.cand_row[pos] = (uint32_t)(row0 + (c * 4 + (idx >> 2)) * 8 + col_l + (idx & 1));
                  ++pos;
                }
              }
            }
          } else {
            if (stage_cnt + total > kCandStage) {
              flush_stage(sm.stage_key[cw], sm.stage_row[cw], stage_cnt, lane, p);
              stage_cnt = 0;
            }
            int pos = stage_cnt + excl;
#pragma unroll
            for (int idx = 0; idx < 16; ++idx) {
              if ((pass >> idx) & 1) {
                sm.stage_key[cw][pos] = ((uint64_t)(uint32_t)qs[(idx >> 1) & 1] << 32) | (uint64_t)(~f32_to_ordered32(sc[idx]));
                sm.stage_row[cw][pos] = (uint32_t)(row0 + (c * 4 + (idx >> 2)) * 8 + col_l + (idx & 1));
                ++pos;
              }
            }
            stage_cnt += total;
            __syncwarp();
          }
        }
      }
    }
    flush_stage(sm.stage_key[cw], sm.stage_row[cw], stage_cnt, lane, p);
  }
  __syncwarp();
  if (C > 1) cluster_sync_all(); else __syncthreads();
}

// Reference similarity pass on CUDA cores (same bf16 inputs, f32 accumulation, same filter):
// used by the tests to validate the wgmma path (env DBX_KNN_REF_GEMM=1), never by default.
__global__ void knn_ref_filter_kernel(const __nv_bfloat16* q, const __nv_bfloat16* c, const __grid_constant__ KnnGemmParams p) {
  const int64_t total = (int64_t)p.nq * p.n_rows;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int qi = (int)(i / p.n_rows);
    const int64_t r = p.n0 + i % p.n_rows;
    const __nv_bfloat16* a = q + (int64_t)qi * p.dim_pad;
    const __nv_bfloat16* b = c + r * p.dim_pad;
    float dot = 0.0f;
    for (int k = 0; k < p.dim_pad; ++k) dot += __bfloat162float(a[k]) * __bfloat162float(b[k]);
    const float s = p.kind == DBX_DIST_COSINE ? dot : 2.0f * dot - p.q_scale[qi] - p.c_scale[r];
    if (s >= p.bound[qi]) {
      unsigned long long pos = atomicAdd(p.cand_count, 1ULL);
      if ((int64_t)pos < p.cand_cap) {
        p.cand_key[pos] = ((uint64_t)(uint32_t)qi << 32) | (uint64_t)(~f32_to_ordered32(s));
        p.cand_row[pos] = (uint32_t)r;
      }
    }
  }
}

// Reference similarity pass for int8 operands on CUDA cores: exact int32 dot product over the same
// padded operands, the same score and the same filter as the int8 wgmma kernel (DBX_KNN_REF_GEMM=1).
__global__ void knn_ref_filter_i8_kernel(const int8_t* q, const int8_t* c, const __grid_constant__ KnnGemmParams p) {
  const int64_t total = (int64_t)p.nq * p.n_rows;
  const bool is_l2 = p.kind != DBX_DIST_COSINE;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int qi = (int)(i / p.n_rows);
    const int64_t r = p.n0 + i % p.n_rows;
    const int8_t* a = q + (int64_t)qi * p.dim_pad;
    const int8_t* b = c + r * p.dim_pad;
    int32_t dot = 0;
    for (int k = 0; k < p.dim_pad; ++k) dot += (int32_t)a[k] * (int32_t)b[k];
    const float s = is_l2 ? i8_score(true, dot, 0.0f, 0.0f, p.q_sq[qi], p.c_sq[r]) : i8_score(false, dot, p.q_scale[qi], p.c_scale[r], 0, 0);
    if (s >= p.bound[qi]) {
      unsigned long long pos = atomicAdd(p.cand_count, 1ULL);
      if ((int64_t)pos < p.cand_cap) {
        p.cand_key[pos] = ((uint64_t)(uint32_t)qi << 32) | (uint64_t)(~f32_to_ordered32(s));
        p.cand_row[pos] = (uint32_t)r;
      }
    }
  }
}

}  // namespace dbx
