// common.cuh — shared host/device helpers for libdbx (sm_90a only).
#pragma once
#ifdef __CUDACC_RTC__  // run-time specialised kernels (agg_jit.cu): no host headers under NVRTC
typedef signed char int8_t;
typedef short int16_t;
typedef int int32_t;
typedef long long int64_t;
typedef unsigned char uint8_t;
typedef unsigned short uint16_t;
typedef unsigned int uint32_t;
typedef unsigned long long uint64_t;
typedef unsigned long long uintptr_t;
#define DBX_DEVICE_ONLY 1
#else
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <string>
#endif

#include "../../include/dbx.h"

namespace dbx {

constexpr int kNumSMs = 132;  // H100 SXM; grids are sized in multiples of this

#ifndef DBX_DEVICE_ONLY
// ---------------------------------------------------------------- error plumbing
struct ErrorSink {
  std::string msg;
  void set(const std::string& m) { msg = m; }
};
extern thread_local ErrorSink g_create_error;  // dbx_last_error(NULL)
extern std::atomic<int64_t> g_launches;        // dbx_kernel_launch_count()

#define DBX_CUDA_TRY(sink, expr)                                                              \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      (sink).set(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " #expr);        \
      return _e == cudaErrorMemoryAllocation ? DBX_ERR_OOM                                    \
             : (_e == cudaErrorNoDevice || _e == cudaErrorInsufficientDriver) ? DBX_ERR_NO_DEVICE \
                                                                              : DBX_ERR_CUDA; \
    }                                                                                         \
  } while (0)

#define DBX_TRY(expr)              \
  do {                             \
    int32_t _s = (expr);           \
    if (_s != DBX_OK) return _s;   \
  } while (0)

inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }
#endif  // !DBX_DEVICE_ONLY

// ---------------------------------------------------------------- dtype helpers
constexpr int kNullableFlag = 0x100;  // OR-ed into input_types[] for Nullable(T) columns

__host__ __device__ inline int dtype_size(int dt) {
  switch (dt) {
    case DBX_I8: case DBX_U8: return 1;
    case DBX_I16: case DBX_U16: return 2;
    case DBX_I32: case DBX_U32: case DBX_F32: return 4;
    case DBX_I64: case DBX_U64: case DBX_F64: return 8;
    default: return 0;
  }
}
// bytes of one row of a column: vectors are dim elements wide; 0 for BOOL (bit-packed)
__host__ __device__ inline int64_t column_row_bytes(int dt, int vec_dim) {
  return dt == DBX_VEC_F32 ? 4LL * vec_dim : dt == DBX_VEC_I8 ? (int64_t)vec_dim : (int64_t)dtype_size(dt);
}
__host__ __device__ inline bool is_vector_dtype(int dt) { return dt == DBX_VEC_F32 || dt == DBX_VEC_I8; }
enum ValClass : int { VC_INT = 0, VC_UINT = 1, VC_FLT = 2 };
__host__ __device__ inline int dtype_class(int dt) {
  switch (dt) {
    case DBX_I8: case DBX_I16: case DBX_I32: case DBX_I64: return VC_INT;
    case DBX_F32: case DBX_F64: return VC_FLT;
    default: return VC_UINT;
  }
}

// Device view of one input column (Buffer<T> + Bitmap), passed by value in kernel params.
struct DevCol {
  const void* data;
  const uint8_t* validity;  // nullptr: all valid
  int64_t vbit_off;
  int64_t dbit_off;         // DBX_BOOL data: bit offset of row 0
  uint64_t const_bits;      // is_const: the value widened to 64 bits (i64 / u64 / f64 bits)
  int32_t dtype;
  int32_t is_const;         // 1: BlockEntry::Const; 2: const NULL
};

// ---------------------------------------------------------------- device helpers
#ifdef __CUDACC__

// L2 cache policies (sm_90a has no .L2::evict_* qualifier on plain loads: every load takes a
// createpolicy descriptor through .L2::cache_hint).
__device__ __forceinline__ uint64_t make_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t make_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// Streaming loads: read-only path, no L1 allocation, evict-first in L2 so the column stream
// does not push the hash table out of the 50 MB L2.
struct u64x4 { uint64_t x, y, z, w; };
__device__ __forceinline__ uint64_t policy_evict_first_hoistable() {  // not volatile: loops share one policy
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// 32 bytes as two 128-bit loads (sm_90a has no 256-bit load)
__device__ __forceinline__ u64x4 ld_stream_256(const void* p) {
  const uint64_t pol = policy_evict_first_hoistable();
  u64x4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(r.x), "=l"(r.y) : "l"(p), "l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;"
               : "=l"(r.z), "=l"(r.w)
               : "l"((const char*)p + 16), "l"(pol));
  return r;
}
__device__ __forceinline__ uint4 ld_stream_128(const void* p, uint64_t pol) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint64_t ld_stream_u64(const void* p, uint64_t pol) {
  uint64_t r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint32_t ld_stream_u32(const void* p, uint64_t pol) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint16_t ld_stream_u16(const void* p, uint64_t pol) {
  uint16_t r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint8_t ld_stream_u8(const void* p, uint64_t pol) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
  return (uint8_t)r;
}

// Table accesses go to L2 (the point of coherence for the atomics).
__device__ __forceinline__ uint64_t ld_table_u64(const void* p) {
  uint64_t r;
  asm volatile("ld.global.relaxed.gpu.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void red_add_u64(void* p, uint64_t v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_add_f64(void* p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
// same, with an L2 eviction-priority hint (evict_last keeps the hash table resident while the
// column stream, loaded evict_first, passes through)
__device__ __forceinline__ void red_add_u64_hint(void* p, uint64_t v, uint64_t pol) {
  asm volatile("red.global.add.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void red_add_f64_hint(void* p, double v, uint64_t pol) {
  asm volatile("red.global.add.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void red_min_s64(void* p, int64_t v) {
  asm volatile("red.global.min.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_max_s64(void* p, int64_t v) {
  asm volatile("red.global.max.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_min_u64(void* p, uint64_t v) {
  asm volatile("red.global.min.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_max_u64(void* p, uint64_t v) {
  asm volatile("red.global.max.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// agg_hash for primitive keys (reference: src/query/expression/src/aggregate/group_hash.rs:555-570).
// Using the reference's hash keeps radix partitions compatible with a CPU operator.
__host__ __device__ __forceinline__ uint64_t agg_hash_u64(uint64_t x) {
  x ^= x >> 32;
  x *= 0xd6e8feb86659fd93ULL;
  x ^= x >> 32;
  x *= 0xd6e8feb86659fd93ULL;
  x ^= x >> 32;
  return x;
}
constexpr uint64_t kNullHashVal = 0xd1cefa08eb382d69ULL;  // group_hash.rs:38
// 128-bit packed keys (multi-column GROUP BY and join keys wider than 64 bits)
__device__ __forceinline__ uint64_t agg_hash_wide(uint64_t k0, uint64_t k1) {
  return agg_hash_u64(k0 ^ (agg_hash_u64(k1) + 0x9e3779b97f4a7c15ULL));
}

// Owner / partition of a hash among n parts: the top 32 hash bits scaled to [0, n), i.e.
// mulhi32(hash >> 32, n) — radix partitioning on the top bits (partitioned_payload.rs:44-57)
// generalised to any n.  Written with __umulhi on the device: the equivalent 64-bit
// multiply-and-shift form was miscompiled by ptxas 12.9 inside a shared-memory histogram loop
// (misaligned ATOMS address, found with compute-sanitizer).
__host__ __device__ __forceinline__ int hash_to_part(uint64_t h, int n) {
  const uint32_t hi = (uint32_t)(h >> 32);
#ifdef __CUDA_ARCH__
  return (int)__umulhi(hi, (uint32_t)n);
#else
  return (int)(((uint64_t)hi * (uint32_t)n) >> 32);
#endif
}

// Order-preserving map double -> u64 under OrderedFloat (NaN greatest, all NaN equal).
__device__ __forceinline__ uint64_t f64_to_ordered(double d) {
  if (d != d) return 0xFFFFFFFFFFFFFFFFULL;
  uint64_t b = (uint64_t)__double_as_longlong(d);
  return (b & 0x8000000000000000ULL) ? ~b : (b | 0x8000000000000000ULL);
}
#ifndef DBX_DEVICE_ONLY
__host__ __device__ __forceinline__ double ordered_to_f64(uint64_t o) {
  uint64_t b;
  if (o == 0xFFFFFFFFFFFFFFFFULL) b = 0x7FF8000000000000ULL;
  else b = (o & 0x8000000000000000ULL) ? (o & 0x7FFFFFFFFFFFFFFFULL) : ~o;
  double d;
  memcpy(&d, &b, 8);
  return d;
}
#endif

__device__ __forceinline__ bool bit_test(const uint8_t* bits, int64_t i) { return (bits[i >> 3] >> (i & 7)) & 1; }

// ---------------------------------------------------------------- mbarriers and bulk copies
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// `bytes` (a multiple of 16) from global `src` (16-byte aligned) to shared `dst` on the bulk-copy unit; the
// bytes are counted against `bar`'s transaction count.  `pol`: L2 cache policy of the reads.
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
               : "memory");
}

#endif  // __CUDACC__

}  // namespace dbx
