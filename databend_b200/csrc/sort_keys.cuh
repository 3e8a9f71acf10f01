// sort_keys.cuh — order-preserving key images and the stable multi-key device sort shared by
// DBX_OP_TOPK (ORDER BY without a LIMIT, sorts/...) and DBX_OP_WINDOW (WindowPartition's sort by
// PARTITION BY then ORDER BY keys).
#pragma once
#include <algorithm>

#include "radix_sort.cuh"
#include "runtime.h"

namespace dbx {
namespace {

// ================================================================ key images
// Key classes: VC_INT / VC_UINT / VC_FLT (Float64 bits) and KC_F32, a Float32 key carried in its own
// 32 bits.  A float -> double -> float round trip quiets a signalling NaN on sm_90 (0x7F800001 comes
// back as 0x7FC00001), and the result must return every row's key bit for bit.
constexpr int KC_F32 = 3;
inline int key_class(int dtype) {
  if (dtype == DBX_F32) return KC_F32;
  return dtype == DBX_U64 ? VC_UINT : (dtype_class(dtype) == VC_FLT ? VC_FLT : VC_INT);
}

__device__ __forceinline__ uint64_t key_to_ord(uint64_t bits, int cls, bool asc) {
  uint64_t o;
  if (cls == VC_FLT || cls == KC_F32) {
    double d = cls == KC_F32 ? (double)__uint_as_float((uint32_t)bits) : __longlong_as_double((long long)bits);
    if (d == 0.0) d = 0.0;  // -0 == +0
    o = f64_to_ordered(d);
  } else if (cls == VC_INT) {
    o = bits ^ 0x8000000000000000ULL;
  } else {
    o = bits;
  }
  return asc ? o : ~o;
}

// integers sign- or zero-extended to 64 bits; Float32 keeps its own 32 bits (see KC_F32)
__device__ __forceinline__ uint64_t load_widened(const DevCol& c, int64_t row, uint64_t pol) {
  const char* base = (const char*)c.data;
  switch (c.dtype) {
    case DBX_I64: case DBX_U64: case DBX_F64: return ld_stream_u64(base + row * 8, pol);
    case DBX_I32: return (uint64_t)(int64_t)(int32_t)ld_stream_u32(base + row * 4, pol);
    case DBX_U32: case DBX_F32: return ld_stream_u32(base + row * 4, pol);
    case DBX_I16: return (uint64_t)(int64_t)(int16_t)ld_stream_u16(base + row * 2, pol);
    case DBX_U16: return ld_stream_u16(base + row * 2, pol);
    case DBX_I8: return (uint64_t)(int64_t)(int8_t)ld_stream_u8(base + row, pol);
    default: return ld_stream_u8(base + row, pol);
  }
}

__device__ __forceinline__ void store_narrow_key(void* out, int64_t i, int dtype, uint64_t b) {
  switch (dtype) {
    case DBX_I8: case DBX_U8: ((uint8_t*)out)[i] = (uint8_t)b; break;
    case DBX_I16: case DBX_U16: ((uint16_t*)out)[i] = (uint16_t)b; break;
    case DBX_I32: case DBX_U32: case DBX_F32: ((uint32_t*)out)[i] = (uint32_t)b; break;
    default: ((uint64_t*)out)[i] = b; break;
  }
}

inline int grid_1d(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)kNumSMs * 8)); }

__global__ void pack_bits_kernel(const uint8_t* bytes, int64_t n, uint8_t* bits) {
  const int64_t nb = (n + 7) / 8;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (int64_t)gridDim.x * blockDim.x) {
    uint32_t v = 0;
    for (int k = 0; k < 8; ++k) {
      const int64_t i = b * 8 + k;
      if (i < n && bytes[i]) v |= 1u << k;
    }
    bits[b] = (uint8_t)v;
  }
}

// ================================================================ full sort: ingest
// Appends one chunk of the key column to the (ord, row id | NULL flag, original bits) arrays.
__global__ void __launch_bounds__(256) sort_ingest_kernel(const __grid_constant__ DevCol col, int64_t n, int64_t row_base, int cls, int asc,
                                                          uint64_t* ord, uint32_t* rid, uint64_t* bits, unsigned long long* n_null,
                                                          unsigned long long* inexact) {
  const uint64_t pol = make_policy_evict_first();
  unsigned int nulls = 0;
  bool lossy = false;  // -0.0 and NaN payloads do not survive key -> ordered image -> key
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const bool ok = !col.validity || bit_test(col.validity, col.vbit_off + i);
    const uint64_t v = ok ? load_widened(col, i, pol) : 0;
    ord[row_base + i] = ok ? key_to_ord(v, cls, asc != 0) : 0;  // NULL rows: placed by the extra pass on the flag
    rid[row_base + i] = (uint32_t)(row_base + i) | (ok ? 0u : 0x80000000u);
    if (bits) bits[row_base + i] = v;
    nulls += !ok;
    if (ok && cls == VC_FLT) {
      const double d = __longlong_as_double((long long)v);
      lossy |= (d != d && v != 0x7FF8000000000000ULL) || (d == 0.0 && (v >> 63));
    } else if (ok && cls == KC_F32) {
      const float f = __uint_as_float((uint32_t)v);
      lossy |= (f != f && v != 0x7FC00000u) || (f == 0.0f && (v >> 31));
    }
  }
  if (inexact && __any_sync(0xffffffffu, lossy) && (threadIdx.x & 31) == 0) *inexact = 1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nulls += __shfl_xor_sync(0xffffffffu, nulls, o);
  if ((threadIdx.x & 31) == 0 && nulls) atomicAdd(n_null, (unsigned long long)nulls);
}
// Multi-column ORDER BY: the keys of column c in the order the less significant columns have
// established so far (perm = sorted row id | flag of the previous step; nullptr = input order).
__global__ void __launch_bounds__(256) sort_gather_kernel(const uint64_t* ord_c, const uint32_t* rid_c, const uint32_t* perm, int64_t n,
                                                          uint64_t* o_ord, uint32_t* o_rid) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t r = perm ? (perm[i] & 0x7FFFFFFFu) : (uint32_t)i;
    o_ord[i] = ord_c[r];
    o_rid[i] = r | (rid_c[r] & 0x80000000u);
  }
}

// Stable sort of n rows by keys 0 .. n_keys - 1 (key 0 most significant).  ord[k] / rid[k] are
// what sort_ingest_kernel wrote for key k, in input order; n_nulls[k] its NULL rows.  One stable
// radix sort of (key image, row id) per key, least significant first, each in the order the
// previous steps established, so earlier keys dominate and input order breaks the last ties.
// The result (*sorted_ord, *sorted_rid: key 0's image and row id | key 0's NULL flag) lives in
// w_ord[*] / w_rid[*].  Needs n_keys >= 1 and n >= 2.
inline int32_t sort_rows_by_keys(ErrorSink& err, cudaStream_t stream, RadixSorter& sorter, int n_keys, const uint64_t* const* ord,
                                 const uint32_t* const* rid, const int64_t* n_nulls, const int32_t* nulls_first, int64_t n,
                                 DevBuf (&w_ord)[2], DevBuf (&w_rid)[2], const uint64_t** sorted_ord, const uint32_t** sorted_rid) {
  for (int i = 0; i < 2; ++i) { DBX_CUDA_TRY(err, w_ord[i].ensure((size_t)n * 8)); DBX_CUDA_TRY(err, w_rid[i].ensure((size_t)n * 4)); }
  int res = 1;  // which work pair holds the current order (none yet: the first gather goes to pair 0)
  const uint32_t* perm = nullptr;
  for (int c = n_keys - 1; c >= 0; --c) {
    const int in = res ^ 1;
    sort_gather_kernel<<<grid_1d(n), 256, 0, stream>>>(ord[c], rid[c], perm, n, (uint64_t*)w_ord[in].p, (uint32_t*)w_rid[in].p);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    int rb = 0;
    DBX_TRY(sorter.sort(err, stream, (uint64_t*)w_ord[in].p, (uint64_t*)w_ord[in ^ 1].p, (uint32_t*)w_rid[in].p, (uint32_t*)w_rid[in ^ 1].p, n, 0,
                        64, n_nulls[c] > 0, nulls_first[c], n_nulls[c], &rb));
    res = rb ? (in ^ 1) : in;
    perm = (const uint32_t*)w_rid[res].p;
  }
  *sorted_ord = (const uint64_t*)w_ord[res].p;
  *sorted_rid = (const uint32_t*)w_rid[res].p;
  return DBX_OK;
}

}  // namespace
}  // namespace dbx
