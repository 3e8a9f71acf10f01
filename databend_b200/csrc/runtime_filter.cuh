// runtime_filter.cuh — device tests of one join runtime-filter part, shared by the apply kernel
// (runtime_filter.cu) and the join's probe kernel (join.cu), plus the host interface between them.
//
// Reference (paths relative to the databend source tree, src/query):
//   split-block bloom filter: SALT, block index, mask, check    catalog/src/sbbf.rs:97-170,220-222
//   bloom hash of a KeysU8/U16/U32/U64 key (murmur3 fmix64)      common/hashtable/src/traits.rs:227-251
//   min-max / IN-list of the build keys                          service/.../hash_join/runtime_filter/local_builder.rs:94-118
//
// A key enters every test as the 64-bit image the join compares (load_key: sign- or zero-extended),
// which orders correctly in the pair's common type (signed: as int64, unsigned: as uint64).  The
// bloom hash reads the common type's bits: the image masked to its width, zero-extended.
#pragma once
#include <memory>

#include "runtime.h"

namespace dbx {

struct RfPartDev {
  const uint32_t* bloom;   // n_blocks blocks of 8 words, or null (no bloom)
  const uint64_t* inlist;  // n_inlist sorted images, or null (no IN-list)
  uint64_t lo, hi;         // min-max bounds (images); lo > hi rejects every key
  uint64_t mask;           // the common type's width
  uint32_t n_blocks;
  int32_t n_inlist;
  int32_t is_signed;       // common type signed: bounds and IN-list compare as int64
  int32_t has_min_max;
};

__host__ __device__ __forceinline__ uint64_t rf_fmix64(uint64_t h) {
  h ^= h >> 33;
  h *= 0xff51afd7ed558ccdULL;
  h ^= h >> 33;
  h *= 0xc4ceb9fe1a85ec53ULL;
  h ^= h >> 33;
  return h;
}
__host__ __device__ __forceinline__ uint32_t rf_salt(int i) {
  switch (i) {
    case 0: return 0x47b6137bu; case 1: return 0x44974d91u; case 2: return 0x8824ad5bu; case 3: return 0xa2b7289du;
    case 4: return 0x705495c7u; case 5: return 0x2df1424bu; case 6: return 0x9efc4947u; default: return 0x5c6bfb31u;
  }
}
__host__ __device__ __forceinline__ uint32_t rf_block_index(uint64_t h, uint32_t n_blocks) {
  return (uint32_t)(((h >> 32) * (uint64_t)n_blocks) >> 32);
}
__device__ __forceinline__ bool rf_less(uint64_t a, uint64_t b, bool is_signed) {
  return is_signed ? (int64_t)a < (int64_t)b : a < b;
}
__device__ __forceinline__ bool rf_min_max_pass(const RfPartDev& f, uint64_t v) {
  return !f.has_min_max || (!rf_less(v, f.lo, f.is_signed) && !rf_less(f.hi, v, f.is_signed));
}
// one 32-byte block = one sector: two 128-bit loads, every salted bit must be set
__device__ __forceinline__ bool rf_bloom_pass(const RfPartDev& f, uint64_t v) {
  if (!f.bloom) return true;
  const uint64_t h = rf_fmix64(v & f.mask);
  const uint4* blk = (const uint4*)(f.bloom + (size_t)rf_block_index(h, f.n_blocks) * 8);
  const uint4 a = __ldg(blk), b = __ldg(blk + 1);
  const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  const uint32_t x = (uint32_t)h;
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 8; ++i) ok &= (w[i] >> ((x * rf_salt(i)) >> 27)) & 1u;
  return ok;
}

// ---- host side: the built filter, shared by the handle and the join that probes with it
struct RfPart {
  int key_dtype = 0, probe_dtype = 0;
  bool has_min_max = false, has_inlist = false, has_bloom = false, any_key = false;
  bool is_signed = false;
  uint64_t mask = 0, lo = 0, hi = 0;
  int64_t n_inlist = 0, bloom_bytes = 0;
  DevBuf bloom, inlist;
  RfPartDev dev() const {
    RfPartDev d;
    memset(&d, 0, sizeof(d));
    d.bloom = has_bloom ? (const uint32_t*)bloom.p : nullptr;
    d.inlist = has_inlist ? (const uint64_t*)inlist.p : nullptr;
    d.n_inlist = (int32_t)n_inlist;
    d.n_blocks = (uint32_t)(bloom_bytes / 32);
    d.lo = any_key ? lo : 1;  // no non-NULL build key: an empty range
    d.hi = any_key ? hi : 0;
    d.mask = mask;
    d.is_signed = is_signed;
    d.has_min_max = has_min_max;
    return d;
  }
};
struct RfData {
  int device = 0;
  int n_parts = 0;
  int64_t build_rows = 0;
  RfPart parts[DBX_MAX_JOIN_KEYS];
  DevBuf probe_rejected;  // one counter, added to by the probe kernel
  std::atomic<int64_t> probe_checked{0};
  std::atomic<bool> in_probe{false};
};

// one build key column of the join: HBM-resident values and one validity byte per row (or null)
struct RfBuildKey {
  const void* data;
  const uint8_t* valid_bytes;
  int build_dtype, probe_dtype;
};
int32_t build_runtime_filter(ErrorSink& err, cudaStream_t stream, int device, const dbx_runtime_filter_params& p,
                             const RfBuildKey* keys, int n_keys, int64_t build_rows, std::shared_ptr<RfData>* out);
// the handle behind dbx_runtime_filter*
dbx_runtime_filter* make_runtime_filter_handle(std::shared_ptr<RfData> d);

}  // namespace dbx
