// sort.cu — DBX_OP_TOPK: `ORDER BY key [ASC|DESC] [NULLS FIRST|LAST] [LIMIT k]` on the device.
//
// Reference pipeline replaced (paths relative to the databend source tree):
//   TransformSortPartial (per block sort + limit)   src/query/pipeline/transforms/src/processors/transforms/sorts/sort_partial.rs:24-60
//     DataBlock::sort_with_type / SortCompare       src/query/expression/src/kernels/sort.rs:91-111, sort_compare.rs:197-296
//   limit-aware k-way merge                         sorts/sort_merge*.rs, sorts/core/{merger,loser_tree}.rs
//   fused TopN with a runtime boundary filter       src/query/service/src/pipelines/processors/transforms/top_n/transform_partial_top_n.rs:73-130
//
// Every key is mapped to an order-preserving u64 (OrderedFloat order: NaN greatest, -0 == +0,
// src/common/base/src/base/ordered_float.rs:147-201); ties are broken by ascending row id, as in
// the oracle.  Everything below is hand-written (no CUB):
//
//   several keys, LIMIT k the same streaming top-k on a composite order image of all keys (W <= 5
//   (k <= 4 Mi)           64-bit words, see "streaming top-k over several keys" below)
//   LIMIT k (k <= 4 Mi)   streaming top-k: the column is read ONCE (8 B/row, 256-bit streaming
//                         loads); a row survives only if it beats the boundary (the k-th best key
//                         so far — the reference's TopN boundary filter), kept in DEVICE memory and
//                         tightened by a one-CTA radix-select ("cut") kernel that runs between
//                         scan launches.  No host synchronisation between chunks: the host only
//                         chooses chunk sizes that provably fit the candidate list, or launches
//                         one optimistic scan over the rest and checks an overflow flag once.
//   no LIMIT (limit = 0)  full sort: (ordered key, row id) pairs are radix-sorted with a
//                         onesweep-style LSD sort (one global histogram pass for all digits, then
//                         one read+write pass per 8-bit digit with decoupled look-back between
//                         tiles); LSD passes are stable, so equal keys stay in row order.
#include <algorithm>
#include <vector>

#include "sort_keys.cuh"

namespace dbx {

namespace {

// (the key images and the multi-key sort live in sort_keys.cuh, the radix sort in radix_sort.cuh)
// ================================================================ streaming top-k
// Device state words of one candidate list
enum : int { ST_COUNT = 0, ST_BOUND = 1, ST_OVERFLOW = 2, ST_WORDS = 4 };

struct CandList {
  uint64_t* ord;    // order-preserving image (nullptr: list keyed by row id only — the NULL rows)
  uint64_t* rowid;  // global row ordinal
  uint64_t* bits;   // original value bits (nullptr for the NULL list)
  unsigned long long* state;  // [ST_WORDS]
  int64_t cap;
};

__device__ __forceinline__ void cand_append_warp(const CandList& l, bool keep, uint64_t o, uint64_t rid, uint64_t b, int lane) {
  const uint32_t bal = __ballot_sync(0xffffffffu, keep);
  if (!bal) return;
  unsigned long long base = 0;
  if (lane == __ffs(bal) - 1) base = atomicAdd(&l.state[ST_COUNT], (unsigned long long)__popc(bal));
  base = __shfl_sync(0xffffffffu, base, __ffs(bal) - 1);
  if (keep) {
    const unsigned long long pos = base + __popc(bal & ((1u << lane) - 1));
    if ((int64_t)pos < l.cap) {
      if (l.ord) l.ord[pos] = o;
      l.rowid[pos] = rid;
      if (l.bits) l.bits[pos] = b;
    } else {
      l.state[ST_OVERFLOW] = 1;  // never silently: the host replays the chunk in pieces that fit
    }
  }
}

// One pass over `n` rows of the key column.  Only ord <= boundary (read from device memory) can
// still be in the top k.  FAST: 8-byte column, 32 B aligned, no validity: a tile is 2048 rows, two
// 256-bit loads per thread, and the next tile's two loads are issued before this tile is examined
// (128 B in flight per thread); the grid is exactly the number of resident CTAs.
template <bool FAST>
__global__ void __launch_bounds__(256) topk_scan_kernel(const __grid_constant__ DevCol col, int64_t n, int64_t row_base, int cls,
                                                        int asc, const __grid_constant__ CandList cand,
                                                        const __grid_constant__ CandList nulls) {
  const uint64_t pol = make_policy_evict_first();
  const int lane = threadIdx.x & 31;
  const uint64_t boundary = cand.state[ST_BOUND];
  const uint64_t null_boundary = nulls.rowid ? nulls.state[ST_BOUND] : 0;
  if (FAST) {
    const int64_t n_tiles = n / 2048;  // whole tiles; the tail goes through the generic loop below
    const char* base = (const char*)col.data;
    u64x4 q0, q1;
    q0.x = q0.y = q0.z = q0.w = q1.x = q1.y = q1.z = q1.w = 0;
    int64_t tile = blockIdx.x;
    if (tile < n_tiles) {
      q0 = ld_stream_256(base + (tile * 2048 + 4 * (int64_t)threadIdx.x) * 8);
      q1 = ld_stream_256(base + (tile * 2048 + 1024 + 4 * (int64_t)threadIdx.x) * 8);
    }
    for (; tile < n_tiles; tile += gridDim.x) {
      __syncwarp();
      const u64x4 c0 = q0, c1 = q1;
      const int64_t nt = tile + gridDim.x;
      if (nt < n_tiles) {
        q0 = ld_stream_256(base + (nt * 2048 + 4 * (int64_t)threadIdx.x) * 8);
        q1 = ld_stream_256(base + (nt * 2048 + 1024 + 4 * (int64_t)threadIdx.x) * 8);
      }
      const uint64_t v[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      uint64_t o[8];
      bool any = false;
#pragma unroll
      for (int j = 0; j < 8; ++j) { o[j] = key_to_ord(v[j], cls, asc != 0); any |= o[j] <= boundary; }
      if (!__any_sync(0xffffffffu, any)) continue;  // the common case once the boundary is tight
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int64_t r = tile * 2048 + (j >> 2) * 1024 + 4 * (int64_t)threadIdx.x + (j & 3);
        cand_append_warp(cand, o[j] <= boundary, o[j], (uint64_t)(row_base + r), v[j], lane);
      }
    }
  }
  const int64_t first = FAST ? (n / 2048) * 2048 : 0;
  const int64_t n_tiles = (n - first + 1023) / 1024;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    __syncwarp();
    const int64_t r0 = first + tile * 1024 + 4 * (int64_t)threadIdx.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool in = r0 + j < n;
      const bool ok = in && (!col.validity || bit_test(col.validity, col.vbit_off + r0 + j));
      const uint64_t v = ok ? load_widened(col, r0 + j, pol) : 0;
      const uint64_t o = key_to_ord(v, cls, asc != 0);
      const uint64_t rid = (uint64_t)(row_base + r0 + j);
      cand_append_warp(cand, ok && o <= boundary, o, rid, v, lane);
      if (nulls.rowid) cand_append_warp(nulls, in && !ok && rid <= null_boundary, 0, rid, 0, lane);
    }
  }
}

// Radix select inside ONE CTA: keep the k smallest entries of a candidate list under the
// (ord, rowid) order, compact them to the front and publish the new boundary (the k-th entry's
// ord; for the NULL list its row id).  MSD passes over 8-bit digits of the 128-bit key only build
// a 256-bin histogram of the entries that still match the prefix found so far; the loop ends as
// soon as the bucket that contains the k-th entry is taken whole.  Does nothing when the list
// holds <= threshold entries.
struct CutArgs {
  CandList l;
  uint64_t* alt_ord;    // [k] scratch
  uint64_t* alt_rowid;
  uint64_t* alt_bits;
  int64_t k;
  int64_t threshold;
};
constexpr int kCutActive = 4096;  // entries of the bucket under examination kept in shared memory
// bucket that contains the k_rem-th entry of a 256-bin histogram: warp 0, eight bins per lane
__device__ __forceinline__ void cut_find_bucket(const unsigned int* hist, int64_t k_rem, unsigned int* out3, int tid) {
  if (tid >= 32) return;
  unsigned int c[8], sum = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) { c[j] = hist[tid * 8 + j]; sum += c[j]; }
  unsigned int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int up = __shfl_up_sync(0xffffffffu, incl, o);
    if (tid >= o) incl += up;
  }
  unsigned int cum = incl - sum;
  // the lane whose range [cum, cum + sum) contains the k_rem-th entry (k_rem >= 1)
  const bool mine = (int64_t)cum < k_rem && k_rem <= (int64_t)cum + sum;
  const unsigned int total = __shfl_sync(0xffffffffu, incl, 31);
  if (mine) {
    int b = 0;
    for (; b < 7; ++b) {
      if ((int64_t)cum + c[b] >= k_rem) break;
      cum += c[b];
    }
    out3[0] = (unsigned)(tid * 8 + b); out3[1] = cum; out3[2] = c[b];
  } else if (tid == 31 && (int64_t)total < k_rem) {  // cannot happen (k_rem <= matching entries); keep the state sane
    out3[0] = 255; out3[1] = total - c[7]; out3[2] = c[7];
  }
}
__global__ void __launch_bounds__(1024) topk_cut_kernel(const __grid_constant__ CutArgs a) {
  __shared__ unsigned int s_hist[256];
  __shared__ unsigned int s_pick[3];  // bucket, entries before it, entries in it
  __shared__ unsigned int s_out, s_nact;
  extern __shared__ __align__(16) uint64_t s_cut_dyn[];  // active set (ord, rowid) once the bucket is small
  uint64_t* s_ao = s_cut_dyn;
  uint64_t* s_ar = s_cut_dyn + kCutActive;
  const CandList& l = a.l;
  const int64_t cnt = (int64_t)l.state[ST_COUNT];
  const int64_t n = cnt < l.cap ? cnt : l.cap;
  if (n <= a.threshold || n <= a.k) return;
  const int tid = threadIdx.x, lane = tid & 31;
  uint64_t th_hi = 0, th_lo = 0;  // prefix of the threshold key (ord, rowid)
  int64_t k_rem = a.k;
  bool closed = false;
  bool in_smem = false;   // the entries that still match the prefix sit in s_ao / s_ar
  int64_t n_act = n;      // entries matching the prefix found so far
  for (int p = l.ord ? 0 : 8; p < 16 && !closed; ++p) {
    if (tid < 256) s_hist[tid] = 0;
    if (tid == 0) s_nact = 0;
    __syncthreads();
    const int sh = 56 - 8 * (p & 7);
    // a bucket that fits is first copied to shared memory (same pass as its histogram)
    const bool gather = !in_smem && n_act <= kCutActive;
    const int64_t n_scan = in_smem ? n_act : n;
    for (int64_t i0 = tid - lane; i0 < n_scan; i0 += 1024) {
      const int64_t i = i0 + lane;
      bool m = i < n_scan;
      int d = 0;
      uint64_t o = 0, r = 0;
      if (m) {
        if (in_smem) { o = s_ao[i]; r = s_ar[i]; }
        else { o = l.ord ? l.ord[i] : 0; r = l.rowid[i]; }
        if (p < 8) {
          m = in_smem || p == 0 || (o >> (sh + 8)) == (th_hi >> (sh + 8));
          d = (int)((o >> sh) & 255);
        } else {
          m = in_smem || (o == th_hi && (p == 8 || (r >> (sh + 8)) == (th_lo >> (sh + 8))));
          d = (int)((r >> sh) & 255);
        }
      }
      const unsigned mm = __ballot_sync(0xffffffffu, m);
      if (!mm) continue;
      if (gather) {  // (all matching entries of this pass: exactly n_act of them)
        unsigned int base = 0;
        if (lane == __ffs(mm) - 1) base = atomicAdd(&s_nact, (unsigned)__popc(mm));
        base = __shfl_sync(0xffffffffu, base, __ffs(mm) - 1);
        if (m) {
          const unsigned int q = base + __popc(mm & ((1u << lane) - 1));
          if (q < (unsigned)kCutActive) { s_ao[q] = o; s_ar[q] = r; }
        }
      }
      const int d0 = __shfl_sync(0xffffffffu, d, __ffs(mm) - 1);
      const unsigned same = __ballot_sync(0xffffffffu, m && d == d0);
      if (same == mm) { if (lane == __ffs(mm) - 1) atomicAdd(&s_hist[d0], (unsigned)__popc(mm)); }
      else if (m) atomicAdd(&s_hist[d], 1u);
    }
    __syncthreads();
    cut_find_bucket(s_hist, k_rem, s_pick, tid);
    __syncthreads();
    const uint64_t bkt = s_pick[0];
    if (p < 8) th_hi |= bkt << sh; else th_lo |= bkt << sh;
    k_rem -= s_pick[1];
    if (gather) {
      // the gathered set matched the OLD prefix; keep only the chosen bucket for the next passes
      in_smem = true;
      __syncthreads();
      // in-place compaction by one warp-strided sweep through a second counter
      if (tid == 0) s_out = 0;
      __syncthreads();
      uint64_t ko[(kCutActive + 1023) / 1024], kr[(kCutActive + 1023) / 1024];
      bool kk[(kCutActive + 1023) / 1024];
#pragma unroll
      for (int t = 0; t < (kCutActive + 1023) / 1024; ++t) {
        const int64_t i = tid + 1024 * t;
        kk[t] = false;
        if (i < n_act) {
          ko[t] = s_ao[i]; kr[t] = s_ar[i];
          const int d = p < 8 ? (int)((ko[t] >> sh) & 255) : (int)((kr[t] >> sh) & 255);
          kk[t] = d == (int)bkt;
        }
      }
      __syncthreads();
#pragma unroll
      for (int t = 0; t < (kCutActive + 1023) / 1024; ++t) {
        if (kk[t]) { const unsigned int q = atomicAdd(&s_out, 1u); s_ao[q] = ko[t]; s_ar[q] = kr[t]; }
      }
      __syncthreads();
    } else if (in_smem) {
      // narrow the shared-memory set to the chosen bucket
      if (tid == 0) s_out = 0;
      __syncthreads();
      uint64_t ko[(kCutActive + 1023) / 1024], kr[(kCutActive + 1023) / 1024];
      bool kk[(kCutActive + 1023) / 1024];
#pragma unroll
      for (int t = 0; t < (kCutActive + 1023) / 1024; ++t) {
        const int64_t i = tid + 1024 * t;
        kk[t] = false;
        if (i < n_act) {
          ko[t] = s_ao[i]; kr[t] = s_ar[i];
          const int d = p < 8 ? (int)((ko[t] >> sh) & 255) : (int)((kr[t] >> sh) & 255);
          kk[t] = d == (int)bkt;
        }
      }
      __syncthreads();
#pragma unroll
      for (int t = 0; t < (kCutActive + 1023) / 1024; ++t) {
        if (kk[t]) { const unsigned int q = atomicAdd(&s_out, 1u); s_ao[q] = ko[t]; s_ar[q] = kr[t]; }
      }
      __syncthreads();
    }
    n_act = s_pick[2];
    if ((int64_t)s_pick[2] == k_rem) {  // the whole bucket is in: every key with this prefix passes
      const uint64_t low = sh ? ((1ULL << sh) - 1) : 0;
      if (p < 8) { th_hi |= low; th_lo = ~0ULL; } else { th_lo |= low; }
      closed = true;
    }
    __syncthreads();
  }
  // compaction of the entries <= threshold into the scratch arrays (at most k of them)
  if (tid == 0) s_out = 0;
  __syncthreads();
  for (int64_t i0 = tid - lane; i0 < n; i0 += 1024) {
    const int64_t i = i0 + lane;
    uint64_t o = 0, r = 0;
    bool keep = false;
    if (i < n) {
      o = l.ord ? l.ord[i] : 0;
      r = l.rowid[i];
      keep = o < th_hi || (o == th_hi && r <= th_lo);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (!bal) continue;
    unsigned int base = 0;
    if (lane == __ffs(bal) - 1) base = atomicAdd(&s_out, (unsigned)__popc(bal));
    base = __shfl_sync(0xffffffffu, base, __ffs(bal) - 1);
    if (keep) {
      const unsigned int q = base + __popc(bal & ((1u << lane) - 1));
      if ((int64_t)q < a.k) {
        if (l.ord) a.alt_ord[q] = o;
        a.alt_rowid[q] = r;
        if (l.bits) a.alt_bits[q] = l.bits[i];
      }
    }
  }
  __syncthreads();
  const int64_t kept = (int64_t)s_out < a.k ? (int64_t)s_out : a.k;
  for (int64_t i = tid; i < kept; i += 1024) {
    if (l.ord) l.ord[i] = a.alt_ord[i];
    l.rowid[i] = a.alt_rowid[i];
    if (l.bits) l.bits[i] = a.alt_bits[i];
  }
  if (tid == 0) {
    l.state[ST_COUNT] = (unsigned long long)kept;
    l.state[ST_BOUND] = l.ord ? th_hi : th_lo;
  }
}

// Sort n <= 4096 candidates by (ord, rowid) inside one CTA by counting, for every entry, the
// entries that precede it (n^2 / 1024 comparisons per thread out of shared memory).
__global__ void __launch_bounds__(1024) small_rank_sort_kernel(const uint64_t* ord, const uint64_t* rowid, const uint64_t* bits, int n,
                                                               uint64_t* out_rowid, uint64_t* out_bits) {
  extern __shared__ __align__(16) uint64_t s_kr[];  // [n] ord, [n] rowid
  uint64_t* s_o = s_kr;
  uint64_t* s_r = s_kr + n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { s_o[i] = ord ? ord[i] : 0; s_r[i] = rowid[i]; }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const uint64_t o = s_o[i], r = s_r[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += (s_o[j] < o) || (s_o[j] == o && s_r[j] < r);
    out_rowid[rank] = r;
    if (bits) out_bits[rank] = bits[i];
  }
}

__global__ void topk_reset_kernel(unsigned long long* state) {
  if (threadIdx.x < 3 * ST_WORDS) state[threadIdx.x] = (threadIdx.x % ST_WORDS) == ST_BOUND && threadIdx.x < 2 * ST_WORDS ? ~0ULL : 0ULL;
}
__global__ void iota_u32_kernel(uint32_t* p, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = (uint32_t)i;
}
__global__ void gather_u64_kernel(const uint64_t* src, const uint32_t* idx, uint64_t* dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}

// Assemble the result block on the device: [key (original dtype, Nullable), row_id Int64].
struct EmitArgs {
  const uint64_t* bits;    // sorted valid rows: original value bits
  const uint64_t* rowid;   // sorted valid rows
  const uint64_t* null_rowid;  // sorted NULL rows
  int64_t take_valid, take_null;
  int32_t nulls_first, dtype;
  void* out_key;
  int64_t* out_row;
  uint8_t* out_valid_bytes;  // one byte per row
};
__global__ void topk_emit_kernel(const __grid_constant__ EmitArgs a) {
  const int64_t n_out = a.take_valid + a.take_null;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t first = a.nulls_first ? a.take_null : a.take_valid;
    const bool in_first = i < first;
    const bool is_null = a.nulls_first ? in_first : !in_first;
    const int64_t j = in_first ? i : i - first;
    if (is_null) {
      store_narrow_key(a.out_key, i, a.dtype, 0);
      a.out_row[i] = (int64_t)a.null_rowid[j];
      a.out_valid_bytes[i] = 0;
    } else {
      store_narrow_key(a.out_key, i, a.dtype, a.bits[j]);
      a.out_row[i] = (int64_t)a.rowid[j];
      a.out_valid_bytes[i] = 1;
    }
  }
}
struct SortEmitArgs {
  const uint32_t* rid;   // sorted: row id | NULL flag
  const uint64_t* bits;  // by original row id; nullptr: invert the sorted ordered images instead (no gather)
  const uint64_t* ord;   // sorted ordered images
  int32_t cls, asc;
  int64_t n;
  int32_t dtype;
  void* out_key;
  int64_t* out_row;
  uint8_t* out_valid_bytes;  // nullptr: key not nullable
};
__global__ void sort_emit_kernel(const __grid_constant__ SortEmitArgs a) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t r = a.rid[i];
    const uint32_t row = r & 0x7FFFFFFFu;
    const bool is_null = r >> 31;
    uint64_t b = 0;
    if (!is_null) {
      if (a.bits) b = a.bits[row];
      else {
        const uint64_t o = a.asc ? a.ord[i] : ~a.ord[i];
        if (a.cls == KC_F32) {  // the image of a NaN decodes to the canonical 0x7FC00000 (others are gathered)
          const double d = ordered_to_f64(o);
          b = d != d ? 0x7FC00000u : __float_as_uint((float)d);
        } else {
          b = a.cls == VC_FLT ? (uint64_t)__double_as_longlong(ordered_to_f64(o)) : (a.cls == VC_INT ? o ^ 0x8000000000000000ULL : o);
        }
      }
    }
    store_narrow_key(a.out_key, i, a.dtype, b);
    a.out_row[i] = (int64_t)row;
    if (a.out_valid_bytes) a.out_valid_bytes[i] = is_null ? 0 : 1;
  }
}

// ================================================================ streaming top-k over several keys
// ORDER BY k0, k1, ... LIMIT k runs the same candidate list / boundary / cut machinery as one key,
// on a composite order image: every row's keys packed into one big-endian unsigned integer of W
// 64-bit words whose lexicographic order is the ORDER BY order (the reference builds the same thing
// as a byte-comparable row encoding, sorts/core/row_convert/fixed_encode.rs:22-57).  Per key, most
// significant first:
//   nullable key   one placement bit: NULLS FIRST: NULL 0, valid 1; NULLS LAST: NULL 1, valid 0
//   value          the key's natural width (8/16/32/64 bits); signed integers with the sign bit
//                  flipped, floats as their OrderedFloat image (-0 == +0, every NaN greatest),
//                  complemented for DESC; 0 on a NULL row, so NULL rows tie and later keys decide
// Fields may straddle words: the image is only compared, never decoded.  4 x 65 bits: W <= 5.
constexpr int kMaxImageWords = 5;
enum : int { MST_NULLS = 3, MST_BOUND = ST_WORDS };  // multi-key state: [count, -, overflow, nulls emitted, boundary[W]]

struct MultiKeys {
  DevCol col[DBX_MAX_SORT_KEYS];      // col[0] is the first key
  int32_t off[DBX_MAX_SORT_KEYS];     // bit offset of the key's first field, from the image's top bit
  int32_t width[DBX_MAX_SORT_KEYS];   // value field bits
  int32_t nullable[DBX_MAX_SORT_KEYS];
  int32_t nulls_first[DBX_MAX_SORT_KEYS];
  int32_t asc[DBX_MAX_SORT_KEYS];
  int32_t n_keys;
  int32_t lead_bits;  // bits taken by the first key (placement bit + value): <= 65
};

// Host side of the layout: field offsets per key and the number of image words.
inline int multi_key_layout(const int* dtypes, const bool* nullable, int n_keys, MultiKeys* mk) {
  int bit = 0;
  for (int k = 0; k < n_keys; ++k) {
    mk->off[k] = bit;
    mk->nullable[k] = nullable[k] ? 1 : 0;
    mk->width[k] = 8 * dtype_size(dtypes[k]);
    bit += mk->nullable[k] + mk->width[k];
    if (k == 0) mk->lead_bits = bit;
  }
  mk->n_keys = n_keys;
  return (bit + 63) / 64;
}

// The value field of one key (widened bits as load_widened returns them), `width` bits wide.
__device__ __forceinline__ uint64_t key_field(uint64_t v, int dtype, int width, bool asc) {
  const uint64_t mask = width == 64 ? ~0ULL : (1ULL << width) - 1;
  uint64_t o;
  if (dtype == DBX_F64) {
    double d = __longlong_as_double((long long)v);
    if (d == 0.0) d = 0.0;  // -0 == +0
    o = f64_to_ordered(d);
  } else if (dtype == DBX_F32) {
    float f = __uint_as_float((uint32_t)v);
    uint32_t u;
    if (f != f) u = 0xFFFFFFFFu;
    else {
      if (f == 0.0f) f = 0.0f;
      u = __float_as_uint(f);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    }
    o = u;
  } else if (dtype == DBX_I8 || dtype == DBX_I16 || dtype == DBX_I32 || dtype == DBX_I64) {
    o = (v ^ (1ULL << (width - 1))) & mask;
  } else {
    o = v & mask;
  }
  return asc ? o : o ^ mask;
}

// OR the `wd`-bit value v into the image at bit `off` (counted from the top bit of word 0)
template <int W>
__device__ __forceinline__ void img_put(uint64_t (&img)[W], int off, int wd, uint64_t v) {
  const int w0 = off >> 6, end = (off & 63) + wd;  // end <= 128
#pragma unroll
  for (int w = 0; w < W; ++w) {
    if (w == w0) img[w] |= end <= 64 ? v << (64 - end) : v >> (end - 64);
    if (w == w0 + 1 && end > 64) img[w] |= v << (128 - end);
  }
}

template <int W>
__device__ __forceinline__ void img_put_key(const MultiKeys& mk, int k, bool ok, uint64_t v, uint64_t (&img)[W]) {
  int off = mk.off[k];
  if (mk.nullable[k]) { img_put(img, off, 1, (uint64_t)(ok == (mk.nulls_first[k] != 0))); ++off; }
  if (ok) img_put(img, off, mk.width[k], key_field(v, mk.col[k].dtype, mk.width[k], mk.asc[k] != 0));
}

template <int W>
__device__ __forceinline__ bool img_le(const uint64_t (&a)[W], const uint64_t (&b)[W]) {
#pragma unroll
  for (int w = 0; w < W; ++w)
    if (a[w] != b[w]) return a[w] < b[w];
  return true;
}

// The image of row r (first key already loaded: ok0, v0) if it can still be in the top k, i.e.
// image <= boundary.  The first key's fields are compared first (bl0, bl1: the same bits of the
// boundary); the later key columns are read only when they are not greater.
template <int W>
__device__ __forceinline__ bool multi_row(const MultiKeys& mk, int64_t r, bool ok0, uint64_t v0, const uint64_t (&bound)[W], uint64_t bl0,
                                          uint64_t bl1, uint64_t pol, uint64_t (&img)[W]) {
#pragma unroll
  for (int w = 0; w < W; ++w) img[w] = 0;
  img_put_key(mk, 0, ok0, v0, img);
  if (img[0] > bl0) return false;
  if (W > 1 && img[0] == bl0 && img[W > 1 ? 1 : 0] > bl1) return false;  // word 1 holds first-key bits only for a 65-bit key
#pragma unroll
  for (int k = 1; k < DBX_MAX_SORT_KEYS; ++k) {
    if (k >= mk.n_keys) break;
    const DevCol& c = mk.col[k];
    const bool ok = !c.validity || bit_test(c.validity, c.vbit_off + r);
    img_put_key(mk, k, ok, ok ? load_widened(c, r, pol) : 0, img);
  }
  return img_le(img, bound);
}

// One candidate list for all rows (NULL rows included: their placement bits order them).
struct MultiList {
  uint64_t* img;    // [W][cap]: image word w of entry i at img[w * cap + i]
  uint64_t* rowid;  // global row ordinal
  uint64_t* bits;   // the first key's original value bits (as load_widened returns them), 0 for NULL
  unsigned long long* state;  // MST_* words
  int64_t cap;
};

template <int W>
__device__ __forceinline__ void mcand_append_warp(const MultiList& l, bool keep, const uint64_t (&img)[W], uint64_t rid, uint64_t b, int lane) {
  const uint32_t bal = __ballot_sync(0xffffffffu, keep);
  if (!bal) return;
  unsigned long long base = 0;
  if (lane == __ffs(bal) - 1) base = atomicAdd(&l.state[ST_COUNT], (unsigned long long)__popc(bal));
  base = __shfl_sync(0xffffffffu, base, __ffs(bal) - 1);
  if (keep) {
    const unsigned long long pos = base + __popc(bal & ((1u << lane) - 1));
    if ((int64_t)pos < l.cap) {
#pragma unroll
      for (int w = 0; w < W; ++w) l.img[w * l.cap + pos] = img[w];
      l.rowid[pos] = rid;
      l.bits[pos] = b;
    } else {
      l.state[ST_OVERFLOW] = 1;
    }
  }
}

// topk_scan_kernel for a composite image: the first key is read densely (FAST: 8-byte column, 32 B
// aligned, no validity: 256-bit streaming loads with the next tile prefetched); a row whose first
// key is beyond the boundary's is rejected without touching the other key columns.  Launched with
// 256 threads; 80 registers (3 CTAs per SM) leave the W = 1 .. 5 instantiations without spills.
template <int W, bool FAST>
__global__ void __maxnreg__(80) topk_multi_scan_kernel(const __grid_constant__ MultiKeys mk, int64_t n, int64_t row_base,
                                                              const __grid_constant__ MultiList cand) {
  const uint64_t pol = make_policy_evict_first();
  const int lane = threadIdx.x & 31;
  uint64_t bound[W];
#pragma unroll
  for (int w = 0; w < W; ++w) bound[w] = cand.state[MST_BOUND + w];
  const int lb = mk.lead_bits;
  const uint64_t bl0 = bound[0] & (lb >= 64 ? ~0ULL : ~(~0ULL >> lb));
  const uint64_t bl1 = W > 1 && lb > 64 ? bound[W > 1 ? 1 : 0] & 0x8000000000000000ULL : 0;
  const DevCol& col = mk.col[0];
  uint64_t img[W];
  if (FAST) {
    const int64_t n_tiles = n / 2048;
    const char* base = (const char*)col.data;
    u64x4 q0, q1;
    q0.x = q0.y = q0.z = q0.w = q1.x = q1.y = q1.z = q1.w = 0;
    int64_t tile = blockIdx.x;
    if (tile < n_tiles) {
      q0 = ld_stream_256(base + (tile * 2048 + 4 * (int64_t)threadIdx.x) * 8);
      q1 = ld_stream_256(base + (tile * 2048 + 1024 + 4 * (int64_t)threadIdx.x) * 8);
    }
    for (; tile < n_tiles; tile += gridDim.x) {
      __syncwarp();
      const u64x4 c0 = q0, c1 = q1;
      const int64_t nt = tile + gridDim.x;
      if (nt < n_tiles) {
        q0 = ld_stream_256(base + (nt * 2048 + 4 * (int64_t)threadIdx.x) * 8);
        q1 = ld_stream_256(base + (nt * 2048 + 1024 + 4 * (int64_t)threadIdx.x) * 8);
      }
      const uint64_t v[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      bool any = false;
#pragma unroll
      for (int j = 0; j < 8; ++j) {  // first key only (a non-nullable 64-bit key: one word)
        const uint64_t f = key_field(v[j], col.dtype, 64, mk.asc[0] != 0);
        any |= f <= bl0;
      }
      if (!__any_sync(0xffffffffu, any)) continue;  // the common case once the boundary is tight
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int64_t r = tile * 2048 + (j >> 2) * 1024 + 4 * (int64_t)threadIdx.x + (j & 3);
        const bool keep = multi_row(mk, r, true, v[j], bound, bl0, bl1, pol, img);
        mcand_append_warp(cand, keep, img, (uint64_t)(row_base + r), v[j], lane);
      }
    }
  }
  const int64_t first = FAST ? (n / 2048) * 2048 : 0;
  const int64_t n_tiles = (n - first + 1023) / 1024;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    __syncwarp();
    const int64_t r0 = first + tile * 1024 + 4 * (int64_t)threadIdx.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool in = r0 + j < n;
      const bool ok = in && (!col.validity || bit_test(col.validity, col.vbit_off + r0 + j));
      const uint64_t v = ok ? load_widened(col, r0 + j, pol) : 0;
      bool keep = false;
      if (in) keep = multi_row(mk, r0 + j, ok, v, bound, bl0, bl1, pol, img);
      mcand_append_warp(cand, keep, img, (uint64_t)(row_base + r0 + j), v, lane);
    }
  }
}

// topk_cut_kernel over (W image words, row id): MSD 8-bit digit passes over 8 (W + 1) digits; the
// loop ends as soon as the bucket that contains the k-th entry is taken whole.  Publishes the
// k-th image (or an upper bound of it) as the W-word boundary.
struct MultiCutArgs {
  MultiList l;
  uint64_t* alt_img;  // [W][k] scratch
  uint64_t* alt_rowid;
  uint64_t* alt_bits;
  int64_t k;
  int64_t threshold;
};
template <int E>
__device__ __forceinline__ uint64_t word_at(const uint64_t (&e)[E], int q) {
  uint64_t x = e[0];
#pragma unroll
  for (int w = 1; w < E; ++w)
    if (q == w) x = e[w];
  return x;
}
template <int W>
__global__ void __launch_bounds__(1024) topk_multi_cut_kernel(const __grid_constant__ MultiCutArgs a) {
  constexpr int E = W + 1;  // entry: image words, row id
  constexpr int T = (kCutActive + 1023) / 1024;
  __shared__ unsigned int s_hist[256];
  __shared__ unsigned int s_pick[3];
  __shared__ unsigned int s_out, s_nact;
  extern __shared__ __align__(16) uint64_t s_cut_dyn[];  // active set: [E][kCutActive]
  const MultiList& l = a.l;
  const int64_t cnt = (int64_t)l.state[ST_COUNT];
  const int64_t n = cnt < l.cap ? cnt : l.cap;
  if (n <= a.threshold || n <= a.k) return;
  const int tid = threadIdx.x, lane = tid & 31;
  auto load_entry = [&](int64_t i, uint64_t (&e)[E]) {
#pragma unroll
    for (int w = 0; w < W; ++w) e[w] = l.img[w * l.cap + i];
    e[W] = l.rowid[i];
  };
  uint64_t th[E];
#pragma unroll
  for (int w = 0; w < E; ++w) th[w] = 0;
  int64_t k_rem = a.k;
  bool closed = false;
  bool in_smem = false;
  int64_t n_act = n;
  for (int p = 0; p < 8 * E && !closed; ++p) {
    if (tid < 256) s_hist[tid] = 0;
    if (tid == 0) s_nact = 0;
    __syncthreads();
    const int q = p >> 3, sh = 56 - 8 * (p & 7);
    const uint64_t thq = word_at(th, q);
    const bool gather = !in_smem && n_act <= kCutActive;
    const int64_t n_scan = in_smem ? n_act : n;
    for (int64_t i0 = tid - lane; i0 < n_scan; i0 += 1024) {
      const int64_t i = i0 + lane;
      bool m = i < n_scan;
      int d = 0;
      uint64_t e[E];
#pragma unroll
      for (int w = 0; w < E; ++w) e[w] = 0;
      if (m) {
        if (in_smem) {
#pragma unroll
          for (int w = 0; w < E; ++w) e[w] = s_cut_dyn[w * kCutActive + i];
        } else {
          load_entry(i, e);
        }
        const uint64_t eq = word_at(e, q);
        if (!in_smem) {
#pragma unroll
          for (int w = 0; w < E; ++w)
            if (w < q) m &= e[w] == th[w];
          if ((p & 7) != 0) m &= (eq >> (sh + 8)) == (thq >> (sh + 8));
        }
        d = (int)((eq >> sh) & 255);
      }
      const unsigned mm = __ballot_sync(0xffffffffu, m);
      if (!mm) continue;
      if (gather) {
        unsigned int base = 0;
        if (lane == __ffs(mm) - 1) base = atomicAdd(&s_nact, (unsigned)__popc(mm));
        base = __shfl_sync(0xffffffffu, base, __ffs(mm) - 1);
        if (m) {
          const unsigned int qq = base + __popc(mm & ((1u << lane) - 1));
          if (qq < (unsigned)kCutActive) {
#pragma unroll
            for (int w = 0; w < E; ++w) s_cut_dyn[w * kCutActive + qq] = e[w];
          }
        }
      }
      const int d0 = __shfl_sync(0xffffffffu, d, __ffs(mm) - 1);
      const unsigned same = __ballot_sync(0xffffffffu, m && d == d0);
      if (same == mm) { if (lane == __ffs(mm) - 1) atomicAdd(&s_hist[d0], (unsigned)__popc(mm)); }
      else if (m) atomicAdd(&s_hist[d], 1u);
    }
    __syncthreads();
    cut_find_bucket(s_hist, k_rem, s_pick, tid);
    __syncthreads();
    const uint64_t bkt = s_pick[0];
#pragma unroll
    for (int w = 0; w < E; ++w)
      if (w == q) th[w] |= bkt << sh;
    k_rem -= s_pick[1];
    if (gather || in_smem) {
      // keep only the chosen bucket of the shared-memory set (gathered under the OLD prefix)
      const int64_t n_have = n_act;  // <= kCutActive
      in_smem = true;
      if (tid == 0) s_out = 0;
      __syncthreads();
      uint64_t ke[T][E];
      bool kk[T];
#pragma unroll
      for (int t = 0; t < T; ++t) {
        const int64_t i = tid + 1024 * t;
        kk[t] = false;
        if (i < n_have) {
#pragma unroll
          for (int w = 0; w < E; ++w) ke[t][w] = s_cut_dyn[w * kCutActive + i];
          kk[t] = (int)((word_at(ke[t], q) >> sh) & 255) == (int)bkt;
        }
      }
      __syncthreads();
#pragma unroll
      for (int t = 0; t < T; ++t) {
        if (kk[t]) {
          const unsigned int qq = atomicAdd(&s_out, 1u);
#pragma unroll
          for (int w = 0; w < E; ++w) s_cut_dyn[w * kCutActive + qq] = ke[t][w];
        }
      }
      __syncthreads();
    }
    n_act = s_pick[2];
    if ((int64_t)s_pick[2] == k_rem) {  // the whole bucket is in: every entry with this prefix passes
      const uint64_t low = sh ? ((1ULL << sh) - 1) : 0;
#pragma unroll
      for (int w = 0; w < E; ++w) {
        if (w == q) th[w] |= low;
        if (w > q) th[w] = ~0ULL;
      }
      closed = true;
    }
    __syncthreads();
  }
  // compaction of the entries <= threshold into the scratch arrays (at most k of them)
  if (tid == 0) s_out = 0;
  __syncthreads();
  for (int64_t i0 = tid - lane; i0 < n; i0 += 1024) {
    const int64_t i = i0 + lane;
    uint64_t e[E];
    bool keep = false;
    if (i < n) {
      load_entry(i, e);
      keep = img_le(e, th);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (!bal) continue;
    unsigned int base = 0;
    if (lane == __ffs(bal) - 1) base = atomicAdd(&s_out, (unsigned)__popc(bal));
    base = __shfl_sync(0xffffffffu, base, __ffs(bal) - 1);
    if (keep) {
      const unsigned int qq = base + __popc(bal & ((1u << lane) - 1));
      if ((int64_t)qq < a.k) {
#pragma unroll
        for (int w = 0; w < W; ++w) a.alt_img[w * a.k + qq] = e[w];
        a.alt_rowid[qq] = e[W];
        a.alt_bits[qq] = l.bits[i];
      }
    }
  }
  __syncthreads();
  const int64_t kept = (int64_t)s_out < a.k ? (int64_t)s_out : a.k;
  for (int64_t i = tid; i < kept; i += 1024) {
#pragma unroll
    for (int w = 0; w < W; ++w) l.img[w * l.cap + i] = a.alt_img[w * a.k + i];
    l.rowid[i] = a.alt_rowid[i];
    l.bits[i] = a.alt_bits[i];
  }
  if (tid == 0) {
    l.state[ST_COUNT] = (unsigned long long)kept;
#pragma unroll
    for (int w = 0; w < W; ++w) l.state[MST_BOUND + w] = th[w];
  }
}

// n <= 4096 candidates ranked by (image, row id) inside one CTA; out_idx[rank] = entry.
template <int W>
__global__ void __launch_bounds__(1024) small_rank_sort_multi_kernel(const uint64_t* img, int64_t stride, const uint64_t* rowid, int n,
                                                                     uint32_t* out_idx) {
  constexpr int E = W + 1;
  extern __shared__ __align__(16) uint64_t s_ent[];  // [E][n]
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
#pragma unroll
    for (int w = 0; w < W; ++w) s_ent[w * n + i] = img[w * stride + i];
    s_ent[W * n + i] = rowid[i];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    uint64_t e[E];
#pragma unroll
    for (int w = 0; w < E; ++w) e[w] = s_ent[w * n + i];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      bool lt = false;  // entry j < entry i
#pragma unroll
      for (int w = E - 1; w >= 0; --w) {
        const uint64_t x = s_ent[w * n + j];
        lt = x < e[w] || (x == e[w] && lt);
      }
      rank += lt;
    }
    out_idx[rank] = (uint32_t)i;
  }
}

// Result block [first key, row id] from the sorted permutation; a row is NULL when its placement
// bit (the image's top bit) says so.
struct MultiEmitArgs {
  const uint32_t* idx;
  const uint64_t* img0;
  const uint64_t* rowid;
  const uint64_t* bits;
  int64_t n;
  int32_t dtype, nullable, nulls_first;
  void* out_key;
  int64_t* out_row;
  uint8_t* out_valid_bytes;
  unsigned long long* n_null;
};
__global__ void topk_multi_emit_kernel(const __grid_constant__ MultiEmitArgs a) {
  unsigned int nulls = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t j = a.idx[i];
    const bool ok = !a.nullable || (int)(a.img0[j] >> 63) == (a.nulls_first != 0);
    store_narrow_key(a.out_key, i, a.dtype, ok ? a.bits[j] : 0);
    a.out_row[i] = (int64_t)a.rowid[j];
    a.out_valid_bytes[i] = ok ? 1 : 0;
    nulls += !ok;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) nulls += __shfl_xor_sync(0xffffffffu, nulls, o);
  if ((threadIdx.x & 31) == 0 && nulls) atomicAdd(a.n_null, (unsigned long long)nulls);
}

}  // namespace

// ================================================================ operator
class TopkOp : public Op {
 public:
  dbx_topk_params prm;
  int n_cols = 0;
  int key_dtype = 0;
  bool key_nullable = false;
  int cls = 0;
  bool full_sort = false;
  Stager stager;
  RadixSorter sorter;
  // ---- top-k mode
  DevBuf ord, rowid, bits, null_rowid, state, alt_ord, alt_rowid, alt_bits, alt_null;
  DevBuf f_idx0, f_idx1, f_key0, f_key1, f_rowid, f_bits, f_null;  // finish(): sorted candidates
  PinnedBuf host;
  int64_t cap = 0;
  int64_t count_ub = 0, null_ub = 0;   // upper bounds on the list sizes known to the host without a sync
  int64_t rows_seen = 0;
  int64_t rows_at_last_cut = 0;
  int scan_ctas_per_sm = 0;
  DevBuf snap_ord, snap_rowid, snap_bits, snap_null;  // candidate lists as they were before the first optimistic scan of a push
  // ---- full-sort mode
  DevBuf s_ord[2], s_rid[2], s_bits;
  int64_t s_cap = 0;
  // further sort keys (ORDER BY a, b, ...): ordered images and row id | NULL flag per key, in input order
  int n_extra = 0;
  int x_dtype[DBX_MAX_SORT_KEYS - 1] = {}, x_cls[DBX_MAX_SORT_KEYS - 1] = {};
  bool x_nullable[DBX_MAX_SORT_KEYS - 1] = {};
  DevBuf x_ord[DBX_MAX_SORT_KEYS - 1], x_rid[DBX_MAX_SORT_KEYS - 1], x_cnt, w_ord[2], w_rid[2];
  // ---- streaming top-k over several keys: one candidate list of composite images (rowid, bits and
  // alt_rowid, alt_bits as in top-k mode; no NULL list)
  bool multi = false;
  int mw = 0;    // image words
  MultiKeys mk;  // image layout; the columns of the block being pushed
  DevBuf m_img, m_state, alt_img, snap_img;
  int scan_multi_ctas_per_sm = 0;
  std::unique_ptr<OwnedBlock> result;
  bool pulled = false;

  int32_t init(const dbx_topk_params* p, const int32_t* types, int32_t n, int dev) {
    DBX_TRY(base_init(dev));
    prm = *p;
    n_cols = n;
    if (p->key_col < 0 || p->key_col >= n) { err.set("top-k: key column outside the input schema"); return DBX_ERR_INVALID; }
    if (p->limit < 0) { err.set("top-k: negative limit"); return DBX_ERR_INVALID; }
    key_dtype = types[p->key_col] & 0xFF;
    key_nullable = (types[p->key_col] & DBX_NULLABLE) != 0;
    if (dtype_size(key_dtype) == 0) { err.set("top-k: key must be a numeric column"); return DBX_ERR_UNSUPPORTED; }
    cls = key_class(key_dtype);
    full_sort = p->limit == 0 || p->limit > (1 << 22);  // no LIMIT (or one too large for the candidate list): sort everything, then cut
    n_extra = p->n_extra_keys;
    if (n_extra < 0 || n_extra > DBX_MAX_SORT_KEYS - 1) { err.set("sort: at most 4 sort keys"); return DBX_ERR_INVALID; }
    for (int j = 0; j < n_extra; ++j) {
      const int c = p->extra_key_cols[j];
      if (c < 0 || c >= n) { err.set("sort: key column outside the input schema"); return DBX_ERR_INVALID; }
      x_dtype[j] = types[c] & 0xFF;
      x_nullable[j] = (types[c] & DBX_NULLABLE) != 0;
      if (dtype_size(x_dtype[j]) == 0) { err.set("sort: keys must be numeric columns"); return DBX_ERR_UNSUPPORTED; }
      x_cls[j] = key_class(x_dtype[j]);
    }
    // several keys with a LIMIT: streaming top-k over the composite order image
    multi = n_extra > 0 && !full_sort;
    DBX_CUDA_TRY(err, x_cnt.ensure(64));
    DBX_TRY(stager.init(dev, stream, &err));
    DBX_CUDA_TRY(err, host.ensure(256));
    DBX_CUDA_TRY(err, state.ensure(8 * ST_WORDS * 3 + 64));
    if (multi) {
      int dts[DBX_MAX_SORT_KEYS] = {key_dtype};
      bool nul[DBX_MAX_SORT_KEYS] = {key_nullable};
      memset(&mk, 0, sizeof(mk));
      mk.asc[0] = p->asc; mk.nulls_first[0] = p->nulls_first;
      for (int j = 0; j < n_extra; ++j) {
        dts[1 + j] = x_dtype[j]; nul[1 + j] = x_nullable[j];
        mk.asc[1 + j] = p->extra_asc[j]; mk.nulls_first[1 + j] = p->extra_nulls_first[j];
      }
      mw = multi_key_layout(dts, nul, 1 + n_extra, &mk);
      DBX_CUDA_TRY(err, m_state.ensure(8 * (ST_WORDS + kMaxImageWords)));
    }
    if (!full_sort) {
      const int64_t k = p->limit;
      // candidate list: large enough that a whole device-resident column usually fits behind the
      // boundary of its first few million rows; 3 x 8 B per entry ((W + 2) x 8 B for W image words)
      static const int64_t cap_env = getenv("DBX_TOPK_CAP") ? atoll(getenv("DBX_TOPK_CAP")) : 0;
      cap = cap_env > 0 ? cap_env : std::max<int64_t>(1 << 22, 8 * k);
      cap = std::max<int64_t>(cap, 4 * k + 4096);
      if (multi) {
        DBX_CUDA_TRY(err, m_img.ensure(mw * cap * 8));
        DBX_CUDA_TRY(err, rowid.ensure(cap * 8));
        DBX_CUDA_TRY(err, bits.ensure(cap * 8));
        DBX_CUDA_TRY(err, alt_img.ensure(mw * k * 8));
        DBX_CUDA_TRY(err, alt_rowid.ensure(k * 8));
        DBX_CUDA_TRY(err, alt_bits.ensure(k * 8));
        return reset();
      }
      DBX_CUDA_TRY(err, ord.ensure(cap * 8));
      DBX_CUDA_TRY(err, rowid.ensure(cap * 8));
      DBX_CUDA_TRY(err, bits.ensure(cap * 8));
      DBX_CUDA_TRY(err, alt_ord.ensure(k * 8));
      DBX_CUDA_TRY(err, alt_rowid.ensure(k * 8));
      DBX_CUDA_TRY(err, alt_bits.ensure(k * 8));
      if (key_nullable) {
        DBX_CUDA_TRY(err, null_rowid.ensure(cap * 8));
        DBX_CUDA_TRY(err, alt_null.ensure(k * 8));
      }
    }
    return reset();
  }

  int32_t reset() override {
    topk_reset_kernel<<<1, 32, 0, stream>>>((unsigned long long*)state.p);  // count 0, boundary = everything passes
    count_launch();
    DBX_CUDA_TRY(err, cudaMemsetAsync(x_cnt.p, 0, 64, stream));
    if (multi) {  // count 0, boundary all ones: everything passes
      DBX_CUDA_TRY(err, cudaMemsetAsync(m_state.p, 0, 8 * MST_BOUND, stream));
      DBX_CUDA_TRY(err, cudaMemsetAsync((unsigned long long*)m_state.p + MST_BOUND, 0xFF, 8 * mw, stream));
    }
    DBX_CUDA_TRY(err, cudaGetLastError());
    count_ub = null_ub = 0;
    rows_seen = 0;
    rows_at_last_cut = 0;
    result.reset();
    pulled = false;
    return DBX_OK;
  }

  CandList cand_list() const {
    CandList l;
    l.ord = (uint64_t*)ord.p; l.rowid = (uint64_t*)rowid.p; l.bits = (uint64_t*)bits.p;
    l.state = (unsigned long long*)state.p;
    l.cap = cap;
    return l;
  }
  CandList null_list() const {
    CandList l;
    l.ord = nullptr; l.rowid = (uint64_t*)null_rowid.p; l.bits = nullptr;  // rowid == nullptr: key not nullable
    l.state = (unsigned long long*)state.p + ST_WORDS;
    l.cap = cap;
    return l;
  }

  MultiList multi_list() const {
    MultiList l;
    l.img = (uint64_t*)m_img.p; l.rowid = (uint64_t*)rowid.p; l.bits = (uint64_t*)bits.p;
    l.state = (unsigned long long*)m_state.p;
    l.cap = cap;
    return l;
  }
  // calls f(std::integral_constant<int, W>) for this operator's image width
  template <class F>
  int32_t by_words(F&& f) {
    switch (mw) {
      case 1: return f(std::integral_constant<int, 1>());
      case 2: return f(std::integral_constant<int, 2>());
      case 3: return f(std::integral_constant<int, 3>());
      case 4: return f(std::integral_constant<int, 4>());
      case 5: return f(std::integral_constant<int, 5>());
      default: err.set("internal: composite sort image wider than 5 words"); return DBX_ERR_INVALID;
    }
  }
  template <int W>
  int32_t multi_cut_w(int64_t threshold) {
    MultiCutArgs a;
    a.l = multi_list();
    a.alt_img = (uint64_t*)alt_img.p; a.alt_rowid = (uint64_t*)alt_rowid.p; a.alt_bits = (uint64_t*)alt_bits.p;
    a.k = prm.limit; a.threshold = threshold;
    const int smem = kCutActive * (W + 1) * 8;  // 192 KiB at W = 5
    static std::atomic<bool> attr_set[64];
    if (!attr_set[device]) {
      DBX_CUDA_TRY(err, cudaFuncSetAttribute(topk_multi_cut_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      attr_set[device] = true;
    }
    topk_multi_cut_kernel<W><<<1, 1024, smem, stream>>>(a);
    count_launch();
    return DBX_OK;
  }
  template <int W>
  int32_t multi_scan_w(const MultiKeys& k, int64_t m, int64_t row_base, bool fast) {
    if (scan_multi_ctas_per_sm == 0) {
      int a = 0, b2 = 0;
      DBX_CUDA_TRY(err, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, topk_multi_scan_kernel<W, true>, 256, 0));
      DBX_CUDA_TRY(err, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b2, topk_multi_scan_kernel<W, false>, 256, 0));
      scan_multi_ctas_per_sm = std::max(1, std::min(a, b2));
    }
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((m + 2047) / 2048, (int64_t)kNumSMs * scan_multi_ctas_per_sm));
    if (fast) topk_multi_scan_kernel<W, true><<<grid, 256, 0, stream>>>(k, m, row_base, multi_list());
    else topk_multi_scan_kernel<W, false><<<grid, 256, 0, stream>>>(k, m, row_base, multi_list());
    count_launch();
    return DBX_OK;
  }
  int32_t launch_multi_scan(int64_t off, int64_t m, int64_t row_base) {
    MultiKeys k = mk;
    for (int c = 0; c < mk.n_keys; ++c) {
      k.col[c].data = (const char*)mk.col[c].data + off * dtype_size(mk.col[c].dtype);
      if (k.col[c].validity) k.col[c].vbit_off += off;
    }
    const bool fast = !key_nullable && dtype_size(key_dtype) == 8 && !k.col[0].validity && ((reinterpret_cast<uintptr_t>(k.col[0].data) & 31) == 0);
    DBX_TRY(by_words([&](auto w) { return multi_scan_w<decltype(w)::value>(k, m, row_base, fast); }));
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }

  // cut both lists back to k when they hold more than `threshold` entries (device decides)
  int32_t launch_cuts(int64_t threshold, int64_t rows_so_far) {
    if (multi) {
      DBX_TRY(by_words([&](auto w) { return multi_cut_w<decltype(w)::value>(threshold); }));
      DBX_CUDA_TRY(err, cudaGetLastError());
      count_ub = std::min(count_ub, std::max(threshold, prm.limit));
      rows_at_last_cut = rows_so_far;
      return DBX_OK;
    }
    CutArgs a;
    a.l = cand_list();
    a.alt_ord = (uint64_t*)alt_ord.p; a.alt_rowid = (uint64_t*)alt_rowid.p; a.alt_bits = (uint64_t*)alt_bits.p;
    a.k = prm.limit; a.threshold = threshold;
    static std::atomic<bool> attr_set[64];
    if (!attr_set[device]) {
      DBX_CUDA_TRY(err, cudaFuncSetAttribute(topk_cut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kCutActive * 16));
      attr_set[device] = true;
    }
    topk_cut_kernel<<<1, 1024, kCutActive * 16, stream>>>(a);
    count_launch();
    if (key_nullable) {
      CutArgs b;
      b.l = null_list();
      b.alt_ord = nullptr; b.alt_rowid = (uint64_t*)alt_null.p; b.alt_bits = nullptr;
      b.k = prm.limit; b.threshold = threshold;
      topk_cut_kernel<<<1, 1024, kCutActive * 16, stream>>>(b);
      count_launch();
    }
    DBX_CUDA_TRY(err, cudaGetLastError());
    count_ub = std::min(count_ub, std::max(threshold, prm.limit));
    null_ub = std::min(null_ub, std::max(threshold, prm.limit));
    rows_at_last_cut = rows_so_far;
    return DBX_OK;
  }

  int32_t launch_scan(const DevCol& col, int64_t off, int64_t m, int64_t row_base) {
    if (multi) return launch_multi_scan(off, m, row_base);  // mk.col[] holds the pushed block's keys
    DevCol c = col;
    const int esz = dtype_size(key_dtype);
    c.data = (const char*)col.data + off * esz;
    if (c.validity) c.vbit_off += off;
    const bool fast = esz == 8 && !c.validity && ((reinterpret_cast<uintptr_t>(c.data) & 31) == 0);
    if (scan_ctas_per_sm == 0) {
      int a = 0, b2 = 0;
      DBX_CUDA_TRY(err, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, topk_scan_kernel<true>, 256, 0));
      DBX_CUDA_TRY(err, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b2, topk_scan_kernel<false>, 256, 0));
      scan_ctas_per_sm = std::max(1, std::min(a, b2));
    }
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((m + 2047) / 2048, (int64_t)kNumSMs * scan_ctas_per_sm));
    CandList nl = null_list();
    if (!key_nullable) nl.rowid = nullptr;
    if (fast) topk_scan_kernel<true><<<grid, 256, 0, stream>>>(c, m, row_base, cls, prm.asc, cand_list(), nl);
    else topk_scan_kernel<false><<<grid, 256, 0, stream>>>(c, m, row_base, cls, prm.asc, cand_list(), nl);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }

  // rows [off, off + m) in pieces that provably fit the lists; a cut follows every piece
  int32_t scan_guaranteed(const DevCol& col, int64_t off, int64_t m) {
    const int64_t k = prm.limit;
    int64_t done = 0;
    while (done < m) {
      int64_t room = cap - std::max(count_ub, null_ub);
      if (room < cap / 2) { DBX_TRY(launch_cuts(2 * k, rows_seen + off + done)); room = cap - std::max(count_ub, null_ub); }
      const int64_t piece = std::min(m - done, room);
      DBX_TRY(launch_scan(col, off + done, piece, rows_seen + off + done));
      count_ub += piece;
      if (key_nullable && !multi) null_ub += piece;
      done += piece;
    }
    return DBX_OK;
  }

  // One pushed block.  Chunks grow geometrically (x8), each followed by a cut that tightens the
  // device-resident boundary, so a chunk adds about 8k survivors however long the column is.  A
  // chunk that provably fits the candidate list is "guaranteed"; larger ones are launched
  // optimistically (expected survivors << capacity) behind a snapshot of the lists, and the
  // overflow flags are checked ONCE at the end of the push: an overflow restores the snapshot and
  // replays the range in guaranteed pieces.  No host synchronisation otherwise.
  int32_t push_topk(const DevCol& col, int64_t n) {
    const int64_t k = prm.limit;
    int64_t done = 0;
    int64_t chunk = std::max<int64_t>(8 * k, 1 << 14);
    bool snap = false;
    int64_t snap_done = 0, snap_count_ub = 0, snap_null_ub = 0, snap_cut_pos = 0;
    unsigned long long* st = (unsigned long long*)(multi ? m_state.p : state.p);
    const size_t st_bytes = multi ? 8 * (MST_BOUND + mw) : 8 * ST_WORDS * 2;  // <= 72 B
    while (done < n) {
      const int64_t seen = rows_seen + done;
      const int64_t rest = n - done;
      int64_t room = cap - std::max(count_ub, null_ub);
      const int64_t m = std::min(rest, chunk);
      if (room < m && std::max(count_ub, null_ub) > 2 * k) {  // the host's bounds are pessimistic: let the device cut
        DBX_TRY(launch_cuts(2 * k, seen));
        room = cap - std::max(count_ub, null_ub);
      }
      if (m > room && !snap) {  // first optimistic chunk of this push: snapshot the (cut) lists and their state
        DBX_TRY(launch_cuts(k, seen));
        DBX_CUDA_TRY(err, snap_rowid.ensure(k * 8));
        DBX_CUDA_TRY(err, snap_bits.ensure(k * 8));
        if (multi) {
          DBX_CUDA_TRY(err, snap_img.ensure(mw * k * 8));
          DBX_CUDA_TRY(err, cudaMemcpy2DAsync(snap_img.p, k * 8, m_img.p, cap * 8, k * 8, mw, cudaMemcpyDeviceToDevice, stream));
        } else {
          DBX_CUDA_TRY(err, snap_ord.ensure(k * 8));
          DBX_CUDA_TRY(err, cudaMemcpyAsync(snap_ord.p, ord.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        }
        DBX_CUDA_TRY(err, cudaMemcpyAsync(snap_rowid.p, rowid.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        DBX_CUDA_TRY(err, cudaMemcpyAsync(snap_bits.p, bits.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        if (key_nullable && !multi) {
          DBX_CUDA_TRY(err, snap_null.ensure(k * 8));
          DBX_CUDA_TRY(err, cudaMemcpyAsync(snap_null.p, null_rowid.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        }
        DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, st, st_bytes, cudaMemcpyDeviceToHost, stream));
        snap = true;
        snap_done = done; snap_count_ub = count_ub; snap_null_ub = null_ub; snap_cut_pos = rows_at_last_cut;
      }
      DBX_TRY(launch_scan(col, done, m, seen));
      count_ub += m;
      if (key_nullable && !multi) null_ub += m;
      done += m;
      // cut when the rows seen have doubled since the last cut (always inside a multi-chunk push)
      if (rows_seen + done - rows_at_last_cut >= rows_at_last_cut || done < n) DBX_TRY(launch_cuts(2 * k, rows_seen + done));
      chunk *= 8;
    }
    if (snap) {
      DBX_CUDA_TRY(err, cudaMemcpyAsync((char*)host.p + 128, st, st_bytes, cudaMemcpyDeviceToHost, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      const unsigned long long* before = (const unsigned long long*)host.p;
      const unsigned long long* after = (const unsigned long long*)((char*)host.p + 128);
      if (after[ST_OVERFLOW] || (!multi && after[ST_WORDS + ST_OVERFLOW])) {
        // an optimistic chunk did not fit: back to the snapshot, then the same rows in pieces that do
        unsigned long long back[MST_BOUND + kMaxImageWords];
        memcpy(back, before, st_bytes);
        back[ST_OVERFLOW] = 0;
        if (!multi) back[ST_WORDS + ST_OVERFLOW] = 0;
        if (multi) DBX_CUDA_TRY(err, cudaMemcpy2DAsync(m_img.p, cap * 8, snap_img.p, k * 8, k * 8, mw, cudaMemcpyDeviceToDevice, stream));
        else DBX_CUDA_TRY(err, cudaMemcpyAsync(ord.p, snap_ord.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        DBX_CUDA_TRY(err, cudaMemcpyAsync(rowid.p, snap_rowid.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        DBX_CUDA_TRY(err, cudaMemcpyAsync(bits.p, snap_bits.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        if (key_nullable && !multi) DBX_CUDA_TRY(err, cudaMemcpyAsync(null_rowid.p, snap_null.p, k * 8, cudaMemcpyDeviceToDevice, stream));
        DBX_CUDA_TRY(err, cudaMemcpyAsync(st, back, st_bytes, cudaMemcpyHostToDevice, stream));
        DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
        count_ub = std::min<int64_t>(snap_count_ub, (int64_t)before[ST_COUNT]);
        null_ub = multi ? 0 : std::min<int64_t>(snap_null_ub, (int64_t)before[ST_WORDS + ST_COUNT]);
        rows_at_last_cut = snap_cut_pos;
        DBX_TRY(scan_guaranteed(col, snap_done, n - snap_done));
      }
    }
    return DBX_OK;
  }

  // grow the full-sort arrays, keeping their contents
  int32_t sort_reserve(int64_t rows) {
    if (rows <= s_cap) return DBX_OK;
    int64_t ncap = std::max<int64_t>(rows, std::max<int64_t>(s_cap * 2, 1 << 20));
    auto grow = [&](DevBuf& b, size_t elt, bool keep) -> int32_t {
      DevBuf nb;
      DBX_CUDA_TRY(err, nb.ensure((size_t)ncap * elt));
      if (keep && b.p && rows_seen) DBX_CUDA_TRY(err, cudaMemcpyAsync(nb.p, b.p, (size_t)rows_seen * elt, cudaMemcpyDeviceToDevice, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      b = std::move(nb);
      return DBX_OK;
    };
    DBX_TRY(grow(s_ord[0], 8, true));
    DBX_TRY(grow(s_rid[0], 4, true));
    DBX_TRY(grow(s_bits, 8, true));
    for (int j = 0; j < n_extra; ++j) { DBX_TRY(grow(x_ord[j], 8, true)); DBX_TRY(grow(x_rid[j], 4, true)); }
    s_cap = ncap;
    return DBX_OK;
  }

  int32_t push(const dbx_block* b) override {
    if (b->num_cols != n_cols) { err.set("push: block column count differs from the operator's input schema"); return DBX_ERR_INVALID; }
    const dbx_column& kc = b->cols[prm.key_col];
    if (kc.dtype != key_dtype || kc.len != b->num_rows) { err.set("push: key column does not match the input schema"); return DBX_ERR_INVALID; }
    const int64_t n = b->num_rows;
    if (n == 0) return DBX_OK;
    if (kc.is_const) { err.set("top-k over a constant key column is not supported"); return DBX_ERR_UNSUPPORTED; }
    if (kc.validity && !key_nullable) { err.set("push: validity bitmap on a key column declared non-nullable"); return DBX_ERR_INVALID; }
    DevCol col;
    DBX_TRY(stager.begin());
    DBX_TRY(stager.stage(kc, 0, &col));
    DBX_TRY(timing_begin());
    if (full_sort) {
      if (rows_seen + n > rs::kMaxRows) { err.set("sort: more than 2^30 - 1 rows are not supported"); return DBX_ERR_UNSUPPORTED; }
      DBX_TRY(sort_reserve(rows_seen + n));
      sort_ingest_kernel<<<grid_1d(n), 256, 0, stream>>>(col, n, rows_seen, cls, prm.asc, (uint64_t*)s_ord[0].p, (uint32_t*)s_rid[0].p,
                                                         (uint64_t*)s_bits.p, (unsigned long long*)state.p + ST_WORDS + ST_COUNT,
                                                         (unsigned long long*)state.p + ST_WORDS + ST_OVERFLOW);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      for (int j = 0; j < n_extra; ++j) {
        const dbx_column& xc = b->cols[prm.extra_key_cols[j]];
        if (xc.dtype != x_dtype[j] || xc.len != n || xc.is_const) { err.set("push: sort key column does not match the input schema (constant keys unsupported)"); return DBX_ERR_INVALID; }
        if (xc.validity && !x_nullable[j]) { err.set("push: validity bitmap on a key column declared non-nullable"); return DBX_ERR_INVALID; }
        DevCol xcol;
        DBX_TRY(stager.stage(xc, 1 + j, &xcol));
        sort_ingest_kernel<<<grid_1d(n), 256, 0, stream>>>(xcol, n, rows_seen, x_cls[j], prm.extra_asc[j], (uint64_t*)x_ord[j].p, (uint32_t*)x_rid[j].p,
                                                           nullptr, (unsigned long long*)x_cnt.p + j, nullptr);
        count_launch();
        DBX_CUDA_TRY(err, cudaGetLastError());
      }
    } else {
      if (multi) {
        mk.col[0] = col;
        mk.col[0].dtype = key_dtype;
        for (int j = 0; j < n_extra; ++j) {
          const dbx_column& xc = b->cols[prm.extra_key_cols[j]];
          if (xc.dtype != x_dtype[j] || xc.len != n || xc.is_const) { err.set("push: sort key column does not match the input schema (constant keys unsupported)"); return DBX_ERR_INVALID; }
          if (xc.validity && !x_nullable[j]) { err.set("push: validity bitmap on a key column declared non-nullable"); return DBX_ERR_INVALID; }
          DBX_TRY(stager.stage(xc, 1 + j, &mk.col[1 + j]));
          mk.col[1 + j].dtype = x_dtype[j];
        }
      }
      DBX_TRY(push_topk(col, n));
    }
    rows_seen += n;
    DBX_TRY(timing_end());
    DBX_TRY(stager.end());
    return DBX_OK;
  }

  int32_t dev_alloc(OwnedBlock* ob, size_t bytes, void** p) {
    DBX_CUDA_TRY(err, pool_alloc(device, stream, bytes ? bytes : 1, p));
    ob->dev_allocs.push_back(*p);
    return DBX_OK;
  }

  int32_t finish_full_sort() {
    const int64_t n = rows_seen;
    auto ob = std::make_unique<OwnedBlock>();
    ob->stream = stream;  // freed in order behind this operator's enqueued work
    ob->device = device;
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, (unsigned long long*)state.p + ST_WORDS, 8 * ST_WORDS, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const int64_t n_nulls = (int64_t)((unsigned long long*)host.p)[ST_COUNT];
    const bool needs_gather = ((unsigned long long*)host.p)[ST_OVERFLOW] != 0;  // a -0.0 or a NaN with a payload was ingested
    int buf = 0;
    const uint64_t* sorted_ord = nullptr;
    const uint32_t* sorted_rid = nullptr;
    if (n_extra > 0 && n > 1) {
      unsigned long long xn[DBX_MAX_SORT_KEYS] = {};
      DBX_CUDA_TRY(err, cudaMemcpyAsync(xn, x_cnt.p, 8 * (DBX_MAX_SORT_KEYS - 1), cudaMemcpyDeviceToHost, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      const uint64_t* k_ord[DBX_MAX_SORT_KEYS] = {(const uint64_t*)s_ord[0].p};
      const uint32_t* k_rid[DBX_MAX_SORT_KEYS] = {(const uint32_t*)s_rid[0].p};
      int64_t k_nulls[DBX_MAX_SORT_KEYS] = {n_nulls};
      int32_t k_nulls_first[DBX_MAX_SORT_KEYS] = {prm.nulls_first};
      for (int j = 0; j < n_extra; ++j) {
        k_ord[1 + j] = (const uint64_t*)x_ord[j].p; k_rid[1 + j] = (const uint32_t*)x_rid[j].p;
        k_nulls[1 + j] = (int64_t)xn[j]; k_nulls_first[1 + j] = prm.extra_nulls_first[j];
      }
      DBX_TRY(sort_rows_by_keys(err, stream, sorter, 1 + n_extra, k_ord, k_rid, k_nulls, k_nulls_first, n, w_ord, w_rid, &sorted_ord, &sorted_rid));
    } else if (n > 1) {
      DBX_CUDA_TRY(err, s_ord[1].ensure((size_t)s_cap * 8));
      DBX_CUDA_TRY(err, s_rid[1].ensure((size_t)s_cap * 4));
      DBX_TRY(sorter.sort(err, stream, (uint64_t*)s_ord[0].p, (uint64_t*)s_ord[1].p, (uint32_t*)s_rid[0].p, (uint32_t*)s_rid[1].p, n, 0,
                          64, n_nulls > 0, prm.nulls_first, n_nulls, &buf));
    }
    if (!sorted_ord) { sorted_ord = (const uint64_t*)s_ord[buf].p; sorted_rid = (const uint32_t*)s_rid[buf].p; }
    const int64_t n_in = n;
    const int64_t n_out = prm.limit > 0 ? std::min<int64_t>(n_in, prm.limit) : n_in;  // LIMIT > 4 Mi: cut the sorted rows
    // the first key's NULL rows are one run at the start (NULLS FIRST) or the end of the sorted rows
    const int64_t out_nulls = prm.nulls_first ? std::min(n_nulls, n_out) : std::max<int64_t>(0, n_out - (n_in - n_nulls));
    void *okey = nullptr, *orow = nullptr, *ovb = nullptr, *obits = nullptr;
    const int esz = dtype_size(key_dtype);
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out * esz, &okey));
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out * 8, &orow));
    if (key_nullable) {
      DBX_TRY(dev_alloc(ob.get(), (size_t)n_out, &ovb));
      DBX_TRY(dev_alloc(ob.get(), (size_t)(n_out + 7) / 8 + 8, &obits));
    }
    if (n_out) {
      SortEmitArgs ea;
      ea.rid = sorted_rid; ea.bits = needs_gather ? (const uint64_t*)s_bits.p : nullptr; ea.n = n_out; ea.dtype = key_dtype;
      ea.ord = sorted_ord; ea.cls = cls; ea.asc = prm.asc;
      ea.out_key = okey; ea.out_row = (int64_t*)orow; ea.out_valid_bytes = (uint8_t*)ovb;
      sort_emit_kernel<<<grid_1d(n_out), 256, 0, stream>>>(ea);
      count_launch();
      if (key_nullable) { pack_bits_kernel<<<grid_1d((n_out + 7) / 8), 256, 0, stream>>>((const uint8_t*)ovb, n_out, (uint8_t*)obits); count_launch(); }
      DBX_CUDA_TRY(err, cudaGetLastError());
    }
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, sorter.meta.p ? (void*)sorter.fail() : state.p, 4, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    if (sorter.meta.p && n > 1 && *(unsigned int*)host.p) { err.set("internal: radix sort look-back timed out"); return DBX_ERR_CUDA; }
    dbx_column kcol;
    memset(&kcol, 0, sizeof(kcol));
    kcol.dtype = key_dtype; kcol.mem = DBX_MEM_DEVICE; kcol.len = n_out; kcol.data = okey;
    if (key_nullable) { kcol.validity = (const uint8_t*)obits; kcol.null_count = out_nulls; }
    dbx_column rcol;
    memset(&rcol, 0, sizeof(rcol));
    rcol.dtype = DBX_I64; rcol.mem = DBX_MEM_DEVICE; rcol.len = n_out; rcol.data = orow;
    ob->cols.push_back(kcol);
    ob->cols.push_back(rcol);
    result = std::move(ob);
    return DBX_OK;
  }

  // sort `n` (ord?, rowid, bits?) entries by (ord, rowid) into out_rowid / out_bits
  int32_t sort_candidates(const uint64_t* c_ord, const uint64_t* c_rowid, const uint64_t* c_bits, int64_t n, uint64_t* out_rowid,
                          uint64_t* out_bits) {
    if (n == 0) return DBX_OK;
    if (n <= 4096) {
      static std::atomic<bool> attr_set[64];
      if (!attr_set[device]) {
        DBX_CUDA_TRY(err, cudaFuncSetAttribute(small_rank_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 16));
        attr_set[device] = true;
      }
      small_rank_sort_kernel<<<1, 1024, (size_t)n * 16, stream>>>(c_ord, c_rowid, c_bits, (int)n, out_rowid, out_bits);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      return DBX_OK;
    }
    // two stable radix sorts of a permutation: by row id, then by the ordered key
    DBX_CUDA_TRY(err, f_idx0.ensure(n * 4));
    DBX_CUDA_TRY(err, f_idx1.ensure(n * 4));
    DBX_CUDA_TRY(err, f_key0.ensure(n * 8));
    DBX_CUDA_TRY(err, f_key1.ensure(n * 8));
    iota_u32_kernel<<<grid_1d(n), 256, 0, stream>>>((uint32_t*)f_idx0.p, n);
    count_launch();
    DBX_CUDA_TRY(err, cudaMemcpyAsync(f_key0.p, c_rowid, n * 8, cudaMemcpyDeviceToDevice, stream));
    int buf = 0;
    DBX_TRY(sorter.sort(err, stream, (uint64_t*)f_key0.p, (uint64_t*)f_key1.p, (uint32_t*)f_idx0.p, (uint32_t*)f_idx1.p, n, 0, 48, false, 0, 0, &buf));
    uint32_t* idx = (uint32_t*)(buf ? f_idx1.p : f_idx0.p);
    uint32_t* idx_other = (uint32_t*)(buf ? f_idx0.p : f_idx1.p);
    if (c_ord) {
      uint64_t* kb = (uint64_t*)(buf ? f_key0.p : f_key1.p);  // the buffer the first sort left free
      uint64_t* kb_other = (uint64_t*)(buf ? f_key1.p : f_key0.p);
      gather_u64_kernel<<<grid_1d(n), 256, 0, stream>>>(c_ord, idx, kb, n);
      count_launch();
      int buf2 = 0;
      DBX_TRY(sorter.sort(err, stream, kb, kb_other, idx, idx_other, n, 0, 64, false, 0, 0, &buf2));
      if (buf2) idx = idx_other;
    }
    gather_u64_kernel<<<grid_1d(n), 256, 0, stream>>>(c_rowid, idx, out_rowid, n);
    if (c_bits) gather_u64_kernel<<<grid_1d(n), 256, 0, stream>>>(c_bits, idx, out_bits, n);
    count_launch(2);
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }

  // the sorted order of n <= k multi-key candidates as a permutation of the list (`*idx`)
  template <int W>
  int32_t multi_order_w(int64_t n, uint32_t** idx) {
    DBX_CUDA_TRY(err, f_idx0.ensure(std::max<int64_t>(n, 1) * 4));
    *idx = (uint32_t*)f_idx0.p;
    if (n == 0) return DBX_OK;
    const uint64_t* img = (const uint64_t*)m_img.p;
    if (n <= 4096) {
      static std::atomic<bool> attr_set[64];
      if (!attr_set[device]) {
        DBX_CUDA_TRY(err, cudaFuncSetAttribute(small_rank_sort_multi_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * (W + 1) * 8));
        attr_set[device] = true;
      }
      small_rank_sort_multi_kernel<W><<<1, 1024, (size_t)n * (W + 1) * 8, stream>>>(img, cap, (const uint64_t*)rowid.p, (int)n, *idx);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      return DBX_OK;
    }
    // W + 1 stable radix sorts of a permutation: by row id, then by the image words from the least
    // significant to the most significant
    DBX_CUDA_TRY(err, f_idx1.ensure(n * 4));
    DBX_CUDA_TRY(err, f_key0.ensure(n * 8));
    DBX_CUDA_TRY(err, f_key1.ensure(n * 8));
    uint32_t* cur = (uint32_t*)f_idx0.p;
    uint32_t* other = (uint32_t*)f_idx1.p;
    iota_u32_kernel<<<grid_1d(n), 256, 0, stream>>>(cur, n);
    count_launch();
    DBX_CUDA_TRY(err, cudaMemcpyAsync(f_key0.p, rowid.p, n * 8, cudaMemcpyDeviceToDevice, stream));
    int rid_bits = 8;
    while (rid_bits < 64 && ((uint64_t)std::max<int64_t>(rows_seen - 1, 0) >> rid_bits)) rid_bits += 8;
    for (int w = W; w >= 0; --w) {
      if (w < W) {
        gather_u64_kernel<<<grid_1d(n), 256, 0, stream>>>(img + (size_t)w * cap, cur, (uint64_t*)f_key0.p, n);
        count_launch();
      }
      int buf = 0;
      DBX_TRY(sorter.sort(err, stream, (uint64_t*)f_key0.p, (uint64_t*)f_key1.p, cur, other, n, 0, w == W ? rid_bits : 64, false, 0, 0, &buf));
      if (buf) std::swap(cur, other);
    }
    *idx = cur;
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }

  int32_t finish_multi() {
    const int64_t k = prm.limit;
    DBX_TRY(launch_cuts(k, rows_seen));  // the list down to <= k entries
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, m_state.p, 8 * ST_WORDS, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const unsigned long long* h = (const unsigned long long*)host.p;
    if (h[ST_OVERFLOW]) { err.set("internal: top-k candidate list overflow"); return DBX_ERR_CUDA; }
    const int64_t n_out = std::min<int64_t>((int64_t)h[ST_COUNT], k);
    uint32_t* idx = nullptr;
    DBX_TRY(by_words([&](auto w) { return multi_order_w<decltype(w)::value>(n_out, &idx); }));
    auto ob = std::make_unique<OwnedBlock>();
    ob->stream = stream;  // freed in order behind this operator's enqueued work
    ob->device = device;
    const int esz = dtype_size(key_dtype);
    void *okey = nullptr, *orow = nullptr, *ovb = nullptr, *obits = nullptr;
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out * esz, &okey));
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out * 8, &orow));
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out + 1, &ovb));
    DBX_TRY(dev_alloc(ob.get(), (size_t)(n_out + 7) / 8 + 8, &obits));
    if (n_out) {
      MultiEmitArgs ea;
      ea.idx = idx; ea.img0 = (const uint64_t*)m_img.p; ea.rowid = (const uint64_t*)rowid.p; ea.bits = (const uint64_t*)bits.p;
      ea.n = n_out; ea.dtype = key_dtype; ea.nullable = key_nullable; ea.nulls_first = prm.nulls_first;
      ea.out_key = okey; ea.out_row = (int64_t*)orow; ea.out_valid_bytes = (uint8_t*)ovb;
      ea.n_null = (unsigned long long*)m_state.p + MST_NULLS;
      topk_multi_emit_kernel<<<grid_1d(n_out), 256, 0, stream>>>(ea);
      pack_bits_kernel<<<grid_1d((n_out + 7) / 8), 256, 0, stream>>>((const uint8_t*)ovb, n_out, (uint8_t*)obits);
      count_launch(2);
      DBX_CUDA_TRY(err, cudaGetLastError());
    }
    const bool radix = n_out > 4096 && sorter.meta.p;
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, (unsigned long long*)m_state.p + MST_NULLS, 8, cudaMemcpyDeviceToHost, stream));
    if (radix) DBX_CUDA_TRY(err, cudaMemcpyAsync((char*)host.p + 8, (void*)sorter.fail(), 4, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const int64_t n_nulls = (int64_t)*(const unsigned long long*)host.p;
    if (radix && *(const unsigned int*)((char*)host.p + 8)) { err.set("internal: radix sort look-back timed out"); return DBX_ERR_CUDA; }
    dbx_column kcol;
    memset(&kcol, 0, sizeof(kcol));
    kcol.dtype = key_dtype; kcol.mem = DBX_MEM_DEVICE; kcol.len = n_out; kcol.data = okey;
    if (key_nullable) { kcol.validity = (const uint8_t*)obits; kcol.null_count = n_nulls; }
    dbx_column rcol;
    memset(&rcol, 0, sizeof(rcol));
    rcol.dtype = DBX_I64; rcol.mem = DBX_MEM_DEVICE; rcol.len = n_out; rcol.data = orow;
    ob->cols.push_back(kcol);
    ob->cols.push_back(rcol);
    result = std::move(ob);
    return DBX_OK;
  }

  int32_t finish() override {
    if (full_sort) return finish_full_sort();
    if (multi) return finish_multi();
    const int64_t k = prm.limit;
    DBX_TRY(launch_cuts(k, rows_seen));  // both lists down to <= k entries
    unsigned long long* st = (unsigned long long*)state.p;
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, st, 8 * ST_WORDS * 2, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const unsigned long long* h = (const unsigned long long*)host.p;
    if (h[ST_OVERFLOW] || h[ST_WORDS + ST_OVERFLOW]) { err.set("internal: top-k candidate list overflow"); return DBX_ERR_CUDA; }
    const int64_t n_valid = std::min<int64_t>((int64_t)h[ST_COUNT], k);
    const int64_t n_nulls = key_nullable ? std::min<int64_t>((int64_t)h[ST_WORDS + ST_COUNT], k) : 0;
    int64_t take_null, take_valid;
    if (prm.nulls_first) { take_null = n_nulls; take_valid = std::min<int64_t>(k - take_null, n_valid); }
    else { take_valid = n_valid; take_null = std::min<int64_t>(k - take_valid, n_nulls); }
    const int64_t n_out = take_null + take_valid;
    DBX_CUDA_TRY(err, f_rowid.ensure(std::max<int64_t>(n_valid, 1) * 8));
    DBX_CUDA_TRY(err, f_bits.ensure(std::max<int64_t>(n_valid, 1) * 8));
    DBX_TRY(sort_candidates((const uint64_t*)ord.p, (const uint64_t*)rowid.p, (const uint64_t*)bits.p, n_valid, (uint64_t*)f_rowid.p, (uint64_t*)f_bits.p));
    if (n_nulls) {
      DBX_CUDA_TRY(err, f_null.ensure(n_nulls * 8));
      DBX_TRY(sort_candidates(nullptr, (const uint64_t*)null_rowid.p, nullptr, n_nulls, (uint64_t*)f_null.p, nullptr));
    }
    // output block: [key (original dtype, nullable), row_id Int64], assembled on the device
    auto ob = std::make_unique<OwnedBlock>();
    ob->stream = stream;  // freed in order behind this operator's enqueued work
    ob->device = device;
    const int esz = dtype_size(key_dtype);
    void *okey = nullptr, *orow = nullptr, *ovb = nullptr, *obits = nullptr;
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out * esz, &okey));
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out * 8, &orow));
    DBX_TRY(dev_alloc(ob.get(), (size_t)n_out + 1, &ovb));
    DBX_TRY(dev_alloc(ob.get(), (size_t)(n_out + 7) / 8 + 8, &obits));
    if (n_out) {
      EmitArgs ea;
      ea.bits = (const uint64_t*)f_bits.p; ea.rowid = (const uint64_t*)f_rowid.p; ea.null_rowid = (const uint64_t*)f_null.p;
      ea.take_valid = take_valid; ea.take_null = take_null; ea.nulls_first = prm.nulls_first; ea.dtype = key_dtype;
      ea.out_key = okey; ea.out_row = (int64_t*)orow; ea.out_valid_bytes = (uint8_t*)ovb;
      topk_emit_kernel<<<grid_1d(n_out), 256, 0, stream>>>(ea);
      pack_bits_kernel<<<grid_1d((n_out + 7) / 8), 256, 0, stream>>>((const uint8_t*)ovb, n_out, (uint8_t*)obits);
      count_launch(2);
      DBX_CUDA_TRY(err, cudaGetLastError());
    }
    dbx_column kcol;
    memset(&kcol, 0, sizeof(kcol));
    kcol.dtype = key_dtype; kcol.mem = DBX_MEM_DEVICE; kcol.len = n_out; kcol.data = okey;
    if (key_nullable) { kcol.validity = (const uint8_t*)obits; kcol.null_count = take_null; }
    dbx_column rcol;
    memset(&rcol, 0, sizeof(rcol));
    rcol.dtype = DBX_I64; rcol.mem = DBX_MEM_DEVICE; rcol.len = n_out; rcol.data = orow;
    ob->cols.push_back(kcol);
    ob->cols.push_back(rcol);
    result = std::move(ob);
    return DBX_OK;
  }

  int32_t pull(int32_t out_mem, dbx_block* out, int32_t* has_block) override;
};

}  // namespace dbx

namespace dbx {

int32_t TopkOp::pull(int32_t out_mem, dbx_block* out, int32_t* has_block) {
  if (!finished) { err.set("pull before finish"); return DBX_ERR_STATE; }
  if (pulled || !result) { *has_block = 0; return DBX_OK; }
  pulled = true;
  *has_block = 1;
  return pull_owned_block(result, device, stream, err, out_mem, out);
}

Op* make_topk_op(const dbx_topk_params* p, const int32_t* types, int32_t n, int device, int32_t* st) {
  auto* op = new TopkOp();
  *st = op->init(p, types, n, device);
  if (*st != DBX_OK) { g_create_error.set(op->err.msg); delete op; return nullptr; }
  return op;
}

}  // namespace dbx
