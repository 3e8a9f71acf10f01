// join.cu — DBX_OP_JOIN: hash join on one integer key column (INNER, LEFT, LEFT SEMI / ANTI, RIGHT,
// RIGHT SEMI / ANTI, FULL).
//
// Reference replaced (paths relative to the databend source tree, src/query/service/src/pipelines/processors/transforms):
//   Join trait (add_block / final_build / probe_block -> JoinStream / final_probe)   new_hash_join/join.rs:26-53
//   TransformHashJoin stage machine Build -> BuildFinal -> Probe                    new_hash_join/transform_hash_join.rs:39-230
//   BasicHashJoin::{add_block, final_build}                                         new_hash_join/memory/basic.rs:77-160
//   HashJoinHashTable::{with_build_row_num, insert, probe}                          hash_join_table/hashjoin_hashtable.rs:95-190
//   InnerHashJoin::probe_block / InnerHashJoinStream::next                          new_hash_join/memory/inner_join.rs:122-262
//
// Design.  Build rows stay in HBM as columns.  The table is an open-addressed multimap of
// 32-byte entries {key, build_row + 1 | validity flags, payload0, payload1} = one sector = two
// 128-bit loads: the probe of a row with up to two 8-byte build columns next to the key touches
// ONE random sector (the reference reads an 8-byte header, then chases the entry chain, then
// gathers the build row).  A 1e9-row probe into a 1e7-row build side is bound by HBM's
// random-sector rate, not by bytes: every avoided gather is worth as much as the probe itself.
// Build columns that do not fit the entry are gathered by build row as before.  The probe kernel streams the probe key column once, walks
// buckets until it sees an empty entry, and writes each joined row directly into the output
// columns at a position claimed with a warp-aggregated atomic: no (probe,build) index pairs are
// materialised and no second gather pass runs (the reference does DataBlock::take +
// take_column_vec).  Output row order is therefore unspecified — like the reference's when
// several threads build the chains — and results are compared as multisets.
// NULL keys never match (fixed_keys.rs: rows with a NULL key are skipped on both sides).
//
// Composite keys (up to four key pairs, HashMethodFixedKeys in new_hash_join/hashtable/fixed_keys.rs)
// are packed into one or two 64-bit words, one bit field per pair (KeyPartDev, as the aggregate's
// multi-column GROUP BY).  Up to 64 bits the entry is the same as for one key; up to 128 bits it is
// {k0, k1, row1, p0}: still one sector, with one inlined build column instead of two.  The kernels
// are templated on the key width KW (words) and on PACKED (key loaded from several columns); the
// single-key instantiations <1, false> read the one key column directly.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "plan.h"
#include "runtime.h"
#include "runtime_filter.cuh"

namespace dbx {

namespace {

constexpr int kJoinBlock = 256;
constexpr int kMaxJoinCols = 16;

template <int KW> struct JEntry;
template <> struct JEntry<1> {
  uint64_t key;
  uint64_t row1;  // (build row + 1) | validity of p0 << 62 | validity of p1 << 63; 0 = empty
  uint64_t p0, p1;  // raw bytes of up to two build columns (zero-extended to 8 bytes)
};
template <> struct JEntry<2> {  // 128-bit key
  uint64_t key, key1;
  uint64_t row1;  // (build row + 1) | validity of p0 << 62; 0 = empty
  uint64_t p0;
};
using JoinEntry = JEntry<1>;
static_assert(sizeof(JEntry<1>) == 32 && sizeof(JEntry<2>) == 32, "one entry = one 32-byte sector");
constexpr uint64_t kRowMask = (1ULL << 62) - 1;

__device__ __forceinline__ void clear_entry(JEntry<1>& e) { e.key = e.row1 = e.p0 = e.p1 = 0; }
__device__ __forceinline__ void clear_entry(JEntry<2>& e) { e.key = e.key1 = e.row1 = e.p0 = 0; }
__device__ __forceinline__ bool key_eq(const JEntry<1>& e, uint64_t k, uint64_t) { return e.key == k; }
__device__ __forceinline__ bool key_eq(const JEntry<2>& e, uint64_t k, uint64_t kh) { return e.key == k && e.key1 == kh; }
__device__ __forceinline__ uint64_t key_hi(const JEntry<1>&) { return 0; }
__device__ __forceinline__ uint64_t key_hi(const JEntry<2>& e) { return e.key1; }
__device__ __forceinline__ uint64_t entry_p1(const JEntry<1>& e) { return e.p1; }
__device__ __forceinline__ uint64_t entry_p1(const JEntry<2>&) { return 0; }
__device__ __forceinline__ void fill_entry(JEntry<1>* e, uint64_t k, uint64_t, uint64_t p0, uint64_t p1) { e->key = k; e->p0 = p0; e->p1 = p1; }
__device__ __forceinline__ void fill_entry(JEntry<2>* e, uint64_t k, uint64_t kh, uint64_t p0, uint64_t) { e->key = k; e->key1 = kh; e->p0 = p0; }

// Composite key of one side: its key columns and the bit field of each (KeyPartDev: shift, mask,
// dtype; slot = column index).  Both sides share shifts and masks and differ in dtypes.
struct JoinKeyPack {
  DevCol cols[DBX_MAX_JOIN_KEYS];
  KeyPartDev parts[DBX_MAX_JOIN_KEYS];
  int32_t n;
  int32_t pad;
};

struct JoinTableDev {
  JoinEntry* entries;  // cap entries (power of two), one per 32-byte sector
  int64_t cap;
};
template <int KW = 1>
__device__ __forceinline__ int64_t join_home(const JoinTableDev& t, uint64_t k, uint64_t kh = 0) {
  const uint64_t h = KW == 1 ? agg_hash_u64(k) : agg_hash_wide(k, kh);
  return (int64_t)(h & (uint64_t)(t.cap - 1));
}

// build column carried inside the table entry
struct InlineColDev {
  const void* src;
  const uint8_t* valid_bytes;  // one byte per build row, or null
  int32_t size;
  int32_t on;
};

// One column copied into the output for every match.
struct JoinColDev {
  const void* src;
  void* dst;
  const uint8_t* src_validity;  // may be null
  int64_t src_vbit_off;
  uint8_t* dst_valid;           // one byte per output row, or null
  int32_t size;                 // bytes per value
  int32_t from;                 // build side: 0 gather by build row, 1 the entry's key, 2 entry.p0, 3 entry.p1,
                                // 4 + s: the packed key's bit field at shift s (composite keys)
};

// One value slot of the residual predicate (RESID kernels): a probe column, read once per probe row,
// or a build column, read per candidate pair from the source JoinColDev::from names for it.
constexpr int kResidSlots = 8;  // comp_row_cond's value slots
struct ResidSlotDev {
  DevCol probe;                // side 0: the probe block's column
  const void* src;             // side 1, from = 0: the build column, gathered by build row
  const uint8_t* valid_bytes;  // side 1, from = 0: one byte per build row, or null (all valid)
  int32_t side;                // 0 probe, 1 build
  int32_t from;                // build side: as JoinColDev::from
  int32_t dtype;
  int32_t size;
};

struct JoinProbeParams {
  DevCol key;
  JoinTableDev table;
  JoinColDev probe_cols[kMaxJoinCols];
  JoinColDev build_cols[kMaxJoinCols];
  int32_t n_probe_cols, n_build_cols;
  int32_t kind, pad;  // dbx_join_kind
  int64_t n_rows;
  int64_t out_cap;
  unsigned long long* cursor;  // number of matches (may exceed out_cap: then the host retries)
  uint8_t* matched;            // build-side kinds: one byte per build row, set when a probe row matches it
  JoinKeyPack pack;            // composite keys (PACKED kernels): the probe key columns
  RfPartDev rf;                // RF kernels: the runtime filter's min-max and bloom (runtime_filter.cuh)
  unsigned long long* rf_rejected;  // RF kernels: rows the filter turned away
  // RESID kernels (kept behind every field above, so the other kernels see the same layout): the
  // residual predicate's program, its COLUMN nodes naming slots of resid_slots
  int32_t resid_n_nodes, resid_n_slots;
  ResidSlotDev resid_slots[kResidSlots];
  NodeDev resid_nodes[kMaxExprNodes];
};

__device__ __forceinline__ uint64_t load_key(const DevCol& c, int64_t row) {
  const char* base = (const char*)c.data;
  switch (c.dtype) {
    case DBX_I64: case DBX_U64: return ((const uint64_t*)base)[row];
    case DBX_I32: return (uint64_t)(int64_t)((const int32_t*)base)[row];
    case DBX_U32: return ((const uint32_t*)base)[row];
    case DBX_I16: return (uint64_t)(int64_t)((const int16_t*)base)[row];
    case DBX_U16: return ((const uint16_t*)base)[row];
    case DBX_I8: return (uint64_t)(int64_t)((const int8_t*)base)[row];
    default: return ((const uint8_t*)base)[row];
  }
}

// HashJoinHashTable::insert (hashjoin_hashtable.rs:110-141): every build row with a valid key
// claims the first free entry along its probe sequence (CAS on the row field; the key is written
// afterwards — build and probe are separated by a kernel boundary).
__device__ __forceinline__ uint64_t load_raw(const void* base, int size, int64_t row) {
  switch (size) {
    case 8: return ((const uint64_t*)base)[row];
    case 4: return ((const uint32_t*)base)[row];
    case 2: return ((const uint16_t*)base)[row];
    default: return ((const uint8_t*)base)[row];
  }
}
// Composite key of row r: false if any key column is NULL there (the row never matches).  Each
// value is widened to 64 bits (load_key), masked to its field and shifted into word shift / 64.
template <int KW>
__device__ __forceinline__ bool load_packed_key(const JoinKeyPack& pk, int64_t r, uint64_t& k, uint64_t& kh) {
  k = kh = 0;
#pragma unroll
  for (int i = 0; i < DBX_MAX_JOIN_KEYS; ++i) {
    if (i >= pk.n) break;
    const DevCol& c = pk.cols[i];
    if (c.validity && !bit_test(c.validity, c.vbit_off + r)) return false;
    const KeyPartDev& f = pk.parts[i];
    const uint64_t v = (load_key(c, r) & f.mask) << (f.shift & 63);
    if (KW == 1 || f.shift < 64) k |= v;
    else kh |= v;
  }
  return true;
}

template <int KW, bool PACKED>
__global__ void join_build_kernel(const __grid_constant__ DevCol key, int64_t n_rows,
                                  const __grid_constant__ JoinTableDev t, const __grid_constant__ InlineColDev i0,
                                  const __grid_constant__ InlineColDev i1, const __grid_constant__ JoinKeyPack pk) {
  const int64_t mask = t.cap - 1;
  JEntry<KW>* const entries = (JEntry<KW>*)t.entries;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t k, kh = 0;
    if (PACKED) {
      if (!load_packed_key<KW>(pk, r, k, kh)) continue;
    } else {
      if (key.validity && !bit_test(key.validity, key.vbit_off + r)) continue;
      k = load_key(key, r);
    }
    uint64_t tag = (uint64_t)(r + 1);
    uint64_t p0 = 0, p1 = 0;
    if (i0.on) { p0 = load_raw(i0.src, i0.size, r); if (!i0.valid_bytes || i0.valid_bytes[r]) tag |= 1ULL << 62; }
    if (KW == 1 && i1.on) { p1 = load_raw(i1.src, i1.size, r); if (!i1.valid_bytes || i1.valid_bytes[r]) tag |= 1ULL << 63; }
    int64_t s = join_home<KW>(t, k, kh);
    for (;;) {
      JEntry<KW>* e = entries + s;
      unsigned long long old = atomicCAS((unsigned long long*)&e->row1, 0ULL, (unsigned long long)tag);
      if (old == 0ULL) { fill_entry(e, k, kh, p0, p1); break; }
      s = (s + 1) & mask;
    }
  }
}

__device__ __forceinline__ void store_value(const JoinColDev& c, uint64_t bits, bool valid, int64_t dst_row) {
  switch (c.size) {
    case 8: ((uint64_t*)c.dst)[dst_row] = bits; break;
    case 4: ((uint32_t*)c.dst)[dst_row] = (uint32_t)bits; break;
    case 2: ((uint16_t*)c.dst)[dst_row] = (uint16_t)bits; break;
    default: ((uint8_t*)c.dst)[dst_row] = (uint8_t)bits; break;
  }
  if (c.dst_valid) c.dst_valid[dst_row] = valid ? 1 : 0;
}

__device__ __forceinline__ void copy_value(const JoinColDev& c, int64_t src_row, int64_t dst_row) {
  switch (c.size) {
    case 8: ((uint64_t*)c.dst)[dst_row] = ((const uint64_t*)c.src)[src_row]; break;
    case 4: ((uint32_t*)c.dst)[dst_row] = ((const uint32_t*)c.src)[src_row]; break;
    case 2: ((uint16_t*)c.dst)[dst_row] = ((const uint16_t*)c.src)[src_row]; break;
    default: ((uint8_t*)c.dst)[dst_row] = ((const uint8_t*)c.src)[src_row]; break;
  }
  if (c.dst_valid) c.dst_valid[dst_row] = c.src_validity ? (uint8_t)bit_test(c.src_validity, c.src_vbit_off + src_row) : 1;
}

__device__ __forceinline__ JoinEntry load_entry(const JoinEntry* e) {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  JoinEntry r;  // 32 bytes as two 128-bit loads (sm_90a has no 256-bit load)
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(r.key), "=l"(r.row1) : "l"(e), "l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(r.p0), "=l"(r.p1) : "l"((const char*)e + 16), "l"(pol));
  return r;
}
__device__ __forceinline__ JEntry<2> load_entry(const JEntry<2>* e) {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  JEntry<2> r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(r.key), "=l"(r.key1) : "l"(e), "l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(r.row1), "=l"(r.p0) : "l"((const char*)e + 16), "l"(pol));
  return r;
}
// PACKED: the build key columns are decoded from the entry's packed key (from = 4 + field shift),
// which saves the random gather by build row that a key column would otherwise cost.
template <bool PACKED = false, int KW>
__device__ __forceinline__ void emit_match(const JoinProbeParams& p, int64_t r, const JEntry<KW>& e, int64_t pos) {
  if (pos >= p.out_cap) return;
  for (int c = 0; c < p.n_probe_cols; ++c) copy_value(p.probe_cols[c], r, pos);
  for (int c = 0; c < p.n_build_cols; ++c) {
    const JoinColDev& jc = p.build_cols[c];
    if (jc.from == 0) copy_value(jc, (int64_t)(e.row1 & kRowMask) - 1, pos);
    else if (jc.from == 1) store_value(jc, e.key, true, pos);
    else if (jc.from == 2) store_value(jc, e.p0, (e.row1 >> 62) & 1, pos);
    else if (!PACKED || jc.from == 3) store_value(jc, entry_p1(e), (e.row1 >> 63) & 1, pos);
    else {
      const int s = jc.from - 4;
      store_value(jc, (s < 64 ? e.key : key_hi(e)) >> (s & 63), true, pos);
    }
  }
}

// ---- residual predicate (HashJoinDesc::other_predicate, hash_join/desc.rs:156-190): the ON clause's
// non-equi conditions, evaluated on every candidate pair (equal keys) inside the probe.  A pair whose
// predicate is NULL or false is no match, for every kind.  The values of one pair sit in up to eight
// slots: the probe row's are loaded once before its walk, the build row's per candidate from the entry
// (key, p0, p1, packed key field) or by a gather by build row.
struct ResidRow { uint64_t v[kResidSlots]; };

// value image (load_image's) of a build value held as its raw bytes, zero-extended: integers sign- or
// zero-extended to 64 bits, F32 as the f64 bits of its value
__device__ __forceinline__ uint64_t raw_image(uint64_t raw, int dtype) {
  if (dtype == DBX_F32) return (uint64_t)__double_as_longlong((double)__uint_as_float((uint32_t)raw));
  return wrap_int(raw, dtype);
}

__device__ __forceinline__ void resid_load_probe(const JoinProbeParams& p, int64_t r, ResidRow& row, uint32_t& valid) {
  valid = 0;
#pragma unroll
  for (int s = 0; s < kResidSlots; ++s) {
    row.v[s] = 0;
    if (s >= p.resid_n_slots || p.resid_slots[s].side != 0) continue;
    bool ok;
    load_column(p.resid_slots[s].probe, r, p.resid_slots[s].dtype, row.v[s], ok);
    valid |= (ok ? 1u : 0u) << s;
  }
}

// The RESID kernels share ONE out-of-line copy of the interpreter, for the reason agg_kernels.cuh's
// comp_row_interp gives: inlined, it would multiply their code and build time.  NULL counts as false
// (the reference's is_true wrapper); the predicate cannot raise (dbx_op_create_join refuses such).
static __device__ __noinline__ bool resid_true(const JoinProbeParams& p, const ResidRow row, uint32_t valid) {
  bool ok = false;
  int err = 0;
  const CompDev cd{0, p.resid_n_nodes, 0, 1};
  const uint64_t v = comp_row_cond(cd, p.resid_nodes, row.v, valid, ok, err);
  return ok && v != 0;
}

// Is the candidate pair (probe row `row`, build entry e) a matching pair?
template <int KW>
__device__ __forceinline__ bool resid_match(const JoinProbeParams& p, const JEntry<KW>& e, ResidRow row, uint32_t valid) {
#pragma unroll
  for (int s = 0; s < kResidSlots; ++s) {
    if (s >= p.resid_n_slots || p.resid_slots[s].side == 0) continue;
    const ResidSlotDev& rs = p.resid_slots[s];
    uint64_t raw;
    bool ok = true;
    if (rs.from == 0) {
      const int64_t b = (int64_t)(e.row1 & kRowMask) - 1;
      raw = load_raw(rs.src, rs.size, b);
      ok = !rs.valid_bytes || rs.valid_bytes[b];
    } else if (rs.from == 1) {
      raw = e.key;
    } else if (rs.from == 2) {
      raw = e.p0;
      ok = (e.row1 >> 62) & 1;
    } else if (rs.from == 3) {
      raw = entry_p1(e);
      ok = (e.row1 >> 63) & 1;
    } else {
      const int sh = rs.from - 4;
      raw = (sh < 64 ? e.key : key_hi(e)) >> (sh & 63);
    }
    row.v[s] = ok ? raw_image(raw, rs.dtype) : 0;
    valid |= (ok ? 1u : 0u) << s;
  }
  return resid_true(p, row, valid);
}

// Does any key occur twice on the build side?  One thread per slot walks the rest of the slot's
// probe sequence (short at load factor <= 0.5).  A build side without duplicates (the usual
// primary-key dimension table) lets the probe stop at its first match instead of walking on to the
// next empty entry: one dependent L2 round trip per probe row instead of two or more.
template <int KW>
__global__ void join_dup_check_kernel(const __grid_constant__ JoinTableDev t, unsigned int* dup) {
  const int64_t mask = t.cap - 1;
  const JEntry<KW>* const entries = (const JEntry<KW>*)t.entries;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < t.cap; i += (int64_t)gridDim.x * blockDim.x) {
    const JEntry<KW> e = entries[i];
    if (e.row1 == 0) continue;
    int64_t s = (i + 1) & mask;
    for (;;) {
      const JEntry<KW> f = entries[s];
      if (f.row1 == 0) break;
      if (key_eq(f, e.key, key_hi(e))) { *dup = 1; break; }
      s = (s + 1) & mask;
      if (s == i) break;
    }
  }
}

// probe_block + JoinStream::next fused, two probe rows per thread: both rows' entry loads are in
// flight together (the probe is bound by dependent L2 round trips, not by bytes).  Per step of 512
// rows a CTA (1) walks every row's probe sequence, counting its matches and keeping the first
// matching entry in registers, (2) reserves the step's output rows with ONE atomic on the global
// cursor (block scan of the counts; a per-warp reservation costs millions of same-address atomics
// per block and was the bottleneck), (3) writes the first match from registers and re-walks the
// sequence only for rows with several matches.  UNIQUE: the build side has no duplicate keys, so
// a row's walk ends at its first match.
// MARK (the build-side kinds RIGHT, RIGHT SEMI, RIGHT ANTI, FULL): every matching entry's build
// row is marked in p.matched for the final scan.  Racing stores all write 1, so no atomics.  RIGHT
// then emits like INNER, FULL like LEFT, RIGHT SEMI / ANTI emit nothing here.
// KW / PACKED: key width in words and composite keys (see the top of the file); a probe row with a
// NULL in any key column is a miss.  The PACKED instantiations, and the non-unique RF ones
// (the two widest single-key kernels), ask for three resident blocks per SM: without a minimum ptxas caps them near 64 registers and spills, with one it takes up to 94
// registers (two blocks per SM), and the probe is bound by latency, so occupancy counts.
// RF (single key): the join's runtime filter tests min-max and bloom before the table walk; a
// rejected row cannot match and takes the no-match path, which is right for every kind.  The
// RF = false instantiations carry none of it.
// RESID: the residual predicate decides, on every key match (candidate pair), whether the pair is a
// matching pair; only matching pairs are counted, marked, kept as `first` and emitted, so every kind's
// rule ("matched", "no match") reads as "has a matching pair".  The probe row's slots are loaded once
// before the walk; the re-walk evaluates the predicate again and skips the first matching pair.  LEFT
// SEMI / ANTI without MARK stop at the first matching pair.  The RESID = false instantiations carry none
// of it.
template <int KW, bool PACKED, bool UNIQUE, bool MARK, bool RF = false, bool RESID = false>
__global__ void __launch_bounds__(kJoinBlock, (PACKED || (RF && !UNIQUE)) ? 3 : 0) join_probe2_kernel(const __grid_constant__ JoinProbeParams p) {
  __shared__ unsigned int s_warp[kJoinBlock / 32];
  __shared__ unsigned long long s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t mask = p.table.cap - 1;
  const int64_t step = (int64_t)gridDim.x * blockDim.x * 2;
  const int64_t n_iter = (p.n_rows + step - 1) / step;
  const JEntry<KW>* const entries = (const JEntry<KW>*)p.table.entries;
  unsigned int rf_rej = 0;
  // LEFT SEMI / ANTI only ask whether a matching pair exists (with MARK every match is marked)
  const bool stop_at_first = UNIQUE || (RESID && !MARK && (p.kind == DBX_JOIN_LEFT_SEMI || p.kind == DBX_JOIN_LEFT_ANTI));
  for (int64_t it = 0; it < n_iter; ++it) {
    int64_t r[2];
    r[0] = it * step + (int64_t)blockIdx.x * blockDim.x * 2 + threadIdx.x;
    r[1] = r[0] + blockDim.x;
    bool in_range[2], go[2];
    uint64_t k[2] = {0, 0}, kh[2] = {0, 0};
    int64_t b0[2] = {0, 0}, sl[2] = {0, 0};
    unsigned int n_match[2] = {0, 0};
    JEntry<KW> first[2];
    ResidRow prow[2];      // RESID: the probe row's slots
    uint32_t pvalid[2] = {0, 0};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      clear_entry(first[j]);
      in_range[j] = r[j] < p.n_rows;
      if (PACKED) go[j] = in_range[j] && load_packed_key<KW>(p.pack, r[j], k[j], kh[j]);
      else go[j] = in_range[j] && !(p.key.validity && !bit_test(p.key.validity, p.key.vbit_off + r[j]));
      if (RF && go[j]) {
        const uint64_t v = load_key(p.key, r[j]);
        if (!rf_min_max_pass(p.rf, v) || !rf_bloom_pass(p.rf, v)) { go[j] = false; ++rf_rej; }
      }
      if (go[j]) {
        if (!PACKED) k[j] = load_key(p.key, r[j]);
        b0[j] = join_home<KW>(p.table, k[j], kh[j]);
        sl[j] = b0[j];
        if (RESID) resid_load_probe(p, r[j], prow[j], pvalid[j]);
      }
    }
    while (go[0] || go[1]) {  // an empty entry ends a probe sequence
      JEntry<KW> e[2];
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (go[j]) e[j] = load_entry(entries + sl[j]);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (!go[j]) continue;
        if (e[j].row1 == 0) { go[j] = false; continue; }
        if (key_eq(e[j], k[j], kh[j])) {
          if (!RESID || resid_match<KW>(p, e[j], prow[j], pvalid[j])) {
            if (MARK) {  // read first: a dimension row hit by many facts is written once, not per match
              uint8_t* m = p.matched + (int64_t)(e[j].row1 & kRowMask) - 1;
              if (*m == 0) *m = 1;
            }
            if (n_match[j] == 0) first[j] = e[j];
            ++n_match[j];
            if (stop_at_first) { go[j] = false; continue; }
          }
          if (RESID && UNIQUE) { go[j] = false; continue; }  // the row's only candidate
        }
        sl[j] = (sl[j] + 1) & mask;
      }
    }
    bool outer_null[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      // semi / anti: the probe row itself is the output, at most once (a NULL key counts as no match)
      if (p.kind == DBX_JOIN_LEFT_SEMI) n_match[j] = n_match[j] ? 1u : 0u;
      else if (p.kind == DBX_JOIN_LEFT_ANTI) n_match[j] = (in_range[j] && n_match[j] == 0) ? 1u : 0u;
      else if (MARK && (p.kind == DBX_JOIN_RIGHT_SEMI || p.kind == DBX_JOIN_RIGHT_ANTI)) n_match[j] = 0;  // marked only
      outer_null[j] = (p.kind == DBX_JOIN_LEFT || (MARK && p.kind == DBX_JOIN_FULL)) && in_range[j] && n_match[j] == 0;  // preserved row without a match
      if (outer_null[j]) n_match[j] = 1;
    }
    // block-wide exclusive scan of the match counts -> one reservation per CTA and step
    const unsigned int mine = n_match[0] + n_match[1];
    unsigned int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int tot = 0;
      for (int w = 0; w < kJoinBlock / 32; ++w) { const unsigned int c = s_warp[w]; s_warp[w] = tot; tot += c; }
      s_base = tot ? atomicAdd(p.cursor, (unsigned long long)tot) : 0ULL;
    }
    __syncthreads();
    int64_t pos = (int64_t)s_base + s_warp[warp] + incl - mine;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (outer_null[j]) {
        if (pos < p.out_cap) {
          for (int c = 0; c < p.n_probe_cols; ++c) copy_value(p.probe_cols[c], r[j], pos);
          for (int c = 0; c < p.n_build_cols; ++c) store_value(p.build_cols[c], 0, false, pos);
        }
        ++pos;
      } else if (n_match[j] && (p.kind == DBX_JOIN_LEFT_SEMI || p.kind == DBX_JOIN_LEFT_ANTI)) {
        if (pos < p.out_cap)
          for (int c = 0; c < p.n_probe_cols; ++c) copy_value(p.probe_cols[c], r[j], pos);
        ++pos;
      } else if (n_match[j]) {
        emit_match<PACKED>(p, r[j], first[j], pos++);
        if (!UNIQUE && n_match[j] > 1) {  // duplicates of the key on the build side: walk again, skip the first
          int64_t b = b0[j];
          unsigned int seen = 0;
          for (;;) {
            const JEntry<KW> e = load_entry(entries + b);
            if (e.row1 == 0) break;
            if (key_eq(e, k[j], kh[j]) && (!RESID || resid_match<KW>(p, e, prow[j], pvalid[j])) && seen++ > 0)
              emit_match<PACKED>(p, r[j], e, pos++);
            b = (b + 1) & mask;
          }
        }
      }
    }
  }
  if (RF) {  // RuntimeFilterStats: one atomic per warp
    const unsigned int w = __reduce_add_sync(0xffffffffu, rf_rej);
    if (lane == 0 && w) atomicAdd(p.rf_rejected, (unsigned long long)w);
  }
}

// Join::final_probe of the build-side kinds: stream the matched map and compact the selected build
// rows (want = 1: rows matched at least once, RIGHT SEMI; want = 0: rows never matched, RIGHT /
// RIGHT ANTI / FULL, NULL-key rows included since they were never inserted).  Every build column is
// gathered by build row from its HBM-resident column; positions are reserved like the probe's: a
// block-wide scan, then one cursor atomic per CTA and step.  With out_cap = 0 it only counts.
struct FinalColDev {
  const void* src;
  const uint8_t* src_valid;  // one byte per build row, or null (all valid)
  void* dst;
  uint8_t* dst_valid;        // one byte per output row, or null
  int32_t size;
  int32_t pad;
};
struct JoinFinalParams {
  FinalColDev cols[kMaxJoinCols];
  int32_t n_cols;
  int32_t want;
  const uint8_t* matched;
  int64_t n_rows;
  int64_t out_cap;
  unsigned long long* cursor;
};
__global__ void __launch_bounds__(kJoinBlock) join_final_scan_kernel(const __grid_constant__ JoinFinalParams p) {
  __shared__ unsigned int s_warp[kJoinBlock / 32];
  __shared__ unsigned long long s_base;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  const int64_t n_iter = (p.n_rows + step - 1) / step;
  for (int64_t it = 0; it < n_iter; ++it) {
    const int64_t r = it * step + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool sel = r < p.n_rows && (p.matched[r] != 0) == (p.want != 0);
    const unsigned int ballot = __ballot_sync(0xffffffffu, sel);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int tot = 0;
      for (int w = 0; w < kJoinBlock / 32; ++w) { const unsigned int c = s_warp[w]; s_warp[w] = tot; tot += c; }
      s_base = tot ? atomicAdd(p.cursor, (unsigned long long)tot) : 0ULL;
    }
    __syncthreads();
    const int64_t pos = (int64_t)s_base + s_warp[warp] + __popc(ballot & ((1u << lane) - 1u));
    __syncthreads();
    if (sel && pos < p.out_cap) {
      for (int c = 0; c < p.n_cols; ++c) {
        const FinalColDev& fc = p.cols[c];
        switch (fc.size) {
          case 8: ((uint64_t*)fc.dst)[pos] = ((const uint64_t*)fc.src)[r]; break;
          case 4: ((uint32_t*)fc.dst)[pos] = ((const uint32_t*)fc.src)[r]; break;
          case 2: ((uint16_t*)fc.dst)[pos] = ((const uint16_t*)fc.src)[r]; break;
          default: ((uint8_t*)fc.dst)[pos] = ((const uint8_t*)fc.src)[r]; break;
        }
        if (fc.dst_valid) fc.dst_valid[pos] = fc.src_valid ? fc.src_valid[r] : 1;
      }
    }
  }
}

__global__ void pack_bits_kernel(const uint8_t* bytes, int64_t n, uint8_t* bits) {
  int64_t nb = (n + 7) / 8;
  for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (int64_t)gridDim.x * blockDim.x) {
    uint32_t v = 0;
    for (int k = 0; k < 8; ++k) {
      int64_t i = b * 8 + k;
      if (i < n && bytes[i]) v |= 1u << k;
    }
    bits[b] = (uint8_t)v;
  }
}

inline int64_t next_pow2_i64(int64_t x) {
  int64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}
// the kinds that keep build rows: they mark matches during the probe and emit from final_probe
inline bool build_side_kind(int kind) { return kind >= DBX_JOIN_RIGHT && kind <= DBX_JOIN_FULL; }
inline int grid_rows(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + kJoinBlock - 1) / kJoinBlock, (int64_t)kNumSMs * 8)); }

// Device column that grows by appending pushed blocks (build side).
struct GrowCol {
  DevBuf data, valid_bytes;  // validity kept as one byte per row (simplifies appends at any offset)
  int64_t rows = 0;
  int size = 8;
  bool nullable = false;
};

__global__ void bits_to_bytes_kernel(const uint8_t* bits, int64_t bit_off, int64_t n, uint8_t* bytes) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    bytes[i] = bits ? (uint8_t)bit_test(bits, bit_off + i) : 1;
}

}  // namespace

class JoinOp : public Op {
 public:
  dbx_join_params prm;
  int n_build_cols = 0, n_probe_cols = 0;
  int build_dtype[kMaxJoinCols], probe_dtype[kMaxJoinCols];
  bool build_nullable[kMaxJoinCols], probe_nullable[kMaxJoinCols];
  Stager stager;
  std::vector<GrowCol> build;
  int64_t build_rows = 0;
  DevBuf table_buf, cursor;
  int64_t table_cap = 0;
  PinnedBuf host;
  int inline_col[2] = {-1, -1};
  bool build_unique = false;  // no key occurs twice on the build side (checked after the build)
  JoinTableDev table_view() const { return JoinTableDev{(JoinEntry*)table_buf.p, table_cap}; }
  std::vector<std::unique_ptr<OwnedBlock>> outputs;  // joined blocks waiting to be pulled (device resident)
  size_t next_out = 0;
  DevBuf matched;             // build-side kinds: one byte per build row, 1 once any probe row matched it
  std::shared_ptr<RfData> rf_probe;  // runtime filter the probe kernel tests (single key), shared with its handle
  bool final_probed = false;  // Join::final_probe ran: no more probe blocks until reset
  // key pairs (1 + n_extra_keys); packed: composite key of key_words words, fields in *_part
  int n_keys = 1, key_words = 1;
  bool packed = false;
  int key_build_col[DBX_MAX_JOIN_KEYS], key_probe_col[DBX_MAX_JOIN_KEYS];
  KeyPartDev build_part[DBX_MAX_JOIN_KEYS], probe_part[DBX_MAX_JOIN_KEYS];
  // bit field of build column c in the packed key, -1 if c is not a key column
  int build_key_shift(int c) const {
    for (int i = 0; i < n_keys; ++i) if (key_build_col[i] == c) return build_part[i].shift;
    return -1;
  }

  // input_types = build schema (params.n_build_cols columns) followed by the probe schema.
  int32_t init(const dbx_join_params* p, const int32_t* types, int32_t n, int dev) {
    DBX_TRY(base_init(dev));
    prm = *p;
    if (p->kind < DBX_JOIN_INNER || p->kind > DBX_JOIN_FULL) { err.set("join: unknown dbx_join_kind"); return DBX_ERR_UNSUPPORTED; }
    n_build_cols = p->n_build_cols;
    n_probe_cols = n - n_build_cols;
    if (n_build_cols <= 0 || n_probe_cols <= 0 || n_build_cols > kMaxJoinCols || n_probe_cols > kMaxJoinCols) {
      err.set("join: input_types must hold the build schema (params.n_build_cols columns) followed by the probe schema");
      return DBX_ERR_INVALID;
    }
    for (int i = 0; i < n_build_cols; ++i) { build_dtype[i] = types[i] & 0xFF; build_nullable[i] = (types[i] & DBX_NULLABLE) != 0; }
    for (int i = 0; i < n_probe_cols; ++i) { probe_dtype[i] = types[n_build_cols + i] & 0xFF; probe_nullable[i] = (types[n_build_cols + i] & DBX_NULLABLE) != 0; }
    if (p->build_key_col < 0 || p->build_key_col >= n_build_cols || p->probe_key_col < 0 || p->probe_key_col >= n_probe_cols) { err.set("join: key column outside the schema"); return DBX_ERR_INVALID; }
    if (p->n_extra_keys < 0 || p->n_extra_keys > DBX_MAX_JOIN_KEYS - 1) { err.set("join: n_extra_keys must be 0 .. DBX_MAX_JOIN_KEYS - 1"); return DBX_ERR_INVALID; }
    n_keys = 1 + p->n_extra_keys;
    for (int i = 0; i < n_keys; ++i) {
      key_build_col[i] = i == 0 ? p->build_key_col : p->extra_build_key_cols[i - 1];
      key_probe_col[i] = i == 0 ? p->probe_key_col : p->extra_probe_key_cols[i - 1];
      if (key_build_col[i] < 0 || key_build_col[i] >= n_build_cols || key_probe_col[i] < 0 || key_probe_col[i] >= n_probe_cols) { err.set("join: key column outside the schema"); return DBX_ERR_INVALID; }
    }
    auto int_key = [](int dt) { return dt != DBX_BOOL && dt != DBX_F32 && dt != DBX_F64 && dtype_size(dt) > 0; };
    for (int i = 0; i < n_keys; ++i)
      if (!int_key(build_dtype[key_build_col[i]]) || !int_key(probe_dtype[key_probe_col[i]])) { err.set("join: keys must be integer columns"); return DBX_ERR_UNSUPPORTED; }
    for (int i = 0; i < n_build_cols; ++i) if (dtype_size(build_dtype[i]) == 0) { err.set("join: only fixed-width numeric columns are supported"); return DBX_ERR_UNSUPPORTED; }
    for (int i = 0; i < n_probe_cols; ++i) if (dtype_size(probe_dtype[i]) == 0) { err.set("join: only fixed-width numeric columns are supported"); return DBX_ERR_UNSUPPORTED; }
    // keys of different widths/signedness compare by value: both are widened to 64 bits
    // (sign-extended if signed), the common super type of the reference's key cast.  The one pair
    // with no 64-bit super type is (signed, UInt64): the widened images of -1 and 2^64-1 coincide,
    // so it is refused here (the reference's type checker casts both sides to a wider type first;
    // a caller wanting that join casts the keys before the operator, as the reference's planner does).
    for (int i = 0; i < n_keys; ++i) {
      const int bk = build_dtype[key_build_col[i]], pk = probe_dtype[key_probe_col[i]];
      const bool bs = dtype_class(bk) == VC_INT, ps = dtype_class(pk) == VC_INT;
      if ((bk == DBX_U64 && ps) || (pk == DBX_U64 && bs)) { err.set("join: a signed key cannot be compared with a UInt64 key without a cast (no common 64-bit type)"); return DBX_ERR_UNSUPPORTED; }
    }
    // composite keys: one bit field per pair, as wide as the pair's common type (same signedness:
    // the larger size; signed S with unsigned U: max(S, 2U) bytes, which holds both value ranges),
    // packed from bit 0 upward; a field never straddles the two words (the aggregate's rule)
    packed = n_keys > 1;
    key_words = 1;
    if (packed) {
      int bits = 0;
      for (int i = 0; i < n_keys; ++i) {
        const int bk = build_dtype[key_build_col[i]], pk = probe_dtype[key_probe_col[i]];
        const int bsz = dtype_size(bk), psz = dtype_size(pk);
        const bool bs = dtype_class(bk) == VC_INT, ps = dtype_class(pk) == VC_INT;
        const int bytes = bs == ps ? std::max(bsz, psz) : (bs ? std::max(bsz, 2 * psz) : std::max(psz, 2 * bsz));
        const int w = 8 * bytes;
        if (bits < 64 && bits + w > 64) bits = 64;
        for (KeyPartDev* kp : {&build_part[i], &probe_part[i]}) {
          memset(kp, 0, sizeof(*kp));
          kp->shift = bits;
          kp->null_shift = -1;  // NULL rows never enter the table or match: no NULL flags
          kp->mask = w == 64 ? ~0ULL : ((1ULL << w) - 1);
        }
        build_part[i].slot = key_build_col[i]; build_part[i].dtype = bk;
        probe_part[i].slot = key_probe_col[i]; probe_part[i].dtype = pk;
        bits += w;
      }
      if (bits > 128) { err.set("join: composite keys wider than 128 bits need 256-bit or serialised join keys: not built"); return DBX_ERR_UNSUPPORTED; }
      key_words = bits > 64 ? 2 : 1;
    }
    build.resize(n_build_cols);
    for (int i = 0; i < n_build_cols; ++i) { build[i].size = dtype_size(build_dtype[i]); build[i].nullable = build_nullable[i]; }
    DBX_TRY(stager.init(dev, stream, &err));
    DBX_CUDA_TRY(err, cursor.ensure(64));
    DBX_CUDA_TRY(err, host.ensure(64));
    return DBX_OK;
  }

  // Join::add_block (build side): append the block's columns to the HBM-resident build side
  int32_t push(const dbx_block* b) override {
    if (b->num_cols != n_build_cols) { err.set("add_block: block does not match the build schema"); return DBX_ERR_INVALID; }
    const int64_t n = b->num_rows;
    if (n == 0) return DBX_OK;
    DBX_TRY(stager.begin());
    for (int c = 0; c < n_build_cols; ++c) {
      const dbx_column& col = b->cols[c];
      if (col.dtype != build_dtype[c] || col.len != n || col.is_const) { err.set("add_block: column dtype/length mismatch (const build columns unsupported)"); return DBX_ERR_INVALID; }
      DevCol dc;
      DBX_TRY(stager.stage(col, c, &dc));
      GrowCol& g = build[c];
      const size_t need = (size_t)(build_rows + n) * g.size;
      if (need > g.data.bytes) {  // grow, preserving the rows already appended (the hint avoids re-allocations)
        DevBuf nb;
        DBX_CUDA_TRY(err, nb.ensure(std::max({need, g.data.bytes * 2, (size_t)std::max<int64_t>(prm.expected_build_rows, 0) * g.size})));
        if (build_rows) DBX_CUDA_TRY(err, cudaMemcpyAsync(nb.p, g.data.p, (size_t)build_rows * g.size, cudaMemcpyDeviceToDevice, stream));
        DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
        g.data = std::move(nb);
      }
      DBX_CUDA_TRY(err, cudaMemcpyAsync((char*)g.data.p + (size_t)build_rows * g.size, dc.data, (size_t)n * g.size, cudaMemcpyDeviceToDevice, stream));
      if (g.nullable) {
        const size_t vneed = (size_t)(build_rows + n);
        if (vneed > g.valid_bytes.bytes) {
          DevBuf nb;
          DBX_CUDA_TRY(err, nb.ensure(std::max({vneed, g.valid_bytes.bytes * 2, (size_t)std::max<int64_t>(prm.expected_build_rows, 0)})));
          if (build_rows) DBX_CUDA_TRY(err, cudaMemcpyAsync(nb.p, g.valid_bytes.p, (size_t)build_rows, cudaMemcpyDeviceToDevice, stream));
          DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
          g.valid_bytes = std::move(nb);
        }
        bits_to_bytes_kernel<<<grid_rows(n), kJoinBlock, 0, stream>>>(dc.validity, dc.vbit_off, n, (uint8_t*)g.valid_bytes.p + build_rows);
        count_launch();
      }
    }
    build_rows += n;
    DBX_TRY(stager.end());
    return DBX_OK;
  }

  // Join::final_build: size the table for the build row count and insert every row
  int32_t finish() override {
    table_cap = std::max<int64_t>(next_pow2_i64(2 * std::max<int64_t>(build_rows, 1)), 1024);  // with_build_row_num
    if (build_rows >= (int64_t)kRowMask) { err.set("join: too many build rows"); return DBX_ERR_UNSUPPORTED; }
    DBX_CUDA_TRY(err, table_buf.ensure((size_t)table_cap * sizeof(JoinEntry)));
    DBX_CUDA_TRY(err, cudaMemsetAsync(table_buf.p, 0, (size_t)table_cap * sizeof(JoinEntry), stream));
    if (build_side_kind(prm.kind)) {  // the matched map, indexed by build row (NULL-key rows stay 0)
      DBX_CUDA_TRY(err, matched.ensure((size_t)std::max<int64_t>(build_rows, 1)));
      DBX_CUDA_TRY(err, cudaMemsetAsync(matched.p, 0, (size_t)std::max<int64_t>(build_rows, 1), stream));
    }
    if (build_rows) {
      GrowCol& kc = build[prm.build_key_col];
      DevCol key;
      memset(&key, 0, sizeof(key));
      key.data = kc.data.p;
      key.dtype = build_dtype[prm.build_key_col];
      // build-side validity is stored as bytes; expose it as a bitmap-free predicate by packing
      DevBuf kbits;
      if (kc.nullable && !packed) {
        DBX_CUDA_TRY(err, kbits.ensure((size_t)(build_rows + 7) / 8 + 8));
        pack_bits_kernel<<<grid_rows((build_rows + 7) / 8), kJoinBlock, 0, stream>>>((const uint8_t*)kc.valid_bytes.p, build_rows, (uint8_t*)kbits.p);
        count_launch();
        key.validity = (const uint8_t*)kbits.p;
      }
      // composite keys: every key column, NULL bitmaps packed from the stored bytes as above
      JoinKeyPack pk;
      memset(&pk, 0, sizeof(pk));
      DevBuf pk_bits[DBX_MAX_JOIN_KEYS];
      if (packed) {
        pk.n = n_keys;
        for (int i = 0; i < n_keys; ++i) {
          const GrowCol& g = build[key_build_col[i]];
          pk.cols[i].data = g.data.p;
          pk.cols[i].dtype = build_dtype[key_build_col[i]];
          pk.parts[i] = build_part[i];
          if (g.nullable) {
            DBX_CUDA_TRY(err, pk_bits[i].ensure((size_t)(build_rows + 7) / 8 + 8));
            pack_bits_kernel<<<grid_rows((build_rows + 7) / 8), kJoinBlock, 0, stream>>>((const uint8_t*)g.valid_bytes.p, build_rows, (uint8_t*)pk_bits[i].p);
            count_launch();
            pk.cols[i].validity = (const uint8_t*)pk_bits[i].p;
          }
        }
      }
      JoinTableDev t = table_view();
      // the first two non-key build columns travel inside the entries (one with a 128-bit key)
      InlineColDev ic[2];
      memset(ic, 0, sizeof(ic));
      inline_col[0] = inline_col[1] = -1;
      const int n_inline = key_words == 2 ? 1 : 2;
      for (int c = 0, k = 0; c < n_build_cols && k < n_inline; ++c) {
        if (packed ? build_key_shift(c) >= 0 : c == prm.build_key_col) continue;
        inline_col[k] = c;
        ic[k].src = build[c].data.p;
        ic[k].valid_bytes = build[c].nullable ? (const uint8_t*)build[c].valid_bytes.p : nullptr;
        ic[k].size = build[c].size;
        ic[k].on = 1;
        ++k;
      }
      const int grid = grid_rows(build_rows);
      if (!packed) join_build_kernel<1, false><<<grid, kJoinBlock, 0, stream>>>(key, build_rows, t, ic[0], ic[1], pk);
      else if (key_words == 1) join_build_kernel<1, true><<<grid, kJoinBlock, 0, stream>>>(key, build_rows, t, ic[0], ic[1], pk);
      else join_build_kernel<2, true><<<grid, kJoinBlock, 0, stream>>>(key, build_rows, t, ic[0], ic[1], pk);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      DBX_CUDA_TRY(err, cudaMemsetAsync(cursor.p, 0, 16, stream));
      if (key_words == 2) join_dup_check_kernel<2><<<grid_rows(table_cap), kJoinBlock, 0, stream>>>(t, (unsigned int*)cursor.p + 2);
      else join_dup_check_kernel<1><<<grid_rows(table_cap), kJoinBlock, 0, stream>>>(t, (unsigned int*)cursor.p + 2);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, (unsigned int*)cursor.p + 2, 4, cudaMemcpyDeviceToHost, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      build_unique = *(unsigned int*)host.p == 0 && !getenv("DBX_JOIN_NO_UNIQUE");
    } else {
      build_unique = true;
    }
    return DBX_OK;
  }

  // Residual predicate (dbx_op_create_join): the type-checked program, its COLUMN nodes renumbered to
  // slots; resid_col[s] = schema column of slot s (build columns, then the probe columns)
  int resid_n_nodes = 0, resid_n_slots = 0;
  NodeDev resid_nodes[kMaxExprNodes];
  int resid_col[kResidSlots];

  int32_t set_residual(const dbx_expr* e) {
    if (!e || e->n_nodes == 0) return DBX_OK;
    const int n = n_build_cols + n_probe_cols;
    int dtypes[2 * kMaxJoinCols];
    bool nullable[2 * kMaxJoinCols];
    for (int c = 0; c < n_build_cols; ++c) { dtypes[c] = build_dtype[c]; nullable[c] = build_nullable[c]; }
    for (int c = 0; c < n_probe_cols; ++c) { dtypes[n_build_cols + c] = probe_dtype[c]; nullable[n_build_cols + c] = probe_nullable[c]; }
    int dt = 0;
    bool out_nullable = false;
    const int32_t st = infer_expr_types(*e, n, dtypes, nullable, resid_nodes, &dt, &out_nullable, err);
    if (st != DBX_OK) { err.set("join other_predicate: " + err.msg); return st; }
    if (dt != DBX_BOOL) { err.set("join other_predicate: the predicate must be Boolean (nullable or not)"); return DBX_ERR_INVALID; }
    if (expr_can_raise(resid_nodes, e->n_nodes)) {
      err.set("join other_predicate: a predicate that can raise (`/`, `div` or `%` by a non-constant or zero divisor, an overflowing "
              "cast, a negation of an Int64 / UInt64) is not built: the reference's selector evaluates AND / OR children under an "
              "adaptive order (expression/src/filter/selector.rs:182-300), so which pairs reach it there is not deterministic");
      return DBX_ERR_UNSUPPORTED;
    }
    int n_slots = 0;
    for (int i = 0; i < e->n_nodes; ++i) {
      if (resid_nodes[i].kind != DBX_EXPR_COLUMN) continue;
      const int c = resid_nodes[i].col;
      int s = 0;
      while (s < n_slots && resid_col[s] != c) ++s;
      if (s == n_slots) {
        if (n_slots == kResidSlots) {
          err.set("join other_predicate: the predicate references more than 8 distinct columns (the interpreter has 8 value slots)");
          return DBX_ERR_UNSUPPORTED;
        }
        resid_col[n_slots++] = c;
      }
      resid_nodes[i].col = s;
    }
    resid_n_nodes = e->n_nodes;
    resid_n_slots = n_slots;
    return DBX_OK;
  }
  // the device slot table of one probe block (probe columns `cols`)
  void fill_residual(JoinProbeParams& pp, const DevCol* cols) {
    pp.resid_n_nodes = resid_n_nodes;
    pp.resid_n_slots = resid_n_slots;
    memcpy(pp.resid_nodes, resid_nodes, sizeof(NodeDev) * resid_n_nodes);
    for (int s = 0; s < resid_n_slots; ++s) {
      ResidSlotDev& rs = pp.resid_slots[s];
      const int c = resid_col[s];
      if (c >= n_build_cols) {
        rs.side = 0;
        rs.probe = cols[c - n_build_cols];
        rs.dtype = probe_dtype[c - n_build_cols];
        continue;
      }
      rs.side = 1;
      rs.dtype = build_dtype[c];
      rs.size = build[c].size;
      if (packed && build_key_shift(c) >= 0) rs.from = 4 + build_key_shift(c);  // the packed key's field
      else rs.from = c == prm.build_key_col ? 1 : (c == inline_col[0] ? 2 : (c == inline_col[1] ? 3 : 0));
      rs.src = build[c].data.p;
      rs.valid_bytes = build[c].nullable ? (const uint8_t*)build[c].valid_bytes.p : nullptr;
    }
  }

  template <int KW, bool PACKED, bool RF = false, bool RESID = false>
  void launch_probe2(const JoinProbeParams& pp, int grid) {
    if (pp.matched) {
      if (build_unique) join_probe2_kernel<KW, PACKED, true, true, RF, RESID><<<grid, kJoinBlock, 0, stream>>>(pp);
      else join_probe2_kernel<KW, PACKED, false, true, RF, RESID><<<grid, kJoinBlock, 0, stream>>>(pp);
    } else {
      if (build_unique) join_probe2_kernel<KW, PACKED, true, false, RF, RESID><<<grid, kJoinBlock, 0, stream>>>(pp);
      else join_probe2_kernel<KW, PACKED, false, false, RF, RESID><<<grid, kJoinBlock, 0, stream>>>(pp);
    }
  }
  template <bool RESID>
  void launch_probe_as(const JoinProbeParams& pp, int grid) {
    if (packed) {
      if (key_words == 2) launch_probe2<2, true, false, RESID>(pp, grid);
      else launch_probe2<1, true, false, RESID>(pp, grid);
      return;
    }
    if (rf_probe) { launch_probe2<1, false, true, RESID>(pp, grid); return; }
    launch_probe2<1, false, false, RESID>(pp, grid);
  }
  void launch_probe(const JoinProbeParams& pp, int64_t rows) {
    const int grid = grid_rows((rows + 1) / 2);
    if (resid_n_nodes) launch_probe_as<true>(pp, grid);
    else launch_probe_as<false>(pp, grid);
  }

  // Join::probe_block: join one probe block; the joined block is queued for dbx_op_pull
  int32_t probe(const dbx_block* b) {
    if (!finished) { err.set("probe before final_build"); return DBX_ERR_STATE; }
    if (final_probed) { err.set("probe_block after final_probe (reset the operator first)"); return DBX_ERR_STATE; }
    if (b->num_cols != n_probe_cols) { err.set("probe_block: block does not match the probe schema"); return DBX_ERR_INVALID; }
    const int64_t n = b->num_rows;
    if (n == 0) return DBX_OK;
    if (rf_probe) rf_probe->probe_checked += n;
    DevCol cols[kMaxJoinCols];
    DBX_TRY(stager.begin());
    for (int c = 0; c < n_probe_cols; ++c) {
      const dbx_column& col = b->cols[c];
      if (col.dtype != probe_dtype[c] || col.len != n || col.is_const) { err.set("probe_block: column dtype/length mismatch (const probe columns unsupported)"); return DBX_ERR_INVALID; }
      DBX_TRY(stager.stage(col, c, &cols[c]));
    }
    // RIGHT SEMI / RIGHT ANTI only mark the matched map here: no output columns, no blocks
    const bool marks_only = prm.kind == DBX_JOIN_RIGHT_SEMI || prm.kind == DBX_JOIN_RIGHT_ANTI;
    int64_t out_cap = marks_only ? 0 : n + n / 8 + 1024;  // optimistic: about one match per probe row
    DBX_TRY(timing_begin());
    for (int attempt = 0; attempt < 2; ++attempt) {
      auto ob = std::make_unique<OwnedBlock>();
    ob->stream = stream;  // freed in order behind this operator's enqueued work
      ob->device = device;
      JoinProbeParams pp;
      memset(&pp, 0, sizeof(pp));
      pp.key = cols[prm.probe_key_col];
      pp.table = table_view();
      pp.n_probe_cols = marks_only ? 0 : n_probe_cols;
      pp.n_build_cols = (prm.kind == DBX_JOIN_INNER || prm.kind == DBX_JOIN_LEFT || prm.kind == DBX_JOIN_RIGHT || prm.kind == DBX_JOIN_FULL) ? n_build_cols : 0;
      pp.kind = prm.kind;
      pp.n_rows = n;
      pp.out_cap = out_cap;
      pp.cursor = (unsigned long long*)cursor.p;
      pp.matched = build_side_kind(prm.kind) ? (uint8_t*)matched.p : nullptr;
      if (rf_probe) {  // a retried probe must not count its rejections twice
        pp.rf = rf_probe->parts[0].dev();
        pp.rf_rejected = attempt == 0 ? (unsigned long long*)rf_probe->probe_rejected.p : (unsigned long long*)cursor.p + 4;
      }
      if (packed) {
        pp.pack.n = n_keys;
        for (int i = 0; i < n_keys; ++i) {
          pp.pack.cols[i] = cols[key_probe_col[i]];
          pp.pack.parts[i] = probe_part[i];
        }
      }
      if (resid_n_nodes) fill_residual(pp, cols);
      std::vector<uint8_t*> valid_bytes;
      auto add_out = [&](JoinColDev& jc, int dtype, bool nullable) -> int32_t {
        void* d = nullptr;
        DBX_CUDA_TRY(err, pool_alloc(device, stream, (size_t)out_cap * dtype_size(dtype), &d));
        ob->dev_allocs.push_back(d);
        jc.dst = d;
        jc.size = dtype_size(dtype);
        uint8_t* vb = nullptr;
        if (nullable) {
          DBX_CUDA_TRY(err, pool_alloc(device, stream, (size_t)out_cap, (void**)&vb));
          ob->dev_allocs.push_back(vb);
        }
        jc.dst_valid = vb;
        valid_bytes.push_back(vb);
        dbx_column oc;
        memset(&oc, 0, sizeof(oc));
        oc.dtype = dtype; oc.mem = DBX_MEM_DEVICE; oc.data = d; oc.null_count = nullable ? -1 : 0;
        ob->cols.push_back(oc);
        return DBX_OK;
      };
      // output column order = probe projection then build projection (inner_join.rs:236-245);
      // RIGHT and FULL return the probe columns Nullable in every block (their final blocks carry NULLs there)
      const bool probe_null = prm.kind == DBX_JOIN_RIGHT || prm.kind == DBX_JOIN_FULL;
      for (int c = 0; c < pp.n_probe_cols; ++c) {
        pp.probe_cols[c].src = cols[c].data;
        pp.probe_cols[c].src_validity = cols[c].validity;
        pp.probe_cols[c].src_vbit_off = cols[c].vbit_off;
        DBX_TRY(add_out(pp.probe_cols[c], probe_dtype[c], probe_nullable[c] || probe_null));
      }
      DevBuf build_bits[kMaxJoinCols];
      for (int c = 0; c < pp.n_build_cols; ++c) {
        pp.build_cols[c].src = build[c].data.p;
        if (packed && build_key_shift(c) >= 0) pp.build_cols[c].from = 4 + build_key_shift(c);  // decoded from the entry's key
        else pp.build_cols[c].from = c == prm.build_key_col ? 1 : (c == inline_col[0] ? 2 : (c == inline_col[1] ? 3 : 0));
        if (build[c].nullable && pp.build_cols[c].from == 0) {  // bytes -> use the byte array directly through a 1-byte "bitmap" trick: pack once
          DBX_CUDA_TRY(err, build_bits[c].ensure((size_t)(build_rows + 7) / 8 + 8));
          pack_bits_kernel<<<grid_rows((build_rows + 7) / 8), kJoinBlock, 0, stream>>>((const uint8_t*)build[c].valid_bytes.p, build_rows, (uint8_t*)build_bits[c].p);
          count_launch();
          pp.build_cols[c].src_validity = (const uint8_t*)build_bits[c].p;
        }
        DBX_TRY(add_out(pp.build_cols[c], build_dtype[c], build_nullable[c] || prm.kind == DBX_JOIN_LEFT || prm.kind == DBX_JOIN_FULL));
      }
      DBX_CUDA_TRY(err, cudaMemsetAsync(cursor.p, 0, 8, stream));
      launch_probe(pp, n);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, cursor.p, 8, cudaMemcpyDeviceToHost, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      const int64_t matches = (int64_t)*(unsigned long long*)host.p;
      if (matches > out_cap) {  // many-to-many: retry once with the exact size
        out_cap = matches;
        continue;
      }
      for (size_t i = 0; i < ob->cols.size(); ++i) {
        ob->cols[i].len = matches;
        if (valid_bytes[i]) {
          uint8_t* bits = nullptr;
          DBX_CUDA_TRY(err, pool_alloc(device, stream, (size_t)(matches + 7) / 8 + 8, (void**)&bits));
          ob->dev_allocs.push_back(bits);
          pack_bits_kernel<<<grid_rows((matches + 7) / 8 + 1), kJoinBlock, 0, stream>>>(valid_bytes[i], matches, bits);
          count_launch();
          ob->cols[i].validity = bits;
        }
      }
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      if (matches > 0) outputs.push_back(std::move(ob));
      break;
    }
    DBX_TRY(timing_end());
    DBX_TRY(stager.end());
    return DBX_OK;
  }

  // Join::final_probe (right_join.rs, right_join_semi.rs, right_join_anti.rs; FULL as in
  // hash_join_probe_state.rs:455-567): once every probe block is done, queue the build rows that were
  // never matched (RIGHT, RIGHT ANTI, FULL) or matched at least once (RIGHT SEMI), for dbx_op_pull.
  // RIGHT and FULL put Const NULL entries on the probe side (the reference's null_block), so
  // nothing is written for them.  A no-op for the probe-side kinds, and for a second call.
  int32_t final_probe() {
    if (!finished) { err.set("final_probe before final_build"); return DBX_ERR_STATE; }
    if (final_probed) return DBX_OK;
    final_probed = true;
    if (!build_side_kind(prm.kind) || build_rows == 0) return DBX_OK;
    JoinFinalParams fp;
    memset(&fp, 0, sizeof(fp));
    fp.n_cols = n_build_cols;
    fp.want = prm.kind == DBX_JOIN_RIGHT_SEMI ? 1 : 0;
    fp.matched = (const uint8_t*)matched.p;
    fp.n_rows = build_rows;
    fp.cursor = (unsigned long long*)cursor.p;
    // pass 1 counts (out_cap = 0), so the output is allocated exactly
    DBX_TRY(timing_begin());
    DBX_CUDA_TRY(err, cudaMemsetAsync(cursor.p, 0, 8, stream));
    join_final_scan_kernel<<<grid_rows(build_rows), kJoinBlock, 0, stream>>>(fp);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    DBX_TRY(timing_end());
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, cursor.p, 8, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const int64_t rows = (int64_t)*(unsigned long long*)host.p;
    if (rows == 0) return DBX_OK;
    auto ob = std::make_unique<OwnedBlock>();
    ob->stream = stream;
    ob->device = device;
    if (prm.kind == DBX_JOIN_RIGHT || prm.kind == DBX_JOIN_FULL) {
      for (int c = 0; c < n_probe_cols; ++c) {
        dbx_column oc;
        memset(&oc, 0, sizeof(oc));
        oc.dtype = probe_dtype[c]; oc.mem = DBX_MEM_DEVICE; oc.is_const = 1; oc.len = rows; oc.null_count = rows;
        oc.konst.dtype = probe_dtype[c]; oc.konst.is_null = 1;
        ob->cols.push_back(oc);
      }
    }
    std::vector<uint8_t*> valid_bytes;
    for (int c = 0; c < n_build_cols; ++c) {
      const int sz = build[c].size;
      void* d = nullptr;
      DBX_CUDA_TRY(err, pool_alloc(device, stream, (size_t)rows * sz, &d));
      ob->dev_allocs.push_back(d);
      uint8_t* vb = nullptr;
      if (build_nullable[c] || prm.kind == DBX_JOIN_FULL) {
        DBX_CUDA_TRY(err, pool_alloc(device, stream, (size_t)rows, (void**)&vb));
        ob->dev_allocs.push_back(vb);
      }
      valid_bytes.push_back(vb);
      fp.cols[c] = FinalColDev{build[c].data.p, build[c].nullable ? (const uint8_t*)build[c].valid_bytes.p : nullptr, d, vb, sz, 0};
      dbx_column oc;
      memset(&oc, 0, sizeof(oc));
      oc.dtype = build_dtype[c]; oc.mem = DBX_MEM_DEVICE; oc.data = d; oc.len = rows; oc.null_count = vb ? -1 : 0;
      ob->cols.push_back(oc);
    }
    fp.out_cap = rows;
    DBX_TRY(timing_begin());
    DBX_CUDA_TRY(err, cudaMemsetAsync(cursor.p, 0, 8, stream));
    join_final_scan_kernel<<<grid_rows(build_rows), kJoinBlock, 0, stream>>>(fp);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    DBX_TRY(timing_end());
    const size_t first_build = ob->cols.size() - (size_t)n_build_cols;
    for (int c = 0; c < n_build_cols; ++c) {
      if (!valid_bytes[c]) continue;
      uint8_t* bits = nullptr;
      DBX_CUDA_TRY(err, pool_alloc(device, stream, (size_t)(rows + 7) / 8 + 8, (void**)&bits));
      ob->dev_allocs.push_back(bits);
      pack_bits_kernel<<<grid_rows((rows + 7) / 8 + 1), kJoinBlock, 0, stream>>>(valid_bytes[c], rows, bits);
      count_launch();
      ob->cols[first_build + c].validity = bits;
    }
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    outputs.push_back(std::move(ob));
    return DBX_OK;
  }

  // JoinStream::next
  int32_t pull(int32_t out_mem, dbx_block* out, int32_t* has_block) override {
    if (next_out >= outputs.size()) { *has_block = 0; outputs.clear(); next_out = 0; return DBX_OK; }
    std::unique_ptr<OwnedBlock> ob = std::move(outputs[next_out++]);
    *has_block = 1;
    if (out_mem == DBX_MEM_DEVICE) return fill_owned_block(ob.release(), out);
    auto hb = std::make_unique<OwnedBlock>();
    hb->device = device;
    for (const dbx_column& dc : ob->cols) {
      dbx_column c = dc;
      c.mem = DBX_MEM_HOST;
      if (dc.is_const) { hb->cols.push_back(c); continue; }  // Const entries carry no data
      size_t bytes = (size_t)dc.len * dtype_size(dc.dtype);
      void* hp = nullptr;
      DBX_CUDA_TRY(err, pinned_alloc(bytes, &hp));
      hb->host_allocs.push_back(hp);
      if (bytes) DBX_CUDA_TRY(err, cudaMemcpyAsync(hp, dc.data, bytes, cudaMemcpyDeviceToHost, stream));
      c.data = hp;
      if (dc.validity) {
        size_t vb = (size_t)(dc.len + 7) / 8;
        void* hv = nullptr;
        DBX_CUDA_TRY(err, pinned_alloc(vb, &hv));
        hb->host_allocs.push_back(hv);
        if (vb) DBX_CUDA_TRY(err, cudaMemcpyAsync(hv, dc.validity, vb, cudaMemcpyDeviceToHost, stream));
        c.validity = (const uint8_t*)hv;
      }
      hb->cols.push_back(c);
    }
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    return fill_owned_block(hb.release(), out);
  }

  // Join runtime filter (runtime_filter.cu) of the finished build side; in_probe also hands it to the
  // probe kernel until reset
  int32_t runtime_filter(const dbx_runtime_filter_params* p, dbx_runtime_filter** out) {
    const int k = prm.kind;
    if (k == DBX_JOIN_LEFT || k == DBX_JOIN_LEFT_ANTI || k == DBX_JOIN_FULL) {
      err.set("runtime filter: LEFT, LEFT ANTI and FULL joins keep every probe row, so no filter is built for them");
      return DBX_ERR_UNSUPPORTED;
    }
    if (!finished) { err.set("runtime filter before final_build"); return DBX_ERR_STATE; }
    if (p->in_probe && packed) { err.set("runtime filter: in_probe is built for single-key joins only (apply the filter to probe blocks instead)"); return DBX_ERR_UNSUPPORTED; }
    RfBuildKey keys[DBX_MAX_JOIN_KEYS];
    for (int i = 0; i < n_keys; ++i) {
      const GrowCol& g = build[key_build_col[i]];
      keys[i] = RfBuildKey{g.data.p, g.nullable ? (const uint8_t*)g.valid_bytes.p : nullptr, build_dtype[key_build_col[i]],
                           probe_dtype[key_probe_col[i]]};
    }
    std::shared_ptr<RfData> d;
    DBX_TRY(build_runtime_filter(err, stream, device, *p, keys, n_keys, build_rows, &d));
    drop_runtime_filter();
    if (p->in_probe && (d->parts[0].has_min_max || d->parts[0].has_bloom)) {
      rf_probe = d;
      d->in_probe = true;
    }
    *out = make_runtime_filter_handle(std::move(d));
    if (!*out) { drop_runtime_filter(); err.set("runtime filter: could not create the handle's stream"); return DBX_ERR_CUDA; }
    return DBX_OK;
  }
  void drop_runtime_filter() {
    if (rf_probe) rf_probe->in_probe = false;
    rf_probe.reset();
  }
  ~JoinOp() override { drop_runtime_filter(); }
  const char* kernel_variant() override { return rf_probe ? "precompiled kernels; runtime filter in the probe" : Op::kernel_variant(); }

  int32_t reset() override {
    drop_runtime_filter();
    build_rows = 0;
    final_probed = false;  // the matched map is cleared by the next final_build
    outputs.clear();
    next_out = 0;
    return DBX_OK;
  }
};

Op* make_join_op(const dbx_join_params* p, const int32_t* types, int32_t n, int device, int32_t* st) {
  auto* op = new JoinOp();
  *st = op->init(p, types, n, device);
  if (*st != DBX_OK) { g_create_error.set(op->err.msg); delete op; return nullptr; }
  return op;
}

}  // namespace dbx

using namespace dbx;

extern "C" int32_t dbx_op_create_join(const dbx_join_params* params, const int32_t* input_types, int32_t n_input_cols,
                                      const dbx_expr* other_predicate, int32_t device, dbx_op** out) {
  if (!out || !params || !input_types) { g_create_error.set("dbx_op_create_join: null argument"); return DBX_ERR_INVALID; }
  *out = nullptr;
  int32_t ndev = 0;
  DBX_TRY(dbx_device_count(&ndev));
  if (device < 0 || device >= ndev) { g_create_error.set("dbx_op_create: device index out of range"); return DBX_ERR_INVALID; }
  int32_t st = DBX_OK;
  Op* op = make_join_op(params, input_types, n_input_cols, device, &st);
  if (!op) return st == DBX_OK ? DBX_ERR_INVALID : st;
  st = static_cast<JoinOp*>(op)->set_residual(other_predicate);
  if (st != DBX_OK) { g_create_error.set(op->err.msg); delete op; return st; }
  op->kind = DBX_OP_JOIN;
  *out = reinterpret_cast<dbx_op*>(op);
  return DBX_OK;
}

extern "C" int32_t dbx_join_probe(dbx_op* op, const dbx_block* block) {
  if (!op || !block) return DBX_ERR_INVALID;
  Op* o = reinterpret_cast<Op*>(op);
  if (o->kind != DBX_OP_JOIN) { o->err.set("dbx_join_probe: not a join operator"); return DBX_ERR_INVALID; }
  DBX_CUDA_TRY(o->err, cudaSetDevice(o->device));
  return static_cast<JoinOp*>(o)->probe(block);
}

extern "C" int32_t dbx_join_final_probe(dbx_op* op) {
  if (!op) return DBX_ERR_INVALID;
  Op* o = reinterpret_cast<Op*>(op);
  if (o->kind != DBX_OP_JOIN) { o->err.set("dbx_join_final_probe: not a join operator"); return DBX_ERR_INVALID; }
  DBX_CUDA_TRY(o->err, cudaSetDevice(o->device));
  return static_cast<JoinOp*>(o)->final_probe();
}

extern "C" int32_t dbx_join_runtime_filter(dbx_op* op, const dbx_runtime_filter_params* params, dbx_runtime_filter** out) {
  if (!op || !params || !out) { g_create_error.set("dbx_join_runtime_filter: null argument"); return DBX_ERR_INVALID; }
  *out = nullptr;
  Op* o = reinterpret_cast<Op*>(op);
  if (o->kind != DBX_OP_JOIN) { o->err.set("dbx_join_runtime_filter: not a join operator"); g_create_error.set(o->err.msg); return DBX_ERR_INVALID; }
  DBX_CUDA_TRY(o->err, cudaSetDevice(o->device));
  const int32_t st = static_cast<JoinOp*>(o)->runtime_filter(params, out);
  if (st != DBX_OK) g_create_error.set(o->err.msg);
  return st;
}
