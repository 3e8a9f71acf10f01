// plan.h — host-normalised, device-consumable description of a fused
// [TransformFilter ->] TransformPartialAggregate step.  Built once per operator from
// dbx_agg_params / dbx_predicate (include/dbx.h), passed BY VALUE to the kernels.
#pragma once
#include "common.cuh"
#include "eval_kernels.cuh"

namespace dbx {

constexpr int kMaxSlots = 8;    // distinct input columns one kernel reads
constexpr int kMaxUpdates = 16; // state-word updates per passing row
constexpr int kMaxWords = 15;   // state words per group (entry = key + words)
constexpr int kMaxComputed = DBX_MAX_COMPUTED_COLS;  // computed columns one operator evaluates
constexpr int kMaxCompNodes = 32;                    // postfix nodes of all its computed columns together

// x % d for a runtime-constant divisor without a hardware divide: Granlund–Montgomery
// round-up method (N = 64):  m' = floor(2^64 (2^l - d) / d) + 1,
//   t = mulhi(m', n);  q = (t + ((n - t) >> sh1)) >> sh2;  r = n - q d.
// The reference strength-reduces the same way for unsigned divisors
// (arithmetic_modulo.rs:119-147, crate strength_reduce); signed operands go through |x|, |d|
// and take the sign of the dividend (Rust `%` truncates), MIN % -1 = 0 falls out (|d| = 1).
struct ModMagic {
  uint64_t d;   // |divisor|
  uint64_t m;   // m'
  int32_t sh1, sh2;
};

#ifndef DBX_DEVICE_ONLY
inline ModMagic make_mod_magic(uint64_t d) {
  ModMagic mm;
  mm.d = d;
  int l = 0;
  while (l < 64 && ((unsigned __int128)1 << l) < (unsigned __int128)d) ++l;  // l = ceil(log2 d)
  unsigned __int128 num = (((unsigned __int128)1 << l) - d) << 64;
  mm.m = (uint64_t)(num / d) + 1;
  mm.sh1 = l < 1 ? l : 1;
  mm.sh2 = l - 1 > 0 ? l - 1 : 0;
  return mm;
}
#endif

__host__ __device__ __forceinline__ uint64_t mulhi_u64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
__host__ __device__ __forceinline__ uint64_t umod_magic(uint64_t n, const ModMagic& mm) {
  uint64_t t = mulhi_u64(mm.m, n);
  uint64_t q = (t + ((n - t) >> mm.sh1)) >> mm.sh2;
  return n - q * mm.d;
}
__host__ __device__ __forceinline__ int64_t smod_magic(int64_t x, const ModMagic& mm) {
  uint64_t ux = x < 0 ? (uint64_t)0 - (uint64_t)x : (uint64_t)x;
  uint64_t r = umod_magic(ux, mm);
  return x < 0 ? -(int64_t)r : (int64_t)r;
}

// Exact divisibility test  d | n  without computing the remainder (Granlund–Montgomery /
// Hacker's Delight 10-17): with d = d' 2^k, d' odd and inv = d'^-1 mod 2^64,
//   d | n  <=>  rotr(n * inv, k) <= floor((2^64 - 1) / d).
// Used for `x % d = 0` / `x % d <> 0`, the shape the configs filter on.
#ifndef DBX_DEVICE_ONLY
inline ModMagic make_div_magic(uint64_t d) {
  ModMagic mm;
  int k = 0;
  uint64_t dp = d;
  while ((dp & 1) == 0) { dp >>= 1; ++k; }
  uint64_t inv = dp;  // correct to 3 bits; each Newton step doubles the precision
  for (int i = 0; i < 6; ++i) inv *= 2 - dp * inv;
  mm.m = inv;
  mm.sh1 = k;
  mm.sh2 = 0;
  mm.d = ~0ULL / d;
  return mm;
}
#endif
__host__ __device__ __forceinline__ bool divisible_magic(uint64_t n, const ModMagic& mm) {
  uint64_t q = n * mm.m;
  q = (q >> mm.sh1) | (mm.sh1 ? (q << (64 - mm.sh1)) : 0);
  return q <= mm.d;
}

// One flattened SelectExpr node (postfix).  CMP: lhs = slot (optional modulo), rhs = const or slot.
struct PredNodeDev {
  int32_t kind;        // dbx_pred_kind
  int32_t cmp;         // dbx_cmp_op
  int32_t n_children;  // AND / OR
  int32_t value;       // CONST value / BOOLCOL slot
  int32_t cls;         // comparison class (ValClass) after widening
  int32_t l_slot;
  int32_t l_mod;       // 1: lhs = slot % mod; 2: divisibility test (slot % d  =/<>  0), mod = make_div_magic(d)
  int32_t r_slot;      // -1: rhs is r_const
  uint64_t r_const;    // bits in class `cls`
  double mod_f;        // FLT modulo divisor
  ModMagic mod;
};

enum UpdOp : int32_t {
  UPD_INC = 0,        // word += 1                      (row count / count(*))
  UPD_INC_VALID = 1,  // word += 1 if slot valid        (count(col), OrNull flag of a nullable arg)
  UPD_ADD_INT = 2,    // word += value (two's complement wrapping == i64/u64 wrapping add)
  UPD_ADD_F64 = 3,    // word(f64) += value
  UPD_MIN_S64 = 4, UPD_MAX_S64 = 5, UPD_MIN_U64 = 6, UPD_MAX_U64 = 7,
  UPD_MIN_F64 = 8, UPD_MAX_F64 = 9  // on the order-preserving u64 image of the double
};
struct UpdateDev {
  int32_t op;
  int32_t slot;  // input slot (unused for UPD_INC)
  int32_t word;  // state word index
  int32_t pad;
};

// Device hash table of groups.
//   keys[cap + 2]              cap = 4 * n_buckets (power of two); a bucket is 4 consecutive keys =
//                              one 32-byte sector, probed with ONE 256-bit load; bucket of a key =
//                              agg_hash(key) & (n_buckets - 1), linear probing over buckets;
//                              keys[cap] / keys[cap + 1] are 0/1 "present" flags of the two special
//                              groups: the key equal to the EMPTY sentinel, and the NULL key;
//   states[(cap + 2) * n_words] row-major: state word w of slot i at states[i * n_words + w], so the
//                              REDs of one row fall into one or two sectors
constexpr uint64_t kEmptyKey = 0x8000000000000000ULL;
struct TableDev {
  uint64_t* keys;
  uint64_t* states;
  int64_t cap;
  int32_t n_words;
  int32_t probe_limit;             // buckets examined before a row is sent to the overflow list
  int32_t key_words;               // 1: 64-bit keys, buckets of 4; 2: 128-bit packed keys (HashMethodKeysU128,
                                   // kernels/group_by.rs:66-79): keys[2 i], keys[2 i + 1], buckets of 2 = one sector
  unsigned long long* n_groups;    // device counter: groups inserted so far
  unsigned long long* n_overflow;  // device counter
  uint32_t* overflow_rows;         // rows that could not be placed (nullptr: provably not needed)
  // groups of a CTA's hot-group cache that could not be placed when the cache was merged (table full):
  // exchange-format rows [key][0][words...], merged by the host after the table has grown
  uint64_t* hot_spill;             // nullptr: a failed merge is counted in n_overflow (cannot happen below the load-factor budget)
  unsigned long long* n_hot_spill;
  unsigned long long* n_hot_rows;  // rows the hot-group caches absorbed (the host turns the cache off when it absorbs next to nothing)
};

__host__ __device__ __forceinline__ uint64_t* word_ptr(const TableDev& t, int64_t slot, int w) {
  return t.states + slot * t.n_words + w;
}

// Multi-column GROUP BY packed into one 64-bit key (the reference's HashMethodKeysU64 idea,
// kernels/group_by.rs:66-79: fixed-size key columns whose bytes + NULL flags fit one word):
// column j contributes (value & mask) << shift, a nullable column additionally one NULL bit; a
// NULL value contributes zero value bits, so (NULL, x) and (0, x) stay different groups.
struct KeyPartDev {
  int32_t slot;        // input slot of the column
  int32_t shift;       // bit position of the value field (0..127: word = shift >> 6; a field never straddles words)
  int32_t null_shift;  // bit position of the NULL flag (same word as the value), -1: column is not Nullable
  int32_t dtype;
  uint64_t mask;       // value field mask (unshifted)
};

struct AggKernelParams {
  DevCol cols[kMaxSlots];
  PredNodeDev nodes[DBX_MAX_PRED_NODES];
  UpdateDev upd[kMaxUpdates];
  KeyPartDev key_parts[DBX_MAX_GROUP_COLS];
  TableDev table;
  int64_t n_rows;
  const uint32_t* row_index;  // indirect mode: process rows row_index[0..n_rows)
  unsigned long long* single_state;  // ungrouped: word array accumulated with one atomic per CTA
  int32_t n_slots, n_nodes, n_updates;
  int32_t key_slot;     // -1: no GROUP BY
  int32_t key_nullable; // key column may carry a validity bitmap
  int32_t n_key_parts;  // > 1: the key is packed from key_parts[] (key_slot is unused)
  int32_t key_is_float; // 1: the (single) key is a float column: every NaN is one group (group_hash.rs:599-619)
  uint32_t row_base;    // added to in-launch row numbers when recording overflow rows
  int32_t debug_flags;  // perf bisecting only (env DBX_AGG_DEBUG): 1 = skip state updates, 2 = skip table probe
  int32_t hot_cache;                // 1: per-CTA shared-memory cache of hot groups (skewed keys), flushed at kernel end
  // computed columns (kept behind every field above, so plans without them see the same layout):
  // comp[0, comp_pred) feed the predicate and are evaluated before it, comp[comp_pred, n_comp) after it
  int32_t n_comp, comp_pred;
  uint32_t fresh_slots;             // slots that hold a computed value only (no input column is loaded into them)
  int32_t pad_comp;
  CompDev comp[kMaxComputed];
  NodeDev cnodes[kMaxCompNodes];
  int64_t expr_row0;                // number (since create / reset) of the row this launch's row 0 stands for
  unsigned long long* expr_err;     // min over failing selected rows of (row << 8 | code); nullptr: the plan cannot raise
};

// The plan fields the fused kernels read per row, as ONE constexpr object: a run-time specialised
// build (agg_jit.cu) emits `__device__ constexpr StaticPlan jit_plan = {...}` from the operator's
// plan, and agg_kernels.cuh reads `jit_plan.f` where the precompiled kernels read `p.f`.
struct StaticPlan {
  int32_t n_nodes, n_updates, key_slot, key_is_float, n_key_parts, debug_flags, n_words, hot_cache;
  PredNodeDev nodes[DBX_MAX_PRED_NODES];
  UpdateDev upd[kMaxUpdates];
  KeyPartDev key_parts[DBX_MAX_GROUP_COLS];
  // computed columns, last: agg_jit_plan_text writes them only when there are some, so the text of every
  // other plan (and the kernel compiled from it) does not change
  int32_t n_comp, comp_pred;
  uint32_t fresh_slots;
  int32_t raises;                   // 1: a computed column after the predicate can raise (errors are recorded)
  CompDev comp[kMaxComputed];
  NodeDev cnodes[kMaxCompNodes];
};

}  // namespace dbx
