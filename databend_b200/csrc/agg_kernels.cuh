// agg_kernels.cuh — fused [filter ->] hash-aggregate kernels for sm_90a.
//
// Replaces, for one pushed DataBlock, the reference's per-block chain
//   TransformFilter (FilterExecutor::select + take)           filter_executor.rs:82-160
//   -> AggregateHashTable::add_groups                         aggregate_hashtable.rs:168-292
//        group_hash_entries / HashIndex::probe_and_create     group_hash.rs:40, hash_index/index.rs:148-214
//        accumulate_keys for sum / count / avg / min / max    aggregate_sum.rs:106-111, aggregate_count.rs:123-157,
//                                                             aggregate_avg.rs:75-80
// with ONE pass over HBM: each input column is read exactly once with 256-bit streaming
// loads (evict-first), the predicate is evaluated in registers, and surviving rows update an
// L2-resident hash table with fire-and-forget `red.global` atomics.
//
// HBM-bound integer work: no tensor cores; the levers are coalescing, bytes in flight,
// keeping the table in L2, and keeping every lane busy in the table phase.
//
// Table layout (see TableDev in plan.h): like the reference's HashIndex (8 ctrl bytes per
// group probed with one SIMD compare, hash_index/group.rs:24-55) the keys are probed a group
// at a time — here a bucket of four 64-bit keys = one 32-byte sector = one 256-bit load.
#pragma once
#include "plan.h"

namespace dbx {

// Plan access.  The precompiled kernels read the plan from the by-value kernel parameters
// (constant bank).  A run-time specialised build (agg_jit.cu: NVRTC, one compilation per plan
// shape) defines DBX_JIT and a `__device__ constexpr StaticPlan jit_plan` before including this
// header: every plan field then is a compile-time constant, the update / predicate loops unroll and
// the per-row interpretation (op if-chains, slot selects, runtime-shift rotates) folds away.
// Computed columns: the precompiled kernels take them through a template flag (EXPR), so that the
// instantiations serving plans without them stay as they were; a specialised build knows from the plan.
#ifdef DBX_JIT
#define PLN(f) (jit_plan.f)
#define PLN_TABLE(f) (jit_plan.f)
#define PLN_UNROLL _Pragma("unroll")
#define PLN_COMP(EXPR) (jit_plan.n_comp > 0)
#define PLN_RAISES (jit_plan.raises != 0)
#else
#define PLN(f) (p.f)
#define PLN_TABLE(f) (p.table.f)
#define PLN_UNROLL
#define PLN_COMP(EXPR) (EXPR)
#define PLN_RAISES (p.expr_err != nullptr)
#endif

constexpr int kBlock = 256;       // threads per CTA
constexpr int kRowsPerThread = 4; // one 256-bit load per 8-byte column per tile
constexpr int kTileRows = kBlock * kRowsPerThread;
constexpr int kWarpsPerBlock = kBlock / 32;
constexpr int kStageCap = 160;    // staged rows per warp: up to 31 carried over + 128 new

struct RowVals {
  uint64_t v[kRowsPerThread];
};

// ---------------------------------------------------------------- column tile loads
template <typename T>
__device__ __forceinline__ uint64_t widen(T x);
template <> __device__ __forceinline__ uint64_t widen<int8_t>(int8_t x) { return (uint64_t)(int64_t)x; }
template <> __device__ __forceinline__ uint64_t widen<int16_t>(int16_t x) { return (uint64_t)(int64_t)x; }
template <> __device__ __forceinline__ uint64_t widen<int32_t>(int32_t x) { return (uint64_t)(int64_t)x; }
template <> __device__ __forceinline__ uint64_t widen<uint8_t>(uint8_t x) { return x; }
template <> __device__ __forceinline__ uint64_t widen<uint16_t>(uint16_t x) { return x; }
template <> __device__ __forceinline__ uint64_t widen<uint32_t>(uint32_t x) { return x; }

__device__ __forceinline__ uint64_t f32_bits_to_f64_bits(uint32_t b) {
  return (uint64_t)__double_as_longlong((double)__uint_as_float(b));
}

// Row r of a tile belongs to thread (r / 4): each thread owns 4 consecutive rows, so an 8-byte
// column is one 256-bit load per thread and tile, a 4-byte column one 128-bit load.
template <bool INDIRECT>
__device__ __forceinline__ void load_slot(const DevCol& c, int64_t tile_base, int64_t n_rows, const uint32_t* row_index,
                                          uint64_t pol, RowVals& out, uint32_t& valid_mask) {
  valid_mask = 0xF;
  if (c.is_const) {
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) out.v[j] = c.const_bits;
    if (c.is_const == 2) valid_mask = 0;
    return;
  }
  const int64_t r0 = tile_base + (int64_t)kRowsPerThread * threadIdx.x;
  int64_t rows[kRowsPerThread];
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    int64_t r = r0 + j;
    if (INDIRECT) rows[j] = r < n_rows ? (int64_t)row_index[r] : -1;
    else rows[j] = r < n_rows ? r : -1;
  }
  const bool full = !INDIRECT && (r0 + kRowsPerThread <= n_rows);
  const char* base = (const char*)c.data;
  const int dt = c.dtype;
  if (dt == DBX_I64 || dt == DBX_U64 || dt == DBX_F64) {
    if (full && ((reinterpret_cast<uintptr_t>(base) & 31) == 0)) {
      u64x4 q = ld_stream_256(base + r0 * 8);
      out.v[0] = q.x; out.v[1] = q.y; out.v[2] = q.z; out.v[3] = q.w;
    } else {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) out.v[j] = rows[j] >= 0 ? ld_stream_u64(base + rows[j] * 8, pol) : 0;
    }
  } else if (dt == DBX_I32 || dt == DBX_U32 || dt == DBX_F32) {
    uint32_t w[kRowsPerThread];
    if (full && ((reinterpret_cast<uintptr_t>(base) & 15) == 0)) {
      uint4 q = ld_stream_128(base + r0 * 4, pol);
      w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w;
    } else {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) w[j] = rows[j] >= 0 ? ld_stream_u32(base + rows[j] * 4, pol) : 0;
    }
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
      out.v[j] = dt == DBX_I32 ? widen<int32_t>((int32_t)w[j]) : (dt == DBX_U32 ? (uint64_t)w[j] : f32_bits_to_f64_bits(w[j]));
  } else if (dt == DBX_I16 || dt == DBX_U16) {
    uint16_t w[kRowsPerThread];
    if (full && ((reinterpret_cast<uintptr_t>(base) & 7) == 0)) {
      uint64_t q = ld_stream_u64(base + r0 * 2, pol);
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) w[j] = (uint16_t)(q >> (16 * j));
    } else {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) w[j] = rows[j] >= 0 ? ld_stream_u16(base + rows[j] * 2, pol) : 0;
    }
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) out.v[j] = dt == DBX_I16 ? widen<int16_t>((int16_t)w[j]) : (uint64_t)w[j];
  } else if (dt == DBX_I8 || dt == DBX_U8) {
    uint8_t w[kRowsPerThread];
    if (full && ((reinterpret_cast<uintptr_t>(base) & 3) == 0)) {
      uint32_t q = ld_stream_u32(base + r0, pol);
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) w[j] = (uint8_t)(q >> (8 * j));
    } else {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) w[j] = rows[j] >= 0 ? ld_stream_u8(base + rows[j], pol) : 0;
    }
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) out.v[j] = dt == DBX_I8 ? widen<int8_t>((int8_t)w[j]) : (uint64_t)w[j];
  } else if (dt == DBX_BOOL) {
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
      out.v[j] = rows[j] >= 0 ? (uint64_t)bit_test((const uint8_t*)base, c.dbit_off + rows[j]) : 0;
  } else {
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) out.v[j] = 0;
  }
  if (c.validity) {
    uint32_t m = 0;
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
      if (rows[j] >= 0 && bit_test(c.validity, c.vbit_off + rows[j])) m |= 1u << j;
    valid_mask = m;
  }
}

template <int NS>
__device__ __forceinline__ uint64_t pick(const RowVals (&vals)[NS], int slot, int j) {
  uint64_t r = vals[0].v[j];
#pragma unroll
  for (int s = 1; s < NS; ++s)
    if (slot == s) r = vals[s].v[j];
  return r;
}
template <int NS>
__device__ __forceinline__ uint32_t pick_mask(const uint32_t (&m)[NS], int slot) {
  uint32_t r = m[0];
#pragma unroll
  for (int s = 1; s < NS; ++s)
    if (slot == s) r = m[s];
  return r;
}

// ---------------------------------------------------------------- computed columns
// One computed column's postfix program on one row: a value stack held in registers (push / pop shift
// them), COLUMN nodes read the row's slot values v[] / validity bits.  Returns the value (0 when NULL).
template <typename V>
__device__ __forceinline__ uint64_t comp_row(const CompDev& cd, const NodeDev* cnodes, const V& v, uint32_t valid, bool& ok, int& err) {
  uint64_t s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0, s5 = 0, s6 = 0, s7 = 0;
  bool n0 = false, n1 = false, n2 = false, n3 = false, n4 = false, n5 = false, n6 = false, n7 = false;
  PLN_UNROLL
  for (int i = cd.first; i < cd.first + cd.n_nodes; ++i) {
    const NodeDev nd = cnodes[i];
    if (nd.kind == DBX_EXPR_COLUMN || nd.kind == DBX_EXPR_CONST) {
      s7 = s6; s6 = s5; s5 = s4; s4 = s3; s3 = s2; s2 = s1; s1 = s0;
      n7 = n6; n6 = n5; n5 = n4; n4 = n3; n3 = n2; n2 = n1; n1 = n0;
      if (nd.kind == DBX_EXPR_COLUMN) { n0 = (valid >> nd.col) & 1; s0 = n0 ? v[nd.col] : 0; }
      else { n0 = !nd.c_null; s0 = n0 ? nd.c_bits : 0; }
    } else if (nd.kind == DBX_EXPR_CAST) {
      apply_cast(nd, s0, n0, err);
    } else if (nd.func == DBX_FN_NOT || nd.func == DBX_FN_NEGATE || nd.func == DBX_FN_IS_NULL || nd.func == DBX_FN_IS_NOT_NULL) {
      apply_unary(nd, s0, n0, err);
    } else {
      apply_binary(nd, s1, n1, s0, n0, err);  // s1 op s0 -> s1, then pop
      s0 = s1; s1 = s2; s2 = s3; s3 = s4; s4 = s5; s5 = s6; s6 = s7;
      n0 = n1; n1 = n2; n2 = n3; n3 = n4; n4 = n5; n5 = n6; n6 = n7;
    }
  }
  ok = n0;
  return n0 ? s0 : 0;
}
// The same for a program with IF / ASSUME_NOT_NULL (CompDev::branches) is comp_row_cond (eval_kernels.cuh).
#ifndef DBX_JIT
// The precompiled kernels share ONE out-of-line copy of the interpreter (inlined into every
// instantiation it would multiply their code and build time); a specialised build inlines comp_row
// with constexpr nodes, where it folds into straight-line code.  Under the 64-register bound of these
// kernels the call costs spills (DESIGN §4: computed columns); the specialised build has none of them.
// The out-of-line copy is the per-slot-flag form for every program: it gives the same values and errors
// as comp_row where both apply, and fewer spill bytes in its callers than comp_row or than both behind a
// branch.
struct SlotRow { uint64_t v[kMaxSlots]; };
struct CompOut { uint64_t v; int32_t ok, err; };
static __device__ __noinline__ CompOut comp_row_interp(const AggKernelParams& p, int c, const SlotRow row, uint32_t valid) {
  bool o = false;
  int e = 0;
  CompOut r;
  r.v = comp_row_cond(p.comp[c], p.cnodes, row.v, valid, o, e);
  r.ok = o;
  r.err = e;
  return r;
}
#endif

// Evaluates computed columns [c0, c1) on the thread's rows (EvalScalar between the filter and the
// aggregate, fused); the result replaces the value and validity of the column's slot.  A failing call is
// recorded only on rows of `record` (rows the predicate kept), as the first failing row since the
// operator's create / reset.
template <int NS, bool INDIRECT>
__device__ __forceinline__ void eval_computed(const AggKernelParams& p, int c0, int c1, RowVals (&vals)[NS], uint32_t (&vmask)[NS],
                                              uint32_t record, int64_t r0) {
  PLN_UNROLL
  for (int c = c0; c < c1; ++c) {
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      uint32_t valid = 0;
#pragma unroll
      for (int s = 0; s < NS; ++s) valid |= ((vmask[s] >> j) & 1u) << s;
      bool ok = false;
      int err = 0;
#ifdef DBX_JIT
      uint64_t v[NS];
#pragma unroll
      for (int s = 0; s < NS; ++s) v[s] = vals[s].v[j];
      const CompDev cd = PLN(comp[c]);
      const uint64_t out = cd.branches ? comp_row_cond(cd, jit_plan.cnodes, v, valid, ok, err) : comp_row(cd, jit_plan.cnodes, v, valid, ok, err);
#else
      SlotRow row;
#pragma unroll
      for (int s = 0; s < kMaxSlots; ++s) row.v[s] = s < NS ? vals[s].v[j] : 0;
      const CompOut co = comp_row_interp(p, c, row, valid);
      const uint64_t out = co.v;
      ok = co.ok != 0;
      err = co.err;
      const CompDev cd = p.comp[c];
#endif
      if (PLN_RAISES && err && ((record >> j) & 1)) {
        const int64_t row = p.expr_row0 + (INDIRECT ? (int64_t)p.row_index[r0 + j] : (int64_t)p.row_base + r0 + j);
        atomicMin(p.expr_err, ((unsigned long long)row << 8) | (unsigned long long)err);
      }
#pragma unroll
      for (int s = 0; s < NS; ++s)
        if (s == cd.slot) {
          vals[s].v[j] = out;
          vmask[s] = (vmask[s] & ~(1u << j)) | ((ok ? 1u : 0u) << j);
        }
    }
  }
}

// OrderedFloat compare (src/common/base/src/base/ordered_float.rs:147-201)
__device__ __forceinline__ int cmp_f64_ordered(double a, double b) {
  bool an = a != a, bn = b != b;
  if (an | bn) return an == bn ? 0 : (an ? 1 : -1);
  return a < b ? -1 : (a > b ? 1 : 0);
}

// ---------------------------------------------------------------- predicate
__device__ __forceinline__ bool apply_cmp(int op, int c) {
  // if-chain (uniform branches) rather than a jump table: keeps the kernel small and off BRX
  if (op == DBX_EQ) return c == 0;
  if (op == DBX_NE) return c != 0;
  if (op == DBX_LT) return c < 0;
  if (op == DBX_LE) return c <= 0;
  if (op == DBX_GT) return c > 0;
  return c >= 0;
}

// One Compare node on one row.  a/b are the 64-bit images of the operands in class nd.cls.
__device__ __forceinline__ bool eval_cmp(const PredNodeDev& nd, uint64_t a, uint64_t b) {
  if (nd.l_mod == 2) {  // `x % d (= | <>) 0` on integers: exact divisibility test, no remainder needed
    uint64_t ux = a;
    if (nd.cls == VC_INT && (int64_t)a < 0) ux = (uint64_t)0 - a;
    bool div = divisible_magic(ux, nd.mod);
    return nd.cmp == DBX_EQ ? div : !div;
  }
  int c;
  if (nd.cls == VC_INT) {
    int64_t x = (int64_t)a;
    if (nd.l_mod) x = smod_magic(x, nd.mod);
    int64_t y = (int64_t)b;
    c = x < y ? -1 : (x > y ? 1 : 0);
  } else if (nd.cls == VC_UINT) {
    uint64_t x = a;
    if (nd.l_mod) x = umod_magic(x, nd.mod);
    c = x < b ? -1 : (x > b ? 1 : 0);
  } else {
    double x = __longlong_as_double((long long)a);
    if (nd.l_mod) x = fmod(x, nd.mod_f);
    c = cmp_f64_ordered(x, __longlong_as_double((long long)b));
  }
  return apply_cmp(nd.cmp, c);
}

// Evaluates the flattened SelectExpr tree for the thread's kRowsPerThread rows; returns a
// bitmask of selected rows.  NULL operands make a Compare false (select_column_scalar.rs).
template <int NS>
__device__ __forceinline__ uint32_t eval_predicate(const AggKernelParams& p, const RowVals (&vals)[NS],
                                                   const uint32_t (&vmask)[NS], uint32_t in_range) {
  if (PLN(n_nodes) == 0) return in_range;
  uint32_t stack[kRowsPerThread];
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) stack[j] = 0;
  PLN_UNROLL
  for (int n = 0; n < PLN(n_nodes); ++n) {
    const PredNodeDev nd = PLN(nodes[n]);
    if (nd.kind == DBX_PRED_CMP) {
      uint32_t lm = pick_mask<NS>(vmask, nd.l_slot);
      uint32_t rm = nd.r_slot >= 0 ? pick_mask<NS>(vmask, nd.r_slot) : 0xF;
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) {
        uint64_t a = pick<NS>(vals, nd.l_slot, j);
        uint64_t b = nd.r_slot >= 0 ? pick<NS>(vals, nd.r_slot, j) : nd.r_const;
        bool r = eval_cmp(nd, a, b) && ((lm >> j) & 1) && ((rm >> j) & 1);
        stack[j] = (stack[j] << 1) | (r ? 1u : 0u);
      }
    } else if (nd.kind == DBX_PRED_AND || nd.kind == DBX_PRED_OR) {
      uint32_t k = (1u << nd.n_children) - 1;
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) {
        uint32_t top = stack[j] & k;
        uint32_t r = nd.kind == DBX_PRED_AND ? (top == k) : (top != 0);
        stack[j] = ((stack[j] >> nd.n_children) << 1) | r;
      }
    } else if (nd.kind == DBX_PRED_BOOLCOL) {
      uint32_t m = pick_mask<NS>(vmask, nd.value);
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) {
        uint32_t r = (pick<NS>(vals, nd.value, j) != 0) && ((m >> j) & 1);
        stack[j] = (stack[j] << 1) | r;
      }
    } else {
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) stack[j] = (stack[j] << 1) | (nd.value ? 1u : 0u);
    }
  }
  uint32_t sel = 0;
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) sel |= (stack[j] & 1u) << j;
  return sel & in_range;
}

// Float group keys (group_hash.rs:599-619, payload_row.rs match_column_type on OrderedFloat): rows
// group by the value's bit pattern, except that every NaN is ONE group (canonical NaN); -0.0 and
// +0.0 hash differently in the reference and are separate groups here too.
__device__ __forceinline__ uint64_t canonical_float_key(uint64_t bits) {
  const double d = __longlong_as_double((long long)bits);
  return d != d ? 0x7FF8000000000000ULL : bits;
}

// ---------------------------------------------------------------- table
// Coherent load of one 32-byte bucket (4 keys) as two 128-bit loads: goes to L2, the point of
// coherence of the CAS.
__device__ __forceinline__ u64x4 ld_bucket(const uint64_t* p) {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  u64x4 r;
  asm volatile("ld.global.relaxed.gpu.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(r.x), "=l"(r.y) : "l"(p), "l"(pol) : "memory");
  asm volatile("ld.global.relaxed.gpu.L2::cache_hint.v2.b64 {%0, %1}, [%2], %3;" : "=l"(r.z), "=l"(r.w) : "l"(p + 2), "l"(pol) : "memory");
  return r;
}
__device__ __forceinline__ int bucket_match(const u64x4& k, uint64_t key) {
  return k.x == key ? 0 : (k.y == key ? 1 : (k.z == key ? 2 : (k.w == key ? 3 : -1)));
}

// HashIndex::find_or_insert (hash_index/index.rs:92-111) past the first probe: walks buckets
// linearly; inserts into the first EMPTY position of the first non-full bucket with a CAS.
// Returns the slot, or -1 if the probe limit was hit (the row then goes to the overflow list).
__device__ __noinline__ int64_t find_or_insert_slow(const TableDev& t, uint64_t key, int64_t b, u64x4 kb,
                                                    uint32_t& new_groups) {
  const int64_t nb_mask = (t.cap >> 2) - 1;
  int probes = 0, retries = 0;
  while (probes < t.probe_limit) {
    int m = bucket_match(kb, key);
    if (m >= 0) return 4 * b + m;
    int e = kb.x == kEmptyKey ? 0 : (kb.y == kEmptyKey ? 1 : (kb.z == kEmptyKey ? 2 : (kb.w == kEmptyKey ? 3 : -1)));
    if (e >= 0 && retries < 64) {
      unsigned long long old = atomicCAS((unsigned long long*)(t.keys + 4 * b + e), (unsigned long long)kEmptyKey,
                                         (unsigned long long)key);
      if (old == kEmptyKey) { ++new_groups; return 4 * b + e; }
      if (old == key) return 4 * b + e;
      ++retries;  // lost the race to another key: look at this bucket again
      kb = ld_bucket(t.keys + 4 * b);
      continue;
    }
    b = (b + 1) & nb_mask;
    ++probes;
    retries = 0;
    kb = ld_bucket(t.keys + 4 * b);
  }
  return -1;
}

// ---- 128-bit packed keys: slot i holds keys[2 i], keys[2 i + 1]; a bucket is 2 slots = one 32-byte
// sector = one 256-bit probe; insertion is ONE 128-bit compare-and-swap (atom.cas.b128, sm_90+).
// The EMPTY pattern is both words == kEmptyKey; a real key equal to it lives in the special slot cap.
// (agg_hash_wide is in common.cuh: the join hashes its 128-bit keys with it too.)
__device__ __forceinline__ void cas_b128(uint64_t* addr, uint64_t c0, uint64_t c1, uint64_t v0, uint64_t v1, uint64_t& o0, uint64_t& o1) {
  asm volatile(
      "{\n\t"
      ".reg .b128 cmp, val, old;\n\t"
      "mov.b128 cmp, {%2, %3};\n\t"
      "mov.b128 val, {%4, %5};\n\t"
      "atom.global.relaxed.gpu.cas.b128 old, [%6], cmp, val;\n\t"
      "mov.b128 {%0, %1}, old;\n\t"
      "}"
      : "=l"(o0), "=l"(o1)
      : "l"(c0), "l"(c1), "l"(v0), "l"(v1), "l"(addr)
      : "memory");
}
__device__ __forceinline__ int bucket_match_wide(const u64x4& k, uint64_t k0, uint64_t k1) {
  return (k.x == k0 && k.y == k1) ? 0 : ((k.z == k0 && k.w == k1) ? 1 : -1);
}
__device__ __noinline__ int64_t find_or_insert_wide(const TableDev& t, uint64_t k0, uint64_t k1, int64_t b, u64x4 kb, uint32_t& new_groups) {
  const int64_t nb_mask = (t.cap >> 1) - 1;
  int probes = 0, retries = 0;
  while (probes < t.probe_limit) {
    const int m = bucket_match_wide(kb, k0, k1);
    if (m >= 0) return 2 * b + m;
    const int e = (kb.x == kEmptyKey && kb.y == kEmptyKey) ? 0 : ((kb.z == kEmptyKey && kb.w == kEmptyKey) ? 1 : -1);
    if (e >= 0 && retries < 64) {
      uint64_t o0, o1;
      cas_b128(t.keys + 4 * b + 2 * e, kEmptyKey, kEmptyKey, k0, k1, o0, o1);
      if (o0 == kEmptyKey && o1 == kEmptyKey) { ++new_groups; return 2 * b + e; }
      if (o0 == k0 && o1 == k1) return 2 * b + e;
      ++retries;
      kb = ld_bucket(t.keys + 4 * b);
      continue;
    }
    b = (b + 1) & nb_mask;
    ++probes;
    retries = 0;
    kb = ld_bucket(t.keys + 4 * b);
  }
  return -1;
}
__device__ __forceinline__ int64_t resolve_slot_wide(const TableDev& t, uint64_t k0, uint64_t k1, uint32_t& new_groups) {
  if (k0 == kEmptyKey && k1 == kEmptyKey) {  // the key equal to the EMPTY pattern: special slot cap, word 0 is its "present" flag
    if (atomicExch((unsigned long long*)(t.keys + 2 * t.cap), 1ULL) == kEmptyKey) ++new_groups;
    return t.cap;
  }
  const int64_t b = (int64_t)(agg_hash_wide(k0, k1) & (uint64_t)((t.cap >> 1) - 1));
  const u64x4 kb = ld_bucket(t.keys + 4 * b);
  const int m = bucket_match_wide(kb, k0, k1);
  return m >= 0 ? 2 * b + m : find_or_insert_wide(t, k0, k1, b, kb, new_groups);
}

__device__ __forceinline__ void apply_update(int op, void* w, uint64_t val, bool valid) {
  if (op == UPD_INC) { red_add_u64(w, 1); return; }
  if (!valid) return;
  if (op == UPD_ADD_INT) { red_add_u64(w, val); return; }
  if (op == UPD_ADD_F64) { red_add_f64(w, __longlong_as_double((long long)val)); return; }
  if (op == UPD_INC_VALID) { red_add_u64(w, 1); return; }
  if (op == UPD_MIN_S64) { red_min_s64(w, (int64_t)val); return; }
  if (op == UPD_MAX_S64) { red_max_s64(w, (int64_t)val); return; }
  if (op == UPD_MIN_U64) { red_min_u64(w, val); return; }
  if (op == UPD_MAX_U64) { red_max_u64(w, val); return; }
  if (op == UPD_MIN_F64) { red_min_u64(w, f64_to_ordered(__longlong_as_double((long long)val))); return; }
  red_max_u64(w, f64_to_ordered(__longlong_as_double((long long)val)));
}

// Slot of a special key: the key equal to the EMPTY sentinel lives at slot cap, the NULL key
// at slot cap + 1; keys[] there is a 0/1 "present" flag.
__device__ __forceinline__ int64_t special_slot(const TableDev& t, bool key_null, uint32_t& new_groups) {
  int64_t slot = t.cap + (key_null ? 1 : 0);
  if (atomicExch((unsigned long long*)(t.keys + slot), 1ULL) == kEmptyKey) ++new_groups;
  return slot;
}

// ---------------------------------------------------------------- fused kernel (GROUP BY)
// Per tile of 1024 rows (8 warps x 128 rows):
//   1. every input column is read once with 256-bit streaming loads (4 consecutive rows / thread);
//   2. the predicate is evaluated in registers;
//   3. each warp appends its surviving rows to a warp-private shared-memory stage with ballot
//      compaction (values of every slot, validity bits, row id);
//   4. whenever >= 32 rows are staged the warp runs the table phase on exactly 32 of them, one
//      per lane: hash -> one 256-bit bucket probe -> fire-and-forget RED per state word.
//      Leftovers (< 32) are carried to the next tile, so no lane idles on filtered-out rows.
// FAST: plain 8-byte device columns, no validity, 32 B aligned, whole tiles, at most one
// Compare: straight-line loads, and the next tile is prefetched into registers before the
// table phase so the HBM stream overlaps the L2 atomics.
template <int NS>
struct StageWarp {
  uint64_t val[NS][kStageCap];
  uint32_t row[kStageCap];
  uint8_t vm[kStageCap];
};

// ---- hot-group cache (skewed keys).  A few keys taking a large share of the rows serialise on the L2
// atomic unit of their state words (log-uniform keys over 1e6: 57 ms instead of 7.6 ms).  Each CTA
// therefore keeps kHotSlots groups in shared memory: a key may claim the slot its hash selects only
// when it occurs at least twice among the 32 rows its warp is working on (so uniformly distributed keys
// never claim, and pay one shared-memory load per row), rows of a cached key are accumulated with
// shared-memory atomics and touch neither the table nor L2, and the CTA merges its cache into the table
// once, at the end of the kernel.
constexpr int kHotSlots = 128;
constexpr int kHotWords = 8;  // plans with more state words run without the cache
constexpr size_t kHotBytes = (size_t)kHotSlots * (1 + kHotWords) * 8;
__device__ __forceinline__ uint64_t hot_identity(int op) {
  if (op == UPD_MIN_S64) return 0x7FFFFFFFFFFFFFFFULL;
  if (op == UPD_MAX_S64) return 0x8000000000000000ULL;
  if (op == UPD_MIN_U64 || op == UPD_MIN_F64) return ~0ULL;
  return 0;  // counters, sums (+0.0), unsigned / ordered-float maxima
}
// 64-bit add to a shared-memory word as native 32-bit shared atomics (a 64-bit shared atomicAdd is a
// compare-and-swap loop on sm_90): low half, then the high half plus the low half's carry.  The word is
// exact (mod 2^64) once every add has completed; nothing reads it in between.
__device__ __forceinline__ void smem_add_u64(uint64_t* w, uint64_t v) {
  unsigned int* h = reinterpret_cast<unsigned int*>(w);
  const unsigned int lo = (unsigned int)v, hi = (unsigned int)(v >> 32);
  const unsigned int old = atomicAdd(h, lo);
  const unsigned int up = hi + (old + lo < old ? 1u : 0u);
  if (up) atomicAdd(h + 1, up);
}
__device__ __forceinline__ void hot_update(int op, uint64_t* w, uint64_t val, bool valid) {
  if (op == UPD_INC) { smem_add_u64(w, 1); return; }
  if (!valid) return;
  if (op == UPD_ADD_INT) { smem_add_u64(w, val); return; }
  if (op == UPD_ADD_F64) { atomicAdd((double*)w, __longlong_as_double((long long)val)); return; }
  if (op == UPD_INC_VALID) { smem_add_u64(w, 1); return; }
  if (op == UPD_MIN_S64) { atomicMin((long long*)w, (long long)val); return; }
  if (op == UPD_MAX_S64) { atomicMax((long long*)w, (long long)val); return; }
  if (op == UPD_MIN_U64) { atomicMin((unsigned long long*)w, (unsigned long long)val); return; }
  if (op == UPD_MAX_U64) { atomicMax((unsigned long long*)w, (unsigned long long)val); return; }
  const unsigned long long o = f64_to_ordered(__longlong_as_double((long long)val));
  if (op == UPD_MIN_F64) atomicMin((unsigned long long*)w, o); else atomicMax((unsigned long long*)w, o);
}
__device__ __forceinline__ void hot_flush_word(int op, void* w, uint64_t v) {
  if (op == UPD_ADD_F64) { red_add_f64(w, __longlong_as_double((long long)v)); return; }
  if (op == UPD_MIN_S64) { red_min_s64(w, (int64_t)v); return; }
  if (op == UPD_MAX_S64) { red_max_s64(w, (int64_t)v); return; }
  if (op == UPD_MIN_U64 || op == UPD_MIN_F64) { red_min_u64(w, v); return; }
  if (op == UPD_MAX_U64 || op == UPD_MAX_F64) { red_max_u64(w, v); return; }
  red_add_u64(w, v);
}

template <int NS, bool FAST, int KW = 1>
__device__ __forceinline__ void table_phase32(const AggKernelParams& p, const StageWarp<NS>& sw, int first, int count,
                                              int lane, uint32_t& new_groups, uint64_t* hot = nullptr) {
  const TableDev& t = p.table;
  const int i = first + lane;
  const bool act = lane < count;
  uint64_t key = 0, key_hi = 0;
  uint32_t vm = 0xFF;
  bool key_null = false;
  if (act) {
    if (!FAST) vm = sw.vm[i];
    if (KW == 2) {  // 128-bit packed key: a field lives in word (shift >> 6)
      for (int j = 0; j < p.n_key_parts; ++j) {
        const KeyPartDev kp = p.key_parts[j];
        const bool ok = (vm >> kp.slot) & 1;
        const uint64_t bits = ok ? (sw.val[kp.slot][i] & kp.mask) << (kp.shift & 63) : 1ULL << (kp.null_shift & 63);
        if ((ok ? kp.shift : kp.null_shift) >> 6) key_hi |= bits; else key |= bits;
      }
    } else if (PLN(n_key_parts) > 1) {  // packed multi-column key; NULLs are encoded inside the key
      PLN_UNROLL
      for (int j = 0; j < PLN(n_key_parts); ++j) {
        const KeyPartDev kp = PLN(key_parts[j]);
        const bool ok = (vm >> kp.slot) & 1;
        if (ok) key |= (sw.val[kp.slot][i] & kp.mask) << kp.shift;
        else key |= 1ULL << kp.null_shift;
      }
    } else {
      key = sw.val[PLN(key_slot)][i];
      if (PLN(key_is_float)) key = canonical_float_key(key);
      key_null = !((vm >> PLN(key_slot)) & 1);
    }
  }
  const bool special = KW == 2 ? false : (key_null || key == kEmptyKey);
  const uint64_t hash = KW == 2 ? 0 : agg_hash_u64(key);
  const int64_t b = KW == 2 ? 0 : (int64_t)(hash & (uint64_t)((t.cap >> 2) - 1));
  bool cached = false;
  if (KW == 1 && hot) {
    const bool cand = act && !special;
    // idle lanes vote with throw-away values (a chance match only lets a key claim a slot a little earlier)
    const unsigned peers = __match_any_sync(0xffffffffu, cand ? key : (0x8000000000000001ULL + (uint64_t)lane));
    if (cand) {
      const int hs = (int)((hash >> 37) & (kHotSlots - 1));
      uint64_t ck = ((volatile uint64_t*)hot)[hs];
      if (ck == kEmptyKey && __popc(peers) >= 2) {
        const unsigned long long old = atomicCAS((unsigned long long*)(hot + hs), (unsigned long long)kEmptyKey, (unsigned long long)key);
        ck = old == kEmptyKey ? key : (uint64_t)old;
      }
      if (ck == key) {
        cached = true;
        uint64_t* hw = hot + kHotSlots + (size_t)hs * kHotWords;
        PLN_UNROLL
        for (int u = 0; u < PLN(n_updates); ++u) {
          const UpdateDev ud = PLN(upd[u]);
          hot_update(ud.op, hw + ud.word, sw.val[ud.slot][i], (vm >> ud.slot) & 1);
        }
      }
    }
  }
  u64x4 kb;
  kb.x = kb.y = kb.z = kb.w = 0;
  if (KW == 1 && act && !special && !cached) kb = ld_bucket(t.keys + 4 * b);
  if (act && !cached) {
    int64_t slot;
    if (KW == 2) {
      slot = resolve_slot_wide(t, key, key_hi, new_groups);
    } else if (special) {
      slot = special_slot(t, key_null, new_groups);
    } else {
      int m = bucket_match(kb, key);
      slot = m >= 0 ? 4 * b + m : find_or_insert_slow(t, key, b, kb, new_groups);
    }
    if (slot < 0) {
      unsigned long long idx = atomicAdd(t.n_overflow, 1ULL);
      if (t.overflow_rows) t.overflow_rows[idx] = sw.row[i];
    } else if (!(PLN(debug_flags) & 1)) {
      uint64_t* row = t.states + slot * PLN_TABLE(n_words);
      PLN_UNROLL
      for (int u = 0; u < PLN(n_updates); ++u) {
        const UpdateDev ud = PLN(upd[u]);
        apply_update(ud.op, row + ud.word, sw.val[ud.slot][i], (vm >> ud.slot) & 1);
      }
    }
  }
  __syncwarp();
}

template <int NS, bool EXPR = false>
__device__ __forceinline__ void prefetch_tile(const AggKernelParams& p, int64_t tile, RowVals (&vals)[NS]) {
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    if (PLN_COMP(EXPR) && ((PLN(fresh_slots) >> s) & 1)) continue;  // a computed column's own slot: nothing to load
    u64x4 q = ld_stream_256((const char*)p.cols[s].data + (tile * kTileRows + (int64_t)kRowsPerThread * threadIdx.x) * 8);
    vals[s].v[0] = q.x; vals[s].v[1] = q.y; vals[s].v[2] = q.z; vals[s].v[3] = q.w;
  }
}

template <int NS, bool FAST, bool INDIRECT, int KW = 1, bool EXPR = false>
__device__ __forceinline__ void filter_group_agg_body(const AggKernelParams& p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  StageWarp<NS>& sw = reinterpret_cast<StageWarp<NS>*>(smem_raw)[warp];
  // hot-group cache behind the row stages: [kHotSlots keys][kHotSlots x kHotWords state words]
  uint64_t* hot = nullptr;
  if (KW == 1 && PLN(hot_cache) && p.hot_cache) {  // plan capability (compile-time when specialised) and this launch's choice
    hot = reinterpret_cast<uint64_t*>(smem_raw + ((sizeof(StageWarp<NS>) * kWarpsPerBlock + 15) & ~(size_t)15));
    for (int e = threadIdx.x; e < kHotSlots; e += kBlock) {
      hot[e] = kEmptyKey;
      uint64_t* hw = hot + kHotSlots + (size_t)e * kHotWords;
      for (int w = 0; w < kHotWords; ++w) hw[w] = 0;
      PLN_UNROLL
      for (int u = 0; u < PLN(n_updates); ++u) { const UpdateDev ud = PLN(upd[u]); hw[ud.word] = hot_identity(ud.op); }
    }
    __syncthreads();
  }
  const int64_t n_tiles = FAST ? p.n_rows / kTileRows : (p.n_rows + kTileRows - 1) / kTileRows;
  const uint32_t lt_mask = (1u << lane) - 1;
  uint32_t new_groups = 0;
  const uint64_t pol = make_policy_evict_first();
  int n_staged = 0;  // warp-uniform

  RowVals vals[NS];
  uint32_t vmask[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) vmask[s] = 0xF;

  int64_t tile = blockIdx.x;
  if (FAST && tile < n_tiles) prefetch_tile<NS, EXPR>(p, tile, vals);
  for (; tile < n_tiles; tile += gridDim.x) {
    __syncwarp();  // lanes enter every tile together (diverged lanes would serialise the warp)
    const int64_t tile_base = tile * kTileRows;
    const int64_t r0 = tile_base + (int64_t)kRowsPerThread * threadIdx.x;
    uint32_t sel;
    if (FAST) {
      sel = 0xF;
      if (PLN_COMP(EXPR)) eval_computed<NS, INDIRECT>(p, 0, PLN(comp_pred), vals, vmask, 0, r0);
      if (PLN(n_nodes)) {
        const PredNodeDev nd = PLN(nodes[0]);
#pragma unroll
        for (int j = 0; j < kRowsPerThread; ++j)
          if (!eval_cmp(nd, pick<NS>(vals, nd.l_slot, j), nd.r_const)) sel &= ~(1u << j);
      }
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) load_slot<INDIRECT>(p.cols[s], tile_base, p.n_rows, p.row_index, pol, vals[s], vmask[s]);
      uint32_t in_range = 0;
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j)
        if (r0 + j < p.n_rows) in_range |= 1u << j;
      if (PLN_COMP(EXPR)) eval_computed<NS, INDIRECT>(p, 0, PLN(comp_pred), vals, vmask, 0, r0);
      sel = eval_predicate<NS>(p, vals, vmask, in_range);
    }
    if (PLN_COMP(EXPR)) eval_computed<NS, INDIRECT>(p, PLN(comp_pred), PLN(n_comp), vals, vmask, sel, r0);
    if (PLN(debug_flags) & 2) sel = 0;
    // ballot compaction: append the surviving rows behind the carried-over ones
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      const bool on = (sel >> j) & 1;
      const uint32_t bal = __ballot_sync(0xffffffffu, on);
      if (on) {
        const int o = n_staged + __popc(bal & lt_mask);
        uint32_t m = 0;
#pragma unroll
        for (int s = 0; s < NS; ++s) {
          sw.val[s][o] = vals[s].v[j];
          if (!FAST) m |= ((vmask[s] >> j) & 1u) << s;
        }
        if (!FAST) sw.vm[o] = (uint8_t)m;
        sw.row[o] = INDIRECT ? p.row_index[r0 + j] : (uint32_t)(r0 + j) + p.row_base;
      }
      n_staged += __popc(bal);
    }
    if (FAST) {  // prefetch the next tile: the loads fly while this warp works on the table
      const int64_t nt = tile + gridDim.x;
      if (nt < n_tiles) prefetch_tile<NS, EXPR>(p, nt, vals);
    }
    __syncwarp();
    while (n_staged >= 32) {
      n_staged -= 32;
      table_phase32<NS, FAST, KW>(p, sw, n_staged, 32, lane, new_groups, hot);
    }
  }
  __syncwarp();
  if (n_staged > 0) table_phase32<NS, FAST, KW>(p, sw, 0, n_staged, lane, new_groups, hot);
  if (hot) {  // merge this CTA's cached groups into the table: one find-or-insert and one RED per word and group
    __syncthreads();
    for (int e = threadIdx.x; e < kHotSlots; e += kBlock) {
      const uint64_t key = hot[e];
      if (key == kEmptyKey) continue;
      const TableDev& t = p.table;
      const int64_t b = (int64_t)(agg_hash_u64(key) & (uint64_t)((t.cap >> 2) - 1));
      const u64x4 kb = ld_bucket(t.keys + 4 * b);
      const int m = bucket_match(kb, key);
      const int64_t slot = m >= 0 ? 4 * b + m : find_or_insert_slow(t, key, b, kb, new_groups);
      const uint64_t* hw = hot + kHotSlots + (size_t)e * kHotWords;
      atomicAdd(t.n_hot_rows, (unsigned long long)hw[0]);  // word 0 = rows of the group
      if (slot < 0) {  // table full: hand the group to the host, which merges it after growing the table
        if (!t.hot_spill) { atomicAdd(t.n_overflow, 1ULL); continue; }
        uint64_t* row = t.hot_spill + atomicAdd(t.n_hot_spill, 1ULL) * (unsigned long long)(2 + t.n_words);
        row[0] = key; row[1] = 0;
        for (int w = 0; w < t.n_words; ++w) row[2 + w] = hw[w];
        continue;
      }
      PLN_UNROLL
      for (int u = 0; u < PLN(n_updates); ++u) {
        const UpdateDev ud = PLN(upd[u]);
        hot_flush_word(ud.op, word_ptr(t, slot, ud.word), hw[ud.word]);
      }
    }
  }
  // one counter update per warp
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) new_groups += __shfl_xor_sync(0xffffffffu, new_groups, o);
  if (lane == 0 && new_groups) atomicAdd(p.table.n_groups, (unsigned long long)new_groups);
}

#ifndef DBX_JIT
// (4 CTAs/SM at 62 registers: 5-6 CTAs spill and queue up behind the L2 atomics, 2-3 CTAs hide less latency)
template <int NS, bool FAST, bool INDIRECT, bool EXPR = false>
__global__ void __launch_bounds__(kBlock, 4) filter_group_agg_kernel(const __grid_constant__ AggKernelParams p) {
  filter_group_agg_body<NS, FAST, INDIRECT, 1, EXPR>(p);
}
// 128-bit packed group keys (two key words per slot): any column layout, direct or replayed rows
template <int NS, bool INDIRECT, bool EXPR = false>
__global__ void __launch_bounds__(kBlock, 4) filter_group_agg_wide_kernel(const __grid_constant__ AggKernelParams p) {
  filter_group_agg_body<NS, false, INDIRECT, 2, EXPR>(p);
}
#endif

// ---------------------------------------------------------------- pass 1 of the partitioned aggregation
// Tables larger than L2 (>= ~1.5e6 groups of configs[1]'s shape) turn every reduction into a DRAM
// round trip (2e6 / 1e7 keys: 28 / 44 ms per 1e9 rows instead of 7.6).  For those the operator makes
// two passes (SURVEY 3.1's fallback): this kernel filters the rows and scatters the survivors'
// slot values into P partitions by TABLE SLICE — slice = the top bits of the row's bucket index —
// and pass 2 aggregates each partition against its slice of the table only (slice_agg_kernel: the
// slice in shared memory; tables with too many slices for that: the fused kernel with the slice held
// in L2).  The table, the final merge and the exchange are unchanged; only the order in which rows
// reach the table differs.
//
// With hundreds of partitions a 1024-row tile has less than one surviving row per partition, so a CTA
// collects the survivors of several tiles in shared memory (unsorted, each tagged with its partition
// and its rank inside the partition) before it reserves one run per non-empty partition with one
// global atomic each and copies the rows out in partition order: consecutive threads store
// consecutive addresses of a run, and runs of one partition from different CTAs are reserved next to
// each other, so L2 completes the sectors before they reach DRAM.
constexpr int kMaxPartitions = 1024;
struct PartitionOut {
  uint64_t* out[kMaxSlots];       // per slot: [P][cap_p] 64-bit images
  unsigned long long* counts;     // [P] rows written per partition; [P] = overflow flag
  int64_t cap_p;
  uint64_t nb_mask;               // (cap >> 2) - 1
  int32_t region_shift;           // partition = (hash & nb_mask) >> region_shift
  int32_t n_parts;
};
// survivors a CTA collects before it copies them out (about 100 KB of shared memory: two CTAs per SM)
template <int NS>
__host__ __device__ constexpr int partition_stash_rows() { return NS <= 3 ? 3072 : (NS <= 5 ? 2048 : 1024); }
template <int NS>
__host__ __device__ constexpr size_t partition_smem_bytes() { return (size_t)partition_stash_rows<NS>() * (8 * NS + 4 + 2); }

// GROUP BY key of row j of a thread's tile, for rows without validity (the partitioned path only
// takes columns without NULLs, so a packed key never carries a NULL flag)
template <int NS>
__device__ __forceinline__ uint64_t plain_row_key(const AggKernelParams& p, const RowVals (&vals)[NS], int j) {
  uint64_t key = 0;
  if (PLN(n_key_parts) > 1) {
    PLN_UNROLL
    for (int k = 0; k < PLN(n_key_parts); ++k) { const KeyPartDev kp = PLN(key_parts[k]); key |= (pick<NS>(vals, kp.slot, j) & kp.mask) << kp.shift; }
  } else {
    key = pick<NS>(vals, PLN(key_slot), j);
    if (PLN(key_is_float)) key = canonical_float_key(key);
  }
  return key;
}

// Barrier `BAR` over the kBlock threads 0 .. kBlock - 1: barrier 0 is __syncthreads; the ring variant of pass 1
// synchronises its consumer threads on barrier 1, which its producer warp never joins.
template <int BAR>
__device__ __forceinline__ void block_sync() {
  if (BAR == 0) __syncthreads();
  else asm volatile("bar.sync %0, %1;" ::"n"(BAR), "n"(kBlock) : "memory");
}

// exclusive prefix sum of cnt[0, n) into off[0, n) by threads 0 .. kBlock - 1, n <= 4 * kBlock; ends with
// those threads synchronised on barrier BAR
static_assert(kMaxPartitions <= 4 * kBlock, "block_exclusive_scan: four counts per thread");
template <int BAR = 0>
__device__ __forceinline__ void block_exclusive_scan(const unsigned int* cnt, unsigned int* off, int n) {
  __shared__ unsigned int s_warp[kWarpsPerBlock];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = (n + kBlock - 1) / kBlock;
  unsigned int loc[4], sum = 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = threadIdx.x * per + q;
    loc[q] = (q < per && i < n) ? cnt[i] : 0u;
    sum += loc[q];
  }
  unsigned int inc = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) s_warp[warp] = inc;
  block_sync<BAR>();
  unsigned int ex = inc - sum;
  for (int w = 0; w < warp; ++w) ex += s_warp[w];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = threadIdx.x * per + q;
    if (q < per && i < n) off[i] = ex;
    ex += loc[q];
  }
  block_sync<BAR>();
}

// Filters the thread's rows of one tile (vals / vmask: the tile's slot values, loaded by the caller), tags each
// survivor with its partition and its rank inside the partition, and appends the survivors to the stash:
// warps in order, rows of a warp in ballot order.  Threads 0 .. kBlock - 1 take part, synchronised on barrier BAR.
template <int NS, bool EXPR, int R, int BAR>
__device__ __forceinline__ void partition_stash_tile(const AggKernelParams& p, const PartitionOut& po, RowVals (&vals)[NS], uint32_t (&vmask)[NS],
                                                     int64_t tile_base, uint64_t* stash, uint32_t* tag, unsigned int* s_cnt,
                                                     unsigned int (&s_wcnt)[2][kWarpsPerBlock], int& n_stash, int& parity) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t lt_mask = (1u << lane) - 1;
  const int64_t r0 = tile_base + (int64_t)kRowsPerThread * threadIdx.x;
  uint32_t in_range = 0;
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j)
    if (r0 + j < p.n_rows) in_range |= 1u << j;
  // computed values are stashed with the inputs: pass 2 reads them and evaluates nothing
  if (PLN_COMP(EXPR)) eval_computed<NS, false>(p, 0, PLN(comp_pred), vals, vmask, 0, r0);
  const uint32_t sel = eval_predicate<NS>(p, vals, vmask, in_range);
  if (PLN_COMP(EXPR)) eval_computed<NS, false>(p, PLN(comp_pred), PLN(n_comp), vals, vmask, sel, r0);
  uint32_t tg[kRowsPerThread], bal[kRowsPerThread];
  int warp_n = 0;
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    tg[j] = 0;
    if ((sel >> j) & 1) {
      const uint64_t key = plain_row_key<NS>(p, vals, j);
      const int part = key == kEmptyKey ? 0 : (int)((agg_hash_u64(key) & po.nb_mask) >> po.region_shift);
      tg[j] = ((uint32_t)part << 16) | atomicAdd(&s_cnt[part], 1u);
    }
    bal[j] = __ballot_sync(0xffffffffu, (sel >> j) & 1);
    warp_n += __popc(bal[j]);
  }
  // s_wcnt alternates between two buffers, so a warp that runs ahead into the next tile never overwrites
  // counts still being read
  if (lane == 0) s_wcnt[parity][warp] = warp_n;
  block_sync<BAR>();
  int pos = n_stash, total = 0;
  for (int w = 0; w < kWarpsPerBlock; ++w) {
    const int c = s_wcnt[parity][w];
    if (w < warp) pos += c;
    total += c;
  }
  parity ^= 1;
#pragma unroll
  for (int j = 0; j < kRowsPerThread; ++j) {
    if ((sel >> j) & 1) {
      const int i = pos + __popc(bal[j] & lt_mask);
#pragma unroll
      for (int s = 0; s < NS; ++s) stash[(size_t)s * R + i] = vals[s].v[j];
      tag[i] = tg[j];
    }
    pos += __popc(bal[j]);
  }
  n_stash += total;
}

// Copies the n_stash collected survivors out in partition order: one global reservation per non-empty
// partition, then consecutive threads store consecutive rows of a run.  Empties the stash and the counts.
template <int NS, int R, int BAR>
__device__ __forceinline__ void partition_copy_out(const PartitionOut& po, const uint64_t* stash, const uint32_t* tag, uint16_t* perm,
                                                   unsigned int* s_cnt, unsigned int* s_off, unsigned long long* s_base, int& n_stash) {
  block_sync<BAR>();
  block_exclusive_scan<BAR>(s_cnt, s_off, po.n_parts);
  for (int r = threadIdx.x; r < po.n_parts; r += kBlock) {
    const unsigned int c = s_cnt[r];
    s_base[r] = c ? atomicAdd(&po.counts[r], (unsigned long long)c) : 0ULL;
  }
  for (int i = threadIdx.x; i < n_stash; i += kBlock) perm[s_off[tag[i] >> 16] + (tag[i] & 0xFFFF)] = (uint16_t)i;
  block_sync<BAR>();
  for (int li = threadIdx.x; li < n_stash; li += kBlock) {
    const int i = perm[li];
    const uint32_t part = tag[i] >> 16;
    const unsigned long long at = s_base[part] + (tag[i] & 0xFFFF);
    if (at >= (unsigned long long)po.cap_p) { po.counts[po.n_parts] = 1; continue; }  // the host falls back to the one-pass path
    const unsigned long long d = (unsigned long long)part * (unsigned long long)po.cap_p + at;
#pragma unroll
    for (int s = 0; s < NS; ++s) po.out[s][d] = stash[(size_t)s * R + i];
  }
  for (int r = threadIdx.x; r < po.n_parts; r += kBlock) s_cnt[r] = 0;
  n_stash = 0;
  block_sync<BAR>();  // shared buffers are reused by the next tiles
}

template <int NS, bool EXPR = false>
__device__ __forceinline__ void filter_partition_body(const AggKernelParams& p, const PartitionOut& po) {
  constexpr int R = partition_stash_rows<NS>();
  // dynamic shared memory: [NS][R] survivors in arrival order, [R] tags (partition << 16 | rank), [R] copy-out order
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* stash = reinterpret_cast<uint64_t*>(smem_raw);
  uint32_t* tag = reinterpret_cast<uint32_t*>(stash + (size_t)NS * R);
  uint16_t* perm = reinterpret_cast<uint16_t*>(tag + R);
  __shared__ unsigned int s_cnt[kMaxPartitions];
  __shared__ unsigned int s_off[kMaxPartitions];
  __shared__ unsigned long long s_base[kMaxPartitions];
  __shared__ unsigned int s_wcnt[2][kWarpsPerBlock];
  const int64_t n_tiles = (p.n_rows + kTileRows - 1) / kTileRows;
  const uint64_t pol = make_policy_evict_first();
  for (int r = threadIdx.x; r < po.n_parts; r += kBlock) s_cnt[r] = 0;
  __syncthreads();
  int n_stash = 0;  // block-uniform
  int parity = 0;
  RowVals vals[NS];
  uint32_t vmask[NS];
  int64_t tile = blockIdx.x;
  if (tile < n_tiles) {
#pragma unroll
    for (int s = 0; s < NS; ++s) load_slot<false>(p.cols[s], tile * kTileRows, p.n_rows, nullptr, pol, vals[s], vmask[s]);
  }
  for (; tile < n_tiles; tile += gridDim.x) {
    partition_stash_tile<NS, EXPR, R, 0>(p, po, vals, vmask, tile * kTileRows, stash, tag, s_cnt, s_wcnt, n_stash, parity);
    // the next tile's loads fly while this one is stashed and copied out
    const int64_t next = tile + gridDim.x;
    if (next < n_tiles) {
#pragma unroll
      for (int s = 0; s < NS; ++s) load_slot<false>(p.cols[s], next * kTileRows, p.n_rows, nullptr, pol, vals[s], vmask[s]);
    }
    if (n_stash + kTileRows <= R && next < n_tiles) continue;
    partition_copy_out<NS, R, 0>(po, stash, tag, perm, s_cnt, s_off, s_base, n_stash);
  }
}

// ---------------------------------------------------------------- pass 1, bulk-copy ring variant
// Same filter, tags, stash and copy-out as filter_partition_body, with the column reads taken off the
// threads that filter.  One persistent CTA per SM: warps 0-7 (kBlock threads, barrier 1) filter and
// scatter, warp 8 only moves data.  One lane of it copies each whole tile of every column slot with the
// bulk-copy unit (cp.async.bulk, evict-first) into a ring of D stages, gated by a full / empty mbarrier
// pair per stage.  The consumers read a stage into registers and hand it back at once.  So the ring is
// refilled while they filter, stash, and copy the survivors out, and D tiles of reads stay in flight
// through a copy-out; the plain kernel has one prefetched tile then.  The ring also frees the registers
// and the second CTA the plain kernel needs to hide its loads, which leaves room for a larger stash and
// so longer store runs per partition.  A bulk copy needs a 16-byte aligned source: the host runs this
// kernel only when every column slot starts 16-byte aligned.  A partial last tile is loaded with
// load_slot, so no copy reads past a column.
constexpr int kRingThreads = kBlock + 32;
constexpr size_t kRingSlotBytes = (size_t)kTileRows * 8;  // one slot of a stage: one tile of the widest column
constexpr size_t kRingSmemBudget = 209 << 10;             // dynamic shared memory: 227 KB less the 17.1 KB of static arrays
template <int NS>
__host__ __device__ constexpr int ring_stages() { return NS <= 4 ? 3 : 2; }
template <int NS>
__host__ __device__ constexpr size_t ring_bytes() { return (size_t)ring_stages<NS>() * NS * kRingSlotBytes; }
// the stash takes the rest, in multiples of 256 rows, at most 8192 (NS = 1 .. 8: 8192, 7424, 4608, 2816, 2816, 2048, 1536, 1024)
template <int NS>
__host__ __device__ constexpr int ring_stash_rows() {
  return (kRingSmemBudget - 128 - ring_bytes<NS>()) / (8 * NS + 6) / 256 * 256 > 8192 ? 8192
                                                                                      : (int)((kRingSmemBudget - 128 - ring_bytes<NS>()) / (8 * NS + 6) / 256 * 256);
}
template <int NS>
__host__ __device__ constexpr size_t ring_smem_bytes() { return 128 + ring_bytes<NS>() + (size_t)ring_stash_rows<NS>() * (8 * NS + 4 + 2); }

// The thread's kRowsPerThread rows of one column tile in a ring stage, widened as load_slot widens them.
__device__ __forceinline__ void ring_slot(const unsigned char* st, int dt, RowVals& out) {
  const int t = threadIdx.x;
  if (dt == DBX_I64 || dt == DBX_U64 || dt == DBX_F64) {
    const ulonglong2 a = reinterpret_cast<const ulonglong2*>(st)[2 * t], b = reinterpret_cast<const ulonglong2*>(st)[2 * t + 1];
    out.v[0] = a.x; out.v[1] = a.y; out.v[2] = b.x; out.v[3] = b.y;
  } else if (dt == DBX_I32 || dt == DBX_U32 || dt == DBX_F32) {
    const uint4 q = reinterpret_cast<const uint4*>(st)[t];
    const uint32_t w[kRowsPerThread] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
      out.v[j] = dt == DBX_I32 ? widen<int32_t>((int32_t)w[j]) : (dt == DBX_U32 ? (uint64_t)w[j] : f32_bits_to_f64_bits(w[j]));
  } else if (dt == DBX_I16 || dt == DBX_U16) {
    const uint64_t q = reinterpret_cast<const uint64_t*>(st)[t];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      const uint16_t w = (uint16_t)(q >> (16 * j));
      out.v[j] = dt == DBX_I16 ? widen<int16_t>((int16_t)w) : (uint64_t)w;
    }
  } else {  // DBX_I8, DBX_U8: the host sends no other type through the ring
    const uint32_t q = reinterpret_cast<const uint32_t*>(st)[t];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
      const uint8_t w = (uint8_t)(q >> (8 * j));
      out.v[j] = dt == DBX_I8 ? widen<int8_t>((int8_t)w) : (uint64_t)w;
    }
  }
}

template <int NS, bool EXPR = false>
__device__ __forceinline__ void filter_partition_ring_body(const AggKernelParams& p, const PartitionOut& po) {
  constexpr int R = ring_stash_rows<NS>();
  constexpr int D = ring_stages<NS>();
  static_assert(R >= kTileRows, "the stash holds at least one tile");
  // dynamic shared memory: [D] full and [D] empty barriers (128 B), the ring [D][NS][kRingSlotBytes], then the
  // stash as in filter_partition_body
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw);  // completes when the stage holds its tile
  uint64_t* empty = full + D;                               // completes when every consumer warp has read the stage
  unsigned char* ring = smem_raw + 128;
  uint64_t* stash = reinterpret_cast<uint64_t*>(ring + ring_bytes<NS>());
  uint32_t* tag = reinterpret_cast<uint32_t*>(stash + (size_t)NS * R);
  uint16_t* perm = reinterpret_cast<uint16_t*>(tag + R);
  __shared__ unsigned int s_cnt[kMaxPartitions];
  __shared__ unsigned int s_off[kMaxPartitions];
  __shared__ unsigned long long s_base[kMaxPartitions];
  __shared__ unsigned int s_wcnt[2][kWarpsPerBlock];
  const int64_t n_tiles = (p.n_rows + kTileRows - 1) / kTileRows;
  const int64_t n_full = p.n_rows / kTileRows;  // whole tiles come through the ring
  if (threadIdx.x == 0) {
    for (int d = 0; d < D; ++d) { mbar_init(&full[d], 1); mbar_init(&empty[d], kWarpsPerBlock); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int r = threadIdx.x; r < po.n_parts; r += kRingThreads) s_cnt[r] = 0;
  __syncthreads();  // the last CTA-wide barrier: from here on the consumers synchronise on barrier 1 only
  if (threadIdx.x >= kBlock) {  // the producer warp
    if (threadIdx.x == kBlock) {
      const uint64_t pol = make_policy_evict_first();
      uint32_t tile_bytes = 0;
#pragma unroll
      for (int s = 0; s < NS; ++s)
        if (!p.cols[s].is_const) tile_bytes += kTileRows * dtype_size(p.cols[s].dtype);
      int k = 0;
      for (int64_t tile = blockIdx.x; tile < n_full; tile += gridDim.x, ++k) {
        const int st = k % D;
        mbar_wait(&empty[st], ((k / D) & 1) ^ 1);  // the first round finds every stage free
        mbar_expect_tx(&full[st], tile_bytes);
#pragma unroll
        for (int s = 0; s < NS; ++s) {
          if (p.cols[s].is_const) continue;
          const int w = dtype_size(p.cols[s].dtype);
          bulk_copy_g2s(ring + ((size_t)st * NS + s) * kRingSlotBytes, (const char*)p.cols[s].data + tile * kTileRows * w,
                        (uint32_t)(kTileRows * w), &full[st], pol);
        }
      }
    }
    return;
  }
  const uint64_t pol = make_policy_evict_first();
  int n_stash = 0;  // uniform over the consumer threads
  int parity = 0;
  RowVals vals[NS];
  uint32_t vmask[NS];
  int k = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++k) {
    if (tile < n_full) {
      const int st = k % D;
      mbar_wait(&full[st], (k / D) & 1);
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        if (p.cols[s].is_const) load_slot<false>(p.cols[s], tile * kTileRows, p.n_rows, nullptr, pol, vals[s], vmask[s]);
        else { ring_slot(ring + ((size_t)st * NS + s) * kRingSlotBytes, p.cols[s].dtype, vals[s]); vmask[s] = 0xF; }
      }
      __syncwarp();
      if ((threadIdx.x & 31) == 0) mbar_arrive(&empty[st]);  // the stage is in registers: the producer may refill it
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) load_slot<false>(p.cols[s], tile * kTileRows, p.n_rows, nullptr, pol, vals[s], vmask[s]);
    }
    partition_stash_tile<NS, EXPR, R, 1>(p, po, vals, vmask, tile * kTileRows, stash, tag, s_cnt, s_wcnt, n_stash, parity);
    if (n_stash + kTileRows <= R && tile + gridDim.x < n_tiles) continue;
    partition_copy_out<NS, R, 1>(po, stash, tag, perm, s_cnt, s_off, s_base, n_stash);
  }
}

// ---------------------------------------------------------------- pass 2: one CTA per table slice
// CTA i aggregates partition i against slice i of the table (slice_slots consecutive slots = whole
// buckets) held in shared memory: the slice's keys and state words are loaded from the table, the
// partition's rows are streamed from pass 1's buffers, every row is probed in the slice in the same
// linear bucket order as find_or_insert_slow and updates its group with shared-memory atomics
// (slice_update_words), and the slice is stored back with plain stores (no other CTA touches it).  A row is
// deferred to a list, which the fused kernel then runs against the whole table, when its probe
// would leave the slice (this includes the wrap from the last bucket to bucket 0), when it reaches
// probe_limit (or kSliceProbes), or when its key is the EMPTY pattern: these are the only rows this
// kernel could place somewhere a global probe would not.  As nothing is ever deleted, every key keeps
// exactly one slot.  A row whose key is new is also deferred once the slice holds kSliceFillNum /
// kSliceFillDen of its slots: a table with more groups than it was sized for then stops filling here,
// and the host grows it before the deferred rows run (a full table would make each of them walk
// probe_limit buckets before it overflows).  Any deferred row is probed globally, so deferring more
// rows never changes a result.  The deferred rows' values are copied to a compact list, so the fused
// kernel reads them directly.
//
// The cost of a row is a chain of shared-memory accesses (bucket loads, then atomics whose returned
// values feed the next step), so what matters is how many rows are in flight per SM, and that no warp
// waits for another.  kSliceBlock = 1024 threads (32 warps per SM, at most 64 registers) each stream
// their own rows: the partition is cut into blocks of slice_warp_rows<NS>() rows (32 x RPT), block b
// belongs to warp b mod 32, and each warp copies its blocks into its own kSliceRing buffers in shared
// memory with cp.async (the next block is in flight while this one is aggregated), synchronised with
// __syncwarp only.  So a warp slowed by a long probe, a compare-and-swap retry or a deferred-row
// reservation holds back no other warp, and the CTA meets at a barrier only after the slice is loaded
// and before it is stored back.  No row values are held in registers across a block.  Each thread
// handles its RPT rows in phases: it loads the first bucket of every row (two 128-bit shared loads
// each) before it resolves any slot, then issues the updates of all rows and all state words phase by
// phase (slice_update_words), so that independent atomics are in flight together.
constexpr int kSliceBlock = 1024;
constexpr int kSliceWarps = kSliceBlock / 32;
constexpr int kSliceRing = 2;  // row buffers per warp
constexpr int kSliceFillNum = 3, kSliceFillDen = 4;
// Buckets a row probes in its slice before it is deferred.  Below the load-factor budget chains this
// long are rare; a slice that fills up (more groups than the table was sized for) defers its rows after
// a few probes instead of walking every full bucket to the slice's end.
constexpr int kSliceProbes = 8;
constexpr size_t kSliceBytes = 128 << 10;       // shared memory for one slice: keys + state words
constexpr size_t kSliceStageBytes = 96 << 10;   // every warp's row buffers: a full slice and its rows take 224 of the 227 KB a CTA may use
// Rows of one per-warp block: 64 (two per lane) or 32 where kSliceRing buffers of NS slots for each of the
// 32 warps fit kSliceStageBytes (more rows per thread spill at 64 registers); NS = 7 and 8 only fit 24
// (lanes 24..31 idle, so 768 rows of the CTA are in flight).  A multiple of 8, so every buffer and every
// block's first row stays 16-byte aligned for cp.async.
template <int NS>
__host__ __device__ constexpr int slice_warp_rows() {
  int r = 64;
  while (r > 8 && (size_t)kSliceWarps * kSliceRing * NS * 8 * r > kSliceStageBytes) r -= r > 32 ? 32 : 8;
  return r;
}
template <int NS>
__host__ __device__ constexpr size_t slice_stage_bytes() { return (size_t)kSliceWarps * kSliceRing * NS * 8 * slice_warp_rows<NS>(); }
struct SliceIn {
  const uint64_t* in[kMaxSlots];  // pass 1's partitions: per slot [P][cap_p]
  const unsigned long long* counts;
  int64_t cap_p;
  int64_t slice_slots;
  uint64_t* deferred[kMaxSlots];  // per slot: the deferred rows' values, in no particular order
  unsigned long long* n_deferred; // [0] deferred rows, [1] slices that reached the fill limit
};

__device__ __forceinline__ void cp_async_16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
// Rows [r0, r0 + min(WR, n - r0)) of the partition at `base`, every slot, into buf[NS][WR] as one cp.async
// group of the calling warp (every lane commits one, so the lanes' group counts agree).  The copy moves
// whole 16-byte pairs of rows: a partition's buffer holds cap_p >= n rows and cap_p is a multiple of 4,
// so the pair that holds the last row stays inside it (its other row is not used).
template <int NS, int WR>
__device__ __forceinline__ void slice_warp_copy(const SliceIn& si, int64_t base, int64_t r0, int64_t n, uint64_t* buf, int lane) {
  const int pairs = (int)((min((int64_t)WR, n - r0) + 1) >> 1);
#pragma unroll
  for (int s = 0; s < NS; ++s)
    for (int c = lane; c < pairs; c += 32) cp_async_16(buf + (size_t)s * WR + 2 * c, si.in[s] + base + r0 + 2 * c);
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// One 32-byte bucket of the slice as two 128-bit shared loads; volatile: other threads insert keys meanwhile.
__device__ __forceinline__ u64x4 lds_bucket(const uint64_t* b) {
  u64x4 r;
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(b);
  asm volatile("ld.volatile.shared.v2.u64 {%0, %1}, [%2];" : "=l"(r.x), "=l"(r.y) : "r"(a) : "memory");
  asm volatile("ld.volatile.shared.v2.u64 {%0, %1}, [%2+16];" : "=l"(r.z), "=l"(r.w) : "r"(a) : "memory");
  return r;
}

// GROUP BY key of row i of a stage (slot s of row i at st[s * B + i]); no validity, as in plain_row_key
template <int B>
__device__ __forceinline__ uint64_t stage_row_key(const AggKernelParams& p, const uint64_t* st, int i) {
  uint64_t key = 0;
  if (PLN(n_key_parts) > 1) {
    PLN_UNROLL
    for (int k = 0; k < PLN(n_key_parts); ++k) { const KeyPartDev kp = PLN(key_parts[k]); key |= (st[(size_t)kp.slot * B + i] & kp.mask) << kp.shift; }
  } else {
    key = st[(size_t)PLN(key_slot) * B + i];
    if (PLN(key_is_float)) key = canonical_float_key(key);
  }
  return key;
}

// The probe of one row from its first bucket lb (contents kb) on: the slot, -1 when the row is deferred
// because its probe leaves the slice or reaches max_probes, -2 when it is a new group for a slice at
// its fill limit.
__device__ __noinline__ int64_t slice_probe(uint64_t* skeys, uint64_t key, int64_t lb, u64x4 kb, int64_t nbs, int max_probes,
                                            unsigned int* s_fill, unsigned int fill_limit) {
  int probes = 0;
  while (true) {
    const int m = bucket_match(kb, key);
    if (m >= 0) return 4 * lb + m;
    const int e = kb.x == kEmptyKey ? 0 : (kb.y == kEmptyKey ? 1 : (kb.z == kEmptyKey ? 2 : (kb.w == kEmptyKey ? 3 : -1)));
    if (e >= 0) {
      if (*(volatile unsigned int*)s_fill >= fill_limit) return -2;
      const unsigned long long old = atomicCAS((unsigned long long*)(skeys + 4 * lb + e), (unsigned long long)kEmptyKey, (unsigned long long)key);
      if (old == kEmptyKey) { atomicAdd(s_fill, 1u); return 4 * lb + e; }
      if (old == key) return 4 * lb + e;
      kb = lds_bucket(skeys + 4 * lb);  // another key took the slot: look at this bucket again (it has one EMPTY slot less)
      continue;
    }
    if (++lb == nbs) return -1;  // the probe leaves the slice
    if (++probes >= max_probes) return -1;
    kb = lds_bucket(skeys + 4 * lb);
  }
}

// (state word, row) pairs per call of slice_update_words: the specialised build takes every word of its
// plan at once (the plan is a constant, so the phases unroll to straight-line code); the precompiled one
// reads the plan at run time and takes a few words at a time, so that what the first phase returns fits
// its registers.
#ifdef DBX_JIT
constexpr int kSliceUpdPairs = 32;
#else
constexpr int kSliceUpdPairs = 4;
#endif

// Update words upd[u0, u0 + G) of a thread's RPT rows (row r is lane + 32 r of the warp's block `st`; bit r
// of `on`: it has slot slot[r]), phase by phase over all rows and words, so that no shared-memory access
// waits on a result it does not need:
//  1. the low halves of the integer words (counts and integer sums are two native 32-bit shared adds plus
//     a carry, as in smem_add_u64) and the first load of every f64 sum;
//  2. the high halves with their carries, the first compare-and-swap of every f64 sum, and the minima and
//     maxima (hot_update's shared-memory atomics);
//  3. one retry loop over the (row, f64 word) pairs whose compare-and-swap lost a race.
template <int RPT, int G, int WR>
__device__ __forceinline__ void slice_update_words(const AggKernelParams& p, int u0, const uint64_t* st, int lane, uint64_t* sst, int nw,
                                                   const int (&slot)[RPT], uint32_t on) {
  static_assert(G * RPT <= 32, "one pending bit per (word, row)");
  auto word = [&](int u, int r) { return sst + slot[r] * nw + PLN(upd[u]).word; };
  auto val = [&](int u, int r) { return st[PLN(upd[u]).slot * WR + lane + 32 * r]; };
  auto is_int = [](int op) { return op == UPD_INC || op == UPD_INC_VALID || op == UPD_ADD_INT; };
  uint64_t got[G][RPT];  // what phase 1 returned: the old low half of an integer word, the f64 word
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int u = u0 + g;
    if (u >= PLN(n_updates)) break;
    const int op = PLN(upd[u]).op;
#pragma unroll
    for (int r = 0; r < RPT; ++r) {
      if (!((on >> r) & 1)) continue;
      if (is_int(op)) got[g][r] = atomicAdd(reinterpret_cast<unsigned int*>(word(u, r)), op == UPD_ADD_INT ? (unsigned int)val(u, r) : 1u);
      else if (op == UPD_ADD_F64) got[g][r] = *reinterpret_cast<volatile unsigned long long*>(word(u, r));
    }
  }
  uint32_t pend = 0;  // bit g * RPT + r: row r's compare-and-swap of word u0 + g lost a race
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int u = u0 + g;
    if (u >= PLN(n_updates)) break;
    const int op = PLN(upd[u]).op;
#pragma unroll
    for (int r = 0; r < RPT; ++r) {
      if (!((on >> r) & 1)) continue;
      const uint64_t v = op == UPD_INC || op == UPD_INC_VALID ? 1 : val(u, r);
      if (is_int(op)) {
        const unsigned int old = (unsigned int)got[g][r], lo = (unsigned int)v, up = (unsigned int)(v >> 32) + (old + lo < old ? 1u : 0u);
        if (up) atomicAdd(reinterpret_cast<unsigned int*>(word(u, r)) + 1, up);
      } else if (op == UPD_ADD_F64) {
        const unsigned long long cur = got[g][r];
        const unsigned long long nv = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)cur) + __longlong_as_double((long long)v));
        const unsigned long long o = atomicCAS(reinterpret_cast<unsigned long long*>(word(u, r)), cur, nv);
        if (o != cur) pend |= 1u << (g * RPT + r);
        got[g][r] = o;
      } else {
        hot_update(op, word(u, r), v, true);
      }
    }
  }
  while (pend) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int u = u0 + g;
      if (u >= PLN(n_updates)) break;
      if (PLN(upd[u]).op != UPD_ADD_F64) continue;
#pragma unroll
      for (int r = 0; r < RPT; ++r) {
        if (!((pend >> (g * RPT + r)) & 1)) continue;
        const unsigned long long cur = got[g][r];
        const unsigned long long nv = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)cur) + __longlong_as_double((long long)val(u, r)));
        const unsigned long long o = atomicCAS(reinterpret_cast<unsigned long long*>(word(u, r)), cur, nv);
        if (o == cur) pend &= ~(1u << (g * RPT + r));
        got[g][r] = o;
      }
    }
  }
}

template <int NS>
__device__ __forceinline__ void slice_agg_body(const AggKernelParams& p, const SliceIn& si) {
  constexpr int WR = slice_warp_rows<NS>();
  constexpr int RPT = (WR + 31) / 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ unsigned int s_fill, s_fill0;  // occupied slots of the slice: now, and when it was loaded
  const TableDev& t = p.table;
  // the nw state words of a slot are one row-major entry, so the slice's entries are one contiguous run of the table
  const int nw = PLN_TABLE(n_words);
  const int64_t S = si.slice_slots;
  uint64_t* skeys = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t* sst = skeys + S;                 // state word w of slot i at sst[i * nw + w]
  uint64_t* stage = sst + S * nw;            // per warp, kSliceRing buffers of [NS][WR] row values
  const int64_t slot0 = (int64_t)blockIdx.x * S;
  const int64_t n = (int64_t)si.counts[blockIdx.x];
  const int64_t base = (int64_t)blockIdx.x * si.cap_p;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t* ring = stage + (size_t)warp * kSliceRing * NS * WR;
  // block b of the partition (rows [b * WR, b * WR + WR)) belongs to warp b mod kSliceWarps
  const int64_t n_blocks = (n + WR - 1) / WR;
  const int my_blocks = warp < n_blocks ? (int)((n_blocks - 1 - warp) / kSliceWarps) + 1 : 0;
  if (my_blocks > 0) slice_warp_copy<NS, WR>(si, base, (int64_t)warp * WR, n, ring, lane);  // in flight while the slice is loaded
  if (threadIdx.x == 0) s_fill = s_fill0 = 0;
  __syncthreads();
  ulonglong2* gkeys = reinterpret_cast<ulonglong2*>(t.keys + slot0);
  ulonglong2* gst = reinterpret_cast<ulonglong2*>(t.states + slot0 * nw);
  unsigned int occupied = 0;
#pragma unroll 2
  for (int64_t i = threadIdx.x; i < S / 2; i += kSliceBlock) {
    const ulonglong2 k = gkeys[i];
    reinterpret_cast<ulonglong2*>(skeys)[i] = k;
    occupied += (k.x != kEmptyKey ? 1u : 0u) + (k.y != kEmptyKey ? 1u : 0u);
  }
  if (occupied) { atomicAdd(&s_fill, occupied); atomicAdd(&s_fill0, occupied); }
#pragma unroll 4
  for (int64_t e = threadIdx.x; e < S * nw / 2; e += kSliceBlock) reinterpret_cast<ulonglong2*>(sst)[e] = gst[e];
  const unsigned int fill_limit = (unsigned int)(S * kSliceFillNum / kSliceFillDen);
  const int64_t nbs = S >> 2;  // buckets per slice
  const uint64_t nb_mask = (uint64_t)(t.cap >> 2) - 1;
  const int max_probes = min(t.probe_limit, kSliceProbes);
  bool hit_limit = false;
  __syncthreads();  // the slice is loaded; from here on each warp runs on its own until the store-back
  for (int j = 0; j < my_blocks; ++j) {
    const int64_t r0 = ((int64_t)j * kSliceWarps + warp) * WR;
    const uint64_t* st = ring + (size_t)(j % kSliceRing) * NS * WR;
    if (j + 1 < my_blocks) {
      slice_warp_copy<NS, WR>(si, base, r0 + (int64_t)kSliceWarps * WR, n, ring + (size_t)((j + 1) % kSliceRing) * NS * WR, lane);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncwarp();  // this block's rows, copied by every lane, are visible to the whole warp
    const int m = (int)min((int64_t)WR, n - r0);
    // phase 1: the first bucket of every row, then the slots
    uint64_t key[RPT];
    int64_t lb[RPT];
    u64x4 kb[RPT];
    uint32_t probe = 0;  // rows with a key to probe (the EMPTY pattern is deferred)
#pragma unroll
    for (int r = 0; r < RPT; ++r) {
      const int i = lane + 32 * r;
      key[r] = i < m ? stage_row_key<WR>(p, st, i) : kEmptyKey;
      lb[r] = 0;
      kb[r].x = kb[r].y = kb[r].z = kb[r].w = 0;
      if (i < m && key[r] != kEmptyKey) {
        probe |= 1u << r;
        lb[r] = (int64_t)(agg_hash_u64(key[r]) & nb_mask) - (int64_t)blockIdx.x * nbs;
        kb[r] = lds_bucket(skeys + 4 * lb[r]);
      }
    }
    int slot[RPT];
#pragma unroll
    for (int r = 0; r < RPT; ++r) {
      slot[r] = -1;
      if (!((probe >> r) & 1)) continue;
      const int mt = bucket_match(kb[r], key[r]);
      if (mt >= 0) {
        slot[r] = (int)(4 * lb[r] + mt);
      } else {
        const int64_t s = slice_probe(skeys, key[r], lb[r], kb[r], nbs, max_probes, &s_fill, fill_limit);
        if (s == -2) hit_limit = true;
        slot[r] = s < 0 ? -1 : (int)s;
      }
    }
    // the deferred rows (live, no slot), reserved once per warp and row position
#pragma unroll
    for (int r = 0; r < RPT; ++r) {
      const int i = lane + 32 * r;
      const bool defer = i < m && slot[r] < 0;
      const unsigned dm = __ballot_sync(0xffffffffu, defer);
      if (dm) {
        unsigned long long d = 0;
        if (lane == 0) d = atomicAdd(si.n_deferred, (unsigned long long)__popc(dm));
        d = __shfl_sync(0xffffffffu, d, 0) + __popc(dm & ((1u << lane) - 1));
        if (defer) {
#pragma unroll
          for (int s = 0; s < NS; ++s) si.deferred[s][d] = st[(size_t)s * WR + i];
        }
      }
    }
    // phase 2: the updates of every row and state word
    uint32_t on = 0;
#pragma unroll
    for (int r = 0; r < RPT; ++r)
      if (slot[r] >= 0) on |= 1u << r;
    constexpr int G = kSliceUpdPairs / RPT;
    PLN_UNROLL
    for (int u0 = 0; u0 < PLN(n_updates); u0 += G) slice_update_words<RPT, G, WR>(p, u0, st, lane, sst, nw, slot, on);
    __syncwarp();  // every lane is done with this buffer before the warp's next copy overwrites it
  }
  const int any_hit = __syncthreads_or(hit_limit);
#pragma unroll 2
  for (int64_t i = threadIdx.x; i < S / 2; i += kSliceBlock) gkeys[i] = reinterpret_cast<const ulonglong2*>(skeys)[i];
#pragma unroll 4
  for (int64_t e = threadIdx.x; e < S * nw / 2; e += kSliceBlock) gst[e] = reinterpret_cast<const ulonglong2*>(sst)[e];
  if (threadIdx.x == 0) {
    if (s_fill > s_fill0) atomicAdd(t.n_groups, (unsigned long long)(s_fill - s_fill0));
    if (any_hit) atomicAdd(si.n_deferred + 1, 1ULL);
  }
}

#ifndef DBX_JIT  // everything below is compiled offline only
// the precompiled passes (no NVRTC on the machine, a plan that could not be specialised, DBX_AGG_JIT=0)
template <int NS, bool EXPR = false>
__global__ void __launch_bounds__(kBlock, 2) filter_partition_kernel(const __grid_constant__ AggKernelParams p, const __grid_constant__ PartitionOut po) {
  filter_partition_body<NS, EXPR>(p, po);
}
template <int NS, bool EXPR = false>
__global__ void __launch_bounds__(kRingThreads, 1) filter_partition_ring_kernel(const __grid_constant__ AggKernelParams p,
                                                                                const __grid_constant__ PartitionOut po) {
  filter_partition_ring_body<NS, EXPR>(p, po);
}
template <int NS>
__global__ void __launch_bounds__(kSliceBlock, 1) slice_agg_kernel(const __grid_constant__ AggKernelParams p, const __grid_constant__ SliceIn si) {
  slice_agg_body<NS>(p, si);
}

// ---------------------------------------------------------------- fused kernel (no GROUP BY)
// PartialSingleStateAggregator (transform_single_key.rs:93-141): a pure streaming reduce.
// Per-thread accumulators -> warp shuffle -> one atomic per warp into the single state.
__device__ __forceinline__ uint64_t upd_identity(int op) {
  if (op == UPD_MIN_S64) return (uint64_t)INT64_MAX;
  if (op == UPD_MAX_S64) return (uint64_t)INT64_MIN;
  if (op == UPD_MIN_U64 || op == UPD_MIN_F64) return ~0ULL;
  return 0;
}
__device__ __forceinline__ uint64_t upd_combine(int op, uint64_t a, uint64_t b) {
  if (op == UPD_ADD_F64) return (uint64_t)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
  if (op == UPD_MIN_S64) return (uint64_t)min((int64_t)a, (int64_t)b);
  if (op == UPD_MAX_S64) return (uint64_t)max((int64_t)a, (int64_t)b);
  if (op == UPD_MIN_U64 || op == UPD_MIN_F64) return a < b ? a : b;
  if (op == UPD_MAX_U64 || op == UPD_MAX_F64) return a > b ? a : b;
  return a + b;
}
__device__ __forceinline__ void merge_word(int op, void* w, uint64_t v) {
  if (op == UPD_ADD_F64) { red_add_f64(w, __longlong_as_double((long long)v)); return; }
  if (op == UPD_MIN_S64) { red_min_s64(w, (int64_t)v); return; }
  if (op == UPD_MAX_S64) { red_max_s64(w, (int64_t)v); return; }
  if (op == UPD_MIN_U64 || op == UPD_MIN_F64) { red_min_u64(w, v); return; }
  if (op == UPD_MAX_U64 || op == UPD_MAX_F64) { red_max_u64(w, v); return; }
  red_add_u64(w, v);
}

template <int NS, bool EXPR = false>
__global__ void __launch_bounds__(kBlock, 4) filter_single_agg_kernel(const __grid_constant__ AggKernelParams p) {
  const int64_t n_tiles = (p.n_rows + kTileRows - 1) / kTileRows;
  __shared__ uint64_t s_acc[kWarpsPerBlock][kMaxUpdates];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t pol = make_policy_evict_first();
  // per-thread accumulators live in shared memory indexed by update (dynamic index without
  // local-memory spills); one column of 32 lanes per warp would be too big, so each thread
  // keeps its partials in registers for up to 4 updates and falls back to shared beyond that.
  uint64_t acc0 = upd_identity(p.n_updates > 0 ? p.upd[0].op : 0);
  uint64_t acc1 = upd_identity(p.n_updates > 1 ? p.upd[1].op : 0);
  uint64_t acc2 = upd_identity(p.n_updates > 2 ? p.upd[2].op : 0);
  uint64_t acc3 = upd_identity(p.n_updates > 3 ? p.upd[3].op : 0);
  if (lane == 0)
    for (int u = 0; u < kMaxUpdates; ++u) s_acc[warp][u] = upd_identity(u < p.n_updates ? p.upd[u].op : 0);
  __syncwarp();

  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    __syncwarp();
    const int64_t tile_base = tile * kTileRows;
    RowVals vals[NS];
    uint32_t vmask[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) load_slot<false>(p.cols[s], tile_base, p.n_rows, nullptr, pol, vals[s], vmask[s]);
    const int64_t r0 = tile_base + (int64_t)kRowsPerThread * threadIdx.x;
    uint32_t in_range = 0;
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
      if (r0 + j < p.n_rows) in_range |= 1u << j;
    if (EXPR) eval_computed<NS, false>(p, 0, p.comp_pred, vals, vmask, 0, r0);
    const uint32_t sel = eval_predicate<NS>(p, vals, vmask, in_range);
    if (EXPR) eval_computed<NS, false>(p, p.comp_pred, p.n_comp, vals, vmask, sel, r0);
    for (int u = 0; u < p.n_updates; ++u) {
      const UpdateDev ud = p.upd[u];
      const uint32_t m = sel & (ud.op == UPD_INC ? 0xFu : pick_mask<NS>(vmask, ud.slot));
      uint64_t part = upd_identity(ud.op);
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) {
        if (!((m >> j) & 1)) continue;
        uint64_t val = pick<NS>(vals, ud.slot, j);
        uint64_t x = (ud.op == UPD_INC || ud.op == UPD_INC_VALID) ? 1
                     : (ud.op == UPD_MIN_F64 || ud.op == UPD_MAX_F64) ? f64_to_ordered(__longlong_as_double((long long)val))
                                                                       : val;
        part = upd_combine(ud.op, part, x);
      }
      if (u == 0) acc0 = upd_combine(ud.op, acc0, part);
      else if (u == 1) acc1 = upd_combine(ud.op, acc1, part);
      else if (u == 2) acc2 = upd_combine(ud.op, acc2, part);
      else if (u == 3) acc3 = upd_combine(ud.op, acc3, part);
      else {  // rare: more than 4 state words — reduce across the warp right away
        uint64_t a = part;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a = upd_combine(ud.op, a, __shfl_xor_sync(0xffffffffu, a, o));
        if (lane == 0) s_acc[warp][u] = upd_combine(ud.op, s_acc[warp][u], a);
      }
    }
  }
  __syncwarp();
  for (int u = 0; u < p.n_updates; ++u) {
    const int op = p.upd[u].op;
    uint64_t a = u == 0 ? acc0 : u == 1 ? acc1 : u == 2 ? acc2 : u == 3 ? acc3 : upd_identity(op);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a = upd_combine(op, a, __shfl_xor_sync(0xffffffffu, a, o));
    if (lane == 0) {
      if (u >= 4) a = s_acc[warp][u];
      merge_word(op, word_ptr(p.table, 0, p.upd[u].word), a);
    }
  }
}

// ---------------------------------------------------------------- standalone filter (TransformFilter)
// FilterExecutor::filter = select + take (filter_executor.rs:82-160, kernels/filter.rs:36-70,
// kernels/take.rs:43-60): rows for which the predicate is true, in input order, for every column.
//   pass 1  filter_select_kernel: predicate in registers -> 4-bit selection per thread + per-tile count
//   (scan of the tile counts)
//   pass 2  filter_take_kernel: every thread knows its output position (tile offset + block scan of
//           the popcounts) and copies its selected rows of every column — order preserved, no atomics.
template <int NS, bool EXPR = false>
__global__ void __launch_bounds__(kBlock) filter_select_kernel(const __grid_constant__ AggKernelParams p, uint8_t* sel_nibbles,
                                                               uint32_t* tile_counts) {
  __shared__ uint32_t s_cnt[kWarpsPerBlock];
  const int64_t n_tiles = (p.n_rows + kTileRows - 1) / kTileRows;
  const uint64_t pol = make_policy_evict_first();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t tile_base = tile * kTileRows;
    RowVals vals[NS];
    uint32_t vmask[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) load_slot<false>(p.cols[s], tile_base, p.n_rows, nullptr, pol, vals[s], vmask[s]);
    const int64_t r0 = tile_base + (int64_t)kRowsPerThread * threadIdx.x;
    uint32_t in_range = 0;
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j)
      if (r0 + j < p.n_rows) in_range |= 1u << j;
    if (EXPR) eval_computed<NS, false>(p, 0, p.n_comp, vals, vmask, 0, r0);  // predicate inputs only: they cannot raise
    const uint32_t sel = eval_predicate<NS>(p, vals, vmask, in_range);
    sel_nibbles[tile * kBlock + threadIdx.x] = (uint8_t)sel;
    uint32_t c = __popc(sel);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_cnt[warp] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t t = 0;
      for (int w = 0; w < kWarpsPerBlock; ++w) t += s_cnt[w];
      tile_counts[tile] = t;
    }
    __syncthreads();
  }
}

struct TakeCol {
  const void* src;
  const uint8_t* src_valid;  // bitmap or nullptr
  int64_t src_vbit_off, src_dbit_off;
  void* dst;                 // values (BOOL: one byte per row, packed afterwards)
  uint8_t* dst_valid;        // one byte per row or nullptr
  int32_t dtype, is_const;
  uint64_t const_bits;
};
struct TakeParams {
  TakeCol cols[64];
  int32_t n_cols;
  int64_t n_rows;
  const uint8_t* sel_nibbles;
  const uint32_t* tile_offsets;  // exclusive scan of the tile counts
};
__global__ void __launch_bounds__(kBlock) filter_take_kernel(const __grid_constant__ TakeParams p) {
  __shared__ uint32_t s_warp[kWarpsPerBlock];
  const int64_t n_tiles = (p.n_rows + kTileRows - 1) / kTileRows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const uint32_t sel = p.sel_nibbles[tile * kBlock + threadIdx.x];
    const uint32_t n = __popc(sel);
    uint32_t incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0;
    for (int w = 0; w < warp; ++w) wbase += s_warp[w];
    __syncthreads();
    if (!sel) continue;
    const int64_t out0 = (int64_t)p.tile_offsets[tile] + wbase + incl - n;
    const int64_t r0 = tile * kTileRows + (int64_t)kRowsPerThread * threadIdx.x;
    for (int c = 0; c < p.n_cols; ++c) {
      const TakeCol& tc = p.cols[c];
      const int esz = dtype_size(tc.dtype);
      int64_t o = out0;
#pragma unroll
      for (int j = 0; j < kRowsPerThread; ++j) {
        if (!((sel >> j) & 1)) continue;
        const int64_t r = r0 + j;
        if (tc.dtype == DBX_BOOL) {
          ((uint8_t*)tc.dst)[o] = tc.is_const ? (uint8_t)(tc.const_bits != 0) : (uint8_t)bit_test((const uint8_t*)tc.src, tc.src_dbit_off + r);
        } else if (tc.is_const) {
          if (esz == 8) ((uint64_t*)tc.dst)[o] = tc.const_bits;
          else if (esz == 4) ((uint32_t*)tc.dst)[o] = tc.dtype == DBX_F32 ? __float_as_uint((float)__longlong_as_double((long long)tc.const_bits)) : (uint32_t)tc.const_bits;
          else if (esz == 2) ((uint16_t*)tc.dst)[o] = (uint16_t)tc.const_bits;
          else ((uint8_t*)tc.dst)[o] = (uint8_t)tc.const_bits;
        } else {
          if (esz == 8) ((uint64_t*)tc.dst)[o] = ((const uint64_t*)tc.src)[r];
          else if (esz == 4) ((uint32_t*)tc.dst)[o] = ((const uint32_t*)tc.src)[r];
          else if (esz == 2) ((uint16_t*)tc.dst)[o] = ((const uint16_t*)tc.src)[r];
          else ((uint8_t*)tc.dst)[o] = ((const uint8_t*)tc.src)[r];
        }
        if (tc.dst_valid) tc.dst_valid[o] = tc.is_const == 2 ? 0 : (tc.src_valid ? (uint8_t)bit_test(tc.src_valid, tc.src_vbit_off + r) : 1);
        ++o;
      }
    }
  }
}

// ---------------------------------------------------------------- table maintenance
struct WordInit {
  uint64_t w[kMaxWords];
};
__global__ void table_init_kernel(const __grid_constant__ TableDev t, const __grid_constant__ WordInit init) {
  const int64_t n_slots = t.cap + 2;
  const int64_t n_keys = n_slots * t.key_words;
  const int64_t total = n_keys + n_slots * t.n_words;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < n_keys) t.keys[i] = kEmptyKey;
    else t.states[i - n_keys] = init.w[(i - n_keys) % t.n_words];
  }
}

// Kinds of state words, for merging two states of the same group
// (batch_merge_states: aggregate_sum.rs:126-129, aggregate_avg.rs:82-86, count: += , min/max).
struct WordKinds {
  int32_t op[kMaxWords];  // UPD_ADD_INT (also counts), UPD_ADD_F64, UPD_MIN_*, UPD_MAX_* (ordered image for F64)
};

// Resolve the destination slot of a (key, key_kind) pair. key_kind: 0 normal, 1 key == EMPTY
// sentinel, 2 NULL key.
__device__ __forceinline__ int64_t resolve_slot(const TableDev& t, uint64_t key, int key_kind, uint32_t& new_groups) {
  if (key_kind != 0) return special_slot(t, key_kind == 2, new_groups);
  const int64_t b = (int64_t)(agg_hash_u64(key) & (uint64_t)((t.cap >> 2) - 1));
  u64x4 kb = ld_bucket(t.keys + 4 * b);
  int m = bucket_match(kb, key);
  return m >= 0 ? 4 * b + m : find_or_insert_slow(t, key, b, kb, new_groups);
}

// AggregateHashTable::combine_payload (aggregate_hashtable.rs:349-380) / resize (:463-489):
// every occupied slot of `src` is found-or-inserted in `dst` and its words merged.
__global__ void table_merge_kernel(const __grid_constant__ TableDev src, const __grid_constant__ TableDev dst,
                                   const __grid_constant__ WordKinds kinds) {
  uint32_t new_groups = 0;
  const int64_t n_slots = src.cap + 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t d;
    if (src.key_words == 2) {
      uint64_t k0 = src.keys[2 * i], k1 = src.keys[2 * i + 1];
      if (i >= src.cap) { if (i > src.cap || k0 == kEmptyKey) continue; k0 = k1 = kEmptyKey; }  // special slot: the EMPTY-pattern key
      else if (k0 == kEmptyKey && k1 == kEmptyKey) continue;
      d = resolve_slot_wide(dst, k0, k1, new_groups);
    } else {
      uint64_t key = src.keys[i];
      if (key == kEmptyKey) continue;
      int key_kind = i >= src.cap ? (int)(i - src.cap) + 1 : 0;
      d = resolve_slot(dst, key, key_kind, new_groups);
    }
    if (d < 0) { atomicAdd(dst.n_overflow, 1ULL); continue; }
    for (int w = 0; w < src.n_words; ++w) merge_word(kinds.op[w], word_ptr(dst, d, w), *word_ptr(src, i, w));
  }
  __syncwarp();
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) new_groups += __shfl_xor_sync(0xffffffffu, new_groups, o);
  if ((threadIdx.x & 31) == 0 && new_groups) atomicAdd(dst.n_groups, (unsigned long long)new_groups);
}

// Exchange rows for the partial -> final shuffle: [key:8][key_kind:8][words: 8*n_words].
// Owner of a group = high 32 bits of agg_hash scaled to n_parts, i.e. radix partitioning on
// the top hash bits like PartitionedPayload (partitioned_payload.rs:44-57) but for any n_parts.
__device__ __forceinline__ int owner_of(uint64_t key, int key_kind, int n_parts) {
  uint64_t h = key_kind == 2 ? kNullHashVal : agg_hash_u64(key_kind == 1 ? kEmptyKey : key);
  return hash_to_part(h, n_parts);
}

__global__ void table_partition_count_kernel(const __grid_constant__ TableDev src, int n_parts,
                                             unsigned long long* counts) {
  extern __shared__ unsigned int s_cnt[];
  for (int i = threadIdx.x; i < n_parts; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  const int64_t n_slots = src.cap + 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t key = src.keys[i];
    if (key == kEmptyKey) continue;
    int key_kind = i >= src.cap ? (int)(i - src.cap) + 1 : 0;
    atomicAdd(&s_cnt[owner_of(key, key_kind, n_parts)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_parts; i += blockDim.x)
    if (s_cnt[i]) atomicAdd(&counts[i], (unsigned long long)s_cnt[i]);
}

__global__ void table_partition_scatter_kernel(const __grid_constant__ TableDev src, int n_parts,
                                               unsigned long long* cursors /* pre-set to part offsets */,
                                               uint64_t* rows_out) {
  const int row_words = 2 + src.n_words;
  const int64_t n_slots = src.cap + 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_slots; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t key = src.keys[i];
    if (key == kEmptyKey) continue;
    int key_kind = i >= src.cap ? (int)(i - src.cap) + 1 : 0;
    unsigned long long pos = atomicAdd(&cursors[owner_of(key, key_kind, n_parts)], 1ULL);
    uint64_t* r = rows_out + pos * row_words;
    r[0] = key_kind ? 0 : key;
    r[1] = (uint64_t)key_kind;
    for (int w = 0; w < src.n_words; ++w) r[2 + w] = *word_ptr(src, i, w);
  }
}

// TransformFinalAggregate::handle_meta on received payload rows (transform_aggregate_final.rs:201-303)
__global__ void rows_merge_kernel(const uint64_t* rows, int64_t n_rows, const __grid_constant__ TableDev dst,
                                  const __grid_constant__ WordKinds kinds) {
  uint32_t new_groups = 0;
  const int row_words = 2 + dst.n_words;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rows; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t* r = rows + i * row_words;
    int64_t d = resolve_slot(dst, r[0], (int)r[1], new_groups);
    if (d < 0) { atomicAdd(dst.n_overflow, 1ULL); continue; }
    for (int w = 0; w < dst.n_words; ++w) merge_word(kinds.op[w], word_ptr(dst, d, w), r[2 + w]);
  }
  __syncwarp();
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) new_groups += __shfl_xor_sync(0xffffffffu, new_groups, o);
  if ((threadIdx.x & 31) == 0 && new_groups) atomicAdd(dst.n_groups, (unsigned long long)new_groups);
}

// Same, but ONE thread merges the rows in the order given: used for per-rank single states
// (no GROUP BY), where the row order is the rank order and f64 sums must be reproducible.
__global__ void rows_merge_ordered_kernel(const uint64_t* rows, int64_t n_rows, const __grid_constant__ TableDev dst,
                                          const __grid_constant__ WordKinds kinds) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  uint32_t new_groups = 0;
  const int row_words = 2 + dst.n_words;
  for (int64_t i = 0; i < n_rows; ++i) {
    const uint64_t* r = rows + i * row_words;
    int64_t d = resolve_slot(dst, r[0], (int)r[1], new_groups);
    if (d < 0) { atomicAdd(dst.n_overflow, 1ULL); continue; }
    for (int w = 0; w < dst.n_words; ++w) {
      merge_word(kinds.op[w], word_ptr(dst, d, w), r[2 + w]);
      __threadfence();  // keep the order of the f64 additions to one word
    }
  }
  if (new_groups) atomicAdd(dst.n_groups, (unsigned long long)new_groups);
}

// ---------------------------------------------------------------- partial -> final exchange over peer memory
// One process per GPU; every rank owns a receive buffer in its HBM that all peers map (CUDA IPC
// over NVLink / NVSwitch).  The partial's groups are hash-partitioned by owner and each row is
// stored DIRECTLY into the owner's receive region by the scatter kernel (no staging copy, no
// count exchange, no NCCL on the data path); a release-flag per (source, owner) tells the owner's
// merge kernel that the region is complete.  Mirrors build_partition_bucket.rs:41-131 + the
// Flight exchange of AggregateMeta partitions, as one fused partition+send kernel.
constexpr int kMaxRanks = 16;
struct ExchangeHeader {
  unsigned long long count[2][kMaxRanks];  // [parity][source rank]: rows that source wrote
  unsigned long long flag[kMaxRanks];      // [source rank]: last epoch the source completed
  unsigned long long overflow[2][kMaxRanks];  // [parity][source rank]: epoch in which the region was too small
  unsigned long long pad[16];
};
struct ExchangeScatterParams {
  TableDev src;
  void* peer_base[kMaxRanks];  // receive buffer (header first) of every rank, as mapped here
  unsigned long long* cursors; // [n_ranks] rows reserved per owner (zeroed before the launch)
  unsigned int* done;          // CTAs finished (zeroed before the launch)
  int64_t region_rows;
  unsigned long long epoch;
  int32_t n_ranks, rank, row_words, parity;
  int32_t clear_src;  // 1: re-initialise every source slot once it was read (fused table clear)
  int32_t pad;
  WordInit init;
};
__device__ __forceinline__ uint64_t* exchange_region(void* base, int n_ranks, int parity, int src, int64_t region_rows, int row_words) {
  return reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(base) + sizeof(ExchangeHeader)) +
         ((int64_t)(parity * n_ranks + src) * region_rows) * row_words;
}

constexpr int kExchMaxRowWords = 2 + kMaxWords;
constexpr int kScatterSlots = 4;  // table slots per thread and step
__global__ void __launch_bounds__(256) exchange_scatter_kernel(const __grid_constant__ ExchangeScatterParams x) {
  // Per step of 1024 slots (4 per thread): count the step's groups per owner, reserve a run in every
  // owner's region with ONE atomic per owner, lay the rows out owner after owner in shared memory,
  // then copy each owner's run with consecutive 8-byte stores — NVLink sees full 128-byte lines
  // instead of scattered 8-byte writes, and the barriers are amortised over four slots per thread.
  extern __shared__ __align__(16) uint64_t s_rows[];  // [1024][row_words]
  __shared__ unsigned int s_cnt[kMaxRanks];
  __shared__ unsigned int s_off[kMaxRanks + 1];
  __shared__ unsigned long long s_base[kMaxRanks];
  __shared__ int s_last;
  const TableDev& src = x.src;
  const int rw = x.row_words;
  const int64_t n_slots = src.cap + 2;
  const int64_t step_slots = 256 * kScatterSlots;
  const int64_t n_steps = (n_slots + step_slots - 1) / step_slots;
  for (int64_t st = blockIdx.x; st < n_steps; st += gridDim.x) {
    if (threadIdx.x < kMaxRanks) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const int64_t i0 = st * step_slots + threadIdx.x;
    uint64_t key[kScatterSlots];
    int owner[kScatterSlots];
    unsigned int local[kScatterSlots];
#pragma unroll
    for (int j = 0; j < kScatterSlots; ++j) {
      const int64_t i = i0 + (int64_t)j * 256;
      key[j] = i < n_slots ? src.keys[i] : kEmptyKey;
    }
#pragma unroll
    for (int j = 0; j < kScatterSlots; ++j) {
      const int64_t i = i0 + (int64_t)j * 256;
      owner[j] = -1;
      local[j] = 0;
      if (key[j] != kEmptyKey) {
        const int key_kind = i >= src.cap ? (int)(i - src.cap) + 1 : 0;
        owner[j] = owner_of(key[j], key_kind, x.n_ranks);
        local[j] = atomicAdd(&s_cnt[owner[j]], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int o = 0;
      for (int r = 0; r < x.n_ranks; ++r) { s_off[r] = o; o += s_cnt[r]; }
      s_off[x.n_ranks] = o;
    }
    if (threadIdx.x < x.n_ranks && s_cnt[threadIdx.x])
      s_base[threadIdx.x] = atomicAdd(&x.cursors[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kScatterSlots; ++j) {
      if (owner[j] < 0) continue;
      const int64_t i = i0 + (int64_t)j * 256;
      const int key_kind = i >= src.cap ? (int)(i - src.cap) + 1 : 0;
      uint64_t* r = s_rows + (size_t)(s_off[owner[j]] + local[j]) * rw;
      r[0] = key_kind ? 0 : key[j];
      r[1] = (uint64_t)key_kind;
      for (int w = 0; w < src.n_words; ++w) r[2 + w] = *word_ptr(src, i, w);
      if (x.clear_src) {  // the slot is read by this thread only: leave the table ready for the next query
        src.keys[i] = kEmptyKey;
        for (int w = 0; w < src.n_words; ++w) *word_ptr(src, i, w) = x.init.w[w];
      }
    }
    __syncthreads();
    for (int o = 0; o < x.n_ranks; ++o) {
      const unsigned int cnt = s_cnt[o];
      if (!cnt) continue;
      const unsigned long long base = s_base[o];
      // rows beyond the region are dropped here and reported through the overflow flag
      const int64_t room = x.region_rows - (int64_t)base;
      const int64_t n_ok = room <= 0 ? 0 : (room < (int64_t)cnt ? room : (int64_t)cnt);
      uint64_t* dst = exchange_region(x.peer_base[o], x.n_ranks, x.parity, x.rank, x.region_rows, rw) + base * rw;
      const uint64_t* from = s_rows + (size_t)s_off[o] * rw;
      for (int64_t j = threadIdx.x; j < n_ok * rw; j += blockDim.x) dst[j] = from[j];
    }
    __syncthreads();
  }
  // publish: the last CTA to finish writes the row counts and then the completion flags
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(x.done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (s_last && threadIdx.x < x.n_ranks) {
    __threadfence_system();
    const unsigned long long cnt = atomicAdd(&x.cursors[threadIdx.x], 0ULL);
    ExchangeHeader* h = reinterpret_cast<ExchangeHeader*>(x.peer_base[threadIdx.x]);
    const bool over = (int64_t)cnt > x.region_rows;
    h->count[x.parity][x.rank] = over ? (unsigned long long)x.region_rows : cnt;
    if (over) h->overflow[x.parity][x.rank] = x.epoch;
    __threadfence_system();
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&h->flag[x.rank]), "l"(x.epoch) : "memory");
  }
}

struct ExchangeMergeParams {
  TableDev dst;
  WordKinds kinds;
  void* base;  // this rank's receive buffer
  unsigned long long* status;  // [0] != 0: timed out waiting for a peer; [1] != 0: a region overflowed;
                               // [2] nanoseconds the wait kernel spent until every source had released
  int64_t region_rows;
  unsigned long long epoch;
  long long spin_limit_ns;
  int32_t n_ranks, row_words, parity, pad;
};
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// One warp waits until every source has released its region for this epoch (one lane per
// source, acquire loads at system scope on flags in LOCAL memory that the peers store to over
// NVLink).  A separate 1-CTA kernel in front of the merge: nothing else spins, the merge grid
// starts only when its input is complete, and a peer that never arrives costs `spin_limit_ns`,
// not a hung GPU.
__global__ void __launch_bounds__(32) exchange_wait_kernel(const __grid_constant__ ExchangeMergeParams x) {
  ExchangeHeader* h = reinterpret_cast<ExchangeHeader*>(x.base);
  const unsigned long long t0 = globaltimer_ns();
  bool fail = false;
  if ((int)threadIdx.x < x.n_ranks) {
    while (true) {
      unsigned long long f;
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(f) : "l"(&h->flag[threadIdx.x]) : "memory");
      if (f >= x.epoch) break;
      if ((long long)(globaltimer_ns() - t0) > x.spin_limit_ns) { fail = true; break; }
      __nanosleep(100);
    }
    if (!fail && h->overflow[x.parity][threadIdx.x] == x.epoch) atomicExch(&x.status[1], 1ULL);
  }
  const unsigned any_fail = __ballot_sync(0xffffffffu, fail);
  if (threadIdx.x == 0) {
    if (any_fail) atomicExch(&x.status[0], 1ULL);
    x.status[2] = globaltimer_ns() - t0;
  }
}
// TransformFinalAggregate over the received regions (transform_aggregate_final.rs:201-303):
// every row of every source is found-or-inserted in the final table and its words merged.
__global__ void __launch_bounds__(256) exchange_merge_kernel(const __grid_constant__ ExchangeMergeParams x) {
  const ExchangeHeader* h = reinterpret_cast<const ExchangeHeader*>(x.base);
  if (*reinterpret_cast<volatile unsigned long long*>(&x.status[0])) return;  // a peer never arrived: reported by the host
  uint32_t new_groups = 0;
  for (int s = 0; s < x.n_ranks; ++s) {
    const int64_t cnt = (int64_t)h->count[x.parity][s];
    const uint64_t* rows = exchange_region(x.base, x.n_ranks, x.parity, s, x.region_rows, x.row_words);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (int64_t)gridDim.x * blockDim.x) {
      const uint64_t* r = rows + i * x.row_words;
      int64_t d = resolve_slot(x.dst, r[0], (int)r[1], new_groups);
      if (d < 0) { atomicAdd(x.dst.n_overflow, 1ULL); continue; }
      for (int w = 0; w < x.dst.n_words; ++w) merge_word(x.kinds.op[w], word_ptr(x.dst, d, w), r[2 + w]);
    }
  }
  __syncwarp();
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) new_groups += __shfl_xor_sync(0xffffffffu, new_groups, o);
  if ((threadIdx.x & 31) == 0 && new_groups) atomicAdd(x.dst.n_groups, (unsigned long long)new_groups);
}

// ---------------------------------------------------------------- finalize
// AggregateHashTable::merge_result -> batch_merge_result (aggregate_hashtable.rs:382-408):
// compacts the table into dense output columns [aggs..., keys...] (payload.rs:284-286).
struct FinalAgg {
  int32_t kind;       // dbx_agg_kind
  int32_t acc_word;   // sum/avg/min/max accumulator word (-1: none)
  int32_t cnt_word;   // word holding the number of non-NULL inputs
  int32_t arg_dtype;  // dbx_dtype of the argument (decides result type / narrowing)
  void* out;          // result values (8 B each except min/max of narrow types)
  uint8_t* out_valid; // one byte per group (packed to a bitmap afterwards); nullptr for count
};
struct FinalizeParams {
  FinalAgg aggs[DBX_MAX_AGGS];
  int32_t n_aggs;
  int32_t key_dtype;      // -1: no key output
  void* out_key;
  uint8_t* out_key_valid; // byte per group or nullptr
  // packed multi-column keys (n_key_parts > 1): one output column per part
  int32_t n_key_parts;
  int32_t pad;
  KeyPartDev key_parts[DBX_MAX_GROUP_COLS];
  void* out_keys[DBX_MAX_GROUP_COLS];
  uint8_t* out_keys_valid[DBX_MAX_GROUP_COLS];
  unsigned long long* out_count;
  int64_t out_capacity;   // rows the output columns can hold
};

__device__ __forceinline__ void store_narrow(void* out, int64_t idx, int dtype, uint64_t bits) {
  if (dtype == DBX_I8 || dtype == DBX_U8) ((uint8_t*)out)[idx] = (uint8_t)bits;
  else if (dtype == DBX_I16 || dtype == DBX_U16) ((uint16_t*)out)[idx] = (uint16_t)bits;
  else if (dtype == DBX_I32 || dtype == DBX_U32) ((uint32_t*)out)[idx] = (uint32_t)bits;
  else if (dtype == DBX_F32) ((float*)out)[idx] = (float)__longlong_as_double((long long)bits);
  else ((uint64_t*)out)[idx] = bits;
}

__global__ void __launch_bounds__(256) table_finalize_kernel(const __grid_constant__ TableDev src, const __grid_constant__ FinalizeParams fp) {
  __shared__ unsigned int s_warp_cnt[8];
  __shared__ unsigned long long s_block_base;
  const int64_t n_slots = src.cap + 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n_iter = (n_slots + stride - 1) / stride;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t it = 0; it < n_iter; ++it) {
    int64_t i = it * stride + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t key = kEmptyKey, key_hi = kEmptyKey;
    if (i < n_slots) {
      if (src.key_words == 2) {
        key = src.keys[2 * i]; key_hi = src.keys[2 * i + 1];
        if (i == src.cap && key != kEmptyKey) key = key_hi = kEmptyKey ^ 1;  // occupied marker, values restored below
        else if (i > src.cap) key = key_hi = kEmptyKey;
      } else key = src.keys[i];
    }
    bool occ = src.key_words == 2 ? !(key == kEmptyKey && key_hi == kEmptyKey) : key != kEmptyKey;
    // output slot allocation: one atomic per CTA and step (warp ballots + an 8-entry scan)
    const unsigned ballot = __ballot_sync(0xffffffffu, occ);
    if (lane == 0) s_warp_cnt[warp] = __popc(ballot);
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int tot = 0;
      for (int w = 0; w < 8; ++w) { const unsigned int c = s_warp_cnt[w]; s_warp_cnt[w] = tot; tot += c; }
      s_block_base = tot ? atomicAdd(fp.out_count, (unsigned long long)tot) : 0ULL;
    }
    __syncthreads();
    const unsigned long long base = s_block_base + s_warp_cnt[warp];
    __syncthreads();
    if (!occ) continue;
    int64_t o = (int64_t)base + __popc(ballot & ((1u << lane) - 1));
    if (o >= fp.out_capacity) continue;  // the host re-runs with a larger output (never silently)
    int key_kind = i >= src.cap ? (int)(i - src.cap) + 1 : 0;
    if (fp.n_key_parts > 1) {
      const uint64_t kb = key_kind == 1 ? kEmptyKey : key;
      const uint64_t kb_hi = key_kind == 1 ? kEmptyKey : key_hi;  // 128-bit keys only
      for (int j = 0; j < fp.n_key_parts; ++j) {
        const KeyPartDev kp = fp.key_parts[j];
        const uint64_t w = (kp.shift >> 6) ? kb_hi : kb;
        const bool is_null = kp.null_shift >= 0 && ((w >> (kp.null_shift & 63)) & 1);
        store_narrow(fp.out_keys[j], o, kp.dtype, is_null ? 0 : ((w >> (kp.shift & 63)) & kp.mask));
        if (fp.out_keys_valid[j]) fp.out_keys_valid[j][o] = is_null ? 0 : 1;
      }
    } else if (fp.key_dtype >= 0) {
      uint64_t kb = key_kind == 1 ? kEmptyKey : (key_kind == 2 ? 0 : key);
      store_narrow(fp.out_key, o, fp.key_dtype, kb);
      if (fp.out_key_valid) fp.out_key_valid[o] = key_kind == 2 ? 0 : 1;
    }
    for (int a = 0; a < fp.n_aggs; ++a) {
      const FinalAgg& fa = fp.aggs[a];
      uint64_t cnt = *word_ptr(src, i, fa.cnt_word);
      uint64_t acc = fa.acc_word >= 0 ? *word_ptr(src, i, fa.acc_word) : 0;
      int cls = dtype_class(fa.arg_dtype);
      if (fa.kind == DBX_AGG_COUNT) ((uint64_t*)fa.out)[o] = cnt;
      else if (fa.kind == DBX_AGG_SUM) ((uint64_t*)fa.out)[o] = cnt ? acc : 0;
      else if (fa.kind == DBX_AGG_AVG) {  // aggregate_avg.rs:88-96: value as f64 / count as f64
        double num = cls == VC_FLT ? __longlong_as_double((long long)acc)
                                   : (cls == VC_INT ? (double)(int64_t)acc : (double)acc);
        ((double*)fa.out)[o] = cnt ? num / (double)cnt : 0.0;
      } else {  // min / max keep the argument type
        uint64_t bits = acc;
        if (cls == VC_FLT) bits = (uint64_t)__double_as_longlong(ordered_to_f64(acc));
        store_narrow(fa.out, o, fa.arg_dtype, cnt ? bits : 0);
      }
      if (fa.out_valid) fa.out_valid[o] = cnt ? 1 : 0;
    }
  }
}

// ---------------------------------------------------------------- spill_schema serde of partial states
// AggregatorParams::spill_schema (aggregator_params.rs:103-117): one Tuple column `agg_i` per
// aggregate function holding its serialised state (StateSerde::serialize_type), then the group
// columns.  The C-ABI carries every tuple FLATTENED into consecutive columns; the fields are
//   count(..)            [UInt64 count]                                   aggregate_count.rs:170-172
//   sum(T)               [TSum value]                                     aggregate_sum.rs:155-157
//   avg(T)               [TSum sum, UInt64 count]                         aggregate_avg.rs:106-111
//   min(T) / max(T)      [Boolean has_value, T value]                     aggregate_min_max_any.rs:315-321
// followed, for every function but count, by one Boolean per wrapping adaptor: the null adaptor of a
// Nullable argument (aggregate_null_adaptor.rs:508-517) and the or-null adaptor every non-count
// function gets (aggregate_ornull_adaptor.rs:184-190, aggregate_function_factory.rs:219-249); both
// flags are "a non-NULL input was seen".  Rows come from / go to the fixed-width exchange rows
// [key][key kind][state words...] (table_partition_scatter_kernel / rows_merge_kernel).
constexpr int kMaxSpillFields = 5 * DBX_MAX_AGGS;
enum SpillFieldKind : int32_t { SPF_CNT = 0, SPF_ACC = 1, SPF_FLAG = 2, SPF_VALUE = 3 };
struct SpillFieldDev {
  int32_t kind;      // SpillFieldKind
  int32_t word;      // SPF_ACC / SPF_VALUE: accumulator word; SPF_CNT / SPF_FLAG: counter word
  int32_t cnt_word;  // word holding the number of non-NULL inputs (gates SPF_VALUE / SPF_ACC defaults)
  int32_t dtype;     // SPF_VALUE: argument dtype (narrow store, floats leave the ordered image)
  void* out;         // 8 B per row (CNT / ACC), dtype-wide (VALUE), 1 byte per row (FLAG; packed afterwards)
};
struct SpillOutParams {
  SpillFieldDev f[kMaxSpillFields];
  int32_t n_fields, row_words;
  int32_t key_dtype, n_key_parts;  // key_dtype -1: no group columns
  void* out_key;
  uint8_t* out_key_valid;
  KeyPartDev key_parts[DBX_MAX_GROUP_COLS];
  void* out_keys[DBX_MAX_GROUP_COLS];
  uint8_t* out_keys_valid[DBX_MAX_GROUP_COLS];
};

__global__ void __launch_bounds__(256) rows_to_spill_kernel(const uint64_t* rows, int64_t n, const __grid_constant__ SpillOutParams sp) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t* row = rows + r * sp.row_words;
    const uint64_t key = row[0];
    const int key_kind = (int)row[1];
    if (sp.n_key_parts > 1) {
      const uint64_t kb = key_kind == 1 ? kEmptyKey : key;
      for (int j = 0; j < sp.n_key_parts; ++j) {
        const KeyPartDev kp = sp.key_parts[j];
        const bool is_null = kp.null_shift >= 0 && ((kb >> kp.null_shift) & 1);
        store_narrow(sp.out_keys[j], r, kp.dtype, is_null ? 0 : ((kb >> kp.shift) & kp.mask));
        if (sp.out_keys_valid[j]) sp.out_keys_valid[j][r] = is_null ? 0 : 1;
      }
    } else if (sp.key_dtype >= 0) {
      store_narrow(sp.out_key, r, sp.key_dtype, key_kind == 1 ? kEmptyKey : (key_kind == 2 ? 0 : key));
      if (sp.out_key_valid) sp.out_key_valid[r] = key_kind == 2 ? 0 : 1;
    }
    for (int i = 0; i < sp.n_fields; ++i) {
      const SpillFieldDev& f = sp.f[i];
      const uint64_t w = row[2 + f.word];
      const uint64_t cnt = row[2 + f.cnt_word];
      if (f.kind == SPF_CNT) ((uint64_t*)f.out)[r] = w;
      else if (f.kind == SPF_ACC) ((uint64_t*)f.out)[r] = cnt ? w : 0;
      else if (f.kind == SPF_FLAG) ((uint8_t*)f.out)[r] = w ? 1 : 0;
      else {
        uint64_t bits = w;
        if (dtype_class(f.dtype) == VC_FLT) bits = (uint64_t)__double_as_longlong(ordered_to_f64(w));
        store_narrow(f.out, r, f.dtype, cnt ? bits : 0);
      }
    }
  }
}

// 64-bit image of row r of a numeric / boolean column as the table kernels widen it
__device__ __forceinline__ uint64_t column_image(const DevCol& c, int64_t r) {
  const char* b = (const char*)c.data;
  switch (c.dtype) {
    case DBX_I64: case DBX_U64: case DBX_F64: return ((const uint64_t*)b)[r];
    case DBX_I32: return (uint64_t)(int64_t)((const int32_t*)b)[r];
    case DBX_U32: return ((const uint32_t*)b)[r];
    case DBX_F32: return f32_bits_to_f64_bits(((const uint32_t*)b)[r]);
    case DBX_I16: return (uint64_t)(int64_t)((const int16_t*)b)[r];
    case DBX_U16: return ((const uint16_t*)b)[r];
    case DBX_I8: return (uint64_t)(int64_t)((const int8_t*)b)[r];
    case DBX_U8: return ((const uint8_t*)b)[r];
    case DBX_BOOL: return (uint64_t)bit_test((const uint8_t*)b, c.dbit_off + r);
    default: return 0;
  }
}
enum WordSrcMode : int32_t { WS_CNT_EXACT = 0, WS_CNT_FLAG = 1, WS_CNT_ONE = 2, WS_ACC_RAW = 3, WS_ACC_VALUE = 4 };
struct WordSrcDev {
  int32_t mode;
  int32_t col;       // input column of the value (CNT_EXACT / CNT_FLAG / ACC_*)
  int32_t flag_col;  // ACC_*: Boolean column saying the accumulator holds a value; -1: always
  int32_t pad;
  uint64_t init;     // identity of the word (what an accumulator without a value merges as)
};
struct SpillInParams {
  DevCol cols[kMaxSpillFields + DBX_MAX_GROUP_COLS];
  WordSrcDev w[kMaxWords];
  int32_t n_words, row_words;
  int32_t key_col, n_key_parts;  // key_col: first group column; -1: none
  int32_t key_is_float, pad;
  KeyPartDev key_parts[DBX_MAX_GROUP_COLS];  // .slot = input column index here
};
__global__ void __launch_bounds__(256) spill_to_rows_kernel(const __grid_constant__ SpillInParams sp, int64_t n, uint64_t* rows) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    uint64_t* row = rows + r * sp.row_words;
    uint64_t key = 0;
    int key_kind = 0;
    if (sp.n_key_parts > 1) {
      for (int j = 0; j < sp.n_key_parts; ++j) {
        const KeyPartDev kp = sp.key_parts[j];
        const DevCol& c = sp.cols[kp.slot];
        const bool ok = !c.validity || bit_test(c.validity, c.vbit_off + r);
        if (ok) key |= (column_image(c, r) & kp.mask) << kp.shift;
        else key |= 1ULL << kp.null_shift;
      }
      if (key == kEmptyKey) { key = 0; key_kind = 1; }
    } else if (sp.key_col >= 0) {
      const DevCol& c = sp.cols[sp.key_col];
      const bool ok = !c.validity || bit_test(c.validity, c.vbit_off + r);
      key = ok ? column_image(c, r) : 0;
      if (ok && sp.key_is_float) key = canonical_float_key(key);
      if (!ok) key_kind = 2;
      else if (key == kEmptyKey) { key = 0; key_kind = 1; }
    }
    row[0] = key;
    row[1] = (uint64_t)key_kind;
    for (int w = 0; w < sp.n_words; ++w) {
      const WordSrcDev ws = sp.w[w];
      uint64_t v;
      if (ws.mode == WS_CNT_ONE) v = 1;
      else if (ws.mode == WS_CNT_EXACT) v = column_image(sp.cols[ws.col], r);
      else if (ws.mode == WS_CNT_FLAG) v = column_image(sp.cols[ws.col], r) ? 1 : 0;
      else {
        const bool has = ws.flag_col < 0 || column_image(sp.cols[ws.flag_col], r) != 0;
        if (!has) v = ws.init;
        else {
          v = column_image(sp.cols[ws.col], r);
          if (ws.mode == WS_ACC_VALUE && dtype_class(sp.cols[ws.col].dtype) == VC_FLT) v = f64_to_ordered(__longlong_as_double((long long)v));
        }
      }
      row[2 + w] = v;
    }
  }
}
__global__ void pack_bytes_kernel(const uint8_t* bytes, int64_t n, uint8_t* bits) {
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

// bytes (0/1) -> LSB-first bitmap (MutableBitmap layout), one output byte per thread
__global__ void pack_validity_kernel(const uint8_t* bytes, const unsigned long long* n_dev, int64_t n_max, uint8_t* bits) {
  const int64_t n = min((int64_t)*n_dev, n_max);
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

#endif  // !DBX_JIT

}  // namespace dbx
