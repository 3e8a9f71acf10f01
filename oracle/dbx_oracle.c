/*
 * dbx_oracle.c — CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the reference's algorithms for the hot path, used ONLY by
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs as
 * the checker and the timed CPU baseline.  libdbx never links, loads or calls this file.
 *
 * The reference (Rust, nightly-2025-12-11) cannot be compiled in this environment, so this
 * is a "port" oracle.  It is pinned against the reference's own golden vectors
 * (tests/golden/ JSON files, extracted from the reference's testdata with file:line citations)
 * by tests/test_oracle_golden.py.
 *
 * Each function cites the reference file:line it follows (paths relative to the databend source tree).
 *
 * Third-party arithmetic restated from its published algorithm (not vendored in the reference):
 *   ndarray 0.15.6 (Cargo.lock) `numeric_util::unrolled_fold` — 8 interleaved partial sums —
 *   used by cosine_distance via `(&a * &b).sum()` (src/common/vector/src/distance.rs:28-34).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif
#if defined(__SSE4_2__)
#include <nmmintrin.h>
#endif

#include "../include/dbx.h"
#include "dbx_oracle.h"

/* ------------------------------------------------------------------ helpers */

static inline int bit_get(const uint8_t* bits, int64_t i) { return (bits[i >> 3] >> (i & 7)) & 1; }

static inline int col_valid(const dbx_column* c, int64_t row) {
  if (c->is_const) return !c->konst.is_null;
  if (!c->validity) return 1;
  return bit_get(c->validity, c->validity_bit_offset + row);
}

typedef enum { VC_INT = 0, VC_UINT = 1, VC_FLT = 2 } vclass;
typedef struct {
  vclass cls;
  int64_t i;
  uint64_t u;
  double f;
} val;

static inline vclass dtype_class(int32_t dt) {
  switch (dt) {
    case DBX_I8: case DBX_I16: case DBX_I32: case DBX_I64: return VC_INT;
    case DBX_BOOL: case DBX_U8: case DBX_U16: case DBX_U32: case DBX_U64: return VC_UINT;
    default: return VC_FLT;
  }
}

static inline val scalar_val(const dbx_scalar* s) {
  val v;
  v.cls = dtype_class(s->dtype);
  v.i = s->v.i64;
  v.u = s->v.u64;
  v.f = s->v.f64;
  if (v.cls == VC_INT) { v.u = (uint64_t)v.i; v.f = (double)v.i; }
  else if (v.cls == VC_UINT) { v.i = (int64_t)v.u; v.f = (double)v.u; }
  return v;
}

static inline val col_val(const dbx_column* c, int64_t row) {
  val v;
  if (c->is_const) return scalar_val(&c->konst);
  v.cls = dtype_class(c->dtype);
  v.i = 0; v.u = 0; v.f = 0;
  switch (c->dtype) {
    case DBX_BOOL: v.u = (uint64_t)bit_get((const uint8_t*)c->data, c->data_bit_offset + row); break;
    case DBX_I8: v.i = ((const int8_t*)c->data)[row]; break;
    case DBX_I16: v.i = ((const int16_t*)c->data)[row]; break;
    case DBX_I32: v.i = ((const int32_t*)c->data)[row]; break;
    case DBX_I64: v.i = ((const int64_t*)c->data)[row]; break;
    case DBX_U8: v.u = ((const uint8_t*)c->data)[row]; break;
    case DBX_U16: v.u = ((const uint16_t*)c->data)[row]; break;
    case DBX_U32: v.u = ((const uint32_t*)c->data)[row]; break;
    case DBX_U64: v.u = ((const uint64_t*)c->data)[row]; break;
    case DBX_F32: v.f = ((const float*)c->data)[row]; break;
    case DBX_F64: v.f = ((const double*)c->data)[row]; break;
    default: break;
  }
  if (v.cls == VC_INT) { v.u = (uint64_t)v.i; v.f = (double)v.i; }
  else if (v.cls == VC_UINT) { v.i = (int64_t)v.u; v.f = (double)v.u; }
  return v;
}

/* ------------------------------------------------------------------ modulo */
/* arithmetic_modulo.rs:72-97 (push_modulo_result): rhs == 0 -> per-row error "Division by
 * zero"; signed MIN % -1 -> 0; else Rust `%` (truncated: sign of the dividend) computed in
 * the LeastSuper type (numeric_basic_arithmetic.rs:492-522), i.e. i64 / u64 / f64 here.   */
static inline int modulo_val(val a, val b, val* out) {
  if (a.cls == VC_FLT || b.cls == VC_FLT) {
    if (b.f == 0.0) return 1;
    out->cls = VC_FLT;
    out->f = fmod(a.f, b.f); /* Rust f64 % = C fmod */
    return 0;
  }
  if (a.cls == VC_UINT && b.cls == VC_UINT) {
    if (b.u == 0) return 1;
    out->cls = VC_UINT;
    out->u = a.u % b.u;
    out->i = (int64_t)out->u;
    out->f = (double)out->u;
    return 0;
  }
  /* any signed operand: LeastSuper is a signed integer (u64 mixed with signed is F64 in the
   * reference, arithmetics_type.rs; not reachable from the configs, computed in i64 here) */
  if ((b.cls == VC_INT && b.i == 0) || (b.cls == VC_UINT && b.u == 0)) return 1;
  {
    int64_t x = a.cls == VC_INT ? a.i : (int64_t)a.u;
    int64_t y = b.cls == VC_INT ? b.i : (int64_t)b.u;
    out->cls = VC_INT;
    if (x == INT64_MIN && y == -1) out->i = 0; /* is_signed_min_modulo_minus_one */
    else out->i = x % y;                       /* C99 % truncates like Rust */
    out->u = (uint64_t)out->i;
    out->f = (double)out->i;
  }
  return 0;
}

/* OrderedFloat total order (src/common/base/src/base/ordered_float.rs:147-201):
 * NaN is the greatest value and all NaNs are equal; -0 == +0. Returns -1/0/1. */
static inline int ordered_cmp_f64(double a, double b) {
  int an = isnan(a), bn = isnan(b);
  if (an || bn) return an == bn ? 0 : (an ? 1 : -1);
  return a < b ? -1 : (a > b ? 1 : 0);
}

static inline int cmp_val(val a, val b) {
  if (a.cls == VC_FLT || b.cls == VC_FLT) return ordered_cmp_f64(a.f, b.f);
  if (a.cls == VC_INT && b.cls == VC_INT) return a.i < b.i ? -1 : (a.i > b.i ? 1 : 0);
  if (a.cls == VC_UINT && b.cls == VC_UINT) return a.u < b.u ? -1 : (a.u > b.u ? 1 : 0);
  if (a.cls == VC_INT) { /* int vs uint */
    if (a.i < 0) return -1;
    return (uint64_t)a.i < b.u ? -1 : ((uint64_t)a.i > b.u ? 1 : 0);
  }
  if (b.i < 0) return 1;
  return a.u < (uint64_t)b.i ? -1 : (a.u > (uint64_t)b.i ? 1 : 0);
}

static inline int apply_cmp(int op, int c) {
  switch (op) {
    case DBX_EQ: return c == 0;
    case DBX_NE: return c != 0;
    case DBX_LT: return c < 0;
    case DBX_LE: return c <= 0;
    case DBX_GT: return c > 0;
    default: return c >= 0;
  }
}

/* Evaluate one operand for one row. Returns 0 ok, 1 NULL, 2 division by zero. */
static inline int eval_operand(const dbx_block* blk, const dbx_operand* o, int64_t row, val* out) {
  if (o->is_const) {
    if (o->c.is_null) return 1;
    *out = scalar_val(&o->c);
    return 0;
  }
  const dbx_column* c = &blk->cols[o->col];
  if (!col_valid(c, row)) return 1; /* passthrough_nullable */
  *out = col_val(c, row);
  if (o->arith == DBX_ARITH_MODULO) {
    if (o->c.is_null) return 1;
    val r;
    if (modulo_val(*out, scalar_val(&o->c), &r)) return 2;
    *out = r;
  }
  return 0;
}

/* ------------------------------------------------------------------ filter */
/* FilterExecutor::select (filter_executor.rs:106-116) -> Selector::select over the
 * SelectExpr tree (selector.rs:64-180): AND = every child true, OR = any child true,
 * Compare = select_column_scalar (select_value/select_column_scalar.rs:27-140) where a NULL
 * on either side is "not selected". Row-at-a-time restatement: the result (ascending
 * true_selection) is identical. */
static int eval_pred_row(const dbx_block* blk, const dbx_predicate* p, int64_t row, int* divzero) {
  int stack[DBX_MAX_PRED_NODES];
  int sp = 0;
  for (int n = 0; n < p->n_nodes; ++n) {
    const dbx_pred_node* nd = &p->nodes[n];
    switch (nd->kind) {
      case DBX_PRED_CMP: {
        val a, b;
        int ra = eval_operand(blk, &nd->lhs, row, &a);
        int rb = eval_operand(blk, &nd->rhs, row, &b);
        if (ra == 2 || rb == 2) { *divzero = 1; stack[sp++] = 0; break; }
        if (ra || rb) { stack[sp++] = 0; break; }
        stack[sp++] = apply_cmp(nd->cmp, cmp_val(a, b));
        break;
      }
      case DBX_PRED_AND: {
        int r = 1;
        for (int k = 0; k < nd->n_children; ++k) r &= stack[--sp];
        stack[sp++] = r;
        break;
      }
      case DBX_PRED_OR: {
        int r = 0;
        for (int k = 0; k < nd->n_children; ++k) r |= stack[--sp];
        stack[sp++] = r;
        break;
      }
      case DBX_PRED_BOOLCOL: {
        const dbx_column* c = &blk->cols[nd->value];
        stack[sp++] = col_valid(c, row) && col_val(c, row).u != 0;
        break;
      }
      default: stack[sp++] = nd->value != 0; break;
    }
  }
  return sp ? stack[sp - 1] : 1;
}

int orc_filter_select(const dbx_block* blk, const dbx_predicate* pred, uint32_t* sel, int64_t* n_sel,
                      int64_t* err_row) {
  int64_t n = 0;
  *err_row = -1;
  for (int64_t r = 0; r < blk->num_rows; ++r) {
    int dz = 0;
    int pass = eval_pred_row(blk, pred, r, &dz);
    if (dz) { /* evaluator.rs:234-244: the first failing row aborts the expression */
      *err_row = r;
      *n_sel = 0;
      return DBX_ERR_BAD_ARGUMENTS;
    }
    /* select_column_scalar.rs:118-131: branch-free  sel[n] = idx; n += ret */
    sel[n] = (uint32_t)r;
    n += pass;
  }
  *n_sel = n;
  return DBX_OK;
}

static size_t dtype_size(int32_t dt) {
  switch (dt) {
    case DBX_I8: case DBX_U8: return 1;
    case DBX_I16: case DBX_U16: return 2;
    case DBX_I32: case DBX_U32: case DBX_F32: return 4;
    default: return 8;
  }
}

/* DataBlock::take (kernels/take.rs:43-60,255): gather rows by u32 index; validity gathered
 * bit by bit.  out_data holds n_sel elements, out_valid one BYTE per row (1 = valid). */
int orc_take_column(const dbx_column* c, const uint32_t* sel, int64_t n_sel, void* out_data, uint8_t* out_valid) {
  size_t w = dtype_size(c->dtype);
  if (c->dtype == DBX_BOOL || c->dtype == DBX_VEC_F32) return DBX_ERR_UNSUPPORTED;
  for (int64_t i = 0; i < n_sel; ++i) {
    int64_t r = sel[i];
    if (c->is_const) {
      val v = scalar_val(&c->konst);
      switch (c->dtype) {
        case DBX_F32: ((float*)out_data)[i] = (float)v.f; break;
        case DBX_F64: ((double*)out_data)[i] = v.f; break;
        default: memcpy((char*)out_data + i * w, &v.u, w); break; /* little-endian truncation */
      }
    } else {
      memcpy((char*)out_data + i * w, (const char*)c->data + r * w, w);
    }
    if (out_valid) out_valid[i] = (uint8_t)col_valid(c, r);
  }
  return DBX_OK;
}

/* ------------------------------------------------------------------ group hash */
/* group_hash.rs:555-570 (impl_agg_hash_for_primitive_types) */
uint64_t orc_agg_hash_u64(uint64_t x) {
  x ^= x >> 32;
  x *= 0xd6e8feb86659fd93ULL;
  x ^= x >> 32;
  x *= 0xd6e8feb86659fd93ULL;
  x ^= x >> 32;
  return x;
}
#define ORC_NULL_HASH_VAL 0xd1cefa08eb382d69ULL /* group_hash.rs:38 */

/* key word of one group column for one row: the value `as u64` (sign-extended for signed
 * ints, group_hash.rs:559 `*self as u64`; floats hash their canonical-NaN bits, :599-619). */
static inline uint64_t key_word(const dbx_column* c, int64_t row) {
  val v = col_val(c, row);
  if (v.cls == VC_FLT) {
    if (c->dtype == DBX_F32) {
      float f = (float)v.f;
      uint32_t b;
      if (isnan(f)) f = NAN;
      memcpy(&b, &f, 4);
      return b;
    } else {
      double d = v.f;
      uint64_t b;
      if (isnan(d)) d = NAN;
      memcpy(&b, &d, 8);
      return b;
    }
  }
  return v.u;
}

/* group_hash_entries (group_hash.rs:40-62) + combine (:267-282): first column h = agg_hash,
 * later columns h = h * NULL_HASH_VAL ^ agg_hash; NULL hashes to NULL_HASH_VAL (:177-205). */
static inline uint64_t group_hash_row(const dbx_block* blk, const dbx_agg_params* p, int64_t row, uint64_t* words,
                                      uint8_t* valids) {
  uint64_t h = 0;
  for (int g = 0; g < p->n_group_cols; ++g) {
    const dbx_column* c = &blk->cols[p->group_cols[g]];
    int ok = col_valid(c, row);
    uint64_t w = ok ? key_word(c, row) : 0;
    uint64_t hi = ok ? orc_agg_hash_u64(w) : ORC_NULL_HASH_VAL;
    words[g] = w;
    valids[g] = (uint8_t)ok;
    h = g == 0 ? hi : (h * ORC_NULL_HASH_VAL) ^ hi;
  }
  return h;
}

/* ------------------------------------------------------------------ aggregate states */
/* One state per (group, aggregate), restating
 *   NumberSumState{value}                 aggregate_sum.rs:41-45,106-111   (value += v as TSum, wrapping: Cargo.toml:577)
 *   AggregateCountFunction state {count}  aggregate_count.rs:52-54,123-157
 *   NumberAvgState{value,count}           aggregate_avg.rs:54-104
 *   min/max scalar states                 aggregate_min_max_any.rs (value + has-value)
 *   OrNull flag ("had a non-NULL input")  adaptors/aggregate_ornull_adaptor.rs:41-140
 * TSum: unsigned -> u64, signed -> i64, float -> f64 (arithmetics_type.rs:844-1071).       */
typedef struct {
  union { int64_t i; uint64_t u; double f; } acc;
  uint64_t count; /* non-NULL inputs seen: avg divisor, count result, OrNull flag (count>0) */
} agg_state;

static inline void state_init(agg_state* s) { s->acc.u = 0; s->count = 0; }

static inline void state_add(agg_state* s, int kind, vclass cls, val v) {
  switch (kind) {
    case DBX_AGG_SUM:
    case DBX_AGG_AVG:
      if (cls == VC_FLT) s->acc.f += v.f;
      else s->acc.u += v.u; /* two's complement wrapping add == i64 wrapping add */
      break;
    case DBX_AGG_MIN:
      if (s->count == 0) { if (cls == VC_FLT) s->acc.f = v.f; else s->acc.u = v.u; }
      else if (cls == VC_FLT) { if (ordered_cmp_f64(v.f, s->acc.f) < 0) s->acc.f = v.f; }
      else if (cls == VC_INT) { if (v.i < s->acc.i) s->acc.i = v.i; }
      else { if (v.u < s->acc.u) s->acc.u = v.u; }
      break;
    case DBX_AGG_MAX:
      if (s->count == 0) { if (cls == VC_FLT) s->acc.f = v.f; else s->acc.u = v.u; }
      else if (cls == VC_FLT) { if (ordered_cmp_f64(v.f, s->acc.f) > 0) s->acc.f = v.f; }
      else if (cls == VC_INT) { if (v.i > s->acc.i) s->acc.i = v.i; }
      else { if (v.u > s->acc.u) s->acc.u = v.u; }
      break;
    default: break; /* count: only the counter */
  }
  s->count += 1;
}

/* batch_merge_states / merge (aggregate_sum.rs:126-129, aggregate_avg.rs:82-86) */
static inline void state_merge(agg_state* d, const agg_state* s, int kind, vclass cls) {
  if (s->count == 0) return;
  switch (kind) {
    case DBX_AGG_SUM:
    case DBX_AGG_AVG:
      if (cls == VC_FLT) d->acc.f += s->acc.f; else d->acc.u += s->acc.u;
      break;
    case DBX_AGG_MIN:
    case DBX_AGG_MAX: {
      val v; v.cls = cls; v.i = s->acc.i; v.u = s->acc.u; v.f = s->acc.f;
      uint64_t keep = d->count;
      state_add(d, kind, cls, v);
      d->count = keep; /* count merged below */
      break;
    }
    default: break;
  }
  d->count += s->count;
}

/* ------------------------------------------------------------------ hash table */
/* Restates AggregateHashTable (aggregate_hashtable.rs:168-292) + HashIndex
 * (hash_index/index.rs:92-214): open addressing, slot = hash & mask, linear probing,
 * grows when count*LOAD_FACTOR(1.35) > capacity (aggregate/mod.rs:55).  The 7-bit tag /
 * 8-wide ctrl groups only accelerate the probe; the found-or-inserted slot is the same. */
typedef struct {
  int64_t cap, count;
  int32_t n_gc, n_aggs;
  int64_t* slot_group; /* cap entries: -1 empty else group index */
  uint64_t* hashes;    /* per group */
  uint64_t* kwords;    /* per group: n_gc words */
  uint8_t* kvalid;     /* per group: n_gc bytes */
  agg_state* states;   /* per group: n_aggs states */
  int64_t gcap;
} otable;

static void ot_init(otable* t, int n_gc, int n_aggs, int64_t cap) {
  t->cap = cap; t->count = 0; t->n_gc = n_gc; t->n_aggs = n_aggs;
  t->slot_group = (int64_t*)malloc(sizeof(int64_t) * cap);
  for (int64_t i = 0; i < cap; ++i) t->slot_group[i] = -1;
  t->gcap = 1024;
  t->hashes = (uint64_t*)malloc(sizeof(uint64_t) * t->gcap);
  t->kwords = (uint64_t*)malloc(sizeof(uint64_t) * t->gcap * (n_gc ? n_gc : 1));
  t->kvalid = (uint8_t*)malloc(t->gcap * (n_gc ? n_gc : 1));
  t->states = (agg_state*)malloc(sizeof(agg_state) * t->gcap * (n_aggs ? n_aggs : 1));
}
static void ot_free(otable* t) {
  free(t->slot_group); free(t->hashes); free(t->kwords); free(t->kvalid); free(t->states);
}
static void ot_resize(otable* t) { /* aggregate_hashtable.rs:463-489 */
  int64_t ncap = t->cap * 2;
  free(t->slot_group);
  t->slot_group = (int64_t*)malloc(sizeof(int64_t) * ncap);
  for (int64_t i = 0; i < ncap; ++i) t->slot_group[i] = -1;
  for (int64_t g = 0; g < t->count; ++g) {
    int64_t s = (int64_t)(t->hashes[g] & (uint64_t)(ncap - 1));
    while (t->slot_group[s] >= 0) s = (s + 1) & (ncap - 1);
    t->slot_group[s] = g;
  }
  t->cap = ncap;
}
static int64_t ot_find_or_insert(otable* t, uint64_t h, const uint64_t* words, const uint8_t* valids) {
  int n_gc = t->n_gc;
  if ((double)(t->count + 1) * 1.35 > (double)t->cap) ot_resize(t);
  int64_t mask = t->cap - 1;
  int64_t s = (int64_t)(h & (uint64_t)mask);
  for (;;) {
    int64_t g = t->slot_group[s];
    if (g < 0) break;
    if (t->hashes[g] == h) { /* row_match_entries (payload_row.rs:324-400) */
      int same = 1;
      for (int k = 0; k < n_gc; ++k)
        if (t->kvalid[g * n_gc + k] != valids[k] || (valids[k] && t->kwords[g * n_gc + k] != words[k])) { same = 0; break; }
      if (same) return g;
    }
    s = (s + 1) & mask;
  }
  if (t->count == t->gcap) {
    t->gcap *= 2;
    t->hashes = (uint64_t*)realloc(t->hashes, sizeof(uint64_t) * t->gcap);
    t->kwords = (uint64_t*)realloc(t->kwords, sizeof(uint64_t) * t->gcap * (n_gc ? n_gc : 1));
    t->kvalid = (uint8_t*)realloc(t->kvalid, t->gcap * (n_gc ? n_gc : 1));
    t->states = (agg_state*)realloc(t->states, sizeof(agg_state) * t->gcap * (t->n_aggs ? t->n_aggs : 1));
  }
  int64_t g = t->count++;
  t->slot_group[s] = g;
  t->hashes[g] = h;
  for (int k = 0; k < n_gc; ++k) { t->kwords[g * n_gc + k] = words[k]; t->kvalid[g * n_gc + k] = valids[k]; }
  for (int a = 0; a < t->n_aggs; ++a) state_init(&t->states[g * t->n_aggs + a]);
  return g;
}

/* ------------------------------------------------------------------ filter -> group-by */
#define ORC_BLOCK_ROWS 65536 /* max_block_size, settings_default.rs:142-143 */
#define ORC_RADIX_BITS 7     /* MAX_RADIX_BITS, aggregate/mod.rs:66-67 -> 128 buckets */

static vclass agg_arg_class(const dbx_block* blk, const dbx_agg_desc* a) {
  if (a->arg_col < 0) return VC_UINT;
  return dtype_class(blk->cols[a->arg_col].dtype);
}

/* One thread's TransformFilter -> TransformPartialAggregate::execute_one_block
 * (filter_predicate.rs:70-93, transform_aggregate_partial.rs:179-240) over rows [r0,r1). */
static int partial_rows(const dbx_block* blk, const dbx_agg_params* p, int64_t r0, int64_t r1, otable* t,
                        int64_t* err_row) {
  uint64_t words[DBX_MAX_GROUP_COLS];
  uint8_t valids[DBX_MAX_GROUP_COLS];
  for (int64_t r = r0; r < r1; ++r) {
    if (p->filter.n_nodes) {
      int dz = 0;
      int pass = eval_pred_row(blk, &p->filter, r, &dz);
      if (dz) { *err_row = r; return DBX_ERR_BAD_ARGUMENTS; }
      if (!pass) continue;
    }
    int64_t g;
    if (p->n_group_cols) {
      uint64_t h = group_hash_row(blk, p, r, words, valids);
      g = ot_find_or_insert(t, h, words, valids);
    } else {
      if (t->count == 0) g = ot_find_or_insert(t, 0, words, valids); else g = 0;
    }
    for (int a = 0; a < p->n_aggs; ++a) { /* accumulate_keys (aggregate_hashtable.rs:251-262) */
      const dbx_agg_desc* ad = &p->aggs[a];
      agg_state* s = &t->states[g * p->n_aggs + a];
      if (ad->arg_col < 0) { s->count += 1; continue; } /* count(*) */
      const dbx_column* c = &blk->cols[ad->arg_col];
      if (!col_valid(c, r)) continue;                     /* NULL inputs are skipped */
      state_add(s, ad->kind, dtype_class(c->dtype), col_val(c, r));
    }
  }
  return DBX_OK;
}

static void finalize_into(const dbx_block* blk, const dbx_agg_params* p, const otable* t, orc_agg_result* out,
                          int64_t base) {
  for (int64_t g = 0; g < t->count; ++g) {
    for (int k = 0; k < p->n_group_cols; ++k) {
      out->key_bits[k][base + g] = t->kwords[g * t->n_gc + k];
      out->key_valid[k][base + g] = t->kvalid[g * t->n_gc + k];
    }
    for (int a = 0; a < p->n_aggs; ++a) {
      const agg_state* s = &t->states[g * p->n_aggs + a];
      vclass cls = agg_arg_class(blk, &p->aggs[a]);
      uint64_t bits = 0;
      uint8_t ok = 1;
      switch (p->aggs[a].kind) {
        case DBX_AGG_COUNT: bits = s->count; ok = 1; break; /* aggregate_count.rs:66-70: never NULL */
        case DBX_AGG_AVG: {                                 /* aggregate_avg.rs:88-96 */
          double num = cls == VC_FLT ? s->acc.f : (cls == VC_INT ? (double)s->acc.i : (double)s->acc.u);
          double r = s->count ? num / (double)s->count : 0.0;
          memcpy(&bits, &r, 8);
          ok = s->count > 0;
          break;
        }
        default: bits = s->count ? s->acc.u : 0; ok = s->count > 0; break; /* OrNull: NULL iff no input */
      }
      out->agg_bits[a][base + g] = bits;
      out->agg_valid[a][base + g] = ok;
    }
  }
}

static int result_dtype(const dbx_block* blk, const dbx_agg_desc* a) {
  vclass cls = agg_arg_class(blk, a);
  switch (a->kind) {
    case DBX_AGG_COUNT: return DBX_U64;
    case DBX_AGG_AVG: return DBX_F64;
    case DBX_AGG_SUM: return cls == VC_FLT ? DBX_F64 : (cls == VC_INT ? DBX_I64 : DBX_U64);
    default: return blk->cols[a->arg_col].dtype; /* min/max keep the argument type */
  }
}

static void result_alloc(orc_agg_result* out, const dbx_block* blk, const dbx_agg_params* p, int64_t n) {
  memset(out, 0, sizeof(*out));
  out->n_groups = n;
  out->n_group_cols = p->n_group_cols;
  out->n_aggs = p->n_aggs;
  int64_t m = n ? n : 1;
  for (int k = 0; k < p->n_group_cols; ++k) {
    out->key_bits[k] = (uint64_t*)malloc(sizeof(uint64_t) * m);
    out->key_valid[k] = (uint8_t*)malloc(m);
  }
  for (int a = 0; a < p->n_aggs; ++a) {
    out->agg_bits[a] = (uint64_t*)malloc(sizeof(uint64_t) * m);
    out->agg_valid[a] = (uint8_t*)malloc(m);
    out->agg_dtype[a] = result_dtype(blk, &p->aggs[a]);
  }
}

void orc_agg_result_free(orc_agg_result* r) {
  for (int k = 0; k < DBX_MAX_GROUP_COLS; ++k) { free(r->key_bits[k]); free(r->key_valid[k]); }
  for (int a = 0; a < DBX_MAX_AGGS; ++a) { free(r->agg_bits[a]); free(r->agg_valid[a]); }
  memset(r, 0, sizeof(*r));
}

/* Two-phase group-by, structured like the reference pipeline:
 *   phase 1: `threads` TransformPartialAggregate instances pull 65 536-row blocks
 *            (physical_aggregate_partial.rs:223-235) into thread-local tables;
 *   phase 2: groups are radix-partitioned on hash bits (partitioned_payload.rs:44-57,
 *            build_partition_bucket.rs:75-121) and each bucket is merged by one
 *            TransformFinalAggregate (combine_payload + merge_result,
 *            aggregate_hashtable.rs:349-408).
 * threads <= 1 runs the same code on one thread. */
int orc_filter_group_agg(const dbx_block* blk, const dbx_agg_params* p, int threads, orc_agg_result* out,
                         int64_t* err_row) {
  if (threads < 1) threads = 1;
  *err_row = -1;
  int64_t n = blk->num_rows;
  int64_t n_blocks = (n + ORC_BLOCK_ROWS - 1) / ORC_BLOCK_ROWS;
  otable* parts = (otable*)malloc(sizeof(otable) * threads);
  for (int t = 0; t < threads; ++t) ot_init(&parts[t], p->n_group_cols, p->n_aggs, 1024);
  int status = DBX_OK;
  int64_t first_err = INT64_MAX;

#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int64_t b = 0; b < n_blocks; ++b) {
    int tid = 0;
#ifdef _OPENMP
    tid = omp_get_thread_num();
#endif
    int64_t r0 = b * ORC_BLOCK_ROWS, r1 = r0 + ORC_BLOCK_ROWS;
    if (r1 > n) r1 = n;
    int64_t er = -1;
    int st = partial_rows(blk, p, r0, r1, &parts[tid], &er);
    if (st != DBX_OK) {
#pragma omp critical
      { status = st; if (er < first_err) first_err = er; }
    }
  }
  if (status != DBX_OK) {
    for (int t = 0; t < threads; ++t) ot_free(&parts[t]);
    free(parts);
    *err_row = first_err;
    memset(out, 0, sizeof(*out));
    return status;
  }

  if (p->n_group_cols == 0) { /* FinalSingleStateAggregator (transform_single_key.rs:232-278) */
    otable fin;
    ot_init(&fin, 0, p->n_aggs, 1024);
    uint64_t w0 = 0; uint8_t v0 = 0;
    ot_find_or_insert(&fin, 0, &w0, &v0);
    for (int t = 0; t < threads; ++t)
      if (parts[t].count)
        for (int a = 0; a < p->n_aggs; ++a)
          state_merge(&fin.states[a], &parts[t].states[a], p->aggs[a].kind, agg_arg_class(blk, &p->aggs[a]));
    result_alloc(out, blk, p, 1);
    finalize_into(blk, p, &fin, out, 0);
    ot_free(&fin);
    for (int t = 0; t < threads; ++t) ot_free(&parts[t]);
    free(parts);
    return DBX_OK;
  }

  const int NB = 1 << ORC_RADIX_BITS;
  otable* finals = (otable*)malloc(sizeof(otable) * NB);
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int bkt = 0; bkt < NB; ++bkt) {
    otable* f = &finals[bkt];
    ot_init(f, p->n_group_cols, p->n_aggs, 1024);
    for (int t = 0; t < threads; ++t) {
      const otable* s = &parts[t];
      for (int64_t g = 0; g < s->count; ++g) {
        /* partition = hash bits [48-radix, 48) (partitioned_payload.rs:44-57) */
        if ((int)((s->hashes[g] >> (48 - ORC_RADIX_BITS)) & (NB - 1)) != bkt) continue;
        int64_t d = ot_find_or_insert(f, s->hashes[g], &s->kwords[g * s->n_gc], &s->kvalid[g * s->n_gc]);
        for (int a = 0; a < p->n_aggs; ++a)
          state_merge(&f->states[d * p->n_aggs + a], &s->states[g * p->n_aggs + a], p->aggs[a].kind,
                      agg_arg_class(blk, &p->aggs[a]));
      }
    }
  }
  int64_t total = 0;
  int64_t* base = (int64_t*)malloc(sizeof(int64_t) * NB);
  for (int b = 0; b < NB; ++b) { base[b] = total; total += finals[b].count; }
  result_alloc(out, blk, p, total);
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads)
  for (int b = 0; b < NB; ++b) finalize_into(blk, p, &finals[b], out, base[b]);
  for (int b = 0; b < NB; ++b) ot_free(&finals[b]);
  free(finals); free(base);
  for (int t = 0; t < threads; ++t) ot_free(&parts[t]);
  free(parts);
  return DBX_OK;
}

/* ------------------------------------------------------------------ hash join */
/* FastHash for u64 keys (src/common/hashtable/src/traits.rs:195-214): CRC32C(u64::MAX, k)
 * under SSE4.2 (a 32-bit hash), else the murmur3 finaliser. */
static inline uint64_t join_hash_u64(uint64_t k, int* bits) {
#if defined(__SSE4_2__)
  *bits = 32;
  return (uint64_t)_mm_crc32_u64(~0ULL, k);
#else
  *bits = 64;
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return k;
#endif
}

/* Inner hash join on one integer key column.
 * build: HashJoinHashTable::with_build_row_num + insert (hashjoin_hashtable.rs:95-141):
 *   capacity = max(next_pow2(2*rows), 1024); index = hash >> (hash_bits - log2 cap);
 *   each bucket heads a chain (newest first).  The 16-bit tag only skips chain walks.
 * probe: probe / next_matched (hashjoin_hashtable.rs:144-190, fixed_keys.rs:82-166): for every
 *   probe row walk the chain, comparing keys; emit (probe_idx, build_idx) per match.
 * NULL keys never match (fixed_keys.rs: build rows with NULL key are skipped via the
 * validity bitmap; probe rows with NULL key get pointer 0).
 * Output pairs are in probe order; within a probe row in chain order (LIFO of build order). */
int orc_hash_join_inner(const dbx_column* build_key, const dbx_column* probe_key, int64_t** out_probe_idx,
                        int64_t** out_build_idx, int64_t* n_out) {
  int64_t nb = build_key->len, np = probe_key->len;
  int64_t cap = 1024;
  while (cap < nb * 2) cap <<= 1;
  int lg = 0;
  while ((1LL << lg) < cap) ++lg;
  int hbits = 64;
  (void)join_hash_u64(0, &hbits);
  int shift = hbits - lg;
  int64_t* head = (int64_t*)malloc(sizeof(int64_t) * cap);
  int64_t* next = (int64_t*)malloc(sizeof(int64_t) * (nb ? nb : 1));
  for (int64_t i = 0; i < cap; ++i) head[i] = -1;
  for (int64_t r = 0; r < nb; ++r) {
    if (!col_valid(build_key, r)) { next[r] = -1; continue; }
    uint64_t k = key_word(build_key, r);
    uint64_t h = join_hash_u64(k, &hbits);
    int64_t idx = shift >= 64 ? 0 : (int64_t)(h >> shift);
    next[r] = head[idx];
    head[idx] = r;
  }
  int64_t ocap = np > 16 ? np : 16, no = 0;
  int64_t* op = (int64_t*)malloc(sizeof(int64_t) * ocap);
  int64_t* ob = (int64_t*)malloc(sizeof(int64_t) * ocap);
  for (int64_t r = 0; r < np; ++r) {
    if (!col_valid(probe_key, r)) continue;
    uint64_t k = key_word(probe_key, r);
    uint64_t h = join_hash_u64(k, &hbits);
    int64_t idx = shift >= 64 ? 0 : (int64_t)(h >> shift);
    for (int64_t e = head[idx]; e >= 0; e = next[e]) {
      if (key_word(build_key, e) != k) continue;
      if (no == ocap) {
        ocap *= 2;
        op = (int64_t*)realloc(op, sizeof(int64_t) * ocap);
        ob = (int64_t*)realloc(ob, sizeof(int64_t) * ocap);
      }
      op[no] = r; ob[no] = e; ++no;
    }
  }
  free(head); free(next);
  *out_probe_idx = op; *out_build_idx = ob; *n_out = no;
  return DBX_OK;
}

/* Probe-side ("left") join kinds on top of the same table walk
 * (new_hash_join/memory/left_join.rs, left_join_semi.rs, left_join_anti.rs):
 *   kind 0 INNER       every (probe, build) match
 *   kind 1 LEFT SEMI   probe rows with at least one match, once; build index -1
 *   kind 2 LEFT ANTI   probe rows with no match (a NULL key never matches); build index -1
 *   kind 3 LEFT        every match, plus (probe, -1) for probe rows with no match
 * Pairs come out in probe order (the reference's filter_with_bitmap keeps the probe order for
 * semi/anti; the unmatched rows of a LEFT join follow each probed block: unspecified order). */
int orc_hash_join(int kind, const dbx_column* build_key, const dbx_column* probe_key, int64_t** out_probe_idx,
                  int64_t** out_build_idx, int64_t* n_out) {
  int64_t *ip = NULL, *ib = NULL, ni = 0;
  int st = orc_hash_join_inner(build_key, probe_key, &ip, &ib, &ni);
  if (st != DBX_OK) return st;
  if (kind == 0) { *out_probe_idx = ip; *out_build_idx = ib; *n_out = ni; return DBX_OK; }
  int64_t np = probe_key->len;
  int64_t cap = ni + np + 1, no = 0;
  int64_t* op = (int64_t*)malloc(sizeof(int64_t) * cap);
  int64_t* ob = (int64_t*)malloc(sizeof(int64_t) * cap);
  int64_t j = 0; /* inner pairs are in probe order */
  for (int64_t r = 0; r < np; ++r) {
    int64_t first = j;
    while (j < ni && ip[j] == r) ++j;
    int64_t m = j - first;
    if (kind == 1) { if (m) { op[no] = r; ob[no] = -1; ++no; } }
    else if (kind == 2) { if (!m) { op[no] = r; ob[no] = -1; ++no; } }
    else { /* LEFT */
      for (int64_t t = first; t < j; ++t) { op[no] = r; ob[no] = ib[t]; ++no; }
      if (!m) { op[no] = r; ob[no] = -1; ++no; }
    }
  }
  free(ip); free(ib);
  *out_probe_idx = op; *out_build_idx = ob; *n_out = no;
  return DBX_OK;
}

void orc_free(void* p) { free(p); }

/* ------------------------------------------------------------------ sort / top-k */
/* DataBlock::sort_with_type + SortCompare (kernels/sort.rs:91-111, sort_compare.rs:197-296):
 * a u32 permutation ordered by the key (numbers: Ord; floats: OrderedFloat), `asc` flag,
 * NULLs by nulls_first, LimitRows(k).  Ties are arbitrary in the reference
 * (sort_unstable_by); the oracle breaks them by ascending row id so results are a
 * deterministic function of the input (the GPU path uses the same rule). */
typedef struct { const dbx_column* c; int asc; int nulls_first; } sort_ctx;
static sort_ctx g_sort; /* single-threaded use (qsort has no context argument) */

static int perm_cmp(const void* pa, const void* pb) {
  int64_t a = *(const int64_t*)pa, b = *(const int64_t*)pb;
  const dbx_column* c = g_sort.c;
  int va = col_valid(c, a), vb = col_valid(c, b);
  int r;
  if (!va || !vb) {
    if (va == vb) r = 0;
    else r = (!va) ? (g_sort.nulls_first ? -1 : 1) : (g_sort.nulls_first ? 1 : -1);
  } else {
    r = cmp_val(col_val(c, a), col_val(c, b));
    if (!g_sort.asc) r = -r;
  }
  if (r) return r;
  return a < b ? -1 : (a > b ? 1 : 0);
}

/* Structured like the reference pipeline: per 65 536-row block sort + limit
 * (TransformSortPartial, sorts/sort_partial.rs:56-58), then a limit-aware merge of the
 * per-block candidates (sort_merge*.rs).  out_idx receives min(k, n) global row ids. */
int orc_topk(const dbx_column* key, int asc, int nulls_first, int64_t k, int64_t* out_idx, int64_t* n_out) {
  int64_t n = key->len;
  if (k > n) k = n;
  g_sort.c = key; g_sort.asc = asc; g_sort.nulls_first = nulls_first;
  int64_t n_blocks = (n + ORC_BLOCK_ROWS - 1) / ORC_BLOCK_ROWS;
  int64_t ccap = n_blocks * (k < ORC_BLOCK_ROWS ? k : ORC_BLOCK_ROWS) + 1, nc = 0;
  int64_t* cand = (int64_t*)malloc(sizeof(int64_t) * ccap);
  int64_t* perm = (int64_t*)malloc(sizeof(int64_t) * ORC_BLOCK_ROWS);
  for (int64_t b = 0; b < n_blocks; ++b) {
    int64_t r0 = b * ORC_BLOCK_ROWS, r1 = r0 + ORC_BLOCK_ROWS;
    if (r1 > n) r1 = n;
    int64_t m = r1 - r0;
    for (int64_t i = 0; i < m; ++i) perm[i] = r0 + i;
    qsort(perm, (size_t)m, sizeof(int64_t), perm_cmp);
    int64_t keep = m < k ? m : k;
    memcpy(cand + nc, perm, sizeof(int64_t) * keep);
    nc += keep;
  }
  qsort(cand, (size_t)nc, sizeof(int64_t), perm_cmp);
  memcpy(out_idx, cand, sizeof(int64_t) * k);
  *n_out = k;
  free(cand); free(perm);
  return DBX_OK;
}

/* ------------------------------------------------------------------ vector distance */
/* ndarray 0.15.6 numeric_util::unrolled_fold (third party, restated): eight interleaved
 * accumulators p0..p7 over full chunks of 8, folded as
 *   acc = 0; acc += (p0+p4); acc += (p1+p5); acc += (p2+p6); acc += (p3+p7);
 * then the <8 tail elements are added sequentially. */
static float unrolled_sum_products(const float* a, const float* b, int64_t n) {
  float p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  int64_t i = 0;
  for (; i + 8 <= n; i += 8)
    for (int j = 0; j < 8; ++j) {
      volatile float prod = a[i + j] * b[i + j]; /* `&a * &b` materialises f32 products: no FMA */
      p[j] = p[j] + prod;
    }
  float acc = 0.0f;
  acc = acc + (p[0] + p[4]);
  acc = acc + (p[1] + p[5]);
  acc = acc + (p[2] + p[6]);
  acc = acc + (p[3] + p[7]);
  for (; i < n; ++i) {
    volatile float prod = a[i] * b[i];
    acc = acc + prod;
  }
  return acc;
}

/* cosine_distance (src/common/vector/src/distance.rs:19-35):
 *   1 - sum(a*b) / (sqrt(sum(a*a)) * sqrt(sum(b*b)))   all in f32; zero vector -> NaN */
float orc_cosine_distance(const float* a, const float* b, int64_t n) {
  float aa = unrolled_sum_products(a, a, n);
  float bb = unrolled_sum_products(b, b, n);
  float ab = unrolled_sum_products(a, b, n);
  volatile float den = sqrtf(aa) * sqrtf(bb);
  volatile float q = ab / den;
  return 1.0f - q;
}

/* l2_distance (distance.rs:65-80): sequential f32 fold of (a-b)^2, then sqrt */
float orc_l2_distance(const float* a, const float* b, int64_t n) {
  float acc = 0.0f;
  for (int64_t i = 0; i < n; ++i) {
    volatile float d = a[i] - b[i];
    volatile float sq = d * d;
    acc = acc + sq;
  }
  return sqrtf(acc);
}

/* calculate_distance (scalars/vector.rs:497-556): row-wise driver; either side may be a
 * single (const) vector.  out[i] for i < rows. */
void orc_distance_rows(int kind, const float* lhs, int lhs_const, const float* rhs, int rhs_const, int64_t rows,
                       int64_t dim, float* out, int threads) {
  if (threads < 1) threads = 1;
#pragma omp parallel for schedule(static) num_threads(threads)
  for (int64_t i = 0; i < rows; ++i) {
    const float* a = lhs + (lhs_const ? 0 : i * dim);
    const float* b = rhs + (rhs_const ? 0 : i * dim);
    out[i] = kind == DBX_DIST_COSINE ? orc_cosine_distance(a, b, dim) : orc_l2_distance(a, b, dim);
  }
}

/* ------------------------------------------------------------------ synthetic data */
/* Same counter-based generator as dbx_synth_fill (include/dbx.h), so that the host oracle
 * and the device see bit-identical columns. */
static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ULL;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
  return x ^ (x >> 31);
}

int orc_synth_fill(int kind, uint64_t seed, int64_t a, int64_t first_row, int64_t len, void* out, int threads) {
  if (threads < 1) threads = 1;
  if (kind == 4) {
#pragma omp parallel for schedule(static) num_threads(threads)
    for (int64_t i = 0; i < len; ++i) {
      uint64_t ctr = (uint64_t)(first_row + i);
      uint64_t r = splitmix64(seed + (ctr >> 1));
      float u1 = ((float)((r >> 40) + 1)) * (1.0f / 16777216.0f); /* (0,1] */
      float u2 = ((float)((r >> 8) & 0xFFFFFF)) * (1.0f / 16777216.0f);
      float rad = sqrtf(-2.0f * logf(u1));
      float ang = 6.28318530717958647692f * u2;
      ((float*)out)[i] = (ctr & 1) ? rad * sinf(ang) : rad * cosf(ang);
    }
    return DBX_OK;
  }
#pragma omp parallel for schedule(static) num_threads(threads)
  for (int64_t i = 0; i < len; ++i) {
    uint64_t row = (uint64_t)(first_row + i);
    uint64_t r = splitmix64(seed + row);
    switch (kind) {
      case 0: ((int64_t*)out)[i] = (int64_t)(((unsigned __int128)r * (unsigned __int128)(uint64_t)a) >> 64); break;
      case 1: ((int64_t*)out)[i] = (int64_t)(int32_t)(uint32_t)(r >> 32); break;
      case 2: ((double*)out)[i] = (double)(r >> (64 - a)); break;
      case 3: ((double*)out)[i] = (double)(r >> 11) * (1.0 / 9007199254740992.0); break;
      case 5: { /* bijection on [0, 2^a): odd multiply + xorshift, both invertible mod 2^a */
        uint64_t m = a >= 64 ? ~0ULL : ((1ULL << a) - 1);
        uint64_t x = row & m;
        x = (x * 0x9E3779B97F4A7C15ULL + seed) & m;
        x ^= x >> (a / 2 + 1);
        x = (x * 0xBF58476D1CE4E5B9ULL) & m;
        x ^= x >> (a / 2 + 1);
        ((int64_t*)out)[i] = (int64_t)x;
        break;
      }
      default: break;
    }
  }
  return DBX_OK;
}

int orc_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
