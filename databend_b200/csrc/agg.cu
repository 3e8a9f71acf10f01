// agg.cu — DBX_OP_AGG_PARTIAL / DBX_OP_AGG_FINAL: host side of the fused
// [TransformFilter ->] TransformPartialAggregate -> TransformFinalAggregate path.
//
// Reference operators replaced (paths relative to the databend source tree):
//   TransformFilter                    src/query/pipeline/transforms/src/processors/transforms/filters/filter_predicate.rs:35-104
//   TransformPartialAggregate          src/query/service/src/pipelines/processors/transforms/aggregator/transform_aggregate_partial.rs:117-304
//   PartialSingleStateAggregator       .../aggregator/transform_single_key.rs:42-188
//   TransformFinalAggregate            .../aggregator/transform_aggregate_final.rs:67-330
//   FinalSingleStateAggregator         .../aggregator/transform_single_key.rs:190-279
//   AggregateHashTable                 src/query/expression/src/aggregate/aggregate_hashtable.rs:168-408
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "agg_kernels.cuh"
#include "agg_jit.h"
#include "runtime.h"

namespace dbx {

namespace {

constexpr int64_t kChunkRows = 1LL << 28;        // rows per kernel launch (u32 overflow row ids)
constexpr int64_t kDefaultTableBytes = 64 << 20; // default table: 1e6 groups of config 2's shape without growth
constexpr int kProbeLimit = 64;  // buckets (x4 slots)

inline int grid_for_rows(int64_t n_rows) {
  int64_t tiles = (n_rows + kTileRows - 1) / kTileRows;
  int64_t g = (int64_t)kNumSMs * 8;  // 8 resident CTAs of 256 threads per SM = full occupancy
  return (int)std::max<int64_t>(1, std::min(tiles, g));
}
inline int grid_for_entries(int64_t n) {
  int64_t g = (n + 255) / 256;
  return (int)std::max<int64_t>(1, std::min<int64_t>(g, (int64_t)kNumSMs * 8));
}

// ---------------------------------------------------------------- plan
constexpr int kMaxCols = 64 + kMaxComputed;  // input columns, then computed columns

struct AggPlan {
  dbx_agg_params params;
  int n_cols = 0;   // input columns (the pushed blocks' schema)
  int n_comp = 0;   // computed columns: column n_cols + i is computed[i]
  int col_dtype[kMaxCols];
  bool col_nullable[kMaxCols];

  int n_slots = 0;
  // input column loaded into each slot; -1: the slot holds a computed value only.  While the plan is
  // built with computed columns these are virtual slots (one per column, computed ones included), mapped
  // onto at most kMaxSlots by allocate_slots.
  int slot_col[kMaxCols];
  // computed columns: the type-checked programs (COLUMN nodes name input columns), and what the
  // kernels evaluate after allocate_slots (only the computed columns the plan uses)
  NodeDev comp_nodes[kMaxComputed][kMaxExprNodes];
  int comp_n_nodes[kMaxComputed] = {};
  bool comp_raises[kMaxComputed] = {};
  int n_comp_ev = 0, comp_pred = 0, n_cnodes = 0;
  CompDev comp[kMaxComputed];
  NodeDev cnodes[kMaxCompNodes];
  uint32_t fresh_slots = 0;
  bool comp_nullable = false;  // a computed column the kernels evaluate may be NULL
  bool can_raise = false;      // a computed column evaluated after the predicate can raise: errors are recorded

  int n_nodes = 0;
  PredNodeDev nodes[DBX_MAX_PRED_NODES];
  bool div_by_zero = false;

  bool grouped = false;
  int key_slot = -1, key_dtype = -1;
  bool key_nullable = false;
  bool key_is_float = false;
  int n_key_parts = 0;  // > 1: packed multi-column key
  int key_words = 1;    // 2: the packed key needs 65..128 bits (HashMethodKeysU128)
  KeyPartDev key_parts[DBX_MAX_GROUP_COLS];

  int n_words = 0;
  WordInit init;
  WordKinds kinds;
  int n_updates = 0;
  UpdateDev upd[kMaxUpdates];
  FinalAgg fin[DBX_MAX_AGGS];  // out pointers filled at finalize time
  // tuning knobs, read from the environment once per operator (experiments sweep them in one process)
  bool l2_persist = true;    // persisting L2 access-policy window over the table
  int debug_flags = 0;
  bool hot_cache = false;    // per-CTA shared-memory cache of hot groups (skewed keys); DBX_AGG_HOT=0 turns it off

  int slot_of(int col, ErrorSink* err) {
    for (int s = 0; s < n_slots; ++s)
      if (slot_col[s] == col) return s;
    if (n_slots == (n_comp ? kMaxCols : kMaxSlots)) { err->set("operator reads more than 8 distinct columns"); return -1; }
    slot_col[n_slots] = col;
    return n_slots++;
  }
  int add_word(uint64_t init_v, int kind) {
    init.w[n_words] = init_v;
    kinds.op[n_words] = kind;
    return n_words++;
  }
};

// widened class of a column as loaded by load_slot: every integer type narrower than 64 bits is
// exactly representable as i64.
inline int loaded_class(int dtype) {
  switch (dtype) {
    case DBX_U64: return VC_UINT;
    case DBX_F32: case DBX_F64: return VC_FLT;
    default: return VC_INT;
  }
}
inline int flip_cmp(int op) {
  switch (op) {
    case DBX_LT: return DBX_GT;
    case DBX_LE: return DBX_GE;
    case DBX_GT: return DBX_LT;
    case DBX_GE: return DBX_LE;
    default: return op;
  }
}
inline double scalar_as_double(const dbx_scalar& s) {
  int c = dtype_class(s.dtype);
  return c == VC_FLT ? s.v.f64 : (c == VC_INT ? (double)s.v.i64 : (double)s.v.u64);
}
inline int cmp3_d(double a, double b) {
  bool an = a != a, bn = b != b;
  if (an || bn) return an == bn ? 0 : (an ? 1 : -1);
  return a < b ? -1 : (a > b ? 1 : 0);
}
inline bool apply_cmp_host(int op, int c) {
  switch (op) {
    case DBX_EQ: return c == 0;
    case DBX_NE: return c != 0;
    case DBX_LT: return c < 0;
    case DBX_LE: return c <= 0;
    case DBX_GT: return c > 0;
    default: return c >= 0;
  }
}

int32_t lower_cmp(AggPlan* pl, const dbx_pred_node& in, PredNodeDev* out, ErrorSink* err) {
  memset(out, 0, sizeof(*out));
  out->kind = DBX_PRED_CMP;
  out->r_slot = -1;
  dbx_operand l = in.lhs, r = in.rhs;
  int cmp = in.cmp;
  if (l.is_const && r.is_const) {  // constant folding -> BooleanScalar
    out->kind = DBX_PRED_CONST;
    if (l.c.is_null || r.c.is_null) { out->value = 0; return DBX_OK; }
    int cl = dtype_class(l.c.dtype), cr = dtype_class(r.c.dtype);
    int c3;
    if (cl == VC_FLT || cr == VC_FLT || cl != cr) c3 = cmp3_d(scalar_as_double(l.c), scalar_as_double(r.c));
    else if (cl == VC_INT) c3 = l.c.v.i64 < r.c.v.i64 ? -1 : (l.c.v.i64 > r.c.v.i64 ? 1 : 0);
    else c3 = l.c.v.u64 < r.c.v.u64 ? -1 : (l.c.v.u64 > r.c.v.u64 ? 1 : 0);
    out->value = apply_cmp_host(cmp, c3);
    return DBX_OK;
  }
  if (l.is_const) { std::swap(l, r); cmp = flip_cmp(cmp); }
  if (l.col < 0 || l.col >= pl->n_cols + pl->n_comp) { err->set("predicate references a column outside the input schema"); return DBX_ERR_INVALID; }
  if (!r.is_const && r.arith != DBX_ARITH_NONE) { err->set("arithmetic on the right-hand column of a comparison is not supported"); return DBX_ERR_UNSUPPORTED; }
  int lcls = loaded_class(pl->col_dtype[l.col]);
  out->l_slot = pl->slot_of(l.col, err);
  if (out->l_slot < 0) return DBX_ERR_UNSUPPORTED;
  out->cmp = cmp;
  if (l.arith == DBX_ARITH_MODULO) {
    if (l.c.is_null) { out->kind = DBX_PRED_CONST; out->value = 0; return DBX_OK; }  // x % NULL is NULL
    int ccls = dtype_class(l.c.dtype);
    if (lcls == VC_FLT || ccls == VC_FLT) {
      if (lcls != VC_FLT) { err->set("integer column % float literal is not supported"); return DBX_ERR_UNSUPPORTED; }
      double d = scalar_as_double(l.c);
      if (d == 0.0) pl->div_by_zero = true;
      out->mod_f = d;
    } else {
      uint64_t ad;
      if (ccls == VC_INT) ad = l.c.v.i64 < 0 ? (uint64_t)0 - (uint64_t)l.c.v.i64 : (uint64_t)l.c.v.i64;
      else ad = l.c.v.u64;
      if (lcls == VC_UINT && ccls == VC_INT && l.c.v.i64 < 0) { err->set("UInt64 % negative literal is not supported"); return DBX_ERR_UNSUPPORTED; }
      if (lcls == VC_INT && ccls == VC_UINT && l.c.v.u64 > (uint64_t)INT64_MAX) { err->set("Int64 % literal above i64::MAX is not supported"); return DBX_ERR_UNSUPPORTED; }
      if (ad == 0) { pl->div_by_zero = true; ad = 1; }
      out->mod = make_mod_magic(ad);
    }
    out->l_mod = 1;
  } else if (l.arith != DBX_ARITH_NONE) {
    err->set("unknown arithmetic op in predicate");
    return DBX_ERR_INVALID;
  }
  if (!r.is_const) {
    if (r.col < 0 || r.col >= pl->n_cols + pl->n_comp) { err->set("predicate references a column outside the input schema"); return DBX_ERR_INVALID; }
    int rcls = loaded_class(pl->col_dtype[r.col]);
    if (rcls != lcls) { err->set("comparison between columns of different numeric classes is not supported"); return DBX_ERR_UNSUPPORTED; }
    out->r_slot = pl->slot_of(r.col, err);
    if (out->r_slot < 0) return DBX_ERR_UNSUPPORTED;
    out->cls = lcls;
    return DBX_OK;
  }
  if (r.c.is_null) { out->kind = DBX_PRED_CONST; out->value = 0; return DBX_OK; }  // cmp with NULL is never true
  int rcls = dtype_class(r.c.dtype);
  // `x % d = 0` / `x % d <> 0` on integers: exact divisibility test instead of a remainder
  if (out->l_mod == 1 && lcls != VC_FLT && rcls != VC_FLT && r.c.v.u64 == 0 && (cmp == DBX_EQ || cmp == DBX_NE) &&
      !pl->div_by_zero && !getenv("DBX_AGG_NO_DIVTEST")) {
    out->mod = make_div_magic(out->mod.d);
    out->l_mod = 2;
  }
  if (lcls == VC_FLT) {
    out->cls = VC_FLT;
    out->r_const = scalar_bits(r.c, VC_FLT);
  } else if (rcls == VC_FLT) {
    err->set("integer column compared with a float literal is not supported");
    return DBX_ERR_UNSUPPORTED;
  } else if (lcls == VC_INT) {
    out->cls = VC_INT;
    if (rcls == VC_UINT && r.c.v.u64 > (uint64_t)INT64_MAX) {  // literal above every i64: fold, keep NULL handling
      bool always = cmp == DBX_LT || cmp == DBX_LE || cmp == DBX_NE;
      out->cmp = always ? DBX_LE : DBX_GT;
      out->r_const = (uint64_t)INT64_MAX;
    } else {
      out->r_const = r.c.v.u64;
    }
  } else {
    out->cls = VC_UINT;
    if (rcls == VC_INT && r.c.v.i64 < 0) {  // literal below every u64
      bool always = cmp == DBX_GT || cmp == DBX_GE || cmp == DBX_NE;
      out->cmp = always ? DBX_GE : DBX_LT;
      out->r_const = 0;
    } else {
      out->r_const = r.c.v.u64;
    }
  }
  return DBX_OK;
}

int32_t lower_predicate(AggPlan* pl, const dbx_predicate& pred, ErrorSink* err) {
  if (pred.n_nodes < 0 || pred.n_nodes > DBX_MAX_PRED_NODES) { err->set("predicate: bad node count"); return DBX_ERR_INVALID; }
  pl->n_nodes = pred.n_nodes;
  int depth = 0;
  for (int i = 0; i < pred.n_nodes; ++i) {
    const dbx_pred_node& in = pred.nodes[i];
    PredNodeDev* out = &pl->nodes[i];
    switch (in.kind) {
      case DBX_PRED_CMP: DBX_TRY(lower_cmp(pl, in, out, err)); depth += 1; break;
      case DBX_PRED_AND:
      case DBX_PRED_OR:
        memset(out, 0, sizeof(*out));
        out->kind = in.kind;
        out->n_children = in.n_children;
        if (in.n_children < 2 || in.n_children > depth || in.n_children > 16) { err->set("predicate: malformed AND/OR"); return DBX_ERR_INVALID; }
        depth -= in.n_children - 1;
        break;
      case DBX_PRED_BOOLCOL:
        memset(out, 0, sizeof(*out));
        out->kind = DBX_PRED_BOOLCOL;
        if (in.value < 0 || in.value >= pl->n_cols + pl->n_comp || pl->col_dtype[in.value] != DBX_BOOL) { err->set("predicate: BooleanColumn must reference a Boolean column"); return DBX_ERR_INVALID; }
        out->value = pl->slot_of(in.value, err);
        if (out->value < 0) return DBX_ERR_UNSUPPORTED;
        depth += 1;
        break;
      case DBX_PRED_CONST:
        memset(out, 0, sizeof(*out));
        out->kind = DBX_PRED_CONST;
        out->value = in.value != 0;
        depth += 1;
        break;
      default: err->set("predicate: unknown node kind"); return DBX_ERR_INVALID;
    }
    if (depth > 30) { err->set("predicate: expression too deep"); return DBX_ERR_UNSUPPORTED; }
  }
  if (pred.n_nodes && depth != 1) { err->set("predicate: postfix tree does not reduce to one value"); return DBX_ERR_INVALID; }
  return DBX_OK;
}

// Type-checks the computed columns (dbx_eval_scalar's inference over the input schema) and appends
// them to the plan's columns.
int32_t add_computed(AggPlan* pl, const dbx_expr* comp, int n_comp, ErrorSink* err) {
  if (n_comp < 0 || n_comp > kMaxComputed) { err->set("computed columns: n_computed outside 0 .. DBX_MAX_COMPUTED_COLS"); return DBX_ERR_INVALID; }
  if (n_comp > 0 && !comp) { err->set("computed columns: null list"); return DBX_ERR_INVALID; }
  if (pl->n_cols + n_comp > 64) { err->set("computed columns: more than 64 input and computed columns"); return DBX_ERR_INVALID; }
  for (int i = 0; i < n_comp; ++i) {
    const dbx_expr& e = comp[i];
    for (int k = 0; k < e.n_nodes && k < DBX_MAX_EXPR_NODES; ++k)
      if (e.nodes[k].kind == DBX_EXPR_COLUMN && e.nodes[k].col >= pl->n_cols && e.nodes[k].col < pl->n_cols + n_comp) {
        err->set("computed column " + std::to_string(i) + " references a computed column (only input columns may be referenced)");
        return DBX_ERR_INVALID;
      }
    int dt = 0;
    bool nullable = false;
    const int32_t st = infer_expr_types(e, pl->n_cols, pl->col_dtype, pl->col_nullable, pl->comp_nodes[i], &dt, &nullable, *err);
    if (st != DBX_OK) { err->set("computed column " + std::to_string(i) + ": " + err->msg); return st; }
    pl->comp_n_nodes[i] = e.n_nodes;
    pl->comp_raises[i] = expr_can_raise(pl->comp_nodes[i], e.n_nodes);
    pl->col_dtype[pl->n_cols + i] = dt;
    pl->col_nullable[pl->n_cols + i] = nullable;
  }
  pl->n_comp = n_comp;
  return DBX_OK;
}

// Maps the plan's virtual slots (one per column it reads) onto at most kMaxSlots.  Per tile the kernels
// load the inputs, evaluate the computed columns the predicate uses, the predicate, then the other
// computed columns; a computed column takes the slot of a value whose last use is at or before its own
// evaluation (an input only the predicate or earlier expressions read), else a new slot.
int32_t allocate_slots(AggPlan* pl, ErrorSink* err) {
  const int nv0 = pl->n_slots;
  bool pred_use[kMaxCols] = {}, late_use[kMaxCols] = {};
  for (int i = 0; i < pl->n_nodes; ++i) {
    const PredNodeDev& n = pl->nodes[i];
    if (n.kind == DBX_PRED_CMP) { pred_use[n.l_slot] = true; if (n.r_slot >= 0) pred_use[n.r_slot] = true; }
    else if (n.kind == DBX_PRED_BOOLCOL) pred_use[n.value] = true;
  }
  if (pl->grouped) {
    if (pl->n_key_parts > 1) for (int j = 0; j < pl->n_key_parts; ++j) late_use[pl->key_parts[j].slot] = true;
    else late_use[pl->key_slot] = true;
  }
  for (int u = 0; u < pl->n_updates; ++u)
    if (pl->upd[u].op != UPD_INC) late_use[pl->upd[u].slot] = true;
  // evaluation order: computed columns the predicate reads, then the others the plan reads
  int order[kMaxComputed], n_ord = 0, n_pred = 0;
  for (int phase = 0; phase < 2; ++phase)
    for (int v = 0; v < nv0; ++v) {
      const int c = pl->slot_col[v] - pl->n_cols;
      if (c < 0 || pred_use[v] != (phase == 0)) continue;
      if (pl->comp_raises[c] && phase == 0) {
        err->set("computed column " + std::to_string(c) + " is used by the predicate and can raise (division by a column or by zero, an overflowing cast or the negation of a 64-bit integer): "
                 "which rows reach it would depend on the evaluation order of the filter");
        return DBX_ERR_UNSUPPORTED;
      }
      order[n_ord++] = c;
      n_pred += phase == 0;
    }
  // the inputs of the evaluated computed columns
  for (int k = 0; k < n_ord; ++k) {
    const int c = order[k];
    for (int i = 0; i < pl->comp_n_nodes[c]; ++i)
      if (pl->comp_nodes[c][i].kind == DBX_EXPR_COLUMN && pl->slot_of(pl->comp_nodes[c][i].col, err) < 0) return DBX_ERR_UNSUPPORTED;
  }
  const int nv = pl->n_slots;
  // positions: 0 load, 1 .. n_pred predicate's computed columns, n_pred + 1 predicate, then the others
  auto comp_pos = [&](int c) { for (int k = 0; k < n_ord; ++k) if (order[k] == c) return k < n_pred ? 1 + k : 2 + k; return -1; };
  const int kEnd = 1 << 20;
  int last[kMaxCols], def[kMaxCols];
  for (int v = 0; v < nv; ++v) {
    const int c = pl->slot_col[v] - pl->n_cols;
    def[v] = c < 0 ? 0 : comp_pos(c);
    last[v] = late_use[v] ? kEnd : (pred_use[v] ? n_pred + 1 : 0);
  }
  for (int k = 0; k < n_ord; ++k) {
    const int c = order[k];
    for (int i = 0; i < pl->comp_n_nodes[c]; ++i)
      if (pl->comp_nodes[c][i].kind == DBX_EXPR_COLUMN) {
        const int v = pl->slot_of(pl->comp_nodes[c][i].col, err);
        last[v] = std::max(last[v], comp_pos(c));
      }
  }
  // inputs first (all are live at the load), then the computed columns in evaluation order
  int phys[kMaxCols], occ_last[kMaxSlots], phys_col[kMaxSlots], n_phys = 0;
  uint32_t fresh = 0;
  for (int v = 0; v < nv; ++v) {
    phys[v] = -1;
    if (pl->slot_col[v] >= pl->n_cols) continue;
    if (n_phys == kMaxSlots) break;
    phys_col[n_phys] = pl->slot_col[v];
    occ_last[n_phys] = last[v];
    phys[v] = n_phys++;
  }
  for (int k = 0; k < n_ord; ++k) {
    int v = 0;
    while (pl->slot_col[v] != pl->n_cols + order[k]) ++v;
    int s = 0;
    while (s < n_phys && occ_last[s] > def[v]) ++s;
    if (s == n_phys) {
      if (n_phys == kMaxSlots) break;
      phys_col[n_phys] = -1;
      fresh |= 1u << n_phys;
      ++n_phys;
    }
    occ_last[s] = last[v];
    phys[v] = s;
  }
  for (int v = 0; v < nv; ++v)
    if (phys[v] < 0) {
      err->set("the plan needs more than 8 values per row (input and computed columns), even with computed columns taking the slots of inputs they outlive: not supported");
      return DBX_ERR_UNSUPPORTED;
    }
  // rewrite every slot reference
  for (int i = 0; i < pl->n_nodes; ++i) {
    PredNodeDev& n = pl->nodes[i];
    if (n.kind == DBX_PRED_CMP) { n.l_slot = phys[n.l_slot]; if (n.r_slot >= 0) n.r_slot = phys[n.r_slot]; }
    else if (n.kind == DBX_PRED_BOOLCOL) n.value = phys[n.value];
  }
  if (pl->grouped) {
    for (int j = 0; j < pl->n_key_parts; ++j) pl->key_parts[j].slot = phys[pl->key_parts[j].slot];
    pl->key_slot = phys[pl->key_slot];
  }
  for (int u = 0; u < pl->n_updates; ++u) pl->upd[u].slot = pl->upd[u].op == UPD_INC ? 0 : phys[pl->upd[u].slot];
  pl->n_cnodes = 0;
  pl->comp_nullable = false;
  pl->can_raise = false;
  for (int k = 0; k < n_ord; ++k) {
    const int c = order[k];
    if (pl->n_cnodes + pl->comp_n_nodes[c] > kMaxCompNodes) { err->set("computed columns: more than 32 expression nodes evaluated per row"); return DBX_ERR_UNSUPPORTED; }
    int v = 0;
    while (pl->slot_col[v] != pl->n_cols + c) ++v;
    CompDev& cd = pl->comp[k];
    memset(&cd, 0, sizeof(cd));
    cd.first = pl->n_cnodes; cd.n_nodes = pl->comp_n_nodes[c]; cd.slot = phys[v];
    cd.branches = expr_has_branches(pl->comp_nodes[c], pl->comp_n_nodes[c]) ? 1 : 0;
    for (int i = 0; i < pl->comp_n_nodes[c]; ++i) {
      NodeDev nd = pl->comp_nodes[c][i];
      if (nd.kind == DBX_EXPR_COLUMN) nd.col = phys[pl->slot_of(nd.col, err)];
      pl->cnodes[pl->n_cnodes++] = nd;
    }
    pl->comp_nullable |= pl->col_nullable[pl->n_cols + c];
    pl->can_raise |= pl->comp_raises[c];
  }
  pl->n_comp_ev = n_ord;
  pl->comp_pred = n_pred;
  pl->fresh_slots = fresh;
  pl->n_slots = n_phys;
  for (int s = 0; s < n_phys; ++s) pl->slot_col[s] = phys_col[s];
  return DBX_OK;
}

int32_t build_plan(const dbx_agg_params* p, const int32_t* types, int32_t n_cols, const dbx_expr* comp, int32_t n_comp, AggPlan* pl,
                   ErrorSink* err) {
  if (n_cols < 0 || n_cols > 64) { err->set("too many input columns"); return DBX_ERR_INVALID; }
  pl->params = *p;
  pl->n_cols = n_cols;
  for (int i = 0; i < n_cols; ++i) {
    pl->col_dtype[i] = types[i] & 0xFF;
    pl->col_nullable[i] = (types[i] & DBX_NULLABLE) != 0;
  }
  DBX_TRY(add_computed(pl, comp, n_comp, err));
  n_cols += pl->n_comp;  // below, a column index may name a computed column
  if (p->n_aggs < 0 || p->n_aggs > DBX_MAX_AGGS) { err->set("bad aggregate count"); return DBX_ERR_INVALID; }
  if (p->n_group_cols < 0 || p->n_group_cols > DBX_MAX_GROUP_COLS) { err->set("bad group column count"); return DBX_ERR_INVALID; }
  DBX_TRY(lower_predicate(pl, p->filter, err));

  pl->grouped = p->n_group_cols > 0;
  pl->n_key_parts = 0;
  if (p->n_group_cols > 1) {
    // several fixed-width integer key columns whose bits (+ one NULL bit per Nullable column) fit
    // 64 bits are packed into one word, like HashMethodKeysU64 (kernels/group_by.rs:66-79); the
    // table, exchange and merge code then see an ordinary 64-bit key
    int bits = 0;
    for (int g = 0; g < p->n_group_cols; ++g) {
      const int kc = p->group_cols[g];
      if (kc < 0 || kc >= n_cols) { err->set("group column outside the input schema"); return DBX_ERR_INVALID; }
      const int dt = pl->col_dtype[kc];
      if (dtype_class(dt) == VC_FLT || dt == DBX_BOOL || dtype_size(dt) == 0) { err->set("GROUP BY keys must be integer columns (float/bool keys not built yet)"); return DBX_ERR_UNSUPPORTED; }
      KeyPartDev& kp = pl->key_parts[g];
      memset(&kp, 0, sizeof(kp));
      kp.slot = pl->slot_of(kc, err);
      if (kp.slot < 0) return DBX_ERR_UNSUPPORTED;
      kp.dtype = dt;
      const int w = 8 * dtype_size(dt);
      const int need = w + (pl->col_nullable[kc] ? 1 : 0);
      if (bits < 64 && bits + need > 64) bits = 64;  // a field (value + its NULL flag) never straddles the two key words
      kp.shift = bits;
      kp.mask = w == 64 ? ~0ULL : ((1ULL << w) - 1);
      bits += w;
      kp.null_shift = -1;
      if (pl->col_nullable[kc]) kp.null_shift = bits++;
    }
    if (bits > 128) { err->set("multi-column GROUP BY keys wider than 128 bits (incl. NULL flags) need 256-bit or serialised keys: not built (SURVEY 8f.1)"); return DBX_ERR_UNSUPPORTED; }
    pl->key_words = bits > 64 ? 2 : 1;  // HashMethodKeysU64 / HashMethodKeysU128 (kernels/group_by.rs:66-79)
    pl->n_key_parts = p->n_group_cols;
    pl->key_slot = pl->key_parts[0].slot;
    pl->key_dtype = DBX_U64;
    pl->key_nullable = false;
  } else if (pl->grouped) {
    int kc = p->group_cols[0];
    if (kc < 0 || kc >= n_cols) { err->set("group column outside the input schema"); return DBX_ERR_INVALID; }
    int dt = pl->col_dtype[kc];
    if (dt == DBX_BOOL || dtype_size(dt) == 0) { err->set("GROUP BY key must be a numeric column (bool/string keys not built yet)"); return DBX_ERR_UNSUPPORTED; }
    pl->key_is_float = dtype_class(dt) == VC_FLT;
    pl->key_slot = pl->slot_of(kc, err);
    if (pl->key_slot < 0) return DBX_ERR_UNSUPPORTED;
    pl->key_dtype = dt;
    pl->key_nullable = pl->col_nullable[kc];
  }

  // state words: word 0 = number of rows of the group (count(*), and the OrNull flag / avg
  // divisor of every aggregate whose argument type is not Nullable)
  memset(&pl->init, 0, sizeof(pl->init));
  memset(&pl->kinds, 0, sizeof(pl->kinds));
  pl->add_word(0, UPD_ADD_INT);
  pl->upd[pl->n_updates++] = UpdateDev{UPD_INC, 0, 0, 0};
  int cnt_word_of_col[kMaxCols], acc_word_of_col[kMaxCols];
  for (int i = 0; i < kMaxCols; ++i) cnt_word_of_col[i] = acc_word_of_col[i] = -1;

  for (int a = 0; a < p->n_aggs; ++a) {
    const dbx_agg_desc& ad = p->aggs[a];
    FinalAgg& fa = pl->fin[a];
    memset(&fa, 0, sizeof(fa));
    fa.kind = ad.kind;
    fa.acc_word = -1;
    if (ad.arg_col < 0) {
      if (ad.kind != DBX_AGG_COUNT) { err->set("only count() may omit its argument"); return DBX_ERR_INVALID; }
      fa.cnt_word = 0;
      fa.arg_dtype = DBX_U64;
      continue;
    }
    if (ad.arg_col >= n_cols) { err->set("aggregate argument outside the input schema"); return DBX_ERR_INVALID; }
    int dt = pl->col_dtype[ad.arg_col];
    if (dtype_size(dt) == 0) { err->set("aggregate argument must be a numeric column"); return DBX_ERR_UNSUPPORTED; }
    fa.arg_dtype = dt;
    int slot = pl->slot_of(ad.arg_col, err);
    if (slot < 0) return DBX_ERR_UNSUPPORTED;
    if (pl->n_words + 2 > kMaxWords || pl->n_updates + 2 > kMaxUpdates) { err->set("too many aggregate states"); return DBX_ERR_UNSUPPORTED; }
    if (!pl->col_nullable[ad.arg_col]) {
      fa.cnt_word = 0;
    } else {
      if (cnt_word_of_col[ad.arg_col] < 0) {
        cnt_word_of_col[ad.arg_col] = pl->add_word(0, UPD_ADD_INT);
        pl->upd[pl->n_updates++] = UpdateDev{UPD_INC_VALID, slot, cnt_word_of_col[ad.arg_col], 0};
      }
      fa.cnt_word = cnt_word_of_col[ad.arg_col];
    }
    int cls = loaded_class(dt);
    switch (ad.kind) {
      case DBX_AGG_COUNT: break;
      case DBX_AGG_SUM:
      case DBX_AGG_AVG:
        if (acc_word_of_col[ad.arg_col] < 0) {
          int op = cls == VC_FLT ? UPD_ADD_F64 : UPD_ADD_INT;
          acc_word_of_col[ad.arg_col] = pl->add_word(0, op);
          pl->upd[pl->n_updates++] = UpdateDev{op, slot, acc_word_of_col[ad.arg_col], 0};
        }
        fa.acc_word = acc_word_of_col[ad.arg_col];
        break;
      case DBX_AGG_MIN:
      case DBX_AGG_MAX: {
        bool mn = ad.kind == DBX_AGG_MIN;
        int op = cls == VC_FLT ? (mn ? UPD_MIN_F64 : UPD_MAX_F64) : cls == VC_UINT ? (mn ? UPD_MIN_U64 : UPD_MAX_U64) : (mn ? UPD_MIN_S64 : UPD_MAX_S64);
        uint64_t iv = op == UPD_MIN_S64 ? (uint64_t)INT64_MAX : op == UPD_MAX_S64 ? (uint64_t)INT64_MIN : (op == UPD_MIN_U64 || op == UPD_MIN_F64) ? ~0ULL : 0ULL;
        fa.acc_word = pl->add_word(iv, op);
        pl->upd[pl->n_updates++] = UpdateDev{op, slot, fa.acc_word, 0};
        break;
      }
      default: err->set("unknown aggregate kind"); return DBX_ERR_INVALID;
    }
  }
  if (pl->n_slots == 0) {  // e.g. count(*) without filter: still need a row source
    if (pl->n_cols == 0) { err->set("operator needs at least one input column"); return DBX_ERR_INVALID; }
    pl->slot_of(0, err);
  }
  if (pl->n_comp) DBX_TRY(allocate_slots(pl, err));
  pl->debug_flags = getenv("DBX_AGG_DEBUG") ? atoi(getenv("DBX_AGG_DEBUG")) : 0;
  pl->hot_cache = pl->grouped && pl->key_words == 1 && pl->n_words <= kHotWords &&
                  !(getenv("DBX_AGG_HOT") && atoi(getenv("DBX_AGG_HOT")) == 0);
  pl->l2_persist = !(getenv("DBX_AGG_L2_PERSIST") && atoi(getenv("DBX_AGG_L2_PERSIST")) == 0);
  return DBX_OK;
}

// ---------------------------------------------------------------- device table
struct DeviceTable {
  DevBuf mem;       // one allocation: [keys: (cap + 2) u64, padded to 256 B][states: (cap + 2) * n_words u64]
                    // (contiguous so ONE L2 access-policy window can cover the whole table)
  void* keys_p = nullptr;
  void* states_p = nullptr;
  DevBuf counters;  // [0] n_groups, [1] n_overflow
  int64_t cap = 0;
  int n_words = 0;
  int key_words = 1;

  unsigned long long* n_groups() const { return (unsigned long long*)counters.p; }
  unsigned long long* n_overflow() const { return (unsigned long long*)counters.p + 1; }
  size_t bytes() const { return (size_t)(cap + 2) * 8 * (key_words + n_words); }

  int32_t create(int64_t capacity, const AggPlan& pl, cudaStream_t stream, ErrorSink* err) {
    cap = capacity < 4 ? 4 : capacity;
    n_words = pl.n_words;
    key_words = pl.key_words;
    const size_t kbytes = ((size_t)(cap + 2) * 8 * key_words + 32 + 255) & ~(size_t)255;
    DBX_CUDA_TRY(*err, mem.ensure(kbytes + (size_t)(cap + 2) * 8 * n_words));
    keys_p = mem.p;
    states_p = (char*)mem.p + kbytes;
    DBX_CUDA_TRY(*err, counters.ensure(64));
    return clear(pl, stream, err);
  }
  int32_t clear(const AggPlan& pl, cudaStream_t stream, ErrorSink* err) {
    DBX_CUDA_TRY(*err, cudaMemsetAsync(counters.p, 0, 64, stream));
    int64_t total = (cap + 2) * (key_words + n_words);
    int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)kNumSMs * 16);
    table_init_kernel<<<grid, 256, 0, stream>>>(view(nullptr), pl.init);
    count_launch();
    DBX_CUDA_TRY(*err, cudaGetLastError());
    if (!pl.grouped) {  // the single state is slot 0 (key 0) and always exists
      uint64_t zero = 0;
      DBX_CUDA_TRY(*err, cudaMemcpyAsync(keys_p, &zero, 8, cudaMemcpyHostToDevice, stream));
      unsigned long long one = 1;
      DBX_CUDA_TRY(*err, cudaMemcpyAsync(counters.p, &one, 8, cudaMemcpyHostToDevice, stream));
    }
    return DBX_OK;
  }
  TableDev view(uint32_t* overflow_rows) const {
    TableDev t;
    t.keys = (uint64_t*)keys_p;
    t.states = (uint64_t*)states_p;
    t.cap = cap;
    t.n_words = n_words;
    t.key_words = key_words;
    t.n_groups = n_groups();
    t.n_overflow = n_overflow();
    t.overflow_rows = overflow_rows;
    t.hot_spill = nullptr;
    t.n_hot_spill = (unsigned long long*)counters.p + 2;
    t.n_hot_rows = (unsigned long long*)counters.p + 3;
    t.probe_limit = (int32_t)std::min<int64_t>(kProbeLimit, cap >> (key_words == 2 ? 1 : 2));
    return t;
  }
  void swap(DeviceTable& o) {
    std::swap(mem, o.mem);
    std::swap(keys_p, o.keys_p);
    std::swap(states_p, o.states_p);
    std::swap(counters, o.counters);
    std::swap(cap, o.cap);
    std::swap(n_words, o.n_words);
    std::swap(key_words, o.key_words);
  }
};

inline int64_t next_pow2(int64_t x) {
  int64_t p = 1;
  while (p < x) p <<= 1;
  return p;
}

}  // namespace

static std::atomic<size_t> g_persist_limit[64];  // cudaLimitPersistingL2CacheSize as last set, per device

// calls f(std::integral_constant<int, NS>) for a run-time slot count (1..8; anything else: 8)
template <class F>
static auto by_slots(int ns, F&& f) {
  switch (ns) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 3: return f(std::integral_constant<int, 3>());
    case 4: return f(std::integral_constant<int, 4>());
    case 5: return f(std::integral_constant<int, 5>());
    case 6: return f(std::integral_constant<int, 6>());
    case 7: return f(std::integral_constant<int, 7>());
    default: return f(std::integral_constant<int, 8>());
  }
}

// sizeof(StageWarp<NS>) for a run-time slot count
static size_t kMaxSlotsStageBytes(int ns) { return by_slots(ns, [](auto s) { return sizeof(StageWarp<decltype(s)::value>); }); }

// dynamic shared memory of the partitioned passes for a run-time slot count: pass 1's stash, pass 2's row buffers
static size_t partition_smem_for(int ns) { return by_slots(ns, [](auto s) { return partition_smem_bytes<decltype(s)::value>(); }); }
static size_t ring_smem_for(int ns) { return by_slots(ns, [](auto s) { return ring_smem_bytes<decltype(s)::value>(); }); }
static size_t slice_stage_bytes_for(int ns) { return by_slots(ns, [](auto s) { return slice_stage_bytes<decltype(s)::value>(); }); }

// ================================================================ partial
class AggPartialOp : public Op {
 public:
  AggPlan plan;
  DeviceTable table;
  Stager stager;
  DevBuf ovf[2];
  PinnedBuf host_counters;
  int64_t groups_known = 0;    // exact group count at the last counter read
  int64_t rows_since_read = 0; // rows pushed since (upper bound on new groups)
  bool pulled = false;
  int64_t rows_in = 0;
  int64_t initial_cap = 0;
  bool table_ready = false;
  bool table_clean = false;  // the exchange scatter left the table empty (fused clear): reset costs no kernel
  void* window_base = nullptr;  // L2 access-policy window currently set on the stream
  size_t window_bytes = 0;
  AggJitKernels jit;            // kernels compiled for this plan (agg_jit.h); empty: precompiled kernels
  std::string jit_status = "off";
  ~AggPartialOp() override {
    if (window_base) {  // give the persisting L2 lines back (other operators / the kNN GEMM want the whole L2)
      cudaSetDevice(device);
      if (stream) cudaStreamSynchronize(stream);
      cudaCtxResetPersistingL2Cache();
    }
  }

  int32_t init(const dbx_agg_params* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int dev) {
    DBX_TRY(base_init(dev));
    DBX_TRY(build_plan(p, types, n, comp, n_comp, &plan, &err));
    DBX_TRY(stager.init(dev, stream, &err));
    DBX_CUDA_TRY(err, host_counters.ensure(64));
    if (plan.can_raise) {
      DBX_CUDA_TRY(err, expr_err.ensure(8));
      DBX_CUDA_TRY(err, cudaMemsetAsync(expr_err.p, 0xFF, 8, stream));
    }
    int64_t cap;
    if (!plan.grouped) cap = 4;
    else if (p->expected_groups > 0) cap = next_pow2(std::max<int64_t>(2 * p->expected_groups, 1024));
    else cap = std::max<int64_t>(1024, next_pow2(kDefaultTableBytes / (8 * (1 + plan.n_words)) + 1) / 2);
    initial_cap = cap;
    DBX_TRY(ensure_table());
    specialise();
    return DBX_OK;
  }

  std::string variant_text;
  const char* kernel_variant() override {
    variant_text = jit_status;
    if (plan.n_comp_ev)  // which kernels evaluated the computed columns (tests assert the path they target)
      variant_text += "; computed columns: straight-line launches " + std::to_string(comp_fast_launches) + ", generic launches " +
                      std::to_string(comp_generic_launches) + ", rows absorbed by the hot-group cache " + std::to_string(hot_absorbed_seen);
    if (partitioned_chunks || partition_fallbacks)
      variant_text += "; two-pass (partitioned by table slice) chunks: " + std::to_string(partitioned_chunks) + " (pass 2 in shared memory: " +
                      std::to_string(slice_chunks) + ", in L2 regions: " + std::to_string(partitioned_chunks - slice_chunks) +
                      "), one-pass fallbacks (skew): " + std::to_string(partition_fallbacks) + "; specialised launches: pass 1 " +
                      std::to_string(part_jit_launches) + " of " + std::to_string(partitioned_chunks + partition_fallbacks) + ", pass 2 " +
                      std::to_string(slice_jit_launches) + " of " + std::to_string(slice_chunks) + "; pass 1 on the bulk-copy ring: " +
                      std::to_string(part_ring_launches) + " of " + std::to_string(partitioned_chunks + partition_fallbacks);
    return variant_text.c_str();
  }
  // Ask for kernels compiled for this plan (grouped plans with 64-bit keys).  Failure is not an
  // error: the precompiled kernels serve the operator, jit_status says why.
  void specialise() {
    const char* e = getenv("DBX_AGG_JIT");
    if (e && atoi(e) == 0) { jit_status = "off (DBX_AGG_JIT=0)"; return; }
    if (!plan.grouped || plan.key_words != 1) { jit_status = "off (plan shape not specialised)"; return; }
    StaticPlan sp;
    memset(&sp, 0, sizeof(sp));
    sp.n_nodes = plan.n_nodes; sp.n_updates = plan.n_updates; sp.key_slot = plan.key_slot; sp.key_is_float = plan.key_is_float ? 1 : 0;
    sp.n_key_parts = plan.n_key_parts; sp.debug_flags = plan.debug_flags; sp.n_words = plan.n_words; sp.hot_cache = plan.hot_cache ? 1 : 0;
    memcpy(sp.nodes, plan.nodes, sizeof(PredNodeDev) * plan.n_nodes);
    memcpy(sp.upd, plan.upd, sizeof(UpdateDev) * plan.n_updates);
    memcpy(sp.key_parts, plan.key_parts, sizeof(plan.key_parts));
    if (plan.n_comp_ev) {
      sp.n_comp = plan.n_comp_ev; sp.comp_pred = plan.comp_pred; sp.fresh_slots = plan.fresh_slots; sp.raises = plan.can_raise ? 1 : 0;
      memcpy(sp.comp, plan.comp, sizeof(plan.comp));
      memcpy(sp.cnodes, plan.cnodes, sizeof(NodeDev) * plan.n_cnodes);
    }
    std::string why;
    if (!agg_jit_get(agg_jit_plan_text(sp), plan.n_slots, &jit, &why)) { jit = AggJitKernels(); jit_status = "precompiled kernels (" + why + ")"; return; }
    // the row stages of 5+ slots exceed the 48 KB default: opt the specialised kernels in on this device
    const size_t smem = (((size_t)(kMaxSlotsStageBytes(plan.n_slots)) * kWarpsPerBlock + 15) & ~(size_t)15) + kHotBytes;
    cudaError_t ce = cudaSuccess;
    if (smem > 48 * 1024) {
      ce = cudaKernelSetAttributeForDevice(jit.fast, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem, device);
      if (ce == cudaSuccess) ce = cudaKernelSetAttributeForDevice(jit.gen, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem, device);
    }
    if (ce != cudaSuccess) {
      cudaGetLastError();
      jit = AggJitKernels();
      jit_status = std::string("precompiled kernels (shared-memory opt-in of the specialised kernel failed: ") + cudaGetErrorString(ce) + ")";
      return;
    }
    jit_status = "specialised";
    // the two passes of the partitioned path: both use more than 48 KB of dynamic shared memory
    ce = cudaKernelSetAttributeForDevice(jit.part, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)partition_smem_for(plan.n_slots), device);
    if (ce == cudaSuccess)
      ce = cudaKernelSetAttributeForDevice(jit.part_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring_smem_for(plan.n_slots), device);
    if (ce == cudaSuccess)
      ce = cudaKernelSetAttributeForDevice(jit.slice, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSliceBytes + slice_stage_bytes_for(plan.n_slots)), device);
    if (ce != cudaSuccess) drop_two_pass_jit("shared-memory opt-in", ce);
  }
  // the partitioned passes go back to the precompiled kernels; the fused kernels stay specialised
  void drop_two_pass_jit(const char* what, cudaError_t ce) {
    cudaGetLastError();
    jit.part = jit.part_ring = jit.slice = nullptr;
    jit_status += std::string(" (two-pass: precompiled kernels, ") + what + " of the specialised kernel failed: " + cudaGetErrorString(ce) + ")";
  }

  // Pin the hash table in L2 while the column stream passes through: a persisting access-policy
  // window over the table's allocation on this operator's stream (the column loads are outside
  // the window and carry evict_first).  DBX_AGG_L2_PERSIST=0 turns it off.
  int32_t apply_l2_window() {
    if (!plan.l2_persist || !plan.grouped) return DBX_OK;
    if (part_threshold > 0 && (int64_t)table.bytes() > part_threshold) {
      // a table beyond L2 is aggregated region by region (partitioned_rows): a window over all of it would
      // only take capacity away from the region that is being worked on
      if (window_base) {
        cudaStreamAttrValue off;
        memset(&off, 0, sizeof(off));
        DBX_CUDA_TRY(err, cudaStreamSetAttribute(stream, cudaStreamAttributeAccessPolicyWindow, &off));
        DBX_CUDA_TRY(err, cudaCtxResetPersistingL2Cache());
        window_base = nullptr; window_bytes = 0;
      }
      return DBX_OK;
    }
    if (table.mem.p == window_base && table.bytes() == window_bytes) return DBX_OK;
    window_base = table.mem.p;
    window_bytes = table.bytes();
    int max_persist = 0, max_window = 0;
    DBX_CUDA_TRY(err, cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, device));
    DBX_CUDA_TRY(err, cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, device));
    if (max_persist <= 0 || max_window <= 0) return DBX_OK;
    const size_t bytes = std::min<size_t>(table.bytes() + 512, (size_t)max_window);
    const size_t want = std::min<size_t>(bytes, (size_t)max_persist);
    if (g_persist_limit[device] < want) {  // the set-aside only ever grows (it is a device-wide limit shared by all operators)
      DBX_CUDA_TRY(err, cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want));
      g_persist_limit[device] = want;
    }
    cudaStreamAttrValue av;
    memset(&av, 0, sizeof(av));
    av.accessPolicyWindow.base_ptr = table.mem.p;
    av.accessPolicyWindow.num_bytes = bytes;
    av.accessPolicyWindow.hitRatio = bytes <= want ? 1.0f : (float)want / (float)bytes;
    av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    av.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
    DBX_CUDA_TRY(err, cudaStreamSetAttribute(stream, cudaStreamAttributeAccessPolicyWindow, &av));
    return DBX_OK;
  }

  // (Re-)create or clear the table lazily: after a final operator adopted it, or after reset().
  int32_t ensure_table() {
    if (table_ready) return DBX_OK;
    if (table.cap != initial_cap || !table.keys_p) DBX_TRY(table.create(initial_cap, plan, stream, &err));
    else if (!table_clean) DBX_TRY(table.clear(plan, stream, &err));
    table_clean = false;
    hot_absorbed_seen = 0;  // the counters were cleared with the table
    DBX_TRY(apply_l2_window());
    table_ready = true;
    groups_known = plan.grouped ? 0 : 1;
    rows_since_read = 0;
    return DBX_OK;
  }

  int64_t prev_query_groups = 0;  // groups of the query before the last reset (exact at its last counter read)
  int32_t reset() override {
    if (batch_open) { batch_open = false; batch_rows = 0; DBX_TRY(stager.join_aux()); DBX_TRY(stager.end()); }
    prev_query_groups = groups_known;
    table_ready = false;
    DBX_TRY(ensure_table());
    groups_known = plan.grouped ? 0 : 1;
    rows_since_read = 0;
    pulled = false;
    rows_in = 0;
    if (plan.can_raise) DBX_CUDA_TRY(err, cudaMemsetAsync(expr_err.p, 0xFF, 8, stream));
    return DBX_OK;
  }

  unsigned long long hot_spilled = 0;  // read_counters: groups the hot-group caches could not place
  bool hot_on = true;                  // adaptive: see read_counters
  int64_t hot_probe_rows = 0;          // input rows launched with the cache on since the last evaluation
  unsigned long long hot_absorbed_seen = 0;
  int64_t hot_launches = 0;
  bool want_hot() { return plan.hot_cache && (hot_on || (hot_launches++ % 32) == 31); }
  DevBuf hot_spill;
  int32_t read_counters(unsigned long long* n_groups, unsigned long long* n_overflow) {
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host_counters.p, table.counters.p, 32, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    *n_groups = ((unsigned long long*)host_counters.p)[0];
    *n_overflow = ((unsigned long long*)host_counters.p)[1];
    hot_spilled = ((unsigned long long*)host_counters.p)[2];
    // the hot-group cache pays for itself only on skewed keys: keep it while it absorbs >= 0.5 % of the
    // rows it saw, turn it off otherwise (uniform keys: +3 % kernel time for nothing); re-probed every 32 launches
    const unsigned long long absorbed = ((unsigned long long*)host_counters.p)[3];
    if (hot_probe_rows > 0) {
      hot_on = (absorbed - std::min(absorbed, hot_absorbed_seen)) * 200 >= (unsigned long long)hot_probe_rows;
      hot_probe_rows = 0;
    }
    hot_absorbed_seen = absorbed;
    groups_known = (int64_t)*n_groups;
    rows_since_read = 0;
    return DBX_OK;
  }

  // resize (aggregate_hashtable.rs:463-489): rebuild into a larger table on the device
  int32_t grow_to(int64_t new_cap) {
    DeviceTable nt;
    DBX_TRY(nt.create(new_cap, plan, stream, &err));
    table_merge_kernel<<<grid_for_entries(table.cap + 2), 256, 0, stream>>>(table.view(nullptr), nt.view(nullptr), plan.kinds);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));  // old table is freed below
    table.swap(nt);
    DBX_TRY(apply_l2_window());
    return DBX_OK;
  }

  int64_t comp_fast_launches = 0, comp_generic_launches = 0;
  template <int NS, bool FAST, bool INDIRECT>
  int32_t launch_one(const AggKernelParams& kp) {
    if (kp.n_comp > 0) {
      ++(FAST ? comp_fast_launches : comp_generic_launches);
      return launch_kernel<NS, FAST, INDIRECT, true>(kp);
    }
    return launch_kernel<NS, FAST, INDIRECT>(kp);
  }
  template <int NS, bool FAST, bool INDIRECT, bool EXPR = false>
  int32_t launch_kernel(const AggKernelParams& kp) {
    static std::atomic<bool> attr_set[64];
    if (device < 0 || device >= 64) { err.set("device index out of range"); return DBX_ERR_INVALID; }
    // the row stages, then the hot-group cache
    const size_t smem = ((sizeof(StageWarp<NS>) * kWarpsPerBlock + 15) & ~(size_t)15) + kHotBytes;
    auto kern = filter_group_agg_kernel<NS, FAST, INDIRECT, EXPR>;
    if (!attr_set[device]) {
      DBX_CUDA_TRY(err, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr_set[device] = true;
    }
    int grid = grid_for_rows(kp.n_rows);
    static const int per_sm = getenv("DBX_AGG_GRID") ? atoi(getenv("DBX_AGG_GRID")) : 0;
    if (per_sm > 0 && !(kp.table.hot_spill && per_sm > 8))  // the spill buffer of the hot-group caches is sized for 8 CTAs per SM
      grid = (int)std::max<int64_t>(1, std::min<int64_t>((kp.n_rows + kTileRows - 1) / kTileRows, (int64_t)kNumSMs * per_sm));
    if (!INDIRECT && jit.ok() && !no_filter_) {  // same grid, block and shared memory: only the code differs
      void* args[] = {(void*)&kp};
      const cudaError_t ce = cudaLaunchKernel((const void*)(FAST ? jit.fast : jit.gen), dim3(grid), dim3(kBlock), args, smem, stream);
      if (ce == cudaSuccess) { count_launch(); return DBX_OK; }
      cudaGetLastError();
      jit = AggJitKernels();
      jit_status = std::string("precompiled kernels (launch of the specialised kernel failed: ") + cudaGetErrorString(ce) + ")";
    }
    kern<<<grid, kBlock, smem, stream>>>(kp);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }
  template <int NS, bool INDIRECT, bool EXPR>
  int32_t launch_wide(const AggKernelParams& kp) {
    static std::atomic<bool> attr_set[64];
    if (device < 0 || device >= 64) { err.set("device index out of range"); return DBX_ERR_INVALID; }
    const size_t smem = (sizeof(StageWarp<NS>) * kWarpsPerBlock + 15) & ~(size_t)15;
    if (!attr_set[device]) {
      DBX_CUDA_TRY(err, cudaFuncSetAttribute(filter_group_agg_wide_kernel<NS, INDIRECT, EXPR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr_set[device] = true;
    }
    filter_group_agg_wide_kernel<NS, INDIRECT, EXPR><<<grid_for_rows(kp.n_rows), kBlock, smem, stream>>>(kp);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }
  template <bool INDIRECT>
  int32_t launch_wide_ns(const AggKernelParams& kp) {
    return by_slots(plan.n_slots, [&](auto s) {
      constexpr int NS = decltype(s)::value;
      return kp.n_comp > 0 ? launch_wide<NS, INDIRECT, true>(kp) : launch_wide<NS, INDIRECT, false>(kp);
    });
  }
  template <bool FAST, bool INDIRECT>
  int32_t launch_ns(const AggKernelParams& kp) {
    return by_slots(plan.n_slots, [&](auto s) { return launch_one<decltype(s)::value, FAST, INDIRECT>(kp); });
  }
  // The straight-line variant applies to plain 8-byte device columns (no validity, 32 B aligned)
  // with at most one Compare; it covers whole tiles, the generic kernel takes the remainder.
  bool fast_eligible(const AggKernelParams& kp) const {
    if (getenv("DBX_AGG_NO_FAST")) return false;
    if (kp.n_nodes > 1) return false;
    if (kp.n_nodes == 1 && (kp.nodes[0].kind != DBX_PRED_CMP || kp.nodes[0].r_slot >= 0)) return false;
    if (kp.n_comp > 0 && plan.comp_nullable) return false;  // the straight-line kernel stages no validity
    for (int s = 0; s < kp.n_slots; ++s) {
      if (kp.n_comp > 0 && ((kp.fresh_slots >> s) & 1)) continue;
      const DevCol& c = kp.cols[s];
      if (c.is_const || c.validity) return false;
      if (c.dtype != DBX_I64 && c.dtype != DBX_U64 && c.dtype != DBX_F64) return false;
      if (reinterpret_cast<uintptr_t>(c.data) & 31) return false;
    }
    return true;
  }
  int32_t launch_grouped(const AggKernelParams& kp, bool indirect) {
    if (plan.key_words == 2) return indirect ? launch_wide_ns<true>(kp) : launch_wide_ns<false>(kp);
    if (indirect) return launch_ns<false, true>(kp);
    if (!fast_eligible(kp) || kp.n_rows < kTileRows) return launch_ns<false, false>(kp);
    AggKernelParams a = kp;
    const int64_t n_fast = kp.n_rows / kTileRows * kTileRows;
    a.n_rows = n_fast;
    DBX_TRY((launch_ns<true, false>(a)));
    if (n_fast < kp.n_rows) {
      AggKernelParams b = kp;
      for (int s = 0; s < kp.n_slots; ++s) b.cols[s].data = (const char*)kp.cols[s].data + n_fast * 8;
      b.n_rows = kp.n_rows - n_fast;
      b.row_base = kp.row_base + (uint32_t)n_fast;
      DBX_TRY((launch_ns<false, false>(b)));
    }
    return DBX_OK;
  }
  int32_t launch_single(const AggKernelParams& kp) {
    int grid = std::min(grid_for_rows(kp.n_rows), kNumSMs * 4);
    by_slots(plan.n_slots, [&](auto s) {
      constexpr int NS = decltype(s)::value;
      if (kp.n_comp > 0) filter_single_agg_kernel<NS, true><<<grid, kBlock, 0, stream>>>(kp);
      else filter_single_agg_kernel<NS, false><<<grid, kBlock, 0, stream>>>(kp);
    });
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }

  void fill_params(AggKernelParams* kp, const DevCol* cols, int64_t row0, int64_t n) {
    memset(kp, 0, sizeof(*kp));
    for (int s = 0; s < plan.n_slots; ++s) {
      DevCol c = cols[s];
      if (!c.is_const) {
        if (c.dtype == DBX_BOOL) c.dbit_off += row0;
        else c.data = (const char*)c.data + row0 * dtype_size(c.dtype);
        if (c.validity) c.vbit_off += row0;
      }
      kp->cols[s] = c;
    }
    memcpy(kp->nodes, plan.nodes, sizeof(PredNodeDev) * plan.n_nodes);
    memcpy(kp->upd, plan.upd, sizeof(UpdateDev) * plan.n_updates);
    kp->n_rows = n;
    kp->n_slots = plan.n_slots;
    kp->n_nodes = no_filter_ ? 0 : plan.n_nodes;  // pass 2 of the partitioned path: the rows are the survivors already
    kp->n_updates = plan.n_updates;
    kp->key_slot = plan.key_slot;
    kp->key_nullable = plan.key_nullable;
    kp->key_is_float = plan.key_is_float ? 1 : 0;
    kp->n_key_parts = plan.n_key_parts;
    memcpy(kp->key_parts, plan.key_parts, sizeof(plan.key_parts));
    kp->debug_flags = plan.debug_flags;
    // computed columns, except over pass 1's buffers (they hold the computed values already)
    if (plan.n_comp_ev && !no_filter_) {
      kp->n_comp = plan.n_comp_ev;
      kp->comp_pred = plan.comp_pred;
      kp->fresh_slots = plan.fresh_slots;
      memcpy(kp->comp, plan.comp, sizeof(plan.comp));
      memcpy(kp->cnodes, plan.cnodes, sizeof(NodeDev) * plan.n_cnodes);
      kp->expr_row0 = expr_base + row0;
      kp->expr_err = plan.can_raise ? (unsigned long long*)expr_err.p : nullptr;
    }
  }
  // the DevCol of a slot that holds a computed value only: a constant, so the loads touch no memory
  static DevCol fresh_col() {
    DevCol c;
    memset(&c, 0, sizeof(c));
    c.dtype = DBX_U64;
    c.is_const = 1;
    return c;
  }

  int32_t push(const dbx_block* b) override {
    if (b->num_cols != plan.n_cols) { err.set("push: block column count differs from the operator's input schema"); return DBX_ERR_INVALID; }
    for (int i = 0; i < plan.n_cols; ++i) {
      if (b->cols[i].dtype != plan.col_dtype[i]) { err.set("push: block column dtype differs from the operator's input schema"); return DBX_ERR_INVALID; }
      if (b->cols[i].len != b->num_rows) { err.set("push: column length differs from num_rows"); return DBX_ERR_INVALID; }
      if (b->cols[i].validity && !plan.col_nullable[i] && !b->cols[i].is_const) { err.set("push: validity bitmap on a column declared non-nullable"); return DBX_ERR_INVALID; }
    }
    const int64_t n = b->num_rows;
    if (n == 0) return DBX_OK;
    if (plan.div_by_zero) {  // rem_scalar: divisor literal 0 fails the whole block (arithmetic_modulo.rs:137-140)
      err.set("Division by zero, during run expr: modulo (first failing row 0)");
      return DBX_ERR_BAD_ARGUMENTS;
    }
    DBX_TRY(ensure_table());
    table_clean = false;
    // Small host blocks (the reference pushes 65 536-row DataBlocks, settings_default.rs:142) are
    // coalesced: their columns are DMA'd back to back into one staging generation and the fused
    // kernel runs once per ~4 Mi rows instead of once per block.
    if (batchable(b)) {
      if (batch_open && batch_rows + n > kBatchCapRows) DBX_TRY(flush_batch());
      if (!batch_open) { DBX_TRY(stager.begin()); batch_open = true; batch_rows = 0; batch_row0 = rows_in; }
      for (int s = 0; s < plan.n_slots; ++s) {
        if (plan.slot_col[s] < 0) { batch_cols[s] = fresh_col(); continue; }
        DBX_TRY(stager.stage_at(b->cols[plan.slot_col[s]], s, batch_rows, kBatchCapRows, &batch_cols[s]));
      }
      batch_rows += n;
      rows_in += n;
      return DBX_OK;
    }
    DBX_TRY(flush_batch());
    DevCol cols[kMaxSlots];
    DBX_TRY(stager.begin());
    for (int s = 0; s < plan.n_slots; ++s) {
      if (plan.slot_col[s] < 0) { cols[s] = fresh_col(); continue; }
      DBX_TRY(stager.stage(b->cols[plan.slot_col[s]], s, &cols[s]));
    }
    expr_base = rows_in;
    rows_in += n;
    DBX_TRY(process_rows(cols, n));
    DBX_TRY(stager.end());
    return DBX_OK;
  }

  // ---- coalescing of small pushes
  static constexpr int64_t kBatchCapRows = 4 << 20;
  static constexpr int64_t kBatchMaxBlockRows = 1 << 20;
  bool batch_open = false;
  int64_t batch_rows = 0;
  int64_t batch_row0 = 0;  // number of the batch's first row since create / reset
  int64_t expr_base = 0;   // number of the first row of the rows process_rows works on
  DevBuf expr_err;         // plans that can raise: min over failing rows of (row << 8 | code), ~0: none
  PinnedBuf expr_err_host;
  DevCol batch_cols[kMaxSlots];
  bool batchable(const dbx_block* b) const {
    if (no_batching || b->num_rows > kBatchMaxBlockRows) return false;
    for (int s = 0; s < plan.n_slots; ++s) {
      if (plan.slot_col[s] < 0) continue;
      const dbx_column& c = b->cols[plan.slot_col[s]];
      if (c.mem != DBX_MEM_HOST || c.is_const || c.validity || c.dtype == DBX_BOOL) return false;
    }
    return true;
  }
  // dbx_op_inputs_consumed: copies of a still-open batch run on the stager's auxiliary streams
  int32_t wait_inputs() override {
    DBX_TRY(stager.join_aux());
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    return DBX_OK;
  }
  int32_t flush_batch() {
    if (!batch_open) return DBX_OK;
    batch_open = false;
    DBX_TRY(stager.join_aux());
    expr_base = batch_row0;
    if (batch_rows > 0) DBX_TRY(process_rows(batch_cols, batch_rows));
    batch_rows = 0;
    DBX_TRY(stager.end());
    return DBX_OK;
  }
  bool no_batching = getenv("DBX_AGG_NO_BATCH") != nullptr;

  // the fused kernel(s) over n rows whose needed columns are on the device
  // ---- two-pass aggregation for tables that do not fit L2 (see filter_partition_kernel)
  bool no_filter_ = false;
  DevBuf part_buf[kMaxSlots], part_cnt;
  PinnedBuf part_host;
  // defaults sized to the 50 MB L2: tables beyond ~80% of it go two-pass, in regions of ~40% of it
  int64_t part_threshold = getenv("DBX_AGG_PARTITION_BYTES") ? atoll(getenv("DBX_AGG_PARTITION_BYTES")) : (40LL << 20);
  int64_t part_region_bytes = getenv("DBX_AGG_REGION_BYTES") ? atoll(getenv("DBX_AGG_REGION_BYTES")) : (20LL << 20);
  int64_t partitioned_chunks = 0, partition_fallbacks = 0, slice_chunks = 0;
  static constexpr int64_t kPartChunkRows = 1LL << 28;
  static constexpr int kMaxRegions = 64;  // partitions of the L2-region pass 2
  bool partition_eligible(const DevCol* cols, int64_t m) const {
    if (!plan.grouped || plan.key_words != 1 || part_threshold <= 0) return false;
    if ((int64_t)table.bytes() <= part_threshold || m < (1 << 16)) return false;
    // every partition pass pulls its table region into L2 again: worth it only when the rows outweigh the table
    if (m * 8 * plan.n_slots < 4 * (int64_t)table.bytes() && !getenv("DBX_AGG_PARTITION_ALWAYS")) return false;
    if (plan.comp_nullable) return false;  // the partitions carry value images only
    for (int s = 0; s < plan.n_slots; ++s)
      if (plan.slot_col[s] >= 0 && (cols[s].is_const || cols[s].validity)) return false;
    return true;
  }
  bool region_window_on = false;
  void region_window(void* base, size_t bytes) {  // best effort: a failure only costs speed
    int max_persist = 0, max_window = 0;
    cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, device);
    cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, device);
    cudaStreamAttrValue av;
    memset(&av, 0, sizeof(av));
    if (base && bytes && max_persist > 0 && max_window > 0) {
      const size_t win = std::min<size_t>(bytes, (size_t)max_window);
      const size_t want = std::min<size_t>(win, (size_t)max_persist);
      if (device >= 0 && device < 64 && g_persist_limit[device] < want) { cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want); g_persist_limit[device] = want; }
      av.accessPolicyWindow.base_ptr = base;
      av.accessPolicyWindow.num_bytes = win;
      av.accessPolicyWindow.hitRatio = win <= want ? 1.0f : (float)want / (float)win;
      av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      av.accessPolicyWindow.missProp = cudaAccessPropertyNormal;
      region_window_on = true;
    } else if (!region_window_on) {
      return;
    } else {
      region_window_on = false;
    }
    cudaStreamSetAttribute(stream, cudaStreamAttributeAccessPolicyWindow, &av);
    if (!region_window_on) cudaCtxResetPersistingL2Cache();
    cudaGetLastError();
  }
  int jit_part_per_sm = 0;  // resident CTAs per SM of the specialised pass 1, 0: not asked yet
  int jit_ring_per_sm = -1; // the same for its ring variant, -1: not asked yet
  int64_t part_jit_launches = 0, slice_jit_launches = 0, part_ring_launches = 0;
  // DBX_AGG_PART_RING=0: pass 1 never takes the bulk-copy ring (both variants can then be compared in one process)
  bool part_ring = !(getenv("DBX_AGG_PART_RING") && atoi(getenv("DBX_AGG_PART_RING")) == 0);
  // The ring variant of pass 1 copies whole tiles of every column slot with the bulk-copy unit: it needs
  // byte-sized integer or float columns that start 16-byte aligned (a tile is then a multiple of 16 bytes).
  bool ring_fits(const AggKernelParams& kp) const {
    if (!part_ring) return false;
    for (int s = 0; s < plan.n_slots; ++s) {
      const DevCol& c = kp.cols[s];
      if (c.is_const) continue;
      if (dtype_size(c.dtype) == 0 || ((uintptr_t)c.data & 15)) return false;
    }
    return true;
  }
  template <int NS>
  int32_t launch_partition(const AggKernelParams& kp, const PartitionOut& po) {
    if (device < 0 || device >= 64) { err.set("device index out of range"); return DBX_ERR_INVALID; }
    const int64_t n_tiles = (kp.n_rows + kTileRows - 1) / kTileRows;
    const bool ring = ring_fits(kp);
    if (jit.two_pass_ok() && ring && jit_ring_per_sm < 0) {
      int n = 0;
      const cudaError_t ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, (const void*)jit.part_ring, kRingThreads, ring_smem_bytes<NS>());
      if (ce == cudaSuccess) jit_ring_per_sm = n;
      else drop_two_pass_jit("occupancy query", ce);
    }
    if (jit.two_pass_ok() && ring && jit_ring_per_sm > 0) {  // one persistent CTA per SM
      const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(n_tiles, (int64_t)kNumSMs * jit_ring_per_sm));
      void* args[] = {(void*)&kp, (void*)&po};
      const cudaError_t ce = cudaLaunchKernel((const void*)jit.part_ring, dim3(grid), dim3(kRingThreads), args, ring_smem_bytes<NS>(), stream);
      if (ce == cudaSuccess) { ++part_jit_launches; ++part_ring_launches; return DBX_OK; }
      drop_two_pass_jit("launch", ce);
    }
    const size_t smem = partition_smem_bytes<NS>();
    if (jit.two_pass_ok() && !jit_part_per_sm) {  // the occupancy of the kernel that will run
      int n = 0;
      const cudaError_t ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, (const void*)jit.part, kBlock, smem);
      if (ce == cudaSuccess) jit_part_per_sm = std::max(1, n);
      else drop_two_pass_jit("occupancy query", ce);
    }
    if (jit.two_pass_ok()) {
      const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(n_tiles, (int64_t)kNumSMs * jit_part_per_sm));
      void* args[] = {(void*)&kp, (void*)&po};
      const cudaError_t ce = cudaLaunchKernel((const void*)jit.part, dim3(grid), dim3(kBlock), args, smem, stream);
      if (ce == cudaSuccess) { ++part_jit_launches; return DBX_OK; }
      drop_two_pass_jit("launch", ce);
    }
    if (kp.n_comp > 0) return ring ? launch_partition_ring_kernel<NS, true>(kp, po) : launch_partition_kernel<NS, true>(kp, po);
    return ring ? launch_partition_ring_kernel<NS, false>(kp, po) : launch_partition_kernel<NS, false>(kp, po);
  }
  template <int NS, bool EXPR>
  int32_t launch_partition_kernel(const AggKernelParams& kp, const PartitionOut& po) {
    static std::atomic<int> per_sm[64];  // resident CTAs per SM, 0: not asked yet
    const size_t smem = partition_smem_bytes<NS>();
    if (!per_sm[device]) {
      cudaFuncSetAttribute(filter_partition_kernel<NS, EXPR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      int n = 0;
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, filter_partition_kernel<NS, EXPR>, kBlock, smem);
      per_sm[device] = std::max(1, n);
    }
    // one resident wave: a CTA copies its survivors out only every few tiles, more CTAs would only add partial batches
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((kp.n_rows + kTileRows - 1) / kTileRows, (int64_t)kNumSMs * per_sm[device]));
    filter_partition_kernel<NS, EXPR><<<grid, kBlock, smem, stream>>>(kp, po);
    return DBX_OK;
  }
  template <int NS, bool EXPR>
  int32_t launch_partition_ring_kernel(const AggKernelParams& kp, const PartitionOut& po) {
    static std::atomic<int> per_sm[64];  // resident CTAs per SM, -1: the kernel does not fit, 0: not asked yet
    const size_t smem = ring_smem_bytes<NS>();
    if (!per_sm[device]) {
      cudaFuncSetAttribute(filter_partition_ring_kernel<NS, EXPR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      int n = 0;
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, filter_partition_ring_kernel<NS, EXPR>, kRingThreads, smem);
      cudaGetLastError();
      per_sm[device] = n > 0 ? n : -1;
    }
    if (per_sm[device] < 0) return launch_partition_kernel<NS, EXPR>(kp, po);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((kp.n_rows + kTileRows - 1) / kTileRows, (int64_t)kNumSMs * per_sm[device]));
    filter_partition_ring_kernel<NS, EXPR><<<grid, kRingThreads, smem, stream>>>(kp, po);
    ++part_ring_launches;
    return DBX_OK;
  }
  template <int NS>
  int32_t launch_slice_agg(const AggKernelParams& kp, const SliceIn& si, int n_parts, size_t slice_bytes) {
    static std::atomic<bool> attr_set[64];
    if (device < 0 || device >= 64) { err.set("device index out of range"); return DBX_ERR_INVALID; }
    const size_t smem = slice_bytes + slice_stage_bytes<NS>();  // the slice, then the two row buffers
    if (jit.two_pass_ok()) {
      void* args[] = {(void*)&kp, (void*)&si};
      const cudaError_t ce = cudaLaunchKernel((const void*)jit.slice, dim3(n_parts), dim3(kSliceBlock), args, smem, stream);
      if (ce == cudaSuccess) { ++slice_jit_launches; return DBX_OK; }
      drop_two_pass_jit("launch", ce);
    }
    if (!attr_set[device]) {
      cudaFuncSetAttribute(slice_agg_kernel<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSliceBytes + slice_stage_bytes<NS>()));
      attr_set[device] = true;
    }
    slice_agg_kernel<NS><<<n_parts, kSliceBlock, smem, stream>>>(kp, si);
    return DBX_OK;
  }
  // Slots per shared-memory slice of the table (whole buckets, a power of two), or 0 when the table
  // has more slices than pass 1 can partition into, or when the groups (known so far, or of the previous
  // query) would fill more than half of it: a slice that fills up defers most of its rows, which then
  // overflow and replay through the fused kernel.  Pass 2 then runs the fused kernel per L2-sized region.
  int64_t slice_slots() const {
    if (2 * std::max(groups_known, prev_query_groups) > table.cap) return 0;
    int64_t s = 4;
    while (2 * s * 8 * (1 + table.n_words) <= (int64_t)kSliceBytes && 2 * s <= table.cap) s *= 2;
    return table.cap / s <= kMaxPartitions ? s : 0;
  }
  // rows [row0, row0 + m) in two passes; *done = false when a partition overflowed (skewed keys): the caller takes the one-pass path
  int32_t partitioned_rows(const DevCol* cols, int64_t row0, int64_t m, bool* done) {
    *done = false;
    const int64_t slice = slice_slots();
    int n_parts = 2;
    if (slice) n_parts = (int)(table.cap / slice);
    else while (n_parts < kMaxRegions && (int64_t)table.bytes() / n_parts > part_region_bytes) n_parts <<= 1;
    const int64_t nb = table.cap >> 2;
    int lg_nb = 0, lg_p = 0;
    while ((1LL << lg_nb) < nb) ++lg_nb;
    while ((1 << lg_p) < n_parts) ++lg_p;
    if (lg_nb < lg_p) return DBX_OK;
    const int64_t cap_p = ((m / n_parts) * 3 / 2 + 8192 + 3) & ~3LL;  // hash-uniform partitions; skew overflows and falls back
    AggKernelParams kp;
    fill_params(&kp, cols, row0, m);
    PartitionOut po;
    memset(&po, 0, sizeof(po));
    for (int s = 0; s < plan.n_slots; ++s) {
      DBX_CUDA_TRY(err, part_buf[s].ensure((size_t)n_parts * cap_p * 8));
      po.out[s] = (uint64_t*)part_buf[s].p;
    }
    DBX_CUDA_TRY(err, part_cnt.ensure((kMaxPartitions + 1) * 8));
    DBX_CUDA_TRY(err, part_host.ensure((kMaxPartitions + 3) * 8));  // [P] overflow flag; [kMaxPartitions + 1, + 2] slice_agg_kernel's counts
    DBX_CUDA_TRY(err, cudaMemsetAsync(part_cnt.p, 0, (kMaxPartitions + 1) * 8, stream));
    po.counts = (unsigned long long*)part_cnt.p; po.cap_p = cap_p; po.nb_mask = (uint64_t)(nb - 1);
    po.region_shift = lg_nb - lg_p; po.n_parts = n_parts;
    DBX_TRY(by_slots(plan.n_slots, [&](auto s) { return launch_partition<decltype(s)::value>(kp, po); }));
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    DBX_CUDA_TRY(err, cudaMemcpyAsync(part_host.p, part_cnt.p, (size_t)(n_parts + 1) * 8, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const unsigned long long* hc = (const unsigned long long*)part_host.p;
    if (hc[n_parts]) { ++partition_fallbacks; return DBX_OK; }
    no_filter_ = true;
    int32_t rc = slice ? slice_pass(kp, po, slice, n_parts) : region_pass(n_parts, cap_p);
    no_filter_ = false;
    if (rc == DBX_OK) { *done = true; ++partitioned_chunks; slice_chunks += slice ? 1 : 0; }
    return rc;
  }
  // pass 2 in shared memory: one slice_agg_kernel launch, then the deferred rows through the fused kernel
  DevBuf deferred[kMaxSlots], n_deferred;
  int32_t slice_pass(AggKernelParams kp, const PartitionOut& po, int64_t slice, int n_parts) {
    const unsigned long long* hc = (const unsigned long long*)part_host.p;
    int64_t survivors = 0;
    for (int pi = 0; pi < n_parts; ++pi) survivors += (int64_t)hc[pi];
    for (int s = 0; s < plan.n_slots; ++s) DBX_CUDA_TRY(err, deferred[s].ensure((size_t)std::max<int64_t>(survivors, 1) * 8));
    DBX_CUDA_TRY(err, n_deferred.ensure(16));
    DBX_CUDA_TRY(err, cudaMemsetAsync(n_deferred.p, 0, 16, stream));
    SliceIn si;
    memset(&si, 0, sizeof(si));
    for (int s = 0; s < plan.n_slots; ++s) si.in[s] = po.out[s];
    si.counts = po.counts; si.cap_p = po.cap_p; si.slice_slots = slice;
    for (int s = 0; s < plan.n_slots; ++s) si.deferred[s] = (uint64_t*)deferred[s].p;
    si.n_deferred = (unsigned long long*)n_deferred.p;
    kp.table = table.view(nullptr);
    const size_t smem = (size_t)slice * 8 * (1 + plan.n_words);
    DBX_TRY(by_slots(plan.n_slots, [&](auto s) { return launch_slice_agg<decltype(s)::value>(kp, si, n_parts, smem); }));
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    DBX_CUDA_TRY(err, cudaMemcpyAsync((char*)part_host.p + (kMaxPartitions + 1) * 8, n_deferred.p, 16, cudaMemcpyDeviceToHost, stream));
    unsigned long long ng = 0, no = 0;
    DBX_TRY(read_counters(&ng, &no));
    const int64_t n_def = (int64_t)((const unsigned long long*)part_host.p)[kMaxPartitions + 1];
    const int64_t n_full = (int64_t)((const unsigned long long*)part_host.p)[kMaxPartitions + 2];
    // slices at their fill limit: the table holds fewer slots than the groups need; grow it (the rule of
    // agg_rows' overflow path) before the deferred rows run, instead of letting them find it full
    if (n_full > 0) DBX_TRY(grow_to(next_pow2(std::max<int64_t>(table.cap * 4, 2 * (int64_t)ng))));
    if (n_def > 0) {
      DevCol pc[kMaxSlots];
      for (int s = 0; s < plan.n_slots; ++s) {
        memset(&pc[s], 0, sizeof(DevCol));
        pc[s].dtype = DBX_U64;  // 64-bit images as the loads would have widened them
        pc[s].data = deferred[s].p;
      }
      return agg_rows(pc, 0, n_def);
    }
    if ((int64_t)ng * 2 > table.cap) DBX_TRY(grow_to(next_pow2(4 * (int64_t)ng)));
    return DBX_OK;
  }
  // pass 2 through the fused kernel, one launch per partition, with the partition's table region pinned in L2
  int32_t region_pass(int n_parts, int64_t cap_p) {
    const unsigned long long* hc = (const unsigned long long*)part_host.p;
    int32_t rc = DBX_OK;
    const int64_t cap_at_start = table.cap;
    for (int pi = 0; pi < n_parts && rc == DBX_OK; ++pi) {
      const int64_t cnt = (int64_t)hc[pi];
      if (!cnt) continue;
      // keep the state words of THIS region in L2 while its rows stream through (they take the reductions;
      // the key buckets are read with evict-last hints)
      if (plan.l2_persist && table.cap == cap_at_start) {
        const int64_t slots = table.cap / n_parts;
        region_window((char*)table.states_p + (size_t)pi * slots * plan.n_words * 8, (size_t)slots * plan.n_words * 8);
      }
      DevCol pc[kMaxSlots];
      for (int s = 0; s < plan.n_slots; ++s) {
        memset(&pc[s], 0, sizeof(DevCol));
        pc[s].dtype = DBX_U64;  // 64-bit images as the loads would have widened them
        pc[s].data = (const char*)part_buf[s].p + (size_t)pi * cap_p * 8;
      }
      rc = agg_rows(pc, 0, cnt);
    }
    region_window(nullptr, 0);
    return rc;
  }

  int32_t process_rows(const DevCol* cols, int64_t n) {
    DBX_TRY(timing_begin());
    for (int64_t row0 = 0; row0 < n; row0 += kChunkRows) {
      const int64_t m = std::min(kChunkRows, n - row0);
      if (partition_eligible(cols, m)) {
        for (int64_t sub = 0; sub < m; sub += kPartChunkRows) {
          const int64_t mm = std::min(kPartChunkRows, m - sub);
          bool done = false;
          DBX_TRY(partitioned_rows(cols, row0 + sub, mm, &done));
          if (!done) DBX_TRY(agg_rows(cols, row0 + sub, mm));
        }
        continue;
      }
      DBX_TRY(agg_rows(cols, row0, m));
    }
    DBX_TRY(timing_end());
    return DBX_OK;
  }
  // one chunk through the fused kernel (grouped: with overflow replay and growth)
  int32_t agg_rows(const DevCol* cols, int64_t row0, int64_t m) {
    {
      AggKernelParams kp;
      fill_params(&kp, cols, row0, m);
      if (!plan.grouped) {
        kp.table = table.view(nullptr);
        kp.single_state = (unsigned long long*)table.states_p;
        DBX_TRY(launch_single(kp));
        return DBX_OK;
      }
      // Insertions are provably within the load-factor budget when even "every row is a new
      // group" keeps the table at most half full: no overflow list, no host sync.
      const bool safe = (groups_known + rows_since_read + m) * 2 <= table.cap;
      if (safe) {
        kp.table = table.view(nullptr);
        if (want_hot()) { kp.hot_cache = 1; hot_probe_rows += m; }
        DBX_TRY(launch_grouped(kp, false));
        rows_since_read += m;
        return DBX_OK;
      }
      DBX_CUDA_TRY(err, ovf[0].ensure((size_t)m * 4));
      kp.table = table.view((uint32_t*)ovf[0].p);
      if (want_hot()) {  // groups a full table refuses at the end of the kernel come back as rows (merged below)
        hot_probe_rows += m;
        const size_t row_bytes = (size_t)(2 + plan.n_words) * 8;
        DBX_CUDA_TRY(err, hot_spill.ensure((size_t)kNumSMs * 8 * kHotSlots * row_bytes));
        kp.table.hot_spill = (uint64_t*)hot_spill.p;
        kp.hot_cache = 1;
      }
      DBX_TRY(launch_grouped(kp, false));
      unsigned long long ng = 0, no = 0;
      DBX_TRY(read_counters(&ng, &no));
      const unsigned long long n_spilled = hot_spilled;
      int cur = 0;
      while (no > 0) {  // rows whose group did not fit: grow and replay just those rows
        int64_t want = next_pow2(std::max<int64_t>(table.cap * 4, 2 * (int64_t)ng));
        DBX_TRY(grow_to(want));
        DBX_CUDA_TRY(err, cudaMemsetAsync(table.n_overflow(), 0, 8, stream));
        DBX_CUDA_TRY(err, ovf[cur ^ 1].ensure((size_t)no * 4));
        AggKernelParams kr;
        fill_params(&kr, cols, row0, (int64_t)no);
        kr.row_index = (const uint32_t*)ovf[cur].p;
        kr.table = table.view((uint32_t*)ovf[cur ^ 1].p);
        DBX_TRY(launch_grouped(kr, true));
        cur ^= 1;
        DBX_TRY(read_counters(&ng, &no));
      }
      if (n_spilled) {  // cached groups that found the table full: merge them now that it has room
        if (((int64_t)ng + (int64_t)n_spilled) * 2 > table.cap) DBX_TRY(grow_to(next_pow2(4 * ((int64_t)ng + (int64_t)n_spilled))));
        DBX_CUDA_TRY(err, cudaMemsetAsync((unsigned long long*)table.counters.p + 2, 0, 8, stream));
        rows_merge_kernel<<<grid_for_entries((int64_t)n_spilled), 256, 0, stream>>>((const uint64_t*)hot_spill.p, (int64_t)n_spilled, table.view(nullptr), plan.kinds);
        count_launch();
        DBX_CUDA_TRY(err, cudaGetLastError());
        DBX_TRY(read_counters(&ng, &no));
        if (no) { err.set("internal: aggregate table overflow while merging cached groups"); return DBX_ERR_CUDA; }
      }
      if ((int64_t)ng * 2 > table.cap) DBX_TRY(grow_to(next_pow2(4 * (int64_t)ng)));
    }
    return DBX_OK;
  }

  // Plans whose computed columns can raise read the error word here (the one synchronisation they add);
  // a failure poisons the operator until reset, so no state built from the failed input leaves it.
  int32_t finish() override {
    DBX_TRY(flush_batch());
    return check_expr_error();
  }
  // Every hand-off of the partial's state (finish, merge into a final, partition / serialize, exchange)
  // runs this after flushing, so state built from rows that failed to evaluate never leaves the operator.
  int32_t check_expr_error() {
    if (poisoned) { err.set(poison_msg); return DBX_ERR_STATE; }
    if (!plan.can_raise) return DBX_OK;
    DBX_CUDA_TRY(err, expr_err_host.ensure(8));
    DBX_CUDA_TRY(err, cudaMemcpyAsync(expr_err_host.p, expr_err.p, 8, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const unsigned long long w = *(const unsigned long long*)expr_err_host.p;
    if (w == ~0ULL) return DBX_OK;
    const int code = (int)(w & 0xFF);
    const int64_t row = (int64_t)(w >> 8);
    const char* msg = code == ERR_DIV_ZERO ? "Division by zero" : code == ERR_DIVIDED_BY_ZERO ? "divided by zero" : "number overflowed";
    poison(std::string(msg) + " while evaluating a computed column (first failing row " + std::to_string(row) + ")");
    return DBX_ERR_BAD_ARGUMENTS;
  }

  // The partial emits one metadata-only block (AggregateMeta::AggregatePayload): the payload
  // stays in HBM and is referenced through block.meta.
  int32_t pull(int32_t, dbx_block* out, int32_t* has_block) override {
    if (!finished) { err.set("pull before finish"); return DBX_ERR_STATE; }
    if (pulled) { *has_block = 0; return DBX_OK; }
    memset(out, 0, sizeof(*out));
    out->meta = this;
    *has_block = 1;
    pulled = true;
    return DBX_OK;
  }

  int32_t exact_groups(int64_t* n) {
    unsigned long long ng, no;
    DBX_TRY(flush_batch());
    DBX_TRY(ensure_table());
    DBX_TRY(read_counters(&ng, &no));
    if (no) { err.set("internal: rows were dropped by the partial table (overflow in safe mode)"); return DBX_ERR_CUDA; }
    *n = (int64_t)ng;
    return DBX_OK;
  }
};

// ================================================================ final
class AggFinalOp;
int32_t exchange_launch_merge(dbx_agg_exchange* x, AggFinalOp* f, int64_t cap);

class AggFinalOp : public Op {
 public:
  AggPlan plan;
  DeviceTable table;
  bool has_table = false;
  PinnedBuf host_counters;
  std::unique_ptr<OwnedBlock> result_dev;  // finalized columns in HBM
  int64_t result_rows = 0;
  bool pulled = false;
  unsigned long long* exchange_status = nullptr;  // device: set by a peer-memory exchange merge
  dbx_agg_exchange* exchange_src = nullptr;       // the exchange whose regions this table was merged from
  int64_t last_groups = 0;                        // result size of the previous query (sizing hint, survives reset)
  cudaEvent_t ev_fin_end = nullptr;               // recorded behind the finalize kernels (per-phase timing)
  bool fin_timed = false;
  ~AggFinalOp() override { if (ev_fin_end) cudaEventDestroy(ev_fin_end); }

  int32_t init(const dbx_agg_params* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int dev) {
    DBX_TRY(base_init(dev));
    DBX_TRY(build_plan(p, types, n, comp, n_comp, &plan, &err));
    DBX_CUDA_TRY(err, host_counters.ensure(64));
    DBX_CUDA_TRY(err, cudaEventCreate(&ev_fin_end));
    return DBX_OK;
  }
  int32_t reset() override {
    has_table = false;
    exchange_status = nullptr;
    exchange_src = nullptr;
    result_dev.reset();
    result_rows = 0;
    pulled = false;
    return DBX_OK;
  }

  int32_t read_groups(int64_t* ng, int64_t* no) {
    DBX_CUDA_TRY(err, cudaMemcpyAsync(host_counters.p, table.counters.p, 16, cudaMemcpyDeviceToHost, stream));
    if (exchange_status) DBX_CUDA_TRY(err, cudaMemcpyAsync((char*)host_counters.p + 16, exchange_status, 16, cudaMemcpyDeviceToHost, stream));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    *ng = (int64_t)((unsigned long long*)host_counters.p)[0];
    *no = (int64_t)((unsigned long long*)host_counters.p)[1];
    if (exchange_status) {
      const unsigned long long* st = (const unsigned long long*)host_counters.p + 2;
      if (st[0]) { err.set("exchange: timed out waiting for a peer rank's partition"); return DBX_ERR_STATE; }
      if (st[1]) { err.set("exchange: a peer had more groups for this rank than the receive region holds"); return DBX_ERR_OOM; }
    }
    return DBX_OK;
  }

  int32_t ensure_capacity(int64_t incoming) {
    if (!has_table) {
      int64_t cap = plan.grouped ? next_pow2(std::max<int64_t>(1024, 2 * incoming)) : 4;
      DBX_TRY(table.create(cap, plan, stream, &err));
      has_table = true;
      return DBX_OK;
    }
    if (!plan.grouped) return DBX_OK;
    int64_t ng, no;
    DBX_TRY(read_groups(&ng, &no));
    if ((ng + incoming) * 2 > table.cap) {
      DeviceTable nt;
      DBX_TRY(nt.create(next_pow2(2 * (ng + incoming)), plan, stream, &err));
      table_merge_kernel<<<grid_for_entries(table.cap + 2), 256, 0, stream>>>(table.view(nullptr), nt.view(nullptr), plan.kinds);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      table.swap(nt);
    }
    return DBX_OK;
  }

  // combine_payload of one partial's table (AggregateMeta::AggregatePayload)
  int32_t merge_partial(AggPartialOp* part) {
    if (finished) { err.set("merge after finish"); return DBX_ERR_STATE; }
    if (part->device != device) { err.set("partial and final operators live on different devices"); return DBX_ERR_INVALID; }
    if (part->plan.n_words != plan.n_words || part->plan.grouped != plan.grouped ||
        memcmp(&part->plan.kinds, &plan.kinds, sizeof(WordKinds)) != 0) {
      err.set("partial and final operators were created with different aggregate parameters");
      return DBX_ERR_INVALID;
    }
    {
      int32_t st = part->flush_batch();
      if (st == DBX_OK) st = part->check_expr_error();
      if (st == DBX_OK) st = part->ensure_table();
      if (st != DBX_OK) { err.set(part->err.msg); return st; }
    }
    DBX_CUDA_TRY(err, cudaStreamSynchronize(part->stream));  // partial's kernels precede the merge
    if (!has_table) {  // first partial: adopt its table (swap buffers), nothing to merge
      unsigned long long ng = 0, no = 0;
      int32_t st = part->read_counters(&ng, &no);
      if (st != DBX_OK) { err.set(part->err.msg); return st; }
      if (no) { err.set("internal: rows were dropped by the partial table (overflow in safe mode)"); return DBX_ERR_CUDA; }
      table.swap(part->table);
      has_table = true;
      part->table_ready = false;  // whatever buffer it now holds is re-created / cleared lazily
      part->table_clean = false;
      return DBX_OK;
    }
    int64_t pg = 0;
    {
      int32_t st = part->exact_groups(&pg);
      if (st != DBX_OK) { err.set(part->err.msg); return st; }
    }
    DBX_TRY(ensure_capacity(pg));
    table_merge_kernel<<<grid_for_entries(part->table.cap + 2), 256, 0, stream>>>(part->table.view(nullptr), table.view(nullptr), plan.kinds);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    int64_t ng, no;
    DBX_TRY(read_groups(&ng, &no));
    if (no) { err.set("internal: final table overflow during merge"); return DBX_ERR_CUDA; }
    return DBX_OK;
  }

  int32_t merge_rows(const void* dev_rows, int64_t n_rows) {
    if (finished) { err.set("merge after finish"); return DBX_ERR_STATE; }
    if (plan.key_words != 1) { err.set("128-bit packed group keys: exchange rows carry 64-bit keys only"); return DBX_ERR_UNSUPPORTED; }
    DBX_TRY(ensure_capacity(n_rows));
    if (n_rows == 0) return DBX_OK;
    // no GROUP BY: the rows are per-rank single states (FinalSingleStateAggregator,
    // transform_single_key.rs:232-278): merged by ONE thread in row (= rank) order, so f64 sums
    // are reproducible; grouped rows merge concurrently with REDs
    if (!plan.grouped) rows_merge_ordered_kernel<<<1, 32, 0, stream>>>((const uint64_t*)dev_rows, n_rows, table.view(nullptr), plan.kinds);
    else rows_merge_kernel<<<grid_for_entries(n_rows), 256, 0, stream>>>((const uint64_t*)dev_rows, n_rows, table.view(nullptr), plan.kinds);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    int64_t ng, no;
    DBX_TRY(read_groups(&ng, &no));
    if (no) { err.set("internal: final table overflow during merge"); return DBX_ERR_CUDA; }
    return DBX_OK;
  }

  // Final input port: blocks whose meta references a partial payload.
  int32_t push(const dbx_block* b) override {
    if (!b->meta) { err.set("AGG_FINAL consumes partial payload blocks (block.meta) or dbx_agg_final_merge_*"); return DBX_ERR_INVALID; }
    return merge_partial(reinterpret_cast<AggPartialOp*>(b->meta));
  }

  static int result_dtype(const FinalAgg& fa) {
    int cls = dtype_class(fa.arg_dtype);
    switch (fa.kind) {
      case DBX_AGG_COUNT: return DBX_U64;
      case DBX_AGG_AVG: return DBX_F64;
      case DBX_AGG_SUM: return cls == VC_FLT ? DBX_F64 : (cls == VC_INT ? DBX_I64 : DBX_U64);
      default: return fa.arg_dtype;
    }
  }

  // merge_result: compact the table into [aggs..., keys...] columns in HBM
  // The output columns are sized for the most groups a healthy table holds (half its slots) and
  // the finalize kernel is enqueued right away; the group count is read back afterwards, so the
  // whole operator costs ONE host synchronisation.  (A fuller table — only possible after merges
  // the host did not size — repeats the pass with the exact count.)
  int32_t finish() override {
    if (!has_table) DBX_TRY(ensure_capacity(0));
    int64_t ng = 0, no = 0;
    int32_t st = finalize_pass(plan.grouped ? table.cap / 2 + 2 : 1, &ng, &no);
    if (st != DBX_OK) return st;
    if (no && exchange_src) {
      // the table was sized from the previous query's result and this one has more groups: the
      // received regions are still intact, so merge them again into a worst-case table
      result_dev.reset();
      has_table = false;
      DBX_TRY(exchange_launch_merge(exchange_src, this, 0));
      DBX_TRY(finalize_pass(table.cap / 2 + 2, &ng, &no));
    }
    if (no) { err.set("internal: rows were dropped by the aggregate table (overflow)"); return DBX_ERR_CUDA; }
    last_groups = ng;
    if (ng > result_capacity) {
      result_dev.reset();
      DBX_TRY(finalize_pass(ng, &ng, &no));
    }
    result_rows = ng;
    for (dbx_column& c : result_dev->cols) c.len = ng;
    return DBX_OK;
  }

  int64_t result_capacity = 0;
  int32_t finalize_pass(int64_t capacity, int64_t* ng_out, int64_t* no_out) {
    auto ob = std::make_unique<OwnedBlock>();
    ob->stream = stream;  // freed in order behind this operator's enqueued work
    ob->device = device;
    const int64_t cap_rows = std::max<int64_t>(capacity, 1);
    const int64_t ng = cap_rows;  // column lengths are patched by finish() once the count is known
    result_capacity = cap_rows;
    auto dev_alloc = [&](size_t bytes, void** p) -> int32_t {
      DBX_CUDA_TRY(err, pool_alloc(device, stream, bytes, p));
      ob->dev_allocs.push_back(*p);
      return DBX_OK;
    };
    FinalizeParams fp;
    memset(&fp, 0, sizeof(fp));
    fp.n_aggs = plan.params.n_aggs;
    std::vector<uint8_t*> valid_bytes;  // per output column (nullptr = not nullable)
    for (int a = 0; a < fp.n_aggs; ++a) {
      fp.aggs[a] = plan.fin[a];
      int rdt = result_dtype(plan.fin[a]);
      void* vals = nullptr;
      DBX_TRY(dev_alloc((size_t)cap_rows * dtype_size(rdt), &vals));
      fp.aggs[a].out = vals;
      uint8_t* vb = nullptr;
      if (plan.fin[a].kind != DBX_AGG_COUNT) DBX_TRY(dev_alloc((size_t)cap_rows, (void**)&vb));
      fp.aggs[a].out_valid = vb;
      valid_bytes.push_back(vb);
      dbx_column c;
      memset(&c, 0, sizeof(c));
      c.dtype = rdt;
      c.mem = DBX_MEM_DEVICE;
      c.len = ng;
      c.data = vals;
      c.null_count = vb ? -1 : 0;
      ob->cols.push_back(c);
    }
    fp.key_dtype = -1;
    fp.n_key_parts = 0;
    if (plan.grouped && plan.n_key_parts > 1) {  // packed key -> one output column per group column
      fp.n_key_parts = plan.n_key_parts;
      memcpy(fp.key_parts, plan.key_parts, sizeof(plan.key_parts));
      for (int j = 0; j < plan.n_key_parts; ++j) {
        const int dt = plan.key_parts[j].dtype;
        void* kv = nullptr;
        DBX_TRY(dev_alloc((size_t)cap_rows * dtype_size(dt), &kv));
        fp.out_keys[j] = kv;
        uint8_t* vb = nullptr;
        if (plan.key_parts[j].null_shift >= 0) DBX_TRY(dev_alloc((size_t)cap_rows, (void**)&vb));
        fp.out_keys_valid[j] = vb;
        valid_bytes.push_back(vb);
        dbx_column c;
        memset(&c, 0, sizeof(c));
        c.dtype = dt;
        c.mem = DBX_MEM_DEVICE;
        c.len = ng;
        c.data = kv;
        c.null_count = vb ? -1 : 0;
        ob->cols.push_back(c);
      }
    } else if (plan.grouped) {
      fp.key_dtype = plan.key_dtype;
      void* kv = nullptr;
      DBX_TRY(dev_alloc((size_t)cap_rows * dtype_size(plan.key_dtype), &kv));
      fp.out_key = kv;
      uint8_t* vb = nullptr;
      if (plan.key_nullable) DBX_TRY(dev_alloc((size_t)cap_rows, (void**)&vb));
      fp.out_key_valid = vb;
      valid_bytes.push_back(vb);
      dbx_column c;
      memset(&c, 0, sizeof(c));
      c.dtype = plan.key_dtype;
      c.mem = DBX_MEM_DEVICE;
      c.len = ng;
      c.data = kv;
      c.null_count = vb ? -1 : 0;
      ob->cols.push_back(c);
    }
    unsigned long long* out_count = nullptr;
    DBX_TRY(dev_alloc(8, (void**)&out_count));
    DBX_CUDA_TRY(err, cudaMemsetAsync(out_count, 0, 8, stream));
    fp.out_count = out_count;
    fp.out_capacity = cap_rows;
    table_finalize_kernel<<<grid_for_entries(table.cap + 2), 256, 0, stream>>>(table.view(nullptr), fp);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    // validity bytes -> LSB-first bitmaps
    for (size_t i = 0; i < valid_bytes.size(); ++i) {
      if (!valid_bytes[i]) continue;
      uint8_t* bits = nullptr;
      DBX_TRY(dev_alloc((size_t)(cap_rows + 7) / 8 + 8, (void**)&bits));
      pack_validity_kernel<<<grid_for_entries((ng + 7) / 8 + 1), 256, 0, stream>>>(valid_bytes[i], out_count, cap_rows, bits);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      ob->cols[i].validity = bits;
      ob->cols[i].validity_bit_offset = 0;
    }
    result_dev = std::move(ob);
    DBX_CUDA_TRY(err, cudaEventRecord(ev_fin_end, stream));
    fin_timed = true;
    return read_groups(ng_out, no_out);  // the one synchronisation: also completes the kernels above
  }

  int32_t pull(int32_t out_mem, dbx_block* out, int32_t* has_block) override {
    if (!finished) { err.set("pull before finish"); return DBX_ERR_STATE; }
    if (pulled || !result_dev) { *has_block = 0; return DBX_OK; }
    pulled = true;
    *has_block = 1;
    return pull_owned_block(result_dev, device, stream, err, out_mem, out);
  }
};

// exclusive prefix sum of the per-tile selection counts: ONE CTA walks the array in chunks of
// 1024 with a running carry (<= 2 Mi tiles: a few microseconds); offsets[n] = total
__global__ void __launch_bounds__(1024) tile_scan_kernel(const uint32_t* counts, uint32_t* offsets, int64_t n) {
  constexpr int kPer = 8;  // consecutive tiles per thread and step
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int64_t i0 = 0; i0 < n; i0 += 1024 * kPer) {
    const int64_t i = i0 + (int64_t)threadIdx.x * kPer;
    uint32_t c[kPer], sum = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) { c[j] = i + j < n ? counts[i + j] : 0; sum += c[j]; }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint32_t w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += up;
      }
      s_warp[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const uint32_t base = s_carry + (warp ? s_warp[warp - 1] : 0);
    uint32_t run = base + incl - sum;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      if (i + j < n) offsets[i + j] = run;
      run += c[j];
    }
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = base + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) offsets[n] = s_carry;
}

// ================================================================ standalone filter
// TransformFilter (filter_predicate.rs:35-104): Transform::transform(DataBlock) -> DataBlock, one
// output block per pushed block, rows in input order.  BlockEntry::Const columns stay const.
class FilterOp : public Op {
 public:
  AggPlan plan;
  Stager stager;
  DevBuf nibbles, tile_counts, tile_offsets, dev_total;
  PinnedBuf host;
  std::vector<std::unique_ptr<OwnedBlock>> out_q;
  size_t out_head = 0;
  int64_t rows_in = 0, rows_out = 0;

  int32_t init(const dbx_predicate* pred, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int dev) {
    DBX_TRY(base_init(dev));
    dbx_agg_params ap;
    memset(&ap, 0, sizeof(ap));
    ap.filter = *pred;
    DBX_TRY(build_plan(&ap, types, n, comp, n_comp, &plan, &err));
    for (int i = 0; i < n; ++i)
      if (plan.col_dtype[i] != DBX_BOOL && dtype_size(plan.col_dtype[i]) == 0) { err.set("filter: unsupported column type (numeric and boolean columns only)"); return DBX_ERR_UNSUPPORTED; }
    DBX_TRY(stager.init(dev, stream, &err));
    DBX_CUDA_TRY(err, host.ensure(64));
    DBX_CUDA_TRY(err, dev_total.ensure(64));
    return DBX_OK;
  }
  int32_t reset() override { out_q.clear(); out_head = 0; rows_in = rows_out = 0; return DBX_OK; }

  int32_t push(const dbx_block* b) override {
    if (b->num_cols != plan.n_cols) { err.set("push: block column count differs from the operator's input schema"); return DBX_ERR_INVALID; }
    for (int i = 0; i < plan.n_cols; ++i) {
      if (b->cols[i].dtype != plan.col_dtype[i]) { err.set("push: block column dtype differs from the operator's input schema"); return DBX_ERR_INVALID; }
      if (b->cols[i].len != b->num_rows) { err.set("push: column length differs from num_rows"); return DBX_ERR_INVALID; }
    }
    const int64_t n = b->num_rows;
    if (n >= (1LL << 31)) { err.set("filter: blocks of 2^31 rows or more are not supported"); return DBX_ERR_UNSUPPORTED; }
    if (plan.div_by_zero && n > 0) {  // rem_scalar: divisor literal 0 fails the whole block (arithmetic_modulo.rs:137-140)
      err.set("Division by zero, during run expr: modulo (first failing row 0)");
      return DBX_ERR_BAD_ARGUMENTS;
    }
    rows_in += n;
    auto ob = std::make_unique<OwnedBlock>();
    ob->stream = stream;  // freed in order behind this operator's enqueued work
    ob->device = device;
    const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
    int64_t total = 0;
    DevCol pcols[kMaxSlots];
    DevCol ccols[64];
    if (n > 0) {
      DBX_TRY(stager.begin());
      int col_slot[64];
      for (int c = 0; c < plan.n_cols; ++c) col_slot[c] = -1;
      for (int s = 0; s < plan.n_slots; ++s) {
        if (plan.slot_col[s] < 0) { memset(&pcols[s], 0, sizeof(DevCol)); pcols[s].dtype = DBX_U64; pcols[s].is_const = 1; continue; }
        DBX_TRY(stager.stage(b->cols[plan.slot_col[s]], s, &pcols[s]));
        col_slot[plan.slot_col[s]] = s;
      }
      for (int c = 0; c < plan.n_cols; ++c) {
        if (col_slot[c] >= 0) ccols[c] = pcols[col_slot[c]];
        else DBX_TRY(stager.stage(b->cols[c], plan.n_slots + c, &ccols[c]));
      }
      DBX_CUDA_TRY(err, nibbles.ensure((size_t)n_tiles * kBlock));
      DBX_CUDA_TRY(err, tile_counts.ensure((size_t)(n_tiles + 1) * 4));
      DBX_CUDA_TRY(err, tile_offsets.ensure((size_t)(n_tiles + 1) * 4));
      AggKernelParams kp;
      memset(&kp, 0, sizeof(kp));
      for (int s = 0; s < plan.n_slots; ++s) kp.cols[s] = pcols[s];
      memcpy(kp.nodes, plan.nodes, sizeof(PredNodeDev) * plan.n_nodes);
      kp.n_rows = n; kp.n_slots = plan.n_slots; kp.n_nodes = plan.n_nodes; kp.key_slot = -1;
      if (plan.n_comp_ev) {  // computed predicate operands (they cannot raise: allocate_slots refuses those)
        kp.n_comp = plan.n_comp_ev; kp.comp_pred = plan.comp_pred; kp.fresh_slots = plan.fresh_slots;
        memcpy(kp.comp, plan.comp, sizeof(plan.comp));
        memcpy(kp.cnodes, plan.cnodes, sizeof(NodeDev) * plan.n_cnodes);
      }
      const int grid = grid_for_rows(n);
      DBX_TRY(timing_begin());
      by_slots(plan.n_slots, [&](auto s) {
        constexpr int NS = decltype(s)::value;
        if (kp.n_comp > 0) filter_select_kernel<NS, true><<<grid, kBlock, 0, stream>>>(kp, (uint8_t*)nibbles.p, (uint32_t*)tile_counts.p);
        else filter_select_kernel<NS><<<grid, kBlock, 0, stream>>>(kp, (uint8_t*)nibbles.p, (uint32_t*)tile_counts.p);
      });
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      tile_scan_kernel<<<1, 1024, 0, stream>>>((const uint32_t*)tile_counts.p, (uint32_t*)tile_offsets.p, n_tiles);
      count_launch();
      uint32_t* h = (uint32_t*)host.p;
      DBX_CUDA_TRY(err, cudaMemcpyAsync(h, (uint32_t*)tile_offsets.p + n_tiles, 4, cudaMemcpyDeviceToHost, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      total = (int64_t)h[0];
      unsigned long long t64 = (unsigned long long)total;
      DBX_CUDA_TRY(err, cudaMemcpyAsync(dev_total.p, &t64, 8, cudaMemcpyHostToDevice, stream));
    }
    rows_out += total;
    auto dev_alloc = [&](size_t bytes, void** p) -> int32_t {
      DBX_CUDA_TRY(err, pool_alloc(device, stream, bytes ? bytes : 1, p));
      ob->dev_allocs.push_back(*p);
      return DBX_OK;
    };
    TakeParams tp;
    memset(&tp, 0, sizeof(tp));
    struct Pack { uint8_t* bytes; int col; bool is_data; };
    std::vector<Pack> packs;
    int n_take = 0;
    for (int c = 0; c < plan.n_cols; ++c) {
      const dbx_column& ic = b->cols[c];
      dbx_column oc;
      memset(&oc, 0, sizeof(oc));
      oc.dtype = ic.dtype; oc.mem = DBX_MEM_DEVICE; oc.len = total; oc.vec_dim = 0; oc.null_count = 0;
      if (ic.is_const) {  // BlockEntry::Const survives a filter as a shorter const entry
        oc.is_const = 1; oc.konst = ic.konst; oc.mem = DBX_MEM_HOST;
        ob->cols.push_back(oc);
        continue;
      }
      if (total > 0) {
        TakeCol& tc = tp.cols[n_take++];
        tc.src = ccols[c].data; tc.src_valid = ccols[c].validity; tc.src_vbit_off = ccols[c].vbit_off; tc.src_dbit_off = ccols[c].dbit_off;
        tc.dtype = ic.dtype; tc.is_const = 0;
        void* vals = nullptr;
        DBX_TRY(dev_alloc(ic.dtype == DBX_BOOL ? (size_t)total : (size_t)total * dtype_size(ic.dtype), &vals));
        tc.dst = vals;
        oc.data = vals;
        if (ic.dtype == DBX_BOOL) packs.push_back(Pack{(uint8_t*)vals, (int)ob->cols.size(), true});
        if (ic.validity) {
          uint8_t* vb = nullptr;
          DBX_TRY(dev_alloc((size_t)total, (void**)&vb));
          tc.dst_valid = vb;
          packs.push_back(Pack{vb, (int)ob->cols.size(), false});
          oc.null_count = -1;
        }
      }
      ob->cols.push_back(oc);
    }
    if (total > 0) {
      tp.n_cols = n_take; tp.n_rows = n; tp.sel_nibbles = (const uint8_t*)nibbles.p; tp.tile_offsets = (const uint32_t*)tile_offsets.p;
      filter_take_kernel<<<grid_for_rows(n), kBlock, 0, stream>>>(tp);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      for (const Pack& pk : packs) {
        uint8_t* bits = nullptr;
        DBX_TRY(dev_alloc((size_t)(total + 7) / 8 + 8, (void**)&bits));
        pack_validity_kernel<<<grid_for_entries((total + 7) / 8 + 1), 256, 0, stream>>>(pk.bytes, (const unsigned long long*)dev_total.p, total, bits);
        count_launch();
        DBX_CUDA_TRY(err, cudaGetLastError());
        if (pk.is_data) { ob->cols[pk.col].data = bits; ob->cols[pk.col].data_bit_offset = 0; }
        else { ob->cols[pk.col].validity = bits; ob->cols[pk.col].validity_bit_offset = 0; }
      }
    }
    if (n > 0) {
      DBX_TRY(timing_end());
      DBX_TRY(stager.end());
    }
    out_q.push_back(std::move(ob));
    return DBX_OK;
  }

  int32_t finish() override { return DBX_OK; }

  // Transform is 1:1: output blocks can be pulled as soon as they were pushed
  int32_t pull(int32_t out_mem, dbx_block* out, int32_t* has_block) override {
    if (out_head >= out_q.size()) { *has_block = 0; return DBX_OK; }
    std::unique_ptr<OwnedBlock> ob = std::move(out_q[out_head++]);
    if (out_head == out_q.size()) { out_q.clear(); out_head = 0; }
    *has_block = 1;
    const int64_t rows = ob->cols.empty() ? 0 : ob->cols[0].len;
    int32_t st = pull_owned_block(ob, device, stream, err, out_mem, out);
    if (st == DBX_OK) out->num_rows = rows;
    return st;
  }
};

Op* make_filter_op(const dbx_predicate* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int device, int32_t* st) {
  auto* op = new FilterOp();
  *st = op->init(p, types, n, comp, n_comp, device);
  if (*st != DBX_OK) { g_create_error.set(op->err.msg); delete op; return nullptr; }
  return op;
}

Op* make_agg_partial_op(const dbx_agg_params* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int device,
                        int32_t* st) {
  auto* op = new AggPartialOp();
  *st = op->init(p, types, n, comp, n_comp, device);
  if (*st != DBX_OK) { g_create_error.set(op->err.msg); delete op; return nullptr; }
  return op;
}
Op* make_agg_final_op(const dbx_agg_params* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int device,
                      int32_t* st) {
  auto* op = new AggFinalOp();
  *st = op->init(p, types, n, comp, n_comp, device);
  if (*st != DBX_OK) { g_create_error.set(op->err.msg); delete op; return nullptr; }
  return op;
}

}  // namespace dbx

using namespace dbx;

extern "C" {

int32_t dbx_agg_final_merge_partial(dbx_op* final_op, dbx_op* partial_op) {
  if (!final_op || !partial_op) return DBX_ERR_INVALID;
  Op* f = reinterpret_cast<Op*>(final_op);
  Op* p = reinterpret_cast<Op*>(partial_op);
  if (f->kind != DBX_OP_AGG_FINAL || p->kind != DBX_OP_AGG_PARTIAL) { f->err.set("merge_partial: wrong operator kinds"); return DBX_ERR_INVALID; }
  DBX_CUDA_TRY(f->err, cudaSetDevice(f->device));
  return static_cast<AggFinalOp*>(f)->merge_partial(static_cast<AggPartialOp*>(p));
}

int32_t dbx_agg_partial_partition(dbx_op* partial_op, int32_t n_parts, void** dev_rows, int64_t* part_offsets,
                                  int32_t* row_bytes) {
  if (!partial_op || !dev_rows || !part_offsets || !row_bytes || n_parts < 1 || n_parts > 4096) return DBX_ERR_INVALID;
  Op* o = reinterpret_cast<Op*>(partial_op);
  if (o->kind != DBX_OP_AGG_PARTIAL) { o->err.set("partition: not a partial aggregate operator"); return DBX_ERR_INVALID; }
  AggPartialOp* p = static_cast<AggPartialOp*>(o);
  if (p->plan.key_words != 1) { p->err.set("128-bit packed group keys: the row exchange / serialisation formats carry 64-bit keys only (single-GPU partial -> final hand-off works)"); return DBX_ERR_UNSUPPORTED; }
  DBX_CUDA_TRY(p->err, cudaSetDevice(p->device));
  DBX_TRY(p->flush_batch());
  DBX_TRY(p->check_expr_error());
  DevBuf counts;
  DBX_CUDA_TRY(p->err, counts.ensure((size_t)n_parts * 8));
  DBX_CUDA_TRY(p->err, cudaMemsetAsync(counts.p, 0, (size_t)n_parts * 8, p->stream));
  TableDev tv = p->table.view(nullptr);
  int grid = grid_for_entries(tv.cap + 2);
  table_partition_count_kernel<<<grid, 256, (size_t)n_parts * 4, p->stream>>>(tv, n_parts, (unsigned long long*)counts.p);
  count_launch();
  DBX_CUDA_TRY(p->err, cudaGetLastError());
  std::vector<unsigned long long> h((size_t)n_parts);
  DBX_CUDA_TRY(p->err, cudaMemcpyAsync(h.data(), counts.p, (size_t)n_parts * 8, cudaMemcpyDeviceToHost, p->stream));
  DBX_CUDA_TRY(p->err, cudaStreamSynchronize(p->stream));
  std::vector<unsigned long long> cursors((size_t)n_parts);
  int64_t total = 0;
  for (int i = 0; i < n_parts; ++i) { part_offsets[i] = total; cursors[i] = (unsigned long long)total; total += (int64_t)h[i]; }
  part_offsets[n_parts] = total;
  const int rb = 8 * (2 + p->plan.n_words);
  *row_bytes = rb;
  void* rows = nullptr;
  DBX_CUDA_TRY(p->err, pool_alloc(p->device, p->stream, (size_t)std::max<int64_t>(total, 1) * rb, &rows));
  DBX_CUDA_TRY(p->err, cudaMemcpyAsync(counts.p, cursors.data(), (size_t)n_parts * 8, cudaMemcpyHostToDevice, p->stream));
  table_partition_scatter_kernel<<<grid, 256, 0, p->stream>>>(tv, n_parts, (unsigned long long*)counts.p, (uint64_t*)rows);
  count_launch();
  DBX_CUDA_TRY(p->err, cudaGetLastError());
  DBX_CUDA_TRY(p->err, cudaStreamSynchronize(p->stream));
  *dev_rows = rows;  // caller frees with dbx_device_free (stream-ordered pool)
  return DBX_OK;
}

// ---- spill_schema serde (see the layout comment above rows_to_spill_kernel)
namespace {
struct SpillFieldHost { int kind, word, cnt_word, dtype; };
struct SpillLayout {
  int n_fields = 0;
  SpillFieldHost f[dbx::kMaxSpillFields];
  int arity[DBX_MAX_AGGS] = {};
};
int sum_dtype(int arg_dtype) {  // ResultTypeOfUnary::Sum (arithmetics_type.rs:259-267)
  const int c = dbx::dtype_class(arg_dtype);
  return c == dbx::VC_FLT ? DBX_F64 : (c == dbx::VC_INT ? DBX_I64 : DBX_U64);
}
void spill_layout(const dbx::AggPlan& pl, SpillLayout* L) {
  using namespace dbx;
  for (int a = 0; a < pl.params.n_aggs; ++a) {
    const FinalAgg& fa = pl.fin[a];
    const int arg_col = pl.params.aggs[a].arg_col;
    const bool nullable_arg = arg_col >= 0 && pl.col_nullable[arg_col];
    const int first = L->n_fields;
    auto add = [&](int kind, int word, int dtype) { L->f[L->n_fields++] = SpillFieldHost{kind, word, fa.cnt_word, dtype}; };
    switch (fa.kind) {
      case DBX_AGG_COUNT: add(SPF_CNT, fa.cnt_word, DBX_U64); break;
      case DBX_AGG_SUM: add(SPF_ACC, fa.acc_word, sum_dtype(fa.arg_dtype)); break;
      case DBX_AGG_AVG: add(SPF_ACC, fa.acc_word, sum_dtype(fa.arg_dtype)); add(SPF_CNT, fa.cnt_word, DBX_U64); break;
      default: add(SPF_FLAG, fa.cnt_word, DBX_BOOL); add(SPF_VALUE, fa.acc_word, fa.arg_dtype); break;
    }
    if (fa.kind != DBX_AGG_COUNT) {
      if (nullable_arg) add(SPF_FLAG, fa.cnt_word, DBX_BOOL);  // AggregateNullUnaryAdaptor<true>
      add(SPF_FLAG, fa.cnt_word, DBX_BOOL);                    // AggregateFunctionOrNullAdaptor
    }
    L->arity[a] = L->n_fields - first;
  }
}
}  // namespace

int32_t dbx_agg_partial_serialize(dbx_op* partial_op, int32_t out_mem, dbx_block* out, int32_t* tuple_arity) {
  using namespace dbx;
  if (!partial_op || !out || !tuple_arity) return DBX_ERR_INVALID;
  Op* o = reinterpret_cast<Op*>(partial_op);
  if (o->kind != DBX_OP_AGG_PARTIAL) { o->err.set("serialize: not a partial aggregate operator"); return DBX_ERR_INVALID; }
  AggPartialOp* p = static_cast<AggPartialOp*>(o);
  const AggPlan& pl = p->plan;
  void* rows = nullptr;
  int64_t offs[2] = {0, 0};
  int32_t row_bytes = 0;
  DBX_TRY(dbx_agg_partial_partition(partial_op, 1, &rows, offs, &row_bytes));
  const int64_t n = offs[1];
  struct RowsGuard { int dev; void* p; cudaStream_t s; ~RowsGuard() { pool_free(dev, p, s); } } rows_guard{p->device, rows, p->stream};
  SpillLayout L;
  spill_layout(pl, &L);
  for (int a = 0; a < pl.params.n_aggs; ++a) tuple_arity[a] = L.arity[a];
  auto ob = std::make_unique<OwnedBlock>();
  ob->stream = p->stream;
  ob->device = p->device;
  const int64_t cap = std::max<int64_t>(n, 1);
  auto dev_alloc = [&](size_t bytes, void** q) -> int32_t {
    DBX_CUDA_TRY(p->err, pool_alloc(p->device, p->stream, bytes, q));
    ob->dev_allocs.push_back(*q);
    return DBX_OK;
  };
  SpillOutParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.n_fields = L.n_fields;
  sp.row_words = row_bytes / 8;
  std::vector<uint8_t*> bool_bytes, valid_bytes;  // per output column: byte-per-row staging to pack
  for (int i = 0; i < L.n_fields; ++i) {
    const SpillFieldHost& f = L.f[i];
    const size_t w = f.kind == SPF_FLAG ? 1 : (size_t)dtype_size(f.dtype);
    void* d = nullptr;
    DBX_TRY(dev_alloc((size_t)cap * w, &d));
    sp.f[i] = SpillFieldDev{f.kind, f.word, f.cnt_word, f.dtype, d};
    dbx_column c;
    memset(&c, 0, sizeof(c));
    c.dtype = f.dtype; c.mem = DBX_MEM_DEVICE; c.len = n; c.data = d;
    ob->cols.push_back(c);
    bool_bytes.push_back(f.kind == SPF_FLAG ? (uint8_t*)d : nullptr);
    valid_bytes.push_back(nullptr);
  }
  sp.key_dtype = -1;
  auto add_key = [&](int dt, bool nullable, void** kv, uint8_t** vb) -> int32_t {
    DBX_TRY(dev_alloc((size_t)cap * dtype_size(dt), kv));
    *vb = nullptr;
    if (nullable) DBX_TRY(dev_alloc((size_t)cap, (void**)vb));
    dbx_column c;
    memset(&c, 0, sizeof(c));
    c.dtype = dt; c.mem = DBX_MEM_DEVICE; c.len = n; c.data = *kv; c.null_count = nullable ? -1 : 0;
    ob->cols.push_back(c);
    bool_bytes.push_back(nullptr);
    valid_bytes.push_back(*vb);
    return DBX_OK;
  };
  if (pl.grouped && pl.n_key_parts > 1) {
    sp.n_key_parts = pl.n_key_parts;
    memcpy(sp.key_parts, pl.key_parts, sizeof(pl.key_parts));
    for (int j = 0; j < pl.n_key_parts; ++j) DBX_TRY(add_key(pl.key_parts[j].dtype, pl.key_parts[j].null_shift >= 0, &sp.out_keys[j], &sp.out_keys_valid[j]));
  } else if (pl.grouped) {
    sp.key_dtype = pl.key_dtype;
    DBX_TRY(add_key(pl.key_dtype, pl.key_nullable, &sp.out_key, &sp.out_key_valid));
  }
  if (n) {
    rows_to_spill_kernel<<<grid_for_entries(n), 256, 0, p->stream>>>((const uint64_t*)rows, n, sp);
    count_launch();
    DBX_CUDA_TRY(p->err, cudaGetLastError());
  }
  for (size_t i = 0; i < ob->cols.size(); ++i) {
    for (int pass = 0; pass < 2; ++pass) {
      uint8_t* bytes = pass == 0 ? bool_bytes[i] : valid_bytes[i];
      if (!bytes) continue;
      uint8_t* bits = nullptr;
      DBX_TRY(dev_alloc((size_t)(cap + 7) / 8 + 8, (void**)&bits));
      if (n) { pack_bytes_kernel<<<grid_for_entries((n + 7) / 8), 256, 0, p->stream>>>(bytes, n, bits); count_launch(); }
      if (pass == 0) { ob->cols[i].data = bits; ob->cols[i].data_bit_offset = 0; }
      else { ob->cols[i].validity = bits; ob->cols[i].validity_bit_offset = 0; }
    }
  }
  DBX_CUDA_TRY(p->err, cudaGetLastError());
  int32_t rc = pull_owned_block(ob, p->device, p->stream, p->err, out_mem, out);
  if (rc == DBX_OK) out->num_rows = n;
  return rc;
}

int32_t dbx_agg_final_merge_serialized(dbx_op* final_op, const dbx_block* block) {
  using namespace dbx;
  if (!final_op || !block) return DBX_ERR_INVALID;
  Op* o = reinterpret_cast<Op*>(final_op);
  if (o->kind != DBX_OP_AGG_FINAL) { o->err.set("merge_serialized: not a final aggregate operator"); return DBX_ERR_INVALID; }
  AggFinalOp* f = static_cast<AggFinalOp*>(o);
  const AggPlan& pl = f->plan;
  DBX_CUDA_TRY(f->err, cudaSetDevice(f->device));
  SpillLayout L;
  spill_layout(pl, &L);
  const int n_keys = !pl.grouped ? 0 : (pl.n_key_parts > 1 ? pl.n_key_parts : 1);
  if (block->num_cols != L.n_fields + n_keys) { f->err.set("merge_serialized: block does not have the spill schema's column count"); return DBX_ERR_INVALID; }
  const int64_t n = block->num_rows;
  SpillInParams sp;
  memset(&sp, 0, sizeof(sp));
  std::vector<DevBuf> owned;
  for (int c = 0; c < block->num_cols; ++c) {
    const dbx_column& col = block->cols[c];
    const int want = c < L.n_fields ? L.f[c].dtype : (pl.n_key_parts > 1 ? pl.key_parts[c - L.n_fields].dtype : pl.key_dtype);
    if (col.dtype != want || col.len != n || col.is_const) { f->err.set("merge_serialized: column " + std::to_string(c) + " does not match the spill schema"); return DBX_ERR_INVALID; }
    DevCol& dc = sp.cols[c];
    dc.dtype = col.dtype;
    if (col.mem == DBX_MEM_DEVICE) { dc.data = col.data; dc.validity = col.validity; dc.vbit_off = col.validity_bit_offset; dc.dbit_off = col.data_bit_offset; continue; }
    const bool is_bool = col.dtype == DBX_BOOL;
    const int64_t b0 = is_bool ? col.data_bit_offset >> 3 : 0;
    const size_t bytes = is_bool ? (size_t)(((col.data_bit_offset + n + 7) >> 3) - b0) : (size_t)n * dtype_size(col.dtype);
    owned.emplace_back();
    DBX_CUDA_TRY(f->err, owned.back().ensure(bytes ? bytes : 1));
    if (bytes) DBX_CUDA_TRY(f->err, cudaMemcpyAsync(owned.back().p, (const char*)col.data + b0, bytes, cudaMemcpyHostToDevice, f->stream));
    dc.data = owned.back().p;
    dc.dbit_off = is_bool ? (col.data_bit_offset & 7) : 0;
    if (col.validity) {
      const int64_t v0 = col.validity_bit_offset >> 3, v1 = (col.validity_bit_offset + n + 7) >> 3;
      owned.emplace_back();
      DBX_CUDA_TRY(f->err, owned.back().ensure((size_t)std::max<int64_t>(v1 - v0, 1)));
      if (v1 > v0) DBX_CUDA_TRY(f->err, cudaMemcpyAsync(owned.back().p, col.validity + v0, (size_t)(v1 - v0), cudaMemcpyHostToDevice, f->stream));
      dc.validity = (const uint8_t*)owned.back().p;
      dc.vbit_off = col.validity_bit_offset & 7;
    }
  }
  // where each state word comes from: an exact counter beats a flag beats "a group has >= 1 row"
  sp.n_words = pl.n_words;
  sp.row_words = 2 + pl.n_words;
  int rank[kMaxWords];
  for (int w = 0; w < pl.n_words; ++w) { sp.w[w] = WordSrcDev{WS_CNT_ONE, -1, -1, 0, pl.init.w[w]}; rank[w] = 0; }
  for (int i = 0; i < L.n_fields; ++i) {
    const SpillFieldHost& fd = L.f[i];
    if (fd.kind == SPF_CNT && rank[fd.word] < 3) { sp.w[fd.word] = WordSrcDev{WS_CNT_EXACT, i, -1, 0, pl.init.w[fd.word]}; rank[fd.word] = 3; }
    else if (fd.kind == SPF_FLAG && rank[fd.word] < 2) { sp.w[fd.word] = WordSrcDev{WS_CNT_FLAG, i, -1, 0, pl.init.w[fd.word]}; rank[fd.word] = 2; }
  }
  {
    int col = 0;
    for (int a = 0; a < pl.params.n_aggs; ++a) {
      const int first = col, last = col + L.arity[a] - 1;  // the last field of a non-count tuple is the or-null flag
      for (; col <= last; ++col) {
        const SpillFieldHost& fd = L.f[col];
        if (fd.kind == SPF_ACC) sp.w[fd.word] = WordSrcDev{WS_ACC_RAW, col, last, 0, pl.init.w[fd.word]};
        else if (fd.kind == SPF_VALUE) sp.w[fd.word] = WordSrcDev{WS_ACC_VALUE, col, first, 0, pl.init.w[fd.word]};
      }
    }
  }
  sp.key_col = pl.grouped ? L.n_fields : -1;
  sp.n_key_parts = pl.grouped && pl.n_key_parts > 1 ? pl.n_key_parts : 0;
  sp.key_is_float = pl.key_is_float ? 1 : 0;
  memcpy(sp.key_parts, pl.key_parts, sizeof(pl.key_parts));
  for (int j = 0; j < sp.n_key_parts; ++j) sp.key_parts[j].slot = L.n_fields + j;
  DevBuf rows;
  DBX_CUDA_TRY(f->err, rows.ensure((size_t)std::max<int64_t>(n, 1) * sp.row_words * 8));
  if (n) {
    spill_to_rows_kernel<<<grid_for_entries(n), 256, 0, f->stream>>>(sp, n, (uint64_t*)rows.p);
    count_launch();
    DBX_CUDA_TRY(f->err, cudaGetLastError());
  }
  return f->merge_rows(rows.p, n);  // synchronises the stream: the staging buffers can go
}

int32_t dbx_agg_final_merge_rows(dbx_op* final_op, const void* dev_rows, int64_t n_rows) {
  if (!final_op || (n_rows > 0 && !dev_rows) || n_rows < 0) return DBX_ERR_INVALID;
  Op* f = reinterpret_cast<Op*>(final_op);
  if (f->kind != DBX_OP_AGG_FINAL) { f->err.set("merge_rows: not a final aggregate operator"); return DBX_ERR_INVALID; }
  DBX_CUDA_TRY(f->err, cudaSetDevice(f->device));
  return static_cast<AggFinalOp*>(f)->merge_rows(dev_rows, n_rows);
}

}  // extern "C"

// ================================================================ peer-memory exchange
struct dbx_agg_exchange {
  dbx::ErrorSink err;
  int device = 0, rank = 0, n_ranks = 1, row_words = 0;
  int64_t region_rows = 0, table_cap = 0;
  dbx::DevBuf recv, scratch, status;  // scratch: [n_ranks] cursors + done counter
  dbx::PinnedBuf host_status;
  void* peer_base[dbx::kMaxRanks] = {};
  bool peer_is_ipc[dbx::kMaxRanks] = {};
  bool connected = false;
  bool fused_clear = true;
  long long spin_limit_ns = 5000LL * 1000 * 1000;
  unsigned long long epoch = 0;
  cudaEvent_t ev_scatter = nullptr, ev_merge = nullptr;  // cross-stream ordering (no timing)
  // per-phase timing of the last query: [0] scatter begin, [1] scatter end (partial's stream);
  // [2] wait begin, [3] wait end = merge begin, [4] merge end (final's stream)
  cudaEvent_t ev_t[5] = {};
  dbx::AggFinalOp* last_final = nullptr;
  size_t recv_bytes() const {
    return sizeof(dbx::ExchangeHeader) + (size_t)2 * n_ranks * region_rows * row_words * 8;
  }
};

extern "C" {

const char* dbx_agg_exchange_last_error(const dbx_agg_exchange* x) { return x ? x->err.msg.c_str() : g_create_error.msg.c_str(); }

int32_t dbx_agg_exchange_create(dbx_op* partial_op, int32_t rank, int32_t n_ranks, int64_t region_rows, dbx_agg_exchange** out,
                                void* ipc_handle_out) {
  if (!partial_op || !out || n_ranks < 1 || n_ranks > kMaxRanks || rank < 0 || rank >= n_ranks) { g_create_error.set("dbx_agg_exchange_create: bad argument"); return DBX_ERR_INVALID; }
  Op* o = reinterpret_cast<Op*>(partial_op);
  if (o->kind != DBX_OP_AGG_PARTIAL) { g_create_error.set("dbx_agg_exchange_create: not a partial aggregate operator"); return DBX_ERR_INVALID; }
  AggPartialOp* p = static_cast<AggPartialOp*>(o);
  if (!p->plan.grouped) { g_create_error.set("dbx_agg_exchange_create: aggregation without GROUP BY has no key to partition by: use dbx_agg_single_allreduce"); return DBX_ERR_UNSUPPORTED; }
  if (p->plan.key_words != 1) { g_create_error.set("dbx_agg_exchange_create: 128-bit packed group keys are not carried by the exchange rows (64-bit keys only)"); return DBX_ERR_UNSUPPORTED; }
  ErrorSink& err = g_create_error;
  std::unique_ptr<dbx_agg_exchange> x(new dbx_agg_exchange());
  x->device = p->device; x->rank = rank; x->n_ranks = n_ranks; x->row_words = 2 + p->plan.n_words;
  // a source can send at most all of its groups to one owner; a partial table holds at most cap/2
  x->region_rows = region_rows > 0 ? region_rows : std::max<int64_t>(p->initial_cap / 2 + 2, 1024);
  x->table_cap = std::max<int64_t>(p->initial_cap, next_pow2(2 * x->region_rows - 4));
  x->fused_clear = !(getenv("DBX_EXCH_FUSED_CLEAR") && atoi(getenv("DBX_EXCH_FUSED_CLEAR")) == 0);
  if (getenv("DBX_EXCH_SPIN_MS")) x->spin_limit_ns = atoll(getenv("DBX_EXCH_SPIN_MS")) * 1000000LL;
  DBX_CUDA_TRY(err, cudaSetDevice(x->device));
  DBX_CUDA_TRY(err, x->recv.ensure(x->recv_bytes()));
  DBX_CUDA_TRY(err, cudaMemset(x->recv.p, 0, sizeof(ExchangeHeader)));
  DBX_CUDA_TRY(err, x->scratch.ensure(8 * (kMaxRanks + 2)));
  DBX_CUDA_TRY(err, x->status.ensure(64));
  DBX_CUDA_TRY(err, cudaMemset(x->status.p, 0, 64));
  DBX_CUDA_TRY(err, x->host_status.ensure(64));
  DBX_CUDA_TRY(err, cudaEventCreateWithFlags(&x->ev_scatter, cudaEventDisableTiming));
  DBX_CUDA_TRY(err, cudaEventCreateWithFlags(&x->ev_merge, cudaEventDisableTiming));
  for (auto& e : x->ev_t) DBX_CUDA_TRY(err, cudaEventCreate(&e));
  if (ipc_handle_out) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t hd;
    DBX_CUDA_TRY(err, cudaIpcGetMemHandle(&hd, x->recv.p));
    memcpy(ipc_handle_out, &hd, 64);
  }
  *out = x.release();
  return DBX_OK;
}

int32_t dbx_agg_exchange_local_buffer(dbx_agg_exchange* x, void** base, int64_t* region_rows, int32_t* row_bytes) {
  if (!x) return DBX_ERR_INVALID;
  if (base) *base = x->recv.p;
  if (region_rows) *region_rows = x->region_rows;
  if (row_bytes) *row_bytes = x->row_words * 8;
  return DBX_OK;
}

/* all_handles: n_ranks x 64 bytes (cudaIpcMemHandle_t of every rank, own entry ignored), or
 * NULL when `same_process_ptrs` gives the receive buffers directly (ranks simulated in one process). */
int32_t dbx_agg_exchange_connect(dbx_agg_exchange* x, const void* all_handles, void* const* same_process_ptrs) {
  if (!x || (!all_handles && !same_process_ptrs)) return DBX_ERR_INVALID;
  DBX_CUDA_TRY(x->err, cudaSetDevice(x->device));
  for (int r = 0; r < x->n_ranks; ++r) {
    if (r == x->rank) { x->peer_base[r] = x->recv.p; continue; }
    if (same_process_ptrs) { x->peer_base[r] = same_process_ptrs[r]; continue; }
    cudaIpcMemHandle_t hd;
    memcpy(&hd, (const char*)all_handles + (size_t)r * 64, 64);
    void* p = nullptr;
    DBX_CUDA_TRY(x->err, cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess));
    x->peer_base[r] = p;
    x->peer_is_ipc[r] = true;
  }
  x->connected = true;
  return DBX_OK;
}

/* Hash-partition the finished partial's groups by owner and store every row straight into the
 * owner's receive region (peer memory).  Enqueued on the partial's stream; no host sync.  The
 * same pass re-initialises the partial's table, so the operator is re-armed for the next query
 * without a separate clear (dbx_op_reset on it then costs no kernel). */
int32_t dbx_agg_exchange_scatter(dbx_agg_exchange* x, dbx_op* partial_op) {
  if (!x || !partial_op) return DBX_ERR_INVALID;
  if (!x->connected) { x->err.set("exchange: scatter before connect"); return DBX_ERR_STATE; }
  AggPartialOp* p = static_cast<AggPartialOp*>(reinterpret_cast<Op*>(partial_op));
  DBX_CUDA_TRY(x->err, cudaSetDevice(x->device));
  { int32_t st = p->flush_batch(); if (st == DBX_OK) st = p->check_expr_error(); if (st == DBX_OK) st = p->ensure_table(); if (st != DBX_OK) { x->err.set(p->err.msg); return st; } }
  if (2 + p->plan.n_words != x->row_words) { x->err.set("exchange: operator state layout differs from the exchange's"); return DBX_ERR_INVALID; }
  x->epoch += 1;
  // region reuse: this rank's merge of the previous epoch must precede the scatter that lets peers move on
  DBX_CUDA_TRY(x->err, cudaStreamWaitEvent(p->stream, x->ev_merge, 0));
  DBX_CUDA_TRY(x->err, cudaEventRecord(x->ev_t[0], p->stream));
  DBX_CUDA_TRY(x->err, cudaMemsetAsync(x->scratch.p, 0, 8 * (kMaxRanks + 2), p->stream));
  ExchangeScatterParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.src = p->table.view(nullptr);
  for (int r = 0; r < x->n_ranks; ++r) sp.peer_base[r] = x->peer_base[r];
  sp.cursors = (unsigned long long*)x->scratch.p;
  sp.done = (unsigned int*)((unsigned long long*)x->scratch.p + kMaxRanks);
  sp.region_rows = x->region_rows;
  sp.epoch = x->epoch;
  sp.n_ranks = x->n_ranks; sp.rank = x->rank; sp.row_words = x->row_words; sp.parity = (int)(x->epoch & 1);
  sp.clear_src = x->fused_clear ? 1 : 0;
  sp.init = p->plan.init;
  {
    static std::atomic<bool> attr_set[64];
    if (!attr_set[x->device]) {
      DBX_CUDA_TRY(x->err, cudaFuncSetAttribute(exchange_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 256 * kScatterSlots * kExchMaxRowWords * 8));
      attr_set[x->device] = true;
    }
  }
  exchange_scatter_kernel<<<grid_for_entries((sp.src.cap + 2 + kScatterSlots - 1) / kScatterSlots), 256, (size_t)256 * kScatterSlots * x->row_words * 8, p->stream>>>(sp);
  count_launch();
  DBX_CUDA_TRY(x->err, cudaGetLastError());
  if (x->fused_clear) {  // the table is empty again: only the counters are left to reset
    DBX_CUDA_TRY(x->err, cudaMemsetAsync(p->table.counters.p, 0, 64, p->stream));
    p->table_clean = true;
    p->hot_absorbed_seen = 0;
  }
  DBX_CUDA_TRY(x->err, cudaEventRecord(x->ev_t[1], p->stream));
  DBX_CUDA_TRY(x->err, cudaEventRecord(x->ev_scatter, p->stream));
  return DBX_OK;
}

/* Merge every source's region of the current epoch into the final operator's table; a one-warp
 * kernel waits on the sources' release flags (device side), the merge grid follows it in stream
 * order.  Enqueued on the final's stream; no host sync. */
int32_t dbx_agg_exchange_merge(dbx_agg_exchange* x, dbx_op* final_op) {
  if (!x || !final_op) return DBX_ERR_INVALID;
  Op* o = reinterpret_cast<Op*>(final_op);
  if (o->kind != DBX_OP_AGG_FINAL) { x->err.set("exchange: merge target is not a final aggregate operator"); return DBX_ERR_INVALID; }
  AggFinalOp* f = static_cast<AggFinalOp*>(o);
  DBX_CUDA_TRY(x->err, cudaSetDevice(x->device));
  if (f->finished) { x->err.set("merge after finish"); return DBX_ERR_STATE; }
  if (f->has_table) { x->err.set("exchange: the final operator already holds merged state (reset it first; an exchange merge always starts a fresh table)"); return DBX_ERR_STATE; }
  // table size: from the previous query's result when there is one (an owner holds ~1/n_ranks of
  // the groups, so this is far smaller than the worst case and cheaper to clear and scan); finish()
  // falls back to the worst-case size if it turns out too small
  int64_t cap = 0;
  if (f->last_groups > 0) cap = std::min<int64_t>(x->table_cap, next_pow2(std::max<int64_t>(4 * f->last_groups, 1024)));
  DBX_TRY(exchange_launch_merge(x, f, cap));
  return DBX_OK;
}

/* Per-phase device times (ms, CUDA events) of the last scatter/merge pair, for bench.py's N > 1
 * line: out8[0] scatter kernel, [1] wait for the peers' flags (wait kernel, event-timed),
 * [2] merge kernel, [3] finalize (merge end -> result columns ready), [4] the wait kernel's own
 * measure of its spin (globaltimer), [5..7] reserved (0).  Call after the final's finish(). */
int32_t dbx_agg_exchange_phase_ms(dbx_agg_exchange* x, float* out8) {
  if (!x || !out8) return DBX_ERR_INVALID;
  DBX_CUDA_TRY(x->err, cudaSetDevice(x->device));
  for (int i = 0; i < 8; ++i) out8[i] = 0.f;
  if (x->epoch == 0) { x->err.set("exchange: no query timed yet"); return DBX_ERR_STATE; }
  DBX_CUDA_TRY(x->err, cudaEventSynchronize(x->ev_t[1]));
  DBX_CUDA_TRY(x->err, cudaEventSynchronize(x->ev_t[4]));
  DBX_CUDA_TRY(x->err, cudaEventElapsedTime(&out8[0], x->ev_t[0], x->ev_t[1]));
  DBX_CUDA_TRY(x->err, cudaEventElapsedTime(&out8[1], x->ev_t[2], x->ev_t[3]));
  DBX_CUDA_TRY(x->err, cudaEventElapsedTime(&out8[2], x->ev_t[3], x->ev_t[4]));
  if (x->last_final && x->last_final->fin_timed) {
    DBX_CUDA_TRY(x->err, cudaEventSynchronize(x->last_final->ev_fin_end));
    DBX_CUDA_TRY(x->err, cudaEventElapsedTime(&out8[3], x->ev_t[4], x->last_final->ev_fin_end));
  }
  DBX_CUDA_TRY(x->err, cudaMemcpy(x->host_status.p, x->status.p, 32, cudaMemcpyDeviceToHost));
  out8[4] = (float)(((unsigned long long*)x->host_status.p)[2] * 1e-6);
  return DBX_OK;
}

}  // extern "C"

namespace dbx {
// (re-)create the final's table with `cap` slots (0 = worst case) and merge the current epoch's regions
int32_t exchange_launch_merge(dbx_agg_exchange* x, AggFinalOp* f, int64_t cap) {
  if (cap <= 0) cap = x->table_cap;
  {
    int32_t st = f->table.create(cap, f->plan, f->stream, &f->err);
    if (st != DBX_OK) { x->err.set(f->err.msg); return st; }
    f->has_table = true;
  }
  DBX_CUDA_TRY(x->err, cudaStreamWaitEvent(f->stream, x->ev_scatter, 0));
  ExchangeMergeParams mp;
  memset(&mp, 0, sizeof(mp));
  mp.dst = f->table.view(nullptr);
  mp.kinds = f->plan.kinds;
  mp.base = x->recv.p;
  mp.status = (unsigned long long*)x->status.p;
  mp.region_rows = x->region_rows;
  mp.epoch = x->epoch;
  mp.spin_limit_ns = x->spin_limit_ns;  // a peer that never arrives must not hang the GPU
  mp.n_ranks = x->n_ranks; mp.row_words = x->row_words; mp.parity = (int)(x->epoch & 1);
  DBX_CUDA_TRY(x->err, cudaEventRecord(x->ev_t[2], f->stream));
  exchange_wait_kernel<<<1, 32, 0, f->stream>>>(mp);
  DBX_CUDA_TRY(x->err, cudaEventRecord(x->ev_t[3], f->stream));
  exchange_merge_kernel<<<grid_for_entries(x->region_rows), 256, 0, f->stream>>>(mp);
  count_launch(2);
  DBX_CUDA_TRY(x->err, cudaGetLastError());
  DBX_CUDA_TRY(x->err, cudaEventRecord(x->ev_t[4], f->stream));
  DBX_CUDA_TRY(x->err, cudaEventRecord(x->ev_merge, f->stream));
  f->exchange_status = (unsigned long long*)x->status.p;
  f->exchange_src = x;
  x->last_final = f;
  return DBX_OK;
}
}  // namespace dbx

extern "C" {

int32_t dbx_agg_exchange_destroy(dbx_agg_exchange* x) {
  if (!x) return DBX_OK;
  cudaSetDevice(x->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < x->n_ranks; ++r)
    if (x->peer_is_ipc[r] && x->peer_base[r]) cudaIpcCloseMemHandle(x->peer_base[r]);
  if (x->ev_scatter) cudaEventDestroy(x->ev_scatter);
  if (x->ev_merge) cudaEventDestroy(x->ev_merge);
  for (auto& e : x->ev_t)
    if (e) cudaEventDestroy(e);
  delete x;
  return DBX_OK;
}

}  // extern "C"
