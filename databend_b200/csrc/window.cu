// window.cu — DBX_OP_WINDOW: one WindowPartition and the chain of Window nodes that share its
// PARTITION BY / ORDER BY, on the device.
//
// Reference pipeline replaced (paths relative to the databend source tree):
//   WindowPartition (sort by partition + order keys)   src/query/service/src/physical_plans/physical_window_partition.rs
//   Window (one result column per node)                src/query/service/src/physical_plans/physical_window.rs
//   TransformWindow::add_block / merge_result_...      src/query/pipeline/transforms/src/processors/transforms/window/
//                                                      transform_window.rs:481-660, 1003-1153
//
// The reference walks the sorted rows one by one, advancing partition, peer group and frame bounds.
// Here every row's bounds come from scans over the sorted rows instead, so no row depends on the
// previous one:
//   push      every pushed block is copied to the device as it comes (dbx_block_concat of one block:
//             the caller's buffers are read before push returns)
//   finish    1. the blocks are concatenated and one stable sort by (partition keys, order keys) gives
//                the window order (sort_rows_by_keys, shared with ORDER BY);
//             2. the boundary kernel flags partition starts and peer-group starts from the sorted key
//                images and NULL flags (an image alone cannot tell a NULL from a value);
//             3. scans (reduce-then-scan over 2048-row tiles: a reduce pass, one CTA over the tile
//                totals, a scan pass with the tile's carry, so no CTA waits on another) give every
//                row its partition start / end, peer start / end (reverse scans for the ends), the
//                dense rank, and per aggregate argument a prefix sum and non-NULL count (global,
//                wrapping: differences are exact for integers) or a segmented running / suffix
//                sum, min or max (frames open on one side);
//             4. one emit kernel per function computes the row's frame [start, end) and its value;
//                frames bounded on both sides add (or compare) their rows one by one in row order,
//                which is the reference's order, so Float sums over them are bit-exact;
//             5. the input columns are gathered once into window order (dbx_block_take).
#include <algorithm>
#include <vector>

#include "sort_keys.cuh"

namespace dbx {

namespace {

// ================================================================ scans
constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems;
constexpr int kSpineThreads = 1024;

struct OpSumU32 { using T = uint32_t; __device__ static T id() { return 0; } __device__ static T f(T a, T b) { return a + b; } };
struct OpMaxU32 { using T = uint32_t; __device__ static T id() { return 0; } __device__ static T f(T a, T b) { return a > b ? a : b; } };
struct OpMinU32 { using T = uint32_t; __device__ static T id() { return 0xFFFFFFFFu; } __device__ static T f(T a, T b) { return a < b ? a : b; } };
struct OpSumU64 { using T = uint64_t; __device__ static T id() { return 0; } __device__ static T f(T a, T b) { return a + b; } };
struct OpMinU64 { using T = uint64_t; __device__ static T id() { return ~0ULL; } __device__ static T f(T a, T b) { return a < b ? a : b; } };
struct OpMaxU64 { using T = uint64_t; __device__ static T id() { return 0; } __device__ static T f(T a, T b) { return a > b ? a : b; } };
struct OpSumF64 {  // f64 bits
  using T = uint64_t;
  __device__ static T id() { return 0; }
  __device__ static T f(T a, T b) { return (T)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b)); }
};

// What a scan reads at physical row i: a value and (segmented scans) whether a segment starts there.
enum : int { SRC_START_IDX = 0, SRC_END_IDX = 1, SRC_FLAGS = 2, SRC_VALUES = 3, SRC_VALID = 4 };
struct ScanSrc {
  int32_t mode;
  int32_t segmented;         // SRC_VALUES: restart at partition starts (forward) / ends (reverse)
  const uint8_t* flags;      // SRC_START_IDX / SRC_END_IDX / SRC_FLAGS: boundary flags; segmented: partition starts
  const uint64_t* vals;      // SRC_VALUES
  const uint8_t* valid;      // SRC_VALUES / SRC_VALID: nullptr = all valid
  int64_t n;
};

template <class Op, bool REV>
__device__ __forceinline__ void scan_src(const ScanSrc& s, int64_t i, typename Op::T& v, bool& h) {
  using T = typename Op::T;
  h = false;
  switch (s.mode) {
    case SRC_START_IDX: v = s.flags[i] ? (T)i : (T)0; break;
    case SRC_END_IDX: v = (i + 1 < s.n && s.flags[i + 1]) ? (T)(i + 1) : (T)s.n; break;
    case SRC_FLAGS: v = s.flags[i]; break;
    case SRC_VALID: v = (!s.valid || s.valid[i]) ? 1 : 0; break;
    default:
      v = (!s.valid || s.valid[i]) ? (T)s.vals[i] : Op::id();
      if (s.segmented) h = REV ? (i + 1 == s.n || s.flags[i + 1]) : (s.flags[i] != 0);
      break;
  }
}

// (h, v) pairs under the segmented operator: (ha, va) . (hb, vb) = (ha | hb, hb ? vb : va op vb)
template <class Op>
struct Seg {
  typename Op::T v;
  bool h;
  __device__ __forceinline__ static Seg make(typename Op::T v, bool h) { Seg s; s.v = v; s.h = h; return s; }
  __device__ __forceinline__ Seg then(const Seg& b) const { return make(b.h ? b.v : Op::f(v, b.v), h || b.h); }
};

// Exclusive scan of one Seg per thread over the CTA (blockDim.x a multiple of 32, <= 1024); returns
// the thread's exclusive prefix and sets *total.
template <class Op>
__device__ __forceinline__ Seg<Op> block_exclusive(Seg<Op> x, Seg<Op>* total) {
  __shared__ typename Op::T s_v[32];
  __shared__ bool s_h[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  Seg<Op> inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Seg<Op> up = Seg<Op>::make(__shfl_up_sync(0xffffffffu, inc.v, o), __shfl_up_sync(0xffffffffu, inc.h, o));
    if (lane >= o) inc = up.then(inc);
  }
  if (lane == 31) { s_v[warp] = inc.v; s_h[warp] = inc.h; }
  __syncthreads();
  if (warp == 0) {
    Seg<Op> w = lane < n_warps ? Seg<Op>::make(s_v[lane], s_h[lane]) : Seg<Op>::make(Op::id(), false);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      Seg<Op> up = Seg<Op>::make(__shfl_up_sync(0xffffffffu, w.v, o), __shfl_up_sync(0xffffffffu, w.h, o));
      if (lane >= o) w = up.then(w);
    }
    s_v[lane] = w.v; s_h[lane] = w.h;  // inclusive over warps
  }
  __syncthreads();
  Seg<Op> wexc = Seg<Op>::make(__shfl_up_sync(0xffffffffu, inc.v, 1), __shfl_up_sync(0xffffffffu, inc.h, 1));
  if (lane == 0) wexc = Seg<Op>::make(Op::id(), false);
  Seg<Op> r = wexc;
  if (warp > 0) r = Seg<Op>::make(s_v[warp - 1], s_h[warp - 1]).then(wexc);
  *total = Seg<Op>::make(s_v[n_warps - 1], s_h[n_warps - 1]);
  __syncthreads();  // s_v / s_h are reused by the next call
  return r;
}

template <class Op, bool REV>
__device__ __forceinline__ void load_items(const ScanSrc& s, int64_t tile, Seg<Op> (&it)[kScanItems]) {
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t j = tile * kScanTile + (int64_t)threadIdx.x * kScanItems + k;
    typename Op::T v = Op::id();
    bool h = false;
    if (j < s.n) scan_src<Op, REV>(s, REV ? s.n - 1 - j : j, v, h);
    it[k] = Seg<Op>::make(v, h);
  }
}

template <class Op, bool REV>
__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(const __grid_constant__ ScanSrc s, typename Op::T* tile_v, uint8_t* tile_h) {
  Seg<Op> it[kScanItems];
  load_items<Op, REV>(s, blockIdx.x, it);
  Seg<Op> a = it[0];
#pragma unroll
  for (int k = 1; k < kScanItems; ++k) a = a.then(it[k]);
  Seg<Op> total;
  block_exclusive<Op>(a, &total);
  if (threadIdx.x == 0) { tile_v[blockIdx.x] = total.v; tile_h[blockIdx.x] = total.h; }
}

// one CTA: exclusive prefix of the tile totals (each thread walks a run of consecutive tiles)
template <class Op>
__global__ void __launch_bounds__(kSpineThreads) scan_spine_kernel(typename Op::T* tile_v, const uint8_t* tile_h, int64_t n_tiles) {
  const int64_t per = (n_tiles + kSpineThreads - 1) / kSpineThreads;
  const int64_t t0 = (int64_t)threadIdx.x * per, t1 = t0 + per < n_tiles ? t0 + per : n_tiles;
  Seg<Op> a = Seg<Op>::make(Op::id(), false);
  for (int64_t t = t0; t < t1; ++t) a = a.then(Seg<Op>::make(tile_v[t], tile_h[t] != 0));
  Seg<Op> total;
  Seg<Op> run = block_exclusive<Op>(a, &total);
  for (int64_t t = t0; t < t1; ++t) {
    const Seg<Op> x = Seg<Op>::make(tile_v[t], tile_h[t] != 0);
    tile_v[t] = run.v;  // exclusive carry of tile t
    run = run.then(x);
  }
}

template <class Op, bool REV>
__global__ void __maxnreg__(64) scan_tile_kernel(const __grid_constant__ ScanSrc s, const typename Op::T* tile_v, typename Op::T* out) {
  Seg<Op> it[kScanItems];
  load_items<Op, REV>(s, blockIdx.x, it);
  Seg<Op> a = it[0];
#pragma unroll
  for (int k = 1; k < kScanItems; ++k) a = a.then(it[k]);
  Seg<Op> total;
  Seg<Op> run = Seg<Op>::make(tile_v[blockIdx.x], false).then(block_exclusive<Op>(a, &total));
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t j = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems + k;
    run = run.then(it[k]);
    if (j < s.n) out[REV ? s.n - 1 - j : j] = run.v;
  }
}

// ================================================================ boundaries, gathers, emit
struct BoundArgs {
  const uint64_t* ord[DBX_MAX_SORT_KEYS];
  const uint32_t* rid[DBX_MAX_SORT_KEYS];
  int32_t n_keys, n_part;   // keys [0, n_part) are partition keys
  const uint32_t* perm;     // sorted row id | NULL flag; nullptr: input order
  int64_t n;
  uint8_t* part;            // 1 where a partition starts
  uint8_t* peer;            // 1 where a peer group starts (partition starts included)
  uint32_t* rows;           // sorted row ids
};
__global__ void __launch_bounds__(256) window_bounds_kernel(const __grid_constant__ BoundArgs a) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t r = a.perm ? (a.perm[i] & 0x7FFFFFFFu) : (uint32_t)i;
    bool part = i == 0, peer = i == 0;
    if (i > 0) {
      const uint32_t q = a.perm ? (a.perm[i - 1] & 0x7FFFFFFFu) : (uint32_t)(i - 1);
      for (int k = 0; k < a.n_keys; ++k) {
        const bool differs = a.ord[k][r] != a.ord[k][q] || ((a.rid[k][r] ^ a.rid[k][q]) >> 31);
        if (k < a.n_part) part |= differs;
        peer |= differs;
      }
    }
    a.part[i] = part;
    a.peer[i] = peer;
    a.rows[i] = r;
  }
}

// A function's argument in window order: the widened value bits (RAW, as load_widened returns them),
// the value as f64 bits (F64) or as an order image whose unsigned order is the value order (ORD:
// integers with the sign bit flipped, floats as f64_to_ordered, NaN greatest, -0 < +0 as in the
// aggregate path's min / max).
enum : int { GV_RAW = 0, GV_F64 = 1, GV_ORD = 2 };
__global__ void __launch_bounds__(256) window_gather_arg_kernel(const __grid_constant__ DevCol c, const uint32_t* rows, int64_t n, int mode,
                                                                uint64_t* vals, uint8_t* valid) {
  const uint64_t pol = make_policy_evict_first();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = rows[i];
    bool ok;
    uint64_t v;
    if (c.is_const) { ok = c.is_const == 1; v = c.const_bits; }
    else { ok = !c.validity || bit_test(c.validity, c.vbit_off + r); v = ok ? load_widened(c, r, pol) : 0; }
    if (mode != GV_RAW && ok) {
      const int cls = dtype_class(c.dtype);
      if (cls == VC_FLT) {
        const double d = c.dtype == DBX_F32 ? (double)__uint_as_float((uint32_t)v) : __longlong_as_double((long long)v);
        v = mode == GV_F64 ? (uint64_t)__double_as_longlong(d) : f64_to_ordered(d);
      } else if (mode == GV_F64) {
        v = (uint64_t)__double_as_longlong(cls == VC_INT ? (double)(int64_t)v : (double)v);
      } else if (cls == VC_INT) {
        v ^= 0x8000000000000000ULL;
      }
    }
    vals[i] = ok ? v : 0;
    valid[i] = ok;
  }
}

struct EmitArgs {
  int32_t kind, agg, arg_cls, arg_dtype;   // arg_cls: dtype_class of the argument
  int32_t units, start, end;               // frame (dbx_frame_units / dbx_frame_bound)
  int32_t empty;                           // the start bound lies after the end bound: every frame is empty
  int64_t so, eo;                          // frame offsets
  int64_t n, fn_n;                         // rows; NTILE buckets / LAG, LEAD offset / NTH_VALUE index
  const uint32_t *ps, *pe, *gs, *ge, *dr;  // partition start / end, peer start / end, peer starts so far
  const uint64_t* val;                     // argument in window order (GV_* as the function needs)
  const uint8_t* valid;
  const uint64_t* dval;                    // LAG / LEAD default in window order (nullptr: NULL)
  const uint8_t* dvalid;
  const uint64_t* pre;                     // integer sum: inclusive prefix sum (wrapping) over all rows
  const uint64_t* cnt;                     // inclusive prefix count of non-NULL arguments
  const uint64_t* seg;                     // segmented running (start UNBOUNDED) or suffix (end UNBOUNDED) sum / min / max
  void* out;
  uint8_t* out_valid;                      // one byte per row, nullptr: not nullable
  int32_t out_dtype;
};

__device__ __forceinline__ void frame_of(const EmitArgs& a, int64_t i, int64_t ps, int64_t pe, int64_t& s, int64_t& e) {
  switch (a.start) {
    case DBX_BOUND_UNBOUNDED_PRECEDING: s = ps; break;
    case DBX_BOUND_CURRENT_ROW: s = a.units == DBX_FRAME_RANGE ? (int64_t)a.gs[i] : i; break;
    case DBX_BOUND_PRECEDING: s = i - a.so > ps ? i - a.so : ps; break;
    default: s = i + a.so < pe ? i + a.so : pe; break;  // FOLLOWING
  }
  switch (a.end) {
    case DBX_BOUND_UNBOUNDED_FOLLOWING: e = pe; break;
    case DBX_BOUND_CURRENT_ROW: e = a.units == DBX_FRAME_RANGE ? (int64_t)a.ge[i] : i + 1; break;
    case DBX_BOUND_PRECEDING: e = i - a.eo + 1 > ps ? i - a.eo + 1 : ps; break;
    default: e = i + a.eo + 1 < pe ? i + a.eo + 1 : pe; break;  // FOLLOWING
  }
  if (e < s) e = s;
}

__device__ __forceinline__ uint64_t ntile_bucket(uint64_t n, uint64_t row_in_part, uint64_t rows) {  // compute_nitle
  if (n > rows) return row_in_part;
  const uint64_t per = rows / n, extra = rows % n, boundary = (per + 1) * extra, r = row_in_part - 1;
  return r < boundary ? r / (per + 1) + 1 : (r - extra) / per + 1;
}

__global__ void __launch_bounds__(256) window_emit_kernel(const __grid_constant__ EmitArgs a) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ps = a.ps[i], pe = a.pe[i], psize = pe - ps;
    uint64_t v = 0;
    bool ok = true;
    switch (a.kind) {
      case DBX_WIN_ROW_NUMBER: v = (uint64_t)(i - ps + 1); break;
      case DBX_WIN_RANK: v = (uint64_t)(a.gs[i] - ps + 1); break;
      case DBX_WIN_DENSE_RANK: v = (uint64_t)(a.dr[i] - a.dr[ps] + 1); break;
      case DBX_WIN_PERCENT_RANK: {
        const double p = psize <= 1 ? 0.0 : (double)(a.gs[i] - ps) / (double)(psize - 1);
        v = (uint64_t)__double_as_longlong(p);
        break;
      }
      case DBX_WIN_CUME_DIST: v = (uint64_t)__double_as_longlong((double)(a.ge[i] - ps) / (double)psize); break;
      case DBX_WIN_NTILE: v = ntile_bucket((uint64_t)a.fn_n, (uint64_t)(i - ps + 1), (uint64_t)psize); break;
      case DBX_WIN_LAG: case DBX_WIN_LEAD: {
        const int64_t t = a.kind == DBX_WIN_LAG ? i - a.fn_n : i + a.fn_n;
        if (t >= ps && t < pe) { v = a.val[t]; ok = a.valid[t]; }
        else if (a.dval) { v = a.dval[i]; ok = a.dvalid[i]; }
        else ok = false;
        break;
      }
      case DBX_WIN_NTH_VALUE: {
        int64_t s, e;
        frame_of(a, i, ps, pe, s, e);
        const int64_t t = a.fn_n == 0 ? e - 1 : s + a.fn_n - 1;
        if (a.empty || s >= e || t >= e) ok = false;
        else { v = a.val[t]; ok = a.valid[t]; }
        break;
      }
      default: {  // DBX_WIN_AGGREGATE
        int64_t s = 0, e = 0;
        if (!a.empty) frame_of(a, i, ps, pe, s, e);
        uint64_t c = e - s;  // count(*)
        if (a.cnt && e > s) c = a.cnt[e - 1] - (s > 0 ? a.cnt[s - 1] : 0);
        else if (a.cnt) c = 0;
        if (a.agg == DBX_AGG_COUNT) { v = c; break; }
        ok = c > 0;
        if (!ok) break;
        uint64_t acc;
        if (a.agg == DBX_AGG_SUM || a.agg == DBX_AGG_AVG) {
          if (a.arg_cls != VC_FLT) {
            acc = a.pre[e - 1] - (s > 0 ? a.pre[s - 1] : 0);
          } else if (a.seg) {
            // + 0.0: the reference's state starts at +0.0, so a frame of -0.0 values sums to +0.0
            acc = (uint64_t)__double_as_longlong(__longlong_as_double((long long)(a.start == DBX_BOUND_UNBOUNDED_PRECEDING ? a.seg[e - 1] : a.seg[s])) + 0.0);
          } else {  // both bounds finite: the frame's rows in row order, as the reference adds them
            double d = 0.0;
            for (int64_t t = s; t < e; ++t)
              if (a.valid[t]) d += __longlong_as_double((long long)a.val[t]);
            acc = (uint64_t)__double_as_longlong(d);
          }
          if (a.agg == DBX_AGG_AVG) {
            const double num = a.arg_cls == VC_FLT ? __longlong_as_double((long long)acc) : (a.arg_cls == VC_INT ? (double)(int64_t)acc : (double)acc);
            acc = (uint64_t)__double_as_longlong(num / (double)c);
          }
          v = acc;
          break;
        }
        // min / max over order images
        const bool is_min = a.agg == DBX_AGG_MIN;
        if (a.seg) {
          acc = a.start == DBX_BOUND_UNBOUNDED_PRECEDING ? a.seg[e - 1] : a.seg[s];
        } else {
          acc = is_min ? ~0ULL : 0;
          for (int64_t t = s; t < e; ++t) {
            if (!a.valid[t]) continue;
            const uint64_t x = a.val[t];
            acc = is_min ? (x < acc ? x : acc) : (x > acc ? x : acc);
          }
        }
        if (a.arg_cls == VC_FLT) {
          const double d = ordered_to_f64(acc);
          v = a.arg_dtype != DBX_F32 ? (uint64_t)__double_as_longlong(d) : d != d ? 0x7FC00000u : (uint64_t)__float_as_uint((float)d);
        } else {
          v = a.arg_cls == VC_INT ? acc ^ 0x8000000000000000ULL : acc;
        }
        break;
      }
    }
    store_narrow_key(a.out, i, a.out_dtype, ok ? v : 0);
    if (a.out_valid) a.out_valid[i] = ok;
  }
}

}  // namespace

// ================================================================ operator
class WindowOp : public Op {
 public:
  dbx_window_params prm;
  std::vector<int32_t> types;  // input schema (with DBX_NULLABLE)
  std::vector<dbx_block> parts;  // library-owned device copies of the pushed blocks
  int64_t rows_seen = 0;
  RadixSorter sorter;
  DevBuf k_ord[DBX_MAX_SORT_KEYS], k_rid[DBX_MAX_SORT_KEYS], k_cnt, w_ord[2], w_rid[2];
  DevBuf part8, peer8, rows32, idx[5], tile_v, tile_h, g_val, g_valid, d_val, d_valid, pre, cnt, seg;
  PinnedBuf host;
  std::unique_ptr<OwnedBlock> result;
  bool pulled = false;

  ~WindowOp() override { release_parts(); }

  void release_parts() {
    for (dbx_block& b : parts) dbx_block_release(&b);
    parts.clear();
  }

  int32_t invalid(const char* m) { err.set(m); return DBX_ERR_INVALID; }
  int32_t unsupported(const char* m) { err.set(m); return DBX_ERR_UNSUPPORTED; }

  bool col_ok(int c) const { return c >= 0 && c < (int)types.size(); }
  int dt(int c) const { return types[(size_t)c] & 0xFF; }
  bool nullable(int c) const { return (types[(size_t)c] & DBX_NULLABLE) != 0; }

  int32_t init(const dbx_window_params* p, const int32_t* t, int32_t n, int dev) {
    DBX_TRY(base_init(dev));
    prm = *p;
    if (n < 0 || n > 64 || (n > 0 && !t)) return invalid("window: 0 .. 64 input columns");
    types.assign(t, t + n);
    const int np = p->n_partition_cols, no = p->n_order_cols;
    if (np < 0 || no < 0 || np + no > DBX_MAX_SORT_KEYS) return invalid("window: at most 4 partition and order keys together");
    for (int k = 0; k < np + no; ++k) {
      const int c = k < np ? p->partition_cols[k] : p->order_cols[k - np];
      if (!col_ok(c)) return invalid("window: key column outside the input schema");
      if (dtype_size(dt(c)) == 0) return invalid("window: keys must be numeric columns");
    }
    if (p->n_funcs < 1 || p->n_funcs > DBX_MAX_WINDOW_FUNCS) return invalid("window: 1 .. 8 functions");
    for (int f = 0; f < p->n_funcs; ++f) {
      dbx_window_func& w = prm.funcs[f];
      if ((w.kind == DBX_WIN_LAG || w.kind == DBX_WIN_LEAD) && w.n < 0 && w.n != INT64_MIN) {  // lag(x, -n) is lead(x, n)
        w.kind = w.kind == DBX_WIN_LAG ? DBX_WIN_LEAD : DBX_WIN_LAG;
        w.n = -w.n;
      }
      const dbx_window_frame& fr = w.frame;
      const bool has_frame = fr.units || fr.start || fr.end || fr.start_offset || fr.end_offset;
      if (w.ignore_nulls) return unsupported("window: IGNORE NULLS is not supported");
      if (w.distinct) return unsupported("window: DISTINCT window aggregates are not supported");
      switch (w.kind) {
        case DBX_WIN_ROW_NUMBER: case DBX_WIN_RANK: case DBX_WIN_DENSE_RANK: case DBX_WIN_PERCENT_RANK: case DBX_WIN_CUME_DIST:
          break;
        case DBX_WIN_NTILE:
          if (w.n < 1) return invalid("window: ntile needs a positive number of buckets");
          break;
        case DBX_WIN_LAG: case DBX_WIN_LEAD:
          if (w.n < 0) return invalid("window: lag / lead offset out of range");
          if (!col_ok(w.arg_col)) return invalid("window: argument column outside the input schema");
          if (w.default_col != -1 && !col_ok(w.default_col)) return invalid("window: default column outside the input schema");
          if (w.default_col != -1 && dt(w.default_col) != dt(w.arg_col)) return invalid("window: the default column must have the argument's type");
          break;
        case DBX_WIN_NTH_VALUE:
          if (w.n < 0) return invalid("window: negative nth_value index");
          if (!col_ok(w.arg_col)) return invalid("window: argument column outside the input schema");
          break;
        case DBX_WIN_AGGREGATE:
          if (w.agg_kind < DBX_AGG_SUM || w.agg_kind > DBX_AGG_MAX) return invalid("window: unknown aggregate");
          if (w.arg_col == -1 ? w.agg_kind != DBX_AGG_COUNT : !col_ok(w.arg_col)) return invalid("window: argument column outside the input schema");
          if (w.arg_col >= 0 && dtype_size(dt(w.arg_col)) == 0) return invalid("window: aggregate arguments must be numeric (not Boolean or Vector)");
          break;
        default: return invalid("window: unknown function kind");
      }
      if ((w.kind == DBX_WIN_LAG || w.kind == DBX_WIN_LEAD || w.kind == DBX_WIN_NTH_VALUE) && dtype_size(dt(w.arg_col)) == 0)
        return unsupported("window: lag / lead / nth_value of Boolean or Vector columns are not supported");
      const bool takes_frame = w.kind == DBX_WIN_AGGREGATE || w.kind == DBX_WIN_NTH_VALUE;
      if (!takes_frame) {
        if (has_frame) return invalid("window: this function takes no frame (the binder gives it one)");
        continue;
      }
      if (fr.units != DBX_FRAME_ROWS && fr.units != DBX_FRAME_RANGE) return invalid("window: frame units must be ROWS or RANGE");
      if (fr.start < DBX_BOUND_UNBOUNDED_PRECEDING || fr.start > DBX_BOUND_FOLLOWING) return invalid("window: bad frame start");
      if (fr.end < DBX_BOUND_PRECEDING || fr.end > DBX_BOUND_UNBOUNDED_FOLLOWING) return invalid("window: bad frame end");
      if (fr.start_offset < 0 || fr.end_offset < 0) return invalid("window: negative frame offset");
      const bool s_off = fr.start == DBX_BOUND_PRECEDING || fr.start == DBX_BOUND_FOLLOWING;
      const bool e_off = fr.end == DBX_BOUND_PRECEDING || fr.end == DBX_BOUND_FOLLOWING;
      if ((!s_off && fr.start_offset) || (!e_off && fr.end_offset)) return invalid("window: an offset on a bound that takes none");
      if (fr.units == DBX_FRAME_RANGE && (s_off || e_off)) return unsupported("window: RANGE frames with an offset are not supported");
    }
    DBX_CUDA_TRY(err, host.ensure(64));
    DBX_CUDA_TRY(err, k_cnt.ensure(8 * DBX_MAX_SORT_KEYS));
    return DBX_OK;
  }

  int32_t reset() override {
    release_parts();
    rows_seen = 0;
    result.reset();
    pulled = false;
    return DBX_OK;
  }

  int32_t push(const dbx_block* b) override {
    if (b->num_cols != (int)types.size()) return invalid("push: block column count differs from the operator's input schema");
    for (int c = 0; c < b->num_cols; ++c) {
      const dbx_column& col = b->cols[c];
      if (col.dtype != dt(c) || col.len != b->num_rows) return invalid("push: column does not match the input schema");
      if (!col.is_const && col.validity && !nullable(c)) return invalid("push: validity bitmap on a column declared non-nullable");
    }
    const int64_t n = b->num_rows;
    if (n == 0) return DBX_OK;
    if (rows_seen + n > rs::kMaxRows) return unsupported("window: more than 2^30 - 1 rows are not supported");
    dbx_block copy;
    memset(&copy, 0, sizeof(copy));
    const int32_t st = dbx_block_concat(device, b, 1, DBX_MEM_DEVICE, &copy);  // read completely before it returns
    if (st != DBX_OK) { err.set(dbx_last_error(nullptr)); return st; }
    parts.push_back(copy);
    rows_seen += n;
    return DBX_OK;
  }

  template <class Op, bool REV>
  int32_t scan(const ScanSrc& s, typename Op::T* out) {
    const int64_t tiles = (s.n + kScanTile - 1) / kScanTile;
    DBX_CUDA_TRY(err, tile_v.ensure((size_t)tiles * 8));
    DBX_CUDA_TRY(err, tile_h.ensure((size_t)tiles));
    scan_reduce_kernel<Op, REV><<<(unsigned)tiles, kScanThreads, 0, stream>>>(s, (typename Op::T*)tile_v.p, (uint8_t*)tile_h.p);
    scan_spine_kernel<Op><<<1, kSpineThreads, 0, stream>>>((typename Op::T*)tile_v.p, (const uint8_t*)tile_h.p, tiles);
    scan_tile_kernel<Op, REV><<<(unsigned)tiles, kScanThreads, 0, stream>>>(s, (const typename Op::T*)tile_v.p, out);
    count_launch(3);
    DBX_CUDA_TRY(err, cudaGetLastError());
    return DBX_OK;
  }

  // the device view of column c of the concatenated input (Const entries carry their value)
  DevCol dev_col(const dbx_column& col) const {
    DevCol d;
    memset(&d, 0, sizeof(d));
    d.dtype = col.dtype;
    if (col.is_const) {
      d.is_const = col.konst.is_null ? 2 : 1;
      if (col.dtype == DBX_F32) { const float f = (float)col.konst.v.f64; uint32_t u; memcpy(&u, &f, 4); d.const_bits = u; }
      else d.const_bits = col.konst.v.u64;
      return d;
    }
    d.data = col.data; d.validity = col.validity; d.vbit_off = col.validity_bit_offset; d.dbit_off = col.data_bit_offset;
    return d;
  }

  int32_t alloc_out(OwnedBlock* ob, size_t bytes, void** p) {
    DBX_CUDA_TRY(err, pool_alloc(device, stream, bytes ? bytes : 1, p));
    ob->dev_allocs.push_back(*p);
    return DBX_OK;
  }

  int32_t empty_result() {
    auto ob = std::make_unique<OwnedBlock>();
    ob->device = device;
    ob->stream = stream;
    for (int c = 0; c < (int)types.size() + prm.n_funcs; ++c) {
      dbx_column oc;
      memset(&oc, 0, sizeof(oc));
      oc.mem = DBX_MEM_DEVICE;
      if (c < (int)types.size()) oc.dtype = dt(c);
      else oc.dtype = result_dtype(prm.funcs[c - types.size()]);
      void* d = nullptr;
      DBX_TRY(alloc_out(ob.get(), 8, &d));
      oc.data = d;
      if ((c < (int)types.size() && nullable(c)) || (c >= (int)types.size() && result_nullable(prm.funcs[c - types.size()]))) oc.validity = (const uint8_t*)d;
      ob->cols.push_back(oc);
    }
    result = std::move(ob);
    return DBX_OK;
  }

  int result_dtype(const dbx_window_func& w) const {
    switch (w.kind) {
      case DBX_WIN_PERCENT_RANK: case DBX_WIN_CUME_DIST: return DBX_F64;
      case DBX_WIN_LAG: case DBX_WIN_LEAD: case DBX_WIN_NTH_VALUE: return dt(w.arg_col);
      case DBX_WIN_AGGREGATE: {
        if (w.agg_kind == DBX_AGG_COUNT) return DBX_U64;
        if (w.agg_kind == DBX_AGG_AVG) return DBX_F64;
        const int cls = dtype_class(dt(w.arg_col));
        if (w.agg_kind == DBX_AGG_SUM) return cls == VC_FLT ? DBX_F64 : (cls == VC_INT ? DBX_I64 : DBX_U64);
        return dt(w.arg_col);
      }
      default: return DBX_U64;
    }
  }
  bool result_nullable(const dbx_window_func& w) const {
    switch (w.kind) {
      case DBX_WIN_LAG: case DBX_WIN_LEAD: return w.default_col < 0 || nullable(w.default_col) || nullable(w.arg_col);
      case DBX_WIN_NTH_VALUE: return true;
      case DBX_WIN_AGGREGATE: return w.agg_kind != DBX_AGG_COUNT;
      default: return false;
    }
  }

  // FrameBound order (frame_bound.rs:50-80): UNBOUNDED PRECEDING < n PRECEDING (larger n first) <
  // CURRENT ROW < n FOLLOWING (smaller n first) < UNBOUNDED FOLLOWING
  static bool bound_after(int sb, int64_t so, int eb, int64_t eo) {
    auto key = [](int b, int64_t o) { return b == DBX_BOUND_PRECEDING ? -o : (b == DBX_BOUND_FOLLOWING ? o : 0); };
    return sb != eb ? sb > eb : key(sb, so) > key(eb, eo);
  }

  int32_t emit_function(const dbx_window_func& w, const dbx_block& in, int64_t n, const uint32_t* rows, OwnedBlock* ob) {
    const int out_dt = result_dtype(w);
    const bool out_null = result_nullable(w);
    void *out = nullptr, *ovb = nullptr, *obits = nullptr;
    DBX_TRY(alloc_out(ob, (size_t)n * dtype_size(out_dt), &out));
    if (out_null) {
      DBX_TRY(alloc_out(ob, (size_t)n, &ovb));
      DBX_TRY(alloc_out(ob, (size_t)(n + 7) / 8 + 8, &obits));
    }
    EmitArgs a;
    memset(&a, 0, sizeof(a));
    a.kind = w.kind; a.agg = w.agg_kind; a.n = n; a.fn_n = w.n;
    a.units = w.frame.units; a.start = w.frame.start; a.end = w.frame.end;
    a.so = std::min<int64_t>(w.frame.start_offset, 1LL << 40); a.eo = std::min<int64_t>(w.frame.end_offset, 1LL << 40);  // beyond any partition
    a.fn_n = std::min<int64_t>(w.n, 1LL << 40);
    a.ps = (const uint32_t*)idx[0].p; a.pe = (const uint32_t*)idx[1].p; a.gs = (const uint32_t*)idx[2].p;
    a.ge = (const uint32_t*)idx[3].p; a.dr = (const uint32_t*)idx[4].p;
    a.out = out; a.out_valid = (uint8_t*)ovb; a.out_dtype = out_dt;
    const bool framed = w.kind == DBX_WIN_AGGREGATE || w.kind == DBX_WIN_NTH_VALUE;
    if (framed) a.empty = bound_after(w.frame.start, w.frame.start_offset, w.frame.end, w.frame.end_offset);
    if (w.arg_col >= 0 && w.kind >= DBX_WIN_LAG) {
      const int adt = dt(w.arg_col);
      a.arg_dtype = adt; a.arg_cls = dtype_class(adt);
      const bool is_agg = w.kind == DBX_WIN_AGGREGATE;
      const bool flt = a.arg_cls == VC_FLT;
      const int mode = !is_agg ? GV_RAW : (w.agg_kind == DBX_AGG_MIN || w.agg_kind == DBX_AGG_MAX) ? GV_ORD : (flt ? GV_F64 : GV_RAW);
      DBX_CUDA_TRY(err, g_val.ensure((size_t)n * 8));
      DBX_CUDA_TRY(err, g_valid.ensure((size_t)n));
      window_gather_arg_kernel<<<grid_1d(n), 256, 0, stream>>>(dev_col(in.cols[w.arg_col]), rows, n, mode, (uint64_t*)g_val.p, (uint8_t*)g_valid.p);
      count_launch();
      a.val = (const uint64_t*)g_val.p; a.valid = (const uint8_t*)g_valid.p;
      if ((w.kind == DBX_WIN_LAG || w.kind == DBX_WIN_LEAD) && w.default_col >= 0) {
        DBX_CUDA_TRY(err, d_val.ensure((size_t)n * 8));
        DBX_CUDA_TRY(err, d_valid.ensure((size_t)n));
        window_gather_arg_kernel<<<grid_1d(n), 256, 0, stream>>>(dev_col(in.cols[w.default_col]), rows, n, GV_RAW, (uint64_t*)d_val.p, (uint8_t*)d_valid.p);
        count_launch();
        a.dval = (const uint64_t*)d_val.p; a.dvalid = (const uint8_t*)d_valid.p;
      }
      if (is_agg) {
        ScanSrc s;
        memset(&s, 0, sizeof(s));
        s.n = n; s.vals = a.val; s.valid = a.valid; s.flags = (const uint8_t*)part8.p;
        DBX_CUDA_TRY(err, cnt.ensure((size_t)n * 8));
        s.mode = SRC_VALID;
        DBX_TRY((scan<OpSumU64, false>(s, (uint64_t*)cnt.p)));
        a.cnt = (const uint64_t*)cnt.p;
        s.mode = SRC_VALUES;
        const bool sum_like = w.agg_kind == DBX_AGG_SUM || w.agg_kind == DBX_AGG_AVG;
        if (sum_like && !flt) {
          DBX_CUDA_TRY(err, pre.ensure((size_t)n * 8));
          DBX_TRY((scan<OpSumU64, false>(s, (uint64_t*)pre.p)));
          a.pre = (const uint64_t*)pre.p;
        } else if (w.agg_kind != DBX_AGG_COUNT && !a.empty) {
          const bool fwd = w.frame.start == DBX_BOUND_UNBOUNDED_PRECEDING, rev = !fwd && w.frame.end == DBX_BOUND_UNBOUNDED_FOLLOWING;
          if (fwd || rev) {
            DBX_CUDA_TRY(err, seg.ensure((size_t)n * 8));
            s.segmented = 1;
            uint64_t* o = (uint64_t*)seg.p;
            if (sum_like) DBX_TRY(fwd ? (scan<OpSumF64, false>(s, o)) : (scan<OpSumF64, true>(s, o)));
            else if (w.agg_kind == DBX_AGG_MIN) DBX_TRY(fwd ? (scan<OpMinU64, false>(s, o)) : (scan<OpMinU64, true>(s, o)));
            else DBX_TRY(fwd ? (scan<OpMaxU64, false>(s, o)) : (scan<OpMaxU64, true>(s, o)));
            a.seg = o;
          }
        }
      }
    }
    window_emit_kernel<<<grid_1d(n), 256, 0, stream>>>(a);
    count_launch();
    if (out_null) { pack_bits_kernel<<<grid_1d((n + 7) / 8), 256, 0, stream>>>((const uint8_t*)ovb, n, (uint8_t*)obits); count_launch(); }
    DBX_CUDA_TRY(err, cudaGetLastError());
    dbx_column oc;
    memset(&oc, 0, sizeof(oc));
    oc.dtype = out_dt; oc.mem = DBX_MEM_DEVICE; oc.len = n; oc.data = out;
    if (out_null) { oc.validity = (const uint8_t*)obits; oc.null_count = -1; }
    ob->cols.push_back(oc);
    return DBX_OK;
  }

  int32_t finish() override {
    if (parts.empty()) return empty_result();
    // 1. one device block of every pushed row, then the sort
    dbx_block in;
    memset(&in, 0, sizeof(in));
    if (parts.size() == 1) {
      in = parts[0];
      parts.clear();
    } else {
      const int32_t st = dbx_block_concat(device, parts.data(), (int32_t)parts.size(), DBX_MEM_DEVICE, &in);
      if (st != DBX_OK) { err.set(dbx_last_error(nullptr)); return st; }
      release_parts();
    }
    struct Guard { dbx_block* b; ~Guard() { dbx_block_release(b); } } guard{&in};
    const int64_t n = in.num_rows;
    // four timed phases in the handle's event ring (dbx_op_kernel_ms, back = 3 .. 0): key images and
    // sort, boundaries and scans, emit, gather
    DBX_TRY(timing_begin());
    const int np = prm.n_partition_cols, no = prm.n_order_cols;
    // Const keys are equal on every row: they neither order nor split anything
    BoundArgs ba;
    memset(&ba, 0, sizeof(ba));
    int nk = 0, nkp = 0;
    const uint64_t* ord[DBX_MAX_SORT_KEYS] = {};
    const uint32_t* rid[DBX_MAX_SORT_KEYS] = {};
    int32_t nulls_first[DBX_MAX_SORT_KEYS] = {};
    DBX_CUDA_TRY(err, cudaMemsetAsync(k_cnt.p, 0, 8 * DBX_MAX_SORT_KEYS, stream));
    for (int k = 0; k < np + no; ++k) {
      const int c = k < np ? prm.partition_cols[k] : prm.order_cols[k - np];
      const dbx_column& col = in.cols[c];
      if (col.is_const) continue;
      const int asc = k < np ? 1 : prm.order_asc[k - np];
      nulls_first[nk] = k < np ? 0 : prm.order_nulls_first[k - np];
      DBX_CUDA_TRY(err, k_ord[nk].ensure((size_t)n * 8));
      DBX_CUDA_TRY(err, k_rid[nk].ensure((size_t)n * 4));
      sort_ingest_kernel<<<grid_1d(n), 256, 0, stream>>>(dev_col(col), n, 0, key_class(col.dtype), asc, (uint64_t*)k_ord[nk].p, (uint32_t*)k_rid[nk].p,
                                                         nullptr, (unsigned long long*)k_cnt.p + nk, nullptr);
      count_launch();
      ord[nk] = (const uint64_t*)k_ord[nk].p; rid[nk] = (const uint32_t*)k_rid[nk].p;
      if (k < np) ++nkp;
      ++nk;
    }
    DBX_CUDA_TRY(err, cudaGetLastError());
    const uint32_t* perm = nullptr;
    if (nk > 0 && n > 1) {
      DBX_CUDA_TRY(err, cudaMemcpyAsync(host.p, k_cnt.p, 8 * DBX_MAX_SORT_KEYS, cudaMemcpyDeviceToHost, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      int64_t n_nulls[DBX_MAX_SORT_KEYS];
      for (int k = 0; k < DBX_MAX_SORT_KEYS; ++k) n_nulls[k] = (int64_t)((const unsigned long long*)host.p)[k];
      const uint64_t* sorted_ord = nullptr;
      DBX_TRY(sort_rows_by_keys(err, stream, sorter, nk, ord, rid, n_nulls, nulls_first, n, w_ord, w_rid, &sorted_ord, &perm));
    }
    DBX_TRY(timing_end());
    DBX_TRY(timing_begin());
    // 2. boundaries  3. row indices
    DBX_CUDA_TRY(err, part8.ensure((size_t)n));
    DBX_CUDA_TRY(err, peer8.ensure((size_t)n));
    DBX_CUDA_TRY(err, rows32.ensure((size_t)n * 4));
    for (int k = 0; k < nk; ++k) { ba.ord[k] = ord[k]; ba.rid[k] = rid[k]; }
    ba.n_keys = nk; ba.n_part = nkp; ba.perm = perm; ba.n = n;
    ba.part = (uint8_t*)part8.p; ba.peer = (uint8_t*)peer8.p; ba.rows = (uint32_t*)rows32.p;
    window_bounds_kernel<<<grid_1d(n), 256, 0, stream>>>(ba);
    count_launch();
    for (auto& b : idx) DBX_CUDA_TRY(err, b.ensure((size_t)n * 4));
    ScanSrc s;
    memset(&s, 0, sizeof(s));
    s.n = n;
    s.mode = SRC_START_IDX; s.flags = (const uint8_t*)part8.p;
    DBX_TRY((scan<OpMaxU32, false>(s, (uint32_t*)idx[0].p)));
    s.mode = SRC_END_IDX;
    DBX_TRY((scan<OpMinU32, true>(s, (uint32_t*)idx[1].p)));
    s.mode = SRC_START_IDX; s.flags = (const uint8_t*)peer8.p;
    DBX_TRY((scan<OpMaxU32, false>(s, (uint32_t*)idx[2].p)));
    s.mode = SRC_END_IDX;
    DBX_TRY((scan<OpMinU32, true>(s, (uint32_t*)idx[3].p)));
    s.mode = SRC_FLAGS;
    DBX_TRY((scan<OpSumU32, false>(s, (uint32_t*)idx[4].p)));
    DBX_TRY(timing_end());
    DBX_TRY(timing_begin());
    // 4. one column per function
    auto fob = std::make_unique<OwnedBlock>();
    fob->device = device;
    fob->stream = stream;
    for (int f = 0; f < prm.n_funcs; ++f) DBX_TRY(emit_function(prm.funcs[f], in, n, (const uint32_t*)rows32.p, fob.get()));
    DBX_TRY(timing_end());
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    const unsigned int* fail = sorter.meta.p ? sorter.fail() : nullptr;
    if (fail && nk > 0 && n > 1) {
      DBX_CUDA_TRY(err, cudaMemcpy(host.p, fail, 4, cudaMemcpyDeviceToHost));
      if (*(const unsigned int*)host.p) { err.set("internal: radix sort look-back timed out"); return DBX_ERR_CUDA; }
    }
    // 5. the input columns in window order
    dbx_block taken;
    memset(&taken, 0, sizeof(taken));
    DBX_TRY(timing_begin());  // the gather is synchronous on its own stream: this pair brackets the call
    const int32_t st = dbx_block_take(device, &in, (const uint32_t*)rows32.p, n, DBX_MEM_DEVICE, DBX_MEM_DEVICE, &taken);
    if (st != DBX_OK) { err.set(dbx_last_error(nullptr)); return st; }
    DBX_TRY(timing_end());
    std::unique_ptr<OwnedBlock> ob((OwnedBlock*)taken.owner);
    ob->stream = stream;
    for (const dbx_column& c : fob->cols) ob->cols.push_back(c);
    ob->dev_allocs.insert(ob->dev_allocs.end(), fob->dev_allocs.begin(), fob->dev_allocs.end());
    fob->dev_allocs.clear();
    result = std::move(ob);
    return DBX_OK;
  }

  int32_t pull(int32_t out_mem, dbx_block* out, int32_t* has_block) override {
    if (!finished) { err.set("pull before finish"); return DBX_ERR_STATE; }
    if (pulled || !result) { *has_block = 0; return DBX_OK; }
    pulled = true;
    *has_block = 1;
    return pull_owned_block(result, device, stream, err, out_mem, out);
  }
};

Op* make_window_op(const dbx_window_params* p, const int32_t* types, int32_t n, int device, int32_t* st) {
  auto* op = new WindowOp();
  *st = op->init(p, types, n, device);
  if (*st != DBX_OK) { g_create_error.set(op->err.msg); delete op; return nullptr; }
  return op;
}

}  // namespace dbx
