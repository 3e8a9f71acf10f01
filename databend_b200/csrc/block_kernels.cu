// block_kernels.cu — DataBlock::take / take_ranges / scatter / concat on the device.
//
// Reference kernels replaced (paths relative to the databend source tree, src/query/expression/src/kernels):
//   DataBlock::take(indices)              take.rs:43-60        (gather by u32 row indices)
//   DataBlock::take_ranges(ranges, n)     take_ranges.rs:40    (concatenation of row ranges)
//   DataBlock::scatter(indices, n)        scatter.rs:21        (row i goes to block indices[i], order kept)
//   DataBlock::concat(blocks)             concat.rs:62
// Every column kind libdbx carries is handled: numeric Buffer<T>, Boolean (bit-packed), Vector(Float32)
// and Vector(Int8) (flat row-major), Nullable (validity Bitmap with a bit offset), BlockEntry::Const (stays const).
// HBM-bound byte moving: one thread per output row and column element, coalesced on the output side.
#include <algorithm>
#include <vector>

#include "radix_sort.cuh"
#include "runtime.h"

namespace dbx {
namespace {

struct GatherCol {
  const void* src;
  const uint8_t* src_valid;   // bitmap or nullptr
  int64_t src_vbit_off, src_dbit_off;
  void* dst;                  // values (BOOL: one byte per row, packed afterwards)
  uint8_t* dst_valid;         // one byte per row or nullptr
  int32_t elt;                // bytes per row (vectors: 4 * dim or dim); 0 = BOOL
  int32_t pad;
};
struct GatherParams {
  GatherCol cols[64];
  int32_t n_cols;
  int32_t pad;
  int64_t n_out;
  const uint32_t* idx;   // out row i <- src row idx[i]; nullptr: src row = src_row0 + i
  int64_t src_row0;
  int64_t dst_row0;      // first output row (concat writes blocks one after another)
};

__global__ void __launch_bounds__(256) gather_rows_kernel(const __grid_constant__ GatherParams p) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n_out; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = p.idx ? (int64_t)p.idx[i] : p.src_row0 + i;
    const int64_t o = p.dst_row0 + i;
    for (int c = 0; c < p.n_cols; ++c) {
      const GatherCol& gc = p.cols[c];
      if (gc.elt == 0) ((uint8_t*)gc.dst)[o] = (uint8_t)bit_test((const uint8_t*)gc.src, gc.src_dbit_off + r);
      else if (gc.elt == 8) ((uint64_t*)gc.dst)[o] = ((const uint64_t*)gc.src)[r];
      else if (gc.elt == 4) ((uint32_t*)gc.dst)[o] = ((const uint32_t*)gc.src)[r];
      else if (gc.elt == 2) ((uint16_t*)gc.dst)[o] = ((const uint16_t*)gc.src)[r];
      else if (gc.elt == 1) ((uint8_t*)gc.dst)[o] = ((const uint8_t*)gc.src)[r];
      else if ((gc.elt & 3) == 0) {  // Vector(Float32), or Vector(Int8) whose dim is a multiple of 4
        const uint32_t* s = (const uint32_t*)((const char*)gc.src + r * gc.elt);
        uint32_t* d = (uint32_t*)((char*)gc.dst + o * gc.elt);
        for (int k = 0; k < gc.elt / 4; ++k) d[k] = s[k];
      } else {  // Vector(Int8) of any other dim
        const uint8_t* s = (const uint8_t*)gc.src + r * gc.elt;
        uint8_t* d = (uint8_t*)gc.dst + o * gc.elt;
        for (int k = 0; k < gc.elt; ++k) d[k] = s[k];
      }
      if (gc.dst_valid) gc.dst_valid[o] = gc.src_valid ? (uint8_t)bit_test(gc.src_valid, gc.src_vbit_off + r) : 1;
    }
  }
}
__global__ void bytes_to_bits_kernel(const uint8_t* bytes, int64_t n, uint8_t* bits) {
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
__global__ void expand_ranges_kernel(const uint32_t* starts, const int64_t* out_off, int64_t n_ranges, int64_t n_out, uint32_t* idx) {
  // one warp per range
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n_ranges; r += n_warps) {
    const int64_t o0 = out_off[r], len = out_off[r + 1] - o0;
    for (int64_t j = lane; j < len; j += 32) idx[o0 + j] = starts[r] + (uint32_t)j;
  }
}
__global__ void widen_u32_iota_kernel(const uint32_t* part, int64_t n, uint64_t* keys, uint32_t* rows) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = part[i];
    rows[i] = (uint32_t)i;
  }
}
__global__ void count_parts_kernel(const uint32_t* part, int64_t n, int n_parts, unsigned long long* counts, unsigned int* bad) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t q = part[i];
    if (q >= (uint32_t)n_parts) { atomicExch(bad, 1u); continue; }
    atomicAdd(&counts[q], 1ULL);
  }
}

inline int grid_n(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)kNumSMs * 8)); }

// A block whose columns are all addressable on the device (host columns are copied in).
struct DeviceView {
  std::vector<DevCol> cols;      // data / validity pointers on the device
  std::vector<DevBuf> owned;
  int32_t load(ErrorSink& err, cudaStream_t st, const dbx_block* b) {
    cols.resize((size_t)b->num_cols);
    for (int c = 0; c < b->num_cols; ++c) {
      const dbx_column& col = b->cols[c];
      DevCol& dc = cols[(size_t)c];
      memset(&dc, 0, sizeof(dc));
      dc.dtype = col.dtype;
      if (col.len != b->num_rows) { err.set("block kernel: column length differs from num_rows"); return DBX_ERR_INVALID; }
      if (col.is_const) { dc.is_const = 1; continue; }
      const bool is_bool = col.dtype == DBX_BOOL;
      const int64_t elt = column_row_bytes(col.dtype, col.vec_dim);
      if (!is_bool && elt == 0) { err.set("block kernel: unsupported column type"); return DBX_ERR_UNSUPPORTED; }
      if (col.mem == DBX_MEM_DEVICE) {
        dc.data = col.data; dc.validity = col.validity; dc.vbit_off = col.validity_bit_offset; dc.dbit_off = col.data_bit_offset;
        continue;
      }
      if (is_bool) {
        const int64_t b0 = col.data_bit_offset >> 3, b1 = (col.data_bit_offset + col.len + 7) >> 3;
        owned.emplace_back();
        DBX_CUDA_TRY(err, owned.back().ensure((size_t)std::max<int64_t>(b1 - b0, 1)));
        if (b1 > b0) DBX_CUDA_TRY(err, cudaMemcpyAsync(owned.back().p, (const uint8_t*)col.data + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, st));
        dc.data = owned.back().p; dc.dbit_off = col.data_bit_offset & 7;
      } else {
        owned.emplace_back();
        DBX_CUDA_TRY(err, owned.back().ensure((size_t)std::max<int64_t>(col.len * elt, 1)));
        if (col.len) DBX_CUDA_TRY(err, cudaMemcpyAsync(owned.back().p, col.data, (size_t)(col.len * elt), cudaMemcpyHostToDevice, st));
        dc.data = owned.back().p;
      }
      if (col.validity) {
        const int64_t b0 = col.validity_bit_offset >> 3, b1 = (col.validity_bit_offset + col.len + 7) >> 3;
        owned.emplace_back();
        DBX_CUDA_TRY(err, owned.back().ensure((size_t)std::max<int64_t>(b1 - b0, 1)));
        if (b1 > b0) DBX_CUDA_TRY(err, cudaMemcpyAsync(owned.back().p, col.validity + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, st));
        dc.validity = (const uint8_t*)owned.back().p; dc.vbit_off = col.validity_bit_offset & 7;
      }
    }
    return DBX_OK;
  }
};

// Output columns of `n_out` rows with the schema of `proto`; returns the gather descriptors.
struct OutputBuilder {
  std::unique_ptr<OwnedBlock> ob;
  std::vector<uint8_t*> valid_bytes, bool_bytes;  // per column, nullptr when unused
  int32_t begin(ErrorSink& err, int device, cudaStream_t st, const dbx_block* proto, const bool* nullable, int64_t n_out) {
    ob = std::make_unique<OwnedBlock>();
    ob->device = device;
    valid_bytes.assign((size_t)proto->num_cols, nullptr);
    bool_bytes.assign((size_t)proto->num_cols, nullptr);
    for (int c = 0; c < proto->num_cols; ++c) {
      const dbx_column& pc = proto->cols[c];
      dbx_column oc;
      memset(&oc, 0, sizeof(oc));
      oc.dtype = pc.dtype; oc.vec_dim = pc.vec_dim; oc.len = n_out; oc.mem = DBX_MEM_DEVICE;
      if (pc.is_const) { oc.is_const = 1; oc.konst = pc.konst; oc.mem = DBX_MEM_HOST; ob->cols.push_back(oc); continue; }
      const int64_t elt = pc.dtype == DBX_BOOL ? 1 : column_row_bytes(pc.dtype, pc.vec_dim);
      void* d = nullptr;
      DBX_CUDA_TRY(err, pool_alloc(device, st, (size_t)std::max<int64_t>(n_out * elt, 1), &d));
      ob->dev_allocs.push_back(d);
      oc.data = d;
      if (pc.dtype == DBX_BOOL) bool_bytes[(size_t)c] = (uint8_t*)d;
      if (nullable[c]) {
        void* v = nullptr;
        DBX_CUDA_TRY(err, pool_alloc(device, st, (size_t)std::max<int64_t>(n_out, 1), &v));
        ob->dev_allocs.push_back(v);
        valid_bytes[(size_t)c] = (uint8_t*)v;
        oc.null_count = -1;
      }
      ob->cols.push_back(oc);
    }
    return DBX_OK;
  }
  // descriptors for copying rows of `src` (same schema) into the output
  void fill(GatherParams* gp, const DeviceView& src, const dbx_block* proto) const {
    memset(gp, 0, sizeof(*gp));
    int k = 0;
    for (int c = 0; c < proto->num_cols; ++c) {
      if (proto->cols[c].is_const) continue;
      GatherCol& gc = gp->cols[k++];
      const DevCol& dc = src.cols[(size_t)c];
      gc.src = dc.data; gc.src_valid = dc.validity; gc.src_vbit_off = dc.vbit_off; gc.src_dbit_off = dc.dbit_off;
      gc.dst = (void*)ob->cols[(size_t)c].data;
      gc.dst_valid = valid_bytes[(size_t)c];
      gc.elt = (int32_t)column_row_bytes(proto->cols[c].dtype, proto->cols[c].vec_dim);
    }
    gp->n_cols = k;
  }
  // byte-per-row validity / boolean data -> LSB-first bitmaps, then hand the block out
  int32_t finish(ErrorSink& err, int device, cudaStream_t st, int64_t n_out, int32_t out_mem, dbx_block* out) {
    for (size_t c = 0; c < ob->cols.size(); ++c) {
      for (int which = 0; which < 2; ++which) {
        uint8_t* bytes = which ? valid_bytes[c] : bool_bytes[c];
        if (!bytes) continue;
        void* bits = nullptr;
        DBX_CUDA_TRY(err, pool_alloc(device, st, (size_t)(n_out + 7) / 8 + 8, &bits));
        ob->dev_allocs.push_back(bits);
        if (n_out) { bytes_to_bits_kernel<<<grid_n((n_out + 7) / 8), 256, 0, st>>>(bytes, n_out, (uint8_t*)bits); count_launch(); }
        if (which) { ob->cols[c].validity = (const uint8_t*)bits; ob->cols[c].validity_bit_offset = 0; }
        else { ob->cols[c].data = bits; ob->cols[c].data_bit_offset = 0; }
      }
    }
    DBX_CUDA_TRY(err, cudaGetLastError());
    int32_t st_ = pull_owned_block(ob, device, st, err, out_mem, out);
    if (st_ == DBX_OK) out->num_rows = n_out;
    return st_;
  }
};

struct CallCtx {
  cudaStream_t st = nullptr;
  ~CallCtx() { if (st) cudaStreamDestroy(st); }
  int32_t init(ErrorSink& err, int device) {
    int32_t ndev = 0;
    DBX_TRY(dbx_device_count(&ndev));
    if (device < 0 || device >= ndev) { err.set("device index out of range"); return DBX_ERR_INVALID; }
    DBX_CUDA_TRY(err, cudaSetDevice(device));
    DBX_CUDA_TRY(err, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    return DBX_OK;
  }
};

int32_t idx_to_device(ErrorSink& err, cudaStream_t st, const uint32_t* idx, int64_t n, int32_t mem, DevBuf& buf, const uint32_t** out) {
  if (mem == DBX_MEM_DEVICE) { *out = idx; return DBX_OK; }
  DBX_CUDA_TRY(err, buf.ensure((size_t)std::max<int64_t>(n, 1) * 4));
  if (n) DBX_CUDA_TRY(err, cudaMemcpyAsync(buf.p, idx, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  *out = (const uint32_t*)buf.p;
  return DBX_OK;
}

void nullable_flags(const dbx_block* b, bool* out) {
  for (int c = 0; c < b->num_cols; ++c) out[c] = b->cols[c].validity != nullptr && !b->cols[c].is_const;
}

}  // namespace
}  // namespace dbx

using namespace dbx;

extern "C" {

int32_t dbx_block_take(int32_t device, const dbx_block* block, const uint32_t* indices, int64_t n_indices, int32_t indices_mem,
                       int32_t out_mem, dbx_block* out) {
  ErrorSink& err = g_create_error;
  if (!block || !out || n_indices < 0 || (n_indices > 0 && !indices) || block->num_cols < 0 || block->num_cols > 64) { err.set("dbx_block_take: bad argument"); return DBX_ERR_INVALID; }
  CallCtx cx;
  DBX_TRY(cx.init(err, device));
  DeviceView src;
  DBX_TRY(src.load(err, cx.st, block));
  DevBuf ibuf;
  const uint32_t* didx = nullptr;
  DBX_TRY(idx_to_device(err, cx.st, indices, n_indices, indices_mem, ibuf, &didx));
  if (indices_mem == DBX_MEM_HOST)  // an index outside the block would read out of bounds: reject it up front
    for (int64_t i = 0; i < n_indices; ++i)
      if ((int64_t)indices[i] >= block->num_rows) { err.set("dbx_block_take: index out of range"); return DBX_ERR_INVALID; }
  bool nullable[64];
  nullable_flags(block, nullable);
  OutputBuilder ob;
  DBX_TRY(ob.begin(err, device, cx.st, block, nullable, n_indices));
  GatherParams gp;
  ob.fill(&gp, src, block);
  gp.n_out = n_indices; gp.idx = didx;
  if (n_indices && gp.n_cols) { gather_rows_kernel<<<grid_n(n_indices), 256, 0, cx.st>>>(gp); count_launch(); }
  return ob.finish(err, device, cx.st, n_indices, out_mem, out);
}

int32_t dbx_block_take_ranges(int32_t device, const dbx_block* block, const uint32_t* starts, const uint32_t* lens, int64_t n_ranges,
                              int32_t out_mem, dbx_block* out) {
  ErrorSink& err = g_create_error;
  if (!block || !out || n_ranges < 0 || (n_ranges > 0 && (!starts || !lens)) || block->num_cols > 64) { err.set("dbx_block_take_ranges: bad argument"); return DBX_ERR_INVALID; }
  CallCtx cx;
  DBX_TRY(cx.init(err, device));
  std::vector<int64_t> off((size_t)n_ranges + 1, 0);
  for (int64_t r = 0; r < n_ranges; ++r) {
    if ((int64_t)starts[r] + (int64_t)lens[r] > block->num_rows) { err.set("dbx_block_take_ranges: range outside the block"); return DBX_ERR_INVALID; }
    off[(size_t)r + 1] = off[(size_t)r] + lens[r];
  }
  const int64_t n_out = off[(size_t)n_ranges];
  DeviceView src;
  DBX_TRY(src.load(err, cx.st, block));
  DevBuf d_starts, d_off, d_idx;
  DBX_CUDA_TRY(err, d_starts.ensure((size_t)std::max<int64_t>(n_ranges, 1) * 4));
  DBX_CUDA_TRY(err, d_off.ensure((size_t)(n_ranges + 1) * 8));
  DBX_CUDA_TRY(err, d_idx.ensure((size_t)std::max<int64_t>(n_out, 1) * 4));
  if (n_ranges) DBX_CUDA_TRY(err, cudaMemcpyAsync(d_starts.p, starts, (size_t)n_ranges * 4, cudaMemcpyHostToDevice, cx.st));
  DBX_CUDA_TRY(err, cudaMemcpyAsync(d_off.p, off.data(), (size_t)(n_ranges + 1) * 8, cudaMemcpyHostToDevice, cx.st));
  if (n_out) { expand_ranges_kernel<<<grid_n(n_ranges * 32), 256, 0, cx.st>>>((const uint32_t*)d_starts.p, (const int64_t*)d_off.p, n_ranges, n_out, (uint32_t*)d_idx.p); count_launch(); }
  bool nullable[64];
  nullable_flags(block, nullable);
  OutputBuilder ob;
  DBX_TRY(ob.begin(err, device, cx.st, block, nullable, n_out));
  GatherParams gp;
  ob.fill(&gp, src, block);
  gp.n_out = n_out; gp.idx = (const uint32_t*)d_idx.p;
  if (n_out && gp.n_cols) { gather_rows_kernel<<<grid_n(n_out), 256, 0, cx.st>>>(gp); count_launch(); }
  int32_t st = ob.finish(err, device, cx.st, n_out, out_mem, out);
  DBX_CUDA_TRY(err, cudaStreamSynchronize(cx.st));  // `off` and the index buffers live on this frame
  return st;
}

int32_t dbx_block_scatter(int32_t device, const dbx_block* block, const uint32_t* indices, int32_t indices_mem, int32_t n_parts,
                          int32_t out_mem, dbx_block* outs) {
  ErrorSink& err = g_create_error;
  if (!block || !outs || n_parts < 1 || n_parts > 65536 || (block->num_rows > 0 && !indices) || block->num_cols > 64) { err.set("dbx_block_scatter: bad argument"); return DBX_ERR_INVALID; }
  const int64_t n = block->num_rows;
  if (n > rs::kMaxRows) { err.set("dbx_block_scatter: more than 2^30 - 1 rows"); return DBX_ERR_UNSUPPORTED; }
  CallCtx cx;
  DBX_TRY(cx.init(err, device));
  DeviceView src;
  DBX_TRY(src.load(err, cx.st, block));
  DevBuf ibuf, counts, keys0, keys1, rows0, rows1;
  const uint32_t* dpart = nullptr;
  DBX_TRY(idx_to_device(err, cx.st, indices, n, indices_mem, ibuf, &dpart));
  // rows of each target block, in input order = one STABLE radix pass (two above 256 targets) on the target index
  DBX_CUDA_TRY(err, counts.ensure((size_t)n_parts * 8 + 16));
  DBX_CUDA_TRY(err, cudaMemsetAsync(counts.p, 0, (size_t)n_parts * 8 + 16, cx.st));
  DBX_CUDA_TRY(err, keys0.ensure((size_t)std::max<int64_t>(n, 1) * 8));
  DBX_CUDA_TRY(err, keys1.ensure((size_t)std::max<int64_t>(n, 1) * 8));
  DBX_CUDA_TRY(err, rows0.ensure((size_t)std::max<int64_t>(n, 1) * 4));
  DBX_CUDA_TRY(err, rows1.ensure((size_t)std::max<int64_t>(n, 1) * 4));
  unsigned int* bad = (unsigned int*)((unsigned long long*)counts.p + n_parts);
  int buf = 0;
  RadixSorter sorter;
  if (n) {
    count_parts_kernel<<<grid_n(n), 256, 0, cx.st>>>(dpart, n, n_parts, (unsigned long long*)counts.p, bad);
    widen_u32_iota_kernel<<<grid_n(n), 256, 0, cx.st>>>(dpart, n, (uint64_t*)keys0.p, (uint32_t*)rows0.p);
    count_launch(2);
    DBX_TRY(sorter.sort(err, cx.st, (uint64_t*)keys0.p, (uint64_t*)keys1.p, (uint32_t*)rows0.p, (uint32_t*)rows1.p, n, 0, n_parts > 256 ? 16 : 8, false, 0,
                        0, &buf));
  }
  std::vector<unsigned long long> h((size_t)n_parts + 2, 0);
  DBX_CUDA_TRY(err, cudaMemcpyAsync(h.data(), counts.p, (size_t)n_parts * 8 + 16, cudaMemcpyDeviceToHost, cx.st));
  DBX_CUDA_TRY(err, cudaStreamSynchronize(cx.st));
  if (*(unsigned int*)&h[(size_t)n_parts]) { err.set("dbx_block_scatter: scatter index outside [0, n_parts)"); return DBX_ERR_INVALID; }
  const uint32_t* order = (const uint32_t*)(buf ? rows1.p : rows0.p);
  bool nullable[64];
  nullable_flags(block, nullable);
  int64_t off = 0;
  for (int q = 0; q < n_parts; ++q) {
    const int64_t m = (int64_t)h[(size_t)q];
    OutputBuilder ob;
    DBX_TRY(ob.begin(err, device, cx.st, block, nullable, m));
    GatherParams gp;
    ob.fill(&gp, src, block);
    gp.n_out = m; gp.idx = order + off;
    if (m && gp.n_cols) { gather_rows_kernel<<<grid_n(m), 256, 0, cx.st>>>(gp); count_launch(); }
    int32_t st = ob.finish(err, device, cx.st, m, out_mem, &outs[q]);
    if (st != DBX_OK) {
      for (int j = 0; j < q; ++j) dbx_block_release(&outs[j]);
      return st;
    }
    off += m;
  }
  DBX_CUDA_TRY(err, cudaStreamSynchronize(cx.st));
  return DBX_OK;
}

int32_t dbx_block_concat(int32_t device, const dbx_block* blocks, int32_t n_blocks, int32_t out_mem, dbx_block* out) {
  ErrorSink& err = g_create_error;
  if (!blocks || !out || n_blocks < 1) { err.set("dbx_block_concat: bad argument"); return DBX_ERR_INVALID; }
  const dbx_block* first = &blocks[0];
  if (first->num_cols > 64) { err.set("dbx_block_concat: too many columns"); return DBX_ERR_INVALID; }
  int64_t total = 0;
  bool nullable[64] = {};
  bool all_const[64];
  for (int c = 0; c < first->num_cols; ++c) all_const[c] = true;
  for (int b = 0; b < n_blocks; ++b) {
    if (blocks[b].num_cols != first->num_cols) { err.set("Unable to concat blocks with different number of columns"); return DBX_ERR_INVALID; }  // concat.rs:70-75
    for (int c = 0; c < first->num_cols; ++c) {
      const dbx_column& col = blocks[b].cols[c];
      if (col.dtype != first->cols[c].dtype || col.vec_dim != first->cols[c].vec_dim) { err.set("Unable to concat blocks with different schemas"); return DBX_ERR_INVALID; }
      if (col.validity || (col.is_const && col.konst.is_null)) nullable[c] = true;
      // a column stays BlockEntry::Const only if every block carries the same constant (concat.rs:96-110)
      if (!col.is_const) all_const[c] = false;
      else if (first->cols[c].is_const && (col.konst.is_null != first->cols[c].konst.is_null || col.konst.v.u64 != first->cols[c].konst.v.u64)) all_const[c] = false;
    }
    total += blocks[b].num_rows;
  }
  for (int c = 0; c < first->num_cols; ++c)
    if (!all_const[c] && is_vector_dtype(first->cols[c].dtype))
      for (int b = 0; b < n_blocks; ++b)
        if (blocks[b].cols[c].is_const) { err.set("dbx_block_concat: constant vector columns cannot be materialised"); return DBX_ERR_UNSUPPORTED; }
  CallCtx cx;
  DBX_TRY(cx.init(err, device));
  // prototype of the output schema: const only where every input is the same const
  std::vector<dbx_column> proto_cols(first->cols, first->cols + first->num_cols);
  for (int c = 0; c < first->num_cols; ++c) if (!all_const[c]) proto_cols[(size_t)c].is_const = 0;
  dbx_block proto = *first;
  proto.cols = proto_cols.data();
  OutputBuilder ob;
  DBX_TRY(ob.begin(err, device, cx.st, &proto, nullable, total));
  std::vector<DeviceView> views((size_t)n_blocks);
  int64_t off = 0;
  for (int b = 0; b < n_blocks; ++b) {
    const int64_t m = blocks[b].num_rows;
    // const entries that must be materialised become device columns of the repeated value
    dbx_block tmp = blocks[b];
    std::vector<dbx_column> tcols(blocks[b].cols, blocks[b].cols + blocks[b].num_cols);
    std::vector<DevBuf> fills;
    for (int c = 0; c < first->num_cols; ++c) {
      dbx_column& col = tcols[(size_t)c];
      if (!col.is_const || all_const[c]) continue;
      const int sz = col.dtype == DBX_BOOL ? 1 : dtype_size(col.dtype);
      std::vector<uint8_t> hostv((size_t)std::max<int64_t>(m, 1) * sz, 0);
      if (!col.konst.is_null) {
        for (int64_t i = 0; i < m; ++i) {
          uint8_t* d = hostv.data() + (size_t)i * sz;
          if (col.dtype == DBX_BOOL) d[0] = col.konst.v.u64 ? 1 : 0;
          else if (col.dtype == DBX_F32) { float f = (float)col.konst.v.f64; memcpy(d, &f, 4); }
          else if (col.dtype == DBX_F64) memcpy(d, &col.konst.v.f64, 8);
          else memcpy(d, &col.konst.v.u64, (size_t)sz);  // little endian: low bytes of the 64-bit image
        }
      }
      fills.emplace_back();
      if (col.dtype == DBX_BOOL) {
        std::vector<uint8_t> bits((size_t)(m + 7) / 8 + 1, 0);
        for (int64_t i = 0; i < m; ++i) if (hostv[(size_t)i]) bits[(size_t)(i >> 3)] |= (uint8_t)(1u << (i & 7));
        DBX_CUDA_TRY(err, fills.back().ensure(bits.size()));
        DBX_CUDA_TRY(err, cudaMemcpyAsync(fills.back().p, bits.data(), bits.size(), cudaMemcpyHostToDevice, cx.st));
        DBX_CUDA_TRY(err, cudaStreamSynchronize(cx.st));
      } else {
        DBX_CUDA_TRY(err, fills.back().ensure(hostv.size()));
        DBX_CUDA_TRY(err, cudaMemcpyAsync(fills.back().p, hostv.data(), hostv.size(), cudaMemcpyHostToDevice, cx.st));
        DBX_CUDA_TRY(err, cudaStreamSynchronize(cx.st));
      }
      const bool was_null = col.konst.is_null;
      col.is_const = 0; col.mem = DBX_MEM_DEVICE; col.data = fills.back().p; col.data_bit_offset = 0; col.validity = nullptr;
      if (was_null) {  // a NULL constant: all-zero validity
        fills.emplace_back();
        DBX_CUDA_TRY(err, fills.back().ensure((size_t)(m + 7) / 8 + 8));
        DBX_CUDA_TRY(err, cudaMemsetAsync(fills.back().p, 0, (size_t)(m + 7) / 8 + 8, cx.st));
        col.validity = (const uint8_t*)fills.back().p; col.validity_bit_offset = 0;
      }
    }
    tmp.cols = tcols.data();
    DBX_TRY(views[(size_t)b].load(err, cx.st, &tmp));
    GatherParams gp;
    ob.fill(&gp, views[(size_t)b], &proto);
    gp.n_out = m; gp.idx = nullptr; gp.src_row0 = 0; gp.dst_row0 = off;
    if (m && gp.n_cols) { gather_rows_kernel<<<grid_n(m), 256, 0, cx.st>>>(gp); count_launch(); }
    DBX_CUDA_TRY(err, cudaStreamSynchronize(cx.st));  // `fills` of this block are released at the end of the iteration
    off += m;
  }
  return ob.finish(err, device, cx.st, total, out_mem, out);
}

}  // extern "C"
