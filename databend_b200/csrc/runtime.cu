// runtime.cu — host runtime + the operator-independent part of the C-ABI.
#include "runtime.h"

#include <set>

#include <mutex>
#include <unordered_map>
#include <vector>

namespace dbx {

thread_local ErrorSink g_create_error;
std::atomic<int64_t> g_launches{0};

// ---------------------------------------------------------------- allocators
namespace {
std::mutex g_alloc_mu;
cudaStream_t g_util_stream[64] = {};
bool g_pool_ready[64] = {};
std::unordered_map<void*, size_t> g_pinned_live;            // ptr -> size class
std::unordered_map<size_t, std::vector<void*>> g_pinned_free;  // size class -> blocks

cudaError_t ensure_pool(int device) {
  if (g_pool_ready[device]) return cudaSuccess;
  cudaMemPool_t pool;
  cudaError_t e = cudaDeviceGetDefaultMemPool(&pool, device);
  if (e != cudaSuccess) return e;
  uint64_t thr = ~0ULL;
  e = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  if (e != cudaSuccess) return e;
  e = cudaStreamCreateWithFlags(&g_util_stream[device], cudaStreamNonBlocking);
  if (e != cudaSuccess) return e;
  g_pool_ready[device] = true;
  return cudaSuccess;
}
}  // namespace

cudaError_t pool_alloc(int device, cudaStream_t stream, size_t bytes, void** out) {
  {
    std::lock_guard<std::mutex> lk(g_alloc_mu);
    cudaError_t e = ensure_pool(device);
    if (e != cudaSuccess) return e;
  }
  return cudaMallocAsync(out, bytes ? bytes : 1, stream);
}
// streams of live operators: a buffer is freed on its producer's stream only while that stream exists
static std::set<cudaStream_t> g_live_streams;
void pool_free(int device, void* p, cudaStream_t producer) {
  if (!p) return;
  cudaStream_t s;
  {
    std::lock_guard<std::mutex> lk(g_alloc_mu);
    s = (producer && g_live_streams.count(producer)) ? producer : g_util_stream[device];
  }
  cudaFreeAsync(p, s);
}
cudaError_t pinned_alloc(size_t bytes, void** out) {
  size_t cls = 4096;
  while (cls < bytes) cls <<= 1;
  {
    std::lock_guard<std::mutex> lk(g_alloc_mu);
    auto it = g_pinned_free.find(cls);
    if (it != g_pinned_free.end() && !it->second.empty()) {
      *out = it->second.back();
      it->second.pop_back();
      g_pinned_live[*out] = cls;
      return cudaSuccess;
    }
  }
  cudaError_t e = cudaMallocHost(out, cls);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(g_alloc_mu);
  g_pinned_live[*out] = cls;
  return cudaSuccess;
}
void pinned_free(void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(g_alloc_mu);
  auto it = g_pinned_live.find(p);
  if (it == g_pinned_live.end()) { cudaFreeHost(p); return; }
  g_pinned_free[it->second].push_back(p);
  g_pinned_live.erase(it);
}

// ---------------------------------------------------------------- Stager
int32_t Stager::init(int device, cudaStream_t stream, ErrorSink* err) {
  device_ = device;
  stream_ = stream;
  err_ = err;
  for (auto& g : gens_) DBX_CUDA_TRY(*err_, cudaEventCreateWithFlags(&g.done, cudaEventDisableTiming));
  gather_ = !getenv("DBX_STAGE_NO_GATHER");
  if (!getenv("DBX_STAGE_ONE_STREAM")) {
    for (int i = 0; i < kAux; ++i) {
      DBX_CUDA_TRY(*err_, cudaStreamCreateWithFlags(&aux_[i], cudaStreamNonBlocking));
      DBX_CUDA_TRY(*err_, cudaEventCreateWithFlags(&aux_ev_[i], cudaEventDisableTiming));
    }
  }
  return DBX_OK;
}
Stager::~Stager() {
  for (auto& g : gens_)
    if (g.done) cudaEventDestroy(g.done);
  for (int i = 0; i < kAux; ++i) {
    if (aux_[i]) { cudaStreamSynchronize(aux_[i]); cudaStreamDestroy(aux_[i]); }
    if (aux_ev_[i]) cudaEventDestroy(aux_ev_[i]);
  }
}
// One CTA row (blockIdx.y) per segment, gridDim.x CTAs striding over its 16-byte words.
__global__ void __launch_bounds__(256) gather_segments_kernel(const Stager::Segment* segs) {
  const Stager::Segment sg = segs[blockIdx.y];
  const uint4* src = (const uint4*)sg.src;
  uint4* dst = (uint4*)sg.dst;
  const unsigned long long n16 = sg.bytes >> 4;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (unsigned long long)gridDim.x * blockDim.x)
    dst[i] = __ldcs(src + i);
  if (blockIdx.x == 0 && threadIdx.x < (sg.bytes & 15)) {  // tail bytes (columns narrower than 16 B per row)
    const unsigned long long o = (n16 << 4) + threadIdx.x;
    ((unsigned char*)sg.dst)[o] = ((const unsigned char*)sg.src)[o];
  }
}

int32_t Stager::join_aux() {
  if (!segs_.empty()) {
    const size_t bytes = segs_.size() * sizeof(Segment);
    DBX_CUDA_TRY(*err_, seg_host_[cur_].ensure(bytes));
    DBX_CUDA_TRY(*err_, seg_dev_[cur_].ensure(bytes));
    memcpy(seg_host_[cur_].p, segs_.data(), bytes);
    DBX_CUDA_TRY(*err_, cudaMemcpyAsync(seg_dev_[cur_].p, seg_host_[cur_].p, bytes, cudaMemcpyHostToDevice, stream_));
    const dim3 grid(8, (unsigned)segs_.size());
    gather_segments_kernel<<<grid, 256, 0, stream_>>>((const Segment*)seg_dev_[cur_].p);
    count_launch();
    DBX_CUDA_TRY(*err_, cudaGetLastError());
    segs_.clear();
  }
  for (int i = 0; i < kAux; ++i) {
    if (!aux_used_[i]) continue;
    aux_used_[i] = false;
    DBX_CUDA_TRY(*err_, cudaEventRecord(aux_ev_[i], aux_[i]));
    DBX_CUDA_TRY(*err_, cudaStreamWaitEvent(stream_, aux_ev_[i], 0));
  }
  return DBX_OK;
}
int32_t Stager::begin() {
  cur_ = (cur_ + 1) % kGenerations;
  Gen& g = gens_[cur_];
  if (g.pending) {
    DBX_CUDA_TRY(*err_, cudaEventSynchronize(g.done));
    g.pending = false;
  }
  return DBX_OK;
}
int32_t Stager::stage(const dbx_column& c, int slot, DevCol* out) {
  Gen& g = gens_[cur_];
  memset(out, 0, sizeof(*out));
  out->dtype = c.dtype;
  if (c.is_const) {
    out->is_const = c.konst.is_null ? 2 : 1;
    int cls = dtype_class(c.dtype);
    out->const_bits = scalar_bits(c.konst, cls);
    return DBX_OK;
  }
  const int64_t n = c.len;
  const bool is_bool = c.dtype == DBX_BOOL;
  if (!is_bool && dtype_size(c.dtype) == 0) {
    err_->set("unsupported column dtype for this operator");
    return DBX_ERR_UNSUPPORTED;
  }
  if (c.mem == DBX_MEM_DEVICE) {
    out->data = c.data;
    out->validity = c.validity;
    out->vbit_off = c.validity_bit_offset;
    out->dbit_off = c.data_bit_offset;
    return DBX_OK;
  }
  if ((int)g.data.size() <= slot) { g.data.resize(slot + 1); g.validity.resize(slot + 1); }
  if (is_bool) {
    int64_t b0 = c.data_bit_offset >> 3, b1 = (c.data_bit_offset + n + 7) >> 3;
    size_t bytes = (size_t)(b1 - b0);
    DBX_CUDA_TRY(*err_, g.data[slot].ensure(bytes ? bytes : 1));
    if (bytes) DBX_CUDA_TRY(*err_, cudaMemcpyAsync(g.data[slot].p, (const uint8_t*)c.data + b0, bytes, cudaMemcpyHostToDevice, stream_));
    out->dbit_off = c.data_bit_offset & 7;
    h2d_bytes += bytes;
  } else {
    size_t bytes = (size_t)n * dtype_size(c.dtype);
    DBX_CUDA_TRY(*err_, g.data[slot].ensure(bytes ? bytes : 1));
    if (bytes) DBX_CUDA_TRY(*err_, cudaMemcpyAsync(g.data[slot].p, c.data, bytes, cudaMemcpyHostToDevice, stream_));
    h2d_bytes += bytes;
  }
  out->data = g.data[slot].p;
  if (c.validity) {
    int64_t b0 = c.validity_bit_offset >> 3, b1 = (c.validity_bit_offset + n + 7) >> 3;
    size_t bytes = (size_t)(b1 - b0);
    DBX_CUDA_TRY(*err_, g.validity[slot].ensure(bytes ? bytes : 1));
    if (bytes) DBX_CUDA_TRY(*err_, cudaMemcpyAsync(g.validity[slot].p, c.validity + b0, bytes, cudaMemcpyHostToDevice, stream_));
    out->validity = (const uint8_t*)g.validity[slot].p;
    out->vbit_off = c.validity_bit_offset & 7;
    h2d_bytes += bytes;
  }
  return DBX_OK;
}
// Append `c` (a HOST column without validity) at row `row_off` of the generation's buffer for `slot`;
// the buffer holds `cap_rows` rows.  `out->data` is the buffer base (rows [0, row_off + c.len) valid).
int32_t Stager::stage_at(const dbx_column& c, int slot, int64_t row_off, int64_t cap_rows, DevCol* out) {
  Gen& g = gens_[cur_];
  const int esz = dtype_size(c.dtype);
  if (esz == 0 || c.is_const || c.validity || c.mem != DBX_MEM_HOST || row_off + c.len > cap_rows) {
    err_->set("internal: stage_at on a column that cannot be coalesced");
    return DBX_ERR_INVALID;
  }
  if ((int)g.data.size() <= slot) { g.data.resize(slot + 1); g.validity.resize(slot + 1); }
  if (g.data[slot].bytes < (size_t)cap_rows * esz) {
    if (row_off != 0) { err_->set("internal: staging buffer too small in the middle of a batch"); return DBX_ERR_INVALID; }
    DBX_CUDA_TRY(*err_, g.data[slot].ensure((size_t)cap_rows * esz));
  }
  h2d_bytes += (size_t)c.len * esz;
  memset(out, 0, sizeof(*out));
  out->dtype = c.dtype;
  out->data = g.data[slot].p;
  if (gather_ && c.len && ((uintptr_t)c.data & 15) == 0 && (((size_t)row_off * esz) & 15) == 0 && segs_.size() < 60000) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, c.data) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) {
      segs_.push_back(Segment{at.devicePointer, (char*)g.data[slot].p + (size_t)row_off * esz, (unsigned long long)c.len * esz});
      return DBX_OK;
    }
    cudaGetLastError();  // pageable memory: the DMA path below
  }
  cudaStream_t cs = stream_;
  if (aux_[0]) { cs = aux_[slot % kAux]; aux_used_[slot % kAux] = true; }
  if (c.len) DBX_CUDA_TRY(*err_, cudaMemcpyAsync((char*)g.data[slot].p + (size_t)row_off * esz, c.data, (size_t)c.len * esz, cudaMemcpyHostToDevice, cs));
  return DBX_OK;
}
int32_t Stager::end() {
  Gen& g = gens_[cur_];
  DBX_CUDA_TRY(*err_, cudaEventRecord(g.done, stream_));
  g.pending = true;
  return DBX_OK;
}

// ---------------------------------------------------------------- Op base
int32_t Op::base_init(int dev) {
  device = dev;
  DBX_CUDA_TRY(err, cudaSetDevice(device));
  DBX_CUDA_TRY(err, cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  { std::lock_guard<std::mutex> lk(g_alloc_mu); g_live_streams.insert(stream); }
  for (auto& pr : ev_ring)
    for (auto& e : pr) DBX_CUDA_TRY(err, cudaEventCreate(&e));
  return DBX_OK;
}
Op::~Op() {
  for (auto& pr : ev_ring)
    for (auto& e : pr)
      if (e) cudaEventDestroy(e);
  if (stream) {
    // blocks this operator produced may outlive it: finish its work first, so that their buffers
    // can go back to the pool on the utility stream afterwards
    cudaStreamSynchronize(stream);
    { std::lock_guard<std::mutex> lk(g_alloc_mu); g_live_streams.erase(stream); }
    cudaStreamDestroy(stream);
  }
}
int32_t Op::timing_begin() {
  ev_idx += 1;
  DBX_CUDA_TRY(err, cudaEventRecord(ev_ring[ev_idx % kEvRing][0], stream));
  return DBX_OK;
}
int32_t Op::timing_end() {
  DBX_CUDA_TRY(err, cudaEventRecord(ev_ring[ev_idx % kEvRing][1], stream));
  timed = true;
  return DBX_OK;
}

int32_t fill_owned_block(OwnedBlock* ob, dbx_block* out) {
  out->num_cols = (int32_t)ob->cols.size();
  out->cols = ob->cols.data();
  out->num_rows = ob->cols.empty() ? 0 : ob->cols[0].len;
  out->meta = nullptr;
  out->owner = ob;
  out->reserved = 0;
  return DBX_OK;
}

// Hand a finished device-resident result to the caller: as is (device), or copied into pinned
// host memory (zero-copy wrappable by the caller, released through dbx_block_release).
// BOOL columns hold packed bits (like validity).
int32_t pull_owned_block(std::unique_ptr<OwnedBlock>& result_dev, int device, cudaStream_t stream, ErrorSink& err, int32_t out_mem,
                         dbx_block* out) {
  if (out_mem == DBX_MEM_DEVICE) {
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    OwnedBlock* ob = result_dev.release();
    return fill_owned_block(ob, out);
  }
  auto hb = std::make_unique<OwnedBlock>();
  hb->device = device;
  for (const dbx_column& dc : result_dev->cols) {
    dbx_column c = dc;
    c.mem = DBX_MEM_HOST;
    if (dc.is_const) { hb->cols.push_back(c); continue; }
    size_t bytes = dc.dtype == DBX_BOOL ? (size_t)(dc.data_bit_offset + dc.len + 7) / 8
                 : (size_t)dc.len * column_row_bytes(dc.dtype, dc.vec_dim);
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
  for (dbx_column& c : hb->cols) {
    if (!c.validity) continue;
    int64_t nulls = 0;
    for (int64_t i = 0; i < c.len; ++i) nulls += !((c.validity[i >> 3] >> (i & 7)) & 1);
    c.null_count = nulls;
  }
  result_dev.reset();
  return fill_owned_block(hb.release(), out);
}


// factories implemented next to each operator
Op* make_agg_partial_op(const dbx_agg_params* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int device,
                        int32_t* st);
Op* make_agg_final_op(const dbx_agg_params* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int device,
                      int32_t* st);
Op* make_filter_op(const dbx_predicate* p, const int32_t* types, int32_t n, const dbx_expr* comp, int32_t n_comp, int device, int32_t* st);
Op* make_topk_op(const dbx_topk_params* p, const int32_t* types, int32_t n, int device, int32_t* st);
Op* make_join_op(const dbx_join_params* p, const int32_t* types, int32_t n, int device, int32_t* st);
Op* make_window_op(const dbx_window_params* p, const int32_t* types, int32_t n, int device, int32_t* st);

}  // namespace dbx

using namespace dbx;

// ================================================================ C-ABI (generic part)
extern "C" {

int32_t dbx_abi_version(void) { return DBX_ABI_VERSION; }

int32_t dbx_device_count(int32_t* n) {
  int c = 0;
  cudaError_t e = cudaGetDeviceCount(&c);
  if (e != cudaSuccess || c == 0) {
    if (n) *n = 0;
    g_create_error.set(std::string("no usable CUDA device: ") + cudaGetErrorString(e) + " (libdbx has no CPU fallback)");
    return DBX_ERR_NO_DEVICE;
  }
  if (n) *n = c;
  return DBX_OK;
}

const char* dbx_last_error(const dbx_op* op) {
  if (!op) return g_create_error.msg.c_str();
  return reinterpret_cast<const Op*>(op)->err.msg.c_str();
}

int32_t dbx_host_alloc(size_t bytes, void** out) {
  DBX_CUDA_TRY(g_create_error, cudaMallocHost(out, bytes ? bytes : 1));
  return DBX_OK;
}
int32_t dbx_host_free(void* p) {
  DBX_CUDA_TRY(g_create_error, cudaFreeHost(p));
  return DBX_OK;
}
int32_t dbx_host_register(void* p, size_t bytes) {
  DBX_CUDA_TRY(g_create_error, cudaHostRegister(p, bytes, cudaHostRegisterDefault));
  return DBX_OK;
}
int32_t dbx_host_unregister(void* p) {
  DBX_CUDA_TRY(g_create_error, cudaHostUnregister(p));
  return DBX_OK;
}
int32_t dbx_device_alloc(int32_t device, size_t bytes, void** out) {
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(device));
  DBX_CUDA_TRY(g_create_error, cudaMalloc(out, bytes ? bytes : 1));
  return DBX_OK;
}
int32_t dbx_device_free(int32_t device, void* p) {
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(device));
  DBX_CUDA_TRY(g_create_error, cudaFree(p));
  return DBX_OK;
}
int32_t dbx_memcpy_h2d(int32_t device, void* dst, const void* src, size_t bytes) {
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(device));
  DBX_CUDA_TRY(g_create_error, cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
  return DBX_OK;
}
int32_t dbx_memcpy_d2h(int32_t device, void* dst, const void* src, size_t bytes) {
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(device));
  DBX_CUDA_TRY(g_create_error, cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return DBX_OK;
}
int32_t dbx_memcpy_d2d(int32_t device, void* dst, const void* src, size_t bytes) {
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(device));
  DBX_CUDA_TRY(g_create_error, cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToDevice));
  return DBX_OK;
}
int32_t dbx_device_synchronize(int32_t device) {
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(device));
  DBX_CUDA_TRY(g_create_error, cudaDeviceSynchronize());
  return DBX_OK;
}

int32_t dbx_op_create(int32_t kind, const void* params, const int32_t* input_types, int32_t n_input_cols,
                      int32_t device, dbx_op** out) {
  return dbx_op_create_computed(kind, params, input_types, n_input_cols, nullptr, 0, device, out);
}

int32_t dbx_op_create_computed(int32_t kind, const void* params, const int32_t* input_types, int32_t n_input_cols,
                               const dbx_expr* computed, int32_t n_computed, int32_t device, dbx_op** out) {
  if (!out || !params) { g_create_error.set("dbx_op_create: null argument"); return DBX_ERR_INVALID; }
  if (n_computed < 0 || n_computed > DBX_MAX_COMPUTED_COLS) { g_create_error.set("dbx_op_create_computed: n_computed outside 0 .. DBX_MAX_COMPUTED_COLS"); return DBX_ERR_INVALID; }
  if (n_computed > 0 && !computed) { g_create_error.set("dbx_op_create_computed: null computed list"); return DBX_ERR_INVALID; }
  if (n_computed > 0 && n_input_cols + n_computed > 64) { g_create_error.set("dbx_op_create_computed: more than 64 input and computed columns"); return DBX_ERR_INVALID; }
  if (n_computed > 0 && (kind == DBX_OP_TOPK || kind == DBX_OP_JOIN || kind == DBX_OP_WINDOW)) {
    g_create_error.set("dbx_op_create_computed: computed columns are taken by the filter and aggregate operators only");
    return DBX_ERR_UNSUPPORTED;
  }
  *out = nullptr;
  int32_t ndev = 0;
  DBX_TRY(dbx_device_count(&ndev));
  if (device < 0 || device >= ndev) { g_create_error.set("dbx_op_create: device index out of range"); return DBX_ERR_INVALID; }
  int32_t st = DBX_OK;
  Op* op = nullptr;
  switch (kind) {
    case DBX_OP_AGG_PARTIAL: op = make_agg_partial_op((const dbx_agg_params*)params, input_types, n_input_cols, computed, n_computed, device, &st); break;
    case DBX_OP_AGG_FINAL: op = make_agg_final_op((const dbx_agg_params*)params, input_types, n_input_cols, computed, n_computed, device, &st); break;
    case DBX_OP_FILTER: op = make_filter_op((const dbx_predicate*)params, input_types, n_input_cols, computed, n_computed, device, &st); break;
    case DBX_OP_TOPK: op = make_topk_op((const dbx_topk_params*)params, input_types, n_input_cols, device, &st); break;
    case DBX_OP_JOIN: op = make_join_op((const dbx_join_params*)params, input_types, n_input_cols, device, &st); break;
    case DBX_OP_WINDOW: op = make_window_op((const dbx_window_params*)params, input_types, n_input_cols, device, &st); break;
    default: g_create_error.set("dbx_op_create: unknown operator kind"); return DBX_ERR_INVALID;
  }
  if (!op) return st == DBX_OK ? DBX_ERR_INVALID : st;
  op->kind = kind;
  *out = reinterpret_cast<dbx_op*>(op);
  return DBX_OK;
}

int32_t dbx_op_destroy(dbx_op* op) {
  if (!op) return DBX_OK;
  Op* o = reinterpret_cast<Op*>(op);
  cudaSetDevice(o->device);
  if (o->stream) cudaStreamSynchronize(o->stream);
  delete o;
  return DBX_OK;
}

#define DBX_OP_ENTER_ANY(op)                                                   \
  if (!(op)) return DBX_ERR_INVALID;                                           \
  Op* o = reinterpret_cast<Op*>(op);                                           \
  DBX_CUDA_TRY(o->err, cudaSetDevice(o->device));
// a poisoned handle (its input failed to evaluate) takes reset and destroy only
#define DBX_OP_ENTER(op)                                                       \
  DBX_OP_ENTER_ANY(op)                                                         \
  if (o->poisoned) { o->err.set("the operator's input failed to evaluate (" + o->poison_msg + "): reset it"); return DBX_ERR_STATE; }

int32_t dbx_op_push(dbx_op* op, const dbx_block* block) {
  DBX_OP_ENTER(op);
  if (!block) { o->err.set("push: null block"); return DBX_ERR_INVALID; }
  if (o->finished) { o->err.set("push after finish"); return DBX_ERR_STATE; }
  return o->push(block);
}
int32_t dbx_op_finish(dbx_op* op) {
  DBX_OP_ENTER(op);
  if (o->finished) return DBX_OK;
  int32_t st = o->finish();
  if (st == DBX_OK) o->finished = true;
  return st;
}
int32_t dbx_op_pull(dbx_op* op, int32_t out_mem, dbx_block* out, int32_t* has_block) {
  DBX_OP_ENTER(op);
  if (!out || !has_block) { o->err.set("pull: null argument"); return DBX_ERR_INVALID; }
  *has_block = 0;
  return o->pull(out_mem, out, has_block);
}
int32_t dbx_op_reset(dbx_op* op) {
  DBX_OP_ENTER_ANY(op);
  int32_t st = o->reset();
  if (st == DBX_OK) { o->finished = false; o->poisoned = false; }
  return st;
}
int32_t dbx_block_release(dbx_block* block) {
  if (!block || !block->owner) return DBX_OK;
  OwnedBlock* ob = reinterpret_cast<OwnedBlock*>(block->owner);
  cudaSetDevice(ob->device);
  delete ob;
  block->owner = nullptr;
  block->cols = nullptr;
  block->num_cols = 0;
  return DBX_OK;
}

int64_t dbx_kernel_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int32_t dbx_op_kernel_ms(dbx_op* op, int32_t back, float* ms) {
  DBX_OP_ENTER(op);
  if (!o->timed || back < 0 || back >= Op::kEvRing || back > o->ev_idx) { o->err.set("no timed kernel that far back on this handle"); return DBX_ERR_STATE; }
  cudaEvent_t* pr = o->ev_ring[(o->ev_idx - back) % Op::kEvRing];
  DBX_CUDA_TRY(o->err, cudaEventSynchronize(pr[1]));
  DBX_CUDA_TRY(o->err, cudaEventElapsedTime(ms, pr[0], pr[1]));
  return DBX_OK;
}
int32_t dbx_op_last_kernel_ms(dbx_op* op, float* ms) { return dbx_op_kernel_ms(op, 0, ms); }
int32_t dbx_op_kernel_variant(dbx_op* op, char* out, int32_t cap) {
  if (!op || !out || cap <= 0) return DBX_ERR_INVALID;
  snprintf(out, (size_t)cap, "%s", reinterpret_cast<Op*>(op)->kernel_variant());
  return DBX_OK;
}
int32_t dbx_op_stream(dbx_op* op, void** stream) {
  DBX_OP_ENTER(op);
  *stream = (void*)o->stream;
  return DBX_OK;
}
int32_t dbx_op_inputs_consumed(dbx_op* op) {
  DBX_OP_ENTER(op);
  return o->wait_inputs();
}
int32_t dbx_op_synchronize(dbx_op* op) {
  DBX_OP_ENTER(op);
  DBX_TRY(o->wait_inputs());  // reads recorded but not yet enqueued (coalesced small pushes) first: the header promises them consumed
  DBX_CUDA_TRY(o->err, cudaStreamSynchronize(o->stream));
  return DBX_OK;
}

}  // extern "C"
