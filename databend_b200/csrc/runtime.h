// runtime.h — host runtime of libdbx: operator base class, device buffers, host->HBM staging.
#pragma once
#include <memory>
#include <vector>

#include "common.cuh"

namespace dbx {

// RAII device allocation on a fixed device.
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  int device = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
  DevBuf& operator=(DevBuf&& o) noexcept {
    release();
    p = o.p; bytes = o.bytes; device = o.device;
    o.p = nullptr; o.bytes = 0;
    return *this;
  }
  ~DevBuf() { release(); }
  void release() {
    if (p) { cudaFree(p); p = nullptr; bytes = 0; }
  }
  // grow-only; contents are NOT preserved
  cudaError_t ensure(size_t need) {
    if (need <= bytes) return cudaSuccess;
    release();
    size_t cap = need + need / 4 + 256;
    cudaError_t e = cudaMalloc(&p, cap);
    if (e == cudaSuccess) bytes = cap; else p = nullptr;
    return e;
  }
};

struct PinnedBuf {
  void* p = nullptr;
  size_t bytes = 0;
  ~PinnedBuf() { if (p) cudaFreeHost(p); }
  cudaError_t ensure(size_t need) {
    if (need <= bytes) return cudaSuccess;
    if (p) { cudaFreeHost(p); p = nullptr; bytes = 0; }
    cudaError_t e = cudaMallocHost(&p, need);
    if (e == cudaSuccess) bytes = need;
    return e;
  }
};

// Stream-ordered device allocations from the device's default memory pool (release threshold
// raised so freed blocks are reused instead of returned to the driver): per-query result and
// exchange buffers cost microseconds instead of a cudaMalloc/cudaFree round trip.
cudaError_t pool_alloc(int device, cudaStream_t stream, size_t bytes, void** out);
void pool_free(int device, void* p, cudaStream_t producer = nullptr);
// Cached pinned host allocations (cudaMallocHost is milliseconds per call): power-of-two size
// classes, freed blocks are kept for reuse.
cudaError_t pinned_alloc(size_t bytes, void** out);
void pinned_free(void* p);

// Library-owned output block: columns + the buffers that back them.
struct OwnedBlock {
  std::vector<dbx_column> cols;
  std::vector<void*> host_allocs;  // pinned_alloc
  std::vector<void*> dev_allocs;   // pool_alloc
  int device = 0;
  // Stream of the operator that produced the device buffers: they are returned to the pool IN
  // ORDER behind whatever that stream still has enqueued (a block dropped right after a push may
  // still be written by the kernels of that push).  Operators that are gone have synchronised
  // their stream on destruction, and null means "the producer already waited".
  cudaStream_t stream = nullptr;
  ~OwnedBlock() {
    for (void* p : host_allocs) pinned_free(p);
    for (void* p : dev_allocs) pool_free(device, p, stream);
  }
};

// Host -> HBM staging of the columns an operator reads from a pushed block.
// A ring of generations lets push(i+1) copy while the kernel of push(i) still runs;
// a generation is reused only after the event recorded behind its consumer has fired.
class Stager {
 public:
  struct Segment { const void* src; void* dst; unsigned long long bytes; };
  static constexpr int kGenerations = 4;
  int32_t init(int device, cudaStream_t stream, ErrorSink* err);
  ~Stager();
  // Begin staging for one push: waits until the next generation is free.
  int32_t begin();
  // Make column `c` of the pushed block available on the device (copying if it lives on the
  // host) and describe it as a DevCol.  `slot` indexes the per-generation buffers.
  int32_t stage(const dbx_column& c, int slot, DevCol* out);
  // Coalescing of small host blocks: append the column at row `row_off` of a `cap_rows`-row buffer.
  int32_t join_aux();
  int32_t stage_at(const dbx_column& c, int slot, int64_t row_off, int64_t cap_rows, DevCol* out);
  // Record that all kernels consuming this generation have been enqueued.
  int32_t end();
  int64_t h2d_bytes = 0;  // instrumentation

 private:
  struct Gen {
    std::vector<DevBuf> data, validity;
    cudaEvent_t done = nullptr;
    bool pending = false;
  };
  Gen gens_[kGenerations];
  int cur_ = -1;
  int device_ = 0;
  cudaStream_t stream_ = nullptr;
  // Coalesced small pushes (stage_at) spread their copies over a few auxiliary streams: a 512 KB
  // transfer leaves the copy engine idle for a few microseconds between descriptors, several
  // engines in flight keep PCIe busy.  join_aux() makes the operator stream wait for them.
  // Pinned (mapped) host columns are not copied by the DMA engines at all: stage_at only records
  // {source, destination, bytes}, and join_aux() launches ONE gather kernel per batch whose CTAs
  // read the host columns over PCIe with 128-bit loads (gather_segments_kernel) — no per-block
  // CUDA call is left on the submitting thread.
  std::vector<Segment> segs_;
  PinnedBuf seg_host_[kGenerations];
  DevBuf seg_dev_[kGenerations];
  bool gather_ = true;
  static constexpr int kAux = 3;
  cudaStream_t aux_[kAux] = {};
  cudaEvent_t aux_ev_[kAux] = {};
  bool aux_used_[kAux] = {};
  ErrorSink* err_ = nullptr;
};

// Operator handle behind `dbx_op*` (the Processor shell of the reference: event()/process()
// are driven by the caller; push = transform/consume, finish = on_finish, pull = output port).
class Op {
 public:
  virtual ~Op();
  int32_t base_init(int device);
  virtual int32_t push(const dbx_block* b) = 0;
  virtual int32_t finish() = 0;
  virtual int32_t pull(int32_t out_mem, dbx_block* out, int32_t* has_block) = 0;
  virtual int32_t reset() { err.set("reset not supported by this operator"); return DBX_ERR_UNSUPPORTED; }
  // Block until every pushed block has been read completely (see dbx_op_inputs_consumed).  The
  // consumers of a pushed block are all enqueued on `stream` before push returns.
  virtual int32_t wait_inputs() {
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
    return DBX_OK;
  }
  // which build of the hot kernel serves this handle ("specialised" / "precompiled kernels (why)")
  virtual const char* kernel_variant() { return "precompiled kernels"; }

  int kind = -1;
  int device = 0;
  cudaStream_t stream = nullptr;
  ErrorSink err;
  // event pairs bracketing the dominant kernel(s) of the most recent pushes (a small ring, so the
  // kernel of push i can still be read after push i+1 was enqueued)
  static constexpr int kEvRing = 8;
  cudaEvent_t ev_ring[kEvRing][2] = {};
  int64_t ev_idx = -1;
  int32_t timing_begin();
  int32_t timing_end();
  bool timed = false;
  bool finished = false;
  // an evaluation error of the pushed input: every call but reset / destroy fails until reset
  bool poisoned = false;
  std::string poison_msg;
  void poison(const std::string& m) { poisoned = true; poison_msg = m; err.set(m); }
};

// Converts a scalar to the 64-bit image the kernels use for its class (i64 / u64 / f64 bits).
inline uint64_t scalar_bits(const dbx_scalar& s, int as_class) {
  int cls = dtype_class(s.dtype);
  if (as_class == VC_FLT) {
    double d = cls == VC_FLT ? s.v.f64 : (cls == VC_INT ? (double)s.v.i64 : (double)s.v.u64);
    uint64_t b;
    memcpy(&b, &d, 8);
    return b;
  }
  return s.v.u64;  // i64 and u64 share the two's complement image
}

int32_t fill_owned_block(OwnedBlock* ob, dbx_block* out);
// Hand a finished device-resident block to the caller: as is (device), or copied into pinned host
// memory (zero-copy wrappable by the caller, released through dbx_block_release).
int32_t pull_owned_block(std::unique_ptr<OwnedBlock>& result_dev, int device, cudaStream_t stream, ErrorSink& err, int32_t out_mem,
                         dbx_block* out);

// ---- hash partitioning of device columns (partition.cu)
constexpr int kMaxParts = 64;
constexpr int kMaxPartCols = 16;
struct PartCol {
  const void* src;
  void* dst;
  int32_t size;
  int32_t pad;
};
struct PartParams {
  DevCol key;
  PartCol cols[kMaxPartCols];
  int32_t n_cols, n_parts;
  int64_t n_rows;
  unsigned long long* counters;  // [n_parts]: counts (pass 1) / cursors (pass 2)
};
// owner of a key (common.cuh: hash_to_part)
__host__ __device__ __forceinline__ int part_owner(uint64_t key, int n_parts) { return hash_to_part(agg_hash_u64(key), n_parts); }
int32_t hash_partition_device(ErrorSink& err, cudaStream_t stream, const PartParams& params, unsigned long long* counters,
                              int64_t* host_offsets);

}  // namespace dbx
