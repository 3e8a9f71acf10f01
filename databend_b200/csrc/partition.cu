// partition.cu — dbx_hash_partition: radix/hash partitioning of a device-resident block by the
// owner of its key column, the step in front of the all-to-all of a partitioned hash join
// (BASELINE configs[2]; the reference shuffles both join sides by key hash between nodes:
// src/query/service/src/servers/flight/v1/scatter/flight_scatter_hash.rs, and within a node
// partitions build rows in new_hash_join/grace/*).  The owner rule is the one the aggregate
// exchange uses (agg_kernels.cuh: owner_of), so both shuffles agree.
#include <algorithm>
#include <vector>

#include "runtime.h"

namespace dbx {
namespace {

__device__ __forceinline__ uint64_t part_load_key(const DevCol& c, int64_t row) {
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
__global__ void __launch_bounds__(256) partition_count_kernel(const __grid_constant__ PartParams p) {
  __shared__ unsigned int s_cnt[kMaxParts];
  if (threadIdx.x < kMaxParts) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  // (the owner is passed through an opaque asm: with nvcc 12.9 -O3 the peeled remainder of this
  // loop otherwise folds the scaled index into a wrong loop-invariant multiplier — seen in SASS as
  // base + hash_hi * (7 n_parts + ...) and caught by compute-sanitizer as a misaligned ATOMS)
#pragma unroll 1
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n_rows; i += (int64_t)gridDim.x * blockDim.x) {
    int owner = part_owner(part_load_key(p.key, i), p.n_parts);
    asm volatile("" : "+r"(owner));
    atomicAdd(&s_cnt[owner], 1u);
  }
  __syncthreads();
  if (threadIdx.x < p.n_parts && s_cnt[threadIdx.x]) atomicAdd(&p.counters[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
}

// per step of 1024 rows (4 per thread): one reservation per (CTA, owner); the step's values are
// laid out owner after owner in shared memory and copied out in runs, so the stores are coalesced
// per partition and the barriers are amortised over four rows per thread
constexpr int kPartRows = 4;
__global__ void __launch_bounds__(256) partition_scatter_kernel(const __grid_constant__ PartParams p) {
  __shared__ unsigned int s_cnt[kMaxParts];
  __shared__ unsigned int s_off[kMaxParts + 1];
  __shared__ unsigned long long s_base[kMaxParts];
  __shared__ unsigned long long s_dst[256 * kPartRows];
  __shared__ uint64_t s_val[256 * kPartRows];
  const int64_t step_rows = (int64_t)blockDim.x * kPartRows;
  const int64_t n_steps = (p.n_rows + step_rows - 1) / step_rows;
#pragma unroll 1
  for (int64_t st = blockIdx.x; st < n_steps; st += gridDim.x) {
    if (threadIdx.x < kMaxParts) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const int64_t i0 = st * step_rows + threadIdx.x;
    int owner[kPartRows];
    unsigned int slot[kPartRows];
#pragma unroll
    for (int j = 0; j < kPartRows; ++j) {
      const int64_t i = i0 + (int64_t)j * blockDim.x;
      owner[j] = -1;
      slot[j] = 0;
      if (i < p.n_rows) {
        int o = part_owner(part_load_key(p.key, i), p.n_parts);
        asm volatile("" : "+r"(o));
        owner[j] = o;
        slot[j] = atomicAdd(&s_cnt[o], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int o = 0;
      for (int r = 0; r < p.n_parts; ++r) { s_off[r] = o; o += s_cnt[r]; }
      s_off[p.n_parts] = o;
    }
    if (threadIdx.x < p.n_parts && s_cnt[threadIdx.x])
      s_base[threadIdx.x] = atomicAdd(&p.counters[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kPartRows; ++j) {
      if (owner[j] >= 0) {
        const unsigned int local = slot[j];
        slot[j] = s_off[owner[j]] + local;
        s_dst[slot[j]] = s_base[owner[j]] + local;
      }
    }
    const unsigned int total = s_off[p.n_parts];
    for (int c = 0; c < p.n_cols; ++c) {
      const PartCol& pc = p.cols[c];
      __syncthreads();
#pragma unroll
      for (int j = 0; j < kPartRows; ++j) {
        if (owner[j] < 0) continue;
        const int64_t i = i0 + (int64_t)j * blockDim.x;
        uint64_t v;
        if (pc.size == 8) v = ((const uint64_t*)pc.src)[i];
        else if (pc.size == 4) v = ((const uint32_t*)pc.src)[i];
        else if (pc.size == 2) v = ((const uint16_t*)pc.src)[i];
        else v = ((const uint8_t*)pc.src)[i];
        s_val[slot[j]] = v;
      }
      __syncthreads();
      for (unsigned int t = threadIdx.x; t < total; t += blockDim.x) {
        const int64_t o = (int64_t)s_dst[t];
        const uint64_t v = s_val[t];
        if (pc.size == 8) ((uint64_t*)pc.dst)[o] = v;
        else if (pc.size == 4) ((uint32_t*)pc.dst)[o] = (uint32_t)v;
        else if (pc.size == 2) ((uint16_t*)pc.dst)[o] = (uint16_t)v;
        else ((uint8_t*)pc.dst)[o] = (uint8_t)v;
      }
    }
    __syncthreads();
  }
}

}  // namespace


// Stream-ordered hash partition of device columns (used by dbx_hash_partition).  `counters`:
// device scratch of kMaxParts u64.  host_counts/host_offsets: host arrays; the call synchronises the stream once (the counts are needed to place the runs).
int32_t hash_partition_device(ErrorSink& err, cudaStream_t stream, const PartParams& params, unsigned long long* counters,
                              int64_t* host_offsets) {
  PartParams p = params;
  p.counters = counters;
  DBX_CUDA_TRY(err, cudaMemsetAsync(counters, 0, (size_t)kMaxParts * 8, stream));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((p.n_rows + 1023) / 1024, (int64_t)kNumSMs * 8));
  if (p.n_rows > 0) {
    partition_count_kernel<<<grid, 256, 0, stream>>>(p);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
  }
  std::vector<unsigned long long> h((size_t)p.n_parts);
  DBX_CUDA_TRY(err, cudaMemcpyAsync(h.data(), counters, (size_t)p.n_parts * 8, cudaMemcpyDeviceToHost, stream));
  DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
  std::vector<unsigned long long> cur((size_t)p.n_parts);
  int64_t total = 0;
  for (int i = 0; i < p.n_parts; ++i) { host_offsets[i] = total; cur[i] = (unsigned long long)total; total += (int64_t)h[i]; }
  host_offsets[p.n_parts] = total;
  if (p.n_rows > 0 && p.n_cols > 0) {
    DBX_CUDA_TRY(err, cudaMemcpyAsync(counters, cur.data(), (size_t)p.n_parts * 8, cudaMemcpyHostToDevice, stream));
    partition_scatter_kernel<<<grid, 256, 0, stream>>>(p);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
    DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));  // `cur` lives on this stack frame
  }
  return DBX_OK;
}

}  // namespace dbx

using namespace dbx;

extern "C" int32_t dbx_hash_partition(int32_t device, const dbx_block* block, int32_t key_col, int32_t n_parts,
                                      void* const* out_cols, int64_t* part_offsets) {
  ErrorSink& err = g_create_error;
  if (!block || !out_cols || !part_offsets || n_parts < 1 || n_parts > kMaxParts) { err.set("dbx_hash_partition: bad argument"); return DBX_ERR_INVALID; }
  if (block->num_cols < 1 || block->num_cols > kMaxPartCols || key_col < 0 || key_col >= block->num_cols) { err.set("dbx_hash_partition: bad column count / key column"); return DBX_ERR_INVALID; }
  int32_t ndev = 0;
  DBX_TRY(dbx_device_count(&ndev));
  DBX_CUDA_TRY(err, cudaSetDevice(device));
  PartParams p;
  memset(&p, 0, sizeof(p));
  p.n_cols = block->num_cols; p.n_parts = n_parts; p.n_rows = block->num_rows;
  for (int c = 0; c < block->num_cols; ++c) {
    const dbx_column& col = block->cols[c];
    if (col.mem != DBX_MEM_DEVICE || col.is_const || col.validity || dtype_size(col.dtype) == 0 || col.len != block->num_rows) {
      err.set("dbx_hash_partition: columns must be device-resident, non-nullable, non-const numeric columns");
      return DBX_ERR_UNSUPPORTED;
    }
    p.cols[c].src = col.data; p.cols[c].dst = out_cols[c]; p.cols[c].size = dtype_size(col.dtype);
  }
  if (dtype_class(block->cols[key_col].dtype) == VC_FLT) { err.set("dbx_hash_partition: key must be an integer column"); return DBX_ERR_UNSUPPORTED; }
  p.key.data = block->cols[key_col].data; p.key.dtype = block->cols[key_col].dtype;
  DevBuf counters;
  DBX_CUDA_TRY(err, counters.ensure((size_t)kMaxParts * 8));
  return hash_partition_device(err, nullptr, p, (unsigned long long*)counters.p, part_offsets);
}
