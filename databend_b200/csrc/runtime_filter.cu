// runtime_filter.cu — join runtime filters: min-max, IN-list and split-block bloom filter built on
// the device from the join's HBM-resident build keys, and applied to probe blocks.
//
// Reference replaced (paths relative to the databend source tree, src/query):
//   RuntimeFilterLocalBuilder (thresholds on the running build rows, IN-list dedup)
//                                               service/.../hash_join/runtime_filter/local_builder.rs:86-274
//   bloom enabling rule (build_table_rows, selectivity)   .../hash_join/runtime_filter/builder.rs:17-57
//   build_runtime_filter_infos / build_bloom_filter        .../hash_join/runtime_filter/convert.rs:50-117,242-272
//   Sbbf::new_with_ndv_fpp / insert_hash / check_hash      catalog/src/sbbf.rs:220-291
//   ExprBloomFilter::apply (the probe-side bitmap)         storages/fuse/src/pruning/expr_bloom_filter.rs:31-44
//
// Build: per key pair one min/max reduction over the non-NULL keys (warp shuffles, one atomic per
// CTA; it also counts them), the IN-list in one CTA (first occurrences ranked among the distinct
// values: sorted and de-duplicated without a sort pass, n <= DBX_RF_MAX_INLIST), and the bloom
// insert (one atomicOr per word, eight words per block).  Apply: one thread per probe row, one
// ballot per 32 rows writes the bit-packed result; the IN-lists sit in shared memory.
#include <algorithm>
#include <cmath>
#include <vector>

#include "runtime_filter.cuh"

namespace dbx {

namespace {

constexpr int kRfBlock = 256;

__device__ __forceinline__ uint64_t rf_load(const void* base, int dtype, int64_t row) {
  switch (dtype) {
    case DBX_I64: case DBX_U64: return ((const uint64_t*)base)[row];
    case DBX_I32: return (uint64_t)(int64_t)((const int32_t*)base)[row];
    case DBX_U32: return ((const uint32_t*)base)[row];
    case DBX_I16: return (uint64_t)(int64_t)((const int16_t*)base)[row];
    case DBX_U16: return ((const uint16_t*)base)[row];
    case DBX_I8: return (uint64_t)(int64_t)((const int8_t*)base)[row];
    default: return ((const uint8_t*)base)[row];
  }
}

// out[0] = min image, out[1] = max image (pre-set to the neutral bounds), out[2] = non-NULL rows
__global__ void __launch_bounds__(kRfBlock) rf_min_max_kernel(const void* data, int dtype, const uint8_t* valid_bytes, int64_t n,
                                                              int is_signed, unsigned long long* out) {
  __shared__ uint64_t s_lo[kRfBlock / 32], s_hi[kRfBlock / 32];
  __shared__ unsigned long long s_cnt[kRfBlock / 32];
  uint64_t lo = is_signed ? (uint64_t)INT64_MAX : ~0ULL, hi = is_signed ? (uint64_t)INT64_MIN : 0ULL;
  unsigned long long cnt = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    if (valid_bytes && !valid_bytes[r]) continue;
    const uint64_t v = rf_load(data, dtype, r);
    if (is_signed) { lo = (int64_t)v < (int64_t)lo ? v : lo; hi = (int64_t)v > (int64_t)hi ? v : hi; }
    else { lo = v < lo ? v : lo; hi = v > hi ? v : hi; }
    ++cnt;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint64_t l2 = __shfl_down_sync(0xffffffffu, lo, o), h2 = __shfl_down_sync(0xffffffffu, hi, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    if (is_signed) { lo = (int64_t)l2 < (int64_t)lo ? l2 : lo; hi = (int64_t)h2 > (int64_t)hi ? h2 : hi; }
    else { lo = l2 < lo ? l2 : lo; hi = h2 > hi ? h2 : hi; }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_lo[warp] = lo; s_hi[warp] = hi; s_cnt[warp] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kRfBlock / 32; ++w) {
      if (is_signed) { lo = (int64_t)s_lo[w] < (int64_t)lo ? s_lo[w] : lo; hi = (int64_t)s_hi[w] > (int64_t)hi ? s_hi[w] : hi; }
      else { lo = s_lo[w] < lo ? s_lo[w] : lo; hi = s_hi[w] > hi ? s_hi[w] : hi; }
      cnt += s_cnt[w];
    }
    if (cnt) {
      if (is_signed) { atomicMin((long long*)&out[0], (long long)lo); atomicMax((long long*)&out[1], (long long)hi); }
      else { atomicMin(&out[0], (unsigned long long)lo); atomicMax(&out[1], (unsigned long long)hi); }
      atomicAdd(&out[2], cnt);
    }
  }
}

// The distinct non-NULL keys in ascending order (array_distinct of local_builder.rs:251-274, then
// sorted for the binary search of apply).  One CTA: a key's first occurrence is written at its rank
// among the first occurrences.  *count = distinct keys.
__global__ void __launch_bounds__(1024) rf_inlist_kernel(const void* data, int dtype, const uint8_t* valid_bytes, int n, int is_signed,
                                                         uint64_t* out, unsigned long long* count) {
  extern __shared__ uint64_t s_vals[];
  uint8_t* s_valid = (uint8_t*)(s_vals + n);
  uint8_t* s_first = s_valid + n;
  __shared__ unsigned int s_n;
  if (threadIdx.x == 0) s_n = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    s_valid[i] = valid_bytes ? (valid_bytes[i] != 0) : 1;
    s_vals[i] = rf_load(data, dtype, i);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    bool first = s_valid[i];
    for (int j = 0; j < i && first; ++j) first = !(s_valid[j] && s_vals[j] == s_vals[i]);
    s_first[i] = first;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (!s_first[i]) continue;
    const uint64_t v = s_vals[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) rank += s_first[j] && rf_less(s_vals[j], v, is_signed);
    out[rank] = v;
    atomicAdd(&s_n, 1u);
  }
  __syncthreads();
  if (threadIdx.x == 0) *count = s_n;
}

// Sbbf::insert_hash (sbbf.rs:272-275, BlockAtomic::insert :198-203): one hash per non-NULL build row,
// duplicates included
__global__ void __launch_bounds__(kRfBlock) rf_bloom_insert_kernel(const void* data, int dtype, const uint8_t* valid_bytes, int64_t n,
                                                                   uint64_t mask, uint32_t* words, uint32_t n_blocks) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    if (valid_bytes && !valid_bytes[r]) continue;
    const uint64_t h = rf_fmix64(rf_load(data, dtype, r) & mask);
    uint32_t* blk = words + (size_t)rf_block_index(h, n_blocks) * 8;
    const uint32_t x = (uint32_t)h;
#pragma unroll
    for (int i = 0; i < 8; ++i) atomicOr(blk + i, 1u << ((x * rf_salt(i)) >> 27));
  }
}

struct RfApplyParams {
  RfPartDev parts[DBX_MAX_JOIN_KEYS];
  DevCol keys[DBX_MAX_JOIN_KEYS];
  int32_t inlist_off[DBX_MAX_JOIN_KEYS];  // offset of part i's IN-list in shared memory (values)
  int32_t n_parts;
  int32_t pad;
  int64_t n_rows;
  uint32_t* out;                  // ceil(n_rows / 32) words, LSB first
  unsigned long long* passed;
};

__global__ void __launch_bounds__(kRfBlock) rf_apply_kernel(const __grid_constant__ RfApplyParams p) {
  extern __shared__ uint64_t s_in[];
  for (int i = 0; i < p.n_parts; ++i)
    for (int j = threadIdx.x; j < p.parts[i].n_inlist; j += blockDim.x) s_in[p.inlist_off[i] + j] = p.parts[i].inlist[j];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t n_words = (p.n_rows + 31) / 32;
  const int64_t wstep = (int64_t)gridDim.x * (blockDim.x / 32);
  unsigned long long passed = 0;
  for (int64_t w = (int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); w < n_words; w += wstep) {
    const int64_t r = w * 32 + lane;
    bool pass = r < p.n_rows;
    for (int i = 0; i < p.n_parts && pass; ++i) {
      const DevCol& c = p.keys[i];
      const RfPartDev& f = p.parts[i];
      if (c.validity && !bit_test(c.validity, c.vbit_off + r)) { pass = false; break; }
      const uint64_t v = rf_load(c.data, c.dtype, r);
      pass = rf_min_max_pass(f, v);
      if (pass && f.inlist) {
        const uint64_t* s = s_in + p.inlist_off[i];
        int lo = 0, hi = f.n_inlist;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (rf_less(s[mid], v, f.is_signed)) lo = mid + 1; else hi = mid;
        }
        pass = lo < f.n_inlist && s[lo] == v;
      }
      if (pass) pass = rf_bloom_pass(f, v);
    }
    const unsigned int bits = __ballot_sync(0xffffffffu, pass);
    if (lane == 0) { p.out[w] = bits; passed += __popc(bits); }
  }
  if (lane == 0 && passed) atomicAdd(p.passed, passed);
}

inline int rf_grid(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + kRfBlock - 1) / kRfBlock, (int64_t)kNumSMs * 8)); }

// the pair's common type: the join's key rule (same signedness: the larger size; signed S with
// unsigned U: max(S, 2 U) bytes); signed with UInt64 never gets here (the join refuses it)
void common_key_type(int b, int p, int* dtype, bool* is_signed, uint64_t* mask) {
  const bool bs = dtype_class(b) == VC_INT, ps = dtype_class(p) == VC_INT;
  const int bz = dtype_size(b), pz = dtype_size(p);
  const int bytes = bs == ps ? std::max(bz, pz) : (bs ? std::max(bz, 2 * pz) : std::max(pz, 2 * bz));
  *is_signed = bs || ps;
  static const int kSigned[9] = {0, DBX_I8, DBX_I16, 0, DBX_I32, 0, 0, 0, DBX_I64};
  static const int kUnsigned[9] = {0, DBX_U8, DBX_U16, 0, DBX_U32, 0, 0, 0, DBX_U64};
  *dtype = *is_signed ? kSigned[bytes] : kUnsigned[bytes];
  *mask = bytes == 8 ? ~0ULL : ((1ULL << (8 * bytes)) - 1);
}

// num_of_bits_from_ndv_fpp (sbbf.rs:236-239) with fpp = 0.01, then optimal_num_of_bytes (:225-229):
// the same f64 expression, and Rust's saturating `as usize`
int64_t bloom_bytes_for(uint64_t ndv) {
  const double bits = -8.0 * (double)ndv / std::log(1.0 - std::pow(0.01, 1.0 / 8.0));
  const uint64_t nbits = bits >= 18446744073709551616.0 ? ~0ULL : (bits > 0 ? (uint64_t)bits : 0ULL);
  uint64_t bytes = std::min<uint64_t>(nbits / 8, 128ULL << 20);
  bytes = std::max<uint64_t>(bytes, 32);
  uint64_t p2 = 1;
  while (p2 < bytes) p2 <<= 1;
  return (int64_t)p2;
}

// should_enable_runtime_filter (builder.rs:17-57)
bool bloom_selective(int64_t build_rows, int64_t build_table_rows, uint64_t threshold) {
  if (build_rows <= 0 || build_table_rows <= 0) return false;
  return (double)build_rows / (double)build_table_rows * 100.0 < (double)threshold;
}

struct RfHandle {
  std::shared_ptr<RfData> d;
  cudaStream_t stream = nullptr;
  std::unique_ptr<Stager> stager;
  ErrorSink err;
  DevBuf passed;
  PinnedBuf host;
  int64_t apply_checked = 0, apply_rejected = 0;
  ~RfHandle() {
    if (stream) cudaStreamSynchronize(stream);
    stager.reset();
    if (stream) cudaStreamDestroy(stream);
  }
};

int32_t fail(int32_t st, const std::string& msg) {
  g_create_error.set(msg);
  return st;
}

}  // namespace

int32_t build_runtime_filter(ErrorSink& err, cudaStream_t stream, int device, const dbx_runtime_filter_params& p,
                             const RfBuildKey* keys, int n_keys, int64_t build_rows, std::shared_ptr<RfData>* out) {
  if (p.inlist_threshold < 0 || p.inlist_threshold > DBX_RF_MAX_INLIST) { err.set("runtime filter: inlist_threshold must be 0 .. DBX_RF_MAX_INLIST"); return DBX_ERR_INVALID; }
  if (p.bloom_threshold < 0 || p.build_table_rows < 0) { err.set("runtime filter: negative bloom_threshold or build_table_rows"); return DBX_ERR_INVALID; }
  auto d = std::make_shared<RfData>();
  d->device = device;
  d->n_parts = n_keys;
  d->build_rows = build_rows;
  DBX_CUDA_TRY(err, d->probe_rejected.ensure(8));
  DBX_CUDA_TRY(err, cudaMemsetAsync(d->probe_rejected.p, 0, 8, stream));
  for (int i = 0; i < n_keys; ++i) {
    RfPart& f = d->parts[i];
    common_key_type(keys[i].build_dtype, keys[i].probe_dtype, &f.key_dtype, &f.is_signed, &f.mask);
    f.probe_dtype = keys[i].probe_dtype;
  }
  // a packet with no build rows carries no filters (local_builder.rs:231-233)
  if (build_rows > 0) {
    const bool bloom_on = p.enable_bloom && build_rows <= p.bloom_threshold && bloom_selective(build_rows, p.build_table_rows, p.selectivity_threshold);
    DevBuf scratch;
    DBX_CUDA_TRY(err, scratch.ensure(32));
    unsigned long long* sc = (unsigned long long*)scratch.p;
    PinnedBuf hbuf;
    DBX_CUDA_TRY(err, hbuf.ensure(32));
    unsigned long long* hs = (unsigned long long*)hbuf.p;
    for (int i = 0; i < n_keys; ++i) {
      RfPart& f = d->parts[i];
      const RfBuildKey& k = keys[i];
      hs[0] = f.is_signed ? (unsigned long long)INT64_MAX : ~0ULL;
      hs[1] = f.is_signed ? (unsigned long long)INT64_MIN : 0ULL;
      hs[2] = 0;
      DBX_CUDA_TRY(err, cudaMemcpyAsync(sc, hs, 24, cudaMemcpyHostToDevice, stream));
      rf_min_max_kernel<<<rf_grid(build_rows), kRfBlock, 0, stream>>>(k.data, k.build_dtype, k.valid_bytes, build_rows, f.is_signed, sc);
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      DBX_CUDA_TRY(err, cudaMemcpyAsync(hs, sc, 24, cudaMemcpyDeviceToHost, stream));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
      const uint64_t ndv = hs[2];  // non-NULL build keys: the bloom's ndv
      f.any_key = ndv > 0;
      f.lo = hs[0];
      f.hi = hs[1];
      f.has_min_max = p.enable_min_max && (uint64_t)build_rows <= p.min_max_threshold;
      if (p.enable_inlist && build_rows <= p.inlist_threshold) {
        f.has_inlist = true;
        DBX_CUDA_TRY(err, f.inlist.ensure((size_t)std::max<int64_t>(build_rows, 1) * 8));
        const int n = (int)build_rows;
        const size_t smem = (size_t)n * 10;
        DBX_CUDA_TRY(err, cudaFuncSetAttribute(rf_inlist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 1)));
        rf_inlist_kernel<<<1, 1024, smem, stream>>>(k.data, k.build_dtype, k.valid_bytes, n, f.is_signed, (uint64_t*)f.inlist.p, sc + 3);
        count_launch();
        DBX_CUDA_TRY(err, cudaGetLastError());
        DBX_CUDA_TRY(err, cudaMemcpyAsync(hs + 3, sc + 3, 8, cudaMemcpyDeviceToHost, stream));
        DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
        f.n_inlist = (int64_t)hs[3];
      }
      if (bloom_on) {
        f.has_bloom = true;
        f.bloom_bytes = bloom_bytes_for(ndv);
        DBX_CUDA_TRY(err, f.bloom.ensure((size_t)f.bloom_bytes));
        DBX_CUDA_TRY(err, cudaMemsetAsync(f.bloom.p, 0, (size_t)f.bloom_bytes, stream));
        rf_bloom_insert_kernel<<<rf_grid(build_rows), kRfBlock, 0, stream>>>(k.data, k.build_dtype, k.valid_bytes, build_rows, f.mask,
                                                                             (uint32_t*)f.bloom.p, (uint32_t)(f.bloom_bytes / 32));
        count_launch();
        DBX_CUDA_TRY(err, cudaGetLastError());
      }
    }
  }
  DBX_CUDA_TRY(err, cudaStreamSynchronize(stream));
  *out = std::move(d);
  return DBX_OK;
}

dbx_runtime_filter* make_runtime_filter_handle(std::shared_ptr<RfData> d) {
  auto h = std::make_unique<RfHandle>();
  h->d = std::move(d);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
  h->stager = std::make_unique<Stager>();
  if (h->stager->init(h->d->device, h->stream, &h->err) != DBX_OK) return nullptr;
  if (h->passed.ensure(8) != cudaSuccess) return nullptr;
  if (h->host.ensure(8) != cudaSuccess) return nullptr;
  return reinterpret_cast<dbx_runtime_filter*>(h.release());
}

}  // namespace dbx

using namespace dbx;

extern "C" {

int32_t dbx_runtime_filter_info(dbx_runtime_filter* rf, dbx_rf_info* out) {
  if (!rf || !out) return fail(DBX_ERR_INVALID, "dbx_runtime_filter_info: null argument");
  RfHandle* h = reinterpret_cast<RfHandle*>(rf);
  const RfData& d = *h->d;
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(d.device));
  memset(out, 0, sizeof(*out));
  out->n_parts = d.n_parts;
  out->in_probe = d.in_probe.load() ? 1 : 0;
  out->build_rows = d.build_rows;
  out->apply_rows_checked = h->apply_checked;
  out->apply_rows_rejected = h->apply_rejected;
  out->probe_rows_checked = d.probe_checked.load();
  unsigned long long rej = 0;
  DBX_CUDA_TRY(g_create_error, cudaMemcpy(&rej, d.probe_rejected.p, 8, cudaMemcpyDeviceToHost));
  out->probe_rows_rejected = (int64_t)rej;
  for (int i = 0; i < d.n_parts; ++i) {
    const RfPart& f = d.parts[i];
    dbx_rf_part_info& pi = out->parts[i];
    pi.has_min_max = f.has_min_max;
    pi.has_inlist = f.has_inlist;
    pi.has_bloom = f.has_bloom;
    pi.key_dtype = f.key_dtype;
    pi.min.dtype = pi.max.dtype = f.key_dtype;
    pi.min.is_null = pi.max.is_null = f.any_key ? 0 : 1;
    pi.min.v.u64 = f.any_key ? f.lo : 0;
    pi.max.v.u64 = f.any_key ? f.hi : 0;
    pi.inlist_len = f.n_inlist;
    pi.bloom_bytes = f.bloom_bytes;
  }
  return DBX_OK;
}

int32_t dbx_runtime_filter_export(dbx_runtime_filter* rf, int32_t part, uint32_t* bloom_words, int64_t bloom_cap, int64_t* inlist,
                                  int64_t inlist_cap) {
  if (!rf) return fail(DBX_ERR_INVALID, "dbx_runtime_filter_export: null handle");
  RfHandle* h = reinterpret_cast<RfHandle*>(rf);
  const RfData& d = *h->d;
  if (part < 0 || part >= d.n_parts) return fail(DBX_ERR_INVALID, "dbx_runtime_filter_export: part out of range");
  const RfPart& f = d.parts[part];
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(d.device));
  if (bloom_words && f.has_bloom) {
    if (bloom_cap < f.bloom_bytes / 4) return fail(DBX_ERR_INVALID, "dbx_runtime_filter_export: bloom buffer too small");
    DBX_CUDA_TRY(g_create_error, cudaMemcpy(bloom_words, f.bloom.p, (size_t)f.bloom_bytes, cudaMemcpyDeviceToHost));
  }
  if (inlist && f.has_inlist && f.n_inlist) {
    if (inlist_cap < f.n_inlist) return fail(DBX_ERR_INVALID, "dbx_runtime_filter_export: IN-list buffer too small");
    DBX_CUDA_TRY(g_create_error, cudaMemcpy(inlist, f.inlist.p, (size_t)f.n_inlist * 8, cudaMemcpyDeviceToHost));
  }
  return DBX_OK;
}

int32_t dbx_runtime_filter_apply(dbx_runtime_filter* rf, const dbx_block* block, const int32_t* key_cols, int32_t out_mem, dbx_block* out,
                                 int64_t* n_passed) {
  if (!rf || !block || !key_cols || !out) return fail(DBX_ERR_INVALID, "dbx_runtime_filter_apply: null argument");
  RfHandle* h = reinterpret_cast<RfHandle*>(rf);
  const RfData& d = *h->d;
  DBX_CUDA_TRY(g_create_error, cudaSetDevice(d.device));
  const int64_t n = block->num_rows;
  RfApplyParams ap;
  memset(&ap, 0, sizeof(ap));
  ap.n_parts = d.n_parts;
  ap.n_rows = n;
  int smem_vals = 0;
  for (int i = 0; i < d.n_parts; ++i) {
    const int c = key_cols[i];
    if (c < 0 || c >= block->num_cols) return fail(DBX_ERR_INVALID, "dbx_runtime_filter_apply: key column outside the block");
    const dbx_column& col = block->cols[c];
    if (col.dtype != d.parts[i].probe_dtype || col.len != n || col.is_const)
      return fail(DBX_ERR_INVALID, "dbx_runtime_filter_apply: key column must be a non-const column of the join's probe key dtype");
    ap.parts[i] = d.parts[i].dev();
    ap.inlist_off[i] = smem_vals;
    smem_vals += ap.parts[i].inlist ? ap.parts[i].n_inlist : 0;
  }
  int32_t st = h->stager->begin();
  for (int i = 0; i < d.n_parts && st == DBX_OK; ++i) st = h->stager->stage(block->cols[key_cols[i]], i, &ap.keys[i]);
  if (st != DBX_OK) return fail(st, h->err.msg);
  auto ob = std::make_unique<OwnedBlock>();
  ob->device = d.device;
  ob->stream = h->stream;
  const int64_t n_words = (n + 31) / 32;
  void* words = nullptr;
  DBX_CUDA_TRY(g_create_error, pool_alloc(d.device, h->stream, (size_t)std::max<int64_t>(n_words, 1) * 4, &words));
  ob->dev_allocs.push_back(words);
  ap.out = (uint32_t*)words;
  ap.passed = (unsigned long long*)h->passed.p;
  DBX_CUDA_TRY(g_create_error, cudaMemsetAsync(h->passed.p, 0, 8, h->stream));
  if (n_words) {
    const size_t smem = (size_t)smem_vals * 8;
    if (smem > 48 * 1024)
      DBX_CUDA_TRY(g_create_error, cudaFuncSetAttribute(rf_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_words + kRfBlock / 32 - 1) / (kRfBlock / 32), (int64_t)kNumSMs * 8));
    rf_apply_kernel<<<grid, kRfBlock, smem, h->stream>>>(ap);
    count_launch();
    DBX_CUDA_TRY(g_create_error, cudaGetLastError());
  }
  DBX_CUDA_TRY(g_create_error, cudaMemcpyAsync(h->host.p, h->passed.p, 8, cudaMemcpyDeviceToHost, h->stream));
  st = h->stager->end();
  if (st != DBX_OK) return fail(st, h->err.msg);
  DBX_CUDA_TRY(g_create_error, cudaStreamSynchronize(h->stream));
  const int64_t passed = (int64_t)*(unsigned long long*)h->host.p;
  h->apply_checked += n;
  h->apply_rejected += n - passed;
  if (n_passed) *n_passed = passed;
  dbx_column oc;
  memset(&oc, 0, sizeof(oc));
  oc.dtype = DBX_BOOL; oc.mem = DBX_MEM_DEVICE; oc.data = words; oc.len = n; oc.null_count = 0;
  ob->cols.push_back(oc);
  st = pull_owned_block(ob, d.device, h->stream, h->err, out_mem, out);
  if (st != DBX_OK) return fail(st, h->err.msg);
  return DBX_OK;
}

int32_t dbx_runtime_filter_destroy(dbx_runtime_filter* rf) {
  if (!rf) return DBX_OK;
  RfHandle* h = reinterpret_cast<RfHandle*>(rf);
  cudaSetDevice(h->d->device);
  delete h;
  return DBX_OK;
}

}  // extern "C"
