// knn.cu — dbx_eval_distance (row-wise cosine_distance / l2_distance) and dbx_knn_* (brute-force
// `ORDER BY distance(c, q) LIMIT k` for a batch of queries).
//
// Reference replaced (paths relative to the databend source tree):
//   cosine_distance / l2_distance            src/common/vector/src/distance.rs:19-35,65-80
//   calculate_distance (row-wise driver)     src/query/functions/src/scalars/vector.rs:497-556
//   EvalScalar -> TopN pipeline (SURVEY 3.5) blocks/block_operator.rs:90-98 + top_n/*.rs
//
// kNN plan (one call = one batch of queries):
//   1. corpus: bf16 copy + per-row scale, made once at dbx_knn_create and kept in HBM next to
//      the f32 corpus;
//   2. similarity GEMM on tensor cores in passes of geometrically growing corpus ranges; the
//      epilogue keeps only entries that beat the per-query boundary (k'-th best so far, k' = 8k
//      rounded up to 64), exactly like the top-k operator's boundary filter;
//   3. between passes the candidate list is cut back to k' per query (radix sort by
//      (query, similarity)), which tightens the boundaries;
//   4. the surviving k' candidates per query are re-evaluated EXACTLY in f32 with the reference's
//      evaluation order and sorted by (distance, row id): returned distances are bit-identical to
//      the row-wise function, the bf16 GEMM only decides which rows get that far.
// A Vector(Int8) corpus takes the same plan with an int8 operand (no bf16 copy) and the s8 wgmma:
// its dot products and norms are exact integers, so the only error left between the GEMM's score
// and the reference distance is the f32 evaluation of the score itself.
#include <cuda.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <limits>
#include <vector>

#include "knn_kernels.cuh"
#include "radix_sort.cuh"
#include "runtime.h"

namespace dbx {

namespace {

inline int grid_1d(int64_t n, int block = 256) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + block - 1) / block, (int64_t)kNumSMs * 16));
}
inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// per query: [start, end) of its run in the sorted candidate keys
// (n_dev != nullptr: the candidate count lives on the device — no host sync in front of the cut)
__global__ void seg_bounds_kernel(const uint64_t* keys, int64_t n_host, const unsigned long long* n_dev, int nq, int64_t* seg) {
  const int64_t n = n_dev ? (int64_t)*n_dev : n_host;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q <= nq; q += gridDim.x * blockDim.x) {
    const uint64_t target = (uint64_t)q << 32;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      int64_t mid = (lo + hi) >> 1;
      if (keys[mid] < target) lo = mid + 1; else hi = mid;
    }
    seg[q] = lo;
  }
}
// keep the best k' of every query: compact them to the front (query after query) and publish the
// new boundary (similarity of the k'-th, or -inf while a query has fewer than k' candidates).
// Step 1 (one block): exclusive scan of min(len, k') over the queries -> off[q], total.
__global__ void retain_scan_kernel(const int64_t* seg, int nq, int kprime, int64_t* off, unsigned long long* out_count) {
  __shared__ int64_t s_warp[32];
  __shared__ int64_t s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int q0 = 0; q0 < nq; q0 += blockDim.x) {
    const int q = q0 + threadIdx.x;
    const int64_t len = q < nq ? min((int64_t)kprime, seg[q + 1] - seg[q]) : 0;
    int64_t incl = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int64_t w = lane < (int)(blockDim.x >> 5) ? s_warp[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t up = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += up;
      }
      s_warp[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const int64_t base = s_carry + (warp ? s_warp[warp - 1] : 0);
    if (q < nq) off[q] = base + incl - len;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = base + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) { off[nq] = s_carry; *out_count = (unsigned long long)s_carry; }
}
// Step 2: one warp per query copies its survivors and writes the boundary.
__global__ void retain_copy_kernel(const uint64_t* keys, const uint32_t* rows, const int64_t* seg, const int64_t* off, int nq, int kprime,
                                   uint64_t* out_keys, uint32_t* out_rows, float* bound) {
  const int lane = threadIdx.x & 31;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nq; q += n_warps) {
    const int64_t src = seg[q], dst = off[q];
    const int len = (int)(off[q + 1] - dst);
    for (int j = lane; j < len; j += 32) { out_keys[dst + j] = keys[src + j]; out_rows[dst + j] = rows[src + j]; }
    if (lane == 0) {
      float b = -INFINITY;
      if (len == kprime) {
        const uint32_t o = ~(uint32_t)(keys[src + len - 1] & 0xFFFFFFFFu);
        const uint32_t bits = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
        b = __uint_as_float(bits);
      }
      bound[q] = b;
    }
  }
}
// exact f32 distance of every retained (query, row) pair
__device__ __forceinline__ uint32_t dist_to_ordered32(float d) {  // OrderedFloat: NaN last, -0 == +0
  if (d != d) return 0xFFFFFFFFu;
  if (d == 0.0f) return 0x80000000u;
  const uint32_t b = __float_as_uint(d);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
template <typename T>
__global__ void rerank_kernel(int kind, const T* queries, const T* corpus, int dim, const uint64_t* keys,
                              const uint32_t* rows, int64_t n, uint64_t* out_keys, float* out_dist) {
  if (kind == DBX_DIST_COSINE) {
    const int lane = threadIdx.x & 31, g = lane >> 3;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t base = warp * 4; base < n; base += n_warps * 4) {
      const int64_t i = base + g < n ? base + g : n - 1;
      const uint32_t q = (uint32_t)(keys[i] >> 32);
      const float d = exact_cosine_g8(corpus + (int64_t)rows[i] * dim, queries + (int64_t)q * dim, dim, lane);
      if (base + g < n && (lane & 7) == 0) {
        out_dist[i] = d;
        out_keys[i] = ((uint64_t)q << 32) | dist_to_ordered32(d);
      }
    }
    return;
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t q = (uint32_t)(keys[i] >> 32);
    const float d = exact_l2(corpus + (int64_t)rows[i] * dim, queries + (int64_t)q * dim, dim);
    out_dist[i] = d;
    out_keys[i] = ((uint64_t)q << 32) | dist_to_ordered32(d);  // ascending distance, NaN last (OrderedFloat)
  }
}
// Certificate of exactness.  Every corpus row that is NOT among a query's candidates has an
// approximate similarity <= bound[q] (it was filtered against a boundary that only rises, or cut
// below the k'-th best).  If E bounds (exact similarity - approximate similarity) plus the f32
// error of the distance the ranking uses, and the k-th returned row beats bound + E, the candidate
// set provably held the exact top k; otherwise the query is re-done on the exact path.
//
// Error budget (u = 2^-8 for bf16 round-to-nearest-even, f32 unit 2^-24, n = dim):
//  * bf16 operands: RNE moves a value by at most u/(1+u) of itself, either way, so a product
//    moves by at most (1 + u/(1+u))^2 - 1 = 0.0077972 of |q_i c_i| (a product of two values
//    rounded up; two values rounded down give 1 - (1+u)^-2 = 0.0077670), and by Cauchy-Schwarz
//    the dot product by 0.0077972 |q||c|;
//  * the f32 accumulation inside wgmma (bf16 products are exact in f32): the tensor core's adder
//    is NOT assumed to round to nearest.  The budget assumes each product enters the accumulator
//    truncated by less than one f32 ulp of the running magnitude and each accumulate truncates
//    once more, i.e. at most 2 n 2^-23 sum|q^_i c^_i| <= 2 n 2^-23 * 1.008 |q||c|;
//  * normalisation (cosine, prep_rows_kernel): rsqrtf (2 ulp), the lane-strided f32 sum of
//    squares (n/32 + 6 roundings) and the scaling multiply, both operands:
//    2^-21 + (n/32 + 8) 2^-24;
//  * the f32 distance the ranking uses (exact_cosine_g8: chains of n/8 + 13 roundings for ab, aa,
//    bb, then sqrt, mul, div, sub): 2 (n/8 + 13) 2^-24 + 4 2^-24; exact_l2: n + 3 roundings of
//    non-negative terms, i.e. a relative error of the squared distance below (n + 16) 2^-23;
//  * 32 2^-24 (cosine) / n 2^-120 (L2, absolute) for the f32 compare and subnormal flushes.
// The constants are computed for the corpus's dim on the host (certificate_constants).  The budget
// holds for rows whose squared norms are in range (prep_rows_kernel): a query out of range, or a
// corpus with a row out of range that is not NaN for every query, is answered exactly.
//
// Int8 corpora (s8 wgmma, exact int32 accumulators, prep_rows_i8_kernel, i8_score): the bf16,
// accumulator and normalisation terms are gone — ab, |q|^2 and |c|^2 are exact integers.  Left:
//  * cosine: the score (f32(ab) * 1/|q|) * 1/|c| — f32(ab) 2^-24, each reciprocal norm from an
//    f32-rounded sum, an f32 sqrt and an f32 division <= 2.5 2^-24, two multiplies 2 2^-24 —
//    is within 8 2^-24 of the similarity (|similarity| <= 1); the budget takes 16 2^-24, plus the
//    reference's f32 evaluation (`exact` above) and the 32 2^-24 compare term;
//  * L2: the score -S is exact before its one rounding to f32, 2^-24 S <= 2^-23 (|q|^2 + |c|^2);
//    |q|^2 and cmax^2 in the certificate are themselves f32-rounded (a few 2^-24), and so is the
//    compare: l2_norms = 2^-21 covers all of it, l2_cross = 0; l2_rel and l2_floor as above.
// int8 has no inf or NaN, so no row is outside the range (corpus_unsafe = 0); zero rows are NaN
// for every query under cosine and harmless, as above.  Every term stays strictly positive even
// where the score is exact: with int8 data exact ties in distance are ordinary (duplicate rows, or
// distinct integer similarities that round to one f32 distance), the cut keeps tied rows in an
// arbitrary order, and only a positive margin sends a tie at the boundary to the exact path instead
// of returning a higher row id.
struct KnnCertificate {
  float cos_margin;  // cosine: certified iff 1 - d_k >= bound + cos_margin
  float l2_cross;    // L2: e = l2_cross |q| cmax + l2_norms (|q|^2 + cmax^2) + l2_floor (1 + |q|)
  float l2_norms;
  float l2_floor;
  float l2_rel;      // L2: certified iff d_k^2 (1 + l2_rel) < -bound - e
  int corpus_unsafe;
};
__global__ void certify_kernel(int kind, int nq, int k, int kk, const int64_t* seg, const float* bound, const float* q_scale,
                               const unsigned int* max_norm_bits, const float* out_dist, KnnCertificate cert, uint8_t* flags) {
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
    const int64_t m = seg[q + 1] - seg[q];
    const float qs = q_scale[q];  // cosine: 1/|q|, L2: |q|^2
    const bool q_in_range = kind == DBX_DIST_COSINE ? (qs >= 8.8817842e-16f && qs <= 1.1258999e15f)  // 1/|q| in [2^-50, 2^50]
                                                    : qs <= kCertNormHi;
    bool ok;
    if (m < kk) ok = false;
    else if (kk == 0) ok = true;
    else if (cert.corpus_unsafe || !q_in_range) ok = false;
    else if (bound[q] == -INFINITY) ok = true;  // every row with a non-NaN similarity is a candidate
    else {
      const float dk = out_dist[(int64_t)q * k + kk - 1];
      if (kind == DBX_DIST_COSINE) {
        ok = (1.0f - dk) >= bound[q] + cert.cos_margin;
      } else {
        const float nq_ = sqrtf(qs), cmax = __uint_as_float(*max_norm_bits);
        const float e = cert.l2_cross * nq_ * cmax + cert.l2_norms * (qs + cmax * cmax) + cert.l2_floor * (1.0f + nq_);
        ok = dk * dk * (1.0f + cert.l2_rel) < -bound[q] - e;
      }
    }
    flags[q] = ok ? 0 : 1;
  }
}
KnnCertificate certificate_constants(int kind, int dim, int corpus_unsafe, bool int8) {
  const double n = dim, f32 = std::ldexp(1.0, -24), u = std::ldexp(1.0, -8);
  const double bf16 = (1.0 + u / (1.0 + u)) * (1.0 + u / (1.0 + u)) - 1.0;  // 0.0077972
  const double acc = 2.0 * n * std::ldexp(1.0, -23) * 1.008;
  KnnCertificate c;
  memset(&c, 0, sizeof(c));
  c.corpus_unsafe = corpus_unsafe;
  if (int8) {
    if (kind == DBX_DIST_COSINE) {
      const double exact = (2.0 * (n / 8 + 13) + 4) * f32;
      c.cos_margin = (float)(16 * f32 + exact + 32 * f32);
    } else {
      c.l2_norms = (float)std::ldexp(1.0, -21);
      c.l2_floor = (float)(n * std::ldexp(1.0, -120));
      c.l2_rel = (float)((n + 16) * std::ldexp(1.0, -23));
    }
    return c;
  }
  if (kind == DBX_DIST_COSINE) {
    const double norm = std::ldexp(1.0, -21) + (n / 32 + 8) * f32;
    const double exact = (2.0 * (n / 8 + 13) + 4) * f32;
    c.cos_margin = (float)(bf16 + acc + norm + exact + 32 * f32);
  } else {
    // cmax and |q| come from the same f32 sums of squares: (n/32 + 8) 2^-24 relative covers them
    const double norm_rel = (n / 32 + 8) * f32;
    c.l2_cross = (float)((2.0 * (bf16 + acc) + std::ldexp(1.0, -21)) * (1.0 + 2.0 * norm_rel));
    c.l2_norms = (float)(norm_rel + std::ldexp(1.0, -23));
    c.l2_floor = (float)(n * std::ldexp(1.0, -120));
    c.l2_rel = (float)((n + 16) * std::ldexp(1.0, -23));
  }
  return c;
}
// exact path: keys of one query's distances to every corpus row
// After a similarity pass without a host check: a pass that appended more than the list holds is
// dropped on the device (count back to what it was) and flagged; the host sees the flag at the
// end of the search and repeats the search with per-pass checks.
__global__ void knn_post_pass_kernel(unsigned long long* count, const unsigned long long* prev, long long cap, unsigned long long* overflow) {
  if (threadIdx.x == 0 && (long long)*count > cap) { *count = *prev; *overflow = 1; }
}
// Per-query cut (per-query candidate lists): ONE CTA per query keeps the k' best of its list —
// radix select on the 32-bit key image in shared memory — compacts them to the front of the list
// and tightens the query's boundary to the k'-th best score.  Replaces sort + segment search +
// scan + copy of the shared-list cut with one launch.
__global__ void __launch_bounds__(256) knn_cut_perq_kernel(uint64_t* cand_key, uint32_t* cand_row, unsigned int* qcount, int qcap, int kprime,
                                                           float* bound) {
  extern __shared__ __align__(16) uint32_t s_dyn[];
  uint32_t* s_k = s_dyn;          // [qcap] low 32 key bits: ~ordered(score), smaller = better
  uint32_t* s_r = s_dyn + qcap;   // [qcap] corpus rows
  __shared__ unsigned int s_hist[256];
  __shared__ unsigned int s_pick[3];
  __shared__ unsigned int s_out, s_max;
  const int q = blockIdx.x, tid = threadIdx.x;
  const unsigned int cnt = qcount[q];
  const int n = (int)(cnt < (unsigned)qcap ? cnt : (unsigned)qcap);
  if (n < kprime) return;  // fewer than k' candidates so far: nothing to cut, the boundary stays
  uint64_t* kq = cand_key + (size_t)q * qcap;
  uint32_t* rq = cand_row + (size_t)q * qcap;
  for (int i = tid; i < n; i += 256) { s_k[i] = (uint32_t)kq[i]; s_r[i] = rq[i]; }
  if (tid == 0) { s_out = 0; s_max = 0; }
  __syncthreads();
  uint32_t th = 0xFFFFFFFFu;  // keep key <= th
  if (n > kprime) {
    uint32_t prefix = 0;
    int k_rem = kprime;
    bool closed = false;
    for (int p = 0; p < 4 && !closed; ++p) {
      s_hist[tid] = 0;
      __syncthreads();
      const int sh = 24 - 8 * p;
      for (int i = tid; i < n; i += 256) {
        const uint32_t key = s_k[i];
        if (p == 0 || (key >> (sh + 8)) == (prefix >> (sh + 8))) atomicAdd(&s_hist[(key >> sh) & 255], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        unsigned int cum = 0;
        int b = 0;
        for (; b < 255; ++b) {
          if ((int)(cum + s_hist[b]) >= k_rem) break;
          cum += s_hist[b];
        }
        s_pick[0] = (unsigned)b; s_pick[1] = cum; s_pick[2] = s_hist[b];
      }
      __syncthreads();
      prefix |= s_pick[0] << sh;
      k_rem -= (int)s_pick[1];
      if ((int)s_pick[2] == k_rem) { prefix |= sh ? ((1u << sh) - 1) : 0u; closed = true; }
      __syncthreads();
    }
    th = prefix;
  }
  // entries strictly better than the threshold always fit; ties at the threshold fill what is left
  for (int i = tid; i < n; i += 256) {
    const uint32_t key = s_k[i];
    if (key < th || (key == th && n <= kprime)) {
      const unsigned int pos = atomicAdd(&s_out, 1u);
      kq[pos] = ((uint64_t)(uint32_t)q << 32) | key;
      rq[pos] = s_r[i];
      atomicMax(&s_max, key);
    }
  }
  __syncthreads();
  if (n > kprime) {
    for (int i = tid; i < n; i += 256) {
      const uint32_t key = s_k[i];
      if (key == th) {
        const unsigned int pos = atomicAdd(&s_out, 1u);
        if ((int)pos < kprime) {
          kq[pos] = ((uint64_t)(uint32_t)q << 32) | key;
          rq[pos] = s_r[i];
          atomicMax(&s_max, key);
        }
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    const unsigned int kept = s_out < (unsigned)kprime ? s_out : (unsigned)kprime;
    qcount[q] = kept;
    if ((int)kept == kprime) {  // the k'-th best score so far
      const uint32_t o = ~s_max;
      const uint32_t bits = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
      bound[q] = __uint_as_float(bits);
    }
  }
}
// Shared candidate list (what the similarity GEMM's epilogue appends to, in coalesced bursts) ->
// per-query lists: every candidate goes to the list of its query (warp-aggregated reservation:
// consecutive candidates mostly share their query).  Keeps the hot GEMM epilogue untouched and
// still lets ONE kernel per pass do the cut.
__global__ void __launch_bounds__(256) perq_distribute_kernel(const uint64_t* keys, const uint32_t* rows, const unsigned long long* n_dev, long long cap,
                                                              unsigned int* qcount, int qcap, uint64_t* q_keys, uint32_t* q_rows,
                                                              unsigned long long* overflow) {
  const long long cnt = (long long)*n_dev;
  if (cnt > cap) { if (blockIdx.x == 0 && threadIdx.x == 0) *overflow = 1; }  // the shared list itself overflowed in this pass
  const long long n = cnt < cap ? cnt : cap;
  const int lane = threadIdx.x & 31;
  for (long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) - lane; i0 < n; i0 += (long long)gridDim.x * blockDim.x) {
    const long long i = i0 + lane;
    const bool in = i < n;
    const uint64_t key = in ? keys[i] : 0;
    const uint32_t q = (uint32_t)(key >> 32);
    const unsigned peers = __match_any_sync(0xffffffffu, in ? q : 0xFFFFFFFFu - (uint32_t)lane);
    const int leader = __ffs(peers) - 1;
    unsigned int base = 0;
    if (in && lane == leader) base = atomicAdd(qcount + q, (unsigned int)__popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (in) {
      const unsigned int pos = base + __popc(peers & ((1u << lane) - 1));
      if ((int)pos < qcap) {
        q_keys[(size_t)q * qcap + pos] = key;
        q_rows[(size_t)q * qcap + pos] = rows[i];
      } else {
        *overflow = 1;  // never silently: the host repeats the search in checked mode
      }
    }
  }
}
// per-query lists -> one flat list for the re-rank: prefix over min(count, k') (one CTA), then copy
__global__ void __launch_bounds__(1024) perq_offsets_kernel(const unsigned int* qcount, int nq, int kprime, int64_t* off, unsigned long long* out_count) {
  __shared__ int64_t s_warp[32];
  __shared__ int64_t s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int q0 = 0; q0 < nq; q0 += 1024) {
    const int q = q0 + threadIdx.x;
    const int64_t len = q < nq ? (int64_t)(qcount[q] < (unsigned)kprime ? qcount[q] : (unsigned)kprime) : 0;
    int64_t incl = len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int64_t w = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t up = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += up;
      }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int64_t base = s_carry + (warp ? s_warp[warp - 1] : 0);
    if (q < nq) off[q] = base + incl - len;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = base + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) { off[nq] = s_carry; *out_count = (unsigned long long)s_carry; }
}
__global__ void perq_flatten_kernel(const uint64_t* keys, const uint32_t* rows, int qcap, const int64_t* off, int nq, uint64_t* out_keys, uint32_t* out_rows) {
  const int lane = threadIdx.x & 31;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; q < nq; q += n_warps) {
    const int64_t dst = off[q];
    const int len = (int)(off[q + 1] - dst);
    for (int j = lane; j < len; j += 32) { out_keys[dst + j] = keys[(size_t)q * qcap + j]; out_rows[dst + j] = rows[(size_t)q * qcap + j]; }
  }
}
__global__ void exact_keys_kernel(const float* dist, int64_t n, uint64_t* keys, uint32_t* rows) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = dist_to_ordered32(dist[i]);
    rows[i] = (uint32_t)i;
  }
}
__global__ void exact_emit_kernel(const uint32_t* sorted_rows, const float* dist, int kk, int k, int64_t* out_idx, float* out_dist) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < kk) { out_idx[j] = (int64_t)sorted_rows[j]; out_dist[j] = dist[sorted_rows[j]]; }
  else if (j < k) { out_idx[j] = -1; out_dist[j] = nanf(""); }
}
__global__ void fill_f32_kernel(float* p, int64_t n, float v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void iota32_kernel(uint32_t* p, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = (uint32_t)i;
}
__global__ void widen_u32_kernel(const uint32_t* src, uint64_t* dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[i];
}
__global__ void gather_key_kernel(const uint64_t* src, const uint32_t* idx, uint64_t* dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}
__global__ void emit_topk_kernel(const uint64_t* sorted_keys, const uint32_t* perm, const uint32_t* rows, const float* dist,
                                 const int64_t* seg, int nq, int k, int64_t* out_idx, float* out_dist) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nq * k; i += gridDim.x * blockDim.x) {
    const int q = i / k, j = i % k;
    const int64_t s = seg[q] + j;
    if (s < seg[q + 1]) {
      const uint32_t src = perm[s];
      out_idx[i] = (int64_t)rows[src];
      out_dist[i] = dist[src];
    } else {
      out_idx[i] = -1;
      out_dist[i] = nanf("");
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}
// bf16 / int8 matrix [rows, dim_pad] row-major, box = [one 128-byte k-block, box_rows], 128-byte
// swizzle.  int8 is described as UINT8 (there is no signed 8-bit tensor-map type; TMA moves bytes).
bool make_tmap(CUtensorMap* m, const void* base, int64_t rows, int dim_pad, int box_rows, bool int8) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return false;
  const int es = int8 ? 1 : 2;
  cuuint64_t dims[2] = {(cuuint64_t)dim_pad, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)dim_pad * es};
  cuuint32_t box[2] = {(cuuint32_t)(kKBlockBytes / es), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, int8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

}  // namespace dbx

using namespace dbx;

struct dbx_knn {
  ErrorSink err;
  int device = 0;
  int kind = 0;
  bool int8 = false;  // Vector(Int8) corpus: int8 operands, s8 wgmma; else Vector(Float32), bf16 operands
  int dim = 0, dim_pad = 0;
  int64_t n = 0;
  cudaStream_t stream = nullptr;
  const void* corpus = nullptr;  // f32 / i8 [n, dim] in HBM (borrowed if the caller passed device memory)
  DevBuf corpus_own, corpus_op, c_scale, c_sq;  // corpus_op: the GEMM operand (bf16 or int8, [n + 128, dim_pad])
  // per-search scratch (grow-only)
  DevBuf q_raw, q_op, q_scale, q_sq, bound, seg, seg_off, cand_key[2], cand_row[2], counters, perm[2], key_tmp, sort_alt, dist, qcount;
  DevBuf out_idx_dev, out_dist_dev, max_norm, flags, ex_dist, ex_key[2], ex_row[2], ex_tmp;
  PinnedBuf host, host_flags;
  int corpus_unsafe = 0;  // rows outside the certificate's norm range (prep_rows_kernel)
  int64_t stat_certified = 0, stat_exact = 0, stat_candidates = 0, stat_passes = 0, stat_cluster = 0, stat_grid = 0, stat_us_passes = 0, stat_us_rerank = 0;
  int64_t cand_cap = 0;
  int64_t last_gemm_launches = 0;
  float last_gemm_ms = 0.f;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  RadixSorter sorter;
  std::vector<cudaEvent_t> pass_ev;  // event pairs around the similarity passes of one search
  ~dbx_knn() { for (cudaEvent_t e : pass_ev) cudaEventDestroy(e); }
};

// Launch plumbing of the similarity GEMM for a cluster size C in {1,2,4,8} and operand type T.
template <int C, typename T>
static int32_t gemm_prepare_t(ErrorSink& err, int* max_clusters) {
  static int cached = -1;
  if (cached < 0) {
    const int smem = (int)(sizeof(GemmSmem) + 1024);
    DBX_CUDA_TRY(err, cudaFuncSetAttribute(knn_gemm_filter_kernel<C, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int n = kNumSMs / C;
    if (C > 1) {
      cudaLaunchConfig_t cfg;
      memset(&cfg, 0, sizeof(cfg));
      cfg.gridDim = dim3(C * (kNumSMs / C));
      cfg.blockDim = dim3(kGemmThreads);
      cfg.dynamicSmemBytes = smem;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = C; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      int q = 0;
      DBX_CUDA_TRY(err, cudaOccupancyMaxActiveClusters(&q, knn_gemm_filter_kernel<C, T>, &cfg));
      if (q < 1) { err.set("similarity GEMM: no co-resident cluster fits on this device"); return DBX_ERR_CUDA; }
      n = std::min(n, q);
    }
    cached = n;
  }
  *max_clusters = cached;
  return DBX_OK;
}
template <int C, typename T>
static int32_t gemm_launch_t(ErrorSink& err, int n_clusters, cudaStream_t st, const CUtensorMap& tq, const CUtensorMap& tc, const KnnGemmParams& gp) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(n_clusters * C);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = sizeof(GemmSmem) + 1024;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = C; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  DBX_CUDA_TRY(err, cudaLaunchKernelEx(&cfg, knn_gemm_filter_kernel<C, T>, tq, tc, gp));
  return DBX_OK;
}
template <typename T>
static int32_t knn_gemm_prepare_t(ErrorSink& err, int cluster, int* max_clusters) {
  switch (cluster) {
    case 1: return gemm_prepare_t<1, T>(err, max_clusters);
    case 2: return gemm_prepare_t<2, T>(err, max_clusters);
    case 4: return gemm_prepare_t<4, T>(err, max_clusters);
    default: return gemm_prepare_t<8, T>(err, max_clusters);
  }
}
template <typename T>
static int32_t knn_gemm_launch_t(ErrorSink& err, int cluster, int n_clusters, cudaStream_t st, const CUtensorMap& tq, const CUtensorMap& tc,
                                 const KnnGemmParams& gp) {
  switch (cluster) {
    case 1: return gemm_launch_t<1, T>(err, n_clusters, st, tq, tc, gp);
    case 2: return gemm_launch_t<2, T>(err, n_clusters, st, tq, tc, gp);
    case 4: return gemm_launch_t<4, T>(err, n_clusters, st, tq, tc, gp);
    default: return gemm_launch_t<8, T>(err, n_clusters, st, tq, tc, gp);
  }
}
static int32_t knn_gemm_prepare(ErrorSink& err, bool int8, int cluster, int* max_clusters) {
  return int8 ? knn_gemm_prepare_t<int8_t>(err, cluster, max_clusters) : knn_gemm_prepare_t<__nv_bfloat16>(err, cluster, max_clusters);
}
static int32_t knn_gemm_launch(ErrorSink& err, bool int8, int cluster, int n_clusters, cudaStream_t st, const CUtensorMap& tq, const CUtensorMap& tc,
                               const KnnGemmParams& gp) {
  return int8 ? knn_gemm_launch_t<int8_t>(err, cluster, n_clusters, st, tq, tc, gp)
              : knn_gemm_launch_t<__nv_bfloat16>(err, cluster, n_clusters, st, tq, tc, gp);
}

// Exact answer for one query: distance to every corpus row (row-wise kernel, reference evaluation
// order), stable radix sort by the OrderedFloat key (ties keep ascending row id), first k.
static int32_t knn_exact_query(dbx_knn* h, int q, int k, int kk) {
  ErrorSink& err = h->err;
  cudaStream_t st = h->stream;
  const int64_t n = h->n;
  int64_t* oi = (int64_t*)h->out_idx_dev.p + (int64_t)q * k;
  float* od = (float*)h->out_dist_dev.p + (int64_t)q * k;
  int ex_buf = 0;
  if (n > 0) {
    DBX_CUDA_TRY(err, h->ex_dist.ensure((size_t)n * 4));
    for (int i = 0; i < 2; ++i) {
      DBX_CUDA_TRY(err, h->ex_key[i].ensure((size_t)n * 8));
      DBX_CUDA_TRY(err, h->ex_row[i].ensure((size_t)n * 4));
    }
    const int grid = grid_1d(h->kind == DBX_DIST_COSINE ? n * 8 : n, 128);
    if (h->int8)
      distance_rows_kernel<<<grid, 128, 0, st>>>(h->kind, (const int8_t*)h->corpus, 0, (const int8_t*)h->q_raw.p + (int64_t)q * h->dim, 1, n, h->dim,
                                                 nullptr, 0, nullptr, 0, (float*)h->ex_dist.p, nullptr);
    else
      distance_rows_kernel<<<grid, 128, 0, st>>>(h->kind, (const float*)h->corpus, 0, (const float*)h->q_raw.p + (int64_t)q * h->dim, 1, n, h->dim,
                                                 nullptr, 0, nullptr, 0, (float*)h->ex_dist.p, nullptr);
    exact_keys_kernel<<<grid_1d(n), 256, 0, st>>>((const float*)h->ex_dist.p, n, (uint64_t*)h->ex_key[0].p, (uint32_t*)h->ex_row[0].p);
    // stable LSD radix sort on the 32 significant key bits: ties keep ascending row ids
    DBX_TRY(h->sorter.sort(err, st, (uint64_t*)h->ex_key[0].p, (uint64_t*)h->ex_key[1].p, (uint32_t*)h->ex_row[0].p, (uint32_t*)h->ex_row[1].p, n, 0, 32,
                           false, 0, 0, &ex_buf));
    count_launch(3);
  }
  exact_emit_kernel<<<(k + 255) / 256, 256, 0, st>>>((const uint32_t*)h->ex_row[ex_buf].p, (const float*)h->ex_dist.p, kk, k, oi, od);
  count_launch();
  DBX_CUDA_TRY(err, cudaGetLastError());
  return DBX_OK;
}

extern "C" {

const char* dbx_knn_last_error(const dbx_knn* h) { return h ? h->err.msg.c_str() : g_create_error.msg.c_str(); }

int32_t dbx_knn_create(int32_t kind, int32_t device, const dbx_column* corpus, dbx_knn** out) {
  if (!corpus || !out) { g_create_error.set("dbx_knn_create: null argument"); return DBX_ERR_INVALID; }
  *out = nullptr;
  if (kind != DBX_DIST_COSINE && kind != DBX_DIST_L2) { g_create_error.set("dbx_knn_create: unknown distance kind"); return DBX_ERR_INVALID; }
  if ((corpus->dtype != DBX_VEC_F32 && corpus->dtype != DBX_VEC_I8) || corpus->vec_dim <= 0) {
    g_create_error.set("dbx_knn_create: corpus must be a VECTOR(Float32) or VECTOR(Int8) column");
    return DBX_ERR_INVALID;
  }
  if (corpus->dtype == DBX_VEC_I8 && corpus->vec_dim >= 131072) {  // the s8 wgmma's int32 accumulators hold |sum ab| < 2^31
    g_create_error.set("dbx_knn_create: VECTOR(Int8) corpora are limited to dim < 131072");
    return DBX_ERR_UNSUPPORTED;
  }
  if (corpus->validity) { g_create_error.set("dbx_knn_create: NULL vectors in the corpus are not supported yet"); return DBX_ERR_UNSUPPORTED; }
  if (corpus->len >= (1LL << 31)) { g_create_error.set("dbx_knn_create: corpus too large for 32-bit row ids"); return DBX_ERR_UNSUPPORTED; }
  int32_t ndev = 0;
  DBX_TRY(dbx_device_count(&ndev));
  std::unique_ptr<dbx_knn> h(new dbx_knn());
  ErrorSink& err = g_create_error;
  h->device = device; h->kind = kind; h->int8 = corpus->dtype == DBX_VEC_I8; h->dim = corpus->vec_dim; h->n = corpus->len;
  h->dim_pad = round_up(corpus->vec_dim, h->int8 ? kBlockK<int8_t> : kBlockK<__nv_bfloat16>);
  const int es = h->int8 ? 1 : 4, op_es = h->int8 ? 1 : 2;  // bytes per element of the corpus / of the GEMM operand
  DBX_CUDA_TRY(err, cudaSetDevice(device));
  DBX_CUDA_TRY(err, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  DBX_CUDA_TRY(err, cudaEventCreate(&h->ev0));
  DBX_CUDA_TRY(err, cudaEventCreate(&h->ev1));
  const size_t bytes = (size_t)h->n * h->dim * es;
  if (corpus->mem == DBX_MEM_DEVICE) {
    h->corpus = corpus->data;
  } else {
    DBX_CUDA_TRY(err, h->corpus_own.ensure(bytes ? bytes : 4));
    DBX_CUDA_TRY(err, cudaMemcpyAsync(h->corpus_own.p, corpus->data, bytes, cudaMemcpyHostToDevice, h->stream));
    h->corpus = h->corpus_own.p;
  }
  // the operand copy is padded by one GEMM tile of rows so that every TMA box stays inside the tensor
  const int64_t n_alloc = h->n + kGemmBN;
  DBX_CUDA_TRY(err, h->corpus_op.ensure((size_t)n_alloc * h->dim_pad * op_es));
  DBX_CUDA_TRY(err, cudaMemsetAsync(h->corpus_op.p, 0, (size_t)n_alloc * h->dim_pad * op_es, h->stream));
  DBX_CUDA_TRY(err, h->c_scale.ensure((size_t)n_alloc * 4));
  DBX_CUDA_TRY(err, cudaMemsetAsync(h->c_scale.p, 0, (size_t)n_alloc * 4, h->stream));
  if (h->int8) {
    DBX_CUDA_TRY(err, h->c_sq.ensure((size_t)n_alloc * 4));
    DBX_CUDA_TRY(err, cudaMemsetAsync(h->c_sq.p, 0, (size_t)n_alloc * 4, h->stream));
  }
  DBX_CUDA_TRY(err, h->max_norm.ensure(8));  // [0] largest row norm (bits), [1] rows outside the certificate's range
  DBX_CUDA_TRY(err, cudaMemsetAsync(h->max_norm.p, 0, 8, h->stream));
  if (h->n) {
    if (h->int8)
      prep_rows_i8_kernel<<<grid_1d(h->n * 32), 256, 0, h->stream>>>((const int8_t*)h->corpus, h->n, h->dim, h->dim_pad, (int8_t*)h->corpus_op.p,
                                                                   (int32_t*)h->c_sq.p, (float*)h->c_scale.p, kind, (unsigned int*)h->max_norm.p);
    else
      prep_rows_kernel<<<grid_1d(h->n * 32), 256, 0, h->stream>>>((const float*)h->corpus, h->n, h->dim, h->dim_pad, (__nv_bfloat16*)h->corpus_op.p,
                                                                (float*)h->c_scale.p, kind, (unsigned int*)h->max_norm.p,
                                                                (unsigned int*)h->max_norm.p + 1);
    count_launch();
    DBX_CUDA_TRY(err, cudaGetLastError());
  }
  DBX_CUDA_TRY(err, h->counters.ensure(64));
  DBX_CUDA_TRY(err, h->host.ensure(64));
  DBX_CUDA_TRY(err, cudaMemcpyAsync(h->host.p, h->max_norm.p, 8, cudaMemcpyDeviceToHost, h->stream));
  DBX_CUDA_TRY(err, cudaStreamSynchronize(h->stream));
  h->corpus_unsafe = ((const unsigned int*)h->host.p)[1] != 0;
  *out = h.release();
  return DBX_OK;
}

int32_t dbx_knn_destroy(dbx_knn* h) {
  if (!h) return DBX_OK;
  cudaSetDevice(h->device);
  if (h->stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); }
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
  return DBX_OK;
}

int32_t dbx_knn_last_gemm_ms(dbx_knn* h, float* ms, int64_t* launches) {
  if (!h) return DBX_ERR_INVALID;
  if (ms) *ms = h->last_gemm_ms;
  if (launches) *launches = h->last_gemm_launches;
  return DBX_OK;
}

int32_t dbx_knn_search(dbx_knn* h, const dbx_column* queries, int32_t k, int32_t out_mem, int64_t* out_idx, float* out_dist) {
  if (!h) return DBX_ERR_INVALID;
  ErrorSink& err = h->err;
  if (!queries || !out_idx || !out_dist || k <= 0) { err.set("dbx_knn_search: bad argument"); return DBX_ERR_INVALID; }
  if (queries->dtype != (h->int8 ? DBX_VEC_I8 : DBX_VEC_F32)) {
    // the reference would answer 0.0 (or NULL) on every row of a mixed Int8 / Float32 pair
    err.set(h->int8 ? "dbx_knn_search: queries must be VECTOR(Int8) like the corpus" : "dbx_knn_search: queries must be VECTOR(Float32) like the corpus");
    return DBX_ERR_INVALID;
  }
  if (queries->vec_dim != h->dim) { err.set("Vector length not equal: query dimension differs from the corpus"); return DBX_ERR_INVALID; }
  if (queries->validity) { err.set("dbx_knn_search: NULL query vectors are not supported yet"); return DBX_ERR_UNSUPPORTED; }
  if (k > 1024) { err.set("dbx_knn_search: k > 1024 is not supported"); return DBX_ERR_UNSUPPORTED; }
  DBX_CUDA_TRY(err, cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const int nq = (int)queries->len;
  if (nq == 0) return DBX_OK;
  if (nq > 65536) { err.set("dbx_knn_search: more than 65536 queries per batch"); return DBX_ERR_UNSUPPORTED; }
  // cluster size of the similarity GEMM (corpus tile multicast to `cluster` query blocks); must
  // divide the number of 128-query blocks so that no padded query block is computed
  int cluster = 1;
  {
    const int n_mblk = round_up(nq, kGemmBM) / kGemmBM;
    if (n_mblk % 2 == 0) cluster = 2;  // halves the corpus-tile traffic per CTA; larger clusters leave SMs idle
    if (const char* e = getenv("DBX_KNN_CLUSTER")) {
      const int c = atoi(e);
      if (c == 1 || c == 2 || c == 4 || c == 8) cluster = c;
    }
  }
  const int nq_pad = round_up(nq, kGemmBM * cluster);
  const int dim = h->dim, dim_pad = h->dim_pad;
  const int kprime = round_up(std::max(8 * k, 64), 64);

  // ---- queries: f32 / i8 as given (exact re-rank) + GEMM operand (bf16 / int8) + scale
  const int es = h->int8 ? 1 : 4, op_es = h->int8 ? 1 : 2;
  DBX_CUDA_TRY(err, h->q_raw.ensure((size_t)nq_pad * dim * es));
  DBX_CUDA_TRY(err, h->q_op.ensure((size_t)nq_pad * dim_pad * op_es));
  DBX_CUDA_TRY(err, h->q_scale.ensure((size_t)nq_pad * 4));
  DBX_CUDA_TRY(err, h->bound.ensure((size_t)nq_pad * 4));
  DBX_CUDA_TRY(err, h->seg.ensure((size_t)(nq + 2) * 8));
  DBX_CUDA_TRY(err, h->seg_off.ensure((size_t)(nq + 2) * 8));
  DBX_CUDA_TRY(err, cudaMemsetAsync(h->q_raw.p, 0, (size_t)nq_pad * dim * es, st));
  DBX_CUDA_TRY(err, cudaMemcpyAsync(h->q_raw.p, queries->data, (size_t)nq * dim * es,
                                    queries->mem == DBX_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
  if (h->int8) {
    DBX_CUDA_TRY(err, h->q_sq.ensure((size_t)nq_pad * 4));
    prep_rows_i8_kernel<<<grid_1d((int64_t)nq_pad * 32), 256, 0, st>>>((const int8_t*)h->q_raw.p, nq_pad, dim, dim_pad, (int8_t*)h->q_op.p,
                                                                     (int32_t*)h->q_sq.p, (float*)h->q_scale.p, h->kind, nullptr);
  } else {
    prep_rows_kernel<<<grid_1d((int64_t)nq_pad * 32), 256, 0, st>>>((const float*)h->q_raw.p, nq_pad, dim, dim_pad, (__nv_bfloat16*)h->q_op.p,
                                                                  (float*)h->q_scale.p, h->kind, nullptr, nullptr);
  }
  count_launch();

  // ---- candidate storage
  const int64_t want_cap = std::max<int64_t>(1 << 22, 4LL * nq * kprime);
  if (want_cap > h->cand_cap) {
    for (int i = 0; i < 2; ++i) {
      DBX_CUDA_TRY(err, h->cand_key[i].ensure((size_t)want_cap * 8));
      DBX_CUDA_TRY(err, h->cand_row[i].ensure((size_t)want_cap * 4));
      DBX_CUDA_TRY(err, h->perm[i].ensure((size_t)want_cap * 4));
    }
    DBX_CUDA_TRY(err, h->key_tmp.ensure((size_t)want_cap * 8));
    DBX_CUDA_TRY(err, h->sort_alt.ensure((size_t)want_cap * 8));
    DBX_CUDA_TRY(err, h->dist.ensure((size_t)want_cap * 4));
    h->cand_cap = want_cap;
  }
  const int64_t cap = h->cand_cap;
  unsigned long long* d_count = (unsigned long long*)h->counters.p;  // [0] candidates, [1] count before the pass, [2] overflow flag
  unsigned long long* d_prev = d_count + 1;
  unsigned long long* d_over = d_count + 2;
  int cur = 0;           // candidates live in cand_*[cur][0..n_cand)
  int64_t n_cand = 0;

  int q_bits = 1;
  while ((1 << q_bits) < nq) ++q_bits;
  const int key_bits = 32 + q_bits;  // (query << 32) | score: the sorts skip the unused high bits
  int row_bits = 1;
  while (row_bits < 32 && (1LL << row_bits) < h->n) ++row_bits;
  auto t_start = std::chrono::steady_clock::now();
  // Default: NO host synchronisation between the similarity passes — the candidate count stays on
  // the device (the cut's radix sort, segment search and copy read it there), passes grow on a
  // fixed geometric schedule, and a pass that would overflow the candidate list is dropped and
  // flagged on the device; the flag is read once, before the re-rank, and an overflow repeats the
  // search with a host check after every pass (DBX_KNN_SYNC=1 forces that mode).
  bool async_mode = getenv("DBX_KNN_SYNC") == nullptr;
  // per-query candidate lists (the asynchronous mode's layout): capacity per query
  int qcap = (int)std::min<int64_t>(4096, cap / nq_pad / 256 * 256);
  const bool qcap_forced = getenv("DBX_KNN_QCAP") != nullptr;  // tests: a small capacity forces the overflow fallback
  if (qcap_forced) qcap = std::min(qcap, std::max(256, atoi(getenv("DBX_KNN_QCAP")) / 256 * 256));
  bool perq = async_mode && qcap >= 4 * kprime && (qcap >= 1024 || qcap_forced) && !getenv("DBX_KNN_SHARED_LIST");
  unsigned int* d_qcount = nullptr;
  if (perq) {
    DBX_CUDA_TRY(err, h->qcount.ensure((size_t)nq_pad * 4));
    d_qcount = (unsigned int*)h->qcount.p;
    static std::atomic<bool> attr_set[64];
    if (!attr_set[h->device]) {
      DBX_CUDA_TRY(err, cudaFuncSetAttribute(knn_cut_perq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 8));
      attr_set[h->device] = true;
    }
  }
  auto select = [&]() -> int32_t {  // cut every query back to its best k', tighten boundaries
    if (perq) {  // shared list (cand_*[1], filled by the GEMM) -> per-query lists (cand_*[0]) -> one cut kernel
      perq_distribute_kernel<<<kNumSMs * 8, 256, 0, st>>>((const uint64_t*)h->cand_key[1].p, (const uint32_t*)h->cand_row[1].p, d_count, (long long)cap,
                                                          d_qcount, qcap, (uint64_t*)h->cand_key[0].p, (uint32_t*)h->cand_row[0].p, d_over);
      DBX_CUDA_TRY(err, cudaMemsetAsync(d_count, 0, 8, st));
      knn_cut_perq_kernel<<<nq, 256, (size_t)qcap * 8, st>>>((uint64_t*)h->cand_key[0].p, (uint32_t*)h->cand_row[0].p, d_qcount, qcap, kprime,
                                                            (float*)h->bound.p);
      count_launch(2);
      DBX_CUDA_TRY(err, cudaGetLastError());
      return DBX_OK;
    }
    if (!async_mode && n_cand == 0) return DBX_OK;
    const unsigned long long* nd = async_mode ? d_count : nullptr;
    int rb = 0;
    DBX_TRY(h->sorter.sort(err, st, (uint64_t*)h->cand_key[cur].p, (uint64_t*)h->cand_key[cur ^ 1].p, (uint32_t*)h->cand_row[cur].p,
                           (uint32_t*)h->cand_row[cur ^ 1].p, async_mode ? cap : n_cand, 0, key_bits, false, 0, 0, &rb, nd));
    const int src = rb ? (cur ^ 1) : cur, dst = src ^ 1;
    seg_bounds_kernel<<<grid_1d(nq + 1), 256, 0, st>>>((const uint64_t*)h->cand_key[src].p, n_cand, nd, nq, (int64_t*)h->seg.p);
    retain_scan_kernel<<<1, 1024, 0, st>>>((const int64_t*)h->seg.p, nq, kprime, (int64_t*)h->seg_off.p, d_count);
    retain_copy_kernel<<<grid_1d((int64_t)nq * 32), 256, 0, st>>>((const uint64_t*)h->cand_key[src].p, (const uint32_t*)h->cand_row[src].p,
                                                                 (const int64_t*)h->seg.p, (const int64_t*)h->seg_off.p, nq, kprime,
                                                                 (uint64_t*)h->cand_key[dst].p, (uint32_t*)h->cand_row[dst].p, (float*)h->bound.p);
    count_launch(3);
    DBX_CUDA_TRY(err, cudaGetLastError());
    cur = dst;
    if (!async_mode) {
      DBX_CUDA_TRY(err, cudaMemcpyAsync(h->host.p, d_count, 8, cudaMemcpyDeviceToHost, st));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(st));
      n_cand = (int64_t)*(unsigned long long*)h->host.p;
    }
    return DBX_OK;
  };

  // ---- similarity passes over geometrically growing corpus ranges
  CUtensorMap tmap_q, tmap_c;
  const bool use_ref = getenv("DBX_KNN_REF_GEMM") != nullptr;
  int max_clusters = kNumSMs / cluster;
  if (!use_ref) {
    if (!make_tmap(&tmap_q, h->q_op.p, nq_pad, dim_pad, kGemmBM, h->int8) ||
        !make_tmap(&tmap_c, h->corpus_op.p, h->n + kGemmBN, dim_pad, kGemmBN / cluster, h->int8)) {
      err.set("cuTensorMapEncodeTiled failed (TMA descriptors for the similarity GEMM)");
      return DBX_ERR_CUDA;
    }
    DBX_TRY(knn_gemm_prepare(err, h->int8, cluster, &max_clusters));
    h->stat_cluster = cluster; h->stat_grid = (int64_t)max_clusters * cluster;
  }
  for (int attempt = 0; attempt < 2; ++attempt) {
    fill_f32_kernel<<<grid_1d(nq_pad), 256, 0, st>>>((float*)h->bound.p, nq_pad, -std::numeric_limits<float>::infinity());
    count_launch();
    DBX_CUDA_TRY(err, cudaMemsetAsync(d_count, 0, 24, st));
    if (perq) DBX_CUDA_TRY(err, cudaMemsetAsync(d_qcount, 0, (size_t)nq_pad * 4, st));
    cur = 0;
    n_cand = 0;
    h->last_gemm_ms = 0.f;
    h->last_gemm_launches = 0;
    int64_t done = 0;
    size_t n_ev = 0;
    // first pass: small enough that even "everything passes" fits the candidate list
    int64_t chunk = std::max<int64_t>(kGemmBN, std::min<int64_t>((cap / 2) / std::max(nq, 1) / kGemmBN * kGemmBN, 1 << 16));
    if (perq) chunk = std::max<int64_t>(kGemmBN, std::min<int64_t>(chunk, (qcap / 2) / kGemmBN * kGemmBN));  // even "everything passes" fits a query's list
    while (done < h->n) {
      const int64_t m = std::min<int64_t>(chunk, h->n - done);
      KnnGemmParams gp;
      memset(&gp, 0, sizeof(gp));
      gp.kind = h->kind; gp.nq = nq; gp.nq_pad = nq_pad; gp.dim_pad = dim_pad; gp.n0 = done; gp.n_rows = m;
      gp.q_scale = (const float*)h->q_scale.p; gp.c_scale = (const float*)h->c_scale.p; gp.bound = (const float*)h->bound.p;
      gp.cand_key = (uint64_t*)h->cand_key[perq ? 1 : cur].p; gp.cand_row = (uint32_t*)h->cand_row[perq ? 1 : cur].p; gp.cand_count = d_count; gp.cand_cap = cap;
      gp.q_sq = (const int32_t*)h->q_sq.p; gp.c_sq = (const int32_t*)h->c_sq.p;
      cudaEvent_t e0 = h->ev0, e1 = h->ev1;
      if (async_mode) {
        if (!perq) DBX_CUDA_TRY(err, cudaMemcpyAsync(d_prev, d_count, 8, cudaMemcpyDeviceToDevice, st));
        while (h->pass_ev.size() < n_ev + 2) {
          cudaEvent_t e = nullptr;
          DBX_CUDA_TRY(err, cudaEventCreate(&e));
          h->pass_ev.push_back(e);
        }
        e0 = h->pass_ev[n_ev]; e1 = h->pass_ev[n_ev + 1];
        n_ev += 2;
      }
      DBX_CUDA_TRY(err, cudaEventRecord(e0, st));
      if (use_ref && h->int8) {
        knn_ref_filter_i8_kernel<<<grid_1d((int64_t)nq * m), 256, 0, st>>>((const int8_t*)h->q_op.p, (const int8_t*)h->corpus_op.p, gp);
      } else if (use_ref) {
        knn_ref_filter_kernel<<<grid_1d((int64_t)nq * m), 256, 0, st>>>((const __nv_bfloat16*)h->q_op.p, (const __nv_bfloat16*)h->corpus_op.p, gp);
      } else {
        const int64_t tiles = ((m + kGemmBN - 1) / kGemmBN) * (nq_pad / (kGemmBM * cluster));
        const int n_clusters = (int)std::min<int64_t>(tiles, max_clusters);
        DBX_TRY(knn_gemm_launch(err, h->int8, cluster, n_clusters, st, tmap_q, tmap_c, gp));
      }
      count_launch();
      DBX_CUDA_TRY(err, cudaGetLastError());
      DBX_CUDA_TRY(err, cudaEventRecord(e1, st));
      if (async_mode) {
        if (!perq) {
          knn_post_pass_kernel<<<1, 32, 0, st>>>(d_count, d_prev, (long long)cap, d_over);
          count_launch();
        }
        h->last_gemm_launches += 1;
        done += m;
        DBX_TRY(select());
        chunk = std::min<int64_t>(chunk * 8, 1LL << 24);
        continue;
      }
      DBX_CUDA_TRY(err, cudaMemcpyAsync(h->host.p, d_count, 8, cudaMemcpyDeviceToHost, st));
      DBX_CUDA_TRY(err, cudaStreamSynchronize(st));
      float ms = 0.f;
      cudaEventElapsedTime(&ms, e0, e1);
      const int64_t cnt = (int64_t)*(unsigned long long*)h->host.p;
      if (cnt > cap) {  // more survivors than the list holds: drop this pass, tighten, retry smaller
        unsigned long long back = (unsigned long long)n_cand;
        DBX_CUDA_TRY(err, cudaMemcpyAsync(d_count, &back, 8, cudaMemcpyHostToDevice, st));
        DBX_TRY(select());
        if (m <= kGemmBN) { err.set("kNN candidate list too small for one GEMM tile"); return DBX_ERR_CUDA; }
        chunk = std::max<int64_t>(kGemmBN, (m / 4) / kGemmBN * kGemmBN);
        continue;
      }
      h->last_gemm_ms += ms;
      h->last_gemm_launches += 1;
      n_cand = cnt;
      done += m;
      DBX_TRY(select());
      chunk = std::min<int64_t>(chunk * 8, 1LL << 24);
    }
    h->stat_passes = h->last_gemm_launches;
    if (!async_mode) break;
    if (perq) {  // per-query lists -> one flat list (cand_*[1]) for the re-rank
      perq_offsets_kernel<<<1, 1024, 0, st>>>(d_qcount, nq, kprime, (int64_t*)h->seg_off.p, d_count);
      perq_flatten_kernel<<<grid_1d((int64_t)nq * 32), 256, 0, st>>>((const uint64_t*)h->cand_key[0].p, (const uint32_t*)h->cand_row[0].p, qcap,
                                                                    (const int64_t*)h->seg_off.p, nq, (uint64_t*)h->cand_key[1].p, (uint32_t*)h->cand_row[1].p);
      count_launch(2);
      cur = 1;
    }
    // the one host check of the asynchronous mode
    DBX_CUDA_TRY(err, cudaMemcpyAsync(h->host.p, d_count, 24, cudaMemcpyDeviceToHost, st));
    DBX_CUDA_TRY(err, cudaStreamSynchronize(st));
    n_cand = (int64_t)((unsigned long long*)h->host.p)[0];
    for (size_t i = 0; i + 1 < n_ev; i += 2) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, h->pass_ev[i], h->pass_ev[i + 1]);
      h->last_gemm_ms += ms;
    }
    if (((unsigned long long*)h->host.p)[2] == 0) break;
    async_mode = false;  // a pass overflowed a candidate list: once more, shared list, with a host check after every pass
    perq = false;
  }

  auto t_passes = std::chrono::steady_clock::now();
  // ---- exact re-rank of the k' survivors per query, ordered by (distance, row id)
  DBX_CUDA_TRY(err, h->out_idx_dev.ensure((size_t)nq * k * 8));
  DBX_CUDA_TRY(err, h->out_dist_dev.ensure((size_t)nq * k * 4));
  const uint64_t* final_keys = (const uint64_t*)h->key_tmp.p;
  const uint32_t* final_perm = (const uint32_t*)h->perm[0].p;
  if (n_cand > 0) {
    // exact distances, then two stable LSD radix sorts of a permutation: by row id, then by
    // (query, exact distance) -> ties keep ascending row ids
    if (h->int8)
      rerank_kernel<<<grid_1d(n_cand), 256, 0, st>>>(h->kind, (const int8_t*)h->q_raw.p, (const int8_t*)h->corpus, dim, (const uint64_t*)h->cand_key[cur].p,
                                                     (const uint32_t*)h->cand_row[cur].p, n_cand, (uint64_t*)h->key_tmp.p, (float*)h->dist.p);
    else
      rerank_kernel<<<grid_1d(n_cand), 256, 0, st>>>(h->kind, (const float*)h->q_raw.p, (const float*)h->corpus, dim, (const uint64_t*)h->cand_key[cur].p,
                                                     (const uint32_t*)h->cand_row[cur].p, n_cand, (uint64_t*)h->key_tmp.p, (float*)h->dist.p);
    iota32_kernel<<<grid_1d(n_cand), 256, 0, st>>>((uint32_t*)h->perm[0].p, n_cand);
    uint64_t* ka = (uint64_t*)h->cand_key[cur ^ 1].p;
    uint64_t* kb = (uint64_t*)h->sort_alt.p;
    widen_u32_kernel<<<grid_1d(n_cand), 256, 0, st>>>((const uint32_t*)h->cand_row[cur].p, ka, n_cand);
    count_launch(3);
    int rb1 = 0, rb2 = 0;
    DBX_TRY(h->sorter.sort(err, st, ka, kb, (uint32_t*)h->perm[0].p, (uint32_t*)h->perm[1].p, n_cand, 0, row_bits, false, 0, 0, &rb1));
    uint32_t* p_sorted = (uint32_t*)h->perm[rb1].p;
    uint32_t* p_other = (uint32_t*)h->perm[rb1 ^ 1].p;
    gather_key_kernel<<<grid_1d(n_cand), 256, 0, st>>>((const uint64_t*)h->key_tmp.p, p_sorted, ka, n_cand);
    count_launch();
    DBX_TRY(h->sorter.sort(err, st, ka, kb, p_sorted, p_other, n_cand, 0, key_bits, false, 0, 0, &rb2));
    final_keys = rb2 ? kb : ka;
    final_perm = rb2 ? p_other : p_sorted;
    seg_bounds_kernel<<<grid_1d(nq + 1), 256, 0, st>>>(final_keys, n_cand, nullptr, nq, (int64_t*)h->seg.p);
    count_launch();
  } else {
    DBX_CUDA_TRY(err, cudaMemsetAsync(h->seg.p, 0, (size_t)(nq + 2) * 8, st));
  }
  emit_topk_kernel<<<grid_1d((int64_t)nq * k), 256, 0, st>>>(final_keys, final_perm, (const uint32_t*)h->cand_row[cur].p,
                                                            (const float*)h->dist.p, (const int64_t*)h->seg.p, nq, k, (int64_t*)h->out_idx_dev.p,
                                                            (float*)h->out_dist_dev.p);
  count_launch();
  DBX_CUDA_TRY(err, cudaGetLastError());

  // ---- certificate; queries that fail it are answered by the exact path
  const int kk = (int)std::min<int64_t>(k, h->n);
  DBX_CUDA_TRY(err, h->flags.ensure((size_t)nq));
  DBX_CUDA_TRY(err, h->host_flags.ensure((size_t)nq));
  certify_kernel<<<grid_1d(nq), 256, 0, st>>>(h->kind, nq, k, kk, (const int64_t*)h->seg.p, (const float*)h->bound.p, (const float*)h->q_scale.p,
                                             (const unsigned int*)h->max_norm.p, (const float*)h->out_dist_dev.p,
                                             certificate_constants(h->kind, dim, h->corpus_unsafe, h->int8), (uint8_t*)h->flags.p);
  count_launch();
  DBX_CUDA_TRY(err, cudaGetLastError());
  DBX_CUDA_TRY(err, cudaMemcpyAsync(h->host_flags.p, h->flags.p, (size_t)nq, cudaMemcpyDeviceToHost, st));
  DBX_CUDA_TRY(err, cudaStreamSynchronize(st));
  auto t_rerank = std::chrono::steady_clock::now();
  h->stat_us_passes = std::chrono::duration_cast<std::chrono::microseconds>(t_passes - t_start).count();
  h->stat_us_rerank = std::chrono::duration_cast<std::chrono::microseconds>(t_rerank - t_passes).count();
  h->stat_candidates = n_cand;
  h->stat_exact = 0;
  const uint8_t* hf = (const uint8_t*)h->host_flags.p;
  const bool force_exact = getenv("DBX_KNN_FORCE_EXACT") != nullptr;
  for (int q = 0; q < nq; ++q) {
    if (!hf[q] && !force_exact) continue;
    DBX_TRY(knn_exact_query(h, q, k, kk));
    h->stat_exact += 1;
  }
  h->stat_certified = nq - h->stat_exact;

  const cudaMemcpyKind ck = out_mem == DBX_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  DBX_CUDA_TRY(err, cudaMemcpyAsync(out_idx, h->out_idx_dev.p, (size_t)nq * k * 8, ck, st));
  DBX_CUDA_TRY(err, cudaMemcpyAsync(out_dist, h->out_dist_dev.p, (size_t)nq * k * 4, ck, st));
  DBX_CUDA_TRY(err, cudaStreamSynchronize(st));
  return DBX_OK;
}

int32_t dbx_knn_last_stats(dbx_knn* h, int64_t* out8) {
  if (!h || !out8) return DBX_ERR_INVALID;
  memset(out8, 0, 8 * sizeof(int64_t));
  out8[0] = h->stat_certified; out8[1] = h->stat_exact; out8[2] = h->stat_candidates; out8[3] = h->stat_passes; out8[4] = h->stat_cluster; out8[5] = h->stat_grid; out8[6] = h->stat_us_passes; out8[7] = h->stat_us_rerank;
  return DBX_OK;
}

// ScalarFunction::eval for cosine_distance / l2_distance (scalars/vector.rs:263-281,497-556)
int32_t dbx_eval_distance(int32_t kind, int32_t device, const dbx_column* lhs, const dbx_column* rhs, dbx_column* out) {
  ErrorSink& err = g_create_error;
  if (!lhs || !rhs || !out) { err.set("dbx_eval_distance: null argument"); return DBX_ERR_INVALID; }
  if (kind != DBX_DIST_COSINE && kind != DBX_DIST_L2) { err.set("dbx_eval_distance: unknown distance kind"); return DBX_ERR_INVALID; }
  if (!is_vector_dtype(lhs->dtype) || !is_vector_dtype(rhs->dtype)) {
    err.set("dbx_eval_distance: arguments must be VECTOR(Float32) or VECTOR(Int8)");
    return DBX_ERR_INVALID;
  }
  // A Vector(Int8) / Vector(Float32) pair passes the reference's type check (dims are compared only
  // for equal element types, scalars/vector.rs:458-494), then calculate_distance's `(_, _)` arm marks
  // every row invalid and writes 0.0: 0.0 everywhere, NULL everywhere when the result is Nullable.
  const bool mixed = lhs->dtype != rhs->dtype;
  if (!mixed && lhs->vec_dim != rhs->vec_dim) {  // distance.rs:20-26
    err.set("Vector length not equal: " + std::to_string(lhs->vec_dim) + " != " + std::to_string(rhs->vec_dim));
    return DBX_ERR_INVALID;
  }
  const int64_t rows = out->len;
  if ((!lhs->is_const && lhs->len != rows) || (!rhs->is_const && rhs->len != rows)) { err.set("dbx_eval_distance: column lengths differ"); return DBX_ERR_INVALID; }
  if (out->dtype != DBX_F32 || !out->data) { err.set("dbx_eval_distance: out must be a caller-provided Float32 column"); return DBX_ERR_INVALID; }
  int32_t ndev = 0;
  DBX_TRY(dbx_device_count(&ndev));
  DBX_CUDA_TRY(err, cudaSetDevice(device));
  if (rows == 0) return DBX_OK;
  if (mixed) {
    if (out->mem == DBX_MEM_DEVICE) DBX_CUDA_TRY(err, cudaMemset((void*)out->data, 0, (size_t)rows * 4));
    else memset((void*)out->data, 0, (size_t)rows * 4);
    if (out->validity) {
      if (out->mem == DBX_MEM_DEVICE) DBX_CUDA_TRY(err, cudaMemset((void*)out->validity, 0, (size_t)(rows + 7) / 8));
      else memset((void*)out->validity, 0, (size_t)(rows + 7) / 8);
      out->null_count = rows;
      out->validity_bit_offset = 0;
    }
    return DBX_OK;
  }
  const int dim = lhs->vec_dim;
  const int es = lhs->dtype == DBX_VEC_I8 ? 1 : 4;
  // const sides carry their single vector in `data` (len 1)
  DevBuf la, ra, lvb, rvb, ob, ovb, obits;
  auto to_dev = [&](const dbx_column* c, DevBuf& buf, const void** p) -> int32_t {
    const size_t bytes = (size_t)(c->is_const ? 1 : c->len) * dim * es;
    if (c->is_const && (c->konst.is_null || !c->data)) {  // NULL constant: every output row is NULL
      DBX_CUDA_TRY(err, buf.ensure(bytes));
      DBX_CUDA_TRY(err, cudaMemset(buf.p, 0, bytes));
      *p = buf.p;
      return DBX_OK;
    }
    if (c->mem == DBX_MEM_DEVICE) { *p = c->data; return DBX_OK; }
    DBX_CUDA_TRY(err, buf.ensure(bytes));
    DBX_CUDA_TRY(err, cudaMemcpy(buf.p, c->data, bytes, cudaMemcpyHostToDevice));
    *p = buf.p;
    return DBX_OK;
  };
  auto valid_to_dev = [&](const dbx_column* c, DevBuf& buf, const uint8_t** p, int64_t* off) -> int32_t {
    *p = nullptr; *off = 0;
    if (!c->validity || c->is_const) return DBX_OK;
    if (c->mem == DBX_MEM_DEVICE) { *p = c->validity; *off = c->validity_bit_offset; return DBX_OK; }
    const int64_t b0 = c->validity_bit_offset >> 3, b1 = (c->validity_bit_offset + c->len + 7) >> 3;
    DBX_CUDA_TRY(err, buf.ensure((size_t)(b1 - b0) + 1));
    DBX_CUDA_TRY(err, cudaMemcpy(buf.p, c->validity + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice));
    *p = (const uint8_t*)buf.p; *off = c->validity_bit_offset & 7;
    return DBX_OK;
  };
  const void *lp, *rp;
  const uint8_t *lv, *rv;
  int64_t lvo, rvo;
  DBX_TRY(to_dev(lhs, la, &lp));
  DBX_TRY(to_dev(rhs, ra, &rp));
  DBX_TRY(valid_to_dev(lhs, lvb, &lv, &lvo));
  DBX_TRY(valid_to_dev(rhs, rvb, &rv, &rvo));
  const bool const_null = (lhs->is_const && (lhs->konst.is_null || !lhs->data)) || (rhs->is_const && (rhs->konst.is_null || !rhs->data));
  float* op = (float*)out->data;
  if (out->mem != DBX_MEM_DEVICE) { DBX_CUDA_TRY(err, ob.ensure((size_t)rows * 4)); op = (float*)ob.p; }
  uint8_t* ovalid = nullptr;
  const bool want_valid = out->validity != nullptr;
  if (want_valid) { DBX_CUDA_TRY(err, ovb.ensure((size_t)rows)); ovalid = (uint8_t*)ovb.p; }
  if ((lv || rv || const_null) && !want_valid) { err.set("dbx_eval_distance: nullable inputs need out->validity"); return DBX_ERR_INVALID; }
  const int grid = grid_1d(kind == DBX_DIST_COSINE ? rows * 8 : rows, 128);
  if (es == 1)
    distance_rows_kernel<<<grid, 128>>>(kind, (const int8_t*)lp, lhs->is_const, (const int8_t*)rp, rhs->is_const, rows, dim, lv, lvo, rv, rvo, op, ovalid);
  else
    distance_rows_kernel<<<grid, 128>>>(kind, (const float*)lp, lhs->is_const, (const float*)rp, rhs->is_const, rows, dim, lv, lvo, rv, rvo, op, ovalid);
  count_launch();
  DBX_CUDA_TRY(err, cudaGetLastError());
  if (out->mem != DBX_MEM_DEVICE) DBX_CUDA_TRY(err, cudaMemcpy((void*)out->data, op, (size_t)rows * 4, cudaMemcpyDeviceToHost));
  if (want_valid) {
    std::vector<uint8_t> hb((size_t)rows);
    DBX_CUDA_TRY(err, cudaMemcpy(hb.data(), ovalid, (size_t)rows, cudaMemcpyDeviceToHost));
    std::vector<uint8_t> bits((size_t)(rows + 7) / 8, 0);
    int64_t nulls = 0;
    for (int64_t i = 0; i < rows; ++i) {
      bool ok = hb[i] && !const_null;
      if (ok) bits[i >> 3] |= (uint8_t)(1u << (i & 7)); else ++nulls;
    }
    if (out->mem == DBX_MEM_DEVICE) DBX_CUDA_TRY(err, cudaMemcpy((void*)out->validity, bits.data(), bits.size(), cudaMemcpyHostToDevice));
    else memcpy((void*)out->validity, bits.data(), bits.size());
    out->null_count = nulls;
    out->validity_bit_offset = 0;
  }
  DBX_CUDA_TRY(err, cudaDeviceSynchronize());
  return DBX_OK;
}

}  // extern "C"
