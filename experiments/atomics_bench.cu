// experiments/atomics_bench.cu — what does the GPU give for "stream 24 B/row + random L2 atomics"?
// Variants isolate the stream, the probe load and the REDs of the fused filter->hash-agg kernel.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o atomics_bench atomics_bench.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

struct u64x4 { uint64_t x, y, z, w; };
__device__ __forceinline__ u64x4 ld256(const void* p) {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  u64x4 r;  // two 128-bit loads: sm_90a has no 256-bit load
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0,%1}, [%2], %3;" : "=l"(r.x), "=l"(r.y) : "l"(p), "l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.b64 {%0,%1}, [%2], %3;" : "=l"(r.z), "=l"(r.w) : "l"((const char*)p + 16), "l"(pol));
  return r;
}
__device__ __forceinline__ uint64_t mix(uint64_t x) {
  x ^= x >> 32; x *= 0xd6e8feb86659fd93ULL; x ^= x >> 32; x *= 0xd6e8feb86659fd93ULL; x ^= x >> 32; return x;
}
__device__ __forceinline__ void red64(void* p, uint64_t v) { asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void redf64(void* p, double v) { asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ void red32(void* p, uint32_t v) { asm volatile("red.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void redf32x4(void* p, float a, float b, float c, float d) { asm volatile("red.global.v4.f32.add [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory"); }
__device__ __forceinline__ void redf32x2(void* p, float a, float b) { asm volatile("red.global.v2.f32.add [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory"); }
__device__ __forceinline__ uint64_t ldtab(const void* p) { uint64_t r; asm volatile("ld.global.relaxed.gpu.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory"); return r; }

// MODE 0: stream only (sum to keep loads alive)   1: + probe load   2: + 1 RED   3: + 3 REDs same sector (AoS 32B)
// MODE 4: probe + 3 REDs AoS (the real thing, no CAS)  5: 3 REDs SoA   6: stream k only-if-selected (predicated loads)
template <int MODE>
__global__ void __launch_bounds__(256, 4) k(const uint64_t* kc, const int64_t* vc, const double* xc, int64_t n, uint8_t* tab,
                                            uint64_t mask, uint64_t* sink, uint64_t* soa) {
  int64_t tiles = n / 1024;
  uint64_t acc = 0;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    int64_t r0 = t * 1024 + 4 * threadIdx.x;
    u64x4 v = ld256(vc + r0);
    u64x4 kk, xx;
    if (MODE != 6) { kk = ld256(kc + r0); xx = ld256(xc + r0); }
    int64_t vv[4] = {(int64_t)v.x, (int64_t)v.y, (int64_t)v.z, (int64_t)v.w};
    uint32_t sel = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) sel |= (vv[j] % 3 == 0) << j;
    if (MODE == 6) {
      if (sel) { kk = ld256(kc + r0); xx = ld256(xc + r0); } else { kk = v; xx = v; }
    }
    uint64_t ks[4] = {kk.x, kk.y, kk.z, kk.w};
    uint64_t xs[4] = {xx.x, xx.y, xx.z, xx.w};
    if (MODE == 0 || MODE == 6) {
#pragma unroll
      for (int j = 0; j < 4; ++j) if ((sel >> j) & 1) acc += ks[j] + xs[j];
      continue;
    }
    uint64_t first[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint64_t slot = mix(ks[j]) & mask;
      first[j] = 0;
      if (((sel >> j) & 1) && (MODE == 1 || MODE == 4)) first[j] = ldtab(tab + slot * 32);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!((sel >> j) & 1)) continue;
      uint64_t slot = mix(ks[j]) & mask;
      uint8_t* e = tab + slot * 32;
      if (MODE == 1) { acc += first[j]; continue; }
      if (MODE == 2) { red64(e + 8, (uint64_t)vv[j]); continue; }
      if (MODE == 3 || MODE == 4) {
        if (MODE == 4 && first[j] == 0x1234567) acc += 1;
        red64(e + 8, 1); red64(e + 16, (uint64_t)vv[j]); redf64(e + 24, __longlong_as_double((long long)xs[j]));
        continue;
      }
      if (MODE == 7) { uint32_t* s32 = (uint32_t*)soa; red32(s32 + slot, 1); red32(s32 + (mask + 1) + slot, (uint32_t)vv[j]); red32(s32 + 2 * (mask + 1) + slot, (uint32_t)xs[j]); continue; }
      if (MODE == 8) { redf32x4((float*)soa + slot * 4, 1.0f, (float)vv[j], (float)xs[j], 2.0f); continue; }
      if (MODE == 9) { red64(soa + slot, 1); red64(soa + (mask + 1) + slot, (uint64_t)vv[j]); continue; }
      if (MODE == 10) { redf64(soa + slot, 1.0); redf64(soa + (mask + 1) + slot, (double)vv[j]); redf64(soa + 2 * (mask + 1) + slot, __longlong_as_double((long long)xs[j])); continue; }
      if (MODE == 11) { red32((uint32_t*)soa + slot, 1); red64(soa + (mask + 1) + slot, (uint64_t)vv[j]); redf64(soa + 2 * (mask + 1) + slot, __longlong_as_double((long long)xs[j])); continue; }
      if (MODE == 12) { redf32x2((float*)soa + slot * 2, 1.0f, (float)vv[j]); continue; }
      if (MODE == 13) { red64(soa + slot * 4, 1); red64(soa + slot * 4 + 1, (uint64_t)vv[j]); redf64(soa + slot * 4 + 2, __longlong_as_double((long long)xs[j])); red64(soa + slot * 4 + 3, 1); continue; }
      if (MODE == 5) {
        red64(soa + slot, 1); red64(soa + (mask + 1) + slot, (uint64_t)vv[j]); redf64(soa + 2 * (mask + 1) + slot, __longlong_as_double((long long)xs[j]));
      }
    }
  }
  if (acc == 0xdeadbeef) *sink = acc;
}

__global__ void fill(uint64_t* kc, int64_t* vc, double* xc, int64_t n, uint64_t nkeys) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t r = mix(i * 0x9E3779B97F4A7C15ULL + 1);
    kc[i] = __umul64hi(r, nkeys);
    vc[i] = (int64_t)(int32_t)(mix(r) >> 32);
    xc[i] = (double)(mix(r + 7) >> 44);
  }
}

template <int MODE>
void run(const char* name, const uint64_t* kc, const int64_t* vc, const double* xc, int64_t n, uint8_t* tab, uint64_t mask, uint64_t* sink, uint64_t* soa, int grid) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  k<MODE><<<grid, 256>>>(kc, vc, xc, n, tab, mask, sink, soa);
  cudaDeviceSynchronize();
  float best = 1e9;
  for (int it = 0; it < 3; ++it) {
    cudaEventRecord(a);
    k<MODE><<<grid, 256>>>(kc, vc, xc, n, tab, mask, sink, soa);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (ms < best) best = ms;
  }
  printf("%-46s grid %5d  %8.3f ms  %7.1f Grows/s  %7.1f GB/s(24B/row)\n", name, grid, best, n / best / 1e6, 24.0 * n / best / 1e6);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) printf("CUDA error %s\n", cudaGetErrorString(e));
}

// MODE B0: per surviving row ONE 16-byte TMA bulk reduction (.add.u64 on {cnt, sum_v})
// MODE B1: B0 + one f64 RED (sum_x)      MODE B2: two bulk reductions (u64 16 B + f64 16 B)
// AoS entry 32 B: [cnt][sum_v][sum_x][key]
// round-2 candidates: GEN = staging generations per thread, `lanes` = bit mask of the lanes that use
// the bulk path (the others update cnt and sum_v with two plain REDs), PROBE = also load the key
// bucket first (what the real kernel does)
template <int MODE, int GEN = 2, bool PROBE = false>
__global__ void __launch_bounds__(256, 4) kbulk(const uint64_t* kc, const int64_t* vc, const double* xc, int64_t n, uint8_t* tab,
                                                uint64_t mask, uint64_t* sink, uint32_t lanes = 0xFFFFFFFFu) {
  constexpr int W = MODE == 2 ? 4 : 2;
  extern __shared__ __align__(16) uint64_t stage_raw[];
  uint64_t (*stage)[256][4][W] = reinterpret_cast<uint64_t (*)[256][4][W]>(stage_raw);
  int64_t tiles = n / 1024;
  uint64_t acc = 0;
  int gen = 0;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    int64_t r0 = t * 1024 + 4 * threadIdx.x;
    u64x4 v = ld256(vc + r0);
    u64x4 kk = ld256(kc + r0), xx = ld256(xc + r0);
    int64_t vv[4] = {(int64_t)v.x, (int64_t)v.y, (int64_t)v.z, (int64_t)v.w};
    uint64_t ks[4] = {kk.x, kk.y, kk.z, kk.w};
    uint64_t xs[4] = {xx.x, xx.y, xx.z, xx.w};
    uint32_t sel = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) sel |= (vv[j] % 3 == 0) << j;
    // the slots of this generation were handed to TMA GEN iterations ago: wait until it has read them
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(GEN - 1) : "memory");
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!((sel >> j) & 1)) continue;
      uint64_t* s = stage[gen][threadIdx.x][j];
      s[0] = 1; s[1] = (uint64_t)vv[j];
      if (MODE == 2) { s[2] = xs[j]; s[3] = 0; }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!((sel >> j) & 1)) continue;
      uint64_t slot = mix(ks[j]) & mask;
      uint8_t* e = tab + slot * 32;
      if (PROBE && ldtab(e + 24) == 0x1234567) acc += 1;
      uint32_t sa = (uint32_t)__cvta_generic_to_shared(stage[gen][threadIdx.x][j]);
      if ((lanes >> (threadIdx.x & 31)) & 1) {
        asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.u64 [%0], [%1], 16;" ::"l"(e), "r"(sa) : "memory");
      } else {
        red64(e, 1); red64(e + 8, (uint64_t)vv[j]);
      }
      if (MODE == 1) redf64(e + 16, __longlong_as_double((long long)xs[j]));
      if (MODE == 2) asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f64 [%0], [%1], 16;" ::"l"(e + 16), "r"(sa + 16) : "memory");
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    gen = (gen + 1) % GEN;
    acc += sel;
  }
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  if (acc == 0xdeadbeefULL << 20) *sink = acc;
}
template <int MODE, int GEN = 2, bool PROBE = false>
void runbulk(const char* name, const uint64_t* kc, const int64_t* vc, const double* xc, int64_t n, uint8_t* tab, uint64_t mask, uint64_t* sink, int grid,
             uint32_t lanes = 0xFFFFFFFFu) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  const int smem = GEN * 256 * 4 * (MODE == 2 ? 4 : 2) * 8;
  cudaFuncSetAttribute(kbulk<MODE, GEN, PROBE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  kbulk<MODE, GEN, PROBE><<<grid, 256, smem>>>(kc, vc, xc, n, tab, mask, sink, lanes);
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("%s: CUDA error %s\n", name, cudaGetErrorString(e)); return; }
  float best = 1e9;
  for (int it = 0; it < 3; ++it) {
    cudaEventRecord(a);
    kbulk<MODE, GEN, PROBE><<<grid, 256, smem>>>(kc, vc, xc, n, tab, mask, sink, lanes);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (ms < best) best = ms;
  }
  printf("%-46s grid %5d  %8.3f ms  %7.1f Grows/s  %7.1f GB/s(24B/row)\n", name, grid, best, n / best / 1e6, 24.0 * n / best / 1e6);
}

int main(int argc, char** argv) {
  int64_t n = argc > 1 ? atoll(argv[1]) : 1000000000LL;
  n = n / 1024 * 1024;
  uint64_t nkeys = argc > 2 ? atoll(argv[2]) : 1000000;
  uint64_t cap = 1; while (cap < 2 * nkeys) cap <<= 1;
  uint64_t *kc, *sink, *soa; int64_t* vc; double* xc; uint8_t* tab;
  cudaMalloc(&kc, n * 8); cudaMalloc(&vc, n * 8); cudaMalloc(&xc, n * 8); cudaMalloc(&tab, cap * 32); cudaMalloc(&sink, 8); cudaMalloc(&soa, cap * 32);
  cudaMemset(tab, 0, cap * 32); cudaMemset(soa, 0, cap * 32);
  fill<<<148 * 16, 256>>>(kc, vc, xc, n, nkeys);
  cudaDeviceSynchronize();
  printf("rows %lld keys %llu table %llu slots x 32 B = %.1f MB\n", (long long)n, (unsigned long long)nkeys, (unsigned long long)cap, cap * 32 / 1e6);
  for (int occ : {4, 8, 16, 64}) {
    int grid = 148 * occ;
    run<0>("0 stream 3 cols", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  }
  int grid = 148 * 4;
  run<6>("6 stream v, k/x only when selected", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<1>("1 stream + probe load", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<2>("2 stream + 1 RED", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<3>("3 stream + 3 RED same sector", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<4>("4 stream + probe + 3 RED same sector", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<5>("5 stream + 3 RED SoA", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<7>("7 stream + 3 RED u32 SoA", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<8>("8 stream + 1 RED f32x4", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<12>("12 stream + 1 RED f32x2", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<9>("9 stream + 2 RED u64 SoA", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<10>("10 stream + 3 RED f64 SoA", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<11>("11 stream + u32 + u64 + f64 SoA", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  run<13>("13 stream + 4 RED same sector", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  // correctness probe of the bulk reduction: table zeroed, one pass, check a few entries
  cudaMemset(tab, 0, cap * 32);
  cudaFuncSetAttribute(kbulk<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 256 * 4 * 4 * 8);
  kbulk<2><<<grid, 256, 2 * 256 * 4 * 4 * 8>>>(kc, vc, xc, n, tab, cap - 1, sink);
  { cudaError_t e = cudaDeviceSynchronize(); if (e != cudaSuccess) printf("bulk probe: CUDA error %s\n", cudaGetErrorString(e)); }
  {
    uint64_t h[8]; cudaMemcpy(h, tab, 64, cudaMemcpyDeviceToHost);
    uint64_t tot = 0; uint64_t* all = (uint64_t*)malloc(cap * 32); cudaMemcpy(all, tab, cap * 32, cudaMemcpyDeviceToHost);
    for (uint64_t i = 0; i < cap; ++i) tot += all[i * 4];
    printf("bulk check: entry0 cnt=%llu sumv=%lld sumx=%f ; total cnt over table = %llu (expect ~n/3 = %lld)\n", (unsigned long long)h[0], (long long)h[1], *(double*)&h[2], (unsigned long long)tot, (long long)(n / 3));
    free(all);
  }
  runbulk<0>("B0 stream + 1 bulk-reduce 16B u64x2", kc, vc, xc, n, tab, cap - 1, sink, grid);
  runbulk<1>("B1 stream + bulk u64x2 + RED f64", kc, vc, xc, n, tab, cap - 1, sink, grid);
  runbulk<2>("B2 stream + bulk u64x2 + bulk f64x2", kc, vc, xc, n, tab, cap - 1, sink, grid);
  // round-2 candidates (not measured yet): deeper staging, RED/TMA lane mixes, with the probe
  runbulk<1, 4>("B1 GEN=4", kc, vc, xc, n, tab, cap - 1, sink, grid);
  runbulk<1, 2>("B1 3/4 lanes bulk", kc, vc, xc, n, tab, cap - 1, sink, grid, 0x77777777u);
  runbulk<1, 2>("B1 1/2 lanes bulk", kc, vc, xc, n, tab, cap - 1, sink, grid, 0x55555555u);
  runbulk<1, 2>("B1 1/4 lanes bulk", kc, vc, xc, n, tab, cap - 1, sink, grid, 0x11111111u);
  runbulk<1, 2, true>("B1 + probe", kc, vc, xc, n, tab, cap - 1, sink, grid);
  runbulk<1, 2, true>("B1 + probe, 1/2 lanes bulk", kc, vc, xc, n, tab, cap - 1, sink, grid, 0x55555555u);
  grid = 148 * 8;
  run<4>("4 (grid x8 -> occupancy-limited to 4/SM)", kc, vc, xc, n, tab, cap - 1, sink, soa, grid);
  return 0;
}
