// Dev microbenchmark: what random 4-byte gather rate can an H100 sustain, by mechanism and index distribution?
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/ubench_gather scripts/ubench_gather.cu
// run:   /tmp/ubench_gather [scale]   or   /tmp/ubench_gather 27 sms  (L2-resident gathers confined to S SMs, DESIGN §5)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../lux_b200/csrc/build.cuh"
using namespace luxb;
namespace luxb { void set_error(const char*, ...) {} }

__global__ void gen_idx(uint32_t* idx, uint64_t m, int mode, int scale, uint32_t n) {
  uint64_t sm = splitmix64(27);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    if (mode == 0) idx[i] = (uint32_t)(splitmix64(i ^ 0x1234) % n);
    else { uint32_t s, d; rmat_edge(sm, i, scale, n, s, d); idx[i] = s; }
  }
}

template <int U, int HINT>
__global__ void gather_ldg(const uint32_t* __restrict__ idx, const float* __restrict__ x, uint64_t m, float* out) {
  float acc = 0.f;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t pol = 0;
  if (HINT == 1) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  if (HINT == 2) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; base < m; base += stride * U) {
    uint32_t id[U]; float v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) { uint64_t i = base + k * stride; id[k] = i < m ? __ldg(idx + i) : 0; }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (HINT == 0) v[k] = __ldg(x + id[k]);
      else asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v[k]) : "l"(x + id[k]), "l"(pol));
    }
#pragma unroll
    for (int k = 0; k < U; ++k) acc += v[k];
  }
  if (acc == 123.456f) out[0] = acc;
}

// cp.async 4B global->shared, deep queue, then consume
template <int U>
__global__ void gather_cpasync(const uint32_t* __restrict__ idx, const float* __restrict__ x, uint64_t m, float* out) {
  extern __shared__ float sm[];
  float acc = 0.f;
  uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; base < m; base += stride * U) {
#pragma unroll
    for (int k = 0; k < U; ++k) {
      uint64_t i = base + k * stride;
      uint32_t id = i < m ? __ldg(idx + i) : 0;
      uint32_t dst = (uint32_t)__cvta_generic_to_shared(sm + k * blockDim.x + threadIdx.x);
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(x + id));
    }
    asm volatile("cp.async.commit_group;");
    asm volatile("cp.async.wait_group 0;");
#pragma unroll
    for (int k = 0; k < U; ++k) acc += sm[k * blockDim.x + threadIdx.x];
  }
  if (acc == 123.456f) out[0] = acc;
}

// random gathers confined to the SMs with %smid < s_max: CTAs placed elsewhere leave at once, the others claim chunks of
// 2048 gathers from a counter.  Does the gather rate scale with SMs, or is it a limit of the whole device?
__global__ void gather_on_sms(const uint32_t* __restrict__ idx, const float* __restrict__ x, uint64_t m, float* out, uint32_t s_max,
                              unsigned long long* next) {
  uint32_t smid;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
  if (smid >= s_max) return;
  __shared__ unsigned long long base;
  float acc = 0.f;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) base = atomicAdd(next, 2048ull);
    __syncthreads();
    const uint64_t b = base;
    if (b >= m) break;
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { const uint64_t i = b + k * 256 + threadIdx.x; v[k] = i < m ? __ldg(x + __ldg(idx + i)) : 0.f; }
#pragma unroll
    for (int k = 0; k < 8; ++k) acc += v[k];
  }
  if (acc == 123.456f) out[0] = acc;
}

template <class F>
float timeit(F f, int reps = 3) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  f(); cudaDeviceSynchronize();
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) { cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best; }
  return best;
}

int main(int argc, char** argv) {
  int scale = argc > 1 ? atoi(argv[1]) : 27;
  uint32_t n = 1u << scale;
  uint64_t m = 1ull << 29;
  float* x; uint32_t* idx; float* out;
  cudaMalloc(&x, (size_t)n * 4); cudaMalloc(&idx, m * 4); cudaMalloc(&out, 4);
  cudaMemset(x, 0, (size_t)n * 4);
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  if (argc > 2 && !strcmp(argv[2], "sms")) {  // ubench_gather 27 sms: uniform gathers into 24 MB (L2-resident) on S SMs
    const uint32_t n24 = 6u << 20;
    unsigned long long* next; cudaMalloc(&next, 8);
    gen_idx<<<sms * 16, 256>>>(idx, m, 0, scale, n24);
    cudaDeviceSynchronize();
    for (int s : {sms, sms - 16, sms - 32, sms - 48, 40, 32}) {
      float ms = timeit([&] { cudaMemsetAsync(next, 0, 8); gather_on_sms<<<sms * 8, 256>>>(idx, x, m, out, s, next); });
      printf("  24 MB array, uniform, 8 gathers in flight per thread, %3d SMs: %7.3f ms  %6.1f Ggather/s\n", s, ms, m / ms / 1e6);
    }
    return 0;
  }
  for (int mode = 0; mode < 2; ++mode) {
    gen_idx<<<sms * 16, 256>>>(idx, m, mode, scale, n);
    cudaDeviceSynchronize();
    printf("== n=2^%d floats (%.0f MB), m=2^29 gathers, index dist: %s\n", scale, n * 4.0 / 1e6, mode ? "rmat-src" : "uniform");
    for (int bpsm : {2, 4, 8}) {
      int grid = sms * bpsm;
#define RUN(U, H, name) { float ms = timeit([&] { gather_ldg<U, H><<<grid, 256>>>(idx, x, m, out); }); \
      printf("  ldg U=%2d hint=%s blocks/SM=%d (%2d warps): %7.3f ms  %6.1f Ggather/s\n", U, name, bpsm, bpsm * 8, ms, m / ms / 1e6); }
      RUN(1, 0, "none") RUN(4, 0, "none") RUN(8, 0, "none") RUN(16, 0, "none")
      RUN(8, 1, "evict_last") RUN(8, 2, "evict_first")
#define RUNC(U) { cudaFuncSetAttribute(gather_cpasync<U>, cudaFuncAttributeMaxDynamicSharedMemorySize, U * 256 * 4); \
      float ms = timeit([&] { gather_cpasync<U><<<grid, 256, U * 256 * 4>>>(idx, x, m, out); }); \
      printf("  cp.async U=%2d blocks/SM=%d: %7.3f ms  %6.1f Ggather/s\n", U, bpsm, ms, m / ms / 1e6); }
      RUNC(8) RUNC(16)
    }
  }
  // sequential (coalesced) baseline for reference
  return 0;
}
