// tools/arith_sweep.cu — standalone tuning harness (not part of the product library):
// times variants of the streaming f64 add (2 loads + 1 store per 16 B) to pick the
// bytes-in-flight / occupancy point for k_arith. Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o arith_sweep arith_sweep.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>

__device__ __forceinline__ uint4 ld16(const void *p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ld16_plain(const void *p) { return *reinterpret_cast<const uint4 *>(p); }
__device__ __forceinline__ void st16(void *p, uint4 v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st16_plain(void *p, uint4 v) { *reinterpret_cast<uint4 *>(p) = v; }

__device__ __forceinline__ uint4 add2(uint4 a, uint4 b) {
  double a0 = __hiloint2double(a.y, a.x), a1 = __hiloint2double(a.w, a.z);
  double b0 = __hiloint2double(b.y, b.x), b1 = __hiloint2double(b.w, b.z);
  double c0 = __dadd_rn(a0, b0), c1 = __dadd_rn(a1, b1);
  return make_uint4(__double2loint(c0), __double2hiint(c0), __double2loint(c1), __double2hiint(c1));
}

// U 16-byte vectors per thread per iteration, warp-contiguous (512 B per warp access)
template <int U, int THREADS, int MINB, int HINT>
__global__ void __launch_bounds__(THREADS, MINB) k_add(const uint4 *__restrict__ a, const uint4 *__restrict__ b, uint4 *__restrict__ o, int64_t nvec) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * THREADS) >> 5;
  const int64_t groups = nvec / (32 * U);
  for (int64_t g = warp; g < groups; g += nwarps) {
    const int64_t base = g * 32 * U + lane;
    uint4 va[U], vb[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      va[k] = HINT ? ld16(a + base + k * 32) : ld16_plain(a + base + k * 32);
      vb[k] = HINT ? ld16(b + base + k * 32) : ld16_plain(b + base + k * 32);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      uint4 c = add2(va[k], vb[k]);
      if (HINT) st16(o + base + k * 32, c); else st16_plain(o + base + k * 32, c);
    }
  }
}

template <int U, int THREADS, int MINB, int HINT>
void run(const char *name, const uint4 *a, const uint4 *b, uint4 *o, int64_t nvec, int sms, int oversub) {
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_add<U, THREADS, MINB, HINT>, THREADS, 0);
  int grid = sms * per_sm * oversub;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 2; ++i) k_add<U, THREADS, MINB, HINT><<<grid, THREADS>>>(a, b, o, nvec);
  cudaEventRecord(e0);
  const int reps = 5;
  for (int i = 0; i < reps; ++i) k_add<U, THREADS, MINB, HINT><<<grid, THREADS>>>(a, b, o, nvec);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= reps;
  printf("%-34s U=%d thr=%4d minb=%d hint=%d occ=%d grid=%5d  %.3f ms  %.1f GB/s\n", name, U, THREADS, MINB, HINT, per_sm, grid, ms, 48.0 * nvec / ms / 1e6);
}

int main() {
  int64_t n = 1000000000; int64_t nvec = n / 2;
  uint4 *a, *b, *o;
  cudaMalloc(&a, n * 8); cudaMalloc(&b, n * 8); cudaMalloc(&o, n * 8);
  cudaMemset(a, 1, n * 8); cudaMemset(b, 2, n * 8);
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  // reference: plain copy with cudaMemcpy D2D
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaMemcpy(o, a, n * 8, cudaMemcpyDeviceToDevice);
  cudaEventRecord(e0); for (int i = 0; i < 5; ++i) cudaMemcpyAsync(o, a, n * 8, cudaMemcpyDeviceToDevice); cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1); printf("cudaMemcpy D2D 8 GB: %.3f ms, %.1f GB/s (read+write)\n", ms / 5, 16.0 * n / (ms / 5) / 1e6);
  run<4, 256, 4, 1>("base(U4,256,mb4)", a, b, o, nvec, sms, 1);
  run<4, 256, 4, 0>("plain ld/st", a, b, o, nvec, sms, 1);
  run<2, 256, 8, 1>("U2 mb8", a, b, o, nvec, sms, 1);
  run<2, 256, 6, 1>("U2 mb6", a, b, o, nvec, sms, 1);
  run<8, 256, 2, 1>("U8 mb2", a, b, o, nvec, sms, 1);
  run<8, 256, 3, 1>("U8 mb3", a, b, o, nvec, sms, 1);
  run<4, 512, 2, 1>("U4 512thr mb2", a, b, o, nvec, sms, 1);
  run<4, 128, 8, 1>("U4 128thr mb8", a, b, o, nvec, sms, 1);
  run<4, 1024, 1, 1>("U4 1024thr", a, b, o, nvec, sms, 1);
  run<1, 256, 8, 1>("U1 mb8", a, b, o, nvec, sms, 1);
  run<4, 256, 4, 1>("base x2 oversub", a, b, o, nvec, sms, 2);
  run<4, 256, 4, 1>("base x8 oversub", a, b, o, nvec, sms, 8);
  run<2, 256, 8, 1>("U2 mb8 x8 oversub", a, b, o, nvec, sms, 8);
  run<1, 256, 8, 1>("U1 mb8 x16 oversub", a, b, o, nvec, sms, 16);
  return 0;
}
