// Latency micro-benchmarks for the quantities the step kernel's cycle model depends on (H100 SXM, sm_90a; one CTA per SM on its 132 SMs):
// dependent-chain latency of the f64 ops, shared-memory load->use, warp shuffles, and the cost of streaming never-seen
// straight-line code (instruction fetch) for 1 warp and for 10 lockstep warps per SM.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench ubench.cu && ./ubench
#include <cstdio>
#include <cuda_runtime.h>
#define N 256
#define CHAIN(name, init, stmt) \
__global__ void k_##name(double* out, long long* cyc, double a, double b) { double x = init; long long t0 = clock64(); \
  _Pragma("unroll") for (int i = 0; i < N; i++) { stmt; } long long t1 = clock64(); if (threadIdx.x == 0) { cyc[0] = t1 - t0; } out[threadIdx.x] = x; }
CHAIN(dfma, a, x = fma(x, b, a))
CHAIN(dmul, a, x = x * b)
CHAIN(dadd, a, x = x + b)
CHAIN(ddiv, a, x = b / x + a)
CHAIN(drcp, a, x = 1.0 / x + a)
CHAIN(dsqrt, a, x = sqrt(x) + a)
CHAIN(drsqrt, a, x = rsqrt(x) + a)
CHAIN(dsin, a, x = sin(x) + a)
CHAIN(dacos, a, x = acos(x * 0.1) + a)
CHAIN(dasin, a, x = asin(x * 0.1) + a)
CHAIN(dexp, a, x = exp(-x) + a)
CHAIN(shfl, a, x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31) + a)
CHAIN(ffma, a, x = (double)fmaf((float)x, 1.0001f, 0.5f))
__global__ void k_lds(double* out, long long* cyc, int stride) { __shared__ double s[1024]; for (int i = threadIdx.x; i < 1024; i += blockDim.x) s[i] = (double)((i + stride) & 1023); __syncthreads();
  double x = threadIdx.x; long long t0 = clock64();
  #pragma unroll
  for (int i = 0; i < N; i++) x = s[(int)x];
  long long t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0; out[threadIdx.x] = x; }
__global__ void k_sts_lds(double* out, long long* cyc) { __shared__ double s[64]; double x = threadIdx.x; long long t0 = clock64();
  #pragma unroll
  for (int i = 0; i < N; i++) { s[threadIdx.x] = x; __syncwarp(); x = s[(threadIdx.x + 1) & 31] + 1.0; __syncwarp(); }
  long long t1 = clock64(); if (threadIdx.x == 0) cyc[0] = t1 - t0; out[threadIdx.x] = x; }
// straight-line code of a given size: BODY x REP dependent DFMAs interleaved with independent IMADs (never looped)
template <int REP> __device__ __forceinline__ double body(double x, double b, double a) {
  #pragma unroll
  for (int i = 0; i < REP; i++) { x = fma(x, b, a); x = fma(x, a, b); x = fma(x, b, b); x = fma(x, a, a); }
  return x; }
template <int REP> __global__ void k_code(double* out, long long* cyc, double a, double b, int iters) { double x = a + threadIdx.x;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) { x = body<REP>(x, b, a); __syncthreads(); }
  long long t1 = clock64(); if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0; out[blockIdx.x * blockDim.x + threadIdx.x] = x; }
int main() {
  double* out; long long* cyc; cudaMalloc(&out, 1 << 20); cudaMalloc(&cyc, 4096); long long h[512];
  #define RUN(name, ...) for (int r = 0; r < 2; r++) { k_##name<<<1, 32>>>(out, cyc, __VA_ARGS__); cudaMemcpy(h, cyc, 8, cudaMemcpyDeviceToHost); } printf("%-10s %7.1f cycles per dependent op\n", #name, (double)h[0] / N);
  RUN(dfma, 1.0, 0.999) RUN(dmul, 1.0, 0.999) RUN(dadd, 1.0, 0.5) RUN(ddiv, 1.5, 0.7) RUN(drcp, 1.5, 0.7) RUN(dsqrt, 1.5, 0.7) RUN(drsqrt, 1.5, 0.7)
  RUN(dsin, 0.5, 0.7) RUN(dacos, 0.5, 0.7) RUN(dasin, 0.5, 0.7) RUN(dexp, 0.5, 0.7) RUN(shfl, 0.5, 0.7) RUN(ffma, 0.5, 0.7)
  for (int r = 0; r < 2; r++) { k_lds<<<1, 32>>>(out, cyc, 7); cudaMemcpy(h, cyc, 8, cudaMemcpyDeviceToHost); } printf("%-10s %7.1f cycles per dependent LDS.64 (pointer chase)\n", "lds", (double)h[0] / N);
  for (int r = 0; r < 2; r++) { k_sts_lds<<<1, 32>>>(out, cyc); cudaMemcpy(h, cyc, 8, cudaMemcpyDeviceToHost); } printf("%-10s %7.1f cycles per STS -> syncwarp -> LDS(other lane) -> DADD -> syncwarp\n", "sts_lds", (double)h[0] / N);
  // instruction streaming: code bodies of 4*REP DFMAs (16 B each)
  #define CODE(REP) for (int w = 1; w <= 10; w += 9) for (int iters = 1; iters <= 4; iters += 3) { for (int r = 0; r < 2; r++) { k_code<REP><<<132, 32 * w>>>(out, cyc, 1.0, 0.999, iters); cudaMemcpy(h, cyc, 8 * 132, cudaMemcpyDeviceToHost); } \
      double m = 0; for (int i = 0; i < 132; i++) m += h[i]; m /= 132; printf("code %5d KB  warps/SM %2d  passes %d: %7.2f cycles per instruction (dependent DFMA chain)\n", (REP) * 4 * 16 / 1024, w, iters, m / ((double)(REP) * 4 * iters)); }
  CODE(256) CODE(2048) CODE(8192) CODE(16384)
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0; }
