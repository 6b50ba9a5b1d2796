// Instruction-fetch bandwidth for never-looped straight-line code with HIGH ILP (8 independent FFMA/DFMA chains): cycles per
// instruction vs code size, for 1 warp and 10 lockstep warps per SM.  Each size runs twice (the second run finds the code in L2).
#include <cstdio>
#include <cuda_runtime.h>
template <int REP, typename T> __device__ __forceinline__ void body(T* x, T a, T b) {
  #pragma unroll
  for (int i = 0; i < REP; i++) {
    #pragma unroll
    for (int j = 0; j < 8; j++) x[j] = x[j]*a + b; } }
template <int REP, typename T> __global__ void k_code(T* out, long long* cyc, T a, T b, int iters) {
  T x[8]; for (int j = 0; j < 8; j++) x[j] = a + threadIdx.x + j;
  long long t0 = clock64();
  for (int it = 0; it < iters; it++) { body<REP, T>(x, a, b); __syncthreads(); }
  long long t1 = clock64(); if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
  T s = 0; for (int j = 0; j < 8; j++) s += x[j]; out[blockIdx.x*blockDim.x + threadIdx.x] = s; }
template <int REP, typename T> void run(const char* name, void* out, long long* cyc) {
  long long h[132];
  for (int w = 1; w <= 10; w += 9) for (int iters = 1; iters <= 3; iters += 2) {
    for (int r = 0; r < 2; r++) { k_code<REP, T><<<132, 32*w>>>((T*)out, cyc, (T)0.999, (T)0.001, iters); cudaMemcpy(h, cyc, 8*132, cudaMemcpyDeviceToHost); }
    double m = 0; for (int i = 0; i < 132; i++) m += h[i]; m /= 132;
    printf("%s code %5d KB  warps/SM %2d  passes %d: %6.2f cycles per instruction  (%.2f bytes of code per cycle per SM)\n", name, REP*8*16/1024, w, iters, m/((double)REP*8*iters), (double)REP*8*16*iters/m); } }
int main() {
  void* out; long long* cyc; cudaMalloc(&out, 1 << 22); cudaMalloc(&cyc, 4096);
  run<32, float>("ffma", out, cyc); run<256, float>("ffma", out, cyc); run<1024, float>("ffma", out, cyc); run<4096, float>("ffma", out, cyc); run<8192, float>("ffma", out, cyc);
  run<32, double>("dfma", out, cyc); run<1024, double>("dfma", out, cyc); run<8192, double>("dfma", out, cyc);
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize())); return 0; }
