// Isolated timing of the bordered 34 x 34 solve (legs model): shuffle-based chol_reg32b vs the row-register chol_rs32b, and chol_rs<32> for scale.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I../../myosuite_b200/csrc -o ubench_chol34 ubench_chol34.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "myo_solver.cuh"
__global__ void __launch_bounds__(320) k(double* out, long long* cyc, int reps, int mode, int n) {
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, nt = n*(n+1)/2;
  double* H = smem + wid*(36*37/2 + 2*36 + 8); double* x = H + 36*37/2;
  long long tot = 0;
  for (int r = 0; r < reps; r++) {
    for (int i = lane; i < nt; i += 32) { int a, b; tri_index(i, a, b); H[i] = (a == b) ? 10.0 + a : 1.0/(1 + a + b); }
    for (int i = lane; i < n; i += 32) x[i] = 1.0 + i;
    __syncwarp();
    long long t0 = clock64();
    if (mode == 0) chol_reg32b<4>(H, n, x, lane); else if (mode == 1) chol_rs32b<2>(H, x, n, lane); else chol_rs<32>(H, x, n, lane);
    long long t1 = clock64(); tot += t1 - t0; }
  if (lane == 0) cyc[blockIdx.x*(blockDim.x >> 5) + wid] = tot / reps;
  out[(blockIdx.x*blockDim.x + threadIdx.x)*2] = x[lane]; out[(blockIdx.x*blockDim.x + threadIdx.x)*2+1] = x[32 + (lane & 1)];
}
int main() {
  double* out; long long* cyc; cudaMalloc(&out, 1 << 24); cudaMalloc(&cyc, 1 << 16); long long h[4096]; const char* nm[3] = {"chol_reg32b<4> (shuffles)", "chol_rs32b<2> (row registers, static border)", "chol_rs<32>"};
  for (int mode = 0; mode < 3; mode++) for (int w = 1; w <= 7; w += 6) {
    size_t sm = (size_t)w*(36*37/2 + 2*36 + 8)*8; int n = mode == 2 ? 32 : 34;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    for (int r = 0; r < 2; r++) { k<<<132, 32*w, sm>>>(out, cyc, 20, mode, n); cudaMemcpy(h, cyc, 8*132*w, cudaMemcpyDeviceToHost); }
    double m = 0; for (int i = 0; i < 132*w; i++) m += h[i];
    double hx[8]; cudaMemcpy(hx, out, 64, cudaMemcpyDeviceToHost);
    printf("%s n=%d: %d warps/SM: %.0f cycles per solve (%s); x0 %.12g x1 %.12g x32 %.12g\n", nm[mode], n, w, m/(132*w), cudaGetErrorString(cudaGetLastError()), hx[0], hx[2], hx[1]); }
  return 0; }
