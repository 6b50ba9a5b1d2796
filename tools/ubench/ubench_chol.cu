// Isolated timing of the dense solver (row-register LDL') exactly as the step kernel compiles it: cycles per solve for one warp,
// and with 10 warps per SM (all solving).  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I../../myosuite_b200/csrc -o ubench_chol ubench_chol.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "myo_solver.cuh"
template <int NM>
__global__ void k(double* out, long long* cyc, int reps, int mode) {
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, n = NM, nt = n*(n+1)/2;
  double* H = smem + wid*(nt + 2*n + 8); double* x = H + nt; double* H0 = x + n;   // H0 unused; keep a pristine copy in registers instead
  long long tot = 0;
  for (int r = 0; r < reps; r++) {
    for (int i = lane; i < nt; i += 32) { int a, b; tri_index(i, a, b); H[i] = (a == b) ? 10.0 + a : 1.0/(1 + a + b); }
    for (int i = lane; i < n; i += 32) x[i] = 1.0 + i;
    __syncwarp();
    long long t0 = clock64();
    if (mode) chol_rs<NM>(H, x, n, lane); else chol_rot<24>(H, x, n, lane);
    long long t1 = clock64(); tot += t1 - t0; }
  if (lane == 0) cyc[blockIdx.x*(blockDim.x >> 5) + wid] = tot / reps;
  out[blockIdx.x*blockDim.x + threadIdx.x] = x[lane % n];
}
int main() {
  double* out; long long* cyc; cudaMalloc(&out, 1 << 22); cudaMalloc(&cyc, 1 << 16); long long h[4096];
  for (int mode = 0; mode < 2; mode++) for (int w = 1; w <= 10; w += 9) {
    size_t sm = (size_t)w*(23*24/2 + 2*23 + 8)*8;
    cudaFuncSetAttribute(k<23>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    for (int r = 0; r < 2; r++) { k<23><<<132, 32*w, sm>>>(out, cyc, 20, mode); cudaMemcpy(h, cyc, 8*132*w, cudaMemcpyDeviceToHost); }
    double m = 0; for (int i = 0; i < 132*w; i++) m += h[i]; printf("%s n=23: %d warps/SM: %.0f cycles per solve, x[0..2] check below (%s)\n", mode ? "chol_rs (unrolled)" : "chol_rot (rolled)", w, m/(132*w), cudaGetErrorString(cudaGetLastError())); }
  double hx[64]; cudaMemcpy(hx, out, 64*8, cudaMemcpyDeviceToHost); printf("solution head: %.12g %.12g %.12g\n", hx[0], hx[1], hx[2]);
  return 0; }
