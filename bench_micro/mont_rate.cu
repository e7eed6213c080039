// Microbenchmark: sustained rate of the tile Montgomery square / multiply (pai_core.cuh) on sm_90a.
//   build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o mont_rate mont_rate.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../python-paillier_b200/csrc/pai_core.cuh"
using namespace pai;

template <int NT, int NTHR, int VAR>
__global__ void __launch_bounds__(NTHR, 1) k_rate(uint32_t* out, const uint32_t* in, int nsqr, int nmul, long long* cyc) {
  extern __shared__ u4 smem[];
  const int Q = 2 * NT;
  u4* cst = smem;                       // N (Q quads) + ninv (2 quads)
  u4* bx = smem + Q + 2;                    // 3 buffers
  u4* by = NTHR > 128 ? bx : bx + Q * NTHR;          // 2-buffer mode: Y aliases X (read-only operand)
  u4* bz = NTHR > 128 ? bx + Q * NTHR : by + Q * NTHR;
  int tid = threadIdx.x;
  for (int i = tid; i < Q; i += NTHR) { u4 v; v.x = in[4 * i] | 1u; v.y = in[4 * i + 1]; v.z = in[4 * i + 2]; v.w = in[4 * i + 3] | 0x80000000u; cst[i] = v; }
  for (int q = 0; q < Q; q++) { u4 v; v.x = in[q + tid]; v.y = in[q * 3 + tid]; v.z = q * tid; v.w = in[q] >> 1; bx[q * NTHR + tid] = v; by[q * NTHR + tid] = v; }
  if (tid < 2) { u4 v; v.x = in[100 + 4 * tid]; v.y = in[101 + 4 * tid]; v.z = in[102]; v.w = in[103]; cst[Q + tid] = v; }
  __syncthreads();
  Opnd X{bx + tid, NTHR}, Y{by + tid, NTHR}, Z{bz + tid, NTHR}, N{cst, 1}, ninv{cst + Q, 1};
  long long t0 = clock64();
  for (int i = 0; i < nsqr; i++) { mont_sqr<NT>(Z, X, N, ninv); Opnd t = X; X = Z; Z = t; }
  for (int i = 0; i < nmul; i++) { mont_mul<NT>(Z, X, Y, N, ninv); Opnd t = X; X = Z; Z = t; }
  long long t1 = clock64();
  uint32_t s = 0;
  for (int q = 0; q < Q; q++) { u4 v = X.p[q * X.s]; s ^= v.x ^ v.y ^ v.z ^ v.w; }
  out[blockIdx.x * NTHR + tid] = s;
  if (tid == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int NT, int NTHR, int VAR>
void bench(int nsqr, int nmul, const char* name) {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  int nsm = p.multiProcessorCount;
  size_t smem = (size_t)(2 * NT) * 16 * (1 + (NTHR > 128 ? 2 : 3) * NTHR) + 32;
  cudaFuncSetAttribute(k_rate<NT, NTHR, VAR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int occ = 0; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_rate<NT, NTHR, VAR>, NTHR, smem);
  int grid = nsm * occ;
  uint32_t *out, *in; long long* cyc;
  cudaMalloc(&out, (size_t)grid * NTHR * 4); cudaMalloc(&in, 1 << 20); cudaMalloc(&cyc, grid * 8);
  cudaMemset(in, 0x5b, 1 << 20);
  k_rate<NT, NTHR, VAR><<<grid, NTHR, smem>>>(out, in, nsqr, nmul, cyc);
  cudaError_t e = cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k_rate<NT, NTHR, VAR><<<grid, NTHR, smem>>>(out, in, nsqr, nmul, cyc);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  long long* h = (long long*)malloc(grid * 8); cudaMemcpy(h, cyc, grid * 8, cudaMemcpyDeviceToHost);
  double mx = 0; for (int i = 0; i < grid; i++) if (h[i] > mx) mx = (double)h[i];
  // tile products actually executed
  double tiles_mul = 2.0 * NT * NT + NT /*m*/ , tiles_sqr = NT * (NT - 1) / 2.0 + NT + NT * NT + NT;
  double macs = 64.0 * (nsqr * tiles_sqr + nmul * tiles_mul);
  double canon = (double)(nsqr + nmul) * (2.0 * (8 * NT) * (8 * NT) + 8 * NT);
  printf("{\"kernel\": \"%s\", \"var\": %d, \"NT\": %d, \"threads\": %d, \"ctas_per_sm\": %d, \"err\": \"%s\", \"ms\": %.3f, \"cycles\": %.0f, "
         "\"exec_mac_per_clk_sm\": %.2f, \"canon_mac_per_clk_sm\": %.2f, \"modmul_per_s\": %.3e, \"canon_mac_per_s\": %.3e}\n",
         name, VAR, NT, NTHR, occ, cudaGetErrorString(e), ms, mx, macs * NTHR * occ / mx, canon * NTHR * occ / mx,
         (double)(nsqr + nmul) * grid * NTHR / (ms * 1e-3), canon * grid * NTHR / (ms * 1e-3));
  free(h); cudaFree(out); cudaFree(in); cudaFree(cyc);
}

int main() {
  bench<16, 128, 0>(40, 0, "sqr4096");
  bench<16, 128, 0>(0, 40, "mul4096");
  bench<16, 224, 0>(40, 0, "sqr4096_224thr_2buf");
  bench<16, 224, 0>(0, 40, "mul4096_224thr_2buf");
  bench<8, 128, 0>(80, 0, "sqr2048");
  bench<8, 128, 0>(0, 80, "mul2048");
  bench<24, 96, 0>(20, 0, "sqr6144_96thr");
  bench<4, 128, 0>(160, 0, "sqr1024");
  return 0;
}
