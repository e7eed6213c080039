// FP64-pipe big-integer product microbenchmark for sm_90a.
// A 52x52 -> 104-bit product as two round-toward-zero DFMAs and one DADD (the double-precision split used by
// Emmart, Zheng & Weems, ARITH 2018):  hi = fma_rz(a, b, 2^104), lo = fma_rz(a, b, (2^104 + 2^52) - hi); the bit
// patterns of hi / lo carry the high / low 52 bits of a*b in their mantissas and are summed as 64-bit integers.
// Measures products / clk / SM of an 8x8-limb tile product (64 products into 16 column sums) in the
// thread-per-element form the Paillier kernels use, against the 25.1 MAC(32x32)/clk/SM of the IMAD.WIDE carry chains.
//   build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dfma_peak dfma_peak.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#define ITERS 1024
#define C1 20282409603651670423947251286016.0   /* 2^104 */
#define C2 20282409603651674927546878656512.0   /* 2^104 + 2^52 */

__device__ __forceinline__ void prod52(double a, double b, uint64_t& acc_lo, uint64_t& acc_hi) {
  double hi = __fma_rz(a, b, C1);
  double sub = C2 - hi;
  double lo = __fma_rz(a, b, sub);
  acc_hi += (uint64_t)__double_as_longlong(hi);
  acc_lo += (uint64_t)__double_as_longlong(lo);
}

// 3-input form: the two 64-bit addends of a column are added in one IADD3 / IADD3.X pair
__device__ __forceinline__ void prod52_pair(double a0, double b0, double a1, double b1, uint64_t& acc_lo, uint64_t& acc_hi) {
  double h0 = __fma_rz(a0, b0, C1), h1 = __fma_rz(a1, b1, C1);
  double l0 = __fma_rz(a0, b0, C2 - h0), l1 = __fma_rz(a1, b1, C2 - h1);
  acc_hi += (uint64_t)__double_as_longlong(h0) + (uint64_t)__double_as_longlong(h1);
  acc_lo += (uint64_t)__double_as_longlong(l0) + (uint64_t)__double_as_longlong(l1);
}

template <int MODE>
__device__ __forceinline__ void tile_mac52(uint64_t (&acc)[17], const double (&a)[8], const double (&b)[8]) {
  if (MODE == 0) {
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
      for (int j = 0; j < 8; j++) prod52(a[i], b[j], acc[i + j], acc[i + j + 1]);
  } else {
    // walk the columns; pair the products of a column
#pragma unroll
    for (int k = 0; k < 15; k++) {
      const int i0 = k < 8 ? 0 : k - 7, i1 = k < 8 ? k : 7;
#pragma unroll
      for (int i = i0; i <= i1; i += 2) {
        if (i + 1 <= i1) prod52_pair(a[i], b[k - i], a[i + 1], b[k - i - 1], acc[k], acc[k + 1]);
        else prod52(a[i], b[k - i], acc[k], acc[k + 1]);
      }
    }
  }
}

template <int MODE>
__global__ void k_tile(uint64_t* out, const double* in, long long* cyc) {
  double a[8], b[8];
  uint64_t acc[17];
  for (int i = 0; i < 8; i++) { a[i] = in[(threadIdx.x + i * 7) & 255]; b[i] = in[(threadIdx.x + 100 + i) & 255]; }
  for (int i = 0; i < 17; i++) acc[i] = i;
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
    tile_mac52<MODE>(acc, a, b);
    // keep the operands changing without extra FP64 work: swap roles through the integer side
    a[it & 7] = __longlong_as_double((__double_as_longlong(a[it & 7]) & ~0xfffffll) | (acc[3] & 0xfffff));
  }
  long long t1 = clock64();
  uint64_t s = 0;
  for (int i = 0; i < 17; i++) s ^= acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// operands from shared memory in the interleaved layout (limb l of thread t at base[l * nthreads + t])
template <int MODE>
__global__ void k_tile_smem(uint64_t* out, const double* in, long long* cyc, int ntiles) {
  extern __shared__ double sm[];
  const int nt = blockDim.x;
  for (int i = threadIdx.x; i < 2 * ntiles * 8 * nt; i += nt) sm[i] = in[i & 255];
  __syncthreads();
  uint64_t acc[17];
  for (int i = 0; i < 17; i++) acc[i] = i;
  const double2* A = (const double2*)sm;
  const double2* B = A + ntiles * 4 * nt;
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS / 8; it++) {
#pragma unroll 1
    for (int ta = 0; ta < ntiles; ta++) {
      double a[8], b[8];
#pragma unroll
      for (int q = 0; q < 4; q++) { double2 v = A[(ta * 4 + q) * nt + threadIdx.x]; a[2 * q] = v.x; a[2 * q + 1] = v.y; }
#pragma unroll
      for (int q = 0; q < 4; q++) { double2 v = B[((ntiles - 1 - ta) * 4 + q) * nt + threadIdx.x]; b[2 * q] = v.x; b[2 * q + 1] = v.y; }
      tile_mac52<MODE>(acc, a, b);
    }
  }
  long long t1 = clock64();
  uint64_t s = 0;
  for (int i = 0; i < 17; i++) s ^= acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// exactness check of the split against 128-bit integer arithmetic
__global__ void k_check(const uint64_t* x, const uint64_t* y, int n, int* bad) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t a = x[i] & ((1ull << 52) - 1), b = y[i] & ((1ull << 52) - 1);
  if (i == 0) a = b = (1ull << 52) - 1;
  if (i == 1) a = 0;
  uint64_t lo = 0, hi = 0;
  prod52((double)a, (double)b, lo, hi);
  lo -= 0x4330000000000000ull; hi -= 0x4670000000000000ull;
  uint64_t pl = a * b, ph = __umul64hi(a, b);
  uint64_t el = pl & ((1ull << 52) - 1), eh = (pl >> 52) | (ph << 12);
  if (lo != el || hi != eh) atomicAdd(bad, 1);
}

template <typename F>
static double run(F launch, int blocks, long long* d_cyc) {
  launch(); launch();
  cudaDeviceSynchronize();
  long long* h = new long long[blocks];
  cudaMemcpy(h, d_cyc, blocks * sizeof(long long), cudaMemcpyDeviceToHost);
  double s = 0;
  for (int i = 0; i < blocks; i++) s += (double)h[i];
  delete[] h;
  return s / blocks;
}

int main() {
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) { printf("{\"error\": \"no device\"}\n"); return 1; }
  const int sms = p.multiProcessorCount;
  double* d_in; uint64_t* d_out; long long* d_cyc; int* d_bad; uint64_t *d_x, *d_y;
  cudaMalloc(&d_in, 256 * 8); cudaMalloc(&d_out, sms * 1024 * 8); cudaMalloc(&d_cyc, sms * 8); cudaMalloc(&d_bad, 4);
  double h_in[256]; uint64_t hx[4096], hy[4096];
  uint64_t s = 88172645463325252ull;
  for (int i = 0; i < 256; i++) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; h_in[i] = (double)(s & ((1ull << 52) - 1)); }
  for (int i = 0; i < 4096; i++) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; hx[i] = s; s ^= s << 13; s ^= s >> 7; s ^= s << 17; hy[i] = s; }
  cudaMemcpy(d_in, h_in, sizeof h_in, cudaMemcpyHostToDevice);
  cudaMalloc(&d_x, sizeof hx); cudaMalloc(&d_y, sizeof hy);
  cudaMemcpy(d_x, hx, sizeof hx, cudaMemcpyHostToDevice); cudaMemcpy(d_y, hy, sizeof hy, cudaMemcpyHostToDevice);
  cudaMemset(d_bad, 0, 4);
  k_check<<<16, 256>>>(d_x, d_y, 4096, d_bad);
  int bad = -1; cudaMemcpy(&bad, d_bad, 4, cudaMemcpyDeviceToHost);
  printf("{\"split_mismatches\": %d, \"sms\": %d", bad, sms);
  const int thr[] = {128, 192, 256, 384, 512};
  for (int mode = 0; mode < 2; mode++)
    for (int t : thr) {
      double c = mode == 0 ? run([&] { k_tile<0><<<sms, t>>>(d_out, d_in, d_cyc); }, sms, d_cyc)
                           : run([&] { k_tile<1><<<sms, t>>>(d_out, d_in, d_cyc); }, sms, d_cyc);
      printf(", \"tile_reg_mode%d_%dthr\": %.2f", mode, t, (double)ITERS * 64 * t / c);
    }
  cudaFuncSetAttribute(k_tile_smem<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  cudaFuncSetAttribute(k_tile_smem<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  for (int mode = 0; mode < 2; mode++)
    for (int t : {128, 160, 192}) {
      const int ntiles = 5; size_t smem = (size_t)2 * ntiles * 64 * t;
      double c = mode == 0 ? run([&] { k_tile_smem<0><<<sms, t, smem>>>(d_out, d_in, d_cyc, ntiles); }, sms, d_cyc)
                           : run([&] { k_tile_smem<1><<<sms, t, smem>>>(d_out, d_in, d_cyc, ntiles); }, sms, d_cyc);
      printf(", \"tile_smem_mode%d_%dthr\": %.2f", mode, t, (double)(ITERS / 8) * ntiles * 64 * t / c);
    }
  printf(", \"unit\": \"52x52-bit products / clk / SM (x2.64 = 32x32 MAC equivalents)\", \"err\": \"%s\"}\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
