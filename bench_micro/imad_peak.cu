// Integer-pipe microbenchmark for sm_90a: measures the sustained issue rate of the
// instructions the Montgomery kernels are built from, so that roofline.peak in bench.py
// is a MEASURED number, not the nominal 64 IMAD/clk/SM.
//   build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o imad_peak imad_peak.cu
//   run  : ./imad_peak            (prints one JSON object)
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#define ITERS 2048

// ---- wide MAC carry chain: 4 x IMAD.WIDE.U32(.X) + IADD3.X  (what the tile MAC uses)
__device__ __forceinline__ void chain4(uint32_t* acc, const uint32_t* a, uint32_t b) {
  asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(acc[0]), "+r"(acc[1]) : "r"(a[0]), "r"(b));
  asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(acc[2]), "+r"(acc[3]) : "r"(a[1]), "r"(b));
  asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(acc[4]), "+r"(acc[5]) : "r"(a[2]), "r"(b));
  asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(acc[6]), "+r"(acc[7]) : "r"(a[3]), "r"(b));
  asm volatile("addc.u32 %0, %0, 0;" : "+r"(acc[8]));
}

template <int NCHAIN>
__global__ void k_wide_chain(uint32_t* out, const uint32_t* in, long long* cyc) {
  uint32_t a[4], b[NCHAIN], acc[NCHAIN][9];
  for (int i = 0; i < 4; i++) a[i] = in[threadIdx.x + i * 7];
  for (int c = 0; c < NCHAIN; c++) { b[c] = in[threadIdx.x + 100 + c]; for (int i = 0; i < 9; i++) acc[c][i] = in[c * 9 + i]; }
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int c = 0; c < NCHAIN; c++) chain4(acc[c], a, b[c]);
  }
  long long t1 = clock64();
  uint32_t s = 0;
  for (int c = 0; c < NCHAIN; c++) for (int i = 0; i < 9; i++) s ^= acc[c][i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// ---- independent ops, NACC accumulators
template <int OP, int NACC>
__global__ void k_indep(uint32_t* out, const uint32_t* in, long long* cyc) {
  uint32_t a = in[threadIdx.x], b = in[threadIdx.x + 64];
  uint32_t lo[NACC], hi[NACC], x[NACC], y[NACC];
  double d[NACC];
  for (int i = 0; i < NACC; i++) { lo[i] = in[i]; hi[i] = in[i + 32]; d[i] = (double)in[i]; x[i] = in[i + 3]; y[i] = in[i + 5]; }
  double da = (double)a * 1e-9, db = (double)b * 1e-9;
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int r = 0; r < 4; r++) {
#pragma unroll
      for (int i = 0; i < NACC; i++) {
        if (OP == 0) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(lo[i]) : "r"(a), "r"(b));
        if (OP == 1) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(lo[i]) : "r"(a), "r"(b));
        if (OP == 2) { uint64_t v = ((uint64_t)hi[i] << 32) | lo[i];
                       asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(v) : "r"(lo[i]), "r"(b));
                       lo[i] = (uint32_t)v; hi[i] = (uint32_t)(v >> 32); }
        if (OP == 3) asm volatile("fma.rn.f64 %0, %1, %2, %0;" : "+d"(d[i]) : "d"(da), "d"(db));
        if (OP == 4) asm volatile("shfl.sync.idx.b32 %0, %0, %1, 0x1f, 0xffffffff;" : "+r"(lo[i]) : "r"(a & 31));
        if (OP == 5) asm volatile("add.cc.u32 %0, %0, %2; addc.u32 %1, %1, %3;" : "+r"(lo[i]), "+r"(hi[i]) : "r"(a), "r"(b));
        if (OP == 6) asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.u32 %1, %2, %3, %1;" : "+r"(lo[i]), "+r"(hi[i]) : "r"(lo[(i + 1) % NACC]), "r"(b));
        // 7: the same multiplier WITHOUT a 64-bit addend (IMAD.WIDE.U32 Rd, Ra, Rb, RZ): separates the multiplier's rate from
        //    the cost of reading the addend pair
        if (OP == 7) { uint64_t v;
                       asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(v) : "r"(lo[i]), "r"(b));
                       lo[i] = (uint32_t)v ^ (uint32_t)(v >> 32); }
        // 8: wide MAC pair + two independent ALU adds per MAC (do IADD3s issue in the shadow of the half-rate IMAD.WIDE?)
        if (OP == 8) { asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.u32 %1, %2, %3, %1;" : "+r"(lo[i]), "+r"(hi[i]) : "r"(lo[(i + 1) % NACC]), "r"(b));
                       asm volatile("add.u32 %0, %0, %1;" : "+r"(x[i]) : "r"(a));
                       asm volatile("add.u32 %0, %0, %1;" : "+r"(y[i]) : "r"(b)); }
      }
    }
  }
  long long t1 = clock64();
  uint32_t s = 0;
  for (int i = 0; i < NACC; i++) s ^= lo[i] ^ hi[i] ^ (uint32_t)d[i] ^ x[i] ^ y[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// ---- LDS.128 throughput (conflict-free, interleaved layout)
__global__ void k_lds(uint32_t* out, const uint32_t* in, long long* cyc) {
  extern __shared__ uint4 sm[];
  for (int i = threadIdx.x; i < 16 * blockDim.x; i += blockDim.x) sm[i] = make_uint4(in[i & 255], i, i * 3, i * 7);
  __syncthreads();
  uint4 acc = make_uint4(0, 0, 0, 0);
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; it++) {
#pragma unroll
    for (int q = 0; q < 16; q++) { uint4 v = sm[q * blockDim.x + threadIdx.x]; acc.x ^= v.x; acc.y += v.y; acc.z ^= v.z; acc.w += v.w; }
  }
  long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc.x ^ acc.y ^ acc.z ^ acc.w;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

struct Res { double per_clk_sm; double mhz; double ms; };

template <typename F>
static Res run(F launch, int grid, int block, double ops_per_thread, int nsm) {
  uint32_t *out, *in; long long* cyc;
  cudaMalloc(&out, (size_t)grid * block * 4); cudaMalloc(&in, 1 << 20); cudaMalloc(&cyc, grid * 8);
  cudaMemset(in, 0x5a, 1 << 20);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  launch(out, in, cyc); cudaDeviceSynchronize();
  cudaEventRecord(e0);
  for (int r = 0; r < 5; r++) launch(out, in, cyc);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
  long long* h = (long long*)malloc(grid * 8); cudaMemcpy(h, cyc, grid * 8, cudaMemcpyDeviceToHost);
  double mx = 0; for (int i = 0; i < grid; i++) if (h[i] > mx) mx = (double)h[i];
  free(h); cudaFree(out); cudaFree(in); cudaFree(cyc);
  Res r;
  double total_ops = ops_per_thread * grid * block;
  // CTAs per SM resident together = grid/nsm (we always launch multiples of nsm that fit)
  r.per_clk_sm = total_ops / nsm / mx;            // thread-ops per clock per SM (in-kernel clock)
  r.ms = ms;
  r.mhz = mx / (ms * 1e3);                        // cycles / us
  return r;
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  int nsm = p.multiProcessorCount;
  printf("{\"gpu\": \"%s\", \"sms\": %d, \"results\": [\n", p.name, nsm);
  int first = 1;
  auto emit = [&](const char* name, int warps, Res r) {
    printf("%s {\"op\": \"%s\", \"warps_per_sm\": %d, \"thread_ops_per_clk_per_sm\": %.2f, \"eff_mhz\": %.0f, \"ms\": %.3f}",
           first ? "" : ",\n", name, warps, r.per_clk_sm, r.mhz, r.ms);
    first = 0;
  };
  int wlist[] = {4, 8, 16};   // <= 16 warps/SM so that every CTA of the grid is co-resident
  for (int wi = 0; wi < 3; wi++) {
    int warps = wlist[wi]; int block = 128; int cta_per_sm = warps / 4; int grid = nsm * cta_per_sm;
    emit("wide_chain4_x2(IMAD.WIDE.X)", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_wide_chain<2><<<grid, block>>>(o, i, c); }, grid, block, 2.0 * 4 * ITERS, nsm));
    emit("wide_chain4_x4(IMAD.WIDE.X)", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_wide_chain<4><<<grid, block>>>(o, i, c); }, grid, block, 4.0 * 4 * ITERS, nsm));
    emit("wide_chain4_x8(IMAD.WIDE.X)", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_wide_chain<8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("imad_lo", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<0, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("imad_hi", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<1, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("imad_wide_nocarry", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<2, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("imad_wide_pair_x8", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<6, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("imad_wide_pair_x16", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<6, 16><<<grid, block>>>(o, i, c); }, grid, block, 16.0 * 4 * ITERS, nsm));
    emit("mul_wide_no_addend", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<7, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("imad_wide_pair_plus_2_iadd", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<8, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("dfma", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<3, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("shfl", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<4, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS, nsm));
    emit("iadd_cc_pair", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_indep<5, 8><<<grid, block>>>(o, i, c); }, grid, block, 8.0 * 4 * ITERS * 2, nsm));
    emit("lds128", warps, run([&](uint32_t* o, const uint32_t* i, long long* c) { k_lds<<<grid, block, 16 * block * 16>>>(o, i, c); }, grid, block, 16.0 * ITERS, nsm));
  }
  printf("\n]}\n");
  return 0;
}
