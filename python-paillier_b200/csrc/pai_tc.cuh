// pai_tc.cuh -- digit Montgomery arithmetic modulo n^2 with the REDUCTIONS on the tensor cores (Hopper wgmma).
//
// Every Montgomery reduction multiplies a per-ciphertext number by a batch-wide constant twice:
//     m = T_lo * N' mod R        (N' = -n^-1 mod R)          and          hi = floor(m * n / R).
// In base-256 digits, for the 128 ciphertexts of a thread group (one warpgroup) at once, that is  [128 x D] x Toeplitz(const):
// wgmma.mma_async u8 x u8 -> s32 GEMMs (two m64 halves of the 128 rows, K = 32 digits per instruction, column sums
// <= D * 255^2 < 2^25; at D = 384 they pass 2^24, and tc_limbs8 keeps the high word of every shifted sum).  The
// accumulator fragments are computed 32 columns at a time and moved by warp shuffles to the lane that owns the row, which
// propagates the carries (ALU pipe) and has the quotient / the high half as ordinary 32-bit limbs again.  What stays on
// the integer-multiply pipe are only the products of two per-ciphertext numbers (x0*y0, x0*y1 + x1*y0): 100 instead of
// 228 tile products per squaring, 192 instead of 320 per multiplication at 2048-bit keys, and no quotient products.
//
// Exactness of the high half.  GEMM 2 produces the byte columns D-4 .. 2D-5 of m*n (the top three columns 2D-4 .. 2D-2
// are six scalar byte products).  The columns below D-4 are never computed: their sum I is < 1.004 * 256^(D-2), and the
// low half of m*n is KNOWN, m*n mod R = -T_lo mod R =: L.  With S the exactly propagated part (columns >= D-4),
// s = its guard limb (digits D-4 .. D-1) and l the top limb of L:   floor(m*n / R) = floor(S / R) + [s > l]
// (S mod R + I wraps past R exactly when the guard limb exceeds l; checked against integers in tests/test_tc_model.py).
//
// Data flow of one product Z = X*Y*R^-1 mod n^2 (digits X = x0 + n x1 etc., see pai_digit.cuh for the identity):
//   P1  T = x0*y0            (IMAD)   T_lo -> A (the group's MMA operand buffer, row = thread), T_hi -> park (L2)
//   G1  A x Toeplitz(N')     (tensor) E1: m -> A (digits == limb bytes: the buffer is both operand and limb array)
//   G2  A x Toeplitz(n)      (tensor) E2: t = T_hi + hi + [T_lo != 0] -> park;  carry = [t >= n];  A <- W = K - m
//   P2  B = x0*y1 + x1*y0 + W (IMAD)  B_lo -> A (over W, tile by tile), B_hi -> over x0 (dead tile by tile)
//   G1  A x Toeplitz(N')              E1: m' -> A
//   G2  A x Toeplitz(n)               E4: z = B_hi + hi' + ... (< 3n + 3) -> Z1 in place, reduced by digit_reduce3
//   Z0 = t - n*carry: park -> the buffer of x1.       Shared memory per ciphertext: 3 half-buffers (x0, x1, A).
//
// A CTA runs up to four independent groups of 128 threads (named barriers): while one group waits for its GEMMs and runs
// the ALU epilogues, the others keep the integer-multiply pipe busy.  PTX does not promise which rows of A a warp's share
// of a wgmma reads, so after every GEMM chunk the four warps of the group meet at their named barrier before any of them
// rewrites A (tc_ld32).
//
// Compiled twice like everything else: nvcc (sm_90a: wgmma inline PTX) and g++ -DPAI_HOSTSIM, where a "group" is TC_RL
// rows walked phase by phase and the GEMM is an integer loop over the very same operand layouts.
#pragma once
#include "pai_digit.cuh"

namespace pai {

#if defined(PAI_HOSTSIM)
constexpr int TC_RL = 2;                  // rows of a group the simulation walks (placed in varying 8-row groups of the layout)
#else
constexpr int TC_RL = 1;                  // the GPU thread owns one row; state lives in registers
#endif
#define TC_EACH_ROW for (int rw = 0; rw < TC_RL; rw++)
constexpr int TC_M = 128;                 // rows (ciphertexts) of a group = the M of two m64 wgmma halves

// ---- operand layouts (K-major, no swizzle: 8 x 16-byte core matrices) ---------------------------------------------
// A operand [128 x D]: digit k of row r.  Core matrix (r/8, k/16) at ((r/8) * (D/16) + k/16) * 128 bytes.
PAI_HD uint32_t tc_a_off(int D, int r, int k) {
  return ((uint32_t)(r >> 3) * (uint32_t)(D / 16) + (uint32_t)(k >> 4)) * 128u + (uint32_t)(r & 7) * 16u + (uint32_t)(k & 15);
}
// Toeplitz operands are stored as BANDS: for the K block kappa (digits 32 kappa .. 32 kappa + 31) the [D x 32] tile of
// Toeplitz(c)[j][k] = c[j - k + shift] only depends on j - 32 kappa, so all K blocks read windows of ONE [2D-32 x 32]
// matrix band[u][k'] = c[u - (D - 32) + shift - k'], window of block kappa = rows u0 .. u0 + D - 1, u0 = D - 32 - 32 kappa.
// 15 KB per constant at 2048-bit keys instead of a 64 KB D x D matrix.
PAI_HD int tc_band_rows(int NTH) { return 64 * NTH - 32; }
PAI_HD int tc_band_bytes(int NTH) { return 32 * tc_band_rows(NTH); }
PAI_HD uint32_t tc_band_off(int u, int kp) {
  return ((uint32_t)(u >> 3) * 2u + (uint32_t)(kp >> 4)) * 128u + (uint32_t)(u & 7) * 16u + (uint32_t)(kp & 15);
}
// global blob of one modulus for this path: [ band(N') | band(n) ]
PAI_HD int tc_blob_bytes(int NTH) { return 2 * tc_band_bytes(NTH); }

// single-thread setup: N' = -n^-1 mod 256^D, then the two bands.  scratch: 8*NTH limbs.
template <int NTH>
PAI_DEV void tc_setup(const uint32_t* N, uint8_t* blob, uint32_t* scratch) {
  const int D = 32 * NTH, L = 8 * NTH;
  inv_mod_2k(scratch, N, L);
  uint32_t c = 1;
  for (int i = 0; i < L; i++) { uint64_t v = (uint64_t)(~scratch[i]) + c; scratch[i] = (uint32_t)v; c = (uint32_t)(v >> 32); }
  const uint8_t* np = (const uint8_t*)scratch;       // little-endian limbs == base-256 digits
  const uint8_t* nb = (const uint8_t*)N;
  uint8_t* b1 = blob;
  uint8_t* b2 = blob + tc_band_bytes(NTH);
  const int U = tc_band_rows(NTH);
  for (int u = 0; u < U; u++)
    for (int kp = 0; kp < 32; kp++) {
      int i1 = u - (D - 32) - kp;                      // N'[j - k]
      int i2 = u + 28 - kp;                            // n[(D - 4 + j') - k]
      b1[tc_band_off(u, kp)] = (i1 >= 0 && i1 < D) ? np[i1] : 0;
      b2[tc_band_off(u, kp)] = (i2 >= 0 && i2 < D) ? nb[i2] : 0;
    }
}

// ---- per-group context -------------------------------------------------------------------------------------------
template <int NTH>
struct TcCtx {
  DigitEnv* dc;
  u4* X;                    // shared half-buffer of the low digit x0, interleaved: quad q of thread t at X[q * nthr + t]
  Opnd H1;                  // half-buffer of the high digit x1 of row 0 / this thread: shared (stride nthr) when it fits next
                            // to X for the number of groups wanted, else a slot of the thread's table strip in global memory
  u4* A;                    // this group's operand buffer (128 * D bytes, tc_a_off layout)
  const uint8_t* band[2];   // shared: band(N'), band(n)
  Opnd tbl;                 // window table of THIS thread (global, stride nthr); simulation: of row 0
  int slots;                // table entries; entry `slots` is the park slot
  int tid, nthr;            // thread index in the CTA / threads per CTA (simulation: 0 / TC_RL)
  int row0;                 // row of this thread inside the group (simulation: first of the TC_RL rows)
#if defined(PAI_HOSTSIM)
  int32_t tmem[TC_RL][512];
#else
  int which;                // operand band of the current reduction GEMM: 0 = N', 1 = n (see tc_ld32)
  int grp;                  // group index (named barrier 1 + grp)
  long long* prof;          // optional phase profile (PAI_TC_PROF): 16 cycle counters per warp, or null
#endif
};

// phase timing (development aid): adds the cycles since *t to counter i of this warp and restarts the clock
#if !defined(PAI_HOSTSIM)
#define TC_PROF_START(c, t) long long t = (c).prof ? clock64() : 0
#define TC_PROF(c, t, i) do { if ((c).prof) { long long n_ = clock64(); if ((threadIdx.x & 31) == 0) (c).prof[i] += n_ - t; t = n_; } } while (0)
#else
#define TC_PROF_START(c, t) (void)0
#define TC_PROF(c, t, i) (void)0
#endif

// Where the high digit x1 of the running value lives.  Shared memory next to x0 wherever that does not cost a group of
// the CTA; at 192 and 256 digits (1536/2048-bit n, the primes of 3072/4096-bit keys) a third group only fits when x1 moves
// to the thread's table strip in global memory (L2-resident: 256 B per thread), and the third group is worth more.
template <int NTH>
PAI_HD constexpr bool tc_x1_global() { return NTH == 6 || NTH == 8; }

template <int NTH>
PAI_DEV Opnd tc_h(const TcCtx<NTH>& c, int i, int rw) {
  Opnd o;
  if (i == 0) { o.p = c.X + c.tid + rw; o.s = c.nthr; }
  else { o.p = c.H1.p + rw; o.s = c.H1.s; }
  return o;
}
template <int NTH>
PAI_DEV Opnd tc_a(const TcCtx<NTH>& c, int rw) {
  const int r = c.row0 + rw;
  Opnd o; o.p = c.A + (size_t)(r >> 3) * (2 * NTH) * 8 + (r & 7); o.s = 8; return o;
}
template <int NTH>
PAI_DEV Opnd tc_tbl(const TcCtx<NTH>& c, int e, int half, int rw) {
  Opnd o; o.p = c.tbl.p + rw + ((size_t)e * 4 * NTH + (size_t)half * 2 * NTH) * c.tbl.s; o.s = c.tbl.s; return o;
}
template <int NTH>
PAI_DEV Opnd tc_park(const TcCtx<NTH>& c, int rw) { return tc_tbl<NTH>(c, c.slots, 0, rw); }
// the W slot (tc_x1_global only): entry slots + 2 of the strip (slots + 1 is the home of x1)
template <int NTH>
PAI_DEV Opnd tc_wslot(const TcCtx<NTH>& c, int rw) { return tc_tbl<NTH>(c, c.slots + 2, 0, rw); }
template <int NTH>
PAI_DEV SOpnd tc_xs(const TcCtx<NTH>& c, int rw) { return to_shared(tc_h<NTH>(c, 0, rw)); }
// x1 as the operand type of its home: shared-memory loads where it is in shared memory
template <int NTH>
PAI_DEV auto tc_x1(const TcCtx<NTH>& c, int rw) {
  if constexpr (tc_x1_global<NTH>()) return tc_h<NTH>(c, 1, rw);
  else return to_shared(tc_h<NTH>(c, 1, rw));
}
template <int NTH>
PAI_DEV SOpnd tc_as(const TcCtx<NTH>& c, int rw) { return to_shared(tc_a<NTH>(c, rw)); }

// state of one row between the phases of one product
struct TcRow {
  uint32_t ltop, nz, carry, wtop, ovf2;
};

// ---- tensor-core plumbing ------------------------------------------------------------------------------------------
#if !defined(PAI_HOSTSIM)
PAI_DEV uint32_t tc_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// K-major, no-swizzle shared-memory matrix descriptor: LBO = byte distance of core matrices along K, SBO = along M/N
PAI_DEV uint64_t tc_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo >> 4) & 0x3fff) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3fff) << 32;
  return d;
}
// d[64 x 32] (+)= A[64 x 32 digits] x B[32 digits x 32], unsigned 8-bit operands, s32 accumulators
PAI_DEV void tc_wgmma_n32(uint32_t d[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.u8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
        "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
PAI_DEV void tc_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
// x[i] for a lane-dependent i in 0..3 without indexing registers (which would put x in local memory)
PAI_DEV uint32_t tc_pick4(const uint32_t x0, const uint32_t x1, const uint32_t x2, const uint32_t x3, int i) {
  const uint32_t lo = (i & 1) ? x1 : x0, hi = (i & 1) ? x3 : x2;
  return (i & 2) ? hi : lo;
}
#endif

// 32 consecutive column sums of this thread's row, starting at column c0
template <int NTH>
PAI_DEV void tc_ld32(const TcCtx<NTH>& c, int rw, int c0, uint32_t v[32]) {
#if defined(PAI_HOSTSIM)
  for (int j = 0; j < 32; j++) v[j] = (uint32_t)c.tmem[rw][c0 + j];
#else
  // The columns c0 .. c0 + 31 of the GEMM c.which, computed now: both m64 halves, over the K blocks that reach them (both
  // Toeplitz operands are triangular: digit block kappa of A reaches only the columns j >= 32 kappa of A x T(N') and
  // only the columns j' < 32 kappa + 48 of A x T(n)).
  (void)rw;
  const int D = 32 * NTH, t = c0 >> 5;
  uint32_t acc[2][16];
  PAI_UNROLL
  for (int h = 0; h < 2; h++) {
    PAI_UNROLL
    for (int i = 0; i < 16; i++) acc[h][i] = 0;
  }
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
  const uint32_t a0 = tc_smem_u32(c.A), b0 = tc_smem_u32(c.band[c.which]);
  uint32_t more = 0;
  PAI_UNROLL
  for (int kap = 0; kap < NTH; kap++) {
    if (c.which == 0 ? kap > t : kap < t - 1) continue;
    const uint64_t db = tc_desc(b0 + (uint32_t)((D - 32 - 32 * kap + c0) / 8) * 256u, 128u, 256u);
    PAI_UNROLL
    for (int h = 0; h < 2; h++)
      tc_wgmma_n32(acc[h], tc_desc(a0 + (uint32_t)(h * 64 * D + kap * 256), 128u, (uint32_t)(D / 16) * 128u), db, more);
    more = 1;
  }
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  tc_bar_sync(1 + c.grp, TC_M);            // every warp's chunk is complete before any warp rewrites A (E1, E2, P2)
  // Fragment of lane L = 4 g + q: in 8-column block j, acc[h][4j + 2k' + e] = (row g + 8k' of the warp's 16 in half h,
  // column 8j + 2q + e).  Lane L owns the warp's row (L & 15) of half (L >> 4), i.e. local row g' + 8k with g' = L & 7,
  // k = L >> 3 (c.row0).  In round r it takes the column pair 2q' + (0, 1), q' = (r + k) & 3, from lane 4g' + q' -- which
  // sends, in that round, its pair of local row g' + 8((q' - r) & 3).
  const int lane = threadIdx.x & 31, qs = lane & 3, gd = lane & 7, kd = lane >> 3;
  PAI_UNROLL
  for (int j = 0; j < 4; j++) {
    uint32_t got[4][2];
    PAI_UNROLL
    for (int r = 0; r < 4; r++) {
      const int ks = (qs - r) & 3, src = 4 * gd + ((r + kd) & 3);
      PAI_UNROLL
      for (int e = 0; e < 2; e++) {
        const uint32_t s = tc_pick4(acc[0][4 * j + e], acc[0][4 * j + 2 + e], acc[1][4 * j + e], acc[1][4 * j + 2 + e], ks);
        got[r][e] = __shfl_sync(0xffffffffu, s, src);
      }
    }
    PAI_UNROLL
    for (int q = 0; q < 4; q++) {
      const int r = (q - kd) & 3;
      PAI_UNROLL
      for (int e = 0; e < 2; e++) v[8 * j + 2 * q + e] = tc_pick4(got[0][e], got[1][e], got[2][e], got[3][e], r);
    }
  }
#endif
}

// The group's GEMM: accumulator = A x window(band[which]).  All threads of the group call it.
template <int NTH>
PAI_DEV void tc_gemm(TcCtx<NTH>& c, int which) {
#if defined(PAI_HOSTSIM)
  const int D = 32 * NTH;
  const uint8_t* a = (const uint8_t*)c.A;
  TC_EACH_ROW {
    const int r = c.row0 + rw;
    for (int j = 0; j < D; j++) {
      uint32_t sum = 0;                                   // <= D * 255^2 < 2^25
      for (int kap = 0; kap < NTH; kap++) {
        const int u0 = D - 32 - 32 * kap;
        for (int h = 0; h < 2; h++) {                     // 16 contiguous digits of the row x 16 contiguous band bytes
          const uint8_t* pa = a + tc_a_off(D, r, 32 * kap + 16 * h);
          const uint8_t* pb = c.band[which] + tc_band_off(u0 + j, 16 * h);
          uint32_t s16 = 0;
          for (int t = 0; t < 16; t++) s16 += (uint32_t)pa[t] * pb[t];
          sum += s16;
        }
      }
      c.tmem[rw][j] = (int32_t)sum;
    }
  }
#else
  // the GEMM itself runs chunk by chunk as the epilogue reads it (tc_ld32); here the rows of A written through the generic
  // proxy are made visible to the tensor cores
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  tc_bar_sync(1 + c.grp, TC_M);
  c.which = which;
#endif
}

// eight 32-bit limbs from 32 byte-column sums (any 32-bit values) and the running carry.
// On the GPU this is spelled in funnel shifts and add-with-carry chains so that it runs on the ALU pipe: written as 64-bit
// C arithmetic ptxas turned the shifts into IMAD.WIDE (three per limb), i.e. onto the very pipe the products need.
// The high word of every shifted sum is kept: at D = 384 digits (3072-bit n) a column sum reaches 384 * 255^2 > 2^24, so
// v1 << 8 has a high part too.
PAI_DEV void tc_limbs8(const uint32_t v[32], uint32_t& carry, uint32_t out[8]) {
  PAI_UNROLL
  for (int j = 0; j < 8; j++) {
#if defined(PAI_HOSTSIM)
    uint64_t x = (uint64_t)v[4 * j] + ((uint64_t)v[4 * j + 1] << 8) + ((uint64_t)v[4 * j + 2] << 16) + ((uint64_t)v[4 * j + 3] << 24) + carry;
    out[j] = (uint32_t)x;
    carry = (uint32_t)(x >> 32);
#else
    uint32_t lo, hi;
    asm("{\n\t.reg .u32 t1, t2, t3, h1, h2, h3;\n\t"
        "shf.l.wrap.b32 t1, 0, %3, 8;\n\t"          // low word of v1 << 8
        "shf.r.wrap.b32 h1, %3, 0, 24;\n\t"         // v1 >> 24
        "shf.l.wrap.b32 t2, 0, %4, 16;\n\t"         // low word of v2 << 16
        "shf.r.wrap.b32 h2, %4, 0, 16;\n\t"         // v2 >> 16
        "shf.l.wrap.b32 t3, 0, %5, 24;\n\t"         // low word of v3 << 24
        "shf.r.wrap.b32 h3, %5, 0, 8;\n\t"          // v3 >> 8
        "add.cc.u32 %0, %2, t1;\n\t"
        "addc.u32 %1, h2, h3;\n\t"
        "add.cc.u32 %0, %0, t2;\n\t"
        "addc.u32 %1, %1, h1;\n\t"
        "add.cc.u32 %0, %0, t3;\n\t"
        "addc.u32 %1, %1, 0;\n\t"
        "add.cc.u32 %0, %0, %6;\n\t"
        "addc.u32 %1, %1, 0;\n\t}"
        : "=&r"(lo), "=&r"(hi)
        : "r"(v[4 * j]), "r"(v[4 * j + 1]), "r"(v[4 * j + 2]), "r"(v[4 * j + 3]), "r"(carry));
    out[j] = lo;
    carry = hi;
#endif
  }
}

// ---- phases ---------------------------------------------------------------------------------------------------------
PAI_DEV uint32_t tc_or8(const uint32_t v[8], int n) { uint32_t o = 0; for (int i = 0; i < n; i++) o |= v[i]; return o; }

// bookkeeping of a finished low half: nz = [lo != 0], ltop = top limb of (-lo mod R)
struct TcLow {
  uint32_t lowor, top;
};
PAI_DEV void tc_low_tile(TcLow& l, const uint32_t v[8], bool last) {
  if (!last) l.lowor |= tc_or8(v, 8);
  else { l.lowor |= tc_or8(v, 7); l.top = v[7]; }
}

// P1 (multiplication): T = x0 * y0;  T_lo -> A, T_hi + [T_lo != 0] -> park
template <int NTH, class XT>
PAI_FN void tc_prod1_mul(SOpnd A, Opnd P, XT x0, Opnd y0, TcRow* st) {
  Acc acc;
  acc_clear(acc);
  TcLow low; low.lowor = 0; low.top = 0;
  for (int k = 0; k < 2 * NTH; k++) {
    int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
    int hi = k < NTH ? k : NTH - 1;
    // y0 usually comes from the window table in L2: its next tile is requested one tile product ahead
    uint32_t yn[8];
    ld_tile(y0, k - lo, yn);
    for (int i = lo; i <= hi; i++) {
      uint32_t x[8], y[8];
      PAI_UNROLL
      for (int j = 0; j < 8; j++) y[j] = yn[j];
      if (i < hi) ld_tile(y0, k - i - 1, yn);
      ld_tile(x0, i, x);
      tile_mac(acc, x, y);
    }
    if (k == NTH) acc.C[0] += st->nz;
    uint32_t v[8];
    acc_resolve_low(acc, v);
    if (k < NTH) {
      st_tile(A, k, v);
      tc_low_tile(low, v, k == NTH - 1);
      if (k == NTH - 1) { st->nz = (low.lowor | low.top) != 0u; st->ltop = ~low.top + (low.lowor == 0u ? 1u : 0u); }
    } else {
      st_tile(P, k - NTH, v);
    }
    acc_shift8(acc);
  }
}

// r = a + small (8 limbs); returns the carry
PAI_DEV uint32_t add8_small(uint32_t r[8], const uint32_t a[8], uint32_t small) {
  uint32_t b[8];
  b[0] = small;
  PAI_UNROLL
  for (int i = 1; i < 8; i++) b[i] = 0;
  return add8(r, a, b);
}

// P1 (squaring): T = x0^2 = 2 * OFF + DIAG in two passes, so that the doubling is not paid per column:
//   pass A  OFF = sum_{i<j} a_i a_j B^(i+j): plain column scanning with ONE accumulator (the round-1 form kept a second
//           accumulator for the off-diagonal part and resolved, shifted and doubled it in every column), tiles parked
//           where the result will go (A / park);
//   pass B  the squares a_i^2 occupy the tile pairs (2i, 2i+1) without overlapping: T = 2*OFF + a_i^2 + carry, pair by pair.
template <int NTH>
PAI_FN void tc_prod1_sqr(SOpnd A, Opnd P, SOpnd x0, TcRow* st) {
  {
    Acc acc;
    acc_clear(acc);
    for (int k = 0; k < 2 * NTH; k++) {
      int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
      int hs = k == 0 ? -1 : (k - 1) / 2;
      for (int i = lo; i <= hs; i++) {
        uint32_t x[8], y[8];
        ld_tile(x0, i, x); ld_tile(x0, k - i, y);
        tile_mac(acc, x, y);
      }
      uint32_t v[8];
      acc_resolve_low(acc, v);
      if (k < NTH) st_tile(A, k, v);
      else st_tile(P, k - NTH, v);
      acc_shift8(acc);
    }
  }
  uint32_t carry = 0, topbit = 0;
  TcLow low; low.lowor = 0; low.top = 0;
  for (int i = 0; i < NTH; i++) {
    uint32_t dg[2][8];
    {
      Acc d;
      acc_clear(d);
      uint32_t x[8];
      ld_tile(x0, i, x);
      tile_mac(d, x, x);
      acc_resolve_low(d, dg[0]);
      acc_shift8(d);
      acc_resolve_low(d, dg[1]);
    }
    PAI_UNROLL
    for (int h = 0; h < 2; h++) {
      const int t = 2 * i + h;
      uint32_t o[8], o2[8], s1[8], v[8];
      if (t < NTH) ld_tile(A, t, o);
      else ld_tile(P, t - NTH, o);
      o2[0] = (o[0] << 1) | topbit;
      PAI_UNROLL
      for (int j = 1; j < 8; j++) o2[j] = (o[j] << 1) | (o[j - 1] >> 31);
      topbit = o[7] >> 31;
      if (t == NTH) carry += st->nz;                       // T_hi is parked with [T_lo != 0] already added
      uint32_t c1 = add8(s1, o2, dg[h]);
      uint32_t c2 = add8_small(v, s1, carry);
      carry = c1 + c2;
      if (t < NTH) {
        st_tile(A, t, v);
        tc_low_tile(low, v, t == NTH - 1);
        if (t == NTH - 1) { st->nz = (low.lowor | low.top) != 0u; st->ltop = ~low.top + (low.lowor == 0u ? 1u : 0u); }
      } else {
        st_tile(P, t - NTH, v);
      }
    }
  }
}

// E1: quotient m = (column sums of lo * N') mod R -> A (as limbs == digits).  Column block t of the product depends on the
// digit blocks 0 .. t of A only, so the blocks are read from the top down and each one's limbs, without the carry from
// below, replace digit block t as soon as no lower block needs it; a second pass adds the carries.
template <int NTH>
PAI_FN void tc_epi_m(const TcCtx<NTH>* c, int rw, SOpnd A) {
  uint32_t ovf[NTH];
  PAI_UNROLL
  for (int t = NTH - 1; t >= 0; t--) {
    uint32_t v[32], l[8];
    ovf[t] = 0;
    tc_ld32<NTH>(*c, rw, 32 * t, v);
    tc_limbs8(v, ovf[t], l);
    st_tile(A, t, l);
  }
  uint32_t carry = 0;
  PAI_UNROLL
  for (int t = 0; t < NTH; t++) {
    uint32_t l[8], r[8];
    ld_tile(A, t, l);
    const uint32_t cy = add8_small(r, l, carry);
    st_tile(A, t, r);
    carry = ovf[t] + cy;
  }
}

// the high half of m*n, one tile at a time: hi tile j = S-limbs 8j+1 .. 8j+8 (S-limb 0 is the guard limb), the very top
// limb from the three scalar columns.  Usage: tc_hi_begin, then tc_hi_tile for j = 0 .. NTH-1.
template <int NTH>
struct TcHi {
  uint32_t L[8];
  uint32_t carry;
  uint32_t cadd;          // [guard limb > ltop]
};
template <int NTH>
PAI_DEV void tc_hi_begin(const TcCtx<NTH>& c, int rw, uint32_t ltop, TcHi<NTH>& h) {
  uint32_t v[32];
  h.carry = 0;
  tc_ld32<NTH>(c, rw, 0, v);
  tc_limbs8(v, h.carry, h.L);
  h.cadd = h.L[0] > ltop ? 1u : 0u;
}
template <int NTH>
PAI_DEV void tc_hi_tile(const TcCtx<NTH>& c, int rw, int j, const SOpnd& m, const Opnd& N, TcHi<NTH>& h, uint32_t out[8]) {
  PAI_UNROLL
  for (int i = 0; i < 7; i++) out[i] = h.L[i + 1];
  if (j < NTH - 1) {
    uint32_t v[32];
    tc_ld32<NTH>(c, rw, 32 * (j + 1), v);
    tc_limbs8(v, h.carry, h.L);
    out[7] = h.L[0];
  } else {
    // byte columns 2D-4 .. 2D-2: products of the top three digits of m and n
    const uint32_t mt = ld_quad(m, 2 * NTH - 1).w, nt = N.p[(2 * NTH - 1) * N.s].w;
    const uint32_t m1 = (mt >> 8) & 0xffu, m2 = (mt >> 16) & 0xffu, m3 = mt >> 24;
    const uint32_t n1 = (nt >> 8) & 0xffu, n2 = (nt >> 16) & 0xffu, n3 = nt >> 24;
    const uint32_t e0 = m1 * n3 + m2 * n2 + m3 * n1, e1 = m2 * n3 + m3 * n2, e2 = m3 * n3;
    out[7] = h.carry + e0 + (e1 << 8) + (e2 << 16);            // < 2^32: floor(m n / R) < R
  }
}

// E2: t = (T_hi + [T_lo != 0]) + hi + [guard > ltop] -> park (in place); carry = [t >= n]; W = (KL - m) mod R -> A in place
// (x1 in shared memory) or -> the thread's W slot Wd in global memory (tc_x1_global); wtop
template <int NTH, bool WSLOT>
PAI_FN void tc_epi_t(const TcCtx<NTH>* c, int rw, SOpnd A, Opnd Ag, Opnd P, Opnd Wd, const DigitEnv* dc, TcRow* st) {
  constexpr int BL = NTH > 8 ? NTH / 2 : NTH;                   // park tiles loaded together (register budget)
  uint32_t th[BL][8];
  PAI_UNROLL
  for (int j = 0; j < BL; j++) ld_tile(P, j, th[j]);             // park loads in flight before the first GEMM chunk
  TcHi<NTH> h;
  tc_hi_begin<NTH>(*c, rw, st->ltop, h);
  uint32_t cy = h.cadd, bo = 0;
  PAI_UNROLL
  for (int j0 = 0; j0 < NTH; j0 += BL) {
    if (j0 > 0) {
      PAI_UNROLL
      for (int j = 0; j < BL; j++) ld_tile(P, j0 + j, th[j]);
    }
    PAI_UNROLL
    for (int jj = 0; jj < BL; jj++) {
      const int j = j0 + jj;
      uint32_t hi[8], t[8], nt[8], d[8];
      tc_hi_tile<NTH>(*c, rw, j, A, dc->N, h, hi);
      cy = add8c(t, th[jj], hi, cy);
      st_tile(P, j, t);
      ld_tile(dc->N, j, nt);
      bo = sub8b(d, t, nt, bo);
    }
  }
  st->carry = (cy != 0u) | (bo ^ 1u);
  uint32_t wb;
  if constexpr (WSLOT) {                                        // W goes to its global slot: A is about to hold x1' (P2)
    wb = 0;
    for (int t = 0; t < NTH; t++) {
      uint32_t a[8], b[8], r[8];
      ld_tile(dc->KL, t, a); ld_tile(A, t, b);
      wb = sub8b(r, a, b, wb);
      st_tile(Wd, t, r);
    }
  } else {
    wb = big_rsub<NTH>(Ag, dc->KL);
  }
  st->wtop = 1u - wb + st->carry;
}

// P2 (multiplication): B = x0*y1 + x1*y0 + W;  B_lo -> A (over W), B_hi (+ wtop + [B_lo != 0]) -> bh
template <int NTH, class XT, class X1T>
PAI_FN void tc_prod2_mul(SOpnd A, SOpnd bh, XT x0, X1T x1, Opnd y0, Opnd y1, TcRow* st) {
  Acc acc;
  acc_clear(acc);
  TcLow low; low.lowor = 0; low.top = 0;
  uint32_t nz2 = 0;
  for (int k = 0; k < 2 * NTH; k++) {
    int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
    int hi = k < NTH ? k : NTH - 1;
    uint32_t yn1[8], yn0[8];                             // table tiles requested one iteration ahead (L2 latency)
    ld_tile(y1, k - lo, yn1);
    ld_tile(y0, k - lo, yn0);
    if constexpr (tc_x1_global<NTH>()) {                 // ... and so are x1's when it lives in global memory
      uint32_t xn1[8];
      ld_tile(x1, lo, xn1);
      for (int i = lo; i <= hi; i++) {
        uint32_t x[8], xb[8], ya[8], yb[8];
        PAI_UNROLL
        for (int j = 0; j < 8; j++) { ya[j] = yn1[j]; yb[j] = yn0[j]; xb[j] = xn1[j]; }
        if (i < hi) { ld_tile(y1, k - i - 1, yn1); ld_tile(y0, k - i - 1, yn0); ld_tile(x1, i + 1, xn1); }
        ld_tile(x0, i, x);
        tile_mac(acc, x, ya);
        tile_mac(acc, xb, yb);
      }
    } else {
      for (int i = lo; i <= hi; i++) {
        uint32_t x[8], ya[8], yb[8];
        PAI_UNROLL
        for (int j = 0; j < 8; j++) { ya[j] = yn1[j]; yb[j] = yn0[j]; }
        if (i < hi) { ld_tile(y1, k - i - 1, yn1); ld_tile(y0, k - i - 1, yn0); }
        ld_tile(x0, i, x);
        tile_mac(acc, x, ya);
        ld_tile(x1, i, x);
        tile_mac(acc, x, yb);
      }
    }
    uint32_t v[8];
    if (k < NTH) {
      uint32_t w[8];
      ld_tile(A, k, w);
      acc_add_low(acc, w);
      acc_resolve_low(acc, v);
      st_tile(A, k, v);
      tc_low_tile(low, v, k == NTH - 1);
      if (k == NTH - 1) { nz2 = (low.lowor | low.top) != 0u; st->ltop = ~low.top + (low.lowor == 0u ? 1u : 0u); }
    } else {
      if (k == NTH) acc.C[0] += st->wtop + nz2;
      acc_resolve_low(acc, v);
      st_tile(bh, k - NTH, v);
    }
    acc_shift8(acc);
  }
  st->ovf2 = lo32(acc.E[0]) + acc.C[0];
}

// P2 (squaring): B = 2*x0*x1 + W.  x1 is dead after this phase, so it is doubled IN PLACE first (x1' = 2*x1 mod R, top bit
// tb) and the cross products run as a plain product x0 * x1' in one accumulator; tb * x0 * R enters as x0's tiles in the
// upper columns (each read right before B_hi overwrites it).
template <int NTH, class X1T>
PAI_FN void tc_prod2_sqr(SOpnd A, SOpnd bh, SOpnd x0, X1T x1, TcRow* st) {
  uint32_t tb = 0;
  for (int t = 0; t < NTH; t++) {
    uint32_t x[8], y[8];
    ld_tile(x1, t, x);
    y[0] = (x[0] << 1) | tb;
    PAI_UNROLL
    for (int j = 1; j < 8; j++) y[j] = (x[j] << 1) | (x[j - 1] >> 31);
    tb = x[7] >> 31;
    st_tile(x1, t, y);
  }
  Acc acc;
  acc_clear(acc);
  uint32_t nz2 = 0;
  TcLow low; low.lowor = 0; low.top = 0;
  for (int k = 0; k < 2 * NTH; k++) {
    int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
    int hc = k < NTH ? k : NTH - 1;
    for (int i = lo; i <= hc; i++) {
      uint32_t x[8], y[8];
      ld_tile(x0, i, x); ld_tile(x1, k - i, y);
      tile_mac(acc, x, y);
    }
    uint32_t v[8];
    if (k < NTH) {
      uint32_t w[8];
      ld_tile(A, k, w);
      acc_add_low(acc, w);
      acc_resolve_low(acc, v);
      st_tile(A, k, v);
      tc_low_tile(low, v, k == NTH - 1);
      if (k == NTH - 1) { nz2 = (low.lowor | low.top) != 0u; st->ltop = ~low.top + (low.lowor == 0u ? 1u : 0u); }
    } else {
      if (tb) {
        uint32_t w[8];
        ld_tile(x0, k - NTH, w);
        acc_add_low(acc, w);
      }
      if (k == NTH) acc.C[0] += st->wtop + nz2;
      acc_resolve_low(acc, v);
      st_tile(bh, k - NTH, v);
    }
    acc_shift8(acc);
  }
  st->ovf2 = lo32(acc.E[0]) + acc.C[0];
}

// ---- P2 of a squaring with x1 in global memory (tc_x1_global).  Read from L2 tile by tile, each tile of x1 would cross
// NTH times; instead x1' is staged in A for the phase -- A is free because E2 sent W to the thread's global W slot Q.
// W comes back one tile per column (requested before the column's products), B_lo replaces it there tile by tile, and moves
// to A (the MMA operand) when the products are done: 5*NTH tile transfers through L2 per phase instead of 10*NTH.
// (Multiplications keep W in A and prefetch x1: one in seven products, and the staging copies cost them more than they save.)
template <int NTH>
PAI_DEV void tc_q_to_a(SOpnd A, Opnd Q) {
  constexpr int BL = NTH % 4 == 0 ? 4 : (NTH % 3 == 0 ? 3 : (NTH % 2 == 0 ? 2 : 1));      // loads in flight together
  static_assert(NTH % BL == 0, "whole blocks only: a partial block would run past the row");
  PAI_UNROLL
  for (int j0 = 0; j0 < NTH; j0 += BL) {
    uint32_t t[BL][8];
    PAI_UNROLL
    for (int j = 0; j < BL; j++) ld_tile(Q, j0 + j, t[j]);
    PAI_UNROLL
    for (int j = 0; j < BL; j++) st_tile(A, j0 + j, t[j]);
  }
}
template <int NTH>
PAI_FN void tc_prod2_sqr_g(SOpnd A, Opnd Q, SOpnd bh, SOpnd x0, Opnd x1, TcRow* st) {
  uint32_t tb = 0;
  for (int t = 0; t < NTH; t++) {                       // x1' = 2*x1 mod R -> A, top bit tb
    uint32_t x[8], y[8];
    ld_tile(x1, t, x);
    y[0] = (x[0] << 1) | tb;
    PAI_UNROLL
    for (int j = 1; j < 8; j++) y[j] = (x[j] << 1) | (x[j - 1] >> 31);
    tb = x[7] >> 31;
    st_tile(A, t, y);
  }
  Acc acc;
  acc_clear(acc);
  uint32_t nz2 = 0;
  TcLow low; low.lowor = 0; low.top = 0;
  for (int k = 0; k < 2 * NTH; k++) {
    int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
    int hc = k < NTH ? k : NTH - 1;
    uint32_t w[8];
    if (k < NTH) ld_tile(Q, k, w);
    for (int i = lo; i <= hc; i++) {
      uint32_t x[8], y[8];
      ld_tile(x0, i, x); ld_tile(A, k - i, y);
      tile_mac(acc, x, y);
    }
    uint32_t v[8];
    if (k < NTH) {
      acc_add_low(acc, w);
      acc_resolve_low(acc, v);
      st_tile(Q, k, v);
      tc_low_tile(low, v, k == NTH - 1);
      if (k == NTH - 1) { nz2 = (low.lowor | low.top) != 0u; st->ltop = ~low.top + (low.lowor == 0u ? 1u : 0u); }
    } else {
      if (tb) {
        uint32_t xw[8];
        ld_tile(x0, k - NTH, xw);
        acc_add_low(acc, xw);
      }
      if (k == NTH) acc.C[0] += st->wtop + nz2;
      acc_resolve_low(acc, v);
      st_tile(bh, k - NTH, v);
    }
    acc_shift8(acc);
  }
  st->ovf2 = lo32(acc.E[0]) + acc.C[0];
  tc_q_to_a<NTH>(A, Q);
}

// E4: z = B_hi' + hi' + [guard > ltop] (+ ovf2 * R) < 3n + 3, reduced modulo n in place (bh)
template <int NTH>
PAI_FN void tc_epi_z(const TcCtx<NTH>* c, int rw, SOpnd A, SOpnd bh, Opnd bhg, const DigitEnv* dc, TcRow* st) {
  TcHi<NTH> h;
  tc_hi_begin<NTH>(*c, rw, st->ltop, h);
  uint32_t cy = h.cadd, b1 = 0, b2 = 0, b3 = 0;
  for (int j = 0; j < NTH; j++) {
    uint32_t hi[8], th[8], t[8], nt[8], d[8];
    tc_hi_tile<NTH>(*c, rw, j, A, dc->N, h, hi);
    ld_tile(bh, j, th);
    cy = add8c(t, th, hi, cy);
    st_tile(bh, j, t);
    ld_tile(dc->N, j, nt);   b1 = sub8b(d, t, nt, b1);
    ld_tile(dc->N2, j, nt);  b2 = sub8b(d, t, nt, b2);
    ld_tile(dc->N3, j, nt);  b3 = sub8b(d, t, nt, b3);
  }
  digit_reduce3<NTH>(bhg, *dc, st->ovf2 + cy, b1, b2, b3);
}

// Z0 = t - (n & mask): park -> shared half-buffer, all park loads issued together (one L2 round trip, not NTH)
template <int NTH>
PAI_FN void tc_z0_copy(SOpnd dst, Opnd P, Opnd N, uint32_t mask) {
  constexpr int BL = NTH > 8 ? NTH / 2 : NTH;
  uint32_t bo = 0;
  PAI_UNROLL
  for (int j0 = 0; j0 < NTH; j0 += BL) {
    uint32_t t[BL][8];
    PAI_UNROLL
    for (int j = 0; j < BL; j++) ld_tile(P, j0 + j, t[j]);
    PAI_UNROLL
    for (int j = 0; j < BL; j++) {
      uint32_t y[8], r[8];
      ld_tile(N, j0 + j, y);
      PAI_UNROLL
      for (int i = 0; i < 8; i++) y[i] &= mask;
      bo = sub8b(r, t[j], y, bo);
      st_tile(dst, j0 + j, r);
    }
  }
}

// ---- one product, all phases.  Operand resolvers map a row to its operand (rows differ only in their base address):
//   x0: low digit of the first factor (the shared buffer X, or a generic operand for rows read straight from global
//   memory); x1: its high digit (generic); y0, y1: digits of the second factor (generic; ignored for SQR).
//   Result: Z0 in X (buffer 0), Z1 in buffer 1 -- Z1 is built in X (over x0, whose tiles are dead by then), moved to
//   buffer 1 at the end, and Z0 = t - n*carry comes in from the park slot.
template <int NTH, bool SQR, class FX0, class FX1, class FY0, class FY1>
PAI_DEV void tc_op(TcCtx<NTH>& c, FX0 x0, FX1 x1, FY0 y0, FY1 y1) {
  TcRow st[TC_RL];
  TC_PROF_START(c, t0);
  TC_EACH_ROW {
    st[rw].nz = 0;
    if constexpr (SQR) tc_prod1_sqr<NTH>(tc_as<NTH>(c, rw), tc_park<NTH>(c, rw), x0(rw), &st[rw]);
    else tc_prod1_mul<NTH>(tc_as<NTH>(c, rw), tc_park<NTH>(c, rw), x0(rw), y0(rw), &st[rw]);
  }
  TC_PROF(c, t0, SQR ? 0 : 8);
  tc_gemm<NTH>(c, 0);
  TC_PROF(c, t0, 1);
  TC_EACH_ROW tc_epi_m<NTH>(&c, rw, tc_as<NTH>(c, rw));
  TC_PROF(c, t0, 2);
  tc_gemm<NTH>(c, 1);
  TC_PROF(c, t0, 3);
  constexpr bool SWAP = SQR && tc_x1_global<NTH>();      // squarings with x1 in global memory stage it in A (tc_prod2_sqr_g)
  TC_EACH_ROW tc_epi_t<NTH, SWAP>(&c, rw, tc_as<NTH>(c, rw), tc_a<NTH>(c, rw), tc_park<NTH>(c, rw), tc_wslot<NTH>(c, rw), c.dc, &st[rw]);
  TC_PROF(c, t0, 4);
  TC_EACH_ROW {
    if constexpr (SWAP) tc_prod2_sqr_g<NTH>(tc_as<NTH>(c, rw), tc_wslot<NTH>(c, rw), tc_xs<NTH>(c, rw), x0(rw), x1(rw), &st[rw]);
    else if constexpr (SQR) tc_prod2_sqr<NTH>(tc_as<NTH>(c, rw), tc_xs<NTH>(c, rw), x0(rw), x1(rw), &st[rw]);
    else tc_prod2_mul<NTH>(tc_as<NTH>(c, rw), tc_xs<NTH>(c, rw), x0(rw), x1(rw), y0(rw), y1(rw), &st[rw]);
  }
  TC_PROF(c, t0, SQR ? 5 : 9);
  tc_gemm<NTH>(c, 0);
  TC_PROF(c, t0, 1);
  TC_EACH_ROW tc_epi_m<NTH>(&c, rw, tc_as<NTH>(c, rw));
  TC_PROF(c, t0, 2);
  tc_gemm<NTH>(c, 1);
  TC_PROF(c, t0, 3);
  TC_EACH_ROW tc_epi_z<NTH>(&c, rw, tc_as<NTH>(c, rw), tc_xs<NTH>(c, rw), tc_h<NTH>(c, 0, rw), c.dc, &st[rw]);
  TC_PROF(c, t0, 6);
  TC_EACH_ROW {
    big_copy<NTH>(tc_h<NTH>(c, 1, rw), tc_h<NTH>(c, 0, rw));                                     // Z1 -> buffer 1
    tc_z0_copy<NTH>(tc_xs<NTH>(c, rw), tc_park<NTH>(c, rw), c.dc->N, 0u - st[rw].carry);        // Z0 -> X
  }
  TC_PROF(c, t0, 7);
#if !defined(PAI_HOSTSIM)
  if (c.prof && (threadIdx.x & 31) == 0) c.prof[SQR ? 10 : 11] += 1;
#endif
}

// in-place forms: (x0, x1) in buffers (0, 1)  ->  (Z0, Z1) in buffers (0, 1)
template <int NTH>
PAI_DEV void tc_sqr_inplace(TcCtx<NTH>& c) {
  auto X = [&](int rw) { return tc_xs<NTH>(c, rw); };
  auto Y = [&](int rw) { return tc_x1<NTH>(c, rw); };
  auto G = [&](int rw) { return tc_h<NTH>(c, 1, rw); };
  tc_op<NTH, true>(c, X, Y, G, G);
}
template <int NTH, class FY0, class FY1>
PAI_DEV void tc_mul_inplace(TcCtx<NTH>& c, FY0 y0, FY1 y1) {
  auto X = [&](int rw) { return tc_xs<NTH>(c, rw); };
  auto Y = [&](int rw) { return tc_x1<NTH>(c, rw); };
  tc_op<NTH, false>(c, X, Y, y0, y1);
}
template <int NTH>
PAI_DEV void tc_tbl_store(TcCtx<NTH>& c, int e) {                 // T[e] = (buffer 0, buffer 1)
  TC_EACH_ROW {
    big_copy<NTH>(tc_tbl<NTH>(c, e, 0, rw), tc_h<NTH>(c, 0, rw));
    big_copy<NTH>(tc_tbl<NTH>(c, e, 1, rw), tc_h<NTH>(c, 1, rw));
  }
}
template <int NTH>
PAI_DEV void tc_tbl_load(TcCtx<NTH>& c, int e) {                  // (buffer 0, buffer 1) = T[e]
  TC_EACH_ROW {
    big_copy<NTH>(tc_h<NTH>(c, 0, rw), tc_tbl<NTH>(c, e, 0, rw));
    big_copy<NTH>(tc_h<NTH>(c, 1, rw), tc_tbl<NTH>(c, e, 1, rw));
  }
}
template <int NTH>
PAI_DEV void tc_set_one(TcCtx<NTH>& c) {                          // (buffer 0, buffer 1) = Montgomery one
  TC_EACH_ROW { big_copy<NTH>(tc_h<NTH>(c, 0, rw), c.dc->ONEM.d0); big_copy<NTH>(tc_h<NTH>(c, 1, rw), c.dc->ONEM.d1); }
}

// Sliding-window exponentiation with the host-built program (see dpow_prog): base in buffers (0, 1), result likewise.
template <int NTH>
PAI_DEV void tc_pow_prog(TcCtx<NTH>& c, const uint32_t* prog, int nops, int nodd) {
  tc_tbl_store<NTH>(c, 0);                                                // T[0] = base
  if (nodd > 1) {
    tc_sqr_inplace<NTH>(c);
    tc_tbl_store<NTH>(c, nodd);                                           // base^2
    tc_tbl_load<NTH>(c, 0);
    for (int k = 1; k < nodd; k++) {                                      // T[k] = T[k-1] * base^2
      tc_mul_inplace<NTH>(c, [&](int rw) { return tc_tbl<NTH>(c, nodd, 0, rw); }, [&](int rw) { return tc_tbl<NTH>(c, nodd, 1, rw); });
      tc_tbl_store<NTH>(c, k);
    }
  }
  tc_tbl_load<NTH>(c, (int)(prog[0] & 0xffffu));
  for (int i = 1; i < nops; i++) {
    const uint32_t op = prog[i];
    const int nsq = (int)(op >> 16), idx = (int)(op & 0xffffu);
    for (int s = 0; s < nsq; s++) tc_sqr_inplace<NTH>(c);
    if (idx != 0xffff)
      tc_mul_inplace<NTH>(c, [&](int rw) { return tc_tbl<NTH>(c, idx, 0, rw); }, [&](int rw) { return tc_tbl<NTH>(c, idx, 1, rw); });
  }
}

// plain number Z0 + n*Z1 of the digits in buffers (0, 1) -> out_row(rw) (a scratch table entry for padding rows)
template <int NTH, class FOUT>
PAI_DEV void tc_store_plain(TcCtx<NTH>& c, FOUT out_row, const bool* store) {
  TC_EACH_ROW {
    DNum z; z.d0 = tc_h<NTH>(c, 0, rw); z.d1 = tc_h<NTH>(c, 1, rw);
    Opnd o;
    if (store[rw]) { o.p = (u4*)out_row(rw); o.s = 1; }
    else o = tc_tbl<NTH>(c, 0, 0, rw);                                   // scratch: table entry 0 (2*NTH tiles)
    digits_to_plain<NTH>(o, z, c.dc->N);
  }
}

// raw_encrypt (phe/paillier.py:102-139) for the rows of one group: c = (1 + n*m) * r^n mod n^2.
//   g: global row index of every row of the group (clamped to batch - 1), store: whether it is a real row.
template <int NTH>
PAI_DEV void tc_encrypt_rows(TcCtx<NTH>& c, const uint32_t* prog, int nops, int nodd, const uint32_t* m, const uint32_t* r,
                             uint32_t* out, const long* g, const bool* store) {
  const DigitEnv& dc = *c.dc;
  const int ln = 8 * NTH, lc = 16 * NTH;
  // (r, 0) * RR: enter the Montgomery domain
  tc_op<NTH, false>(
      c, [&](int rw) { Opnd o; o.p = (u4*)(r + g[rw] * ln); o.s = 1; return o; }, [&](int) { return dc.ZERO; },
      [&](int) { return dc.RR.d0; }, [&](int) { return dc.RR.d1; });
  if (nops <= 0) tc_set_one<NTH>(c);                                      // exponent 0 -> Montgomery one
  else tc_pow_prog<NTH>(c, prog, nops, nodd);
  // times the PLAIN digit pair (1, m) of the nude ciphertext 1 + n*m: leaves the domain
  tc_mul_inplace<NTH>(c, [&](int) { return dc.ONE; }, [&](int rw) { Opnd o; o.p = (u4*)(m + g[rw] * ln); o.s = 1; return o; });
  tc_store_plain<NTH>(c, [&](int rw) { return out + g[rw] * lc; }, store);
}

// ------------------------------------------------------------------------------------------------
// Fixed windows of W bits (secret exponent shared by the batch: no digit is skipped, or per-element exponents with a
// group-uniform window count); the 2^W-entry tables live in global memory.
// table of powers of the base in buffers (0, 1) at entries e0 .. e0 + 2^W - 1: T[0] = 1, T[1] = base, T[i] = T[i-1] * base
template <int NTP, int W>
PAI_DEV void tc_build_table(TcCtx<NTP>& c, int e0) {
  const DigitEnv& dc = *c.dc;
  TC_EACH_ROW { big_copy<NTP>(tc_tbl<NTP>(c, e0, 0, rw), dc.ONEM.d0); big_copy<NTP>(tc_tbl<NTP>(c, e0, 1, rw), dc.ONEM.d1); }
  tc_tbl_store<NTP>(c, e0 + 1);
  tc_sqr_inplace<NTP>(c);
  tc_tbl_store<NTP>(c, e0 + 2);
  for (int i = 3; i < (1 << W); i++) {
    tc_mul_inplace<NTP>(c, [&](int rw) { return tc_tbl<NTP>(c, e0 + 1, 0, rw); }, [&](int rw) { return tc_tbl<NTP>(c, e0 + 1, 1, rw); });
    tc_tbl_store<NTP>(c, e0 + i);
  }
}
// (buffer 0, buffer 1) = entry e(rw) of the table, e differing per row
template <int NTP, class FE>
PAI_DEV void tc_tbl_load_f(TcCtx<NTP>& c, FE e) {
  TC_EACH_ROW {
    const int d = e(rw);
    big_copy<NTP>(tc_h<NTP>(c, 0, rw), tc_tbl<NTP>(c, d, 0, rw));
    big_copy<NTP>(tc_h<NTP>(c, 1, rw), tc_tbl<NTP>(c, d, 1, rw));
  }
}
template <int NTP, int W, class FD>
PAI_DEV void tc_pow_fixed_f(TcCtx<NTP>& c, FD digit, int nwin) {                // digit(rw, window index) -> table entry of row rw
  tc_build_table<NTP, W>(c, 0);
  tc_tbl_load_f<NTP>(c, [&](int rw) { return digit(rw, nwin - 1); });
  for (int wi = nwin - 2; wi >= 0; wi--) {
    for (int s = 0; s < W; s++) tc_sqr_inplace<NTP>(c);
    tc_mul_inplace<NTP>(c, [&](int rw) { return tc_tbl<NTP>(c, digit(rw, wi), 0, rw); },
                        [&](int rw) { return tc_tbl<NTP>(c, digit(rw, wi), 1, rw); });
  }
}
template <int NTP, int W>
PAI_DEV void tc_pow_fixed(TcCtx<NTP>& c, const uint32_t* e, int nl, int nwin) {
  tc_pow_fixed_f<NTP, W>(c, [&](int, int wi) { return (int)exp_digit(e, nl, wi * W, W); }, nwin);
}

// buffers (0, 1) <- Montgomery digit form of the plain 2*NTH-tile numbers base_row(rw) = c_0 + c_1*R:
// (c_0, 0) * R^2 + (c_1, 0) * R^3, accumulated in table entry `tmp`.
template <int NTH, class FROW>
PAI_DEV void tc_enter_wide(TcCtx<NTH>& c, FROW base_row, int tmp) {
  const DigitEnv& dc = *c.dc;
  for (int i = 0; i < 2; i++) {
    const DNum E = i == 0 ? dc.RR : dc.E3;
    tc_op<NTH, false>(
        c, [&](int rw) { Opnd o; o.p = (u4*)(base_row(rw) + (size_t)i * 8 * NTH); o.s = 1; return o; }, [&](int) { return dc.ZERO; },
        [&](int) { return E.d0; }, [&](int) { return E.d1; });
    if (i == 0) tc_tbl_store<NTH>(c, tmp);
    else TC_EACH_ROW {
      DNum acc, add;
      acc.d0 = tc_tbl<NTH>(c, tmp, 0, rw); acc.d1 = tc_tbl<NTH>(c, tmp, 1, rw);
      add.d0 = tc_h<NTH>(c, 0, rw); add.d1 = tc_h<NTH>(c, 1, rw);
      dadd<NTH>(acc, add, dc.N);
    }
  }
  tc_tbl_load<NTH>(c, tmp);
}
// leave the domain and write the plain number to out_row(rw)
template <int NTH, class FOUT>
PAI_DEV void tc_exit_plain(TcCtx<NTH>& c, FOUT out_row, const bool* store) {
  const DigitEnv& dc = *c.dc;
  tc_mul_inplace<NTH>(c, [&](int) { return dc.ONE; }, [&](int) { return dc.ZERO; });
  tc_store_plain<NTH>(c, out_row, store);
}

// c^k mod n^2 with per-element exponents (EncryptedNumber._raw_mul, phe/paillier.py:749-751) -- prog_powmod_digit on
// the tensor-core path.  base rows: plain ciphertexts (2*NTH tiles = c_0 + c_1*R); nwin is uniform over the group.
template <int NTH, int W>
PAI_DEV void tc_powmod_rows(TcCtx<NTH>& c, const uint32_t* base, const uint32_t* exp, int nl, int nwin, uint32_t* out,
                            const long* g, const bool* store) {
  const int lc = 16 * NTH;
  tc_enter_wide<NTH>(c, [&](int rw) { return base + g[rw] * lc; }, 0);
  if (nwin <= 0) tc_set_one<NTH>(c);
  else tc_pow_fixed_f<NTH, W>(c, [&](int rw, int wi) { return (int)exp_digit(exp + g[rw] * nl, nl, wi * W, W); }, nwin);
  tc_exit_plain<NTH>(c, [&](int rw) { return out + g[rw] * lc; }, store);
}

// prod_i c_i^(k_i) mod n^2 over the `gsz` elements of one row's group -- Straus' simultaneous exponentiation: one table of
// 2^W powers per element, ONE chain of squarings shared by the whole group (the encrypted dot product of
// examples/logistic_regression_encrypted_model.py:170-180 costs (2 + 2^W - 1 + nwin) products per element instead of
// (2 + 2^W - 1 + nwin * (W + 1))).  Elements past the end of the batch count as exponent 0.  Table entries of element i:
// 2^W * i ...; the entry after the last table is the entry scratch (then the park slot and, maybe, buffer 1).
template <int NTH, int W>
PAI_DEV void tc_straus_rows(TcCtx<NTH>& c, const uint32_t* base, const uint32_t* exp, int nl, int gsz, int nwin, long batch,
                            uint32_t* out, const long* g, const bool* store) {
  const int lc = 16 * NTH;
  const int tmp = gsz << W;
  auto elem = [&](int rw, int i) { long j = g[rw] * gsz + i; return j < batch ? j : batch - 1; };
  auto digit = [&](int rw, int i, int wi) {
    long j = g[rw] * gsz + i;
    return j < batch ? (int)exp_digit(exp + j * nl, nl, wi * W, W) : 0;
  };
  for (int i = 0; i < gsz; i++) {
    tc_enter_wide<NTH>(c, [&](int rw) { return base + elem(rw, i) * lc; }, tmp);
    tc_build_table<NTH, W>(c, i << W);
  }
  if (nwin <= 0) {
    tc_set_one<NTH>(c);
  } else {
    for (int wi = nwin - 1; wi >= 0; wi--) {
      if (wi < nwin - 1) for (int s = 0; s < W; s++) tc_sqr_inplace<NTH>(c);
      for (int i = 0; i < gsz; i++) {
        if (wi == nwin - 1 && i == 0) tc_tbl_load_f<NTH>(c, [&](int rw) { return digit(rw, 0, wi); });
        else tc_mul_inplace<NTH>(c, [&](int rw) { return tc_tbl<NTH>(c, (i << W) + digit(rw, i, wi), 0, rw); },
                                 [&](int rw) { return tc_tbl<NTH>(c, (i << W) + digit(rw, i, wi), 1, rw); });
      }
    }
  }
  tc_exit_plain<NTH>(c, [&](int rw) { return out + g[rw] * lc; }, store);
}

// ------------------------------------------------------------------------------------------------
// raw_decrypt with CRT (phe/paillier.py:328-374) on the tensor-core path: the same program as prog_decrypt_digit
// (pai_digit.cuh), every product modulo p^2 / q^2 through tc_op.
// one prime side: m_x = L(c^(x-1) mod x^2) * h mod x  -> NTP tiles in the shared buffer X (buffer 0)
template <int NTP, int W>
PAI_DEV void tc_decrypt_half(TcCtx<NTP>& c, DSideC<NTP>& S, const uint8_t* bands, const uint32_t* cbase, const long* g) {
  DigitEnv& dc = S.dc;
  c.dc = &dc;
  c.band[0] = bands;
  c.band[1] = bands + tc_band_bytes(NTP);
  const int lc = 32 * NTP;
  const DNum Ek[4] = {dc.RR, dc.E3, dc.E4, dc.E5};
  // X = c * R mod x^2 from the four NTP-tile pieces of c (accumulated in table entry 0)
  for (int i = 0; i < 4; i++) {
    tc_op<NTP, false>(
        c, [&](int rw) { Opnd o; o.p = (u4*)(cbase + g[rw] * lc + (size_t)i * 8 * NTP); o.s = 1; return o; }, [&](int) { return dc.ZERO; },
        [&](int) { return Ek[i].d0; }, [&](int) { return Ek[i].d1; });
    if (i == 0) tc_tbl_store<NTP>(c, 0);
    else TC_EACH_ROW {
      DNum acc, add;
      acc.d0 = tc_tbl<NTP>(c, 0, 0, rw); acc.d1 = tc_tbl<NTP>(c, 0, 1, rw);
      add.d0 = tc_h<NTP>(c, 0, rw); add.d1 = tc_h<NTP>(c, 1, rw);
      dadd<NTP>(acc, add, dc.N);
    }
  }
  tc_tbl_load<NTP>(c, 0);
  if (S.nwin <= 0) tc_set_one<NTP>(c);
  else tc_pow_fixed<NTP, W>(c, S.e, 8 * NTP, S.nwin);
  tc_mul_inplace<NTP>(c, [&](int) { return dc.ONE; }, [&](int) { return dc.ZERO; });          // plain digits u = u0 + x*u1
  TC_EACH_ROW {
    Opnd u0 = tc_h<NTP>(c, 0, rw), u1 = tc_h<NTP>(c, 1, rw);
    // L(u) = (u-1)//x = u1 if u0 >= 1;  u0 == 0: u1 - 1, and -1 = x - 1 (mod x) if u1 == 0   (pai_digit.cuh)
    uint32_t u0z = big_is_zero<NTP>(u0);
    uint32_t u1z = big_is_zero<NTP>(u1);
    big_sub_masked<NTP>(u1, u1, dc.ONE, 0u - (u0z & (u1z ^ 1u)));
    const uint32_t sel = u0z & u1z;
    for (int t = 0; t < NTP; t++) {
      uint32_t l[8], n[8];
      ld_tile(u1, t, l); ld_tile(dc.N, t, n);
      if (t == 0) n[0] -= 1u;
      PAI_UNROLL
      for (int i = 0; i < 8; i++) l[i] = sel ? n[i] : l[i];
      st_tile(u1, t, l);
    }
    mont_mul<NTP>(u0, u1, S.hM, dc.N, dc.NI);                              // L * h mod x  (over u0's buffer)
  }
}

template <int NTP, int W>
PAI_DEV void tc_decrypt_rows(TcCtx<NTP>& c, DSideC<NTP>& P, DSideC<NTP>& Qs, const Opnd& pinvqM, const uint8_t* bands,
                             const uint32_t* cbase, uint32_t* out, const long* g, const bool* store) {
  const int ln = 16 * NTP;
  tc_decrypt_half<NTP, W>(c, P, bands, cbase, g);
  TC_EACH_ROW { if (store[rw]) store_row(out + g[rw] * ln, tc_h<NTP>(c, 0, rw), 2 * NTP); }      // m_p -> low half of the row
  tc_decrypt_half<NTP, W>(c, Qs, bands + 2 * tc_band_bytes(NTP), cbase, g);
  TC_EACH_ROW {
    uint32_t* out_row = out + g[rw] * ln;
    Opnd mq = tc_h<NTP>(c, 0, rw), mp = tc_a<NTP>(c, rw), uo = tc_h<NTP>(c, 1, rw);
    if (store[rw]) load_row(mp, out_row, 2 * NTP, 2 * NTP);
    else big_copy<NTP>(mp, mq);
    // u = (m_q - m_p) * p^-1 mod q     (m_p < p < q, m_q < q)
    uint32_t bo = big_sub_masked<NTP>(mq, mq, mp, 0xffffffffu);
    big_add_masked<NTP>(mq, mq, Qs.dc.N, 0u - bo);
    mont_mul<NTP>(uo, mq, pinvqM, Qs.dc.N, Qs.dc.NI);
    // m = m_p + u * p : the product goes straight to the output row (a scratch table entry for padding rows)
    Opnd o;
    if (store[rw]) { o.p = (u4*)out_row; o.s = 1; }
    else o = tc_tbl<NTP>(c, 0, 0, rw);
    big_mul<NTP, NTP, 2 * NTP>(o, uo, P.dc.N, 0u);
    uint32_t cy = 0;
    for (int t = 0; t < 2 * NTP; t++) {
      uint32_t x[8], b[8], r[8];
      ld_tile(o, t, x);
      if (t < NTP) ld_tile(mp, t, b);
      else { PAI_UNROLL for (int i = 0; i < 8; i++) b[i] = 0; }
      cy = add8c(r, x, b, cy);
      st_tile(o, t, r);
    }
  }
}

}  // namespace pai
