// pai_core.cuh -- multi-precision primitives of the H100 Paillier engine.
//
// One THREAD owns one big integer ("instance").  Numbers are little-endian arrays of 32-bit limbs
// grouped in TILES of 8 limbs (256 bit).  Operands live in shared memory in an interleaved layout
// (quad q of thread t at  base[q * nthreads + t], 16 bytes each) so that every LDS.128/STS.128 of
// a warp is conflict free; tile products run in registers as chains of IMAD.WIDE.U32(.X) that
// ptxas fuses from  mad.lo.cc / madc.hi.cc  pairs (verified with cuobjdump on sm_90a).
//
// Everything in this header is written once and compiled twice:
//   * by nvcc for sm_90a (the product), and
//   * by g++ with -DPAI_HOSTSIM (tests/hostsim: a TEST-ONLY build that runs the very same
//     templates on the CPU, one simulated thread at a time, so the algorithms can be checked
//     against the oracle in the GPU-less build container).  The product never loads that build.
//
// Reference semantics implemented on top of these primitives (see pai_kernels.cuh):
//   powmod  phe/util.py:38-50      mulmod  phe/util.py:53-64      invert  phe/util.py:85-103
#pragma once
#include <stdint.h>

#if defined(PAI_HOSTSIM)
#define PAI_DEV static inline
#define PAI_FN static
#define PAI_HD static inline
#define PAI_MEM inline
struct pai_u4 { uint32_t x, y, z, w; };
typedef pai_u4 u4;
#define PAI_UNROLL
#else
#define PAI_DEV __device__ __forceinline__
#define PAI_FN __device__ __noinline__
#define PAI_HD __host__ __device__ __forceinline__
#define PAI_MEM __device__ __forceinline__
typedef uint4 u4;
#define PAI_UNROLL _Pragma("unroll")
#endif

namespace pai {

static const int TILE = 8;  // limbs per tile

// CTA barrier used only to keep the warps of a CTA on the same ladder step (instruction-cache locality);
// a no-op in the CPU simulation, where threads run one after the other.
PAI_DEV void cta_step_sync() {
#if !defined(PAI_HOSTSIM)
  __syncthreads();
#endif
}

// ------------------------------------------------------------------------------------------------
// Operand descriptor: quad q (4 limbs) is at p[q * s].
//   per-thread operand in the interleaved shared/global layout: p = base + tid, s = nthreads
//   broadcast operand (per-key constant, same for all threads):  p = base,       s = 1
struct Opnd {
  u4* p;
  int s;
};

PAI_DEV void ld_tile(const Opnd& o, int t, uint32_t a[8]) {
  u4 q0 = o.p[(2 * t) * o.s];
  u4 q1 = o.p[(2 * t + 1) * o.s];
  a[0] = q0.x; a[1] = q0.y; a[2] = q0.z; a[3] = q0.w;
  a[4] = q1.x; a[5] = q1.y; a[6] = q1.z; a[7] = q1.w;
}
PAI_DEV void st_tile(const Opnd& o, int t, const uint32_t a[8]) {
  u4 q0, q1;
  q0.x = a[0]; q0.y = a[1]; q0.z = a[2]; q0.w = a[3];
  q1.x = a[4]; q1.y = a[5]; q1.z = a[6]; q1.w = a[7];
  o.p[(2 * t) * o.s] = q0;
  o.p[(2 * t + 1) * o.s] = q1;
}
PAI_DEV void zero_tile(const Opnd& o, int t) {
  u4 z; z.x = z.y = z.z = z.w = 0;
  o.p[(2 * t) * o.s] = z;
  o.p[(2 * t + 1) * o.s] = z;
}

// Shared-memory operand addressed through the 32-bit shared window (LDS.128 / STS.128 with 32-bit address arithmetic)
// instead of a generic 64-bit pointer: the hot loops of pai_tc.cuh load four quads per tile product, and with generic
// pointers every one of them cost an IMAD.WIDE for the address on the very pipe the products run on, plus the longer
// generic-load path.  The CPU simulation has no address spaces: there an SOpnd is an Opnd.
#if !defined(PAI_HOSTSIM)
struct SOpnd {
  uint32_t a;      // shared address of quad 0
  uint32_t sb;     // byte distance between consecutive quads
};
PAI_DEV SOpnd to_shared(const Opnd& o) {
  SOpnd s;
  s.a = (uint32_t)__cvta_generic_to_shared(o.p);
  s.sb = (uint32_t)o.s * 16u;
  return s;
}
PAI_DEV u4 lds_quad(uint32_t addr) {
  u4 q;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(q.x), "=r"(q.y), "=r"(q.z), "=r"(q.w) : "r"(addr));
  return q;
}
PAI_DEV void sts_quad(uint32_t addr, const u4& q) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(q.x), "r"(q.y), "r"(q.z), "r"(q.w) : "memory");
}
PAI_DEV u4 ld_quad(const SOpnd& o, int q) { return lds_quad(o.a + (uint32_t)q * o.sb); }
PAI_DEV void ld_tile(const SOpnd& o, int t, uint32_t a[8]) {
  const uint32_t base = o.a + (uint32_t)(2 * t) * o.sb;
  u4 q0 = lds_quad(base), q1 = lds_quad(base + o.sb);
  a[0] = q0.x; a[1] = q0.y; a[2] = q0.z; a[3] = q0.w;
  a[4] = q1.x; a[5] = q1.y; a[6] = q1.z; a[7] = q1.w;
}
PAI_DEV void st_tile(const SOpnd& o, int t, const uint32_t a[8]) {
  const uint32_t base = o.a + (uint32_t)(2 * t) * o.sb;
  u4 q0, q1;
  q0.x = a[0]; q0.y = a[1]; q0.z = a[2]; q0.w = a[3];
  q1.x = a[4]; q1.y = a[5]; q1.z = a[6]; q1.w = a[7];
  sts_quad(base, q0);
  sts_quad(base + o.sb, q1);
}
#else
typedef Opnd SOpnd;
PAI_DEV SOpnd to_shared(const Opnd& o) { return o; }
PAI_DEV u4 ld_quad(const SOpnd& o, int q) { return o.p[q * o.s]; }
#endif
PAI_DEV u4 ld_quad_g(const Opnd& o, int q) { return o.p[q * o.s]; }

// ------------------------------------------------------------------------------------------------
// Carry-chain primitives.  Each is ONE asm block so the carry flag never crosses a statement.

PAI_DEV uint32_t lo32(uint64_t x) { return (uint32_t)x; }
PAI_DEV uint32_t hi32(uint64_t x) { return (uint32_t)(x >> 32); }
PAI_DEV uint64_t pack64(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// X[0..3] (four 64-bit column pairs) += {a0,a1,a2,a3} * b, one product per pair, carries rippling
// from pair to pair; the final carry-out is added to cw.
// The accumulator limbs are held as 64-bit values so that ptxas keeps every (lo, hi) in an aligned
// register pair: each mad.lo.cc/madc.hi.cc couple becomes ONE in-place IMAD.WIDE.U32(.X) with no register
// shuffling (with separate 32-bit registers the r01 ncu capture showed ~35 MOVs per 64 MACs).
PAI_DEV void mac_chain4(uint64_t* X, uint32_t& cw, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b) {
#if !defined(PAI_HOSTSIM)
  asm("{\n\t"
      ".reg .u32 l0, h0, l1, h1, l2, h2, l3, h3;\n\t"
      "mov.b64 {l0, h0}, %0;\n\t"
      "mov.b64 {l1, h1}, %1;\n\t"
      "mov.b64 {l2, h2}, %2;\n\t"
      "mov.b64 {l3, h3}, %3;\n\t"
      "mad.lo.cc.u32 l0, %5, %9, l0;\n\t"
      "madc.hi.cc.u32 h0, %5, %9, h0;\n\t"
      "madc.lo.cc.u32 l1, %6, %9, l1;\n\t"
      "madc.hi.cc.u32 h1, %6, %9, h1;\n\t"
      "madc.lo.cc.u32 l2, %7, %9, l2;\n\t"
      "madc.hi.cc.u32 h2, %7, %9, h2;\n\t"
      "madc.lo.cc.u32 l3, %8, %9, l3;\n\t"
      "madc.hi.cc.u32 h3, %8, %9, h3;\n\t"
      "addc.u32 %4, %4, 0;\n\t"
      "mov.b64 %0, {l0, h0};\n\t"
      "mov.b64 %1, {l1, h1};\n\t"
      "mov.b64 %2, {l2, h2};\n\t"
      "mov.b64 %3, {l3, h3};\n\t"
      "}"
      : "+l"(X[0]), "+l"(X[1]), "+l"(X[2]), "+l"(X[3]), "+r"(cw)
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b));
#else
  const uint32_t av[4] = {a0, a1, a2, a3};
  uint32_t c = 0;
  for (int i = 0; i < 4; i++) {
    unsigned __int128 v = (unsigned __int128)X[i] + (uint64_t)av[i] * b + c;
    X[i] = (uint64_t)v;
    c = (uint32_t)(v >> 64);
  }
  cw += c;
#endif
}

// r[0..7] = a[0..7] + b[0..7]; returns carry-out (0/1)
PAI_DEV uint32_t add8(uint32_t r[8], const uint32_t a[8], const uint32_t b[8]) {
  uint32_t c;
#if !defined(PAI_HOSTSIM)
  asm("add.cc.u32 %0, %9, %17;\n\t"
      "addc.cc.u32 %1, %10, %18;\n\t"
      "addc.cc.u32 %2, %11, %19;\n\t"
      "addc.cc.u32 %3, %12, %20;\n\t"
      "addc.cc.u32 %4, %13, %21;\n\t"
      "addc.cc.u32 %5, %14, %22;\n\t"
      "addc.cc.u32 %6, %15, %23;\n\t"
      "addc.cc.u32 %7, %16, %24;\n\t"
      "addc.u32 %8, 0, 0;"
      : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]), "=r"(c)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
        "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
#else
  uint64_t cc = 0;
  for (int i = 0; i < 8; i++) { cc += (uint64_t)a[i] + b[i]; r[i] = (uint32_t)cc; cc >>= 32; }
  c = (uint32_t)cc;
#endif
  return c;
}

// r = a + b + cin ; returns carry-out.  cin in {0,1}
PAI_DEV uint32_t add8c(uint32_t r[8], const uint32_t a[8], const uint32_t b[8], uint32_t cin) {
  uint32_t c;
#if !defined(PAI_HOSTSIM)
  asm("add.cc.u32 %8, %25, 0xffffffff;\n\t"   // sets CF = cin
      "addc.cc.u32 %0, %9, %17;\n\t"
      "addc.cc.u32 %1, %10, %18;\n\t"
      "addc.cc.u32 %2, %11, %19;\n\t"
      "addc.cc.u32 %3, %12, %20;\n\t"
      "addc.cc.u32 %4, %13, %21;\n\t"
      "addc.cc.u32 %5, %14, %22;\n\t"
      "addc.cc.u32 %6, %15, %23;\n\t"
      "addc.cc.u32 %7, %16, %24;\n\t"
      "addc.u32 %8, 0, 0;"
      : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]), "=&r"(c)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
        "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]), "r"(cin));
#else
  uint64_t cc = cin;
  for (int i = 0; i < 8; i++) { cc += (uint64_t)a[i] + b[i]; r[i] = (uint32_t)cc; cc >>= 32; }
  c = (uint32_t)cc;
#endif
  return c;
}

// r = a - b - bin ; returns borrow-out (0/1).  bin in {0,1}
PAI_DEV uint32_t sub8b(uint32_t r[8], const uint32_t a[8], const uint32_t b[8], uint32_t bin) {
  uint32_t bo;
#if !defined(PAI_HOSTSIM)
  asm("sub.cc.u32 %8, 0, %25;\n\t"            // 0 - bin : borrow set iff bin == 1
      "subc.cc.u32 %0, %9, %17;\n\t"
      "subc.cc.u32 %1, %10, %18;\n\t"
      "subc.cc.u32 %2, %11, %19;\n\t"
      "subc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, %21;\n\t"
      "subc.cc.u32 %5, %14, %22;\n\t"
      "subc.cc.u32 %6, %15, %23;\n\t"
      "subc.cc.u32 %7, %16, %24;\n\t"
      "subc.u32 %8, 0, 0;"                     // 0 - 0 - borrow  -> 0 or 0xffffffff
      : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]), "=&r"(bo)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
        "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]), "r"(bin));
  bo &= 1u;
#else
  uint64_t bb = bin;
  for (int i = 0; i < 8; i++) {
    uint64_t d = (uint64_t)a[i] - b[i] - bb;
    r[i] = (uint32_t)d;
    bb = (d >> 63) & 1;
  }
  bo = (uint32_t)bb;
#endif
  return bo;
}

// ------------------------------------------------------------------------------------------------
// Column accumulator.  Value = sum_i E[i]*2^(64 i) + sum_i O[i]*2^(64 i + 32) + sum_i C[i]*2^(32 i).
//   E[i] : 64-bit pair on columns (2i, 2i+1)   -- targets of chains that start on an even column
//   O[i] : 64-bit pair on columns (2i+1, 2i+2) -- targets of chains that start on an odd column
//   C[i] : small counters that collect the carry-out of every chain (never a product target, so they
//          cannot overflow); keeping them separate makes every tile MAC exact without rippling.
struct Acc {
  uint64_t E[8], O[8];
  uint32_t C[17];
};

PAI_DEV void acc_clear(Acc& A) {
  PAI_UNROLL
  for (int i = 0; i < 8; i++) { A.E[i] = 0; A.O[i] = 0; }
  PAI_UNROLL
  for (int i = 0; i < 17; i++) A.C[i] = 0;
}

// A += a[0..7] * b[0..7]   (64 wide MACs + 16 carry captures)
PAI_DEV void tile_mac(Acc& A, const uint32_t a[8], const uint32_t b[8]) {
  PAI_UNROLL
  for (int j = 0; j < 8; j++) {
    if ((j & 1) == 0) {
      mac_chain4(&A.E[j / 2], A.C[j + 8], a[0], a[2], a[4], a[6], b[j]);          // columns j   .. j+7
      mac_chain4(&A.O[j / 2], A.C[j + 9], a[1], a[3], a[5], a[7], b[j]);          // columns j+1 .. j+8
    } else {
      mac_chain4(&A.O[(j - 1) / 2], A.C[j + 8], a[0], a[2], a[4], a[6], b[j]);    // columns j   .. j+7
      mac_chain4(&A.E[(j + 1) / 2], A.C[j + 9], a[1], a[3], a[5], a[7], b[j]);    // columns j+1 .. j+8
    }
  }
}

// the low 8 columns of E and of O as 32-bit vectors
PAI_DEV void acc_low_vectors(const Acc& A, uint32_t e[8], uint32_t o[8]) {
  PAI_UNROLL
  for (int i = 0; i < 4; i++) { e[2 * i] = lo32(A.E[i]); e[2 * i + 1] = hi32(A.E[i]); }
  o[0] = 0;
  o[1] = lo32(A.O[0]); o[2] = hi32(A.O[0]);
  o[3] = lo32(A.O[1]); o[4] = hi32(A.O[1]);
  o[5] = lo32(A.O[2]); o[6] = hi32(A.O[2]);
  o[7] = lo32(A.O[3]);
}

// v = low 8 limbs of the accumulator value; their carry is pushed into C[8]
PAI_DEV void acc_resolve_low(Acc& A, uint32_t v[8]) {
  uint32_t e[8], o[8], t[8];
  acc_low_vectors(A, e, o);
  uint32_t c1 = add8(t, e, o);
  uint32_t c2 = add8(v, t, A.C);
  A.C[8] += c1 + c2;
}

// v = low 8 limbs of the accumulator value WITHOUT recording their carry (the limbs stay in place;
// a later acc_resolve_low over the same limbs accounts for the carry exactly once)
PAI_DEV void acc_peek_low(const Acc& A, uint32_t v[8]) {
  uint32_t e[8], o[8], t[8];
  acc_low_vectors(A, e, o);
  add8(t, e, o);
  add8(v, t, A.C);
}

// The low 8 limbs of the accumulator VALUE are known to be 0 mod 2^256 (right after acc += m * n0 in a
// Montgomery step): their carry into limb 8 is k = (E + O + C at limb 7, + 2) >> 32 -- the limbs below 7 sum to
// delta * 2^224 with delta in {0, 1, 2}, so limb 7 holds k*2^32 - delta.  Replaces two 8-limb carry chains.
PAI_DEV void acc_carry_of_zero_low(Acc& A) {
  uint64_t s7 = (uint64_t)hi32(A.E[3]) + lo32(A.O[3]) + A.C[7] + 2u;
  A.C[8] += (uint32_t)(s7 >> 32);
}

// A.low8 += d[0..7]  (carry captured in C[8])
PAI_DEV void acc_add_low(Acc& A, const uint32_t d[8]) {
  uint32_t e[8], t[8];
  PAI_UNROLL
  for (int i = 0; i < 4; i++) { e[2 * i] = lo32(A.E[i]); e[2 * i + 1] = hi32(A.E[i]); }
  uint32_t c = add8(t, e, d);
  PAI_UNROLL
  for (int i = 0; i < 4; i++) A.E[i] = pack64(t[2 * i], t[2 * i + 1]);
  A.C[8] += c;
}

// A >>= 256 bits (the low 8 limbs must already have been consumed)
PAI_DEV void acc_shift8(Acc& A) {
  uint32_t straddle = hi32(A.O[3]);            // column 8 of the pair (7, 8): becomes column 0
  PAI_UNROLL
  for (int i = 0; i < 4; i++) { A.E[i] = A.E[i + 4]; A.E[i + 4] = 0; }
  A.O[0] = A.O[4]; A.O[1] = A.O[5]; A.O[2] = A.O[6];
  A.O[3] = 0; A.O[4] = 0; A.O[5] = 0; A.O[6] = 0;
  PAI_UNROLL
  for (int i = 0; i < 8; i++) { A.C[i] = A.C[i + 8]; A.C[i + 8] = 0; }
  A.C[8] = A.C[16];
  A.C[16] = 0;
  uint64_t s = A.E[0] + straddle;               // fold it into the pair (0, 1); carry -> column 2
  A.C[2] += (s < A.E[0]) ? 1u : 0u;
  A.E[0] = s;
}

// Short chains for the truncated product below: X[0..NP) += {a0..} * b on NP pairs; the carry out of the
// last pair is added to cw.
template <int NP>
PAI_DEV void mac_chain_n(uint64_t* X, uint32_t& cw, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b) {
#if !defined(PAI_HOSTSIM)
  if (NP == 1) {
    asm("{\n\t.reg .u32 l0, h0;\n\t"
        "mov.b64 {l0, h0}, %0;\n\t"
        "mad.lo.cc.u32 l0, %2, %3, l0;\n\t"
        "madc.hi.cc.u32 h0, %2, %3, h0;\n\t"
        "addc.u32 %1, %1, 0;\n\t"
        "mov.b64 %0, {l0, h0};\n\t}"
        : "+l"(X[0]), "+r"(cw) : "r"(a0), "r"(b));
  } else if (NP == 2) {
    asm("{\n\t.reg .u32 l0, h0, l1, h1;\n\t"
        "mov.b64 {l0, h0}, %0;\n\t"
        "mov.b64 {l1, h1}, %1;\n\t"
        "mad.lo.cc.u32 l0, %3, %5, l0;\n\t"
        "madc.hi.cc.u32 h0, %3, %5, h0;\n\t"
        "madc.lo.cc.u32 l1, %4, %5, l1;\n\t"
        "madc.hi.cc.u32 h1, %4, %5, h1;\n\t"
        "addc.u32 %2, %2, 0;\n\t"
        "mov.b64 %0, {l0, h0};\n\t"
        "mov.b64 %1, {l1, h1};\n\t}"
        : "+l"(X[0]), "+l"(X[1]), "+r"(cw) : "r"(a0), "r"(a1), "r"(b));
  } else if (NP == 3) {
    asm("{\n\t.reg .u32 l0, h0, l1, h1, l2, h2;\n\t"
        "mov.b64 {l0, h0}, %0;\n\t"
        "mov.b64 {l1, h1}, %1;\n\t"
        "mov.b64 {l2, h2}, %2;\n\t"
        "mad.lo.cc.u32 l0, %4, %7, l0;\n\t"
        "madc.hi.cc.u32 h0, %4, %7, h0;\n\t"
        "madc.lo.cc.u32 l1, %5, %7, l1;\n\t"
        "madc.hi.cc.u32 h1, %5, %7, h1;\n\t"
        "madc.lo.cc.u32 l2, %6, %7, l2;\n\t"
        "madc.hi.cc.u32 h2, %6, %7, h2;\n\t"
        "addc.u32 %3, %3, 0;\n\t"
        "mov.b64 %0, {l0, h0};\n\t"
        "mov.b64 %1, {l1, h1};\n\t"
        "mov.b64 %2, {l2, h2};\n\t}"
        : "+l"(X[0]), "+l"(X[1]), "+l"(X[2]), "+r"(cw) : "r"(a0), "r"(a1), "r"(a2), "r"(b));
  } else {
    mac_chain4(X, cw, a0, a1, a2, a3, b);
  }
#else
  const uint32_t av[4] = {a0, a1, a2, a3};
  uint32_t c = 0;
  for (int i = 0; i < NP; i++) {
    unsigned __int128 v = (unsigned __int128)X[i] + (uint64_t)av[i] * b + c;
    X[i] = (uint64_t)v;
    c = (uint32_t)(v >> 64);
  }
  cw += c;
#endif
}

// m = (v * w) mod 2^256: only the products with i + j <= 7 matter, and those on the anti-diagonal
// i + j = 7 only through their low halves: 28 wide MACs + 8 plain IMADs instead of 64 wide MACs.
PAI_DEV void mul_lo8(uint32_t m[8], const uint32_t v[8], const uint32_t w[8]) {
  uint64_t E[4] = {0, 0, 0, 0};    // column pairs (0,1) (2,3) (4,5) (6,7)
  uint64_t O[3] = {0, 0, 0};       // column pairs (1,2) (3,4) (5,6)
  // row j (multiplier w[j]); product v[i]*w[j] lands on columns (i+j, i+j+1) and is kept iff i + j <= 6
  // j = 0: even i 0,2,4,6 -> E[0..3];  odd i 1,3,5 -> O[0..2]
  uint32_t d = 0, junk = 0;        // d: column 7 (carries out of the O chains + anti-diagonal); junk: column 8
  mac_chain_n<4>(&E[0], junk, v[0], v[2], v[4], v[6], w[0]);
  mac_chain_n<3>(&O[0], d, v[1], v[3], v[5], 0, w[0]);
  // j = 1: even i 0,2,4 -> O[0..2];   odd i 1,3,5 -> E[1..3]
  mac_chain_n<3>(&O[0], d, v[0], v[2], v[4], 0, w[1]);
  mac_chain_n<3>(&E[1], junk, v[1], v[3], v[5], 0, w[1]);
  // j = 2: even i 0,2,4 -> E[1..3];   odd i 1,3 -> O[1..2]
  mac_chain_n<3>(&E[1], junk, v[0], v[2], v[4], 0, w[2]);
  mac_chain_n<2>(&O[1], d, v[1], v[3], 0, 0, w[2]);
  // j = 3: even i 0,2 -> O[1..2];     odd i 1,3 -> E[2..3]
  mac_chain_n<2>(&O[1], d, v[0], v[2], 0, 0, w[3]);
  mac_chain_n<2>(&E[2], junk, v[1], v[3], 0, 0, w[3]);
  // j = 4: even i 0,2 -> E[2..3];     odd i 1 -> O[2]
  mac_chain_n<2>(&E[2], junk, v[0], v[2], 0, 0, w[4]);
  mac_chain_n<1>(&O[2], d, v[1], 0, 0, 0, w[4]);
  // j = 5: even i 0 -> O[2];          odd i 1 -> E[3]
  mac_chain_n<1>(&O[2], d, v[0], 0, 0, 0, w[5]);
  mac_chain_n<1>(&E[3], junk, v[1], 0, 0, 0, w[5]);
  // j = 6: even i 0 -> E[3]
  mac_chain_n<1>(&E[3], junk, v[0], 0, 0, 0, w[6]);
  // anti-diagonal, low halves only -> column 7
  PAI_UNROLL
  for (int i = 0; i < 8; i++) d += v[i] * w[7 - i];
  uint32_t e[8], o[8], t[8];
  PAI_UNROLL
  for (int i = 0; i < 4; i++) { e[2 * i] = lo32(E[i]); e[2 * i + 1] = hi32(E[i]); }
  o[0] = 0;
  o[1] = lo32(O[0]); o[2] = hi32(O[0]);
  o[3] = lo32(O[1]); o[4] = hi32(O[1]);
  o[5] = lo32(O[2]); o[6] = hi32(O[2]);
  o[7] = d;
  add8(t, e, o);
  PAI_UNROLL
  for (int i = 0; i < 8; i++) m[i] = t[i];
}

// ------------------------------------------------------------------------------------------------
// Whole-number helpers on interleaved operands (NT tiles each).

// borrow of (a - b); nothing stored
template <int NT>
PAI_DEV uint32_t big_sub_borrow(const Opnd& a, const Opnd& b) {
  uint32_t bo = 0;
  for (int t = 0; t < NT; t++) {
    uint32_t x[8], y[8], r[8];
    ld_tile(a, t, x); ld_tile(b, t, y);
    bo = sub8b(r, x, y, bo);
  }
  return bo;
}

// out = a - (b & mask)   (mask = 0 or 0xffffffff); returns borrow
template <int NT>
PAI_DEV uint32_t big_sub_masked(const Opnd& out, const Opnd& a, const Opnd& b, uint32_t mask) {
  uint32_t bo = 0;
  for (int t = 0; t < NT; t++) {
    uint32_t x[8], y[8], r[8];
    ld_tile(a, t, x); ld_tile(b, t, y);
    PAI_UNROLL
    for (int i = 0; i < 8; i++) y[i] &= mask;
    bo = sub8b(r, x, y, bo);
    st_tile(out, t, r);
  }
  return bo;
}

// out = a + (b & mask); returns carry
template <int NT>
PAI_DEV uint32_t big_add_masked(const Opnd& out, const Opnd& a, const Opnd& b, uint32_t mask) {
  uint32_t c = 0;
  for (int t = 0; t < NT; t++) {
    uint32_t x[8], y[8], r[8];
    ld_tile(a, t, x); ld_tile(b, t, y);
    PAI_UNROLL
    for (int i = 0; i < 8; i++) y[i] &= mask;
    c = add8c(r, x, y, c);
    st_tile(out, t, r);
  }
  return c;
}

// x = x - N if (force || x >= N)    -> canonical residue when x < 2N (or x + force*2^(256NT) < 2N)
template <int NT>
PAI_DEV uint32_t big_cond_sub(const Opnd& x, const Opnd& N, uint32_t force) {
  uint32_t bo = big_sub_borrow<NT>(x, N);
  uint32_t need = ((force != 0u) | (bo ^ 1u)) & 1u;
  big_sub_masked<NT>(x, x, N, 0u - need);
  return need;                                   // 1 iff N was subtracted
}

template <int NT>
PAI_DEV void big_copy(const Opnd& dst, const Opnd& src) {
  for (int q = 0; q < 2 * NT; q++) dst.p[q * dst.s] = src.p[q * src.s];
}

template <int NT>
PAI_DEV uint32_t big_is_zero(const Opnd& a) {
  uint32_t acc = 0;
  for (int q = 0; q < 2 * NT; q++) { u4 v = a.p[q * a.s]; acc |= v.x | v.y | v.z | v.w; }
  return acc == 0 ? 1u : 0u;
}

// ------------------------------------------------------------------------------------------------
// Plain product, column (product) scanning over tiles:
//   out[0..NCOL) = low NCOL tiles of  (a * b + addend),  a: NTA tiles, b: NTB tiles, addend < 2^32
template <int NTA, int NTB, int NCOL>
PAI_DEV void big_mul(const Opnd& out, const Opnd& a, const Opnd& b, uint32_t addend) {
  Acc acc;
  acc_clear(acc);
  acc.E[0] = addend;   // 64-bit pair on columns (0, 1)
  for (int k = 0; k < NCOL; k++) {
    int lo = k - NTB + 1 > 0 ? k - NTB + 1 : 0;
    int hi = k < NTA - 1 ? k : NTA - 1;
    for (int i = lo; i <= hi; i++) {
      uint32_t x[8], y[8];
      ld_tile(a, i, x); ld_tile(b, k - i, y);
      tile_mac(acc, x, y);
    }
    uint32_t v[8];
    acc_resolve_low(acc, v);
    st_tile(out, k, v);
    acc_shift8(acc);
  }
}

// ------------------------------------------------------------------------------------------------
// Montgomery multiplication, tile-level finely integrated product scanning (R = 2^(256 NT)):
//   out = a * b / R mod N, canonical (< N) provided a*b < R*N.
//   `out` doubles as the store for the quotient tiles m_i (dead before the result tile that
//   replaces them is written), so out must not alias a or b.  N is a broadcast operand,
//   NI = tile holding -N^-1 mod 2^256.
template <int NT>
PAI_FN void mont_mul(Opnd out, Opnd a, Opnd b, Opnd N, Opnd NI) {
  Acc acc;
  acc_clear(acc);
  uint32_t bo = 0;
  uint32_t n0[8], ninv[8];
  ld_tile(N, 0, n0);
  ld_tile(NI, 0, ninv);
  for (int k = 0; k < 2 * NT; k++) {
    int lo = k - NT + 1 > 0 ? k - NT + 1 : 0;
    int hi = k < NT ? k - 1 : NT - 1;
    // terms that have both a product and a reduction partner: i in [lo, hi], j = k - i >= 1
    for (int i = lo; i <= hi; i++) {
      uint32_t x[8], y[8], u[8], w[8];
      ld_tile(a, i, x); ld_tile(b, k - i, y);
      ld_tile(out, i, u); ld_tile(N, k - i, w);
      tile_mac(acc, x, y);
      tile_mac(acc, u, w);
    }
    uint32_t v[8];
    if (k < NT) {
      uint32_t x[8], y[8], m[8];
      ld_tile(a, k, x); ld_tile(b, 0, y);
      tile_mac(acc, x, y);
      acc_peek_low(acc, v);
      mul_lo8(m, v, ninv);
      st_tile(out, k, m);
      tile_mac(acc, m, n0);
      acc_carry_of_zero_low(acc);       // low tile == 0 by construction; its carry goes to C[8]
    } else {
      acc_resolve_low(acc, v);
      st_tile(out, k - NT, v);
      uint32_t nt[8], d[8];
      ld_tile(N, k - NT, nt);
      bo = sub8b(d, v, nt, bo);                  // running borrow of (result - N): no separate compare pass
    }
    acc_shift8(acc);
  }
  uint32_t ovf = lo32(acc.E[0]) + acc.C[0];   // what is left is 0 or 1, in column 0
  uint32_t need = (ovf != 0u) | (bo ^ 1u);
  big_sub_masked<NT>(out, out, N, 0u - need);
}

// Montgomery squaring: out = a*a/R mod N.  Off-diagonal tile products are accumulated once in a
// second accumulator S, doubled on the way into the main accumulator (136 instead of 256 product
// tiles at NT = 16).
template <int NT>
PAI_FN void mont_sqr(Opnd out, Opnd a, Opnd N, Opnd NI) {
  Acc acc, S;
  acc_clear(acc);
  acc_clear(S);
  uint32_t n0[8], ninv[8];
  ld_tile(N, 0, n0);
  ld_tile(NI, 0, ninv);
  uint32_t topbit = 0, bo = 0;
  for (int k = 0; k < 2 * NT; k++) {
    int lo = k - NT + 1 > 0 ? k - NT + 1 : 0;
    int hi = k < NT ? k - 1 : NT - 1;
    // off-diagonal pairs i < j = k - i  <=>  i <= (k-1)/2
    int hs = (k - 1) / 2;
    if (k == 0) hs = -1;
    // i in [lo, hs]: an off-diagonal product tile (into S) and a reduction tile m_i * N_(k-i) (into acc) --
    // two independent accumulators, so the two wavefronts of IMAD.WIDE chains interleave
    int i = lo;
    for (; i <= hs; i++) {
      uint32_t x[8], y[8], u[8], w[8];
      ld_tile(a, i, x); ld_tile(a, k - i, y);
      ld_tile(out, i, u); ld_tile(N, k - i, w);
      tile_mac(S, x, y);
      tile_mac(acc, u, w);
    }
    // remaining reduction partners, i in (hs, hi]
    for (; i <= hi; i++) {
      uint32_t x[8], y[8];
      ld_tile(out, i, x); ld_tile(N, k - i, y);
      tile_mac(acc, x, y);
    }
    if ((k & 1) == 0) {
      uint32_t x[8];
      ld_tile(a, k >> 1, x);
      tile_mac(acc, x, x);
    }
    // main += 2 * (low tile of S)
    {
      uint32_t d[8], d2[8];
      acc_resolve_low(S, d);
      acc_shift8(S);
      d2[0] = (d[0] << 1) | topbit;
      PAI_UNROLL
      for (int i = 1; i < 8; i++) d2[i] = (d[i] << 1) | (d[i - 1] >> 31);
      topbit = d[7] >> 31;
      acc_add_low(acc, d2);
    }
    uint32_t v[8];
    if (k < NT) {
      uint32_t m[8];
      acc_peek_low(acc, v);
      mul_lo8(m, v, ninv);
      st_tile(out, k, m);
      tile_mac(acc, m, n0);
      acc_carry_of_zero_low(acc);
    } else {
      acc_resolve_low(acc, v);
      st_tile(out, k - NT, v);
      uint32_t nt[8], d[8];
      ld_tile(N, k - NT, nt);
      bo = sub8b(d, v, nt, bo);
    }
    acc_shift8(acc);
  }
  uint32_t ovf = lo32(acc.E[0]) + acc.C[0] + topbit;
  uint32_t need = (ovf != 0u) | (bo ^ 1u);
  big_sub_masked<NT>(out, out, N, 0u - need);
}

}  // namespace pai
