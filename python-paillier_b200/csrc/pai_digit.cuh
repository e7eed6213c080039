// pai_digit.cuh -- Montgomery arithmetic modulo n^2 on base-n digits.
//
// Paillier's moduli are squares (n^2, p^2, q^2).  Write an element of Z_{n^2} as X = X0 + n*X1 with
// digits 0 <= X0, X1 < n, and let R = 2^(256*NTH) be the Montgomery radix OF n (half the width of n^2).
// With A = X0*Y0 and the ordinary Montgomery reduction modulo n,  A + m*n = t*R  (m = -A/n mod R),
//
//     X*Y = A + n*(X0*Y1 + X1*Y0)            (mod n^2)
//         = t*R + n*(X0*Y1 + X1*Y0 - m)
//     X*Y*R^-1 = t + n * REDC_n(X0*Y1 + X1*Y0 - m)          (mod n^2)
// (t < 2n: when it is reduced to t - n the high digit gains +1, i.e. +R inside the second REDC)
//
// because n*a mod n^2 only depends on a mod n.  So one multiplication modulo n^2 (in Montgomery form with
// radix R) costs two half-width Montgomery passes: REDC_n(X0*Y0) (keeping its quotient m) and
// REDC_n(X0*Y1 + X1*Y0 + (K - m)) with K a multiple of n that keeps the sum non-negative.
// In tile products (NTH = tiles of n):   multiply 5*NTH^2 + 2*NTH  instead of 8*NTH^2 + 2*NTH,
//                                        square   ~3.5*NTH^2 + 2.5*NTH instead of ~6*NTH^2 + 3*NTH
// (2048-bit key: 336 vs 528 and 244 vs 408) -- and no arithmetic is done on 2x-wide numbers at all.
// For decryption there is a bonus: with u = u0 + p*u1 the function L(u) = (u-1)//p (phe/paillier.py:362)
// is just the high digit u1 (minus one when u0 = 0, reproducing Python's floor division).
//
// Results are bit-identical to any other exact method (unique canonical residues); the parity tests do not
// know which path produced them.
#pragma once
#include "pai_kernels.cuh"

namespace pai {

// a number in digit form: two operands of NTH tiles each
struct DNum {
  Opnd d0, d1;
};

// the two halves of an operand buffer of 2*NTH tiles
template <int NTH>
PAI_DEV Opnd half_lo(const Opnd& b) { return b; }
template <int NTH>
PAI_DEV Opnd half_hi(const Opnd& b) {
  Opnd o;
  o.p = b.p + (size_t)(2 * NTH) * b.s;
  o.s = b.s;
  return o;
}

struct DigitEnv {
  Opnd N, NI, KL, ONE, ZERO;
  Opnd N2, N3, TOPS;          // 2n mod R, 3n mod R, and their overflow words (TOPS tile: [top2, top3, ...])
  DNum RR, ONEM, E3, E4, E5;
};

// x = K - x (NT tiles); returns the borrow (1 if x > K)
template <int NT>
PAI_DEV uint32_t big_rsub(const Opnd& x, const Opnd& K) {
  uint32_t bo = 0;
  for (int t = 0; t < NT; t++) {
    uint32_t a[8], b[8], r[8];
    ld_tile(K, t, a); ld_tile(x, t, b);
    bo = sub8b(r, a, b, bo);
    st_tile(x, t, r);
  }
  return bo;
}

// Reduction of the second phase: V = olo + ovf*R < 3n + 2.  b1, b2, b3 are the borrows of olo - (c*n mod R)
// gathered while the result tiles were produced; q = #{c : V >= c*n}; one masked subtraction of q*n.
template <int NTH>
PAI_DEV void digit_reduce3(const Opnd& olo, const DigitEnv& dc, uint32_t ovf, uint32_t b1, uint32_t b2, uint32_t b3) {
  const u4 tops = dc.TOPS.p[0];
  const int s1 = (int)ovf - (int)b1;
  const int s2 = (int)ovf - (int)tops.x - (int)b2;
  const int s3 = (int)ovf - (int)tops.y - (int)b3;
  const int q = (s1 >= 0) + (s2 >= 0) + (s3 >= 0);
  Opnd sel = q == 2 ? dc.N2 : (q == 3 ? dc.N3 : dc.N);
  big_sub_masked<NTH>(olo, olo, sel, q ? 0xffffffffu : 0u);
}

template <int NTH>
PAI_FN void dmul(Opnd olo, Opnd ohi, Opnd x0, Opnd x1, Opnd y0, Opnd y1, const DigitEnv* dcp) {
  const DigitEnv& dc = *dcp;
  const Opnd N = dc.N, NI = dc.NI, KL = dc.KL;
  uint32_t n0[8], ninv[8];
  ld_tile(N, 0, n0);
  ld_tile(NI, 0, ninv);
  uint32_t carry = 0;
  // ---- phase 1: A = x0*y0, m -> olo, t = (A + m n)/R -> ohi
  {
    Acc acc;
    acc_clear(acc);
    uint32_t b1 = 0;
    for (int k = 0; k < 2 * NTH; k++) {
      int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
      int hi = k < NTH ? k - 1 : NTH - 1;
      for (int i = lo; i <= hi; i++) {
        uint32_t x[8], y[8], u[8], w[8];
        ld_tile(x0, i, x); ld_tile(y0, k - i, y);
        ld_tile(olo, i, u); ld_tile(N, k - i, w);
        tile_mac(acc, x, y);
        tile_mac(acc, u, w);
      }
      uint32_t v[8];
      if (k < NTH) {
        uint32_t x[8], y[8], m[8];
        ld_tile(x0, k, x); ld_tile(y0, 0, y);
        tile_mac(acc, x, y);
        acc_peek_low(acc, v);
        mul_lo8(m, v, ninv);
        st_tile(olo, k, m);
        tile_mac(acc, m, n0);
        acc_carry_of_zero_low(acc);
      } else {
        acc_resolve_low(acc, v);
        st_tile(ohi, k - NTH, v);
        uint32_t nt[8], d[8];
        ld_tile(N, k - NTH, nt);
        b1 = sub8b(d, v, nt, b1);
      }
      acc_shift8(acc);
    }
    uint32_t ovf = lo32(acc.E[0]) + acc.C[0];
    carry = (ovf != 0u) | (b1 ^ 1u);
    big_sub_masked<NTH>(ohi, ohi, N, 0u - carry);
  }
  // ---- W = (R + KL) - m  >= 0:  low NTH tiles in olo, top part wtop.  Reducing the low digit by n carries
  // +1 into the high digit; adding R to B adds exactly 1 to REDC_n(B), so the carry rides on wtop.
  uint32_t wtop = 1u - big_rsub<NTH>(olo, KL) + carry;
  // ---- phase 2: B = x0*y1 + x1*y0 + W, quotient tiles m' overwrite W tile by tile, result Z1 -> olo
  {
    Acc acc;
    acc_clear(acc);
    uint32_t b1 = 0, b2 = 0, b3 = 0;
    for (int k = 0; k < 2 * NTH; k++) {
      int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
      int hi = k < NTH ? k - 1 : NTH - 1;
      for (int i = lo; i <= hi; i++) {
        uint32_t x[8], y[8];
        ld_tile(x0, i, x); ld_tile(y1, k - i, y);
        tile_mac(acc, x, y);
        ld_tile(x1, i, x); ld_tile(y0, k - i, y);
        tile_mac(acc, x, y);
        ld_tile(olo, i, x); ld_tile(N, k - i, y);
        tile_mac(acc, x, y);
      }
      uint32_t v[8];
      if (k < NTH) {
        uint32_t x[8], y[8], m[8];
        ld_tile(x0, k, x); ld_tile(y1, 0, y);
        tile_mac(acc, x, y);
        ld_tile(x1, k, x); ld_tile(y0, 0, y);
        tile_mac(acc, x, y);
        ld_tile(olo, k, x);                                   // W_k
        acc_add_low(acc, x);
        acc_peek_low(acc, v);
        mul_lo8(m, v, ninv);
        st_tile(olo, k, m);
        tile_mac(acc, m, n0);
        acc_carry_of_zero_low(acc);
      } else {
        if (k == NTH) acc.C[0] += wtop;
        acc_resolve_low(acc, v);
        st_tile(olo, k - NTH, v);
        uint32_t nt[8], d[8];
        ld_tile(N, k - NTH, nt);      b1 = sub8b(d, v, nt, b1);
        ld_tile(dc.N2, k - NTH, nt);  b2 = sub8b(d, v, nt, b2);
        ld_tile(dc.N3, k - NTH, nt);  b3 = sub8b(d, v, nt, b3);
      }
      acc_shift8(acc);
    }
    uint32_t ovf = lo32(acc.E[0]) + acc.C[0];
    digit_reduce3<NTH>(olo, dc, ovf, b1, b2, b3);
  }
}

// Z = X^2 * R^-1 mod n^2 in digit form (X0, X1 canonical).  Output as in dmul.
template <int NTH>
PAI_FN void dsqr(Opnd olo, Opnd ohi, Opnd x0, Opnd x1, const DigitEnv* dcp) {
  const DigitEnv& dc = *dcp;
  const Opnd N = dc.N, NI = dc.NI, KL = dc.KL;
  uint32_t n0[8], ninv[8];
  ld_tile(N, 0, n0);
  ld_tile(NI, 0, ninv);
  uint32_t carry = 0;
  // ---- phase 1: A = x0^2 (off-diagonal tiles once, doubled through S), m -> olo, t -> ohi
  {
    Acc acc, S;
    acc_clear(acc);
    acc_clear(S);
    uint32_t topbit = 0, b1 = 0;
    for (int k = 0; k < 2 * NTH; k++) {
      int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
      int hi = k < NTH ? k - 1 : NTH - 1;
      int hs = k == 0 ? -1 : (k - 1) / 2;
      int i = lo;
      for (; i <= hs; i++) {
        uint32_t x[8], y[8], u[8], w[8];
        ld_tile(x0, i, x); ld_tile(x0, k - i, y);
        ld_tile(olo, i, u); ld_tile(N, k - i, w);
        tile_mac(S, x, y);
        tile_mac(acc, u, w);
      }
      for (; i <= hi; i++) {
        uint32_t x[8], y[8];
        ld_tile(olo, i, x); ld_tile(N, k - i, y);
        tile_mac(acc, x, y);
      }
      if ((k & 1) == 0) {
        uint32_t x[8];
        ld_tile(x0, k >> 1, x);
        tile_mac(acc, x, x);
      }
      {
        uint32_t d[8], d2[8];
        acc_resolve_low(S, d);
        acc_shift8(S);
        d2[0] = (d[0] << 1) | topbit;
        PAI_UNROLL
        for (int j = 1; j < 8; j++) d2[j] = (d[j] << 1) | (d[j - 1] >> 31);
        topbit = d[7] >> 31;
        acc_add_low(acc, d2);
      }
      uint32_t v[8];
      if (k < NTH) {
        uint32_t m[8];
        acc_peek_low(acc, v);
        mul_lo8(m, v, ninv);
        st_tile(olo, k, m);
        tile_mac(acc, m, n0);
        acc_carry_of_zero_low(acc);
      } else {
        acc_resolve_low(acc, v);
        st_tile(ohi, k - NTH, v);
        uint32_t nt[8], d[8];
        ld_tile(N, k - NTH, nt);
        b1 = sub8b(d, v, nt, b1);
      }
      acc_shift8(acc);
    }
    uint32_t ovf = lo32(acc.E[0]) + acc.C[0] + topbit;
    carry = (ovf != 0u) | (b1 ^ 1u);
    big_sub_masked<NTH>(ohi, ohi, N, 0u - carry);
  }
  uint32_t wtop = 1u - big_rsub<NTH>(olo, KL) + carry;
  // ---- phase 2: B = 2*x0*x1 + W  (all NTH^2 cross tiles once in S, doubled on the way in)
  {
    Acc acc, S;
    acc_clear(acc);
    acc_clear(S);
    uint32_t topbit = 0, b1 = 0, b2 = 0, b3 = 0;
    for (int k = 0; k < 2 * NTH; k++) {
      int lo = k - NTH + 1 > 0 ? k - NTH + 1 : 0;
      int hi = k < NTH ? k - 1 : NTH - 1;            // reduction partners i in [lo, hi]; cross tiles i in [lo, hc]
      int hc = k < NTH ? k : NTH - 1;
      int i = lo;
      for (; i <= hi; i++) {
        uint32_t x[8], y[8], u[8], w[8];
        ld_tile(x0, i, x); ld_tile(x1, k - i, y);
        ld_tile(olo, i, u); ld_tile(N, k - i, w);
        tile_mac(S, x, y);
        tile_mac(acc, u, w);
      }
      for (; i <= hc; i++) {
        uint32_t x[8], y[8];
        ld_tile(x0, i, x); ld_tile(x1, k - i, y);
        tile_mac(S, x, y);
      }
      {
        uint32_t d[8], d2[8];
        acc_resolve_low(S, d);
        acc_shift8(S);
        d2[0] = (d[0] << 1) | topbit;
        PAI_UNROLL
        for (int j = 1; j < 8; j++) d2[j] = (d[j] << 1) | (d[j - 1] >> 31);
        topbit = d[7] >> 31;
        acc_add_low(acc, d2);
      }
      uint32_t v[8];
      if (k < NTH) {
        uint32_t x[8], m[8];
        ld_tile(olo, k, x);                                   // W_k
        acc_add_low(acc, x);
        acc_peek_low(acc, v);
        mul_lo8(m, v, ninv);
        st_tile(olo, k, m);
        tile_mac(acc, m, n0);
        acc_carry_of_zero_low(acc);
      } else {
        if (k == NTH) acc.C[0] += wtop;
        acc_resolve_low(acc, v);
        st_tile(olo, k - NTH, v);
        uint32_t nt[8], d[8];
        ld_tile(N, k - NTH, nt);      b1 = sub8b(d, v, nt, b1);
        ld_tile(dc.N2, k - NTH, nt);  b2 = sub8b(d, v, nt, b2);
        ld_tile(dc.N3, k - NTH, nt);  b3 = sub8b(d, v, nt, b3);
      }
      acc_shift8(acc);
    }
    uint32_t ovf = lo32(acc.E[0]) + acc.C[0] + topbit;
    digit_reduce3<NTH>(olo, dc, ovf, b1, b2, b3);
  }
}


// ------------------------------------------------------------------------------------------------
// Constants blob of one digit modulus (uint32 limbs, h = 8*NTH), appended to the ordinary blob of n:
//   [ blob(n): N | R1 | R2 | R3 | ONE | NINV(8) ]  [ KL (h) | RR (2h) | ONEM (2h) | ZERO (h) | E3 (2h) | E4 (2h) | E5 (2h) | N2 (h) | N3 (h) | TOPS (8) ]
// RR = digits of R^2 mod n^2, ONEM = digits of R mod n^2, Ek = digits of R^k mod n^2 (entry constants for
// double-width inputs: c = sum c_i R^i  ->  c*R = sum dmul((c_i, 0), E(i+2))).
PAI_HD int dc_extra_limbs(int NTH) { return 8 * NTH * (1 + 2 + 2 + 1 + 2 + 2 + 2 + 1 + 1) + 8; }
PAI_HD int dc_limbs(int NTH) { return 5 * 8 * NTH + 8 + dc_extra_limbs(NTH); }



template <int NTH>
PAI_DEV void digit_bind(DigitEnv& d, u4* blob) {
  const int Q = 2 * NTH;
  d.N.p = blob;               d.N.s = 1;
  d.ONE.p = blob + 4 * Q;     d.ONE.s = 1;
  d.NI.p = blob + 5 * Q;      d.NI.s = 1;
  u4* e = blob + 5 * Q + 2;
  d.KL.p = e;                 d.KL.s = 1;
  d.RR.d0.p = e + Q;          d.RR.d0.s = 1;
  d.RR.d1.p = e + 2 * Q;      d.RR.d1.s = 1;
  d.ONEM.d0.p = e + 3 * Q;    d.ONEM.d0.s = 1;
  d.ONEM.d1.p = e + 4 * Q;    d.ONEM.d1.s = 1;
  d.ZERO.p = e + 5 * Q;       d.ZERO.s = 1;
  d.E3.d0.p = e + 6 * Q;      d.E3.d0.s = 1;
  d.E3.d1.p = e + 7 * Q;      d.E3.d1.s = 1;
  d.E4.d0.p = e + 8 * Q;      d.E4.d0.s = 1;
  d.E4.d1.p = e + 9 * Q;      d.E4.d1.s = 1;
  d.E5.d0.p = e + 10 * Q;     d.E5.d0.s = 1;
  d.E5.d1.p = e + 11 * Q;     d.E5.d1.s = 1;
  d.N2.p = e + 12 * Q;        d.N2.s = 1;
  d.N3.p = e + 13 * Q;        d.N3.s = 1;
  d.TOPS.p = e + 14 * Q;      d.TOPS.s = 1;
}

// Compact constant area of the encrypt kernel (only what prog_encrypt_digit touches, so that 224 threads x
// 1 KB of operands still fit the 227 KB of shared memory at 2048-bit keys):
//   [ N (h) | ONE (h) | NINV (8) | KL (h) | RR (2h) | N2 (h) | N3 (h) | TOPS (8) ]
// (the all-zero operand is read from the global digit blob: it is only touched when entering/leaving the domain)
PAI_HD int dc_enc_limbs(int NTH) { return 8 * NTH * 7 + 16; }
// the scalar-multiplication kernel appends [ ONEM (2h) | E3 (2h) ] to the same prefix
PAI_HD int dc_pow_limbs(int NTH) { return 8 * NTH * 11 + 16; }
// offset (limbs) of the ZERO region inside the global digit blob
PAI_HD int dc_zero_offset(int NTH) { return 5 * 8 * NTH + 8 + 5 * 8 * NTH; }
template <int NTH>
PAI_DEV void digit_bind_enc(DigitEnv& d, u4* c, const uint32_t* gzero) {
  const int Q = 2 * NTH;
  d.N.p = c;                  d.N.s = 1;
  d.ONE.p = c + Q;            d.ONE.s = 1;
  d.NI.p = c + 2 * Q;         d.NI.s = 1;
  d.KL.p = c + 2 * Q + 2;     d.KL.s = 1;
  d.RR.d0.p = c + 3 * Q + 2;  d.RR.d0.s = 1;
  d.RR.d1.p = c + 4 * Q + 2;  d.RR.d1.s = 1;
  d.ZERO.p = (u4*)gzero;      d.ZERO.s = 1;
  d.N2.p = c + 5 * Q + 2;     d.N2.s = 1;
  d.N3.p = c + 6 * Q + 2;     d.N3.s = 1;
  d.TOPS.p = c + 7 * Q + 2;   d.TOPS.s = 1;
  d.ONEM = d.RR; d.E3 = d.RR; d.E4 = d.RR; d.E5 = d.RR;      // not used by encrypt
}
template <int NTH>
PAI_DEV void digit_bind_pow(DigitEnv& d, u4* c, const uint32_t* gzero) {
  const int Q = 2 * NTH;
  digit_bind_enc<NTH>(d, c, gzero);
  d.ONEM.d0.p = c + 7 * Q + 4;  d.ONEM.d0.s = 1;
  d.ONEM.d1.p = c + 8 * Q + 4;  d.ONEM.d1.s = 1;
  d.E3.d0.p = c + 9 * Q + 4;    d.E3.d0.s = 1;
  d.E3.d1.p = c + 10 * Q + 4;   d.E3.d1.s = 1;
}

// single-thread setup of the extra constants; blob(n) (N, R1, ..., NINV) must already be set up.
//   scratch: 4 * h limbs
template <int NTH>
PAI_DEV void digit_setup(uint32_t* blob, uint32_t* scratch) {
  const int h = 8 * NTH;
  const uint32_t* N = blob;
  const uint32_t* R1 = blob + h;
  uint32_t* e = blob + 5 * h + 8;
  uint32_t* KL = e;
  uint32_t* RR = e + h;
  uint32_t* ONEM = e + 3 * h;
  uint32_t* ZERO = e + 5 * h;
  uint32_t* E3 = e + 6 * h;
  uint32_t* E4 = e + 8 * h;
  uint32_t* E5 = e + 10 * h;
  { uint32_t bo = 0; for (int i = 0; i < h; i++) { uint64_t d = (uint64_t)N[i] - R1[i] - bo; KL[i] = (uint32_t)d; bo = (uint32_t)(d >> 63); } }
  for (int i = 0; i < h; i++) ZERO[i] = 0;
  // digits of 2^k mod n^2 by doubling from (1, 0); snapshot at k = 32h (R) and k = 64h (R^2)
  uint32_t* d0 = scratch;
  uint32_t* d1 = scratch + h;
  uint32_t* t = scratch + 2 * h;
  for (int i = 0; i < h; i++) { d0[i] = (i == 0); d1[i] = 0; }
  bool n_is_one = (N[0] == 1);
  for (int i = 1; i < h && n_is_one; i++) if (N[i]) n_is_one = false;
  if (n_is_one) d0[0] = 0;
  for (int it = 0; it < 64 * h; it++) {
    if (it == 32 * h) for (int i = 0; i < h; i++) { ONEM[i] = d0[i]; ONEM[h + i] = d1[i]; }
    // d0 = 2 d0; carry c0 = (2 d0 >= n)
    uint32_t c = 0;
    for (int i = 0; i < h; i++) { uint32_t v = d0[i]; d0[i] = (v << 1) | c; c = v >> 31; }
    uint32_t bo = 0;
    for (int i = 0; i < h; i++) { uint64_t d = (uint64_t)d0[i] - N[i] - bo; t[i] = (uint32_t)d; bo = (uint32_t)(d >> 63); }
    uint32_t c0 = (c || !bo) ? 1u : 0u;
    if (c0) for (int i = 0; i < h; i++) d0[i] = t[i];
    // d1 = 2 d1 + c0 mod n
    c = c0;
    for (int i = 0; i < h; i++) { uint32_t v = d1[i]; d1[i] = (v << 1) | c; c = v >> 31; }
    bo = 0;
    for (int i = 0; i < h; i++) { uint64_t d = (uint64_t)d1[i] - N[i] - bo; t[i] = (uint32_t)d; bo = (uint32_t)(d >> 63); }
    if (c || !bo) for (int i = 0; i < h; i++) d1[i] = t[i];
  }
  for (int i = 0; i < h; i++) { RR[i] = d0[i]; RR[h + i] = d1[i]; }
  // E3 = RR*RR/R = R^3, E4 = E3*RR/R, E5 = E4*RR/R   (digit Montgomery products, stride-1 operands)
  // N2 = 2n mod R, N3 = 3n mod R and their overflow words
  uint32_t* N2 = e + 12 * h;
  uint32_t* N3 = e + 13 * h;
  uint32_t* TOPS = e + 14 * h;
  {
    uint64_t c = 0;
    for (int i = 0; i < h; i++) { c += 2ull * N[i]; N2[i] = (uint32_t)c; c >>= 32; }
    TOPS[0] = (uint32_t)c;
    c = 0;
    for (int i = 0; i < h; i++) { c += 3ull * N[i]; N3[i] = (uint32_t)c; c >>= 32; }
    TOPS[1] = (uint32_t)c;
    for (int i = 2; i < 8; i++) TOPS[i] = 0;
  }
  DigitEnv env;
  digit_bind<NTH>(env, (u4*)blob);
  Opnd r0{(u4*)RR, 1}, r1{(u4*)(RR + h), 1};
  Opnd tmp{(u4*)scratch, 1};                                  // 2h limbs: lo | hi
  uint32_t* Es[3] = {E3, E4, E5};
  Opnd p0 = r0, p1 = r1;
  for (int k = 0; k < 3; k++) {
    dmul<NTH>(half_lo<NTH>(tmp), half_hi<NTH>(tmp), p0, p1, r0, r1, &env);
    for (int i = 0; i < h; i++) { Es[k][i] = scratch[h + i]; Es[k][h + i] = scratch[i]; }     // (Z0 = hi, Z1 = lo)
    p0.p = (u4*)Es[k]; p1.p = (u4*)(Es[k] + h);
  }
}

// ------------------------------------------------------------------------------------------------
// Exponentiation in digit form with a host-built sliding-window program (see sliding_program in
// pai_engine.cu): two shared-memory buffers of 2*NTH tiles; a number sits in a buffer either as
// [d0 | d1] (swapped = 0) or, right after dmul/dsqr, as [d1 | d0] (swapped = 1).  Table entries live in
// global memory as [d0 | d1] and are consumed from there.
template <int NTH>
struct DPowEnv {
  Opnd buf[2];
  Opnd tbl;           // entry e, quad q at tbl.p[(e * 4*NTH + q) * tbl.s]
  DigitEnv* dc;
  int step_sync;      // 1: every thread of the CTA runs the same ladder -> barrier before each step (I-cache locality)
};

template <int NTH>
PAI_DEV DNum dview(const Opnd& b, int swapped) {
  DNum d;
  d.d0 = swapped ? half_hi<NTH>(b) : half_lo<NTH>(b);
  d.d1 = swapped ? half_lo<NTH>(b) : half_hi<NTH>(b);
  return d;
}
template <int NTH>
PAI_DEV DNum dtbl_entry(const DPowEnv<NTH>& E, int e) {
  Opnd o;
  o.p = E.tbl.p + (size_t)e * 4 * NTH * E.tbl.s;
  o.s = E.tbl.s;
  return dview<NTH>(o, 0);
}
template <int NTH>
PAI_DEV void dtbl_store(const DPowEnv<NTH>& E, int e, const DNum& x) {
  DNum t = dtbl_entry<NTH>(E, e);
  for (int q = 0; q < 2 * NTH; q++) { t.d0.p[q * t.d0.s] = x.d0.p[q * x.d0.s]; t.d1.p[q * t.d1.s] = x.d1.p[q * x.d1.s]; }
}

// base in (buf[bi], swapped sw).  Returns buffer index; *sw_out = its orientation.
template <int NTH>
PAI_DEV int dpow_prog(const DPowEnv<NTH>& E, int bi, int sw, const uint32_t* prog, int nops, int nodd, int* sw_out) {
  const DigitEnv& dc = *E.dc;
  int cur = bi, oth = bi ^ 1;
  if (nops <= 0) {                                                        // exponent 0 -> Montgomery one
    DNum o = dview<NTH>(E.buf[oth], 0);
    big_copy<NTH>(o.d0, dc.ONEM.d0);
    big_copy<NTH>(o.d1, dc.ONEM.d1);
    *sw_out = 0;
    return oth;
  }
  DNum x = dview<NTH>(E.buf[cur], sw);
  dtbl_store<NTH>(E, 0, x);                                               // T[0] = base
  if (nodd > 1) {
    dsqr<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, &dc);
    dtbl_store<NTH>(E, nodd, dview<NTH>(E.buf[oth], 1));                  // base^2
    const DNum b2 = dtbl_entry<NTH>(E, nodd);
    for (int k = 1; k < nodd; k++) {                                      // T[k] = T[k-1] * base^2
      x = dview<NTH>(E.buf[cur], sw);
      dmul<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, b2.d0, b2.d1, &dc);
      { int t = cur; cur = oth; oth = t; }
      sw = 1;
      dtbl_store<NTH>(E, k, dview<NTH>(E.buf[cur], sw));
    }
  }
  {                                                                       // initial value T[idx]
    const DNum t0 = dtbl_entry<NTH>(E, (int)(prog[0] & 0xffffu));
    DNum c = dview<NTH>(E.buf[cur], 0);
    big_copy<NTH>(c.d0, t0.d0);
    big_copy<NTH>(c.d1, t0.d1);
    sw = 0;
  }
  for (int i = 1; i < nops; i++) {
    const uint32_t op = prog[i];
    const int nsq = (int)(op >> 16), idx = (int)(op & 0xffffu);
    for (int s = 0; s < nsq; s++) {
      if (E.step_sync) cta_step_sync();
      x = dview<NTH>(E.buf[cur], sw);
      dsqr<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, &dc);
      int t = cur; cur = oth; oth = t;
      sw = 1;
    }
    if (idx != 0xffff) {
      if (E.step_sync) cta_step_sync();
      x = dview<NTH>(E.buf[cur], sw);
      const DNum te = dtbl_entry<NTH>(E, idx);
      dmul<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, te.d0, te.d1, &dc);
      int t = cur; cur = oth; oth = t;
      sw = 1;
    }
  }
  *sw_out = sw;
  return cur;
}

// out (2*NTH tiles) = d0 + n * d1   (plain integer from canonical digits); out must not alias d0/d1
template <int NTH>
PAI_DEV void digits_to_plain(const Opnd& out, const DNum& x, const Opnd& N) {
  big_mul<NTH, NTH, 2 * NTH>(out, x.d1, N, 0u);
  uint32_t c = 0;
  for (int t = 0; t < 2 * NTH; t++) {
    uint32_t a[8], b[8], r[8];
    ld_tile(out, t, a);
    if (t < NTH) ld_tile(x.d0, t, b);
    else { PAI_UNROLL for (int i = 0; i < 8; i++) b[i] = 0; }
    c = add8c(r, a, b, c);
    st_tile(out, t, r);
  }
}

// raw_encrypt in digit form (phe/paillier.py:102-139):  c = (1 + n*m) * r^n mod n^2.
//   (r, 0) enters the Montgomery domain by a product with RR; the final product with the PLAIN digit pair
//   (1, m) of the nude ciphertext 1 + n*m leaves it again; r and m are read straight from their global rows.
template <int NTH>
PAI_DEV void prog_encrypt_digit(const DPowEnv<NTH>& E, const uint32_t* prog, int nops, int nodd,
                                const uint32_t* m_row, const uint32_t* r_row, uint32_t* out_row, bool store) {
  const DigitEnv& dc = *E.dc;
  Opnd r_op{(u4*)r_row, 1}, m_op{(u4*)m_row, 1};
  dmul<NTH>(half_lo<NTH>(E.buf[0]), half_hi<NTH>(E.buf[0]), r_op, dc.ZERO, dc.RR.d0, dc.RR.d1, &dc);
  int sw = 1;
  int cur = dpow_prog<NTH>(E, 0, 1, prog, nops, nodd, &sw);
  int oth = cur ^ 1;
  DNum x = dview<NTH>(E.buf[cur], sw);
  dmul<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, dc.ONE, m_op, &dc);
  digits_to_plain<NTH>(E.buf[cur], dview<NTH>(E.buf[oth], 1), dc.N);
  if (store) store_row(out_row, E.buf[cur], 4 * NTH);
}


// ------------------------------------------------------------------------------------------------
// Fixed-window exponentiation in digit form (secret exponent shared by the batch: decrypt's p-1 / q-1;
// no digit is skipped).  Table: T[0] = 1, T[1] = base, T[i] = T[i-1]*base, 2^W entries in global memory.
template <int NTH, int W>
PAI_DEV int dpow_fixed(const DPowEnv<NTH>& E, int bi, int sw, const uint32_t* e, int nl, int nwin, int* sw_out) {
  const DigitEnv& dc = *E.dc;
  int cur = bi, oth = bi ^ 1;
  if (nwin <= 0) {
    DNum o = dview<NTH>(E.buf[oth], 0);
    big_copy<NTH>(o.d0, dc.ONEM.d0);
    big_copy<NTH>(o.d1, dc.ONEM.d1);
    *sw_out = 0;
    return oth;
  }
  DNum x = dview<NTH>(E.buf[cur], sw);
  dtbl_store<NTH>(E, 0, dc.ONEM);
  dtbl_store<NTH>(E, 1, x);
  const DNum t1 = dtbl_entry<NTH>(E, 1);
  dsqr<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, &dc);
  { int t = cur; cur = oth; oth = t; }
  sw = 1;
  dtbl_store<NTH>(E, 2, dview<NTH>(E.buf[cur], sw));
  for (int i = 3; i < (1 << W); i++) {
    x = dview<NTH>(E.buf[cur], sw);
    dmul<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, t1.d0, t1.d1, &dc);
    { int t = cur; cur = oth; oth = t; }
    dtbl_store<NTH>(E, i, dview<NTH>(E.buf[cur], sw));
  }
  {
    const DNum t0 = dtbl_entry<NTH>(E, (int)exp_digit(e, nl, (nwin - 1) * W, W));
    DNum c = dview<NTH>(E.buf[cur], 0);
    big_copy<NTH>(c.d0, t0.d0);
    big_copy<NTH>(c.d1, t0.d1);
    sw = 0;
  }
  for (int wi = nwin - 2; wi >= 0; wi--) {
    for (int s = 0; s < W; s++) {
      if (E.step_sync) cta_step_sync();
      x = dview<NTH>(E.buf[cur], sw);
      dsqr<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, &dc);
      int t = cur; cur = oth; oth = t;
      sw = 1;
    }
    if (E.step_sync) cta_step_sync();
    x = dview<NTH>(E.buf[cur], sw);
    const DNum te = dtbl_entry<NTH>(E, (int)exp_digit(e, nl, wi * W, W));
    dmul<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, te.d0, te.d1, &dc);
    int t = cur; cur = oth; oth = t;
    sw = 1;
  }
  *sw_out = sw;
  return cur;
}

// a += b in digit form (canonical digits in, canonical digits out)
template <int NTH>
PAI_DEV void dadd(const DNum& a, const DNum& b, const Opnd& N) {
  uint32_t c = big_add_masked<NTH>(a.d0, a.d0, b.d0, 0xffffffffu);
  uint32_t carry = big_cond_sub<NTH>(a.d0, N, c);
  // a.d1 = a.d1 + b.d1 + carry  (< 2n) then one conditional subtraction
  uint32_t cc = carry;
  for (int t = 0; t < NTH; t++) {
    uint32_t x[8], y[8], r[8];
    ld_tile(a.d1, t, x); ld_tile(b.d1, t, y);
    cc = add8c(r, x, y, cc);
    st_tile(a.d1, t, r);
  }
  big_cond_sub<NTH>(a.d1, N, cc);
}

// ------------------------------------------------------------------------------------------------
// raw_decrypt with CRT in digit form (phe/paillier.py:328-374).
// One prime side x in {p, q}: constants = digit blob of x (digit_bind layout) followed by hM (h(x)*R mod x,
// Montgomery form mod x) and the exponent x - 1.
template <int NTP>
struct DSideC {
  DigitEnv dc;
  Opnd R1;            // (unused placeholder for symmetry with the blob layout)
  Opnd hM;
  const uint32_t* e;
  int nwin;
};
template <int NTP>
PAI_HD int dside_limbs() { return dc_limbs(NTP) + 2 * 8 * NTP; }
template <int NTP>
PAI_DEV void dside_bind(DSideC<NTP>& S, u4* base, int nwin) {
  digit_bind<NTP>(S.dc, base);
  u4* p = base + dc_limbs(NTP) / 4;
  S.hM.p = p; S.hM.s = 1;
  S.R1 = S.hM;
  S.e = (const uint32_t*)(p + 2 * NTP);
  S.nwin = nwin;
}

// out: m_x = L(c^(x-1) mod x^2) * h mod x  (NTP tiles) in the LOW half of buf[ret]
template <int NTP, int W>
PAI_DEV int decrypt_half_digit(DPowEnv<NTP>& E, DSideC<NTP>& S, const uint32_t* c_row) {
  DigitEnv& dc = S.dc;
  E.dc = &dc;
  const DNum Ek[4] = {dc.RR, dc.E3, dc.E4, dc.E5};
  // X = c * R mod x^2:  c = sum_i c_i R^i (four pieces of NTP tiles, read from the global row)
  Opnd c0{(u4*)c_row, 1};
  dmul<NTP>(half_lo<NTP>(E.buf[0]), half_hi<NTP>(E.buf[0]), c0, dc.ZERO, Ek[0].d0, Ek[0].d1, &dc);
  for (int i = 1; i < 4; i++) {
    Opnd ci{(u4*)(c_row + (size_t)i * 8 * NTP), 1};
    dmul<NTP>(half_lo<NTP>(E.buf[1]), half_hi<NTP>(E.buf[1]), ci, dc.ZERO, Ek[i].d0, Ek[i].d1, &dc);
    dadd<NTP>(dview<NTP>(E.buf[0], 1), dview<NTP>(E.buf[1], 1), dc.N);
  }
  int sw = 1;
  int cur = dpow_fixed<NTP, W>(E, 0, 1, S.e, 8 * NTP, S.nwin, &sw);      // c^(x-1) * R mod x^2
  int oth = cur ^ 1;
  DNum x = dview<NTP>(E.buf[cur], sw);
  dmul<NTP>(half_lo<NTP>(E.buf[oth]), half_hi<NTP>(E.buf[oth]), x.d0, x.d1, dc.ONE, dc.ZERO, &dc);
  // plain digits u = u0 + x*u1:  L(u) = (u-1)//x = u1 if u0 >= 1;  u0 == 0: u1 - 1, and -1 = x - 1 (mod x) if u1 == 0
  DNum u = dview<NTP>(E.buf[oth], 1);
  uint32_t u0z = big_is_zero<NTP>(u.d0);
  uint32_t u1z = big_is_zero<NTP>(u.d1);
  big_sub_masked<NTP>(u.d1, u.d1, dc.ONE, 0u - (u0z & (u1z ^ 1u)));
  {
    const uint32_t sel = u0z & u1z;
    for (int t = 0; t < NTP; t++) {
      uint32_t l[8], n[8];
      ld_tile(u.d1, t, l); ld_tile(dc.N, t, n);
      if (t == 0) n[0] -= 1u;                                             // x is odd: no borrow
      PAI_UNROLL
      for (int i = 0; i < 8; i++) l[i] = sel ? n[i] : l[i];
      st_tile(u.d1, t, l);
    }
  }
  mont_mul<NTP>(half_lo<NTP>(E.buf[cur]), u.d1, S.hM, dc.N, dc.NI);        // L * h mod x
  return cur;
}

template <int NTP, int W>
PAI_DEV void prog_decrypt_digit(DPowEnv<NTP>& E, DSideC<NTP>& P, DSideC<NTP>& Qs, const Opnd& pinvqM,
                                const uint32_t* c_row, uint32_t* out_row, bool store) {
  int ip = decrypt_half_digit<NTP, W>(E, P, c_row);
  if (store) store_row(out_row, half_lo<NTP>(E.buf[ip]), 2 * NTP);        // m_p -> global (low half of the row)
  int c = decrypt_half_digit<NTP, W>(E, Qs, c_row);
  int o = c ^ 1;
  Opnd mq = half_lo<NTP>(E.buf[c]), mp = half_hi<NTP>(E.buf[c]);
  if (store) load_row(mp, out_row, 2 * NTP, 2 * NTP);
  else big_copy<NTP>(mp, mq);
  // u = (m_q - m_p) * p^-1 mod q     (m_p < p < q, m_q < q)
  uint32_t bo = big_sub_masked<NTP>(mq, mq, mp, 0xffffffffu);
  big_add_masked<NTP>(mq, mq, Qs.dc.N, 0u - bo);
  Opnd uo = half_lo<NTP>(E.buf[o]), mp2 = half_hi<NTP>(E.buf[o]);
  mont_mul<NTP>(uo, mq, pinvqM, Qs.dc.N, Qs.dc.NI);
  big_copy<NTP>(mp2, mp);
  // m = m_p + u * p
  big_mul<NTP, NTP, 2 * NTP>(E.buf[c], uo, P.dc.N, 0u);
  uint32_t cy = 0;
  for (int t = 0; t < 2 * NTP; t++) {
    uint32_t a[8], b[8], r[8];
    ld_tile(E.buf[c], t, a);
    if (t < NTP) ld_tile(mp2, t, b);
    else { PAI_UNROLL for (int i = 0; i < 8; i++) b[i] = 0; }
    cy = add8c(r, a, b, cy);
    st_tile(E.buf[c], t, r);
  }
  if (store) store_row(out_row, E.buf[c], 4 * NTP);
}


// ------------------------------------------------------------------------------------------------
// Encryption with the private key (pai_priv_encrypt): c = (1 + n*m) * r^n mod n^2 through the CRT, n = p*q with p < q.
// For x in {p, q} and y the other prime:
//   r^n = (r^x)^y = s^x (mod x^2),  s = (r mod x)^(y mod (x-1)) mod x     (x-th powers mod x^2 depend on r mod x only,
//                                                                          and r^x mod x^2 has order dividing x - 1)
//   1 + n*m = 1 + x*((y*m) mod x)  (mod x^2): the plain digit pair (1, t_x), t_x = y*m mod x
//   c = c_p + p^2 * h,  h = (c_q - c_p) * p^-2 mod q^2                    (Garner; c_p < p^2 < q^2, so c < n^2 as it stands)
// Both exponents are secret and run through fixed windows with no digit skipped.  x | r gives s = 0 (y mod (x-1) >= 1),
// hence r^n = 0 mod x^2, as it must.
// The warp-per-ciphertext route computes r^n mod x^2 as r^(n mod x(x-1)) on the warp kernels and passes the plain results
// in (pre_p / pre_q): n mod x(x-1) = x * (y mod (x-1)) >= x, so that form holds for every r, x | r included.
// Constants of one side:  [ digit blob of x (dc_limbs) | yR = y*R mod x | yR2 = y*R^2 mod x | e1 = y mod (x-1) ]
// after the two sides:    [ K1 = p^-2*R | K1N = -p^-2*R | K2N = -p^-2*R^2 (mod q^2, digit pairs [d0 | d1]) | P2 = p^2 (plain) ]
template <int NTH>
PAI_DEV void digit_enter(const DPowEnv<NTH>& E, const uint32_t* base_row);

template <int NTP>
struct PESideC {
  DigitEnv dc;
  Opnd R1, R2, R3;    // R^k mod x (blob of x)
  Opnd yR, yR2;
  const uint32_t* e1;
  int nwin;           // windows of both exponents (bit length of x)
};
template <int NTP>
struct PEncC {
  PESideC<NTP> P, Q;
  DNum K1, K1N, K2N;
  Opnd P2;
};
template <int NTP>
PAI_HD int pe_side_limbs() { return dc_limbs(NTP) + 3 * 8 * NTP; }
template <int NTP>
PAI_HD int pe_const_limbs() { return 2 * pe_side_limbs<NTP>() + 4 * 16 * NTP; }
// table slots per thread: the 2^W window entries, then [t_p | t_q] and the parked c_p
PAI_HD int pe_slots(int W) { return (1 << W) + 2; }

template <int NTP>
PAI_DEV void pe_side_bind(PESideC<NTP>& S, u4* base, int nwin) {
  const int Q = 2 * NTP;
  digit_bind<NTP>(S.dc, base);
  S.R1.p = base + Q;          S.R1.s = 1;
  S.R2.p = base + 2 * Q;      S.R2.s = 1;
  S.R3.p = base + 3 * Q;      S.R3.s = 1;
  u4* p = base + dc_limbs(NTP) / 4;
  S.yR.p = p;                 S.yR.s = 1;
  S.yR2.p = p + Q;            S.yR2.s = 1;
  S.e1 = (const uint32_t*)(p + 2 * Q);
  S.nwin = nwin;
}
template <int NTP>
PAI_DEV void pe_bind(PEncC<NTP>& C, u4* smem, int nwin_p, int nwin_q) {
  const int Q = 2 * NTP;
  pe_side_bind<NTP>(C.P, smem, nwin_p);
  pe_side_bind<NTP>(C.Q, smem + pe_side_limbs<NTP>() / 4, nwin_q);
  u4* k = smem + 2 * (pe_side_limbs<NTP>() / 4);
  DNum* ks[3] = {&C.K1, &C.K1N, &C.K2N};
  for (int i = 0; i < 3; i++) {
    ks[i]->d0.p = k + 2 * i * Q;       ks[i]->d0.s = 1;
    ks[i]->d1.p = k + (2 * i + 1) * Q; ks[i]->d1.s = 1;
  }
  C.P2.p = k + 6 * Q;         C.P2.s = 1;
}

// t = y*m mod x = m0*yR/R + m1*yR2/R (m = m0 + m1*R, any m < R^2); tmp: NTP tiles of scratch
template <int NTP>
PAI_DEV void pe_msg_digit(const Opnd& t, const Opnd& tmp, const PESideC<NTP>& S, const uint32_t* m_row) {
  Opnd m0{(u4*)m_row, 1}, m1{(u4*)(m_row + 8 * NTP), 1};
  mont_mul<NTP>(t, m0, S.yR, S.dc.N, S.dc.NI);
  mont_mul<NTP>(tmp, m1, S.yR2, S.dc.N, S.dc.NI);
  uint32_t c = big_add_masked<NTP>(t, t, tmp, 0xffffffffu);
  big_cond_sub<NTP>(t, S.dc.N, c);
}

// Step 1: base^e * R mod x by fixed windows (no digit skipped) on half-width operands.  The base (Montgomery form mod x)
// is in the low half of buf[0]; window entry i is the low half of table slot i.  Returns the operand holding the result.
template <int NTP, int W>
PAI_DEV Opnd mpow_fixed(const DPowEnv<NTP>& E, const PESideC<NTP>& S, const uint32_t* e, int nwin) {
  const Opnd N = S.dc.N, NI = S.dc.NI;
  const Opnd b = half_lo<NTP>(E.buf[0]);
  Opnd cur = half_lo<NTP>(E.buf[1]), oth = half_hi<NTP>(E.buf[1]);
  big_copy<NTP>(dtbl_entry<NTP>(E, 0).d0, S.R1);
  big_copy<NTP>(dtbl_entry<NTP>(E, 1).d0, b);
  mont_sqr<NTP>(cur, b, N, NI);
  big_copy<NTP>(dtbl_entry<NTP>(E, 2).d0, cur);
  for (int i = 3; i < (1 << W); i++) {
    mont_mul<NTP>(oth, cur, b, N, NI);
    { Opnd t = cur; cur = oth; oth = t; }
    big_copy<NTP>(dtbl_entry<NTP>(E, i).d0, cur);
  }
  big_copy<NTP>(cur, dtbl_entry<NTP>(E, (int)exp_digit(e, 8 * NTP, (nwin - 1) * W, W)).d0);
  for (int wi = nwin - 2; wi >= 0; wi--) {
    for (int s = 0; s < W; s++) {
      if (E.step_sync) cta_step_sync();
      mont_sqr<NTP>(oth, cur, N, NI);
      Opnd t = cur; cur = oth; oth = t;
    }
    if (E.step_sync) cta_step_sync();
    mont_mul<NTP>(oth, cur, dtbl_entry<NTP>(E, (int)exp_digit(e, 8 * NTP, wi * W, W)).d0, N, NI);
    Opnd t = cur; cur = oth; oth = t;
  }
  return cur;
}

// r^n mod x^2 in Montgomery digit form -> (buf[ret], orientation *sw).  r = r0 + r1*R (any r < R^2).
template <int NTP, int W>
PAI_DEV int pe_pow_side(DPowEnv<NTP>& E, PESideC<NTP>& S, const uint32_t* r_row, int* sw) {
  DigitEnv& dc = S.dc;
  E.dc = &dc;
  Opnd r0{(u4*)r_row, 1}, r1{(u4*)(r_row + 8 * NTP), 1};
  const Opnd a = half_lo<NTP>(E.buf[0]), t = half_hi<NTP>(E.buf[0]), u = half_lo<NTP>(E.buf[1]);
  mont_mul<NTP>(t, r0, S.R2, dc.N, dc.NI);                                // r0 * R
  mont_mul<NTP>(u, r1, S.R3, dc.N, dc.NI);                                // r1 * R^2
  uint32_t c = big_add_masked<NTP>(a, t, u, 0xffffffffu);
  big_cond_sub<NTP>(a, dc.N, c);                                          // r * R mod x
  const Opnd s = mpow_fixed<NTP, W>(E, S, S.e1, S.nwin);                  // s * R mod x
  // (s*R mod x, 0) read as a Montgomery digit pair stands for some s' = s (mod x), and s'^x = s^x (mod x^2)
  big_copy<NTP>(a, s);
  big_copy<NTP>(t, dc.ZERO);
  return dpow_fixed<NTP, W>(E, 0, 0, (const uint32_t*)dc.N.p, 8 * NTP, S.nwin, sw);   // s^x * R mod x^2
}

// The tail shared by the thread-per-ciphertext and the warp-per-ciphertext routes.  Side p: c_p = omega_p * (1, t_p) as a
// plain number, parked in table slot 2^W + 1.  omega: r^n mod p^2 in Montgomery digit form in (buf[cur], sw).
template <int NTP, int W>
PAI_DEV void pe_finish_p(const DPowEnv<NTP>& E, const PEncC<NTP>& C, int cur, int sw) {
  const DigitEnv& dc = C.P.dc;
  const int oth = cur ^ 1;
  const DNum x = dview<NTP>(E.buf[cur], sw);
  dmul<NTP>(half_lo<NTP>(E.buf[oth]), half_hi<NTP>(E.buf[oth]), x.d0, x.d1, dc.ONE, dtbl_entry<NTP>(E, 1 << W).d0, &dc);
  digits_to_plain<NTP>(E.buf[cur], dview<NTP>(E.buf[oth], 1), dc.N);
  big_copy<2 * NTP>(dtbl_entry<NTP>(E, (1 << W) + 1).d0, E.buf[cur]);
}
// Side q and the CRT: h = (omega_q * (1, t_q) - c_p) * p^-2 mod q^2, c = c_p + p^2 * h (4*NTP tiles, buf[0] and buf[1]
// read as one operand: the two buffers of a thread are adjacent in the interleaved layout).
template <int NTP, int W>
PAI_DEV void pe_finish_q(const DPowEnv<NTP>& E, const PEncC<NTP>& C, int cur, int sw, uint32_t* out_row, bool store) {
  const DigitEnv& dc = C.Q.dc;
  const int oth = cur ^ 1;
  const Opnd cp = dtbl_entry<NTP>(E, (1 << W) + 1).d0;                    // c_p = cp_lo + cp_hi * R
  const Opnd cp_hi{cp.p + (size_t)(2 * NTP) * cp.s, cp.s};
  DNum x = dview<NTP>(E.buf[cur], sw);
  dmul<NTP>(half_lo<NTP>(E.buf[oth]), half_hi<NTP>(E.buf[oth]), x.d0, x.d1, C.K1.d0, C.K1.d1, &dc);        // omega_q p^-2 R
  x = dview<NTP>(E.buf[oth], 1);
  dmul<NTP>(half_lo<NTP>(E.buf[cur]), half_hi<NTP>(E.buf[cur]), x.d0, x.d1, dc.ONE, dtbl_entry<NTP>(E, 1 << W).d1, &dc);   // c_q p^-2
  dmul<NTP>(half_lo<NTP>(E.buf[oth]), half_hi<NTP>(E.buf[oth]), cp, dc.ZERO, C.K1N.d0, C.K1N.d1, &dc);      // -cp_lo p^-2
  dadd<NTP>(dview<NTP>(E.buf[cur], 1), dview<NTP>(E.buf[oth], 1), dc.N);
  dmul<NTP>(half_lo<NTP>(E.buf[oth]), half_hi<NTP>(E.buf[oth]), cp_hi, dc.ZERO, C.K2N.d0, C.K2N.d1, &dc);   // -cp_hi R p^-2
  dadd<NTP>(dview<NTP>(E.buf[cur], 1), dview<NTP>(E.buf[oth], 1), dc.N);                                   // h, digits
  const Opnd h = dtbl_entry<NTP>(E, 0).d0;
  digits_to_plain<NTP>(E.buf[oth], dview<NTP>(E.buf[cur], 1), dc.N);
  big_copy<2 * NTP>(h, E.buf[oth]);
  big_mul<2 * NTP, 2 * NTP, 4 * NTP>(E.buf[0], h, C.P2, 0u);
  uint32_t cy = 0;
  for (int t = 0; t < 4 * NTP; t++) {
    uint32_t a[8], b[8], r[8];
    ld_tile(E.buf[0], t, a);
    if (t < 2 * NTP) ld_tile(cp, t, b);
    else { PAI_UNROLL for (int i = 0; i < 8; i++) b[i] = 0; }
    cy = add8c(r, a, b, cy);
    st_tile(E.buf[0], t, r);
  }
  if (store) store_row(out_row, E.buf[0], 8 * NTP);
}

// One ciphertext.  pre_p / pre_q (plain rows r^n mod x^2 computed by the warp kernels) replace the two exponentiations.
template <int NTP, int W>
PAI_DEV void prog_priv_encrypt_digit(DPowEnv<NTP>& E, PEncC<NTP>& C, const uint32_t* m_row, const uint32_t* r_row,
                                     const uint32_t* pre_p, const uint32_t* pre_q, uint32_t* out_row, bool store) {
  const DNum tpq = dtbl_entry<NTP>(E, 1 << W);                            // [t_p | t_q]
  pe_msg_digit<NTP>(half_lo<NTP>(E.buf[0]), half_hi<NTP>(E.buf[0]), C.P, m_row);
  big_copy<NTP>(tpq.d0, half_lo<NTP>(E.buf[0]));
  pe_msg_digit<NTP>(half_lo<NTP>(E.buf[0]), half_hi<NTP>(E.buf[0]), C.Q, m_row);
  big_copy<NTP>(tpq.d1, half_lo<NTP>(E.buf[0]));
  PESideC<NTP>* sides[2] = {&C.P, &C.Q};
  const uint32_t* pre[2] = {pre_p, pre_q};
  for (int i = 0; i < 2; i++) {
    int cur = 0, sw = 1;
    if (pre[i]) {
      E.dc = &sides[i]->dc;
      digit_enter<NTP>(E, pre[i]);
    } else {
      cur = pe_pow_side<NTP, W>(E, *sides[i], r_row, &sw);
    }
    if (i == 0) pe_finish_p<NTP, W>(E, C, cur, sw);
    else pe_finish_q<NTP, W>(E, C, cur, sw, out_row, store);
  }
}


// ------------------------------------------------------------------------------------------------
// Entering and leaving the digit-Montgomery domain of n^2 for a plain ciphertext row (2*NTH tiles = c_0 + c_1*R).
// Entry: c*R = dmul((c_0, 0), RR) + dmul((c_1, 0), E3), left in buf[0] as [d1 | d0] (swapped = 1); uses both buffers.
template <int NTH>
PAI_DEV void digit_enter(const DPowEnv<NTH>& E, const uint32_t* base_row) {
  const DigitEnv& dc = *E.dc;
  Opnd c0{(u4*)base_row, 1}, c1{(u4*)(base_row + 8 * NTH), 1};
  dmul<NTH>(half_lo<NTH>(E.buf[0]), half_hi<NTH>(E.buf[0]), c0, dc.ZERO, dc.RR.d0, dc.RR.d1, &dc);
  dmul<NTH>(half_lo<NTH>(E.buf[1]), half_hi<NTH>(E.buf[1]), c1, dc.ZERO, dc.E3.d0, dc.E3.d1, &dc);
  dadd<NTH>(dview<NTH>(E.buf[0], 1), dview<NTH>(E.buf[1], 1), dc.N);
}
// Exit: the number in (buf[cur], orientation sw) times (1, 0), then the plain integer d0 + n*d1 -> out_row (4*NTH quads).
template <int NTH>
PAI_DEV void digit_leave_store(const DPowEnv<NTH>& E, int cur, int sw, uint32_t* out_row, bool store) {
  const DigitEnv& dc = *E.dc;
  int oth = cur ^ 1;
  DNum x = dview<NTH>(E.buf[cur], sw);
  dmul<NTH>(half_lo<NTH>(E.buf[oth]), half_hi<NTH>(E.buf[oth]), x.d0, x.d1, dc.ONE, dc.ZERO, &dc);
  digits_to_plain<NTH>(E.buf[cur], dview<NTH>(E.buf[oth], 1), dc.N);
  if (store) store_row(out_row, E.buf[cur], 4 * NTH);
}

// c^k mod n^2 with per-element exponents in digit form (EncryptedNumber._raw_mul, phe/paillier.py:749-751).
//   base row: plain ciphertext, 2*NTH tiles = c_0 + c_1*R;  e: exponent limbs of this element; nwin uniform.
template <int NTH, int W>
PAI_DEV void prog_powmod_digit(DPowEnv<NTH>& E, const uint32_t* base_row, const uint32_t* e, int nl, int nwin,
                               uint32_t* out_row, bool store) {
  digit_enter<NTH>(E, base_row);
  int sw = 1;
  int cur = dpow_fixed<NTH, W>(E, 0, 1, e, nl, nwin, &sw);
  digit_leave_store<NTH>(E, cur, sw, out_row, store);
}

// ------------------------------------------------------------------------------------------------
// Plaintext matrix (CSR) times ciphertext vector (pai_raw_matvec): out[j] = prod_t T[col_t, sign_t] ^ mag_t mod n^2.
// Window tables are built once per base and shared by every row.  Slot s < ncols holds the powers of c[s], slot
// ncols + i those of c[i]^-1 (built only for columns used with a negative scalar).  Entry k = 1 .. 2^w - 1 of a slot is
// base^k * R in digit form, [d0 | d1] with stride 1, at quad (s * (2^w - 1) + k - 1) * 4*NTH of the table.
template <int NTH>
PAI_DEV DNum mv_entry(const u4* tbl, long slot, int w, uint32_t k) {
  Opnd o;
  o.p = (u4*)tbl + ((size_t)slot * ((1u << w) - 1u) + (k - 1u)) * 4 * NTH;
  o.s = 1;
  return dview<NTH>(o, 0);
}
template <int NTH>
PAI_DEV void dnum_copy(const DNum& dst, const DNum& src) {
  big_copy<NTH>(dst.d0, src.d0);
  big_copy<NTH>(dst.d1, src.d1);
}

// the 2^w - 1 entries of one slot: T[1] = base * R, T[k] = T[k-1] * T[1]  (2^w - 2 products, serial)
template <int NTH>
PAI_DEV void prog_matvec_table(const DPowEnv<NTH>& E, const uint32_t* base_row, u4* tbl, long slot, int w) {
  digit_enter<NTH>(E, base_row);
  const DNum t1 = mv_entry<NTH>(tbl, slot, w, 1);
  dnum_copy<NTH>(t1, dview<NTH>(E.buf[0], 1));
  int cur = 0;
  for (uint32_t k = 2; k < (1u << w); k++) {
    DNum x = dview<NTH>(E.buf[cur], 1);
    dmul<NTH>(half_lo<NTH>(E.buf[cur ^ 1]), half_hi<NTH>(E.buf[cur ^ 1]), x.d0, x.d1, t1.d0, t1.d1, E.dc);
    cur ^= 1;
    dnum_copy<NTH>(mv_entry<NTH>(tbl, slot, w, k), dview<NTH>(E.buf[cur], 1));
  }
}

// One output row by Straus' method over the row's entries [lo, hi): the accumulator starts at one (R in digit form);
// window wi (top down) costs w squarings (none for the top window) and one product per entry whose digit is non-zero.
template <int NTH>
PAI_DEV void prog_matvec_row(const DPowEnv<NTH>& E, const u4* tbl, long ncols, int w, int nwin, const int32_t* indices,
                             const uint32_t* mag, int ml, const uint8_t* neg, long lo, long hi, uint32_t* out_row, bool store) {
  const DigitEnv& dc = *E.dc;
  int cur = 0, sw = 0;
  dnum_copy<NTH>(dview<NTH>(E.buf[0], 0), dc.ONEM);
  for (int wi = nwin - 1; wi >= 0; wi--) {
    if (wi != nwin - 1) {
      for (int s = 0; s < w; s++) {
        DNum x = dview<NTH>(E.buf[cur], sw);
        dsqr<NTH>(half_lo<NTH>(E.buf[cur ^ 1]), half_hi<NTH>(E.buf[cur ^ 1]), x.d0, x.d1, &dc);
        cur ^= 1;
        sw = 1;
      }
    }
    for (long t = lo; t < hi; t++) {
      const uint32_t dg = exp_digit(mag + t * ml, ml, wi * w, w);
      if (!dg) continue;
      const long slot = (neg && neg[t]) ? ncols + indices[t] : (long)indices[t];
      const DNum te = mv_entry<NTH>(tbl, slot, w, dg);
      DNum x = dview<NTH>(E.buf[cur], sw);
      dmul<NTH>(half_lo<NTH>(E.buf[cur ^ 1]), half_hi<NTH>(E.buf[cur ^ 1]), x.d0, x.d1, te.d0, te.d1, &dc);
      cur ^= 1;
      sw = 1;
    }
  }
  digit_leave_store<NTH>(E, cur, sw, out_row, store);
}

}  // namespace pai
