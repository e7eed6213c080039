// pai_kernels.cuh -- per-thread "programs" of the Paillier hot path, built on pai_core.cuh.
//
// Each program is the work ONE thread does for ONE batch element.  The __global__ wrappers in
// pai_engine.cu run them in a persistent grid (thousands of elements per launch); tests/hostsim
// runs the same programs on the CPU (test-only).  Reference semantics, file:line in
// data61/python-paillier 1.5.0:
//   prog_encrypt   PaillierPublicKey.raw_encrypt          phe/paillier.py:102-139
//   prog_decrypt   PaillierPrivateKey.raw_decrypt + crt   phe/paillier.py:328-374
//   prog_mulmod    EncryptedNumber._raw_add / util.mulmod phe/paillier.py:705-719, phe/util.py:53-64
//   prog_powmod    EncryptedNumber._raw_mul / util.powmod phe/paillier.py:749-751, phe/util.py:38-50
//   prog_invert    util.invert                            phe/util.py:85-103
//   mod_setup      Montgomery constants of a modulus (no reference counterpart; replaces what GMP
//                  derives internally inside mpz_powm)
#pragma once
#include "pai_core.cuh"

namespace pai {

// ------------------------------------------------------------------------------------------------
// Per-modulus constant blob (uint32 limbs, L = 8*NT):  N | R1 | R2 | R3 | ONE | NINV(8)
//   R1 = R mod N (Montgomery form of 1), R2 = R^2 mod N, R3 = R^3 mod N, ONE = integer 1,
//   NINV = -N^-1 mod 2^256,  R = 2^(32 L).
PAI_HD int mc_limbs(int NT) { return 5 * 8 * NT + 8; }

struct ModC {
  Opnd N, R1, R2, R3, ONE, ninv;
};

PAI_DEV void modc_bind(ModC& m, u4* blob, int NT) {
  const int Q = 2 * NT;
  m.N.p = blob;           m.N.s = 1;
  m.R1.p = blob + Q;      m.R1.s = 1;
  m.R2.p = blob + 2 * Q;  m.R2.s = 1;
  m.R3.p = blob + 3 * Q;  m.R3.s = 1;
  m.ONE.p = blob + 4 * Q; m.ONE.s = 1;
  m.ninv.p = blob + 5 * Q; m.ninv.s = 1;
}

// ------------------------------------------------------------------------------------------------
// Global <-> interleaved helpers.  Rows in global memory are little-endian limb arrays, 16-byte aligned.
PAI_DEV void load_row(const Opnd& dst, const uint32_t* row, int nq_src, int nq_total) {
  const u4* r = (const u4*)row;
  for (int q = 0; q < nq_src; q++) dst.p[q * dst.s] = r[q];
  u4 z; z.x = z.y = z.z = z.w = 0;
  for (int q = nq_src; q < nq_total; q++) dst.p[q * dst.s] = z;
}
PAI_DEV void store_row(uint32_t* row, const Opnd& src, int nq) {
  u4* r = (u4*)row;
  for (int q = 0; q < nq; q++) r[q] = src.p[q * src.s];
}

// bits [pos, pos+w) of the little-endian limb array e[0..nl)
PAI_DEV uint32_t exp_digit(const uint32_t* e, int nl, int pos, int w) {
  int li = pos >> 5, sh = pos & 31;
  uint32_t v = e[li] >> sh;
  if (sh + w > 32 && li + 1 < nl) v |= e[li + 1] << (32 - sh);
  return v & ((1u << w) - 1u);
}
PAI_DEV int limbs_bitlen(const uint32_t* e, int nl) {
  for (int i = nl - 1; i >= 0; i--) {
    uint32_t v = e[i];
    if (v) { int b = 0; while (v) { b++; v >>= 1; } return 32 * i + b; }
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Fixed-window Montgomery exponentiation.  Three operand buffers; the 2^W-entry table of powers
// lives in global memory (HBM/L2) in the same interleaved layout, so a warp's table traffic is
// fully coalesced 512-byte segments.
template <int NT>
struct PowEnv {
  Opnd buf[3];
  Opnd tbl;   // entry e, quad q  at  tbl.p[(e * 2*NT + q) * tbl.s]
  ModC* mc;
};

template <int NT>
PAI_DEV void tbl_store(const PowEnv<NT>& E, int e, const Opnd& src) {
  for (int q = 0; q < 2 * NT; q++) E.tbl.p[(e * 2 * NT + q) * E.tbl.s] = src.p[q * src.s];
}
template <int NT>
PAI_DEV void tbl_load(const PowEnv<NT>& E, int e, const Opnd& dst) {
  for (int q = 0; q < 2 * NT; q++) dst.p[q * dst.s] = E.tbl.p[(e * 2 * NT + q) * E.tbl.s];
}

// base (Montgomery form, canonical) in buf[bi]; exponent limbs e[0..nl), nwin windows of W bits.
// Returns the index of the buffer that holds base^e in Montgomery form.
// SKIPZERO: skip the multiplication for zero digits (only for exponents shared by the whole batch
// and public, i.e. encrypt; per-element digits would diverge, secret ones would leak).
template <int NT, int W, bool SKIPZERO>
PAI_DEV int mont_pow(const PowEnv<NT>& E, int bi, const uint32_t* e, int nl, int nwin) {
  const ModC& mc = *E.mc;
  int y = bi == 2 ? 0 : bi + 1;
  int z = y == 2 ? 0 : y + 1;
  if (nwin <= 0) {
    big_copy<NT>(E.buf[y], mc.R1);
    return y;
  }
  // table of powers: T[0] = 1, T[1] = base, T[i] = T[i-1] * base
  tbl_store<NT>(E, 0, mc.R1);
  tbl_store<NT>(E, 1, E.buf[bi]);
  mont_sqr<NT>(E.buf[y], E.buf[bi], mc.N, mc.ninv);
  tbl_store<NT>(E, 2, E.buf[y]);
  {
    int p = y, o = z;
    for (int i = 3; i < (1 << W); i++) {
      mont_mul<NT>(E.buf[o], E.buf[p], E.buf[bi], mc.N, mc.ninv);
      tbl_store<NT>(E, i, E.buf[o]);
      int t = p; p = o; o = t;
    }
  }
  int cur = y, oth = z;
  tbl_load<NT>(E, (int)exp_digit(e, nl, (nwin - 1) * W, W), E.buf[cur]);
  for (int wi = nwin - 2; wi >= 0; wi--) {
    for (int s = 0; s < W; s++) {
      mont_sqr<NT>(E.buf[oth], E.buf[cur], mc.N, mc.ninv);
      int t = cur; cur = oth; oth = t;
    }
    int d = (int)exp_digit(e, nl, wi * W, W);
    if (SKIPZERO && d == 0) continue;
    tbl_load<NT>(E, d, E.buf[bi]);
    mont_mul<NT>(E.buf[oth], E.buf[cur], E.buf[bi], mc.N, mc.ninv);
    int t = cur; cur = oth; oth = t;
  }
  return cur;
}

// Two-buffer exponentiation: table entries are consumed straight from the global table as the `b` operand of
// mont_mul (never staged in shared memory), so a thread needs 2 x 32*NT bytes of shared memory instead
// of 3 x -- at 4096-bit moduli that is 224 instead of 128 resident threads per SM.
template <int NT>
PAI_DEV Opnd tbl_entry(const PowEnv<NT>& E, int e) {
  Opnd o;
  o.p = E.tbl.p + (size_t)e * 2 * NT * E.tbl.s;
  o.s = E.tbl.s;
  return o;
}

// Sliding-window exponentiation driven by a host-built "exponent program" (public exponent shared by
// the whole batch: encrypt's n).  prog[i] = (nsq << 16) | idx : square nsq times, then multiply by the
// odd power T[idx] = base^(2 idx + 1)  (idx = 0xffff: no multiplication).  prog[0] only selects the
// initial value T[idx].  Table slots: T[0 .. 2^(w-1)) odd powers, slot 2^(w-1) = base^2 (build helper).
// Two shared-memory buffers, table entries consumed straight from global memory.
template <int NT>
PAI_DEV int mont_pow_prog(const PowEnv<NT>& E, int bi, const uint32_t* prog, int nops, int nodd) {
  const ModC& mc = *E.mc;
  int cur = bi, oth = bi ^ 1;
  if (nops <= 0) {                                   // exponent 0
    big_copy<NT>(E.buf[oth], mc.R1);
    return oth;
  }
  tbl_store<NT>(E, 0, E.buf[cur]);                                        // T[0] = base
  if (nodd > 1) {
    mont_sqr<NT>(E.buf[oth], E.buf[cur], mc.N, mc.ninv);                  // base^2
    tbl_store<NT>(E, nodd, E.buf[oth]);
    const Opnd b2 = tbl_entry<NT>(E, nodd);
    for (int k = 1; k < nodd; k++) {                                      // T[k] = T[k-1] * base^2
      mont_mul<NT>(E.buf[oth], E.buf[cur], b2, mc.N, mc.ninv);
      { int t = cur; cur = oth; oth = t; }
      tbl_store<NT>(E, k, E.buf[cur]);
    }
  }
  tbl_load<NT>(E, (int)(prog[0] & 0xffffu), E.buf[cur]);
  for (int i = 1; i < nops; i++) {
    const uint32_t op = prog[i];
    const int nsq = (int)(op >> 16), idx = (int)(op & 0xffffu);
    for (int s = 0; s < nsq; s++) {
      mont_sqr<NT>(E.buf[oth], E.buf[cur], mc.N, mc.ninv);
      int t = cur; cur = oth; oth = t;
    }
    if (idx != 0xffff) {
      mont_mul<NT>(E.buf[oth], E.buf[cur], tbl_entry<NT>(E, idx), mc.N, mc.ninv);
      int t = cur; cur = oth; oth = t;
    }
  }
  return cur;
}

// raw_encrypt:  c = (1 + n*m) * r^n mod n^2          (phe/paillier.py:102-139)
// Both reference branches for the nude ciphertext (:125-134) equal n*(m mod n)+1 mod n^2
// (because (1+n*a)^-1 = 1-n*a mod n^2), and the final Montgomery multiplication reduces any
// m, r < 2^(32*Ln) for free, so no inversion and no range split is needed here.
//   NT  = tiles of n^2 (even); n, m, r have NT/2 tiles.  mc = constants of n^2.
//   nbc = n as a broadcast operand (NT/2 tiles); e = limbs of n (the exponent), nwin windows.
// (full-width Montgomery variant with two shared-memory buffers; the default path is prog_encrypt_digit)
template <int NT>
PAI_DEV void prog_encrypt2(const PowEnv<NT>& E, const Opnd& nbc, const uint32_t* prog, int nops, int nodd,
                           const uint32_t* m_row, const uint32_t* r_row, uint32_t* out_row, bool store) {
  const ModC& mc = *E.mc;
  load_row(E.buf[0], r_row, NT, 2 * NT);
  mont_mul<NT>(E.buf[1], E.buf[0], mc.R2, mc.N, mc.ninv);                 // r*R mod n^2
  int cur = mont_pow_prog<NT>(E, 1, prog, nops, nodd);                    // (r^n)*R mod n^2
  tbl_store<NT>(E, 0, E.buf[cur]);                                        // park it in table slot 0
  int a = cur, b = cur ^ 1;
  load_row(E.buf[a], m_row, NT, NT);
  big_mul<NT / 2, NT / 2, NT>(E.buf[b], E.buf[a], nbc, 1u);               // n*m + 1
  mont_mul<NT>(E.buf[a], E.buf[b], tbl_entry<NT>(E, 0), mc.N, mc.ninv);   // (n*m+1) * r^n mod n^2
  if (store) store_row(out_row, E.buf[a], 2 * NT);
}

// ------------------------------------------------------------------------------------------------
// a*b mod N for any a, b < 2^(32 L)                   (phe/util.py:53-64, phe/paillier.py:719)
template <int NT>
PAI_DEV void prog_mulmod(const Opnd buf[3], const ModC& mc, const uint32_t* a_row, const uint32_t* b_row,
                         uint32_t* out_row, bool store) {
  load_row(buf[0], a_row, 2 * NT, 2 * NT);
  load_row(buf[1], b_row, 2 * NT, 2 * NT);
  mont_mul<NT>(buf[2], buf[0], mc.R2, mc.N, mc.ninv);                     // a*R mod N (canonical)
  mont_mul<NT>(buf[0], buf[2], buf[1], mc.N, mc.ninv);                    // a*b mod N
  if (store) store_row(out_row, buf[0], 2 * NT);
}

// ------------------------------------------------------------------------------------------------
// base^e mod N with a per-element or shared exponent  (phe/util.py:38-50, phe/paillier.py:749-751)
//   base: nqb quads (<= 4*NT: a double-width base is reduced through R2/R3 like GMP reduces it)
//   e: exponent limbs (nl), nwin windows (uniform loop bound; leading zero digits multiply by 1)
template <int NT, int W>
PAI_DEV void prog_powmod(const PowEnv<NT>& E, const uint32_t* base_row, int base_tiles, const uint32_t* e, int nl,
                         int nwin, uint32_t* out_row, bool store) {
  const ModC& mc = *E.mc;
  if (base_tiles <= NT) {
    load_row(E.buf[0], base_row, 2 * base_tiles, 2 * NT);
    mont_mul<NT>(E.buf[1], E.buf[0], mc.R2, mc.N, mc.ninv);
  } else {                                                                 // base = lo + hi * R
    load_row(E.buf[0], base_row, 2 * NT, 2 * NT);
    mont_mul<NT>(E.buf[2], E.buf[0], mc.R2, mc.N, mc.ninv);                // lo * R
    load_row(E.buf[0], base_row + 8 * NT, 2 * (base_tiles - NT), 2 * NT);
    mont_mul<NT>(E.buf[1], E.buf[0], mc.R3, mc.N, mc.ninv);                // hi * R^2
    uint32_t c = big_add_masked<NT>(E.buf[1], E.buf[1], E.buf[2], 0xffffffffu);
    big_cond_sub<NT>(E.buf[1], mc.N, c);
  }
  int cur = mont_pow<NT, W, false>(E, 1, e, nl, nwin);
  int a = cur == 2 ? 0 : cur + 1;
  mont_mul<NT>(E.buf[a], E.buf[cur], mc.ONE, mc.N, mc.ninv);              // leave the Montgomery domain
  if (store) store_row(out_row, E.buf[a], 2 * NT);
}

// ------------------------------------------------------------------------------------------------
// Modular inverse for an odd modulus, binary extended gcd   (phe/util.py:85-103)
//   buf[0..3]: u, v, x1, x2.  Returns 0 and stores a^-1 mod N, or 1 if gcd(a, N) != 1
//   (the reference raises ZeroDivisionError there).

// x = (x + (N & mask)) >> 1  (the carry of the addition becomes the top bit)
template <int NT>
PAI_DEV void big_halve_mod(const Opnd& x, const Opnd& N, uint32_t mask) {
  uint32_t prev[8], s[8], y[8];
  uint32_t c = 0;
  for (int t = 0; t < NT; t++) {
    ld_tile(x, t, s); ld_tile(N, t, y);
    PAI_UNROLL
    for (int i = 0; i < 8; i++) y[i] &= mask;
    c = add8c(s, s, y, c);
    if (t > 0) {
      uint32_t o[8];
      PAI_UNROLL
      for (int i = 0; i < 7; i++) o[i] = (prev[i] >> 1) | (prev[i + 1] << 31);
      o[7] = (prev[7] >> 1) | (s[0] << 31);
      st_tile(x, t - 1, o);
    }
    PAI_UNROLL
    for (int i = 0; i < 8; i++) prev[i] = s[i];
  }
  uint32_t o[8];
  PAI_UNROLL
  for (int i = 0; i < 7; i++) o[i] = (prev[i] >> 1) | (prev[i + 1] << 31);
  o[7] = (prev[7] >> 1) | (c << 31);
  st_tile(x, NT - 1, o);
}

PAI_DEV uint32_t low_limb(const Opnd& x) { return x.p[0].x; }

template <int NT>
PAI_DEV uint32_t big_is_one(const Opnd& a) {
  uint32_t acc = 0;
  for (int q = 0; q < 2 * NT; q++) { u4 v = a.p[q * a.s]; acc |= (q == 0 ? (v.x ^ 1u) : v.x) | v.y | v.z | v.w; }
  return acc == 0 ? 1u : 0u;
}

template <int NT>
PAI_DEV int prog_invert(const Opnd buf[4], const ModC& mc, const uint32_t* a_row, int a_tiles, uint32_t* out_row, bool store) {
  const Opnd &u = buf[0], &v = buf[1], &x1 = buf[2], &x2 = buf[3];
  // u = a mod N (canonical) through the Montgomery domain and back
  load_row(x1, a_row, 2 * a_tiles, 2 * NT);
  mont_mul<NT>(x2, x1, mc.R2, mc.N, mc.ninv);
  mont_mul<NT>(u, x2, mc.ONE, mc.N, mc.ninv);
  big_copy<NT>(v, mc.N);
  big_copy<NT>(x1, mc.ONE);
  for (int q = 0; q < 2 * NT; q++) { u4 zq; zq.x = zq.y = zq.z = zq.w = 0; x2.p[q * x2.s] = zq; }
  int fail = 0;
  if (big_is_one<NT>(mc.N)) {
    // everything is 0 mod 1 (never on the Paillier path)
  } else {
    const int maxit = 2 * 256 * NT + 8;      // each step removes a bit of u or v
    int it = 0;
    while (!big_is_zero<NT>(u) && it < 2 * maxit) {
      it++;
      if ((low_limb(u) & 1u) == 0) {
        big_halve_mod<NT>(u, mc.N, 0u);
        big_halve_mod<NT>(x1, mc.N, 0u - (low_limb(x1) & 1u));
      } else if ((low_limb(v) & 1u) == 0) {
        big_halve_mod<NT>(v, mc.N, 0u);
        big_halve_mod<NT>(x2, mc.N, 0u - (low_limb(x2) & 1u));
      } else if (big_sub_borrow<NT>(u, v) == 0) {                          // u >= v
        big_sub_masked<NT>(u, u, v, 0xffffffffu);
        uint32_t bo = big_sub_masked<NT>(x1, x1, x2, 0xffffffffu);
        big_add_masked<NT>(x1, x1, mc.N, 0u - bo);
      } else {
        big_sub_masked<NT>(v, v, u, 0xffffffffu);
        uint32_t bo = big_sub_masked<NT>(x2, x2, x1, 0xffffffffu);
        big_add_masked<NT>(x2, x2, mc.N, 0u - bo);
      }
    }
    if (!big_is_one<NT>(v)) fail = 1;
  }
  if (store) {
    if (fail) for (int q = 0; q < 2 * NT; q++) { u4 zq; zq.x = zq.y = zq.z = zq.w = 0; x2.p[q * x2.s] = zq; }
    store_row(out_row, x2, 2 * NT);
  }
  return fail;
}

// ------------------------------------------------------------------------------------------------
// raw_decrypt with CRT                                  (phe/paillier.py:328-374)
// Constants of one prime side (all broadcast, pointing into the kernel's constant area):
template <int NTP>
struct SideC {
  ModC sq;            // modulus x^2  (2*NTP tiles)
  ModC pr;            // modulus x    (NTP tiles)
  Opnd xinv;          // x^-1 mod 2^(256 NTP)             -> exact division in L(u) = (u-1)/x  (:362-364)
  Opnd hM;            // h(x) * R_x mod x  (h_function, :356-360), Montgomery form mod x
  const uint32_t* e;  // x - 1  (8*NTP limbs)
  int nwin;           // windows of the exponent
};

// one CRT half: out_small (NTP tiles, in buf[ret]) = L(c^(x-1) mod x^2) * h mod x
template <int NTP, int W>
PAI_DEV int decrypt_half(PowEnv<2 * NTP>& E, const SideC<NTP>& S, const uint32_t* c_row, const uint32_t* pre_row = nullptr) {
  const int NT2 = 2 * NTP;
  const ModC& mq = S.sq;
  int a, b;
  if (pre_row) {                                                           // u = c^(x-1) mod x^2 computed elsewhere
    a = 1; b = 2;
    load_row(E.buf[a], pre_row, 2 * NT2, 2 * NT2);
  } else {
    // c mod x^2 in Montgomery form: c = lo + hi*R  ->  lo*R + hi*R^2   (GMP reduces the base the same way)
    load_row(E.buf[0], c_row, 2 * NT2, 2 * NT2);
    mont_mul<NT2>(E.buf[2], E.buf[0], mq.R2, mq.N, mq.ninv);
    load_row(E.buf[0], c_row + 8 * NT2, 2 * NT2, 2 * NT2);
    mont_mul<NT2>(E.buf[1], E.buf[0], mq.R3, mq.N, mq.ninv);
    uint32_t cy = big_add_masked<NT2>(E.buf[1], E.buf[1], E.buf[2], 0xffffffffu);
    big_cond_sub<NT2>(E.buf[1], mq.N, cy);
    E.mc = const_cast<ModC*>(&S.sq);
    int cur = mont_pow<NT2, W, false>(E, 1, S.e, 8 * NTP, S.nwin);        // c^(x-1) * R mod x^2
    a = cur == 2 ? 0 : cur + 1;
    b = a == 2 ? 0 : a + 1;
    mont_mul<NT2>(E.buf[a], E.buf[cur], mq.ONE, mq.N, mq.ninv);           // u = c^(x-1) mod x^2
  }
  // L(u) = (u - 1) // x.  u = 1 mod x whenever gcd(c, x) = 1, so the division is exact and equals
  // (u-1) * x^-1 mod 2^(256 NTP).  Otherwise x | c and u == 0: Python's floor division gives
  // (0-1)//x = -1, which the following mulmod(., h, x) sees as x - 1.
  uint32_t uz = big_is_zero<NT2>(E.buf[a]);
  big_sub_masked<NT2>(E.buf[a], E.buf[a], mq.ONE, 0u - (uz ^ 1u));        // u - 1 (kept 0 when u == 0)
  big_mul<NTP, NTP, NTP>(E.buf[b], E.buf[a], S.xinv, 0u);                 // low half of (u-1) * x^-1
  {                                                                       // u == 0  ->  x - 1
    Opnd xm1 = S.pr.N;
    for (int t = 0; t < NTP; t++) {
      uint32_t l[8], n[8];
      ld_tile(E.buf[b], t, l); ld_tile(xm1, t, n);
      if (t == 0) n[0] -= 1u;                                             // x is odd: no borrow
      PAI_UNROLL
      for (int i = 0; i < 8; i++) l[i] = uz ? n[i] : l[i];
      st_tile(E.buf[b], t, l);
    }
  }
  mont_mul<NTP>(E.buf[a], E.buf[b], S.hM, S.pr.N, S.pr.ninv);             // L * h mod x
  return a;
}

// full decrypt of one ciphertext.  pinvqM = (p^-1 mod q) * R_q mod q  (:233, used by crt :373).
// out_row (2*NTP tiles = limbs of n) doubles as the spill slot for m_p between the halves.
template <int NTP, int W>
PAI_DEV void prog_decrypt(PowEnv<2 * NTP>& E, const SideC<NTP>& P, const SideC<NTP>& Qs, const Opnd& pinvqM,
                          const uint32_t* c_row, uint32_t* out_row, bool store, const uint32_t* pre_p = nullptr,
                          const uint32_t* pre_q = nullptr) {
  const int NT2 = 2 * NTP;
  int ip = decrypt_half<NTP, W>(E, P, c_row, pre_p);
  if (store) store_row(out_row, E.buf[ip], 2 * NTP);                      // m_p -> global (low half)
  int iq = decrypt_half<NTP, W>(E, Qs, c_row, pre_q);
  int a = iq == 2 ? 0 : iq + 1;
  int b = a == 2 ? 0 : a + 1;
  if (store) load_row(E.buf[a], out_row, 2 * NTP, 2 * NTP);
  else big_copy<NTP>(E.buf[a], E.buf[iq]);                                 // inactive lane: any valid value
  // u = (m_q - m_p) * p^-1 mod q   (m_p < p < q, m_q < q)
  uint32_t bo = big_sub_masked<NTP>(E.buf[iq], E.buf[iq], E.buf[a], 0xffffffffu);
  big_add_masked<NTP>(E.buf[iq], E.buf[iq], Qs.pr.N, 0u - bo);
  mont_mul<NTP>(E.buf[b], E.buf[iq], pinvqM, Qs.pr.N, Qs.pr.ninv);
  // m = m_p + u * p
  big_mul<NTP, NTP, NT2>(E.buf[iq], E.buf[b], P.pr.N, 0u);
  for (int t = NTP; t < NT2; t++) zero_tile(E.buf[a], t);
  big_add_masked<NT2>(E.buf[iq], E.buf[iq], E.buf[a], 0xffffffffu);
  if (store) store_row(out_row, E.buf[iq], 2 * NT2);
}

// ------------------------------------------------------------------------------------------------
// Montgomery constants of one modulus (single thread; operands are plain arrays, stride 1).
//   blob: mc_limbs(NT) limbs with N already filled in; scratch: 3 * 8*NT limbs.
// x * N = 1 mod 2^(32 nl): limb-serial Hensel lifting.  N odd.
PAI_DEV void inv_mod_2k(uint32_t* x, const uint32_t* N, int nl) {
  // 32-bit inverse of N[0] by Newton
  uint32_t n0 = N[0], i0 = n0;
  for (int i = 0; i < 5; i++) i0 *= 2u - n0 * i0;
  // t = x*N - 1 must vanish limb by limb; keep t (nl limbs, mod 2^(32 nl)) in x's upper workspace-free way
  // simple O(nl^2): x_i = -t_i * i0, t += x_i * N << (32 i)
  for (int i = 0; i < nl; i++) x[i] = 0;
  // t stored temporarily in-place is not possible; recompute column-wise with a running carry
  // Use the identity: t_i (the i-th limb of x*N - 1 given x_0..x_{i-1}) computed on the fly.
  // Maintain the full running product in a small rolling window via 64-bit accumulators.
  uint64_t carry_lo = 0, carry_hi = 0;   // 128-bit running carry into column i
  for (int i = 0; i < nl; i++) {
    // column sum of known terms: sum_{j<i} x_j * N_{i-j} + carry
    uint64_t lo = carry_lo, hi = carry_hi;
    for (int j = 0; j < i; j++) {
      uint64_t p = (uint64_t)x[j] * N[i - j];
      lo += p; if (lo < p) hi++;
    }
    // want (lo + x_i * n0) = (i == 0 ? 1 : 0) mod 2^32
    uint32_t target = (i == 0) ? 1u : 0u;
    uint32_t xi = (target - (uint32_t)lo) * i0;
    x[i] = xi;
    uint64_t p = (uint64_t)xi * n0;
    lo += p; if (lo < p) hi++;
    // shift the 128-bit column sum right by one limb
    carry_lo = (lo >> 32) | (hi << 32);
    carry_hi = hi >> 32;
  }
}

template <int NT>
PAI_DEV void mod_setup(uint32_t* blob, uint32_t* scratch) {
  const int L = 8 * NT;
  uint32_t* N = blob;
  uint32_t* R1 = blob + L;
  uint32_t* R2 = blob + 2 * L;
  uint32_t* R3 = blob + 3 * L;
  uint32_t* ONE = blob + 4 * L;
  uint32_t* NINV = blob + 5 * L;
  uint32_t* t0 = scratch;
  uint32_t* t1 = scratch + L;
  for (int i = 0; i < L; i++) ONE[i] = (i == 0);
  // NINV = -N^-1 mod 2^256
  {
    uint32_t inv[8];
    inv_mod_2k(inv, N, 8);
    uint32_t c = 1;
    for (int i = 0; i < 8; i++) { uint64_t v = (uint64_t)(~inv[i]) + c; NINV[i] = (uint32_t)v; c = (uint32_t)(v >> 32); }
  }
  // R1 = 2^(32 L) mod N by doubling x = 1 (x < N throughout)
  for (int i = 0; i < L; i++) t0[i] = (i == 0);
  {
    // N == 1 -> everything is 0
    bool n_is_one = (N[0] == 1);
    for (int i = 1; i < L && n_is_one; i++) if (N[i]) n_is_one = false;
    if (n_is_one) t0[0] = 0;
  }
  for (int it = 0; it < 32 * L + NT; it++) {
    if (it == 32 * L) for (int i = 0; i < L; i++) R1[i] = t0[i];
    uint32_t c = 0;
    for (int i = 0; i < L; i++) { uint32_t v = t0[i]; t0[i] = (v << 1) | c; c = v >> 31; }
    // subtract N if carry or t0 >= N
    uint32_t bo = 0;
    for (int i = 0; i < L; i++) { uint64_t d = (uint64_t)t0[i] - N[i] - bo; t1[i] = (uint32_t)d; bo = (uint32_t)(d >> 63); }
    if (c || !bo) for (int i = 0; i < L; i++) t0[i] = t1[i];
  }
  // t0 = 2^NT * R mod N (Montgomery form of 2^NT).  Eight Montgomery squarings give 2^(256 NT) * R = R^2.
  Opnd ninv{(u4*)NINV, 1};
  Opnd oN{(u4*)N, 1}, a{(u4*)t0, 1}, b{(u4*)t1, 1};
  for (int s = 0; s < 8; s++) {
    mont_sqr<NT>(b, a, oN, ninv);
    Opnd t = a; a = b; b = t;
  }
  for (int i = 0; i < L; i++) R2[i] = ((uint32_t*)a.p)[i];
  Opnd oR2{(u4*)R2, 1}, oR3{(u4*)R3, 1};
  mont_mul<NT>(oR3, oR2, oR2, oN, ninv);                                   // R^2 * R^2 / R = R^3
}

// ------------------------------------------------------------------------------------------------
// Miller-Rabin on a BATCH of candidates, one thread per candidate (util.miller_rabin, phe/util.py:381-417; the
// reference's key generation tests one candidate at a time, phe/util.py:106-124).  Every candidate is its own modulus,
// so each thread derives its own Montgomery constants (mod_setup) in a private strip of global memory and runs the
// generic window ladder on stride-1 operands.  `bases`: `rounds` random rows per candidate (any value < 2^(32 L); reduced
// here; a base congruent to 0 or +-1 passes its round, as it tells nothing).  result: 1 = probably prime, 0 = composite.
//   ws (limbs per thread): mc_limbs(NT) | 3L setup scratch | 3 buffers of L | 2^W table entries of L | d (L)
template <int NT, int W>
PAI_HD long mr_ws_limbs() { return mc_limbs(NT) + (long)(3 + 3 + (1 << W) + 1) * 8 * NT; }

template <int NT, int W>
PAI_DEV void prog_miller_rabin(uint32_t* ws, const uint32_t* cand, const uint32_t* bases, int rounds, int32_t* result) {
  const int L = 8 * NT;
  uint32_t* blob = ws;
  uint32_t* scratch = blob + mc_limbs(NT);
  uint32_t* b0 = scratch + 3 * L;
  uint32_t* tblp = b0 + 3 * L;
  uint32_t* d = tblp + (long)(1 << W) * L;
  for (int i = 0; i < L; i++) blob[i] = cand[i];
  // tiny / even candidates are the host's business (trial division comes first); keep the kernel total anyway
  if (!(cand[0] & 1u)) { *result = 0; return; }
  mod_setup<NT>(blob, scratch);
  ModC mc;
  modc_bind(mc, (u4*)blob, NT);
  // n - 1 = 2^s * d
  int s = 0;
  {
    for (int i = 0; i < L; i++) d[i] = cand[i];
    d[0] &= ~1u;                                             // n - 1 (n odd)
    int nz = 0;
    for (int i = 0; i < L; i++) if (d[i]) nz = 1;
    if (!nz) { *result = 0; return; }                         // n == 1
    while (!(d[0] & 1u)) {
      for (int i = 0; i < L - 1; i++) d[i] = (d[i] >> 1) | (d[i + 1] << 31);
      d[L - 1] >>= 1;
      s++;
    }
  }
  const int nwin = (limbs_bitlen(d, L) + W - 1) / W;
  PowEnv<NT> E;
  for (int i = 0; i < 3; i++) { E.buf[i].p = (u4*)(b0 + i * L); E.buf[i].s = 1; }
  E.tbl.p = (u4*)tblp; E.tbl.s = 1;
  E.mc = &mc;
  // minus one in Montgomery form: N - R1
  int prime = 1;
  for (int r = 0; r < rounds && prime; r++) {
    load_row(E.buf[0], bases + (long)r * L, 2 * NT, 2 * NT);
    mont_mul<NT>(E.buf[1], E.buf[0], mc.R2, mc.N, mc.ninv);                 // a * R mod N (any a < 2^(32 L))
    // a = 0, 1, -1 (mod N): uninformative
    uint32_t is0 = big_is_zero<NT>(E.buf[1]);
    uint32_t is1 = 1, ism1 = 1;
    {
      uint32_t bo = 0;
      for (int t = 0; t < NT; t++) {
        uint32_t x[8], y[8], o[8], n[8], m1[8];
        ld_tile(E.buf[1], t, x); ld_tile(mc.R1, t, y); ld_tile(mc.N, t, n);
        bo = sub8b(m1, n, y, bo);                                            // N - R1, tile by tile
        for (int i = 0; i < 8; i++) { if (x[i] != y[i]) is1 = 0; if (x[i] != m1[i]) ism1 = 0; o[i] = 0; }
        (void)o;
      }
    }
    if (is0 | is1 | ism1) continue;
    int cur = mont_pow<NT, W, false>(E, 1, d, L, nwin);                      // a^d in Montgomery form
    int pass = 0;
    for (int it = 0; it < s && !pass; it++) {
      uint32_t eq1 = 1, eqm1 = 1, bo = 0;
      for (int t = 0; t < NT; t++) {
        uint32_t x[8], y[8], n[8], m1[8];
        ld_tile(E.buf[cur], t, x); ld_tile(mc.R1, t, y); ld_tile(mc.N, t, n);
        bo = sub8b(m1, n, y, bo);
        for (int i = 0; i < 8; i++) { if (x[i] != y[i]) eq1 = 0; if (x[i] != m1[i]) eqm1 = 0; }
      }
      if (eqm1 || (it == 0 && eq1)) { pass = 1; break; }
      if (eq1) break;                                                        // a nontrivial square root of 1: composite
      if (it + 1 < s) {
        int nxt = cur == 2 ? 0 : cur + 1;
        mont_sqr<NT>(E.buf[nxt], E.buf[cur], mc.N, mc.ninv);
        cur = nxt;
      }
    }
    if (!pass) prime = 0;
  }
  *result = prime;
}

}  // namespace pai
