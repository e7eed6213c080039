// pai_pack.cuh -- packed fixed-point plaintexts (DESIGN.md §3.10): K signed slots of b bits in one plaintext row,
// P = sum_j s_j * 2^(b j), stored as P mod n.  With |s_j| <= 2^(b-1) - 1 and K = (bits(n) - 1) / b,
// |P| < 2^(bK-1) <= 2^(bits(n)-2) < n/2, so the centre lift of P mod n gives P back and its balanced base-2^b digits are the
// slots.  Those digits are unique and never -2^(b-1), so unpack refuses that digit: it accepts exactly what pack makes.  One thread per row: the
// work per row is a few hundred word operations, nothing next to the encryption or decryption of that row.
#pragma once
#include "pai_core.cuh"

namespace pai {

typedef __int128 pack_i128;

// m[0..ln) <- P mod n for the slots s[0..cnt) (slots cnt..K-1 are 0).  Returns 1, with the row zeroed, when a slot lies
// outside (-2^(b-1), 2^(b-1)).
PAI_DEV int pack_row(const int64_t* s, int cnt, int b, const uint32_t* n, int ln, uint32_t* m) {
  const int64_t lim = (int64_t)1 << (b - 1);
  int bad = 0, neg = 0;
  for (int j = 0; j < cnt; j++) {
    const int64_t v = s[j];
    bad |= (v >= lim) | (v <= -lim);
    if (v) neg = v < 0;                                  // P has the sign of its highest nonzero slot
  }
  if (bad) {
    for (int i = 0; i < ln; i++) m[i] = 0;
    return 1;
  }
  // limb i of P (two's complement) is the low word of acc once every slot that starts below bit 32(i+1) is in; a negative
  // P gets n added on the way, which leaves n + P = P mod n
  pack_i128 acc = 0;
  uint64_t carry = 0;
  int j = 0;
  for (int i = 0; i < ln; i++) {
    for (; j < cnt && b * j < 32 * i + 32; j++) acc += (pack_i128)s[j] << (b * j - 32 * i);
    const uint64_t t = (uint64_t)(uint32_t)acc + (neg ? n[i] : 0u) + carry;
    m[i] = (uint32_t)t;
    carry = t >> 32;
    acc >>= 32;
  }
  return 0;
}

// s[0..cnt) <- the first cnt slots of row m[0..ln) (cnt <= K).  Returns 1, with the slots zeroed, when the row is not a
// packing: m >= n, a digit is -2^(b-1) (no slot pack accepts), or the centre-lifted value has a nonzero part above
// slot K-1.
PAI_DEV int unpack_row(const uint32_t* m, const uint32_t* n, int ln, int b, int K, int64_t* s, int cnt) {
  // from the top limb down: m against n, and 2m against n (m > (n-1)/2 <=> 2m > n, n odd)
  int ge = -1, neg = (int)(m[ln - 1] >> 31);
  int neg_known = neg;
  for (int i = ln - 1; i >= 0; i--) {
    if (ge < 0 && m[i] != n[i]) ge = m[i] > n[i];
    const uint32_t t = (m[i] << 1) | (i ? m[i - 1] >> 31 : 0u);
    if (!neg_known && t != n[i]) { neg = t > n[i]; neg_known = 1; }
  }
  int bad = ge != 0;                                     // ge = -1: m == n
  if (!bad) {
    // V = P in two's complement: m, or m - n when m > (n-1)/2; streamed limb by limb into acc, which holds the bits of
    // V above the digits taken so far (nb of them loaded), less those digits' borrows
    pack_i128 acc = 0;
    int nb = 0, i = 0;
    uint32_t borrow = 0;
    const int sh = 64 - b;
    const int64_t dmin = -((int64_t)1 << (b - 1));
    for (int j = 0; j < K; j++) {
      while (nb < b) {                                   // b K <= bits(n) - 1 <= 32 ln: the limbs never run out here
        uint32_t v = m[i];
        if (neg) { const uint64_t d = (uint64_t)m[i] - n[i] - borrow; v = (uint32_t)d; borrow = (uint32_t)(d >> 63); }
        acc += (pack_i128)v << nb;
        nb += 32;
        i++;
      }
      const int64_t d = (int64_t)((uint64_t)acc << sh) >> sh;   // the low b bits as a digit in [-2^(b-1), 2^(b-1))
      if (j < cnt) s[j] = d;
      bad |= d == dmin;
      acc = (acc - d) >> b;
      nb -= b;
    }
    // the rest, acc + 2^nb * (V >> 32 i), must be zero: its loaded bits first, then each remaining limb, then the sign
    bad |= (acc & (((pack_i128)1 << nb) - 1)) != 0;
    acc >>= nb;
    for (; i < ln; i++) {
      uint32_t v = m[i];
      if (neg) { const uint64_t d = (uint64_t)m[i] - n[i] - borrow; v = (uint32_t)d; borrow = (uint32_t)(d >> 63); }
      acc += v;
      bad |= (uint32_t)acc != 0;
      acc >>= 32;
    }
    bad |= acc != (pack_i128)neg;                        // V's infinite top is -neg: acc - neg must vanish
  }
  if (bad)
    for (int j = 0; j < cnt; j++) s[j] = 0;
  return bad;
}

}  // namespace pai
