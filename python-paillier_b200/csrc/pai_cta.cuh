// pai_cta.cuh -- CTA-level bodies of the kernels: shared-memory map, persistent chunk loop.
//
// Shared memory map of every kernel:   [ constants (broadcast operands) | buf0 | buf1 | buf2 (| buf3) ]
// with each buffer holding 2*NT quads for each of the CTA's threads in the interleaved layout.
// A body has two phases separated by a CTA barrier: phase 0 copies the per-key constants into
// shared memory cooperatively, phase 1 is the per-thread persistent loop (no barriers: threads are
// independent).  The __global__ kernels in pai_engine.cu call phase 0, __syncthreads(), phase 1;
// tests/hostsim calls phase 0 for every simulated thread, then phase 1 for every simulated thread.
#pragma once
#include "pai_kernels.cuh"
#include "pai_digit.cuh"
#include "pai_rng.cuh"
#include "pai_radix.cuh"
#include "pai_coop.cuh"
#include "pai_tc.cuh"

namespace pai {

struct CtaId {
  int tid, nthr, cta, ncta;
};

// Row scheduler of the persistent kernels.  Work is handed out in groups of 32 consecutive rows (one
// group per warp per iteration) from a global counter, so a warp that has a scheduler to itself (e.g.
// the 7th warp of a 224-thread CTA) simply takes more groups than warps that share one, and the last
// wave of a launch balances itself.  The CPU simulation (no warps, no atomics) uses the equivalent
// static round-robin.
struct RowSched {
  unsigned long long* counter;   // zeroed by the host before the launch
  long ngroups;                  // ceil(batch / gw)
  int gw;                        // rows per group: 32 (the simulation build runs CTAs narrower than a warp)
  long sim_next, sim_stride;     // simulation only
};
PAI_DEV RowSched sched_init(const CtaId& id, unsigned long long* counter, long batch) {
  RowSched s;
  s.counter = counter;
  s.gw = id.nthr < 32 ? id.nthr : 32;
  s.ngroups = (batch + s.gw - 1) / s.gw;
  const long warps_per_cta = (id.nthr + s.gw - 1) / s.gw;
  s.sim_next = (long)id.cta * warps_per_cta + id.tid / s.gw;
  s.sim_stride = (long)id.ncta * warps_per_cta;
  return s;
}
// next row for this thread, or -1 when the batch is exhausted
PAI_DEV long sched_next_row(RowSched& s, const CtaId& id) {
  long grp;
#if !defined(PAI_HOSTSIM)
  unsigned long long w = 0;
  if ((id.tid & 31) == 0) w = atomicAdd(s.counter, 1ull);
  w = __shfl_sync(0xffffffffu, w, 0);
  grp = (long)w;
#else
  grp = s.sim_next;
  s.sim_next += s.sim_stride;
#endif
  if (grp >= s.ngroups) return -1;
  return grp * s.gw + (id.tid % s.gw);
}

// phase 0: constants -> shared
PAI_DEV void cta_load_consts(u4* smem, const CtaId& id, const uint32_t* src, int nquads) {
  const u4* s = (const u4*)src;
  for (int i = id.tid; i < nquads; i += id.nthr) smem[i] = s[i];
}

template <int NT>
PAI_DEV void cta_bufs(Opnd* buf, int nbuf, u4* smem, int const_quads, const CtaId& id) {
  for (int b = 0; b < nbuf; b++) {
    buf[b].p = smem + const_quads + b * (2 * NT) * id.nthr + id.tid;
    buf[b].s = id.nthr;
  }
}

template <int NT, int W>
PAI_DEV Opnd cta_table(u4* tbl, const CtaId& id) {
  Opnd t;
  t.p = tbl + (size_t)id.cta * ((size_t)(1 << W) * 2 * NT * id.nthr) + id.tid;
  t.s = id.nthr;
  return t;
}

// ---- encrypt.  consts = [ blob(n^2) | n (4*NT limbs) ]
template <int NT>
PAI_DEV int enc_const_quads() { return mc_limbs(NT) / 4 + NT; }

// table slots per thread of the encrypt kernel: 2^(w-1) odd powers + base^2
template <int NT>
PAI_DEV Opnd cta_table_slots(u4* tbl, const CtaId& id, int slots) {
  Opnd t;
  t.p = tbl + (size_t)id.cta * ((size_t)slots * 2 * NT * id.nthr) + id.tid;
  t.s = id.nthr;
  return t;
}

template <int NT>
PAI_DEV void cta_encrypt(u4* smem, const CtaId& id, const uint32_t* prog, int nops, int nodd, const uint32_t* m, const uint32_t* r,
                         uint32_t* out, long batch, u4* tbl, unsigned long long* counter) {
  ModC mc;
  modc_bind(mc, smem, NT);
  PowEnv<NT> E;
  cta_bufs<NT>(E.buf, 2, smem, enc_const_quads<NT>(), id);       // two operand buffers (mont_pow_prog)
  E.tbl = cta_table_slots<NT>(tbl, id, nodd + 1);
  E.mc = &mc;
  Opnd nbc{smem + mc_limbs(NT) / 4, 1};
  const int ln = 4 * NT, lc = 8 * NT;
  RowSched sched = sched_init(id, counter, batch);
  for (long g = sched_next_row(sched, id); g >= 0; g = sched_next_row(sched, id)) {
    bool store = g < batch;
    if (!store) g = batch - 1;
    prog_encrypt2<NT>(E, nbc, prog, nops, nodd, m + g * ln, r + g * ln, out + g * lc, store);
  }
}

// ---- encrypt in digit form (pai_digit.cuh).  consts = compact encrypt constants (dc_enc_limbs(NTH)); two buffers of
// 2*NTH tiles per thread; r and m are read straight from their global rows.
template <int NTH>
PAI_DEV void cta_encrypt_digit(u4* smem, const CtaId& id, const uint32_t* prog, int nops, int nodd, const uint32_t* m,
                               const uint32_t* r, uint32_t* out, long batch, u4* tbl, unsigned long long* counter,
                               const uint32_t* gzero) {
  DigitEnv dc;
  digit_bind_enc<NTH>(dc, smem, gzero);
  DPowEnv<NTH> E;
  cta_bufs<2 * NTH>(E.buf, 2, smem, dc_enc_limbs(NTH) / 4, id);
  E.tbl = cta_table_slots<2 * NTH>(tbl, id, nodd + 1);
  E.dc = &dc;
  E.step_sync = 1;
  const int ln = 8 * NTH, lc = 16 * NTH;
  (void)counter;
  // static chunks: every thread of the CTA runs the same number of identical ladders, so the per-step barrier is safe
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g = chunk * id.nthr + id.tid;
    bool store = g < batch;
    if (!store) g = batch - 1;
    prog_encrypt_digit<NTH>(E, prog, nops, nodd, m + g * ln, r + g * ln, out + g * lc, store);
  }
}

// ---- kernels with the reductions on the tensor cores (pai_tc.cuh).  Shared memory map of all of them:
//   [ constants | pad | bands (2 per digit modulus) | X | H1 (unless tc_x1_global) | A (one per 128-thread group) ]
// X/H1: the half-buffers of the digits x0 / x1 of every thread (interleaved, stride nthr); A: the groups' MMA operand buffers.
template <int NTH>
PAI_HD size_t tc_smem_bytes(int const_limbs, int nbands, int nthr) {
  const int groups = nthr >= TC_M ? nthr / TC_M : 1;
  return (size_t)const_limbs * 4 + 256 + (size_t)nbands * tc_band_bytes(NTH) + (tc_x1_global<NTH>() ? 1 : 2) * (size_t)(2 * NTH) * nthr * 16 +
         (size_t)groups * TC_M * 32 * NTH;
}
template <int NTH>
PAI_HD size_t tc_enc_smem_bytes(int nthr) { return tc_smem_bytes<NTH>(dc_enc_limbs(NTH), 2, nthr); }
template <int NTH>
PAI_HD size_t tc_pow_smem_bytes(int nthr) { return tc_smem_bytes<NTH>(dc_pow_limbs(NTH), 2, nthr); }
template <int NTP>
PAI_HD size_t tc_dec_smem_bytes(int nthr) { return tc_smem_bytes<NTP>((2 * (dside_limbs<NTP>() / 4) + 2 * NTP) * 4, 4, nthr); }
// Set-up shared by the tensor-core kernels: copies the bands to shared memory and fills in the context of the calling
// thread.  Returns the shared-memory address of the bands.  `entries`: user table entries per thread; three more follow:
// the park slot and (tc_x1_global) the home of the high digit x1 and the W slot.
template <int NTH>
PAI_DEV uint8_t* tc_cta_begin(TcCtx<NTH>& c, u4* smem, const CtaId& id, int const_limbs, int nbands, const uint8_t* gbands, u4* tbl,
                              int entries, int stagger_cycles) {
  constexpr bool x1_global = tc_x1_global<NTH>();
  const int D = 32 * NTH;
  uint8_t* base = (uint8_t*)smem;
  size_t off = (size_t)const_limbs * 4;
#if !defined(PAI_HOSTSIM)
  off += (128u - ((tc_smem_u32(base) + (uint32_t)off) & 127u)) & 127u;     // operands of the MMA: 128-byte aligned
#else
  off = (off + 127) & ~(size_t)127;
#endif
  uint8_t* bands = base + off;
  u4* X = (u4*)(bands + (size_t)nbands * tc_band_bytes(NTH));
  u4* H1s = X + (size_t)(2 * NTH) * id.nthr;
  uint8_t* A0 = (uint8_t*)(x1_global ? H1s : H1s + (size_t)(2 * NTH) * id.nthr);
  c.X = X;
  c.band[0] = bands; c.band[1] = bands + tc_band_bytes(NTH);
  c.slots = entries;                                         // park slot = entry `entries`, x1 home = entry `entries` + 1
  c.nthr = id.nthr;
  const size_t tbl_cta = (size_t)(entries + 3) * 4 * NTH * id.nthr;
  (void)D;
#if defined(PAI_HOSTSIM)
  // one call walks the TC_RL rows of the CTA (id.nthr == TC_RL); they sit in different 8-row groups of the operand
  // layout from CTA to CTA so that the (row / 8) and (row % 8) parts of the addressing are exercised too
  for (int i = 0; i < nbands * tc_band_bytes(NTH); i++) bands[i] = gbands[i];
  c.A = (u4*)A0;
  c.tid = 0;
  c.row0 = 8 * (id.cta % 16) + (TC_RL < 8 ? TC_RL * ((id.cta / 2) % (8 / TC_RL)) : 0);
  c.tbl.p = tbl + (size_t)id.cta * tbl_cta;
  c.tbl.s = id.nthr;
  (void)stagger_cycles;
#else
  {
    const u4* src = (const u4*)gbands;
    u4* dst = (u4*)bands;
    for (int i = id.tid; i < nbands * tc_band_bytes(NTH) / 16; i += id.nthr) dst[i] = src[i];
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");         // the bands are wgmma operands
  __syncthreads();
  const int grp = id.tid / TC_M, lane = id.tid & 31;
  c.grp = grp;
  c.which = 0;
  c.A = (u4*)(A0 + (size_t)grp * TC_M * D);
  c.tid = id.tid;
  // the row of the group whose column sums tc_ld32 brings to this lane: row (lane & 15) of this warp's 16 in m64 half lane >> 4
  c.row0 = 64 * (lane >> 4) + 16 * ((id.tid % TC_M) >> 5) + (lane & 15);
  c.prof = nullptr;
  c.tbl.p = tbl + (size_t)id.cta * tbl_cta + id.tid;
  c.tbl.s = id.nthr;
  if (grp > 0 && stagger_cycles > 0) {                 // put the groups out of phase: some multiply while the others reduce
    const long long t0 = clock64();
    while (clock64() - t0 < (long long)stagger_cycles * grp / (id.nthr / TC_M) * 2) {}
  }
#endif
  if (x1_global) c.H1 = tc_tbl<NTH>(c, entries + 1, 0, 0);
  else { c.H1.p = H1s + c.tid; c.H1.s = id.nthr; }
  return bands;
}
// rows of this thread (simulation: of the TC_RL rows of the CTA) in chunk `chunk`
PAI_DEV void tc_chunk_rows(const CtaId& id, long chunk, long batch, long* g, bool* store) {
  TC_EACH_ROW {
    g[rw] = chunk * id.nthr + id.tid + rw;
    store[rw] = g[rw] < batch;
    if (!store[rw]) g[rw] = batch - 1;
  }
}

template <int NTH>
PAI_DEV void cta_encrypt_tc(u4* smem, const CtaId& id, const uint32_t* prog, int nops, int nodd, const uint32_t* m, const uint32_t* r,
                            uint32_t* out, long batch, u4* tbl, const uint32_t* gzero, const uint8_t* gbands, int stagger_cycles,
                            long long* prof = nullptr) {
  DigitEnv dc;
  digit_bind_enc<NTH>(dc, smem, gzero);
  TcCtx<NTH> c;
  c.dc = &dc;
  tc_cta_begin<NTH>(c, smem, id, dc_enc_limbs(NTH), 2, gbands, tbl, nodd + 1, stagger_cycles);
#if !defined(PAI_HOSTSIM)
  c.prof = prof ? prof + ((size_t)id.cta * (id.nthr / 32) + id.tid / 32) * 16 : nullptr;
#else
  (void)prof;
#endif
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g[TC_RL]; bool store[TC_RL];
    tc_chunk_rows(id, chunk, batch, g, store);
    tc_encrypt_rows<NTH>(c, prog, nops, nodd, m, r, out, g, store);
  }
}

// ---- c^k mod n^2 (raw_mul) on the tensor-core path.  consts = compact constants with ONEM and E3 (dc_pow_limbs); the
// window count is made uniform over the 128-thread group (the groups are independent of each other).
template <int NTH, int W>
PAI_DEV void cta_powmod_tc(u4* smem, const CtaId& id, const uint32_t* base, const uint32_t* exp, int exp_limbs, uint32_t* out, long batch,
                           u4* tbl, const uint32_t* gzero, const uint8_t* gbands, int stagger_cycles) {
  DigitEnv dc;
  digit_bind_pow<NTH>(dc, smem, gzero);
  TcCtx<NTH> c;
  c.dc = &dc;
  tc_cta_begin<NTH>(c, smem, id, dc_pow_limbs(NTH), 2, gbands, tbl, (1 << W), stagger_cycles);
#if !defined(PAI_HOSTSIM)
  __shared__ int s_nwin[4];
#endif
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g[TC_RL]; bool store[TC_RL];
    tc_chunk_rows(id, chunk, batch, g, store);
    int nwin = 0;
    TC_EACH_ROW { int w = (limbs_bitlen(exp + g[rw] * exp_limbs, exp_limbs) + W - 1) / W; nwin = w > nwin ? w : nwin; }
#if !defined(PAI_HOSTSIM)
    if (c.row0 == 0) s_nwin[c.grp] = 0;
    tc_bar_sync(1 + c.grp, TC_M);
    nwin = __reduce_max_sync(0xffffffffu, nwin);
    if ((id.tid & 31) == 0) atomicMax(&s_nwin[c.grp], nwin);
    tc_bar_sync(1 + c.grp, TC_M);
    nwin = s_nwin[c.grp];
    tc_bar_sync(1 + c.grp, TC_M);
#endif
    tc_powmod_rows<NTH, W>(c, base, exp, exp_limbs, nwin, out, g, store);
  }
}

// ---- prod_i c_i^(k_i) over groups of gsz elements per thread (Straus, tc_straus_rows): one output row per group.
template <int NTH, int W>
PAI_DEV void cta_straus_tc(u4* smem, const CtaId& id, const uint32_t* base, const uint32_t* exp, int exp_limbs, int gsz, uint32_t* out,
                           long batch, u4* tbl, const uint32_t* gzero, const uint8_t* gbands, int stagger_cycles) {
  DigitEnv dc;
  digit_bind_pow<NTH>(dc, smem, gzero);
  TcCtx<NTH> c;
  c.dc = &dc;
  tc_cta_begin<NTH>(c, smem, id, dc_pow_limbs(NTH), 2, gbands, tbl, (gsz << W) + 1, stagger_cycles);
  const long ngroups = (batch + gsz - 1) / gsz;
#if !defined(PAI_HOSTSIM)
  __shared__ int s_nwin[4];
#endif
  for (long chunk = id.cta; chunk * id.nthr < ngroups; chunk += id.ncta) {
    long g[TC_RL]; bool store[TC_RL];
    tc_chunk_rows(id, chunk, ngroups, g, store);
    int nwin = 0;
    TC_EACH_ROW {
      for (int i = 0; i < gsz; i++) {
        long j = g[rw] * gsz + i;
        if (j >= batch) break;
        int w = (limbs_bitlen(exp + j * exp_limbs, exp_limbs) + W - 1) / W;
        nwin = w > nwin ? w : nwin;
      }
    }
#if !defined(PAI_HOSTSIM)
    if (c.row0 == 0) s_nwin[c.grp] = 0;
    tc_bar_sync(1 + c.grp, TC_M);
    nwin = __reduce_max_sync(0xffffffffu, nwin);
    if ((id.tid & 31) == 0) atomicMax(&s_nwin[c.grp], nwin);
    tc_bar_sync(1 + c.grp, TC_M);
    nwin = s_nwin[c.grp];
    tc_bar_sync(1 + c.grp, TC_M);
#endif
    tc_straus_rows<NTH, W>(c, base, exp, exp_limbs, gsz, nwin, batch, out, g, store);
  }
}

// ---- decrypt with the reductions on the tensor cores.  consts = [ P side | Q side | pinvqM ] as in cta_decrypt_digit;
// bands: p (2), q (2)
template <int NTP, int W>
PAI_DEV void cta_decrypt_tc(u4* smem, const CtaId& id, int nwin_p, int nwin_q, const uint32_t* cin, uint32_t* out, long batch, u4* tbl,
                            const uint8_t* gbands, int stagger_cycles) {
  DSideC<NTP> P, Qs;
  dside_bind<NTP>(P, smem, nwin_p);
  dside_bind<NTP>(Qs, smem + dside_limbs<NTP>() / 4, nwin_q);
  Opnd pinvqM{smem + 2 * (dside_limbs<NTP>() / 4), 1};
  TcCtx<NTP> c;
  c.dc = &P.dc;
  uint8_t* bands = tc_cta_begin<NTP>(c, smem, id, (2 * (dside_limbs<NTP>() / 4) + 2 * NTP) * 4, 4, gbands, tbl, (1 << W), stagger_cycles);
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g[TC_RL]; bool store[TC_RL];
    tc_chunk_rows(id, chunk, batch, g, store);
    tc_decrypt_rows<NTP, W>(c, P, Qs, pinvqM, bands, cin, out, g, store);
  }
}

// ---- mulmod.  consts = [ blob ]
template <int NT>
PAI_DEV void cta_mulmod(u4* smem, const CtaId& id, const uint32_t* a, const uint32_t* b, uint32_t* out, long batch) {
  ModC mc;
  modc_bind(mc, smem, NT);
  Opnd buf[3];
  cta_bufs<NT>(buf, 3, smem, mc_limbs(NT) / 4, id);
  const int l = 8 * NT;
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g = chunk * id.nthr + id.tid;
    bool store = g < batch;
    if (!store) g = batch - 1;
    prog_mulmod<NT>(buf, mc, a + g * l, b + g * l, out + g * l, store);
  }
}

// ---- product of many rows modulo N (homomorphic SUM of a ciphertext vector: sum(), np.mean over EncryptedNumbers,
// phe/tests/math_test.py:44-58).  consts = [ blob ]; three buffers.  No row is ever converted to Montgomery form:
// every mont_mul of two numbers carrying R-exponents e1, e2 (value * R^e) gives e1 + e2 - 1, a plain row has e = 0, so a
// product tree over L rows ends at e = 1 - L however it is shaped.  The deficit is repaid by CORRECTION rows
// K_i = R^(2^i + 1) mod N (one per set bit of L, a per-key table): as leaves of the same tree they bring the total to
// e = 1, and one multiplication by 1 leaves the domain.  Every thread multiplies its strided share of the rows (read
// straight from global memory), the CTA folds its threads' partials in a shared-memory tree; threads without rows
// contribute R mod N (e = 1, neutral).  final = 0: the CTA's partial goes to row `cta` of out (input of the second
// launch); final = 1: canonical result in row 0.  corr_bits: set bits = correction rows to append to the input.
PAI_DEV const uint32_t* reduce_row(const uint32_t* rows, long batch, int l, const uint32_t* corr, unsigned long long corr_bits, long v) {
  if (v < batch) return rows + v * l;
  long j = v - batch;
  for (int i = 0; i < 64; i++)
    if ((corr_bits >> i) & 1ull) { if (j == 0) return corr + (long)i * l; j--; }
  return corr;
}
PAI_DEV int popcount64(unsigned long long x) { int c = 0; while (x) { c += (int)(x & 1ull); x >>= 1; } return c; }

template <int NT>
PAI_DEV void cta_reduce_mul(u4* smem, const CtaId& id, const uint32_t* rows, long batch, uint32_t* out, const uint32_t* corr,
                            unsigned long long corr_bits, int final) {
  ModC mc;
  modc_bind(mc, smem, NT);
  Opnd buf[3];
  cta_bufs<NT>(buf, 3, smem, mc_limbs(NT) / 4, id);
  const int l = 8 * NT;
  const long T = (long)id.ncta * id.nthr;
  const long total = batch + popcount64(corr_bits);
  long g = (long)id.cta * id.nthr + id.tid;
  int cur = 0;
  if (g < total) {
    load_row(buf[0], reduce_row(rows, batch, l, corr, corr_bits, g), 2 * NT, 2 * NT);
    for (g += T; g < total; g += T) {
      Opnd r{(u4*)reduce_row(rows, batch, l, corr, corr_bits, g), 1};
      mont_mul<NT>(buf[cur ^ 1], buf[cur], r, mc.N, mc.ninv);
      cur ^= 1;
    }
  } else {
    big_copy<NT>(buf[0], mc.R1);
  }
  // `cur` differs between threads (different row counts): settle every partial in buf[2]
  big_copy<NT>(buf[2], buf[cur]);
  int src = 2;
#if !defined(PAI_HOSTSIM)
  for (int step = 1; step < id.nthr; step <<= 1) {
    const int dst = (src + 1) % 3;
    __syncthreads();
    if ((id.tid & (2 * step - 1)) == 0) {
      if (id.tid + step < id.nthr) {
        Opnd other = buf[src];
        other.p += step;                                           // the partner's buffer in the interleaved layout
        mont_mul<NT>(buf[dst], buf[src], other, mc.N, mc.ninv);
      } else {
        big_copy<NT>(buf[dst], buf[src]);                          // no partner on this level
      }
    }
    src = dst;
  }
  const bool writer = id.tid == 0;
  const int shift = 0;
#else
  // the simulation runs the threads of a CTA one after the other: the last one folds everybody's partials serially
  const bool writer = id.tid == id.nthr - 1;
  const int shift = id.tid;
  if (writer) {
    Opnd acc = buf[src], o = buf[(src + 1) % 3];
    acc.p -= shift; o.p -= shift;                                  // thread 0's buffers
    for (int t = 1; t < id.nthr; t++) {
      Opnd a = buf[src];
      a.p += t - shift;
      mont_mul<NT>(o, acc, a, mc.N, mc.ninv);
      big_copy<NT>(acc, o);
    }
  }
#endif
  if (writer) {
    Opnd res = buf[src], tmp = buf[(src + 1) % 3];
    res.p -= shift; tmp.p -= shift;
    uint32_t* orow = out + (final ? 0 : (long)id.cta * l);
    if (final) { mont_mul<NT>(tmp, res, mc.ONE, mc.N, mc.ninv); store_row(orow, tmp, 2 * NT); }
    else store_row(orow, res, 2 * NT);
  }
}

// correction rows of cta_reduce_mul: K_0 = R^2, K_(i+1) = K_i^2 / R = R^(2^(i+1) + 1)   (single thread, once per modulus)
template <int NT>
PAI_DEV void reduce_corr_setup(u4* smem, const CtaId& id, uint32_t* tbl, int rows) {
  if (id.cta != 0 || id.tid != 0) return;
  ModC mc;
  modc_bind(mc, smem, NT);
  Opnd buf[2];
  cta_bufs<NT>(buf, 2, smem, mc_limbs(NT) / 4, id);
  const int l = 8 * NT;
  big_copy<NT>(buf[0], mc.R2);
  for (int i = 0; i < rows; i++) {
    store_row(tbl + (long)i * l, buf[i & 1], 2 * NT);
    mont_sqr<NT>(buf[(i & 1) ^ 1], buf[i & 1], mc.N, mc.ninv);
  }
}

// ---- powmod.  consts = [ blob ].  exp rows in global memory (exp_stride = 0: one shared exponent).
// nwin_fixed >= 0: uniform window count given by the host; < 0: per element from the bit length
// (made warp-uniform on the device so that a warp never diverges in the ladder).
template <int NT, int W>
PAI_DEV void cta_powmod(u4* smem, const CtaId& id, const uint32_t* base, int base_tiles, const uint32_t* exp, int exp_limbs,
                        long exp_stride, int nwin_fixed, uint32_t* out, long batch, u4* tbl, unsigned long long* counter) {
  ModC mc;
  modc_bind(mc, smem, NT);
  PowEnv<NT> E;
  cta_bufs<NT>(E.buf, 3, smem, mc_limbs(NT) / 4, id);
  E.tbl = cta_table<NT, W>(tbl, id);
  E.mc = &mc;
  const int l = 8 * NT;
  RowSched sched = sched_init(id, counter, batch);
  for (long g = sched_next_row(sched, id); g >= 0; g = sched_next_row(sched, id)) {
    bool store = g < batch;
    if (!store) g = batch - 1;
    const uint32_t* e = exp + g * exp_stride;
    int nwin = nwin_fixed;
    if (nwin < 0) {
      nwin = (limbs_bitlen(e, exp_limbs) + W - 1) / W;
#if !defined(PAI_HOSTSIM)
      nwin = __reduce_max_sync(0xffffffffu, nwin);
#endif
    }
    prog_powmod<NT, W>(E, base + g * (long)(8 * base_tiles), base_tiles, e, exp_limbs, nwin, out + g * l, store);
  }
}

// ---- invert.  consts = [ blob ]; four buffers.  flags (optional): 0 -> plain copy of a.
template <int NT>
PAI_DEV void cta_invert(u4* smem, const CtaId& id, const uint32_t* a, int a_tiles, const int32_t* flags, uint32_t* out,
                        int32_t* status, long batch) {
  ModC mc;
  modc_bind(mc, smem, NT);
  Opnd buf[4];
  cta_bufs<NT>(buf, 4, smem, mc_limbs(NT) / 4, id);
  const int l = 8 * NT;
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g = chunk * id.nthr + id.tid;
    if (g >= batch) continue;
    if (flags && !flags[g]) {
      const u4* src = (const u4*)(a + g * (long)(8 * a_tiles));
      u4* dst = (u4*)(out + g * l);
      u4 z; z.x = z.y = z.z = z.w = 0;
      for (int q = 0; q < 2 * NT; q++) dst[q] = q < 2 * a_tiles ? src[q] : z;
      if (status) status[g] = 0;
      continue;
    }
    int fail = prog_invert<NT>(buf, mc, a + g * (long)(8 * a_tiles), a_tiles, out + g * l, true);
    if (status) status[g] = fail;
  }
}

// ---- invert, amortised (Montgomery's simultaneous inversion): the negative-scalar branch of _raw_mul needs invert(c, n^2)
// for every flagged row (phe/paillier.py:745-749); a binary extended gcd per row costs as much as hundreds of modular
// multiplications.  Here a thread owns a SEGMENT of `seg` consecutive rows: prefix products of the flagged rows in the
// Montgomery domain (parked in the output rows), ONE extended gcd of the segment's product, then the back substitution
// inv_i = I * P_(i-1), I <- I * a_i -- six multiplications per row.  If the product has no inverse (some row shares a factor
// with N, or is 0) the segment falls back to one gcd per row so that every row gets its own status.  Unflagged rows are copied.
// Four buffers (those of prog_invert).
template <int NT>
PAI_DEV void cta_invert_batch(u4* smem, const CtaId& id, const uint32_t* a, const int32_t* flags, uint32_t* out, int32_t* status,
                              long batch, int seg) {
  ModC mc;
  modc_bind(mc, smem, NT);
  Opnd buf[4];
  cta_bufs<NT>(buf, 4, smem, mc_limbs(NT) / 4, id);
  const int l = 8 * NT;
  const long nseg = (batch + seg - 1) / seg;
  for (long sg = (long)id.cta * id.nthr + id.tid; sg < nseg; sg += (long)id.ncta * id.nthr) {
    const long lo = sg * seg, hi = lo + seg < batch ? lo + seg : batch;
    // forward: P_i = P_(i-1) * a_i * R  (Montgomery form of the running product) -> out row i; unflagged rows copied
    long last = -1, nflag = 0;
    int cur = 0;                                             // running product in buf[cur] (0 or 1)
    for (long i = lo; i < hi; i++) {
      const uint32_t* row = a + i * l;
      if (!flags[i]) {
        const u4* src = (const u4*)row;
        u4* dst = (u4*)(out + i * l);
        for (int q = 0; q < 2 * NT; q++) dst[q] = src[q];
        status[i] = 0;
        continue;
      }
      load_row(buf[2], row, 2 * NT, 2 * NT);
      if (last < 0) mont_mul<NT>(buf[cur], buf[2], mc.R2, mc.N, mc.ninv);                    // a_i * R
      else {
        mont_mul<NT>(buf[3], buf[2], mc.R2, mc.N, mc.ninv);
        mont_mul<NT>(buf[cur ^ 1], buf[cur], buf[3], mc.N, mc.ninv);
        cur ^= 1;
      }
      store_row(out + i * l, buf[cur], 2 * NT);
      last = i;
      nflag++;
    }
    if (last < 0) continue;
    // one inversion of the segment's product: (A R)^-1 = A^-1 R^-1 (plain gcd), times R^3 -> A^-1 R
    int fail = prog_invert<NT>(buf, mc, out + last * l, NT, out + last * l, false);         // result in buf[3] (x2)
    if (fail) {
      for (long i = lo; i < hi; i++)
        if (flags[i]) status[i] = prog_invert<NT>(buf, mc, a + i * l, NT, out + i * l, true);
      continue;
    }
    mont_mul<NT>(buf[0], buf[3], mc.R3, mc.N, mc.ninv);      // I = (a_lo .. a_last)^-1 in Montgomery form
    int ic = 0;                                              // I lives in buf[ic] (0 or 1)
    long prev = last;
    for (long i = last; i >= lo; i--) {
      if (!flags[i]) continue;
      // find the previous flagged row (its out row holds P_prev)
      long pj = i - 1;
      while (pj >= lo && !flags[pj]) pj--;
      if (pj >= lo) {
        Opnd pp{(u4*)(out + pj * l), 1};
        mont_mul<NT>(buf[2], buf[ic], pp, mc.N, mc.ninv);    // a_i^-1 (Montgomery form)
      } else {
        big_copy<NT>(buf[2], buf[ic]);                       // first flagged row: I itself
      }
      mont_mul<NT>(buf[3], buf[2], mc.ONE, mc.N, mc.ninv);   // leave the domain
      if (pj >= lo) {                                        // I <- I * a_i (before row i is overwritten)
        Opnd ai{(u4*)(a + i * l), 1};
        mont_mul<NT>(buf[2], ai, mc.R2, mc.N, mc.ninv);
        mont_mul<NT>(buf[ic ^ 1], buf[ic], buf[2], mc.N, mc.ninv);
        ic ^= 1;
      }
      store_row(out + i * l, buf[3], 2 * NT);
      status[i] = 0;
      (void)prev;
    }
  }
}

// ---- raw_mul preparation (phe/paillier.py:742-749): s >= n - max_int  ->  flag, exponent n - s
// Plain one-thread-per-element kernel body over global memory (a few hundred integer ops per element).
//   n, thresh (= n - max_int): ln limbs.
PAI_DEV void rawmul_prep(const uint32_t* n, const uint32_t* thresh, int ln, const uint32_t* s, uint32_t* e_out,
                         int32_t* flag, long g) {
  const uint32_t* sr = s + g * ln;
  uint32_t* eo = e_out + g * ln;
  uint32_t bo = 0;
  for (int i = 0; i < ln; i++) { uint64_t d = (uint64_t)sr[i] - thresh[i] - bo; bo = (uint32_t)(d >> 63); }
  int neg = bo ? 0 : 1;                                    // s >= thresh
  flag[g] = neg;
  if (neg) {
    uint32_t b2 = 0;
    for (int i = 0; i < ln; i++) { uint64_t d = (uint64_t)n[i] - sr[i] - b2; eo[i] = (uint32_t)d; b2 = (uint32_t)(d >> 63); }
  } else {
    for (int i = 0; i < ln; i++) eo[i] = sr[i];
  }
}

// ---- decrypt.  consts = [ P side | Q side | pinvqM ], side = [ blob(x^2) | blob(x) | xinv | hM | e ]
template <int NTP>
PAI_DEV int side_quads() { return mc_limbs(2 * NTP) / 4 + mc_limbs(NTP) / 4 + 3 * 2 * NTP; }
template <int NTP>
PAI_DEV int dec_const_quads() { return 2 * side_quads<NTP>() + 2 * NTP; }

template <int NTP>
PAI_DEV void side_bind(SideC<NTP>& S, u4* base, int nwin) {
  modc_bind(S.sq, base, 2 * NTP);
  u4* p = base + mc_limbs(2 * NTP) / 4;
  modc_bind(S.pr, p, NTP);
  p += mc_limbs(NTP) / 4;
  S.xinv.p = p; S.xinv.s = 1;
  p += 2 * NTP;
  S.hM.p = p; S.hM.s = 1;
  p += 2 * NTP;
  S.e = (const uint32_t*)p;
  S.nwin = nwin;
}

template <int NTP, int W>
PAI_DEV void cta_decrypt(u4* smem, const CtaId& id, int nwin_p, int nwin_q, const uint32_t* c, uint32_t* out, long batch, u4* tbl,
                         unsigned long long* counter, const uint32_t* pre_p = nullptr, const uint32_t* pre_q = nullptr) {
  SideC<NTP> P, Qs;
  side_bind<NTP>(P, smem, nwin_p);
  side_bind<NTP>(Qs, smem + side_quads<NTP>(), nwin_q);
  Opnd pinvqM{smem + 2 * side_quads<NTP>(), 1};
  PowEnv<2 * NTP> E;
  cta_bufs<2 * NTP>(E.buf, 3, smem, dec_const_quads<NTP>(), id);
  E.tbl = cta_table<2 * NTP, W>(tbl, id);
  E.mc = &P.sq;
  const int lc = 32 * NTP, ln = 16 * NTP;
  RowSched sched = sched_init(id, counter, batch);
  for (long g = sched_next_row(sched, id); g >= 0; g = sched_next_row(sched, id)) {
    bool store = g < batch;
    if (!store) g = batch - 1;
    prog_decrypt<NTP, W>(E, P, Qs, pinvqM, c + g * lc, out + g * ln, store, pre_p ? pre_p + g * ln : nullptr,
                         pre_q ? pre_q + g * ln : nullptr);
  }
}


// ---- decrypt in digit form.  consts = [ P side | Q side | pinvqM ], side = dside_limbs<NTP>() limbs
template <int NTP>
PAI_DEV int ddec_const_quads() { return 2 * (dside_limbs<NTP>() / 4) + 2 * NTP; }

template <int NTP, int W>
PAI_DEV void cta_decrypt_digit(u4* smem, const CtaId& id, int nwin_p, int nwin_q, const uint32_t* c, uint32_t* out, long batch,
                               u4* tbl, unsigned long long* counter) {
  DSideC<NTP> P, Qs;
  dside_bind<NTP>(P, smem, nwin_p);
  dside_bind<NTP>(Qs, smem + dside_limbs<NTP>() / 4, nwin_q);
  Opnd pinvqM{smem + 2 * (dside_limbs<NTP>() / 4), 1};
  DPowEnv<NTP> E;
  cta_bufs<2 * NTP>(E.buf, 2, smem, ddec_const_quads<NTP>(), id);
  E.tbl = cta_table_slots<2 * NTP>(tbl, id, 1 << W);
  E.dc = &P.dc;
  E.step_sync = 1;
  const int lc = 32 * NTP, ln = 16 * NTP;
  (void)counter;
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g = chunk * id.nthr + id.tid;
    bool store = g < batch;
    if (!store) g = batch - 1;
    prog_decrypt_digit<NTP, W>(E, P, Qs, pinvqM, c + g * lc, out + g * ln, store);
  }
}

// ---- encrypt with the private key in digit form (pai_priv_encrypt).  consts = pe_const_limbs<NTP>(); two buffers of
// 2*NTP tiles per thread and the static chunks of cta_decrypt_digit.  pre_p / pre_q: r^n mod p^2 / q^2 from the warp
// kernels (then no ladder runs), or null.
template <int NTP, int W>
PAI_DEV void cta_priv_encrypt_digit(u4* smem, const CtaId& id, int nwin_p, int nwin_q, const uint32_t* m, const uint32_t* r,
                                    const uint32_t* pre_p, const uint32_t* pre_q, uint32_t* out, long batch, u4* tbl) {
  PEncC<NTP> C;
  pe_bind<NTP>(C, smem, nwin_p, nwin_q);
  DPowEnv<NTP> E;
  cta_bufs<2 * NTP>(E.buf, 2, smem, pe_const_limbs<NTP>() / 4, id);
  E.tbl = cta_table_slots<2 * NTP>(tbl, id, pe_slots(W));
  E.dc = &C.P.dc;
  E.step_sync = 1;
  const int ln = 16 * NTP, lc = 32 * NTP;
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g = chunk * id.nthr + id.tid;
    bool store = g < batch;
    if (!store) g = batch - 1;
    prog_priv_encrypt_digit<NTP, W>(E, C, m + g * ln, r + g * ln, pre_p ? pre_p + g * ln : nullptr, pre_q ? pre_q + g * ln : nullptr,
                                    out + g * lc, store);
  }
}


// ---- c^k mod n^2 in digit form (raw_mul).  consts = compact constants with ONEM and E3 (dc_pow_limbs).
// Exponents differ per element; the window count is made CTA-uniform (max over the CTA through one shared word)
// so that the per-step barrier of the ladder is safe here too.
template <int NTH, int W>
PAI_DEV void cta_powmod_digit(u4* smem, const CtaId& id, const uint32_t* base, const uint32_t* exp, int exp_limbs, uint32_t* out,
                              long batch, u4* tbl, unsigned long long* counter, const uint32_t* gzero) {
  DigitEnv dc;
  digit_bind_pow<NTH>(dc, smem, gzero);
  DPowEnv<NTH> E;
  cta_bufs<2 * NTH>(E.buf, 2, smem, dc_pow_limbs(NTH) / 4, id);
  E.tbl = cta_table_slots<2 * NTH>(tbl, id, 1 << W);
  E.dc = &dc;
  E.step_sync = 1;
  const int lc = 16 * NTH;
  (void)counter;
#if !defined(PAI_HOSTSIM)
  __shared__ int s_nwin;
#endif
  for (long chunk = id.cta; chunk * id.nthr < batch; chunk += id.ncta) {
    long g = chunk * id.nthr + id.tid;
    bool store = g < batch;
    if (!store) g = batch - 1;
    const uint32_t* e = exp + g * exp_limbs;
    int nwin = (limbs_bitlen(e, exp_limbs) + W - 1) / W;
#if !defined(PAI_HOSTSIM)
    if (id.tid == 0) s_nwin = 0;
    __syncthreads();
    nwin = __reduce_max_sync(0xffffffffu, nwin);
    if ((id.tid & 31) == 0) atomicMax(&s_nwin, nwin);
    __syncthreads();
    nwin = s_nwin;
#endif
    prog_powmod_digit<NTH, W>(E, base + g * lc, e, exp_limbs, nwin, out + g * lc, store);
  }
}

// ---- plaintext CSR matrix times ciphertext vector in digit form (pai_raw_matvec).  consts = dc_pow_limbs, two buffers.
// Tables: one thread per slot (see prog_matvec_table); slot ncols + i is built from cinv[i] only where flag[i] is set.
template <int NTH>
PAI_DEV void cta_matvec_table(u4* smem, const CtaId& id, const uint32_t* c, const uint32_t* cinv, const int32_t* flag,
                              long ncols, long nslots, int w, u4* tbl, const uint32_t* gzero) {
  DigitEnv dc;
  digit_bind_pow<NTH>(dc, smem, gzero);
  DPowEnv<NTH> E;
  cta_bufs<2 * NTH>(E.buf, 2, smem, dc_pow_limbs(NTH) / 4, id);
  E.tbl = E.buf[0];                                         // (the shared tables are addressed by mv_entry)
  E.dc = &dc;
  E.step_sync = 0;
  const int lc = 16 * NTH;
  for (long s = (long)id.cta * id.nthr + id.tid; s < nslots; s += (long)id.ncta * id.nthr) {
    const bool inv = s >= ncols;
    const long col = inv ? s - ncols : s;
    if (inv && !flag[col]) continue;
    prog_matvec_table<NTH>(E, (inv ? cinv : c) + col * lc, tbl, s, w);
  }
}

// Rows: one thread per output row, handed out by the row scheduler.  The window count comes from the largest magnitude
// of the row, made warp-uniform, so the lanes of a warp run the same squaring chain.  Rows beyond the last one repeat it
// without storing (the warp stays complete for the reduction).
template <int NTH>
PAI_DEV void cta_matvec_digit(u4* smem, const CtaId& id, const u4* tbl, long ncols, int w, const int64_t* indptr,
                              const int32_t* indices, const uint32_t* mag, int ml, const uint8_t* neg, uint32_t* out,
                              long nrows, unsigned long long* counter, const uint32_t* gzero) {
  DigitEnv dc;
  digit_bind_pow<NTH>(dc, smem, gzero);
  DPowEnv<NTH> E;
  cta_bufs<2 * NTH>(E.buf, 2, smem, dc_pow_limbs(NTH) / 4, id);
  E.tbl = E.buf[0];
  E.dc = &dc;
  E.step_sync = 0;
  const int lc = 16 * NTH;
  RowSched sched = sched_init(id, counter, nrows);
  for (long g = sched_next_row(sched, id); g >= 0; g = sched_next_row(sched, id)) {
    bool store = g < nrows;
    if (!store) g = nrows - 1;
    const long lo = indptr[g], hi = indptr[g + 1];
    int nbits = 0;
    for (long t = lo; t < hi; t++) {
      const int b = limbs_bitlen(mag + t * ml, ml);
      nbits = b > nbits ? b : nbits;
    }
    int nwin = (nbits + w - 1) / w;
#if !defined(PAI_HOSTSIM)
    nwin = __reduce_max_sync(0xffffffffu, nwin);
#endif
    prog_matvec_row<NTH>(E, tbl, ncols, w, nwin, indices, mag, ml, neg, lo, hi, out + g * lc, store);
  }
}

}  // namespace pai
