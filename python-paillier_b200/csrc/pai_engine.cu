// pai_engine.cu -- host orchestration + C ABI of libpaillier_b200.so (see include/paillier_b200.h).
//
// Product build:   nvcc -gencode arch=compute_90a,code=sm_90a ... -shared  (python-paillier_b200/build.py)
// Test-only build: g++ -x c++ -DPAI_HOSTSIM ...  -> tests/hostsim/libpaillier_b200_hostsim.so
//                  (same orchestration, kernels run on the CPU; never loaded by the product package)
//
// All big-integer work happens in the kernels (pai_cta.cuh / pai_kernels.cuh / pai_core.cuh).  The
// host side only pads limb arrays, multiplies p*q / n*n once per key (schoolbook, a few thousand
// word operations), sizes launches and workspaces, and sequences kernels on the caller's stream.
#include "pai_rt.h"
#include "pai_pack.cuh"

#include <algorithm>
#include <cstdio>
#include <deque>
#include <map>
#include <mutex>
#include <new>

using namespace pai;

// ------------------------------------------------------------------------------------------------
// kernel bodies (functors launched through rt_launch / k_body)
namespace {

template <int NT>
struct SetupBody {
  const uint32_t* consts; int const_quads;
  uint32_t* blob; uint32_t* scratch;
  PAI_MEM void run(u4*, const CtaId& id) const { if (id.tid == 0 && id.cta == 0) mod_setup<NT>(blob, scratch); }
};
// x^-1 mod 2^(32 nl) for the L function (single thread)
struct XinvBody {
  const uint32_t* consts; int const_quads;
  uint32_t* out; const uint32_t* x; int nl;
  PAI_MEM void run(u4*, const CtaId& id) const { if (id.tid == 0 && id.cta == 0) inv_mod_2k(out, x, nl); }
};
template <int NT>
struct EncBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* prog; int nops, nodd; const uint32_t* m; const uint32_t* r; uint32_t* out; long batch; u4* tbl;
  unsigned long long* counter;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_encrypt<NT>(smem, id, prog, nops, nodd, m, r, out, batch, tbl, counter); }
};
template <int NTH>
struct DigitSetupBody {
  const uint32_t* consts; int const_quads;
  uint32_t* blob; uint32_t* scratch;
  PAI_MEM void run(u4*, const CtaId& id) const { if (id.tid == 0 && id.cta == 0) digit_setup<NTH>(blob, scratch); }
};
template <int NTH>
struct EncDigitBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* prog; int nops, nodd; const uint32_t* m; const uint32_t* r; uint32_t* out; long batch; u4* tbl;
  unsigned long long* counter; const uint32_t* gzero;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_encrypt_digit<NTH>(smem, id, prog, nops, nodd, m, r, out, batch, tbl, counter, gzero); }
};
// tensor-core path (pai_tc.cuh)
template <int NTH>
struct TcSetupBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* N; uint8_t* blob; uint32_t* scratch;
  PAI_MEM void run(u4*, const CtaId& id) const { if (id.tid == 0 && id.cta == 0) tc_setup<NTH>(N, blob, scratch); }
};
template <int NTH>
struct TcEncBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* prog; int nops, nodd; const uint32_t* m; const uint32_t* r; uint32_t* out; long batch; u4* tbl;
  const uint32_t* gzero; const uint8_t* bands; int stagger; long long* prof;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_encrypt_tc<NTH>(smem, id, prog, nops, nodd, m, r, out, batch, tbl, gzero, bands, stagger, prof); }
};
template <int NTH, int W>
struct TcPowBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* base; const uint32_t* exp; int exp_limbs; uint32_t* out; long batch; u4* tbl; const uint32_t* gzero;
  const uint8_t* bands; int stagger;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_powmod_tc<NTH, W>(smem, id, base, exp, exp_limbs, out, batch, tbl, gzero, bands, stagger); }
};
template <int NTH, int W>
struct TcStrausBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* base; const uint32_t* exp; int exp_limbs; int gsz; uint32_t* out; long batch; u4* tbl; const uint32_t* gzero;
  const uint8_t* bands; int stagger;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_straus_tc<NTH, W>(smem, id, base, exp, exp_limbs, gsz, out, batch, tbl, gzero, bands, stagger); }
};
template <int NTP, int W>
struct TcDecBody {
  const uint32_t* consts; int const_quads;
  int nwin_p, nwin_q; const uint32_t* c; uint32_t* out; long batch; u4* tbl; const uint8_t* bands; int stagger;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_decrypt_tc<NTP, W>(smem, id, nwin_p, nwin_q, c, out, batch, tbl, bands, stagger); }
};
template <int NTH, int W>
struct PowDigitBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* base; const uint32_t* exp; int exp_limbs; uint32_t* out; long batch; u4* tbl; unsigned long long* counter;
  const uint32_t* gzero;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_powmod_digit<NTH, W>(smem, id, base, exp, exp_limbs, out, batch, tbl, counter, gzero); }
};
// matrix-vector product (pai_raw_matvec): column flags, shared window tables, rows
struct MatFlagBody {
  const uint32_t* consts; int const_quads;
  const int32_t* indices; const uint8_t* neg; long nnz; int32_t* flag;
  PAI_MEM void run(u4*, const CtaId& id) const {
    for (long t = (long)id.cta * id.nthr + id.tid; t < nnz; t += (long)id.ncta * id.nthr)
      if (neg[t]) flag[indices[t]] = 1;
  }
};
template <int NTH>
struct MatTblBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* c; const uint32_t* cinv; const int32_t* flag; long ncols, nslots; int w; u4* tbl; const uint32_t* gzero;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_matvec_table<NTH>(smem, id, c, cinv, flag, ncols, nslots, w, tbl, gzero); }
};
template <int NTH>
struct MatRowBody {
  const uint32_t* consts; int const_quads;
  const u4* tbl; long ncols; int w; const int64_t* indptr; const int32_t* indices; const uint32_t* mag; int ml;
  const uint8_t* neg; uint32_t* out; long nrows; unsigned long long* counter; const uint32_t* gzero;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    cta_matvec_digit<NTH>(smem, id, tbl, ncols, w, indptr, indices, mag, ml, neg, out, nrows, counter, gzero);
  }
};
template <int NT>
struct MulBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* a; const uint32_t* b; uint32_t* out; long batch;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_mulmod<NT>(smem, id, a, b, out, batch); }
};
template <int NT>
struct ReduceBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* rows; long batch; uint32_t* out; const uint32_t* corr; unsigned long long corr_bits; int final;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_reduce_mul<NT>(smem, id, rows, batch, out, corr, corr_bits, final); }
};
template <int NT>
struct ReduceCorrBody {
  const uint32_t* consts; int const_quads;
  uint32_t* tbl; int rows;
  PAI_MEM void run(u4* smem, const CtaId& id) const { reduce_corr_setup<NT>(smem, id, tbl, rows); }
};
template <int NT, int W>
struct PowBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* base; int base_tiles; const uint32_t* exp; int exp_limbs; long exp_stride; int nwin_fixed;
  uint32_t* out; long batch; u4* tbl; unsigned long long* counter;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    cta_powmod<NT, W>(smem, id, base, base_tiles, exp, exp_limbs, exp_stride, nwin_fixed, out, batch, tbl, counter);
  }
};
template <int NT>
struct InvBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* a; int a_tiles; const int32_t* flags; uint32_t* out; int32_t* status; long batch;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_invert<NT>(smem, id, a, a_tiles, flags, out, status, batch); }
};
template <int NT>
struct InvBatchBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* a; const int32_t* flags; uint32_t* out; int32_t* status; long batch; int seg;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_invert_batch<NT>(smem, id, a, flags, out, status, batch, seg); }
};
template <int NT, int W>
struct MillerRabinBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* cand; const uint32_t* bases; int rounds; int32_t* result; uint32_t* ws; long batch;
  PAI_MEM void run(u4*, const CtaId& id) const {
    const int L = 8 * NT;
    for (long g = (long)id.cta * id.nthr + id.tid; g < batch; g += (long)id.ncta * id.nthr)
      prog_miller_rabin<NT, W>(ws + ((long)id.cta * id.nthr + id.tid) * mr_ws_limbs<NT, W>(), cand + g * L, bases + g * (long)rounds * L, rounds,
                               result + g);
  }
};
struct RngBody {
  const uint32_t* consts; int const_quads;
  uint32_t key[8]; unsigned long long nonce; const uint32_t* n; int ln, nbits; uint32_t* out; long batch;
  PAI_MEM void run(u4*, const CtaId& id) const {
    for (long g = (long)id.cta * id.nthr + id.tid; g < batch; g += (long)id.ncta * id.nthr)
      rng_fill_lt_n(key, nonce, (uint64_t)g, n, ln, nbits, out + g * ln);
  }
};
// ---- warp-per-ciphertext bodies (pai_coop.cuh): small batches
template <int K>
struct CoopPowBody {
  const uint32_t* consts; int const_quads;
  int nsides;                               // 1, or 2 = both CRT halves of one ciphertext on two warps
  const uint32_t* blob[2]; uint32_t n0inv[2]; const uint32_t* e[2]; int e_limbs; int nwin[2]; uint32_t* out[2];
  const uint32_t* base; int base_limbs; int out_limbs; long batch;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    const int warp = COOP_WARPS == 1 ? 0 : id.tid >> 5, nwarp = COOP_WARPS == 1 ? 1 : id.nthr >> 5;
    uint32_t* tbl = (uint32_t*)smem + (size_t)warp * ((1 << COOP_W) * K * 32);
    const long items = batch * nsides;
    for (long it = (long)id.cta * nwarp + warp; it < items; it += (long)id.ncta * nwarp) {
      const int sd = (int)(it % nsides);
      const long g = it / nsides;
      coop_powmod<K>(blob[sd], n0inv[sd], base + g * base_limbs, base_limbs, e[sd], e_limbs, nwin[sd],
                     out[sd] + g * out_limbs, out_limbs, tbl);
    }
  }
};
template <int K>
struct CoopEncBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* blob; uint32_t n0inv; const uint32_t* nrow; int n_limbs; int nwin;
  const uint32_t* m; const uint32_t* r; uint32_t* out; long batch;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    const int warp = COOP_WARPS == 1 ? 0 : id.tid >> 5, nwarp = COOP_WARPS == 1 ? 1 : id.nthr >> 5;
    uint32_t* tbl = (uint32_t*)smem + (size_t)warp * ((1 << COOP_W) * K * 32);
    for (long g = (long)id.cta * nwarp + warp; g < batch; g += (long)id.ncta * nwarp)
      coop_encrypt<K>(blob, n0inv, nrow, n_limbs, nrow, nwin, m + g * n_limbs, r + g * n_limbs, out + g * 2 * n_limbs,
                      2 * n_limbs, tbl);
  }
};
struct ToDecBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* limbs; int L; uint8_t* text; int chunks; long batch;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    for (long g = (long)id.cta * id.nthr + id.tid; g < batch; g += (long)id.ncta * id.nthr)
      radix_to_decimal((uint32_t*)smem, id.tid, id.nthr, limbs + g * L, L, text + g * (long)chunks * 9, chunks);
  }
};
struct FromDecBody {
  const uint32_t* consts; int const_quads;
  const uint8_t* text; int width; uint32_t* limbs; int L; int32_t* status; long batch;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    for (long g = (long)id.cta * id.nthr + id.tid; g < batch; g += (long)id.ncta * id.nthr) {
      int st = radix_from_decimal((uint32_t*)smem, id.tid, id.nthr, text + g * (long)width, width, limbs + g * L, L);
      if (status) status[g] = st;
    }
  }
};
// packed fixed-point rows (pai_pack.cuh), one thread per plaintext row; n (ln limbs) is the CTA's constant area
struct PackBody {
  const uint32_t* consts; int const_quads;
  const int64_t* s; long count; int b, K, ln; uint32_t* m; int32_t* status; long rows;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    for (long r = (long)id.cta * id.nthr + id.tid; r < rows; r += (long)id.ncta * id.nthr) {
      const long lo = r * K;
      status[r] = pack_row(s + lo, count - lo < K ? (int)(count - lo) : K, b, (const uint32_t*)smem, ln, m + r * ln);
    }
  }
};
struct UnpackBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* m; int b, K, ln; int64_t* s; long count; int32_t* status; long rows;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    for (long r = (long)id.cta * id.nthr + id.tid; r < rows; r += (long)id.ncta * id.nthr) {
      const long lo = r * K;
      status[r] = unpack_row(m + r * ln, (const uint32_t*)smem, ln, b, K, s + lo, count - lo < K ? (int)(count - lo) : K);
    }
  }
};
struct PrepBody {
  const uint32_t* consts; int const_quads;
  const uint32_t* n; const uint32_t* thresh; int ln; const uint32_t* s; uint32_t* e_out; int32_t* flag; long batch;
  PAI_MEM void run(u4*, const CtaId& id) const {
    for (long g = (long)id.cta * id.nthr + id.tid; g < batch; g += (long)id.ncta * id.nthr) rawmul_prep(n, thresh, ln, s, e_out, flag, g);
  }
};
template <int NTP, int W>
struct DecBody {
  const uint32_t* consts; int const_quads;
  int nwin_p, nwin_q; const uint32_t* c; uint32_t* out; long batch; u4* tbl; unsigned long long* counter;
  const uint32_t* pre_p; const uint32_t* pre_q;      // c^(p-1) mod p^2, c^(q-1) mod q^2 already computed (pai_coop.cuh), or null
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    cta_decrypt<NTP, W>(smem, id, nwin_p, nwin_q, c, out, batch, tbl, counter, pre_p, pre_q);
  }
};
template <int NTP, int W>
struct DecDigitBody {
  const uint32_t* consts; int const_quads;
  int nwin_p, nwin_q; const uint32_t* c; uint32_t* out; long batch; u4* tbl; unsigned long long* counter;
  PAI_MEM void run(u4* smem, const CtaId& id) const { cta_decrypt_digit<NTP, W>(smem, id, nwin_p, nwin_q, c, out, batch, tbl, counter); }
};
template <int NTP, int W>
struct PrivEncDigitBody {
  const uint32_t* consts; int const_quads;
  int nwin_p, nwin_q; const uint32_t* m; const uint32_t* r;
  const uint32_t* pre_p; const uint32_t* pre_q;      // r^n mod p^2, r^n mod q^2 already computed (warp kernels), or null
  uint32_t* out; long batch; u4* tbl;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    cta_priv_encrypt_digit<NTP, W>(smem, id, nwin_p, nwin_q, m, r, pre_p, pre_q, out, batch, tbl);
  }
};
// one CRT half with h = 1 (used once per key to derive hp / hq): out = L(g^(x-1) mod x^2) mod x
template <int NTP, int W>
struct LBody {
  const uint32_t* consts; int const_quads;   // one side: [ blob(x^2) | blob(x) | xinv | hM | e ]
  int nwin; const uint32_t* c; uint32_t* out; u4* tbl;
  PAI_MEM void run(u4* smem, const CtaId& id) const {
    if (id.cta != 0 || id.tid != 0) return;
    SideC<NTP> S;
    side_bind<NTP>(S, smem, nwin);
    PowEnv<2 * NTP> E;
    cta_bufs<2 * NTP>(E.buf, 3, smem, side_quads<NTP>(), id);
    E.tbl = cta_table<2 * NTP, W>(tbl, id);
    E.mc = &S.sq;
    int r = decrypt_half<NTP, W>(E, S, c);
    store_row(out, E.buf[r], 2 * NTP);
  }
};

}  // namespace
#if !defined(PAI_HOSTSIM)
// tensor-core kernels of digit moduli with at most 4 tiles (128 base-256 digits: 2048-bit-key decrypt, 1024-bit-key encrypt)
// keep 3 x 128 bytes per thread in shared memory, so FOUR 128-thread groups fit an SM:
// 16 warps instead of 8 to keep the integer pipe busy while other groups wait for their GEMMs -- at 128 registers a thread
namespace pai {
template <int W> struct BodyMaxThreads<TcDecBody<2, W>> { static const int v = 512; };
template <int W> struct BodyMaxThreads<TcDecBody<4, W>> { static const int v = 512; };
template <> struct BodyMaxThreads<TcEncBody<2>> { static const int v = 512; };
template <> struct BodyMaxThreads<TcEncBody<4>> { static const int v = 512; };
template <int W> struct BodyMaxThreads<TcPowBody<2, W>> { static const int v = 512; };
template <int W> struct BodyMaxThreads<TcPowBody<4, W>> { static const int v = 512; };
template <int W> struct BodyMaxThreads<TcStrausBody<2, W>> { static const int v = 512; };
template <int W> struct BodyMaxThreads<TcStrausBody<4, W>> { static const int v = 512; };
// 192 / 256 digits: THREE groups (384 threads, 168 registers) once the high digit x1 lives in the thread's table strip in
// L2 instead of shared memory
template <int W> struct BodyMaxThreads<TcDecBody<6, W>> { static const int v = 384; };
template <int W> struct BodyMaxThreads<TcDecBody<8, W>> { static const int v = 384; };
template <> struct BodyMaxThreads<TcEncBody<6>> { static const int v = 384; };
template <> struct BodyMaxThreads<TcEncBody<8>> { static const int v = 384; };
template <int W> struct BodyMaxThreads<TcPowBody<6, W>> { static const int v = 384; };
template <int W> struct BodyMaxThreads<TcPowBody<8, W>> { static const int v = 384; };
template <int W> struct BodyMaxThreads<TcStrausBody<6, W>> { static const int v = 384; };
template <int W> struct BodyMaxThreads<TcStrausBody<8, W>> { static const int v = 384; };
}  // namespace pai
#endif
namespace {
const int W_ENC = 6, W_DEC = 5, W_VAR = 4;   // W_ENC: sliding window (32 odd powers); W_DEC/W_VAR: fixed windows
#if defined(PAI_HOSTSIM)
const int NTHR_MAX = 2;      // the CPU simulation runs lanes one after the other: keep CTAs tiny
#else
const int NTHR_MAX = 256;
#endif

int pick_nt(int tiles_needed) {
  static const int sup[] = {1, 2, 3, 4, 6, 8, 12, 16, 24, 32};
  for (int v : sup) if (v >= tiles_needed) return v;
  return -1;
}
int pick_ntp(int tiles_needed) {
  static const int sup[] = {1, 2, 3, 4, 6, 8};
  for (int v : sup) if (v >= tiles_needed) return v;
  return -1;
}

// little host helpers on limb vectors (per-key setup only)
typedef std::vector<uint32_t> limbs_t;
int eff_limbs(const uint32_t* a, int n) { while (n > 0 && a[n - 1] == 0) n--; return n; }
int bit_length(const limbs_t& a) {
  int n = eff_limbs(a.data(), (int)a.size());
  if (!n) return 0;
  uint32_t v = a[n - 1]; int b = 0; while (v) { b++; v >>= 1; }
  return 32 * (n - 1) + b;
}
limbs_t h_mul(const limbs_t& a, const limbs_t& b) {
  limbs_t r(a.size() + b.size(), 0);
  for (size_t i = 0; i < a.size(); i++) {
    uint64_t c = 0;
    for (size_t j = 0; j < b.size(); j++) { uint64_t t = (uint64_t)a[i] * b[j] + r[i + j] + c; r[i + j] = (uint32_t)t; c = t >> 32; }
    r[i + b.size()] = (uint32_t)c;
  }
  return r;
}
limbs_t h_sub_small(const limbs_t& a, uint32_t s) {
  limbs_t r(a); uint64_t bo = s;
  for (size_t i = 0; i < r.size() && bo; i++) { uint64_t d = (uint64_t)r[i] - bo; r[i] = (uint32_t)d; bo = (d >> 63) & 1; }
  return r;
}
limbs_t h_add_small(const limbs_t& a, uint32_t s) {
  limbs_t r(a); uint64_t c = s;
  for (size_t i = 0; i < r.size() && c; i++) { uint64_t d = (uint64_t)r[i] + c; r[i] = (uint32_t)d; c = d >> 32; }
  return r;
}
limbs_t h_div_small(const limbs_t& a, uint32_t d) {
  limbs_t q(a.size(), 0); uint64_t rem = 0;
  for (int i = (int)a.size() - 1; i >= 0; i--) { uint64_t t = (rem << 32) | a[i]; q[i] = (uint32_t)(t / d); rem = t % d; }
  return q;
}
limbs_t h_sub(const limbs_t& a, const limbs_t& b) {
  limbs_t r(a.size()); uint64_t bo = 0;
  for (size_t i = 0; i < a.size(); i++) { uint64_t d = (uint64_t)a[i] - (i < b.size() ? b[i] : 0) - bo; r[i] = (uint32_t)d; bo = (d >> 63) & 1; }
  return r;
}
int h_cmp(const uint32_t* a, const uint32_t* b, int n) {
  for (int i = n - 1; i >= 0; i--) if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  return 0;
}
limbs_t padded(const uint32_t* a, int n, int total) {
  limbs_t r(total, 0);
  for (int i = 0; i < n && i < total; i++) r[i] = a[i];
  return r;
}
// a = quo * m + rem (m > 0) by binary long division with one masked subtraction per bit: the operands are key material
void h_divmod(const limbs_t& a, const limbs_t& m, limbs_t* quo, limbs_t* rem) {
  const size_t L = m.size() + 1;
  limbs_t r(L, 0), t(L, 0);
  if (quo) quo->assign(a.size(), 0);
  for (long i = 32 * (long)a.size() - 1; i >= 0; i--) {
    uint32_t c = (a[i >> 5] >> (i & 31)) & 1u;
    for (size_t j = 0; j < L; j++) { uint32_t v = r[j]; r[j] = (v << 1) | c; c = v >> 31; }
    uint64_t bo = 0;
    for (size_t j = 0; j < L; j++) { uint64_t d = (uint64_t)r[j] - (j < m.size() ? m[j] : 0u) - bo; t[j] = (uint32_t)d; bo = (d >> 63) & 1; }
    const uint32_t keep = 0u - (uint32_t)bo;                 // r < m: r stays
    for (size_t j = 0; j < L; j++) r[j] = (r[j] & keep) | (t[j] & ~keep);
    if (quo) (*quo)[i >> 5] |= (uint32_t)(1 - bo) << (i & 31);
  }
  if (rem) { *rem = r; rem->resize(m.size()); }
  std::fill(r.begin(), r.end(), 0);
  std::fill(t.begin(), t.end(), 0);
}
limbs_t h_mod(const limbs_t& a, const limbs_t& m) { limbs_t r; h_divmod(a, m, nullptr, &r); return r; }
limbs_t h_shl_limbs(const limbs_t& a, int k) { limbs_t r(k, 0); r.insert(r.end(), a.begin(), a.end()); return r; }

// Sliding-window program of a public exponent (see mont_pow_prog): left-to-right, windows of at most w
// bits that start and end on a 1 bit.  entry = (nsq << 16) | idx, idx = (window value - 1) / 2 or 0xffff.
std::vector<uint32_t> sliding_program(const limbs_t& e, int w) {
  std::vector<uint32_t> prog;
  int nbits = bit_length(e);
  auto bit = [&](int i) { return (e[i >> 5] >> (i & 31)) & 1u; };
  int i = nbits - 1;
  uint32_t pending = 0;                      // squarings owed before the next multiplication
  bool first = true;
  while (i >= 0) {
    if (!bit(i)) { pending++; i--; continue; }
    int l = std::min(w, i + 1);
    while (!bit(i - l + 1)) l--;             // window [i-l+1, i] ends on a 1
    uint32_t v = 0;
    for (int k = 0; k < l; k++) v = (v << 1) | bit(i - k);
    if (first) { prog.push_back((0u << 16) | ((v - 1) / 2)); first = false; }
    else {
      uint32_t nsq = pending + (uint32_t)l;
      while (nsq > 0xfff0u) { prog.push_back((0xfff0u << 16) | 0xffffu); nsq -= 0xfff0u; }
      prog.push_back((nsq << 16) | ((v - 1) / 2));
    }
    pending = 0;
    i -= l;
  }
  while (pending > 0) { uint32_t c = std::min(pending, 0xfff0u); prog.push_back((c << 16) | 0xffffu); pending -= c; }
  return prog;
}

// Device memory a context owns.  It knows its size, so a context holding key material can zero it before the free
// (`release(true)`: a memset and a sync on the current device, which the destroy functions set first).
template <class T = void>
struct DevBuf {
  T* p = nullptr; size_t bytes = 0;
  int ensure(size_t need) {
    if (need <= bytes) return 0;
    release();
    int rc = rt_malloc((void**)&p, need);
    if (rc) return rc;
    bytes = need;
    return 0;
  }
  void release(bool wipe = false) {
    if (wipe && p) { rt_memset(p, 0, bytes, 0); rt_sync(0); }
    rt_free(p); p = nullptr; bytes = 0;
  }
};
// a temporary device buffer, freed on every return path
struct TmpBuf {
  void* p = nullptr;
  TmpBuf() = default;
  TmpBuf(const TmpBuf&) = delete;
  TmpBuf& operator=(const TmpBuf&) = delete;
  ~TmpBuf() { rt_free(p); }
  int alloc(size_t bytes) { return rt_malloc(&p, bytes); }
  uint32_t* u32() const { return (uint32_t*)p; }
};

// work counters of the persistent kernels: a ring of zero-initialised 64-bit counters per (context, stream);
// each launch takes the next one and re-zeroes it on the launch stream first (launches on one stream are
// ordered, so a counter is never re-armed while a previous kernel on that stream still uses it).
struct Counters {
  DevBuf<> buf; int next = 0;
  int take(rt_stream s, unsigned long long** out) {
    int rc = buf.ensure(64 * 8);
    if (rc) return rc;
    unsigned long long* p = (unsigned long long*)buf.p + next;
    next = (next + 1) % 64;
    rc = rt_memset(p, 0, 8, s);
    *out = p;
    return rc;
  }
};

// Everything a launch borrows from its context while it runs: the window-table workspace, the work counters and the
// intermediate rows of multi-kernel operations.  One set per CUDA stream the context has been used on, so calls on
// different streams never share scratch memory (launches on ONE stream are ordered and may).  Looked up under the
// context's mutex; lives until the context is destroyed.
struct StreamWs {
  DevBuf<> tbl, w_base, w_exp, w_flag, coop_u, red_a, red_b, mv_tbl;
  Counters ctr;
  void release(bool wipe) {
    for (DevBuf<>* b : {&tbl, &w_base, &w_exp, &w_flag, &coop_u, &red_a, &red_b, &mv_tbl, &ctr.buf}) b->release(wipe);
  }
};
struct WsMap {
  std::map<rt_stream, StreamWs> m;
  StreamWs& get(rt_stream s) { return m[s]; }
  void release(bool wipe = false) { for (auto& kv : m) kv.second.release(wipe); m.clear(); }
};
typedef std::lock_guard<std::recursive_mutex> CtxLock;

// launch geometry for a body with `nbuf` operand buffers of NT tiles
struct Geom { int nthr, grid; size_t smem; };
template <class Body>
int geometry(int device, int NT, int const_quads, int nbuf, long batch, Geom& g) {
  size_t max_smem = rt_max_smem(device);
  int nthr = NTHR_MAX;
  size_t smem;
  for (;;) {
    smem = ((size_t)const_quads + (size_t)nbuf * 2 * NT * nthr) * 16;
    if (smem <= max_smem || nthr <= 32) break;
    nthr -= 32;   // (never reached in the simulation build)
  }
  if (smem > max_smem) { g_err = "operand size does not fit shared memory"; return PAI_E_ARG; }
  int occ = rt_occupancy<Body>(nthr, smem);
  if (occ <= 0) { g_err = "kernel cannot be resident (occupancy 0)"; return PAI_E_CUDA; }
  long chunks = (batch + nthr - 1) / nthr;
  long maxgrid = (long)rt_sm_count(device) * occ;
  g.nthr = nthr; g.smem = smem; g.grid = (int)std::max(1L, std::min(chunks, maxgrid));
  return 0;
}
long wave_rows(const Geom& g) { return (long)g.grid * g.nthr; }

// What a persistent kernel with a window table needs from its launcher, stated once per body: operand tiles, constant
// quads, operand buffers and table entries per thread (2 * tiles quads each)
struct Shape { int nt, cq, nbuf; long entries; };
// rows one full grid of B holds (0 when B cannot be resident)
template <class B>
long wave_of(int device, const Shape& sh) {
  Geom g;
  return geometry<B>(device, sh.nt, sh.cq, sh.nbuf, 1L << 40, g) ? 0 : wave_rows(g);
}
// geometry, the window-table workspace, a work counter and the launch of a persistent kernel B over `batch` rows;
// make(tbl, counter) builds the body
template <class B, class Make>
int launch_persistent(int device, StreamWs& w, const Shape& sh, long batch, rt_stream s, Make make) {
  Geom g;
  int rc = geometry<B>(device, sh.nt, sh.cq, sh.nbuf, batch, g);
  if (!rc) rc = w.tbl.ensure((size_t)g.grid * sh.entries * 2 * sh.nt * g.nthr * 16);
  unsigned long long* ctr = nullptr;
  if (!rc) rc = w.ctr.take(s, &ctr);
  if (rc) return rc;
  return rt_launch(make((u4*)w.tbl.p, ctr), g.grid, g.nthr, g.smem, s);
}
// a one-thread setup kernel (per key): `scratch_bytes` of device scratch, one 32-thread CTA, waited for; make(scratch)
// builds the body
template <class Make>
int run_setup(size_t scratch_bytes, rt_stream s, Make make) {
  TmpBuf scratch;
  int rc = scratch.alloc(scratch_bytes);
  if (!rc) rc = rt_launch(make(scratch.u32()), 1, 32, 0, s);
  if (!rc) rc = rt_sync(s);
  return rc;
}

}  // namespace

// kernel family of a context; the values are the codes pai_*_kernel_path returns
enum Family { FULL = 0, DIGIT = 1, TC = 2 };

// ------------------------------------------------------------------------------------------------
struct pai_mod {
  int device = 0, NT = 0, L = 0;
  DevBuf<uint32_t> d_blob;          // mc_limbs(NT) (+ extra room requested by the owner)
  limbs_t h_N;                      // padded modulus
  DevBuf<> tmp_a, tmp_b, tmp_o, tmp_s, tmp_e;   // staging of the host-pointer entry points (used under `mu`, stream 0)
  WsMap ws;                         // per-stream workspaces
  std::recursive_mutex mu;          // serialises host threads on this context (recursive: coop constants are built
                                    // through the context's own entry points)
  // warp-per-ciphertext layout (pai_coop.cuh), built on first use (then coopK != 0): [ N | R^2 mod N | R^3 mod N ],
  // R = 2^(32*32*coopK)
  DevBuf<uint32_t> d_coop; int coopK = 0; uint32_t coop_n0inv = 0; bool coop_building = false;
  DevBuf<uint32_t> d_corr;          // correction rows R^(2^i + 1) mod N of the product reduction (cta_reduce_mul), built on first use
};
struct pai_pub {
  pai_mod* nsq = nullptr;           // modulus n^2; its blob is followed by n (4*NT limbs) for encrypt
  int ln = 0;                       // limbs of n (= 4*NT)
  uint32_t* d_nth = nullptr;        // [ n | n - max_int ]  (ln limbs each) for raw_mul's branch test
  DevBuf<> h_m, h_r, h_c, h_s;      // staging of the host-pointer entry points (under `mu`)
  WsMap ws;                         // per-stream intermediates of raw_mul / reductions
  std::recursive_mutex mu;
  limbs_t h_n;
  uint32_t* d_prog = nullptr;       // sliding-window program of the exponent n (encrypt)
  int nops = 0, nodd = 0;
  pai_mod* nmod = nullptr;          // modulus n with the digit-form constants appended (pai_digit.cuh)
  uint32_t* d_enc_consts = nullptr; // compact constant area of the encrypt kernel (dc_enc_limbs)
  Family family = DIGIT;            // of encrypt and raw_mul (pick_family)
  uint8_t* d_tc = nullptr;          // family TC only: [ band(N') | band(n) ] (pai_tc.cuh)
  int tc_stagger = 0;               // family TC: start-up delay (cycles) of the second thread group
  long wave = 0;                    // ciphertexts per wave of the throughput encrypt kernel (lazily measured)
};
struct pai_priv {
  int device = 0, NTP = 0;
  pai_mod *p2 = nullptr, *q2 = nullptr, *p1 = nullptr, *q1 = nullptr;
  DevBuf<uint32_t> d_consts;        // [ P side | Q side | pinvqM ]  (full-width path, also used to derive hp/hq)
  pai_mod *pd = nullptr, *qd = nullptr;   // p, q with digit-form constants (pai_digit.cuh)
  DevBuf<uint32_t> d_dconsts;       // digit path: [ P: dblob(p) | hM | e ][ Q: ... ][ pinvqM ]
  Family family = DIGIT;            // of decrypt (pick_family)
  DevBuf<uint8_t> d_tc;             // family TC only: [ band(p') | band(p) | band(q') | band(q) ]
  int tc_stagger = 0;
  int nwin_p = 0, nwin_q = 0;
  limbs_t h_p, h_q, h_pinv, h_hp, h_hq;   // 16*NTP limbs each (padded)
  DevBuf<> h_c, h_m;                // staging of pai_decrypt_host (under `mu`)
  WsMap ws;                         // per-stream window tables, counters, warp-path intermediates
  std::recursive_mutex mu;
  long wave = 0;                    // ciphertexts per wave of the throughput decrypt kernel (lazily measured)
  DevBuf<uint32_t> d_coop_e;        // [ p - 1 | q - 1 ] (8*NTP limbs each) for the warp-per-ciphertext path
  // encryption with the private key (pai_priv_encrypt), built on its first call:
  DevBuf<uint32_t> d_pe_consts;     // pe_const_limbs<NTP>() limbs (pai_digit.cuh)
  DevBuf<uint32_t> d_pe_coop_e;     // [ n mod p(p-1) | n mod q(q-1) ] (16*NTP limbs each) for its warp-per-ciphertext route
  int pe_nwin_p = 0, pe_nwin_q = 0, pe_coop_nwin[2] = {0, 0};
  long pe_wave = 0;                 // rows per wave of its throughput kernel (routing only)
  DevBuf<> h_r;                     // staging of pai_priv_encrypt_host (with h_m and h_c, under `mu`)
};

// ------------------------------------------------------------------------------------------------
#define DISPATCH_K(KV, CALL)                                                                          \
  switch (KV) {                                                                                       \
    case 1: { constexpr int K = 1; CALL; } break;                                                     \
    case 2: { constexpr int K = 2; CALL; } break;                                                     \
    case 3: { constexpr int K = 3; CALL; } break;                                                     \
    case 4: { constexpr int K = 4; CALL; } break;                                                     \
    case 6: { constexpr int K = 6; CALL; } break;                                                     \
    case 8: { constexpr int K = 8; CALL; } break;                                                     \
    default: g_err = "unsupported operand size"; rc = PAI_E_ARG;                                      \
  }
#define DISPATCH_NT(NTV, CALL)                                                                        \
  switch (NTV) {                                                                                      \
    case 1: { constexpr int NT = 1; CALL; } break;                                                    \
    case 2: { constexpr int NT = 2; CALL; } break;                                                    \
    case 3: { constexpr int NT = 3; CALL; } break;                                                    \
    case 4: { constexpr int NT = 4; CALL; } break;                                                    \
    case 6: { constexpr int NT = 6; CALL; } break;                                                    \
    case 8: { constexpr int NT = 8; CALL; } break;                                                    \
    case 12: { constexpr int NT = 12; CALL; } break;                                                  \
    case 16: { constexpr int NT = 16; CALL; } break;                                                  \
    case 24: { constexpr int NT = 24; CALL; } break;                                                  \
    case 32: { constexpr int NT = 32; CALL; } break;                                                  \
    default: g_err = "unsupported operand size"; rc = PAI_E_ARG;                                      \
  }
#define DISPATCH_NTP(NTV, CALL)                                                                       \
  switch (NTV) {                                                                                      \
    case 1: { constexpr int NTP = 1; CALL; } break;                                                   \
    case 2: { constexpr int NTP = 2; CALL; } break;                                                   \
    case 3: { constexpr int NTP = 3; CALL; } break;                                                   \
    case 4: { constexpr int NTP = 4; CALL; } break;                                                   \
    case 6: { constexpr int NTP = 6; CALL; } break;                                                   \
    case 8: { constexpr int NTP = 8; CALL; } break;                                                   \
    default: g_err = "unsupported key size"; rc = PAI_E_ARG;                                          \
  }

#define DISPATCH_NTH(NTV, CALL)                                                                       \
  switch (NTV) {                                                                                      \
    case 2: { constexpr int NTH = 2; CALL; } break;                                                   \
    case 4: { constexpr int NTH = 4; CALL; } break;                                                   \
    case 6: { constexpr int NTH = 6; CALL; } break;                                                   \
    case 8: { constexpr int NTH = 8; CALL; } break;                                                   \
    case 12: { constexpr int NTH = 12; CALL; } break;                                                 \
    case 16: { constexpr int NTH = 16; CALL; } break;                                                 \
    default: g_err = "unsupported key size"; rc = PAI_E_ARG;                                          \
  }

#define DISPATCH_TC(NTV, CALL)                                                                        \
  switch (NTV) {                                                                                      \
    case 2: { constexpr int NTH = 2; CALL; } break;                                                   \
    case 4: { constexpr int NTH = 4; CALL; } break;                                                   \
    case 6: { constexpr int NTH = 6; CALL; } break;                                                   \
    case 8: { constexpr int NTH = 8; CALL; } break;                                                   \
    case 12: { constexpr int NTH = 12; CALL; } break;                                                 \
    default: g_err = "key size not supported by the tensor-core path"; rc = PAI_E_ARG;                \
  }

namespace {

// tile counts the tensor-core kernels are instantiated for (DISPATCH_TC), up to `max_tiles`
bool tc_supported(int tiles, int max_tiles) { return (tiles == 2 || tiles == 4 || tiles == 6 || tiles == 8 || tiles == 12) && tiles <= max_tiles; }
// `path_var`=full (PAI_ENCRYPT_PATH / PAI_DECRYPT_PATH) selects the full-width Montgomery kernels; otherwise PAI_TC=2
// selects the tensor-core kernels where they cover the key (`tc_ok`).  By default the integer-pipe digit kernels run,
// which measure faster on the H100 at every key size both families cover (DESIGN.md section 4).
Family pick_family(const char* path_var, bool tc_ok) {
  const char* e = getenv(path_var);
  if (e && std::string(e) == "full") return FULL;
  const char* tc = getenv("PAI_TC");
  return tc_ok && tc && std::string(tc) == "2" ? TC : DIGIT;
}
// start-up delay (cycles) of the second thread group of the tensor-core kernels
int tc_stagger_cycles() {
  const char* st = getenv("PAI_TC_STAGGER");
  return st && *st ? atoi(st) : 40000;
}

template <int NT>
int do_setup(pai_mod* m, rt_stream s) {
  return run_setup((size_t)3 * 8 * NT * 4, s, [&](uint32_t* scratch) { return SetupBody<NT>{nullptr, 0, m->d_blob.p, scratch}; });
}

// create a modulus context; extra_limbs of device room are left after the blob
int mod_create_impl(const uint32_t* modulus, int limbs, int device, int force_nt, int extra_limbs, pai_mod** out) {
  if (!modulus || !out || limbs <= 0) { g_err = "null/empty modulus"; return PAI_E_ARG; }
  int eff = eff_limbs(modulus, limbs);
  if (eff == 0 || !(modulus[0] & 1u)) { g_err = "modulus must be odd and non-zero"; return PAI_E_ARG; }
  if (eff == 1 && modulus[0] == 1u) { g_err = "modulus must be > 1"; return PAI_E_ARG; }
  int NT = force_nt > 0 ? force_nt : pick_nt((eff + 7) / 8);
  if (NT < 0 || 8 * NT < eff) { g_err = "modulus too large (max 8192 bits)"; return PAI_E_ARG; }
  if (rt_device_count() <= device) { g_err = "no such CUDA device (this engine has no CPU fallback)"; return PAI_E_CUDA; }
  int rc = rt_set_device(device);
  if (rc) return rc;
  pai_mod* m = new (std::nothrow) pai_mod();
  if (!m) return PAI_E_ARG;
  m->device = device; m->NT = NT; m->L = 8 * NT;
  m->h_N = padded(modulus, eff, m->L);
  rc = m->d_blob.ensure(((size_t)mc_limbs(NT) + extra_limbs) * 4);
  if (!rc) rc = rt_memset(m->d_blob.p, 0, m->d_blob.bytes, 0);
  if (!rc) rc = rt_h2d(m->d_blob.p, m->h_N.data(), (size_t)m->L * 4, 0);
  if (!rc) { DISPATCH_NT(NT, rc = do_setup<NT>(m, 0)); }
  if (rc) { m->d_blob.release(); delete m; return rc; }
  *out = m;
  return 0;
}
// `wipe`: the modulus is part of a private key -- zero every buffer before it is freed, and the host copy of the modulus.
// The coop constants are zeroed in any case.
void mod_free(pai_mod* m, bool wipe) {
  if (!m) return;
  rt_set_device(m->device);
  m->d_blob.release(wipe);
  m->d_corr.release(wipe);
  m->d_coop.release(true);
  m->ws.release(wipe);
  for (DevBuf<>* b : {&m->tmp_a, &m->tmp_b, &m->tmp_o, &m->tmp_s, &m->tmp_e}) b->release(wipe);
  if (wipe) std::fill(m->h_N.begin(), m->h_N.end(), 0);
  delete m;
}

template <int NT>
int do_mulmod(pai_mod* m, const uint32_t* consts, int cq, const uint32_t* a, const uint32_t* b, uint32_t* out, long batch, rt_stream s) {
  typedef MulBody<NT> B;
  Geom g;
  int rc = geometry<B>(m->device, NT, cq, 3, batch, g);
  if (rc) return rc;
  B body{consts, cq, a, b, out, batch};
  return rt_launch(body, g.grid, g.nthr, g.smem, s);
}

template <int NT>
int do_powmod(pai_mod* m, const uint32_t* base, int base_tiles, const uint32_t* d_exp, int exp_limbs, long exp_stride,
              int nwin_fixed, uint32_t* out, long batch, rt_stream s) {
  const Shape sh{NT, mc_limbs(NT) / 4, 3, 1 << W_VAR};
  return launch_persistent<PowBody<NT, W_VAR>>(m->device, m->ws.get(s), sh, batch, s, [&](u4* tbl, unsigned long long* ctr) {
    return PowBody<NT, W_VAR>{m->d_blob.p, sh.cq, base, base_tiles, d_exp, exp_limbs, exp_stride, nwin_fixed, out, batch, tbl, ctr};
  });
}

// product of `batch` rows modulo N -> one canonical row (two launches: per-CTA partial products, then their product
// together with the correction rows; one launch when a single CTA covers the batch)
const int REDUCE_CORR_ROWS = 44;
template <int NT>
int do_reduce_mul(pai_mod* m, const uint32_t* rows, long batch, uint32_t* out, rt_stream s) {
  typedef ReduceBody<NT> B;
  Geom g;
  const int cq = mc_limbs(NT) / 4;
  int rc = geometry<B>(m->device, NT, cq, 3, batch, g);
  if (rc) return rc;
  if (!m->d_corr.p) {                                 // per-modulus table R^(2^i + 1), built on first use
    rc = m->d_corr.ensure((size_t)REDUCE_CORR_ROWS * m->L * 4);
    if (rc) return rc;
    ReduceCorrBody<NT> cb{m->d_blob.p, cq, m->d_corr.p, REDUCE_CORR_ROWS};
    rc = rt_launch(cb, 1, g.nthr, g.smem, s);
    if (!rc) rc = rt_sync(s);
    if (rc) { m->d_corr.release(); return rc; }
  }
  const unsigned long long bits = (unsigned long long)batch;
  if (g.grid == 1) {
    B body{m->d_blob.p, cq, rows, batch, out, m->d_corr.p, bits, 1};
    return rt_launch(body, 1, g.nthr, g.smem, s);
  }
  StreamWs& w = m->ws.get(s);
  rc = w.red_a.ensure((size_t)g.grid * m->L * 4);
  if (rc) return rc;
  B first{m->d_blob.p, cq, rows, batch, (uint32_t*)w.red_a.p, m->d_corr.p, 0ull, 0};
  rc = rt_launch(first, g.grid, g.nthr, g.smem, s);
  if (rc) return rc;
  B second{m->d_blob.p, cq, (const uint32_t*)w.red_a.p, (long)g.grid, out, m->d_corr.p, bits, 1};
  return rt_launch(second, 1, g.nthr, g.smem, s);
}

template <int NT>
int do_invert(pai_mod* m, const uint32_t* a, int a_tiles, const int32_t* flags, uint32_t* out, int32_t* status, long batch, rt_stream s) {
  typedef InvBody<NT> B;
  Geom g;
  int cq = mc_limbs(NT) / 4;
  int rc = geometry<B>(m->device, NT, cq, 4, batch, g);
  if (rc) return rc;
  B body{m->d_blob.p, cq, a, a_tiles, flags, out, status, batch};
  return rt_launch(body, g.grid, g.nthr, g.smem, s);
}

// flagged rows inverted with one extended gcd per segment of rows (cta_invert_batch); unflagged rows copied
template <int NT>
int do_invert_flagged(pai_mod* m, const uint32_t* a, const int32_t* flags, uint32_t* out, int32_t* status, long batch, rt_stream s) {
  typedef InvBatchBody<NT> B;
  Geom g;
  int cq = mc_limbs(NT) / 4;
  int rc = geometry<B>(m->device, NT, cq, 4, 1L << 40, g);                 // full grid
  if (rc) return rc;
  const long T = (long)g.grid * g.nthr;
  long seg = (batch + T - 1) / T;                                          // rows per thread when the whole grid is busy
  if (seg < 1) seg = 1;
  if (seg > 32) seg = 32;
  const long nseg = (batch + seg - 1) / seg;
  g.grid = (int)std::max(1L, std::min((long)g.grid, (nseg + g.nthr - 1) / g.nthr));
  B body{m->d_blob.p, cq, a, flags, out, status, batch, (int)seg};
  return rt_launch(body, g.grid, g.nthr, g.smem, s);
}

template <int NT>
Shape enc_shape(const pai_pub* k) { return {NT, mc_limbs(NT) / 4 + NT, 2, k->nodd + 1}; }
template <int NT>
int do_encrypt(pai_pub* k, const uint32_t* m_, const uint32_t* r, uint32_t* c, long batch, rt_stream s) {
  pai_mod* m = k->nsq;
  const Shape sh = enc_shape<NT>(k);
  return launch_persistent<EncBody<NT>>(m->device, m->ws.get(s), sh, batch, s, [&](u4* tbl, unsigned long long* ctr) {
    return EncBody<NT>{m->d_blob.p, sh.cq, k->d_prog, k->nops, k->nodd, m_, r, c, batch, tbl, ctr};
  });
}

template <int NTH>
int do_digit_setup(pai_mod* m, rt_stream s) {
  return run_setup((size_t)4 * 8 * NTH * 4, s, [&](uint32_t* scratch) { return DigitSetupBody<NTH>{nullptr, 0, m->d_blob.p, scratch}; });
}

template <int NTH>
Shape enc_digit_shape(const pai_pub* k) { return {2 * NTH, dc_enc_limbs(NTH) / 4, 2, k->nodd + 1}; }
template <int NTH>
int do_encrypt_digit(pai_pub* k, const uint32_t* m_, const uint32_t* r, uint32_t* c, long batch, rt_stream s) {
  pai_mod* m = k->nmod;
  const Shape sh = enc_digit_shape<NTH>(k);
  return launch_persistent<EncDigitBody<NTH>>(m->device, m->ws.get(s), sh, batch, s, [&](u4* tbl, unsigned long long* ctr) {
    return EncDigitBody<NTH>{k->d_enc_consts, sh.cq, k->d_prog, k->nops, k->nodd, m_, r, c, batch, tbl, ctr, m->d_blob.p + dc_zero_offset(NTH)};
  });
}

// launch geometry of a tensor-core kernel: as many 128-thread groups per CTA as the body's register budget
// (BodyMaxThreads) and shared memory (tc_x1_global decides where the high digit lives) allow.
// PAI_TC_GROUPS=<n> caps the group count (experiments).
template <class B, int NTH, class SmemFn>
int tc_geometry_of(int device, SmemFn smem_bytes, long batch, Geom& g) {
#if defined(PAI_HOSTSIM)
  g.nthr = TC_RL;
  g.smem = smem_bytes(TC_M);
  long chunks = (batch + g.nthr - 1) / g.nthr;
  g.grid = (int)std::max(1L, std::min(chunks, 3L));
  (void)device;
  return 0;
#else
  const size_t max_smem = rt_max_smem(device);
  const char* eg = getenv("PAI_TC_GROUPS");
  const int want_groups = eg && *eg ? atoi(eg) : 0;
  for (int groups = 4; groups >= 1; groups--) {
    const int nthr = groups * TC_M;
    if (nthr > BodyMaxThreads<B>::v || (want_groups && groups > want_groups)) continue;
    size_t smem = smem_bytes(nthr);
    if (smem + 128 > max_smem) continue;
    int occ = rt_occupancy<B>(nthr, smem);
    if (occ <= 0) continue;
    const long slots = (long)rt_sm_count(device) * occ;
    int use = groups;
    // less than one wave of rows (a small batch, or the tail the callers split off): the fewest groups per CTA that still
    // hold it in one wave -- a group sharing its SM with fewer others runs faster, and more SMs are busy
    if (!want_groups) while (use > 1 && (long)(use - 1) * TC_M * slots >= batch) use--;
    g.nthr = use * TC_M;
    g.smem = smem_bytes(g.nthr);
    long chunks = (batch + g.nthr - 1) / g.nthr;
    g.grid = (int)std::max(1L, std::min(chunks, slots));
    return 0;
  }
  g_err = "tensor-core kernel cannot be resident";
  return PAI_E_CUDA;
#endif
}
// The tensor-core kernels run whole waves in one launch and a tail of less than a wave in a second launch with a
// geometry of its own (tc_geometry_of).  launch(off, rows) runs rows [off, off + rows).
template <class Launch>
int tc_split(long wave, long batch, Launch launch) {
  if (batch <= wave || batch % wave == 0) return launch(0L, batch);
  const long head = batch - batch % wave;
  int rc = launch(0L, head);
  return rc ? rc : launch(head, batch - head);
}
// geometry (tc_geometry_of), the window-table workspace and the launch of a tensor-core kernel B over `batch` rows, with
// `entries` table entries of 4 * NTH quads per thread; make(tbl) builds the body
template <class B, int NTH, class SmemFn, class Make>
int launch_tc(int device, StreamWs& w, SmemFn smem_bytes, long entries, long batch, rt_stream s, Make make) {
  Geom g;
  int rc = tc_geometry_of<B, NTH>(device, smem_bytes, batch, g);
  if (!rc) rc = w.tbl.ensure((size_t)g.grid * entries * 4 * NTH * g.nthr * 16);
  if (rc) return rc;
  return rt_launch_group(make((u4*)w.tbl.p), g.grid, g.nthr, g.smem, s);
}
// rows one full grid of the tensor-core kernel B holds (0 when B cannot be resident)
template <class B, int NTH>
long tc_wave(int device, size_t (*smem_bytes)(int)) {
  Geom g;
  return tc_geometry_of<B, NTH>(device, smem_bytes, 1L << 40, g) ? 0 : wave_rows(g);
}
template <int NTH>
int do_encrypt_tc(pai_pub* k, const uint32_t* m_, const uint32_t* r, uint32_t* c, long batch, rt_stream s) {
  typedef TcEncBody<NTH> B;
  pai_mod* m = k->nmod;
  Geom g;
  int rc = tc_geometry_of<B, NTH>(m->device, tc_enc_smem_bytes<NTH>, batch, g);
  if (rc) return rc;
  rc = m->ws.get(s).tbl.ensure((size_t)g.grid * (size_t)(k->nodd + 4) * 4 * NTH * g.nthr * 16);
  if (rc) return rc;
  B body{k->d_enc_consts, dc_enc_limbs(NTH) / 4, k->d_prog, k->nops, k->nodd, m_, r, c, batch, (u4*)m->ws.get(s).tbl.p,
         m->d_blob.p + dc_zero_offset(NTH), k->d_tc, k->tc_stagger, nullptr};
#if !defined(PAI_HOSTSIM)
  // development aid: PAI_TC_PROF=<file> dumps per-warp cycle counters of the phases of tc_op after a synchronous launch
  if (const char* pf = getenv("PAI_TC_PROF")) {
    const size_t nw = (size_t)g.grid * (g.nthr / 32), bytes = nw * 16 * sizeof(long long);
    void* d = nullptr;
    rc = rt_malloc(&d, bytes);
    if (!rc) rc = rt_memset(d, 0, bytes, s);
    body.prof = (long long*)d;
    if (!rc) rc = rt_launch_group(body, g.grid, g.nthr, g.smem, s);
    std::vector<long long> h(nw * 16);
    if (!rc) rc = rt_d2h(h.data(), d, bytes, s);
    if (!rc) rc = rt_sync(s);
    if (!rc) if (FILE* f = fopen(pf, "w")) {
      for (size_t w = 0; w < nw; w++) { for (int i = 0; i < 16; i++) fprintf(f, "%lld ", h[w * 16 + i]); fprintf(f, "\n"); }
      fclose(f);
    }
    rt_free(d);
    return rc;
  }
#endif
  return rt_launch_group(body, g.grid, g.nthr, g.smem, s);
}
template <int NTH>
int do_powmod_tc(pai_pub* k, const uint32_t* base, const uint32_t* d_exp, int exp_limbs, uint32_t* out, long batch, rt_stream s) {
  typedef TcPowBody<NTH, W_VAR> B;
  pai_mod* m = k->nmod;
  return launch_tc<B, NTH>(m->device, m->ws.get(s), tc_pow_smem_bytes<NTH>, (1 << W_VAR) + 3, batch, s, [&](u4* tbl) {
    return B{k->d_enc_consts, dc_pow_limbs(NTH) / 4, base, d_exp, exp_limbs, out, batch, tbl, m->d_blob.p + dc_zero_offset(NTH), k->d_tc, k->tc_stagger};
  });
}
// Straus groups: one thread per group of gsz elements; gsz is chosen so that the groups fill about one wave
template <int NTH>
int do_straus_tc(pai_pub* k, const uint32_t* base, const uint32_t* d_exp, int exp_limbs, long batch, uint32_t* partial, long* ngroups_out,
                 rt_stream s) {
  typedef TcStrausBody<NTH, W_VAR> B;
  pai_mod* m = k->nmod;
  Geom g;
  int rc = tc_geometry_of<B, NTH>(m->device, tc_pow_smem_bytes<NTH>, 1L << 40, g);
  if (rc) return rc;
  const long wave = (long)g.grid * g.nthr;
  long gsz = (batch + wave - 1) / wave;
  if (gsz < 1) gsz = 1;
  if (gsz > 32) gsz = 32;
  const long ngroups = (batch + gsz - 1) / gsz;
  *ngroups_out = ngroups;
  return launch_tc<B, NTH>(m->device, m->ws.get(s), tc_pow_smem_bytes<NTH>, (gsz << W_VAR) + 4, ngroups, s, [&](u4* tbl) {
    return B{k->d_enc_consts, dc_pow_limbs(NTH) / 4, base, d_exp, exp_limbs, (int)gsz, partial, batch, tbl, m->d_blob.p + dc_zero_offset(NTH), k->d_tc, k->tc_stagger};
  });
}
template <int NTH>
int do_tc_setup(pai_pub* k, rt_stream s) {
  int rc = rt_malloc((void**)&k->d_tc, (size_t)tc_blob_bytes(NTH));
  if (rc) return rc;
  return run_setup((size_t)8 * NTH * 4, s, [&](uint32_t* scratch) { return TcSetupBody<NTH>{nullptr, 0, k->nmod->d_blob.p, k->d_tc, scratch}; });
}

template <int NTH>
int do_powmod_digit(pai_pub* k, const uint32_t* base, const uint32_t* d_exp, int exp_limbs, uint32_t* out, long batch, rt_stream s) {
  pai_mod* m = k->nmod;
  const Shape sh{2 * NTH, dc_pow_limbs(NTH) / 4, 2, 1 << W_VAR};
  return launch_persistent<PowDigitBody<NTH, W_VAR>>(m->device, m->ws.get(s), sh, batch, s, [&](u4* tbl, unsigned long long* ctr) {
    return PowDigitBody<NTH, W_VAR>{k->d_enc_consts, sh.cq, base, d_exp, exp_limbs, out, batch, tbl, ctr, m->d_blob.p + dc_zero_offset(NTH)};
  });
}

// Window width of the matrix-vector product: the w in 1..8 with the fewest modular multiplications,
//   tabled * (2^w - 2)  +  nrows * bits  +  nnz * ceil(bits / w)       (tables, squarings, products)
// among the widths whose tables fit MATVEC_TABLE_BUDGET.  w = 1 needs no table products (a table entry is the base
// itself, the size of the vector), so it is taken when nothing wider fits: the columns are never split into blocks.
#if defined(PAI_HOSTSIM)
const size_t MATVEC_TABLE_BUDGET = (size_t)64 << 10;       // the CPU simulation reaches w = 1 at small shapes
#else
const size_t MATVEC_TABLE_BUDGET = (size_t)2 << 30;
#endif
int matvec_window(long tabled, long nrows, long nnz, int bits, size_t entry_bytes) {
  int best = 1;
  double best_cost = 0;
  for (int w = 1; w <= 8; w++) {
    if (w > 1 && (double)tabled * ((1 << w) - 1) * (double)entry_bytes > (double)MATVEC_TABLE_BUDGET) break;
    const double cost = (double)tabled * ((1 << w) - 2) + (double)nrows * bits + (double)nnz * ((bits + w - 1) / w);
    if (w == 1 || cost < best_cost) { best = w; best_cost = cost; }
  }
  return best;
}
size_t matvec_entry_bytes(int NTH) { return (size_t)4 * NTH * 16; }

template <int NTH>
int do_matvec_digit(pai_pub* k, StreamWs& w, const uint32_t* c, const uint32_t* cinv, const int32_t* flag, long ncols,
                    long nslots, int win, const int64_t* indptr, const int32_t* indices, const uint32_t* mag, int ml,
                    const uint8_t* neg, long nnz, long nrows, uint32_t* out, rt_stream s) {
  pai_mod* m = k->nmod;
  const int cq = dc_pow_limbs(NTH) / 4;
  const uint32_t* gzero = m->d_blob.p + dc_zero_offset(NTH);
  int rc = 0;
  if (nnz > 0) {
    typedef MatTblBody<NTH> TB;
    Geom g;
    rc = geometry<TB>(m->device, 2 * NTH, cq, 2, nslots, g);
    if (!rc) rc = w.mv_tbl.ensure((size_t)nslots * ((1u << win) - 1u) * matvec_entry_bytes(NTH));
    if (rc) return rc;
    TB tb{k->d_enc_consts, cq, c, cinv, flag, ncols, nslots, win, (u4*)w.mv_tbl.p, gzero};
    rc = rt_launch(tb, g.grid, g.nthr, g.smem, s);
    if (rc) return rc;
  }
  return launch_persistent<MatRowBody<NTH>>(m->device, w, {2 * NTH, cq, 2, 0}, nrows, s, [&](u4*, unsigned long long* ctr) {
    return MatRowBody<NTH>{k->d_enc_consts, cq, (const u4*)w.mv_tbl.p, ncols, win, indptr, indices, mag, ml, neg, out, nrows, ctr, gzero};
  });
}

// constant quads of one CRT side of the full-width decrypt: [ blob(x^2) | blob(x) | xinv | hM | e ]
int side_quads_of(int NTP) { return mc_limbs(2 * NTP) / 4 + mc_limbs(NTP) / 4 + 6 * NTP; }
// constant quads of the digit and tensor-core decrypt: [ P: dblob(p) | hM | e ][ Q: ... ][ pinvqM ]
template <int NTP>
int dconst_quads() { return 2 * (dside_limbs<NTP>() / 4) + 2 * NTP; }

template <int NTP>
Shape dec_shape() { return {2 * NTP, 2 * side_quads_of(NTP) + 2 * NTP, 3, 1 << W_DEC}; }
template <int NTP>
int do_decrypt(pai_priv* k, const uint32_t* c, uint32_t* out, long batch, rt_stream s, const uint32_t* pre_p = nullptr,
               const uint32_t* pre_q = nullptr) {
  const Shape sh = dec_shape<NTP>();
  return launch_persistent<DecBody<NTP, W_DEC>>(k->device, k->ws.get(s), sh, batch, s, [&](u4* tbl, unsigned long long* ctr) {
    return DecBody<NTP, W_DEC>{k->d_consts.p, sh.cq, k->nwin_p, k->nwin_q, c, out, batch, tbl, ctr, pre_p, pre_q};
  });
}

template <int NTP>
Shape dec_digit_shape() { return {2 * NTP, dconst_quads<NTP>(), 2, 1 << W_DEC}; }
template <int NTP>
int do_decrypt_digit(pai_priv* k, const uint32_t* c, uint32_t* out, long batch, rt_stream s) {
  const Shape sh = dec_digit_shape<NTP>();
  return launch_persistent<DecDigitBody<NTP, W_DEC>>(k->device, k->ws.get(s), sh, batch, s, [&](u4* tbl, unsigned long long* ctr) {
    return DecDigitBody<NTP, W_DEC>{k->d_dconsts.p, sh.cq, k->nwin_p, k->nwin_q, c, out, batch, tbl, ctr};
  });
}

template <int NTP>
int do_decrypt_tc(pai_priv* k, const uint32_t* c, uint32_t* out, long batch, rt_stream s) {
  typedef TcDecBody<NTP, W_DEC> B;
  return launch_tc<B, NTP>(k->device, k->ws.get(s), tc_dec_smem_bytes<NTP>, (1 << W_DEC) + 3, batch, s, [&](u4* tbl) {
    return B{k->d_dconsts.p, dconst_quads<NTP>(), k->nwin_p, k->nwin_q, c, out, batch, tbl, k->d_tc.p, k->tc_stagger};
  });
}
template <int NTP>
int do_priv_tc_setup(pai_priv* k, rt_stream s) {
  int rc = k->d_tc.ensure((size_t)2 * tc_blob_bytes(NTP));
  pai_mod* md[2] = {k->pd, k->qd};
  for (int i = 0; i < 2 && !rc; i++) {
    rc = run_setup((size_t)8 * NTP * 4, s, [&](uint32_t* scratch) {
      return TcSetupBody<NTP>{nullptr, 0, md[i]->d_blob.p, k->d_tc.p + (size_t)i * tc_blob_bytes(NTP), scratch};
    });
  }
  return rc;
}

// digit-form constants of the private key, assembled from the digit blobs of p and q and from the
// h / exponent / p^-1 constants the full-width setup has already derived.
template <int NTP>
int do_priv_digit_setup(pai_priv* k, rt_stream s) {
  const int L1 = 8 * NTP;
  int rc = mod_create_impl(k->h_p.data(), L1, k->device, NTP, dc_extra_limbs(NTP), &k->pd);
  if (!rc) rc = mod_create_impl(k->h_q.data(), L1, k->device, NTP, dc_extra_limbs(NTP), &k->qd);
  if (!rc) rc = do_digit_setup<NTP>(k->pd, s);
  if (!rc) rc = do_digit_setup<NTP>(k->qd, s);
  if (!rc) rc = k->d_dconsts.ensure((size_t)dconst_quads<NTP>() * 16);
  if (rc) return rc;
  const int side = dside_limbs<NTP>();
  const int old_side = 4 * side_quads_of(NTP);                          // [ blob(x^2) | blob(x) | xinv | hM | e ]
  const int old_hM = mc_limbs(2 * NTP) + mc_limbs(NTP) + L1;
  pai_mod* md[2] = {k->pd, k->qd};
  for (int i = 0; i < 2 && !rc; i++) {
    uint32_t* dst = k->d_dconsts.p + (size_t)i * side;
    const uint32_t* old = k->d_consts.p + (size_t)i * old_side;
    rc = rt_d2d(dst, md[i]->d_blob.p, (size_t)dc_limbs(NTP) * 4, s);
    if (!rc) rc = rt_d2d(dst + dc_limbs(NTP), old + old_hM, (size_t)2 * L1 * 4, s);      // hM | e
  }
  if (!rc) rc = rt_d2d(k->d_dconsts.p + (size_t)2 * side, k->d_consts.p + (size_t)2 * old_side, (size_t)L1 * 4, s);   // pinvqM
  if (!rc) rc = rt_sync(s);
  return rc;
}

// ---- encryption with the private key
template <int NTP>
Shape priv_enc_shape() { return {2 * NTP, pe_const_limbs<NTP>() / 4, 2, pe_slots(W_DEC)}; }
template <int NTP>
int do_priv_encrypt_digit(pai_priv* k, const uint32_t* m, const uint32_t* r, uint32_t* c, long batch, rt_stream s,
                          const uint32_t* pre_p, const uint32_t* pre_q) {
  typedef PrivEncDigitBody<NTP, W_DEC> B;
  const Shape sh = priv_enc_shape<NTP>();
  return launch_persistent<B>(k->device, k->ws.get(s), sh, batch, s, [&](u4* tbl, unsigned long long*) {
    return B{k->d_pe_consts.p, sh.cq, k->pe_nwin_p, k->pe_nwin_q, m, r, pre_p, pre_q, c, batch, tbl};
  });
}
// The constants of pai_priv_encrypt (pai_digit.cuh), derived on the host from p, q and p^-1 mod q and uploaded once; the
// digit blobs of p and q are copied from pd / qd.
// Host scratch for the key-derived values: every result of a helper is moved into it (never copied, never dropped as a
// temporary), so each intermediate of the derivation lives in exactly one buffer, and every buffer is zeroed on exit.
// (h_divmod zeroes its own working rows.)
struct KeyScratch {
  std::deque<limbs_t> v;
  limbs_t& operator()(limbs_t x) { v.push_back(std::move(x)); return v.back(); }
  ~KeyScratch() { for (limbs_t& x : v) std::fill(x.begin(), x.end(), 0); }
};
template <int NTP>
int do_priv_enc_setup(pai_priv* k, rt_stream s) {
  const int L1 = 8 * NTP, L2 = 16 * NTP, side = pe_side_limbs<NTP>();
  KeyScratch S;
  const limbs_t* x[2] = {&S(padded(k->h_p.data(), L1, L1)), &S(padded(k->h_q.data(), L1, L1))};
  const limbs_t* x2[2] = {&S(h_mul(*x[0], *x[0])), &S(h_mul(*x[1], *x[1]))};
  const limbs_t& n = S(h_mul(*x[0], *x[1]));
  limbs_t& img = S(limbs_t(2 * side + 4 * L2, 0));
  limbs_t& coop_e = S(limbs_t(2 * L2, 0));
  auto put = [](const limbs_t& v, uint32_t* o, size_t limbs) { std::copy(v.begin(), v.begin() + limbs, o); };
  for (int i = 0; i < 2; i++) {                                   // [ yR | yR2 | e1 ] after the digit blob of x
    const limbs_t& y = *x[i ^ 1];
    const limbs_t& xm1 = S(h_sub_small(*x[i], 1));
    const limbs_t& xx1 = S(h_mul(*x[i], xm1));
    uint32_t* o = img.data() + (size_t)i * side + dc_limbs(NTP);
    put(S(h_mod(S(h_shl_limbs(y, L1)), *x[i])), o, L1);
    put(S(h_mod(S(h_shl_limbs(y, 2 * L1)), *x[i])), o + L1, L1);
    put(S(h_mod(y, xm1)), o + 2 * L1, L1);
    put(S(h_mod(n, xx1)), coop_e.data() + (size_t)i * L2, L2);
    k->pe_coop_nwin[i] = (bit_length(xx1) + COOP_W - 1) / COOP_W;
  }
  k->pe_nwin_p = (bit_length(*x[0]) + W_DEC - 1) / W_DEC;
  k->pe_nwin_q = (bit_length(*x[1]) + W_DEC - 1) / W_DEC;
  // u = p^-2 mod q^2 by one Newton step from (p^-1 mod q)^2 mod q: u = u0 * (2 - p^2 u0) mod q^2
  const limbs_t& q = *x[1];
  const limbs_t& q2 = *x2[1];
  const limbs_t& u0 = S(h_mod(S(h_mul(k->h_pinv, k->h_pinv)), q));
  const limbs_t& t = S(h_mod(S(h_mul(*x2[0], u0)), q2));
  const limbs_t& s2 = S(h_mod(S(h_sub(S(h_add_small(S(padded(q2.data(), (int)q2.size(), (int)q2.size() + 1)), 2)), t)), q2));
  const limbs_t& u = S(h_mod(S(h_mul(u0, s2)), q2));
  const limbs_t& uR = S(h_mod(S(h_shl_limbs(u, L1)), q2));
  const limbs_t& uR2 = S(h_mod(S(h_shl_limbs(u, 2 * L1)), q2));
  const limbs_t* kv[3] = {&uR, &S(h_mod(S(h_sub(q2, uR)), q2)), &S(h_mod(S(h_sub(q2, uR2)), q2))};
  for (int j = 0; j < 3; j++) {                                   // K1 = u R, K1N = -u R, K2N = -u R^2 as digits base q
    limbs_t& d0 = S(limbs_t());
    limbs_t& d1 = S(limbs_t());
    h_divmod(*kv[j], q, &d1, &d0);
    uint32_t* o = img.data() + 2 * (size_t)side + (size_t)j * L2;
    put(d0, o, L1);
    put(d1, o + L1, L1);
  }
  put(*x2[0], img.data() + 2 * (size_t)side + 3 * L2, L2);
  int rc = k->d_pe_consts.ensure(img.size() * 4);
  if (!rc) rc = k->d_pe_coop_e.ensure(coop_e.size() * 4);
  if (!rc) rc = rt_h2d(k->d_pe_consts.p, img.data(), img.size() * 4, s);
  pai_mod* md[2] = {k->pd, k->qd};
  for (int i = 0; i < 2 && !rc; i++) rc = rt_d2d(k->d_pe_consts.p + (size_t)i * side, md[i]->d_blob.p, (size_t)dc_limbs(NTP) * 4, s);
  if (!rc) rc = rt_h2d(k->d_pe_coop_e.p, coop_e.data(), coop_e.size() * 4, s);
  if (!rc) rc = rt_sync(s);                                      // the host images are read before they are wiped
  if (!rc) k->pe_wave = std::max(1L, wave_of<PrivEncDigitBody<NTP, W_DEC>>(k->device, priv_enc_shape<NTP>()));
  if (rc) { k->d_pe_consts.release(true); k->d_pe_coop_e.release(true); }
  return rc;
}

// derive one side's constants on the device.  side layout: [ blob(x^2) | blob(x) | xinv | hM | e ]
template <int NTP>
int do_side(pai_priv* k, pai_mod* m2, pai_mod* m1, const limbs_t& x, const limbs_t& g_pad, uint32_t* d_side, int nwin,
            limbs_t& h_out, rt_stream s) {
  const int NT2 = 2 * NTP, L1 = 8 * NTP;
  uint32_t* d_b2 = d_side;
  uint32_t* d_b1 = d_b2 + mc_limbs(NT2);
  uint32_t* d_xinv = d_b1 + mc_limbs(NTP);
  uint32_t* d_hM = d_xinv + L1;
  uint32_t* d_e = d_hM + L1;
  int rc = rt_d2d(d_b2, m2->d_blob.p, (size_t)mc_limbs(NT2) * 4, s);
  if (!rc) rc = rt_d2d(d_b1, m1->d_blob.p, (size_t)mc_limbs(NTP) * 4, s);
  // x^-1 mod 2^(256 NTP)
  if (!rc) { XinvBody xb{nullptr, 0, d_xinv, d_b1 /* N of blob(x) */, L1}; rc = rt_launch(xb, 1, 32, 0, s); }
  // exponent x - 1
  limbs_t e = h_sub_small(x, 1);
  if (!rc) rc = rt_h2d(d_e, e.data(), (size_t)L1 * 4, s);
  // h = 1 for now: hM = R1 of blob(x)
  if (!rc) rc = rt_d2d(d_hM, d_b1 + L1, (size_t)L1 * 4, s);
  if (rc) return rc;
  // l = L(g^(x-1) mod x^2) mod x  via one CRT half with h = 1 on the "ciphertext" g = n + 1
  TmpBuf d_g, d_l, d_h, d_st, d_hm;
  rc = d_g.alloc((size_t)2 * 8 * NT2 * 4);
  if (!rc) rc = d_l.alloc((size_t)L1 * 4);
  if (!rc) rc = d_h.alloc((size_t)L1 * 4);
  if (!rc) rc = d_hm.alloc((size_t)L1 * 4);
  if (!rc) rc = d_st.alloc(16);
  if (!rc) rc = rt_h2d(d_g.p, g_pad.data(), (size_t)2 * 8 * NT2 * 4, s);
  if (!rc) {
    typedef LBody<NTP, W_DEC> B;
    const int cq = side_quads_of(NTP);
    Geom g;
    rc = geometry<B>(k->device, NT2, cq, 3, 1, g);
    if (!rc) rc = k->ws.get(s).tbl.ensure((size_t)g.grid * ((size_t)1 << W_DEC) * 2 * NT2 * g.nthr * 16);
    if (!rc) { B body{d_side, cq, nwin, d_g.u32(), d_l.u32(), (u4*)k->ws.get(s).tbl.p}; rc = rt_launch(body, 1, g.nthr, g.smem, s); }
  }
  // h = l^-1 mod x  (phe/paillier.py:360), then hM = h * R mod x
  if (!rc) rc = do_invert<NTP>(m1, d_l.u32(), NTP, nullptr, d_h.u32(), (int32_t*)d_st.p, 1, s);
  int32_t st = 0;
  if (!rc) rc = rt_d2h(&st, d_st.p, 4, s);
  if (!rc) rc = rt_sync(s);
  if (!rc && st) { g_err = "h_function: inverse does not exist"; rc = PAI_E_NOINV; }
  if (!rc) rc = do_mulmod<NTP>(m1, m1->d_blob.p, mc_limbs(NTP) / 4, d_h.u32(), m1->d_blob.p + L1 /* R1 as a plain number */, d_hm.u32(), 1, s);
  if (!rc) rc = rt_d2d(d_hM, d_hm.p, (size_t)L1 * 4, s);
  h_out.assign(L1, 0);
  if (!rc) rc = rt_d2h(h_out.data(), d_h.p, (size_t)L1 * 4, s);
  if (!rc) rc = rt_sync(s);
  return rc;
}

template <int NTP>
int do_priv_setup(pai_priv* k, rt_stream s) {
  const int L1 = 8 * NTP, NT2 = 2 * NTP;
  const int sideq = side_quads_of(NTP);
  int rc = k->d_consts.ensure(((size_t)2 * sideq + 2 * NTP) * 16);
  if (!rc) rc = rt_memset(k->d_consts.p, 0, k->d_consts.bytes, s);
  if (rc) return rc;
  limbs_t p = padded(k->h_p.data(), L1, L1), q = padded(k->h_q.data(), L1, L1);
  limbs_t n = h_mul(p, q);                         // 2*L1 limbs
  limbs_t g = h_add_small(n, 1);                   // g = n + 1 (phe/paillier.py:87); cannot overflow 2*L1 limbs for n = p*q odd < 2^k - 1
  limbs_t g_pad = padded(g.data(), (int)g.size(), 2 * 8 * NT2);
  k->nwin_p = (bit_length(h_sub_small(p, 1)) + W_DEC - 1) / W_DEC;
  k->nwin_q = (bit_length(h_sub_small(q, 1)) + W_DEC - 1) / W_DEC;
  uint32_t* d_P = k->d_consts.p;
  uint32_t* d_Q = k->d_consts.p + (size_t)sideq * 4;
  uint32_t* d_pinvqM = k->d_consts.p + (size_t)2 * sideq * 4;
  rc = do_side<NTP>(k, k->p2, k->p1, p, g_pad, d_P, k->nwin_p, k->h_hp, s);
  if (!rc) rc = do_side<NTP>(k, k->q2, k->q1, q, g_pad, d_Q, k->nwin_q, k->h_hq, s);
  if (rc) return rc;
  // p_inverse = p^-1 mod q (phe/paillier.py:233); pinvqM = p_inverse * R mod q
  TmpBuf d_p, d_pi, d_st, d_pm;
  rc = d_p.alloc((size_t)L1 * 4);
  if (!rc) rc = d_pi.alloc((size_t)L1 * 4);
  if (!rc) rc = d_pm.alloc((size_t)L1 * 4);
  if (!rc) rc = d_st.alloc(16);
  if (!rc) rc = rt_h2d(d_p.p, p.data(), (size_t)L1 * 4, s);
  if (!rc) rc = do_invert<NTP>(k->q1, d_p.u32(), NTP, nullptr, d_pi.u32(), (int32_t*)d_st.p, 1, s);
  int32_t st = 0;
  if (!rc) rc = rt_d2h(&st, d_st.p, 4, s);
  if (!rc) rc = rt_sync(s);
  if (!rc && st) { g_err = "p has no inverse mod q"; rc = PAI_E_NOINV; }
  if (!rc) rc = do_mulmod<NTP>(k->q1, k->q1->d_blob.p, mc_limbs(NTP) / 4, d_pi.u32(), k->q1->d_blob.p + L1, d_pm.u32(), 1, s);
  if (!rc) rc = rt_d2d(d_pinvqM, d_pm.p, (size_t)L1 * 4, s);
  k->h_pinv.assign(L1, 0);
  if (!rc) rc = rt_d2h(k->h_pinv.data(), d_pi.p, (size_t)L1 * 4, s);
  if (!rc) rc = rt_sync(s);
  return rc;
}

}  // namespace

// ================================================================================================ C ABI
// ---- warp-per-ciphertext path (pai_coop.cuh) -------------------------------------------------------------------
// A batch, or the tail of a batch beyond whole waves of the throughput kernel, of at most coop_limit(wave) elements
// takes it.  A wave of the thread-per-ciphertext kernel costs the same whether it holds one ciphertext or a full wave,
// while the warp kernels run at a fraction of its full-wave throughput with a small floor -- so they win up to about a
// third of a wave.
// PAI_COOP_MAX overrides the limit with an absolute element count (0 disables the path).
static long coop_limit(long wave) {
  const char* e = getenv("PAI_COOP_MAX");
  if (e && *e) return atol(e);
#ifdef PAI_HOSTSIM
  (void)wave;
  return 0;            // the simulation build of the tests exercises the throughput kernels unless asked otherwise
#else
  return wave * 3 / 10;
#endif
}
// rows [batch - n, batch) that go to the warp kernels
static long coop_rows(long batch, long wave) {
  const long lim = coop_limit(wave);
  if (batch <= lim) return batch;
  const long tail = wave > 0 ? batch % wave : 0;
  return tail <= lim ? tail : 0;
}
// one CTA (= one warp) per item, no grid-stride loop: the hardware block scheduler refills SMs as items finish
template <int K, class B>
static int launch_coop(const B& b, long items, rt_stream s) {
  const int grid = (int)std::min<long>((items + COOP_WARPS - 1) / COOP_WARPS, 1L << 30);
  return rt_launch_coop(b, grid, 32 * COOP_WARPS, (size_t)COOP_WARPS * (1 << COOP_W) * K * 32 * 4, s);
}
// constants of the modulus in the warp layout, computed once with the generic kernels: 2^(64 Lc) and 2^(96 Lc) mod N
static int ensure_coop(pai_mod* m, rt_stream s) {
  if (m->coopK) return 0;
  const int Lc = (m->L + 31) / 32 * 32, K = Lc / 32;
  if (K != 1 && K != 2 && K != 3 && K != 4 && K != 6 && K != 8) { g_err = "unsupported operand size"; return PAI_E_ARG; }
  TmpBuf tmp_buf;
  int rc = m->d_coop.ensure((size_t)3 * Lc * 4);
  if (!rc) rc = tmp_buf.alloc((size_t)2 * m->L * 4);
  uint32_t* blob = m->d_coop.p;
  uint32_t* tmp = tmp_buf.u32();
  if (!rc) rc = rt_memset(blob, 0, m->d_coop.bytes, s);
  if (!rc) rc = rt_h2d(blob, m->h_N.data(), (size_t)m->L * 4, s);
  limbs_t two(m->L, 0);
  two[0] = 2;
  if (!rc) rc = rt_h2d(tmp, two.data(), (size_t)m->L * 4, s);
  m->coop_building = true;
  for (int i = 0; i < 2 && !rc; i++) {
    uint32_t e = (uint32_t)((i + 2) * 32 * Lc);
    rc = pai_mod_powmod_shared(m, tmp, m->L, &e, 1, tmp + m->L, 1, s);
    if (!rc) rc = rt_d2d(blob + (size_t)(i + 1) * Lc, tmp + m->L, (size_t)m->L * 4, s);
  }
  m->coop_building = false;
  if (!rc) rc = rt_sync(s);
  if (rc) { m->d_coop.release(); return rc; }
  uint32_t n0 = m->h_N[0], i0 = n0;
  for (int i = 0; i < 5; i++) i0 *= 2u - n0 * i0;
  m->coop_n0inv = 0u - i0;                       // -N^-1 mod 2^32
  m->coopK = K;
  return 0;
}
template <int K>
static int do_coop_powmod(pai_mod* m, const uint32_t* d_base, int base_limbs, const uint32_t* d_exp, int exp_limbs, int nbits,
                          uint32_t* d_out, long batch, rt_stream s) {
  CoopPowBody<K> b;
  b.consts = nullptr; b.const_quads = 0; b.nsides = 1;
  b.blob[0] = b.blob[1] = m->d_coop.p; b.n0inv[0] = b.n0inv[1] = m->coop_n0inv;
  b.e[0] = b.e[1] = d_exp; b.e_limbs = exp_limbs; b.nwin[0] = b.nwin[1] = (nbits + COOP_W - 1) / COOP_W;
  b.out[0] = b.out[1] = d_out; b.base = d_base; b.base_limbs = base_limbs; b.out_limbs = m->L; b.batch = batch;
  return launch_coop<K>(b, batch, s);
}

template <int K>
static int do_coop_encrypt(pai_pub* k, const uint32_t* d_m, const uint32_t* d_r, uint32_t* d_c, long batch, rt_stream s) {
  pai_mod* m = k->nsq;
  const int nwin = (bit_length(k->h_n) + COOP_W - 1) / COOP_W;
  CoopEncBody<K> b{nullptr, 0, m->d_coop.p, m->coop_n0inv, k->d_nth, k->ln, nwin, d_m, d_r, d_c, batch};
  return launch_coop<K>(b, batch, s);
}
template <int K>
static int do_coop_decrypt_pow(pai_priv* k, const uint32_t* d_c, uint32_t* up, uint32_t* uq, long batch, rt_stream s) {
  const int L1 = 8 * k->NTP, L2 = 16 * k->NTP;
  CoopPowBody<K> b;
  b.consts = nullptr; b.const_quads = 0; b.nsides = 2;
  b.blob[0] = k->p2->d_coop.p; b.blob[1] = k->q2->d_coop.p; b.n0inv[0] = k->p2->coop_n0inv; b.n0inv[1] = k->q2->coop_n0inv;
  b.e[0] = k->d_coop_e.p; b.e[1] = k->d_coop_e.p + L1; b.e_limbs = L1;
  b.nwin[0] = (bit_length(h_sub_small(k->h_p, 1)) + COOP_W - 1) / COOP_W;
  b.nwin[1] = (bit_length(h_sub_small(k->h_q, 1)) + COOP_W - 1) / COOP_W;
  b.out[0] = up; b.out[1] = uq; b.base = d_c; b.base_limbs = 2 * L2; b.out_limbs = L2; b.batch = batch;
  return launch_coop<K>(b, 2 * batch, s);
}
// r^n mod p^2 and mod q^2 as r^(n mod x(x-1)) for pai_priv_encrypt (the two sides of a row on two warps)
template <int K>
static int do_coop_priv_enc_pow(pai_priv* k, const uint32_t* d_r, uint32_t* up, uint32_t* uq, long batch, rt_stream s) {
  const int L2 = 16 * k->NTP;
  CoopPowBody<K> b;
  b.consts = nullptr; b.const_quads = 0; b.nsides = 2;
  b.blob[0] = k->p2->d_coop.p; b.blob[1] = k->q2->d_coop.p; b.n0inv[0] = k->p2->coop_n0inv; b.n0inv[1] = k->q2->coop_n0inv;
  b.e[0] = k->d_pe_coop_e.p; b.e[1] = k->d_pe_coop_e.p + L2; b.e_limbs = L2;
  b.nwin[0] = k->pe_coop_nwin[0]; b.nwin[1] = k->pe_coop_nwin[1];
  b.out[0] = up; b.out[1] = uq; b.base = d_r; b.base_limbs = L2; b.out_limbs = L2; b.batch = batch;
  return launch_coop<K>(b, 2 * batch, s);
}

// ---- batched Miller-Rabin (key generation) -------------------------------------------------------
template <int NT>
static int do_miller_rabin(const uint32_t* d_cand, const uint32_t* d_bases, int rounds, int32_t* d_result, long batch, int device, rt_stream s) {
  typedef MillerRabinBody<NT, 4> B;
#if defined(PAI_HOSTSIM)
  const int nthr = 2;
#else
  const int nthr = 64;
#endif
  long blocks = (batch + nthr - 1) / nthr;
  int grid = (int)std::max(1L, std::min(blocks, (long)rt_sm_count(device) * 8));
  TmpBuf ws;
  int rc = ws.alloc((size_t)grid * nthr * mr_ws_limbs<NT, 4>() * 4);
  if (rc) return rc;
  B body{nullptr, 0, d_cand, d_bases, rounds, d_result, ws.u32(), batch};
  rc = rt_launch(body, grid, nthr, 0, s);
  if (!rc) rc = rt_sync(s);
  return rc;
}

// ---- one entry per operation and kernel family -------------------------------------------------------------------
// rows per full wave of the throughput kernels (measured once per context from the launch geometry)
static int pub_wave(pai_pub* k) {
  if (k->wave) return 0;
  int rc = 0;
  switch (k->family) {
    case TC: DISPATCH_TC(k->nmod->NT, k->wave = (tc_wave<TcEncBody<NTH>, NTH>(k->nmod->device, tc_enc_smem_bytes<NTH>))); break;
    case DIGIT: DISPATCH_NTH(k->nmod->NT, k->wave = wave_of<EncDigitBody<NTH>>(k->nmod->device, enc_digit_shape<NTH>(k))); break;
    case FULL: DISPATCH_NT(k->nsq->NT, k->wave = wave_of<EncBody<NT>>(k->nsq->device, enc_shape<NT>(k))); break;
  }
  if (rc) return rc;
  if (k->wave <= 0) k->wave = 1;
  return 0;
}
static int priv_wave(pai_priv* k) {
  if (k->wave) return 0;
  int rc = 0;
  switch (k->family) {
    case TC: DISPATCH_TC(k->NTP, k->wave = (tc_wave<TcDecBody<NTH, W_DEC>, NTH>(k->device, tc_dec_smem_bytes<NTH>))); break;
    case DIGIT: DISPATCH_NTP(k->NTP, k->wave = (wave_of<DecDigitBody<NTP, W_DEC>>(k->device, dec_digit_shape<NTP>()))); break;
    case FULL: DISPATCH_NTP(k->NTP, k->wave = (wave_of<DecBody<NTP, W_DEC>>(k->device, dec_shape<NTP>()))); break;
  }
  if (rc) return rc;
  if (k->wave <= 0) k->wave = 1;
  return 0;
}
// the throughput encrypt kernels on rows [0, batch) (after pub_wave)
static int encrypt_rows(pai_pub* k, const uint32_t* d_m, const uint32_t* d_r, uint32_t* d_c, long batch, rt_stream s) {
  int rc = 0;
  switch (k->family) {
    case TC:
      DISPATCH_TC(k->nmod->NT, rc = tc_split(k->wave, batch, [&](long off, long rows) {
        return do_encrypt_tc<NTH>(k, d_m + off * 8 * NTH, d_r + off * 8 * NTH, d_c + off * 16 * NTH, rows, s);
      }));
      break;
    case DIGIT: DISPATCH_NTH(k->nmod->NT, rc = do_encrypt_digit<NTH>(k, d_m, d_r, d_c, batch, s)); break;
    case FULL: DISPATCH_NT(k->nsq->NT, rc = do_encrypt<NT>(k, d_m, d_r, d_c, batch, s)); break;
  }
  return rc;
}
// the throughput decrypt kernels on rows [0, batch) (after priv_wave)
static int decrypt_rows(pai_priv* k, const uint32_t* d_c, uint32_t* d_m, long batch, rt_stream s) {
  int rc = 0;
  switch (k->family) {
    case TC:
      DISPATCH_TC(k->NTP, rc = tc_split(k->wave, batch, [&](long off, long rows) {
        return do_decrypt_tc<NTH>(k, d_c + off * 32 * NTH, d_m + off * 16 * NTH, rows, s);
      }));
      break;
    case DIGIT: DISPATCH_NTP(k->NTP, rc = do_decrypt_digit<NTP>(k, d_c, d_m, batch, s)); break;
    case FULL: DISPATCH_NTP(k->NTP, rc = do_decrypt<NTP>(k, d_c, d_m, batch, s)); break;
  }
  return rc;
}

namespace {
struct StageIn { DevBuf<>& buf; const void* src; size_t bytes; };
struct StageOut { DevBuf<>& buf; void* dst; size_t bytes; };   // dst may be null: the device result is not copied back
// A host-pointer entry point: under the context's lock and on its device, copy the inputs into the context's staging
// buffers, size the outputs, run `call` (the device-pointer variant on stream 0) and copy the outputs back.  The lock is
// held until the results are in host memory.
template <class Call>
int run_staged(std::recursive_mutex& mu, int device, long batch, std::initializer_list<StageIn> in, std::initializer_list<StageOut> out,
               Call call) {
  DeviceGuard device_guard_; (void)device_guard_;
  CtxLock lock_(mu);
  if (batch == 0) return 0;
  int rc = rt_set_device(device);
  for (const StageIn& x : in) {
    if (!rc) rc = x.buf.ensure(x.bytes);
    if (!rc) rc = rt_h2d(x.buf.p, x.src, x.bytes, 0);
  }
  for (const StageOut& x : out) if (!rc) rc = x.buf.ensure(x.bytes);
  if (!rc) rc = call();
  for (const StageOut& x : out) if (!rc && x.dst) rc = rt_d2h(x.dst, x.buf.p, x.bytes, 0);
  if (!rc) rc = rt_sync(0);
  return rc;
}
template <class T = uint32_t>
T* dev(const DevBuf<>& b) { return (T*)b.p; }

// pai_pack_slots / pai_unpack_slots: one launch of `b` over the rows of `count` slots, 128 threads per CTA, n in shared
// memory; no workspace, so no lock
template <class Body>
int pack_launch(pai_pub* k, const void* d_in, void* d_out, int32_t* d_status, long count, int slot_bits, void* stream, Body b) {
  DeviceGuard device_guard_; (void)device_guard_;
  const int K = pai_pack_slots_per_row(k, slot_bits);
  if (K < 0) return K;
  if (!d_in || !d_out || !d_status || count < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  if (count == 0) return 0;
  int rc = rt_set_device(k->nsq->device);
  if (rc) return rc;
  const long rows = (count + K - 1) / K;
  b.consts = k->d_nth; b.const_quads = k->ln / 4;
  b.b = slot_bits; b.K = K; b.ln = k->ln; b.count = count; b.status = d_status; b.rows = rows;
  const long blocks = (rows + 127) / 128;
  return rt_launch(b, (int)std::min(blocks, (long)rt_sm_count(k->nsq->device) * 16), 128, (size_t)k->ln * 4, (rt_stream)stream);
}
}  // namespace

extern "C" {

const char* pai_last_error(void) { return g_err.c_str(); }
int pai_version(void) { return 100; }
int pai_device_count(void) { return rt_device_count(); }
long pai_launch_count(void) { return g_launches.load(); }

int pai_mod_create(const uint32_t* modulus, int limbs, int device, pai_mod** out) {
  DeviceGuard device_guard_; (void)device_guard_;
  return mod_create_impl(modulus, limbs, device, 0, 0, out);
}
int pai_mod_destroy(pai_mod* m) { mod_free(m, false); return 0; }
int pai_mod_limbs(const pai_mod* m) { return m ? m->L : PAI_E_ARG; }

int pai_mod_mulmod(pai_mod* m, const uint32_t* d_a, const uint32_t* d_b, uint32_t* d_out, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!m || !d_a || !d_b || !d_out || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(m->mu);
  if (batch == 0) return 0;
  int rc = rt_set_device(m->device);
  if (rc) return rc;
  DISPATCH_NT(m->NT, rc = do_mulmod<NT>(m, m->d_blob.p, mc_limbs(NT) / 4, d_a, d_b, d_out, batch, (rt_stream)stream));
  return rc;
}

static int powmod_common(pai_mod* m, const uint32_t* d_base, int base_limbs, const uint32_t* d_exp, int exp_limbs, long exp_stride,
                         int nwin_fixed, uint32_t* d_out, long batch, void* stream) {
  if (base_limbs != m->L && base_limbs != 2 * m->L) { g_err = "base_limbs must be L or 2L"; return PAI_E_ARG; }
  int rc = 0;
  DISPATCH_NT(m->NT, rc = do_powmod<NT>(m, d_base, base_limbs / 8, d_exp, exp_limbs, exp_stride, nwin_fixed, d_out, batch, (rt_stream)stream));
  return rc;
}

int pai_mod_powmod_shared(pai_mod* m, const uint32_t* d_base, int base_limbs, const uint32_t* exponent, int exp_limbs,
                          uint32_t* d_out, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!m || !d_base || !exponent || !d_out || batch < 0 || exp_limbs <= 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(m->mu);
  if (batch == 0) return 0;
  int rc = rt_set_device(m->device);
  if (rc) return rc;
  limbs_t e(exponent, exponent + exp_limbs);
  int nwin = (bit_length(e) + W_VAR - 1) / W_VAR;
  const bool coop = !m->coop_building && batch <= coop_limit(8192);
  if (coop) {                                   // before the exponent is staged: building the constants uses tmp_e too
    if (base_limbs != m->L && base_limbs != 2 * m->L) { g_err = "base_limbs must be L or 2L"; return PAI_E_ARG; }
    rc = ensure_coop(m, (rt_stream)stream);
    if (rc) return rc;
  }
  rc = m->tmp_e.ensure((size_t)exp_limbs * 4);
  if (!rc) rc = rt_h2d(m->tmp_e.p, exponent, (size_t)exp_limbs * 4, (rt_stream)stream);
  if (!rc) rc = rt_sync((rt_stream)stream);   // `exponent` is caller-owned host memory
  if (rc) return rc;
  if (coop) {
    DISPATCH_K(m->coopK, rc = do_coop_powmod<K>(m, d_base, base_limbs, (const uint32_t*)m->tmp_e.p, exp_limbs, bit_length(e), d_out,
                                                batch, (rt_stream)stream));
    return rc;
  }
  return powmod_common(m, d_base, base_limbs, (const uint32_t*)m->tmp_e.p, exp_limbs, 0, nwin, d_out, batch, stream);
}

int pai_mod_powmod(pai_mod* m, const uint32_t* d_base, int base_limbs, const uint32_t* d_exp, int exp_limbs,
                   uint32_t* d_out, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!m || !d_base || !d_exp || !d_out || batch < 0 || exp_limbs <= 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(m->mu);
  if (batch == 0) return 0;
  int rc = rt_set_device(m->device);
  if (rc) return rc;
  return powmod_common(m, d_base, base_limbs, d_exp, exp_limbs, exp_limbs, -1, d_out, batch, stream);
}

int pai_mod_invert(pai_mod* m, const uint32_t* d_a, int a_limbs, uint32_t* d_out, int32_t* d_status, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!m || !d_a || !d_out || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(m->mu);
  if (a_limbs != m->L) { g_err = "a_limbs must equal pai_mod_limbs()"; return PAI_E_ARG; }
  if (batch == 0) return 0;
  int rc = rt_set_device(m->device);
  if (rc) return rc;
  DISPATCH_NT(m->NT, rc = do_invert<NT>(m, d_a, a_limbs / 8, nullptr, d_out, d_status, batch, (rt_stream)stream));
  return rc;
}

// ---------------------------------------------------------------------------------------- public key
int pai_pub_create(const uint32_t* n, int limbs, int device, pai_pub** out) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!n || !out || limbs <= 0) { g_err = "bad argument"; return PAI_E_ARG; }
  int eff = eff_limbs(n, limbs);
  if (eff == 0 || !(n[0] & 1u)) { g_err = "n must be odd"; return PAI_E_ARG; }
  // n has 2*NTp tiles, n^2 4*NTp, where NTp covers half of n's limbs
  int ntp = pick_ntp((eff + 15) / 16);
  if (ntp < 0) { g_err = "key too large (max 4096 bits)"; return PAI_E_ARG; }
  int NT = 4 * ntp, ln = 4 * NT;
  limbs_t nn = padded(n, eff, ln);
  limbs_t nsq = h_mul(nn, nn);                     // 2*ln = 8*NT limbs
  pai_pub* k = new (std::nothrow) pai_pub();
  if (!k) return PAI_E_ARG;
  k->ln = ln; k->h_n = nn;
  int rc = mod_create_impl(nsq.data(), (int)nsq.size(), device, NT, ln, &k->nsq);
  if (rc) { delete k; return rc; }
  // n right after the blob (encrypt's constant area)
  rc = rt_h2d(k->nsq->d_blob.p + mc_limbs(NT), nn.data(), (size_t)ln * 4, 0);
  // raw_mul branch threshold n - max_int, max_int = n//3 - 1   (phe/paillier.py:90, 745)
  limbs_t maxint = h_sub_small(h_div_small(nn, 3), 1);
  limbs_t thr = h_sub(nn, maxint);
  if (!rc) rc = rt_malloc((void**)&k->d_nth, (size_t)2 * ln * 4);
  if (!rc) rc = rt_h2d(k->d_nth, nn.data(), (size_t)ln * 4, 0);
  if (!rc) rc = rt_h2d(k->d_nth + ln, thr.data(), (size_t)ln * 4, 0);
  // modulus n itself with the digit-form constants (encrypt runs on base-n digits, pai_digit.cuh)
  if (!rc) rc = mod_create_impl(nn.data(), ln, device, 2 * ntp, dc_extra_limbs(2 * ntp), &k->nmod);
  if (!rc) { DISPATCH_NTH(2 * ntp, rc = do_digit_setup<NTH>(k->nmod, 0)); }
  if (!rc) {   // compact encrypt constants: [ N | ONE | NINV | KL | RR | ZERO ] gathered from the digit blob
    const int h = 8 * 2 * ntp;
    const uint32_t* b = k->nmod->d_blob.p;
    const uint32_t* e = b + 5 * h + 8;            // KL | RR(2h) | ONEM(2h) | ZERO | ...
    rc = rt_malloc((void**)&k->d_enc_consts, (size_t)dc_pow_limbs(2 * ntp) * 4);
    uint32_t* c = k->d_enc_consts;
    if (!rc) rc = rt_d2d(c, b, (size_t)h * 4, 0);                                  // N
    if (!rc) rc = rt_d2d(c + h, b + 4 * h, (size_t)(h + 8) * 4, 0);                // ONE | NINV
    if (!rc) rc = rt_d2d(c + 2 * h + 8, e, (size_t)3 * h * 4, 0);                  // KL | RR
    if (!rc) rc = rt_d2d(c + 5 * h + 8, e + 12 * h, (size_t)(2 * h + 8) * 4, 0);   // N2 | N3 | TOPS
    if (!rc) rc = rt_d2d(c + 7 * h + 16, e + 3 * h, (size_t)2 * h * 4, 0);         // ONEM
    if (!rc) rc = rt_d2d(c + 9 * h + 16, e + 6 * h, (size_t)2 * h * 4, 0);         // E3
  }
  // tensor-core reductions (pai_tc.cuh): digit moduli of at most 384 base-256 digits (keys up to 3072 bits; above that
  // the operand buffers of even one 128-thread group no longer fit shared memory)
  k->family = pick_family("PAI_ENCRYPT_PATH", tc_supported(2 * ntp, 12));
  if (!rc && k->family == TC) {
    DISPATCH_TC(2 * ntp, rc = do_tc_setup<NTH>(k, 0));
    k->tc_stagger = tc_stagger_cycles();
  }
  // exponent program for r^n: sliding windows of W_ENC bits over the public exponent n
  std::vector<uint32_t> prog = sliding_program(nn, W_ENC);
  k->nops = (int)prog.size();
  k->nodd = 1 << (W_ENC - 1);
  if (!rc) rc = rt_malloc((void**)&k->d_prog, prog.size() * 4 + 16);
  if (!rc) rc = rt_h2d(k->d_prog, prog.data(), prog.size() * 4, 0);
  if (!rc) rc = rt_sync(0);
  if (rc) { pai_pub_destroy(k); return rc; }
  *out = k;
  return 0;
}
int pai_pub_destroy(pai_pub* k) {
  if (!k) return 0;
  if (k->nsq) rt_set_device(k->nsq->device);
  rt_free(k->d_nth);
  rt_free(k->d_prog);
  rt_free(k->d_enc_consts);
  rt_free(k->d_tc);
  k->ws.release(); k->h_m.release(); k->h_r.release(); k->h_c.release(); k->h_s.release();
  mod_free(k->nsq, false);
  mod_free(k->nmod, false);
  delete k;
  return 0;
}
int pai_pub_n_limbs(const pai_pub* k) { return k ? k->ln : PAI_E_ARG; }
int pai_pub_c_limbs(const pai_pub* k) { return k ? 2 * k->ln : PAI_E_ARG; }
int pai_pub_kernel_path(const pai_pub* k) { return k ? k->family : PAI_E_ARG; }
long pai_pub_wave(pai_pub* k) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k) return PAI_E_ARG;
  CtxLock lock_(k->mu);
  if (rt_set_device(k->nsq->device) || pub_wave(k)) return PAI_E_CUDA;
  return k->wave;
}

int pai_encrypt(pai_pub* k, const uint32_t* d_m, const uint32_t* d_r, uint32_t* d_c, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || !d_m || !d_r || !d_c || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(k->mu);
  if (batch == 0) return 0;
  int rc = rt_set_device(k->nsq->device);
  if (rc) return rc;
  rc = pub_wave(k);
  if (rc) return rc;
  const long ncoop = coop_rows(batch, k->wave);     // small batch / tail: one warp per ciphertext (pai_coop.cuh)
  if (ncoop) {
    pai_mod* m = k->nsq;
    rc = ensure_coop(m, (rt_stream)stream);
    if (rc) return rc;
    const long off = batch - ncoop;
    DISPATCH_K(m->coopK, rc = do_coop_encrypt<K>(k, d_m + off * k->ln, d_r + off * k->ln, d_c + off * 2 * k->ln, ncoop,
                                                 (rt_stream)stream));
    if (rc || off == 0) return rc;
    batch = off;
  }
  return encrypt_rows(k, d_m, d_r, d_c, batch, (rt_stream)stream);
}
int pai_random_lt_n(pai_pub* k, const uint8_t* seed32, unsigned long long nonce, uint32_t* d_r, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || !seed32 || !d_r || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  if (batch == 0) return 0;
  int rc = rt_set_device(k->nsq->device);
  if (rc) return rc;
  RngBody b;
  b.consts = nullptr; b.const_quads = 0;
  memcpy(b.key, seed32, 32);
  b.nonce = nonce; b.n = k->d_nth; b.ln = k->ln; b.nbits = bit_length(k->h_n); b.out = d_r; b.batch = batch;
  long blocks = (batch + 127) / 128;
  return rt_launch(b, (int)std::min(blocks, (long)rt_sm_count(k->nsq->device) * 16), 128, 0, (rt_stream)stream);
}
// ---- batched Miller-Rabin (key generation): do_miller_rabin above
int pai_miller_rabin(const uint32_t* d_cand, int limbs, const uint32_t* d_bases, int rounds, int32_t* d_result, long batch, int device,
                     void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!d_cand || !d_bases || !d_result || batch < 0 || rounds < 1 || limbs < 8 || limbs % 8) { g_err = "bad argument"; return PAI_E_ARG; }
  if (batch == 0) return 0;
  int rc = rt_set_device(device);
  if (rc) return rc;
  DISPATCH_NT(limbs / 8, rc = do_miller_rabin<NT>(d_cand, d_bases, rounds, d_result, batch, device, (rt_stream)stream));
  return rc;
}
// ---- decimal wire format ---------------------------------------------------------------------
static int radix_geometry(int device, int limbs, long batch, int* grid, int* nthr, size_t* smem) {
  if (limbs < 1 || limbs > 1024) { g_err = "limb count not supported"; return PAI_E_ARG; }
  int t = (int)std::min<size_t>(128, (rt_max_smem(device) - 1024) / ((size_t)limbs * 4));
  t = std::min(t, NTHR_MAX);
  if (t >= 32) t &= ~31;
  if (t < 1) { g_err = "limb count not supported"; return PAI_E_ARG; }
  *nthr = t;
  *smem = (size_t)limbs * 4 * t;
  *grid = (int)std::min<long>((batch + t - 1) / t, (long)rt_sm_count(device) * 8);
  return 0;
}
int pai_decimal_width(int limbs) { return limbs > 0 ? 9 * radix_chunks(limbs) : 0; }
int pai_limbs_to_decimal(const uint32_t* d_limbs, int limbs, uint8_t* d_text, long batch, int device, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!d_limbs || !d_text || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  if (batch == 0) return 0;
  int rc = rt_set_device(device);
  if (rc) return rc;
  int grid, nthr; size_t smem;
  if ((rc = radix_geometry(device, limbs, batch, &grid, &nthr, &smem))) return rc;
  ToDecBody b{nullptr, 0, d_limbs, limbs, d_text, radix_chunks(limbs), batch};
  return rt_launch(b, grid, nthr, smem, (rt_stream)stream);
}
int pai_decimal_to_limbs(const uint8_t* d_text, int width, uint32_t* d_limbs, int limbs, int32_t* d_status, long batch, int device,
                         void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!d_limbs || !d_text || batch < 0 || width < 1) { g_err = "bad argument"; return PAI_E_ARG; }
  if (batch == 0) return 0;
  int rc = rt_set_device(device);
  if (rc) return rc;
  int grid, nthr; size_t smem;
  if ((rc = radix_geometry(device, limbs, batch, &grid, &nthr, &smem))) return rc;
  FromDecBody b{nullptr, 0, d_text, width, d_limbs, limbs, d_status, batch};
  return rt_launch(b, grid, nthr, smem, (rt_stream)stream);
}
// ---- packed fixed-point rows (pai_pack.cuh) ------------------------------------------------------
int pai_pack_slots_per_row(const pai_pub* k, int slot_bits) {
  if (!k || slot_bits < 2 || slot_bits > 63) { g_err = "bad argument"; return PAI_E_ARG; }
  const int K = (bit_length(k->h_n) - 1) / slot_bits;
  if (K < 1) { g_err = "slot wider than the key"; return PAI_E_ARG; }
  return K;
}
int pai_pack_slots(pai_pub* k, const int64_t* d_slots, long count, int slot_bits, uint32_t* d_m, int32_t* d_status, void* stream) {
  PackBody b{};
  b.s = d_slots; b.m = d_m;
  return pack_launch(k, d_slots, d_m, d_status, count, slot_bits, stream, b);
}
int pai_unpack_slots(pai_pub* k, const uint32_t* d_m, int slot_bits, int64_t* d_slots, long count, int32_t* d_status, void* stream) {
  UnpackBody b{};
  b.m = d_m; b.s = d_slots;
  return pack_launch(k, d_m, d_slots, d_status, count, slot_bits, stream, b);
}
int pai_raw_add(pai_pub* k, const uint32_t* d_a, const uint32_t* d_b, uint32_t* d_c, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k) { g_err = "bad argument"; return PAI_E_ARG; }
  return pai_mod_mulmod(k->nsq, d_a, d_b, d_c, batch, stream);
}
int pai_raw_sum(pai_pub* k, const uint32_t* d_c, long batch, uint32_t* d_out, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || !d_c || !d_out || batch < 1) { g_err = "bad argument"; return PAI_E_ARG; }
  pai_mod* m = k->nsq;
  CtxLock lock_(m->mu);
  int rc = rt_set_device(m->device);
  if (rc) return rc;
  DISPATCH_NT(m->NT, rc = do_reduce_mul<NT>(m, d_c, batch, d_out, (rt_stream)stream));
  return rc;
}
// raw_mul's branch per element (phe/paillier.py:742-749) into the stream's workspace: exponent s or n - s (w_exp), base
// c or invert(c) mod n^2 (w_base); statuses go to d_status, or to scratch when it is null
static int rawmul_prepare(pai_pub* k, StreamWs& w, const uint32_t* d_a, const uint32_t* d_s, int32_t* d_status, long batch, rt_stream s) {
  const int ln = k->ln;
  int rc = w.w_exp.ensure((size_t)batch * ln * 4);
  if (!rc) rc = w.w_base.ensure((size_t)batch * 2 * ln * 4);
  if (!rc) rc = w.w_flag.ensure((size_t)batch * 4 * 2);
  if (rc) return rc;
  int32_t* flag = (int32_t*)w.w_flag.p;
  PrepBody b{nullptr, 0, k->d_nth, k->d_nth + ln, ln, d_s, (uint32_t*)w.w_exp.p, flag, batch};
  rc = rt_launch(b, (int)std::min((batch + 127) / 128, 65535L), 128, 0, s);
  if (rc) return rc;
  pai_mod* m = k->nsq;
  DISPATCH_NT(m->NT, rc = do_invert_flagged<NT>(m, d_a, flag, (uint32_t*)w.w_base.p, d_status ? d_status : flag + batch, batch, s));
  return rc;
}
// base^exp mod n^2 per element, exponents of ln limbs (raw_mul; raw_dot outside the tensor-core family)
static int powers(pai_pub* k, const uint32_t* d_base, const uint32_t* d_exp, uint32_t* d_out, long batch, rt_stream s) {
  int rc = 0;
  switch (k->family) {
    case TC: DISPATCH_TC(k->nmod->NT, rc = do_powmod_tc<NTH>(k, d_base, d_exp, k->ln, d_out, batch, s)); break;
    case DIGIT: DISPATCH_NTH(k->nmod->NT, rc = do_powmod_digit<NTH>(k, d_base, d_exp, k->ln, d_out, batch, s)); break;
    case FULL: rc = powmod_common(k->nsq, d_base, 2 * k->ln, d_exp, k->ln, k->ln, -1, d_out, batch, s); break;
  }
  return rc;
}
int pai_raw_mul(pai_pub* k, const uint32_t* d_a, const uint32_t* d_s, uint32_t* d_c, int32_t* d_status, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || !d_a || !d_s || !d_c || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(k->mu);
  if (batch == 0) return 0;
  rt_stream s = (rt_stream)stream;
  int rc = rt_set_device(k->nsq->device);
  if (rc) return rc;
  StreamWs& w = k->ws.get(s);
  rc = rawmul_prepare(k, w, d_a, d_s, d_status, batch, s);
  if (rc) return rc;
  return powers(k, (const uint32_t*)w.w_base.p, (const uint32_t*)w.w_exp.p, d_c, batch, s);
}

int pai_raw_dot(pai_pub* k, const uint32_t* d_a, const uint32_t* d_s, uint32_t* d_out, int32_t* d_status, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || !d_a || !d_s || !d_out || batch < 1) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(k->mu);
  pai_mod* m = k->nsq;
  rt_stream s = (rt_stream)stream;
  int rc = rt_set_device(m->device);
  if (rc) return rc;
  StreamWs& w = k->ws.get(s);
  rc = rawmul_prepare(k, w, d_a, d_s, d_status, batch, s);
  if (!rc) rc = w.red_b.ensure((size_t)batch * 2 * k->ln * 4);   // a row per element (an upper bound for the Straus groups)
  if (rc) return rc;
  const uint32_t* base = (const uint32_t*)w.w_base.p;
  const uint32_t* exp = (const uint32_t*)w.w_exp.p;
  long nrows = batch;
  if (k->family == TC) {                               // Straus groups on the tensor-core path -> one row per group
    DISPATCH_TC(k->nmod->NT, rc = do_straus_tc<NTH>(k, base, exp, k->ln, batch, (uint32_t*)w.red_b.p, &nrows, s));
  } else {                                             // every power on its own, then the product
    rc = powers(k, base, exp, (uint32_t*)w.red_b.p, batch, s);
  }
  if (rc) return rc;
  CtxLock lock2_(m->mu);
  DISPATCH_NT(m->NT, rc = do_reduce_mul<NT>(m, (const uint32_t*)w.red_b.p, nrows, d_out, s));
  return rc;
}

int pai_raw_matvec_window(pai_pub* k, long ncols, long nrows, long nnz, int mag_bits, int with_neg) {
  if (!k || ncols < 0 || nrows < 0 || nnz < 0 || mag_bits < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const long tabled = with_neg ? 2 * ncols : ncols;
  return matvec_window(tabled, nrows, nnz, mag_bits, matvec_entry_bytes(k->nmod->NT));
}

int pai_raw_matvec(pai_pub* k, const uint32_t* d_c, long ncols, const int64_t* d_indptr, const int32_t* d_indices,
                   const uint32_t* d_mag, int mag_limbs, int mag_bits, const uint8_t* d_neg, long nnz, long nrows,
                   uint32_t* d_out, int32_t* d_status, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || ncols < 0 || nrows < 0 || nnz < 0 || mag_limbs < 1 || mag_bits < 0 || mag_bits > 32 * mag_limbs ||
      (nrows > 0 && (!d_indptr || !d_out)) || (nnz > 0 && (!d_c || !d_indices || !d_mag || ncols < 1))) {
    g_err = "bad argument";
    return PAI_E_ARG;
  }
  CtxLock lock_(k->mu);
  rt_stream s = (rt_stream)stream;
  int rc = rt_set_device(k->nsq->device);
  if (rc) return rc;
  StreamWs& w = k->ws.get(s);
  const bool inverses = d_neg && nnz > 0;
  if (d_status && ncols > 0 && !inverses) rc = rt_memset(d_status, 0, (size_t)ncols * 4, s);
  if (rc || nrows == 0) return rc;
  const int lc = 2 * k->ln;
  const int bits = mag_bits ? mag_bits : 32 * mag_limbs;
  const long nslots = inverses ? 2 * ncols : ncols;
  const int win = matvec_window(nslots, nrows, nnz, bits, matvec_entry_bytes(k->nmod->NT));
  int32_t* flag = nullptr;
  const uint32_t* cinv = nullptr;
  if (inverses) {   // 1. columns used with a negative scalar, 2. their inverses (the others are copied)
    rc = w.w_flag.ensure((size_t)ncols * 4 * 2);
    if (!rc) rc = w.w_base.ensure((size_t)ncols * lc * 4);
    if (!rc) rc = rt_memset(w.w_flag.p, 0, (size_t)ncols * 4, s);
    if (rc) return rc;
    flag = (int32_t*)w.w_flag.p;
    int32_t* status = d_status ? d_status : flag + ncols;
    MatFlagBody fb{nullptr, 0, d_indices, d_neg, nnz, flag};
    rc = rt_launch(fb, (int)std::min((nnz + 127) / 128, 65535L), 128, 0, s);
    if (rc) return rc;
    pai_mod* m = k->nsq;
    DISPATCH_NT(m->NT, rc = do_invert_flagged<NT>(m, d_c, flag, (uint32_t*)w.w_base.p, status, ncols, s));
    if (rc) return rc;
    cinv = (const uint32_t*)w.w_base.p;
  }
  // 3. shared window tables, 4. one thread per row
  DISPATCH_NTH(k->nmod->NT, rc = do_matvec_digit<NTH>(k, w, d_c, cinv, flag, ncols, nslots, win, d_indptr, d_indices, d_mag,
                                                      mag_limbs, inverses ? d_neg : nullptr, nnz, nrows, d_out, s));
  return rc;
}

// ---------------------------------------------------------------------------------------- private key
int pai_priv_create(const uint32_t* p, const uint32_t* q, int limbs, int device, pai_priv** out) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!p || !q || !out || limbs <= 0) { g_err = "bad argument"; return PAI_E_ARG; }
  int ep = eff_limbs(p, limbs), eq = eff_limbs(q, limbs);
  if (!ep || !eq || !(p[0] & 1u) || !(q[0] & 1u)) { g_err = "p and q must be odd"; return PAI_E_ARG; }
  int ntp = pick_ntp((std::max(ep, eq) + 7) / 8);
  if (ntp < 0) { g_err = "key too large (p and q at most 2048 bits each)"; return PAI_E_ARG; }
  const int L1 = 8 * ntp;
  limbs_t pp = padded(p, ep, L1), qq = padded(q, eq, L1);
  int c = h_cmp(pp.data(), qq.data(), L1);
  if (c == 0) { g_err = "p and q have to be different"; return PAI_E_ARG; }     // phe/paillier.py:220-222
  if (c > 0) std::swap(pp, qq);                                                   // :224-229
  pai_priv* k = new (std::nothrow) pai_priv();
  if (!k) return PAI_E_ARG;
  k->device = device; k->NTP = ntp; k->h_p = pp; k->h_q = qq;
  limbs_t p2 = h_mul(pp, pp), q2 = h_mul(qq, qq);
  int rc = mod_create_impl(p2.data(), (int)p2.size(), device, 2 * ntp, 0, &k->p2);
  if (!rc) rc = mod_create_impl(q2.data(), (int)q2.size(), device, 2 * ntp, 0, &k->q2);
  if (!rc) rc = mod_create_impl(pp.data(), L1, device, ntp, 0, &k->p1);
  if (!rc) rc = mod_create_impl(qq.data(), L1, device, ntp, 0, &k->q1);
  if (!rc) { DISPATCH_NTP(ntp, rc = do_priv_setup<NTP>(k, 0)); }
  if (!rc) { DISPATCH_NTP(ntp, rc = do_priv_digit_setup<NTP>(k, 0)); }
  // tensor-core reductions: p, q of 64 .. 256 base-256 digits (keys up to 4096 bits)
  k->family = pick_family("PAI_DECRYPT_PATH", tc_supported(ntp, 8));
  if (!rc && k->family == TC) {
    DISPATCH_TC(ntp, rc = do_priv_tc_setup<NTH>(k, 0));
    k->tc_stagger = tc_stagger_cycles();
  }
  if (rc) { pai_priv_destroy(k); return rc; }
  *out = k;
  return 0;
}
int pai_priv_destroy(pai_priv* k) {
  if (!k) return 0;
  rt_set_device(k->device);
  k->d_consts.release(true); k->d_dconsts.release(true); k->d_tc.release(true); k->d_coop_e.release(true);
  k->d_pe_consts.release(true); k->d_pe_coop_e.release(true);
  k->ws.release(true); k->h_c.release(true); k->h_m.release(true); k->h_r.release(true);
  for (pai_mod* m : {k->pd, k->qd, k->p2, k->q2, k->p1, k->q1}) mod_free(m, true);
  for (limbs_t* h : {&k->h_p, &k->h_q, &k->h_pinv, &k->h_hp, &k->h_hq}) std::fill(h->begin(), h->end(), 0);
  delete k;
  return 0;
}
int pai_priv_n_limbs(const pai_priv* k) { return k ? 16 * k->NTP : PAI_E_ARG; }
int pai_priv_c_limbs(const pai_priv* k) { return k ? 32 * k->NTP : PAI_E_ARG; }
int pai_priv_kernel_path(const pai_priv* k) { return k ? k->family : PAI_E_ARG; }
long pai_priv_wave(pai_priv* k) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k) return PAI_E_ARG;
  CtxLock lock_(k->mu);
  if (rt_set_device(k->device) || priv_wave(k)) return PAI_E_CUDA;
  return k->wave;
}
int pai_priv_get(const pai_priv* k, uint32_t* p, uint32_t* q, uint32_t* p_inverse, uint32_t* hp, uint32_t* hq) {
  if (!k) return PAI_E_ARG;
  const int ln = 16 * k->NTP, L1 = 8 * k->NTP;
  const limbs_t* src[5] = {&k->h_p, &k->h_q, &k->h_pinv, &k->h_hp, &k->h_hq};
  uint32_t* dst[5] = {p, q, p_inverse, hp, hq};
  for (int i = 0; i < 5; i++) {
    if (!dst[i]) continue;
    memset(dst[i], 0, (size_t)ln * 4);
    memcpy(dst[i], src[i]->data(), (size_t)L1 * 4);
  }
  return 0;
}
int pai_decrypt(pai_priv* k, const uint32_t* d_c, uint32_t* d_m, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || !d_c || !d_m || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(k->mu);
  if (batch == 0) return 0;
  int rc = rt_set_device(k->device);
  if (rc) return rc;
  rc = priv_wave(k);
  if (rc) return rc;
  const long ncoop = coop_rows(batch, k->wave);
  if (ncoop) {
    // both big exponentiations on one warp each (pai_coop.cuh), then L, h and the CRT in the thread-per-ciphertext form
    rt_stream s = (rt_stream)stream;
    const int L1 = 8 * k->NTP, L2 = 16 * k->NTP;
    const long off = batch - ncoop;
    rc = ensure_coop(k->p2, s);
    if (!rc) rc = ensure_coop(k->q2, s);
    if (!rc && !k->d_coop_e.p) {
      limbs_t e = h_sub_small(k->h_p, 1), eq = h_sub_small(k->h_q, 1);
      e.resize(L1, 0); eq.resize(L1, 0);
      e.insert(e.end(), eq.begin(), eq.end());
      rc = k->d_coop_e.ensure((size_t)2 * L1 * 4);
      if (!rc) rc = rt_h2d(k->d_coop_e.p, e.data(), (size_t)2 * L1 * 4, s);
      if (!rc) rc = rt_sync(s);
    }
    StreamWs& w = k->ws.get(s);
    if (!rc) rc = w.coop_u.ensure((size_t)2 * ncoop * L2 * 4);
    if (rc) return rc;
    uint32_t* up = (uint32_t*)w.coop_u.p;
    uint32_t* uq = up + (size_t)ncoop * L2;
    DISPATCH_K(k->p2->coopK, rc = do_coop_decrypt_pow<K>(k, d_c + off * 2 * L2, up, uq, ncoop, s));
    if (rc) return rc;
    DISPATCH_NTP(k->NTP, rc = do_decrypt<NTP>(k, d_c + off * 2 * L2, d_m + off * L2, ncoop, s, up, uq));
    if (rc || off == 0) return rc;
    batch = off;
  }
  return decrypt_rows(k, d_c, d_m, batch, (rt_stream)stream);
}
int pai_priv_encrypt(pai_priv* k, const uint32_t* d_m, const uint32_t* d_r, uint32_t* d_c, long batch, void* stream) {
  DeviceGuard device_guard_; (void)device_guard_;
  if (!k || !d_m || !d_r || !d_c || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  CtxLock lock_(k->mu);
  if (batch == 0) return 0;
  rt_stream s = (rt_stream)stream;
  int rc = rt_set_device(k->device);
  if (!rc && !k->d_pe_consts.p) { DISPATCH_NTP(k->NTP, rc = do_priv_enc_setup<NTP>(k, s)); }
  if (rc) return rc;
  const long ncoop = coop_rows(batch, k->pe_wave);
  if (ncoop) {
    // both exponentiations on one warp each (pai_coop.cuh), then the message factors and the CRT one thread per row
    const int L2 = 16 * k->NTP;
    const long off = batch - ncoop;
    rc = ensure_coop(k->p2, s);
    if (!rc) rc = ensure_coop(k->q2, s);
    StreamWs& w = k->ws.get(s);
    if (!rc) rc = w.coop_u.ensure((size_t)2 * ncoop * L2 * 4);
    if (rc) return rc;
    uint32_t* up = (uint32_t*)w.coop_u.p;
    uint32_t* uq = up + (size_t)ncoop * L2;
    DISPATCH_K(k->p2->coopK, rc = do_coop_priv_enc_pow<K>(k, d_r + off * L2, up, uq, ncoop, s));
    if (rc) return rc;
    DISPATCH_NTP(k->NTP, rc = do_priv_encrypt_digit<NTP>(k, d_m + off * L2, d_r + off * L2, d_c + off * 2 * L2, ncoop, s, up, uq));
    if (rc || off == 0) return rc;
    batch = off;
  }
  DISPATCH_NTP(k->NTP, rc = do_priv_encrypt_digit<NTP>(k, d_m, d_r, d_c, batch, s, nullptr, nullptr));
  return rc;
}

// ---------------------------------------------------------------------------------------- host-pointer variants

int pai_encrypt_host(pai_pub* k, const uint32_t* m, const uint32_t* r, uint32_t* c, long batch) {
  if (!k || !m || !r || !c || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const size_t bn = (size_t)batch * k->ln * 4;
  return run_staged(k->mu, k->nsq->device, batch, {{k->h_m, m, bn}, {k->h_r, r, bn}}, {{k->h_c, c, 2 * bn}},
                    [&] { return pai_encrypt(k, dev(k->h_m), dev(k->h_r), dev(k->h_c), batch, nullptr); });
}
int pai_raw_add_host(pai_pub* k, const uint32_t* a, const uint32_t* b, uint32_t* c, long batch) {
  if (!k || !a || !b || !c || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const size_t bc = (size_t)batch * 2 * k->ln * 4;
  return run_staged(k->mu, k->nsq->device, batch, {{k->h_m, a, bc}, {k->h_r, b, bc}}, {{k->h_c, c, bc}},
                    [&] { return pai_raw_add(k, dev(k->h_m), dev(k->h_r), dev(k->h_c), batch, nullptr); });
}
int pai_raw_mul_host(pai_pub* k, const uint32_t* a, const uint32_t* s, uint32_t* c, int32_t* status, long batch) {
  if (!k || !a || !s || !c || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const size_t bn = (size_t)batch * k->ln * 4;
  return run_staged(k->mu, k->nsq->device, batch, {{k->h_m, a, 2 * bn}, {k->h_s, s, bn}}, {{k->h_c, c, 2 * bn}, {k->h_r, status, (size_t)batch * 4}},
                    [&] { return pai_raw_mul(k, dev(k->h_m), dev(k->h_s), dev(k->h_c), dev<int32_t>(k->h_r), batch, nullptr); });
}
int pai_decrypt_host(pai_priv* k, const uint32_t* c, uint32_t* m, long batch) {
  if (!k || !c || !m || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const size_t bn = (size_t)batch * 16 * k->NTP * 4;
  return run_staged(k->mu, k->device, batch, {{k->h_c, c, 2 * bn}}, {{k->h_m, m, bn}},
                    [&] { return pai_decrypt(k, dev(k->h_c), dev(k->h_m), batch, nullptr); });
}
int pai_priv_encrypt_host(pai_priv* k, const uint32_t* m, const uint32_t* r, uint32_t* c, long batch) {
  if (!k || !m || !r || !c || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const size_t bn = (size_t)batch * 16 * k->NTP * 4;
  return run_staged(k->mu, k->device, batch, {{k->h_m, m, bn}, {k->h_r, r, bn}}, {{k->h_c, c, 2 * bn}},
                    [&] { return pai_priv_encrypt(k, dev(k->h_m), dev(k->h_r), dev(k->h_c), batch, nullptr); });
}
int pai_mod_mulmod_host(pai_mod* m, const uint32_t* a, const uint32_t* b, uint32_t* out, long batch) {
  if (!m || !a || !b || !out || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const size_t bl = (size_t)batch * m->L * 4;
  return run_staged(m->mu, m->device, batch, {{m->tmp_a, a, bl}, {m->tmp_b, b, bl}}, {{m->tmp_o, out, bl}},
                    [&] { return pai_mod_mulmod(m, dev(m->tmp_a), dev(m->tmp_b), dev(m->tmp_o), batch, nullptr); });
}
int pai_mod_powmod_host(pai_mod* m, const uint32_t* base, int base_limbs, const uint32_t* exp, int exp_limbs, int shared_exp,
                        uint32_t* out, long batch) {
  if (!m || !base || !exp || !out || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  const size_t bb = (size_t)batch * base_limbs * 4, bo = (size_t)batch * m->L * 4;
  if (shared_exp)     // the exponent stays in host memory (pai_mod_powmod_shared)
    return run_staged(m->mu, m->device, batch, {{m->tmp_a, base, bb}}, {{m->tmp_o, out, bo}}, [&] {
      return pai_mod_powmod_shared(m, dev(m->tmp_a), base_limbs, exp, exp_limbs, dev(m->tmp_o), batch, nullptr);
    });
  return run_staged(m->mu, m->device, batch, {{m->tmp_a, base, bb}, {m->tmp_b, exp, (size_t)batch * exp_limbs * 4}}, {{m->tmp_o, out, bo}},
                    [&] { return pai_mod_powmod(m, dev(m->tmp_a), base_limbs, dev(m->tmp_b), exp_limbs, dev(m->tmp_o), batch, nullptr); });
}
int pai_mod_invert_host(pai_mod* m, const uint32_t* a, int a_limbs, uint32_t* out, int32_t* status, long batch) {
  if (!m || !a || !out || batch < 0) { g_err = "bad argument"; return PAI_E_ARG; }
  return run_staged(m->mu, m->device, batch, {{m->tmp_a, a, (size_t)batch * a_limbs * 4}},
                    {{m->tmp_o, out, (size_t)batch * m->L * 4}, {m->tmp_s, status, (size_t)batch * 4}},
                    [&] { return pai_mod_invert(m, dev(m->tmp_a), a_limbs, dev(m->tmp_o), dev<int32_t>(m->tmp_s), batch, nullptr); });
}

}  // extern "C"
