/*
 * paillier_b200.h -- C ABI of the H100-native batched Paillier engine (libpaillier_b200.so).
 *
 * This is the drop-in boundary for the big-integer hot path of data61/python-paillier (phe 1.5.0).
 * The reference reaches its bigint engine (gmpy2 -> GMP) through three scalar functions,
 * phe/util.py:38 powmod, :53 mulmod, :85 invert, imported by name at phe/paillier.py:29 and called
 * one Python int at a time from raw_encrypt (:130,137,139), obfuscate (:622-623), raw_decrypt
 * (:346-353), crt (:373), h_function (:360), _raw_add (:719) and _raw_mul (:747-751).  The reference
 * has no batch interface; the entry points below are the batched form of exactly those call sites.
 *
 * Conventions
 *   - Big integers are little-endian arrays of uint32 limbs, row-major [batch][limbs], rows 16-byte
 *     aligned, zero padded to the context's limb counts (pai_*_limbs()).  Results are canonical
 *     residues (fully reduced; never left in Montgomery form).
 *   - Pointers named d_* are DEVICE pointers (e.g. torch tensor.data_ptr()); the *_host variants take
 *     HOST pointers and stage H2D/D2H inside the call (pinned staging, synchronous on return).
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).  Device-pointer calls are
 *     asynchronous on that stream.
 *   - Threads and streams: every entry point that takes a context locks it for the duration of the call
 *     (host-pointer variants: until their results are back in host memory), so one context may be shared by any
 *     number of host threads.  Scratch memory (window tables, work counters, intermediate rows) is kept per
 *     (context, stream): calls on different streams run concurrently on the device without sharing any of it;
 *     each stream a context is used on costs one table workspace (about 1 GB at 2048-bit keys).
 *   - Every function returns 0 on success or a negative PAI_E_* code; pai_last_error() gives text.
 *   - There is NO CPU fallback: without a CUDA device every compute call fails with PAI_E_CUDA.
 *   - Batch size needs no tuning: pai_encrypt / pai_decrypt / pai_mod_powmod_shared route a batch (or the remainder of
 *     a batch beyond whole waves of the thread-per-ciphertext kernels) of up to 0.3 wave to warp-per-ciphertext
 *     kernels with ~10x lower latency.  Environment switches, read at call time / context creation:
 *     PAI_COOP_MAX=<rows> (0 = never use the warp kernels), PAI_TC=2 (the tensor-core reductions for every size they exist
 *     for instead of the default base-n digit kernels on the integer pipe, which measure faster on the H100),
 *     PAI_TC_GROUPS=<1..4> (cap on the 128-thread groups per CTA of the tensor-core kernels; experiments and sanitizer runs),
 *     PAI_ENCRYPT_PATH=full, PAI_DECRYPT_PATH=full (full-width Montgomery kernels instead of the base-n digit kernels).
 *     All variants return identical bits.
 */
#ifndef PAILLIER_B200_H
#define PAILLIER_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PAI_OK 0
#define PAI_E_ARG (-1)      /* bad argument (null pointer, even modulus, size not supported, p >= q ...) */
#define PAI_E_CUDA (-2)     /* CUDA runtime error (no device, launch failure, out of memory) */
#define PAI_E_NOINV (-3)    /* a modular inverse needed for per-key constants does not exist */

typedef struct pai_mod pai_mod;     /* Montgomery context of one odd modulus          */
typedef struct pai_pub pai_pub;     /* public key context:  n, n^2                    */
typedef struct pai_priv pai_priv;   /* private key context: p < q, p^2, q^2, hp, hq   */

const char* pai_last_error(void);
int pai_version(void);
/* number of CUDA devices visible (0 when there is none / no driver); never fails */
int pai_device_count(void);

/* ---- generic modulus contexts: the batched form of the phe/util.py seam -------------------------
 * pai_mod_create: modulus = `limbs` uint32 limbs (odd, > 1, at most 8192 bits).  The context pads it
 * to pai_mod_limbs() limbs (a multiple of 8); all operand rows of this context have that many limbs. */
int pai_mod_create(const uint32_t* modulus, int limbs, int device, pai_mod** out);
int pai_mod_destroy(pai_mod* m);
int pai_mod_limbs(const pai_mod* m);

/* out[i] = a[i] * b[i] mod N                                  (util.mulmod, phe/util.py:53-64) */
int pai_mod_mulmod(pai_mod* m, const uint32_t* d_a, const uint32_t* d_b, uint32_t* d_out, long batch, void* stream);
/* out[i] = base[i] ^ e mod N, one exponent for the whole batch (util.powmod, phe/util.py:38-50).
 * base rows have base_limbs limbs: pai_mod_limbs() or 2*pai_mod_limbs() (a double-width base is
 * reduced first, as GMP does for raw_decrypt's powmod(c, p-1, p^2), phe/paillier.py:347). */
int pai_mod_powmod_shared(pai_mod* m, const uint32_t* d_base, int base_limbs, const uint32_t* exponent, int exp_limbs,
                          uint32_t* d_out, long batch, void* stream);
/* out[i] = base[i] ^ e[i] mod N, per-element exponents, rows of exp_limbs limbs (device) */
int pai_mod_powmod(pai_mod* m, const uint32_t* d_base, int base_limbs, const uint32_t* d_exp, int exp_limbs,
                   uint32_t* d_out, long batch, void* stream);
/* out[i] = a[i]^-1 mod N; d_status[i] = 1 where no inverse exists (util.invert raises
 * ZeroDivisionError there, phe/util.py:96-97,101-102) and out[i] = 0. */
int pai_mod_invert(pai_mod* m, const uint32_t* d_a, int a_limbs, uint32_t* d_out, int32_t* d_status, long batch, void* stream);

/* ---- public key: PaillierPublicKey (phe/paillier.py:71-194) ------------------------------------ */
int pai_pub_create(const uint32_t* n, int limbs, int device, pai_pub** out);
int pai_pub_destroy(pai_pub* k);
int pai_pub_n_limbs(const pai_pub* k);     /* Ln : limbs of plaintexts / r / scalars (multiple of 16) */
int pai_pub_c_limbs(const pai_pub* k);     /* 2*Ln: limbs of ciphertexts                              */
/* rows one full wave of the throughput encrypt kernel holds on this device (a batch that is a multiple of it wastes
 * nothing; host code that pipelines a long vector in chunks sizes the chunks with it).  No reference counterpart:
 * the reference processes one element per call (examples/federated_learning_with_encryption.py:122-133). */
long pai_pub_wave(pai_pub* k);
/* kernel family that serves pai_encrypt for this key: 0 = full-width Montgomery, 1 = base-n digit arithmetic on the
 * integer pipe (pai_digit.cuh), 2 = base-n digits with both multiplications of every Montgomery reduction on the
 * tensor cores (pai_tc.cuh; keys up to 3072 bits).  All families return identical bits; PAI_TC=2 / PAI_ENCRYPT_PATH=full
 * at context creation select family 2 / 0 instead of the default 1.  Instrumentation only (bench.py reports the MACs of the active family). */
int pai_pub_kernel_path(const pai_pub* k);

/* c[i] = (1 + n*m[i]) * r[i]^n mod n^2        raw_encrypt, phe/paillier.py:102-139
 * (= obfuscate of the nude ciphertext, :603-624).  Any m, r < 2^(32 Ln) is accepted and reduced. */
int pai_encrypt(pai_pub* k, const uint32_t* d_m, const uint32_t* d_r, uint32_t* d_c, long batch, void* stream);
/* r[i] uniform in [1, n), the batched form of get_random_lt_n (phe/paillier.py:141-143): ChaCha20 keystream of
 * the 32-byte seed (take it from the OS CSPRNG) and the 64-bit nonce (distinct per call), rejection sampled on the
 * device.  d_r: [batch][pai_pub_n_limbs()]. */
int pai_random_lt_n(pai_pub* k, const uint8_t* seed32, unsigned long long nonce, uint32_t* d_r, long batch, void* stream);
/* c[i] = a[i] * b[i] mod n^2                  _raw_add, phe/paillier.py:705-719 */
int pai_raw_add(pai_pub* k, const uint32_t* d_a, const uint32_t* d_b, uint32_t* d_c, long batch, void* stream);
/* c[i] = a[i] ^ s[i] mod n^2 for 0 <= s[i] < n, with the reference's negative-scalar branch
 * (s >= n - max_int: invert(a, n^2) ^ (n - s)); d_status[i] = 1 where that inverse does not exist.
 *                                             _raw_mul, phe/paillier.py:721-751 */
int pai_raw_mul(pai_pub* k, const uint32_t* d_a, const uint32_t* d_s, uint32_t* d_c, int32_t* d_status, long batch, void* stream);

/* out = c[0] * c[1] * ... * c[batch-1] mod n^2 (one row): the homomorphic SUM of a whole ciphertext vector in two
 * launches -- every thread multiplies its share of the rows in the Montgomery domain (entered once), the CTAs fold
 * their threads' partial products in shared memory, a second launch folds the CTAs'.  The reference's idiom is
 * sum(list_of_EncryptedNumber) / np.mean(...) = batch-1 sequential _raw_add calls (phe/tests/math_test.py:44-58,
 * phe/paillier.py:705-719).  batch >= 1. */
int pai_raw_sum(pai_pub* k, const uint32_t* d_c, long batch, uint32_t* d_out, void* stream);

/* out = prod_i a[i]^s[i] mod n^2 (one row): the encrypted DOT PRODUCT of a ciphertext vector with plaintext scalars
 * 0 <= s[i] < n, with _raw_mul's negative-scalar branch per element (d_status as in pai_raw_mul; may be NULL).  On the
 * tensor-core kernel family the powers are taken by Straus' simultaneous exponentiation (one squaring chain shared by
 * the group of elements a thread owns), then pai_raw_sum's reduction folds the groups.  The reference's idiom is
 * sum(w_i * x_i) over EncryptedNumbers = one _raw_mul and one _raw_add per element
 * (examples/logistic_regression_encrypted_model.py:170-180, phe/tests/math_test.py:50-58).  batch >= 1. */
int pai_raw_dot(pai_pub* k, const uint32_t* d_a, const uint32_t* d_s, uint32_t* d_out, int32_t* d_status, long batch, void* stream);

/* out[j] = prod_{t = indptr[j]}^{indptr[j+1]-1} ( neg[t] ? c[indices[t]]^-1 : c[indices[t]] ) ^ mag[t]  mod n^2
 * A plaintext matrix in CSR form times a ciphertext vector: the encrypted scoring loop of
 * examples/logistic_regression_encrypted_model.py:170-180 (score += x[0, i] * weights[i] over the nonzeros of a row) for
 * every row at once.  c: [ncols][pai_pub_c_limbs()].  indptr: [nrows + 1] int64; indices: [nnz] int32 column numbers in
 * [0, ncols).  mag: [nnz][mag_limbs] magnitudes, 0 <= mag < n.  mag_bits: a bound on the bit length of every magnitude
 * (0 = 32 * mag_limbs); it only steers the choice of the window width (a 0/1 matrix passes 1).
 * Scalars are sign and magnitude, not residues as in pai_raw_mul's s: the reference's rule for an encoding s
 * (phe/paillier.py:742-749: s >= n - max_int -> base invert(c, n^2), exponent n - s) becomes neg = 1, mag = n - s; any
 * other s is neg = 0, mag = s.  neg: [nnz] uint8, or NULL when every scalar is non-negative.
 * status: [ncols] (may be NULL), 1 where c[i] is used with a negative scalar and has no inverse mod n^2 (the outputs of
 * the rows that use it are then unspecified), else 0.  Rows with no entries give 1.
 * Window tables c^1 .. c^(2^w - 1) are built once per column (and per inverse) and shared by all rows; every row runs
 * one squaring chain for all its entries (Straus).  w comes from pai_raw_matvec_window.  One thread per row: a 1 x d
 * product is latency bound, pai_raw_dot is the tool for it.  Asynchronous on `stream`; no host synchronisation. */
int pai_raw_matvec(pai_pub* k, const uint32_t* d_c, long ncols, const int64_t* d_indptr, const int32_t* d_indices,
                   const uint32_t* d_mag, int mag_limbs, int mag_bits, const uint8_t* d_neg, long nnz, long nrows,
                   uint32_t* d_out, int32_t* d_status, void* stream);
/* the window width 1..8 pai_raw_matvec picks for these shapes (bits = mag_bits, or 32 * mag_limbs; with_neg: d_neg given) */
int pai_raw_matvec_window(pai_pub* k, long ncols, long nrows, long nnz, int bits, int with_neg);

/* ---- private key: PaillierPrivateKey (phe/paillier.py:197-380) ---------------------------------
 * p, q: `limbs` limbs each, p*q = n.  Ordered internally so that p < q (:224-229).  All derived
 * constants (p^2, q^2, p^-1 mod q, hp, hq; :230-235) are computed by the engine on the device. */
int pai_priv_create(const uint32_t* p, const uint32_t* q, int limbs, int device, pai_priv** out);
int pai_priv_destroy(pai_priv* k);
int pai_priv_n_limbs(const pai_priv* k);
int pai_priv_c_limbs(const pai_priv* k);
long pai_priv_wave(pai_priv* k);            /* as pai_pub_wave, for the decrypt kernel */
int pai_priv_kernel_path(const pai_priv* k);   /* as pai_pub_kernel_path (tensor-core family: keys up to 4096 bits) */
/* copies of the derived constants (host buffers of pai_priv_n_limbs() limbs each; NULL = skip):
 * p, q (ordered), p_inverse, hp, hq -- for the drop-in key object's attributes */
int pai_priv_get(const pai_priv* k, uint32_t* p, uint32_t* q, uint32_t* p_inverse, uint32_t* hp, uint32_t* hq);
/* m[i] = raw_decrypt(c[i]) with CRT             phe/paillier.py:328-374 */
int pai_decrypt(pai_priv* k, const uint32_t* d_c, uint32_t* d_m, long batch, void* stream);
/* c[i] = (1 + n*m[i]) * r[i]^n mod n^2 for whatever integers the rows hold: the value pai_encrypt returns for the same
 * integers, bit for bit, computed with the private key.  m, r: [batch][pai_priv_n_limbs()]; c: [batch][pai_priv_c_limbs()]
 * (the layout of pai_decrypt).  The key holder's encryption: r^n mod p^2 and mod q^2 from half-length exponentiations
 * (s = (r mod x)^(y mod (x-1)) mod x, then s^x mod x^2 for x, y = p, q and q, p), the message factor per prime, and
 * Garner's CRT to n^2.  Secret exponents run through fixed windows with no digit skipped.  The result is defined for
 * prime p and q, like pai_decrypt's; pai_priv_create does not test primality.  The per-key constants are derived on the
 * first call.  Small batches and the tail beyond whole waves take warp-per-ciphertext exponentiations (PAI_COOP_MAX as
 * for pai_encrypt).  Always on the integer-pipe digit kernels, whatever PAI_TC / PAI_DECRYPT_PATH select.  Asynchronous
 * on `stream`, except for the first call, which waits for the constants' upload. */
int pai_priv_encrypt(pai_priv* k, const uint32_t* d_m, const uint32_t* d_r, uint32_t* d_c, long batch, void* stream);

/* ---- decimal wire format: the radix conversion behind the reference's JSON serialisation ---------
 * (docs/serialisation.rst:24-42 ships ciphertexts as str(int); phe/command_line.py:120-131, 267-276 likewise.)
 * Text rows are fixed-width fields of pai_decimal_width(limbs) ASCII digits, right aligned, '0' padded, row-major
 * [batch][width], device memory.  pai_decimal_to_limbs accepts any width; d_status[i] (may be NULL) = 1 where a row
 * holds a character that is not a digit, 2 where the value needs more than `limbs` limbs (the row is zeroed). */
int pai_decimal_width(int limbs);
int pai_limbs_to_decimal(const uint32_t* d_limbs, int limbs, uint8_t* d_text, long batch, int device, void* stream);
int pai_decimal_to_limbs(const uint8_t* d_text, int width, uint32_t* d_limbs, int limbs, int32_t* d_status, long batch, int device,
                         void* stream);

/* ---- packed fixed-point plaintexts: many signed values per ciphertext --------------------------------------
 * No reference counterpart (BatchCrypt-style packing; DESIGN.md §3.10).  A plaintext row holds K = (bits(n) - 1) / slot_bits
 * signed slots s_j with |s_j| <= 2^(slot_bits-1) - 1 as P = sum_j s_j * 2^(slot_bits*j), stored as P mod n.  Then
 * |P| < 2^(bits(n)-2) < n/2, and raw_add / raw_mul by an integer act on every slot while the slots stay within that bound.  Slot j of row r
 * is value r*K + j of a flat int64 array.  Asynchronous on `stream`; no workspace. */
/* K for this key, or PAI_E_ARG for slot_bits outside 2..63 or when not even one slot fits */
int pai_pack_slots_per_row(const pai_pub* k, int slot_bits);
/* m[r] = (sum_j s[r*K + j] * 2^(slot_bits*j)) mod n for r < ceil(count / K), missing slots 0.  d_status[r] = 1 where a slot
 * of row r is outside (-2^(slot_bits-1), 2^(slot_bits-1)); that row is zeroed.  m: [rows][pai_pub_n_limbs()]. */
int pai_pack_slots(pai_pub* k, const int64_t* d_slots, long count, int slot_bits, uint32_t* d_m, int32_t* d_status, void* stream);
/* inverse: centre-lift mod n (m <= (n-1)/2: P = m, else m - n), balanced base-2^slot_bits digits into the first `count`
 * slots; d_status[r] = 1 where row r is not a packing (m >= n, a digit -2^(slot_bits-1), or a nonzero part above slot
 * K-1), its slots are zeroed.  It accepts exactly the rows pai_pack_slots produces. */
int pai_unpack_slots(pai_pub* k, const uint32_t* d_m, int slot_bits, int64_t* d_slots, long count, int32_t* d_status, void* stream);

/* ---- batched primality testing for key generation ----------------------------------------------------------
 * result[i] = 1 if candidate i passes `rounds` Miller-Rabin rounds with the bases given, 0 if it is composite:
 * util.miller_rabin (phe/util.py:381-417) for a whole batch of candidates, one thread per candidate, each with its own
 * Montgomery constants.  The reference's getprimeover / is_prime (phe/util.py:106-124, 420-443) test one candidate at a
 * time.  cand: [batch][limbs] (limbs a multiple of 8, candidates odd; trial division by small primes stays on the host);
 * bases: [batch][rounds][limbs] random rows (reduced by the kernel; the caller draws them from a CSPRNG).
 * Synchronous on return (device pointers). */
int pai_miller_rabin(const uint32_t* d_cand, int limbs, const uint32_t* d_bases, int rounds, int32_t* d_result, long batch, int device,
                     void* stream);

/* ---- host-pointer convenience variants (H2D + kernel + D2H inside; synchronous) ---------------- */
int pai_encrypt_host(pai_pub* k, const uint32_t* m, const uint32_t* r, uint32_t* c, long batch);
int pai_raw_add_host(pai_pub* k, const uint32_t* a, const uint32_t* b, uint32_t* c, long batch);
int pai_raw_mul_host(pai_pub* k, const uint32_t* a, const uint32_t* s, uint32_t* c, int32_t* status, long batch);
int pai_decrypt_host(pai_priv* k, const uint32_t* c, uint32_t* m, long batch);
int pai_priv_encrypt_host(pai_priv* k, const uint32_t* m, const uint32_t* r, uint32_t* c, long batch);
int pai_mod_mulmod_host(pai_mod* m, const uint32_t* a, const uint32_t* b, uint32_t* out, long batch);
int pai_mod_powmod_host(pai_mod* m, const uint32_t* base, int base_limbs, const uint32_t* exp, int exp_limbs, int shared_exp,
                        uint32_t* out, long batch);
int pai_mod_invert_host(pai_mod* m, const uint32_t* a, int a_limbs, uint32_t* out, int32_t* status, long batch);

/* ---- instrumentation ---------------------------------------------------------------------------
 * number of kernels this library has launched since load (for bench.py's gpu_launches) */
long pai_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* PAILLIER_B200_H */
