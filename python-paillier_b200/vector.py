"""EncryptedVector: a batch of Paillier ciphertexts resident in GPU memory.

The reference has no vector type: callers loop over scalars (examples/federated_learning_with_encryption.py
:122-133, phe/tests/math_test.py:44-58).  This is the batched form of exactly those loops -- one kernel
launch per vector operation, ciphertexts stay in HBM as [B, c_limbs] uint32 limb matrices and are
only converted to Python ints on request.  Semantics per element are those of EncryptedNumber
(exponent alignment before add, phe/paillier.py:695-700; lazy obfuscation, :565-566).
"""
import fractions
import math
import numbers
import operator
import os

import numpy as np

from .encoding import EncodedNumber
from .engine import ints_to_limbs, limbs_to_ints, limbs_to_decimal_dev, decimal_to_limbs_dev, decimal_width


def _torch():
    import torch
    return torch


def _to_dev(arr, ctx):
    """numpy uint32 limb matrix -> torch.int32 tensor on the context's GPU (host tensor only for the test-only
    simulation build, whose "device" pointers are host pointers)."""
    torch = _torch()
    t = torch.from_numpy(np.ascontiguousarray(arr).view(np.int32).copy())
    return t if ctx.eng.simulated else t.to("cuda:%d" % ctx.device, non_blocking=False)


def _to_host(t):
    return t.cpu().numpy().view(np.uint32)


def _stream(ctx):
    """The CUDA stream the engine kernels of this call are launched on: torch's CURRENT stream of the context's
    device, so that they are ordered with the surrounding torch work (allocations, fills, index ops, .cpu()) also
    inside ``with torch.cuda.stream(s)``.  The engine keeps its scratch memory per (context, stream)."""
    if ctx.eng.simulated:
        return None
    return int(_torch().cuda.current_stream(ctx.device).cuda_stream)


def _rows_for(ctx_limbs, t):
    """Zero-pad (or trim all-zero columns of) a device limb matrix to `ctx_limbs` columns."""
    have = int(t.shape[1])
    if have == ctx_limbs:
        return t
    torch = _torch()
    if have < ctx_limbs:
        return torch.nn.functional.pad(t, (0, ctx_limbs - have)).contiguous()
    return t[:, :ctx_limbs].contiguous()


def limbs_to_decimal_strings(ctx, d_limbs):
    """Device limb matrix -> list of decimal strings (str(int) of every row), converted on the GPU."""
    torch = _torch()
    count, limbs = int(d_limbs.shape[0]), int(d_limbs.shape[1])
    if not count:
        return []
    width = decimal_width(limbs, ctx.eng)
    d_text = torch.empty((count, width), dtype=torch.uint8, device=d_limbs.device)
    limbs_to_decimal_dev(d_limbs, limbs, d_text, count, ctx.device, stream=_stream(ctx), engine=ctx.eng)
    raw = d_text.cpu().numpy().tobytes()
    return [(raw[i * width:(i + 1) * width].lstrip(b"0") or b"0").decode("ascii") for i in range(count)]


def decimal_strings_to_limbs(ctx, strings, limbs):
    """List of decimal strings -> device limb matrix [len, limbs] (int() of every string, on the GPU).
    ValueError for anything that is not a non-negative decimal integer fitting `limbs` limbs."""
    torch = _torch()
    count = len(strings)
    width = max([len(t) for t in strings] + [1])
    raw = b"".join(t.encode("ascii").rjust(width, b"0") if isinstance(t, str) else bytes(t).rjust(width, b"0") for t in strings)
    text = np.frombuffer(raw, dtype=np.uint8).reshape(count, width)
    t = torch.from_numpy(text.copy())
    d_text = t if ctx.eng.simulated else t.to("cuda:%d" % ctx.device)
    d_limbs = torch.empty((count, limbs), dtype=torch.int32, device=d_text.device)
    d_status = torch.zeros((count,), dtype=torch.int32, device=d_text.device)
    if count:
        decimal_to_limbs_dev(d_text, width, d_limbs, limbs, d_status, count, ctx.device, stream=_stream(ctx), engine=ctx.eng)
        bad = torch.nonzero(d_status).flatten()
        if bad.numel():
            i = int(bad[0])
            raise ValueError("value %d is not a decimal integer below 2**%d" % (i, 32 * limbs))
    return d_limbs


def random_r_values(n, count):
    """count values uniform in [1, n) from os.urandom (64 surplus bits: bias < 2^-64), the batched
    counterpart of PaillierPublicKey.get_random_lt_n (phe/paillier.py:141-143)."""
    nbytes = (n.bit_length() + 7) // 8 + 8
    raw = os.urandom(nbytes * count)
    span = n - 1
    return [1 + int.from_bytes(raw[i * nbytes:(i + 1) * nbytes], "little") % span for i in range(count)]


# ------------------------------------------------------------------------------------------------------
# Vectorised EncodedNumber.encode / decode: numpy fast paths that give exactly
# the values phe/encoding.py:110-233 computes element by element, with a per-element fallback for
# everything outside the fast path (huge mantissas, precision=..., non-finite values, ints beyond 63 bits).
def _limbs_from_signed(int_rep, n, ln):
    """[B] int64 signed integers -> [B, ln] uint32 limbs of (int_rep mod n), assuming |int_rep| < 2^63 < n."""
    mag = np.abs(int_rep).astype(np.uint64)
    neg = int_rep < 0
    out = np.zeros((int_rep.shape[0], ln), dtype=np.uint32)
    out[:, 0] = (mag & np.uint64(0xffffffff)).astype(np.uint32)
    if ln > 1:
        out[:, 1] = (mag >> np.uint64(32)).astype(np.uint32)
    if neg.any():
        nl = ints_to_limbs([n], ln)[0]
        n_low = np.uint64(int(nl[0]) | ((int(nl[1]) << 32) if ln > 1 else 0))
        m = mag[neg]
        low = n_low - m                                   # wraps modulo 2^64
        borrow = m > n_low
        rows = np.tile(nl, (m.shape[0], 1))
        rows[:, 0] = (low & np.uint64(0xffffffff)).astype(np.uint32)
        if ln > 1:
            rows[:, 1] = (low >> np.uint64(32)).astype(np.uint32)
        j = 2
        while j < ln and borrow.any():
            cur = rows[:, j]
            rows[:, j] = np.where(borrow, cur - np.uint32(1), cur)
            borrow = borrow & (cur == 0)
            j += 1
        out[neg] = rows
    return out


def _encode_fast(public_key, values, max_exponent=None):
    """The numpy fast path of encode_batch: (signed integer representations [B] int64, exponents [B] int64), or None
    when the values need the per-element path."""
    arr = None
    if public_key.n.bit_length() > 80:
        if isinstance(values, np.ndarray) and values.dtype in (np.float64, np.int64, np.int32):
            arr = values
        elif len(values) and all(type(v) is float for v in values):
            arr = np.asarray(values, dtype=np.float64)
        elif len(values) and all(type(v) is int and -2 ** 62 < v < 2 ** 62 for v in values):
            arr = np.asarray(values, dtype=np.int64)
    if arr is not None and arr.dtype == np.float64 and np.isfinite(arr).all():
        m, e = np.frexp(arr)
        mant = np.ldexp(m, 53).astype(np.int64)                       # exact 53-bit signed mantissa
        lsb = e.astype(np.int64) - 53                                 # weight of the last mantissa bit
        exps = np.floor_divide(lsb, 4)                                # floor(lsb / log2(16)), phe/encoding.py:167-174
        if max_exponent is not None:
            exps = np.minimum(exps, np.asarray(max_exponent, dtype=np.int64))
        shift = lsb - 4 * exps
        if (shift <= 9).all():                                        # |int_rep| < 2^62
            return np.left_shift(mant, shift), exps
    elif arr is not None and arr.dtype != np.float64:
        exps = np.zeros(arr.shape[0], dtype=np.int64)
        if max_exponent is None or (np.asarray(max_exponent) >= 0).all():
            return arr.astype(np.int64), exps
    return None


def encode_batch(public_key, values, precision=None, max_exponent=None):
    """Encode a sequence like EncodedNumber.encode does element by element.
    Returns (limbs [B, n_limbs] uint32 of the encodings, exponents [B] int64)."""
    ctx = public_key.engine_context()
    ln = ctx.n_limbs
    if precision is None:
        fast = _encode_fast(public_key, values, max_exponent)
        if fast is not None:
            return _limbs_from_signed(fast[0], public_key.n, ln), fast[1]
    if isinstance(max_exponent, (list, tuple, np.ndarray)):
        mex = [int(x) for x in max_exponent]
    else:
        mex = [max_exponent] * len(values)
    vals = values.tolist() if isinstance(values, np.ndarray) else values
    encs = [v if isinstance(v, EncodedNumber) else EncodedNumber.encode(public_key, v, precision, mx)
            for v, mx in zip(vals, mex)]
    return (ints_to_limbs([x.encoding for x in encs], ln), np.array([x.exponent for x in encs], dtype=np.int64))


def decode_batch(public_key, limbs, exponents):
    """Decode plaintext limbs [B, n_limbs] with exponents [B] like EncodedNumber.decode; returns a list."""
    n = public_key.n
    ln = limbs.shape[1]
    count = limbs.shape[0]
    out = [None] * count
    exps = np.asarray(exponents, dtype=np.int64)
    small_pos = ~limbs[:, 2:].any(axis=1) if ln > 2 else np.ones(count, dtype=bool)
    low = limbs[:, 0].astype(np.uint64) | (limbs[:, 1].astype(np.uint64) << np.uint64(32)) if ln > 1 else limbs[:, 0].astype(np.uint64)
    # negatives are stored as n - |x| (phe/encoding.py:217-219): |x| = n - enc fits 64 bits exactly when the limbs above
    # the low pair equal those of n (no borrow out of the low pair) or of n - 2^64 (borrow)
    nl = ints_to_limbs([n], ln)[0]
    neg_small = np.zeros(count, dtype=bool)
    neg_mag = np.zeros(count, dtype=np.uint64)
    rest = np.nonzero(~small_pos)[0]
    if len(rest) and ln > 2 and n >> 64:
        n_low = int(n & (2 ** 64 - 1))
        hi0 = nl[2:]
        hi1 = ints_to_limbs([(n >> 64) - 1], ln - 2)[0]
        sub = limbs[rest]
        lo = low[rest]
        no_borrow = lo <= np.uint64(n_low)
        same0 = (sub[:, 2:] == hi0).all(axis=1)
        same1 = (sub[:, 2:] == hi1).all(axis=1)
        ok = np.where(no_borrow, same0, same1)
        neg_small[rest] = ok
        neg_mag[rest] = np.uint64(n_low) - lo              # modulo 2^64: the borrow is what `same1` accounts for
    fast = (small_pos | neg_small) & (exps < 0) & (exps > -250) & (public_key.max_int > 2 ** 64)
    if fast.any():
        mag = np.where(small_pos, low, neg_mag)
        val = np.ldexp(mag.astype(np.float64), (4 * exps).astype(np.int32)) if EncodedNumber.BASE == 16 else None
        val = np.where(small_pos, val, -val)
        if fast.all():
            out = val.tolist()
        else:
            for i, v in zip(np.nonzero(fast)[0].tolist(), val[fast].tolist()):
                out[i] = v
    slow = np.nonzero(~fast)[0]
    if len(slow):
        encs = limbs_to_ints(limbs[slow])
        for i, enc in zip(slow, encs):
            out[i] = EncodedNumber(public_key, enc, int(exps[i])).decode()
    return out


# ------------------------------------------------------------------------------------------------------
# Host preparation of EncryptedVector.rmatmul: sign-and-magnitude scalars with the exponent alignment folded in.
def _is_sparse(X):
    try:
        import scipy.sparse as sp
    except ImportError:
        return False
    return sp.issparse(X)


def _plain_values(a):
    """Matrix entries as encode_batch takes them: float64 for every float dtype and int64 for integer and bool dtypes that
    fit it (both give the encodings EncodedNumber.encode gives their Python values), Python objects otherwise."""
    k = a.dtype.kind
    if k == "f":
        return a.astype(np.float64)
    if k in "bi" or (k == "u" and (a.size == 0 or int(a.max()) < 2 ** 63)):
        return a.astype(np.int64)
    return a.astype(object)


def _signed_encodings(public_key, values):
    """encode_batch of `values` as sign and magnitude: (neg [B] bool, mag, exponents [B] int64).  mag is a uint64 array on
    encode_batch's fast path (|int_rep| < 2^62), else a list of Python ints from the per-element path; an encoding s
    is negative where s >= n - max_int, with magnitude n - s (phe/paillier.py:742-749)."""
    fast = _encode_fast(public_key, values)
    if fast is not None:
        int_rep, exps = fast
        return int_rep < 0, np.abs(int_rep).astype(np.uint64), exps
    limbs, exps = encode_batch(public_key, values)
    n, thr = public_key.n, public_key.n - public_key.max_int
    encs = limbs_to_ints(limbs)
    return np.array([e >= thr for e in encs], dtype=bool), [n - e if e >= thr else e for e in encs], exps


def _bitlen64(x):
    """bit lengths of a uint64 array (exact: each 32-bit half converts to float64 without rounding)"""
    def bl32(v):
        return np.frexp(v.astype(np.float64))[1].astype(np.int64)
    hi = x >> np.uint64(32)
    return np.where(hi > 0, 32 + bl32(hi), bl32(x & np.uint64(0xffffffff)))


def _aligned_magnitudes(public_key, mag, delta):
    """|k| * BASE^delta of every entry as a limb matrix: (limbs per row L, bit bound, uint32 [B, L]).  On the fast path
    the shift by 4*delta bits is done on numpy words; a product above max_int raises dot()'s ValueError."""
    max_int = public_key.max_int
    shift = delta.astype(np.int64) * int(EncodedNumber.LOG2_BASE)

    def too_big(m, s):
        raise ValueError('Integer needs to be within +/- %d but got %d' % (max_int, m << s))
    if isinstance(mag, np.ndarray):
        tb = _bitlen64(mag) + shift
        for i in np.nonzero(tb >= max_int.bit_length())[0].tolist():       # at or above the bound: exact check
            if int(mag[i]) << int(shift[i]) > max_int:
                too_big(int(mag[i]), int(shift[i]))
        bits = int(tb.max()) if len(tb) else 1
        L = max(1, (bits + 31) // 32)
        q, r = shift // 32, (shift % 32).astype(np.uint64)
        m32 = np.uint64(0xffffffff)
        a, b = (mag & m32) << r, (mag >> np.uint64(32)) << r                 # each below 2^63
        # words q, q+1, q+2 of every row through a flat index (two spare columns: words above the bound are zero)
        out = np.zeros((len(mag), L + 2), dtype=np.uint32)
        flat = out.reshape(-1)
        at = np.arange(len(mag), dtype=np.int64) * (L + 2) + q
        flat[at] = (a & m32).astype(np.uint32)
        flat[at + 1] = ((a >> np.uint64(32)) | (b & m32)).astype(np.uint32)
        flat[at + 2] = (b >> np.uint64(32)).astype(np.uint32)
        out = np.ascontiguousarray(out[:, :L])
        return L, max(bits, 1), out
    vals = []
    for m, s in zip(mag, shift.tolist()):
        if m << s > max_int:
            too_big(m, s)
        vals.append(m << s)
    bits = max([v.bit_length() for v in vals] + [1])
    L = (bits + 31) // 32
    return L, bits, ints_to_limbs(vals, L)


def _arr_to_dev(arr, ctx):
    """numpy array (any dtype) -> torch tensor on the context's GPU (host tensor for the simulation build)"""
    t = _torch().from_numpy(np.ascontiguousarray(arr))
    return t if ctx.eng.simulated else t.to("cuda:%d" % ctx.device)


class EncryptedVector(object):
    __array_ufunc__ = None          # numpy_array + vector / numpy_array * vector defer to __radd__ / __rmul__

    def __init__(self, public_key, limbs, exponents, obfuscated=False):
        self.public_key = public_key
        self.limbs = limbs                                  # torch.int32 [B, c_limbs] on the key's device
        self.exponents = np.asarray(exponents, dtype=np.int64)
        self._obfuscated = obfuscated

    # ------------------------------------------------------------------ construction
    @classmethod
    def encrypt(cls, public_key, values, precision=None, r_values=None, private_key=None):
        """Encode every value (EncodedNumber.encode) and encrypt the batch in one launch.  With
        r_values None each element gets a fresh random r and is therefore already obfuscated.  With the private key
        given, the encryption runs through the CRT (pai_priv_encrypt) and gives the same ciphertexts."""
        if len(values) and any(isinstance(v, EncodedNumber) for v in (values if not isinstance(values, np.ndarray) else [])):
            encs = [v if isinstance(v, EncodedNumber) else EncodedNumber.encode(public_key, v, precision) for v in values]
            return cls.encrypt_encoded(public_key, [e.encoding for e in encs], [e.exponent for e in encs], r_values, private_key)
        limbs, exps = encode_batch(public_key, values, precision)
        return cls._encrypt_limbs(public_key, limbs, exps, r_values, private_key)

    @classmethod
    def encrypt_encoded(cls, public_key, encodings, exponents, r_values=None, private_key=None):
        ctx = public_key.engine_context()
        return cls._encrypt_limbs(public_key, ints_to_limbs([e % public_key.n for e in encodings], ctx.n_limbs), exponents, r_values,
                                  private_key)

    @classmethod
    def _encrypt_limbs(cls, public_key, m_limbs, exponents, r_values=None, private_key=None):
        return cls._encrypt_dev_rows(public_key, _to_dev(m_limbs, public_key.engine_context()), exponents, r_values, private_key)

    @classmethod
    def _encrypt_dev_rows(cls, public_key, d_m, exponents, r_values=None, private_key=None):
        """Encrypt the plaintext rows d_m [B, n_limbs] (int32, on the key's device) in one launch."""
        ctx = public_key.engine_context()
        count = int(d_m.shape[0])
        obf = r_values is None
        torch = _torch()
        if r_values is None:
            # fresh obfuscators drawn on the device from a ChaCha20 stream keyed by os.urandom (pai_rng.cuh)
            d_r = torch.empty((count, ctx.n_limbs), dtype=torch.int32, device=d_m.device)
            if count:
                ctx.random_lt_n_dev(d_r, count, stream=_stream(ctx))
        else:
            d_r = _to_dev(ints_to_limbs(list(r_values), ctx.n_limbs), ctx)
        if private_key is not None:
            # the private context sizes its rows from max(p, q): re-pad the rows in, trim the all-zero columns out
            pctx = private_key.engine_context()
            d_c = torch.empty((count, pctx.c_limbs), dtype=torch.int32, device=d_m.device)
            if count:
                pctx.encrypt_dev(_rows_for(pctx.n_limbs, d_m), _rows_for(pctx.n_limbs, d_r), d_c, count, stream=_stream(pctx))
            return cls(public_key, _rows_for(ctx.c_limbs, d_c), exponents, obfuscated=obf)
        d_c = torch.empty((count, ctx.c_limbs), dtype=torch.int32, device=d_m.device)
        if count:
            ctx.encrypt_dev(d_m, d_r, d_c, count, stream=_stream(ctx))
        return cls(public_key, d_c, exponents, obfuscated=obf)

    @classmethod
    def from_encrypted_numbers(cls, numbers):
        pk = numbers[0].public_key
        ctx = pk.engine_context()
        limbs = _to_dev(ints_to_limbs([x.ciphertext(be_secure=False) % pk.nsquare for x in numbers], ctx.c_limbs), ctx)
        return cls(pk, limbs, [x.exponent for x in numbers])

    # ------------------------------------------------------------------ access
    def __len__(self):
        return int(self.limbs.shape[0])

    def ciphertexts(self, be_secure=True):
        if be_secure and not self._obfuscated:
            self.obfuscate()
        return limbs_to_ints(_to_host(self.limbs))

    def to_encrypted_numbers(self, be_secure=False):
        from .paillier import EncryptedNumber
        out = []
        for c, e in zip(self.ciphertexts(be_secure), self.exponents.tolist()):
            x = EncryptedNumber(self.public_key, c, int(e))
            if self._obfuscated:
                x._mark_obfuscated()
            out.append(x)
        return out

    def __getitem__(self, i):
        """v[int] -> EncryptedNumber (only that row leaves the device); v[slice / index array / mask] -> EncryptedVector."""
        import numbers
        if isinstance(i, numbers.Integral) and not isinstance(i, (bool, np.bool_)):
            from .paillier import EncryptedNumber
            k = operator.index(i)
            if k < 0:
                k += len(self)
            if not 0 <= k < len(self):
                raise IndexError("EncryptedVector index out of range")
            x = EncryptedNumber(self.public_key, limbs_to_ints(_to_host(self.limbs[k:k + 1]))[0], int(self.exponents[k]))
            if self._obfuscated:
                x._mark_obfuscated()
            return x
        if isinstance(i, np.ndarray):
            i = _torch().from_numpy(i).to(self.limbs.device)
            exps = self.exponents[i.cpu().numpy()]
        else:
            exps = self.exponents[i]
        return EncryptedVector(self.public_key, self.limbs[i].contiguous(), exps, self._obfuscated)

    def obfuscate(self):
        """c_i <- c_i * r_i^n mod n^2 with fresh r_i (phe/paillier.py:603-624): K1 with m = 0, then K3."""
        ctx = self.public_key.engine_context()
        count = len(self)
        if count:
            torch = _torch()
            d_r = torch.empty((count, ctx.n_limbs), dtype=torch.int32, device=self.limbs.device)
            ctx.random_lt_n_dev(d_r, count, stream=_stream(ctx))
            d_zero = torch.zeros((count, ctx.n_limbs), dtype=torch.int32, device=self.limbs.device)
            d_rn = torch.empty_like(self.limbs)
            ctx.encrypt_dev(d_zero, d_r, d_rn, count, stream=_stream(ctx))
            out = torch.empty_like(self.limbs)
            ctx.raw_add_dev(self.limbs, d_rn, out, count, stream=_stream(ctx))
            self.limbs = out
        self._obfuscated = True

    # ------------------------------------------------------------------ arithmetic
    def _raw_mul_rows(self, limbs, scalars):
        """limbs[i] ^ scalars[i] mod n^2 (device), scalars: list of ints in [0, n) or their limb matrix."""
        ctx = self.public_key.engine_context()
        torch = _torch()
        count = int(limbs.shape[0])
        d_s = _to_dev(scalars if isinstance(scalars, np.ndarray) else ints_to_limbs(scalars, ctx.n_limbs), ctx)
        out = torch.empty_like(limbs)
        status = torch.zeros((count,), dtype=torch.int32, device=limbs.device)
        ctx.raw_mul_dev(limbs, d_s, out, status, count, stream=_stream(ctx))
        if bool(status.any().item()):
            raise ZeroDivisionError('invert() no inverse exists')
        return out

    def decrease_exponent_to(self, new_exps):
        """Per-element exponent alignment: elements whose exponent is above new_exps[i] are raised to
        BASE^(delta) (phe/paillier.py:570-601); the others are untouched."""
        new_exps = np.broadcast_to(np.asarray(new_exps, dtype=np.int64), self.exponents.shape)
        if np.any(new_exps > self.exponents):
            raise ValueError('New exponent should be more negative than old exponent')
        idx = np.nonzero(new_exps < self.exponents)[0]
        limbs = self.limbs
        if len(idx):
            torch = _torch()
            ctx = self.public_key.engine_context()
            tidx = torch.from_numpy(idx).to(limbs.device)
            # the scalar BASE**delta is a small positive int: its encoding is the integer itself (exponent 0), so the
            # scalar limb matrix is built per distinct delta without touching EncodedNumber for every element
            deltas = (self.exponents[idx] - new_exps[idx]).astype(np.int64)
            scal = np.zeros((len(idx), ctx.n_limbs), dtype=np.uint32)
            for d in np.unique(deltas):
                factor = pow(EncodedNumber.BASE, int(d))
                if factor > self.public_key.max_int:
                    raise ValueError('Integer needs to be within +/- %d but got %d' % (self.public_key.max_int, factor))
                scal[deltas == d] = ints_to_limbs([factor], ctx.n_limbs)[0]
            sub = limbs[tidx].contiguous()
            out = torch.empty_like(sub)
            status = torch.zeros((len(idx),), dtype=torch.int32, device=limbs.device)
            ctx.raw_mul_dev(sub, _to_dev(scal, ctx), out, status, len(idx), stream=_stream(ctx))
            if bool(status.any().item()):
                raise ZeroDivisionError('invert() no inverse exists')
            limbs = limbs.clone()
            limbs[tidx] = out
        return EncryptedVector(self.public_key, limbs, new_exps.copy(), obfuscated=self._obfuscated and not len(idx))

    def __add__(self, other):
        from .paillier import EncryptedNumber
        ctx = self.public_key.engine_context()
        torch = _torch()
        if isinstance(other, EncryptedNumber):
            # broadcast: one row uploaded and expanded on the device, then the vector + vector path (exponent alignment)
            if self.public_key != other.public_key:
                raise ValueError("Attempted to add numbers encrypted against different public keys!")
            row = _to_dev(ints_to_limbs([other.ciphertext(be_secure=False) % self.public_key.nsquare], ctx.c_limbs), ctx)
            other = EncryptedVector(self.public_key, row.expand(len(self), -1).contiguous(),
                                    np.full(len(self), other.exponent, dtype=np.int64))
        if isinstance(other, EncryptedVector):
            if self.public_key != other.public_key:
                raise ValueError("Attempted to add numbers encrypted against different public keys!")
            if len(other) != len(self):
                raise ValueError("length mismatch")
            new_exps = np.minimum(self.exponents, other.exponents)
            a, b = self.decrease_exponent_to(new_exps), other.decrease_exponent_to(new_exps)
            out = torch.empty_like(a.limbs)
            if len(self):
                ctx.raw_add_dev(a.limbs, b.limbs, out, len(self), stream=_stream(ctx))
            return EncryptedVector(self.public_key, out, new_exps)
        # plaintext operand(s): encode against each element's exponent (phe/paillier.py:626-676)
        scalars = list(other) if hasattr(other, "__len__") else [other] * len(self)
        if len(scalars) != len(self):
            raise ValueError("length mismatch")
        n = self.public_key.n
        if any(isinstance(s, EncodedNumber) for s in scalars):
            encs = [s if isinstance(s, EncodedNumber) else EncodedNumber.encode(self.public_key, s, max_exponent=int(e))
                    for s, e in zip(scalars, self.exponents)]
            new_exps = np.minimum(self.exponents, np.array([e.exponent for e in encs], dtype=np.int64))
            a = self.decrease_exponent_to(new_exps)
            encs = [e.decrease_exponent_to(int(x)) if e.exponent > x else e for e, x in zip(encs, new_exps)]
            encodings = [e.encoding for e in encs]
        else:
            # plain numbers: one vectorised encode against every element's exponent; the encoded exponent never exceeds
            # it (max_exponent), so only `self` may need aligning
            s_limbs, new_exps = encode_batch(self.public_key, other if isinstance(other, np.ndarray) else scalars,
                                             max_exponent=self.exponents)
            a = self.decrease_exponent_to(new_exps)
            encodings = limbs_to_ints(s_limbs)
        nude = [(n * e + 1) % self.public_key.nsquare for e in encodings]          # raw_encrypt(., r=1), phe/paillier.py:673
        d_b = _to_dev(ints_to_limbs(nude, ctx.c_limbs), ctx)
        out = torch.empty_like(a.limbs)
        if len(self):
            ctx.raw_add_dev(a.limbs, d_b, out, len(self), stream=_stream(ctx))
        return EncryptedVector(self.public_key, out, new_exps)

    __radd__ = __add__

    def __mul__(self, other):
        if isinstance(other, EncryptedVector):
            raise NotImplementedError('Good luck with that...')
        scalars = list(other) if hasattr(other, "__len__") else [other] * len(self)
        if len(scalars) != len(self):
            raise ValueError("length mismatch")
        if any(isinstance(s, EncodedNumber) for s in scalars):
            encs = [s if isinstance(s, EncodedNumber) else EncodedNumber.encode(self.public_key, s) for s in scalars]
            s_limbs = ints_to_limbs([e.encoding for e in encs], self.public_key.engine_context().n_limbs)
            s_exps = np.array([e.exponent for e in encs], dtype=np.int64)
        else:
            s_limbs, s_exps = encode_batch(self.public_key, other if isinstance(other, np.ndarray) else scalars)
        out = self._raw_mul_rows(self.limbs, s_limbs) if len(self) else self.limbs
        return EncryptedVector(self.public_key, out, self.exponents + s_exps)

    __rmul__ = __mul__

    def __sub__(self, other):
        return self + (other * -1)

    def __rsub__(self, other):
        return other + (self * -1)

    def __truediv__(self, scalar):
        return self * (1 / scalar)

    def sum(self):
        """Homomorphic sum of all elements -> EncryptedNumber: the product of the ciphertexts modulo n^2 in two launches
        (pai_raw_sum: per-thread strided products, shared-memory tree per CTA, second launch over the CTA partials) --
        the reference's sum(list) / np.mean idiom (phe/tests/math_test.py:44-58) without B - 1 sequential _raw_add calls."""
        from .paillier import EncryptedNumber
        if not len(self):
            raise ValueError("empty vector")
        ctx = self.public_key.engine_context()
        torch = _torch()
        v = self.decrease_exponent_to(int(self.exponents.min()))
        out = torch.empty((1, v.limbs.shape[1]), dtype=torch.int32, device=v.limbs.device)
        ctx.raw_sum_dev(v.limbs, len(v), out, stream=_stream(ctx))
        return EncryptedNumber(self.public_key, limbs_to_ints(_to_host(out))[0], int(v.exponents[0]))

    def sum_chain(self):
        """The round-1 form of sum(): a chain of log2(B) pairwise raw_add launches (kept as the comparison baseline of
        bench.py's `reductions` leg and as a cross-check in the tests)."""
        from .paillier import EncryptedNumber
        if not len(self):
            raise ValueError("empty vector")
        ctx = self.public_key.engine_context()
        torch = _torch()
        v = self.decrease_exponent_to(int(self.exponents.min()))
        limbs = v.limbs
        while limbs.shape[0] > 1:
            half = limbs.shape[0] // 2
            out = torch.empty((half, limbs.shape[1]), dtype=torch.int32, device=limbs.device)
            ctx.raw_add_dev(limbs[:half].contiguous(), limbs[half:2 * half].contiguous(), out, half, stream=_stream(ctx))
            limbs = torch.cat([out, limbs[2 * half:]], dim=0) if limbs.shape[0] % 2 else out
        c = limbs_to_ints(_to_host(limbs))[0]
        return EncryptedNumber(self.public_key, c, int(v.exponents[0]))

    def _encode_scalars(self, scalars):
        if isinstance(scalars, EncryptedVector):
            raise NotImplementedError('Good luck with that...')
        sc = list(scalars) if not isinstance(scalars, np.ndarray) else scalars
        if len(sc) != len(self):
            raise ValueError("length mismatch")
        if not isinstance(sc, np.ndarray) and any(isinstance(x, EncodedNumber) for x in sc):
            encs = [x if isinstance(x, EncodedNumber) else EncodedNumber.encode(self.public_key, x) for x in sc]
            return (ints_to_limbs([e.encoding for e in encs], self.public_key.engine_context().n_limbs),
                    np.array([e.exponent for e in encs], dtype=np.int64))
        return encode_batch(self.public_key, sc)

    def dot(self, scalars):
        """Homomorphic dot product sum_i self[i] * scalars[i] -> EncryptedNumber (the encrypted scoring loop of
        examples/logistic_regression_encrypted_model.py:170-180): pai_raw_dot = Straus' simultaneous exponentiation over
        the group of elements each thread owns (one shared chain of squarings) + the product reduction of sum().
        Element exponents are aligned to the lowest one by folding BASE^delta into the plaintext scalar."""
        from .paillier import EncryptedNumber
        if not len(self):
            raise ValueError("empty vector")
        ctx = self.public_key.engine_context()
        torch = _torch()
        s_limbs, s_exps = self._encode_scalars(scalars)
        exps = self.exponents + s_exps
        emin = int(exps.min())
        up = np.nonzero(exps > emin)[0]
        if len(up):                                   # c^(k * BASE^delta) = (c^k)^(BASE^delta): alignment inside the exponent
            n, max_int = self.public_key.n, self.public_key.max_int
            vals = limbs_to_ints(s_limbs[up])
            new = []
            for k, d in zip(vals, (exps[up] - emin).tolist()):
                f = pow(EncodedNumber.BASE, int(d))
                mag = (n - k) if k >= n - max_int else k
                if mag * f > max_int:
                    raise ValueError('Integer needs to be within +/- %d but got %d' % (max_int, mag * f))
                new.append(k * f % n)
            s_limbs = s_limbs.copy()
            s_limbs[up] = ints_to_limbs(new, s_limbs.shape[1])
        out = torch.empty((1, self.limbs.shape[1]), dtype=torch.int32, device=self.limbs.device)
        status = torch.zeros((len(self),), dtype=torch.int32, device=self.limbs.device)
        ctx.raw_dot_dev(self.limbs, _to_dev(s_limbs, ctx), out, status, len(self), stream=_stream(ctx))
        if bool(status.any().item()):
            raise ZeroDivisionError('invert() no inverse exists')
        return EncryptedNumber(self.public_key, limbs_to_ints(_to_host(out))[0], emin)

    def dot_chain(self, scalars):
        """The round-1 form of dot(): one raw_mul launch, then sum_chain()."""
        return (self * scalars).sum_chain()

    def rmatmul(self, X):
        """X @ self for a plaintext matrix X of shape [N, len(self)] -> EncryptedVector of length N, in one fused product
        on the device (pai_raw_matvec): window tables of every ciphertext are built once and shared by all rows, and
        each row runs one squaring chain for all its entries.  This is the encrypted scoring of
        examples/logistic_regression_encrypted_model.py:170-180 for a whole matrix; ``v.rmatmul(X) + enc_b`` adds the
        intercept.

        X is a 2-D numpy array (float or int) or any scipy.sparse matrix or array.
          - dense X: row j equals ``self.dot(X[j])``, the same ciphertext with the same exponent (the lowest exponent
            over ALL entries of the row, zeros included; zero scalars contribute nothing).
          - sparse X: row j equals the reference's loop ``score += x[0, i] * w[i]`` over ``x.nonzero()`` without an
            intercept (explicitly stored zeros are ignored); an empty row is the ciphertext 1 with exponent 0.
        Exponents are aligned inside the scalars as in dot(), with the same ValueError when |k| * BASE^delta exceeds
        max_int; a ciphertext used with a negative scalar that has no inverse mod n^2 raises ZeroDivisionError.  The
        result is not obfuscated.

        ``X @ v`` reaches this method for numpy X.  ``scipy_matrix @ v`` does NOT: scipy converts v with
        np.asanyarray first, so scipy users call ``v.rmatmul(X)``.  A single row is latency bound here (one thread
        per row): use dot() for a 1 x d product."""
        pk = self.public_key
        ctx = pk.engine_context()
        torch = _torch()
        sparse = _is_sparse(X)
        if not sparse:
            X = np.asarray(X)
            if X.ndim == 1:
                raise ValueError("rmatmul needs a 2-D matrix; use dot() for a 1-D vector of scalars")
        if X.ndim != 2:
            raise ValueError("rmatmul needs a 2-D matrix")
        nrows, ncols = (int(x) for x in X.shape)
        if ncols != len(self):
            raise ValueError("matrix has %d columns, the vector %d elements" % (ncols, len(self)))
        if sparse:
            X = X.tocsr(copy=True)
            X.sum_duplicates()
            X.eliminate_zeros()                           # x.nonzero() skips explicitly stored zeros
            indptr = X.indptr.astype(np.int64)
            cols = X.indices.astype(np.int64)
            vals = _plain_values(X.data)
        else:
            indptr = np.arange(nrows + 1, dtype=np.int64) * ncols
            cols = np.tile(np.arange(ncols, dtype=np.int64), nrows)
            vals = _plain_values(X.reshape(-1))
        rows = np.repeat(np.arange(nrows, dtype=np.int64), np.diff(indptr))
        neg, mag, exps = _signed_encodings(pk, vals)
        # row exponent: the lowest exponent among the row's entries (dense: zeros included); empty rows: 0
        texp = self.exponents[cols] + exps
        row_exp = np.zeros(nrows, dtype=np.int64)
        filled = np.diff(indptr) > 0
        if filled.any():
            row_exp[filled] = np.minimum.reduceat(texp, indptr[:-1][filled])
        delta = texp - row_exp[rows]
        keep = np.nonzero(mag != 0 if isinstance(mag, np.ndarray) else np.array([m != 0 for m in mag], dtype=bool))[0]
        rows, cols, neg, delta = rows[keep], cols[keep], neg[keep], delta[keep]
        mag = mag[keep] if isinstance(mag, np.ndarray) else [mag[i] for i in keep.tolist()]
        mag_limbs, mag_bits, m_limbs = _aligned_magnitudes(pk, mag, delta)
        # rows by decreasing length, so that the rows of a warp are about equally long
        counts = np.bincount(rows, minlength=nrows)
        order = np.argsort(-counts, kind="stable")
        s_indptr = np.zeros(nrows + 1, dtype=np.int64)
        np.cumsum(counts[order], out=s_indptr[1:])
        starts = np.zeros(nrows, dtype=np.int64)
        np.cumsum(counts[:-1], out=starts[1:])
        shift = np.repeat(starts[order] - s_indptr[:-1], counts[order])
        perm = slice(None) if not shift.any() else np.arange(len(keep), dtype=np.int64) + shift
        nnz = len(keep)
        dev = self.limbs.device
        d_indptr = _arr_to_dev(s_indptr, ctx)
        d_indices = _arr_to_dev(cols[perm].astype(np.int32), ctx)
        d_mag = _to_dev(m_limbs[perm], ctx)
        any_neg = bool(neg.any())
        d_neg = _arr_to_dev(neg[perm].astype(np.uint8), ctx) if any_neg else None
        out = torch.empty((nrows, ctx.c_limbs), dtype=torch.int32, device=dev)
        status = torch.zeros((max(ncols, 1),), dtype=torch.int32, device=dev)
        if nrows:
            ctx.raw_matvec_dev(self.limbs, ncols, d_indptr, d_indices, d_mag, mag_limbs, mag_bits, d_neg, nnz, nrows, out,
                               status, stream=_stream(ctx))
            if any_neg and bool(status.any().item()):
                raise ZeroDivisionError('invert() no inverse exists')
        res = torch.empty_like(out)
        res.index_copy_(0, _arr_to_dev(order, ctx), out)
        return EncryptedVector(pk, res, row_exp)

    __rmatmul__ = rmatmul

    # ------------------------------------------------------------------ wire format
    def to_json(self, be_secure=True):
        """The reference's basic JSON scheme (docs/serialisation.rst:24-31): {'public_key': {'n': ...},
        'values': [[str(ciphertext), exponent], ...]} -- readable by an unmodified phe peer."""
        if be_secure and not self._obfuscated:
            self.obfuscate()
        texts = limbs_to_decimal_strings(self.public_key.engine_context(), self.limbs)
        return '{"public_key": {"n": %d}, "values": [%s]}' % (
            self.public_key.n, ", ".join('["%s", %d]' % (t, e) for t, e in zip(texts, self.exponents.tolist())))

    @classmethod
    def from_json(cls, serialised, public_key=None):
        """Inverse of to_json (docs/serialisation.rst:35-42); ciphertexts go straight to the GPU."""
        import json
        from .paillier import PaillierPublicKey
        d = json.loads(serialised)
        pk = public_key or PaillierPublicKey(int(d["public_key"]["n"]))
        if pk.n != int(d["public_key"]["n"]):
            raise ValueError("serialised vector was encrypted against a different key")
        ctx = pk.engine_context()
        texts = [str(v[0]).lstrip("0") or "0" for v in d["values"]]
        bound = str(pk.nsquare)                    # the reference accepts any int; keep rows canonical (< n^2)
        texts = [t if len(t) < len(bound) or (len(t) == len(bound) and t < bound) or not t.isdigit()
                 else str(int(t) % pk.nsquare) for t in texts]
        d_c = decimal_strings_to_limbs(ctx, texts, ctx.c_limbs)
        return cls(pk, d_c, [int(v[1]) for v in d["values"]])

    # ------------------------------------------------------------------ decryption
    def decrypt_encoded(self, private_key):
        if self.public_key != private_key.public_key:
            raise ValueError('encrypted_number was encrypted against a different key!')
        ctx = private_key.engine_context()
        torch = _torch()
        count = len(self)
        plain = limbs_to_ints(self._decrypt_rows(ctx)) if count else []
        return [EncodedNumber(self.public_key, m, int(e)) for m, e in zip(plain, self.exponents)]

    def decrypt(self, private_key):
        """Decrypt and decode (vectorised EncodedNumber.decode) -> list of Python floats / ints."""
        if self.public_key != private_key.public_key:
            raise ValueError('encrypted_number was encrypted against a different key!')
        ctx = private_key.engine_context()
        torch = _torch()
        count = len(self)
        if not count:
            return []
        return decode_batch(self.public_key, self._decrypt_rows(ctx), self.exponents)

    def _decrypt_rows(self, ctx):
        """raw_decrypt of every row -> host uint32 matrix [B, n_limbs of the PUBLIC layout]."""
        return _to_host(self._decrypt_rows_dev(ctx))

    def _decrypt_rows_dev(self, ctx):
        """raw_decrypt of every row -> device int32 matrix [B, n_limbs of the PUBLIC layout].  The private context sizes
        its rows from max(p, q), the public one from n: for unbalanced primes they differ, and the rows are re-padded."""
        torch = _torch()
        count = len(self)
        d_c = _rows_for(ctx.c_limbs, self.limbs)
        d_m = torch.empty((count, ctx.n_limbs), dtype=torch.int32, device=self.limbs.device)
        ctx.decrypt_dev(d_c, d_m, count, stream=_stream(ctx))
        return _rows_for(self.public_key.engine_context().n_limbs, d_m)


# ------------------------------------------------------------------------------------------------------
# Packed fixed-point vectors (DESIGN.md §3.10): K signed b-bit slots per plaintext, packed and unpacked on the device.
def _slot_max(slot_bits):
    return (1 << (slot_bits - 1)) - 1


def _quantise(values, bound, frac_bits, device):
    """values -> (int64 tensor of round_half_even(x * 2^frac_bits) on `device`, shape).  NaN, inf or |x| > bound raise
    ValueError.  Float dtypes go through float64 (exact for every float dtype; the scaling by 2^f is exact), integer dtypes
    take an exact int64 path.  The caller has checked that ceil(bound * 2^f) < 2^62."""
    torch = _torch()
    if isinstance(values, torch.Tensor):
        t = values.detach()
    else:
        a = np.asarray(values)
        if a.dtype.kind == "u" and a.dtype.itemsize == 8:         # torch has no general uint64: range check here
            if a.size and int(a.max()) > bound:
                raise ValueError("a value exceeds the declared bound %r" % (bound,))
            a = a.astype(np.int64)
        if a.dtype.kind not in "biuf":
            raise TypeError("values must be real numbers, got dtype %s" % a.dtype)
        t = torch.as_tensor(a)
    if t.is_complex():
        raise TypeError("values must be real numbers, got dtype %s" % t.dtype)
    shape = tuple(int(x) for x in t.shape)
    t = t.to(device).reshape(-1)
    if t.is_floating_point():
        x = t.to(torch.float64)
        if not bool(torch.isfinite(x).all().item()):
            raise ValueError("values must be finite")
        if bool((x.abs() > float(bound)).any().item()):
            raise ValueError("a value exceeds the declared bound %r" % (bound,))
        return torch.round(x * float(2 ** frac_bits)).to(torch.int64).contiguous(), shape
    x = t.to(torch.int64)
    ib = min(int(math.floor(bound)), 2 ** 63 - 1)
    if bool(((x > ib) | (x < -ib)).any().item()):
        raise ValueError("a value exceeds the declared bound %r" % (bound,))
    # |x| * 2^f <= ceil(bound * 2^f) < 2^62; for f >= 62 that leaves only x = 0
    return (x * (1 << frac_bits) if frac_bits < 62 else x).contiguous(), shape


class PackedEncryptedVector(object):
    """Fixed-point values packed many to a ciphertext (DESIGN.md §3.10).

    Each value x is quantised to the integer slot q = round_half_even(x * 2^frac_bits); slots_per_ciphertext slots of
    slot_bits bits share one plaintext.  Homomorphic addition and multiplication by an integer act on every slot at once.
    slot_bound is a public bound on every |slot|, derived from the bound declared at encryption, never from the data;
    an operation whose result could leave 2^(slot_bits-1) - 1 raises OverflowError before anything runs.

    The rows are an EncryptedVector with exponents 0 (``.ciphertexts``); +, * and obfuscate() are its operations."""
    __array_ufunc__ = None

    def __init__(self, ciphertexts, shape, slot_bits, frac_bits, slot_bound):
        self.ciphertexts = ciphertexts
        self.shape = tuple(int(x) for x in shape)
        self.slot_bits = int(slot_bits)
        self.frac_bits = int(frac_bits)
        self.slot_bound = int(slot_bound)
        self.slots_per_ciphertext = ciphertexts.public_key.engine_context().slots_per_row(self.slot_bits)

    @property
    def public_key(self):
        return self.ciphertexts.public_key

    def __len__(self):
        return math.prod(self.shape)

    # ------------------------------------------------------------------ construction
    @classmethod
    def encrypt(cls, public_key, values, bound, frac_bits=24, headroom=1024, r_values=None, private_key=None):
        """Quantise `values` (torch tensor on any device, numpy array or sequence; float or integer; any shape) with
        frac_bits fractional bits, pack them on the device and encrypt one ciphertext per slots_per_ciphertext values.
        `bound` declares max |x|; the slot width leaves room for `headroom` such vectors to be added.  r_values: one r
        per ciphertext, or None for fresh random r drawn on the device."""
        torch = _torch()
        if isinstance(frac_bits, bool) or not isinstance(frac_bits, numbers.Integral) or frac_bits < 0:
            raise ValueError("frac_bits must be a non-negative integer")
        if isinstance(headroom, bool) or not isinstance(headroom, numbers.Integral) or headroom < 1:
            raise ValueError("headroom must be a positive integer")
        if (isinstance(bound, bool) or not isinstance(bound, numbers.Real) or bound <= 0
                or not (isinstance(bound, numbers.Integral) or math.isfinite(bound))):
            raise ValueError("bound must be a positive finite number")
        frac_bits, headroom = int(frac_bits), int(headroom)
        qmax = math.ceil(fractions.Fraction(bound) * 2 ** frac_bits)
        slot_bits = (qmax * headroom).bit_length() + 1
        if slot_bits > 63:
            raise ValueError("bound * 2^frac_bits * headroom needs %d-bit slots; at most 63 are supported" % slot_bits)
        ctx = public_key.engine_context()
        K = ctx.slots_per_row(slot_bits)
        device = "cpu" if ctx.eng.simulated else "cuda:%d" % ctx.device
        q, shape = _quantise(values, bound, frac_bits, device)
        count = int(q.numel())
        rows = -(-count // K)
        if r_values is not None:
            r_values = list(r_values)
            if len(r_values) != rows:
                raise ValueError("%d r_values for %d ciphertexts" % (len(r_values), rows))
        d_m = torch.empty((rows, ctx.n_limbs), dtype=torch.int32, device=q.device)
        status = torch.zeros((rows,), dtype=torch.int32, device=q.device)
        ctx.pack_slots_dev(q, count, slot_bits, d_m, status, stream=_stream(ctx))
        if bool(status.any().item()):                          # every |q| <= qmax < 2^(slot_bits-1)
            raise RuntimeError("pack_slots rejected a slot within the bound")
        rows_enc = EncryptedVector._encrypt_dev_rows(public_key, d_m, np.zeros(rows, dtype=np.int64), r_values, private_key)
        return cls(rows_enc, shape, slot_bits, frac_bits, qmax)

    # ------------------------------------------------------------------ arithmetic
    def _result(self, ciphertexts, slot_bound):
        return PackedEncryptedVector(ciphertexts, self.shape, self.slot_bits, self.frac_bits, slot_bound)

    def _check_bound(self, slot_bound):
        if slot_bound > _slot_max(self.slot_bits):
            raise OverflowError("the result's slots could reach %d, beyond the %d-bit slots' %d"
                                % (slot_bound, self.slot_bits, _slot_max(self.slot_bits)))

    def _check_layout(self, other):
        if not isinstance(other, PackedEncryptedVector):
            raise ValueError("a packed vector combines only with a packed vector")
        if (self.public_key != other.public_key or self.shape != other.shape or self.slot_bits != other.slot_bits
                or self.frac_bits != other.frac_bits):
            raise ValueError("packed vectors differ in key, shape, slot_bits or frac_bits")

    def __add__(self, other):
        if isinstance(other, numbers.Integral) and not isinstance(other, bool) and other == 0:
            return self                                         # sum() starts from 0
        if not isinstance(other, (PackedEncryptedVector, EncryptedVector)):
            return NotImplemented
        self._check_layout(other)
        bound = self.slot_bound + other.slot_bound
        self._check_bound(bound)
        return self._result(self.ciphertexts + other.ciphertexts, bound)

    __radd__ = __add__

    def __neg__(self):
        return self * -1

    def __sub__(self, other):
        if not isinstance(other, (PackedEncryptedVector, EncryptedVector)):
            return NotImplemented
        self._check_layout(other)
        self._check_bound(self.slot_bound + other.slot_bound)
        return self + (-other)

    def __mul__(self, other):
        if isinstance(other, (PackedEncryptedVector, EncryptedVector)):
            raise NotImplementedError('Good luck with that...')
        if isinstance(other, bool) or not isinstance(other, numbers.Integral):
            raise TypeError("a packed vector is multiplied by integers only; apply a real factor after decryption")
        c = int(other)
        bound = self.slot_bound * abs(c)
        self._check_bound(bound)
        return self._result(self.ciphertexts * c, bound)

    __rmul__ = __mul__

    def obfuscate(self):
        self.ciphertexts.obfuscate()

    # ------------------------------------------------------------------ decryption
    def decrypt_fixed(self, private_key):
        """The exact int64 slots (the quantised values, summed and scaled as the operations did), a tensor of .shape on
        the vector's device.  A ciphertext whose plaintext is not a packing raises ValueError."""
        if self.public_key != private_key.public_key:
            raise ValueError('encrypted_number was encrypted against a different key!')
        torch = _torch()
        ctx = self.public_key.engine_context()
        count, rows = len(self), len(self.ciphertexts)
        dev = self.ciphertexts.limbs.device
        slots = torch.zeros((count,), dtype=torch.int64, device=dev)
        if rows:
            d_m = self.ciphertexts._decrypt_rows_dev(private_key.engine_context())
            status = torch.zeros((rows,), dtype=torch.int32, device=dev)
            ctx.unpack_slots_dev(d_m, self.slot_bits, slots, count, status, stream=_stream(ctx))
            bad = torch.nonzero(status).flatten()
            if bad.numel():
                raise ValueError("ciphertext %d does not decrypt to a packing of %d-bit slots" % (int(bad[0]), self.slot_bits))
        return slots.reshape(self.shape)

    def decrypt(self, private_key):
        """The values as a float64 tensor of .shape on the vector's device: slot * 2^-frac_bits (exact while |slot| < 2^53)."""
        return self.decrypt_fixed(private_key).to(_torch().float64) * (2.0 ** -self.frac_bits)

    # ------------------------------------------------------------------ wire format
    def to_json(self, be_secure=True):
        """{"packing": {shape, slot_bits, frac_bits, slot_bound}, "ciphertexts": <EncryptedVector.to_json>}"""
        import json
        packing = {"shape": list(self.shape), "slot_bits": self.slot_bits, "frac_bits": self.frac_bits,
                   "slot_bound": self.slot_bound}
        return '{"packing": %s, "ciphertexts": %s}' % (json.dumps(packing), self.ciphertexts.to_json(be_secure))

    @classmethod
    def from_json(cls, serialised, public_key=None):
        import json
        d = json.loads(serialised)
        try:
            p = d["packing"]
            shape, b, f, bound = p["shape"], p["slot_bits"], p["frac_bits"], p["slot_bound"]
            cts = d["ciphertexts"]
        except (KeyError, TypeError) as e:
            raise ValueError("not a serialised packed vector") from e

        def is_int(x):
            return isinstance(x, int) and not isinstance(x, bool)
        if (not isinstance(shape, list) or not all(is_int(x) and x >= 0 for x in shape) or not is_int(b) or not 2 <= b <= 63
                or not is_int(f) or f < 0 or not is_int(bound) or not 0 <= bound <= _slot_max(b)):
            raise ValueError("malformed packing layout")
        if not isinstance(cts, dict):
            raise ValueError("malformed ciphertexts")
        try:
            rows = EncryptedVector.from_json(json.dumps(cts), public_key)
        except (KeyError, TypeError, IndexError, AttributeError) as e:
            raise ValueError("malformed ciphertexts") from e
        K = rows.public_key.engine_context().slots_per_row(b)
        if len(rows) != -(-math.prod(shape) // K) or rows.exponents.any():
            raise ValueError("the ciphertexts do not match the packing layout")
        return cls(rows, shape, b, f, bound)
