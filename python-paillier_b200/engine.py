"""ctypes binding of libpaillier_b200.so (C ABI: include/paillier_b200.h) + limb packing.

This is the thin host layer between Python ints and the CUDA engine.  It replaces what
``gmpy2`` is to the reference (phe/util.py:21-25, 50, 63-64, 92): a native bigint engine behind
three functions -- except that here the engine is batched and lives on the GPU.

There is NO CPU fallback.  If the CUDA library is missing or no device is present, loading /
context creation raises ``EngineUnavailable`` -- nothing silently degrades to Python ``pow``.
"""
import ctypes
import os
import threading

import numpy as np

__all__ = ["Engine", "EngineError", "EngineUnavailable", "get_engine", "ints_to_limbs", "limbs_to_ints",
           "PublicContext", "PrivateContext", "ModContext"]

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_NAME = "libpaillier_b200.so"

PAI_E_ARG, PAI_E_CUDA, PAI_E_NOINV = -1, -2, -3


class EngineError(RuntimeError):
    pass


class EngineUnavailable(EngineError):
    """The CUDA engine cannot be used (library not built, or no CUDA device)."""


_u32p = ctypes.POINTER(ctypes.c_uint32)
_i32p = ctypes.POINTER(ctypes.c_int32)
_vp = ctypes.c_void_p

# name -> (restype, argtypes); every symbol include/paillier_b200.h declares
SYMBOLS = {
    "pai_last_error": (ctypes.c_char_p, []),
    "pai_version": (ctypes.c_int, []),
    "pai_device_count": (ctypes.c_int, []),
    "pai_launch_count": (ctypes.c_long, []),
    "pai_mod_create": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    "pai_mod_destroy": (ctypes.c_int, [_vp]),
    "pai_mod_limbs": (ctypes.c_int, [_vp]),
    "pai_mod_mulmod": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long, _vp]),
    "pai_mod_powmod_shared": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, ctypes.c_int, _vp, ctypes.c_long, _vp]),
    "pai_mod_powmod": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, ctypes.c_int, _vp, ctypes.c_long, _vp]),
    "pai_mod_invert": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, _vp, ctypes.c_long, _vp]),
    "pai_pub_create": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    "pai_pub_destroy": (ctypes.c_int, [_vp]),
    "pai_pub_n_limbs": (ctypes.c_int, [_vp]),
    "pai_pub_c_limbs": (ctypes.c_int, [_vp]),
    "pai_pub_wave": (ctypes.c_long, [_vp]),
    "pai_priv_wave": (ctypes.c_long, [_vp]),
    "pai_pub_kernel_path": (ctypes.c_int, [_vp]),
    "pai_priv_kernel_path": (ctypes.c_int, [_vp]),
    "pai_encrypt": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long, _vp]),
    "pai_random_lt_n": (ctypes.c_int, [_vp, ctypes.c_char_p, ctypes.c_ulonglong, _vp, ctypes.c_long, _vp]),
    "pai_decimal_width": (ctypes.c_int, [ctypes.c_int]),
    "pai_limbs_to_decimal": (ctypes.c_int, [_vp, ctypes.c_int, _vp, ctypes.c_long, ctypes.c_int, _vp]),
    "pai_decimal_to_limbs": (ctypes.c_int, [_vp, ctypes.c_int, _vp, ctypes.c_int, _vp, ctypes.c_long, ctypes.c_int, _vp]),
    "pai_pack_slots_per_row": (ctypes.c_int, [_vp, ctypes.c_int]),
    "pai_pack_slots": (ctypes.c_int, [_vp, _vp, ctypes.c_long, ctypes.c_int, _vp, _vp, _vp]),
    "pai_unpack_slots": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, ctypes.c_long, _vp, _vp]),
    "pai_raw_add": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long, _vp]),
    "pai_raw_mul": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, ctypes.c_long, _vp]),
    "pai_miller_rabin": (ctypes.c_int, [_vp, ctypes.c_int, _vp, ctypes.c_int, _vp, ctypes.c_long, ctypes.c_int, _vp]),
    "pai_raw_sum": (ctypes.c_int, [_vp, _vp, ctypes.c_long, _vp, _vp]),
    "pai_raw_dot": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, ctypes.c_long, _vp]),
    "pai_raw_matvec": (ctypes.c_int, [_vp, _vp, ctypes.c_long, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, _vp, ctypes.c_long,
                                      ctypes.c_long, _vp, _vp, _vp]),
    "pai_raw_matvec_window": (ctypes.c_int, [_vp, ctypes.c_long, ctypes.c_long, ctypes.c_long, ctypes.c_int, ctypes.c_int]),
    "pai_priv_create": (ctypes.c_int, [_vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(_vp)]),
    "pai_priv_destroy": (ctypes.c_int, [_vp]),
    "pai_priv_n_limbs": (ctypes.c_int, [_vp]),
    "pai_priv_c_limbs": (ctypes.c_int, [_vp]),
    "pai_priv_get": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "pai_decrypt": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_long, _vp]),
    "pai_priv_encrypt": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long, _vp]),
    "pai_encrypt_host": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long]),
    "pai_raw_add_host": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long]),
    "pai_raw_mul_host": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, ctypes.c_long]),
    "pai_decrypt_host": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_long]),
    "pai_priv_encrypt_host": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long]),
    "pai_mod_mulmod_host": (ctypes.c_int, [_vp, _vp, _vp, _vp, ctypes.c_long]),
    "pai_mod_powmod_host": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, _vp, ctypes.c_long]),
    "pai_mod_invert_host": (ctypes.c_int, [_vp, _vp, ctypes.c_int, _vp, _vp, ctypes.c_long]),
}


# ---------------------------------------------------------------------------- decimal wire format
def limbs_to_decimal_dev(d_limbs, limbs, d_text, batch, device=0, stream=None, engine=None):
    """d_text [batch, decimal_width(limbs)] uint8 <- decimal digits of d_limbs [batch, limbs] (pai_radix.cuh)."""
    eng = engine or get_engine()
    eng.check(eng.lib.pai_limbs_to_decimal(_ptr(d_limbs), limbs, _ptr(d_text), batch, device, _ptr(stream)))


def decimal_to_limbs_dev(d_text, width, d_limbs, limbs, d_status, batch, device=0, stream=None, engine=None):
    eng = engine or get_engine()
    eng.check(eng.lib.pai_decimal_to_limbs(_ptr(d_text), width, _ptr(d_limbs), limbs, _ptr(d_status), batch, device,
                                           _ptr(stream)))


def decimal_width(limbs, engine=None):
    return int((engine or get_engine()).lib.pai_decimal_width(limbs))


def miller_rabin_batch(candidates, rounds=25, device=0, engine=None):
    """[is n probably prime] for a list of odd ints > 3: `rounds` Miller-Rabin rounds per candidate on the device, random
    bases from os.urandom (pai_miller_rabin; util.miller_rabin, phe/util.py:381-417, for a whole batch)."""
    eng = engine or get_engine()
    eng.require_device()
    count = len(candidates)
    if not count:
        return []
    tiles = (max(c.bit_length() for c in candidates) + 255) // 256
    tiles = next((t for t in (1, 2, 3, 4, 6, 8, 12, 16, 24, 32) if t >= tiles), None)       # tile counts the kernels exist for
    if tiles is None:
        raise ValueError("candidates above 8192 bits are not supported")
    limbs = 8 * tiles
    cand = ints_to_limbs(candidates, limbs)
    bases = np.frombuffer(bytearray(os.urandom(count * rounds * limbs * 4)), dtype=np.uint32).reshape(count, rounds, limbs)
    result = np.zeros(count, dtype=np.int32)
    if eng.simulated:
        eng.check(eng.lib.pai_miller_rabin(_ptr(cand), limbs, _ptr(bases), rounds, _ptr(result), count, device, None))
        return [bool(x) for x in result]
    import torch
    dev = "cuda:%d" % device
    d_c = torch.from_numpy(cand.view(np.int32).copy()).to(dev)
    d_b = torch.from_numpy(bases.view(np.int32).copy()).to(dev)
    d_r = torch.zeros(count, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    eng.check(eng.lib.pai_miller_rabin(_ptr(d_c), limbs, _ptr(d_b), rounds, _ptr(d_r), count, device, None))
    return [bool(x) for x in d_r.cpu().tolist()]


# ---------------------------------------------------------------------------- limb packing
def ints_to_limbs(values, limbs):
    """Python ints (0 <= v < 2**(32*limbs)) -> C-contiguous uint32 array [len, limbs], little endian.
    One ``int.to_bytes`` per value (the CPython floor, ~0.4 us at 2048 bits), one join, one frombuffer."""
    nbytes = 4 * limbs
    n = len(values)
    try:
        raw = b"".join(map(int.to_bytes, values, (nbytes,) * n, ("little",) * n))
    except OverflowError as e:
        raise ValueError("integer does not fit %d limbs (or is negative)" % limbs) from e
    # bytearray: callers get a writable array (np.frombuffer of bytes would be read-only)
    return np.frombuffer(bytearray(raw), dtype=np.uint32).reshape(n, limbs)


def limbs_to_ints(arr):
    """uint32 array [n, limbs] -> list of Python ints (one ``int.from_bytes`` per row over a memoryview, no copies)."""
    arr = np.ascontiguousarray(arr, dtype=np.uint32)
    n, limbs = arr.shape
    nbytes = 4 * limbs
    if not n:
        return []
    mv = memoryview(arr).cast("B")
    fb = int.from_bytes
    return [fb(mv[i:i + nbytes], "little") for i in range(0, n * nbytes, nbytes)]


def _ptr(a):
    """void* of a numpy array / torch tensor / raw integer address."""
    if a is None:
        return None
    if isinstance(a, int):
        return ctypes.c_void_p(a)
    if isinstance(a, np.ndarray):
        if not a.flags["C_CONTIGUOUS"]:
            raise ValueError("array must be C-contiguous")
        return ctypes.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):                      # torch tensor (device or pinned host memory)
        if not a.is_contiguous():
            raise ValueError("tensor must be contiguous")
        return ctypes.c_void_p(a.data_ptr())
    raise TypeError("unsupported buffer type %r" % type(a))


# ---------------------------------------------------------------------------- library
class Engine:
    """A loaded libpaillier_b200.so.  ``lib_path`` is for tests (the CPU simulation build under
    tests/hostsim); the product always uses the in-tree CUDA build next to this file."""

    def __init__(self, lib_path=None):
        path = lib_path or os.path.join(_HERE, LIB_NAME)
        if not os.path.exists(path):
            raise EngineUnavailable(
                "%s not found: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
                "This package has no CPU fallback." % path)
        try:
            self.lib = ctypes.CDLL(path)
        except OSError as e:
            raise EngineUnavailable("cannot load %s: %s" % (path, e)) from e
        self.path = path
        # the TEST-ONLY CPU simulation build treats "device" pointers as host pointers
        self.simulated = "hostsim" in os.path.basename(path)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(self.lib, name)            # AttributeError if the ABI is incomplete
            fn.restype = res
            fn.argtypes = args

    def device_count(self):
        return int(self.lib.pai_device_count())

    def require_device(self):
        if self.device_count() < 1:
            raise EngineUnavailable("no CUDA device visible; the Paillier engine runs on the GPU only "
                                    "(there is no CPU fallback)")

    def launch_count(self):
        return int(self.lib.pai_launch_count())

    def check(self, rc):
        if rc == 0:
            return
        msg = (self.lib.pai_last_error() or b"").decode("utf-8", "replace")
        if rc == PAI_E_CUDA:
            raise EngineUnavailable("CUDA error: %s" % msg)
        if rc == PAI_E_NOINV:
            raise ZeroDivisionError('invert() no inverse exists')      # phe/util.py:96-97
        raise EngineError("engine error %d: %s" % (rc, msg))


_engine = None
_engine_lock = threading.Lock()


def get_engine():
    """Process-wide engine (the CUDA build).  Raises EngineUnavailable when it cannot be used."""
    global _engine
    with _engine_lock:
        if _engine is None:
            _engine = Engine()
        return _engine


def _set_engine_for_tests(engine):
    """tests only: install an explicitly constructed Engine (e.g. the hostsim build)."""
    global _engine
    with _engine_lock:
        _engine = engine


# ---------------------------------------------------------------------------- Python-int pipelines
_PIPE_MIN = 1 << 15        # below this many rows a single call is used


def _chunk_ranges(count, wave, target=1 << 16):
    """Split [0, count) in chunks that are whole waves of the throughput kernel (about `target` rows each), so that only
    the last chunk has a partial wave."""
    wave = max(1, int(wave))
    chunk = max(1, round(target / wave)) * wave
    return [(lo, min(count, lo + chunk)) for lo in range(0, count, chunk)]


def _pipeline(ranges, pack, run, unpack):
    """out = concat(unpack(run(pack(lo, hi)))) over the ranges, with the (GIL-holding) int <-> limb conversions of chunk
    i+1 / i-1 running on this thread while the blocking C call of chunk i (which releases the GIL) runs on a worker
    thread.  The C ABI serialises calls on one context, so at most one kernel batch is in flight."""
    from concurrent.futures import ThreadPoolExecutor
    out = []
    with ThreadPoolExecutor(max_workers=1) as ex:
        futs = []
        for i, (lo, hi) in enumerate(ranges):
            futs.append(ex.submit(run, pack(lo, hi)))
            if i:
                out.extend(unpack(futs[i - 1].result()))
                futs[i - 1] = None
        out.extend(unpack(futs[-1].result()))
    return out


def _raw_encrypt_pipelined(ctx, plaintexts, r_values):
    """raw_encrypt of Python ints through ctx.encrypt_host (a public or a private context): m of any sign or size (reduced
    mod n as the reference's ``% nsquare`` does, phe/paillier.py:134), r in [1, n)."""
    n = ctx.n
    lim = 1 << (32 * ctx.n_limbs)
    count = len(plaintexts)
    if len(r_values) != count:
        raise ValueError("plaintexts and r_values differ in length")

    def pack(lo, hi):
        return (ints_to_limbs([p if 0 <= p < lim else p % n for p in plaintexts[lo:hi]], ctx.n_limbs),
                ints_to_limbs(r_values[lo:hi], ctx.n_limbs))
    if count < _PIPE_MIN:
        return limbs_to_ints(ctx.encrypt_host(*pack(0, count)))
    return _pipeline(_chunk_ranges(count, ctx.wave()), pack, lambda a: ctx.encrypt_host(*a), limbs_to_ints)


# ---------------------------------------------------------------------------- contexts
class ModContext:
    """Montgomery context of one odd modulus: batched powmod / mulmod / invert (the phe/util.py seam)."""

    def __init__(self, modulus, device=0, engine=None):
        self.eng = engine or get_engine()
        self.eng.require_device()
        if modulus <= 1 or modulus % 2 == 0:
            raise ValueError("modulus must be odd and > 1")
        self.modulus = modulus
        limbs = (modulus.bit_length() + 31) // 32
        arr = ints_to_limbs([modulus], limbs)          # keep a reference alive across the call
        h = ctypes.c_void_p()
        self.eng.check(self.eng.lib.pai_mod_create(_ptr(arr), limbs, device, ctypes.byref(h)))
        del arr
        self.h = h
        self.limbs = int(self.eng.lib.pai_mod_limbs(h))
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.pai_mod_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # host-array API (numpy uint32 [B, limbs])
    def mulmod_host(self, a, b):
        out = np.empty_like(a)
        self.eng.check(self.eng.lib.pai_mod_mulmod_host(self.h, _ptr(a), _ptr(b), _ptr(out), a.shape[0]))
        return out

    def powmod_host(self, base, exp, shared):
        out = np.empty((base.shape[0], self.limbs), dtype=np.uint32)
        self.eng.check(self.eng.lib.pai_mod_powmod_host(self.h, _ptr(base), base.shape[1], _ptr(exp), exp.shape[-1],
                                                        1 if shared else 0, _ptr(out), base.shape[0]))
        return out

    def invert_host(self, a):
        out = np.empty((a.shape[0], self.limbs), dtype=np.uint32)
        status = np.zeros(a.shape[0], dtype=np.int32)
        self.eng.check(self.eng.lib.pai_mod_invert_host(self.h, _ptr(a), a.shape[1], _ptr(out), _ptr(status), a.shape[0]))
        return out, status

    # Python-int API
    def powmod(self, bases, exponents):
        """[b**e mod N]; `exponents` is one int (shared) or a list (per element).  Bases may be up to
        twice as wide as the modulus (reduced on the device)."""
        single = 2 ** (32 * self.limbs)
        wide = any(b >= single for b in bases)
        base = ints_to_limbs(bases, self.limbs * (2 if wide else 1))
        if isinstance(exponents, int):
            el = max(1, (exponents.bit_length() + 31) // 32)
            exp = ints_to_limbs([exponents], el)
            return limbs_to_ints(self.powmod_host(base, exp, True))
        el = max(1, max((e.bit_length() + 31) // 32 for e in exponents))
        el = (el + 3) // 4 * 4
        exp = ints_to_limbs(exponents, el)
        return limbs_to_ints(self.powmod_host(base, exp, False))

    def mulmod(self, a, b):
        return limbs_to_ints(self.mulmod_host(ints_to_limbs(a, self.limbs), ints_to_limbs(b, self.limbs)))

    def invert(self, a):
        out, status = self.invert_host(ints_to_limbs(a, self.limbs))
        return limbs_to_ints(out), status.tolist()


class PublicContext:
    """Engine context of a public key n: batched raw_encrypt / _raw_add / _raw_mul."""

    def __init__(self, n, device=0, engine=None):
        self.eng = engine or get_engine()
        self.eng.require_device()
        if n <= 1 or n % 2 == 0:
            raise ValueError("n must be odd and > 1")
        self.n = n
        limbs = (n.bit_length() + 31) // 32
        h = ctypes.c_void_p()
        arr = ints_to_limbs([n], limbs)                # keep a reference alive across the call
        self.eng.check(self.eng.lib.pai_pub_create(_ptr(arr), limbs, device, ctypes.byref(h)))
        del arr
        self.h = h
        self.n_limbs = int(self.eng.lib.pai_pub_n_limbs(h))
        self.c_limbs = int(self.eng.lib.pai_pub_c_limbs(h))
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.pai_pub_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- device-pointer API (torch tensors / raw addresses), asynchronous on `stream`
    def encrypt_dev(self, d_m, d_r, d_c, batch, stream=None):
        self.eng.check(self.eng.lib.pai_encrypt(self.h, _ptr(d_m), _ptr(d_r), _ptr(d_c), batch, _ptr(stream)))

    def random_lt_n_dev(self, d_r, batch, seed=None, nonce=0, stream=None):
        """Fill d_r [batch, n_limbs] with r uniform in [1, n) on the device (ChaCha20 of a 32-byte seed; default:
        a fresh seed from os.urandom) -- the batched get_random_lt_n (phe/paillier.py:141-143)."""
        seed = os.urandom(32) if seed is None else bytes(seed)
        if len(seed) != 32:
            raise ValueError("seed must be 32 bytes")
        self.eng.check(self.eng.lib.pai_random_lt_n(self.h, seed, nonce, _ptr(d_r), batch, _ptr(stream)))

    def raw_add_dev(self, d_a, d_b, d_c, batch, stream=None):
        self.eng.check(self.eng.lib.pai_raw_add(self.h, _ptr(d_a), _ptr(d_b), _ptr(d_c), batch, _ptr(stream)))

    def raw_mul_dev(self, d_a, d_s, d_c, d_status, batch, stream=None):
        self.eng.check(self.eng.lib.pai_raw_mul(self.h, _ptr(d_a), _ptr(d_s), _ptr(d_c), _ptr(d_status), batch, _ptr(stream)))

    def raw_sum_dev(self, d_c, batch, d_out, stream=None):
        """d_out[0] = product of the rows of d_c mod n^2 (homomorphic sum of the vector), two launches."""
        self.eng.check(self.eng.lib.pai_raw_sum(self.h, _ptr(d_c), batch, _ptr(d_out), _ptr(stream)))

    def raw_dot_dev(self, d_a, d_s, d_out, d_status, batch, stream=None):
        """d_out[0] = prod_i d_a[i]^d_s[i] mod n^2 (encrypted dot product with plaintext scalars)."""
        self.eng.check(self.eng.lib.pai_raw_dot(self.h, _ptr(d_a), _ptr(d_s), _ptr(d_out), _ptr(d_status), batch, _ptr(stream)))

    def raw_matvec_dev(self, d_c, ncols, d_indptr, d_indices, d_mag, mag_limbs, mag_bits, d_neg, nnz, nrows, d_out,
                       d_status, stream=None):
        """d_out[j] = prod over the CSR entries t of row j of (d_neg[t] ? d_c[col]^-1 : d_c[col]) ^ d_mag[t] mod n^2
        (plaintext matrix times ciphertext vector, include/paillier_b200.h pai_raw_matvec).  d_neg may be None."""
        self.eng.check(self.eng.lib.pai_raw_matvec(self.h, _ptr(d_c), ncols, _ptr(d_indptr), _ptr(d_indices), _ptr(d_mag),
                                                   mag_limbs, mag_bits, _ptr(d_neg), nnz, nrows, _ptr(d_out),
                                                   _ptr(d_status), _ptr(stream)))

    def slots_per_row(self, slot_bits):
        """K, the signed slots of `slot_bits` bits one plaintext row of this key holds (pai_pack_slots_per_row)."""
        k = int(self.eng.lib.pai_pack_slots_per_row(self.h, slot_bits))
        if k < 0:
            raise ValueError("%d-bit slots: slot_bits must be 2..63 and at most bits(n) - 1" % slot_bits)
        return k

    def pack_slots_dev(self, d_slots, count, slot_bits, d_m, d_status, stream=None):
        """d_m [ceil(count / K), n_limbs] <- the int64 slots d_slots [count] packed K to a row, mod n; d_status [rows] = 1
        where a slot does not fit (that row is zeroed)."""
        self.eng.check(self.eng.lib.pai_pack_slots(self.h, _ptr(d_slots), count, slot_bits, _ptr(d_m), _ptr(d_status),
                                                   _ptr(stream)))

    def unpack_slots_dev(self, d_m, slot_bits, d_slots, count, d_status, stream=None):
        """Inverse of pack_slots_dev: d_status [rows] = 1 where a row is not a packing (its slots are zeroed)."""
        self.eng.check(self.eng.lib.pai_unpack_slots(self.h, _ptr(d_m), slot_bits, _ptr(d_slots), count, _ptr(d_status),
                                                     _ptr(stream)))

    def matvec_window(self, ncols, nrows, nnz, bits, with_neg):
        """The window width raw_matvec_dev picks for these shapes."""
        w = int(self.eng.lib.pai_raw_matvec_window(self.h, ncols, nrows, nnz, bits, 1 if with_neg else 0))
        self.eng.check(min(w, 0))
        return w

    # ---- host-array API (numpy uint32 limb matrices), synchronous
    def encrypt_host(self, m, r):
        out = np.empty((m.shape[0], self.c_limbs), dtype=np.uint32)
        self.eng.check(self.eng.lib.pai_encrypt_host(self.h, _ptr(m), _ptr(r), _ptr(out), m.shape[0]))
        return out

    def raw_add_host(self, a, b):
        out = np.empty((a.shape[0], self.c_limbs), dtype=np.uint32)
        self.eng.check(self.eng.lib.pai_raw_add_host(self.h, _ptr(a), _ptr(b), _ptr(out), a.shape[0]))
        return out

    def raw_mul_host(self, a, s):
        out = np.empty((a.shape[0], self.c_limbs), dtype=np.uint32)
        status = np.zeros(a.shape[0], dtype=np.int32)
        self.eng.check(self.eng.lib.pai_raw_mul_host(self.h, _ptr(a), _ptr(s), _ptr(out), _ptr(status), a.shape[0]))
        return out, status

    # ---- Python-int API
    def raw_encrypt(self, plaintexts, r_values):
        """[(1 + n*m) * r^n mod n^2]  for ints m (any sign/size: reduced mod n as the reference's
        ``% nsquare`` does, phe/paillier.py:134) and r in [1, n)."""
        return _raw_encrypt_pipelined(self, plaintexts, r_values)

    def wave(self):
        """Rows per full wave of the throughput encrypt kernel (batches that are multiples of it waste nothing)."""
        return int(self.eng.lib.pai_pub_wave(self.h))

    def kernel_path(self):
        """"full" | "digit" | "tc": the kernel family behind encrypt_dev for this key (include/paillier_b200.h)."""
        return ("full", "digit", "tc")[int(self.eng.lib.pai_pub_kernel_path(self.h))]

    def raw_add(self, a, b):
        return limbs_to_ints(self.raw_add_host(ints_to_limbs(a, self.c_limbs), ints_to_limbs(b, self.c_limbs)))

    def raw_mul(self, a, scalars):
        out, status = self.raw_mul_host(ints_to_limbs(a, self.c_limbs), ints_to_limbs(scalars, self.n_limbs))
        return limbs_to_ints(out), status.tolist()


class PrivateContext:
    """Engine context of a private key (p, q): batched raw_decrypt (CRT), and raw_encrypt through the CRT with the same
    bits as PublicContext's."""

    def __init__(self, p, q, device=0, engine=None):
        self.eng = engine or get_engine()
        self.eng.require_device()
        if p == q:
            raise ValueError('p and q have to be different')
        limbs = (max(p, q).bit_length() + 31) // 32
        h = ctypes.c_void_p()
        pa, qa = ints_to_limbs([p], limbs), ints_to_limbs([q], limbs)   # keep references alive across the call
        self.eng.check(self.eng.lib.pai_priv_create(_ptr(pa), _ptr(qa), limbs, device, ctypes.byref(h)))
        del pa, qa
        self.h = h
        self.n_limbs = int(self.eng.lib.pai_priv_n_limbs(h))
        self.c_limbs = int(self.eng.lib.pai_priv_c_limbs(h))
        bufs = [np.zeros((1, self.n_limbs), dtype=np.uint32) for _ in range(5)]
        self.eng.check(self.eng.lib.pai_priv_get(h, *[_ptr(b) for b in bufs]))
        self.p, self.q, self.p_inverse, self.hp, self.hq = [limbs_to_ints(b)[0] for b in bufs]
        self.n = self.p * self.q
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.pai_priv_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def decrypt_dev(self, d_c, d_m, batch, stream=None):
        self.eng.check(self.eng.lib.pai_decrypt(self.h, _ptr(d_c), _ptr(d_m), batch, _ptr(stream)))

    def decrypt_host(self, c):
        out = np.empty((c.shape[0], self.n_limbs), dtype=np.uint32)
        self.eng.check(self.eng.lib.pai_decrypt_host(self.h, _ptr(c), _ptr(out), c.shape[0]))
        return out

    def encrypt_dev(self, d_m, d_r, d_c, batch, stream=None):
        """d_c = (1 + n*d_m) * d_r^n mod n^2 with the private key (pai_priv_encrypt): the bits PublicContext.encrypt_dev
        gives for the same rows.  Rows of n_limbs / c_limbs columns (this context's layout)."""
        self.eng.check(self.eng.lib.pai_priv_encrypt(self.h, _ptr(d_m), _ptr(d_r), _ptr(d_c), batch, _ptr(stream)))

    def encrypt_host(self, m, r):
        out = np.empty((m.shape[0], self.c_limbs), dtype=np.uint32)
        self.eng.check(self.eng.lib.pai_priv_encrypt_host(self.h, _ptr(m), _ptr(r), _ptr(out), m.shape[0]))
        return out

    def raw_encrypt(self, plaintexts, r_values):
        """As PublicContext.raw_encrypt, computed with the private key."""
        return _raw_encrypt_pipelined(self, plaintexts, r_values)

    def raw_decrypt(self, ciphertexts):
        """raw_decrypt for ints of any size/sign (reduced mod n^2 first; the reference's powmod
        reduces the base the same way, phe/paillier.py:347,351)."""
        nsq = self.n * self.n
        full = 2 ** (32 * self.c_limbs)
        count = len(ciphertexts)

        def pack(lo, hi):
            return ints_to_limbs([x if 0 <= x < full else x % nsq for x in ciphertexts[lo:hi]], self.c_limbs)
        if count < _PIPE_MIN:
            return limbs_to_ints(self.decrypt_host(pack(0, count)))
        return _pipeline(_chunk_ranges(count, self.wave()), pack, self.decrypt_host, limbs_to_ints)

    def wave(self):
        """Rows per full wave of the throughput decrypt kernel."""
        return int(self.eng.lib.pai_priv_wave(self.h))

    def kernel_path(self):
        return ("full", "digit", "tc")[int(self.eng.lib.pai_priv_kernel_path(self.h))]
