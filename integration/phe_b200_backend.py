"""The binding a `phe` maintainer would add: the scalar bigint seam of data61/python-paillier on libpaillier_b200.so.

The reference reaches its native engine (gmpy2) through three functions, ``phe/util.py:38 powmod``, ``:53 mulmod``,
``:85 invert``, selected per call by the module flag ``HAVE_GMP`` (``phe/util.py:21-25, 47, 60, 91``) and imported BY NAME
into ``phe.paillier`` (``phe/paillier.py:29``).  This module is that seam over the C ABI of ``include/paillier_b200.h``
(plain ctypes, no torch, no other part of this repo): ``install(phe)`` rebinds the three names in ``phe.util`` AND in
``phe.paillier`` -- the same backend flip the reference's own tests perform with ``util.HAVE_GMP`` at
``phe/tests/util_test.py:64-75`` -- and ``uninstall(phe)`` restores them.  Everything else of ``phe`` stays untouched.

Library lookup: ``$PHE_B200_LIB``, else ``python-paillier_b200/libpaillier_b200.so`` next to this repo's root.
INTEGRATION.md section 1 quotes this file.
"""
import ctypes
import os
import threading

_USE_MOD_FROM_GMP_SIZE = (1 << (8 * 2))          # same thresholds as phe/util.py:35-36
_USE_MULMOD_FROM_GMP_SIZE = (1 << 1000)
_MAX_BITS = 8192                                  # pai_mod_create's limit

_lib = None
_mods = {}
_lock = threading.Lock()
_saved = {}


def load(path=None):
    """dlopen the engine and declare the few prototypes the seam needs."""
    global _lib
    if _lib is None:
        here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        path = path or os.environ.get("PHE_B200_LIB") or os.path.join(here, "python-paillier_b200", "libpaillier_b200.so")
        lib = ctypes.CDLL(path)
        vp, ci, cl = ctypes.c_void_p, ctypes.c_int, ctypes.c_long
        lib.pai_last_error.restype = ctypes.c_char_p
        lib.pai_device_count.restype = ci
        lib.pai_mod_create.argtypes = [vp, ci, ci, ctypes.POINTER(vp)]
        lib.pai_mod_limbs.argtypes = [vp]
        lib.pai_mod_powmod_host.argtypes = [vp, vp, ci, vp, ci, ci, vp, cl]
        lib.pai_mod_mulmod_host.argtypes = [vp, vp, vp, vp, cl]
        lib.pai_mod_invert_host.argtypes = [vp, vp, ci, vp, vp, cl]
        if lib.pai_device_count() < 1:
            raise OSError("libpaillier_b200: no CUDA device (the engine has no CPU fallback)")
        _lib = lib
    return _lib


def _limbs(x, n):
    """Python int -> n little-endian uint32 limbs."""
    return (ctypes.c_uint32 * n).from_buffer_copy(x.to_bytes(4 * n, "little"))


def _mod(c):
    """One Montgomery context per odd modulus (pai_mod_create), kept for the life of the process."""
    with _lock:
        if c not in _mods:
            n = (c.bit_length() + 31) // 32
            h = ctypes.c_void_p()
            rc = _lib.pai_mod_create(_limbs(c, n), n, 0, ctypes.byref(h))
            if rc:
                raise RuntimeError("pai_mod_create: %s" % _lib.pai_last_error().decode())
            _mods[c] = (h, _lib.pai_mod_limbs(h))
        return _mods[c]


def _on_engine(c):
    return c > _USE_MOD_FROM_GMP_SIZE and c & 1 and c.bit_length() <= _MAX_BITS


def powmod(a, b, c):
    """phe/util.py:38-50: a ** b mod c (the body behind ``HAVE_GMP`` replaced by pai_mod_powmod_host)."""
    if a == 1:
        return 1
    if b < 0 or not _on_engine(c) or max(a, b, c) < _USE_MOD_FROM_GMP_SIZE:
        return pow(a, b, c)
    h, L = _mod(c)
    wide = 2 if (a < 0 or a.bit_length() > 32 * L) else 1          # raw_decrypt passes a 2x-wide base (:347)
    if a < 0 or a.bit_length() > 64 * L:
        a %= c
        wide = 1
    e = (b.bit_length() + 31) // 32 or 1
    out = (ctypes.c_uint32 * L)()
    rc = _lib.pai_mod_powmod_host(h, _limbs(a, wide * L), wide * L, _limbs(b, e), e, 1, out, 1)
    if rc:
        raise RuntimeError("pai_mod_powmod_host: %s" % _lib.pai_last_error().decode())
    return int.from_bytes(bytes(out), "little")


def mulmod(a, b, c):
    """phe/util.py:53-64: a * b mod c, non-negative also for negative a (crt, phe/paillier.py:373)."""
    if not _on_engine(c) or max(a, b, c) < _USE_MULMOD_FROM_GMP_SIZE:
        return a * b % c
    h, L = _mod(c)
    lim = 1 << (32 * L)
    a = a if 0 <= a < lim else a % c
    b = b if 0 <= b < lim else b % c
    out = (ctypes.c_uint32 * L)()
    rc = _lib.pai_mod_mulmod_host(h, _limbs(a, L), _limbs(b, L), out, 1)
    if rc:
        raise RuntimeError("pai_mod_mulmod_host: %s" % _lib.pai_last_error().decode())
    return int.from_bytes(bytes(out), "little")


def invert(a, b):
    """phe/util.py:85-103: a^-1 mod b; ZeroDivisionError('invert() no inverse exists') as at :96-97, 101-102."""
    if not _on_engine(b):
        g, s = b, 0                                    # plain extended Euclid for even / tiny moduli
        r0, r1, s0, s1 = a % b, b, 1, 0
        while r1:
            k = r0 // r1
            r0, r1, s0, s1 = r1, r0 - k * r1, s1, s0 - k * s1
        if r0 != 1:
            raise ZeroDivisionError('invert() no inverse exists')
        return s0 % b
    h, L = _mod(b)
    a = a if 0 <= a < (1 << (32 * L)) else a % b
    out = (ctypes.c_uint32 * L)()
    status = ctypes.c_int32(0)
    rc = _lib.pai_mod_invert_host(h, _limbs(a, L), L, out, ctypes.byref(status), 1)
    if rc:
        raise RuntimeError("pai_mod_invert_host: %s" % _lib.pai_last_error().decode())
    if status.value:
        raise ZeroDivisionError('invert() no inverse exists')
    return int.from_bytes(bytes(out), "little")


def install(phe, lib_path=None):
    """Rebind powmod / mulmod / invert in phe.util and -- because phe/paillier.py:29 imported them by name -- in
    phe.paillier."""
    load(lib_path)
    import phe.paillier as pp        # noqa: F401  (the module objects of the package passed in)
    import phe.util as pu
    for mod in (pu, pp):
        for name, fn in (("powmod", powmod), ("mulmod", mulmod), ("invert", invert)):
            _saved.setdefault((mod.__name__, name), getattr(mod, name))
            setattr(mod, name, fn)


def uninstall(phe):
    import phe.paillier as pp        # noqa: F401
    import phe.util as pu
    for mod in (pu, pp):
        for name in ("powmod", "mulmod", "invert"):
            orig = _saved.pop((mod.__name__, name), None)
            if orig is not None:
                setattr(mod, name, orig)
