"""Encryption with the private key (pai_priv_encrypt) on the test-only host simulation: the CRT arithmetic in pure Python,
bit equality with pai_encrypt and Python pow on edge rows, the routing between the thread-per-ciphertext kernel and the
warp-per-ciphertext route with its launch counts, independence from the kernel-family settings, the argument checks and
the Python API (PaillierPrivateKey.encrypt_batch / raw_encrypt_batch)."""
import contextlib
import importlib
import os
import random

import numpy as np
import pytest

from oracle.golden import H, load_golden

ENV_VARS = ("PAI_TC", "PAI_ENCRYPT_PATH", "PAI_DECRYPT_PATH", "PAI_COOP_MAX")
PAI_E_ARG = -1


@contextlib.contextmanager
def _env(**values):
    saved = {k: os.environ.get(k) for k in ENV_VARS}
    for k in ENV_VARS:
        os.environ.pop(k, None)
    os.environ.update(values)
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _is_prime(c):
    if c < 2:
        return False
    for sp in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if c % sp == 0:
            return c == sp
    d, s = c - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):        # deterministic below 3.3e24
        x = pow(a, d, c)
        if x in (1, c - 1):
            continue
        for _ in range(s - 1):
            x = x * x % c
            if x == c - 1:
                break
        else:
            return False
    return True


def _prime(rng, bits):
    while True:
        c = rng.getrandbits(bits) | (1 << (bits - 1)) | 1
        if _is_prime(c):
            return c


def _key(bits, pbits, seed):
    rng = random.Random(seed)
    while True:
        p, q = _prime(rng, pbits), _prime(rng, bits - pbits)
        if p != q and (p * q).bit_length() == bits:
            return p * q, min(p, q), max(p, q)


# the golden keys, and an unbalanced key whose private rows (two tiles per prime) are wider than its public ones (one)
KEYS = {"k256": "vectors_256.json", "k1024": "vectors_1024.json", "ntp2-300u": (300, 40, 5)}


def _keyof(name):
    k = KEYS[name]
    if isinstance(k, tuple):
        return _key(*k)
    fx = load_golden(k)
    return H(fx["n"]), min(H(fx["p"]), H(fx["q"])), max(H(fx["p"]), H(fx["q"]))


@pytest.fixture(scope="module")
def sim(pkg):
    import __graft_entry__ as ge
    return pkg.Engine(ge.build_hostsim())


@pytest.fixture(scope="module")
def E():
    return importlib.import_module("python-paillier_b200.engine")


def _edge_rows(n, p, q, ln, rng):
    top = (1 << (32 * ln)) - 1
    ms = [0, 1, n - 1, n, top]
    rs = [0, 1, p, q, 3 * p, n - 1, n, (top // q) * q, (top // q - 7) * q, top]
    rows = [(m, r) for m in ms for r in rs]
    rows += [(rng.randrange(n), rng.randrange(1, n)) for _ in range(6)] + [(rng.getrandbits(32 * ln), rng.getrandbits(32 * ln)) for _ in range(3)]
    return [m for m, _ in rows], [r for _, r in rows]


def _want(n, ms, rs):
    n2 = n * n
    return [(1 + n * m) * pow(r, n, n2) % n2 for m, r in zip(ms, rs)]


def _priv_encrypt(E, sim, priv, ms, rs):
    m, r = E.ints_to_limbs(ms, priv.n_limbs), E.ints_to_limbs(rs, priv.n_limbs)
    c = np.zeros((len(ms), priv.c_limbs), np.uint32)
    sim.check(sim.lib.pai_priv_encrypt(priv.h, E._ptr(m), E._ptr(r), E._ptr(c), len(ms), None))
    return E.limbs_to_ints(c)


# ---------------------------------------------------------------------------- the arithmetic, in Python
def test_crt_model_identities():
    """The three identities the kernels rest on, for primes of 10 to 64 bits (balanced and not) and every kind of r."""
    rng = random.Random(2024)
    for trial in range(60):
        pb = rng.randrange(10, 65)
        qb = pb if trial % 2 else rng.randrange(10, 65)
        p, q = _prime(rng, pb), _prime(rng, qb)
        if p == q:
            continue
        p, q = min(p, q), max(p, q)
        n, n2 = p * q, (p * q) ** 2
        for x, y in ((p, q), (q, p)):
            rs = [0, 1, x, 5 * x, n, n - 1, rng.randrange(n2), rng.randrange(1, n)]
            for r in rs:
                want = pow(r, n, x * x)
                s = pow(r % x, y % (x - 1), x)
                assert pow(s, x, x * x) == want                                # two short exponentiations
                assert pow(r, n % (x * (x - 1)), x * x) == want                # the warp route's exponent
        for m in (0, 1, n - 1, n, rng.randrange(n), rng.getrandbits(200)):
            r = rng.randrange(n2)
            cp = pow(r, n, p * p) * (1 + p * (q * m % p)) % (p * p)
            cq = pow(r, n, q * q) * (1 + q * (p * m % q)) % (q * q)
            h = (cq - cp) * pow(p * p, -1, q * q) % (q * q)
            assert cp + p * p * h == (1 + n * m) * pow(r, n, n2) % n2          # Garner, canonical as it stands


# ---------------------------------------------------------------------------- the engine
@pytest.mark.parametrize("key", list(KEYS))
def test_bit_equal_to_public_encrypt(pkg, sim, E, key):
    n, p, q = _keyof(key)
    with _env(PAI_COOP_MAX="0"):
        pub, priv = pkg.PublicContext(n, engine=sim), pkg.PrivateContext(p, q, engine=sim)
        assert priv.n_limbs >= pub.n_limbs
        ms, rs = _edge_rows(n, p, q, pub.n_limbs, random.Random(n % 1000003))
        got = _priv_encrypt(E, sim, priv, ms, rs)
        assert got == _want(n, ms, rs)
        assert got == E.limbs_to_ints(pub.encrypt_host(E.ints_to_limbs(ms, pub.n_limbs), E.ints_to_limbs(rs, pub.n_limbs)))
        assert priv.raw_encrypt(ms, rs) == got
        pub.close(); priv.close()


# launches of one call: first call on a fresh context (constants built on the host: no setup kernel), then a second call
ROUTES = {
    # name: (PAI_COOP_MAX, rows, launches of the first call, of the second)
    "kernel": ("0", 7, 1, 1),
    "tail": ("3", 7, 7, 3),             # one wave (4 rows here) on the kernel, 3 rows on the warp route
    "warp": ("100000", 3, 6, 2),
}


@pytest.mark.parametrize("key", ["k256", "ntp2-300u"])
def test_routes_bit_equal_and_launch_counts(pkg, sim, E, key):
    n, p, q = _keyof(key)
    rng = random.Random(17)
    launches = {}
    for name, (coop, rows, first, second) in ROUTES.items():
        with _env(PAI_COOP_MAX=coop):
            priv = pkg.PrivateContext(p, q, engine=sim)
            ms = [rng.randrange(n) for _ in range(rows - 2)] + [n - 1, 0]
            rs = [rng.randrange(1, n) for _ in range(rows - 2)] + [q, p]
            counts = []
            for _ in range(2):
                before = sim.launch_count()
                got = _priv_encrypt(E, sim, priv, ms, rs)
                counts.append(sim.launch_count() - before)
                assert got == _want(n, ms, rs), name                 # every route gives pai_encrypt's bits
            launches[name] = tuple(counts)
            priv.close()
    assert launches == {name: (v[2], v[3]) for name, v in ROUTES.items()}


@pytest.mark.parametrize("setting", [{"PAI_TC": "2"}, {"PAI_DECRYPT_PATH": "full"}, {"PAI_ENCRYPT_PATH": "full"}])
def test_independent_of_kernel_family(pkg, sim, E, setting):
    """The digit kernel runs whatever family is selected, and the private context keeps reporting decrypt's path and wave."""
    n, p, q = _keyof("k1024")
    ms, rs = [5, n - 1, 0], [n - 2, 3, 7]
    with _env(PAI_COOP_MAX="0", **setting):
        priv = pkg.PrivateContext(p, q, engine=sim)
        path, wave = priv.kernel_path(), priv.wave()
        assert _priv_encrypt(E, sim, priv, ms, rs) == _want(n, ms, rs)
        assert (priv.kernel_path(), priv.wave()) == (path, wave)
        c = E.ints_to_limbs(_want(n, ms, rs), priv.c_limbs)
        assert E.limbs_to_ints(priv.decrypt_host(c)) == [m % n for m in ms]
        priv.close()


def test_argument_checks(pkg, sim, E):
    n, p, q = _keyof("k256")
    with _env(PAI_COOP_MAX="0"):
        priv = pkg.PrivateContext(p, q, engine=sim)
        lib, P = sim.lib, E._ptr
        x = np.zeros((2, priv.c_limbs), np.uint32)
        calls = {
            "device": lambda h, ps, b: lib.pai_priv_encrypt(h, ps[0], ps[1], ps[2], b, None),
            "host": lambda h, ps, b: lib.pai_priv_encrypt_host(h, ps[0], ps[1], ps[2], b),
        }
        for name, fn in calls.items():
            ok = [P(x)] * 3
            assert fn(None, ok, 1) == PAI_E_ARG, name
            for i in range(3):
                assert fn(priv.h, ok[:i] + [None] + ok[i + 1:], 1) == PAI_E_ARG, (name, i)
            assert fn(priv.h, ok, -1) == PAI_E_ARG, name
            before = sim.launch_count()
            assert fn(priv.h, ok, 0) == 0, name
            assert sim.launch_count() == before, name
        priv.close()


# ---------------------------------------------------------------------------- Python API
@pytest.fixture
def api(pkg, sim):
    engine_mod = importlib.import_module("python-paillier_b200.engine")
    engine_mod._set_engine_for_tests(sim)
    yield
    engine_mod._set_engine_for_tests(None)
    importlib.import_module("python-paillier_b200.util")._ctx_cache.clear()


@pytest.mark.parametrize("key", ["k256", "ntp2-300u"])
def test_python_api(pkg, api, key):
    import torch
    n, p, q = _keyof(key)
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    rng = random.Random(3)
    with _env(PAI_COOP_MAX="0"):
        for values, precision in (([0.5, -1.25, 3.0, 1e-3, -7.0], None), ([0, 1, -1, 12345, -(n // 3 - 2)], None),
                                  ([1.5, -2.75, 0.0], 1e-4),
                                  ([pkg.EncodedNumber.encode(pk, 2.5), pkg.EncodedNumber.encode(pk, -3)], None)):
            rs = [rng.randrange(1, n) for _ in values]
            a = pk.encrypt_batch(values, precision=precision, r_values=rs)
            b = sk.encrypt_batch(values, precision=precision, r_values=rs)
            assert torch.equal(a.limbs, b.limbs) and np.array_equal(a.exponents, b.exponents)
            fresh = sk.encrypt_batch(values, precision=precision)
            assert fresh._obfuscated and not b._obfuscated
            assert fresh.decrypt(sk) == a.decrypt(sk)
        ms = [rng.randrange(n) for _ in range(6)] + [-5, n + 3]
        rs = [0, None, rng.randrange(1, n), n * n + 5, n, (1 << (32 * pk.engine_context().n_limbs)) + 11, n * n - 2, 1]
        fixed = [r if r else 9 for r in rs]
        assert sk.raw_encrypt_batch(ms, fixed) == pk.raw_encrypt_batch(ms, fixed) == \
            [pk.raw_encrypt(m, r) for m, r in zip(ms, fixed)]
        falsy = sk.raw_encrypt_batch([4, 5], [0, 0])                   # a fresh r each: decrypts to m
        assert sk.raw_decrypt_batch(falsy) == [4, 5]
