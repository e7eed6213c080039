"""Encryption with the private key (pai_priv_encrypt) on the H100: every row equals pai_encrypt on the same inputs, sampled
rows equal the GMP oracle and edge rows equal Python's pow, for one key per private tile class, over several waves with a
tail, a tail on the warp route and a batch entirely on it; a call on a side stream, private-key encryption and decryption
on one context from two host threads, and the encrypt_batch / decrypt_batch round trip."""
import random
import threading

import numpy as np
import pytest

from oracle import paillier_oracle as orc
from oracle.golden import H, load_golden

pytestmark = pytest.mark.gpu

# name -> (bits of n, bits of the smaller prime) or a golden key; "ntpK" is the private tile class (tiles of 256 bits per
# prime, from the larger prime), checked against pai_priv_n_limbs() = 16 * K before any row runs
KEYS = {"ntp1-500": (500, 250), "ntp2-1000u": (1000, 490), "ntp3-1025u": (1025, 512), "ntp4-2048": "vectors_2048.json",
        "ntp6-2049u": (2049, 1024), "ntp8-4096": "vectors_4096.json"}


def _prime(rng, bits):
    import importlib
    util = importlib.import_module("python-paillier_b200.util")
    while True:
        c = rng.getrandbits(bits) | (1 << (bits - 1)) | 1
        if util.is_prime(c):
            return c


def _key(name):
    k = KEYS[name]
    if isinstance(k, str):
        fx = load_golden(k)
        p, q = H(fx["p"]), H(fx["q"])
        return H(fx["n"]), min(p, q), max(p, q)
    rng = random.Random(k[0] * 31 + k[1])
    while True:
        p, q = _prime(rng, k[1]), _prime(rng, k[0] - k[1])
        if p != q and (p * q).bit_length() == k[0]:
            return p * q, min(p, q), max(p, q)


@pytest.fixture(scope="module")
def gmp():
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    yield
    orc.BACKEND = "python"


def _dev(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int32)).to("cuda:0")


def _edge(n, p, q, ln):
    top = (1 << (32 * ln)) - 1
    ms = [0, 1, n - 1, n, top]
    rs = [0, 1, p, q, 3 * p, n - 1, n, (top // q) * q, top]
    return [(m, r) for m in ms for r in rs]


def _run(pub, priv, m, r, batch, stream=None):
    """(private rows, public rows) as host arrays in the public layout"""
    import torch
    from importlib import import_module
    V = import_module("python-paillier_b200.vector")
    d_m, d_r = _dev(m), _dev(r)
    d_c = torch.empty((batch, pub.c_limbs), dtype=torch.int32, device="cuda:0")
    pub.encrypt_dev(d_m, d_r, d_c, batch)
    d_pc = torch.empty((batch, priv.c_limbs), dtype=torch.int32, device="cuda:0")
    priv.encrypt_dev(V._rows_for(priv.n_limbs, d_m), V._rows_for(priv.n_limbs, d_r), d_pc, batch, stream=stream)
    torch.cuda.synchronize()
    return V._to_host(V._rows_for(pub.c_limbs, d_pc)), V._to_host(d_c)


def _assert_routing_wave(eng, pub, priv, W):
    """pai_priv_encrypt routes by the wave of its own kernel, which it keeps internal; the batches of the test are sized
    from decrypt's wave W (pai_priv_wave).  The launch counts show that the two are equal: after a warm-up (constants,
    warp contexts), floor(0.3 W) rows take two launches (all on the warp route: both exponentiations of a row in one
    launch, then the tail), W rows one (a whole wave, no tail) and W + 1 rows three (one row on the warp route, the wave).
    The first bounds the internal wave w from below (floor(0.3 w) >= floor(0.3 W), so w >= W - 3); among those w only
    w = W gives no tail at W rows and a tail at W + 1."""
    import torch
    from importlib import import_module
    V = import_module("python-paillier_b200.vector")
    B = W + 1
    d_m = torch.zeros((B, priv.n_limbs), dtype=torch.int32, device="cuda:0")
    d_r = torch.zeros((B, pub.n_limbs), dtype=torch.int32, device="cuda:0")
    pub.random_lt_n_dev(d_r, B, seed=bytes(32))
    d_r = V._rows_for(priv.n_limbs, d_r)
    d_c = torch.empty((B, priv.c_limbs), dtype=torch.int32, device="cuda:0")
    priv.encrypt_dev(d_m, d_r, d_c, 1)
    torch.cuda.synchronize()
    launches = {}
    for rows in (W * 3 // 10, W, W + 1):
        before = eng.launch_count()
        priv.encrypt_dev(d_m, d_r, d_c, rows)
        torch.cuda.synchronize()
        launches[rows] = eng.launch_count() - before
    assert launches == {W * 3 // 10: 2, W: 1, W + 1: 3}, (W, launches)


@pytest.mark.parametrize("key", list(KEYS))
def test_rows_equal_public_encrypt_and_oracle(cuda_engine, gmp, pkg, key):
    from importlib import import_module
    E = import_module("python-paillier_b200.engine")
    n, p, q = _key(key)
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    assert priv.n_limbs == 16 * int(key[3]), (key, priv.n_limbs)
    opub = orc.PublicConsts(n)
    ln, W = pub.n_limbs, priv.wave()
    rng = random.Random(n % 999983)
    edge = _edge(n, p, q, ln)
    _assert_routing_wave(cuda_engine, pub, priv, W)
    # several waves and a tail (the tail below 0.3 wave goes to the warp route), a tail above it, and all on the warp route
    for batch in (3 * W + W // 7, 2 * W + W // 2, 7):
        rows = [(rng.randrange(n), rng.randrange(1, n)) for _ in range(batch)]
        at = [0, 1] + ([W - 2, W - 1, W, W + 1] if batch > W + 2 else [])
        for i, j in enumerate(at):                          # edge rows beside ordinary rows and on both sides of a wave boundary
            rows[j] = edge[(i * 7 + batch) % len(edge)]
        if batch == 7:
            rows[2:7] = edge[:5]
        m = np.zeros((batch, ln), np.uint32)
        r = np.zeros((batch, ln), np.uint32)
        m[:] = E.ints_to_limbs([x for x, _ in rows], ln)
        r[:] = E.ints_to_limbs([y for _, y in rows], ln)
        got, want = _run(pub, priv, m, r, batch)
        assert np.array_equal(got, want), (key, batch, np.nonzero((got != want).any(1))[0][:8])
        cs = E.limbs_to_ints(got)
        n2 = n * n
        for j in set(at) | set(range(2, 7) if batch == 7 else []):
            mj, rj = rows[j]
            assert cs[j] == (1 + n * mj) * pow(rj, n, n2) % n2, (key, batch, j)
        for j in random.Random(batch).sample(range(batch), min(64, batch)):
            mj, rj = rows[j]
            if 0 < rj < n:
                assert cs[j] == orc.raw_encrypt(opub, mj % n, rj), (key, batch, j)
    pub.close(); priv.close()


def test_side_stream_and_two_threads(cuda_engine, pkg):
    import torch
    n, p, q = _key("ntp4-2048")
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    rng = random.Random(5)
    B = 3000
    ms = [rng.randrange(n) for _ in range(B)]
    rs = [rng.randrange(1, n) for _ in range(B)]
    s = torch.cuda.Stream()
    from importlib import import_module
    E = import_module("python-paillier_b200.engine")
    m, r = E.ints_to_limbs(ms, pub.n_limbs), E.ints_to_limbs(rs, pub.n_limbs)
    with torch.cuda.stream(s):
        got, want = _run(pub, priv, m, r, B, stream=int(s.cuda_stream))
    assert np.array_equal(got, want)
    cs = E.limbs_to_ints(want)
    out = {}

    def enc():
        out["enc"] = priv.raw_encrypt(ms, rs)

    def dec():
        out["dec"] = priv.raw_decrypt(cs)
    ts = [threading.Thread(target=enc), threading.Thread(target=dec)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert out["enc"] == cs and out["dec"] == ms
    pub.close(); priv.close()


@pytest.mark.parametrize("kb", [2048, 3072])
def test_encrypt_batch_round_trip(cuda_engine, pkg, kb):
    import torch
    fx = load_golden("vectors_%d.json" % kb)
    pk = pkg.PaillierPublicKey(H(fx["n"]))
    sk = pkg.PaillierPrivateKey(pk, H(fx["p"]), H(fx["q"]))
    rng = random.Random(kb)
    vals = [rng.uniform(-1e6, 1e6) for _ in range(5000)] + [0, 1, -1, 2 ** 40]
    v = sk.encrypt_batch(vals)
    assert v._obfuscated
    assert sk.decrypt_batch(v) == pytest.approx(vals, rel=1e-12, abs=1e-9)
    rs = [rng.randrange(1, pk.n) for _ in vals]
    a, b = pk.encrypt_batch(vals, r_values=rs), sk.encrypt_batch(vals, r_values=rs)
    assert torch.equal(a.limbs, b.limbs) and np.array_equal(a.exponents, b.exponents)
