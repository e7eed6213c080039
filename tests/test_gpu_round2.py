"""Round-2 GPU tests: one context on two CUDA streams and on several host threads at once (per-stream scratch, context
lock), the multi-chunk persistent loop at the reference's default key size (>= 2 waves at 3072 bits), the pipelined
Python-int API, and EncryptedVector inside a non-default torch stream."""
import random
import threading

import numpy as np
import pytest

from oracle import paillier_oracle as orc
from oracle.golden import H, load_golden

pytestmark = pytest.mark.gpu


def _key(kb):
    fx = load_golden("vectors_%d.json" % kb)
    return H(fx["n"]), H(fx["p"]), H(fx["q"])


@pytest.fixture(scope="module")
def gmp():
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    yield
    orc.BACKEND = "python"


def _uniform(pub, rows, seed, nonce, stream=None):
    import torch
    t = torch.empty((rows, pub.n_limbs), dtype=torch.int32, device="cuda")
    pub.random_lt_n_dev(t, rows, seed=bytes([seed]) * 32, nonce=nonce, stream=stream)
    return t


def test_two_streams_one_context(pkg, cuda_engine, gmp):
    """Encrypt + decrypt + raw_mul of two different batches issued back to back on two streams of ONE context pair: the
    kernels overlap on the device (each batch is a fraction of a wave) and must not share window tables or counters."""
    import torch
    n, p, q = _key(1024)
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    rows = 20000
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    bufs = []
    for rep in range(3):
        for i, s in enumerate((s1, s2)):
            with torch.cuda.stream(s):
                st = int(s.cuda_stream)
                m = _uniform(pub, rows, 40 + i, 2 * rep, st)
                r = _uniform(pub, rows, 40 + i, 2 * rep + 1, st)
                c = torch.empty((rows, pub.c_limbs), dtype=torch.int32, device="cuda")
                d = torch.empty((rows, pub.n_limbs), dtype=torch.int32, device="cuda")
                k = torch.zeros((rows, pub.n_limbs), dtype=torch.int32, device="cuda")
                k[:, 0] = m[:, 0]
                e = torch.empty_like(c)
                status = torch.zeros((rows,), dtype=torch.int32, device="cuda")
                pub.encrypt_dev(m, r, c, rows, stream=st)
                pub.raw_mul_dev(c, k, e, status, rows, stream=st)
                priv.decrypt_dev(c, d, rows, stream=st)
                bufs.append((m, r, c, d, k, e, status))
    torch.cuda.synchronize()
    opub = orc.PublicConsts(n)
    rng = random.Random(1)
    for m, r, c, d, k, e, status in bufs:
        assert bool((d == m).all().item()) and not bool(status.any().item())
        idx = [0, rows - 1] + [rng.randrange(rows) for _ in range(6)]
        ti = torch.tensor(idx, device="cuda")
        mi, ri, ci, ki, ei = (pkg.limbs_to_ints(t[ti].cpu().numpy().view(np.uint32)) for t in (m, r, c, k, e))
        assert ci == [orc.raw_encrypt(opub, a, b) for a, b in zip(mi, ri)]
        assert ei == [orc.raw_mul(opub, a, b) for a, b in zip(ci, ki)]


def test_host_threads_share_a_key(pkg, cuda_engine, gmp):
    """The scalar phe API from 4 host threads on one key pair (ctypes releases the GIL): every result equals the oracle's."""
    n, p, q = _key(1024)
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    opub = orc.PublicConsts(n)
    errors = []

    def work(seed):
        try:
            rng = random.Random(seed)
            for _ in range(12):
                m, r = rng.randrange(n), rng.randrange(1, n)
                c = pk.raw_encrypt(m, r)
                if c != orc.raw_encrypt(opub, m, r) or sk.raw_decrypt(c) != m:
                    errors.append(seed)
            ms = [rng.randrange(n) for _ in range(300)]
            rs = [rng.randrange(1, n) for _ in range(300)]
            cs = pk.raw_encrypt_batch(ms, rs)
            if cs[::50] != [orc.raw_encrypt(opub, a, b) for a, b in zip(ms[::50], rs[::50])] or sk.raw_decrypt_batch(cs) != ms:
                errors.append(("batch", seed))
        except Exception as e:        # noqa: BLE001
            errors.append(repr(e))
    ts = [threading.Thread(target=work, args=(s,)) for s in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[:4]


def test_3072_bit_more_than_two_waves(pkg, cuda_engine, gmp):
    """The reference's default key size (phe/paillier.py:34) through >= 2 full waves + a ragged tail of the persistent
    kernels: whole-batch round trip on the device and sampled rows (first / last of every wave) against the oracle."""
    import torch
    n, p, q = _key(3072)
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    wave = pub.wave()
    rows = 2 * max(wave, priv.wave()) + wave // 3 + 5        # >= 2 waves of either kernel (their waves differ)
    m, r = _uniform(pub, rows, 7, 0), _uniform(pub, rows, 7, 1)
    c = torch.empty((rows, pub.c_limbs), dtype=torch.int32, device="cuda")
    d = torch.empty((rows, pub.n_limbs), dtype=torch.int32, device="cuda")
    pub.encrypt_dev(m, r, c, rows)
    priv.decrypt_dev(c, d, rows)
    assert bool((d == m).all().item())
    idx = sorted({0, 1, wave - 1, wave, wave + 1, 2 * wave - 1, 2 * wave, 2 * wave + 1, rows - 2, rows - 1,
                  priv.wave() - 1, priv.wave(), 2 * priv.wave()} | {random.Random(3).randrange(rows) for _ in range(20)})
    idx = [i for i in idx if 0 <= i < rows]
    ti = torch.tensor(idx, device="cuda")
    mi, ri, ci = (pkg.limbs_to_ints(t[ti].cpu().numpy().view(np.uint32)) for t in (m, r, c))
    opub = orc.PublicConsts(n)
    assert all(0 < x < n for x in mi + ri)                         # pai_random_lt_n range
    assert ci == [orc.raw_encrypt(opub, a, b) for a, b in zip(mi, ri)]


def test_python_int_pipeline_on_gpu(pkg, cuda_engine, gmp):
    """list[int] -> list[int] through the chunked pipeline (conversions overlapped with the kernels) at 3.5 waves."""
    n, p, q = _key(1024)
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    rows = int(3.5 * pk.engine_context().wave())
    rng = random.Random(2)
    ms = [rng.randrange(n) for _ in range(rows)]
    rs = [rng.randrange(1, n) for _ in range(rows)]
    cs = pk.raw_encrypt_batch(ms, rs)
    assert len(cs) == rows and sk.raw_decrypt_batch(cs) == ms
    opub = orc.PublicConsts(n)
    idx = [0, 1, rows // 2, rows - 1] + [rng.randrange(rows) for _ in range(28)]
    assert [cs[i] for i in idx] == [orc.raw_encrypt(opub, ms[i], rs[i]) for i in idx]


def test_vector_inside_a_torch_stream(pkg, cuda_engine):
    """EncryptedVector work issued inside `with torch.cuda.stream(s)` is ordered with torch's own kernels on that stream."""
    import torch
    n, p, q = _key(1024)
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    vals = np.random.RandomState(1).randn(3000) * 0.1
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        v = pk.encrypt_batch(vals)
        w = (v + v) * 0.5 + 1.0
        w.obfuscate()
        out = sk.decrypt_batch(w)
    assert np.allclose(out, vals + 1.0, rtol=0, atol=1e-12)


def test_fused_reductions_on_gpu(pkg, cuda_engine):
    """EncryptedVector.sum / dot on the GPU (shared-memory product tree, second launch over the CTA partials; the dot
    product's powers on the default digit kernels) against the launch chains and the plaintext results."""
    import torch
    n, p, q = _key(1024)
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    rng = np.random.RandomState(3)
    for count in (1, 5, 300, 70001):
        vals = rng.randint(-10 ** 6, 10 ** 6, size=count).astype(np.int64)
        v = pk.encrypt_batch(vals)
        s_f, s_c = v.sum(), v.sum_chain()
        assert s_f.ciphertext(False) == s_c.ciphertext(False)
        assert sk.decrypt(s_f) == int(vals.sum())
        ks = rng.randint(-2 ** 40, 2 ** 40, size=count).astype(np.int64)
        d_f = v.dot(ks)
        if count <= 300:
            assert d_f.ciphertext(False) == v.dot_chain(ks).ciphertext(False)
        assert sk.decrypt(d_f) == int((vals.astype(object) * ks.astype(object)).sum())
    fl = rng.randn(2000) * 0.1
    w = rng.randn(2000)
    v = pk.encrypt_batch(fl)
    assert abs(sk.decrypt(v.dot(w)) - float(fl @ w)) < 1e-6 and abs(sk.decrypt(v.sum()) - fl.sum()) < 1e-9
    torch.cuda.synchronize()


def test_batched_keygen_on_gpu(pkg, cuda_engine):
    """generate_paillier_keypairs: prime candidates tested by the batched Miller-Rabin kernel; every prime it returns is
    confirmed by the host-side is_prime (the reference's algorithm, phe/util.py:420-443), every key works."""
    import importlib
    import time
    util = importlib.import_module("python-paillier_b200.util")
    t0 = time.perf_counter()
    keys = pkg.generate_paillier_keypairs(12, n_length=2048)
    dt = time.perf_counter() - t0
    assert len(keys) == 12 and len({pk.n for pk, _ in keys}) == 12
    for pk, sk in keys[:4]:
        assert pk.n.bit_length() == 2048 and util.is_prime(sk.p, 8) and util.is_prime(sk.q, 8)
    pk, sk = keys[5]
    assert sk.decrypt(pk.encrypt(3.5) * 2) == 7.0
    cands = [2 ** 521 - 1, (2 ** 521 - 1) * 3 + 2, 3825123056546413051, 2 ** 1279 - 1, (2 ** 607 - 1) * (2 ** 521 - 1)]
    assert util.is_prime_batch(cands) == [True, util.is_prime((2 ** 521 - 1) * 3 + 2), False, True, False]
    print("12 x 2048-bit key pairs in %.1f s" % dt)
