"""The tensor-core kernel family (pai_tc.cuh, PAI_TC=2) on the GPU at the digit sizes with code of their own: three groups
with x1 in L2 and the P2 staging (2048-bit encrypt / raw_mul, 3072-bit decrypt), a single group (3072-bit encrypt) and
four bands (4096-bit decrypt).  One full wave of either kernel plus a ragged tail, compared row for row with the
integer-pipe digit family and on sampled rows with the oracle."""
import random

import numpy as np
import pytest

from oracle import paillier_oracle as orc
from oracle.golden import H, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gmp():
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    yield
    orc.BACKEND = "python"


def _uniform(pub, rows, seed, nonce):
    import torch
    t = torch.empty((rows, pub.n_limbs), dtype=torch.int32, device="cuda")
    pub.random_lt_n_dev(t, rows, seed=bytes([seed]) * 32, nonce=nonce)
    return t


@pytest.mark.parametrize("kb", [2048, 3072, 4096])
def test_tc_family_full_wave_equals_digit_family_and_oracle(pkg, cuda_engine, gmp, monkeypatch, kb):
    import torch
    fx = load_golden("vectors_%d.json" % kb)
    n, p, q = H(fx["n"]), H(fx["p"]), H(fx["q"])
    monkeypatch.setenv("PAI_COOP_MAX", "0")                        # the throughput kernels even for the tail
    ctx = {}
    for family in ("2", "0"):                                      # read at context creation
        monkeypatch.setenv("PAI_TC", family)
        ctx[family] = (pkg.PublicContext(n), pkg.PrivateContext(p, q))
    (tpub, tpriv), (dpub, dpriv) = ctx["2"], ctx["0"]
    assert (tpub.kernel_path(), tpriv.kernel_path()) == ("tc" if kb <= 3072 else "digit", "tc")
    assert (dpub.kernel_path(), dpriv.kernel_path()) == ("digit", "digit")
    rows = max(tpub.wave(), tpriv.wave()) + 77
    m, r = _uniform(tpub, rows, 9, 0), _uniform(tpub, rows, 9, 1)
    k = torch.zeros_like(m)
    k[:, :2] = r[:, :2]                                            # 64-bit scalars
    out = {}
    for family, (pub, priv) in ctx.items():
        c = torch.empty((rows, pub.c_limbs), dtype=torch.int32, device="cuda")
        d = torch.empty_like(m)
        e = torch.empty_like(c)
        status = torch.ones((rows,), dtype=torch.int32, device="cuda")
        pub.encrypt_dev(m, r, c, rows)
        priv.decrypt_dev(c, d, rows)
        pub.raw_mul_dev(c, k, e, status, rows)
        torch.cuda.synchronize()
        out[family] = (c, d, e, status)
    (c, d, e, status), (c0, d0, e0, status0) = out["2"], out["0"]
    assert bool((d == m).all().item()) and bool((d0 == m).all().item())
    assert bool((c == c0).all().item()) and bool((e == e0).all().item())
    assert not bool(status.any().item()) and not bool(status0.any().item())
    waves = sorted({tpub.wave(), tpriv.wave()})
    idx = sorted({0, 1, rows - 2, rows - 1} | {w + o for w in waves for o in (-1, 0, 1)}
                 | {random.Random(kb).randrange(rows) for _ in range(10)})
    idx = [i for i in idx if 0 <= i < rows]
    ti = torch.tensor(idx, device="cuda")
    mi, ri, ci, ki, ei = (pkg.limbs_to_ints(t[ti].cpu().numpy().view(np.uint32)) for t in (m, r, c, k, e))
    opub = orc.PublicConsts(n)
    assert ci == [orc.raw_encrypt(opub, a, b) for a, b in zip(mi, ri)]
    assert ei == [orc.raw_mul(opub, a, b) for a, b in zip(ci, ki)]
    for pub, priv in ctx.values():
        pub.close(); priv.close()


def test_tc_family_straus_dot_product(pkg, cuda_engine, monkeypatch):
    """EncryptedVector.dot on the tensor-core Straus kernels (2048-bit key): a fraction of a wave (one element per Straus
    group) and more elements than a wave (two per group), against the launch chain and the plaintext result."""
    fx = load_golden("vectors_2048.json")
    n, p, q = H(fx["n"]), H(fx["p"]), H(fx["q"])
    monkeypatch.setenv("PAI_TC", "2")
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    assert pk.engine_context().kernel_path() == "tc"
    rng = np.random.RandomState(4)
    for count in (300, pk.engine_context().wave() + 77):
        vals = rng.randint(-10 ** 6, 10 ** 6, size=count).astype(np.int64)
        ks = rng.randint(-2 ** 40, 2 ** 40, size=count).astype(np.int64)
        v = pk.encrypt_batch(vals)
        d = v.dot(ks)
        if count <= 300:
            assert d.ciphertext(False) == v.dot_chain(ks).ciphertext(False)
        assert sk.decrypt(d) == int((vals.astype(object) * ks.astype(object)).sum())
