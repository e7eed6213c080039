"""EncryptedVector.rmatmul on the H100 (pai_raw_matvec: shared window tables, one Straus chain per row): several waves of
rows against the GMP oracle, v.dot and the plaintext product; a skewed sparse matrix; 3072- and 4096-bit keys; a call
inside a non-default torch stream."""
import random

import numpy as np
import pytest

from oracle import paillier_oracle as orc
from oracle.golden import H, load_golden

pytestmark = pytest.mark.gpu
sp = pytest.importorskip("scipy.sparse")


@pytest.fixture(scope="module")
def gmp():
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    yield
    orc.BACKEND = "python"


def _keys(pkg, kb):
    fx = load_golden("vectors_%d.json" % kb)
    pk = pkg.PaillierPublicKey(H(fx["n"]))
    return pk, pkg.PaillierPrivateKey(pk, H(fx["p"]), H(fx["q"]))


def _vector(pk, vals, seed):
    rng = random.Random(seed)
    return pk.encrypt_batch(vals, r_values=[rng.randrange(1, pk.n) for _ in vals])


def _oracle_row(pkg, pk, opub, cs, vexps, cols, vals):
    """prod_t raw_mul(c, enc(x) * BASE^delta mod n) over the row's terms, with dot()'s exponent alignment"""
    encs = [pkg.EncodedNumber.encode(pk, x) for x in vals]
    exps = [int(vexps[i]) + e.exponent for i, e in zip(cols, encs)]
    if not exps:
        return 1, 0
    low = min(exps)
    acc = 1
    for i, e, x in zip(cols, encs, exps):
        s = e.encoding * pkg.EncodedNumber.BASE ** (x - low) % pk.n
        acc = orc.raw_add(opub, acc, orc.raw_mul(opub, cs[i], s))
    return acc, low


def test_dense_waves_against_oracle_dot_and_plaintext(pkg, cuda_engine, gmp):
    pk, sk = _keys(pkg, 2048)
    opub = orc.PublicConsts(pk.n)
    wave = pk.engine_context().wave()
    nrows, d = 2 * wave + wave // 3 + 7, 6
    rng = np.random.default_rng(21)
    w = [float(x) for x in rng.normal(size=d)]
    v = _vector(pk, w, 21)
    X = rng.normal(size=(nrows, d))
    X[rng.random(X.shape) < 0.2] = 0.0
    X[5] = 0.0
    y = v.rmatmul(X)
    got = y.ciphertexts(False)
    cs = v.ciphertexts(False)
    sample = sorted(set([0, 5, nrows - 1, wave, 2 * wave] + random.Random(1).sample(range(nrows), 27)))
    for j in sample:
        c, e = _oracle_row(pkg, pk, opub, cs, v.exponents, list(range(d)), X[j].tolist())
        assert got[j] == c and y.exponents[j] == e, j
    for j in sample[:16]:
        ref = v.dot(X[j])
        assert got[j] == ref.ciphertext(False) and y.exponents[j] == ref.exponent
    assert np.allclose(sk.decrypt_batch(y), X @ np.array(w), rtol=1e-9, atol=1e-9)


def test_skewed_sparse_against_oracle(pkg, cuda_engine, gmp):
    pk, sk = _keys(pkg, 2048)
    opub = orc.PublicConsts(pk.n)
    rng = np.random.default_rng(22)
    nrows, d = 20011, 3000
    lens = rng.geometric(0.15, size=nrows) - 1
    lens[rng.random(nrows) < 0.05] = 0
    lens[[3, 777, 15000]] = [1500, 2000, 900]
    indptr = np.concatenate([[0], np.cumsum(lens)])
    indices = np.concatenate([rng.choice(d, size=k, replace=False) for k in lens]).astype(np.int32)
    data = rng.exponential(0.2, size=int(indptr[-1]))
    X = sp.csr_matrix((data, indices, indptr), shape=(nrows, d))
    w = [float(x) for x in rng.normal(size=d)]
    v = _vector(pk, w, 22)
    y = v.rmatmul(X)
    got = y.ciphertexts(False)
    cs = v.ciphertexts(False)
    empty = int(np.nonzero(lens == 0)[0][0])
    sample = sorted(set([3, 777, 15000, empty, nrows - 1] + random.Random(2).sample(range(nrows), 20)))
    for j in sample:
        row = X[j]
        c, e = _oracle_row(pkg, pk, opub, cs, v.exponents, row.indices.tolist(), row.data.tolist())
        assert got[j] == c and y.exponents[j] == e, j
    dec = sk.decrypt_batch(y)
    assert np.allclose(dec, X @ np.array(w), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("kb", [3072, 4096])
def test_small_dense_large_keys(pkg, cuda_engine, gmp, kb):
    pk, sk = _keys(pkg, kb)
    rng = np.random.default_rng(kb)
    w = [float(x) for x in rng.normal(size=7)]
    w[2] = -4
    v = _vector(pk, w, kb)
    X = rng.normal(size=(40, 7))
    X[:, 1] = rng.integers(-9, 9, size=40)
    X[0] = 0.0
    y = v.rmatmul(X)
    refs = [v.dot(X[j]) for j in range(40)]
    assert y.ciphertexts(False) == [r.ciphertext(False) for r in refs]
    assert y.exponents.tolist() == [r.exponent for r in refs]
    assert np.allclose(sk.decrypt_batch(y), X @ np.array(w), rtol=1e-9, atol=1e-9)


def test_inside_a_non_default_stream(pkg, cuda_engine):
    import torch
    pk, sk = _keys(pkg, 2048)
    rng = np.random.default_rng(23)
    v = _vector(pk, [float(x) for x in rng.normal(size=50)], 23)
    X = sp.random(3000, 50, density=0.1, format="csr", random_state=23)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        y = v.rmatmul(X) + pk.encrypt(0.5, r_value=5)
        y = y.rmatmul(sp.identity(3000, dtype=np.int64, format="csr"))      # int 1: the same rows back
    s.synchronize()
    b = pk.encrypt(0.5, r_value=5)
    ref = v.rmatmul(X) + b
    assert y.ciphertexts(False) == ref.ciphertexts(False) and y.exponents.tolist() == ref.exponents.tolist()
    assert np.allclose(sk.decrypt_batch(y), X @ np.array(v.decrypt(sk)) + 0.5, atol=1e-9)
