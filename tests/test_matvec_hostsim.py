"""EncryptedVector.rmatmul (pai_raw_matvec: plaintext matrix times ciphertext vector with shared window tables) on the
test-only host simulation: every row must equal what the per-row and per-element APIs give, bit for bit."""
import importlib
import random

import numpy as np
import pytest

from oracle.golden import H, load_golden

sp = pytest.importorskip("scipy.sparse")


def _keys_on_hostsim(pkg, golden):
    import __graft_entry__ as ge
    engine_mod = importlib.import_module("python-paillier_b200.engine")
    engine_mod._set_engine_for_tests(pkg.Engine(ge.build_hostsim()))
    fx = load_golden(golden)
    pk = pkg.PaillierPublicKey(H(fx["n"]))
    return engine_mod, (pk, pkg.PaillierPrivateKey(pk, H(fx["p"]), H(fx["q"])), H(fx["p"]))


@pytest.fixture(scope="module", params=["vectors_256.json", "vectors_1024.json"])
def env(request, pkg):
    engine_mod, keys = _keys_on_hostsim(pkg, request.param)
    yield keys
    engine_mod._set_engine_for_tests(None)


@pytest.fixture(scope="module")
def env256(pkg):
    engine_mod, keys = _keys_on_hostsim(pkg, "vectors_256.json")
    yield keys
    engine_mod._set_engine_for_tests(None)


def _vector(pk, vals, seed):
    rng = random.Random(seed)
    return pk.encrypt_batch(vals, r_values=[rng.randrange(1, pk.n) for _ in vals])


def _same(vec, numbers):
    assert vec.ciphertexts(False) == [x.ciphertext(False) for x in numbers]
    assert vec.exponents.tolist() == [x.exponent for x in numbers]


def test_dense_rows_equal_dot(pkg, env):
    pk, sk, _ = env
    rng = np.random.default_rng(1)
    w = [float(x) for x in rng.normal(size=9)]
    w[3] = 5                                              # an int element: exponent 0 next to floats near -13
    w[6] = 1e-9
    v = _vector(pk, w, 1)
    X = rng.normal(size=(13, 9)) * 10.0 ** rng.integers(-3, 4, size=(13, 9))
    X[:, 2] = rng.integers(-50, 50, size=13)              # an int column (integer values in the float matrix)
    X[0, :] = 0.0                                         # a zero row
    X[1, ::2] = 0.0
    X[2, 4] = -0.0
    y = v.rmatmul(X)
    _same(y, [v.dot(X[j]) for j in range(X.shape[0])])
    assert np.allclose(sk.decrypt_batch(y), X @ np.array(w, dtype=float), rtol=1e-9, atol=1e-9)
    _same(X @ v, [v.dot(X[j]) for j in range(X.shape[0])])
    Xi = rng.integers(-1000, 1000, size=(6, 9))           # an int matrix
    _same(v.rmatmul(Xi), [v.dot(Xi[j]) for j in range(6)])
    _same(v.rmatmul(X.astype(np.float32)), [v.dot(X.astype(np.float32)[j]) for j in range(X.shape[0])])
    with pytest.raises(ValueError, match="dot"):
        v.rmatmul(X[0])
    with pytest.raises(ValueError):
        v.rmatmul(X[:, :5])


def _loop(x, weights, intercept=None):
    """the reference's encrypted_score (examples/logistic_regression_encrypted_model.py:170-174) on EncryptedNumbers"""
    _, idx = x.nonzero()
    score = intercept
    for i in idx:
        term = x[0, i] * weights[i]
        score = term if score is None else score + term
    return score


def test_sparse_rows_equal_the_reference_loop(pkg, env):
    pk, sk, _ = env
    rng = np.random.default_rng(2)
    d = 50
    w = [float(x) for x in rng.normal(size=d)]
    w[7] = -3
    v = _vector(pk, w, 2)
    nums = v.to_encrypted_numbers()
    rows = [[], [(4, 0.25)], [(d - 1, -2.0)], [(i, float(rng.uniform(-1, 1))) for i in range(0, d, 1) if i % 5]]
    rows += [[(int(i), float(rng.exponential())) for i in rng.choice(d, size=rng.integers(1, 6), replace=False)] for _ in range(9)]
    rows += [[(3, 0.0), (8, 1.5)], [(11, 0.0)], []]       # explicitly stored zeros
    indptr = np.cumsum([0] + [len(r) for r in rows])
    X = sp.csr_matrix((np.array([x for r in rows for _, x in r], dtype=float), np.array([i for r in rows for i, _ in r], dtype=np.int32),
                       indptr), shape=(len(rows), d))
    assert X.nnz == sum(len(r) for r in rows)
    y = v.rmatmul(X)
    for j in range(len(rows)):
        ref = _loop(X[j], nums)
        if ref is None:
            assert y[j].ciphertext(False) == 1 and y[j].exponent == 0
        else:
            assert y[j].ciphertext(False) == ref.ciphertext(False) and y[j].exponent == ref.exponent
    b = pk.encrypt(0.125, r_value=12345)
    yb = y + b
    _same(yb, [_loop(X[j], nums, intercept=b) for j in range(len(rows))])
    assert np.allclose(sk.decrypt_batch(yb), X @ np.array(w) + 0.125, atol=1e-9)
    for other in (sp.coo_matrix(X), sp.csc_array(X)):
        assert v.rmatmul(other).ciphertexts(False) == y.ciphertexts(False)


def test_indicator_matrix_is_a_segment_sum(pkg, env):
    pk, sk, _ = env
    rng = np.random.default_rng(3)
    count, nseg = 120, 9
    vals = [int(x) for x in rng.integers(-10 ** 6, 10 ** 6, size=count)]
    v = _vector(pk, vals, 3)
    seg = rng.integers(0, nseg - 1, size=count)            # the last segment stays empty
    X = sp.csr_matrix((np.ones(count, dtype=np.int64), (seg, np.arange(count))), shape=(nseg, count))
    ctx = pk.engine_context()
    assert ctx.matvec_window(count, nseg, count, 1, False) == 1    # B = 1: no squarings, no table products
    y = v.rmatmul(X)
    for j in range(nseg - 1):
        s = v[np.nonzero(seg == j)[0]].sum()
        assert y[j].ciphertext(False) == s.ciphertext(False) and y[j].exponent == s.exponent
    assert y[nseg - 1].ciphertext(False) == 1
    assert sk.decrypt_batch(y) == [sum(x for x, s in zip(vals, seg) if s == j) for j in range(nseg)]
    fv = _vector(pk, [float(x) for x in rng.normal(size=count)], 4)      # mixed exponents: BASE^delta in the scalars
    fy = fv.rmatmul(X)
    for j in range(nseg - 1):
        s = fv[np.nonzero(seg == j)[0]].sum()
        assert fy[j].ciphertext(False) == s.ciphertext(False) and fy[j].exponent == s.exponent


def test_large_scalars_and_bounds(pkg, env):
    pk, sk, _ = env
    v = _vector(pk, [3, -1, 7, 2], 5)
    big = np.array([[2 ** 62 - 1, -(2 ** 62) + 1, 1, 0], [2 ** 61, 5, -(2 ** 62) + 3, 2 ** 40]], dtype=np.int64)
    _same(v.rmatmul(big), [v.dot(big[j]) for j in range(2)])
    m = pk.max_int
    edge = np.array([[m, -m, 1, 0], [m // 2, 0, -m // 3, 2 ** 70]], dtype=object)
    _same(v.rmatmul(edge), [v.dot(edge[j]) for j in range(2)])
    mixed = _vector(pk, [3, 0.5], 6)                      # exponents 0 and -14: m is raised by BASE^28
    for row in ([m, 1.0], [-m, -0.25]):
        X = np.array([row], dtype=object)
        with pytest.raises(ValueError):
            mixed.dot(X[0])
        with pytest.raises(ValueError):
            mixed.rmatmul(X)


def test_non_invertible_ciphertext(pkg, env):
    pk, sk, p = env
    c2 = pk.encrypt(4, r_value=77)
    v = pkg.EncryptedVector.from_encrypted_numbers([pkg.EncryptedNumber(pk, p, 0), c2])
    with pytest.raises(ZeroDivisionError):
        v.dot([-1, 2])
    with pytest.raises(ZeroDivisionError):
        v.rmatmul(np.array([[1, 2], [-1, 2]]))
    y = v.rmatmul(np.array([[1, 2], [3, -2], [0, 1]]))
    nsq = pk.nsquare
    c = c2.ciphertext(False)
    assert y.ciphertexts(False) == [p * pow(c, 2, nsq) % nsq, pow(p, 3, nsq) * pow(c, -2, nsq) % nsq, c]


def test_against_python_pow(pkg, env):
    pk, sk, _ = env
    rng = np.random.default_rng(7)
    v = _vector(pk, [int(x) for x in rng.integers(-99, 99, size=11)], 7)
    cs = v.ciphertexts(False)
    nsq = pk.nsquare
    X = rng.integers(-2 ** 31, 2 ** 31, size=(17, 11))
    X[rng.random(X.shape) < 0.3] = 0
    y = v.rmatmul(X)
    want = []
    for row in X.tolist():
        acc = 1
        for c, k in zip(cs, row):
            acc = acc * pow(c, k, nsq) % nsq
        want.append(acc)
    assert y.ciphertexts(False) == want and not y.exponents.any()


@pytest.mark.parametrize("ncols, nrows, bits, want", [(200, 3, 20, 1), (4, 50, 40, 6), (30, 6, 12, 3)])
def test_window_choice(pkg, env256, ncols, nrows, bits, want):
    """the selector's pick for shapes whose tables do (not) fit the simulation's 64 KB table budget (128-byte entries at
    the 256-bit key), and a product at that pick"""
    pk, sk, _ = env256
    ctx = pk.engine_context()
    assert ctx.matvec_window(ncols, nrows, ncols * nrows, bits, False) == want
    rng = np.random.default_rng(ncols)
    v = _vector(pk, [int(x) for x in rng.integers(0, 1000, size=ncols)], 8)
    X = rng.integers(0, 2 ** bits, size=(nrows, ncols))
    X[:, 0] = 2 ** bits - 1                               # every row reaches the full bit length
    y = v.rmatmul(X)
    nsq = pk.nsquare
    cs = v.ciphertexts(False)
    want_rows = []
    for row in X.tolist():
        acc = 1
        for c, k in zip(cs, row):
            acc = acc * pow(c, k, nsq) % nsq
        want_rows.append(acc)
    assert y.ciphertexts(False) == want_rows


def test_vector_plus_encrypted_number(pkg, env):
    pk, sk, _ = env
    vals = [0.5, -2.0, 3, 1e-5]
    v = _vector(pk, vals, 9)
    nums = v.to_encrypted_numbers()
    for b in (pk.encrypt(1.25, r_value=99), pk.encrypt(7, r_value=98), pk.encrypt(-3e-9, r_value=97)):
        _same(v + b, [x + b for x in nums])
        assert np.allclose(sk.decrypt_batch(v + b), np.array(vals, dtype=float) + sk.decrypt(b))
