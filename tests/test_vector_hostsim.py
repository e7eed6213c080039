"""EncryptedVector and the vectorised EncodedNumber encode/decode on the test-only
host simulation: results must equal the per-element reference semantics exactly."""
import importlib
import random

import numpy as np
import pytest

from oracle.golden import H, load_golden


@pytest.fixture(scope="module")
def env(pkg):
    import __graft_entry__ as ge
    engine_mod = importlib.import_module("python-paillier_b200.engine")
    engine_mod._set_engine_for_tests(pkg.Engine(ge.build_hostsim()))
    fx = load_golden("vectors_256.json")
    pk = pkg.PaillierPublicKey(H(fx["n"]))
    sk = pkg.PaillierPrivateKey(pk, H(fx["p"]), H(fx["q"]))
    yield pk, sk, importlib.import_module("python-paillier_b200.vector")
    engine_mod._set_engine_for_tests(None)


def test_encode_decode_batch_exact(pkg, env):
    pk, sk, vec = env
    rng = random.Random(1)
    vals = [rng.gauss(0, 0.1) for _ in range(300)] + [0.0, -0.0, 1.0, -1.0, 1e-300, -1e-300, 1e30, -2.5e-7, float(2 ** 53), 0.1, 5e-324]
    limbs, exps = vec.encode_batch(pk, vals)
    ref = [pkg.EncodedNumber.encode(pk, v) for v in vals]
    assert pkg.limbs_to_ints(limbs) == [e.encoding for e in ref] and exps.tolist() == [e.exponent for e in ref]
    limbs, exps = vec.encode_batch(pk, np.array(vals))
    assert pkg.limbs_to_ints(limbs) == [e.encoding for e in ref]
    ivals = [rng.randrange(-2 ** 40, 2 ** 40) for _ in range(100)] + [0, 1, -1, 2 ** 61, -2 ** 61]
    limbs, exps = vec.encode_batch(pk, ivals)
    assert pkg.limbs_to_ints(limbs) == [pkg.EncodedNumber.encode(pk, v).encoding for v in ivals] and not exps.any()
    limbs, exps = vec.encode_batch(pk, vals[:50], max_exponent=[-15] * 50)
    ref15 = [pkg.EncodedNumber.encode(pk, v, max_exponent=-15) for v in vals[:50]]
    assert pkg.limbs_to_ints(limbs) == [e.encoding for e in ref15] and exps.tolist() == [e.exponent for e in ref15]
    mixed = [1, 2.5, -3, 10 ** 30]                        # falls back to the per-element path
    limbs, exps = vec.encode_batch(pk, mixed)
    assert pkg.limbs_to_ints(limbs) == [pkg.EncodedNumber.encode(pk, v).encoding for v in mixed]
    with pytest.raises(ValueError):
        vec.encode_batch(pk, [pk.max_int + 1, 1])
    encs = ref + [pkg.EncodedNumber.encode(pk, float(v)) for v in ivals]
    ln = pk.engine_context().n_limbs
    dec = vec.decode_batch(pk, pkg.ints_to_limbs([e.encoding for e in encs], ln), [e.exponent for e in encs])
    refd = [e.decode() for e in encs]
    assert all(a == b and type(a) is type(b) for a, b in zip(dec, refd))
    prods = [pkg.EncodedNumber(pk, (a.encoding * b.encoding) % pk.n, a.exponent + b.exponent) for a, b in zip(encs[:200], encs[100:300])]
    dec = vec.decode_batch(pk, pkg.ints_to_limbs([e.encoding for e in prods], ln), [e.exponent for e in prods])
    assert dec == [e.decode() for e in prods]
    with pytest.raises(OverflowError):
        vec.decode_batch(pk, pkg.ints_to_limbs([pk.max_int + 10], ln), [0])


def test_vector_ops_match_scalar_semantics(pkg, env):
    pk, sk, vec = env
    rng = random.Random(4)
    a = [rng.gauss(0, 1) for _ in range(9)] + [3, -4, 0]
    b = [rng.gauss(0, 1e-3) for _ in range(9)] + [1.5, 2, -7]
    ra = [rng.randrange(1, pk.n) for _ in a]
    rb = [rng.randrange(1, pk.n) for _ in b]
    va, vb = pk.encrypt_batch(a, r_values=ra), pk.encrypt_batch(b, r_values=rb)
    sa = [pk.encrypt(x, r_value=r) for x, r in zip(a, ra)]
    sb = [pk.encrypt(x, r_value=r) for x, r in zip(b, rb)]
    assert va.ciphertexts(False) == [x.ciphertext(False) for x in sa]
    for vres, sres in (((va + vb), [x + y for x, y in zip(sa, sb)]),
                       ((va + b), [x + y for x, y in zip(sa, b)]),
                       ((va * b), [x * y for x, y in zip(sa, b)]),
                       ((va - vb), [x - y for x, y in zip(sa, sb)]),
                       ((va / 4), [x / 4 for x in sa])):
        assert vres.ciphertexts(False) == [x.ciphertext(False) for x in sres]
        assert vres.exponents.tolist() == [x.exponent for x in sres]
        assert sk.decrypt_batch(vres) == [sk.decrypt(x) for x in sres]
    # all-float operands take the vectorised encode path (lists and numpy arrays): same bits as element by element
    bf = [float(x) for x in b]
    for operand in (bf, np.array(bf)):
        for vres, sres in (((va + operand), [x + y for x, y in zip(sa, bf)]), ((va * operand), [x * y for x, y in zip(sa, bf)]),
                           ((operand + va), [y + x for x, y in zip(sa, bf)])):
            assert vres.ciphertexts(False) == [x.ciphertext(False) for x in sres]
            assert vres.exponents.tolist() == [x.exponent for x in sres]
    bi = [int(x * 100) for x in b]
    assert (va * bi).ciphertexts(False) == [(x * y).ciphertext(False) for x, y in zip(sa, bi)]
    assert (va + bi).ciphertexts(False) == [(x + y).ciphertext(False) for x, y in zip(sa, bi)]
    assert sk.decrypt((va + vb).sum()) == pytest.approx(sum(a) + sum(b), abs=1e-12)
    fresh = pk.encrypt_batch(a)
    c0 = fresh.ciphertexts(False)
    assert fresh.ciphertexts(True) == c0                    # already obfuscated by the random r
    s = va + vb
    c1 = s.ciphertexts(False)
    assert s.ciphertexts(True) != c1 and sk.decrypt_batch(s) == [sk.decrypt(x + y) for x, y in zip(sa, sb)]
    back = pkg.EncryptedVector.from_encrypted_numbers(sa)
    assert back.ciphertexts(False) == va.ciphertexts(False) and len(back) == len(a)
    assert sk.decrypt(va.dot(b)) == pytest.approx(sum(x * y for x, y in zip(a, b)), abs=1e-12)
    # wire format of docs/serialisation.rst: readable with plain EncryptedNumber objects and back
    import json
    js = va.to_json(be_secure=False)
    d = json.loads(js)
    assert int(d["public_key"]["n"]) == pk.n
    nums = [pkg.EncryptedNumber(pk, int(c), int(e)) for c, e in d["values"]]
    assert [sk.decrypt(x) for x in nums] == sk.decrypt_batch(va)
    rt = pkg.EncryptedVector.from_json(js)
    assert rt.ciphertexts(False) == va.ciphertexts(False) and rt.exponents.tolist() == va.exponents.tolist()
    with pytest.raises(NotImplementedError):
        va * vb
    with pytest.raises(ValueError):
        va + pk.encrypt_batch([1.0])


def test_batched_codec_equals_scalar_codec(pkg):
    """encode_batch / decode_batch (vectorised) against EncodedNumber.encode / decode element by element, including
    magnitudes around 2^64 (the limit of the fast decode path), negatives that borrow across limbs, and values that
    must take the exact slow path."""
    import importlib
    import random
    import __graft_entry__ as ge
    engine_mod = importlib.import_module("python-paillier_b200.engine")
    vec = importlib.import_module("python-paillier_b200.vector")
    engine_mod._set_engine_for_tests(pkg.Engine(ge.build_hostsim()))
    try:
        fx = load_golden("vectors_1024.json")
        pk = pkg.PaillierPublicKey(H(fx["n"]))
        rng = random.Random(11)
        floats = [rng.uniform(-1, 1) * 10 ** rng.randrange(-30, 30) for _ in range(400)]
        floats += [0.0, -0.0, 1.0, -1.0, 2.0 ** 63, -(2.0 ** 63), 2.0 ** 64, -(2.0 ** 64), 2.0 ** 64 * (1 + 2 ** -52), 1e-300, -1e300,
                   float(2 ** 53 - 1), -float(2 ** 53 - 1), 5e-324]
        limbs, exps = vec.encode_batch(pk, floats)
        encs = [pkg.EncodedNumber.encode(pk, v) for v in floats]
        assert pkg.limbs_to_ints(limbs) == [e.encoding for e in encs] and exps.tolist() == [e.exponent for e in encs]
        assert vec.decode_batch(pk, limbs, exps) == [e.decode() for e in encs]
        # encodings built directly: every combination of small / large magnitude, sign and exponent
        n = pk.n
        mags = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1, 2 ** 64, 2 ** 64 + 1, (n & (2 ** 64 - 1)), (n & (2 ** 64 - 1)) + 1, 2 ** 200]
        cases = [(m, e) for m in mags for e in (-1, -13, -60, -249, -250, 0, 3)] + [(n - m, e) for m in mags[1:] for e in (-1, -13, -60, 0)]
        l2 = pkg.ints_to_limbs([c[0] for c in cases], limbs.shape[1])
        e2 = [c[1] for c in cases]
        assert vec.decode_batch(pk, l2, e2) == [pkg.EncodedNumber(pk, c[0], c[1]).decode() for c in cases]
    finally:
        engine_mod._set_engine_for_tests(None)


def test_fused_sum_and_dot_equal_the_launch_chains(pkg, env):
    """EncryptedVector.sum / dot (pai_raw_sum / pai_raw_dot: two-launch product reduction, Straus exponentiation) give the
    same ciphertext as the chains of raw_add / raw_mul launches they replace, and decrypt to the plaintext results --
    mixed exponents, negative and zero scalars, lengths that are not powers of two."""
    pk, sk, vec = env
    rng = random.Random(12)
    for count in (1, 2, 7, 33):
        vals = [rng.gauss(0, 1) for _ in range(count)]
        if count > 2:
            vals[1] = 3                                   # an int among floats: exponent 0 next to -13
        v = pk.encrypt_batch(vals, r_values=[rng.randrange(1, pk.n) for _ in vals])
        s_f, s_c = v.sum(), v.sum_chain()
        assert s_f.ciphertext(False) == s_c.ciphertext(False) and s_f.exponent == s_c.exponent
        assert abs(sk.decrypt(s_f) - sum(vals)) < 1e-9
        ks = [rng.gauss(0, 2) for _ in range(count)]
        if count > 2:
            ks[0], ks[2] = 0.0, -4
        d_f, d_c = v.dot(ks), v.dot_chain(ks)
        assert d_f.ciphertext(False) == d_c.ciphertext(False) and d_f.exponent == d_c.exponent
        assert abs(sk.decrypt(d_f) - sum(a * b for a, b in zip(vals, ks))) < 1e-6
        ki = [rng.randrange(-1000, 1000) for _ in range(count)]
        assert sk.decrypt(v.dot(np.array(ki))) == pytest.approx(sum(a * b for a, b in zip(vals, ki)), abs=1e-6)
    with pytest.raises(ValueError):
        v.dot([1.0])
