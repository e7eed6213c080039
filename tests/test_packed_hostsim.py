"""Packed fixed-point vectors on the test-only host simulation: pai_pack_slots / pai_unpack_slots against a pure-Python model
of the format (DESIGN.md §3.10), their status and argument checks and launch counts, and the PackedEncryptedVector API:
exact slot sums, bound tracking, input kinds, public- and private-key ciphertexts against Python ints, JSON."""
import importlib
import json
import random

import numpy as np
import pytest

from oracle.golden import H, load_golden

PAI_E_ARG = -1


def _prime(rng, bits):
    while True:
        c = rng.getrandbits(bits) | (1 << (bits - 1)) | 1
        if all(pow(a, c - 1, c) == 1 for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)):
            return c


def _golden(name):
    fx = load_golden(name)
    return H(fx["n"]), H(fx["p"]), H(fx["q"])


def _unbalanced_300():
    """n of 300 bits from a 40-bit and a 260-bit prime: the private rows (two tiles per prime) are wider than the public"""
    rng = random.Random(5)
    while True:
        p, q = _prime(rng, 40), _prime(rng, 260)
        if (p * q).bit_length() == 300:
            return p * q, p, q


@pytest.fixture(scope="module")
def E():
    return importlib.import_module("python-paillier_b200.engine")


@pytest.fixture(scope="module")
def sim(pkg, E):
    import __graft_entry__ as ge
    eng = pkg.Engine(ge.build_hostsim())
    E._set_engine_for_tests(eng)
    yield eng
    E._set_engine_for_tests(None)


# ---------------------------------------------------------------------------- the format, in Python
def model_pack(n, b, K, slots):
    return [sum(s << (b * j) for j, s in enumerate(slots[lo:lo + K])) % n for lo in range(0, len(slots), K)]


def model_unpack(n, b, K, m):
    """(K slots, is a packing) of a row m: a packing has balanced digits in (-2^(b-1), 2^(b-1)), the slots pack accepts,
    and nothing above slot K-1"""
    P = m if m <= (n - 1) // 2 else m - n
    out = []
    for _ in range(K):
        d = P & ((1 << b) - 1)
        d -= (1 << b) if d >= 1 << (b - 1) else 0
        out.append(d)
        P = (P - d) >> b
    ok = P == 0 and m < n and -(1 << (b - 1)) not in out
    return (out if ok else [0] * K), ok


def _pack(E, sim, pub, slots, b):
    K = pub.slots_per_row(b)
    rows = -(-len(slots) // K)
    s = np.array(slots, dtype=np.int64)
    m = np.full((rows, pub.n_limbs), 0xdeadbeef, np.uint32)
    st = np.full(rows, 7, np.int32)
    before = sim.launch_count()
    sim.check(sim.lib.pai_pack_slots(pub.h, E._ptr(s), len(slots), b, E._ptr(m), E._ptr(st), None))
    assert sim.launch_count() - before == 1
    return E.limbs_to_ints(m), st.tolist()


def _unpack(E, sim, pub, rows, b, count):
    m = E.ints_to_limbs(rows, pub.n_limbs)
    out = np.full(count, 12345, np.int64)
    st = np.full(len(rows), 7, np.int32)
    before = sim.launch_count()
    sim.check(sim.lib.pai_unpack_slots(pub.h, E._ptr(m), b, E._ptr(out), count, E._ptr(st), None))
    assert sim.launch_count() - before == 1
    return out.tolist(), st.tolist()


MODULI = {"k64": lambda: _golden("vectors_64.json")[0], "k256": lambda: _golden("vectors_256.json")[0],
          "k1024": lambda: _golden("vectors_1024.json")[0], "odd-2^255+1": lambda: 2 ** 255 + 1}


@pytest.mark.parametrize("key", list(MODULI))
@pytest.mark.parametrize("b", [2, 3, 31, 32, 33, 63])
def test_pack_and_unpack_equal_the_model(pkg, E, sim, key, b):
    n = MODULI[key]()
    L = n.bit_length()
    pub = pkg.PublicContext(n, engine=sim)
    K = pub.slots_per_row(b)
    assert K == (L - 1) // b
    top = (1 << (b - 1)) - 1
    rng = random.Random(L * 64 + b)
    cases = [[top] * K, [-top] * K, [(-1) ** j * top for j in range(K)], [-(-1) ** j * top for j in range(K)], [0] * K,
             [0] * (K - 1) + [-1], [1] + [0] * (K - 1), [rng.randint(-top, top) for _ in range(K)]]
    slots = [s for c in cases for s in c] + [rng.randint(-top, top) for _ in range(K // 2 + 1)]   # a last row not full
    for count in (len(slots), len(slots) - 1, 1):
        rows, st = _pack(E, sim, pub, slots[:count], b)
        assert rows == model_pack(n, b, K, slots[:count]) and st == [0] * len(rows), (key, b, count)
        got, st = _unpack(E, sim, pub, rows, b, count)
        assert got == slots[:count] and st == [0] * len(rows), (key, b, count)
    # the extreme packings themselves: |P| just below 2^(bK-1), the widest value the format produces
    extreme = model_pack(n, b, K, [top] * K + [-top] * K)
    assert max(abs(P if P <= n // 2 else P - n) for P in extreme).bit_length() == b * K - 1
    pub.close()


# n just above a power of two: when b divides bits(n) - 1, -(n-1)/2 has balanced digits with a top digit -2^(b-1)
STATUS_MODULI = dict(MODULI, **{"odd-2^256+1": lambda: 2 ** 256 + 1, "odd-2^2047+1": lambda: 2 ** 2047 + 1})


@pytest.mark.parametrize("key", list(STATUS_MODULI))
def test_status_of_slots_and_rows(pkg, E, sim, key):
    n = STATUS_MODULI[key]()
    pub = pkg.PublicContext(n, engine=sim)
    for b in (2, 3, 5, 17, 23, 31, 32, 33, 63):
        K = pub.slots_per_row(b)
        half = 1 << (b - 1)
        ok = [half - 1] * K
        slots = ok + [half] + [0] * (K - 1) + ok + [0] * (K - 1) + [-half] + ok[:1]
        rows, st = _pack(E, sim, pub, slots, b)
        assert st == [0, 1, 0, 1, 0] and rows[1] == 0 and rows[3] == 0, (key, b, st)
        assert rows[0] == rows[2] == model_pack(n, b, K, ok)[0]
        # rows that are not packings: beyond the widest packing, the centre-lift boundary, m >= n
        bK = b * K
        # beyond every packing (|P| < 2^(bK-1)): +-(n-1)/2, +-2^(bK-1); not residues: m >= n
        bad = [(n - 1) // 2, (n + 1) // 2, 1 << (bK - 1), n - (1 << (bK - 1)), n, n + 1, (1 << (32 * pub.n_limbs)) - 1]
        good = model_pack(n, b, K, [half - 1] * K + [1 - half] * K) + [0, n - 1]       # the widest packings, 0 and -1
        rng = random.Random(n % 99991 + b)
        either = [(1 << (bK - 1)) - 1, n - (1 << bK) if bK < n.bit_length() - 1 else n - 2]
        either += [rng.randrange(n) for _ in range(4)] + [rng.randrange(1 << (bK - 1)) * rng.choice([1, -1]) % n for _ in range(4)]
        rows = bad + good + either
        got, st = _unpack(E, sim, pub, rows, b, K * len(rows))
        want = [model_unpack(n, b, K, m) for m in rows]
        assert st == [0 if w[1] else 1 for w in want], (key, b, st)
        assert st[:len(bad) + len(good)] == [1] * len(bad) + [0] * len(good), (key, b, st)
        assert got == [s for w in want for s in w[0]]
        # a digit -2^(b-1) is refused: a row that is a packing but for one slot set to -2^(b-1)
        for j in (0, K - 1):
            sl = [half - 1] * K
            sl[j] = -half
            P = sum(x << (b * i) for i, x in enumerate(sl)) % n
            got, st = _unpack(E, sim, pub, [P], b, K)
            assert st == [1] and got == [0] * K, (key, b, j)
    pub.close()


def test_argument_checks(pkg, E, sim):
    n = _golden("vectors_256.json")[0]
    pub = pkg.PublicContext(n, engine=sim)
    lib = sim.lib
    s = np.zeros(8, np.int64)
    m = np.zeros((8, pub.n_limbs), np.uint32)
    st = np.zeros(8, np.int32)
    before = sim.launch_count()
    for b in (1, 64, 0, -3, 256):
        assert lib.pai_pack_slots_per_row(pub.h, b) == PAI_E_ARG
        assert lib.pai_pack_slots(pub.h, E._ptr(s), 8, b, E._ptr(m), E._ptr(st), None) == PAI_E_ARG
        assert lib.pai_unpack_slots(pub.h, E._ptr(m), b, E._ptr(s), 8, E._ptr(st), None) == PAI_E_ARG
    assert lib.pai_pack_slots_per_row(None, 8) == PAI_E_ARG
    assert lib.pai_pack_slots(pub.h, None, 8, 8, E._ptr(m), E._ptr(st), None) == PAI_E_ARG
    assert lib.pai_pack_slots(pub.h, E._ptr(s), 8, 8, E._ptr(m), None, None) == PAI_E_ARG
    assert lib.pai_pack_slots(pub.h, E._ptr(s), -1, 8, E._ptr(m), E._ptr(st), None) == PAI_E_ARG
    assert lib.pai_unpack_slots(pub.h, None, 8, E._ptr(s), 8, E._ptr(st), None) == PAI_E_ARG
    assert lib.pai_pack_slots(pub.h, E._ptr(s), 0, 8, E._ptr(m), E._ptr(st), None) == 0
    assert lib.pai_unpack_slots(pub.h, E._ptr(m), 8, E._ptr(s), 0, E._ptr(st), None) == 0
    assert sim.launch_count() == before
    assert lib.pai_pack_slots_per_row(pub.h, 63) == 255 // 63 and lib.pai_pack_slots_per_row(pub.h, 2) == 127
    pub.close()
    small = pkg.PublicContext(_golden("vectors_64.json")[0], engine=sim)
    assert lib.pai_pack_slots_per_row(small.h, 63) == 1
    with pytest.raises(ValueError):
        small.slots_per_row(64)
    small.close()


# ---------------------------------------------------------------------------- the Python API
KEYS = {"k256": lambda: _golden("vectors_256.json"), "k1024": lambda: _golden("vectors_1024.json"), "ntp2-300u": _unbalanced_300}


@pytest.fixture(scope="module", params=list(KEYS))
def keys(request, pkg, sim):
    n, p, q = KEYS[request.param]()
    pk = pkg.PaillierPublicKey(n)
    return pk, pkg.PaillierPrivateKey(pk, p, q)


def _quantised(x, f):
    return [round(float(v) * 2 ** f) for v in np.asarray(x, dtype=np.float64).reshape(-1)]


def test_sums_differences_and_scalars_are_exact(pkg, keys):
    import torch
    pk, sk = keys
    rng = np.random.default_rng(11)
    f = 20
    xs = [rng.uniform(-3, 3, size=37) for _ in range(4)]
    xs[0][:6] = [3.0, -3.0, 0.0, 2 ** -21, -(2 ** -21), 3 * 2 ** -21]        # at the bound, ties to even
    vs = [pk.encrypt_packed(x, 3.0, frac_bits=f, headroom=64) for x in xs]
    qs = [np.array(_quantised(x, f), dtype=np.int64) for x in xs]
    assert qs[0][3:6].tolist() == [0, 0, 2]
    total = sum(vs)
    assert total.slot_bound == 4 * vs[0].slot_bound
    assert total.decrypt_fixed(sk).tolist() == sum(qs).tolist()
    d = vs[0] - vs[1]
    assert d.decrypt_fixed(sk).tolist() == (qs[0] - qs[1]).tolist()
    assert (-vs[2]).decrypt_fixed(sk).tolist() == (-qs[2]).tolist()
    for c in (-5, 7, 0, 1, -1, np.int64(-3)):
        assert (vs[3] * c).decrypt_fixed(sk).tolist() == (qs[3] * int(c)).tolist(), c
        assert (c * vs[3]).slot_bound == vs[3].slot_bound * abs(int(c))
    out = sk.decrypt_batch(total)
    assert out.dtype == torch.float64 and tuple(out.shape) == (37,)
    assert out.tolist() == (sum(qs) * 2.0 ** -f).tolist()
    assert np.abs(out.numpy() - sum(xs)).max() <= 4 * 2.0 ** -(f + 1)


def test_bound_tracking(pkg, keys):
    pk, sk = keys
    # bound 1, f = 4: qmax = 16; headroom 4: 64 needs 7 bits, slots of 8 bits hold up to 127 = 7 * 16 + 15
    x = [1.0, -1.0, 0.5, -0.9375]
    v = pk.encrypt_packed(x, 1.0, frac_bits=4, headroom=4)
    assert (v.slot_bits, v.slot_bound) == (8, 16)
    acc = v
    for _ in range(6):
        acc = acc + v
    assert acc.slot_bound == 112
    assert acc.decrypt_fixed(sk).tolist() == [7 * q for q in _quantised(x, 4)]
    with pytest.raises(OverflowError):
        acc + v
    with pytest.raises(OverflowError):
        acc - v
    with pytest.raises(OverflowError):
        sum([v] * 8)
    assert (v * 7).decrypt_fixed(sk).tolist() == [7 * q for q in _quantised(x, 4)]
    assert (v * -7).slot_bound == 112
    for c in (8, -8, 2 ** 40):
        with pytest.raises(OverflowError):
            v * c
    # the bound comes from the declaration: small data under a large bound still gets the large bound
    w = pk.encrypt_packed([0.0, 0.001], 1000.0, frac_bits=0, headroom=1)
    assert (w.slot_bits, w.slot_bound) == (11, 1000)


def test_errors(pkg, keys):
    import torch
    pk, sk = keys
    v = pk.encrypt_packed([0.5, 1.5], 2.0)
    for bad in ([float("nan")], [float("inf")], [2.5], [-2.0000001], np.array([3], dtype=np.int64), torch.tensor([-3])):
        with pytest.raises(ValueError):
            pk.encrypt_packed(bad, 2.0)
    for kw in ({"bound": 0}, {"bound": -1.0}, {"bound": float("nan")}, {"bound": 2.0, "frac_bits": -1},
               {"bound": 2.0, "headroom": 0}, {"bound": 2.0 ** 40, "frac_bits": 24}):        # the last needs 75-bit slots
        with pytest.raises(ValueError):
            pk.encrypt_packed([0.5], **kw)
    with pytest.raises(ValueError):
        pk.encrypt_packed([0.5, 1.5], 2.0, r_values=[1, 2, 3])
    with pytest.raises(TypeError):
        v * 2.0
    with pytest.raises(TypeError):
        v * np.float64(3)
    with pytest.raises(NotImplementedError):
        v * v
    for other in (pk.encrypt_packed([0.5, 1.5], 2.0, frac_bits=23), pk.encrypt_packed([0.5, 1.5, 1.0], 2.0),
                  pk.encrypt_packed([[0.5, 1.5]], 2.0), pk.encrypt_packed([0.5, 1.5], 2.0, headroom=1 << 20),
                  pk.encrypt_batch([0.5, 1.5])):
        with pytest.raises(ValueError):
            v + other
        with pytest.raises(ValueError):
            v - other
    other_pk = pkg.PaillierPublicKey(_golden("vectors_512.json")[0])
    with pytest.raises(ValueError):
        v + other_pk.encrypt_packed([0.5, 1.5], 2.0)
    with pytest.raises(TypeError):
        v + 1.0
    assert 0 + v is v and v + 0 is v
    tiny = pkg.PaillierPublicKey(1000003 * 999983)           # 40 bits: a 42-bit slot does not fit
    with pytest.raises(ValueError):
        tiny.encrypt_packed([1.0], 2.0 ** 30, frac_bits=0, headroom=2 ** 10)
    assert tiny.encrypt_packed([1.0], 2.0 ** 30, frac_bits=0, headroom=2 ** 7).slots_per_ciphertext == 1


@pytest.mark.parametrize("kind", ["list", "np64", "np32", "npint", "torch", "torch-int", "torch-f16"])
def test_input_kinds_keep_the_shape(pkg, keys, kind):
    import torch
    pk, sk = keys
    base = np.array([[0.25, -1.5, 2.0], [3.125, -0.0, 1.0 / 3]])
    ints = np.array([[3, -4, 0], [7, 1, -2]], dtype=np.int64)
    x = {"list": base.tolist(), "np64": base, "np32": base.astype(np.float32), "npint": ints, "torch": torch.from_numpy(base),
         "torch-int": torch.from_numpy(ints).to(torch.int32), "torch-f16": torch.from_numpy(base).to(torch.float16)}[kind]
    v = pk.encrypt_packed(x, 8, frac_bits=10)
    assert v.shape == (2, 3) and len(v) == 6
    ref = np.asarray(x.float().numpy() if kind == "torch-f16" else (x.numpy() if kind.startswith("torch") else x), dtype=np.float64)
    assert v.decrypt_fixed(sk).reshape(-1).tolist() == _quantised(ref, 10)
    assert v.decrypt(sk).numpy().tolist() == (np.array(_quantised(ref, 10)) * 2.0 ** -10).reshape(2, 3).tolist()
    s = pk.encrypt_packed(np.float64(1.5), 2.0)            # a 0-d input
    assert s.shape == () and s.decrypt(sk).item() == 1.5


def test_ciphertexts_equal_python_ints(pkg, keys):
    import torch
    pk, sk = keys
    n, n2 = pk.n, pk.nsquare
    rng = random.Random(n % 1000003)
    x = [rng.uniform(-4, 4) for _ in range(29)] + [4.0, -4.0]
    probe = pk.encrypt_packed(x, 4.0, frac_bits=16, headroom=8)
    b, K = probe.slot_bits, probe.slots_per_ciphertext
    assert K == (n.bit_length() - 1) // b
    rows = -(-len(x) // K)
    rs = [rng.randrange(1, n) for _ in range(rows)]
    a, c = pk.encrypt_packed(x, 4.0, frac_bits=16, headroom=8, r_values=rs), sk.encrypt_packed(x, 4.0, frac_bits=16, headroom=8, r_values=rs)
    assert torch.equal(a.ciphertexts.limbs, c.ciphertexts.limbs) and not a.ciphertexts.exponents.any()
    P = model_pack(n, b, K, _quantised(x, 16))
    assert a.ciphertexts.ciphertexts(False) == [(1 + n * m) * pow(r, n, n2) % n2 for m, r in zip(P, rs)]
    fresh = sk.encrypt_packed(x, 4.0, frac_bits=16, headroom=8)
    assert fresh.ciphertexts._obfuscated and fresh.decrypt_fixed(sk).tolist() == _quantised(x, 16)
    before = a.ciphertexts.ciphertexts(False)
    a.obfuscate()
    assert a.ciphertexts.ciphertexts(False) != before and a.decrypt_fixed(sk).tolist() == _quantised(x, 16)


def test_json_round_trip(pkg, keys):
    pk, sk = keys
    x = np.linspace(-2, 2, 23).reshape(23, 1)
    v = sum([pk.encrypt_packed(x, 2.0, frac_bits=12) for _ in range(3)])
    s = v.to_json()
    d = json.loads(s)
    assert d["packing"] == {"shape": [23, 1], "slot_bits": v.slot_bits, "frac_bits": 12, "slot_bound": v.slot_bound}
    assert len(d["ciphertexts"]["values"]) == len(v.ciphertexts)
    for w in (pkg.PackedEncryptedVector.from_json(s), pkg.PackedEncryptedVector.from_json(s, pk)):
        assert (w.shape, w.slot_bits, w.frac_bits, w.slot_bound) == (v.shape, v.slot_bits, v.frac_bits, v.slot_bound)
        assert w.decrypt_fixed(sk).tolist() == v.decrypt_fixed(sk).tolist()
    other_pk = pkg.PaillierPublicKey(_golden("vectors_512.json")[0])
    with pytest.raises(ValueError):
        pkg.PackedEncryptedVector.from_json(s, other_pk)

    def broken(**change):
        e = json.loads(s)
        e["packing"].update(change)
        return json.dumps(e)
    for bad in (broken(shape=[23, 1000]), broken(shape=[-1]), broken(slot_bits=1), broken(slot_bits=64), broken(slot_bits=True),
                broken(frac_bits=-1), broken(slot_bound=1 << (v.slot_bits - 1)), broken(slot_bound=-1), broken(shape="23"),
                json.dumps({"ciphertexts": d["ciphertexts"]}), json.dumps({"packing": d["packing"], "ciphertexts": "x"}),
                json.dumps({"packing": d["packing"], "ciphertexts": {"values": d["ciphertexts"]["values"]}}),
                json.dumps({"packing": d["packing"], "ciphertexts": {"public_key": d["ciphertexts"]["public_key"]}}),
                json.dumps({"packing": d["packing"], "ciphertexts": dict(d["ciphertexts"], values=[[]])}),
                json.dumps({"packing": d["packing"], "ciphertexts": dict(d["ciphertexts"], values=7)}),
                json.dumps({"packing": d["packing"], "ciphertexts": dict(d["ciphertexts"], public_key=[1])}),
                json.dumps({"packing": d["packing"], "ciphertexts": dict(d["ciphertexts"], values=["12"])})):
        with pytest.raises(ValueError):
            pkg.PackedEncryptedVector.from_json(bad, pk)
    e = json.loads(s)
    e["ciphertexts"]["values"][0][1] = -3                   # a row with an exponent is not a packing's
    with pytest.raises(ValueError):
        pkg.PackedEncryptedVector.from_json(json.dumps(e), pk)


def test_a_row_that_is_not_a_packing_is_refused(pkg, keys):
    pk, sk = keys
    v = pk.encrypt_packed([1.0, -1.0], 1.0, frac_bits=4, headroom=2)
    k = v.slots_per_ciphertext * v.slot_bits
    n = pk.n
    # 2^(bK-1), +-(n-1)/2 and a row whose top slot is -2^(b-1): none is a packing
    top = sum(s << (v.slot_bits * j) for j, s in enumerate([0] * (v.slots_per_ciphertext - 1) + [-(1 << (v.slot_bits - 1))]))
    for m in (2 ** (k - 1), (n - 1) // 2, (n + 1) // 2, top % n):
        v.ciphertexts = pkg.EncryptedVector.encrypt_encoded(pk, [m], [0], r_values=[3])
        with pytest.raises(ValueError):
            v.decrypt_fixed(sk)
