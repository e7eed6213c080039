"""GPU parity at scale through size-independent properties (BASELINE.json configs 2-5 shapes), plus the
drop-in Python layer and EncryptedVector running on the CUDA engine."""
import random

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


def _rand_rows(rng, rows, limbs, top):
    a = rng.integers(0, 2 ** 32, size=(rows, limbs), dtype=np.uint32)
    a[:, top:] = 0
    return a


@pytest.mark.parametrize("kb,batch", [(2048, 40000), (3072, 9000), (1024, 70000)])
def test_roundtrip_and_sampled_oracle(pkg, cuda_engine, gmp, kb, batch):
    """configs[1]/[3] shape: dec(enc(m)) == m for the whole batch on device + sampled bit-exact check."""
    import torch
    n, p, q = _key(kb)
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    rng = np.random.default_rng(kb)
    m = _rand_rows(rng, batch, pub.n_limbs, kb // 32 - 1)
    r = _rand_rows(rng, batch, pub.n_limbs, kb // 32 - 1)
    r[:, 0] |= 1
    # edge rows: m = 0, m = n - 1, r = 1, r = n - 1
    m[0] = 0
    m[1] = pkg.ints_to_limbs([n - 1], pub.n_limbs)[0]
    r[2] = pkg.ints_to_limbs([1], pub.n_limbs)[0]
    r[3] = pkg.ints_to_limbs([n - 1], pub.n_limbs)[0]
    d_m = torch.from_numpy(m.view(np.int32)).cuda()
    d_r = torch.from_numpy(r.view(np.int32)).cuda()
    d_c = torch.empty((batch, pub.c_limbs), dtype=torch.int32, device="cuda")
    d_d = torch.empty((batch, pub.n_limbs), dtype=torch.int32, device="cuda")
    pub.encrypt_dev(d_m, d_r, d_c, batch)
    priv.decrypt_dev(d_c, d_d, batch)
    assert bool((d_d == d_m).all().item())
    idx = [0, 1, 2, 3] + random.Random(kb).sample(range(batch), 60)
    ms = pkg.limbs_to_ints(m[idx])
    rs = pkg.limbs_to_ints(r[idx])
    cs = pkg.limbs_to_ints(d_c[idx].cpu().numpy().view(np.uint32))
    opub = orc.PublicConsts(n)
    assert cs == [orc.raw_encrypt(opub, a, b) for a, b in zip(ms, rs)]


def test_homomorphism_add_mul_at_scale(pkg, cuda_engine, gmp):
    """configs[2] shape (2048-bit): D(E(a)*E(b)) = a+b mod n and D(E(a)^k) = a*k mod n for the whole batch,
    checked on device with plain limb arithmetic for small operands, plus sampled oracle equality."""
    import torch
    kb, batch = 2048, 30000
    n, p, q = _key(kb)
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    rng = np.random.default_rng(5)
    ln, lc = pub.n_limbs, pub.c_limbs
    a = np.zeros((batch, ln), dtype=np.uint32); a[:, 0] = rng.integers(0, 2 ** 31, batch)
    b = np.zeros((batch, ln), dtype=np.uint32); b[:, 0] = rng.integers(0, 2 ** 31, batch)
    k = np.zeros((batch, ln), dtype=np.uint32); k[:, 0] = rng.integers(0, 2 ** 31, batch); k[:, 1] = rng.integers(0, 2 ** 32, batch)
    ra, rb = _rand_rows(rng, batch, ln, kb // 32 - 1), _rand_rows(rng, batch, ln, kb // 32 - 1)
    ra[:, 0] |= 1; rb[:, 0] |= 1
    dev = lambda x: torch.from_numpy(x.view(np.int32)).cuda()
    d_ca = torch.empty((batch, lc), dtype=torch.int32, device="cuda"); d_cb = torch.empty_like(d_ca)
    d_s = torch.empty_like(d_ca); d_t = torch.empty_like(d_ca)
    st = torch.zeros((batch,), dtype=torch.int32, device="cuda")
    pub.encrypt_dev(dev(a), dev(ra), d_ca, batch)
    pub.encrypt_dev(dev(b), dev(rb), d_cb, batch)
    pub.raw_add_dev(d_ca, d_cb, d_s, batch)
    pub.raw_mul_dev(d_ca, dev(k), d_t, st, batch)
    assert not bool(st.any().item())
    d_ds = torch.empty((batch, ln), dtype=torch.int32, device="cuda"); d_dt = torch.empty_like(d_ds)
    priv.decrypt_dev(d_s, d_ds, batch)
    priv.decrypt_dev(d_t, d_dt, batch)
    got_sum = pkg.limbs_to_ints(d_ds.cpu().numpy().view(np.uint32))
    got_mul = pkg.limbs_to_ints(d_dt.cpu().numpy().view(np.uint32))
    av, bv = a[:, 0].astype(object), b[:, 0].astype(object)
    kv = k[:, 0].astype(object) + (k[:, 1].astype(object) << 32)
    assert got_sum == [int(x + y) for x, y in zip(av, bv)]
    assert got_mul == [int(x * y) for x, y in zip(av, kv)]
    opub = orc.PublicConsts(n)
    idx = random.Random(1).sample(range(batch), 40)
    ca = pkg.limbs_to_ints(d_ca[idx].cpu().numpy().view(np.uint32))
    cb = pkg.limbs_to_ints(d_cb[idx].cpu().numpy().view(np.uint32))
    cs = pkg.limbs_to_ints(d_s[idx].cpu().numpy().view(np.uint32))
    ct = pkg.limbs_to_ints(d_t[idx].cpu().numpy().view(np.uint32))
    assert cs == [orc.raw_add(opub, x, y) for x, y in zip(ca, cb)]
    assert ct == [orc.raw_mul(opub, x, int(kv[i])) for x, i in zip(ca, idx)]


@pytest.mark.parametrize("coop_max", ["0", "1024"])
def test_negative_scalars_and_ragged_batches(pkg, cuda_engine, gmp, monkeypatch, coop_max):
    """_raw_mul's inverse branch at 2048 bit, empty / 1 / non-multiple-of-warp batches, on the thread-per-ciphertext
    kernels (PAI_COOP_MAX=0) and on the warp-per-ciphertext ones."""
    monkeypatch.setenv("PAI_COOP_MAX", coop_max)
    n, p, q = _key(2048)
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    opub = orc.PublicConsts(n)
    rng = random.Random(9)
    assert pub.raw_encrypt([], []) == [] and priv.raw_decrypt([]) == [] and pub.raw_add([], []) == []
    for batch in (1, 31, 33, 225):
        m = [rng.randrange(n) for _ in range(batch)]
        r = [rng.randrange(1, n) for _ in range(batch)]
        c = pub.raw_encrypt(m, r)
        assert priv.raw_decrypt(c) == m
    m = [rng.randrange(n) for _ in range(48)]
    c = pub.raw_encrypt(m, [rng.randrange(1, n) for _ in m])
    ks = [n - 1 - rng.getrandbits(rng.choice([8, 53, 64])) for _ in m[:24]] + [rng.getrandbits(64) for _ in m[24:]]
    out, st = pub.raw_mul(c, ks)
    assert st == [0] * 48
    assert out == [orc.raw_mul(opub, x, k) for x, k in zip(c, ks)]
    assert priv.raw_decrypt(out) == [(a * k) % n for a, k in zip(m, ks)]
    out, st = pub.raw_mul([0, n, p, c[0]], [n - 3] * 4)          # non-invertible ciphertexts -> status 1
    assert st == [1, 1, 1, 0]


def test_dropin_api_and_vector_on_gpu(pkg, cuda_engine):
    """The phe-compatible layer on the real engine: config-1 fixture rows (bit-exact ciphertexts), operator
    fixture, and the federated-learning shape with EncryptedVector (configs[4] protocol, small D)."""
    c1 = load_golden("config1_1024.json")
    pk = pkg.PaillierPublicKey(H(c1["n"]))
    sk = pkg.PaillierPrivateKey(pk, H(c1["p"]), H(c1["q"]))
    rows = c1["rows"]
    vec = pk.encrypt_batch([row["x"] for row in rows], r_values=[H(row["r"]) for row in rows])
    assert vec.ciphertexts(be_secure=False) == [H(row["c"]) for row in rows]          # all 256 rows, one launch
    assert sk.decrypt_batch(vec) == [row["x"] for row in rows]
    e = pk.encrypt(rows[0]["x"], r_value=H(rows[0]["r"]))
    assert e.ciphertext(False) == H(rows[0]["c"]) and sk.decrypt(e) == rows[0]["x"]
    api = load_golden("api_1024.json")
    for op in api["ops"]:
        a, b = eval(op["a"]), eval(op["b"])
        ea, eb = pk.encrypt(a, r_value=H(op["ra"])), pk.encrypt(b, r_value=H(op["rb"]))
        for name, val in (("add", ea + eb), ("add_scalar", ea + b), ("mul", ea * b), ("sub", ea - eb), ("div4", ea / 4)):
            assert [val.ciphertext(False), val.exponent] == [H(op[name][0]), op[name][1]], name
            assert repr(sk.decrypt(val)) == op[name][2], name
    # federated protocol shape: 5 clients, gradient of D floats, ring-sum of encrypted vectors, decrypt, / n_clients
    D, n_clients = 600, 5
    grads = [np.random.RandomState(43 + i).randn(D) * 0.1 for i in range(n_clients)]
    acc = pk.encrypt_batch(grads[0].tolist())
    for g in grads[1:]:
        acc = acc + pk.encrypt_batch(g.tolist())
    agg = np.array(sk.decrypt_batch(acc)) / n_clients
    assert np.allclose(agg, np.mean(grads, axis=0), rtol=0, atol=1e-12)
    scaled = sk.decrypt_batch(acc * 0.5)
    assert np.allclose(scaled, 0.5 * np.sum(grads, axis=0), atol=1e-12)
    assert sk.decrypt(acc.sum()) == pytest.approx(float(np.sum(grads)), abs=1e-9)
    lst = acc[:3].to_encrypted_numbers()
    assert [sk.decrypt(x) for x in lst] == sk.decrypt_batch(acc[:3])


def test_streams_and_cuda_graph(pkg, cuda_engine, gmp):
    """Device-pointer entry points are asynchronous on the caller's stream and capturable in a CUDA graph
    (workspaces are sized by a warm-up call; nothing allocates or synchronises during capture)."""
    import torch
    kb, batch = 1024, 4096
    n, p, q = _key(kb)
    pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
    rng = np.random.default_rng(3)
    m = _rand_rows(rng, batch, pub.n_limbs, kb // 32 - 1)
    r = _rand_rows(rng, batch, pub.n_limbs, kb // 32 - 1)
    r[:, 0] |= 1
    d_m = torch.from_numpy(m.view(np.int32)).cuda()
    d_r = torch.from_numpy(r.view(np.int32)).cuda()
    d_c = torch.zeros((batch, pub.c_limbs), dtype=torch.int32, device="cuda")
    d_d = torch.zeros((batch, pub.n_limbs), dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        pub.encrypt_dev(d_m, d_r, d_c, batch, stream=side.cuda_stream)          # warm-up on the side stream
        priv.decrypt_dev(d_c, d_d, batch, stream=side.cuda_stream)
    side.synchronize()
    assert bool((d_d == d_m).all().item())
    ref_c = d_c.clone()
    d_c.zero_(); d_d.zero_()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        pub.encrypt_dev(d_m, d_r, d_c, batch, stream=side.cuda_stream)
        priv.decrypt_dev(d_c, d_d, batch, stream=side.cuda_stream)
    for _ in range(2):
        d_c.zero_(); d_d.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert bool((d_c == ref_c).all().item()) and bool((d_d == d_m).all().item())


def test_all_kernel_paths_agree(pkg, cuda_engine, monkeypatch):
    """The tensor-core reduction kernels (PAI_TC=2, pai_tc.cuh), the base-n digit kernels on the integer pipe (default),
    the full-width Montgomery kernels (PAI_*_PATH=full) and the warp-per-ciphertext kernels (small batches, pai_coop.cuh)
    must give identical bits."""
    n, p, q = _key(1024)
    rng = random.Random(21)
    m = [rng.randrange(n) for _ in range(300)] + [0, 1, n - 1]
    r = [rng.randrange(1, n) for _ in m]
    k = [rng.getrandbits(64) for _ in m[:150]] + [n - 1 - rng.getrandbits(40) for _ in m[150:]]
    results = []
    paths = []
    for env in ({"PAI_TC": "2", "PAI_COOP_MAX": "0"}, {"PAI_TC": "0", "PAI_COOP_MAX": "0"},
                {"PAI_ENCRYPT_PATH": "full", "PAI_DECRYPT_PATH": "full", "PAI_COOP_MAX": "0"}, {"PAI_COOP_MAX": "100000"}):
        for key in ("PAI_ENCRYPT_PATH", "PAI_DECRYPT_PATH", "PAI_COOP_MAX", "PAI_TC"):
            monkeypatch.delenv(key, raising=False)
        for key, val in env.items():
            monkeypatch.setenv(key, val)
        pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)       # the switches are read at context creation
        paths.append((pub.kernel_path(), priv.kernel_path()))
        c = pub.raw_encrypt(m, r)
        t, st = pub.raw_mul(c, k)
        results.append((c, priv.raw_decrypt(c), t, st, priv.raw_decrypt(t)))
        pub.close(); priv.close()
    assert paths[:3] == [("tc", "tc"), ("digit", "digit"), ("full", "full")]
    assert results[0] == results[1] == results[2] == results[3]
    assert results[0][1] == m


def test_device_obfuscators(pkg, cuda_engine):
    """pai_random_lt_n on the GPU: same stream as the simulation build for a seed (the keystream itself is pinned to
    an independent ChaCha20 in tests/test_rng_hostsim.py), 1 <= r < n, distinct rows, fresh per call by default."""
    import torch
    import __graft_entry__ as ge
    n, p, q = _key(2048)
    pub = pkg.PublicContext(n)
    batch = 50000
    d_r = torch.empty((batch, pub.n_limbs), dtype=torch.int32, device="cuda")
    seed = bytes(range(32))
    pub.random_lt_n_dev(d_r, batch, seed=seed, nonce=7)
    torch.cuda.synchronize()
    r = d_r.cpu().numpy().view(np.uint32)
    sim = pkg.Engine(ge.build_hostsim())
    spub = pkg.PublicContext(n, engine=sim)
    ref = np.zeros((64, spub.n_limbs), dtype=np.uint32)
    spub.random_lt_n_dev(ref, 64, seed=seed, nonce=7)
    assert (r[:64] == ref).all()
    vals = pkg.limbs_to_ints(r[:2000])
    assert all(1 <= v < n for v in vals)
    assert len(np.unique(r[:, :4].copy().view([("", np.uint32)] * 4))) == batch
    d_r2 = torch.empty_like(d_r)
    pub.random_lt_n_dev(d_r2, batch)
    assert not bool((d_r2 == d_r).all(dim=1).any().item())
    # and an encrypt/decrypt round trip with device-drawn r
    priv = pkg.PrivateContext(p, q)
    m = _rand_rows(np.random.default_rng(1), batch, pub.n_limbs, 63)
    d_m = torch.from_numpy(m.view(np.int32)).cuda()
    d_c = torch.empty((batch, pub.c_limbs), dtype=torch.int32, device="cuda")
    d_d = torch.empty_like(d_m)
    pub.encrypt_dev(d_m, d_r2, d_c, batch)
    priv.decrypt_dev(d_c, d_d, batch)
    assert bool((d_d == d_m).all().item())


def test_decimal_wire_format_on_gpu(pkg, cuda_engine):
    """pai_limbs_to_decimal / pai_decimal_to_limbs at ciphertext size: equal to Python's str()/int() on a sample,
    lossless round trip of the whole batch on the device, and the JSON scheme of docs/serialisation.rst."""
    import importlib
    import torch
    eng = importlib.import_module("python-paillier_b200.engine")
    n, p, q = _key(2048)
    pub = pkg.PublicContext(n)
    batch, lc = 20000, pub.c_limbs
    c = _rand_rows(np.random.default_rng(3), batch, lc, lc)
    c[0] = 0
    c[1] = 0xffffffff
    c[2, 1:] = 0
    d_c = torch.from_numpy(c.view(np.int32)).cuda()
    width = eng.decimal_width(lc)
    d_text = torch.empty((batch, width), dtype=torch.uint8, device="cuda")
    eng.limbs_to_decimal_dev(d_c, lc, d_text, batch)
    d_back = torch.empty_like(d_c)
    d_status = torch.ones((batch,), dtype=torch.int32, device="cuda")
    eng.decimal_to_limbs_dev(d_text, width, d_back, lc, d_status, batch)
    assert bool((d_back == d_c).all().item()) and not bool(d_status.any().item())
    text = d_text[:200].cpu().numpy()
    assert [bytes(r).decode() for r in text] == [str(v).rjust(width, "0") for v in pkg.limbs_to_ints(c[:200])]
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    v = pk.encrypt_batch([0.5 * i for i in range(-50, 50)])
    back = pkg.EncryptedVector.from_json(v.to_json())
    assert back.ciphertexts(False) == v.ciphertexts(False)
    assert sk.decrypt_batch(back) == [0.5 * i for i in range(-50, 50)]
