"""The engine's host layer on the test-only host simulation: which kernel family each context selects under the three
settings (default, PAI_TC=2, PAI_ENCRYPT_PATH=PAI_DECRYPT_PATH=full), the wave it reports, how many kernels every
entry point launches, and the argument checks of the host-pointer entry points.  The launch counts and waves are pinned
as literals, so a change to how the host code reaches the kernels that launches more, fewer or other kernels shows
here; the outputs of the three families must be bit-equal and correct."""
import contextlib
import hashlib
import os
import random

import numpy as np
import pytest

from oracle.golden import H, load_golden

KEYS = ("vectors_256.json", "vectors_1024.json")
SETTINGS = {
    "default": {},
    "tc": {"PAI_TC": "2"},
    "full": {"PAI_ENCRYPT_PATH": "full", "PAI_DECRYPT_PATH": "full"},
}
ENV_VARS = ("PAI_TC", "PAI_ENCRYPT_PATH", "PAI_DECRYPT_PATH", "PAI_COOP_MAX", "PAI_TC_STAGGER")
B = 3                      # rows per call: below one wave of every kernel, so the coop limit alone decides the routing
BW = 13                    # more than two waves of every kernel, and not a multiple of one
PAI_E_ARG = -1

# kernel family of the public / private context and the rows per wave they report
PATHS = {
    ("vectors_256.json", "default"): (("digit", "digit"), (4, 4)),
    ("vectors_256.json", "tc"): (("tc", "digit"), (6, 4)),                # the tensor-core family covers encrypt only here
    ("vectors_256.json", "full"): (("full", "full"), (4, 4)),
    ("vectors_1024.json", "default"): (("digit", "digit"), (4, 4)),
    ("vectors_1024.json", "tc"): (("tc", "tc"), (6, 6)),
    ("vectors_1024.json", "full"): (("full", "full"), (4, 4)),
}
# kernel launches per call, the same for every key and setting ...
LAUNCHES = {
    "encrypt": 1, "decrypt": 1, "raw_add": 1, "raw_mul": 3, "raw_mul_neg": 3, "raw_sum": 3, "raw_dot": 5, "raw_matvec": 4,
    "mod_mulmod": 1, "mod_powmod": 1, "mod_powmod_shared": 1, "mod_invert": 1,
    "encrypt_host": 1, "raw_add_host": 1, "raw_mul_host": 3, "decrypt_host": 1,
    "mod_mulmod_host": 1, "mod_powmod_host": 1, "mod_powmod_host_shared": 1, "mod_invert_host": 1,
    "encrypt_waves": 1, "decrypt_waves": 1, "encrypt_coop": 3, "decrypt_coop": 6,
}
# ... except where the tensor-core kernels run whole waves and then the tail with a geometry of its own
LAUNCHES_TC = {
    "vectors_256.json": {"encrypt_waves": 2},
    "vectors_1024.json": {"encrypt_waves": 2, "decrypt_waves": 2},
}
# sha256 over every output of one setting: the same for all three settings
DIGESTS = {
    "vectors_256.json": "620825e227fc8133f9ff00669a51df07561091dc744948400c2064ab5667b719",
    "vectors_1024.json": "af127c3296692a758719ed753593dc798ca2aade12e7d484b8107c238038b056",
}


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


@pytest.fixture(scope="module")
def sim(pkg):
    import __graft_entry__ as ge
    return pkg.Engine(ge.build_hostsim())


@pytest.fixture(scope="module")
def runs(pkg, sim):
    cache = {}

    def get(key, setting):
        if (key, setting) not in cache:
            cache[key, setting] = _run(pkg, sim, load_golden(key), SETTINGS[setting])
        return cache[key, setting]
    return get


def _run(pkg, sim, fx, settings):
    """Every entry point once on fixed inputs: (paths and waves, launches per call, digest of the outputs in call order)."""
    from importlib import import_module
    E = import_module("python-paillier_b200.engine")
    lib, P = sim.lib, E._ptr
    n, p, q = H(fx["n"]), H(fx["p"]), H(fx["q"])
    n2 = n * n
    rng = random.Random(11)
    launches, outputs = {}, []

    def call(name, fn, *outs):
        before = sim.launch_count()
        sim.check(fn())
        launches[name] = sim.launch_count() - before
        outputs.extend(np.array(o).copy() for o in outs)

    with _env(PAI_COOP_MAX="0", **settings):
        pub = pkg.PublicContext(n, engine=sim)
        priv = pkg.PrivateContext(p, q, engine=sim)
        mod = pkg.ModContext(n, engine=sim)
        paths = ((pub.kernel_path(), priv.kernel_path()), (pub.wave(), priv.wave()))
        ln, lc, lm = pub.n_limbs, pub.c_limbs, mod.limbs
        ms = [0, n - 1, rng.randrange(n)]
        rs = [1, n - 1, rng.randrange(1, n)]
        m, r = E.ints_to_limbs(ms, ln), E.ints_to_limbs(rs, ln)
        c = np.zeros((B, lc), np.uint32)
        call("encrypt", lambda: lib.pai_encrypt(pub.h, P(m), P(r), P(c), B, None), c)
        cs = E.limbs_to_ints(c)
        assert cs == [(1 + n * mi) * pow(ri, n, n2) % n2 for mi, ri in zip(ms, rs)]
        d = np.zeros((B, ln), np.uint32)
        call("decrypt", lambda: lib.pai_decrypt(priv.h, P(c), P(d), B, None), d)
        assert E.limbs_to_ints(d) == ms
        c2 = np.ascontiguousarray(c[::-1])
        out = np.zeros((B, lc), np.uint32)
        call("raw_add", lambda: lib.pai_raw_add(pub.h, P(c), P(c2), P(out), B, None), out)
        assert E.limbs_to_ints(out) == [a * b % n2 for a, b in zip(cs, cs[::-1])]
        max_int = n // 3 - 1
        for name, ks in (("raw_mul", [0, 5, rng.getrandbits(64)]), ("raw_mul_neg", [n - 1, 7, n - max_int])):
            s, st = E.ints_to_limbs(ks, ln), np.full(B, -9, np.int32)
            call(name, lambda: lib.pai_raw_mul(pub.h, P(c), P(s), P(out), P(st), B, None), out, st)
            want = [pow(a, k, n2) if k < n - max_int else pow(a, k - n, n2) for a, k in zip(cs, ks)]   # negative: c^-1 ^ (n - k)
            assert E.limbs_to_ints(out) == want and st.tolist() == [0] * B
        one = np.zeros((1, lc), np.uint32)
        call("raw_sum", lambda: lib.pai_raw_sum(pub.h, P(c), B, P(one), None), one)
        s, st = E.ints_to_limbs([n - 2, 3, rng.getrandbits(64)], ln), np.full(B, -9, np.int32)
        call("raw_dot", lambda: lib.pai_raw_dot(pub.h, P(c), P(s), P(one), P(st), B, None), one, st)
        indptr, indices = np.array([0, 2, 3], np.int64), np.array([0, 2, 1], np.int32)
        mag, neg = np.array([[3], [1000], [77]], np.uint32), np.array([0, 1, 0], np.uint8)
        rows, st = np.zeros((2, lc), np.uint32), np.full(B, -9, np.int32)
        call("raw_matvec", lambda: lib.pai_raw_matvec(pub.h, P(c), B, P(indptr), P(indices), P(mag), 1, 0, P(neg), 3, 2, P(rows),
                                                      P(st), None), rows, st)
        a, b = E.ints_to_limbs([rng.randrange(1, n) for _ in range(B)], lm), E.ints_to_limbs([rng.randrange(n) for _ in range(B)], lm)
        e = E.ints_to_limbs([rng.getrandbits(100) for _ in range(B)], 4)
        e1 = E.ints_to_limbs([rng.getrandbits(70)], 4)
        mo, mst = np.zeros((B, lm), np.uint32), np.full(B, -9, np.int32)
        call("mod_mulmod", lambda: lib.pai_mod_mulmod(mod.h, P(a), P(b), P(mo), B, None), mo)
        call("mod_powmod", lambda: lib.pai_mod_powmod(mod.h, P(a), lm, P(e), 4, P(mo), B, None), mo)
        call("mod_powmod_shared", lambda: lib.pai_mod_powmod_shared(mod.h, P(a), lm, P(e1), 4, P(mo), B, None), mo)
        call("mod_invert", lambda: lib.pai_mod_invert(mod.h, P(a), lm, P(mo), P(mst), B, None), mo, mst)
        hc = np.zeros((B, lc), np.uint32)
        call("encrypt_host", lambda: lib.pai_encrypt_host(pub.h, P(m), P(r), P(hc), B), hc)
        assert np.array_equal(hc, c)
        call("raw_add_host", lambda: lib.pai_raw_add_host(pub.h, P(c), P(c2), P(out), B), out)
        s, st = E.ints_to_limbs([n - 1, 7, 9], ln), np.full(B, -9, np.int32)
        call("raw_mul_host", lambda: lib.pai_raw_mul_host(pub.h, P(c), P(s), P(out), P(st), B), out, st)
        call("decrypt_host", lambda: lib.pai_decrypt_host(priv.h, P(c), P(d), B), d)
        assert E.limbs_to_ints(d) == ms
        call("mod_mulmod_host", lambda: lib.pai_mod_mulmod_host(mod.h, P(a), P(b), P(mo), B), mo)
        call("mod_powmod_host", lambda: lib.pai_mod_powmod_host(mod.h, P(a), lm, P(e), 4, 0, P(mo), B), mo)
        call("mod_powmod_host_shared", lambda: lib.pai_mod_powmod_host(mod.h, P(a), lm, P(e1), 4, 1, P(mo), B), mo)
        call("mod_invert_host", lambda: lib.pai_mod_invert_host(mod.h, P(a), lm, P(mo), P(mst), B), mo, mst)
        mw, rw = E.ints_to_limbs([rng.randrange(n) for _ in range(BW)], ln), E.ints_to_limbs([rng.randrange(1, n) for _ in range(BW)], ln)
        cw, dw = np.zeros((BW, lc), np.uint32), np.zeros((BW, ln), np.uint32)
        call("encrypt_waves", lambda: lib.pai_encrypt(pub.h, P(mw), P(rw), P(cw), BW, None), cw)
        call("decrypt_waves", lambda: lib.pai_decrypt(priv.h, P(cw), P(dw), BW, None), dw)
        assert np.array_equal(dw, mw)
        with _env(PAI_COOP_MAX="100000", **settings):      # the warp-per-ciphertext kernels take the whole batch
            cc, dd = np.zeros((B, lc), np.uint32), np.zeros((B, ln), np.uint32)
            call("encrypt_coop", lambda: lib.pai_encrypt(pub.h, P(m), P(r), P(cc), B, None), cc)
            call("decrypt_coop", lambda: lib.pai_decrypt(priv.h, P(c), P(dd), B, None), dd)
            assert np.array_equal(cc, c) and E.limbs_to_ints(dd) == ms
        pub.close(); priv.close(); mod.close()
    return paths, launches, hashlib.sha256(b"".join(o.tobytes() for o in outputs)).hexdigest()


@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("key", KEYS)
def test_paths_waves_and_launch_counts(runs, key, setting):
    paths, launches, _ = runs(key, setting)
    assert paths == PATHS[key, setting]
    assert launches == dict(LAUNCHES, **(LAUNCHES_TC[key] if setting == "tc" else {}))


@pytest.mark.parametrize("key", KEYS)
def test_outputs_bit_equal_across_families(runs, key):
    digests = {s: runs(key, s)[2] for s in SETTINGS}
    assert set(digests.values()) == {DIGESTS[key]}, digests


@pytest.mark.parametrize("key", KEYS)
def test_host_entry_points_check_arguments(pkg, sim, key):
    """A null pointer or a negative batch is PAI_E_ARG; batch 0 returns 0 and launches nothing."""
    fx = load_golden(key)
    n = H(fx["n"])
    with _env(PAI_COOP_MAX="0"):
        pub = pkg.PublicContext(n, engine=sim)
        priv = pkg.PrivateContext(H(fx["p"]), H(fx["q"]), engine=sim)
        mod = pkg.ModContext(n, engine=sim)
        lib = sim.lib
        from importlib import import_module
        P = import_module("python-paillier_b200.engine")._ptr
        x = np.zeros((1, 4 * pub.c_limbs), np.uint32)
        st = np.zeros(4, np.int32)
        lm = mod.limbs
        entries = {          # name -> (call(handle, pointers, batch), handle, number of pointers)
            "encrypt_host": (lambda h, ps, b: lib.pai_encrypt_host(h, ps[0], ps[1], ps[2], b), pub.h, 3),
            "raw_add_host": (lambda h, ps, b: lib.pai_raw_add_host(h, ps[0], ps[1], ps[2], b), pub.h, 3),
            "raw_mul_host": (lambda h, ps, b: lib.pai_raw_mul_host(h, ps[0], ps[1], ps[2], P(st), b), pub.h, 3),
            "decrypt_host": (lambda h, ps, b: lib.pai_decrypt_host(h, ps[0], ps[1], b), priv.h, 2),
            "mod_mulmod_host": (lambda h, ps, b: lib.pai_mod_mulmod_host(h, ps[0], ps[1], ps[2], b), mod.h, 3),
            "mod_powmod_host": (lambda h, ps, b: lib.pai_mod_powmod_host(h, ps[0], lm, ps[1], 1, 0, ps[2], b), mod.h, 3),
            "mod_powmod_host_shared": (lambda h, ps, b: lib.pai_mod_powmod_host(h, ps[0], lm, ps[1], 1, 1, ps[2], b), mod.h, 3),
            "mod_invert_host": (lambda h, ps, b: lib.pai_mod_invert_host(h, ps[0], lm, ps[1], P(st), b), mod.h, 2),
        }
        for name, (fn, h, npt) in entries.items():
            ok = [P(x)] * npt
            assert fn(None, ok, 1) == PAI_E_ARG, name
            for i in range(npt):
                assert fn(h, ok[:i] + [None] + ok[i + 1:], 1) == PAI_E_ARG, (name, i)
            assert fn(h, ok, -1) == PAI_E_ARG, name
            before = sim.launch_count()
            assert fn(h, ok, 0) == 0, name
            assert sim.launch_count() == before, name
        pub.close(); priv.close(); mod.close()
