"""The tensor-core kernel family (pai_tc.cuh) on the test-only host simulation, where a thread group is walked phase by
phase and the wgmma GEMM is an integer loop over the very same operand / band layouts: encrypt, CRT decrypt and
raw_mul must equal the oracle and the integer-pipe digit kernels (PAI_TC=0) bit for bit, for every key size the family
covers, including degenerate ciphertexts and batches that are not a multiple of the group."""
import random

import pytest

from oracle import paillier_oracle as orc
from oracle.golden import H, load_golden


@pytest.fixture(scope="module")
def sim(pkg):
    import __graft_entry__ as ge
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    yield pkg.Engine(ge.build_hostsim())
    orc.BACKEND = "python"


def _ctx(pkg, sim, monkeypatch, n, p, q, tc):
    monkeypatch.setenv("PAI_COOP_MAX", "0")
    monkeypatch.setenv("PAI_TC", "2" if tc else "0")          # 2: the tensor-core kernels wherever they exist
    return pkg.PublicContext(n, engine=sim), pkg.PrivateContext(p, q, engine=sim)


@pytest.mark.parametrize("kb,rows", [(1024, 11), (2048, 5), (3072, 3)])
def test_tc_family_equals_oracle_and_digit_family(pkg, sim, monkeypatch, kb, rows):
    fx = load_golden("vectors_%d.json" % kb)
    n, p, q = H(fx["n"]), H(fx["p"]), H(fx["q"])
    opub = orc.PublicConsts(n)
    opriv = orc.PrivateConsts(opub, p, q)
    rng = random.Random(kb)
    ms = [0, n - 1] + [rng.randrange(n) for _ in range(rows - 2)]
    rs = [1, n - 1] + [rng.randrange(1, n) for _ in range(rows - 2)]
    ks = [0, 1, opub.max_int, n - 1, n - opub.max_int][:rows] + [rng.getrandbits(64) for _ in range(max(0, rows - 5))]
    pub, priv = _ctx(pkg, sim, monkeypatch, n, p, q, True)
    assert pub.kernel_path() == "tc" and priv.kernel_path() == "tc"
    cs = pub.raw_encrypt(ms, rs)
    assert cs == [orc.raw_encrypt(opub, m, r) for m, r in zip(ms, rs)]
    xs = cs + [0, 1, n, n * n - 1, p, q, p * p, q * q]
    ds = priv.raw_decrypt(xs)
    assert ds == [orc.raw_decrypt(opriv, c) for c in xs]
    ts, st = pub.raw_mul(cs, ks[:len(cs)])
    assert st == [0] * len(cs) and ts == [orc.raw_mul(opub, c, k) for c, k in zip(cs, ks)]
    if kb <= 2048:
        pub0, priv0 = _ctx(pkg, sim, monkeypatch, n, p, q, False)
        assert pub0.kernel_path() == "digit" and priv0.kernel_path() == "digit"
        assert pub0.raw_encrypt(ms, rs) == cs and priv0.raw_decrypt(xs) == ds and pub0.raw_mul(cs, ks[:len(cs)])[0] == ts


def test_tc_family_key_size_coverage(pkg, sim, monkeypatch):
    """Which keys the tensor-core kernels cover under PAI_TC=2: encrypt for 1024 .. 3072-bit keys, decrypt for 1024 .. 4096-bit
    keys (same bits as the integer-pipe digit kernels, tests/test_edge_keys_hostsim.py).  By default every key, 256 to
    4096 bits, takes the integer-pipe digit kernels."""
    for kb, enc, dec in ((256, "digit", "digit"), (512, "digit", "digit"), (1024, "tc", "tc"), (2048, "tc", "tc"), (3072, "tc", "tc"),
                         (4096, "digit", "tc")):
        fx = load_golden("vectors_%d.json" % kb)
        for forced in (True, False):
            if forced:
                monkeypatch.setenv("PAI_TC", "2")
            else:
                monkeypatch.delenv("PAI_TC", raising=False)
            pub = pkg.PublicContext(H(fx["n"]), engine=sim)
            priv = pkg.PrivateContext(H(fx["p"]), H(fx["q"]), engine=sim)
            if forced and kb >= 1024:
                assert (pub.kernel_path(), priv.kernel_path()) == (enc, dec), kb
            elif not forced:
                assert (pub.kernel_path(), priv.kernel_path()) == ("digit", "digit"), kb
            pub.close(); priv.close()
