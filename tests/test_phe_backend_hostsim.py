"""integration/phe_b200_backend.py -- the ctypes binding of the reference's scalar seam (powmod / mulmod / invert) -- on
the test-only host simulation of the device code: the seam golden vectors the reference computed, the reference's
known answer (phe/tests/paillier_test.py:128-136) through the three functions, and install / uninstall rebinding the
names in stand-in ``phe.util`` / ``phe.paillier`` modules the way the reference's own tests flip backends."""
import importlib.util
import os
import sys
import types

import pytest

from oracle.golden import H, load_golden


@pytest.fixture(scope="module")
def backend():
    import __graft_entry__ as ge
    lib = ge.build_hostsim()
    spec = importlib.util.spec_from_file_location("phe_b200_backend_under_test",
                                                  os.path.join(ge.ROOT, "integration", "phe_b200_backend.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.load(lib)
    yield mod, lib


@pytest.mark.parametrize("kb", [256, 1024])
def test_seam_equals_the_reference_vectors(backend, kb):
    b, _ = backend
    seam = load_golden("vectors_%d.json" % kb)["seam"]
    for e in seam["powmod"]:
        assert b.powmod(H(e["a"]), H(e["b"]), H(e["c"])) == H(e["o"])
    for e in seam["mulmod"]:
        assert b.mulmod(H(e["a"]), H(e["b"]), H(e["c"])) == H(e["o"])
    for e in seam["invert"]:
        if "error" in e:
            with pytest.raises(ZeroDivisionError):
                b.invert(H(e["a"]), H(e["b"]))
        else:
            assert b.invert(H(e["a"]), H(e["b"])) == H(e["o"])
    with pytest.raises(ZeroDivisionError):
        b.invert(2, 4)


def test_reference_known_answer_through_the_seam(backend):
    b, _ = backend
    p, q = 293, 433
    n = p * q
    assert n == 126869
    nsq = n * n
    c = (1 + n * 10100) * b.powmod(74384, n, nsq) % nsq
    assert c == 935906717
    lam = (p - 1) * (q - 1)
    mu = b.invert((b.powmod(n + 1, lam, nsq) - 1) // n, n)
    assert (b.powmod(c, lam, nsq) - 1) // n * mu % n == 10100
    assert b.mulmod(c, c, nsq) == c * c % nsq


def test_install_and_uninstall_rebind_the_seam(backend, monkeypatch):
    b, lib = backend
    orig = {name: (lambda *a, _n=name: ("original", _n)) for name in ("powmod", "mulmod", "invert")}
    phe = types.ModuleType("phe")
    pu, pp = types.ModuleType("phe.util"), types.ModuleType("phe.paillier")
    for mod in (pu, pp):
        for name, fn in orig.items():
            setattr(mod, name, fn)
    phe.util, phe.paillier = pu, pp
    for name, mod in (("phe", phe), ("phe.util", pu), ("phe.paillier", pp)):
        monkeypatch.setitem(sys.modules, name, mod)
    b.install(phe, lib_path=lib)
    try:
        for mod in (pu, pp):
            assert mod.powmod is b.powmod and mod.mulmod is b.mulmod and mod.invert is b.invert
        assert pp.powmod(74384, 126869, 126869 ** 2) == pow(74384, 126869, 126869 ** 2)
    finally:
        b.uninstall(phe)
    for mod in (pu, pp):
        for name, fn in orig.items():
            assert getattr(mod, name) is fn
