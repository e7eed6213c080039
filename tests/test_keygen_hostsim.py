"""Batched key generation: pai_miller_rabin / util.is_prime_batch / getprimeover_batch /
generate_paillier_keypairs on the host simulation -- probable-prime agreement with the reference's is_prime
(phe/util.py:420-443) on primes, composites, Carmichael numbers and strong pseudoprimes to small bases."""
import importlib
import random

import pytest

from oracle.golden import H, load_golden


@pytest.fixture(scope="module")
def env(pkg):
    import __graft_entry__ as ge
    engine_mod = importlib.import_module("python-paillier_b200.engine")
    engine_mod._set_engine_for_tests(pkg.Engine(ge.build_hostsim()))
    yield importlib.import_module("python-paillier_b200.util"), engine_mod
    engine_mod._set_engine_for_tests(None)


def test_miller_rabin_batch_agrees_with_the_reference(pkg, env):
    util, engine_mod = env
    rng = random.Random(5)
    ref = load_golden("is_prime_reference.json")          # the reference's is_prime verdicts on these candidates
    primes = [2 ** 127 - 1, 2 ** 521 - 1, (1 << 255) - 19, 2 ** 89 - 1]
    carmichael = [561 * 1, 41041, 825265, 321197185, 5394826801, 232250619601, 9746347772161, 1436697831295441,
                  60977817398996785, 7156857700403137441, 1791562810662585767521, 87674969936234821377601]
    strong_pseudo = [3215031751, 3825123056546413051, 318665857834031151167461]      # strong pseudoprimes to bases 2, 3, 5, 7 (and more)
    semiprimes = [(2 ** 127 - 1) * ((1 << 255) - 19), (2 ** 89 - 1) * (2 ** 107 - 1)]
    randoms = [rng.getrandbits(256) | 1 | (1 << 255) for _ in range(24)] + [rng.getrandbits(700) | 1 | (1 << 699) for _ in range(6)]
    cands = [c for c in primes + carmichael + strong_pseudo + semiprimes + randoms if c > 20000]
    assert cands == [H(c) for c in ref["candidates"]]
    got = util.is_prime_batch(cands)
    assert got == ref["is_prime"]
    assert got[:4] == [True] * 4 and not any(got[4:4 + len([c for c in carmichael if c > 20000]) + len(strong_pseudo) + len(semiprimes)])
    # raw kernel on survivors only (no trial division): the pseudoprimes must still fall to random bases
    raw = engine_mod.miller_rabin_batch([3215031751, 2 ** 127 - 1, 3825123056546413051, 318665857834031151167461, 2 ** 61 - 1], rounds=25)
    assert raw == [False, True, False, False, True]


def test_batched_keygen(pkg, env):
    util, _ = env
    ps = util.getprimeover_batch(160, 5)
    assert len(ps) == 5 and len(set(ps)) == 5 and all(p.bit_length() == 160 and util.is_prime(p) for p in ps)
    keys = pkg.generate_paillier_keypairs(3, n_length=320)
    assert len({pk.n for pk, _ in keys}) == 3
    for pk, sk in keys:
        assert pk.n.bit_length() == 320 and sk.p * sk.q == pk.n
        assert sk.decrypt(pk.encrypt(-12.5) + 3) == -9.5
    pk, sk = pkg.generate_paillier_keypair(n_length=512)        # the scalar entry point keeps the reference's host-side loop
    assert pk.n.bit_length() == 512 and sk.decrypt(pk.encrypt(7)) == 7
