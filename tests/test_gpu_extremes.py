"""The GPU-only arithmetic at its carry extremes, bit for bit against the oracle (gmp backend).

The host simulation compiles the same templates, but wherever the GPU build uses PTX or warp intrinsics -- the carry
chains of pai_core.cuh, the limb assembly from wgmma column sums in pai_tc.cuh (tc_limbs8, tc_ld32), the warp-uniform
window counts of pai_cta.cuh (__reduce_max_sync) and the warp-per-ciphertext kernels of pai_coop.cuh -- the simulation
runs a plain C++ twin instead.  This module drives the real code with the inputs where such code goes wrong:

* moduli: one key per NTp class (not on a tile boundary; 1025- and 1530-bit keys, a 2049-bit key that is mostly
  padding), unbalanced prime pairs, and public moduli with extreme Montgomery constants: n = 1 mod 2^k (N' mostly 0xff),
  n = -1 mod 2^k (N' = 1 mod 2^k) and n just below a power of two (top limbs all ones);
* operands: 0, 1, n - 1, all-ones limbs, n^2 - 1, n^2 - n, the scalars 0, 1, n - 1, max_int, n - max_int, 2^64 - 1,
  and inputs solved so that the low half T_lo of the first Montgomery product is all ones above its forced zero bits
  (encrypt: r * RR.d0 mod R; raw_mul / dot / decrypt: c mod R * RR.d0 mod R).  Each solved input is checked here before
  it reaches the GPU.  At the 3072-bit n = 1 mod 2^1536 modulus a model of the tensor-core GEMM 1 also checks that the
  solved encrypt and raw_mul / dot inputs give a different quotient m when the limb assembly drops the high word of a
  column sum shifted left by 8, which is what tc_limbs8 did while it assumed every column sum < 2^24;
* placement: extreme rows share warps with ordinary rows, k = 0 sits beside k = n - 1, and extreme rows sit on either
  side of a wave boundary.

Kernel families (read when a context is created; kernel_path() is asserted so that no fallback hides one):
digit (default), tc (PAI_TC=2 where tc_supported covers the size), full (PAI_ENCRYPT_PATH / PAI_DECRYPT_PATH=full),
coop (PAI_COOP_MAX large: encrypt, decrypt and shared-exponent powmod on the warp-per-ciphertext kernels).

What runs (public NTp class from n, private class from the larger prime; "tc" means tc where the class has it):

=========================  ====  ====  ===========================  ==========================================
key / modulus              pub   priv  families                     operations
=========================  ====  ====  ===========================  ==========================================
ntp1-300u (40/260 bits)    1     2     digit tc full coop           encrypt decrypt raw_add raw_mul
ntp1-500                   1     1     digit tc* full coop          encrypt decrypt raw_add raw_mul
ntp2-1000                  2     2     digit tc full coop           encrypt decrypt raw_add raw_mul
ntp3-1025u (512/513)       3     3     digit tc* full coop          encrypt decrypt raw_add raw_mul
ntp3-1530                  3     3     digit tc* full coop          encrypt decrypt raw_add raw_mul, sum, dot
ntp4-2000                  4     4     digit tc full coop           encrypt decrypt raw_add raw_mul
ntp6-2049u (1024/1025)     6     6     digit tc full coop           encrypt decrypt raw_add raw_mul
ntp8-3100u (1100/2000)     8     8     digit tc* full coop          encrypt decrypt raw_add raw_mul
ntp3-n1 (= 1 mod 2^768)    3     -     digit tc full coop           encrypt raw_add raw_mul, wave, sum, dot
ntp3-top (2^1536 - small)  3     -     digit tc full coop           encrypt raw_add raw_mul
ntp6-n1 (= 1 mod 2^1536)   6     -     digit tc full coop           encrypt raw_add raw_mul, wave, Straus dot
ntp6-nm1 (= -1 mod 2^1536) 6     -     digit tc full coop           encrypt raw_add raw_mul
ntp6-top (2^3072 - small)  6     -     digit tc full coop           encrypt raw_add raw_mul
ntp8-n1 (= 1 mod 2^2048)   8     -     digit tc* full coop          encrypt raw_add raw_mul
ModContext, NT = 3         -     -     coop / not coop              powmod (shared, per element), mulmod, invert
=========================  ====  ====  ===========================  ==========================================
(tc*: one side's class has no tensor-core kernels -- decrypt at private class 1 or 3, encrypt at public class 8 --
and kernel_path() must say "digit" for that side.)
"""
import random

import numpy as np
import pytest

from oracle import paillier_oracle as orc

pytestmark = pytest.mark.gpu

NTP = (1, 2, 3, 4, 6, 8)                       # DISPATCH_NTP
SWITCHES = ("PAI_TC", "PAI_ENCRYPT_PATH", "PAI_DECRYPT_PATH", "PAI_COOP_MAX")
FAMILIES = {
    "digit": {"PAI_COOP_MAX": "0"},
    "tc": {"PAI_TC": "2", "PAI_COOP_MAX": "0"},
    "full": {"PAI_ENCRYPT_PATH": "full", "PAI_DECRYPT_PATH": "full", "PAI_COOP_MAX": "0"},
    "coop": {"PAI_COOP_MAX": "1000000"},
}
# name -> (bits of n, bits of the smaller prime) for real keys, or a constructor of a public modulus
REAL = {"ntp1-300u": (300, 40), "ntp1-500": (500, 250), "ntp2-1000": (1000, 500), "ntp3-1025u": (1025, 512),
        "ntp3-1530": (1530, 765), "ntp4-2000": (2000, 1000), "ntp6-2049u": (2049, 1024), "ntp8-3100u": (3100, 1100)}
CRAFTED = {"ntp3-n1": (1536, "one"), "ntp3-top": (1536, "top"), "ntp6-n1": (3072, "one"), "ntp6-nm1": (3072, "minus"),
           "ntp6-top": (3072, "top"), "ntp8-n1": (4096, "one")}


@pytest.fixture(scope="module")
def gmp():
    """The oracle on libgmp; where libgmp is missing, on its pure-Python backend (same results, slower)."""
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    yield
    orc.BACKEND = "python"


def _family(monkeypatch, family):
    for key in SWITCHES:
        monkeypatch.delenv(key, raising=False)
    for key, val in FAMILIES[family].items():
        monkeypatch.setenv(key, val)


def _pick(tiles):
    return next(t for t in NTP if t >= tiles)


def _pub_ntp(n):
    return _pick(((n.bit_length() + 31) // 32 + 15) // 16)


def _priv_ntp(p, q):
    return _pick(((max(p, q).bit_length() + 31) // 32 + 7) // 8)


def _expected_paths(family, n, pq):
    if family == "full":
        return "full", "full"
    if family != "tc":
        return "digit", "digit"
    pub = "tc" if 2 * _pub_ntp(n) in (2, 4, 6, 8, 12) else "digit"            # tc_supported(2 * ntp, 12)
    priv = "tc" if pq and _priv_ntp(*pq) in (2, 4, 6, 8) else "digit"          # tc_supported(ntp, 8)
    return pub, priv


def _ones(x):
    """The largest all-ones number below x."""
    return (1 << (x.bit_length() - 1)) - 1


def _solve_low(d0, R, below):
    """The least x with x * d0 mod R = R - 2^z (z: the trailing zero bits of d0, which every such product has), or None
    when that x is not below `below`."""
    z = (d0 & -d0).bit_length() - 1
    Rz = R >> z
    x = ((Rz - 1) * pow(d0 >> z, -1, Rz)) % Rz
    t_lo = x * d0 % R
    assert t_lo >> z == Rz - 1 and t_lo % (1 << z) == 0          # all ones above the forced zero bits
    return x if x < below else None


def _digit_radix(n):
    """R of the base-n digit kernels (and the tensor-core reductions): 2^(512 * NTp), and RR.d0 = R^2 mod n."""
    R = 1 << (512 * _pub_ntp(n))
    return R, R * R % n


def _gemm1_columns(t_lo, n, R):
    """Byte-column sums of the tensor-core GEMM 1, T_lo x Toeplitz(N') (N' = -n^-1 mod R), columns 0 .. D-1."""
    D = R.bit_length() // 8
    nprime = -pow(n, -1, R) % R
    a = np.frombuffer(t_lo.to_bytes(D, "little"), np.uint8).astype(np.int64)
    b = np.frombuffer(nprime.to_bytes(D, "little"), np.uint8).astype(np.int64)
    return np.convolve(a, b)[:D]


def _gemm1_quotients(t_lo, n, R):
    """m = T_lo * N' mod R assembled from the GEMM-1 column sums as tc_limbs8 does: exactly, and with the bits of v1 << 8
    above 2^32 dropped (what its PTX computed while it assumed every column sum < 2^24)."""
    cols = [int(x) for x in _gemm1_columns(t_lo, n, R)]
    exact = cut = 0
    for j in range(0, len(cols), 4):
        v0, v1, v2, v3 = cols[j:j + 4]
        exact += (v0 + (v1 << 8) + (v2 << 16) + (v3 << 24)) << (8 * j)
        cut += (v0 + ((v1 << 8) & 0xffffffff) + (v2 << 16) + (v3 << 24)) << (8 * j)
    return exact % R, cut % R


def _prime(rng, bits):
    import importlib
    util = importlib.import_module("python-paillier_b200.util")
    while True:
        c = rng.getrandbits(bits) | (1 << (bits - 1)) | 1
        if util.is_prime(c):
            return c


def _crafted(bits, kind, rng):
    """A public modulus of `bits` bits with an extreme Montgomery constant, whose solved encrypt obfuscator is below n."""
    half = bits // 2
    while True:
        t = rng.getrandbits(half - 2)
        if kind == "one":
            n = (1 << (bits - 1)) + (t << half) + 1
        elif kind == "minus":
            n = (1 << (bits - 1)) + ((t | 1) << half) - 1
        else:
            n = (1 << bits) - 2 * (t >> (half - 66)) - 1
        R, d0 = _digit_radix(n)
        if n.bit_length() == bits and _solve_low(d0, R, n) is not None:
            return n


_CASES = {}


def _case(name):
    """Key, operands and oracle results of one key (computed once, shared by the families)."""
    if name in _CASES:
        return _CASES[name]
    rng = random.Random(name)
    if name in REAL:
        bits, pbits = REAL[name]
        while True:
            p, q = _prime(rng, pbits), _prime(rng, bits - pbits)
            n = p * q
            if p != q and n.bit_length() == bits:
                break
        pq = (p, q)
    else:
        n, pq = _crafted(*CRAFTED[name], rng), None
    nsq = n * n
    opub = orc.PublicConsts(n)
    R, d0 = _digit_radix(n)
    r_solved = _solve_low(d0, R, n)
    c0 = _solve_low(d0, R, R)
    c_solved = c0 + R * ((nsq - 1 - c0) // R)                   # low half solved, high half as large as c < n^2 allows
    assert c_solved < nsq and c_solved % R == c0
    if name == "ntp6-n1":             # D = 384: the entry products of encrypt and of raw_mul / dot overflow a v1 column
        for t_lo in (r_solved * d0 % R, c0 * d0 % R):
            exact, cut = _gemm1_quotients(t_lo, n, R)
            assert exact == t_lo * (-pow(n, -1, R) % R) % R and cut != exact
    if name in CRAFTED:
        assert r_solved is not None
    # encrypt: every extreme (m, r) pair on the even rows, ordinary rows between them (one warp holds both)
    ms_x = [0, 1, n - 1, _ones(n), n - opub.max_int, opub.max_int]
    rs_x = [1, n - 1, _ones(n)] + ([r_solved] if r_solved else [])
    ext = [(m, r) for r in rs_x for m in ms_x]
    ms, rs = [], []
    for m, r in ext:
        ms += [m, rng.randrange(n)]
        rs += [r, rng.randrange(1, n)]
    cs = [orc.raw_encrypt(opub, m, r) for m, r in zip(ms, rs)]
    # raw_mul: extreme ciphertexts x extreme scalars, k = 0 next to k = n - 1, ordinary rows between the groups
    cs_x = [1, nsq - 1, nsq - n, _ones(nsq), c_solved]
    ks_x = [0, n - 1, 1, opub.max_int, n - opub.max_int, (1 << 64) - 1]
    ma, mk = [], []
    for c in cs_x:
        ma += [c] * len(ks_x) + [cs[rng.randrange(len(cs))]]
        mk += ks_x + [rng.getrandbits(64)]
    mul = []
    for c, k in zip(ma, mk):
        try:
            mul.append((orc.raw_mul(opub, c, k), 0))
        except ZeroDivisionError:
            mul.append((None, 1))                              # negative branch on a base with no inverse
    adds_a = cs_x + cs[:32]
    adds_b = adds_a[::-1]
    case = dict(n=n, pq=pq, ms=ms, rs=rs, cs=cs, ma=ma, mk=mk, mul=mul, adds=(adds_a, adds_b),
                add=[orc.raw_add(opub, a, b) for a, b in zip(adds_a, adds_b)], c_solved=c_solved, r_solved=r_solved)
    if pq:
        p, q = min(pq), max(pq)
        opriv = orc.PrivateConsts(opub, p, q)
        Rp = 1 << (256 * _priv_ntp(p, q))                       # radix of the smaller prime's side, which runs first
        cp0 = _solve_low(Rp * Rp % p, Rp, Rp)
        cp = cp0 + Rp * ((nsq - 1 - cp0) // Rp)
        assert cp < nsq
        xs = []
        for i, c in enumerate(cs):
            xs.append(c)
            if i % 4 == 0:
                xs.append([0, 1, n, nsq - 1, nsq - n, p, q, p * p, q * q, cp, c_solved, _ones(nsq), nsq - p][i // 4 % 13])
        case.update(xs=xs, dec=[orc.raw_decrypt(opriv, x) for x in xs])
    _CASES[name] = case
    return case


KEYS = list(REAL) + list(CRAFTED)


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("name", KEYS)
def test_key_ops_at_extremes(pkg, cuda_engine, gmp, monkeypatch, name, family):
    """encrypt, raw_add, raw_mul (with its status) and, for real keys, decrypt of the extreme operands."""
    cs = _case(name)
    n, pq = cs["n"], cs["pq"]
    _family(monkeypatch, family)
    pub = pkg.PublicContext(n)
    priv = pkg.PrivateContext(*pq) if pq else None
    want_pub, want_priv = _expected_paths(family, n, pq)
    assert pub.kernel_path() == want_pub
    if priv:
        assert priv.kernel_path() == want_priv
    assert pub.raw_encrypt(cs["ms"], cs["rs"]) == cs["cs"]
    assert pub.raw_add(*cs["adds"]) == cs["add"]
    out, st = pub.raw_mul(cs["ma"], cs["mk"])
    for i, (o, s, (want, wst)) in enumerate(zip(out, st, cs["mul"])):
        assert s == wst, i
        if not wst:
            assert o == want, i
    if priv:
        assert priv.raw_decrypt(cs["xs"]) == cs["dec"]
        priv.close()
    pub.close()


def _dev(pkg, ints, limbs):
    import torch
    return torch.from_numpy(pkg.ints_to_limbs(ints, limbs).view(np.int32).copy()).cuda()


def _ints(pkg, t):
    return pkg.limbs_to_ints(t.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("name,family", [("ntp3-n1", "tc"), ("ntp3-n1", "digit"), ("ntp6-n1", "tc"),
                                         ("ntp6-n1", "digit"), ("ntp3-1530", "tc")])
def test_extreme_rows_on_a_wave_boundary(pkg, cuda_engine, gmp, monkeypatch, name, family):
    """One wave plus a tail of the throughput encrypt, raw_mul and decrypt kernels, with the solved extreme rows and
    k = 0 / k = n - 1 at the first rows, either side of the wave boundary and at the last row."""
    import torch
    cs = _case(name)
    n, pq = cs["n"], cs["pq"]
    _family(monkeypatch, family)
    pub = pkg.PublicContext(n)
    assert pub.kernel_path() == _expected_paths(family, n, pq)[0]
    rows = pub.wave() + 40
    w = pub.wave()
    idx = [0, 1, w - 2, w - 1, w, w + 1, rows - 1]
    m = torch.empty((rows, pub.n_limbs), dtype=torch.int32, device="cuda")
    r = torch.empty_like(m)
    pub.random_lt_n_dev(m, rows, seed=bytes([7]) * 32, nonce=0)
    pub.random_lt_n_dev(r, rows, seed=bytes([7]) * 32, nonce=1)
    ti = torch.tensor(idx, device="cuda")
    ms_x = [0, n - 1, _ones(n), 1, n - 1, 0, _ones(n)]
    rs_x = [cs["r_solved"] or 1, _ones(n), cs["r_solved"] or n - 1, n - 1, cs["r_solved"] or 1, 1, cs["r_solved"] or 1]
    m[ti] = _dev(pkg, ms_x, pub.n_limbs)
    r[ti] = _dev(pkg, rs_x, pub.n_limbs)
    c = torch.empty((rows, pub.c_limbs), dtype=torch.int32, device="cuda")
    pub.encrypt_dev(m, r, c, rows)
    k = torch.zeros_like(m)
    k[:, :2] = r[:, :2]                                                 # 64-bit scalars
    ks_x = [0, n - 1, (1 << 64) - 1, orc.PublicConsts(n).max_int, n - 1, 1, (1 << 64) - 1]
    k[ti] = _dev(pkg, ks_x, pub.n_limbs)
    # the solved base on rows w - 2, w - 1, w + 1 and the last, each with a positive scalar, so that it enters the power
    solved = [2, 3, 5, 6]
    assert all(0 < ks_x[i] < n - orc.PublicConsts(n).max_int for i in solved)
    base = c.clone()
    base[ti[solved]] = _dev(pkg, [cs["c_solved"]] * len(solved), pub.c_limbs)
    e = torch.empty_like(c)
    status = torch.ones((rows,), dtype=torch.int32, device="cuda")
    pub.raw_mul_dev(base, k, e, status, rows)
    torch.cuda.synchronize()
    sample = sorted(set(idx) | set(random.Random(name).sample(range(rows), 8)))
    si = torch.tensor(sample, device="cuda")
    opub = orc.PublicConsts(n)
    mi, ri, ci, bi, ki, ei = (_ints(pkg, t[si]) for t in (m, r, c, base, k, e))
    assert ci == [orc.raw_encrypt(opub, a, b) for a, b in zip(mi, ri)]
    # the crafted moduli have small factors, so a negative scalar may meet a base without an inverse: status 1
    for i, a, b, o, s in zip(sample, bi, ki, ei, status[si].tolist()):
        try:
            want = orc.raw_mul(opub, a, b)
        except ZeroDivisionError:
            assert s == 1, i
            continue
        assert s == 0 and o == want, i
    if pq:
        priv = pkg.PrivateContext(*pq)
        assert priv.kernel_path() == _expected_paths(family, n, pq)[1]
        d = torch.empty_like(m)
        priv.decrypt_dev(c, d, rows)
        torch.cuda.synchronize()
        assert bool((d == m).all().item())
        priv.close()
    pub.close()


@pytest.mark.parametrize("name,family,big", [("ntp3-1530", "digit", False), ("ntp3-1530", "tc", False),
                                             ("ntp3-n1", "digit", False), ("ntp3-n1", "tc", False),
                                             ("ntp6-n1", "tc", False), ("ntp6-n1", "tc", True)])
def test_sum_and_dot_at_extremes(pkg, cuda_engine, gmp, monkeypatch, name, family, big):
    """EncryptedVector.sum and .dot over extreme ciphertexts and scalars (tc: the Straus kernels, one element per group,
    and with `big` more elements than a wave: several per group)."""
    import torch
    cs = _case(name)
    n = cs["n"]
    nsq = n * n
    _family(monkeypatch, family)
    pk = pkg.PaillierPublicKey(n)
    ctx = pk.engine_context()
    assert ctx.kernel_path() == _expected_paths(family, n, None)[0]
    opub = orc.PublicConsts(n)
    c_sol = cs["c_solved"]
    ks_x = [0, n - 1, 1, opub.max_int, n - opub.max_int, (1 << 64) - 1]
    positive = [k for k in ks_x if 0 < k < n - opub.max_int]
    # extreme (ciphertext, scalar) pairs: a negative scalar only where the ciphertext has an inverse (the crafted moduli
    # have small factors); the solved ciphertext with every positive scalar, so that it enters the Straus tables as it is
    pairs = [(c_sol, k) for k in positive]
    pairs += [(c, k) for c in (1, nsq - 1, _ones(nsq)) for k in ks_x
              if k < n - opub.max_int or orc.extended_euclidean_algorithm(c, n)[0] == 1]
    rng = random.Random(name + family)
    count = ctx.wave() + 50 if big else 48
    if big:
        m = torch.empty((count, ctx.n_limbs), dtype=torch.int32, device="cuda")
        r = torch.empty_like(m)
        ctx.random_lt_n_dev(m, count, seed=bytes([5]) * 32, nonce=0)
        ctx.random_lt_n_dev(r, count, seed=bytes([5]) * 32, nonce=1)
        c = torch.empty((count, ctx.c_limbs), dtype=torch.int32, device="cuda")
        ctx.encrypt_dev(m, r, c, count)
        cts = _ints(pkg, c)
    else:
        cts = [cs["cs"][i % len(cs["cs"])] for i in range(count)]
    ks = [rng.getrandbits(40) for _ in range(count)]
    for pos, (x, k) in enumerate(pairs):                                # k = 0 beside k = n - 1; ordinary rows after
        cts[pos], ks[pos] = x, k
    cts[count - 2], ks[count - 2] = c_sol, positive[-1]
    cts[count - 1], ks[count - 1] = c_sol, positive[0]
    assert len(pairs) < 32 and sum(x == c_sol and k in positive for x, k in zip(cts, ks)) == len(positive) + 2
    v = pkg.EncryptedVector(pk, _dev(pkg, cts, ctx.c_limbs), np.zeros(count, dtype=np.int64))
    want_sum = 1
    for x in cts:
        want_sum = want_sum * x % nsq
    assert v.sum().ciphertext(False) == want_sum
    want_dot = 1
    for x, k in zip(cts, ks):
        want_dot = want_dot * orc.raw_mul(opub, x, k) % nsq
    d = v.dot([pkg.EncodedNumber(pk, k, 0) for k in ks])
    assert d.ciphertext(False) == want_dot


MODULI = {"nt3-m1": lambda rng: (1 << 700) + (rng.getrandbits(340) << 350) + 1,
          "nt3-mm1": lambda rng: (1 << 767) + ((rng.getrandbits(380) | 1) << 384) - 1,
          "nt3-top": lambda rng: (1 << 768) - 2 * rng.getrandbits(64) - 1,
          "nt3-rand": lambda rng: rng.getrandbits(600) | (1 << 599) | 1}


@pytest.mark.parametrize("coop_max", ["0", "1000000"])
@pytest.mark.parametrize("name", list(MODULI))
def test_mod_context_nt3_at_extremes(pkg, cuda_engine, gmp, monkeypatch, name, coop_max):
    """ModContext at 513 to 768 bits (NT = 3): powmod with a shared exponent (the warp-per-ciphertext kernels when
    coop_max is large) and with per-element exponents, mulmod and invert."""
    rng = random.Random(name)
    M = MODULI[name](rng)
    _family(monkeypatch, "coop" if coop_max != "0" else "digit")
    ctx = pkg.ModContext(M)
    assert ctx.limbs == 24
    R = 1 << 768
    b_solved = _solve_low(R * R % M, R, M)
    bases = [0, 1, M - 1, _ones(M)] + ([b_solved] if b_solved else []) + [rng.randrange(M) for _ in range(11)]
    exps = [0, 1, M - 1, (1 << 64) - 1, _ones(M), rng.randrange(M)]
    for e in exps:
        assert ctx.powmod(bases, e) == [pow(b, e, M) for b in bases]
    wide = bases + [M * M - 1, (1 << 1536) - 1]
    assert ctx.powmod(wide, M - 2) == [pow(b, M - 2, M) for b in wide]
    per = [exps[i % len(exps)] for i in range(len(bases))]
    assert ctx.powmod(bases, per) == [pow(b, e, M) for b, e in zip(bases, per)]
    a, b = bases, bases[::-1]
    assert ctx.mulmod(a, b) == [x * y % M for x, y in zip(a, b)]
    inv, st = ctx.invert(bases)
    for x, y, s in zip(bases, inv, st):
        g = orc.extended_euclidean_algorithm(x, M)[0]
        assert s == (0 if g == 1 else 1), x
        if g == 1:
            assert y == orc.invert(x, M)
    ctx.close()
