"""Packed fixed-point vectors on the H100: encrypt_packed from CUDA float tensors over several waves of ciphertext rows at
2048, 3072 and 4096 bits, sampled rows against the GMP oracle's raw_encrypt of the model plaintext, the private-key path
bit-identical to the public one, a five-client sum that decrypts to the exact integer sum on the device, and a call
inside torch.cuda.stream(s)."""
import random

import numpy as np
import pytest

from oracle import paillier_oracle as orc
from oracle.golden import H, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gmp():
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    yield
    orc.BACKEND = "python"


def _keys(pkg, kb):
    fx = load_golden("vectors_%d.json" % kb)
    pk = pkg.PaillierPublicKey(H(fx["n"]))
    return pk, pkg.PaillierPrivateKey(pk, H(fx["p"]), H(fx["q"]))


def _model_rows(n, b, K, q, rows):
    """P mod n of the given rows from the quantised slots q (int64 numpy)"""
    return [sum(int(s) << (b * j) for j, s in enumerate(q[r * K:(r + 1) * K])) % n for r in rows]


@pytest.mark.parametrize("kb", [2048, 3072, 4096])
def test_waves_of_rows_equal_the_oracle_and_the_private_path(cuda_engine, gmp, pkg, kb):
    import torch
    pk, sk = _keys(pkg, kb)
    ctx = pk.engine_context()
    W = ctx.wave()
    f, bound = 24, 8.0
    K = ctx.slots_per_row((int(bound * 2 ** f) * 1024).bit_length() + 1)
    rows = 2 * W + W // 3                                 # two whole waves and a tail
    count = rows * K - K // 2                             # the last row not full
    gen = torch.Generator(device="cuda:0").manual_seed(kb)
    x = (torch.rand((count // 3, 3), generator=gen, device="cuda:0", dtype=torch.float64) * 2 - 1) * bound
    x[0, :] = torch.tensor([bound, -bound, 0.0], device="cuda:0")
    count = x.numel()
    rows = -(-count // K)
    rng = random.Random(kb)
    rs = [rng.randrange(1, pk.n) for _ in range(rows)]
    v = pk.encrypt_packed(x, bound, frac_bits=f, r_values=rs)
    w = sk.encrypt_packed(x, bound, frac_bits=f, r_values=rs)
    assert (v.slots_per_ciphertext, len(v.ciphertexts), v.shape) == (K, rows, (count // 3, 3))
    assert v.ciphertexts.limbs.is_cuda and torch.equal(v.ciphertexts.limbs, w.ciphertexts.limbs)
    q = torch.round(x.double() * 2.0 ** f).to(torch.int64).reshape(-1).cpu().numpy()
    assert v.decrypt_fixed(sk).reshape(-1).cpu().numpy().tolist() == q.tolist()
    sample = sorted(set([0, 1, W - 1, W, rows - 1] + random.Random(kb + 1).sample(range(rows), 24)))
    opub = orc.PublicConsts(pk.n)
    cs = v.ciphertexts[np.array(sample)].ciphertexts(False)
    want = [orc.raw_encrypt(opub, m, rs[r]) for m, r in zip(_model_rows(pk.n, v.slot_bits, K, q, sample), sample)]
    assert cs == want, kb


def test_five_client_sum_is_exact_and_stays_on_the_device(cuda_engine, pkg):
    import torch
    pk, sk = _keys(pkg, 2048)
    gen = torch.Generator(device="cuda:0").manual_seed(4)
    grads = [torch.randn(20000, generator=gen, device="cuda:0", dtype=torch.float64) * 0.1 for _ in range(5)]
    grads[0][:2] = torch.tensor([1.0, -1.0], device="cuda:0")
    enc = [pk.encrypt_packed(g, 1.0) for g in grads]
    total = sum(enc)
    qs = [torch.round(g * 2.0 ** 24).to(torch.int64) for g in grads]
    fixed = total.decrypt_fixed(sk)
    assert fixed.is_cuda and torch.equal(fixed, sum(qs))
    out = sk.decrypt_batch(total)
    assert out.is_cuda and out.dtype == torch.float64
    assert float((out - sum(grads)).abs().max()) <= 5 * 2.0 ** -25
    diff = (enc[0] - enc[1]) * -3
    assert torch.equal(diff.decrypt_fixed(sk), (qs[0] - qs[1]) * -3)


def test_inside_a_side_stream(cuda_engine, pkg):
    import torch
    pk, sk = _keys(pkg, 2048)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.linspace(-2, 2, 7001, device="cuda:0", dtype=torch.float64).reshape(7001, 1)
        v = pk.encrypt_packed(x, 2.0, frac_bits=30)
        y = sk.encrypt_packed(x, 2.0, frac_bits=30)
        got = (v + y).decrypt_fixed(sk)
        back = pkg.PackedEncryptedVector.from_json(v.to_json(), pk).decrypt(sk)
    s.synchronize()
    q = torch.round(x * 2.0 ** 30).to(torch.int64)
    assert torch.equal(got, 2 * q) and torch.equal(back, q.double() * 2.0 ** -30)
