"""Target for per-kernel ncu captures of K2/K3/K4: one wave each of decrypt, raw_add, raw_mul (pos + neg scalars)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import paillier_b200 as pb
import importlib
_fx = importlib.import_module("python-paillier_b200.fixtures")
H, load_golden = _fx.H, _fx.load_golden

kb = 2048
fx = load_golden("vectors_%d.json" % kb)
n = H(fx["n"])
pub = pb.PublicContext(n); priv = pb.PrivateContext(H(fx["p"]), H(fx["q"]))
batch = 132 * 224
ln, lc = pub.n_limbs, pub.c_limbs
rng = np.random.default_rng(1)
m = rng.integers(0, 2**32, size=(batch, ln), dtype=np.uint32); m[:, kb // 32 - 1:] = 0
r = rng.integers(0, 2**32, size=(batch, ln), dtype=np.uint32); r[:, kb // 32 - 1:] = 0
dm, dr = torch.from_numpy(m.view(np.int32)).cuda(), torch.from_numpy(r.view(np.int32)).cuda()
dc = torch.empty((batch, lc), dtype=torch.int32, device="cuda"); dc2 = torch.empty_like(dc)
dd = torch.empty((batch, ln), dtype=torch.int32, device="cuda")
st = torch.zeros((batch,), dtype=torch.int32, device="cuda")
ds = torch.zeros((batch, ln), dtype=torch.int32, device="cuda"); ds[:, :2] = dm[:, :2]
neg = pb.ints_to_limbs([n - 12345], ln).view(np.int32)
ds[: batch // 64] = torch.from_numpy(neg.copy()).cuda()          # a few negative scalars -> inverse branch
for _ in range(2):
    pub.encrypt_dev(dm, dr, dc, batch)
    priv.decrypt_dev(dc, dd, batch)
    pub.raw_add_dev(dc, dc, dc2, batch)
    pub.raw_mul_dev(dc, ds, dc2, st, batch)
torch.cuda.synchronize()
assert bool((dd == dm).all().item())
print("ok", batch)
