"""Small workload for compute-sanitizer (memcheck / racecheck): every round-2 kernel on a 1024-bit key -- tensor-core
encrypt / decrypt / raw_mul (forced: PAI_TC=2), amortised inversion, product reduction, Straus dot product, batched
Miller-Rabin, and the same context driven from two CUDA streams.   python sanitize_target.py [rows [key_bits]]
(2048-bit keys with PAI_TC_GROUPS=3 in the environment: three groups per CTA, x1 in L2)"""
import os, sys
os.environ["PAI_TC"] = "2"
os.environ["PAI_COOP_MAX"] = "0"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, random
import paillier_b200 as pb, importlib
_fx = importlib.import_module("python-paillier_b200.fixtures")
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 300
n, p, q = _fx.fixed_key(int(sys.argv[2]) if len(sys.argv) > 2 else 1024)
pk = pb.PaillierPublicKey(n); sk = pb.PaillierPrivateKey(pk, p, q)
pub, priv = pk.engine_context(), sk.engine_context()
assert pub.kernel_path() == "tc" and priv.kernel_path() == "tc"
rng = random.Random(1)
ms = [rng.randrange(n) for _ in range(rows)]; rs = [rng.randrange(1, n) for _ in range(rows)]
cs = pub.raw_encrypt(ms, rs)
assert priv.raw_decrypt(cs) == ms
ks = [rng.getrandbits(40) if i % 2 else n - 1 - rng.getrandbits(30) for i in range(rows)]
out, st = pub.raw_mul(cs, ks)
assert not any(st) and priv.raw_decrypt(out) == [m * (k if k < n // 2 else k - n) % n for m, k in zip(ms, ks)]
vals = np.arange(rows, dtype=np.int64) - rows // 2
v = pk.encrypt_batch(vals)
assert sk.decrypt(v.sum()) == int(vals.sum())
w = np.arange(rows, dtype=np.int64) % 7 - 3
assert sk.decrypt(v.dot(w)) == int((vals * w).sum())
s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
res = []
for s in (s1, s2):
    with torch.cuda.stream(s):
        x = pk.encrypt_batch(vals[:128])
        res.append(((x + x) * 3, s))
torch.cuda.synchronize()
for r, s in res:
    assert sk.decrypt_batch(r) == [int(6 * a) for a in vals[:128]]
util = importlib.import_module("python-paillier_b200.util")
assert util.is_prime_batch([2 ** 127 - 1, 2 ** 127 + 1, 3825123056546413051]) == [True, False, False]
print("sanitize target ok", rows)
