"""Quick device-resident throughput probe (not the contract bench): encrypt / decrypt / add / mul kernels."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import paillier_b200 as pb
import importlib
_fx = importlib.import_module("python-paillier_b200.fixtures")
H, load_golden = _fx.H, _fx.load_golden

def run(kb, batch):
    fx = load_golden("vectors_%d.json" % kb)
    n, p, q = H(fx["n"]), H(fx["p"]), H(fx["q"])
    pub = pb.PublicContext(n); priv = pb.PrivateContext(p, q)
    ln, lc = pub.n_limbs, pub.c_limbs
    rng = np.random.default_rng(1)
    m = rng.integers(0, 2**32, size=(batch, ln), dtype=np.uint32); m[:, (kb // 32) - 1:] = 0
    r = rng.integers(0, 2**32, size=(batch, ln), dtype=np.uint32); r[:, (kb // 32) - 1:] = 0
    dm, dr = torch.from_numpy(m.view(np.int32)).cuda(), torch.from_numpy(r.view(np.int32)).cuda()
    dc = torch.empty((batch, lc), dtype=torch.int32, device="cuda"); dc2 = torch.empty_like(dc)
    dd = torch.empty((batch, ln), dtype=torch.int32, device="cuda")
    st = torch.empty((batch,), dtype=torch.int32, device="cuda")
    res = {"key_bits": kb, "batch": batch}
    def timeit(name, fn, reps=2):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps): fn()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        res[name + "_ms"] = round(ms, 3); res[name + "_per_s"] = round(batch / ms * 1e3, 1)
    timeit("encrypt", lambda: pub.encrypt_dev(dm, dr, dc, batch))
    timeit("decrypt", lambda: priv.decrypt_dev(dc, dd, batch))
    ok = bool((dd[:, :ln] == dm).all().item())
    res["roundtrip_ok"] = ok
    timeit("add", lambda: pub.raw_add_dev(dc, dc, dc2, batch), reps=5)
    ds = torch.zeros((batch, ln), dtype=torch.int32, device="cuda"); ds[:, :2] = dm[:, :2]
    timeit("mul64", lambda: pub.raw_mul_dev(dc, ds, dc2, st, batch))
    print(json.dumps(res), flush=True)

if __name__ == "__main__":
    for kb, b in [(1024, 132 * 256 * 4), (2048, 132 * 224 * 4), (3072, 132 * 128 * 2)]:
        run(kb, b)
