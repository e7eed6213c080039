"""Small-batch latency at a 2048-bit key: warp-per-ciphertext kernels (pai_coop.cuh) against the thread-per-ciphertext
throughput kernels, device-resident inputs, CUDA-event timing (prints one JSON line)."""
import importlib
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pkg = importlib.import_module("python-paillier_b200")
import importlib
_fx = importlib.import_module("python-paillier_b200.fixtures")
H, load_golden = _fx.H, _fx.load_golden

kb = int(os.environ.get("LAT_KEYBITS", 2048))
fx = load_golden("vectors_%d.json" % kb)
n, p, q = H(fx["n"]), H(fx["p"]), H(fx["q"])
pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
rng = np.random.default_rng(0)
sizes = [1, 8, 64, 132, 528, 1024, 2112, 4224, 8448]
hybrid = pub.wave() + 4000       # one full encrypt wave plus a tail
top = max(sizes + [hybrid])
m = rng.integers(0, 2 ** 32, size=(top, pub.n_limbs), dtype=np.uint32); m[:, kb // 32 - 1:] = 0
r = rng.integers(0, 2 ** 32, size=(top, pub.n_limbs), dtype=np.uint32); r[:, kb // 32 - 1:] = 0; r[:, 0] |= 1
d_m = torch.from_numpy(m.view(np.int32)).cuda(); d_r = torch.from_numpy(r.view(np.int32)).cuda()
d_c = torch.empty((top, pub.c_limbs), dtype=torch.int32, device="cuda")
d_d = torch.empty_like(d_m)
out = {"workload": "%d-bit key, ms per call" % kb, "rows": []}
ref = None
for mode, env in (("thread", "0"), ("warp", "1000000")):
    os.environ["PAI_COOP_MAX"] = env
    for b in sizes:
        if mode == "thread" and b not in (1, 132, 1024, 8448):
            continue
        for _ in range(2):
            pub.encrypt_dev(d_m, d_r, d_c, b); priv.decrypt_dev(d_c, d_d, b)
        torch.cuda.synchronize()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record(); pub.encrypt_dev(d_m, d_r, d_c, b)
        e[1].record(); priv.decrypt_dev(d_c, d_d, b)
        e[2].record(); torch.cuda.synchronize()
        ok = bool((d_d[:b] == d_m[:b]).all().item())
        if b == 1024:
            if ref is None:
                ref = d_c[:b].clone()
            else:
                ok = ok and bool((ref == d_c[:b]).all().item())
        out["rows"].append({"path": mode, "batch": b, "encrypt_ms": round(e[0].elapsed_time(e[1]), 3),
                            "decrypt_ms": round(e[1].elapsed_time(e[2]), 3), "roundtrip_ok": ok})
for mode, env in (("thread only", "0"), ("default: waves on threads, tail on warps", None)):
    if env is None:
        os.environ.pop("PAI_COOP_MAX", None)
    else:
        os.environ["PAI_COOP_MAX"] = env
    b = hybrid
    for _ in range(2):
        pub.encrypt_dev(d_m, d_r, d_c, b); priv.decrypt_dev(d_c, d_d, b)
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e[0].record(); pub.encrypt_dev(d_m, d_r, d_c, b)
    e[1].record(); priv.decrypt_dev(d_c, d_d, b)
    e[2].record(); torch.cuda.synchronize()
    out["rows"].append({"path": mode, "batch": b, "encrypt_ms": round(e[0].elapsed_time(e[1]), 3),
                        "decrypt_ms": round(e[1].elapsed_time(e[2]), 3), "roundtrip_ok": bool((d_d[:b] == d_m[:b]).all().item())})
print(json.dumps(out))
