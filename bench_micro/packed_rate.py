"""One federated-learning round (bench.py configs[4]: 5 clients x D float64 gradients, 2048-bit key), unpacked against
packed, on one GPU.

Unpacked is today's path: encrypt_batch per client, `+` over the clients, decrypt_batch.  Packed quantises each gradient
with frac_bits fractional bits under a declared bound (|g| <= --bound; the gradients are randn * 0.1, as in configs[4]),
packs slots_per_ciphertext values into each plaintext on the device and runs the same three steps on the packed rows.
Both paths are warmed up on a small round, then timed alternately --repeats times; each step ends in a device
synchronise.  Per path: the median seconds of encrypt / sum / decrypt, values/s of the whole round, the ciphertext count
of one client, the bytes of one client's to_json, and the max |error| of the decrypted mean against the numpy mean.  The
card's name and power limit are read in the same run.  One JSON file goes to --out.

    python bench_micro/packed_rate.py --out DIR [--dim 100000] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--dim", type=int, default=100000)
    ap.add_argument("--clients", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--bound", type=float, default=1.0)
    ap.add_argument("--frac-bits", type=int, default=24)
    ap.add_argument("--headroom", type=int, default=1024)
    args = ap.parse_args()
    import numpy as np
    import torch
    import paillier_b200 as pkg
    from importlib import import_module
    fixtures = import_module("python-paillier_b200.fixtures")
    if not torch.cuda.is_available():
        raise SystemExit("packed_rate measures on a CUDA device; none is visible")

    name, power = card()
    n, p, q = fixtures.fixed_key(2048)
    pk = pkg.PaillierPublicKey(n)
    sk = pkg.PaillierPrivateKey(pk, p, q)
    D, C = args.dim, args.clients
    grads = [np.random.RandomState(43 + i).randn(D) * 0.1 for i in range(C)]
    assert max(np.abs(g).max() for g in grads) <= args.bound
    mean = np.mean(grads, axis=0)
    d_grads = [torch.from_numpy(g).to("cuda:0") for g in grads]
    kw = dict(frac_bits=args.frac_bits, headroom=args.headroom)

    def step(t, key, fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        t[key] = time.perf_counter() - t0
        return out

    def unpacked(gs, t):
        enc = step(t, "encrypt_s", lambda: [pk.encrypt_batch(g) for g in gs])
        acc = step(t, "sum_s", lambda: sum(enc[1:], enc[0]))
        agg = step(t, "decrypt_s", lambda: np.array(sk.decrypt_batch(acc)) / len(gs))
        return enc[0], agg

    def packed(gs, t):
        enc = step(t, "encrypt_s", lambda: [pk.encrypt_packed(g, args.bound, **kw) for g in gs])
        acc = step(t, "sum_s", lambda: sum(enc))
        agg = step(t, "decrypt_s", lambda: (sk.decrypt_batch(acc) / len(gs)).cpu().numpy())
        return enc[0], agg

    paths = {"unpacked": (unpacked, grads), "packed": (packed, d_grads)}
    for fn, gs in paths.values():                       # warm-up: every call of the round on a small vector
        fn([g[:D // 2 + 7] for g in gs[:2]], {})
    times = {k: [] for k in paths}
    results = {}
    for _ in range(args.repeats):
        for k, (fn, gs) in paths.items():
            t = {}
            results[k] = fn(gs, t)
            t["round_s"] = t["encrypt_s"] + t["sum_s"] + t["decrypt_s"]
            times[k].append(t)
    out = {"bench": "packed_rate", "gpu": name, "power_limit": power, "key_bits": 2048, "clients": C, "dim": D,
           "repeats": args.repeats, "bound": args.bound, **kw}
    for k, ts in times.items():
        first, agg = results[k]
        med = {s: sorted(t[s] for t in ts)[len(ts) // 2] for s in ts[0]}
        rows = len(first.ciphertexts) if k == "packed" else len(first)
        out[k] = {"median_s": med, "times_s": ts, "values_per_s": C * D / med["round_s"], "ciphertexts_per_client": rows,
                  "to_json_bytes_per_client": len(first.to_json()), "max_abs_error_of_mean": float(np.abs(agg - mean).max())}
    pv = results["packed"][0]
    out["packed"].update(slot_bits=pv.slot_bits, slots_per_ciphertext=pv.slots_per_ciphertext)
    # the packed sum of C quantised values is within C * 2^-(f+1) of the float sum, the mean within 2^-(f+1)
    out["packed_sum_within_quantisation"] = bool(out["packed"]["max_abs_error_of_mean"] * C <= C * 2.0 ** -(args.frac_bits + 1))
    out["speedup_round"] = out["unpacked"]["median_s"]["round_s"] / out["packed"]["median_s"]["round_s"]
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "packed_rate.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: out[k] for k in ("gpu", "power_limit", "speedup_round", "packed_sum_within_quantisation")}))
    print(json.dumps({k: {s: out[k][s] for s in ("median_s", "values_per_s", "ciphertexts_per_client",
                                                  "to_json_bytes_per_client", "max_abs_error_of_mean")}
                      for k in paths}))


if __name__ == "__main__":
    main()
