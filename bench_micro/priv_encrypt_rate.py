"""Encryption with the private key (pai_priv_encrypt) against public-key encryption (pai_encrypt) on one GPU.

For the fixed 1024-, 2048-, 3072- and 4096-bit keys (fixtures.fixed_key): m and r are drawn on the device from a seeded
ChaCha20 stream (pai_random_lt_n), the batch is two whole waves of pai_encrypt plus half a wave; both paths are warmed up
and then timed alternately, three times each, with CUDA events around the call.  Per key one JSON line: rows/s of both
paths with the spread (max - min over the median), the 32x32->64 MACs the kernels execute per row counted from the
loops (bench.executed_macs' conventions) and their rate against the integer-pipe peak measured by bench_micro/imad_peak,
the latency of a call of 1, 32 and 1024 rows (median of five), whether all rows of the two paths are equal, and whether
64 sampled rows equal the GMP oracle.  The first line holds the card's name and power limit.

    python bench_micro/priv_encrypt_rate.py [--keys 1024,2048,3072,4096] [--waves 2]
"""
import argparse
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def crt_macs(p, q):
    """32x32->64 MACs of one row of pai_priv_encrypt (pai_digit.cuh), counted from the loops with bench.executed_macs'
    per-product costs; mont_sqr counted as mont_mul"""
    t = max(p, q).bit_length() + 255 >> 8
    t = next(v for v in (1, 2, 3, 4, 6, 8) if v >= t)

    def dsqr():
        return 64 * (t * (t + 1) // 2 + 3 * t * t) + 72 * t

    def dmul():
        return 64 * 5 * t * t + 72 * t

    def mont():
        return 64 * (2 * t * t + t) + 36 * t
    total = 0
    for x in (p, q):
        nwin = -(-x.bit_length() // 5)
        sq, mu = 1 + 5 * (nwin - 1), 29 + (nwin - 1)
        total += (2 + 2 + sq + mu) * mont() + sq * dsqr() + mu * dmul()    # r mod x, t_x, step 1, step 2
    total += 5 * dmul() + 2 * 64 * t * t + 64 * (2 * t) ** 2                # message factors, CRT, digits -> plain
    return total


def timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", default="1024,2048,3072,4096")
    ap.add_argument("--waves", type=int, default=2)
    args = ap.parse_args()
    import torch
    import paillier_b200 as pkg
    from bench import executed_macs, measured_int_peak
    from oracle import paillier_oracle as orc
    from importlib import import_module
    fixtures = import_module("python-paillier_b200.fixtures")
    E = import_module("python-paillier_b200.engine")
    V = import_module("python-paillier_b200.vector")
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"

    name, power = card()
    peak = measured_int_peak()
    peak_mac_s = peak["mac_per_clk_sm"] * peak["mhz"] * 1e6 * peak["sms"]
    print(json.dumps({"bench": "priv_encrypt_rate", "gpu": name, "power_limit": power, "imad_peak": peak,
                      "imad_peak_mac_s": peak_mac_s, "oracle": orc.BACKEND}), flush=True)
    for kb in [int(k) for k in args.keys.split(",")]:
        n, p, q = fixtures.fixed_key(kb)
        p, q = min(p, q), max(p, q)
        pub, priv = pkg.PublicContext(n), pkg.PrivateContext(p, q)
        W = pub.wave()
        B = args.waves * W + W // 2
        ln = pub.n_limbs
        d_m = torch.empty((B, ln), dtype=torch.int32, device="cuda:0")
        d_r = torch.empty((B, ln), dtype=torch.int32, device="cuda:0")
        pub.random_lt_n_dev(d_m, B, seed=bytes(range(32)), nonce=kb)
        pub.random_lt_n_dev(d_r, B, seed=bytes(range(32)), nonce=kb + 1)
        pm, pr = V._rows_for(priv.n_limbs, d_m), V._rows_for(priv.n_limbs, d_r)
        c_pub = torch.empty((B, pub.c_limbs), dtype=torch.int32, device="cuda:0")
        c_priv = torch.empty((B, priv.c_limbs), dtype=torch.int32, device="cuda:0")

        def run_pub(b=B):
            pub.encrypt_dev(d_m, d_r, c_pub, b)

        def run_priv(b=B):
            priv.encrypt_dev(pm, pr, c_priv, b)
        run_pub(); run_priv(); torch.cuda.synchronize()
        t_pub, t_priv = [], []
        for _ in range(3):
            t_pub.append(timed(run_pub))
            t_priv.append(timed(run_priv))
        equal = bool(torch.equal(V._rows_for(pub.c_limbs, c_priv), c_pub))
        idx = random.Random(kb).sample(range(B), 64)
        ms = E.limbs_to_ints(V._to_host(d_m[idx]))
        rs = E.limbs_to_ints(V._to_host(d_r[idx]))
        cs = E.limbs_to_ints(V._to_host(V._rows_for(pub.c_limbs, c_priv[idx])))
        opub = orc.PublicConsts(n)
        oracle_ok = cs == [orc.raw_encrypt(opub, m, r) for m, r in zip(ms, rs)]
        lat = {}
        for rows in (1, 32, 1024):
            for label, fn in (("public", run_pub), ("private", run_priv)):
                fn(rows); torch.cuda.synchronize()
                ts = sorted(timed(lambda: fn(rows)) for _ in range(5))
                lat["%s_%d" % (label, rows)] = ts[2]
        macs_pub = executed_macs(kb, n)["encrypt"]
        macs_priv = crt_macs(p, q)

        def stats(ts, macs):
            med = sorted(ts)[1]
            return {"rows_per_s": B / med, "times_s": ts, "spread": (max(ts) - min(ts)) / med, "executed_macs_per_row": macs,
                    "share_of_imad_peak": macs * B / med / peak_mac_s}
        print(json.dumps({"key_bits": kb, "batch": B, "public_wave": W, "public": stats(t_pub, macs_pub),
                          "private": stats(t_priv, macs_priv), "speedup": sorted(t_pub)[1] / sorted(t_priv)[1],
                          "latency_s": lat, "rows_equal": equal, "oracle_rows_equal": oracle_ok}), flush=True)
        pub.close(); priv.close()


if __name__ == "__main__":
    main()
