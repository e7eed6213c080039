"""Plaintext matrix times encrypted vector (EncryptedVector.rmatmul, pai_raw_matvec) on one GPU at a 2048-bit key.

Prints one JSON line: the card and its power limit, the integer-pipe peak measured by bench_micro/imad_peak, and per
workload: the wall time of rmatmul (host preparation included; warm-up of the same shapes first, a device synchronise
at the end), terms per second, the window width picked, the device time of the pai_raw_matvec call alone (CUDA events
around it: flags, inverses, tables, rows), the 32x32->64 MACs the kernels execute counted from the shapes (an upper
bound: every digit of every term counted non-zero), their rate over the device time against the peak, and the
speed-up over the per-row loop users write today, timed on a sample of rows and scaled.  Every workload's result is
checked against the GMP oracle on sampled rows.

Workloads:
  dense      10 000 x 1 000 Gaussian float64 matrix, encrypted Gaussian weights; per-row loop: v.dot(X[j])
  sparse     100 000 x 20 000 at 0.5 % density, non-negative tf-idf-like values, skewed row lengths (a few rows of
             2 000 entries, some empty); per-row loop: v[x.indices].dot(x.data)
  histogram  0/1 indicator matrix, 10^6 encrypted gradients into 10^4 segments; per-row loop as for sparse

    python bench_micro/matvec_rate.py [--scale 0.1] [--baseline-rows 200] [--parity-rows 64]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def digit_macs(kb):
    """32x32->64 MACs of one dsqr and one dmul of the digit kernels (bench.executed_macs' count)"""
    t = kb // 256
    return 64 * (t * (t + 1) // 2 + 3 * t * t) + 72 * t, 64 * 5 * t * t + 72 * t


def executed_macs(kb, call, w):
    """the kernels' work from the shapes the call passed, by the window rule's own count: table products (and the two
    products of entering the domain per tabled base), squarings at the bit bound, one product per term and window,
    leaving the domain per row"""
    _, ncols, _, _, _, _, bits, d_neg, nnz, nrows = call[:10]
    tabled = ncols * (2 if d_neg is not None else 1)
    sq, mul = digit_macs(kb)
    nwin = -(-bits // w)
    return (tabled * ((1 << w) - 2 + 2) * mul + nrows * (nwin - 1) * w * sq + nnz * nwin * mul + nrows * mul), tabled


def oracle_rows(pkg, orc, opub, pk, cs, vexps, rows):
    """[(ciphertext, exponent)] of rows given as (column list, value list), by dot()'s rule: raw_mul per term"""
    out = []
    for cols, vals in rows:
        encs = [pkg.EncodedNumber.encode(pk, x) for x in vals]
        exps = [int(vexps[i]) + e.exponent for i, e in zip(cols, encs)]
        if not exps:
            out.append((1, 0))
            continue
        low = min(exps)
        acc = 1
        for i, e, x in zip(cols, encs, exps):
            acc = orc.raw_add(opub, acc, orc.raw_mul(opub, cs[i], e.encoding * pkg.EncodedNumber.BASE ** (x - low) % pk.n))
        out.append((acc, low))
    return out


def skewed_csr(sp, rng, nrows, ncols, density, long_rows, long_len, empty_frac):
    """tf-idf-like rows: lognormal row lengths around density * ncols, a few rows of long_len entries, a share of empty
    rows; columns drawn with replacement (a repeated column is summed into one entry, as tocsr() does)"""
    lens = (rng.poisson(density * ncols, size=nrows) * rng.lognormal(-0.25, 0.7, size=nrows)).astype(np.int64)
    lens = np.minimum(lens, ncols)
    lens[rng.random(nrows) < empty_frac] = 0
    lens[rng.choice(nrows, size=long_rows, replace=False)] = long_len
    rows = np.repeat(np.arange(nrows), lens)
    cols = rng.integers(0, ncols, size=len(rows))
    data = rng.exponential(1.0, size=len(rows)) * np.log(1 + ncols / (1 + cols))             # tf * idf
    return sp.csr_matrix((data, (rows, cols)), shape=(nrows, ncols))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every row count (quick runs)")
    ap.add_argument("--baseline-rows", type=int, default=200)
    ap.add_argument("--parity-rows", type=int, default=64)
    args = ap.parse_args()
    import torch
    import scipy.sparse as sp
    import paillier_b200 as pkg
    from bench import measured_int_peak
    from oracle import paillier_oracle as orc
    from oracle.golden import H, load_golden

    name, power = card()
    peak = measured_int_peak()
    peak_mac_s = peak["mac_per_clk_sm"] * peak["mhz"] * 1e6 * peak["sms"]
    kb = 2048
    fx = load_golden("vectors_%d.json" % kb)
    pk = pkg.PaillierPublicKey(H(fx["n"]))
    ctx = pk.engine_context()
    orc.BACKEND = "gmp" if orc.have_gmp() else "python"
    opub = orc.PublicConsts(pk.n)
    rng = np.random.default_rng(2026)
    calls = []
    raw = ctx.raw_matvec_dev

    def recording(*a, **k):                               # the call's shapes, and its device time between two events
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = raw(*a, **k)
        e1.record()
        calls.append((a, e0, e1))
        return r
    ctx.raw_matvec_dev = recording

    def scaled(x):
        return max(1, int(x * args.scale))
    work = {}
    d = 1000
    work["dense"] = (rng.normal(size=(scaled(10000), d)), [float(x) for x in rng.normal(size=d)])
    work["sparse"] = (skewed_csr(sp, rng, scaled(100000), 20000, 0.005, 5, 2000, 0.05), [float(x) for x in rng.normal(size=20000)])
    nv, nseg = scaled(10 ** 6), scaled(10 ** 4)
    seg = rng.integers(0, nseg, size=nv)
    work["histogram"] = (sp.csr_matrix((np.ones(nv, dtype=np.int64), (seg, np.arange(nv))), shape=(nseg, nv)),
                         [float(x) for x in rng.normal(0, 0.1, size=nv)])
    result = {"bench": "matvec_rate", "gpu": name, "power_limit": power, "key_bits": kb, "imad_peak": peak,
              "imad_peak_mac_s": peak_mac_s, "workloads": {}}
    for label, (X, w) in work.items():
        v = pk.encrypt_batch(w)
        sparse = sp.issparse(X)
        nrows = X.shape[0]
        y = v.rmatmul(X)                                  # warm-up of the same shapes, and the result checked below
        torch.cuda.synchronize()
        calls.clear()
        t0 = time.perf_counter()
        y2 = v.rmatmul(X)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        call, e0, e1 = calls[-1]
        device = e0.elapsed_time(e1) / 1e3
        nnz, bits, neg = int(call[8]), int(call[6]), call[7] is not None
        win = ctx.matvec_window(int(call[1]), nrows, nnz, bits, neg)
        macs, tabled = executed_macs(kb, call, win)
        # parity: both runs, against the GMP oracle on sampled rows
        got = y.ciphertexts(False)
        assert got == y2.ciphertexts(False)
        cs = v.ciphertexts(False)
        pr = random.Random(7).sample(range(nrows), min(args.parity_rows, nrows))
        if sparse:
            Xc = X.tocsr()
            rows = [(Xc[j].indices.tolist(), Xc[j].data.tolist()) for j in pr]
        else:
            rows = [(list(range(X.shape[1])), X[j].tolist()) for j in pr]
        ok = all(got[j] == c and int(y.exponents[j]) == e for j, (c, e) in zip(pr, oracle_rows(pkg, orc, opub, pk, cs, v.exponents, rows)))
        # per-row loop on a sample of rows, scaled to all rows
        br = random.Random(8).sample(range(nrows), min(args.baseline_rows, nrows))
        if sparse:
            Xc = X.tocsr()
            br = [j for j in br if Xc.indptr[j + 1] > Xc.indptr[j]] or br
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j in br:
            if sparse:
                x = Xc[j]
                if x.nnz:
                    v[x.indices.astype(np.int64)].dot(x.data)
            else:
                v.dot(X[j])
        torch.cuda.synchronize()
        loop = (time.perf_counter() - t0) * nrows / len(br)
        result["workloads"][label] = {
            "shape": [int(nrows), int(X.shape[1])], "terms": nnz, "mag_limbs": int(call[5]), "mag_bits": bits,
            "negative_scalars": neg, "tabled_bases": int(tabled), "window": win, "wall_s": wall, "terms_per_s": nnz / wall,
            "device_s": device, "executed_macs": int(macs), "executed_mac_per_s_device": macs / device,
            "share_of_imad_peak_device": macs / device / peak_mac_s, "executed_mac_per_s_wall": macs / wall,
            "row_loop_s_scaled": loop, "row_loop_sample_rows": len(br), "speedup_over_row_loop": loop / wall,
            "oracle_rows": len(pr), "oracle_parity": bool(ok)}
        del y, y2, v
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
