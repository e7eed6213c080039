"""Numerical model (numpy, CPU) of the reductions of pai_tc.cuh: the two constant-operand
multiplications of a Montgomery reduction as batch GEMMs in 8-bit digits -- the arithmetic a u8 x u8 -> s32 tensor-core (`wgmma`)
kernel would perform, with the int32 column-sum bounds checked.  Not used by the engine; exercised by
tests/test_redc_gemm_model.py against Python integers.

REDC(t) for t < N*R, R = 256^D:   m = (t mod R) * N' mod R,   u = (t + m*N) / R,   u -= N if u >= N.
  m     = carry_propagate( T_low[batch, D]  @ Toeplitz_low(N')[D, D] )  mod R      (GEMM 1: lower-triangular band)
  hi    = carry_propagate( m[batch, D]      @ Toeplitz_high(N)[D, D] )            (GEMM 2: only the columns >= D)
  u     = t_high + hi + (t_low != 0)      -- the low halves of t and m*N sum to exactly 0 or R
GEMM 2 only computes the G = 4 guard columns below column D and the D columns above it.  The carry of the
discarded low columns into column D is still exact, because low(m*N) = (R - t_low) mod R is known: with
T = guard column sums as an integer (units of 256^(D-G)) and Lq = the top G digits of low(m*N),
S_low - low(m*N) = carry * R  implies  T - Lq = carry * 256^G - delta with an integer 0 <= delta < 2^24.1 < 256^G,
hence carry = ceil((T - Lq) / 256^G).
"""
import numpy as np


def to_digits(values, D):
    raw = b"".join(int(v).to_bytes(D, "little") for v in values)
    return np.frombuffer(raw, dtype=np.uint8).reshape(len(values), D).astype(np.int64)


def from_digits(mat):
    """rows of (possibly unnormalised, non-negative) base-256 column sums -> Python ints"""
    out = []
    for row in mat:
        v = 0
        for i in range(len(row) - 1, -1, -1):
            v = (v << 8) + int(row[i])
        out.append(v)
    return out


def toeplitz(const_digits, rows, cols, shift=0):
    """T[i, j] = const[j + shift - i]: row-vector x times T = columns [shift, shift + cols) of the product x * const"""
    T = np.zeros((rows, cols), dtype=np.int64)
    L = len(const_digits)
    for i in range(rows):
        for j in range(cols):
            k = j + shift - i
            if 0 <= k < L:
                T[i, j] = const_digits[k]
    return T


def carry_propagate(cols, D_out):
    """column sums (int64, < 2^31) -> D_out normalised digits + carry out (vectorised over the batch)"""
    cols = cols.copy()
    carry = np.zeros(cols.shape[0], dtype=np.int64)
    out = np.zeros((cols.shape[0], D_out), dtype=np.int64)
    for j in range(D_out):
        v = cols[:, j] + carry
        out[:, j] = v & 0xFF
        carry = v >> 8
    return out, carry


def redc_gemm(t_values, N, D, guard=4):
    """Batched Montgomery reduction with the two GEMMs; returns (u list, max column sum seen)."""
    R = 1 << (8 * D)
    Np = (-pow(N, -1, R)) % R
    nd, npd = to_digits([N], D)[0], to_digits([Np], D)[0]
    t = to_digits(t_values, 2 * D)
    t_low, t_high = t[:, :D], t[:, D:]
    # GEMM 1: low D columns of t_low * N'
    c1 = t_low @ toeplitz(npd, D, D, 0)
    m, _ = carry_propagate(c1, D)
    # GEMM 2: columns [D - guard, 2D) of m * N; the guard columns only feed the carry into column D
    c2 = m @ toeplitz(nd, D, D + guard, D - guard)
    assert c1.max() < 2 ** 31 and c2.max() < 2 ** 31
    lows_nonzero = (t_low != 0).any(axis=1).astype(np.int64)
    t_low_vals = from_digits(t_low)
    m_vals = from_digits(m)
    # reference: exact high half of m*N on Python integers
    mN_high_exact = [(mv * N) >> (8 * D) for mv in m_vals]
    # kernel route: guard columns + the known low half give the exact carry into column D
    G = guard
    T = [sum(int(c2[r, g]) << (8 * g) for g in range(G)) for r in range(c2.shape[0])]
    Lq = [(((R - tl) % R) >> (8 * (D - G))) for tl in t_low_vals]
    carry_in = np.array([-((Lq_ - T_) // (1 << (8 * G))) for T_, Lq_ in zip(T, Lq)], dtype=np.int64)   # ceil((T - Lq) / 256^G)
    hi_cols = c2[:, G:].copy()
    hi_cols[:, 0] += carry_in
    hi, carry_top = carry_propagate(hi_cols, D)
    hi_vals = [h + (int(c) << (8 * D)) for h, c in zip(from_digits(hi), carry_top)]
    u = []
    for hv, exact, th, nz in zip(hi_vals, mN_high_exact, from_digits(t_high), lows_nonzero):
        val = hv + th + int(nz)
        if val >= N:
            val -= N
        u.append((val, hv == exact))
    return u, int(max(c1.max(), c2.max()))
