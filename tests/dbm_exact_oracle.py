"""Exact log Z and log p*(v) of binary DBMs by enumerating the odd layers (DESIGN.md §5.4f) -- TEST INFRASTRUCTURE ONLY.

Unit layer j = 0..L is v (j = 0) or h_j (tests/dbm_ais_depth_oracle.py).  The odd layers form the state x, numbered by the
integer s whose bits are x_1, then x_3, ... (x_1 in the lowest bits), and v and the even layers are summed out:

    log p*(x) = sum_{odd j} b_j.x_j + sum_{even j} sum_n softplus(z_{j,n}(x))
    log Z     = LSE_x log p*(x)
    log p*(v) = b_v.v + LSE_x [x_1.(v W_0) + g(x)],     g(x) = log p*(x) - sum_n softplus(z_{0,n}(x))

`exact` states this in float64 over chunks of states, for any X (grey rows included); `bf16_split` is the engine's weight
operand hi + lo.
"""
import numpy as np

import dbm_ais_depth_oracle as A


def n_odd(prm):
    w = A.widths(prm)
    return sum(w[j] for j in range(1, len(w), 2))


def _bits(s, lo, n):
    return ((s[:, None] >> (lo + np.arange(n))[None, :]) & 1).astype(np.float64)


def exact(prm, X=None, chunk_bits=16):
    """(log Z, log p*(v) [rows] or None) in float64, enumerating 2^chunk_bits states at a time"""
    Ws, bs = A.unit_layers(prm)
    w = A.widths(prm)
    L = len(w) - 1
    odd = list(range(1, L + 1, 2))
    lo = {}
    k = 0
    for j in odd:
        lo[j] = k
        k += w[j]
    total = 1 << k
    if X is not None:
        X = np.asarray(X, np.float64)
        Q = X @ Ws[0]                                   # [rows, n_1]
        lp_rows = np.full(len(X), -np.inf)
    lz = -np.inf
    step = 1 << min(k, chunk_bits)
    for s0 in range(0, total, step):
        s = np.arange(s0, s0 + step, dtype=np.int64)
        x = {j: _bits(s, lo[j], w[j]) for j in odd}
        lin = sum(x[j] @ bs[j] for j in odd)
        rest = sum((A.softplus(A.z_raw(Ws, x, j) + bs[j]).sum(axis=1) for j in range(2, L + 1, 2)), np.zeros(step))
        sp0 = A.softplus(A.z_raw(Ws, x, 0) + bs[0]).sum(axis=1)
        lz = np.logaddexp(lz, np.logaddexp.reduce(lin + rest + sp0))
        if X is not None:
            t = Q @ x[1].T + (lin + rest)[None, :]
            lp_rows = np.logaddexp(lp_rows, np.logaddexp.reduce(t, axis=1))
    return float(lz), (None if X is None else X @ bs[0] + lp_rows)


def bf16_split(W):
    """hi = bf16(W), lo = bf16(W - hi), both round-to-nearest-even, as float32 arrays"""
    def r(a):
        u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
        u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
        return u.astype(np.uint32).view(np.float32)
    hi = r(W)
    return hi, r(np.asarray(W, np.float32) - hi)
