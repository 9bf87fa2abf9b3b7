"""AIS estimates of log p*(v) of binary DBMs with v clamped (DESIGN.md §5.4g) restated -- TEST INFRASTRUCTURE ONLY.

Unit layers j = 0..L as in dbm_ais_depth_oracle.py (j = 0 is v).  With v clamped to a row X_r the odd hidden layers are summed
out and the even hidden layers h_2, h_4, ... are the chains' state x (x_0 = v):

    log p*_beta(x; v) = beta (b_v.v + sum_{even j >= 2} b_j.x_j) + sum_{odd j} sum_n softplus(beta z_{j,n}),
    z_j = b_j + x_{j-1} W_{j-1} + x_{j+1} W_j^T.

At beta = 1 the sum over x is p*(v); at beta = 0 it is 2^(sum_i H_i).  The b_v.v term is linear in beta, so it is added once,
with log Z_0 = (sum_i H_i) log 2, to every run.

`ais` states the ladder in two arithmetics, as dbm_ais_depth_oracle.ais does: float64 throughout (bf16=False), or the tensor-
core engine's (bf16=True: bf16 weights and bf16(X) in the products, fp32 pre-activations, float32 increments summed in
float64; b_v.X in float64 from the float32 X).  Temperatures, sweeps and the order of the draws are the depth ladder's with
the roles moved up one layer; every layer drawn is sampled.  Chain c = r n_runs + k (run k of row r) draws from Philox row
(row0 + r) n_runs + k at SITE_AIS_CLAMPED, t = 2 j for the initial state of layer j and t = 2 j + 1 for its transition draws,
tick = s k + sweep as in the depth ladder.
"""
import numpy as np

import dbm_ais_depth_oracle as A
from oracle import philox as P
from oracle.dbm_bf16 import _r, softplus_diff
from oracle.rbm import sigmoid

SITE_AIS_CLAMPED = 15            # csrc/bm_rng.cuh
LOG2 = float(np.log(2.))


def log_p_star(prm, X, x, beta=1.0):
    """log p*_beta(x; v) of the even-layer states x[j] (j >= 2) with x_0 = X (rows aligned), float64"""
    Ws, bs = A.unit_layers(prm)
    L = len(Ws)
    x = dict(x)
    x[0] = np.asarray(X, np.float64)
    out = beta * (x[0] @ bs[0])
    for j in range(2, L + 1, 2):
        out = out + beta * (x[j] @ bs[j])
    for j in range(1, L + 1, 2):
        out = out + A.softplus(beta * (A.z_raw(Ws, x, j) + bs[j])).sum(axis=1)
    return out


def enumerated_log_p_v(prm, X):
    """log p*(v) of each row of X by enumerating the even layers (the odd layers summed out), float64"""
    w = A.widths(prm)
    L = len(w) - 1
    even = list(range(2, L + 1, 2))
    X = np.asarray(X, np.float64)
    out = []
    for v in X:
        if even:
            grids = np.meshgrid(*[np.arange(2 ** w[j]) for j in even], indexing='ij')
            x = {j: A.states(w[j])[g.ravel()] for j, g in zip(even, grids)}
            n = len(x[even[0]])
        else:
            x, n = {}, 1
        out.append(float(np.logaddexp.reduce(log_p_star(prm, np.repeat(v[None, :], n, axis=0), x))))
    return np.array(out)


def ais(prm, X, n_runs, n_betas, k, seed, row0=0, bf16=False, beta_dtype=np.float32):
    """[rows, n_runs]: each run's estimate of log p*(v_r) (log Z_0 and b_v.v included) for rows row0.. of the caller's data"""
    Ws, bs = A.unit_layers(prm, bf16)
    L = len(Ws)
    w = A.widths(prm)
    X = np.asarray(X, np.float32)
    rows = X.shape[0]
    N = rows * int(n_runs)
    first = int(row0) * int(n_runs)
    bvx = X.astype(np.float64) @ np.asarray(prm['vb'], np.float32).astype(np.float64)
    if L == 1:                                     # nothing to anneal: the closed form
        z = (_r(X) if bf16 else X).astype(np.float64) @ Ws[0].astype(np.float64) + bs[1].astype(np.float64)
        return np.repeat((bvx + A.softplus(z).sum(axis=1))[:, None], int(n_runs), axis=1)
    dt = np.float32 if bf16 else np.float64
    t = A.temperatures(n_betas, beta_dtype)
    nT = len(t)
    inc = lambda s: (0.0 if s == 0 else t[s - 1], 1.0 if s == nT - 1 else t[s])
    summed, state = list(range(1, L + 1, 2)), list(range(2, L + 1, 2))

    def increment(x, a, b):
        out = np.zeros(N)
        for j in summed:
            z = (A.z_raw(Ws, x, j) + bs[j]).astype(dt)
            if bf16:
                out += softplus_diff(a, b, z).astype(np.float64).sum(axis=1)
            else:
                a64, b64 = float(a), float(b)
                out += np.log1p(sigmoid(a64 * z) * np.expm1((b64 - a64) * z)).sum(axis=1)
        return out

    def prob(pre):
        with np.errstate(over='ignore'):
            return (dt(1) / (dt(1) + np.exp(-pre))).astype(dt)

    def draw(p, j, tick):
        u = P.uniform_at(N, p.shape[1], seed, SITE_AIS_CLAMPED, 2 * j + 1, tick, first)
        return (u.astype(dt) < p).astype(dt)

    x = [None] * (L + 1)
    x[0] = np.repeat((_r(X) if bf16 else X.astype(np.float64)), int(n_runs), axis=0).astype(dt)
    for j in state:
        x[j] = (P.uniform_at(N, w[j], seed, SITE_AIS_CLAMPED, 2 * j, 0, first) < np.float32(0.5)).astype(dt)
    logw = np.zeros(N)
    for s in range(nT):
        beta = dt(t[s])
        for sw in range(int(k)):
            tick = s * int(k) + sw
            if sw == 0 and s >= 1:
                logw += increment(x, *inc(s - 1))
            for j in summed:
                x[j] = draw(prob((beta * (A.z_raw(Ws, x, j) + bs[j]).astype(dt)).astype(dt)), j, tick)
            for j in state:
                x[j] = draw(prob((beta * A.z_raw(Ws, x, j).astype(dt) + beta * bs[j]).astype(dt)), j, tick)
            if sw == int(k) - 1:
                a, b = inc(s)
                for j in state:
                    logw += (float(b) - float(a)) * (x[j].astype(np.float64) @ bs[j].astype(np.float64))
    logw += increment(x, *inc(nT - 1))
    out = logw + sum(w[1:]) * LOG2 + np.repeat(bvx, int(n_runs))
    return out.reshape(rows, int(n_runs))


def log_mean_rows(runs):
    """each row's log-mean-exp over its runs"""
    m = runs.max(axis=1, keepdims=True)
    return m[:, 0] + np.log(np.mean(np.exp(runs - m), axis=1))
