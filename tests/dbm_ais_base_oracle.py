"""AIS log Z of binary DBMs from a base-rate model (DESIGN.md §5.4d) restated -- TEST INFRASTRUCTURE ONLY.

Unit layers j = 0..L as in dbm_ais_depth_oracle.py (j = 0 is v).  The base model p_A(x) ∝ exp(sum_j a_j.x_j) is factorial over
every unit layer; a_j = 0 is the uniform base of §5.4c.  The path is p_beta ∝ p_A^(1 - beta) p_B^beta: every weight scaled by
beta, layer j's bias beta b_j + (1 - beta) a_j.  With u_j = (b_j - a_j) + x_{j-1} W_{j-1} + x_{j+1} W_j^T,

    log p*_beta(x) = sum_{odd j} (beta (b_j - a_j) + a_j).x_j + sum_{even j} sum_n softplus(beta u_{j,n} + a_{j,n}),

every layer is drawn from sigmoid(beta u_j + a_j), the initial states from sigmoid(a_j), and log Z_A = sum_j sum_n softplus(a_j,n)
replaces (V + sum H) log 2.  Temperatures, sweeps and Philox sites are those of dbm_ais_depth_oracle.ais.

`ais` states one ladder in float64 (bf16=False) and in the tensor-core engine's arithmetic (bf16=True: bf16 weights, fp32
u = z_raw + (b - a) with b - a rounded to float32 as the engine uploads it, increments log1p(sigmoid(a' u + a) expm1((b' - a') u))
in float32 summed in float64).
"""
import numpy as np

import dbm_ais_depth_oracle as A
from oracle import philox as P
from oracle.dbm_bf16 import _r
from oracle.rbm import sigmoid


def full_base(prm, base, dtype=np.float64):
    """one vector per unit layer: the base as float32 values (what the engine reads), zeros where it is None"""
    w = A.widths(prm)
    if base is None:
        base = [None] * len(w)
    assert len(base) == len(w)
    return [np.zeros(w[j], dtype) if a is None else np.asarray(a, np.float32).reshape(w[j]).astype(dtype)
            for j, a in enumerate(base)]


def has_base(base):
    return base is not None and any(a is not None for a in base)


def log_Z_A(prm, base):
    """log Z of the base model in float64; without a base the engine's (V + sum H) * float32(log 2)"""
    if not has_base(base):
        return sum(A.widths(prm)) * A.LOG2_F32
    return float(sum(A.softplus(a).sum() for a in full_base(prm, base)))


def log_p_star(prm, x, beta, base):
    """the marginalised log p*_beta of the odd-layer states x[j] on the path from the base, float64"""
    Ws, bs = A.unit_layers(prm)
    a = full_base(prm, base)
    L = len(Ws)
    out = 0.
    for j in range(1, L + 1, 2):
        out = out + x[j] @ (beta * (bs[j] - a[j]) + a[j])
    for j in range(0, L + 1, 2):
        out = out + A.softplus(beta * (A.z_raw(Ws, x, j) + bs[j] - a[j]) + a[j]).sum(axis=1)
    return out


def path_model(prm, beta, base):
    """the parameters of p_beta as a DBM: weights beta W, biases beta b + (1 - beta) a"""
    Ws, bs = A.unit_layers(prm)
    a = full_base(prm, base)
    out = {'vb': beta * bs[0] + (1. - beta) * a[0]}
    for i, W in enumerate(Ws):
        out['W' + A.sfx(i)] = beta * W
        out['hb' + A.sfx(i)] = beta * bs[i + 1] + (1. - beta) * a[i + 1]
    return out


def softplus_diff_base(a, b, u, a0):
    """softplus(b u + a0) - softplus(a u + a0) in float32 (the kernel's closed form with a base)"""
    a, b = np.float32(a), np.float32(b)
    u = np.asarray(u, np.float32)
    with np.errstate(over='ignore'):
        s = np.float32(1.) / (np.float32(1.) + np.exp(-(a * u + a0)))
    return np.log1p(s * np.expm1((b - a) * u))


def ais(prm, n_runs, n_betas, k, seed, base=None, first_run=0, bf16=False, sample_v=True, sample_h=None,
        beta_dtype=np.float32, return_logw=False):
    """log Z estimates of runs [first_run, first_run + n_runs) of the ladder from the base (log Z_A included); with
    return_logw also the log-weights without it"""
    Ws, bs = A.unit_layers(prm, bf16)
    L = len(Ws)
    w = A.widths(prm)
    dt = np.float32 if bf16 else np.float64
    a = full_base(prm, base, np.float32 if bf16 else np.float64)
    d = [(bs[j] - a[j]).astype(dt) for j in range(L + 1)]
    sampled = [bool(sample_v)] + [bool(s) for s in (sample_h if sample_h is not None else [True] * L)]
    assert all(sampled[1::2]), 'the state layers are sampled'
    t = A.temperatures(n_betas, beta_dtype)
    nT = len(t)
    inc = lambda s: (0.0 if s == 0 else t[s - 1], 1.0 if s == nT - 1 else t[s])

    def increment(x, lo, hi):
        out = np.zeros(n_runs)
        for j in range(0, L + 1, 2):
            u = (A.z_raw(Ws, x, j) + d[j]).astype(dt)
            if bf16:
                out += softplus_diff_base(lo, hi, u, a[j]).astype(np.float64).sum(axis=1)
            else:
                lo64, hi64 = float(lo), float(hi)
                out += np.log1p(sigmoid(lo64 * u + a[j]) * np.expm1((hi64 - lo64) * u)).sum(axis=1)
        return out

    def draw(p, j, tick):
        st, gi = A.site(j)
        u = P.uniform_at(n_runs, p.shape[1], seed, st, gi, tick, first_run)
        return (u.astype(dt) < p).astype(dt)

    def prob(pre):
        with np.errstate(over='ignore'):
            return (dt(1) / (dt(1) + np.exp(-pre))).astype(dt)

    x = [None] * (L + 1)
    for j in range(1, L + 1, 2):
        p0 = (np.float32(1) / (np.float32(1) + np.exp(-a[j].astype(np.float32)))).astype(np.float32)
        x[j] = (P.uniform_at(n_runs, w[j], seed, P.SITE_AIS_INIT, (j - 1) // 2, 0, first_run) < p0).astype(dt)
    logw = np.zeros(n_runs)
    for s in range(nT):
        beta = dt(t[s])
        for sw in range(int(k)):
            tick = s * int(k) + sw
            if sw == 0 and s >= 1:
                logw += increment(x, *inc(s - 1))
            for j in range(0, L + 1, 2):
                u = (A.z_raw(Ws, x, j) + d[j]).astype(dt)
                p = prob((beta * u + a[j]).astype(dt))
                x[j] = draw(p, j, tick) if sampled[j] else (_r(p) if bf16 else p)
            for j in range(1, L + 1, 2):
                x[j] = draw(prob((beta * A.z_raw(Ws, x, j).astype(dt) + beta * d[j] + a[j]).astype(dt)), j, tick)
            if sw == int(k) - 1:
                lo, hi = inc(s)
                for j in range(1, L + 1, 2):
                    logw += (float(hi) - float(lo)) * (x[j].astype(np.float64) @ d[j].astype(np.float64))
    logw += increment(x, *inc(nT - 1))
    out = logw + log_Z_A(prm, base)
    return (out, logw) if return_logw else out


def data_base(X):
    """DBM.log_Z(base_rate=X): the visible base logit((sum_r X_r + 1) / (n + 2)) as float32, hidden layers uniform"""
    X = np.asarray(X, np.float64)
    p = (X.sum(axis=0) + 1.) / (X.shape[0] + 2.)
    return np.log(p / (1. - p)).astype(np.float32)
