"""AIS log Z and the variational bound of binary DBMs of any depth (DESIGN.md §5.4c) restated -- TEST INFRASTRUCTURE ONLY.

Unit layer j = 0..L is v (j = 0) or h_j, with weights W_j between layers j and j + 1 (the model's 'W', 'W_1', ...) and biases
b_0 = vb, b_j = hb of h_j.  The odd layers are the state x of the chains; v and the even layers are summed out:

    log p*_beta(x) = beta sum_{odd j} b_j.x_j + sum_{even j} sum_n softplus(beta z_{j,n}),
    z_j = b_j + x_{j-1} W_{j-1} + x_{j+1} W_j^T        (no first term for v, no second for h_L).

`ais` states one ladder in two arithmetics:
  * bf16=False: float64 throughout (the statement);
  * bf16=True: the tensor-core engine's arithmetic (DbmTC::ais_local_layers): bf16 weight operands, fp32 pre-activations,
    increments softplus(b z) - softplus(a z) = log1p(sigmoid(a z) expm1((b - a) z)) in float32 summed in float64, means of
    unsampled layers stored as bf16, draws against the fp32 probability.
Both follow the engine's arrangement: temperatures t_0 = 1/n_betas, t_{s+1} = t_s + 1/n_betas accumulated in float32 (or in
`beta_dtype`) while t_s < 1 - 1/n_betas + 1e-5; transition s runs k sweeps at t_s, each drawing every summed-out layer from
sigmoid(t_s z_j) given the state and then every state layer from sigmoid(t_s z_j) given the summed-out layers; the increment
log p*_b(x) - log p*_a(x) of the state transition s produced is weighed with (a, b) = (t_{s-1} or 0, t_s or 1 for the last).
Draws: v at SITE_AIS_V, hidden layer i = j - 1 at SITE_AIS_H1 (i even) or SITE_AIS_H2 (i odd) with Gibbs index i // 2, the
initial state x_0 ~ Ber(1/2) of layer i at SITE_AIS_INIT with the same index; tick = s k + sweep, row = first_run + r.  At
L = 2 these are the reference's ladder and sites (oracle/dbm.py).

`bound` is dbm.py:743-757 for L layers on the E-step's means: sum_i t_i.mu_i + X.b_v + sum_i mu_i.c_i + sum_i H(clip(mu_i)),
t_i = mu_{i-1} W_i (X W_0 for i = 0), in float64 or on the bf16 emulation's E-step with fp32 products.
"""
import itertools

import numpy as np

from oracle import philox as P
from oracle.dbm import OracleDBM
from oracle.dbm_bf16 import OracleDBMbf16, _r, softplus_diff
from oracle.rbm import sigmoid

LOG2_F32 = float(np.float32(np.log(2.)))


def sfx(i):
    return '' if i == 0 else '_%d' % i


def n_layers(prm):
    return sum(1 for k in prm if k.startswith('W') and not k.startswith('dW'))


def unit_layers(prm, bf16=False):
    """(weights W_0..W_{L-1}, biases b_0..b_L) as the arithmetic reads them"""
    L = n_layers(prm)
    if bf16:
        Ws = [_r(prm['W' + sfx(i)]) for i in range(L)]
        bs = [np.asarray(prm['vb'], np.float32)] + [np.asarray(prm['hb' + sfx(i)], np.float32) for i in range(L)]
    else:
        Ws = [np.asarray(prm['W' + sfx(i)], np.float64) for i in range(L)]
        bs = [np.asarray(prm['vb'], np.float64)] + [np.asarray(prm['hb' + sfx(i)], np.float64) for i in range(L)]
    return Ws, bs


def widths(prm):
    L = n_layers(prm)
    return [prm['W'].shape[0]] + [prm['W' + sfx(i)].shape[1] for i in range(L)]


def z_raw(Ws, x, j):
    """x_{j-1} W_{j-1} + x_{j+1} W_j^T from the layers next to j (without the bias)"""
    L = len(Ws)
    acc = None
    if j >= 1:
        acc = x[j - 1] @ Ws[j - 1]
    if j + 1 <= L:
        up = x[j + 1] @ Ws[j].T
        acc = up if acc is None else acc + up
    return acc


def softplus(z):
    return np.logaddexp(0.0, z)


def log_p_star(prm, x, beta=1.0):
    """the marginalised log p*_beta of the states x[j] (odd j), float64"""
    Ws, bs = unit_layers(prm)
    L = len(Ws)
    out = 0.
    for j in range(1, L + 1, 2):
        out = out + beta * (x[j] @ bs[j])
    for j in range(0, L + 1, 2):
        out = out + softplus(beta * (z_raw(Ws, x, j) + bs[j])).sum(axis=1)
    return out


def states(n):
    return ((np.arange(2 ** n)[:, None] >> np.arange(n)[None, :]) & 1).astype(np.float64)


def exact_log_Z(prm):
    """log Z by enumerating the state layers (the summed-out layers marginalised analytically)"""
    w = widths(prm)
    L = len(w) - 1
    odd = list(range(1, L + 1, 2))
    grids = np.meshgrid(*[np.arange(2 ** w[j]) for j in odd], indexing='ij')
    x = {}
    for j, g in zip(odd, grids):
        x[j] = states(w[j])[g.ravel()]
    return float(np.logaddexp.reduce(log_p_star(prm, x)))


def brute_log_Z(prm):
    """log Z by enumerating every unit of a tiny model"""
    Ws, bs = unit_layers(prm)
    w = widths(prm)
    cfgs = np.array(list(itertools.product((0., 1.), repeat=sum(w))))
    cut = np.cumsum([0] + w)
    xs = [cfgs[:, cut[j]:cut[j + 1]] for j in range(len(w))]
    e = sum(xs[j] @ bs[j] for j in range(len(w))) + sum(((xs[i] @ Ws[i]) * xs[i + 1]).sum(axis=1) for i in range(len(Ws)))
    return float(np.logaddexp.reduce(e))


def brute_log_p_v(prm, X):
    """exact log p*(v) (without -log Z) by enumerating the hidden units"""
    Ws, bs = unit_layers(prm)
    w = widths(prm)
    cfgs = np.array(list(itertools.product((0., 1.), repeat=sum(w[1:]))))
    cut = np.cumsum([0] + w[1:])
    hs = [cfgs[:, cut[j]:cut[j + 1]] for j in range(len(w) - 1)]
    e_h = sum(hs[j] @ bs[j + 1] for j in range(len(hs)))
    e_h = e_h + sum(((hs[i] @ Ws[i + 1]) * hs[i + 1]).sum(axis=1) for i in range(len(hs) - 1))
    X = np.asarray(X, np.float64)
    out = X @ bs[0] + np.logaddexp.reduce((X @ Ws[0]) @ hs[0].T + e_h[None, :], axis=1)
    return out


def temperatures(n_betas, dtype=np.float32):
    d = dtype(1. / n_betas)
    t = [d]
    while t[-1] < dtype(1.) - d + dtype(1e-5):
        t.append(dtype(t[-1] + d))
    return t


def site(j):
    """(site, Gibbs index) of unit layer j"""
    if j == 0:
        return P.SITE_AIS_V, 0
    i = j - 1
    return (P.SITE_AIS_H1 if i % 2 == 0 else P.SITE_AIS_H2), i // 2


def ais(prm, n_runs, n_betas, k, seed, first_run=0, bf16=False, sample_v=True, sample_h=None, beta_dtype=np.float32):
    """log Z estimates of runs [first_run, first_run + n_runs) of the ladder"""
    Ws, bs = unit_layers(prm, bf16)
    L = len(Ws)
    w = widths(prm)
    dt = np.float32 if bf16 else np.float64
    sampled = [bool(sample_v)] + [bool(s) for s in (sample_h if sample_h is not None else [True] * L)]
    assert all(sampled[1::2]), 'the state layers are sampled'
    t = temperatures(n_betas, beta_dtype)
    nT = len(t)
    inc = lambda s: (0.0 if s == 0 else t[s - 1], 1.0 if s == nT - 1 else t[s])

    def increment(x, a, b):
        out = np.zeros(n_runs)
        for j in range(0, L + 1, 2):
            z = (z_raw(Ws, x, j) + bs[j]).astype(dt)
            if bf16:
                out += softplus_diff(a, b, z).astype(np.float64).sum(axis=1)
            else:
                a64, b64 = float(a), float(b)
                out += np.log1p(sigmoid(a64 * z) * np.expm1((b64 - a64) * z)).sum(axis=1)
        return out

    def draw(p, j, tick):
        st, gi = site(j)
        u = P.uniform_at(n_runs, p.shape[1], seed, st, gi, tick, first_run)
        return (u.astype(dt) < p).astype(dt)

    x = [None] * (L + 1)
    for j in range(1, L + 1, 2):
        st, gi = P.SITE_AIS_INIT, (j - 1) // 2
        x[j] = (P.uniform_at(n_runs, w[j], seed, st, gi, 0, first_run) < np.float32(0.5)).astype(dt)
    logw = np.zeros(n_runs)
    for s in range(nT):
        beta = dt(t[s])
        for sw in range(int(k)):
            tick = s * int(k) + sw
            if sw == 0 and s >= 1:
                logw += increment(x, *inc(s - 1))
            for j in range(0, L + 1, 2):
                z = (z_raw(Ws, x, j) + bs[j]).astype(dt)
                with np.errstate(over='ignore'):
                    p = (dt(1) / (dt(1) + np.exp(-(beta * z)))).astype(dt)
                x[j] = draw(p, j, tick) if sampled[j] else (_r(p) if bf16 else p)
            for j in range(1, L + 1, 2):
                pre = (beta * z_raw(Ws, x, j).astype(dt) + beta * bs[j]).astype(dt)
                with np.errstate(over='ignore'):
                    p = (dt(1) / (dt(1) + np.exp(-pre))).astype(dt)
                x[j] = draw(p, j, tick)
            if sw == int(k) - 1:
                a, b = inc(s)
                for j in range(1, L + 1, 2):
                    logw += (float(b) - float(a)) * (x[j].astype(np.float64) @ bs[j].astype(np.float64))
    logw += increment(x, *inc(nT - 1))
    return logw + sum(w) * LOG2_F32


def bound(cfg, prm, X, bf16=False):
    """the per-row variational bound (without -log Z) on the E-step's means, float64 sums"""
    o = (OracleDBMbf16 if bf16 else OracleDBM)(dict(cfg, dtype='float32' if bf16 else 'float64'))
    o.set_params({k: np.asarray(v, np.float32 if bf16 else np.float64) for k, v in prm.items()})
    X = np.asarray(X, np.float32 if bf16 else np.float64)
    rows = X.shape[0]
    o.mean_field(X)
    L = o.L
    mu = [o.p['mu' + sfx(i)][:rows] for i in range(L)]
    Ws, bs = unit_layers(prm, bf16)
    out = X.astype(np.float64) @ bs[0].astype(np.float64)
    for i in range(L):
        below = (_r(X) if bf16 else X) if i == 0 else mu[i - 1]
        t = (below @ Ws[i]).astype(np.float32 if bf16 else np.float64).astype(np.float64)
        m = mu[i].astype(np.float64)
        out = out + (t * m).sum(axis=1) + m @ bs[i + 1].astype(np.float64)
        s = np.clip(mu[i].astype(np.float32), np.float32(1e-7), np.float32(1. - 1e-7)).astype(np.float64) if bf16 else \
            np.clip(m, 1e-7, 1. - 1e-7)
        out = out + (-s * np.log(s) - (1. - s) * np.log(1. - s)).sum(axis=1)
    return out, [m.astype(np.float64) for m in mu]


def bound_given_mu(prm, X, mu, bf16_weights=True):
    """the bound in float64 on given means (the engine's own E-step, read back with get_params), with the weights the engine
    reads (bf16_weights) or the model's"""
    Ws, bs = unit_layers(prm)
    if bf16_weights:
        Ws = [_r(W).astype(np.float64) for W in Ws]
    X = np.asarray(X, np.float64)
    out = X @ bs[0]
    for i, m in enumerate(mu):
        m = np.asarray(m, np.float64)
        below = X if i == 0 else np.asarray(mu[i - 1], np.float64)
        out = out + ((below @ Ws[i]) * m).sum(axis=1) + m @ bs[i + 1]
        s = np.clip(m, 1e-7, 1. - 1e-7)
        out = out + (-s * np.log(s) - (1. - s) * np.log(1. - s)).sum(axis=1)
    return out
