"""Conditional sampling with clamped Gibbs chains (DESIGN.md §5.9, include/bm.h bm_dbm_fill) restated -- TEST INFRASTRUCTURE
ONLY.

`fill` states one call in two arithmetics on the oracles' models:
  * bf16=False: in the model's dtype with the oracle's own conditionals (oracle.dbm.OracleDBM._act and its Philox draws, keyed
    by the row row0 + r), the float64 statement and, for a float32 OracleDBM, what the CUDA-core engine computes;
  * bf16=True: the bf16 emulation of the tensor-core engine (oracle/dbm_bf16.py, tests/dbm_bf16_multinomial.py): bf16 weight
    operands, fp32 pre-activations, means stored as bf16, draws compared against the fp32 mean.
The semantics, for every row r:
  1. v0 = X where observed, act(0 W_0' + b) (sigmoid(b), or b for Gaussian units) where missing;
  2. h0 = the mean-field E-step's approximate-inference pass on v0 (inputs doubled below the top layer); a labelled row of a
     classification DBM starts at its one-hot label;
  3. sweeps t = 1..k: h_1 .. h_L bottom-up (each reading the layer above from the previous sweep), the label reset to e_y on
     labelled rows, then v from the new h_1 and v <- X where observed; draws at (SITE_DBM_H + i | SITE_DBM_V, t, seed, tick,
     row0 + r), sampled as the model's sample_v / sample_h say;
  4. out = the visible means p(v | h_1 of sweep k), X where observed.
`clamp_v=False` / `clamp_y=False` switch off the visible / label clamp in the sweeps: the negative controls of the statistical
tests.  `FillOracleDBM` / `FillClassDBM64` carry `fill` as an engine method, so the Python classes can run on them
(set_engine_factory('dbm', factory)).
"""
import importlib.util
import os

import numpy as np

from oracle import philox as P
from oracle.dbm import OracleDBM
from oracle.dbm_bf16 import _r
from oracle.rbm import sigmoid, multinomial_counts

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_cdbm = _load('class_dbm_oracle')
_mult = _load('dbm_bf16_multinomial')
softmax_rows = _mult.softmax_rows


def _label_layer(o):
    """the engine's index of a classification DBM's label layer, None for a plain DBM"""
    return getattr(o, 'Lm', None) if hasattr(o, 'C') else None


def _one_hot_rows(m, labels):
    if labels is None:
        return m
    m = m.copy()
    rows = np.nonzero(labels >= 0)[0]
    m[rows] = 0.
    m[rows, labels[rows]] = 1.
    return m


def fill(o, X, mask, labels=None, row0=0, k=1, seed=0, tick=0, bf16=False, clamp_v=True, clamp_y=True):
    """One call on rows row0 .. row0 + rows - 1.  Returns (out, states) with states the chain's last two sweeps:
    'v', 'v_prev', 'h', 'h_prev', 'h_1', ... (the label layer: 'y', 'y_prev') and 'mean'."""
    L, Hs, V = o.L, o.Hs, o.V
    rows = X.shape[0]
    dt = np.dtype(np.float32) if bf16 else o.dt
    f = dt.type
    sh = [bool(s) for s in o.cfg.get('sample_h', [True] * L)]
    sv = bool(o.cfg.get('sample_v', True))
    top = _label_layer(o)
    lab = None if labels is None else np.asarray(labels, dtype=np.int64)
    Wf = [(_r(o.W(i)) if bf16 else o.W(i)) for i in range(L)]
    mask = np.asarray(mask).astype(bool)
    Xc = _r(X) if bf16 else np.asarray(X, dtype=dt)

    def draws(fn, n, site, t):
        return fn(rows, n, seed, site, t, tick, row0)

    def hidden(i, below, above, acc, sample, t):
        kind, ns = o.h_kinds[i], o.h_n_samples[i]
        T = below @ Wf[i]
        if above is not None:
            T = T + above @ Wf[i + 1].T
        site = P.SITE_DBM_H + i
        if bf16:
            pre = (np.float32(acc) * T + np.float32(1.) * o.hb(i)).astype(np.float32)
            if kind == 'bernoulli':
                m = sigmoid(pre)
                return (draws(P.uniform_at, Hs[i], site, t) < m).astype(np.float32) if sample else _r(m)
            m = softmax_rows(pre, ns)
            if sample:
                m64 = m.astype(np.float64)
                probs = (m64 / np.cumsum(m64, axis=1)[:, -1:]).astype(np.float32)
                m = multinomial_counts(probs, int(ns), seed, site, t, tick, row0).astype(np.float32)
            return _r(m)
        if acc != 1.:
            T = f(acc) * T
        m = o._act(kind, T, o.hb(i), ns)
        if not sample:
            return m
        if kind == 'bernoulli':
            return (draws(P.uniform_at, Hs[i], site, t).astype(dt) < m).astype(dt)
        probs = (m / m.sum(axis=1, keepdims=True)).astype(np.float32)
        return multinomial_counts(probs, int(ns), seed, site, t, tick, row0).astype(dt)

    def visible(h0, sample, t):
        if bf16:
            T = (h0 @ Wf[0].T).astype(np.float32)
            if o.v_kind == 'bernoulli':
                m = sigmoid(T + o.p['vb'])
                return (draws(P.uniform_at, V, P.SITE_DBM_V, t) < m).astype(np.float32) if sample else _r(m)
            m = (T * o.sigma + o.p['vb']).astype(np.float32)
            if sample:
                m = m + o.sigma * draws(P.normal_at, V, P.SITE_DBM_V, t).astype(np.float32)
            return _r(m)
        m = o._act(o.v_kind, h0 @ Wf[0].T, o.p['vb'])
        if not sample:
            return m
        if o.v_kind == 'bernoulli':
            return (draws(P.uniform_at, V, P.SITE_DBM_V, t).astype(dt) < m).astype(dt)
        return (m + o.sigma * draws(P.normal_at, V, P.SITE_DBM_V, t).astype(dt)).astype(dt)

    v = np.where(mask, Xc, visible(np.zeros((rows, Hs[0]), dtype=dt), False, 0)).astype(dt)
    H = []
    for i in range(L):
        H.append(hidden(i, v if i == 0 else H[i - 1], None, 2. if (i == 0 or i < L - 1) else 1., False, 0))
        if i == top:
            H[i] = _one_hot_rows(H[i], lab)
    v_prev, H_prev = v, H
    for t in range(1, int(k) + 1):
        Hn = []
        for i in range(L):
            Hn.append(hidden(i, v if i == 0 else Hn[i - 1], H[i + 1] if i + 1 < L else None, 1., sh[i], t))
            if i == top and clamp_y:
                Hn[i] = _one_hot_rows(Hn[i], lab)
        vn = visible(Hn[0], sv, t)
        if clamp_v:
            vn = np.where(mask, Xc, vn).astype(dt)
        v_prev, H_prev, v, H = v, H, vn, Hn
    mean = visible(H[0], False, 0)
    out = np.where(mask, np.asarray(X, dtype=dt), mean).astype(dt)
    states = {'v': v, 'v_prev': v_prev, 'mean': mean}
    for i in range(L):
        name = 'y' if i == top else 'h' + ('' if i == 0 else '_%d' % i)
        states[name], states[name + '_prev'] = H[i], H_prev[i]
    return out, states


class _Fill(object):
    bf16 = False

    def fill(self, X, mask, labels=None, row0=0, k=1, seed=0, tick=0):
        X = np.asarray(X, dtype=self.dt)
        return fill(self, X, mask, labels, row0, k, seed, tick, bf16=self.bf16)[0]


class FillOracleDBM(_Fill, OracleDBM):
    pass


class FillClassDBM64(_Fill, _cdbm.ClassDBM64):
    pass


def factory(cfg):
    """the float statement as the engine of DBM / ClassificationDBM (set_engine_factory('dbm', factory))"""
    return FillClassDBM64(cfg) if cfg.get('n_classes') else FillOracleDBM(cfg)


# ---- exact conditionals of models small enough to enumerate ---------------------------------------------------------------
def states(n):
    return ((np.arange(2 ** n)[:, None] >> np.arange(n)) & 1).astype(np.float64)


def exact_log_p_v(d, Hs):
    """log p(v) [2^V] of a binary DBM with 1 or 2 hidden layers (h_1 enumerated for 2, the top layer summed out)"""
    V = d['vb'].shape[0]
    vs = states(V)
    sp = lambda z: np.logaddexp(0., z)
    W0, c0 = d['W'].astype(np.float64), d['hb'].astype(np.float64)
    if len(Hs) == 1:
        lp = vs @ d['vb'] + sp(vs @ W0 + c0).sum(1)
    else:
        W1, c1 = d['W_1'].astype(np.float64), d['hb_1'].astype(np.float64)
        h1 = states(Hs[0])
        e = (vs @ d['vb'])[:, None] + (vs @ W0) @ h1.T + (h1 @ c0)[None, :] + sp(h1 @ W1 + c1).sum(1)[None, :]
        lp = np.logaddexp.reduce(e, axis=1)
    return lp - np.logaddexp.reduce(lp)


def conditional_table(log_p_v, V, obs_idx, x_obs):
    """p(v_missing | v_obs = x_obs) over the 2^(V - |obs|) patterns of the missing units, indexed by sum_j v_miss[j] 2^j"""
    vs = states(V)
    miss = [j for j in range(V) if j not in obs_idx]
    keep = np.all(vs[:, obs_idx] == np.asarray(x_obs)[None, :], axis=1)
    lp = log_p_v[keep]
    idx = (vs[keep][:, miss] @ (2 ** np.arange(len(miss)))).astype(np.int64)
    p = np.zeros(2 ** len(miss))
    p[idx] = np.exp(lp - np.logaddexp.reduce(lp))
    return p


def chi2_per_dof(counts, p, min_expected=5.):
    """Pearson chi-square per degree of freedom of `counts` against probabilities `p`, cells expecting < 5 pooled"""
    n = counts.sum()
    ex = n * p
    keep = ex >= min_expected
    obs, e = np.append(counts[keep], counts[~keep].sum()), np.append(ex[keep], ex[~keep].sum())
    if e[-1] < min_expected:
        obs, e = obs[:-1], e[:-1]
    return float(((obs - e) ** 2 / e).sum() / max(len(e) - 1, 1))
