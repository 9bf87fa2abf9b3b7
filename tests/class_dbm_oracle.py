"""The classification DBM (DESIGN.md §5.7, include/bm.h bm_dbm_cfg.n_classes) restated twice: in float64 on
oracle.dbm.OracleDBM (ClassDBM64, the statement of the model) and on the bf16 emulation of the tensor-core DBM engine
(oracle/dbm_bf16.py, tests/dbm_bf16_multinomial.py; ClassDBMbf16, what the engine computes op for op).

The model x - h_1 - ... - h_L - y is the plain DBM with L + 1 hidden layers whose top layer is multinomial (n_samples 1,
sampled, no sparsity term) and whose last weight is W_{L+1} = U^T.  What the label adds:
  - in the mean-field E-step a row labelled t >= 0 holds the one-hot e_t in the label slot, before the first test and after
    every update (so its change is 0); a row labelled -1 updates it like any multinomial layer;
  - yb takes the plain momentum update from sum q(y) / rows - sum y / M, without a sparsity term;
  - predict_proba = softmax(yb + mu_L U^T) in fp32 from the E-step's final mu_L (y free), by the row kernel's arithmetic.
Names are the engine's: U [C, H_L], yb, dU, dyb, y [M, C], mu_y [B, C]; the other names are the plain DBM's.

ClassDBM64 also takes a `mutation` (for the tests that show the checks can fail): 'no_yb' draws the label particles without
yb, 'below' makes them read h_{L-1} (its first H_L units) instead of h_L.
"""
import importlib.util
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_mult = _load('dbm_bf16_multinomial')
from oracle.dbm import OracleDBM  # noqa: E402
Base = _mult.OracleDBMbf16Multinomial
softmax_rows = _mult.softmax_rows


def sfx(i):
    return '' if i == 0 else '_%d' % i


def plain_cfg(cfg):
    """The engine's DBM underneath: the label as hidden layer L + 1 (multinomial, n_samples 1, sampled, sparsity cost 0)."""
    c = dict(cfg)
    C, L = int(c.pop('n_classes')), len(cfg['n_hiddens'])
    c['n_hiddens'] = list(cfg['n_hiddens']) + [C]
    c['h_kinds'] = list(cfg.get('h_kinds', ['bernoulli'] * L)) + ['multinomial']
    c['h_n_samples'] = list(cfg.get('h_n_samples', [100.] * L)) + [1.]
    c['sample_h'] = list(cfg.get('sample_h', [True] * L)) + [True]
    c['sparsity_target'] = list(cfg.get('sparsity_target', [0.1] * L)) + [0.]
    c['sparsity_cost'] = list(cfg.get('sparsity_cost', [0.] * L)) + [0.]
    return c


def to_plain(d, L):
    """classification names -> the plain DBM's names of the label layer"""
    out = {}
    for k, v in d.items():
        k2 = {'U': 'W', 'dU': 'dW', 'yb': 'hb', 'dyb': 'dhb', 'y': 'h', 'mu_y': 'mu'}.get(k)
        if k2 is None:
            out[k] = v
        else:
            out[k2 + sfx(L)] = np.ascontiguousarray(np.asarray(v).T) if k in ('U', 'dU') else v
    return out


def from_plain(d, L):
    out = {}
    for k, v in d.items():
        for stem, name in (('W', 'U'), ('dW', 'dU'), ('hb', 'yb'), ('dhb', 'dyb'), ('h', 'y'), ('mu', 'mu_y')):
            if k == stem + sfx(L):
                out[name] = np.ascontiguousarray(v.T) if name in ('U', 'dU') else v
                break
        else:
            if not any(k == s + sfx(L) for s in ('q_means', 'mu_means')):
                out[k] = v
    return out


class ClassDBMbf16(Base):
    def __init__(self, cfg):
        self.Lm, self.C = len(cfg['n_hiddens']), int(cfg['n_classes'])
        Base.__init__(self, plain_cfg(cfg))
        self._labels = None                 # [rows] during the E-step of a labelled step

    def set_params(self, d):
        Base.set_params(self, to_plain(d, self.Lm))

    def get_params(self, names=None):
        return from_plain(Base.get_params(self), self.Lm) if names is None else \
            {k: v for k, v in from_plain(Base.get_params(self), self.Lm).items() if k in names}

    def _clamp(self, m):
        if self._labels is None:
            return m
        m = m.copy()
        lab = self._labels[:m.shape[0]]
        rows = np.nonzero(lab >= 0)[0]
        m[rows] = 0.
        m[rows, lab[rows]] = 1.
        return m

    def _hidden(self, i, below, above, sample, seed, site, t, tick, acc_scale=1., bias_scale=1.):
        out = Base._hidden(self, i, below, above, sample, seed, site, t, tick, acc_scale, bias_scale)
        return self._clamp(out) if (i == self.Lm and self._in_mf) else out

    _in_mf = False

    def mean_field(self, X):
        rows = np.asarray(X).shape[0]
        k = 'mu' + sfx(self.Lm)
        self.p[k][:rows] = self._clamp(self.p[k][:rows])
        self._in_mf = True
        try:
            return Base.mean_field(self, X)
        finally:
            self._in_mf = False

    def train_step(self, X, lr, momentum, k, seed, tick, metrics=(), labels=None):
        self._labels = None if labels is None else np.asarray(labels, dtype=np.int64)
        L = self.Lm
        keep = {n + sfx(L): self.p[n + sfx(L)].copy() for n in ('q_means', 'mu_means')}
        try:
            out = Base.train_step(self, X, lr, momentum, k, seed, tick, metrics)
        finally:
            self._labels = None
        for n, v in keep.items():           # the label layer keeps no sparsity statistics
            self.p[n] = v
        return out

    def transform(self, X):
        self.mean_field(X)
        return self.p['mu' + sfx(self.Lm - 1)][:len(X)].copy()

    def predict_proba(self, X):
        self.mean_field(X)
        L = self.Lm
        mu = self.p['mu' + sfx(L - 1)][:len(X)]
        pre = (mu @ self.Wb(L) + self.hb(L)).astype(np.float32)
        return softmax_rows(pre, 1.)


class ClassDBM64(OracleDBM):
    """The float64 statement: OracleDBM with the label as hidden layer L + 1, the clamp in the mean-field E-step, the label
    in the particle sweeps and yb's plain momentum update.  Also an engine for the Python model (``factory``)."""

    def __init__(self, cfg, mutation=None):
        self.Lm, self.C = len(cfg['n_hiddens']), int(cfg['n_classes'])
        c = plain_cfg(cfg)
        c['dtype'] = 'float64'
        OracleDBM.__init__(self, c)
        self.mutation = mutation
        self._labels = None

    def set_params(self, d):
        OracleDBM.set_params(self, to_plain(d, self.Lm))

    def get_params(self, names=None):
        out = from_plain(OracleDBM.get_params(self), self.Lm)
        return out if names is None else {k: out[k] for k in names}

    def _clamp(self, m):
        if self._labels is None:
            return m
        m = m.copy()
        lab = self._labels[:m.shape[0]]
        rows = np.nonzero(lab >= 0)[0]
        m[rows] = 0.
        m[rows, lab[rows]] = 1.
        return m

    def gibbs_step(self, v, H, update_v, sample, seed, t, tick):
        v_new, Hn = OracleDBM.gibbs_step(self, v, H, update_v, sample, seed, t, tick)
        top = self.Lm
        if self.mutation and sample:           # redraw the label particles from the mutated conditional
            hb = self.hb(top) * (0. if self.mutation == 'no_yb' else 1.)
            below = Hn[top - 1] if self.mutation == 'no_yb' else (Hn[top - 2] if top >= 2 else v)[:, :self.Hs[top - 1]]
            m = self._act('multinomial', below @ self.W(top), hb, 1.)
            Hn[top] = self._sample('multinomial', m, 1., seed, P_SITE_DBM_H + top, t, tick)
        if self._in_mf:
            Hn[top] = self._clamp(Hn[top])
        return v_new, Hn

    _in_mf = False

    def mean_field(self, X):
        """OracleDBM.mean_field with the label slot of labelled rows held at e_t (before the first test and after every
        update, so that it never changes)"""
        L = self.L
        X = np.asarray(X, dtype=self.dt)
        rows = X.shape[0]
        k = 'mu' + sfx(self.Lm)
        self.p[k][:rows] = self._clamp(self.p[k][:rows])
        mu = [self.p['mu' + sfx(i)][:rows] for i in range(L)]
        mu_new, T = [], None
        for i in range(L):
            T = 2. * (X @ self.W(0)) if i == 0 else T @ self.W(i) * (2. if i < L - 1 else 1.)
            T = self._act(self.h_kinds[i], T, self.hb(i), self.h_n_samples[i])
            if i == self.Lm:
                T = self._clamp(T)
            mu_new.append(T)
        step, tol = 0, self.cfg.get('mf_tol', 1e-7)
        self._in_mf = True
        try:
            while step < int(self.cfg.get('max_mf_updates', 10)) and \
                    max(np.max(np.abs(a - b)) for a, b in zip(mu, mu_new)) > tol:
                _, Hn = self.gibbs_step(X, mu, update_v=False, sample=False, seed=0, t=0, tick=0)
                mu, mu_new = Hn, mu
                step += 1
        finally:
            self._in_mf = False
        for i in range(L):
            self.p['mu' + sfx(i)][:rows] = mu[i]
        return step

    def train_step(self, X, lr, momentum, k, seed, tick, metrics=(), labels=None):
        """OracleDBM.train_step; the label layer's sparsity cost is 0, so its bias takes the plain momentum update (its
        q_means / mu_means are not variables of the model and are left as they were).  Needs n_classes > n_layers, where
        the reference's element-i quirk of the sparsity statistics finds an element to read."""
        assert self.C > self.Lm, 'the float64 statement needs n_classes > n_layers'
        self._labels = None if labels is None else np.asarray(labels, dtype=np.int64)
        top = self.Lm
        keep = {n + sfx(top): self.p[n + sfx(top)].copy() for n in ('q_means', 'mu_means')}
        try:
            out = OracleDBM.train_step(self, X, lr, momentum, k, seed, tick, metrics)
        finally:
            self._labels = None
        self.p.update(keep)
        return out

    def transform(self, X):
        self.mean_field(X)
        return self.p['mu' + sfx(self.Lm - 1)][:len(X)].copy()

    def predict_proba(self, X):
        X = np.asarray(X, dtype=self.dt)
        self.mean_field(X)
        mu = self.p['mu' + sfx(self.Lm - 1)][:len(X)]
        return self._act('multinomial', mu @ self.W(self.Lm), self.hb(self.Lm), 1.)

    def close(self):
        pass


def factory(cfg):
    """the float64 statement as the engine of boltzmann_machines.ClassificationDBM (set_engine_factory('dbm', factory))"""
    return ClassDBM64(cfg)


P_SITE_DBM_H = 16


def bound_terms(o, X, t):
    """the clamped variational bound per row at the statement's current mu: E_q[-E(x, h, y = t)] + H(q)"""
    L = o.Lm
    mu = [o.p['mu' + sfx(i)][:len(X)] for i in range(L)]
    f = X @ o.p['vb'] + ((X @ o.W(0)) * mu[0]).sum(1)
    for i in range(L):
        f = f + mu[i] @ o.hb(i)
        if i > 0:
            f = f + ((mu[i - 1] @ o.W(i)) * mu[i]).sum(1)
        m = np.clip(mu[i], 1e-300, 1 - 1e-16)
        f = f - (m * np.log(m) + (1 - m) * np.log1p(-m)).sum(1)
    U, yb = o.W(L).T, o.hb(L)
    return f + (U[t] * mu[L - 1]).sum(1) + yb[t]


def exact_log_p_vy(d, Hs):
    """log p(v, y) of a classification DBM with binary units, every (v, y) of V <= 8, h_1..h_{L-1} enumerated (L <= 2 here)
    and h_L summed out: returns [2^V, C]"""
    V, L = d['vb'].shape[0], len(Hs)
    Ws = [d['W' + sfx(i)] for i in range(L)]
    hbs = [d['hb' + sfx(i)] for i in range(L)]
    U, yb = d['U'].astype(np.float64), d['yb'].astype(np.float64)
    vs = ((np.arange(2 ** V)[:, None] >> np.arange(V)) & 1).astype(np.float64)
    sp = lambda z: np.logaddexp(0., z)
    if L == 1:
        a = vs @ Ws[0] + hbs[0]                                               # [2^V, H]
        lp = (vs @ d['vb'])[:, None] + yb[None, :] + sp(a[:, None, :] + U[None, :, :]).sum(2)
    else:
        H1 = Hs[0]
        h1s = ((np.arange(2 ** H1)[:, None] >> np.arange(H1)) & 1).astype(np.float64)
        t = vs @ d['vb']                                                       # [2^V]
        e = t[:, None] + (vs @ Ws[0]) @ h1s.T + (h1s @ hbs[0])[None, :]       # [2^V, 2^H1]
        b2 = h1s @ Ws[1] + hbs[1]                                              # [2^H1, H2]
        top = sp(b2[:, None, :] + U[None, :, :]).sum(2) + yb[None, :]          # [2^H1, C]
        lp = np.logaddexp.reduce(e[:, :, None] + top[None, :, :], axis=1)     # [2^V, C]
    return lp - np.logaddexp.reduce(lp.ravel())
