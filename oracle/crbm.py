"""Float64 numpy statement of the classification RBM (Larochelle & Bengio, ICML 2008) that
``boltzmann_machines.rbm.ClassificationRBM`` trains on the tensor cores (csrc/bm_crbm_tc.cuh), with the engine's
Philox draws.

    o[b,y,j] = hb_j + U[y,j] + (x_b W)_j      F[b,y] = yb_y + sum_j softplus(o[b,y,j])      p(y|x_b) = softmax_y F[b,.]

One step: grad = g_disc + alpha g_gen - l2 (W, U); d <- lr (momentum d + grad); theta += d.  g_disc is the gradient of the
batch mean of log p(t|x); g_gen is CD-k on the joint p(x, y) started from h0 ~ S_t = sigmoid(o[., t, .]): every sweep draws
x | h (site SITE_V), then the label y | h = softmax(yb + h U^T) (site SITE_CRBM_Y), then h | x, y (site SITE_H), all at
t = sweep index; h0 states come from SITE_H0 at t = 0.  ``sample_v`` governs x and the label, ``sample_h`` the hidden
units; the last sweep's h are means.

``_r`` and ``_w`` are the points where the engine rounds to bf16 (identity here; tests/class_rbm_bf16.py overrides them).
"""
import numpy as np

from . import philox as P
from .rbm import multinomial_counts

SITE_CRBM_Y = 12


def _softplus(x):
    return np.logaddexp(x, 0.0)


def _sigmoid(x):
    return 0.5 * (1.0 + np.tanh(0.5 * x))


class OracleCRBM(object):
    NAMES = ('W', 'U', 'vb', 'hb', 'yb', 'dW', 'dU', 'dvb', 'dhb', 'dyb')

    def __init__(self, cfg):
        c = self.cfg = dict(cfg)
        if c.get('dtype', 'float32') != 'float32' or c.get('compute') not in (None, 'bf16'):
            raise NotImplementedError('the classification RBM is defined for float32 models on the tensor cores')
        self.V, self.H, self.C = int(c['n_visible']), int(c['n_hidden']), int(c['n_classes'])
        self.alpha, self.l2 = float(c.get('alpha', 0.01)), float(c.get('l2', 0.))
        self.sample_v, self.sample_h = bool(c.get('sample_v', False)), bool(c.get('sample_h', True))
        V, H, C = self.V, self.H, self.C
        shapes = {'W': (V, H), 'U': (C, H), 'vb': (V,), 'hb': (H,), 'yb': (C,)}
        shapes.update({'d' + k: s for k, s in list(shapes.items())})
        self._shapes = shapes
        self.p = {k: np.zeros(s) for k, s in shapes.items()}

    # ---- rounding hooks --------------------------------------------------------------
    def _r(self, x):
        """an activation as the engine stores it"""
        return x

    def _w(self, name):
        """W or U as the engine's GEMMs read them"""
        return self.p[name]

    # ---- variables -------------------------------------------------------------------
    def set_params(self, d):
        for k, v in d.items():
            self.p[k] = np.array(v, dtype=np.float64).reshape(self._shapes[k])

    def get_params(self, names=None):
        return {k: self.p[k].astype(np.float32) for k in (names or self.NAMES)}

    def init_normal_weights(self, stddev, op_seed_w, op_seed_u):
        self.p['W'] = P.tf_random_normal((self.V, self.H), stddev, op_seed_w, 'float32').astype(np.float64)
        self.p['U'] = P.tf_random_normal((self.C, self.H), stddev, op_seed_u, 'float32').astype(np.float64)

    # ---- the model -------------------------------------------------------------------
    def preactivations(self, X):
        """o [n, C, H] with the input as the engine reads it"""
        A = self._r(np.asarray(X, dtype=np.float64)) @ self._w('W')
        return self._post_A(A)

    def _post_A(self, A):
        return (A + self.p['hb'])[:, None, :] + self.p['U'][None, :, :]

    def free_energies(self, O):
        return self.p['yb'][None, :] + _softplus(O).sum(axis=2)

    def posterior(self, X):
        """(p [n, C], F [n, C], o [n, C, H])"""
        O = self.preactivations(X)
        F = self.free_energies(O)
        Fm = F - F.max(axis=1, keepdims=True)
        Pr = np.exp(Fm)
        Pr /= Pr.sum(axis=1, keepdims=True)
        return Pr, F, O

    def log_p(self, X, y):
        _, F, _ = self.posterior(X)
        m = F.max(axis=1, keepdims=True)
        logz = (m + np.log(np.exp(F - m).sum(axis=1, keepdims=True)))[:, 0]
        return F[np.arange(len(y)), y] - logz

    def disc_gradient(self, X, y):
        """gradients of mean_b log p(t_b|x_b) with respect to W, U, vb, hb, yb"""
        Xr = self._r(np.asarray(X, dtype=np.float64))
        Pr, _, O = self.posterior(X)
        S = _sigmoid(O)
        n = len(y)
        St = S[np.arange(n), y]
        Sh = (Pr[:, :, None] * S).sum(axis=1)
        E = np.zeros_like(Pr)
        E[np.arange(n), y] = 1.0
        return {'W': Xr.T @ (St - Sh) / n, 'U': ((E - Pr)[:, :, None] * S).sum(axis=0) / n, 'vb': np.zeros(self.V),
                'hb': (St - Sh).sum(axis=0) / n, 'yb': (E - Pr).sum(axis=0) / n}

    def chain(self, St, k, seed, tick):
        """CD-k on p(x, y) from S_t: (X_k, Y_k, H_k means)"""
        n = St.shape[0]
        h = (P.uniform_at(n, self.H, seed, P.SITE_H0, 0, tick) < St.astype(np.float32)).astype(np.float64) if self.sample_h else St
        h = self._r(h)
        x = yk = None
        for s in range(1, int(k) + 1):
            xm = _sigmoid(h @ self._w('W').T + self.p['vb'])
            x = (P.uniform_at(n, self.V, seed, P.SITE_V, s, tick) < xm.astype(np.float32)).astype(np.float64) if self.sample_v else xm
            x = self._r(x)
            z = h @ self._w('U').T + self.p['yb']
            ym = np.exp(z - z.max(axis=1, keepdims=True))
            ym /= ym.sum(axis=1, keepdims=True)
            yk = multinomial_counts(ym.astype(np.float32), 1, seed, SITE_CRBM_Y, s, tick) if self.sample_v else ym
            yk = self._r(yk)
            hm = _sigmoid(x @ self._w('W') + yk @ self._w('U') + self.p['hb'])
            if self.sample_h and s < int(k):
                h = (P.uniform_at(n, self.H, seed, P.SITE_H, s, tick) < hm.astype(np.float32)).astype(np.float64)
            else:
                h = hm
            h = self._r(h)
        return x, yk, h

    def train_step(self, X, y, lr, momentum, k, seed, tick, metrics=False):
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.int64).reshape(-1)
        if y.min() < 0 or y.max() >= self.C:
            raise RuntimeError('labels outside [0, n_classes)')
        n = len(y)
        out = None
        if metrics:
            lp = self.log_p(X, y)
            Pr = self.posterior(X)[0]
            out = {'nll': float(-lp.mean()), 'accuracy': float(np.mean(np.argmax(Pr, axis=1) == y))}
        g = self.disc_gradient(X, y)
        if self.alpha > 0:
            Xr = self._r(X)
            O = self.preactivations(X)
            St = _sigmoid(O[np.arange(n), y])
            Y = np.zeros((n, self.C))
            Y[np.arange(n), y] = 1.0
            Xk, Yk, Hk = self.chain(St, k, seed, tick)
            gen = {'W': (Xr.T @ St - Xk.T @ Hk) / n, 'U': (Y.T @ St - Yk.T @ Hk) / n, 'vb': (Xr - Xk).mean(axis=0),
                   'hb': (St - Hk).mean(axis=0), 'yb': (Y - Yk).mean(axis=0)}
            g = {kk: g[kk] + self.alpha * gen[kk] for kk in g}
        for name in ('W', 'U'):
            g[name] = g[name] - self.l2 * self.p[name]
        for name in ('W', 'U', 'vb', 'hb', 'yb'):
            d = lr * (momentum * self.p['d' + name] + g[name])
            self.p['d' + name] = d
            self.p[name] = self.p[name] + d
        return out

    def predict_proba(self, X):
        return self.posterior(X)[0].astype(np.float32)

    def transform(self, X):
        Pr, _, O = self.posterior(X)
        return (Pr[:, :, None] * _sigmoid(O)).sum(axis=1).astype(np.float32)

    def close(self):
        pass


def crbm_factory(cfg):
    """Engine factory for ``boltzmann_machines.base.set_engine_factory('crbm', ...)``: the model's host logic on the CPU."""
    return OracleCRBM(cfg)
