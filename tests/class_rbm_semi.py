"""Semi-supervised classification RBM (Larochelle, Mandel, Pascanu & Bengio, "Learning Algorithms for the Classification
Restricted Boltzmann Machine", JMLR 13, 2012) -- TEST INFRASTRUCTURE ONLY.

Extends the float64 statement of the model (oracle/crbm.py::OracleCRBM) and its bf16 emulation
(tests/class_rbm_bf16.py::OracleCRBMbf16) with rows labelled -1, as csrc/bm_crbm_tc.cuh trains them when beta > 0:

    grad = (1/N) sum_labelled   [ d log p(t|x) + alpha CD-k d log p(x, t) ]
         + (1/N) sum_unlabelled [ beta CD-k d log p(x) ]                      - l2 (W, U)

An unlabelled row's positive phase is exact (W: x S^T, U[y]: p(y|x) s[y], hb: S^, yb: p, vb: x).  Its chain starts from a
label y0 drawn from p(y|x) at site SITE_CRBM_Y0 (t = 0; word 0 of column block 0 of the row, the first y whose CDF exceeds u,
the CDF of the float32 p formed as the multinomial row kernel forms it) and h0 ~ sigmoid(o[., y0, .]) at SITE_H0, exactly as a
labelled row starts from S_t.  Its negative phase is the last sweep of the same chain with weight beta.  A batch without -1
is the labelled-only step of the base classes, unchanged.
"""
import numpy as np

from oracle import philox as P
from oracle.crbm import OracleCRBM
from oracle.rbm import multinomial_counts

from class_rbm_bf16 import OracleCRBMbf16, close_enough, _bf, _mm, _mult, _sigmoid, f32
from class_rbm_bf16 import SITE_CRBM_Y

SITE_CRBM_Y0 = 13


def start_labels(Pr, seed, tick, site=SITE_CRBM_Y0):
    """one categorical draw per row from the float32 posterior Pr [n, C]: the label an unlabelled row's chain starts from"""
    Pr = np.asarray(Pr, np.float32)
    m64 = Pr.astype(np.float64)
    probs = (m64 / np.cumsum(m64, axis=1)[:, -1:]).astype(np.float32)
    return np.argmax(multinomial_counts(probs, 1, seed, site, 0, tick), axis=1)


def _check_labels(y, C, beta):
    unl = y == -1
    if unl.any() and not beta > 0:
        raise RuntimeError('label -1 is outside [0, n_classes) when beta = 0')
    if np.any(y[~unl] < 0) or np.any(y[~unl] >= C):
        raise RuntimeError('labels outside [0, n_classes)')
    return unl


class OracleSemiCRBM(OracleCRBM):
    """the float64 model; cfg['beta'] (default 0) weighs the rows labelled -1"""

    def __init__(self, cfg):
        super(OracleSemiCRBM, self).__init__(cfg)
        self.beta = float(self.cfg.get('beta', 0.))
        if not self.beta >= 0:
            raise RuntimeError('beta must be non-negative')

    def log_px_unnormalised(self, X):
        """log sum_y exp(vb.x + F(x, y)) = log p(x) + log Z"""
        _, F, _ = self.posterior(X)
        m = F.max(axis=1, keepdims=True)
        return self._r(np.asarray(X, np.float64)) @ self.p['vb'] + (m + np.log(np.exp(F - m).sum(axis=1, keepdims=True)))[:, 0]

    def semi_positive(self, X):
        """gradients of mean_b log sum_y exp(vb.x_b + F(x_b, y)) with respect to W, U, vb, hb, yb"""
        Xr = self._r(np.asarray(X, np.float64))
        Pr, _, O = self.posterior(X)
        S = _sigmoid64(O)
        Sh = (Pr[:, :, None] * S).sum(axis=1)
        n = len(Xr)
        return {'W': Xr.T @ Sh / n, 'U': (Pr[:, :, None] * S).sum(axis=0) / n, 'vb': Xr.mean(axis=0),
                'hb': Sh.mean(axis=0), 'yb': Pr.mean(axis=0)}

    def chain_start(self, X, y, seed, tick):
        """(the label each row's chain starts from, S at that label [n, H])"""
        y = np.asarray(y, np.int64).reshape(-1)
        Pr, _, O = self.posterior(X)
        ts = np.where(y < 0, start_labels(Pr.astype(np.float32), seed, tick), y)
        return ts, _sigmoid64(O[np.arange(len(y)), ts])

    def train_step(self, X, y, lr, momentum, k, seed, tick, metrics=False):
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.int64).reshape(-1)
        unl = _check_labels(y, self.C, self.beta)
        if not unl.any():
            return super(OracleSemiCRBM, self).train_step(X, y, lr, momentum, k, seed, tick, metrics)
        lab, n = ~unl, len(y)
        out = None
        if metrics:
            if lab.any():
                lp = self.log_p(X[lab], y[lab])
                Pr = self.posterior(X[lab])[0]
                out = {'nll': float(-lp.mean()), 'accuracy': float(np.mean(np.argmax(Pr, axis=1) == y[lab]))}
            else:
                out = {'nll': float('nan'), 'accuracy': float('nan')}
        names = ('W', 'U', 'vb', 'hb', 'yb')
        g = {kk: np.zeros(self.p[kk].shape) for kk in names}
        if lab.any():
            d = self.disc_gradient(X[lab], y[lab])
            g = {kk: g[kk] + d[kk] * (lab.sum() / n) for kk in names}
        sp = self.semi_positive(X[unl])
        g = {kk: g[kk] + self.beta * sp[kk] * (unl.sum() / n) for kk in names}
        Xr = self._r(X)
        _, St = self.chain_start(X, y, seed, tick)
        Xk, Yk, Hk = self.chain(St, k, seed, tick)
        Y = np.zeros((n, self.C))
        Y[np.where(lab)[0], y[lab]] = 1.0
        w = np.where(lab, self.alpha, self.beta)[:, None]
        a = self.alpha
        g['W'] += (a * Xr[lab].T @ St[lab] - Xk.T @ (w * Hk)) / n
        g['U'] += (a * Y[lab].T @ St[lab] - Yk.T @ (w * Hk)) / n
        g['vb'] += (a * Xr[lab].sum(axis=0) - (w * Xk).sum(axis=0)) / n          # (the unlabelled x are in semi_positive)
        g['hb'] += (a * St[lab].sum(axis=0) - (w * Hk).sum(axis=0)) / n
        g['yb'] += (a * Y[lab].sum(axis=0) - (w * Yk).sum(axis=0)) / n
        for name in ('W', 'U'):
            g[name] = g[name] - self.l2 * self.p[name]
        for name in names:
            d = lr * (momentum * self.p['d' + name] + g[name])
            self.p['d' + name] = d
            self.p[name] = self.p[name] + d
        return out


def _sigmoid64(x):
    return 0.5 * (1.0 + np.tanh(0.5 * x))


def semi_factory(cfg):
    """engine factory for ``set_engine_factory('crbm', ...)``: the semi-supervised model's host logic on the CPU"""
    return OracleSemiCRBM(cfg)


class OracleSemiCRBMbf16(OracleCRBMbf16):
    """the engine's arithmetic for batches with rows labelled -1.  ``start_site`` and ``start_from_mean`` exist to show that
    the comparison sees the start of the unlabelled rows' chain: moving the draw, or starting from S^, breaks its bound."""
    start_site = SITE_CRBM_Y0
    start_from_mean = False

    def __init__(self, cfg):
        super(OracleSemiCRBMbf16, self).__init__(cfg)
        self.beta = float(self.cfg.get('beta', 0.))

    def train_step(self, X, y, lr, momentum, k, seed, tick, metrics=False):
        y = np.asarray(y, np.int64).reshape(-1)
        unl = _check_labels(y, self.C, self.beta)
        if not unl.any():
            return super(OracleSemiCRBMbf16, self).train_step(X, y, lr, momentum, k, seed, tick, metrics)
        p, C, H, V = self.p, self.C, self.H, self.V
        X = np.asarray(X, f32)
        n, lab = len(y), ~unl
        alpha, beta, pos = f32(self.alpha), f32(self.beta), f32(1) + f32(self.alpha)
        Xb = _bf(X)
        O, F, logz, Pr = self._columns_in(X)
        out = None
        if metrics:
            if lab.any():
                r = np.where(lab)[0]
                out = {'nll': float(np.mean(logz[r] - F[r, y[r]])), 'accuracy': float(np.mean(np.argmax(F[r], axis=1) == y[r]))}
            else:
                out = {'nll': float('nan'), 'accuracy': float('nan')}
        S = _sigmoid(O)                                              # [n, C, H]
        ts = np.where(unl, start_labels(Pr, seed, tick, self.start_site), y)
        St = S[np.arange(n), ts]
        Sh = (Pr[:, :, None] * S).sum(axis=1, dtype=f32).astype(f32)
        g = np.where(unl[:, None], beta * Sh, pos * St - Sh).astype(f32)
        E = np.zeros((n, C), f32)
        E[np.where(lab)[0], y[lab]] = 1
        coef = np.where(unl[:, None], beta * Pr, pos * E - Pr).astype(f32)
        gU = (coef[:, :, None] * S).sum(axis=0, dtype=np.float64)
        ghb = g.sum(axis=0, dtype=np.float64)
        gyb = coef.sum(axis=0, dtype=np.float64)
        GW = np.asarray(Xb, np.float64).T @ np.asarray(_bf(g), np.float64)
        # the chain: every row, as for labelled rows; unlabelled rows start from S_{y0}
        Wb, Ub = _bf(p['W']), _bf(p['U'])
        h_src = np.where(unl[:, None], Sh, St).astype(f32) if self.start_from_mean else St
        h = (P.uniform_at(n, H, seed, P.SITE_H0, 0, tick) < h_src).astype(f32) if self.sample_h else _bf(h_src)
        for s in range(1, int(k) + 1):
            xm = _sigmoid(_mm(h, Wb.T) + p['vb'])
            x = (P.uniform_at(n, V, seed, P.SITE_V, s, tick) < xm).astype(f32) if self.sample_v else _bf(xm)
            pre = (_mm(h, Ub.T) + p['yb']).astype(f32)
            ym = _mult.softmax_rows(pre, 1.0)
            yk_ = _mult.multinomial_rows(ym, 1, seed, SITE_CRBM_Y, s, tick) if self.sample_v else _bf(ym)
            hm = _sigmoid((_mm(x, Wb) + _mm(yk_, Ub)).astype(f32) + p['hb'])
            h = (P.uniform_at(n, H, seed, P.SITE_H, s, tick) < hm).astype(f32) if (self.sample_h and s < int(k)) else _bf(hm)
        Xk, Yk, Hk = x, _bf(yk_), h
        w = np.where(unl, beta, alpha).astype(f32)[:, None]
        GW = GW - np.asarray(Xk, np.float64).T @ np.asarray(_bf(w * Hk), np.float64)

        def stats(m):
            Yd, Hd = np.asarray(Yk[m], np.float64), np.asarray(Hk[m], np.float64)
            return Yd.T @ Hd, Hd.sum(axis=0), (Xb[m] - Xk[m]).sum(axis=0, dtype=np.float64), Yd.sum(axis=0)
        yh, hk, xd, yk = stats(lab)
        yhu, hku, xdu, yku = stats(unl)
        a, b = self.alpha, self.beta
        N, l2 = f32(n), f32(self.l2)
        grads = {'W': (GW.astype(f32) / N - l2 * p['W']).astype(f32),
                 'U': ((gU - a * yh - b * yhu).astype(f32) / N - l2 * p['U']).astype(f32),
                 'vb': ((a * xd + b * xdu).astype(f32) / N).astype(f32),
                 'hb': ((ghb - a * hk - b * hku).astype(f32) / N).astype(f32),
                 'yb': ((gyb - a * yk - b * yku).astype(f32) / N).astype(f32)}
        lr, mom = f32(lr), f32(momentum)
        for name in ('W', 'U', 'vb', 'hb', 'yb'):
            d = (lr * (mom * p['d' + name] + grads[name])).astype(f32)
            p['d' + name] = d
            p[name] = (p[name] + d).astype(f32)
        return out


def semi_labels(rng, rows, C, fraction):
    """labels in [0, C) with -1 on no row ('none'), on about a third of the rows ('some'; at least one of each kind) or on
    every row ('all')"""
    y = rng.randint(0, C, size=rows)
    if fraction == 'all':
        return np.full(rows, -1)
    if fraction == 'some':
        m = rng.rand(rows) < 1 / 3.
        m[0], m[1] = True, False
        y[m] = -1
    return y


def compare_semi_with_emulation(make_engine, alpha, beta, C_, sample_v, sample_h, fraction, k=1, V=37, H=70, rows=45, steps=3,
                                before_step=None, on_step=None):
    """Ragged V / H / rows, a new batch with the given unlabelled fraction every step.  Every variable after every step and
    the step's metrics (NaN for a batch without labelled rows): 1 bf16 ulp or 2e-5, whichever is larger (close_enough).
    before_step() runs before and on_step(step, labels) after each engine step (to count the interpreter's launches)."""
    cfg = dict(n_visible=V, n_hidden=H, n_classes=C_, alpha=alpha, beta=beta, l2=1e-3, max_batch=64, sample_v=sample_v,
               sample_h=sample_h)
    eng, emu = make_engine(cfg), OracleSemiCRBMbf16(cfg)
    rng = np.random.RandomState(C_ * 10 + k + int(100 * beta))
    p = {'W': 0.3 * rng.randn(V, H), 'U': 0.3 * rng.randn(C_, H), 'vb': 0.1 * rng.randn(V), 'hb': 0.1 * rng.randn(H),
         'yb': 0.1 * rng.randn(C_)}
    eng.set_params(p)
    emu.set_params(p)
    for step in range(steps):
        X = (rng.rand(rows, V) < 0.4).astype(np.float32)
        y = semi_labels(rng, rows, C_, fraction)
        if before_step:
            before_step()
        got = eng.train_step(X, y, 0.1, 0.5, k, seed=23, tick=step, metrics=True)
        if on_step:
            on_step(step, y)
        want = emu.train_step(X, y, 0.1, 0.5, k, seed=23, tick=step, metrics=True)
        if fraction == 'all':
            assert np.isnan(got['nll']) and np.isnan(got['accuracy']), got
        else:
            assert abs(got['nll'] - want['nll']) <= 1e-5 * max(1.0, want['nll']) and got['accuracy'] == want['accuracy'], \
                (step, got, want)
        g, w = eng.get_params(), emu.get_params()
        for name in w:
            ok = close_enough(g[name], w[name])
            assert ok.all(), (step, name, np.argwhere(~ok)[:5], g[name][~ok][:5], w[name][~ok][:5])
    eng.close()
