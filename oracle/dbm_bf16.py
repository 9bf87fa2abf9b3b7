"""bf16-operand emulation of the DBM path -- TEST INFRASTRUCTURE ONLY.

``OracleDBM`` (oracle/dbm.py) restates the reference in its storage dtype and is the pinned oracle.  This
subclass is the checker of the *tensor-core* DBM engine (`csrc/bm_dbm_tc.cuh`, `compute='bf16'`): the same
control flow, with every value the engine keeps as a bf16 GEMM operand rounded to bf16 at the same point --

  * the weights the GEMMs read (a bf16 shadow of the fp32 variables; updates stay fp32),
  * the batch X as a GEMM operand (the fp32 batch still feeds `mean(X)`, the MSRE and the bound's X.b term),
  * variational parameters mu and particle values whenever they are *means* (samples are exact in bf16),
  * anything the caller sets or initialises (`set_params`, `init_particles`) for mu / v / h,

fp32 accumulation everywhere, and the AIS importance weights accumulated in float64 from
    softplus(b z) - softplus(a z) = log1p(sigmoid(a z) * expm1((b - a) z))        (float32 arithmetic)
over fp32 pre-activations z (bf16 operands).  It exists to state what the bf16 engine is expected to
produce; the parity claims against the reference rest on OracleDBM.  Never imported by the product.
"""
import numpy as np

from . import philox as P
from .dbm import OracleDBM
from .rbm import sigmoid, bf16_round


def _r(x):
    return bf16_round(np.asarray(x, dtype=np.float32))


def softplus_diff(a, b, z):
    """softplus(b z) - softplus(a z) in float32, free of cancellation (csrc/bm_dbm_tc.cuh::softplus_diff)."""
    a, b = np.float32(a), np.float32(b)
    z = np.asarray(z, dtype=np.float32)
    with np.errstate(over='ignore'):
        s = np.float32(1.) / (np.float32(1.) + np.exp(-a * z))
    return np.log1p(s * np.expm1((b - a) * z))


class OracleDBMbf16(OracleDBM):
    def __init__(self, cfg):
        cfg = dict(cfg)
        assert np.dtype(cfg.get('dtype', 'float32')) == np.float32, 'bf16 compute is defined for float32 models'
        super(OracleDBMbf16, self).__init__(cfg)
        assert all(k == 'bernoulli' for k in self.h_kinds) and self.v_kind in ('bernoulli', 'gaussian')

    # -- operands ------------------------------------------------------------------------------
    def Wb(self, i):
        return _r(self.W(i))

    def _state_names(self):
        names = ['v']
        for i in range(self.L):
            names += ['h' + self._sfx(i), 'mu' + self._sfx(i)]
        return names

    def _narrow_state(self):
        for k in self._state_names():
            self.p[k] = _r(self.p[k])

    def set_params(self, d):
        super(OracleDBMbf16, self).set_params(d)
        self._narrow_state()

    def init_particles(self, seed):
        super(OracleDBMbf16, self).init_particles(seed)
        self._narrow_state()

    # -- one conditional: means are rounded to bf16 when they are stored, draws compare against the fp32 mean --
    def _hidden(self, i, below, above, sample, seed, site, t, tick, acc_scale=1., bias_scale=1.):
        T = below @ self.Wb(i)
        if above is not None:
            T = T + above @ self.Wb(i + 1).T
        pre = (np.float32(acc_scale) * T + np.float32(bias_scale) * self.hb(i)).astype(np.float32)
        m = sigmoid(pre)
        if sample:
            u = P.uniform_at(m.shape[0], m.shape[1], seed, site, t, tick, getattr(self, '_row0', 0))
            return (u < m).astype(np.float32)
        return _r(m)

    def _visible(self, h0, sample, seed, site, t, tick):
        T = (h0 @ self.Wb(0).T).astype(np.float32)
        if self.v_kind == 'bernoulli':
            m = sigmoid(T + self.p['vb'])
            if sample:
                u = P.uniform_at(m.shape[0], m.shape[1], seed, site, t, tick)
                return (u < m).astype(np.float32)
            return _r(m)
        m = (T * self.sigma + self.p['vb']).astype(np.float32)
        if sample:
            eps = P.normal_at(m.shape[0], m.shape[1], seed, site, t, tick).astype(np.float32)
            return _r(m + self.sigma * eps)
        return _r(m)

    def gibbs_step(self, v, H, update_v, sample, seed, t, tick):
        L, sh = self.L, self.cfg.get('sample_h', [True] * self.L)
        Hn = [None] * L
        for i in range(L):
            below = v if i == 0 else Hn[i - 1]
            above = H[i + 1] if i + 1 < L else None
            Hn[i] = self._hidden(i, below, above, bool(sample and sh[i]), seed, P.SITE_DBM_H + i, t, tick)
        v_new = v
        if update_v:
            v_new = self._visible(Hn[0], bool(sample and self.cfg.get('sample_v', True)), seed, P.SITE_DBM_V, t, tick)
        return v_new, Hn

    def mean_field(self, X):
        L = self.L
        Xb = _r(X)
        rows = Xb.shape[0]
        mu = [self.p['mu' + self._sfx(i)][:rows] for i in range(L)]
        mu_new = []
        for i in range(L):
            below = Xb if i == 0 else mu_new[i - 1]
            sc = 2. if (i == 0 or i < L - 1) else 1.
            mu_new.append(self._hidden(i, below, None, False, 0, 0, 0, 0, acc_scale=sc))
        step = 0
        tol = np.float32(self.cfg.get('mf_tol', 1e-7))
        self.mf_diffs = []                  # the change every convergence test of this E-step measured
        while step < int(self.cfg.get('max_mf_updates', 10)):
            self.mf_diffs.append(max(np.max(np.abs(a - b)) for a, b in zip(mu, mu_new)))
            if not self.mf_diffs[-1] > tol:
                break
            _, Hn = self.gibbs_step(Xb, mu, update_v=False, sample=False, seed=0, t=0, tick=0)
            mu, mu_new = Hn, mu
            step += 1
        for i in range(L):
            self.p['mu' + self._sfx(i)][:rows] = mu[i]
        return step

    def mf_tol_stopping_at(self, X, stop):
        """An mf_tol under which the E-step on X from the current state stops after exactly `stop` sweeps, halfway (on a log
        scale) between the change it tests after `stop` sweeps and the smallest change before; None if there is no such gap."""
        import copy
        probe = copy.deepcopy(self)
        probe.cfg.update(mf_tol=-1.0, max_mf_updates=stop + 1)
        probe.mean_field(X)
        d = [float(x) for x in probe.mf_diffs]
        if not (0 < d[stop] < min(d[:stop] or [np.inf])):
            return None
        return float(np.sqrt(d[stop] * min(d[:stop]))) if stop else 2 * d[0]

    def reconstruction(self, rows):
        return self._visible(self.p['mu'][:rows], False, 0, 0, 0, 0)

    def train_step(self, X, lr, momentum, k, seed, tick, metrics=()):
        c, p, L = self.cfg, self.p, self.L
        f = np.float32
        X = np.asarray(X, dtype=np.float32)
        Xb = _r(X)
        rows = X.shape[0]
        n_mf = self.mean_field(X)
        self.particles_update(k, True, seed, tick)
        out = None
        if metrics:
            out = {}
            if 'msre' in metrics:
                out['msre'] = float(np.mean(np.square(X - self.reconstruction(rows)), dtype=np.float64))
            if 'n_mf_updates' in metrics:
                out['n_mf_updates'] = float(n_mf)
        N, Mp = f(self.B), f(self.M)
        mu = [p['mu' + self._sfx(i)][:rows] for i in range(L)]
        Hp = [p['h' + self._sfx(i)] for i in range(L)]
        l2 = f(c.get('l2', 0.))
        dvb = X.sum(axis=0) / f(rows) - p['v'].sum(axis=0) / Mp
        pos = [Xb] + mu[:-1]
        neg = [p['v']] + Hp[:-1]
        dW = []
        for i in range(L):
            G = (pos[i].T @ mu[i]) * (f(1) / N) - (neg[i].T @ Hp[i]) * (f(1) / Mp)
            dW.append(G - l2 * self.W(i))
        dhb = [mu[i].sum(axis=0) / f(rows) - Hp[i].sum(axis=0) / Mp for i in range(L)]
        damp = f(c.get('sparsity_damping', 0.9))
        targets = c.get('sparsity_target', [0.1] * L)
        costs = c.get('sparsity_cost', [0.] * L)
        for i in range(L):
            s = self._sfx(i)
            qv = Hp[i].sum(axis=0)
            p['q_means' + s] = (damp * p['q_means' + s] + (f(1) - damp) * qv[i]).astype(f)
            mv = mu[i].sum(axis=0)
            p['mu_means' + s] = (damp * p['mu_means' + s] + (f(1) - damp) * mv[i]).astype(f)
            pen = f(costs[i]) * (p['q_means' + s] - f(targets[i]))
            pen = pen + f(costs[i]) * (p['mu_means' + s] - f(targets[i]))
            dW[i] = dW[i] - pen[None, :]
            dhb[i] = dhb[i] - pen
        lr, mom = f(lr), f(momentum)
        p['dvb'] = (lr * (mom * p['dvb'] + dvb)).astype(f)
        p['vb'] = (p['vb'] + p['dvb']).astype(f)
        for i in range(L):
            s = self._sfx(i)
            p['dW' + s] = (lr * (mom * p['dW' + s] + dW[i])).astype(f)
            p['W' + s] = self._max_norm(p['W' + s] + p['dW' + s])
            p['dhb' + s] = (lr * (mom * p['dhb' + s] + dhb[i])).astype(f)
            p['hb' + s] = (p['hb' + s] + p['dhb' + s]).astype(f)
        return out

    def log_proba(self, X):
        X = np.asarray(X, dtype=np.float32)
        rows = X.shape[0]
        self.mean_field(X)
        mu0, mu1 = self.p['mu'][:rows], self.p['mu_1'][:rows]
        minus_E = ((_r(X) @ self.Wb(0)) * mu0).sum(axis=1) + ((mu0 @ self.Wb(1)) * mu1).sum(axis=1)
        minus_E = minus_E + X @ self.p['vb'] + mu0 @ self.hb(0) + mu1 @ self.hb(1)
        ent = 0.
        for m in (mu0, mu1):
            s = np.clip(m, np.float32(1e-7), np.float32(1. - 1e-7))
            ent = ent + (-s * np.log(s) - (1. - s) * np.log(1. - s)).sum(axis=1)
        return (minus_E + ent).astype(np.float64)

    # -- AIS ---------------------------------------------------------------------------------------
    def _pre(self, x):
        pa = (x @ self.Wb(0).T + self.p['vb']).astype(np.float32)
        pb = (x @ self.Wb(1) + self.hb(1)).astype(np.float32)
        return pa, pb

    def _accum2(self, x, pa, pb, a, b):
        lin = (x @ self.hb(0)).astype(np.float32)
        out = (np.float64(np.float32(b)) - np.float64(np.float32(a))) * lin.astype(np.float64)
        out = out + softplus_diff(a, b, pa).astype(np.float64).sum(axis=1)
        out = out + softplus_diff(a, b, pb).astype(np.float64).sum(axis=1)
        return out

    def _unit(self, pre, beta, sample, seed, site, tick):
        with np.errstate(over='ignore'):
            p = np.float32(1.) / (np.float32(1.) + np.exp(-(np.float32(beta) * pre)))
        if sample:
            u = P.uniform_at(pre.shape[0], pre.shape[1], seed, site, 0, tick, getattr(self, '_row0', 0))
            return (u < p).astype(np.float32)
        return _r(p)

    def _ais(self, n_runs, n_betas, k, seed):
        assert self.L == 2 and self.v_kind == 'bernoulli'
        f = np.float32
        sh = self.cfg.get('sample_h', [True] * self.L)
        sv = self.cfg.get('sample_v', True)
        delta = f(1. / n_betas)
        u = P.uniform_at(int(n_runs), self.Hs[0], seed, P.SITE_AIS_INIT, 0, 0, self._row0)
        x = (u < f(0.5)).astype(f)
        state = {'it': 0}

        def transition(x, beta, pre):
            for s in range(int(k)):
                tick = state['it'] * int(k) + s
                pa, pb = pre if (pre is not None and s == 0) else self._pre(x)
                v = self._unit(pa, beta, sv, seed, P.SITE_AIS_V, tick)
                h2 = self._unit(pb, beta, sh[1], seed, P.SITE_AIS_H2, tick)
                x = self._hidden(0, v, h2, bool(sh[0]), seed, P.SITE_AIS_H1, 0, tick, acc_scale=beta, bias_scale=beta)
            state['it'] += 1
            return x

        x = transition(x, delta, None)
        pre = self._pre(x)
        logw = np.zeros(int(n_runs), dtype=np.float64)
        beta, prev = delta, f(0.)
        while beta < f(1.) - delta + f(1e-5):
            logw += self._accum2(x, pre[0], pre[1], prev, beta)
            x = transition(x, f(beta + delta), pre)
            pre = self._pre(x)
            prev = beta
            beta = f(beta + delta)
        logw += self._accum2(x, pre[0], pre[1], prev, f(1.))
        return logw + (self.V + self.Hs[0] + self.Hs[1]) * float(np.float32(np.log(2.)))


def dbm_bf16_factory(cfg):
    return OracleDBMbf16(cfg)
