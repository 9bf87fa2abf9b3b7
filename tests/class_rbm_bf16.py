"""bf16 emulation of the tensor-core classification RBM (csrc/bm_crbm_tc.cuh) -- TEST INFRASTRUCTURE ONLY.

`oracle/crbm.py::OracleCRBM` states the model in float64.  This subclass computes what the engine computes, rounding where it
rounds:
  * X, the chain's x / label / h and the W / U shadows are bf16 GEMM operands; GEMMs accumulate in fp32 (here: float64 of the
    bf16 values, then float32);
  * the posterior: a = A + hb, o = a + U and softplus(o) in float32, F = yb + the softplus sum in float64, p = float32;
  * the columns: sigmoid(o) in float32, S^ = sum_y p s (float32), G = bf16((1 + alpha) S_t - S^), h0 = (u < S_t) or bf16(S_t);
  * the chain's conditionals in float32 from fp32 pre-activations: x | h and h | x, y through sigmoid (states: u < mean),
    y | h through the multinomial row kernel (tests/dbm_bf16_multinomial.py: softmax_rows / multinomial_rows, one draw);
  * the W gradient from bf16(G) and bf16(alpha H_k); every other sum and the momentum update in float32.
"""
import importlib.util
import os

import numpy as np

from oracle import philox as P
from oracle.crbm import OracleCRBM, SITE_CRBM_Y
from oracle.rbm import bf16_round

_spec = importlib.util.spec_from_file_location('dbm_bf16_multinomial', os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                                    'dbm_bf16_multinomial.py'))
_mult = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_mult)

f32 = np.float32


def _bf(x):
    return bf16_round(np.asarray(x, dtype=f32))


def _mm(a, b):
    """a GEMM of bf16 operands with fp32 accumulation"""
    return (np.asarray(a, np.float64) @ np.asarray(b, np.float64)).astype(f32)


def _sigmoid(x):
    x = np.asarray(x, f32)
    with np.errstate(over='ignore'):
        return (f32(1) / (f32(1) + np.exp(-x))).astype(f32)


def _softplus(x):
    x = np.asarray(x, f32)
    return (np.maximum(x, f32(0)) + np.log1p(np.exp(-np.abs(x)))).astype(f32)


class OracleCRBMbf16(OracleCRBM):
    def set_params(self, d):
        for k, v in d.items():
            self.p[k] = np.array(v, dtype=f32).reshape(self._shapes[k])

    def init_normal_weights(self, stddev, op_seed_w, op_seed_u):
        super(OracleCRBMbf16, self).init_normal_weights(stddev, op_seed_w, op_seed_u)
        self.p['W'], self.p['U'] = self.p['W'].astype(f32), self.p['U'].astype(f32)

    def _columns_in(self, X):
        """o [n, C, H] (float32) and the posterior from bf16 X and the bf16 W shadow"""
        p = self.p
        A = _mm(_bf(X), _bf(p['W']))
        a = (A + p['hb']).astype(f32)
        O = (a[:, None, :] + p['U'][None, :, :]).astype(f32)
        F = p['yb'].astype(np.float64)[None, :] + _softplus(O).astype(np.float64).sum(axis=2)
        m = F.max(axis=1, keepdims=True)
        logz = m + np.log(np.exp(F - m).sum(axis=1, keepdims=True))
        return O, F, logz[:, 0], np.exp(F - logz).astype(f32)

    def predict_proba(self, X):
        return self._columns_in(X)[3]

    def transform(self, X):
        O, _, _, Pr = self._columns_in(X)
        return (Pr[:, :, None] * _sigmoid(O)).sum(axis=1, dtype=f32).astype(f32)

    def train_step(self, X, y, lr, momentum, k, seed, tick, metrics=False):
        p, C, H = self.p, self.C, self.H
        X = np.asarray(X, f32)
        y = np.asarray(y, np.int64).reshape(-1)
        n = len(y)
        alpha, pos = f32(self.alpha), f32(1) + f32(self.alpha)
        Xb = _bf(X)
        O, F, logz, Pr = self._columns_in(X)
        out = None
        if metrics:
            out = {'nll': float(np.mean(logz - F[np.arange(n), y])), 'accuracy': float(np.mean(np.argmax(F, axis=1) == y))}
        S = _sigmoid(O)                                              # [n, C, H]
        St = S[np.arange(n), y]
        Sh = (Pr[:, :, None] * S).sum(axis=1, dtype=f32).astype(f32)
        g = (pos * St - Sh).astype(f32)
        E = np.zeros((n, C), f32)
        E[np.arange(n), y] = 1
        coef = (pos * E - Pr).astype(f32)
        gU = (coef[:, :, None] * S).sum(axis=0, dtype=np.float64)
        ghb = g.sum(axis=0, dtype=np.float64)
        gyb = coef.sum(axis=0, dtype=np.float64)
        GW = np.asarray(Xb, np.float64).T @ np.asarray(_bf(g), np.float64)
        yh = hk = xd = yk = 0.0
        if self.alpha > 0:
            Wb, Ub = _bf(p['W']), _bf(p['U'])
            h = (P.uniform_at(n, H, seed, P.SITE_H0, 0, tick) < St).astype(f32) if self.sample_h else _bf(St)
            for s in range(1, int(k) + 1):
                xm = _sigmoid(_mm(h, Wb.T) + p['vb'])
                x = (P.uniform_at(n, self.V, seed, P.SITE_V, s, tick) < xm).astype(f32) if self.sample_v else _bf(xm)
                pre = (_mm(h, Ub.T) + p['yb']).astype(f32)
                ym = _mult.softmax_rows(pre, 1.0)
                yk_ = _mult.multinomial_rows(ym, 1, seed, SITE_CRBM_Y, s, tick) if self.sample_v else _bf(ym)
                hm = _sigmoid((_mm(x, Wb) + _mm(yk_, Ub)).astype(f32) + p['hb'])
                h = (P.uniform_at(n, H, seed, P.SITE_H, s, tick) < hm).astype(f32) if (self.sample_h and s < int(k)) else _bf(hm)
            Xk, Yk, Hk = x, _bf(yk_), h
            GW = GW - np.asarray(Xk, np.float64).T @ np.asarray(_bf(alpha * Hk), np.float64)
            yh = np.asarray(Yk, np.float64).T @ np.asarray(Hk, np.float64)
            hk = Hk.sum(axis=0, dtype=np.float64)
            xd = (Xb - Xk).sum(axis=0, dtype=np.float64)
            yk = Yk.sum(axis=0, dtype=np.float64)
        N, l2 = f32(n), f32(self.l2)
        grads = {'W': (GW.astype(f32) / N - l2 * p['W']).astype(f32),
                 'U': ((gU - self.alpha * np.asarray(yh)).astype(f32) / N - l2 * p['U']).astype(f32),
                 'vb': (alpha * np.asarray(xd * np.ones(self.V)).astype(f32) / N).astype(f32),
                 'hb': ((ghb - self.alpha * np.asarray(hk)).astype(f32) / N).astype(f32),
                 'yb': ((gyb - self.alpha * np.asarray(yk)).astype(f32) / N).astype(f32)}
        lr, mom = f32(lr), f32(momentum)
        for name in ('W', 'U', 'vb', 'hb', 'yb'):
            d = (lr * (mom * p['d' + name] + grads[name])).astype(f32)
            p['d' + name] = d
            p[name] = (p[name] + d).astype(f32)
        return out


def close_enough(got, want):
    """1 bf16 ulp (2^-8 relative) or 2e-5 absolute, whichever is larger, element by element"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want) <= np.maximum(2e-5, np.abs(want) * 2.0 ** -8)


def compare_with_emulation(make_engine, alpha, k, C_, sample_v, sample_h, V=37, H=70, rows=45, steps=3):
    """Ragged V / H / rows.  Every variable after every step, the step's metrics, then predict_proba and transform:
    1 bf16 ulp or 2e-5, whichever is larger (close_enough)."""
    cfg = dict(n_visible=V, n_hidden=H, n_classes=C_, alpha=alpha, l2=1e-3, max_batch=64, sample_v=sample_v,
               sample_h=sample_h)
    eng, emu = make_engine(cfg), OracleCRBMbf16(cfg)
    rng = np.random.RandomState(C_ * 10 + k)
    p = {'W': 0.3 * rng.randn(V, H), 'U': 0.3 * rng.randn(C_, H), 'vb': 0.1 * rng.randn(V), 'hb': 0.1 * rng.randn(H),
         'yb': 0.1 * rng.randn(C_)}
    eng.set_params(p)
    emu.set_params(p)
    for step in range(steps):
        X = (rng.rand(rows, V) < 0.4).astype(np.float32)
        y = rng.randint(0, C_, size=rows)
        got = eng.train_step(X, y, 0.1, 0.5, k, seed=23, tick=step, metrics=True)
        want = emu.train_step(X, y, 0.1, 0.5, k, seed=23, tick=step, metrics=True)
        assert abs(got['nll'] - want['nll']) <= 1e-5 * max(1.0, want['nll']) and got['accuracy'] == want['accuracy'], (step, got, want)
        g, w = eng.get_params(), emu.get_params()
        for name in w:
            ok = close_enough(g[name], w[name])
            assert ok.all(), (step, name, np.argwhere(~ok)[:5], g[name][~ok][:5], w[name][~ok][:5])
    X = (rng.rand(rows, V) < 0.4).astype(np.float32)
    assert close_enough(eng.predict_proba(X), emu.predict_proba(X)).all()
    assert close_enough(eng.transform(X), emu.transform(X)).all()
    eng.close()
