"""Centered DBMs (DESIGN.md §5.8) restated for the tests -- TEST INFRASTRUCTURE ONLY.

Unit layers j = 0..L: x_0 = v, x_{j+1} = hidden layer j; W_i [n_i, n_{i+1}] joins x_i and x_{i+1}; the stored biases are
b_0 = vb, b_{j+1} = hb....  The centered energy E_c(x) = -sum_i (x_i - o_i)'W_i (x_{i+1} - o_{i+1}) - sum_j (x_j - o_j)'a_j is the
plain DBM with b_j = a_j - c_j, c_j = W_{j-1}'o_{j-1} + W_j o_{j+1}.

* ``centered_mstep``: the engine's formulation in float64 -- stored (W, b), the rank-2 (+ rank-1) correction of the plain
  gradient, the change of c_j taken out of b_j after max-norm, then the offsets' moving average.
* ``LiteralCentered``: the same model kept in centered coordinates (W, a, o): centered products computed directly and the
  conditionals taken from E_c.  It shares no code with ``centered_mstep`` beyond the sparsity and max-norm rules.
* ``CenteredOracleDBMbf16``: the bf16 emulation of the tensor-core engine (oracle/dbm_bf16.py) with the centered update,
  in float32 where the engine computes in fp32.
"""
import numpy as np

from oracle.dbm_bf16 import OracleDBMbf16


def sfx(i):
    return '' if i == 0 else '_%d' % i


def bias_name(j):
    return 'vb' if j == 0 else 'hb' + sfx(j - 1)


def offset_name(j):
    return 'v_offset' if j == 0 else 'h_offset' + sfx(j - 1)


def coupling(W, o):
    """c_j = W_{j-1}' o_{j-1} + W_j o_{j+1} for j = 0..L"""
    L = len(W)
    c = []
    for j in range(L + 1):
        t = np.zeros(len(o[j]))
        if j > 0:
            t = t + W[j - 1].T @ o[j - 1]
        if j < L:
            t = t + W[j] @ o[j + 1]
        c.append(t)
    return c


def max_norm(W, mn):
    n = np.sqrt(np.sum(np.square(W), axis=0))
    return W * np.minimum(n, mn) / np.maximum(n, 1e-8)


def sparsity(state, i, q_sum, mu_sum, cfg):
    """dbm.py:580-590 (element i of the sum vectors: sic); returns the penalty vector and updates the running means"""
    s = sfx(i)
    damp = cfg.get('sparsity_damping', 0.9)
    cost, target = cfg['sparsity_cost'][i], cfg['sparsity_target'][i]
    state['q_means' + s] = damp * state['q_means' + s] + (1 - damp) * q_sum[i]
    state['mu_means' + s] = damp * state['mu_means' + s] + (1 - damp) * mu_sum[i]
    return cost * (state['q_means' + s] - target) + cost * (state['mu_means' + s] - target)


def centered_grads(d, p, o, N, M):
    """G^c_i by the rank-2 formula: G_i - o_i s_{i+1}' - s_i o_{i+1}' + (r / N - 1) o_i o_{i+1}'"""
    r = d[0].shape[0]
    s = [d[j].sum(0) / N - p[j].sum(0) / M for j in range(len(d))]
    out = []
    for i in range(len(d) - 1):
        G = d[i].T @ d[i + 1] / N - p[i].T @ p[i + 1] / M
        out.append(G - np.outer(o[i], s[i + 1]) - np.outer(s[i], o[i + 1]) + (r / N - 1.0) * np.outer(o[i], o[i + 1]))
    return out


def centered_grads_direct(d, p, o, N, M):
    """the centered products themselves: sum (d_i - o_i)(d_{i+1} - o_{i+1})' / N - sum (p_i - o_i)(p_{i+1} - o_{i+1})' / M"""
    return [(d[i] - o[i]).T @ (d[i + 1] - o[i + 1]) / N - (p[i] - o[i]).T @ (p[i + 1] - o[i + 1]) / M for i in range(len(d) - 1)]


def centered_mstep(state, d, p, cfg, lr, mom, rate, x_prod=None):
    """One centered M-step, engine formulation, float64, in place on `state` (the engine's variable names, plus the offsets
    and 'offsets_set').  d: data sides [X, mu_0, ..] (rows present), p: particle sides [v, h_0, ..].  x_prod: the visible data
    the products read when it differs from d[0] (the engine's bf16 operand of a Gaussian batch; sums read the batch itself)."""
    L = len(d) - 1
    N, M = float(cfg['batch_size']), float(cfg['n_particles'])
    rows = d[0].shape[0]
    W = [state['W' + sfx(i)] for i in range(L)]
    dsum = [x.sum(0) for x in d]
    psum = [x.sum(0) for x in p]
    if not state['offsets_set'][0]:
        for j in range(L + 1):
            state[offset_name(j)] = dsum[j] / rows
        state['offsets_set'] = np.ones(1)
    o = [state[offset_name(j)] for j in range(L + 1)]
    c_old = coupling(W, o)
    s_ = [dsum[j] / N - psum[j] / M for j in range(L + 1)]
    dp = d if x_prod is None else [x_prod] + list(d[1:])
    G = [dp[i].T @ dp[i + 1] / N - p[i].T @ p[i + 1] / M - np.outer(o[i], s_[i + 1]) - np.outer(s_[i], o[i + 1])
         + (rows / N - 1.0) * np.outer(o[i], o[i + 1]) for i in range(L)]
    db = [dsum[j] / rows - psum[j] / M for j in range(L + 1)]
    l2 = cfg.get('l2', 0.)
    for i in range(L):
        pen = sparsity(state, i, psum[i + 1], dsum[i + 1], cfg)
        G[i] = G[i] - l2 * W[i] - pen[None, :]
        db[i + 1] = db[i + 1] - pen
    state['dvb'] = lr * (mom * state['dvb'] + db[0])
    state['vb'] = state['vb'] + state['dvb']
    for i in range(L):
        s = sfx(i)
        state['dW' + s] = lr * (mom * state['dW' + s] + G[i])
        state['W' + s] = max_norm(state['W' + s] + state['dW' + s], cfg.get('max_norm', np.inf))
        state['dhb' + s] = lr * (mom * state['dhb' + s] + db[i + 1])
        state['hb' + s] = state['hb' + s] + state['dhb' + s]
    c_new = coupling([state['W' + sfx(i)] for i in range(L)], o)
    for j in range(L + 1):
        state[bias_name(j)] = state[bias_name(j)] - (c_new[j] - c_old[j])
        state[offset_name(j)] = (1 - rate) * o[j] + rate * dsum[j] / rows
    return state


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


class LiteralCentered(object):
    """Bernoulli DBM kept in centered coordinates (W, a, o) with velocities (dW, da), float64."""

    def __init__(self, cfg, W, b, o):
        self.cfg = cfg
        self.L = len(W)
        self.W = [np.array(w, dtype=np.float64) for w in W]
        self.o = [np.array(x, dtype=np.float64) for x in o]
        c = coupling(self.W, self.o)
        self.a = [np.asarray(b[j], dtype=np.float64) + c[j] for j in range(self.L + 1)]
        self.dW = [np.zeros_like(w) for w in self.W]
        self.da = [np.zeros_like(x) for x in self.a]
        self.sp = {}
        for i in range(self.L):
            self.sp['q_means' + sfx(i)] = np.zeros(len(self.a[i + 1]))
            self.sp['mu_means' + sfx(i)] = np.zeros(len(self.a[i + 1]))

    def stored_b(self):
        c = coupling(self.W, self.o)
        return [self.a[j] - c[j] for j in range(self.L + 1)]

    def conditional(self, j, x):
        """p(x_j = 1 | neighbours) from E_c"""
        z = self.a[j].copy()
        if j > 0:
            z = z + (x[j - 1] - self.o[j - 1]) @ self.W[j - 1]
        if j < self.L:
            z = z + (x[j + 1] - self.o[j + 1]) @ self.W[j].T
        return sigmoid(z)

    def step(self, d, p, lr, mom, rate, first):
        cfg = self.cfg
        N, M = float(cfg['batch_size']), float(cfg['n_particles'])
        rows = d[0].shape[0]
        if first:                   # the offsets move to the data means with the distribution (b) held fixed
            b = self.stored_b()
            self.o = [x.mean(0) for x in d]
            c = coupling(self.W, self.o)
            self.a = [b[j] + c[j] for j in range(self.L + 1)]
        G = centered_grads_direct(d, p, self.o, N, M)
        ga = [(d[j] - self.o[j]).sum(0) / rows - (p[j] - self.o[j]).sum(0) / M for j in range(self.L + 1)]
        for i in range(self.L):
            pen = sparsity(self.sp, i, p[i + 1].sum(0), d[i + 1].sum(0), cfg)
            G[i] = G[i] - cfg.get('l2', 0.) * self.W[i] - pen[None, :]
            ga[i + 1] = ga[i + 1] - pen
        for i in range(self.L):
            self.dW[i] = lr * (mom * self.dW[i] + G[i])
            self.W[i] = max_norm(self.W[i] + self.dW[i], cfg.get('max_norm', np.inf))
        for j in range(self.L + 1):
            self.da[j] = lr * (mom * self.da[j] + ga[j])
            self.a[j] = self.a[j] + self.da[j]
        b = self.stored_b()
        self.o = [(1 - rate) * self.o[j] + rate * d[j].mean(0) for j in range(self.L + 1)]
        c = coupling(self.W, self.o)
        self.a = [b[j] + c[j] for j in range(self.L + 1)]


class CenteredOracleDBMbf16(OracleDBMbf16):
    """The tensor-core engine's centered step: OracleDBMbf16's E-step and particle sweeps, then the centered update in
    float32 on the same bf16 operands (coupling in float64, rounded to float32 -- the kernel sums in fp32 with fma)."""

    def __init__(self, cfg, offset_rate):
        super(CenteredOracleDBMbf16, self).__init__(cfg)
        self.rate = np.float32(offset_rate)
        for j in range(self.L + 1):
            self.p[offset_name(j)] = np.zeros(self.V if j == 0 else self.Hs[j - 1], dtype=np.float32)
        self.p['offsets_set'] = np.zeros(1, dtype=np.float32)

    def _coupling32(self, o):
        W = [self.W(i).astype(np.float64) for i in range(self.L)]
        return [c.astype(np.float32) for c in coupling(W, [x.astype(np.float64) for x in o])]

    def train_step(self, X, lr, momentum, k, seed, tick, metrics=()):
        c, p, L, f = self.cfg, self.p, self.L, np.float32
        X = np.asarray(X, dtype=np.float32)
        rows = X.shape[0]
        self.mean_field(X)
        self.particles_update(k, True, seed, tick)
        from oracle.dbm_bf16 import _r
        N, Mp = f(self.B), f(self.M)
        d = [_r(X)] + [p['mu' + sfx(i)][:rows] for i in range(L)]
        P = [p['v']] + [p['h' + sfx(i)] for i in range(L)]
        dsum = [X.sum(axis=0)] + [x.sum(axis=0) for x in d[1:]]
        psum = [x.sum(axis=0) for x in P]
        if not p['offsets_set'][0]:
            for j in range(L + 1):
                p[offset_name(j)] = (dsum[j] / f(rows)).astype(f)
            p['offsets_set'] = np.ones(1, dtype=f)
        o = [p[offset_name(j)] for j in range(L + 1)]
        s = [(dsum[j] * (f(1) / N) - psum[j] * (f(1) / Mp)).astype(f) for j in range(L + 1)]
        corr = f(rows / float(self.B) - 1.0)
        c_old = self._coupling32(o)
        l2 = f(c.get('l2', 0.))
        dW = []
        for i in range(L):
            G = (d[i].T @ d[i + 1]) * (f(1) / N) - (P[i].T @ P[i + 1]) * (f(1) / Mp)
            G = G - np.outer(o[i], s[i + 1]) - np.outer(s[i], o[i + 1]) + corr * np.outer(o[i], o[i + 1])
            dW.append(G - l2 * self.W(i))
        db = [dsum[j] / f(rows) - psum[j] / Mp for j in range(L + 1)]
        damp = f(c.get('sparsity_damping', 0.9))
        for i in range(L):
            q = sfx(i)
            p['q_means' + q] = (damp * p['q_means' + q] + (f(1) - damp) * psum[i + 1][i]).astype(f)
            p['mu_means' + q] = (damp * p['mu_means' + q] + (f(1) - damp) * dsum[i + 1][i]).astype(f)
            cost, target = f(c['sparsity_cost'][i]), f(c['sparsity_target'][i])
            pen = cost * (p['q_means' + q] - target) + cost * (p['mu_means' + q] - target)
            dW[i] = dW[i] - pen[None, :]
            db[i + 1] = db[i + 1] - pen
        lr, mom = f(lr), f(momentum)
        p['dvb'] = (lr * (mom * p['dvb'] + db[0])).astype(f)
        p['vb'] = (p['vb'] + p['dvb']).astype(f)
        for i in range(L):
            q = sfx(i)
            p['dW' + q] = (lr * (mom * p['dW' + q] + dW[i])).astype(f)
            p['W' + q] = self._max_norm(p['W' + q] + p['dW' + q])
            p['dhb' + q] = (lr * (mom * p['dhb' + q] + db[i + 1])).astype(f)
            p['hb' + q] = (p['hb' + q] + p['dhb' + q]).astype(f)
        c_new = self._coupling32(o)
        for j in range(L + 1):
            p[bias_name(j)] = (p[bias_name(j)] - (c_new[j] - c_old[j])).astype(f)
            p[offset_name(j)] = ((f(1) - self.rate) * o[j] + self.rate * (dsum[j] / f(rows))).astype(f)


EPS32 = 2.0 ** -24


def replay_bounds(before, after, X, Xb, cfg, lr, mom, rate):
    """The float64 centered M-step applied to the step's own exported activations (``after``: mu, v, h of slot 0) from the
    variables before the step, with a bound per element for the engine's fp32 arithmetic on the same operands:
      gradient entries: K u sum |terms| (K = rows + n_particles + 4 accumulated terms, u = 2^-24), times lr in W / dW;
      couplings: (n + 2) u sum |W||o| each, twice (before and after); and 8 ulps of every stored value.
    Returns {name: (want, bound)} for W, dW, biases, their velocities and the offsets."""
    L = len(cfg['n_hiddens'])
    rows = X.shape[0]
    st = {k: np.asarray(v, dtype=np.float64).copy() for k, v in before.items()}
    d = [np.asarray(X, np.float64)] + [np.asarray(after['mu' + sfx(i)][:rows], np.float64) for i in range(L)]
    p = [np.asarray(after['v'], np.float64)] + [np.asarray(after['h' + sfx(i)], np.float64) for i in range(L)]
    xp = np.asarray(Xb, np.float64)
    first = not st['offsets_set'][0]
    centered_mstep(st, d, p, cfg, lr, mom, rate, x_prod=xp)
    N, M = float(cfg['batch_size']), float(cfg['n_particles'])
    o = [st[offset_name(j)] if not first else d[j].mean(0) for j in range(L + 1)]
    if not first:     # the offsets used by the step are the ones before it
        o = [np.asarray(before[offset_name(j)], np.float64) for j in range(L + 1)]
    dp = [xp] + d[1:]
    K = rows + M + 4
    out = {}
    absW = [np.abs(np.asarray(before['W' + sfx(i)], np.float64)) for i in range(L)]
    absW_new = [np.abs(st['W' + sfx(i)]) for i in range(L)]
    for i in range(L):
        q = sfx(i)
        A = (np.abs(dp[i]).T @ np.abs(dp[i + 1]) / N + np.abs(p[i]).T @ np.abs(p[i + 1]) / M
             + np.outer(np.abs(o[i]), np.abs(d[i + 1]).sum(0) / N + np.abs(p[i + 1]).sum(0) / M)
             + np.outer(np.abs(d[i]).sum(0) / N + np.abs(p[i]).sum(0) / M, np.abs(o[i + 1]))
             + np.outer(np.abs(o[i]), np.abs(o[i + 1])) + cfg.get('l2', 0.) * absW[i])
        gb = lr * K * EPS32 * A
        out['dW' + q] = (st['dW' + q], gb + 8 * EPS32 * np.abs(st['dW' + q]) + 8 * EPS32 * lr * mom * np.abs(before['dW' + q]))
        out['W' + q] = (st['W' + q], gb + 8 * EPS32 * (absW[i] + absW_new[i]) + out['dW' + q][1])
    for j in range(L + 1):
        n_nb = (len(o[j - 1]) if j > 0 else 0) + (len(o[j + 1]) if j < L else 0) + 2
        C = np.zeros(len(o[j]))
        for Wa in (absW, absW_new):
            if j > 0:
                C = C + Wa[j - 1].T @ np.abs(o[j - 1])
            if j < L:
                C = C + Wa[j] @ np.abs(o[j + 1])
        dn = 'dvb' if j == 0 else 'dhb' + sfx(j - 1)
        gbias = lr * (rows + M + 4) * EPS32 * (np.abs(d[j]).sum(0) / rows + np.abs(p[j]).sum(0) / M + 1.0)
        out[dn] = (st[dn], gbias + 8 * EPS32 * np.abs(st[dn]))
        out[bias_name(j)] = (st[bias_name(j)], gbias + n_nb * EPS32 * C + 8 * EPS32 * (np.abs(st[bias_name(j)]) + C))
        out[offset_name(j)] = (st[offset_name(j)], 8 * EPS32 * (np.abs(st[offset_name(j)]) + np.abs(d[j]).sum(0) / rows) +
                               rows * EPS32 * np.abs(d[j]).sum(0) / rows)
    return out


def check_replay(bounds, after):
    """[(name, worst |engine - float64| / bound)]; raises AssertionError naming the first variable outside its bound"""
    worst = []
    for k, (want, tol) in bounds.items():
        err = np.abs(np.asarray(after[k], np.float64) - want)
        r = float(np.max(err / np.maximum(tol, 1e-300)))
        worst.append((k, r))
        assert r <= 1.0, '%s: max |engine - float64| = %.3g, %.3g of its bound' % (k, float(err.max()), r)
    return worst
