"""Parallel tempering of the DBM's persistent chains, restated on the oracles -- TEST INFRASTRUCTURE ONLY.

The semantics (DESIGN.md §5.4, include/bm.h bm_dbm_cfg.n_temps):

  * ladder betas = [1 = b_0 > b_1 > ... > b_{T-1} >= 0]; slot m holds n_particles chains (v, h_1 .. h_L);
  * a sweep of slot m is the usual sweep (hidden layers bottom-up, each reading the old layer above, then v) with every
    conditional sigmoid(b_m (pre-activation + bias)); its draws use the usual sites and t / tick at row row0 + m M + p,
    so slot 0 draws exactly what the untempered chain draws;
  * every committed particle update (train_step, val_metrics, the first half of sample_v) ends with ONE swap round:
    pairs (m, m+1) with m = tick (mod 2), E(x) = -(v.b + sum_i h_i.c_i + sum_i h_{i-1} W_i h_i), accept when
    log u < (b_m - b_{m+1}) (E(x_m) - E(x_{m+1})), u from Philox (SITE_DBM_PT, t = m, tick) at column 0 of row row0 + p;
    an accepted swap exchanges the two slots' states;
  * slots 1..T-1 are the variables 'v_pt' [T-1, M, V] and 'h_pt', 'h_pt_1', ... [T-1, M, H_i]; slot 0 stays 'v', 'h...'.

`PTOracleDBM` is the float64 (or float32) restatement on oracle.dbm.OracleDBM; `PTOracleDBMbf16` the bf16 emulation of the
tensor-core engine on oracle.dbm_bf16.OracleDBMbf16 (bf16 weight operands, fp32 pre-activations b * acc + b * bias, the
energies from bf16 weights in float64).  `mutation` switches on one deliberate error, so that a statistical test can show
it would notice: 'sign' (acceptance sign flipped), 'no_bias_energy' (E without the bias terms), 'beta_weights_only'
(b_m scales the weight term of the conditionals but not the biases).
"""
import numpy as np

from oracle import philox as P
from oracle.dbm import OracleDBM
from oracle.dbm_bf16 import OracleDBMbf16, _r
from oracle.rbm import sigmoid

SITE_DBM_PT = 14


class _Tempering(object):
    def _pt_setup(self, betas, mutation=None):
        self.betas = [float(b) for b in betas]
        self.T = len(self.betas)
        self.mutation = mutation
        self.pt_accepted = np.zeros(max(self.T - 1, 0), dtype=np.int64)
        self.pt_proposed = np.zeros(max(self.T - 1, 0), dtype=np.int64)
        self.last_swaps = None                      # [T-1, M] decisions of the last round (False where not proposed)
        if self.T > 1:
            sizes = [self.V] + self.Hs
            for idx, name in enumerate(self._pt_names()):
                self.p[name] = np.zeros((self.T - 1, self.M, sizes[idx]), dtype=self.dt)

    def _pt_names(self):
        return ['v_pt'] + ['h_pt' + self._sfx(i) for i in range(self.L)]

    def _base_names(self):
        return ['v'] + ['h' + self._sfx(i) for i in range(self.L)]

    def slot(self, m):
        """(v, [h_0 .. h_{L-1}]) of slot m"""
        if m == 0:
            return self.p['v'], [self.p['h' + self._sfx(i)] for i in range(self.L)]
        names = self._pt_names()
        return self.p[names[0]][m - 1], [self.p[n][m - 1] for n in names[1:]]

    def _set_slot(self, m, v, H):
        if m == 0:
            self.p['v'] = v
            for i in range(self.L):
                self.p['h' + self._sfx(i)] = H[i]
            return
        for name, x in zip(self._pt_names(), [v] + list(H)):
            self.p[name][m - 1] = x

    def init_particles(self, seed):
        super(_Tempering, self).init_particles(seed)
        r0 = self._particle_row0()
        sizes = [self.V] + self.Hs
        for m in range(1, self.T):
            for idx, name in enumerate(self._pt_names()):
                u = P.uniform_at(self.M, sizes[idx], seed, P.SITE_PARTICLE_INIT, idx, 0, r0 + m * self.M)
                self.p[name][m - 1] = self._narrow(u.astype(self.dt))

    def _narrow(self, x):
        return x

    def energy(self, v, H):
        """E(x) per particle, float64"""
        f = np.float64
        with_bias = self.mutation != 'no_bias_energy'
        e = np.zeros(v.shape[0], dtype=f)
        below = v.astype(f)
        if with_bias:
            e -= below @ self.p['vb'].astype(f)
        for i in range(self.L):
            h = H[i].astype(f)
            prod = below @ self._energy_W(i).astype(f)
            e -= (prod * h).sum(axis=1)
            if with_bias:
                e -= h @ self.hb(i).astype(f)
            below = h
        return e

    def _energy_W(self, i):
        return self.W(i)

    def swap_round(self, seed, tick):
        T, M = self.T, self.M
        E = [self.energy(*self.slot(m)) for m in range(T)]
        r0 = self._particle_row0()
        self.last_swaps = np.zeros((T - 1, M), dtype=bool)
        for m in range(int(tick) % 2, T - 1, 2):
            u = P.uniform_at(M, 1, seed, SITE_DBM_PT, m, tick, r0)[:, 0].astype(np.float64)
            with np.errstate(divide='ignore'):
                lu = np.log(u)
            d = (self.betas[m] - self.betas[m + 1]) * (E[m] - E[m + 1])
            ok = lu < (-d if self.mutation == 'sign' else d)
            self.last_swaps[m] = ok
            self.pt_accepted[m] += int(ok.sum())
            self.pt_proposed[m] += M
            (va, Ha), (vb, Hb) = self.slot(m), self.slot(m + 1)
            va, vb = va.copy(), vb.copy()
            Ha, Hb = [h.copy() for h in Ha], [h.copy() for h in Hb]
            va[ok], vb[ok] = vb[ok], va[ok]
            for i in range(self.L):
                Ha[i][ok], Hb[i][ok] = Hb[i][ok], Ha[i][ok]
            self._set_slot(m, va, Ha)
            self._set_slot(m + 1, vb, Hb)

    def particles_update(self, n_steps, sample, seed, tick, t0=0, commit=True):
        if not commit or self.T == 1:
            return super(_Tempering, self).particles_update(n_steps, sample, seed, tick, t0=t0, commit=commit)
        r0 = self._particle_row0()
        for m in range(self.T):
            v, H = self.slot(m)
            for s in range(int(n_steps)):
                v, H = self.tempered_sweep(v, H, self.betas[m], bool(sample), seed, t0 + s + 1, tick, r0 + m * self.M)
            self._set_slot(m, v, list(H))
        self.swap_round(seed, tick)
        return self.slot(0)


class PTOracleDBM(_Tempering, OracleDBM):
    """The float64 / float32 oracle with the tempered ladder."""

    def __init__(self, cfg, betas, mutation=None):
        OracleDBM.__init__(self, cfg)
        self._pt_setup(betas, mutation)

    def tempered_sweep(self, v, H, beta, sample, seed, t, tick, row0):
        L, dt = self.L, self.dt
        bw = dt.type(beta)
        bb = dt.type(1.) if self.mutation == 'beta_weights_only' else bw
        self._row0 = row0
        try:
            Hn = [None] * L
            for i in range(L):
                below = v if i == 0 else Hn[i - 1]
                x = below @ self.W(i)
                if i + 1 < L:
                    x = x + H[i + 1] @ self.W(i + 1).T
                Hn[i] = sigmoid((bw * x + bb * self.hb(i)).astype(dt))
                if sample:
                    Hn[i] = self._sample('bernoulli', Hn[i], 100., seed, P.SITE_DBM_H + i, t, tick)
            v = sigmoid((bw * (Hn[0] @ self.W(0).T) + bb * self.p['vb']).astype(dt))
            if sample:
                v = self._sample('bernoulli', v, 100., seed, P.SITE_DBM_V, t, tick)
        finally:
            self._row0 = 0
        return v, Hn


class PTOracleDBMbf16(_Tempering, OracleDBMbf16):
    """The bf16 emulation of the tensor-core engine with the tempered ladder: each op's pre-activation is
    fp32(b) * (bf16 operands @ bf16 weights) + fp32(b) * bias in float32, as the op's epilogue computes it."""

    def __init__(self, cfg, betas, mutation=None):
        OracleDBMbf16.__init__(self, cfg)
        self._pt_setup(betas, mutation)

    def _state_names(self):
        return OracleDBMbf16._state_names(self) + (self._pt_names() if self.T > 1 else [])

    def _narrow(self, x):
        return _r(x)

    def _energy_W(self, i):
        return self.Wb(i)

    def tempered_sweep(self, v, H, beta, sample, seed, t, tick, row0):
        L, f = self.L, np.float32
        b = f(beta)
        self._row0 = row0
        try:
            Hn = [None] * L
            for i in range(L):
                below = v if i == 0 else Hn[i - 1]
                above = H[i + 1] if i + 1 < L else None
                Hn[i] = self._hidden(i, below, above, sample, seed, P.SITE_DBM_H + i, t, tick, acc_scale=b, bias_scale=b)
        finally:
            self._row0 = 0
        pre = (b * (Hn[0] @ self.Wb(0).T).astype(f) + b * self.p['vb']).astype(f)
        m = sigmoid(pre)
        if sample:
            u = P.uniform_at(m.shape[0], m.shape[1], seed, P.SITE_DBM_V, t, tick, row0)
            v = (u < m).astype(f)
        else:
            v = _r(m)
        return v, Hn


def exact_log_marginal_v(W, hb, vb, beta=1.0):
    """log p_beta(v) over all 2^V visible states of a binary DBM with weights W[i], biases hb[i], vb (enumeration of every
    hidden layer but the last, which is summed out analytically).  Returns (states [2^V, V], log p [2^V])."""
    V = len(vb)
    L = len(W)
    allv = ((np.arange(2 ** V)[:, None] >> np.arange(V)[None, :]) & 1).astype(np.float64)
    def states(n):
        return ((np.arange(2 ** n)[:, None] >> np.arange(n)[None, :]) & 1).astype(np.float64)
    W = [np.asarray(w, np.float64) for w in W]
    hb = [np.asarray(c, np.float64) for c in hb]
    vb = np.asarray(vb, np.float64)
    # log sum over h_0 .. h_{L-2} (enumerated) of exp(-beta E), with h_{L-1} summed out: softplus(beta (h_{L-2} W_{L-1} + c))
    logp = beta * (allv @ vb)
    if L == 1:
        logp = logp + np.logaddexp(0., beta * (allv @ W[0] + hb[0])).sum(axis=1)
    else:
        hs = [states(W[i].shape[1]) for i in range(L - 1)]
        import itertools
        acc = np.full(len(allv), -np.inf)
        for combo in itertools.product(*[range(len(h)) for h in hs]):
            hsel = [hs[i][combo[i]] for i in range(L - 1)]
            t = beta * (allv @ W[0] @ hsel[0] + hsel[0] @ hb[0])
            for i in range(1, L - 1):
                t = t + beta * (hsel[i - 1] @ W[i] @ hsel[i] + hsel[i] @ hb[i])
            last = hsel[L - 2] @ W[L - 1] + hb[L - 1]
            t = t + np.logaddexp(0., beta * last).sum()
            acc = np.logaddexp(acc, t)
        logp = logp + acc
    logp = logp - np.logaddexp.reduce(logp)
    return allv, logp
