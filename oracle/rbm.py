"""CPU restatement (numpy) of the reference's CD-k RBM path -- TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs may import this module; the product package
(``boltzmann-machines_b200/``) never does.

PARITY STATUS: pinned against the reference's OWN SOURCE for the RBM path.  tests/golden/reference_rbm_cases.json holds
results of yell/boltzmann-machines' unmodified `BernoulliRBM / GaussianRBM / MultinomialRBM` classes (`fit` with
schedules, dropout, fixed and variable-length chains, validation metrics, free-energy gap; `transform`; `init`;
`get_tf_params`) executed with `oracle/tf1shim.py` in place of TensorFlow 1.3 (which cannot be installed here) and with
the random ops answered from the Philox layout of oracle/philox.py; tests/test_z_reference_golden.py replays the same
scenarios through the host mirror on this oracle (and, on the GPU, on the CUDA engine) and matches weights, momentum
accumulators, MSRE / PLL / L2 / free-energy-gap logs and transforms to float rounding.  The RNG primitive and TF's
weight-initialiser stream are pinned by the reference's own KAT (oracle/philox.py; reproduced through the reference's
`init()` in the `init_from_seed` golden case).  NOT pinned: TensorFlow's own draw order for the Gibbs stream (it depends
on graph construction order, SURVEY.md §8c -- the engine defines its own counter layout) and TensorFlow's kernels.
Each method cites the lines it restates (paths relative to /root/reference/boltzmann_machines/).

TF-1.3 op semantics relied on: ``tf.nn.dropout(x, keep)`` = x/keep*floor(keep+u);
``tf.nn.l2_loss(w)`` = sum(w**2)/2; ``tf.log_sigmoid(x)`` = -softplus(-x);
``Bernoulli(probs=p).sample()`` = (u < p); ``Normal(loc, scale).sample()`` =
loc + scale*N(0,1); ``Multinomial(M, probs).sample()`` = counts of M categorical
draws.
"""
import numpy as np

from . import philox as P

KINDS = ('bernoulli', 'multinomial', 'gaussian')


def bf16_round(x):
    """Round-to-nearest-even float32 -> bfloat16 -> float32 (what the tensor
    path stores)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32)
    r = ((u >> np.uint32(16)) & np.uint32(1)) + np.uint32(0x7FFF)
    return ((u + r) & np.uint32(0xFFFF0000)).view(np.float32)


def sigmoid(x):
    # 1/(1+exp(-x)) evaluated stably in the array's dtype
    out = np.empty_like(x)
    pos = x >= 0
    out[pos] = 1.0 / (1.0 + np.exp(-x[pos]))
    e = np.exp(x[~pos])
    out[~pos] = e / (1.0 + e)
    return out


def softplus(x):
    return np.logaddexp(x, 0).astype(x.dtype, copy=False)


def multinomial_counts(probs, n_draws, seed, site, t, tick, row0=0):
    """counts[r, j] = #{draws d < n_draws : cdf[r, j-1] <= u[r, d] < cdf[r, j]}.
    CDF in float64 of the float32 probabilities; draw d of row r uses element
    (r, d) of the site's uniform block."""
    rows, K = probs.shape
    u = P.uniform_at(rows, int(n_draws), seed, site, t, tick, row0).astype(np.float64)
    p64 = probs.astype(np.float64)
    cdf = np.cumsum(p64, axis=1)
    cdf /= cdf[:, -1:]
    counts = np.zeros((rows, K), dtype=np.float64)
    for r in range(rows):
        idx = np.searchsorted(cdf[r], u[r], side='right')
        idx = np.minimum(idx, K - 1)
        counts[r] = np.bincount(idx, minlength=K)
    return counts


class OracleRBM(object):
    """State + one training step of ``BaseRBM`` (rbm/base_rbm.py:415-525)."""

    def __init__(self, cfg):
        self.cfg = dict(cfg)
        c = self.cfg
        self.V, self.H = int(c['n_visible']), int(c['n_hidden'])
        self.dt = np.dtype(c.get('dtype', 'float32'))
        self.v_kind, self.h_kind = c.get('v_kind', 'bernoulli'), c.get('h_kind', 'bernoulli')
        assert self.v_kind in KINDS and self.h_kind in KINDS
        self.emulate_bf16 = c.get('compute', 'fp32') == 'bf16'
        sig = c.get('sigma', None)
        self.sigma = None if sig is None else np.broadcast_to(
            np.asarray(sig, dtype=self.dt), (self.V,)).copy()
        z = lambda *s: np.zeros(s, dtype=self.dt)
        self.p = dict(W=z(self.V, self.H), vb=z(self.V), hb=z(self.H),
                      dW=z(self.V, self.H), dvb=z(self.V), dhb=z(self.H), q_means=z(self.H))
        # base_rbm.py:256-262
        self.m_up = self.dt.type(2.0 if c.get('dbm_first', False) else 1.0)
        self.m_dn = self.dt.type(2.0 if c.get('dbm_last', False) else 1.0)

    # -- param access ------------------------------------------------------
    def set_params(self, d):
        for k, v in d.items():
            if k == 'sigma':
                continue
            self.p[k] = np.array(v, dtype=self.dt).reshape(self.p[k].shape)

    def get_params(self, names=None):
        want = list(self.p) + ['sigma'] if names is None else list(names)
        out = {k: self.p[k].copy() for k in want if k in self.p}
        if self.sigma is not None and 'sigma' in want:
            out['sigma'] = self.sigma.copy()
        return out

    def init_normal_W(self, stddev, op_seed):
        # base_rbm.py:277-279: tf.random_normal(stddev=W_init, seed=random_seed)
        self.p['W'] = P.tf_random_normal((self.V, self.H), stddev, op_seed, self.dt.name).astype(self.dt)

    # -- helpers -----------------------------------------------------------
    def _r(self, x):
        return bf16_round(x).astype(self.dt) if self.emulate_bf16 else x

    def _Wc(self):
        return self._r(self.p['W'])

    def _activation(self, kind, x, b, n_samples, sigma):
        # layers.py:47-48 (Bernoulli), :65-66 (Multinomial), :84-86 (Gaussian)
        if kind == 'bernoulli':
            return sigmoid(x + b)
        if kind == 'multinomial':
            z = x + b
            z = z - z.max(axis=1, keepdims=True)
            e = np.exp(z)
            return (self.dt.type(n_samples) * e / e.sum(axis=1, keepdims=True)).astype(self.dt)
        return (x * sigma + b).astype(self.dt)

    def _sample(self, kind, means, n_samples, sigma, seed, site, t, tick, row0):
        # layers.py:34-36,50-51 / :68-70 / :88-89
        rows, n = means.shape
        if kind == 'bernoulli':
            u = P.uniform_at(rows, n, seed, site, t, tick, row0)
            return (u < means.astype(np.float32)).astype(self.dt) if self.dt == np.float32 \
                else (u.astype(np.float64) < means).astype(self.dt)
        if kind == 'multinomial':
            probs = (means / means.sum(axis=1, keepdims=True)).astype(np.float32)
            return multinomial_counts(probs, int(n_samples), seed, site, t, tick, row0).astype(self.dt)
        eps = P.normal_at(rows, n, seed, site, t, tick, row0).astype(self.dt)
        return (means + sigma * eps).astype(self.dt)

    def means_h_given_v(self, v):
        # base_rbm.py:339-345 (+ :329-332)
        x = self.m_up * (v @ self._Wc())
        return self._activation(self.h_kind, x, self.m_up * self.p['hb'],
                                self.cfg.get('h_n_samples', 100), None)

    def means_v_given_h(self, h):
        # base_rbm.py:353-359 (+ :334-337)
        x = self.m_dn * (h @ self._Wc().T)
        return self._activation(self.v_kind, x, self.m_dn * self.p['vb'],
                                self.cfg.get('v_n_samples', 100), self.sigma)

    def _sample_h(self, m, seed, site, t, tick, row0):
        return self._sample(self.h_kind, m, self.cfg.get('h_n_samples', 100), None,
                            seed, site, t, tick, row0)

    def _sample_v(self, m, seed, site, t, tick, row0):
        return self._sample(self.v_kind, m, self.cfg.get('v_n_samples', 100), self.sigma,
                            seed, site, t, tick, row0)

    def prepare_input(self, X, seed, tick, row0=0):
        """GaussianRBM pre-division (rbm/rbm.py:101-107) then dropout
        (base_rbm.py:417-418); in bf16 mode rounded to bf16 like the chain's
        input operand."""
        return self._r(self.prepare_input_fp(X, seed, tick, row0))

    def prepare_input_fp(self, X, seed, tick, row0=0):
        """The prepared batch before any bf16 rounding: what the free energy
        and the PLL read in every mode."""
        X = np.asarray(X, dtype=self.dt)
        if self.v_kind == 'gaussian':
            X = X / self.sigma[None, :]
        keep = self.cfg.get('dropout', None)
        if keep is not None:
            u = P.uniform_at(X.shape[0], X.shape[1], seed, P.SITE_DROPOUT, 0, tick, row0)
            mask = np.floor(np.float32(keep) + u).astype(self.dt)
            X = X / self.dt.type(keep) * mask
        return X

    def chain(self, X, k, seed, tick, row0=0):
        """base_rbm.py:421-426 + :367-384.  X is the prepared batch."""
        c = self.cfg
        h0_means = self.means_h_given_v(X)
        if c.get('sample_h', True):
            h_states = self._sample_h(h0_means, seed, P.SITE_H0, 0, tick, row0)
        else:
            h_states = self._r(h0_means)
        h0_means = self._r(h0_means)
        v_states = v_means = h_means = None
        for t in range(1, int(k) + 1):
            v_means = self.means_v_given_h(h_states)
            if c.get('sample_v', False):
                v_states = self._r(self._sample_v(v_means, seed, P.SITE_V, t, tick, row0))
            else:
                v_states = self._r(v_means)
            v_means = self._r(v_means)
            h_means = self.means_h_given_v(v_states)
            if c.get('sample_h', True) and t < int(k):
                h_states = self._sample_h(h_means, seed, P.SITE_H, t, tick, row0)
            else:
                h_states = self._r(h_means)   # last-step states are never consumed
            h_means = self._r(h_means)
        return h0_means, v_states, v_means, h_states, h_means

    # -- free energies (rbm/rbm.py:17-22, 50-60, 109-116) --------------------
    # In bf16 mode too they read the fp32 W and the unrounded prepared batch: the
    # engine evaluates them on its CUDA-core kernels in fp32, as the reference's
    # graph does (only the chain and MSRE see bf16 operands).
    def free_energy(self, v, seed=0, tick=0, fe_idx=0):
        W = self.p['W']
        if self.h_kind == 'multinomial':
            K, M = self.H, float(self.cfg.get('h_n_samples', 100))
            from math import lgamma
            T1 = -(v @ self.p['vb'])
            T2 = -(v @ W)
            probs = np.full((1, K), 1.0 / K, dtype=np.float32)
            h_hat = multinomial_counts(probs, int(M), seed, P.SITE_MULTINOMIAL_FE, fe_idx, tick)[0]
            T3 = T2 @ h_hat.astype(self.dt)
            fe = np.mean(T1 + T3, dtype=np.float64)
            return float(fe - lgamma(M + K) + lgamma(M + 1) + lgamma(K))
        T_h = -softplus(v @ W + self.p['hb']).sum(axis=1)
        if self.v_kind == 'gaussian':
            T1 = self.p['vb'][None, :] / self.sigma[None, :]
            T3 = 0.5 * np.square(v - T1).sum(axis=1)
            return float(np.mean(T3 + T_h, dtype=np.float64))
        T1 = -(v @ self.p['vb'])
        return float(np.mean(T1 + T_h, dtype=np.float64))

    def pll(self, X, seed, tick, row0=0):
        """base_rbm.py:496-513: flip one random visible per row; V*log_sigmoid of
        the difference of *batch-mean* free energies."""
        rows = X.shape[0]
        idx = (P.site_words(rows, 1, seed, P.SITE_PLL, 0, tick, row0)[:, 0] % np.uint32(self.V)).astype(np.int64)
        Xc = X.copy()
        Xc[np.arange(rows), idx] = 1 - Xc[np.arange(rows), idx]
        d = self.free_energy(Xc, seed, tick, 0) - self.free_energy(X, seed, tick, 1)
        return float(self.V * -np.logaddexp(0.0, -d))

    def _metrics(self, names, X, v_means, seed, tick, row0, X_fp=None):
        """X: the chain's input (MSRE); X_fp: the same batch unrounded (free
        energy, PLL), X itself when not given."""
        X_fp = X if X_fp is None else X_fp
        out = {}
        if 'l2_loss' in names:   # base_rbm.py:482-484
            out['l2_loss'] = float(self.cfg.get('l2', 0.) * 0.5 * np.sum(np.square(self.p['W'], dtype=np.float64)))
        if 'msre' in names:      # :486-488
            out['msre'] = float(np.mean(np.square(X - v_means), dtype=np.float64))
        if 'pll' in names:
            out['pll'] = self.pll(X_fp, seed, tick, row0)
        if 'free_energy' in names:   # :516
            out['free_energy'] = self.free_energy(X_fp, seed, tick, 2)
        return out

    # -- engine interface ----------------------------------------------------
    def train_step(self, X, lr, momentum, k, seed, tick, metrics=(), shard=None):
        """One ``session.run(train_op)`` (base_rbm.py:415-479).  Metrics, when
        requested, see the pre-update parameters.

        ``shard=(rank, nranks, allreduce)`` models the engine's data-parallel mode (no counterpart in
        the single-device reference): X is this rank's slice of a global batch of ``rows * nranks``
        rows, draws are keyed by the global row index, and the four sufficient statistics are
        summed over ranks by ``allreduce(array) -> array`` before the (identical) update."""
        c, p, dt = self.cfg, self.p, self.dt
        rank, nranks, allreduce = shard if shard is not None else (0, 1, None)
        row0 = rank * np.asarray(X).shape[0]
        X_fp = self.prepare_input_fp(X, seed, tick, row0)
        X = self._r(X_fp)
        h0_means, v_states, v_means, _, h_means = self.chain(X, k, seed, tick, row0)
        out = self._metrics(metrics, X, v_means, seed, tick, row0, X_fp) if metrics else None
        self.apply_update(X, h0_means, v_states, h_means, lr, momentum, nranks, allreduce)
        return out

    def apply_update(self, X, h0_means, v_states, h_means, lr, momentum, nranks=1, allreduce=None):
        """Gradients, sparsity and momentum updates of one step from the chain's activations
        (base_rbm.py:443-474).  Separate from ``train_step`` so that full-size tests can apply it to the
        CUDA engine's own activations (a size-independent check of the statistics + update kernels)."""
        c, p, dt = self.cfg, self.p, self.dt
        N = dt.type(X.shape[0] * nranks)
        G = X.T @ h0_means - v_states.T @ h_means
        dvb_sum, dhb_sum, q_sum = (X - v_states).sum(axis=0), (h0_means - h_means).sum(axis=0), h_means.sum(axis=0)
        if allreduce is not None:
            G, dvb_sum, dhb_sum, q_sum = allreduce(G), allreduce(dvb_sum), allreduce(dhb_sum), allreduce(q_sum)
        dW = G / N - dt.type(c.get('l2', 0.)) * p['W']   # :445-449
        dvb = dvb_sum / N                             # :451
        dhb = dhb_sum / N                             # :453
        damp = dt.type(c.get('sparsity_damping', 0.9))
        q = damp * p['q_means'] + (dt.type(1) - damp) * q_sum   # :457-459
        pen = dt.type(c.get('sparsity_cost', 0.)) * (q - dt.type(c.get('sparsity_target', 0.1)))
        p['q_means'] = q.astype(dt)
        dhb = dhb - pen
        dW = dW - pen[None, :]                        # :461-462
        lr, mom = dt.type(lr), dt.type(momentum)
        p['dW'] = (lr * (mom * p['dW'] + dW)).astype(dt)      # :467-474
        p['W'] = (p['W'] + p['dW']).astype(dt)
        p['dvb'] = (lr * (mom * p['dvb'] + dvb)).astype(dt)
        p['vb'] = (p['vb'] + p['dvb']).astype(dt)
        p['dhb'] = (lr * (mom * p['dhb'] + dhb)).astype(dt)
        p['hb'] = (p['hb'] + p['dhb']).astype(dt)

    def transform(self, X, k, seed, tick):
        """base_rbm.py:438-440,687-700: chain-end h_means (E[h|v_k])."""
        Xp = self.prepare_input(X, seed, tick)
        return self.chain(Xp, k, seed, tick)[4]

    def metrics(self, X, k, seed, tick, names):
        """base_rbm.py:573-590 / :592-621 (no parameter update)."""
        X_fp = self.prepare_input_fp(X, seed, tick)
        Xp = self._r(X_fp)
        v_means = None
        if 'msre' in names:
            v_means = self.chain(Xp, k, seed, tick)[2]
        return self._metrics(names, Xp, v_means, seed, tick, 0, X_fp)

    def close(self):
        pass


def rbm_factory(cfg):
    """Engine factory for ``boltzmann_machines.base.set_engine_factory('rbm', ...)``
    -- used by tests to drive the package's host logic on CPU."""
    return OracleRBM(cfg)
