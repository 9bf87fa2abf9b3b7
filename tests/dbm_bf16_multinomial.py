"""bf16 emulation of the tensor-core DBM engine with multinomial hidden layers -- TEST INFRASTRUCTURE ONLY.

`oracle/dbm_bf16.py::OracleDBMbf16` states what the tensor-core engine (csrc/bm_dbm_tc.cuh, compute='bf16') computes for
Bernoulli hidden layers.  This subclass adds multinomial hidden layers (layers.py:54-70), rounding where the engine rounds:

  * the layer's pre-activations acc_scale * (bf16 operands @ bf16 weights) + bias_scale * b in fp32,
  * n_samples * softmax(row) and the categorical draws as the CUDA-core engine's kernels compute them (softmax_rows /
    multinomial_rows in bm_simt.cu, which the engine's fused row kernel reproduces bit for bit): exp in float32, the row sum
    in float64 rounded to float32, probabilities mean / (float64 row sum) rounded to float32, the float64 CDF of
    oracle.rbm.multinomial_counts and the draws of the layer's Philox site,
  * means and counts narrowed to bf16 as GEMM operands (counts above 256 round to 2^-9 relative),

while the fp32 particles of a multinomial layer keep what the row kernel computed -- exact integer counts -- or what the
caller set / initialised, as the engine's get_param('h...') returns them.  Convergence measures of the E-step are recorded as in the base class (mf_diffs).
"""
import numpy as np

from oracle import philox as P
from oracle.dbm import OracleDBM
from oracle.dbm_bf16 import OracleDBMbf16, _r
from oracle.rbm import multinomial_counts


def softmax_rows(pre, scale):
    """softmax_rows_kernel<float>: scale * exp(x - max) / float(sum in float64)."""
    pre = np.asarray(pre, dtype=np.float32)
    m = pre.max(axis=1, keepdims=True)
    with np.errstate(over='ignore', under='ignore'):
        e = np.exp((pre - m).astype(np.float32))
    tot = e.astype(np.float64).sum(axis=1, keepdims=True).astype(np.float32)
    return ((np.float32(scale) * e) / tot).astype(np.float32)


def multinomial_rows(means, n_draws, seed, site, t, tick):
    """multinomial_rows_kernel<float>: probabilities float32(mean / sequential float64 row sum), float64 CDF, first j with
    cdf[j] > u for draw d of row r taken from element (r, d) of the site's uniforms."""
    m64 = np.asarray(means, dtype=np.float32).astype(np.float64)
    tot = np.cumsum(m64, axis=1)[:, -1:]
    probs = (m64 / tot).astype(np.float32)
    return multinomial_counts(probs, int(n_draws), seed, site, t, tick).astype(np.float32)


class OracleDBMbf16Multinomial(OracleDBMbf16):
    def __init__(self, cfg):
        cfg = dict(cfg)
        assert np.dtype(cfg.get('dtype', 'float32')) == np.float32, 'bf16 compute is defined for float32 models'
        OracleDBM.__init__(self, cfg)          # (the base class asserts Bernoulli hidden layers)
        assert all(k in ('bernoulli', 'multinomial') for k in self.h_kinds) and self.v_kind in ('bernoulli', 'gaussian')
        self.exact = {}                        # fp32 particles of multinomial layers where they differ from the bf16 operand
        self._written = {}

    def _multi(self, i):
        return self.h_kinds[i] == 'multinomial'

    def _keep_fp32_particles(self):
        for i in range(self.L):
            if self._multi(i):
                k = 'h' + self._sfx(i)
                self.exact[k] = self.p[k].copy()

    # what the caller sets or initialises is narrowed for the GEMMs; a multinomial layer's fp32 particles keep it as given
    def set_params(self, d):
        OracleDBM.set_params(self, d)
        self._keep_fp32_particles()
        self._narrow_state()

    def init_particles(self, seed):
        OracleDBM.init_particles(self, seed)
        self._keep_fp32_particles()
        self._narrow_state()

    def get_params(self, names=None):
        out = super(OracleDBMbf16Multinomial, self).get_params(names)
        for k, v in self.exact.items():
            if k in out:
                out[k] = v.copy()
        return out

    def _hidden(self, i, below, above, sample, seed, site, t, tick, acc_scale=1., bias_scale=1.):
        if not self._multi(i):
            return super(OracleDBMbf16Multinomial, self)._hidden(i, below, above, sample, seed, site, t, tick, acc_scale, bias_scale)
        T = below @ self.Wb(i)
        if above is not None:
            T = T + above @ self.Wb(i + 1).T
        pre = (np.float32(acc_scale) * T + np.float32(bias_scale) * self.hb(i)).astype(np.float32)
        out = softmax_rows(pre, self.h_n_samples[i])
        if sample:
            out = multinomial_rows(out, int(self.h_n_samples[i]), seed, site, t, tick)
        self._written[i] = out
        return _r(out)

    def particles_update(self, n_steps, sample, seed, tick, t0=0, commit=True):
        self._written = {}
        v, H = super(OracleDBMbf16Multinomial, self).particles_update(n_steps, sample, seed, tick, t0, commit)
        if commit:
            for i, x in self._written.items():
                self.exact['h' + self._sfx(i)] = x
        return v, H

    def log_proba(self, X):
        assert not any(self._multi(i) for i in range(self.L)), 'log_proba is defined for binary hidden layers'
        return super(OracleDBMbf16Multinomial, self).log_proba(X)

    def _ais(self, n_runs, n_betas, k, seed):
        assert not any(self._multi(i) for i in range(self.L)), 'AIS is defined for binary hidden layers'
        return super(OracleDBMbf16Multinomial, self)._ais(n_runs, n_betas, k, seed)
