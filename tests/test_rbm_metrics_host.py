"""Negative controls of the RBM metrics checks (tests/test_zz_rbm_metrics_gpu.py): its checkers, fed the numpy oracle
(oracle/rbm.py, in float64, emulating the bf16 engine's roundings where the case asks for compute='bf16') as a stand-in engine,
accept the oracle's metrics and reject each mutation below at the cases where the mutation changes the result.  The cases
are the GPU file's small ones (130-70 at batch 65, a 37-21 model with batches above max_batch; Gaussian visibles with sigma in
{0.5, 1, 2}; multinomial hidden units), its exactness probes included."""
import numpy as np
import pytest

from oracle import philox as P
from oracle.rbm import OracleRBM
from test_zz_rbm_metrics_gpu import check_epoch, run_case, run_epoch


class StandIn(OracleRBM):
    """the oracle as an engine: exports the chain's input and visible means, runs train_step_at / train_epoch, and applies
    one mutation of the metrics' definition"""

    def __init__(self, cfg, mutation=None):
        super(StandIn, self).__init__(cfg)
        self.mutation = mutation
        self.act = {}
        self.data = None

    def get_activation(self, name, rows):
        a = self.act[name]
        assert a.shape[0] == rows
        return a

    def chain(self, X, k, seed, tick, row0=0):
        out = super(StandIn, self).chain(X, k, seed, tick, row0)
        self.act = dict(X=X, v_means=out[2])
        return out

    def set_data(self, X):
        self.data = np.array(X)

    def train_step_at(self, first_row, rows, lr, momentum, k, seed, tick, metrics=()):
        if self.mutation == 'pll-row0-first-row':
            self._row0 = first_row
        try:
            return self.train_step(self.data[first_row:first_row + rows], lr, momentum, k, seed, tick, metrics)
        finally:
            self._row0 = None

    _row0 = None

    def train_step(self, X, lr, momentum, k, seed, tick, metrics=()):
        if self.mutation != 'after-update' or not metrics:
            return super(StandIn, self).train_step(X, lr, momentum, k, seed, tick, metrics)
        X_fp = self.prepare_input_fp(X, seed, tick)
        Xr = self._r(X_fp)
        h0, v_states, v_means, _, h_means = self.chain(Xr, k, seed, tick)
        self.apply_update(Xr, h0, v_states, h_means, lr, momentum)
        return self._metrics(metrics, Xr, v_means, seed, tick, 0, X_fp)

    def train_epoch(self, X, batch, lr, momentum, k, seed, tick0, metrics=(), every=0, iter0=0):
        nb = (X.shape[0] + batch - 1) // batch
        vals = [self.train_step(X[i * batch:(i + 1) * batch], lr, momentum, k, seed, tick0 + i, metrics) for i in range(nb)]
        rep = [i for i in range(nb) if every and (iter0 + i + 1) % every == 0]
        if self.mutation == 'epoch-shift':
            rep = [i + 1 if i + 1 < nb else i - 1 for i in rep]
        return {m: [vals[i][m] for i in rep] for m in metrics}

    def _metrics(self, names, X, v_means, seed, tick, row0, X_fp=None):
        if self.mutation == 'fe-bf16-input':
            X_fp = X
        if self._row0 is not None:
            row0 = self._row0
        out = super(StandIn, self)._metrics(names, X, v_means, seed, tick, row0, X_fp)
        if self.mutation == 'msre-rows-ldv' and 'msre' in out:
            out['msre'] *= self.V / float((self.V + 63) // 64 * 64 + 64)       # divided by rows * ldv instead of rows * V
        return out

    def free_energy(self, v, seed=0, tick=0, fe_idx=0):
        if self.mutation == 'fe-idx-swap':
            fe_idx = {0: 1, 1: 0}.get(fe_idx, fe_idx)
        if self.mutation == 'fe-bf16-W':
            W = self.p['W']
            self.p['W'] = self._Wc()
            try:
                return super(StandIn, self).free_energy(v, seed, tick, fe_idx)
            finally:
                self.p['W'] = W
        return super(StandIn, self).free_energy(v, seed, tick, fe_idx)

    def pll(self, X, seed, tick, row0=0):
        m = self.mutation
        if m not in ('pll-site', 'pll-row0+1', 'pll-tick+1', 'pll-mod-V+1'):
            return super(StandIn, self).pll(X, seed, tick, row0)
        rows = X.shape[0]
        site = P.SITE_PLL + 1 if m == 'pll-site' else P.SITE_PLL
        row0 = row0 + 1 if m == 'pll-row0+1' else row0
        tick = tick + 1 if m == 'pll-tick+1' else tick
        mod = self.V + 1 if m == 'pll-mod-V+1' else self.V
        idx = (P.site_words(rows, 1, seed, site, 0, tick, row0)[:, 0] % np.uint32(mod)).astype(np.int64)
        Xc = X.copy()
        r = np.flatnonzero(idx < self.V)                 # (the engine's kernel flips nothing in a row whose index is V)
        Xc[r, idx[r]] = 1 - Xc[r, idx[r]]
        d = self.free_energy(Xc, seed, tick, 0) - self.free_energy(X, seed, tick, 1)
        return float(self.V * -np.logaddexp(0.0, -d))


def standin(mutation=None):
    return lambda cfg: StandIn(cfg, mutation)


def run(case, mutation=None):
    shape, probe, compute = case
    if probe == 'epoch':
        run_epoch(shape, compute, dtype='float64', make=standin(mutation))
    else:
        run_case(shape, probe, compute, dtype='float64', make=standin(mutation))


CASES = [(s, p, c) for s, p in [('small', 'bench'), ('small', 'w0'), ('small', 'dyadic'), ('small', 'bf16w'),
                                 ('small-ragged', 'bench'), ('small-ragged', 'w0'), ('small-gauss', 'bench'),
                                 ('small-gauss', 'gauss-x'), ('small-multi', 'dyadic')]
         for c in ('bf16', 'fp32')] + [('small', 'epoch', 'bf16'), ('small', 'epoch', 'fp32')]
MUTATIONS = {          # mutation: the cases that must reject it
    'pll-site': [('small', 'w0', 'fp32'), ('small', 'w0', 'bf16'), ('small-ragged', 'w0', 'bf16')],
    'pll-row0+1': [('small', 'w0', 'fp32'), ('small', 'w0', 'bf16'), ('small-ragged', 'w0', 'bf16')],
    'pll-row0-first-row': [('small', 'w0', 'fp32'), ('small-ragged', 'w0', 'bf16')],        # PLL keyed by the dataset row
    'pll-tick+1': [('small', 'w0', 'fp32'), ('small', 'w0', 'bf16'), ('small-ragged', 'w0', 'bf16')],
    'pll-mod-V+1': [('small', 'w0', 'fp32'), ('small', 'w0', 'bf16'), ('small-ragged', 'w0', 'bf16')],
    'fe-bf16-W': [('small', 'bf16w', 'bf16')],
    'fe-bf16-input': [('small-gauss', 'gauss-x', 'bf16')],
    'after-update': [('small', 'dyadic', 'bf16'), ('small', 'bench', 'fp32'), ('small-multi', 'dyadic', 'fp32')],
    'msre-rows-ldv': [('small', 'bench', 'bf16'), ('small-ragged', 'bench', 'fp32')],
    'fe-idx-swap': [('small-multi', 'dyadic', 'bf16'), ('small-multi', 'dyadic', 'fp32')],
    'epoch-shift': [('small', 'epoch', 'bf16'), ('small', 'epoch', 'fp32')],
}


@pytest.mark.parametrize('case', CASES, ids=['-'.join(c) for c in CASES])
def test_checker_accepts_the_oracle(case):
    run(case)


@pytest.mark.parametrize('mutation,case', [(m, c) for m, cs in MUTATIONS.items() for c in cs],
                         ids=['{0}:{1}'.format(m, '-'.join(c)) for m, cs in MUTATIONS.items() for c in cs])
def test_checker_rejects_the_mutation(mutation, case):
    with pytest.raises(AssertionError):
        run(case, mutation)


def test_epoch_checker_sees_a_shifted_report():
    """check_epoch compares values, not only their count"""
    loop = [{n: float(i) for n in ('l2_loss', 'msre', 'free_energy', 'pll')} for i in range(4)]
    check_epoch({n: [0.0, 2.0] for n in loop[0]}, loop, [0, 2], 'unshifted')
    with pytest.raises(AssertionError):
        check_epoch({n: [1.0, 3.0] for n in loop[0]}, loop, [0, 2], 'shifted')
