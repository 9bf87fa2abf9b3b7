"""Negative controls of the tensor-core DBM replay (tests/test_zz_dbm_tc_replay_gpu.py): its checkers, fed the bf16 emulation
(oracle/dbm_bf16.py) as a stand-in engine at the sizes and learning rates of the GPU cases, accept the emulation's outputs and
reject each mutation below wherever the mutation is materially present.

Where a mutation is not present at a case's values it is not run there (NOT_PRESENT states why); the ragged case
(batch_size 1024 != n_particles 1100, 1000 rows, Gaussian visibles, a mean-valued middle layer) exists for those."""
import functools

import numpy as np
import pytest

from oracle import philox as P
from oracle.dbm_bf16 import OracleDBMbf16
from test_tc_kernel_exact_gpu import bf16r
from test_zz_dbm_tc_replay_gpu import (CASES, Conditionals, check_estep, check_mstep, check_particle_sweep, check_zero_sweeps,
                                       particles, pinned_stale, sfx)


class StandIn(OracleDBMbf16):
    """the emulation as an engine: the column norm of max-norm in double, as colnorm_kernel takes it, and optional mutations of
    the E-step and the particle sweeps"""

    def __init__(self, cfg, mutation=None):
        super(StandIn, self).__init__(cfg)
        self.mutation = mutation

    def _max_norm(self, T):
        n = np.sqrt(np.square(T.astype(np.float64)).sum(axis=0)).astype(np.float32)
        mn = np.float32(self.cfg.get('max_norm', np.inf))
        return (T * np.minimum(n, mn) / np.maximum(n, np.float32(1e-8))).astype(np.float32)

    def _hidden(self, i, below, above, sample, seed, site, t, tick, acc_scale=1., bias_scale=1.):
        if self.mutation == 'approx-without-x2' and acc_scale == 2.:
            acc_scale = 1.
        return super(StandIn, self)._hidden(i, below, above, sample, seed, site, t, tick, acc_scale, bias_scale)

    def _visible(self, h0, sample, seed, site, t, tick):
        if self.mutation == 'v-at-site-h' and site == P.SITE_DBM_V:
            site = P.SITE_DBM_H
        return super(StandIn, self)._visible(h0, sample, seed, site, t, tick)

    def gibbs_step(self, v, H, update_v, sample, seed, t, tick):
        v_new, Hn = super(StandIn, self).gibbs_step(v, H, update_v, sample, seed, t, tick)
        if self.mutation == 'above-from-new-sweep' and not update_v:          # a mean-field sweep: layer i reads layer i+1 new
            for i in range(self.L - 1):
                below = v if i == 0 else Hn[i - 1]
                Hn[i] = self._hidden(i, below, Hn[i + 1], False, seed, 0, t, tick)
        return v_new, Hn


def mstep_fp32(cfg, before, X, after, lr, mom, mutation=None):
    """the stand-in's M-step (OracleDBMbf16.train_step) restated in fp32 with a mutation; returns the variables it writes"""
    f = np.float32
    L = len(cfg['n_hiddens'])
    B, M, rows = f(cfg['batch_size']), f(cfg['n_particles']), f(X.shape[0])
    n_div, m_div = {'swap-divisors': (M, B), 'rows-for-dW': (rows, M)}.get(mutation, (B, M))
    mu = [after['mu' + sfx(i)][:X.shape[0]] for i in range(L)]
    H = [after['h' + sfx(i)] for i in range(L)]
    v = after['v']
    lr, mom = f(lr), f(0.0 if mutation == 'no-momentum' else mom)
    l2, damp = f(cfg.get('l2', 0.)), f(cfg.get('sparsity_damping', 0.9))
    out = {}
    out['dvb'] = (lr * (mom * before['dvb'] + (X.sum(axis=0) / rows - v.sum(axis=0) / M))).astype(f)
    out['vb'] = (before['vb'] + out['dvb']).astype(f)
    pos, neg = [bf16r(X).astype(f)] + mu[:-1], [v] + H[:-1]
    for i in range(L):
        s = sfx(i)
        G = (pos[i].T @ mu[i]) * (f(1) / n_div) - (neg[i].T @ H[i]) * (f(1) / m_div)
        if mutation == 'G-scale' and i == L - 1:
            G = G * f(1.01)
        qv, mv = H[i].sum(axis=0), mu[i].sum(axis=0)
        if mutation != 'penalty-per-unit':
            qv, mv = qv[i], mv[i]
        q = (damp * before['q_means' + s] + (f(1) - damp) * qv).astype(f)
        m = (damp * before['mu_means' + s] + (f(1) - damp) * mv).astype(f)
        cost, target = f(cfg['sparsity_cost'][i]), f(cfg['sparsity_target'][i])
        pen = cost * (q - target) + cost * (m - target)
        if mutation == 'no-penalty':
            pen = np.zeros_like(pen)
        out['q_means' + s], out['mu_means' + s] = q, m
        out['dW' + s] = (lr * (mom * before['dW' + s] + (G - l2 * before['W' + s] - pen[None, :]))).astype(f)
        W = (before['W' + s] + out['dW' + s]).astype(f)
        if mutation != 'no-max-norm':
            n = np.sqrt(np.square(W.astype(np.float64)).sum(axis=0)).astype(f)
            W = (W * np.minimum(n, f(cfg['max_norm'])) / np.maximum(n, f(1e-8))).astype(f)
        out['W' + s] = W
        out['dhb' + s] = (lr * (mom * before['dhb' + s] + (mu[i].sum(axis=0) / rows - H[i].sum(axis=0) / M - pen))).astype(f)
        out['hb' + s] = (before['hb' + s] + out['dhb' + s]).astype(f)
    return dict(after, **out)


@functools.lru_cache(maxsize=None)
def case(name):
    c = CASES[name]()
    if name == 'cfg5-pcd':
        raise ValueError('cfg5-pcd is not a host case')
    return c


@functools.lru_cache(maxsize=None)
def standin_step(name, mutation=None):
    """(before, after) of one PCD-1 train_step of the stand-in from the case's restored state"""
    c = case(name)
    emu = StandIn(c['cfg'], mutation)
    emu.set_params(c['init'])
    before = emu.get_params()
    emu.train_step(c['X'], c['lr'], c['mom'], 1, c['seed'], c['tick'])
    return before, emu.get_params()


def standin_sweeps(c, J, mutation=None):
    L = len(c['cfg']['n_hiddens'])
    out = []
    for j in range(J + 1):
        emu = StandIn(dict(c['cfg'], max_mf_updates=j, mf_tol=-1.0), mutation)
        emu.set_params(c['init'])
        emu.mean_field(c['X'])
        out.append([emu.get_params(['mu' + sfx(i)])['mu' + sfx(i)] for i in range(L)])
    return out


def standin_stops(c, state, mf_tol, mutation=None):
    emu = StandIn(dict(c['cfg'], max_mf_updates=25, mf_tol=mf_tol), mutation)
    emu.set_params(state)
    return emu.mean_field(c['X'])


# ---- each checker on the stand-in, then on each mutation ------------------------------------------------------------------------
def run_estep(name, mutation=None):
    c = case(name)
    L = len(c['cfg']['n_hiddens'])
    stale = [c['init']['mu' + sfx(i)] for i in range(L)]
    check_estep(Conditionals(c['cfg'], c['init']), c['X'], stale, standin_sweeps(c, 2, mutation), name)


def run_zero_sweeps(name, mutation=None):
    c = case(name)
    L = len(c['cfg']['n_hiddens'])
    pinned, tol_stop, tol_go = pinned_stale(Conditionals(c['cfg'], c['init']), c['X'], [c['init']['mu' + sfx(i)] for i in range(L)])
    state = dict(c['init'], **{'mu' + sfx(i): pinned[i] for i in range(L)})
    check_zero_sweeps(standin_stops(c, state, tol_stop, mutation), standin_stops(c, state, tol_go, mutation), name)


def run_particles(name, mutation=None):
    c = case(name)
    L = len(c['cfg']['n_hiddens'])
    before, after = standin_step(name, mutation)
    check_particle_sweep(Conditionals(c['cfg'], before), particles(before, L), particles(after, L), c['seed'], c['tick'], 1, name)


def run_mstep(name, mutation=None):
    c = case(name)
    before, after = standin_step(name)
    if mutation is not None:
        after = mstep_fp32(c['cfg'], before, c['X'], after, c['lr'], c['mom'], mutation)
    check_mstep(c['cfg'], before, c['X'], after, c['lr'], c['mom'], name)


HOST_CASES = ('cfg4', 'cfg4-maxnorm', 'ragged')
CHECKS = {'E-step': run_estep, 'zero sweeps': run_zero_sweeps, 'particles': run_particles, 'M-step': run_mstep}
MUTATIONS = {          # mutation: (the checker that must reject it, the cases where it is materially present)
    'swap-divisors': ('M-step', ('ragged',)),                       # dW with n_particles and batch_size swapped
    'rows-for-dW': ('M-step', ('ragged',)),                         # the rows present instead of batch_size for dW
    'no-penalty': ('M-step', ('cfg4', 'ragged')),
    'penalty-per-unit': ('M-step', ('cfg4', 'ragged')),             # unit j's own sums instead of element `layer`
    'no-max-norm': ('M-step', ('cfg4-maxnorm',)),
    'no-momentum': ('M-step', ('cfg4', 'cfg4-maxnorm', 'ragged')),
    'G-scale': ('M-step', ('cfg4', 'ragged')),                      # a 1 % scale error in G of the top layer
    'approx-without-x2': ('zero sweeps', ('cfg4', 'ragged')),
    'above-from-new-sweep': ('E-step', ('cfg4', 'ragged')),
    'v-at-site-h': ('particles', ('cfg4', 'ragged')),
}
NOT_PRESENT = {
    ('swap-divisors', 'cfg4'): 'batch_size == n_particles == 1024',
    ('rows-for-dW', 'cfg4'): 'the batch has batch_size rows',
    ('no-max-norm', 'cfg4'): 'W ~ 0.02: no column norm comes near max_norm = 6',
    ('no-max-norm', 'ragged'): 'W ~ 0.05: no column norm comes near max_norm = 6',
}


def test_not_present_list_is_complete():
    for m, (_, where) in MUTATIONS.items():
        for n in HOST_CASES:
            if n not in where and n != 'cfg4-maxnorm':
                assert (m, n) in NOT_PRESENT, (m, n)


@pytest.mark.parametrize('check', list(CHECKS))
@pytest.mark.parametrize('name', HOST_CASES)
def test_checker_accepts_the_emulation(name, check):
    CHECKS[check](name)


@pytest.mark.parametrize('mutation,name', [(m, n) for m, (_, where) in MUTATIONS.items() for n in where])
def test_checker_rejects_the_mutation(mutation, name):
    with pytest.raises(AssertionError):
        CHECKS[MUTATIONS[mutation][0]](name, mutation)


def test_unmutated_restatement_is_the_emulation():
    """mstep_fp32 without a mutation writes what the stand-in wrote (so each mutation differs from the emulation only by itself)"""
    c = case('cfg4-maxnorm')
    before, after = standin_step('cfg4-maxnorm')
    again = mstep_fp32(c['cfg'], before, c['X'], after, c['lr'], c['mom'])
    for k, v in after.items():
        np.testing.assert_allclose(again[k], v, rtol=2e-6, atol=1e-9, err_msg=k)
