"""The AIS replay (tests/test_zz_dbm_ais_replay_gpu.py) without a GPU: its float64 ladder is pinned against the committed
float64 oracle at the benchmark's shape and against exact enumeration, and its checker, fed stand-in engines, accepts the
numpy oracles and rejects each mutation of the ladder below wherever the mutation changes a run by more than the bound.

The stand-in (`standin`) is the ladder as the tensor-core engine arranges it -- fp32 pre-activations from bf16 weights, the
increment of x_j taken with the first sweep of transition j + 1, the linear term with the transition that draws the state --
so that each mutation is one wrong index, site or temperature of that arrangement."""
import json
import os

import numpy as np
import pytest

from oracle import philox as P
from oracle.dbm import OracleDBM
from oracle.dbm_bf16 import OracleDBMbf16, softplus_diff
from oracle.rbm import bf16_round
from test_zz_dbm_ais_replay_gpu import (ENGINES, REPORT, Engine, Model, chain, check_runs, dbm_cfg, increments, params, softplus,
                                        temperatures)

HERE = os.path.dirname(os.path.abspath(__file__))
# the float32 numpy oracle rounds beta z before each softplus (one fp32 rounding per evaluation, not per difference)
ENGINES['oracle-fp32'] = Engine('oracle-fp32', 2.0 ** -24, 2.0 ** -21, ENGINES['fp32'].weights, np.float32, False, prod=2.0 ** -24)

SHAPE = (30, (18, 11))


def standin(prm, n_runs, n_betas, k, seed, first_run=0, mutation=None, flip=None):
    """log Z estimates of runs [first_run, first_run + n_runs); `flip` = (run, transition, sweep, site, unit) inverts one draw"""
    f = np.float32
    W0, W1 = bf16_round(prm['W'].astype(f)), bf16_round(prm['W_1'].astype(f))
    b, c1, c2 = prm['vb'].astype(f), prm['hb'].astype(f), prm['hb_1'].astype(f)
    t = [f(x) for x in temperatures(n_betas, np.float64 if mutation == 'beta in float64' else np.float32)]
    inc = increments(t)
    n = len(t)
    row_init = 0 if mutation == 'first_run ignored' else first_run
    row = 0 if mutation in ('first_run ignored', 'first_run at the init site only') else first_run
    site_v, site_h2 = P.SITE_AIS_V, P.SITE_AIS_H2
    if mutation == 'v and h2 sites swapped':
        site_v, site_h2 = site_h2, site_v

    def draw(z, site, tick, r0, addr):
        with np.errstate(over='ignore'):
            p = f(1) / (f(1) + np.exp(-z))
        s = P.uniform_at(n_runs, z.shape[1], seed, site, 0, tick, r0) < p
        if flip is not None and flip[1:4] == addr:
            s[flip[0] - first_run, flip[4]] ^= True
        return s.astype(f)

    def weigh(x, a, b_):
        pa, pb = (x @ W0.T + b).astype(f), (x @ W1 + c2).astype(f)
        return softplus_diff(a, b_, pa).astype(np.float64).sum(axis=1) + softplus_diff(a, b_, pb).astype(np.float64).sum(axis=1)

    x = (P.uniform_at(n_runs, W0.shape[1], seed, P.SITE_AIS_INIT, 0, 0, row_init) < f(0.5)).astype(f)
    logw = np.zeros(n_runs)
    for j in range(n):
        for s in range(k):
            tick = {'tick + 1': j * k + s + 1, 'tick without k': j + s}.get(mutation, j * k + s)
            if j >= 1 and (s == 0 or mutation == 'weighs on every sweep'):
                a, b_ = inc[j if mutation == 'increments one temperature late' else j - 1]
                if not (mutation == 'no increment at every 30th temperature' and j % 30 == 0):
                    logw += weigh(x, a, b_)
            pa, pb = (x @ W0.T + b).astype(f), (x @ W1 + c2).astype(f)
            v = draw(t[j] * pa, site_v, tick, row, (j, s, P.SITE_AIS_V))
            h2 = draw(t[j] * pb, site_h2, tick, row, (j, s, P.SITE_AIS_H2))
            x = draw(t[j] * (v @ W0 + h2 @ W1.T).astype(f) + t[j] * c1, P.SITE_AIS_H1, tick, row, (j, s, P.SITE_AIS_H1))
            if s == k - 1 and mutation != 'linear term dropped':
                a, b_ = inc[j]
                coef = np.float64(t[j]) if mutation == 'linear term at beta' else np.float64(b_) - np.float64(a)
                logw += coef * (x @ c1).astype(np.float64)
    a, b_ = inc[n - 1]
    logw += weigh(x, a, t[n - 1] if mutation == 'last increment at the last beta' else b_)
    if mutation != 'log Z_0 omitted':
        logw += (W0.shape[0] + W0.shape[1] + W1.shape[1]) * float(f(np.log(2.)))
    return logw


CALLS = {'k1': dict(n_runs=24, n_betas=60, k=1, seed=11, first_run=40),
         'k2': dict(n_runs=24, n_betas=60, k=2, seed=12, first_run=40)}
MUTATIONS = {          # mutation: the calls where it changes a run by more than the bound
    'tick + 1': ('k1', 'k2'),
    'tick without k': ('k2',),
    'v and h2 sites swapped': ('k1', 'k2'),
    'first_run ignored': ('k1', 'k2'),
    'first_run at the init site only': ('k1', 'k2'),
    'increments one temperature late': ('k1', 'k2'),
    'linear term dropped': ('k1', 'k2'),
    'linear term at beta': ('k1', 'k2'),
    'no increment at every 30th temperature': ('k1', 'k2'),
    'weighs on every sweep': ('k2',),
    'log Z_0 omitted': ('k1', 'k2'),
}
BELOW_THE_BOUND = {
    ('tick without k', 'k1'): 'k = 1: the same ticks',
    ('weighs on every sweep', 'k1'): 'k = 1: one sweep',
    ('last increment at the last beta', 'k1'): 'the accumulated float32 beta ends within 1e-6 of 1 at 60 temperatures',
    ('last increment at the last beta', 'k2'): 'the accumulated float32 beta ends within 1e-6 of 1 at 60 temperatures',
    ('beta in float64', 'k1'): 'float32(float64 recurrence) differs from the float32 recurrence by an ulp of beta: 1e-7 of a term',
    ('beta in float64', 'k2'): 'as for k = 1',
}


@pytest.fixture(scope='module')
def small():
    prm = params(*SHAPE, scale=0.4, bias=0.5, grid=5)
    return prm, Model(prm)


def run_standin(small, call, mutation=None):
    prm, m = small
    c = CALLS[call]
    got = standin(prm, mutation=mutation, **c)
    return check_runs(m, c['n_betas'], c['k'], c['seed'], c['first_run'], got, call + (': ' + mutation if mutation else ''))


@pytest.mark.parametrize('call', list(CALLS))
def test_checker_accepts_the_standin(small, call):
    assert small[1].exact
    run_standin(small, call)


@pytest.mark.parametrize('mutation,call', [(m_, c) for m_, where in MUTATIONS.items() for c in where])
def test_checker_rejects_the_mutation(small, mutation, call):
    with pytest.raises(AssertionError):
        run_standin(small, call, mutation)


@pytest.mark.parametrize('mutation,call', list(BELOW_THE_BOUND))
def test_mutations_below_the_bound_are_listed_not_forced(small, mutation, call):
    """what the replay cannot see at these calls, stated: the mutated stand-in is accepted"""
    run_standin(small, call, mutation)


def test_last_increment_at_the_last_beta_is_seen_where_the_recurrence_ends_off_one(small):
    """a ladder whose accumulated float32 beta ends 1e-5 away from 1: weighing the last state at it instead of at 1.0 moves a
    run by that much of sum z sigmoid(z), which the replay sees once the pre-activations are wide"""
    shape = (64, (48, 40))
    prm = params(*shape, scale=1.0, bias=1.0, grid=4)
    m = Model(prm)
    n_betas = max(range(900, 1100), key=lambda n: abs(1.0 - float(temperatures(n, np.float32)[-1])))
    assert abs(1.0 - float(temperatures(n_betas, np.float32)[-1])) > 5e-6
    check_runs(m, n_betas, 1, 3, 0, standin(prm, 4, n_betas, 1, 3), 'off-one ladder')
    with pytest.raises(AssertionError):
        check_runs(m, n_betas, 1, 3, 0, standin(prm, 4, n_betas, 1, 3, mutation='last increment at the last beta'), 'off-one ladder')


# ---- the numpy oracles as engines --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['bf16', 'oracle-fp32', 'float64'])
@pytest.mark.parametrize('k', [1, 3])
def test_checker_accepts_the_numpy_oracles(kind, k):
    dtype = 'float64' if kind == 'float64' else 'float32'
    cfg = dbm_cfg(*SHAPE, compute='bf16' if kind == 'bf16' else 'fp32', dtype=dtype)
    prm = params(*SHAPE, scale=0.4, bias=0.5, grid=5 if kind != 'float64' else None)
    ora = (OracleDBMbf16 if kind == 'bf16' else OracleDBM)(cfg)
    ora.set_params({n: np.asarray(v, dtype) for n, v in prm.items()})
    m = Model(prm, cfg['compute'], dtype)
    if kind == 'oracle-fp32':
        m.engine = ENGINES[kind]
    got = ora.ais(16, 40, k, 5, first_run=7)
    check_runs(m, 40, k, 5, 7, got, kind + ' oracle')


def test_replay_reproduces_the_float64_oracle_at_the_benchmark_shape():
    """784-512-1024 x 1000 betas, the parameters of tests/golden/make_ais_benchmark_oracle.py (non-zero biases), identity
    weights and the float64 recurrence: the first runs of the committed float64 oracle to round-off"""
    import sys
    sys.path.insert(0, os.path.join(HERE, 'golden'))
    try:
        import make_ais_benchmark_oracle as G
    finally:
        sys.path.pop(0)
    fx = json.load(open(os.path.join(HERE, 'golden', 'ais_benchmark_shape_oracle.json')))
    sh = fx['shape']
    m = Model(G.weights(), 'fp32', 'float64')
    ref = chain(m, sh['n_betas'], sh['n_gibbs_steps'], sh['seed'], 0, 3)
    np.testing.assert_allclose(ref.logw, fx['log_weights'][:3], rtol=0, atol=1e-8)
    assert ref.bound.max() < 1e-7
    one = chain(m, sh['n_betas'], sh['n_gibbs_steps'], sh['seed'], 2, 1)             # a run replayed on its own
    np.testing.assert_allclose(one.logw[0], fx['log_weights'][2], rtol=0, atol=1e-8)


def test_replay_estimates_the_enumerated_log_Z():
    """7-5-4: the log-mean-exp of the float64 ladder's runs against log Z by enumeration of the 32 states of h_1"""
    m = Model(params(7, (5, 4), scale=0.5, bias=0.5, grid=5))
    ref = chain(m, 200, 1, 3, 0, 256)
    x = ((np.arange(2 ** 5)[:, None] >> np.arange(5)[None, :]) & 1).astype(np.float64)
    zv, zh = x @ m.W0.B.T + m.b, x @ m.W1.B + m.c2
    logZ = np.logaddexp.reduce(x @ m.c1 + softplus(zv).sum(axis=1) + softplus(zh).sum(axis=1))
    est = np.logaddexp.reduce(ref.logw) - np.log(256)
    assert abs(est - logZ) < 0.1, (est, logZ)


# ---- forks -----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def loose():
    """weights off the grid: the draws' tolerance carries the accumulator's worst case, so some draws lie within it"""
    prm = params(*SHAPE, scale=0.4, bias=0.5, grid=None)
    m = Model(prm)
    assert not m.exact
    return prm, m


def test_a_draw_flipped_inside_its_tolerance_is_accepted_and_counted(loose):
    prm, m = loose
    c = dict(CALLS['k2'], n_runs=192)
    ref = chain(m, c['n_betas'], c['k'], c['seed'], c['first_run'], c['n_runs'])
    got0 = standin(prm, **c)
    for r in (r for r in range(c['n_runs']) if ref.near[r]):          # a run with a draw within tolerance whose flip moves it
        addr = ref.near[r][0][2]
        got = standin(prm, flip=(c['first_run'] + r,) + addr, **c)
        if abs(got[r] - ref.logw[r]) > ref.bound[r]:
            break
    else:
        raise AssertionError('no draw within its tolerance among {0} runs'.format(c['n_runs']))
    np.testing.assert_array_equal(np.delete(got, r), np.delete(got0, r))
    before = REPORT['forked']
    assert check_runs(m, c['n_betas'], c['k'], c['seed'], c['first_run'], got, 'flip inside') == 1
    assert REPORT['forked'] == before + 1


def test_a_draw_flipped_outside_its_tolerance_is_rejected(loose):
    prm, m = loose
    c = CALLS['k2']
    ref = chain(m, c['n_betas'], c['k'], c['seed'], c['first_run'], c['n_runs'])
    near = set(a for _, _, a in ref.near[0])
    addr = next(a for a in ((3, 1, P.SITE_AIS_H1, u) for u in range(SHAPE[1][0])) if a not in near)
    got = standin(prm, flip=(c['first_run'],) + addr, **c)
    assert abs(got[0] - ref.logw[0]) > ref.bound[0]
    with pytest.raises(AssertionError, match='run {0}'.format(c['first_run'])):
        check_runs(m, c['n_betas'], c['k'], c['seed'], c['first_run'], got, 'flip outside')
