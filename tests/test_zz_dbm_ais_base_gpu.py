"""AIS log Z from a base-rate model (DESIGN.md §5.4d, DbmTC::ais_local_layers with a base) on the H100: exact enumeration at
L = 1..4, the bf16 emulation run by run (tests/dbm_ais_base_oracle.py), the AIS epilogues with a base vector on the edge operands
of test_tc_kernel_exact_gpu.py, a float64 replay at cfg4's shape with a data-like base, and a zero base at L = 2 against
ais_local."""
import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P

import dbm_ais_base_oracle as B
import dbm_ais_depth_oracle as A
from test_tc_kernel_exact_gpu import (EDGES, ULP, assert_f32_within, assert_guards, bf16_bits_to_f64, check_bernoulli,
                                      edge_operands, product, sigmoid_tol, softplus)
from test_zz_dbm_ais_depth_gpu import AIS_FAR, AIS_LADDER, bf16_params, engine, lm, params

pytestmark = pytest.mark.gpu

SHAPES = {1: (7, (5,)), 2: (6, (5, 4)), 3: (6, (5, 4, 3)), 4: (5, (4, 4, 3, 3))}


def bases(prm, seed):
    rng = np.random.RandomState(seed)
    return [(rng.randn(n) - (1.5 if j == 0 else 0.3)).astype(np.float32) for j, n in enumerate(A.widths(prm))]


# ---- exact enumeration and the emulation -------------------------------------------------------------------------------------
@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('L', [1, 2, 3, 4])
def test_ais_from_a_base_matches_exact_enumeration(L, k):
    """the tolerances of test_zz_dbm_ais_depth_gpu.py::test_ais_matches_exact_enumeration"""
    V, Hs = SHAPES[L]
    n_betas = 240 if k == 1 else 120
    p = params(V, Hs, seed=L)
    base = bases(p, L)
    e = engine(V, Hs, p)
    a = e.ais(32, n_betas, k, 2222, base=base)
    b = B.ais(p, 32, n_betas, k, 2222, base=base, bf16=True)
    assert abs(lm(a) - lm(b)) < 0.1
    assert np.mean(np.abs(a - b) < 2e-3) > 0.8
    exact = A.exact_log_Z(bf16_params(p))
    assert abs(lm(a) - exact) < 0.15, (lm(a), exact)
    e.close()


@pytest.mark.parametrize('which', ['v', 'all'])
@pytest.mark.parametrize('L', [1, 2, 3])
@pytest.mark.parametrize('n_betas', [60, 500])
def test_runs_match_the_emulation(L, which, n_betas):
    V, Hs = {1: (37, (21,)), 2: (29, (19, 11)), 3: (13, (21, 9, 6))}[L]
    p = params(V, Hs, scale=0.5, seed=20 + L)
    base = bases(p, 30 + L)
    if which == 'v':
        base = [base[0]] + [None] * L
    e = engine(V, Hs, p)
    a, b = e.ais(24, n_betas, 1, 41, base=base), B.ais(p, 24, n_betas, 1, 41, base=base, bf16=True)
    assert np.mean(np.abs(a - b) < 2e-3) >= 0.75, np.abs(a - b)
    assert abs(np.mean(a) - np.mean(b)) < 0.05
    e.close()


# ---- the epilogues with a base vector ---------------------------------------------------------------------------------------
def base_of(N, edge):
    return np.random.RandomState(100 + edge).uniform(-4.0, 2.0, N).astype(np.float32)


@pytest.mark.parametrize('edge', [i for i, e in enumerate(EDGES) if (e['bn'] or 0) <= 128])
@pytest.mark.parametrize('temps,mode', [(AIS_LADDER, 'AIS_UNITS'), (AIS_FAR, 'AIS_UNITS_G')], ids=['series', 'closed'])
def test_units_op_with_a_base(edge, temps, mode):
    """u = A B^T + (b - a); logw[m] += sum_n softplus(b' u + a) - softplus(a' u + a); states ~ sigmoid(next u + a)"""
    e = EDGES[edge]
    M, N = e['M'], e['N']
    A1, B1, a_t, b_t, _, bias = edge_operands(e, edge)
    rng = np.random.RandomState(edge)
    A1 = A1 * (rng.rand(*A1.shape) < 0.5)
    a0 = base_of(N, edge)
    u = product(A1, B1, a_t, b_t) + np.asarray(bias, np.float64)[None, :]
    a0d = a0.astype(np.float64)[None, :]
    logw0 = rng.randn(M)
    seed, site = 0xB0 + edge, P.SITE_AIS_V
    out = _native.debug_tc_op([(A1, B1, a_t, b_t, False)], outputs=('state',), ais_kind=1, sample='bernoulli', bias=bias,
                              ais_base=a0, seed=seed, site=site, t=e['t'], tick=e['tick'], tick_off=e['tick_off'],
                              row0=e['row0'], logw=logw0, force_bn=e['bn'] or 0, force_cluster=e['cluster'],
                              **{k: float(v) for k, v in temps.items()})
    assert out['plan']['mode'] == mode, out['plan']
    a, b, nxt = (float(temps[k]) for k in ('ais_a', 'ais_b', 'ais_next'))
    p = 1.0 / (1.0 + np.exp(-(nxt * u + a0d)))
    tol = sigmoid_tol(p, 4.0 * ULP * (np.abs(nxt * u) + np.abs(a0d) + 1.0))
    uu = P.uniform_at(M, N, seed, site, e['t'], e['tick'] + e['tick_off'], e['row0']).astype(np.float64)
    check_bernoulli(out['state'][:M, :N], uu, p, tol, 'unit states')
    term = softplus(b * u + a0d) - softplus(a * u + a0d)
    rel = (4e-6 if mode == 'AIS_UNITS' else 2.0 ** -18) + 70 * ULP
    tolw = rel * np.abs(term).sum(axis=1) + 1e-9
    assert_f32_within((out['logw'][:M] - logw0)[:, None], term.sum(axis=1)[:, None], tolw[:, None], 'logw increment')
    assert_guards(out, M, N)


@pytest.mark.parametrize('edge', [i for i, e in enumerate(EDGES) if (e['bn'] or 0) <= 128])
def test_state_op_with_a_base(edge):
    """x' ~ sigmoid(beta (A B^T + (b - a)) + a); the linear term stays beta-free of a"""
    e = EDGES[edge]
    M, N = e['M'], e['N']
    A1, B1, a_t, b_t, _, bias = edge_operands(e, edge)
    beta, lin = 0.625, 0.37
    a0 = base_of(N, edge)
    logw0 = np.random.RandomState(edge).randn(M)
    seed, site = 0xC0 + edge, P.SITE_AIS_H1
    out = _native.debug_tc_op([(A1, B1, a_t, b_t, False)], outputs=('state',), ais_kind=2, act='sigmoid', sample='bernoulli',
                              acc_scale=beta, bias_scale=beta, bias=bias, ais_base=a0, ais_lin=lin, seed=seed, site=site,
                              t=e['t'], tick=e['tick'], tick_off=e['tick_off'], row0=e['row0'], logw=logw0,
                              force_bn=e['bn'] or 0, force_cluster=e['cluster'])
    assert out['plan']['mode'] == 'AIS_STATE', out['plan']
    a_ = beta * product(A1, B1, a_t, b_t)
    b_ = beta * np.asarray(bias, np.float64) + a0.astype(np.float64)
    p = 1.0 / (1.0 + np.exp(-(a_ + b_[None, :])))
    tol = sigmoid_tol(p, 4.0 * ULP * (np.abs(a_) + np.abs(b_)[None, :] + np.abs(a0)[None, :]))
    u = P.uniform_at(M, N, seed, site, e['t'], e['tick'] + e['tick_off'], e['row0']).astype(np.float64)
    check_bernoulli(out['state'][:M, :N], u, p, tol, 'state draws')
    s = bf16_bits_to_f64(out['state'][:M, :N])
    w = beta * np.asarray(bias, np.float64) * -1.4426950408889634
    inc = lin * (s * w[None, :]).sum(axis=1)
    tolw = 74 * ULP * abs(lin) * np.abs(w).sum() + 1e-9
    assert_f32_within((out['logw'][:M] - logw0)[:, None], inc[:, None], np.full((M, 1), tolw), 'logw increment')
    assert_guards(out, M, N)


def test_a_base_needs_an_ais_op_of_at_most_128_columns():
    e = EDGES[3]
    A1, B1, a_t, b_t, _, bias = edge_operands(e, 3)
    with pytest.raises(RuntimeError, match='128 columns'):
        _native.debug_tc_op([(A1, B1, a_t, b_t, False)], outputs=('state',), ais_kind=1, sample='bernoulli', bias=bias,
                            ais_base=base_of(e['N'], 3), force_bn=256, force_cluster=e['cluster'], **AIS_FAR)


# ---- cfg4's shape --------------------------------------------------------------------------------------------------------------
def test_replay_at_784_500_1000_with_a_data_like_base():
    """16 runs of a 100-temperature ladder with visible biases and base around -3 (mostly-off pixels) against the float64
    statement on the weights the engine reads; runs fork only where a uniform lies within round-off of its probability"""
    V, Hs = 784, (500, 1000)
    p = params(V, Hs, scale=0.03, bias=0.2, seed=6)
    rng = np.random.RandomState(7)
    p['vb'] = (-3.0 + 0.7 * rng.randn(V)).astype(np.float32)
    X = (rng.rand(2000, V) < 1.0 / (1.0 + np.exp(-p['vb']))).astype(np.float32)
    base = [B.data_base(X), None, None]
    e = engine(V, Hs, p)
    got = e.ais(16, 100, 1, 99, first_run=1000, base=base)
    want = B.ais(bf16_params(p), 16, 100, 1, 99, first_run=1000, base=base)
    assert np.mean(np.abs(got - want) < 0.02) >= 0.75, np.abs(got - want)
    assert abs(lm(got) - lm(want)) < 0.05
    e.close()


@pytest.mark.parametrize('n_betas', [60, 500])
def test_zero_base_at_two_layers_is_ais_local(n_betas):
    """the layered ladder with a zero base draws what ais_local draws; the log-weights agree to the order of the fp64 atomics"""
    V, Hs = 784, (500, 1000)
    p = params(V, Hs, scale=0.03, bias=0.2, seed=8)
    e = engine(V, Hs, p)
    today = e.ais(256, n_betas, 1, 5)
    zero = [np.zeros(n, np.float32) for n in (V,) + Hs]
    got = e.ais(256, n_betas, 1, 5, base=zero)
    np.testing.assert_allclose(got - B.log_Z_A(p, zero), today - sum((V,) + Hs) * A.LOG2_F32, rtol=0, atol=1e-9)
    np.testing.assert_array_equal(e.ais(256, n_betas, 1, 5, base=[None] * 3), today)
    e.close()
