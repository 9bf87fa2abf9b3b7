"""AIS log Z and the variational bound of binary DBMs with one, three or more hidden layers on the tensor-core engine
(DESIGN.md §5.4c, DbmTC::ais_local_layers / log_proba_layers) on the H100: exact enumeration, the bf16 emulation run by run
(tests/dbm_ais_depth_oracle.py), the two epilogue shapes only these ladders use, a replay at 784-500-500-1000, identities
between depths at the benchmark's width, and the bound."""
import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P
from oracle.rbm import bf16_round

import dbm_ais_depth_oracle as A
from test_tc_kernel_exact_gpu import (EDGES, ULP, assert_f32_within, assert_guards, bf16_bits_to_f64, check_bernoulli,
                                      edge_operands, product, sigmoid_tol, softplus)

pytestmark = pytest.mark.gpu
sfx = A.sfx


def make_cfg(V, Hs, **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, h_n_samples=[100.] * L,
               dtype='float32', compute='bf16', n_particles=4, batch_size=16, max_mf_updates=10, mf_tol=1e-7, l2=1e-4,
               max_norm=3.0, sample_v=True, sample_h=[True] * L, sparsity_target=[0.2] * L, sparsity_cost=[0.01] * L,
               sparsity_damping=0.9)
    cfg.update(kw)
    return cfg


def params(V, Hs, scale=0.3, bias=0.1, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [V] + list(Hs)
    d = {'vb': (bias * rng.randn(V)).astype(np.float32)}
    for i in range(len(Hs)):
        d['W' + sfx(i)] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + sfx(i)] = (bias * rng.randn(sizes[i + 1])).astype(np.float32)
    return d


def bf16_params(p):
    return {k: (bf16_round(v) if k.startswith('W') else v) for k, v in p.items()}


def engine(V, Hs, p, **kw):
    e = _native.CudaDBM(make_cfg(V, Hs, **kw))
    assert e.compute == 'bf16'
    e.set_params(p)
    return e


def lm(v):
    return float(np.logaddexp.reduce(v) - np.log(len(v)))


def log_mean_se(v):
    """log of the mean of exp(v) and the standard error of that log (delta method)"""
    w = np.exp(v - np.max(v))
    return lm(v), float(np.std(w) / np.mean(w) / np.sqrt(len(v)))


SHAPES = {1: (7, (5,)), 3: (6, (5, 4, 3)), 4: (5, (4, 4, 3, 3))}


# ---- exact enumeration and the emulation -------------------------------------------------------------------------------------
@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('L', [1, 3, 4])
def test_ais_matches_exact_enumeration(L, k):
    """the tolerances of tests/test_zz_dbm_tc_gpu.py::test_ais_matches_exact_enumeration"""
    V, Hs = SHAPES[L]
    n_betas = 240 if k == 1 else 120
    p = params(V, Hs, seed=L)
    e = engine(V, Hs, p)
    a = e.ais(32, n_betas, k, 2222)
    b = A.ais(p, 32, n_betas, k, 2222, bf16=True)
    assert abs(lm(a) - lm(b)) < 0.1
    assert np.mean(np.abs(a - b) < 2e-3) > 0.8           # the same chains, but for a draw at rounding distance of its probability
    exact = A.exact_log_Z(bf16_params(p))
    assert abs(lm(a) - exact) < 0.15, (lm(a), exact)
    e.close()


@pytest.mark.parametrize('L', [1, 3, 4])
def test_fine_ladder_and_unsampled_summed_out_layers_match_the_emulation(L):
    """>= 400 temperatures: the series form of the increment (bm_tc.cu MODE_AIS_UNITS); and v / h_2 as means"""
    V, Hs = SHAPES[L]
    p = params(V, Hs, scale=1.0, seed=10 + L)
    e = engine(V, Hs, p)
    a, b = e.ais(12, 500, 1, 31), A.ais(p, 12, 500, 1, 31, bf16=True)
    assert np.mean(np.abs(a - b) < 2e-3) >= 0.75, np.abs(a - b)
    assert abs(np.mean(a) - np.mean(b)) < 0.05
    e.close()
    if L >= 3:
        sh = [True] * L
        sh[1] = False
        e = engine(V, Hs, p, sample_v=False, sample_h=sh)
        a, b = e.ais(32, 120, 2, 7), A.ais(p, 32, 120, 2, 7, bf16=True, sample_v=False, sample_h=sh)
        assert np.mean(np.abs(a - b) < 2e-3) > 0.8, np.abs(a - b)
        e.close()


# ---- the two epilogue shapes these ladders add -------------------------------------------------------------------------------
AIS_LADDER = dict(ais_a=np.float32(0.5), ais_b=np.float32(0.5 + 1.0 / 500), ais_next=np.float32(0.5 + 2.0 / 500))
AIS_FAR = dict(ais_a=np.float32(0.2), ais_b=np.float32(0.3), ais_next=np.float32(0.4))


@pytest.mark.parametrize('edge', range(len(EDGES)))
@pytest.mark.parametrize('temps,mode', [(AIS_LADDER, 'AIS_UNITS'), (AIS_FAR, 'AIS_UNITS_G')], ids=['series', 'closed'])
def test_units_op_behind_two_pairs(edge, temps, mode):
    """a middle summed-out layer: z = A1 B1^T + A2 B2^T + bias; logw[m] += sum_n softplus(b z) - softplus(a z); states drawn"""
    e = EDGES[edge]
    M, N = e['M'], e['N']
    A1, B1, a_t, b_t, _, bias = edge_operands(e, edge)
    A2, B2, a_t2, b_t2, _, _ = edge_operands(e, edge + 1)
    rng = np.random.RandomState(edge)
    A1 = A1 * (rng.rand(*A1.shape) < 0.5)
    A2 = A2 * (rng.rand(*A2.shape) < 0.5)                # keep z within about [-8, 8]
    z = product(A1, B1, a_t, b_t) + product(A2, B2, a_t2, b_t2) + np.asarray(bias, np.float64)[None, :]
    logw0 = rng.randn(M)
    seed, site = 0xD0 + edge, P.SITE_AIS_H2
    out = _native.debug_tc_op([(A1, B1, a_t, b_t, False), (A2, B2, a_t2, b_t2, False)], outputs=('state',), ais_kind=1,
                              sample='bernoulli', bias=bias, seed=seed, site=site, t=e['t'], tick=e['tick'],
                              tick_off=e['tick_off'], row0=e['row0'], logw=logw0, force_bn=e['bn'] or 0,
                              force_cluster=e['cluster'], **{k: float(v) for k, v in temps.items()})
    assert out['plan']['mode'] == mode, out['plan']
    a, b, nxt = (float(temps[k]) for k in ('ais_a', 'ais_b', 'ais_next'))
    p = 1.0 / (1.0 + np.exp(-nxt * z))
    tol = sigmoid_tol(p, 4.0 * ULP * (np.abs(nxt * z) + 1.0))
    u = P.uniform_at(M, N, seed, site, e['t'], e['tick'] + e['tick_off'], e['row0']).astype(np.float64)
    check_bernoulli(out['state'][:M, :N], u, p, tol, 'unit states')
    term = softplus(b * z) - softplus(a * z)
    rel = (4e-6 if mode == 'AIS_UNITS' else 2.0 ** -18) + 70 * ULP
    tolw = rel * np.abs(term).sum(axis=1) + 1e-9
    assert_f32_within((out['logw'][:M] - logw0)[:, None], term.sum(axis=1)[:, None], tolw[:, None], 'logw increment')
    assert_guards(out, M, N)


@pytest.mark.parametrize('edge', range(len(EDGES)))
def test_state_op_behind_one_pair(edge):
    """h_1 of a one-layer model or h_L of an odd-depth one: x' ~ sigmoid(beta (A B^T + c)) with the linear term, at the
    temperature scaling the ladder uses (acc_scale = bias_scale = beta)"""
    e = EDGES[edge]
    M, N = e['M'], e['N']
    A1, B1, a_t, b_t, _, bias = edge_operands(e, edge)
    beta, lin = 0.625, 0.37
    logw0 = np.random.RandomState(edge).randn(M)
    seed, site = 0xE0 + edge, P.SITE_AIS_H1
    out = _native.debug_tc_op([(A1, B1, a_t, b_t, False)], outputs=('state',), ais_kind=2, act='sigmoid', sample='bernoulli',
                              acc_scale=beta, bias_scale=beta, bias=bias, ais_lin=lin, seed=seed, site=site, t=e['t'],
                              tick=e['tick'], tick_off=e['tick_off'], row0=e['row0'], logw=logw0, force_bn=e['bn'] or 0,
                              force_cluster=e['cluster'])
    assert out['plan']['mode'] == 'AIS_STATE', out['plan']
    a_ = beta * product(A1, B1, a_t, b_t)
    b_ = beta * np.asarray(bias, np.float64)
    p = 1.0 / (1.0 + np.exp(-(a_ + b_[None, :])))
    tol = sigmoid_tol(p, 4.0 * ULP * (np.abs(a_) + np.abs(b_)[None, :]))
    u = P.uniform_at(M, N, seed, site, e['t'], e['tick'] + e['tick_off'], e['row0']).astype(np.float64)
    check_bernoulli(out['state'][:M, :N], u, p, tol, 'state draws')
    s = bf16_bits_to_f64(out['state'][:M, :N])
    w = b_ * -1.4426950408889634
    inc = lin * (s * w[None, :]).sum(axis=1)
    tolw = 74 * ULP * abs(lin) * np.abs(w).sum() + 1e-9
    assert_f32_within((out['logw'][:M] - logw0)[:, None], inc[:, None], np.full((M, 1), tolw), 'logw increment')
    assert_guards(out, M, N)


# ---- a realistic depth ----------------------------------------------------------------------------------------------------------
def test_replay_at_784_500_500_1000():
    """16 runs of a 100-temperature ladder against the float64 statement on the weights the engine reads (bf16), computed
    here.  The two differ only by fp32 sums, so a draw differs only where its uniform lies within round-off of its
    probability; such a fork moves one run, so most runs agree to float32 round-off of their log-weights"""
    V, Hs = 784, (500, 500, 1000)
    p = params(V, Hs, scale=0.03, bias=0.2, seed=5)
    e = engine(V, Hs, p)
    got = e.ais(16, 100, 1, 99, first_run=1000)
    want = A.ais(bf16_params(p), 16, 100, 1, 99, first_run=1000)
    assert np.mean(np.abs(got - want) < 0.02) >= 0.75, np.abs(got - want)
    assert abs(lm(got) - lm(want)) < 0.05
    e.close()


# ---- identities between depths at the benchmark's width -------------------------------------------------------------------
def _identity(V, Hs, n_runs=256, n_betas=300):
    """log Z of a model whose top weights are zero = log Z of its prefix + sum softplus(c_L)"""
    L = len(Hs)
    p = params(V, Hs, scale=0.02, bias=0.1, seed=L)
    p['W' + sfx(L - 1)][:] = 0.
    q = {k: v for k, v in p.items() if k not in ('W' + sfx(L - 1), 'hb' + sfx(L - 1))}
    big, small = engine(V, Hs, p), engine(V, Hs[:-1], q)
    a, sa = log_mean_se(big.ais(n_runs, n_betas, 1, 11))
    b, sb = log_mean_se(small.ais(n_runs, n_betas, 1, 12))
    shift = float(np.logaddexp(0., p['hb' + sfx(L - 1)].astype(np.float64)).sum())
    big.close(); small.close()
    return a, b + shift, 3 * (sa + sb) + 1e-3


def test_zero_top_weights_three_layers_against_the_two_layer_ladder():
    """the new path (L = 3) against the untouched one (L = 2) at 784-512-1024(-512)"""
    a, b, tol = _identity(784, (512, 1024, 512))
    assert abs(a - b) < tol, (a, b, tol)


def test_zero_top_weights_two_layers_against_the_one_layer_ladder():
    """the untouched path (L = 2) against the new one (L = 1) at 784-512(-1024)"""
    a, b, tol = _identity(784, (512, 1024))
    assert abs(a - b) < tol, (a, b, tol)


# ---- the bound --------------------------------------------------------------------------------------------------------------------
def test_bound_of_one_layer_is_the_exact_log_likelihood():
    V, Hs = 7, (5,)
    p = params(V, Hs, scale=0.8, bias=0.3, seed=3)
    e = engine(V, Hs, p)
    X = (np.random.RandomState(2).rand(16, V) < 0.5).astype(np.float32)
    logZ = A.exact_log_Z(bf16_params(p))
    exact = A.brute_log_p_v(bf16_params(p), X) - logZ
    np.testing.assert_allclose(e.log_proba(X) - logZ, exact, atol=2e-3)    # the E-step's bf16 means
    e.close()


@pytest.mark.parametrize('L', [3, 4])
def test_bound_is_below_the_exact_log_likelihood(L):
    V, Hs = SHAPES[L]
    p = params(V, Hs, scale=0.8, bias=0.3, seed=20 + L)
    e = engine(V, Hs, p)
    X = (np.random.RandomState(2).rand(16, V) < 0.5).astype(np.float32)
    exact = A.brute_log_p_v(bf16_params(p), X)
    assert np.all(e.log_proba(X) <= exact + 2e-3)
    e.close()


@pytest.mark.parametrize('V,Hs', [(784, (500, 500, 1000)), (784, (500,)), (30, (18, 11, 7, 5))])
def test_bound_matches_the_float64_restatement_given_the_engines_means(V, Hs):
    L = len(Hs)
    p = params(V, Hs, scale=0.05, bias=0.2, seed=L)
    e = engine(V, Hs, p)
    X = (np.random.RandomState(8).rand(16, V) < 0.3).astype(np.float32)
    got = e.log_proba(X)
    g = e.get_params(['mu' + sfx(i) for i in range(L)])
    want = A.bound_given_mu(p, X, [g['mu' + sfx(i)][:16] for i in range(L)])
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-3)
    e.close()
