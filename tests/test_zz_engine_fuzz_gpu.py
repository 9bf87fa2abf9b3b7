"""Random-shape fuzz of the CUDA engines against the oracles (seeded: the same 60 configurations every run).

The fixed-shape parity tests pin a handful of tile geometries; this one walks ragged sizes (visible / hidden / batch
counts that are not multiples of 8, 64 or 128, single-row batches, K shorter than one MMA chunk), every unit kind,
dropout, sampling flags and chain lengths through `bm_rbm_train_step` / `bm_dbm_train_step` in each compute mode.
"""
import os

import numpy as np
import pytest

from boltzmann_machines import _native
from oracle.rbm import OracleRBM
from oracle.dbm import OracleDBM

pytestmark = pytest.mark.gpu


def rbm_case(i):
    rng = np.random.RandomState(9000 + i)
    pick = lambda xs: xs[rng.randint(len(xs))]
    kind = pick(['bernoulli', 'bernoulli', 'gaussian', 'multinomial'])
    V = int(pick([5, 17, 63, 64, 65, 127, 129, 200, 300, 784, 1000]))
    H = int(pick([3, 8, 15, 16, 17, 64, 70, 128, 130, 257, 512]))
    B = int(pick([1, 2, 7, 31, 33, 64, 100, 128, 129, 255, 300]))
    cfg = dict(n_visible=V, n_hidden=H, dtype='float32', l2=float(pick([0., 1e-4])), max_batch=B,
               sample_v=bool(rng.rand() < 0.5), sample_h=bool(rng.rand() < 0.7), sparsity_cost=float(pick([0., 0.01])),
               sparsity_target=0.2, dropout=pick([None, 0.8]))
    if kind == 'gaussian':
        cfg.update(v_kind='gaussian', h_kind='bernoulli', sigma=np.linspace(0.6, 1.4, V))
    elif kind == 'multinomial':
        cfg.update(v_kind='bernoulli', h_kind='multinomial', h_n_samples=int(pick([5, 20])))
    else:
        cfg.update(v_kind='bernoulli', h_kind='bernoulli')
    k = int(pick([1, 1, 2, 3]))
    init = dict(W=(0.1 * rng.randn(V, H)).astype(np.float32), vb=(0.1 * rng.randn(V)).astype(np.float32),
                hb=(0.1 * rng.randn(H)).astype(np.float32))
    X = rng.randn(2, B, V).astype(np.float32) if kind == 'gaussian' else (rng.rand(2, B, V) < 0.3).astype(np.float32)
    return cfg, k, init, X


@pytest.mark.parametrize('compute', ['fp32', 'bf16'])
@pytest.mark.parametrize('i', range(40))
def test_rbm_two_steps_on_random_shapes(i, compute):
    cfg, k, init, X = rbm_case(i)
    cfg = dict(cfg, compute=compute)
    # every built-in unit kind runs its GEMMs on the tensor cores under compute='bf16' (multinomial layers: GEMM, then row
    # softmax and draws as separate launches, bm_rbm_tc.cu: mixed()): the oracle rounds to bf16 at the same points
    eng, ora = _native.CudaRBM(cfg), OracleRBM(cfg)
    eng.set_params(init), ora.set_params(init)
    for it in range(2):
        eng.train_step(X[it], 0.05, 0.5, k, 4242, it)
        ora.train_step(X[it], 0.05, 0.5, k, 4242, it)
    g, w = eng.get_params(), ora.get_params()
    # fp32: summation order / libm; a draw differs only at rounding-level ties (one flipped unit moves dW by lr/B)
    tol = (5e-5 + 0.06 / X.shape[1]) if compute == 'fp32' else (3e-3 + 0.06 / X.shape[1])
    if cfg['h_kind'] == 'multinomial' and compute == 'bf16':
        tol *= 4.0                       # means up to n_samples (20) carry bf16 rounding of that size
    for name in ('W', 'vb', 'hb', 'dW', 'dvb', 'dhb', 'q_means'):
        assert np.all(np.isfinite(g[name])), name
        np.testing.assert_allclose(g[name], w[name], atol=tol, err_msg='{0} {1}'.format(name, cfg))
    m_g = eng.metrics(X[0], k, 7, 9, ('msre', 'pll', 'free_energy') if cfg['h_kind'] != 'multinomial' else ('msre',))
    m_w = ora.metrics(X[0], k, 7, 9, tuple(m_g))
    for name in m_g:
        assert m_g[name] == pytest.approx(m_w[name], rel=2e-2, abs=2e-2), (name, cfg)
    eng.close()


def dbm_case(i):
    rng = np.random.RandomState(7000 + i)
    pick = lambda xs: xs[rng.randint(len(xs))]
    L = int(pick([1, 2, 2, 3]))
    V = int(pick([9, 30, 65, 130, 784]))
    Hs = [int(pick([4, 11, 18, 64, 70, 129])) for _ in range(L)]
    B, M = int(pick([1, 5, 10, 33, 128])), int(pick([1, 4, 12, 40, 130]))
    gaussian = bool(rng.rand() < 0.25)
    cfg = dict(n_visible=V, n_hiddens=Hs, v_kind='gaussian' if gaussian else 'bernoulli', h_kinds=['bernoulli'] * L,
               h_n_samples=[100.] * L, dtype='float32', compute='fp32', n_particles=M, batch_size=B, max_mf_updates=int(pick([1, 4, 7])),
               mf_tol=float(pick([1e-7, 1e-3])), l2=1e-4, max_norm=float(pick([1.0, 3.0])), sample_v=bool(rng.rand() < 0.7),
               sample_h=[bool(rng.rand() < 0.8) for _ in range(L)], sparsity_target=[0.2] * L,
               sparsity_cost=[float(pick([0., 0.01]))] * L, sparsity_damping=0.9)
    if gaussian:
        cfg['sigma'] = np.linspace(0.7, 1.3, V)
    sizes = [V] + Hs
    init = {'vb': (0.1 * rng.randn(V)).astype(np.float32)}
    for j in range(L):
        s = '' if j == 0 else '_%d' % j
        init['W' + s] = (0.2 * rng.randn(sizes[j], sizes[j + 1])).astype(np.float32)
        init['hb' + s] = (0.1 * rng.randn(sizes[j + 1])).astype(np.float32)
    X = rng.randn(2, B, V).astype(np.float32) if gaussian else (rng.rand(2, B, V) < 0.3).astype(np.float32)
    return cfg, int(pick([1, 2])), init, X


@pytest.mark.parametrize('i', range(20))
def test_dbm_two_steps_on_random_shapes_fp32(i):
    cfg, k, init, X = dbm_case(i)
    eng, ora = _native.CudaDBM(cfg), OracleDBM(cfg)
    for e in (eng, ora):
        e.set_params(init)
        e.init_particles(99)
    for it in range(2):
        a = eng.train_step(X[it], 0.02, 0.5, k, 31337, it, metrics=('msre', 'n_mf_updates'))
        b = ora.train_step(X[it], 0.02, 0.5, k, 31337, it, metrics=('msre', 'n_mf_updates'))
        assert abs(a['n_mf_updates'] - b['n_mf_updates']) <= 1, cfg
        assert a['msre'] == pytest.approx(b['msre'], rel=1e-3), cfg
    g, w = eng.get_params(), ora.get_params()
    tol = 5e-5 + 0.05 / max(cfg['n_particles'], 1)
    for name in w:
        np.testing.assert_allclose(g[name], w[name], atol=tol, err_msg='{0} {1}'.format(name, cfg))
    eng.close()
