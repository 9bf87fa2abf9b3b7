"""Clamped Gibbs chains (bm_dbm_fill, DESIGN.md §5.9) on the H100, replayed against float64 from the chain states the engine
exports (bm_dbm_debug_last_fill).

* cfg4's shape, 784-512-1024 after a few training steps, 1024 rows with the top 14 image rows missing, k = 3: every free unit of
  the last sweep against u < p recomputed in float64 from the sweep before (units within the fp32 bound of u are counted as
  ambiguous and bounded), every clamped unit equal to X's bf16 value in both exported sweeps, the output means against float64
  sigmoid(h_1 W_0' + b) within the bf16 bound, and the observed output units equal to X.
* The same shape with a 10-class label layer: labelled rows hold e_y in both sweeps, free labels follow the CDF of
  softmax(yb + h_L U') at site 16 + L.
* dbm_cifar_naive.py's shape, 3072-5000-1000 with sigma = 1 Gaussian visibles and a multinomial top layer: the Gaussian draws of
  the last sweep equal mean + N at their Philox address within the bf16 bound.
* A 16-visible model with 65 536 chains and 8 observed units: the missing units' distribution matches the exact conditional
  (chi-square per dof <= 2), and the same statistic rejects the unconditional marginal (> 4).
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from oracle import philox as P  # noqa: E402
from oracle.rbm import bf16_round  # noqa: E402
import dbm_fill_oracle as F  # noqa: E402

pytestmark = pytest.mark.gpu


def _native():
    from boltzmann_machines import _native
    return _native


def cfg(Hs, V, B, M=64, **kw):
    L = len(Hs)
    c = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
             n_particles=M, batch_size=B, max_mf_updates=3, mf_tol=1e-7, l2=1e-5, max_norm=1e300, sample_v=True,
             sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[0.] * L, sparsity_damping=0.9)
    c.update(kw)
    return c


def rand_params(c, scale, seed, bias=0.):
    rng = np.random.RandomState(seed)
    sizes = [c['n_visible']] + list(c['n_hiddens'])
    d = {'vb': (bias * rng.randn(sizes[0])).astype(np.float32)}
    for i in range(len(c['n_hiddens'])):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = (bias * rng.randn(sizes[i + 1])).astype(np.float32)
    return d


def digits_like(n, seed):
    rng = np.random.RandomState(seed)
    return (rng.rand(n, 784) < np.linspace(0.02, 0.4, 784)[None, :]).astype(np.float32)


def check_bernoulli_draws(state, p, u, free):
    """state == (u < p) on every free unit whose |u - p| exceeds the fp32 bound; returns the ambiguous count"""
    amb = (np.abs(u - p) <= 1e-4) & free
    bad = (state != (u < p)) & free & ~amb
    assert not bad.any(), 'draws disagree with float64 at {0} units'.format(int(bad.sum()))
    return int(amb.sum())


def sig(x):
    return 1. / (1. + np.exp(-x))


def trained_cfg4(n_classes=0):
    N = _native()
    c = cfg([512, 1024], 784, 1024, M=1024, **({'n_classes': n_classes} if n_classes else {}))
    e = N.CudaDBM(c)
    d = rand_params(c, 0.02, 1)
    if n_classes:
        rng = np.random.RandomState(2)
        d.update(U=(0.05 * rng.randn(n_classes, 1024)).astype(np.float32), yb=np.zeros(n_classes, np.float32))
    e.set_params(d)
    e.init_particles(7)
    X = digits_like(1024, 3)
    y = np.arange(1024) % 10
    for s in range(3):
        e.train_step(X, 0.01, 0.5, 1, seed=11, tick=s, labels=y if n_classes else None)
    return c, e


def replay_chain(e, c, X, mask, seed, tick, row0, k, labels=None):
    """the float64 checks of one fill on a two-layer Bernoulli DBM (+ label layer); returns the ambiguous draws"""
    rows = X.shape[0]
    out = e.fill(X, mask, labels, row0=row0, k=k, seed=seed, tick=tick)
    g = {n: e.debug_last_fill(n, rows).astype(np.float64) for n in ('v', 'v_prev', 'h', 'h_prev', 'h_1', 'h_1_prev', 'mean')}
    if labels is not None:
        for n in ('y', 'y_prev'):
            g[n] = e.debug_last_fill(n, rows).astype(np.float64)
    p = e.get_params(['W', 'W_1', 'vb', 'hb', 'hb_1'] + (['U', 'yb'] if labels is not None else []))
    W0, W1 = bf16_round(p['W']).astype(np.float64), bf16_round(p['W_1']).astype(np.float64)
    m = mask.astype(bool)
    Xb = bf16_round(X).astype(np.float64)
    for n in ('v', 'v_prev'):                                         # clamped units: X's bf16 value in every sweep
        assert np.array_equal(g[n][m], Xb[m]), n
    amb = 0
    u = lambda site, n: P.uniform_at(rows, n, seed, site, k, tick, row0).astype(np.float64)
    pre0 = g['v_prev'] @ W0 + g['h_1_prev'] @ W1.T + p['hb']
    amb += check_bernoulli_draws(g['h'], sig(pre0), u(P.SITE_DBM_H, 512), np.ones_like(g['h'], bool))
    pre1 = g['h'] @ W1 + p['hb_1']
    if labels is not None:
        pre1 = pre1 + g['y_prev'] @ bf16_round(p['U']).astype(np.float64)
    amb += check_bernoulli_draws(g['h_1'], sig(pre1), u(P.SITE_DBM_H + 1, 1024), np.ones_like(g['h_1'], bool))
    pv = sig(g['h'] @ W0.T + p['vb'])
    amb += check_bernoulli_draws(g['v'], pv, u(P.SITE_DBM_V, 784), ~m)
    # output means: float64 act(h_1 W_0' + b) within the bf16 rounding of the mean (plus the fp32 accumulation)
    err = np.abs(out.astype(np.float64) - pv)[~m]
    assert np.all(err <= 2. ** -8 * pv[~m] + 1e-5), float(err.max())
    assert np.array_equal(out[m], X[m])                                # observed output units are X bit for bit
    return amb, g, p


def test_cfg4_shape_replay():
    c, e = trained_cfg4()
    X = digits_like(1024, 5)
    mask = np.ones_like(X, dtype=np.uint8)
    mask[:, :14 * 28] = 0                                              # the top 14 image rows are missing
    before = e.get_params()
    amb, _, _ = replay_chain(e, c, X, mask, seed=1234, tick=3, row0=2048, k=3)
    n_draws = 1024 * (512 + 1024 + 14 * 28)
    assert amb <= 1e-3 * n_draws, amb
    after = e.get_params()
    assert all(np.array_equal(before[n], after[n]) for n in before), 'fill changed a variable'
    print('cfg4 fill: {0} draws checked, {1} ambiguous'.format(n_draws, amb))
    e.close()


def test_cfg4_shape_classes_replay():
    c, e = trained_cfg4(n_classes=10)
    X = digits_like(1024, 6)
    mask = np.ones_like(X, dtype=np.uint8)
    mask[:, :14 * 28] = 0
    y = np.where(np.arange(1024) % 2 == 0, np.arange(1024) % 10, -1).astype(np.int32)
    seed, tick, row0, k = 99, 1, 0, 3
    amb, g, p = replay_chain(e, c, X, mask, seed, tick, row0, k, labels=y)
    lab = y >= 0
    onehot = np.eye(10)[y[lab]]
    for n in ('y', 'y_prev'):
        assert np.array_equal(g[n][lab], onehot), n
    z = g['h_1'] @ bf16_round(p['U']).astype(np.float64).T + p['yb']
    q = np.exp(z - z.max(1, keepdims=True))
    cdf = np.cumsum(q / q.sum(1, keepdims=True), axis=1)
    u = P.uniform_at(1024, 1, seed, P.SITE_DBM_H + 2, k, tick, row0).astype(np.float64)[:, 0]
    want = np.minimum((cdf <= u[:, None]).sum(1), 9)
    near = np.min(np.abs(cdf - u[:, None]), axis=1) <= 1e-4
    got = g['y'].argmax(1)
    assert np.all(g['y'][~lab].sum(1) == 1)
    bad = (got != want) & ~lab & ~near
    assert not bad.any(), int(bad.sum())
    print('cfg4 + 10 classes: {0} ambiguous unit draws, {1} ambiguous labels'.format(amb, int((near & ~lab).sum())))
    e.close()


def test_cifar_naive_shape_gaussian_draws():
    N = _native()
    c = cfg([5000, 1000], 3072, 100, M=100, v_kind='gaussian', sigma=np.ones(3072), h_kinds=['bernoulli', 'multinomial'],
            h_n_samples=[100., 1000.])
    e = N.CudaDBM(c)
    assert e.compute == 'bf16'
    e.set_params(rand_params(c, 0.01, 4, bias=0.1))
    rng = np.random.RandomState(8)
    X = rng.randn(100, 3072).astype(np.float32)
    mask = (rng.rand(100, 3072) < 0.5).astype(np.uint8)
    seed, tick, row0, k = 5, 0, 300, 2
    out = e.fill(X, mask, row0=row0, k=k, seed=seed, tick=tick)
    v, h = e.debug_last_fill('v', 100).astype(np.float64), e.debug_last_fill('h', 100).astype(np.float64)
    p = e.get_params(['W', 'vb'])
    mean = h @ bf16_round(p['W']).astype(np.float64).T + p['vb']
    eps = P.normal_at(100, 3072, seed, P.SITE_DBM_V, k, tick, row0).astype(np.float64)
    free = ~mask.astype(bool)
    want = mean + eps
    err = np.abs(v - want)[free]
    assert np.all(err <= 2. ** -8 * np.abs(want[free]) + 1e-3), float(err.max())
    assert np.array_equal(v[~free], bf16_round(X).astype(np.float64)[~free])
    assert np.array_equal(out[~free], X[~free])
    em = np.abs(out.astype(np.float64) - mean)[free]
    assert np.all(em <= 2. ** -8 * np.abs(mean[free]) + 1e-3), float(em.max())
    e.close()


def test_enumerable_conditional_on_gpu():
    N = _native()
    V, Hs, B = 16, [6], 8192
    c = cfg(Hs, V, B, M=16)
    e = N.CudaDBM(c)
    d = rand_params(c, 0.9, 12, bias=0.5)
    e.set_params(d)
    dd = {k: bf16_round(v).astype(np.float64) if k.startswith('W') else v.astype(np.float64) for k, v in d.items()}
    logp = F.exact_log_p_v(dd, Hs)
    obs = list(range(0, 16, 2))
    x_obs = np.array([1, 0, 1, 1, 0, 0, 1, 0], dtype=np.float64)
    want = F.conditional_table(logp, V, obs, x_obs)
    miss = [j for j in range(V) if j not in obs]
    counts = np.zeros(256)
    X = np.zeros((B, V), np.float32)
    X[:, obs] = x_obs
    mask = np.zeros((B, V), np.uint8)
    mask[:, obs] = 1
    for r0 in range(0, 65536, B):
        e.fill(X, mask, row0=r0, k=30, seed=77, tick=0)
        v = e.debug_last_fill('v', B)
        counts += np.bincount((v[:, miss] @ (2 ** np.arange(8))).astype(np.int64), minlength=256)
    stat = F.chi2_per_dof(counts, want)
    # the unconditional marginal of the missing units (bit j of the table = missing unit j): the statistic must reject it
    vs = F.states(V)
    pm = np.zeros(256)
    np.add.at(pm, (vs[:, miss] @ (2 ** np.arange(8))).astype(np.int64), np.exp(logp))
    ctrl = F.chi2_per_dof(counts, pm)
    print('16-visible model, 65536 chains: chi2/dof {0:.3f}; against the marginal {1:.1f}'.format(stat, ctrl))
    assert stat <= 2.0, stat
    assert ctrl > 2 * 2.0, ctrl
    e.close()
