"""Classification RBM without a GPU: the float64 statement of the model (oracle/crbm.py) against brute force and finite
differences, its chain draws, the public API (boltzmann_machines.rbm.ClassificationRBM) on the oracle engine, and the
engine on the stand-in runtime with every kernel interpreted on the CPU (tests/hostsim, the classification RBM's restatements
linked in by tests/hostsim/build_crbm.sh) against the bf16 emulation (tests/class_rbm_bf16.py)."""
import ctypes as C
import itertools
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import philox as P
from oracle.crbm import OracleCRBM, crbm_factory, SITE_CRBM_Y
from oracle.rbm import multinomial_counts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_crbm.so')


def model(V=7, H=5, C=3, seed=0, **kw):
    cfg = dict(n_visible=V, n_hidden=H, n_classes=C, alpha=0.01, l2=1e-4, max_batch=16)
    cfg.update(kw)
    m = OracleCRBM(cfg)
    rng = np.random.RandomState(seed)
    m.set_params({'W': 0.5 * rng.randn(V, H), 'U': 0.5 * rng.randn(C, H), 'vb': 0.3 * rng.randn(V),
                  'hb': 0.3 * rng.randn(H), 'yb': 0.3 * rng.randn(C)})
    return m, rng


def test_posterior_equals_enumeration_over_h():
    m, rng = model(V=6, H=10, C=4)
    X = (rng.rand(5, 6) < 0.5).astype(np.float64)
    p = m.p
    hs = np.array(list(itertools.product([0.0, 1.0], repeat=10)))            # all 2^10 hidden states
    for b in range(len(X)):
        logp = np.array([np.logaddexp.reduce(hs @ (X[b] @ p['W'] + p['U'][y] + p['hb']) + p['yb'][y]) for y in range(4)])
        want = np.exp(logp - np.logaddexp.reduce(logp))
        np.testing.assert_allclose(m.predict_proba(X[b:b + 1])[0], want, atol=1e-6)      # float32 output
        np.testing.assert_allclose(m.posterior(X[b:b + 1])[0][0], want, rtol=0, atol=1e-10)


def test_discriminative_gradient_equals_finite_differences():
    m, rng = model(V=5, H=4, C=3, seed=1)
    X = rng.rand(6, 5)
    y = rng.randint(0, 3, size=6)
    g = m.disc_gradient(X, y)
    eps = 1e-6
    for name in ('W', 'U', 'vb', 'hb', 'yb'):
        num = np.zeros_like(m.p[name])
        for idx in np.ndindex(*m.p[name].shape):
            keep = m.p[name][idx]
            m.p[name][idx] = keep + eps
            hi = m.log_p(X, y).mean()
            m.p[name][idx] = keep - eps
            lo = m.log_p(X, y).mean()
            m.p[name][idx] = keep
            num[idx] = (hi - lo) / (2 * eps)
        np.testing.assert_allclose(g[name], num, rtol=1e-6, atol=1e-9, err_msg=name)


def test_chain_draws_at_the_documented_sites():
    m, rng = model(V=9, H=6, C=5, sample_v=True, sample_h=True)
    seed, tick, n = 77, 3, 8
    St = rng.rand(n, 6)
    Xk, Yk, Hk = m.chain(St, 2, seed, tick)
    h0 = (P.uniform_at(n, 6, seed, P.SITE_H0, 0, tick) < St.astype(np.float32)).astype(np.float64)
    xm1 = 1 / (1 + np.exp(-(h0 @ m.p['W'].T + m.p['vb'])))
    x1 = (P.uniform_at(n, 9, seed, P.SITE_V, 1, tick) < xm1.astype(np.float32)).astype(np.float64)
    z = h0 @ m.p['U'].T + m.p['yb']
    ym = np.exp(z - z.max(1, keepdims=True))
    ym /= ym.sum(1, keepdims=True)
    y1 = multinomial_counts(ym.astype(np.float32), 1, seed, SITE_CRBM_Y, 1, tick)
    hm1 = 1 / (1 + np.exp(-(x1 @ m.p['W'] + y1 @ m.p['U'] + m.p['hb'])))
    h1 = (P.uniform_at(n, 6, seed, P.SITE_H, 1, tick) < hm1.astype(np.float32)).astype(np.float64)
    xm2 = 1 / (1 + np.exp(-(h1 @ m.p['W'].T + m.p['vb'])))
    x2 = (P.uniform_at(n, 9, seed, P.SITE_V, 2, tick) < xm2.astype(np.float32)).astype(np.float64)
    np.testing.assert_array_equal(Xk, x2)
    assert np.all(Yk.sum(axis=1) == 1) and set(np.unique(Yk)) <= {0.0, 1.0}       # one-hot label draws
    assert SITE_CRBM_Y not in (P.SITE_H0, P.SITE_V, P.SITE_H) and SITE_CRBM_Y < P.SITE_DBM_H


def test_alpha_zero_is_the_discriminative_gradient_step():
    m, rng = model(alpha=0.0, l2=0.0)
    X, y = rng.rand(8, 7), rng.randint(0, 3, size=8)
    g = m.disc_gradient(X, y)
    before = {k: m.p[k].copy() for k in ('W', 'U', 'yb')}
    m.train_step(X, y, lr=0.1, momentum=0.0, k=1, seed=1, tick=0)
    for k in before:
        np.testing.assert_allclose(m.p[k] - before[k], 0.1 * g[k], rtol=1e-12, atol=1e-15)


# ---- public API on the oracle engine ------------------------------------------------------------------------------------
@pytest.fixture
def oracle_crbm():
    from boltzmann_machines.base import set_engine_factory
    old = set_engine_factory('crbm', crbm_factory)
    yield
    set_engine_factory('crbm', old)


def data(n=60, V=12, C=3, seed=0):
    rng = np.random.RandomState(seed)
    protos = rng.rand(C, V)
    y = rng.randint(0, C, size=n)
    return (rng.rand(n, V) < protos[y]).astype(np.float32), y


def test_fit_save_load_predict(oracle_crbm, tmp_path):
    from boltzmann_machines import ClassificationRBM
    X, y = data()
    path = str(tmp_path / 'crbm') + '/'
    m = ClassificationRBM(n_visible=12, n_hidden=8, n_classes=3, alpha=0.01, max_epoch=2, batch_size=16, learning_rate=0.1,
                          random_seed=3, verbose=False, model_path=path, metrics_config=dict(train_metrics_every_iter=2))
    m.fit(X, y, X_val=X[:20], y_val=y[:20])
    P1 = m.predict_proba(X)
    assert P1.shape == (60, 3) and P1.dtype == np.float32
    np.testing.assert_allclose(P1.sum(axis=1), 1.0, atol=1e-6)
    np.testing.assert_array_equal(m.predict(X), np.argmax(P1, axis=1))
    assert m.transform(X).shape == (60, 8)
    assert set(m.get_tf_params(scope='weights')) == {'W', 'U', 'vb', 'hb', 'yb'}
    assert set(m.get_tf_params(scope='grads_accumulators')) == {'dW', 'dU', 'dvb', 'dhb', 'dyb'}
    m2 = ClassificationRBM.load_model(path)
    np.testing.assert_array_equal(m2.predict_proba(X), P1)
    train = [json.loads(l) for l in open(os.path.join(path, 'logs', 'train', 'scalars.jsonl'))]
    val = [json.loads(l) for l in open(os.path.join(path, 'logs', 'val', 'scalars.jsonl'))]
    assert [r['step'] for r in train] == [2, 4, 6, 8] and all('mean_nll' in r and 'accuracy' in r for r in train)
    assert [r['step'] for r in val] == [4, 8] and all(0 <= r['accuracy'] <= 1 for r in val)
    m3 = ClassificationRBM(n_visible=12, n_hidden=8, n_classes=3, verbose=False, model_path=str(tmp_path / 'c3') + '/')
    m3.init_from(m)
    m3.init()
    np.testing.assert_array_equal(m3.get_tf_params(scope='weights')['U'], m.get_tf_params(scope='weights')['U'])


def test_predict_ties_go_to_the_lowest_class(oracle_crbm, tmp_path):
    from boltzmann_machines import ClassificationRBM
    m = ClassificationRBM(n_visible=4, n_hidden=3, n_classes=3, W_init=np.zeros((4, 3)), U_init=np.zeros((3, 3)),
                          verbose=False, model_path=str(tmp_path) + '/').init()
    assert list(m.predict(np.ones((2, 4)))) == [0, 0]


@pytest.mark.parametrize('kw', [dict(dtype='float64'), dict(compute='fp32'), dict(dropout=0.5), dict(sparsity_cost=0.1),
                                dict(dbm_first=True), dict(dbm_last=True)])
def test_refusals_name_the_option(kw):
    from boltzmann_machines import ClassificationRBM
    name = list(kw)[0]
    with pytest.raises(NotImplementedError, match=name if name != 'dtype' else 'float64'):
        ClassificationRBM(n_visible=4, n_hidden=3, n_classes=2, **kw)


def test_bad_labels_are_refused(oracle_crbm, tmp_path):
    from boltzmann_machines import ClassificationRBM
    m = ClassificationRBM(n_visible=12, n_hidden=4, n_classes=3, verbose=False, model_path=str(tmp_path) + '/')
    X, y = data()
    with pytest.raises(ValueError, match='labels'):
        m.fit(X, np.where(y == 0, 3, y))


# ---- the engine's host code on the stand-in runtime -------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_crbm.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(SIM)
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    lib.fakecuda_launches.restype = C.c_long
    lib.fakecuda_launches.argtypes = [C.c_char_p]
    lib.fakecuda_hazard_launches.restype = C.c_long
    lib.fakecuda_set_hazards(2)                 # every program launch, whatever its size
    lib.fakecuda_set_execute(1)
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    yield lib
    lib.fakecuda_set_execute(0)
    lib.fakecuda_set_hazards(1)
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib


def launches(sim, name=b''):
    return sim.fakecuda_launches(name)


def clean(sim):
    """no violation (out-of-bounds copies or tensor maps, hazards between ops of a program launch) and every launch
    interpreted"""
    v, sk = sim.fakecuda_violation().decode(), sim.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


def engine(**kw):
    from boltzmann_machines import _native
    cfg = dict(n_visible=30, n_hidden=20, n_classes=10, alpha=0.01, l2=1e-4, max_batch=100, sample_v=True, sample_h=True)
    cfg.update(kw)
    return _native.CudaCRBM(cfg)


@pytest.mark.parametrize('alpha,k', [(0.0, 1), (0.0, 3), (0.01, 1), (1.0, 3)])
def test_launches_per_step(sim, alpha, k):
    e = engine(alpha=alpha)
    X = np.zeros((70, 30), np.float32)
    y = np.arange(70) % 10
    sim.fakecuda_reset()
    e.train_step(X, y, 0.1, 0.5, k, seed=1, tick=0)
    clean(sim)
    tc = launches(sim, b'tc_')                          # the tensor-core ops: forward and dW (+ 3 per sweep)
    assert launches(sim, b'crbm_posterior_rows') == 1 and launches(sim, b'crbm_columns') == 1
    assert launches(sim, b'crbm_update') == 1
    if alpha == 0:
        assert launches(sim, b'dbm_multinomial_rows') == 0 and launches(sim, b'crbm_chain_stats') == 0
        assert tc == 2
        assert launches(sim) == 2 + 2 + 1 + 1           # + the bf16 conversion of X
    else:
        assert launches(sim, b'dbm_multinomial_rows') == k and launches(sim, b'crbm_chain_stats') == 1
        assert tc == 2 + 3 * k
        assert launches(sim) == 2 + 3 * k + k + 2 + 1 + 1 + 1
    e.close()


def test_predict_and_transform_launches(sim):
    e = engine()
    X = np.zeros((250, 30), np.float32)                 # three chunks of max_batch rows
    sim.fakecuda_reset()
    assert e.predict_proba(X).shape == (250, 10)
    assert launches(sim, b'crbm_posterior_rows') == 3 and launches(sim, b'crbm_columns') == 0
    sim.fakecuda_reset()
    assert e.transform(X).shape == (250, 20)
    assert launches(sim, b'crbm_columns') == 3
    clean(sim)
    e.close()


def test_bad_labels_launch_nothing(sim):
    e = engine()
    X = np.zeros((10, 30), np.float32)
    for bad in (-1, 10):
        y = np.zeros(10, np.int32)
        y[4] = bad
        sim.fakecuda_reset()
        with pytest.raises(RuntimeError, match='outside'):
            e.train_step(X, y, 0.1, 0.5, 1, seed=1, tick=0)
        assert launches(sim) == 0
    e.close()


@pytest.mark.parametrize('kw,word', [(dict(dtype='float64'), 'float64'), (dict(compute='fp32'), 'fp32'),
                                     (dict(dropout=0.8), 'dropout'), (dict(sparsity_cost=0.1), 'sparsity'),
                                     (dict(dbm_first=True), 'dbm_first'), (dict(dbm_last=True), 'dbm_last')])
def test_engine_refusals_launch_nothing(sim, kw, word):
    sim.fakecuda_reset()
    with pytest.raises(NotImplementedError, match=word):
        engine(**kw)
    assert launches(sim) == 0


@pytest.mark.parametrize('C_', [1, 65])
def test_class_count_is_bounded(sim, C_):
    with pytest.raises(RuntimeError, match='n_classes'):
        engine(n_classes=C_)


def test_parameters_round_trip(sim):
    e = engine(n_visible=13, n_hidden=9, n_classes=4)
    rng = np.random.RandomState(0)
    d = {'W': rng.randn(13, 9), 'U': rng.randn(4, 9), 'yb': rng.randn(4), 'dU': rng.randn(4, 9)}
    e.set_params(d)
    got = e.get_params(list(d))
    for k in d:
        np.testing.assert_array_equal(got[k], d[k].astype(np.float32))
    e.close()


# ---- the interpreted engine against the bf16 emulation ---------------------------------------------------------------------
@pytest.mark.parametrize('sample_v,sample_h', [(False, False), (True, True), (True, False), (False, True)])
@pytest.mark.parametrize('C_', [2, 10, 64])
@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('alpha', [0.0, 0.01, 1.0])
def test_interpreter_equals_the_bf16_emulation(sim, alpha, k, C_, sample_v, sample_h):
    from boltzmann_machines import _native
    sim.fakecuda_reset()
    from class_rbm_bf16 import compare_with_emulation
    compare_with_emulation(_native.CudaCRBM, alpha, k, C_, sample_v, sample_h)
    clean(sim)
    assert sim.fakecuda_hazard_launches() == 0         # each tensor-core op is its own launch: no multi-op programs


def test_emulation_detects_a_wrong_label_site():
    """the comparison above is tight enough to see the chain's draws: moving the label draw to another site, or not
    drawing h0, changes the variables by far more than its bound"""
    from class_rbm_bf16 import OracleCRBMbf16, close_enough
    import class_rbm_bf16 as E
    cfg = dict(n_visible=37, n_hidden=70, n_classes=10, alpha=1.0, l2=1e-3, max_batch=64, sample_v=True, sample_h=True)
    rng = np.random.RandomState(0)
    p = {'W': 0.3 * rng.randn(37, 70), 'U': 0.3 * rng.randn(10, 70), 'vb': 0.1 * rng.randn(37), 'hb': 0.1 * rng.randn(70),
         'yb': 0.1 * rng.randn(10)}
    X, y = (rng.rand(45, 37) < 0.4).astype(np.float32), rng.randint(0, 10, size=45)

    def run(**over):
        m = OracleCRBMbf16(dict(cfg, **over))
        m.set_params(p)
        m.train_step(X, y, 0.1, 0.5, 1, seed=23, tick=0)
        return m.get_params()

    ref = run()
    old = E.SITE_CRBM_Y
    try:
        E.SITE_CRBM_Y = 13
        moved = run()
    finally:
        E.SITE_CRBM_Y = old
    no_h0 = run(sample_h=False)
    for other in (moved, no_h0):
        assert not all(close_enough(other[n], ref[n]).all() for n in ('W', 'U', 'yb', 'hb'))
