"""Semi-supervised classification RBM without a GPU (rows labelled -1 with beta > 0): the float64 statement
(tests/class_rbm_semi.py) against finite differences and enumeration, the public API on that statement, and the engine on the
stand-in runtime with every kernel interpreted on the CPU (tests/hostsim/build_crbm_semi.sh) against the bf16 emulation."""
import ctypes as C
import itertools
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import philox as P

from class_rbm_semi import (OracleSemiCRBM, OracleSemiCRBMbf16, SITE_CRBM_Y0, close_enough, compare_semi_with_emulation,
                            semi_factory, semi_labels)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_crbm_semi.so')


def model(V=7, H=5, C=3, seed=0, **kw):
    cfg = dict(n_visible=V, n_hidden=H, n_classes=C, alpha=0.01, beta=0.5, l2=1e-4, max_batch=16)
    cfg.update(kw)
    m = OracleSemiCRBM(cfg)
    rng = np.random.RandomState(seed)
    m.set_params({'W': 0.5 * rng.randn(V, H), 'U': 0.5 * rng.randn(C, H), 'vb': 0.3 * rng.randn(V),
                  'hb': 0.3 * rng.randn(H), 'yb': 0.3 * rng.randn(C)})
    return m, rng


def test_unlabelled_positive_phase_equals_finite_differences():
    """the exact positive phase of an unlabelled row is the gradient of log sum_y exp(vb.x + F(x, y))"""
    m, rng = model(V=5, H=4, C=3, seed=1)
    X = rng.rand(6, 5)
    g = m.semi_positive(X)
    eps = 1e-6
    for name in ('W', 'U', 'vb', 'hb', 'yb'):
        num = np.zeros_like(m.p[name])
        for idx in np.ndindex(*m.p[name].shape):
            keep = m.p[name][idx]
            m.p[name][idx] = keep + eps
            hi = m.log_px_unnormalised(X).mean()
            m.p[name][idx] = keep - eps
            lo = m.log_px_unnormalised(X).mean()
            m.p[name][idx] = keep
            num[idx] = (hi - lo) / (2 * eps)
        np.testing.assert_allclose(g[name], num, rtol=1e-6, atol=1e-9, err_msg=name)


def test_chain_start_is_a_draw_from_p_y_h_given_x():
    """V = 3, H = 2, C = 2: over 40 000 copies of one x, the start (y0, h0) of the unlabelled rows' chain against p(y, h | x)
    by enumeration.  Every one of the 8 cells within 0.01 (4 standard deviations of a frequency at n = 40 000 is <= 0.01)."""
    m, _ = model(V=3, H=2, C=2, seed=4, sample_h=True)
    x = np.array([1.0, 0.0, 1.0])
    n, seed, tick = 40000, 91, 5
    X = np.tile(x, (n, 1))
    y0, S0 = m.chain_start(X, np.full(n, -1), seed, tick)
    h0 = (P.uniform_at(n, 2, seed, P.SITE_H0, 0, tick) < S0.astype(np.float32)).astype(int)
    p = m.p
    cells = list(itertools.product(range(2), itertools.product([0, 1], repeat=2)))
    logw = np.array([p['yb'][y] + np.dot(h, x @ p['W'] + p['U'][y] + p['hb']) for y, h in cells])
    want = np.exp(logw - np.logaddexp.reduce(logw))
    got = np.array([np.mean((y0 == y) & (h0[:, 0] == h[0]) & (h0[:, 1] == h[1])) for y, h in cells])
    assert np.max(np.abs(got - want)) <= 0.01, (got, want)


def test_start_label_uses_its_own_site():
    assert SITE_CRBM_Y0 == 13 and SITE_CRBM_Y0 not in (P.SITE_H0, P.SITE_V, P.SITE_H, 12) and SITE_CRBM_Y0 < P.SITE_DBM_H


def test_labelled_batches_are_the_hybrid_step():
    """without -1 the semi-supervised statement is the hybrid step, whatever beta is"""
    a, rng = model(beta=0.0)
    b, _ = model(beta=0.7)
    X, y = rng.rand(8, 7), rng.randint(0, 3, size=8)
    for m in (a, b):
        m.train_step(X, y, 0.1, 0.5, 1, seed=1, tick=0)
    for k in a.p:
        np.testing.assert_array_equal(a.p[k], b.p[k])


def test_refusals_of_the_statement():
    m, rng = model(beta=0.0)
    with pytest.raises(RuntimeError, match='outside'):
        m.train_step(rng.rand(4, 7), [0, -1, 1, 2], 0.1, 0.5, 1, seed=1, tick=0)
    m, rng = model()
    for bad in (-2, 3):
        with pytest.raises(RuntimeError, match='outside'):
            m.train_step(rng.rand(4, 7), [0, -1, bad, 2], 0.1, 0.5, 1, seed=1, tick=0)


# ---- public API on the float64 statement --------------------------------------------------------------------------------
@pytest.fixture
def semi_engine():
    from boltzmann_machines.base import set_engine_factory
    old = set_engine_factory('crbm', semi_factory)
    yield
    set_engine_factory('crbm', old)


def data(n=64, V=12, C=3, seed=0):
    rng = np.random.RandomState(seed)
    protos = rng.rand(C, V)
    y = rng.randint(0, C, size=n)
    return (rng.rand(n, V) < protos[y]).astype(np.float32), y


def test_fit_with_unlabelled_rows_save_load(semi_engine, tmp_path):
    from boltzmann_machines import ClassificationRBM
    X, y = data()
    y = y.copy()
    y[1::2] = -1
    y[16:32] = -1                        # the second batch of every epoch has no label: it reports nothing
    path = str(tmp_path / 'semi') + '/'
    m = ClassificationRBM(n_visible=12, n_hidden=8, n_classes=3, alpha=0.01, beta=0.5, max_epoch=2, batch_size=16,
                          learning_rate=0.1, random_seed=3, verbose=False, model_path=path,
                          metrics_config=dict(train_metrics_every_iter=1))
    m.fit(X, y, X_val=X[:20], y_val=np.where(y[:20] < 0, 0, y[:20]))
    P1 = m.predict_proba(X)
    assert P1.shape == (64, 3) and np.all(np.isfinite(P1))
    train = [json.loads(l) for l in open(os.path.join(path, 'logs', 'train', 'scalars.jsonl'))]
    assert [r['step'] for r in train] == [1, 3, 4, 5, 7, 8]
    assert all(np.isfinite(r['mean_nll']) and 0 <= r['accuracy'] <= 1 for r in train)
    m2 = ClassificationRBM.load_model(path)
    assert m2.beta == 0.5
    np.testing.assert_array_equal(m2.predict_proba(X), P1)


def test_unlabelled_rows_change_the_model(semi_engine, tmp_path):
    """the same labelled rows with and without the unlabelled ones give different weights (the rows are used)"""
    from boltzmann_machines import ClassificationRBM
    X, y = data()
    ys = y.copy()
    ys[1::2] = -1
    out = []
    for beta, labels in ((0.5, ys), (0.0, None)):
        m = ClassificationRBM(n_visible=12, n_hidden=8, n_classes=3, beta=beta, max_epoch=1, batch_size=16, random_seed=3,
                              verbose=False, model_path=str(tmp_path / str(beta)) + '/')
        if labels is None:
            m.fit(X[0::2], y[0::2])
        else:
            m.fit(X, labels)
        out.append(m.get_tf_params(scope='weights')['W'])
    assert not np.array_equal(out[0], out[1])


def test_label_errors(semi_engine, tmp_path):
    from boltzmann_machines import ClassificationRBM
    X, y = data()
    y = y.copy()
    y[3] = -1
    m = ClassificationRBM(n_visible=12, n_hidden=4, n_classes=3, verbose=False, model_path=str(tmp_path / 'a') + '/')
    with pytest.raises(ValueError, match='beta') as e:
        m.fit(X, y)
    assert 'labels' in str(e.value)
    m = ClassificationRBM(n_visible=12, n_hidden=4, n_classes=3, beta=0.2, verbose=False, model_path=str(tmp_path / 'b') + '/')
    with pytest.raises(ValueError, match='labels'):
        m.fit(X, np.where(y == 0, -2, y))
    with pytest.raises(ValueError, match='labels'):
        m.fit(X, np.where(y == 0, 3, y))
    with pytest.raises(ValueError, match='labels'):
        m.fit(X, np.where(y < 0, 0, y), X_val=X[:8], y_val=y[:8])          # y_val must be fully labelled
    with pytest.raises(ValueError, match='beta'):
        ClassificationRBM(n_visible=12, n_hidden=4, n_classes=3, beta=-0.1, verbose=False)


# ---- the engine's host code on the stand-in runtime -------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_crbm_semi.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(SIM)
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    lib.fakecuda_launches.restype = C.c_long
    lib.fakecuda_launches.argtypes = [C.c_char_p]
    lib.fakecuda_hazard_launches.restype = C.c_long
    lib.fakecuda_set_hazards(2)
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


KERNELS = (b'tc_', b'crbm_posterior_rows', b'crbm_columns', b'crbm_chain_stats', b'crbm_update', b'dbm_multinomial_rows', b'')


def counts(sim):
    return [sim.fakecuda_launches(k) for k in KERNELS]


def clean(sim):
    v, sk = sim.fakecuda_violation().decode(), sim.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


def engine(**kw):
    from boltzmann_machines import _native
    cfg = dict(n_visible=30, n_hidden=20, n_classes=10, alpha=0.01, beta=0.5, l2=1e-4, max_batch=100, sample_v=True,
               sample_h=True)
    cfg.update(kw)
    return _native.CudaCRBM(cfg)


@pytest.mark.parametrize('C_', [2, 10])
@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('alpha', [0.0, 0.01, 1.0])
def test_labelled_batches_are_bitwise_the_beta_zero_step(sim, alpha, k, C_):
    """every row labelled: beta = 0.5 computes the beta = 0 step bit for bit, with the same launches"""
    from boltzmann_machines import _native
    res = []
    for beta in (0.0, 0.5):
        cfg = dict(n_visible=37, n_hidden=70, n_classes=C_, alpha=alpha, beta=beta, l2=1e-3, max_batch=64, sample_v=True,
                   sample_h=True)
        e = _native.CudaCRBM(cfg)
        rng = np.random.RandomState(7)
        e.set_params({'W': 0.3 * rng.randn(37, 70), 'U': 0.3 * rng.randn(C_, 70), 'vb': 0.1 * rng.randn(37),
                      'hb': 0.1 * rng.randn(70), 'yb': 0.1 * rng.randn(C_)})
        metrics, launches = [], []
        for step in range(3):
            X = (rng.rand(45, 37) < 0.4).astype(np.float32)
            y = rng.randint(0, C_, size=45)
            sim.fakecuda_reset()
            metrics.append(e.train_step(X, y, 0.1, 0.5, k, seed=23, tick=step, metrics=True))
            launches.append(counts(sim))
            clean(sim)
        res.append((e.get_params(), metrics, launches))
        e.close()
    (p0, m0, l0), (p1, m1, l1) = res
    assert l0 == l1 and m0 == m1
    for name in p0:
        assert p0[name].tobytes() == p1[name].tobytes(), name


@pytest.mark.parametrize('sample_v,sample_h', [(False, False), (True, True), (True, False), (False, True)])
@pytest.mark.parametrize('C_', [2, 10, 64])
@pytest.mark.parametrize('fraction', ['none', 'some', 'all'])
@pytest.mark.parametrize('alpha', [0.0, 0.01])
@pytest.mark.parametrize('beta', [0.1, 1.0])
def test_interpreter_equals_the_semi_supervised_emulation(sim, beta, alpha, fraction, C_, sample_v, sample_h):
    """every step: the variables to close_enough, no runtime violation or hazard, and the chain (k = 1: 1 statistics kernel,
    1 label row kernel, 3 tensor-core ops) runs at alpha = 0 exactly when the batch holds an unlabelled row"""
    from boltzmann_machines import _native
    sim.fakecuda_reset()
    seen = []

    def on_step(step, y):
        seen.append((bool(np.any(y < 0)), counts(sim)))

    compare_semi_with_emulation(_native.CudaCRBM, alpha, beta, C_, sample_v, sample_h, fraction,
                                before_step=sim.fakecuda_reset, on_step=on_step)
    clean(sim)
    assert sim.fakecuda_hazard_launches() == 0
    for unl, (tc, post, cols, stats, upd, mult, total) in seen:
        chain = alpha > 0 or unl
        assert (post, cols, upd) == (1, 1, 1)
        assert stats == int(chain) and mult == int(chain) and tc == 2 + 3 * int(chain)
        assert total == tc + post + cols + stats + upd + mult + 1          # + the bf16 conversion of X


def test_emulation_detects_a_wrong_start():
    """the comparison above sees the start of the unlabelled rows' chain: drawing its label at another site, or starting
    from S^ instead of S at the drawn label, changes the variables by far more than its bound"""
    cfg = dict(n_visible=37, n_hidden=70, n_classes=10, alpha=1.0, beta=1.0, l2=1e-3, max_batch=64, sample_v=True,
               sample_h=True)
    rng = np.random.RandomState(0)
    p = {'W': 0.3 * rng.randn(37, 70), 'U': 0.3 * rng.randn(10, 70), 'vb': 0.1 * rng.randn(37), 'hb': 0.1 * rng.randn(70),
         'yb': 0.1 * rng.randn(10)}
    X, y = (rng.rand(45, 37) < 0.4).astype(np.float32), semi_labels(rng, 45, 10, 'some')

    def run(**over):
        m = OracleSemiCRBMbf16(cfg)
        for k, v in over.items():
            setattr(m, k, v)
        m.set_params(p)
        m.train_step(X, y, 0.1, 0.5, 1, seed=23, tick=0)
        return m.get_params()

    ref = run()
    for other in (run(start_site=12), run(start_from_mean=True)):
        assert not all(close_enough(other[n], ref[n]).all() for n in ('W', 'U', 'yb', 'hb'))


def test_refusals_launch_nothing(sim):
    X = np.zeros((10, 30), np.float32)
    cases = [(0.0, -1), (0.5, -2), (0.5, 10), (0.0, -2)]
    for beta, bad in cases:
        e = engine(beta=beta)
        y = np.zeros(10, np.int32)
        y[4] = bad
        sim.fakecuda_reset()
        with pytest.raises(RuntimeError, match='outside'):
            e.train_step(X, y, 0.1, 0.5, 1, seed=1, tick=0)
        assert sim.fakecuda_launches(b'') == 0
        e.close()
    for beta in (-0.5, float('nan'), float('inf')):
        sim.fakecuda_reset()
        with pytest.raises(RuntimeError, match='beta'):
            engine(beta=beta)
        assert sim.fakecuda_launches(b'') == 0


def test_all_unlabelled_metrics_are_nan(sim):
    e = engine(alpha=0.0)
    X = (np.random.RandomState(0).rand(12, 30) < 0.5).astype(np.float32)
    m = e.train_step(X, np.full(12, -1), 0.1, 0.5, 1, seed=1, tick=0, metrics=True)
    assert np.isnan(m['nll']) and np.isnan(m['accuracy'])
    y = np.full(12, -1)
    y[:4] = [1, 2, 3, 4]
    m = e.train_step(X, y, 0.1, 0.5, 1, seed=1, tick=1, metrics=True)
    assert np.isfinite(m['nll']) and m['accuracy'] in (0.0, 0.25, 0.5, 0.75, 1.0)
    clean(sim)
    e.close()
