"""Semi-supervised classification RBM on the H100 (rows labelled -1 with beta > 0, csrc/bm_crbm_tc.cuh) against its float64
statement and its bf16 emulation (tests/class_rbm_semi.py).

The float64 statement is evaluated on the operands as the engine rounds them, as in tests/test_zz_class_rbm_gpu.py, and held
to the same bounds: 1e-3 on the variables after three steps of means-only chains.  With sampled chains the engine is held to
the emulation after every step (1 bf16 ulp or 2e-5).

Dry run without a GPU: BM_HOSTSIM=1 python -m pytest tests/test_zz_class_rbm_semi_gpu.py -m gpu (on the stand-in runtime with
the classification RBM's semi-supervised restatements linked in, tests/hostsim/build_crbm_semi.sh)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from class_rbm_semi import OracleSemiCRBM, compare_semi_with_emulation, semi_labels

from oracle.rbm import bf16_round

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM = os.environ.get('BM_HOSTSIM') == '1'


@pytest.fixture(scope='module', autouse=True)
def _hostsim_with_the_crbm_kernels():
    """BM_HOSTSIM=1: run this module on the stand-in runtime that also interprets the classification RBM's kernels"""
    if not HOSTSIM:
        yield
        return
    from boltzmann_machines import _native
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_crbm_semi.sh')], stdout=subprocess.DEVNULL)
    lib = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_crbm_semi.so'))
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    lib.fakecuda_set_execute(0 if os.environ.get('BM_HOSTSIM_EXECUTE') == '0' else 1)
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    yield
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib
    v, sk = lib.fakecuda_violation().decode(), lib.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


class RoundedSemiOracle(OracleSemiCRBM):
    """the float64 model on the engine's bf16 operands"""
    def _r(self, x):
        return bf16_round(x).astype(np.float64)

    def _w(self, name):
        return bf16_round(self.p[name]).astype(np.float64)


@pytest.mark.parametrize('fraction', ['some', 'all'])
@pytest.mark.parametrize('C', [2, 10, 64])
@pytest.mark.parametrize('alpha', [0.0, 0.01])
def test_means_only_semi_steps_against_float64(alpha, C, fraction):
    from boltzmann_machines import _native
    cfg = dict(n_visible=50, n_hidden=70, n_classes=C, alpha=alpha, beta=0.5, l2=1e-4, max_batch=64, sample_v=False,
               sample_h=False)
    eng, ora = _native.CudaCRBM(cfg), RoundedSemiOracle(cfg)
    rng = np.random.RandomState(C)
    p = {'W': 0.3 * rng.randn(50, 70), 'U': 0.3 * rng.randn(C, 70), 'vb': 0.1 * rng.randn(50), 'hb': 0.1 * rng.randn(70),
         'yb': 0.1 * rng.randn(C)}
    p = {k: v.astype(np.float32) for k, v in p.items()}
    eng.set_params(p)
    ora.set_params(p)
    for step in range(3):
        X = (rng.rand(45, 50) < 0.4).astype(np.float32)
        y = semi_labels(rng, 45, C, fraction)
        got = eng.train_step(X, y, 0.1, 0.5, 1, seed=5, tick=step, metrics=True)
        want = ora.train_step(X, y, 0.1, 0.5, 1, seed=5, tick=step, metrics=True)
        if fraction == 'all':
            assert np.isnan(got['nll']) and np.isnan(got['accuracy'])
        else:
            n_lab = int(np.sum(y >= 0))
            assert abs(got['nll'] - want['nll']) < 1e-4 * max(1.0, want['nll'])
            assert abs(got['accuracy'] - want['accuracy']) <= 1 / n_lab + 1e-12
    g, w = eng.get_params(), ora.get_params()
    for name in w:
        np.testing.assert_allclose(g[name], w[name], rtol=0, atol=1e-3, err_msg=name)
    eng.close()


@pytest.mark.parametrize('sample_v,sample_h', [(True, True), (True, False), (False, True)])
@pytest.mark.parametrize('C', [2, 10, 64])
@pytest.mark.parametrize('fraction', ['some', 'all'])
def test_sampled_semi_chain_equals_the_bf16_emulation(fraction, C, sample_v, sample_h):
    """alpha = beta = 1, so that the chain's draws (the start label at site 13, h0 at 1, x at 2, the label at 12, h at 3)
    carry their full weight; every variable is compared after every step"""
    from boltzmann_machines import _native
    compare_semi_with_emulation(_native.CudaCRBM, 1.0, 1.0, C, sample_v, sample_h, fraction)


def synthetic(n, V=784, C=10, seed=0):
    """seeded class-conditional binary data (as tests/test_zz_class_rbm_gpu.py): each class a prototype of per-pixel
    probabilities"""
    rng = np.random.RandomState(seed)
    protos = np.clip(rng.beta(0.5, 0.5, size=(C, V)), 0.05, 0.95)
    y = rng.randint(0, C, size=n)
    return (rng.rand(n, V) < protos[y]).astype(np.float32), y


@pytest.mark.skipif(HOSTSIM, reason='about 4e10 multiply-adds: hours on the scalar interpreter; the H100 runs it')
def test_784_1024_10_semi_supervised_three_epochs_against_the_oracle(tmp_path):
    """Engine and float64 statement trained from the same weights: 3 epochs on 3 000 rows of which every tenth (300) keeps
    its label, beta = 0.1 (alpha 0.01, k 1, learning rate 0.1).  The float64 statement reaches 100.0 % test accuracy and a
    mean NLL of 1.321 nats on this data (its CPU run; at learning rate 0.05 it reached only 19.2 %, so the NLL would have
    been the only informative check there too); the bounds (1 point, 0.05 nats) were chosen before any engine run, as in the
    labelled test."""
    from boltzmann_machines import ClassificationRBM
    from boltzmann_machines.base import set_engine_factory
    from class_rbm_semi import semi_factory
    X, y = synthetic(4000, seed=0)
    Xtr, ytr, Xte, yte = X[:3000], y[:3000].copy(), X[3000:], y[3000:]
    ytr[np.arange(3000) % 10 != 0] = -1
    kw = dict(n_visible=784, n_hidden=1024, n_classes=10, alpha=0.01, beta=0.1, learning_rate=0.1, momentum=0.5,
              max_epoch=3, batch_size=100, random_seed=11, verbose=False, save_after_each_epoch=False)
    res = {}
    for name in ('cuda', 'oracle'):
        old = set_engine_factory('crbm', semi_factory) if name == 'oracle' else None
        try:
            m = ClassificationRBM(model_path=str(tmp_path / name) + '/', **kw)
            m.fit(Xtr, ytr)
            P = m.predict_proba(Xte).astype(np.float64)
        finally:
            if name == 'oracle':
                set_engine_factory('crbm', old)
        res[name] = (np.mean(np.argmax(P, 1) == yte), -np.mean(np.log(np.maximum(P[np.arange(len(yte)), yte], 1e-30))))
    (acc_c, nll_c), (acc_o, nll_o) = res['cuda'], res['oracle']
    assert abs(acc_c - acc_o) <= 0.01, res
    assert abs(nll_c - nll_o) <= 0.05, res
