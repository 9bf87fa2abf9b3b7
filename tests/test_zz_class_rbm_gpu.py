"""Classification RBM on the H100 (csrc/bm_crbm_tc.cuh) against its float64 statement (oracle/crbm.py).

The oracle is evaluated on the operands as the engine rounds them (X and the W shadow in bf16; U, the biases and every
variable in fp32), so what remains is fp32 accumulation and the bf16 rounding of the gradient operands and chain
activations.  The bounds below are set from that: the posterior to 2e-5 (H <= 100 softplus sums in fp32), a few steps of
training to 1e-3 of the variables.  The engine is also held to its bf16 emulation (tests/class_rbm_bf16.py) step by step,
sampled chains included, to 1 bf16 ulp or 2e-5.

Dry run without a GPU: BM_HOSTSIM=1 python -m pytest tests/test_zz_class_rbm_gpu.py -m gpu (on the stand-in runtime with
the classification RBM's restatements linked in, tests/hostsim/build_crbm.sh)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from class_rbm_bf16 import compare_with_emulation

from oracle.crbm import OracleCRBM
from oracle.rbm import bf16_round

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM = os.environ.get('BM_HOSTSIM') == '1'


@pytest.fixture(scope='module', autouse=True)
def _hostsim_with_the_crbm_kernels():
    """BM_HOSTSIM=1: run this module on the stand-in runtime that also interprets the classification RBM's kernels and the
    label's row kernel; no runtime violation and no kernel without a CPU restatement may occur."""
    if not HOSTSIM:
        yield
        return
    from boltzmann_machines import _native
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_crbm.sh')], stdout=subprocess.DEVNULL)
    lib = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_crbm.so'))
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
    print('kernels without a CPU restatement: none')


class RoundedOracle(OracleCRBM):
    """the float64 model on the engine's bf16 operands"""
    def _r(self, x):
        return bf16_round(x).astype(np.float64)

    def _w(self, name):
        return bf16_round(self.p[name]).astype(np.float64)


def pair(V, H, C, seed=0, scale=0.3, **kw):
    from boltzmann_machines import _native
    cfg = dict(n_visible=V, n_hidden=H, n_classes=C, alpha=0.01, l2=1e-4, max_batch=64, sample_v=False, sample_h=False)
    cfg.update(kw)
    eng, ora = _native.CudaCRBM(cfg), RoundedOracle(cfg)
    rng = np.random.RandomState(seed)
    p = {'W': scale * rng.randn(V, H), 'U': scale * rng.randn(C, H), 'vb': 0.1 * rng.randn(V), 'hb': 0.1 * rng.randn(H),
         'yb': 0.1 * rng.randn(C)}
    p = {k: v.astype(np.float32) for k, v in p.items()}
    eng.set_params(p)
    ora.set_params(p)
    return eng, ora, rng


@pytest.mark.parametrize('C', [2, 10, 64])
def test_posterior_and_transform_against_float64(C):
    eng, ora, rng = pair(100, 70, C)
    X = (rng.rand(150, 100) < 0.3).astype(np.float32)          # three chunks of max_batch rows
    np.testing.assert_allclose(eng.predict_proba(X), ora.predict_proba(X), rtol=0, atol=2e-5)
    np.testing.assert_allclose(eng.transform(X), ora.transform(X), rtol=0, atol=2e-5)
    eng.close()


@pytest.mark.parametrize('alpha', [0.0, 0.01, 1.0])
@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('C', [2, 10, 64])
def test_training_steps_against_float64(alpha, k, C):
    eng, ora, rng = pair(50, 70, C, seed=C, alpha=alpha)
    for step in range(3):
        X = (rng.rand(45, 50) < 0.4).astype(np.float32)
        y = rng.randint(0, C, size=45)
        got = eng.train_step(X, y, 0.1, 0.5, k, seed=5, tick=step, metrics=True)
        want = ora.train_step(X, y, 0.1, 0.5, k, seed=5, tick=step, metrics=True)
        # the variables differ by the bf16 rounding of the gradient operands: a relative bound on the NLL, one row on accuracy
        assert abs(got['nll'] - want['nll']) < 1e-4 * max(1.0, want['nll'])
        assert abs(got['accuracy'] - want['accuracy']) <= 1 / 45 + 1e-12
    g, w = eng.get_params(), ora.get_params()
    for name in w:
        np.testing.assert_allclose(g[name], w[name], rtol=0, atol=1e-3, err_msg=name)
    eng.close()


@pytest.mark.parametrize('sample_v,sample_h', [(True, True), (False, True), (True, False)])
def test_sampled_chain_runs_and_stays_close(sample_v, sample_h):
    """the chain's draws follow the engine's bf16 means, so single draws may differ from the oracle's; alpha = 0.01 keeps
    their weight in the update small enough for a 2e-3 bound over three steps"""
    eng, ora, rng = pair(50, 70, 10, seed=4, sample_v=sample_v, sample_h=sample_h)
    for step in range(3):
        X = (rng.rand(45, 50) < 0.4).astype(np.float32)
        y = rng.randint(0, 10, size=45)
        eng.train_step(X, y, 0.1, 0.5, 2, seed=9, tick=step)
        ora.train_step(X, y, 0.1, 0.5, 2, seed=9, tick=step)
    g, w = eng.get_params(), ora.get_params()
    for name in w:
        np.testing.assert_allclose(g[name], w[name], rtol=0, atol=2e-3, err_msg=name)
    eng.close()


@pytest.mark.parametrize('sample_v,sample_h', [(True, True), (True, False), (False, True)])
@pytest.mark.parametrize('C', [2, 10, 64])
@pytest.mark.parametrize('k', [1, 3])
def test_sampled_chain_equals_the_bf16_emulation(k, C, sample_v, sample_h):
    """alpha = 1, so that the chain's draws (h0 at site 1, x at 2, the label at 12, h at 3) carry their full weight; every
    variable is compared after every step"""
    from boltzmann_machines import _native
    compare_with_emulation(_native.CudaCRBM, 1.0, k, C, sample_v, sample_h)


@pytest.mark.parametrize('alpha', [0.0, 0.01])
def test_means_only_steps_equal_the_bf16_emulation(alpha):
    from boltzmann_machines import _native
    compare_with_emulation(_native.CudaCRBM, alpha, 1, 10, False, False)


def synthetic(n, V=784, C=10, seed=0):
    """seeded class-conditional binary data: each class a prototype of per-pixel probabilities"""
    rng = np.random.RandomState(seed)
    protos = np.clip(rng.beta(0.5, 0.5, size=(C, V)), 0.05, 0.95)
    y = rng.randint(0, C, size=n)
    return (rng.rand(n, V) < protos[y]).astype(np.float32), y


@pytest.mark.skipif(HOSTSIM, reason='about 4e10 multiply-adds: hours on the scalar interpreter; the H100 runs it')
def test_784_1024_10_three_epochs_against_the_oracle(tmp_path):
    """Engine and float64 oracle trained from the same weights, 3 epochs of hybrid training (alpha 0.01, k 1).  The oracle
    reaches 89.1 % test accuracy and a mean NLL of 1.490 nats on this data (its CPU run); the bounds (1 point, 0.05 nats)
    were chosen before any engine run and are not derived from a measured spread."""
    from boltzmann_machines import ClassificationRBM
    from boltzmann_machines.base import set_engine_factory
    from oracle.crbm import crbm_factory
    X, y = synthetic(4000, seed=0)
    Xtr, ytr, Xte, yte = X[:3000], y[:3000], X[3000:], y[3000:]
    kw = dict(n_visible=784, n_hidden=1024, n_classes=10, alpha=0.01, learning_rate=0.05, momentum=0.5, max_epoch=3,
              batch_size=100, random_seed=11, verbose=False, save_after_each_epoch=False)
    res = {}
    for name in ('cuda', 'oracle'):
        old = set_engine_factory('crbm', crbm_factory) if name == 'oracle' else None
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
