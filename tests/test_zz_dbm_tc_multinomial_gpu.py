"""Multinomial hidden layers on the tensor-core DBM engine (compute='bf16', csrc/bm_dbm_tc.cuh) on the GPU: the fused row
kernel bit for bit against the CUDA-core engine's softmax_rows + multinomial_rows, the engine against its bf16 emulation
(tests/dbm_bf16_multinomial.py), and dbm_cifar_naive.py's DBM shape against the emulation and the fp32 engine.

Dry run without a GPU: BM_HOSTSIM=1 python -m pytest tests/test_zz_dbm_tc_multinomial_gpu.py -m gpu (on the stand-in runtime
with the row kernel's CPU restatement linked in, tests/hostsim/build_dbm_multinomial.sh)."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P
from oracle.rbm import bf16_round

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B_, M_ = 'bernoulli', 'multinomial'


@pytest.fixture(scope='module', autouse=True)
def _hostsim_with_the_row_kernel():
    """BM_HOSTSIM=1: run this module on the stand-in runtime that also interprets dbm_multinomial_rows_kernel; no runtime
    violation and no kernel without a CPU restatement may occur."""
    if os.environ.get('BM_HOSTSIM') != '1':
        yield
        return
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_multinomial.sh')], stdout=subprocess.DEVNULL)
    lib = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_multinomial.so'))
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


def emulation():
    spec = importlib.util.spec_from_file_location('dbm_bf16_multinomial', os.path.join(ROOT, 'tests', 'dbm_bf16_multinomial.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.OracleDBMbf16Multinomial


def make_cfg(kinds, Hs, V=30, n_samples=300, gaussian=False, B=10, M=12, **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='gaussian' if gaussian else 'bernoulli', h_kinds=list(kinds),
               h_n_samples=[float(n_samples)] * L, dtype='float32', compute='bf16', n_particles=M, batch_size=B,
               max_mf_updates=6, mf_tol=1e-6, l2=1e-4, max_norm=3.0, sample_v=True, sample_h=[True] * L,
               sparsity_target=[0.2] * L, sparsity_cost=[0.01] * L, sparsity_damping=0.9)
    if gaussian:
        cfg['sigma'] = np.ones(V) if V > 100 else np.linspace(0.7, 1.3, V)
    cfg.update(kw)
    return cfg


def init(cfg, engines, scale=0.3, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [cfg['n_visible']] + cfg['n_hiddens']
    d = {'vb': (0.1 * rng.randn(sizes[0])).astype(np.float32)}
    for i in range(len(cfg['n_hiddens'])):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = (0.1 * rng.randn(sizes[i + 1])).astype(np.float32)
    for e in engines:
        e.set_params(d)
        e.init_particles(4242)


def batch(cfg, rows, seed):
    rng = np.random.RandomState(seed)
    if cfg['v_kind'] == 'gaussian':
        return rng.randn(rows, cfg['n_visible']).astype(np.float32)
    return (rng.rand(rows, cfg['n_visible']) < 0.3).astype(np.float32)


def check_counts(cfg, g):
    for i, kind in enumerate(cfg['h_kinds']):
        if kind == 'multinomial' and cfg['sample_h'][i]:
            h = g['h' + ('' if i == 0 else '_%d' % i)]
            assert np.array_equal(h, np.round(h)) and np.all(h >= 0), i
            np.testing.assert_array_equal(h.sum(axis=1), np.full(h.shape[0], cfg['h_n_samples'][i], np.float32))


@pytest.mark.parametrize('rows,cols,n', [(300, 1000, 1000), (64, 7800, 512), (130, 11, 6), (257, 513, 300)])
@pytest.mark.parametrize('draws', [False, True], ids=['means', 'counts'])
def test_row_kernel_is_bit_identical_to_softmax_then_multinomial_rows(rows, cols, n, draws):
    pre = (3.0 * np.random.RandomState(cols).randn(rows, cols)).astype(np.float32)
    out_bf, out_f32, ref_means, ref_counts = _native.debug_dbm_multinomial_rows(pre, n, n if draws else 0, 77, P.SITE_DBM_H + 1, 3, 5)
    want = ref_counts if draws else ref_means
    np.testing.assert_array_equal(out_f32.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(out_bf, (bf16_round(want).view(np.uint32) >> 16).astype(np.uint16))
    if draws:
        np.testing.assert_array_equal(want.sum(axis=1), np.full(rows, n, np.float32))


CASES = [((B_, M_), (18, 11), 6, False), ((M_, B_), (19, 13), 300, False), ((B_, M_, B_), (18, 11, 7), 1000, False),
         ((B_, M_), (18, 11), 300, True), ((M_,), (21,), 1000, False)]


@pytest.mark.parametrize('kinds,Hs,n_samples,gaussian', CASES)
def test_training_and_queries_track_the_emulation(kinds, Hs, n_samples, gaussian):
    """GEMM summation order and the epilogue's ex2-based sigmoid differ from numpy's in the last bits: means agree to about
    one bf16 ulp, a categorical (or Bernoulli) draw may differ where u falls within rounding of a CDF boundary."""
    cfg = make_cfg(kinds, Hs, n_samples=n_samples, gaussian=gaussian)
    eng, emu = _native.CudaDBM(cfg), emulation()(cfg)
    assert eng.compute == 'bf16'
    init(cfg, (eng, emu))
    for it in range(3):
        X = batch(cfg, 10, it)
        a = eng.train_step(X, 0.05, 0.5, 2, 99, it, metrics=('msre', 'n_mf_updates'))
        b = emu.train_step(X, 0.05, 0.5, 2, 99, it, metrics=('msre', 'n_mf_updates'))
        assert a['msre'] == pytest.approx(b['msre'], rel=0.05), it
        assert abs(a['n_mf_updates'] - b['n_mf_updates']) <= 1, it
    g, w = eng.get_params(), emu.get_params()
    for k in w:
        if k.startswith(('W', 'dW', 'vb', 'hb', 'dvb', 'dhb')):
            np.testing.assert_allclose(g[k], w[k], atol=2e-2, err_msg=k)
    check_counts(cfg, g)
    for i, kind in enumerate(kinds):
        k = 'h' + ('' if i == 0 else '_%d' % i)
        assert np.mean(np.any(g[k] != w[k], axis=1)) <= 0.25, (k, np.mean(np.any(g[k] != w[k], axis=1)))
    Xq = batch(cfg, 7, 9)
    top_scale = n_samples if kinds[-1] == M_ else 1          # multinomial means sum to n_samples per row
    np.testing.assert_allclose(eng.transform(Xq), emu.transform(Xq), rtol=2.0 ** -5, atol=2e-2 * top_scale)
    np.testing.assert_allclose(eng.reconstruct(Xq), emu.reconstruct(Xq), rtol=2.0 ** -5, atol=2e-2)
    v = eng.sample_v(2, 11, 4)
    assert v.shape == (12, cfg['n_visible']) and np.all(np.isfinite(v))
    check_counts(cfg, eng.get_params())
    eng.close()


@pytest.mark.parametrize('stop', [2, 5, 7, 'never', 'no-updates'])
def test_e_step_stops_where_the_emulation_does(stop):
    cfg = make_cfg((B_, M_), (18, 11), n_samples=6, max_mf_updates=0 if stop == 'no-updates' else 12, mf_tol=-1.0)
    X = batch(cfg, 7, 9)
    if isinstance(stop, int):
        probe = emulation()(cfg)
        init(cfg, (probe,), scale=0.6)
        cfg['mf_tol'] = probe.mf_tol_stopping_at(X, stop)
        assert cfg['mf_tol'] is not None, 'no tolerance stops the emulation after %d sweeps' % stop
    eng, emu = _native.CudaDBM(cfg), emulation()(cfg)
    init(cfg, (eng, emu), scale=0.6)
    mu0 = eng.get_params(['mu_1'])['mu_1']
    a, b = eng.val_metrics(X, 1, 7, 3), emu.val_metrics(X, 1, 7, 3)
    assert b['n_mf_updates'] == {'never': 12, 'no-updates': 0}.get(stop, stop)
    assert abs(a['n_mf_updates'] - b['n_mf_updates']) <= 1
    assert a['msre'] == pytest.approx(b['msre'], rel=1e-2)
    g, w = eng.get_params(['mu', 'mu_1']), emu.get_params(['mu', 'mu_1'])
    np.testing.assert_allclose(g['mu'], w['mu'], rtol=2.0 ** -7, atol=1e-3)
    np.testing.assert_allclose(g['mu_1'], w['mu_1'], rtol=2.0 ** -6, atol=2e-3)
    if stop == 'no-updates':
        np.testing.assert_array_equal(g['mu_1'], mu0)
    eng.close()


def test_cifar_naive_shape_tracks_the_emulation_and_the_fp32_engine():
    """examples/dbm_cifar_naive.py's DBM: Gaussian 3072 -> Bernoulli 5000 -> multinomial 1000 (n_samples 1000), batch =
    particles = 100, 1 Gibbs step, 10 mean-field updates.  Three steps against the emulation; one step against the fp32 engine:
    MSRE within 2 %, and the bf16 E-step stops no later than the fp32 one (DESIGN §9)."""
    cfg = make_cfg((B_, M_), (5000, 1000), V=3072, n_samples=1000, gaussian=True, B=100, M=100, max_mf_updates=10,
                   mf_tol=1e-7, sparsity_cost=[0., 0.], max_norm=np.inf, l2=1e-5)
    tc, simt, emu = _native.CudaDBM(cfg), _native.CudaDBM(dict(cfg, compute='fp32')), emulation()(cfg)
    assert tc.compute == 'bf16' and simt.compute == 'fp32'
    init(cfg, (tc, simt, emu), scale=0.01)
    for it in range(3):
        X = batch(cfg, 100, it)
        a = tc.train_step(X, 1e-3, 0.5, 1, 7, it, metrics=('msre', 'n_mf_updates'))
        b = emu.train_step(X, 1e-3, 0.5, 1, 7, it, metrics=('msre', 'n_mf_updates'))
        assert a['msre'] == pytest.approx(b['msre'], rel=1e-2), it
        assert abs(a['n_mf_updates'] - b['n_mf_updates']) <= 1, it
        if it == 0:
            c = simt.train_step(X, 1e-3, 0.5, 1, 7, it, metrics=('msre', 'n_mf_updates'))
            assert a['msre'] == pytest.approx(c['msre'], rel=0.02)
            assert 1 <= a['n_mf_updates'] <= c['n_mf_updates']
    g, w = tc.get_params(['W', 'W_1', 'vb', 'hb', 'hb_1', 'h_1']), emu.get_params(['W', 'W_1', 'vb', 'hb', 'hb_1', 'h_1'])
    for k in ('W', 'W_1', 'vb', 'hb', 'hb_1'):
        rel = np.linalg.norm(g[k] - w[k]) / max(np.linalg.norm(w[k]), 1e-12)
        assert rel < 0.02, (k, rel)
    check_counts(cfg, g)
    tc.close(); simt.close()
