"""Every stage of the classification RBM's step (csrc/bm_crbm_tc.cuh) at the benchmark's shapes and at the kernels' edges,
replayed in float64 from the engine's own intermediates (CudaCRBM.debug_last_step; the checks and their bounds are in
tests/class_rbm_replay.py).  The float64 work runs with torch on the same GPU, in row chunks.

Split arithmetic (the engine does not report it).  Row splits: ceil(rows / 64).  Split-K slices of the dW op:
s1 = max(1, min((SMs / 2) / (ceil(V / 256) ceil(H / 256)), ceil(rows / 64))); for 784-1024 on a 132-SM H100 that is
min(66 / 16, ...) = 4 at 4096 rows and 2 at 128 rows.  Column blocks: ceil(H / 128) (8 at H = 1024, 2 at H = 129).

Dry run without a GPU: BM_HOSTSIM=1 python -m pytest tests/test_zz_class_rbm_replay_gpu.py -m gpu runs the small cases on the
stand-in runtime with the classification RBM's kernels restated on the CPU (tests/hostsim/build_crbm_semi.sh)."""
import ctypes as Ct
import os
import subprocess

import numpy as np
import pytest

import class_rbm_replay as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM = os.environ.get('BM_HOSTSIM') == '1'
big = pytest.mark.skipif(HOSTSIM, reason='benchmark size: hours on the scalar interpreter; the H100 runs it')


@pytest.fixture(scope='module', autouse=True)
def _hostsim_with_the_crbm_kernels():
    """BM_HOSTSIM=1: run this module on the stand-in runtime that also interprets the classification RBM's kernels"""
    if not HOSTSIM:
        yield
        return
    from boltzmann_machines import _native
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_crbm_semi.sh')], stdout=subprocess.DEVNULL)
    lib = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_crbm_semi.so'))
    lib.fakecuda_violation.restype = Ct.c_char_p
    lib.fakecuda_skipped.restype = Ct.c_char_p
    lib.fakecuda_set_execute(1)
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    yield
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib
    v, sk = lib.fakecuda_violation().decode(), lib.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


@pytest.fixture(scope='module', autouse=True)
def _report():
    R.reset_report()
    yield
    print('\nclassification RBM replay: draws checked {draws}, ambiguous {ambiguous}; rebuilt h draws {h_rebuilt}, ambiguous '
          '{h_ambiguous}'.format(**R.REPORT))
    for k, v in sorted(R.REPORT['worst'].items()):
        print('  worst |difference| / bound  {0:14s} {1:.3g}'.format(k, v))


def device():
    return 'cpu' if HOSTSIM else 'cuda'


def sm_count():
    import torch
    return 132 if HOSTSIM else torch.cuda.get_device_properties(0).multi_processor_count


def engine(cfg):
    from boltzmann_machines import _native
    return _native.CudaCRBM(cfg)


def cfg_of(V, H, C, max_batch, alpha=0.0, beta=0.0, sample_v=False, sample_h=True, l2=1e-4):
    return dict(n_visible=V, n_hidden=H, n_classes=C, alpha=alpha, beta=beta, l2=l2, max_batch=max_batch, sample_v=sample_v,
                sample_h=sample_h)


def params(rng, V, H, C):
    p = {'W': 0.05 * rng.randn(V, H), 'U': 0.3 * rng.randn(C, H), 'vb': 0.1 * rng.randn(V), 'hb': 0.1 * rng.randn(H),
         'yb': 0.1 * rng.randn(C)}
    p.update({'d' + k: np.zeros_like(v) for k, v in list(p.items())})
    return {k: v.astype(np.float32) for k, v in p.items()}


def data(rng, rows, V, C):
    """class-conditional binary rows: each class a prototype of per-pixel probabilities"""
    protos = np.clip(rng.beta(0.5, 0.5, size=(C, V)), 0.05, 0.95)
    y = rng.randint(0, C, size=rows)
    return (rng.rand(rows, V) < protos[y]).astype(np.float32), y


def two_steps(cfg, rows, k=1, unl=None, seed=5):
    """step 1 at lr 1, momentum 0 (the momenta are the gradients), then step 2 without set_params at lr 0.3, momentum 0.5:
    the update formula and the bf16 shadows step 1 left.  unl(rng, y) marks rows -1."""
    V, H, C = cfg['n_visible'], cfg['n_hidden'], cfg['n_classes']
    rng = np.random.RandomState(V + H + C + rows)
    eng = engine(cfg)
    eng.set_params(params(rng, V, H, C))
    for step, (lr, mom) in enumerate(((1.0, 0.0), (0.3, 0.5))):
        X, y = data(rng, rows, V, C)
        if unl is not None:
            unl(rng, y)
        R.run_step(eng, cfg, X, y, lr, mom, k, seed, step, sm_count(), device())
    eng.close()


# ---- the benchmark's shapes: 784-1024-10, max_batch 4096 ----------------------------------------------------------------------
@big
@pytest.mark.parametrize('rows', [128, 4096])
@pytest.mark.parametrize('alpha,sample_v,sample_h', [(0.0, False, True), (0.01, False, True)])
def test_benchmark_steps(rows, alpha, sample_v, sample_h):
    """alpha = 0 (no chain) and the benchmark's hybrid setting (alpha 0.01, k 1, sample_h)"""
    cfg = cfg_of(784, 1024, 10, 4096, alpha=alpha, sample_v=sample_v, sample_h=sample_h)
    from boltzmann_machines import _native
    ctx = _native.Context.default()
    before = ctx.launch_count()
    two_steps(cfg, rows)
    # premise: the launches a step makes do not depend on reading its buffers (debug_last_step launches nothing)
    eng = engine(cfg)
    rng = np.random.RandomState(1)
    eng.set_params(params(rng, 784, 1024, 10))
    X, y = data(rng, rows, 784, 10)
    n0 = ctx.launch_count()
    eng.train_step(X, y, 0.1, 0.5, 1, seed=3, tick=0)
    n1 = ctx.launch_count()
    eng.debug_last_step(('A', 'P', 'y0', 'G') + (('h0', 'x_k', 'y_k', 'h_k', 'aH') if alpha > 0 else ()))
    assert ctx.launch_count() == n1 and before < n0
    eng.train_step(X, y, 0.1, 0.5, 1, seed=3, tick=1)
    assert ctx.launch_count() - n1 == n1 - n0
    # and reading changes no result: the same two steps without reading, bit for bit
    quiet = engine(cfg)
    quiet.set_params(params(np.random.RandomState(1), 784, 1024, 10))
    for tick in (0, 1):
        quiet.train_step(X, y, 0.1, 0.5, 1, seed=3, tick=tick)
    a, b = eng.get_params(), quiet.get_params()
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    eng.close()
    quiet.close()


@big
@pytest.mark.parametrize('sample_h', [True, False])
def test_benchmark_chain_prefixes(sample_h):
    """alpha = 1, sampled x and label, CD-1 .. CD-5 from the same state at 4096 rows, each sweep replayed"""
    cfg = cfg_of(784, 1024, 10, 4096, alpha=1.0, sample_v=True, sample_h=sample_h)
    rng = np.random.RandomState(11)
    X, y = data(rng, 4096, 784, 10)
    eng = engine(cfg)
    R.check_prefixes(eng, cfg, params(rng, 784, 1024, 10), X, y, 5, 7, 3, sm_count(), device())
    eng.close()


# ---- semi-supervised rows ---------------------------------------------------------------------------------------------------
def edges(rng, y):
    """rows on both sides of two split edges, and the second split wholly unlabelled"""
    y[[63, 64, 127, 128]] = -1
    y[64:128] = -1


def half(rng, y):
    edges(rng, y)
    y[rng.rand(len(y)) < 0.5] = -1


def every(rng, y):
    y[:] = -1


@big
@pytest.mark.parametrize('unl', [half, every], ids=['50%', '100%'])
@pytest.mark.parametrize('alpha', [0.0, 0.01])
def test_semi_supervised_benchmark_steps(unl, alpha):
    two_steps(cfg_of(784, 1024, 10, 4096, alpha=alpha, beta=0.1), 4096, unl=unl)


@big
def test_semi_without_unlabelled_rows_is_the_labelled_step():
    """beta = 0.1 on a batch with no -1 (0 % unlabelled) is the beta = 0 step, bit for bit, and passes the replay"""
    rng = np.random.RandomState(4)
    p = params(rng, 784, 1024, 10)
    X, y = data(rng, 4096, 784, 10)
    out = []
    for beta in (0.1, 0.0):
        cfg = cfg_of(784, 1024, 10, 4096, alpha=0.01, beta=beta)
        eng = engine(cfg)
        eng.set_params(p)
        R.run_step(eng, cfg, X, y, 1.0, 0.0, 1, 5, 0, sm_count(), device())
        out.append(eng.get_params())
        eng.close()
    for k in out[0]:
        assert np.array_equal(out[0][k], out[1][k]), k


# ---- edges: class-count templates, partial column blocks, ragged V, row counts around the splits -----------------------------
EDGES = [  # (V, H, C, rows, max_batch, alpha, beta, sample_v, sample_h, unlabelled)
    (781, 1000, 17, 4033, 4096, 0.01, 0.1, False, True, True),
    (784, 129, 16, 65, 128, 1.0, 0.0, True, True, False),
    (781, 129, 64, 63, 64, 1.0, 0.5, True, False, True),
    (784, 1000, 33, 1, 64, 0.01, 0.0, False, True, False),
    (781, 129, 2, 4033, 4096, 0.0, 0.1, True, True, True),
    (40, 300, 17, 150, 150, 1.0, 0.5, True, True, True),
    (37, 129, 64, 65, 128, 0.5, 0.0, True, True, False),
    (37, 129, 2, 63, 64, 0.0, 0.0, False, True, False),
]


def _small(e):
    return e[0] * e[1] * e[3] <= 1e6


@pytest.mark.parametrize('e', [pytest.param(e, marks=() if _small(e) else big) for e in EDGES],
                         ids=['V{0}-H{1}-C{2}-rows{3}'.format(*e) for e in EDGES])
def test_edges(e):
    V, H, C, rows, mb, alpha, beta, sv, sh, unl = e
    mark = None
    if unl:
        mark = edges if rows > 128 else (lambda rng, y: y.__setitem__(slice(0, None, 3), -1))
    two_steps(cfg_of(V, H, C, mb, alpha=alpha, beta=beta, sample_v=sv, sample_h=sh), rows, unl=mark)


# ---- queries ----------------------------------------------------------------------------------------------------------------
@big
def test_predict_proba_and_transform_ragged_chunks():
    """65 536 + 37 rows at max_batch 4096: 17 chunks, the last of 37 rows; every row within its bound"""
    rng = np.random.RandomState(8)
    cfg = cfg_of(784, 1024, 10, 4096, alpha=0.01)
    eng = engine(cfg)
    p = params(rng, 784, 1024, 10)
    eng.set_params(p)
    X, _ = data(rng, 65536 + 37, 784, 10)
    R.check_queries(p, X, eng.predict_proba(X), eng.transform(X), device())
    with pytest.raises(RuntimeError, match='no training step'):
        eng.debug_last_step(('A',))
    eng.close()


def test_debug_last_step_refusals():
    cfg = cfg_of(37, 129, 10, 64, alpha=0.0)
    eng = engine(cfg)
    rng = np.random.RandomState(2)
    eng.set_params(params(rng, 37, 129, 10))
    X, y = data(rng, 20, 37, 10)
    eng.train_step(X, y, 0.1, 0.5, 1, seed=1, tick=0)
    from boltzmann_machines import _native
    lib = _native.load_library() if not HOSTSIM else _native._lib
    buf = np.empty((20, 129), np.float32)
    assert lib.bm_crbm_debug_last_step(eng.handle, b'A', buf.ctypes.data, buf.nbytes - 4) != 0       # size mismatch
    assert lib.bm_crbm_debug_last_step(eng.handle, b'Q', buf.ctypes.data, buf.nbytes) != 0           # unknown name
    assert lib.bm_crbm_debug_last_step(eng.handle, b'h_k', buf.ctypes.data, 20 * 129 * 2) != 0       # no chain at alpha 0
    assert lib.bm_crbm_debug_last_step(eng.handle, b'A', buf.ctypes.data, buf.nbytes) == 0
    eng.close()
