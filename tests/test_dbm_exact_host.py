"""Exact log Z and log p*(v) of binary DBMs with a narrow odd side (DESIGN.md §5.4f), checked without a GPU.

* The statement (tests/dbm_exact_oracle.py): the chunked float64 enumeration of the odd layers against brute force over every
  unit (dbm_ais_depth_oracle.brute_log_Z / brute_log_p_v) at L = 1, 2, 3 with ragged widths, binary and grey rows.
* The tensor-core engine's host code on the stand-in runtime (tests/hostsim, build_dbm_exact.sh) against the statement within
  1e-4 nats: n_odd from 1 to 18 at L = 1, 2, 3, several launches per call, binary and grey rows, tempered and centered models;
  repeated calls; every refusal before any launch; the Python class.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dbm_ais_depth_oracle as A  # noqa: E402
import dbm_exact_oracle as E  # noqa: E402
from test_dbm_ais_depth_host import _stack, make_cfg, params  # noqa: E402

ROOT = os.path.dirname(HERE)
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_exact.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')

TOL = 1e-4


def rows(V, n=6, seed=0):
    """three binary rows and three grey ones"""
    rng = np.random.RandomState(seed)
    X = (rng.rand(n, V) < 0.4).astype(np.float32)
    X[n // 2:] = rng.rand(n - n // 2, V).astype(np.float32)
    return X


# ---- the statement ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('V,Hs', [(5, (4,)), (4, (3, 4)), (3, (3, 2, 3))], ids=['L1', 'L2', 'L3'])
def test_statement_is_brute_force(V, Hs):
    p = params(V, Hs, scale=0.9, seed=len(Hs))
    X = rows(V)
    for chunk_bits in (1, 16):
        lz, lp = E.exact(p, X, chunk_bits=chunk_bits)
        assert abs(lz - A.brute_log_Z(p)) < 1e-10
        np.testing.assert_allclose(lp, A.brute_log_p_v(p, X), rtol=0, atol=1e-10)


# ---- the engine on the stand-in runtime -------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_exact.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(SIM)
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    lib.fakecuda_reset()
    lib.fakecuda_set_execute(1)
    yield lib
    lib.fakecuda_set_execute(0)
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib


def clean(sim):
    v, sk = sim.fakecuda_violation().decode(), sim.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


def engine(c, d):
    from boltzmann_machines import _native
    e = _native.CudaDBM(c)
    assert e.compute == 'bf16'
    e.set_params(d)
    return e


# (V, Hs, log2 states per launch or 0 for the default): n_odd 1 .. 18; the 14- and 18-bit cases span several launches, the
# 18-bit one runs the two-step (n_odd, n_1 > 16) operands
CASES = [
    (5, (1,), 0), (9, (7,), 0), (11, (14,), 10), (6, (18,), 15),
    (7, (5, 6), 0), (6, (13, 4), 11),
    (5, (4, 3, 5), 0), (4, (6, 3, 8), 9),
]


@pytest.mark.parametrize('V,Hs,chunk', CASES, ids=['%d-%s' % (c[0], '-'.join(map(str, c[1]))) for c in CASES])
def test_engine_equals_the_statement(sim, V, Hs, chunk):
    p = params(V, Hs, scale=0.5, seed=sum(Hs))
    X = rows(V, seed=V)
    e = engine(make_cfg(Hs, V), p)
    if chunk:
        e.debug_exact_chunk(chunk)
    lp, lz = e.exact(X)
    want_z, want_p = E.exact(p, X)
    assert abs(lz - want_z) < TOL, (lz, want_z)
    np.testing.assert_allclose(lp, want_p, rtol=0, atol=TOL)
    assert e.exact(None)[0] is None and e.exact(None)[1] == lz          # log Z alone is the same pass without rows
    e.close()
    clean(sim)


def test_repeated_calls_and_launch_sizes_agree(sim):
    V, Hs = 6, (13, 4)
    p = params(V, Hs, scale=0.5, seed=3)
    X = rows(V, n=70)                                                   # two 64-row blocks of the rows kernel
    e = engine(make_cfg(Hs, V), p)
    lp, lz = e.exact(X)
    lp2, lz2 = e.exact(X)
    assert lz2 == lz and np.array_equal(lp2, lp)
    e.debug_exact_chunk(8)                                              # 32 launches instead of one
    lp3, lz3 = e.exact(X)
    assert abs(lz3 - lz) < 1e-10
    # the rows kernel's exponentials are fp32 against a running max that depends on where a launch starts
    np.testing.assert_allclose(lp3, lp, rtol=0, atol=1e-6)
    e.debug_exact_chunk(0)
    assert e.exact(None)[1] == lz
    e.close()
    clean(sim)


@pytest.mark.parametrize('what', ['tempered', 'centered'])
def test_tempered_and_centered_models_read_the_stored_parameters(sim, what):
    V, Hs = 5, (4, 3, 5)
    p = params(V, Hs, scale=0.5, seed=21)
    kw = dict(pt_betas=[1.0, 0.6, 0.3]) if what == 'tempered' else dict(centering=True, offset_rate=0.05)
    e = engine(make_cfg(Hs, V, **kw), p)
    e.init_particles(3)
    X = rows(V)
    lp, lz = e.exact(X)
    want_z, want_p = E.exact(p, X)
    assert abs(lz - want_z) < TOL
    np.testing.assert_allclose(lp, want_p, rtol=0, atol=TOL)
    e.close()
    clean(sim)


def test_large_pre_activations_stay_finite(sim):
    """|z| up to ~1e3: softplus(z) = max(z, 0) + log1p(exp(-|z|)) neither overflows nor loses the linear part"""
    V, Hs = 8, (6, 5)
    p = params(V, Hs, scale=60.0, bias=200.0, seed=5)
    X = rows(V)
    e = engine(make_cfg(Hs, V), p)
    lp, lz = e.exact(X)
    want_z, want_p = E.exact(p, X)
    assert np.isfinite(lz) and np.all(np.isfinite(lp))
    assert abs(lz - want_z) < 1e-6 * abs(want_z) + TOL, (lz, want_z)
    np.testing.assert_allclose(lp, want_p, rtol=1e-6, atol=TOL)
    e.close()
    clean(sim)


def test_refusals_launch_nothing(sim):
    from boltzmann_machines import _native
    ctx = _native.Context.default()
    V = 6
    X = np.zeros((4, V), np.float32)
    cases = [
        (make_cfg((5, 4), V, v_kind='gaussian', sigma=np.ones(V)), 'binary'),
        (make_cfg((5, 4, 3), V, h_kinds=['bernoulli', 'multinomial', 'bernoulli'], h_n_samples=[100., 3., 100.]), 'binary'),
        (make_cfg((5, 4), V, compute='fp32'), 'tensor-core engine'),
        (make_cfg((5, 4), V, dtype='float64'), 'tensor-core engine'),
        (make_cfg((33,), V), 'n_odd = 33'),
        (make_cfg((20, 4, 13), V), 'n_odd = 33'),
    ]
    for c, msg in cases:
        e = _native.CudaDBM(c)
        e.set_params(params(V, c['n_hiddens']) if c.get('dtype', 'float32') == 'float32' else
                     {k: v.astype(np.float64) for k, v in params(V, c['n_hiddens']).items()})
        n0 = ctx.launch_count()
        for call in (lambda: e.exact(None), lambda: e.exact(X.astype(np.float32))):
            with pytest.raises(NotImplementedError, match=msg):
                call()
        assert ctx.launch_count() == n0, c
        e.close()
    e = engine(make_cfg((5, 4), V), params(V, (5, 4)))
    n0 = ctx.launch_count()
    bad = X.copy()
    bad[2, 3] = np.nan
    with pytest.raises(RuntimeError, match='non-finite'):
        e.exact(bad)
    lib = _native._lib
    out = np.zeros(4)
    lz = C.c_double()
    assert lib.bm_dbm_exact(e.handle, None, 0, None, None) == -1                        # nothing to compute
    assert lib.bm_dbm_exact(e.handle, X.ctypes.data, 0, None, C.byref(lz)) == -1        # X without rows
    assert lib.bm_dbm_exact(e.handle, None, 4, out.ctypes.data, C.byref(lz)) == -1      # rows without X
    assert lib.bm_dbm_exact(e.handle, X.ctypes.data, 4, None, C.byref(lz)) == -1        # rows without log_p_star
    assert lib.bm_dbm_exact(e.handle, X.ctypes.data, -1, out.ctypes.data, C.byref(lz)) == -1
    with pytest.raises(ValueError):
        e.exact(np.zeros((4, V + 1), np.float32))
    assert ctx.launch_count() == n0
    e.close()
    clean(sim)


# ---- the Python class ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sizes', [(7, 5), (6, 5, 4, 3)], ids=['L1', 'L3'])
def test_python_exact_log_Z_and_log_proba(sim, tmp_path, sizes):
    m, X = _stack(tmp_path, list(sizes))
    prm = {n: v for n, v in m.get_tf_params(scope='weights').items()}
    want_z, want_p = E.exact(prm, X[:10])
    lz = m.exact_log_Z()
    assert isinstance(lz, float) and abs(lz - want_z) < TOL
    lp = m.exact_log_proba(X[:10])
    np.testing.assert_allclose(lp, want_p - want_z, rtol=0, atol=2 * TOL)
    np.testing.assert_allclose(m.exact_log_proba(X[:10], log_Z=0.0), want_p, rtol=0, atol=TOL)
    grey = np.random.RandomState(2).rand(3, sizes[0]).astype(np.float32)
    np.testing.assert_allclose(m.exact_log_proba(grey, log_Z=lz), E.exact(prm, grey)[1] - lz, rtol=0, atol=2 * TOL)
    assert m.exact_log_proba(X[:0]).shape == (0,)
    for bad in (X[:3, :-1], X[0], np.where(np.eye(3, sizes[0]) > 0, np.inf, X[:3])):
        with pytest.raises(ValueError):
            m.exact_log_proba(bad)
    clean(sim)


def test_python_refusals(sim, tmp_path):
    m64, X = _stack(tmp_path / 'f64', [6, 5, 4], dtype='float64')
    for call in (m64.exact_log_Z, lambda: m64.exact_log_proba(X[:4])):
        with pytest.raises(NotImplementedError, match='float32'):
            call()
    wide, X = _stack(tmp_path / 'wide', [6, 33])
    with pytest.raises(NotImplementedError, match='n_odd = 33'):
        wide.exact_log_Z()
    from boltzmann_machines.class_dbm import ClassificationDBM
    for name in ('exact_log_Z', 'exact_log_proba'):
        with pytest.raises(NotImplementedError, match='ClassificationDBM'):
            getattr(ClassificationDBM, name)(None)
    clean(sim)
