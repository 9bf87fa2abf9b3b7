"""AIS log Z of binary DBMs from a base-rate model (DESIGN.md §5.4d), checked without a GPU.

* The statement (tests/dbm_ais_base_oracle.py): the marginalised log p*_beta on the path from the base against brute force over
  every unit, at beta = 0 (log Z_A), 0.37 and 1; the float64 ladder against enumeration with a base on every layer; on a model
  with data-like visible biases the data base gives a smaller spread of the log-weights and a smaller error than the uniform one.
* The tensor-core engine's host code on the stand-in runtime (tests/hostsim, build_dbm_ais_base.sh) against the bf16 emulation,
  run by run: L = 1, 2, 3, k = 1 and 3, coarse and fine (>= 400 temperatures) ladders, ragged widths, bases on v only and on
  every layer; slices; the zero and the all-null base against the uniform ladder; every refusal before any launch; the Python
  class.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dbm_ais_base_oracle as B  # noqa: E402
import dbm_ais_depth_oracle as A  # noqa: E402
from test_dbm_ais_depth_host import _stack, clean, engine, log_mean, make_cfg, params, same_runs  # noqa: E402

ROOT = os.path.dirname(HERE)
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_ais_base.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')

SHAPES = {1: (7, (5,)), 2: (6, (5, 4)), 3: (6, (5, 4, 3))}
RAGGED = {1: (37, (21,)), 2: (29, (19, 11)), 3: (13, (21, 9, 6))}


def bases(prm, which, seed=0):
    """a base on v only or on every layer (None elsewhere)"""
    rng = np.random.RandomState(seed)
    w = A.widths(prm)
    out = [None] * len(w)
    for j in (range(len(w)) if which == 'all' else [0]):
        out[j] = (rng.randn(w[j]) - (1.5 if j == 0 else 0.5)).astype(np.float32)
    return out


# ---- the statement ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('beta', [0.0, 0.37, 1.0])
@pytest.mark.parametrize('L', [1, 2, 3])
def test_marginalised_log_p_star_on_the_path_matches_brute_force(L, beta):
    V, Hs = {1: (4, (3,)), 2: (3, (3, 2)), 3: (3, (2, 3, 2))}[L]
    p = params(V, Hs, scale=0.9, seed=L)
    base = bases(p, 'all', seed=L)
    w = A.widths(p)
    odd = list(range(1, L + 1, 2))
    grids = np.meshgrid(*[np.arange(2 ** w[j]) for j in odd], indexing='ij')
    x = {j: A.states(w[j])[g.ravel()] for j, g in zip(odd, grids)}
    summed = float(np.logaddexp.reduce(B.log_p_star(p, x, beta, base)))
    assert abs(summed - A.brute_log_Z(B.path_model(p, beta, base))) < 1e-10
    if beta == 0.0:
        assert abs(summed - B.log_Z_A(p, base)) < 1e-10


@pytest.mark.parametrize('L', [1, 2, 3])
def test_float64_ladder_from_a_base_estimates_the_enumerated_log_Z(L):
    V, Hs = SHAPES[L]
    p = params(V, Hs, scale=0.5)
    est = log_mean(B.ais(p, 256, 200, 1, 3, base=bases(p, 'all', seed=L)))
    assert abs(est - A.exact_log_Z(p)) < 0.05, (est, A.exact_log_Z(p))


def test_zero_base_statement_is_the_uniform_ladder():
    V, Hs = SHAPES[3]
    p = params(V, Hs, scale=0.6)
    zero = [np.zeros(n, np.float32) for n in A.widths(p)]
    _, lw0 = B.ais(p, 16, 30, 2, 4, base=zero, return_logw=True)
    got = A.ais(p, 16, 30, 2, 4) - sum(A.widths(p)) * A.LOG2_F32
    np.testing.assert_allclose(lw0, got, rtol=0, atol=1e-10)


def data_like_model():
    """an enumerable 12-6-4 DBM whose visible units are mostly off (biases around -3), as a model of MNIST-like data is"""
    rng = np.random.RandomState(11)
    V, Hs = 12, (6, 4)
    p = params(V, Hs, scale=0.4, seed=11)
    p['vb'] = (-3.0 + 0.8 * rng.randn(V)).astype(np.float32)
    return p


def test_data_base_narrows_the_log_weights_on_a_data_like_model():
    """measured in float64 with fixed seeds: the spread of the log-weights and the error of log Z-hat, uniform against the
    base sigmoid(a_v) = the model's own visible marginals, at a short ladder (pinned values)"""
    p = data_like_model()
    exact = A.exact_log_Z(p)
    X = (np.random.RandomState(3).rand(4000, 12) < 1. / (1. + np.exp(-p['vb'].astype(np.float64)))).astype(np.float32)
    base = [B.data_base(X), None, None]
    uni = B.ais(p, 400, 20, 1, 9)
    dat = B.ais(p, 400, 20, 1, 9, base=base)
    sd_u, sd_d = float(np.std(uni)), float(np.std(dat))
    err_u, err_d = abs(log_mean(uni) - exact), abs(log_mean(dat) - exact)
    assert sd_d < sd_u and err_d < err_u, (sd_u, sd_d, err_u, err_d)
    np.testing.assert_allclose([sd_u, sd_d, err_u, err_d], PINNED_SPREAD, rtol=1e-6, atol=1e-9)


# (std of log Z-hat per run, uniform / data base; |log mean - exact|, uniform / data base), 20 temperatures, 400 runs
PINNED_SPREAD = [0.14402376861786975, 0.1286358820306841, 0.026638132280966786, 0.019967110430945567]


# ---- the engine on the stand-in runtime -------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_ais_base.sh')], stdout=subprocess.DEVNULL)
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


@pytest.mark.parametrize('which', ['v', 'all'])
@pytest.mark.parametrize('L', [1, 2, 3])
@pytest.mark.parametrize('k,n_betas', [(1, 60), (3, 25), (1, 420)], ids=['k1', 'k3', 'fine'])
def test_engine_equals_the_emulation(sim, L, k, n_betas, which):
    V, Hs = RAGGED[L]
    p = params(V, Hs, scale=0.3, seed=L)
    base = bases(p, which, seed=10 + L)
    e = engine(make_cfg(Hs, V), p)
    got = e.ais(12, n_betas, k, 77, base=base)
    same_runs(got, B.ais(p, 12, n_betas, k, 77, base=base, bf16=True), (L, k, n_betas, which))
    e.close()
    clean(sim)


def test_slices_concatenate_to_the_ladder(sim):
    V, Hs = RAGGED[2]
    p = params(V, Hs, scale=0.3, seed=4)
    base = bases(p, 'all', seed=4)
    e = engine(make_cfg(Hs, V), p)
    whole = e.ais(21, 40, 1, 6, base=base)
    parts = np.concatenate([e.ais(n, 40, 1, 6, first_run=lo, base=base) for lo, n in ((0, 8), (8, 5), (13, 8))])
    np.testing.assert_array_equal(parts, whole)
    e.close()
    clean(sim)


@pytest.mark.parametrize('L', [1, 2, 3])
def test_zero_and_null_bases(sim, L):
    """a zero base runs the layered ladder with today's draws (at L = 2 against ais_local's program); an all-null base is
    today's call"""
    V, Hs = RAGGED[L]
    p = params(V, Hs, scale=0.3, seed=50 + L)
    e = engine(make_cfg(Hs, V), p)
    today = e.ais(12, 40, 2, 3)
    zero = [np.zeros(n, np.float32) for n in A.widths(p)]
    got = e.ais(12, 40, 2, 3, base=zero)
    np.testing.assert_allclose(got - B.log_Z_A(p, zero), today - sum(A.widths(p)) * A.LOG2_F32, rtol=0, atol=1e-9)
    np.testing.assert_array_equal(e.ais(12, 40, 2, 3, base=[None] * (L + 1)), today)
    e.close()
    clean(sim)


BM_EINVAL, BM_EUNSUPPORTED = -1, -5


def rc_of(e, base):
    """the return code of bm_dbm_ais_base for 4 runs of a 10-temperature ladder"""
    keep = [None if a is None else np.ascontiguousarray(a, np.float32) for a in base]
    bp = (C.c_void_p * len(keep))(*[None if a is None else a.ctypes.data for a in keep])
    out = np.empty(4)
    return e._lib.bm_dbm_ais_base(e.handle, 4, 10, 1, 1, bp, out.ctypes.data)


def test_refusals_launch_nothing(sim):
    from boltzmann_machines import _native
    ctx = _native.Context.default()
    V, Hs = 6, (5, 4)
    p = params(V, Hs)
    base = [np.zeros(V, np.float32), None, None]
    cases = [
        (make_cfg(Hs, V, v_kind='gaussian', sigma=np.ones(V)), 'binary'),
        (make_cfg(Hs, V, h_kinds=['bernoulli', 'multinomial'], h_n_samples=[100., 3.]), 'binary'),
        (make_cfg(Hs, V, sample_h=[False, True]), 'sampled states'),
        (make_cfg(Hs, V, compute='fp32'), 'CUDA-core engine'),
        (make_cfg(Hs, V, dtype='float64'), 'CUDA-core engine'),
        (make_cfg(Hs, V, n_classes=3), 'no label layer'),
    ]
    for c, msg in cases:
        e = _native.CudaDBM(c)
        q = params(V, Hs)
        e.set_params({n: v.astype(e.dt) for n, v in q.items()})
        n0 = ctx.launch_count()
        for first_run in (None, 3):
            with pytest.raises(RuntimeError, match=msg):
                e.ais(4, 10, 1, 1, first_run=first_run, base=base)
        assert rc_of(e, base) == BM_EUNSUPPORTED
        assert ctx.launch_count() == n0, c
        e.close()
    e = engine(make_cfg(Hs, V), p)
    n0 = ctx.launch_count()
    bad = [np.zeros(V, np.float32), None, np.array([0., np.nan, 0., 0.], np.float32)]
    with pytest.raises(RuntimeError, match='non-finite'):
        e.ais(4, 10, 1, 1, base=bad)
    assert rc_of(e, bad) == BM_EINVAL
    for args in ((0, 10, 1), (4, 1, 1), (4, 10, 0)):
        with pytest.raises(RuntimeError, match='bad AIS arguments'):
            e.ais(*args, 1, base=base)
    with pytest.raises(ValueError):
        e.ais(4, 10, 1, 1, base=[None, None])
    with pytest.raises(ValueError):
        e.ais(4, 10, 1, 1, base=[np.zeros(V + 1), None, None])
    assert ctx.launch_count() == n0
    e.close()
    clean(sim)


# ---- the Python class ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sizes', [(7, 5), (6, 5, 4), (6, 5, 4, 3)], ids=['L1', 'L2', 'L3'])
def test_python_log_Z_from_the_data(sim, tmp_path, sizes):
    m, X = _stack(tmp_path, list(sizes))
    log_mean_, (lo, hi), values = m.log_Z(n_betas=60, n_runs=32, n_gibbs_steps=1, base_rate=X)
    assert values.shape == (32,) and np.all(np.isfinite(values)) and lo <= log_mean_ <= hi
    prm = {n: v for n, v in m.get_tf_params(scope='weights').items()}
    assert abs(log_mean_ - A.exact_log_Z(prm)) < 0.2
    base = [B.data_base(X)] + [None] * (len(sizes) - 1)
    np.testing.assert_allclose(m._engine.ais(4, 10, 1, 5, base=base), B.ais(prm, 4, 10, 1, 5, base=base, bf16=True), atol=1e-4)
    clean(sim)


def test_python_base_rate_validation_and_refusals(sim, tmp_path):
    m, X = _stack(tmp_path, [6, 5, 4])
    for bad in (X[:, :5], X * 2., [None, None], [np.zeros(6), np.zeros(4), None], [np.full(6, np.inf), None, None]):
        with pytest.raises(ValueError):
            m.log_Z(n_betas=10, n_runs=4, base_rate=bad)
    values = m.log_Z(n_betas=10, n_runs=4, base_rate=[np.zeros(6), None, np.zeros(4)])[2]
    assert values.shape == (4,)
    m2, X2 = _stack(tmp_path / 'u', [6, 5, 4], sample_h_states=[False, True])
    with pytest.raises(NotImplementedError, match='sampled states'):
        m2.log_Z(n_betas=10, n_runs=4, base_rate=X2)
    m64, X64 = _stack(tmp_path / 'f64', [6, 5, 4], dtype='float64')
    with pytest.raises(NotImplementedError, match='float32'):
        m64.log_Z(n_betas=10, n_runs=4, base_rate=X64)
    clean(sim)
