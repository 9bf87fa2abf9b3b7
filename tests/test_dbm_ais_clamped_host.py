"""AIS estimates of log p*(v) of binary DBMs with v clamped (DESIGN.md §5.4g), checked without a GPU.

* The statement (tests/dbm_ais_clamped_oracle.py): log p*_beta(x; v) summed over the even layers against brute force over
  every hidden unit at beta = 0, 0.37 and 1 for L = 2, 3, 4; the float64 ladder against enumeration on tiny models, within its
  own standard error; L = 1 is the closed form.
* The tensor-core engine's host code on the stand-in runtime (tests/hostsim, build_dbm_ais_clamped.sh) against the bf16
  emulation, run by run: L = 2, 3, 4, k = 1 and 3, short and 420-temperature ladders, ragged widths, binary and grey rows,
  sample_h_states false somewhere (still sampled), tempered and centered models; row slices through row0 against one call,
  a row's runs unchanged by other rows, slices of the chain budget; L = 1; every refusal before any launch; the ladder's
  programs pass the dataflow check; the Python class, its refusals and a model left bit-identical.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dbm_ais_clamped_oracle as Q  # noqa: E402
import dbm_ais_depth_oracle as A  # noqa: E402
from test_dbm_ais_depth_host import _stack, clean, engine, make_cfg, params, same_runs  # noqa: E402

ROOT = os.path.dirname(HERE)
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_ais_clamped.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')

SHAPES = {2: (6, (5, 4)), 3: (5, (4, 4, 3)), 4: (4, (3, 4, 3, 3))}
RAGGED = {2: (37, (21, 11)), 3: (29, (19, 9, 13)), 4: (13, (21, 6, 9, 7))}


def rows_of(V, n, grey=False, seed=0):
    rng = np.random.RandomState(seed)
    if grey:
        return rng.rand(n, V).astype(np.float32)
    return (rng.rand(n, V) < 0.4).astype(np.float32)


# ---- the statement ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('beta', [0.0, 0.37, 1.0])
@pytest.mark.parametrize('L', [2, 3, 4])
def test_clamped_log_p_star_matches_brute_force(L, beta):
    V, Hs = {2: (3, (3, 3)), 3: (3, (2, 3, 2)), 4: (2, (2, 2, 3, 2))}[L]
    p = params(V, Hs, scale=0.9, seed=L)
    X = rows_of(V, 3, seed=L)
    w = A.widths(p)
    even = list(range(2, L + 1, 2))
    grids = np.meshgrid(*[np.arange(2 ** w[j]) for j in even], indexing='ij')
    x = {j: A.states(w[j])[g.ravel()] for j, g in zip(even, grids)}
    n = len(x[2])
    for v in X:
        summed = float(np.logaddexp.reduce(Q.log_p_star(p, np.repeat(v[None, :], n, axis=0), x, beta)))
        if beta == 1.0:
            assert abs(summed - A.brute_log_p_v(p, v[None, :])[0]) < 1e-10
        elif beta == 0.0:
            assert abs(summed - sum(Hs) * np.log(2.)) < 1e-10
        else:                                     # the model with every parameter scaled by beta
            scaled = {k: beta * np.asarray(val, np.float64) for k, val in p.items()}
            assert abs(summed - A.brute_log_p_v(scaled, v[None, :])[0]) < 1e-10


@pytest.mark.parametrize('L', [2, 3, 4])
def test_float64_ladder_estimates_the_enumerated_log_p_v(L):
    """each row's estimate within 4 of its own standard errors (+ 0.01 nats) of the enumerated log p*(v)"""
    V, Hs = SHAPES[L]
    p = params(V, Hs, scale=0.5)
    X = np.concatenate([rows_of(V, 3, seed=1), rows_of(V, 2, grey=True, seed=2)])
    runs = Q.ais(p, X, 200, 100, 1, 3)
    est = Q.log_mean_rows(runs)
    exact = Q.enumerated_log_p_v(p, X)
    np.testing.assert_allclose(exact, A.brute_log_p_v(p, X), atol=1e-10)
    w = np.exp(runs - runs.max(axis=1, keepdims=True))
    se = w.std(axis=1) / w.mean(axis=1) / np.sqrt(runs.shape[1])
    assert np.all(np.abs(est - exact) < 4 * se + 0.01), (est - exact, se)


def test_one_layer_is_the_closed_form():
    p = params(7, (5,), scale=0.6)
    X = rows_of(7, 4)
    np.testing.assert_allclose(Q.ais(p, X, 3, 10, 1, 1), np.repeat(A.brute_log_p_v(p, X)[:, None], 3, axis=1), atol=1e-10)


# ---- the engine on the stand-in runtime -------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_ais_clamped.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(SIM)
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    lib.fakecuda_hazard_launches.restype = C.c_long
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


@pytest.mark.parametrize('grey', [False, True], ids=['binary', 'grey'])
@pytest.mark.parametrize('L', [2, 3, 4])
@pytest.mark.parametrize('k,n_betas', [(1, 60), (3, 25), (1, 420)], ids=['k1', 'k3', 'fine'])
def test_engine_equals_the_emulation(sim, L, k, n_betas, grey):
    V, Hs = RAGGED[L]
    p = params(V, Hs, scale=0.3, seed=L)
    X = rows_of(V, 3, grey=grey, seed=L)
    e = engine(make_cfg(Hs, V), p)
    got = e.ais_clamped(X, 5, n_betas, k, 77, row0=2)
    assert got.shape == (3, 5)
    same_runs(got.ravel(), Q.ais(p, X, 5, n_betas, k, 77, row0=2, bf16=True).ravel(), (L, k, n_betas, grey))
    e.close()
    clean(sim)


def test_unsampled_layers_are_still_sampled(sim):
    """the ladder draws every layer it updates whatever sample_v / sample_h say: the same runs as a fully sampled model"""
    V, Hs = RAGGED[3]
    p = params(V, Hs, scale=0.3, seed=9)
    X = rows_of(V, 3, seed=9)
    e = engine(make_cfg(Hs, V, sample_v=False, sample_h=[False, True, False]), p)
    got = e.ais_clamped(X, 4, 40, 2, 5)
    same_runs(got.ravel(), Q.ais(p, X, 4, 40, 2, 5, bf16=True).ravel(), 'unsampled')
    e.close()
    e = engine(make_cfg(Hs, V), p)
    np.testing.assert_array_equal(e.ais_clamped(X, 4, 40, 2, 5), got)
    e.close()
    clean(sim)


@pytest.mark.parametrize('what', ['tempered', 'centered'])
def test_tempered_and_centered_models_read_the_stored_parameters(sim, what):
    V, Hs = RAGGED[2]
    p = params(V, Hs, scale=0.3, seed=21)
    kw = dict(pt_betas=[1.0, 0.6, 0.3]) if what == 'tempered' else dict(centering=True, offset_rate=0.05)
    e = engine(make_cfg(Hs, V, **kw), p)
    e.init_particles(3)
    X = rows_of(V, 3, seed=21)
    got = e.ais_clamped(X, 4, 60, 1, 8)
    same_runs(got.ravel(), Q.ais(p, X, 4, 60, 1, 8, bf16=True).ravel(), what)
    e.close()
    clean(sim)


def test_row_slices_and_chain_slices_match_one_call(sim, monkeypatch):
    V, Hs = RAGGED[3]
    p = params(V, Hs, scale=0.3, seed=4)
    X = rows_of(V, 7, seed=4)
    e = engine(make_cfg(Hs, V), p)
    whole = e.ais_clamped(X, 3, 30, 1, 6)
    parts = np.concatenate([e.ais_clamped(X[lo:hi], 3, 30, 1, 6, row0=lo) for lo, hi in ((0, 2), (2, 3), (3, 7))])
    np.testing.assert_array_equal(parts, whole)
    # a row's runs depend on its index only: the same row with other rows around it
    np.testing.assert_array_equal(e.ais_clamped(X[4:5], 3, 30, 1, 6, row0=4), whole[4:5])
    other = X.copy()
    other[[0, 1, 2, 3, 5, 6]] = 1. - other[[0, 1, 2, 3, 5, 6]]
    np.testing.assert_array_equal(e.ais_clamped(other, 3, 30, 1, 6)[4], whole[4])
    e.close()
    clean(sim)


def test_chain_budget_slices_are_invisible(sim):
    """more chains than one ladder runs (DbmTC::AIS_CLAMPED_CHAINS = 32768): the call cuts them into slices, and the runs
    are those of the rows computed one at a time"""
    V, Hs = 5, (4, 3)
    p = params(V, Hs, scale=0.4, seed=5)
    X = rows_of(V, 3, seed=5)
    e = engine(make_cfg(Hs, V), p)
    n_runs = 12000                                 # 36 000 chains: two slices, the cut inside row 2
    got = e.ais_clamped(X, n_runs, 2, 1, 3)
    np.testing.assert_array_equal(got[2], e.ais_clamped(X[2:3], n_runs, 2, 1, 3, row0=2)[0])
    same_runs(got[2, -200:], Q.ais(p, X[2:3], n_runs, 2, 1, 3, row0=2, bf16=True)[0, -200:], 'budget')
    e.close()
    clean(sim)


def test_one_layer_returns_log_proba(sim):
    V, Hs = 9, (7,)
    p = params(V, Hs, scale=0.5, seed=6)
    X = np.concatenate([rows_of(V, 3, seed=6), rows_of(V, 2, grey=True, seed=7)])
    e = engine(make_cfg(Hs, V, B=4), p)
    got = e.ais_clamped(X, 3, 10, 1, 1)
    assert np.all(got == got[:, :1])
    np.testing.assert_allclose(got[:, 0], e.log_proba(X[:4]).tolist() + e.log_proba(X[4:]).tolist(), rtol=0, atol=0)
    np.testing.assert_allclose(got, Q.ais(p, X, 3, 10, 1, 1, bf16=True), rtol=0, atol=1e-4)
    e.close()
    clean(sim)


BM_EINVAL, BM_EUNSUPPORTED = -1, -5


def rc_of(e, X, rows=None, row0=0, n_runs=2, n_betas=10, k=1, out=True):
    lw = np.empty(max(1, (rows if rows is not None else len(X)) * max(n_runs, 1)))
    return e._lib.bm_dbm_ais_clamped(e.handle, None if X is None else X.ctypes.data, len(X) if rows is None else rows, row0,
                                     n_runs, n_betas, k, 1, lw.ctypes.data if out else None)


def test_refusals_launch_nothing(sim):
    from boltzmann_machines import _native
    ctx = _native.Context.default()
    V, Hs = 6, (5, 4)
    X = rows_of(V, 3)
    cases = [
        (make_cfg(Hs, V, v_kind='gaussian', sigma=np.ones(V)), 'binary'),
        (make_cfg(Hs, V, h_kinds=['bernoulli', 'multinomial'], h_n_samples=[100., 3.]), 'binary'),
        (make_cfg(Hs, V, compute='fp32'), 'CUDA-core engine'),
        (make_cfg(Hs, V, dtype='float64'), 'CUDA-core engine'),
        (make_cfg(Hs, V, n_classes=3), 'classification DBM'),
    ]
    for c, msg in cases:
        e = _native.CudaDBM(c)
        e.set_params({n: v.astype(e.dt) for n, v in params(V, Hs).items()})
        n0 = ctx.launch_count()
        with pytest.raises(NotImplementedError, match=msg):
            e.ais_clamped(X, 2, 10, 1, 1)
        assert rc_of(e, X) == BM_EUNSUPPORTED
        assert ctx.launch_count() == n0, c
        e.close()
    e = engine(make_cfg(Hs, V), params(V, Hs))
    n0 = ctx.launch_count()
    bad = X.copy()
    bad[1, 2] = np.nan
    for args, msg in (((bad, 2, 10, 1, 1), 'non-finite'), ((X, 0, 10, 1, 1), 'bad AIS arguments'),
                      ((X, 2, 1, 1, 1), 'bad AIS arguments'), ((X, 2, 10, 0, 1), 'bad AIS arguments'),
                      ((X[:0], 2, 10, 1, 1), 'bad AIS arguments')):
        with pytest.raises(RuntimeError, match=msg):
            e.ais_clamped(*args)
    with pytest.raises(RuntimeError, match='2\\^32'):
        e.ais_clamped(X, 2, 10, 1, 1, row0=2 ** 31 - 1)
    assert rc_of(e, X, row0=(2 ** 32) // 2 - 3) == BM_EINVAL            # (row0 + 3) * 2 == 2^32
    assert rc_of(e, None, rows=3) == BM_EINVAL
    assert rc_of(e, X, out=False) == BM_EINVAL
    assert rc_of(e, X, rows=0) == BM_EINVAL
    assert ctx.launch_count() == n0
    with pytest.raises(ValueError):
        e.ais_clamped(X[:, :5], 2, 10, 1, 1)
    e.close()
    clean(sim)


@pytest.mark.parametrize('L', [2, 3, 4])
def test_ladder_programs_pass_the_dataflow_check(sim, L):
    """every element an op of a clamped ladder launch reads or writes is ordered by a declared dependency path, 256 chains at a
    time; with one dependency of a summed-out op dropped, the check reports the hazard"""
    V, Hs = SHAPES[L]
    p = params(V, Hs, seed=40 + L)
    X = rows_of(V, 6, seed=L)
    sim.fakecuda_set_hazards(2)
    try:
        n0 = sim.fakecuda_hazard_launches()
        e = engine(make_cfg(Hs, V), p)
        e.ais_clamped(X, 100, 40, 2, 3)                      # 600 chains: three 256-chain blocks, several launches per ladder
        assert sim.fakecuda_hazard_launches() - n0 >= 2
        clean(sim)
        sim.fakecuda_drop_dependency(L, 0)                   # the second sweep's h_1 op stops waiting for the first sweep's h_2
        e.ais_clamped(X, 100, 40, 2, 3)
        assert sim.fakecuda_violation().decode() != ''
        e.close()
    finally:
        sim.fakecuda_drop_dependency(-1, -1)
        sim.fakecuda_set_hazards(0)
        sim.fakecuda_reset()


# ---- the Python class ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sizes', [(7, 5), (6, 5, 4), (6, 5, 4, 3)], ids=['L1', 'L2', 'L3'])
def test_python_ais_log_proba(sim, tmp_path, sizes):
    m, X = _stack(tmp_path, list(sizes))
    prm = {n: v for n, v in m.get_tf_params(scope='weights').items()}
    est, runs = m.ais_log_proba(X[:6], 1.5, n_betas=60, n_runs=16, n_gibbs_steps=1, return_runs=True)
    assert est.shape == (6,) and runs.shape == (6, 16) and est.dtype == np.float64
    np.testing.assert_allclose(est, Q.log_mean_rows(runs) - 1.5, rtol=0, atol=1e-12)
    exact = A.brute_log_p_v(prm, X[:6])
    assert np.all(np.abs(Q.log_mean_rows(runs) - exact) < 0.3), (Q.log_mean_rows(runs), exact)
    np.testing.assert_array_equal(m.ais_log_proba(X[:6], 0.0, n_betas=10, n_runs=2).shape, (6,))
    clean(sim)


def test_python_rows_are_sliced_to_the_chain_budget(sim, tmp_path, monkeypatch):
    from boltzmann_machines import DBM
    m, X = _stack(tmp_path, [6, 5, 4])
    monkeypatch.setattr(DBM, '_AIS_CLAMPED_CHAINS', 10)             # 4 runs: two rows per engine call
    calls = []
    orig = m._engine.ais_clamped

    def spy(Xs, n_runs, n_betas, k, seed, row0=0):
        calls.append((len(Xs), row0, seed))
        return orig(Xs, n_runs, n_betas, k, seed, row0=row0)
    monkeypatch.setattr(m._engine, 'ais_clamped', spy)
    _, sliced = m.ais_log_proba(X[:5], 0.0, n_betas=10, n_runs=4, n_gibbs_steps=1, return_runs=True)
    seed = calls[0][2]
    assert calls == [(2, 0, seed), (2, 2, seed), (1, 4, seed)]
    np.testing.assert_array_equal(sliced, orig(X[:5], 4, 10, 1, seed))
    clean(sim)


def test_python_validation_refusals_and_an_untouched_model(sim, tmp_path):
    m, X = _stack(tmp_path, [6, 5, 4])
    for bad in (X[:, :5], X[0], np.where(np.arange(6) == 2, np.nan, X[:3])):
        with pytest.raises(ValueError):
            m.ais_log_proba(bad, 0.0, n_betas=10, n_runs=2)
    for kw in (dict(n_runs=0), dict(n_betas=1), dict(n_gibbs_steps=0)):
        with pytest.raises(ValueError):
            m.ais_log_proba(X[:2], 0.0, **dict(dict(n_betas=10, n_runs=2), **kw))
    m64, X64 = _stack(tmp_path / 'f64', [6, 5, 4], dtype='float64')
    with pytest.raises(NotImplementedError, match='float32'):
        m64.ais_log_proba(X64[:2], 0.0, n_betas=10, n_runs=2)
    # the model is bit-identical afterwards: every variable and particle, and the next train_step is that of a twin that ran
    # no query
    twin, _ = _stack(tmp_path / 'twin', [6, 5, 4])
    before = m._engine.get_params()
    m.ais_log_proba(X[:5], 0.0, n_betas=20, n_runs=3, n_gibbs_steps=2)
    after = m._engine.get_params()
    for n, v in before.items():
        np.testing.assert_array_equal(after[n], v, err_msg='ais_log_proba moved ' + n)
    for mm in (m, twin):
        mm._engine.train_step(X[:8], 0.01, 0.5, 1, 5, 3)
    a, b = m._engine.get_params(), twin._engine.get_params()
    for n in a:
        np.testing.assert_array_equal(a[n], b[n], err_msg='train_step after ais_log_proba: ' + n)
    clean(sim)


def test_classification_dbm_refuses(sim, tmp_path):
    from boltzmann_machines import ClassificationDBM
    with pytest.raises(NotImplementedError, match='ClassificationDBM: ais_log_proba'):
        ClassificationDBM.ais_log_proba(object(), np.zeros((2, 6)), 0.0)
