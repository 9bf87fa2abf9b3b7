"""AIS log Z and the variational bound of binary DBMs with one, three or more hidden layers (DESIGN.md §5.4c), checked without
a GPU.

* The statement (tests/dbm_ais_depth_oracle.py): the marginalised log p* against brute force over every unit of tiny models at
  L = 1, 3 and 4; the float64 ladder's estimate against log Z from enumerating the state layers; at L = 2 the statement equals
  the reference ladder of oracle/dbm.py run for run, which pins the site rule.
* The tensor-core engine's host code on the stand-in runtime (tests/hostsim, build_dbm_ais_depth.sh) against the bf16
  emulation, run by run: L = 1, 3, 4, k = 1 and 3, coarse and fine (>= 400 temperatures) ladders, unsampled summed-out layers,
  tempered and centered models; slices and chunks of a ladder concatenate to the whole ladder; the bound against its
  emulation; every refusal before any launch; the ladders' programs pass the dataflow check; the Python class.
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
from oracle.dbm import OracleDBM  # noqa: E402

ROOT = os.path.dirname(HERE)
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_ais_depth.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
sfx = A.sfx


def make_cfg(Hs, V, B=8, dtype='float32', compute='bf16', **kw):
    L = len(Hs)
    c = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype=dtype, compute=compute,
             n_particles=8, batch_size=B, max_mf_updates=6, mf_tol=1e-6, l2=1e-4, max_norm=3.0, sample_v=True,
             sample_h=[True] * L, sparsity_target=[0.2] * L, sparsity_cost=[0.01] * L, sparsity_damping=0.9)
    c.update(kw)
    return c


def params(V, Hs, scale=0.6, bias=0.5, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [V] + list(Hs)
    d = {'vb': (bias * rng.randn(V)).astype(np.float32)}
    for i in range(len(Hs)):
        d['W' + sfx(i)] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + sfx(i)] = (bias * rng.randn(sizes[i + 1])).astype(np.float32)
    return d


def log_mean(v):
    return float(np.logaddexp.reduce(v) - np.log(len(v)))


SHAPES = {1: (7, (5,)), 3: (6, (5, 4, 3)), 4: (5, (4, 4, 3, 3))}


# ---- the statement ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('V,Hs', [(4, (3,)), (3, (3, 2, 2)), (3, (2, 3, 2, 2))])
def test_marginalised_log_p_star_matches_brute_force(V, Hs):
    """summing the state layers' exp log p*_1 is log Z over every unit; and at L = 1 log p*_1 over h_1 is log p*(v) summed"""
    p = params(V, Hs, scale=0.9, seed=len(Hs))
    assert abs(A.exact_log_Z(p) - A.brute_log_Z(p)) < 1e-10
    w = A.widths(p)
    x = {j: A.states(w[j])[np.random.RandomState(j).randint(0, 2 ** w[j], 5)] for j in range(1, len(Hs) + 1, 2)}
    if len(Hs) == 1:
        # p*(h_1) = exp(c.h) prod_n (1 + exp(b_n + W_n h)): the brute force over v for each h
        Ws, bs = A.unit_layers(p)
        vs = A.states(V)
        brute = [np.logaddexp.reduce(vs @ bs[0] + h @ bs[1] + ((vs @ Ws[0]) * h).sum(axis=1)) for h in x[1]]
        np.testing.assert_allclose(A.log_p_star(p, x), brute, atol=1e-10)


@pytest.mark.parametrize('L', [1, 3, 4])
def test_float64_ladder_estimates_the_enumerated_log_Z(L):
    V, Hs = SHAPES[L]
    p = params(V, Hs, scale=0.5)
    est = log_mean(A.ais(p, 256, 200, 1, 3))
    assert abs(est - A.exact_log_Z(p)) < 0.05, (est, A.exact_log_Z(p))


@pytest.mark.parametrize('k', [1, 3])
def test_the_rule_at_two_layers_is_the_reference_ladder(k):
    """float64 statement with float64 temperatures against oracle/dbm.py's float64 ladder: the same draws at the same sites,
    run for run to round-off (any other site, Gibbs index or order of the layers changes runs by whole increments)"""
    V, Hs = 7, (5, 4)
    p = params(V, Hs, scale=0.5)
    o = OracleDBM(make_cfg(Hs, V, dtype='float64', compute='fp32'))
    o.set_params({n: v.astype(np.float64) for n, v in p.items()})
    got = A.ais(p, 24, 50, k, 5, first_run=7, beta_dtype=np.float64)
    np.testing.assert_allclose(got, o.ais(24, 50, k, 5, first_run=7), rtol=0, atol=1e-10)


def test_bound_of_one_layer_is_exact_and_of_deeper_models_below():
    for V, Hs in ((7, (5,)), (5, (4, 3, 3))):
        p = params(V, Hs, scale=0.7)
        X = (np.random.RandomState(1).rand(6, V) < 0.5).astype(np.float64)
        b, _ = A.bound(make_cfg(Hs, V, max_mf_updates=50, mf_tol=1e-12), p, X)
        exact = A.brute_log_p_v(p, X)
        if len(Hs) == 1:
            np.testing.assert_allclose(b, exact, atol=1e-9)
        else:
            assert np.all(b <= exact + 1e-9) and np.all(b > exact - 3.0), (b, exact)


# ---- the engine on the stand-in runtime -------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_ais_depth.sh')], stdout=subprocess.DEVNULL)
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


def clean(sim):
    v, sk = sim.fakecuda_violation().decode(), sim.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


def engine(c, d):
    from boltzmann_machines import _native
    e = _native.CudaDBM(c)
    assert e.compute == 'bf16'
    e.set_params(d)
    return e


def same_runs(got, want, what):
    """the engine and the emulation run the same chains: every run to float32 round-off of its increments, but for a draw
    whose uniform lies within an fp32 rounding of its probability (sums in another order), which forks one run"""
    close = np.abs(got - want) < 1e-5
    assert np.mean(close) >= 0.95, (what, np.abs(got - want))


@pytest.mark.parametrize('L', [1, 3, 4])
@pytest.mark.parametrize('k,n_betas', [(1, 60), (3, 25), (1, 420)], ids=['k1', 'k3', 'fine'])
def test_engine_equals_the_emulation(sim, L, k, n_betas):
    V, Hs = SHAPES[L]
    p = params(V, Hs, scale=0.8, seed=L)
    e = engine(make_cfg(Hs, V), p)
    got = e.ais(20, n_betas, k, 77)
    same_runs(got, A.ais(p, 20, n_betas, k, 77, bf16=True), (L, k, n_betas))
    e.close()
    clean(sim)


@pytest.mark.parametrize('L', [3, 4])
def test_unsampled_summed_out_layers(sim, L):
    """v and h_2 take their means (bf16) where they are not sampled: the closed-form epilogue without a draw"""
    V, Hs = SHAPES[L]
    p = params(V, Hs, seed=10 + L)
    sh = [True] * L
    sh[1] = False
    e = engine(make_cfg(Hs, V, sample_v=False, sample_h=sh), p)
    got = e.ais(16, 60, 2, 5)
    same_runs(got, A.ais(p, 16, 60, 2, 5, bf16=True, sample_v=False, sample_h=sh), 'unsampled')
    e.close()
    clean(sim)


@pytest.mark.parametrize('what', ['tempered', 'centered'])
def test_tempered_and_centered_models_read_the_stored_parameters(sim, what):
    V, Hs = SHAPES[3]
    p = params(V, Hs, seed=21)
    kw = dict(pt_betas=[1.0, 0.6, 0.3]) if what == 'tempered' else dict(centering=True, offset_rate=0.05)
    e = engine(make_cfg(Hs, V, **kw), p)
    e.init_particles(3)
    got = e.ais(16, 60, 1, 8)
    same_runs(got, A.ais(p, 16, 60, 1, 8, bf16=True), what)
    e.close()
    clean(sim)


def test_slices_and_chunks_concatenate_to_the_ladder(sim):
    V, Hs = SHAPES[3]
    p = params(V, Hs, seed=4)
    e = engine(make_cfg(Hs, V), p)
    whole = e.ais(21, 40, 1, 6)
    parts = np.concatenate([e.ais(n, 40, 1, 6, first_run=lo) for lo, n in ((0, 8), (8, 5), (13, 8))])
    np.testing.assert_array_equal(parts, whole)
    np.testing.assert_array_equal(e.ais(1, 40, 1, 6, first_run=20), whole[20:])
    e.close()
    clean(sim)


@pytest.mark.parametrize('L', [1, 3])
def test_bound_equals_the_emulation(sim, L):
    V, Hs = SHAPES[L]
    p = params(V, Hs, seed=30 + L)
    c = make_cfg(Hs, V)
    e = engine(c, p)
    X = (np.random.RandomState(5).rand(7, V) < 0.5).astype(np.float32)
    got = e.log_proba(X)
    want, mu = A.bound(c, p, X, bf16=True)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-4)
    g = e.get_params(['mu' + sfx(i) for i in range(L)])
    np.testing.assert_allclose(got, A.bound_given_mu(p, X, [g['mu' + sfx(i)][:7] for i in range(L)]), rtol=0, atol=1e-3)
    e.close()
    clean(sim)


def test_refusals_launch_nothing(sim):
    from boltzmann_machines import _native
    ctx = _native.Context.default()
    V, Hs = 6, (5, 4, 3)
    p = params(V, Hs)
    X = np.zeros((4, V), np.float32)
    cases = [
        (make_cfg(Hs, V, v_kind='gaussian', sigma=np.ones(V)), 'binary', 'binary'),
        (make_cfg(Hs, V, h_kinds=['bernoulli', 'multinomial', 'bernoulli'], h_n_samples=[100., 3., 100.]), 'binary', 'binary'),
        (make_cfg(Hs, V, sample_h=[True, True, False]), 'sampled states', None),
        (make_cfg((5,), V, sample_h=[False]), 'sampled states', None),
    ]
    for c, msg_ais, msg_lp in cases:
        q = params(V, c['n_hiddens'])
        e = _native.CudaDBM(c)
        assert e.compute == 'bf16'
        e.set_params(q)
        n0 = ctx.launch_count()
        with pytest.raises(RuntimeError, match=msg_ais):
            e.ais(4, 10, 1, 1)
        with pytest.raises(RuntimeError, match=msg_ais):
            e.ais(4, 10, 1, 1, first_run=3)
        if msg_lp:
            with pytest.raises(RuntimeError, match=msg_lp):
                e.log_proba(X)
        assert ctx.launch_count() == n0, c
        e.close()
    e = engine(make_cfg(Hs, V), p)
    n0 = ctx.launch_count()
    for bad in ((0, 10, 1), (4, 1, 1), (4, 10, 0)):
        with pytest.raises(RuntimeError, match='bad AIS arguments'):
            e.ais(*bad, 1)
    assert ctx.launch_count() == n0
    e.close()
    # the CUDA-core engine keeps its two-layer refusals, whatever the dtype
    for c in (make_cfg(Hs, V, compute='fp32'), make_cfg(Hs, V, dtype='float64'), make_cfg((5,), V, dtype='float64')):
        e = _native.CudaDBM(c)
        assert e.compute == 'fp32'
        n0 = ctx.launch_count()
        with pytest.raises(RuntimeError, match='2-layer'):
            e.ais(4, 10, 1, 1)
        with pytest.raises(RuntimeError, match='2 hidden'):
            e.log_proba(np.zeros((4, V), e.dt))
        assert ctx.launch_count() == n0
        e.close()
    clean(sim)


@pytest.mark.parametrize('L', [1, 3, 4])
def test_ladder_programs_pass_the_dataflow_check(sim, L):
    """every element an op of a ladder launch reads or writes is ordered by a declared dependency path, 256 runs at a time; with
    one dependency of a summed-out op dropped, the check reports the hazard"""
    V, Hs = SHAPES[L]
    p = params(V, Hs, seed=40 + L)
    sim.fakecuda_set_hazards(2)
    try:
        n0 = sim.fakecuda_hazard_launches()
        e = engine(make_cfg(Hs, V), p)
        e.ais(600, 40, 2, 3)                                 # three 256-run blocks, several launches per ladder
        assert sim.fakecuda_hazard_launches() - n0 >= 2
        clean(sim)
        sim.fakecuda_drop_dependency(L + 1, 0)               # the second sweep's v op stops waiting for the first sweep's h_1
        e.ais(600, 40, 2, 3)
        assert sim.fakecuda_violation().decode() != ''
        e.close()
    finally:
        sim.fakecuda_drop_dependency(-1, -1)
        sim.fakecuda_set_hazards(0)
        sim.fakecuda_reset()


# ---- the Python class ---------------------------------------------------------------------------------------------------------
def _stack(tmp, sizes, dtype='float32', **kw):
    from boltzmann_machines import DBM
    from boltzmann_machines.rbm import BernoulliRBM
    rng = np.random.RandomState(0)
    X = (rng.rand(40, sizes[0]) < 0.4).astype(np.float32)
    rbms, inp = [], X
    for i in range(len(sizes) - 1):
        r = BernoulliRBM(n_visible=sizes[i], n_hidden=sizes[i + 1], max_epoch=1, batch_size=8, random_seed=1 + i, dtype=dtype,
                         model_path=str(tmp / ('r%d' % i)))
        r.fit(inp)
        inp = r.transform(inp)
        rbms.append(r)
    m = DBM(rbms=rbms, n_particles=8, batch_size=8, max_epoch=1, random_seed=4, dtype=dtype, model_path=str(tmp / 'dbm'), **kw)
    m.fit(X)
    return m, X


@pytest.mark.parametrize('sizes', [(7, 5), (6, 5, 4, 3)], ids=['L1', 'L3'])
def test_python_log_Z_and_log_proba(sim, tmp_path, sizes):
    m, X = _stack(tmp_path, list(sizes))
    log_mean_, (lo, hi), values = m.log_Z(n_betas=60, n_runs=32, n_gibbs_steps=1)
    assert values.shape == (32,) and np.all(np.isfinite(values)) and lo <= log_mean_ <= hi
    prm = {n: v for n, v in m.get_tf_params(scope='weights').items()}
    assert abs(log_mean_ - A.exact_log_Z(prm)) < 0.2
    lp = m.log_proba(X[:10], log_mean_)
    assert lp.shape == (10,) and np.all(lp < 0)
    if len(sizes) == 2:          # one layer: the bound is the exact log-likelihood up to bf16 operands and the log Z estimate
        np.testing.assert_allclose(lp, A.brute_log_p_v(prm, X[:10]) - log_mean_, atol=0.1)
    clean(sim)


def test_python_refusals(sim, tmp_path):
    m, X = _stack(tmp_path, [6, 5, 4, 3], sample_h_states=[True, True, False])
    with pytest.raises(NotImplementedError, match='sampled states'):
        m.log_Z(n_betas=10, n_runs=4)
    assert m.log_proba(X[:4], 0.0).shape == (4,)            # the bound needs no sampled layer
    m64, X = _stack(tmp_path / 'f64', [6, 5, 4, 3], dtype='float64')
    for call in (lambda: m64.log_Z(n_betas=10, n_runs=4), lambda: m64.log_proba(X[:4], 0.0)):
        with pytest.raises(NotImplementedError, match='float32'):
            call()
    clean(sim)
