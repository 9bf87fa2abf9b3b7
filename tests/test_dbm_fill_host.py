"""Clamped Gibbs chains (DESIGN.md §5.9, bm_dbm_fill), checked without a GPU.

* The float64 statement (tests/dbm_fill_oracle.py) samples the exact conditionals of models small enough to enumerate:
  p(v_miss | v_obs) of a Bernoulli 6-4 and a 5-4-3 DBM and of a sigma = 1 Gaussian 3-4 DBM, and p(v | y) of a classification
  5-4 DBM with 3 classes (chi-square per dof <= 2); the same statistic rejects the chain without the visible clamp and the one
  with the label left free.
* Both engines' host code on the stand-in runtime (tests/hostsim, build_dbm_fill.sh): the CUDA-core engine draws what the
  statement draws, state for state; the tensor-core engine equals the bf16 emulation -- every chain state exactly, the means to
  one bf16 ulp -- over depths, ragged widths, Gaussian visibles, a multinomial top layer, labelled / mixed / free label layers,
  tempered and centered models, k = 1 and longer chains.
* A call cut into chunks of 7 rows equals one call; a fill leaves every variable as it was and the next training step as it
  would have been; every refusal launches nothing; the Python classes wire it up.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dbm_fill_oracle as F  # noqa: E402
from oracle.dbm_bf16 import OracleDBMbf16  # noqa: E402

ROOT = os.path.dirname(HERE)
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_fill.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
CHI2_LIMIT = 2.0


def sfx(i):
    return '' if i == 0 else '_%d' % i


def make_cfg(Hs, V, B=16, dtype='float32', compute='bf16', **kw):
    L = len(Hs)
    c = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype=dtype, compute=compute,
             n_particles=8, batch_size=B, max_mf_updates=4, mf_tol=1e-6, l2=1e-4, max_norm=3.0, sample_v=True,
             sample_h=[True] * L, sparsity_target=[0.2] * L, sparsity_cost=[0.01] * L, sparsity_damping=0.9)
    c.update(kw)
    return c


def params(cfg, scale=0.8, bias=0.5, seed=0, n_classes=0):
    rng = np.random.RandomState(seed)
    sizes = [cfg['n_visible']] + list(cfg['n_hiddens'])
    d = {'vb': (bias * rng.randn(sizes[0])).astype(np.float32)}
    for i in range(len(cfg['n_hiddens'])):
        d['W' + sfx(i)] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + sfx(i)] = (bias * rng.randn(sizes[i + 1])).astype(np.float32)
    if n_classes:
        d['U'] = (1.5 * rng.randn(n_classes, sizes[-1])).astype(np.float32)
        d['yb'] = (bias * rng.randn(n_classes)).astype(np.float32)
    return d


# ---- the float64 statement samples the exact conditionals --------------------------------------------------------------------
N_CHAINS, K_CHAIN = 20000, 50


def missing_code(v, miss):
    return (np.round(v[:, miss]) @ (2 ** np.arange(len(miss)))).astype(np.int64)


def bernoulli_stat(Hs, V, obs, x_obs, clamp_v=True):
    c = make_cfg(Hs, V, dtype='float64', B=N_CHAINS)
    o = F.FillOracleDBM(c)
    d = params(c, scale=1.5, bias=0.6, seed=3)
    o.set_params(d)
    X = np.zeros((N_CHAINS, V))
    X[:, obs] = x_obs
    mask = np.zeros((N_CHAINS, V), np.uint8)
    mask[:, obs] = 1
    _, st = F.fill(o, X, mask, None, 0, K_CHAIN, 21, 0, clamp_v=clamp_v)
    miss = [j for j in range(V) if j not in obs]
    counts = np.bincount(missing_code(st['v'], miss), minlength=2 ** len(miss))
    want = F.conditional_table(F.exact_log_p_v({k: v.astype(np.float64) for k, v in d.items()}, Hs), V, obs, x_obs)
    return F.chi2_per_dof(counts, want)


@pytest.mark.parametrize('Hs,V,obs,x_obs', [([4], 6, [0, 1, 2], [1, 1, 0]), ([4, 3], 5, [1, 4], [1, 1])])
def test_statement_samples_exact_conditional(Hs, V, obs, x_obs):
    assert bernoulli_stat(Hs, V, obs, x_obs) <= CHI2_LIMIT


def test_chi2_rejects_chain_without_visible_clamp():
    assert bernoulli_stat([4], 6, [0, 1, 2], [1, 1, 0], clamp_v=False) > 5 * CHI2_LIMIT


def class_stat(clamp_y=True):
    c = make_cfg([4], 5, dtype='float64', B=N_CHAINS, n_classes=3, sparsity_cost=[0.])
    o = F.FillClassDBM64(c)
    d = params(c, scale=1.0, bias=0.5, seed=5, n_classes=3)
    o.set_params(d)
    y = (np.arange(N_CHAINS) % 3).astype(np.int32)
    X, mask = np.zeros((N_CHAINS, 5)), np.zeros((N_CHAINS, 5), np.uint8)
    _, st = F.fill(o, X, mask, y, 0, K_CHAIN, 33, 0, clamp_y=clamp_y)
    lp = F._cdbm.exact_log_p_vy({k: v.astype(np.float64) for k, v in d.items()}, [4])        # [2^5, 3]
    stats = []
    for t in range(3):
        p = np.exp(lp[:, t] - np.logaddexp.reduce(lp[:, t]))
        counts = np.bincount(missing_code(st['v'][y == t], list(range(5))), minlength=32)
        stats.append(F.chi2_per_dof(counts, p))
    return max(stats)


def test_statement_samples_class_conditional():
    assert class_stat() <= CHI2_LIMIT


def test_chi2_rejects_free_label():
    assert class_stat(clamp_y=False) > 5 * CHI2_LIMIT


def test_statement_samples_gaussian_conditional():
    """sigma = 1 Gaussian 3-4: p(v_2 | v_0, v_1) is a mixture over h of unit normals, binned at its deciles"""
    from scipy.stats import norm
    V, H = 3, 4
    c = make_cfg([H], V, dtype='float64', B=N_CHAINS, v_kind='gaussian', sigma=np.ones(V))
    o = F.FillOracleDBM(c)
    d = params(c, scale=0.7, bias=0.5, seed=9)
    o.set_params(d)
    x_obs = np.array([1.2, -0.4])
    X = np.zeros((N_CHAINS, V))
    X[:, :2] = x_obs
    mask = np.zeros((N_CHAINS, V), np.uint8)
    mask[:, :2] = 1

    def stat(clamp_v):
        _, st = F.fill(o, X, mask, None, 0, K_CHAIN, 4, 0, clamp_v=clamp_v)
        W, b, cc = d['W'].astype(np.float64), d['vb'].astype(np.float64), d['hb'].astype(np.float64)
        hs = F.states(H)
        mu = b[None, :] + hs @ W.T                                        # p(v | h) = N(b + W h, 1)
        logw = hs @ cc + 0.5 * (mu ** 2).sum(1)                        # log p(h) + const
        logw = logw + norm.logpdf(x_obs[None, :] - mu[:, :2]).sum(1)     # x p(v_obs | h)
        w = np.exp(logw - np.logaddexp.reduce(logw))
        grid = np.linspace(-8, 8, 40001)
        cdf = (w[None, :] * norm.cdf(grid[:, None] - mu[None, :, 2])).sum(1)
        edges = np.interp(np.arange(1, 10) / 10., cdf, grid)
        counts = np.bincount(np.searchsorted(edges, st['v'][:, 2]), minlength=10)
        return F.chi2_per_dof(counts, np.full(10, 0.1))
    assert stat(True) <= CHI2_LIMIT
    assert stat(False) > 5 * CHI2_LIMIT


# ---- the engines on the stand-in runtime ------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_fill.sh')], stdout=subprocess.DEVNULL)
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


def clean(sim, skipped_ok=False):
    v, sk = sim.fakecuda_violation().decode(), sim.fakecuda_skipped().decode()
    assert v == '' and (skipped_ok or sk == ''), (v, sk)


def batch(c, rows, seed, p_obs=0.5):
    rng = np.random.RandomState(seed)
    V = c['n_visible']
    X = (rng.randn(rows, V) if c.get('v_kind') == 'gaussian' else (rng.rand(rows, V) < 0.4)).astype(np.float32)
    return X, (rng.rand(rows, V) < p_obs).astype(np.uint8)


def engine(c, d):
    from boltzmann_machines import _native
    e = _native.CudaDBM(c)
    e.set_params(d)
    return e


def state_names(c):
    L = len(c['n_hiddens'])
    n = ['v'] + ['h' + sfx(i) for i in range(L)] + (['y'] if c.get('n_classes') else [])
    return n + [x + '_prev' for x in n]


def test_cuda_core_engine_draws_what_the_statement_draws(sim):
    for Hs, V, extra in (([5, 4], 7, {}), ([6], 9, dict(v_kind='gaussian', sigma=np.ones(9))),
                         ([5, 4], 7, dict(h_kinds=['bernoulli', 'multinomial'], h_n_samples=[100., 3.]))):
        c = make_cfg(Hs, V, compute='fp32', **extra)
        d = params(c, seed=len(Hs) + V)
        e = engine(c, d)
        o = F.FillOracleDBM(c)
        o.set_params(d)
        X, m = batch(c, 11, 2)
        for k in (1, 4):
            out = e.fill(X, m, row0=5, k=k, seed=17, tick=3)
            ref, st = F.fill(o, X, m, None, 5, k, 17, 3)
            for n in state_names(c):
                got, want = e.debug_last_fill(n, 11), st[n]
                if (n.startswith('v') and c['v_kind'] == 'gaussian') or (k == 1 and n.endswith('_prev')):
                    # Gaussian states and the start's means: the same expressions, fp32 rounding of the layer op's sums
                    assert np.allclose(got, want, rtol=1e-5, atol=1e-5), n
                else:
                    assert np.array_equal(got, want), (Hs, n, k)
            assert np.array_equal(out[m == 1], X[m == 1])
            assert np.allclose(out, ref, rtol=1e-5, atol=1e-6)
        e.close()
    clean(sim)


def tc_cases():
    g = dict(v_kind='gaussian', sigma=np.ones(9))
    return [
        ('L1', make_cfg([6], 9), None),
        ('L2', make_cfg([7, 5], 9), None),
        ('L3-ragged', make_cfg([13, 7, 10], 11), None),
        ('gaussian', make_cfg([6, 4], 9, **g), None),
        ('multinomial-top', make_cfg([6, 5], 9, h_kinds=['bernoulli', 'multinomial'], h_n_samples=[100., 4.]), None),
        ('pt', make_cfg([6, 4], 9, pt_betas=[1.0, 0.6, 0.3]), None),
        ('centered', make_cfg([6, 4], 9, centering=True, offset_rate=0.1), None),
        ('class-all', make_cfg([6, 5], 9, n_classes=4, sparsity_cost=[0.] * 2), 'all'),
        ('class-mixed', make_cfg([6, 5], 9, n_classes=4, sparsity_cost=[0.] * 2), 'mixed'),
        ('class-free', make_cfg([6, 5], 9, n_classes=4, sparsity_cost=[0.] * 2), 'free'),
    ]


def emulation(c):
    if c.get('n_classes'):
        return F._cdbm.ClassDBMbf16(c)
    if any(k == 'multinomial' for k in c['h_kinds']):
        return F._mult.OracleDBMbf16Multinomial(c)
    return OracleDBMbf16(c)


@pytest.mark.parametrize('name,c,labels', tc_cases(), ids=[t[0] for t in tc_cases()])
def test_tensor_core_engine_equals_bf16_emulation(sim, name, c, labels):
    C_ = c.get('n_classes', 0)
    d = params(c, seed=7, n_classes=C_)
    e = engine(c, d)
    e.init_particles(3)
    o = emulation(c)
    o.set_params(d)
    X, m = batch(c, 13, 4)
    y = None
    if labels is not None:
        y = {'all': np.arange(13) % C_, 'mixed': np.where(np.arange(13) % 3 == 0, -1, np.arange(13) % C_),
             'free': np.full(13, -1)}[labels].astype(np.int32)
    for k in (1, 5):
        out = e.fill(X, m, y, row0=40, k=k, seed=91, tick=6)
        ref, st = F.fill(o, X, m, y, 40, k, 91, 6, bf16=True)
        for n in state_names(c):
            assert np.array_equal(e.debug_last_fill(n, 13), st[n]), (name, n, k)
        ulp = np.abs(st['mean']) * 2. ** -8 + 1e-30
        assert np.all(np.abs(e.debug_last_fill('mean', 13) - st['mean']) <= ulp), (name, k)
        assert np.all(np.abs(out - ref) <= np.abs(ref) * 2. ** -8 + 1e-30), (name, k)
        assert np.array_equal(out[m == 1], X[m == 1])
    e.close()
    clean(sim)


@pytest.mark.parametrize('compute', ['fp32', 'bf16'])
def test_chunks_of_7_equal_one_call(sim, compute):
    c = make_cfg([7, 5], 9, compute=compute, B=64)
    d = params(c, seed=2)
    e = engine(c, d)
    X, m = batch(c, 64, 6)
    whole = e.fill(X, m, row0=0, k=3, seed=8, tick=1)
    parts = np.concatenate([e.fill(X[lo:lo + 7], m[lo:lo + 7], row0=lo, k=3, seed=8, tick=1) for lo in range(0, 64, 7)])
    assert np.array_equal(whole, parts)
    e.close()
    clean(sim)


@pytest.mark.parametrize('compute,extra', [('fp32', {}), ('bf16', {}), ('bf16', dict(n_classes=4, sparsity_cost=[0.] * 2))])
def test_fill_leaves_no_trace(sim, compute, extra):
    c = make_cfg([6, 5], 9, compute=compute, **extra)
    d = params(c, seed=3, n_classes=extra.get('n_classes', 0))
    a, b = engine(c, d), engine(c, d)
    for e in (a, b):
        e.init_particles(5)
    X, m = batch(c, 16, 1)
    before = a.get_params()
    y = (np.arange(16) % 4).astype(np.int32) if extra else None
    a.fill(X, m, y, row0=0, k=4, seed=3, tick=0)
    after = a.get_params()
    assert all(np.array_equal(before[n], after[n]) for n in before)
    kw = dict(labels=y) if extra else {}
    for e in (a, b):
        e.train_step(X, 0.05, 0.5, 2, seed=12, tick=1, **kw)
    pa, pb = a.get_params(), b.get_params()
    assert all(np.array_equal(pa[n], pb[n]) for n in pa)
    a.close(); b.close()
    clean(sim)


def test_refusals_launch_nothing(sim):
    from boltzmann_machines import _native
    ctx = _native.Context.default()
    plain = engine(make_cfg([6], 9), params(make_cfg([6], 9)))
    cls = engine(make_cfg([6], 9, n_classes=3, sparsity_cost=[0.]), params(make_cfg([6], 9), n_classes=3))
    X, m = batch(make_cfg([6], 9), 4, 0)
    lib = _native.load_library()
    cases = [
        (plain, X, m, None, dict(k=0), 'n_gibbs_steps'),
        (plain, X, m * 2, None, {}, 'mask byte'),
        (plain, X, m, np.zeros(4, np.int32), {}, 'no label layer'),
        (cls, X, m, np.array([0, 1, 3, -1], np.int32), {}, 'outside [-1, n_classes)'),
        (cls, X, m, np.array([0, -2, 1, -1], np.int32), {}, 'outside [-1, n_classes)'),
        (plain, np.zeros((17, 9), np.float32), np.zeros((17, 9), np.uint8), None, {}, 'rows must lie'),
    ]
    for e, Xc, mc, y, kw, msg in cases:
        n0 = ctx.launch_count()
        with pytest.raises(RuntimeError) as ei:
            e.fill(Xc, mc, y, row0=0, seed=1, tick=0, **kw)
        assert msg in str(ei.value), (msg, str(ei.value))
        assert ctx.launch_count() == n0, msg
    n0 = ctx.launch_count()
    out = (C.c_float * 36)()
    assert lib.bm_dbm_fill(plain.handle, None, m.ctypes.data, None, 4, 0, 1, 0, 0, out) != 0
    assert lib.bm_dbm_fill(plain.handle, X.ctypes.data, None, None, 4, 0, 1, 0, 0, out) != 0
    assert lib.bm_dbm_fill(plain.handle, X.ctypes.data, m.ctypes.data, None, 4, 0, 1, 0, 0, None) != 0
    assert ctx.launch_count() == n0
    with pytest.raises(RuntimeError):
        engine(make_cfg([6], 9), params(make_cfg([6], 9))).debug_last_fill('v', 4)      # before the first fill
    plain.close(); cls.close()
    clean(sim)


def test_launches_per_sweep(sim):
    """one program launch and the visible clamp per sweep (Bernoulli layers), independent of depth"""
    from boltzmann_machines import _native
    ctx = _native.Context.default()
    c = make_cfg([7, 5, 6], 9)
    e = engine(c, params(c))
    X, m = batch(c, 8, 0)
    counts = []
    for k in (2, 12):
        n0 = ctx.launch_count()
        e.fill(X, m, row0=0, k=k, seed=1, tick=0)
        counts.append(ctx.launch_count() - n0)
    assert (counts[1] - counts[0]) == 10 * 2, counts
    e.close()
    clean(sim)


# ---- the Python classes ------------------------------------------------------------------------------------------------------
def _dbm_model(tmp, cls_labels=False):
    from boltzmann_machines import DBM, ClassificationDBM
    from boltzmann_machines.rbm import BernoulliRBM
    from boltzmann_machines.rbm.class_rbm import ClassificationRBM
    rng = np.random.RandomState(0)
    X = (rng.rand(40, 9) < 0.4).astype(np.float32)
    r1 = BernoulliRBM(n_visible=9, n_hidden=6, max_epoch=1, batch_size=8, random_seed=1, model_path=str(tmp / 'r1'))
    r1.fit(X)
    if cls_labels:
        r2 = ClassificationRBM(n_visible=6, n_hidden=5, n_classes=3, max_epoch=1, batch_size=8, random_seed=2,
                               model_path=str(tmp / 'r2'))
        r2.fit(r1.transform(X), np.arange(40) % 3)
        m = ClassificationDBM(rbms=[r1, r2], n_particles=8, batch_size=8, max_epoch=1, random_seed=4,
                              model_path=str(tmp / 'dbm'))
        m.fit(X, np.arange(40) % 3)
    else:
        r2 = BernoulliRBM(n_visible=6, n_hidden=5, max_epoch=1, batch_size=8, random_seed=2, model_path=str(tmp / 'r2'))
        r2.fit(r1.transform(X))
        m = DBM(rbms=[r1, r2], n_particles=8, batch_size=8, max_epoch=1, random_seed=4, model_path=str(tmp / 'dbm'))
        m.fit(X)
    return m, X


@pytest.mark.parametrize('labelled', [False, True])
def test_python_fill_missing(sim, tmp_path, labelled):
    m, X = _dbm_model(tmp_path, labelled)
    mask = (np.random.RandomState(1).rand(*X.shape) < 0.5).astype(np.float32)
    kw = dict(y=np.arange(40) % 3 - (np.arange(40) % 5 == 0)) if labelled else {}
    a = m.fill_missing(X, mask, n_gibbs_steps=3, **kw)
    assert a.shape == X.shape and a.dtype == np.float32
    assert np.array_equal(a[mask == 1], X[mask == 1])
    b = m.fill_missing(X, mask, n_gibbs_steps=3, **kw)
    assert not np.array_equal(a, b)                                   # consecutive calls draw afresh
    cls = type(m)
    again = cls.load_model(str(tmp_path / 'dbm'))
    again.random_seed = m.random_seed
    m2 = cls.load_model(str(tmp_path / 'dbm'))
    assert np.array_equal(again.fill_missing(X, mask, n_gibbs_steps=3, **kw), m2.fill_missing(X, mask, n_gibbs_steps=3, **kw))
    for bad in (dict(mask=mask[:, :4]), dict(mask=mask * 2), dict(X=np.where(mask == 1, np.nan, X))):
        args = dict(X=X, mask=mask)
        args.update(bad)
        with pytest.raises(ValueError):
            m.fill_missing(args['X'], args['mask'], n_gibbs_steps=3, **kw)
    if labelled:
        gen = m.fill_missing(np.zeros((6, 9), np.float32), np.zeros((6, 9)), y=np.arange(6) % 3, n_gibbs_steps=2)
        assert gen.shape == (6, 9) and np.all((gen > 0) & (gen < 1))
    # the ClassificationRBM's pre-training runs kernels this library does not restate (tests/hostsim/build_crbm.sh does)
    clean(sim, skipped_ok=labelled)


def test_python_fill_missing_on_the_statement(tmp_path):
    """DBM.fill_missing under set_engine_factory: the float statement is an engine like the CUDA ones"""
    from boltzmann_machines.base import set_engine_factory
    old = set_engine_factory('dbm', F.factory)
    try:
        m, X = _dbm_model(tmp_path)
        mask = np.ones_like(X)
        mask[:, :4] = 0
        out = m.fill_missing(X, mask, n_gibbs_steps=2)
        assert np.array_equal(out[:, 4:], X[:, 4:]) and np.all((out[:, :4] > 0) & (out[:, :4] < 1))
    finally:
        set_engine_factory('dbm', old)
