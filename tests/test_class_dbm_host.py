"""Classification DBMs (DESIGN.md §5.7), checked without a GPU.

* The float64 statement (tests/class_dbm_oracle.py, ClassDBM64) against the model's mathematics: the labelled positive
  phase is the finite-difference gradient of the clamped variational bound; the persistent chains sweeping v, h.., y sample
  the exact p(v, y) of enumerable models (chi-square), and the same statistic rejects two wrong label samplers.
* The tensor-core engine's host code on the stand-in runtime with every kernel interpreted on the CPU (tests/hostsim;
  tests/hostsim/build_class_dbm.sh links the restatements of the multinomial row kernel and of the label clamp) against the
  bf16 emulation (particles exactly), against the float64 statement (to the bf16 bound) and against the plain DBM engine
  (bit for bit); plus the refusals, the launches of a labelled step and the Python model class."""
import ctypes as C
import importlib.util
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_class_dbm.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')


def oracle():
    spec = importlib.util.spec_from_file_location('class_dbm_oracle', os.path.join(ROOT, 'tests', 'class_dbm_oracle.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_class_dbm.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(SIM)
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    lib.fakecuda_launches.restype = C.c_long
    lib.fakecuda_launches.argtypes = [C.c_char_p]
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    yield lib
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib


@pytest.fixture
def executing(sim):
    sim.fakecuda_reset()
    sim.fakecuda_set_execute(1)
    yield sim
    sim.fakecuda_set_execute(0)


def clean(sim):
    v, sk = sim.fakecuda_violation().decode(), sim.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


def make_cfg(Hs, C=4, V=30, kinds=None, gaussian=False, B=10, M=12, **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='gaussian' if gaussian else 'bernoulli',
               h_kinds=list(kinds or ['bernoulli'] * L), h_n_samples=[50.] * L, dtype='float32', compute='bf16',
               n_particles=M, batch_size=B, max_mf_updates=7, mf_tol=1e-6, l2=1e-4, max_norm=3.0, sample_v=True,
               sample_h=[True] * L, sparsity_target=[0.2] * L, sparsity_cost=[0.01] * L, sparsity_damping=0.9,
               n_classes=C)
    if gaussian:
        cfg['sigma'] = np.linspace(0.7, 1.3, V)
    cfg.update(kw)
    return cfg


def params(cfg, scale=0.3, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [cfg['n_visible']] + cfg['n_hiddens']
    d = {'vb': (0.1 * rng.randn(sizes[0])).astype(np.float32)}
    for i in range(len(cfg['n_hiddens'])):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = (0.1 * rng.randn(sizes[i + 1])).astype(np.float32)
    C = cfg['n_classes']
    d['U'] = (scale * rng.randn(C, sizes[-1])).astype(np.float32)
    d['yb'] = (0.1 * rng.randn(C)).astype(np.float32)
    return d


def batch(cfg, rng, rows=10):
    if cfg['v_kind'] == 'gaussian':
        return rng.randn(rows, cfg['n_visible']).astype(np.float32)
    return (rng.rand(rows, cfg['n_visible']) < 0.3).astype(np.float32)


def labels(kind, rows, C, rng):
    y = rng.randint(0, C, size=rows).astype(np.int32)
    if kind == 'none':
        y[:] = -1
    elif kind == 'mixed':
        y[::3] = -1
    return y


PARTICLES = ('v', 'h', 'h_1', 'h_2', 'y')


def compare(g, w, names=None):
    """the particles exactly (every draw the same, Gaussian visibles included: the sampled value is rounded to bf16 from the
    same fp32 mean and noise); every other variable to one bf16 ulp / 2e-5 (fp32 sums in another order)"""
    for k in (names or w):
        if k in PARTICLES:
            np.testing.assert_array_equal(g[k], w[k], err_msg=k)
        else:
            np.testing.assert_allclose(g[k], w[k], rtol=2.0 ** -7, atol=2e-5, err_msg=k)


# ---- the float64 statement against the model's mathematics ----------------------------------------------------------
def stmt_cfg(Hs, V, C, M=8, B=4, **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, h_n_samples=[1.] * L,
               dtype='float64', n_particles=M, batch_size=B, max_mf_updates=4000, mf_tol=1e-14, l2=0., max_norm=np.inf,
               sample_v=True, sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[0.] * L, sparsity_damping=0.9,
               n_classes=C)
    cfg.update(kw)
    return cfg


def test_labelled_positive_phase_is_the_gradient_of_the_clamped_bound():
    """F(theta) = mean over rows of max_q E_q[-E(x, h, y = t)] + H(q), q factorised over h_1..h_L with y clamped to t, is
    computed by the statement's clamped E-step run to its fixed point.  By stationarity dF/dtheta is the positive phase the
    update uses: x mu_1^T, mu_{i-1} mu_i^T, e_t mu_L^T for U, mu_i and e_t for the biases.  Central differences agree."""
    mod = oracle()
    cfg = stmt_cfg([5, 4], 6, 3)
    d = params(dict(cfg, n_hiddens=[5, 4]), scale=0.5, seed=4)
    d = {k: v.astype(np.float64) for k, v in d.items()}
    rng = np.random.RandomState(2)
    X = (rng.rand(4, 6) < 0.5).astype(np.float64)
    t = np.array([0, 2, 1, 2])

    def F(dd):
        o = mod.ClassDBM64(cfg)
        o.set_params(dd)
        o._labels = t
        o.mean_field(X)
        return float(mod.bound_terms(o, X, t).mean()), o

    _, o = F(d)
    mu0, mu1, q = o.p['mu'][:4], o.p['mu_1'][:4], o.p['mu_2'][:4]
    np.testing.assert_array_equal(q, np.eye(3)[t])
    pos = {'W': X.T @ mu0 / 4, 'W_1': mu0.T @ mu1 / 4, 'U': q.T @ mu1 / 4, 'hb': mu0.mean(0), 'hb_1': mu1.mean(0),
           'yb': q.mean(0)}
    eps = 1e-5
    for name, idx in [('W', (1, 2)), ('W', (5, 0)), ('W_1', (3, 1)), ('W_1', (0, 3)), ('U', (2, 1)), ('U', (1, 3)),
                      ('U', (0, 0)), ('hb', (4,)), ('hb_1', (2,)), ('yb', (1,)), ('yb', (2,))]:
        fd = []
        for sgn in (1, -1):
            dd = {k: v.copy() for k, v in d.items()}
            dd[name][idx] += sgn * eps
            fd.append(F(dd)[0])
        grad = (fd[0] - fd[1]) / (2 * eps)
        assert abs(grad - pos[name][idx]) < 1e-7, (name, idx, grad, pos[name][idx])


CHI2_ROUNDS, CHI2_BURN, CHI2_THIN = 1500, 100, 10      # rounds of one sweep; samples every 10th round after 100
CHI2_LIMIT = 2.0                                       # chi-square / degrees of freedom of a correct sampler (test_dbm_pt_host)


def chi2_vy(Hs, V, C=3, mutation=None, seed=11, M=256):
    """chains of the statement (k = 1 sweeps over v, h_1 .. h_L, y) against the exact p(v, y), chi-square per dof"""
    mod = oracle()
    cfg = stmt_cfg(Hs, V, C, M=M)
    o = mod.ClassDBM64(cfg, mutation=mutation)
    d = params(dict(cfg, n_hiddens=list(Hs)), scale=1.0, seed=3)
    d['yb'] = np.array([0.8, -0.6, 0.1][:C], np.float32)
    o.set_params(d)
    o.init_particles(5)
    pw = 2 ** np.arange(V)
    counts = np.zeros(2 ** V * C)
    for r in range(CHI2_ROUNDS):
        o.particles_update(1, True, seed, r)
        if r >= CHI2_BURN and r % CHI2_THIN == 0:
            v, y = o.p['v'], o.p['h' + mod.sfx(len(Hs))]
            assert np.all(y.sum(1) == 1)
            counts += np.bincount((v @ pw).astype(np.int64) * C + np.argmax(y, 1), minlength=2 ** V * C)
    logp = mod.exact_log_p_vy({k: v.astype(np.float64) for k, v in d.items()}, Hs).ravel()
    n = counts.sum()
    expct = n * np.exp(logp)
    keep = expct >= 5
    obs, ex = np.append(counts[keep], counts[~keep].sum()), np.append(expct[keep], expct[~keep].sum())
    if ex[-1] < 5:
        obs, ex = obs[:-1], ex[:-1]
    return float(((obs - ex) ** 2 / ex).sum() / max(len(ex) - 1, 1))


@pytest.mark.parametrize('Hs,V', [([4], 5), ([4, 3], 5)])
def test_chains_sample_the_exact_joint_of_v_and_y(Hs, V):
    stat = chi2_vy(Hs, V)
    assert stat < CHI2_LIMIT, stat


@pytest.mark.parametrize('mutation', ['no_yb', 'below'])
def test_chi2_rejects_wrong_label_samplers(mutation):
    stat = chi2_vy([4, 3], 5, mutation=mutation)
    assert stat > 4 * CHI2_LIMIT, (mutation, stat)


B_, M_ = 'bernoulli', 'multinomial'
MODELS = {'L1': dict(Hs=(18,)), 'L2': dict(Hs=(18, 11)), 'L3-ragged': dict(Hs=(19, 13, 7), V=29, C=5),
          'gaussian': dict(Hs=(18, 11), gaussian=True), 'multinomial-hL': dict(Hs=(18, 11), kinds=[B_, M_])}


@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('labelled', ['all', 'mixed', 'none'])
@pytest.mark.parametrize('model', sorted(MODELS))
def test_training_and_queries_equal_the_emulation(executing, model, labelled, k):
    from boltzmann_machines import _native
    cfg = make_cfg(**MODELS[model])
    eng, emu = _native.CudaDBM(cfg), oracle().ClassDBMbf16(cfg)
    d = params(cfg)
    for e in (eng, emu):
        e.set_params(d)
        e.init_particles(4242)
    compare(eng.get_params(), emu.get_params())
    rng = np.random.RandomState(5)
    C = cfg['n_classes']
    for it in range(3):
        X = batch(cfg, rng)
        y = labels(labelled, 10, C, rng)
        a = eng.train_step(X, 0.05, 0.5, k, 99, it, metrics=('msre', 'n_mf_updates'), labels=y)
        b = emu.train_step(X, 0.05, 0.5, k, 99, it, metrics=('msre', 'n_mf_updates'), labels=y)
        assert a['n_mf_updates'] == b['n_mf_updates'], it
        assert a['msre'] == pytest.approx(b['msre'], rel=1e-3), it
        g = eng.get_params(['mu_y'])['mu_y'][:10]
        on = y >= 0
        np.testing.assert_array_equal(g[on], np.eye(C, dtype=np.float32)[y[on]])       # clamped rows: exactly one-hot
    g = eng.get_params()
    compare(g, emu.get_params())
    assert np.array_equal(g['y'].sum(axis=1), np.ones(cfg['n_particles'], np.float32))
    Xq = X[:7]
    tol = dict(rtol=2.0 ** -7, atol=2e-5)
    np.testing.assert_allclose(eng.predict_proba(Xq), emu.predict_proba(Xq), err_msg='predict_proba', **tol)
    np.testing.assert_allclose(eng.transform(Xq), emu.transform(Xq), err_msg='transform', **tol)
    compare(eng.get_params(), emu.get_params())
    clean(executing)
    eng.close()


@pytest.mark.parametrize('model', ['L2', 'gaussian'])
def test_engine_e_step_and_queries_near_float64(executing, model):
    """the engine's E-step of a mixed step, predict_proba and transform against the float64 statement on the same state:
    fixed 7 sweeps (mf_tol < 0), every value to 3e-2 (bf16 operands and activations through 7 sweeps); labelled slots exact"""
    from boltzmann_machines import _native
    cfg = make_cfg(**dict(MODELS[model], max_mf_updates=7, mf_tol=-1.0))
    eng, ref = _native.CudaDBM(cfg), oracle().ClassDBM64(cfg)
    d = params(cfg)
    for e in (eng, ref):
        e.set_params(d)
        e.init_particles(4242)
    rng = np.random.RandomState(8)
    X = batch(cfg, rng)
    Xq = batch(cfg, rng)[:7]
    for name, f in (('predict_proba', lambda e: e.predict_proba(Xq)), ('transform', lambda e: e.transform(Xq))):
        np.testing.assert_allclose(f(eng), f(ref), atol=3e-2, err_msg=name)
    y = labels('mixed', 10, cfg['n_classes'], rng)
    eng.train_step(X, 0.05, 0.5, 1, 99, 0, labels=y)
    ref.train_step(X, 0.05, 0.5, 1, 99, 0, labels=y)
    g, w = eng.get_params(), ref.get_params()
    for k in ('mu', 'mu_1', 'mu_y'):
        np.testing.assert_allclose(g[k][:10], w[k][:10], atol=3e-2, err_msg=k)
    np.testing.assert_array_equal(g['mu_y'][:10][y >= 0], w['mu_y'][:10][y >= 0])
    clean(executing)
    eng.close()


def plain_engine(cfg):
    from boltzmann_machines import _native
    return _native.CudaDBM(oracle().plain_cfg(cfg))


@pytest.mark.parametrize('model', ['L1', 'L2', 'L3-ragged', 'gaussian'])
def test_unlabelled_batches_are_the_plain_dbm_bit_for_bit(executing, model):
    """labels of -1 only (and bm_dbm_train_step without labels) = the plain DBM with a multinomial top layer of C units,
    n_samples 1, sampled, sparsity cost 0: every variable bit for bit"""
    from boltzmann_machines import _native
    cfg = make_cfg(**MODELS[model])
    L = len(cfg['n_hiddens'])
    mod = oracle()
    eng, ref = _native.CudaDBM(cfg), plain_engine(cfg)
    d = params(cfg)
    eng.set_params(d)
    ref.set_params(mod.to_plain(d, L))
    for e in (eng, ref):
        e.init_particles(7)
    rng = np.random.RandomState(3)
    for it in range(3):
        X = batch(cfg, rng)
        ref.train_step(X, 0.05, 0.5, 2, 11, it)
        if it == 1:
            eng.train_step(X, 0.05, 0.5, 2, 11, it)
        else:
            eng.train_step(X, 0.05, 0.5, 2, 11, it, labels=np.full(10, -1, np.int32))
    g, w = eng.get_params(), mod.from_plain(ref.get_params(), L)
    assert sorted(g) == sorted(w)
    for k in g:
        np.testing.assert_array_equal(g[k], w[k], err_msg=k)
    X = batch(cfg, rng)
    ref.transform(X)                                  # (returns the label layer's mu: the plain DBM's top layer)
    np.testing.assert_array_equal(eng.transform(X), ref.get_params(['mu' + mod.sfx(L - 1)])['mu' + mod.sfx(L - 1)])
    clean(executing)


def test_refusals_launch_nothing(sim):
    from boltzmann_machines import _native
    sim.fakecuda_reset()
    cfg = make_cfg((18, 11))
    cases = [(dict(n_classes=1), ValueError, 'n_classes'), (dict(n_classes=-2), ValueError, 'n_classes'),
             (dict(compute='fp32'), NotImplementedError, 'compute fp32'),
             (dict(dtype='float64'), NotImplementedError, 'dtype float64'),
             (dict(pt_betas=[1.0, 0.5]), NotImplementedError, 'parallel tempering'),
             (dict(n_hiddens=[5] * 8, h_kinds=[B_] * 8, h_n_samples=[1.] * 8, sample_h=[1] * 8, sparsity_target=[0.] * 8,
                   sparsity_cost=[0.] * 8), ValueError, 'at most 7 hidden layers')]
    for kw, exc, msg in cases:
        c = dict(cfg)
        c.update(kw)
        with pytest.raises(exc, match=msg):
            _native.CudaDBM(c)
    assert sim.fakecuda_launches(b'') == 0
    eng = _native.CudaDBM(cfg)
    eng.set_params(params(cfg))
    sim.fakecuda_reset()
    X = np.zeros((10, 30), np.float32)
    for bad in ([4] + [0] * 9, [-2] + [0] * 9):
        with pytest.raises(RuntimeError, match='outside'):
            eng.train_step(X, 0.05, 0.5, 1, 1, 0, labels=np.array(bad, np.int32))
    with pytest.raises(RuntimeError, match='batch'):
        eng.train_step(np.zeros((11, 30), np.float32), 0.05, 0.5, 1, 1, 0, labels=np.zeros(11, np.int32))
    assert sim.fakecuda_launches(b'') == 0
    for what in ('log_proba', 'ais'):
        with pytest.raises(RuntimeError, match='classification DBM'):
            eng.log_proba(X) if what == 'log_proba' else eng.ais(4, 10, 1, 1)
    plain = plain_engine(cfg)
    with pytest.raises(RuntimeError, match='no label layer'):
        plain.train_step(X, 0.05, 0.5, 1, 1, 0, labels=np.zeros(10, np.int32))
    assert sim.fakecuda_launches(b'') == 0
    eng.close(); plain.close()


def program_launches_per_chunk(sim, make, step):
    """tc_program_kernel launches of one E-step chunk: a step whose E-step runs two chunks minus one that runs one"""
    n = []
    for max_mf in (5, 10):
        eng = make(max_mf)
        sim.fakecuda_reset()
        step(eng)
        n.append(sim.fakecuda_launches(b'tc_program_kernel'))
        eng.close()
    return n[1] - n[0]


def test_an_all_labelled_step_has_the_plain_programs_per_chunk(sim):
    """never-converging E-steps (mf_tol < 0): 5 speculated sweeps per chunk.  All labelled: the label layer runs no op and the
    chunk is ONE program, as for the plain DBM without the label; mixed: the label's row kernel cuts every sweep"""
    from boltzmann_machines import _native
    X = (np.random.RandomState(0).rand(10, 30) < 0.3).astype(np.float32)

    def cls(max_mf):
        cfg = make_cfg((18, 11), max_mf_updates=max_mf, mf_tol=-1.0)
        e = _native.CudaDBM(cfg)
        e.set_params(params(cfg))
        return e

    def plain(max_mf):
        cfg = make_cfg((18, 11), max_mf_updates=max_mf, mf_tol=-1.0)
        cfg.pop('n_classes')
        e = _native.CudaDBM(cfg)
        e.set_params({k: v for k, v in params(make_cfg((18, 11))).items() if k not in ('U', 'yb')})
        return e

    y = np.arange(10, dtype=np.int32) % 4
    per_all = program_launches_per_chunk(sim, cls, lambda e: e.train_step(X, 0.05, 0.5, 1, 1, 0, labels=y))
    per_plain = program_launches_per_chunk(sim, plain, lambda e: e.train_step(X, 0.05, 0.5, 1, 1, 0))
    ym = y.copy()
    ym[::2] = -1
    per_mixed = program_launches_per_chunk(sim, cls, lambda e: e.train_step(X, 0.05, 0.5, 1, 1, 0, labels=ym))
    assert per_plain == 1 and per_all == per_plain
    assert per_mixed == 5
    assert sim.fakecuda_launches(b'cdbm_clamp_labels_kernel') > 0


# ---- the Python model class -------------------------------------------------------------------------------------
def _stack(V=30, H1=18, H2=11, C=4, seed=0):
    from boltzmann_machines import BernoulliRBM, ClassificationRBM
    rng = np.random.RandomState(seed)
    r1 = BernoulliRBM(n_visible=V, n_hidden=H1)
    r2 = ClassificationRBM(n_visible=H1, n_hidden=H2, n_classes=C)
    w1 = {'W': (0.3 * rng.randn(V, H1)).astype(np.float32), 'vb': (0.1 * rng.randn(V)).astype(np.float32),
          'hb': (0.1 * rng.randn(H1)).astype(np.float32)}
    w2 = {'W': (0.3 * rng.randn(H1, H2)).astype(np.float32), 'vb': (0.1 * rng.randn(H1)).astype(np.float32),
          'hb': (0.1 * rng.randn(H2)).astype(np.float32), 'U': (0.3 * rng.randn(C, H2)).astype(np.float32),
          'yb': (0.1 * rng.randn(C)).astype(np.float32)}
    r1.get_tf_params = lambda scope=None: dict(w1)
    r2.get_tf_params = lambda scope=None: dict(w2)
    return [r1, r2], w1, w2


def test_python_class_composes_trains_and_round_trips(executing, tmp_path):
    from boltzmann_machines import ClassificationDBM
    rbms, w1, w2 = _stack()
    path = str(tmp_path / 'cdbm') + '/'
    m = ClassificationDBM(rbms, n_particles=12, batch_size=10, max_epoch=2, n_gibbs_steps=1, max_mf_updates=4,
                          learning_rate=0.01, verbose=False, model_path=path, random_seed=1, train_metrics_every_iter=1)
    m.init()
    got = m.get_tf_params(scope='weights')
    np.testing.assert_array_equal(got['U'], w2['U'])              # copied unchanged (bf16 shadows aside, the fp32 values)
    np.testing.assert_array_equal(got['yb'], w2['yb'])
    np.testing.assert_allclose(got['W'], w1['W'], rtol=0, atol=0)  # two RBMs: W unchanged, hb_0 halved + 0.5 vb_1
    np.testing.assert_allclose(got['hb'], 0.5 * w1['hb'] + 0.5 * w2['vb'], rtol=1e-7)
    np.testing.assert_array_equal(m.get_tf_params(scope='grads_accumulators')['dU'], 0)
    rng = np.random.RandomState(1)
    X = (rng.rand(30, 30) < 0.3).astype(np.float32)
    y = rng.randint(0, 4, 30)
    y[::4] = -1
    m.fit(X, y, X_val=X[:10], y_val=np.abs(y[:10]))
    val = [json.loads(l) for l in open(os.path.join(path, 'logs', 'val', 'scalars.jsonl'))]
    assert any('accuracy' in r and 'mean_nll' in r for r in val)
    assert any('mean_squared_recon_error' in r for r in val)
    before = m.get_tf_params()
    P = m.predict_proba(X[:13])
    assert P.shape == (13, 4) and P.dtype == np.float32
    np.testing.assert_allclose(P.sum(axis=1), 1, rtol=1e-5)
    np.testing.assert_array_equal(m.predict(X[:13]), np.argmax(P, axis=1))
    assert m.transform(X[:13]).shape == (13, 11)
    after = m.get_tf_params()
    for k in before:                                              # the queries leave no trace
        np.testing.assert_array_equal(before[k], after[k], err_msg=k)
    m2 = ClassificationDBM.load_model(path)
    assert m2.n_classes_ == 4
    np.testing.assert_array_equal(m2.predict_proba(X[:13]), P)
    clean(executing)


def test_python_class_refusals(sim):
    from boltzmann_machines import ClassificationDBM, BernoulliRBM
    rbms, _, _ = _stack()
    with pytest.raises(ValueError, match='last RBM'):
        ClassificationDBM(rbms[:1])
    with pytest.raises(ValueError, match='only the last'):
        ClassificationDBM([rbms[1], rbms[1]])
    with pytest.raises(NotImplementedError, match='parallel tempering'):
        ClassificationDBM(rbms, pt_betas=[1.0, 0.5])
    with pytest.raises(NotImplementedError, match='float32'):
        ClassificationDBM(rbms, dtype='float64')
    m = ClassificationDBM(rbms, n_particles=12, batch_size=10, verbose=False, save_after_each_epoch=False)
    with pytest.raises(ValueError, match='needs the labels'):
        m.fit(np.zeros((10, 30), np.float32))
    with pytest.raises(ValueError, match='labels must be integers'):
        m.fit(np.zeros((10, 30), np.float32), np.full(10, 4))
    with pytest.raises(ValueError, match='labels must be integers'):
        m.fit(np.zeros((10, 30), np.float32), np.zeros(10, int), X_val=np.zeros((10, 30), np.float32), y_val=np.full(10, -1))
    for f in (m.log_Z, lambda: m.log_proba(np.zeros((2, 30)), 0.)):
        with pytest.raises(NotImplementedError):
            f()
    assert isinstance(rbms[0], BernoulliRBM)
