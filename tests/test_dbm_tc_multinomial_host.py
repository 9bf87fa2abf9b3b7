"""Multinomial hidden layers on the tensor-core DBM engine (csrc/bm_dbm_tc.cuh), checked without a GPU: the library's host
code on the stand-in runtime with every kernel interpreted on the CPU (tests/hostsim; the multinomial row kernel's restatement
is linked in by tests/hostsim/build_dbm_multinomial.sh), against the bf16 emulation
(tests/dbm_bf16_multinomial.py).  Means agree to one bf16 ulp, counts exactly; plus the dataflow of the cut programs, the
launches and host synchronisations of a step, and which engine a model is routed to."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_multinomial.so')     # + the row kernel's restatement
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')


def emulation():
    spec = importlib.util.spec_from_file_location('dbm_bf16_multinomial', os.path.join(ROOT, 'tests', 'dbm_bf16_multinomial.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.OracleDBMbf16Multinomial


@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_multinomial.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(SIM)
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    lib.fakecuda_hazard_launches.restype = C.c_long
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


def make_cfg(kinds, Hs, V=30, n_samples=300, gaussian=False, B=10, M=12, **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='gaussian' if gaussian else 'bernoulli', h_kinds=list(kinds),
               h_n_samples=[float(n_samples)] * L, dtype='float32', compute='bf16', n_particles=M, batch_size=B,
               max_mf_updates=6, mf_tol=1e-6, l2=1e-4, max_norm=3.0, sample_v=True, sample_h=[True] * L,
               sparsity_target=[0.2] * L, sparsity_cost=[0.01] * L, sparsity_damping=0.9)
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
    return d


def pair(cfg, scale=0.3):
    from boltzmann_machines import _native
    eng, emu = _native.CudaDBM(cfg), emulation()(cfg)
    assert eng.compute == 'bf16'
    d = params(cfg, scale)
    for e in (eng, emu):
        e.set_params(d)
        e.init_particles(4242)
    return eng, emu


def compare(cfg, g, w, names=None):
    """every variable to one bf16 ulp / 2e-5; the particles of multinomial layers exactly"""
    for k in (names or w):
        multi = k.startswith('h') and not k.startswith('hb') and cfg['h_kinds'][int(k[2:] or 0)] == 'multinomial'
        if multi:
            np.testing.assert_array_equal(g[k], w[k], err_msg=k)
        else:
            np.testing.assert_allclose(g[k], w[k], rtol=2.0 ** -7, atol=2e-5, err_msg=k)


def check_counts(cfg, got):
    for i, kind in enumerate(cfg['h_kinds']):
        if kind == 'multinomial' and cfg['sample_h'][i]:
            h = got['h' + ('' if i == 0 else '_%d' % i)]
            assert np.array_equal(h, np.round(h)) and np.all(h >= 0), i
            np.testing.assert_array_equal(h.sum(axis=1), np.full(h.shape[0], cfg['h_n_samples'][i], np.float32))


B_, M_ = 'bernoulli', 'multinomial'
CASES = [((B_, M_), (18, 11), 6, False), ((M_, B_), (19, 13), 300, False), ((B_, M_, B_), (18, 11, 7), 1000, False),
         ((B_, M_), (18, 11), 300, True), ((M_,), (21,), 1000, False)]


@pytest.mark.parametrize('kinds,Hs,n_samples,gaussian', CASES)
def test_training_and_queries_equal_the_emulation(executing, kinds, Hs, n_samples, gaussian):
    cfg = make_cfg(kinds, Hs, n_samples=n_samples, gaussian=gaussian)
    eng, emu = pair(cfg)
    compare(cfg, eng.get_params(), emu.get_params(), ['v'] + ['h' + ('' if i == 0 else '_%d' % i) for i in range(len(Hs))])
    rng = np.random.RandomState(5)
    for it in range(3):
        X = rng.randn(10, cfg['n_visible']).astype(np.float32) if gaussian else (rng.rand(10, cfg['n_visible']) < 0.3).astype(np.float32)
        a = eng.train_step(X, 0.05, 0.5, 2, 99, it, metrics=('msre', 'n_mf_updates'))
        b = emu.train_step(X, 0.05, 0.5, 2, 99, it, metrics=('msre', 'n_mf_updates'))
        assert a['n_mf_updates'] == b['n_mf_updates'], it
        assert a['msre'] == pytest.approx(b['msre'], rel=1e-3), it
    g = eng.get_params()
    compare(cfg, g, emu.get_params())
    check_counts(cfg, g)
    Xq = X[:7]
    tol = dict(rtol=2.0 ** -7, atol=2e-5)
    np.testing.assert_allclose(eng.transform(Xq), emu.transform(Xq), err_msg='transform', **tol)
    np.testing.assert_allclose(eng.reconstruct(Xq), emu.reconstruct(Xq), err_msg='reconstruct', **tol)
    np.testing.assert_allclose(eng.sample_v(2, 11, 4), emu.sample_v(2, 11, 4), err_msg='sample_v', **tol)
    g = eng.get_params()
    compare(cfg, g, emu.get_params())
    check_counts(cfg, g)
    clean(executing)
    eng.close()


@pytest.mark.parametrize('stop', [2, 5, 7, 'never', 'no-updates'])
def test_e_step_stops_where_the_emulation_does(executing, stop):
    """Speculated chunks of up to 5 sweeps, cut at the multinomial layer: the E-step keeps the sweep the emulation's
    sweep-by-sweep loop stops at -- inside the first chunk, at its last sweep, in a later chunk, never, and at
    max_mf_updates = 0."""
    cfg = make_cfg((B_, M_), (18, 11), n_samples=6, max_mf_updates=0 if stop == 'no-updates' else 12, mf_tol=-1.0)
    X = (np.random.RandomState(9).rand(7, cfg['n_visible']) < 0.3).astype(np.float32)
    if isinstance(stop, int):
        probe = emulation()(cfg)
        probe.set_params(params(cfg, 0.6))
        probe.init_particles(4242)
        cfg['mf_tol'] = probe.mf_tol_stopping_at(X, stop)
        assert cfg['mf_tol'] is not None, 'no tolerance stops the emulation after %d sweeps' % stop
    want = {'never': 12, 'no-updates': 0}.get(stop, stop)
    eng, emu = pair(cfg, 0.6)
    mu0 = eng.get_params(['mu_1'])['mu_1']
    a, b = eng.val_metrics(X, 1, 7, 3), emu.val_metrics(X, 1, 7, 3)
    assert a['n_mf_updates'] == b['n_mf_updates'] == want, (a['n_mf_updates'], b['n_mf_updates'])
    assert a['msre'] == pytest.approx(b['msre'], rel=1e-3)
    g, w = eng.get_params(), emu.get_params()
    compare(cfg, g, w, ['mu', 'mu_1', 'h', 'h_1'])
    if stop == 'no-updates':
        np.testing.assert_array_equal(g['mu_1'], mu0)
    clean(executing)
    eng.close()


@pytest.mark.parametrize('kinds', [(M_, B_), (B_, M_), (B_, M_, M_)])
def test_segmented_programs_have_no_dataflow_hazard(executing, kinds):
    """The checker of tools/hazard_check_configs.py on three 256-row blocks: the mean-field and particle programs cut at the
    multinomial layers declare every dependency their units need."""
    executing.fakecuda_set_hazards(2)
    try:
        Hs = (40, 24, 16)[:len(kinds)]
        cfg = make_cfg(kinds, Hs, V=70, B=600, M=520, n_samples=50)
        from boltzmann_machines import _native
        eng = _native.CudaDBM(cfg)
        eng.init_particles(1)
        X = (np.random.RandomState(0).rand(600, 70) < 0.3).astype(np.float32)
        before = executing.fakecuda_hazard_launches()
        eng.train_step(X, 0.05, 0.5, 2, 7, 0)
        assert executing.fakecuda_hazard_launches() - before >= 4
        clean(executing)
        eng.close()
    finally:
        executing.fakecuda_set_hazards(1)


def test_a_step_with_a_multinomial_layer_reads_one_flag_per_chunk(sim):
    """cfg4's shape (784-512-1024, batch = particles = 1024) with a multinomial top layer, 10 sweeps (two chunks of 5), CD-1:
    the step blocks the host exactly once per chunk, as the Bernoulli model does.  Launches: the approximate-inference
    pass adds one row kernel; a chunk of c sweeps runs c programs (each ending at the multinomial op) and c row kernels
    instead of one program; the particle sweep two programs and one row kernel instead of one program."""
    from boltzmann_machines import _native
    X = (np.random.RandomState(0).rand(1024, 784) < 0.2).astype(np.float32)
    counts = {}
    for top in (B_, M_):
        cfg = make_cfg((B_, top), (512, 1024), V=784, B=1024, M=1024, n_samples=100, max_mf_updates=10, mf_tol=-1.0)
        eng = _native.CudaDBM(cfg)
        assert eng.compute == 'bf16'
        eng.init_particles(1)
        eng.train_step(X, 0.01, 0.5, 1, 7, 0)                 # builds the programs
        sim.fakecuda_reset()
        eng.train_step(X, 0.01, 0.5, 1, 7, 1)
        counts[top] = (sim.fakecuda_syncs(), sim.fakecuda_launches(b''), sim.fakecuda_launches(b'tc_program_kernel'),
                       sim.fakecuda_launches(b'dbm_multinomial_rows_kernel'))
        clean(sim)
        eng.close()
    (sb, lb, pb, rb), (sm, lm, pm, rm) = counts[B_], counts[M_]
    assert sb == sm == 2, counts
    assert rb == 0 and rm == 1 + 10 + 1, counts
    assert pm == pb + 2 * 4 + 1, counts                    # two chunks: 5 programs for 1; particles: 2 for 1
    assert lm == lb + rm + (pm - pb), counts


def test_routing_is_opt_in(sim, monkeypatch):
    """Without an explicit request a multinomial model keeps the fp32 engine -- also under BM_COMPUTE=bf16 alone, which
    test sessions set; compute='bf16' or BM_DBM_COMPUTE=bf16 selects the tensor-core engine.  Bernoulli models as before."""
    from boltzmann_machines import _native
    sim.fakecuda_reset()
    for v in ('BM_COMPUTE', 'BM_DBM_COMPUTE'):
        monkeypatch.delenv(v, raising=False)

    def engine(kinds, compute=None, **env):
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            cfg = make_cfg(kinds, (9, 5), V=12)
            cfg.pop('compute')
            if compute:
                cfg['compute'] = compute
            eng = _native.CudaDBM(cfg)
            got = eng.compute
            eng.close()
        return got

    assert engine((B_, M_)) == 'fp32'
    assert engine((B_, M_), BM_COMPUTE='bf16') == 'fp32'
    assert engine((M_, B_), compute='bf16') == 'bf16'
    assert engine((B_, M_), BM_DBM_COMPUTE='bf16') == 'bf16'
    assert engine((B_, M_), BM_COMPUTE='bf16', BM_DBM_COMPUTE='fp32') == 'fp32'
    assert engine((B_, B_)) == 'bf16'
    assert engine((B_, B_), BM_COMPUTE='fp32') == 'fp32'
    clean(sim)


def test_binary_only_queries_refuse_multinomial_layers(sim):
    from boltzmann_machines import _native
    sim.fakecuda_reset()
    eng = _native.CudaDBM(make_cfg((B_, M_), (9, 5), V=12, B=4, M=4))
    with pytest.raises(RuntimeError, match='binary'):
        eng.log_proba(np.zeros((4, 12), np.float32))
    with pytest.raises(RuntimeError, match='binary'):
        eng.ais(4, 5, 1, 1)
    eng.close()
    clean(sim)


def test_particle_read_back_keeps_exact_counts(executing):
    """n_samples = 1000: the GEMM operand rounds counts above 256 to bf16, get_param returns the integers the draws produced
    (summing to n_samples per row) -- before and after other variables are set."""
    cfg = make_cfg((B_, M_), (18, 11), n_samples=1000, sparsity_cost=[0.0, 0.0])
    eng, emu = pair(cfg)
    X = (np.random.RandomState(3).rand(10, 30) < 0.3).astype(np.float32)
    eng.train_step(X, 0.05, 0.5, 1, 99, 0)
    emu.train_step(X, 0.05, 0.5, 1, 99, 0)
    h = eng.get_params(['h_1'])['h_1']
    check_counts(cfg, {'h_1': h})
    from oracle.rbm import bf16_round
    assert not np.array_equal(bf16_round(h), h)            # some counts are not representable in bf16
    np.testing.assert_array_equal(h, emu.get_params(['h_1'])['h_1'])
    eng.set_params({'vb': np.zeros(30, np.float32)})
    np.testing.assert_array_equal(eng.get_params(['h_1'])['h_1'], h)
    clean(executing)
    eng.close()
