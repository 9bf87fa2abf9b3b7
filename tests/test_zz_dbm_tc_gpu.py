"""Tensor-core DBM engine (compute='bf16', csrc/bm_dbm_tc.cuh) against its bf16-operand emulation
(oracle/dbm_bf16.py), the pinned fp32 oracle and exact enumeration.  The engine is the default for float32 models with
Bernoulli hidden layers."""
import os

import numpy as np
import pytest

from boltzmann_machines import _native
from oracle.dbm import OracleDBM
from oracle.dbm_bf16 import OracleDBMbf16
from oracle.rbm import bf16_round

pytestmark = pytest.mark.gpu


def make_cfg(V=30, Hs=(18, 11), **kw):
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * len(Hs),
               h_n_samples=[100.] * len(Hs), dtype='float32', compute='bf16', n_particles=12, batch_size=10,
               max_mf_updates=6, mf_tol=1e-6, l2=1e-4, max_norm=3.0, sample_v=True, sample_h=[True] * len(Hs),
               sparsity_target=[0.2] * len(Hs), sparsity_cost=[0.01] * len(Hs), sparsity_damping=0.9)
    cfg.update(kw)
    return cfg


def init(cfg, engines, seed=0, scale=0.3):
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
    return d


def batch(cfg, rows, seed=1):
    return (np.random.RandomState(seed).rand(rows, cfg['n_visible']) < 0.3).astype(np.float32)


def close_bf16(got, want, name, frac=0.1):
    """bf16-stored means: equal up to one bf16 ulp almost everywhere (the kernel's sigmoid is ex2/rcp based)."""
    np.testing.assert_allclose(got, want, rtol=2.0 ** -6, atol=1e-3, err_msg=name)
    assert np.mean(got != want) <= frac, name


def test_state_roundtrip_is_bf16_for_activations_and_fp32_for_variables():
    cfg = make_cfg()
    eng = _native.CudaDBM(cfg)
    assert eng.compute == 'bf16'
    d = init(cfg, (eng,))
    g = eng.get_params()
    for k in ('W', 'W_1', 'vb', 'hb', 'hb_1'):
        np.testing.assert_array_equal(g[k], d[k])
    emu = OracleDBMbf16(cfg); init(cfg, (emu,))
    w = emu.get_params()
    for k in ('v', 'h', 'h_1'):
        np.testing.assert_array_equal(g[k], w[k])
    eng.close()


@pytest.mark.parametrize('Hs', [(18,), (18, 11), (18, 11, 7), (70, 130)])
def test_mean_field_and_queries(Hs):
    """The second operand pair of a conditional reads a transposed shadow of W_{i+1}: both pairs MN-major."""
    cfg = make_cfg(Hs=Hs)
    eng, emu = _native.CudaDBM(cfg), OracleDBMbf16(cfg)
    init(cfg, (eng, emu))
    Xq = batch(cfg, 7, seed=9)
    close_bf16(eng.transform(Xq), emu.transform(Xq), 'transform')
    close_bf16(eng.reconstruct(Xq), emu.reconstruct(Xq), 'reconstruct')
    if len(Hs) == 2:
        np.testing.assert_allclose(eng.log_proba(Xq), emu.log_proba(Xq), atol=0.05)
    g, w = eng.get_params(['mu']), emu.get_params(['mu'])
    close_bf16(g['mu'][:7], w['mu'][:7], 'mu')
    eng.close()


@pytest.mark.parametrize('Hs', [(18,), (18, 11), (18, 11, 7)])
def test_training_steps_track_the_emulation(Hs):
    cfg = make_cfg(Hs=Hs)
    eng, emu = _native.CudaDBM(cfg), OracleDBMbf16(cfg)
    init(cfg, (eng, emu))
    for it in range(3):
        X = batch(cfg, 10, seed=it)
        got = eng.train_step(X, 0.05, 0.5, 2, 99, it, metrics=('msre', 'n_mf_updates'))
        want = emu.train_step(X, 0.05, 0.5, 2, 99, it, metrics=('msre', 'n_mf_updates'))
        assert got['msre'] == pytest.approx(want['msre'], rel=0.05)
        assert abs(got['n_mf_updates'] - want['n_mf_updates']) <= 1
    g, w = eng.get_params(), emu.get_params()
    for k in w:
        if k.startswith(('W', 'dW', 'vb', 'hb', 'dvb', 'dhb')):
            np.testing.assert_allclose(g[k], w[k], atol=2e-2, err_msg=k)
    assert set(np.unique(g['h'])) <= {0.0, 1.0}
    # a Bernoulli draw may differ only where u is within rounding of p: particles agree almost everywhere
    assert np.mean(g['h'] != w['h']) < 0.1
    eng.close()


def test_first_gibbs_sweep_is_the_philox_draw():
    """One sampled sweep from identical particles: states equal the emulation's except at rounding-level ties."""
    cfg = make_cfg(V=784, Hs=(512, 256), n_particles=256, batch_size=16)
    eng, emu = _native.CudaDBM(cfg), OracleDBMbf16(cfg)
    init(cfg, (eng, emu), scale=0.05)
    X = batch(cfg, 16)
    eng.val_metrics(X, 1, 77, 3); emu.val_metrics(X, 1, 77, 3)
    g, w = eng.get_params(['v', 'h', 'h_1']), emu.get_params(['v', 'h', 'h_1'])
    for k in w:
        assert set(np.unique(g[k])) <= {0.0, 1.0}, k
        assert np.mean(g[k] != w[k]) < 0.01, (k, np.mean(g[k] != w[k]))
    eng.close()


_EMU_AIS = {}


def _emulated_ladder(cfg, k, n_betas):
    """the bf16 emulation's ladder (numpy loops: a minute per call), computed once per model"""
    key = (k, n_betas, tuple(cfg['sample_h']))
    if key not in _EMU_AIS:
        emu = OracleDBMbf16(cfg)
        init(cfg, (emu,))
        _EMU_AIS[key] = (emu.ais(32, n_betas, k, 2222), emu.get_params())
    return _EMU_AIS[key]


@pytest.mark.parametrize('k', [1, 3])
def test_ais_matches_exact_enumeration(k):
    """Weight increments and unit updates inside the epilogues of the three tensor-core ops of a temperature step, up to 30
    steps per persistent launch (a model whose first hidden layer is sampled)."""
    cfg = make_cfg(V=7, Hs=(5, 4), n_particles=4, batch_size=4)
    n_betas = 240 if k == 1 else 120
    eng = _native.CudaDBM(cfg)
    init(cfg, (eng,))
    a = eng.ais(32, n_betas, k, 2222)
    b, p = _emulated_ladder(cfg, k, n_betas)
    lm = lambda v: np.logaddexp.reduce(v) - np.log(len(v))
    assert abs(lm(a) - lm(b)) < 0.1
    assert np.mean(np.abs(a - b) < 2e-3) > 0.8           # the same chains, but for a draw at rounding distance of its probability
    W0, W1 = bf16_round(p['W']).astype(np.float64), bf16_round(p['W_1']).astype(np.float64)
    terms = []
    for s in range(2 ** 5):
        x = np.array([(s >> i) & 1 for i in range(5)], dtype=np.float64)
        terms.append(x @ p['hb'] + np.logaddexp(0, W0 @ x + p['vb']).sum() + np.logaddexp(0, x @ W1 + p['hb_1']).sum())
    exact = np.logaddexp.reduce(terms)
    assert abs(lm(a) - exact) < 0.15, (lm(a), exact)
    eng.close()


@pytest.mark.parametrize('k', [1, 3])
def test_ais_of_a_mean_valued_first_layer_matches_the_emulation(k):
    """A model whose first hidden layer is not sampled runs the ladder over fp32 pre-activations in memory, one fused pass over
    them per temperature (DbmTC::ais_local_passes): same expressions, same Philox sites as the emulation."""
    cfg = make_cfg(V=7, Hs=(5, 4), n_particles=4, batch_size=4, sample_h=[False, True])
    n_betas = 240 if k == 1 else 120
    eng = _native.CudaDBM(cfg)
    init(cfg, (eng,))
    a = eng.ais(32, n_betas, k, 2222)
    b, _ = _emulated_ladder(cfg, k, n_betas)
    lm = lambda v: np.logaddexp.reduce(v) - np.log(len(v))
    assert abs(lm(a) - lm(b)) < 0.1
    assert np.mean(np.abs(a - b) < 2e-3) > 0.8           # the same chains, but for a draw at rounding distance of its probability
    eng.close()


def test_ais_fine_ladder_takes_the_series_form_and_matches_the_emulation():
    """ladders of >= 400 temperatures compute the weight increment of a unit as t * sigmoid(m z), the sigmoid taken as a
    third-order series around the one the draw needs (bm_tc.cu: MODE_AIS_UNITS): same chains and log-weights as the emulation's
    closed form softplus(b z) - softplus(a z)."""
    cfg = make_cfg(V=7, Hs=(5, 4), n_particles=4, batch_size=4)
    eng, emu = _native.CudaDBM(cfg), OracleDBMbf16(cfg)
    init(cfg, (eng, emu), scale=1.0)                      # pre-activations of several units in magnitude
    a, b = eng.ais(12, 500, 1, 31), emu.ais(12, 500, 1, 31)
    assert np.mean(np.abs(a - b) < 2e-3) >= 0.75, np.abs(a - b)
    assert abs(np.mean(a) - np.mean(b)) < 0.05
    eng.close()


def test_ais_is_within_one_nat_of_the_pinned_oracle():
    """BASELINE.json: AIS log Z within +-1.0 of the reference path (784-64-32, 64 runs x 200 betas)."""
    cfg = make_cfg(V=784, Hs=(64, 32), n_particles=4, batch_size=4)
    eng, ref = _native.CudaDBM(cfg), OracleDBM(dict(cfg, compute='fp32'))
    init(cfg, (eng, ref), scale=0.05)
    a = eng.ais(64, 200, 1, 1)
    b = ref.ais(64, 200, 1, 1)
    lm = lambda v: np.logaddexp.reduce(v) - np.log(len(v))
    assert abs(lm(a) - lm(b)) < 1.0
    eng.close()


def test_ais_at_the_benchmark_shape_is_within_one_nat_of_the_float64_oracle():
    """north_star's gate at BASELINE.json configs[3]'s own shape: DBM 784-512-1024, 256 runs x 1000 betas -- the tensor-core
    ladder (bf16 operands, epilogue-fused) against the float64 oracle on identical weights, and against the fp32 CUDA-core
    engine (same chains up to rounding).  The oracle's 256 log-weights are a committed fixture (minutes of numpy:
    tests/golden/make_ais_benchmark_oracle.py; tests/test_oracle_fixtures.py re-derives some of its chains on the CPU)."""
    import json
    fx = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ais_benchmark_shape_oracle.json')))
    sh = fx['shape']
    cfg = make_cfg(V=sh['V'], Hs=tuple(sh['Hs']), n_particles=4, batch_size=4)
    eng, simt = _native.CudaDBM(cfg), _native.CudaDBM(dict(cfg, compute='fp32'))
    assert eng.compute == 'bf16'
    init(cfg, (eng, simt), seed=sh['weight_seed'], scale=sh['weight_scale'])
    lm = lambda v: np.logaddexp.reduce(v) - np.log(len(v))
    n = fx['n_runs']
    a, b = eng.ais(n, sh['n_betas'], sh['n_gibbs_steps'], sh['seed']), simt.ais(n, sh['n_betas'], sh['n_gibbs_steps'], sh['seed'])
    c = np.asarray(fx['log_weights'], dtype=np.float64)
    assert abs(lm(a) - lm(c)) < 1.0, (lm(a), lm(c))
    assert abs(lm(b) - lm(c)) < 1.0, (lm(b), lm(c))
    assert abs(np.mean(a) - np.mean(c)) < 1.0 and abs(np.mean(b) - np.mean(c)) < 1.0
    # the ladder's spread is the chains' own (std 0.17 nats in the oracle), not rounding noise on top of it
    assert np.std(a) < 3 * np.std(c) + 0.05 and np.std(b) < 3 * np.std(c) + 0.05
    eng.close(); simt.close()


def test_cfg4_shape_step_agrees_with_the_fp32_engine():
    """BASELINE.json configs[3] shape: DBM 784-512-1024, 1024 particles, batch 1024, 25 mean-field updates."""
    base = make_cfg(V=784, Hs=(512, 1024), n_particles=1024, batch_size=1024, max_mf_updates=25, mf_tol=1e-7,
                    max_norm=6.0, sparsity_cost=[0., 0.])
    tc, simt = _native.CudaDBM(base), _native.CudaDBM(dict(base, compute='fp32'))
    assert tc.compute == 'bf16' and simt.compute == 'fp32'
    init(base, (tc, simt), scale=0.02)
    X = batch(base, 1024)
    a = tc.train_step(X, 2e-3, 0.5, 1, 7, 0, metrics=('msre', 'n_mf_updates'))
    b = simt.train_step(X, 2e-3, 0.5, 1, 7, 0, metrics=('msre', 'n_mf_updates'))
    assert a['msre'] == pytest.approx(b['msre'], rel=0.02)
    ga, gb = tc.get_params(['W', 'W_1', 'vb', 'hb', 'hb_1']), simt.get_params(['W', 'W_1', 'vb', 'hb', 'hb_1'])
    for k in ga:
        rel = np.linalg.norm(ga[k] - gb[k]) / max(np.linalg.norm(gb[k]), 1e-12)
        assert rel < 0.02, (k, rel)
    tc.close(); simt.close()


@pytest.mark.parametrize('Hs,rows,stop', [(Hs, rows, stop) for Hs, rows in (((18, 11), 10), ((18, 11, 7), 10))
                                           for stop in (2, 5, 7, 'never', 'no-updates')] +
                                          [((512, 1024), 300, stop) for stop in (2, 5, 'never', 'no-updates')])
def test_mean_field_programs_equal_the_emulation(Hs, rows, stop):
    """The E-step runs as persistent dataflow programs of up to 5 speculated sweeps per launch (DbmTC::MF_CHUNK); the first
    sweep index whose convergence test passes is picked afterwards, so mu and n_mf_updates are those of the emulation's
    sweep-by-sweep loop up to fp32 summation order.  Stops inside the first program (2), at its last sweep (5), in a later one
    (7), at max_mf_updates = 8 (never converged: a second program of 3 sweeps), and at max_mf_updates = 0 (mu unchanged); the
    tolerance for a stop is read off the emulation's convergence measures.  The 784-512-1024 model converges to a one-ulp
    oscillation by its sixth sweep, so its later program is reached through max_mf_updates only."""
    V = 30 if Hs[0] < 100 else 784
    scale = 0.6 if V == 30 else 0.04
    cfg = make_cfg(V=V, Hs=Hs, batch_size=max(rows, 10), max_mf_updates=0 if stop == 'no-updates' else 8, mf_tol=-1.0)
    if isinstance(stop, int):
        probe = OracleDBMbf16(cfg)
        init(cfg, (probe,), scale=scale)
        cfg['mf_tol'] = probe.mf_tol_stopping_at(batch(cfg, rows, seed=0), stop)
        assert cfg['mf_tol'] is not None, 'no tolerance stops the emulation after %d sweeps' % stop
    eng, emu = _native.CudaDBM(cfg), OracleDBMbf16(cfg)
    init(cfg, (eng, emu), scale=scale)
    mu0 = eng.get_params(['mu'])['mu']
    names = ['mu' + ('' if i == 0 else '_%d' % i) for i in range(len(Hs))]
    for it in range(2):                      # the second E-step starts from the first one's mu (stale-mu quirk)
        X = batch(cfg, rows, seed=it)
        a, b = eng.val_metrics(X, 1, 5, it), emu.val_metrics(X, 1, 5, it)
        if it == 0:
            assert b['n_mf_updates'] == {'never': 8, 'no-updates': 0}.get(stop, stop)
        # only the order in which a consumer adds its K chunks may follow the producers' completion order (granule-level
        # dataflow), i.e. fp32 rounding before the bf16 store
        assert abs(a['n_mf_updates'] - b['n_mf_updates']) <= 1
        assert a['msre'] == pytest.approx(b['msre'], rel=1e-2)
        ga, gb = eng.get_params(names), emu.get_params(names)
        for k in names:
            np.testing.assert_allclose(ga[k], gb[k], rtol=2.0 ** -7, atol=1e-3, err_msg=k)
            assert np.mean(ga[k] != gb[k]) < 0.02, k
    if stop == 'no-updates':
        np.testing.assert_array_equal(ga['mu'], mu0)
    eng.close()


@pytest.mark.parametrize('Hs,k', [((18,), 3), ((18, 11), 1), ((18, 11, 7), 2), ((512,), 5), ((512, 256), 2)])
def test_particle_sweep_program_equals_the_emulation(Hs, k):
    """The k committed sweeps of the persistent chains (k x (L + 1) ops) run as ONE persistent dataflow program; same
    ops, same Philox sites as the emulation -> the same particles up to draws at rounding-level ties."""
    V = 30 if Hs[0] < 100 else 784
    cfg = make_cfg(V=V, Hs=Hs, n_particles=12 if V == 30 else 300, batch_size=10)
    eng, emu = _native.CudaDBM(cfg), OracleDBMbf16(cfg)
    init(cfg, (eng, emu), scale=0.3 if V == 30 else 0.03)
    X = batch(cfg, 10)
    for it in range(2):
        eng.val_metrics(X, k, 5, it), emu.val_metrics(X, k, 5, it)
        names = ['v'] + ['h' + ('' if i == 0 else '_%d' % i) for i in range(len(Hs))]
        ga, gb = eng.get_params(names), emu.get_params(names)
        for n in names:
            assert set(np.unique(ga[n])) <= {0.0, 1.0}, n
            assert np.mean(ga[n] != gb[n]) < 0.05, (n, np.mean(ga[n] != gb[n]))
    eng.close()


@pytest.mark.parametrize('M,N,K1,K2', [(200, 512, 784, 1024), (1024, 512, 784, 1024), (33, 18, 30, 11), (300, 130, 70, 257)])
def test_raw_two_pair_op_with_uniform_layouts(M, N, K1, K2):
    """The op shape the tensor-core DBM engine uses by default: two pairs, both with K-major A and MN-major B
    (x W_i + y (W_{i+1}^T) with the transposed shadow)."""
    rng = np.random.RandomState(M + N + 1)
    A1, B1 = rng.rand(M, K1), 0.1 * rng.randn(K1, N)
    A2, B2 = rng.rand(M, K2), 0.1 * rng.randn(K2, N)
    C = _native.debug_tc_gemm(A1, B1, a_t=False, b_t=True, A2=A2, B2=B2)
    r = lambda x: bf16_round(x).astype(np.float64)
    np.testing.assert_allclose(C, r(A1) @ r(B1) + r(A2) @ r(B2), atol=5e-2, rtol=1e-3)
