"""Parallel tempering of the DBM's persistent chains, checked without a GPU.

* The float64 restatement (tests/dbm_pt_oracle.py) samples the right distributions: on models small enough to enumerate,
  every slot's empirical distribution of v matches the exact p_{beta_m}(v) (chi-square), and the same statistic rejects
  three deliberate errors of the restatement.
* The tensor-core engine's host code on the stand-in runtime (tests/hostsim, with build_dbm_pt.sh's restatement of the swap
  kernel) against the bf16 emulation: particles of every slot, swap counts and parameters after several steps.
* The ladder [1.0] is the engine without tempering, bit for bit; refusals carry their messages.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from dbm_pt_oracle import PTOracleDBM, PTOracleDBMbf16, exact_log_marginal_v

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_pt.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')


def make_cfg(Hs, V, M, B=8, dtype='float32', **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype=dtype, compute='bf16',
               n_particles=M, batch_size=B, max_mf_updates=4, mf_tol=1e-6, l2=1e-4, max_norm=3.0, sample_v=True,
               sample_h=[True] * L, sparsity_target=[0.2] * L, sparsity_cost=[0.01] * L, sparsity_damping=0.9)
    cfg.update(kw)
    return cfg


def params(cfg, scale=0.8, bias=0.6, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [cfg['n_visible']] + cfg['n_hiddens']
    d = {'vb': (bias * rng.randn(sizes[0])).astype(np.float32)}
    for i in range(len(cfg['n_hiddens'])):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = (bias * rng.randn(sizes[i + 1])).astype(np.float32)
    return d


# ---- the float64 restatement samples p_beta -----------------------------------------------------------------------------
CHI2_ROUNDS, CHI2_BURN, CHI2_THIN = 1500, 100, 10      # rounds of one sweep + one swap round; samples every 10th round after 100
CHI2_LIMIT = 2.0                                       # chi-square / degrees of freedom of a correct sampler stays below this


def chi2_per_slot(Hs, V, betas, mutation=None, seed=11, M=256):
    cfg = make_cfg(Hs, V, M, dtype='float64')
    o = PTOracleDBM(cfg, betas, mutation=mutation)
    d = params(cfg, scale=1.0, bias=1.0, seed=3)
    o.set_params(d)
    o.init_particles(5)
    L = len(Hs)
    W = [d['W' + ('' if i == 0 else '_%d' % i)] for i in range(L)]
    hb = [d['hb' + ('' if i == 0 else '_%d' % i)] for i in range(L)]
    pw = 2 ** np.arange(V)
    counts = np.zeros((len(betas), 2 ** V))
    for r in range(CHI2_ROUNDS):
        o.particles_update(1, True, seed, r)
        if r >= CHI2_BURN and r % CHI2_THIN == 0:
            for m in range(len(betas)):
                v = o.slot(m)[0]
                counts[m] += np.bincount((v @ pw).astype(np.int64), minlength=2 ** V)
    stats = []
    for m, b in enumerate(betas):
        _, logp = exact_log_marginal_v(W, hb, d['vb'], beta=b)
        n = counts[m].sum()
        expct = n * np.exp(logp)
        keep = expct >= 5
        obs, ex = np.append(counts[m][keep], counts[m][~keep].sum()), np.append(expct[keep], expct[~keep].sum())
        if ex[-1] < 5:
            obs, ex = obs[:-1], ex[:-1]
        stats.append(float(((obs - ex) ** 2 / ex).sum() / max(len(ex) - 1, 1)))
    return stats, o


@pytest.mark.parametrize('Hs,V', [([4], 6), ([4, 3], 5)])
def test_oracle_slots_sample_their_temperature(Hs, V):
    stats, o = chi2_per_slot(Hs, V, [1.0, 0.7, 0.45, 0.2])
    assert max(stats) < CHI2_LIMIT, stats
    acc = o.pt_accepted / np.maximum(o.pt_proposed, 1)
    assert np.all(acc > 0.05), acc


@pytest.mark.parametrize('mutation', ['sign', 'no_bias_energy', 'beta_weights_only'])
def test_chi2_rejects_oracle_mutations(mutation):
    stats, _ = chi2_per_slot([4], 6, [1.0, 0.7, 0.45, 0.2], mutation=mutation)
    assert max(stats) > 4 * CHI2_LIMIT, (mutation, stats)


# ---- the engine's host code on the stand-in runtime -----------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_pt.sh')], stdout=subprocess.DEVNULL)
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


def engine(cfg, betas):
    from boltzmann_machines import _native
    c = dict(cfg)
    if betas is not None:
        c['pt_betas'] = betas
    return _native.CudaDBM(c)


PARTICLES = ('v', 'h', 'h_1', 'v_pt', 'h_pt', 'h_pt_1')


@pytest.mark.parametrize('Hs,V,M', [([24], 37, 20), ([19, 13], 29, 17)])
def test_engine_matches_bf16_emulation(sim, Hs, V, M):
    betas = [1.0, 0.8, 0.55, 0.3, 0.0]
    cfg = make_cfg(Hs, V, M, B=6)
    eng, emu = engine(cfg, betas), PTOracleDBMbf16(cfg, betas)
    d = params(cfg, scale=0.3, bias=0.3)
    for e in (eng, emu):
        e.set_params(d)
        e.init_particles(4242)
    X = (np.random.RandomState(1).rand(6, V) < 0.4).astype(np.float32)
    for step in range(4):
        k = (1, 2, 8, 1)[step]                 # k = 8: 5 slots x 8 sweeps x (L + 1) ops are cut into launches between sweeps
        eng.train_step(X, lr=0.05, momentum=0.5, k=k, seed=99, tick=step)
        emu.train_step(X, lr=0.05, momentum=0.5, k=k, seed=99, tick=step)
        g, w = eng.get_params(), emu.get_params()
        for name in PARTICLES:
            if name in g:
                np.testing.assert_array_equal(g[name], w[name], err_msg='%s after step %d' % (name, step))
        acc, prop = eng.pt_counts()
        np.testing.assert_array_equal(acc, emu.pt_accepted, err_msg='swaps after step %d' % step)
        np.testing.assert_array_equal(prop, emu.pt_proposed)
    for k in g:
        if k not in PARTICLES:
            np.testing.assert_allclose(g[k], w[k], rtol=2.0 ** -7, atol=2e-5, err_msg=k)
    assert emu.pt_accepted.sum() > 0 and emu.pt_accepted.sum() < emu.pt_proposed.sum()
    # sample_v: the committed half tempers and swaps, the output is slot 0's
    got = eng.sample_v(2, 7, 10)
    want = emu.sample_v(2, 7, 10)
    np.testing.assert_allclose(got, want, rtol=2.0 ** -7, atol=2e-5)
    g, w = eng.get_params(), emu.get_params()
    for name in ('v_pt', 'h_pt'):
        np.testing.assert_array_equal(g[name], w[name], err_msg=name)
    clean(sim)


def test_single_temperature_is_the_plain_engine(sim):
    cfg = make_cfg([24, 13], 29, 17, B=6)
    a, b = engine(cfg, [1.0]), engine(cfg, None)
    d = params(cfg, scale=0.3, bias=0.3)
    for e in (a, b):
        e.set_params(d)
        e.init_particles(3)
    X = (np.random.RandomState(2).rand(6, 29) < 0.4).astype(np.float32)
    for step in range(3):
        for e in (a, b):
            e.train_step(X, lr=0.05, momentum=0.5, k=2, seed=5, tick=step)
    ga, gb = a.get_params(), b.get_params()
    assert set(ga) == set(gb)
    for k in ga:
        np.testing.assert_array_equal(ga[k], gb[k], err_msg=k)
    np.testing.assert_array_equal(a.sample_v(2, 5, 9), b.sample_v(2, 5, 9))
    clean(sim)


def test_tempered_slots_set_and_get(sim):
    cfg = make_cfg([24], 37, 20)
    e = engine(cfg, [1.0, 0.5, 0.25])
    v = (np.random.RandomState(0).rand(2, 20, 37) < 0.5).astype(np.float32)
    e.set_params({'v_pt': v})
    np.testing.assert_array_equal(e.get_params(['v_pt'])['v_pt'], v)
    with pytest.raises(RuntimeError, match='no tempered chains'):
        engine(cfg, None).pt_counts()


@pytest.mark.parametrize('change,betas,exc,msg', [
    (dict(), [0.9, 0.5], ValueError, 'betas\\[0\\] must be 1'),
    (dict(), [1.0, 0.5, 0.5], ValueError, 'decrease strictly'),
    (dict(), [1.0, -0.1], ValueError, 'decrease strictly'),
    (dict(sample_v=False), [1.0, 0.5], ValueError, 'sampled visible states'),
    (dict(sample_h=[True, False]), [1.0, 0.5], ValueError, 'sampled hidden states'),
    (dict(compute='fp32'), [1.0, 0.5], NotImplementedError, 'tensor-core engine only'),
    (dict(dtype='float64'), [1.0, 0.5], NotImplementedError, 'tensor-core engine only'),
    (dict(v_kind='gaussian', sigma=np.ones(29)), [1.0, 0.5], NotImplementedError, 'gaussian visibles'),
    (dict(h_kinds=['bernoulli', 'multinomial']), [1.0, 0.5], NotImplementedError, 'multinomial hidden layers'),
])
def test_engine_refusals(sim, change, betas, exc, msg):
    cfg = make_cfg([24, 13], 29, 17)
    cfg.update(change)
    with pytest.raises(exc, match=msg):
        engine(cfg, betas)


def test_dbm_constructor_refusals():
    from boltzmann_machines import DBM
    with pytest.raises(ValueError, match='pt_betas'):
        DBM(pt_betas=[1.0, 1.0])
    with pytest.raises(ValueError, match='pt_betas'):
        DBM(pt_betas=[0.5])
    with pytest.raises(ValueError, match='sampled states'):
        DBM(pt_betas=[1.0, 0.5], sample_v_states=False)
    with pytest.raises(NotImplementedError, match='float32'):
        DBM(pt_betas=[1.0, 0.5], dtype='float64')
    assert DBM(pt_betas=[1.0, 0.5]).pt_betas == [1.0, 0.5]


def test_saved_state_continues_bit_identically(sim):
    """model.npz holds engine.get_params() -- with the tempered slots -- and load_model restores it with set_params: a restored
    engine's next steps (swap pairs keyed by the tick) are those of the engine kept in memory"""
    cfg = make_cfg([19, 13], 29, 17, B=6)
    betas = [1.0, 0.6, 0.3]
    a = engine(cfg, betas)
    a.set_params(params(cfg, scale=0.3, bias=0.3))
    a.init_particles(8)
    X = (np.random.RandomState(4).rand(6, 29) < 0.4).astype(np.float32)
    for t in range(3):
        a.train_step(X, lr=0.05, momentum=0.5, k=2, seed=13, tick=t)
    saved = a.get_params()
    assert {'v_pt', 'h_pt', 'h_pt_1'} <= set(saved)
    b = engine(cfg, betas)
    b.set_params(saved)
    for t in range(3, 5):
        for e in (a, b):
            e.train_step(X, lr=0.05, momentum=0.5, k=2, seed=13, tick=t)
    ga, gb = a.get_params(), b.get_params()
    for k in ga:
        np.testing.assert_array_equal(ga[k], gb[k], err_msg=k)
    # the queries' snapshot (DBM._snapshot: variational parameters and negative particles) covers every slot
    from boltzmann_machines import DBM
    m = DBM(pt_betas=betas)
    m.n_layers_ = 2
    snap = m._scopes()['negative_particles']
    assert {'v', 'h', 'h_1', 'v_pt', 'h_pt', 'h_pt_1'} <= set(snap)
    keep = b.get_params(list(snap))
    b.transform(X)
    b.sample_v(2, 3, 9)
    b.set_params(keep)
    after = b.get_params(list(snap))
    for k in keep:
        np.testing.assert_array_equal(after[k], keep[k], err_msg=k)
    clean(sim)


def test_ladder_longer_than_one_program(sim):
    """46 slots of a one-layer model: a sweep is 92 ops, more than one program holds -- it is cut inside the sweep, and the
    slots outnumber nothing here but still share the grid's CTA pairs; every slot and swap count as the emulation"""
    betas = list(np.linspace(1.0, 0.0, 46))
    cfg = make_cfg([12], 10, 4, B=4)
    eng, emu = engine(cfg, betas), PTOracleDBMbf16(cfg, betas)
    d = params(cfg, scale=0.4, bias=0.3)
    for e in (eng, emu):
        e.set_params(d)
        e.init_particles(17)
    X = (np.random.RandomState(5).rand(4, 10) < 0.4).astype(np.float32)
    for step, k in enumerate((2, 1)):
        eng.train_step(X, lr=0.05, momentum=0.5, k=k, seed=21, tick=step)
        emu.train_step(X, lr=0.05, momentum=0.5, k=k, seed=21, tick=step)
    g, w = eng.get_params(), emu.get_params()
    for name in ('v', 'h', 'v_pt', 'h_pt'):
        np.testing.assert_array_equal(g[name], w[name], err_msg=name)
    acc, prop = eng.pt_counts()
    np.testing.assert_array_equal(acc, emu.pt_accepted)
    np.testing.assert_array_equal(prop, emu.pt_proposed)
    clean(sim)


def test_unrelated_create_errors_stay_runtime_errors(sim):
    """only the refusals of the tempering option become ValueError / NotImplementedError"""
    cfg = make_cfg([12], 10, 4, B=4, n_particles=0)
    with pytest.raises(RuntimeError, match='n_particles and batch_size must be positive') as got:
        engine(cfg, [1.0, 0.5])
    assert type(got.value) is RuntimeError
