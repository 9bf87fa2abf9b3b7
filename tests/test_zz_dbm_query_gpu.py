"""The DBM queries -- transform, reconstruct, the two-layer bound log_proba, sample_v and the validation MSRE -- at the
benchmark's shapes on the tensor-core engine, the fp32 CUDA-core engine and a float64 model, against the float64 statements of
tests/dbm_query_replay.py (which states each query and derives its bounds).  Also: the tempered and centered models, the ragged
Gaussian model of the step replay, and the Python class's chunked queries at cfg4's shape replayed chunk by chunk with the stale
mu carried across chunks.

The benchmark-size cases are skipped on the host simulation; the 30-18-11 cases run there."""
import numpy as np
import pytest

import dbm_query_replay as Q
from boltzmann_machines import _native
from test_tc_kernel_exact_gpu import HOSTSIM
from test_zz_dbm_tc_replay_gpu import _bench, batch, cfg4_case, ragged_cfg, restored_state, sfx, small_cfg

pytestmark = pytest.mark.gpu
big = pytest.mark.skipif(HOSTSIM, reason='benchmark-size queries: hours on the interpreter')

SEED, TICK, LR, MOM = 0x5EED, 4, 2e-3, 0.5
J = 6                            # the E-step sweep checked: one chunk of 5 sweeps and one of 1 on the tensor-core engine
PREC_CFG = {'bf16': dict(compute='bf16'), 'fp32': dict(compute='fp32'), 'float64': dict(compute='fp32', dtype='float64')}


def saturated(cfg, d):
    """four units per hidden layer with mu exactly 1 and four exactly 0 on float32 models, so that the bound's entropy clip
    binds (binary visibles only: the Gaussian model keeps its state)"""
    if cfg.get('v_kind', 'bernoulli') == 'bernoulli':
        for i in range(len(cfg['n_hiddens'])):
            hb = d['hb' + sfx(i)].copy()
            hb[:4], hb[4:8] = 30.0, -120.0
            d['hb' + sfx(i)] = hb
    return d


def engine(cfg, **over):
    return _native.CudaDBM(dict(cfg, **over))


def with_engine(cfg, state, fn, **over):
    eng = engine(cfg, **over)
    try:
        eng.set_params(state)
        return fn(eng)
    finally:
        eng.close()


def mu_of(eng, L):
    return Q.mus(eng.get_params(['mu' + sfx(i) for i in range(L)]), L)


def run_queries(name, cfg, init, X, prec, queries, ks=(0, 1, 2), T=1):
    """every query in `queries` from the restored state `init` on the engine of arithmetic `prec`"""
    cfg = dict(cfg, **PREC_CFG[prec])
    what = '{0} {1}'.format(name, prec)
    L = len(cfg['n_hiddens'])
    m = Q.Model(cfg, init, prec)
    stale = [init['mu' + sfx(i)] for i in range(L)]
    qcfg = dict(max_mf_updates=J, mf_tol=-1.0)
    sweeps, out = {}, {}
    for j in (J - 1, J):
        def run(eng):
            out[j] = eng.transform(X)
            return mu_of(eng, L)
        sweeps[j] = with_engine(cfg, init, run, max_mf_updates=j, mf_tol=-1.0)
    Q.check_estep_sweep(m, X, sweeps[J], sweeps[J - 1], stale, what)
    Q.check_transform(out[J], sweeps[J], what)
    eng = engine(cfg, **qcfg)
    try:
        recon = None
        if 'reconstruct' in queries or 'val_metrics' in queries:
            eng.set_params(init)
            recon = eng.reconstruct(X)
            Q.check_same_mu(mu_of(eng, L), sweeps[J], what + ' reconstruct')
            Q.check_reconstruct(m, sweeps[J][0], recon, what)
        if 'log_proba' in queries:
            eng.set_params(init)
            lp = eng.log_proba(X)
            Q.check_same_mu(mu_of(eng, L), sweeps[J], what + ' log_proba')
            Q.check_bound(m, init, X, sweeps[J], lp, what)
            Q.bound_gap(m, init, X, sweeps[J], lp, name)
        if 'val_metrics' in queries:
            eng.set_params(init)
            got = eng.val_metrics(X, 1, SEED, TICK)
            assert got['n_mf_updates'] == J, (what, got)
            after_vm = eng.get_params()
            Q.check_same_mu(Q.mus(after_vm, L), sweeps[J], what + ' val_metrics')
            Q.check_msre(X, recon, got['msre'], what)
            eng.set_params(init)
            eng.train_step(X, LR, MOM, 1, SEED, TICK)
            Q.check_same_particles(eng.get_params(), after_vm, L, T, what + ': val_metrics against train_step')
        if 'sample_v' in queries:
            for k in ks:
                eng.set_params(init)
                eng.val_metrics(X, k, SEED, TICK)
                committed = eng.get_params()
                eng.set_params(init)
                v = eng.sample_v(k, SEED, TICK)
                Q.check_sample_v(m, committed, eng.get_params(), v, k, T, sample_v_chain(eng, k), what)
    finally:
        eng.close()


def sample_v_chain(eng, k):
    """{t: sweep t} of the last sample_v's uncommitted half, t = k - 1 (if >= 1) and k, read through the engine's hook"""
    names = ['v'] + ['h' + sfx(i) for i in range(eng.L)]
    chain = {}
    if k >= 1:
        chain[k] = {n: eng.debug_last_sample_v(n) for n in names}
    if k >= 2:
        chain[k - 1] = {n: eng.debug_last_sample_v(n + '_prev') for n in names}
    return chain


ALL = ('reconstruct', 'log_proba', 'val_metrics', 'sample_v')


def cfg4():
    c = cfg4_case()
    return c['cfg'], saturated(c['cfg'], c['init']), c['X']


@big
@pytest.mark.parametrize('prec', ['bf16', 'fp32', 'float64'])
def test_cfg4_queries(prec):
    cfg, init, X = cfg4()
    run_queries('cfg4', cfg, init, X, prec, ALL)


@big
def test_cfg4_ragged_rows():
    """1000 of 1024 rows: rows >= 1000 of mu stay as they were, every query on the rows present"""
    cfg, init, X = cfg4()
    run_queries('cfg4 1000 rows', cfg, init, X[:1000], 'bf16', ALL, ks=(1,))


@big
def test_cfg5_pcd_queries():
    cfg = _bench().dbm_cfg('bf16', [4096], 4096, 784, pcd_only=True)
    init = saturated(cfg, restored_state(cfg, 0.01, 31))
    run_queries('cfg5-pcd', cfg, init, batch(cfg, 4096, 3), 'bf16', ('reconstruct', 'sample_v'), ks=(1, 2))


@big
def test_ragged_gaussian_queries():
    cfg = ragged_cfg()
    init = restored_state(cfg, 0.05, 31)
    X = batch(cfg, 1000, 3)
    run_queries('ragged', cfg, init, X, 'bf16', ('reconstruct', 'sample_v'), ks=(1, 2))
    eng = engine(cfg)
    try:
        eng.set_params(init)
        with pytest.raises(RuntimeError, match='binary'):
            eng.log_proba(X)
    finally:
        eng.close()


@big
def test_tempered_sample_v():
    """T = 4: the committed sweeps run every slot and end with a swap round (also at k = 0), the uncommitted ones slot 0"""
    cfg = dict(_bench().dbm_cfg('bf16'), pt_betas=[1.0, 0.9, 0.8, 0.7])
    init = saturated(cfg, restored_state(cfg, 0.02, 31))
    rng = np.random.RandomState(8)
    init['v_pt'] = (rng.rand(3, cfg['n_particles'], cfg['n_visible']) < 0.3).astype(np.float32)
    for i, H in enumerate(cfg['n_hiddens']):
        init['h_pt' + sfx(i)] = (rng.rand(3, cfg['n_particles'], H) < 0.5).astype(np.float32)
    X = batch(cfg, 1024, 3)
    run_queries('tempered', cfg, init, X, 'bf16', ('val_metrics', 'sample_v'), ks=(0, 1, 2), T=4)


@big
def test_centered_queries():
    """the queries of a centered model read the plain (W, b), whatever the offsets"""
    cfg = dict(_bench().dbm_cfg('bf16'), centering=True, offset_rate=0.05)
    init = saturated(cfg, restored_state(cfg, 0.02, 31))
    X = batch(cfg, 1024, 3)
    rng = np.random.RandomState(9)
    init['v_offset'] = X.mean(axis=0).astype(np.float32)
    for i, H in enumerate(cfg['n_hiddens']):
        init['h_offset' + sfx(i)] = rng.uniform(0.1, 0.6, H).astype(np.float32)
    init['offsets_set'] = np.ones(1, np.float32)
    run_queries('centered', cfg, init, X, 'bf16', ('reconstruct', 'log_proba'))


@pytest.mark.parametrize('prec', ['bf16', 'fp32'])
def test_sample_v_hook_is_read_only(prec):
    """the hook adds no launch and changes no result: an engine that read every sweep through it takes the same next train_step
    as one that did not; it refuses after k = 0 and once a particle update has run since"""
    cfg = dict(small_cfg(), **PREC_CFG[prec])
    init = saturated(cfg, restored_state(cfg, 0.6, 31))
    X = batch(cfg, 10, 3)
    a, b = engine(cfg), engine(cfg)
    try:
        for e in (a, b):
            e.set_params(init)
            e.sample_v(2, SEED, TICK)
        n0 = a.ctx.launch_count()
        sample_v_chain(a, 2)
        assert a.ctx.launch_count() == n0
        for e in (a, b):
            e.train_step(X, LR, MOM, 1, SEED, TICK + 1)
        Q.check_unchanged(b.get_params(), a.get_params(), 'train_step after the sample_v hook')
        with pytest.raises(RuntimeError, match='sample_v_debug'):
            a.debug_last_sample_v('v')
        a.sample_v(0, SEED, TICK)
        with pytest.raises(RuntimeError, match='sample_v_debug'):
            a.debug_last_sample_v('v')
        a.sample_v(1, SEED, TICK)
        a.debug_last_sample_v('h_1')
        with pytest.raises(RuntimeError, match='committed particles'):
            a.debug_last_sample_v('v_prev')
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize('prec', ['bf16', 'fp32', 'float64'])
def test_small_queries(prec):
    """30-18-11, batch 10, 12 particles: every query, and 7 of 10 rows (also on the host simulation)"""
    cfg = small_cfg()
    init = saturated(cfg, restored_state(cfg, 0.6, 31))
    X = batch(cfg, 10, 3)
    run_queries('small', cfg, init, X, prec, ALL)
    run_queries('small 7 rows', cfg, init, X[:7], prec, ALL, ks=(1,))


# ---- the Python class: chunked queries --------------------------------------------------------------------------------------
def python_dbm(cfg, state, path):
    """a DBM of the Python class on an engine holding `state` (max_mf_updates = 1, mf_tol = -1: one sweep per chunk, reading
    the stale mu of the layer above)"""
    from boltzmann_machines import DBM
    L = len(cfg['n_hiddens'])
    m = DBM(rbms=None, n_particles=cfg['n_particles'], batch_size=cfg['batch_size'], max_mf_updates=1, mf_tol=-1.0,
            l2=cfg['l2'], max_norm=cfg['max_norm'], sample_v_states=True, sample_h_states=[True] * L,
            sparsity_target=list(cfg['sparsity_target']), sparsity_cost=list(cfg['sparsity_cost']), random_seed=11,
            model_path=str(path) + '/', pt_betas=cfg.get('pt_betas'), centering=cfg.get('centering', False),
            offset_rate=cfg.get('offset_rate', 0.01))
    m.n_layers_, m.n_visible_, m.n_hiddens_ = L, cfg['n_visible'], list(cfg['n_hiddens'])
    m.layers_ = dict(v=dict(kind='bernoulli'), h=[dict(kind='bernoulli') for _ in range(L)])
    m.initialized_ = True
    m._engine = m._make_engine()
    m._engine.set_params(state)
    return m


def test_python_chunked_queries(tmp_path):
    """transform, reconstruct and log_proba on 3 batches + 37 rows (cfg4's shape, a tempered and centered model; 3 x 10 + 7 rows
    of the 30-18-11 model on the host simulation), each chunk replayed on its own from the mu the chunk before left; afterwards
    every variable, particle, tempered slot and offset is as before, the next train_step is that of a model that ran no query,
    and sample_v restores or commits exactly its committed particles"""
    if HOSTSIM:
        cfg, B = small_cfg(), 10
        init = saturated(cfg, restored_state(cfg, 0.6, 31))
    else:
        cfg = dict(_bench().dbm_cfg('bf16'), pt_betas=[1.0, 0.8], centering=True, offset_rate=0.05)
        B = cfg['batch_size']
        init = saturated(cfg, restored_state(cfg, 0.02, 31))
        rng = np.random.RandomState(8)
        init['v_pt'] = (rng.rand(1, cfg['n_particles'], cfg['n_visible']) < 0.3).astype(np.float32)
        for i, H in enumerate(cfg['n_hiddens']):
            init['h_pt' + sfx(i)] = (rng.rand(1, cfg['n_particles'], H) < 0.5).astype(np.float32)
            init['h_offset' + sfx(i)] = rng.uniform(0.1, 0.6, H).astype(np.float32)
        init['v_offset'] = rng.uniform(0.05, 0.3, cfg['n_visible']).astype(np.float32)
        init['offsets_set'] = np.ones(1, np.float32)
    L = len(cfg['n_hiddens'])
    T = len(cfg.get('pt_betas') or [1.0])
    X = batch(cfg, 3 * B + (37 if B > 100 else 7), 5)
    model = python_dbm(cfg, init, tmp_path / 'q')
    twin = python_dbm(cfg, init, tmp_path / 'twin')
    try:
        before = model._engine.get_params()
        got = {'transform': model.transform(X), 'reconstruct': model.reconstruct(X), 'log_proba': model.log_proba(X, 0.0)}
        after = model._engine.get_params()
        for n, a in before.items():
            np.testing.assert_array_equal(after[n], a, err_msg='python queries moved ' + n)
        # the chunk-by-chunk replay: chunk c starts from the mu chunk c - 1 left
        qcfg = dict(cfg, max_mf_updates=1, mf_tol=-1.0)
        pm = Q.Model(qcfg, init, 'bf16')
        state = dict(init)
        for lo in range(0, len(X), B):
            Xc = X[lo:lo + B]
            what = 'python chunk at row {0}'.format(lo)
            eng = engine(qcfg)
            try:
                eng.set_params(state)
                t = eng.transform(Xc)
                mu = mu_of(eng, L)
            finally:
                eng.close()
            np.testing.assert_array_equal(got['transform'][lo:lo + B], t, err_msg=what + ': transform')
            Q.check_estep_sweep(pm, Xc, mu, [state['mu' + sfx(i)] for i in range(L)], [state['mu' + sfx(i)] for i in range(L)],
                                what)
            Q.check_reconstruct(pm, mu[0], got['reconstruct'][lo:lo + B], what)
            Q.check_bound(pm, init, Xc, mu, got['log_proba'][lo:lo + B], what)
            state = dict(state, **{'mu' + sfx(i): mu[i] for i in range(L)})
        # the next train_step is that of the twin, which ran no query
        Xt = batch(cfg, B, 6)
        for mm_ in (model, twin):
            mm_._engine.train_step(Xt, LR, MOM, 1, SEED, TICK)
        a, b = model._engine.get_params(), twin._engine.get_params()
        for n in a:
            np.testing.assert_array_equal(a[n], b[n], err_msg='train_step after the queries: ' + n)
        # sample_v: save_model=False leaves the model as it was; save_model=True exactly the committed particles
        before = model._engine.get_params()
        model.sample_v(n_gibbs_steps=2, save_model=False)
        after = model._engine.get_params()
        for n, v in before.items():
            np.testing.assert_array_equal(after[n], v, err_msg='sample_v(save_model=False) moved ' + n)
        seed = model._rng.get_state()
        model.sample_v(n_gibbs_steps=2, save_model=True)
        saved = model._engine.get_params()
        model._rng.set_state(seed)
        call_seed = model.make_random_seed()
        eng = engine(dict(cfg, max_mf_updates=1, mf_tol=-1.0))
        try:
            eng.set_params(before)
            eng.val_metrics(X[:B], 2, call_seed, 0)
            committed = eng.get_params()
        finally:
            eng.close()
        Q.check_same_particles(saved, committed, L, T, 'sample_v(save_model=True)', [n for n in Q.particle_names(L, T) if n != 'v'])
        for n, v in before.items():
            if n not in Q.particle_names(L, T):
                np.testing.assert_array_equal(saved[n], v, err_msg='sample_v(save_model=True) moved ' + n)
    finally:
        model.close()
        twin.close()


def test_report():
    """(runs last in this file) what the cases above checked"""
    print('\n' + Q.report_line('dbm-query'))
    assert Q.off_within_limit(), Q.REPORT
