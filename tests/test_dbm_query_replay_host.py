"""Negative controls of the DBM query replay (tests/test_zz_dbm_query_gpu.py): its checkers (tests/dbm_query_replay.py), fed the
bf16 emulation (oracle/dbm_bf16.py, with the tempered ladder of tests/dbm_pt_oracle.py) as a stand-in engine, accept the
emulation and reject each planted mutation wherever it is materially present.  NOT_PRESENT states where a mutation is below its
bound, and why."""
import functools

import numpy as np
import pytest

import dbm_query_replay as Q
from dbm_pt_oracle import PTOracleDBMbf16
from oracle import philox as P
from oracle.dbm_bf16 import _r
from test_zz_dbm_query_gpu import J, LR, MOM, SEED, TICK, sample_v_chain, saturated
from test_zz_dbm_tc_replay_gpu import _bench, batch, ragged_cfg, restored_state, sfx, small_cfg

f32 = np.float32


class StandIn(PTOracleDBMbf16):
    """the emulation as an engine: the bound and the MSRE summed in double as the engine's row kernels do, and one mutation"""

    def __init__(self, cfg, mutation=None):
        super(StandIn, self).__init__(cfg, cfg.get('pt_betas') or [1.0])
        self.mutation = mutation

    # E-step: the stale mu of a chunk, and the approximate pass (kept for 'recon-approx')
    def _hidden(self, i, below, above, sample, seed, site, t, tick, acc_scale=1., bias_scale=1.):
        if self.mutation == 'uncommitted-sampled' and getattr(self, '_uncommitted', False) and self.cfg.get('sample_h', [True])[i]:
            sample, seed, site, t = True, SEED, P.SITE_DBM_H + i, 99
        return super(StandIn, self)._hidden(i, below, above, sample, seed, site, t, tick, acc_scale, bias_scale)

    def mean_field(self, X):
        rows = X.shape[0]
        if self.mutation in ('chunk-zeros', 'chunk-approx'):
            for i in range(self.L):
                if self.mutation == 'chunk-zeros':
                    self.p['mu' + sfx(i)][:rows] = 0.
            if self.mutation == 'chunk-approx':
                below = _r(X)
                for i in range(self.L):
                    sc = 2. if (i == 0 or i < self.L - 1) else 1.
                    below = self._hidden(i, below, None, False, 0, 0, 0, 0, acc_scale=sc)
                    self.p['mu' + sfx(i)][:rows] = below
        self._approx = _r(self._hidden(0, _r(X), None, False, 0, 0, 0, 0, acc_scale=2.))
        return super(StandIn, self).mean_field(X)

    def reconstruction(self, rows):
        if self.mutation == 'recon-approx':
            return self._visible(self._approx[:rows], False, 0, 0, 0, 0)
        return super(StandIn, self).reconstruction(rows)

    def val_metrics(self, X, k, seed, tick):
        X = np.asarray(X, f32)
        rows = X.shape[0]
        n_mf = self.mean_field(X)
        self.particles_update(k, True, seed, tick)
        d = X.astype(np.float64) - self.reconstruction(rows).astype(np.float64)
        s = float(np.sum(d * d))
        n = d.size
        if self.mutation == 'msre-padded':            # over the padded leading dimension of the bf16 buffers
            n = rows * (-(-self.V // 64) * 64)
        return {'msre': s / n, 'n_mf_updates': float(n_mf)}

    def log_proba(self, X):
        X = np.asarray(X, f32)
        rows = X.shape[0]
        self.mean_field(X)
        mu0, mu1 = self.p['mu'][:rows], self.p['mu_1'][:rows]
        W0, W1 = (self.W(0), self.W(1)) if self.mutation == 'bound-fp32-W' else (self.Wb(0), self.Wb(1))
        t0 = (_r(X) @ W0).astype(f32)
        t1 = (mu1 @ W1 if self.mutation == 'bound-mu-swapped' else mu0 @ W1).astype(f32)
        w1 = mu0 if self.mutation == 'bound-mu-swapped' else mu1
        d = np.float64
        out = (t0.astype(d) * mu0).sum(axis=1) + (t1.astype(d) * w1).sum(axis=1)
        out += X.astype(d) @ self.p['vb'].astype(d) + mu0.astype(d) @ self.hb(0).astype(d) + mu1.astype(d) @ self.hb(1).astype(d)
        for m in (mu0, mu1):
            if self.mutation == 'bound-no-clip':
                s = m.astype(d)
            elif self.mutation == 'bound-clip-double':
                s = np.clip(m.astype(d), 1e-7, 1. - 1e-7)
            else:
                s = np.clip(m, f32(1e-7), f32(1. - 1e-7)).astype(d)
            with np.errstate(divide='ignore', invalid='ignore'):
                out += (-s * np.log(s) - (1. - s) * np.log(1. - s)).sum(axis=1)
        return out

    def sample_v(self, k, seed, tick):
        """k committed sweeps, then k uncommitted ones on a ping-pong of scratch (sweep t in slot t % 2), as the engine runs them"""
        start = (self.p['v'].copy(), [self.p['h' + sfx(i)].copy() for i in range(self.L)])
        self.particles_update(k, True, seed, tick)
        committed = (self.p['v'], [self.p['h' + sfx(i)] for i in range(self.L)])
        v, H = start if self.mutation == 'uncommitted-from-precommit' else committed
        if not hasattr(self, '_scratch'):
            self._scratch = {t: (np.zeros_like(self.p['v']), [np.zeros_like(h) for h in committed[1]]) for t in (0, 1)}
        self._uncommitted = True
        try:
            for s in range(int(k)):
                if s == 1 and self.mutation == 'uncommitted-second-skipped':
                    break
                if s >= 1 and self.mutation == 'uncommitted-second-reads-committed':
                    v, H = committed
                v, H = self.gibbs_step(v, H, True, False, seed, int(k) + s + 1, tick)
                self._scratch[(s + 1) % 2] = (v, H)
        finally:
            self._uncommitted = False
        if self.mutation == 'uncommitted-writes-h' and k > 0:
            for i in range(self.L):
                self.p['h' + sfx(i)] = H[i]
        self.p['v'] = v
        self._sv_k = int(k)
        return v.copy()

    def debug_last_sample_v(self, name):
        """the engine's hook: sweep k (or k - 1 with '_prev') from the scratch it ran on"""
        t = self._sv_k - (1 if name.endswith('_prev') else 0)
        v, H = self._scratch[t % 2]
        base = name[:-5] if name.endswith('_prev') else name
        return v.copy() if base == 'v' else H[[sfx(i) for i in range(self.L)].index(base[1:])].copy()


# ---- cases ---------------------------------------------------------------------------------------------------------------------
def square_cfg():
    return dict(small_cfg(), n_hiddens=[16, 16])


CFGS = {
    'cfg4': lambda: (_bench().dbm_cfg('bf16'), 0.02, 1024),
    'small': lambda: (small_cfg(), 0.6, 10),
    'square': lambda: (square_cfg(), 0.6, 10),
    'ragged': lambda: (ragged_cfg(), 0.05, 1000),
}


@functools.lru_cache(maxsize=None)
def case(name):
    cfg, scale, rows = CFGS[name]()
    return cfg, saturated(cfg, restored_state(cfg, scale, 31)), batch(cfg, rows, 3)


def standin(name, mutation=None, **over):
    cfg, init, _ = case(name)
    s = StandIn(dict(cfg, **over), mutation)
    s.set_params(init)
    return s


def mu_of(s):
    return [s.p['mu' + sfx(i)].copy() for i in range(s.L)]


# ---- each query through the checkers -------------------------------------------------------------------------------------------
def run_estep(name, mutation=None):
    cfg, init, X = case(name)
    sweeps = {}
    for j in (J - 1, J):
        s = standin(name, mutation, max_mf_updates=j, mf_tol=-1.0)
        out = s.transform(X)
        sweeps[j] = mu_of(s)
    m = Q.Model(cfg, init, 'bf16')
    Q.check_estep_sweep(m, X, sweeps[J], sweeps[J - 1], Q.mus(init, m.L), name)
    Q.check_transform(out, sweeps[J], name)


def run_reconstruct(name, mutation=None):
    cfg, init, X = case(name)
    s = standin(name, mutation, max_mf_updates=J, mf_tol=-1.0)
    rec = s.reconstruct(X)
    Q.check_reconstruct(Q.Model(cfg, init, 'bf16'), mu_of(s)[0], rec, name)


def run_bound(name, mutation=None):
    cfg, init, X = case(name)
    s = standin(name, mutation, max_mf_updates=J, mf_tol=-1.0)
    lp = s.log_proba(X)
    Q.check_bound(Q.Model(cfg, init, 'bf16'), init, X, mu_of(s), lp, name)


def run_val_metrics(name, mutation=None):
    cfg, init, X = case(name)
    s = standin(name, mutation, max_mf_updates=J, mf_tol=-1.0)
    got = s.val_metrics(X, 1, SEED, TICK)
    assert got['n_mf_updates'] == J
    after = s.get_params()
    r = standin(name, None, max_mf_updates=J, mf_tol=-1.0)
    rec = r.reconstruct(X)
    Q.check_same_mu(Q.mus(after, len(cfg['n_hiddens'])), mu_of(r), name)
    Q.check_msre(X, rec, got['msre'], name)
    t = standin(name, None, max_mf_updates=J, mf_tol=-1.0)
    t.train_step(X, LR, MOM, 1, SEED, TICK)
    Q.check_same_particles(t.get_params(), after, len(cfg['n_hiddens']), 1, name)


def run_sample_v(name, mutation=None):
    """k = 0, 1, 2 for the emulation; a mutation at k = 2 only, where the uncommitted half has a second sweep"""
    cfg, init, X = case(name)
    m = Q.Model(cfg, init, 'bf16')
    for k in ((2,) if mutation else (0, 1, 2)):
        c = standin(name)
        c.val_metrics(X, k, SEED, TICK)
        s = standin(name, mutation)
        v = s.sample_v(k, SEED, TICK)
        Q.check_sample_v(m, c.get_params(), s.get_params(), v, k, 1, sample_v_chain(s, k), name)


def run_chunks(name, mutation=None):
    """the chunked E-step of the Python queries: 3 batches + a ragged one, each from the mu the chunk before left (one sweep)"""
    cfg, init, _ = case(name)
    B = cfg['batch_size']
    X = batch(cfg, 3 * B + 7, 5)
    m = Q.Model(dict(cfg, max_mf_updates=1, mf_tol=-1.0), init, 'bf16')
    s = standin(name, mutation, max_mf_updates=1, mf_tol=-1.0)
    for lo in range(0, len(X), B):
        stale = mu_of(s)
        s.transform(X[lo:lo + B])
        Q.check_estep_sweep(m, X[lo:lo + B], mu_of(s), stale, stale, '{0} chunk at {1}'.format(name, lo))


def run_snapshot(name, mutation=None):
    """the Python class's sample_v(save_model=False) on a tempered stand-in leaves every variable as it was"""
    from boltzmann_machines import DBM
    from boltzmann_machines.base import set_engine_factory
    cfg, init, _ = case(name)
    cfg = dict(cfg, pt_betas=[1.0, 0.8])
    L = len(cfg['n_hiddens'])
    old = set_engine_factory('dbm', lambda c: StandIn(c))
    orig = DBM._snapshot
    if mutation == 'snapshot-no-tempered':
        DBM._snapshot = lambda self: self._engine.get_params(['mu' + sfx(i) for i in range(L)] + Q.particle_names(L, 1))
    try:
        dbm = DBM(rbms=None, n_particles=cfg['n_particles'], batch_size=cfg['batch_size'], sample_h_states=[True] * L,
                  sparsity_target=list(cfg['sparsity_target']), sparsity_cost=list(cfg['sparsity_cost']), random_seed=11,
                  pt_betas=cfg['pt_betas'])
        dbm.n_layers_, dbm.n_visible_, dbm.n_hiddens_ = L, cfg['n_visible'], list(cfg['n_hiddens'])
        dbm.layers_ = dict(v=dict(kind='bernoulli'), h=[dict(kind='bernoulli') for _ in range(L)])
        dbm.initialized_ = True
        dbm._engine = dbm._make_engine()
        rng = np.random.RandomState(8)
        slots = {'v_pt': (rng.rand(1, cfg['n_particles'], cfg['n_visible']) < 0.3).astype(f32)}
        for i, H in enumerate(cfg['n_hiddens']):
            slots['h_pt' + sfx(i)] = (rng.rand(1, cfg['n_particles'], H) < 0.5).astype(f32)
        dbm._engine.set_params(dict(init, **slots))
        before = dbm._engine.get_params()
        dbm.sample_v(n_gibbs_steps=1, save_model=False)
        Q.check_unchanged(before, dbm._engine.get_params(), name + ' sample_v(save_model=False)')
    finally:
        DBM._snapshot = orig
        set_engine_factory('dbm', old)


CHECKS = {'E-step': run_estep, 'reconstruct': run_reconstruct, 'log_proba': run_bound, 'val_metrics': run_val_metrics,
          'sample_v': run_sample_v, 'chunks': run_chunks, 'snapshot': run_snapshot}
ACCEPT = [('cfg4', c) for c in CHECKS] + [('small', c) for c in CHECKS] + [('square', 'log_proba'), ('ragged', 'reconstruct'),
                                                                            ('ragged', 'sample_v')]
MUTATIONS = {          # mutation: (the checker that must reject it, the cases where it is materially present)
    'bound-no-clip': ('log_proba', ('cfg4', 'small')),             # mu exactly 0 or 1: 0 log 0
    'bound-fp32-W': ('log_proba', ('small',)),
    'bound-mu-swapped': ('log_proba', ('square',)),                 # mu_1 W_1 weighted by mu_0
    'recon-approx': ('reconstruct', ('cfg4', 'small')),
    'chunk-zeros': ('chunks', ('cfg4', 'small')),
    'chunk-approx': ('chunks', ('cfg4', 'small')),
    'uncommitted-sampled': ('sample_v', ('cfg4', 'small')),
    'uncommitted-writes-h': ('sample_v', ('cfg4', 'small')),
    'uncommitted-from-precommit': ('sample_v', ('cfg4', 'small')),
    'uncommitted-second-skipped': ('sample_v', ('cfg4', 'small')),          # k = 2 returns the first sweep's means
    'uncommitted-second-reads-committed': ('sample_v', ('cfg4', 'small')),  # sweep 2 from the committed particles, not sweep 1
    'bound-clip-double': ('log_proba', ()),                                 # the entropy clip in double on a float32 model
    'msre-padded': ('val_metrics', ('cfg4', 'small')),
    'snapshot-no-tempered': ('snapshot', ('cfg4', 'small')),
}
NOT_PRESENT = {
    ('bound-fp32-W', 'cfg4'): 'not detected: bf16 rounding of W ~ N(0, 0.02^2) moves the bound by 0.0082 nats per row on average '
                              'and 0.025 at most (the reported gap), inside the rigorous accumulation bound of the 784- and '
                              '512-term t GEMMs (~0.23 nats per row)',
    ('bound-clip-double', 'cfg4'): 'not detected: at the 8 saturated units of a row the float32 and double clips differ by '
                                   '~2.5e-6 nats, far inside the bound (~0.23 nats per row)',
    ('bound-clip-double', 'small'): 'not detected: ~2.5e-6 nats per row against a bound of ~2.6e-4',
    ('bound-mu-swapped', 'cfg4'): 'H_0 != H_1: mu_1 W_1 does not exist; a row kernel that strides mu_1 by H_0 is caught on the GPU',
    ('bound-mu-swapped', 'small'): 'H_0 != H_1 (18, 11): mu_1 W_1 does not exist',
}


def test_not_present_list_is_complete():
    for m, (_, where) in MUTATIONS.items():
        for n in ('cfg4', 'small'):
            if n not in where:
                assert (m, n) in NOT_PRESENT, (m, n)


@pytest.mark.parametrize('name,check', ACCEPT)
def test_checker_accepts_the_emulation(name, check):
    CHECKS[check](name)


@pytest.mark.parametrize('mutation,name', [(m, n) for m, (_, where) in MUTATIONS.items() for n in where])
def test_checker_rejects_the_mutation(mutation, name):
    with pytest.raises(AssertionError):
        CHECKS[MUTATIONS[mutation][0]](name, mutation)
