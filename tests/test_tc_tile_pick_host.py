"""The tile picker on the host simulation: the headline workload's ops (BernoulliRBM 784-1024, batch 4096, CD-k) are planned
at 256 columns on CTA pairs -- one unit per pair for a chain half-step instead of two at 128 columns -- and ops too small to
fill the GPU at that width keep narrower tiles."""
import numpy as np
import pytest

from test_hostsim import sim, clean          # noqa: F401  (module fixture: the library on the stand-in runtime)


def plan_of(M, N, K, a_t, b_t, outputs=('f32',), splits=1, n_pairs=1, **kw):
    from boltzmann_machines import _native
    A = np.zeros((K, M) if a_t else (M, K), np.float32)
    B = np.zeros((K, N) if b_t else (N, K), np.float32)
    pairs = [(A, B, a_t, b_t, False)] + ([(A, B, a_t, b_t, True)] if n_pairs == 2 else [])
    return _native.debug_tc_op(pairs, outputs=outputs, splits=splits, **kw)['plan']


@pytest.mark.parametrize('name,M,N,K,a_t,b_t,outputs,splits,n_pairs,units', [
    ('h', 4096, 1024, 784, False, True, ('mean', 'state'), 1, 1, 64),      # v -> h: W as MN-major B
    ('v', 4096, 784, 1024, False, False, ('mean',), 1, 1, 64),              # h -> v: W as K-major B
    ('dW', 786, 1024, 4096, True, True, ('f32',), 4, 2, 64),               # X^T h0 - v^T h: MN-major operands, split over K
])
def test_headline_ops_plan_256_columns(sim, name, M, N, K, a_t, b_t, outputs, splits, n_pairs, units):
    sim.fakecuda_reset()
    p = plan_of(M, N, K, a_t, b_t, outputs, splits, n_pairs,
                act='linear' if name == 'dW' else 'sigmoid', sample='bernoulli' if 'state' in outputs else None)
    assert (p['bn'], p['cluster'], p['units']) == (256, 2, units), p
    assert p['ctas'] == 2 * units
    clean(sim)


def test_small_op_keeps_narrow_tiles(sim):
    sim.fakecuda_reset()
    p = plan_of(256, 130, 64, False, False)
    assert p['bn'] == 64, p
    clean(sim)


def test_headline_program_plan(sim):
    """The program of one cfg2 training step, as the engine plans it (launches recorded, not interpreted): h0, five pairs of
    chain half-steps and the two statistics ops in one launch; every chain op 256 columns wide on the first 64 CTA pairs and
    following its producer granule by granule; the statistics split over K on all 66 pairs."""
    from boltzmann_machines import _native
    V, H, B, k = 784, 1024, 4096, 5
    sim.fakecuda_reset()
    sim.fakecuda_set_execute(0)
    eng = _native.CudaRBM(dict(n_visible=V, n_hidden=H, v_kind='bernoulli', h_kind='bernoulli', dtype='float32', compute='bf16',
                               l2=1e-5, sample_v=False, sample_h=True, max_batch=B))
    eng.init_normal_W(0.01, 1337)
    eng.train_step((np.random.RandomState(3).rand(B, V) < 0.13).astype(np.float32), 0.05, 0.5, k, 7, 0)
    plan = eng.debug_tc_plan()
    eng.close()
    chain = plan[:1 + 2 * k]
    modes = ['SIG_BERN_MEAN_STATE'] + ['SIG_MEAN', 'SIG_BERN_STATE'] * (k - 1) + ['SIG_MEAN', 'SIG_MEAN']
    assert [p['mode'] for p in chain] == modes, plan
    assert len(plan) == len(chain) + 2 and all(p['launch'] == 0 for p in plan), plan
    for i, p in enumerate(chain):
        assert (p['bn'], p['m_groups'], p['n_tiles'], p['splits']) == (256, 16, 4, 1), (i, p)
        assert (p['pair_begin'], p['pair_count'], p['follows_granules']) == (0, 64, i > 0), (i, p)
    for p in plan[len(chain):]:
        assert p['mode'] == 'RAW_F32' and p['splits'] > 1 and not p['follows_granules'], p
        assert (p['pair_begin'], p['pair_count']) == (0, 66), p
    clean(sim)
