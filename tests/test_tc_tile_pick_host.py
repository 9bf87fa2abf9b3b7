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
