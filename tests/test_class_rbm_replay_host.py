"""The stage-by-stage replay of tests/class_rbm_replay.py on the bf16 emulation of the classification RBM as a stand-in
engine (SplitEmulation: sums in 64-row fp32 splits, split-K slices of the W gradient, bf16 shadows refreshed by the update).

The unmutated emulation passes every check at shapes with several row splits (rows 150: 64 + 64 + 22), several 128-column
blocks (H = 300), three split-K slices (s1 = 3 for 132 SMs), C = 17 (the kernels' 64-class template) and semi-supervised rows
at the split edges.  Each planted mutation must be rejected: the test prints which check saw it."""
import numpy as np
import pytest

import class_rbm_replay as R

SM = 132
V, H, C, ROWS = 40, 300, 17, 150


def params(rng, V_=V, H_=H, C_=C):
    p = {'W': 0.3 * rng.randn(V_, H_), 'U': 0.3 * rng.randn(C_, H_), 'vb': 0.1 * rng.randn(V_), 'hb': 0.1 * rng.randn(H_),
         'yb': 0.1 * rng.randn(C_)}
    p.update({'d' + k: np.zeros_like(v) for k, v in list(p.items())})
    return {k: v.astype(np.float32) for k, v in p.items()}


def labels(rng, rows, C_, unlabelled):
    y = rng.randint(0, C_, size=rows)
    if unlabelled:
        y[[63, 64, 127, 128]] = -1          # both sides of two split edges ...
        y[64:128] = -1                       # ... and one split wholly unlabelled
        y[rng.rand(rows) < 0.2] = -1
    return y


def two_steps(eng, cfg, k=1, unlabelled=True, seed=5, rows=ROWS, C_=C):
    """step 1 (lr 1, momentum 0: the momenta are the gradients), then step 2 without set_params (lr 0.3, momentum 0.5)"""
    rng = np.random.RandomState(7)
    eng.set_params(params(rng, cfg['n_visible'], cfg['n_hidden'], C_))
    for step, (lr, mom) in enumerate(((1.0, 0.0), (0.3, 0.5))):
        X = (rng.rand(rows, cfg['n_visible']) < 0.4).astype(np.float32)
        y = labels(rng, rows, C_, unlabelled)
        R.run_step(eng, cfg, X, y, lr, mom, k, seed, step, SM, 'cpu')


def cfg_of(alpha, beta, sample_v, sample_h, C_=C, l2=1e-3):
    return dict(n_visible=V, n_hidden=H, n_classes=C_, alpha=alpha, beta=beta, l2=l2, max_batch=ROWS, sample_v=sample_v,
                sample_h=sample_h)


MUTATED_CFG = cfg_of(1.0, 0.5, True, True)


@pytest.mark.parametrize('alpha,beta,sample_v,sample_h,C_,unlabelled', [
    (1.0, 0.5, True, True, 17, True), (0.0, 0.0, False, True, 17, False), (0.01, 0.0, False, True, 10, False),
    (0.0, 0.1, True, False, 2, True), (1.0, 0.0, False, False, 16, False), (0.01, 0.1, False, True, 64, True)])
def test_unmutated_emulation_passes(alpha, beta, sample_v, sample_h, C_, unlabelled):
    cfg = cfg_of(alpha, beta, sample_v, sample_h, C_)
    R.reset_report()
    two_steps(R.SplitEmulation(cfg, SM), cfg, unlabelled=unlabelled, C_=C_)
    print('accepted', cfg, R.REPORT)


@pytest.mark.parametrize('sample_h', [True, False])
def test_unmutated_emulation_passes_cd_prefixes(sample_h):
    cfg = cfg_of(1.0, 0.5, True, sample_h)
    R.reset_report()
    rng = np.random.RandomState(3)
    p = params(rng)
    X = (rng.rand(ROWS, V) < 0.4).astype(np.float32)
    R.check_prefixes(R.SplitEmulation(cfg, SM), cfg, p, X, labels(rng, ROWS, C, True), 4, 9, 2, SM, 'cpu')
    print('accepted prefixes', R.REPORT)


def test_split_arithmetic():
    assert R.split_k(V, H, ROWS, SM) == 3 and R.splits(ROWS) == 3
    assert R.split_k(784, 1024, 128, SM) == 2 and R.split_k(784, 1024, 4096, SM) == 4
    assert R.splits(4033) == 64 and 4033 - 63 * 64 == 1


@pytest.mark.parametrize('mutation', R.MUTATIONS)
def test_mutation_is_rejected(mutation):
    with pytest.raises(AssertionError) as e:
        two_steps(R.SplitEmulation(MUTATED_CFG, SM, mutation), MUTATED_CFG)
    print('rejected', mutation, '--', str(e.value).split('\n')[0][:160])
