"""Centered DBMs on the H100 (DESIGN.md §5.8).

* Every centered M-step -- the first (the offsets set from the batch) and the second (the moving average) -- replayed in float64
  from the step's own exported activations, at cfg4's shape, at the cfg5-pcd shape, on a ragged three-layer model with Gaussian
  visibles and a multinomial top layer, and on a ragged three-layer model with four tempered slots (the bounds:
  tests/dbm_centered_oracle.py::replay_bounds).
* Zero offsets with offset_rate 0 are the plain step at cfg4, bit for bit.
* Training from scratch on 4x4 bars-and-stripes and on its flip 1 - D: exact average log-likelihood of plain and centered
  16-16-8 DBMs over 5 seeds (tools/bench_dbm_centered.py prints the table), and AIS log Z of a trained centered model against
  the exact one.
"""
import itertools

import numpy as np
import pytest

from dbm_centered_oracle import check_replay, replay_bounds, sfx
from oracle.rbm import bf16_round

pytestmark = pytest.mark.gpu


def cfg_of(V, Hs, M, B=None, **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
               n_particles=M, batch_size=B or M, max_mf_updates=10, mf_tol=1e-7, l2=1e-5, max_norm=1.5, sample_v=True,
               sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[1e-4] * L, sparsity_damping=0.9,
               centering=True, offset_rate=0.05)
    cfg.update(kw)
    return cfg


def params(V, Hs, scale, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [V] + list(Hs)
    d = {'vb': (0.1 * rng.randn(V)).astype(np.float32)}
    for i in range(len(Hs)):
        d['W' + sfx(i)] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + sfx(i)] = (0.1 * rng.randn(sizes[i + 1])).astype(np.float32)
    return d


def engine(cfg):
    from boltzmann_machines import _native
    return _native.CudaDBM(cfg)


CASES = {
    'cfg4': (784, [512, 1024], 1024, 1024, {}, 0.02),
    'cfg5-pcd': (784, [4096], 4096, 4096, {}, 0.01),
    'ragged-gauss-mult': (301, [203, 77, 9], 130, 100,
                          dict(v_kind='gaussian', sigma=np.ones(301), sample_v=False, h_kinds=['bernoulli', 'bernoulli', 'multinomial'],
                               h_n_samples=[100., 100., 4.], sparsity_cost=[1e-4, 1e-4, 0.]), 0.05),
    'ragged-pt4': (301, [203, 77, 45], 130, 100, dict(pt_betas=[1.0, 0.75, 0.5, 0.25]), 0.05),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_centered_msteps_against_float64(case):
    V, Hs, M, B, kw, scale = CASES[case]
    cfg = cfg_of(V, Hs, M, B, **kw)
    eng = engine(cfg)
    eng.set_params(params(V, Hs, scale))
    eng.init_particles(7)
    rng = np.random.RandomState(1)
    worst = []
    for step in range(2):
        rows = B if step == 0 else B - 37                   # the second batch is partial
        if kw.get('v_kind') == 'gaussian':
            X = rng.randn(rows, V).astype(np.float32)
        else:
            X = (rng.rand(rows, V) < 0.13).astype(np.float32)
        before = eng.get_params()
        eng.train_step(X, lr=0.01, momentum=0.5 if step else 0.0, k=1, seed=5, tick=step)
        after = eng.get_params()
        assert after['offsets_set'][0] == 1
        worst += check_replay(replay_bounds(before, after, X, bf16_round(X), cfg, 0.01, 0.5 if step else 0.0, 0.05), after)
    print(case, 'largest |engine - float64| / bound:', max(w for _, w in worst))
    eng.close()


def test_zero_offsets_without_motion_are_the_plain_step_at_cfg4():
    V, Hs, M = 784, [512, 1024], 1024
    a = engine(cfg_of(V, Hs, M, offset_rate=0.0))
    b = engine(cfg_of(V, Hs, M, centering=False))
    d = params(V, Hs, 0.02)
    for e in (a, b):
        e.set_params(d)
        e.init_particles(3)
    a.set_params({'offsets_set': np.ones(1, np.float32)})
    X = (np.random.RandomState(2).rand(M, V) < 0.13).astype(np.float32)
    for step in range(2):
        for e in (a, b):
            e.train_step(X, lr=0.01, momentum=0.5, k=1, seed=9, tick=step)
    ga, gb = a.get_params(), b.get_params()
    for k in gb:
        np.testing.assert_array_equal(ga[k], gb[k], err_msg=k)
    a.close(); b.close()


# ---- training from scratch on bars and stripes -----------------------------------------------------------------------------
def bars_and_stripes():
    """the 30 distinct 4x4 bars-and-stripes images (each row or each column all on or all off), as [30, 16].  The set is
    closed under x -> 1 - x, so 1 - D holds the same images in another order"""
    out = set()
    for bits in itertools.product([0, 1], repeat=4):
        a = np.array(bits, dtype=np.float32)
        out.add(tuple(np.repeat(a[:, None], 4, 1).ravel()))
        out.add(tuple(np.repeat(a[None, :], 4, 0).ravel()))
    return np.array(sorted(out), dtype=np.float64)


def exact_log_likelihood(W0, W1, b0, b1, b2, X):
    """mean log p(x) of a binary v-h1-h2 DBM: h1 enumerated, v and h2 summed out analytically (float64)"""
    H1 = np.array(list(itertools.product([0., 1.], repeat=W0.shape[1])))
    sp = lambda z: np.logaddexp(0.0, z)
    top = sp(H1 @ W1 + b2).sum(1)
    logZ = np.logaddexp.reduce(H1 @ b1 + sp(H1 @ W0.T + b0).sum(1) + top)
    lp = [np.logaddexp.reduce(x @ b0 + H1 @ b1 + H1 @ (W0.T @ x) + top) for x in X]
    return float(np.mean(lp) - logZ), float(logZ)


def train_bas(data, centered, seed, tmp, epochs=300):
    from boltzmann_machines import DBM
    from boltzmann_machines.rbm import BernoulliRBM
    X = np.tile(data, (4, 1)).astype(np.float32)                        # 120 rows, 4 batches of 30 per epoch
    rbms = [BernoulliRBM(n_visible=16, n_hidden=16, model_path=str(tmp / 'r1'), random_seed=seed).init(),
            BernoulliRBM(n_visible=16, n_hidden=8, model_path=str(tmp / 'r2'), random_seed=seed + 100).init()]
    m = DBM(rbms, n_particles=100, batch_size=30, max_epoch=epochs, n_gibbs_steps=1, max_mf_updates=10, mf_tol=1e-7,
            learning_rate=0.05, momentum=0.5, model_path=str(tmp / 'dbm'), random_seed=seed, centering=centered,
            offset_rate=0.01, train_metrics_every_iter=0, save_after_each_epoch=False)
    vb, Ws, hbs = m._composed_init()
    ll0 = exact_log_likelihood(Ws[0].astype(np.float64), Ws[1].astype(np.float64), vb.astype(np.float64),
                               hbs[0].astype(np.float64), hbs[1].astype(np.float64), data)[0]
    m.fit(X)
    p = m.get_tf_params(scope='weights')
    ll, logZ = exact_log_likelihood(*(p[k].astype(np.float64) for k in ('W', 'W_1', 'vb', 'hb', 'hb_1')), data)
    return ll0, ll, logZ, m


SEEDS = (1, 2, 3, 4, 5)


def bas_table(tmp_path_factory):
    D = bars_and_stripes()
    out = {}
    for name, data in (('D', D), ('1-D', 1.0 - D)):
        for centered in (False, True):
            runs = [train_bas(data, centered, s, tmp_path_factory.mktemp('bas'))[:2] for s in SEEDS]
            out[(name, centered)] = (np.array([r[0] for r in runs]), np.array([r[1] for r in runs]))
    return out


def test_training_from_scratch_on_bars_and_stripes(tmp_path_factory):
    t = bas_table(tmp_path_factory)
    for (name, centered), (ll0, ll) in sorted(t.items()):
        print('%-4s %-8s initial %.3f  final %.3f +- %.3f  (%s)' % (name, 'centered' if centered else 'plain', ll0.mean(),
                                                                    ll.mean(), ll.std(), ' '.join('%.3f' % x for x in ll)))
        assert np.all(ll > ll0 + 1.0), (name, centered, ll0, ll)      # every run learns
    # measured on an H100 80GB HBM3 (700 W): plain -9.661 +- 0.126, centered -8.677 +- 0.111 nats on D and on 1 - D alike
    cP, cD, cF = t[('D', False)][1], t[('D', True)][1], t[('1-D', True)][1]
    spread = max(cP.std(), cD.std(), cF.std())
    assert cD.mean() > cP.mean() + 3 * spread, (cP, cD)
    # centering is flip invariant: the two data sets give the same distribution of results up to the seeds' spread
    assert abs(cD.mean() - cF.mean()) <= 4 * spread + 0.1, (cD, cF)


def test_ais_reads_the_stored_parameters(tmp_path):
    D = bars_and_stripes()
    _, _, logZ, m = train_bas(1.0 - D, True, 1, tmp_path, epochs=100)
    log_mean, _, _ = m.log_Z(n_betas=2000, n_runs=500, n_gibbs_steps=1)
    assert abs(log_mean - logZ) < 1.0, (log_mean, logZ)
