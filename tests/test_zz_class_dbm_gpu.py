"""Classification DBMs on the H100 (csrc/bm_cdbm_tc.cuh, DESIGN.md §5.7) at cfg4's shape 784-512-1024 with 10 classes,
batch = particles = 1024.

- A batch labelled -1 throughout is the plain DBM with a multinomial top layer of 10 units (n_samples 1, sampled, sparsity
  cost 0), bit for bit, over several steps.
- One all-labelled and one mixed step replayed against float64 from the engine's own state: the labelled rows' label slots
  are exactly one-hot; the E-step's mu_1, mu_2 and label slots are the float64 statement's clamped E-step to 2e-2; every label particle is the categorical draw u < CDF at site 16 + L (Philox, word 0 of column block
  0 of the particle's row) from softmax(yb + h_L U^T) of the pre-update U, ambiguous only where u is within 2e-4 of a CDF
  step (the fp32 accumulation of the 1024-term logits); U and yb after the update equal the float64 momentum / l2 / max-norm update computed from the engine's mu_L, q(y),
  h_L and y, to 1e-5 of the largest term.
- predict_proba equals float64 softmax(yb + mu_L U^T) of the returned transform (U as the engine's bf16 shadow) to fp32
  rounding.
- A learning run from a BernoulliRBM and a ClassificationRBM pretrained on a seeded synthetic task, on the engine and on the
  float64 statement."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle():
    spec = importlib.util.spec_from_file_location('class_dbm_oracle', os.path.join(ROOT, 'tests', 'class_dbm_oracle.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def bf16(x):
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


V, HS, C, B, M = 784, [512, 1024], 10, 1024, 1024


def cfg4(**kw):
    cfg = dict(n_visible=V, n_hiddens=list(HS), v_kind='bernoulli', h_kinds=['bernoulli'] * 2, h_n_samples=[100.] * 2,
               dtype='float32', compute='bf16', n_particles=M, batch_size=B, max_mf_updates=10, mf_tol=1e-7, l2=1e-5,
               max_norm=4.0, sample_v=True, sample_h=[True] * 2, sparsity_target=[0.1] * 2, sparsity_cost=[0.] * 2,
               sparsity_damping=0.9, n_classes=C)
    cfg.update(kw)
    return cfg


def params(seed=0, scale=0.02):
    rng = np.random.RandomState(seed)
    sizes = [V] + HS
    d = {'vb': (0.1 * rng.randn(V)).astype(np.float32)}
    for i in range(2):
        s = '' if i == 0 else '_1'
        d['W' + s] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = (0.1 * rng.randn(sizes[i + 1])).astype(np.float32)
    d['U'] = (0.3 * rng.randn(C, HS[-1])).astype(np.float32)
    d['yb'] = (0.1 * rng.randn(C)).astype(np.float32)
    return d


def data(rows=B, seed=1):
    rng = np.random.RandomState(seed)
    protos = np.clip(rng.beta(0.5, 0.5, size=(C, V)), 0.05, 0.95)
    y = rng.randint(0, C, size=rows)
    return (rng.rand(rows, V) < protos[y]).astype(np.float32), y.astype(np.int32)


def test_unlabelled_batches_are_the_plain_dbm_bit_for_bit():
    from boltzmann_machines import _native
    mod = oracle()
    cfg = cfg4()
    eng, ref = _native.CudaDBM(cfg), _native.CudaDBM(mod.plain_cfg(cfg))
    d = params()
    eng.set_params(d)
    ref.set_params(mod.to_plain(d, 2))
    for e in (eng, ref):
        e.init_particles(5)
    for it in range(3):
        X, _ = data(seed=10 + it)
        ref.train_step(X, 0.01, 0.9, 1, 77, it)
        eng.train_step(X, 0.01, 0.9, 1, 77, it, labels=np.full(B, -1, np.int32))
    g, w = eng.get_params(), mod.from_plain(ref.get_params(), 2)
    assert sorted(g) == sorted(w)
    for k in g:
        np.testing.assert_array_equal(g[k], w[k], err_msg=k)
    eng.close(); ref.close()


def _uniform_col0(seed, site, t, tick, rows):
    from oracle import philox as P
    return P.uniform_at(rows, 1, seed, site, t, tick, 0)[:, 0].astype(np.float64)


@pytest.mark.parametrize('labelled', ['all', 'mixed'])
def test_one_step_replayed_against_float64(labelled):
    from boltzmann_machines import _native
    eng = _native.CudaDBM(cfg4())
    d = params(seed=3)
    eng.set_params(d)
    eng.init_particles(9)
    X, y = data(seed=4)
    if labelled == 'mixed':
        y[::2] = -1
    before = eng.get_params()
    lr, mom, seed, tick = 0.01, 0.9, 1234, 3
    eng.train_step(X, lr, mom, 1, seed, tick, labels=y)
    g = eng.get_params()
    # the E-step: labelled label slots exactly one-hot, unlabelled ones a distribution
    q = g['mu_y']
    on = y >= 0
    np.testing.assert_array_equal(q[on], np.eye(C, dtype=np.float32)[y[on]])
    if (~on).any():
        np.testing.assert_allclose(q[~on].sum(axis=1), 1, atol=2e-2)
    # the E-step's result against the float64 statement's clamped E-step from the same state (both stop at the same cap
    # of 10 sweeps or earlier at convergence): bf16 operands and activations keep every value within 2e-2
    ref = oracle().ClassDBM64(cfg4())
    ref.set_params(before)
    ref._labels = y
    ref.mean_field(X)
    for k in ('mu', 'mu_1', 'mu_2'):
        name = {'mu_2': 'mu_y'}.get(k, k)
        np.testing.assert_allclose(g[name][:B], ref.p[k][:B], atol=2e-2, err_msg=name)
    # the label draws: y ~ softmax(yb + h_L U^T) with the new h_L and the pre-update U, yb (bf16 shadow of U)
    hL, Y = g['h_1'].astype(np.float64), g['y']
    logits = hL @ bf16(before['U']).astype(np.float64).T + before['yb'].astype(np.float64)
    p = np.exp(logits - logits.max(axis=1, keepdims=True))
    p /= p.sum(axis=1, keepdims=True)
    cdf = np.cumsum(p, axis=1)
    u = _uniform_col0(seed, 16 + 2, 1, tick, M)
    pick = np.argmax(cdf > u[:, None], axis=1)
    assert np.all(Y.sum(axis=1) == 1)
    got = np.argmax(Y, axis=1)
    ambiguous = np.min(np.abs(cdf - u[:, None]), axis=1) < 2e-4      # fp32 logits of a 1024-term product
    bad = (got != pick) & ~ambiguous
    assert not bad.any(), np.nonzero(bad)[0][:10]
    # the update of U and yb from the engine's statistics, in float64
    mu = g['mu_1'][:B].astype(np.float64)
    qq = q[:B].astype(np.float64)
    G = (qq.T @ mu) / B - (Y.astype(np.float64).T @ hL) / M                    # [C, H_L]
    U0 = before['U'].astype(np.float64)
    dU = lr * (mom * before['dU'].astype(np.float64) + G - 1e-5 * U0)
    Un = U0 + dU
    norm = np.sqrt((Un ** 2).sum(axis=1, keepdims=True))                       # columns of W_{L+1} = U^T: rows of U
    Un = Un * np.minimum(norm, 4.0) / np.maximum(norm, 1e-8)
    scale = lr * (np.abs(qq.T) @ np.abs(mu) / B + np.abs(Y.T) @ np.abs(hL) / M).max()
    assert np.max(np.abs(g['U'] - Un)) <= 1e-5 * max(scale, 1e-3) + 1e-6
    dyb = lr * (mom * before['dyb'].astype(np.float64) + qq.sum(0) / B - Y.sum(0) / M)
    np.testing.assert_allclose(g['yb'], before['yb'] + dyb, atol=1e-6)
    eng.close()


def test_predict_proba_is_the_softmax_of_the_returned_transform():
    from boltzmann_machines import _native
    eng = _native.CudaDBM(cfg4())
    d = params(seed=6)
    eng.set_params(d)
    eng.init_particles(1)
    X, _ = data(rows=3000, seed=7)
    P, T = [], []
    for i in range(0, 3000, B):                 # both queries from the same E-step start (mu enters the first sweep)
        keep = eng.get_params(['mu', 'mu_1', 'mu_y'])
        P.append(eng.predict_proba(X[i:i + B]))
        eng.set_params(keep)
        T.append(eng.transform(X[i:i + B]))
        eng.set_params(keep)
    P, T = np.concatenate(P), np.concatenate(T)
    logits = bf16(T).astype(np.float64) @ bf16(d['U']).astype(np.float64).T + d['yb'].astype(np.float64)
    want = np.exp(logits - logits.max(axis=1, keepdims=True))
    want /= want.sum(axis=1, keepdims=True)
    np.testing.assert_allclose(P, want, rtol=1e-4, atol=1e-6)
    eng.close()


def _scores(P, y):
    P = np.asarray(P, dtype=np.float64)
    return float(np.mean(np.argmax(P, 1) == y)), float(-np.mean(np.log(np.maximum(P[np.arange(len(y)), y], 1e-30))))


def test_learning_run_against_the_float64_statement(tmp_path):
    """A BernoulliRBM 784-256 and a ClassificationRBM 256-128 (10 classes, on the first layer's means) pretrained on the
    synthetic task, composed into a ClassificationDBM, then two epochs with a quarter of the labels set to -1 -- once on the
    engine and once on the float64 statement (tests/class_dbm_oracle.py, ClassDBM64, on the CPU) from the same stack, data
    and seeds.  Bounds, chosen before any run: the engine's test accuracy within 3 points and its mean NLL within 0.05 nats
    of the statement's, and on both the NLL after training below the composed model's.  Measured on an H100 80GB HBM3 (700 W),
    test accuracy / mean NLL: ClassificationRBM 0.415 / 2.192; composed DBM 0.407 / 2.1924 on both; after two epochs engine
    0.597 / 2.1903, float64 statement 0.598 / 2.1903.  The weak pretraining (5 epochs each, lr 0.1 / 0.05) keeps every
    posterior close to uniform; the check is that the engine learns what the statement learns from the same stack."""
    from boltzmann_machines import BernoulliRBM, ClassificationRBM, ClassificationDBM
    from boltzmann_machines.base import set_engine_factory
    mod = oracle()
    X, y = data(rows=4000, seed=0)
    Xtr, ytr, Xte, yte = X[:3000], y[:3000], X[3000:], y[3000:]
    r1 = BernoulliRBM(n_visible=V, n_hidden=256, W_init=0.01, learning_rate=0.1, momentum=0.5, max_epoch=5, batch_size=100,
                      n_gibbs_steps=1, random_seed=1, verbose=False, model_path=str(tmp_path / 'r1') + '/')
    r1.fit(Xtr)
    r2 = ClassificationRBM(n_visible=256, n_hidden=128, n_classes=C, alpha=0.01, learning_rate=0.05, momentum=0.5,
                           max_epoch=5, batch_size=100, random_seed=2, verbose=False, model_path=str(tmp_path / 'r2') + '/')
    r2.fit(r1.transform(Xtr), ytr)
    crbm = _scores(r2.predict_proba(r1.transform(Xte)), yte)
    ysemi = ytr.copy()
    ysemi[::4] = -1
    res = {}
    for name in ('cuda', 'float64'):
        old = set_engine_factory('dbm', mod.factory) if name == 'float64' else None
        try:
            m = ClassificationDBM([r1, r2], n_particles=100, batch_size=100, max_epoch=2, n_gibbs_steps=1, max_mf_updates=10,
                                  learning_rate=0.001, momentum=0.9, random_seed=3, verbose=False,
                                  model_path=str(tmp_path / name) + '/', save_after_each_epoch=False)
            m.init()
            start = _scores(m.predict_proba(Xte), yte)
            m.fit(Xtr, ysemi)
            res[name] = (start, _scores(m.predict_proba(Xte), yte))
        finally:
            if name == 'float64':
                set_engine_factory('dbm', old)
    print('classification DBM learning run (accuracy, mean NLL): ClassificationRBM %s; composed DBM -> after 2 epochs: '
          'engine %s -> %s, float64 %s -> %s' % (crbm, res['cuda'][0], res['cuda'][1], res['float64'][0], res['float64'][1]))
    (c0, c1), (o0, o1) = res['cuda'], res['float64']
    assert abs(c1[0] - o1[0]) <= 0.03 and abs(c1[1] - o1[1]) <= 0.05, res
    assert c1[1] < c0[1] and o1[1] < o0[1], res
