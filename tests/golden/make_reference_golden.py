"""Golden vectors from the REFERENCE'S OWN RBM AND DBM CODE: tests/golden/reference_rbm_cases.json,
tests/golden/reference_dbm_cases.json.

Needs a checkout of yell/boltzmann-machines, named by the BM_REFERENCE_DIR environment variable:

    python tests/golden/make_reference_golden.py

yell/boltzmann-machines is imported unmodified from that checkout with `oracle/tf1shim.py` registered as
`tensorflow` (TensorFlow 1.3 itself cannot be installed here).  For every case below the reference's own
`BernoulliRBM/GaussianRBM/MultinomialRBM(...).fit(X, X_val)`, `.transform(X)`, `.get_tf_params(...)` and `.init()` run:
its graph construction (base_rbm.py:244-525), its fit loop (:533-655), its persistence round trip between public calls
(tf_model.py:10-40,117-162).  Every random op of the graph asks the provider below, which answers from the Philox
layout the oracle and the CUDA engine share (oracle/philox.py): draw site from the op's name scope, Gibbs index from
the `gibbs_step[_i]` scope (or the while_loop iteration), tick = index of the Session.run call inside the public call,
seed = the graph-level seed the reference sets from its own RNG (`tf.set_random_seed(model.make_random_seed())`).

What the golden file pins: the oracle's (and, on the GPU, the engine's) gradients, sparsity term, momentum updates,
metrics (MSRE, PLL with its batch-mean quirk, L2, free-energy gap), schedules, dropout, the Gaussian / Multinomial unit
types and the fixed / variable-length Gibbs chain AGAINST THE REFERENCE'S SOURCE executing those formulas.  What it
does not pin: TensorFlow's own random stream (substituted, see above) and TensorFlow's kernels (numpy here).
"""
import json
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import philox as P                      # noqa: E402
from oracle import tf1shim                          # noqa: E402
from oracle.rbm import multinomial_counts           # noqa: E402

FALLBACK_SEED = 0            # seed of public calls that do not reseed the graph (init, get_tf_params)


def gibbs_index(req):
    """(is_chain_step, t): t-th Gibbs step (1-based) from the `gibbs_step[_i]` scope or the while_loop iteration."""
    for part in req.scope.split('/'):
        if part == 'gibbs_step' or part.startswith('gibbs_step_'):
            if req.loop_iter is not None:
                return True, req.loop_iter + 1
            return True, (int(part.split('_')[-1]) if part != 'gibbs_step' else 0) + 1
    return False, 0


AIS = {'seed': None, 'k': 1, 'sites': [P.SITE_AIS_V, P.SITE_AIS_H2, P.SITE_AIS_H1]}     # set around DBM.log_Z: the mirror draws a dedicated AIS seed per call (dbm.py:701)


def dbm_provider(req, seed, tick, shape):
    """Random ops of the reference's DBM graph (dbm.py:362-383 particle initialisers, :385-427 Gibbs step,
    :641-648 sample_v, :660-736 AIS) -> the draw sites of oracle/dbm.py."""
    parts = req.scope.split('/')
    if parts[0] == 'negative_particles':            # layer.init(batch_size=n_particles); *_new buffers are never read
        leaf = req.name.split('/')[-1].split(':')[0]
        if leaf.endswith('_1'):
            return np.zeros(shape, dtype=req.dtype)
        idx = 0
        if len(parts) > 1:
            idx = 1 + (0 if parts[1] == 'h_particle' else int(parts[1].split('_')[-1]))
        ais_ops = [t for t in req.graph.by_name.values()
                   if getattr(t, 'random_kind', None) == 'bernoulli' and getattr(t, 'op_seed', None) is not None]
        assert len(ais_ops) == 1                     # Bernoulli(logits).sample(seed=self.make_random_seed()), dbm.py:701
        draw = P.normal_at if req.kind == 'normal' else P.uniform_at       # GaussianLayer.init multiplies by sigma itself
        return draw(shape[0], shape[1], int(ais_ops[0].op_seed), P.SITE_PARTICLE_INIT, idx, 0).astype(req.dtype)
    if 'annealed_importance_sampling' in parts:
        assert req.kind == 'bernoulli'
        p = np.asarray(req.args[0])
        if req.op_seed is not None:                  # x_0 ~ Ber(0.5)
            u = P.uniform_at(shape[0], shape[1], AIS['seed'], P.SITE_AIS_INIT, 0, 0)
            return (u < np.float32(0.5)).astype(np.int32)
        stack = req.loop_stack
        it, s = (0, stack[0]) if len(stack) == 1 else (stack[0] + 1, stack[1])
        # sample, sample_1, sample_2 in creation order: v, h2, x_hat -- those of them the model samples (dbm.py:669-684)
        leaf = req.name.split('/')[-1].split(':')[0]
        site = AIS['sites'][0 if leaf == 'sample' else int(leaf.split('_')[-1])]
        u = P.uniform_at(shape[0], shape[1], AIS['seed'], site, 0, it * AIS['k'] + s)
        return (u.astype(p.dtype) < p).astype(np.int32)
    assert 'gibbs_chain' in parts, (req.scope, req.kind)
    leaf = [q for q in parts if q.startswith('sample_')][-1]
    site = P.SITE_DBM_V if leaf.startswith('sample_v_hat') else P.SITE_DBM_H + int(leaf[len('sample_h'):].split('_')[0])
    p = np.asarray(req.args[0])
    if req.kind == 'normal_loc_scale':
        scale = np.asarray(req.args[1])
        return (p + scale * P.normal_at(shape[0], shape[1], seed, site, req.loop_iter + 1, tick).astype(p.dtype)).astype(p.dtype)
    assert req.kind == 'bernoulli', req.kind
    u = P.uniform_at(shape[0], shape[1], seed, site, req.loop_iter + 1, tick)
    return (u.astype(p.dtype) < p).astype(np.int32)


def provider(req):
    seed = req.graph_seed if req.graph_seed is not None else FALLBACK_SEED
    tick = req.run_index
    shape = tuple(int(s) for s in req.shape)
    top = req.scope.split('/')[0]
    if top in ('negative_particles', 'annealed_importance_sampling') or \
            (('gibbs_chain/while' in req.scope) and 'sample_h_given_v' not in req.scope and 'sample_v_given_h' not in req.scope):
        return dbm_provider(req, seed, tick, shape)
    if req.kind == 'normal':                        # W initialiser: tf.random_normal(..., seed=random_seed)
        assert req.scope.startswith('weights') and req.op_seed is not None, req.scope
        return P.tf_random_normal(shape, req.stddev, int(req.op_seed), np.dtype(req.dtype).name)
    if req.kind == 'dropout_uniform':
        return P.uniform_at(shape[0], shape[1], seed, P.SITE_DROPOUT, 0, tick)
    if req.kind == 'uniform_int':
        assert 'pseudo_loglik' in req.scope
        return P.site_words(shape[0], 1, seed, P.SITE_PLL, 0, tick)[:, 0]
    in_step, t = gibbs_index(req)
    if 'free_energy' in req.scope:                  # MultinomialRBM._free_energy: h_hat ~ Multinomial(M, uniform)
        assert req.kind == 'multinomial'
        leaf = [p for p in req.scope.split('/') if p.startswith('free_energy')][0]
        fe_idx = 2 if not req.scope.startswith('pseudo_loglik') else (0 if leaf == 'free_energy' else 1)
        K = shape[-1]
        probs = np.full((1, K), 1.0 / K, dtype=np.float32)
        return multinomial_counts(probs, int(req.total_count), seed, P.SITE_MULTINOMIAL_FE, fe_idx, tick)[0].astype(np.float32)
    if 'sample_h_given_v' in req.scope:
        site = P.SITE_H if in_step else P.SITE_H0
    elif 'sample_v_given_h' in req.scope:
        site = P.SITE_V
    else:
        raise AssertionError('unmapped random op: {0} {1}'.format(req.kind, req.name))
    rows, n = shape
    if req.kind == 'bernoulli':
        p = np.asarray(req.args[0])
        u = P.uniform_at(rows, n, seed, site, t, tick)
        return ((u < p) if p.dtype == np.float32 else (u.astype(np.float64) < p)).astype(np.int32)
    if req.kind == 'multinomial':                   # tf.multinomial is shift-invariant per row
        p = np.asarray(req.args[0], dtype=np.float64)
        probs = (p / p.sum(axis=1, keepdims=True)).astype(np.float32)
        return multinomial_counts(probs, int(req.total_count), seed, site, t, tick).astype(np.float32)
    if req.kind == 'normal_loc_scale':
        loc, scale = np.asarray(req.args[0]), np.asarray(req.args[1])
        return (loc + scale * P.normal_at(rows, n, seed, site, t, tick).astype(loc.dtype)).astype(loc.dtype)
    raise AssertionError(req.kind)


def cases():
    rng = np.random.RandomState(7)
    Xb = (rng.rand(40, 20) < 0.3).astype(np.float32)
    Xb_val = (rng.rand(16, 20) < 0.3).astype(np.float32)
    Xg = rng.randn(36, 16).astype(np.float32)
    Xg_val = rng.randn(12, 16).astype(np.float32)
    mc = dict(msre=True, pll=True, l2_loss=True, feg=True, train_metrics_every_iter=2, val_metrics_every_epoch=1,
              feg_every_epoch=2, n_batches_for_feg=3)
    W20 = (0.1 * rng.randn(20, 12)).astype(np.float32)
    out = []
    out.append(dict(name='bernoulli_cd1_schedules', cls='BernoulliRBM', X=Xb, X_val=Xb_val, transform_rows=10,
                    kw=dict(n_visible=20, n_hidden=12, W_init=W20, vb_init=-0.5, hb_init=0.1, n_gibbs_steps=1,
                            learning_rate=[0.05, 0.02], momentum=[0.5, 0.9], max_epoch=3, batch_size=8, l2=1e-3,
                            sparsity_target=0.2, sparsity_cost=0.05, sparsity_damping=0.8, random_seed=1337,
                            metrics_config=dict(mc), verbose=False, save_after_each_epoch=True)))
    out.append(dict(name='bernoulli_variable_k_dropout_sample_v', cls='BernoulliRBM', X=Xb, X_val=Xb_val, transform_rows=8,
                    kw=dict(n_visible=20, n_hidden=12, W_init=W20, n_gibbs_steps=[1, 2, 3], learning_rate=0.03,
                            momentum=0.7, max_epoch=3, batch_size=16, l2=1e-4, sample_v_states=True, dropout=0.8,
                            dbm_first=True, random_seed=42, metrics_config=dict(mc), verbose=False,
                            save_after_each_epoch=False)))
    out.append(dict(name='bernoulli_fixed_k3_means_only', cls='BernoulliRBM', X=Xb, X_val=None, transform_rows=8,
                    kw=dict(n_visible=20, n_hidden=12, W_init=W20, n_gibbs_steps=3, learning_rate=0.05, momentum=0.5,
                            max_epoch=2, batch_size=10, l2=0., sample_h_states=False, dbm_last=True, random_seed=5,
                            metrics_config=dict(msre=True, train_metrics_every_iter=1), verbose=False,
                            save_after_each_epoch=False)))
    out.append(dict(name='bernoulli_float64', cls='BernoulliRBM', X=Xb.astype(np.float64), X_val=Xb_val.astype(np.float64),
                    transform_rows=6,
                    kw=dict(n_visible=20, n_hidden=12, W_init=W20.astype(np.float64), n_gibbs_steps=2, learning_rate=0.05,
                            momentum=0.6, max_epoch=2, batch_size=8, l2=1e-3, sparsity_cost=0.01, random_seed=11,
                            dtype='float64', metrics_config=dict(mc), verbose=False, save_after_each_epoch=False)))
    out.append(dict(name='gaussian_sigma_vector', cls='GaussianRBM', X=Xg, X_val=Xg_val, transform_rows=9,
                    kw=dict(n_visible=16, n_hidden=10, W_init=(0.05 * rng.randn(16, 10)).astype(np.float32),
                            sigma=np.linspace(0.6, 1.4, 16).tolist(), n_gibbs_steps=1, learning_rate=2e-3, momentum=0.8,
                            max_epoch=3, batch_size=12, l2=1e-3, sample_v_states=True, random_seed=3,
                            metrics_config=dict(mc), verbose=False, save_after_each_epoch=False)))
    out.append(dict(name='multinomial_hidden', cls='MultinomialRBM', X=Xb, X_val=Xb_val, transform_rows=7,
                    kw=dict(n_visible=20, n_hidden=6, n_samples=10, W_init=(0.1 * rng.randn(20, 6)).astype(np.float32),
                            n_gibbs_steps=1, learning_rate=0.01, momentum=0.5, max_epoch=2, batch_size=8, l2=1e-3,
                            random_seed=9, metrics_config=dict(mc), verbose=False, save_after_each_epoch=False)))
    out.append(dict(name='bernoulli_resume_after_load_model', cls='BernoulliRBM', X=Xb, X_val=Xb_val, transform_rows=5,
                    resume_max_epoch=4,
                    kw=dict(n_visible=20, n_hidden=12, W_init=W20, n_gibbs_steps=[1, 1, 2], learning_rate=[0.05, 0.04, 0.03, 0.02],
                            momentum=[0.5, 0.6, 0.7], max_epoch=2, batch_size=10, l2=1e-3, sparsity_cost=0.02, random_seed=77,
                            metrics_config=dict(mc), verbose=False, save_after_each_epoch=True)))
    out.append(dict(name='bernoulli_init_from_another_rbm', cls='BernoulliRBM', X=Xb, X_val=None, transform_rows=5,
                    pre_kw=dict(n_visible=20, n_hidden=12, W_init=W20, n_gibbs_steps=1, learning_rate=0.05, momentum=0.5,
                                max_epoch=2, batch_size=10, l2=1e-3, random_seed=31, verbose=False, save_after_each_epoch=False),
                    kw=dict(n_visible=20, n_hidden=12, n_gibbs_steps=2, learning_rate=0.02, momentum=0.9, max_epoch=4,
                            batch_size=8, l2=1e-4, sparsity_cost=0.01, random_seed=32,
                            metrics_config=dict(msre=True, train_metrics_every_iter=3), verbose=False,
                            save_after_each_epoch=False)))
    # found by --fuzz: with no scalar metric enabled the reference still runs the session once per validation batch (an
    # empty fetch list is a tick of the public call) and still writes its train / validation summary events
    out.append(dict(name='bernoulli_no_scalar_metrics_feg_only', cls='BernoulliRBM', X=Xb, X_val=Xb_val, transform_rows=6,
                    kw=dict(n_visible=20, n_hidden=12, W_init=W20, n_gibbs_steps=[2, 1], learning_rate=0.04, momentum=0.6,
                            max_epoch=3, batch_size=12, l2=1e-4, sample_v_states=True, dropout=0.9, random_seed=2024,
                            metrics_config=dict(msre=False, pll=False, l2_loss=False, feg=True, train_metrics_every_iter=3,
                                                val_metrics_every_epoch=1, feg_every_epoch=2, n_batches_for_feg=2),
                            verbose=False, save_after_each_epoch=False)))
    out.append(dict(name='init_from_seed', cls='BernoulliRBM', X=None, X_val=None, transform_rows=0,
                    kw=dict(n_visible=20, n_hidden=12, W_init=0.01, vb_init=0.25, random_seed=1337, verbose=False)))
    return out


def fuzz_cases(n, seed):
    """Random public-API scenarios (same record format as `cases()`): the oracle and the host mirror are fuzzed against
    the reference's own source with them --
        python tests/golden/make_reference_golden.py --fuzz 40 --seed 1 --out /tmp/fuzz.json
        BM_GOLDEN_RBM_CASES=/tmp/fuzz.json python -m pytest tests/test_z_reference_golden.py -k public_api -m 'not gpu'
    (nothing is committed: a disagreement found this way becomes a named case in `cases()`)."""
    rng = np.random.RandomState(seed)
    pick = lambda xs: xs[rng.randint(len(xs))]
    out = []
    for i in range(n):
        cls = pick(['BernoulliRBM', 'BernoulliRBM', 'BernoulliRBM', 'GaussianRBM', 'MultinomialRBM'])
        dt = pick(['float32', 'float32', 'float32', 'float64'])
        V, H = int(rng.randint(6, 25)), int(rng.randint(3, 15))
        n_rows, n_val = int(rng.randint(17, 46)), int(pick([0, 9, 14]))
        epochs = int(rng.randint(1, 4))
        sched = lambda lo, hi: (float(rng.uniform(lo, hi)) if rng.rand() < 0.5 else
                                [float(rng.uniform(lo, hi)) for _ in range(int(rng.randint(1, epochs + 2)))])
        if cls == 'GaussianRBM':
            X = rng.randn(n_rows, V).astype(dt)
            X_val = rng.randn(n_val, V).astype(dt) if n_val else None
        else:
            X = (rng.rand(n_rows, V) < 0.3).astype(dt)
            X_val = (rng.rand(n_val, V) < 0.3).astype(dt) if n_val else None
        mc = dict(msre=bool(rng.rand() < 0.8), pll=bool(rng.rand() < 0.6), l2_loss=bool(rng.rand() < 0.5),
                  feg=bool(n_val and rng.rand() < 0.6), train_metrics_every_iter=int(rng.randint(1, 4)),
                  val_metrics_every_epoch=int(rng.randint(1, 3)), feg_every_epoch=int(rng.randint(1, 3)),
                  n_batches_for_feg=int(rng.randint(1, 4)))
        kw = dict(n_visible=V, n_hidden=H,
                  W_init=(0.1 * rng.randn(V, H)).astype(dt) if rng.rand() < 0.7 else float(rng.uniform(0.01, 0.1)),
                  vb_init=float(rng.uniform(-0.5, 0.5)), hb_init=float(rng.uniform(-0.3, 0.3)),
                  n_gibbs_steps=(int(rng.randint(1, 4)) if rng.rand() < 0.5 else
                                 [int(rng.randint(1, 4)) for _ in range(int(rng.randint(1, epochs + 2)))]),
                  learning_rate=sched(2e-3, 5e-2) if cls != 'GaussianRBM' else sched(5e-4, 3e-3),
                  momentum=sched(0.3, 0.9), max_epoch=epochs, batch_size=int(rng.randint(4, 17)),
                  l2=float(pick([0., 1e-4, 1e-3])), sparsity_target=float(rng.uniform(0.05, 0.3)),
                  sparsity_cost=float(pick([0., 0.01, 0.05])), sparsity_damping=float(rng.uniform(0.5, 0.95)),
                  sample_v_states=bool(rng.rand() < 0.5), sample_h_states=bool(rng.rand() < 0.7),
                  dropout=pick([None, None, 0.7, 0.9]), dbm_first=bool(rng.rand() < 0.25), dbm_last=bool(rng.rand() < 0.25),
                  random_seed=int(rng.randint(1, 10 ** 6)), dtype=dt, metrics_config=mc, verbose=False,
                  save_after_each_epoch=bool(rng.rand() < 0.5))
        if cls == 'GaussianRBM':
            kw['sigma'] = float(rng.uniform(0.6, 1.5)) if rng.rand() < 0.5 else rng.uniform(0.6, 1.5, size=V).tolist()
        if cls == 'MultinomialRBM':
            kw['n_samples'] = int(rng.randint(3, 12))
        case = dict(name='fuzz_{0}_{1}_{2}'.format(seed, i, cls), cls=cls, X=X, X_val=X_val,
                    transform_rows=int(rng.randint(1, n_rows)), kw=kw)
        r = rng.rand()
        if r < 0.2:                                  # load_model + more epochs in a "new process"
            case['resume_max_epoch'] = epochs + int(rng.randint(1, 3))
        elif r < 0.35 and isinstance(kw['W_init'], np.ndarray):      # init_from a briefly trained model of the same class
            pre = dict(kw)
            pre.update(max_epoch=1, random_seed=int(rng.randint(1, 10 ** 6)), metrics_config=dict(mc), save_after_each_epoch=False)
            case['pre_kw'] = pre
            case['kw'] = {k: v for k, v in kw.items() if k not in ('W_init', 'vb_init', 'hb_init')}
            if case['X_val'] is not None and rng.rand() < 0.5:
                case['X_val'] = None
        out.append(case)
    return out


def dbm_spec(variant):
    """(X, X_val, rbm_cls, rbm_kw, dbm_kw, with_ais) of the three committed variants."""
    rng = np.random.RandomState({'bernoulli_2layer': 21, 'gaussian_visible_2layer': 22, 'bernoulli_3layer': 23,
                                 'bernoulli_2layer_partial_sampling': 24}[variant])
    V = 16
    sizes = [V, 10, 6] if variant != 'bernoulli_3layer' else [V, 10, 8, 5]
    L = len(sizes) - 1
    if variant == 'gaussian_visible_2layer':
        X = rng.randn(24, V).astype(np.float32)
        X_val = rng.randn(16, V).astype(np.float32)
    else:
        X = (rng.rand(24, V) < 0.3).astype(np.float32)
        X_val = (rng.rand(16, V) < 0.3).astype(np.float32)
    rbm_cls, rbm_kw = [], []
    for i in range(L):
        kw = dict(n_visible=sizes[i], n_hidden=sizes[i + 1], W_init=(0.1 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32),
                  n_gibbs_steps=1 + (i % 2), learning_rate=0.05, momentum=0.5, max_epoch=2, batch_size=8, l2=1e-3,
                  dbm_first=(i == 0), dbm_last=(i == L - 1), random_seed=101 * (i + 1), verbose=False, save_after_each_epoch=False)
        cls = 'BernoulliRBM'
        if i == 0 and variant == 'gaussian_visible_2layer':
            cls = 'GaussianRBM'
            kw.update(sigma=np.linspace(0.7, 1.3, V).tolist(), learning_rate=5e-3, sample_v_states=True)
        rbm_cls.append(cls)
        rbm_kw.append(kw)
    dbm_kw = dict(n_particles=8, n_gibbs_steps=[1, 2], max_mf_updates=5, mf_tol=1e-5, learning_rate=[0.02, 0.01],
                  momentum=[0.5, 0.9], max_epoch=3, batch_size=8, l2=1e-4, max_norm=0.6, sample_v_states=True,
                  sample_h_states=[True] * L, sparsity_target=[0.2, 0.1, 0.15][:L], sparsity_cost=[1e-2, 5e-3, 2e-3][:L],
                  sparsity_damping=0.8, train_metrics_every_iter=2, val_metrics_every_epoch=1, verbose=False,
                  save_after_each_epoch=True, random_seed=303)
    if variant == 'gaussian_visible_2layer':
        dbm_kw.update(learning_rate=[2e-3, 1e-3], max_norm=1.5)
    if variant == 'bernoulli_2layer_partial_sampling':      # found by --fuzz: fewer sample ops in the AIS transition; no max-norm
        dbm_kw.update(sample_v_states=False, sample_h_states=[True, False], max_norm=np.inf, n_gibbs_steps=2, mf_tol=1e-2)
    return X, X_val, rbm_cls, rbm_kw, dbm_kw, variant.startswith('bernoulli_2layer')


def fuzz_dbm_spec(seed, i):
    """A random DBM scenario of the same shape (see fuzz_cases): 2 or 3 layers, binary or Gaussian visibles, random
    schedules / particle counts / mean-field limits / sparsity / max-norm / sampling flags."""
    rng = np.random.RandomState(100003 * seed + i)
    pick = lambda xs: xs[rng.randint(len(xs))]
    L = int(pick([2, 2, 3]))
    dt = pick(['float32', 'float32', 'float32', 'float64'])
    gaussian = bool(rng.rand() < 0.25)
    V = int(rng.randint(8, 20))
    sizes = [V] + [int(rng.randint(4, 12)) for _ in range(L)]
    # the reference's variational parameters are a [batch_size, H] variable: every batch it sees (training, validation,
    # the 16 / 8 rows of the queries) must be full
    dbm_batch = int(pick([4, 8]))
    n_rows, n_val = int(pick([16, 24, 32])), 16
    if gaussian:
        X, X_val = rng.randn(n_rows, V).astype(dt), rng.randn(n_val, V).astype(dt)
    else:
        X, X_val = (rng.rand(n_rows, V) < 0.3).astype(dt), (rng.rand(n_val, V) < 0.3).astype(dt)
    rbm_cls, rbm_kw = [], []
    for j in range(L):
        kw = dict(n_visible=sizes[j], n_hidden=sizes[j + 1], W_init=(0.1 * rng.randn(sizes[j], sizes[j + 1])).astype(dt), dtype=dt,
                  n_gibbs_steps=int(rng.randint(1, 3)), learning_rate=float(rng.uniform(0.01, 0.05)), momentum=float(rng.uniform(0.3, 0.9)),
                  max_epoch=int(rng.randint(1, 3)), batch_size=int(rng.randint(5, 13)), l2=float(pick([0., 1e-3])),
                  dbm_first=(j == 0), dbm_last=(j == L - 1), random_seed=int(rng.randint(1, 10 ** 6)), verbose=False,
                  save_after_each_epoch=False)
        cls = 'BernoulliRBM'
        if j == 0 and gaussian:
            cls = 'GaussianRBM'
            kw.update(sigma=rng.uniform(0.7, 1.3, size=V).tolist(), learning_rate=5e-3, sample_v_states=True)
        rbm_cls.append(cls)
        rbm_kw.append(kw)
    epochs = int(rng.randint(1, 4))
    sched = lambda lo, hi: (float(rng.uniform(lo, hi)) if rng.rand() < 0.5 else
                            [float(rng.uniform(lo, hi)) for _ in range(int(rng.randint(1, epochs + 2)))])
    dbm_kw = dict(n_particles=int(rng.randint(3, 13)),
                  n_gibbs_steps=(int(rng.randint(1, 4)) if rng.rand() < 0.5 else [int(rng.randint(1, 4)) for _ in range(int(rng.randint(1, epochs + 2)))]),
                  max_mf_updates=int(rng.randint(1, 8)), mf_tol=float(pick([1e-7, 1e-5, 1e-2])),
                  learning_rate=sched(1e-3, 2e-2) if not gaussian else sched(5e-4, 2e-3), momentum=sched(0.3, 0.9),
                  max_epoch=epochs, batch_size=dbm_batch, l2=float(pick([0., 1e-4])),
                  max_norm=float(pick([0.6, 1.5, np.inf])), sample_v_states=bool(rng.rand() < 0.7),
                  sample_h_states=[bool(rng.rand() < 0.8) for _ in range(L)],
                  sparsity_target=[float(rng.uniform(0.05, 0.3)) for _ in range(L)],
                  sparsity_cost=[float(pick([0., 1e-2, 5e-3])) for _ in range(L)], sparsity_damping=float(rng.uniform(0.5, 0.95)),
                  train_metrics_every_iter=int(rng.randint(1, 4)), val_metrics_every_epoch=int(rng.randint(1, 3)), verbose=False,
                  save_after_each_epoch=bool(rng.rand() < 0.5), random_seed=int(rng.randint(1, 10 ** 6)), dtype=dt)
    resume = epochs + int(rng.randint(1, 3)) if rng.rand() < 0.3 else None     # load_model + load_rbms + more epochs
    return X, X_val, rbm_cls, rbm_kw, dbm_kw, (L == 2 and not gaussian), resume


def run_dbm_case(ref, workdir, variant, spec=None):
    """Greedy pre-training of the RBM stack, then DBM.fit / transform / reconstruct / sample_v (/ log_proba / log_Z for
    the 2-layer binary model, the only one the reference implements them for) -- dbm_mnist.py's sequence in miniature --
    all through the reference's public API.  Variants: 2 binary layers; Gaussian visibles (dbm_cifar*.py); 3 layers."""
    spec = tuple(spec if spec is not None else dbm_spec(variant))
    X, X_val, rbm_cls, rbm_kw, dbm_kw, with_ais = spec[:6]
    resume_max_epoch = spec[6] if len(spec) > 6 else None
    L = len(rbm_kw)
    rbms, inp, Q = [], X, None
    for i in range(L):
        r = getattr(ref.rbm, rbm_cls[i])(model_path=os.path.join(workdir, variant, 'rbm%d' % i) + '/', **rbm_kw[i])
        r.fit(inp)
        if i < L - 1:
            inp = r.transform(inp)
            if i == 0:
                Q = inp
        rbms.append(r)
    dbm = ref.DBM(rbms=rbms, model_path=os.path.join(workdir, variant, 'dbm') + '/', **dbm_kw)
    log = {'train': [], 'val': []}
    for meth, key in (('_train_epoch', 'train'), ('_run_val_metrics', 'val')):
        orig = getattr(dbm, meth)

        def wrapped(*a, _orig=orig, _key=key, **k):
            r = _orig(*a, **k)
            log[_key].append([None if v is None else float(v) for v in r])
            return r
        setattr(dbm, meth, wrapped)
    dbm.fit(X, X_val)
    dbm_summaries = summaries_of(dbm)
    if resume_max_epoch:
        # what dbm_mnist.py does in a new process: DBM.load_model(path), load_rbms(rbms), then more epochs
        dbm = ref.DBM.load_model(os.path.join(workdir, variant, 'dbm') + '/')
        dbm.load_rbms(rbms)
        dbm.set_params(max_epoch=resume_max_epoch)
        for meth, key in (('_train_epoch', 'train'), ('_run_val_metrics', 'val')):
            orig = getattr(dbm, meth)

            def wrapped2(*a, _orig=orig, _key=key, **k):
                r = _orig(*a, **k)
                log[_key].append([None if v is None else float(v) for v in r])
                return r
            setattr(dbm, meth, wrapped2)
        dbm.fit(X, X_val)
    rec = {'summaries': dbm_summaries, 'variant': variant, 'rbm_cls': rbm_cls,
           'rbm_kw': [{k: (tolist(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items()} for kw in rbm_kw],
           'dbm_kw': {k: ('inf' if isinstance(v, float) and np.isinf(v) else v) for k, v in dbm_kw.items()}, 'X': tolist(X), 'X_val': tolist(X_val), 'Q': tolist(Q), 'log': log,
           'epoch_': int(dbm.epoch_), 'iter_': int(dbm.iter_), 'resume_max_epoch': resume_max_epoch}
    scopes = ('weights', 'grads_accumulators', 'variational_params', 'hidden_means_accumulators', 'negative_particles')
    rec['after_fit'] = {sc: {k: tolist(v) for k, v in dbm.get_tf_params(scope=sc).items()} for sc in scopes}
    rec['transform'] = tolist(dbm.transform(X[:16]))
    rec['reconstruct'] = tolist(dbm.reconstruct(X[:8]))
    rec['sample_v'] = tolist(dbm.sample_v(n_gibbs_steps=2))
    if with_ais:
        rec['log_proba'] = tolist(dbm.log_proba(X_val, log_Z=0.0))
        # the mirror's log_Z draws the call seed and then a dedicated AIS seed from the model's RNG
        peek = type(dbm._rng)(seed=None).set_state(json.loads(json.dumps(dbm._rng.get_state())))
        peek.randint(2 ** 31 - 1)
        AIS['seed'], AIS['k'] = int(peek.randint(2 ** 31 - 1)), 2
        AIS['sites'] = ([P.SITE_AIS_V] if dbm_kw['sample_v_states'] else []) + \
                       ([P.SITE_AIS_H2] if dbm_kw['sample_h_states'][1] else []) + ([P.SITE_AIS_H1] if dbm_kw['sample_h_states'][0] else [])
        log_mean, (log_low, log_high), values = dbm.log_Z(n_betas=20, n_runs=6, n_gibbs_steps=2)
        rec['log_Z'] = {'n_betas': 20, 'n_runs': 6, 'n_gibbs_steps': 2, 'log_mean': float(log_mean), 'log_low': float(log_low),
                        'log_high': float(log_high), 'values': tolist(values)}
    rec['after_queries'] = {sc: {k: tolist(v) for k, v in dbm.get_tf_params(scope=sc).items()}
                            for sc in ('weights', 'negative_particles')}
    return rec


def summaries_of(model):
    """What the reference handed to its TensorBoard writers during the last public call: the steps of the merged
    train summaries and the (step, {tag: value}) records of the validation writer (tf_model.py:110-115)."""
    val = []
    for step, proto in model._tf_val_writer.events:
        val.append([int(step), {v.tag: float(v.simple_value) for v in proto.value}])
    return {'train_steps': [int(step) for step, _ in model._tf_train_writer.events], 'val': val}


def tolist(a):
    return None if a is None else np.asarray(a).tolist()


def run_case(ref_rbm, case, workdir):
    cls = getattr(ref_rbm, case['cls'])
    kw = dict(case['kw'])
    kw['model_path'] = os.path.join(workdir, case['name']) + '/'
    model = cls(**kw)
    if case.get('pre_kw'):                           # momentum accumulators and weights carried over (base_rbm.py:657-678)
        pre_kw = dict(case['pre_kw'])
        pre_kw['model_path'] = os.path.join(workdir, case['name'] + '_pre') + '/'
        pre = cls(**pre_kw)
        pre.fit(case['X'])
        model.init_from(pre)
        # init_from also copies `initialized_` (base_rbm.py:675-678), after which the reference would try to restore a
        # graph that was never saved under the new model_path; a user has to clear the flag (the host mirror does so itself)
        model.initialized_ = False
    log = {'train': [], 'val': [], 'feg': []}
    for meth, key in (('_train_epoch', 'train'), ('_run_val_metrics', 'val'), ('_run_feg', 'feg')):
        orig = getattr(model, meth)

        def wrapped(*a, _orig=orig, _key=key, **k):
            r = _orig(*a, **k)
            log[_key].append(r if not isinstance(r, dict) else {m: (None if v is None else float(v)) for m, v in r.items()})
            return r
        setattr(model, meth, wrapped)
    rec = {'name': case['name'], 'cls': case['cls'], 'kw': {k: (tolist(v) if isinstance(v, np.ndarray) else v) for k, v in case['kw'].items()},
           'X': tolist(case['X']), 'X_val': tolist(case['X_val']), 'transform_rows': case['transform_rows'],
           'resume_max_epoch': case.get('resume_max_epoch'),
           'pre_kw': None if not case.get('pre_kw') else {k: (tolist(v) if isinstance(v, np.ndarray) else v) for k, v in case['pre_kw'].items()}}
    if case['X'] is None:
        model.init()
    else:
        model.fit(case['X'], case['X_val'])
        rec['summaries'] = summaries_of(model)
        if case.get('resume_max_epoch'):
            # a new process would do exactly this: load_model (params.json, random_state.json), more epochs
            model = cls.load_model(kw['model_path'])
            model.set_params(max_epoch=case['resume_max_epoch'])
            for meth, key in (('_train_epoch', 'train'), ('_run_val_metrics', 'val'), ('_run_feg', 'feg')):
                orig = getattr(model, meth)

                def wrapped2(*a, _orig=orig, _key=key, **k):
                    r = _orig(*a, **k)
                    log[_key].append(r if not isinstance(r, dict) else {m: (None if v is None else float(v)) for m, v in r.items()})
                    return r
                setattr(model, meth, wrapped2)
            model.fit(case['X'], case['X_val'])
            rec['summaries_resumed'] = summaries_of(model)
        rec['transform'] = tolist(model.transform(case['X'][:case['transform_rows']]))
    rec['weights'] = {k: tolist(v) for k, v in model.get_tf_params(scope='weights').items()}
    rec['grads_accumulators'] = {k: tolist(v) for k, v in model.get_tf_params(scope='grads_accumulators').items()}
    rec['log'] = {'train': log['train'], 'val': log['val'], 'feg': [float(v) for v in log['feg']]}
    rec['epoch_'], rec['iter_'] = int(model.epoch_), int(model.iter_)
    return rec


def write_layer_goldens(ref):
    """tests/golden/reference_layers.json: the reference's layers.py plug-ins (layers.py:39-89) evaluated on the shim --
    `activation(x, b)` of the three unit types in both dtypes and the shape / dtype of `init` -- for the host mirror's
    layers.py, which keeps that surface with numpy semantics."""
    tf = sys.modules['tensorflow']
    L = ref.layers
    rng = np.random.RandomState(11)
    recs = []
    for dt in ('float32', 'float64'):
        for name, make in (('BernoulliLayer', lambda n: L.BernoulliLayer(n_units=n, dtype=dt)),
                           ('MultinomialLayer', lambda n: L.MultinomialLayer(n_samples=7, n_units=n, dtype=dt)),
                           ('GaussianLayer', lambda n: L.GaussianLayer(sigma=np.linspace(0.5, 1.5, n), n_units=n, dtype=dt))):
            n = 6
            layer = make(n)
            x = (2.0 * rng.randn(5, n)).astype(dt)
            b = (0.5 * rng.randn(n)).astype(dt)
            saved = tf1shim.default_random_provider          # `init` draws: only its shape / dtype are recorded
            tf1shim.default_random_provider = lambda req: np.zeros(tuple(int(v) for v in req.shape), dtype=req.dtype)
            try:
                tf.reset_default_graph()                     # a graph takes its provider when it is created
                with tf.Session() as sess:
                    act = sess.run(layer.activation(tf.constant(x), tf.constant(b)))
                    init = sess.run(layer.init(batch_size=4, random_seed=5))
            finally:
                tf1shim.default_random_provider = saved
            recs.append({'cls': name, 'dtype': dt, 'x': x.tolist(), 'b': b.tolist(), 'activation': np.asarray(act).tolist(),
                         'activation_dtype': str(np.asarray(act).dtype), 'init_shape': list(np.asarray(init).shape),
                         'init_dtype': str(np.asarray(init).dtype)})
    path = os.path.join(HERE, 'reference_layers.json')
    with open(path, 'w') as fh:
        json.dump({'source': 'yell/boltzmann-machines boltzmann_machines/layers.py on oracle/tf1shim.py', 'cases': recs}, fh)
    print('wrote', path, len(recs), 'cases')


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument('--fuzz', type=int, default=0, help='write N random RBM scenarios instead of the committed goldens')
    ap.add_argument('--seed', type=int, default=1)
    ap.add_argument('--out', default=None)
    ap.add_argument('--fuzz-dbm', type=int, default=10)
    ap.add_argument('--out-dbm', default=None, help='also write --fuzz-dbm random DBM scenarios (BM_GOLDEN_DBM_CASES)')
    args = ap.parse_args()
    tf1shim.default_random_provider = provider
    tf1shim.install()
    REF_DIR = os.path.abspath(os.environ['BM_REFERENCE_DIR'])
    sys.path[:0] = [REF_DIR, os.path.join(REF_DIR, 'boltzmann_machines')]
    # rbm/rbm.py imports `layers` as a top-level module (rbm/env.py puts the package directory on sys.path) while dbm.py
    # imports `.layers`: two module objects, and DBM.log_Z / log_proba assert isinstance(layer, BernoulliLayer) across
    # them (dbm.py:927,948).  Serve the one module under both names -- an import alias, no source change.
    import importlib.abc
    import importlib.util

    class _LayersAlias(importlib.abc.MetaPathFinder, importlib.abc.Loader):
        def find_spec(self, name, path=None, target=None):
            if name == 'layers' and 'boltzmann_machines.layers' in sys.modules:
                return importlib.util.spec_from_loader(name, self)
            return None

        def create_module(self, spec):
            return sys.modules['boltzmann_machines.layers']

        def exec_module(self, module):
            pass
    sys.meta_path.insert(0, _LayersAlias())
    import boltzmann_machines as ref                     # the reference package, unmodified
    assert ref.__file__.startswith(REF_DIR + os.sep), ref.__file__
    if not args.fuzz:
        write_layer_goldens(ref)
    work = tempfile.mkdtemp(prefix='bm_golden_')
    cwd = os.getcwd()
    try:
        os.chdir(work)
        if args.fuzz:
            recs = []
            for c in fuzz_cases(args.fuzz, args.seed):
                try:
                    recs.append(run_case(ref.rbm, c, work))
                except Exception as e:           # a configuration the reference itself rejects is not a test case
                    print('  skipped', c['name'], type(e).__name__, str(e)[:120])
            with open(args.out, 'w') as fh:
                json.dump({'source': 'fuzz seed {0}'.format(args.seed), 'cases': recs}, fh)
            print('wrote', args.out, len(recs), 'cases')
            if args.out_dbm:
                drecs = {}
                for i in range(args.fuzz_dbm):
                    name = 'fuzz_{0}_{1}'.format(args.seed, i)
                    try:
                        drecs[name] = run_dbm_case(ref, work, name, spec=fuzz_dbm_spec(args.seed, i))
                    except Exception as e:
                        print('  skipped DBM', name, type(e).__name__, str(e)[:160])
                with open(args.out_dbm, 'w') as fh:
                    json.dump({'source': 'fuzz seed {0}'.format(args.seed), 'cases': drecs}, fh)
                print('wrote', args.out_dbm, len(drecs), 'DBM cases')
            return
        recs = [run_case(ref.rbm, c, work) for c in cases()]
        dbm_recs = {v: run_dbm_case(ref, work, v) for v in ('bernoulli_2layer', 'gaussian_visible_2layer', 'bernoulli_3layer',
                                                                  'bernoulli_2layer_partial_sampling')}
    finally:
        os.chdir(cwd)
        shutil.rmtree(work, ignore_errors=True)
    out = {'source': 'yell/boltzmann-machines (boltzmann_machines/rbm, layers.py, base/tf_model.py) executed unmodified on '
                     'oracle/tf1shim.py; random draws from the shared Philox layout (tests/golden/make_reference_golden.py)',
           'cases': recs}
    path = os.path.join(HERE, 'reference_rbm_cases.json')
    with open(path, 'w') as fh:
        json.dump(out, fh)
    print('wrote', path, os.path.getsize(path), 'bytes;', len(recs), 'cases')
    dpath = os.path.join(HERE, 'reference_dbm_cases.json')
    with open(dpath, 'w') as fh:
        json.dump({'source': out['source'].replace('boltzmann_machines/rbm, layers.py', 'boltzmann_machines/dbm.py, rbm, layers.py'),
                   'cases': dbm_recs}, fh)
    print('wrote', dpath, os.path.getsize(dpath), 'bytes')
    for v, r in dbm_recs.items():
        print(' ', v, 'log', r['log'], 'log_Z', r.get('log_Z', {}).get('log_mean'))
    for r in recs:
        print(' ', r['name'], 'iter_', r['iter_'], 'train log', r['log']['train'][-1:] , 'feg', r['log']['feg'])


if __name__ == '__main__':
    main()
