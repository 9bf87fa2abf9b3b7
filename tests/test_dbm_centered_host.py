"""Centered DBMs (DESIGN.md §5.8), checked without a GPU.

* The algebra: the rank-2 (+ rank-1) correction of the plain gradient is the centered products, for full and partial batches.
* Two independent restatements -- the engine's formulation (stored W, b) and a model kept in centered coordinates (W, a, o)
  with conditionals from E_c -- train 20 steps to the same (W, b).
* Flip equivariance (Melchior, Fischer & Wiskott, JMLR 2016): with exact expectations, the centered step commutes with
  x -> 1 - x of a layer; the plain step does not.
* The tensor-core engine's host code on the stand-in runtime (tests/hostsim, build_dbm_centered.sh): against the bf16
  emulation and against the float64 M-step on its own activations (PT, multinomial top layer, Gaussian visibles); zero offsets
  with offset_rate 0 are the plain step bit for bit; save / restore, queries and refusals.
"""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

from dbm_centered_oracle import (LiteralCentered, CenteredOracleDBMbf16, bias_name, centered_grads, centered_grads_direct,
                                 centered_mstep, check_replay, offset_name, replay_bounds, sfx)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_dbm_centered.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')


def make_cfg(Hs, V, M, B=8, **kw):
    L = len(Hs)
    cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
               n_particles=M, batch_size=B, max_mf_updates=4, mf_tol=1e-6, l2=1e-3, max_norm=1.2, sample_v=True,
               sample_h=[True] * L, sparsity_target=[0.2] * L, sparsity_cost=[0.05] * L, sparsity_damping=0.9)
    cfg.update(kw)
    return cfg


def params(cfg, scale=0.3, bias=0.3, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [cfg['n_visible']] + cfg['n_hiddens']
    d = {'vb': (bias * rng.randn(sizes[0])).astype(np.float32)}
    for i in range(len(cfg['n_hiddens'])):
        d['W' + sfx(i)] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + sfx(i)] = (bias * rng.randn(sizes[i + 1])).astype(np.float32)
    return d


# ---- 1. the algebra ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('L', [1, 2, 3])
@pytest.mark.parametrize('rows', [16, 11])
def test_rank2_correction_is_the_centered_products(L, rows):
    rng = np.random.RandomState(L * 100 + rows)
    sizes = [9, 7, 6, 5][:L + 1]
    N, M = 16, 13
    d = [rng.rand(rows, n) for n in sizes]
    p = [(rng.rand(M, n) < 0.5).astype(float) for n in sizes]
    o = [rng.rand(n) for n in sizes]
    for a, b in zip(centered_grads(d, p, o, N, M), centered_grads_direct(d, p, o, N, M)):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-13)


# ---- 2. two restatements ---------------------------------------------------------------------------------------------------
def _run_both(L, steps=20, seed=3):
    rng = np.random.RandomState(seed)
    sizes = [10, 8, 7, 6][:L + 1]
    cfg = dict(batch_size=12, n_particles=9, l2=1e-3, max_norm=0.9, n_hiddens=sizes[1:], sparsity_target=[0.2] * L,
               sparsity_cost=[0.05] * L, sparsity_damping=0.9)
    W = [0.4 * rng.randn(sizes[i], sizes[i + 1]) for i in range(L)]
    b = [0.3 * rng.randn(n) for n in sizes]
    D = (rng.rand(12 * 3 - 5, sizes[0]) < 0.35).astype(float)           # a partial last batch: 31 rows in batches of 12
    st = {'vb': b[0].copy(), 'dvb': np.zeros(sizes[0]), 'offsets_set': np.zeros(1)}
    for j in range(L + 1):
        st[offset_name(j)] = np.zeros(sizes[j])
    for i in range(L):
        st.update({'W' + sfx(i): W[i].copy(), 'dW' + sfx(i): np.zeros_like(W[i]), 'hb' + sfx(i): b[i + 1].copy(),
                   'dhb' + sfx(i): np.zeros(sizes[i + 1]), 'q_means' + sfx(i): np.zeros(sizes[i + 1]),
                   'mu_means' + sfx(i): np.zeros(sizes[i + 1])})
    lit = LiteralCentered(cfg, W, b, [np.zeros(n) for n in sizes])
    parts = [rng.rand(9, n) for n in sizes]                               # particle states, swept on each side
    parts_lit = [x.copy() for x in parts]
    for t in range(steps):
        lo = (t * 12) % 36
        X = D[lo:lo + 12]
        mom = 0.5 if t < 5 else 0.9
        u = [rng.rand(9, n) for n in sizes]

        def sweep(cond, x):
            x = [y.copy() for y in x]
            for j in list(range(1, L + 1)) + [0]:
                x[j] = (u[j] < cond(j, x)).astype(float)
            return x

        def cond_plain(j, x):
            z = st[bias_name(j)].copy()
            if j > 0:
                z = z + x[j - 1] @ st['W' + sfx(j - 1)]
            if j < L:
                z = z + x[j + 1] @ st['W' + sfx(j)].T
            return 1 / (1 + np.exp(-z))

        def mf(cond):
            mu = [X] + [np.full((len(X), n), 0.5) for n in sizes[1:]]
            for _ in range(6):
                for j in range(1, L + 1):
                    mu[j] = cond(j, mu)
            return mu

        d_e = mf(cond_plain)
        parts = sweep(cond_plain, parts)
        d_l = mf(lit.conditional)
        parts_lit = sweep(lit.conditional, parts_lit)
        centered_mstep(st, d_e, parts, cfg, 0.05, mom, 0.1)
        lit.step(d_l, parts_lit, 0.05, mom, 0.1, first=(t == 0))
    return st, lit


@pytest.mark.parametrize('L', [1, 2, 3])
def test_engine_formulation_equals_centered_coordinates(L):
    st, lit = _run_both(L)
    b = lit.stored_b()
    for i in range(L):
        np.testing.assert_allclose(st['W' + sfx(i)], lit.W[i], rtol=0, atol=1e-10)
    for j in range(L + 1):
        np.testing.assert_allclose(st[bias_name(j)], b[j], rtol=0, atol=1e-10)
        np.testing.assert_allclose(st[offset_name(j)], lit.o[j], rtol=0, atol=1e-12)
    assert np.max(np.abs(st['W'])) > 0.05                                # the runs moved the model


# ---- 3. flip equivariance ------------------------------------------------------------------------------------------------------
SIZES = (6, 5, 4)


def _states(n):
    return np.array(list(itertools.product([0., 1.], repeat=n)))


def _exact_moments(W, b, X):
    """data side: per row the exact posterior over (h1, h2) given v; model side: the exact joint.  First moments per layer
    and the pairwise moments of adjacent layers, as 'rows' of weights"""
    S = [_states(n) for n in SIZES]
    h = list(itertools.product(range(len(S[1])), range(len(S[2]))))
    H1 = np.array([S[1][a] for a, _ in h]); H2 = np.array([S[2][c] for _, c in h])
    negE_h = H1 @ b[1] + H2 @ b[2] + np.einsum('ki,ij,kj->k', H1, W[1], H2)
    # data: p(h | v) for each row
    data = []
    for x in X:
        le = negE_h + H1 @ (W[0].T @ x)
        w = np.exp(le - le.max()); w /= w.sum()
        data.append((x, w))
    V = S[0]
    lv = (V @ b[0])[:, None] + negE_h[None, :] + (V @ W[0]) @ H1.T
    pj = np.exp(lv - lv.max()); pj /= pj.sum()
    return data, (V, H1, H2, pj)


def _exact_step(W, b, o, X, lr, rate, centered, first):
    """one step with exact expectations (N = rows, M -> exact), no momentum, sparsity cost 0, max-norm; float64"""
    data, (V, H1, H2, pj) = _exact_moments(W, b, X)
    rows = len(X)
    Ed = [X.mean(0), sum(w @ H1 for _, w in data) / rows, sum(w @ H2 for _, w in data) / rows]
    Em = [pj.sum(1) @ V, pj.sum(0) @ H1, pj.sum(0) @ H2]
    Pd = [sum(np.outer(x, w @ H1) for x, w in data) / rows, sum(H1.T @ (w[:, None] * H2) for _, w in data) / rows]
    Pm = [V.T @ pj @ H1, H1.T @ (pj.sum(0)[:, None] * H2)]
    if centered and first:
        o = [e.copy() for e in Ed]
    if not centered:
        o = [np.zeros(n) for n in SIZES]
    from dbm_centered_oracle import coupling, max_norm
    c_old = coupling(W, o)
    s = [Ed[j] - Em[j] for j in range(3)]
    G = [Pd[i] - Pm[i] - np.outer(o[i], s[i + 1]) - np.outer(s[i], o[i + 1]) for i in range(2)]
    Wn = [max_norm(W[i] + lr * (G[i] - 1e-3 * W[i]), 0.8) for i in range(2)]
    bn = [b[j] + lr * s[j] for j in range(3)]
    c_new = coupling(Wn, o)
    bn = [bn[j] - (c_new[j] - c_old[j]) for j in range(3)]
    on = [(1 - rate) * o[j] + rate * Ed[j] for j in range(3)]
    return Wn, bn, on


def _flip(W, b, o, f):
    """the model of x' with x'_f = 1 - x_f: W_{f-1}, W_f and b_f negate, the neighbours' biases absorb W 1, o_f -> 1 - o_f"""
    W, b, o = [w.copy() for w in W], [x.copy() for x in b], [x.copy() for x in o]
    if f > 0:
        b[f - 1] = b[f - 1] + W[f - 1].sum(1)
        W[f - 1] = -W[f - 1]
    if f < 2:
        b[f + 1] = b[f + 1] + W[f].sum(0)
        W[f] = -W[f]
    b[f] = -b[f]
    o[f] = 1 - o[f]
    return W, b, o


@pytest.mark.parametrize('f', [0, 1])
def test_flip_equivariance(f):
    rng = np.random.RandomState(7 + f)
    W = [0.6 * rng.randn(SIZES[i], SIZES[i + 1]) for i in range(2)]
    b = [0.4 * rng.randn(n) for n in SIZES]
    o0 = [np.zeros(n) for n in SIZES]
    X = (rng.rand(10, SIZES[0]) < 0.3).astype(float)
    Xf = 1 - X if f == 0 else X
    errs = {}
    for centered in (True, False):
        # one step, then the step of the flipped model on the flipped data, compared in the flipped coordinates
        W1, b1, o1 = _exact_step(W, b, o0, X, 0.5, 0.1, centered, True)
        Wf, bf, of = _flip(W, b, o0 if not centered else [np.zeros(n) for n in SIZES], f)
        if f != 0:
            # a flipped hidden layer: its data means are 1 - the unflipped ones, which the first step's offsets pick up
            pass
        W2, b2, o2 = _exact_step(Wf, bf, of, Xf, 0.5, 0.1, centered, True)
        W1f, b1f, _ = _flip(W1, b1, o1, f)
        errs[centered] = max([np.max(np.abs(a - c)) for a, c in zip(W2, W1f)] + [np.max(np.abs(a - c)) for a, c in zip(b2, b1f)])
    assert errs[True] < 1e-12, errs
    assert errs[False] > 1e-3, errs


# ---- 4.-6. the engine's host code on the stand-in runtime ---------------------------------------------------------------------
@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_dbm_centered.sh')], stdout=subprocess.DEVNULL)
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


def engine(cfg, rate=0.05, centering=True):
    from boltzmann_machines import _native
    c = dict(cfg)
    if centering:
        c.update(centering=True, offset_rate=rate)
    return _native.CudaDBM(c)


OFFSET_NAMES = lambda L: ['v_offset'] + ['h_offset' + sfx(i) for i in range(L)] + ['offsets_set']


@pytest.mark.parametrize('Hs,V,M,rows', [([24], 37, 20, 6), ([19, 13], 29, 17, 4)])
def test_engine_matches_bf16_emulation(sim, Hs, V, M, rows):
    cfg = make_cfg(Hs, V, M, B=6)
    eng, emu = engine(cfg), CenteredOracleDBMbf16(cfg, 0.05)
    d = params(cfg)
    for e in (eng, emu):
        e.set_params(d)
        e.init_particles(4242)
    X = (np.random.RandomState(1).rand(6, V) < 0.4).astype(np.float32)
    for step in range(4):
        Xs = X if step < 3 else X[:rows]                  # the last batch is partial in the second case
        eng.train_step(Xs, lr=0.05, momentum=0.5, k=2, seed=99, tick=step)
        emu.train_step(Xs, lr=0.05, momentum=0.5, k=2, seed=99, tick=step)
        g, w = eng.get_params(), emu.get_params()
        for name in ('v', 'h', 'h_1'):
            if name in g:
                np.testing.assert_array_equal(g[name], w[name], err_msg='%s after step %d' % (name, step))
    assert g['offsets_set'][0] == 1
    for k in g:
        if k in w and k not in ('v', 'h', 'h_1'):
            np.testing.assert_allclose(g[k], w[k], rtol=2.0 ** -7, atol=2e-5, err_msg=k)
    clean(sim)


@pytest.mark.parametrize('case', ['L1', 'L2_ragged', 'pt3', 'multinomial_top', 'gaussian'])
def test_engine_mstep_against_float64(sim, case):
    """every step's update, first step included, against the float64 M-step on the step's own exported activations"""
    kw, Hs, V, M, betas = {}, [24], 37, 20, None
    if case == 'L2_ragged':
        Hs, V, M = [19, 13], 29, 17
    if case == 'pt3':
        Hs, V, M, betas = [19, 13], 29, 17, [1.0, 0.6, 0.3]
    if case == 'multinomial_top':
        Hs, kw = [19, 6], dict(h_kinds=['bernoulli', 'multinomial'], h_n_samples=[100., 3.], sparsity_cost=[0.05, 0.0])
    if case == 'gaussian':
        Hs, kw = [19, 13], dict(v_kind='gaussian', sigma=np.ones(V), sample_v=False)
    cfg = make_cfg(Hs, V, M, B=6, **kw)
    if betas:
        cfg['pt_betas'] = betas
    eng = engine(cfg)
    eng.set_params(params(cfg))
    eng.init_particles(11)
    rng = np.random.RandomState(2)
    for step in range(3):
        rows = 6 if step < 2 else 5
        X = (rng.randn(rows, V) if case == 'gaussian' else (rng.rand(rows, V) < 0.4)).astype(np.float32)
        before = eng.get_params()
        eng.train_step(X, lr=0.05, momentum=0.5, k=2, seed=3, tick=step)
        after = eng.get_params()
        from oracle.dbm_bf16 import _r
        check_replay(replay_bounds(before, after, X, _r(X), cfg, 0.05, 0.5, 0.05), after)
    clean(sim)


def test_zero_offsets_without_motion_are_the_plain_step(sim):
    cfg = make_cfg([19, 13], 29, 17, B=6)
    a, b = engine(cfg, rate=0.0), engine(cfg, centering=False)
    d = params(cfg)
    for e in (a, b):
        e.set_params(d)
        e.init_particles(5)
    a.set_params({'offsets_set': np.ones(1, np.float32)})          # offsets stay at 0: set, and moved at rate 0
    X = (np.random.RandomState(2).rand(6, 29) < 0.4).astype(np.float32)
    for step in range(3):
        for e in (a, b):
            e.train_step(X if step < 2 else X[:4], lr=0.05, momentum=0.5, k=2, seed=5, tick=step)
    ga, gb = a.get_params(), b.get_params()
    for k in gb:
        np.testing.assert_array_equal(ga[k], gb[k], err_msg=k)
    assert not np.any(ga['v_offset']) and not np.any(ga['h_offset_1'])
    clean(sim)


def test_saved_state_continues_bit_identically(sim):
    """model.npz holds engine.get_params() -- with the offsets and their flag -- and load_model restores it with set_params:
    a restored engine's next steps are those of the engine kept in memory; queries leave the offsets as they were"""
    cfg = make_cfg([19, 13], 29, 17, B=6)
    a = engine(cfg)
    a.set_params(params(cfg))
    a.init_particles(8)
    X = (np.random.RandomState(4).rand(6, 29) < 0.4).astype(np.float32)
    for t in range(3):
        a.train_step(X, lr=0.05, momentum=0.5, k=2, seed=13, tick=t)
    saved = a.get_params()
    assert set(OFFSET_NAMES(2)) <= set(saved) and saved['offsets_set'][0] == 1
    b = engine(cfg)
    b.set_params(saved)
    for t in range(3, 5):
        for e in (a, b):
            e.train_step(X, lr=0.05, momentum=0.5, k=2, seed=13, tick=t)
    ga, gb = a.get_params(), b.get_params()
    for k in ga:
        np.testing.assert_array_equal(ga[k], gb[k], err_msg=k)
    keep = b.get_params(OFFSET_NAMES(2))
    b.transform(X)
    b.reconstruct(X)
    b.sample_v(2, 3, 9)
    after = b.get_params(OFFSET_NAMES(2))
    for k in keep:
        np.testing.assert_array_equal(after[k], keep[k], err_msg=k)
    clean(sim)


def test_model_saves_and_restores_offsets(sim, tmp_path):
    """DBM(centering=True) from init()-only RBMs: params.json keeps centering / offset_rate, model.npz the offsets"""
    from boltzmann_machines import DBM
    from boltzmann_machines.rbm import BernoulliRBM
    X = (np.random.RandomState(0).rand(24, 12) < 0.4).astype(np.float32)
    rbms = [BernoulliRBM(n_visible=12, n_hidden=8, model_path=str(tmp_path / 'r1'), random_seed=1).init(),
            BernoulliRBM(n_visible=8, n_hidden=5, model_path=str(tmp_path / 'r2'), random_seed=2).init()]
    m = DBM(rbms, n_particles=8, batch_size=8, max_epoch=1, n_gibbs_steps=1, learning_rate=0.05,
            model_path=str(tmp_path / 'dbm'), random_seed=3, centering=True, offset_rate=0.1, train_metrics_every_iter=0)
    m.fit(X)
    mine = m.get_tf_params(scope='offsets')
    assert mine['offsets_set'][0] == 1 and np.any(mine['v_offset'])
    again = DBM.load_model(str(tmp_path / 'dbm'))
    assert again.centering and again.offset_rate == 0.1
    got = again.get_tf_params(scope='offsets')
    for k in mine:
        np.testing.assert_array_equal(got[k], mine[k], err_msg=k)
    clean(sim)


@pytest.mark.parametrize('change,exc,msg', [
    (dict(offset_rate=1.5), ValueError, 'offset_rate must lie in'),
    (dict(offset_rate=-0.1), ValueError, 'offset_rate must lie in'),
    (dict(compute='fp32'), NotImplementedError, 'centering runs on the tensor-core engine only'),
    (dict(dtype='float64'), NotImplementedError, 'centering runs on the tensor-core engine only'),
    (dict(n_classes=3), NotImplementedError, 'centering is not supported for classification'),
])
def test_engine_refusals(sim, change, exc, msg):
    cfg = make_cfg([24, 13], 29, 17)
    rate = change.pop('offset_rate', 0.05)
    cfg.update(change)
    with pytest.raises(exc, match=msg):
        engine(cfg, rate=rate)


def test_model_refusals():
    from boltzmann_machines import DBM, ClassificationDBM
    with pytest.raises(ValueError, match='offset_rate'):
        DBM(centering=True, offset_rate=2.0)
    with pytest.raises(NotImplementedError, match='centering'):
        DBM(centering=True, dtype='float64')
    with pytest.raises(NotImplementedError, match='centering'):
        ClassificationDBM(centering=True)
    m = DBM(centering=True, offset_rate=0.2)
    assert m.get_params()['centering'] is True and m.get_params()['offset_rate'] == 0.2
    m.n_layers_ = 2
    assert m._scopes()['offsets'] == ('v_offset', 'h_offset', 'h_offset_1', 'offsets_set')
    assert DBM()._scopes()['offsets'] == ()
