"""Training groups (bm_rbm_group_*, fit_many) without a GPU: the library's host code on the stand-in runtime with every kernel
interpreted on the CPU (tests/hostsim/build_group.sh adds the group kernels' restatement).  A member trained in a group must end
bit for bit where its own epoch ends; a step launches its program cuts and one update, whatever the number of members; the
members keep their solo plans on CTA pairs of their own; group programs have no dataflow hazard; refusals launch nothing."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_group.so')
OBJ = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
NAMES = ('W', 'vb', 'hb', 'dW', 'dvb', 'dhb', 'q_means')


@pytest.fixture(scope='module')
def sim():
    if not (os.path.isdir(OBJ) and any(f.endswith('.o') for f in os.listdir(OBJ))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_group.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(SIM)
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    lib.fakecuda_hazard_launches.restype = C.c_long
    lib.fakecuda_launches.restype = C.c_long
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    yield lib
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib


@pytest.fixture
def executing(sim):
    sim.fakecuda_reset()
    sim.fakecuda_set_execute(1)
    yield sim
    sim.fakecuda_set_execute(0)


def clean(sim):
    v, sk = sim.fakecuda_violation().decode(), sim.fakecuda_skipped().decode()
    assert v == '' and sk == '', (v, sk)


def member_cfg(g, V, H, gaussian, batch):
    cfg = dict(n_visible=V, n_hidden=H, v_kind='gaussian' if gaussian else 'bernoulli', h_kind='bernoulli', dtype='float32',
               compute='bf16', sample_v=bool(g % 2), sample_h=g % 3 != 2, l2=1e-4 * (g + 1), max_batch=batch,
               sparsity_target=0.1 + 0.05 * g, sparsity_cost=1e-3 * (g % 2), sparsity_damping=0.9, dbm_first=g == 1)
    if gaussian:
        cfg['sigma'] = np.linspace(0.8, 1.2 + 0.1 * g, V)
    return cfg


def make(g, V, H, gaussian, batch):
    from boltzmann_machines import _native
    e = _native.CudaRBM(member_cfg(g, V, H, gaussian, batch))
    rng = np.random.RandomState(100 + g)
    e.set_params({'W': (0.1 * rng.randn(V, H)).astype(np.float32), 'vb': (0.1 * rng.randn(V)).astype(np.float32),
                  'hb': (0.1 * rng.randn(H)).astype(np.float32)})
    return e


def data(G, N, V, kind, seed=0):
    rng = np.random.RandomState(seed)
    if kind == 'bytes':
        return (rng.rand(G, N, V) < 0.3).astype(np.float32)
    return rng.rand(G, N, V).astype(np.float32)


def epoch_args(G, k):
    return dict(lr=[0.05 + 0.01 * g for g in range(G)], momentum=[0.5 + 0.1 * g for g in range(G)], k=k,
                seed=[1234 + 7 * g for g in range(G)], tick0=[3 * g for g in range(G)], metrics=[('msre',)] * G,
                every=[1 + g % 2 for g in range(G)], iter0=[g for g in range(G)])


def solo_epoch(e, X, batch, a, g):
    return e.train_epoch(X, batch, a['lr'][g], a['momentum'][g], a['k'], a['seed'][g], a['tick0'][g],
                         metrics=a['metrics'][g], every=a['every'][g], iter0=a['iter0'][g])


@pytest.mark.parametrize('G,V,H,gaussian,kind,k', [(1, 20, 12, False, 'bytes', 1), (2, 37, 70, True, 'real', 2),
                                                   (5, 20, 12, False, 'real', 1), (5, 33, 40, True, 'bytes', 3)])
def test_members_end_where_their_own_epochs_end(executing, G, V, H, gaussian, kind, k):
    """W, vb, hb, dW, dvb, dhb, q_means and the MSRE of every reporting batch, bit for bit; 21 rows in batches of 8 (a short
    last batch), every member with its own seed, tick, lr, momentum, sigma, l2, sparsity, dbm_first and sampling flags"""
    from boltzmann_machines import _native
    batch, N = 8, 21
    X = data(G, N, V, kind)
    a = epoch_args(G, k)
    solo = [make(g, V, H, gaussian, batch) for g in range(G)]
    want = []
    for g, e in enumerate(solo):
        Xg = e.pin(X[g])
        want.append(solo_epoch(e, Xg, batch, a, g))
        e.unpin(Xg)
    members = [make(g, V, H, gaussian, batch) for g in range(G)]
    grp = _native.CudaRBMGroup(members)
    P = grp.pin(list(X))
    got = grp.train_epoch(P, batch, **a)
    grp.unpin(P)
    clean(executing)
    for g in range(G):
        w, m = solo[g].get_params(NAMES), members[g].get_params(NAMES)
        for n in NAMES:
            np.testing.assert_array_equal(m[n], w[n], err_msg='member {0}: {1}'.format(g, n))
        assert got[g] == want[g] and len(got[g]['msre']) > 0, g
    grp.close()


def per_step_launches(sim, G, k, steps=3, V=20, H=12, batch=8):
    from boltzmann_machines import _native
    members = [make(g, V, H, False, batch) for g in range(G)]
    grp = _native.CudaRBMGroup(members)
    X = data(G, steps * batch, V, 'bytes')
    P = grp.pin(list(X))
    a = epoch_args(G, k)
    a['metrics'] = [()] * G
    grp.train_epoch(P, batch, **a)                 # first epoch: descriptor uploads
    sim.fakecuda_reset()
    grp.train_epoch(P, batch, **a)
    counts = {n: sim.fakecuda_launches(n.encode()) / steps for n in ('', 'tc_program_kernel', 'cd_tail_group_kernel',
                                                                       'group_input_kernel')}
    grp.unpin(P)
    grp.close()
    return counts


def test_launches_per_step_do_not_grow_with_the_group(sim):
    """one program launch per cut of TC_PROGRAM_OPS ops (whole members), one update launch, one input conversion; nothing else"""
    one, five = per_step_launches(sim, 1, 1), per_step_launches(sim, 5, 1)
    assert one == five == {'': 3, 'tc_program_kernel': 1, 'cd_tail_group_kernel': 1, 'group_input_kernel': 1}, (one, five)
    # CD-20: 2k + 3 = 43 ops per member (the statistics do not overlap the chain at this size): two members per launch
    cut = per_step_launches(sim, 5, 20)
    assert cut == {'': 5, 'tc_program_kernel': 3, 'cd_tail_group_kernel': 1, 'group_input_kernel': 1}, cut


def test_members_keep_their_solo_plans_on_pairs_of_their_own(executing):
    from boltzmann_machines import _native
    G, V, H, batch, k = 5, 300, 200, 48, 1
    X = data(G, batch, V, 'bytes')
    a = epoch_args(G, k)
    solo = make(0, V, H, False, batch)
    Xs = solo.pin(X[0])
    solo_epoch(solo, Xs, batch, a, 0)
    solo.unpin(Xs)
    want = solo.debug_tc_plan()
    members = [make(0, V, H, False, batch) for _ in range(G)]
    grp = _native.CudaRBMGroup(members)
    P = grp.pin(list(X))
    grp.train_epoch(P, batch, **a)
    grp.unpin(P)
    plans = [m.debug_tc_plan() for m in members]
    keys = ('mode', 'bn', 'm_groups', 'n_tiles', 'splits', 'follows_granules')
    chain = [i for i, r in enumerate(want) if r['pair_begin'] == 0 and r['pair_count'] < 66]
    assert chain, want
    ranges = []
    for plan in plans:
        assert [{q: r[q] for q in keys} for r in plan] == [{q: r[q] for q in keys} for r in want]
        assert len({r['launch'] for r in plan}) == 1
        mine = {(plan[i]['pair_begin'], plan[i]['pair_count']) for i in chain}
        assert len(mine) == 1
        ranges.append(mine.pop())
    ranges.sort()
    for (b0, c0), (b1, _) in zip(ranges, ranges[1:]):
        assert b0 + c0 <= b1, ranges
    assert ranges[-1][0] + ranges[-1][1] <= 66
    clean(executing)
    grp.close()


def test_group_programs_have_no_dataflow_hazard(executing):
    from boltzmann_machines import _native
    executing.fakecuda_set_hazards(2)
    try:
        G, V, H, batch = 3, 20, 12, 8
        for k in (1, 20):
            members = [make(g, V, H, False, batch) for g in range(G)]
            grp = _native.CudaRBMGroup(members)
            P = grp.pin(list(data(G, 2 * batch, V, 'real')))
            before = executing.fakecuda_hazard_launches()
            grp.train_epoch(P, batch, **epoch_args(G, k))
            assert executing.fakecuda_hazard_launches() - before >= 2
            grp.unpin(P)
            grp.close()
        clean(executing)
    finally:
        executing.fakecuda_set_hazards(1)


def test_refusals_launch_nothing(sim):
    from boltzmann_machines import _native
    sim.fakecuda_reset()
    base = make(0, 20, 12, False, 8)
    cases = [(dict(n_hidden=13), ValueError, 'n_hidden'), (dict(n_visible=21), ValueError, 'n_visible'),
             (dict(max_batch=9), ValueError, 'max_batch'), (dict(v_kind='gaussian', sigma=np.ones(20)), ValueError, 'v_kind'),
             (dict(h_kind='multinomial'), NotImplementedError, 'multinomial'),
             (dict(compute='fp32'), NotImplementedError, 'fp32'), (dict(dropout=0.5), NotImplementedError, 'dropout')]
    for change, exc, word in cases:
        cfg = dict(member_cfg(0, 20, 12, False, 8))
        cfg.update(change)
        other = _native.CudaRBM(cfg)
        if change.get('h_kind') == 'multinomial':      # both members multinomial: refused for the layer, not a mismatch
            members = [other, _native.CudaRBM(cfg)]
        elif exc is NotImplementedError:
            members = [other, other]
        else:
            members = [base, other]
        n = sim.fakecuda_launches(b'')
        with pytest.raises((RuntimeError, NotImplementedError)) as err:
            _native.CudaRBMGroup(members)
        assert isinstance(err.value, NotImplementedError) == (exc is NotImplementedError), (change, err.value)
        assert word in str(err.value), (change, err.value)
        assert sim.fakecuda_launches(b'') == n
    grp = _native.CudaRBMGroup([base])
    P = grp.pin([data(1, 8, 20, 'bytes')[0]])
    n = sim.fakecuda_launches(b'')
    with pytest.raises(NotImplementedError, match='43'):
        grp.train_epoch(P, 8, **epoch_args(1, 44))
    assert sim.fakecuda_launches(b'') == n
    grp.unpin(P)
    grp.close()


# ---- fit_many ------------------------------------------------------------------------------------------------------------
def models(path, G, **kw):
    from boltzmann_machines import GaussianRBM
    out = []
    for g in range(G):
        p = dict(n_visible=24, n_hidden=16, batch_size=8, max_epoch=2, n_gibbs_steps=1, learning_rate=[0.01, 0.005],
                 momentum=[0.5, 0.9], sample_v_states=True, sample_h_states=True, sparsity_cost=1e-3, dbm_first=True,
                 random_seed=9000 + g, verbose=False, model_path=os.path.join(path, str(g)) + '/',
                 metrics_config=dict(msre=True, pll=True, feg=True, train_metrics_every_iter=2, feg_every_epoch=1))
        p.update(kw)
        out.append(GaussianRBM(**p))
    return out


def read(path):
    out = {}
    for kind in ('train', 'val'):
        with open(os.path.join(path, 'logs', kind, 'scalars.jsonl')) as fh:
            out[kind] = [json.loads(line) for line in fh]
    return out


def test_fit_many_equals_sequential_fit(executing, tmp_path):
    from boltzmann_machines import fit_many
    G = 3
    rng = np.random.RandomState(5)
    Xs = [rng.randn(20, 24).astype(np.float32) for _ in range(G)]
    Xv = [rng.randn(9, 24).astype(np.float32) for _ in range(G)]
    a, b = models(str(tmp_path / 'solo'), G), models(str(tmp_path / 'group'), G)
    for m, X, V in zip(a, Xs, Xv):
        m.fit(X, V)
    fit_many(b, Xs, Xv)
    clean(executing)
    for g in range(G):
        sa, sb = a[g]._engine.get_params(), b[g]._engine.get_params()
        for n in sa:
            np.testing.assert_array_equal(sb[n], sa[n], err_msg=n)
        assert (a[g].iter_, a[g].epoch_, a[g]._tick) == (b[g].iter_, b[g].epoch_, b[g]._tick)
        pa, pb = str(tmp_path / 'solo' / str(g)), str(tmp_path / 'group' / str(g))
        assert read(pa) == read(pb)
        for f in ('model.npz', 'model-1.npz', 'model-2.npz'):
            with np.load(os.path.join(pa, f)) as za, np.load(os.path.join(pb, f)) as zb:
                for n in za.files:
                    np.testing.assert_array_equal(zb[n], za[n], err_msg=f + ':' + n)


def test_fit_many_refuses_mismatched_models(sim, tmp_path):
    from boltzmann_machines import fit_many, BernoulliRBM
    X = [np.zeros((8, 24), np.float32)] * 2
    for attr, value in (('n_hidden', 17), ('batch_size', 4), ('n_gibbs_steps', 2), ('max_epoch', 3)):
        ms = models(str(tmp_path), 2)
        ms[1] = models(str(tmp_path), 1, **{attr: value})[0]
        with pytest.raises(ValueError, match=attr):
            fit_many(ms, X)
    with pytest.raises(ValueError, match='class'):
        fit_many([models(str(tmp_path), 1)[0], BernoulliRBM(n_visible=24, n_hidden=16, batch_size=8, max_epoch=2)], X)
    with pytest.raises(NotImplementedError, match='dropout'):
        fit_many(models(str(tmp_path), 2, dropout=0.9), X)
