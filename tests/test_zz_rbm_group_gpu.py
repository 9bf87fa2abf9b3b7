"""Training groups on the H100 (fit_many, csrc/bm_rbm_group.cu): every model trained in a group against a clone trained by its own
fit(), bit for bit in every weight, accumulator, scalars.jsonl line and checkpoint.

  (a) the CIFAR-10 recipe's patch RBMs (examples/dbm_cifar.py of the reference): 26 GaussianRBMs 192-300, batch 48, CD-1, sampled
      states, sparsity, dbm_first, a per-epoch momentum schedule; 2 epochs on seeded synthetic data
  (b) 20 BernoulliRBMs 784-500 at CD-3: more ops per step than one program launch holds, so a step is cut into several
  (c) one model

Dry run without a GPU: BM_HOSTSIM=1 python -m pytest tests/test_zz_rbm_group_gpu.py -m gpu -k single (the stand-in runtime with the
group kernels' restatement, tests/hostsim/build_group.sh; the large cases take long there)."""
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM = os.environ.get('BM_HOSTSIM') == '1'


@pytest.fixture(scope='module', autouse=True)
def _hostsim_with_the_group_kernels():
    if not HOSTSIM:
        yield
        return
    from boltzmann_machines import _native
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_group.sh')], stdout=subprocess.DEVNULL)
    lib = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim_group.so'))
    lib.fakecuda_set_execute(1)
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    yield
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib


def patch_models(path, G):
    from boltzmann_machines import GaussianRBM
    return [GaussianRBM(n_visible=192, n_hidden=300, W_init=0.001, vb_init=0., hb_init=0., n_gibbs_steps=1,
                        learning_rate=[0.0005] * 2, momentum=[0.5, 0.9], max_epoch=2, batch_size=48, l2=1e-3,
                        sample_v_states=True, sample_h_states=True, sparsity_cost=1e-3, sparsity_target=0.1,
                        dbm_first=True, metrics_config=dict(msre=True, feg=True, train_metrics_every_iter=20,
                                                            val_metrics_every_epoch=1, feg_every_epoch=1, n_batches_for_feg=4),
                        verbose=False, random_seed=9000 + g, model_path=os.path.join(path, 'rbm_%d' % g) + '/')
            for g in range(G)]


def bernoulli_models(path, G, k=3):
    from boltzmann_machines import BernoulliRBM
    return [BernoulliRBM(n_visible=784, n_hidden=500, W_init=0.01, n_gibbs_steps=k, learning_rate=0.01 * (1 + g % 3),
                         momentum=[0.5, 0.9], max_epoch=2, batch_size=100, l2=1e-5, sample_v_states=g % 2 == 0,
                         metrics_config=dict(msre=True, pll=True, train_metrics_every_iter=5), verbose=False,
                         random_seed=1337 + g, model_path=os.path.join(path, 'rbm_%d' % g) + '/')
            for g in range(G)]


def read(path):
    out = {}
    for kind in ('train', 'val'):
        f = os.path.join(path, 'logs', kind, 'scalars.jsonl')
        out[kind] = open(f).read().splitlines() if os.path.isfile(f) else None
    return out


def same_as_fit(make, Xs, Xv, tmp_path):
    from boltzmann_machines import fit_many
    solo, group = make(str(tmp_path / 'solo')), make(str(tmp_path / 'group'))
    for m, X, V in zip(solo, Xs, Xv if Xv is not None else [None] * len(Xs)):
        m.fit(X, V)
    fit_many(group, Xs, Xv)
    for g, (a, b) in enumerate(zip(solo, group)):
        pa, pb = a._engine.get_params(), b._engine.get_params()
        for n in pa:
            np.testing.assert_array_equal(pb[n], pa[n], err_msg='model {0}: {1}'.format(g, n))
        assert (a.iter_, a.epoch_, a._tick) == (b.iter_, b.epoch_, b._tick)
        da, db = os.path.dirname(a._model_filepath), os.path.dirname(b._model_filepath)
        la, lb = read(da), read(db)
        assert la == lb and la['train'], g
        for f in sorted(os.listdir(da)):
            if f.endswith('.npz'):
                with np.load(os.path.join(da, f)) as za, np.load(os.path.join(db, f)) as zb:
                    assert za.files == zb.files
                    for n in za.files:
                        np.testing.assert_array_equal(zb[n], za[n], err_msg='model {0}: {1}:{2}'.format(g, f, n))
    return group


@pytest.mark.skipif(HOSTSIM, reason='26 models of 192-300 take long on the interpreter')
def test_cifar_patch_rbms(tmp_path):
    rng = np.random.RandomState(9000)
    G, N = 26, 960
    Xs = [(rng.randn(N, 192) * (0.5 + 0.02 * g)).astype(np.float32) for g in range(G)]
    Xv = [rng.randn(96, 192).astype(np.float32) for _ in range(G)]
    same_as_fit(lambda p: patch_models(p, G), Xs, Xv, tmp_path)


@pytest.mark.skipif(HOSTSIM, reason='20 models of 784-500 take long on the interpreter')
def test_bernoulli_784_500_cd3_cut_into_several_launches(tmp_path):
    rng = np.random.RandomState(7)
    G, N = 20, 1000
    protos = rng.rand(10, 784)
    Xs = [(rng.rand(N, 784) < protos[rng.randint(0, 10, N)]).astype(np.float32) for _ in range(G)]
    group = same_as_fit(lambda p: bernoulli_models(p, G), Xs, None, tmp_path)
    # 2k + 3 = 9 ops per member (more with the statistics beside the chain): a step of 20 members takes several launches
    launches = [max(r['launch'] for r in m._engine.debug_tc_plan()) for m in group]
    assert launches[0] == 0 and launches[-1] >= 1 and launches == sorted(launches), launches


def test_single_model(tmp_path):
    rng = np.random.RandomState(3)
    Xs = [rng.rand(130, 64).astype(np.float32)]
    from boltzmann_machines import BernoulliRBM

    def make(p):
        return [BernoulliRBM(n_visible=64, n_hidden=48, max_epoch=2, batch_size=32, n_gibbs_steps=2, learning_rate=0.05,
                             metrics_config=dict(msre=True, pll=True, feg=True, train_metrics_every_iter=2, feg_every_epoch=1),
                             verbose=False, random_seed=11, model_path=os.path.join(p, 'one') + '/')]
    same_as_fit(make, Xs, [rng.rand(40, 64).astype(np.float32)], tmp_path)
