"""Port of the reference's RBM tests
(the reference's boltzmann_machines/rbm/tests/test_rbm.py) exercising the
package's host logic -- schedules, save/load, resume, determinism -- with the
numpy oracle plugged in as the engine (CPU, `-m "not gpu"`), and with the CUDA
engine in both compute modes (`-m gpu`): the `engines` fixture is parametrised."""
import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_almost_equal

from boltzmann_machines.rbm import BernoulliRBM, MultinomialRBM, GaussianRBM, logit_mean
from boltzmann_machines.utils import RNG

N_VISIBLE, N_HIDDEN = 12, 8
CASES = [(BernoulliRBM, 'float32'), (BernoulliRBM, 'float64'),
         (MultinomialRBM, 'float32'), (GaussianRBM, 'float32')]


def data():
    return RNG(seed=1337).rand(16, N_VISIBLE), RNG(seed=42).rand(8, N_VISIBLE)


def config():
    return dict(n_visible=N_VISIBLE, n_hidden=N_HIDDEN, sample_v_states=True, sample_h_states=True,
                dropout=0.9, verbose=False, display_filters=False, random_seed=1337)


def same_weights(a, b):
    wa, wb = a.get_tf_params(scope='weights'), b.get_tf_params(scope='weights')
    for k in ('W', 'hb', 'vb'):
        assert_allclose(wa[k], wb[k])


def same_transforms(a, b, X_val):
    Ha, Hb = a.transform(X_val), b.transform(X_val)
    assert Ha.shape == (len(X_val), N_HIDDEN) == Hb.shape
    assert_allclose(Ha, Hb)


def test_W_init_shape_validation():
    for C in (BernoulliRBM, MultinomialRBM, GaussianRBM):
        for bad in ((4, 2), (3, 3), (3, 2)):
            with pytest.raises(ValueError):
                C(n_visible=4, n_hidden=3, W_init=np.zeros(bad))
        C(n_visible=4, n_hidden=3, W_init=np.zeros((4, 3)))
        C(n_visible=1, n_hidden=1, W_init=np.zeros((1, 1)))


def test_unknown_kwarg_raises():
    with pytest.raises(AttributeError):
        BernoulliRBM(n_visible=4, n_hidden=3, no_such_parameter=1)


def test_use_before_fit_raises(engines, workdir):
    with pytest.raises(RuntimeError):
        BernoulliRBM(n_visible=4, n_hidden=3, model_path='m/').transform(np.zeros((2, 4)))


def test_set_params_rejects_unknown(engines):
    with pytest.raises(ValueError):
        BernoulliRBM(n_visible=4, n_hidden=3).set_params(bogus=1)


@pytest.mark.parametrize('C,dtype', CASES)
def test_initialization_kat(engines, workdir, C, dtype):
    rbm = C(max_epoch=2, model_path='test_rbm_1/', dtype=dtype, **config())
    rbm.init()
    w00 = rbm.get_tf_params(scope='weights')['W'][0][0]
    assert_almost_equal(w00, -0.0094548017 if dtype == 'float32' else -0.0077341544416)


@pytest.mark.parametrize('C,dtype', CASES)
def test_consistency(engines, workdir, C, dtype):
    X, X_val = data()
    mk = lambda path: C(max_epoch=2, model_path=path, dtype=dtype, **config())
    r1, r2 = mk('test_rbm_1/'), mk('test_rbm_2/')
    r1.fit(X), r2.fit(X)
    same_weights(r1, r2), same_transforms(r1, r2, X_val)
    w_after_2 = r1.get_tf_params(scope='weights')['W'].copy()

    for r in (r1, r2):
        r.set_params(max_epoch=r.max_epoch + 1).fit(X)
    same_weights(r1, r2), same_transforms(r1, r2, X_val)
    assert not np.allclose(w_after_2, r1.get_tf_params(scope='weights')['W'])   # it did train on

    r1, r2 = C.load_model('test_rbm_1/'), C.load_model('test_rbm_2/')
    assert r1.epoch_ == 3 and r1.iter_ == 3 * 2
    same_weights(r1, r2), same_transforms(r1, r2, X_val)

    for r in (r1, r2):
        r.set_params(max_epoch=r.max_epoch + 1).fit(X)
    same_weights(r1, r2), same_transforms(r1, r2, X_val)


def test_consistency_val(engines, workdir):
    X, X_val = data()
    mk = lambda path: BernoulliRBM(max_epoch=2, model_path=path,
                                   metrics_config=dict(msre=True, pll=True, feg=True, l2_loss=True,
                                                       train_metrics_every_iter=1),
                                   **config())
    r1, r2 = mk('test_rbm_1/'), mk('test_rbm_2/')
    r1.fit(X, X_val), r2.fit(X, X_val)
    same_weights(r1, r2), same_transforms(r1, r2, X_val)


def test_resume_equals_reload(engines, workdir):
    """continuing in memory == reloading from disk and continuing"""
    X, _ = data()
    a = BernoulliRBM(max_epoch=2, model_path='a/', **config()).fit(X)
    b = BernoulliRBM(max_epoch=2, model_path='b/', **config()).fit(X)
    a.set_params(max_epoch=3).fit(X)
    b = BernoulliRBM.load_model('b/')
    b.set_params(max_epoch=3).fit(X)
    same_weights(a, b)


def test_init_from(engines, workdir):
    X, _ = data()
    a = BernoulliRBM(max_epoch=1, model_path='a/', **config()).fit(X)
    b = BernoulliRBM(max_epoch=2, model_path='b/', **config())
    b.init_from(a)
    assert b.epoch_ == 1
    b.init()
    same_weights(a, b)
    with pytest.raises(ValueError):
        GaussianRBM(n_visible=N_VISIBLE, n_hidden=N_HIDDEN).init_from(a)


def test_get_tf_params_scopes(engines, workdir):
    r = BernoulliRBM(n_visible=5, n_hidden=3, model_path='m/', random_seed=1).init()
    assert set(r.get_tf_params(scope='weights')) == {'W', 'vb', 'hb'}
    assert set(r.get_tf_params(scope='grads_accumulators')) == {'dW', 'dvb', 'dhb'}
    assert 'weights/W' in r.get_tf_params()


def test_logit_mean():
    X = np.array([[0., 1.], [0., 1.], [1., 1.]])
    q = logit_mean(X)
    assert_allclose(q[0], np.log((1 / 3.) / (2 / 3.)))
    assert np.isfinite(q).all()
