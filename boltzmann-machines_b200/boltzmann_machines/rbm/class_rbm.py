"""Classification RBM (Larochelle & Bengio, ICML 2008, "Classification using Discriminative Restricted Boltzmann
Machines"): an RBM over binary inputs x and a one-of-C label y, whose class posterior p(y|x) is exact.

Energy E(x, y, h) = -x'W h - e_y'U h - vb'x - hb'h - yb'e_y.  Training follows the paper's hybrid objective: the gradient
of the batch mean of log p(t|x) plus ``alpha`` times CD-k on the joint p(x, y) (``alpha=0`` is purely discriminative and
runs no Gibbs chain; the default 0.01 is the value the paper reports for MNIST), minus ``l2`` times W and U, applied with
the momentum update of BaseRBM.  The whole step runs in one native call (``bm_crbm_train_step``, csrc/bm_crbm_tc.cuh) on
the tensor cores.

Semi-supervised training (Larochelle, Mandel, Pascanu & Bengio, JMLR 13, 2012): with ``beta > 0`` a label of -1 marks an
unlabelled row, which adds ``beta`` times CD-k of log p(x) -- an exact positive phase and a chain started from a label drawn
from p(y|x) -- so unlabelled data shapes the same joint model the labels train.
"""
import numpy as np

from ..ebm import EnergyBasedModel
from ..base import run_in_tf_session, is_attribute_name, get_engine_factory
from ..utils import make_list_from, batch_bounds, epoch_iter, write_during_training
from ..utils.utils import _maybe_bar
from ..utils.testing import assert_len, assert_shape

_METRIC_DEFAULTS = (('train_metrics_every_iter', 10), ('val_metrics_every_epoch', 1),
                    ('nll_fmt', '.4f'), ('accuracy_fmt', '.4f'))


def _vector(value, n, dtype):
    return np.asarray(value, dtype=dtype) if hasattr(value, '__iter__') else np.full(n, value, dtype=dtype)


class ClassificationRBM(EnergyBasedModel):
    """Classification RBM trained with the hybrid discriminative / generative gradient.

    Parameters
    ----------
    n_visible, n_hidden : positive int
    n_classes : int in [2, 64]
    alpha : weight of the generative (CD-k on p(x, y)) gradient; 0 trains purely discriminatively
    beta : weight of the unlabelled rows' gradient (CD-k on p(x)); with beta > 0, ``fit`` accepts -1 in ``y`` for a row
        without a label.  0 (the default) accepts labelled rows only
    W_init : float (std of the N(0, .) init of W and U) or (n_visible, n_hidden) array for W
    U_init : None (drawn like W from its own op seed) or (n_classes, n_hidden) array
    vb_init, hb_init, yb_init : float or array
    n_gibbs_steps, learning_rate, momentum : scalar or per-epoch list
    max_epoch, batch_size : int
    l2 : weight decay of W and U
    sample_v_states : the chain draws x and the label (one-hot) instead of passing their means
    sample_h_states : the chain draws h
    metrics_config : dict with ``train_metrics_every_iter`` and ``val_metrics_every_epoch``
    dropout, sparsity_cost, dbm_first, dbm_last, compute : accepted for the error message only: any value other than
        the default (None, 0, False, False, None / 'bf16') raises NotImplementedError; float64 models likewise
    """
    _SCOPES = {
        'weights': ('W', 'U', 'vb', 'hb', 'yb'),
        'grads_accumulators': ('dW', 'dU', 'dvb', 'dhb', 'dyb'),
    }

    def __init__(self, n_visible=784, n_hidden=256, n_classes=10, alpha=0.01,
                 W_init=0.01, U_init=None, vb_init=0., hb_init=0., yb_init=0., n_gibbs_steps=1,
                 learning_rate=0.01, momentum=0.9, max_epoch=10, batch_size=10, l2=1e-4,
                 sample_v_states=False, sample_h_states=True,
                 dropout=None, sparsity_cost=0., dbm_first=False, dbm_last=False, compute=None,
                 metrics_config=None, verbose=True, save_after_each_epoch=True,
                 model_path='class_rbm_model/', beta=0., *args, **kwargs):
        super(ClassificationRBM, self).__init__(model_path=model_path, *args, **kwargs)
        for name, value, default in (('dropout', dropout, None), ('sparsity_cost', sparsity_cost, 0.),
                                     ('dbm_first', dbm_first, False), ('dbm_last', dbm_last, False)):
            if value != default:
                raise NotImplementedError('ClassificationRBM does not support {0}={1!r}'.format(name, value))
        if compute not in (None, 'bf16'):
            raise NotImplementedError("ClassificationRBM runs on the tensor cores only (compute={0!r})".format(compute))
        if self.dtype != 'float32':
            raise NotImplementedError("ClassificationRBM supports float32 models only (dtype={0!r})".format(self.dtype))
        if not 2 <= int(n_classes) <= 64:
            raise ValueError('n_classes must be in [2, 64], got {0}'.format(n_classes))
        self.n_visible, self.n_hidden, self.n_classes = n_visible, n_hidden, n_classes
        self.alpha = alpha
        if not float(beta) >= 0.:
            raise ValueError('beta must be non-negative, got {0!r}'.format(beta))
        self.beta = beta
        self.dropout, self.sparsity_cost, self.dbm_first, self.dbm_last, self.compute = \
            dropout, sparsity_cost, dbm_first, dbm_last, compute

        self.W_init = W_init
        if hasattr(self.W_init, '__iter__'):
            self.W_init = np.asarray(self.W_init)
            assert_shape(self, 'W_init', (self.n_visible, self.n_hidden))
        self.U_init = U_init
        if self.U_init is not None:
            self.U_init = np.asarray(self.U_init)
            assert_shape(self, 'U_init', (self.n_classes, self.n_hidden))
        for name, n in (('vb_init', n_visible), ('hb_init', n_hidden), ('yb_init', n_classes)):
            v = locals()[name]
            if hasattr(v, '__iter__'):
                v = np.asarray(v)
            setattr(self, name, v)
            if hasattr(v, '__iter__'):
                assert_len(self, name, n)
        self._acc_init = None                 # momentum accumulators, filled by `init_from`

        self.n_gibbs_steps = make_list_from(n_gibbs_steps)
        self.learning_rate = make_list_from(learning_rate)
        self.momentum = make_list_from(momentum)
        self.max_epoch = max_epoch
        self.batch_size = batch_size
        self.l2 = l2
        self.sample_v_states = sample_v_states
        self.sample_h_states = sample_h_states

        self.metrics_config = dict(metrics_config or {})
        for key, default in _METRIC_DEFAULTS:
            self.metrics_config.setdefault(key, default)
        self.verbose = verbose
        self.save_after_each_epoch = save_after_each_epoch

        self.epoch_ = 0
        self.iter_ = 0

    # ---- engine wiring ---------------------------------------------------------------
    def _engine_cfg(self):
        return dict(n_visible=int(self.n_visible), n_hidden=int(self.n_hidden), n_classes=int(self.n_classes),
                    alpha=float(self.alpha), beta=float(self.beta), l2=float(self.l2), dtype=self.dtype, compute=self.compute,
                    sample_v=bool(self.sample_v_states), sample_h=bool(self.sample_h_states),
                    max_batch=int(self.batch_size), dropout=self.dropout, sparsity_cost=float(self.sparsity_cost),
                    dbm_first=bool(self.dbm_first), dbm_last=bool(self.dbm_last))

    def _make_engine(self):
        return get_engine_factory('crbm')(self._engine_cfg())

    _make_tf_model = _make_engine

    def _init_engine_vars(self):
        V, H, Cn = self.n_visible, self.n_hidden, self.n_classes
        eng = self._engine
        std = 0.01 if hasattr(self.W_init, '__iter__') else float(self.W_init)
        # W from op seed random_seed (as BaseRBM), U from op seed random_seed + 1
        op_seed = self.random_seed
        if op_seed is None:
            op_seed = int(np.random.SeedSequence().generate_state(1)[0])
        eng.init_normal_weights(std, int(op_seed), int(op_seed) + 1)
        if hasattr(self.W_init, '__iter__'):
            eng.set_params({'W': np.asarray(self.W_init, dtype=np.float32)})
        if self.U_init is not None:
            eng.set_params({'U': np.asarray(self.U_init, dtype=np.float32)})
        eng.set_params({'vb': _vector(self.vb_init, V, np.float32), 'hb': _vector(self.hb_init, H, np.float32),
                        'yb': _vector(self.yb_init, Cn, np.float32)})
        acc = self._acc_init or {}
        shapes = {'dW': (V, H), 'dU': (Cn, H), 'dvb': (V,), 'dhb': (H,), 'dyb': (Cn,)}
        eng.set_params({k: np.asarray(acc[k], np.float32) if k in acc else np.zeros(s, np.float32) for k, s in shapes.items()})

    # ---- training ------------------------------------------------------------------------
    def _scheduled(self, values):
        return values[min(self.epoch_, len(values) - 1)]

    def _labels(self, y, n, unlabelled=False):
        """y as int32; -1 (a row without a label) is accepted where ``unlabelled`` allows it and beta > 0"""
        y = np.asarray(y).reshape(-1)
        if y.shape[0] != n:
            raise ValueError('{0} labels for {1} rows'.format(y.shape[0], n))
        if y.size and not np.all(y == np.round(y)):
            raise ValueError('labels must be integers in [0, {0})'.format(self.n_classes))
        if y.size and unlabelled and y.min() == -1 and not float(self.beta) > 0:
            raise ValueError('labels of -1 (unlabelled rows) need beta > 0; beta is {0!r}'.format(self.beta))
        low = -1 if unlabelled and float(self.beta) > 0 else 0
        if y.size and (y.min() < low or y.max() >= self.n_classes):
            raise ValueError('labels must be integers in [{0}, {1})'.format(low, self.n_classes))
        return np.ascontiguousarray(y, dtype=np.int32)

    def _train_epoch(self, X, y):
        every = self.metrics_config['train_metrics_every_iter']
        lr, mom, k = (float(self._scheduled(self.learning_rate)), float(self._scheduled(self.momentum)),
                      int(self._scheduled(self.n_gibbs_steps)))
        got = []
        for lo, hi in _maybe_bar(batch_bounds(len(X), self.batch_size), self.verbose, leave=False, ncols=64, desc='epoch'):
            self.iter_ += 1
            # metrics come from the batch's labelled rows: a reporting batch without one logs nothing
            reporting = bool(every and self.iter_ % every == 0) and bool(np.any(y[lo:hi] >= 0))
            m = self._engine.train_step(X[lo:hi], y[lo:hi], lr, mom, k, self._call_seed, self._next_tick(), metrics=reporting)
            if reporting:
                got.append(m)
                self._log_scalars('train', self.iter_, {'mean_nll': m['nll'], 'accuracy': m['accuracy']})
        if not got:
            return {}
        return {'nll': float(np.mean([g['nll'] for g in got])), 'accuracy': float(np.mean([g['accuracy'] for g in got]))}

    def _scores(self, X, y):
        P = self._proba(X)
        p_t = P[np.arange(len(y)), y].astype(np.float64)
        return {'nll': float(np.mean(-np.log(np.maximum(p_t, np.finfo(np.float64).tiny)))),
                'accuracy': float(np.mean(np.argmax(P, axis=1) == y))}

    def _fit(self, X, y=None, X_val=None, y_val=None):
        if y is None:
            raise ValueError('ClassificationRBM.fit needs the labels y')
        X = np.ascontiguousarray(X, dtype=np.float32)
        y = self._labels(y, len(X), unlabelled=True)
        if X_val is not None:
            X_val = np.ascontiguousarray(X_val, dtype=np.float32)
            y_val = self._labels(y_val, len(X_val))
        mc = self.metrics_config
        for self.epoch_ in epoch_iter(start_epoch=self.epoch_, max_epoch=self.max_epoch, verbose=self.verbose):
            train = self._train_epoch(X, y)
            val = {}
            if X_val is not None and mc['val_metrics_every_epoch'] and self.epoch_ % mc['val_metrics_every_epoch'] == 0:
                val = self._scores(X_val, y_val)
                self._log_scalars('val', self.iter_, {'mean_nll': val['nll'], 'accuracy': val['accuracy']})
            if self.verbose:
                line = 'epoch: {0:{1}}/{2}'.format(self.epoch_, len(str(self.max_epoch)), self.max_epoch)
                for prefix, res in (('', train), ('val.', val)):
                    for m in sorted(res):
                        line += '; {0}{1}: {2:{3}}'.format(prefix, m, res[m], mc[m + '_fmt'])
                write_during_training(line)
            if self.save_after_each_epoch:
                self._save_model(global_step=self.epoch_)

    def fit(self, X, y=None, X_val=None, y_val=None):
        """Train on X [n, n_visible] with labels y [n] in [0, n_classes); validation data optional.

        With ``beta > 0``, y may hold -1 for rows without a label (``y_val`` must be fully labelled).  Batches are taken in
        row order, as for labelled data, so the order of X decides how labelled and unlabelled rows share a batch: shuffle
        or interleave them beforehand to mix them."""
        return super(ClassificationRBM, self).fit(X, X_val=X_val, y=y, y_val=y_val)

    # ---- inference -------------------------------------------------------------------------
    def _proba(self, X):
        X = np.ascontiguousarray(X, dtype=np.float32)
        return np.concatenate([self._engine.predict_proba(X[lo:hi]) for lo, hi in batch_bounds(len(X), self.batch_size)]
                              or [np.zeros((0, self.n_classes), np.float32)])

    @run_in_tf_session()
    def predict_proba(self, X):
        """p(y|x) [n, n_classes] (float32), exact."""
        return self._proba(X)

    def predict(self, X):
        """argmax_y p(y|x); a tie goes to the lowest class index."""
        return np.argmax(self.predict_proba(X), axis=1)

    @run_in_tf_session()
    def transform(self, X):
        """E[h|x] = sum_y p(y|x) sigmoid(hb + U_y + x W) [n, n_hidden]."""
        X = np.ascontiguousarray(X, dtype=np.float32)
        return np.concatenate([self._engine.transform(X[lo:hi]) for lo, hi in batch_bounds(len(X), self.batch_size)]
                              or [np.zeros((0, self.n_hidden), np.float32)])

    def init_from(self, model):
        """Start from another ClassificationRBM's weights, momentum accumulators and trailing-underscore attributes."""
        if type(self) != type(model):
            raise ValueError('an attempt to initialize `{0}` from `{1}`'.format(self.__class__.__name__, model.__class__.__name__))
        w = model.get_tf_params(scope='weights')
        self.W_init, self.U_init, self.vb_init, self.hb_init, self.yb_init = w['W'], w['U'], w['vb'], w['hb'], w['yb']
        self._acc_init = model.get_tf_params(scope='grads_accumulators')
        for k, v in vars(model).items():
            if is_attribute_name(k):
                setattr(self, k, v)
        self.initialized_ = False
        self.close()
