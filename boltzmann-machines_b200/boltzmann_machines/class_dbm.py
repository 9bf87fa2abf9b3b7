"""Classification DBM: a DBM with a one-of-C label layer y above its top hidden layer h_L (no counterpart in the reference,
whose README lists classification DBMs as future work; DESIGN.md §5.7).

Energy: the DBM energy - e_y'U h_L - yb'e_y, with U [n_classes, H_L] and yb [n_classes]; y connects to h_L only.  The model
learns p(x, y) with the DBM's own procedure: in the mean-field E-step the label of a labelled row is held at its one-hot value
and the label of a row labelled -1 is inferred like any hidden layer; the persistent chains sweep v, h_1 .. h_L and y; U takes
the l2, momentum and max-norm of every W, yb the plain momentum update.  ``predict_proba`` runs the E-step with y free and
returns softmax(yb + mu_L U^T) from its final mu_L.  The whole step runs on the tensor-core DBM engine
(``bm_dbm_train_step_labeled``, csrc/bm_cdbm_tc.cuh).
"""
import numpy as np

from .base import run_in_tf_session
from .dbm import DBM
from .layers import BernoulliLayer
from .rbm.class_rbm import ClassificationRBM
from .utils import batch_bounds, epoch_iter, write_during_training
from .utils.utils import _maybe_bar


class _PosteriorRBM(object):
    """What DBM.load_rbms reads of a stacked RBM, for the (x, h) part of a ClassificationRBM."""
    def __init__(self, crbm):
        self.n_visible, self.n_hidden = crbm.n_visible, crbm.n_hidden
        w = crbm.get_tf_params(scope='weights')
        self._weights = {k: w[k] for k in ('W', 'vb', 'hb')}
        self._v_layer, self._h_layer = BernoulliLayer(crbm.n_visible), BernoulliLayer(crbm.n_hidden)

    def get_tf_params(self, scope=None):
        return dict(self._weights)


class ClassificationDBM(DBM):
    """DBM over x with a label layer above the top hidden layer, trained on labelled and unlabelled rows.

    Parameters: those of ``DBM``, except

    rbms : a stack of pre-trained RBMs whose LAST member is a ``ClassificationRBM`` (ValueError otherwise).  Their
        (W, vb, hb) are composed exactly as ``DBM`` composes its stack; U and yb are the ClassificationRBM's, unchanged, and
        their momenta start at zero.
    pt_betas : must be None, and the model float32 (NotImplementedError otherwise): the classification DBM runs on the
        tensor-core engine without parallel tempering.

    ``fit(X, y)`` takes labels in {-1, 0, .., n_classes - 1}; -1 marks an unlabelled row.  Validation logs the DBM's
    msre and n_mf_updates and the ``mean_nll`` and ``accuracy`` of ``predict_proba``.  ``log_Z`` and ``log_proba`` are not
    available: the AIS ladder and the variational bound have no label layer.
    """

    def __init__(self, rbms=None, pt_betas=None, model_path='class_dbm_model/', *args, **kwargs):
        if pt_betas is not None:
            raise NotImplementedError('ClassificationDBM does not support parallel tempering (pt_betas)')
        if kwargs.get('centering'):
            raise NotImplementedError('ClassificationDBM does not support centering')
        self.n_classes_ = None
        super(ClassificationDBM, self).__init__(rbms=rbms, pt_betas=None, model_path=model_path, *args, **kwargs)
        if np.dtype(self.dtype) != np.float32:
            raise NotImplementedError('ClassificationDBM supports float32 models only (dtype={0!r})'.format(self.dtype))

    # ---- composition ----------------------------------------------------------------------------------------
    def load_rbms(self, rbms):
        if rbms is None:
            return
        rbms = list(rbms)
        if not rbms or not isinstance(rbms[-1], ClassificationRBM):
            raise ValueError('the last RBM of a ClassificationDBM must be a ClassificationRBM')
        if any(isinstance(r, ClassificationRBM) for r in rbms[:-1]):
            raise ValueError('only the last RBM of a ClassificationDBM may be a ClassificationRBM')
        crbm = rbms[-1]
        w = crbm.get_tf_params(scope='weights')
        self._U_init = np.array(w['U'], dtype=np.float32)
        self._yb_init = np.array(w['yb'], dtype=np.float32)
        self.n_classes_ = int(crbm.n_classes)
        super(ClassificationDBM, self).load_rbms(rbms[:-1] + [_PosteriorRBM(crbm)])

    def _scopes(self):
        s = dict(super(ClassificationDBM, self)._scopes())
        s['weights'] = s['weights'] + ('U', 'yb')
        s['grads_accumulators'] = s['grads_accumulators'] + ('dU', 'dyb')
        s['variational_params'] = s['variational_params'] + ('mu_y',)
        s['negative_particles'] = s['negative_particles'] + ('y',)
        return s

    def _engine_cfg(self):
        cfg = super(ClassificationDBM, self)._engine_cfg()
        cfg['n_classes'] = int(self.n_classes_)
        return cfg

    def _init_engine_vars(self):
        super(ClassificationDBM, self)._init_engine_vars()
        Cn, H = self._U_init.shape
        self._engine.set_params({'U': self._U_init, 'yb': self._yb_init,
                                 'dU': np.zeros((Cn, H), np.float32), 'dyb': np.zeros(Cn, np.float32)})

    # ---- training -----------------------------------------------------------------------------------------------
    def _labels(self, y, n, unlabelled):
        y = np.asarray(y).reshape(-1)
        if y.shape[0] != n:
            raise ValueError('{0} labels for {1} rows'.format(y.shape[0], n))
        low = -1 if unlabelled else 0
        if y.size and (not np.all(y == np.round(y)) or y.min() < low or y.max() >= self.n_classes_):
            raise ValueError('labels must be integers in [{0}, {1})'.format(low, self.n_classes_))
        return np.ascontiguousarray(y, dtype=np.int32)

    def _train_epoch_labeled(self, X, y):
        msres, n_mfs = [], []
        for lo, hi in _maybe_bar(batch_bounds(len(X), self.batch_size), self.verbose, leave=False, ncols=64, desc='epoch'):
            self.iter_ += 1
            report = ('msre', 'n_mf_updates') if (self.train_metrics_every_iter and
                                                  self.iter_ % self.train_metrics_every_iter == 0) else ()
            got = self._engine.train_step(X[lo:hi], tick=self._next_tick(), metrics=report, labels=y[lo:hi],
                                          **self._step_args())
            if report:
                msres.append(got['msre']); n_mfs.append(got['n_mf_updates'])
                self._log_scalars('train', self.iter_, {'mean_squared_recon_error': got['msre'],
                                                        'n_mf_updates': got['n_mf_updates']})
        return (float(np.mean(msres)) if msres else None, float(np.mean(n_mfs)) if n_mfs else None)

    def _scores(self, X, y):
        P = self._per_batch(X, self.n_classes_, self._engine.predict_proba, 'predict_proba', np.float32)
        p_t = P[np.arange(len(y)), y].astype(np.float64)
        return {'nll': float(np.mean(-np.log(np.maximum(p_t, np.finfo(np.float64).tiny)))),
                'accuracy': float(np.mean(np.argmax(P, axis=1) == y))}

    def _fit(self, X, y=None, X_val=None, y_val=None):
        if y is None:
            raise ValueError('ClassificationDBM.fit needs the labels y')
        X = np.ascontiguousarray(X, dtype=self._np_dtype)
        y = self._labels(y, len(X), unlabelled=True)
        if X_val is not None:
            X_val = np.ascontiguousarray(X_val, dtype=self._np_dtype)
            y_val = self._labels(y_val, len(X_val), unlabelled=False) if y_val is not None else None
        for self.epoch_ in epoch_iter(start_epoch=self.epoch_, max_epoch=self.max_epoch, verbose=self.verbose):
            train_msre, train_n_mf = self._train_epoch_labeled(X, y)
            val = {}
            if X_val is not None and self.val_metrics_every_epoch and self.epoch_ % self.val_metrics_every_epoch == 0:
                val['msre'], val['n_mf'] = self._run_val_metrics(X_val)
                if y_val is not None:
                    s = self._scores(X_val, y_val)
                    val.update(s)
                    self._log_scalars('val', self.iter_, {'mean_nll': s['nll'], 'accuracy': s['accuracy']})
            if self.verbose:
                line = 'epoch: {0:{1}}/{2}'.format(self.epoch_, len(str(self.max_epoch)), self.max_epoch)
                if train_msre:
                    line += '; msre: {0:.5f}'.format(train_msre)
                if train_n_mf:
                    line += '; n_mf_upds: {0:.1f}'.format(train_n_mf)
                for key, fmt in (('msre', '.5f'), ('n_mf', '.1f'), ('nll', '.4f'), ('accuracy', '.4f')):
                    if key in val:
                        line += '; val.{0}: {1:{2}}'.format(key, val[key], fmt)
                write_during_training(line)
            if self.save_after_each_epoch:
                self._save_model(global_step=self.epoch_)

    def fit(self, X, y=None, X_val=None, y_val=None):
        """Train on X [n, n_visible] with labels y [n] in {-1, 0, .., n_classes - 1} (-1: unlabelled row); validation data
        optional (``y_val`` fully labelled, or None for the DBM's metrics only)."""
        return super(ClassificationDBM, self).fit(X, X_val=X_val, y=y, y_val=y_val)

    # ---- queries ------------------------------------------------------------------------------------------------
    @run_in_tf_session()
    def predict_proba(self, X):
        """softmax(yb + mu_L U^T) [n, n_classes] (float32), mu_L from the mean-field E-step with y free.  This is the
        mean-field approximation of p(y|x), not the exact posterior.  Leaves the variational parameters and particles as
        they were."""
        return self._per_batch(X, self.n_classes_, self._engine.predict_proba, 'predict_proba', np.float32)

    @run_in_tf_session(update_seed=True)
    def fill_missing(self, X, mask, y=None, n_gibbs_steps=100):
        """``DBM.fill_missing`` with labels: y [n] in {-1, 0, .., n_classes - 1} (None: all -1).  A row labelled t holds
        its label at e_t in every sweep, so its chain samples p(v_missing | v_observed, y = t); -1 leaves the label free.
        Class-conditional generation is ``fill_missing(np.zeros((n, V)), np.zeros((n, V)), y=labels)``."""
        labels = None if y is None else self._labels(y, len(np.asarray(X)), unlabelled=True)
        return self._fill(X, mask, labels, n_gibbs_steps)

    def predict(self, X):
        """argmax of ``predict_proba``; a tie goes to the lowest class index."""
        return np.argmax(self.predict_proba(X), axis=1)

    def log_Z(self, *args, **kwargs):
        raise NotImplementedError('ClassificationDBM: log_Z is not available (the AIS ladder has no label layer)')

    def exact_log_Z(self, *args, **kwargs):
        raise NotImplementedError('ClassificationDBM: exact_log_Z is not available (the enumeration has no label layer)')

    def exact_log_proba(self, *args, **kwargs):
        raise NotImplementedError('ClassificationDBM: exact_log_proba is not available (the enumeration has no label layer)')

    def log_proba(self, *args, **kwargs):
        raise NotImplementedError('ClassificationDBM: log_proba is not available (the variational bound has no label layer)')

    def ais_log_proba(self, *args, **kwargs):
        raise NotImplementedError('ClassificationDBM: ais_log_proba is not available (the AIS ladder has no label layer)')
