"""Train many RBMs of one shape at once: ``fit_many``.

A small RBM's training step leaves most of the GPU idle, so models that differ only in data, seed or hyper-parameters --
the patch RBMs of a convolutional pipeline, a hyper-parameter sweep -- train faster side by side than one after another.
``fit_many`` runs their epochs as grouped native epochs (``bm_rbm_group_train_epoch``: the members' steps share program
launches) and everything else exactly as each model's own ``fit`` does, so each model ends where its own ``fit`` ends.
"""
import numpy as np

from ..base import get_engine_factory
from ..utils import batch_bounds, epoch_iter
from .base_rbm import BaseRBM

__all__ = ['fit_many']

_SHARED = ('n_visible', 'n_hidden', 'batch_size', 'n_gibbs_steps', 'max_epoch', 'epoch_')


def fit_many(rbms, Xs, X_vals=None):
    """Fit every ``rbms[i]`` to ``Xs[i]`` (validation data ``X_vals[i]``, optional) as ``rbms[i].fit(Xs[i], X_vals[i])`` would:
    the same weights, accumulators, ticks, ``iter_`` / ``epoch_``, ``logs/*/scalars.jsonl`` and checkpoints, bit for bit.

    The models must be of one class with the same ``n_visible``, ``n_hidden``, ``batch_size``, ``n_gibbs_steps`` schedule,
    ``max_epoch`` and current ``epoch_`` (``ValueError`` naming the attribute otherwise), and the training sets must have the
    same number of rows.  Seeds, learning rates, momenta, sigma, ``l2``, sparsity, ``dbm_first`` / ``dbm_last``, sampling flags
    and metrics may differ.  Options the grouped engine does not run (multinomial layers, dropout, user-defined layers,
    float64 or ``compute='fp32'`` models) raise ``NotImplementedError``.  Returns ``rbms``."""
    rbms = list(rbms)
    if not rbms:
        raise ValueError('fit_many needs at least one model')
    Xs = list(Xs)
    X_vals = [None] * len(rbms) if X_vals is None else list(X_vals)
    if len(Xs) != len(rbms) or len(X_vals) != len(rbms):
        raise ValueError('fit_many needs one training set (and one validation set, if any) per model')
    first = rbms[0]
    for m in rbms:
        if not isinstance(m, BaseRBM) or type(m) is not type(first):
            raise ValueError('fit_many: the models must be of one class (got {0} and {1})'
                             .format(type(first).__name__, type(m).__name__))
        for attr in _SHARED:
            if getattr(m, attr) != getattr(first, attr):
                raise ValueError('fit_many: the models must share `{0}` ({1!r} != {2!r})'
                                 .format(attr, getattr(first, attr), getattr(m, attr)))
        if m._v_layer.kind is None or m._h_layer.kind is None:
            raise NotImplementedError('fit_many: user-defined layers (their conditionals run on the host between launches)')
    Xs = [np.ascontiguousarray(X, dtype=m._np_dtype) for m, X in zip(rbms, Xs)]
    if any(X.ndim != 2 or X.shape != Xs[0].shape for X in Xs):
        raise ValueError('fit_many: the training sets must have one shape (rows, n_visible)')
    X_vals = [None if Xv is None else np.ascontiguousarray(Xv, dtype=m._np_dtype) for m, Xv in zip(rbms, X_vals)]

    # what the decorator of `fit` does before the call (base/native_model.py run_in_tf_session)
    for m in rbms:
        m._call_seed = m.make_random_seed()
        m._tick = 0
        if m._engine is None:
            m._engine = m._make_engine()
            if m.initialized_:
                m._restore_engine()
            else:
                m._init_engine_vars()
    group = None
    pinned = None
    try:
        group = get_engine_factory('rbm_group')([m._engine for m in rbms])
        for m in rbms:
            m.initialized_ = True
        pinned = group.pin(Xs)
        n_batches = len(batch_bounds(Xs[0].shape[0], first.batch_size))
        for epoch in epoch_iter(start_epoch=first.epoch_, max_epoch=first.max_epoch, verbose=first.verbose):
            args, wanted = [], []
            for m in rbms:
                m.epoch_ = epoch
                args.append(m._step_args())
                wanted.append(m._enabled(m._TRAIN_METRICS))
            got = group.train_epoch(pinned, first.batch_size, lr=[a['lr'] for a in args], momentum=[a['momentum'] for a in args],
                                    k=args[0]['k'], seed=[a['seed'] for a in args], tick0=[m._tick for m in rbms],
                                    metrics=wanted, every=[m.metrics_config['train_metrics_every_iter'] or 0 for m in rbms],
                                    iter0=[m.iter_ for m in rbms])
            for i, m in enumerate(rbms):
                m._end_epoch(pinned[i], X_vals[i], m._log_train_epoch(got[i], n_batches))
        for m in rbms:
            m._save_model()
    finally:
        if pinned is not None:
            group.unpin(pinned)
        if group is not None:
            group.close()
        for m in rbms:
            m._flush_scalars()
    return rbms
