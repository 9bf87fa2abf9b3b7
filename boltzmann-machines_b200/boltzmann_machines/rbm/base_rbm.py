"""CD-k Restricted Boltzmann Machine: host-side training loop over the native engine.

Interface parity target: /root/reference/boltzmann_machines/rbm/base_rbm.py
(constructor kwargs :95-105, ``metrics_config`` keys :166-178, epoch/batch loop
:549-666, ``init_from`` :668-685, ``transform`` :687-700).  Where the reference
builds a TF graph (``_make_tf_model``) this class hands a configuration to the
engine (``_make_engine``); where it calls ``session.run(train_op, feed_dict)``
per mini-batch (:566) this class makes one C-ABI call, ``engine.train_step``,
which runs the whole CD-k step -- h0, k Gibbs sweeps, dW/dvb/dhb, sparsity,
momentum update -- in hand-written sm_90a CUDA.
"""
import numpy as np

from ..ebm import EnergyBasedModel
from ..base import run_in_tf_session, is_attribute_name, get_engine_factory
from ..utils import make_list_from, batch_bounds, epoch_iter, write_during_training
from ..utils.utils import _maybe_bar
from ..utils.testing import assert_len, assert_shape

_METRIC_DEFAULTS = (
    ('l2_loss', False), ('msre', False), ('pll', False), ('feg', False),
    ('l2_loss_fmt', '.2e'), ('msre_fmt', '.4f'), ('pll_fmt', '.3f'), ('feg_fmt', '.2f'),
    ('train_metrics_every_iter', 10), ('val_metrics_every_epoch', 1),
    ('feg_every_epoch', 2), ('n_batches_for_feg', 10),
)


def _as_vector(value, n, dtype):
    if hasattr(value, '__iter__'):
        return np.asarray(value, dtype=dtype)
    return np.full(n, value, dtype=dtype)


class BaseRBM(EnergyBasedModel):
    """Generic RBM trained with k-step Contrastive Divergence.

    Parameters (identical names and meaning to the reference)
    ----------
    n_visible, n_hidden : positive int
    v_layer_cls, h_layer_cls : layer classes from ``boltzmann_machines.layers``
    v_layer_params, h_layer_params : dict, extra layer kwargs
    W_init : float (std of N(0, .) init) or (n_visible, n_hidden) array
    vb_init, hb_init : float or array
    n_gibbs_steps, learning_rate, momentum : scalar or per-epoch list
    max_epoch, batch_size : int
    l2 : weight decay
    sample_v_states, sample_h_states : bool
    dropout : None or keep-probability of a visible unit
    sparsity_target, sparsity_cost, sparsity_damping : floats
    dbm_first, dbm_last : bool, double the bottom-up / top-down input (DBM pre-training)
    metrics_config : dict (keys in ``_METRIC_DEFAULTS``)
    verbose, save_after_each_epoch : bool
    display_filters, display_hidden_activations, v_shape : accepted for
        compatibility (TensorBoard image summaries are out of scope)
    """
    _SCOPES = {
        'weights': ('W', 'vb', 'hb'),
        'grads_accumulators': ('dW', 'dvb', 'dhb'),
        'hidden_activations_means': ('q_means',),
    }
    # summary tags of the reference (base_rbm.py:179-184)
    _METRIC_TAGS = {'feg': 'free_energy_gap', 'l2_loss': 'l2_loss', 'msre': 'mean_squared_reconstruction_error',
                    'pll': 'pseudo_loglikelihood'}
    _TRAIN_METRICS = ('l2_loss', 'msre', 'pll')
    _VAL_METRICS = ('msre', 'pll')

    def __init__(self,
                 n_visible=784, v_layer_cls=None, v_layer_params=None,
                 n_hidden=256, h_layer_cls=None, h_layer_params=None,
                 W_init=0.01, vb_init=0., hb_init=0., n_gibbs_steps=1,
                 learning_rate=0.01, momentum=0.9, max_epoch=10, batch_size=10, l2=1e-4,
                 sample_v_states=False, sample_h_states=True, dropout=None,
                 sparsity_target=0.1, sparsity_cost=0., sparsity_damping=0.9,
                 dbm_first=False, dbm_last=False,
                 metrics_config=None, verbose=True, save_after_each_epoch=True,
                 display_filters=0, display_hidden_activations=0, v_shape=(28, 28),
                 model_path='rbm_model/', *args, **kwargs):
        super(BaseRBM, self).__init__(model_path=model_path, *args, **kwargs)
        self.n_visible = n_visible
        self.n_hidden = n_hidden

        vp = dict(v_layer_params or {})
        vp.setdefault('n_units', self.n_visible)
        vp.setdefault('dtype', self.dtype)
        hp = dict(h_layer_params or {})
        hp.setdefault('n_units', self.n_hidden)
        hp.setdefault('dtype', self.dtype)
        self._v_layer = v_layer_cls(**vp)
        self._h_layer = h_layer_cls(**hp)

        self.W_init = W_init
        if hasattr(self.W_init, '__iter__'):
            self.W_init = np.asarray(self.W_init)
            assert_shape(self, 'W_init', (self.n_visible, self.n_hidden))
        self.vb_init = vb_init
        if hasattr(self.vb_init, '__iter__'):
            self.vb_init = np.asarray(self.vb_init)
            assert_len(self, 'vb_init', self.n_visible)
        self.hb_init = hb_init
        if hasattr(self.hb_init, '__iter__'):
            self.hb_init = np.asarray(self.hb_init)
            assert_len(self, 'hb_init', self.n_hidden)

        # momentum accumulators, filled by `init_from`
        self._dW_init = None
        self._dvb_init = None
        self._dhb_init = None

        self.n_gibbs_steps = make_list_from(n_gibbs_steps)
        self.learning_rate = make_list_from(learning_rate)
        self.momentum = make_list_from(momentum)
        self.max_epoch = max_epoch
        self.batch_size = batch_size
        self.l2 = l2

        self.sample_h_states = sample_h_states
        self.sample_v_states = sample_v_states
        self.dropout = dropout

        self.sparsity_target = sparsity_target
        self.sparsity_cost = sparsity_cost
        self.sparsity_damping = sparsity_damping

        self.dbm_first = dbm_first
        self.dbm_last = dbm_last

        self.metrics_config = dict(metrics_config or {})
        for key, default in _METRIC_DEFAULTS:
            self.metrics_config.setdefault(key, default)

        self.verbose = verbose
        self.save_after_each_epoch = save_after_each_epoch

        assert self.n_hidden >= display_filters
        self.display_filters = display_filters
        assert self.n_hidden >= display_hidden_activations
        self.display_hidden_activations = display_hidden_activations
        self.v_shape = tuple(v_shape)
        if len(self.v_shape) == 2:
            self.v_shape = self.v_shape + (1,)

        self.epoch_ = 0
        self.iter_ = 0

    # ---- engine wiring -----------------------------------------------------------
    def _engine_cfg(self):
        cfg = dict(
            n_visible=int(self.n_visible), n_hidden=int(self.n_hidden),
            v_kind=self._v_layer.kind, h_kind=self._h_layer.kind,
            dtype=self.dtype, l2=float(self.l2),
            sample_v=bool(self.sample_v_states), sample_h=bool(self.sample_h_states),
            dropout=None if self.dropout is None else float(self.dropout),
            sparsity_target=float(self.sparsity_target),
            sparsity_cost=float(self.sparsity_cost),
            sparsity_damping=float(self.sparsity_damping),
            dbm_first=bool(self.dbm_first), dbm_last=bool(self.dbm_last),
            max_batch=int(self.batch_size),
        )
        for side, layer in (('v', self._v_layer), ('h', self._h_layer)):
            if layer.kind is None:
                continue                       # user-defined layer: the host-driven plugin engine (_make_engine)
            ep = layer.engine_params()
            if 'n_samples' in ep:
                cfg[side + '_n_samples'] = float(ep['n_samples'])
            if 'sigma' in ep:
                if side != 'v':
                    raise NotImplementedError('gaussian hidden units are not supported')
                cfg['sigma'] = np.broadcast_to(np.asarray(ep['sigma'], dtype=np.float64),
                                               (self.n_visible,)).copy()
        return cfg

    def _make_engine(self):
        if self._v_layer.kind is None or self._h_layer.kind is None:
            # a layer that is none of the built-in kinds (layers.py:8-36): GEMMs on the GPU, the layer's own
            # activation / _sample on the host in between (boltzmann_machines/_plugin.py)
            from .._plugin import HostLayerRBM
            return HostLayerRBM(self._engine_cfg(), self._v_layer, self._h_layer)
        return get_engine_factory('rbm')(self._engine_cfg())

    _make_tf_model = _make_engine      # the reference's hook name

    def _init_engine_vars(self):
        dt = self._np_dtype
        V, H = self.n_visible, self.n_hidden
        eng = self._engine
        if hasattr(self.W_init, '__iter__'):
            eng.set_params({'W': np.asarray(self.W_init, dtype=dt)})
        else:
            # same stream as `tf.random_normal(..., stddev=W_init, seed=random_seed)`
            # (base_rbm.py:277-279); pinned by the reference's KAT, test_rbm.py:65-67
            op_seed = self.random_seed
            if op_seed is None:
                op_seed = int(np.random.SeedSequence().generate_state(1)[0])
            eng.init_normal_W(float(self.W_init), int(op_seed))
        z = lambda a, n: np.zeros(n, dtype=dt) if a is None else np.asarray(a, dtype=dt)
        eng.set_params({
            'vb': _as_vector(self.vb_init, V, dt),
            'hb': _as_vector(self.hb_init, H, dt),
            'dW': z(self._dW_init, (V, H)),
            'dvb': z(self._dvb_init, V),
            'dhb': z(self._dhb_init, H),
            'q_means': np.zeros(H, dtype=dt),
        })

    # ---- per-epoch schedules ---------------------------------------------------------
    def _scheduled(self, values):
        return values[min(self.epoch_, len(values) - 1)]

    def _step_args(self, n_gibbs_steps=None):
        k = self._scheduled(self.n_gibbs_steps) if n_gibbs_steps is None else n_gibbs_steps
        return dict(lr=float(self._scheduled(self.learning_rate)),
                    momentum=float(self._scheduled(self.momentum)),
                    k=int(k), seed=self._call_seed)

    # ---- training ------------------------------------------------------------------
    def _enabled(self, names):
        return tuple(m for m in names if self.metrics_config[m])

    def _train_epoch(self, X):
        wanted = self._enabled(self._TRAIN_METRICS)
        every = self.metrics_config['train_metrics_every_iter']
        sums = {m: [] for m in wanted}
        bounds = batch_bounds(len(X), self.batch_size)
        if hasattr(self._engine, 'train_epoch'):
            # the whole batch loop in native calls: same ticks, same results, uploads overlapped.  verbose: the epoch goes in
            # up to 16 calls of whole batches so that the progress bar still moves (the results do not depend on the cut)
            n_calls = min(16, len(bounds)) if self.verbose else 1
            cuts = [len(bounds) * c // n_calls for c in range(n_calls + 1)]
            got = {m: [] for m in wanted}
            for c in _maybe_bar(range(n_calls), self.verbose, leave=False, ncols=64, desc='epoch'):
                b0, b1 = cuts[c], cuts[c + 1]
                if b0 == b1:
                    continue
                part = self._engine.train_epoch(X[bounds[b0][0]:bounds[b1 - 1][1]], self.batch_size, tick0=self._tick + b0,
                                                metrics=wanted, every=every or 0, iter0=self.iter_ + b0, **self._step_args())
                for m in wanted:
                    got[m].extend(part[m])
            return self._log_train_epoch(got, len(bounds))
        for lo, hi in _maybe_bar(bounds, self.verbose, leave=False, ncols=64, desc='epoch'):
            self.iter_ += 1
            reporting = bool(every and self.iter_ % every == 0)
            report = wanted if reporting else ()
            got = self._engine.train_step(X[lo:hi], tick=self._next_tick(),
                                          metrics=report, **self._step_args())
            for m in report:
                sums[m].append(got[m])
            if reporting:
                # the reference writes its merged summaries at every reporting iteration, whether or not a scalar
                # train metric is enabled (base_rbm.py:554-564)
                self._log_scalars('train', self.iter_, {self._METRIC_TAGS[m]: got[m] for m in report}, allow_empty=True)
        return {m: (float(np.mean(v)) if v else None) for m, v in sums.items()}

    def _log_train_epoch(self, got, n_batches):
        """Bookkeeping of an epoch the engine ran in one go: ticks, iterations and the train scalars of the reporting batches
        (`got`: {metric: [value of every reporting batch]}).  Returns the epoch's mean of every metric."""
        every = self.metrics_config['train_metrics_every_iter']
        self._tick += n_batches
        if every:
            steps = [self.iter_ + i + 1 for i in range(n_batches) if (self.iter_ + i + 1) % every == 0]
            for j, step in enumerate(steps):
                self._log_scalars('train', step, {self._METRIC_TAGS[m]: got[m][j] for m in got}, allow_empty=True)
        self.iter_ += n_batches
        return {m: (float(np.mean(v)) if v else None) for m, v in got.items()}

    def _run_val_metrics(self, X_val):
        wanted = self._enabled(self._VAL_METRICS)
        acc = {m: [] for m in wanted}
        a = self._step_args()
        for lo, hi in batch_bounds(len(X_val), self.batch_size):
            # the reference runs the session once per validation batch even when no validation metric is enabled
            # (`run_ops == []`, base_rbm.py:575-579): the call still counts as a tick of this public call
            tick = self._next_tick()
            if not wanted:
                continue
            got = self._engine.metrics(X_val[lo:hi], k=a['k'], seed=a['seed'], tick=tick, names=wanted)
            for m in wanted:
                acc[m].append(got[m])
        res = {m: (float(np.mean(v)) if v else None) for m, v in acc.items()}
        # base_rbm.py:584-589: the summary is written even when it holds no value
        self._log_scalars('val', self.iter_, {self._METRIC_TAGS[m]: v for m, v in res.items()}, allow_empty=True)
        return res

    def _mean_free_energy(self, X):
        a = self._step_args()
        n = self.metrics_config['n_batches_for_feg']
        vals = [self._engine.metrics(X[lo:hi], k=a['k'], seed=a['seed'], tick=self._next_tick(),
                                     names=('free_energy',))['free_energy']
                for lo, hi in batch_bounds(len(X), self.batch_size)[:n]]
        return float(np.mean(vals))

    def _run_feg(self, X, X_val):
        """Free-energy gap (validation minus training): ~0 when not overfitting."""
        train_fe = self._mean_free_energy(X)
        feg = self._mean_free_energy(X_val) - train_fe
        self._log_scalars('val', self.iter_, {self._METRIC_TAGS['feg']: feg})                      # base_rbm.py:617-621
        return feg

    def _fit(self, X, X_val=None, *args, **kwargs):
        X = np.ascontiguousarray(X, dtype=self._np_dtype)
        if X_val is not None:
            X_val = np.ascontiguousarray(X_val, dtype=self._np_dtype)
        pinned = self._engine.pin(X) if hasattr(self._engine, 'pin') else None   # page-locked copy: async uploads
        if pinned is not None:
            X = pinned
        try:
            for self.epoch_ in epoch_iter(start_epoch=self.epoch_, max_epoch=self.max_epoch,
                                          verbose=self.verbose):
                self._end_epoch(X, X_val, self._train_epoch(X))
        finally:
            if pinned is not None:
                self._engine.unpin(pinned)

    def _end_epoch(self, X, X_val, train_results):
        """What follows the training batches of an epoch: validation metrics, free-energy gap, verbose line, checkpoint."""
        mc = self.metrics_config
        val_results, feg = {}, None
        if X_val is not None and self.epoch_ % mc['val_metrics_every_epoch'] == 0:
            val_results = self._run_val_metrics(X_val)
        if X_val is not None and mc['feg'] and self.epoch_ % mc['feg_every_epoch'] == 0:
            feg = self._run_feg(X, X_val)

        if self.verbose:
            line = 'epoch: {0:{1}}/{2}'.format(self.epoch_, len(str(self.max_epoch)), self.max_epoch)
            for prefix, res in (('', train_results), ('val.', val_results)):
                for m in sorted(res):
                    if res[m] is not None:
                        line += '; {0}{1}: {2:{3}}'.format(prefix, m, res[m], mc[m + '_fmt'])
            if feg is not None:
                line += ' ; feg: {0:{1}}'.format(feg, mc['feg_fmt'])
            write_during_training(line)

        if self.save_after_each_epoch:
            self._save_model(global_step=self.epoch_)

    def init_from(self, rbm):
        """Start from another RBM's weights, momentum accumulators and
        trailing-underscore attributes (a model of the same class)."""
        if type(self) != type(rbm):
            raise ValueError('an attempt to initialize `{0}` from `{1}`'
                             .format(self.__class__.__name__, rbm.__class__.__name__))
        weights = rbm.get_tf_params(scope='weights')
        self.W_init, self.vb_init, self.hb_init = weights['W'], weights['vb'], weights['hb']
        acc = rbm.get_tf_params(scope='grads_accumulators')
        self._dW_init, self._dvb_init, self._dhb_init = acc['dW'], acc['dvb'], acc['dhb']
        for k, v in vars(rbm).items():
            if is_attribute_name(k):
                setattr(self, k, v)
        # the reference also copies `initialized_=True`, after which its next call
        # tries to restore a checkpoint this (new) model never wrote; a copy starts
        # un-initialised so that `init()`/`fit()` build it from the values above
        self.initialized_ = False
        self.close()

    @run_in_tf_session(update_seed=True)
    def transform(self, X, np_dtype=None):
        """Hidden activation probabilities at the end of the Gibbs chain started
        at ``X`` (the reference's ``transform_op``, base_rbm.py:438-440)."""
        np_dtype = np_dtype or self._np_dtype
        X = np.ascontiguousarray(X, dtype=self._np_dtype)
        H = np.zeros((len(X), self.n_hidden), dtype=np_dtype)
        a = self._step_args()
        for lo, hi in _maybe_bar(batch_bounds(len(X), self.batch_size), self.verbose,
                                 leave=False, ncols=64, desc='transform'):
            H[lo:hi] = self._engine.transform(X[lo:hi], k=a['k'], seed=a['seed'],
                                              tick=self._next_tick())
        return H
