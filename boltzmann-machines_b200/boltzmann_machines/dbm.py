"""Deep Boltzmann Machine: host-side training loop over the native engine.

Interface parity target: /root/reference/boltzmann_machines/dbm.py (constructor kwargs
:89-99, ``load_rbms`` :207-231, composition of the initial weights from pre-trained RBMs
:266-291, epoch/batch loop :793-857, public methods :859-957).  What the reference runs
inside ``session.run`` -- the mean-field E-step, the PCD particle update, gradients,
sparsity, momentum, max-norm, AIS, the variational bound -- happens in the engine
(``bm_dbm_*`` in include/bm.h).

Session semantics: in the reference every public call opens a session, restores the
variables from disk and (unless it saves) throws its changes away.  ``transform``,
``reconstruct``, ``log_proba``, ``log_Z`` and ``sample_v(save_model=False)`` therefore must
not leave traces in the persistent state (variational parameters, particles): they snapshot
and restore it around the call.
"""
import numpy as np

from .base import run_in_tf_session, get_engine_factory
from .ebm import EnergyBasedModel
from .layers import BernoulliLayer
from .utils import (make_list_from, write_during_training, batch_bounds, epoch_iter,
                    log_sum_exp, log_diff_exp, log_mean_exp, log_std_exp)
from .utils.utils import _maybe_bar


def _sfx(i):
    """TF uniquifies repeated variable names: W, W_1, W_2, ... (dbm_mnist.py:367-371)."""
    return '' if i == 0 else '_{0}'.format(i)


class DBM(EnergyBasedModel):
    """Deep Boltzmann Machine trained with PCD and mean-field variational inference.

    Parameters (identical names and meaning to the reference)
    ----------
    rbms : list of pre-trained RBMs, visible side first
    n_particles : number of persistent Markov chains
    v_particle_init, h_particles_init : optional initial particle states
    n_gibbs_steps : PCD sweeps per update (scalar or per-epoch list)
    max_mf_updates, mf_tol : mean-field iteration cap and sup-norm tolerance
    learning_rate, momentum : scalar or per-epoch list
    max_epoch, batch_size : ints (``len(X)`` should be divisible by ``batch_size``)
    l2, max_norm : weight decay; column-norm constraint
    sample_v_states, sample_h_states : bool, list of bool per hidden layer
    sparsity_target, sparsity_cost : scalar or per-layer; sparsity_damping
    train_metrics_every_iter, val_metrics_every_epoch, verbose, save_after_each_epoch
    display_filters, display_particles, v_shape : accepted for compatibility
    pt_betas : None (default), or a ladder of inverse temperatures 1 = b_0 > b_1 > ... > b_{T-1} >= 0 for parallel
        tempering of the persistent chains (not in the reference; Desjardins et al., AISTATS 2010): slot m holds
        ``n_particles`` chains swept at b_m, and every particle update ends with one round of swaps between neighbouring
        slots.  The gradient, ``sample_v`` and the particles ``v`` / ``h...`` are slot 0's.  Needs the tensor-core engine
        (float32, Bernoulli units) and sampled states in every layer; ``pt_swap_rates_`` holds the last epoch's
        acceptance rate of each pair (m, m+1) (None for a pair the epoch did not propose).
    centering : False (default), or True to train the centered DBM (not in the reference; Montavon & Mueller, *Deep
        Boltzmann machines and the centering trick*, 2012): every layer's states are taken relative to an offset, the data
        mean of the layer, which conditions the gradient so that a DBM can be trained from scratch.  The model's
        distribution and every query are those of the stored (W, b); only the training step changes.  The offsets (scope
        ``offsets``) are set from the first batch and then follow an exponential moving average of the batch means with
        rate ``offset_rate`` in [0, 1].  Needs the tensor-core engine (float32); not for ``ClassificationDBM``.
    """
    _MUTABLE_PREFIXES = ('mu', 'v', 'h')

    def __init__(self, rbms=None,
                 n_particles=100, v_particle_init=None, h_particles_init=None,
                 n_gibbs_steps=5, max_mf_updates=10, mf_tol=1e-7,
                 learning_rate=0.0005, momentum=0.9, max_epoch=10, batch_size=100,
                 l2=0., max_norm=np.inf,
                 sample_v_states=True, sample_h_states=None,
                 sparsity_target=0.1, sparsity_cost=0., sparsity_damping=0.9,
                 train_metrics_every_iter=10, val_metrics_every_epoch=1,
                 verbose=False, save_after_each_epoch=True,
                 display_filters=0, display_particles=0, v_shape=(28, 28),
                 model_path='dbm_model/', pt_betas=None, centering=False, offset_rate=0.01, *args, **kwargs):
        super(DBM, self).__init__(model_path=model_path, *args, **kwargs)
        self.n_layers_ = len(rbms) if rbms is not None else None
        self.n_visible_ = None
        self.n_hiddens_ = []
        self.layers_ = None                  # unit kinds/params, persisted so that a loaded model can run
        self._rbms = None
        self.load_rbms(rbms)

        self.n_particles = n_particles
        self._v_particle_init = v_particle_init
        self._h_particles_init = h_particles_init

        self.n_gibbs_steps = make_list_from(n_gibbs_steps)
        self.max_mf_updates = max_mf_updates
        self.mf_tol = mf_tol

        self.learning_rate = make_list_from(learning_rate)
        self.momentum = make_list_from(momentum)
        self.max_epoch = max_epoch
        self.batch_size = batch_size
        self.l2 = l2
        self.max_norm = max_norm

        self.sample_v_states = sample_v_states
        self.sample_h_states = sample_h_states or ([True] * self.n_layers_ if self.n_layers_ else None)

        self.sparsity_target = make_list_from(sparsity_target)
        self.sparsity_cost = make_list_from(sparsity_cost)
        if self.n_layers_ is not None and self.n_layers_ > 1:
            for x in (self.sparsity_target, self.sparsity_cost):
                if len(x) == 1:
                    x *= self.n_layers_
        self.sparsity_damping = sparsity_damping

        self.train_metrics_every_iter = train_metrics_every_iter
        self.val_metrics_every_epoch = val_metrics_every_epoch
        self.verbose = verbose
        self.save_after_each_epoch = save_after_each_epoch

        for nh in self.n_hiddens_:
            assert nh >= display_filters
        self.display_filters = display_filters
        assert display_particles <= self.n_particles
        self.display_particles = display_particles
        self.v_shape = tuple(v_shape)
        if len(self.v_shape) == 2:
            self.v_shape = self.v_shape + (1,)

        self.pt_betas = None if pt_betas is None else [float(b) for b in np.asarray(pt_betas, dtype=np.float64).ravel()]
        self._check_pt()
        self.pt_swap_rates_ = None

        self.centering = bool(centering)
        self.offset_rate = float(offset_rate)
        self._check_centering()

        self.epoch_ = 0
        self.iter_ = 0
        self.n_samples_generated_ = 0

    def _check_pt(self):
        """The refusals of the engine (include/bm.h, bm_dbm_cfg.n_temps) as far as the constructor can tell."""
        if self.pt_betas is None:
            return
        b = self.pt_betas
        if not b or b[0] != 1.0 or not all(np.isfinite(x) for x in b) or any(y >= x for x, y in zip(b, b[1:])) or b[-1] < 0:
            raise ValueError('pt_betas must decrease strictly from 1.0 and stay >= 0, got {0}'.format(b))
        if not self.sample_v_states or not all(self.sample_h_states or []):
            raise ValueError('parallel tempering needs sampled states in every layer (sample_v_states, sample_h_states)')
        if np.dtype(self.dtype) != np.float32:
            raise NotImplementedError('parallel tempering runs on the tensor-core engine: float32 models only')
        if self.layers_ is not None:
            if self.layers_['v']['kind'] != 'bernoulli':
                raise NotImplementedError('parallel tempering is not supported with gaussian visibles')
            if any(h['kind'] != 'bernoulli' for h in self.layers_['h']):
                raise NotImplementedError('parallel tempering is not supported with multinomial hidden layers')

    def _check_centering(self):
        """The refusals of the engine (include/bm.h, bm_dbm_cfg.centering) as far as the constructor can tell."""
        if not (0.0 <= self.offset_rate <= 1.0):
            raise ValueError('offset_rate must lie in [0, 1], got {0}'.format(self.offset_rate))
        if not self.centering:
            return
        if np.dtype(self.dtype) != np.float32:
            raise NotImplementedError('centering runs on the tensor-core engine: float32 models only')

    # ---- composition from pre-trained RBMs (dbm.py:207-231, 266-291) ---------------------
    def load_rbms(self, rbms):
        if rbms is None:
            return
        self._rbms = rbms
        self.n_layers_ = len(rbms)
        self.n_visible_ = rbms[0].n_visible
        self.n_hiddens_ = [rbm.n_hidden for rbm in rbms]
        self._W_init, self._vb_init, self._hb_init = [], [], []
        for rbm in rbms:
            w = rbm.get_tf_params(scope='weights')
            self._W_init.append(w['W']); self._vb_init.append(w['vb']); self._hb_init.append(w['hb'])
        self._v_layer = rbms[0]._v_layer
        self._h_layers = [rbm._h_layer for rbm in rbms]
        self._v_layer.dtype = self.dtype
        for h in self._h_layers:
            h.dtype = self.dtype
        desc = lambda layer: dict(kind=layer.kind, **{k: (np.asarray(v).tolist() if hasattr(v, '__iter__') else v)
                                                      for k, v in layer.engine_params().items()})
        self.layers_ = dict(v=desc(self._v_layer), h=[desc(h) for h in self._h_layers])
        if getattr(self, 'sample_h_states', None) is None:
            self.sample_h_states = [True] * self.n_layers_

    def _composed_init(self):
        """Halve what is counted twice when RBMs are stacked (dbm.py:266-291)."""
        L = self.n_layers_
        W_init, hb_init = [], []
        vb_init = np.array(self._vb_init[0], dtype=self._np_dtype)
        for i in range(L):
            W = np.array(self._W_init[i], dtype=self._np_dtype)
            vb = np.array(self._vb_init[i], dtype=self._np_dtype)
            hb = np.array(self._hb_init[i], dtype=self._np_dtype)
            if 0 < i < L - 1:                  # intermediate RBMs: both directions were doubled
                W *= 0.5; vb *= 0.5; hb *= 0.5
            W_init.append(W)
            if i == 0:
                hb_init.append(0.5 * hb)
            else:
                hb_init[i - 1] = hb_init[i - 1] + 0.5 * vb
                hb_init.append(0.5 * hb if i < L - 1 else hb)
        return vb_init, W_init, hb_init

    # ---- engine wiring ---------------------------------------------------------------------------
    def _scopes(self):
        L = self.n_layers_ or 0
        per = lambda stem: tuple(stem + _sfx(i) for i in range(L))
        tempered = ('v_pt',) + per('h_pt') if self.pt_betas is not None and len(self.pt_betas) > 1 else ()
        return {
            'weights': ('vb',) + per('W') + per('hb'),
            'grads_accumulators': ('dvb',) + per('dW') + per('dhb'),
            'variational_params': per('mu'),
            'hidden_means_accumulators': per('q_means') + per('mu_means'),
            'negative_particles': ('v',) + per('h') + tempered,
            'offsets': ('v_offset',) + per('h_offset') + ('offsets_set',) if self.centering else (),
        }

    def _tf_name(self, scope, name):
        # the hidden particles are created inside `tf.name_scope('h_particle')` (dbm.py:371-383): TF names them
        # negative_particles/h_particle/h, negative_particles/h_particle_1/h, ...
        if scope == 'negative_particles' and name.startswith('h') and not name.startswith('h_pt'):
            i = name[2:]
            return 'h_particle{0}/h'.format('_' + i if i else '')
        return name

    def _engine_cfg(self):
        if self.layers_ is None:
            raise RuntimeError('the DBM has no layer description: call `load_rbms` (or load a saved model)')
        lay = self.layers_
        cfg = dict(
            n_visible=int(self.n_visible_), n_hiddens=[int(h) for h in self.n_hiddens_],
            v_kind=lay['v']['kind'], h_kinds=[h['kind'] for h in lay['h']],
            h_n_samples=[float(h.get('n_samples', 100.)) for h in lay['h']],
            dtype=self.dtype, n_particles=int(self.n_particles), batch_size=int(self.batch_size),
            max_mf_updates=int(self.max_mf_updates), mf_tol=float(self.mf_tol),
            l2=float(self.l2), max_norm=float(self.max_norm),
            sample_v=bool(self.sample_v_states), sample_h=[bool(s) for s in self.sample_h_states],
            sparsity_target=[float(x) for x in self.sparsity_target],
            sparsity_cost=[float(x) for x in self.sparsity_cost],
            sparsity_damping=float(self.sparsity_damping),
        )
        if self.pt_betas is not None:
            cfg['pt_betas'] = list(self.pt_betas)
        if self.centering:
            cfg['centering'] = True
            cfg['offset_rate'] = self.offset_rate
        if 'sigma' in lay['v']:
            cfg['sigma'] = np.broadcast_to(np.asarray(lay['v']['sigma'], dtype=np.float64), (self.n_visible_,)).copy()
        return cfg

    def _make_engine(self):
        return get_engine_factory('dbm')(self._engine_cfg())

    _make_tf_model = _make_engine

    def _init_engine_vars(self):
        if self._rbms is None:
            raise RuntimeError('`load_rbms` must be called before the first `fit`/`init`')
        dt = self._np_dtype
        vb, Ws, hbs = self._composed_init()
        d = {'vb': vb}
        for i in range(self.n_layers_):
            d['W' + _sfx(i)] = Ws[i]
            d['hb' + _sfx(i)] = hbs[i]
        self._engine.set_params(d)
        # persistent particles: the layers' own initialisers unless given (dbm.py:362-383)
        self._engine.init_particles(self.make_random_seed() if self.random_seed is not None
                                    else int(np.random.SeedSequence().generate_state(1)[0]))
        given = {}
        if self._v_particle_init is not None:
            given['v'] = np.asarray(self._v_particle_init, dtype=dt)
        if self._h_particles_init is not None:
            for i, h in enumerate(self._h_particles_init):
                if h is not None:
                    given['h' + _sfx(i)] = np.asarray(h, dtype=dt).reshape(self.n_particles, self.n_hiddens_[i])
        if given:
            self._engine.set_params(given)

    def _snapshot(self):
        names = [n for sc in ('variational_params', 'negative_particles') for n in self._scopes()[sc]]
        return self._engine.get_params(names)

    # ---- schedules -----------------------------------------------------------------------------------
    def _scheduled(self, values):
        return values[min(self.epoch_, len(values) - 1)]

    def _step_args(self, n_gibbs_steps=None):
        k = self._scheduled(self.n_gibbs_steps) if n_gibbs_steps is None else n_gibbs_steps
        return dict(lr=float(self._scheduled(self.learning_rate)), momentum=float(self._scheduled(self.momentum)),
                    k=int(k), seed=self._call_seed)

    # ---- training ------------------------------------------------------------------------------------
    def _train_epoch(self, X):
        pt = self.pt_betas is not None and len(self.pt_betas) > 1
        if pt:
            acc0, prop0 = self._engine.pt_counts()
        msres, n_mfs = [], []
        for lo, hi in _maybe_bar(batch_bounds(len(X), self.batch_size), self.verbose, leave=False, ncols=64, desc='epoch'):
            self.iter_ += 1
            report = ('msre', 'n_mf_updates') if (self.train_metrics_every_iter and
                                                  self.iter_ % self.train_metrics_every_iter == 0) else ()
            got = self._engine.train_step(X[lo:hi], tick=self._next_tick(), metrics=report, **self._step_args())
            if report:
                msres.append(got['msre']); n_mfs.append(got['n_mf_updates'])
                self._log_scalars('train', self.iter_, {'mean_squared_recon_error': got['msre'],        # dbm.py:636-639
                                                        'n_mf_updates': got['n_mf_updates']})
        if pt:                             # the epoch's swap acceptance rate of each neighbouring pair (m, m+1)
            acc1, prop1 = self._engine.pt_counts()
            dp = (prop1 - prop0).astype(np.float64)
            # None for a pair not proposed in the epoch (params.json stays standard JSON)
            self.pt_swap_rates_ = [float(a) / float(p) if p > 0 else None for a, p in zip(acc1 - acc0, dp)]
            self._log_scalars('train', self.iter_, {'pt_swap_acceptance_{0}'.format(m): r
                                                    for m, r in enumerate(self.pt_swap_rates_) if r is not None})
        return (float(np.mean(msres)) if msres else None, float(np.mean(n_mfs)) if n_mfs else None)

    def _run_val_metrics(self, X_val):
        a = self._step_args()
        msres, n_mfs = [], []
        for lo, hi in batch_bounds(len(X_val), self.batch_size):
            got = self._engine.val_metrics(X_val[lo:hi], k=a['k'], seed=a['seed'], tick=self._next_tick())
            msres.append(got['msre']); n_mfs.append(got['n_mf_updates'])
        self._log_scalars('val', self.iter_, {'mean_squared_recon_error': np.mean(msres),              # dbm.py:818-823
                                              'n_mf_updates': np.mean(n_mfs)})
        return float(np.mean(msres)), float(np.mean(n_mfs))

    def _fit(self, X, X_val=None, *args, **kwargs):
        X = np.ascontiguousarray(X, dtype=self._np_dtype)
        if X_val is not None:
            X_val = np.ascontiguousarray(X_val, dtype=self._np_dtype)
        val_msre, val_n_mf = None, None
        for self.epoch_ in epoch_iter(start_epoch=self.epoch_, max_epoch=self.max_epoch, verbose=self.verbose):
            train_msre, train_n_mf = self._train_epoch(X)
            if X_val is not None and self.epoch_ % self.val_metrics_every_epoch == 0:
                val_msre, val_n_mf = self._run_val_metrics(X_val)
            if self.verbose:
                s = 'epoch: {0:{1}}/{2}'.format(self.epoch_, len(str(self.max_epoch)), self.max_epoch)
                if train_msre:
                    s += '; msre: {0:.5f}'.format(train_msre)
                if train_n_mf:
                    s += '; n_mf_upds: {0:.1f}'.format(train_n_mf)
                if val_msre:
                    s += '; val.msre: {0:.5f}'.format(val_msre)
                if val_n_mf:
                    s += '; val.n_mf_upds: {0:.1f}'.format(val_n_mf)
                write_during_training(s)
            if self.save_after_each_epoch:
                self._save_model(global_step=self.epoch_)

    # ---- queries -------------------------------------------------------------------------------------
    def _per_batch(self, X, width, fn, desc, dtype=None):
        X = np.ascontiguousarray(X, dtype=self._np_dtype)
        out = np.zeros((len(X), width) if width else (len(X),), dtype=dtype or self._np_dtype)
        keep = self._snapshot()
        try:
            for lo, hi in _maybe_bar(batch_bounds(len(X), self.batch_size), self.verbose, leave=False, ncols=64, desc=desc):
                out[lo:hi] = fn(X[lo:hi])
        finally:
            self._engine.set_params(keep)
        return out

    @run_in_tf_session()
    def transform(self, X, np_dtype=None):
        """Activation probabilities of the last hidden layer after the mean-field E-step."""
        return self._per_batch(X, self.n_hiddens_[-1], self._engine.transform, 'transform', np_dtype)

    @run_in_tf_session(update_seed=True)
    def reconstruct(self, X):
        """p(v | h_0 = q) with q the mean-field posterior of the first hidden layer."""
        return self._per_batch(X, self.n_visible_, self._engine.reconstruct, 'reconstruction')

    @run_in_tf_session(update_seed=True)
    def sample_v(self, n_gibbs_steps=0, save_model=False):
        """Visible activation probabilities of the particles after ``n_gibbs_steps`` sweeps."""
        keep = None if save_model else self._snapshot()
        v = self._engine.sample_v(int(n_gibbs_steps), self._call_seed, self._next_tick())
        if save_model:
            self.n_samples_generated_ += n_gibbs_steps
            self._save_model()
        else:
            self._engine.set_params(keep)
        return v

    @run_in_tf_session(update_seed=True)
    def fill_missing(self, X, mask, n_gibbs_steps=100):
        """Conditional sampling (DESIGN.md §5.9): fill in the units of X where ``mask`` is 0 with a Gibbs chain that holds
        the units where it is 1 at X.

        Every row runs its own chain: v starts at X where observed and at the visible mean act(vb) elsewhere, the hidden
        layers at the mean-field E-step's first pass on it; then ``n_gibbs_steps`` sweeps of the model's sampler (as the
        persistent chains sweep, with ``sample_v_states`` / ``sample_h_states``), the observed units reset to X after every
        visible update.  Returns the visible means p(v | h_1) of the last sweep [n, n_visible] in the model's dtype, with the
        observed units equal to X.  For binary and sigma = 1 Gaussian visibles the chain samples p(v_missing | v_observed);
        with another sigma the DBM's Gaussian conditionals belong to no joint distribution and it is the engine's Gibbs
        sampler only.  A row's result depends on its own X, mask and index in X and on the call's seed, not on
        ``batch_size``.  The model's variables, accumulators and particles stay as they were.
        """
        return self._fill(X, mask, None, n_gibbs_steps)

    def _fill(self, X, mask, labels, n_gibbs_steps):
        X = np.ascontiguousarray(X, dtype=self._np_dtype)
        if X.ndim != 2 or X.shape[1] != self.n_visible_:
            raise ValueError('X has shape {0}, expected (n, {1})'.format(X.shape, self.n_visible_))
        mask = np.asarray(mask)
        if mask.shape != X.shape:
            raise ValueError('mask has shape {0}, expected {1}'.format(mask.shape, X.shape))
        if not np.all((mask == 0) | (mask == 1)):
            raise ValueError('mask must hold 0 (missing) or 1 (observed) only')
        if not np.all(np.isfinite(X)):
            raise ValueError('X must be finite')
        k = int(n_gibbs_steps)
        if k < 1:
            raise ValueError('n_gibbs_steps must be >= 1')
        mask = np.ascontiguousarray(mask, dtype=np.uint8)
        out = np.empty_like(X)
        tick = self._next_tick()
        for lo, hi in _maybe_bar(batch_bounds(len(X), self.batch_size), self.verbose, leave=False, ncols=64, desc='fill_missing'):
            out[lo:hi] = self._engine.fill(X[lo:hi], mask[lo:hi], labels=None if labels is None else labels[lo:hi],
                                           row0=lo, k=k, seed=self._call_seed, tick=tick)
        return out

    @run_in_tf_session(update_seed=True)
    def log_Z(self, n_betas=100, n_runs=100, n_gibbs_steps=5, base_rate=None):
        """Annealed-importance-sampling estimate of the log partition function of a binary DBM.

        The chains run over the odd hidden layers h_1, h_3, ...; v and the even layers are summed out analytically
        (DESIGN.md §5.4c).  Two hidden layers run on either engine.  Any other number of layers runs on the tensor-core
        engine (float32 models, ``compute='bf16'``), with the odd layers sampled (``sample_h_states``); otherwise
        ``NotImplementedError`` names what is missing.  Tempered and centered models need nothing extra.

        ``base_rate`` starts the ladder from a factorial base-rate model instead of the uniform one (DESIGN.md §5.4d;
        Salakhutdinov & Hinton 2009), which needs far fewer temperatures for a model of data whose units are mostly off:
          * None: the uniform start;
          * a training-data array ``X`` [n, n_visible] with values in [0, 1]: visible base biases
            logit((sum_r X_r + 1) / (n + 2)), hidden layers uniform;
          * a list or tuple of ``n_layers + 1`` entries (v, h_1 .. h_L), each None (uniform) or the layer's base biases.
        A base runs on the tensor-core engine at every depth, with the odd layers sampled.

        Returns ``log_mean, (log_low, log_high), values``: log of the mean estimate, of the mean
        minus / plus one standard deviation, and the ``n_runs`` individual estimates (log Z_A included).
        """
        base = self._base_rates(base_rate) if base_rate is not None else None
        if base is not None:
            self._check_depth('log_Z from a base-rate model', ais=True)
        elif self.n_layers_ == 2:
            assert self.layers_['v']['kind'] == 'bernoulli' and all(h['kind'] == 'bernoulli' for h in self.layers_['h'])
        else:
            self._check_depth('log_Z', ais=True)
        ais_seed = self.make_random_seed()           # dbm.py:701
        if base is None:
            values = self._engine.ais(int(n_runs), int(n_betas), int(n_gibbs_steps), ais_seed)
        else:
            values = self._engine.ais(int(n_runs), int(n_betas), int(n_gibbs_steps), ais_seed, base=base)
        log_mean = log_mean_exp(values)
        log_std = log_std_exp(values, log_mean_exp_x=log_mean)
        log_high = log_sum_exp([log_std, log_mean])
        log_low = log_diff_exp([log_std, log_mean])[0]
        return log_mean, (log_low, log_high), values

    @run_in_tf_session()
    def log_proba(self, X_test, log_Z):
        """Variational lower bound on log p(v) for the rows of ``X_test`` given an estimate of log Z.

        Two hidden layers run on either engine; any other number of binary layers on the tensor-core engine (float32
        models, ``compute='bf16'``), as for `log_Z`."""
        if self.n_layers_ == 2:
            assert self.layers_['v']['kind'] == 'bernoulli' and all(h['kind'] == 'bernoulli' for h in self.layers_['h'])
        else:
            self._check_depth('log_proba', ais=False)
        P = self._per_batch(X_test, 0, self._engine.log_proba, 'log_proba', np.float64)
        return P - log_Z

    @run_in_tf_session()
    def exact_log_Z(self):
        """Exact log partition function of a binary DBM whose odd hidden layers h_1, h_3, ... hold at most 32 units together.

        Every state of the odd layers is enumerated on the tensor-core engine, with v and the even layers summed out
        analytically (DESIGN.md §5.4f), for the model as stored (float32 weights and biases).  A one-layer DBM is an RBM
        with at most 32 hidden units.  Tempered and centered models need nothing extra.  Refusals raise
        ``NotImplementedError`` naming the reason: non-binary layers, float64 models, ``compute='fp32'``, a
        `ClassificationDBM`, or more than 32 odd-layer units."""
        self._check_exact('exact_log_Z')
        return float(self._engine.exact(None)[1])

    @run_in_tf_session()
    def exact_log_proba(self, X_test, log_Z=None):
        """Exact log p(v) = log p*(v) - log Z of the rows of ``X_test`` [n, n_visible] (float64 [n]), for the models
        `exact_log_Z` accepts.  The values of X are used as given, as in `log_proba`: for binary rows this is log p(v).
        ``log_Z=None`` takes the exact log Z from the same enumeration.  Each slice of up to 16384 rows is one pass over
        the states."""
        self._check_exact('exact_log_proba')
        X = np.asarray(X_test, dtype=np.float32)
        if X.ndim != 2 or X.shape[1] != self.n_visible_:
            raise ValueError('X_test has shape {0}, expected (n, {1})'.format(X.shape, self.n_visible_))
        if not np.all(np.isfinite(X)):
            raise ValueError('X_test must be finite')
        out = np.empty(len(X), dtype=np.float64)
        for lo in range(0, len(X), self._EXACT_ROWS):
            hi = min(len(X), lo + self._EXACT_ROWS)
            out[lo:hi], lz = self._engine.exact(X[lo:hi])
            if log_Z is None:
                log_Z = lz
        if log_Z is None:                              # no rows
            log_Z = self._engine.exact(None)[1]
        return out - float(log_Z)

    _EXACT_ROWS = 16384

    @run_in_tf_session(update_seed=True)
    def ais_log_proba(self, X_test, log_Z, n_betas=100, n_runs=100, n_gibbs_steps=5, return_runs=False):
        """AIS estimate of log p(v) for the rows of ``X_test`` [n, n_visible] given an estimate of log Z (DESIGN.md §5.4g;
        Salakhutdinov & Hinton 2009).

        Each row runs ``n_runs`` AIS chains with v clamped to it: the odd hidden layers h_1, h_3, ... are summed out
        analytically and the even ones are annealed from the uniform model to the DBM, with the temperatures and sweeps of
        `log_Z` (whose defaults these are, so the two read alike; trained models want far more temperatures than 100).  Like
        `log_Z`'s ladder it weighs each state at the temperature it was just drawn at, which biases the estimate up by
        O(1 / n_betas): +0.08 nats at 1000 temperatures on a trained 784-24-1000 model, +0.8 at 100.  `log_proba`'s bound
        sits below log p(v) by the variational gap instead.  Every layer the chains draw is sampled, whatever
        ``sample_h_states`` says.  The values of X are used as given, as in `log_proba`; grey rows enter the products as bf16.
        A one-layer DBM has nothing to anneal: every run is `log_proba`'s value, which is exact there.

        Runs on the tensor-core engine (float32 models, ``compute='bf16'``) with binary layers; otherwise
        ``NotImplementedError`` names what is missing.  Tempered and centered models need nothing extra.  A row's runs
        depend only on its index in ``X_test`` and the call's seed.  Returns float64 [n]: each row's log-mean-exp over its
        runs minus ``log_Z``; with ``return_runs=True`` also the [n, n_runs] per-run estimates of log p*(v).
        """
        self._check_depth('ais_log_proba', ais=False, clamped=True)
        X = np.asarray(X_test, dtype=np.float32)
        if X.ndim != 2 or X.shape[1] != self.n_visible_:
            raise ValueError('X_test has shape {0}, expected (n, {1})'.format(X.shape, self.n_visible_))
        if not np.all(np.isfinite(X)):
            raise ValueError('X_test must be finite')
        n_runs, n_betas, k = int(n_runs), int(n_betas), int(n_gibbs_steps)
        if n_runs < 1 or n_betas < 2 or k < 1:
            raise ValueError('ais_log_proba needs n_runs >= 1, n_betas >= 2 and n_gibbs_steps >= 1')
        seed = self.make_random_seed()
        runs = np.empty((len(X), n_runs), dtype=np.float64)
        step = max(1, self._AIS_CLAMPED_CHAINS // n_runs)
        keep = self._snapshot() if self.n_layers_ == 1 else None      # one layer: the engine's log_proba writes the E-step's means
        try:
            for lo in range(0, len(X), step):
                hi = min(len(X), lo + step)
                runs[lo:hi] = self._engine.ais_clamped(X[lo:hi], n_runs, n_betas, k, seed, row0=lo)
        finally:
            if keep is not None:
                self._engine.set_params(keep)
        m = runs.max(axis=1, keepdims=True)
        est = (m[:, 0] + np.log(np.mean(np.exp(runs - m), axis=1))) - float(log_Z)
        return (est, runs) if return_runs else est

    # chains per engine call of ais_log_proba (DbmTC::AIS_CLAMPED_CHAINS: one ladder slice; at least log_Z's 20 000 runs)
    _AIS_CLAMPED_CHAINS = 32768

    def _check_exact(self, what):
        """The refusals of bm_dbm_exact (include/bm.h), raised before the engine is called."""
        if self.layers_['v']['kind'] != 'bernoulli' or any(h['kind'] != 'bernoulli' for h in self.layers_['h']):
            raise NotImplementedError(what + ' is defined for binary layers (Bernoulli visible and hidden units)')
        if np.dtype(self.dtype) != np.float32:
            raise NotImplementedError(what + ' runs on the tensor-core engine: float32 models only')
        if getattr(self._engine, 'compute', 'bf16') != 'bf16':
            raise NotImplementedError(what + " runs on the tensor-core engine, not on the fp32 CUDA-core engine (compute='fp32')")
        n_odd = sum(int(n) for n in self.n_hiddens_[0::2])
        if n_odd > 32:
            raise NotImplementedError('{0} enumerates the odd layers h_1, h_3, ...: n_odd = {1} units, at most 32'.format(what, n_odd))

    def _base_rates(self, base_rate):
        """log_Z's ``base_rate`` as one float32 vector or None per unit layer (v, h_1 .. h_L)"""
        widths = [self.n_visible_] + [int(n) for n in self.n_hiddens_]
        if isinstance(base_rate, (list, tuple)):
            if len(base_rate) != len(widths):
                raise ValueError('base_rate: {0} per-layer entries (v, h_1 .. h_L), got {1}'.format(len(widths), len(base_rate)))
            base = []
            for j, a in enumerate(base_rate):
                if a is not None:
                    a = np.asarray(a, dtype=np.float64).ravel()
                    if a.size != widths[j]:
                        raise ValueError('base_rate[{0}] has {1} entries, layer {0} has {2} units'.format(j, a.size, widths[j]))
                    if not np.all(np.isfinite(a)):
                        raise ValueError('base_rate[{0}] has non-finite entries'.format(j))
                    a = a.astype(np.float32)
                base.append(a)
            return base
        X = np.asarray(base_rate, dtype=np.float64)
        if X.ndim != 2 or X.shape[1] != widths[0] or X.shape[0] < 1:
            raise ValueError('base_rate: data [n, {0}] or {1} per-layer vectors (v, h_1 .. h_L), got shape {2}'.format(
                widths[0], len(widths), X.shape))
        if not np.all((X >= 0.) & (X <= 1.)):
            raise ValueError('base_rate: data values must lie in [0, 1]')
        p = (X.sum(axis=0) + 1.) / (X.shape[0] + 2.)
        return [np.log(p / (1. - p)).astype(np.float32)] + [None] * self.n_layers_

    def _check_depth(self, what, ais, clamped=False):
        """The refusals of the engine (include/bm.h, bm_dbm_ais / bm_dbm_ais_base / bm_dbm_log_proba) at a depth other than 2,
        of AIS from a base-rate model at any depth and, with ``clamped``, of bm_dbm_ais_clamped at any depth."""
        where = what if ('base-rate' in what or clamped) else '{0} at {1} hidden layers'.format(what, self.n_layers_)
        if self.layers_['v']['kind'] != 'bernoulli' or any(h['kind'] != 'bernoulli' for h in self.layers_['h']):
            raise NotImplementedError(where + ' is defined for binary layers (Bernoulli visible and hidden units)')
        if np.dtype(self.dtype) != np.float32:
            raise NotImplementedError(where + ' runs on the tensor-core engine: float32 models only')
        if getattr(self._engine, 'compute', 'bf16') != 'bf16':
            raise NotImplementedError(where + " runs on the tensor-core engine, not on the fp32 CUDA-core engine (compute='fp32')")
        if ais and not all(self.sample_h_states[0::2]):
            raise NotImplementedError(where + ' needs sampled states in the odd layers h_1, h_3, ... (sample_h_states)')
