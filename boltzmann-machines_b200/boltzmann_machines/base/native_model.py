"""Runtime shim between the model classes and the native engine.

Plays the role of the reference's ``TensorFlowModel``
(/root/reference/boltzmann_machines/base/tf_model.py:10-202): the same public
methods (``init``, ``fit``, ``load_model``, ``get_tf_params``,
``update_working_paths``, ``compute_working_paths``), the same on-disk layout
(``params.json`` + ``random_state.json`` next to the weights) and the same
error behaviour (``RuntimeError`` before ``fit``/``init``), but instead of a
``tf.Session`` a decorated call runs against an *engine*: a handle into
``libbm.so`` (hand-written sm_90a CUDA behind the C-ABI of ``include/bm.h``).

The engine is produced by a factory looked up in ``ENGINE_FACTORIES``.  The
default factories come from ``boltzmann_machines._native`` and raise loudly when
the CUDA library or a GPU is missing -- there is no CPU fallback in this
package.  The test-suite swaps in its numpy oracle through
``set_engine_factory`` to exercise this host logic without a GPU.
"""
import os
import json
import glob
from functools import wraps

import numpy as np

from .base import is_param_name
from .base_model import BaseModel
from .mixin import DtypeMixin

ENGINE_FACTORIES = {}
_FALLBACK_SEED = 0x5EED5EED


def set_engine_factory(kind, factory):
    """Register ``factory(cfg) -> engine`` for ``kind`` in {'rbm', 'dbm'}.
    Returns the previous factory (``None`` = built-in CUDA engine)."""
    old = ENGINE_FACTORIES.get(kind)
    if factory is None:
        ENGINE_FACTORIES.pop(kind, None)
    else:
        ENGINE_FACTORIES[kind] = factory
    return old


def get_engine_factory(kind):
    f = ENGINE_FACTORIES.get(kind)
    if f is None:
        from .. import _native          # raises if libbm.so is absent
        f = _native.default_factory(kind)
    return f


def run_in_tf_session(check_initialized=True, update_seed=False):
    """Decorator for public model methods (name kept from tf_model.py:10-40).

    Before the wrapped method runs: draw the per-call seed (``update_seed``),
    rewind the per-call draw counter, and make sure an engine exists -- restored
    from ``<model_path>`` if the model was initialised earlier, freshly built
    (``check_initialized=False``) otherwise.
    """
    def wrap(f):
        @wraps(f)
        def wrapped_f(model, *args, **kwargs):
            model._call_seed = model.make_random_seed() if update_seed else _FALLBACK_SEED
            model._tick = 0
            if model._engine is None:
                if model.initialized_:
                    model._engine = model._make_engine()
                    model._restore_engine()
                elif check_initialized:
                    raise RuntimeError('`fit` or `init` must be called before calling `{0}`'
                                       .format(f.__name__))
                else:
                    model._engine = model._make_engine()
                    model._init_engine_vars()
            try:
                return f(model, *args, **kwargs)
            finally:
                model._flush_scalars()          # the scalar logs of the call are on disk when it returns
        return wrapped_f
    return wrap


run_in_session = run_in_tf_session


class NativeModel(BaseModel, DtypeMixin):
    # scope name -> variable names, in the order the reference creates them
    _SCOPES = {}

    def __init__(self, model_path='tf_model/', paths=None,
                 tf_session_config=None, tf_saver_params=None, json_params=None,
                 *args, **kwargs):
        super(NativeModel, self).__init__(*args, **kwargs)
        self._model_dirpath = None
        self._model_filepath = None
        self._params_filepath = None
        self._random_state_filepath = None
        self._train_summary_dirpath = None
        self._val_summary_dirpath = None
        self._tf_meta_graph_filepath = None
        self.update_working_paths(model_path=model_path, paths=paths)

        self._tf_session_config = tf_session_config   # accepted, unused (no TF)
        self.tf_saver_params = tf_saver_params or {}
        self.json_params = json_params or {}
        self.json_params.setdefault('sort_keys', True)
        self.json_params.setdefault('indent', 4)
        self.initialized_ = False

        self._engine = None
        self._call_seed = _FALLBACK_SEED
        self._tick = 0

    # ---- paths (tf_model.py:71-99) -----------------------------------------
    @staticmethod
    def compute_working_paths(model_path):
        """``model_path`` is a directory (trailing slash) or a file path."""
        head, tail = os.path.split(model_path)
        head = head or '.'
        if not head.endswith('/'):
            head += '/'
        tail = tail or 'model'
        model_filepath = os.path.join(head, tail)
        return {
            'model_dirpath': head,
            'model_filepath': model_filepath,
            'params_filepath': os.path.join(head, 'params.json'),
            'random_state_filepath': os.path.join(head, 'random_state.json'),
            'train_summary_dirpath': os.path.join(head, 'logs/train'),
            'val_summary_dirpath': os.path.join(head, 'logs/val'),
            'tf_meta_graph_filepath': model_filepath + '.meta',
        }

    def update_working_paths(self, model_path=None, paths=None):
        paths = paths or NativeModel.compute_working_paths(model_path=model_path)
        for k, v in paths.items():
            setattr(self, '_' + k, v)

    # ---- hooks for subclasses ------------------------------------------------
    def _make_engine(self):
        raise NotImplementedError('`_make_engine` is not implemented')

    def _init_engine_vars(self):
        """Push initial values of every engine variable (fresh model)."""
        raise NotImplementedError('`_init_engine_vars` is not implemented')

    def _fit(self, X, X_val=None, *args, **kwargs):
        raise NotImplementedError('`fit` is not implemented')

    def _next_tick(self):
        t = self._tick
        self._tick += 1
        return t

    # ---- persistence (tf_model.py:117-162) -----------------------------------
    def _weights_filepath(self, global_step=None):
        base = self._model_filepath
        if global_step is not None:
            base = '{0}-{1}'.format(base, global_step)
        return base + '.npz'

    def _restore_engine(self):
        path = self._weights_filepath()
        if not os.path.isfile(path):
            raise RuntimeError("no saved weights at '{0}'".format(path))
        with np.load(path) as z:
            self._engine.set_params({k: z[k] for k in z.files})

    # ---- scalar summaries (tf_model.py:110-115: tf.summary.FileWriter on logs/train, logs/val) ----------
    def _log_scalars(self, kind, step, values, allow_empty=False):
        """Append ``{"step": step, tag: value, ...}`` to ``<model>/logs/<kind>/scalars.jsonl`` -- the
        scalar summaries the reference hands to its TensorBoard writers, as one JSON object per line
        (``kind`` in {'train', 'val'}; tags are the reference's summary tags)."""
        values = {k: float(v) for k, v in values.items() if v is not None}
        if not values and not allow_empty:
            return
        rec = {'step': int(step)}
        rec.update(values)
        # buffered: one append per public call (or per 4096 records), not one open / write / close per training iteration
        buf = self.__dict__.setdefault('_scalar_buf', {'train': [], 'val': []})
        buf[kind].append(json.dumps(rec, sort_keys=True))
        if len(buf[kind]) >= 4096:
            self._flush_scalars()

    def _flush_scalars(self):
        buf = self.__dict__.get('_scalar_buf')
        if not buf:
            return
        for kind, lines in buf.items():
            if not lines:
                continue
            d = self._train_summary_dirpath if kind == 'train' else self._val_summary_dirpath
            if not os.path.isdir(d):
                os.makedirs(d)
            with open(os.path.join(d, 'scalars.jsonl'), 'a') as fh:
                fh.write('\n'.join(lines) + '\n')
            del lines[:]

    def _save_model(self, global_step=None):
        for d in (self._train_summary_dirpath, self._val_summary_dirpath):
            if not os.path.exists(d):
                os.makedirs(d)

        params = self._serialize(self.get_params(deep=False))
        params['__class_name__'] = self.__class__.__name__
        with open(self._params_filepath, 'w') as fh:
            json.dump(params, fh, **self.json_params)

        if self.random_seed is not None:
            with open(self._random_state_filepath, 'w') as fh:
                json.dump(self._rng.get_state(), fh)

        state = self._engine.get_params()
        np.savez(self._weights_filepath(), **state)
        if global_step is not None:
            np.savez(self._weights_filepath(global_step), **state)
            keep = self.tf_saver_params.get('max_to_keep', 5)
            if keep:
                old = sorted(glob.glob(self._model_filepath + '-*.npz'),
                             key=lambda p: int(p[len(self._model_filepath) + 1:-4]))
                for p in old[:-keep]:
                    os.remove(p)

    @classmethod
    def load_model(cls, model_path):
        paths = NativeModel.compute_working_paths(model_path)
        with open(paths['params_filepath'], 'r') as fh:
            params = json.load(fh)
        class_name = params.pop('__class_name__')
        if class_name != cls.__name__:
            raise RuntimeError("attempt to load {0} with class {1}".format(class_name, cls.__name__))
        model = cls(paths=paths, **{k: params[k] for k in params if is_param_name(k)})
        model.set_params(**model._deserialize(params))
        if os.path.isfile(model._random_state_filepath):
            with open(model._random_state_filepath, 'r') as fh:
                model._rng.set_state(json.load(fh))
        return model       # the engine is created lazily by the next decorated call

    # ---- public API -----------------------------------------------------------
    @run_in_tf_session(check_initialized=False)
    def init(self):
        if not self.initialized_:
            self.initialized_ = True
            self._save_model()
        return self

    @run_in_tf_session(check_initialized=False, update_seed=True)
    def fit(self, X, X_val=None, *args, **kwargs):
        """Fit the model to the training data (validation data optional)."""
        self.initialized_ = True
        self._fit(X, X_val=X_val, *args, **kwargs)
        self._save_model()
        return self

    @run_in_tf_session()
    def get_tf_params(self, scope=None):
        """Engine variables as numpy arrays.  With ``scope`` the keys are bare
        variable names (``W, vb, hb`` for ``'weights'``); without, they are
        ``'<scope>/<name>'`` like TF's global-variable names."""
        state = self._engine.get_params()
        out = {}
        for sc, names in self._scopes().items():
            if scope and scope not in sc:
                continue
            for n in names:
                if n in state:
                    shown = self._tf_name(sc, n)
                    out[shown if scope else '{0}/{1}'.format(sc, shown)] = state[n]
        return out

    def _tf_name(self, scope, name):
        """Key under which the reference's ``get_tf_params`` reports engine variable ``name`` (TF variable name
        minus the scope prefix); identical to the engine's name unless a subclass says otherwise."""
        return name

    def _scopes(self):
        return self._SCOPES

    def close(self):
        """Release the engine (device memory).  The model stays usable: the next
        call restores from disk."""
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# name used by the reference's class hierarchy and tests
TensorFlowModel = NativeModel
