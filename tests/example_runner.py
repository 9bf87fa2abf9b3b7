"""TEST INFRASTRUCTURE: runs the reference's example scripts (examples/rbm_mnist.py, examples/dbm_mnist.py) UNCHANGED against
this repository's `boltzmann_machines` package.

The scripts are Python 2 (print statements, tuple parameters) and import Keras and an MNIST loader, none of which exist in
this image, so the runner
  * reads the script from the reference checkout (never copied into the repository) and rewrites, in memory, exactly the two
    Python-2 constructs the examples use -- `print x` statements and tuple parameters in `def` headers;
  * provides stand-ins for what is out of scope of the hot path (SURVEY.md section 8): `keras` (the MLP fine-tuning: fit is a
    no-op, predict is uniform), `boltzmann_machines.utils.dataset.load_mnist` (synthetic binary 'MNIST'), the Keras optimizer
    `MultiAdam`, and the examples' `env` path shim;
  * executes the script as `__main__` with the given command line.
Everything the script does with BernoulliRBM / DBM -- constructor keywords, fit, transform, load_model, load_rbms,
get_tf_params -- goes through the package under test.
"""
import ast
import os
import re
import sys
import types

import numpy as np


# ---- Python 2 -> 3, for the constructs the examples use ------------------------------------------------------------------
def _split_top_level(text):
    parts, depth, cur = [], 0, ''
    for ch in text:
        if ch in '([{':
            depth += 1
        elif ch in ')]}':
            depth -= 1
        if ch == ',' and depth == 0:
            parts.append(cur)
            cur = ''
        else:
            cur += ch
    if cur.strip():
        parts.append(cur)
    return parts


def translate(src):
    """`print x` -> `print(x)`; `def f((a, b), c):` -> `def f(_t0, c):` + `a, b = _t0` as the first statement."""
    out, lines, i = [], src.split('\n'), 0
    while i < len(lines):
        line = lines[i]
        m = re.match(r'^(\s*)print\s+(?!\()(.*\S)\s*$', line) or re.match(r'^(\s*)print\s+(\(.*\)\s*%.*|".*)$', line)
        if m and not line.lstrip().startswith('#'):
            out.append('{0}print({1})'.format(m.group(1), m.group(2)))
            i += 1
            continue
        if re.match(r'^\s*def\s+\w+\s*\(', line):
            header, j = line, i
            while header.count('(') != header.count(')') or not header.rstrip().endswith(':'):
                j += 1
                header += '\n' + lines[j]
            indent = re.match(r'^(\s*)', line).group(1)
            name, rest = re.match(r'^\s*def\s+(\w+)\s*\((.*)\)\s*:\s*$', header, flags=re.S).groups()
            args, unpack = [], []
            for a in _split_top_level(rest):
                a = a.strip()
                if a.startswith('('):
                    tmp = '_t{0}'.format(len(unpack))
                    unpack.append('{0}    {1} = {2}'.format(indent, a, tmp))
                    args.append(tmp)
                elif a:
                    args.append(a)
            out.append('{0}def {1}({2}):'.format(indent, name, ', '.join(args)))
            out.extend(unpack)
            i = j + 1
            continue
        out.append(line)
        i += 1
    return '\n'.join(out)


# ---- stand-ins ---------------------------------------------------------------------------------------------------------
def synthetic_mnist(n, seed):
    """binary 'digits' in 0 / 255 from a random 784-32 teacher RBM + labels derived from the hidden code"""
    rng = np.random.RandomState(seed)
    W = 0.6 * rng.randn(784, 32)
    h = (rng.rand(n, 32) < 0.5).astype(np.float64)
    p = 1.0 / (1.0 + np.exp(-(h @ W.T - 2.0)))
    X = (rng.rand(n, 784) < p).astype(np.float32) * 255.0
    y = (h[:, :4] @ np.array([1, 2, 4, 8])).astype(np.int64) % 10
    return X, y


def _stub_modules(n_train, n_test):
    mods = {}

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        mods[name] = m
        return m

    class Layer(object):
        def __init__(self, *a, **kw):
            self.units = a[0] if a else None
            w = kw.get('weights')
            self._weights = [np.asarray(w[0]), np.asarray(w[1])] if w is not None else [np.zeros((1, 1)), np.zeros(1)]

        def get_weights(self):
            return self._weights

    class Sequential(object):
        def __init__(self, layers=()):
            self.layers = list(layers)

        def compile(self, *a, **kw):
            pass

        def fit(self, *a, **kw):
            print('[stand-in keras] MLP fine-tuning is out of scope: fit() skipped')

        def predict(self, X):
            return np.full((len(X), 10), 0.1)

    class Anything(object):
        def __init__(self, *a, **kw):
            pass

    keras = mod('keras')
    keras.regularizers = mod('keras.regularizers', l2=lambda *a, **kw: None)
    keras.callbacks = mod('keras.callbacks', EarlyStopping=Anything, ReduceLROnPlateau=Anything)
    keras.initializers = mod('keras.initializers', glorot_uniform=lambda *a, **kw: None)
    keras.models = mod('keras.models', Sequential=Sequential)
    keras.layers = mod('keras.layers', Dense=Layer, Activation=Layer)
    mod('env')

    def load_mnist(mode='train', path='.'):
        return synthetic_mnist(n_train if mode == 'train' else n_test, 7 if mode == 'train' else 8)
    mod('boltzmann_machines.utils.dataset', load_mnist=load_mnist)
    mod('boltzmann_machines.utils.optimizers', MultiAdam=Anything)
    return mods


def run_example(path, argv, n_train=640, n_test=128):
    """Executes the example at `path` as __main__ with command line `argv`.  Returns the script's globals.

    No test calls it: the examples are the reference project's source and are not stored here.  It is kept for running them by
    hand against a checkout of the reference, e.g. `run_example('<checkout>/examples/rbm_mnist.py', ['--n-train', '512'])`."""
    src = open(path).read()
    py3 = translate(src)
    code = compile(py3, path, 'exec')
    stubs = _stub_modules(n_train, n_test)
    saved = {k: sys.modules.get(k) for k in stubs}
    old_argv = sys.argv
    sys.modules.update(stubs)
    sys.argv = [os.path.basename(path)] + list(argv)
    g = {'__name__': '__main__', '__file__': path, '__doc__': ast.get_docstring(ast.parse(py3))}
    try:
        exec(code, g)
    finally:
        sys.argv = old_argv
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return g
