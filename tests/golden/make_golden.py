"""Generates tests/golden/reference_utils.json by IMPORTING the reference's own modules.

Needs a checkout of yell/boltzmann-machines, named by the BM_REFERENCE_DIR environment variable:

    python tests/golden/make_golden.py

The reference's compute path (TensorFlow 1.3 graphs) cannot be imported here; the parts of the path that are plain
numpy can: `boltzmann_machines/utils/utils.py` (batching + the log-domain statistics that post-process the AIS
log-weights, dbm.py:843-870) and `boltzmann_machines/utils/rng.py` (the host RNG whose draws seed every run_in_tf_session
call and whose state is persisted in random_state.json).  Their outputs on seeded inputs are the golden vectors the
host mirror (boltzmann-machines_b200/boltzmann_machines/utils) is compared with in tests/test_golden_utils.py.
"""
import importlib.util
import json
import os

import numpy as np

REF = os.path.join(os.environ['BM_REFERENCE_DIR'], 'boltzmann_machines', 'utils')
HERE = os.path.dirname(os.path.abspath(__file__))


def load(name):
    spec = importlib.util.spec_from_file_location('ref_' + name, os.path.join(REF, name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    U, R = load('utils'), load('rng')
    rng = np.random.RandomState(20260923)
    out = {'source': 'yell/boltzmann-machines boltzmann_machines/utils/{utils,rng}.py, imported unmodified', 'log_stats': [],
           'batch_iter': [], 'epoch_iter': [], 'make_list_from': [], 'one_hot': [], 'rng': []}
    # log-domain statistics on AIS-like log-weights (large offsets, wide spread)
    for n, loc, scale in ((1, 0., 1.), (5, 0., 1.), (64, 330., 4.), (1000, -750., 25.), (20000, 431.2, 2.5)):
        x = (loc + scale * rng.randn(n)).astype(np.float64)
        rec = {'x_seed': [n, loc, scale], 'x': x.tolist() if n <= 64 else None,
               'log_sum_exp': float(U.log_sum_exp(x)), 'log_mean_exp': float(U.log_mean_exp(x))}
        if n > 1:
            rec['log_std_exp'] = float(U.log_std_exp(x))
            xs = np.sort(x)
            rec['log_diff_exp_sorted_head'] = [float(v) for v in U.log_diff_exp(xs)[:8]]
        out['log_stats'].append(rec)
    for n, bs in ((10, 3), (7, 7), (5, 8), (1, 1), (12, 4)):
        X = np.arange(n * 2).reshape(n, 2)
        out['batch_iter'].append({'n': n, 'batch_size': bs,
                                  'batches': [b.tolist() for b in U.batch_iter(X, batch_size=bs)]})
    for s, m in ((0, 3), (2, 5), (4, 4)):
        out['epoch_iter'].append({'start': s, 'max': m, 'epochs': [int(e) for e in U.epoch_iter(s, m)]})
    for v in (3, 0.5, [1, 2], (4,), 'ab'):
        try:
            out['make_list_from'].append({'in': v if not isinstance(v, tuple) else list(v), 'tuple': isinstance(v, tuple),
                                          'out': list(U.make_list_from(v))})
        except Exception as e:          # pragma: no cover
            out['make_list_from'].append({'in': repr(v), 'error': type(e).__name__})
    y = [2, 0, 1, 2]
    out['one_hot'].append({'y': y, 'one_hot': np.asarray(U.one_hot(y)).tolist(),
                           'unhot': np.asarray(U.unhot(U.one_hot(y))).tolist()})
    for seed in (1337, 0, 42):
        g = R.RNG(seed=seed)
        rec = {'seed': seed, 'rand3': [float(v) for v in g.rand(3)],
               # SeedMixin.make_random_seed (base/mixin.py:34-35) draws exactly this from the model's RNG
               'make_random_seed': [int(g.randint(2 ** 31 - 1)) for _ in range(3)]}
        state = g.get_state()
        rec['next_after_state'] = float(g.rand())
        g2 = R.RNG(seed=None)
        g2.set_state(json.loads(json.dumps(state)))
        rec['replayed_after_state'] = float(g2.rand())
        rec['reseeded_first'] = float(g.reseed().rand()) if hasattr(g, 'reseed') else None
        out['rng'].append(rec)
    with open(os.path.join(HERE, 'reference_utils.json'), 'w') as fh:
        json.dump(out, fh, indent=1, sort_keys=True)
    print('wrote', os.path.join(HERE, 'reference_utils.json'))


if __name__ == '__main__':
    main()
