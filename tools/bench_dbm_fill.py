"""Time DBM.fill_missing's clamped Gibbs chains (bm_dbm_fill, DESIGN.md §5.9) on the tensor-core engine.

Per shape, rounds alternate one fill of k sweeps with sample_v(k / 2) on the same card: sample_v sweeps the same number of
chains (n_particles = rows) k times in all (k / 2 committed sweeps, then k / 2 more), so the gap per sweep is what the fill's
extra work costs -- the visible clamp's launch cut and kernel.  Prints one JSON line per shape with the median ms per sweep of
each, and the card's name, power limit and SM clock read in the same call.

    python tools/bench_dbm_fill.py [--rounds R]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'boltzmann-machines_b200')]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def shape_cfg(V, Hs, rows, **kw):
    L = len(Hs)
    c = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
             n_particles=rows, batch_size=rows, max_mf_updates=10, mf_tol=1e-7, l2=0., max_norm=1e300, sample_v=True,
             sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[0.] * L, sparsity_damping=0.9)
    c.update(kw)
    return c


def run(name, c, k, rounds):
    from boltzmann_machines import _native
    e = _native.CudaDBM(c)
    rng = np.random.RandomState(0)
    sizes = [c['n_visible']] + c['n_hiddens']
    d = {'vb': np.zeros(sizes[0], np.float32)}
    for i in range(len(c['n_hiddens'])):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (0.02 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = np.zeros(sizes[i + 1], np.float32)
    e.set_params(d)
    e.init_particles(1)
    rows, V = c['batch_size'], c['n_visible']
    X = (rng.rand(rows, V) < 0.3).astype(np.float32) if c['v_kind'] == 'bernoulli' else rng.randn(rows, V).astype(np.float32)
    mask = np.ones((rows, V), np.uint8)
    mask[:, :V // 2] = 0
    e.fill(X, mask, k=k, seed=1, tick=0)                      # warm-up: programs built, buffers allocated
    e.sample_v(k // 2, 1, 0)
    tf, ts = [], []
    for r in range(rounds):
        t0 = time.perf_counter(); e.fill(X, mask, k=k, seed=2, tick=r); tf.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); e.sample_v(k // 2, 2, r); ts.append(time.perf_counter() - t0)
    e.close()
    out = dict(shape=name, rows=rows, k=k, fill_ms_per_sweep=1e3 * float(np.median(tf)) / k,
               sample_v_ms_per_sweep=1e3 * float(np.median(ts)) / (2 * (k // 2)), rounds=rounds, card=card())
    print(json.dumps(out))
    sys.stdout.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=20)
    a = ap.parse_args()
    run('cfg4 784-512-1024', shape_cfg(784, [512, 1024], 1024), 10, a.rounds)
    run('cfg4 784-512-1024', shape_cfg(784, [512, 1024], 1024), 100, max(3, a.rounds // 4))
    run('dbm_cifar_naive 3072-5000-1000', shape_cfg(3072, [5000, 1000], 100, v_kind='gaussian', sigma=np.ones(3072),
                                                    h_kinds=['bernoulli', 'multinomial'], h_n_samples=[100., 1000.]),
        10, a.rounds)


if __name__ == '__main__':
    main()
