"""Time the tensor-core engine's AIS ladder (bm_dbm_ais, DESIGN.md §5.4c) at one, two and three hidden layers at MNIST widths.

Per depth: one warm-up ladder, then `--rounds` ladders of `--runs` runs and `--betas` temperatures (k = 1); prints one JSON
line per depth with the median ms per temperature, the algorithmic GFLOP per temperature (4 sum_i n_{i-1} n_i per run: each
W is read by one summed-out op and one state op) and the card's name, power limit and SM clock read in the same call.
L = 2 runs the two-layer ladder (DbmTC::ais_local), L = 1 and 3 the ladder of any depth (DbmTC::ais_local_layers).

    python tools/bench_dbm_ais_depth.py [--runs 20000] [--betas 200] [--rounds 5]
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

SHAPES = {1: (784, [500]), 2: (784, [500, 1000]), 3: (784, [500, 500, 1000])}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def run(L, runs, betas, rounds):
    from boltzmann_machines import _native
    V, Hs = SHAPES[L]
    c = dict(n_visible=V, n_hiddens=Hs, v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
             n_particles=16, batch_size=16, max_mf_updates=10, mf_tol=1e-7, l2=0., max_norm=1e300, sample_v=True,
             sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[0.] * L, sparsity_damping=0.9)
    e = _native.CudaDBM(c)
    assert e.compute == 'bf16'
    rng = np.random.RandomState(0)
    sizes = [V] + Hs
    d = {'vb': np.zeros(V, np.float32)}
    for i in range(L):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (0.02 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = np.zeros(sizes[i + 1], np.float32)
    e.set_params(d)
    e.ais(runs, betas, 1, 1)                                  # warm-up: modules loaded, descriptors built
    ts = []
    for r in range(rounds):
        t0 = time.perf_counter()
        e.ais(runs, betas, 1, 2 + r)                          # returns after the device synchronises
        ts.append(time.perf_counter() - t0)
    e.close()
    gflop = 4.0 * sum(sizes[i] * sizes[i + 1] for i in range(L)) * runs / 1e9
    ms = 1e3 * float(np.median(ts)) / betas
    print(json.dumps(dict(layers=L, shape='-'.join(map(str, sizes)), runs=runs, betas=betas, k=1, ms_per_temperature=ms,
                          gflop_per_temperature=gflop, tflops=gflop / ms, rounds=rounds, card=card())))
    sys.stdout.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20000)
    ap.add_argument('--betas', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    a = ap.parse_args()
    for L in (1, 2, 3):
        run(L, a.runs, a.betas, a.rounds)


if __name__ == '__main__':
    main()
