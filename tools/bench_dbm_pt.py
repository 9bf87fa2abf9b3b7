"""Time parallel tempering of the DBM's persistent chains (csrc/bm_dbm_tc.cuh): ms per bm_dbm_train_step at the cfg4 shape
(784-512-1024, 1024 particles, k = 1) and the cfg5-pcd shape (784-4096, 4096 particles, k = 25) with T = 1, 2, 4, 8 slots on
a geometric ladder, each timed in rounds that alternate with the plain step (no tempering) on the same card.  The models
are bench.py's, except that cfg5-pcd samples its visible states (tempering compares energies of states).  One JSON line per
measurement, plus the card.

    python tools/bench_dbm_pt.py [--steps 50] [--warmup 10] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'boltzmann-machines_b200'))
sys.path.insert(0, ROOT)

from boltzmann_machines import _native  # noqa: E402
import bench  # noqa: E402


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                                        '--format=csv,noheader'], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def engine(shape, T):
    if shape == 'cfg5-pcd':
        cfg = bench.dbm_cfg('bf16', [4096], 4096, 784, pcd_only=True)
        cfg['sample_v'] = True
        k, scale, lr = 25, 0.01, 0.01
    else:
        cfg = bench.dbm_cfg('bf16')
        k, scale, lr = 1, 0.02, 2e-3
    if T is not None:
        cfg['pt_betas'] = [float(0.7 ** m) for m in range(T)] if T > 1 else [1.0]
    e = _native.CudaDBM(cfg)
    e.set_params(bench.dbm_params(cfg, scale=scale))
    e.init_particles(4242)
    X = (np.random.RandomState(0).rand(cfg['batch_size'], cfg['n_visible']) < 0.13).astype(np.float32)
    return e, X, k, lr


def time_steps(e, X, k, lr, steps, tick0):
    ctx = e.ctx
    ctx.sync()
    ctx.timer_start()
    for i in range(steps):
        e.train_step(X, lr, 0.9, k, seed=7, tick=tick0 + i)
    return ctx.timer_stop() / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--shapes', default='cfg4,cfg5-pcd')
    a = ap.parse_args()
    print(json.dumps({'card': card()}))
    for shape in a.shapes.split(','):
        steps = a.steps if shape == 'cfg4' else max(5, a.steps // 5)
        for T in (1, 2, 4, 8):
            pt, X, k, lr = engine(shape, T)
            plain, _, _, _ = engine(shape, None)
            for e in (pt, plain):
                for i in range(a.warmup):
                    e.train_step(X, lr, 0.9, k, seed=7, tick=i)
            t_pt, t_plain = [], []
            tick = a.warmup
            for _ in range(a.rounds):                # alternate: the two engines see the same clocks
                t_pt.append(time_steps(pt, X, k, lr, steps, tick))
                t_plain.append(time_steps(plain, X, k, lr, steps, tick))
                tick += steps
            rec = {'shape': shape, 'k': k, 'T': T, 'ms_per_step_pt': round(float(np.median(t_pt)), 4),
                   'ms_per_step_plain': round(float(np.median(t_plain)), 4),
                   'ratio': round(float(np.median(t_pt) / np.median(t_plain)), 3),
                   'rounds_pt': [round(x, 4) for x in t_pt], 'rounds_plain': [round(x, 4) for x in t_plain]}
            if T > 1:
                acc, prop = pt.pt_counts()
                rec['swap_rates'] = [round(float(x), 3) for x in acc / np.maximum(prop, 1)]
            print(json.dumps(rec), flush=True)
            pt.close()
            plain.close()


if __name__ == '__main__':
    main()
