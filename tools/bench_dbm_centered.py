"""Measure centered DBM training (csrc/bm_dbm_tc.cuh, DESIGN.md §5.8).

1. Step cost: ms per bm_dbm_train_step of the centered and the plain step at the cfg4 shape (784-512-1024, 1024 particles,
   k = 1) and the cfg5-pcd shape (784-4096, 4096 particles, k = 25), timed in rounds that alternate the two engines on the same
   card (median over rounds), and the kernel launches of one step.  The models are bench.py's.
2. Training from scratch (--bas): exact average log-likelihood of 16-16-8 DBMs built from init()-only RBMs, plain and centered,
   5 seeds, on 4x4 bars-and-stripes D and on 1 - D (tests/test_zz_dbm_centered_gpu.py states the runs).
One JSON line per measurement, plus the card.

    python tools/bench_dbm_centered.py [--steps 50] [--warmup 10] [--rounds 3] [--bas]
"""
import argparse
import json
import os
import pathlib
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'boltzmann-machines_b200'))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from boltzmann_machines import _native  # noqa: E402
import bench  # noqa: E402


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                                        '--format=csv,noheader'], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def engine(shape, centered):
    if shape == 'cfg5-pcd':
        cfg = bench.dbm_cfg('bf16', [4096], 4096, 784, pcd_only=True)
        k, scale, lr = 25, 0.01, 0.01
    else:
        cfg = bench.dbm_cfg('bf16')
        k, scale, lr = 1, 0.02, 2e-3
    if centered:
        cfg.update(centering=True, offset_rate=0.01)
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


def launches(e, X, k, lr, tick):
    n0 = e.ctx.launch_count()
    e.train_step(X, lr, 0.9, k, seed=7, tick=tick)
    e.ctx.sync()
    return e.ctx.launch_count() - n0


def step_cost(a):
    for shape in a.shapes.split(','):
        steps = a.steps if shape == 'cfg4' else max(5, a.steps // 5)
        cen, X, k, lr = engine(shape, True)
        plain, _, _, _ = engine(shape, False)
        for e in (cen, plain):
            for i in range(a.warmup):
                e.train_step(X, lr, 0.9, k, seed=7, tick=i)
        t_c, t_p = [], []
        tick = a.warmup
        for _ in range(a.rounds):                    # alternate: the two engines see the same clocks
            t_c.append(time_steps(cen, X, k, lr, steps, tick))
            t_p.append(time_steps(plain, X, k, lr, steps, tick))
            tick += steps
        rec = {'shape': shape, 'k': k, 'ms_per_step_centered': round(float(np.median(t_c)), 4),
               'ms_per_step_plain': round(float(np.median(t_p)), 4), 'ratio': round(float(np.median(t_c) / np.median(t_p)), 4),
               'rounds_centered': [round(x, 4) for x in t_c], 'rounds_plain': [round(x, 4) for x in t_p],
               'launches_centered': launches(cen, X, k, lr, tick), 'launches_plain': launches(plain, X, k, lr, tick)}
        print(json.dumps(rec), flush=True)
        cen.close()
        plain.close()


def bas(a):
    import test_zz_dbm_centered_gpu as T
    D = T.bars_and_stripes()
    with tempfile.TemporaryDirectory() as tmp:
        for name, data in (('D', D), ('1-D', 1.0 - D)):
            for centered in (False, True):
                runs = [T.train_bas(data, centered, s, pathlib.Path(tempfile.mkdtemp(dir=tmp)))[:2] for s in T.SEEDS]
                ll = np.array([r[1] for r in runs])
                print(json.dumps({'data': name, 'centered': centered, 'initial_ll': round(float(np.mean([r[0] for r in runs])), 4),
                                  'final_ll_mean': round(float(ll.mean()), 4), 'final_ll_std': round(float(ll.std()), 4),
                                  'final_ll': [round(float(x), 4) for x in ll]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--shapes', default='cfg4,cfg5-pcd')
    ap.add_argument('--bas', action='store_true', help='also train the bars-and-stripes DBMs')
    a = ap.parse_args()
    print(json.dumps({'card': card()}))
    step_cost(a)
    if a.bas:
        bas(a)


if __name__ == '__main__':
    main()
