"""Time the classification DBM (csrc/bm_cdbm_tc.cuh, DESIGN.md §5.7) at cfg4's shape: 784-512-1024 with a 10-class label
layer, 1024 rows and 1024 particles, k = 1, max_mf_updates 10.  ms per training step with every row labelled, half the rows
labelled -1 and every row labelled -1, each timed in rounds that alternate with the plain 784-512-1024 DBM step (bench.py's
model at max_mf_updates 10) on the same card; then predict_proba rows per second.  One JSON line per measurement, plus the
card (name, power limit, max SM clock) read in the same call.

    python tools/bench_class_dbm.py [--steps 50] [--warmup 10] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'boltzmann-machines_b200'))
sys.path.insert(0, ROOT)

from boltzmann_machines import _native  # noqa: E402
import bench  # noqa: E402

C = 10


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                        '--format=csv,noheader'], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def engine(classes):
    cfg = bench.dbm_cfg('bf16')
    cfg['max_mf_updates'] = 10
    d = bench.dbm_params(cfg)
    if classes:
        cfg['n_classes'] = C
        rng = np.random.RandomState(3)
        d['U'] = (0.02 * rng.randn(C, cfg['n_hiddens'][-1])).astype(np.float32)
        d['yb'] = np.zeros(C, np.float32)
    e = _native.CudaDBM(cfg)
    e.set_params(d)
    e.init_particles(4242)
    return e, cfg


def time_steps(e, X, y, steps, tick0):
    ctx = e.ctx
    ctx.sync()
    ctx.timer_start()
    for i in range(steps):
        e.train_step(X, 2e-3, 0.9, 1, seed=7, tick=tick0 + i, labels=y)
    return ctx.timer_stop() / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    if _native.device_count() < 1:
        raise SystemExit('no GPU: nothing is measured')
    print(json.dumps({'card': card()}), flush=True)
    plain, cfg = engine(False)
    cls, _ = engine(True)
    rows = cfg['batch_size']
    X = (np.random.RandomState(0).rand(rows, cfg['n_visible']) < 0.13).astype(np.float32)
    y = (np.arange(rows) % C).astype(np.int32)
    half = y.copy()
    half[::2] = -1
    runs = {'plain': (plain, None), 'all_labelled': (cls, y), 'half_unlabelled': (cls, half),
            'all_unlabelled': (cls, np.full(rows, -1, np.int32))}
    for name, (e, lab) in runs.items():
        time_steps(e, X, lab, a.warmup, 0)
    res = {k: [] for k in runs}
    for r in range(a.rounds):
        for name, (e, lab) in runs.items():
            res[name].append(time_steps(e, X, lab, a.steps, 1000 * (r + 1)))
    for name, ms in res.items():
        print(json.dumps({'run': name, 'ms_per_step': [round(x, 4) for x in ms], 'median_ms': round(float(np.median(ms)), 4),
                          'vs_plain': round(float(np.median(ms) / np.median(res['plain'])), 3)}), flush=True)
    Xq = (np.random.RandomState(1).rand(rows * 8, cfg['n_visible']) < 0.13).astype(np.float32)
    cls.predict_proba(Xq[:rows])
    cls.ctx.sync()
    t0 = time.perf_counter()
    for _ in range(a.rounds):
        cls.predict_proba(Xq)                        # returns after its last device-to-host copy has completed
    dt = (time.perf_counter() - t0) / a.rounds
    print(json.dumps({'run': 'predict_proba', 'rows': len(Xq), 'rows_per_s': round(len(Xq) / dt, 1)}), flush=True)


if __name__ == '__main__':
    main()
