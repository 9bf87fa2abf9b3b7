"""Time the classification RBM (csrc/bm_crbm_tc.cuh) at 784-1024-10: bm_crbm_train_step at batches 128 and 4096 with
alpha = 0 (discriminative, no chain) and alpha = 0.01 (hybrid, k = 1), the tensor-core kernel's share of a step
(bm_ctx_profile_tc, in a run of its own), and predict_proba rows/s.  Then semi-supervised steps (beta = 0.1, alpha = 0.01,
k = 1) at the same batches with 0 %, 50 % and 100 % of the rows unlabelled, and the test accuracy on the seeded synthetic task
of tests/test_zz_class_rbm_gpu.py with 100 labelled rows alone and with 2 900 unlabelled rows beside them.  One JSON line
per measurement, plus the card.

    python tools/bench_class_rbm.py [--steps 50] [--warmup 10]
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

from boltzmann_machines import _native  # noqa: E402

V, H, C = 784, 1024, 10


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                                        '--format=csv,noheader'],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def engine(batch, alpha, beta=0.0):
    e = _native.CudaCRBM(dict(n_visible=V, n_hidden=H, n_classes=C, alpha=alpha, beta=beta, l2=1e-4, max_batch=batch,
                              sample_v=False, sample_h=True))
    e.init_normal_weights(0.01, 1, 2)
    return e


def data(rows, seed=0):
    rng = np.random.RandomState(seed)
    protos = rng.rand(C, V)
    y = rng.randint(0, C, size=rows)
    return (rng.rand(rows, V) < protos[y]).astype(np.float32), y.astype(np.int32)


def time_steps(e, X, y, steps, warmup):
    ctx = e.ctx
    for i in range(warmup):
        e.train_step(X, y, 0.05, 0.5, 1, seed=3, tick=i)
    ctx.sync()
    ctx.timer_start()
    for i in range(steps):
        e.train_step(X, y, 0.05, 0.5, 1, seed=3, tick=warmup + i)
    return ctx.timer_stop() / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    a = ap.parse_args()
    print(json.dumps({'card': card()}))
    for batch in (128, 4096):
        X, y = data(batch)
        for alpha in (0.0, 0.01):
            e = engine(batch, alpha)
            ms = time_steps(e, X, y, a.steps, a.warmup)
            e.ctx.profile_tc(True)                     # separate run: per-launch events slow the host
            e.ctx.profile_read()
            e.ctx.timer_start()
            for i in range(a.steps):
                e.train_step(X, y, 0.05, 0.5, 1, seed=3, tick=i)
            prof_total = e.ctx.timer_stop()
            _, tc_ms, launches = e.ctx.profile_read()
            e.ctx.profile_tc(False)
            print(json.dumps({'shape': '784-1024-10', 'batch': batch, 'alpha': alpha, 'k': 1, 'ms_per_step': round(ms, 4),
                              'tc_share': round(tc_ms / prof_total, 3), 'tc_launches_per_step': launches / a.steps}))
            e.close()
    e = engine(4096, 0.01)
    X, _ = data(65536, seed=1)
    e.predict_proba(X[:4096])
    e.ctx.sync()
    t0 = time.perf_counter()
    reps = 5
    for _ in range(reps):
        e.predict_proba(X)
    dt = (time.perf_counter() - t0) / reps
    print(json.dumps({'predict_proba_rows': len(X), 'max_batch': 4096, 'rows_per_s': round(len(X) / dt),
                      'note': 'host clock, includes the host-device copies'}))
    e.close()
    for batch in (128, 4096):
        X, y = data(batch)
        for frac in (0.0, 0.5, 1.0):
            yu = y.copy()
            yu[np.arange(batch) < int(round(frac * batch))] = -1
            e = engine(batch, 0.01, beta=0.1)
            ms = time_steps(e, X, yu, a.steps, a.warmup)
            print(json.dumps({'shape': '784-1024-10', 'batch': batch, 'alpha': 0.01, 'beta': 0.1, 'k': 1,
                              'unlabelled': frac, 'ms_per_step': round(ms, 4)}))
            e.close()
    semi_accuracy()


def synthetic(n, seed=0):
    """tests/test_zz_class_rbm_gpu.py's seeded class-conditional task"""
    rng = np.random.RandomState(seed)
    protos = np.clip(rng.beta(0.5, 0.5, size=(C, V)), 0.05, 0.95)
    y = rng.randint(0, C, size=n)
    return (rng.rand(n, V) < protos[y]).astype(np.float32), y


def semi_accuracy(epochs=10):
    """test accuracy with the first 100 training rows labelled, alone (beta = 0) and with the other 2 900 rows unlabelled
    (beta = 0.1); rows are interleaved, one labelled row before every 29 unlabelled ones"""
    import tempfile
    from boltzmann_machines import ClassificationRBM
    X, y = synthetic(4000)
    Xtr, ytr, Xte, yte = X[:3000], y[:3000], X[3000:], y[3000:]
    lab = np.arange(100)
    order = np.concatenate([[i] + list(range(100 + 29 * i, 129 + 29 * i)) for i in lab])      # 1 labelled, 29 unlabelled
    runs = {'100 labels': (Xtr[lab], ytr[lab], 0.0),
            '100 labels + 2900 unlabelled': (Xtr[order], np.where(order < 100, ytr[order], -1), 0.1)}
    for name, (Xf, yf, beta) in runs.items():
        with tempfile.TemporaryDirectory() as d:
            m = ClassificationRBM(n_visible=V, n_hidden=H, n_classes=C, alpha=0.01, beta=beta, learning_rate=0.1, momentum=0.5,
                                  max_epoch=epochs, batch_size=100, random_seed=11, verbose=False,
                                  save_after_each_epoch=False, model_path=d + '/')
            m.fit(Xf, yf)
            P = m.predict_proba(Xte).astype(np.float64)
        acc = float(np.mean(np.argmax(P, 1) == yte))
        nll = float(-np.mean(np.log(np.maximum(P[np.arange(len(yte)), yte], 1e-30))))
        print(json.dumps({'semi_supervised_task': name, 'epochs': epochs, 'beta': beta, 'steps_per_epoch': -(-len(Xf) // 100),
                          'test_accuracy': round(acc, 4), 'test_nll': round(nll, 4)}))


if __name__ == '__main__':
    main()
