"""Time the CIFAR-10 recipe's patch RBMs (examples/dbm_cifar.py of the reference: 26 GaussianRBMs 192-300, batch 48, CD-1, sampled
states, sparsity 1e-3, dbm_first) trained one after another with train_epoch against one grouped epoch (bm_rbm_group_train_epoch,
what fit_many runs), on seeded synthetic data: wall time per epoch (host clock around work that ends in a device synchronise),
kernel launches per step, and whether the grouped models end bit for bit where the sequential ones end.  Alternates the two
ways --reps times.  One JSON line per measurement, plus the card.

    python tools/bench_rbm_group.py [--models 26] [--rows 4800] [--reps 3]
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

V, H, BATCH = 192, 300, 48


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm',
                                        '--format=csv,noheader'],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def engines(G):
    out = []
    for g in range(G):
        e = _native.CudaRBM(dict(n_visible=V, n_hidden=H, v_kind='gaussian', h_kind='bernoulli', dtype='float32', compute='bf16',
                                 sample_v=True, sample_h=True, l2=1e-3, sparsity_cost=1e-3, sparsity_target=0.1,
                                 dbm_first=True, max_batch=BATCH, sigma=np.ones(V)))
        e.init_normal_W(0.001, 9000 + g)
        out.append(e)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--models', type=int, default=26)
    ap.add_argument('--rows', type=int, default=4800)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    G = a.models
    rng = np.random.RandomState(0)
    X = rng.randn(G, a.rows, V).astype(np.float32)
    nb = (a.rows + BATCH - 1) // BATCH
    print(json.dumps({'card': card(), 'models': G, 'rows': a.rows, 'batches_per_epoch': nb}))
    seq, grouped = engines(G), engines(G)
    grp = _native.CudaRBMGroup(grouped)
    P = grp.pin(list(X))
    Ps = [seq[g].pin(X[g]) for g in range(G)]
    ctx = seq[0].ctx
    lr, mom, seeds = [5e-4] * G, [0.9] * G, [9000 + g for g in range(G)]
    tick = [0]

    def run_seq():
        for g in range(G):
            seq[g].train_epoch(Ps[g], BATCH, lr[g], mom[g], 1, seeds[g], tick[0])

    def run_group():
        grp.train_epoch(P, BATCH, lr=lr, momentum=mom, k=1, seed=seeds, tick0=[tick[0]] * G, metrics=[()] * G, every=[0] * G,
                        iter0=[0] * G)

    for name, fn in (('sequential', run_seq), ('group', run_group)):       # warm-up epoch: descriptors, module loads
        fn()
    ctx.sync()
    tick[0] += nb
    times = {'sequential': [], 'group': []}
    launches = {}
    for rep in range(a.reps):
        for name, fn in (('sequential', run_seq), ('group', run_group)):
            n0 = ctx.launch_count()
            ctx.sync()
            t0 = time.perf_counter()
            fn()
            ctx.sync()
            times[name].append(time.perf_counter() - t0)
            launches[name] = (ctx.launch_count() - n0) / nb
        tick[0] += nb
    names = ('W', 'vb', 'hb', 'dW', 'dvb', 'dhb', 'q_means')
    identical = all(np.array_equal(seq[g].get_params([n])[n], grouped[g].get_params([n])[n]) for g in range(G) for n in names)
    for name in times:
        t = times[name]
        print(json.dumps({'way': name, 'epoch_s_min': min(t), 'epoch_s_max': max(t), 'epoch_s': t,
                          'ms_per_step_min': 1e3 * min(t) / nb, 'launches_per_step': launches[name]}))
    print(json.dumps({'speedup_min_over_min': min(times['sequential']) / min(times['group']), 'bit_identical': bool(identical)}))
    grp.unpin(P)
    for e, p in zip(seq, Ps):
        e.unpin(p)
    grp.close()


if __name__ == '__main__':
    main()
