"""Training-step time of DBMs with a multinomial top layer on both DBM engines, on one GPU:

    python tools/bench_dbm_multinomial.py [--shape naive|cifar] [--batch 100 1024] [--steps 10] [--warmup 2] [--rounds 3]

naive: examples/dbm_cifar_naive.py's DBM, Gaussian 3072 -> Bernoulli 5000 -> multinomial 1000 (n_samples 1000).
cifar: examples/dbm_cifar.py's DBM, Gaussian 3072 -> Bernoulli 7800 -> multinomial 512 (n_samples 512).
Both with 1 Gibbs step and 10 mean-field updates (mf_tol 1e-7), batch = particles.  The engine call bm_dbm_train_step is
timed for the tensor-core engine (compute='bf16') and the CUDA-core engine (compute='fp32') in alternating rounds on the same
card, from the same parameters; each round runs `steps` steps after `warmup` untimed ones and ends in a device synchronise.
Per engine and batch one JSON line: median ms/step over the rounds, library kernel launches per step, flag read-backs per step
(host synchronisations of the E-step, from n_mf_updates: one per chunk of 5 speculated sweeps on the tensor-core engine, one
per convergence test on the CUDA-core one), and the tensor-core kernels' device time per step (bm_ctx_profile_tc, in a
separate profiled round).  The card's name and power limit are printed first."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'boltzmann-machines_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)

SHAPES = {'naive': (3072, 5000, 1000, 1000), 'cifar': (3072, 7800, 512, 512)}
MAX_MF, MF_CHUNK = 10, 5


def make_cfg(shape, batch, compute):
    V, H0, H1, n = SHAPES[shape]
    return dict(n_visible=V, n_hiddens=[H0, H1], v_kind='gaussian', sigma=np.ones(V), h_kinds=['bernoulli', 'multinomial'],
                h_n_samples=[100., float(n)], dtype='float32', compute=compute, n_particles=batch, batch_size=batch,
                max_mf_updates=MAX_MF, mf_tol=1e-7, l2=1e-5, max_norm=np.inf, sample_v=True, sample_h=[True, True],
                sparsity_target=[0.1, 0.1], sparsity_cost=[0., 0.], sparsity_damping=0.9)


def flag_readbacks(compute, n_mf):
    if compute == 'bf16':
        return n_mf // MF_CHUNK + (0 if n_mf == MAX_MF and n_mf % MF_CHUNK == 0 else 1)
    return n_mf if n_mf == MAX_MF else n_mf + 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shape', choices=sorted(SHAPES), default='naive')
    ap.add_argument('--batch', type=int, nargs='+', default=[100, 1024])
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    from boltzmann_machines import _native
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout.strip()
    print(json.dumps({'card': card}), flush=True)
    ctx = _native.Context.default()
    for batch in a.batch:
        V = SHAPES[a.shape][0]
        rng = np.random.RandomState(0)
        sizes = [V] + make_cfg(a.shape, batch, 'bf16')['n_hiddens']
        params = {'vb': np.zeros(V, np.float32)}
        for i in range(2):
            s = '' if i == 0 else '_1'
            params['W' + s] = (0.01 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
            params['hb' + s] = np.zeros(sizes[i + 1], np.float32)
        X = rng.randn(batch, V).astype(np.float32)
        engines = {}
        for compute in ('bf16', 'fp32'):
            eng = _native.CudaDBM(make_cfg(a.shape, batch, compute), ctx)
            assert eng.compute == compute
            eng.set_params(params)
            eng.init_particles(1)
            engines[compute] = eng
        times = {c: [] for c in engines}
        launches, n_mf, tc_ms = {}, {}, {}
        tick = 0
        for r in range(a.rounds):
            for c, eng in engines.items():
                for _ in range(a.warmup):
                    eng.train_step(X, 1e-3, 0.5, 1, 7, tick); tick += 1
                ctx.sync()
                l0 = ctx.launch_count()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    eng.train_step(X, 1e-3, 0.5, 1, 7, tick); tick += 1
                ctx.sync()
                times[c].append((time.perf_counter() - t0) * 1e3 / a.steps)
                launches[c] = (ctx.launch_count() - l0) / a.steps
        for c, eng in engines.items():
            n_mf[c] = eng.train_step(X, 1e-3, 0.5, 1, 7, tick, metrics=('n_mf_updates',))['n_mf_updates']; tick += 1
            ctx.sync()
            ctx.profile_tc(True)
            for _ in range(a.steps):
                eng.train_step(X, 1e-3, 0.5, 1, 7, tick); tick += 1
            ctx.sync()
            _, ms, _ = ctx.profile_read()
            ctx.profile_tc(False)
            tc_ms[c] = ms / a.steps
        for c in engines:
            print(json.dumps({'shape': a.shape, 'batch': batch, 'particles': batch, 'engine': c,
                              'ms_per_step': float(np.median(times[c])), 'ms_per_step_rounds': [round(t, 3) for t in times[c]],
                              'launches_per_step': launches[c], 'n_mf_updates': n_mf[c],
                              'flag_readbacks_per_step': flag_readbacks(c, int(n_mf[c])),
                              'tensor_core_ms_per_step': tc_ms[c]}), flush=True)
        for eng in engines.values():
            eng.close()


if __name__ == '__main__':
    main()
