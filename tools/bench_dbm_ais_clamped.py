"""Cost of AIS with v clamped (bm_dbm_ais_clamped, DESIGN.md §5.4g) on the tensor-core engine, and what it tells a user.

cost:    ms per temperature at 784-500-1000 and 784-512-1024 for --rows rows x --runs runs (k = 1), alternated in the same call
         with log_Z's ladder at rows x runs runs; achieved TFLOP/s from the algorithm's FLOPs per chain and temperature
         (clamped: 2 sum_{j >= 1} n_j (n_{j-1} + n_{j+1}); log_Z: the same sum from j = 0; n_{L+1} = 0).
truth:   a 784-24-1000 DBM fitted for --epochs epochs on seeded synthetic binary "digits" (tools/bench_dbm_ais_base.py): per row
         the exact log p(v), the variational bound and the AIS estimate at several temperature counts over 4 seeds.
gap:     a 784-500-1000 DBM fitted the same way: AIS minus the bound, per row, at --betas temperatures.
Prints one JSON line per measurement with the card's name, power limit and SM clock read in the same call.

    python tools/bench_dbm_ais_clamped.py [--what cost,truth,gap] [--rows 200] [--runs 100] [--rounds 3] [--out file.jsonl]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'boltzmann-machines_b200'), os.path.join(ROOT, 'tools')]

from bench_dbm_ais_base import card, data_base, digits  # noqa: E402

OUT = None


def emit(**kw):
    line = json.dumps(dict(kw, card=card()))
    print(line)
    sys.stdout.flush()
    if OUT:
        with open(OUT, 'a') as f:
            f.write(line + '\n')


def flops(widths, first):
    """FLOPs per chain and temperature: one GEMM per updated layer j >= first against its neighbours"""
    n = list(widths) + [0]
    return sum(2 * n[j] * ((n[j - 1] if j >= 1 else 0) + n[j + 1]) for j in range(first, len(widths)))


def n_temps(n_betas):
    d = np.float32(1. / n_betas)
    t = [d]
    while t[-1] < np.float32(1.) - d + np.float32(1e-5):
        t.append(np.float32(t[-1] + d))
    return len(t)


def cost(rows, runs, betas, rounds):
    from boltzmann_machines import _native
    X = digits(rows, seed=1)
    for Hs in ([500, 1000], [512, 1024]):
        L = len(Hs)
        c = dict(n_visible=784, n_hiddens=Hs, v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
                 n_particles=16, batch_size=16, max_mf_updates=10, mf_tol=1e-7, l2=0., max_norm=1e300, sample_v=True,
                 sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[0.] * L, sparsity_damping=0.9)
        e = _native.CudaDBM(c)
        rng = np.random.RandomState(0)
        sizes = [784] + Hs
        d = {'vb': data_base(X)}
        for i in range(L):
            s = '' if i == 0 else '_%d' % i
            d['W' + s] = (0.02 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
            d['hb' + s] = np.zeros(sizes[i + 1], np.float32)
        e.set_params(d)
        chains = rows * runs
        e.ais_clamped(X, runs, 10, 1, 1)                           # warm-up of both ladders
        e.ais(chains, 10, 1, 1)
        t_c, t_z = [], []
        for r in range(rounds):                                    # alternated; each call ends with a device synchronise
            t0 = time.perf_counter()
            e.ais_clamped(X, runs, betas, 1, 2 + r)
            t_c.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            e.ais(chains, betas, 1, 2 + r)
            t_z.append(time.perf_counter() - t0)
        e.close()
        nT = n_temps(betas)
        for name, ts, first in (('clamped', t_c, 1), ('log_Z', t_z, 0)):
            med = float(np.median(ts))
            f = flops(sizes, first)
            emit(what='cost', ladder=name, shape='-'.join(map(str, sizes)), chains=chains, temperatures=nT, k=1,
                 seconds=med, seconds_all=ts, ms_per_temperature=1e3 * med / nT, mflop_per_chain_temperature=f / 1e6,
                 tflops=f * chains * nT / med / 1e12)


def fit(Hs, epochs, X, tmp):
    from boltzmann_machines import DBM
    from boltzmann_machines.rbm import BernoulliRBM
    rbms, inp = [], X
    sizes = [784] + list(Hs)
    for i in range(len(Hs)):
        r = BernoulliRBM(n_visible=sizes[i], n_hidden=sizes[i + 1], max_epoch=epochs, batch_size=100, learning_rate=0.05,
                         random_seed=1 + i, dtype='float32', model_path=os.path.join(tmp, 'r%d' % i), verbose=False)
        r.fit(inp)
        inp = r.transform(inp)
        rbms.append(r)
    m = DBM(rbms=rbms, n_particles=100, batch_size=100, max_epoch=epochs, random_seed=3, dtype='float32',
            model_path=os.path.join(tmp, 'dbm'), verbose=False)
    m.fit(X)
    return m


def truth(rows, runs, epochs, temps):
    X = digits(10000, seed=0)
    tmp = tempfile.mkdtemp()
    try:
        m = fit([24, 1000], epochs, X, tmp)
        T = X[:rows]
        exact_Z = m.exact_log_Z()
        exact = m.exact_log_proba(T, log_Z=exact_Z)
        bound = m.log_proba(T, exact_Z)
        ais = {}
        for nb in temps:
            est, secs = [], []
            for _ in range(4):
                t0 = time.perf_counter()
                est.append(m.ais_log_proba(T, exact_Z, n_betas=nb, n_runs=runs, n_gibbs_steps=1))
                secs.append(time.perf_counter() - t0)
            est = np.array(est)
            ais[str(nb)] = dict(mean_minus_exact=float((est - exact).mean()), seed_std_per_row=float(est.std(axis=0).mean()),
                                max_abs_minus_exact=float(np.abs(est - exact).max()), seconds=secs,
                                rows_first8=est[:, :8].tolist())
        emit(what='truth', shape='784-24-1000', epochs=epochs, rows=rows, runs=runs, k=1, exact_log_Z=exact_Z,
             mean_exact=float(exact.mean()), mean_bound_minus_exact=float((bound - exact).mean()),
             exact_first8=exact[:8].tolist(), bound_first8=bound[:8].tolist(), ais=ais)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def gap(rows, runs, betas, epochs):
    X = digits(10000, seed=0)
    tmp = tempfile.mkdtemp()
    try:
        m = fit([500, 1000], epochs, X, tmp)
        T = X[:rows]
        bound = m.log_proba(T, 0.0)
        t0 = time.perf_counter()
        est = m.ais_log_proba(T, 0.0, n_betas=betas, n_runs=runs, n_gibbs_steps=1)
        secs = time.perf_counter() - t0
        g = est - bound
        emit(what='gap', shape='784-500-1000', epochs=epochs, rows=rows, runs=runs, betas=betas, k=1, seconds=secs,
             mean_ais_minus_bound=float(g.mean()), min=float(g.min()), max=float(g.max()), first8=g[:8].tolist())
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    global OUT
    ap = argparse.ArgumentParser()
    ap.add_argument('--what', default='cost,truth,gap')
    ap.add_argument('--rows', type=int, default=200)
    ap.add_argument('--runs', type=int, default=100)
    ap.add_argument('--betas', type=int, default=1000)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--temps', default='100,1000,10000')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    OUT = a.out
    if 'cost' in a.what:
        cost(a.rows, a.runs, a.betas, a.rounds)
    if 'truth' in a.what:
        truth(a.rows, a.runs, a.epochs, [int(t) for t in a.temps.split(',')])
    if 'gap' in a.what:
        gap(a.rows, a.runs, a.betas, a.epochs)


if __name__ == '__main__':
    main()
