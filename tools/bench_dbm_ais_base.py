"""Cost and benefit of AIS from a base-rate model (bm_dbm_ais_base, DESIGN.md §5.4d) on the tensor-core engine.

cost:    ms per temperature of the uniform ladder and of the ladder from a data-like visible base, alternated round by round,
         at `--runs` runs (k = 1) for 784-500-1000 and 784-500-500-1000.
benefit: a 784-500-1000 DBM fitted for a few epochs on seeded synthetic binary "digits" (nothing downloaded): for 1000 and 5000
         temperatures and 8 seeds, log Z-hat of each seed, their spread (std over seeds) and the mean per-run std of the
         log-weights, uniform against the data base logit((sum X + 1) / (n + 2)).
Prints one JSON line per measurement with the card's name, power limit and SM clock read in the same call.

    python tools/bench_dbm_ais_base.py [--runs 20000] [--betas 200] [--rounds 5] [--what cost,benefit]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'boltzmann-machines_b200')]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def emit(**kw):
    print(json.dumps(dict(kw, card=card())))
    sys.stdout.flush()


def digits(n, seed=0):
    """binary 28x28 "digits": ten seeded stroke prototypes, shifted by up to 2 pixels, with 2% of the pixels flipped"""
    rng = np.random.RandomState(seed)
    protos = np.zeros((10, 28, 28), np.float32)
    for c in range(10):
        for _ in range(3):                                    # three thick strokes per class
            r0, c0, r1, c1 = rng.randint(5, 23, 4)
            for s in np.linspace(0., 1., 40):
                r, q = int(round(r0 + s * (r1 - r0))), int(round(c0 + s * (c1 - c0)))
                protos[c, max(r - 1, 0):r + 2, max(q - 1, 0):q + 2] = 1.
    y = rng.randint(0, 10, n)
    X = np.empty((n, 784), np.float32)
    for i in range(n):
        img = np.roll(np.roll(protos[y[i]], rng.randint(-2, 3), axis=0), rng.randint(-2, 3), axis=1)
        X[i] = img.ravel()
    flip = rng.rand(n, 784) < 0.02
    return np.where(flip, 1. - X, X).astype(np.float32)


def data_base(X):
    p = (X.astype(np.float64).sum(axis=0) + 1.) / (X.shape[0] + 2.)
    return np.log(p / (1. - p)).astype(np.float32)


def cost(runs, betas, rounds):
    from boltzmann_machines import _native
    X = digits(2000, seed=1)
    for Hs in ([500, 1000], [500, 500, 1000]):
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
        base = [data_base(X)] + [None] * L
        for b in (None, base):                                # warm-up of both
            e.ais(runs, betas, 1, 1, base=b)
        ts = {'uniform': [], 'base': []}
        for r in range(rounds):
            for name, b in (('uniform', None), ('base', base)):
                t0 = time.perf_counter()
                e.ais(runs, betas, 1, 2 + r, base=b)          # returns after the device synchronises
                ts[name].append(time.perf_counter() - t0)
        e.close()
        emit(what='cost', shape='-'.join(map(str, sizes)), runs=runs, betas=betas, k=1, rounds=rounds,
             ms_per_temperature={k: 1e3 * float(np.median(v)) / betas for k, v in ts.items()},
             ms_per_temperature_all={k: [1e3 * x / betas for x in v] for k, v in ts.items()})


def benefit(runs, epochs):
    from boltzmann_machines import DBM
    from boltzmann_machines.rbm import BernoulliRBM
    X = digits(10000, seed=0)
    tmp = tempfile.mkdtemp()
    try:
        t0 = time.perf_counter()
        r1 = BernoulliRBM(n_visible=784, n_hidden=500, max_epoch=epochs, batch_size=100, learning_rate=0.05, random_seed=1,
                          dtype='float32', model_path=os.path.join(tmp, 'r1'), verbose=False)
        r1.fit(X)
        H = r1.transform(X)
        r2 = BernoulliRBM(n_visible=500, n_hidden=1000, max_epoch=epochs, batch_size=100, learning_rate=0.05, random_seed=2,
                          dtype='float32', model_path=os.path.join(tmp, 'r2'), verbose=False)
        r2.fit(H)
        m = DBM(rbms=[r1, r2], n_particles=100, batch_size=100, max_epoch=epochs, random_seed=3, dtype='float32',
                model_path=os.path.join(tmp, 'dbm'), verbose=False)
        m.fit(X)
        fit_s = time.perf_counter() - t0
        base = [data_base(X), None, None]
        for betas in (1000, 5000):
            res = {}
            for name, b in (('uniform', None), ('base', base)):
                est, sd = [], []
                for seed in range(8):
                    v = m._engine.ais(runs, betas, 1, 1000 + seed, base=b)
                    est.append(float(np.logaddexp.reduce(v) - np.log(len(v))))
                    sd.append(float(np.std(v)))
                res[name] = dict(log_Z=est, spread_over_seeds=float(np.std(est)), per_run_std=float(np.mean(sd)))
            emit(what='benefit', shape='784-500-1000', epochs=epochs, fit_seconds=fit_s, runs=runs, betas=betas, k=1, **res)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=20000)
    ap.add_argument('--betas', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--benefit-runs', type=int, default=1000)
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--what', default='cost,benefit')
    a = ap.parse_args()
    if 'cost' in a.what:
        cost(a.runs, a.betas, a.rounds)
    if 'benefit' in a.what:
        benefit(a.benefit_runs, a.epochs)


if __name__ == '__main__':
    main()
