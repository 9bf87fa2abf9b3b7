"""Cost of exact log Z / log p(v) (bm_dbm_exact, DESIGN.md §5.4f) on the tensor-core engine, and AIS measured against it.

log_Z:   seconds per exact log Z for n_odd in --bits at 784-n and 784-n-1000 (W ~ N(0, 0.02^2), data-like visible biases),
         after one warm-up call at 20 bits; median of --rounds calls.
proba:   rows x states per second of exact log p*(v) at 784-24 for 1024 rows (the pass with rows minus the pass without).
truth:   a 784-24-1000 DBM fitted for --epochs epochs on seeded synthetic binary "digits" (tools/bench_dbm_ais_base.py): exact
         log Z against AIS from the uniform base and from the data base, 8 seeds each at --runs runs x --betas temperatures.
Prints one JSON line per measurement with the card's name, power limit and SM clock read in the same call.

    python tools/bench_dbm_exact.py [--bits 20,24,28,32] [--rounds 3] [--what log_Z,proba,truth] [--out file.jsonl]
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


def engine(Hs, X):
    from boltzmann_machines import _native
    L = len(Hs)
    c = dict(n_visible=784, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
             n_particles=16, batch_size=16, max_mf_updates=10, mf_tol=1e-7, l2=0., max_norm=1e300, sample_v=True,
             sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[0.] * L, sparsity_damping=0.9)
    e = _native.CudaDBM(c)
    rng = np.random.RandomState(0)
    sizes = [784] + list(Hs)
    d = {'vb': data_base(X)}
    for i in range(L):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (0.02 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = np.zeros(sizes[i + 1], np.float32)
    e.set_params(d)
    return e


def timed(f, rounds):
    ts, out = [], None
    for _ in range(rounds):
        t0 = time.perf_counter()
        out = f()                                             # returns after the device synchronises
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), ts, out


def log_Z(bits, rounds):
    X = digits(2000, seed=1)
    warm = engine([20], X)
    warm.exact(None)
    warm.close()
    for n in bits:
        for Hs in ([n], [n, 1000]):
            e = engine(Hs, X)
            med, ts, (_, lz) = timed(lambda: e.exact(None), rounds)
            N = 784 + sum(Hs[1::2])
            emit(what='log_Z', shape='-'.join(map(str, [784] + Hs)), n_odd=n, seconds=med, seconds_all=ts, log_Z=lz,
                 softplus_per_second=float(2 ** n * N / med))
            e.close()


def proba(rounds):
    X = digits(2000, seed=1)
    e = engine([24], X)
    rows = X[:1024]
    e.exact(rows)
    t_rows, ts_rows, _ = timed(lambda: e.exact(rows), rounds)
    t_z, ts_z, _ = timed(lambda: e.exact(None), rounds)
    emit(what='proba', shape='784-24', rows=len(rows), seconds_with_rows=t_rows, seconds_log_Z_only=t_z,
         rows_states_per_second=float(len(rows) * 2 ** 24 / max(t_rows - t_z, 1e-9)),
         seconds_all={'rows': ts_rows, 'log_Z': ts_z})
    e.close()


def truth(runs, betas, epochs):
    from boltzmann_machines import DBM
    from boltzmann_machines.rbm import BernoulliRBM
    X = digits(10000, seed=0)
    tmp = tempfile.mkdtemp()
    try:
        t0 = time.perf_counter()
        r1 = BernoulliRBM(n_visible=784, n_hidden=24, max_epoch=epochs, batch_size=100, learning_rate=0.05, random_seed=1,
                          dtype='float32', model_path=os.path.join(tmp, 'r1'), verbose=False)
        r1.fit(X)
        r2 = BernoulliRBM(n_visible=24, n_hidden=1000, max_epoch=epochs, batch_size=100, learning_rate=0.05, random_seed=2,
                          dtype='float32', model_path=os.path.join(tmp, 'r2'), verbose=False)
        r2.fit(r1.transform(X))
        m = DBM(rbms=[r1, r2], n_particles=100, batch_size=100, max_epoch=epochs, random_seed=3, dtype='float32',
                model_path=os.path.join(tmp, 'dbm'), verbose=False)
        m.fit(X)
        fit_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        exact = m.exact_log_Z()
        exact_s = time.perf_counter() - t0
        ll = float(np.mean(m.exact_log_proba(X[:1000], log_Z=exact)))
        res = {}
        for name, b in (('uniform', None), ('base', [data_base(X), None, None])):
            est = []
            for seed in range(8):
                v = m._engine.ais(runs, betas, 1, 1000 + seed, base=b)
                est.append(float(np.logaddexp.reduce(v) - np.log(len(v))))
            res[name] = dict(log_Z=est, gap_to_exact=[x - exact for x in est], mean_gap=float(np.mean(est) - exact))
        emit(what='truth', shape='784-24-1000', epochs=epochs, fit_seconds=fit_s, exact_log_Z=exact, exact_seconds=exact_s,
             mean_exact_log_p_train=ll, runs=runs, betas=betas, k=1, **res)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    global OUT
    ap = argparse.ArgumentParser()
    ap.add_argument('--bits', default='20,24,28,32')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--runs', type=int, default=1000)
    ap.add_argument('--betas', type=int, default=1000)
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--what', default='log_Z,proba,truth')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    OUT = a.out
    if 'log_Z' in a.what:
        log_Z([int(b) for b in a.bits.split(',')], a.rounds)
    if 'proba' in a.what:
        proba(a.rounds)
    if 'truth' in a.what:
        truth(a.runs, a.betas, a.epochs)


if __name__ == '__main__':
    main()
