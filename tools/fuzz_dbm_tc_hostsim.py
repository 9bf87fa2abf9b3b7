"""Random configurations of the tensor-core DBM engine (compute='bf16'), its kernels interpreted on the CPU (tests/hostsim),
against the bf16 emulation oracle (oracle/dbm_bf16.py): training steps, queries and AIS on ragged shapes, Gaussian visibles,
sampled and mean-valued layers (an unsampled first hidden layer takes the AIS ladder over fp32 pre-activations), 1-3 hidden
layers and now and then several 256-row blocks.

    python tools/fuzz_dbm_tc_hostsim.py [--n 200] [--seed 0]

Prints one line per failing configuration (with the seed that reproduces it) and a summary; exit code 1 if any failed."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import traceback

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'boltzmann-machines_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)


def draw(rng):
    L = int(rng.choice([1, 2, 2, 3]))
    wide = rng.rand() < 0.12                      # several column tiles / more than a handful of K chunks per op
    V = int(rng.choice([rng.randint(2, 40), rng.randint(40, 200)]) if not wide else rng.randint(200, 640))
    # (layer i needs more than i units: the reference's sparsity update indexes element i of layer i's vector, and the engine
    # refuses narrower layers like the reference's graph does)
    Hs = [max(i + 1, int(rng.choice([rng.randint(2, 30), rng.randint(30, 150)]) if not wide else rng.randint(100, 640))) for i in range(L)]
    gaussian = bool(rng.rand() < 0.25)
    cfg = dict(n_visible=V, n_hiddens=Hs, v_kind='gaussian' if gaussian else 'bernoulli', h_kinds=['bernoulli'] * L,
               h_n_samples=[100.] * L, dtype='float32', compute='bf16', n_particles=int(rng.randint(1, 40)),
               batch_size=int(rng.randint(1, 40)), max_mf_updates=int(rng.randint(1, 9)),
               mf_tol=float(rng.choice([1e-6, 1e-6, 3e-3])), l2=float(rng.choice([0., 1e-4, 1e-2])),
               max_norm=float(rng.choice([np.inf, 3.0, 0.8])), sample_v=bool(rng.rand() < 0.5),
               sample_h=[bool(rng.rand() < 0.7) for _ in range(L)], sparsity_target=[float(rng.uniform(0.05, 0.5)) for _ in range(L)],
               sparsity_cost=[float(rng.choice([0., 0.01, 0.1])) for _ in range(L)], sparsity_damping=float(rng.uniform(0.5, 0.99)))
    if gaussian:
        cfg['sigma'] = rng.uniform(0.6, 1.5, V)
    if rng.rand() < 0.1:
        # several 256-row blocks: the programs' row-block dependencies are then checked block by block (the interpreter shadows
        # every element a program launch touches and reports hazards no declared dependency covers)
        cfg['batch_size'], cfg['n_particles'] = int(rng.randint(257, 700)), int(rng.randint(257, 700))
    run = dict(k=int(rng.randint(1, 4)), steps=int(rng.randint(1, 4)), lr=float(rng.choice([0.01, 0.05, 0.2])),
               momentum=float(rng.choice([0., 0.5, 0.9])), scale=float(rng.choice([0.05, 0.3, 1.0])),
               rows=[int(rng.randint(1, cfg['batch_size'] + 1)) if rng.rand() < 0.3 else cfg['batch_size'] for _ in range(3)])
    return cfg, run


def close(got, want, what, rtol=2.0 ** -7, atol=3e-5):
    """Engine and emulation accumulate in different orders, so a float32 value that sits on a bf16 rounding boundary may round
    either way; one such ulp in a mean-valued state (sample_h False, Gaussian visibles) travels through the next product.  Those
    are isolated elements a fraction of a percent apart.  A wiring error -- wrong operand, scale, site, buffer -- moves most
    elements by O(0.1)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    d = np.abs(got - want)
    bad = d > atol + rtol * np.abs(want)
    assert bad.sum() <= max(3, 0.03 * bad.size) and (d.max() if d.size else 0.0) <= 0.02 * max(1.0, float(np.abs(want).max())), \
        '{0}: {1} of {2} elements off, max |diff| {3:.3g}'.format(what, int(bad.sum()), bad.size, float(d.max()))


def one(cfg, run, seed, sim=None):
    """One configuration.  `sim`: the host-simulation library, whose runtime checks are then asserted too (None: the
    engine runs on a real GPU)."""
    from boltzmann_machines import _native
    from oracle.dbm_bf16 import OracleDBMbf16
    if sim is not None:
        sim.fakecuda_reset()
    eng, emu = _native.CudaDBM(cfg), OracleDBMbf16(cfg)
    assert eng.compute == 'bf16', 'engine fell back to ' + eng.compute
    rng = np.random.RandomState(seed)
    sizes = [cfg['n_visible']] + cfg['n_hiddens']
    d = {'vb': (0.1 * rng.randn(sizes[0])).astype(np.float32)}
    for i in range(len(cfg['n_hiddens'])):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (run['scale'] * rng.randn(sizes[i], sizes[i + 1]) / np.sqrt(sizes[i])).astype(np.float32)
        d['hb' + s] = (0.1 * rng.randn(sizes[i + 1])).astype(np.float32)
    for e in (eng, emu):
        e.set_params(d)
        e.init_particles(seed + 1)
    V, gaussian = cfg['n_visible'], cfg['v_kind'] == 'gaussian'
    for it in range(run['steps']):
        rows = run['rows'][it]
        X = rng.randn(rows, V).astype(np.float32) if gaussian else (rng.rand(rows, V) < 0.3).astype(np.float32)
        a = eng.train_step(X, run['lr'], run['momentum'], run['k'], 99, it, metrics=('msre', 'n_mf_updates'))
        b = emu.train_step(X, run['lr'], run['momentum'], run['k'], 99, it, metrics=('msre', 'n_mf_updates'))
        if a['n_mf_updates'] != b['n_mf_updates']:
            # a sweep whose change lands within bf16 rounding of the tolerance may stop one sweep apart: not a wiring error,
            # but the states diverge from here on
            return 'mf-count'
        np.testing.assert_allclose(a['msre'], b['msre'], rtol=2e-3, err_msg='msre step %d' % it)
        # One step from identical states.  Then the emulation continues from the ENGINE's state: a weight that rounds to
        # the other bf16 neighbour (float32 sums in another order) would otherwise grow step by step into percent-level
        # differences that say nothing about the wiring.
        g, w = eng.get_params(), emu.get_params()
        flips = sum(int((np.abs(g[k] - w[k]) > 0.5).sum()) for k in w if k == 'v' or (k.startswith('h') and not k.startswith('hb')))
        if 0 < flips <= 2:
            return 'sample-flip'          # a uniform within float32 rounding of its probability: the chains part here
        for k in w:
            close(g[k], w[k], 'after training step {0}: {1}'.format(it, k))
        emu.set_params(g)
    nq = min(5, cfg['batch_size'])                 # a DBM query may not exceed batch_size rows
    Xq = rng.randn(nq, V).astype(np.float32) if gaussian else (rng.rand(nq, V) < 0.3).astype(np.float32)
    close(eng.transform(Xq), emu.transform(Xq), 'transform')
    close(eng.reconstruct(Xq), emu.reconstruct(Xq), 'reconstruct')
    close(eng.sample_v(2, 11, 4), emu.sample_v(2, 11, 4), 'sample_v')
    if len(cfg['n_hiddens']) == 2 and not gaussian:
        # float32 log-weight sums in different orders: ~1e-5 relative; a chain that took another sample differs by ~0.1
        # (a single mean-valued unit on a rounding boundary moves one run by a few 1e-3)
        a, b = eng.ais(6, 25, run['k'], 2222), emu.ais(6, 25, run['k'], 2222)
        d = np.abs(a - b)
        assert (d > 5e-4 + 2e-5 * np.abs(b)).sum() <= 1 and d.max() < 1.0, 'ais: {0} vs {1}'.format(a, b)    # (one run may take another sample)
    if sim is not None:
        v = sim.fakecuda_violation().decode()
        assert v == '', v
        sk = sim.fakecuda_skipped().decode()
        assert sk == '', 'not interpreted: ' + sk
    eng.close()
    return 'ok'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=200)
    ap.add_argument('--seed', type=int, default=0)
    args = ap.parse_args()
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    sim = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim.so'))
    sim.fakecuda_violation.restype = C.c_char_p
    sim.fakecuda_skipped.restype = C.c_char_p
    sim.fakecuda_set_execute(1)
    sim.fakecuda_set_hazards(2)               # shadow every program launch, whatever its size
    _native._lib = sim
    counts = {}
    sim.fakecuda_hazard_launches.restype = C.c_long
    for i in range(args.n):
        seed = args.seed * 100000 + i
        cfg, run = draw(np.random.RandomState(seed))
        try:
            r = one(cfg, run, seed, sim)
        except Exception as e:            # noqa: BLE001 -- report and go on
            r = 'FAIL'
            msg = ' '.join(str(e).split())[:400]
            print('FAIL seed={0} cfg={1} run={2}\n     {3}'.format(seed, {k: v for k, v in cfg.items() if k != 'sigma'}, run, msg),
                  flush=True)
            if not isinstance(e, AssertionError):
                traceback.print_exc()
        counts[r] = counts.get(r, 0) + 1
    print(counts, '-- program launches checked for dataflow hazards:', sim.fakecuda_hazard_launches(),
          '; declared dependencies the kernel would not wait for:', sim.fakecuda_unhonoured_dependencies())
    sys.exit(1 if counts.get('FAIL') else 0)


if __name__ == '__main__':
    main()
