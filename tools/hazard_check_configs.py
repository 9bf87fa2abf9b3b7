"""Dataflow-hazard check of the step programs at BASELINE.json's full sizes, on the host simulation (no GPU):

    python tools/hazard_check_configs.py [cfg2] [cfg3] [cfg4] [ais-depth] [ais-clamped]

Every element a program launch reads or writes is shadowed while the launch is interpreted (tests/hostsim/kernels_cpu.cpp,
`Hazards`); a read of / write over something another op of the launch touched must be covered by a declared dependency path,
256-row block by 256-row block.  cfg2: Bernoulli RBM 784-1024, batch 4096, CD-5 (the benchmark's program, 16 row blocks).
cfg3: Gaussian RBM 3072-5000, batch 512 (host batch and resident-dataset step).  cfg4: the tensor-core DBM engine's mean-field
and particle programs, 784-512-1024, batch = particles = 1024.  ais-depth (not run by default): the AIS ladders of
DbmTC::ais_local_layers at one, three and four hidden layers (100-64, 100-64-48-32, 100-64-48-32-16; 600 runs = three 256-run
blocks, 40 temperatures, k = 2, several launches per ladder).  ais-clamped (not run by default): the same ladders with v clamped
(DESIGN.md §5.4g) at two, three and four hidden layers, 6 rows x 100 runs, on the host-simulation library that also restates
the clamped ladder's operand kernel (build_dbm_ais_clamped.sh).  About 3 minutes, 2 GB."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'boltzmann-machines_b200')):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    which = sys.argv[1:] or ['cfg2', 'cfg3', 'cfg4']
    name = 'dbm_ais_clamped' if 'ais-clamped' in which else ''
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build_' + name + '.sh' if name else 'build.sh')],
                          stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    sim = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim' + ('_' + name if name else '') + '.so'))
    sim.fakecuda_violation.restype = C.c_char_p
    sim.fakecuda_hazard_launches.restype = C.c_long
    sim.fakecuda_set_execute(1)
    sim.fakecuda_set_hazards(2)
    _native._lib = sim
    rng = np.random.RandomState(0)
    t0 = time.time()

    def report(what):
        v = sim.fakecuda_violation().decode()
        print('{0}: program launches checked so far {1}, violations: {2}  [{3:.0f} s]'.format(
            what, sim.fakecuda_hazard_launches(), v or 'none', time.time() - t0), flush=True)
        return v == ''

    ok = True
    if 'cfg2' in which:
        B, V, H = 4096, 784, 1024
        eng = _native.CudaRBM(dict(n_visible=V, n_hidden=H, dtype='float32', compute='bf16', l2=1e-5, sample_v=False, sample_h=True,
                                   max_batch=B))
        eng.init_normal_W(0.01, 1)
        eng.train_step((rng.rand(B, V) < 0.2).astype(np.float32), 0.05, 0.5, 5, 7, 0)
        ok = report('cfg2 step') and ok
        eng.close()
    if 'cfg3' in which:
        B, V, H = 512, 3072, 5000
        eng = _native.CudaRBM(dict(n_visible=V, n_hidden=H, dtype='float32', compute='bf16', l2=1e-5, sample_v=False, sample_h=True,
                                   max_batch=B, v_kind='gaussian', h_kind='bernoulli', sigma=np.ones(V)))
        eng.init_normal_W(0.001, 1)
        X = rng.randn(2 * B, V).astype(np.float32)
        eng.train_step(X[:B], 0.001, 0.5, 1, 7, 0)
        ok = report('cfg3 step') and ok
        eng.set_data(X)
        eng.train_step_at(B, B, 0.001, 0.5, 1, 7, 1)
        ok = report('cfg3 resident-dataset step') and ok
        eng.close()
    if 'cfg4' in which:
        V, Hs, B = 784, (512, 1024), 1024
        cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * 2, h_n_samples=[100.] * 2,
                   dtype='float32', compute='bf16', n_particles=B, batch_size=B, max_mf_updates=8, mf_tol=1e-6, l2=1e-4,
                   max_norm=3.0, sample_v=True, sample_h=[True] * 2, sparsity_target=[0.2] * 2, sparsity_cost=[0.01] * 2,
                   sparsity_damping=0.9)
        eng = _native.CudaDBM(cfg)
        eng.set_params({'vb': np.zeros(V, np.float32), 'W': (0.01 * rng.randn(V, 512)).astype(np.float32),
                        'hb': np.zeros(512, np.float32), 'W_1': (0.01 * rng.randn(512, 1024)).astype(np.float32),
                        'hb_1': np.zeros(1024, np.float32)})
        eng.init_particles(1)
        eng.train_step((rng.rand(B, V) < 0.2).astype(np.float32), 0.01, 0.5, 5, 7, 0)
        ok = report('cfg4 DBM programs') and ok
        eng.close()
    if 'ais-depth' in which:
        for Hs in ((64,), (64, 48, 32), (64, 48, 32, 16)):
            V, L = 100, len(Hs)
            cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32',
                       compute='bf16', n_particles=16, batch_size=16, sample_v=True, sample_h=[True] * L)
            eng = _native.CudaDBM(cfg)
            sizes = [V] + list(Hs)
            d = {'vb': np.zeros(V, np.float32)}
            for i in range(L):
                s = '' if i == 0 else '_%d' % i
                d['W' + s] = (0.1 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
                d['hb' + s] = np.zeros(sizes[i + 1], np.float32)
            eng.set_params(d)
            eng.ais(600, 40, 2, 3)
            ok = report('AIS ladder at {0} hidden layers'.format(L)) and ok
            eng.close()
    if 'ais-clamped' in which:
        for Hs in ((64, 48), (64, 48, 32), (64, 48, 32, 16)):
            V, L = 100, len(Hs)
            cfg = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32',
                       compute='bf16', n_particles=16, batch_size=16, sample_v=True, sample_h=[True] * L)
            eng = _native.CudaDBM(cfg)
            sizes = [V] + list(Hs)
            d = {'vb': np.zeros(V, np.float32)}
            for i in range(L):
                s = '' if i == 0 else '_%d' % i
                d['W' + s] = (0.1 * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
                d['hb' + s] = np.zeros(sizes[i + 1], np.float32)
            eng.set_params(d)
            eng.ais_clamped((rng.rand(6, V) < 0.3).astype(np.float32), 100, 40, 2, 3)
            ok = report('clamped AIS ladder at {0} hidden layers'.format(L)) and ok
            eng.close()
    sys.exit(0 if ok else 1)


if __name__ == '__main__':
    main()
