"""bench.py's own control flow on the CPU: the headline benchmark script run end to end on the stand-in CUDA runtime
(tests/hostsim, launches recorded and checked but not interpreted -- timings are meaningless there).  Checks the JSON
contract of the line it prints and that no launch, copy or tensor map of the benchmark-sized run breaks a runtime rule
(the run that first showed a dataset conversion launch beyond the grid limit)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

RUNNER = r'''
import sys, runpy, ctypes as C
sys.path[:0] = [{root!r}, {pkg!r}]
from boltzmann_machines import _native
sim = _native.load_library({sim!r})
sim.fakecuda_violation.restype = C.c_char_p
_native._lib = sim
sys.argv = ['bench.py', '--steps', '6', '--warmup', '3', '--no-cpu-baseline', '--dump-outputs', 'dump']
try:
    runpy.run_path({bench!r}, run_name='__main__')
finally:
    print('VIOLATIONS=' + sim.fakecuda_violation().decode())
'''


def test_bench_contract_on_the_host_simulation(tmp_path):
    obj = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
    if not (os.path.isdir(obj) and any(f.endswith('.o') for f in os.listdir(obj))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build.sh')], stdout=subprocess.DEVNULL)
    code = RUNNER.format(root=ROOT, pkg=os.path.join(ROOT, 'boltzmann-machines_b200'),
                         sim=os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim.so'), bench=os.path.join(ROOT, 'bench.py'))
    # 20 batches = 81920 rows: still taller than grid.y can index (the refused-launch case), half the host-side data shuffling
    env = dict(os.environ, BM_BENCH_BATCHES='20', BM_BENCH_FIT_STEPS='40')
    res = subprocess.run([sys.executable, '-c', code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, cwd=str(tmp_path), env=env)
    assert res.returncode == 0, res.stdout[-3000:]
    assert 'VIOLATIONS=\n' in res.stdout + '\n', res.stdout[-1500:]
    line = [l for l in res.stdout.splitlines() if l.startswith('{"metric"')]
    assert len(line) == 1, res.stdout[-1500:]
    out = json.loads(line[0])
    for key in ('metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling', 'vs_baseline',
                'dtype', 'data', 'config', 'gpu_launches', 'clocks', 'roofline', 'e2e'):
        assert key in out, key
    assert out['n_gpus'] == 1 and out['steps'] == 6 and out['higher_is_better'] is True and out['scaling'] == 'weak'
    assert out['config']['workload'].startswith('BernoulliRBM 784-1024') and 'model' not in out['config']
    assert set(out['roofline']) >= {'bound', 'achieved', 'peak', 'unit', 'frac', 'traffic'}
    assert set(out['e2e']) >= {'value', 'unit', 'h2d_bytes_per_step', 'd2h_bytes_per_step'}
    assert out['e2e']['h2d_bytes_per_step'] == 4096 * 784          # one byte per visible unit and row
    assert 'fit_region_failed' not in out['e2e'] and out['e2e']['path'].startswith('Model(**kwargs).fit(X)')
    assert out['gpu_launches'] == 2 * out['steps']                  # the step's program and the update kernel
    # --dump-outputs: the model the last timed step left behind, float32, under the cap
    import numpy as np
    dump = tmp_path / 'dump'
    got = {f.name: np.load(str(f)) for f in dump.iterdir()}
    assert set(got) == {'W.npy', 'vb.npy', 'hb.npy'}, sorted(got)
    assert got['W.npy'].shape == (784, 1024) and got['vb.npy'].shape == (784,) and got['hb.npy'].shape == (1024,)
    assert all(a.dtype == np.float32 for a in got.values())


def test_dump_outputs_samples_what_exceeds_the_cap(tmp_path, monkeypatch):
    """bench.dump_outputs: float64 stays float64, other arrays become float32; an array that would take the total past the cap
    is replaced by a fixed, seeded sample of its elements plus their indices, and the same input gives the same files."""
    import importlib.util
    import numpy as np
    # a private copy of the module: other tests import `bench` with their own environment
    spec = importlib.util.spec_from_file_location('bench_under_test', os.path.join(ROOT, 'bench.py'))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    monkeypatch.setattr(bench, 'DUMP_BYTES', 4000)
    arrays = {'small': np.arange(10, dtype=np.float64), 'big': np.arange(5000, dtype=np.int32).reshape(50, 100)}
    for d in ('a', 'b'):
        bench.dump_outputs(str(tmp_path / d), arrays)
    small, big, idx = (np.load(str(tmp_path / 'a' / n)) for n in ('small.npy', 'big.npy', 'big_index.npy'))
    assert small.dtype == np.float64 and np.array_equal(small, arrays['small'])
    assert big.dtype == np.float32 and np.array_equal(big, arrays['big'].reshape(-1)[idx].astype(np.float32))
    assert np.all(np.diff(idx) > 0) and 0 < big.size < 5000
    total = sum(f.stat().st_size for f in (tmp_path / 'a').iterdir())
    assert total <= 4000 + 3 * 128                                      # (+ the .npy headers)
    for n in ('small.npy', 'big.npy', 'big_index.npy'):
        assert np.array_equal(np.load(str(tmp_path / 'a' / n)), np.load(str(tmp_path / 'b' / n)))


def test_reference_arm_prints_the_same_config_and_runs_exactly_the_steps_it_was_given(tmp_path):
    """`bench.py --impl reference --steps K --warmup W`: the oracle port on the host cores; same `config` object as the CUDA arm,
    exactly K timed steps (each a bounded sample of the workload's step when K full steps would not fit the time budget), and the
    cpu_baseline / e2e objects the contract asks of this arm."""
    env = dict(os.environ, BM_BENCH_REFERENCE_SECONDS='3', BM_BENCH_BATCHES='20')
    res = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '7', '--warmup', '2'],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, cwd=str(tmp_path), env=env)
    assert res.returncode == 0, res.stdout[-3000:]
    out = json.loads([l for l in res.stdout.splitlines() if l.startswith('{"impl"')][0])
    assert out['impl'] == 'reference' and out['steps'] == 7 and out['warmup'] == 2 and out['n_gpus'] == 1
    assert out['metric'] == 'gibbs_updates_per_sec' and out['unit'] == 'updates/s' and out['higher_is_better'] is True
    sys.path.insert(0, ROOT)
    try:
        os.environ['BM_BENCH_BATCHES'] = '20'
        import importlib
        bench = importlib.import_module('bench')
        assert out['config'] == bench.rbm_config('cfg2', 1)
    finally:
        os.environ.pop('BM_BENCH_BATCHES', None)
        sys.path.remove(ROOT)
    assert out['cpu_baseline']['kind'] == 'port' and out['cpu_baseline']['value'] == out['value'] and out['cpu_baseline']['cores'] >= 1
    assert 'rows each of the batch of 4096' in out['cpu_baseline']['sample']          # 9 full steps do not fit 3 seconds
    assert out['e2e'] == {'value': out['value'], 'unit': 'updates/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}


def test_bench_with_two_ranks_on_the_host_simulation(tmp_path):
    """the launch the driver uses for N > 1 (torchrun, one rank per GPU) with both ranks on the stand-in runtime and the shared-memory
    stand-in for NCCL: rank 0 prints one line for the whole job, the engine-level regions and fit() run data parallel, nothing
    breaks a runtime rule"""
    pytest.importorskip('torch')
    obj = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
    if not (os.path.isdir(obj) and any(f.endswith('.o') for f in os.listdir(obj))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build.sh')], stdout=subprocess.DEVNULL)
    env = dict(os.environ, BM_BENCH_BATCHES='4', BM_BENCH_FIT_STEPS='8',
               BM_NCCL_LIB=os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libfakenccl.so'))
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
           '--master-port', str(29900 + os.getpid() % 90), os.path.join(ROOT, 'tools', 'hostsim_run.py'), os.path.join(ROOT, 'bench.py'),
           '--gpus', '2', '--steps', '6', '--warmup', '3', '--no-cpu-baseline']
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert res.returncode == 0, res.stdout[-3000:]
    lines = [l for l in res.stdout.splitlines() if l.startswith('{"metric"')]
    assert len(lines) == 1, res.stdout[-2000:]
    out = json.loads(lines[0])
    assert out['n_gpus'] == 2 and out['steps'] == 6 and out['scaling'] == 'weak'
    assert out['config']['parallelism'] == 'dp2' and out['config']['global_batch'] == 2 * 4096
    assert out['e2e']['h2d_bytes_per_step'] == 2 * 4096 * 784 and out['e2e']['steps'] >= 8 and 'fit_region_failed' not in out['e2e']
    assert res.stdout.count('violations: none') == 2, res.stdout[-2000:]
