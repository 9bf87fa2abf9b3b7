import os
import sys

# The oracle is numpy on small matrices: on a many-core host (the GPU box has 128 hardware threads) a BLAS pool of that size
# spends its time waking threads up -- the AIS ladders of the tiny test models took minutes there and a second here.
for _v in ('OPENBLAS_NUM_THREADS', 'OMP_NUM_THREADS', 'MKL_NUM_THREADS'):
    os.environ.setdefault(_v, '8')

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG_PARENT = os.path.join(ROOT, 'boltzmann-machines_b200')
for p in (ROOT, PKG_PARENT):
    if p not in sys.path:
        sys.path.insert(0, p)


def _build_if_missing():
    """A fresh checkout has no native artefacts (they are git-ignored): build them once, like __graft_entry__.build() does, so
    that the suite does not depend on who ran first.  nvcc cross-compiles without a GPU; without nvcc the tests that need the
    library say so themselves."""
    import shutil
    import subprocess
    lib = os.path.join(PKG_PARENT, 'boltzmann_machines', 'libbm.so')
    if os.path.isfile(lib) or os.environ.get('BM_NO_AUTOBUILD') == '1':
        return
    if shutil.which('nvcc') is None and not os.path.isfile('/usr/local/cuda/bin/nvcc'):
        return
    sys.stderr.write('[conftest] libbm.so is missing: building it (build.sh, about two minutes)\n')
    subprocess.check_call(['bash', os.path.join(ROOT, 'build.sh')], stdout=subprocess.DEVNULL)
    subprocess.call(['make', '-C', os.path.join(ROOT, 'oracle')], stdout=subprocess.DEVNULL)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')
    if not hasattr(config, 'workerinput'):            # (pytest-xdist: only the controller builds)
        _build_if_missing()
    if os.environ.get('BM_HOSTSIM') == '1':
        # Dry run of the GPU tests WITHOUT a GPU: the library's objects on the stand-in runtime, kernels interpreted on the
        # CPU (tests/hostsim).  `BM_HOSTSIM=1 python -m pytest tests/test_dbm_gpu.py -m gpu` -- shapes of benchmark size
        # take minutes per GEMM there; meant for the small-shape tests and for checking a test's own logic and tolerances.
        import ctypes as C
        import subprocess
        subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build.sh')], stdout=subprocess.DEVNULL)
        from boltzmann_machines import _native
        lib = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim.so'))
        lib.fakecuda_violation.restype = C.c_char_p
        lib.fakecuda_skipped.restype = C.c_char_p
        # BM_HOSTSIM_EXECUTE=0: record and check the launches without interpreting them (fast scan of the big-shape tests
        # for refused launches, bad tensor maps and out-of-bounds copies; their numeric assertions then fail, of course)
        lib.fakecuda_set_execute(0 if os.environ.get('BM_HOSTSIM_EXECUTE') == '0' else 1)
        _native._lib = lib
        config._bm_hostsim = lib


# GPU tests not yet run on an H100 (they pass on the host simulation, tests/hostsim): run them after the tests that
# have already passed on the hardware, so that `-x` reports a surprise in one of them without hiding the rest of the suite.
NOT_YET_RUN_ON_A_GPU = ()


def pytest_collection_modifyitems(config, items):
    # combinations that do not exist: float64 models never take the bf16 engine, and the fuzz corpus has its own bf16 test
    # (test_bf16_engine_replays_the_corpus) -- dropped at collection instead of showing up as skips
    void = [it for it in items if 'matches_the_reference[' in it.nodeid and
            any(t in it.nodeid for t in ('bf16-fuzz_', 'bf16-bernoulli_float64'))]
    if void:
        ids = set(id(it) for it in void)
        items[:] = [it for it in items if id(it) not in ids]
        config.hook.pytest_deselected(items=void)
    late = [it for it in items if it.get_closest_marker('gpu') and any(tag in it.nodeid for tag in NOT_YET_RUN_ON_A_GPU)]
    if late:
        ids = set(id(it) for it in late)
        items[:] = [it for it in items if id(it) not in ids] + late


def pytest_unconfigure(config):
    lib = getattr(config, '_bm_hostsim', None)
    if lib is not None:
        v, sk = lib.fakecuda_violation().decode(), lib.fakecuda_skipped().decode()
        print('\n[hostsim] runtime violations: {0}; kernels without a CPU restatement: {1}; program launches checked for dataflow '
              'hazards: {2}, declared dependencies the kernel would not wait for: {3}'.format(
                  v or 'none', sk or 'none', lib.fakecuda_hazard_launches(), lib.fakecuda_unhonoured_dependencies()))


@pytest.fixture(scope='session', autouse=True)
def _bounded_blas_pool():
    """the same bound for a numpy that was imported before this file set the environment"""
    try:
        from threadpoolctl import threadpool_limits
    except ImportError:
        yield
        return
    with threadpool_limits(limits=int(os.environ.get('OPENBLAS_NUM_THREADS', '8')), user_api='blas'):
        yield


@pytest.fixture
def oracle_engines():
    """Route the package's models to the numpy oracle (host-logic tests on CPU)."""
    from boltzmann_machines.base import set_engine_factory
    from oracle.rbm import rbm_factory
    old = set_engine_factory('rbm', rbm_factory)
    try:
        from oracle.dbm import dbm_factory
        old_d = set_engine_factory('dbm', dbm_factory)
    except ImportError:
        old_d = None
    yield
    set_engine_factory('rbm', old)
    set_engine_factory('dbm', old_d)


@pytest.fixture(params=['oracle',
                        pytest.param('cuda-fp32', marks=pytest.mark.gpu),
                        pytest.param('cuda-bf16', marks=pytest.mark.gpu)])
def engines(request, monkeypatch):
    """The engine behind the package's models: numpy oracle (CPU) or libbm.so (GPU)."""
    from boltzmann_machines.base import set_engine_factory
    if request.param == 'oracle':
        from oracle.rbm import rbm_factory
        from oracle.dbm import dbm_factory
        old = set_engine_factory('rbm', rbm_factory)
        old_d = set_engine_factory('dbm', dbm_factory)
        yield request.param
        set_engine_factory('rbm', old)
        set_engine_factory('dbm', old_d)
    else:
        monkeypatch.setenv('BM_COMPUTE', request.param.split('-')[1])
        old = set_engine_factory('rbm', None)
        old_d = set_engine_factory('dbm', None)
        yield request.param
        set_engine_factory('rbm', old)
        set_engine_factory('dbm', old_d)


@pytest.fixture
def workdir(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    return tmp_path


@pytest.fixture(scope='session')
def hostsim_library():
    """tests/hostsim: libbm's own objects linked against the stand-in CUDA runtime, kernels interpreted on the CPU."""
    import ctypes as C
    import subprocess
    obj = os.path.join(ROOT, 'boltzmann-machines_b200', 'build')
    if not (os.path.isdir(obj) and any(f.endswith('.o') for f in os.listdir(obj))):
        pytest.skip('library objects not built (run build.sh / __graft_entry__.build())')
    subprocess.check_call(['bash', os.path.join(ROOT, 'tests', 'hostsim', 'build.sh')], stdout=subprocess.DEVNULL)
    from boltzmann_machines import _native
    lib = _native.load_library(os.path.join(ROOT, 'tests', 'hostsim', '_build', 'libbm_hostsim.so'))
    lib.fakecuda_violation.restype = C.c_char_p
    lib.fakecuda_skipped.restype = C.c_char_p
    return lib


@pytest.fixture
def hostsim_engines(hostsim_library, monkeypatch):
    """Route the package's CUDA engines to the host simulation (fp32 compute, launches interpreted); checks on exit that
    nothing was skipped and no runtime rule was violated."""
    from boltzmann_machines import _native
    from boltzmann_machines.base import set_engine_factory
    lib = hostsim_library
    old_lib, old_ctx = _native._lib, dict(_native.Context._default)
    _native._lib = lib
    _native.Context._default.clear()
    lib.fakecuda_reset()
    lib.fakecuda_set_execute(1)
    monkeypatch.setenv('BM_COMPUTE', 'fp32')
    old = set_engine_factory('rbm', None), set_engine_factory('dbm', None)
    yield lib
    set_engine_factory('rbm', old[0])
    set_engine_factory('dbm', old[1])
    lib.fakecuda_set_execute(0)
    violation, skipped = lib.fakecuda_violation().decode(), lib.fakecuda_skipped().decode()
    _native.Context._default.clear()
    _native.Context._default.update(old_ctx)
    _native._lib = old_lib
    assert violation == '', violation
    assert skipped == '', skipped
