"""The C-ABI library loads on a CPU-only box and exports every symbol include/bm.h
declares; without a GPU it refuses to create a context instead of falling back."""
import os
import re

import pytest

from boltzmann_machines import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, 'include', 'bm.h')).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(bm_[a-z0-9_]+)\s*\(', text)))


def test_header_and_binding_agree():
    assert declared_symbols() == sorted(_native.EXPORTS)


def test_library_exports_every_declared_symbol():
    lib = _native.load_library()
    for name in declared_symbols():
        assert hasattr(lib, name), name
    assert b'sm_90a' in lib.bm_version()


def test_no_cpu_fallback_without_gpu():
    if _native.device_count() > 0:
        pytest.skip('a GPU is visible')
    with pytest.raises(RuntimeError, match='no CUDA device'):
        _native.Context()
    with pytest.raises(RuntimeError):
        from boltzmann_machines.rbm import BernoulliRBM
        BernoulliRBM(n_visible=4, n_hidden=3, model_path='/tmp/_bm_nofallback/').init()


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, 'boltzmann-machines_b200')
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                src = open(os.path.join(d, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle\b', src, flags=re.M), os.path.join(d, f)


def test_as_bytes_is_lossless_or_declines():
    """engine.pin keeps a training set as bytes only when that is exact (bm_rbm_train_epoch_u8)."""
    import numpy as np
    from boltzmann_machines import _native
    X = (np.random.RandomState(0).rand(7, 5) < 0.3).astype(np.float32)
    Xb = _native.as_bytes(X)
    assert Xb.dtype == np.uint8 and np.array_equal(Xb.astype(np.float32), X)
    assert _native.as_bytes(np.arange(256, dtype=np.float64).reshape(16, 16)).dtype == np.uint8
    assert _native.as_bytes(X * 0.5) is None                      # grey levels
    assert _native.as_bytes(X - 1.0) is None                      # negative
    assert _native.as_bytes(X + 255.0) is None                    # out of range
    assert _native.as_bytes(np.array([[np.nan, 1.0]], dtype=np.float32)) is None
    assert _native.as_bytes(np.zeros((0, 5), dtype=np.float32)) is None
