"""Exact log Z and log p(v) of binary DBMs with a narrow odd side (bm_dbm_exact, DESIGN.md §5.4f) on the H100.

* 784-20 (L = 1) and 784-16-500 (L = 2) with data-like visible biases: log Z and log p*(v) of 256 binary and grey rows against
  the chunked float64 enumeration (tests/dbm_exact_oracle.py) within 1e-4 nats.
* n_odd = 32 end to end: a 784-32 RBM whose hidden units 0-15 see only v[0:392] and units 16-31 only v[392:784] has
  log Z = log Z of the two 392-16 halves, each enumerated in float64; its rows have the closed form
  log p*(v) = b_v.v + sum softplus(c + v W).
* |z| ~ 1e3: finite, and equal to float64 to 1e-6 relative.
* AIS against the truth at 784-20 and 784-20-500 (W rounded to bf16 first, so that the chains and the sum see one model):
  the uniform ladder (256 runs x 1000 temperatures) within 1 nat; the data base's gap is printed, not gated.
* Repeated calls agree to 1e-12.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dbm_exact_oracle as E  # noqa: E402
from test_dbm_ais_depth_host import make_cfg  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _native():
    from boltzmann_machines import _native as n
    try:
        n.load_library()
        if n.device_count() < 1:
            pytest.skip('no CUDA device')
    except RuntimeError as e:
        pytest.skip(str(e))
    return n


def sfx(i):
    return '' if i == 0 else '_%d' % i


def model(Hs, scale=0.1, seed=0, V=784):
    """data-like: visible biases around -2.5 (most pixels off), hidden biases around -1"""
    rng = np.random.RandomState(seed)
    sizes = [V] + list(Hs)
    d = {'vb': (rng.randn(V) - 2.5).astype(np.float32)}
    for i in range(len(Hs)):
        d['W' + sfx(i)] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + sfx(i)] = (0.5 * rng.randn(sizes[i + 1]) - 1.0).astype(np.float32)
    return d


def data_rows(V=784, n=256, seed=1):
    rng = np.random.RandomState(seed)
    X = (rng.rand(n, V) < 0.12).astype(np.float32)
    X[n // 2:] = (rng.rand(n - n // 2, V) * 0.3).astype(np.float32)
    return X


def engine(n, Hs, p, V=784, **kw):
    e = n.CudaDBM(make_cfg(Hs, V, **kw))
    assert e.compute == 'bf16'
    e.set_params(p)
    return e


def softplus(z):
    return np.logaddexp(0.0, z)


@pytest.mark.parametrize('Hs', [(20,), (16, 500)], ids=['784-20', '784-16-500'])
def test_against_float64(Hs):
    n = _native()
    p = model(Hs, seed=len(Hs))
    X = data_rows()
    e = engine(n, Hs, p)
    lp, lz = e.exact(X)
    want_z, want_p = E.exact(p, X, chunk_bits=14)
    print('%s: log Z %.6f (float64 %.6f), max |d log p*| %.2e' % (Hs, lz, want_z, np.max(np.abs(lp - want_p))))
    assert abs(lz - want_z) < TOL
    np.testing.assert_allclose(lp, want_p, rtol=0, atol=TOL)
    lp2, lz2 = e.exact(X)
    assert abs(lz2 - lz) < 1e-12 and np.max(np.abs(lp2 - lp)) < 1e-12
    assert abs(e.exact(None)[1] - lz) < 1e-12
    e.close()


def test_thirty_two_odd_units():
    n = _native()
    p = model((32,), seed=7)
    p['W'][:392, 16:] = 0.
    p['W'][392:, :16] = 0.
    halves = []
    for cols, rows_ in ((slice(0, 16), slice(0, 392)), (slice(16, 32), slice(392, 784))):
        q = {'vb': p['vb'][rows_], 'W': p['W'][rows_, cols], 'hb': p['hb'][cols]}
        halves.append(E.exact(q)[0])
    X = data_rows(n=64, seed=3)
    e = engine(n, (32,), p)
    lp, lz = e.exact(X)
    W, vb, hb = (p[k].astype(np.float64) for k in ('W', 'vb', 'hb'))
    want_p = X.astype(np.float64) @ vb + softplus(X.astype(np.float64) @ W + hb).sum(axis=1)
    print('784-32: log Z %.6f (halves %.6f), max |d log p*| %.2e' % (lz, sum(halves), np.max(np.abs(lp - want_p))))
    assert abs(lz - sum(halves)) < TOL
    np.testing.assert_allclose(lp, want_p, rtol=0, atol=TOL)
    e.close()


def test_extreme_pre_activations():
    n = _native()
    Hs = (12,)
    rng = np.random.RandomState(5)
    p = {'vb': (300. * rng.randn(784)).astype(np.float32), 'W': (4. * rng.randn(784, 12)).astype(np.float32),
         'hb': (500. * rng.randn(12)).astype(np.float32)}
    X = data_rows(n=32)
    e = engine(n, Hs, p)
    lp, lz = e.exact(X)
    want_z, want_p = E.exact(p, X)
    z = X @ p['W'] + p['hb']
    print('|z| up to %.0f; log Z %.6f (float64 %.6f)' % (np.abs(z).max(), lz, want_z))
    assert np.abs(z).max() > 500.
    assert np.isfinite(lz) and np.all(np.isfinite(lp))
    assert abs(lz - want_z) < 1e-6 * abs(want_z)
    np.testing.assert_allclose(lp, want_p, rtol=1e-6, atol=TOL)
    e.close()


@pytest.mark.parametrize('Hs', [(20,), (20, 500)], ids=['784-20', '784-20-500'])
def test_ais_against_the_truth(Hs):
    n = _native()
    p = model(Hs, scale=0.05, seed=11)
    for k in p:
        if k.startswith('W'):
            p[k] = E.bf16_split(p[k])[0]                     # the chains read bf16(W): give the sum the same model
    e = engine(n, Hs, p)
    exact = e.exact(None)[1]
    rng = np.random.RandomState(4)
    X = (rng.rand(5000, 784) < 1. / (1. + np.exp(-p['vb']))).astype(np.float32)
    pr = (X.astype(np.float64).sum(axis=0) + 1.) / (len(X) + 2.)
    base = [np.log(pr / (1. - pr)).astype(np.float32)] + [None] * len(Hs)
    uni = e.ais(256, 1000, 1, 1)
    bas = e.ais(256, 1000, 1, 1, base=base)
    est_u = float(np.logaddexp.reduce(uni) - np.log(len(uni)))
    est_b = float(np.logaddexp.reduce(bas) - np.log(len(bas)))
    print('%s: exact log Z %.4f, uniform AIS gap %+.4f, data-base AIS gap %+.4f' % (Hs, exact, est_u - exact, est_b - exact))
    assert abs(est_u - exact) < 1.0
    e.close()
