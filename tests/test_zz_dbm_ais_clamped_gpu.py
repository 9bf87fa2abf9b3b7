"""AIS estimates of log p*(v) with v clamped (bm_dbm_ais_clamped, DESIGN.md §5.4g) on the H100.

* Run by run against the bf16 emulation (tests/dbm_ais_clamped_oracle.py) at small ragged shapes (L = 2, 3, 4; k = 1, 3;
  binary and grey rows) and at cfg4's shape 784-512-1024 (a few rows, runs and temperatures).
* Identity at the benchmark shape: at 784-512-1024 with W_1 = 0 and b_2 = 0 every increment is deterministic, and each run
  must equal b_v.v + sum softplus(b_1 + v bf16(W_0)) + H_2 log 2 within IDENTITY_TOL (derived below).
* Against the truth: 784-20-500 (L = 2) and 784-12-300-12 (L = 3, n_odd = 24) with data-like biases, W rounded to bf16 so that
  the chains and the enumeration see one model; 128 binary and 128 grey rows (grey values rounded to bf16).  The per-row AIS
  estimate (100 runs x 1000 temperatures, k = 1) against bm_dbm_exact's log p*(v), gated against the float64 ladder's own
  measured bias (TRUTH_BIAS below).
* Repeated calls with one seed agree bit for bit.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dbm_ais_clamped_oracle as Q  # noqa: E402
from oracle.dbm_bf16 import _r  # noqa: E402
from test_dbm_ais_depth_host import make_cfg, params, same_runs  # noqa: E402

pytestmark = pytest.mark.gpu

RAGGED = {2: (37, (21, 11)), 3: (29, (19, 9, 13)), 4: (13, (21, 6, 9, 7))}


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


def engine(n, Hs, p, V, **kw):
    e = n.CudaDBM(make_cfg(Hs, V, **kw))
    assert e.compute == 'bf16'
    e.set_params(p)
    return e


def model(Hs, scale=0.1, seed=0, V=784):
    """data-like (as test_zz_dbm_exact_gpu.model): visible biases around -2.5, hidden biases around -1; W rounded to bf16"""
    rng = np.random.RandomState(seed)
    sizes = [V] + list(Hs)
    d = {'vb': (rng.randn(V) - 2.5).astype(np.float32)}
    for i in range(len(Hs)):
        d['W' + sfx(i)] = _r(scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + sfx(i)] = (0.5 * rng.randn(sizes[i + 1]) - 1.0).astype(np.float32)
    return d


def data_rows(V=784, n=256, seed=1):
    """n / 2 binary rows, then n / 2 grey rows with values rounded to bf16"""
    rng = np.random.RandomState(seed)
    X = (rng.rand(n, V) < 0.12).astype(np.float32)
    X[n // 2:] = _r(rng.rand(n - n // 2, V) * 0.3).astype(np.float32)
    return X


@pytest.mark.parametrize('grey', [False, True], ids=['binary', 'grey'])
@pytest.mark.parametrize('L', [2, 3, 4])
@pytest.mark.parametrize('k,n_betas', [(1, 60), (3, 25)], ids=['k1', 'k3'])
def test_small_shapes_equal_the_emulation(L, k, n_betas, grey):
    n = _native()
    V, Hs = RAGGED[L]
    p = params(V, Hs, scale=0.3, seed=L)
    rng = np.random.RandomState(L)
    X = (rng.rand(6, V) if grey else (rng.rand(6, V) < 0.4)).astype(np.float32)
    e = engine(n, Hs, p, V)
    try:
        got = e.ais_clamped(X, 8, n_betas, k, 77, row0=3)
    finally:
        e.close()
    same_runs(got.ravel(), Q.ais(p, X, 8, n_betas, k, 77, row0=3, bf16=True).ravel(), (L, k, n_betas, grey))


def test_benchmark_shape_equals_the_emulation():
    n = _native()
    Hs = (512, 1024)
    p = model(Hs, scale=0.05, seed=3)
    X = data_rows(n=4, seed=3)
    e = engine(n, Hs, p, 784)
    try:
        got = e.ais_clamped(X, 3, 12, 1, 5)
    finally:
        e.close()
    want = Q.ais(p, X, 3, 12, 1, 5, bf16=True)
    same_runs(got.ravel(), want.ravel(), '784-512-1024')


# Each run telescopes to b_v.v + sum_n [softplus(z_n) - log 2] + (H_1 + H_2) log 2 with z = b_1 + v bf16(W_0).  What differs
# from the float64 value: z_n, an fp32 sum of K = 784 exact bf16 products, is off by at most K u sum_k |v_k W_kn| (u = 2^-24),
# and softplus' <= 1 passes that on; the n_T float32 increments of unit n, each softplus(b z) - softplus(a z) of one sign, are
# off by a few u of their sum |softplus(z_n) - log 2| each, and the epilogue's float32 partial sums over up to H_1 units add
# H_1 u of that.  IDENTITY_TOL = 784 u A + (H_1 + 16) u B with A = sum_n sum_k |v_k W_kn|, B = sum_n |softplus(z_n) - log 2|.
U32 = 2.0 ** -24


def test_identity_at_the_benchmark_shape():
    n = _native()
    Hs = (512, 1024)
    p = model(Hs, scale=0.05, seed=4)
    p['W_1'] = np.zeros_like(p['W_1'])
    p['hb_1'] = np.zeros_like(p['hb_1'])
    X = data_rows(n=16, seed=4)
    e = engine(n, Hs, p, 784)
    try:
        got = e.ais_clamped(X, 4, 50, 1, 9)
    finally:
        e.close()
    W0 = p['W'].astype(np.float64)
    Xr = _r(X).astype(np.float64)
    z = Xr @ W0 + p['hb'].astype(np.float64)
    sp = np.logaddexp(0.0, z)
    want = X.astype(np.float64) @ p['vb'].astype(np.float64) + sp.sum(axis=1) + Hs[1] * np.log(2.)
    A = (np.abs(Xr) @ np.abs(W0)).sum(axis=1)
    B = np.abs(sp - np.log(2.)).sum(axis=1)
    tol = 784 * U32 * A + (Hs[0] + 16) * U32 * B
    err = np.abs(got - want[:, None])
    assert np.all(err <= tol[:, None]), (err.max(axis=1), tol)


# The gate against the truth.  The ladder weighs each state with the increment of the temperature it was just drawn at (the
# depth ladder's arrangement, DESIGN.md §5.4g), which biases the estimate up by O(1/n_T).  The float64 ladder on the CPU at these
# models and settings (100 runs x 1000 temperatures, k = 1; 16 binary and 16 grey rows of the same data) sits TRUTH_BIAS nats
# above the exact log p*(v) on average, with per-row standard errors up to 0.043.  Gate: the mean of AIS - exact within 0.05 of
# that bias, and every row within 5 of its own standard errors + 0.05 of it.
TRUTH_RUNS, TRUTH_BETAS = 100, 1000
TRUTH_BIAS = {'784-20-500': 0.129, '784-12-300-12': 0.070}


@pytest.mark.parametrize('Hs', [(20, 500), (12, 300, 12)], ids=['784-20-500', '784-12-300-12'])
def test_against_the_exact_log_p_v(Hs):
    n = _native()
    p = model(Hs, scale=0.1, seed=7)
    X = data_rows(n=256, seed=8)
    e = engine(n, Hs, p, 784)
    try:
        runs = e.ais_clamped(X, TRUTH_RUNS, TRUTH_BETAS, 1, 11)
        exact, _ = e.exact(X)
    finally:
        e.close()
    est = Q.log_mean_rows(runs)
    w = np.exp(runs - runs.max(axis=1, keepdims=True))
    se = w.std(axis=1) / w.mean(axis=1) / np.sqrt(TRUTH_RUNS)
    d = est - exact - TRUTH_BIAS['-'.join(map(str, (784,) + Hs))]
    print('AIS - exact - bias at', Hs, ': mean %.4f, |max| %.4f, max se %.4f' % (d.mean(), np.abs(d).max(), se.max()))
    assert abs(d.mean()) < 0.05, d.mean()
    assert np.all(np.abs(d) < 5.0 * se + 0.05), (d, se)


def test_repeated_calls_agree_bit_for_bit():
    n = _native()
    V, Hs = RAGGED[3]
    p = params(V, Hs, scale=0.3, seed=12)
    X = (np.random.RandomState(12).rand(5, V) < 0.4).astype(np.float32)
    e = engine(n, Hs, p, V)
    try:
        a = e.ais_clamped(X, 50, 40, 2, 3)
        b = e.ais_clamped(X, 50, 40, 2, 3)
    finally:
        e.close()
    np.testing.assert_array_equal(a, b)
