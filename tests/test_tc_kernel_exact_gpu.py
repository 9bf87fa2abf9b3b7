"""The tensor-core op kernel (csrc/bm_tc.cu) element by element, through the one-op hook `_native.debug_tc_op`.

References are float64, computed from the bf16-rounded operands, with the Philox draws of oracle/philox.py.  Operands are
small integers, so every product and partial sum is exact in fp32 and the accumulator is exactly known whatever the kernel's
accumulation order: raw GEMMs must match bit for bit, and an epilogue may differ from its float64 statement only by its own
arithmetic, whose error is bounded per element below.  Every output buffer has guard rows and columns filled with a sentinel,
and every case checks that nothing outside the op's window was written.

The contract on the edges of an output: rows >= M are never written; fp32 columns >= N are never written; bf16 columns
>= round_up(N, 8) are never written.  bf16 columns [N, round_up(N, 8)) of rows < M are exempt: the TMA store of a granule is
clipped to [M, N], but a clip inside a 16-byte unit may overwrite the rest of that unit."""
import os

import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P

pytestmark = pytest.mark.gpu

HOSTSIM = os.environ.get('BM_HOSTSIM') == '1'
LOG2E = 1.4426950408889634
ULP = 2.0 ** -24                      # unit roundoff of fp32
# documented accuracy of the fast intrinsics the epilogue uses (CUDA C Programming Guide, PTX ISA)
LOGF_ABS = 2.0 ** -21.41              # __logf on [0.5, 2]; 3 ulp elsewhere
SINCOS_ABS = 2.0 ** -20.5             # sin.approx / cos.approx over |x| <= 100 pi (__sincosf on [0, 2 pi))


# ---- helpers -------------------------------------------------------------------------------------------------------------
def bf16_bits_to_f64(b):
    return (np.asarray(b).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def bf16r(x):
    """x rounded to fp32, then to the nearest bf16 (ties to even): what the kernel's pack does to its fp32 value."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def first(mask):
    idx = np.argwhere(mask)
    return tuple(int(i) for i in idx[0])


def assert_equal(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want))) if got.dtype.kind == 'f' else got != want
    if bad.any():
        at = first(bad)
        raise AssertionError('{0}: {1} of {2} elements differ, first at (m, n) = {3}: got {4!r}, want {5!r}'.format(
            what, int(bad.sum()), bad.size, at, got[at], want[at]))


def assert_bf16_within(bits, ref, tol, what):
    """bf16 output `bits` [M, N] against float64 `ref` whose fp32 computation may be off by `tol`: the kernel's value must be
    the rounding of some value in [ref - tol, ref + tol], and never more than one bf16 ulp from bf16(ref).  Returns the
    number of elements that differ from bf16(ref) (values within `tol` of a rounding midpoint)."""
    got = bf16_bits_to_f64(bits)
    lo, hi, near = bf16r(ref - tol), bf16r(ref + tol), bf16r(ref)
    ulp = np.maximum(np.abs(near), 2.0 ** -126) * 2.0 ** -7
    bad = ~((got >= lo) & (got <= hi) & (np.abs(got - near) <= ulp))
    if bad.any():
        at = first(bad)
        raise AssertionError('{0}: {1} of {2} elements outside the rounding of ref +- tol, first at (m, n) = {3}: got {4!r}, '
                             'ref {5!r}, tol {6:.3g}'.format(what, int(bad.sum()), bad.size, at, got[at], ref[at],
                                                            np.broadcast_to(tol, ref.shape)[at]))
    return int((got != near).sum())


def assert_f32_within(got, ref, tol, what):
    d = np.abs(np.asarray(got, np.float64) - ref)
    bad = ~(d <= tol)
    if bad.any():
        at = first(bad)
        raise AssertionError('{0}: {1} of {2} elements off by more than tol, first at (m, n) = {3}: got {4!r}, ref {5!r}, '
                             'tol {6:.3g}'.format(what, int(bad.sum()), bad.size, at, got[at], ref[at],
                                                 np.broadcast_to(tol, ref.shape)[at]))


def assert_guards(out, M, N):
    """nothing outside the op's window was written (see the module docstring for the exempt bf16 padding columns)"""
    n8 = (N + 7) // 8 * 8
    for name in ('mean', 'state'):
        if name in out:
            b = out[name]
            assert_equal(b[M:], np.full_like(b[M:], _native.BF16_SENTINEL), name + ' guard rows')
            assert_equal(b[:M, n8:], np.full_like(b[:M, n8:], _native.BF16_SENTINEL), name + ' guard columns')
    if 'f32' in out:
        b = out['f32'].view(np.uint32)
        for s in range(b.shape[0]):
            assert_equal(b[s, M:], np.full_like(b[s, M:], _native.F32_SENTINEL), 'f32 guard rows (split %d)' % s)
            assert_equal(b[s, :M, N:], np.full_like(b[s, :M, N:], _native.F32_SENTINEL), 'f32 guard columns (split %d)' % s)
    if 'logw' in out:
        assert out['logw'][M] == _native.LOGW_SENTINEL, 'logw guard entry written: %r' % out['logw'][M]


def operands(rng, M, N, K, a_t, b_t, lo=-3, hi=3, density=1.0):
    """integer operands in [lo, hi] (exact in bf16), a `density` fraction of them nonzero"""
    def draw(shape):
        x = rng.randint(lo, hi + 1, size=shape).astype(np.float32)
        if density < 1.0:
            x *= rng.rand(*shape) < density
        return x
    A = draw((K, M) if a_t else (M, K))
    B = draw((K, N) if b_t else (N, K))
    return A, B


def product(A, B, a_t, b_t):
    A = np.asarray(A, np.float64)
    B = np.asarray(B, np.float64)
    return (A.T if a_t else A) @ (B.T if b_t else B).T


def bf16_values(x):
    return bf16r(x).astype(np.float32)


# ---- 1. exact GEMMs ------------------------------------------------------------------------------------------------------
MS = (1, 63, 65, 128, 129, 255, 257, 600)
NS = (1, 8, 17, 70, 130, 784)
KS = (1, 15, 16, 63, 64, 65, 840)
LAYOUTS = ((False, False), (False, True), (True, False), (True, True))


def exact_cases():
    """A covering design instead of the cross product: every (layout, forced width) once -- all multiples of 16 up to 256
    for a K-major B, 64 / 128 / 192 / 256 for an MN-major B -- with both row groupings, and M, N, K cycled through their
    lists with co-prime strides so that every value of each axis meets several values of the others."""
    cases = []
    i = 0
    for a_t, b_t in LAYOUTS:
        widths = (64, 128, 192, 256) if b_t else tuple(range(16, 257, 16))
        for bn in widths:
            cases.append(dict(M=MS[i % len(MS)], N=NS[(5 * i + 1) % len(NS)], K=KS[(3 * i + 2) % len(KS)], a_t=a_t, b_t=b_t,
                              bn=bn, cluster=1 + (i // 2) % 2, pitch=1 + i % 2))
            i += 1
    return cases


@pytest.mark.parametrize('case', exact_cases(), ids=lambda c: 'M{M}-N{N}-K{K}-at{a_t:d}-bt{b_t:d}-bn{bn}-cl{cluster}-ld{pitch}'.format(**c))
def test_exact_gemm(case):
    M, N, K = case['M'], case['N'], case['K']
    rng = np.random.RandomState(M * 7 + N * 11 + K * 13 + case['bn'])
    A, B = operands(rng, M, N, K, case['a_t'], case['b_t'])
    out = _native.debug_tc_op([(A, B, case['a_t'], case['b_t'], False)], outputs=('f32',), force_bn=case['bn'],
                              force_cluster=case['cluster'], f32_ld=(N + 7) // 8 * 8 + case['pitch'])   # odd / even row pitch
    assert out['plan']['mode'] == 'RAW_F32' and out['plan']['bn'] == case['bn'] and out['plan']['cluster'] == case['cluster']
    assert_equal(out['f32'][0, :M, :N], product(A, B, case['a_t'], case['b_t']).astype(np.float32), 'C')
    assert_guards(out, M, N)


@pytest.mark.parametrize('M,N,K1,K2,b_t1,b_t2,neg1,neg2,bn,cluster', [
    (600, 784, 840, 130, True, False, False, True, 128, 2),       # the DBM shape: x W_i (MN-major B) + y W_{i+1}^T (K-major)
    (257, 130, 65, 1000, False, True, True, False, 64, 1),
    (129, 70, 15, 63, False, False, True, True, 112, 2),
    (65, 17, 64, 16, True, True, False, True, 192, 1),
])
def test_exact_two_pairs(M, N, K1, K2, b_t1, b_t2, neg1, neg2, bn, cluster):
    rng = np.random.RandomState(M + N + K1 + K2)
    A1, B1 = operands(rng, M, N, K1, False, b_t1)
    A2, B2 = operands(rng, M, N, K2, True, b_t2)
    out = _native.debug_tc_op([(A1, B1, False, b_t1, neg1), (A2, B2, True, b_t2, neg2)], force_bn=bn, force_cluster=cluster)
    want = (-1.0 if neg1 else 1.0) * product(A1, B1, False, b_t1) + (-1.0 if neg2 else 1.0) * product(A2, B2, True, b_t2)
    assert out['plan']['mode'] == 'RAW_F32'
    assert_equal(out['f32'][0, :M, :N], want.astype(np.float32), 'C')
    assert_guards(out, M, N)


@pytest.mark.parametrize('M,N,K1,K2,splits', [(784, 1024, 320, 0, 5), (300, 130, 200, 200, 7), (65, 70, 128, 0, 2),
                                               (129, 17, 130, 65, 5)])
def test_exact_split_k(M, N, K1, K2, splits):
    """split s writes its partial sums to slab s; with K2 the splits cut across the two pairs (dW: X^T h0 - v^T h).
    splits = total K chunks: one chunk per split."""
    rng = np.random.RandomState(splits)
    A1, B1 = operands(rng, M, N, K1, True, True)
    pairs = [(A1, B1, True, True, False)]
    want = product(A1, B1, True, True)
    if K2:
        A2, B2 = operands(rng, M, N, K2, True, True)
        pairs.append((A2, B2, True, True, True))
        want = want - product(A2, B2, True, True)
    out = _native.debug_tc_op(pairs, splits=splits)
    assert out['plan']['units'] % splits == 0
    partial = out['f32'][:, :M, :N].astype(np.float64)
    assert_equal(partial.sum(axis=0).astype(np.float32), want.astype(np.float32), 'sum of the split-K partials')
    assert_guards(out, M, N)


# ---- epilogues -----------------------------------------------------------------------------------------------------------
def sigmoid_tol(p, e_pre):
    """error of ex2.approx / rcp.approx sigmoid of a pre-activation that is itself off by e_pre"""
    return p * (1.0 - p) * e_pre + 2.0 ** -21 * p


def gaussian_noise(M, N, seed, site, t, tick, row0):
    """float64 Box-Muller of the element's two Philox words (oracle/philox.py's layout), and the bound of the kernel's
    __logf / __sincosf version's error"""
    n4 = (N + 3) // 4 * 4
    w = P.site_words(M, n4, seed, site, t, tick, row0).reshape(M, n4 // 4, 2, 2)
    u1 = np.maximum(P.u32_to_float(w[..., 0]).astype(np.float64), np.float32(1e-7))
    th = 2.0 * np.pi * P.u32_to_float(w[..., 1]).astype(np.float64)
    L = np.log(u1)
    r = np.sqrt(-2.0 * L)
    dL = np.where(u1 >= 0.5, LOGF_ABS, 4.0 * 2.0 ** -23 * np.abs(L))
    dr = np.minimum(dL / np.maximum(r, 1e-30), np.sqrt(2.0 * dL)) + 2.0 * ULP * r
    dtrig = SINCOS_ABS + 2.0 * ULP * th
    g = np.stack([np.sin(th) * r, np.cos(th) * r], axis=-1).reshape(M, n4)[:, :N]
    dg = np.repeat((dr + r * dtrig)[..., None], 2, axis=-1).reshape(M, n4)[:, :N] + 2.0 * ULP * np.abs(g)
    return g, dg


REPORT = {'bernoulli_ties': 0, 'bernoulli_checked': 0, 'gauss_max_dev': 0.0}


def check_epilogue(out, C, spec, M, N):
    """every output of a non-AIS op against the float64 statement of its epilogue"""
    acc_scale, bias_scale = spec.get('acc_scale', 1.0), spec.get('bias_scale', 1.0)
    sigma = spec.get('sigma')
    bias = spec.get('bias')
    a = acc_scale * C * (1.0 if sigma is None else np.asarray(sigma, np.float64)[None, :])
    b = np.zeros(N) if bias is None else bias_scale * np.asarray(bias, np.float64)
    pre = a + b[None, :]
    # fp32 scale, sigma multiply, bias add (and the folded -log2 e of the sigmoid): a few roundings of the operands' size
    e_pre = 4.0 * ULP * (np.abs(a) + np.abs(b)[None, :])
    act = spec.get('act', 'linear')
    if act == 'sigmoid':
        mean = 1.0 / (1.0 + np.exp(-pre))
        tol = sigmoid_tol(mean, e_pre)
    elif act == 'softplus':
        mean = np.logaddexp(0.0, pre)
        # max(x, 0) + log1pf(__expf(-|x|)): the pre-activation's error times softplus' = sigmoid, __expf's 2 + 1.173 |x|
        # ulp carried through log1p, log1pf's and the final add's roundings
        e = np.exp(-np.abs(pre))
        tol = (1.0 / (1.0 + np.exp(-pre))) * e_pre + (2.0 + 1.173 * np.abs(pre)) * ULP * e / (1.0 + e) + 4.0 * ULP * mean
    else:
        mean, tol = pre, e_pre + ULP * np.abs(pre)
    seed, site, t = spec.get('seed', 0), spec.get('site', 0), spec.get('t', 0)
    tick, row0 = spec.get('tick', 0) + spec.get('tick_off', 0), spec.get('row0', 0)
    sample = spec.get('sample')
    if 'mean' in out:
        assert_bf16_within(out['mean'][:M, :N], mean, tol, 'bf16 means')
    if 'f32' in out:
        if act == 'linear' and sigma is None and bias is None:
            assert_equal(out['f32'][0, :M, :N], mean.astype(np.float32), 'raw fp32 accumulators')
        else:
            assert_f32_within(out['f32'][0, :M, :N], mean, tol + 2.0 * ULP * np.abs(mean), 'fp32 means')
    if 'state' in out:
        if sample == 'bernoulli':
            u = P.uniform_at(M, N, seed, site, t, tick, row0).astype(np.float64)
            check_bernoulli(out['state'][:M, :N], u, mean, tol, 'Bernoulli states')
        elif sample == 'gaussian':
            ns = np.ones(N) if spec.get('noise_sigma') is None else np.asarray(spec['noise_sigma'], np.float64)
            g, dg = gaussian_noise(M, N, seed, site, t, tick, row0)
            st = mean + ns[None, :] * g
            stol = tol + np.abs(ns)[None, :] * dg + 2.0 * ULP * np.abs(st)
            got = bf16_bits_to_f64(out['state'][:M, :N])
            REPORT['gauss_max_dev'] = max(REPORT['gauss_max_dev'], float(np.abs(got - bf16r(st)).max()))
            assert_bf16_within(out['state'][:M, :N], st, stol, 'Gaussian states')
        else:
            assert_bf16_within(out['state'][:M, :N], mean, tol, 'states (no sampling)')
    assert_guards(out, M, N)


def check_bernoulli(bits, u, p, tol, what):
    """states are exactly u < p; a disagreement is allowed only where |u - p| is within the kernel's error of p"""
    s = bf16_bits_to_f64(bits)
    assert_equal(np.isin(s, (0.0, 1.0)), np.ones(s.shape, bool), what + ' are 0 / 1')
    want = (u < p).astype(np.float64)
    differ = s != want
    tie = np.abs(u - p) <= tol
    bad = differ & ~tie
    if bad.any():
        at = first(bad)
        raise AssertionError('{0}: {1} of {2} draws are not u < p, first at (m, n) = {3}: state {4}, u {5!r}, p {6!r}'.format(
            what, int(bad.sum()), bad.size, at, s[at], u[at], p[at]))
    REPORT['bernoulli_ties'] += int(differ.sum())
    REPORT['bernoulli_checked'] += s.size


# the edges every mode runs over: ragged M across the 64- and 128-row edges, ragged N across 64-column edges, row0 0 / 1000,
# nonzero t and tick, widths 64 / 128 / 192 / 256 and both row groupings (bn None: the tile heuristic)
EDGES = [dict(M=63, N=70, bn=64, cluster=1, row0=0, t=3, tick=5, tick_off=0),
         dict(M=129, N=130, bn=128, cluster=2, row0=1000, t=1, tick=9, tick_off=2),
         dict(M=257, N=200, bn=192, cluster=2, row0=0, t=7, tick=2, tick_off=1),
         dict(M=200, N=321, bn=256, cluster=1, row0=1000, t=2, tick=11, tick_off=0),
         dict(M=65, N=64, bn=None, cluster=0, row0=1000, t=5, tick=1, tick_off=3)]


def edge_operands(e, i):
    """sparse {-1, 0, 1} operands (exact) and a power-of-two acc_scale that spread acc_scale * C over about [-8, 8]"""
    rng = np.random.RandomState(100 + i)
    K, acc_scale = (96, 1.0) if i % 2 == 0 else (384, 0.5)
    A, B = operands(rng, e['M'], e['N'], K, i % 2 == 1, i % 3 == 1, lo=-1, hi=1, density=0.55)
    bias = bf16_values(rng.uniform(-2.0, 2.0, e['N']))
    return A, B, i % 2 == 1, i % 3 == 1, acc_scale, bias


MODE_SPECS = {
    'SIG_BERN_MEAN_STATE': dict(act='sigmoid', sample='bernoulli', outputs=('mean', 'state')),
    'SIG_BERN_STATE': dict(act='sigmoid', sample='bernoulli', outputs=('state',)),
    'SIG_MEAN': dict(act='sigmoid', outputs=('mean',)),
    'RAW_F32': dict(act='linear', outputs=('f32',), bias=False),
    'GENERIC-gauss-sigma': dict(act='linear', sample='gaussian', outputs=('mean', 'state'), sigma=True, noise_sigma=True),
    'GENERIC-softplus': dict(act='softplus', outputs=('mean', 'f32')),
    'GENERIC-sigmoid-f32': dict(act='sigmoid', sample='bernoulli', outputs=('state', 'f32')),
    'GENERIC-linear-bf16': dict(act='linear', outputs=('mean',)),
}


def run_mode(name, e, i, **over):
    spec = dict(MODE_SPECS[name])
    A, B, a_t, b_t, acc_scale, bias = edge_operands(e, i)
    N = e['N']
    rng = np.random.RandomState(7 + i)
    kw = dict(act=spec['act'], sample=spec.get('sample'), acc_scale=acc_scale, bias_scale=1.0 if i % 2 else 0.5,
              bias=bias if spec.get('bias', True) else None, seed=0xC0FFEE + i, site=P.SITE_H if i % 2 else P.SITE_V,
              t=e['t'], tick=e['tick'], tick_off=e['tick_off'], row0=e['row0'], force_bn=e['bn'] or 0,
              force_cluster=e['cluster'])
    if spec.get('sigma'):
        kw['sigma'] = bf16_values(rng.uniform(0.5, 1.5, N))
    if spec.get('noise_sigma'):
        kw['noise_sigma'] = bf16_values(rng.uniform(0.25, 2.0, N))
    kw.update(over)
    f32_ld = (N + 7) // 8 * 8 + 1 + i % 2            # odd and even row pitches: scalar and float2 stores
    out = _native.debug_tc_op([(A, B, a_t, b_t, False)], outputs=spec['outputs'], f32_ld=f32_ld, **kw)
    return out, product(A, B, a_t, b_t), kw


@pytest.mark.parametrize('edge', range(len(EDGES)))
@pytest.mark.parametrize('mode', list(MODE_SPECS))
def test_epilogue_mode(mode, edge):
    e = EDGES[edge]
    out, C, kw = run_mode(mode, e, edge)
    assert out['plan']['mode'] == mode.split('-')[0], out['plan']
    if e['bn']:
        assert (out['plan']['bn'], out['plan']['cluster']) == (e['bn'], e['cluster'])
    check_epilogue(out, C, kw, e['M'], e['N'])


def test_many_units_per_cta():
    """M = 4096, N = 1024 at BN = 64: several units per CTA (pair), bf16 means AND states, so the staging FIFO, the
    accumulator-stage and unit-barrier parities wrap many times within each CTA.  The unit and CTA counts are asserted so
    that a later heuristic change cannot shrink the test."""
    M, N, K = 4096, 1024, 96
    rng = np.random.RandomState(4096)
    A, B = operands(rng, M, N, K, False, False, lo=-1, hi=1, density=0.55)
    bias = bf16_values(rng.uniform(-2.0, 2.0, N))
    C = product(A, B, False, False)
    for cluster, units in ((1, 32 * 16), (2, 16 * 16)):
        kw = dict(act='sigmoid', sample='bernoulli', bias=bias, seed=77, site=P.SITE_H0, t=2, tick=3, row0=1000,
                  force_bn=64, force_cluster=cluster)
        out = _native.debug_tc_op([(A, B, False, False, False)], outputs=('mean', 'state'), **kw)
        plan = out['plan']
        assert plan['mode'] == 'SIG_BERN_MEAN_STATE'
        assert (plan['bn'], plan['cluster'], plan['units']) == (64, cluster, units), plan
        assert plan['ctas'] == 132 and plan['units'] > 2 * plan['ctas'] // cluster, plan
        check_epilogue(out, C, kw, M, N)


# ---- AIS epilogues -------------------------------------------------------------------------------------------------------
def softplus(x):
    return np.logaddexp(0.0, x)


AIS_LADDER = dict(ais_a=np.float32(0.5), ais_b=np.float32(0.5 + 1.0 / 500), ais_next=np.float32(0.5 + 2.0 / 500))   # 500 steps
AIS_FAR = dict(ais_a=np.float32(0.2), ais_b=np.float32(0.3), ais_next=np.float32(0.4))


@pytest.mark.parametrize('edge', range(len(EDGES)))
@pytest.mark.parametrize('mode,temps,sample,with_logw', [
    ('AIS_UNITS', AIS_LADDER, 'bernoulli', True),
    ('AIS_UNITS_S', AIS_LADDER, 'bernoulli', False),
    ('AIS_UNITS_G', AIS_FAR, 'bernoulli', True),
    ('AIS_UNITS_G', AIS_FAR, None, True),
    ('AIS_UNITS_G', AIS_LADDER, None, True),
], ids=['series', 'states-only', 'closed-sampled', 'closed-unsampled', 'closed-unsampled-close'])
def test_ais_units(mode, temps, sample, with_logw, edge):
    """z = C + bias.  logw[m] += sum_n softplus(b z) - softplus(a z); states = sample(sigmoid(next z))."""
    e = EDGES[edge]
    M, N = e['M'], e['N']
    A, B, a_t, b_t, _, bias = edge_operands(e, edge)
    if edge % 2:
        A = A * (np.random.RandomState(edge).rand(*A.shape) < 0.5)        # K = 384: keep z within about [-8, 8]
    z = product(A, B, a_t, b_t) + np.asarray(bias, np.float64)[None, :]
    logw0 = np.random.RandomState(edge).randn(M)
    seed, site = 0xA15 + edge, P.SITE_AIS_H1
    out = _native.debug_tc_op([(A, B, a_t, b_t, False)], outputs=('state',), ais_kind=1, sample=sample, bias=bias, seed=seed,
                              site=site, t=e['t'], tick=e['tick'], tick_off=e['tick_off'], row0=e['row0'],
                              logw=logw0 if with_logw else None, force_bn=e['bn'] or 0, force_cluster=e['cluster'],
                              **{k: float(v) for k, v in temps.items()})
    assert out['plan']['mode'] == mode, out['plan']
    a, b, nxt = (float(temps[k]) for k in ('ais_a', 'ais_b', 'ais_next'))
    p = 1.0 / (1.0 + np.exp(-nxt * z))
    tol = sigmoid_tol(p, 4.0 * ULP * (np.abs(nxt * z) + 1.0))
    if sample == 'bernoulli':
        u = P.uniform_at(M, N, seed, site, e['t'], e['tick'] + e['tick_off'], e['row0']).astype(np.float64)
        check_bernoulli(out['state'][:M, :N], u, p, tol, 'unit states')
    else:
        assert_bf16_within(out['state'][:M, :N], p, tol, 'unit means')
    if with_logw:
        term = softplus(b * z) - softplus(a * z)
        inc = term.sum(axis=1)
        # per term: the series form's truncation (AIS_MAX_CT / AIS_MAX_CD: < 3e-6 relative) or the closed form's
        # intrinsics; then fp32 sums of up to 64 columns per thread and tile
        rel = (4e-6 if mode == 'AIS_UNITS' else 2.0 ** -18) + 70 * ULP
        tolw = rel * np.abs(term).sum(axis=1) + 1e-9
        got = out['logw'][:M] - logw0
        assert_f32_within(got[:, None], inc[:, None], tolw[:, None], 'logw increment')
    assert_guards(out, M, N)


@pytest.mark.parametrize('edge', range(len(EDGES)))
def test_ais_state(edge):
    """a sampled sigmoid op that also adds ais_lin * sum_n s_n * bias_scale * bias_n * (-log2 e) to logw[m]"""
    e = EDGES[edge]
    M, N = e['M'], e['N']
    A, B, a_t, b_t, acc_scale, bias = edge_operands(e, edge)
    bias_scale, lin, seed, site = (1.0, 0.37, 31 + edge, P.SITE_AIS_V) if edge % 2 else (0.5, -1.25, 31 + edge, P.SITE_AIS_H2)
    logw0 = np.random.RandomState(edge).randn(M)
    out = _native.debug_tc_op([(A, B, a_t, b_t, False)], outputs=('state',), ais_kind=2, act='sigmoid', sample='bernoulli',
                              acc_scale=acc_scale, bias_scale=bias_scale, bias=bias, ais_lin=lin, seed=seed, site=site,
                              t=e['t'], tick=e['tick'], tick_off=e['tick_off'], row0=e['row0'], logw=logw0,
                              force_bn=e['bn'] or 0, force_cluster=e['cluster'])
    assert out['plan']['mode'] == 'AIS_STATE', out['plan']
    C = product(A, B, a_t, b_t)
    a_ = acc_scale * C
    b_ = bias_scale * np.asarray(bias, np.float64)
    p = 1.0 / (1.0 + np.exp(-(a_ + b_[None, :])))
    tol = sigmoid_tol(p, 4.0 * ULP * (np.abs(a_) + np.abs(b_)[None, :]))
    u = P.uniform_at(M, N, seed, site, e['t'], e['tick'] + e['tick_off'], e['row0']).astype(np.float64)
    check_bernoulli(out['state'][:M, :N], u, p, tol, 'AIS states')
    s = bf16_bits_to_f64(out['state'][:M, :N])
    w = b_ * -LOG2E
    inc = lin * (s * w[None, :]).sum(axis=1)
    tolw = (70 * ULP + 4 * ULP) * abs(lin) * np.abs(w).sum() + 1e-9
    assert_f32_within((out['logw'][:M] - logw0)[:, None], inc[:, None], np.full((M, 1), tolw), 'logw increment')
    assert_guards(out, M, N)


# ---- refusals ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('what,kw,b_t', [
    ('bf16 output at a width that is not whole 64-column granules', dict(outputs=('mean',), act='sigmoid', force_bn=48), False),
    ('MN-major B at a width that is not whole 64-column boxes', dict(outputs=('f32',), force_bn=80), True),
    ('split-K with a bf16 output', dict(outputs=('mean', 'f32'), splits=2), False),
])
def test_refused_ops_launch_nothing(what, kw, b_t):
    rng = np.random.RandomState(0)
    A, B = operands(rng, 130, 200, 256, False, b_t)
    ctx = _native.Context.default()
    n0 = ctx.launch_count()
    with pytest.raises(RuntimeError, match='libbm'):
        _native.debug_tc_op([(A, B, False, b_t, False)], **kw)
    assert ctx.launch_count() == n0, what


# ---- 4. schedule invariance ----------------------------------------------------------------------------------------------
def schedules(bf16_out, b_t):
    widths = (64, 128, 192, 256) if (bf16_out or b_t) else tuple(range(16, 257, 16))
    return [(0, 0)] + [(bn, cl) for cl in (1, 2) for bn in widths]


def assert_same_outputs(ref, out, what):
    for k in ('mean', 'state', 'f32'):
        if k in ref:
            assert_equal(out[k].view(np.uint32 if k == 'f32' else np.uint16), ref[k].view(np.uint32 if k == 'f32' else np.uint16),
                         '{0}: {1}'.format(what, k))


INVARIANT = ['SIG_BERN_MEAN_STATE', 'SIG_BERN_STATE', 'SIG_MEAN', 'RAW_F32', 'GENERIC-gauss-sigma', 'GENERIC-softplus',
             'GENERIC-sigmoid-f32', 'GENERIC-linear-bf16', 'AIS_UNITS_S', 'AIS_STATE']


@pytest.mark.parametrize('mode', INVARIANT)
def test_schedule_invariance(mode):
    """Every output bit is the same for every allowed (tile width, row grouping) and for the heuristic's choice: the unit
    -> CTA assignment must not change any result (ops without atomics or split-K)."""
    e = dict(EDGES[3])
    M, N = e['M'], e['N']
    A, B, a_t, b_t, acc_scale, bias = edge_operands(e, 2)       # K-major A / B: every width is allowed for fp32 outputs
    if mode.startswith('AIS'):
        spec_out = ('state',)
        kw = dict(ais_kind=1, sample='bernoulli', bias=bias, **{k: float(v) for k, v in AIS_LADDER.items()}) \
            if mode == 'AIS_UNITS_S' else dict(ais_kind=2, act='sigmoid', sample='bernoulli', bias=bias, ais_lin=0.5)
    else:
        spec = MODE_SPECS[mode]
        spec_out = spec['outputs']
        kw = dict(act=spec['act'], sample=spec.get('sample'), acc_scale=acc_scale, bias=bias if spec.get('bias', True) else None)
        if spec.get('sigma'):
            kw['sigma'] = bf16_values(np.linspace(0.5, 1.5, N))
        if spec.get('noise_sigma'):
            kw['noise_sigma'] = bf16_values(np.linspace(2.0, 0.25, N))
    kw.update(seed=5, site=3, t=4, tick=6, row0=1000)
    bf16_out = 'mean' in spec_out or 'state' in spec_out
    ref = None
    for bn, cl in schedules(bf16_out, b_t):
        out = _native.debug_tc_op([(A, B, a_t, b_t, False)], outputs=spec_out, force_bn=bn, force_cluster=cl, **kw)
        assert out['plan']['mode'] == mode.split('-')[0], out['plan']
        if ref is None:
            ref = out
        else:
            assert_same_outputs(ref, out, 'BN {0}, row grouping {1}'.format(bn, cl))


@pytest.mark.skipif(HOSTSIM, reason='benchmark-size op: minutes on the interpreter')
def test_schedule_invariance_many_units():
    M, N, K = 4096, 1024, 96
    rng = np.random.RandomState(11)
    A, B = operands(rng, M, N, K, False, False, lo=-1, hi=1, density=0.55)
    bias = bf16_values(rng.uniform(-2.0, 2.0, N))
    ref = None
    for bn, cl in schedules(True, False):
        out = _native.debug_tc_op([(A, B, False, False, False)], outputs=('mean', 'state'), act='sigmoid', sample='bernoulli',
                                  bias=bias, seed=9, site=1, t=0, tick=1, force_bn=bn, force_cluster=cl)
        if ref is None:
            ref = out
        else:
            assert_same_outputs(ref, out, 'BN {0}, row grouping {1}'.format(bn, cl))


def test_schedule_invariance_random_normal_operands():
    """Random-normal bf16 operands (inexact products and sums): the per-element accumulation order does not depend on the
    tile width or the row grouping, so the raw accumulators are bit-identical across schedules."""
    M, N, K = 300, 321, 840
    rng = np.random.RandomState(12)
    A, B = rng.randn(M, K), rng.randn(N, K)
    ref = None
    for bn, cl in schedules(False, False):
        out = _native.debug_tc_op([(A, B, False, False, False)], force_bn=bn, force_cluster=cl)
        if ref is None:
            ref = out
        else:
            assert_same_outputs(ref, out, 'BN {0}, row grouping {1}'.format(bn, cl))


def test_report():
    """(runs last in this file) the tie and deviation counts of the cases above"""
    print('\n[tc-exact] Bernoulli draws checked: {0}, disagreements at rounding ties: {1}; max |Gaussian state - bf16(ref)|: '
          '{2:.3g}'.format(REPORT['bernoulli_checked'], REPORT['bernoulli_ties'], REPORT['gauss_max_dev']))
