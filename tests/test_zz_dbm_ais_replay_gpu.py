"""The AIS ladder of the DBM engines (DbmTC::ais_local in csrc/bm_dbm_tc.cuh, Dbm<T>::ais_local / ais_slice in csrc/bm_dbm.cu)
run by run against a float64 statement of the ladder, at the benchmark's size.

The ladder, from the definition (oracle/dbm.py:_ais; dbm.py:650-736).  Temperatures beta_1 = delta = dtype(1 / n_betas),
beta_{i+1} = dtype(beta_i + delta) while beta_i < dtype(1) - delta + dtype(1e-5), in the model's storage dtype; n of them.
Run r (global index first_run + r) starts at x_0 = [u < 1/2] (SITE_AIS_INIT, tick 0) and makes n transitions; transition i =
1..n at beta_i is k sweeps  v = [u < s(beta z_v(x))], h2 = [u < s(beta z_h2(x))], x' = [u < s(beta (v W_0 + h2 W_1^T + c_1))]
with z_v(x) = x W_0^T + b, z_h2(x) = x W_1 + c_2, at SITE_AIS_V / _H2 / _H1, t = 0, tick = (i - 1) k + sweep, row first_run + r.
The state x_i it leaves is weighed with  log p*_b(x_i) - log p*_a(x_i),  a = beta_{i-1} (beta_0 = 0), b = beta_i, and b = 1.0
exactly for the last one, where  log p*_beta(x) = beta x.c_1 + sum softplus(beta z_v) + sum softplus(beta z_h2).  log Z_0 =
(V + H_1 + H_2) float32(log 2).

Why a run can be compared on its own.  With every layer sampled, each GEMM operand of the ladder is exact (binary states, the
weights as the engine's GEMMs read them: bf16(W) on the tensor cores, W otherwise), the draws are u < p at the addresses
above, and the runs are independent.  A float64 chain with the same uniforms is the engine's chain unless some u lies within
the engine's rounding distance of its p, and the log-weight is then a float64 sum.

Bounds (per run, summed over the ladder; `Engine` below holds the constants).
  z        a pre-activation is a sum of K exact products: off by at most K u sum|a b| in any order (u = 2^-23 for the
           truncating tensor-core accumulator, 2^-24 fp32, 2^-53 float64), and by nothing where the weights lie on a grid
           2^-q so coarse that every partial sum is exact in fp32 (`sums_exact`); then one rounding for the bias.  The weight
           term moves by at most (b - a)(1 + |z| / 4) per unit of z's error.
  units    tensor cores: the closed form log1p(sigmoid(a z) expm1((b - a) z)) from ex2.approx / rcp.approx and short series,
           2^-18 of the term; where |b - a| <= 2.5e-3 and |next - (a + b) / 2| <= 4e-3 the series form t sigmoid(m z) may run
           instead (bm_tc.cu: AIS_MAX_CT / AIS_MAX_CD), whose truncations are |t|^3 max|sigmoid''| / 24 (midpoint rule, t =
           (b - a) z) and |t| d^4 max|sigmoid''''| / 24 (third-order series in d = (next - m) z); fp32 partial sums of at most
           64 columns per thread and tile and a 4-lane shuffle, 70 u of sum|term|; fp64 red.add across tiles.  fp32 / float64
           engines: softplus in double, 2^-45 of the two sums.
  linear   tensor cores: sum s c_1 beta (-log2 e) in fp32 times fl32((b - a) / (beta -log2 e)): 74 u of (b - a) sum s |c_1|;
           elsewhere a dot product of H_1 terms in the storage dtype or better.
  draws    |p_engine - p| <= p (1 - p) e_pre + 2^-21 p (tests/test_tc_kernel_exact_gpu.py::sigmoid_tol), e_pre the
           pre-activation's error times beta plus four roundings.

A run whose engine value is outside its bound must be explained by flipped draws inside their own tolerance: the float64 chain
is forked at the run's closest draws (smallest |u - p| first, at most 8, only those within tolerance; a fork that is still
off may be forked again behind its flip, MAX_FLIPS deep) and one fork must match.  Otherwise the failure names the run and
its closest draws (transition, sweep, site, unit).

With the benchmark's own weights (N(0, 0.02^2), not on a grid) the z term dominates: about 0.2 nats over 1000 temperatures,
honest but wide.  So the same calls are also made with weights on the grid 2^-8 (`dyadic`, same scale), where z is exact and
the bound is the arithmetic alone, about 1e-3 nats; the ladder's bookkeeping does not depend on the weights.

Not replayed here: models with a mean-valued layer (DbmTC::ais_local_passes; unsampled v / h2).  Their chains carry bf16
means whose roundings perturb every long run; they stay on the comparison with the bf16 emulation (test_zz_dbm_tc_gpu.py).
Ladders sharded over several GPUs.

The checker is a plain function of (model, call, the engine's values): tests/test_dbm_ais_replay_host.py feeds it the numpy
oracles and mutations of them.  The benchmark-size cases are skipped on the host simulation."""
import time

import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P
from test_tc_kernel_exact_gpu import HOSTSIM, bf16r

pytestmark = pytest.mark.gpu
big = pytest.mark.skipif(HOSTSIM, reason='benchmark-size replay: hours on the interpreter')

PROGRAM_OPS = 90                 # TC_PROGRAM_OPS: the ladder's 3 k n + 2 ops go in launches of 90
CHUNK = 32768                    # runs per ais_local call (Dbm::ais_slice)
AIS_MAX_CT, AIS_MAX_CD = np.float32(2.5e-3), np.float32(4.0e-3)
MAX_FORKS, MAX_FLIPS = 8, 3
MAX_FORKED = 0.25                # share of the replayed runs that may need a flipped draw
REPORT = dict(runs=0, temperatures=0, draws=0, forked=0, flips=0, worst=0.0, worst_at='', t0=time.time())

_BENCH = []


def _bench():
    """a private copy of bench.py, kept out of sys.modules (its module constants read the environment at import)"""
    if not _BENCH:
        import importlib.util
        import os
        path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'bench.py')
        spec = importlib.util.spec_from_file_location('_bench_for_ais_replay', path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _BENCH.append(mod)
    return _BENCH[0]


# ---- engines ---------------------------------------------------------------------------------------------------------------
class Engine(object):
    """what the replay has to know about an engine's arithmetic"""

    def __init__(self, name, u, sig, weights, beta, fused, prod=2.0 ** -53):
        self.name, self.u, self.sig, self.weights, self.beta, self.fused, self.prod = name, u, sig, weights, beta, fused, prod


ENGINES = {
    'bf16': Engine('bf16', 2.0 ** -23, 2.0 ** -21, bf16r, np.float32, True),
    'fp32': Engine('fp32', 2.0 ** -24, 2.0 ** -21, lambda w: np.asarray(w, np.float32).astype(np.float64), np.float32, False),
    'float64': Engine('float64', 2.0 ** -53, 2.0 ** -50, lambda w: np.asarray(w, np.float64), np.float64, False),
}
ULP = 2.0 ** -24


def sums_exact(W, K):
    """every partial sum of K products of a 0 / 1 state and an element of W is exact in fp32: W on a grid 2^-q, K max|W| 2^q < 2^24"""
    for q in range(0, 16):
        s = np.asarray(W, np.float64) * 2.0 ** q
        if np.all(s == np.rint(s)):
            return K * float(np.abs(s).max()) < 2.0 ** 24
    return False


_DEV = []


def _device():
    if not _DEV:
        dev = None
        if not HOSTSIM:
            try:
                import torch
                dev = torch.device('cuda') if torch.cuda.is_available() else None
            except ImportError:
                pass
        _DEV.append(dev)
    return _DEV[0]


class Operand(object):
    """a float64 matrix the chain multiplies states with: on the GPU through torch (DGEMM, K 2^-53) when there is one and the
    batch is worth the copies, numpy otherwise"""

    def __init__(self, B):
        self.B = np.ascontiguousarray(B, np.float64)
        self.dev = None

    def rmul(self, A):
        if A.shape[0] < 32 or _device() is None:
            return A @ self.B
        import torch
        if self.dev is None:
            self.dev = torch.from_numpy(self.B).to(_device())
        return (torch.from_numpy(np.ascontiguousarray(A, np.float64)).to(_device()) @ self.dev).cpu().numpy()


class Model(object):
    """a 2-layer binary DBM as one engine's ladder reads it"""

    def __init__(self, params, compute='bf16', dtype='float32'):
        self.engine = e = ENGINES['float64' if np.dtype(dtype) == np.float64 else compute]
        st = np.dtype(dtype)
        W0, W1 = e.weights(np.asarray(params['W'], st)), e.weights(np.asarray(params['W_1'], st))
        self.V, self.H0, self.H1 = W0.shape[0], W0.shape[1], W1.shape[1]
        self.b = np.asarray(params['vb'], st).astype(np.float64)
        self.c1 = np.asarray(params['hb'], st).astype(np.float64)
        self.c2 = np.asarray(params['hb_1'], st).astype(np.float64)
        self.exact = e.name != 'float64' and sums_exact(W0, self.V + self.H1) and sums_exact(W1, self.V + self.H1)
        self.W0, self.W0T, self.W1, self.W1T = Operand(W0), Operand(W0.T), Operand(W1), Operand(W1.T)
        if not self.exact:
            self.A0, self.A0T, self.A1, self.A1T = (Operand(np.abs(o.B)) for o in (self.W0, self.W0T, self.W1, self.W1T))

    def pre(self, x):
        """(z, its error bound) of the two unit layers: z_v = x W_0^T + b, z_h2 = x W_1 + c_2"""
        u, K = self.engine.u, self.H0
        out = []
        for op, ab, bias in ((self.W0T, None if self.exact else self.A0T, self.b), (self.W1, None if self.exact else self.A1, self.c2)):
            acc = op.rmul(x)
            e = u * (np.abs(acc) + np.abs(bias)[None, :]) * (bias != 0)[None, :]
            if not self.exact:
                e = e + K * u * ab.rmul(x)
            out.append((acc + bias[None, :], e))
        return out

    def hidden(self, v, h2, beta):
        """(beta (v W_0 + h2 W_1^T + c_1), its error bound)"""
        u, K = self.engine.u, self.V + self.H1
        acc = self.W0.rmul(v) + self.W1T.rmul(h2)
        e = 4.0 * u * beta * (np.abs(acc) + np.abs(self.c1)[None, :])
        if not self.exact:
            e = e + beta * K * u * (self.A0.rmul(v) + self.A1T.rmul(h2))
        return beta * (acc + self.c1[None, :]), e


def temperatures(n_betas, dt):
    """beta_1..beta_n of the transitions, the recurrence in the storage dtype"""
    dt = np.dtype(dt).type
    delta = dt(1.0 / n_betas)
    t = [delta]
    while t[-1] < dt(1.0) - delta + dt(1e-5):
        t.append(dt(t[-1] + delta))
    return t


def increments(t):
    """(a_i, b_i) of the state each transition leaves"""
    zero, one = type(t[0])(0.0), type(t[0])(1.0)
    return [(zero if i == 0 else t[i - 1], one if i == len(t) - 1 else t[i]) for i in range(len(t))]


def series_form(a, b, nxt):
    """whether the tensor-core units op of this increment may take the series form (bm_tc.cu::epilogue_mode, in fp32)"""
    a, b, nxt = np.float32(a), np.float32(b), np.float32(nxt)
    return bool(abs(b - a) <= AIS_MAX_CT and abs(nxt - np.float32(0.5) * (a + b)) <= AIS_MAX_CD)


def sigmoid(z):
    with np.errstate(over='ignore'):
        return 1.0 / (1.0 + np.exp(-z))


def softplus(z):
    return np.logaddexp(0.0, z)


SITE_NAMES = {P.SITE_AIS_V: 'v', P.SITE_AIS_H2: 'h2', P.SITE_AIS_H1: 'h1'}


class Chains(object):
    """what a replayed batch of runs returns: per row the log Z estimate, its bound, and the draws within their tolerance
    [(|u - p|, tolerance, (transition, sweep, site, unit))] sorted by |u - p|"""

    def __init__(self, R):
        self.logw, self.bound, self.near, self.draws = np.zeros(R), np.zeros(R), [[] for _ in range(R)], 0


def chain(m, n_betas, k, seed, first, n, forks=None):
    """float64 ladder of runs [first, first + n); with `forks` (a list of flip tuples, each flip the address (transition, sweep,
    site, unit) of a draw to invert) instead len(forks) copies of run `first`, one per tuple"""
    e = m.engine
    t = temperatures(n_betas, e.beta)
    inc = increments(t)
    R = n if forks is None else len(forks)
    rows = n if forks is None else 1
    flips = {}
    for f, fl in enumerate(forks or ()):
        for (it, s, site, unit) in fl:
            flips.setdefault((it, s, site), []).append((f, unit))
    after = [max(fl) if fl else None for fl in (forks or [()] * R)]
    out = Chains(R)

    def draw(p, tol, site, it, s):
        u = P.uniform_at(rows, p.shape[1], seed, site, 0, it * k + s, first).astype(np.float64)
        st = (u < p)
        for f, unit in flips.get((it, s, site), ()):
            st[f, unit] = ~st[f, unit]
        gap = np.abs(u - p)
        rr, cc = np.nonzero(gap <= tol)
        for r, c in zip(rr, cc):
            addr = (it, s, site, int(c))
            if after[r] is None or addr > after[r]:
                out.near[r].append((float(gap[r, c]), float(tol[r, c]), addr))
        out.draws += p.size
        return st.astype(np.float64)

    def tol_of(p, e_pre):
        return p * (1.0 - p) * e_pre + e.sig * p

    u0 = P.uniform_at(rows, m.H0, seed, P.SITE_AIS_INIT, 0, 0, first)
    x = np.broadcast_to((u0 < np.float32(0.5)).astype(np.float64), (R, m.H0)).copy()
    z = m.pre(x)
    for it, beta in enumerate(t):
        beta = float(beta)
        for s in range(k):
            units = []
            for (zz, ez), site in zip(z, (P.SITE_AIS_V, P.SITE_AIS_H2)):
                p = sigmoid(beta * zz)
                units.append(draw(p, tol_of(p, beta * ez + 4.0 * ULP * np.abs(beta * zz)), site, it, s))
            zx, ex = m.hidden(units[0], units[1], beta)
            p = sigmoid(zx)
            x = draw(p, tol_of(p, ex), P.SITE_AIS_H1, it, s)
            z = m.pre(x)
        a, b = float(inc[it][0]), float(inc[it][1])
        lin = np.abs(x * m.c1[None, :]).sum(axis=1)
        out.logw += (b - a) * (x @ m.c1)
        out.bound += (74.0 if e.fused else m.H0) * e.u * (b - a) * lin
        close = e.fused and it + 1 < len(t) and series_form(a, b, t[it + 1])
        for zz, ez in z:
            sb, sa = softplus(b * zz), softplus(a * zz)
            term = sb - sa
            out.logw += term.sum(axis=1)
            out.bound += ((b - a) * (1.0 + 0.25 * np.abs(zz)) * ez).sum(axis=1)
            if e.fused:
                out.bound += (2.0 ** -18 + 70.0 * e.u) * np.abs(term).sum(axis=1)
                if close:
                    tt = np.abs((b - a) * zz)
                    d = np.abs((float(t[it + 1]) - 0.5 * (a + b)) * zz)
                    out.bound += (tt ** 3 * (0.09623 / 24.0) + tt * d ** 4 * (0.125 / 24.0)).sum(axis=1)
            else:
                out.bound += 2.0 ** -45 * (sb + sa).sum(axis=1) + e.prod * (np.abs(b * zz) + np.abs(a * zz)).sum(axis=1)
    logZ0 = (m.V + m.H0 + m.H1) * float(np.float32(np.log(2.0)))
    out.logw += logZ0
    out.bound += 2.0 ** -50 * (np.abs(out.logw) + logZ0) + 1e-12
    for r in range(R):
        out.near[r].sort()
    out.temperatures = len(t)
    return out


def describe(near):
    return ', '.join('transition {0} sweep {1} {2}[{3}] |u - p| {4:.3g} (tol {5:.3g})'.format(
        a[0] + 1, a[1], SITE_NAMES[a[2]], a[3], g, tl) for g, tl, a in near[:MAX_FORKS]) or 'none'


def explain(m, n_betas, k, seed, run, got, near, flips=()):
    """the flips (a tuple of draw addresses) under which the float64 chain of `run` gives `got`, or None"""
    width = MAX_FORKS if not flips else MAX_FORKS // 2
    cands = [flips + (addr,) for _, _, addr in near[:width]]
    if not cands:
        return None
    res = chain(m, n_betas, k, seed, run, 1, forks=cands)
    for f, fl in enumerate(cands):
        if abs(res.logw[f] - got) <= res.bound[f]:
            return fl, abs(res.logw[f] - got) / res.bound[f]
    if len(flips) + 1 < MAX_FLIPS:
        for f, fl in enumerate(cands):
            hit = explain(m, n_betas, k, seed, run, got, res.near[f], fl)
            if hit:
                return hit
    return None


def check_runs(m, n_betas, k, seed, first, got, what, case=None):
    """got[r]: the engine's log Z estimate of run first + r.  Returns the number of runs that needed flipped draws."""
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), '{0}: non-finite estimate'.format(what)
    ref = chain(m, n_betas, k, seed, first, len(got))
    ratio = np.abs(got - ref.logw) / ref.bound
    forked = 0
    for r in np.nonzero(ratio > 1.0)[0]:
        hit = explain(m, n_betas, k, seed, first + int(r), got[r], ref.near[r])
        if hit is None:
            raise AssertionError('{0}: run {1}: engine {2!r}, float64 {3!r}, |difference| {4:.3g} > bound {5:.3g}, and no fork at '
                                 'its closest draws ({6}) reproduces it'.format(what, first + int(r), got[r], ref.logw[r],
                                                                                abs(got[r] - ref.logw[r]), ref.bound[r],
                                                                                describe(ref.near[r])))
        forked += 1
        REPORT['flips'] += len(hit[0])
        ratio[r] = hit[1]
    if case is not None:
        case.bound = max(case.bound, float(ref.bound.max()))
    REPORT['runs'] += len(got)
    REPORT['temperatures'] += len(got) * ref.temperatures
    REPORT['draws'] += ref.draws
    REPORT['forked'] += forked
    if ratio.max() > REPORT['worst']:
        REPORT['worst'], REPORT['worst_at'] = float(ratio.max()), '{0}, run {1}, bound {2:.3g}'.format(
            what, first + int(ratio.argmax()), ref.bound[ratio.argmax()])
    return forked


# ---- models and engine calls ---------------------------------------------------------------------------------------------------
def dyadic(w, q=8):
    """w on the grid 2^-q: exact partial sums in fp32, exact in bf16 while |w| 2^q < 256"""
    return (np.rint(np.asarray(w, np.float64) * 2.0 ** q) / 2.0 ** q).astype(np.float32)


def dbm_cfg(V, Hs, compute='bf16', dtype='float32'):
    return dict(compute=compute, n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * 2,
                h_n_samples=[100.] * 2, dtype=dtype, n_particles=4, batch_size=4, max_mf_updates=6, mf_tol=1e-6, l2=1e-4,
                max_norm=6.0, sample_v=True, sample_h=[True, True], sparsity_target=[0.2, 0.1], sparsity_cost=[1e-4, 5e-5],
                sparsity_damping=0.9)


def params(V, Hs, scale, bias=0.0, seed=2, grid=8):
    """W ~ N(0, scale^2) (on the grid 2^-grid unless grid is None) and biases ~ N(0, bias^2), not bf16 values"""
    d = _bench().dbm_params(dict(n_visible=V, n_hiddens=list(Hs)), seed=seed, scale=scale)
    rng = np.random.RandomState(seed + 1)
    for name in ('vb', 'hb', 'hb_1'):
        d[name] = (bias * rng.randn(d[name].size)).astype(np.float32)
    if grid is not None:
        d['W'], d['W_1'] = dyadic(d['W'], grid), dyadic(d['W_1'], grid)
    return d


class Case(object):
    """an engine with its parameters set, and the replay's model of it"""

    def __init__(self, cfg, prm):
        self.cfg = cfg
        self.eng = _native.CudaDBM(cfg)
        st = np.dtype(cfg['dtype'])
        self.eng.set_params({k_: np.asarray(v, st) for k_, v in prm.items()})
        self.m = Model(prm, cfg['compute'], cfg['dtype'])
        self.bound = 0.0                 # the largest bound of a replayed run

    def close(self):
        self.eng.close()

    def check(self, n_runs, n_betas, k, seed, slices, what, first_run=None):
        """one engine call; the runs of `slices` [(lo, hi)] (indices into the call) replayed.  Returns the call's values."""
        got = self.eng.ais(n_runs, n_betas, k, seed, first_run=first_run)
        assert got.shape == (n_runs,)
        for lo, hi in slices:
            check_runs(self.m, n_betas, k, seed, (first_run or 0) + lo, got[lo:hi],
                       '{0}: ais({1}, {2}, {3}) runs {4}..{5}'.format(what, n_runs, n_betas, k, lo, hi), self)
        return got


BENCH_SHAPE = (784, (512, 1024))


@pytest.fixture(scope='module')
def cfg4():
    """the benchmark's model on the grid 2^-8 (the tight bound), zero biases as bench.py sets them"""
    c = Case(_bench().dbm_cfg(), params(*BENCH_SHAPE, scale=0.02))
    assert c.m.exact
    yield c
    c.close()


@big
def test_benchmark_call_with_the_benchmarks_weights():
    """ais(20000, 1000, 1, 2222) on bench.dbm_params(scale=0.02): exactly what `bench.py --config cfg4-ais` times.  The weights
    are not on a grid, so the bound carries the accumulators' worst case (see the docstring)."""
    b = _bench()
    cfg = b.dbm_cfg()
    c = Case(cfg, b.dbm_params(cfg, scale=0.02))
    try:
        assert not c.m.exact
        c.check(20000, 1000, 1, 2222, [(0, 16), (19984, 20000)], 'cfg4-ais')
    finally:
        c.close()


@big
def test_benchmark_call_and_its_slices(cfg4):
    """the same call on grid weights: the first runs, runs straddling a 256-run block in the middle (9984 = 39 x 256), the last
    runs; then ais_rows(300, .., first_run=19700) (one full 256-block and a ragged 44: its first runs and those around its block
    edge replayed) must be the same runs of the full call.  Not bit for bit: the tile width of an op
    is picked from the number of runs, so the fp32 partial sums of a row regroup between a 20000-run and a 300-run call (7.7e-8
    measured); each call is within the runs' bound of the same float64 value, so the two are within twice the bound (a wrong
    first_run is off by nats)"""
    full = cfg4.check(20000, 1000, 1, 2222, [(0, 32), (9968, 10000), (19968, 20000)], 'cfg4-ais grid')
    part = cfg4.check(300, 1000, 1, 2222, [(0, 16), (240, 300)], 'cfg4-ais grid slice', first_run=19700)
    assert np.abs(part - full[19700:20000]).max() <= 2.0 * cfg4.bound, np.abs(part - full[19700:20000]).max()


@big
@pytest.mark.parametrize('n_betas', [1000, 400])
def test_biased_model_with_wide_preactivations(n_betas):
    """W ~ 0.1 and N(0, 1) biases that are not bf16 values: |z| reaches 20-30, every bias path and the linear term carry weight
    (the benchmark's biases are zero)"""
    c = Case(_bench().dbm_cfg(), params(*BENCH_SHAPE, scale=0.1, bias=1.0, grid=6))
    try:
        assert c.m.exact and np.any(bf16r(c.m.c1) != c.m.c1)
        c.check(64, n_betas, 1, 77, [(0, 64)], 'biased')
    finally:
        c.close()


def modes_of(n_betas):
    """the number of increments of a k = 1 ladder that take the series form, by the rule of bm_tc.cu::epilogue_mode"""
    t = temperatures(n_betas, np.float32)
    inc = increments(t)
    return sum(series_form(inc[i][0], inc[i][1], t[i + 1]) for i in range(len(t) - 1)), len(t) - 1


@big
@pytest.mark.parametrize('n_betas', [2, 3, 30, 31, 32, 399, 400, 401])
def test_ladder_lengths(cfg4, n_betas):
    """one launch exactly full (30 temperatures: 3 x 30 ops + the 2 of the last increment spill into a second), around it, and
    around the switch between the closed and the series form of the increment at 400 temperatures"""
    cfg4.check(32, n_betas, 1, 31 + n_betas, [(0, 32)], 'ladder length')


@pytest.mark.parametrize('n_betas,series', [(399, 'none'), (400, 'some'), (401, 'all')])
def test_form_of_the_increment_around_400_temperatures(n_betas, series):
    """Which form an op takes is observable through debug_tc_op's plan for the op's own (a, b, next): the rule restated in
    `series_form` is the kernel's at the ladder's first, a middle and the last fused increment.  At 400 temperatures
    |b - a| sits on AIS_MAX_CT and float32 round-off of the accumulated beta decides, op by op."""
    n_series, n_ops = modes_of(n_betas)
    assert {'none': n_series == 0, 'some': 0 < n_series < n_ops, 'all': n_series == n_ops}[series], (n_series, n_ops)
    t = temperatures(n_betas, np.float32)
    inc = increments(t)
    rng = np.random.RandomState(0)
    A, B = rng.randint(-2, 3, (8, 16)).astype(np.float32), rng.randint(-2, 3, (8, 16)).astype(np.float32)
    seen = set()
    for i in list(range(0, len(t) - 1, max(1, len(t) // 40))) + [len(t) - 2]:
        a, b, nxt = float(inc[i][0]), float(inc[i][1]), float(t[i + 1])
        out = _native.debug_tc_op([(A, B, False, False, False)], outputs=('state',), ais_kind=1, sample='bernoulli',
                                  bias=np.zeros(8, np.float32), logw=np.zeros(8), ais_a=a, ais_b=b, ais_next=nxt)
        want = 'AIS_UNITS' if series_form(a, b, nxt) else 'AIS_UNITS_G'
        assert out['plan']['mode'] == want, (i, a, b, nxt, out['plan'])
        seen.add(want)
    if series == 'some':
        assert seen == {'AIS_UNITS', 'AIS_UNITS_G'}, seen


@big
@pytest.mark.parametrize('k,n_betas', [(2, 64), (4, 64), (7, 64), (30, 3)])
def test_gibbs_steps(cfg4, k, n_betas):
    """k sweeps per temperature: 3 k does not divide 90 for k = 4, 7 (a launch boundary inside a temperature), and k = 30 is
    one temperature per launch.  Only sweep 0 weighs, ticks run (i - 1) k + sweep."""
    assert (PROGRAM_OPS % (3 * k) != 0) == (k in (4, 7))
    cfg4.check(32, n_betas, k, 5 + k, [(0, 32)], 'Gibbs steps')


@pytest.mark.parametrize('shape', [(781, (130, 70)), (7, (5, 4))], ids=['781-130-70', '7-5-4'])
@pytest.mark.parametrize('k', [1, 3])
def test_ragged_shapes(shape, k):
    if HOSTSIM and shape[0] > 7:
        pytest.skip('benchmark-size replay: hours on the interpreter')
    c = Case(dbm_cfg(*shape), params(*shape, scale=0.25, bias=0.5, grid=5))
    n_betas = 24 if HOSTSIM else 240 if shape[0] == 7 else 120
    try:
        assert c.m.exact
        for R in ((1, 33) if HOSTSIM else (1, 33, 257)):
            c.check(R, n_betas, k, 100 + R, [(0, R)], 'ragged')
        c.check(33, n_betas, k, 9, [(0, 33)], 'ragged rows', first_run=1000)
    finally:
        c.close()


@big
def test_chunking():
    """more runs than one ais_local call takes: the runs around the chunk boundary replayed, and the call equal to two
    ais_rows calls cut there"""
    shape = (64, (32, 16))
    c = Case(dbm_cfg(*shape), params(*shape, scale=0.25, bias=0.5, grid=5))
    try:
        full = c.check(CHUNK + 64, 4, 1, 12, [(CHUNK - 68, CHUNK + 64)], 'chunking')
        two = np.concatenate([c.eng.ais(CHUNK, 4, 1, 12, first_run=0), c.eng.ais(64, 4, 1, 12, first_run=CHUNK)])
        np.testing.assert_array_equal(full, two)
    finally:
        c.close()


@big
def test_fp32_engine():
    """compute='fp32': fp32 GEMMs on unrounded weights (on the grid, so exact), the weights from float64 softplus sums"""
    c = Case(_bench().dbm_cfg('fp32'), params(*BENCH_SHAPE, scale=0.02, bias=0.3, grid=12))
    try:
        assert c.m.exact and c.m.engine.name == 'fp32' and np.any(bf16r(c.m.W0.B) != c.m.W0.B)
        c.check(32, 1000, 1, 8, [(0, 32)], 'fp32 engine')
    finally:
        c.close()


@big
def test_float64_model():
    """a float64 model: the beta recurrence in float64, everything to about 1e-9 with no flipped draw"""
    shape = (781, (130, 70))
    c = Case(dbm_cfg(*shape, compute='fp32', dtype='float64'), params(*shape, scale=0.1, bias=0.5, grid=None))
    try:
        before = REPORT['forked']
        c.check(64, 240, 1, 5, [(0, 64)], 'float64 model')
        assert REPORT['forked'] == before
    finally:
        c.close()


def test_report():
    """(runs last in this file) what the replays above checked"""
    name, power = 'no CUDA device', ''
    if _device() is not None:
        import subprocess
        import torch
        name = torch.cuda.get_device_name(0)
        try:
            power = ', power limit ' + subprocess.check_output(
                ['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], timeout=20).decode().strip()
        except (OSError, subprocess.SubprocessError):
            power = ', power limit not read'
    print('\n[dbm-ais-replay] runs replayed: {0}, temperatures: {1}, draws: {2}; runs that needed flipped draws: {3} ({4} flips); '
          'largest |difference| / bound: {5:.3g} ({6}); {7:.0f} s on {8}{9}'.format(
              REPORT['runs'], REPORT['temperatures'], REPORT['draws'], REPORT['forked'], REPORT['flips'], REPORT['worst'],
              REPORT['worst_at'], time.time() - REPORT['t0'], name, power))
    assert REPORT['runs'] > 0
    assert REPORT['forked'] <= MAX_FORKED * REPORT['runs'], REPORT
