"""The RBM engines' training and validation metrics -- L2 loss, MSRE, free energy and PLL -- at the benchmark's own sizes, against
a float64 statement of each metric as the engine defines it (csrc/bm_rbm.h run_metrics / free_energy / finish_metrics).

Definitions (the same in every compute mode; DESIGN §1 row a13 and §6).  Parameters are the ones the step starts from.

  l2_loss      l2/2 sum W^2 of the fp32 (storage-precision) W.
  msre         mean (X - v_means)^2 over the chain's own input and visible means, as the engine exports them (get_activation):
               the bf16 engine's bf16 operand and bf16 means, the storage-precision engine's prepared batch and means.
  free_energy  batch mean of FE(x) = -x.vb - sum_j softplus(x W + hb)_j (Gaussian visibles: 1/2 |x - vb/sigma|^2 instead of
               -x.vb), with the fp32 W and the UNROUNDED prepared batch (x / sigma for Gaussian visibles) -- also on the bf16 engine,
               whose chain reads bf16 operands.  Multinomial hidden units: -x.vb - (x W).h_hat with h_hat drawn from the uniform
               multinomial at SITE_MULTINOMIAL_FE, fe_idx 2, plus -lgamma(M + H) + lgamma(M + 1) + lgamma(H).
  pll          i_r = site_words(rows, 1, seed, SITE_PLL, 0, tick, row0)[r] % V (row0 = rank * rows: never the dataset row of a
               resident batch), X~ = X with x[r, i_r] -> 1 - x[r, i_r], d = mean FE(X~) - mean FE(X), pll = V log sigmoid(d);
               multinomial hidden units draw h_hat with fe_idx 0 for X~ and 1 for X.  FE(X~) is FE(X) with a rank-1 change per
               row: X~ W = X W + (x~ - x)[r] W[i_r, :].

The float64 products run on the GPU through torch when it has one (tests/test_zz_dbm_tc_replay_gpu.py: mm).

Error bound of the engine's value (u = 2^-24 for float32 models in both compute modes, 2^-53 for float64 ones):

  GEMM         x W is an FMA chain over K = V terms (layer_op_kernel): |acc - sum_i x_i W_ij| <= K 2u sum_i |x_i W_ij| (one
               rounding per add, at most 2u of a partial sum bounded by sum_i |x_i W_ij|, with a factor 2 for the order).  When
               x, W and hb lie on dyadic grids and every partial sum fits the significand (24 bits), the GEMM and the bias add
               are exact and this term is 0 (`exact`).
  bias add     u |x W + hb| (0 when exact).
  softplus     fmaxf(z, 0) + log1pf(expf(-|z|)): expf is within 2 ulp and log1pf within 1 ulp (CUDA C++ Programming Guide,
               single-precision mathematical functions, full-range, no fast math).  An expf error of 2 ulp moves log1p(e) by at
               most e 2^-22 / (1 + e) <= 2^-23, log1pf adds 2^-23 ln 2 and the final add u softplus(z): <= 4u + u softplus(z) per
               element, plus sigmoid(z) times the error of z.
  row sums     rowdot / fe_visible sum in double and cast the row to T: u |row| each; the products x vb in T: u |x vb| each;
               Gaussian visibles: d = x - vb/sigma and d*d in T: 2u |d| (|vb/sigma| + |d|) per element.
  mean         mean_combine sums in double: 2^-50 |mean|.

  FE bound     mean over rows of the row bounds e_r.
  PLL bound    |d_engine - d| <= D = mean_r (e_r(X~) + e_r(X)), where a row with W[i_r, :] == 0 has bit-identical hidden terms for
               X~ and X (fma(x, 0, acc) == acc), so only its visible terms count; then |pll - pll_engine| <= V sigmoid(-(d - D)) D.
  MSRE bound   bf16 engine: the differences of two bf16 values and their squares in fp32, 8 FMAs per partial: 16u of the
               value; then (n + 2) 2^-53 of it for the double sum of n terms (the only term of the storage-precision engines,
               whose differences are exact in double).
  L2 bound     (n + 2) 2^-53 of the value (double sum of n squares).

A worst-case fp32 bound is loose for PLL: at cfg2 K 2u sum |xW| summed over 1024 softplus terms is ~1e-2 per row, ~15 nats of PLL
once multiplied by V.  So two kinds of cases:

  exactness probes  fp32 arithmetic exact or nearly so, bounds ~1e-6 relative, where a definitional slip shows by a wide margin:
                    `w0` (W = 0, spread dyadic vb: PLL is the index stream alone, a wrong site / tick / row0 / modulus moves it by
                    tens of nats), `dyadic` (few-bit W, biases: exact GEMMs), `bf16w` (10-bit W that bf16 always rounds up: FE
                    on the bf16 shadow misses by nats per row), `gauss-x` (11-bit Gaussian inputs that bf16 always rounds away
                    from zero: FE on the rounded input misses by ~5 per row).
  realistic models  bench-like random W on the benchmark's data generators, held to the worst-case bound above.

Entry points: metrics() on a validation set (taller than one batch in the ragged case), train_step(metrics=...) with the chain's
own X / v_means, train_step_at on a resident dataset at first_row != 0, and train_epoch with float32, byte and bf16 feeds, a
ragged last batch, every = 2 and iter0 = 0 / 1, each reported batch bit-identical to a train_step loop whose values are checked.
The benchmark-size cases are skipped on the host simulation; the small ones run there."""
import threading

import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P
from oracle.rbm import bf16_round, multinomial_counts
from test_tc_kernel_exact_gpu import HOSTSIM
from test_zz_dbm_tc_replay_gpu import mm

pytestmark = pytest.mark.gpu
big = pytest.mark.skipif(HOSTSIM, reason='benchmark-size metrics: hours on the interpreter')

NAMES = ('l2_loss', 'msre', 'free_energy', 'pll')
REPORT = dict(checked=0, worst={n: (0.0, 0.0) for n in NAMES}, pll_nats=0.0)


def _bench():
    import bench
    return bench


# ---- float64 statement ------------------------------------------------------------------------------------------------------
def softplus(z):
    return np.maximum(z, 0.0) + np.log1p(np.exp(-np.abs(z)))


def sigmoid(z):
    return 0.5 * (1.0 + np.tanh(0.5 * z))


def grid(a):
    """the smallest q <= 40 with a * 2^q all integers, or None"""
    a = np.asarray(a, np.float64)
    for q in range(41):
        s = a * 2.0 ** q
        if np.array_equal(s, np.round(s)):
            return q
    return None


class Statement(object):
    """float64 metrics of the engine's definition at one parameter state, each with the bound of the engine's value"""

    def __init__(self, cfg, params):
        self.V, self.H = int(cfg['n_visible']), int(cfg['n_hidden'])
        self.f64 = np.dtype(cfg.get('dtype', 'float32')) == np.float64
        self.T = np.float64 if self.f64 else np.float32
        self.bf16 = cfg.get('compute', 'bf16') == 'bf16'        # (float64 engines run with compute='fp32')
        self.u = 2.0 ** -53 if self.f64 else 2.0 ** -24
        self.W = np.asarray(params['W'], self.T).astype(np.float64)
        self.vb = np.asarray(params['vb'], self.T).astype(np.float64)
        self.hb = np.asarray(params['hb'], self.T).astype(np.float64)
        self.absW = np.abs(self.W)
        self.gauss = cfg.get('v_kind', 'bernoulli') == 'gaussian'
        self.multi = cfg.get('h_kind', 'bernoulli') == 'multinomial'
        self.M = float(cfg.get('h_n_samples', 100))
        sig = cfg.get('sigma', None) if self.gauss else None
        self.sigma = np.ones(self.V) if sig is None else \
            np.broadcast_to(np.asarray(sig, np.float64).astype(self.T), (self.V,)).astype(np.float64)
        self.l2 = float(cfg.get('l2', 0.))
        self.qW, self.qb = grid(self.W), grid(self.hb)

    def hhat(self, seed, tick, fe_idx):
        probs = np.full((1, self.H), 1.0 / self.H, dtype=np.float32)
        return multinomial_counts(probs, int(self.M), seed, P.SITE_MULTINOMIAL_FE, fe_idx, tick)[0]

    def exact(self, X, absA):
        """every partial sum of X W (and + hb) is exact in the engine's arithmetic"""
        qx = grid(X)
        if qx is None or self.qW is None or (not self.multi and (self.qb is None or self.qb > qx + self.qW)):
            return False
        top = float(absA.max()) + (0.0 if self.multi else float(np.abs(self.hb).max()))
        return top * 2.0 ** (qx + self.qW) < 2.0 ** (53 if self.f64 else 24)

    def visible(self, X):
        u = self.u
        if self.gauss:
            c = self.vb / self.sigma
            d = X - c[None, :]
            vis = 0.5 * np.square(d).sum(axis=1)
            e = 2.0 * u * (np.abs(d) * (np.abs(c)[None, :] + np.abs(d))).sum(axis=1)
        else:
            vis = -(X @ self.vb)
            e = u * (np.abs(X) @ np.abs(self.vb))
        return vis, e + u * np.abs(vis)

    def rows(self, X, A, absA, exact, hhat):
        """per row: FE, its bound, and the bound of the visible part alone"""
        u = self.u
        gemm = 0.0 if exact else self.V * 2.0 * u * absA
        if self.multi:
            t = A @ hhat
            hid = -t
            eh = (gemm @ hhat if not exact else 0.0) + u * np.abs(t)
        else:
            z = A + self.hb[None, :]
            sp = softplus(z)
            ez = gemm + (0.0 if exact else u * np.abs(z))
            s = sp.sum(axis=1)
            hid = -s
            eh = (sigmoid(z) * ez + 4.0 * u + u * sp).sum(axis=1) + u * s
        vis, ev = self.visible(X)
        return vis + hid, ev + eh, ev

    def metrics(self, names, X_fp, seed, tick, row0=0, X_in=None, v_means=None):
        """{name: (value, bound)}.  X_fp: the prepared batch the free energies read; X_in / v_means: the exported chain input and
        visible means (msre)."""
        out = {}
        X = np.asarray(X_fp, self.T).astype(np.float64)
        if 'l2_loss' in names:
            v = self.l2 * 0.5 * float(np.square(self.W).sum())
            out['l2_loss'] = (v, (self.W.size + 2) * 2.0 ** -53 * v)
        if 'msre' in names:
            d = np.asarray(X_in, np.float64) - np.asarray(v_means, np.float64)
            v = float(np.mean(np.square(d)))
            out['msre'] = (v, ((16.0 * 2.0 ** -24 if self.bf16 else 0.0) + (d.size + 2) * 2.0 ** -53) * v)
        if 'free_energy' not in names and 'pll' not in names:
            return out
        A, absA = mm(X, self.W), mm(np.abs(X), self.absW)
        ex = self.exact(X, absA)
        const = 0.0
        if self.multi:
            from math import lgamma
            const = -lgamma(self.M + self.H) + lgamma(self.M + 1.0) + lgamma(float(self.H))
        if 'free_energy' in names:
            fe, e, _ = self.rows(X, A, absA, ex, self.hhat(seed, tick, 2) if self.multi else None)
            m = float(fe.mean())
            out['free_energy'] = (m + const, float(e.mean()) + 2.0 ** -50 * (abs(m) + abs(const)))
        if 'pll' in names:
            rows = X.shape[0]
            r = np.arange(rows)
            idx = (P.site_words(rows, 1, seed, P.SITE_PLL, 0, tick, row0)[:, 0] % np.uint32(self.V)).astype(np.int64)
            x = X[r, idx]
            xt = (self.T(1) - x.astype(self.T)).astype(np.float64)       # T(1) - x, in the engine's type
            Xt = X.copy()
            Xt[r, idx] = xt
            At = A + (xt - x)[:, None] * self.W[idx]
            absAt = absA + (np.abs(xt) - np.abs(x))[:, None] * self.absW[idx]
            ft, et, evt = self.rows(Xt, At, absAt, self.exact(Xt, absAt), self.hhat(seed, tick, 0) if self.multi else None)
            fx, e1, evx = self.rows(X, A, absA, ex, self.hhat(seed, tick, 1) if self.multi else None)
            same = np.zeros(rows, bool) if self.multi else ~self.W[idx].any(axis=1)
            D = float(np.where(same, evt + evx, et + e1).mean()) + 2.0 ** -50 * (abs(ft.mean()) + abs(fx.mean()))
            d = float(ft.mean() - fx.mean())
            out['pll'] = (-self.V * float(softplus(-d)), self.V * float(sigmoid(-(d - D))) * D + 1e-12 * self.V)
        return out


def check_metrics(got, ref, what):
    for n, v in got.items():
        val, bound = ref[n]
        err = abs(float(v) - val)
        REPORT['checked'] += 1
        we, wb = REPORT['worst'][n]
        if err * wb >= we * bound:              # the largest err / bound so far
            REPORT['worst'][n] = (err, bound)
        if n == 'pll':
            REPORT['pll_nats'] = max(REPORT['pll_nats'], err)
        assert err <= bound, '{0}: {1} = {2!r}, float64 statement {3!r}: |difference| {4:.3g} > bound {5:.3g}'.format(
            what, n, float(v), val, err, bound)


def check_input(st, X_in, X_fp, what):
    """the chain's exported input is the prepared batch, rounded to bf16 on the bf16 engine"""
    want = np.asarray(X_fp, st.T)
    if st.bf16:
        want = bf16_round(want)
    np.testing.assert_array_equal(np.asarray(X_in, st.T), want, err_msg=what + ': exported X')


def check_engine_metrics(eng, cfg, params, X, k, seed, tick, what):
    """metrics() of a batch (validation path, row0 = 0)"""
    got = eng.metrics(X, k, seed, tick, NAMES)
    st = Statement(cfg, params)
    Xp = prepared(cfg, X)
    Xi, vm = eng.get_activation('X', X.shape[0]), eng.get_activation('v_means', X.shape[0])
    check_input(st, Xi, Xp, what)
    check_metrics(got, st.metrics(NAMES, Xp, seed, tick, 0, Xi, vm), what + ': metrics()')
    return got


def check_step_metrics(got, eng, cfg, before, Xp, seed, tick, what):
    """metrics a training step returned: pre-update parameters, the step's own exported X / v_means, row0 = 0 (one rank)"""
    st = Statement(cfg, before)
    rows = Xp.shape[0]
    Xi, vm = eng.get_activation('X', rows), eng.get_activation('v_means', rows)
    check_input(st, Xi, Xp, what)
    check_metrics(got, st.metrics(NAMES, Xp, seed, tick, 0, Xi, vm), what)


def check_epoch(reports, loop, rep, what):
    """an epoch's reports are the train_step loop's values of the reporting batches `rep`, bit for bit"""
    for n in NAMES:
        want = [loop[i][n] for i in rep]
        assert reports[n] == want, '{0}: {1} reports {2} differ from the train_step loop {3} (batches {4})'.format(
            what, n, reports[n], want, rep)


def prepared(cfg, X):
    """the prepared batch the engine's free energies read: x / sigma in the model's type (no dropout in these cases)"""
    T = np.dtype(cfg.get('dtype', 'float32')).type
    X = np.asarray(X, T)
    if cfg.get('v_kind') == 'gaussian':
        X = X / np.broadcast_to(np.asarray(cfg['sigma'], np.float64).astype(T), (X.shape[1],))[None, :]
    return X


# ---- cases ----------------------------------------------------------------------------------------------------------------
# name: (v_kind, h_kind, V, H, batch rows, max_batch, validation rows, k)
SHAPES = {
    'cfg2': ('bernoulli', 'bernoulli', 784, 1024, 4096, 4096, 4096, 5),
    'cfg3': ('gaussian', 'bernoulli', 3072, 5000, 2048, 2048, 2048, 1),
    'cfg5': ('bernoulli', 'bernoulli', 784, 4096, 4096, 4096, 4096, 25),
    'multinomial': ('bernoulli', 'multinomial', 784, 1024, 4096, 4096, 4096, 2),
    'ragged': ('bernoulli', 'bernoulli', 781, 1001, 1500, 1000, 2500, 3),
    'small': ('bernoulli', 'bernoulli', 130, 70, 65, 65, 65, 2),
    'small-ragged': ('bernoulli', 'bernoulli', 37, 21, 40, 16, 50, 2),
    'small-gauss': ('gaussian', 'bernoulli', 130, 70, 65, 65, 65, 2),
    'small-multi': ('bernoulli', 'multinomial', 130, 70, 65, 65, 65, 2),
}


def model_cfg(shape, compute, dtype='float32'):
    vk, hk, V, H, _, mb, _, _ = SHAPES[shape]
    cfg = dict(n_visible=V, n_hidden=H, v_kind=vk, h_kind=hk, dtype=dtype, compute=compute, l2=1e-5, max_batch=mb,
               sample_v=False, sample_h=True, sparsity_target=0.1, sparsity_cost=0.0, sparsity_damping=0.9, h_n_samples=100)
    if vk == 'gaussian':            # (small-gauss: sigma in {0.5, 1, 2}, so that x / sigma keeps the probes' inputs exact)
        cfg['sigma'] = np.ones(V) if shape != 'small-gauss' else np.array([0.5, 1.0, 2.0])[np.arange(V) % 3]
    return cfg


def probe_params(probe, V, H, seed, gauss=False):
    """every variable a step reads (so set_params restores the whole state)"""
    rng = np.random.RandomState(seed)
    f = np.float32
    if probe == 'bench':
        p = dict(W=((0.01 if gauss else 0.05) * rng.randn(V, H)).astype(f), vb=((0.05 if gauss else 0.1) * rng.randn(V)).astype(f),
                 hb=(0.1 * rng.randn(H)).astype(f))
    elif probe == 'w0':              # PLL = the index stream: d = mean_r -(x~ - x) vb[i_r], vb >= 0 keeps d < 0 where PLL ~ V d
        p = dict(W=np.zeros((V, H), f), vb=(rng.randint(0, 64, V) / 8.).astype(f), hb=(rng.randint(-16, 17, H) / 8.).astype(f))
    elif probe == 'dyadic':          # 4-bit W: every partial sum of x W exact in fp32
        p = dict(W=(rng.randint(-8, 9, (V, H)) / 64.).astype(f), vb=(rng.randint(-16, 17, V) / 16.).astype(f),
                 hb=(rng.randint(-32, 33, H) / 16.).astype(f))
    elif probe == 'bf16w':           # 10 significant bits ending in 11: bf16 rounds every weight up by 2^-13
        p = dict(W=((512 + 4 * rng.randint(0, 128, (V, H)) + 3) * 2.0 ** -13).astype(f), vb=(rng.randint(-16, 17, V) / 16.).astype(f),
                 hb=(np.round(-0.1 * V) / 8. + rng.randint(-16, 17, H) / 8.).astype(f))     # x W ~ 0.0125 V
    elif probe == 'gauss-x':         # W = 0: the visible term sees the input rounding alone
        p = dict(W=np.zeros((V, H), f), vb=(rng.randint(-4, 5, V) / 8.).astype(f), hb=(rng.randint(-16, 17, H) / 8.).astype(f))
    else:
        raise ValueError(probe)
    p.update(dW=np.zeros((V, H), f), dvb=np.zeros(V, f), dhb=np.zeros(H, f), q_means=np.full(H, 0.1, f))
    return p


def probe_data(probe, shape, rows, seed):
    vk, _, V = SHAPES[shape][:3]
    if probe == 'gauss-x':           # +-(1024 + 8j + 7) 2^-10: 11 bits, bf16 keeps 8 and rounds away from zero
        rng = np.random.RandomState(seed)
        m = 1024 + 8 * rng.randint(0, 128, (rows, V)) + 7
        return (np.where(rng.rand(rows, V) < 0.5, -1.0, 1.0) * m * 2.0 ** -10).astype(np.float32)
    if vk == 'gaussian':
        return _bench().synth_cifar(rows, n_vis=V, seed=seed)
    return _bench().synth_mnist(rows, seed=seed, n_vis=V)


def run_case(shape, probe, compute, dtype='float32', seed=0x3E7, tick=5, lr=0.05, mom=0.5, make=None):
    """metrics(), train_step(metrics=...) and train_step_at(first_row = 37) of one model, each against the float64 statement.
    make(cfg): the engine (a CudaRBM by default)"""
    vk, _, V, H, B, _, NV, k = SHAPES[shape]
    cfg = model_cfg(shape, compute, dtype)
    init = probe_params(probe, V, H, 11, vk == 'gaussian')
    what = '{0}/{1}/{2}'.format(shape, probe, compute if dtype == 'float32' else dtype)
    eng = (make or _native.CudaRBM)(cfg)
    try:
        eng.set_params(init)
        Xv = probe_data(probe, shape, NV, 5)
        check_engine_metrics(eng, cfg, init, Xv, k, seed, tick, what)
        X = probe_data(probe, shape, B, 6)
        eng.set_params(init)
        got = eng.train_step(X, lr, mom, k, seed, tick + 1, metrics=NAMES)
        check_step_metrics(got, eng, cfg, init, prepared(cfg, X), seed, tick + 1, what + ': train_step')
        assert not np.array_equal(eng.get_params(['W'])['W'], init['W']) or probe in ('w0', 'gauss-x'), what + ': no update'
        first = 37
        Xall = probe_data(probe, shape, first + B + 11, 7)
        eng.set_params(init)
        eng.set_data(Xall)
        got = eng.train_step_at(first, B, lr, mom, k, seed, tick + 2, metrics=NAMES)
        check_step_metrics(got, eng, cfg, init, prepared(cfg, Xall[first:first + B]), seed, tick + 2, what + ': train_step_at')
    finally:
        eng.close()


CASES = [('cfg2', p) for p in ('bench', 'w0', 'dyadic', 'bf16w')] + [('cfg3', 'bench'), ('cfg3', 'gauss-x'), ('cfg5', 'bench')] + \
        [('multinomial', 'bench'), ('multinomial', 'dyadic'), ('ragged', 'bench'), ('ragged', 'w0')]
SMALL = [('small', 'bench'), ('small', 'w0'), ('small', 'dyadic'), ('small', 'bf16w'), ('small-ragged', 'bench'), ('small-ragged', 'w0'),
         ('small-gauss', 'bench'), ('small-gauss', 'gauss-x'), ('small-multi', 'dyadic')]


@big
@pytest.mark.parametrize('compute', ['bf16', 'fp32'])
@pytest.mark.parametrize('shape,probe', CASES)
def test_metrics_at_benchmark_sizes(shape, probe, compute):
    run_case(shape, probe, compute)


@big
def test_metrics_float64_ragged():
    run_case('ragged', 'bench', 'fp32', dtype='float64')
    run_case('ragged', 'w0', 'fp32', dtype='float64')


@pytest.mark.parametrize('compute', ['bf16', 'fp32'])
@pytest.mark.parametrize('shape,probe', SMALL)
def test_metrics_small(shape, probe, compute):
    """130-70 at batch 65 (Bernoulli, Gaussian with sigma in {0.5, 1, 2}, multinomial hidden units), and a 37-21 model whose
    batches (40 rows) and validation set (50 rows) exceed max_batch (16); these also run on the host simulation"""
    run_case(shape, probe, compute)


# ---- train_epoch ------------------------------------------------------------------------------------------------------------
def epoch_feeds(eng, compute, nrows, V):
    """(label, what train_epoch gets, the float32 rows a train_step loop gets)"""
    Xb = _bench().synth_mnist(nrows, seed=31, n_vis=V)
    rng = np.random.RandomState(32)
    Xr = np.clip(Xb * 0.7 + 0.3 * rng.rand(nrows, V), 0.0, 1.0).astype(np.float32)      # real-valued: not bf16 values
    if eng is None:
        return [('float32', Xr, Xr)]
    feeds = [('float32', Xr, Xr), ('u8', eng.pin(Xb), Xb)]
    assert feeds[1][1].dtype == np.uint8
    if compute == 'bf16':
        P16 = _native.as_bf16(Xr)
        feeds.append(('bf16', P16, P16.widen()))
    return feeds


def run_epoch(shape, compute, dtype='float32', make=None):
    """3 full batches and a ragged last one; every = 2 with iter0 = 1 reports batches 0 and 2, iter0 = 0 batches 1 and 3 (the second
    half of the epoch double buffer, and the ragged batch).  Each feed's reports must be the values of a train_step loop over
    the same rows, which are checked against the float64 statement step by step (pre-update parameters of each step)."""
    _, _, V, H, B, _, _, k = SHAPES[shape]
    cfg = model_cfg(shape, compute, dtype)
    init = probe_params('bench', V, H, 12)
    nrows, seed, tick0, lr, mom = 3 * B + (1000 if B > 1000 else B // 3), 0xE9, 40, 0.05, 0.5
    nb = 4
    eng = (make or _native.CudaRBM)(cfg)
    pinned = []
    try:
        if make is None:
            feeds = epoch_feeds(eng, compute, nrows, V)
        else:
            Xr = epoch_feeds(None, None, nrows, V)[0][1]
            feeds = [(dtype, Xr, Xr)]
        for label, feed, Xloop in feeds:
            if getattr(feed, 'dtype', None) == np.uint8:
                pinned.append(feed)
            what = '{0}/{1}/{2} feed'.format(shape, compute, label)
            eng.set_params(init)
            loop = []
            for i in range(nb):
                before = eng.get_params()
                Xi = np.ascontiguousarray(Xloop[i * B:(i + 1) * B])
                got = eng.train_step(Xi, lr, mom, k, seed, tick0 + i, metrics=NAMES)
                check_step_metrics(got, eng, cfg, before, prepared(cfg, Xi), seed, tick0 + i, '{0}: step {1}'.format(what, i))
                loop.append(got)
            after_loop = eng.get_params(['W'])['W']
            for iter0 in (1, 0):
                eng.set_params(init)
                rep = eng.train_epoch(feed, B, lr, mom, k, seed, tick0, metrics=NAMES, every=2, iter0=iter0)
                check_epoch(rep, loop, [i for i in range(nb) if (iter0 + i + 1) % 2 == 0], '{0}, iter0 {1}'.format(what, iter0))
                np.testing.assert_array_equal(eng.get_params(['W'])['W'], after_loop, err_msg=what + ': W after the epoch')
    finally:
        for p in pinned:
            eng.unpin(p)
        eng.close()


@big
@pytest.mark.parametrize('compute', ['bf16', 'fp32'])
def test_epoch_reports_are_the_checked_step_loop(compute):
    """cfg2: float32 (real-valued), byte and (bf16 engine) bfloat16 feeds; 3 batches of 4096 rows and one of 1000"""
    run_epoch('cfg2', compute)


# ---- two contexts on one device ------------------------------------------------------------------------------------------------
@big
def test_two_contexts_on_one_device_from_two_threads():
    """The MSRE / L2 reductions' partial sums belong to the context: two contexts of one device, two threads, each computing
    the metrics of its own model once, get what each got alone.  (One run may not make the two streams' reductions overlap; it
    checks that they do not interfere when they do.)"""
    lib = _native.load_library()
    ctxs = [_native.Context(0), _native.Context(0)]
    engines = []
    try:
        for j, c in enumerate(ctxs):
            cfg = model_cfg('cfg2', 'fp32')
            e = _native.CudaRBM(cfg, ctx=c)
            e.set_params(probe_params('bench', 784, 1024, 20 + j))
            engines.append(e)
        Xs = [_bench().synth_mnist(4096, seed=40 + j) for j in range(2)]
        names = ('l2_loss', 'msre')
        alone = [e.metrics(X, 1, 9, 3, names) for e, X in zip(engines, Xs)]
        together = [None, None]

        def run(j):
            together[j] = engines[j].metrics(Xs[j], 1, 9, 3, names)
        threads = [threading.Thread(target=run, args=(j,)) for j in range(2)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert together == alone
        assert alone[0] != alone[1]
    finally:
        for e in engines:
            e.close()
        for c in ctxs:
            lib.bm_ctx_destroy(c.handle)


def test_report():
    """(runs last in this file) what the cases above checked"""
    w = REPORT['worst']
    print('\n[rbm-metrics] metrics checked: {0}; largest |engine - float64| against its bound (at the largest ratio): {1}; '
          'largest PLL difference {2:.3g} nats'.format(
              REPORT['checked'], ', '.join('{0} {1:.3g} / {2:.3g}'.format(n, w[n][0], w[n][1]) for n in NAMES), REPORT['pll_nats']))
