"""What a user reads from a DBM -- transform, reconstruct, the two-layer bound log_proba, sample_v and the validation MSRE --
stated in float64 as the engines define them (csrc/bm_dbm_tc.cuh DbmTC, csrc/bm_dbm.cu DbmImpl), with the bound of each engine's
value derived from its own arithmetic.  Plain functions of exported arrays (no GPU call): tests/test_zz_dbm_query_gpu.py feeds
them the engines, tests/test_dbm_query_replay_host.py the bf16 emulation (oracle/dbm_bf16.py) and mutations of it.

Three arithmetics (`prec`):
  bf16     the tensor-core engine: GEMM operands are exact bf16 values (binary X and states, bf16 means, bf16(W)), so every
           product is exact in fp32 and an accumulator of K products is off by at most K 2^-23 sum |a b| (ACC); means are stored
           as bf16 (check_bf16: the rounding of a value within the bound, at most one bf16 ulp from bf16(ref)).
  fp32     the CUDA-core engine of a float32 model: fp32 FMA chains on the fp32 W (K 2^-24 sum |a b|, bounded by ACC), fp32
           means (|got - ref| <= bound + 2^-24 |ref|).
  float64  the CUDA-core engine of a float64 model: the same with 2^-52 per add.
The sigmoid adds sigmoid_tol's term (the approximate ex2 / rcp of the tensor-core epilogue; expf's few ulp on the fp32 engine).

The queries, each from one restored state:
  E-step      with mf_tol = -1, engines built with max_mf_updates = J - 1 and J stop after exactly that many sweeps.  Sweep J of
              layer i is the float64 conditional of layer i - 1 of sweep J (X for i = 0) and layer i + 1 of sweep J - 1 (sweep 1
              reads the stale mu).  transform(X) is mu_{L-1}[:rows] bit for bit; rows >= rows of mu stay untouched; the E-step of
              reconstruct, log_proba and val_metrics leaves the same mu bit for bit.
  reconstruct act(mu_0 W_0^T + vb): sigmoid, or (mu_0 W_0^T) sigma + vb for Gaussian visibles, on the engine's own mu_0.
  log_proba   (L = 2) sum t_0.mu_0 + t_1.mu_1 + X.vb + mu_0.hb_0 + mu_1.hb_1 + H(clip(mu_0)) + H(clip(mu_1)), t_0 = X W_0, t_1 =
              mu_0 W_1 with the W the engine reads (bf16(W) on the tensor cores) and the biases as stored, H(s) = -s log s - (1 - s)
              log(1 - s).  The clip to [1e-7, 1 - 1e-7] is taken in float32 on float32 models (csrc/bm_dbm.cu
              dbm_bound_rows_kernel) and in double on float64 ones.  Bound per row: the accumulation bound of the two t GEMMs
              weighted by |mu| (sum_j K ACC (|below| |W|)_j |mu_j|), the storage rounding of t, and the double sums (2^-53 per
              add over every term).  The float32 clip moves H by ~3e-7 nats per unit at exactly 1.0, far inside that bound at
              the benchmark's shapes, so it is pinned by value only where mu is saturated (`entropy` states both clips).
              What bf16 weights cost: `bound_gap` reports (does not gate) the float64 bound with the model's own W minus the
              engine's value.
  val_metrics msre is the float64 mean of (X - recon)^2 over rows x n_visible, recon being the engine's reconstruction of the
              same mu; the kernel sums in double (sqdiff_partial_kernel: 592 x 256 strided partial sums, then a tree), so the
              bound is (rows V / (592 256) + 600) 2^-53 sum (X - recon)^2 / (rows V).  n_mf_updates is the E-step's sweep count.
              The particles it leaves are bit-identical to those of train_step from the same state and key.
  sample_v    k committed sampled sweeps (the particles val_metrics(k) leaves, bit for bit, every tempered slot and the swap
              round included), then k uncommitted sweeps of means from them at t = k + 1 .. 2k (slot 0 only): no draws, the
              hidden particles unchanged, v replaced by the final visible means.

sample_v's uncommitted sweeps run on scratch the engine does not export as variables, so it exports them through a read-only
hook (option (b): bm_dbm_debug_last_sample_v, CudaDBM.debug_last_sample_v, the pattern of bm_crbm_debug_last_step): the last
sweep k and the sweep before it, copied from the ping-pong buffers they ran on, with no launch.  Each exported sweep is then
checked on its own, like a mean-field sweep: every layer against the float64 conditional of the exported values it read (sweep
1 reads the committed particles), with the one-op bound above, and sample_v's result must be the last sweep's visible means bit
for bit.  So the cases use k <= 2, where every sweep is exported.  A bound carried through the chain instead (option (a)) was
measured too wide at the benchmark's shapes: at cfg4 the worst-case accumulation bound of a hidden mean, pushed through |W| for
two sweeps, admits ~0.05 on visible means near 0.5 (~0.1 without rounding the intermediates to bf16), while a second sweep
skipped or fed the committed particles moves them by ~5e-3.

The float64 products run on the GPU through torch when it has one, in numpy otherwise (test_zz_dbm_tc_replay_gpu.mm)."""
import numpy as np

from dbm_ais_depth_oracle import bound_given_mu
from test_tc_kernel_exact_gpu import ULP, bf16r, sigmoid_tol
from test_zz_dbm_tc_replay_gpu import f64, mm, sfx
from test_zz_rbm_tc_chain_gpu import ACC, MAX_OFF, check_bf16

DACC = 2.0 ** -52                # one float64 add
D_ULP = 2.0 ** -53
SQ_PARTIALS = 592 * 256          # strided partial sums of sqdiff_partial_kernel (csrc/bm_simt.cu)

REPORT = dict(queries=0, means=0, off=0, worst={}, gap={})


def record(what, got, ref, tol):
    """the largest |got - ref| / bound of each query (keyed by the query: the text after the case's name)"""
    d = np.abs(f64(got) - f64(ref))
    r = float(np.max(d / np.maximum(f64(tol), 1e-300))) if d.size else 0.0
    kind = what.split(': ')[-1].split(',')[0].split('(')[0].strip()
    REPORT['worst'][kind] = max(REPORT['worst'].get(kind, 0.0), r)


def within(got, ref, tol, what):
    g, ref, tol = f64(got), f64(ref), np.broadcast_to(f64(tol), np.shape(ref))
    bad = ~(np.abs(g - ref) <= tol)
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError('{0}: {1} of {2} elements off by more than the bound, first at {3}: got {4!r}, ref {5!r}, '
                             'bound {6:.3g}'.format(what, int(bad.sum()), bad.size, at, g[at], ref[at], tol[at]))


class Model(object):
    """float64 conditionals of one parameter state as an engine of arithmetic `prec` reads it, each with the bound of the
    engine's value; inputs may carry bounds of their own (propagated through |W|)"""

    def __init__(self, cfg, params, prec):
        assert prec in ('bf16', 'fp32', 'float64')
        self.prec = prec
        self.L = len(cfg['n_hiddens'])
        dt = np.float64 if prec == 'float64' else np.float32
        read = (lambda w: bf16r(np.asarray(w, np.float32))) if prec == 'bf16' else (lambda w: np.asarray(w, dt).astype(np.float64))
        self.W = [read(params['W' + sfx(i)]) for i in range(self.L)]
        self.absW = [np.abs(w) for w in self.W]
        self.hb = [np.asarray(params['hb' + sfx(i)], dt).astype(np.float64) for i in range(self.L)]
        self.vb = np.asarray(params['vb'], dt).astype(np.float64)
        self.acc, self.rnd = (DACC, D_ULP) if prec == 'float64' else (ACC, ULP)
        self.gauss = cfg.get('v_kind', 'bernoulli') == 'gaussian'
        V = self.W[0].shape[0]
        self.sigma = (np.broadcast_to(np.asarray(cfg['sigma'], dt), (V,)) if self.gauss else np.ones(V, dt)).astype(np.float64)

    def operand(self, X):
        """the batch as the GEMMs read it"""
        return bf16r(X) if self.prec == 'bf16' else f64(X)

    def _sigmoid(self, a, b, e):
        p = 1.0 / (1.0 + np.exp(-(a + b)))
        if self.prec == 'float64':
            return p, p * (1.0 - p) * e + 8.0 * D_ULP * p
        return p, sigmoid_tol(p, e)

    def hidden(self, i, below, above, e_below=None, e_above=None):
        """p(h_i | below, above) = sigmoid(below W_i + above W_{i+1}^T + hb_i) and the bound of the engine's value"""
        below = f64(below)
        a, e, K = mm(below, self.W[i]), mm(np.abs(below), self.absW[i]), below.shape[1]
        if above is not None:
            above = f64(above)
            a, e, K = a + mm(above, self.W[i + 1].T), e + mm(np.abs(above), self.absW[i + 1].T), K + above.shape[1]
        b = self.hb[i][None, :]
        e = K * self.acc * e + 4.0 * self.rnd * (np.abs(a) + np.abs(b))
        if e_below is not None:
            e = e + mm(e_below, self.absW[i]) * (1.0 + 2.0 ** -20)
        if e_above is not None:
            e = e + mm(e_above, self.absW[i + 1].T) * (1.0 + 2.0 ** -20)
        return self._sigmoid(a, b, e)

    def visible(self, h0, e_h0=None):
        """E[v | h_0]: sigmoid(h_0 W_0^T + vb), or (h_0 W_0^T) sigma + vb for Gaussian visibles, and its bound"""
        h0 = f64(h0)
        a = mm(h0, self.W[0].T) * self.sigma[None, :]
        b = self.vb[None, :]
        e = h0.shape[1] * self.acc * mm(np.abs(h0), self.absW[0].T) * self.sigma[None, :] + 4.0 * self.rnd * (np.abs(a) + np.abs(b))
        if e_h0 is not None:
            e = e + mm(e_h0, self.absW[0].T) * self.sigma[None, :] * (1.0 + 2.0 ** -20)
        if self.gauss:
            mean = a + b
            return mean, e + self.rnd * np.abs(mean)
        return self._sigmoid(a, b, e)

    def check(self, got, ref, tol, what):
        """a stored mean against its float64 value"""
        REPORT['means'] += np.size(ref)
        if self.prec == 'bf16':
            off = check_bf16(got, ref, tol, what)
            REPORT['off'] += off
            record(what, got, ref, tol + 2.0 ** -9 * np.abs(bf16r(ref)) + 2.0 ** -126)
            return
        tol = tol + self.rnd * np.abs(ref) + (2.0 ** -126 if self.prec == 'fp32' else 0.0)      # fp32: sigmoid underflows to 0
        record(what, got, ref, tol)
        within(got, ref, tol, what)


def mus(d, L):
    return [d['mu' + sfx(i)] for i in range(L)]


# ---- E-step and transform ------------------------------------------------------------------------------------------------------
def check_estep_sweep(m, X, sweep, before, stale, what):
    """sweep = every layer's mu after J sweeps, before = after J - 1 (the stale mu when J = 1), all batch_size rows"""
    rows, Xo = X.shape[0], m.operand(X)
    for i in range(m.L):
        below = Xo if i == 0 else f64(sweep[i - 1][:rows])
        above = f64(before[i + 1][:rows]) if i + 1 < m.L else None
        p, t = m.hidden(i, below, above)
        m.check(sweep[i][:rows], p, t, '{0}: E-step, mu{1}'.format(what, sfx(i)))
        np.testing.assert_array_equal(sweep[i][rows:], stale[i][rows:],
                                      err_msg='{0}: the E-step wrote rows >= {1} of mu{2}'.format(what, rows, sfx(i)))
    REPORT['queries'] += 1


def check_transform(out, mu, what):
    """transform's output is the top layer's mu, bit for bit"""
    rows = out.shape[0]
    np.testing.assert_array_equal(out, mu[-1][:rows], err_msg='{0}: transform is not mu{1}[:rows]'.format(what, sfx(len(mu) - 1)))
    REPORT['queries'] += 1


def check_same_mu(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(g, w, err_msg='{0}: mu{1} differs from the E-step of the other query'.format(what, sfx(i)))


# ---- reconstruct ---------------------------------------------------------------------------------------------------------------
def check_reconstruct(m, mu0, recon, what):
    """recon = act(mu_0 W_0^T + vb) on the engine's own mu_0 (the rows of recon)"""
    rows = recon.shape[0]
    p, t = m.visible(f64(mu0[:rows]))
    m.check(recon, p, t, what + ': reconstruct')
    REPORT['queries'] += 1


# ---- log_proba at two layers ---------------------------------------------------------------------------------------------------
def entropy(m, f32_clip):
    """H(clip(m)) per element: the clip in float32 (float32 models) or in double (float64 models)"""
    m = f64(m)
    if f32_clip:
        s = np.clip(m.astype(np.float32), np.float32(1e-7), np.float32(1. - 1e-7)).astype(np.float64)
    else:
        s = np.clip(m, 1e-7, 1. - 1e-7)
    return -s * np.log(s) - (1. - s) * np.log(1. - s)


def params_of(m, prm):
    """the model's own weights and biases (as stored) for bound_given_mu"""
    keys = ['vb'] + ['W' + sfx(i) for i in range(m.L)] + ['hb' + sfx(i) for i in range(m.L)]
    return {k: f64(prm[k]) for k in keys}


def bound_ref(m, prm, X, mu):
    """the float64 bound on the engine's means with the W the engine reads and its clip, and the per-row bound of the engine's
    value"""
    rows = X.shape[0]
    mu = [f64(x[:rows]) for x in mu]
    f32_clip = m.prec != 'float64'
    ref = bound_given_mu(params_of(m, prm), X, mu, bf16_weights=(m.prec == 'bf16'))
    ref = ref + sum((entropy(x, f32_clip) - entropy(x, False)).sum(axis=1) for x in mu)
    tol = np.zeros(rows)
    mag = mm(np.abs(f64(X)), np.abs(m.vb)[:, None])[:, 0]
    below, n = m.operand(X), f64(X).shape[1]
    for i, x in enumerate(mu):
        K = below.shape[1]
        t = mm(below, m.W[i])
        tol += (K * m.acc * mm(np.abs(below), m.absW[i]) * np.abs(x)).sum(axis=1) + (m.rnd * np.abs(t * x)).sum(axis=1)
        mag += (np.abs(t * x) + np.abs(x * m.hb[i][None, :]) + entropy(x, f32_clip)).sum(axis=1)
        n += x.shape[1]
        below = x
    tol += (n + 64) * D_ULP * mag
    return ref, tol


def check_bound(m, prm, X, mu, got, what):
    ref, tol = bound_ref(m, prm, X, mu)
    record(what + ': log_proba', got, ref, tol)
    within(got, ref, tol, what + ': log_proba')
    REPORT['queries'] += 1
    return ref


def bound_gap(m, prm, X, mu, got, what=''):
    """(per-row gap, mean gap): the engine's value minus the float64 bound with the model's own W on the same means, what bf16
    weights cost"""
    rows = X.shape[0]
    full = bound_given_mu(params_of(m, prm), X, [f64(x[:rows]) for x in mu], bf16_weights=False)
    gap = f64(got) - full
    if m.prec == 'bf16':
        REPORT['gap'][what] = (float(np.mean(gap)), float(np.max(np.abs(gap))))
    return gap, float(np.mean(gap))


# ---- val_metrics ---------------------------------------------------------------------------------------------------------------
def check_msre(X, recon, msre, what):
    d = f64(X) - f64(recon)
    n = d.size
    s = float(np.sum(d * d))
    ref = s / n
    tol = (n / SQ_PARTIALS + 600.0) * D_ULP * ref
    record(what + ': msre', np.array([msre]), np.array([ref]), np.array([max(tol, 1e-300)]))
    within(np.array([msre]), np.array([ref]), np.array([tol]), what + ': msre')
    REPORT['queries'] += 1


def particle_names(L, T=1):
    names = ['v'] + ['h' + sfx(i) for i in range(L)]
    if T > 1:
        names += ['v_pt'] + ['h_pt' + sfx(i) for i in range(L)]
    return names


def check_same_particles(got, want, L, T, what, names=None):
    for n in (names or particle_names(L, T)):
        np.testing.assert_array_equal(got[n], want[n], err_msg='{0}: particle {1} differs'.format(what, n))


# ---- sample_v --------------------------------------------------------------------------------------------------------------------
def check_mean_sweep(m, prev, cur, what):
    """one unsampled particle sweep: cur = {'v': .., 'h': .., 'h_1': ..} after it, prev before it.  Layer i is the float64
    conditional of the new layer below (prev's v for i = 0) and the old layer above; v that of the new h"""
    for i in range(m.L):
        below = f64(prev['v']) if i == 0 else f64(cur['h' + sfx(i - 1)])
        above = f64(prev['h' + sfx(i + 1)]) if i + 1 < m.L else None
        p, t = m.hidden(i, below, above)
        m.check(cur['h' + sfx(i)], p, t, '{0}, h{1}'.format(what, sfx(i)))
    p, t = m.visible(f64(cur['h']))
    m.check(cur['v'], p, t, what + ', v')


def check_sample_v(m, committed, after, out, k, T, chain, what):
    """committed: the particles val_metrics(k) left from the same state; after: every particle after sample_v(k); out: its
    return value; chain: {t: sweep t of the uncommitted half} for t = k - 1 (if >= 1) and k, as the engine exports them"""
    L = m.L
    hidden = [n for n in particle_names(L, T) if n != 'v']
    check_same_particles(after, committed, L, T, what + ': sample_v committed half', hidden)
    np.testing.assert_array_equal(after['v'], out, err_msg=what + ': sample_v returned something else than v')
    if k == 0:
        np.testing.assert_array_equal(out, committed['v'], err_msg=what + ': sample_v(0) moved v')
    else:
        assert sorted(chain) == list(range(max(k - 1, 1), k + 1)), (what, sorted(chain))
        for t in sorted(chain):
            prev = committed if t == 1 else chain.get(t - 1)
            if prev is not None:
                check_mean_sweep(m, prev, chain[t], '{0}: sample_v({1}) uncommitted sweep {2}'.format(what, k, t))
        np.testing.assert_array_equal(out, chain[k]['v'], err_msg='{0}: sample_v({1}) did not return the visible means of its '
                                                                  'last sweep'.format(what, k))
    REPORT['queries'] += 1


def check_unchanged(before, after, what):
    """every variable of `before` is in `after`, bit for bit"""
    for n, v in before.items():
        np.testing.assert_array_equal(after[n], v, err_msg='{0}: {1} moved'.format(what, n))


def report_line(tag):
    w = ', '.join('{0} {1:.3g}'.format(k, v) for k, v in sorted(REPORT['worst'].items()))
    gap = '; '.join('{0}: mean {1:.4g} nats, largest |row| {2:.4g}'.format(k, *v) for k, v in sorted(REPORT['gap'].items())) or 'n/a'
    return ('[{0}] queries checked: {1}; means checked: {2}, off bf16(ref): {3}; the bf16 engine\'s bound minus the bound on '
            'the model\'s own W: {4}; largest |difference| / bound: {5}'.format(tag, REPORT['queries'], REPORT['means'],
                                                                             REPORT['off'], gap, w))


def off_within_limit():
    return REPORT['off'] <= MAX_OFF * max(REPORT['means'], 1)
