"""Every mean-field sweep, particle sweep and M-step of the tensor-core DBM engine (csrc/bm_dbm_tc.cuh, DbmTC) at the
benchmark's own sizes, against a float64 statement of each operation.

Everything a DBM step reads or writes is a variable `CudaDBM.get_params` exports and `set_params` restores (mu*, the particles
v / h*, W*, dW*, vb, dvb, hb*, dhb*, q_means*, mu_means*), and every draw is keyed by (seed, site, t, tick, row0) with site
SITE_DBM_H + i or SITE_DBM_V and t the sweep index (oracle/philox.py), not by the number of sweeps.  So, from one restored state:

  E-step      an engine stopped after j sweeps (max_mf_updates = j, mf_tol = -1: never converged) for j = 0..J.  Sweep j of
              layer i is the float64 conditional of layer i-1 of sweep j and layer i+1 of sweep j-1 (sweep 1 reads the stale
              mu, not the approximate pass: oracle/dbm.py:184-186).  Rows >= rows of mu are never written.
  decision    the sweep outputs give the engine's convergence measures d_t = max_i max |mu_i^(t) - mu_i^(t-1)| exactly (bf16
              operands, an fp32 difference); with mf_tol = d_t the engine must stop after exactly t sweeps (diff == tol stops)
              and leave mu^(t).  The t = 0 test (stale mu against the approximate pass, which is doubled for every layer below
              the top and for layer 0, bias not doubled) is pinned with a stale mu built from the float64 approximate pass.
  particles   PCD-j for j = j0..j1: sweep j of run j against run j-1's exported particles -- h_0 | v, h_1 (u < p at
              SITE_DBM_H, t = j), each higher layer | the new layer below (and the old layer above), v | h_0 (SITE_DBM_V), a
              layer that is not sampled as bf16 means.  mu is bit-identical across the runs (the E-step does not depend on k).
  M-step      the parameters each run leaves against float64 formulas on that run's own activations (oracle/dbm.py:232-284:
              dW divided by the configured batch_size and n_particles, the bias means by the rows present, l2, the sparsity
              penalty with its "element `layer` of the sum vector" quirk, momentum, max-norm).
  next step   a second train_step without set_params, replayed from the state the first one left: the only place where a
              stale bf16 shadow of W (Wb / WbT, rebuilt by refresh_shadow after the update) would show.

Error bounds.  The GEMM operands are exact bf16 values (binary X and states, bf16 means, bf16(W)), so every product is exact in
fp32 and an accumulator of K products in any order is off by at most K 2^-23 sum |a b| (K = K_below + K_above for the two-pair
op of a hidden layer).  The epilogue adds the per-mode terms of tests/test_tc_kernel_exact_gpu.py.  The M-step's bounds start
from the same accumulation bound for the split-K gradient GEMMs and the fp32 column sums, add a few fp32 roundings of every
term of each update expression, and for W the rescale W min(n, c) / max(n, 1e-8), which moves W by up to two ulps even where
max-norm does not bind, plus the column norm's own error where it does.  dW is compared on its own scale.

The checkers are plain functions of exported arrays (no GPU call): tests/test_dbm_tc_replay_host.py feeds them the bf16
emulation (oracle/dbm_bf16.py) and mutations of it.  The float64 products run on the GPU through torch when it has one (a
DGEMM's own error, K 2^-53, is far below every bound here), in numpy otherwise.  The benchmark-size cases are skipped on the host
simulation; the 30-18-11 case runs there."""
import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P
from test_tc_kernel_exact_gpu import HOSTSIM, ULP, bf16r, check_bernoulli, gaussian_noise, sigmoid_tol
from test_zz_rbm_tc_chain_gpu import ACC, MAX_OFF, bits, check_bf16

pytestmark = pytest.mark.gpu
big = pytest.mark.skipif(HOSTSIM, reason='benchmark-size replay: hours on the interpreter')

PROGRAM_OPS = 90                 # TC_PROGRAM_OPS: committed particle sweeps run as one program while k (L + 1) fits
REPORT = dict(draws=0, ambiguous=0, max_gap=0.0, means=0, off=0, sweeps=0, decisions=0, msteps=0)


_BENCH = []


def _bench():
    """a private copy of bench.py, loaded on first use and kept out of sys.modules: its module constants read
    BM_BENCH_BATCHES at import, which a host test of bench.py sets for its own `import bench` (the host test of this file's
    checkers runs in the same session)"""
    if not _BENCH:
        import importlib.util
        import os
        path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'bench.py')
        spec = importlib.util.spec_from_file_location('_bench_for_dbm_replay', path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _BENCH.append(mod)
    return _BENCH[0]


def sfx(i):
    return '' if i == 0 else '_%d' % i


# ---- float64 products ----------------------------------------------------------------------------------------------------
_DEV = []


def mm(a, b):
    """a @ b in float64"""
    if not _DEV:
        dev = None
        if not HOSTSIM:
            try:
                import torch
                dev = torch.device('cuda') if torch.cuda.is_available() else None
            except ImportError:
                pass
        _DEV.append(dev)
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if _DEV[0] is None:
        return a @ b
    import torch
    return (torch.from_numpy(np.ascontiguousarray(a)).to(_DEV[0]) @ torch.from_numpy(np.ascontiguousarray(b)).to(_DEV[0])).cpu().numpy()


def f32(x):
    """a scalar as the engine holds it (fp32), widened"""
    return float(np.float32(x))


def rounding(n, *terms):
    """n fp32 roundings of an expression whose terms have these sizes"""
    return n * ULP * sum(np.abs(t) for t in terms)


# ---- 1. float64 conditionals -------------------------------------------------------------------------------------------------
class Conditionals(object):
    """float64 conditionals of the DBM at one parameter state, with the per-element bound of the kernel's value"""

    def __init__(self, cfg, params):
        self.L = len(cfg['n_hiddens'])
        self.Wb = [bf16r(np.asarray(params['W' + sfx(i)], np.float32)) for i in range(self.L)]
        self.absW = [np.abs(w) for w in self.Wb]
        self.hb = [np.asarray(params['hb' + sfx(i)], np.float32).astype(np.float64) for i in range(self.L)]
        self.vb = np.asarray(params['vb'], np.float32).astype(np.float64)
        self.gauss = cfg.get('v_kind', 'bernoulli') == 'gaussian'
        V = self.Wb[0].shape[0]
        sig = np.broadcast_to(np.asarray(cfg['sigma'], np.float32), (V,)) if self.gauss else np.ones(V, np.float32)
        self.sigma = sig.astype(np.float64)
        self.sample_v = bool(cfg.get('sample_v', True))
        self.sample_h = [bool(s) for s in cfg.get('sample_h', [True] * self.L)]

    def hidden(self, i, below, above, s=1.0):
        """p(h_i | below, above) = sigmoid(s (below Wb_i + above Wb_{i+1}^T) + hb_i) and its bound: one two-pair op"""
        a, e, K = mm(below, self.Wb[i]), mm(np.abs(below), self.absW[i]), below.shape[1]
        if above is not None:
            a, e, K = a + mm(above, self.Wb[i + 1].T), e + mm(np.abs(above), self.absW[i + 1].T), K + above.shape[1]
        a, b = s * a, self.hb[i][None, :]
        e = s * K * ACC * e + 4.0 * ULP * (np.abs(a) + np.abs(b))
        p = 1.0 / (1.0 + np.exp(-(a + b)))
        return p, sigmoid_tol(p, e)

    def approximate(self, X):
        """the approximate-inference pass (oracle/dbm.py:169-176): x2 for layer 0 and every layer below the top, each layer
        reading the bf16 rounding of the float64 value below (the engine reads its own bf16 slot)"""
        out, below = [], X
        for i in range(self.L):
            p, t = self.hidden(i, below, None, 2.0 if (i == 0 or i < self.L - 1) else 1.0)
            out.append((p, t))
            below = bf16r(p)
        return out

    def visible(self, h0):
        """E[v | h_0]: sigmoid(h0 Wb_0^T + vb), or (h0 Wb_0^T) sigma + vb for Gaussian visibles"""
        a = mm(h0, self.Wb[0].T) * self.sigma[None, :]
        b = self.vb[None, :]
        e = h0.shape[1] * ACC * mm(np.abs(h0), self.absW[0].T) * self.sigma[None, :] + 4.0 * ULP * (np.abs(a) + np.abs(b))
        if self.gauss:
            mean = a + b
            return mean, e + ULP * np.abs(mean)
        p = 1.0 / (1.0 + np.exp(-(a + b)))
        return p, sigmoid_tol(p, e)


def check_means(got, ref, tol, what):
    off = check_bf16(got, ref, tol, what)
    REPORT['means'] += ref.size
    REPORT['off'] += off
    return off


def check_draws(got, u, p, tol, what):
    """u < p, a disagreement only where |u - p| is within the bound of p"""
    s = np.asarray(got, np.float64)
    differ = s != (u < p)
    check_bernoulli(bits(got), u, p, tol, what)
    REPORT['draws'] += s.size
    REPORT['ambiguous'] += int(differ.sum())
    if differ.any():
        REPORT['max_gap'] = max(REPORT['max_gap'], float(np.abs(u - p)[differ].max()))


def f64(a):
    return np.asarray(a, np.float64)


# ---- 2. E-step ---------------------------------------------------------------------------------------------------------------
def check_estep(cm, X, stale, sweeps, what):
    """sweeps[j]: every layer's mu after j sweeps (all batch_size rows); sweeps[0] must be the stale mu itself.  Returns the
    convergence measures [d_1, .., d_J] of the engine's own sweeps."""
    rows, Xb = X.shape[0], bf16r(X)                 # the GEMMs read the bf16 batch
    L = cm.L
    for i in range(L):
        np.testing.assert_array_equal(sweeps[0][i], stale[i], err_msg='{0}: mu{1} after 0 sweeps'.format(what, sfx(i)))
    diffs = []
    for j in range(1, len(sweeps)):
        for i in range(L):
            below = Xb if i == 0 else f64(sweeps[j][i - 1][:rows])
            above = f64(sweeps[j - 1][i + 1][:rows]) if i + 1 < L else None
            p, t = cm.hidden(i, below, above)
            check_means(sweeps[j][i][:rows], p, t, '{0}: sweep {1}, mu{2}'.format(what, j, sfx(i)))
            np.testing.assert_array_equal(sweeps[j][i][rows:], stale[i][rows:],
                                          err_msg='{0}: sweep {1} wrote rows >= {2} of mu{3}'.format(what, j, rows, sfx(i)))
        REPORT['sweeps'] += 1
        diffs.append(max(float(np.max(np.abs(f64(sweeps[j][i][:rows]) - f64(sweeps[j - 1][i][:rows])))) for i in range(L)))
    return diffs


def stopping_points(diffs, d0_floor):
    """(t, mf_tol = d_t) for every sweep t whose measure is below all earlier ones (and below the t = 0 measure): the E-step
    with that tolerance stops after exactly t sweeps"""
    out = []
    for t in range(1, len(diffs) + 1):
        d = diffs[t - 1]
        if d < min(diffs[:t - 1] or [np.inf]) and d < d0_floor:
            out.append((t, d))
    return out


def d0_floor(cm, X, stale):
    """a lower bound of the t = 0 measure max |stale - approximate pass|"""
    rows = X.shape[0]
    return min(float(np.max(np.abs(f64(stale[i][:rows]) - p) - t)) for i, (p, t) in enumerate(cm.approximate(bf16r(X))))


ZERO_BUMP = 2.0 ** -4


def pinned_stale(cm, X, stale):
    """A stale mu equal to bf16 of the float64 approximate pass except one element of layer 0 raised by about 2^-4.  The t = 0
    measure is then that raise to within a slack: one bf16 ulp of a mean in [0, 1) (2^-8) twice over, for the pass's own
    roundings and their propagation through the next layer, or twice the largest bound if that is wider.  So mf_tol = raise +
    slack must stop with 0 sweeps and mf_tol = raise - slack must not.  A pass without the x2, or with a doubled bias, moves
    the means by far more.  Returns (stale, tol_stop, tol_go)."""
    rows = X.shape[0]
    out = [np.array(s, np.float32) for s in stale]
    slack = 2.0 ** -7
    for i, (p, t) in enumerate(cm.approximate(bf16r(X))):
        out[i][:rows] = bf16r(p)
        slack = max(slack, 2.0 * float(t.max()))
    r, c = np.unravel_index(np.argmin(np.abs(out[0][:rows] - 0.5)), out[0][:rows].shape)
    base = float(out[0][r, c])
    out[0][r, c] = bf16r(np.float32(base + ZERO_BUMP)).item()
    raise_ = float(out[0][r, c]) - base
    assert raise_ > 2.0 * slack, (raise_, slack)
    return out, raise_ + slack, raise_ - slack


def check_zero_sweeps(n_stop, n_go, what):
    assert n_stop == 0, '{0}: {1} sweeps where the stale mu is the approximate pass to within the bound'.format(what, n_stop)
    assert n_go >= 1, '{0}: no sweep where the stale mu is 2^-4 off the approximate pass'.format(what)


# ---- 4. particle sweeps --------------------------------------------------------------------------------------------------------
def particles(d, L):
    return f64(d['v']), [f64(d['h' + sfx(i)]) for i in range(L)]


def check_particle_sweep(cm, prev, cur, seed, tick, t, what):
    """sweep t: cur = (v, [h_i]) exported after it, prev = before it"""
    v0, H0 = prev
    v1, H1 = cur
    M = v0.shape[0]
    below = v0
    for i in range(cm.L):
        above = H0[i + 1] if i + 1 < cm.L else None
        p, tol = cm.hidden(i, below, above)
        name = '{0}: sweep {1}, h{2}'.format(what, t, sfx(i))
        if cm.sample_h[i]:
            u = P.uniform_at(M, p.shape[1], seed, P.SITE_DBM_H + i, t, tick).astype(np.float64)
            check_draws(H1[i], u, p, tol, name)
        else:
            check_means(H1[i], p, tol, name + ' (means)')
        below = H1[i]
    mean, tol = cm.visible(H1[0])
    name = '{0}: sweep {1}, v'.format(what, t)
    if not cm.sample_v:
        check_means(v1, mean, tol, name + ' (means)')
    elif cm.gauss:
        g, dg = gaussian_noise(M, mean.shape[1], seed, P.SITE_DBM_V, t, tick, 0)
        st = mean + cm.sigma[None, :] * g
        check_bf16(v1, st, tol + cm.sigma[None, :] * dg + 2.0 * ULP * np.abs(st), name + ' (Gaussian)')
    else:
        u = P.uniform_at(M, mean.shape[1], seed, P.SITE_DBM_V, t, tick).astype(np.float64)
        check_draws(v1, u, mean, tol, name)


# ---- 5. M-step -----------------------------------------------------------------------------------------------------------------
def assert_within(got, ref, tol, what):
    g = np.asarray(got, np.float64)
    bad = ~(np.abs(g - ref) <= tol)
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError('{0}: {1} of {2} elements off by more than the bound, first at {3}: got {4!r}, ref {5!r}, '
                             'tol {6:.3g}'.format(what, int(bad.sum()), bad.size, at, g[at], ref[at], tol[at]))


CS_RSPLIT = 64                   # row slabs of the bf16 column sums (csrc/bm_tc_util.cu)


def colsum(a):
    """float64 column sum of an fp32 column sum over the rows, and its bound.  The column sums (colsum_bf16_*) add in a fixed
    tree: 8 lanes stride over each of 64 row slabs, then the 8 lanes, then the 64 slabs, in order -- no element passes through
    more than ceil(slab / 8) + 8 + 64 adds.  (The sparsity quirk feeds a whole column sum into every unit's penalty, so the
    K 2^-23 bound of an unknown order, 15 times wider at 1100 rows, would hide a 1 % error in G behind the penalty's bound.)"""
    a = f64(a)
    depth = -(-(-(-a.shape[0] // CS_RSPLIT)) // 8) + 8 + CS_RSPLIT
    return a.sum(axis=0), depth * ACC * np.abs(a).sum(axis=0)


def expected_mstep(cfg, before, X, after, lr, mom):
    """float64 values of every variable the M-step writes, from the step's own activations (X, the exported mu rows, the final
    particles) and the state before it, each with its per-element bound: {name: (value, bound)}"""
    L = len(cfg['n_hiddens'])
    B, M = int(cfg['batch_size']), int(cfg['n_particles'])
    rows = X.shape[0]
    lr, mom = f32(lr), f32(mom)
    l2 = f32(cfg.get('l2', 0.0))
    damp = f32(cfg.get('sparsity_damping', 0.9))
    omd = float(np.float32(1) - np.float32(damp))
    costs = [f32(c) for c in cfg.get('sparsity_cost', [0.0] * L)]
    targets = [f32(t) for t in cfg.get('sparsity_target', [0.1] * L)]
    c = f32(cfg.get('max_norm', np.inf)) if np.isfinite(cfg.get('max_norm', np.inf)) else np.inf
    inv_n, inv_m = float(np.float32(1) / np.float32(B)), float(np.float32(1) / np.float32(M))
    mu = [f64(after['mu' + sfx(i)][:rows]) for i in range(L)]
    v, H = particles(after, L)
    Xb = bf16r(X)
    out = {}
    # visible bias (:553, :595-596): the mean over the rows present
    xs = f64(X).sum(axis=0)
    exs = 2.0 * ULP * np.abs(xs)
    vs, evs = colsum(v)
    g = xs / rows - vs / M
    eg = exs / rows + evs / M + rounding(3, xs / rows, vs / M)
    d = lr * (mom * f64(before['dvb']) + g)
    ed = lr * (eg + rounding(3, mom * f64(before['dvb']), g)) + ULP * np.abs(d)
    out['dvb'] = (d, ed)
    out['vb'] = (f64(before['vb']) + d, ed + rounding(1, before['vb'], d))
    pos, neg = [Xb] + mu[:-1], [v] + H[:-1]
    for i in range(L):
        s = sfx(i)
        # the sparsity penalty (:580-590): element `i` of the sum vectors (sic)
        ms, ems = colsum(mu[i])
        hs, ehs = colsum(H[i])
        q0, m0 = f64(before['q_means' + s]), f64(before['mu_means' + s])
        q = damp * q0 + omd * hs[i]
        eq = omd * ehs[i] + rounding(3, damp * q0, omd * hs[i])
        mm_ = damp * m0 + omd * ms[i]
        emm = omd * ems[i] + rounding(3, damp * m0, omd * ms[i])
        out['q_means' + s] = (q, eq)
        out['mu_means' + s] = (mm_, emm)
        pen = costs[i] * (q - targets[i]) + costs[i] * (mm_ - targets[i])
        epen = costs[i] * (eq + emm) + rounding(4, costs[i] * q, costs[i] * mm_, costs[i] * targets[i] * 2)
        # hidden bias (:575, :613-614)
        g = ms / rows - hs / M - pen
        eg = ems / rows + ehs / M + epen + rounding(3, ms / rows, hs / M, pen)
        dh = lr * (mom * f64(before['dhb' + s]) + g)
        edh = lr * (eg + rounding(3, mom * f64(before['dhb' + s]), g)) + ULP * np.abs(dh)
        out['dhb' + s] = (dh, edh)
        out['hb' + s] = (f64(before['hb' + s]) + dh, edh + rounding(1, before['hb' + s], dh))
        # weights (:558-568, :602-606, :511-513): G = pos^T mu / batch_size - neg^T h / n_particles, split-K over the rows
        A, eA = mm(pos[i].T, mu[i]), rows * ACC * mm(np.abs(pos[i]).T, np.abs(mu[i]))
        Bn, eB = mm(neg[i].T, H[i]), M * ACC * mm(np.abs(neg[i]).T, np.abs(H[i]))
        G = A * inv_n - Bn * inv_m
        eG = eA * inv_n + eB * inv_m + rounding(3, A * inv_n, Bn * inv_m)
        w, dw0 = f64(before['W' + s]), f64(before['dW' + s])
        g = G - l2 * w - pen[None, :]
        eg = eG + epen[None, :] + rounding(3, G, l2 * w, pen[None, :])
        dW = lr * (mom * dw0 + g)
        edW = lr * (eg + rounding(3, mom * dw0, g)) + ULP * np.abs(dW)
        wn = w + dW
        ewn = edW + rounding(1, w, dW)
        n = np.sqrt((wn * wn).sum(axis=0))
        en = np.sqrt((ewn * ewn).sum(axis=0)) + 2.0 * ULP * n
        W = wn * (np.minimum(n, c) / np.maximum(n, 1e-8))[None, :]
        eW = ewn + np.abs(W) * (en / np.maximum(n, 1e-8) + 4.0 * ULP)[None, :]
        out['dW' + s] = (dW, edW)
        out['W' + s] = (W, eW)
        out['norm' + s] = n
    return out


def check_mstep(cfg, before, X, after, lr, mom, what):
    """the variables the step left against expected_mstep; returns the column norms of the updated W_i"""
    exp = expected_mstep(cfg, before, X, after, lr, mom)
    for name, val in exp.items():
        if not name.startswith('norm'):
            assert_within(after[name], val[0], val[1], '{0}: {1}'.format(what, name))
    REPORT['msteps'] += 1
    return [exp['norm' + sfx(i)] for i in range(len(cfg['n_hiddens']))]


# ---- the engine's runs ---------------------------------------------------------------------------------------------------------
def mu_names(L):
    return ['mu' + sfx(i) for i in range(L)]


def engine(cfg, **over):
    return _native.CudaDBM(dict(cfg, **over))


def estep_sweeps(cfg, init, X, J):
    """every layer's mu after j = 0..J sweeps of the engine's E-step (one engine per j, the state restored)"""
    L = len(cfg['n_hiddens'])
    out = []
    for j in range(J + 1):
        eng = engine(cfg, max_mf_updates=j, mf_tol=-1.0)
        try:
            eng.set_params(init)
            eng.transform(X)
            g = eng.get_params(mu_names(L))
            out.append([g[n] for n in mu_names(L)])
        finally:
            eng.close()
    return out


def stops(cfg, init, X, mf_tol, max_mf):
    """(n_mf_updates, mu) of an E-step with this tolerance"""
    eng = engine(cfg, max_mf_updates=max_mf, mf_tol=mf_tol)
    try:
        eng.set_params(init)
        n = eng.val_metrics(X, 1, 5, 0)['n_mf_updates']
        g = eng.get_params(mu_names(len(cfg['n_hiddens'])))
        return int(n), [g[k] for k in mu_names(len(cfg['n_hiddens']))]
    finally:
        eng.close()


def replay_estep(c):
    cfg, init, X = c['cfg'], c['init'], c['X']
    L = len(cfg['n_hiddens'])
    cm = Conditionals(cfg, init)
    stale = [init['mu' + sfx(i)] for i in range(L)]
    sweeps = estep_sweeps(cfg, init, X, c['J'])
    diffs = check_estep(cm, X, stale, sweeps, c['name'] + ' E-step')
    points = stopping_points(diffs, d0_floor(cm, X, stale))
    assert points, diffs
    for t, d in points:
        n, mu = stops(cfg, init, X, d, max(int(cfg['max_mf_updates']), c['J']))
        assert n == t, '{0}: mf_tol = d_{1} = {2!r} stopped after {3} sweeps (measures {4})'.format(c['name'], t, d, n, diffs)
        for i in range(L):
            np.testing.assert_array_equal(mu[i], sweeps[t][i], err_msg='{0}: mu{1} after stopping at {2}'.format(c['name'], sfx(i), t))
        REPORT['decisions'] += 1
    pinned, tol_stop, tol_go = pinned_stale(cm, X, stale)
    state = dict(init, **{'mu' + sfx(i): pinned[i] for i in range(L)})
    n_stop, mu = stops(cfg, state, X, tol_stop, 25)
    n_go, _ = stops(cfg, state, X, tol_go, 25)
    check_zero_sweeps(n_stop, n_go, c['name'])
    for i in range(L):
        np.testing.assert_array_equal(mu[i], pinned[i], err_msg='{0}: mu{1} after 0 sweeps'.format(c['name'], sfx(i)))
    return diffs


def replay_particles(c, js, after_launches=None):
    """PCD-j for j in js (and the run before the first) from the restored state; sweep j of every j in js replayed from the run
    before it, the M-step of every run.  Returns ({j: exported state}, {j: launches of the step}, column norms)."""
    cfg, init, X = c['cfg'], c['init'], c['X']
    L = len(cfg['n_hiddens'])
    cm = Conditionals(cfg, init)
    seed, tick, lr, mom = c['seed'], c['tick'], c['lr'], c['mom']
    runs, launches, norms = {}, {}, None
    base = js[0] - 1
    eng = engine(cfg)
    try:
        for j in [base] + list(js):
            eng.set_params(init)
            n0 = eng.ctx.launch_count()
            if j > 0:
                eng.train_step(X, lr, mom, j, seed, tick)
            launches[j] = eng.ctx.launch_count() - n0
            runs[j] = eng.get_params()
        for j in js:
            what = '{0} PCD-{1}'.format(c['name'], j)
            prev = particles(runs[j - 1] if j - 1 in runs else init, L)
            check_particle_sweep(cm, prev, particles(runs[j], L), seed, tick, j, what)
            for n in mu_names(L):
                np.testing.assert_array_equal(runs[j][n], runs[js[0]][n], err_msg='{0}: {1} depends on k'.format(what, n))
            norms = check_mstep(cfg, init, X, runs[j], lr, mom, what)
        return runs, launches, norms
    finally:
        eng.close()


def replay_two_steps(c):
    """train_step on X, then on a new batch without set_params: each replayed (one E-step sweep, PCD-1, M-step) from the state
    before it -- the second from the engine's own update and its own bf16 shadows"""
    cfg = dict(c['cfg'], max_mf_updates=1, mf_tol=-1.0)
    L = len(cfg['n_hiddens'])
    eng = engine(cfg)
    try:
        eng.set_params(c['init'])
        before = eng.get_params()
        for step, X in enumerate((c['X'], c['X2'])):
            tick = c['tick'] + step
            eng.train_step(X, c['lr'], c['mom'], 1, c['seed'], tick)
            after = eng.get_params()
            what = '{0} step {1}'.format(c['name'], step + 1)
            cm = Conditionals(cfg, before)
            stale = [before['mu' + sfx(i)] for i in range(L)]
            check_estep(cm, X, stale, [stale, [after[n] for n in mu_names(L)]], what)
            check_particle_sweep(cm, particles(before, L), particles(after, L), c['seed'], tick, 1, what)
            check_mstep(cfg, before, X, after, c['lr'], c['mom'], what)
            before = after
    finally:
        eng.close()


# ---- 7. cases ------------------------------------------------------------------------------------------------------------------
def restored_state(cfg, w_scale, seed):
    """the benchmark's W init and every other variable a step reads, non-zero (momentum accumulators, sparsity means, biases,
    stale mu, particles), so that set_params restores the whole state"""
    d = _bench().dbm_params(cfg, scale=w_scale)
    rng = np.random.RandomState(seed)
    V, Hs, B, M = cfg['n_visible'], cfg['n_hiddens'], cfg['batch_size'], cfg['n_particles']
    gauss = cfg.get('v_kind') == 'gaussian'
    sh = cfg.get('sample_h', [True] * len(Hs))
    d['vb'] = (0.1 * rng.randn(V)).astype(np.float32)
    d['dvb'] = (1e-2 * rng.randn(V)).astype(np.float32)
    if gauss:
        d['v'] = bf16r(np.asarray(cfg['sigma'], np.float64) * rng.randn(M, V)).astype(np.float32)
    else:
        d['v'] = (rng.rand(M, V) < 0.3).astype(np.float32)
    for i, H in enumerate(Hs):
        s = sfx(i)
        d['hb' + s] = (0.3 * rng.randn(H)).astype(np.float32)
        d['dhb' + s] = (1e-2 * rng.randn(H)).astype(np.float32)
        d['dW' + s] = (1e-3 * rng.randn(*d['W' + s].shape)).astype(np.float32)
        d['q_means' + s] = rng.uniform(0.05, 0.3, H).astype(np.float32)
        d['mu_means' + s] = rng.uniform(0.05, 0.3, H).astype(np.float32)
        d['mu' + s] = bf16r(rng.rand(B, H)).astype(np.float32)
        d['h' + s] = ((rng.rand(M, H) < 0.5) if sh[i] else bf16r(rng.rand(M, H))).astype(np.float32)
    return d


def batch(cfg, rows, seed):
    if cfg.get('v_kind') == 'gaussian':
        return _bench().synth_cifar(rows, n_vis=cfg['n_visible'], seed=seed)
    return _bench().synth_mnist(rows, seed=seed, n_vis=cfg['n_visible'])


def make_case(name, cfg, rows, w_scale, lr, J, js, seed=31):
    return dict(name=name, cfg=cfg, init=restored_state(cfg, w_scale, seed), X=batch(cfg, rows, 3), X2=batch(cfg, rows, 4),
                lr=lr, mom=0.5, J=J, js=js, seed=0x5EED, tick=4)


def cfg4_case(name='cfg4', w_scale=0.02):
    return make_case(name, _bench().dbm_cfg('bf16'), 1024, w_scale, 2e-3, 25, (1, 2, 3))


def cfg5_pcd_case():
    cfg = _bench().dbm_cfg('bf16', [4096], 4096, 784, pcd_only=True)
    return make_case('cfg5-pcd', cfg, 4096, 0.01, 0.01, 1, tuple(range(1, 26)))


def ragged_cfg():
    V, Hs = 781, [509, 1001, 67]
    sigma = np.random.RandomState(5).uniform(0.5, 1.5, V).astype(np.float32)
    return dict(compute='bf16', n_visible=V, n_hiddens=Hs, v_kind='gaussian', sigma=sigma, h_kinds=['bernoulli'] * 3,
                h_n_samples=[100.] * 3, dtype='float32', n_particles=1100, batch_size=1024, max_mf_updates=25, mf_tol=1e-7,
                l2=1e-4, max_norm=6.0, sample_v=True, sample_h=[True, False, True], sparsity_target=[0.2, 0.1, 0.1],
                sparsity_cost=[0.1, 0.1, 0.1], sparsity_damping=0.9)


def ragged_case():
    return make_case('ragged', ragged_cfg(), 1000, 0.05, 0.05, 12, (1, 2, 3))


def small_cfg():
    return dict(compute='bf16', n_visible=30, n_hiddens=[18, 11], v_kind='bernoulli', h_kinds=['bernoulli'] * 2,
                h_n_samples=[100.] * 2, dtype='float32', n_particles=12, batch_size=10, max_mf_updates=8, mf_tol=1e-7, l2=1e-4,
                max_norm=1.5, sample_v=True, sample_h=[True, True], sparsity_target=[0.2, 0.1], sparsity_cost=[0.1, 0.1],
                sparsity_damping=0.9)


CASES = {
    'cfg4': cfg4_case,
    'cfg4-maxnorm': lambda: cfg4_case('cfg4-maxnorm', 0.25),
    'cfg5-pcd': cfg5_pcd_case,
    'ragged': ragged_case,
}


def replay_case(c):
    replay_estep(c)
    _, _, norms = replay_particles(c, c['js'])
    replay_two_steps(c)
    return norms


@big
@pytest.mark.parametrize('name', list(CASES))
def test_dbm_step_replay(name):
    c = CASES[name]()
    norms = replay_case(c)
    mn = c['cfg']['max_norm']
    bind = sum(int((n > mn).sum()) for n in norms)
    if name == 'cfg4-maxnorm':
        assert bind > 0, 'no column norm above max_norm: the rescale is not exercised'
    elif name == 'cfg5-pcd':
        assert c['cfg']['sample_v'] is False and len(c['cfg']['n_hiddens']) == 1


@big
def test_particle_program_and_per_op_launches():
    """k (L + 1) <= 90 ops run as one program, longer chains one launch per op: j = 29, 30 are replayed within the program path
    (from run 28), j = 32, 33 within the per-op path (from run 31).  The two paths are not assumed bit-identical."""
    cfg = _bench().dbm_cfg('bf16', rows=512)
    cfg['max_mf_updates'] = 1
    c = make_case('program-boundary', cfg, 512, 0.02, 2e-3, 1, None)
    L = len(cfg['n_hiddens'])
    for js in ((29, 30), (32, 33)):
        _, launches, _ = replay_particles(c, js)
        for j, n in launches.items():
            if j * (L + 1) <= PROGRAM_OPS:
                assert n < j * (L + 1), (j, n)             # one program launch for the particle sweeps
            else:
                assert n >= j * (L + 1), (j, n)            # one launch per op


def test_small_dbm_replay():
    """30-18-11, batch 10 of 10, 12 particles, max-norm binding: items 2-5 (also on the host simulation)"""
    c = make_case('small', small_cfg(), 10, 0.6, 0.05, 8, (1, 2, 3))
    replay_case(c)
    c = make_case('small-rows', small_cfg(), 7, 0.6, 0.05, 4, (1, 2))
    replay_case(c)


def test_report():
    """(runs last in this file) what the replays above checked"""
    print('\n[dbm-tc-replay] mean-field sweeps: {0}, stopping decisions: {1}, M-steps: {2}; draws checked: {3}, ambiguous '
          'disagreements: {4} (largest |u - p| {5:.3g}); means off bf16(ref): {6} of {7}'.format(
              REPORT['sweeps'], REPORT['decisions'], REPORT['msteps'], REPORT['draws'], REPORT['ambiguous'], REPORT['max_gap'],
              REPORT['off'], REPORT['means']))
    assert REPORT['off'] <= MAX_OFF * max(REPORT['means'], 1), REPORT
