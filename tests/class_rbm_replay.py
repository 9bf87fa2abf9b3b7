"""Float64 replay of one classification-RBM step (csrc/bm_crbm_tc.cuh) from the engine's own intermediates -- TEST
INFRASTRUCTURE ONLY.  Shared by tests/test_class_rbm_replay_host.py (the bf16 emulation below as a stand-in engine) and
tests/test_zz_class_rbm_replay_gpu.py (the engine, through CudaCRBM.debug_last_step).

Each stage is checked on the inputs the engine itself used, read back after the step, so an error cannot hide behind the
chaos of a sampled chain:

  A    = X bf16(W)             tensor-core accumulator: |err| <= K 2^-23 sum_k |x_k w_k|  (exact bf16 products, K = V)
  P    from the engine's A      o = fp32(fp32(A + hb) + U) is formed exactly here; softplus(o) in fp32 is off by at most
                                2^-24 sp + 2^-21 log1p(e^-|o|) (expf 2 ulp, log1pf 1 ulp, the final add); F sums H of them in
                                double; p = exp(F - log Z) moves by at most p * 2 max_y |dF_y| before its fp32 rounding
  NLL, accuracy                 the batch means the step returns; an argmax whose gap is within the F bounds is ambiguous
  y0   exact, given P           start_labels (tests/class_rbm_semi.py): the multinomial row kernel's CDF rule at
                                SITE_CRBM_Y0, row r, word 0
  G    bf16 of a value within the bound of (1 + alpha) s_t - sum_y p_y s_y (beta sum_y p_y s_y on an unlabelled row), with
       s = 1 / (1 + expf(-o)) off by at most s (1 - s) 2^-22 + s 2^-23 and one fp32 rounding per product and add
  h0   u < S_t at SITE_H0 (a draw within the bound of S_t is ambiguous), or bf16(S_t); S_{y0} on unlabelled rows
  chain  x_j | h_{j-1} at SITE_V, y_j | h_{j-1} by the row kernel's CDF rule at SITE_CRBM_Y, h_j | x_j, y_j (means: the
       last sweep never samples h), with the bounds of tests/test_zz_rbm_tc_chain_gpu.py (accumulator, 4 fp32 roundings of
       the epilogue, the approximate sigmoid).  h_{j-1} comes from h0 (j = 1) or from the CD-(j-1) run's h_k: with sample_h
       it is rebuilt as u < h at SITE_H, and a draw whose u lies within one bf16 ulp plus the mean's bound is ambiguous.
       Instead of a flip search, an ambiguous draw widens its row's pre-activation bound by |W| of its column: the largest
       change one flip can make, so the check stays rigorous whatever the kernel drew.
  aH   exact: bf16(w_r h_k), w_r = alpha (beta on unlabelled rows)
  gradients and update  from the engine's own P, A, G, x_k, y_k, h_k, aH.  W: the accumulator bound over both pairs
       (K = 2 rows) plus the fp32 sum of the s1 split-K slices; U, hb, yb, vb: in-order fp32 sums of at most 64 rows per
       split, then over the splits ((64 + splits) 2^-24 sum |terms|).  Then c / N - l2 theta, d = lr (mom d + g) and
       theta + d with one rounding each; theta_new == fp32(theta_old + d_new) bit for bit.

REPORT collects draws checked, ambiguous draws and the largest |difference| / bound per quantity."""
import numpy as np
import torch

from oracle import philox as P
from oracle.crbm import SITE_CRBM_Y
from class_rbm_bf16 import _bf, _mm, _mult, _sigmoid, _softplus, f32
from class_rbm_semi import OracleSemiCRBMbf16, SITE_CRBM_Y0, _check_labels, start_labels

U24 = 2.0 ** -24                 # fp32 unit roundoff
ACC = 2.0 ** -23                 # one truncating add of a tensor-core accumulator
ROWS_PER_SPLIT = 64              # CRBM_ROWS_PER_SPLIT
COLS = 128                       # CRBM_COLS
REPORT = dict(draws=0, ambiguous=0, h_rebuilt=0, h_ambiguous=0, worst={})


def reset_report():
    REPORT.update(draws=0, ambiguous=0, h_rebuilt=0, h_ambiguous=0, worst={})


def split_k(V, H, rows, sm_count):
    """the dW op's slice count, as hybrid_step picks it: min(SM pairs / 256 x 256 tiles, 64-row groups)"""
    tiles = ((V + 255) // 256) * ((H + 255) // 256)
    return max(1, min((sm_count // 2) // max(tiles, 1), (rows + 63) // 64))


def splits(rows):
    return (rows + ROWS_PER_SPLIT - 1) // ROWS_PER_SPLIT


def _t(x, dev):
    return torch.as_tensor(np.ascontiguousarray(x), device=dev)


def _d(x, dev):
    return _t(np.asarray(x, np.float64), dev)


def bf16r(x):
    """x rounded to fp32, then to the nearest bf16 (ties to even)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def bf16_ulp(x):
    return np.maximum(np.abs(x), 2.0 ** -126) * 2.0 ** -7


def within(name, got, ref, tol):
    """|got - ref| <= tol everywhere (float64); records the worst ratio"""
    got, ref, tol = (np.asarray(a, np.float64) for a in (got, ref, tol))
    diff = np.abs(got - ref)
    tol = np.broadcast_to(tol, diff.shape)
    ratio = float(np.max(diff / np.maximum(tol, 1e-300))) if diff.size else 0.0
    REPORT['worst'][name] = max(REPORT['worst'].get(name, 0.0), ratio)
    bad = ~(diff <= tol)
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError('{0}: {1} of {2} elements off by more than the bound, first at {3}: got {4!r}, ref {5!r}, '
                             'bound {6:.3g}'.format(name, int(bad.sum()), bad.size, at, got[at], ref[at], tol[at]))


def bf16_within(name, got, ref, tol):
    """got is the bf16 rounding of some value within ref +- tol"""
    got, ref, tol = np.asarray(got, np.float64), np.asarray(ref, np.float64), np.broadcast_to(tol, np.shape(ref))
    lo, hi = bf16r(ref - tol), bf16r(ref + tol)
    bad = ~((got >= lo) & (got <= hi))
    near = bf16r(ref)
    REPORT['worst'][name] = max(REPORT['worst'].get(name, 0.0),      # |got - ref| / (bound + half a bf16 ulp)
                                float(np.max(np.abs(got - ref) / (tol + 0.5 * bf16_ulp(near)))) if got.size else 0.0)
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError('{0}: {1} of {2} bf16 values outside the rounding of ref +- bound, first at {3}: got {4!r}, '
                             'ref {5!r}, bound {6:.3g}'.format(name, int(bad.sum()), bad.size, at, got[at], ref[at], tol[at]))


def bernoulli(name, got, u, p, tol):
    """states are u < p; a disagreement only where |u - p| <= tol"""
    got = np.asarray(got, np.float64)
    assert np.isin(got, (0.0, 1.0)).all(), name + ': states are not 0 / 1'
    want = (u < p).astype(np.float64)
    amb = np.abs(u - p) <= tol
    bad = (got != want) & ~amb
    REPORT['draws'] += got.size
    REPORT['ambiguous'] += int(amb.sum())
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError('{0}: {1} of {2} draws are not u < p, first at {3}: state {4}, u {5!r}, p {6!r}, bound {7:.3g}'
                             .format(name, int(bad.sum()), bad.size, at, got[at], u[at], p[at], tol[at]))


def sigmoid_tc_tol(p, e_pre):
    """the tensor-core epilogue's approximate sigmoid (ex2.approx / rcp.approx) of a pre-activation off by e_pre; results
    below fp32's smallest normal (2^-126) may flush to zero"""
    return p * (1.0 - p) * e_pre + 2.0 ** -21 * p + 2.0 ** -126


# ---- the posterior and the columns, from the engine's A and P -------------------------------------------------------------
class Columns(object):
    """per-row float64 quantities of the posterior and column kernels, in row chunks (o is [rows, C, H])"""

    def __init__(self, params, A, alpha, dev, chunk=256):
        self.dev, self.chunk = dev, chunk
        self.A = _t(np.asarray(A, np.float32), dev)
        self.hb = _t(np.asarray(params['hb'], np.float32), dev)
        self.U = _t(np.asarray(params['U'], np.float32), dev)
        self.yb = _d(np.asarray(params['yb'], np.float32), dev)
        self.pos = np.float32(np.float32(1) + np.float32(alpha))

    def o(self, r0, r1):
        """fp32(fp32(A + hb) + U): formed exactly as the kernels form it"""
        a = self.A[r0:r1] + self.hb
        return (a[:, None, :] + self.U[None, :, :]).double()

    def free_energy(self):
        """F [rows, C] and its bound"""
        Fs, Es = [], []
        for r0 in range(0, self.A.shape[0], self.chunk):
            o = self.o(r0, r0 + self.chunk)
            sp = torch.logaddexp(o, torch.zeros((), dtype=o.dtype, device=o.device))
            l = torch.log1p(torch.exp(-o.abs()))
            Fs.append(self.yb + sp.sum(2))
            Es.append((U24 * sp + 2.0 ** -21 * l).sum(2) + o.shape[2] * 2.0 ** -52 * sp.sum(2))
        return torch.cat(Fs).cpu().numpy(), torch.cat(Es).cpu().numpy()

    def sigmoids(self, r0, r1):
        """s [n, C, H] in float64 and the bound of the kernel's fp32 1 / (1 + expf(-o)) (which is 0 where expf overflows:
        there s < 2^-126)"""
        s = torch.sigmoid(self.o(r0, r1))
        return s, s * (1 - s) * 2.0 ** -22 + s * 2.0 ** -23 + 2.0 ** -126


def posterior_reference(F, eF):
    """p [rows, C] and its bound from F and the bound of F"""
    m = F.max(axis=1, keepdims=True)
    logz = m + np.log(np.exp(F - m).sum(axis=1, keepdims=True))
    p = np.exp(F - logz)
    e = eF.max(axis=1, keepdims=True)
    return p, logz[:, 0], p * (2.0 * e * 1.01 + U24) + 2.0 ** -149


def check_posterior(Pe, F, eF, y, metrics):
    """P element by element; the step's NLL and accuracy over the labelled rows"""
    p, logz, ep = posterior_reference(F, eF)
    within('P', Pe, p, ep)
    if metrics is None:
        return
    lab = np.where(y >= 0)[0]
    if not len(lab):
        assert np.isnan(metrics['nll']) and np.isnan(metrics['accuracy']), metrics
        return
    emax = eF.max(axis=1)
    nll = logz[lab] - F[lab, y[lab]]
    within('NLL', metrics['nll'], nll.mean(), 2.0 * emax[lab].mean() + 1e-12 * max(1.0, abs(nll.mean())))
    # a class can be the kernel's argmax if its F is within both bounds of the largest; ties go to the lowest class
    cand = F[lab] >= (F[lab].max(axis=1, keepdims=True) - 2.0 * emax[lab, None])
    sure = cand.sum(axis=1) == 1
    hit = cand[np.arange(len(lab)), y[lab]]
    lo, hi = int((hit & sure).sum()), int(hit.sum())
    REPORT['ambiguous'] += int((~sure).sum())
    got = metrics['accuracy'] * len(lab)
    assert lo - 1e-6 <= got <= hi + 1e-6, ('accuracy', got, lo, hi)


def column_terms(cols, Pe, y, y0, alpha, beta, r0, r1):
    """for rows [r0, r1): g (the value G rounds) and its bound, S_t (the chain's start mean) and its bound, the gU terms
    coef s and their bound, coef and its bound (all float64 torch on the device)"""
    dev = cols.dev
    s, es = cols.sigmoids(r0, r1)
    n = r1 - r0
    p = _d(np.asarray(Pe[r0:r1], np.float32), dev)
    yy = np.asarray(y[r0:r1])
    unl = _t(yy < 0, dev)
    ts = _t(np.where(yy < 0, np.asarray(y0[r0:r1]) if y0 is not None else 0, yy), dev).long()
    ar = torch.arange(n, device=dev)
    C = p.shape[1]
    ps = p[:, :, None] * s
    sh = ps.sum(1)
    esh = (p[:, :, None] * es).sum(1) + (C + 1) * U24 * ps.sum(1)
    st, est = s[ar, ts], es[ar, ts]
    pos, b = float(cols.pos), float(np.float32(beta))
    g = torch.where(unl[:, None], b * sh, pos * st - sh)
    eg = torch.where(unl[:, None], b * esh + U24 * b * sh, pos * est + U24 * pos * st + esh) + U24 * g.abs()
    E = torch.zeros_like(p)
    E[ar[~unl], ts[~unl]] = 1.0
    coef = torch.where(unl[:, None], b * p, pos * E - p)
    ecoef = U24 * coef.abs()
    terms = coef[:, :, None] * s
    eterms = coef.abs()[:, :, None] * es + s * ecoef[:, :, None] + U24 * terms.abs()
    return g, eg, st, est, terms, eterms, coef, ecoef


# ---- one step ---------------------------------------------------------------------------------------------------------------
def check_step(cfg, before, after, X, y, k, seed, tick, lr, mom, dbg, metrics, sm_count, dev, h_prev=None):
    """every stage of one train_step from `before` to `after` (variables and momenta), given the step's debug buffers.
    h_prev: (h_{k-1} states or means, ambiguous mask, tolerance) of a CD-k prefix for k > 1 (None: the x / y half-steps of
    the last sweep are checked only at k = 1, from h0)."""
    V, H, C = int(cfg['n_visible']), int(cfg['n_hidden']), int(cfg['n_classes'])
    alpha, beta, l2 = float(cfg.get('alpha', 0.01)), float(cfg.get('beta', 0.0)), float(cfg.get('l2', 0.0))
    sample_v, sample_h = bool(cfg.get('sample_v', False)), bool(cfg.get('sample_h', True))
    X = np.asarray(X, np.float32)
    y = np.asarray(y, np.int64).reshape(-1)
    n = len(y)
    unl = y < 0
    semi = bool(unl.any())
    gen = alpha > 0 or semi
    Xb = bf16r(X)
    Wb, Ub = bf16r(before['W']), bf16r(before['U'])

    # A = X bf16(W)
    Xt, Wt = _d(Xb, dev), _d(Wb, dev)
    Aref = (Xt @ Wt).cpu().numpy()
    eA = (V * ACC * (Xt.abs() @ Wt.abs())).cpu().numpy() + U24 * np.abs(Aref)       # (+ the fp32 store)
    within('A', dbg['A'], Aref, eA)

    cols = Columns(before, dbg['A'], alpha, dev)
    F, eF = cols.free_energy()
    check_posterior(dbg['P'], F, eF, y, metrics)
    y0 = None
    if semi:
        y0 = np.asarray(dbg['y0'])
        want = start_labels(np.asarray(dbg['P'], np.float32), seed, tick)
        bad = unl & (y0 != want)
        assert not bad.any(), ('y0', np.where(bad)[0][:5], y0[bad][:5], want[bad][:5])
        REPORT['draws'] += int(unl.sum())

    # columns: G, h0, and the discriminative sums with their bounds
    nU = (C, H)
    gU, egU = np.zeros(nU), np.zeros(nU)
    ghb, eghb, gyb, egyb = np.zeros(H), np.zeros(H), np.zeros(C), np.zeros(C)
    absU, absH, absY = np.zeros(nU), np.zeros(H), np.zeros(C)
    u0 = P.uniform_at(n, H, seed, P.SITE_H0, 0, tick) if gen and k == 1 and sample_h else None
    for r0 in range(0, n, ROWS_PER_SPLIT * 4):
        r1 = min(n, r0 + ROWS_PER_SPLIT * 4)
        g, eg, st, est, terms, eterms, coef, ecoef = column_terms(cols, dbg['P'], y, y0, alpha, beta, r0, r1)
        g_, eg_ = g.cpu().numpy(), eg.cpu().numpy()
        bf16_within('G', dbg['G'][r0:r1], g_, eg_)
        gU += terms.sum(0).cpu().numpy(); egU += eterms.sum(0).cpu().numpy(); absU += terms.abs().sum(0).cpu().numpy()
        ghb += g_.sum(0); eghb += eg_.sum(0); absH += np.abs(g_).sum(0)
        gyb += coef.sum(0).cpu().numpy(); egyb += ecoef.sum(0).cpu().numpy(); absY += coef.abs().sum(0).cpu().numpy()
        if gen and k == 1:
            st_, est_ = st.cpu().numpy(), est.cpu().numpy()
            h0 = dbg['h0'][r0:r1]
            if sample_h:
                bernoulli('h0', h0, u0[r0:r1], st_, est_)
            else:
                bf16_within('h0', h0, st_, est_)
    s2 = splits(n)
    sum_err = lambda absum, ns: (ROWS_PER_SPLIT + ns) * U24 * absum
    grad = {'W': None, 'U': [gU, egU + sum_err(absU, s2)], 'hb': [ghb, eghb + sum_err(absH, s2)],
            'yb': [gyb, egyb + sum_err(absY, s2)], 'vb': [np.zeros(V), np.zeros(V)]}

    # dW = X^T G - X_k^T aH: the engine's own operands
    G = _d(dbg['G'], dev)
    Wsum, Wabs = Xt.T @ G, Xt.T.abs() @ G.abs()
    if gen:
        xk, yk, hk = (np.asarray(dbg[nm], np.float64) for nm in ('x_k', 'y_k', 'h_k'))
        w = np.where(unl, np.float32(beta), np.float32(alpha)).astype(np.float32)[:, None]
        aH_want = bf16r(w * np.asarray(hk, np.float32))
        assert np.array_equal(np.asarray(dbg['aH'], np.float64), aH_want), \
            ('aH', np.argwhere(np.asarray(dbg['aH']) != aH_want)[:5])
        check_chain(cfg, before, dbg, k, seed, tick, dev, h_prev, sample_v, sample_h)
        XK, AH = _d(xk, dev), _d(dbg['aH'], dev)
        Wsum, Wabs = Wsum - XK.T @ AH, Wabs + XK.T.abs() @ AH.abs()
        for m, wt in ((~unl, alpha), (unl, beta)):
            if not m.any():
                continue
            YH = yk[m].T @ hk[m]
            grad['U'][0] -= wt * YH
            grad['U'][1] += wt * sum_err(YH, s2) + U24 * wt * np.abs(YH)
            grad['hb'][0] -= wt * hk[m].sum(0)
            grad['hb'][1] += wt * sum_err(hk[m].sum(0), s2) + U24 * wt * hk[m].sum(0)
            grad['yb'][0] -= wt * yk[m].sum(0)
            grad['yb'][1] += wt * sum_err(yk[m].sum(0), s2) + U24 * wt * yk[m].sum(0)
            dx = Xb[m] - xk[m]
            grad['vb'][0] += wt * dx.sum(0)
            grad['vb'][1] += wt * sum_err(np.abs(dx).sum(0), s2) + U24 * wt * np.abs(dx.sum(0))
    s1 = split_k(V, H, n, sm_count)
    K = 2 * n if gen else n
    Wabs = Wabs.cpu().numpy()
    grad['W'] = [Wsum.cpu().numpy(), (K * ACC + s1 * U24) * Wabs]
    for name in ('W', 'U', 'vb', 'hb', 'yb'):
        c, ec = grad[name]
        ec = ec + 2 * U24 * np.abs(c)                              # c = a - alpha b (- beta b_u): the subtractions
        th = np.asarray(before[name], np.float32).astype(np.float64)
        decay = l2 * th if name in ('W', 'U') else 0.0
        g = c / n - decay
        eg = ec / n + U24 * (np.abs(c) / n + 2 * np.abs(decay) + np.abs(g))
        d_old = np.asarray(before['d' + name], np.float32).astype(np.float64)
        md = np.float32(mom) * d_old
        d_ref = np.float32(lr) * (md + g)
        e_d = float(np.float32(lr)) * (eg + U24 * (np.abs(md) + np.abs(md + g))) + U24 * np.abs(d_ref)
        within('d' + name, after['d' + name], d_ref, e_d)
        want = (np.asarray(before[name], np.float32) + np.asarray(after['d' + name], np.float32)).astype(np.float32)
        assert np.array_equal(np.asarray(after[name], np.float32), want), (name, 'theta + d is not the stored variable')
    return s1


def run_step(eng, cfg, X, y, lr, mom, k, seed, tick, sm_count, dev, h_prev=None):
    """one train_step of `eng` (CudaCRBM or SplitEmulation) checked stage by stage; returns its debug buffers"""
    y = np.asarray(y).reshape(-1)
    gen = float(cfg.get('alpha', 0.01)) > 0 or bool((y < 0).any())
    before = eng.get_params()
    metrics = eng.train_step(X, y, lr, mom, k, seed=seed, tick=tick, metrics=True)
    names = ['A', 'P', 'y0', 'G'] + ((['x_k', 'y_k', 'h_k', 'aH'] + (['h0'] if k == 1 else [])) if gen else [])
    dbg = eng.debug_last_step(names)
    check_step(cfg, before, eng.get_params(), X, y, k, seed, tick, lr, mom, dbg, metrics, sm_count, dev, h_prev)
    return dbg


def check_prefixes(eng, cfg, params, X, y, K, seed, tick, sm_count, dev):
    """CD-1 .. CD-K from the same variables (momenta zero), each run's last sweep replayed from the previous run's h_k"""
    h_prev = None
    for j in range(1, K + 1):
        eng.set_params(params)
        dbg = run_step(eng, cfg, X, y, 1.0, 0.0, j, seed, tick, sm_count, dev, h_prev)
        h_prev = rebuild_h(dbg['h_k'], h_bound(cfg, params, dbg), seed, tick, j, bool(cfg.get('sample_h', True)))


def check_chain(cfg, before, dbg, k, seed, tick, dev, h_prev, sample_v, sample_h):
    """the last sweep (j = k): x_k | h_{k-1}, y_k | h_{k-1} (at k = 1 from h0, else from h_prev) and h_k | x_k, y_k.
    Returns (h_k, its bound) for the next prefix."""
    Wb, Ub = _d(bf16r(before['W']), dev), _d(bf16r(before['U']), dev)
    vb, hb, yb = (np.asarray(before[nm], np.float32).astype(np.float64) for nm in ('vb', 'hb', 'yb'))
    xk, yk, hk = (np.asarray(dbg[nm], np.float64) for nm in ('x_k', 'y_k', 'h_k'))
    n, V = xk.shape
    H, C = hk.shape[1], yk.shape[1]
    # h_k | x_k, y_k: one two-pair op, K = V + C
    XK, YK = _d(xk, dev), _d(yk, dev)
    a = (XK @ Wb + YK @ Ub).cpu().numpy()
    ea = ((V + C) * ACC * (XK.abs() @ Wb.abs() + YK.abs() @ Ub.abs())).cpu().numpy() + 4 * U24 * (np.abs(a) + np.abs(hb))
    ph = 1.0 / (1.0 + np.exp(-(a + hb)))
    tol_h = sigmoid_tc_tol(ph, ea)
    bf16_within('h_k', hk, ph, tol_h)
    if k == 1:
        hp, amb = np.asarray(dbg['h0'], np.float64), np.zeros(hk.shape, bool)
    elif h_prev is not None:
        hp, amb = h_prev
    else:
        return
    HP, AMB = _d(hp, dev), _d(amb.astype(np.float64), dev)
    # x_k | h_{k-1}
    a = (HP @ Wb.T).cpu().numpy()
    ea = (H * ACC * (HP.abs() @ Wb.abs().T) + AMB @ Wb.abs().T).cpu().numpy() + 4 * U24 * (np.abs(a) + np.abs(vb))
    px = 1.0 / (1.0 + np.exp(-(a + vb)))
    tol = sigmoid_tc_tol(px, ea)
    if sample_v:
        bernoulli('x_k', xk, P.uniform_at(n, V, seed, P.SITE_V, k, tick), px, tol)
    else:
        bf16_within('x_k', xk, px, tol)
    # y_k | h_{k-1}: a raw fp32 op, then the multinomial row kernel (fp32 softmax; with sample_v one draw by its CDF rule)
    a = (HP @ Ub.T).cpu().numpy() + yb
    ea = (H * ACC * (HP.abs() @ Ub.abs().T) + AMB @ Ub.abs().T).cpu().numpy() + 4 * U24 * (np.abs(a) + np.abs(yb))
    q = np.exp(a - a.max(axis=1, keepdims=True))
    q /= q.sum(axis=1, keepdims=True)
    eq = q * (2.0 * ea.max(axis=1, keepdims=True) * 1.01 + 2.0 ** -20)
    if not sample_v:
        bf16_within('y_k', yk, q, eq)
        return
    assert np.isin(yk, (0.0, 1.0)).all() and (yk.sum(1) == 1).all(), 'y_k is not one-of-C'
    pick = yk.argmax(1)
    cdf = np.cumsum(q, axis=1)
    ecdf = np.cumsum(eq, axis=1) + (C + 2) * 2.0 ** -23 * cdf
    u = P.uniform_at(n, 1, seed, SITE_CRBM_Y, k, tick)[:, 0].astype(np.float64)
    lo = np.where(pick > 0, cdf[np.arange(n), np.maximum(pick - 1, 0)] - ecdf[np.arange(n), np.maximum(pick - 1, 0)], -1.0)
    hi = np.where(pick < C - 1, cdf[np.arange(n), pick] + ecdf[np.arange(n), pick], 2.0)
    bad = ~((u >= lo) & (u < hi))
    sure = np.minimum((cdf > u[:, None]).argmax(1), C - 1)
    REPORT['draws'] += n
    REPORT['ambiguous'] += int((np.abs(cdf - u[:, None]) <= ecdf).any(axis=1).sum())
    assert not bad.any(), ('y_k draws outside their CDF interval', np.where(bad)[0][:5], pick[bad][:5], sure[bad][:5])


def rebuild_h(h_k, tol_h, seed, tick, j, sample_h):
    """h_j as sweep j + 1 of a longer chain sees it, from the CD-j run's exported h_k (a bf16 mean) and its bound: with
    sample_h the states u < mean at SITE_H, t = j, ambiguous where u is within one bf16 ulp plus the bound of the mean"""
    h_k = np.asarray(h_k, np.float64)
    if not sample_h:
        return h_k, np.zeros(h_k.shape, bool)
    u = P.uniform_at(h_k.shape[0], h_k.shape[1], seed, P.SITE_H, j, tick).astype(np.float64)
    amb = np.abs(u - h_k) <= bf16_ulp(h_k) + tol_h
    REPORT['h_rebuilt'] += h_k.size
    REPORT['h_ambiguous'] += int(amb.sum())
    return (u < h_k).astype(np.float64), amb


def h_bound(cfg, params, dbg):
    """the bound of the kernel's fp32 mean behind the exported h_k"""
    Wb, Ub = bf16r(params['W']), bf16r(params['U'])
    xk, yk = np.asarray(dbg['x_k'], np.float64), np.asarray(dbg['y_k'], np.float64)
    hb = np.asarray(params['hb'], np.float32).astype(np.float64)
    a = xk @ Wb + yk @ Ub
    ea = (xk.shape[1] + yk.shape[1]) * ACC * (np.abs(xk) @ np.abs(Wb) + yk @ np.abs(Ub)) + 4 * U24 * (np.abs(a) + np.abs(hb))
    p = 1.0 / (1.0 + np.exp(-(a + hb)))
    return sigmoid_tc_tol(p, ea)


def check_queries(params, X, Pe, She, dev, chunk=2048):
    """predict_proba and transform row by row, from X alone: A's accumulator bound carried through o, F, p and S^"""
    Wb = _d(bf16r(params['W']), dev)
    hb = _d(np.asarray(params['hb'], np.float32), dev)
    U = _d(np.asarray(params['U'], np.float32), dev)
    yb = _d(np.asarray(params['yb'], np.float32), dev)
    V = Wb.shape[0]
    for r0 in range(0, len(X), chunk):
        Xt = _d(bf16r(X[r0:r0 + chunk]), dev)
        A = Xt @ Wb
        a = A + hb
        o = a[:, None, :] + U[None]
        eo = (V * ACC * (Xt @ Wb.abs()) + U24 * (a.abs() + A.abs()))[:, None, :] + U24 * o.abs()
        sp = torch.logaddexp(o, torch.zeros((), dtype=o.dtype, device=o.device))
        s = torch.sigmoid(o)
        F = yb + sp.sum(2)
        eF = (s * eo + U24 * sp + 2.0 ** -21 * torch.log1p(torch.exp(-o.abs()))).sum(2)
        p, _, ep = posterior_reference(F.cpu().numpy(), eF.cpu().numpy())
        within('predict_proba', Pe[r0:r0 + chunk], p, ep)
        pt, ept = _t(p, dev), _t(ep, dev)
        es = s * (1 - s) * (eo + 2.0 ** -22) + s * 2.0 ** -23 + 2.0 ** -126
        sh = (pt[:, :, None] * s).sum(1)
        esh = (ept[:, :, None] * s + pt[:, :, None] * es).sum(1) + (s.shape[1] + 1) * U24 * sh
        within('transform', She[r0:r0 + chunk], sh.cpu().numpy(), esh.cpu().numpy())


# ---- the bf16 emulation as a stand-in engine ---------------------------------------------------------------------------------
MUTATIONS = ('no_pos', 'next_row_p', 'drop_last_split', 'drop_w_slice', 'gyb_every_block', 'unl_alpha', 'y0_word1',
             'y0_next_row', 'label_at_site_v', 'sample_last_h', 'u_shadow_transposed', 'l2_hb', 'skip_last_class',
             'no_momentum')


class SplitEmulation(OracleSemiCRBMbf16):
    """OracleCRBMbf16 / OracleSemiCRBMbf16 summing as the kernels do -- in 64-row fp32 splits, the W gradient in s1 split-K
    slices -- with the chain reading bf16 shadows of W and U refreshed by the update, and the step's buffers kept for
    debug_last_step.  `mutation` (one of MUTATIONS) plants one wrong term, to show that the checks above see it."""

    def __init__(self, cfg, sm_count=132, mutation=None):
        super(SplitEmulation, self).__init__(cfg)
        assert mutation in (None,) + MUTATIONS, mutation
        self.sm_count, self.mut, self.last = sm_count, mutation, None
        self._shadows()

    def _shadows(self):
        self.Wsh = _bf(self.p['W'])
        self.Ush = _bf(self.p['U'].T).reshape(self.C, self.H) if self.mut == 'u_shadow_transposed' else _bf(self.p['U'])

    def set_params(self, d):
        super(SplitEmulation, self).set_params(d)
        self._shadows()

    def debug_last_step(self, names=None):
        return {k: v for k, v in self.last.items() if names is None or k in names}

    def _y0(self, Pr, seed, tick):
        n = len(Pr)
        u = P.uniform_at(n + 1, 2, seed, SITE_CRBM_Y0, 0, tick).astype(np.float64)
        u = u[1:, 0] if self.mut == 'y0_next_row' else u[:n, 1] if self.mut == 'y0_word1' else u[:n, 0]
        q = (Pr.astype(np.float64) / np.cumsum(Pr.astype(np.float64), axis=1)[:, -1:]).astype(np.float32).astype(np.float64)
        cdf = np.cumsum(q, axis=1)
        return np.minimum((cdf / cdf[:, -1:] > u[:, None]).argmax(1), self.C - 1)

    def train_step(self, X, y, lr, momentum, k, seed, tick, metrics=False):
        p, C, H, V, mut = self.p, self.C, self.H, self.V, self.mut
        y = np.asarray(y, np.int64).reshape(-1)
        unl = _check_labels(y, C, self.beta)
        X = np.asarray(X, f32)
        n, lab = len(y), ~unl
        semi = bool(unl.any())
        gen = self.alpha > 0 or semi
        alpha, beta = f32(self.alpha), f32(self.beta)
        pos = f32(1) if mut == 'no_pos' else f32(1) + alpha
        Xb = _bf(X)
        A = _mm(Xb, self.Wsh)
        O = ((A + p['hb']).astype(f32)[:, None, :] + p['U'][None]).astype(f32)
        used = C - 1 if (mut == 'skip_last_class' and C > 16) else C
        F = p['yb'].astype(np.float64)[None, :] + np.pad(_softplus(O[:, :used]).astype(np.float64).sum(axis=2),
                                                         ((0, 0), (0, C - used)))
        m = F.max(axis=1, keepdims=True)
        logz = (m + np.log(np.exp(F - m).sum(axis=1, keepdims=True)))[:, 0]
        Pr = np.exp(F - logz[:, None]).astype(f32)
        out = None
        if metrics:
            r = np.where(lab)[0]
            out = {'nll': float(np.mean(logz[r] - F[r, y[r]])) if len(r) else float('nan'),
                   'accuracy': float(np.mean(np.argmax(F[r], axis=1) == y[r])) if len(r) else float('nan')}
        y0 = self._y0(Pr, seed, tick) if semi else np.zeros(n, np.int64)
        S = _sigmoid(O)
        S[:, used:] = 0
        ts = np.where(unl, y0, y)
        St = S[np.arange(n), ts]
        Pm = np.roll(Pr, -1, axis=0) if mut == 'next_row_p' else Pr
        Sh = (Pm[:, :, None] * S).sum(axis=1, dtype=f32).astype(f32)
        g = np.where(unl[:, None], beta * Sh, pos * St - Sh).astype(f32)
        E = np.zeros((n, C), f32)
        E[np.where(lab)[0], y[lab]] = 1
        coef = np.where(unl[:, None], beta * Pr, pos * E - Pr).astype(f32)
        s2 = splits(n)
        keep = range(s2 - 1) if mut == 'drop_last_split' else range(s2)
        sl = [slice(s * ROWS_PER_SPLIT, min(n, (s + 1) * ROWS_PER_SPLIT)) for s in range(s2)]
        gU = sum(((coef[sl[s], :, None] * S[sl[s]]).sum(axis=0, dtype=f32) for s in keep), np.zeros((C, H), f32))
        ghb = sum((g[sl[s]].sum(axis=0, dtype=f32) for s in keep), np.zeros(H, f32))
        blocks = (H + COLS - 1) // COLS if mut == 'gyb_every_block' else 1
        gyb = sum((coef[sl[s]].sum(axis=0, dtype=f32) * f32(blocks) for s in keep), np.zeros(C, f32))
        G = _bf(g)
        last = {'A': A, 'P': Pr, 'y0': y0.astype(np.int32), 'G': G}
        XK, AH = None, None
        yh = yhu = np.zeros((C, H), f32)
        hk = hku = np.zeros(H, f32)
        xd = xdu = np.zeros(V, f32)
        yk = yku = np.zeros(C, f32)
        if gen:
            h = (P.uniform_at(n, H, seed, P.SITE_H0, 0, tick) < St).astype(f32) if self.sample_h else _bf(St)
            if int(k) == 1:
                last['h0'] = h
            ysite = P.SITE_V if mut == 'label_at_site_v' else SITE_CRBM_Y
            for s in range(1, int(k) + 1):
                xm = _sigmoid(_mm(h, self.Wsh.T) + p['vb'])
                x = (P.uniform_at(n, V, seed, P.SITE_V, s, tick) < xm).astype(f32) if self.sample_v else _bf(xm)
                ym = _mult.softmax_rows((_mm(h, self.Ush.T) + p['yb']).astype(f32), 1.0)
                yv = _mult.multinomial_rows(ym, 1, seed, ysite, s, tick) if self.sample_v else _bf(ym)
                hm = _sigmoid((_mm(x, self.Wsh) + _mm(yv, self.Ush)).astype(f32) + p['hb'])
                samp = self.sample_h and (s < int(k) or mut == 'sample_last_h')
                h = (P.uniform_at(n, H, seed, P.SITE_H, s, tick) < hm).astype(f32) if samp else _bf(hm)
            XK, YK, HK = x, _bf(yv), h
            w = np.where(unl & (mut != 'unl_alpha'), beta, alpha).astype(f32)[:, None]
            AH = _bf(w * HK)
            last.update(x_k=XK, y_k=YK, h_k=HK, aH=AH)

            def stats(m):
                acc = [np.zeros((C, H), f32), np.zeros(H, f32), np.zeros(V, f32), np.zeros(C, f32)]
                for s in range(s2):
                    r = np.arange(sl[s].start, sl[s].stop)
                    r = r[m[r]]
                    acc[0] += (YK[r, :, None] * HK[r, None, :]).sum(axis=0, dtype=f32)
                    acc[1] += HK[r].sum(axis=0, dtype=f32)
                    acc[2] += (Xb[r] - XK[r]).sum(axis=0, dtype=f32)
                    acc[3] += YK[r].sum(axis=0, dtype=f32)
                return acc
            yh, hk, xd, yk = stats(lab)
            yhu, hku, xdu, yku = stats(unl)
        s1 = split_k(V, H, n, self.sm_count)
        step = -(-n // s1)
        GW = np.zeros((V, H), f32)
        for s in range(s1 - 1 if mut == 'drop_w_slice' else s1):
            r = slice(s * step, min(n, (s + 1) * step))
            part = Xb[r].T.astype(np.float64) @ G[r].astype(np.float64)
            if gen:
                part -= XK[r].T.astype(np.float64) @ AH[r].astype(np.float64)
            GW += part.astype(f32)
        N, l2 = f32(n), f32(self.l2)
        grads = {'W': (GW / N - l2 * p['W']).astype(f32),
                 'U': ((gU - alpha * yh - beta * yhu).astype(f32) / N - l2 * p['U']).astype(f32),
                 'vb': ((alpha * xd + beta * xdu).astype(f32) / N).astype(f32),
                 'hb': ((ghb - alpha * hk - beta * hku).astype(f32) / N - (l2 * p['hb'] if mut == 'l2_hb' else 0)).astype(f32),
                 'yb': ((gyb - alpha * yk - beta * yku).astype(f32) / N).astype(f32)}
        lr, mom = f32(lr), f32(0 if mut == 'no_momentum' else momentum)
        for name in ('W', 'U', 'vb', 'hb', 'yb'):
            d = (lr * (mom * p['d' + name] + grads[name])).astype(f32)
            p['d' + name] = d
            p[name] = (p[name] + d).astype(f32)
        self._shadows()
        self.last = last
        return out
