"""Every Gibbs half-step of the tensor-core CD-k program (csrc/bm_rbm_tc.cu run_program, csrc/bm_tc.cu launch_tc_program) at
the benchmark's own sizes, against a float64 statement of each conditional.

Chain prefixes.  Every half-step draws from the Philox stream keyed by (seed, site, t, tick, row0), and the key does not depend
on k, so the chain of a CD-j step is, half-step by half-step, the first j steps of any longer chain.  For one parameter state,
batch, seed and tick the engine runs CD-1, CD-2, ..., CD-K (parameters restored before each run), and the activations CD-j
exports are checked against a float64 replay from those of CD-(j-1):

  v_j | h_{j-1}  h_{j-1} is never exported.  It is rebuilt from CD-(j-1)'s v_states: p = sigmoid(m (v W_bf16) + m hb) in
                 float64 and s = u < p with u = Philox(SITE_H, j - 1) (CD-1 uses the exported h0_states; with sample_h off the
                 state is CD-(j-1)'s exported h_means itself).  CD-j's v_means must then equal the float64 conditional of s
                 (see the bound below); with sample_v its v_states must be u < p at SITE_V, or Box-Muller for Gaussian visibles.
  h_j | v_j      CD-j's h_means against the float64 conditional of its own v_states.
  update         the parameters left by every CD-j run against the oracle's formulas on that run's activations.

Ambiguous draws.  The kernel compares u with its own fp32 p, so a draw with |u - p| within the error bound of p may come out
either way.  Such draws are resolved row by row: a row of v_j that does not match the replay of s is tried again with one of its
ambiguous hidden draws flipped (closest |u - p| first), then with two of the 8 closest.  A flip changes the row's pre-activation
by +- m W[:, col]: a cheap update of one row.  A row that matches none of these fails the test, and at most 1 % of the rebuilt
rows may need a flip.

Error bound.  The operands are exact bf16 values (binary states, bf16 means, the bf16 shadow of W), so every product is exact
in fp32 (8-bit x 8-bit significands).  The accumulator sums K of them in an order the tests do not assume; with adds that may
truncate, each add is off by less than 2^-23 of a partial sum that is at most sum_k |a_k b_k|, so

    |acc - sum_k a_k b_k| <= K 2^-23 sum_k |a_k b_k|          (K = V for a hidden half-step, H for a visible one).

The epilogue's own arithmetic adds the per-mode bounds of tests/test_tc_kernel_exact_gpu.py (scale, sigma and bias roundings,
the approximate sigmoid, the Box-Muller intrinsics).  A bf16 mean must be the rounding of some value within the bound of the
float64 reference, and at most one bf16 ulp from bf16(reference) (unless the bound itself is wider than that ulp: a Gaussian
mean near zero).  The bound is loose on purpose (wgmma's accumulation order and
rounding are not documented), so the fraction of means that differ from bf16(reference) at all is bounded separately.

Also here: the resident dataset and the epoch double buffer as inputs, chains cut into several launches, bit-identical
activations across the tile widths that promise them, and a read-only plan report (`CudaRBM.debug_tc_plan`) that makes each
case assert its own premise.  The benchmark-size cases are skipped on the host simulation; the 130-70 case runs there."""
import itertools

import numpy as np
import pytest

from boltzmann_machines import _native
from oracle import philox as P
from oracle.rbm import OracleRBM
from test_tc_kernel_exact_gpu import HOSTSIM, ULP, assert_bf16_within, bf16r, check_bernoulli, gaussian_noise, sigmoid_tol

pytestmark = pytest.mark.gpu
big = pytest.mark.skipif(HOSTSIM, reason='benchmark-size chain: hours on the interpreter')

ACC = 2.0 ** -23                 # one truncating fp32 add: less than 2^-23 of the partial sum
MAX_FLIP_ROWS = 0.01             # rows of a rebuilt hidden state that may need a flipped draw
MAX_OFF = 0.005                  # means that may differ from bf16(float64 reference)
PROGRAM_OPS = 90                 # ops per launch of a chain (csrc/bm_rbm_tc.cu)
REPORT = dict(draws=0, rebuilt=0, flips=0, flip_rows=0, flip_max_gap=0.0, means=0, off=0)


def _bench():
    """bench.py, imported on first use: its module constants read BM_BENCH_BATCHES at import, which a host test of bench.py sets
    for its own import"""
    import bench
    return bench


# ---- float64 statement of the two conditionals ---------------------------------------------------------------------------
def bits(a):
    """bf16 bit patterns of exported activations (widened bf16 values: the low 16 bits are zero)"""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    assert not (u & 0xFFFF).any(), 'exported activation is not a bf16 value'
    return (u >> 16).astype(np.uint16)


def bf16_ulp(x):
    return np.maximum(np.abs(x), 2.0 ** -126) * 2.0 ** -7


def rows_within(got, ref, tol):
    """per row: every element passes check_bf16"""
    lo, hi, near = bf16r(ref - tol), bf16r(ref + tol), bf16r(ref)
    ulp = bf16_ulp(near)
    return ((got >= lo) & (got <= hi) & ((np.abs(got - near) <= ulp) | (tol >= ulp))).all(axis=1)


class Conditionals(object):
    """float64 conditionals of the engine's model at one parameter state, with the per-element bound of the kernel's value"""

    def __init__(self, cfg, params):
        self.Wb = bf16r(np.asarray(params['W'], np.float32))          # the bf16 shadow of W
        self.absW = np.abs(self.Wb).astype(np.float32)
        self.vb = np.asarray(params['vb'], np.float32).astype(np.float64)
        self.hb = np.asarray(params['hb'], np.float32).astype(np.float64)
        self.mu = 2.0 if cfg.get('dbm_first') else 1.0
        self.md = 2.0 if cfg.get('dbm_last') else 1.0
        self.gauss = cfg.get('v_kind') == 'gaussian'
        V = self.Wb.shape[0]
        sig = np.broadcast_to(np.asarray(cfg['sigma'], np.float32), (V,)) if self.gauss else np.ones(V, np.float32)
        self.sigma = sig.astype(np.float64)
        self.sample_v, self.sample_h = bool(cfg.get('sample_v', False)), bool(cfg.get('sample_h', True))

    def up(self, v):
        """p(h | v) and its bound"""
        a = self.mu * (v @ self.Wb)
        b = self.mu * self.hb[None, :]
        e = self.mu * v.shape[1] * ACC * (np.abs(v).astype(np.float32) @ self.absW) + 4.0 * ULP * (np.abs(a) + np.abs(b))
        p = 1.0 / (1.0 + np.exp(-(a + b)))
        return p, sigmoid_tol(p, e)

    def down(self, h):
        """E[v | h] and its bound: sigmoid for binary visibles, m (h W^T) sigma + m vb for Gaussian ones"""
        scale = self.md * self.sigma[None, :]
        a = (h @ self.Wb.T) * scale
        b = self.md * self.vb[None, :]
        e = h.shape[1] * ACC * (np.abs(h).astype(np.float32) @ self.absW.T) * scale + 4.0 * ULP * (np.abs(a) + np.abs(b))
        if self.gauss:
            mean = a + b
            return mean, e + ULP * np.abs(mean)
        p = 1.0 / (1.0 + np.exp(-(a + b)))
        return p, sigmoid_tol(p, e)


def check_bf16(got, ref, tol, what):
    """assert_bf16_within (the rounding of a value within ref +- tol, at most one bf16 ulp from bf16(ref)), except where the
    bound itself is wider than one ulp of the result: there only the bound applies.  That happens to a Gaussian mean near a
    zero crossing, where m (h W^T) sigma and m vb cancel: the bound is absolute, the ulp of the result is not."""
    g = np.asarray(got, np.float64)
    wide = tol >= bf16_ulp(bf16r(ref))
    bad = wide & ~((g >= bf16r(ref - tol)) & (g <= bf16r(ref + tol)))
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError('{0}: {1} elements outside the rounding of ref +- tol, first at (m, n) = {2}: got {3!r}, ref {4!r}, '
                             'tol {5:.3g}'.format(what, int(bad.sum()), at, g[at], ref[at], tol[at]))
    assert_bf16_within(bits(got), np.where(wide, g, ref), np.where(wide, 0.0, tol), what)    # (wide elements: checked above)
    return int((g != bf16r(ref)).sum())


def check_means(got, ref, tol, what):
    off = check_bf16(got, ref, tol, what)
    REPORT['means'] += ref.size
    REPORT['off'] += off
    return off


def rebuild_hidden(cm, s, u, p, tol, got_v, what):
    """The hidden states the kernel drew: s = (u < p) row by row, or with one or two of the row's ambiguous draws flipped,
    whichever reproduces the next visible means `got_v`.  Returns (states, E[v | states], bound, rows that needed a flip)."""
    got_v = np.asarray(got_v, np.float64)
    ref, rtol = cm.down(s)
    ok = rows_within(got_v, ref, rtol)
    flipped = 0
    for r in np.flatnonzero(~ok):
        gap = np.abs(u[r] - p[r])
        cand = np.flatnonzero(gap <= tol[r])
        cand = cand[np.argsort(gap[cand], kind='stable')]
        tries = [(c,) for c in cand] + list(itertools.combinations(cand[:8], 2))
        hit = None
        if tries:
            S = np.repeat(s[r][None, :], len(tries), axis=0)
            for i, t in enumerate(tries):
                S[i, list(t)] = 1.0 - S[i, list(t)]
            R, T = cm.down(S)
            good = np.flatnonzero(rows_within(np.broadcast_to(got_v[r], R.shape), R, T))
            hit = int(good[0]) if good.size else None
        if hit is None:
            lo, hi, near = bf16r(ref[r] - rtol[r]), bf16r(ref[r] + rtol[r]), bf16r(ref[r])
            bad = np.flatnonzero((got_v[r] < lo) | (got_v[r] > hi) | (np.abs(got_v[r] - near) > np.abs(near) * 2.0 ** -7))
            c = int(bad[0])
            raise AssertionError('{0}: row {1} matches neither u < p nor any flip of its {2} ambiguous draws: {3} of {4} means '
                                 'off, first at column {5}: got {6!r}, ref {7!r}, tol {8:.3g}'.format(
                                     what, r, cand.size, bad.size, got_v.shape[1], c, got_v[r, c], ref[r, c], rtol[r, c]))
        s[r], ref[r], rtol[r] = S[hit], R[hit], T[hit]
        flipped += 1
        REPORT['flips'] += len(tries[hit])
        REPORT['flip_max_gap'] = max(REPORT['flip_max_gap'], float(gap[list(tries[hit])].max()))
    REPORT['flip_rows'] += flipped
    REPORT['rebuilt'] += s.shape[0]
    REPORT['draws'] += s.size
    return s, ref, rtol, flipped


# ---- the engine's runs ---------------------------------------------------------------------------------------------------
NAMES = ('X', 'h0_means', 'h0_states', 'v_means', 'v_states', 'h_means')


def activations(eng, rows):
    return {n: eng.get_activation(n, rows) for n in NAMES}


def check_update(g, cfg, init, A, lr, mom, what):
    """(c) the parameters `g` left by the step equal the oracle's formulas on the step's own activations"""
    ora = OracleRBM(cfg)
    ora.set_params(init)
    ora.apply_update(A['X'], A['h0_means'], A['v_states'], A['h_means'], lr, mom)
    w = ora.get_params()
    for n in ('dW', 'W', 'dvb', 'vb', 'dhb', 'hb', 'q_means'):
        scale = max(1e-6, float(np.abs(w[n]).max()))
        np.testing.assert_allclose(g[n], w[n], atol=2e-5 * scale + 1e-7, rtol=1e-5, err_msg='{0}: {1}'.format(what, n))


def replay_chain(eng, cfg, init, X, step, k_first, k_last, seed, tick, update=None):
    """Run CD-j for j = max(1, k_first - 1) .. k_last through `step(eng, j)` from the parameters `init` and check half-steps
    v_j | h_{j-1} and h_j | v_j of every j >= k_first (h_j | v_j also for the run before).  X: the batch as the engine must
    have prepared it (checked against the exported X).  update: (lr, mom) to check the parameter update of every run."""
    cm = Conditionals(cfg, init)
    B, V = X.shape
    H = cm.Wb.shape[1]
    first = prev = None
    flip_rows = rebuilt = 0
    means0, off0 = REPORT['means'], REPORT['off']
    for j in range(max(1, k_first - 1), k_last + 1):
        eng.set_params(init)
        step(eng, j)
        A = activations(eng, B)
        what = 'CD-{0}'.format(j)
        if first is None:
            np.testing.assert_array_equal(A['X'], X, err_msg='the batch the chain started from')
            p0, t0 = cm.up(np.asarray(X, np.float64))
            check_means(A['h0_means'], p0, t0, what + ': h0_means')
            if cm.sample_h:
                u0 = P.uniform_at(B, H, seed, P.SITE_H0, 0, tick).astype(np.float64)
                check_bernoulli(bits(A['h0_states']), u0, p0, t0, what + ': h0_states')
                REPORT['draws'] += u0.size
            else:
                np.testing.assert_array_equal(A['h0_states'], A['h0_means'])
            first = A
        else:
            for n in ('X', 'h0_means', 'h0_states'):     # the same prefix: bit for bit
                np.testing.assert_array_equal(A[n], first[n], err_msg='{0}: {1} differs from the first run'.format(what, n))
        if j >= k_first:
            # v_j | h_{j-1}
            if j == 1:
                s = A['h0_states'].astype(np.float64)
                ref, rtol = cm.down(s)
            elif cm.sample_h:
                _, ph, th = prev
                u = P.uniform_at(B, H, seed, P.SITE_H, j - 1, tick).astype(np.float64)
                s = (u < ph).astype(np.float64)
                s, ref, rtol, f = rebuild_hidden(cm, s, u, ph, th, A['v_means'], what + ': v_means')
                flip_rows += f
                rebuilt += B
            else:
                ref, rtol = cm.down(prev[0]['h_means'].astype(np.float64))
            check_means(A['v_means'], ref, rtol, what + ': v_means')
            if not cm.sample_v:
                np.testing.assert_array_equal(A['v_states'], A['v_means'], err_msg=what + ': v_states (sample_v off)')
            elif cm.gauss:
                g, dg = gaussian_noise(B, V, seed, P.SITE_V, j, tick, 0)
                st = ref + cm.sigma[None, :] * g
                check_bf16(A['v_states'], st, rtol + cm.sigma[None, :] * dg + 2.0 * ULP * np.abs(st), what + ': Gaussian v_states')
            else:
                uv = P.uniform_at(B, V, seed, P.SITE_V, j, tick).astype(np.float64)
                check_bernoulli(bits(A['v_states']), uv, ref, rtol, what + ': v_states')
                REPORT['draws'] += uv.size
        # h_j | v_j
        ph, th = cm.up(A['v_states'].astype(np.float64))
        check_means(A['h_means'], ph, th, what + ': h_means')
        if update is not None:
            check_update(eng.get_params(), cfg, init, A, update[0], update[1], what)
        prev = (A, ph, th)
    assert flip_rows <= MAX_FLIP_ROWS * max(rebuilt, 1), (flip_rows, rebuilt)
    means, off = REPORT['means'] - means0, REPORT['off'] - off0
    assert off <= MAX_OFF * means, 'means off bf16(ref): {0} of {1}'.format(off, means)
    return prev[0]


def params(V, H, w_std, seed, gauss=False):
    """every variable a step reads, so that set_params restores the whole state before each run"""
    rng = np.random.RandomState(seed)
    return dict(W=(w_std * rng.randn(V, H)).astype(np.float32), vb=((0.05 if gauss else 0.1) * rng.randn(V)).astype(np.float32),
                hb=(0.1 * rng.randn(H)).astype(np.float32), dW=(1e-3 * w_std * rng.randn(V, H)).astype(np.float32),
                dvb=(1e-3 * rng.randn(V)).astype(np.float32), dhb=(1e-3 * rng.randn(H)).astype(np.float32),
                q_means=rng.uniform(0.05, 0.2, H).astype(np.float32))


def data(kind, rows, V, seed):
    return _bench().synth_cifar(rows, n_vis=V, seed=seed) if kind == 'gaussian' else _bench().synth_mnist(rows, seed=seed, n_vis=V)


def train_step(X, lr, mom, seed, tick):
    return lambda eng, j: eng.train_step(X, lr, mom, j, seed, tick)


def chain_ops(plan, k):
    """the h0 op and the 2k half-steps (when the positive statistics run beside the chain, they sit right after h0)"""
    return [p for p in plan if p['mode'] != 'RAW_F32'][:1 + 2 * k]


def assert_granule_dataflow(ops, V, H):
    """every half-step whose K (the producer's width: H for a visible half-step, V for a hidden one) fits the granule-ordered
    K list of 32 chunks follows its producer granule by granule; h0 has no producer"""
    want = [False] + [(H if i % 2 else V) <= 32 * 64 for i in range(1, len(ops))]
    assert [p['follows_granules'] for p in ops] == want, ops


# ---- 1. chain replay at the benchmark's own shapes -----------------------------------------------------------------------
def bench_case(name, k, w_std=None, **over):
    """the benchmark's model config, shape, learning rate and W init scale (bench.RBM_WORKLOADS)"""
    kind, V, H, B, _, lr, std = _bench().RBM_WORKLOADS[name][:7]
    cfg = _bench().model_cfg('bf16', name)
    cfg.update(over)
    return dict(cfg=cfg, kind=kind, V=V, H=H, B=B, k=k, lr=lr, w_std=w_std or std)


def ragged_case(k=4, w_std=0.05, **over):
    cfg = dict(n_visible=781, n_hidden=1001, v_kind='bernoulli', h_kind='bernoulli', dtype='float32', compute='bf16', l2=1e-5,
               max_batch=4000, sample_v=True, sample_h=True, sparsity_target=0.1, sparsity_cost=0.01, sparsity_damping=0.9)
    cfg.update(over)
    return dict(cfg=cfg, kind='bernoulli', V=781, H=1001, B=4000, k=k, lr=0.05, w_std=w_std)


CASES = {
    'cfg2': lambda: bench_case('cfg2', _bench().K_GIBBS),
    'cfg2-w05': lambda: bench_case('cfg2', 3, w_std=0.05),
    'cfg5-shard-k25': lambda: bench_case('cfg5', 25),
    'cfg3-k3': lambda: bench_case('cfg3', 3),
    'cfg3-k3-sampled-v': lambda: bench_case('cfg3', 3, sample_v=True),
    'ragged-sampled-v': lambda: ragged_case(),
    'ragged-mean-h-dbm': lambda: ragged_case(sample_h=False, dbm_first=True, dbm_last=True, w_std=0.02),
    'ragged-dropout': lambda: ragged_case(dropout=0.8),
}


def run_case(c, seed=0x5EED, tick=4, mom=0.5):
    cfg, B, V, H = c['cfg'], c['B'], c['V'], c['H']
    init = params(V, H, c['w_std'], 11, c['kind'] == 'gaussian')
    X = data(c['kind'], B, V, 3)
    eng = _native.CudaRBM(cfg)
    Xp = OracleRBM(cfg).prepare_input(X, seed, tick)
    try:
        replay_chain(eng, cfg, init, Xp, train_step(X, c['lr'], mom, seed, tick), 1, c['k'], seed, tick, update=(c['lr'], mom))
        return eng.debug_tc_plan()
    finally:
        eng.close()


@big
@pytest.mark.parametrize('name', list(CASES))
def test_chain_replay(name):
    c = CASES[name]()
    plan = run_case(c)
    ops = chain_ops(plan, c['k'])
    assert len(ops) == 1 + 2 * c['k'] and all(p['launch'] == 0 for p in plan), plan
    assert_granule_dataflow(ops, c['V'], c['H'])
    if name == 'cfg2':
        assert all((p['bn'], p['pair_count']) == (256, 64) for p in ops), ops


def test_chain_replay_small():
    """130-70, batch 65, CD-3 with sampled visibles and wide weights (also on the host simulation)"""
    cfg = dict(n_visible=130, n_hidden=70, v_kind='bernoulli', h_kind='bernoulli', dtype='float32', compute='bf16', l2=1e-5,
               max_batch=65, sample_v=True, sample_h=True, sparsity_cost=0.01)
    plan = run_case(dict(cfg=cfg, kind='bernoulli', V=130, H=70, B=65, k=3, lr=0.05, w_std=0.05))
    assert len(chain_ops(plan, 3)) == 7


# ---- 2. input paths and batch cursors ------------------------------------------------------------------------------------
@big
def test_resident_dataset_at_an_unaligned_row():
    """set_data + train_step_at(1000, B): the replay starts from dataset rows [1000, 1000 + B), while the Philox rows stay
    batch-local (row0 = 0)"""
    c = bench_case('cfg2', 3)
    cfg, V, H, B = c['cfg'], c['V'], c['H'], c['B']
    first = 1000
    Xall = _bench().synth_mnist(first + B + 77, seed=21)
    init = params(V, H, c['w_std'], 12)
    seed, tick = 0xDA7A, 9
    eng = _native.CudaRBM(cfg)
    try:
        eng.set_data(Xall)
        step = lambda e, j: e.train_step_at(first, B, c['lr'], 0.5, j, seed, tick)
        replay_chain(eng, cfg, init, Xall[first:first + B], step, 1, 3, seed, tick, update=(c['lr'], 0.5))
    finally:
        eng.close()


@big
def test_epoch_double_buffer():
    """train_epoch over 4 batches of a byte-valued set (converted on the copy stream into the two halves of the epoch buffer):
    the last step reads the second half.  lr = mom = 0 leaves W bit-identical; the last batch's chain is replayed at tick0 + 3."""
    c = bench_case('cfg2', 3)
    cfg, V, H, B = c['cfg'], c['V'], c['H'], c['B']
    nb, seed, tick0 = 4, 0xE90C, 30
    X = _bench().synth_mnist(nb * B, seed=22)
    X[-B:] = _bench().synth_mnist(B, seed=23)           # (the generator tiles 8192 rows: make the last batch its own)
    init = params(V, H, c['w_std'], 13)
    eng = _native.CudaRBM(cfg)
    Xh = eng.pin(X)
    assert Xh.dtype == np.uint8
    try:
        def step(e, j):
            e.train_epoch(Xh, B, 0.0, 0.0, j, seed, tick0)
            np.testing.assert_array_equal(e.get_params(['W'])['W'], init['W'], err_msg='W after an epoch at lr = 0')
        replay_chain(eng, cfg, init, X[-B:], step, 1, 3, seed, tick0 + nb - 1)
    finally:
        eng.unpin(Xh)
        eng.close()


# ---- 3. chains cut across launches ---------------------------------------------------------------------------------------
@big
def test_chains_cut_across_launches():
    """cfg2 widths at batch 1024, k = 43 .. 46: 2k + 3 ops, so k = 43 fits one launch of 90 ops, and op 90 -- the first of the
    second launch -- is the dW op at k = 44, the last hidden half-step at k = 45 and a sampled mid-chain one at k = 46.  Steps
    43 to 46 are replayed, each from its predecessor."""
    c = bench_case('cfg2', 46)
    cfg, V, H = c['cfg'], c['V'], c['H']
    B, seed, tick = 1024, 0xC47, 2
    cfg['max_batch'] = B
    X = _bench().synth_mnist(B, seed=24)
    init = params(V, H, c['w_std'], 14)
    plans = {}
    eng = _native.CudaRBM(cfg)

    def step(e, j):
        e.train_step(X, c['lr'], 0.5, j, seed, tick)
        plans[j] = e.debug_tc_plan()
    try:
        replay_chain(eng, cfg, init, X, step, 43, 46, seed, tick, update=(c['lr'], 0.5))
    finally:
        eng.close()
    for k in range(43, 47):
        plan = plans[k]
        assert len(plan) == 2 * k + 3, (k, len(plan))
        assert [p['launch'] for p in plan] == [i // PROGRAM_OPS for i in range(2 * k + 3)], k
        if k > 43:
            head = plan[PROGRAM_OPS]              # the first op of the second launch waits for nothing inside it
            assert not head['follows_granules'], (k, head)
    assert plans[46][PROGRAM_OPS + 1]['follows_granules']        # ... and the op after it follows it granule by granule


# ---- 4. schedule invariance at the program level -------------------------------------------------------------------------
def run_once(cfg, init, X, k, seed, tick, lr=0.05, env=(), monkeypatch=None):
    """one CD-k step on a fresh engine (the chain's pair lanes are planned once per cached program) under `env`"""
    for n, v in env:
        monkeypatch.setenv(n, str(v))
    eng = _native.CudaRBM(cfg)
    try:
        eng.set_params(init)
        eng.train_step(X, lr, 0.5, k, seed, tick)
        return activations(eng, X.shape[0]), eng.get_params(), eng.debug_tc_plan()
    finally:
        eng.close()
        for n, _ in env:
            monkeypatch.delenv(n)


def assert_same_activations(A, R, what):
    for n in NAMES:
        got, want = bits(A[n]), bits(R[n])
        bad = got != want
        if bad.any():
            at = tuple(int(i) for i in np.argwhere(bad)[0])
            raise AssertionError('{0}: {1} differs in {2} elements, first at {3}: {4!r} vs {5!r}'.format(
                what, n, int(bad.sum()), at, A[n][at], R[n][at]))


@big
def test_tile_widths_128_and_256_give_identical_chains(monkeypatch):
    """A 256-wide producer is consumed in the K order of a 128-wide one, so forcing either width on either half-step changes
    no bit of any activation"""
    c = bench_case('cfg2', _bench().K_GIBBS)
    cfg, V, H, B, k = c['cfg'], c['V'], c['H'], c['B'], c['k']
    init = params(V, H, c['w_std'], 15)
    X = _bench().synth_mnist(B, seed=25)
    R, _, plan = run_once(cfg, init, X, k, 7, 3, monkeypatch=monkeypatch)
    ops = chain_ops(plan, k)
    assert all(p['bn'] == 256 for p in ops), ops
    assert_granule_dataflow(ops, V, H)
    for up, down in itertools.product((128, 256), (128, 256)):
        A, _, plan = run_once(cfg, init, X, k, 7, 3, env=(('BM_TC_BN_UP', up), ('BM_TC_BN_DOWN', down)), monkeypatch=monkeypatch)
        ops = chain_ops(plan, k)
        assert [p['bn'] for p in ops] == [up] + [down, up] * k, ops
        assert_granule_dataflow(ops, V, H)
        assert_same_activations(A, R, 'BN up {0}, down {1}'.format(up, down))


@big
def test_dw_overlap_changes_no_activation(monkeypatch):
    """cfg2 widths at batch 512 leave CTA pairs idle beside the chain: the positive statistics run there unless
    BM_TC_DW_OVERLAP=0.  Activations are bit-identical either way; the parameters differ only by the split-K order of dW."""
    c = bench_case('cfg2', _bench().K_GIBBS)
    cfg, V, H, k = c['cfg'], c['V'], c['H'], c['k']
    B = 512
    cfg['max_batch'] = B
    init = params(V, H, c['w_std'], 16)
    X = _bench().synth_mnist(B, seed=26)
    runs = {}
    for ov in (1, 0):
        A, prm, plan = run_once(cfg, init, X, k, 8, 5, env=(('BM_TC_DW_OVERLAP', ov),), monkeypatch=monkeypatch)
        chain_pairs = max(p['pair_count'] for p in chain_ops(plan, k))
        spare = [p for p in plan if p['mode'] == 'RAW_F32' and p['pair_begin'] >= chain_pairs]
        assert bool(spare) == bool(ov), (ov, plan)
        runs[ov] = A
        check_update(prm, cfg, init, A, c['lr'], 0.5, 'BM_TC_DW_OVERLAP={0}'.format(ov))
    assert_same_activations(runs[0], runs[1], 'dW beside the chain or after it')


@big
@pytest.mark.parametrize('up,down', [(192, 64), (64, 192)])
def test_widths_with_their_own_k_order(up, down, monkeypatch):
    """64- and 192-wide producers are consumed in their own K order (not bit-identical to the others): replayed"""
    c = bench_case('cfg2', 3)
    cfg, V, H, B = c['cfg'], c['V'], c['H'], c['B']
    init = params(V, H, c['w_std'], 17)
    X = _bench().synth_mnist(B, seed=27)
    seed, tick = 0x64, 6
    monkeypatch.setenv('BM_TC_BN_UP', str(up))
    monkeypatch.setenv('BM_TC_BN_DOWN', str(down))
    eng = _native.CudaRBM(cfg)
    try:
        replay_chain(eng, cfg, init, X, train_step(X, c['lr'], 0.5, seed, tick), 1, 3, seed, tick, update=(c['lr'], 0.5))
        ops = chain_ops(eng.debug_tc_plan(), 3)
    finally:
        eng.close()
    assert [p['bn'] for p in ops] == [up] + [down, up] * 3, ops
    assert_granule_dataflow(ops, V, H)


@big
def test_transform_runs_the_same_chain():
    """transform(X, k, seed, tick) runs the program without the dW ops: its hidden means are train_step's, bit for bit"""
    c = bench_case('cfg2', _bench().K_GIBBS)
    cfg, V, H, B, k = c['cfg'], c['V'], c['H'], c['B'], c['k']
    init = params(V, H, c['w_std'], 18)
    X = _bench().synth_mnist(B, seed=28)
    eng = _native.CudaRBM(cfg)
    try:
        eng.set_params(init)
        eng.train_step(X, c['lr'], 0.5, k, 31, 7)
        want = eng.get_activation('h_means', B)
        assert any(p['mode'] == 'RAW_F32' for p in eng.debug_tc_plan())
        eng.set_params(init)
        got = eng.transform(X, k, 31, 7)
        plan = eng.debug_tc_plan()
    finally:
        eng.close()
    assert len(plan) == 1 + 2 * k and not any(p['mode'] == 'RAW_F32' for p in plan), plan
    np.testing.assert_array_equal(bits(got), bits(want))


def test_report():
    """(runs last in this file) what the replays above checked"""
    print('\n[tc-chain] hidden draws checked: {0}, rebuilt rows needing a flip: {1} of {2} ({3} draws flipped, largest |u - p| '
          '{4:.3g}); means off bf16(ref): {5} of {6}'.format(
              REPORT['draws'], REPORT['flip_rows'], REPORT['rebuilt'], REPORT['flips'], REPORT['flip_max_gap'], REPORT['off'],
              REPORT['means']))
