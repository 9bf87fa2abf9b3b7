"""Parallel tempering on the H100 (csrc/bm_dbm_tc.cuh): one committed update -- a tempered sweep of every slot and a swap
round -- replayed in float64 from the particles before it, at the benchmark's shapes; the ladder [1.0] against the plain
step; slot 0 against exact enumeration; and a two-mode model that plain PCD cannot cross.

Replay of one update (k = 1).  Every final slot holds the swept state of its own slot or, where its pair was proposed and
accepted, of its neighbour.  For each candidate source s, each unit of the final state is checked against the float64
conditional sigmoid(b_s (pre + bias)) of the source's inputs (the layer below read from the final state itself, as the sweep
reads the new layer below) and the uniform the engine draws at row s M + p: state == (u < p), unless |u - p| is within the
bound of the fp32 accumulation of the bf16 operands (then the unit is ambiguous and either state is accepted).  The source
that explains a particle's state decides whether the pair was swapped; that outcome is then checked against the decision rule
on float64 energies, a decision within the energies' bound of its threshold counting as ambiguous.  The report counts both."""
import numpy as np
import pytest

from oracle import philox as P
from oracle.rbm import bf16_round

pytestmark = pytest.mark.gpu

SITE_DBM_PT = 14


def sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def cfg_of(V, Hs, M, **kw):
    L = len(Hs)
    c = dict(n_visible=V, n_hiddens=list(Hs), v_kind='bernoulli', h_kinds=['bernoulli'] * L, dtype='float32', compute='bf16',
             n_particles=M, batch_size=min(M, 256), max_mf_updates=3, mf_tol=1e-7, l2=0., max_norm=1e9, sample_v=True,
             sample_h=[True] * L, sparsity_target=[0.1] * L, sparsity_cost=[0.] * L, sparsity_damping=0.9)
    c.update(kw)
    return c


def params(V, Hs, scale, seed=0):
    rng = np.random.RandomState(seed)
    sizes = [V] + list(Hs)
    d = {'vb': (0.5 * rng.randn(V)).astype(np.float32)}
    for i in range(len(Hs)):
        s = '' if i == 0 else '_%d' % i
        d['W' + s] = (scale * rng.randn(sizes[i], sizes[i + 1])).astype(np.float32)
        d['hb' + s] = (0.5 * rng.randn(sizes[i + 1])).astype(np.float32)
    return d


def slots(g, L, T):
    """[(v, [h_0..]) per slot] from get_params"""
    sfx = lambda i: '' if i == 0 else '_%d' % i
    out = [(g['v'].astype(np.float64), [g['h' + sfx(i)].astype(np.float64) for i in range(L)])]
    for m in range(1, T):
        out.append((g['v_pt'][m - 1].astype(np.float64), [g['h_pt' + sfx(i)][m - 1].astype(np.float64) for i in range(L)]))
    return out


def make(V, Hs, M, betas, scale, seed=0):
    from boltzmann_machines import _native
    c = cfg_of(V, Hs, M)
    if betas is not None:
        c['pt_betas'] = betas
    e = _native.CudaDBM(c)
    d = params(V, Hs, scale, seed)
    e.set_params(d)
    e.init_particles(77)
    return e, d


def replay_update(V, Hs, M, betas, scale, warm=2, seed=1234, report=None):
    L, T = len(Hs), len(betas)
    e, d = make(V, Hs, M, betas, scale)
    X = (np.random.RandomState(3).rand(min(M, 256), V) < 0.3).astype(np.float32)
    for t in range(warm):                       # lr = 0: the update moves the particles only
        e.train_step(X, lr=0.0, momentum=0.0, k=1, seed=seed, tick=t)
    tick = warm
    before = slots(e.get_params(), L, T)
    acc0, _ = e.pt_counts()
    e.train_step(X, lr=0.0, momentum=0.0, k=1, seed=seed, tick=tick)
    after = slots(e.get_params(), L, T)
    acc1, _ = e.pt_counts()
    sfx = lambda i: '' if i == 0 else '_%d' % i
    Wb = [bf16_round(d['W' + sfx(i)]).astype(np.float64) for i in range(L)]
    hb = [d['hb' + sfx(i)].astype(np.float64) for i in range(L)]
    vb = d['vb'].astype(np.float64)
    eps = 2.0 ** -22

    def unexplained(s, fin):
        """per particle: units of final state `fin` that slot s's sweep cannot have produced; and the ambiguous ones"""
        v_in, H_in = before[s]
        b = betas[s]
        bad = np.zeros(M, np.int64)
        amb = np.zeros(M, np.int64)
        fv, fH = fin
        for i in range(L):
            below = v_in if i == 0 else fH[i - 1]
            pre = below @ Wb[i]
            mag = np.abs(below) @ np.abs(Wb[i])
            K = below.shape[1]
            if i + 1 < L:
                pre = pre + H_in[i + 1] @ Wb[i + 1].T
                mag = mag + np.abs(H_in[i + 1]) @ np.abs(Wb[i + 1]).T
                K += H_in[i + 1].shape[1]
            p = sig(b * (pre + hb[i]))
            u = P.uniform_at(M, Hs[i], seed, P.SITE_DBM_H + i, 1, tick, s * M).astype(np.float64)
            bound = 0.25 * b * (K * eps * mag + eps * np.abs(pre + hb[i])) + 1e-6
            wrong = fH[i] != (u < p)
            a = np.abs(u - p) <= bound
            bad += (wrong & ~a).sum(axis=1)
            amb += (wrong & a).sum(axis=1)
        pre = fH[0] @ Wb[0].T
        mag = np.abs(fH[0]) @ np.abs(Wb[0]).T
        p = sig(b * (pre + vb))
        u = P.uniform_at(M, V, seed, P.SITE_DBM_V, 1, tick, s * M).astype(np.float64)
        bound = 0.25 * b * (Hs[0] * eps * mag + eps * np.abs(pre + vb)) + 1e-6
        wrong = fv != (u < p)
        a = np.abs(u - p) <= bound
        bad += (wrong & ~a).sum(axis=1)
        amb += (wrong & a).sum(axis=1)
        return bad, amb

    def energy(x):
        v, H = x
        e_ = -(v @ vb)
        bnd = np.zeros(M)
        below = v
        for i in range(L):
            prod = below @ Wb[i] + hb[i]
            mag = np.abs(below) @ np.abs(Wb[i]) + np.abs(hb[i])
            e_ -= (H[i] * prod).sum(axis=1)
            bnd += (H[i] * (below.shape[1] * eps * mag)).sum(axis=1)
            below = H[i]
        return e_, bnd + 1e-9

    stats = dict(ambiguous_units=0, ambiguous_decisions=0, swaps=0, proposed=0)
    swapped = np.zeros((T - 1, M), bool)
    for m in range(tick % 2, T - 1, 2):
        keep_a, amb_a = unexplained(m, after[m])
        keep_b, amb_b = unexplained(m + 1, after[m + 1])
        sw_a, samb_a = unexplained(m + 1, after[m])
        sw_b, samb_b = unexplained(m, after[m + 1])
        keep = (keep_a == 0) & (keep_b == 0)
        swp = (sw_a == 0) & (sw_b == 0)
        assert np.all(keep | swp), 'pair %d: %d particles explained by neither outcome' % (m, int((~(keep | swp)).sum()))
        sw = swp & ~keep
        same = keep & swp                        # both slots ended in the same state: the outcome is not observable
        swapped[m] = sw
        stats['ambiguous_units'] += int(np.where(sw, samb_a + samb_b, amb_a + amb_b).sum())
        # the decision, on the states before the swap
        va = np.where(sw[:, None], after[m + 1][0], after[m][0])
        vb_ = np.where(sw[:, None], after[m][0], after[m + 1][0])
        Ha = [np.where(sw[:, None], after[m + 1][1][i], after[m][1][i]) for i in range(L)]
        Hb = [np.where(sw[:, None], after[m][1][i], after[m + 1][1][i]) for i in range(L)]
        Ea, ba = energy((va, Ha))
        Eb, bb = energy((vb_, Hb))
        u = P.uniform_at(M, 1, seed, SITE_DBM_PT, m, tick, 0)[:, 0].astype(np.float64)
        with np.errstate(divide='ignore'):
            lu = np.log(u)
        thr = (betas[m] - betas[m + 1]) * (Ea - Eb)
        near = np.abs(lu - thr) <= (betas[m] - betas[m + 1]) * (ba + bb)
        want = lu < thr
        assert np.all((want == sw) | near | same), 'pair %d: %d decisions disagree' % (m, int(((want != sw) & ~near & ~same).sum()))
        stats['unobservable'] = stats.get('unobservable', 0) + int(same.sum())
        stats['ambiguous_decisions'] += int(near.sum())
        stats['swaps'] += int(sw.sum())
        stats['proposed'] += M
    for m in range(T):                          # slots outside every proposed pair keep their own swept state
        if (m % 2 == tick % 2 and m + 1 < T) or (m >= 1 and (m - 1) % 2 == tick % 2):
            continue
        bad, amb = unexplained(m, after[m])
        assert np.all(bad == 0), 'slot %d: %d particles not explained' % (m, int((bad > 0).sum()))
        stats['ambiguous_units'] += int(amb.sum())
    assert stats['swaps'] <= int((acc1 - acc0).sum()) <= stats['swaps'] + stats.get('unobservable', 0)
    if report is not None:
        report.append(stats)
    print('PT replay V=%d Hs=%s M=%d T=%d: %s' % (V, Hs, M, T, stats))
    return stats


def test_replay_cfg4_shape_eight_temperatures():
    stats = replay_update(784, [512, 1024], 1024, [1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3], scale=0.05)
    assert stats['swaps'] > 0
    assert stats['ambiguous_decisions'] < 0.05 * stats['proposed']


def test_replay_cfg5_pcd_shape_four_temperatures():
    stats = replay_update(784, [4096], 4096, [1.0, 0.95, 0.9, 0.85], scale=0.01, warm=1)
    assert stats['swaps'] > 0


def test_replay_ragged_three_layers():
    stats = replay_update(100, [70, 45, 33], 300, [1.0, 0.75, 0.5, 0.3, 0.1], scale=0.3)
    assert stats['swaps'] > 0


def replay_last_sweep(V, Hs, M, betas, k, scale, tick, seed=4321):
    """Sweep k of a k-sweep update, replayed in float64: the update runs twice from the same state (val_metrics: no parameter
    update), once with k - 1 and once with k sweeps, same seed and tick.  The first k - 1 sweeps of both are the same chain,
    and both end with a swap round over the same pairs (the pairs follow the tick) with the same uniforms, so with A the
    particles after the (k-1)-sweep update, each proposed pair (m, m+1) of the k-sweep update is explained by two flags:
    whether the round after sweep k - 1 swapped it (sweep k of slot s then starts from A of the other slot) and whether the
    round after sweep k did (the final slot m then holds slot m+1's sweep).  Every unit of the final state is checked against
    u < p at row s M + p, t = k, and both decisions against the float64 energies."""
    L, T = len(Hs), len(betas)
    e, d = make(V, Hs, M, betas, scale)
    X = (np.random.RandomState(3).rand(min(M, 256), V) < 0.3).astype(np.float32)
    for t in range(2):
        e.val_metrics(X, k=1, seed=seed, tick=100 + t)
    start = e.get_params()
    e.val_metrics(X, k=k - 1, seed=seed, tick=tick)
    A = slots(e.get_params(), L, T)
    e.set_params(start)
    e.val_metrics(X, k=k, seed=seed, tick=tick)
    F = slots(e.get_params(), L, T)
    sfx = lambda i: '' if i == 0 else '_%d' % i
    Wb = [bf16_round(d['W' + sfx(i)]).astype(np.float64) for i in range(L)]
    hb = [d['hb' + sfx(i)].astype(np.float64) for i in range(L)]
    vb = d['vb'].astype(np.float64)
    eps = 2.0 ** -22
    memo = {}

    def mm(key, x, W):
        if key not in memo:
            memo[key] = (x @ W, np.abs(x) @ np.abs(W))
        return memo[key]

    draws = {}

    def u_at(site, n, s):
        if (site, s) not in draws:
            draws[(site, s)] = P.uniform_at(M, n, seed, site, k, tick, s * M).astype(np.float64)
        return draws[(site, s)]

    def unexplained(s, j, f):
        """units of final slot f that sweep k of slot s, started from A[j], cannot have produced (and the ambiguous ones)"""
        b = betas[s]
        fv, fH = F[f]
        bad = np.zeros(M, np.int64)
        amb = np.zeros(M, np.int64)
        def tally(state, pre, mag, K, site, n):
            p = sig(b * pre)
            u = u_at(site, n, s)
            bound = 0.25 * b * (K * eps * mag + eps * np.abs(pre)) + 1e-6
            wrong = state != (u < p)
            a = np.abs(u - p) <= bound
            return (wrong & ~a).sum(axis=1), (wrong & a).sum(axis=1)
        for i in range(L):
            pre, mag = mm(('A', j, 'v') if i == 0 else ('F', f, i - 1), A[j][0] if i == 0 else fH[i - 1], Wb[i])
            K = Wb[i].shape[0]
            if i + 1 < L:
                pa, ma = mm(('A', j, 'up', i + 1), A[j][1][i + 1], Wb[i + 1].T)
                pre, mag, K = pre + pa, mag + ma, K + Wb[i + 1].shape[1]
            x, y = tally(fH[i], pre + hb[i], mag, K, P.SITE_DBM_H + i, Hs[i])
            bad += x; amb += y
        pre, mag = mm(('F', f, 'down'), fH[0], Wb[0].T)
        x, y = tally(fv, pre + vb, mag, Hs[0], P.SITE_DBM_V, V)
        return bad + x, amb + y

    def energy(v, H):
        e_ = -(v @ vb)
        bnd = np.zeros(M)
        below = v
        for i in range(L):
            e_ -= (H[i] * (below @ Wb[i] + hb[i])).sum(axis=1)
            bnd += (H[i] * (below.shape[1] * eps * (np.abs(below) @ np.abs(Wb[i]) + np.abs(hb[i])))).sum(axis=1)
            below = H[i]
        return e_, bnd + 1e-9

    def pick(flag, x, y):
        return (np.where(flag[:, None], y[0], x[0]), [np.where(flag[:, None], b_, a_) for a_, b_ in zip(x[1], y[1])])

    def check_decision(m, flag, state_m, state_n, valid):
        """the swap round's decision for pair m on the states before it: flag == (log u < (b_m - b_n)(E_m - E_n)), for the
        particles whose outcome the replay determined (`valid`)"""
        Ea, ba = energy(*state_m)
        Eb, bb = energy(*state_n)
        u = P.uniform_at(M, 1, seed, SITE_DBM_PT, m, tick, 0)[:, 0].astype(np.float64)
        with np.errstate(divide='ignore'):
            lu = np.log(u)
        thr = (betas[m] - betas[m + 1]) * (Ea - Eb)
        near = (np.abs(lu - thr) <= (betas[m] - betas[m + 1]) * (ba + bb)) | ~valid
        assert np.all(((lu < thr) == flag) | near), 'pair %d: %d decisions disagree' % (m, int((((lu < thr) != flag) & ~near).sum()))
        return int((near & valid).sum())

    stats = dict(k=k, ambiguous_units=0, ambiguous_decisions=0, several_explanations=0, swaps_before=0, swaps_last=0, proposed=0)
    paired = set()
    for m in range(tick % 2, T - 1, 2):
        n = m + 1
        paired |= {m, n}
        fits = {}
        for a in (0, 1):                        # a: the round after sweep k - 1 swapped the pair
            for c in (0, 1):                    # c: the round after sweep k did
                src_m, src_n = (n, m) if c else (m, n)                    # whose sweep each final slot holds
                inp = lambda s: (n if s == m else m) if a else s           # the A slot that sweep starts from
                bm_, am_ = unexplained(src_m, inp(src_m), m)
                bn_, an_ = unexplained(src_n, inp(src_n), n)
                fits[(a, c)] = ((bm_ == 0) & (bn_ == 0), am_ + an_)
        ok = np.stack([fits[h][0] for h in sorted(fits)])
        assert np.all(ok.any(axis=0)), 'pair %d: %d particles explained by no hypothesis' % (m, int((~ok.any(axis=0)).sum()))
        stats['several_explanations'] += int((ok.sum(axis=0) > 1).sum())
        first = np.argmax(ok, axis=0)                                     # the first hypothesis that explains the particle
        hyp = sorted(fits)
        a = np.array([hyp[h][0] for h in first], bool)
        c = np.array([hyp[h][1] for h in first], bool)
        stats['ambiguous_units'] += int(sum(fits[hyp[h]][1][p] for p, h in enumerate(first)))
        unique = ok.sum(axis=0) == 1
        # decision after sweep k - 1, on the states before that round (A with the swap undone)
        before_m, before_n = pick(a, A[m], A[n]), pick(a, A[n], A[m])
        stats['ambiguous_decisions'] += check_decision(m, a, before_m, before_n, unique)
        # decision after sweep k, on the swept states (F with the swap undone)
        swept_m, swept_n = pick(c, F[m], F[n]), pick(c, F[n], F[m])
        stats['ambiguous_decisions'] += check_decision(m, c, swept_m, swept_n, unique)
        stats['swaps_before'] += int(a.sum()); stats['swaps_last'] += int(c.sum()); stats['proposed'] += M
    for s in range(T):                          # slots outside every proposed pair: their own sweep from their own state
        if s in paired:
            continue
        bad, amb = unexplained(s, s, s)
        assert np.all(bad == 0), 'slot %d: %d particles not explained' % (s, int((bad > 0).sum()))
        stats['ambiguous_units'] += int(amb.sum())
    print('PT last-sweep replay V=%d Hs=%s M=%d T=%d: %s' % (V, Hs, M, T, stats))
    return stats


def test_replay_last_sweep_cfg5_pcd_shape_k25():
    """cfg5-pcd's chain: k = 25 sweeps of 4 slots are 200 ops in three launches (cuts after sweeps 11 and 22)"""
    stats = replay_last_sweep(784, [4096], 4096, [1.0, 0.95, 0.9, 0.85], k=25, scale=0.01, tick=2)
    assert stats['swaps_last'] > 0 and stats['swaps_before'] > 0
    assert stats['several_explanations'] < 0.001 * stats['proposed']


def test_replay_last_sweep_cfg4_shape_k4():
    """cfg4's shape at T = 8: 24 ops a sweep, k = 4 is 96 ops in two launches; an odd tick leaves slots 0 and 7 unpaired"""
    stats = replay_last_sweep(784, [512, 1024], 1024, [1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.3], k=4, scale=0.05, tick=3)
    assert stats['swaps_last'] > 0
    assert stats['several_explanations'] < 0.001 * stats['proposed']


def test_replay_ladder_longer_than_a_program():
    """46 slots of a one-layer model: a sweep of 92 ops is cut inside the sweep, and the slots share CTA pairs"""
    stats = replay_update(100, [64], 256, [float(b) for b in np.linspace(1.0, 0.0, 46)], scale=0.3)
    assert stats['swaps'] > 0


def test_single_temperature_is_the_plain_step_at_cfg4():
    a, _ = make(784, [512, 1024], 1024, [1.0], scale=0.05)
    b, _ = make(784, [512, 1024], 1024, None, scale=0.05)
    X = (np.random.RandomState(3).rand(256, 784) < 0.3).astype(np.float32)
    for t in range(3):
        for e in (a, b):
            e.train_step(X, lr=2e-3, momentum=0.9, k=1, seed=9, tick=t)
    ga, gb = a.get_params(), b.get_params()
    for k in ga:
        np.testing.assert_array_equal(ga[k], gb[k], err_msg=k)


def exact_v(W, hb, vb):
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from dbm_pt_oracle import exact_log_marginal_v
    return exact_log_marginal_v(W, hb, vb)


def test_slot0_matches_enumeration_with_65536_particles():
    V, Hs, M = 6, [4], 65536
    betas = [1.0, 0.7, 0.45, 0.2]
    e, d = make(V, Hs, M, betas, scale=1.0)
    X = np.zeros((256, V), np.float32)
    for t in range(60):
        e.train_step(X, lr=0.0, momentum=0.0, k=1, seed=21, tick=t)
    v = e.get_params(['v'])['v']
    _, logp = exact_v([bf16_round(d['W']).astype(np.float64)], [d['hb']], d['vb'])
    counts = np.bincount((v @ (2 ** np.arange(V))).astype(np.int64), minlength=2 ** V)
    ex = M * np.exp(logp)
    keep = ex >= 5
    chi2 = float(((counts[keep] - ex[keep]) ** 2 / ex[keep]).sum() / max(keep.sum() - 1, 1))
    print('slot 0 vs enumeration: chi2/dof = %.3f over %d bins' % (chi2, int(keep.sum())))
    assert chi2 < 2.0


MIX_BETAS = [1.0, 0.8, 0.64, 0.5, 0.38, 0.28, 0.2, 0.13, 0.07, 0.0]


def two_mode(betas):
    """p(v) ~ exp(-3 n) (1 + exp(6 n - 48)), n = number of units on: modes at n = 0 and n = 16 of equal mass"""
    from boltzmann_machines import _native
    V, M = 16, 2048
    c = cfg_of(V, [1], M, batch_size=64)
    if betas is not None:
        c['pt_betas'] = betas
    e = _native.CudaDBM(c)
    d = {'W': np.full((V, 1), 6.0, np.float32), 'hb': np.array([-48.0], np.float32), 'vb': np.full(V, -3.0, np.float32)}
    e.set_params(d)
    z = {'v': np.zeros((M, V), np.float32), 'h': np.zeros((M, 1), np.float32)}
    if betas is not None and len(betas) > 1:
        z['v_pt'] = np.zeros((len(betas) - 1, M, V), np.float32)
        z['h_pt'] = np.zeros((len(betas) - 1, M, 1), np.float32)
    e.set_params(z)                              # every chain starts in the n = 0 mode
    X = np.zeros((64, V), np.float32)
    for t in range(400):
        e.train_step(X, lr=0.0, momentum=0.0, k=1, seed=31, tick=t)
    v = e.get_params(['v'])['v']
    return float((v.sum(axis=1) >= 8).mean()), e


def test_tempering_crosses_between_modes():
    W, hb, vb = [np.full((16, 1), 6.0)], [np.array([-48.0])], np.full(16, -3.0)
    allv, logp = exact_v(W, hb, vb)
    exact = float(np.exp(logp)[allv.sum(axis=1) >= 8].sum())
    with_pt, e = two_mode(MIX_BETAS)
    without, _ = two_mode(None)
    acc, prop = e.pt_counts()
    rates = acc / np.maximum(prop, 1)
    print('two-mode model: exact mass of the upper mode %.4f; slot 0 with PT %.4f, without %.4f; swap rates %s'
          % (exact, with_pt, without, np.round(rates, 3).tolist()))
    assert abs(with_pt - exact) < 0.06
    assert without < 0.01
