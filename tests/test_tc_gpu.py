"""Tensor-core (wgmma) path: the raw GEMM in every operand layout, then the bf16 RBM engine
against the oracle that rounds at the same points (bf16 operands, fp32 accumulation)."""
import numpy as np
import pytest

from boltzmann_machines import _native
from oracle.rbm import OracleRBM, bf16_round

pytestmark = pytest.mark.gpu


def ref_gemm(A, B, a_t, b_t):
    A = bf16_round(A).astype(np.float64)
    B = bf16_round(B).astype(np.float64)
    A = A.T if a_t else A
    B = B.T if b_t else B
    return A @ B.T


SHAPES = [(128, 256, 64), (128, 64, 128), (300, 200, 100), (1000, 784, 520), (257, 1024, 784), (64, 16, 784)]


@pytest.mark.parametrize('a_t', [False, True])
@pytest.mark.parametrize('b_t', [False, True])
@pytest.mark.parametrize('M,N,K', SHAPES)
def test_raw_gemm_all_layouts(M, N, K, a_t, b_t):
    rng = np.random.RandomState(M + N + K)
    A = rng.randn(K, M) if a_t else rng.randn(M, K)
    B = rng.randn(K, N) if b_t else rng.randn(N, K)
    C = _native.debug_tc_gemm(A, B, a_t=a_t, b_t=b_t)
    want = ref_gemm(A, B, a_t, b_t)
    np.testing.assert_allclose(C, want, atol=2e-3 * np.sqrt(K), rtol=1e-3)


@pytest.mark.parametrize('cluster,bn', [(2, 128), (2, 256), (2, 64), (2, 208), (2, 32), (2, 224), (1, 112), (1, 256)])
@pytest.mark.parametrize('a_t', [False, True])
@pytest.mark.parametrize('b_t', [False, True])
def test_cta_pair_tiles(cluster, bn, a_t, b_t):
    """Forced tile widths (whole 64-column wgmma blocks plus a last block of 16 / 32 / 48 columns), with CTA pairs taking
    256-row groups or single CTAs taking 128-row blocks; ragged row-block pairs (M = 5 tiles -> the last pair has an empty
    peer), ragged column tiles, many K chunks."""
    if b_t and bn % 64:
        pytest.skip('MN-major B: a tile holds whole 64-column boxes')
    rng = np.random.RandomState(cluster * 1000 + bn)
    M, N, K = 600, 784, 840
    A = rng.randn(K, M) if a_t else rng.randn(M, K)
    B = rng.randn(K, N) if b_t else rng.randn(N, K)
    C = _native.debug_tc_gemm(A, B, a_t=a_t, b_t=b_t, force_bn=bn, force_cluster=cluster)
    np.testing.assert_allclose(C, ref_gemm(A, B, a_t, b_t), atol=2e-3 * np.sqrt(K), rtol=1e-3)


@pytest.mark.parametrize('splits', [1, 3, 5])
def test_two_pair_negated_split_k(splits):
    """The dW shape: C = A1^T-layout * B1 - A2 * B2 with both operands MN-major, split over K."""
    rng = np.random.RandomState(splits)
    M, N, K = 784, 1024, 320
    A1, B1 = rng.rand(K, M) < 0.2, rng.rand(K, N)
    A2, B2 = rng.rand(K, M), rng.rand(K, N)
    C = _native.debug_tc_gemm(A1, B1, a_t=True, b_t=True, A2=A2, B2=B2, neg2=True, splits=splits)
    want = ref_gemm(A1, B1, True, True) - ref_gemm(A2, B2, True, True)
    np.testing.assert_allclose(C, want, atol=5e-2, rtol=1e-3)


def test_two_pair_accumulate_mixed_layouts():
    """The DBM shape: v W0 + h2 W1^T into one accumulator (B MN-major, then B K-major)."""
    rng = np.random.RandomState(9)
    M, N, K1, K2 = 200, 512, 784, 1024
    A1, B1 = rng.rand(M, K1), 0.1 * rng.randn(K1, N)      # W0 stored [K1, N]
    A2, B2 = rng.rand(M, K2), 0.1 * rng.randn(N, K2)      # W1 stored [N, K2]
    ctx = _native.Context.default()
    # the hook shares orientations between pairs, so check the two orientations separately and summed on host
    C1 = _native.debug_tc_gemm(A1, B1, a_t=False, b_t=True)
    C2 = _native.debug_tc_gemm(A2, B2, a_t=False, b_t=False)
    want = ref_gemm(A1, B1, False, True) + ref_gemm(A2, B2, False, False)
    np.testing.assert_allclose(C1 + C2, want, atol=5e-2, rtol=1e-3)


# ------------------------------------------------------------------------------------------------
def make_cfg(kind, V, H, B, **kw):
    cfg = dict(n_visible=V, n_hidden=H, dtype='float32', compute='bf16', l2=1e-4, max_batch=B,
               sample_v=False, sample_h=True, sparsity_cost=0.01, sparsity_target=0.2)
    if kind == 'gaussian':
        cfg.update(v_kind='gaussian', h_kind='bernoulli', sigma=np.linspace(0.5, 1.5, V))
    elif kind == 'multinomial':
        cfg.update(v_kind='bernoulli', h_kind='multinomial', h_n_samples=20)
    elif kind == 'multinomial-v':
        cfg.update(v_kind='multinomial', h_kind='bernoulli', v_n_samples=30, sample_v=True)
    else:
        cfg.update(v_kind='bernoulli', h_kind='bernoulli')
    cfg.update(kw)
    return cfg


def make_pair(cfg, seed=0):
    rng = np.random.RandomState(seed)
    V, H = cfg['n_visible'], cfg['n_hidden']
    init = dict(W=(0.1 * rng.randn(V, H)).astype(np.float32), vb=(0.1 * rng.randn(V)).astype(np.float32),
                hb=(0.1 * rng.randn(H)).astype(np.float32))
    eng, ora = _native.CudaRBM(cfg), OracleRBM(cfg)
    eng.set_params(init), ora.set_params(init)
    return eng, ora


def data(cfg, B, seed=1):
    rng = np.random.RandomState(seed)
    if cfg['v_kind'] == 'gaussian':
        return rng.randn(B, cfg['n_visible']).astype(np.float32)
    return (rng.rand(B, cfg['n_visible']) < 0.3).astype(np.float32)


def close_bf16(got, want, name, frac=2e-3):
    """bf16-stored quantities: equal up to one bf16 ulp, and almost everywhere exactly equal."""
    np.testing.assert_allclose(got, want, rtol=2.0 ** -7, atol=1e-6, err_msg=name)
    assert np.mean(got != want) <= 0.05, name


@pytest.mark.parametrize('kind', ['bernoulli', 'gaussian'])
@pytest.mark.parametrize('V,H,B', [(784, 16, 32), (130, 70, 65), (784, 1024, 256)])
def test_bf16_cd1_matches_rounding_oracle(kind, V, H, B):
    cfg = make_cfg(kind, V, H, B, dropout=0.9)
    eng, ora = make_pair(cfg)
    X = data(cfg, B)
    seed, tick = 0xABCDEF, 2
    Xp = ora.prepare_input(X, seed, tick)
    h0_means, v_states, v_means, _, h_means = ora.chain(Xp, 1, seed, tick)
    eng.train_step(X, 0.05, 0.5, 1, seed, tick)
    close_bf16(eng.get_activation('X', B), Xp, 'X')
    close_bf16(eng.get_activation('h0_means', B), h0_means, 'h0_means')
    # a Bernoulli draw may differ only where u is within rounding of p
    bad = np.mean(eng.get_activation('v_means', B) != v_means)
    assert bad < 0.2, bad
    np.testing.assert_allclose(eng.get_activation('v_means', B), v_means, atol=2e-2, rtol=2e-2)
    np.testing.assert_allclose(eng.get_activation('h_means', B), h_means, atol=2e-2)
    ora.train_step(X, 0.05, 0.5, 1, seed, tick)
    g, w = eng.get_params(), ora.get_params()
    for k in ('W', 'vb', 'hb', 'dW', 'dvb', 'dhb', 'q_means'):
        np.testing.assert_allclose(g[k], w[k], atol=2e-3, err_msg=k)
    eng.close()


def test_bf16_sampled_states_are_exactly_the_philox_draw():
    """Given the engine's own h0_means, its h0_states must be exactly (u < p) of the shared stream."""
    from oracle import philox as P
    cfg = make_cfg('bernoulli', 784, 1024, 128)
    eng, _ = make_pair(cfg)
    X = data(cfg, 128)
    eng.train_step(X, 0.05, 0.5, 1, 555, 7)
    p = eng.get_activation('h0_means', 128)
    s = eng.get_activation('h0_states', 128)
    u = P.uniform_at(128, 1024, 555, P.SITE_H0, 0, 7)
    # p was rounded to bf16 after the comparison, so only draws within one bf16 ulp of p may disagree
    disagree = (s != (u < p))
    assert np.all(np.abs(u - p)[disagree] <= 2.0 ** -8 * np.maximum(p[disagree], 1e-3))
    assert disagree.mean() < 0.01
    assert set(np.unique(s)) <= {0.0, 1.0}
    eng.close()


def test_bf16_training_tracks_fp32_statistically():
    """20 CD-1 steps on the same data: bf16 tensor-core engine vs fp32 CUDA-core engine end near each
    other (same RNG stream; flips only at rounding level)."""
    V, H, B = 784, 256, 512
    rng = np.random.RandomState(3)
    proto = (rng.rand(8, V) < 0.2)
    engines = []
    for compute in ('fp32', 'bf16'):
        cfg = make_cfg('bernoulli', V, H, B, compute=compute, sparsity_cost=0.0)
        eng = _native.CudaRBM(cfg)
        eng.set_params(dict(W=(0.01 * np.random.RandomState(0).randn(V, H)).astype(np.float32)))
        engines.append(eng)
    for it in range(20):
        idx = rng.randint(0, 8, size=B)
        flip = rng.rand(B, V) < 0.02
        X = np.logical_xor(proto[idx], flip).astype(np.float32)
        for eng in engines:
            eng.train_step(X, 0.05, 0.5, 1, 99, it)
    Wa, Wb = engines[0].get_params(['W'])['W'], engines[1].get_params(['W'])['W']
    rel = np.linalg.norm(Wa - Wb) / np.linalg.norm(Wa)
    assert rel < 0.05, rel
    m = engines[1].metrics(X, 1, 5, 0, ('msre', 'pll', 'free_energy'))
    m0 = engines[0].metrics(X, 1, 5, 0, ('msre', 'pll', 'free_energy'))
    assert abs(m['pll'] - m0['pll']) < 0.5          # BASELINE.json: PLL within 0.5 nats
    assert m['msre'] == pytest.approx(m0['msre'], rel=0.05)
    for e in engines:
        e.close()


@pytest.mark.parametrize('kind', ['multinomial', 'multinomial-v'])
@pytest.mark.parametrize('V,H,B,k', [(130, 70, 65, 1), (784, 256, 128, 2), (37, 29, 19, 3)])
def test_multinomial_layers_on_the_tensor_cores_match_the_rounding_oracle(kind, V, H, B, k):
    """layers.py:54-70 with the GEMMs on the tensor cores (raw fp32 pre-activations -> row softmax -> categorical draws on the unrounded
    means -> bf16 operands of the next GEMM), against the oracle that rounds at the same points: activations to a bf16 ulp,
    counts from the shared Philox stream, the whole update."""
    cfg = make_cfg(kind, V, H, B)
    eng, ora = make_pair(cfg)
    assert eng.compute == 'bf16'
    X = data(cfg, B) if kind == 'multinomial' else np.random.RandomState(2).multinomial(30, np.ones(V) / V, size=B).astype(np.float32)
    seed, tick = 0xBEEF, 4
    Xp = ora.prepare_input(X, seed, tick)
    h0_means, v_states, v_means, _, h_means = ora.chain(Xp, k, seed, tick)
    eng.train_step(X, 0.05, 0.5, k, seed, tick)
    np.testing.assert_allclose(eng.get_activation('h0_means', B), h0_means, rtol=2.0 ** -6, atol=2e-3, err_msg='h0_means')
    if k == 1:
        # (one categorical draw landing in a neighbouring bin moves two counts by one)
        assert np.mean(eng.get_activation('v_states', B) != v_states) < 0.02
        np.testing.assert_allclose(eng.get_activation('h_means', B), h_means, rtol=0.05, atol=0.05)
    ora.train_step(X, 0.05, 0.5, k, seed, tick)
    g, w = eng.get_params(), ora.get_params()
    tol = 3e-3 + 0.06 * (30 if kind == 'multinomial-v' else 20) / 20 / B
    for name in ('W', 'vb', 'hb', 'dW', 'dvb', 'dhb', 'q_means'):
        np.testing.assert_allclose(g[name], w[name], atol=tol * max(1.0, float(np.abs(w[name]).max())), err_msg=name)
    np.testing.assert_allclose(eng.transform(X, k, 5, 9), ora.transform(X, k, 5, 9), rtol=0.05, atol=0.05)
    eng.close()


def test_chains_longer_than_one_program_run_as_consecutive_launches():
    """CD-50 (103 ops, a program holds 96; the reference's chain has no limit, base_rbm.py:386-405) against the rounding oracle:
    same draws (one Philox stream whatever the cut), same update."""
    cfg = make_cfg('bernoulli', 130, 70, 65)
    eng, ora = make_pair(cfg)
    X = data(cfg, 65)
    l0 = _native.Context.default().launch_count()
    eng.train_step(X, 0.05, 0.5, 50, 0xC0FFEE, 1)
    assert _native.Context.default().launch_count() - l0 >= 4            # input conversion, two program launches, the update
    ora.train_step(X, 0.05, 0.5, 50, 0xC0FFEE, 1)
    g, w = eng.get_params(), ora.get_params()
    for name in ('W', 'vb', 'hb', 'dW', 'dvb', 'dhb', 'q_means'):
        np.testing.assert_allclose(g[name], w[name], atol=3e-3 + 0.06 / 65, err_msg=name)
    eng.close()
