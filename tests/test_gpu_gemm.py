"""GPU: the wgmma + TMA contraction kernel (3xTF32 split) against a float64 numpy reference."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 128, 256), (256, 384, 512), (200, 130, 100), (1026, 1026, 96), (37, 5, 9)])
def test_gemm_nt_tf32x3(engine, M, N, K):
    rng = np.random.RandomState(M * 7 + N * 3 + K)
    A = rng.randn(M, K).astype(np.float32)
    B = (rng.randn(N, K) * rng.lognormal(0, 2, (N, 1))).astype(np.float32)      # rows of very different scale
    C = engine.debug_gemm_nt(A, B)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    scale = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T         # sum |a||b| bounds the rounding
    err = np.abs(C - ref) / np.maximum(scale, 1e-30)
    assert err.max() < 2e-6, err.max()            # fp32-faithful: ~2^-22 split error + fp32 accumulation
    # plain TF32 (10-bit mantissa) would sit at ~1e-3: make sure the split really is in effect
    assert np.median(err) < 5e-7


@pytest.mark.parametrize("M,K", [(128, 64), (300, 100), (1026, 512), (129, 33)])
def test_gemm_gram_mode_is_symmetric_and_exact_enough(engine, M, K):
    """A == B: only the tiles on or above the diagonal are computed, the rest are stored as their transposes."""
    rng = np.random.RandomState(M + K)
    A = (rng.randn(M, K) * rng.lognormal(0, 1, (M, 1))).astype(np.float32)
    C = engine.debug_gemm_nt(A, A)
    np.testing.assert_array_equal(C, C.T)
    ref = A.astype(np.float64) @ A.astype(np.float64).T
    scale = np.abs(A).astype(np.float64) @ np.abs(A).astype(np.float64).T
    err = np.abs(C - ref) / np.maximum(scale, 1e-30)
    off = err.copy(); np.fill_diagonal(off, 0.0)
    assert off.max() < 2e-6, off.max()
    # a Gram DIAGONAL sums only positive products, so the tensor cores' not-round-to-nearest accumulation (gemm_tc.cu header) drifts one way:
    # ~2^-25 per accumulation, 3 * K / 8 accumulations -- the reason callers bound every chain to TC_KCHUNK = 512 terms
    assert np.diag(err).max() < 2e-6 + 3.0 * K / 8 * 2.0 ** -23, np.diag(err).max()


def test_gemm_many_tiles_per_cta(engine):
    """More tiles than SMs: every persistent CTA walks several tiles through the smem ring."""
    rng = np.random.RandomState(5)
    A = rng.randn(2500, 96).astype(np.float32)
    B = rng.randn(1700, 96).astype(np.float32)                      # 20 x 14 = 280 tiles
    C = engine.debug_gemm_nt(A, B)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    scale = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T
    assert (np.abs(C - ref) / scale).max() < 2e-6
