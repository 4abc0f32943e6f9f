"""The contraction kernels against float64 numpy references: the wgmma + TMA kernel (3xTF32 split, gemm_tc.cu) with its split
and partial-sum helpers, and the FP64 tensor-core (DMMA) kernel (gemm_f64.cu).

The TF32 kernel runs in the geometries its callers launch (Ridge's fold Grams and CG product, LogisticRegression's two
products, the kernel SVMs' Gram), rebuilt here from the callers' own formulas, twice: with integer inputs whose every
product and partial sum is exact in float32 (the result must equal float64 bit for bit, whatever the summation order), and
with float inputs against the float64 rounding bound.  C starts as a signalling-NaN sentinel: every element outside a batch's
window must keep it, so a store outside the window fails."""
import numpy as np
import pytest

from spark_sklearn_b200.engine import EngineError

GS_ERR_ARG = -2
TC_KCHUNK, GRAD_KCHUNK, KCH = 512, 256, 2048   # common.cuh, logreg.cu and TronRounds: the callers' K-chunks
SNAN = np.uint32(0x7FA00000)                   # a signalling NaN: no arithmetic result has this bit pattern
TF32_VMAX, F64_VMAX = 15, 1023                 # integer ranges of the exact tests


def _r(x, m):
    return (x + m - 1) // m * m


def _sentinel(n):
    return np.full(n, SNAN, np.uint32).view(np.float32)


def _ints(vmax, dtype=np.float32):
    """integers in [-vmax, vmax], each row scaled by its own power of two; every row holds +-vmax once, so the scale is
    max|row| / vmax"""
    def draw(rng, rows, K):
        v = rng.randint(-vmax, vmax + 1, (rows, K)).astype(np.float64)
        v[np.arange(rows), rng.randint(0, K, rows)] = vmax * rng.choice([-1.0, 1.0], rows)
        return (v * 2.0 ** rng.randint(-6, 7, (rows, 1))).astype(dtype)
    return draw


def _floats(rng, rows, K):
    return (rng.randn(rows, K) * rng.lognormal(0, 1, (rows, 1))).astype(np.float32)


class Case:
    """One batched launch: A [rows_a][K], B [rows_b][K] (None: symmetric, A is both operands), batches [n][6] =
    a_row0, b_row0, k0, k1, c_offset, ldc, output C [c_elems]; n_sum > 0: the partial sum of the first n_sum blocks of per"""

    def __init__(self, A, B, batches, M, N, c_elems, symmetric=False, n_sum=0, per=0):
        self.A, self.B, self.M, self.N, self.c_elems = A, B, M, N, c_elems
        self.batches = np.asarray(batches, np.int64).reshape(-1, 6)
        self.symmetric, self.n_sum, self.per = symmetric, n_sum, per

    def window(self, off, ldc):
        return off + np.arange(self.M)[:, None] * ldc + np.arange(self.N)[None, :]

    def refs(self):
        """per batch: float64 product, sum |a||b| and chain length"""
        A = self.A.astype(np.float64)
        B = A if self.B is None else self.B.astype(np.float64)
        out = []
        for a0, b0, k0, k1, _, _ in self.batches:
            a, b = A[a0:a0 + self.M, k0:k1], B[b0:b0 + self.N, k0:k1]
            out.append((a @ b.T, np.abs(a) @ np.abs(b).T, int(k1 - k0)))
        return out

    def summed_refs(self):
        """the float64 partial sum over the windows that land in [0, n_sum * per), and which of its elements they cover"""
        ref, scale, covered = np.zeros(self.per), np.zeros(self.per), np.zeros(self.per, bool)
        for (_, _, _, _, off, ldc), (r, s, _) in zip(self.batches, self.refs()):
            if off < self.n_sum * self.per:
                idx = self.window(off % self.per, ldc)
                ref[idx] += r; scale[idx] += s; covered[idx] = True
        return ref, scale, covered

    def run(self, engine):
        """C from a sentinel-filled buffer, twice (bitwise identical); checks the guard bands, the bitwise symmetry of
        symmetric windows and the partial sum against float32(sum of float64(partials)) in chunk order.  -> (windows, C, S)"""
        outs = []
        for _ in range(2):
            r = engine.debug_gemm_tc(self.A, self.B, self.batches, self.M, self.N, _sentinel(self.c_elems), self.symmetric,
                                     self.n_sum, self.per)
            outs.append(r if self.n_sum else (r, None))
        (C, S), (C2, S2) = outs
        np.testing.assert_array_equal(C.view(np.uint32), C2.view(np.uint32))
        inside = np.zeros(self.c_elems, bool)
        for off, ldc in self.batches[:, 4:]:
            inside[self.window(off, ldc)] = True
        stray = np.flatnonzero(C.view(np.uint32)[~inside] != SNAN)
        assert stray.size == 0, "stores outside every window at %s" % np.flatnonzero(~inside)[stray[:8]]
        wins = [C[self.window(off, ldc)] for off, ldc in self.batches[:, 4:]]
        if self.symmetric:
            for w in wins:
                np.testing.assert_array_equal(w.view(np.uint32), w.T.view(np.uint32))
        if self.n_sum:
            np.testing.assert_array_equal(S.view(np.uint32), S2.view(np.uint32))
            _, _, covered = self.summed_refs()
            chk = np.zeros(self.per)
            with np.errstate(invalid="ignore"):                  # the sentinel outside the windows
                for c in range(self.n_sum):                      # chunk order, float64, one rounding at the end
                    chk += C[c * self.per:(c + 1) * self.per].astype(np.float64)
            np.testing.assert_array_equal(S[covered].view(np.uint32), chk.astype(np.float32)[covered].view(np.uint32))
        return wins, C, S


# ---- the callers' geometries, from the callers' formulas ----

def ridge_grams(draw, rng, d, lengths=(32, TC_KCHUNK, 96, 224)):
    """linear.cu: Z^T [Dp][ldz] (features + y + ones), one symmetric batch per fold chunk [poff[q], poff[q+1]), C = the
    chunk Grams [nq][Dp][Dp] at ldc = Dp"""
    D = d + 2
    Dp = _r(D, 32)
    poff = np.concatenate([[0], np.cumsum(lengths)])
    Z = draw(rng, Dp, int(poff[-1]))
    nq = len(lengths)
    return Case(Z, None, [[0, 0, poff[q], poff[q + 1], q * Dp * Dp, Dp] for q in range(nq)], D, D, nq * Dp * Dp, symmetric=True)


def ridge_cg(draw, rng, n_cand, d, groups=3):
    """linear.cu: Q = P A_g, P [nsys][dp] (n_cand rows per group), A_g [groups * dp][dp]; batch (kc, g) reads rows
    g * n_cand and g * dp, K-chunk kc of TC_KCHUNK, writes partial kc; the partials are summed when nkc > 1"""
    dp = _r(d, 32)
    nsys, nkc = groups * n_cand, (dp + TC_KCHUNK - 1) // TC_KCHUNK
    P, Ag = draw(rng, nsys, dp), draw(rng, groups * dp, dp)
    batches = [[g * n_cand, g * dp, kc * TC_KCHUNK, min(dp, (kc + 1) * TC_KCHUNK), kc * nsys * dp + g * n_cand * dp, dp]
               for kc in range(nkc) for g in range(groups)]
    return Case(P, Ag, batches, n_cand, dp, nkc * nsys * dp, n_sum=nkc if nkc > 1 else 0, per=nsys * dp)


def logreg_z(draw, rng, ncol, n, d):
    """logreg.cu: Z^T = W Xa^T, W [ncol][nvp], Xa [n][nvp], C [ncol][npad]"""
    nvp, npad = _r(d + 1, 32), _r(n, 32)
    return Case(draw(rng, ncol, nvp), draw(rng, n, nvp), [[0, 0, 0, nvp, 0, npad]], ncol, n, ncol * npad)


def logreg_grad(draw, rng, ncol, n, d):
    """logreg.cu: G = R Xa, R [ncol][npad], Xa^T [nvp][npad], K split into GRAD_KCHUNK chunks, partial q at q ncol nvp
    (ldc nvp, N = nv), then launch_sum_partials"""
    nv = d + 1
    nvp, npad = _r(nv, 32), _r(n, 32)
    nchunk = (npad + GRAD_KCHUNK - 1) // GRAD_KCHUNK
    batches = [[0, 0, q * GRAD_KCHUNK, min(npad, (q + 1) * GRAD_KCHUNK), q * ncol * nvp, nvp] for q in range(nchunk)]
    return Case(draw(rng, ncol, npad), draw(rng, nvp, npad), batches, ncol, nv, nchunk * ncol * nvp, n_sum=nchunk,
                per=ncol * nvp)


def svc_gram(draw, rng, n, d):
    """kernel_svm.cu (GS_GRAM_TENSOR): X [n][dpad], one symmetric batch, C [n][ld32]"""
    dpad, ld32 = _r(d, 32), _r(n, 4)
    return Case(draw(rng, n, dpad), None, [[0, 0, 0, dpad, 0, ld32]], n, n, n * ld32, symmetric=True)


CASES = {}
for _D in (127, 128, 129, 255, 256, 257):                          # D = d + 2 around one and two 128-row tiles
    CASES["ridge_gram_D%d" % _D] = (lambda D: lambda dr, rng: ridge_grams(dr, rng, D - 2))(_D)
for _nc in (1, 7, 130):
    for _dp in (32, 160, 544):                                     # 544: two K-chunks
        CASES["ridge_cg_%dx%d" % (_nc, _dp)] = (lambda nc, dp: lambda dr, rng: ridge_cg(dr, rng, nc, dp))(_nc, _dp)
CASES["logreg_z_10x300"] = lambda dr, rng: logreg_z(dr, rng, 10, 300, 40)
CASES["logreg_z_150x1100"] = lambda dr, rng: logreg_z(dr, rng, 150, 1100, 20)
CASES["logreg_grad_10x300"] = lambda dr, rng: logreg_grad(dr, rng, 10, 300, 40)
CASES["logreg_grad_150x1100"] = lambda dr, rng: logreg_grad(dr, rng, 150, 1100, 20)   # npad 1120: a ragged last chunk
CASES["svc_gram_129"] = lambda dr, rng: svc_gram(dr, rng, 129, 64)
CASES["svc_gram_1026"] = lambda dr, rng: svc_gram(dr, rng, 1026, 40)


def _seed(name):
    return sum(map(ord, name))


def _tf32_split_is_exact(X):
    hi = (X.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return np.array_equal(hi, X)


def _row_units(X, vmax):
    """the power-of-two scale of every row of an _ints draw"""
    s = np.abs(X.astype(np.float64)).max(1) / vmax
    assert np.array_equal(s, 2.0 ** np.round(np.log2(s)))
    return s


@pytest.mark.parametrize("name", list(CASES))
def test_exact_inputs_keep_every_float32_partial_sum_exact(name):
    """CPU: with the integer draws, lo = 0 after the TF32 split and every chain's sum |a||b| (in units of the two row scales)
    stays below 2^24, so every product and every partial sum in any order is a float32 value: the kernel's result must be
    bitwise the float64 product.  Also the float64 sum of the partials, which launch_sum_partials rounds once."""
    case = CASES[name](_ints(TF32_VMAX), np.random.RandomState(_seed(name)))
    B = case.A if case.B is None else case.B
    assert _tf32_split_is_exact(case.A) and _tf32_split_is_exact(B)
    ua, ub = _row_units(case.A, TF32_VMAX), _row_units(B, TF32_VMAX)
    units = np.zeros(case.per)
    for (a0, b0, k0, k1, off, ldc), (ref, scale, k) in zip(case.batches, case.refs()):
        assert k <= TC_KCHUNK
        u = np.outer(ua[a0:a0 + case.M], ub[b0:b0 + case.N])
        assert (scale / u).max() < 2.0 ** 24
        if case.n_sum:
            units[case.window(off % case.per, ldc)] = u                 # the same rows in every chunk
        # and float32 really reproduces the float64 result summed forwards and backwards (a few rows of the window)
        rows = np.unique([0, min(1, case.M - 1), case.M // 2, case.M - 1])
        prod = case.A[a0 + rows, k0:k1][:, None, :] * B[b0:b0 + case.N, k0:k1][None, :, :]
        for order in (slice(None), slice(None, None, -1)):
            np.testing.assert_array_equal(np.cumsum(prod[:, :, order], axis=2, dtype=np.float32)[:, :, -1], ref[rows])
    if case.n_sum:
        _, scale, covered = case.summed_refs()
        assert (scale[covered] / units[covered]).max() < 2.0 ** 24


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_tc_caller_geometry_exact(engine, name):
    """integer inputs: every window (and the partial sum) equals the float64 product bit for bit"""
    case = CASES[name](_ints(TF32_VMAX), np.random.RandomState(_seed(name)))
    wins, _, S = case.run(engine)
    for w, (ref, _, _) in zip(wins, case.refs()):
        np.testing.assert_array_equal(w.astype(np.float64), ref)
    if case.n_sum:
        ref, _, covered = case.summed_refs()
        np.testing.assert_array_equal(S[covered].astype(np.float64), ref[covered])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_tc_caller_geometry_vs_float64(engine, name):
    """float inputs with rows of different scale: 2e-6 sum|a||b| off a Gram diagonal, the drift bar on it"""
    case = CASES[name](_floats, np.random.RandomState(_seed(name) + 1))
    wins, _, S = case.run(engine)
    for w, (ref, scale, k) in zip(wins, case.refs()):
        err = np.abs(w - ref) / np.maximum(scale, 1e-30)
        if case.symmetric:
            assert np.diag(err).max() < 2e-6 + 3.0 * k / 8 * 2.0 ** -23, np.diag(err).max()
            np.fill_diagonal(err, 0.0)
        assert err.max() < 2e-6, err.max()
        assert np.median(err) < 5e-7                     # plain TF32 would sit at ~1e-3: the split is in effect
    if case.n_sum:
        ref, scale, covered = case.summed_refs()
        err = np.abs(S[covered] - ref[covered]) / np.maximum(scale[covered], 1e-30)
        assert err.max() < 2e-6, err.max()


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [False, True])
def test_tc_store_paths_agree(engine, symmetric):
    """float2 stores (even ldc, 16-byte aligned C), scalar stores (odd ldc) and scalar stores (C one float off): the same
    bits.  symmetric: the diagonal tiles and the mirror at ldc != N."""
    rng = np.random.RandomState(17)
    M = N = 200
    A = _floats(rng, 230, 96)
    B = None if symmetric else _floats(rng, 210, 96)
    got = []
    for off, ldc in [(0, 208), (0, 207), (1, 208)]:
        case = Case(A, B, [[3 if not symmetric else 0, 0 if symmetric else 7, 32, 96, off, ldc]], M, N, off + M * ldc + 5,
                    symmetric)
        wins, _, _ = case.run(engine)
        ref, scale, _ = case.refs()[0]
        err = np.abs(wins[0] - ref) / scale
        if symmetric:
            np.fill_diagonal(err, 0.0)
        assert err.max() < 2e-6
        got.append(wins[0].view(np.uint32))
    np.testing.assert_array_equal(got[0], got[1])
    np.testing.assert_array_equal(got[0], got[2])


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [False, True])
def test_tc_ring_across_batches_of_unequal_length(engine, symmetric):
    """64 batches of 1, 2, 3 and 16 k-blocks interleaved, more tiles than SMs: every persistent CTA's 3-stage ring runs
    across batches of unequal length, some shorter than the ring.  Each window must equal its batch launched alone, and the
    gaps between windows keep the sentinel."""
    rng = np.random.RandomState(23)
    M = N = 256
    nkb = [1, 2, 3, 16] * 16
    A = _floats(rng, M + 64, 5 * 32 + 16 * 32)
    B = None if symmetric else _floats(rng, N + 64, A.shape[1])
    batches = []
    for z, nk in enumerate(nkb):
        a0 = (8 * z) % 64
        k0 = (z % 5) * 32
        batches.append([a0, a0 if symmetric else (24 * z) % 64, k0, k0 + 32 * nk, z * (M * N + 32), N])
    case = Case(A, B, batches, M, N, len(nkb) * (M * N + 32), symmetric)
    wins, _, _ = case.run(engine)
    for z, (w, (ref, scale, _)) in enumerate(zip(wins, case.refs())):
        alone = engine.debug_gemm_tc(A, B, [batches[z][:4] + [0, N]], M, N, _sentinel(M * N), symmetric).reshape(M, N)
        np.testing.assert_array_equal(w.view(np.uint32), alone.view(np.uint32), err_msg="batch %d" % z)
        err = np.abs(w - ref) / scale
        if symmetric:
            np.fill_diagonal(err, 0.0)
        assert err.max() < 2e-6


def test_tc_args_keep_batches_in_bounds():
    """CPU: the geometry builders above keep every batch inside its operands and C (what the hook checks)"""
    for name, make in CASES.items():
        case = make(_floats, np.random.RandomState(0))
        rows_b = case.A.shape[0] if case.B is None else case.B.shape[0]
        for a0, b0, k0, k1, off, ldc in case.batches:
            assert k0 % 32 == 0 and (k1 - k0) % 32 == 0 and 0 <= k0 < k1 <= case.A.shape[1], name
            assert a0 + case.M <= case.A.shape[0] and b0 + case.N <= rows_b, name
            assert ldc >= case.N and off + (case.M - 1) * ldc + case.N <= case.c_elems, name


@pytest.mark.gpu
def test_tc_hook_refuses_every_out_of_bounds_geometry(engine):
    """each invalid argument is refused (GS_ERR_ARG) before anything runs, and the handle works afterwards"""
    rng = np.random.RandomState(3)
    A, B = _floats(rng, 40, 64), _floats(rng, 50, 64)
    M, N, ce = 30, 40, 30 * 40
    good = [0, 0, 0, 64, 0, N]
    bad = [
        (A, B, [0, 0, 16, 48, 0, N], M, N, ce, False, 0, 0),            # k0 not a multiple of 32
        (A, B, [0, 0, 0, 48, 0, N], M, N, ce, False, 0, 0),             # length not a multiple of 32
        (A, B, [0, 0, 32, 96, 0, N], M, N, ce, False, 0, 0),            # k1 > K
        (A, B, [0, 0, -32, 32, 0, N], M, N, ce, False, 0, 0),           # k0 < 0
        (A, B, [11, 0, 0, 64, 0, N], M, N, ce, False, 0, 0),            # a_row0 + M > rows_a
        (A, B, [-1, 0, 0, 64, 0, N], M, N, ce, False, 0, 0),            # a_row0 < 0
        (A, B, [0, 11, 0, 64, 0, N], M, N, ce, False, 0, 0),            # b_row0 + N > rows_b
        (A, B, [0, 0, 0, 64, 1, N], M, N, ce, False, 0, 0),             # window one past C
        (A, B, [0, 0, 0, 64, -1, N], M, N, ce, False, 0, 0),            # c_offset < 0
        (A, B, [0, 0, 0, 64, 0, N + 1], M, N, ce, False, 0, 0),         # ldc pushes the last row past C
        (A, B, [0, 0, 0, 64, 0, N - 1], M, N, ce, False, 0, 0),         # ldc < N
        (A, B, [good, [0, 0, 0, 64, ce - N, N]], M, N, ce, False, 0, 0),  # the second batch's window past C
        (A, None, good, M, N, ce, True, 0, 0),                          # symmetric with M != N
        (A, B, [0, 0, 0, 64, 0, M], M, M, M * M, True, 0, 0),           # symmetric with a B operand
        (A, B, good, M, N, ce, False, 2, ce // 2 + 1),                  # partial sum past C
    ]
    for i, (a, b, bt, m, n, c_elems, sym, n_sum, per) in enumerate(bad):
        with pytest.raises(EngineError) as e:
            engine.debug_gemm_tc(a, b, bt, m, n, _sentinel(c_elems), sym, n_sum, per)
        assert e.value.status == GS_ERR_ARG, i
    for kchunk in (0, -16, 8, 520):
        with pytest.raises(EngineError) as e:
            engine.debug_gemm_f64(A.astype(np.float64), B.astype(np.float64), kchunk)
        assert e.value.status == GS_ERR_ARG, kchunk
    case = Case(A, B, [good], M, N, ce)
    wins, _, _ = case.run(engine)
    ref, scale, _ = case.refs()[0]
    assert (np.abs(wins[0] - ref) / scale).max() < 2e-6
    C = engine.debug_gemm_f64(A.astype(np.float64), B.astype(np.float64), 32)
    np.testing.assert_allclose(C, A.astype(np.float64) @ B.astype(np.float64).T, rtol=0, atol=1e-9 * np.abs(C).max())


# ---- the public single-batch wrapper (one batch over the zero-padded K; B is A: symmetric) ----

@pytest.mark.gpu
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


@pytest.mark.gpu
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


@pytest.mark.gpu
def test_gemm_many_tiles_per_cta(engine):
    """More tiles than SMs: every persistent CTA walks several tiles through the smem ring."""
    rng = np.random.RandomState(5)
    A = rng.randn(2500, 96).astype(np.float32)
    B = rng.randn(1700, 96).astype(np.float32)                      # 20 x 14 = 280 tiles
    C = engine.debug_gemm_nt(A, B)
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    scale = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T
    assert (np.abs(C - ref) / scale).max() < 2e-6


# ---- the FP64 tensor-core kernel in TRON's geometries (linear_search.cu) ----

# name: M (fits x decision rows), N, K, kchunk.  M and N are not multiples of 64 (the hook pads them).
F64_CASES = {
    "tron_z": (70, 300, 96, 96),              # Z = V Xa^T: K = nvp in one chunk
    "tron_grad_4096": (70, 100, 4096, KCH),   # Gp = R Xat^T: K = npad split at KCH, a whole number of chunks
    "tron_grad_5000": (70, 100, 5000, KCH),   # 2048, 2048 and a ragged 904 (912 after padding K to 16)
}


@pytest.mark.parametrize("name", list(F64_CASES))
def test_f64_exact_inputs_fit_the_float64_mantissa(name):
    """CPU: the integer draws keep every partial sum of the exact FP64 tests below 2^53 units"""
    M, N, K, _ = F64_CASES[name]
    rng = np.random.RandomState(_seed(name))
    A, B = _ints(F64_VMAX, np.float64)(rng, M, K), _ints(F64_VMAX, np.float64)(rng, N, K)
    units = np.outer(_row_units(A, F64_VMAX), _row_units(B, F64_VMAX))
    assert ((np.abs(A) @ np.abs(B).T) / units).max() < 2.0 ** 53


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(F64_CASES))
def test_f64_tron_geometry_exact(engine, name):
    """integer inputs: every chunk and the in-place chunk sum are exact, so C is the float64 product bit for bit (a dropped,
    repeated or stale 16-wide k-step fails), twice the same"""
    M, N, K, kchunk = F64_CASES[name]
    rng = np.random.RandomState(_seed(name))
    A, B = _ints(F64_VMAX, np.float64)(rng, M, K), _ints(F64_VMAX, np.float64)(rng, N, K)
    C = engine.debug_gemm_f64(A, B, kchunk)
    np.testing.assert_array_equal(C, A @ B.T)
    np.testing.assert_array_equal(C.view(np.uint64), engine.debug_gemm_f64(A, B, kchunk).view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(F64_CASES))
def test_f64_tron_geometry_vs_float64(engine, name):
    """float inputs: within K eps64 sum|a||b| of the float64 product, the bound of a reordered float64 sum"""
    M, N, K, kchunk = F64_CASES[name]
    rng = np.random.RandomState(_seed(name) + 1)
    A = rng.standard_normal((M, K)) * rng.lognormal(0, 1, (M, 1))
    B = rng.standard_normal((N, K)) * rng.lognormal(0, 1, (N, 1))
    C = engine.debug_gemm_f64(A, B, kchunk)
    assert np.all(np.abs(C - A @ B.T) <= K * np.finfo(np.float64).eps * (np.abs(A) @ np.abs(B).T))
    np.testing.assert_array_equal(C.view(np.uint64), engine.debug_gemm_f64(A, B, kchunk).view(np.uint64))


@pytest.mark.gpu
def test_gemm_f64_matches_numpy(engine):
    rng = np.random.RandomState(0)
    for M, N, K in [(5, 7, 3), (70, 130, 257), (64, 300, 5000)]:          # the last one runs split-K (K > 1024)
        A, B = rng.standard_normal((M, K)), rng.standard_normal((N, K))
        got = engine.debug_gemm_f64(A, B)
        ref = A @ B.T
        bound = 2 * K * np.finfo(np.float64).eps * (np.abs(A) @ np.abs(B).T)   # float64 rounding of a K-term sum
        assert np.all(np.abs(got - ref) <= bound)
