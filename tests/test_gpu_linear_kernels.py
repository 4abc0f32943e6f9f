"""The Ridge / Lasso / ElasticNet fold-Gram pipeline (csrc/linear.cu), one stage at a time, against float64 references in numpy.

Every GPU test takes one stage's own inputs from the gs_debug_linear hook (Engine.debug_linear) and judges its output at that
stage's precision: the shifts, the tensor-core block Grams and their float64 sums, the centred systems (against the training
rows themselves, which is what measures folds whose mean lies far from the global one), the batched CG, the quadratic forms,
the scores (against scikit-learn's metrics on float64 predictions from the GPU's own coefficients), the R^2 edge rules and
the coordinate descent (against a float64 restatement of enet_cd_kernel).  The restatement and the score references are
checked against the oracle and scikit-learn on the CPU, so they can be trusted without a GPU."""
import numpy as np
import pytest
from sklearn.metrics import mean_squared_error, r2_score

gpu = pytest.mark.gpu
U64 = 2.0 ** -53                   # unit roundoff of float64
KCHUNK = 512                       # rows per tensor-core chunk (TC_KCHUNK): the accumulation chain inside the MMA accumulator
CG_TOL = 1e-6
SCORE_DEFAULT, NEG_MSE, NEG_RMSE = 0, 16, 17


# ------------------------------------------------------------------------------------------------ references ----------
def chunk_coef(nrows):
    """Per-row factor of the error bound of a tensor-core Gram entry, |G - Z^T Z| <= sum_r c_r |z_r| |z_r|^T: each product of
    the 3xTF32 split drops lo*lo' and rounds both lo parts to TF32 (3 * 2^-22 <= 2^-20), the chunk's fp32 accumulator may
    truncate at every one of its K additions (K * 2^-23), and z = x - m is rounded to float32 (2 * 2^-24)."""
    c = np.empty(nrows)
    for r0 in range(0, nrows, KCHUNK):
        k = min(KCHUNK, nrows - r0)
        c[r0:r0 + k] = 2.0 ** -20 + k * 2.0 ** -23 + 2.0 ** -23
    return c


def zloc(X, y, rows, m, sw=None):
    """[X - m | y - m_y | 1] of the rows of a block about its float32 mean m, rounded as build_zt_kernel rounds it (float64
    array of the float32 values); sw: the sqrt(w)-scaled copy"""
    Z = np.concatenate([X[rows] - m[:-1], (y[rows] - m[-1])[:, None], np.ones((len(rows), 1), np.float32)], 1).astype(np.float32)
    if sw is not None:
        Z = Z * np.sqrt(sw[rows].astype(np.float32))[:, None]
    return Z.astype(np.float64)


def lift(M, delta):
    """L^T M L with L = I + e_{D-1} delta^T: a Gram about the block mean moved to the common shift (delta = m_b - c, 0 in the
    last column)"""
    L = np.eye(M.shape[0])
    L[-1, :-1] = delta
    return L.T @ M @ L


def masks(n, splits):
    """uint64 [n][2] test / training masks of (train, test) index pairs"""
    te, tr = np.zeros((n, 2), np.uint64), np.zeros((n, 2), np.uint64)
    for k, (a, b) in enumerate(splits):
        bit = np.uint64(1) << np.uint64(k & 63)
        tr[a, k >> 6] |= bit
        te[b, k >> 6] |= bit
    return te, tr


def load(engine, X, y, fold_id=None, splits=None, sw=None, kind=SCORE_DEFAULT):
    if splits is None:
        engine.set_data(X, fold_id, int(fold_id.max()) + 1, y_target=y)
    else:
        engine.set_data(X, -np.ones(len(y), np.int8), len(splits), y_target=y)
        engine.set_splits(*masks(len(y), splits), len(splits))
    engine.set_sample_weight(sw)
    engine.set_scoring(kind)


def train_test(h, g, n):
    """caller rows of group g's training and test sets"""
    tb, trb = h["test_block"][g], h["train_block"][g]
    test = h["blocks"][tb] if tb >= 0 else np.zeros(0, int)
    if trb >= 0:
        return h["blocks"][trb], test
    return np.setdiff1d(np.arange(n), test), test


def score_ref(y, pred, kind):
    """the scorer of scikit-learn on float64 predictions"""
    if kind == NEG_MSE:
        return -mean_squared_error(y, pred)
    if kind == NEG_RMSE:
        return -np.sqrt(mean_squared_error(y, pred))
    return r2_score(y, pred) if len(y) >= 2 else np.nan


def intercept(means, shift, w):
    """intercept in the caller's coordinates: the training means are of X - c, y - c_y (as gs_ridge_refit assembles it)"""
    d = len(w)
    return (means[d] + np.float64(shift[d])) - (means[:d] + shift[:d].astype(np.float64)) @ w


def dp_ni(d):
    dp = (d + 31) // 32 * 32
    return 1 if dp <= 128 else 2 if dp <= 256 else 4 if dp <= 512 else 8


def cd_gram(A, b, ntr, yy, alpha_c, l1, tol_rel, max_iter, ni):
    """float64 restatement of enet_cd_kernel<ni> on one system: scikit-learn's cyclic coordinate descent (_cd_fast.pyx
    enet_coordinate_descent) in the Gram domain, q = rhs - A w, with the kernel's coordinate order, gap-safe screening and
    stopping rule.  -> (w, n_iter, gap, tol, checks [(sweep, gap)])"""
    A = np.asarray(A, np.float64)
    b = np.asarray(b, np.float64)
    d = len(b)
    alpha, beta, tol = alpha_c * l1 * ntr, alpha_c * (1.0 - l1) * ntr, tol_rel * yy
    q, w, excl = b.copy(), np.zeros(d), np.zeros(d, bool)
    order = [k for r in range(4 * ni) for lane in range(32) for k in [128 * (r >> 2) + 4 * lane + (r & 3)] if k < d]
    st = dict(gap=0.0)
    checks = []

    def converged(sweep):
        mx = np.abs(q - beta * w).max()
        wb, wq, l1n, l2, qq = w @ b, w @ q, np.abs(w).sum(), w @ w, q @ q
        rn2, ry = yy - wb - wq, yy - wb
        if alpha == 0.0:
            dn = qq
            gap = qq if beta == 0.0 else rn2 + 0.5 * beta * l2 - ry + qq / (2.0 * beta)
        else:
            dn = mx
            primal = 0.5 * (rn2 + beta * l2) + alpha * l1n
            scale = alpha / dn if dn > alpha else 1.0
            gap = primal - (-0.5 * scale * scale * (rn2 + beta * l2) + scale * ry)
        st["gap"] = gap
        checks.append((sweep, gap))
        if gap <= tol:
            return True
        if alpha > 0.0:
            thr, den = np.sqrt(2.0 * gap) / alpha, max(alpha, dn)
            with np.errstate(divide="ignore", invalid="ignore"):
                dk = (1.0 - np.abs((q - beta * w) / den)) / np.sqrt(np.diag(A) + beta)
            nw = ~excl & ~(dk <= thr)
            for k in order:
                if nw[k] and w[k] != 0.0:
                    q[:] += w[k] * A[k]
                    w[k] = 0.0
            excl[:] |= nw
        return False

    n_iter = 0
    if not converged(0):
        it = 0
        while it < max_iter:
            w_max = d_w_max = 0.0
            for j in range(d):
                if excl[j] or A[j, j] == 0.0:
                    continue
                wj = w[j]
                tmp = q[j] + wj * A[j, j]
                mag = max(abs(tmp) - alpha, 0.0) / (A[j, j] + beta)
                wn = mag if tmp > 0 else -mag if tmp < 0 else 0.0
                if wn != wj:
                    q += (wj - wn) * A[j]
                    w[j] = wn
                d_w_max, w_max = max(d_w_max, abs(wn - wj)), max(w_max, abs(wn))
            if (w_max == 0.0 or d_w_max / w_max <= tol_rel or it == max_iter - 1) and converged(it + 1):
                break
            it += 1
        n_iter = it + 1 if it < max_iter else max_iter
    return w, n_iter, st["gap"], tol, checks


# ------------------------------------------------------------------------------------------------ data -----------------
def regression(n, d, seed, noise=0.5):
    rng = np.random.RandomState(seed)
    X = rng.randn(n, d).astype(np.float32)
    y = (X @ rng.randn(d) / np.sqrt(d) + noise * rng.randn(n) + 2.0).astype(np.float32)
    return X, y


def offset_groups(ratio, n_groups=5, per=300, d=12, seed=0):
    """rows in n_groups groups, each with its own offset (ratio x the in-group spread) in every column and in y; the
    test fold of GroupKFold is one group"""
    rng = np.random.RandomState(seed)
    off = rng.randn(n_groups, d + 1) * ratio
    g = np.repeat(np.arange(n_groups), per)
    X = (off[g, :d] + rng.randn(len(g), d)).astype(np.float32)
    beta = rng.randn(d)
    y = ((X - off[g, :d]) @ beta + off[g, d] + 0.3 * rng.randn(len(g))).astype(np.float32)
    return X, y, g.astype(np.int8)


# ------------------------------------------------------------------------------------------------ stage checks ---------
def check_grams(h, X, y, sw=None):
    """shift, block means, block Grams, T and Tw against float64 references from the float32 data"""
    n, d = X.shape
    c = h["shift"]
    X64 = np.concatenate([X, y[:, None]], 1).astype(np.float64)
    if c.any():                                                        # fit_intercept: c = float32 of the float64 mean
        want = (X64.mean(0)).astype(np.float32)
        ulp = np.spacing(np.abs(want))
        assert (np.abs(c.astype(np.float64) - want) <= ulp).all()
        assert (c == want).mean() >= 0.99
    npl = len(h["blocks"])
    for b, rows in enumerate(h["blocks"]):
        if len(rows):
            m = X64[rows].mean(0)
            assert (np.abs(h["block_shift"][b] - m) <= np.spacing(np.abs(m.astype(np.float32)))).all(), b
            yb = y[rows].astype(np.float64)
            np.testing.assert_allclose(h["ystat"][b], [yb.mean(), ((yb - yb.mean()) ** 2).sum()], rtol=1e-12,
                                       atol=1e-12 * (yb ** 2).sum())
    copies = [(b, b, None) for b in range(npl)] + ([(npl + b, b, sw) for b in range(npl)] if h["weighted_copies"] else [])
    Tref, Twref = np.zeros_like(h["T"]), np.zeros_like(h["T"])
    worst = 0.0
    for gb, b, w in copies:
        rows, G = h["blocks"][b], h["G"][gb]
        m = h["block_shift"][b]
        delta = m.astype(np.float64) - c.astype(np.float64)
        Z = zloc(X, y, rows, m, w)
        ref = lift(Z.T @ Z, delta)
        cz = np.abs(Z) * np.sqrt(chunk_coef(len(rows)))[:, None]
        # the contraction error about the block mean, carried through |L|; plus the float64 rounding of the move to c
        bound = lift(cz.T @ cz, np.abs(delta)) + 8 * U64 * lift(np.abs(Z).T @ np.abs(Z), np.abs(delta)) + 1e-300
        r = np.abs(G - ref) / bound
        worst = max(worst, r.max())
        assert r.max() <= 1.0, (gb, r.max(), np.unravel_index(r.argmax(), r.shape))
        np.testing.assert_array_equal(G, G.T)
        if w is None:
            assert G[-1, -1] == len(rows)
            Tref += G
        else:
            Twref += G
    # T, Tw: float64 sums of the blocks (in block order), each addition rounded once
    absum = np.abs(h["G"][:npl]).sum(0)
    assert (np.abs(h["T"] - Tref) <= npl * U64 * absum).all()
    if h["weighted_copies"]:
        assert (np.abs(h["Tw"] - Twref) <= npl * U64 * np.abs(h["G"][npl:]).sum(0)).all()
    return worst


def check_systems(h, X, y, sw=None, fit_intercept=True):
    """A, rhs and the training means of every group against the training rows themselves, centred first in float64.  The bar
    is scikit-learn's own float32 path (centre, then a float32 product over K rows): 2^-24 K |Xc|^T |Xc|."""
    n, d = X.shape
    c = h["shift"].astype(np.float64)
    worst = 0.0
    for g in range(len(h["test_block"])):
        tr, _ = train_test(h, g, n)
        Xt, yt = X[tr].astype(np.float64), y[tr].astype(np.float64)
        wt = np.ones(len(tr)) if sw is None else sw[tr].astype(np.float32).astype(np.float64)
        if fit_intercept:
            xm, ym = (wt @ Xt) / wt.sum(), (wt @ yt) / wt.sum()
        else:
            xm, ym = np.zeros(d), 0.0
        s = np.sqrt(wt)[:, None]
        Xc, yc = (Xt - xm) * s, (yt - ym) * s[:, 0]
        A_ref, b_ref = Xc.T @ Xc, Xc.T @ yc
        K = len(tr)
        barA = 2.0 ** -24 * K * (np.abs(Xc).T @ np.abs(Xc)) + 1e-300
        barb = 2.0 ** -24 * K * (np.abs(Xc).T @ np.abs(yc)) + 1e-300
        rA, rb = np.abs(h["A"][g] - A_ref) / barA, np.abs(h["rhs"][g] - b_ref) / barb
        worst = max(worst, rA.max(), rb.max())
        assert rA.max() <= 1.0 and rb.max() <= 1.0, (g, rA.max(), rb.max())
        mg = h["means"][g]
        if fit_intercept:
            sx = (np.abs(Xt - c[:d]) * wt[:, None]).sum(0) / wt.sum()
            assert (np.abs(mg[:d] - (xm - c[:d])) <= 2.0 ** -14 * sx + 1e-12).all(), g
        if sw is None:
            assert mg[d + 1] == K
        yyc = (yc ** 2).sum()
        assert abs(mg[d + 2] - yyc) <= 2.0 ** -14 * (np.abs(yc) ** 2).sum() + 1e-300 + 2.0 ** -14 * yyc, g
    return worst


def check_scores(h, X, y, kind, fit_intercept=True):
    """test / training scores against scikit-learn's metrics on float64 predictions from the GPU's own coefficients and
    intercept.  What is left is the Gram algebra: RSS = v^T G v with v = [-w, 1, -b0] over the block Grams, whose error
    is the contraction bound of check_grams carried through |v| plus the float64 rounding of the D^2-term quadratic form."""
    n, d = X.shape
    D = d + 2
    c = h["shift"]
    X64, y64 = X.astype(np.float64), y.astype(np.float64)
    worst = 0.0
    for g in range(len(h["test_block"])):
        tr, te = train_test(h, g, n)
        mg = h["means"][g]
        for ci in range(h["coef"].shape[1]):
            w = h["coef"][g, ci].astype(np.float64)
            b0g = (mg[d] - mg[:d] @ w) if fit_intercept else 0.0
            b0 = intercept(mg, c, w) if fit_intercept else 0.0
            v = np.concatenate([-w, [1.0, -b0g]])
            for side, rows in ((0, te), (1, tr)):
                pred = X64[rows] @ w + b0
                ref = score_ref(y64[rows], pred, kind)
                got = h["scores"][g, ci, side]
                blocks = [h["test_block"][g]] if side == 0 else (
                    [h["train_block"][g]] if h["train_block"][g] >= 0 else range(len(h["blocks"])))
                e_rss = 0.0
                for b in blocks:
                    rb = h["blocks"][b]
                    m = h["block_shift"][b]
                    delta = m.astype(np.float64) - c.astype(np.float64)
                    u = np.abs(v).copy()
                    u[-1] += np.abs(delta) @ np.abs(v[:-1])
                    Z = zloc(X, y, rb, m)
                    e_rss += (chunk_coef(len(rb)) * (np.abs(Z) @ u) ** 2).sum()
                zg = np.concatenate([X64 - c[:d], (y64 - c[d])[:, None], np.ones((n, 1))], 1)
                e_rss += 4 * D * D * U64 * ((np.abs(zg) @ np.abs(v)) ** 2).sum()   # the training side subtracts from T
                m_rows = len(rows)
                rss = ((y64[rows] - pred) ** 2).sum()
                if kind == NEG_MSE:
                    bound = e_rss / m_rows
                elif kind == NEG_RMSE:
                    bound = e_rss / m_rows / max(np.sqrt(rss / m_rows), 1e-300)
                else:
                    tss = ((y64[rows] - y64[rows].mean()) ** 2).sum()
                    if m_rows < 2:
                        assert np.isnan(got)
                        continue
                    if tss == 0:
                        assert got == (1.0 if rss == 0 else 0.0)
                        continue
                    bound = e_rss / tss
                bound += 1e-12 * max(1.0, abs(ref))
                worst = max(worst, abs(got - ref) / bound)
                assert abs(got - ref) <= bound, (g, ci, side, got, ref, bound)
    return worst


# ------------------------------------------------------------------------------------------------ GPU tests ------------
@gpu
@pytest.mark.parametrize("d", [1, 29, 30, 31, 94, 126, 127, 128])
def test_grams_across_column_tiles(engine, d):
    """D = d + 2 across multiples of 32 and the 128-wide tile; folds of 511, 512, 513 and 1025 rows and a fold -1 block"""
    sizes = [511, 512, 513, 1025]
    n = sum(sizes) + 37
    X, y = regression(n, d, d)
    X[:, 0] += 100.0                                                   # one column far from zero: the shift matters
    fold_id = np.concatenate([np.full(s, k, np.int8) for k, s in enumerate(sizes)] + [-np.ones(37, np.int8)])
    fold_id = fold_id[np.random.RandomState(d).permutation(n)]
    load(engine, X, y, fold_id)
    h = engine.debug_linear([1.0, 10.0])
    assert [len(b) for b in h["blocks"]] == sizes + [37]
    check_grams(h, X, y)
    check_systems(h, X, y)
    check_scores(h, X, y, SCORE_DEFAULT)


@gpu
@pytest.mark.parametrize("refit", [False, True])
def test_grams_general_splits_weights_and_refit(engine, refit):
    from sklearn.model_selection import ShuffleSplit
    n, d = 1500, 40
    X, y = regression(n, d, 5)
    sw = np.random.RandomState(1).rand(n) * 3
    sw[::7] = 0.0
    splits = list(ShuffleSplit(4, test_size=0.3, random_state=0).split(X))
    load(engine, X, y, splits=splits, sw=sw)
    h = engine.debug_linear([0.1] if refit else [0.1, 3.0], refit=refit)
    assert h["weighted_copies"]
    check_grams(h, X, y, sw)
    check_systems(h, X, y, sw)
    if not refit:
        for kind in (SCORE_DEFAULT, NEG_MSE):
            engine.set_scoring(kind)
            check_scores(engine.debug_linear([0.1, 3.0]), X, y, kind)
    engine.set_sample_weight(None)


@gpu
@pytest.mark.parametrize("ratio", [1e1, 1e2, 1e3, 1e4])
def test_systems_and_scores_with_fold_local_offsets(engine, ratio):
    """every group (= GroupKFold test fold) has its own offset, ratio x its spread: the training statistics T - G_k and the
    test fold's RSS must be as accurate as centring first would make them"""
    X, y, g = offset_groups(ratio)
    for kind in (SCORE_DEFAULT, NEG_MSE, NEG_RMSE):
        load(engine, X, y, g, kind=kind)
        h = engine.debug_linear([1e-3, 1.0, 100.0])
        if kind == SCORE_DEFAULT:
            check_grams(h, X, y)
            check_systems(h, X, y)
        check_scores(h, X, y, kind)


@gpu
def test_scores_all_kinds_partition_and_general_weighted(engine):
    from sklearn.model_selection import KFold
    n, d = 900, 70                                                     # d > 64: two column tiles of the quadratic forms
    X, y = regression(n, d, 11)
    sw = np.random.RandomState(2).rand(n) + 0.2
    fold_id = np.zeros(n, np.int8)
    for k, (_, te) in enumerate(KFold(5, shuffle=True, random_state=0).split(X)):
        fold_id[te] = k
    splits = list(KFold(4, shuffle=True, random_state=1).split(X))
    for kind in (SCORE_DEFAULT, NEG_MSE, NEG_RMSE):
        for spl in (None, splits):
            load(engine, X, y, fold_id, splits=spl, sw=sw, kind=kind)
            check_scores(engine.debug_linear(np.logspace(-2, 2, 5)), X, y, kind)
    load(engine, X, y, fold_id)
    check_scores(engine.debug_linear([0.5], fit_intercept=False), X, y, SCORE_DEFAULT, fit_intercept=False)


@gpu
@pytest.mark.parametrize("d,n_cand", [(513, 1), (600, 63), (700, 64), (1100, 65), (800, 130)])
def test_cg_solutions_and_true_residual(engine, d, n_cand):
    """the batched CG (nkc = 2 and 3 K-chunks of the tensor-core product) against a float64 solve (by eigendecomposition) of
    the hook's own float32 system, alpha from 1e-6 to 1e6 of trace(A) / d"""
    from scipy import linalg
    n = 4 * d
    X, y = regression(n, d, d)
    load(engine, X, y, (np.arange(n) % 4).astype(np.int8))
    h0 = engine.debug_linear([1.0])
    scale = np.trace(h0["A"][0].astype(np.float64)) / d
    alphas = scale * np.logspace(-6, 6, n_cand) if n_cand > 1 else np.array([scale])
    h = engine.debug_linear(alphas)
    assert h["cg_iterations"] >= 1
    for g in range(len(h["test_block"])):
        A, b = h["A"][g].astype(np.float64), h["rhs"][g].astype(np.float64)
        ev, V = linalg.eigh(A)                                        # float64 solve of every (A + alpha I) w = b at once
        vb = V.T @ b
        for ci, a in enumerate(alphas):
            M = A + a * np.eye(d)
            w = h["coef"][g, ci].astype(np.float64)
            ref = V @ (vb / (ev + a))
            kappa = (ev[-1] + a) / (max(ev[0], 0.0) + a)
            # the stop is on the recursive residual (<= CG_TOL); the true one also carries the 3xTF32 product error and the
            # float32 rounding of x and r: 2^-20 ||M|| ||w|| / ||b|| with a factor 10 of room
            res_bound = 10 * CG_TOL + 10 * 2.0 ** -20 * (ev[-1] + a) * np.linalg.norm(w) / np.linalg.norm(b)
            res = np.linalg.norm(b - M @ w) / np.linalg.norm(b)
            assert res <= res_bound, (g, ci, res, res_bound)
            err = np.linalg.norm(w - ref) / np.linalg.norm(ref)
            assert err <= kappa * res_bound * 4, (g, ci, err, kappa)


@gpu
def test_cg_ill_conditioned_fails_loudly_or_is_right(engine):
    """near-collinear columns and alpha = 1e-6 trace(A) / d: CG either converges to a solution within the bound or the search
    fails with GS_ERR_NUMERIC; a wrong answer reported as success fails the test"""
    from scipy import linalg
    from spark_sklearn_b200.engine import EngineError
    n, d = 2100, 520
    X, y = regression(n, d, 3)
    X[:, 1::2] = X[:, 0::2][:, :d // 2] + 1e-3 * X[:, 1::2]
    load(engine, X, y, (np.arange(n) % 3).astype(np.int8))
    scale = np.trace(engine.debug_linear([1.0])["A"][0].astype(np.float64)) / d
    try:
        h = engine.debug_linear([1e-6 * scale])
    except EngineError as e:
        assert e.status == -5 and "did not converge" in str(e)
        return
    for g in range(3):
        A, b = h["A"][g].astype(np.float64), h["rhs"][g].astype(np.float64)
        M = A + 1e-6 * scale * np.eye(d)
        w = h["coef"][g, 0].astype(np.float64)
        res = np.linalg.norm(b - M @ w) / np.linalg.norm(b)
        ev = np.linalg.eigvalsh(M)
        assert res <= 10 * CG_TOL + 10 * 2.0 ** -20 * ev[-1] * np.linalg.norm(w) / np.linalg.norm(b)
        ref = linalg.solve(M, b, assume_a="pos")
        assert np.linalg.norm(w - ref) / np.linalg.norm(ref) <= 4 * ev[-1] / ev[0] * 20 * CG_TOL


@gpu
@pytest.mark.parametrize("d,n_cand", [(70, 3), (150, 65), (200, 130)])
def test_quadratic_forms(engine, d, n_cand):
    """qk = w^T G_k w and qt = w^T M w (M = T or the split's training Gram) against float64 from the hook's own G, T and w:
    several 64-wide column tiles and more than 64 candidates (two system tiles)"""
    from sklearn.model_selection import ShuffleSplit
    n = 3 * d + 100
    X, y = regression(n, d, d + 1)
    for spl in (None, list(ShuffleSplit(3, test_size=0.25, random_state=0).split(X))):
        load(engine, X, y, (np.arange(n) % 3).astype(np.int8), splits=spl)
        h = engine.debug_linear(np.logspace(-3, 3, n_cand))
        for g in range(len(h["test_block"])):
            tb, trb = h["test_block"][g], h["train_block"][g]
            Gk = h["G"][tb][:d, :d]
            M = (h["G"][trb] if trb >= 0 else h["T"])[:d, :d]
            for ci in range(n_cand):
                w = h["coef"][g, ci].astype(np.float64)
                aw = np.abs(w)
                for got, MM in ((h["qk"][g, ci], Gk), (h["qt"][g, ci], M)):
                    ref = w @ MM @ w
                    assert abs(got - ref) <= (2 * d + 16) * U64 * (aw @ np.abs(MM) @ aw) + 1e-300, (g, ci, got, ref)


@gpu
def test_r2_one_row_and_constant_test_folds(engine):
    """scikit-learn's r2_score edge rules: a one-row test set scores NaN, a constant-target test set 0.0 (not a perfect fit)"""
    n, d = 60, 4
    X, y = regression(n, d, 7)
    load(engine, X, y, np.arange(n).astype(np.int8))                  # LeaveOneOut = KFold(n) on the partition path
    h = engine.debug_linear([0.1, 1.0])
    assert np.isnan(h["scores"][:, :, 0]).all() and np.isfinite(h["scores"][:, :, 1]).all()
    check_scores(h, X, y, SCORE_DEFAULT)
    engine.set_scoring(NEG_MSE)
    assert np.isfinite(engine.debug_linear([0.1])["scores"]).all()
    # a general split whose test set is one row
    splits = [(np.arange(1, n), np.array([0])), (np.arange(30), np.arange(30, n))]
    load(engine, X, y, splits=splits)
    s = engine.debug_linear([0.1])["scores"]
    assert np.isnan(s[0, 0, 0]) and np.isfinite(s[1, 0, 0])
    # a fold whose target is constant: exactly 0.0 on the test side, on both paths
    yc = y.copy()
    fold_id = (np.arange(n) % 4).astype(np.int8)
    yc[fold_id == 2] = np.float32(3.25)
    for spl in (None, [(np.flatnonzero(fold_id != k), np.flatnonzero(fold_id == k)) for k in range(4)]):
        load(engine, X, yc, fold_id, splits=spl)
        h = engine.debug_linear([0.1, 10.0])
        assert (h["scores"][2, :, 0] == 0.0).all()
        check_scores(h, X, yc, SCORE_DEFAULT)


def _compare_cv_results(a, b, n_splits):
    for k in range(n_splits):
        for side in ("test", "train"):
            key = "split%d_%s_score" % (k, side)
            np.testing.assert_allclose(a.cv_results_[key], b.cv_results_[key], rtol=0, atol=5e-5, equal_nan=True, err_msg=key)
    for key in ("mean_test_score", "mean_train_score"):
        np.testing.assert_allclose(a.cv_results_[key], b.cv_results_[key], rtol=0, atol=5e-5, equal_nan=True, err_msg=key)


@gpu
@pytest.mark.parametrize("est", ["ridge", "lasso"])
def test_public_api_leave_one_out_and_constant_group(engine, est):
    import warnings
    from sklearn.linear_model import Lasso, Ridge
    from sklearn.model_selection import GridSearchCV as SkGrid, GroupKFold, LeaveOneOut
    from spark_sklearn_b200 import GridSearchCV
    n, d = 40, 5
    X, y = regression(n, d, 13)
    make = (lambda: Ridge()) if est == "ridge" else (lambda: Lasso(tol=1e-8, max_iter=5000))
    grid = {"alpha": [0.01, 0.1, 1.0]}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a = GridSearchCV(None, make(), grid, cv=LeaveOneOut(), return_train_score=True).fit(X, y)
        b = SkGrid(make(), grid, cv=LeaveOneOut(), return_train_score=True).fit(X, y)
    assert np.isnan(a.cv_results_["mean_test_score"]).all() and np.isnan(b.cv_results_["mean_test_score"]).all()
    _compare_cv_results(a, b, n)
    groups = np.arange(n) % 5
    yc = y.copy()
    yc[groups == 3] = np.float32(-1.5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a = GridSearchCV(None, make(), grid, cv=GroupKFold(5), return_train_score=True).fit(X, yc, groups=groups)
        b = SkGrid(make(), grid, cv=GroupKFold(5), return_train_score=True).fit(X, yc, groups=groups)
    _compare_cv_results(a, b, 5)
    assert a.best_index_ == b.best_index_
    k3 = [k for k, (_, te) in enumerate(GroupKFold(5).split(X, yc, groups)) if (groups[te] == 3).all()][0]
    assert (a.cv_results_["split%d_test_score" % k3] == 0.0).all()


@gpu
@pytest.mark.parametrize("d", [100, 150, 200, 400, 1000])
def test_coordinate_descent_against_gram_restatement(engine, d):
    """enet_cd_kernel<NI> (NI = 1, 2, 2, 4, 8 by d; 150 is the first d past the 128-wide instance) against cd_gram on the hook's own float32 A, rhs and means: l1_ratio 0
    (formulation B), 0.5 and 1, a zero column, a duplicated column, an alpha past alpha_max (w = 0, no sweep) and a
    max_iter stop.  w within 1e-10 of max |w| (the gap's warp-reduction order); n_iter and gap equal, or the gap test
    within 1e-9 of tol where they part"""
    n = 400
    X, y = regression(n, d, d + 3)
    X[:, 3] = 0.0
    X[:, 5] = X[:, 4]
    fold_id = (np.arange(n) % 4).astype(np.int8)
    load(engine, X, y, fold_id)
    amax = np.abs(X.T.astype(np.float64) @ (y - y.mean())).max() / n
    max_iter = 12 if d == 1000 else 200
    cands = [(1e3 * amax, 1.0), (0.05 * amax, 1.0), (0.05 * amax, 0.5), (0.5, 0.0), (0.002 * amax, 1.0)]
    alphas, l1 = [a for a, _ in cands], [r for _, r in cands]
    for mi in (max_iter, 3):
        h = engine.debug_linear(alphas, l1_ratio=l1, tol=1e-4, max_iter=mi)
        assert (h["n_iter"][:, 0] == 0).all() and (h["coef"][:, 0] == 0).all()
        for g in range(2):
            mg = h["means"][g]
            for ci, (a, r) in enumerate(cands):
                w, it, gap, tol, checks = cd_gram(h["A"][g], h["rhs"][g], mg[d + 1], mg[d + 2], a, r, 1e-4, mi, dp_ni(d))
                got_it, got_gap = h["n_iter"][g, ci], h["gap"][g, ci]
                if got_it != it:
                    stop = min(got_it, it)
                    near = [abs(gp - tol) <= 1e-9 * tol for s, gp in checks if s == stop]
                    assert near and all(near), (g, ci, got_it, it, checks)
                    continue
                scale = max(np.abs(w).max(), 1e-300)
                assert np.abs(h["coef"][g, ci] - w).max() <= 1e-10 * scale + 2.0 ** -24 * np.abs(w).max(), (g, ci)
                assert abs(got_gap - gap) <= 1e-9 * max(abs(gap), tol), (g, ci, got_gap, gap)
                if mi == 3 and ci == 4:
                    assert got_it == 3


# ------------------------------------------------------------------------------------------------ CPU checks of the references
def test_cd_gram_restatement_matches_oracle_x_domain():
    """cd_gram on the float64 Gram of a centred problem reproduces oracle.enet_cd (scikit-learn's X-domain loop) with a zero
    and a duplicated column, l1_ratio 0, 0.5 and 1, alpha past alpha_max and a max_iter stop"""
    from oracle import oracle as O
    rng = np.random.RandomState(0)
    n, d = 80, 14
    X = rng.randn(n, d)
    X[:, 2] = 0.0
    X[:, 6] = X[:, 5]
    y = X @ rng.randn(d) + 0.3 * rng.randn(n)
    Xc, yc = X - X.mean(0), y - y.mean()
    A, b, yy = Xc.T @ Xc, Xc.T @ yc, yc @ yc
    amax = np.abs(b).max() / n
    for a, r, mi in ((1e3 * amax, 1.0, 100), (0.05 * amax, 1.0, 1000), (0.05 * amax, 0.5, 1000), (0.5, 0.0, 1000),
                     (0.001 * amax, 1.0, 3)):
        w, it, gap, tol, _ = cd_gram(A, b, n, yy, a, r, 1e-4, mi, 1)
        wo, gapo, tolo, ito = O.enet_cd(np.asfortranarray(Xc), yc, a * r * n, a * (1 - r) * n, 1e-4, mi)
        assert it == ito, (a, r, it, ito)
        np.testing.assert_allclose(w, wo, rtol=0, atol=1e-9 * max(np.abs(wo).max(), 1e-300))
        assert abs(gap - gapo) <= 1e-8 * max(abs(gapo), tolo)


def test_score_references_match_scikit_learn():
    """intercept() from centred training means and a shift gives scikit-learn Ridge's intercept, and score_ref its scores"""
    from sklearn.linear_model import Ridge
    rng = np.random.RandomState(1)
    X = rng.randn(50, 6) + 5.0
    y = X @ rng.randn(6) + 3.0 + 0.1 * rng.randn(50)
    m = Ridge(alpha=0.7).fit(X, y)
    c = (X.mean(0) + 0.25).astype(np.float32)
    shift = np.concatenate([c, [np.float32(y.mean() - 1.0)]])
    means = np.concatenate([X.mean(0) - shift[:6].astype(np.float64), [y.mean() - np.float64(shift[6])]])
    assert abs(intercept(means, shift, m.coef_) - m.intercept_) <= 1e-12 * abs(m.intercept_) + 1e-12
    pred = m.predict(X)
    assert score_ref(y, pred, SCORE_DEFAULT) == m.score(X, y)
    assert score_ref(y, pred, NEG_MSE) == -mean_squared_error(y, pred)
    assert np.isnan(score_ref(y[:1], pred[:1], SCORE_DEFAULT))
    assert score_ref(np.full(5, 2.0), np.arange(5.0), SCORE_DEFAULT) == r2_score(np.full(5, 2.0), np.arange(5.0)) == 0.0
