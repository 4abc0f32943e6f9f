"""The kernel-SVM scoring kernels (csrc/score.cu) and the kernel-matrix guard (csrc/gram.cu), one kernel at a time, against
float64 / integer references in numpy.

The GPU tests feed each kernel through its test hook (gs_debug_decision, gs_debug_score, gs_debug_kernel_matrix) and compare
number for number: decision values within a rounding-error bound of a long-double sum over the GPU's own float64 Gram,
votes, class counts and AUC pair counts exactly, residual sums exactly on integer data and within a bound on random data.
The references themselves are checked against scikit-learn on the CPU (the tests without the gpu mark), so they can be
trusted on a machine without a GPU."""
import numpy as np
import pytest

gpu = pytest.mark.gpu
U = 2.0 ** -53                     # unit roundoff of float64
TJ = 32                            # support rows per tile of score.cu's decision_kernel
FLT_MIN = np.float32(np.finfo(np.float32).tiny)


# ------------------------------------------------------------------------------------------------ references ----------
def _powi(base, times):
    """libsvm's powi on arrays, every multiplication rounded on its own"""
    tmp, ret = base.copy(), np.ones_like(base)
    t = times
    while t > 0:
        if t % 2 == 1:
            ret = ret * tmp
        tmp = tmp * tmp
        t //= 2
    return ret


def kernel_rows(S, xsq, rows, kernel, gamma, degree, coef0):
    """float64 k(x_r, x_j) for the rows r of the slice `rows` and every j, in libsvm's evaluation order"""
    s = S[rows]
    if kernel == "rbf":
        return np.exp(-gamma * ((xsq[rows, None] + xsq[None, :]) - 2.0 * s))
    if kernel == "poly":
        return _powi(gamma * s + coef0, degree)
    if kernel == "sigmoid":
        return np.tanh(gamma * s + coef0)
    return s.copy()


def decision_ref(S, xsq, coef, kernel, gamma=0.0, degree=3, coef0=0.0, block=256):
    """(dec [ncols][n] summed in long double, sum_j |k(r, j)| |coef[c][j]| [ncols][n]) in row blocks of `block`"""
    n = S.shape[0]
    cl, ca = coef.astype(np.longdouble).T.copy(), np.abs(coef).T.copy()
    ref, mag = np.zeros(coef.shape, np.longdouble), np.zeros(coef.shape)
    for r0 in range(0, n, block):
        rows = slice(r0, min(n, r0 + block))
        k = kernel_rows(S, xsq, rows, kernel, gamma, degree, coef0)
        ref[:, rows] = (k.astype(np.longdouble) @ cl).T
        mag[:, rows] = (np.abs(k) @ ca).T
    return ref, mag


def vote_predict(dv, n_classes):
    """libsvm's one-vs-one vote (svm.cpp svm_predict_values) on dv [n_pairs][n] = dec - rho, pairs (0,1), (0,2), ..., (1,2),
    ...: dv > 0 votes for the lower class of the pair, anything else (0 included) for the higher; the first maximum wins"""
    votes = np.zeros((n_classes, dv.shape[1]), np.int64)
    p = 0
    for a in range(n_classes):
        for b in range(a + 1, n_classes):
            pos = dv[p] > 0
            votes[a] += pos
            votes[b] += ~pos
            p += 1
    return np.argmax(votes, axis=0)


def vote_counts(pred, y, te, tr):
    """[test correct, test rows, training correct, training rows]"""
    ok = pred == y
    return np.array([np.sum(ok & te), np.sum(te), np.sum(ok & tr), np.sum(tr)])


def class_counts(pred, y, te, tr, n_classes):
    """[split (test, training)][class][support, true positives, predicted]"""
    out = np.zeros((2, n_classes, 3), np.int64)
    for sp, m in enumerate((te, tr)):
        out[sp, :, 0] = np.bincount(y[m], minlength=n_classes)
        out[sp, :, 1] = np.bincount(y[m & (pred == y)], minlength=n_classes)
        out[sp, :, 2] = np.bincount(pred[m], minlength=n_classes)
    return out


def auc_pairs(s, pos, masks):
    """[wins, ties] of the pairs (p positive, q negative) inside each mask: s_p > s_q, s_p == s_q (integers)"""
    out = []
    for m in masks:
        neg = np.sort(s[m & ~pos])
        p = s[m & pos]
        lo, hi = np.searchsorted(neg, p, "left"), np.searchsorted(neg, p, "right")
        out += [int(lo.sum()), int((hi - lo).sum())]
    return out


def residual_sum(z, dec, rho, m):
    """(sum over the rows of m of e^2 in long double, the float64 e^2 summed), e = z - (dec - rho) in float64"""
    e = z[m] - (dec[m] - rho)
    e2 = e * e
    return np.sum(e2.astype(np.longdouble)), e2


# ------------------------------------------------------------------------------------------------ helpers -------------
def _pack(bits):
    """bool [n][n_splits] -> uint64 [n][2] membership masks (bit k of word k / 64)"""
    out = np.zeros((bits.shape[0], 2), np.uint64)
    for k in range(bits.shape[1]):
        out[:, k >> 6] |= bits[:, k].astype(np.uint64) << np.uint64(k & 63)
    return out


def _random_splits(rng, n, n_splits):
    """ShuffleSplit-like membership: test, training or neither, independently per split"""
    u = rng.random((n, n_splits))
    return u < 0.25, u > 0.45


def _classification(engine, rng, n, n_classes, n_splits=None, d=16):
    """random X, labels covering every class in shuffled order (the engine sorts rows by class), optional random splits"""
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = rng.permutation(np.arange(n) % n_classes).astype(np.int32)
    engine.set_data(X, np.zeros(n, np.int8), 1, y_class=y)
    te = tr = None
    if n_splits:
        te, tr = _random_splits(rng, n, n_splits)
        engine.set_splits(_pack(te), _pack(tr), n_splits)
    return X, y, te, tr


# ------------------------------------------------------------------------------------------------ decision values -----
# (kernel, gamma, degree, coef0, n, ncols, forced slab counts); every case also runs the search's own slab count
DECISION_CASES = [
    ("linear", 0.0, 3, 0.0, 1, 1, [1, 2]),
    ("linear", 0.0, 3, 0.0, 31, 7, [1, 3]),
    ("rbf", 1 / 16, 3, 0.0, 33, 9, [1, 2]),
    ("poly", 1 / 16, 3, -1.0, 33, 8, [1, 10]),
    ("rbf", 1 / 32, 3, 0.0, 65, 95, [1, 16]),
    ("poly", 1 / 16, 1, -2.0, 257, 96, [2, 3]),
    ("sigmoid", 1 / 16, 3, -0.5, 257, 97, [1, 10]),
    ("poly", 1 / 16, 5, -0.25, 1000, 193, [1, 3]),
    ("rbf", 1 / 16, 3, 0.0, 1000, 40, [16]),
    ("poly", 1 / 16, 2, -1.0, 4100, 9, [1, 16]),
    ("sigmoid", 1 / 16, 3, -0.5, 4100, 8, [2, 16]),
    ("rbf", 1 / 16, 3, 0.0, 4608, 40, [1]),
    ("poly", 1 / 16, 4, -0.5, 4608, 1, [10]),
    ("linear", 0.0, 3, 0.0, 4608, 7, [3]),
]


@gpu
@pytest.mark.parametrize("case", DECISION_CASES, ids=lambda c: "%s-n%d-c%d" % (c[0], c[4], c[5]))
def test_decision_values_against_long_double_sums(engine, case):
    """dec[c][r] = sum_j k64(r, j) coef[c][j] on every slab split: within the rounding-error bound of the kernel's sum
    (jlen fmas per slab, then the slab sum) of a long-double reference, and with a median relative error of a float64
    computation (a float32 kernel value would be ~1e-8).  The coefficients are ~1 on a random "training" set and 0 elsewhere,
    so one support row dropped or counted twice misses the bound by orders of magnitude."""
    kernel, gamma, degree, coef0, n, ncols, forced = case
    rng = np.random.default_rng(n * 1000 + ncols)
    _classification(engine, rng, n, 2)
    S, xsq = engine.debug_gram()
    train = rng.random((ncols, n)) < 0.8
    coef = np.where(train, rng.uniform(0.5, 1.5, (ncols, n)) * rng.choice([-1.0, 1.0], (ncols, n)), 0.0)
    ref, mag = decision_ref(S, xsq, coef, kernel, gamma, degree, coef0)
    seen = set()
    for jchunks in [0] + forced:
        dec, used = engine.debug_decision(kernel, gamma, coef, degree=degree, coef0=coef0, jchunks=jchunks)
        if jchunks:
            assert used == jchunks
        seen.add(used)
        jlen = (n + used - 1) // used                              # support rows per slab, whole tiles
        jlen = (jlen + TJ - 1) // TJ * TJ
        err = np.abs(dec.astype(np.longdouble) - ref).astype(np.float64)
        bound = (jlen + used + 2) * U * mag
        worst = np.unravel_index(np.argmax(err - bound), err.shape)
        assert np.all(err <= bound), (jchunks, used, worst, err[worst], bound[worst])
        nz = ref != 0
        rel = err[nz] / np.abs(ref[nz]).astype(np.float64)
        assert np.median(rel) < 1e-14, (jchunks, used, np.median(rel))
    if n == 4608 and ncols == 40:
        assert max(seen) > 1, "the search's slab count at n = 4608, 40 columns should split the support rows"


# ------------------------------------------------------------------------------------------------ votes ---------------
def _vote_decisions(rng, n, n_classes, n_sets):
    """n_sets consecutive blocks of n_pairs decision columns; dec == rho exactly on every 5th row of each column"""
    n_pairs = n_classes * (n_classes - 1) // 2
    ncols = n_pairs * n_sets
    rho = rng.standard_normal(ncols)
    dec = rho[:, None] + rng.standard_normal((ncols, n))
    dec[:, rng.random(n) < 0.2] = rho[:, None]
    return dec, rho, n_pairs


@gpu
@pytest.mark.parametrize("n_classes", [2, 3, 7, 32])
def test_votes_and_class_counts_exact(engine, n_classes):
    """vote_kernel and vote_classes_kernel equal the restatement of libsvm's vote on every (column set, split) task: rows
    with dec - rho == 0 (a vote for the higher class), tied vote counts (the first maximum), rows in neither set, and
    100 splits, so that the tasks of splits 64..99 read the second mask word"""
    rng = np.random.default_rng(n_classes)
    n, n_splits = 700, 100
    _, y, te, tr = _classification(engine, rng, n, n_classes, n_splits, d=2)
    dec, rho, n_pairs = _vote_decisions(rng, n, n_classes, 2)
    preds = [vote_predict(dec[s:s + n_pairs] - rho[s:s + n_pairs, None], n_classes) for s in (0, n_pairs)]
    if n_classes > 2:                                               # the data does hold ties
        dv = dec[:n_pairs] - rho[:n_pairs, None]
        votes = np.zeros((n_classes, n), np.int64)
        p = 0
        for a in range(n_classes):
            for b in range(a + 1, n_classes):
                votes[a] += dv[p] > 0
                votes[b] += ~(dv[p] > 0)
                p += 1
        assert np.sum(np.sum(votes == votes.max(0), 0) > 1) > 10
    first_col = np.repeat([0, n_pairs], n_splits)
    fold = np.tile(np.arange(n_splits), 2)
    got_v = engine.debug_score("vote", dec, rho, first_col, fold)
    got_c = engine.debug_score("class_counts", dec, rho, first_col, fold)
    for t, (c0, k) in enumerate(zip(first_col, fold)):
        pred = preds[c0 // n_pairs]
        np.testing.assert_array_equal(got_v[t], vote_counts(pred, y, te[:, k], tr[:, k]), err_msg=str((t, c0, k)))
        np.testing.assert_array_equal(got_c[t], class_counts(pred, y, te[:, k], tr[:, k], n_classes), err_msg=str((t, c0, k)))


@gpu
def test_votes_beyond_one_launch_of_tasks(engine):
    """~40 000 tasks on three shared binary columns: the launches of 32 768 tasks each must write at their own offsets"""
    rng = np.random.default_rng(40000)
    n, n_splits = 300, 100
    _, y, te, tr = _classification(engine, rng, n, 2, n_splits, d=2)
    dec, rho, _ = _vote_decisions(rng, n, 2, 3)
    t = np.arange(40003)
    first_col, fold = (t % 3).astype(np.int32), ((t * 7 + t // 300) % n_splits).astype(np.int32)
    preds = [vote_predict(dec[c:c + 1] - rho[c], 2) for c in range(3)]
    want_v = np.array([[vote_counts(preds[c], y, te[:, k], tr[:, k]) for k in range(n_splits)] for c in range(3)])
    want_c = np.array([[class_counts(preds[c], y, te[:, k], tr[:, k], 2) for k in range(n_splits)] for c in range(3)])
    np.testing.assert_array_equal(engine.debug_score("vote", dec, rho, first_col, fold), want_v[first_col, fold])
    np.testing.assert_array_equal(engine.debug_score("class_counts", dec, rho, first_col, fold), want_c[first_col, fold])


# ------------------------------------------------------------------------------------------------ AUC -----------------
def _tied_scores(rng, ncols, n):
    """half-integer scores with many exact ties, +0.0 and -0.0 both present; a part of the rows moved by 1e-12, which
    separates them in float64 but not in float32"""
    s = rng.integers(-3, 4, (ncols, n)) * 0.5
    zero = s == 0
    s[zero] = np.where(rng.random(zero.sum()) < 0.5, 0.0, -0.0)
    nudge = rng.random((ncols, n)) < 0.3
    s[nudge] += rng.choice([-1e-12, 1e-12], nudge.sum())
    return s


@gpu
@pytest.mark.parametrize("n_neg,n_pos", [(300, 517), (300, 1), (600, 700)])
def test_auc_pair_counts_exact(engine, n_neg, n_pos):
    """auc_pairs_kernel<double> with the SVC search's sign (-1 on dec) and auc_pairs_kernel<float> with LogisticRegression's
    (+1 on (float)dec) equal integer win / tie counts over the test and training rows of every split, 100 splits"""
    rng = np.random.default_rng(n_neg * 7 + n_pos)
    n, n_splits = n_neg + n_pos, 100
    X = rng.standard_normal((n, 2)).astype(np.float32)
    y = rng.permutation(np.r_[np.zeros(n_neg), np.ones(n_pos)]).astype(np.int32)
    engine.set_data(X, np.zeros(n, np.int8), 1, y_class=y)
    te, tr = _random_splits(rng, n, n_splits)
    if n_pos == 1:                                                  # the single positive row is tested by half the splits
        te[y == 1], tr[y == 1] = np.arange(n_splits) % 2 == 0, np.arange(n_splits) % 2 == 1
    engine.set_splits(_pack(te), _pack(tr), n_splits)
    dec = _tied_scores(rng, 2, n)
    first_col = np.repeat([0, 1], n_splits)
    fold = np.tile(np.arange(n_splits), 2)
    pos = y == 1
    for kind, score in (("auc_f64", -dec), ("auc_f32", dec.astype(np.float32))):
        got = engine.debug_score(kind, dec, None, first_col, fold)
        want = np.array([auc_pairs(score[c], pos, (te[:, k], tr[:, k])) for c, k in zip(first_col, fold)], np.uint64)
        np.testing.assert_array_equal(got, want, err_msg=kind)
        assert n_pos == 1 or (want[:, 1].sum() > 0 and want[:, 0].sum() > 0)
    f64 = [auc_pairs(-dec[0], pos, (te[:, k],)) for k in range(n_splits)]
    f32 = [auc_pairs(dec[0].astype(np.float32), pos, (te[:, k],)) for k in range(n_splits)]
    assert n_pos == 1 or f64 != f32                                 # the float32 instance sees its own ties


# ------------------------------------------------------------------------------------------------ RSS -----------------
def _regression(engine, rng, n, z, n_splits):
    X = rng.standard_normal((n, 2)).astype(np.float32)
    engine.set_data(X, rng.integers(0, 5, n).astype(np.int8), 5, y_target=z.astype(np.float32))
    engine.set_targets_f64(z)
    te, tr = _random_splits(rng, n, n_splits)
    engine.set_splits(_pack(te), _pack(tr), n_splits)
    return te, tr


@gpu
def test_rss_bit_exact_on_integers(engine):
    """small-integer targets, decision values and intercepts: every residual, square and partial sum is exact in float64,
    so the fixed-order reduction must return the exact sum"""
    rng = np.random.default_rng(5)
    n, n_splits = 4999, 70
    z = rng.integers(-20, 21, n).astype(np.float64)
    te, tr = _regression(engine, rng, n, z, n_splits)
    dec = rng.integers(-20, 21, (3, n)).astype(np.float64)
    rho = np.array([0.0, 3.0, -7.0])
    first_col, fold = np.repeat(np.arange(3), n_splits), np.tile(np.arange(n_splits), 3)
    got = engine.debug_score("rss", dec, rho, first_col, fold)
    want = [[float(residual_sum(z, dec[c], rho[c], m)[0]) for m in (te[:, k], tr[:, k])] for c, k in zip(first_col, fold)]
    np.testing.assert_array_equal(got, np.array(want))


@gpu
def test_rss_within_summation_bound(engine):
    rng = np.random.default_rng(6)
    n, n_splits = 3001, 70
    z = rng.standard_normal(n) * 10
    te, tr = _regression(engine, rng, n, z, n_splits)
    dec = z + rng.standard_normal((2, n))
    rho = rng.standard_normal(2)
    first_col, fold = np.repeat(np.arange(2), n_splits), np.tile(np.arange(n_splits), 2)
    got = engine.debug_score("rss", dec, rho, first_col, fold)
    for t, (c, k) in enumerate(zip(first_col, fold)):
        for sp, m in enumerate((te[:, k], tr[:, k])):
            ref, e2 = residual_sum(z, dec[c], rho[c], m)
            err = abs(float(np.longdouble(got[t, sp]) - ref))
            assert err <= (m.sum() + 8) * U * e2.sum(), (t, sp, err)


# ------------------------------------------------------------------------------------------------ hook arguments ------
@gpu
def test_score_hook_rejects_bad_tasks(engine):
    from spark_sklearn_b200.engine import EngineError
    rng = np.random.default_rng(9)
    n = 50
    _, y, te, tr = _classification(engine, rng, n, 3, n_splits=4, d=2)
    dec, rho = rng.standard_normal((3, n)), np.zeros(3)
    for first_col, fold in (([1], [0]), ([-1], [0]), ([0], [4]), ([0], [-1])):
        with pytest.raises(EngineError):
            engine.debug_score("vote", dec, rho, first_col, fold)
    for kind in ("auc_f64", "rss"):                                 # three classes; no regression targets
        with pytest.raises(EngineError):
            engine.debug_score(kind, dec, rho, [0], [0])
    with pytest.raises(EngineError):
        engine._check(engine._L.gs_debug_score(engine._h, 5, dec.ctypes.data, rho.ctypes.data, 3,
                                               np.zeros(1, np.int32).ctypes.data, np.zeros(1, np.int32).ctypes.data, 1,
                                               np.zeros(16, np.int32).ctypes.data))
    np.testing.assert_array_equal(engine.debug_score("vote", dec, rho, [0], [3])[0],            # the valid call still runs
                                  vote_counts(vote_predict(dec, 3), y, te[:, 3], tr[:, 3]))


# ------------------------------------------------------------------------------------------------ guard flag and qd ---
def _special(K):
    return bool(np.any(~((K > 0) & (K >= FLT_MIN) & np.isfinite(K))))


def _far_pair(n):
    """a cluster near the origin and, in the last two rows, two points at distance 2 from each other"""
    X = np.random.default_rng(n).uniform(-0.05, 0.05, (n, 2)).astype(np.float32)
    X[n - 2], X[n - 1] = (-1, 0), (1, 0)
    return X


def _sigmoid_zero_diagonal(n):
    """tanh(x.x - 1) == 0 only at (n-1, n-1): the last row is (1, 0), every other row has x.x' >= ~3.6"""
    X = np.random.default_rng(n).uniform(-0.05, 0.05, (n, 2)).astype(np.float32)
    X[:, 0] += 2
    X[n - 1] = (1, 0)
    return X


def _guard_cases(n):
    """(X, kernel, gamma, degree, coef0, the flag expected, the rows of the special entries or None)"""
    rng = np.random.default_rng(n + 1)
    R = rng.standard_normal((n, 8)).astype(np.float32)
    cases = [(R * 0.3, "rbf", 0.5, 3, 0.0, False, None),
             (R, "poly", 0.5, 2, 1.0, False, None),
             (R, "poly", 0.25, 4, 0.5, False, None),
             (_sigmoid_zero_diagonal(n), "sigmoid", 1.0, 3, -1.0, True, [(n - 1, n - 1)])]
    if n > 1:
        cases += [(_far_pair(n), "rbf", 95 / 4, 3, 0.0, True, [(n - 2, n - 1), (n - 1, n - 2)]),      # exp(-95): subnormal
                  (_far_pair(n), "rbf", 120 / 4, 3, 0.0, True, [(n - 2, n - 1), (n - 1, n - 2)]),     # exp(-120): 0 in float32
                  (R, "linear", 0.0, 3, 0.0, True, None),
                  (R, "sigmoid", 0.125, 3, -0.5, True, None)]
    return cases


@gpu
@pytest.mark.parametrize("n", [1, 33, 1024, 1025])
def test_kernel_matrix_guard_flag_and_diagonal(engine, n):
    """the guard flag is raised exactly when K holds a zero, subnormal, negative or non-finite float32 (the single special
    entry sits in the last column / the last row, so warp tails and the second column block are covered); qd is libsvm's
    float64 diagonal: exact for poly, within one ulp of tanh for sigmoid"""
    for X, kernel, gamma, degree, coef0, want, where in _guard_cases(n):
        engine.set_data(X, np.zeros(n, np.int8), 1, y_class=np.zeros(n, np.int32))
        _, xsq = engine.debug_gram()
        K, qd, flag = engine.debug_kernel_matrix(kernel, gamma, degree=degree, coef0=coef0, return_guard=True)
        label = (n, kernel, gamma, degree, coef0)
        assert flag == int(_special(K)), label
        assert flag == int(want), label
        if where is not None:
            bad = ~((K > 0) & (K >= FLT_MIN) & np.isfinite(K))
            assert sorted(zip(*np.nonzero(bad))) == sorted(where), label
        if kernel == "poly":
            np.testing.assert_array_equal(qd, _powi(gamma * xsq + coef0, degree), err_msg=str(label))
        elif kernel == "sigmoid":
            # CUDA's float64 tanh is specified to 2 ulp (CUDA Math API), and it does differ from the host's tanh by more
            # than one ulp on some of these arguments: compare with the long-double tanh of the same float64 argument
            ref = np.tanh((gamma * xsq + coef0).astype(np.longdouble))
            ulps = np.abs(qd - ref) / np.spacing(np.abs(ref.astype(np.float64)))
            assert np.all(ulps <= 2), (label, float(ulps.max()))
        else:
            assert qd is None


# ------------------------------------------------------------------------------------------------ end to end ----------
@gpu
def test_svc_roc_auc_search_on_the_slab_path(engine):
    """roc_auc ranks the decision values themselves, so it sees errors an accuracy cannot: a search over 4600 rows of the
    config-2 data (n >= 4096: the decision values run on the split support-row range) against scikit-learn's GridSearchCV"""
    import warnings
    from sklearn.model_selection import GridSearchCV as SkGrid
    from sklearn.svm import SVC
    from spark_sklearn_b200 import GridSearchCV, workloads as W
    w = W.make_workload("c2")
    X, y = w["X"][:4600], w["y"][:4600]
    grid = {"C": [1.0, 10.0], "gamma": [1 / 512]}
    a = GridSearchCV(None, SVC(), grid, cv=3, scoring="roc_auc", refit=False).fit(X, y)
    assert engine.n == 4600 and engine.debug_decision("rbf", 1 / 512, np.zeros((6, 4600)))[1] > 1
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        b = SkGrid(SVC(), grid, cv=3, scoring="roc_auc", return_train_score=True, refit=False).fit(X, y)
    for k in range(3):
        for part in ("test", "train"):
            key = "split%d_%s_score" % (k, part)
            np.testing.assert_allclose(a.cv_results_[key], b.cv_results_[key], rtol=0, atol=1e-12, err_msg=key)
    np.testing.assert_array_equal(a.cv_results_["rank_test_score"], b.cv_results_["rank_test_score"])


# ------------------------------------------------------------------------------------------------ the references (CPU) -
def test_vote_reference_matches_svc_predict():
    from sklearn.datasets import make_blobs
    from sklearn.svm import SVC
    for n_classes in (2, 4):
        X, y = make_blobs(240, n_features=3, centers=n_classes, cluster_std=3.0, random_state=n_classes)
        clf = SVC(decision_function_shape="ovo").fit(X, y)
        df = clf.decision_function(X)
        dv = -df[None, :] if n_classes == 2 else df.T               # scikit-learn negates libsvm's binary value only
        np.testing.assert_array_equal(clf.classes_[vote_predict(dv, n_classes)], clf.predict(X))
    # hand-made: a zero votes for the higher class; a three-way tie goes to the first class
    np.testing.assert_array_equal(vote_predict(np.array([[0.0, 1.0]]), 2), [1, 0])
    np.testing.assert_array_equal(vote_predict(np.array([[1.0], [-1.0], [1.0]]), 3), [0])


def test_decision_reference_matches_svc_decision_function():
    from sklearn.datasets import make_blobs
    from sklearn.svm import SVC
    X, y = make_blobs(200, n_features=4, centers=2, cluster_std=4.0, random_state=0)
    X64 = X.astype(np.float32).astype(np.float64)
    S = X64 @ X64.T
    xsq = np.einsum("ij,ij->i", X64, X64)
    for kernel, kw in (("rbf", dict(gamma=0.05)), ("poly", dict(gamma=0.05, degree=3, coef0=-1.0)),
                       ("sigmoid", dict(gamma=0.01, coef0=-0.5)), ("linear", {})):
        clf = SVC(kernel=kernel, **kw).fit(X64, y)
        coef = np.zeros((1, len(y)))
        coef[0, clf.support_] = clf.dual_coef_[0]
        ref, _ = decision_ref(S, xsq, coef, kernel, kw.get("gamma", 0.0), kw.get("degree", 3), kw.get("coef0", 0.0), block=64)
        np.testing.assert_allclose(ref[0].astype(np.float64) + clf.intercept_[0], clf.decision_function(X64), rtol=0,
                                   atol=1e-9, err_msg=kernel)


def test_auc_reference_matches_roc_auc_score():
    from sklearn.metrics import roc_auc_score
    rng = np.random.default_rng(3)
    for n_neg, n_pos in ((300, 517), (300, 1), (37, 600)):
        y = rng.permutation(np.r_[np.zeros(n_neg, bool), np.ones(n_pos, bool)])
        s = _tied_scores(rng, 1, len(y))[0]
        w, t = auc_pairs(s, y, (np.ones(len(y), bool),))
        assert abs((w + 0.5 * t) / (n_neg * n_pos) - roc_auc_score(y, s)) <= 1e-12


def test_rss_reference_matches_r2_score():
    from sklearn.metrics import r2_score
    rng = np.random.default_rng(4)
    z = rng.standard_normal(500) * 3
    dec, rho = z + rng.standard_normal(500), 0.7
    m = rng.random(500) < 0.4
    rss, _ = residual_sum(z, dec, rho, m)
    tss = np.sum((z[m] - z[m].mean()) ** 2)
    assert abs((1 - float(rss) / tss) - r2_score(z[m], dec[m] - rho)) <= 1e-12
