"""The SAG oracle (tests/sag_oracle.c) against scikit-learn's LogisticRegression(solver='sag' | 'saga') and sag_solver:
coef_, intercept_ and n_iter_ bit for bit, for both solvers, binary and 3-class, float64 and float32 X, every penalty, class
and sample weights, fit_intercept=False, the max_iter stop, the mid-epoch rescale and the squared loss.  The oracle uses the
same libm as scikit-learn, so the logistic gradients are exact here."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import LogisticRegression

from sag_oracle import SAGOracle, draws, sag_fit

RNG = np.random.RandomState(0)
X = RNG.randn(80, 6)
Y2 = (X[:, 0] + 0.5 * RNG.randn(80) > 0).astype(int)
Y3 = RNG.randint(0, 3, 80)


def _same(sk, o):
    assert sk.coef_.dtype == o.coef_.dtype and sk.intercept_.dtype == o.intercept_.dtype
    np.testing.assert_array_equal(sk.coef_, o.coef_)
    np.testing.assert_array_equal(sk.intercept_, o.intercept_)
    np.testing.assert_array_equal(sk.n_iter_, o.n_iter_)


def _fit(X, y, sample_weight=None, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return LogisticRegression(**kw).fit(X, y, sample_weight=sample_weight)


PENALTIES = [dict(l1_ratio=0.0), dict(l1_ratio=0.5), dict(l1_ratio=1.0), dict(C=np.inf), dict(C=1e-4),
             dict(C=3e-4, l1_ratio=0.5), dict(max_iter=3)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("solver", ["sag", "saga"])
@pytest.mark.parametrize("y", [Y2, Y3], ids=["binary", "3-class"])
def test_logistic_regression(dtype, solver, y):
    for pen in PENALTIES:
        if solver == "sag" and pen.get("l1_ratio", 0.0) > 0:
            continue
        kw = dict(solver=solver, random_state=1, max_iter=200)
        kw.update(pen)
        _same(_fit(X.astype(dtype), y, **kw), SAGOracle(X.astype(dtype), y, **kw))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_weights_and_switches(dtype):
    sw = RNG.uniform(0, 2, 80)
    sw[::5] = 0.0
    for y in (Y2, Y3):
        for extra in (dict(class_weight="balanced"), dict(class_weight={0: 2.0, 1: 0.5}), dict(fit_intercept=False),
                      dict(solver="sag", l1_ratio=0.0, class_weight="balanced", C=0.1)):
            kw = dict(solver="saga", l1_ratio=0.5, random_state=4, max_iter=100)
            kw.update(extra)
            Xd = X.astype(dtype)
            _same(_fit(Xd, y, sample_weight=sw, **kw), SAGOracle(Xd, y, sample_weight=sw, **kw))
            _same(_fit(Xd, y, **kw), SAGOracle(Xd, y, **kw))


def test_mid_epoch_rescale_and_max_iter():
    """a small C rescales every few samples (wscale < 1e-9), including on an epoch's last sample with the L1 term, whose
    end-of-epoch lagged update then replays the epoch's cumulative sums; max_iter stops with status 1"""
    o = SAGOracle(X, Y2, solver="saga", C=1e-4, l1_ratio=0.5, random_state=2, max_iter=50)
    assert o.status in (0, 1)
    for n in range(40, 80):                    # a rescale period that divides the training size
        for C in (1e-4, 2e-4, 5e-4):
            kw = dict(solver="saga", C=C, l1_ratio=0.5, random_state=2, max_iter=20)
            _same(_fit(X[:n], Y2[:n], **kw), SAGOracle(X[:n], Y2[:n], **kw))
    o = SAGOracle(X, Y3, solver="sag", random_state=0, max_iter=2)
    assert o.status == 1 and o.n_iter == 2


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("saga", [False, True])
def test_squared_loss_equals_sag_solver(dtype, saga):
    from sklearn.linear_model._sag import get_auto_step_size, sag_solver
    from sklearn.utils.extmath import row_norms
    Xd = X.astype(dtype)
    y = (X @ RNG.randn(6) + 0.1 * RNG.randn(80)).astype(dtype)
    sw = RNG.uniform(0, 2, 80).astype(dtype)
    sw[::4] = 0
    for alpha, beta, fi in [(1.0, 0.0, True), (0.1, 0.5, True), (1e3, 0.0, False), (0.0, 2.0, False)]:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", ConvergenceWarning)
            init = {"coef": np.zeros((Xd.shape[1] + int(fi), 1), dtype)}
            coef, n_iter, _ = sag_solver(Xd, y, sw, "squared", alpha, beta, 30, 1e-4, 0, 7, False, None, init, is_saga=saga)
        n = len(Xd)
        step = get_auto_step_size(row_norms(Xd, squared=True).max(), alpha / n, "squared", fi, n_samples=n, is_saga=saga)
        seed = np.random.RandomState(7).randint(1, np.iinfo(np.int32).max)
        got, it, st, steps = sag_fit(Xd, y, sw, "squared", step, alpha / n, beta / n, seed, saga, 1e-4, 30, fi)
        assert it == n_iter and steps == n * it
        np.testing.assert_array_equal(got[0, :Xd.shape[1]], coef[:Xd.shape[1]])
        if fi:
            assert got[0, -1] == coef[-1]


def test_draws():
    d = draws(12345, 20, 1000)
    assert d.min() >= 0 and d.max() < 20 and len(set(d)) == 20
