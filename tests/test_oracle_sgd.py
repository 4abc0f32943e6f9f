"""The SGD oracle (tests/sgd_oracle.c) against scikit-learn's SGDClassifier / SGDRegressor: coef_, intercept_, n_iter_ and
t_ bit for bit, for every loss x penalty x learning rate, binary and one-vs-rest, float64 and float32 X, class and sample
weights, and the stop rules.  The oracle uses the same libm as scikit-learn, so log_loss and invscaling are exact here."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import SGDClassifier, SGDRegressor

from sgd_oracle import SGDOracle, perm

RNG = np.random.RandomState(0)
X = RNG.randn(90, 7)
Y2 = (X[:, 0] + 0.3 * RNG.randn(90) > 0).astype(int)
Y3 = RNG.randint(0, 3, 90)
YR = X @ RNG.randn(7) + 0.1 * RNG.randn(90)
PENALTIES = [None, "l2", "l1", "elasticnet"]
RATES = ["optimal", "constant", "invscaling", "adaptive"]


def _same(sk, o):
    assert sk.coef_.dtype == o.coef_.dtype
    np.testing.assert_array_equal(sk.coef_, o.coef_)
    assert sk.intercept_.dtype == o.intercept_.dtype
    np.testing.assert_array_equal(sk.intercept_, o.intercept_)
    assert sk.n_iter_ == o.n_iter_ and sk.t_ == o.t_


def _fit(cls, X, y, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return cls(**kw).fit(X, y)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("loss", ["hinge", "perceptron", "squared_hinge", "modified_huber", "log_loss"])
@pytest.mark.parametrize("penalty", PENALTIES)
def test_classifier(dtype, loss, penalty):
    for lr in RATES:
        for y in (Y2, Y3):
            kw = dict(loss=loss, penalty=penalty, learning_rate=lr, eta0=0.01, random_state=3, max_iter=30)
            _same(_fit(SGDClassifier, X.astype(dtype), y, **kw), SGDOracle(X.astype(dtype), y, **kw))


@pytest.mark.parametrize("loss", ["squared_error", "huber", "epsilon_insensitive", "squared_epsilon_insensitive"])
@pytest.mark.parametrize("penalty", PENALTIES)
def test_regressor_float64(loss, penalty):
    for lr in RATES:
        kw = dict(loss=loss, penalty=penalty, learning_rate=lr, eta0=0.01, random_state=3, max_iter=30)
        _same(_fit(SGDRegressor, X, YR, **kw), SGDOracle(X, YR, classifier=False, **kw))


@pytest.mark.parametrize("penalty", PENALTIES)
def test_regressor_float32(penalty):
    for loss in ["squared_error", "huber", "epsilon_insensitive", "squared_epsilon_insensitive"]:
        for lr in RATES:
            kw = dict(loss=loss, penalty=penalty, learning_rate=lr, eta0=0.01, random_state=3, max_iter=30)
            X32, y32 = X.astype(np.float32), YR.astype(np.float32)
            _same(_fit(SGDRegressor, X32, y32, **kw), SGDOracle(X32, y32, classifier=False, **kw))


def test_weights_and_switches():
    sw = RNG.uniform(0, 2, 90)
    sw[::5] = 0.0
    for y in (Y2, Y3):
        for extra in (dict(class_weight={0: 2.0, 1: 0.5}), dict(class_weight="balanced"), dict(fit_intercept=False),
                      dict(shuffle=False), dict(tol=None, max_iter=7), dict(n_iter_no_change=2, tol=1e-1)):
            kw = dict(random_state=5, max_iter=50)
            kw.update(extra)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", ConvergenceWarning)
                sk = SGDClassifier(**kw).fit(X, y, sample_weight=sw)
            _same(sk, SGDOracle(X, y, sample_weight=sw, **kw))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        sk = SGDRegressor(random_state=5, max_iter=50).fit(X, YR, sample_weight=sw)
    _same(sk, SGDOracle(X, YR, classifier=False, sample_weight=sw, random_state=5, max_iter=50))


def test_stop_rule_and_max_iter_warning():
    o = SGDOracle(X, Y2, random_state=0, tol=1e-1)
    assert o.status == [0] and o.n_iter_ < 1000
    with pytest.warns(ConvergenceWarning, match="Maximum number of iteration"):
        sk = SGDClassifier(random_state=0, max_iter=3).fit(X, Y2)
    o = SGDOracle(X, Y2, random_state=0, max_iter=3)
    assert o.status == [1] and sk.n_iter_ == o.n_iter_ == 3


def test_perm_is_a_permutation():
    p = perm(12345, 20)
    assert sorted(p) == list(range(20)) and not np.array_equal(p, np.arange(20))
