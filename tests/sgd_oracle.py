"""TEST INFRASTRUCTURE, NOT PRODUCT CODE: the SGD oracle.

sgd_oracle.c restates scikit-learn's _plain_sgd (both dtypes), WeightVector and the xorshift32 shuffle; this module builds
it (into a temporary directory: the source tree is left as it is) and wraps it as SGDClassifier.fit / SGDRegressor.fit do:
the seed draws of fit_binary / _fit_multiclass / _fit_regressor, the label encoding, class weights, one-vs-rest, t_.
Only tests import it.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "sgd_oracle.c")
_LIB = None
MAX_INT = int(np.iinfo(np.int32).max)
LOSSES = ["hinge", "perceptron", "squared_hinge", "modified_huber", "log_loss", "squared_error", "huber",
          "epsilon_insensitive", "squared_epsilon_insensitive"]
PENALTIES = {None: 0, "l1": 1, "l2": 2, "elasticnet": 3}
RATES = {"constant": 1, "optimal": 2, "invscaling": 3, "adaptive": 4}


def _lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha1(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "sgd_oracle_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, i, d, u = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_uint32
        L.oracle_sgd_fit.argtypes = [vp, i, i, i, vp, vp, i, d, i, d, d, i, d, d, d, i, i, i, i, u, d, d, vp, vp, vp]
        L.oracle_sgd_fit.restype = i
        L.oracle_sgd_perm.argtypes = [u, i, vp]
        L.oracle_sgd_perm.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def perm(seed, n):
    """pi: the permutation the shuffle with this seed applies every epoch"""
    out = np.zeros(n, np.int32)
    _lib().oracle_sgd_perm(int(seed), int(n), _p(out))
    return out


def loss_param(loss, epsilon):
    return 0.0 if loss == "perceptron" else (epsilon if LOSSES.index(loss) >= 5 else 1.0)


def fit_one(X, y_enc, sw, seed, wpos=1.0, wneg=1.0, loss="hinge", penalty="l2", alpha=1e-4, l1_ratio=0.15, epsilon=0.1,
            learning_rate="optimal", eta0=0.01, power_t=0.5, tol=1e-3, max_iter=1000, n_iter_no_change=5, fit_intercept=True,
            shuffle=True):
    """one _plain_sgd call -> (coef [d] float64, intercept, n_iter, status: 0 stopped, 1 max_iter, 2 non-finite)"""
    f32 = X.dtype == np.float32
    X = np.ascontiguousarray(X, np.float32 if f32 else np.float64)
    y_enc = np.ascontiguousarray(y_enc, np.float64)
    sw = np.ascontiguousarray(sw, np.float64)
    coef = np.zeros(X.shape[1])
    icpt = np.zeros(1)
    st = np.zeros(1, np.int32)
    it = _lib().oracle_sgd_fit(_p(X), int(f32), X.shape[0], X.shape[1], _p(y_enc), _p(sw), LOSSES.index(loss),
                               loss_param(loss, epsilon), PENALTIES[penalty], float(alpha),
                               float(0.0 if l1_ratio is None else l1_ratio), RATES[learning_rate], float(eta0), float(power_t),
                               -np.inf if tol is None else float(tol), int(max_iter), int(n_iter_no_change),
                               int(bool(fit_intercept)), int(bool(shuffle)), int(seed), float(wpos), float(wneg), _p(coef),
                               _p(icpt), _p(st))
    return coef, float(icpt[0]), int(it), int(st[0])


_FIT_KEYS = ("loss", "penalty", "alpha", "l1_ratio", "epsilon", "learning_rate", "eta0", "power_t", "tol", "max_iter",
             "n_iter_no_change", "fit_intercept", "shuffle")


def classifier_seeds(random_state, n_classes):
    """the shuffle seed of each class fit: binary fit_binary draws make_dataset's seed, then the shuffle seed; one-vs-rest
    first draws one seed per class and each class fit makes the two draws from RandomState(seed)"""
    from sklearn.utils import check_random_state
    rs = check_random_state(random_state)
    if n_classes == 2:
        rs.randint(1, MAX_INT)
        return [int(rs.randint(MAX_INT))]
    out = []
    for s in rs.randint(MAX_INT, size=n_classes):
        r = np.random.RandomState(s)
        r.randint(1, MAX_INT)
        out.append(int(r.randint(MAX_INT)))
    return out


def regressor_seed(random_state):
    """_fit_regressor draws the shuffle seed first, then make_dataset's"""
    from sklearn.utils import check_random_state
    return int(check_random_state(random_state).randint(0, MAX_INT))


class SGDOracle:
    """Fitted SGDClassifier (classes given) / SGDRegressor: coef_, intercept_, n_iter_, t_, status (per class fit).
    seeds: the shuffle seeds (None: drawn from random_state as scikit-learn draws them)."""

    def __init__(self, X, y, classifier=True, random_state=None, sample_weight=None, class_weight=None, seeds=None, **kw):
        from sklearn.linear_model import SGDClassifier, SGDRegressor
        params = (SGDClassifier if classifier else SGDRegressor)().get_params()
        params.update(kw)
        X = np.asarray(X)
        f32 = X.dtype == np.float32
        sw = np.ones(len(X)) if sample_weight is None else np.asarray(sample_weight, np.float64)
        fit_kw = {k: params[k] for k in _FIT_KEYS if k in params}
        if classifier:
            from sklearn.utils.class_weight import compute_class_weight
            self.classes_ = np.unique(y)
            k = len(self.classes_)
            cw = compute_class_weight(class_weight, classes=self.classes_, y=y)
            self.seeds = classifier_seeds(random_state, k) if seeds is None else list(seeds)
            log = fit_kw.get("loss") == "log_loss"
            rows = [(1, cw[1], cw[0])] if k == 2 else [(i, cw[i], 1.0) for i in range(k)]
            res = []
            for (ci, wp, wn), s in zip(rows, self.seeds):
                enc = np.where(y == self.classes_[ci], 1.0, 0.0 if log else -1.0)
                res.append(fit_one(X, enc, sw, s, wp, wn, **fit_kw))
        else:
            self.seeds = [regressor_seed(random_state)] if seeds is None else list(seeds)
            res = [fit_one(X, np.asarray(y, np.float64), sw, self.seeds[0], **fit_kw)]
        dt = np.float32 if f32 else np.float64
        self.coef_ = np.array([r[0] for r in res], dt)
        self.intercept_ = np.array([r[1] for r in res], dt if classifier and len(res) > 1 else np.float64)
        self.status = [r[3] for r in res]
        self.n_iters = [r[2] for r in res]
        self.n_iter_ = max(self.n_iters)
        self.t_ = 1.0 + self.n_iter_ * len(X)
        if not classifier:
            self.coef_ = self.coef_[0]
