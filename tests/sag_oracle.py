"""TEST INFRASTRUCTURE, NOT PRODUCT CODE: the SAG / SAGA oracle.

sag_oracle.c restates scikit-learn's sag64 / sag32 and our_rand_r; this module builds it (into a temporary directory: the
source tree is left as it is) and wraps it as scikit-learn calls it: sag_solver's scaled penalties and step size, and
LogisticRegression.fit's penalty resolution, class x sample weights in X's dtype, label encoding and make_dataset's seed
draw.  Only tests import it.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "sag_oracle.c")
_LIB = None
MAX_INT = int(np.iinfo(np.int32).max)
LOSSES = {"log": 0, "multinomial": 1, "squared": 2}


def _lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha1(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "sag_oracle_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, i, d, u = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_uint32
        for f in (L.oracle_sag64, L.oracle_sag32):
            f.argtypes = [vp, i, i, i, vp, vp, i, i, d, d, d, d, i, i, u, vp, vp, vp]
            f.restype = i
        L.oracle_sag_draws.argtypes = [u, i, i, vp]
        L.oracle_sag_draws.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def draws(seed, n, count):
    """the first count sample positions dataset.random draws over n rows"""
    out = np.zeros(int(count), np.int32)
    _lib().oracle_sag_draws(int(seed), int(n), int(count), _p(out))
    return out


def sag_fit(X, y, sw, loss, step, alpha_scaled, beta_scaled, seed, saga=False, tol=1e-3, max_iter=1000, fit_intercept=True,
            n_classes=1):
    """one sag64 / sag32 call (X's dtype) -> (coef [n_classes][d + 1] float64: weights then intercept, n_iter, status:
    0 stopped, 1 max_iter, 2 non-finite, sample steps)"""
    dt = np.float32 if X.dtype == np.float32 else np.float64
    X = np.ascontiguousarray(X, dt)
    y = np.ascontiguousarray(y, dt)
    sw = np.ascontiguousarray(sw, dt)
    coef = np.zeros((n_classes, X.shape[1] + 1))
    st = np.zeros(1, np.int32)
    steps = np.zeros(1, np.int64)
    fn = _lib().oracle_sag32 if dt == np.float32 else _lib().oracle_sag64
    it = fn(_p(X), X.shape[0], X.shape[1], int(n_classes), _p(y), _p(sw), LOSSES[loss], int(bool(saga)), float(step),
            float(alpha_scaled), float(beta_scaled), float(tol), int(max_iter), int(bool(fit_intercept)), int(seed), _p(coef),
            _p(st), _p(steps))
    return coef, int(it), int(st[0]), int(steps[0])


def resolve_penalty(C, l1_ratio, penalty="deprecated"):
    """LogisticRegression.fit / _logistic_regression_path: (alpha, beta) of sag_solver before the 1 / n scaling"""
    if penalty == "deprecated":
        pen = "l2" if l1_ratio in (0, None) else ("l1" if l1_ratio == 1 else "elasticnet")
        if C == np.inf:
            pen = None
    else:
        pen = penalty
    if penalty is None:
        C = np.inf
        pen = "l2"
    if pen == "l1":
        return 0.0, 1.0 / C
    if pen == "l2":
        return 1.0 / C, 0.0
    return (1.0 / C) * (1 - l1_ratio), (1.0 / C) * l1_ratio


def problem(X, y, sample_weight=None, class_weight=None):
    """(classes, dataset y in X's dtype, sample weights in X's dtype, loss, n_classes) as _logistic_regression_path sets
    them up"""
    from sklearn.utils.class_weight import compute_class_weight
    dt = np.float32 if X.dtype == np.float32 else np.float64
    classes, enc = np.unique(y, return_inverse=True)
    sw = None
    if sample_weight is not None or class_weight is not None:
        sw = np.ones(len(X), dt) if sample_weight is None else np.asarray(sample_weight).astype(dt)
    if class_weight is not None:
        cw = compute_class_weight(class_weight, classes=classes, y=y, sample_weight=sw)
        sw = sw * cw[enc].astype(dt)
    if sw is None:
        sw = np.ones(len(X), dt)
    if len(classes) == 2:
        return classes, (enc == 1).astype(dt), sw, "log", 1
    return classes, enc.astype(dt), sw, "multinomial", len(classes)


def make_dataset_seed(random_state):
    from sklearn.utils import check_random_state
    return int(check_random_state(random_state).randint(1, MAX_INT))


def step_and_penalties(X, C, l1_ratio, solver, fit_intercept, loss, penalty="deprecated"):
    """(step, alpha_scaled, beta_scaled) as sag_solver computes them for LogisticRegression"""
    from sklearn.linear_model._sag import get_auto_step_size
    from sklearn.utils.extmath import row_norms
    alpha, beta = resolve_penalty(C, l1_ratio, penalty)
    n = X.shape[0]
    a, b = float(alpha) / n, float(beta) / n
    mss = row_norms(X, squared=True).max()
    return get_auto_step_size(mss, a, loss, fit_intercept, n_samples=n, is_saga=solver == "saga"), a, b


class SAGOracle:
    """Fitted LogisticRegression(solver='sag' | 'saga'): coef_, intercept_ (X's dtype), n_iter_, status, steps.
    seed: make_dataset's draw (None: drawn from random_state as scikit-learn draws it)."""

    def __init__(self, X, y, sample_weight=None, seed=None, **kw):
        from sklearn.linear_model import LogisticRegression
        p = LogisticRegression().get_params()
        p.update(kw)
        X = np.asarray(X)
        dt = np.float32 if X.dtype == np.float32 else np.float64
        self.classes_, yd, sw, loss, K = problem(X, y, sample_weight, p["class_weight"])
        step, a, b = step_and_penalties(X, p["C"], p["l1_ratio"], p["solver"], p["fit_intercept"], loss, p["penalty"])
        self.seed = make_dataset_seed(p["random_state"]) if seed is None else int(seed)
        coef, self.n_iter, self.status, self.steps = sag_fit(X, yd, sw, loss, step, a, b, self.seed, p["solver"] == "saga",
                                                            p["tol"], p["max_iter"], p["fit_intercept"], K)
        d = X.shape[1]
        self.coef_ = coef[:, :d].astype(dt)
        self.intercept_ = coef[:, d].astype(dt) if p["fit_intercept"] else np.zeros(K, dt)
        self.n_iter_ = np.array([self.n_iter], np.int32)
