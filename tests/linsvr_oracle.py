"""TEST INFRASTRUCTURE, NOT PRODUCT CODE: the LinearSVR oracle.

linsvr_oracle.c restates liblinear's SVR solvers (11: TRON on l2r_l2_svr_fun; 12 / 13: solve_l2r_l1l2_svr, the dual
coordinate descent), train's zero-weight removal, std::mt19937 and bounded_rand_int in float64; this module builds it (into
a temporary directory: the source tree is left as it is) and wraps it as scikit-learn's LinearSVR.fit / _fit_liblinear do
(dual resolution, the solver of (loss, dual), the seed drawn from random_state, bias = intercept_scaling).  Only tests
import it.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "linsvr_oracle.c")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha1(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "linsvr_oracle_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, i, d, u = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_uint32
        L.oracle_linsvr_train.argtypes = [vp, i, i, vp, vp, d, d, d, d, i, i, u, i, vp, vp]
        L.oracle_linsvr_train.restype = ctypes.c_int
        L.oracle_mt_draws.argtypes = [u, i, vp]
        L.oracle_mt_draws.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def mt_draws(seed, k):
    """the first k outputs of std::mt19937(seed)"""
    out = np.zeros(k, np.uint32)
    _lib().oracle_mt_draws(int(seed), int(k), _p(out))
    return out


def solver_of(loss, dual, n_rows, n_features):
    """scikit-learn's _validate_dual_parameter on a training set of n_rows x n_features, then _get_liblinear_solver_type"""
    from sklearn.svm._base import _get_liblinear_solver_type
    from sklearn.svm._classes import _validate_dual_parameter
    dual = _validate_dual_parameter(dual, loss, "l2", "ovr", np.empty((n_rows, n_features), np.bool_))
    return _get_liblinear_solver_type("ovr", "l2", loss, dual)


def seed_of(random_state):
    """the seed _fit_liblinear hands to liblinear: check_random_state(random_state).randint(np.iinfo('i').max)"""
    from sklearn.utils import check_random_state
    return int(check_random_state(random_state).randint(np.iinfo("i").max))


class LinearSVROracle:
    """Fitted LinearSVR: coef_, intercept_, n_iter_, raw_coef_ (liblinear's w, the bias weight last), solver, seed, steps
    (coordinate steps of the CD).  seed: the liblinear seed (None: drawn from random_state as scikit-learn draws it).
    kernel_order: sum the CD dot products in csrc/linsvr.cu's order."""

    def __init__(self, X, y, C=1.0, epsilon=0.0, loss="epsilon_insensitive", dual="auto", tol=1e-4, max_iter=1000,
                 fit_intercept=True, intercept_scaling=1.0, random_state=None, sample_weight=None, seed=None,
                 kernel_order=False):
        X = np.ascontiguousarray(X, np.float64)
        y = np.ascontiguousarray(y, np.float64)
        sw = np.ones(len(X)) if sample_weight is None else np.ascontiguousarray(sample_weight, np.float64)
        self.solver = solver_of(loss, dual, X.shape[0], X.shape[1])
        self.seed = seed_of(random_state) if seed is None else int(seed)
        bias = float(intercept_scaling) if fit_intercept else -1.0
        n = X.shape[1] + (1 if fit_intercept else 0)
        raw = np.zeros(n)
        steps = np.zeros(1, np.int64)
        it = _lib().oracle_linsvr_train(_p(X), X.shape[0], X.shape[1], _p(y), _p(sw), float(C), float(epsilon), bias,
                                        float(tol), int(max_iter), int(self.solver), self.seed, int(bool(kernel_order)),
                                        _p(raw), _p(steps))
        if it < 0:
            raise ValueError("no row has positive weight")
        self.raw_coef_ = raw
        self.coef_ = raw[:X.shape[1]].copy()
        self.intercept_ = intercept_scaling * raw[X.shape[1]:] if fit_intercept else 0.0
        self.n_iter_ = int(it)
        self.steps = int(steps[0])

    def predict(self, X):
        return np.asarray(X, np.float64) @ self.coef_ + self.intercept_
