"""TEST INFRASTRUCTURE, NOT PRODUCT CODE: the LinearSVC oracle.

linsvc_oracle.c restates liblinear's primal squared-hinge solver (train / train_one / l2r_l2_svc_fun / TRON) in float64; this
module builds it (into a temporary directory: the source tree is left as it is) and wraps it as scikit-learn's _fit_liblinear
does (LabelEncoder, compute_class_weight, bias = intercept_scaling, intercept_ = intercept_scaling x the bias weight).  Only
tests import it.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "linsvc_oracle.c")
TRACE_W = 10
TRACE_FIELDS = ("iter", "accepted", "actred", "prered", "delta", "f", "gnorm", "cg_iter", "snorm", "fnew")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha1(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "linsvc_oracle_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, i, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
        L.oracle_linsvc_train.argtypes = [vp, i, i, vp, vp, i, d, vp, d, d, i, vp, vp, vp, i, vp]
        L.oracle_linsvc_train.restype = ctypes.c_int
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class LinearSVCOracle:
    """Fitted LinearSVC(penalty='l2', loss='squared_hinge', dual=False): coef_, intercept_, n_iter_ (max over one-vs-rest
    fits), n_iter_per_fit, and trace[fit] = a list of per-iteration dicts (TRACE_FIELDS) when trace=True."""

    def __init__(self, X, y, C=1.0, tol=1e-4, max_iter=1000, fit_intercept=True, intercept_scaling=1.0, class_weight=None,
                 sample_weight=None, trace=False, trace_cap=4096):
        from sklearn.preprocessing import LabelEncoder
        from sklearn.utils.class_weight import compute_class_weight
        X = np.ascontiguousarray(X, np.float64)
        enc = LabelEncoder()
        y_ind = enc.fit_transform(y).astype(np.int32)
        self.classes_ = enc.classes_
        sw = np.ones(len(X)) if sample_weight is None else np.ascontiguousarray(sample_weight, np.float64)
        cw = np.ascontiguousarray(compute_class_weight(class_weight, classes=self.classes_, y=y, sample_weight=sample_weight),
                                  np.float64)
        nc = len(self.classes_)
        rows = 1 if nc == 2 else nc
        bias = float(intercept_scaling) if fit_intercept else -1.0
        n = X.shape[1] + (1 if fit_intercept else 0)
        raw = np.zeros((rows, n))
        it = np.zeros(rows, np.int32)
        tr = np.zeros((rows, trace_cap, TRACE_W)) if trace else None
        tl = np.zeros(rows, np.int32)
        st = _lib().oracle_linsvc_train(_p(X), X.shape[0], X.shape[1], _p(np.ascontiguousarray(y_ind)), _p(sw), nc, float(C),
                                        _p(cw), bias, float(tol), int(max_iter), _p(raw), _p(it),
                                        None if tr is None else _p(tr), trace_cap, _p(tl))
        if st != 0:
            raise ValueError("a class has no row of positive weight")
        self.raw_coef_ = raw
        self.coef_ = raw[:, :X.shape[1]]
        self.intercept_ = intercept_scaling * raw[:, -1] if fit_intercept else 0.0
        self.n_iter_per_fit = it
        self.n_iter_ = int(it.max())
        self.trace = None if tr is None else [[dict(zip(TRACE_FIELDS, rec)) for rec in tr[q, :tl[q]]] for q in range(rows)]

    def decision_function(self, X):
        d = np.asarray(X, np.float64) @ self.coef_.T + self.intercept_
        return d[:, 0] if d.shape[1] == 1 else d

    def predict(self, X):
        d = self.decision_function(X)
        return self.classes_[(d > 0).astype(int)] if d.ndim == 1 else self.classes_[np.argmax(d, 1)]
