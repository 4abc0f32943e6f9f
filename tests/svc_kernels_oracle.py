"""TEST INFRASTRUCTURE, NOT PRODUCT CODE: the C-SVC oracle for the poly and sigmoid kernels.

svc_kernels_oracle.c runs the solver of oracle/svc_oracle.c on a given float32 kernel matrix and float64 diagonal; this
module builds it (into a temporary directory: the source tree is left as it is), forms libsvm's kernel values from one
float64 Gram and assembles the one-vs-one model as oracle.SVCModel does.  Only tests import it.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle.oracle import folds_from_cv, resolve_gamma  # noqa: F401  (re-exported for the tests)

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "svc_kernels_oracle.c")
_BASE = os.path.join(os.path.dirname(_HERE), "oracle", "svc_oracle.c")
KERNEL_ID = {"linear": 0, "rbf": 1, "poly": 2, "sigmoid": 3}
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha1(open(_SRC, "rb").read() + open(_BASE, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "svc_kernels_oracle_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        dp, ip, fp, i, d, lg = (ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_float),
                                ctypes.c_int, ctypes.c_double, ctypes.c_long)
        L.oracle_gram.argtypes = [dp, i, i, dp]
        L.oracle_gram.restype = None
        L.oracle_kernel_from_gram.argtypes = [dp, i, i, d, i, d, fp, dp]
        L.oracle_kernel_from_gram.restype = None
        L.oracle_svc_solve_kqd.argtypes = [fp, lg, dp, ip, i, i, d, d, i, i, dp, dp, ip, dp]
        L.oracle_svc_solve_kqd.restype = ctypes.c_int
        L.oracle_kernel_decision.argtypes = [dp, i, ip, i, dp, d, i, d, i, d, ip, i, dp]
        L.oracle_kernel_decision.restype = None
        _LIB = L
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(ctypes.POINTER(t))


def gram_ddot(X):
    """float64 X X^T with one BLAS ddot per entry: the dot product libsvm's dense Kernel::dot takes in scikit-learn, so the
    kernel values -- and the unrounded diagonal QD -- match its bit for bit.  O(n^2) calls: small problems only."""
    X64 = np.ascontiguousarray(X, np.float64)
    return np.array([[np.dot(a, b) for b in X64] for a in X64])


def gram(X):
    """float64 X X^T, one sequential dot product per entry (fast; differs from gram_ddot in the last bit of a few entries)"""
    X64 = np.ascontiguousarray(X, np.float64)
    n, d = X64.shape
    S = np.empty((n, n))
    _lib().oracle_gram(_p(X64, ctypes.c_double), n, d, _p(S, ctypes.c_double))
    return S


def kernel_matrix(S, kernel, gamma, degree=3, coef0=0.0):
    """(K [n][n] float32, QD [n] float64) of the poly or sigmoid kernel, from the Gram S"""
    S = np.ascontiguousarray(S, np.float64)
    n = len(S)
    K = np.empty((n, n), np.float32)
    QD = np.empty(n)
    _lib().oracle_kernel_from_gram(_p(S, ctypes.c_double), n, KERNEL_ID[kernel], float(gamma), int(degree), float(coef0),
                                   _p(K, ctypes.c_float), _p(QD, ctypes.c_double))
    return K, QD


def solve(K, QD, rows, n_pos, C, tol=1e-3, shrinking=True, max_iter=-1):
    """One binary sub-problem -> (coef [l] = alpha*y in sub-problem order, rho, n_iter)"""
    K = np.ascontiguousarray(K, np.float32)
    QD = np.ascontiguousarray(QD, np.float64)
    rows = np.ascontiguousarray(rows, np.int32)
    coef = np.zeros(len(rows))
    rho, obj, it = ctypes.c_double(), ctypes.c_double(), ctypes.c_int()
    _lib().oracle_svc_solve_kqd(_p(K, ctypes.c_float), K.shape[1], _p(QD, ctypes.c_double), _p(rows, ctypes.c_int), len(rows),
                                int(n_pos), float(C), float(tol), int(bool(shrinking)), int(max_iter), _p(coef, ctypes.c_double),
                                ctypes.byref(rho), ctypes.byref(it), ctypes.byref(obj))
    return coef, rho.value, it.value


def decision(S, rows, coef, rho, kernel, gamma, degree, coef0, trows):
    rows = np.ascontiguousarray(rows, np.int32)
    trows = np.ascontiguousarray(trows, np.int32)
    coef = np.ascontiguousarray(coef, np.float64)
    out = np.zeros(len(trows))
    _lib().oracle_kernel_decision(_p(S, ctypes.c_double), len(S), _p(rows, ctypes.c_int), len(rows), _p(coef, ctypes.c_double),
                                  float(rho), KERNEL_ID[kernel], float(gamma), int(degree), float(coef0),
                                  _p(trows, ctypes.c_int), len(trows), _p(out, ctypes.c_double))
    return out


class KernelSVCModel:
    """Fitted one-vs-one C-SVC with the poly or sigmoid kernel (svm.cpp:2441-2523 training loop, :2821-2904 prediction).
    S: the float64 Gram of all rows; train: the training rows (original order inside each class, as svm_group_classes)."""

    def __init__(self, X, S, y, train, kernel="poly", gamma="scale", C=1.0, degree=3, coef0=0.0, tol=1e-3, shrinking=True,
                 max_iter=-1, KQD=None):
        train = np.asarray(train)
        self.S, self.kernel, self.degree, self.coef0 = S, kernel, int(degree), float(coef0)
        self.classes = np.unique(y[train])
        self.gamma = resolve_gamma(gamma, np.asarray(X, np.float64)[train])
        K, QD = KQD if KQD is not None else kernel_matrix(S, kernel, self.gamma, degree, coef0)
        self.pairs, self.n_iter = [], []
        by_class = [train[y[train] == c] for c in self.classes]
        for a in range(len(self.classes)):
            for b in range(a + 1, len(self.classes)):
                rows = np.concatenate([by_class[a], by_class[b]]).astype(np.int32)
                coef, rho, it = solve(K, QD, rows, len(by_class[a]), C, tol, shrinking, max_iter)
                self.pairs.append((a, b, rows, coef, rho))
                self.n_iter.append(it)

    def decision_pairs(self, rows):
        return np.stack([decision(self.S, r, coef, rho, self.kernel, self.gamma, self.degree, self.coef0, rows)
                         for (_, _, r, coef, rho) in self.pairs], 1)

    def predict(self, rows):
        dec = self.decision_pairs(rows)
        votes = np.zeros((len(rows), len(self.classes)), np.int64)
        for p, (a, b, _, _, _) in enumerate(self.pairs):
            pos = dec[:, p] > 0
            votes[pos, a] += 1
            votes[~pos, b] += 1
        return self.classes[np.argmax(votes, 1)]

    @property
    def n_sv(self):
        """support vectors of the model (a row is counted once even when several pairs use it)"""
        rows = set()
        for (_, _, r, coef, _) in self.pairs:
            rows.update(r[coef != 0].tolist())
        return len(rows)
