"""TEST INFRASTRUCTURE, NOT PRODUCT CODE: the nu-SVC / nu-SVR oracle.

nu_oracle.c restates libsvm's Solver_NU; this module builds it (into a temporary directory: the source tree is left as it
is) and does what scikit-learn's svm.cpp does around it: the float32 kernel values (tests/svr_oracle.py kernel_rows), the
one-vs-one pairs and the set-up of solve_nu_svc (C = 1 per row, nu_l = sum of nu x C in row order, the greedy starting
alpha per sign, then alpha y / r and rho / r) and solve_nu_svr (2l variables, linear term -/+ z, C per variable, the halved
sum of C x nu handed out greedily to both copies of a row), and the feasibility check of svm_check_parameter.  The fitted
models are assembled by the package's own materialize_svc / materialize_svr.  tests/test_oracle_nu.py pins it against
sklearn.svm.NuSVC / NuSVR.  Only tests import it.
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from svr_oracle import kernel_rows

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "nu_oracle.c")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha1(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "nu_oracle_%d_%s.so" % (os.getuid(), h))
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        vp, i, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
        L.oracle_nu_solve.argtypes = [vp, vp, vp, vp, vp, vp, i, d, i, i, i, vp, vp, vp]
        L.oracle_nu_solve.restype = ctypes.c_int
        _LIB = L
    return _LIB


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def solve(K, QD, y, p, C, alpha, tol, shrinking, max_iter, rebuild_at_stop=False):
    """One Solver_NU solve -> (alpha, rho, r, n_iter, timed_out)"""
    K = np.ascontiguousarray(K, np.float32)
    QD, p, C = (np.ascontiguousarray(a, np.float64) for a in (QD, p, C))
    y = np.ascontiguousarray(y, np.int8)
    alpha = np.array(alpha, np.float64)
    rho, r, to = ctypes.c_double(), ctypes.c_double(), ctypes.c_int()
    it = _lib().oracle_nu_solve(_ptr(K), _ptr(QD), _ptr(y), _ptr(p), _ptr(C), _ptr(alpha), len(y), float(tol),
                                int(bool(shrinking)), int(max_iter), int(bool(rebuild_at_stop)), ctypes.byref(rho),
                                ctypes.byref(r), ctypes.byref(to))
    return alpha, rho.value, r.value, it, bool(to.value)


def _greedy(total, C):
    """alpha_i = min(C_i, remaining) in order (solve_nu_svc / solve_nu_svr)"""
    a = np.zeros(len(C))
    for i, c in enumerate(C):
        a[i] = min(c, total)
        total -= a[i]
    return a


def nusvc_infeasible(nu, y_class):
    """svm_check_parameter: nu (n1 + n2) / 2 > min(n1, n2) for some pair of the classes present"""
    n = [float(c) for c in np.bincount(y_class) if c > 0]
    return any(nu * (n[a] + n[b]) / 2 > min(n[a], n[b]) for a in range(len(n)) for b in range(a + 1, len(n)))


def nusvc_fit(X, y_class, nu, kernel="rbf", gamma=1.0, tol=1e-3, shrinking=True, max_iter=-1, rebuild_at_stop=False):
    """One NuSVC fit -> (pair_coef [n_pairs][n] = alpha y / r by row, rho [n_pairs] = rho / r, n_iter [n_pairs]).
    y_class: class indices 0..k-1 (scikit-learn's sorted classes)."""
    if nusvc_infeasible(nu, y_class):
        raise ValueError("specified nu is infeasible")
    K, QD = kernel_rows(X, kernel, gamma)
    nc = int(y_class.max()) + 1
    n = len(X)
    coef, rhos, its = [], [], []
    for a in range(nc):
        for b in range(a + 1, nc):
            rows = np.concatenate([np.flatnonzero(y_class == a), np.flatnonzero(y_class == b)])
            l, na = len(rows), int((y_class == a).sum())
            yy = np.where(np.arange(l) < na, 1, -1)
            C = np.ones(l)
            nu_l = 0.0
            for c in C:
                nu_l += nu * c
            alpha = np.concatenate([_greedy(nu_l / 2, C[:na]), _greedy(nu_l / 2, C[na:])])
            al, rho, r, it, _ = solve(K[np.ix_(rows, rows)], QD[rows], yy, np.zeros(l), C, alpha, tol, shrinking, max_iter,
                                      rebuild_at_stop)
            pc = np.zeros(n)
            pc[rows] = al * (yy / r)                                  # svm.cpp:1701: alpha[i] *= y[i] / r
            coef.append(pc)
            rhos.append(rho / r)
            its.append(it)
    return np.array(coef), np.array(rhos), np.array(its, np.int32)


def nusvr_fit(X, z, nu, C=1.0, kernel="rbf", gamma=1.0, tol=1e-3, shrinking=True, max_iter=-1, rebuild_at_stop=False):
    """One NuSVR fit -> (coef [n] = alpha+ - alpha-, rho, n_iter)"""
    z = np.asarray(z, np.float64)
    K, QD = kernel_rows(X, kernel, gamma)
    l = len(X)
    Cv = np.full(l, float(C))
    s = 0.0
    for c in Cv:
        s += c * nu
    s /= 2
    a = _greedy(s, Cv)
    alpha = np.concatenate([a, a])
    K2 = np.block([[K, K], [K, K]])
    y2 = np.concatenate([np.ones(l), -np.ones(l)])
    al, rho, _, it, _ = solve(K2, np.concatenate([QD, QD]), y2, np.concatenate([-z, z]), np.concatenate([Cv, Cv]), alpha,
                              tol, shrinking, max_iter, rebuild_at_stop)
    return al[:l] - al[l:], rho, it
