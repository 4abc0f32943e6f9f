"""TEST INFRASTRUCTURE, NOT PRODUCT CODE: a CPU restatement of libsvm's epsilon-SVR solver in numpy.

scikit-learn's SVR (sklearn/svm/src/libsvm/svm.cpp, "svm.cpp" below) solves epsilon-SVR as the C-SVC Solver on 2l
variables (solve_epsilon_svr): positions t < l are the rows with y = +1 and linear term eps - z, positions t >= l the same
rows with y = -1 and linear term eps + z; Q_st = y_s y_t (float)K(x_s, x_t) (SVR_Q, Qfloat = float32).  This module follows
that Solver step for step (svm.cpp Solver::Solve, select_working_set, do_shrinking, reconstruct_gradient, calculate_rho),
so it reproduces libsvm's iterate sequence: tests/test_oracle_svr.py pins it bit for bit against sklearn.svm.SVR.

Every float64 operation is a separately rounded numpy elementwise operation or a Python float operation (no fused
multiply-add), in libsvm's order.  The float32 kernel entries are formed as libsvm forms them: float64 kernel value, then
rounded to float32.  Only tests import this module.
"""
import numpy as np

TAU = 1e-12
LOWER, UPPER, FREE = 0, 1, 2


def kernel_rows(X, kernel, gamma):
    """float32 kernel matrix of the rows of X (libsvm Kernel::kernel_linear / kernel_rbf, then (Qfloat))."""
    X = np.asarray(X, np.float64)
    S = X @ X.T
    # the float64 diagonal enters QD unrounded: one BLAS ddot per row, as libsvm's Kernel::dot computes it
    xsq = np.array([np.dot(x, x) for x in X])
    if kernel == "linear":
        return S.astype(np.float32), xsq
    K = np.exp(-gamma * ((xsq[:, None] + xsq[None, :]) - 2 * S))
    return K.astype(np.float32), np.ones(len(X))


def svr_solve(X, z, C, epsilon, kernel="rbf", gamma=1.0, tol=1e-3, shrinking=True, max_iter=-1, K32=None):
    """One epsilon-SVR fit on the rows of X (in the given order) -> (coef [l] = alpha+ - alpha-, rho, n_iter).
    The prediction of the fitted model is sum_k coef_k K(x, x_k) - rho (float64 kernel values)."""
    z = np.asarray(z, np.float64)
    n = len(z)
    if K32 is None:
        K32, qd_rows = kernel_rows(X, kernel, gamma)
    else:
        qd_rows = np.ones(n) if kernel == "rbf" else np.array([np.dot(x, x) for x in np.asarray(X, np.float64)])
    l = 2 * n
    # state by position; orig[pos] = variable index 0..2n-1 (svm.cpp active_set / swap_index)
    orig = np.arange(l)
    y = np.where(orig < n, 1.0, -1.0)
    p = np.concatenate([epsilon - z, epsilon + z])                 # svm.cpp solve_epsilon_svr: linear_term
    alpha = np.zeros(l)
    G = p.copy()                                                     # alpha = 0: G = p
    Gbar = np.zeros(l)
    QD = np.concatenate([qd_rows, qd_rows])
    st = np.full(l, LOWER, np.int8)
    Cv = C

    def row_of(pos):
        return orig[pos] % n

    def q_row(pos, upto):
        """signed float32 Q row of position pos over positions [0, upto), as float64 (exact widening)"""
        r = K32[row_of(pos)][orig[:upto] % n].astype(np.float64)
        return r * (y[pos] * y[:upto])                             # sign flips are exact

    def status(a):
        return UPPER if a >= Cv else (LOWER if a <= 0 else FREE)

    active = l
    unshrink = False

    def reconstruct():
        if active == l:
            return
        G[active:] = Gbar[active:] + p[active:]
        for f in range(active):                                    # both libsvm branches add in ascending free order
            if st[f] == FREE:
                G[active:] += alpha[f] * q_row(f, l)[active:]

    def select():
        Gmax = -np.inf
        gi = -1
        a = slice(0, active)
        yp, s, g = y[a], st[a], G[a]
        up = np.where(yp > 0, s != UPPER, s != LOWER)
        v = np.where(yp > 0, -g, g)
        if up.any():
            cand = np.where(up, v, -np.inf)
            m = cand.max()
            gi = int(np.flatnonzero(cand == m)[-1])              # ">=": the last maximum wins
            Gmax = m
        Qi = q_row(gi, active) if gi >= 0 else None
        low = np.where(yp > 0, s != LOWER, s != UPPER)
        w = np.where(yp > 0, g, -g)
        Gmax2 = w[low].max() if low.any() else -np.inf
        gj = -1
        if gi >= 0:
            gd = Gmax + w
            ok = low & (gd > 0)
            if ok.any():
                quad = np.where(yp > 0, (QD[gi] + QD[a]) - 2.0 * y[gi] * Qi, (QD[gi] + QD[a]) + 2.0 * y[gi] * Qi)
                gd2 = gd * gd
                od = np.where(quad > 0, -gd2 / np.where(quad > 0, quad, 1.0), -gd2 / TAU)
                od = np.where(ok, od, np.inf)
                m = od.min()
                gj = int(np.flatnonzero(od == m)[-1])            # "<=": the last minimum wins
        if Gmax + Gmax2 < tol or gj == -1:
            return None
        return gi, gj

    def be_shrunk(i, g1, g2):
        if st[i] == UPPER:
            return (-G[i] > g1) if y[i] > 0 else (-G[i] > g2)
        if st[i] == LOWER:
            return (G[i] > g2) if y[i] > 0 else (G[i] > g1)
        return False

    def swap(i, j):
        for arr in (orig, y, st, alpha, G, Gbar, p, QD):
            arr[i], arr[j] = arr[j], arr[i]

    def do_shrinking():
        nonlocal active, unshrink
        g1 = g2 = -np.inf
        for i in range(active):
            if y[i] > 0:
                if st[i] != UPPER and -G[i] >= g1: g1 = -G[i]
                if st[i] != LOWER and G[i] >= g2: g2 = G[i]
            else:
                if st[i] != UPPER and -G[i] >= g2: g2 = -G[i]
                if st[i] != LOWER and G[i] >= g1: g1 = G[i]
        if not unshrink and g1 + g2 <= tol * 10:
            unshrink = True
            reconstruct()
            active = l
        i = 0
        while i < active:
            if be_shrunk(i, g1, g2):
                active -= 1
                while active > i:
                    if not be_shrunk(active, g1, g2):
                        swap(i, active)
                        break
                    active -= 1
            i += 1

    it = 0
    counter = min(l, 1000) + 1
    while True:
        if max_iter != -1 and it >= max_iter:
            if active < l:                                           # svm.cpp: reconstruct before calculate_rho
                reconstruct()
                active = l
            break
        counter -= 1
        if counter == 0:
            counter = min(l, 1000)
            if shrinking:
                do_shrinking()
        ij = select()
        if ij is None:
            reconstruct()
            active = l
            ij = select()
            if ij is None:
                break
            counter = 1
        it += 1
        i, j = ij
        Qi, Qj = q_row(i, l), q_row(j, l)
        Ci = Cj = Cv
        oai, oaj = alpha[i], alpha[j]
        ai, aj = float(oai), float(oaj)
        if y[i] != y[j]:
            quad = QD[i] + QD[j] + 2 * Qi[j]
            if quad <= 0: quad = TAU
            delta = (-G[i] - G[j]) / quad
            diff = ai - aj
            ai += delta; aj += delta
            if diff > 0:
                if aj < 0: aj = 0.0; ai = diff
            else:
                if ai < 0: ai = 0.0; aj = -diff
            if diff > Ci - Cj:
                if ai > Ci: ai = Ci; aj = Ci - diff
            else:
                if aj > Cj: aj = Cj; ai = Cj + diff
        else:
            quad = QD[i] + QD[j] - 2 * Qi[j]
            if quad <= 0: quad = TAU
            delta = (G[i] - G[j]) / quad
            s = ai + aj
            ai -= delta; aj += delta
            if s > Ci:
                if ai > Ci: ai = Ci; aj = s - Ci
            else:
                if aj < 0: aj = 0.0; ai = s
            if s > Cj:
                if aj > Cj: aj = Cj; ai = s - Cj
            else:
                if ai < 0: ai = 0.0; aj = s
        alpha[i], alpha[j] = ai, aj
        dai, daj = ai - oai, aj - oaj
        G[:active] += Qi[:active] * dai + Qj[:active] * daj
        ui, uj = st[i] == UPPER, st[j] == UPPER
        st[i], st[j] = status(ai), status(aj)
        if ui != (st[i] == UPPER):
            if ui: Gbar -= Ci * Qi
            else: Gbar += Ci * Qi
        if uj != (st[j] == UPPER):
            if uj: Gbar -= Cj * Qj
            else: Gbar += Cj * Qj
    # calculate_rho
    nfree, ub, lb, ssum = 0, np.inf, -np.inf, 0.0
    for t in range(active):
        yG = y[t] * G[t]
        if st[t] == UPPER:
            if y[t] < 0: ub = min(ub, yG)
            else: lb = max(lb, yG)
        elif st[t] == LOWER:
            if y[t] > 0: ub = min(ub, yG)
            else: lb = max(lb, yG)
        else:
            nfree += 1; ssum += yG
    rho = ssum / nfree if nfree > 0 else (ub + lb) / 2
    a2 = np.zeros(l)
    a2[orig] = alpha
    return a2[:n] - a2[n:], rho, it


def predict(Xtrain, coef, rho, Xq, kernel="rbf", gamma=1.0):
    Xtrain = np.asarray(Xtrain, np.float64); Xq = np.asarray(Xq, np.float64)
    sv = coef != 0
    if kernel == "linear":
        Kq = Xq @ Xtrain[sv].T
    else:
        d2 = ((Xq[:, None, :] - Xtrain[sv][None, :, :]) ** 2).sum(-1)
        Kq = np.exp(-gamma * d2)
    return Kq @ coef[sv] - rho


def r2(ytrue, ypred):
    ytrue = np.asarray(ytrue, np.float64)
    return 1.0 - ((ytrue - ypred) ** 2).sum() / ((ytrue - ytrue.mean()) ** 2).sum()


def cv_scores_svr(X, y, splits, cands, base=None):
    """test r2 and n_iter per (candidate, split); each fit sees X[train] in the order the split lists it"""
    te = np.zeros((len(cands), len(splits)))
    it = np.zeros((len(cands), len(splits)), np.int64)
    for i, c in enumerate(cands):
        p = dict(dict(kernel="rbf", C=1.0, epsilon=0.1, gamma="scale", tol=1e-3, shrinking=True, max_iter=-1), **(base or {}), **c)
        for k, (tr, ts) in enumerate(splits):
            Xtr = np.asarray(X[tr], np.float64)
            g = p["gamma"]
            if g == "scale":
                v = Xtr.var()
                g = 1.0 / (X.shape[1] * v) if v != 0 else 1.0
            elif g == "auto":
                g = 1.0 / X.shape[1]
            coef, rho, n_it = svr_solve(Xtr, y[tr], p["C"], p["epsilon"], p["kernel"], g, p["tol"], p["shrinking"], p["max_iter"])
            te[i, k] = r2(y[ts], predict(Xtr, coef, rho, X[ts], p["kernel"], g))
            it[i, k] = n_it
    return te, it
