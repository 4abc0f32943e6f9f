"""ctypes binding of libb200gs.so (include/b200gs.h) -- the only way the package computes.

There is deliberately no CPU fallback: if the CUDA library is missing or no sm_90 GPU is visible,
``Engine()`` raises.  The oracle under ``oracle/`` is test infrastructure and is never imported here.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200gs.so")

GS_RETURN_TRAIN, GS_GRAM_TENSOR, GS_NO_SHRINKING, GS_TARGET_F32 = 1, 2, 4, 8
KNN_WEIGHTS = {"uniform": 0, "distance": 1}
KNN_METRIC = {"euclidean": 0, "manhattan": 1}
KERNEL_ID = {"linear": 0, "rbf": 1, "poly": 2, "sigmoid": 3}
_PARAM_KERNELS = (2, 3)            # the kernels that read degree / coef0 (gs_set_kernel_params)

_lib = None


class GsProfile(ctypes.Structure):
    _fields_ = [("ms_total", ctypes.c_float), ("ms_h2d", ctypes.c_float), ("ms_gram", ctypes.c_float),
                ("ms_kernel_matrix", ctypes.c_float), ("ms_solve", ctypes.c_float), ("ms_score", ctypes.c_float),
                ("launches", ctypes.c_int64), ("smo_iterations", ctypes.c_int64),
                ("solve_bytes", ctypes.c_double), ("gram_flops", ctypes.c_double), ("gram_bytes", ctypes.c_double),
                ("h2d_bytes", ctypes.c_int64), ("d2h_bytes", ctypes.c_int64),
                ("ms_tensor", ctypes.c_float), ("tensor_flops", ctypes.c_double)]


class EngineError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("libb200gs status %d: %s" % (status, msg))
        self.status = status


def load_library():
    """dlopen libb200gs.so and declare the prototypes of include/b200gs.h.  Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "spark_sklearn_b200: %s is missing -- build it with `python -m spark_sklearn_b200.build` "
            "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    c = ctypes
    vp, i32, i64, u32, dbl = c.c_void_p, c.c_int32, c.c_int64, c.c_uint32, c.c_double
    L.gs_version.restype = c.c_int
    L.gs_device_count.restype = c.c_int
    L.gs_set_splits.argtypes = [vp, vp, vp, i32]
    L.gs_set_splits.restype = c.c_int
    L.gs_set_class_weight.argtypes = [vp, vp, i32]
    L.gs_set_class_weight.restype = c.c_int
    L.gs_set_kernel_params.argtypes = [vp, vp, vp, i32]
    L.gs_set_kernel_params.restype = c.c_int
    L.gs_set_sample_weight.argtypes = [vp, vp]
    L.gs_set_sample_weight.restype = c.c_int
    L.gs_set_scoring.argtypes = [vp, i32, i32]
    L.gs_set_scoring.restype = c.c_int
    L.gs_create.argtypes = [c.c_int, c.POINTER(vp)]
    L.gs_destroy.argtypes = [vp]
    L.gs_destroy.restype = None
    L.gs_last_error.argtypes = [vp]
    L.gs_last_error.restype = c.c_char_p
    L.gs_set_data.argtypes = [vp, vp, i32, i64, i64, vp, vp, vp, i32]
    L.gs_svc.argtypes = [vp, i32, vp, vp, vp, dbl, i32, u32, vp, vp, vp, vp, vp, vp]
    L.gs_svc_refit.argtypes = [vp, i32, dbl, dbl, dbl, i32, u32, vp, vp, vp]
    L.gs_ridge.argtypes = [vp, i32, vp, i32, u32, vp, vp, vp, vp]
    L.gs_ridge_refit.argtypes = [vp, dbl, i32, vp]
    L.gs_enet.argtypes = [vp, i32, vp, vp, i32, dbl, i32, u32, vp, vp, vp, vp, vp]
    L.gs_enet_refit.argtypes = [vp, dbl, dbl, i32, dbl, i32, vp, vp, vp]
    L.gs_set_targets_f64.argtypes = [vp, vp]
    L.gs_svr.argtypes = [vp, i32, vp, vp, vp, vp, dbl, i32, u32, vp, vp, vp, vp, vp, vp]
    L.gs_svr_refit.argtypes = [vp, i32, dbl, dbl, dbl, dbl, i32, u32, vp, vp, vp]
    L.gs_logreg.argtypes = [vp, i32, vp, dbl, i32, i32, u32, vp, vp, vp, vp, vp]
    L.gs_logreg_refit.argtypes = [vp, dbl, dbl, i32, i32, vp, vp]
    L.gs_linsvc.argtypes = [vp, i32, vp, dbl, i32, i32, dbl, u32, vp, vp, vp, vp, vp]
    L.gs_linsvc_refit.argtypes = [vp, dbl, dbl, i32, i32, dbl, vp, vp]
    L.gs_debug_gemm_f64.argtypes = [vp, vp, i32, vp, i32, i32, vp]
    L.gs_knn.argtypes = [vp, i32, vp, vp, vp, u32, vp, vp, vp, vp]
    L.gs_debug_knn_neighbors.argtypes = [vp, i32, i32, i32, vp, vp]
    L.gs_get_profile.argtypes = [vp, c.POINTER(GsProfile)]
    L.gs_debug_gram.argtypes = [vp, vp, vp]
    L.gs_debug_kernel_matrix.argtypes = [vp, i32, dbl, vp, vp, vp]
    L.gs_debug_decision.argtypes = [vp, i32, dbl, i32, dbl, vp, i32, i32, vp, vp]
    L.gs_debug_score.argtypes = [vp, i32, vp, vp, i32, vp, vp, i32, vp]
    L.gs_debug_gemm_nt.argtypes = [vp, vp, i32, vp, i32, i32, vp]
    L.gs_svc_predicted_iterations.argtypes = [i32, dbl, dbl, i32]
    L.gs_svc_predicted_iterations.restype = dbl
    L.gs_svc_cluster_count.argtypes = [vp, i32, i32]
    L.gs_svc_cluster_count.restype = i32
    L.gs_svc_schedule.argtypes = [vp, i32, i32, vp, vp]
    L.gs_svc_schedule.restype = None
    for f in ("gs_create", "gs_set_data", "gs_svc", "gs_svc_refit", "gs_ridge", "gs_ridge_refit", "gs_enet", "gs_enet_refit", "gs_set_targets_f64",
              "gs_svr", "gs_svr_refit", "gs_logreg",
              "gs_logreg_refit", "gs_linsvc", "gs_linsvc_refit", "gs_get_profile", "gs_debug_gram", "gs_debug_kernel_matrix",
              "gs_debug_decision", "gs_debug_score", "gs_debug_gemm_nt", "gs_debug_gemm_f64", "gs_knn", "gs_debug_knn_neighbors"):
        getattr(L, f).restype = c.c_int
    _lib = L
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


_device_count = None


def device_count():
    """sm_90 GPUs visible to this process (0 without a GPU or without the library's CUDA runtime); asked once per process."""
    global _device_count
    if _device_count is None:
        _device_count = int(load_library().gs_device_count())
    return _device_count


class Engine:
    """One handle = one GPU (reference analogue: the SparkContext `sc`, util.py:51-58)."""

    def __init__(self, device=None):
        self._L = load_library()
        if device is None:
            device = int(os.environ.get("LOCAL_RANK", "0"))
        h = ctypes.c_void_p()
        st = self._L.gs_create(int(device), ctypes.byref(h))
        if st != 0:
            raise EngineError(st, (self._L.gs_last_error(None) or b"").decode())
        self._h = h
        self.device = int(device)
        self.n = self.d = self.n_splits = 0

    def close(self):
        if getattr(self, "_h", None):
            self._L.gs_destroy(self._h)
            self._h = None

    __del__ = close

    def _check(self, st):
        if st != 0:
            raise EngineError(st, (self._L.gs_last_error(self._h) or b"").decode())

    def set_splits(self, test_mask, train_mask, n_splits):
        """General CV splits (include/b200gs.h gs_set_splits): uint64 [n][2] membership masks, after set_data."""
        te = np.ascontiguousarray(test_mask, np.uint64)
        tr = np.ascontiguousarray(train_mask, np.uint64)
        assert te.shape == (self.n, 2) and tr.shape == (self.n, 2)
        self.n_splits = int(n_splits)
        self._check(self._L.gs_set_splits(self._h, _ptr(te), _ptr(tr), int(n_splits)))

    def set_class_weight(self, w=None):
        """[n_sets][n_classes] class weights of the following svc / svc_refit calls (None: all ones)."""
        if w is None:
            self._check(self._L.gs_set_class_weight(self._h, None, 0))
            return
        w = np.ascontiguousarray(np.atleast_2d(w), np.float64)
        self._check(self._L.gs_set_class_weight(self._h, _ptr(w), w.shape[0]))

    def set_sample_weight(self, w=None):
        """fit_params={'sample_weight': w} of the following ridge / enet / logreg calls (None: unweighted)"""
        if w is None:
            self._check(self._L.gs_set_sample_weight(self._h, None))
            return
        w = np.ascontiguousarray(w, np.float64)
        if w.shape != (self.n,):
            raise ValueError("sample_weight has shape %r; expected (%d,)" % (w.shape, self.n))
        self._check(self._L.gs_set_sample_weight(self._h, _ptr(w)))

    def set_scoring(self, kind=0, pos_class=1):
        """Scorer of the following search calls (include/b200gs.h GS_SCORE_*): reference base_search.py:43 check_scoring."""
        self._check(self._L.gs_set_scoring(self._h, int(kind), int(pos_class)))

    # -- the "broadcast" (reference base_search.py:63-65) --
    def set_data(self, X, fold_id, n_splits, y_class=None, y_target=None):
        X = np.ascontiguousarray(X, np.float32 if np.asarray(X).dtype == np.float32 else np.float64)
        fold_id = np.ascontiguousarray(fold_id, np.int8)
        yc = None if y_class is None else np.ascontiguousarray(y_class, np.int32)
        yt = None if y_target is None else np.ascontiguousarray(y_target, np.float32)
        self.n, self.d = X.shape
        self.n_splits = int(n_splits)
        self.n_classes = 0 if yc is None else int(yc.max()) + 1
        self._check(self._L.gs_set_data(self._h, _ptr(X), 0 if X.dtype == np.float32 else 1, X.shape[0], X.shape[1], _ptr(yc), _ptr(yt),
                                        _ptr(fold_id), int(n_splits)))

    # -- map(fun).collect() for SVC and epsilon-SVR (reference base_search.py:74-95) --
    def _kernel_svm(self, fn, kernel, C, per_cand, gamma, tol, max_iter, shrinking, return_train, flags):
        """gs_svc / gs_svr: kernel names or ids, C and the estimator's other per-candidate arrays (per_cand), gamma per
        candidate or per (candidate, split) -> the per-(candidate, split) outputs"""
        kernel = np.ascontiguousarray([KERNEL_ID[k] if isinstance(k, str) else int(k) for k in kernel], np.int32)
        C = np.ascontiguousarray(C, np.float64)
        n_cand = len(C)
        gamma = np.ascontiguousarray(np.broadcast_to(np.asarray(gamma, np.float64).reshape(n_cand, -1),
                                                     (n_cand, self.n_splits)))
        shape = (n_cand, self.n_splits)
        out = dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.zeros(shape, np.int32),
                   n_sv=np.zeros(shape, np.int32), fit_ms=np.zeros(shape, np.float32),
                   score_ms=np.zeros(shape, np.float32))
        fl = int(flags) | (GS_RETURN_TRAIN if return_train else 0) | (0 if shrinking else GS_NO_SHRINKING)
        self._check(fn(self._h, n_cand, _ptr(kernel), _ptr(C), *[_ptr(a) for a in per_cand], _ptr(gamma), float(tol),
                       int(max_iter), fl, _ptr(out["test"]), _ptr(out["train"]), _ptr(out["n_iter"]), _ptr(out["n_sv"]),
                       _ptr(out["fit_ms"]), _ptr(out["score_ms"])))
        if not return_train:
            out["train"] = None
        return out

    def _with_kernel_params(self, kernel_ids, degree, coef0, call):
        """call() with gs_set_kernel_params set to degree / coef0 (scalars or one per candidate) when a poly or sigmoid
        candidate is present, reset afterwards; a call without one sets nothing"""
        if not any(k in _PARAM_KERNELS for k in kernel_ids):
            return call()
        n = len(kernel_ids)
        deg = np.ascontiguousarray(np.broadcast_to(np.asarray(3 if degree is None else degree, np.int64), (n,)), np.int32)
        c0 = np.ascontiguousarray(np.broadcast_to(np.asarray(0.0 if coef0 is None else coef0, np.float64), (n,)))
        self._check(self._L.gs_set_kernel_params(self._h, _ptr(deg), _ptr(c0), n))
        try:
            return call()
        finally:
            self._L.gs_set_kernel_params(self._h, None, None, 0)

    def svc(self, kernel, C, gamma, tol=1e-3, max_iter=-1, shrinking=True, return_train=True, flags=0, degree=None, coef0=None):
        """degree / coef0: scalars or one per candidate, read by the poly and sigmoid candidates (defaults 3 / 0.0)"""
        ids = [KERNEL_ID[k] if isinstance(k, str) else int(k) for k in kernel]
        return self._with_kernel_params(ids, degree, coef0, lambda: self._kernel_svm(
            self._L.gs_svc, ids, C, [], gamma, tol, max_iter, shrinking, return_train, flags))

    def svc_refit(self, kernel, C, gamma, n_classes, tol=1e-3, max_iter=-1, shrinking=True, degree=3, coef0=0.0):
        n_pairs = n_classes * (n_classes - 1) // 2
        coef = np.zeros((n_pairs, self.n))
        rho = np.zeros(n_pairs)
        it = np.zeros(n_pairs, np.int32)
        k = KERNEL_ID[kernel] if isinstance(kernel, str) else int(kernel)
        self._with_kernel_params([k], degree, coef0, lambda: self._check(self._L.gs_svc_refit(
            self._h, k, float(C), float(gamma), float(tol), int(max_iter), 0 if shrinking else GS_NO_SHRINKING, _ptr(coef),
            _ptr(rho), _ptr(it))))
        return coef, rho, it

    def set_targets_f64(self, y):
        """float64 regression targets [n] (caller's row order) of the following svr / svr_refit calls, after set_data"""
        y = np.ascontiguousarray(y, np.float64)
        if y.shape != (self.n,):
            raise ValueError("y has shape %r; expected (%d,)" % (y.shape, self.n))
        self._check(self._L.gs_set_targets_f64(self._h, _ptr(y)))

    def svr(self, kernel, C, epsilon, gamma, tol=1e-3, max_iter=-1, shrinking=True, return_train=True, flags=0):
        epsilon = np.ascontiguousarray(np.broadcast_to(np.asarray(epsilon, np.float64), (len(C),)))
        return self._kernel_svm(self._L.gs_svr, kernel, C, [epsilon], gamma, tol, max_iter, shrinking, return_train, flags)

    def svr_refit(self, kernel, C, epsilon, gamma, tol=1e-3, max_iter=-1, shrinking=True, flags=0):
        """-> (coef [n] by row: alpha+ - alpha-, rho, n_iter); prediction = sum coef k(x, x_row) - rho"""
        coef = np.zeros(self.n)
        rho = np.zeros(1)
        it = np.zeros(1, np.int32)
        k = KERNEL_ID[kernel] if isinstance(kernel, str) else int(kernel)
        fl = int(flags) | (0 if shrinking else GS_NO_SHRINKING)
        self._check(self._L.gs_svr_refit(self._h, k, float(C), float(epsilon), float(gamma), float(tol), int(max_iter),
                                         fl, _ptr(coef), _ptr(rho), _ptr(it)))
        return coef, float(rho[0]), int(it[0])

    def ridge(self, alpha, fit_intercept=True, return_train=True):
        alpha = np.ascontiguousarray(alpha, np.float64)
        shape = (len(alpha), self.n_splits)
        out = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape, np.float32),
                   score_ms=np.zeros(shape, np.float32))
        self._check(self._L.gs_ridge(self._h, len(alpha), _ptr(alpha), int(bool(fit_intercept)),
                                     GS_RETURN_TRAIN if return_train else 0, _ptr(out["test"]), _ptr(out["train"]),
                                     _ptr(out["fit_ms"]), _ptr(out["score_ms"])))
        if not return_train:
            out["train"] = None
        return out

    def ridge_refit(self, alpha, fit_intercept=True):
        coef = np.zeros(self.d + 1)
        self._check(self._L.gs_ridge_refit(self._h, float(alpha), int(bool(fit_intercept)), _ptr(coef)))
        return coef[:-1].copy(), float(coef[-1])

    def enet(self, alpha, l1_ratio, fit_intercept=True, tol=1e-4, max_iter=1000, return_train=True):
        alpha = np.ascontiguousarray(alpha, np.float64)
        l1_ratio = np.ascontiguousarray(np.broadcast_to(np.asarray(l1_ratio, np.float64), alpha.shape))
        shape = (len(alpha), self.n_splits)
        out = dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.zeros(shape, np.int32),
                   fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32))
        self._check(self._L.gs_enet(self._h, len(alpha), _ptr(alpha), _ptr(l1_ratio), int(bool(fit_intercept)), float(tol),
                                    int(max_iter), GS_RETURN_TRAIN if return_train else 0, _ptr(out["test"]), _ptr(out["train"]),
                                    _ptr(out["n_iter"]), _ptr(out["fit_ms"]), _ptr(out["score_ms"])))
        if not return_train:
            out["train"] = None
        return out

    def enet_refit(self, alpha, l1_ratio=1.0, fit_intercept=True, tol=1e-4, max_iter=1000):
        coef = np.zeros(self.d + 1)
        it = np.zeros(1, np.int32)
        gap = np.zeros(1)
        self._check(self._L.gs_enet_refit(self._h, float(alpha), float(l1_ratio), int(bool(fit_intercept)), float(tol),
                                          int(max_iter), _ptr(coef), _ptr(it), _ptr(gap)))
        return coef[:-1].copy(), float(coef[-1]), int(it[0]), float(gap[0])

    def logreg(self, C, tol=1e-4, max_iter=100, fit_intercept=True, return_train=True):
        C = np.ascontiguousarray(C, np.float64)
        shape = (len(C), self.n_splits)
        out = dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.zeros(shape, np.int32),
                   fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32))
        self._check(self._L.gs_logreg(self._h, len(C), _ptr(C), float(tol), int(max_iter), int(bool(fit_intercept)),
                                      GS_RETURN_TRAIN if return_train else 0, _ptr(out["test"]), _ptr(out["train"]),
                                      _ptr(out["n_iter"]), _ptr(out["fit_ms"]), _ptr(out["score_ms"])))
        if not return_train:
            out["train"] = None
        return out

    def logreg_refit(self, C, tol=1e-4, max_iter=100, fit_intercept=True):
        """-> (coef, intercept, n_iter): binary [d], float; three or more classes (multinomial) [n_classes][d], [n_classes]"""
        rows = self.n_classes if self.n_classes > 2 else 1
        coef = np.zeros((rows, self.d + 1))
        it = np.zeros(1, np.int32)
        self._check(self._L.gs_logreg_refit(self._h, float(C), float(tol), int(max_iter), int(bool(fit_intercept)),
                                            _ptr(coef), _ptr(it)))
        if rows == 1:
            return coef[0, :-1].copy(), float(coef[0, -1]), int(it[0])
        return coef[:, :-1].copy(), coef[:, -1].copy(), int(it[0])

    def linsvc(self, C, tol=1e-4, max_iter=1000, fit_intercept=True, intercept_scaling=1.0, return_train=True):
        """LinearSVC (squared hinge, L2, primal TRON) per (candidate, split); n_iter = LinearSVC.n_iter_ of each fit"""
        C = np.ascontiguousarray(C, np.float64)
        shape = (len(C), self.n_splits)
        out = dict(test=np.zeros(shape), train=np.zeros(shape), n_iter=np.zeros(shape, np.int32),
                   fit_ms=np.zeros(shape, np.float32), score_ms=np.zeros(shape, np.float32))
        self._check(self._L.gs_linsvc(self._h, len(C), _ptr(C), float(tol), int(max_iter), int(bool(fit_intercept)),
                                      float(intercept_scaling), GS_RETURN_TRAIN if return_train else 0, _ptr(out["test"]),
                                      _ptr(out["train"]), _ptr(out["n_iter"]), _ptr(out["fit_ms"]), _ptr(out["score_ms"])))
        if not return_train:
            out["train"] = None
        return out

    def linsvc_refit(self, C, tol=1e-4, max_iter=1000, fit_intercept=True, intercept_scaling=1.0):
        """-> (raw [rows][d + 1]: liblinear's weights, the bias feature's last; n_iter [rows]); rows = 1 (binary) or n_classes"""
        rows = self.n_classes if self.n_classes > 2 else 1
        raw = np.zeros((rows, self.d + 1))
        it = np.zeros(rows, np.int32)
        self._check(self._L.gs_linsvc_refit(self._h, float(C), float(tol), int(max_iter), int(bool(fit_intercept)),
                                            float(intercept_scaling), _ptr(raw), _ptr(it)))
        return raw, it

    def knn(self, n_neighbors, weights, metric, return_train=True, y_f32=False):
        """k-NN scores per (candidate, split) from one neighbour selection per metric (include/b200gs.h gs_knn); weights and
        metric are names (KNN_WEIGHTS, KNN_METRIC) or codes.  NaN where n_neighbors exceeds the split's training rows."""
        nn = np.ascontiguousarray(n_neighbors, np.int32)
        w = np.ascontiguousarray([KNN_WEIGHTS[v] if isinstance(v, str) else int(v) for v in weights], np.int32)
        m = np.ascontiguousarray([KNN_METRIC[v] if isinstance(v, str) else int(v) for v in metric], np.int32)
        shape = (len(nn), self.n_splits)
        out = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape, np.float32),
                   score_ms=np.zeros(shape, np.float32))
        fl = (GS_RETURN_TRAIN if return_train else 0) | (GS_TARGET_F32 if y_f32 else 0)
        self._check(self._L.gs_knn(self._h, len(nn), _ptr(nn), _ptr(w), _ptr(m), fl, _ptr(out["test"]), _ptr(out["train"]),
                                   _ptr(out["fit_ms"]), _ptr(out["score_ms"])))
        if not return_train:
            out["train"] = None
        return out

    # -- test hooks --
    def debug_knn_neighbors(self, metric, k, split):
        """-> (idx [n][k] original row indices, -1 past the split's training rows; dist [n][k]): the sorted neighbour lists
        gs_knn votes from, every row against the training rows of split `split`"""
        idx = np.zeros((self.n, k), np.int32)
        dist = np.zeros((self.n, k))
        m = KNN_METRIC[metric] if isinstance(metric, str) else int(metric)
        self._check(self._L.gs_debug_knn_neighbors(self._h, m, int(k), int(split), _ptr(idx), _ptr(dist)))
        return idx, dist

    def debug_gram(self):
        S = np.zeros((self.n, self.n))
        xsq = np.zeros(self.n)
        self._check(self._L.gs_debug_gram(self._h, _ptr(S), _ptr(xsq)))
        return S, xsq

    def debug_kernel_matrix(self, kernel, gamma, degree=3, coef0=0.0, return_guard=False):
        """K [n][n] float32; with return_guard: (K, qd, flag), qd the float64 diagonal (poly / sigmoid, else None) and flag
        the kernel-matrix kernel's guard (1: K holds a zero, subnormal, negative or non-finite value)"""
        K = np.zeros((self.n, self.n), np.float32)
        k = KERNEL_ID[kernel] if isinstance(kernel, str) else int(kernel)
        qd = np.zeros(self.n) if return_guard and k in _PARAM_KERNELS else None
        flag = np.zeros(1, np.int32) if return_guard else None
        self._with_kernel_params([k], degree, coef0, lambda: self._check(self._L.gs_debug_kernel_matrix(
            self._h, k, float(gamma), _ptr(K), _ptr(qd), _ptr(flag))))
        return (K, qd, int(flag[0])) if return_guard else K

    def debug_decision(self, kernel, gamma, coef, degree=3, coef0=0.0, jchunks=0):
        """coef [ncols][n] -> (dec [ncols][n] float64 decision values, slab count used); jchunks 0 = the search's choice"""
        coef = np.ascontiguousarray(np.atleast_2d(coef), np.float64)
        if coef.shape[1] != self.n:
            raise ValueError("debug_decision: coef has %d columns; expected n = %d" % (coef.shape[1], self.n))
        dec = np.zeros_like(coef)
        used = np.zeros(1, np.int32)
        k = KERNEL_ID[kernel] if isinstance(kernel, str) else int(kernel)
        self._check(self._L.gs_debug_decision(self._h, k, float(gamma), int(degree), float(coef0), _ptr(coef), coef.shape[0],
                                              int(jchunks), _ptr(dec), _ptr(used)))
        return dec, int(used[0])

    SCORE_KINDS = {"vote": 0, "class_counts": 1, "auc_f64": 2, "auc_f32": 3, "rss": 4}

    def debug_score(self, kind, dec, rho, first_col, fold):
        """One scorer kernel (include/b200gs.h gs_debug_score) on dec [ncols][n] and rho [ncols] for the tasks
        (first_col[t], fold[t]) -> vote [t][4] int32, class_counts [t][2][n_classes][3] int32, auc_f64 / auc_f32 [t][4]
        uint64, rss [t][2] float64"""
        k = self.SCORE_KINDS[kind]
        dec = np.ascontiguousarray(np.atleast_2d(dec), np.float64)
        rho = None if rho is None else np.ascontiguousarray(rho, np.float64)
        first_col = np.ascontiguousarray(first_col, np.int32)
        fold = np.ascontiguousarray(fold, np.int32)
        t = len(first_col)
        if fold.shape != (t,) or dec.shape[1] != self.n or (rho is not None and rho.shape != (dec.shape[0],)):
            raise ValueError("debug_score: first_col / fold / dec / rho shapes disagree")
        if kind == "vote":
            out = np.zeros((t, 4), np.int32)
        elif kind == "class_counts":
            out = np.zeros((t, 2, self.n_classes, 3), np.int32)
        elif kind == "rss":
            out = np.zeros((t, 2))
        else:
            out = np.zeros((t, 4), np.uint64)
        self._check(self._L.gs_debug_score(self._h, k, _ptr(dec), _ptr(rho), dec.shape[0], _ptr(first_col), _ptr(fold), t,
                                           _ptr(out)))
        return out

    def debug_gemm_nt(self, A, B):
        A = np.ascontiguousarray(A, np.float32)
        B = np.ascontiguousarray(B, np.float32)
        C = np.zeros((A.shape[0], B.shape[0]), np.float32)
        self._check(self._L.gs_debug_gemm_nt(self._h, _ptr(A), A.shape[0], _ptr(B), B.shape[0], A.shape[1], _ptr(C)))
        return C

    def debug_gemm_f64(self, A, B):
        A = np.ascontiguousarray(A, np.float64)
        B = np.ascontiguousarray(B, np.float64)
        C = np.zeros((A.shape[0], B.shape[0]))
        self._check(self._L.gs_debug_gemm_f64(self._h, _ptr(A), A.shape[0], _ptr(B), B.shape[0], A.shape[1], _ptr(C)))
        return C

    def profile(self):
        p = GsProfile()
        self._check(self._L.gs_get_profile(self._h, ctypes.byref(p)))
        return {k: getattr(p, k) for k, _ in GsProfile._fields_}
