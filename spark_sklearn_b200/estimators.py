"""Estimator adapters: turn (estimator, candidate dicts, folds) into the scalar tables the C ABI takes,
and turn refit buffers back into genuine fitted scikit-learn estimators for ``best_estimator_``
(reference base_search.py:165-174 delegates ``predict`` & co. to it).

Only estimators with a CUDA path are accepted (SVC with the linear, rbf, poly and sigmoid kernels, SVR rbf/linear, Ridge,
Lasso / ElasticNet, LogisticRegression, LinearSVC with the primal squared-hinge solver -- the families the reference ships
examples for -- and KNeighborsClassifier / KNeighborsRegressor); anything else raises: no CPU fallback.
"""
import numbers
import warnings

import numpy as np
from sklearn.base import clone

from .engine import Engine, EngineError

_ENGINES = {}


def get_engine(device=None):
    """One cached handle per device: GPU allocations stay warm across searches."""
    import os
    dev = int(os.environ.get("LOCAL_RANK", "0")) if device is None else int(device)
    if dev not in _ENGINES:
        _ENGINES[dev] = Engine(dev)
    return _ENGINES[dev]


def fold_ids_from_splits(splits, n):
    """fold_id[row] = index of the split whose TEST set holds the row -- the compact form for the splitters every
    (Stratified)KFold/GroupKFold/LeaveOneOut-style cv gives: disjoint test sets whose complement is the training set.
    Raises NotImplementedError for any other splitter (see split_masks)."""
    if len(splits) > 127:
        raise NotImplementedError("more than 127 CV splits")
    fold_id = np.full(n, -1, np.int8)
    seen = np.zeros(n, bool)
    for k, (tr, te) in enumerate(splits):
        te = np.asarray(te)
        if np.any(fold_id[te] != -1):
            raise NotImplementedError("CV splitter with overlapping test sets needs split masks")
        fold_id[te] = k
        # train == complement of test  <=>  sizes add up to n, no row twice, none of them a test row
        seen[:] = False
        seen[te] = True
        seen[np.asarray(tr)] = True
        if len(tr) + len(te) != n or not seen.all():
            raise NotImplementedError("CV splitter whose train set is not the complement of its test set needs split masks")
    return fold_id


def split_masks(splits, n):
    """(test_mask, train_mask): uint64 [n][2], bit k of word k // 64 = the row belongs to the test / training set of split k
    (include/b200gs.h gs_set_splits).  The general form of the reference's per-task index arrays (base_search.py:81-82): fits
    ShuffleSplit, RepeatedKFold, PredefinedSplit with -1 entries ... up to 128 splits."""
    if len(splits) > 128:
        raise NotImplementedError("more than 128 CV splits")
    te_m = np.zeros((n, 2), np.uint64)
    tr_m = np.zeros((n, 2), np.uint64)
    for k, (tr, te) in enumerate(splits):
        bit = np.uint64(1) << np.uint64(k & 63)
        te_m[np.asarray(te, np.int64), k >> 6] |= bit
        tr_m[np.asarray(tr, np.int64), k >> 6] |= bit
    if np.any(te_m & tr_m):
        raise ValueError("a row is in both the training and the test set of a CV split")
    return te_m, tr_m


class Folds:
    """The CV splits of one search in the forms the engine takes: fold ids when the splits are a partition (every estimator),
    split masks otherwise (SVC, LogisticRegression)."""

    def __init__(self, splits, n):
        self.n_splits = len(splits)
        self.n = n
        try:
            self.fold_id = fold_ids_from_splits(splits, n)
            self.masks = None
        except NotImplementedError:
            self.fold_id = None
            self.masks = split_masks(splits, n)

    @property
    def partition(self):
        return self.fold_id is not None

    def train_rows(self, k):
        """boolean [n]: the training rows of split k (all rows for k < 0)"""
        if k < 0:
            return np.ones(self.n, bool)
        if self.fold_id is not None:
            return self.fold_id != k
        return (self.masks[1][:, k >> 6] >> np.uint64(k & 63)) & np.uint64(1) == 1


def adapter_for(estimator):
    from sklearn.linear_model import ElasticNet, Lasso, LogisticRegression, Ridge
    from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor
    from sklearn.pipeline import Pipeline
    from sklearn.svm import SVC, SVR, LinearSVC
    t = type(estimator)
    if t is SVC:
        return SVCAdapter
    if t is SVR:
        return SVRAdapter
    if t is Ridge:
        return RidgeAdapter
    if t is LogisticRegression:
        return LogRegAdapter
    if t in (Lasso, ElasticNet):
        return ENetAdapter
    if t is LinearSVC:
        return LinearSVCAdapter
    if t in (KNeighborsClassifier, KNeighborsRegressor):
        return KNeighborsAdapter if t is KNeighborsClassifier else KNeighborsRegressorAdapter
    if t is Pipeline and len(estimator.steps) == 1:
        # the reference's own search tests wrap the estimator in a one-step Pipeline and search 'step__param'
        # (python/spark_sklearn/tests/test_search_2.py:69-93): the step's adapter runs, the names are translated
        return PipelineAdapter(estimator.steps[0][0], adapter_for(estimator.steps[0][1]))
    raise NotImplementedError(
        "spark_sklearn_b200 has CUDA paths for SVC, SVR, Ridge, Lasso, ElasticNet, LogisticRegression, LinearSVC, "
        "KNeighborsClassifier and KNeighborsRegressor (bare or as the only step of a Pipeline); got %s (no CPU fallback)"
        % t.__name__)


def _as_matrix(X):
    import scipy.sparse as sp
    if sp.issparse(X):
        X = X.toarray()                               # the engine is dense (SURVEY.md 8: small dense data)
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError("X must be 2-dimensional")
    if X.dtype == np.float32:
        return np.ascontiguousarray(X)
    return np.ascontiguousarray(X, np.float64)        # scikit-learn upcasts everything else to float64


def _pad_scores(arr_list, my):
    return None if not my else np.concatenate(arr_list, 0)


# scoring= names with a fused CUDA scorer (include/b200gs.h GS_SCORE_*); None = the estimator's own score
CLASSIFICATION_SCORERS = {None: 0, "accuracy": 0, "balanced_accuracy": 1, "f1": 2, "precision": 3, "recall": 4, "roc_auc": 5,
                          "f1_macro": 6, "f1_micro": 7, "f1_weighted": 8}
REGRESSION_SCORERS = {None: 0, "r2": 0, "neg_mean_squared_error": 16, "neg_root_mean_squared_error": 17}


class _Plan:
    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        self.estimator, self.cands = estimator, cands
        self.X, self.y, self.n_splits = _as_matrix(X), y, n_splits
        if isinstance(fold_id, Folds):
            self.folds, self.fold_id = fold_id, fold_id.fold_id
        else:
            self.folds, self.fold_id = None, fold_id
        self.engine = get_engine(device)
        self._prof = {}
        self.score_kind, self.score_pos = 0, 1

    def profile(self):
        return dict(self._prof)

    def _set_data(self, X, **kw):
        """gs_set_data (+ gs_set_splits when the splits are no partition)"""
        if self.folds is not None and not self.folds.partition:
            if not self.general_splits:
                raise NotImplementedError("%s needs a CV splitter whose test sets partition the rows (KFold-like); the fold-Gram "
                                          "algorithm has no CUDA path for %d overlapping / partial splits"
                                          % (type(self.estimator).__name__, self.n_splits))
            self.engine.set_data(X, np.full(len(X), -1, np.int8), self.n_splits, **kw)
            self.engine.set_splits(self.folds.masks[0], self.folds.masks[1], self.n_splits)
        else:
            self.engine.set_data(X, self.fold_id, self.n_splits, **kw)

    general_splits = True
    supports_sample_weight = False

    def set_fit_params(self, fit_params):
        """reference base_search.py:69,83-87: fit_params go to every task's estimator.fit.  The CUDA paths take
        sample_weight (Ridge, Lasso, ElasticNet, LogisticRegression); anything else has no device counterpart."""
        fit_params = dict(fit_params or {})
        sw = fit_params.pop("sample_weight", None)
        if fit_params:
            raise NotImplementedError("fit_params %s have no CUDA path (sample_weight does)" % sorted(fit_params))
        if sw is not None and not self.supports_sample_weight:
            raise NotImplementedError("sample_weight has no CUDA path for %s (class_weight does)" % type(self.estimator).__name__)
        self.sample_weight = None if sw is None else np.asarray(sw, np.float64)
        if self.sample_weight is not None and self.sample_weight.shape != (len(self.X),):
            raise ValueError("sample_weight has shape %r; expected (%d,)" % (self.sample_weight.shape, len(self.X)))
        self.engine.set_sample_weight(self.sample_weight)

    def _class_weights(self, cw, k):
        """scikit-learn's class_weight_ of one fit (svm/_base.py, linear_model/_logistic.py: compute_class_weight(class_weight, classes, y_train)):
        None -> ones; dict -> by label (missing labels 1.0); 'balanced' -> n / (n_classes * bincount) on the TRAINING rows of
        split k (k < 0: all rows)."""
        from sklearn.utils.class_weight import compute_class_weight
        rows = self._train_rows(k)
        sw = getattr(self, "sample_weight", None)        # 'balanced' counts the classes by weight (_logistic.py:431-433)
        return compute_class_weight(cw, classes=self.classes, y=np.asarray(self.y)[rows],
                                    sample_weight=None if sw is None else sw[rows])

    def _set_class_weight(self, cw, refit=False):
        if cw is None:
            self.engine.set_class_weight(None)
            return np.ones(len(self.classes))
        ks = [-1] if refit else range(self.n_splits)
        w = np.stack([self._class_weights(cw, k) for k in ks])
        self.engine.set_class_weight(w)
        return w[0]

    def _train_rows(self, k):
        if self.folds is not None:
            return self.folds.train_rows(k)
        return self.fold_id != k if k >= 0 else np.ones(len(self.fold_id), bool)

    scorers = {None: 0}

    def set_scoring(self, scoring):
        """reference base_search.py:43: check_scoring(estimator, scoring).  Only scorers with a fused CUDA path are accepted
        (strings; callables and multi-metric dicts would need the fitted estimator on the host: no CPU fallback)."""
        if scoring is not None and not isinstance(scoring, str):
            raise NotImplementedError("scoring must be None or a scorer name; callables / multi-metric scoring have no CUDA path")
        if scoring not in self.scorers:
            raise NotImplementedError("scoring=%r has no CUDA path for %s (available: %s)" % (
                scoring, type(self.estimator).__name__, sorted(k for k in self.scorers if k)))
        self.score_kind, self.score_pos = self.scorers[scoring], 1
        if self.score_kind in (2, 3, 4):                      # precision / recall / f1: scikit-learn's pos_label=1
            classes = list(getattr(self, "classes", []))
            if len(classes) != 2:
                raise ValueError("Target is multiclass but average='binary'. Please choose another average setting")
            if 1 not in classes:
                raise ValueError("pos_label=1 is not a valid label. It should be one of %s" % classes)
            self.score_pos = classes.index(1)
        elif self.score_kind == 5 and len(getattr(self, "classes", [])) != 2:
            raise NotImplementedError("scoring='roc_auc' has a CUDA path for binary problems only")

    def costs(self):
        """Predicted relative cost of every candidate (None: all alike) -- used to balance candidates over GPUs."""
        return None

    def close(self):
        pass

    def _base_params(self, cand):
        base = getattr(self, "_est_params", None)
        if base is None:                                  # the search's estimator is fixed: introspect it once, not per candidate
            base = self._est_params = self.estimator.get_params(deep=False)
        p = dict(base)
        unknown = set(cand) - set(p)
        if unknown:
            raise ValueError("Invalid parameter(s) %s for estimator %s" % (sorted(unknown), self.estimator))
        p.update(cand)
        return p

    def _finish(self, res, return_train, error_score, n_my):
        test, train = res["test"], res.get("train")
        bad = ~np.isfinite(test)
        if bad.any():
            if error_score == 'raise':
                raise FloatingPointError("non-finite score from the CUDA path")
            warnings.warn("non-finite scores replaced by error_score=%r" % (error_score,))
            test[bad] = error_score
            if train is not None:
                train[~np.isfinite(train)] = error_score
        return dict(test=test, train=train if return_train else None,
                    fit_time=res["fit_ms"] * 1e-3, score_time=res["score_ms"] * 1e-3)


# ------------------------------------------------------------------ SVC -----------------------
class SVCAdapter:
    multi_device = True        # plan(..., device=d): one plan per GPU of the in-process scheduler
    scorers = CLASSIFICATION_SCORERS

    @staticmethod
    def plan(estimator, cands, X, y, fold_id, n_splits, device=None):
        return SVCPlan(estimator, cands, X, y, fold_id, n_splits, device)


class _KernelGamma:
    """What the SVC and SVR plans share: the gamma of one libsvm fit (sklearn svm/_base.py:278-286) and the Gram mode."""

    def _gamma(self, g, k):
        """'scale' uses the variance of the TRAINING fold (float64); k < 0: all rows."""
        if isinstance(g, str):
            if g == "auto":
                return 1.0 / self.X.shape[1]
            if g == "scale":
                cache = self.__dict__.setdefault("_var_cache", {})
                if k not in cache:
                    cache[k] = np.asarray(self.X[self._train_rows(k)], np.float64).var()
                v = cache[k]
                return 1.0 / (self.X.shape[1] * v) if v != 0 else 1.0
            raise ValueError("gamma=%r" % (g,))
        if not (isinstance(g, numbers.Real) and g >= 0):
            raise ValueError("gamma must be >= 0 or 'scale'/'auto'; got %r" % (g,))
        return float(g)

    def _flags(self):
        import os
        # B200GS_GRAM=tensor: opt-in wgmma Gram (fp32-faithful; scores match to solver tolerance, not bit for bit)
        return 2 if os.environ.get("B200GS_GRAM", "exact") == "tensor" else 0


class SVCPlan(_KernelGamma, _Plan):
    """sklearn.svm.SVC (C-SVC).  Scalars per candidate: kernel, C, gamma (resolved per fold for every kernel but linear),
    degree and coef0 (poly, sigmoid)."""
    scorers = CLASSIFICATION_SCORERS

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("SVC needs y")
        self.classes, self.y_class = np.unique(np.asarray(y), return_inverse=True)
        if len(self.classes) < 2:
            raise ValueError("The number of classes has to be greater than one; got %d class" % len(self.classes))
        self._set_data(self.X, y_class=self.y_class.astype(np.int32))
        self._var_cache = {}

    def _check(self, p):
        if p["kernel"] not in ("rbf", "linear", "poly", "sigmoid"):
            raise NotImplementedError("SVC kernel=%r has no CUDA path (linear, rbf, poly and sigmoid do)" % (p["kernel"],))
        # scikit-learn's parameter constraints (SVC._parameter_constraints), checked whatever the kernel
        if not (isinstance(p["degree"], numbers.Integral) and p["degree"] >= 0):
            raise ValueError("The 'degree' parameter of SVC must be an int in the range [0, inf); got %r" % (p["degree"],))
        if not isinstance(p["coef0"], numbers.Real):
            raise ValueError("The 'coef0' parameter of SVC must be a float; got %r" % (p["coef0"],))
        if p["degree"] > np.iinfo(np.int32).max:
            raise NotImplementedError("SVC degree=%r: the CUDA path takes a 32-bit degree" % (p["degree"],))
        if p.get("probability") not in (False, "deprecated", None):
            raise NotImplementedError("SVC probability=True is not supported by the CUDA path")
        if p.get("break_ties"):
            raise NotImplementedError("SVC break_ties=True is not supported by the CUDA path")
        if not (isinstance(p["C"], numbers.Real) and p["C"] > 0):
            raise ValueError("C must be a positive number; got %r" % (p["C"],))

    def costs(self):
        """Predicted SMO iterations per candidate from the library's own model (gs_svc_predicted_iterations: the one
        gs_svc orders its sub-problems by)."""
        from .engine import load_library, KERNEL_ID
        L = load_library()
        d = self.X.shape[1]
        out = np.ones(len(self.cands))
        try:
            for i, cand in enumerate(self.cands):
                p = self._base_params(cand)
                g = self._gamma(p["gamma"], -1) if p["kernel"] == "rbf" else 0.0
                out[i] = L.gs_svc_predicted_iterations(KERNEL_ID[p["kernel"]], float(p["C"]), float(g), int(d))
        except Exception:
            return None                                 # invalid candidates are reported by evaluate()
        return out

    def evaluate(self, my, return_train=True, error_score='raise'):
        ns = self.n_splits
        shape = (len(my), ns)
        res = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape), score_ms=np.zeros(shape),
                   n_iter=np.zeros(shape, np.int64))
        groups = {}
        params = []
        for j, ci in enumerate(my):
            p = self._base_params(self.cands[ci])
            self._check(p)
            params.append(p)
            cw = p.get("class_weight")
            cwk = None if cw is None else (cw if isinstance(cw, str) else tuple(sorted(cw.items())))
            groups.setdefault((float(p["tol"]), int(p["max_iter"]), bool(p["shrinking"]), cwk), []).append(j)
        prof = {}
        for (tol, max_iter, shrinking, _cwk), idx in groups.items():
            self._set_class_weight(params[idx[0]].get("class_weight"))
            kern = [params[j]["kernel"] for j in idx]
            C = [float(params[j]["C"]) for j in idx]
            gam = np.array([[self._gamma(params[j]["gamma"], k) if params[j]["kernel"] != "linear" else 0.0
                             for k in range(ns)] for j in idx])
            self.engine.set_scoring(self.score_kind, self.score_pos)
            r = self.engine.svc(kern, C, gam, tol=tol, max_iter=max_iter, shrinking=shrinking,
                                return_train=return_train, flags=self._flags(),
                                degree=[int(params[j]["degree"]) for j in idx], coef0=[float(params[j]["coef0"]) for j in idx])
            for key in ("test", "fit_ms", "score_ms", "n_iter"):
                res[key][idx] = r[key]
            if return_train:
                res["train"][idx] = r["train"]
            for k, v in self.engine.profile().items():
                prof[k] = prof.get(k, 0) + v
        self.engine.set_class_weight(None)
        self._prof = prof
        self.n_iter_ = res["n_iter"]
        return self._finish(res, return_train, error_score, len(my))

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        gamma = self._gamma(p["gamma"], -1)          # all rows train (svm/_base.py:278-286)
        cw_ = self._set_class_weight(p.get("class_weight"), refit=True)
        coef, rho, n_iter = self.engine.svc_refit(p["kernel"], p["C"], gamma if p["kernel"] != "linear" else 0.0,
                                                  len(self.classes), tol=p["tol"], max_iter=p["max_iter"],
                                                  shrinking=p["shrinking"], degree=int(p["degree"]), coef0=float(p["coef0"]))
        self.engine.set_class_weight(None)
        est = clone(self.estimator).set_params(**best_params)
        est = materialize_svc(est, self.X, self.y_class, self.classes, coef, rho, n_iter, gamma)
        est.class_weight_ = np.asarray(cw_, np.float64)
        return est


def materialize_svc(est, X, y_class, classes, pair_coef, rho, n_iter, gamma):
    """Fill a (cloned, parametrised) sklearn.svm.SVC with the fitted state libsvm would have produced
    (sklearn svm.cpp:2529-2640 model assembly; svm/_base.py:300-327 attribute post-processing)."""
    n_class = len(classes)
    X64 = np.ascontiguousarray(X, np.float64)
    order = np.argsort(y_class, kind="stable")                    # svm_group_classes: by class, stable
    nonzero = np.any(pair_coef != 0, axis=0)
    sv = order[nonzero[order]]                                    # SV rows in libsvm's grouped order
    sv_class = y_class[sv]
    n_support = np.array([(sv_class == c).sum() for c in range(n_class)], np.int32)
    dual = np.zeros((n_class - 1, len(sv)))
    p = 0
    for i in range(n_class):
        for j in range(i + 1, n_class):
            mi, mj = sv_class == i, sv_class == j
            dual[j - 1, mi] = pair_coef[p, sv[mi]]                # svm.cpp:2611-2632
            dual[i, mj] = pair_coef[p, sv[mj]]
            p += 1
    est.classes_ = classes
    est.class_weight_ = np.ones(n_class)
    est._sparse = False
    est._gamma = float(gamma)
    est.support_ = sv.astype(np.int32)
    est.support_vectors_ = X64[sv]
    est._n_support = n_support
    est._dual_coef_ = dual
    est._intercept_ = -np.asarray(rho, np.float64)                # libsvm wrapper stores -rho
    est.dual_coef_ = dual.copy()
    est.intercept_ = est._intercept_.copy()
    if n_class == 2:                                              # svm/_base.py:305-308
        est.intercept_ *= -1
        est.dual_coef_ = -est.dual_coef_
    est._probA = np.empty(0)
    est._probB = np.empty(0)
    est._effective_probability = False
    est.fit_status_ = 0
    est._num_iter = np.asarray(n_iter, np.int32)
    est.n_iter_ = est._num_iter
    est.shape_fit_ = X.shape
    est.n_features_in_ = X.shape[1]
    return est


# ------------------------------------------------------------------ SVR -----------------------
class SVRAdapter:
    multi_device = True        # plan(..., device=d): one plan per GPU of the in-process scheduler
    scorers = REGRESSION_SCORERS

    @staticmethod
    def plan(estimator, cands, X, y, fold_id, n_splits, device=None):
        return SVRPlan(estimator, cands, X, y, fold_id, n_splits, device)


class SVRPlan(_KernelGamma, _Plan):
    """sklearn.svm.SVR (epsilon-SVR).  Scalars per candidate: kernel, C, epsilon, gamma (resolved per fold).  Each fit runs
    libsvm's solver on its training rows in ascending row order, as scikit-learn's X[train] does for KFold-like splitters."""
    scorers = REGRESSION_SCORERS

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("SVR needs y")
        y = np.asarray(y)
        if y.ndim == 2 and y.shape[1] == 1:               # scikit-learn: column_or_1d(y, warn=True)
            from sklearn.exceptions import DataConversionWarning
            warnings.warn("A column-vector y was passed when a 1d array was expected. Please change the shape of y to "
                          "(n_samples, ), for example using ravel().", DataConversionWarning, stacklevel=2)
            y = y[:, 0]
        if y.ndim != 1:
            raise ValueError("SVR needs a 1d target; got y of shape %r" % (y.shape,))
        self.y = y.astype(np.float64)                     # scikit-learn fits SVR on float64 y
        self._set_data(self.X, y_target=self.y.astype(np.float32))
        self.engine.set_targets_f64(self.y)

    def _check(self, p):
        if p["kernel"] not in ("rbf", "linear"):
            raise NotImplementedError("SVR kernel=%r has no CUDA path (rbf and linear do)" % (p["kernel"],))
        if not (isinstance(p["C"], numbers.Real) and p["C"] > 0):
            raise ValueError("C must be a positive number; got %r" % (p["C"],))
        if not (isinstance(p["epsilon"], numbers.Real) and p["epsilon"] >= 0):
            raise ValueError("epsilon must be a non-negative number; got %r" % (p["epsilon"],))

    max_rows = 8192        # training rows of one fit: 2 x 8192 solver variables, the largest resident-state SMO instance

    def _check_rows(self, k):
        m = int(np.count_nonzero(self._train_rows(k)))
        if m > self.max_rows:
            raise NotImplementedError("SVR fit on %d training rows: the CUDA solver handles up to %d" % (m, self.max_rows))

    def check_refit(self):
        """the refit trains on every row: raise before the search when that fit is too large"""
        self._check_rows(-1)

    def evaluate(self, my, return_train=True, error_score='raise'):
        ns = self.n_splits
        shape = (len(my), ns)
        res = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape), score_ms=np.zeros(shape),
                   n_iter=np.zeros(shape, np.int64))
        for k in range(ns):
            self._check_rows(k)
        groups = {}
        params = []
        for j, ci in enumerate(my):
            p = self._base_params(self.cands[ci])
            self._check(p)
            params.append(p)
            groups.setdefault((float(p["tol"]), int(p["max_iter"]), bool(p["shrinking"])), []).append(j)
        prof = {}
        for (tol, max_iter, shrinking), idx in groups.items():
            kern = [params[j]["kernel"] for j in idx]
            C = [float(params[j]["C"]) for j in idx]
            eps = [float(params[j]["epsilon"]) for j in idx]
            gam = np.array([[self._gamma(params[j]["gamma"], k) if params[j]["kernel"] == "rbf" else 0.0
                             for k in range(ns)] for j in idx])
            self.engine.set_scoring(self.score_kind, self.score_pos)
            r = self.engine.svr(kern, C, eps, gam, tol=tol, max_iter=max_iter, shrinking=shrinking,
                                return_train=return_train, flags=self._flags())
            for key in ("test", "fit_ms", "score_ms", "n_iter"):
                res[key][idx] = r[key]
            if return_train:
                res["train"][idx] = r["train"]
            for k, v in self.engine.profile().items():
                prof[k] = prof.get(k, 0) + v
        self._prof = prof
        self.n_iter_ = res["n_iter"]
        return self._finish(res, return_train, error_score, len(my))

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        self._check_rows(-1)
        gamma = self._gamma(p["gamma"], -1)          # all rows train (svm/_base.py:278-286)
        coef, rho, n_iter = self.engine.svr_refit(p["kernel"], p["C"], p["epsilon"], gamma if p["kernel"] == "rbf" else 0.0,
                                                  tol=p["tol"], max_iter=p["max_iter"], shrinking=p["shrinking"],
                                                  flags=self._flags())
        est = clone(self.estimator).set_params(**best_params)
        est = materialize_svr(est, self.X, coef, rho, n_iter, gamma)
        if p["max_iter"] != -1 and n_iter >= p["max_iter"]:        # svm/_base.py: fit_status_ 1 and its warning
            from sklearn.exceptions import ConvergenceWarning
            est.fit_status_ = 1
            warnings.warn("Solver terminated early (max_iter=%i).  Consider pre-processing your data with StandardScaler "
                          "or MinMaxScaler." % p["max_iter"], ConvergenceWarning)
        return est


def materialize_svr(est, X, coef, rho, n_iter, gamma):
    """Fill a (cloned, parametrised) sklearn.svm.SVR with the fitted state libsvm would have produced for epsilon-SVR
    (svm.cpp svm_train: support vectors = rows with a non-zero coefficient, ascending; sklearn _libsvm.pyx fit: _n_support
    = [n_SV, n_SV] for regression; svm/_base.py fit: intercept_ = -rho, n_iter_ a plain int)."""
    X64 = np.ascontiguousarray(X, np.float64)
    coef = np.asarray(coef, np.float64)
    sv = np.flatnonzero(coef != 0)
    est._sparse = False
    est._gamma = np.float64(gamma)
    est.support_ = sv.astype(np.int32)
    est.support_vectors_ = X64[sv]
    est._n_support = np.array([len(sv), len(sv)], np.int32)
    est._dual_coef_ = coef[sv].reshape(1, -1)
    est._intercept_ = np.array([-float(rho)])
    est.dual_coef_ = est._dual_coef_.copy()
    est.intercept_ = est._intercept_.copy()
    est._probA = np.empty(0)
    est._probB = np.empty(0)
    est._effective_probability = False
    est.fit_status_ = 0
    est._num_iter = np.array([n_iter], np.int32)
    est.n_iter_ = int(n_iter)
    est.shape_fit_ = X.shape
    est.n_features_in_ = X.shape[1]
    return est


# ------------------------------------------------------------------ Ridge ---------------------
class RidgeAdapter:
    multi_device = True        # plan(..., device=d): one plan per GPU of the in-process scheduler
    scorers = REGRESSION_SCORERS

    @staticmethod
    def plan(estimator, cands, X, y, fold_id, n_splits, device=None):
        return RidgePlan(estimator, cands, X, y, fold_id, n_splits, device)


class RidgePlan(_Plan):
    scorers = REGRESSION_SCORERS
    supports_sample_weight = True
    general_splits = True          # partitions: T - G_fold; other splitters: one Gram per training / test row list

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        y = np.asarray(y)
        if y.ndim != 1:
            raise NotImplementedError("multi-output %s is not supported by the CUDA path" % type(estimator).__name__)
        if self.X.dtype != np.float32:
            # scikit-learn solves float64 input in float64; the tensor-core Grams are fp32-faithful (3xTF32 split)
            warnings.warn("spark_sklearn_b200 %s computes in float32: float64 X is rounded to float32 before the "
                          "search (scores agree with scikit-learn's float64 fit to about 1e-6 relative)"
                          % type(estimator).__name__, UserWarning)
        self._set_data(self.X.astype(np.float32, copy=False), y_target=y.astype(np.float32))

    def _check(self, p):
        if p.get("solver", "auto") not in ("auto", "cholesky"):
            raise NotImplementedError("Ridge solver=%r has no CUDA path (auto/cholesky do)" % (p["solver"],))
        if p.get("positive"):
            raise NotImplementedError("Ridge positive=True is not supported by the CUDA path")
        if not (isinstance(p["alpha"], numbers.Real) and p["alpha"] >= 0):
            raise ValueError("alpha must be a non-negative number; got %r" % (p["alpha"],))

    def evaluate(self, my, return_train=True, error_score='raise'):
        shape = (len(my), self.n_splits)
        res = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape), score_ms=np.zeros(shape))
        groups = {}
        for j, ci in enumerate(my):
            p = self._base_params(self.cands[ci])
            self._check(p)
            groups.setdefault(bool(p["fit_intercept"]), []).append((j, float(p["alpha"])))
        prof = {}
        for fi, items in groups.items():
            idx = [j for j, _ in items]
            self.engine.set_scoring(self.score_kind, self.score_pos)
            r = self.engine.ridge([a for _, a in items], fit_intercept=fi, return_train=return_train)
            for key in ("test", "fit_ms", "score_ms"):
                res[key][idx] = r[key]
            if return_train:
                res["train"][idx] = r["train"]
            for k, v in self.engine.profile().items():
                prof[k] = prof.get(k, 0) + v
        self._prof = prof
        return self._finish(res, return_train, error_score, len(my))

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        w, b = self.engine.ridge_refit(p["alpha"], p["fit_intercept"])
        est = clone(self.estimator).set_params(**best_params)
        dt = np.float32 if self.X.dtype == np.float32 else np.float64
        est.coef_ = w.astype(dt)
        est.intercept_ = dt(b) if p["fit_intercept"] else 0.0
        est.n_iter_ = None
        est.solver_ = "cholesky"
        est.n_features_in_ = self.X.shape[1]
        return est


# ------------------------------------------------------------------ Lasso / ElasticNet -------
class ENetAdapter:
    multi_device = True
    scorers = REGRESSION_SCORERS

    @staticmethod
    def plan(estimator, cands, X, y, fold_id, n_splits, device=None):
        return ENetPlan(estimator, cands, X, y, fold_id, n_splits, device)


class ENetPlan(RidgePlan):
    """sklearn.linear_model.Lasso / ElasticNet on the fold Grams of the Ridge path: cyclic coordinate descent with
    scikit-learn's stopping rule (linear_model/_cd_fast.pyx:243-506) in the Gram domain, csrc/linear.cu enet_cd_kernel."""

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        y = np.asarray(y)
        self._y2d = y.ndim == 2 and y.shape[1] == 1      # column-vector y (reference test_search_2.py:79): one target
        if self._y2d:
            y = y[:, 0]
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)

    def _check(self, p):
        if p.get("positive"):
            raise NotImplementedError("positive=True is not supported by the CUDA path")
        if p.get("selection", "cyclic") != "cyclic":
            raise NotImplementedError("selection='random' is not supported by the CUDA path (cyclic is)")
        if p.get("warm_start"):
            raise NotImplementedError("warm_start=True is not supported by the CUDA path")
        if isinstance(p.get("precompute", False), np.ndarray):
            raise NotImplementedError("a user-supplied Gram matrix is not supported by the CUDA path")
        if not (isinstance(p["alpha"], numbers.Real) and p["alpha"] >= 0):
            raise ValueError("alpha must be a non-negative number; got %r" % (p["alpha"],))
        l1 = p.get("l1_ratio", 1.0)
        if not (isinstance(l1, numbers.Real) and 0 <= l1 <= 1):
            raise ValueError("l1_ratio must be in [0, 1]; got %r" % (l1,))
        if self.X.shape[1] > 1024:
            raise NotImplementedError("more than 1024 features is not supported by the coordinate-descent kernel")

    def evaluate(self, my, return_train=True, error_score='raise'):
        shape = (len(my), self.n_splits)
        res = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape), score_ms=np.zeros(shape),
                   n_iter=np.zeros(shape, np.int64))
        groups = {}
        for j, ci in enumerate(my):
            p = self._base_params(self.cands[ci])
            self._check(p)
            key = (bool(p["fit_intercept"]), float(p["tol"]), int(p["max_iter"]))
            groups.setdefault(key, []).append((j, float(p["alpha"]), float(p.get("l1_ratio", 1.0))))
        prof = {}
        for (fi, tol, max_iter), items in groups.items():
            idx = [j for j, _, _ in items]
            self.engine.set_scoring(self.score_kind, self.score_pos)
            r = self.engine.enet([a for _, a, _ in items], [l for _, _, l in items], fit_intercept=fi, tol=tol,
                                 max_iter=max_iter, return_train=return_train)
            for key in ("test", "fit_ms", "score_ms", "n_iter"):
                res[key][idx] = r[key]
            if return_train:
                res["train"][idx] = r["train"]
            for k, v in self.engine.profile().items():
                prof[k] = prof.get(k, 0) + v
        self._prof = prof
        self.n_iter_ = res["n_iter"]
        return self._finish(res, return_train, error_score, len(my))

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        w, b, n_iter, gap = self.engine.enet_refit(p["alpha"], p.get("l1_ratio", 1.0), p["fit_intercept"], p["tol"], p["max_iter"])
        est = clone(self.estimator).set_params(**best_params)
        dt = np.float32 if self.X.dtype == np.float32 else np.float64
        est.coef_ = w.astype(dt)[None, :] if self._y2d else w.astype(dt)
        b = dt(b) if p["fit_intercept"] else 0.0
        est.intercept_ = np.array([b], dt) if self._y2d else b
        est.n_iter_ = n_iter
        est.dual_gap_ = dt(gap / len(self.X))        # _coordinate_descent.py:862
        est.n_features_in_ = self.X.shape[1]
        return est


# ------------------------------------------------------------------ one-step Pipeline ---------
class PipelineAdapter:
    """Pipeline([(name, estimator)]) searched through 'name__param' (reference tests/test_search_2.py:69-93): the step's plan
    with the prefix stripped; the refit estimator is returned inside a fitted clone of the Pipeline."""

    def __init__(self, step, inner):
        self.step, self.inner = step, inner
        self.multi_device = getattr(inner, "multi_device", False)
        self.scorers = inner.scorers

    def _strip(self, cand):
        pre = self.step + "__"
        out = {}
        for k, v in cand.items():
            if not k.startswith(pre):
                raise NotImplementedError("Pipeline parameter %r: only '%s<param>' of the single step has a CUDA path" % (k, pre))
            out[k[len(pre):]] = v
        return out

    def plan(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        inner_plan = self.inner.plan(estimator.steps[0][1], [self._strip(c) for c in cands], X, y, fold_id, n_splits, device)
        return _PipelinePlan(self, estimator, inner_plan)


class _PipelinePlan:
    def __init__(self, adapter, pipeline, inner):
        self._adapter, self._pipeline, self._inner = adapter, pipeline, inner

    def __getattr__(self, name):                      # evaluate, set_scoring, costs, profile, engine, close ...
        return getattr(self._inner, name)

    def set_fit_params(self, fit_params):
        self._inner.set_fit_params(self._adapter._strip(fit_params or {}))

    def refit(self, best_params):
        from sklearn.pipeline import Pipeline
        fitted = self._inner.refit(self._adapter._strip(best_params))
        pipe = clone(self._pipeline)
        pipe.steps = [(self._adapter.step, fitted)]
        return pipe


# ------------------------------------------------------------------ LogisticRegression --------
class LogRegAdapter:
    multi_device = True        # plan(..., device=d): one plan per GPU of the in-process scheduler
    scorers = CLASSIFICATION_SCORERS

    @staticmethod
    def plan(estimator, cands, X, y, fold_id, n_splits, device=None):
        return LogRegPlan(estimator, cands, X, y, fold_id, n_splits, device)


class LogRegPlan(_Plan):
    scorers = CLASSIFICATION_SCORERS
    supports_sample_weight = True

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        self.classes, self.y_class = np.unique(np.asarray(y), return_inverse=True)
        if len(self.classes) < 2:
            raise ValueError("LogisticRegression needs samples of at least 2 classes; got %d" % len(self.classes))
        if len(self.classes) > 64:
            raise NotImplementedError("LogisticRegression CUDA path handles up to 64 classes (got %d)" % len(self.classes))
        if self.X.dtype != np.float32:
            warnings.warn("spark_sklearn_b200 LogisticRegression computes in float32: float64 X is rounded to float32 "
                          "before the search", UserWarning)
        self._set_data(self.X.astype(np.float32, copy=False), y_class=self.y_class.astype(np.int32))

    def _check(self, p):
        if p.get("solver", "lbfgs") != "lbfgs":
            raise NotImplementedError("LogisticRegression solver=%r has no CUDA path (lbfgs does)" % (p["solver"],))
        # scikit-learn 1.9: penalty='deprecated' (the default) or 'l2' with l1_ratio None/0 is the L2 problem the kernel
        # solves; penalty=None (no regularisation, C ignored), 'l1', 'elasticnet' or any l1_ratio > 0 are other problems
        if p.get("penalty", "l2") not in ("l2", "deprecated") or p.get("l1_ratio") not in (None, 0, 0.0):
            raise NotImplementedError("LogisticRegression penalty=%r, l1_ratio=%r has no CUDA path (only the L2 penalty does)"
                                      % (p.get("penalty"), p.get("l1_ratio")))
        if not (isinstance(p["C"], numbers.Real) and p["C"] > 0):
            raise ValueError("C must be a positive number; got %r" % (p["C"],))

    def evaluate(self, my, return_train=True, error_score='raise'):
        shape = (len(my), self.n_splits)
        res = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape), score_ms=np.zeros(shape))
        groups = {}
        for j, ci in enumerate(my):
            p = self._base_params(self.cands[ci])
            self._check(p)
            cw = p.get("class_weight")
            cwk = None if cw is None else (cw if isinstance(cw, str) else tuple(sorted(cw.items())))
            groups.setdefault((float(p["tol"]), int(p["max_iter"]), bool(p["fit_intercept"]), cwk), []).append((j, float(p["C"]), cw))
        prof = {}
        for (tol, mi, fi, _cwk), items in groups.items():
            idx = [j for j, _, _ in items]
            self._set_class_weight(items[0][2])
            self.engine.set_scoring(self.score_kind, self.score_pos)
            r = self.engine.logreg([c for _, c, _ in items], tol=tol, max_iter=mi, fit_intercept=fi,
                                   return_train=return_train)
            for key in ("test", "fit_ms", "score_ms"):
                res[key][idx] = r[key]
            if return_train:
                res["train"][idx] = r["train"]
            for k, v in self.engine.profile().items():
                prof[k] = prof.get(k, 0) + v
        self.engine.set_class_weight(None)
        self._prof = prof
        return self._finish(res, return_train, error_score, len(my))

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        self._set_class_weight(p.get("class_weight"), refit=True)
        w, b, it = self.engine.logreg_refit(p["C"], p["tol"], p["max_iter"], p["fit_intercept"])
        self.engine.set_class_weight(None)
        est = clone(self.estimator).set_params(**best_params)
        est.classes_ = self.classes
        if len(self.classes) > 2:                        # multinomial: one weight row per class (_logistic.py:1355 fit)
            est.coef_ = np.asarray(w)
            est.intercept_ = np.asarray(b) if p["fit_intercept"] else np.zeros(len(self.classes))
        else:
            est.coef_ = w.reshape(1, -1)
            est.intercept_ = np.array([b if p["fit_intercept"] else 0.0])
        est.n_iter_ = np.array([it], np.int32)
        est.n_features_in_ = self.X.shape[1]
        return est


# ------------------------------------------------------------------ LinearSVC -----------------
class LinearSVCAdapter:
    multi_device = True        # plan(..., device=d): one plan per GPU of the in-process scheduler
    scorers = CLASSIFICATION_SCORERS

    @staticmethod
    def plan(estimator, cands, X, y, fold_id, n_splits, device=None):
        return LinearSVCPlan(estimator, cands, X, y, fold_id, n_splits, device)


class LinearSVCPlan(_Plan):
    """sklearn.svm.LinearSVC with liblinear's primal solver (L2R_L2LOSS_SVC: TRON, csrc/linsvc.cu).  X reaches the device in
    float32 or float64 and is widened exactly, as scikit-learn's fit converts it to float64.  Every fit resolves dual='auto'
    from its own training set, as LinearSVC.fit does; a fit that resolves to the dual solver has no CUDA path."""
    scorers = CLASSIFICATION_SCORERS
    supports_sample_weight = True

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("LinearSVC needs y")
        self.classes, self.y_class = np.unique(np.asarray(y), return_inverse=True)
        if len(self.classes) < 2:
            raise ValueError("This solver needs samples of at least 2 classes in the data, but the data contains only one "
                             "class: %r" % (self.classes[0],))
        if len(self.classes) > 64:
            raise NotImplementedError("LinearSVC CUDA path handles up to 64 classes (got %d)" % len(self.classes))
        self._set_data(self.X, y_class=self.y_class.astype(np.int32))

    def _check(self, p, n_rows):
        """scikit-learn's own checks in LinearSVC.fit's order (parameter constraints, dual resolution on a training set of
        n_rows rows, the liblinear solver of the combination: ValueError), then the combinations without a CUDA path"""
        from sklearn.svm import LinearSVC
        from sklearn.svm._base import _get_liblinear_solver_type
        from sklearn.svm._classes import _validate_dual_parameter
        LinearSVC(**p)._validate_params()
        dual = _validate_dual_parameter(p["dual"], p["loss"], p["penalty"], p["multi_class"],
                                        np.empty((n_rows, self.X.shape[1]), np.bool_))
        if p["multi_class"] == "crammer_singer":
            raise NotImplementedError("LinearSVC multi_class='crammer_singer' has no CUDA path (one-vs-rest does)")
        _get_liblinear_solver_type(p["multi_class"], p["penalty"], p["loss"], dual)
        if dual:
            raise NotImplementedError(
                "LinearSVC fit on %d rows x %d features resolves to the dual solver (dual=%r), which has no CUDA path (the "
                "primal solver, dual=False with at least as many rows as features, does)" % (n_rows, self.X.shape[1], p["dual"]))
        if p["penalty"] != "l2":
            raise NotImplementedError("LinearSVC penalty=%r has no CUDA path (l2 does)" % (p["penalty"],))

    def _params(self, cand, ks):
        p = self._base_params(cand)
        for k in ks:
            self._check(p, int(np.count_nonzero(self._train_rows(k))))
        return p

    def evaluate(self, my, return_train=True, error_score='raise'):
        shape = (len(my), self.n_splits)
        res = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape), score_ms=np.zeros(shape),
                   n_iter=np.zeros(shape, np.int64))
        groups = {}
        for j, ci in enumerate(my):
            p = self._params(self.cands[ci], range(self.n_splits))
            cw = p.get("class_weight")
            cwk = None if cw is None else (cw if isinstance(cw, str) else tuple(sorted(cw.items())))
            key = (float(p["tol"]), int(p["max_iter"]), bool(p["fit_intercept"]), float(p["intercept_scaling"]), cwk)
            groups.setdefault(key, []).append((j, float(p["C"]), cw))
        prof = {}
        for (tol, mi, fi, isc, _cwk), items in groups.items():
            idx = [j for j, _, _ in items]
            self._set_class_weight(items[0][2])
            self.engine.set_scoring(self.score_kind, self.score_pos)
            r = self.engine.linsvc([c for _, c, _ in items], tol=tol, max_iter=mi, fit_intercept=fi, intercept_scaling=isc,
                                   return_train=return_train)
            for key in ("test", "fit_ms", "score_ms", "n_iter"):
                res[key][idx] = r[key]
            if return_train:
                res["train"][idx] = r["train"]
            for k, v in self.engine.profile().items():
                prof[k] = prof.get(k, 0) + v
        self.engine.set_class_weight(None)
        self._prof = prof
        self.n_iter_ = res["n_iter"]
        return self._finish(res, return_train, error_score, len(my))

    def refit(self, best_params):
        p = self._params(best_params, [-1])
        self._set_class_weight(p.get("class_weight"), refit=True)
        raw, n_iter = self.engine.linsvc_refit(p["C"], p["tol"], p["max_iter"], p["fit_intercept"], p["intercept_scaling"])
        self.engine.set_class_weight(None)
        est = clone(self.estimator).set_params(**best_params)
        return materialize_linsvc(est, self.classes, raw, n_iter, self.X.shape[1])


def materialize_linsvc(est, classes, raw, n_iter, n_features):
    """Fill a (cloned, parametrised) sklearn.svm.LinearSVC with the fitted state of liblinear's raw weights raw
    [rows][n_features + 1] (the bias feature's weight last) and the per-fit iteration counts (svm/_base.py:1296-1310
    _fit_liblinear, svm/_classes.py:330-351 LinearSVC.fit), with scikit-learn's ConvergenceWarning."""
    raw = np.asarray(raw, np.float64)
    est.classes_ = np.asarray(classes)
    if est.fit_intercept:
        est.coef_ = raw[:, :n_features].copy()
        est.intercept_ = est.intercept_scaling * raw[:, n_features]
    else:
        est.coef_ = raw[:, :n_features].copy()
        est.intercept_ = 0.0
    est.n_iter_ = int(np.max(n_iter))
    est.n_features_in_ = int(n_features)
    if est.n_iter_ >= est.max_iter:
        from sklearn.exceptions import ConvergenceWarning
        warnings.warn("Liblinear failed to converge, increase the number of iterations.", ConvergenceWarning)
    return est


# ------------------------------------------------------------------ k-nearest neighbours ------
class KNeighborsAdapter:
    # One GPU: the neighbour selection is the cost of the whole search and every candidate shares it, so dealing candidates
    # to several GPUs would repeat it on each.  Under torchrun each rank still evaluates the candidates it is dealt.
    multi_device = False
    scorers = CLASSIFICATION_SCORERS

    @staticmethod
    def plan(estimator, cands, X, y, fold_id, n_splits, device=None):
        return KNeighborsPlan(estimator, cands, X, y, fold_id, n_splits, device)


class KNeighborsRegressorAdapter(KNeighborsAdapter):
    scorers = REGRESSION_SCORERS


_KNN_METRICS = {"euclidean": "euclidean", "l2": "euclidean", "manhattan": "manhattan", "l1": "manhattan",
                "cityblock": "manhattan"}


class KNeighborsPlan(_Plan):
    """sklearn.neighbors.KNeighborsClassifier / KNeighborsRegressor (csrc/knn.cu).  A fit stores its training rows; every
    (candidate, split) task's scorer queries the neighbours of its test rows (and, for the train score, of its training
    rows).  The engine selects the max n_neighbors nearest training rows once per (split, metric) and every candidate votes
    from those lists.  The refit is scikit-learn's own fit (it stores the data, plus a tree index when scikit-learn builds
    one: there is no arithmetic for the device to take over)."""
    max_neighbors = 256

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        from sklearn.neighbors import KNeighborsClassifier
        name = type(estimator).__name__
        if y is None:
            raise ValueError("%s needs y" % name)
        self.classifier = isinstance(estimator, KNeighborsClassifier)
        self.scorers = CLASSIFICATION_SCORERS if self.classifier else REGRESSION_SCORERS
        y = np.asarray(y)
        if y.ndim != 1:
            raise NotImplementedError("multi-output %s is not supported by the CUDA path" % name)
        if self.classifier:
            self.classes, self.y_class = np.unique(y, return_inverse=True)
            if len(self.classes) > 64:
                raise NotImplementedError("%s CUDA path handles up to 64 classes (got %d)" % (name, len(self.classes)))
            self._set_data(self.X, y_class=self.y_class.astype(np.int32))
        else:
            # scikit-learn keeps y's dtype: float32 y gives float32 uniform means
            self.y_f32 = y.dtype == np.float32
            self.y64 = y.astype(np.float64)
            self._set_data(self.X, y_target=self.y64.astype(np.float32))
            self.engine.set_targets_f64(self.y64)

    def _check(self, p):
        """scikit-learn's own parameter checks (ValueError), then what the CUDA path does not cover -> (n_neighbors, weights,
        metric name)"""
        type(self.estimator)(**p)._validate_params()
        nn = p["n_neighbors"]
        if nn > self.max_neighbors:
            raise NotImplementedError("n_neighbors=%d: the CUDA path handles up to %d neighbours" % (nn, self.max_neighbors))
        if callable(p["weights"]):
            raise NotImplementedError("a callable weights has no CUDA path ('uniform' and 'distance' do)")
        if p.get("metric_params") is not None:
            raise NotImplementedError("metric_params has no CUDA path")
        metric = p["metric"]
        if metric == "minkowski":
            if p["p"] not in (1, 2):
                raise NotImplementedError("minkowski p=%r has no CUDA path (p=1 and p=2 do)" % (p["p"],))
            metric = "manhattan" if p["p"] == 1 else "euclidean"
        elif not isinstance(metric, str) or metric not in _KNN_METRICS:
            raise NotImplementedError("metric=%r has no CUDA path (minkowski with p 1 or 2, %s do)"
                                      % (metric, ", ".join(sorted(_KNN_METRICS))))
        return int(nn), p["weights"], _KNN_METRICS[metric]

    def evaluate(self, my, return_train=True, error_score='raise'):
        ns = self.n_splits
        shape = (len(my), ns)
        checked = [self._check(self._base_params(self.cands[ci])) for ci in my]
        m_train = [int(np.count_nonzero(self._train_rows(k))) for k in range(ns)]
        too_many = np.array([[nn > m_train[k] for k in range(ns)] for nn, _, _ in checked], bool).reshape(shape)
        if too_many.any() and error_score == 'raise':
            j, k = map(int, np.argwhere(too_many)[0])
            n_test = int(np.count_nonzero(self._test_rows(k)))
            raise ValueError("Expected n_neighbors <= n_samples_fit, but n_neighbors = %d, n_samples_fit = %d, n_samples = %d"
                             % (checked[j][0], m_train[k], n_test))
        res = dict(test=np.full(shape, np.nan), train=np.full(shape, np.nan), fit_ms=np.zeros(shape), score_ms=np.zeros(shape))
        if my:
            self.engine.set_scoring(self.score_kind, self.score_pos)
            r = self.engine.knn([c[0] for c in checked], [c[1] for c in checked], [c[2] for c in checked],
                                return_train=return_train, y_f32=not self.classifier and self.y_f32)
            for key in ("test", "fit_ms", "score_ms"):
                res[key][:] = r[key]
            if return_train:
                res["train"][:] = r["train"]
            self._prof = self.engine.profile()
        res["test"][too_many] = np.nan
        res["train"][too_many] = np.nan
        return self._finish(res, return_train, error_score, len(my))

    def _test_rows(self, k):
        if self.folds is not None and not self.folds.partition:
            return (self.folds.masks[0][:, k >> 6] >> np.uint64(k & 63)) & np.uint64(1) == 1
        fold_id = self.fold_id if self.folds is None else self.folds.fold_id
        return fold_id == k

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        return clone(self.estimator).set_params(**best_params).fit(self.X, self.y)
