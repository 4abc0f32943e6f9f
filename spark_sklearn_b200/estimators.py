"""Estimator plans: turn (estimator, candidate dicts, folds) into the scalar tables the C ABI takes,
and turn refit buffers back into genuine fitted scikit-learn estimators for ``best_estimator_``
(reference base_search.py:165-174 delegates ``predict`` & co. to it).

Only estimators with a CUDA path are accepted (SVC with the linear, rbf, poly and sigmoid kernels, SVR rbf/linear, Ridge,
Lasso / ElasticNet, LogisticRegression (lbfgs, sag, saga), LinearSVC with the primal squared-hinge solver -- the families the reference ships
examples for -- LinearSVR, SGDClassifier / SGDRegressor, and KNeighborsClassifier / KNeighborsRegressor); anything else raises: no CPU fallback.
"""
import copy
import numbers
import threading
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
        # every split's training indices as the splitter yields them: a fit whose result depends on the order of X[train]
        # (LinearSVR's coordinate descent) sees its rows in this order
        self.train_order = [np.asarray(tr, np.int64) for tr, _ in splits]
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

    def test_rows(self, k):
        """boolean [n]: the test rows of split k"""
        if self.fold_id is not None:
            return self.fold_id == k
        return (self.masks[0][:, k >> 6] >> np.uint64(k & 63)) & np.uint64(1) == 1


def adapter_for(estimator):
    """The plan class of an estimator: plan(estimator, cands, X, y, fold_id, n_splits, device=None), multi_device, scorers"""
    from sklearn.linear_model import ElasticNet, Lasso, LogisticRegression, Ridge, SGDClassifier, SGDRegressor
    from sklearn.neighbors import KNeighborsClassifier, KNeighborsRegressor
    from sklearn.pipeline import Pipeline
    from sklearn.svm import SVC, SVR, LinearSVC, LinearSVR, NuSVC, NuSVR
    plans = {SVC: SVCPlan, SVR: SVRPlan, NuSVC: NuSVCPlan, NuSVR: NuSVRPlan, Ridge: RidgePlan, Lasso: ENetPlan,
             ElasticNet: ENetPlan, LogisticRegression: LogRegPlan, LinearSVC: LinearSVCPlan, LinearSVR: LinearSVRPlan,
             SGDClassifier: SGDPlan, SGDRegressor: SGDRegressorPlan, KNeighborsClassifier: KNeighborsPlan,
             KNeighborsRegressor: KNeighborsRegressorPlan}
    t = type(estimator)
    if t in plans:
        return plans[t]
    if t is Pipeline and len(estimator.steps) == 1:
        # the reference's own search tests wrap the estimator in a one-step Pipeline and search 'step__param'
        # (python/spark_sklearn/tests/test_search_2.py:69-93): the step's adapter runs, the names are translated
        return PipelineAdapter(estimator.steps[0][0], adapter_for(estimator.steps[0][1]))
    raise NotImplementedError(
        "spark_sklearn_b200 has CUDA paths for SVC, SVR, NuSVC, NuSVR, Ridge, Lasso, ElasticNet, LogisticRegression, LinearSVC, "
        "LinearSVR, SGDClassifier, SGDRegressor, KNeighborsClassifier and KNeighborsRegressor (bare or as the only step of a Pipeline); got %s (no CPU fallback)"
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


# scoring= names with a fused CUDA scorer (include/b200gs.h GS_SCORE_*); None = the estimator's own score
CLASSIFICATION_SCORERS = {None: 0, "accuracy": 0, "balanced_accuracy": 1, "f1": 2, "precision": 3, "recall": 4, "roc_auc": 5,
                          "f1_macro": 6, "f1_micro": 7, "f1_weighted": 8}
REGRESSION_SCORERS = {None: 0, "r2": 0, "neg_mean_squared_error": 16, "neg_root_mean_squared_error": 17}


_INT_MAX = int(np.iinfo("i").max)
_SEED_LOCK = threading.Lock()


def _random_state(random_state):
    """check_random_state(random_state) as one fit sees it: an int or a RandomState gives every fit the same draws (clone
    deep-copies the parameter, so the caller's RandomState is not advanced); None draws from numpy's global RandomState."""
    from sklearn.utils import check_random_state
    if random_state is not None and not isinstance(random_state, (numbers.Integral, np.random.RandomState)):
        raise ValueError("%r cannot be used to seed a numpy.random.RandomState instance" % (random_state,))
    return check_random_state(copy.deepcopy(random_state) if isinstance(random_state, np.random.RandomState) else random_state)


def fit_seed(random_state, low):
    """The seed of one fit: check_random_state(random_state).randint(low, np.iinfo('i').max).  low 0: the seed
    _fit_liblinear hands to liblinear; low 1: make_dataset's seed of a LogisticRegression(solver='sag' | 'saga') fit."""
    return int(_random_state(random_state).randint(low, _INT_MAX))


def _class_weight_key(cw):
    """class_weight as a group key: None, 'balanced' or the sorted items of a dict"""
    return cw if cw is None or isinstance(cw, str) else tuple(sorted(cw.items()))


def _target_1d(y, name):
    """scikit-learn's column_or_1d(y, warn=True): a column vector is raveled with a DataConversionWarning"""
    y = np.asarray(y)
    if y.ndim == 2 and y.shape[1] == 1:
        from sklearn.exceptions import DataConversionWarning
        warnings.warn("A column-vector y was passed when a 1d array was expected. Please change the shape of y to "
                      "(n_samples, ), for example using ravel().", DataConversionWarning, stacklevel=3)
        y = y[:, 0]
    if y.ndim != 1:
        raise ValueError("%s needs a 1d target; got y of shape %r" % (name, y.shape))
    return y


def _overflow(epoch):
    """the ValueError of an SGD or SAG fit that went non-finite"""
    return ValueError("Floating-point under-/overflow occurred at epoch #%d. Scaling input data with StandardScaler or "
                      "MinMaxScaler might help." % epoch)


class _Plan:
    """One search of one estimator on one device.  A plan class is its own adapter: adapter_for(estimator).plan(...).
    Each plan checks its candidates (_candidate) and makes one engine call per group of candidates (_search); evaluate
    does the rest."""
    multi_device = True        # plan(..., device=d): one plan per GPU of the in-process scheduler
    scorers = {None: 0}
    class_weighted = False     # the estimator has class_weight: one gs_set_class_weight per group
    fail_warning = None        # fits can fail (SGD, SAG): the warning that gives them error_score
    _seed = None               # random_state -> one fit's seeds: the plan draws a seed table (_seed_table)

    @classmethod
    def plan(cls, estimator, cands, X, y, fold_id, n_splits, device=None):
        return cls(estimator, cands, X, y, fold_id, n_splits, device)

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        self.estimator, self.cands = estimator, cands
        self.X, self.y, self.n_splits = _as_matrix(X), y, n_splits
        if isinstance(fold_id, Folds):
            self.folds, self.fold_id = fold_id, fold_id.fold_id
        else:                                             # a bare fold_id array: the splits are a partition
            self.folds, self.fold_id = None, fold_id
        self.engine = get_engine(device)
        self._prof = {}
        self._seeds = None
        self.score_kind, self.score_pos = 0, 1

    def _candidate(self, p, error_score):
        """check one candidate's parameters p -> (group key, engine-call values)"""
        raise NotImplementedError

    def _prepare(self, my, error_score):
        """every candidate of my checked, before any device work -> ([(params, group key, values)], the [len(my)][n_splits]
        fits that fail on the host, or None)"""
        prepared = []
        for ci in my:
            p = self._base_params(self.cands[ci])
            prepared.append((p,) + tuple(self._candidate(p, error_score)))
        return prepared, None

    def _search(self, key, values, cands, return_train):
        """one engine call for the candidates cands (indices into self.cands) of one group -> the engine's outputs"""
        raise NotImplementedError

    def _undefined(self):
        """[n_splits] bool: the splits whose test score scikit-learn itself leaves NaN (None: none)"""
        return None

    def evaluate(self, my, return_train=True, error_score='raise'):
        """the (candidate, split) fits of the candidates my: one engine call per group of candidates that share the call's
        settings (and class weights), groups in order of first appearance"""
        prepared, failed = self._prepare(my, error_score)
        if self._seed is not None:
            self._seed_table()
        groups = {}
        for j, (p, key, _) in enumerate(prepared):
            cwk = _class_weight_key(p.get("class_weight")) if self.class_weighted else None
            groups.setdefault((key, cwk), []).append(j)
        shape = (len(my), self.n_splits)
        res = dict(test=np.zeros(shape), train=np.zeros(shape), fit_ms=np.zeros(shape), score_ms=np.zeros(shape))
        prof = {}
        try:
            for (key, _), idx in groups.items():
                if self.class_weighted:
                    self._set_class_weight(prepared[idx[0]][0].get("class_weight"))
                self.engine.set_scoring(self.score_kind, self.score_pos)
                r = self._search(key, [prepared[j][2] for j in idx], [my[j] for j in idx], return_train)
                for k, v in r.items():
                    if v is None:
                        continue
                    if k not in res:                          # n_iter, status, per-fit counters: int64
                        res[k] = np.zeros(shape + v.shape[2:], np.float64 if v.dtype.kind == "f" else np.int64)
                    res[k][idx] = v
                for k, v in self.engine.profile().items():
                    prof[k] = prof.get(k, 0) + v
        finally:
            if self.class_weighted:
                self.engine.set_class_weight(None)
        self._prof = prof
        for k in ("n_iter", "stats", "cd_stats"):
            if k in res:
                setattr(self, k + "_", res[k])
        bad = np.zeros(shape, bool) if failed is None else failed
        if "status" in res:
            bad = bad | (res["status"] == 2)                  # the engine's non-finite fits
        if bad.any():
            if self.fail_warning is None:
                fill = np.nan                                 # k-NN: NaN, which _finish reports
            elif error_score == 'raise':
                j, k = map(int, np.argwhere(bad)[0])
                raise _overflow(int(res["n_iter"][j, k]))
            else:
                warnings.warn(self.fail_warning % (int(bad.sum()), error_score))
                fill = error_score
            res["test"][bad] = fill
            res["train"][bad] = fill
        return self._finish(res, return_train, error_score, self._undefined())

    def _seed_table(self):
        """The seeds of every fit of the search, [n_cand][n_splits] + the shape of one fit's seeds, drawn as scikit-learn's
        GridSearchCV draws them: candidate-major, split-minor, random_state=None from numpy's global RandomState.  A search
        whose candidates draw from the global RandomState computes the table once for all of its per-GPU plans (they share
        the Folds); the plan keeps it."""
        if self._seeds is None:
            states = [self._base_params(c)["random_state"] for c in self.cands]
            draw = lambda: np.array([[self._seed(rs) for _ in range(self.n_splits)] if rs is None
                                     else [self._seed(rs)] * self.n_splits for rs in states], np.int64)
            if any(rs is None for rs in states) and self.folds is not None:
                with _SEED_LOCK:
                    if getattr(self.folds, "_search_seeds", None) is None:
                        self.folds._search_seeds = draw()
                    self._seeds = self.folds._search_seeds
            else:
                self._seeds = draw()
        return self._seeds

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
        """boolean [n]: the training rows of split k (all rows for k < 0)"""
        if self.folds is not None:
            return self.folds.train_rows(k)
        return self.fold_id != k if k >= 0 else np.ones(len(self.fold_id), bool)

    def _test_rows(self, k):
        """boolean [n]: the test rows of split k"""
        return self.folds.test_rows(k) if self.folds is not None else self.fold_id == k

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

    def _finish(self, res, return_train, error_score, undefined=None):
        """undefined: [n_splits] bool, the splits whose test score scikit-learn itself leaves NaN (kept, not an error)"""
        test, train = res["test"], res.get("train")
        bad = ~np.isfinite(test)
        if undefined is not None:
            bad &= ~undefined[None, :]
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

    def _gammas(self, p, kernels):
        """[n_splits] gamma of candidate p's fits: 0 unless its kernel is one of kernels"""
        return [self._gamma(p["gamma"], k) if p["kernel"] in kernels else 0.0 for k in range(self.n_splits)]

    def _nu_kw(self):
        """engine keyword of the nu solvers (NuSVCPlan / NuSVRPlan set nu = True)"""
        return {"nu": True} if self.nu else {}

    def _flags(self):
        import os
        # B200GS_GRAM=tensor: opt-in wgmma Gram (fp32-faithful; scores match to solver tolerance, not bit for bit)
        return 2 if os.environ.get("B200GS_GRAM", "exact") == "tensor" else 0


class SVCPlan(_KernelGamma, _Plan):
    """sklearn.svm.SVC (C-SVC).  Scalars per candidate: kernel, C, gamma (resolved per fold for every kernel but linear),
    degree and coef0 (poly, sigmoid)."""
    scorers = CLASSIFICATION_SCORERS
    class_weighted = True

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("SVC needs y")
        self.classes, self.y_class = np.unique(np.asarray(y), return_inverse=True)
        if len(self.classes) < 2:
            raise ValueError("The number of classes has to be greater than one; got %d class" % len(self.classes))
        self._set_data(self.X, y_class=self.y_class.astype(np.int32))
        self._var_cache = {}

    nu = False                 # NuSVCPlan: the nu-SVC solver, with nu where SVC has C
    penalty = "C"

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
        self._check_penalty(p)

    def _check_penalty(self, p):
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

    def _candidate(self, p, error_score):
        self._check(p)
        return (float(p["tol"]), int(p["max_iter"]), bool(p["shrinking"])), (p, self._gammas(p, ("rbf", "poly", "sigmoid")))

    def _search(self, key, values, cands, return_train):
        tol, max_iter, shrinking = key
        ps = [p for p, _ in values]
        return self.engine.svc([p["kernel"] for p in ps], [float(p[self.penalty]) for p in ps], np.array([g for _, g in values]),
                               tol=tol, max_iter=max_iter, shrinking=shrinking, return_train=return_train, flags=self._flags(),
                               degree=[int(p["degree"]) for p in ps], coef0=[float(p["coef0"]) for p in ps], **self._nu_kw())

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        gamma = self._gamma(p["gamma"], -1)          # all rows train (svm/_base.py:278-286)
        cw_ = self._set_class_weight(p.get("class_weight"), refit=True)
        coef, rho, n_iter = self.engine.svc_refit(p["kernel"], p[self.penalty], gamma if p["kernel"] != "linear" else 0.0,
                                                  len(self.classes), tol=p["tol"], max_iter=p["max_iter"],
                                                  shrinking=p["shrinking"], degree=int(p["degree"]), coef0=float(p["coef0"]),
                                                  **self._nu_kw())
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


# ------------------------------------------------------------------ NuSVC ---------------------
class NuSVCPlan(SVCPlan):
    """sklearn.svm.NuSVC (libsvm's nu-SVC): SVCPlan with nu in place of C.  class_weight is accepted and reported in
    class_weight_ but, as in libsvm, does not change a nu-SVC fit."""
    nu = True
    penalty = "nu"

    def _check_penalty(self, p):
        type(self.estimator)(**p)._validate_params()          # scikit-learn's own ValueError, e.g. nu outside (0, 1]

    def _infeasible(self, nu, k):
        """libsvm svm_check_parameter: nu is infeasible for the training rows of split k (k < 0: all rows) when some class
        pair has nu (n1 + n2) / 2 > min(n1, n2)"""
        n = np.bincount(self.y_class[self._train_rows(k)], minlength=len(self.classes)).astype(np.float64)
        n = n[n > 0]
        return any(nu * (n[a] + n[b]) / 2 > min(n[a], n[b]) for a in range(len(n)) for b in range(a + 1, len(n)))

    def costs(self):
        return None                                           # no iteration model for nu-SVC: candidates are dealt uniformly

    def _candidate(self, p, error_score):
        if error_score == 'raise':                            # scikit-learn's fit raises before any solve
            self._check(p)
            if any(self._infeasible(float(p["nu"]), k) for k in range(self.n_splits)):
                raise ValueError("specified nu is infeasible")
        return super()._candidate(p, error_score)

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        if self._infeasible(float(p["nu"]), -1):
            raise ValueError("specified nu is infeasible")
        return super().refit(best_params)


# ------------------------------------------------------------------ SVR -----------------------
class SVRPlan(_KernelGamma, _Plan):
    """sklearn.svm.SVR (epsilon-SVR).  Scalars per candidate: kernel, C, epsilon, gamma (resolved per fold).  Each fit runs
    libsvm's solver on its training rows in ascending row order, as scikit-learn's X[train] does for KFold-like splitters."""
    scorers = REGRESSION_SCORERS

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("SVR needs y")
        self.y = _target_1d(y, "SVR").astype(np.float64)  # scikit-learn fits SVR on float64 y
        self._set_data(self.X, y_target=self.y.astype(np.float32))
        self.engine.set_targets_f64(self.y)

    nu = False                 # NuSVRPlan: the nu-SVR solver, with nu where SVR has epsilon
    tube = "epsilon"

    def _check(self, p):
        if p["kernel"] not in ("rbf", "linear"):
            raise NotImplementedError("%s kernel=%r has no CUDA path (rbf and linear do)" % (type(self.estimator).__name__, p["kernel"]))
        self._check_tube(p)

    def _check_tube(self, p):
        if not (isinstance(p["C"], numbers.Real) and p["C"] > 0):
            raise ValueError("C must be a positive number; got %r" % (p["C"],))
        if not (isinstance(p["epsilon"], numbers.Real) and p["epsilon"] >= 0):
            raise ValueError("epsilon must be a non-negative number; got %r" % (p["epsilon"],))

    max_rows = 8192        # training rows of one fit: 2 x 8192 solver variables, the largest resident-state SMO instance

    def _check_rows(self, k):
        m = int(np.count_nonzero(self._train_rows(k)))
        if m > self.max_rows:
            raise NotImplementedError("%s fit on %d training rows: the CUDA solver handles up to %d"
                                      % (type(self.estimator).__name__, m, self.max_rows))

    def check_refit(self):
        """the refit trains on every row: raise before the search when that fit is too large"""
        self._check_rows(-1)

    def _prepare(self, my, error_score):
        for k in range(self.n_splits):
            self._check_rows(k)
        return super()._prepare(my, error_score)

    def _candidate(self, p, error_score):
        self._check(p)
        return (float(p["tol"]), int(p["max_iter"]), bool(p["shrinking"])), (p, self._gammas(p, ("rbf",)))

    def _search(self, key, values, cands, return_train):
        tol, max_iter, shrinking = key
        ps = [p for p, _ in values]
        return self.engine.svr([p["kernel"] for p in ps], [float(p["C"]) for p in ps], [float(p[self.tube]) for p in ps],
                               np.array([g for _, g in values]), tol=tol, max_iter=max_iter, shrinking=shrinking,
                               return_train=return_train, flags=self._flags(), **self._nu_kw())

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        self._check_rows(-1)
        gamma = self._gamma(p["gamma"], -1)          # all rows train (svm/_base.py:278-286)
        coef, rho, n_iter = self.engine.svr_refit(p["kernel"], p["C"], p[self.tube], gamma if p["kernel"] == "rbf" else 0.0,
                                                  tol=p["tol"], max_iter=p["max_iter"], shrinking=p["shrinking"],
                                                  flags=self._flags(), **self._nu_kw())
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


# ------------------------------------------------------------------ NuSVR ---------------------
class NuSVRPlan(SVRPlan):
    """sklearn.svm.NuSVR (libsvm's nu-SVR): SVRPlan with nu in place of epsilon; materialize_svr builds the fitted NuSVR."""
    nu = True
    tube = "nu"

    def _check_tube(self, p):
        type(self.estimator)(**p)._validate_params()          # scikit-learn's own ValueError, e.g. nu outside (0, 1]


# ------------------------------------------------------------------ Ridge ---------------------
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

    def _undefined(self):
        """r2 of a test set of fewer than two rows is NaN (r2_score: UndefinedMetricWarning), as in scikit-learn's search"""
        if self.score_kind != 0:
            return None
        return np.array([np.count_nonzero(self._test_rows(k)) < 2 for k in range(self.n_splits)])

    def _check(self, p):
        if p.get("solver", "auto") not in ("auto", "cholesky"):
            raise NotImplementedError("Ridge solver=%r has no CUDA path (auto/cholesky do)" % (p["solver"],))
        if p.get("positive"):
            raise NotImplementedError("Ridge positive=True is not supported by the CUDA path")
        if not (isinstance(p["alpha"], numbers.Real) and p["alpha"] >= 0):
            raise ValueError("alpha must be a non-negative number; got %r" % (p["alpha"],))

    def _candidate(self, p, error_score):
        self._check(p)
        return bool(p["fit_intercept"]), float(p["alpha"])

    def _search(self, fit_intercept, alpha, cands, return_train):
        return self.engine.ridge(alpha, fit_intercept=fit_intercept, return_train=return_train)

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

    def _candidate(self, p, error_score):
        self._check(p)
        return (bool(p["fit_intercept"]), float(p["tol"]), int(p["max_iter"])), (float(p["alpha"]), float(p.get("l1_ratio", 1.0)))

    def _search(self, key, values, cands, return_train):
        fi, tol, max_iter = key
        return self.engine.enet([a for a, _ in values], [l for _, l in values], fit_intercept=fi, tol=tol, max_iter=max_iter,
                                return_train=return_train)

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
class LogRegPlan(_Plan):
    scorers = CLASSIFICATION_SCORERS
    supports_sample_weight = True
    class_weighted = True

    @classmethod
    def plan(cls, estimator, cands, X, y, fold_id, n_splits, device=None):
        """lbfgs candidates run LogRegPlan, sag / saga candidates LogRegSAGPlan; one search runs one of the two"""
        base = estimator.get_params(deep=False).get("solver", "lbfgs")
        solvers = {c.get("solver", base) for c in cands} or {base}
        if solvers & {"sag", "saga"}:
            if not solvers <= {"sag", "saga"}:
                raise NotImplementedError("LogisticRegression: a search that mixes solver='sag' / 'saga' with %s has no CUDA path "
                                          "(search the two in separate searches)" % sorted(solvers - {"sag", "saga"}))
            return LogRegSAGPlan(estimator, cands, X, y, fold_id, n_splits, device)
        return cls(estimator, cands, X, y, fold_id, n_splits, device)

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

    def _candidate(self, p, error_score):
        self._check(p)
        return (float(p["tol"]), int(p["max_iter"]), bool(p["fit_intercept"])), float(p["C"])

    def _search(self, key, C, cands, return_train):
        tol, max_iter, fit_intercept = key
        return self.engine.logreg(C, tol=tol, max_iter=max_iter, fit_intercept=fit_intercept, return_train=return_train)

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


class LogRegSAGPlan(_Plan):
    """sklearn.linear_model.LogisticRegression(solver='sag' | 'saga') (csrc/sag.cu): sag_solver restated step for step, one
    warp per (candidate, split) fit.  X reaches the device dense in its own dtype (float32 runs sag32, float64 sag64, as
    scikit-learn does).  The step size and the scaled penalties of every fit come from scikit-learn's own functions on that
    fit's training rows, which reach the device in the splitter's order (the sample draws index them)."""
    scorers = CLASSIFICATION_SCORERS
    supports_sample_weight = True
    class_weighted = True
    fail_warning = ("%d fits failed (a floating-point under-/overflow, or step_size * alpha_scaled == 1); their scores are "
                    "error_score=%r")
    max_coef = 512             # features x weight rows held in registers (include/b200gs.h GS_SAG_MAX_COEF)

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        import scipy.sparse as sp
        if sp.issparse(X):
            raise NotImplementedError("LogisticRegression(solver='sag' | 'saga') on sparse X has no CUDA path (scikit-learn's "
                                      "sparse SAG decays the intercept and lags its updates per stored entry): pass a dense X")
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("LogisticRegression needs y")
        self.classes, self.y_class = np.unique(np.asarray(y), return_inverse=True)
        if len(self.classes) < 2:
            raise ValueError("This solver needs samples of at least 2 classes in the data, but the data contains only one "
                             "class: %r" % (self.classes[0],))
        if len(self.classes) > 64:
            raise NotImplementedError("LogisticRegression CUDA path handles up to 64 classes (got %d)" % len(self.classes))
        self.kc = len(self.classes) if len(self.classes) > 2 else 1
        self.loss = "multinomial" if self.kc > 1 else "log"
        if self.X.shape[1] * self.kc > self.max_coef:
            raise NotImplementedError("LogisticRegression(solver='sag' | 'saga') with %d features x %d weight rows: the CUDA "
                                      "path handles up to %d" % (self.X.shape[1], self.kc, self.max_coef))
        self._set_data(self.X, y_class=self.y_class.astype(np.int32))
        if self.folds is not None:
            self.engine.set_train_order(self.folds.train_order)
        self._mss = {}

    def _resolve(self, p):
        """LogisticRegression.fit's checks and penalty resolution (scikit-learn 1.9): ValueError as scikit-learn raises it;
        -> (solver, alpha, beta, C) with alpha / beta sag_solver's L2 and L1 terms before the 1 / n scaling"""
        from sklearn.linear_model import LogisticRegression
        from sklearn.linear_model._logistic import _check_solver
        LogisticRegression(**p)._validate_params()
        if p["penalty"] == "deprecated":
            l1r = p["l1_ratio"]
            if l1r == 0 or l1r is None:
                penalty = "l2"
                if l1r is None:
                    warnings.warn("'l1_ratio=None' was deprecated in version 1.8 and will trigger an error in 1.10. Use "
                                  "0<=l1_ratio<=1 instead.", FutureWarning)
            elif l1r == 1:
                penalty = "l1"
            else:
                penalty = "elasticnet"
            if p["C"] == np.inf:
                penalty = None
        else:
            penalty = p["penalty"]
            warnings.warn("'penalty' was deprecated in version 1.8 and will be removed in 1.10. To avoid this warning, leave "
                          "'penalty' set to its default value and use 'l1_ratio' or 'C' instead. Use l1_ratio=0 instead of "
                          "penalty='l2', l1_ratio=1 instead of penalty='l1', l1_ratio set to a float between 0 and 1 instead "
                          "of penalty='elasticnet', and C=np.inf instead of penalty=None.", FutureWarning)
        solver = _check_solver(p["solver"], penalty, p["dual"])
        if penalty == "elasticnet" and p["l1_ratio"] is None:
            raise ValueError("l1_ratio must be specified when penalty is elasticnet.")
        C = np.inf if p["penalty"] is None else p["C"]
        if p["penalty"] is None:
            penalty = "l2"
        if penalty == "l1":
            alpha, beta = 0.0, 1.0 / C
        elif penalty == "l2":
            alpha, beta = 1.0 / C, 0.0
        else:
            alpha, beta = (1.0 / C) * (1 - p["l1_ratio"]), (1.0 / C) * p["l1_ratio"]
        return solver, alpha, beta

    def _rows(self, k):
        """the training rows of split k in the order the fit sees them (k < 0: every row)"""
        if k < 0:
            return np.arange(len(self.X))
        if self.folds is not None:
            return self.folds.train_order[k]
        return np.flatnonzero(self.fold_id != k)

    def _step(self, k, solver, alpha, beta, fit_intercept):
        """sag_solver's (step, alpha_scaled, beta_scaled) on split k's training rows, computed by scikit-learn's functions in
        X's dtype; ZeroDivisionError where sag_solver raises it"""
        from sklearn.linear_model._sag import get_auto_step_size
        from sklearn.utils.extmath import row_norms
        rows = self._rows(k)
        if k not in self._mss:
            self._mss[k] = row_norms(self.X[rows], squared=True).max()
        n = len(rows)
        a, b = float(alpha) / n, float(beta) / n
        step = get_auto_step_size(self._mss[k], a, self.loss, fit_intercept, n_samples=n, is_saga=solver == "saga")
        if step * a == 1:
            raise ZeroDivisionError("Current sag implementation does not handle the case step_size * alpha_scaled == 1")
        return float(step), a, b

    def _class_weights(self, cw, k):
        """_logistic_regression_path: compute_class_weight on the training rows with their sample weights in X's dtype"""
        from sklearn.utils.class_weight import compute_class_weight
        rows = self._train_rows(k)
        sw = getattr(self, "sample_weight", None)
        sw = np.ones(int(rows.sum())) if sw is None else sw[rows]
        return compute_class_weight(cw, classes=self.classes, y=np.asarray(self.y)[rows], sample_weight=sw.astype(self.X.dtype))

    def _seed(self, random_state):
        return fit_seed(random_state, 1)

    def _candidate(self, p, error_score):
        """-> [n_splits][4] (solver, step, alpha_scaled, beta_scaled) and the [n_splits] fits where sag_solver raises
        ZeroDivisionError"""
        solver, alpha, beta = self._resolve(p)
        fits = np.zeros((self.n_splits, 4))
        zero_div = np.zeros(self.n_splits, bool)
        for k in range(self.n_splits):
            try:
                fits[k] = (solver == "saga",) + self._step(k, solver, alpha, beta, bool(p["fit_intercept"]))
            except ZeroDivisionError:
                if error_score == 'raise':
                    raise
                zero_div[k] = True
                fits[k] = (solver == "saga", 1.0, 0.0, 0.0)
        return (float(p["tol"]), int(p["max_iter"]), bool(p["fit_intercept"])), (fits, zero_div)

    def _prepare(self, my, error_score):
        prepared, _ = super()._prepare(my, error_score)
        return prepared, np.array([zd for _, _, (_, zd) in prepared], bool).reshape(len(my), self.n_splits)

    def _search(self, key, values, cands, return_train):
        tol, max_iter, fit_intercept = key
        f = np.array([fits for fits, _ in values])
        return self.engine.logreg_sag(f[..., 0].astype(np.int64), f[..., 2], f[..., 3], f[..., 1], self._seed_table()[cands],
                                      self.loss, tol=tol, max_iter=max_iter, fit_intercept=fit_intercept,
                                      return_train=return_train, return_stats=True)

    def refit(self, best_params):
        p = self._base_params(best_params)
        solver, alpha, beta = self._resolve(p)
        step, a, b = self._step(-1, solver, alpha, beta, bool(p["fit_intercept"]))
        seed = self._seed(p["random_state"])                  # the refit's own draw, after every search fit's
        self._set_class_weight(p["class_weight"], refit=True)
        try:
            coef, n_iter, status = self.engine.logreg_sag_refit(solver, a, b, step, seed, self.loss, tol=p["tol"],
                                                                max_iter=p["max_iter"], fit_intercept=p["fit_intercept"])
        finally:
            self.engine.set_class_weight(None)
        if status == 2:
            raise _overflow(n_iter)
        est = clone(self.estimator).set_params(**best_params)
        return materialize_logreg_sag(est, self.X, coef, n_iter, self.classes)


def materialize_logreg_sag(est, X, coef, n_iter, classes):
    """Fill a (cloned, parametrised) LogisticRegression with the fitted state of one sag_solver fit coef [K][d + 1] (weights,
    then intercept): coef_ [K][d] and intercept_ [K] in X's dtype (zeros without an intercept), n_iter_ = array([n_iter]),
    classes_, n_features_in_ (linear_model/_logistic.py LogisticRegression.fit), with sag_solver's ConvergenceWarning."""
    d = X.shape[1]
    dt = np.float32 if X.dtype == np.float32 else np.float64
    coef = np.asarray(coef, np.float64)
    est.classes_ = np.asarray(classes)
    est.coef_ = coef[:, :d].astype(dt)
    est.intercept_ = coef[:, d].astype(dt) if est.fit_intercept else np.zeros(len(coef), dt)
    est.n_iter_ = np.array([n_iter], np.int32)
    est.n_features_in_ = int(d)
    if n_iter == est.max_iter:
        from sklearn.exceptions import ConvergenceWarning
        warnings.warn("The max_iter was reached which means the coef_ did not converge", ConvergenceWarning)
    return est


# ------------------------------------------------------------------ LinearSVC -----------------
class LinearSVCPlan(_Plan):
    """sklearn.svm.LinearSVC with liblinear's primal solver (L2R_L2LOSS_SVC: TRON, csrc/linsvc.cu).  X reaches the device in
    float32 or float64 and is widened exactly, as scikit-learn's fit converts it to float64.  Every fit resolves dual='auto'
    from its own training set, as LinearSVC.fit does; a fit that resolves to the dual solver has no CUDA path."""
    scorers = CLASSIFICATION_SCORERS
    supports_sample_weight = True
    class_weighted = True

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

    def _candidate(self, p, error_score):
        for k in range(self.n_splits):
            self._check(p, int(np.count_nonzero(self._train_rows(k))))
        return (float(p["tol"]), int(p["max_iter"]), bool(p["fit_intercept"]), float(p["intercept_scaling"])), float(p["C"])

    def _search(self, key, C, cands, return_train):
        tol, max_iter, fit_intercept, intercept_scaling = key
        return self.engine.linsvc(C, tol=tol, max_iter=max_iter, fit_intercept=fit_intercept,
                                  intercept_scaling=intercept_scaling, return_train=return_train)

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p, len(self.X))
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


# ------------------------------------------------------------------ LinearSVR -----------------
class LinearSVRPlan(_Plan):
    """sklearn.svm.LinearSVR with liblinear's solvers (csrc/linsvr.cu): the dual coordinate descent for
    loss='epsilon_insensitive' (13) and for the squared loss when dual resolves to True (12), TRON otherwise (11).  dual='auto'
    is resolved per training set, as LinearSVR.fit does, so one search can mix 11 and 12.  X reaches the device in float32 or
    float64 and is widened exactly; y is float64.  The CD shuffles the positions of X[train], so every split's training rows
    reach the device in the splitter's order."""
    scorers = REGRESSION_SCORERS
    supports_sample_weight = True
    max_features = 512         # the CD keeps w in registers (include/b200gs.h GS_LINSVR_MAX_FEATURES)

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("LinearSVR needs y")
        y = _target_1d(y, "LinearSVR")
        if self.X.shape[1] > self.max_features:
            raise NotImplementedError("LinearSVR on %d features: the CUDA path handles up to %d"
                                      % (self.X.shape[1], self.max_features))
        self.y = y.astype(np.float64)
        self._set_data(self.X, y_target=self.y.astype(np.float32))
        self.engine.set_targets_f64(self.y)
        if self.folds is not None:
            self.engine.set_train_order(self.folds.train_order)

    def _check(self, p, n_rows):
        """scikit-learn's own checks in LinearSVR.fit's order (parameter constraints, dual resolution on a training set of
        n_rows rows, the liblinear solver of (loss, dual), _fit_liblinear's intercept_scaling test: ValueError), then the
        values without a CUDA path.  Returns the liblinear solver (11, 12 or 13)."""
        from sklearn.svm import LinearSVR
        from sklearn.svm._base import _get_liblinear_solver_type
        from sklearn.svm._classes import _validate_dual_parameter
        LinearSVR(**p)._validate_params()
        dual = _validate_dual_parameter(p["dual"], p["loss"], "l2", "ovr", np.empty((n_rows, self.X.shape[1]), np.bool_))
        solver = _get_liblinear_solver_type("ovr", "l2", p["loss"], dual)
        if p["fit_intercept"] and p["intercept_scaling"] <= 0:
            raise ValueError("Intercept scaling is %r but needs to be greater than 0. To disable fitting an intercept, set "
                             "fit_intercept=False." % p["intercept_scaling"])
        if p["epsilon"] < 0:
            raise NotImplementedError("LinearSVR epsilon=%r has no CUDA path (epsilon >= 0 does)" % (p["epsilon"],))
        return int(solver)

    def _seed(self, random_state):
        return fit_seed(random_state, 0)

    def _candidate(self, p, error_score):
        solvers = [self._check(p, int(np.count_nonzero(self._train_rows(k)))) for k in range(self.n_splits)]
        return ((float(p["tol"]), int(p["max_iter"]), bool(p["fit_intercept"]), float(p["intercept_scaling"])),
                (float(p["C"]), float(p["epsilon"]), solvers))

    def _search(self, key, values, cands, return_train):
        tol, max_iter, fit_intercept, intercept_scaling = key
        return self.engine.linsvr([v[0] for v in values], [v[1] for v in values], [v[2] for v in values],
                                  self._seed_table()[cands], tol=tol, max_iter=max_iter, fit_intercept=fit_intercept,
                                  intercept_scaling=intercept_scaling, return_train=return_train, return_stats=True)

    def refit(self, best_params):
        p = self._base_params(best_params)
        solver = self._check(p, len(self.X))
        seed = self._seed(p["random_state"])                # the refit's own draw, after every search fit's
        raw, n_iter = self.engine.linsvr_refit(p["C"], p["epsilon"], solver, seed, p["tol"], p["max_iter"], p["fit_intercept"],
                                               p["intercept_scaling"])
        est = clone(self.estimator).set_params(**best_params)
        return materialize_linsvr(est, raw, n_iter, self.X.shape[1])


def materialize_linsvr(est, raw, n_iter, n_features):
    """Fill a (cloned, parametrised) sklearn.svm.LinearSVR with the fitted state of liblinear's raw weights raw [n_features + 1]
    (the bias feature's weight last) and the fit's iteration count (svm/_base.py _fit_liblinear, svm/_classes.py
    LinearSVR.fit: coef_ raveled, intercept_ = intercept_scaling x the bias weight as a 1-element array, or 0.0; n_iter_ an
    int), with scikit-learn's ConvergenceWarning."""
    raw = np.asarray(raw, np.float64)
    est.coef_ = raw[:n_features].copy()
    est.intercept_ = est.intercept_scaling * raw[n_features:n_features + 1] if est.fit_intercept else 0.0
    est.n_iter_ = int(n_iter)
    est.n_features_in_ = int(n_features)
    if est.n_iter_ >= est.max_iter:
        from sklearn.exceptions import ConvergenceWarning
        warnings.warn("Liblinear failed to converge, increase the number of iterations.", ConvergenceWarning)
    return est


# ------------------------------------------------------------------ SGDClassifier / SGDRegressor
def sgd_seeds(random_state, n_classes):
    """The shuffle seeds scikit-learn hands to _plain_sgd for one fit (n_classes 0: a regressor), drawing from
    check_random_state(random_state) as fit does: binary fit_binary draws make_dataset's seed, then the shuffle seed;
    one-vs-rest draws one seed per class and each class fit makes those two draws from RandomState(seed); _fit_regressor
    draws the shuffle seed, then make_dataset's (_random_state)."""
    rs = _random_state(random_state)
    if n_classes == 0:
        seed = int(rs.randint(0, _INT_MAX))
        rs.randint(1, _INT_MAX)
        return [seed]
    if n_classes == 2:
        rs.randint(1, _INT_MAX)
        return [int(rs.randint(_INT_MAX))]
    out = []
    for s in rs.randint(_INT_MAX, size=n_classes):
        r = np.random.RandomState(s)
        r.randint(1, _INT_MAX)
        out.append(int(r.randint(_INT_MAX)))
    return out


class SGDPlan(_Plan):
    """sklearn.linear_model.SGDClassifier / SGDRegressor (csrc/sgd.cu): _plain_sgd restated step for step, one warp per
    (candidate, split, one-vs-rest class) fit.  X reaches the device in its own dtype (float32 runs _plain_sgd32, as
    scikit-learn does), dense; the shuffle permutes the positions of X[train], so every split's training rows reach the
    device in the splitter's order."""
    scorers = CLASSIFICATION_SCORERS
    supports_sample_weight = True
    class_weighted = True
    fail_warning = "%d fits failed with a floating-point under-/overflow; their scores are error_score=%r"
    max_features = 512         # w and q live in registers (include/b200gs.h GS_SGD_MAX_FEATURES)

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        import scipy.sparse as sp
        from sklearn.linear_model import SGDClassifier
        name = type(estimator).__name__
        if sp.issparse(X):
            raise NotImplementedError("%s on sparse X has no CUDA path (scikit-learn's sparse SGD decays the intercept and "
                                      "touches only the stored entries): pass a dense X" % name)
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        if y is None:
            raise ValueError("%s needs y" % name)
        self.classifier = isinstance(estimator, SGDClassifier)
        if self.X.shape[1] > self.max_features:
            raise NotImplementedError("%s on %d features: the CUDA path handles up to %d" % (name, self.X.shape[1], self.max_features))
        y = np.asarray(y)
        if self.classifier:
            self.classes, self.y_class = np.unique(y, return_inverse=True)
            if len(self.classes) < 2:
                raise ValueError("The number of classes has to be greater than one; got %d class" % len(self.classes))
            if len(self.classes) > 64:
                raise NotImplementedError("%s CUDA path handles up to 64 classes (got %d)" % (name, len(self.classes)))
            self._set_data(self.X, y_class=self.y_class.astype(np.int32))
            self.kc = len(self.classes) if len(self.classes) > 2 else 1
        else:
            if y.ndim != 1:
                raise NotImplementedError("multi-output %s is not supported by the CUDA path" % name)
            self.y = y.astype(np.float64)
            self._set_data(self.X, y_target=self.y.astype(np.float32))
            self.engine.set_targets_f64(self.y)
            self.kc = 1
        if self.folds is not None:
            self.engine.set_train_order(self.folds.train_order)

    def _check(self, p):
        """scikit-learn's own checks (ValueError), then the settings without a CUDA path"""
        est = type(self.estimator)(**p)
        est._validate_params()
        est._more_validate_params()
        name = type(self.estimator).__name__
        if p["early_stopping"]:
            raise NotImplementedError("%s early_stopping=True has no CUDA path" % name)
        if p["average"] is not False and p["average"] != 0:
            raise NotImplementedError("%s average=%r has no CUDA path" % (name, p["average"]))
        if p["learning_rate"] in ("pa1", "pa2"):
            raise NotImplementedError("%s learning_rate=%r has no CUDA path" % (name, p["learning_rate"]))
        return est

    def _class_weights(self, cw, k):
        """SGD's class weights ignore sample weights: compute_class_weight(class_weight, classes, y_train)"""
        from sklearn.utils.class_weight import compute_class_weight
        return compute_class_weight(cw, classes=self.classes, y=np.asarray(self.y)[self._train_rows(k)])

    def _seed(self, random_state):
        return sgd_seeds(random_state, len(self.classes) if self.classifier else 0)

    @staticmethod
    def _fit_args(p):
        return dict(loss=p["loss"], penalty=p["penalty"], alpha=float(p["alpha"]),
                    l1_ratio=float(0.0 if p["l1_ratio"] is None else p["l1_ratio"]), epsilon=float(p["epsilon"]),
                    learning_rate=p["learning_rate"], eta0=float(p["eta0"]), power_t=float(p["power_t"]))

    def _candidate(self, p, error_score):
        self._check(p)
        key = (None if p["tol"] is None else float(p["tol"]), int(p["max_iter"]), int(p["n_iter_no_change"]),
               bool(p["fit_intercept"]), bool(p["shuffle"]))
        return key, self._fit_args(p)

    def _search(self, key, args, cands, return_train):
        tol, max_iter, n_iter_no_change, fit_intercept, shuffle = key
        return self.engine.sgd(*[[a[k] for a in args] for k in ("loss", "penalty", "alpha", "l1_ratio", "epsilon", "learning_rate",
                                                                "eta0", "power_t")],
                               self._seed_table()[cands], tol=tol, max_iter=max_iter, n_iter_no_change=n_iter_no_change,
                               fit_intercept=fit_intercept, shuffle=shuffle, return_train=return_train, return_stats=True)

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        seeds = self._seed(p["random_state"])                   # the refit's own draw, after every search fit's
        cw_ = self._set_class_weight(p["class_weight"], refit=True) if self.classifier else None
        try:
            coef, n_iter, status = self.engine.sgd_refit(**self._fit_args(p), seed=seeds, tol=p["tol"], max_iter=p["max_iter"],
                                                         n_iter_no_change=p["n_iter_no_change"], fit_intercept=p["fit_intercept"],
                                                         shuffle=p["shuffle"])
        finally:
            if self.classifier:
                self.engine.set_class_weight(None)
        if (status == 2).any():
            raise _overflow(int(n_iter[int(np.argmax(status == 2))]))
        est = clone(self.estimator).set_params(**best_params)
        return materialize_sgd(est, self.X, coef, n_iter, self.classes if self.classifier else None, cw_)


class SGDRegressorPlan(SGDPlan):
    scorers = REGRESSION_SCORERS
    class_weighted = False


def materialize_sgd(est, X, coef, n_iter, classes, class_weight):
    """Fill a (cloned, parametrised) SGDClassifier / SGDRegressor with the fitted state of its per-class fits coef
    [KC][d + 1] (coef, then intercept) and n_iter [KC] (linear_model/_stochastic_gradient.py _fit_binary, _fit_multiclass,
    _fit_regressor: coef_ in X's dtype; intercept_ float64 but for one-vs-rest; n_iter_ the maximum over the classes;
    t_ = 1 + n_iter_ x n_samples; the classifier's _loss_function_), with scikit-learn's ConvergenceWarning."""
    d = X.shape[1]
    dt = np.float32 if X.dtype == np.float32 else np.float64
    coef = np.asarray(coef, np.float64)
    if classes is not None:
        est.classes_ = np.asarray(classes)
        est._expanded_class_weight = np.asarray(class_weight, np.float64)
        est.coef_ = coef[:, :d].astype(dt)
        est.intercept_ = coef[:, d].astype(dt if len(classes) > 2 else np.float64)
    else:
        est.coef_ = coef[0, :d].astype(dt)
        est.intercept_ = coef[0, d:].astype(np.float64)
    est.n_iter_ = int(np.max(n_iter))
    est.t_ = 1.0 + est.n_iter_ * X.shape[0]
    est.n_features_in_ = int(d)
    if classes is not None:                                   # SGDClassifier.fit keeps its loss object; the regressor does not
        est._loss_function_ = est._get_loss_function(est.loss)
    if est.tol is not None and est.tol > -np.inf and est.n_iter_ == est.max_iter:
        from sklearn.exceptions import ConvergenceWarning
        warnings.warn("Maximum number of iteration reached before convergence. Consider increasing max_iter to improve the "
                      "fit.", ConvergenceWarning)
    return est


# ------------------------------------------------------------------ k-nearest neighbours ------
_KNN_METRICS = {"euclidean": "euclidean", "l2": "euclidean", "manhattan": "manhattan", "l1": "manhattan",
                "cityblock": "manhattan"}


class KNeighborsPlan(_Plan):
    """sklearn.neighbors.KNeighborsClassifier / KNeighborsRegressor (csrc/knn.cu).  A fit stores its training rows; every
    (candidate, split) task's scorer queries the neighbours of its test rows (and, for the train score, of its training
    rows).  The engine selects the max n_neighbors nearest training rows once per (split, metric) and every candidate votes
    from those lists.  The refit is scikit-learn's own fit (it stores the data, plus a tree index when scikit-learn builds
    one: there is no arithmetic for the device to take over)."""
    # One GPU: the neighbour selection is the cost of the whole search and every candidate shares it, so dealing candidates
    # to several GPUs would repeat it on each.  Under torchrun each rank still evaluates the candidates it is dealt.
    multi_device = False
    scorers = CLASSIFICATION_SCORERS
    max_neighbors = 256

    def __init__(self, estimator, cands, X, y, fold_id, n_splits, device=None):
        super().__init__(estimator, cands, X, y, fold_id, n_splits, device)
        from sklearn.neighbors import KNeighborsClassifier
        name = type(estimator).__name__
        if y is None:
            raise ValueError("%s needs y" % name)
        self.classifier = isinstance(estimator, KNeighborsClassifier)
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

    def _candidate(self, p, error_score):
        return (), self._check(p)                         # one group: every candidate shares the neighbour selection

    def _prepare(self, my, error_score):
        """a fit whose n_neighbors exceeds its training rows fails, as scikit-learn's predict does"""
        prepared, _ = super()._prepare(my, error_score)
        m_train = [int(np.count_nonzero(self._train_rows(k))) for k in range(self.n_splits)]
        too_many = np.array([[nn > m_train[k] for k in range(self.n_splits)] for _, _, (nn, _, _) in prepared],
                            bool).reshape(len(my), self.n_splits)
        if too_many.any() and error_score == 'raise':
            j, k = map(int, np.argwhere(too_many)[0])
            n_test = int(np.count_nonzero(self._test_rows(k)))
            raise ValueError("Expected n_neighbors <= n_samples_fit, but n_neighbors = %d, n_samples_fit = %d, n_samples = %d"
                             % (prepared[j][2][0], m_train[k], n_test))
        return prepared, too_many

    def _search(self, key, values, cands, return_train):
        return self.engine.knn([v[0] for v in values], [v[1] for v in values], [v[2] for v in values],
                               return_train=return_train, y_f32=not self.classifier and self.y_f32)

    def refit(self, best_params):
        p = self._base_params(best_params)
        self._check(p)
        return clone(self.estimator).set_params(**best_params).fit(self.X, self.y)


class KNeighborsRegressorPlan(KNeighborsPlan):
    scorers = REGRESSION_SCORERS


# The names the plan classes had when adapters were separate classes: code that imports them keeps working.
SVCAdapter, NuSVCAdapter, SVRAdapter, NuSVRAdapter = SVCPlan, NuSVCPlan, SVRPlan, NuSVRPlan
RidgeAdapter, ENetAdapter, LogRegAdapter = RidgePlan, ENetPlan, LogRegPlan
LinearSVCAdapter, LinearSVRAdapter, SGDClassifierAdapter, SGDRegressorAdapter = LinearSVCPlan, LinearSVRPlan, SGDPlan, SGDRegressorPlan
KNeighborsAdapter, KNeighborsRegressorAdapter = KNeighborsPlan, KNeighborsRegressorPlan
