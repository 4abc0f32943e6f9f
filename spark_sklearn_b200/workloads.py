"""Synthetic workloads for the BASELINE.json configs (SURVEY.md §8d recipes).

Every recipe is deterministic (``random_state=0``), fp32, C-contiguous.  They are
shared by ``bench.py``, the parity tests and ``tests/golden/make_goldens.py`` so
that the GPU path, the oracle and the committed goldens all see identical bytes.

A workload is a dict: ``X, y, estimator (name), param_grid | param_distributions,
cv, search ("grid" | "random"), n_iter, random_state``.
"""
import numpy as np

__all__ = ["make_workload", "WORKLOADS"]


def _c1():
    from sklearn.datasets import load_iris
    iris = load_iris()
    return dict(name="c1_iris_svc", X=np.ascontiguousarray(iris.data), y=iris.target,
                estimator="SVC", est_params={"gamma": "auto"},
                param_grid={"kernel": ("linear", "rbf"), "C": [1, 10]}, cv=5, search="grid")


def _svc_data(n=10000, d=512):
    from sklearn.datasets import make_classification
    from sklearn.preprocessing import StandardScaler
    X, y = make_classification(n_samples=n, n_features=d, n_informative=d // 8, n_redundant=0,
                               n_classes=2, class_sep=1.0, flip_y=0.01, random_state=0)
    X = StandardScaler().fit_transform(X).astype(np.float32)
    return np.ascontiguousarray(X), y.astype(np.int64)


def _c2(n=10000, d=512, nc=8, ng=8, cv=5, name="c2_svc_rbf_8x8"):
    X, y = _svc_data(n, d)
    grid = {"C": np.logspace(-1, 2.5, nc), "gamma": np.geomspace(8.0 / (d * 64), 8.0 / (d * 4), ng)}
    # d=512 -> gamma in [1/4096, 1/256] exactly as SURVEY.md §8d states
    return dict(name=name, X=X, y=y, estimator="SVC", est_params={"kernel": "rbf"},
                param_grid=grid, cv=cv, search="grid")


def _c4():
    return _c2(nc=16, ng=16, name="c4_svc_rbf_16x16")


def _c3(n=50000, d=256, n_iter=256, cv=5, name="c3_logreg_random256"):
    from sklearn.datasets import make_classification
    from sklearn.preprocessing import StandardScaler
    from scipy.stats import loguniform
    X, y = make_classification(n_samples=n, n_features=d, n_informative=d // 8, n_redundant=0,
                               n_classes=2, class_sep=0.5, flip_y=0.02, random_state=0)
    X = np.ascontiguousarray(StandardScaler().fit_transform(X).astype(np.float32))
    return dict(name=name, X=X, y=y.astype(np.int64), estimator="LogisticRegression", est_params={},
                param_distributions={"C": loguniform(1e-4, 1e2)}, n_iter=n_iter, random_state=0,
                cv=cv, search="random")


def _c5(n=20000, d=1024, n_alpha=512, cv=10, name="c5_ridge_512"):
    from sklearn.datasets import make_regression
    X, y = make_regression(n_samples=n, n_features=d, n_informative=d // 8, noise=10.0, random_state=0)
    return dict(name=name, X=np.ascontiguousarray(X.astype(np.float32)), y=y.astype(np.float32),
                estimator="Ridge", est_params={}, param_grid={"alpha": np.logspace(-3, 5, n_alpha)},
                cv=cv, search="grid")


def _lasso(n=20000, d=1024, n_alpha=32, cv=10, name="lasso_1024", enet=False):
    """The estimator of the reference's own search tests (tests/test_search_2.py:69-119) on config 5's data recipe."""
    w = _c5(n=n, d=d, n_alpha=2, cv=cv, name=name)
    if enet:
        w.update(estimator="ElasticNet", param_grid={"alpha": np.logspace(-2, 1.5, n_alpha), "l1_ratio": [0.2, 0.7]})
    else:
        w.update(estimator="Lasso", param_grid={"alpha": np.logspace(-2, 2, n_alpha)})
    return w


def _svr(n=1000, d=32, grid=None, cv=5, name="svr_small"):
    """epsilon-SVR: make_regression, X standardised then fp32, y standardised in float64 (SVR's epsilon is in y units)."""
    from sklearn.datasets import make_regression
    from sklearn.preprocessing import StandardScaler
    X, y = make_regression(n_samples=n, n_features=d, n_informative=8, noise=10.0, random_state=0)
    X = np.ascontiguousarray(StandardScaler().fit_transform(X).astype(np.float32))
    y = (y - y.mean()) / y.std()
    if grid is None:
        grid = {"C": [0.1, 1.0, 10.0, 100.0], "gamma": [1.0 / 256, 1.0 / 32, "scale"], "epsilon": [0.05, 0.2]}
    return dict(name=name, X=X, y=y.astype(np.float64), estimator="SVR", est_params={"kernel": "rbf"},
                param_grid=grid, cv=cv, search="grid")


def _svc_kernels(n=3000, d=128, cv=5, name="svc_kernels_mid"):
    """SVC over the poly and sigmoid kernels (with a few rbf and linear candidates) on the config-2 data recipe: the
    list-of-dicts grid shape of the reference's own cv_results_ example (grid_search.py:120-160)."""
    X, y = _svc_data(n, d)
    grid = [{"kernel": ["poly"], "degree": [2, 3], "coef0": [0.0, 1.0], "C": [0.1, 1.0, 10.0]},
            {"kernel": ["sigmoid"], "gamma": [1.0 / 1024, "scale"], "coef0": [-1.0, 0.0], "C": [0.1, 1.0, 10.0]},
            {"kernel": ["rbf"], "gamma": [1.0 / 512], "C": [1.0, 10.0]},
            {"kernel": ["linear"], "C": [0.01]}]
    return dict(name=name, X=X, y=y, estimator="SVC", est_params={}, param_grid=grid, cv=cv, search="grid")


def _linsvc(which="small"):
    """LinearSVC (primal TRON): the config-3 data with 8 C values (small), a 3-class set (multi), and config 3's own
    search shape on its data (c3: 256 random C candidates x 5 folds = 1280 fits of 40000 x 256, all primal)."""
    from scipy.stats import loguniform
    if which == "multi":
        from sklearn.datasets import make_classification
        from sklearn.preprocessing import StandardScaler
        X, y = make_classification(n_samples=3000, n_features=64, n_informative=16, n_redundant=0, n_classes=3,
                                   class_sep=0.8, flip_y=0.02, random_state=0)
        X = np.ascontiguousarray(StandardScaler().fit_transform(X).astype(np.float32))
        return dict(name="linsvc_multi", X=X, y=y.astype(np.int64), estimator="LinearSVC", est_params={},
                    param_grid={"C": np.logspace(-3, 1, 6)}, cv=5, search="grid")
    if which == "c3":
        w = _c3(name="linsvc_c3")
        w.update(estimator="LinearSVC", param_distributions={"C": loguniform(1e-4, 1e2)})
        return w
    w = _c3(n=4000, d=32, name="linsvc_small")
    w.update(estimator="LinearSVC", search="grid", param_grid={"C": np.logspace(-4, 2, 8)})
    return w


def _knn(which="small"):
    """k-nearest neighbours: config 3's recipe at 2000 x 32 (small, binary), a 4-class set (multi), the SVR recipe (reg_small),
    config 2's data with a 200-fit grid (c2) and config 3's 50000 x 256 data with a smaller grid (c3: the row-slab case)."""
    grid = {"n_neighbors": [1, 3, 5, 15], "weights": ["uniform", "distance"], "p": [1, 2]}
    if which == "reg_small":
        w = _svr(name="knn_reg_small", grid=grid)
        w.update(estimator="KNeighborsRegressor", est_params={})
        return w
    if which == "multi":
        from sklearn.datasets import make_classification
        from sklearn.preprocessing import StandardScaler
        X, y = make_classification(n_samples=2000, n_features=32, n_informative=12, n_redundant=0, n_classes=4,
                                   class_sep=1.0, flip_y=0.02, random_state=0)
        X = np.ascontiguousarray(StandardScaler().fit_transform(X).astype(np.float32))
        return dict(name="knn_multi", X=X, y=y.astype(np.int64), estimator="KNeighborsClassifier", est_params={},
                    param_grid=grid, cv=5, search="grid")
    if which == "c2":
        X, y = _svc_data()
        return dict(name="knn_c2", X=X, y=y, estimator="KNeighborsClassifier", est_params={},
                    param_grid={"n_neighbors": [1, 2, 3, 5, 8, 13, 21, 34, 55, 89], "weights": ["uniform", "distance"],
                                "p": [1, 2]}, cv=5, search="grid")
    if which == "c3":
        w = _c3(name="knn_c3")
        w.update(estimator="KNeighborsClassifier", est_params={}, search="grid",
                 param_grid={"n_neighbors": [5, 21], "weights": ["uniform", "distance"], "p": [1, 2]})
        return w
    w = _c3(n=2000, d=32, name="knn_small")
    w.update(estimator="KNeighborsClassifier", est_params={}, search="grid", param_grid=grid)
    return w


WORKLOADS = {
    "c1": _c1, "c2": _c2, "c3": _c3, "c4": _c4, "c5": _c5,
    # reduced-size variants: same recipes, sizes the CPU oracle finishes in seconds
    "c2_small": lambda: _c2(n=1000, d=64, nc=4, ng=4, name="c2_small"),
    "c2_mid": lambda: _c2(n=3000, d=128, nc=4, ng=4, name="c2_mid"),
    "c3_small": lambda: _c3(n=4000, d=32, n_iter=16, name="c3_small"),
    "c5_small": lambda: _c5(n=2000, d=64, n_alpha=32, cv=10, name="c5_small"),
    # SURVEY.md 8f-2: Lasso / ElasticNet on the fold Grams
    "lasso_1024": _lasso,
    "lasso_small": lambda: _lasso(n=2000, d=64, n_alpha=16, cv=5, name="lasso_small"),
    "enet_small": lambda: _lasso(n=1500, d=200, n_alpha=6, cv=4, name="enet_small", enet=True),
    # epsilon-SVR (SURVEY.md 8f-2): svr_c6 is the measurement config (8 x 8 C x gamma, 8000 training rows per fit)
    "svr_small": _svr,
    "svr_mid": lambda: _svr(n=5000, d=128, grid={"C": [0.3, 3.0, 30.0], "gamma": [1.0 / 1024, 1.0 / 128, "scale"],
                                                 "epsilon": [0.1]}, name="svr_mid"),
    "svr_c6": lambda: _svr(n=10000, d=512, grid={"C": np.logspace(-1, 2.5, 8), "gamma": np.geomspace(1.0 / 4096, 1.0 / 256, 8),
                                                 "epsilon": [0.1]}, name="svr_c6"),
    # SVC poly / sigmoid: the golden-sized grid and the same grid on config-2 data (tools/bench_kernels.py)
    "svc_kernels_mid": _svc_kernels,
    "svc_kernels_c2": lambda: _svc_kernels(n=10000, d=512, name="svc_kernels_c2"),
    # LinearSVC, primal TRON (csrc/linsvc.cu): golden-sized binary and 3-class grids, and config 3's search (tools/bench_linsvc.py)
    "linsvc_small": _linsvc,
    "linsvc_multi": lambda: _linsvc("multi"),
    "linsvc_c3": lambda: _linsvc("c3"),
    # k-nearest neighbours (csrc/knn.cu): one neighbour selection per (split, metric) serves every candidate
    "knn_small": _knn,
    "knn_multi": lambda: _knn("multi"),
    "knn_reg_small": lambda: _knn("reg_small"),
    "knn_c2": lambda: _knn("c2"),
    "knn_c3": lambda: _knn("c3"),
}


def make_workload(key):
    return WORKLOADS[key]()


def make_estimator(w):
    """Instantiate the sklearn estimator a workload names."""
    if w["estimator"] == "SVC":
        from sklearn.svm import SVC
        return SVC(**w["est_params"])
    if w["estimator"] == "LogisticRegression":
        from sklearn.linear_model import LogisticRegression
        return LogisticRegression(**w["est_params"])
    if w["estimator"] == "Ridge":
        from sklearn.linear_model import Ridge
        return Ridge(**w["est_params"])
    if w["estimator"] == "SVR":
        from sklearn.svm import SVR
        return SVR(**w["est_params"])
    if w["estimator"] == "LinearSVC":
        from sklearn.svm import LinearSVC
        return LinearSVC(**w["est_params"])
    if w["estimator"] in ("KNeighborsClassifier", "KNeighborsRegressor"):
        import sklearn.neighbors as nb
        return getattr(nb, w["estimator"])(**w["est_params"])
    if w["estimator"] in ("Lasso", "ElasticNet"):
        import sklearn.linear_model as lm
        return getattr(lm, w["estimator"])(**w["est_params"])
    raise ValueError(w["estimator"])


def candidates(w):
    """The candidate list exactly as the reference enumerates it
    (ParameterGrid: reference grid_search.py:246; ParameterSampler: random_search.py:222)."""
    from sklearn.model_selection import ParameterGrid, ParameterSampler
    if w["search"] == "grid":
        return list(ParameterGrid(w["param_grid"]))
    return list(ParameterSampler(w["param_distributions"], w["n_iter"], random_state=w["random_state"]))
