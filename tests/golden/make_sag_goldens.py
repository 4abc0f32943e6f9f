"""Write the LogisticRegression(solver='sag' | 'saga') goldens (tests/golden/sag_small.npz, sag_multi.npz) with
scikit-learn 1.9 on the CPU: the workload's GridSearchCV (cv=5) split test scores and mean test scores, best_index_, every
(candidate, split) fit's n_iter_ (fitted one task at a time, in GridSearchCV's order) and the refit's coef_ / intercept_ /
n_iter_.  Run from the repository root: python tests/golden/make_sag_goldens.py"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    from sklearn.base import clone
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.model_selection import GridSearchCV, ParameterGrid, StratifiedKFold
    from spark_sklearn_b200 import workloads as W
    warnings.simplefilter("ignore", ConvergenceWarning)
    for key in ("sag_small", "sag_multi"):
        w = W.make_workload(key)
        X, y = w["X"], w["y"]
        est = W.make_estimator(w)
        gs = GridSearchCV(est, w["param_grid"], cv=5).fit(X, y)
        cands = list(ParameterGrid(w["param_grid"]))
        splits = list(StratifiedKFold(5).split(X, y))
        n_iter = np.array([[clone(est).set_params(**c).fit(X[tr], y[tr]).n_iter_[0] for tr, _ in splits] for c in cands])
        be = gs.best_estimator_
        np.savez(os.path.join(ROOT, "tests", "golden", key + ".npz"),
                 split_test=np.stack([gs.cv_results_["split%d_test_score" % k] for k in range(5)], 1),
                 mean_test=gs.cv_results_["mean_test_score"], best_index=gs.best_index_,
                 n_iter=n_iter, refit_coef=be.coef_, refit_intercept=be.intercept_, refit_n_iter=be.n_iter_)
        print(key, gs.best_params_, n_iter.min(), n_iter.max())


if __name__ == "__main__":
    main()
