"""Regenerate the k-NN golden from scikit-learn (1.9): every split's test and train score of the knn_c2 search (config 2's
10000 x 512 data, 10 n_neighbors x 2 weights x 2 metrics, StratifiedKFold(5): 200 fits), as scikit-learn's own
GridSearchCV(return_train_score=True) computes them.

    python tests/golden/make_knn_goldens.py            # knn_c2.npz (minutes on 8 cores)
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from spark_sklearn_b200 import workloads as W  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    from sklearn.model_selection import GridSearchCV
    w = W.make_workload("knn_c2")
    cands = W.candidates(w)
    s = GridSearchCV(W.make_estimator(w), w["param_grid"], cv=w["cv"], return_train_score=True, n_jobs=os.cpu_count(),
                     refit=False).fit(w["X"], w["y"])
    r = s.cv_results_
    assert [dict(p) for p in r["params"]] == cands
    ns = w["cv"]
    test = np.stack([r["split%d_test_score" % k] for k in range(ns)], 1)
    train = np.stack([r["split%d_train_score" % k] for k in range(ns)], 1)
    np.savez_compressed(os.path.join(HERE, "knn_c2.npz"), test=test, train=train, best_index=np.int32(s.best_index_))
    print("knn_c2: best", s.best_params_, "mean_test_score %.6f" % s.best_score_)


if __name__ == "__main__":
    main()
