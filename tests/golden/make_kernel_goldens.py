"""Regenerate the SVC poly / sigmoid golden from scikit-learn itself (sklearn.svm.SVC, libsvm):

    python tests/golden/make_kernel_goldens.py [--jobs N]

svc_kernels_mid.npz holds, for the workload's ParameterGrid order (a list of grids: poly, sigmoid, rbf, linear) x its
StratifiedKFold splits: test_scores, train_scores (accuracy), n_iter (n_iter_ summed over the one-vs-one pairs) and n_sv
(support vectors) of SVC(**est_params, **candidate).fit(X[train], y[train]).
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def _fit(X, y, params, train, test):
    from sklearn.svm import SVC
    m = SVC(**params).fit(X[train], y[train])
    return m.score(X[test], y[test]), m.score(X[train], y[train]), int(np.sum(m.n_iter_)), int(np.sum(m.n_support_))


def make(key, jobs):
    from joblib import Parallel, delayed
    from sklearn.model_selection import check_cv
    from spark_sklearn_b200 import workloads as W
    w = W.make_workload(key)
    X, y = w["X"], w["y"]
    cands = W.candidates(w)
    splits = list(check_cv(w["cv"], y, classifier=True).split(X, y))
    out = Parallel(n_jobs=jobs)(delayed(_fit)(X, y, dict(w["est_params"], **c), a, b) for c in cands for a, b in splits)
    out = np.array(out).reshape(len(cands), len(splits), 4)
    np.savez_compressed(os.path.join(HERE, key + ".npz"), test_scores=out[..., 0], train_scores=out[..., 1],
                        n_iter=out[..., 2].astype(np.int64), n_sv=out[..., 3].astype(np.int64))
    print(key, out.shape[:2], "n_iter %d..%d" % (out[..., 2].min(), out[..., 2].max()),
          "accuracy %.3f..%.3f" % (out[..., 0].min(), out[..., 0].max()))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("keys", nargs="*", default=["svc_kernels_mid"])
    ap.add_argument("--jobs", type=int, default=-1)
    a = ap.parse_args()
    for key in a.keys:
        make(key, a.jobs)
