#!/usr/bin/env python
"""Run one BASELINE workload through the C ABI on cuda:0, print the device profile, save the score
arrays to <name>_gpu.npz in the current directory and compare with tests/golden/<name>.npz when it exists."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spark_sklearn_b200 import workloads as W  # noqa: E402
from spark_sklearn_b200.estimators import get_engine, fold_ids_from_splits  # noqa: E402


def main(key, reps=2):
    from sklearn.model_selection import check_cv
    w = W.make_workload(key)
    X, y = w["X"], w["y"]
    cands = W.candidates(w)
    eng = get_engine(0)
    cv = check_cv(w["cv"], y, classifier=w["estimator"] in ("SVC", "LogisticRegression"))
    splits = list(cv.split(X, y))
    fold_id = fold_ids_from_splits(splits, len(y))
    out = None
    for rep in range(reps):
        t0 = time.time()
        if w["estimator"] == "SVC":
            eng.set_data(X, fold_id, len(splits), y_class=y.astype(np.int32))
            t1 = time.time()
            d = X.shape[1]
            kern = [c.get("kernel", w["est_params"].get("kernel", "rbf")) for c in cands]
            gam = [1.0 / d if c.get("gamma", w["est_params"].get("gamma")) == "auto" else float(c.get("gamma", 0)) for c in cands]
            out = eng.svc(kern, [float(c["C"]) for c in cands], np.array(gam)[:, None])
        elif w["estimator"] == "Ridge":
            eng.set_data(X, fold_id, len(splits), y_target=y)
            t1 = time.time()
            out = eng.ridge([float(c["alpha"]) for c in cands])
        elif w["estimator"] in ("Lasso", "ElasticNet"):
            eng.set_data(X, fold_id, len(splits), y_target=y)
            t1 = time.time()
            out = eng.enet([float(c["alpha"]) for c in cands], [float(c.get("l1_ratio", 1.0)) for c in cands])
        else:
            eng.set_data(X, fold_id, len(splits), y_class=y.astype(np.int32))
            t1 = time.time()
            out = eng.logreg([float(c["C"]) for c in cands])
        t2 = time.time()
        p = eng.profile()
        nfit = len(cands) * len(splits)
        print("%s rep%d: set_data %.1f ms, search %.1f ms wall -> %.1f fits/s | profile %s"
              % (key, rep, (t1 - t0) * 1e3, (t2 - t1) * 1e3, nfit / (t2 - t1),
                 {k: (round(v, 3) if isinstance(v, float) else v) for k, v in p.items()}), flush=True)
    np.savez(w["name"] + "_gpu.npz", **{k: v for k, v in out.items() if v is not None})
    gp = os.path.join(ROOT, "tests", "golden", w["name"] + ".npz")
    if os.path.exists(gp):
        g = np.load(gp)
        dt = np.abs(out["test"] - g["test_scores"])
        print("parity vs golden: max|d split test| %.3g  max|d mean_test| %.3g  n_iter equal: %s"
              % (dt.max(), np.abs(out["test"].mean(1) - g["test_scores"].mean(1)).max(),
                 np.array_equal(out.get("n_iter"), g["diag"][:, :, 0].astype(np.int32)) if "n_iter" in out else "n/a"))
    if "n_iter" in out:
        it = out["n_iter"]
        print("n_iter: min %d median %d max %d total %d; fit_ms max %.1f" % (it.min(), np.median(it), it.max(), it.sum(), out["fit_ms"].max()))

    if "n_iter" in out and os.environ.get("B200GS_PRINT_US"):
        us = out["fit_ms"] * 1e3 / np.maximum(out["n_iter"], 1)
        o = np.argsort(-out["n_iter"].ravel())
        print("us/iter: longest10 %s | median all %.2f | min %.2f max %.2f" % (np.round(us.ravel()[o[:10]], 2), np.median(us), us.min(), us.max()))


if __name__ == "__main__":
    main(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 2)
