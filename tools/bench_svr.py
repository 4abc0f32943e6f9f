"""Measure the epsilon-SVR search on one GPU: fits/s from CUDA events with X resident, the phase split, the SMO solve's
HBM traffic as a fraction of the H100's 3.35 TB/s, and scikit-learn's GridSearchCV(n_jobs=cores) on a subset of the
candidates for comparison (with a parity check on that subset).

    python tools/bench_svr.py [--workload svr_c6] [--steps 1] [--sk-cands 2]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM5 80 GB peak
# smo_hbm_fraction counts the l K entries of the training rows read per gathered row (2 rows per iteration).  Fits with
# 2049..4096 training rows run on the bulk-row-copy instance, which moves whole K rows (n floats): there the bytes actually
# moved are n / l times the count.  svr_c6 (8000-row fits) runs on the gather instance, where the count is the traffic.


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="svr_c6")
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--sk-cands", type=int, default=2, help="candidates scikit-learn fits for comparison (0: skip)")
    a = ap.parse_args()

    from sklearn.model_selection import GridSearchCV as SkGridSearchCV, KFold, ParameterGrid
    from sklearn.svm import SVR
    from spark_sklearn_b200.estimators import Folds, SVRPlan
    from spark_sklearn_b200 import workloads as W

    w = W.make_workload(a.workload)
    X, y, cv = w["X"], w["y"], w["cv"]
    cands = list(ParameterGrid(w["param_grid"]))
    splits = list(KFold(cv).split(X))
    plan = SVRPlan.plan(SVR(**w["est_params"]), cands, X, y, Folds(splits, len(X)), cv)   # X, y resident from here
    n_fits = len(cands) * cv

    plan.evaluate([0])                                            # warm-up: library load, kernel attributes, buffers
    runs = []
    for _ in range(a.steps):
        res = plan.evaluate(list(range(len(cands))))
        runs.append(dict(plan.profile()))
    prof = min(runs, key=lambda p: p["ms_total"])
    ms = prof["ms_total"]
    solve_s = prof["ms_solve"] * 1e-3
    out = dict(workload=a.workload, n=int(X.shape[0]), d=int(X.shape[1]), candidates=len(cands), folds=cv, fits=n_fits,
               gpu_ms=round(ms, 2), fits_per_s=round(n_fits / (ms * 1e-3), 2),
               ms_gram=round(prof["ms_gram"], 2), ms_kernel_matrix=round(prof["ms_kernel_matrix"], 2),
               ms_solve=round(prof["ms_solve"], 2), ms_score=round(prof["ms_score"], 2),
               smo_iterations=int(prof["smo_iterations"]),
               smo_hbm_fraction=round(prof["solve_bytes"] / solve_s / HBM_BYTES_PER_S, 4) if solve_s > 0 else None,
               steps=a.steps, all_gpu_ms=[round(p["ms_total"], 2) for p in runs])

    if a.sk_cands > 0:
        # the candidates with the smallest C: the cheapest for libsvm, so the comparison finishes
        pick = sorted(range(len(cands)), key=lambda i: (cands[i]["C"], i))[:a.sk_cands]
        sub = [cands[i] for i in pick]
        grid = [{k: [v] for k, v in c.items()} for c in sub]
        t0 = time.perf_counter()
        sk = SkGridSearchCV(SVR(**w["est_params"]), grid, cv=KFold(cv), n_jobs=os.cpu_count(), refit=False).fit(X, y)
        sk_s = time.perf_counter() - t0
        ref = np.stack([sk.cv_results_["split%d_test_score" % k] for k in range(cv)], 1)
        got = res["test"][pick]
        out.update(sklearn_fits=len(sub) * cv, sklearn_s=round(sk_s, 2), sklearn_fits_per_s=round(len(sub) * cv / sk_s, 3),
                   sklearn_cores=os.cpu_count(), parity_max_abs_split_score_diff=float(np.abs(got - ref).max()))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
