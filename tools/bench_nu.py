"""Measure the NuSVC and NuSVR searches on one GPU: fits/s from CUDA events with X resident, the phase split (Gram, kernel
matrices, SMO solve, scoring), and scikit-learn's GridSearchCV(n_jobs=16) on a subset of the candidates for comparison (with
a parity check on that subset).  The solve time includes the gradient initialisation from the non-zero starting alpha: the
library has no separate timer for it, so it is reported as not measured.  The card's name and power limit are printed with
the numbers.

    python tools/bench_nu.py [--workloads nusvc_c2,nusvr_mid] [--steps 2] [--sk-cands 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def run(key, steps, sk_cands):
    from sklearn.model_selection import GridSearchCV as SkGridSearchCV, KFold, ParameterGrid, StratifiedKFold
    from spark_sklearn_b200 import workloads as W
    from spark_sklearn_b200.estimators import Folds, adapter_for

    w = W.make_workload(key)
    X, y, cv = w["X"], w["y"], w["cv"]
    est = W.make_estimator(w)
    cands = list(ParameterGrid(w["param_grid"]))
    splitter = KFold(cv) if w["estimator"] == "NuSVR" else StratifiedKFold(cv)
    splits = list(splitter.split(X, y))
    plan = adapter_for(est).plan(est, cands, X, y, Folds(splits, len(X)), cv)      # X, y resident from here
    n_fits = len(cands) * cv
    plan.evaluate([0])                                                                # warm-up
    runs = []
    for _ in range(steps):
        res = plan.evaluate(list(range(len(cands))))
        runs.append(dict(plan.profile()))
    prof = min(runs, key=lambda p: p["ms_total"])
    ms = prof["ms_total"]
    out = dict(workload=key, n=int(X.shape[0]), d=int(X.shape[1]), candidates=len(cands), folds=cv, fits=n_fits,
               gpu_ms=round(ms, 2), fits_per_s=round(n_fits / (ms * 1e-3), 2),
               ms_gram=round(prof["ms_gram"], 2), ms_kernel_matrix=round(prof["ms_kernel_matrix"], 2),
               ms_gradient_init="not measured (inside ms_solve)",
               ms_solve=round(prof["ms_solve"], 2), ms_score=round(prof["ms_score"], 2),
               smo_iterations=int(prof["smo_iterations"]), steps=steps, all_gpu_ms=[round(p["ms_total"], 2) for p in runs])
    if sk_cands > 0:
        # the smallest-nu candidates: the fewest support vectors, the cheapest fits for libsvm
        pick = sorted(range(len(cands)), key=lambda i: (cands[i]["nu"], i))[:sk_cands]
        grid = [{k: [v] for k, v in cands[i].items()} for i in pick]
        t0 = time.perf_counter()
        sk = SkGridSearchCV(W.make_estimator(w), grid, cv=splitter, n_jobs=16, refit=False).fit(X, y)
        sk_s = time.perf_counter() - t0
        ref = np.stack([sk.cv_results_["split%d_test_score" % k] for k in range(cv)], 1)
        out.update(sklearn_fits=len(pick) * cv, sklearn_s=round(sk_s, 2), sklearn_fits_per_s=round(len(pick) * cv / sk_s, 3),
                   sklearn_n_jobs=16, parity_max_abs_split_score_diff=float(np.abs(res["test"][pick] - ref).max()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="nusvc_c2,nusvr_mid")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--sk-cands", type=int, default=2, help="candidates scikit-learn fits for comparison (0: skip)")
    a = ap.parse_args()
    card = _card()
    for key in a.workloads.split(","):
        out = run(key, a.steps, a.sk_cands)
        out["card"] = card
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
