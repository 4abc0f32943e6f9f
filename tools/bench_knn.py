"""Measure the k-NN search on one GPU: fits/s from CUDA events with X resident, the phase split (distances / selection /
votes), the distance phase's achieved FP64 rate against the H100 SXM data sheet's 34 TFLOP/s (FP64 without tensor cores:
the tile kernel runs on the FP64 pipes), the selection's bytes/s, and scikit-learn's GridSearchCV(n_jobs=cores) on a sample
of the candidates (with a parity check on that sample).  The card's name and power limit are read in the same run.

    python tools/bench_knn.py [--workload knn_c2] [--steps 3] [--sk-cands 4]
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

FP64_FLOPS = 34e12                 # H100 SXM data sheet, FP64 (non-tensor), a 700 W card


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="knn_c2")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--sk-cands", type=int, default=4, help="candidates scikit-learn fits for comparison (0: skip)")
    a = ap.parse_args()

    from sklearn.model_selection import GridSearchCV as SkGridSearchCV, StratifiedKFold
    from spark_sklearn_b200.estimators import Folds, adapter_for
    from spark_sklearn_b200 import workloads as W

    w = W.make_workload(a.workload)
    X, y, cv = w["X"], w["y"], w["cv"]
    cands = W.candidates(w)
    est = W.make_estimator(w)
    splits = list(StratifiedKFold(cv).split(X, y))
    plan = adapter_for(est).plan(est, cands, X, y, Folds(splits, len(X)), cv)      # X resident from here
    plan.set_scoring(None)
    n_fits = len(cands) * cv

    plan.evaluate([0])                                            # warm-up: library load, buffers
    runs = []
    for _ in range(a.steps):
        res = plan.evaluate(list(range(len(cands))))
        runs.append(dict(plan.profile()))
    prof = min(runs, key=lambda p: p["ms_total"])
    ms = prof["ms_total"]
    rate = prof["gram_flops"] / (prof["ms_gram"] * 1e-3) if prof["ms_gram"] > 0 else None
    out = dict(workload=a.workload, card=card(), n=int(X.shape[0]), d=int(X.shape[1]), candidates=len(cands), folds=cv,
               fits=n_fits, gpu_ms=round(ms, 2), fits_per_s=round(n_fits / (ms * 1e-3), 2),
               ms_distances=round(prof["ms_gram"], 2), ms_selection=round(prof["ms_solve"], 2),
               ms_votes=round(prof["ms_score"], 2), launches=int(prof["launches"]),
               distance_fp64_tflops=round(rate / 1e12, 2) if rate else None,
               distance_fraction_of_datasheet=round(rate / FP64_FLOPS, 3) if rate else None,
               selection_gb_per_s=round(prof["solve_bytes"] / (prof["ms_solve"] * 1e-3) / 1e9, 1) if prof["ms_solve"] > 0 else None,
               steps=a.steps, all_gpu_ms=[round(p["ms_total"], 2) for p in runs])

    if a.sk_cands > 0:
        pick = list(np.linspace(0, len(cands) - 1, a.sk_cands).round().astype(int))
        grid = [{k: [v] for k, v in cands[i].items()} for i in pick]
        t0 = time.perf_counter()
        sk = SkGridSearchCV(W.make_estimator(w), grid, cv=StratifiedKFold(cv), n_jobs=os.cpu_count(), refit=False,
                            return_train_score=True).fit(X, y)
        sk_s = time.perf_counter() - t0
        ref = np.stack([sk.cv_results_["split%d_test_score" % k] for k in range(cv)], 1)
        ref_tr = np.stack([sk.cv_results_["split%d_train_score" % k] for k in range(cv)], 1)
        got, got_tr = res["test"][pick], res["train"][pick]
        out.update(sklearn_fits=len(pick) * cv, sklearn_s=round(sk_s, 2), sklearn_fits_per_s=round(len(pick) * cv / sk_s, 3),
                   sklearn_cores=os.cpu_count(), parity_max_abs_split_score_diff=float(max(np.abs(got - ref).max(),
                                                                                            np.abs(got_tr - ref_tr).max())))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
