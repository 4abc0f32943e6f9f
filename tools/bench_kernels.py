"""Measure SVC searches over the poly and sigmoid kernels on one GPU, next to rbf and linear candidates on the same data:
per kernel, fits/s from CUDA events with X resident, the phase split, the time per kernel matrix (where the poly / sigmoid
arithmetic replaces rbf's exp), SMO iterations, solve time per iteration and the solve phase's HBM traffic as a fraction of
the H100's 3.35 TB/s.  With --timeline the library prints when each solver tier starts and ends (B200GS_SMO_TIMELINE).

    python tools/bench_kernels.py [--workload svc_kernels_c2] [--steps 2] [--timeline]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM5 80 GB peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="svc_kernels_c2")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--timeline", action="store_true", help="print the solver tiers' start / end times (stderr)")
    a = ap.parse_args()

    from sklearn.model_selection import check_cv
    from sklearn.svm import SVC
    from spark_sklearn_b200.estimators import Folds, SVCPlan
    from spark_sklearn_b200 import workloads as W

    w = W.make_workload(a.workload)
    X, y = w["X"], w["y"]
    cands = W.candidates(w)
    splits = list(check_cv(w["cv"], y, classifier=True).split(X, y))
    ns = len(splits)
    plan = SVCPlan.plan(SVC(**w["est_params"]), cands, X, y, Folds(splits, len(X)), ns)   # X, y resident from here
    plan.evaluate([0])                                            # warm-up: library load, kernel attributes, buffers
    if a.timeline:
        os.environ["B200GS_SMO_TIMELINE"] = "1"

    out = dict(workload=a.workload, n=int(X.shape[0]), d=int(X.shape[1]), folds=ns, steps=a.steps, kernels={})
    for kern in ("poly", "sigmoid", "rbf", "linear"):
        my = [i for i, c in enumerate(cands) if c["kernel"] == kern]
        if not my:
            continue
        # kernel matrices of the search: one per (kernel, per-split gamma, degree, coef0) -- 'scale' differs per split
        mats = set()
        for i in my:
            p = dict(SVC(**w["est_params"]).get_params(), **cands[i])
            for k in range(ns):
                mats.add((kern, plan._gamma(p["gamma"], k) if kern != "linear" else 0.0,
                          p["degree"] if kern == "poly" else 0, p["coef0"] if kern in ("poly", "sigmoid") else 0.0))
        runs = []
        for _ in range(a.steps):
            plan.evaluate(my)
            runs.append(dict(plan.profile()))
        prof = min(runs, key=lambda p: p["ms_total"])
        ms, solve_ms, it = prof["ms_total"], prof["ms_solve"], int(prof["smo_iterations"])
        fits = len(my) * ns
        out["kernels"][kern] = dict(
            candidates=len(my), fits=fits, kernel_matrices=len(mats), gpu_ms=round(ms, 2), fits_per_s=round(fits / (ms * 1e-3), 1),
            ms_gram=round(prof["ms_gram"], 2), ms_kernel_matrix=round(prof["ms_kernel_matrix"], 2),
            ms_per_kernel_matrix=round(prof["ms_kernel_matrix"] / len(mats), 3), ms_solve=round(solve_ms, 2),
            ms_score=round(prof["ms_score"], 2), smo_iterations=it,
            solve_ns_per_iteration=round(solve_ms * 1e6 / it, 2) if it else None,
            smo_hbm_fraction=round(prof["solve_bytes"] / (solve_ms * 1e-3) / HBM_BYTES_PER_S, 4) if solve_ms > 0 else None,
            all_gpu_ms=[round(p["ms_total"], 2) for p in runs])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
