"""Measure the LogisticRegression(solver='saga') search on one GPU: fits/s from CUDA events with X resident on the usual grid
of 10 C x 5 l1_ratio values x cv=5 on 20000 x 128 rows (binary and 4 classes), the solve / score split, the epoch range, SM
cycles per sample step inside the fits (median), cycles per sample step at d = 32, 128 and 512 on the same rows, and
scikit-learn's GridSearchCV(n_jobs=cores) on a few sampled candidates (with the largest split-score difference on that
sample).  The card's name and power limit are read in the same run.

    python tools/bench_sag.py [--workloads sag_c2,sag_c4] [--steps 2] [--sk-cands 3]
"""
import argparse
import json
import os
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_linsvr import card  # noqa: E402


def _plan(X, y, cands, cv, est):
    from sklearn.model_selection import StratifiedKFold
    from spark_sklearn_b200.estimators import Folds, LogRegPlan
    splits = list(StratifiedKFold(cv).split(X, y))
    plan = LogRegPlan.plan(est, cands, X, y, Folds(splits, len(X)), cv)
    plan.set_scoring(None)
    return plan


def _cycles_per_step(plan):
    st = plan.stats_
    return float(np.median(st[..., 1] / np.maximum(st[..., 0], 1)))


def bench(key, steps, sk_cands):
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.linear_model import LogisticRegression
    from sklearn.model_selection import GridSearchCV as SkGridSearchCV, StratifiedKFold
    from spark_sklearn_b200 import workloads as W

    w = W.make_workload(key)
    X, y, cv = w["X"], w["y"], w["cv"]
    cands = W.candidates(w)
    est = LogisticRegression(**w["est_params"])
    plan = _plan(X, y, cands, cv, est)
    n_fits = len(cands) * cv
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        plan.evaluate([0])                                        # warm-up: library load, buffers
        runs = []
        for _ in range(steps):
            res = plan.evaluate(list(range(len(cands))))
            runs.append((dict(plan.profile()), plan.stats_.copy(), plan.n_iter_.copy()))
    prof, stats, n_iter = min(runs, key=lambda r: r[0]["ms_total"])
    ms = prof["ms_total"]
    samples, cyc = stats[..., 0], stats[..., 1]
    out = dict(workload=key, n=int(X.shape[0]), d=int(X.shape[1]), classes=int(len(np.unique(y))), candidates=len(cands),
               folds=cv, fits=n_fits, gpu_ms=round(ms, 2), fits_per_s=round(n_fits / (ms * 1e-3), 2),
               ms_solve=round(prof["ms_solve"], 2), ms_score=round(prof["ms_score"], 2),
               n_iter_range=[int(n_iter.min()), int(n_iter.max())], sample_steps=int(samples.sum()),
               sm_cycles_per_step_in_fit_median=round(float(np.median(cyc / np.maximum(samples, 1))), 1),
               launches=int(prof["launches"]), steps=steps, all_gpu_ms=[round(p["ms_total"], 2) for p, _, _ in runs])

    # cycles per sample step against d: one saga candidate on the first 4000 rows, features tiled to d
    rng = np.random.RandomState(0)
    per_d = {}
    k = len(np.unique(y))
    for d in (32, 128, 512):
        if d * (k if k > 2 else 1) > 512:
            continue
        Xd = np.ascontiguousarray(np.tile(X[:4000], (1, (d + X.shape[1] - 1) // X.shape[1]))[:, :d] + 0.01 * rng.randn(4000, d))
        p = _plan(Xd, y[:4000], [{"C": 1.0, "l1_ratio": 0.5}], cv, LogisticRegression(solver="saga", random_state=0, max_iter=5))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            p.evaluate([0])
        per_d[d] = round(_cycles_per_step(p), 1)
    out["sm_cycles_per_step_by_d"] = per_d

    if sk_cands > 0:
        pick = list(np.linspace(0, len(cands) - 1, sk_cands).round().astype(int))
        grid = [{kk: [v] for kk, v in cands[i].items()} for i in pick]
        cores = os.cpu_count()
        t0 = time.perf_counter()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", ConvergenceWarning)
            sk = SkGridSearchCV(est, grid, cv=StratifiedKFold(cv), n_jobs=cores, refit=False).fit(X, y)
        sk_s = time.perf_counter() - t0
        ref = np.stack([sk.cv_results_["split%d_test_score" % kk] for kk in range(cv)], 1)
        got = res["test"][pick]
        out.update(sklearn_fits=len(pick) * cv, sklearn_s=round(sk_s, 2), sklearn_fits_per_s=round(len(pick) * cv / sk_s, 3),
                   sklearn_n_jobs=cores, parity_max_abs_split_score_diff=float(np.abs(got - ref).max()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="sag_c2,sag_c4")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--sk-cands", type=int, default=3, help="candidates scikit-learn fits for comparison (0: skip)")
    a = ap.parse_args()
    c = card()
    for key in a.workloads.split(","):
        out = bench(key, a.steps, a.sk_cands)
        out["card"] = c
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
