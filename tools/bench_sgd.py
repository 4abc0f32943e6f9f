"""Measure the SGDClassifier search on one GPU: fits/s from CUDA events with X resident, the solve / score split, the epoch
range, SM cycles per sample inside one fit (median) and the share of a fit's cycles spent drawing and applying the shuffle,
cycles per sample at d = 32, 128 and 512 on the same rows, and scikit-learn's GridSearchCV(n_jobs=16) on a sample of the
candidates (with a parity check on that sample).  The card's name and power limit are read in the same run.

    python tools/bench_sgd.py [--workload sgd_c] [--steps 2] [--sk-cands 4]
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
    from spark_sklearn_b200.estimators import Folds, SGDPlan
    splits = list(StratifiedKFold(cv).split(X, y))
    plan = SGDPlan.plan(est, cands, X, y, Folds(splits, len(X)), cv)
    plan.set_scoring(None)
    return plan


def _cycles_per_sample(plan):
    st = plan.stats_
    return float(np.median(st[..., 2] / np.maximum(st[..., 0], 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="sgd_c")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--sk-cands", type=int, default=4, help="candidates scikit-learn fits for comparison (0: skip)")
    a = ap.parse_args()

    from sklearn.exceptions import ConvergenceWarning
    from sklearn.linear_model import SGDClassifier
    from sklearn.model_selection import GridSearchCV as SkGridSearchCV, StratifiedKFold
    from spark_sklearn_b200 import workloads as W

    w = W.make_workload(a.workload)
    X, y, cv = w["X"], w["y"], w["cv"]
    cands = W.candidates(w)
    est = SGDClassifier(**w["est_params"])
    plan = _plan(X, y, cands, cv, est)
    n_fits = len(cands) * cv
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        plan.evaluate([0])                                        # warm-up: library load, buffers
        runs = []
        for _ in range(a.steps):
            res = plan.evaluate(list(range(len(cands))))
            runs.append((dict(plan.profile()), plan.stats_.copy(), plan.n_iter_.copy()))
    prof, stats, n_iter = min(runs, key=lambda r: r[0]["ms_total"])
    ms = prof["ms_total"]
    samples, shuf, cyc = stats[..., 0], stats[..., 1], stats[..., 2]
    out = dict(workload=a.workload, card=card(), n=int(X.shape[0]), d=int(X.shape[1]), classes=int(len(np.unique(y))),
               candidates=len(cands), folds=cv, fits=n_fits, class_fits=int(samples.size), gpu_ms=round(ms, 2),
               fits_per_s=round(n_fits / (ms * 1e-3), 2), ms_solve=round(prof["ms_solve"], 2), ms_score=round(prof["ms_score"], 2),
               n_iter_range=[int(n_iter.min()), int(n_iter.max())], samples=int(samples.sum()),
               ns_per_sample_aggregate=round(prof["ms_solve"] * 1e6 / max(int(samples.sum()), 1), 4),
               sm_cycles_per_sample_in_fit_median=round(float(np.median(cyc / np.maximum(samples, 1))), 1),
               shuffle_share_of_fit_cycles=round(float(shuf.sum() / max(cyc.sum(), 1)), 4),
               launches=int(prof["launches"]), steps=a.steps, all_gpu_ms=[round(p["ms_total"], 2) for p, _, _ in runs])

    # cycles per sample against d: the default candidate on the first 4000 rows, features tiled to d
    rng = np.random.RandomState(0)
    per_d = {}
    for d in (32, 128, 512):
        Xd = np.ascontiguousarray(np.tile(X[:4000], (1, (d + X.shape[1] - 1) // X.shape[1]))[:, :d]
                                  + 0.01 * rng.randn(4000, d).astype(np.float32))
        p = _plan(Xd, y[:4000], [{"alpha": 1e-4}], cv, SGDClassifier(random_state=0, max_iter=20))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            p.evaluate([0])
        per_d[d] = round(_cycles_per_sample(p), 1)
    out["sm_cycles_per_sample_by_d"] = per_d

    if a.sk_cands > 0:
        pick = list(np.linspace(0, len(cands) - 1, a.sk_cands).round().astype(int))
        grid = [{k: [v] for k, v in cands[i].items()} for i in pick]
        t0 = time.perf_counter()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", ConvergenceWarning)
            sk = SkGridSearchCV(est, grid, cv=StratifiedKFold(cv), n_jobs=16, refit=False).fit(X, y)
        sk_s = time.perf_counter() - t0
        ref = np.stack([sk.cv_results_["split%d_test_score" % k] for k in range(cv)], 1)
        got = res["test"][pick]
        out.update(sklearn_fits=len(pick) * cv, sklearn_s=round(sk_s, 2), sklearn_fits_per_s=round(len(pick) * cv / sk_s, 3),
                   sklearn_n_jobs=16, sklearn_cores=os.cpu_count(), parity_split_scores_equal=bool(np.array_equal(got, ref)),
                   parity_max_abs_split_score_diff=float(np.abs(got - ref).max()))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
