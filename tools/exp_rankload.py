"""Development: run ONE rank's share of an N-GPU weak-scaling grid on a single GPU (the ranks are independent)."""
import sys, os, time, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from spark_sklearn_b200 import workloads as WL, dist as D
from spark_sklearn_b200.estimators import adapter_for, fold_ids_from_splits
from sklearn.base import is_classifier
from sklearn.model_selection import check_cv
n_gpus = int(sys.argv[1]); ranks = [int(r) for r in sys.argv[2:]] or [0]
w = bench.scaled_workload("c2", n_gpus)
est = WL.make_estimator(w); X, y = w["X"], w["y"]; cands = WL.candidates(w)
splits = list(check_cv(w["cv"], y, classifier=is_classifier(est)).split(X, y))
fold_id = fold_ids_from_splits(splits, len(y))
plan = adapter_for(est).plan(est, cands, X, y, fold_id, len(splits))
parts = D.assign_for_plan(plan, len(cands), n_gpus)
for r in ranks:
    for rep in range(3):
        out = plan.evaluate(parts[r], return_train=True); p = plan.profile()
    it = out["n_iter"] if "n_iter" in out else None
    print("N=%d rank %d: %d candidates, step %.1f ms (solve %.1f, score %.1f), iterations %s" % (
        n_gpus, r, len(parts[r]), p["ms_total"], p["ms_solve"], p["ms_score"], int(p.get("smo_iterations", 0))), flush=True)
