"""Regenerate the LinearSVC goldens from scikit-learn (1.9): per (candidate, split) test and train scores and n_iter_, and
one refit's coef_ / intercept_.

    python tests/golden/make_linsvc_goldens.py            # linsvc_small.npz, linsvc_multi.npz
    python tests/golden/make_linsvc_goldens.py --c3       # also linsvc_c3.npz (1280 fits of 40000 x 256: minutes on 8 cores)

Variants of the small workloads: class_weight None / 'balanced' / a dict, and sample weights that include zeros.  The
splits are the search's: StratifiedKFold(5) (check_cv of an integer cv for a classifier).
"""
import os
import sys
from multiprocessing import Pool

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from spark_sklearn_b200 import workloads as W  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
VARIANTS = {"none": {}, "balanced": {"class_weight": "balanced"}, "dict": {"class_weight": {0: 2.0, 1: 0.5}}, "sw": {}}
# the dict variant weights class 0 up and class 1 down; a third class keeps weight 1


def sample_weight(n):
    """the 'sw' variant's weights: a deterministic mix of zeros and weights in [0.5, 2)"""
    rng = np.random.RandomState(1)
    w = rng.uniform(0.5, 2.0, n)
    w[rng.rand(n) < 0.1] = 0.0
    return w


def _fit(args):
    from sklearn.svm import LinearSVC
    X, y, tr, te, params, sw = args
    est = LinearSVC(**params).fit(X[tr], y[tr], sample_weight=None if sw is None else sw[tr])
    return est.score(X[te], y[te]), est.score(X[tr], y[tr]), est.n_iter_


def splits(w):
    from sklearn.model_selection import StratifiedKFold
    return list(StratifiedKFold(w["cv"]).split(w["X"], w["y"]))


def run(w, variant, pool):
    cands = W.candidates(w)
    sp = splits(w)
    sw = sample_weight(len(w["X"])) if variant == "sw" else None
    extra = VARIANTS[variant]
    jobs = [(w["X"], w["y"], tr, te, dict(w["est_params"], **extra, **c), sw) for c in cands for tr, te in sp]
    out = np.array(pool.map(_fit, jobs, chunksize=1)).reshape(len(cands), len(sp), 3)
    return out[..., 0], out[..., 1], out[..., 2].astype(np.int32)


def main():
    from sklearn.svm import LinearSVC
    keys = ["linsvc_small", "linsvc_multi"] + (["linsvc_c3"] if "--c3" in sys.argv else [])
    with Pool() as pool:
        for key in keys:
            w = W.make_workload(key)
            arrays = {}
            for variant in (VARIANTS if key != "linsvc_c3" else ["none"]):
                te, trs, it = run(w, variant, pool)
                arrays.update({"%s_test" % variant: te, "%s_train" % variant: trs, "%s_n_iter" % variant: it})
                print(key, variant, "n_iter range", it.min(), it.max(), flush=True)
            best = dict(W.candidates(w)[0] if key == "linsvc_c3" else W.candidates(w)[len(W.candidates(w)) // 2])
            est = LinearSVC(**dict(w["est_params"], **best)).fit(w["X"], w["y"])
            arrays.update(refit_C=np.float64(best["C"]), refit_coef=est.coef_, refit_intercept=np.atleast_1d(est.intercept_),
                          refit_n_iter=np.int32(est.n_iter_))
            np.savez_compressed(os.path.join(HERE, key + ".npz"), **arrays)


if __name__ == "__main__":
    main()
