"""Regenerate the LinearSVR goldens from scikit-learn (1.9): per (candidate, split) test and train R^2 and n_iter_, and one
refit's coef_ / intercept_ / n_iter_.

    python tests/golden/make_linsvr_goldens.py            # linsvr_small.npz, linsvr_wide.npz

Variants: the workload's own estimator (none), dual=True (the squared loss on the dual CD, solver 12), sample weights that
include zeros (sw), fit_intercept=False (nofi) and intercept_scaling=2.5 (scaling).  The splits are the search's: KFold(5)
(check_cv of an integer cv for a regressor).
"""
import os
import sys
from multiprocessing import Pool

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
from spark_sklearn_b200 import workloads as W  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
VARIANTS = {"none": {}, "dual": {"dual": True}, "sw": {}, "nofi": {"fit_intercept": False}, "scaling": {"intercept_scaling": 2.5}}
KEYS = {"linsvr_small": list(VARIANTS), "linsvr_wide": ["none", "sw"]}


def sample_weight(n):
    """the 'sw' variant's weights: a deterministic mix of zeros and weights in [0.5, 2)"""
    rng = np.random.RandomState(1)
    w = rng.uniform(0.5, 2.0, n)
    w[rng.rand(n) < 0.1] = 0.0
    return w


def _fit(args):
    import warnings
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.svm import LinearSVR
    X, y, tr, te, params, sw = args
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        est = LinearSVR(**params).fit(X[tr], y[tr], sample_weight=None if sw is None else sw[tr])
    return est.score(X[te], y[te]), est.score(X[tr], y[tr]), est.n_iter_


def splits(w):
    from sklearn.model_selection import KFold
    return list(KFold(w["cv"]).split(w["X"], w["y"]))


def run(w, variant, pool):
    cands = W.candidates(w)
    sp = splits(w)
    sw = sample_weight(len(w["X"])) if variant == "sw" else None
    jobs = [(w["X"], w["y"], tr, te, dict(w["est_params"], **VARIANTS[variant], **c), sw) for c in cands for tr, te in sp]
    out = np.array(pool.map(_fit, jobs, chunksize=1)).reshape(len(cands), len(sp), 3)
    return out[..., 0], out[..., 1], out[..., 2].astype(np.int32)


def main():
    import warnings
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.svm import LinearSVR
    with Pool() as pool:
        for key, variants in KEYS.items():
            w = W.make_workload(key)
            arrays = {}
            for variant in variants:
                te, trs, it = run(w, variant, pool)
                arrays.update({"%s_test" % variant: te, "%s_train" % variant: trs, "%s_n_iter" % variant: it})
                print(key, variant, "n_iter range", it.min(), it.max(), flush=True)
            cands = W.candidates(w)
            best = dict(cands[len(cands) // 2])
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", ConvergenceWarning)
                est = LinearSVR(**dict(w["est_params"], **best)).fit(w["X"], w["y"])
            arrays.update(refit_index=np.int32(len(cands) // 2), refit_coef=est.coef_,
                          refit_intercept=np.atleast_1d(est.intercept_), refit_n_iter=np.int32(est.n_iter_))
            np.savez_compressed(os.path.join(HERE, key + ".npz"), **arrays)


if __name__ == "__main__":
    main()
