"""``GridSearchCV`` with the reference's constructor and ``fit`` (reference
python/spark_sklearn/grid_search.py:212-246), evaluated on H100 GPUs instead of a Spark cluster."""
from collections.abc import Mapping, Sequence

import numpy as np
from sklearn.model_selection import ParameterGrid

from .base_search import B200BaseSearchCV


def _check_param_grid(param_grid):
    """Restates sklearn<0.20 ``_check_param_grid`` that the reference calls (grid_search.py:226)."""
    if hasattr(param_grid, 'items'):
        param_grid = [param_grid]
    for p in param_grid:
        if not isinstance(p, Mapping):
            raise ValueError("Parameter grid is not a dict or a list of dicts ({!r})".format(p))
        for name, v in p.items():
            if isinstance(v, np.ndarray) and v.ndim > 1:
                raise ValueError("Parameter array should be one-dimensional.")
            if isinstance(v, str) or not isinstance(v, (np.ndarray, Sequence)):
                raise ValueError("Parameter values for parameter ({0}) need to be a sequence"
                                 "(but not a string) or np.ndarray.".format(name))
            if len(v) == 0:
                raise ValueError("Parameter values for parameter ({0}) need to be a non-empty sequence.".format(name))


class GridSearchCV(B200BaseSearchCV):
    """Exhaustive search over specified parameter values for an estimator, on H100 GPUs.

    Signature, defaults (``cv=3``, ``iid=True``, ``return_train_score=True``, ``error_score='raise'``)
    and fitted attributes follow ``spark_sklearn.GridSearchCV`` (reference grid_search.py:10-246).
    ``sc`` is accepted for drop-in compatibility and never touched (no Spark here); ``n_jobs`` and
    ``pre_dispatch`` are ignored exactly as the reference documents (grid_search.py:46-50).
    """

    def __init__(self, sc, estimator, param_grid, scoring=None, fit_params=None, n_jobs=1, iid=True, refit=True,
                 cv=3, verbose=0, pre_dispatch='2*n_jobs', error_score='raise', return_train_score=True):
        super(GridSearchCV, self).__init__(
            estimator=estimator, scoring=scoring, n_jobs=n_jobs, iid=iid, refit=refit, cv=cv, verbose=verbose,
            pre_dispatch=pre_dispatch, error_score=error_score, return_train_score=return_train_score)
        self.fit_params = fit_params if fit_params is not None else {}
        self.sc = sc
        self.param_grid = param_grid
        self.cv_results_ = None
        _check_param_grid(param_grid)

    def fit(self, X, y=None, groups=None):
        """Run fit with all sets of parameters (reference grid_search.py:228-246)."""
        return self._fit(X, y, groups, ParameterGrid(self.param_grid))
