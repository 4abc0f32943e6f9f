"""``RandomizedSearchCV`` with the reference's constructor and ``fit`` (reference
python/spark_sklearn/random_search.py:186-226), evaluated on H100 GPUs instead of a Spark cluster."""
from sklearn.model_selection import ParameterSampler

from .base_search import B200BaseSearchCV


class RandomizedSearchCV(B200BaseSearchCV):
    """Randomized search on hyper parameters, on H100 GPUs.

    Follows ``spark_sklearn.RandomizedSearchCV`` (reference random_search.py:9-226): candidates are drawn
    by scikit-learn's own ``ParameterSampler(param_distributions, n_iter, random_state)`` so the
    candidate list is identical to the reference's; no ``return_train_score`` keyword (train scores
    are always returned, reference random_search.py:195-199).
    """

    def __init__(self, sc, estimator, param_distributions, n_iter=10, scoring=None, fit_params=None, n_jobs=1,
                 iid=True, refit=True, cv=None, verbose=0, pre_dispatch='2*n_jobs', random_state=None,
                 error_score='raise'):
        self.param_distributions = param_distributions
        self.n_iter = n_iter
        self.random_state = random_state
        super(RandomizedSearchCV, self).__init__(
            estimator=estimator, scoring=scoring, fit_params=fit_params, n_jobs=n_jobs, iid=iid, refit=refit,
            cv=cv, verbose=verbose, pre_dispatch=pre_dispatch, error_score=error_score)
        self.fit_params = fit_params if fit_params is not None else {}
        self.sc = sc
        self.cv_results_ = None

    def fit(self, X, y=None, groups=None):
        """Run fit on the estimator with randomly drawn parameters (reference random_search.py:204-226)."""
        sampled_params = ParameterSampler(self.param_distributions, self.n_iter, random_state=self.random_state)
        return self._fit(X, y, groups, sampled_params)
