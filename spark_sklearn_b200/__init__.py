"""spark_sklearn_b200 -- H100-native drop-in for the cross-validated search classes of
databricks/spark-sklearn (reference python/spark_sklearn/__init__.py:1-9 exports):

    from spark_sklearn_b200 import GridSearchCV, RandomizedSearchCV
    GridSearchCV(sc, SVC(), {"C": [...], "gamma": [...]}, cv=5).fit(X, y).cv_results_

The (candidate x fold) fit-and-score tasks run as hand-written sm_90a CUDA kernels in
``libb200gs.so`` (C ABI: include/b200gs.h) -- there is no Spark, no joblib and no CPU fallback.
"""
from .grid_search import GridSearchCV
from .random_search import RandomizedSearchCV

__all__ = ["GridSearchCV", "RandomizedSearchCV"]
__version__ = "0.1.0"
