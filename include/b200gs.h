/*
 * b200gs.h -- C ABI of libb200gs.so, the H100 (sm_90a) cross-validated grid-search engine.
 *
 * Drop-in boundary.  The reference (databricks/spark-sklearn) is pure Python and has no FFI of
 * its own; the seam this library replaces is the per-task closure that the reference maps over
 * a Spark RDD and collects:
 *
 *     python/spark_sklearn/base_search.py:74-88   fun(tup) -> (index, _fit_and_score(...))
 *     python/spark_sklearn/base_search.py:62-65   sc.parallelize(tasks), sc.broadcast(X|y|groups)
 *     python/spark_sklearn/base_search.py:89-95   .map(fun).collect(), re-ordered by task index
 *
 * Instead of one task per (candidate, fold), ONE call evaluates the whole task list: the dataset
 * is copied to the GPU once (gs_set_data == the broadcast), gs_svc / gs_ridge / gs_logreg map every
 * (candidate, fold) task with CUDA kernels (== map(fun)), and the score arrays come back in the
 * reference's task order, candidate-major / fold-minor (== collect + re-order, base_search.py:56-61,
 * 100-108).  The ctypes binding a maintainer adds on the reference side is in INTEGRATION.md.
 *
 * Conventions: C linkage; plain pointers + sizes; every function returns 0 on success or a
 * negative gs_status, never throws; gs_last_error() returns a human-readable message for the last
 * failure on that handle.  All pointers are HOST pointers owned by the caller and need only live
 * for the duration of the call.  A handle is bound to one CUDA device and is not thread-safe.
 * There is no CPU fallback: without a usable sm_90 device gs_create fails.
 */
#ifndef B200GS_H
#define B200GS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gs_handle gs_handle;

enum gs_status {
    GS_OK = 0,
    GS_ERR_CUDA = -1,        /* CUDA runtime/driver error (message has the call site)       */
    GS_ERR_ARG = -2,         /* invalid argument                                             */
    GS_ERR_NO_DATA = -3,     /* search called before gs_set_data                             */
    GS_ERR_UNSUPPORTED = -4, /* configuration the CUDA path does not implement (no fallback) */
    GS_ERR_NUMERIC = -5      /* non-finite result (maps to the reference's error_score)      */
};

enum gs_kernel { GS_KERNEL_LINEAR = 0, GS_KERNEL_RBF = 1, GS_KERNEL_POLY = 2, GS_KERNEL_SIGMOID = 3 };
enum gs_dtype { GS_F32 = 0, GS_F64 = 1 };

enum gs_flags {
    GS_RETURN_TRAIN = 1,     /* also fill train_scores (reference return_train_score=True)   */
    GS_GRAM_TENSOR = 2,      /* build the Gram on wgmma tensor cores (3xTF32 split, fp32-faithful)
                                instead of the float64 Gram that reproduces libsvm bit for bit */
    GS_NO_SHRINKING = 4      /* SVC(shrinking=False)                                         */
};

/* ---- lifecycle ------------------------------------------------------------------------- */
/* Replaces: SparkContext creation (reference util.py:51-58) -- one handle per process/GPU.    */
int gs_create(int device, gs_handle **out);
void gs_destroy(gs_handle *h);
const char *gs_last_error(const gs_handle *h);      /* h may be NULL: last gs_create failure  */
int gs_version(void);
/* General CV splits.  Replaces: the per-task (train, test) index arrays of the reference (base_search.py:81-82,
 * islice(cv.split(X, y, groups))) for splitters whose test sets overlap or whose training set is not the complement of the
 * test set (ShuffleSplit, RepeatedKFold, PredefinedSplit with -1).  Call after gs_set_data (whose fold ids may all be -1).
 * test_mask / train_mask: [n][2] uint64, bit k of word k/64 = row belongs to the test / training set of split k; a row may be
 * in neither.  gs_svc, gs_logreg and gs_ridge honour the masks (gs_ridge then contracts one Gram per training / test row
 * list of a split instead of the fold Grams T - G_fold of a partition). */
int gs_set_splits(gs_handle *h, const uint64_t *test_mask, const uint64_t *train_mask, int32_t n_splits);

/* Class weights of the following gs_svc / gs_svc_refit calls: the C of a training row is C x w[class of the row].
 * Replaces: SVC(class_weight=...) forwarded through clone(estimator).set_params / fit_params into every task (reference
 * base_search.py:69,83-87); scikit-learn computes `class_weight_` from the TRAINING labels of each fit ('balanced' differs
 * per fold), hence one weight set per split: w is [n_sets][n_classes], n_sets = n_splits (search), 1 (refit, or the same
 * weights for every split); w == NULL resets to all ones. */
int gs_set_class_weight(gs_handle *h, const double *w, int32_t n_sets);

/* Polynomial / sigmoid kernel parameters of the next gs_svc (n = n_cand), gs_svc_refit or gs_debug_kernel_matrix (n = 1):
 * SVC(degree=..., coef0=...), one value per candidate.  libsvm's kernels (svm.cpp Kernel): poly = powi(gamma x.y + coef0,
 * degree), sigmoid = tanh(gamma x.y + coef0); gamma is resolved per split as for rbf and may be any finite value >= 0.
 * Linear and rbf candidates ignore both values.  degree == NULL resets every candidate to scikit-learn's defaults (degree 3,
 * coef0 0), as does gs_set_data.  A call whose count differs from its n_cand fails with GS_ERR_ARG, as does a degree < 0 or a
 * coef0 that is not finite.  gs_svr keeps rejecting the poly and sigmoid kernels (GS_ERR_UNSUPPORTED). */
int gs_set_kernel_params(gs_handle *h, const int32_t *degree, const double *coef0, int32_t n);

/* Sample weights of the following gs_ridge / gs_enet / gs_logreg calls and their refits.  Replaces: fit_params={'sample_weight': w}
 * handed to every task's estimator.fit (reference base_search.py:69,83-87; scikit-learn's _fit_and_score slices it by the
 * training rows and weights the FIT only -- the scores stay unweighted).  w: [n] in the caller's row order, >= 0; NULL resets.
 * gs_ridge / gs_enet contract a second, sqrt(w)-scaled copy of the row blocks for the weighted training statistics;
 * gs_logreg multiplies the pointwise loss and gradient.  gs_svc rejects them (its kernels take a C per class, not per row).
 * gs_set_data resets the weights. */
int gs_set_sample_weight(gs_handle *h, const double *w);

/* Scorer of the following gs_svc / gs_logreg / gs_ridge calls.  Replaces: check_scoring(estimator, scoring) and the scorer
 * call inside _fit_and_score (reference base_search.py:43,83-87; grid_search.py:212-214 `scoring=`).  The score is
 * computed on the device from the decision values / Gram statistics already in HBM.  pos_class: class id (index into the
 * sorted labels) that precision / recall / f1 treat as positive (scikit-learn's pos_label=1). */
enum {
    GS_SCORE_DEFAULT = 0,            /* accuracy (classifiers) / r2 (Ridge): estimator.score                */
    GS_SCORE_BALANCED_ACCURACY = 1,
    GS_SCORE_F1 = 2, GS_SCORE_PRECISION = 3, GS_SCORE_RECALL = 4,          /* binary, class pos_class      */
    GS_SCORE_ROC_AUC = 5,            /* binary: rank statistic of the decision values                        */
    GS_SCORE_F1_MACRO = 6, GS_SCORE_F1_MICRO = 7, GS_SCORE_F1_WEIGHTED = 8,
    GS_SCORE_NEG_MSE = 16, GS_SCORE_NEG_RMSE = 17                          /* Ridge                         */
};
int gs_set_scoring(gs_handle *h, int32_t kind, int32_t pos_class);   /* gs_set_data resets scoring, class and sample weights to their defaults */

/* Number of sm_90 GPUs this process can drive (0: none).  Replaces: the executor count Spark reports to the driver
 * (reference base_search.py:62 sc.parallelize(..., len(tasks)) leaves placement to Spark); the in-process scheduler of
 * spark_sklearn_b200/base_search.py opens one handle per device and deals the candidates over them. */
int gs_device_count(void);

/* ---- data: the "broadcast" (reference base_search.py:63-65) ------------------------------ */
/*
 * X        [n][d] row-major, x_dtype = GS_F32 (float32: the dtype of the BASELINE configs; exact in the
 *          float64 Gram) or GS_F64 (float64: what scikit-learn upcasts every other input to).
 * y_class  [n] int32 class ids 0..n_classes-1 in sorted-label order, or NULL for regression.
 * y_target [n] float32 regression targets, or NULL for classification.
 * fold_id  [n] int8: index of the CV split whose TEST set holds the row (reference
 *          base_search.py:81-82 recomputes cv.split per task; here the splits arrive once);
 *          -1 = row is in no test set (always train).  n_splits = number of splits.
 */
int gs_set_data(gs_handle *h, const void *X, int32_t x_dtype, int64_t n, int64_t d,
                const int32_t *y_class, const float *y_target,
                const int8_t *fold_id, int32_t n_splits);

/* ---- searches: map(fun).collect() for one estimator family ------------------------------- */
/*
 * SVC (C-SVC, one-vs-one; replaces _fit_and_score -> SVC.fit/score = sklearn libsvm,
 * svm.cpp:2365 svm_train, :666 Solver::Solve, :2821 svm_predict_values).
 *   kernel[n_cand] (GS_KERNEL_*; poly / sigmoid read degree and coef0 from gs_set_kernel_params), C[n_cand];
 *   gamma[n_cand*n_splits] (already resolved per fold: 'scale' depends
 *   on the training fold, sklearn svm/_base.py:278-286).  tol = SVC.tol, max_iter = SVC.max_iter
 *   (-1: none).  Outputs, all [n_cand*n_splits], candidate-major: test_scores / train_scores
 *   (accuracy, float64; train may be NULL without GS_RETURN_TRAIN), n_iter (sum over OvO pairs),
 *   n_sv (support vectors), fit_ms / score_ms (device time attributed to the task; may be NULL).
 */
int gs_svc(gs_handle *h, int32_t n_cand, const int32_t *kernel, const double *C, const double *gamma,
           double tol, int32_t max_iter, uint32_t flags,
           double *test_scores, double *train_scores, int32_t *n_iter, int32_t *n_sv,
           float *fit_ms, float *score_ms);

/*
 * Refit (reference base_search.py:165-174) of one SVC on ALL rows.  Outputs, indexed by ORIGINAL
 * dataset row: pair_coef [n_pairs][n] = alpha_k*y_k of each one-vs-one sub-model (0 for rows outside
 * the pair / non-SVs; pair order (0,1),(0,2),...,(1,2),... as svm.cpp:2484), rho [n_pairs],
 * n_iter [n_pairs].  The Python side assembles a fitted sklearn.svm.SVC from them.
 */
int gs_svc_refit(gs_handle *h, int32_t kernel, double C, double gamma, double tol, int32_t max_iter,
                 uint32_t flags, double *pair_coef, double *rho, int32_t *n_iter);

/*
 * Ridge (replaces Ridge.fit/score: sklearn linear_model/_ridge.py:919, _solve_cholesky :215-227,
 * r2 base.py:716).  alpha[n_cand].  Scores are R^2.  coef_out (may be NULL): refit on all rows of
 * candidate refit_cand -> [d] weights + intercept at [d].
 */
int gs_ridge(gs_handle *h, int32_t n_cand, const double *alpha, int32_t fit_intercept, uint32_t flags,
             double *test_scores, double *train_scores, float *fit_ms, float *score_ms);
int gs_ridge_refit(gs_handle *h, double alpha, int32_t fit_intercept, double *coef_out);

/*
 * ElasticNet / Lasso (replaces ElasticNet.fit/score and Lasso.fit/score -- the estimator of the reference's own search tests,
 * python/spark_sklearn/tests/test_search_2.py:69-119: sklearn linear_model/_coordinate_descent.py:1170-1280 fit, :781-782
 * penalty scaling, _cd_fast.pyx:243-506 enet_coordinate_descent, :162-240 duality gap).  alpha[n_cand], l1_ratio[n_cand]
 * (1.0 = Lasso); tol / max_iter as scikit-learn's; selection='cyclic', positive=False.  Same fold Grams, scorers and split
 * handling as gs_ridge; the solve is cyclic coordinate descent with scikit-learn's stopping rule and gap-safe screening, run
 * in the Gram domain (one warp per (candidate, split)).  n_iter (may be NULL): [n_cand][n_splits] sweeps.  No more than 1024
 * features.  A fit that stops at max_iter is returned as it is (scikit-learn: ConvergenceWarning).
 * gs_enet_refit: all rows -> [d] weights + intercept at [d]; n_iter / dual_gap (may be NULL): sweeps and the duality gap
 * (scikit-learn's dual_gap_ = gap / n_samples).
 */
int gs_enet(gs_handle *h, int32_t n_cand, const double *alpha, const double *l1_ratio, int32_t fit_intercept, double tol,
            int32_t max_iter, uint32_t flags, double *test_scores, double *train_scores, int32_t *n_iter, float *fit_ms,
            float *score_ms);
int gs_enet_refit(gs_handle *h, double alpha, double l1_ratio, int32_t fit_intercept, double tol, int32_t max_iter,
                  double *coef_out, int32_t *n_iter, double *dual_gap);

/*
 * LogisticRegression (L2, lbfgs; replaces sklearn linear_model/_logistic.py:219 _logistic_regression_path, objective
 * _linear_loss.py:47-64).  C[n_cand].  Scores are accuracy unless gs_set_scoring says otherwise.  Two classes: the binomial
 * loss on one weight row.  Three to 64 classes: scikit-learn's multinomial loss (_logistic.py:527-545, _loss/_loss.pyx
 * closs_grad_half_multinomial), one weight row per class, predictions by the first arg-max.
 * gs_logreg_refit: coef_out is [rows][d + 1] (weights, then the intercept), rows = 1 (binary) or n_classes.
 */
int gs_logreg(gs_handle *h, int32_t n_cand, const double *C, double tol, int32_t max_iter,
              int32_t fit_intercept, uint32_t flags,
              double *test_scores, double *train_scores, int32_t *n_iter, float *fit_ms, float *score_ms);
int gs_logreg_refit(gs_handle *h, double C, double tol, int32_t max_iter, int32_t fit_intercept,
                    double *coef_out, int32_t *n_iter);

/*
 * epsilon-SVR (replaces SVR.fit/score: sklearn libsvm svm.cpp solve_epsilon_svr on 2l variables, r2 base.py RegressorMixin).
 * gs_set_targets_f64: the float64 targets y[n] in the caller's row order (scikit-learn fits SVR on float64 y; gs_set_data keeps
 * float32 targets only).  Valid after a regression gs_set_data, which resets them.
 * gs_svr: kernel[n_cand], C[n_cand], epsilon[n_cand]; gamma[n_cand*n_splits] resolved per split as for gs_svc.  tol / max_iter
 * as SVR's; flags GS_RETURN_TRAIN, GS_NO_SHRINKING, GS_GRAM_TENSOR.  Splits: gs_set_data's fold ids or gs_set_splits masks; a
 * fit's variables are its training rows in ascending original index (scikit-learn's X[train] for partition splitters).
 * Scores: r2, or GS_SCORE_NEG_MSE / GS_SCORE_NEG_RMSE (gs_set_scoring).  Outputs as gs_svc's, n_iter per fit.
 * At most 8192 training rows per fit, gs_svr_refit's all-row fit included (GS_ERR_UNSUPPORTED beyond); sample and class
 * weights are rejected.  r2 of a split with fewer than two rows is NaN (scikit-learn: UndefinedMetricWarning).
 * gs_svr_refit: all rows; coef[n] = dual coefficient (alpha+ - alpha-) by ORIGINAL row, *rho (prediction = sum coef k - rho),
 * *n_iter.
 */
int gs_set_targets_f64(gs_handle *h, const double *y);
int gs_svr(gs_handle *h, int32_t n_cand, const int32_t *kernel, const double *C, const double *epsilon, const double *gamma,
           double tol, int32_t max_iter, uint32_t flags, double *test_scores, double *train_scores, int32_t *n_iter,
           int32_t *n_sv, float *fit_ms, float *score_ms);
int gs_svr_refit(gs_handle *h, int32_t kernel, double C, double epsilon, double gamma, double tol, int32_t max_iter,
                 uint32_t flags, double *coef, double *rho, int32_t *n_iter);

/*
 * LinearSVC (penalty='l2', loss='squared_hinge', primal: replaces LinearSVC.fit/score = sklearn liblinear linear.cpp train /
 * train_one with L2R_L2LOSS_SVC, l2r_l2_svc_fun and tron.cpp TRON, the trust-region Newton method with conjugate gradients).
 * C[n_cand]; tol / max_iter as LinearSVC's.  fit_intercept != 0: every row gets the regularised feature intercept_scaling
 * (> 0, scikit-learn's bias).  Two classes: one fit per (candidate, split), class 0 = -1.  Three or more: one-vs-rest, one fit
 * per class, whose negative rows get the unweighted C (linear.cpp train).  Class weights: gs_set_class_weight (one set per
 * split or one for all); sample weights: gs_set_sample_weight, float64, a row with weight 0 leaves the fit.  Splits: fold ids
 * or gs_set_splits masks.  Each fit follows liblinear's iterate in float64 (X is widened exactly; the products run on the
 * FP64 tensor cores).  Scores: accuracy or gs_set_scoring's scorer from the float64 decision values (binary: > 0 ->
 * class 1; one-vs-rest: first arg-max).  n_iter: [n_cand][n_splits], TRON iterations, the maximum over the one-vs-rest
 * fits (LinearSVC.n_iter_).  Every class needs a row of positive weight in every training set (GS_ERR_UNSUPPORTED).
 * gs_linsvc_refit: all rows; coef_out [rows][d + 1] = liblinear's raw weights (features, then the weight of the bias
 * feature: intercept_ = intercept_scaling x that; 0 without an intercept), rows = 1 (binary) or n_classes; n_iter [rows].
 */
int gs_linsvc(gs_handle *h, int32_t n_cand, const double *C, double tol, int32_t max_iter, int32_t fit_intercept,
              double intercept_scaling, uint32_t flags, double *test_scores, double *train_scores, int32_t *n_iter,
              float *fit_ms, float *score_ms);
int gs_linsvc_refit(gs_handle *h, double C, double tol, int32_t max_iter, int32_t fit_intercept, double intercept_scaling,
                    double *coef_out, int32_t *n_iter);

/*
 * k-nearest neighbours (replaces KNeighborsClassifier / KNeighborsRegressor .fit/score: a fit stores its training rows,
 * the scorer's predict runs scikit-learn's brute-force ArgKmin, sklearn/metrics/_pairwise_distances_reduction, and the
 * vote of neighbors/_classification.py, _regression.py, _base.py _get_weights).  n_neighbors[n_cand]
 * (1..GS_KNN_MAX_NEIGHBORS), weights[n_cand] (GS_KNN_UNIFORM, GS_KNN_DISTANCE), metric[n_cand] (GS_KNN_EUCLIDEAN,
 * GS_KNN_MANHATTAN).  For each metric present the call computes the distances once, in row slabs (no n x n matrix is
 * kept): Euclidean orders by scikit-learn's surrogate xsq[c] - 2 x_r.x_c (float64) and its distance is
 * sqrt(max(surrogate + xsq[r], 0)) (float32 X: both rounded to float32, as EuclideanDistance32 does), a row's distance
 * to itself being exactly 0; Manhattan is the float64 sum of the differences rounded in X's dtype, in feature order,
 * then rounded to X's dtype (ManhattanDistance32/64.dist).  One selection per metric then keeps, for every evaluated
 * row and split, the K_max = max n_neighbors nearest training rows sorted by (key, original row index): an exact tie
 * goes to the lower index (scikit-learn's ArgKmin heap usually, but not always, keeps the same rows).  Every candidate
 * votes from those lists: uniform (proba = count / k) or 1 / distance (the indicator of zero distance when a neighbour
 * is at distance 0; sums in numpy's pairwise order), prediction = first arg-max; regressor: mean of the neighbours' y
 * (float32 when flags has GS_TARGET_F32: numpy keeps float32 y) or sum w y / sum w in float64.  Classifier: labels from
 * gs_set_data, up to 64 classes, every gs_set_scoring classifier scorer (roc_auc: binary, on predict_proba[:, 1]).
 * Regressor: float64 targets from gs_set_targets_f64, r2 / GS_SCORE_NEG_MSE / GS_SCORE_NEG_RMSE.  Splits: fold ids or
 * gs_set_splits masks; flags GS_RETURN_TRAIN also scores every split's training rows.  A task whose n_neighbors exceeds
 * its split's training rows scores NaN (scikit-learn's kneighbors raises ValueError).  Sample and class weights are
 * rejected.  fit_ms / score_ms (may be NULL): the call's distance + selection time and its vote time, each divided
 * evenly over the tasks.  gs_profile: ms_gram the distances, ms_solve the selection, ms_score votes and scorers.
 */
enum { GS_KNN_UNIFORM = 0, GS_KNN_DISTANCE = 1 };
enum { GS_KNN_EUCLIDEAN = 0, GS_KNN_MANHATTAN = 1 };
enum { GS_KNN_MAX_NEIGHBORS = 256 };
enum { GS_TARGET_F32 = 8 };          /* gs_knn flag: the regression targets are float32 */
int gs_knn(gs_handle *h, int32_t n_cand, const int32_t *n_neighbors, const int32_t *weights, const int32_t *metric,
           uint32_t flags, double *test_scores, double *train_scores, float *fit_ms, float *score_ms);

/* ---- test hooks (used by tests/ to localise a parity failure to one kernel) ---------------- */
/* The sorted neighbour lists gs_knn votes from, for every row (original order) against the training rows of split `split`:
 * idx_out [n][k] original row indices (-1 past the split's training rows), dist_out [n][k] distances (+inf there); either
 * may be NULL.  metric: GS_KNN_EUCLIDEAN or GS_KNN_MANHATTAN; 1 <= k <= GS_KNN_MAX_NEIGHBORS. */
int gs_debug_knn_neighbors(gs_handle *h, int32_t metric, int32_t k, int32_t split, int32_t *idx_out, double *dist_out);
/* S_out [n][n] float64 Gram X X^T and xsq_out [n] (either may be NULL), in ORIGINAL row order.  */
int gs_debug_gram(gs_handle *h, double *S_out, double *xsq_out);
/* K_out [n][n] float32 kernel matrix (the SMO solver's Q without the y_i*y_j sign), original order; poly / sigmoid take
 * degree and coef0 from gs_set_kernel_params (n = 1).  Optional outputs (NULL: not computed): qd_out [n] the float64
 * diagonal k(x_r, x_r) the solver reads (poly / sigmoid only, GS_ERR_ARG for the other kernels); *special_out the guard
 * flag that sends a search to the general SMO instance: 1 when K holds a zero, a subnormal, a negative or a non-finite
 * value, else 0. */
int gs_debug_kernel_matrix(gs_handle *h, int32_t kernel, double gamma, float *K_out, double *qd_out, int32_t *special_out);
/* dec_out [ncols][n] = sum_j k64(r, j) coef[c][j], the float64 decision values of the SVC / SVR scorers (kernel recomputed
 * in float64 from the Gram; rows r, j in original order).  jchunks = 0: the search's own split of the support rows into
 * slabs, reported in *jchunks_used (may be NULL); 1..64: that many slabs. */
int gs_debug_decision(gs_handle *h, int32_t kernel, double gamma, int32_t degree, double coef0, const double *coef, int32_t ncols,
                      int32_t jchunks, double *dec_out, int32_t *jchunks_used);
/* One scorer kernel on the dataset's labels / targets and splits.  dec [ncols][n] decision values (original row order),
 * rho [ncols] (unused by the AUC kinds); task t reads the columns from first_col[t] (n_classes (n_classes - 1) / 2 of them
 * for the vote kinds, one otherwise) with split fold[t].  out, per task:
 *   GS_DEBUG_SCORE_VOTE          int32 [4] = {test correct, test rows, training correct, training rows}
 *   GS_DEBUG_SCORE_CLASS_COUNTS  int32 [2 (test, training)][n_classes][3 = support, true positives, predicted]
 *   GS_DEBUG_SCORE_AUC_F64       uint64 [4] = {test wins, test ties, training wins, training ties} of the pairs (row of class
 *                                1, row of class 0) on -dec (the SVC search's sign); two classes
 *   GS_DEBUG_SCORE_AUC_F32       the same on (float)dec, sign +1 (LogisticRegression's float32 z)
 *   GS_DEBUG_SCORE_RSS           float64 [2] = residual sums of squares sum (z - (dec - rho))^2 over the test / training rows
 *                                (regression dataset after gs_set_targets_f64) */
enum { GS_DEBUG_SCORE_VOTE = 0, GS_DEBUG_SCORE_CLASS_COUNTS = 1, GS_DEBUG_SCORE_AUC_F64 = 2, GS_DEBUG_SCORE_AUC_F32 = 3,
       GS_DEBUG_SCORE_RSS = 4 };
int gs_debug_score(gs_handle *h, int32_t kind, const double *dec, const double *rho, int32_t ncols, const int32_t *first_col,
                   const int32_t *fold, int32_t n_tasks, void *out);

/* C[M][N] = sum_k A[M][k]*B[N][k] on the wgmma tensor-core path (3xTF32 split), host fp32 row-major in/out. */
int gs_debug_gemm_nt(gs_handle *h, const float *A, int32_t M, const float *B, int32_t N, int32_t K, float *C);
/* C[M][N] = sum_k A[M][k]*B[N][k] on the FP64 tensor-core path of gs_linsvc (K > 1024: split-K with the fixed-order sum of
 * the partials), host float64 row-major in/out. */
int gs_debug_gemm_f64(gs_handle *h, const double *A, int32_t M, const double *B, int32_t N, int32_t K, double *C);

/* ---- planning helpers (host only, no device work; used by gs_svc itself and by the multi-GPU host driver) -------- */
/* Predicted SMO iterations (thousands, for ~8000 training rows) of one C-SVC sub-problem: the model that orders the
 * sub-problems of a search and deals candidates to GPUs.  kernel: GS_KERNEL_*; d = number of features.  Only ratios
 * between candidates are meaningful. */
double gs_svc_predicted_iterations(int32_t kernel, double C, double gamma, int32_t d);
/* Number of sub-problems a search puts on 4-CTA clusters, given the predicted costs sorted in DESCENDING order and
 * the SM count (the makespan model documented in DESIGN.md section 4). */
int32_t gs_svc_cluster_count(const double *cost_desc, int32_t n, int32_t sm_count);
/* Three-tier schedule of the slot-layout solver: of problems sorted by descending predicted cost, *n_cluster go on 4-CTA
 * clusters, the next *n_exclusive get an SM each, the rest share SMs two by two.  The split is the one whose predicted
 * makespan is smallest (the closed-form model documented in csrc/api.cu and DESIGN.md section 4). */
void gs_svc_schedule(const double *cost_desc, int32_t n, int32_t sm_count, int32_t *n_cluster, int32_t *n_exclusive);

/* ---- measurement ----------------------------------------------------------------------- */
typedef struct gs_profile {
    /* last search call; device times from CUDA events on the engine's stream */
    float ms_total;            /* whole call incl. host<->device copies of parameters/results  */
    float ms_h2d;              /* gs_set_data: host->device copy of X/y/fold ids (last call)   */
    float ms_gram;             /* Gram / fold-statistics build                                 */
    float ms_kernel_matrix;    /* exp() materialisation of K_gamma (SVC)                        */
    float ms_solve;            /* SMO / Cholesky / L-BFGS                                       */
    float ms_score;            /* decision values + accuracy / R^2                              */
    int64_t launches;          /* kernels launched by the call                                  */
    int64_t smo_iterations;    /* SVC: total SMO iterations over all sub-problems               */
    double solve_bytes;        /* algorithmic HBM bytes of the dominant solve kernel (DESIGN.md)*/
    double gram_flops;         /* algorithmic flops of the Gram build                           */
    double gram_bytes;         /* algorithmic bytes of the Gram build                           */
    int64_t h2d_bytes;         /* bytes copied host->device by gs_set_data + the search         */
    int64_t d2h_bytes;         /* bytes copied device->host by the search                       */
    float ms_tensor;           /* CUDA-event time of the wgmma contraction launches of the call */
    double tensor_flops;       /* TF32 tensor-core flops those launches executed (3 MMAs per product) */
} gs_profile;
int gs_get_profile(const gs_handle *h, gs_profile *out);

#ifdef __cplusplus
}
#endif
#endif /* B200GS_H */
