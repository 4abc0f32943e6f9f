/* TEST INFRASTRUCTURE, NOT PRODUCT CODE: scikit-learn's SAG / SAGA solver (linear_model/_sag_fast.pyx.tp sag64 / sag32,
 * lagged_update, scale_weights, predict_sample on a dense ArrayDataset), its sample draw (utils/_random.pxd our_rand_r,
 * utils/_seq_dataset.pyx.tp _get_random_index) and the gradients of _loss/_loss.pyx.tp (cgradient_half_binomial,
 * cgradient_half_squared_error, CyHalfMultinomialLoss.cy_gradient) restated in C.  The body below is compiled twice, with
 * T = double (sag64) and T = float (sag32), so every value scikit-learn keeps in T and every operation C evaluates in T or
 * in double is typed as the Cython-generated C types it.  The arrays (cumulative_sums, feature_hist, the gradient memory)
 * are kept as scikit-learn keeps them.  libm's exp as scikit-learn's; built with -ffp-contract=off by sag_oracle.py. */
#ifndef SAG_T
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { LOSS_LOG = 0, LOSS_MULTINOMIAL = 1, LOSS_SQUARED = 2 };

static uint32_t our_rand_r(uint32_t *seed)
{
    if (seed[0] == 0) seed[0] = 1u;
    seed[0] ^= (uint32_t)(seed[0] << 13);
    seed[0] ^= (uint32_t)(seed[0] >> 17);
    seed[0] ^= (uint32_t)(seed[0] << 5);
    return seed[0] % ((uint32_t)0x7fffffff + 1u);
}

/* the first count sample positions dataset.random draws over n rows from this seed */
void oracle_sag_draws(uint32_t seed, int n, int count, int32_t *out)
{
    for (int i = 0; i < count; i++) out[i] = (int)(our_rand_r(&seed) % (uint32_t)n);
}

static double cgradient_half_binomial(double y_true, double raw_prediction)
{
    double exp_tmp;
    if (raw_prediction > -37) {
        exp_tmp = exp(-raw_prediction);
        return ((1 - y_true) - y_true * exp_tmp) / (1 + exp_tmp);
    }
    return exp(raw_prediction) - y_true;
}

#define SAG_T double
#define SAG_FN oracle_sag64
#define SAG_FMAX fmax64
#define SAG_SOFT soft64
#define SAG_LAGGED lagged_update64
#define SAG_SCALE scale_weights64
#include __FILE__
#undef SAG_T
#undef SAG_FN
#undef SAG_FMAX
#undef SAG_SOFT
#undef SAG_LAGGED
#undef SAG_SCALE
#define SAG_T float
#define SAG_FN oracle_sag32
#define SAG_FMAX fmax32
#define SAG_SOFT soft32
#define SAG_LAGGED lagged_update32
#define SAG_SCALE scale_weights32
#include __FILE__

#else  /* ---- the body, once per dtype ---- */

static inline SAG_T SAG_FMAX(SAG_T x, SAG_T y) { return x > y ? x : y; }
static inline SAG_T SAG_SOFT(SAG_T x, SAG_T shrinkage) { return SAG_FMAX(x - shrinkage, 0) - SAG_FMAX(-x - shrinkage, 0); }

/* lagged_update over every feature (dense X: xnnz = n_features, x_ind_ptr = 0 .. n_features - 1) */
static int SAG_LAGGED(SAG_T *weights, SAG_T wscale, int n_features, int n_samples, int n_classes, int sample_itr,
                           SAG_T *cumulative_sums, SAG_T *cumulative_sums_prox, int *feature_hist, int prox, SAG_T *sum_gradient,
                           int reset)
{
    for (int feature_ind = 0; feature_ind < n_features; feature_ind++) {
        const int f_idx = feature_ind * n_classes;
        SAG_T cum_sum = cumulative_sums[sample_itr - 1], cum_sum_prox = 0;
        if (prox) cum_sum_prox = cumulative_sums_prox[sample_itr - 1];
        if (feature_hist[feature_ind] != 0) {
            cum_sum -= cumulative_sums[feature_hist[feature_ind] - 1];
            if (prox) cum_sum_prox -= cumulative_sums_prox[feature_hist[feature_ind] - 1];
        }
        if (!prox) {
            for (int class_ind = 0; class_ind < n_classes; class_ind++) {
                const int idx = f_idx + class_ind;
                weights[idx] -= cum_sum * sum_gradient[idx];
                if (reset) {
                    weights[idx] *= wscale;
                    if (!isfinite(weights[idx])) return -1;
                }
            }
        } else {
            for (int class_ind = 0; class_ind < n_classes; class_ind++) {
                const int idx = f_idx + class_ind;
                if (fabs(sum_gradient[idx] * cum_sum) < cum_sum_prox) {
                    weights[idx] -= cum_sum * sum_gradient[idx];
                    weights[idx] = SAG_SOFT(weights[idx], cum_sum_prox);
                } else {
                    int last_update_ind = feature_hist[feature_ind];
                    if (last_update_ind == -1) last_update_ind = sample_itr - 1;
                    for (int lagged_ind = sample_itr - 1; lagged_ind > last_update_ind - 1; lagged_ind--) {
                        SAG_T grad_step, prox_step;
                        if (lagged_ind > 0) {
                            grad_step = cumulative_sums[lagged_ind] - cumulative_sums[lagged_ind - 1];
                            prox_step = cumulative_sums_prox[lagged_ind] - cumulative_sums_prox[lagged_ind - 1];
                        } else {
                            grad_step = cumulative_sums[lagged_ind];
                            prox_step = cumulative_sums_prox[lagged_ind];
                        }
                        weights[idx] -= sum_gradient[idx] * grad_step;
                        weights[idx] = SAG_SOFT(weights[idx], prox_step);
                    }
                }
                if (reset) {
                    weights[idx] *= wscale;
                    if (!isfinite(weights[idx])) return -1;
                }
            }
        }
        feature_hist[feature_ind] = reset ? sample_itr % n_samples : sample_itr;
    }
    if (reset) {
        cumulative_sums[sample_itr - 1] = 0.0;
        if (prox) cumulative_sums_prox[sample_itr - 1] = 0.0;
    }
    return 0;
}

static int SAG_SCALE(SAG_T *weights, SAG_T *wscale, int n_features, int n_samples, int n_classes, int sample_itr,
                          SAG_T *cumulative_sums, SAG_T *cumulative_sums_prox, int *feature_hist, int prox, SAG_T *sum_gradient)
{
    const int status = SAG_LAGGED(weights, wscale[0], n_features, n_samples, n_classes, sample_itr + 1, cumulative_sums,
                                       cumulative_sums_prox, feature_hist, prox, sum_gradient, 1);
    if (status == 0) wscale[0] = 1.0;
    return status;
}

/* One sag_solver call on X [n][d] (positions in the order scikit-learn sees X[train]) with the dataset's y [n] (0 / 1 for
 * 'log', label codes for 'multinomial', targets for 'squared') and sample weights sw [n], both in T.  n_classes: 1, or the
 * number of classes for 'multinomial'.  alpha / beta are alpha_scaled / beta_scaled; step the step size; intercept_decay 1.
 * coef [n_classes][d + 1]: the weights, then the intercept (coef_init.T).  Returns n_iter; *status 0 stopped by the tol
 * rule, 1 ran max_iter epochs, 2 non-finite (n_iter is that epoch); *steps the samples drawn. */
int SAG_FN(const SAG_T *X, int n_samples, int n_features, int n_classes, const SAG_T *Y, const SAG_T *SW, int loss, int saga,
           double step_size, double alpha, double beta, double tol, int max_iter, int fit_intercept, uint32_t seed, double *coef,
           int *status_out, int64_t *steps)
{
    const int nw = n_features * n_classes;
    SAG_T *weights = calloc(nw ? nw : 1, sizeof(SAG_T)), *sum_gradient = calloc(nw ? nw : 1, sizeof(SAG_T));
    SAG_T *previous_weights = calloc(nw ? nw : 1, sizeof(SAG_T));
    SAG_T *gradient_memory = calloc((size_t)n_samples * n_classes, sizeof(SAG_T));
    SAG_T *cumulative_sums = calloc(n_samples, sizeof(SAG_T)), *cumulative_sums_prox = calloc(n_samples, sizeof(SAG_T));
    SAG_T *intercept = calloc(n_classes, sizeof(SAG_T)), *intercept_sum_gradient = calloc(n_classes, sizeof(SAG_T));
    SAG_T *prediction = calloc(n_classes, sizeof(SAG_T)), *gradient = calloc(n_classes, sizeof(SAG_T));
    int *feature_hist = calloc(n_features ? n_features : 1, sizeof(int)), *seen = calloc(n_samples, sizeof(int));
    const double intercept_decay = 1.0;
    const SAG_T wscale_update = 1.0 - step_size * alpha;
    SAG_T wscale = 1.0;
    int status = 0, num_seen = 0, n_iter = 0, stopped = 0;
    const int prox = beta > 0 && saga;
    int64_t nsteps = 0;
    cumulative_sums[0] = 0.0;

    for (n_iter = 0; n_iter < max_iter; n_iter++) {
        int sample_itr;
        for (sample_itr = 0; sample_itr < n_samples; sample_itr++) {
            const int sample_ind = (int)(our_rand_r(&seed) % (uint32_t)n_samples);
            const SAG_T *x = X + (size_t)sample_ind * n_features;
            const SAG_T y = Y[sample_ind], sample_weight = SW[sample_ind];
            const int s_idx = sample_ind * n_classes;
            nsteps++;
            if (seen[sample_ind] == 0) { num_seen += 1; seen[sample_ind] = 1; }
            if (sample_itr > 0) {
                status = SAG_LAGGED(weights, wscale, n_features, n_samples, n_classes, sample_itr, cumulative_sums,
                                         cumulative_sums_prox, feature_hist, prox, sum_gradient, 0);
                if (status == -1) break;
            }
            /* predict_sample */
            for (int class_ind = 0; class_ind < n_classes; class_ind++) {
                SAG_T innerprod = 0.0;
                for (int j = 0; j < n_features; j++) innerprod += weights[j * n_classes + class_ind] * x[j];
                prediction[class_ind] = wscale * innerprod + intercept[class_ind];
            }
            if (loss == LOSS_MULTINOMIAL) {          /* CyHalfMultinomialLoss.cy_gradient, sum_exp_minus_max */
                double max_value = prediction[0], sum_exps = 0;
                for (int k = 1; k < n_classes; k++)
                    if (max_value < prediction[k]) max_value = prediction[k];
                for (int k = 0; k < n_classes; k++) {
                    gradient[k] = exp(prediction[k] - max_value);
                    sum_exps += gradient[k];
                }
                for (int k = 0; k < n_classes; k++) {
                    gradient[k] /= sum_exps;
                    gradient[k] = (gradient[k] - (y == k)) * sample_weight;
                }
            } else if (loss == LOSS_LOG) {
                gradient[0] = cgradient_half_binomial(y, prediction[0]) * sample_weight;
            } else {
                gradient[0] = ((double)prediction[0] - (double)y) * sample_weight;
            }
            wscale *= wscale_update;
            for (int j = 0; j < n_features; j++) {
                const SAG_T val = x[j];
                const int f_idx = j * n_classes;
                for (int class_ind = 0; class_ind < n_classes; class_ind++) {
                    const SAG_T gradient_correction = val * (gradient[class_ind] - gradient_memory[s_idx + class_ind]);
                    if (saga)
                        weights[f_idx + class_ind] -= (gradient_correction * step_size * (1 - 1. / num_seen) / wscale);
                    sum_gradient[f_idx + class_ind] += gradient_correction;
                }
            }
            if (fit_intercept) {
                for (int class_ind = 0; class_ind < n_classes; class_ind++) {
                    SAG_T gradient_correction = (gradient[class_ind] - gradient_memory[s_idx + class_ind]);
                    intercept_sum_gradient[class_ind] += gradient_correction;
                    gradient_correction *= step_size * (1. - 1. / num_seen);
                    if (saga)
                        intercept[class_ind] -= (step_size * intercept_sum_gradient[class_ind] / num_seen * intercept_decay) +
                                                gradient_correction;
                    else
                        intercept[class_ind] -= (step_size * intercept_sum_gradient[class_ind] / num_seen * intercept_decay);
                    if (!isfinite(intercept[class_ind])) { status = -1; break; }
                }
                if (status == -1) break;
            }
            for (int class_ind = 0; class_ind < n_classes; class_ind++) gradient_memory[s_idx + class_ind] = gradient[class_ind];
            if (sample_itr == 0) {
                cumulative_sums[0] = step_size / (wscale * num_seen);
                if (prox) cumulative_sums_prox[0] = step_size * beta / wscale;
            } else {
                cumulative_sums[sample_itr] = (cumulative_sums[sample_itr - 1] + step_size / (wscale * num_seen));
                if (prox) cumulative_sums_prox[sample_itr] = (cumulative_sums_prox[sample_itr - 1] + step_size * beta / wscale);
            }
            if (wscale < 1e-9) {
                status = SAG_SCALE(weights, &wscale, n_features, n_samples, n_classes, sample_itr, cumulative_sums,
                                        cumulative_sums_prox, feature_hist, prox, sum_gradient);
                if (status == -1) break;
            }
        }
        if (status == -1) break;
        status = SAG_SCALE(weights, &wscale, n_features, n_samples, n_classes, n_samples - 1, cumulative_sums,
                                cumulative_sums_prox, feature_hist, prox, sum_gradient);
        if (status == -1) break;
        SAG_T max_change = 0.0, max_weight = 0.0;
        for (int idx = 0; idx < nw; idx++) {
            max_weight = SAG_FMAX(max_weight, fabs(weights[idx]));
            max_change = SAG_FMAX(max_change, fabs(weights[idx] - previous_weights[idx]));
            previous_weights[idx] = weights[idx];
        }
        if ((max_weight != 0 && max_change / max_weight <= tol) || (max_weight == 0 && max_change == 0)) { stopped = 1; break; }
    }
    /* Cython leaves a finished range() loop's variable at its last value: max_iter epochs give n_iter = max_iter */
    if (!stopped && status != -1) n_iter = max_iter > 0 ? max_iter - 1 : 0;
    n_iter += 1;
    *status_out = status == -1 ? 2 : (stopped ? 0 : 1);
    *steps = nsteps;
    for (int k = 0; k < n_classes; k++) {
        for (int j = 0; j < n_features; j++) coef[(size_t)k * (n_features + 1) + j] = weights[j * n_classes + k];
        coef[(size_t)k * (n_features + 1) + n_features] = intercept[k];
    }
    free(weights); free(sum_gradient); free(previous_weights); free(gradient_memory); free(cumulative_sums);
    free(cumulative_sums_prox); free(intercept); free(intercept_sum_gradient); free(prediction); free(gradient);
    free(feature_hist); free(seen);
    return n_iter;
}

#endif
