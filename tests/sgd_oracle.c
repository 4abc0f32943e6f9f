/* TEST INFRASTRUCTURE, NOT PRODUCT CODE: scikit-learn's plain SGD (_sgd_fast.pyx.tp _plain_sgd, utils/_weight_vector.pyx.tp
 * WeightVector, utils/_seq_dataset.pyx.tp ArrayDataset.shuffle with our_rand_r) restated in C, for float64 X (_plain_sgd64)
 * and float32 X (_plain_sgd32: every value scikit-learn keeps in float is rounded to float -- w, q, the local wscale copies
 * of add() and reset_wscale(), norm() and l1norm() -- while WeightVector32's wscale, sq_norm and l1_norm stay double; a
 * float operation made in double and rounded once gives the float result).  Built with -ffp-contract=off by sgd_oracle.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { HINGE, PERCEPTRON, SQUARED_HINGE, MODIFIED_HUBER, LOG_LOSS, SQUARED_ERROR, HUBER, EPS_INS, SQ_EPS_INS };
enum { P_NONE = 0, P_L1 = 1, P_L2 = 2, P_EN = 3 };
enum { CONSTANT = 1, OPTIMAL = 2, INVSCALING = 3, ADAPTIVE = 4 };

static int F32;
static double R(double v) { return F32 ? (double)(float)v : v; }

static double log1pexp(double x)
{
    if (x <= -37) return exp(x);
    if (x <= -2) return log1p(exp(x));
    if (x <= 18) return log(1. + exp(x));
    if (x <= 33.3) return x + exp(-x);
    return x;
}

static double loss_of(int loss, double th, double y, double p)
{
    double z, r, a;
    switch (loss) {
    case HINGE: case PERCEPTRON: z = p * y; return z <= th ? th - z : 0.0;
    case SQUARED_HINGE: z = th - p * y; return z > 0 ? z * z : 0.0;
    case MODIFIED_HUBER: z = p * y; if (z >= 1.0) return 0.0; if (z >= -1.0) return (1.0 - z) * (1.0 - z); return -4.0 * z;
    case LOG_LOSS: return log1pexp(p) - y * p;
    case SQUARED_ERROR: return 0.5 * (p - y) * (p - y);
    case HUBER: a = fabs(y - p); return a <= th ? 0.5 * (a * a) : th * (a - 0.5 * th);
    case EPS_INS: r = fabs(y - p) - th; return r > 0 ? r : 0;
    default: r = fabs(y - p) - th; return r > 0 ? r * r : 0;
    }
}

double oracle_sgd_dloss(int loss, double th, double y, double p)
{
    double z, e, r;
    switch (loss) {
    case HINGE: case PERCEPTRON: return p * y <= th ? -y : 0.0;
    case SQUARED_HINGE: z = th - p * y; return z > 0 ? -2 * y * z : 0.0;
    case MODIFIED_HUBER: z = p * y; if (z >= 1.0) return 0.0; if (z >= -1.0) return 2.0 * (1.0 - z) * -y; return -4.0 * y;
    case LOG_LOSS: if (p > -37) { e = exp(-p); return ((1 - y) - y * e) / (1 + e); } return exp(p) - y;
    case SQUARED_ERROR: return p - y;
    case HUBER: r = p - y; return fabs(r) <= th ? r : (r >= 0 ? th : -th);
    case EPS_INS: return y - p > th ? -1 : (p - y > th ? 1 : 0);
    default: z = y - p; if (z > th) return -2 * (z - th); if (z < -th) return 2 * (-z - th); return 0;
    }
}

/* pi: ArrayDataset.shuffle(seed) applied to the identity */
void oracle_sgd_perm(uint32_t seed, int n, int *ind)
{
    for (int i = 0; i < n; i++) ind[i] = i;
    uint32_t s = seed ? seed : 1u;
    for (unsigned i = 0; i + 1 < (unsigned)n; i++) {
        s ^= (uint32_t)(s << 13);
        s ^= (uint32_t)(s >> 17);
        s ^= (uint32_t)(s << 5);
        unsigned j = i + (s % (0x7fffffffu + 1u)) % (unsigned)(n - i);
        int t = ind[i]; ind[i] = ind[j]; ind[j] = t;
    }
}

/* One fit.  X [n][d] (float64, or float32 when f32), y [n] already encoded (+1 / -1, 1 / 0 for log_loss, or targets),
 * sw [n].  Returns n_iter; *status 0 stopped, 1 max_iter epochs, 2 non-finite (n_iter is that epoch).  coef [d], *icpt. */
int oracle_sgd_fit(const void *Xv, int f32, int n, int d, const double *y, const double *sw, int loss, double th, int penalty,
                   double alpha, double l1_ratio, int lr, double eta0, double power_t, double tol, int max_iter, int n_iter_no_change,
                   int fit_intercept, int shuffle, uint32_t seed, double wpos, double wneg, double *coef, double *icpt, int *status)
{
    F32 = f32;
    const double *X64 = (const double *)Xv;
    const float *X32 = (const float *)Xv;
    double *w = calloc(d, sizeof(double)), *q = calloc(d, sizeof(double)), *x = malloc(sizeof(double) * (d ? d : 1));
    int *ind = malloc(sizeof(int) * n);
    for (int i = 0; i < n; i++) ind[i] = i;
    double wscale = 1.0, sq_norm = 0.0, l1_norm = 0.0, intercept = 0.0, t = 1.0, eta = eta0, u = 0.0, best = INFINITY;
    const double thr = f32 ? 1e-6 : 1e-9;
    if (penalty == P_L2) l1_ratio = 0.0;
    else if (penalty == P_L1) l1_ratio = 1.0;
    double optimal_init = 0.0;
    if (lr == OPTIMAL) {
        double typw = sqrt(1.0 / sqrt(alpha));
        double g = oracle_sgd_dloss(loss, th, 1.0, -typw);
        double ie = typw / (g > 1.0 ? g : 1.0);
        optimal_init = 1.0 / (ie * alpha);
    }
    const double cwp = R(wpos), cwn = R(wneg);
    int epoch, nic = 0, st = 1;
    for (epoch = 0; epoch < max_iter; epoch++) {
        double obj = 0;
        if (shuffle) {
            uint32_t s = seed ? seed : 1u;
            for (unsigned i = 0; i + 1 < (unsigned)n; i++) {
                s ^= (uint32_t)(s << 13);
                s ^= (uint32_t)(s >> 17);
                s ^= (uint32_t)(s << 5);
                unsigned j = i + (s % (0x7fffffffu + 1u)) % (unsigned)(n - i);
                int tmp = ind[i]; ind[i] = ind[j]; ind[j] = tmp;
            }
        }
        for (int ii = 0; ii < n; ii++) {
            const int r = ind[ii];
            for (int j = 0; j < d; j++) x[j] = f32 ? (double)X32[(size_t)r * d + j] : X64[(size_t)r * d + j];
            const double yy = R(y[r]), s_w = R(sw[r]);
            double acc = 0.0;
            for (int j = 0; j < d; j++) acc += R(w[j] * x[j]);
            acc *= wscale;
            const double p = R(acc) + intercept;
            if (lr == OPTIMAL) eta = 1.0 / (alpha * (optimal_init + t - 1));
            else if (lr == INVSCALING) eta = eta0 / pow(t, power_t);
            obj += loss_of(loss, th, yy, p);
            if (penalty > 0) {
                const double nrm = R(sqrt(sq_norm));
                obj += alpha * ((1 - l1_ratio) * 0.5 * (nrm * nrm) + l1_ratio * R(l1_norm));
            }
            const double cw = yy > 0.0 ? cwp : cwn;
            double dl = oracle_sgd_dloss(loss, th, yy, p);
            if (dl < -1e12) dl = -1e12;
            else if (dl > 1e12) dl = 1e12;
            double update = -eta * dl;
            update *= R(cw * s_w);
            if (penalty >= P_L2) {
                double c = 1.0 - ((1.0 - l1_ratio) * eta * alpha);
                c = R(c > 0 ? c : 0.0);
                wscale = wscale * c;
                sq_norm = sq_norm * R(c * c);
                l1_norm = l1_norm * fabs(c);
                if (wscale < thr) {
                    for (int j = 0; j < d; j++) w[j] = R(w[j] * R(wscale));
                    wscale = 1.0;
                }
            }
            if (update != 0.0) {
                const double wsf = R(wscale), cu = R(R(update) / wsf);
                double a2 = 0.0, a1 = 0.0;
                for (int j = 0; j < d; j++) {
                    w[j] = R(w[j] + x[j] * cu);
                    a2 += R(w[j] * w[j]);
                    a1 += fabs(w[j]);
                }
                sq_norm = a2 * R(wsf * wsf);
                l1_norm = a1 * wsf;
            }
            if (fit_intercept && update != 0) intercept += update;
            if (penalty == P_L1 || penalty == P_EN) {
                u += (l1_ratio * eta * alpha);
                for (int j = 0; j < d; j++) {
                    const double z = w[j];
                    if (wscale * z > 0.0) { const double v = w[j] - ((u + q[j]) / wscale); w[j] = R(v > 0.0 ? v : 0.0); }
                    else if (wscale * z < 0.0) { const double v = w[j] + ((u - q[j]) / wscale); w[j] = R(v < 0.0 ? v : 0.0); }
                    q[j] = R(q[j] + wscale * (w[j] - z));
                }
            }
            t += 1;
        }
        int bad = !isfinite(intercept);
        for (int j = 0; j < d; j++) bad |= !isfinite(w[j]);
        if (bad) { st = 2; break; }
        const double mean = obj / n;
        if (tol > -INFINITY && mean > best - tol) nic++;
        else nic = 0;
        if (mean < best) best = mean;
        if (nic >= n_iter_no_change) {
            if (lr == ADAPTIVE && eta > 1e-6) { eta = eta / 5; nic = 0; }
            else { st = 0; break; }
        }
    }
    for (int j = 0; j < d; j++) coef[j] = R(w[j] * R(wscale));
    *icpt = intercept;
    *status = st;
    free(w); free(q); free(x); free(ind);
    return st == 1 ? max_iter : epoch + 1;
}
