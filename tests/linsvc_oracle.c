/* linsvc_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE: liblinear's primal L2-regularised squared-hinge solver
 * (L2R_L2LOSS_SVC) restated in float64 on a dense matrix, the checker of csrc/linsvc.cu.
 *
 * Restates, from the liblinear sources scikit-learn 1.9 ships (sklearn/svm/src/liblinear):
 *   linear.cpp:2453-2578 train        remove_zero_weight; rows grouped by class in label order, stable; weighted_C[i] =
 *                                     C x weight[i]; binary: class 0 -> -1, train_one(Cp = weighted_C[1], Cn = weighted_C[0]);
 *                                     one-vs-rest: class i -> +1, train_one(Cp = weighted_C[i], Cn = C)
 *   linear.cpp:2309-2362 train_one    C_i = W_i x (Cp | Cn), primal_solver_tol = eps x max(min(pos, neg), 1) / l
 *   linear.cpp:228-390 l2r_l2_svc_fun fun / grad / Hv with the active set I of the latest grad(), Xv / subXv / subXTv as
 *                                     sequential loops over each row's non-zero features (liblinear_helper.c dense_to_sparse
 *                                     drops zeros and appends the bias feature)
 *   tron.cpp:44-209 TRON::tron, trcg  eta0 1e-4, eta1 0.25, eta2 0.75, sigma1 0.25, sigma2 0.5, sigma3 4; delta = min(delta,
 *                                     snorm) on the first iteration; three stop tests; returns --iter
 * dot / nrm2 / axpy are sequential loops here (scikit-learn's go through scipy's BLAS), so results agree with scikit-learn
 * to the rounding of reordered float64 sums, not bit for bit.
 *
 * Trace (optional): one record of TRACE_W doubles per TRON iteration -- iter, accepted, actred, prered, delta (after the
 * update), f (before the step), gnorm (before the step), cg_iter, snorm, fnew.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define TRACE_W 10

typedef struct {
    int l, n;              /* rows, variables (features + bias) */
    const double *X;       /* [l][nx] rows of the problem, in problem order */
    int nx;                /* features */
    double bias;           /* <= 0: no bias feature */
    double *y, *C, *z;
    int *I, sizeI;
} fun_t;

static double dot(int n, const double *a, const double *b) { double s = 0; for (int i = 0; i < n; i++) s += a[i] * b[i]; return s; }
static double nrm2(int n, const double *a) { return sqrt(dot(n, a, a)); }
static void axpy(int n, double a, const double *x, double *y) { for (int i = 0; i < n; i++) y[i] += a * x[i]; }
static void scal(int n, double a, double *x) { for (int i = 0; i < n; i++) x[i] *= a; }

static double row_dot(const fun_t *F, int i, const double *v)
{
    const double *x = F->X + (size_t)i * F->nx;
    double s = 0;
    for (int j = 0; j < F->nx; j++) if (x[j] != 0) s += v[j] * x[j];
    if (F->bias > 0) s += v[F->nx] * F->bias;
    return s;
}
static void row_axpy(const fun_t *F, int i, double a, double *out)
{
    const double *x = F->X + (size_t)i * F->nx;
    for (int j = 0; j < F->nx; j++) if (x[j] != 0) out[j] += a * x[j];
    if (F->bias > 0) out[F->nx] += a * F->bias;
}

static double fun(fun_t *F, const double *w)
{
    double f = 0;
    for (int i = 0; i < F->l; i++) F->z[i] = row_dot(F, i, w);
    for (int i = 0; i < F->n; i++) f += w[i] * w[i];
    f /= 2.0;
    for (int i = 0; i < F->l; i++) {
        F->z[i] = F->y[i] * F->z[i];
        double d = 1 - F->z[i];
        if (d > 0) f += F->C[i] * d * d;
    }
    return f;
}

static void grad(fun_t *F, const double *w, double *g)
{
    F->sizeI = 0;
    for (int i = 0; i < F->l; i++)
        if (F->z[i] < 1) {
            F->z[F->sizeI] = F->C[i] * F->y[i] * (F->z[i] - 1);
            F->I[F->sizeI] = i;
            F->sizeI++;
        }
    memset(g, 0, sizeof(double) * F->n);
    for (int i = 0; i < F->sizeI; i++) row_axpy(F, F->I[i], F->z[i], g);
    for (int i = 0; i < F->n; i++) g[i] = w[i] + 2 * g[i];
}

static void Hv(fun_t *F, const double *s, double *Hs)
{
    double *wa = malloc(sizeof(double) * (F->sizeI + 1));
    for (int i = 0; i < F->sizeI; i++) wa[i] = F->C[F->I[i]] * row_dot(F, F->I[i], s);
    memset(Hs, 0, sizeof(double) * F->n);
    for (int i = 0; i < F->sizeI; i++) row_axpy(F, F->I[i], wa[i], Hs);
    for (int i = 0; i < F->n; i++) Hs[i] = s[i] + 2 * Hs[i];
    free(wa);
}

static int trcg(fun_t *F, double delta, const double *g, double *s, double *r)
{
    const int n = F->n;
    double *d = malloc(sizeof(double) * n), *Hd = malloc(sizeof(double) * n);
    for (int i = 0; i < n; i++) { s[i] = 0; r[i] = -g[i]; d[i] = r[i]; }
    const double cgtol = 0.1 * nrm2(n, g);
    int cg_iter = 0;
    double rTr = dot(n, r, r);
    while (1) {
        if (nrm2(n, r) <= cgtol) break;
        cg_iter++;
        Hv(F, d, Hd);
        double alpha = rTr / dot(n, d, Hd);
        axpy(n, alpha, d, s);
        if (nrm2(n, s) > delta) {
            alpha = -alpha;
            axpy(n, alpha, d, s);
            double std = dot(n, s, d), sts = dot(n, s, s), dtd = dot(n, d, d), dsq = delta * delta;
            double rad = sqrt(std * std + dtd * (dsq - sts));
            if (std >= 0) alpha = (dsq - sts) / (std + rad);
            else alpha = (rad - std) / dtd;
            axpy(n, alpha, d, s);
            alpha = -alpha;
            axpy(n, alpha, Hd, r);
            break;
        }
        alpha = -alpha;
        axpy(n, alpha, Hd, r);
        double rnewTrnew = dot(n, r, r);
        double beta = rnewTrnew / rTr;
        scal(n, beta, d);
        axpy(n, 1.0, r, d);
        rTr = rnewTrnew;
    }
    free(d); free(Hd);
    return cg_iter;
}

static int tron(fun_t *F, double *w, double eps, int max_iter, double *trace, int trace_cap, int *trace_len)
{
    const double eta0 = 1e-4, eta1 = 0.25, eta2 = 0.75, sigma1 = 0.25, sigma2 = 0.5, sigma3 = 4;
    const int n = F->n;
    double *s = malloc(sizeof(double) * n), *r = malloc(sizeof(double) * n), *w_new = malloc(sizeof(double) * n),
           *g = malloc(sizeof(double) * n);
    int search = 1, iter = 1;
    for (int i = 0; i < n; i++) w[i] = 0;
    double f = fun(F, w);
    grad(F, w, g);
    double delta = nrm2(n, g), gnorm1 = delta, gnorm = gnorm1;
    if (gnorm <= eps * gnorm1) search = 0;
    while (iter <= max_iter && search) {
        const int cg_iter = trcg(F, delta, g, s, r);
        memcpy(w_new, w, sizeof(double) * n);
        axpy(n, 1.0, s, w_new);
        const double gs = dot(n, g, s);
        const double prered = -0.5 * (gs - dot(n, s, r));
        const double fnew = fun(F, w_new);
        const double actred = f - fnew;
        const double snorm = nrm2(n, s);
        double alpha;
        if (iter == 1) delta = fmin(delta, snorm);
        if (fnew - f - gs <= 0) alpha = sigma3;
        else alpha = fmax(sigma1, -0.5 * (gs / (fnew - f - gs)));
        if (actred < eta0 * prered) delta = fmin(fmax(alpha, sigma1) * snorm, sigma2 * delta);
        else if (actred < eta1 * prered) delta = fmax(sigma1 * delta, fmin(alpha * snorm, sigma2 * delta));
        else if (actred < eta2 * prered) delta = fmax(sigma1 * delta, fmin(alpha * snorm, sigma3 * delta));
        else delta = fmax(delta, fmin(alpha * snorm, sigma3 * delta));
        const int accepted = actred > eta0 * prered;
        if (trace && *trace_len < trace_cap) {
            double *t = trace + (size_t)(*trace_len)++ * TRACE_W;
            t[0] = iter; t[1] = accepted; t[2] = actred; t[3] = prered; t[4] = delta; t[5] = f; t[6] = gnorm; t[7] = cg_iter;
            t[8] = snorm; t[9] = fnew;
        }
        if (accepted) {
            iter++;
            memcpy(w, w_new, sizeof(double) * n);
            f = fnew;
            grad(F, w, g);
            gnorm = nrm2(n, g);
            if (gnorm <= eps * gnorm1) break;
        }
        if (f < -1.0e+32) break;
        if (fabs(actred) <= 0 && prered <= 0) break;
        if (fabs(actred) <= 1.0e-12 * fabs(f) && fabs(prered) <= 1.0e-12 * fabs(f)) break;
    }
    free(s); free(r); free(w_new); free(g);
    return --iter;
}

/* X [l][nx] dense rows, y [l] class ids 0..nc-1, W [l] sample weights, cw [nc] class weights (scikit-learn's class_weight_),
 * bias > 0: the bias feature.  w_out [rows][nx + (bias > 0)], rows = 1 (nc == 2) or nc; n_iter [rows].
 * trace: [rows][trace_cap][TRACE_W] (may be NULL), trace_len [rows].  Returns -1 when a class has no row of positive weight. */
int oracle_linsvc_train(const double *X, int l0, int nx, const int *y0, const double *W0, int nc, double Cval, const double *cw,
                        double bias, double tol, int max_iter, double *w_out, int *n_iter, double *trace, int trace_cap,
                        int *trace_len)
{
    const int n = nx + (bias > 0 ? 1 : 0);
    /* remove_zero_weight, then group_classes: by class, stable */
    int l = 0;
    int *count = calloc(nc, sizeof(int));
    for (int i = 0; i < l0; i++) if (W0[i] > 0) { l++; count[y0[i]]++; }
    for (int c = 0; c < nc; c++) if (count[c] == 0) { free(count); return -1; }
    int *start = malloc(sizeof(int) * nc), *perm = malloc(sizeof(int) * l), *fill = calloc(nc, sizeof(int));
    start[0] = 0;
    for (int c = 1; c < nc; c++) start[c] = start[c - 1] + count[c - 1];
    for (int i = 0; i < l0; i++) if (W0[i] > 0) perm[start[y0[i]] + fill[y0[i]]++] = i;
    double *Xp = malloc(sizeof(double) * (size_t)l * nx), *W = malloc(sizeof(double) * l);
    for (int k = 0; k < l; k++) { memcpy(Xp + (size_t)k * nx, X + (size_t)perm[k] * nx, sizeof(double) * nx); W[k] = W0[perm[k]]; }
    double *wC = malloc(sizeof(double) * nc);
    for (int c = 0; c < nc; c++) wC[c] = Cval * cw[c];

    fun_t F;
    F.l = l; F.n = n; F.X = Xp; F.nx = nx; F.bias = bias;
    F.y = malloc(sizeof(double) * l); F.C = malloc(sizeof(double) * l); F.z = malloc(sizeof(double) * l); F.I = malloc(sizeof(int) * l);
    const int rows = nc == 2 ? 1 : nc;
    for (int q = 0; q < rows; q++) {
        double Cp, Cn;
        if (nc == 2) {
            for (int k = 0; k < l; k++) F.y[k] = k < start[0] + count[0] ? -1 : +1;
            Cp = wC[1]; Cn = wC[0];
        } else {
            for (int k = 0; k < l; k++) F.y[k] = (k >= start[q] && k < start[q] + count[q]) ? +1 : -1;
            Cp = wC[q]; Cn = Cval;
        }
        int pos = 0;
        for (int k = 0; k < l; k++) if (F.y[k] > 0) pos++;
        const int neg = l - pos;
        const int m = pos < neg ? pos : neg;
        const double primal_solver_tol = tol * (m > 1 ? m : 1) / l;
        for (int k = 0; k < l; k++) F.C[k] = F.y[k] > 0 ? W[k] * Cp : W[k] * Cn;
        if (trace_len) trace_len[q] = 0;
        n_iter[q] = tron(&F, w_out + (size_t)q * n, primal_solver_tol, max_iter,
                         trace ? trace + (size_t)q * trace_cap * TRACE_W : NULL, trace_cap, trace_len ? trace_len + q : NULL);
    }
    free(F.y); free(F.C); free(F.z); free(F.I);
    free(count); free(start); free(perm); free(fill); free(Xp); free(W); free(wC);
    return 0;
}
