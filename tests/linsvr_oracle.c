/* linsvr_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE: liblinear's three L2-regularised SVR solvers restated in
 * float64 on a dense matrix, the checker of csrc/linsvr.cu.
 *
 * Restates, from the liblinear sources scikit-learn 1.9 ships (sklearn/svm/src/liblinear, newrand/newrand.h):
 *   train                    remove_zero_weight (rows of weight <= 0 dropped, order kept); a regression problem is one
 *                            train_one on every remaining row
 *   train_one                L2R_L2LOSS_SVR (11): C_i = C W_i, TRON(eps = tol) on l2r_l2_svr_fun;
 *                            L2R_L2LOSS_SVR_DUAL (12) / L2R_L1LOSS_SVR_DUAL (13): solve_l2r_l1l2_svr
 *   solve_l2r_l1l2_svr       dual coordinate descent: lambda_i = 0.5 / C_i and no upper bound (12), lambda 0 and
 *                            |beta_i| <= C_i (13); a Fisher-Yates shuffle of the active set every epoch with
 *                            bounded_rand_int; shrinking against Gmax_old; the |d| < 1e-12 skip; the stop
 *                            Gnorm1 <= eps Gnorm1_init, which unshrinks and continues while the active set is not full
 *   l2r_l2_svr_fun           f = w'w / 2 + sum C_i (|z_i - y_i| - p)_+^2, g = w + 2 X_I' C_I (d -/+ p), Hs on the same set
 *   newrand.h                std::mt19937 seeded by set_seed; bounded_rand_int = Lemire's multiply-shift with rejection
 * Rows are sparse in liblinear (liblinear_helper.c drops zeros and appends the bias feature): dot, nrm2_sq and axpy are
 * sequential loops over the non-zero features, then the bias.  TRON's vector operations go through BLAS in scikit-learn and
 * are sequential loops here, so solver 11 agrees with scikit-learn to the rounding of reordered sums, not bit for bit.
 *
 * kernel_order != 0 sums every CD dot product in the order of csrc/linsvr.cu instead: 32 lanes, lane L sums features
 * L, L + 32, ... in ascending order, then an xor butterfly over 16, 8, 4, 2, 1.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- std::mt19937 and bounded_rand_int ---- */
static uint32_t mt[624];
static int mti = 625;

void oracle_mt_seed(uint32_t s)
{
    mt[0] = s;
    for (int i = 1; i < 624; i++) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
    mti = 624;
}

uint32_t oracle_mt_next(void)
{
    if (mti >= 624) {
        for (int i = 0; i < 624; i++) {
            const uint32_t y = (mt[i] & 0x80000000u) | (mt[(i + 1) % 624] & 0x7fffffffu);
            mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        mti = 0;
    }
    uint32_t y = mt[mti++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

uint32_t oracle_bounded_rand_int(uint32_t range)
{
    uint32_t x = oracle_mt_next();
    uint64_t m = (uint64_t)x * (uint64_t)range;
    uint32_t l = (uint32_t)m;
    if (l < range) {
        uint32_t t = -range;
        if (t >= range) {
            t -= range;
            if (t >= range) t %= range;
        }
        while (l < t) {
            x = oracle_mt_next();
            m = (uint64_t)x * (uint64_t)range;
            l = (uint32_t)m;
        }
    }
    return (uint32_t)(m >> 32);
}

/* ---- the problem: dense rows, the bias as feature nx when bias > 0 ---- */
typedef struct {
    int l, n, nx;
    const double *X;
    double bias;
    const double *y, *C;
    double p;
    double *z;
    int *I, sizeI;
} prob_t;

static double row_dot(const prob_t *P, int i, const double *v)
{
    const double *x = P->X + (size_t)i * P->nx;
    double s = 0;
    for (int j = 0; j < P->nx; j++) if (x[j] != 0) s += v[j] * x[j];
    if (P->bias > 0) s += v[P->nx] * P->bias;
    return s;
}

/* the dot product of csrc/linsvr.cu's warp: per-lane sequential partial sums, then the xor butterfly */
static double row_dot_kernel(const prob_t *P, int i, const double *v)
{
    const double *x = P->X + (size_t)i * P->nx;
    double part[32];
    for (int L = 0; L < 32; L++) {
        double s = 0;
        for (int j = L; j < P->n; j += 32) {
            const double xj = j < P->nx ? x[j] : P->bias;
            s += v[j] * xj;
        }
        part[L] = s;
    }
    for (int m = 16; m; m >>= 1) {
        double nxt[32];
        for (int L = 0; L < 32; L++) nxt[L] = part[L] + part[L ^ m];
        memcpy(part, nxt, sizeof part);
    }
    return part[0];
}

static void row_axpy(const prob_t *P, int i, double a, double *out)
{
    const double *x = P->X + (size_t)i * P->nx;
    for (int j = 0; j < P->nx; j++) if (x[j] != 0) out[j] += a * x[j];
    if (P->bias > 0) out[P->nx] += a * P->bias;
}

static double row_nrm2_sq(const prob_t *P, int i)
{
    const double *x = P->X + (size_t)i * P->nx;
    double s = 0;
    for (int j = 0; j < P->nx; j++) if (x[j] != 0) s += x[j] * x[j];
    if (P->bias > 0) s += P->bias * P->bias;
    return s;
}

/* ---- solve_l2r_l1l2_svr ---- */
#define INF HUGE_VAL
static int solve_svr_dual(const prob_t *P, double *w, int l1loss, double eps, int max_iter, int kernel_order, int64_t *steps)
{
    const int l = P->l, w_size = P->n;
    int i, s, iter = 0, active_size = l;
    int *index = malloc(sizeof(int) * l);
    double d, G, H, Gmax_old = INF, Gmax_new, Gnorm1_new, Gnorm1_init = -1.0;
    double *beta = malloc(sizeof(double) * l), *QD = malloc(sizeof(double) * l);
    double *lambda = malloc(sizeof(double) * l), *upper_bound = malloc(sizeof(double) * l);
    for (i = 0; i < l; i++) {
        if (l1loss) { lambda[i] = 0; upper_bound[i] = P->C[i]; }
        else { lambda[i] = 0.5 / P->C[i]; upper_bound[i] = INF; }
    }
    for (i = 0; i < l; i++) beta[i] = 0;
    for (i = 0; i < w_size; i++) w[i] = 0;
    for (i = 0; i < l; i++) {
        QD[i] = row_nrm2_sq(P, i);
        row_axpy(P, i, beta[i], w);
        index[i] = i;
    }
    *steps = 0;
    while (iter < max_iter) {
        Gmax_new = 0;
        Gnorm1_new = 0;
        for (i = 0; i < active_size; i++) {
            int j = i + (int)oracle_bounded_rand_int((uint32_t)(active_size - i));
            int t = index[i]; index[i] = index[j]; index[j] = t;
        }
        for (s = 0; s < active_size; s++) {
            (*steps)++;
            i = index[s];
            G = -P->y[i] + lambda[i] * beta[i];
            H = QD[i] + lambda[i];
            if (kernel_order) G += row_dot_kernel(P, i, w);
            else {                                   /* scikit-learn's copy accumulates the row into G itself */
                const double *x = P->X + (size_t)i * P->nx;
                for (int j = 0; j < P->nx; j++) if (x[j] != 0) G += x[j] * w[j];
                if (P->bias > 0) G += P->bias * w[P->nx];
            }
            double Gp = G + P->p, Gn = G - P->p, violation = 0;
            if (beta[i] == 0) {
                if (Gp < 0) violation = -Gp;
                else if (Gn > 0) violation = Gn;
                else if (Gp > Gmax_old && Gn < -Gmax_old) {
                    active_size--;
                    int t = index[s]; index[s] = index[active_size]; index[active_size] = t;
                    s--;
                    continue;
                }
            } else if (beta[i] >= upper_bound[i]) {
                if (Gp > 0) violation = Gp;
                else if (Gp < -Gmax_old) {
                    active_size--;
                    int t = index[s]; index[s] = index[active_size]; index[active_size] = t;
                    s--;
                    continue;
                }
            } else if (beta[i] <= -upper_bound[i]) {
                if (Gn < 0) violation = -Gn;
                else if (Gn > Gmax_old) {
                    active_size--;
                    int t = index[s]; index[s] = index[active_size]; index[active_size] = t;
                    s--;
                    continue;
                }
            } else if (beta[i] > 0) violation = fabs(Gp);
            else violation = fabs(Gn);
            Gmax_new = Gmax_new < violation ? violation : Gmax_new;
            Gnorm1_new += violation;
            if (Gp < H * beta[i]) d = -Gp / H;
            else if (Gn > H * beta[i]) d = -Gn / H;
            else d = -beta[i];
            if (fabs(d) < 1.0e-12) continue;
            double beta_old = beta[i];
            double lo = beta[i] + d;
            lo = lo < -upper_bound[i] ? -upper_bound[i] : lo;                 /* max(beta + d, -ub) */
            beta[i] = upper_bound[i] < lo ? upper_bound[i] : lo;               /* min(., ub) */
            d = beta[i] - beta_old;
            if (d != 0) row_axpy(P, i, d, w);
        }
        if (iter == 0) Gnorm1_init = Gnorm1_new;
        iter++;
        if (Gnorm1_new <= eps * Gnorm1_init) {
            if (active_size == l) break;
            active_size = l;
            Gmax_old = INF;
            continue;
        }
        Gmax_old = Gmax_new;
    }
    free(index); free(beta); free(QD); free(lambda); free(upper_bound);
    return iter;
}

/* ---- l2r_l2_svr_fun and TRON (as tests/linsvc_oracle.c restates it) ---- */
static double dot(int n, const double *a, const double *b) { double s = 0; for (int i = 0; i < n; i++) s += a[i] * b[i]; return s; }
static double nrm2(int n, const double *a) { return sqrt(dot(n, a, a)); }
static void axpy(int n, double a, const double *x, double *y) { for (int i = 0; i < n; i++) y[i] += a * x[i]; }
static void scal(int n, double a, double *x) { for (int i = 0; i < n; i++) x[i] *= a; }

static double fun(prob_t *P, const double *w)
{
    double f = 0;
    for (int i = 0; i < P->l; i++) P->z[i] = row_dot(P, i, w);
    for (int i = 0; i < P->n; i++) f += w[i] * w[i];
    f /= 2;
    for (int i = 0; i < P->l; i++) {
        const double d = P->z[i] - P->y[i];
        if (d < -P->p) f += P->C[i] * (d + P->p) * (d + P->p);
        else if (d > P->p) f += P->C[i] * (d - P->p) * (d - P->p);
    }
    return f;
}

static void grad(prob_t *P, const double *w, double *g)
{
    P->sizeI = 0;
    for (int i = 0; i < P->l; i++) {
        const double d = P->z[i] - P->y[i];
        if (d < -P->p) { P->z[P->sizeI] = P->C[i] * (d + P->p); P->I[P->sizeI++] = i; }
        else if (d > P->p) { P->z[P->sizeI] = P->C[i] * (d - P->p); P->I[P->sizeI++] = i; }
    }
    memset(g, 0, sizeof(double) * P->n);
    for (int i = 0; i < P->sizeI; i++) row_axpy(P, P->I[i], P->z[i], g);
    for (int i = 0; i < P->n; i++) g[i] = w[i] + 2 * g[i];
}

static void Hv(prob_t *P, const double *s, double *Hs)
{
    double *wa = malloc(sizeof(double) * (P->sizeI + 1));
    for (int i = 0; i < P->sizeI; i++) wa[i] = P->C[P->I[i]] * row_dot(P, P->I[i], s);
    memset(Hs, 0, sizeof(double) * P->n);
    for (int i = 0; i < P->sizeI; i++) row_axpy(P, P->I[i], wa[i], Hs);
    for (int i = 0; i < P->n; i++) Hs[i] = s[i] + 2 * Hs[i];
    free(wa);
}

static void trcg(prob_t *P, double delta, const double *g, double *s, double *r)
{
    const int n = P->n;
    double *d = malloc(sizeof(double) * n), *Hd = malloc(sizeof(double) * n);
    for (int i = 0; i < n; i++) { s[i] = 0; r[i] = -g[i]; d[i] = r[i]; }
    const double cgtol = 0.1 * nrm2(n, g);
    double rTr = dot(n, r, r);
    while (1) {
        if (nrm2(n, r) <= cgtol) break;
        Hv(P, d, Hd);
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
}

static int tron(prob_t *P, double *w, double eps, int max_iter)
{
    const double eta0 = 1e-4, eta1 = 0.25, eta2 = 0.75, sigma1 = 0.25, sigma2 = 0.5, sigma3 = 4;
    const int n = P->n;
    double *s = malloc(sizeof(double) * n), *r = malloc(sizeof(double) * n), *w_new = malloc(sizeof(double) * n),
           *g = malloc(sizeof(double) * n);
    int search = 1, iter = 1;
    for (int i = 0; i < n; i++) w[i] = 0;
    double f = fun(P, w);
    grad(P, w, g);
    double delta = nrm2(n, g), gnorm1 = delta, gnorm = gnorm1;
    if (gnorm <= eps * gnorm1) search = 0;
    while (iter <= max_iter && search) {
        trcg(P, delta, g, s, r);
        memcpy(w_new, w, sizeof(double) * n);
        axpy(n, 1.0, s, w_new);
        const double gs = dot(n, g, s);
        const double prered = -0.5 * (gs - dot(n, s, r));
        const double fnew = fun(P, w_new);
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
        if (actred > eta0 * prered) {
            iter++;
            memcpy(w, w_new, sizeof(double) * n);
            f = fnew;
            grad(P, w, g);
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

/* X [l0][nx] rows in training order, y [l0], W [l0] sample weights; solver 11, 12 or 13; bias > 0: the bias feature.
 * w_out [nx + (bias > 0)]; steps: coordinate steps of the CD (0 for TRON).  Returns n_iter, or -1 when no row has positive
 * weight. */
int oracle_linsvr_train(const double *X, int l0, int nx, const double *y0, const double *W0, double C, double p, double bias,
                        double tol, int max_iter, int solver, uint32_t seed, int kernel_order, double *w_out, int64_t *steps)
{
    int l = 0;
    for (int i = 0; i < l0; i++) if (W0[i] > 0) l++;
    if (l == 0) return -1;
    double *Xp = malloc(sizeof(double) * (size_t)l * nx), *y = malloc(sizeof(double) * l), *Ci = malloc(sizeof(double) * l);
    for (int i = 0, k = 0; i < l0; i++)
        if (W0[i] > 0) {
            memcpy(Xp + (size_t)k * nx, X + (size_t)i * nx, sizeof(double) * nx);
            y[k] = y0[i];
            Ci[k] = W0[i] * C;
            k++;
        }
    prob_t P;
    P.l = l; P.nx = nx; P.n = nx + (bias > 0 ? 1 : 0); P.X = Xp; P.bias = bias; P.y = y; P.C = Ci; P.p = p;
    P.z = malloc(sizeof(double) * l); P.I = malloc(sizeof(int) * l); P.sizeI = 0;
    oracle_mt_seed(seed);
    int it;
    *steps = 0;
    if (solver == 11) it = tron(&P, w_out, tol, max_iter);
    else it = solve_svr_dual(&P, w_out, solver == 13, tol, max_iter, kernel_order, steps);
    free(Xp); free(y); free(Ci); free(P.z); free(P.I);
    return it;
}

void oracle_mt_draws(uint32_t seed, int k, uint32_t *out)
{
    oracle_mt_seed(seed);
    for (int i = 0; i < k; i++) out[i] = oracle_mt_next();
}
