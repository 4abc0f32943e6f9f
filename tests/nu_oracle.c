/*
 * tests/nu_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A plain-C restatement of libsvm's Solver_NU as scikit-learn 1.9 ships it (sklearn/svm/src/libsvm/svm.cpp, "svm.cpp"
 * below): Solver::Solve (l. 666-943) with Solver_NU's select_working_set, be_shrunk, do_shrinking and calculate_rho
 * (l. 1169-1421), reconstruct_gradient (l. 624-664) and swap_index.  The caller (tests/nu_oracle.py) does the set-up of
 * solve_nu_svc (l. 1649) and solve_nu_svr (l. 1798): y, the linear term p, C and the greedy starting alpha.
 *
 * The kernel is given as a float32 matrix K[l][l] (the Qfloat values libsvm computes, before the y_i y_j sign) and the
 * float64 diagonal QD, both in the problem's original order; the solver permutes its own state as libsvm does and reads
 * K through that permutation.  Every operation is libsvm's, in libsvm's order.
 *
 * Build: gcc -O2 -ffp-contract=off (no fused multiply-add, as libsvm's x86-64 build).
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define INF HUGE_VAL
#define TAU 1e-12
enum { LOWER = 0, UPPER = 1, FREE = 2 };

typedef struct {
    int l, active;
    const float *K;
    const double *QD0;
    int *idx;
    signed char *y;
    double *alpha, *G, *Gbar, *p, *C;
    char *st;
    double eps;
    int unshrink;
} Solver;

static double QD(const Solver *s, int i) { return s->QD0[s->idx[i]]; }
/* Q_i[j] = (Qfloat)(y_i y_j k(i, j)): the sign of a float is exact */
static float Q(const Solver *s, int i, int j)
{
    const float k = s->K[(size_t)s->idx[i] * s->l + s->idx[j]];
    return s->y[i] == s->y[j] ? k : -k;
}
static void update_status(Solver *s, int i)
{
    if (s->alpha[i] >= s->C[i]) s->st[i] = UPPER;
    else if (s->alpha[i] <= 0) s->st[i] = LOWER;
    else s->st[i] = FREE;
}
#define SWAPT(T, a, i, j) do { T t_ = (a)[i]; (a)[i] = (a)[j]; (a)[j] = t_; } while (0)
static void swap_index(Solver *s, int i, int j)
{
    SWAPT(int, s->idx, i, j); SWAPT(signed char, s->y, i, j); SWAPT(double, s->G, i, j); SWAPT(char, s->st, i, j);
    SWAPT(double, s->alpha, i, j); SWAPT(double, s->p, i, j); SWAPT(double, s->Gbar, i, j); SWAPT(double, s->C, i, j);
}

/* svm.cpp:624-664 (both of its loop orders add alpha_j Q_ij to G_i in ascending j) */
static void reconstruct_gradient(Solver *s)
{
    if (s->active == s->l) return;
    for (int j = s->active; j < s->l; j++) s->G[j] = s->Gbar[j] + s->p[j];
    for (int i = 0; i < s->active; i++)
        if (s->st[i] == FREE)
            for (int j = s->active; j < s->l; j++) s->G[j] += s->alpha[i] * Q(s, i, j);
}

/* svm.cpp:1189-1299 */
static int select_working_set(Solver *s, int *out_i, int *out_j)
{
    double Gmaxp = -INF, Gmaxp2 = -INF, Gmaxn = -INF, Gmaxn2 = -INF, obj_diff_min = INF;
    int Gmaxp_idx = -1, Gmaxn_idx = -1, Gmin_idx = -1;
    const double *G = s->G;
    for (int t = 0; t < s->active; t++)
        if (s->y[t] == +1) {
            if (s->st[t] != UPPER && -G[t] >= Gmaxp) { Gmaxp = -G[t]; Gmaxp_idx = t; }
        } else {
            if (s->st[t] != LOWER && G[t] >= Gmaxn) { Gmaxn = G[t]; Gmaxn_idx = t; }
        }
    const int ip = Gmaxp_idx, in = Gmaxn_idx;
    for (int j = 0; j < s->active; j++) {
        if (s->y[j] == +1) {
            if (s->st[j] != LOWER) {
                const double grad_diff = Gmaxp + G[j];
                if (G[j] >= Gmaxp2) Gmaxp2 = G[j];
                if (grad_diff > 0) {
                    const double quad_coef = QD(s, ip) + QD(s, j) - 2 * Q(s, ip, j);
                    const double obj_diff = quad_coef > 0 ? -(grad_diff * grad_diff) / quad_coef : -(grad_diff * grad_diff) / TAU;
                    if (obj_diff <= obj_diff_min) { Gmin_idx = j; obj_diff_min = obj_diff; }
                }
            }
        } else {
            if (s->st[j] != UPPER) {
                const double grad_diff = Gmaxn - G[j];
                if (-G[j] >= Gmaxn2) Gmaxn2 = -G[j];
                if (grad_diff > 0) {
                    const double quad_coef = QD(s, in) + QD(s, j) - 2 * Q(s, in, j);
                    const double obj_diff = quad_coef > 0 ? -(grad_diff * grad_diff) / quad_coef : -(grad_diff * grad_diff) / TAU;
                    if (obj_diff <= obj_diff_min) { Gmin_idx = j; obj_diff_min = obj_diff; }
                }
            }
        }
    }
    const double a = Gmaxp + Gmaxp2, b = Gmaxn + Gmaxn2;
    if ((a < b ? b : a) < s->eps || Gmin_idx == -1) return 1;
    *out_i = s->y[Gmin_idx] == +1 ? Gmaxp_idx : Gmaxn_idx;
    *out_j = Gmin_idx;
    return 0;
}

/* svm.cpp:1301-1319 */
static int be_shrunk(const Solver *s, int i, double Gmax1, double Gmax2, double Gmax3, double Gmax4)
{
    if (s->st[i] == UPPER) return s->y[i] == +1 ? -s->G[i] > Gmax1 : -s->G[i] > Gmax4;
    if (s->st[i] == LOWER) return s->y[i] == +1 ? s->G[i] > Gmax2 : s->G[i] > Gmax3;
    return 0;
}

/* svm.cpp:1321-1371 */
static void do_shrinking(Solver *s)
{
    double Gmax1 = -INF, Gmax2 = -INF, Gmax3 = -INF, Gmax4 = -INF;
    for (int i = 0; i < s->active; i++) {
        if (s->st[i] != UPPER) {
            if (s->y[i] == +1) { if (-s->G[i] > Gmax1) Gmax1 = -s->G[i]; }
            else if (-s->G[i] > Gmax4) Gmax4 = -s->G[i];
        }
        if (s->st[i] != LOWER) {
            if (s->y[i] == +1) { if (s->G[i] > Gmax2) Gmax2 = s->G[i]; }
            else if (s->G[i] > Gmax3) Gmax3 = s->G[i];
        }
    }
    const double a = Gmax1 + Gmax2, b = Gmax3 + Gmax4;
    if (!s->unshrink && (a < b ? b : a) <= s->eps * 10) {
        s->unshrink = 1;
        reconstruct_gradient(s);
        s->active = s->l;
    }
    for (int i = 0; i < s->active; i++)
        if (be_shrunk(s, i, Gmax1, Gmax2, Gmax3, Gmax4)) {
            s->active--;
            while (s->active > i) {
                if (!be_shrunk(s, s->active, Gmax1, Gmax2, Gmax3, Gmax4)) { swap_index(s, i, s->active); break; }
                s->active--;
            }
        }
}

/* svm.cpp:1373-1421 */
static double calculate_rho(const Solver *s, double *r_out)
{
    int nf1 = 0, nf2 = 0;
    double ub1 = INF, ub2 = INF, lb1 = -INF, lb2 = -INF, sf1 = 0, sf2 = 0;
    for (int i = 0; i < s->active; i++) {
        const double g = s->G[i];
        if (s->y[i] == +1) {
            if (s->st[i] == UPPER) lb1 = lb1 < g ? g : lb1;
            else if (s->st[i] == LOWER) ub1 = g < ub1 ? g : ub1;
            else { ++nf1; sf1 += g; }
        } else {
            if (s->st[i] == UPPER) lb2 = lb2 < g ? g : lb2;
            else if (s->st[i] == LOWER) ub2 = g < ub2 ? g : ub2;
            else { ++nf2; sf2 += g; }
        }
    }
    const double r1 = nf1 > 0 ? sf1 / nf1 : (ub1 + lb1) / 2;
    const double r2 = nf2 > 0 ? sf2 / nf2 : (ub2 + lb2) / 2;
    *r_out = (r1 + r2) / 2;
    return (r1 - r2) / 2;
}

/*
 * One Solver_NU solve.  K [l][l] float32, QD [l], y [l] (+1 / -1), p [l], C [l], alpha [l] (in: the starting point, out:
 * the solution, by original position).  rebuild_at_stop != 0 reconstructs the gradient of the shrunk variables before rho
 * at a max_iter stop (a variant kept for the test that shows which of the two scikit-learn does).  Returns n_iter;
 * rho, r and timed_out out.
 */
int oracle_nu_solve(const float *K, const double *QD0, const signed char *y_, const double *p_, const double *C_, double *alpha_,
                    int l, double eps, int shrinking, int max_iter, int rebuild_at_stop, double *rho, double *r, int *timed_out)
{
    Solver s;
    memset(&s, 0, sizeof s);
    s.l = l; s.K = K; s.QD0 = QD0; s.eps = eps; s.active = l;
    s.idx = malloc(sizeof(int) * l); s.y = malloc(l); s.st = malloc(l);
    s.alpha = malloc(sizeof(double) * l); s.G = malloc(sizeof(double) * l); s.Gbar = malloc(sizeof(double) * l);
    s.p = malloc(sizeof(double) * l); s.C = malloc(sizeof(double) * l);
    for (int i = 0; i < l; i++) {
        s.idx[i] = i; s.y[i] = y_[i]; s.alpha[i] = alpha_[i]; s.p[i] = p_[i]; s.C[i] = C_[i];
        update_status(&s, i);
    }
    for (int i = 0; i < l; i++) { s.G[i] = s.p[i]; s.Gbar[i] = 0; }
    for (int i = 0; i < l; i++)
        if (s.st[i] != LOWER) {
            const double ai = s.alpha[i];
            for (int j = 0; j < l; j++) s.G[j] += ai * Q(&s, i, j);
            if (s.st[i] == UPPER)
                for (int j = 0; j < l; j++) s.Gbar[j] += s.C[i] * Q(&s, i, j);
        }
    int iter = 0, counter = (l < 1000 ? l : 1000) + 1;
    *timed_out = 0;
    for (;;) {
        if (max_iter != -1 && iter >= max_iter) { *timed_out = 1; break; }
        if (--counter == 0) {
            counter = l < 1000 ? l : 1000;
            if (shrinking) do_shrinking(&s);
        }
        int i, j;
        if (select_working_set(&s, &i, &j) != 0) {
            reconstruct_gradient(&s);
            s.active = l;
            if (select_working_set(&s, &i, &j) != 0) break;
            counter = 1;
        }
        ++iter;
        const double C_i = s.C[i], C_j = s.C[j];
        const double old_ai = s.alpha[i], old_aj = s.alpha[j];
        double *alpha = s.alpha, *G = s.G;
        if (s.y[i] != s.y[j]) {                                   /* never taken by Solver_NU: i and j share a sign */
            double quad_coef = QD(&s, i) + QD(&s, j) + 2 * Q(&s, i, j);
            if (quad_coef <= 0) quad_coef = TAU;
            const double delta = (-G[i] - G[j]) / quad_coef, diff = alpha[i] - alpha[j];
            alpha[i] += delta; alpha[j] += delta;
            if (diff > 0) { if (alpha[j] < 0) { alpha[j] = 0; alpha[i] = diff; } }
            else { if (alpha[i] < 0) { alpha[i] = 0; alpha[j] = -diff; } }
            if (diff > C_i - C_j) { if (alpha[i] > C_i) { alpha[i] = C_i; alpha[j] = C_i - diff; } }
            else { if (alpha[j] > C_j) { alpha[j] = C_j; alpha[i] = C_j + diff; } }
        } else {
            double quad_coef = QD(&s, i) + QD(&s, j) - 2 * Q(&s, i, j);
            if (quad_coef <= 0) quad_coef = TAU;
            const double delta = (G[i] - G[j]) / quad_coef, sum = alpha[i] + alpha[j];
            alpha[i] -= delta; alpha[j] += delta;
            if (sum > C_i) { if (alpha[i] > C_i) { alpha[i] = C_i; alpha[j] = sum - C_i; } }
            else { if (alpha[j] < 0) { alpha[j] = 0; alpha[i] = sum; } }
            if (sum > C_j) { if (alpha[j] > C_j) { alpha[j] = C_j; alpha[i] = sum - C_j; } }
            else { if (alpha[i] < 0) { alpha[i] = 0; alpha[j] = sum; } }
        }
        const double dai = alpha[i] - old_ai, daj = alpha[j] - old_aj;
        for (int k = 0; k < s.active; k++) G[k] += Q(&s, i, k) * dai + Q(&s, j, k) * daj;
        const int ui = s.st[i] == UPPER, uj = s.st[j] == UPPER;
        update_status(&s, i);
        update_status(&s, j);
        if (ui != (s.st[i] == UPPER)) {
            if (ui) for (int k = 0; k < l; k++) s.Gbar[k] -= C_i * Q(&s, i, k);
            else for (int k = 0; k < l; k++) s.Gbar[k] += C_i * Q(&s, i, k);
        }
        if (uj != (s.st[j] == UPPER)) {
            if (uj) for (int k = 0; k < l; k++) s.Gbar[k] -= C_j * Q(&s, j, k);
            else for (int k = 0; k < l; k++) s.Gbar[k] += C_j * Q(&s, j, k);
        }
    }
    if (*timed_out && rebuild_at_stop) { reconstruct_gradient(&s); s.active = l; }
    *rho = calculate_rho(&s, r);
    for (int i = 0; i < l; i++) alpha_[s.idx[i]] = s.alpha[i];
    free(s.idx); free(s.y); free(s.st); free(s.alpha); free(s.G); free(s.Gbar); free(s.p); free(s.C);
    return iter;
}
