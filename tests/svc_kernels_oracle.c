/*
 * tests/svc_kernels_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The poly and sigmoid kernels for the C-SVC oracle of oracle/svc_oracle.c, whose solver steps (working-set selection,
 * shrinking, gradient reconstruction, bias) are reused as they are: this file includes it.  What the two kernels add is
 * libsvm's kernel value (scikit-learn svm.cpp Kernel::kernel_poly / kernel_sigmoid and powi) and a float64 diagonal QD
 * that is neither 1 (rbf) nor the squared norm (linear), so the solve entry point below takes the float32 kernel matrix
 * and that diagonal as inputs.  tests/test_oracle_kernels.py pins it against sklearn.svm.SVC.
 *
 * Build: gcc -O2 -ffp-contract=off (no fused multiply-add, as libsvm's x86-64 build).
 */
#include "../oracle/svc_oracle.c"

enum { KERNEL_POLY = 2, KERNEL_SIGMOID = 3 };

/* svm.cpp powi: square and multiply */
static double powi_(double base, int times)
{
    double tmp = base, ret = 1.0;
    for (int t = times; t > 0; t /= 2) {
        if (t % 2 == 1) ret *= tmp;
        tmp = tmp * tmp;
    }
    return ret;
}

static double kernel_of_dot(int kernel, double s, double gamma, int degree, double coef0)
{
    if (kernel == KERNEL_POLY) return powi_(gamma * s + coef0, degree);
    return tanh(gamma * s + coef0);
}

/* S[n][n] = X X^T, one sequential dot product per entry (the summation order of dot_rows in oracle/svc_oracle.c) */
void oracle_gram(const double *X, int n, int d, double *S)
{
    for (int a = 0; a < n; a++)
        for (int b = a; b < n; b++) {
            const double *pa = X + (size_t)a * d, *pb = X + (size_t)b * d;
            double s = 0.0;
            for (int k = 0; k < d; k++) s += pa[k] * pb[k];
            S[(size_t)a * n + b] = S[(size_t)b * n + a] = s;
        }
}

/* K[r][c] = (float)k(x_r, x_c) (unsigned Q, svm.cpp SVC_Q::get_Q) and QD[r] = k(x_r, x_r) in float64 (svm.cpp SVC_Q) */
void oracle_kernel_from_gram(const double *S, int n, int kernel, double gamma, int degree, double coef0, float *K, double *QD)
{
    for (int r = 0; r < n; r++) {
        for (int c = 0; c < n; c++) K[(size_t)r * n + c] = (float)kernel_of_dot(kernel, S[(size_t)r * n + c], gamma, degree, coef0);
        QD[r] = kernel_of_dot(kernel, S[(size_t)r * n + r], gamma, degree, coef0);
    }
}

/*
 * One binary C-SVC sub-problem on a given float32 kernel matrix K[n][ldk] and float64 diagonal QD[n], both indexed by dataset
 * row -- the loop of oracle_svc_solve (svm.cpp:1600-1647 solve_c_svc, :670-944 Solver::Solve) with QD taken from the caller.
 * rows[l]: dataset rows in sub-problem order, the first n_pos labelled +1.  Outputs as oracle_svc_solve.
 */
int oracle_svc_solve_kqd(const float *K, long ldk, const double *QD, const int *rows, int l, int n_pos,
                         double C, double eps, int shrinking, int max_iter,
                         double *coef, double *rho, int *n_iter, double *obj)
{
    qmat_t q; smo_t s;
    memset(&q, 0, sizeof q); memset(&s, 0, sizeof s);
    q.l = l; q.rows = rows; q.Kpre = K; q.ldk = ldk; q.kernel = KERNEL_LINEAR;
    q.y0 = (signed char *)malloc(l);
    q.qrow = (float **)calloc(l, sizeof(float *));
    s.l = s.active = l; s.eps = eps; s.q = &q;
    s.orig = (int *)malloc(sizeof(int) * l); s.y = (signed char *)malloc(l); s.st = (char *)malloc(l);
    s.alpha = (double *)calloc(l, sizeof(double)); s.G = (double *)malloc(sizeof(double) * l);
    s.Gbar = (double *)calloc(l, sizeof(double)); s.QD = (double *)malloc(sizeof(double) * l);
    s.Cv = (double *)malloc(sizeof(double) * l);
    for (int i = 0; i < l; i++) {
        q.y0[i] = s.y[i] = i < n_pos ? +1 : -1;
        s.orig[i] = i; s.Cv[i] = C; s.G[i] = -1.0;
        s.QD[i] = QD[rows[i]];
        set_status(&s, i);
    }

    int iter = 0, timed_out = 0;
    int counter = (l < 1000 ? l : 1000) + 1;
    for (;;) {
        if (max_iter != -1 && iter >= max_iter) { timed_out = 1; break; }
        if (--counter == 0) { counter = l < 1000 ? l : 1000; if (shrinking) shrink(&s); }
        int i, j;
        if (pick_pair(&s, &i, &j)) {
            rebuild_gradient(&s);
            s.active = l;
            if (pick_pair(&s, &i, &j)) break;
            counter = 1;
        }
        iter++;
        const float *Qi = q_row(&q, s.orig[i]), *Qj = q_row(&q, s.orig[j]);
        double Ci = s.Cv[i], Cj = s.Cv[j], oai = s.alpha[i], oaj = s.alpha[j];
        if (s.y[i] != s.y[j]) {
            double quad = s.QD[i] + s.QD[j] + 2 * QP(&s, Qi, j);
            if (quad <= 0) quad = TAU_;
            double delta = (-s.G[i] - s.G[j]) / quad, diff = s.alpha[i] - s.alpha[j];
            s.alpha[i] += delta; s.alpha[j] += delta;
            if (diff > 0) { if (s.alpha[j] < 0) { s.alpha[j] = 0; s.alpha[i] = diff; } }
            else          { if (s.alpha[i] < 0) { s.alpha[i] = 0; s.alpha[j] = -diff; } }
            if (diff > Ci - Cj) { if (s.alpha[i] > Ci) { s.alpha[i] = Ci; s.alpha[j] = Ci - diff; } }
            else                { if (s.alpha[j] > Cj) { s.alpha[j] = Cj; s.alpha[i] = Cj + diff; } }
        } else {
            double quad = s.QD[i] + s.QD[j] - 2 * QP(&s, Qi, j);
            if (quad <= 0) quad = TAU_;
            double delta = (s.G[i] - s.G[j]) / quad, sum = s.alpha[i] + s.alpha[j];
            s.alpha[i] -= delta; s.alpha[j] += delta;
            if (sum > Ci) { if (s.alpha[i] > Ci) { s.alpha[i] = Ci; s.alpha[j] = sum - Ci; } }
            else          { if (s.alpha[j] < 0)  { s.alpha[j] = 0;  s.alpha[i] = sum; } }
            if (sum > Cj) { if (s.alpha[j] > Cj) { s.alpha[j] = Cj; s.alpha[i] = sum - Cj; } }
            else          { if (s.alpha[i] < 0)  { s.alpha[i] = 0;  s.alpha[j] = sum; } }
        }
        double dai = s.alpha[i] - oai, daj = s.alpha[j] - oaj;
        for (int k = 0; k < s.active; k++) s.G[k] += QP(&s, Qi, k) * dai + QP(&s, Qj, k) * daj;
        int ui = s.st[i] == ST_UPPER, uj = s.st[j] == ST_UPPER;
        set_status(&s, i); set_status(&s, j);
        if (ui != (s.st[i] == ST_UPPER)) {
            if (ui) for (int k = 0; k < l; k++) s.Gbar[k] -= Ci * QP(&s, Qi, k);
            else    for (int k = 0; k < l; k++) s.Gbar[k] += Ci * QP(&s, Qi, k);
        }
        if (uj != (s.st[j] == ST_UPPER)) {
            if (uj) for (int k = 0; k < l; k++) s.Gbar[k] -= Cj * QP(&s, Qj, k);
            else    for (int k = 0; k < l; k++) s.Gbar[k] += Cj * QP(&s, Qj, k);
        }
    }
    *rho = bias_term(&s);
    double v = 0;
    for (int i = 0; i < l; i++) v += s.alpha[i] * (s.G[i] + (-1.0));
    *obj = v / 2;
    for (int i = 0; i < l; i++) coef[s.orig[i]] = s.alpha[i] * s.y[i];
    *n_iter = iter;
    for (int i = 0; i < l; i++) free(q.qrow[i]);
    free(q.qrow); free(q.y0);
    free(s.orig); free(s.y); free(s.st); free(s.alpha); free(s.G); free(s.Gbar); free(s.QD); free(s.Cv);
    return timed_out;
}

/* out[t] = sum_k coef_k k(x_trows[t], x_rows[k]) - rho from the Gram S[n][n], float64 kernel values, non-SVs skipped
 * (svm.cpp:2821-2904 svm_predict_values with k_function) */
void oracle_kernel_decision(const double *S, int n, const int *rows, int l, const double *coef, double rho, int kernel,
                            double gamma, int degree, double coef0, const int *trows, int nt, double *out)
{
    for (int t = 0; t < nt; t++) {
        double sum = 0;
        for (int k = 0; k < l; k++) {
            if (coef[k] == 0) continue;
            sum += coef[k] * kernel_of_dot(kernel, S[(size_t)trows[t] * n + rows[k]], gamma, degree, coef0);
        }
        out[t] = sum - rho;
    }
}
