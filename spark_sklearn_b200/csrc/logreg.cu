// logreg.cu -- batched binary L2 logistic regression, one L-BFGS-B run per (candidate C, fold) column.
//
// Replaces (reference base_search.py:83-87 -> sklearn _fit_and_score -> LogisticRegression.fit/score):
//   sklearn/linear_model/_logistic.py:580-604   scipy.optimize.minimize(method="L-BFGS-B", maxcor=10, maxls=50,
//                                               gtol=tol, ftol=64*eps, maxiter=max_iter)
//   sklearn/linear_model/_linear_loss.py:47-64  f(w,b) = (1/n) sum_i [log(1+e^{z_i}) - y_i z_i] + (l2/2)|w|^2,
//                                               z = Xw + b, l2 = 1/(C n), intercept not penalised
//   sklearn/linear_model/_base.py:416           predict: z > 0 -> classes_[1]
//
// scipy's L-BFGS-B stops after 5-9 iterations at gtol=1e-4, i.e. NOT at the optimum, so "solve exactly" is not
// "match" (SURVEY.md H4: a fully converged fit moves mean_test_score by up to 1e-4).  This file restates the
// algorithm for the unconstrained case op for op: steepest descent first step with stp = 1/|d|, then
// d = -H g by the two-loop recursion with H0 = I/theta (theta = y'y/s'y, mathematically the compact-form
// subspace step of L-BFGS-B when no bound is active), the More'-Thuente line search dcsrch/dcstep (ftol 1e-3,
// gtol 0.9, xtol 0.1), the curvature-skip rule, and the stopping tests in scipy's order
// (projected-gradient max-norm <= gtol, relative f-reduction <= ftol, iteration cap).
//
// Batching: every function/gradient evaluation of ALL columns is two tensor-core contractions (gemm_tc.cu):
//   Z^T[col][row] = W[col][:] . Xa[row][:]      (Xa = [X | 1], K = features)
//   G[col][feat]  = R[col][:] . Xa^T[feat][:]   (R = masked (sigmoid(z) - y)/n_train, K = rows)
// with a fused element-wise pass between them (loss, residual, fold mask, hi/lo split of R); the per-column
// optimiser state machine runs one warp per column between evaluations.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

constexpr int MCOR = 10;               // maxcor
constexpr int GRAD_KCHUNK = 256;       // accumulation-chain bound of the gradient contraction (heavily cancelled sum)
constexpr double LS_FTOL = 1e-3, LS_GTOL = 0.9, LS_XTOL = 0.1, STPMX = 1e10;
constexpr double EPSMCH = 2.220446049250313e-16;
enum { T_FG_START = 0, T_FG_LNSRCH = 1, T_DONE = 2 };
enum { R_PGTOL = 1, R_FTOL = 2, R_MAXITER = 3, R_ABNORMAL = 4, R_MAXFUN = 5 };

struct LbScalars {                     // per column
    int task, iter, nfev, col, head, iback, reason, stage, brackt, fresh;
    double f, fold, theta, stp, dnorm, gd, gdold, sbgnrm;
    double ginit, gtest, gx, gy, finit, fx, fy, stx, sty, stmin, stmax, width, width1;
    double l2, loss_acc;               // l2_reg_strength; loss accumulator written by the element-wise pass
    double rho[MCOR];
};

// ---------------------------------------------------------------- MINPACK-2 dcstep / dcsrch ------------
__device__ void dcstep(double &stx, double &fx, double &dx, double &sty, double &fy, double &dy, double &stp,
                       double fp, double dp, int &brackt, double stpmin, double stpmax)
{
    const double sgnd = dp * (dx / fabs(dx));
    double stpf, stpc, stpq, theta, s, gamma, p, q, r;
    if (fp > fx) {
        theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
        s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
        gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
        if (stp < stx) gamma = -gamma;
        p = (gamma - dx) + theta; q = ((gamma - dx) + gamma) + dp; r = p / q;
        stpc = stx + r * (stp - stx);
        stpq = stx + ((dx / ((fx - fp) / (stp - stx) + dx)) / 2.0) * (stp - stx);
        stpf = fabs(stpc - stx) < fabs(stpq - stx) ? stpc : stpc + (stpq - stpc) / 2.0;
        brackt = 1;
    } else if (sgnd < 0.0) {
        theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
        s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
        gamma = s * sqrt((theta / s) * (theta / s) - (dx / s) * (dp / s));
        if (stp > stx) gamma = -gamma;
        p = (gamma - dp) + theta; q = ((gamma - dp) + gamma) + dx; r = p / q;
        stpc = stp + r * (stx - stp);
        stpq = stp + (dp / (dp - dx)) * (stx - stp);
        stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
        brackt = 1;
    } else if (fabs(dp) < fabs(dx)) {
        theta = 3.0 * (fx - fp) / (stp - stx) + dx + dp;
        s = fmax(fabs(theta), fmax(fabs(dx), fabs(dp)));
        gamma = s * sqrt(fmax(0.0, (theta / s) * (theta / s) - (dx / s) * (dp / s)));
        if (stp > stx) gamma = -gamma;
        p = (gamma - dp) + theta; q = (gamma + (dx - dp)) + gamma; r = p / q;
        if (r < 0.0 && gamma != 0.0) stpc = stp + r * (stx - stp);
        else stpc = stp > stx ? stpmax : stpmin;
        stpq = stp + (dp / (dp - dx)) * (stx - stp);
        if (brackt) {
            stpf = fabs(stpc - stp) < fabs(stpq - stp) ? stpc : stpq;
            if (stp > stx) stpf = fmin(stp + 0.66 * (sty - stp), stpf);
            else stpf = fmax(stp + 0.66 * (sty - stp), stpf);
        } else {
            stpf = fabs(stpc - stp) > fabs(stpq - stp) ? stpc : stpq;
            stpf = fmin(stpmax, stpf); stpf = fmax(stpmin, stpf);
        }
    } else {
        if (brackt) {
            theta = 3.0 * (fp - fy) / (sty - stp) + dy + dp;
            s = fmax(fabs(theta), fmax(fabs(dy), fabs(dp)));
            gamma = s * sqrt((theta / s) * (theta / s) - (dy / s) * (dp / s));
            if (stp > sty) gamma = -gamma;
            p = (gamma - dp) + theta; q = ((gamma - dp) + gamma) + dy; r = p / q;
            stpc = stp + r * (sty - stp);
            stpf = stpc;
        } else stpf = stp > stx ? stpmax : stpmin;
    }
    if (fp > fx) { sty = stp; fy = fp; dy = dp; }
    else {
        if (sgnd < 0.0) { sty = stx; fy = fx; dy = dx; }
        stx = stp; fx = fp; dx = dp;
    }
    stp = stpf;
}

// returns 0 = evaluate f,g at the new stp; 1 = converged; 2 = warning (line search ends at the current stp)
__device__ int dcsrch(LbScalars &S, double f, double g, bool start)
{
    const double stpmin = 0.0, stpmax = STPMX, xtrapl = 1.1, xtrapu = 4.0;
    if (start) {
        S.brackt = 0; S.stage = 1; S.finit = f; S.ginit = g; S.gtest = LS_FTOL * g;
        S.width = stpmax - stpmin; S.width1 = S.width / 0.5;
        S.stx = 0; S.fx = f; S.gx = g; S.sty = 0; S.fy = f; S.gy = g;
        S.stmin = 0; S.stmax = S.stp + xtrapu * S.stp;
        return 0;
    }
    const double ftest = S.finit + S.stp * S.gtest;
    if (S.stage == 1 && f <= ftest && g >= 0.0) S.stage = 2;
    int ret = 0;
    if (S.brackt && (S.stp <= S.stmin || S.stp >= S.stmax)) ret = 2;
    if (S.brackt && S.stmax - S.stmin <= LS_XTOL * S.stmax) ret = 2;
    if (S.stp == stpmax && f <= ftest && g <= S.gtest) ret = 2;
    if (S.stp == stpmin && (f > ftest || g >= S.gtest)) ret = 2;
    if (f <= ftest && fabs(g) <= LS_GTOL * (-S.ginit)) ret = 1;
    if (ret) return ret;
    if (S.stage == 1 && f <= S.fx && f > ftest) {
        double fm = f - S.stp * S.gtest, fxm = S.fx - S.stx * S.gtest, fym = S.fy - S.sty * S.gtest;
        double gm = g - S.gtest, gxm = S.gx - S.gtest, gym = S.gy - S.gtest;
        dcstep(S.stx, fxm, gxm, S.sty, fym, gym, S.stp, fm, gm, S.brackt, S.stmin, S.stmax);
        S.fx = fxm + S.stx * S.gtest; S.fy = fym + S.sty * S.gtest; S.gx = gxm + S.gtest; S.gy = gym + S.gtest;
    } else {
        dcstep(S.stx, S.fx, S.gx, S.sty, S.fy, S.gy, S.stp, f, g, S.brackt, S.stmin, S.stmax);
    }
    if (S.brackt) {
        if (fabs(S.sty - S.stx) >= 0.66 * S.width1) S.stp = S.stx + 0.5 * (S.sty - S.stx);
        S.width1 = S.width; S.width = fabs(S.sty - S.stx);
    }
    if (S.brackt) { S.stmin = fmin(S.stx, S.sty); S.stmax = fmax(S.stx, S.sty); }
    else { S.stmin = S.stp + xtrapl * (S.stp - S.stx); S.stmax = S.stp + xtrapu * (S.stp - S.stx); }
    S.stp = fmax(S.stp, stpmin); S.stp = fmin(S.stp, stpmax);
    if ((S.brackt && (S.stp <= S.stmin || S.stp >= S.stmax)) || (S.brackt && S.stmax - S.stmin <= LS_XTOL * S.stmax)) S.stp = S.stx;
    return 0;
}

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int m = 16; m; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    return v;
}
__device__ __forceinline__ double warp_max(double v)
{
#pragma unroll
    for (int m = 16; m; m >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, m));
    return v;
}

// vectors of a column live at V + col * VSTRIDE: x, g, t (x at line-search start), r (g at line-search start), d,
// then WS[MCOR][nvp], WY[MCOR][nvp]; nvp = padded number of variables
struct LbLayout { int nv, nvp; };
__device__ __forceinline__ double *vec(double *V, int which, int nvp) { return V + (size_t)which * nvp; }

// One warp per fit: consume the f/g just evaluated at the trial point and advance the optimiser until the next
// trial point is ready (or the fit is done).  Writes the float32 trial weights (hi/lo split) for the next GEMM.
// The variables of a fit are n_class blocks of `per` entries (the first nv of each block are real: features, then the
// intercept; binary problems have one block), i.e. n_class consecutive rows of the weight / gradient matrices of the GEMMs.
#define LB_FOR(j) for (int j = lane; j < nvp; j += 32) if ((j % per) < nv)
__global__ void lbfgs_advance_kernel(LbScalars *__restrict__ Sc, double *__restrict__ Vall, const float *__restrict__ Gmat,
                                     int64_t ldg, int ncol, int nv, int per, int n_class, int n_feat_pen, double pgtol, double factr_eps,
                                     int maxiter, int maxfun, int maxls, float *__restrict__ Wh, float *__restrict__ Wl, int64_t ldw,
                                     int *__restrict__ n_open)
{
    const int nvp = per * n_class;                                          // length of a fit's vectors
    const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (c >= ncol) return;
    LbScalars S = Sc[c];
    if (S.task == T_DONE) return;
    double *V = Vall + (size_t)c * (5 + 2 * MCOR) * nvp;
    double *x = vec(V, 0, nvp), *g = vec(V, 1, nvp), *t = vec(V, 2, nvp), *r = vec(V, 3, nvp), *d = vec(V, 4, nvp);
    double *WS = vec(V, 5, nvp), *WY = vec(V, 5 + MCOR, nvp);

    // ---- finish f and g at the trial point: f = loss/n + (l2/2)|w|^2, g = G + l2 w (intercept not penalised) ----
    double ww = 0;
    LB_FOR(j) {
        const double w = x[j];
        double gj = (double)Gmat[(size_t)c * ldg + j];
        if ((j % per) < n_feat_pen) { gj += S.l2 * w; ww += w * w; }
        g[j] = gj;
    }
    ww = warp_sum(ww);
    const double f = S.loss_acc + 0.5 * S.l2 * ww;
    S.nfev++;

    bool need_direction = false;
    if (S.task == T_FG_START) {
        S.f = f;
        double m = 0;
        LB_FOR(j) m = fmax(m, fabs(g[j]));
        S.sbgnrm = warp_max(m);
        if (S.sbgnrm <= pgtol) { S.task = T_DONE; S.reason = R_PGTOL; }
        else need_direction = true;
    } else {
        // ---- inside the line search (lnsrlb): gd = g.d at the trial point ----
        double gd = 0;
        LB_FOR(j) gd += g[j] * d[j];
        gd = warp_sum(gd);
        S.gd = gd;
        const int ret = dcsrch(S, f, gd, false);
        if (ret == 0) {
            S.iback++;
            if (S.iback >= maxls) {
                // too many backtracks: restore the point; refresh the memory or give up (lnsrlb info = -3... handling)
                LB_FOR(j) { x[j] = t[j]; g[j] = r[j]; }
                S.f = S.fold;
                if (S.col == 0) { S.task = T_DONE; S.reason = R_ABNORMAL; }
                else { S.col = 0; S.head = 0; S.theta = 1.0; S.fresh = 1; need_direction = true; }
            } else {
                LB_FOR(j) x[j] = (S.stp == 1.0) ? t[j] + d[j] : S.stp * d[j] + t[j];
            }
        } else {
            // ---- line search finished: new iterate ----
            S.f = f;
            S.iter++;
            double m = 0;
            LB_FOR(j) m = fmax(m, fabs(g[j]));
            S.sbgnrm = warp_max(m);
            if (S.iter >= maxiter) { S.task = T_DONE; S.reason = R_MAXITER; }
            else if (S.nfev > maxfun) { S.task = T_DONE; S.reason = R_MAXFUN; }
            else if (S.sbgnrm <= pgtol) { S.task = T_DONE; S.reason = R_PGTOL; }
            else {
                const double ddum = fmax(fmax(fabs(S.fold), fabs(S.f)), 1.0);
                if (S.fold - S.f <= factr_eps * ddum) { S.task = T_DONE; S.reason = R_FTOL; }
                else {
                    // ---- BFGS pair: y = g - g_old, s = stp * d (mainlb after label 777) ----
                    double rr = 0, dr, ddum2;
                    LB_FOR(j) { const double yj = g[j] - r[j]; r[j] = yj; rr += yj * yj; }
                    rr = warp_sum(rr);
                    if (S.stp == 1.0) { dr = S.gd - S.gdold; ddum2 = -S.gdold; }
                    else {
                        dr = (S.gd - S.gdold) * S.stp; ddum2 = -S.gdold * S.stp;
                        LB_FOR(j) d[j] *= S.stp;
                    }
                    if (!(dr <= EPSMCH * ddum2)) {
                        const int slot = S.col < MCOR ? (S.head + S.col) % MCOR : S.head;
                        LB_FOR(j) { WS[(size_t)slot * nvp + j] = d[j]; WY[(size_t)slot * nvp + j] = r[j]; }
                        S.rho[slot] = 1.0 / dr;
                        if (S.col < MCOR) S.col++; else S.head = (S.head + 1) % MCOR;
                        S.theta = rr / dr;
                    }
                    need_direction = true;
                }
            }
        }
    }

    if (need_direction && S.task != T_DONE) {
        // ---- direction d = -H g: two-loop recursion, H0 = I/theta (== L-BFGS-B subspace step with no active bound) ----
        __syncwarp();
        double alpha_i[MCOR];
        LB_FOR(j) d[j] = g[j];                      // q
        for (int k = S.col - 1; k >= 0; k--) {
            const int slot = (S.head + k) % MCOR;
            double a = 0;
            LB_FOR(j) a += WS[(size_t)slot * nvp + j] * d[j];
            a = warp_sum(a) * S.rho[slot];
            alpha_i[k] = a;
            LB_FOR(j) d[j] -= a * WY[(size_t)slot * nvp + j];
        }
        const double h0 = 1.0 / S.theta;
        LB_FOR(j) d[j] *= h0;
        for (int k = 0; k < S.col; k++) {
            const int slot = (S.head + k) % MCOR;
            double b = 0;
            LB_FOR(j) b += WY[(size_t)slot * nvp + j] * d[j];
            b = warp_sum(b) * S.rho[slot];
            const double cf = alpha_i[k] - b;
            LB_FOR(j) d[j] += cf * WS[(size_t)slot * nvp + j];
        }
        double dtd = 0, gd = 0;
        LB_FOR(j) { const double dj = -d[j]; d[j] = dj; dtd += dj * dj; gd += g[j] * dj; }
        dtd = warp_sum(dtd); gd = warp_sum(gd);
        if (gd >= 0.0) {                                                    // not a descent direction: refresh the memory
            if (S.col == 0) { S.task = T_DONE; S.reason = R_ABNORMAL; }
            else {
                S.col = 0; S.head = 0; S.theta = 1.0;
                dtd = 0; gd = 0;
                LB_FOR(j) { const double dj = -g[j]; d[j] = dj; dtd += dj * dj; gd += g[j] * dj; }
                dtd = warp_sum(dtd); gd = warp_sum(gd);
            }
        }
        if (S.task != T_DONE) {
            // ---- start the line search (lnsrlb): stp = 1/|d| on the very first iteration, else 1 ----
            S.dnorm = sqrt(dtd);
            S.stp = S.iter == 0 ? fmin(1.0 / S.dnorm, STPMX) : 1.0;
            S.fold = S.f; S.iback = 0; S.gd = gd; S.gdold = gd;
            LB_FOR(j) { t[j] = x[j]; r[j] = g[j]; }
            dcsrch(S, S.f, gd, true);
            LB_FOR(j) x[j] = (S.stp == 1.0) ? t[j] + d[j] : S.stp * d[j] + t[j];
            S.task = T_FG_LNSRCH;
        }
    }
    __syncwarp();
    // ---- publish: scalars, and the float32 trial point for the next evaluation ----
    if (S.task != T_DONE) {
        for (int j = lane; j < nvp; j += 32) {
            const float v = (j % per) < nv ? (float)x[j] : 0.f;
            const float hh = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
            Wh[(size_t)c * ldw + j] = hh; Wl[(size_t)c * ldw + j] = v - hh;
        }
        if (lane == 0) atomicAdd(n_open, 1);
    }
    S.loss_acc = 0.0;
    if (lane == 0) Sc[c] = S;
}

// write float32 weights of every column (final iterate) for the scoring GEMM
__global__ void lbfgs_export_kernel(const double *__restrict__ Vall, int ncol, int nv, int per, int n_class, float *__restrict__ Wh,
                                    float *__restrict__ Wl, int64_t ldw)
{
    const int c = blockIdx.x, nvp = per * n_class;
    const double *x = Vall + (size_t)c * (5 + 2 * MCOR) * nvp;
    for (int j = threadIdx.x; j < nvp; j += blockDim.x) {
        const float v = (j % per) < nv ? (float)x[j] : 0.f;
        const float hh = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
        Wh[(size_t)c * ldw + j] = hh; Wl[(size_t)c * ldw + j] = v - hh;
    }
}

// Element-wise pass over Z^T [ncol][ldz]: loss, masked residual (hi/lo split), per-column loss sum.
// column c trains on rows whose fold id != fold_of_col[c] (or on all rows when fold_of_col[c] < 0).
__global__ void logistic_residual_kernel(const float *__restrict__ Zt, int64_t ldz, int n, const int *__restrict__ y,
                                         SplitMasks sm, const int *__restrict__ fold_of_col,
                                         const double *__restrict__ inv_ntrain, const float *__restrict__ cw /* [ncol][2] class weights or null */,
                                         const float *__restrict__ sw /* [n] sample weights or null */,
                                         LbScalars *__restrict__ Sc, float *__restrict__ Rh, float *__restrict__ Rl)
{
    const int c = blockIdx.y;
    if (Sc[c].task == T_DONE) return;
    const int fc = fold_of_col[c];
    const float invn = (float)inv_ntrain[c];
    double acc = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const size_t idx = (size_t)c * ldz + i;
        float rres = 0.f;
        if (split_train(sm, i, fc)) {
            const float z = Zt[idx];
            const float yi = (float)y[i];
            // half binomial loss log(1+e^z) - y z, evaluated the numerically stable way
            const float lz = z > 0.f ? z + log1pf(expf(-z)) : log1pf(expf(z));
            const float p = 1.f / (1.f + expf(-z));
            if (cw || sw) {                              // sample_weight (x class_weight_[y]) multiplies the pointwise loss and gradient
                const float wi = (sw ? sw[i] : 1.f) * (cw ? cw[c * 2 + y[i]] : 1.f);   // (_logistic.py: sample_weight *= class_weight_[y]; _loss: loss_out *= sample_weight)
                acc += (double)(wi * (lz - yi * z));
                rres = (wi * (p - yi)) * invn;
            } else {
                acc += (double)(lz - yi * z);
                rres = (p - yi) * invn;
            }
        }
        const float hh = __uint_as_float(__float_as_uint(rres) & 0xffffe000u);
        Rh[idx] = hh; Rl[idx] = rres - hh;
    }
    __shared__ double sh[8];
#pragma unroll
    for (int m = 16; m; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sh[w];
        atomicAdd(&Sc[c].loss_acc, s * inv_ntrain[c]);
    }
}

// accuracy counts: z > 0 -> class 1
__global__ void logistic_count_kernel(const float *__restrict__ Zt, int64_t ldz, int n, const int *__restrict__ y,
                                      SplitMasks sm, const int *__restrict__ fold_of_col, int *__restrict__ counts)
{
    const int c = blockIdx.y, fc = fold_of_col[c];
    int cte = 0, nte = 0, ctr = 0, ntr = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int pred = Zt[(size_t)c * ldz + i] > 0.f ? 1 : 0;
        const bool ok = pred == y[i];
        if (split_test(sm, i, fc)) { nte++; cte += ok; }
        if (split_train(sm, i, fc)) { ntr++; ctr += ok; }
    }
#pragma unroll
    for (int m = 16; m; m >>= 1) {
        cte += __shfl_xor_sync(0xffffffffu, cte, m); nte += __shfl_xor_sync(0xffffffffu, nte, m);
        ctr += __shfl_xor_sync(0xffffffffu, ctr, m); ntr += __shfl_xor_sync(0xffffffffu, ntr, m);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&counts[c * 4 + 0], cte); atomicAdd(&counts[c * 4 + 1], nte);
        atomicAdd(&counts[c * 4 + 2], ctr); atomicAdd(&counts[c * 4 + 3], ntr);
    }
}

// per-class counts for the count-based scorers: counts[col][split (0 test, 1 train)][class (0, 1)][3 = support, tp, predicted]
__global__ void logistic_classes_kernel(const float *__restrict__ Zt, int64_t ldz, int n, const int *__restrict__ y,
                                        SplitMasks sm, const int *__restrict__ fold_of_col, int *__restrict__ counts)
{
    __shared__ int sh[12];
    if (threadIdx.x < 12) sh[threadIdx.x] = 0;
    __syncthreads();
    const int c = blockIdx.y, fc = fold_of_col[c];
    int loc[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int pred = Zt[(size_t)c * ldz + i] > 0.f ? 1 : 0, yc = y[i];
        const int sp = split_test(sm, i, fc) ? 0 : (split_train(sm, i, fc) ? 1 : 2);     // 2: in neither set
#pragma unroll
        for (int q = 0; q < 4; q++) {                                   // (split, class) = q
            const int qs = q >> 1, qc = q & 1;
            loc[q * 3 + 0] += (sp == qs && yc == qc);
            loc[q * 3 + 1] += (sp == qs && yc == qc && pred == qc);
            loc[q * 3 + 2] += (sp == qs && pred == qc);
        }
    }
#pragma unroll
    for (int e = 0; e < 12; e++) {
#pragma unroll
        for (int m = 16; m; m >>= 1) loc[e] += __shfl_xor_sync(0xffffffffu, loc[e], m);
        if ((threadIdx.x & 31) == 0 && loc[e]) atomicAdd(&sh[e], loc[e]);
    }
    __syncthreads();
    if (threadIdx.x < 12 && sh[threadIdx.x]) atomicAdd(&counts[(size_t)c * 12 + threadIdx.x], sh[threadIdx.x]);
}

// Multinomial counterpart of logistic_residual_kernel (n_class >= 3: sklearn/_loss/_loss.pyx closs_grad_half_multinomial --
// loss_i = logsumexp(z_i) - z_i[y_i], gradient softmax(z_i) - onehot(y_i)).  A fit owns n_class consecutive rows of Z^T / R.
__global__ void multinomial_residual_kernel(const float *__restrict__ Zt, int64_t ldz, int n, int K, const int *__restrict__ y,
                                            SplitMasks sm, const int *__restrict__ fold_of_col,
                                            const double *__restrict__ inv_ntrain, const float *__restrict__ cw /* [nfit][K] or null */,
                                            const float *__restrict__ sw /* [n] sample weights or null */,
                                            LbScalars *__restrict__ Sc, float *__restrict__ Rh, float *__restrict__ Rl)
{
    const int f = blockIdx.y;
    if (Sc[f].task == T_DONE) return;
    const int fc = fold_of_col[f];
    const float invn = (float)inv_ntrain[f];
    double acc = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const size_t base = (size_t)f * K * ldz + i;
        if (split_train(sm, i, fc)) {
            float mx = -INFINITY;
            for (int k = 0; k < K; k++) mx = fmaxf(mx, Zt[base + (size_t)k * ldz]);
            float se = 0.f;
            for (int k = 0; k < K; k++) se += expf(Zt[base + (size_t)k * ldz] - mx);
            const int yi = y[i];
            const float wi = (sw ? sw[i] : 1.f) * (cw ? cw[(size_t)f * K + yi] : 1.f);
            acc += (double)(wi * (logf(se) + mx - Zt[base + (size_t)yi * ldz]));
            const float inv_se = 1.f / se;
            for (int k = 0; k < K; k++) {
                const float p = expf(Zt[base + (size_t)k * ldz] - mx) * inv_se;
                const float rres = (wi * (p - (k == yi ? 1.f : 0.f))) * invn;
                const float hh = __uint_as_float(__float_as_uint(rres) & 0xffffe000u);
                Rh[base + (size_t)k * ldz] = hh; Rl[base + (size_t)k * ldz] = rres - hh;
            }
        } else {
            for (int k = 0; k < K; k++) { Rh[base + (size_t)k * ldz] = 0.f; Rl[base + (size_t)k * ldz] = 0.f; }
        }
    }
    __shared__ double sh[8];
#pragma unroll
    for (int m = 16; m; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sh[w];
        atomicAdd(&Sc[f].loss_acc, s * inv_ntrain[f]);
    }
}

// Multinomial predictions (first arg-max of the n_class decision values, like np.argmax in LinearClassifierMixin.predict):
// accuracy counts [nfit][4] and, when ccounts != null, the per-class counts [nfit][2 splits][K][3] of the count-based scorers
__global__ void multinomial_count_kernel(const float *__restrict__ Zt, int64_t ldz, int n, int K, const int *__restrict__ y,
                                         SplitMasks sm, const int *__restrict__ fold_of_col, int *__restrict__ counts,
                                         int *__restrict__ ccounts)
{
    extern __shared__ int shc[];                                         // [2][K][3]
    const int f = blockIdx.y, fc = fold_of_col[f];
    if (ccounts) {
        for (int e = threadIdx.x; e < 6 * K; e += blockDim.x) shc[e] = 0;
        __syncthreads();
    }
    int cte = 0, nte = 0, ctr = 0, ntr = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const size_t base = (size_t)f * K * ldz + i;
        int pred = 0;
        float best = Zt[base];
        for (int k = 1; k < K; k++) { const float z = Zt[base + (size_t)k * ldz]; if (z > best) { best = z; pred = k; } }
        const int yc = y[i];
        const bool ok = pred == yc;
        const int sp = split_test(sm, i, fc) ? 0 : (split_train(sm, i, fc) ? 1 : 2);
        if (sp == 0) { nte++; cte += ok; }
        if (sp == 1) { ntr++; ctr += ok; }
        if (ccounts && sp < 2) {
            atomicAdd(&shc[(sp * K + yc) * 3 + 0], 1);
            if (ok) atomicAdd(&shc[(sp * K + yc) * 3 + 1], 1);
            atomicAdd(&shc[(sp * K + pred) * 3 + 2], 1);
        }
    }
#pragma unroll
    for (int m = 16; m; m >>= 1) {
        cte += __shfl_xor_sync(0xffffffffu, cte, m); nte += __shfl_xor_sync(0xffffffffu, nte, m);
        ctr += __shfl_xor_sync(0xffffffffu, ctr, m); ntr += __shfl_xor_sync(0xffffffffu, ntr, m);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&counts[f * 4 + 0], cte); atomicAdd(&counts[f * 4 + 1], nte);
        atomicAdd(&counts[f * 4 + 2], ctr); atomicAdd(&counts[f * 4 + 3], ntr);
    }
    if (ccounts) {
        __syncthreads();
        for (int e = threadIdx.x; e < 6 * K; e += blockDim.x)
            if (shc[e]) atomicAdd(&ccounts[(size_t)f * 6 * K + e], shc[e]);
    }
}

// Xa = [X | 1] padded to [n][nvp] and its transpose [nvp][npad]
__global__ void build_xa_kernel(const float *__restrict__ X, int n, int d, int fit_intercept, int nvp, int64_t npad,
                                float *__restrict__ Xa, float *__restrict__ Xat)
{
    __shared__ float tile[32][33];
    const int i0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
    const int i = i0 + threadIdx.y, j = j0 + threadIdx.x;
    float v = 0.f;
    if (i < n) {
        if (j < d) v = X[(size_t)i * d + j];
        else if (j == d && fit_intercept) v = 1.f;
    }
    if (i < n && j < nvp) Xa[(size_t)i * nvp + j] = v;
    tile[threadIdx.y][threadIdx.x] = v;
    __syncthreads();
    const int jt = j0 + threadIdx.y, it = i0 + threadIdx.x;
    if (jt < nvp && it < npad) Xat[(size_t)jt * npad + it] = it < n ? tile[threadIdx.x][threadIdx.y] : 0.f;
}

int logreg_run(gs_handle *h, int n_cand, const double *Cv, double tol, int max_iter, int fit_intercept, bool refit,
               double *test_scores, double *train_scores, int32_t *n_iter, double *coef_out, float *ms_solve, float *ms_score)
{
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) { gs_set_error(h, "gs_logreg: no dataset (call gs_set_data first)"); return GS_ERR_NO_DATA; }
    if (!h->classification || h->n_classes < 2) { gs_set_error(h, "gs_logreg: needs a classification dataset with at least two classes"); return GS_ERR_UNSUPPORTED; }
    if (h->n_classes > 64) { gs_set_error(h, "gs_logreg: more than 64 classes is not supported"); return GS_ERR_UNSUPPORTED; }
    if (n_cand <= 0 || !Cv) { gs_set_error(h, "gs_logreg: bad arguments"); return GS_ERR_ARG; }
    for (int c = 0; c < n_cand; c++)
        if (!(Cv[c] > 0)) { gs_set_error(h, "gs_logreg: C must be > 0"); return GS_ERR_ARG; }
    const int kind = refit ? GS_SCORE_DEFAULT : h->score_kind;
    if (int e = check_scorer(h, "gs_logreg", kind)) return e;
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int n = (int)h->n, d = (int)h->d, ns = refit ? 1 : h->n_splits;
    const int nv = d + (fit_intercept ? 1 : 0), nvp = (nv + 31) & ~31;
    const int64_t npad = ((int64_t)n + 31) & ~31LL;
    const int nfit = n_cand * ns;                              // optimiser instances: one per (candidate, split)
    const int nc = h->n_classes;
    const int KC = nc > 2 ? nc : 1;                            // weight rows of a fit: 1 (binary: the class-1 logit) or one per class (multinomial)
    const int ncol = nfit * KC;                                // rows of W / Z^T / R / G in the two contractions
    const bool multi = KC > 1;

    h->evp.reset(); h->tt.reset();
    cudaEvent_t ev[3];
    for (auto &e : ev) e = h->evp.get();
    cudaEventRecord(ev[0], st);

    // ---- buffers ----
    DevBuf &bXa = h->dWork[0], &bXs = h->dWork[1], &bZ = h->dWork[2], &bR = h->dWork[3], &bW = h->dWork[4], &bV = h->dWork[5],
           &bS = h->dWork[6], &bMeta = h->dWork[7];
    GS_CUDA(bXa.reserve(((size_t)n * nvp + (size_t)nvp * npad) * 4));
    GS_CUDA(bXs.reserve(((size_t)n * nvp + (size_t)nvp * npad) * 4 * 2));
    GS_CUDA(bZ.reserve((size_t)ncol * npad * 4));
    GS_CUDA(bR.reserve((size_t)ncol * npad * 4 * 2));
    const int nchunk = (int)((npad + GRAD_KCHUNK - 1) / GRAD_KCHUNK);          // split-K of the gradient contraction
    GS_CUDA(bW.reserve((size_t)ncol * nvp * 4 * (3 + (size_t)nchunk)));
    GS_CUDA(bV.reserve((size_t)ncol * (5 + 2 * MCOR) * nvp * 8));          // nfit vectors of KC * nvp
    GS_CUDA(bS.reserve((size_t)nfit * sizeof(LbScalars)));
    GS_CUDA(bMeta.reserve((size_t)nfit * (4 + 8 + 16) + (size_t)nfit * std::max(2, KC) * 4 + (size_t)(nchunk + 4) * sizeof(TcBatch) + 256));
    float *dXa = bXa.as<float>(), *dXat = dXa + (size_t)n * nvp;
    // hi parts of [Xa | Xa^T] contiguous, then the lo parts: one split launch covers both matrices
    float *dXah = bXs.as<float>(), *dXath = dXah + (size_t)n * nvp, *dXal = dXath + (size_t)nvp * npad, *dXatl = dXal + (size_t)n * nvp;
    float *dZ = bZ.as<float>(), *dRh = bR.as<float>(), *dRl = dRh + (size_t)ncol * npad;
    float *dWh = bW.as<float>(), *dWl = dWh + (size_t)ncol * nvp, *dG = dWl + (size_t)ncol * nvp, *dGp = dG + (size_t)ncol * nvp;
    double *dV = bV.as<double>();
    LbScalars *dS = bS.as<LbScalars>();
    unsigned char *mp = bMeta.as<unsigned char>();
    const int CWS = std::max(2, KC);                           // class weights of a fit
    double *dInv = reinterpret_cast<double *>(mp); mp += (size_t)nfit * 8;
    float *dCwBuf = reinterpret_cast<float *>(mp); mp += (size_t)nfit * CWS * 4;
    int *dFoldOf = reinterpret_cast<int *>(mp); mp += (size_t)nfit * 4;
    int *dCounts = reinterpret_cast<int *>(mp); mp += (size_t)nfit * 16;
    int *dOpen = reinterpret_cast<int *>(mp); mp += 16;
    TcBatch *dBatch = reinterpret_cast<TcBatch *>(((uintptr_t)mp + 15) & ~(uintptr_t)15);

    // per-column constants
    // sum of the sample weights (1 without gs_set_sample_weight) of the training rows of every split, and per class
    const bool has_sw = !h->sample_w.empty();
    std::vector<double> ntrain(std::max(ns, 1), 0.0), ntrain_c((size_t)std::max(ns, 1) * nc, 0.0);
    for (int k = 0; k < ns; k++)
        for (int i = 0; i < n; i++)
            if (refit || h->is_train(i, k)) {
                const double wi = has_sw ? (double)h->sample_w[i] : 1.0;
                ntrain[k] += wi; ntrain_c[(size_t)k * nc + h->yc[i]] += wi;
            }
    const float *dSw = has_sw ? h->dSw.as<float>() : nullptr;
    if (int e = check_class_weight_sets(h, "gs_logreg", ns)) return e;
    const bool weighted = h->class_w_sets > 0;
    std::vector<float> cwcol((size_t)nfit * CWS, 1.f);
    std::vector<LbScalars> hs(nfit);
    std::vector<double> inv(nfit);
    std::vector<int> foldof(nfit);
    for (int c = 0; c < n_cand; c++)
        for (int k = 0; k < ns; k++) {
            const int col = c * ns + k;
            double sw_sum = (double)ntrain[k];                     // sum of the sample weights of the training rows
            if (weighted) {
                const double *cw = &h->class_w[(size_t)(h->class_w_sets == 1 ? 0 : k) * nc];
                sw_sum = 0;
                for (int q = 0; q < nc; q++) {
                    cwcol[(size_t)col * CWS + q] = (float)cw[q];
                    sw_sum += (double)((float)cw[q]) * ntrain_c[(size_t)k * nc + q];
                }
            }
            memset(&hs[col], 0, sizeof(LbScalars));
            hs[col].task = T_FG_START; hs[col].theta = 1.0; hs[col].fresh = 1;
            hs[col].l2 = 1.0 / (Cv[c] * sw_sum);
            inv[col] = 1.0 / sw_sum;
            foldof[col] = refit ? -100 : k;
        }
    GS_CUDA(cudaMemcpyAsync(dS, hs.data(), (size_t)nfit * sizeof(LbScalars), cudaMemcpyHostToDevice, st));
    GS_CUDA(cudaMemcpyAsync(dInv, inv.data(), (size_t)nfit * 8, cudaMemcpyHostToDevice, st));
    const float *dCw = nullptr;
    if (weighted) {
        GS_CUDA(cudaMemcpyAsync(dCwBuf, cwcol.data(), cwcol.size() * 4, cudaMemcpyHostToDevice, st));
        dCw = dCwBuf;
    }
    GS_CUDA(cudaMemcpyAsync(dFoldOf, foldof.data(), (size_t)nfit * 4, cudaMemcpyHostToDevice, st));
    GS_CUDA(cudaMemsetAsync(dV, 0, (size_t)ncol * (5 + 2 * MCOR) * nvp * 8, st));        // x0 = 0
    GS_CUDA(cudaMemsetAsync(dWh, 0, (size_t)ncol * nvp * 4 * 2, st));                      // trial point = x0
    GS_CUDA(cudaMemsetAsync(dRh, 0, (size_t)ncol * npad * 4 * 2, st));
    std::vector<TcBatch> hb;
    hb.push_back(TcBatch{0, 0, 0, nvp, dZ, npad});                                       // Z^T = W Xa^T (K = features: short)
    for (int q = 0; q < nchunk; q++)                                                     // G partials, K = rows in chunks
        hb.push_back(TcBatch{0, 0, q * GRAD_KCHUNK, (int)std::min<int64_t>(npad, (int64_t)(q + 1) * GRAD_KCHUNK),
                             dGp + (size_t)q * ncol * nvp, (int64_t)nvp});
    GS_CUDA(cudaMemcpyAsync(dBatch, hb.data(), hb.size() * sizeof(TcBatch), cudaMemcpyHostToDevice, st));
    int64_t launches = 0;

    {   // Xa, Xa^T and their hi/lo splits
        dim3 grid((unsigned)((npad + 31) / 32), (nvp + 31) / 32), block(32, 32);
        build_xa_kernel<<<grid, block, 0, st>>>(h->dX.as<float>(), n, d, fit_intercept, nvp, npad, dXa, dXat);
        GS_CUDA(cudaGetLastError());
        GS_CUDA(launch_split_tf32(dXa, dXah, dXal, (size_t)n * nvp + (size_t)nvp * npad, st));    // both arrays are contiguous
        launches += 2;
    }
    TcMap mXh, mXl, mXth, mXtl, mWh, mWl, mRh, mRl;
    GS_CUDA(tc_make_map(&mXh, dXah, n, nvp, nvp)); GS_CUDA(tc_make_map(&mXl, dXal, n, nvp, nvp));
    GS_CUDA(tc_make_map(&mXth, dXath, nvp, npad, npad)); GS_CUDA(tc_make_map(&mXtl, dXatl, nvp, npad, npad));
    GS_CUDA(tc_make_map(&mWh, dWh, ncol, nvp, nvp)); GS_CUDA(tc_make_map(&mWl, dWl, ncol, nvp, nvp));
    GS_CUDA(tc_make_map(&mRh, dRh, ncol, npad, npad)); GS_CUDA(tc_make_map(&mRl, dRl, ncol, npad, npad));

    const double factr_eps = 64.0 * EPSMCH;                  // ftol = factr * epsmch
    const int maxfun = 15000;
    int open = 1, rounds = 0;
    const int warps_per_block = 4;
    while (open > 0 && rounds < 4000) {
        // f, g at every open column's trial point: Z^T = W Xa^T ; R = residual(Z) ; G = R Xa
        h->tt.begin(h->evp, st);
        GS_CUDA(launch_gemm_nt_tf32x3(mWh, mWl, mXh, mXl, dBatch, 1, ncol, n, st));
        h->tt.end(h->evp, st, 3.0 * 2.0 * (double)ncol * n * nvp);
        dim3 grid(64, nfit);
        if (multi) multinomial_residual_kernel<<<grid, 256, 0, st>>>(dZ, npad, n, KC, h->dY.as<int>(), h->masks(), dFoldOf, dInv, dCw, dSw, dS, dRh, dRl);
        else logistic_residual_kernel<<<grid, 256, 0, st>>>(dZ, npad, n, h->dY.as<int>(), h->masks(), dFoldOf, dInv, dCw, dSw, dS, dRh, dRl);
        GS_CUDA(cudaGetLastError());
        h->tt.begin(h->evp, st);
        GS_CUDA(launch_gemm_nt_tf32x3(mRh, mRl, mXth, mXtl, dBatch + 1, nchunk, ncol, nv, st));
        h->tt.end(h->evp, st, 3.0 * 2.0 * (double)ncol * nv * (double)npad);
        GS_CUDA(launch_sum_partials(dGp, nchunk, (int64_t)ncol * nvp, dG, st));
        GS_CUDA(cudaMemsetAsync(dOpen, 0, 4, st));
        lbfgs_advance_kernel<<<(nfit + warps_per_block - 1) / warps_per_block, warps_per_block * 32, 0, st>>>(
            dS, dV, dG, (int64_t)nvp * KC, nfit, nv, nvp, KC, d, tol, factr_eps, max_iter, maxfun, 50, dWh, dWl, (int64_t)nvp * KC, dOpen);
        GS_CUDA(cudaGetLastError());
        GS_CUDA(cudaMemcpyAsync(&open, dOpen, 4, cudaMemcpyDeviceToHost, st));
        GS_CUDA(cudaStreamSynchronize(st));
        launches += 5;
        rounds++;
    }
    cudaEventRecord(ev[1], st);

    std::vector<LbScalars> fin(nfit);
    GS_CUDA(cudaMemcpyAsync(fin.data(), dS, (size_t)nfit * sizeof(LbScalars), cudaMemcpyDeviceToHost, st));
    if (!refit) {
        // ---- scoring: z at the final iterate for every row, accuracy split by fold ----
        lbfgs_export_kernel<<<nfit, 128, 0, st>>>(dV, nfit, nv, nvp, KC, dWh, dWl, (int64_t)nvp * KC);
        GS_CUDA(cudaGetLastError());
        h->tt.begin(h->evp, st);
        GS_CUDA(launch_gemm_nt_tf32x3(mWh, mWl, mXh, mXl, dBatch, 1, ncol, n, st));
        h->tt.end(h->evp, st, 3.0 * 2.0 * (double)ncol * n * nvp);
        GS_CUDA(cudaMemsetAsync(dCounts, 0, (size_t)nfit * 16, st));
        dim3 grid(64, nfit);
        // non-default scorers (gs_set_scoring): class counts or ROC-AUC pair counts from the z values already in HBM
        std::vector<int> ccounts;
        std::vector<unsigned long long> araw;
        const int per_fit = 6 * nc;                                          // [2 splits][nc][support, tp, predicted]
        if (multi) {
            int *d_cc = nullptr;
            if (kind != GS_SCORE_DEFAULT) {
                GS_CUDA(h->dScore.reserve((size_t)nfit * per_fit * 4));
                GS_CUDA(cudaMemsetAsync(h->dScore.p, 0, (size_t)nfit * per_fit * 4, st));
                d_cc = h->dScore.as<int>();
            }
            multinomial_count_kernel<<<grid, 256, (size_t)per_fit * 4, st>>>(dZ, npad, n, KC, h->dY.as<int>(), h->masks(), dFoldOf, dCounts, d_cc);
            GS_CUDA(cudaGetLastError());
            if (d_cc) {
                ccounts.resize((size_t)nfit * per_fit);
                GS_CUDA(cudaMemcpyAsync(ccounts.data(), d_cc, ccounts.size() * 4, cudaMemcpyDeviceToHost, st));
            }
        } else {
            logistic_count_kernel<<<grid, 256, 0, st>>>(dZ, npad, n, h->dY.as<int>(), h->masks(), dFoldOf, dCounts);
            GS_CUDA(cudaGetLastError());
        }
        launches += 3;
        std::vector<int> counts((size_t)nfit * 4);
        GS_CUDA(cudaMemcpyAsync(counts.data(), dCounts, counts.size() * 4, cudaMemcpyDeviceToHost, st));
        if (kind == GS_SCORE_ROC_AUC) {
            std::vector<int> meta((size_t)nfit * 2);
            for (int col = 0; col < nfit; col++) { meta[col] = col; meta[nfit + col] = refit ? -100 : col % ns; }
            GS_CUDA(h->dScore.reserve((size_t)nfit * 40));
            unsigned long long *d_auc = h->dScore.as<unsigned long long>();
            int *d_meta = (int *)(d_auc + (size_t)nfit * 4);
            GS_CUDA(cudaMemcpyAsync(d_meta, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice, st));
            GS_CUDA(cudaMemsetAsync(d_auc, 0, (size_t)nfit * 32, st));
            GS_CUDA(launch_auc_pairs_f32(dZ, npad, n, h->class_start[1], h->masks(), d_meta, d_meta + nfit, nfit, +1, d_auc, st));
            araw.resize((size_t)nfit * 4);
            GS_CUDA(cudaMemcpyAsync(araw.data(), d_auc, (size_t)nfit * 32, cudaMemcpyDeviceToHost, st));
            launches++;
        } else if (kind != GS_SCORE_DEFAULT && !multi) {
            GS_CUDA(h->dScore.reserve((size_t)nfit * 48));
            GS_CUDA(cudaMemsetAsync(h->dScore.p, 0, (size_t)nfit * 48, st));
            logistic_classes_kernel<<<grid, 256, 0, st>>>(dZ, npad, n, h->dY.as<int>(), h->masks(), dFoldOf, h->dScore.as<int>());
            GS_CUDA(cudaGetLastError());
            ccounts.resize((size_t)nfit * 12);
            GS_CUDA(cudaMemcpyAsync(ccounts.data(), h->dScore.p, ccounts.size() * 4, cudaMemcpyDeviceToHost, st));
            launches++;
        }
        cudaEventRecord(ev[2], st);
        GS_CUDA(cudaStreamSynchronize(st));
        const SplitScoreStats ss(h, ns, kind);
        for (int col = 0; col < nfit; col++) {
            for (int sp = 0; sp < 2; sp++) {
                double *out = sp == 0 ? test_scores : train_scores;
                if (!out) continue;
                if (kind == GS_SCORE_DEFAULT) out[col] = SplitScoreStats::accuracy(&counts[(size_t)col * 4 + sp * 2]);
                else if (kind == GS_SCORE_ROC_AUC) out[col] = ss.auc(col % ns, sp, &araw[(size_t)col * 4 + sp * 2]);
                else out[col] = ss.counts(&ccounts[(size_t)col * per_fit + sp * 3 * nc]);
            }
            if (n_iter) n_iter[col] = fin[col].iter;
        }
    } else {
        std::vector<double> x((size_t)nvp * KC);
        GS_CUDA(cudaMemcpyAsync(x.data(), dV, x.size() * 8, cudaMemcpyDeviceToHost, st));
        cudaEventRecord(ev[2], st);
        GS_CUDA(cudaStreamSynchronize(st));
        for (int q = 0; q < KC; q++) {                                       // [KC][d + 1]: weights, then the intercept
            for (int j = 0; j < d; j++) coef_out[(size_t)q * (d + 1) + j] = x[(size_t)q * nvp + j];
            coef_out[(size_t)q * (d + 1) + d] = fit_intercept ? x[(size_t)q * nvp + d] : 0.0;
        }
        if (n_iter) n_iter[0] = fin[0].iter;
    }
    for (int col = 0; col < nfit; col++)
        if (fin[col].task != T_DONE) { gs_set_error(h, "gs_logreg: optimiser did not terminate"); return GS_ERR_NUMERIC; }
    linear_profile(h, ev, launches, ms_solve, ms_score);
    gs_profile &pf = h->prof;
    pf.smo_iterations = rounds;                                 // function-evaluation rounds
    pf.gram_flops = (double)rounds * 2.0 * 2.0 * (double)n * nv * ncol;
    pf.d2h_bytes = (int64_t)nfit * (16 + sizeof(LbScalars));
    return GS_OK;
}

}  // namespace

extern "C" {

int gs_logreg(gs_handle *h, int32_t n_cand, const double *C, double tol, int32_t max_iter, int32_t fit_intercept, uint32_t flags,
              double *test_scores, double *train_scores, int32_t *n_iter, float *fit_ms, float *score_ms)
{
    if (h && !test_scores) { gs_set_error(h, "gs_logreg: test_scores is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    const int st = logreg_run(h, n_cand, C, tol, max_iter, fit_intercept, false, test_scores,
                              (flags & GS_RETURN_TRAIN) ? train_scores : nullptr, n_iter, nullptr, &a, &b);
    if (st) return st;
    spread_call_ms(n_cand * h->n_splits, a, b, fit_ms, score_ms);
    return GS_OK;
}

int gs_logreg_refit(gs_handle *h, double C, double tol, int32_t max_iter, int32_t fit_intercept, double *coef_out, int32_t *n_iter)
{
    if (h && !coef_out) { gs_set_error(h, "gs_logreg_refit: coef_out is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    return logreg_run(h, 1, &C, tol, max_iter, fit_intercept, true, nullptr, nullptr, n_iter, coef_out, &a, &b);
}

}  // extern "C"
