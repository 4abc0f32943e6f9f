// linsvc.cu -- batched LinearSVC (L2-regularised squared hinge, primal): one liblinear TRON run per column.
//
// Replaces (reference base_search.py:83-87 -> sklearn _fit_and_score -> LinearSVC.fit/score):
//   sklearn/svm/_base.py:1230-1310 _fit_liblinear       class_weight_, bias = intercept_scaling, intercept_ = bias * w[-1]
//   liblinear linear.cpp:2453-2578 train                remove_zero_weight, classes grouped in sorted-label order; binary:
//                                                       class 0 -> y = -1, train_one(Cp = C w_1, Cn = C w_0); one-vs-rest:
//                                                       class i -> +1 with C w_i, every other row C
//   linear.cpp:2309-2362 train_one                      C_i = W_i Cp|Cn, eps = tol max(min(pos, neg), 1) / l
//   linear.cpp:228-390 l2r_l2_svc_fun                   f = w'w/2 + sum C_i max(0, 1 - y_i w'x_i)^2,
//                                                       g = w + 2 X_I' (C y (z - 1))_I, Hs = s + 2 X_I' (C X_I s)_I
//   tron.cpp:44-209 TRON::tron / trcg                   trust-region Newton with conjugate gradients, restated op for op
//
// A column is one (candidate, split, one-vs-rest class) fit.  Every round, each open column submits one float64 vector v
// (the trial point w + s of fun(), or the CG direction d of Hv()), and the round computes for all columns at once
//   Z^T[col][row] = v[col] . Xa[row]                  (FP64 tensor cores, K = d + 1; Xa = [X | bias])
//   R[col][row]   = the element-wise pass below
//   G[col][f]     = sum_row R[col][row] Xa[row][f]    (FP64 tensor cores, split-K over rows, partials summed in order)
// then one warp per column (tron_advance_kernel) consumes G and moves TRON to its next submission.
//   fun mode: z = y Z; loss partials C (1 - z)^2 for z < 1; R = C y (z - 1) for z < 1 (the gradient of the trial point,
//             needed only if TRON accepts the step) and the trial point's active set {z < 1} into the column's spare
//             mask, which becomes current on acceptance -- a rejected step leaves w, f, g and the active set as they were.
//   Hv mode:  R = C (X d) on the current active set.
// liblinear's grad() reads the z of the latest fun() and Hv() the active set of the latest grad(): grad() only ever follows
// an accepted fun(), so both are the trial point's, which is what the spare mask holds.
// The host loop of the rounds and the scoring of the final weights are linear_search.cu's (TronRounds, score_linear_fits).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

constexpr double ETA0 = 1e-4, ETA1 = 0.25, ETA2 = 0.75, SIGMA1 = 0.25, SIGMA2 = 0.5, SIGMA3 = 4;
// M_FUN / M_HV / M_DONE, PW_BLOCKS, NVEC and TrState are in common.cuh: linsvr.cu drives the same TRON

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int m = 16; m; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    return v;
}

// One warp per column.  dot / nrm2: strided per-lane sums, then a fixed xor tree (deterministic).  axpy is a fused
// multiply-add per element, as the BLAS daxpy scikit-learn links; scalar formulas are rounded operation by operation.
#define TR_FOR(j) for (int j = lane; j < nvp; j += 32)
__global__ void tron_advance_kernel(TrState *__restrict__ St, double *__restrict__ Vec, double *__restrict__ V,
                                    const double *__restrict__ Gp, int nchunk, int64_t gp_stride, const double *__restrict__ fpart,
                                    int ncol, int nvp, int max_iter, int *__restrict__ n_open)
{
    const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (c >= ncol) return;
    TrState S = St[c];
    if (S.mode == M_DONE) return;
    double *w = Vec + (size_t)c * NVEC * nvp, *g = w + nvp, *s = g + nvp, *r = s + nvp, *d = r + nvp;
    double *v = V + (size_t)c * nvp;
    const double *G = Gp + (size_t)c * nvp;
    auto Gat = [&](int j) {
        double x = G[j];
        for (int q = 1; q < nchunk; q++) x += G[(size_t)q * gp_stride + j];
        return x;
    };
    auto dot = [&](const double *a, const double *b) {
        double x = 0;
        TR_FOR(j) x = __dadd_rn(x, __dmul_rn(a[j], b[j]));
        return warp_sum(x);
    };

    bool start_cg = false, finish_cg = false;
    if (S.mode == M_FUN) {
        double fl = 0;
        for (int b = 0; b < PW_BLOCKS; b++) fl += fpart[(size_t)c * PW_BLOCKS + b];
        const double fnew = __dadd_rn(__ddiv_rn(dot(v, v), 2.0), fl);          // fun(): w'w / 2, then the loss terms
        if (S.init) {                                                          // tron(): f = fun(0); grad(0, g)
            S.init = 0;
            S.f = fnew;
            TR_FOR(j) g[j] = __dadd_rn(v[j], __dmul_rn(2.0, Gat(j)));
            S.cur ^= 1;
            S.delta = sqrt(dot(g, g));
            S.gnorm1 = S.delta;
            if (S.gnorm1 <= __dmul_rn(S.eps, S.gnorm1) || S.iter > max_iter) { S.mode = M_DONE; S.n_iter = S.iter - 1; }
            else start_cg = true;
        } else {
            const double f = S.f;
            const double gs = dot(g, s);
            const double prered = __dmul_rn(-0.5, __dsub_rn(gs, dot(s, r)));
            const double actred = __dsub_rn(f, fnew);
            const double snorm = sqrt(dot(s, s));
            if (S.iter == 1) S.delta = fmin(S.delta, snorm);
            double alpha;
            const double den = __dsub_rn(__dsub_rn(fnew, f), gs);
            if (den <= 0) alpha = SIGMA3;
            else alpha = fmax(SIGMA1, __dmul_rn(-0.5, __ddiv_rn(gs, den)));
            double delta = S.delta;
            if (actred < __dmul_rn(ETA0, prered)) delta = fmin(__dmul_rn(fmax(alpha, SIGMA1), snorm), __dmul_rn(SIGMA2, delta));
            else if (actred < __dmul_rn(ETA1, prered)) delta = fmax(__dmul_rn(SIGMA1, delta), fmin(__dmul_rn(alpha, snorm), __dmul_rn(SIGMA2, delta)));
            else if (actred < __dmul_rn(ETA2, prered)) delta = fmax(__dmul_rn(SIGMA1, delta), fmin(__dmul_rn(alpha, snorm), __dmul_rn(SIGMA3, delta)));
            else delta = fmax(delta, fmin(__dmul_rn(alpha, snorm), __dmul_rn(SIGMA3, delta)));
            S.delta = delta;
            bool stop = false;
            if (actred > __dmul_rn(ETA0, prered)) {                           // accept: w, f, g and the active set move
                S.iter++;
                TR_FOR(j) { w[j] = v[j]; g[j] = __dadd_rn(v[j], __dmul_rn(2.0, Gat(j))); }
                S.f = fnew;
                S.cur ^= 1;
                const double gnorm = sqrt(dot(g, g));
                if (gnorm <= __dmul_rn(S.eps, S.gnorm1)) stop = true;
            }
            if (!stop) {
                if (S.f < -1.0e+32) stop = true;
                else if (fabs(actred) <= 0 && prered <= 0) stop = true;
                else if (fabs(actred) <= __dmul_rn(1.0e-12, fabs(S.f)) && fabs(prered) <= __dmul_rn(1.0e-12, fabs(S.f))) stop = true;
            }
            if (stop || S.iter > max_iter) { S.mode = M_DONE; S.n_iter = S.iter - 1; }
            else start_cg = true;
        }
    } else {                                                                   // M_HV: Hd = d + 2 G
        __syncwarp();
        double dHd = 0;
        TR_FOR(j) dHd = __dadd_rn(dHd, __dmul_rn(d[j], __dadd_rn(d[j], __dmul_rn(2.0, Gat(j)))));
        dHd = warp_sum(dHd);
        double alpha = __ddiv_rn(S.rTr, dHd);
        TR_FOR(j) s[j] = fma(alpha, d[j], s[j]);
        __syncwarp();
        if (sqrt(dot(s, s)) > S.delta) {                                      // trcg: the step reaches the trust-region boundary
            alpha = -alpha;
            TR_FOR(j) s[j] = fma(alpha, d[j], s[j]);
            __syncwarp();
            const double std_ = dot(s, d), sts = dot(s, s), dtd = dot(d, d);
            const double dsq = __dmul_rn(S.delta, S.delta);
            const double rad = sqrt(__dadd_rn(__dmul_rn(std_, std_), __dmul_rn(dtd, __dsub_rn(dsq, sts))));
            if (std_ >= 0) alpha = __ddiv_rn(__dsub_rn(dsq, sts), __dadd_rn(std_, rad));
            else alpha = __ddiv_rn(__dsub_rn(rad, std_), dtd);
            TR_FOR(j) s[j] = fma(alpha, d[j], s[j]);
            alpha = -alpha;
            TR_FOR(j) r[j] = fma(alpha, __dadd_rn(d[j], __dmul_rn(2.0, Gat(j))), r[j]);
            finish_cg = true;
        } else {
            alpha = -alpha;
            TR_FOR(j) r[j] = fma(alpha, __dadd_rn(d[j], __dmul_rn(2.0, Gat(j))), r[j]);
            __syncwarp();
            const double rnew = dot(r, r);
            const double beta = __ddiv_rn(rnew, S.rTr);
            TR_FOR(j) d[j] = __dadd_rn(__dmul_rn(beta, d[j]), r[j]);
            S.rTr = rnew;
            if (sqrt(rnew) <= S.cgtol) finish_cg = true;
            else { S.cg_iter++; TR_FOR(j) v[j] = d[j]; }
        }
    }
    if (start_cg) {                                                            // trcg entry: s = 0, r = -g, d = r
        __syncwarp();
        TR_FOR(j) { s[j] = 0.0; r[j] = -g[j]; d[j] = -g[j]; }
        __syncwarp();
        S.cgtol = __dmul_rn(0.1, sqrt(dot(g, g)));
        S.rTr = dot(r, r);
        S.cg_iter = 0;
        if (sqrt(S.rTr) <= S.cgtol) finish_cg = true;
        else { S.mode = M_HV; S.cg_iter = 1; TR_FOR(j) v[j] = d[j]; }
    }
    if (finish_cg) {                                                           // w_new = w + s: the next fun()
        __syncwarp();
        TR_FOR(j) v[j] = __dadd_rn(w[j], s[j]);
        S.mode = M_FUN;
    }
    __syncwarp();
    if (lane == 0) {
        St[c] = S;
        if (S.mode != M_DONE) atomicAdd(n_open, 1);
    }
}

// The element-wise pass between the two contractions (see the file comment).  Column c trains on the rows of split
// St[c].fold (every row for the refit) whose weight is positive.  Loss partials: fpart[c][block], fixed-order tree.
__global__ void linsvc_pointwise_kernel(const double *__restrict__ Zt, int64_t ldz, int n, const int *__restrict__ y,
                                        SplitMasks sm, const double *__restrict__ W, const TrState *__restrict__ St,
                                        unsigned char *__restrict__ mask, int64_t mask_stride, double *__restrict__ R,
                                        double *__restrict__ fpart)
{
    __shared__ double sh[256];
    const int c = blockIdx.y;
    const TrState &S = St[c];
    const int mode = S.mode, fold = S.fold, pos = S.pos;
    const double Cp = S.Cp, Cn = S.Cn;
    const unsigned char *mcur = mask + (size_t)S.cur * mask_stride + (size_t)c * ldz;
    unsigned char *mnext = mask + (size_t)(S.cur ^ 1) * mask_stride + (size_t)c * ldz;
    double acc = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const size_t idx = (size_t)c * ldz + i;
        double res = 0.0;
        if (mode != M_DONE && split_train(sm, i, fold) && W[i] > 0) {
            const double yi = y[i] == pos ? 1.0 : -1.0;
            const double Ci = __dmul_rn(W[i], yi > 0 ? Cp : Cn);
            if (mode == M_FUN) {
                const double z = __dmul_rn(yi, Zt[idx]);
                const double dd = __dsub_rn(1.0, z);
                if (dd > 0) acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(Ci, dd), dd));
                const bool act = z < 1;
                if (act) res = __dmul_rn(__dmul_rn(Ci, yi), __dsub_rn(z, 1.0));
                mnext[i] = act;
            } else if (mcur[i]) {
                res = __dmul_rn(Ci, Zt[idx]);
            }
        } else if (mode == M_FUN) {
            mnext[i] = 0;
        }
        R[idx] = res;
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int m = blockDim.x >> 1; m; m >>= 1) {
        if ((int)threadIdx.x < m) sh[threadIdx.x] += sh[threadIdx.x + m];
        __syncthreads();
    }
    if (threadIdx.x == 0) fpart[(size_t)c * PW_BLOCKS + blockIdx.x] = sh[0];
}

// Xa = [X | bias | 0 ...] in float64 ([npad][nvp], rows >= n zero) and its transpose [nvp][npad]
__global__ void build_xa64_kernel(const float *__restrict__ X32, const double *__restrict__ X64, int n, int d, double bias, int nvp,
                                  int64_t npad, double *__restrict__ Xa, double *__restrict__ Xat)
{
    __shared__ double tile[32][33];
    const int i0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
    const int i = i0 + threadIdx.y, j = j0 + threadIdx.x;
    double v = 0.0;
    if (i < n) {
        if (j < d) v = X64 ? X64[(size_t)i * d + j] : (double)X32[(size_t)i * d + j];
        else if (j == d) v = bias;
    }
    if (i < npad && j < nvp) Xa[(size_t)i * nvp + j] = v;
    tile[threadIdx.y][threadIdx.x] = v;
    __syncthreads();
    const int jt = j0 + threadIdx.y, it = i0 + threadIdx.x;
    if (jt < nvp && it < npad) Xat[(size_t)jt * npad + it] = tile[threadIdx.x][threadIdx.y];
}

// final weights of every column -> the submission rows (one more forward contraction gives the decision values)
__global__ void export_w_kernel(const double *__restrict__ Vec, int ncol, int nvp, double *__restrict__ V)
{
    const int c = blockIdx.x;
    if (c >= ncol) return;
    for (int j = threadIdx.x; j < nvp; j += blockDim.x) V[(size_t)c * nvp + j] = Vec[(size_t)c * NVEC * nvp + j];
}

// Per-class counts of fit f's predictions from its KC decision rows (KC == 1: z > 0 -> class 1; else the first arg-max):
// counts[f][split (0 test, 1 train)][class][3 = support, tp, predicted]
__global__ void linsvc_count_kernel(const double *__restrict__ Zt, int64_t ldz, int n, int K, int KC, const int *__restrict__ y,
                                    SplitMasks sm, const int *__restrict__ fold_of_fit, int *__restrict__ counts)
{
    extern __shared__ int shc[];                                         // [2][K][3]
    const int f = blockIdx.y, fc = fold_of_fit[f];
    for (int e = threadIdx.x; e < 6 * K; e += blockDim.x) shc[e] = 0;
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const size_t base = (size_t)f * KC * ldz + i;
        int pred;
        if (KC == 1) pred = Zt[base] > 0.0 ? 1 : 0;
        else {
            pred = 0;
            double best = Zt[base];
            for (int k = 1; k < KC; k++) { const double z = Zt[base + (size_t)k * ldz]; if (z > best) { best = z; pred = k; } }
        }
        const int yc = y[i];
        const int sp = split_test(sm, i, fc) ? 0 : (split_train(sm, i, fc) ? 1 : 2);
        if (sp < 2) {
            atomicAdd(&shc[(sp * K + yc) * 3 + 0], 1);
            if (pred == yc) atomicAdd(&shc[(sp * K + yc) * 3 + 1], 1);
            atomicAdd(&shc[(sp * K + pred) * 3 + 2], 1);
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 6 * K; e += blockDim.x)
        if (shc[e]) atomicAdd(&counts[(size_t)f * 6 * K + e], shc[e]);
}

int linsvc_run(gs_handle *h, int n_cand, const double *Cv, double tol, int max_iter, int fit_intercept, double intercept_scaling,
               bool refit, double *test_scores, double *train_scores, int32_t *n_iter, double *coef_out, float *ms_solve,
               float *ms_score)
{
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) { gs_set_error(h, "gs_linsvc: no dataset (call gs_set_data first)"); return GS_ERR_NO_DATA; }
    if (!h->classification || h->n_classes < 2) { gs_set_error(h, "gs_linsvc: needs a classification dataset with at least two classes"); return GS_ERR_UNSUPPORTED; }
    if (h->n_classes > 64) { gs_set_error(h, "gs_linsvc: more than 64 classes is not supported"); return GS_ERR_UNSUPPORTED; }
    if (n_cand <= 0 || !Cv || !(tol > 0) || max_iter < 0) { gs_set_error(h, "gs_linsvc: bad arguments"); return GS_ERR_ARG; }
    if (fit_intercept && !(intercept_scaling > 0 && std::isfinite(intercept_scaling))) {
        gs_set_error(h, "gs_linsvc: intercept_scaling must be > 0 with an intercept"); return GS_ERR_ARG;
    }
    for (int c = 0; c < n_cand; c++)
        if (!(Cv[c] > 0) || !std::isfinite(Cv[c])) { gs_set_error(h, "gs_linsvc: C must be > 0 and finite"); return GS_ERR_ARG; }
    const int ns = refit ? 1 : h->n_splits, nc = h->n_classes;
    const int KC = nc > 2 ? nc : 1;
    if (int e = check_class_weight_sets(h, "gs_linsvc", ns)) return e;
    if (int e = check_scorer(h, "gs_linsvc", refit ? GS_SCORE_DEFAULT : h->score_kind)) return e;
    const bool weighted = h->class_w_sets > 0;
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int n = (int)h->n, d = (int)h->d;
    const int nvp = (int)round_up(d + 1, 64);
    const int64_t npad = round_up(n, 64);
    const int nfit = n_cand * ns, ncol = nfit * KC;

    // training rows of positive weight per (split, class): liblinear's l, pos, neg after remove_zero_weight
    const bool has_sw = !h->sample_w.empty();
    std::vector<double> W64(n, 1.0);
    if (has_sw) W64 = h->sample_w64;
    std::vector<int64_t> cnt((size_t)ns * nc, 0);
    for (int k = 0; k < ns; k++)
        for (int i = 0; i < n; i++)
            if ((refit || h->is_train(i, k)) && W64[i] > 0) cnt[(size_t)k * nc + h->yc[i]]++;
    for (size_t e = 0; e < cnt.size(); e++)
        if (cnt[e] == 0) { gs_set_error(h, "gs_linsvc: a class has no training row of positive weight in a split"); return GS_ERR_UNSUPPORTED; }

    h->evp.reset(); h->tt.reset();
    cudaEvent_t ev[3];
    for (auto &e : ev) e = h->evp.get();
    cudaEventRecord(ev[0], st);

    DevBuf &bXa = h->dWork[0], &bZ = h->dWork[1];
    const size_t xa_elems = (size_t)npad * nvp;
    GS_CUDA(bXa.reserve(xa_elems * 2 * 8 + (size_t)npad * 8));
    GS_CUDA(bZ.reserve((size_t)round_up(ncol, 64) * npad * 8));
    double *dXa = bXa.as<double>(), *dXat = dXa + xa_elems, *dW = dXat + xa_elems, *dZ = bZ.as<double>();
    TronRounds tr;
    if (int e = tr.reserve(h, ncol)) return e;

    std::vector<TrState> hs(ncol);
    for (int c = 0; c < n_cand; c++)
        for (int k = 0; k < ns; k++) {
            const int fit = c * ns + k;
            const double *cw = weighted ? &h->class_w[(size_t)(h->class_w_sets == 1 ? 0 : k) * nc] : nullptr;
            int64_t l = 0;
            for (int q = 0; q < nc; q++) l += cnt[(size_t)k * nc + q];
            for (int q = 0; q < KC; q++) {
                TrState &S = hs[(size_t)fit * KC + q];
                memset(&S, 0, sizeof S);
                S.mode = M_FUN; S.iter = 1; S.init = 1; S.fold = refit ? -100 : k;
                S.pos = KC == 1 ? 1 : q;
                S.Cp = cw ? Cv[c] * cw[S.pos] : Cv[c];                          // weighted_C[i] = C x weight[i]
                S.Cn = KC == 1 ? (cw ? Cv[c] * cw[0] : Cv[c]) : Cv[c];         // one-vs-rest negatives: the unweighted C
                const int64_t pos = cnt[(size_t)k * nc + S.pos], neg = l - pos;
                S.eps = tol * (double)std::max<int64_t>(std::min(pos, neg), 1) / (double)l;
            }
        }
    GS_CUDA(cudaMemcpyAsync(tr.St, hs.data(), (size_t)ncol * sizeof(TrState), cudaMemcpyHostToDevice, st));
    GS_CUDA(cudaMemcpyAsync(dW, W64.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    GS_CUDA(launch_build_xa64(h->x_dtype == GS_F64 ? nullptr : h->dX.as<float>(), h->x_dtype == GS_F64 ? h->dX64.as<double>() : nullptr,
                              n, d, fit_intercept ? intercept_scaling : 0.0, nvp, npad, dXa, dXat, st));
    int64_t launches = 1;
    const int *Y = h->dY.as<int>();
    auto pointwise = [&]() {
        linsvc_pointwise_kernel<<<dim3(PW_BLOCKS, ncol), 256, 0, st>>>(dZ, npad, n, Y, h->masks(), dW, tr.St, tr.mask,
                                                                       (int64_t)ncol * npad, tr.R, tr.F);
        return cudaGetLastError();
    };
    if (int e = tr.run(h, "gs_linsvc", dXa, dXat, dZ, max_iter, pointwise, launches)) return e;
    cudaEventRecord(ev[1], st);

    std::vector<TrState> fin(ncol);
    GS_CUDA(cudaMemcpyAsync(fin.data(), tr.St, (size_t)ncol * sizeof(TrState), cudaMemcpyDeviceToHost, st));
    if (!refit) {
        // ---- scoring: float64 decision values of the final weights for every row ----
        export_w_kernel<<<ncol, 128, 0, st>>>(tr.Vec, ncol, nvp, tr.V);
        GS_CUDA(cudaGetLastError());
        launches++;
        if (int e = score_linear_fits(h, tr.V, dXa, dZ, nfit, KC, ns, h->score_kind, test_scores, train_scores, ev[2], launches)) return e;
        for (int f = 0; f < nfit && n_iter; f++) {
            int it = 0;
            for (int q = 0; q < KC; q++) it = std::max(it, fin[(size_t)f * KC + q].n_iter);
            n_iter[f] = it;
        }
    } else {
        std::vector<double> x((size_t)KC * NVEC * nvp);
        GS_CUDA(cudaMemcpyAsync(x.data(), tr.Vec, x.size() * 8, cudaMemcpyDeviceToHost, st));
        cudaEventRecord(ev[2], st);
        GS_CUDA(cudaStreamSynchronize(st));
        for (int q = 0; q < KC; q++) {
            for (int j = 0; j <= d; j++) coef_out[(size_t)q * (d + 1) + j] = x[(size_t)q * NVEC * nvp + j];
            if (n_iter) n_iter[q] = fin[q].n_iter;
        }
    }
    linear_profile(h, ev, launches, ms_solve, ms_score);
    h->prof.smo_iterations = tr.rounds;                         // TRON rounds: one fun() or Hv() per open column each
    h->prof.d2h_bytes = (int64_t)ncol * sizeof(TrState);
    return GS_OK;
}

}  // namespace

// ---- the pieces linear_search.cu (TronRounds, the classification scorers), linsvr.cu, sgd.cu and sag.cu (Xa) share ----
cudaError_t launch_tron_advance(TrState *St, double *Vec, double *V, const double *Gp, int nchunk, int64_t gp_stride,
                                const double *fpart, int ncol, int nvp, int max_iter, int *n_open, cudaStream_t st)
{
    tron_advance_kernel<<<(ncol + 3) / 4, 128, 0, st>>>(St, Vec, V, Gp, nchunk, gp_stride, fpart, ncol, nvp, max_iter, n_open);
    return cudaGetLastError();
}

cudaError_t launch_build_xa64(const float *X32, const double *X64, int n, int d, double bias, int nvp, int64_t npad, double *Xa,
                              double *Xat, cudaStream_t st)
{
    dim3 grid((unsigned)((npad + 31) / 32), (nvp + 31) / 32), block(32, 32);
    build_xa64_kernel<<<grid, block, 0, st>>>(X32, X64, n, d, bias, nvp, npad, Xa, Xat);
    return cudaGetLastError();
}

cudaError_t launch_linsvc_count(const double *Zt, int64_t ldz, int n, int K, int KC, const int *y, SplitMasks sm,
                                const int *fold_of_fit, int nfit, int *counts, cudaStream_t st)
{
    linsvc_count_kernel<<<dim3(64, nfit), 256, (size_t)6 * K * 4, st>>>(Zt, ldz, n, K, KC, y, sm, fold_of_fit, counts);
    return cudaGetLastError();
}

extern "C" {

int gs_linsvc(gs_handle *h, int32_t n_cand, const double *C, double tol, int32_t max_iter, int32_t fit_intercept,
              double intercept_scaling, uint32_t flags, double *test_scores, double *train_scores, int32_t *n_iter,
              float *fit_ms, float *score_ms)
{
    if (h && !test_scores) { gs_set_error(h, "gs_linsvc: test_scores is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    const int st = linsvc_run(h, n_cand, C, tol, max_iter, fit_intercept, intercept_scaling, false, test_scores,
                              (flags & GS_RETURN_TRAIN) ? train_scores : nullptr, n_iter, nullptr, &a, &b);
    if (st) return st;
    spread_call_ms(n_cand * h->n_splits, a, b, fit_ms, score_ms);
    return GS_OK;
}

int gs_linsvc_refit(gs_handle *h, double C, double tol, int32_t max_iter, int32_t fit_intercept, double intercept_scaling,
                    double *coef_out, int32_t *n_iter)
{
    if (h && !coef_out) { gs_set_error(h, "gs_linsvc_refit: coef_out is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    return linsvc_run(h, 1, &C, tol, max_iter, fit_intercept, intercept_scaling, true, nullptr, nullptr, n_iter, coef_out, &a, &b);
}

}  // extern "C"
