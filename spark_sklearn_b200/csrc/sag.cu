// sag.cu -- batched LogisticRegression(solver='sag' | 'saga'): scikit-learn's SAG / SAGA solver restated step for step, one
// warp per (candidate, split) fit.
//
// Replaces (reference base_search.py:83-87 -> sklearn _fit_and_score -> LogisticRegression.fit / score):
//   linear_model/_logistic.py _logistic_regression_path  the targets (binary 0 / 1 with classes_[1] positive, 'log'; three
//                                             or more classes label-encoded, 'multinomial'), class x sample weights in X's
//                                             dtype; the penalties, step size and seed come from the host per fit
//   linear_model/_sag_fast.pyx.tp sag64 / sag32  the sample loop on a dense ArrayDataset: rand_int draws with replacement,
//                                             seen / num_seen, lagged_update, predict_sample, the gradient, wscale, the sum
//                                             of gradients, the SAGA correction, the intercept, the gradient memory, the
//                                             cumulative sums, scale_weights mid-epoch (wscale < 1e-9) and at every epoch
//                                             end, the max_change / max_weight stop, the non-finite status
//   _loss/_loss.pyx.tp                        cgradient_half_binomial, the half squared error, CyHalfMultinomialLoss.cy_gradient
//
// A fit is one warp.  Its weights and sum_gradient live in registers, in scikit-learn's [feature][class] layout: lane L holds
// entries q = L, L + 32, ... of the d x K array.  Lane k holds class k's intercept and intercept gradient sum (k and k + 32).
// Every lane computes the same scalars (wscale, num_seen, the cumulative sums).  The gradient memory [l][K], seen [l] and
// previous_weights live in HBM.  Dense X touches every feature at every step, so feature_hist is one scalar and the
// cumulative sums the lagged update reads are two registers; the arrays are kept in HBM as well for SAGA with an L1 term,
// whose lagged update replays every step since the last update when a mid-epoch rescale lands on an epoch's last sample.
// predict_sample's sums are made in feature order (each lane writes its products to shared memory; lane k adds class k's in
// sequence), every operation is rounded on its own (no contraction), and float32 X runs sag32: every value scikit-learn
// keeps in float -- the weights, wscale, the cumulative sums, the gradients -- is rounded to float where its C expression
// is, while the step size and the penalties stay double.  Only exp (the logistic gradients) comes from CUDA's math library.
// The training order and the scoring of the final weights are linear_search.cu's (train_rows, score_linear_fits).
#include "common.cuh"
#include "sequential.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

constexpr int SAG_WARPS = 4;            // fits per block
constexpr int MAX_S = GS_SAG_MAX_COEF / 32;

struct SagFit {
    int off, l;            // training positions: order[off .. off + l), internal rows in the splitter's order
    int out;               // row block of V / n_iter / status / stats
    int cwset;             // class-weight set (-1: none)
    uint32_t seed;         // make_dataset's seed
    int saga;
    double step, alpha, beta;   // the step size, alpha_scaled, beta_scaled
};

template <typename T> __device__ __forceinline__ double soft_threshold(double x, double sh)
{
    const double a = rnd<T>(__dsub_rn(x, sh)), b = rnd<T>(__dsub_rn(-x, sh));
    return rnd<T>(__dsub_rn(a > 0.0 ? a : 0.0, b > 0.0 ? b : 0.0));
}

__device__ __forceinline__ double warp_max(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const double u = __shfl_xor_sync(0xffffffffu, v, o); v = u > v ? u : v; }
    return v;
}

// per-fit HBM scratch, in bytes: gradient memory [l][K], previous weights [d K], the cumulative sums [l] x 2, seen [l]
__host__ __device__ inline size_t sag_scratch_bytes(int l, int dk, int K, int tsize)
{
    const size_t a = ((size_t)l * K * tsize + 255) & ~(size_t)255, b = ((size_t)dk * tsize + 255) & ~(size_t)255;
    const size_t c = ((size_t)l * tsize + 255) & ~(size_t)255, e = ((size_t)l + 255) & ~(size_t)255;
    return a + b + 2 * c + e;
}

// lagged_update of every weight of this lane (the shortcut or the unrolled prox loop, as scikit-learn picks them).
// sample_itr and fh as scikit-learn's; cum / cump = cumulative_sums[sample_itr - 1] - cumulative_sums[fh - 1] and the prox
// sums alike; the replay (more than one lagged step) reads the arrays cs / csp.
template <int S, typename T>
__device__ __forceinline__ void sag_lagged(double (&w)[S], const double (&sg)[S], int dk, int lane, bool prox, int sample_itr,
                                           int fh, double cum, double cump, const T *cs, const T *csp)
{
#pragma unroll
    for (int i = 0; i < S; i++) {
        if (lane + 32 * i >= dk) continue;
        if (!prox) { w[i] = rnd<T>(__dsub_rn(w[i], rnd<T>(__dmul_rn(cum, sg[i])))); continue; }
        if (fabs(rnd<T>(__dmul_rn(sg[i], cum))) < cump) {
            w[i] = soft_threshold<T>(rnd<T>(__dsub_rn(w[i], rnd<T>(__dmul_rn(cum, sg[i])))), cump);
        } else {
            for (int li = sample_itr - 1; li > fh - 1; li--) {       // one step but after a rescale at an epoch's last sample
                double gs = cum, ps = cump;
                if (sample_itr - fh > 1) {
                    gs = li > 0 ? rnd<T>(__dsub_rn((double)cs[li], (double)cs[li - 1])) : (double)cs[li];
                    ps = li > 0 ? rnd<T>(__dsub_rn((double)csp[li], (double)csp[li - 1])) : (double)csp[li];
                }
                w[i] = soft_threshold<T>(rnd<T>(__dsub_rn(w[i], rnd<T>(__dmul_rn(sg[i], gs)))), ps);
            }
        }
    }
}

template <int S, typename T>
__global__ void __launch_bounds__(SAG_WARPS * 32)
sag_kernel(const SagFit *__restrict__ fits, int nfits, const T *__restrict__ X, int d, int K, int loss, const int *__restrict__ yc,
           const double *__restrict__ z, const double *__restrict__ sw, const double *__restrict__ cw, int nc,
           const int *__restrict__ order, unsigned char *__restrict__ scratch, size_t fit_stride, double tol, int max_iter,
           int fit_intercept, double *__restrict__ V, int nvp, int *__restrict__ n_iter_out, int *__restrict__ status_out,
           long long *__restrict__ stats)
{
    extern __shared__ double sag_sh[];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.x * SAG_WARPS + wid;
    if (f >= nfits) return;                                   // whole warps only: nothing below syncs the block
    const long long t_begin = clock64();
    const int dk = d * K, kp = (K + 1) & ~1;
    double *prod = sag_sh + (size_t)wid * (((dk + 1) & ~1) + 3 * kp), *predS = prod + ((dk + 1) & ~1), *pS = predS + kp,
           *gcS = pS + kp;
    const SagFit F = fits[f];
    const int l = F.l;
    unsigned char *scr = scratch + (size_t)f * fit_stride;
    T *gm = (T *)scr;
    T *prev = (T *)(scr + (((size_t)l * K * sizeof(T) + 255) & ~(size_t)255));
    T *cs = (T *)((unsigned char *)prev + (((size_t)dk * sizeof(T) + 255) & ~(size_t)255));
    T *csp = (T *)((unsigned char *)cs + (((size_t)l * sizeof(T) + 255) & ~(size_t)255));
    unsigned char *seen = (unsigned char *)csp + (((size_t)l * sizeof(T) + 255) & ~(size_t)255);
    const double *cwk = F.cwset >= 0 ? cw + (size_t)F.cwset * nc : nullptr;

    int fk[S];                                                  // slot i: (feature << 8) | class
    double w[S], sg[S], xs[S];
#pragma unroll
    for (int i = 0; i < S; i++) {
        const int q = lane + 32 * i, fe = q < dk ? q / K : 0;
        fk[i] = q < dk ? (fe << 8) | (q - fe * K) : 0;
        w[i] = 0.0; sg[i] = 0.0;
    }
    double icpt[2] = {0.0, 0.0}, isg[2] = {0.0, 0.0};
    const bool prox = F.beta > 0 && F.saga;
    const double step = F.step, wsu = rnd<T>(__dsub_rn(1.0, __dmul_rn(step, F.alpha))), stepbeta = __dmul_rn(step, F.beta);
    double wscale = 1.0, cs_last = 0.0, cs_fh = 0.0, csp_last = 0.0, csp_fh = 0.0;
    int fh = 0, num_seen = 0, status = 1, epoch;
    uint32_t seed = F.seed;
    long long steps = 0;

    // scale_weights at sample_itr = s: the lagged update with reset (and the non-finite check), feature_hist = (s + 1) % l,
    // cumulative_sums[s] = 0, wscale = 1.  Returns false on a non-finite weight.
    auto rescale = [&](int s) -> bool {
        const double cum = fh != 0 ? rnd<T>(__dsub_rn(cs_last, cs_fh)) : cs_last;
        const double cump = fh != 0 ? rnd<T>(__dsub_rn(csp_last, csp_fh)) : csp_last;
        sag_lagged<S, T>(w, sg, dk, lane, prox, s + 1, fh, cum, cump, cs, csp);
        bool bad = false;
#pragma unroll
        for (int i = 0; i < S; i++) {
            if (lane + 32 * i >= dk) continue;
            w[i] = rnd<T>(__dmul_rn(w[i], wscale));
            bad |= !isfinite(w[i]);
        }
        if (__any_sync(0xffffffffu, bad)) return false;
        fh = (s + 1) % l;
        cs_last = 0.0; cs_fh = 0.0; csp_last = 0.0; csp_fh = 0.0;
        if (prox && lane == 0) { cs[s] = (T)0; csp[s] = (T)0; }
        wscale = 1.0;
        return true;
    };

    for (epoch = 0; epoch < max_iter; epoch++) {
        int s;
        for (s = 0; s < l; s++) {
            steps++;
            const int pos = (int)(our_rand_r(seed) % (uint32_t)l);
            const int r = order[F.off + pos];
            const T *xr = X + (size_t)r * d;
#pragma unroll
            for (int i = 0; i < S; i++) xs[i] = lane + 32 * i < dk ? (double)xr[fk[i] >> 8] : 0.0;
            const int ycl = yc ? yc[r] : 0;
            const double y = loss == GS_SAG_SQUARED ? rnd<T>(z[r]) : (loss == GS_SAG_LOG ? (ycl == 1 ? 1.0 : 0.0) : (double)ycl);
            double swT = sw ? rnd<T>(sw[r]) : 1.0;
            if (cwk) swT = rnd<T>(__dmul_rn(swT, rnd<T>(cwk[ycl])));
            int sn = lane == 0 ? (int)seen[pos] : 0;
            sn = __shfl_sync(0xffffffffu, sn, 0);
            if (!sn) { num_seen++; if (lane == 0) seen[pos] = 1; }

            // ---- lagged_update ----
            if (s > 0) {
                const double cum = fh != 0 ? rnd<T>(__dsub_rn(cs_last, cs_fh)) : cs_last;
                const double cump = fh != 0 ? rnd<T>(__dsub_rn(csp_last, csp_fh)) : csp_last;
                if (prox && s - fh > 1) __syncwarp();                 // the replay reads lane 0's cumulative sums
                sag_lagged<S, T>(w, sg, dk, lane, prox, s, fh, cum, cump, cs, csp);
                fh = s; cs_fh = cs_last; csp_fh = csp_last;
            }
            // ---- predict_sample: class k's sum in feature order, by lane k ----
            __syncwarp();
#pragma unroll
            for (int i = 0; i < S; i++) {
                const int q = lane + 32 * i;
                if (q < dk) prod[q] = rnd<T>(__dmul_rn(w[i], xs[i]));
            }
            __syncwarp();
            double pred[2] = {0.0, 0.0};
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int k = lane + 32 * h;
                if (k < K) pred[h] = rnd<T>(__dadd_rn(rnd<T>(__dmul_rn(wscale, seq_sum<T>(prod + k, d, K))), icpt[h]));
            }
            // ---- the gradient of class k, by lane k ----
            double g[2] = {0.0, 0.0};
            if (loss == GS_SAG_MULTINOMIAL) {                       // sum_exp_minus_max, then (p_k - (y == k)) sw
#pragma unroll
                for (int h = 0; h < 2; h++) if (lane + 32 * h < K) predS[lane + 32 * h] = pred[h];
                __syncwarp();
                double mx = predS[0];
                for (int k = 1; k < K; k++) if (mx < predS[k]) mx = predS[k];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int k = lane + 32 * h;
                    if (k < K) { g[h] = rnd<T>(exp(__dsub_rn(pred[h], mx))); pS[k] = g[h]; }
                }
                __syncwarp();
                double sum = 0.0;
                for (int k = 0; k < K; k++) sum = __dadd_rn(sum, pS[k]);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int k = lane + 32 * h;
                    if (k < K) {
                        g[h] = rnd<T>(__ddiv_rn(g[h], sum));
                        g[h] = rnd<T>(__dmul_rn(rnd<T>(__dsub_rn(g[h], y == (double)k ? 1.0 : 0.0)), swT));
                    }
                }
            } else if (lane == 0) {
                g[0] = rnd<T>(__dmul_rn(loss == GS_SAG_LOG ? grad_half_binomial(y, pred[0]) : __dsub_rn(pred[0], y), swT));
            }
            wscale = rnd<T>(__dmul_rn(wscale, wsu));
            const double omn = __dsub_rn(1.0, __ddiv_rn(1.0, (double)num_seen));
            double diff[2] = {0.0, 0.0};
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int k = lane + 32 * h;
                if (k < K) {
                    T *gmp = gm + (size_t)pos * K + k;
                    diff[h] = rnd<T>(__dsub_rn(g[h], (double)*gmp));
                    gcS[k] = diff[h];
                    *gmp = (T)g[h];
                }
            }
            __syncwarp();
            // ---- the sum of gradients and the SAGA correction ----
#pragma unroll
            for (int i = 0; i < S; i++) {
                if (lane + 32 * i >= dk) continue;
                const double gcx = rnd<T>(__dmul_rn(xs[i], gcS[fk[i] & 255]));
                if (F.saga) w[i] = rnd<T>(__dsub_rn(w[i], __ddiv_rn(__dmul_rn(__dmul_rn(gcx, step), omn), wscale)));
                sg[i] = rnd<T>(__dadd_rn(sg[i], gcx));
            }
            // ---- the intercept ----
            if (fit_intercept) {
                bool bad = false;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (lane + 32 * h >= K) continue;
                    isg[h] = rnd<T>(__dadd_rn(isg[h], diff[h]));
                    const double gci = rnd<T>(__dmul_rn(diff[h], __dmul_rn(step, omn)));
                    double dec = __dmul_rn(__ddiv_rn(__dmul_rn(step, isg[h]), (double)num_seen), 1.0);
                    if (F.saga) dec = __dadd_rn(dec, gci);
                    icpt[h] = rnd<T>(__dsub_rn(icpt[h], dec));
                    bad |= !isfinite(icpt[h]);
                }
                if (__any_sync(0xffffffffu, bad)) { status = 2; break; }
            }
            // ---- the cumulative sums ----
            {
                const double a = __ddiv_rn(step, rnd<T>(__dmul_rn(wscale, (double)num_seen)));
                cs_last = s == 0 ? rnd<T>(a) : rnd<T>(__dadd_rn(cs_last, a));
                if (prox) {
                    const double b = __ddiv_rn(stepbeta, wscale);
                    csp_last = s == 0 ? rnd<T>(b) : rnd<T>(__dadd_rn(csp_last, b));
                    if (lane == 0) { cs[s] = (T)cs_last; csp[s] = (T)csp_last; }
                }
            }
            if (wscale < 1e-9 && !rescale(s)) { status = 2; break; }
        }
        if (status == 2) break;
        if (prox) __syncwarp();
        if (!rescale(l - 1)) { status = 2; break; }
        // ---- the stop test: max |w - previous| / max |w| <= tol ----
        double mw = 0.0, mc = 0.0;
#pragma unroll
        for (int i = 0; i < S; i++) {
            const int q = lane + 32 * i;
            if (q >= dk) continue;
            const double a = fabs(w[i]), c = fabs(rnd<T>(__dsub_rn(w[i], (double)prev[q])));
            mw = a > mw ? a : mw;
            mc = c > mc ? c : mc;
            prev[q] = (T)w[i];
        }
        mw = warp_max(mw);
        mc = warp_max(mc);
        if ((mw != 0.0 && rnd<T>(__ddiv_rn(mc, mw)) <= tol) || (mw == 0.0 && mc == 0.0)) { status = 0; break; }
    }
    const int n_iter = status == 1 ? (max_iter > 0 ? max_iter : 1) : epoch + 1;
    const int nvK = nvp;
#pragma unroll
    for (int i = 0; i < S; i++) {
        const int q = lane + 32 * i;
        if (q < dk) V[((size_t)F.out * K + (fk[i] & 255)) * nvK + (fk[i] >> 8)] = w[i];
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
        if (lane + 32 * h < K) V[((size_t)F.out * K + lane + 32 * h) * nvK + d] = icpt[h];
    if (lane == 0) {
        n_iter_out[F.out] = n_iter;
        status_out[F.out] = status;
        if (stats) {
            stats[(size_t)F.out * 2 + 0] = steps;
            stats[(size_t)F.out * 2 + 1] = clock64() - t_begin;
        }
    }
}

__global__ void sag_draws_kernel(uint32_t seed, int n, int count, int *out)
{
    for (int i = 0; i < count; i++) out[i] = (int)(our_rand_r(seed) % (uint32_t)n);
}

size_t sag_smem(int dk, int K) { return (size_t)SAG_WARPS * (((dk + 1) & ~1) + 3 * ((K + 1) & ~1)) * sizeof(double); }

template <int S, typename T>
cudaError_t launch_sag_t(const SagFit *fits, int nfits, const T *X, int d, int K, int loss, const int *yc, const double *z,
                         const double *sw, const double *cw, int nc, const int *order, unsigned char *scratch, size_t stride,
                         double tol, int max_iter, int fi, double *V, int nvp, int *n_iter, int *status, long long *stats,
                         cudaStream_t st)
{
    const size_t smem = sag_smem(d * K, K);
    const dim3 grid((nfits + SAG_WARPS - 1) / SAG_WARPS), block(SAG_WARPS * 32);
    cudaFuncSetAttribute(sag_kernel<S, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    sag_kernel<S, T><<<grid, block, smem, st>>>(fits, nfits, X, d, K, loss, yc, z, sw, cw, nc, order, scratch, stride, tol,
                                                 max_iter, fi, V, nvp, n_iter, status, stats);
    return cudaGetLastError();
}

template <typename T>
cudaError_t launch_sag(int s, const SagFit *fits, int nfits, const T *X, int d, int K, int loss, const int *yc, const double *z,
                       const double *sw, const double *cw, int nc, const int *order, unsigned char *scratch, size_t stride,
                       double tol, int max_iter, int fi, double *V, int nvp, int *n_iter, int *status, long long *stats,
                       cudaStream_t st)
{
#define SAG_CASE(N) if (s <= N) return launch_sag_t<N, T>(fits, nfits, X, d, K, loss, yc, z, sw, cw, nc, order, scratch, stride, tol, max_iter, fi, V, nvp, n_iter, status, stats, st)
    SAG_CASE(1); SAG_CASE(2); SAG_CASE(4); SAG_CASE(8); SAG_CASE(MAX_S);
#undef SAG_CASE
    return cudaErrorInvalidValue;
}

// refit: one fit on every row (in row order), ns = 1; coef_out [K][d + 1], n_iter / status [1]
int sag_run(gs_handle *h, int n_cand, const int32_t *solver, const double *alpha_scaled, const double *beta_scaled,
            const double *step, const uint32_t *seed, int loss, double tol, int max_iter, int fit_intercept, bool refit,
            double *test_scores, double *train_scores, int32_t *n_iter, int32_t *fit_status, double *coef_out, int64_t *stats_out,
            float *ms_solve, float *ms_score)
{
    const char *who = refit ? "gs_logreg_sag_refit" : "gs_logreg_sag";
    auto fail = [&](int code, const std::string &msg) { gs_set_error(h, std::string(who) + ": " + msg); return code; };
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) return fail(GS_ERR_NO_DATA, "no dataset (call gs_set_data first)");
    const bool cls = h->classification;
    if (loss != GS_SAG_LOG && loss != GS_SAG_MULTINOMIAL && loss != GS_SAG_SQUARED) return fail(GS_ERR_ARG, "loss code out of range");
    if (loss == GS_SAG_SQUARED) {
        if (cls || h->z64.empty()) return fail(GS_ERR_NO_DATA, "the squared loss needs float64 targets (gs_set_targets_f64 after a regression gs_set_data)");
        if (!coef_out) return fail(GS_ERR_ARG, "the squared loss reports coef_out only (it is NULL)");
        if (h->class_w_sets > 0) return fail(GS_ERR_ARG, "class weights do not apply to the squared loss");
    } else {
        if (!cls) return fail(GS_ERR_ARG, "the logistic losses need class labels");
        if (h->n_classes < 2) return fail(GS_ERR_UNSUPPORTED, "needs at least two classes");
        if (h->n_classes > 64) return fail(GS_ERR_UNSUPPORTED, "more than 64 classes is not supported");
        if ((loss == GS_SAG_LOG) != (h->n_classes == 2)) return fail(GS_ERR_ARG, "'log' is the binary loss, 'multinomial' the loss of three or more classes");
    }
    const int ns = refit ? 1 : h->n_splits;
    if (n_cand <= 0 || !solver || !alpha_scaled || !beta_scaled || !step || !seed || std::isnan(tol) || max_iter < 0)
        return fail(GS_ERR_ARG, "bad arguments");
    for (int t = 0; t < n_cand * ns; t++) {
        if (solver[t] != GS_SAG_SOLVER_SAG && solver[t] != GS_SAG_SOLVER_SAGA) return fail(GS_ERR_ARG, "solver must be GS_SAG_SOLVER_SAG or GS_SAG_SOLVER_SAGA");
        if (!(alpha_scaled[t] >= 0) || !std::isfinite(alpha_scaled[t]) || !(beta_scaled[t] >= 0) || !std::isfinite(beta_scaled[t]))
            return fail(GS_ERR_ARG, "alpha_scaled and beta_scaled must be finite and >= 0");
        if (!(step[t] > 0) || !std::isfinite(step[t])) return fail(GS_ERR_ARG, "step must be finite and > 0");
    }
    const int nc = cls ? h->n_classes : 1;
    const int K = loss == GS_SAG_MULTINOMIAL ? nc : 1;
    const int n = (int)h->n, d = (int)h->d, dk = d * K;
    if (dk > GS_SAG_MAX_COEF) return fail(GS_ERR_UNSUPPORTED, "features x weight rows above GS_SAG_MAX_COEF (" + std::to_string(GS_SAG_MAX_COEF) + ")");
    const int kind = refit || !cls ? GS_SCORE_DEFAULT : h->score_kind;
    if (int e = check_scorer(h, who, kind)) return e;
    if (int e = check_class_weight_sets(h, who, ns)) return e;
    const bool weighted = cls && h->class_w_sets > 0;
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int S = std::max(1, (dk + 31) / 32);
    const int nvp = (int)round_up(d + 1, 64);
    const int64_t npad = round_up(n, 64);
    const bool has_sw = !h->sample_w.empty();
    const bool f64 = h->x_dtype == GS_F64;
    const int tsize = f64 ? 8 : 4;

    // ---- every split's training rows in the splitter's order (internal rows); zero-weight rows stay (they count in n) ----
    std::vector<int> order, sp_off;
    const int lmax = train_rows(h, ns, refit, false, order, sp_off);
    if (lmax == 0) return fail(GS_ERR_UNSUPPORTED, "a split has no training row");

    const int nfit = n_cand * ns;
    std::vector<SagFit> hf(nfit);
    for (int c = 0; c < n_cand; c++)
        for (int k = 0; k < ns; k++) {
            const int t = c * ns + k;
            SagFit &F = hf[t];
            F.off = sp_off[k]; F.l = sp_off[k + 1] - sp_off[k]; F.out = t;
            F.cwset = weighted ? (h->class_w_sets == 1 ? 0 : k) : -1;
            F.seed = seed[t]; F.saga = solver[t] == GS_SAG_SOLVER_SAGA;
            F.step = step[t]; F.alpha = alpha_scaled[t]; F.beta = beta_scaled[t];
        }
    const int mpad = (int)round_up((int64_t)nfit * K, 64);

    h->evp.reset(); h->tt.reset();
    cudaEvent_t ev[3];
    for (auto &e : ev) e = h->evp.get();
    cudaEventRecord(ev[0], st);

    DevBuf &bXa = h->dWork[0], &bZ = h->dWork[1], &bFit = h->dWork[2], &bScr = h->dWork[3], &bOut = h->dWork[4];
    const size_t xa_elems = (size_t)npad * nvp;
    GS_CUDA(bXa.reserve((xa_elems * 2 + (size_t)n + (size_t)std::max(1, h->class_w_sets) * nc) * 8));
    double *dXa = bXa.as<double>(), *dXat = dXa + xa_elems, *dSw = dXat + xa_elems, *dCw = dSw + n;
    const size_t fit_bytes = (size_t)nfit * sizeof(SagFit);
    GS_CUDA(bFit.reserve(round_up(fit_bytes, 256) + order.size() * 4 + 256));
    SagFit *dFits = bFit.as<SagFit>();
    int *dOrder = reinterpret_cast<int *>(bFit.as<unsigned char>() + round_up(fit_bytes, 256));
    GS_CUDA(bOut.reserve((size_t)mpad * nvp * 8 + (size_t)nfit * (2 * 8 + 8) + 256));
    double *dV = bOut.as<double>();
    long long *dStats = reinterpret_cast<long long *>(dV + (size_t)mpad * nvp);
    int *dIter = reinterpret_cast<int *>(dStats + (size_t)nfit * 2), *dStatus = dIter + nfit;
    GS_CUDA(cudaMemsetAsync(dV, 0, (size_t)mpad * nvp * 8, st));
    GS_CUDA(cudaMemcpyAsync(dFits, hf.data(), fit_bytes, cudaMemcpyHostToDevice, st));
    GS_CUDA(cudaMemcpyAsync(dOrder, order.data(), order.size() * 4, cudaMemcpyHostToDevice, st));
    if (has_sw) GS_CUDA(cudaMemcpyAsync(dSw, h->sample_w64.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    if (weighted) GS_CUDA(cudaMemcpyAsync(dCw, h->class_w.data(), h->class_w.size() * 8, cudaMemcpyHostToDevice, st));

    // ---- the fits, in waves that fit the free device memory ----
    const size_t stride = round_up((int64_t)sag_scratch_bytes(lmax, dk, K, tsize), 256);
    size_t free_b = 0, total_b = 0;
    GS_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t budget = free_b / 10 * 7 + bScr.cap;
    const int wave = (int)std::max<size_t>(1, std::min<size_t>((size_t)nfit, budget / stride));
    GS_CUDA(bScr.reserve((size_t)wave * stride));
    const float *X32 = h->dX.as<float>();
    const double *X64 = f64 ? h->dX64.as<double>() : nullptr;
    const int *Yc = cls ? h->dY.as<int>() : nullptr;
    const double *Z = cls ? nullptr : h->dZ64.as<double>();
    int64_t launches = 0;
    for (int first = 0; first < nfit; first += wave) {
        const int cnt = std::min(wave, nfit - first);
        GS_CUDA(cudaMemsetAsync(bScr.p, 0, (size_t)cnt * stride, st));
        const cudaError_t e = f64 ? launch_sag<double>(S, dFits + first, cnt, X64, d, K, loss, Yc, Z, has_sw ? dSw : nullptr, weighted ? dCw : nullptr, nc, dOrder, bScr.as<unsigned char>(), stride, tol, max_iter, fit_intercept, dV, nvp, dIter, dStatus, dStats, st)
                                  : launch_sag<float>(S, dFits + first, cnt, X32, d, K, loss, Yc, Z, has_sw ? dSw : nullptr, weighted ? dCw : nullptr, nc, dOrder, bScr.as<unsigned char>(), stride, tol, max_iter, fit_intercept, dV, nvp, dIter, dStatus, dStats, st);
        GS_CUDA(e);
        launches++;
    }
    cudaEventRecord(ev[1], st);

    std::vector<int> iters(nfit), status(nfit);
    std::vector<long long> stats((size_t)nfit * 2);
    GS_CUDA(cudaMemcpyAsync(iters.data(), dIter, (size_t)nfit * 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaMemcpyAsync(status.data(), dStatus, (size_t)nfit * 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaMemcpyAsync(stats.data(), dStats, stats.size() * 8, cudaMemcpyDeviceToHost, st));
    std::vector<double> wraw;
    if (coef_out) {
        wraw.resize((size_t)nfit * K * nvp);
        GS_CUDA(cudaMemcpyAsync(wraw.data(), dV, wraw.size() * 8, cudaMemcpyDeviceToHost, st));
    }

    // ---- scoring: decision values [X | 1] . [coef | intercept] of every fit in one FP64 contraction ----
    const bool score = !refit && cls;
    if (score) {
        GS_CUDA(launch_build_xa64(f64 ? nullptr : X32, X64, n, d, 1.0, nvp, npad, dXa, dXat, st));
        launches++;
        GS_CUDA(bZ.reserve((size_t)mpad * npad * 8));
        if (int e = score_linear_fits(h, dV, dXa, bZ.as<double>(), nfit, K, ns, kind, test_scores, train_scores, ev[2], launches)) return e;
    } else {
        cudaEventRecord(ev[2], st);
        GS_CUDA(cudaStreamSynchronize(st));
    }

    for (int f = 0; f < nfit; f++) {
        if (score && status[f] == 2) { test_scores[f] = NAN; if (train_scores) train_scores[f] = NAN; }   // a non-finite fit
        if (n_iter) n_iter[f] = iters[f];
        if (fit_status) fit_status[f] = status[f];
        if (coef_out)
            for (int q = 0; q < K; q++)
                for (int j = 0; j <= d; j++) coef_out[((size_t)f * K + q) * (d + 1) + j] = wraw[((size_t)f * K + q) * nvp + j];
        if (stats_out) for (int e = 0; e < 2; e++) stats_out[(size_t)f * 2 + e] = stats[(size_t)f * 2 + e];
    }
    linear_profile(h, ev, launches, ms_solve, ms_score);
    int64_t total = 0;
    for (int t = 0; t < nfit; t++) total += stats[(size_t)t * 2];
    h->prof.smo_iterations = total;                                  // SAG sample steps
    return GS_OK;
}

}  // namespace

extern "C" {

int gs_logreg_sag(gs_handle *h, int32_t n_cand, const int32_t *solver, const double *alpha_scaled, const double *beta_scaled,
                  const double *step, const uint32_t *seed, int32_t loss, double tol, int32_t max_iter, int32_t fit_intercept,
                  uint32_t flags, double *test_scores, double *train_scores, int32_t *n_iter, int32_t *fit_status, float *fit_ms,
                  float *score_ms, double *coef_out, int64_t *stats)
{
    if (h && !test_scores && loss != GS_SAG_SQUARED) { gs_set_error(h, "gs_logreg_sag: test_scores is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    const int st = sag_run(h, n_cand, solver, alpha_scaled, beta_scaled, step, seed, loss, tol, max_iter, fit_intercept, false,
                           test_scores, (flags & GS_RETURN_TRAIN) ? train_scores : nullptr, n_iter, fit_status, coef_out, stats,
                           &a, &b);
    if (st) return st;
    spread_call_ms(n_cand * h->n_splits, a, b, fit_ms, score_ms);
    return GS_OK;
}

int gs_logreg_sag_refit(gs_handle *h, int32_t solver, double alpha_scaled, double beta_scaled, double step, uint32_t seed,
                        int32_t loss, double tol, int32_t max_iter, int32_t fit_intercept, double *coef_out, int32_t *n_iter,
                        int32_t *fit_status)
{
    if (h && !coef_out) { gs_set_error(h, "gs_logreg_sag_refit: coef_out is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    return sag_run(h, 1, &solver, &alpha_scaled, &beta_scaled, &step, &seed, loss, tol, max_iter, fit_intercept, true, nullptr,
                   nullptr, n_iter, fit_status, coef_out, nullptr, &a, &b);
}

int gs_debug_sag_draws(gs_handle *h, uint32_t seed, int32_t n, int32_t count, int32_t *out)
{
    if (!h) return GS_ERR_ARG;
    if (n <= 0 || count <= 0 || !out) { gs_set_error(h, "gs_debug_sag_draws: bad arguments"); return GS_ERR_ARG; }
    GS_CUDA(cudaSetDevice(h->device));
    GS_CUDA(h->dScore.reserve((size_t)count * 4));
    sag_draws_kernel<<<1, 1, 0, h->stream>>>(seed, n, count, h->dScore.as<int>());
    GS_CUDA(cudaGetLastError());
    GS_CUDA(cudaMemcpyAsync(out, h->dScore.p, (size_t)count * 4, cudaMemcpyDeviceToHost, h->stream));
    GS_CUDA(cudaStreamSynchronize(h->stream));
    return GS_OK;
}

}  // extern "C"
