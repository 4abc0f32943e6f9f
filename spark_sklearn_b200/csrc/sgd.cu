// sgd.cu -- batched SGDClassifier / SGDRegressor: scikit-learn's plain SGD restated step for step, one warp per fit.
//
// Replaces (reference base_search.py:83-87 -> sklearn _fit_and_score -> SGDClassifier / SGDRegressor .fit / score):
//   linear_model/_stochastic_gradient.py      fit_binary (binary: one fit, y = +1 for classes_[1]; one-vs-rest: one fit per
//                                             class, negatives weighted 1.0), _fit_regressor; seeds drawn on the host
//   linear_model/_sgd_fast.pyx.tp _plain_sgd  the sample loop: dot, learning rate, objective, class x sample weight, the
//                                             L2 scale, add, intercept, the L1 truncated gradient, the stop rule, the
//                                             adaptive eta / 5, the non-finite check after every epoch
//   utils/_weight_vector.pyx.tp               WeightVector: w times wscale, reset below 1e-9 (float64) / 1e-6 (float32),
//                                             add() recomputing sq_norm and l1_norm over every feature
//   utils/_seq_dataset.pyx.tp shuffle          Fisher-Yates on xorshift32 (our_rand_r) with the seed passed by value: every
//                                             epoch applies the same swaps, so epoch e's order is epoch e-1's gathered
//                                             through one permutation pi, drawn once per fit (sgd_draw_perm)
//
// A fit is one warp.  w (and q, the L1 bookkeeping) live in registers: lane L holds features L, L + 32, ...  Every lane
// computes the same scalars.  The sums scikit-learn makes in feature order -- the dot product and add()'s squared and
// absolute norms -- are made in that order: each lane writes its terms to shared memory and every lane adds them up in
// sequence (broadcast reads), so a fit equals scikit-learn's bit for bit wherever the arithmetic is IEEE (no contraction;
// log_loss's exp / log1p and invscaling's pow come from CUDA's math library).  The norms feed only the objective, so they
// are summed only when the stop rule reads a penalised objective, and a sample's norms are summed together with the next
// sample's dot product (two independent chains in one loop).  float32 X runs _plain_sgd32: w, q, y, the weights and the
// float copies WeightVector32 makes (wscale in add() and reset_wscale(), norm(), l1norm()) are float32 values, while its
// wscale, sq_norm and l1_norm stay double; every operation scikit-learn rounds to float is rounded to float (a float
// operation made in double and rounded once gives the float result: 53 >= 2 x 24 + 2).
// The training order and the scoring of the final weights are linear_search.cu's (train_rows, score_linear_fits).
#include "common.cuh"
#include "sequential.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

constexpr int SGD_WARPS = 4;           // fits per block
constexpr int MAX_NT = GS_SGD_MAX_FEATURES / 32;
enum { OPTIMAL = 2, INVSCALING = 3, ADAPTIVE = 4 };

struct SgdCand {
    int loss, penalty, lr;
    double alpha, l1_ratio, lparam, eta0, power_t, optimal_init;   // lparam: hinge threshold or epsilon
};

struct SgdFit {
    int off, l;            // training positions: order[off .. off + l), internal rows in the splitter's order
    int out;               // row of V / n_iter / status / stats: (candidate x split) x KC + class
    int cand;
    int pos;               // classifier: the class whose rows are +1 (log_loss: 1, others 0 / -1); regressor -1
    int ovr;               // one-vs-rest: the intercept is stored in intercept_[class], in X's dtype
    uint32_t seed;         // the shuffle seed
    double wpos, wneg;     // class weights of the +1 and the other rows
};

// sklearn's log1pexp (_loss.pyx.tp)
__host__ __device__ inline double log1pexp(double x)
{
    if (x <= -37) return exp(x);
    if (x <= -2) return log1p(exp(x));
    if (x <= 18) return log(1. + exp(x));
    if (x <= 33.3) return x + exp(-x);
    return x;
}

// loss(y, p) and its derivative in p, as _sgd_fast.pyx.tp / _loss.pyx.tp compute them (rounding op by op)
__host__ __device__ inline double sgd_dloss(int loss, double th, double y, double p)
{
    switch (loss) {
    case GS_SGD_HINGE: case GS_SGD_PERCEPTRON: return p * y <= th ? -y : 0.0;
    case GS_SGD_SQUARED_HINGE: { const double z = th - p * y; return z > 0 ? -2 * y * z : 0.0; }
    case GS_SGD_MODIFIED_HUBER: {
        const double z = p * y;
        if (z >= 1.0) return 0.0;
        if (z >= -1.0) return 2.0 * (1.0 - z) * -y;
        return -4.0 * y;
    }
    case GS_SGD_LOG_LOSS:
        if (p > -37) { const double e = exp(-p); return ((1 - y) - y * e) / (1 + e); }
        return exp(p) - y;
    case GS_SGD_SQUARED_ERROR: return p - y;
    case GS_SGD_HUBER: { const double r = p - y; return fabs(r) <= th ? r : (r >= 0 ? th : -th); }
    case GS_SGD_EPSILON_INSENSITIVE: return y - p > th ? -1.0 : (p - y > th ? 1.0 : 0.0);
    default: {                                                   // squared_epsilon_insensitive
        const double z = y - p;
        if (z > th) return -2 * (z - th);
        if (z < -th) return 2 * (-z - th);
        return 0.0;
    }
    }
}

__device__ __forceinline__ double sgd_loss(int loss, double th, double y, double p)
{
    switch (loss) {
    case GS_SGD_HINGE: case GS_SGD_PERCEPTRON: { const double z = __dmul_rn(p, y); return z <= th ? __dsub_rn(th, z) : 0.0; }
    case GS_SGD_SQUARED_HINGE: { const double z = __dsub_rn(th, __dmul_rn(p, y)); return z > 0 ? __dmul_rn(z, z) : 0.0; }
    case GS_SGD_MODIFIED_HUBER: {
        const double z = __dmul_rn(p, y);
        if (z >= 1.0) return 0.0;
        if (z >= -1.0) return __dmul_rn(__dsub_rn(1.0, z), __dsub_rn(1.0, z));
        return __dmul_rn(-4.0, z);
    }
    case GS_SGD_LOG_LOSS: return __dsub_rn(log1pexp(p), __dmul_rn(y, p));
    case GS_SGD_SQUARED_ERROR: return __dmul_rn(__dmul_rn(0.5, __dsub_rn(p, y)), __dsub_rn(p, y));
    case GS_SGD_HUBER: {
        const double a = fabs(__dsub_rn(y, p));
        return a <= th ? __dmul_rn(0.5, __dmul_rn(a, a)) : __dmul_rn(th, __dsub_rn(a, __dmul_rn(0.5, th)));
    }
    case GS_SGD_EPSILON_INSENSITIVE: { const double r = __dsub_rn(fabs(__dsub_rn(y, p)), th); return r > 0 ? r : 0.0; }
    default: { const double r = __dsub_rn(fabs(__dsub_rn(y, p)), th); return r > 0 ? __dmul_rn(r, r) : 0.0; }
    }
}

// the device copy of sgd_dloss with every operation rounded on its own
__device__ __forceinline__ double sgd_dloss_rn(int loss, double th, double y, double p)
{
    switch (loss) {
    case GS_SGD_HINGE: case GS_SGD_PERCEPTRON: return __dmul_rn(p, y) <= th ? -y : 0.0;
    case GS_SGD_SQUARED_HINGE: { const double z = __dsub_rn(th, __dmul_rn(p, y)); return z > 0 ? __dmul_rn(__dmul_rn(-2.0, y), z) : 0.0; }
    case GS_SGD_MODIFIED_HUBER: {
        const double z = __dmul_rn(p, y);
        if (z >= 1.0) return 0.0;
        if (z >= -1.0) return __dmul_rn(__dmul_rn(2.0, __dsub_rn(1.0, z)), -y);
        return __dmul_rn(-4.0, y);
    }
    case GS_SGD_LOG_LOSS: return grad_half_binomial(y, p);
    case GS_SGD_SQUARED_ERROR: return __dsub_rn(p, y);
    case GS_SGD_HUBER: { const double r = __dsub_rn(p, y); return fabs(r) <= th ? r : (r >= 0 ? th : -th); }
    case GS_SGD_EPSILON_INSENSITIVE: return __dsub_rn(y, p) > th ? -1.0 : (__dsub_rn(p, y) > th ? 1.0 : 0.0);
    default: {
        const double z = __dsub_rn(y, p);
        if (z > th) return __dmul_rn(-2.0, __dsub_rn(z, th));
        if (z < -th) return __dmul_rn(2.0, __dsub_rn(-z, th));
        return 0.0;
    }
    }
}

// pi: ArrayDataset.shuffle(seed) applied to the identity over l positions (Fisher-Yates, our_rand_r), one thread
__device__ void sgd_draw_perm(uint32_t seed, int l, int *perm)
{
    for (int i = 0; i < l; i++) perm[i] = i;
    uint32_t s = seed;
    for (int i = 0; i < l - 1; i++) {
        const int j = i + (int)(our_rand_r(s) % (uint32_t)(l - i));
        const int a = perm[i];
        perm[i] = perm[j];
        perm[j] = a;
    }
}

template <int NT, typename T, bool L1>
__global__ void __launch_bounds__(SGD_WARPS * 32)
sgd_kernel(const SgdFit *__restrict__ fits, int nfits, const SgdCand *__restrict__ cands, const T *__restrict__ X, int d,
           const int *__restrict__ yc, const double *__restrict__ z, const double *__restrict__ sw, const int *__restrict__ order,
           int *__restrict__ idx_all, int64_t lstride, double tol, int max_iter, int n_iter_no_change, int fit_intercept,
           int shuffle, double *__restrict__ V, int nvp, int *__restrict__ n_iter_out, int *__restrict__ status_out,
           long long *__restrict__ stats)
{
    extern __shared__ double sgd_sh[];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.x * SGD_WARPS + wid;
    if (f >= nfits) return;                                   // whole warps only: nothing below syncs the block
    const long long t_begin = clock64();
    const int dp = (d + 1) & ~1;
    double *sd = sgd_sh + (size_t)wid * 3 * dp, *s2 = sd + dp, *s3 = s2 + dp;
    const SgdFit F = fits[f];
    const SgdCand P = cands[F.cand];
    const int l = F.l;
    int *perm = idx_all + (size_t)f * 3 * lstride, *cur = perm + lstride, *nxt = cur + lstride;
    for (int i = lane; i < l; i += 32) cur[i] = order[F.off + i];
    long long shuffle_cycles = 0;
    if (shuffle) {
        const long long t0 = clock64();
        if (lane == 0) sgd_draw_perm(F.seed, l, perm);
        shuffle_cycles += clock64() - t0;
    }
    __syncwarp();

    const bool is_log = P.loss == GS_SGD_LOG_LOSS;
    const int pen = P.penalty;
    const double alpha = P.alpha, th = P.lparam;
    const double l1r = pen == GS_SGD_L2 ? 0.0 : (pen == GS_SGD_L1 ? 1.0 : P.l1_ratio);
    const bool need_obj = tol > -HUGE_VAL;                     // the objective only feeds the stop rule
    const bool need_norms = need_obj && pen != GS_SGD_NONE;
    const double thresh = sizeof(T) == 4 ? 1e-6 : 1e-9;
    const double wposT = rnd<T>(F.wpos), wnegT = rnd<T>(F.wneg);
    auto target = [&](int r) -> double {
        if (F.pos < 0) return rnd<T>(z[r]);
        return yc[r] == F.pos ? 1.0 : (is_log ? 0.0 : -1.0);
    };

    T w[NT], q[NT];
#pragma unroll
    for (int t = 0; t < NT; t++) { w[t] = 0; q[t] = 0; }
    double wscale = 1.0, sq_norm = 0.0, l1_norm = 0.0, pend_ws = 1.0;
    bool pend = false;
    double intercept = 0.0, tt = 1.0, eta = P.eta0, u = 0.0;
    double best = HUGE_VAL;
    int nic = 0, epoch = 0, status = 1;
    long long steps = 0;

    for (epoch = 0; epoch < max_iter; epoch++) {
        double obj = 0.0;
        if (shuffle) {                                         // this epoch's order: the last one gathered through pi
            const long long t0 = clock64();
            for (int i = lane; i < l; i += 32) nxt[i] = cur[perm[i]];
            int *s = cur; cur = nxt; nxt = s;
            __syncwarp();
            shuffle_cycles += clock64() - t0;
        }
        T xn[NT];
        int rn = cur[0];
        {
            const T *xr = X + (size_t)rn * d;
#pragma unroll
            for (int t = 0; t < NT; t++) { const int j = lane + 32 * t; xn[t] = j < d ? xr[j] : (T)0; }
        }
        for (int i = 0; i < l; i++) {
            steps++;
            const int r = rn;
            T x[NT];
#pragma unroll
            for (int t = 0; t < NT; t++) x[t] = xn[t];
            const double y = target(r), swT = sw ? rnd<T>(sw[r]) : 1.0;
            if (i + 1 < l) {                                   // the next position's row, loaded during this step
                rn = cur[i + 1];
                const T *xr = X + (size_t)rn * d;
#pragma unroll
                for (int t = 0; t < NT; t++) { const int j = lane + 32 * t; xn[t] = j < d ? xr[j] : (T)0; }
            }
            // ---- p = w.dot(x) + intercept; the norms of the last add() ----
            __syncwarp();
#pragma unroll
            for (int t = 0; t < NT; t++) {
                const int j = lane + 32 * t;
                if (j < d) sd[j] = rnd<T>(__dmul_rn((double)w[t], (double)x[t]));
            }
            __syncwarp();
            double dot;
            if (pend) {
                double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll 4
                for (int j = 0; j < d; j++) {
                    a0 = __dadd_rn(a0, sd[j]);
                    a1 = __dadd_rn(a1, s2[j]);
                    a2 = __dadd_rn(a2, s3[j]);
                }
                dot = a0;
                sq_norm = __dmul_rn(a1, rnd<T>(__dmul_rn(pend_ws, pend_ws)));
                l1_norm = __dmul_rn(a2, pend_ws);
                pend = false;
            } else {
                dot = seq_sum<double>(sd, d, 1);
            }
            const double p = __dadd_rn(rnd<T>(__dmul_rn(dot, wscale)), intercept);
            if (P.lr == OPTIMAL) eta = __ddiv_rn(1.0, __dmul_rn(alpha, __dsub_rn(__dadd_rn(P.optimal_init, tt), 1.0)));
            else if (P.lr == INVSCALING) eta = __ddiv_rn(P.eta0, pow(tt, P.power_t));
            if (need_obj) {
                obj = __dadd_rn(obj, sgd_loss(P.loss, th, y, p));
                if (pen != GS_SGD_NONE) {
                    const double nrm = rnd<T>(sqrt(sq_norm));
                    obj = __dadd_rn(obj, __dmul_rn(alpha, __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(1.0, l1r), 0.5), __dmul_rn(nrm, nrm)),
                                                                    __dmul_rn(l1r, rnd<T>(l1_norm)))));
                }
            }
            const double cw = y > 0.0 ? wposT : wnegT;
            double dl = sgd_dloss_rn(P.loss, th, y, p);
            dl = dl < -1e12 ? -1e12 : (dl > 1e12 ? 1e12 : dl);
            double update = __dmul_rn(-eta, dl);
            update = __dmul_rn(update, rnd<T>(__dmul_rn(cw, swT)));
            if (pen == GS_SGD_L2 || pen == GS_SGD_ELASTICNET) {   // w.scale(max(0, 1 - (1 - l1_ratio) eta alpha))
                double c = __dsub_rn(1.0, __dmul_rn(__dmul_rn(__dsub_rn(1.0, l1r), eta), alpha));
                c = rnd<T>(c > 0 ? c : 0.0);
                wscale = __dmul_rn(wscale, c);
                if (need_norms) {
                    sq_norm = __dmul_rn(sq_norm, rnd<T>(__dmul_rn(c, c)));
                    l1_norm = __dmul_rn(l1_norm, fabs(c));
                }
                if (wscale < thresh) {                        // reset_wscale: scal by wscale in X's dtype
                    const double wsf = rnd<T>(wscale);
#pragma unroll
                    for (int t = 0; t < NT; t++) w[t] = (T)rnd<T>(__dmul_rn((double)w[t], wsf));
                    wscale = 1.0;
                }
            }
            if (update != 0.0) {                              // w.add(x, update)
                const double wsf = rnd<T>(wscale), cu = rnd<T>(__ddiv_rn(rnd<T>(update), wsf));
#pragma unroll
                for (int t = 0; t < NT; t++) w[t] = (T)rnd<T>(__dadd_rn((double)w[t], __dmul_rn((double)x[t], cu)));
                if (need_norms) {
                    __syncwarp();
#pragma unroll
                    for (int t = 0; t < NT; t++) {
                        const int j = lane + 32 * t;
                        if (j < d) { s2[j] = rnd<T>(__dmul_rn((double)w[t], (double)w[t])); s3[j] = fabs((double)w[t]); }
                    }
                    pend = true;
                    pend_ws = wsf;
                }
                if (fit_intercept) intercept = __dadd_rn(intercept, update);
            }
            if (L1) {                                         // l1penalty: truncated gradient with the q / u bookkeeping
                u = __dadd_rn(u, __dmul_rn(__dmul_rn(l1r, eta), alpha));
#pragma unroll
                for (int t = 0; t < NT; t++) {
                    const double zz = (double)w[t];
                    double nw = zz;
                    if (__dmul_rn(wscale, zz) > 0.0) {
                        const double v = __dsub_rn(zz, __ddiv_rn(__dadd_rn(u, (double)q[t]), wscale));
                        nw = rnd<T>(v > 0.0 ? v : 0.0);
                    } else if (__dmul_rn(wscale, zz) < 0.0) {
                        const double v = __dadd_rn(zz, __ddiv_rn(__dsub_rn(u, (double)q[t]), wscale));
                        nw = rnd<T>(v < 0.0 ? v : 0.0);
                    }
                    w[t] = (T)nw;
                    q[t] = (T)rnd<T>(__dadd_rn((double)q[t], __dmul_rn(wscale, __dsub_rn(nw, zz))));
                }
            }
            tt = __dadd_rn(tt, 1.0);
        }
        // ---- the epoch's checks: non-finite weights, then the stop rule ----
        bool bad = !isfinite(intercept);
#pragma unroll
        for (int t = 0; t < NT; t++) bad |= !isfinite((double)w[t]);
        if (__any_sync(0xffffffffu, bad)) { status = 2; break; }
        const double mean = __ddiv_rn(obj, (double)l);
        if (need_obj && mean > __dsub_rn(best, tol)) nic++;
        else nic = 0;
        if (mean < best) best = mean;
        if (nic >= n_iter_no_change) {
            if (P.lr == ADAPTIVE && eta > 1e-6) { eta = __ddiv_rn(eta, 5.0); nic = 0; }
            else { status = 0; break; }
        }
    }
    const int n_iter = status == 1 ? max_iter : epoch + 1;
#pragma unroll
    for (int t = 0; t < NT; t++) {
        const int j = lane + 32 * t;
        if (j < d) V[(size_t)F.out * nvp + j] = rnd<T>(__dmul_rn((double)w[t], rnd<T>(wscale)));   // reset_wscale
    }
    if (lane == 0) {
        V[(size_t)F.out * nvp + d] = F.ovr ? rnd<T>(intercept) : intercept;
        n_iter_out[F.out] = n_iter;
        status_out[F.out] = status;
        if (stats) {
            stats[(size_t)F.out * 3 + 0] = steps;
            stats[(size_t)F.out * 3 + 1] = shuffle_cycles;
            stats[(size_t)F.out * 3 + 2] = clock64() - t_begin;
        }
    }
}

__global__ void sgd_perm_kernel(uint32_t seed, int l, int *out) { sgd_draw_perm(seed, l, out); }

template <int NT, typename T>
cudaError_t launch_sgd_t(bool l1, const SgdFit *fits, int nfits, const SgdCand *cands, const T *X, int d, const int *yc,
                         const double *z, const double *sw, const int *order, int *idx, int64_t lstride, double tol, int max_iter,
                         int nic, int fi, int shuffle, double *V, int nvp, int *n_iter, int *status, long long *stats,
                         cudaStream_t st)
{
    const size_t smem = (size_t)SGD_WARPS * 3 * ((d + 1) & ~1) * sizeof(double);
    const dim3 grid((nfits + SGD_WARPS - 1) / SGD_WARPS), block(SGD_WARPS * 32);
    if (l1) {
        cudaFuncSetAttribute(sgd_kernel<NT, T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        sgd_kernel<NT, T, true><<<grid, block, smem, st>>>(fits, nfits, cands, X, d, yc, z, sw, order, idx, lstride, tol, max_iter,
                                                           nic, fi, shuffle, V, nvp, n_iter, status, stats);
    } else {
        cudaFuncSetAttribute(sgd_kernel<NT, T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        sgd_kernel<NT, T, false><<<grid, block, smem, st>>>(fits, nfits, cands, X, d, yc, z, sw, order, idx, lstride, tol, max_iter,
                                                            nic, fi, shuffle, V, nvp, n_iter, status, stats);
    }
    return cudaGetLastError();
}

template <typename T>
cudaError_t launch_sgd(int nt, bool l1, const SgdFit *fits, int nfits, const SgdCand *cands, const T *X, int d, const int *yc,
                       const double *z, const double *sw, const int *order, int *idx, int64_t lstride, double tol, int max_iter,
                       int nic, int fi, int shuffle, double *V, int nvp, int *n_iter, int *status, long long *stats, cudaStream_t st)
{
#define SGD_CASE(K) if (nt <= K) return launch_sgd_t<K, T>(l1, fits, nfits, cands, X, d, yc, z, sw, order, idx, lstride, tol, max_iter, nic, fi, shuffle, V, nvp, n_iter, status, stats, st)
    SGD_CASE(1); SGD_CASE(2); SGD_CASE(3); SGD_CASE(4); SGD_CASE(6); SGD_CASE(8); SGD_CASE(12); SGD_CASE(MAX_NT);
#undef SGD_CASE
    return cudaErrorInvalidValue;
}

// refit: one fit on every row (in row order), ns = 1; coef_out [KC][d + 1], n_iter / status [KC]
int sgd_run(gs_handle *h, int n_cand, const int32_t *loss, const int32_t *penalty, const double *alpha, const double *l1_ratio,
            const double *epsilon, const int32_t *lr, const double *eta0, const double *power_t, const uint32_t *seed, double tol,
            int max_iter, int n_iter_no_change, int fit_intercept, int shuffle, bool refit, double *test_scores, double *train_scores,
            int32_t *n_iter, int32_t *fit_status, double *coef_out, int64_t *stats_out, float *ms_solve, float *ms_score)
{
    const char *who = refit ? "gs_sgd_refit" : "gs_sgd";
    auto fail = [&](int code, const std::string &msg) { gs_set_error(h, std::string(who) + ": " + msg); return code; };
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) return fail(GS_ERR_NO_DATA, "no dataset (call gs_set_data first)");
    const bool cls = h->classification;
    if (cls && h->n_classes < 2) return fail(GS_ERR_UNSUPPORTED, "needs at least two classes");
    if (cls && h->n_classes > 64) return fail(GS_ERR_UNSUPPORTED, "more than 64 classes is not supported");
    if (!cls && h->z64.empty()) return fail(GS_ERR_NO_DATA, "no float64 targets (call gs_set_targets_f64 after gs_set_data)");
    if (!cls && h->class_w_sets > 0) return fail(GS_ERR_ARG, "class weights do not apply to a regressor");
    if (n_cand <= 0 || !loss || !penalty || !alpha || !l1_ratio || !epsilon || !lr || !eta0 || !power_t || !seed ||
        std::isnan(tol) || tol == HUGE_VAL || max_iter < 1 || n_iter_no_change < 1)
        return fail(GS_ERR_ARG, "bad arguments");
    if (h->d > GS_SGD_MAX_FEATURES) return fail(GS_ERR_UNSUPPORTED, "more than " + std::to_string(GS_SGD_MAX_FEATURES) + " features");
    for (int c = 0; c < n_cand; c++) {
        if (cls ? !(loss[c] >= 0 && loss[c] <= GS_SGD_SQUARED_EPSILON_INSENSITIVE) : !(loss[c] >= GS_SGD_SQUARED_ERROR && loss[c] <= GS_SGD_SQUARED_EPSILON_INSENSITIVE))
            return fail(GS_ERR_ARG, "loss code out of range for this dataset");
        if (penalty[c] < GS_SGD_NONE || penalty[c] > GS_SGD_ELASTICNET) return fail(GS_ERR_ARG, "penalty code out of range");
        if (lr[c] < 1 || lr[c] > 4) return fail(GS_ERR_ARG, "learning_rate must be constant, optimal, invscaling or adaptive");
        if (!(alpha[c] >= 0) || !std::isfinite(alpha[c]) || (lr[c] == OPTIMAL && !(alpha[c] > 0))) return fail(GS_ERR_ARG, "alpha must be >= 0 (> 0 with 'optimal') and finite");
        if (!(l1_ratio[c] >= 0 && l1_ratio[c] <= 1)) return fail(GS_ERR_ARG, "l1_ratio must be in [0, 1]");
        if (!(epsilon[c] >= 0) || !std::isfinite(epsilon[c])) return fail(GS_ERR_ARG, "epsilon must be >= 0 and finite");
        if (!(eta0[c] >= 0) || !std::isfinite(eta0[c]) || !std::isfinite(power_t[c])) return fail(GS_ERR_ARG, "eta0 must be >= 0, eta0 and power_t finite");
    }
    const int kind = refit ? GS_SCORE_DEFAULT : h->score_kind;
    const int ns = refit ? 1 : h->n_splits, nc = cls ? h->n_classes : 1;
    const int KC = cls && nc > 2 ? nc : 1;
    if (int e = check_scorer(h, who, kind)) return e;
    if (int e = check_class_weight_sets(h, who, ns)) return e;
    const bool weighted = cls && h->class_w_sets > 0;
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int n = (int)h->n, d = (int)h->d;
    const int nt = std::max(1, (d + 31) / 32);
    const int nvp = (int)round_up(d + 1, 64);
    const int64_t npad = round_up(n, 64);
    const bool has_sw = !h->sample_w.empty();

    // ---- every split's training rows in the splitter's order (internal rows); zero-weight rows stay (they scale w) ----
    std::vector<int> order, sp_off;
    const int lmax = train_rows(h, ns, refit, false, order, sp_off);
    if (lmax == 0) return fail(GS_ERR_UNSUPPORTED, "a split has no training row");

    std::vector<SgdCand> hc(n_cand);
    for (int c = 0; c < n_cand; c++) {
        SgdCand &P = hc[c];
        P.loss = loss[c]; P.penalty = penalty[c]; P.lr = lr[c];
        P.alpha = alpha[c]; P.l1_ratio = l1_ratio[c]; P.eta0 = eta0[c]; P.power_t = power_t[c];
        P.lparam = loss[c] == GS_SGD_PERCEPTRON ? 0.0 : (loss[c] <= GS_SGD_LOG_LOSS ? 1.0 : epsilon[c]);
        P.optimal_init = 0.0;
        if (lr[c] == OPTIMAL) {                                   // _plain_sgd: eta of the first sample = typw / max(1, dloss(1, -typw))
            const double typw = std::sqrt(1.0 / std::sqrt(alpha[c]));
            const double g = sgd_dloss(loss[c], P.lparam, 1.0, -typw);
            const double initial_eta0 = typw / (g > 1.0 ? g : 1.0);
            P.optimal_init = 1.0 / (initial_eta0 * alpha[c]);
        }
    }
    std::vector<SgdFit> hf;
    hf.reserve((size_t)n_cand * ns * KC);
    for (int c = 0; c < n_cand; c++)
        for (int k = 0; k < ns; k++)
            for (int q = 0; q < KC; q++) {
                const int t = (c * ns + k) * KC + q;
                SgdFit F;
                F.off = sp_off[k]; F.l = sp_off[k + 1] - sp_off[k]; F.out = t; F.cand = c; F.seed = seed[t];
                F.pos = cls ? (KC == 1 ? 1 : q) : -1;
                F.ovr = KC > 1;
                const double *cw = weighted ? &h->class_w[(size_t)(h->class_w_sets == 1 ? 0 : k) * nc] : nullptr;
                F.wpos = cw ? cw[F.pos] : 1.0;                       // binary: cw[1] / cw[0]; one-vs-rest: cw[k] / 1.0
                F.wneg = cw && KC == 1 ? cw[0] : 1.0;
                hf.push_back(F);
            }
    // the instance with L1 bookkeeping carries q in registers: the fits are launched in two groups
    auto plain = [&](const SgdFit &F) { return penalty[F.cand] != GS_SGD_L1 && penalty[F.cand] != GS_SGD_ELASTICNET; };
    std::stable_partition(hf.begin(), hf.end(), plain);
    const int nfit_all = (int)hf.size(), nplain = (int)std::count_if(hf.begin(), hf.end(), plain);
    const int nfit = n_cand * ns;
    const int mpad = (int)round_up(nfit_all, 64);

    h->evp.reset(); h->tt.reset();
    cudaEvent_t ev[3];
    for (auto &e : ev) e = h->evp.get();
    cudaEventRecord(ev[0], st);

    DevBuf &bXa = h->dWork[0], &bZ = h->dWork[1], &bFit = h->dWork[2], &bIdx = h->dWork[3], &bOut = h->dWork[4];
    const size_t xa_elems = (size_t)npad * nvp;
    GS_CUDA(bXa.reserve((xa_elems * 2 + (size_t)n) * 8));
    double *dXa = bXa.as<double>(), *dXat = dXa + xa_elems, *dSw = dXat + xa_elems;
    const size_t fit_bytes = (size_t)nfit_all * sizeof(SgdFit), cand_bytes = (size_t)n_cand * sizeof(SgdCand);
    GS_CUDA(bFit.reserve(round_up(fit_bytes, 256) + round_up(cand_bytes, 256) + order.size() * 4 + 256));
    SgdFit *dFits = bFit.as<SgdFit>();
    SgdCand *dCands = reinterpret_cast<SgdCand *>(bFit.as<unsigned char>() + round_up(fit_bytes, 256));
    int *dOrder = reinterpret_cast<int *>(bFit.as<unsigned char>() + round_up(fit_bytes, 256) + round_up(cand_bytes, 256));
    const int64_t lstride = round_up(lmax, 32);
    GS_CUDA(bIdx.reserve((size_t)nfit_all * 3 * lstride * 4));
    GS_CUDA(bOut.reserve((size_t)mpad * nvp * 8 + (size_t)nfit_all * (3 * 8 + 8) + 256));
    double *dV = bOut.as<double>();
    long long *dStats = reinterpret_cast<long long *>(dV + (size_t)mpad * nvp);
    int *dIter = reinterpret_cast<int *>(dStats + (size_t)nfit_all * 3), *dStatus = dIter + nfit_all;
    GS_CUDA(cudaMemsetAsync(dV, 0, (size_t)mpad * nvp * 8, st));
    GS_CUDA(cudaMemcpyAsync(dFits, hf.data(), fit_bytes, cudaMemcpyHostToDevice, st));
    GS_CUDA(cudaMemcpyAsync(dCands, hc.data(), cand_bytes, cudaMemcpyHostToDevice, st));
    GS_CUDA(cudaMemcpyAsync(dOrder, order.data(), order.size() * 4, cudaMemcpyHostToDevice, st));
    if (has_sw) GS_CUDA(cudaMemcpyAsync(dSw, h->sample_w64.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    const bool f64 = h->x_dtype == GS_F64;
    const float *X32 = h->dX.as<float>();
    const double *X64 = f64 ? h->dX64.as<double>() : nullptr;
    const int *Yc = cls ? h->dY.as<int>() : nullptr;
    const double *Z = cls ? nullptr : h->dZ64.as<double>();
    const double *SW = has_sw ? dSw : nullptr;
    int64_t launches = 0;
    for (int g = 0; g < 2; g++) {
        const int first = g ? nplain : 0, cnt = g ? nfit_all - nplain : nplain;
        if (!cnt) continue;
        int *idx = bIdx.as<int>() + (size_t)first * 3 * lstride;
        const cudaError_t e = f64 ? launch_sgd<double>(nt, g == 1, dFits + first, cnt, dCands, X64, d, Yc, Z, SW, dOrder, idx, lstride, tol, max_iter, n_iter_no_change, fit_intercept, shuffle, dV, nvp, dIter, dStatus, dStats, st)
                                  : launch_sgd<float>(nt, g == 1, dFits + first, cnt, dCands, X32, d, Yc, Z, SW, dOrder, idx, lstride, tol, max_iter, n_iter_no_change, fit_intercept, shuffle, dV, nvp, dIter, dStatus, dStats, st);
        GS_CUDA(e);
        launches++;
    }
    cudaEventRecord(ev[1], st);

    std::vector<int> iters(nfit_all), status(nfit_all);
    std::vector<long long> stats((size_t)nfit_all * 3);
    GS_CUDA(cudaMemcpyAsync(iters.data(), dIter, (size_t)nfit_all * 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaMemcpyAsync(status.data(), dStatus, (size_t)nfit_all * 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaMemcpyAsync(stats.data(), dStats, stats.size() * 8, cudaMemcpyDeviceToHost, st));
    std::vector<double> wraw;
    if (coef_out) {
        wraw.resize((size_t)nfit_all * nvp);
        GS_CUDA(cudaMemcpyAsync(wraw.data(), dV, wraw.size() * 8, cudaMemcpyDeviceToHost, st));
    }

    // ---- scoring: decision values [X | 1] . [coef | intercept] of every fit in one FP64 contraction ----
    if (!refit) {
        GS_CUDA(launch_build_xa64(f64 ? nullptr : X32, X64, n, d, 1.0, nvp, npad, dXa, dXat, st));
        launches++;
        GS_CUDA(bZ.reserve((size_t)mpad * npad * 8));
        if (int e = score_linear_fits(h, dV, dXa, bZ.as<double>(), nfit, KC, ns, kind, test_scores, train_scores, ev[2], launches)) return e;
    } else {
        cudaEventRecord(ev[2], st);
        GS_CUDA(cudaStreamSynchronize(st));
    }

    // n_iter / status per (candidate, split): the maximum over the classes; a non-finite class fit (the first in class
    // order, as one-vs-rest raises it) gives status 2, its epoch and NaN scores.  The refit reports each class.
    for (int f = 0; f < nfit; f++)
        for (int q = 0; q < KC; q++) {
            const int t = f * KC + q;
            if (refit) {
                if (n_iter) n_iter[q] = iters[t];
                if (fit_status) fit_status[q] = status[t];
            }
            if (coef_out) for (int j = 0; j <= d; j++) coef_out[(size_t)t * (d + 1) + j] = wraw[(size_t)t * nvp + j];
            if (stats_out) for (int e = 0; e < 3; e++) stats_out[(size_t)t * 3 + e] = stats[(size_t)t * 3 + e];
        }
    if (!refit)
        for (int f = 0; f < nfit; f++) {
            int it = 0, s = 1, bad_it = 0;
            bool stopped_all = true, bad = false;
            for (int q = 0; q < KC; q++) {
                const int t = f * KC + q;
                it = std::max(it, iters[t]);
                if (status[t] == 2 && !bad) { bad = true; bad_it = iters[t]; }
                stopped_all &= status[t] == 0;
            }
            s = bad ? 2 : (stopped_all ? 0 : 1);
            if (n_iter) n_iter[f] = bad ? bad_it : it;
            if (fit_status) fit_status[f] = s;
            if (bad) { test_scores[f] = NAN; if (train_scores) train_scores[f] = NAN; }
        }
    linear_profile(h, ev, launches, ms_solve, ms_score);
    int64_t total = 0;
    for (int t = 0; t < nfit_all; t++) total += stats[(size_t)t * 3];
    h->prof.smo_iterations = total;                                  // SGD samples processed
    return GS_OK;
}

}  // namespace

extern "C" {

int gs_sgd(gs_handle *h, int32_t n_cand, const int32_t *loss, const int32_t *penalty, const double *alpha, const double *l1_ratio,
           const double *epsilon, const int32_t *learning_rate, const double *eta0, const double *power_t, const uint32_t *seed,
           double tol, int32_t max_iter, int32_t n_iter_no_change, int32_t fit_intercept, int32_t shuffle, uint32_t flags,
           double *test_scores, double *train_scores, int32_t *n_iter, int32_t *fit_status, float *fit_ms, float *score_ms,
           double *coef_out, int64_t *stats)
{
    if (h && !test_scores) { gs_set_error(h, "gs_sgd: test_scores is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    const int st = sgd_run(h, n_cand, loss, penalty, alpha, l1_ratio, epsilon, learning_rate, eta0, power_t, seed, tol, max_iter,
                           n_iter_no_change, fit_intercept, shuffle, false, test_scores, (flags & GS_RETURN_TRAIN) ? train_scores : nullptr,
                           n_iter, fit_status, coef_out, stats, &a, &b);
    if (st) return st;
    spread_call_ms(n_cand * h->n_splits, a, b, fit_ms, score_ms);
    return GS_OK;
}

int gs_sgd_refit(gs_handle *h, int32_t loss, int32_t penalty, double alpha, double l1_ratio, double epsilon, int32_t learning_rate,
                 double eta0, double power_t, const uint32_t *seed, double tol, int32_t max_iter, int32_t n_iter_no_change,
                 int32_t fit_intercept, int32_t shuffle, double *coef_out, int32_t *n_iter, int32_t *fit_status)
{
    if (h && (!coef_out || !seed)) { gs_set_error(h, "gs_sgd_refit: coef_out or seed is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    return sgd_run(h, 1, &loss, &penalty, &alpha, &l1_ratio, &epsilon, &learning_rate, &eta0, &power_t, seed, tol, max_iter,
                   n_iter_no_change, fit_intercept, shuffle, true, nullptr, nullptr, n_iter, fit_status, coef_out, nullptr, &a, &b);
}

int gs_debug_sgd_perm(gs_handle *h, uint32_t seed, int32_t l, int32_t *out)
{
    if (!h) return GS_ERR_ARG;
    if (l <= 0 || !out) { gs_set_error(h, "gs_debug_sgd_perm: bad arguments"); return GS_ERR_ARG; }
    GS_CUDA(cudaSetDevice(h->device));
    GS_CUDA(h->dScore.reserve((size_t)l * 4));
    sgd_perm_kernel<<<1, 1, 0, h->stream>>>(seed, l, h->dScore.as<int>());
    GS_CUDA(cudaGetLastError());
    GS_CUDA(cudaMemcpyAsync(out, h->dScore.p, (size_t)l * 4, cudaMemcpyDeviceToHost, h->stream));
    GS_CUDA(cudaStreamSynchronize(h->stream));
    return GS_OK;
}

}  // extern "C"
