// linsvr.cu -- batched LinearSVR: liblinear's dual coordinate descent (solvers 12 and 13) one warp per fit, and its primal
// TRON (solver 11) on the FP64 tensor-core contractions of linsvc.cu.
//
// Replaces (reference base_search.py:83-87 -> sklearn _fit_and_score -> LinearSVR.fit/score):
//   sklearn/svm/_classes.py LinearSVR.fit      dual resolved per training set; coef_ = raw[:d], intercept_ = scaling x raw[d]
//   sklearn/svm/_base.py _fit_liblinear        seed = check_random_state(random_state).randint(INT_MAX), bias = scaling
//   liblinear linear.cpp train                 remove_zero_weight (order kept); one train_one on the remaining rows
//   linear.cpp solve_l2r_l1l2_svr              the dual CD, restated step for step in linsvr_cd_kernel:
//                                              12 (squared loss): lambda_i = 0.5 / C_i, no bound; 13: lambda 0, |beta_i| <= C_i;
//                                              per epoch a Fisher-Yates shuffle of the active set (bounded_rand_int on
//                                              std::mt19937), shrinking against Gmax_old, the |d| < 1e-12 skip, the clip,
//                                              and the stop Gnorm1 <= eps Gnorm1_init that unshrinks while the set is not full
//   linear.cpp l2r_l2_svr_fun + tron.cpp        solver 11: linsvr_pointwise_kernel between the two contractions, TRON itself
//                                              is linsvc.cu's tron_advance_kernel, its rounds linear_search.cu's TronRounds
//
// A CD fit is one warp.  w lives in registers (lane L holds features L, L + 32, ...; the bias is feature d), beta and the
// index permutation live in HBM (beta by internal row, the permutation as internal rows), the mt19937 state in shared memory.
// Every lane computes the same scalars: the dot product is a per-lane sequential sum and an xor butterfly, whose result is
// the same on all lanes, so the update, the shrink decision and the stores need no broadcast.  Scalar arithmetic is rounded
// operation by operation as liblinear's (no contraction); only the dot product's summation order differs from liblinear,
// which accumulates the row into G in feature order (tests/linsvr_oracle.c restates both orders).
// The training order and the scoring of the final weights are linear_search.cu's (train_rows, score_linear_fits).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int CD_WARPS = 4;            // fits per block
constexpr int MAX_NT = 17;             // 17 x 32 = 544 >= 512 features + the bias
constexpr int MT_N = 624;

__device__ __forceinline__ uint32_t mt_temper(uint32_t y)
{
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

// std::mt19937 held by one warp: state in shared memory, the next outputs buffered one per lane (lanes [0, have) valid).
struct WarpMt {
    uint32_t *mt;
    int used;                          // outputs of the current state block already pulled into the buffer
    uint32_t buf;
    int have;

    __device__ void seed(uint32_t s, int lane)
    {
        if (lane == 0) {
            mt[0] = s;
            for (int i = 1; i < MT_N; i++) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
        }
        __syncwarp();
        used = MT_N; have = 0; buf = 0;
    }
    // the generation step, 32 words at a time: word i reads words i + 1 (not yet rewritten, or word 0 for i = 623, already
    // rewritten as in the sequential loop) and i + 397 (old for i < 227) or i - 227 (rewritten in an earlier chunk)
    __device__ void twist(int lane)
    {
        for (int c = 0; c < (MT_N + 31) / 32; c++) {
            const int i = c * 32 + lane;
            uint32_t nv = 0;
            if (i < MT_N) {
                const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1 == MT_N ? 0 : i + 1] & 0x7fffffffu);
                nv = mt[i < MT_N - 397 ? i + 397 : i - (MT_N - 397)] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
            }
            __syncwarp();
            if (i < MT_N) mt[i] = nv;
            __syncwarp();
        }
    }
    // fill lanes [have, 32) with the next outputs of the stream
    __device__ void refill(int lane)
    {
        const int need = 32 - have, k = lane - have;
        uint32_t raw = 0;
        if (k >= 0 && used + k < MT_N) raw = mt[used + k];
        if (used + need > MT_N) {
            twist(lane);
            if (k >= 0 && used + k >= MT_N) raw = mt[used + k - MT_N];
            used = used + need - MT_N;
        } else {
            used += need;
        }
        __syncwarp();
        if (k >= 0) buf = mt_temper(raw);
        have = 32;
    }
    __device__ void consume(int take)
    {
        buf = __shfl_down_sync(FULL, buf, take);
        have -= take;
    }
};

struct CdFit {
    int off, l;            // the fit's training rows: order[off .. off + l), internal rows in liblinear's position order
    int out;               // row of V / n_iter / stats
    uint32_t seed;
    double C, p;           // C and epsilon
};

__device__ __forceinline__ double warp_sum_rn(double v)
{
#pragma unroll
    for (int m = 16; m; m >>= 1) v = __dadd_rn(v, __shfl_xor_sync(FULL, v, m));
    return v;
}

template <int NT, bool L1, typename TX>
__global__ void __launch_bounds__(CD_WARPS * 32)
linsvr_cd_kernel(const CdFit *__restrict__ fits, int nfits, const TX *__restrict__ X, int d, double bias,
                 const int *__restrict__ order, const double *__restrict__ QD, const double *__restrict__ y,
                 const double *__restrict__ W, double *__restrict__ beta_all, int *__restrict__ index_all, int64_t idx_stride,
                 int n, double eps, int max_iter, double *__restrict__ V, int nvp, int *__restrict__ n_iter_out,
                 long long *__restrict__ stats)
{
    __shared__ uint32_t mts[CD_WARPS][MT_N];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.x * CD_WARPS + wid;
    if (f >= nfits) return;                                   // whole warps only: nothing below syncs the block
    const long long t_begin = clock64();
    const CdFit F = fits[f];
    const int l = F.l;
    double *beta = beta_all + (size_t)f * n;
    int *index = index_all + (size_t)f * idx_stride;
    for (int i = lane; i < l; i += 32) {
        const int r = order[F.off + i];
        index[i] = r;
        beta[r] = 0.0;
    }
    WarpMt rng;
    rng.mt = mts[wid];
    rng.seed(F.seed, lane);                                   // ends in __syncwarp: index / beta are visible to every lane
    const double C = F.C, p = F.p;
    // a row's part of this lane's features (the bias is feature d) and its scalars: beta, y, C_i = W_i C, QD
    auto load_row = [&](int row, double (&xx)[NT], double &b, double &yy, double &cc, double &qq) {
        const TX *xr = X + (size_t)row * d;
#pragma unroll
        for (int t = 0; t < NT; t++) {
            const int j = lane + 32 * t;
            xx[t] = j < d ? (double)xr[j] : (j == d ? bias : 0.0);
        }
        b = beta[row];
        yy = y[row];
        cc = W ? __dmul_rn(W[row], C) : C;                    // C_[i] = W[i] * C
        qq = QD[row];
    };

    double w[NT];
#pragma unroll
    for (int t = 0; t < NT; t++) w[t] = 0.0;
    int iter = 0, active = l;
    double Gmax_old = HUGE_VAL, Gnorm1_init = -1.0;
    long long steps = 0, shuffle_cycles = 0;

    while (iter < max_iter) {
        double Gmax_new = 0, Gnorm1_new = 0;
        // ---- for i in [0, active): swap(index[i], index[i + bounded_rand_int(active - i)]) ----
        const long long t0 = clock64();
        for (int i0 = 0; i0 < active;) {
            if (rng.have < 32) rng.refill(lane);
            const bool valid = i0 + lane < active;
            const uint32_t r = valid ? (uint32_t)(active - i0 - lane) : 1u;
            const uint64_t m = (uint64_t)rng.buf * (uint64_t)r;
            const uint32_t lo = (uint32_t)m;
            bool rej = false;
            if (valid && lo < r) rej = lo < (0u - r) % r;     // Lemire's rejection: the output is redrawn
            const unsigned rm = __ballot_sync(FULL, rej);
            const int nvalid = min(32, active - i0);
            const int q = rm ? __ffs(rm) - 1 : nvalid;        // draws of this batch that stand
            const int jj = i0 + lane + (int)(m >> 32);
            for (int k = 0; k < q; k++) {
                const int j = __shfl_sync(FULL, jj, k), a = i0 + k;
                const int va = index[a], vj = index[j];
                index[a] = vj;
                index[j] = va;
            }
            i0 += q;
            rng.consume(rm ? q + 1 : nvalid);
        }
        shuffle_cycles += clock64() - t0;

        // ---- one pass over the active set.  Each step loads its own row: loading the next position's row during the
        // current step measured slower on an H100 (1304 against 1161 SM cycles per step on linsvr_c). ----
        int s = 0;
        int cur = active > 0 ? index[0] : 0;
        while (s < active) {
            steps++;
            const int row = cur;
            const int nxt = s + 1 < active ? index[s + 1] : 0;   // the next position, or
            const int last = index[active - 1];                  // the row a shrink swaps in
            double x[NT], b, yi, Ci, qd;
            load_row(row, x, b, yi, Ci, qd);
            double part = 0.0;
#pragma unroll
            for (int t = 0; t < NT; t++) part = __dadd_rn(part, __dmul_rn(w[t], x[t]));
            part = warp_sum_rn(part);
            const double lambda = L1 ? 0.0 : __ddiv_rn(0.5, Ci);
            const double ub = L1 ? Ci : HUGE_VAL;
            double G = __dadd_rn(-yi, __dmul_rn(lambda, b));
            const double H = __dadd_rn(qd, lambda);
            G = __dadd_rn(G, part);
            const double Gp = __dadd_rn(G, p), Gn = __dsub_rn(G, p);
            double violation = 0;
            bool shrink = false;
            if (b == 0) {
                if (Gp < 0) violation = -Gp;
                else if (Gn > 0) violation = Gn;
                else if (Gp > Gmax_old && Gn < -Gmax_old) shrink = true;
            } else if (b >= ub) {
                if (Gp > 0) violation = Gp;
                else if (Gp < -Gmax_old) shrink = true;
            } else if (b <= -ub) {
                if (Gn < 0) violation = -Gn;
                else if (Gn > Gmax_old) shrink = true;
            } else if (b > 0) violation = fabs(Gp);
            else violation = fabs(Gn);
            if (shrink) {                                        // swap(index[s], index[--active]); the same s again
                active--;
                index[s] = last;
                index[active] = row;
                cur = last;
                continue;
            }
            Gmax_new = Gmax_new < violation ? violation : Gmax_new;
            Gnorm1_new = __dadd_rn(Gnorm1_new, violation);
            const double Hb = __dmul_rn(H, b);
            double dd;
            if (Gp < Hb) dd = __ddiv_rn(-Gp, H);
            else if (Gn > Hb) dd = __ddiv_rn(-Gn, H);
            else dd = -b;
            s++;
            cur = nxt;
            if (fabs(dd) < 1.0e-12) continue;
            double nb = __dadd_rn(b, dd);
            nb = nb < -ub ? -ub : nb;                            // max(beta + d, -ub)
            nb = ub < nb ? ub : nb;                              // min(., ub)
            dd = __dsub_rn(nb, b);
            beta[row] = nb;
            if (dd != 0) {
#pragma unroll
                for (int t = 0; t < NT; t++)
                    if (x[t] != 0) w[t] = __dadd_rn(w[t], __dmul_rn(dd, x[t]));
            }
        }
        if (iter == 0) Gnorm1_init = Gnorm1_new;
        iter++;
        if (Gnorm1_new <= __dmul_rn(eps, Gnorm1_init)) {
            if (active == l) break;
            active = l;
            Gmax_old = HUGE_VAL;
            continue;
        }
        Gmax_old = Gmax_new;
    }
#pragma unroll
    for (int t = 0; t < NT; t++) {
        const int j = lane + 32 * t;
        if (j < nvp) V[(size_t)F.out * nvp + j] = w[t];
    }
    if (lane == 0) {
        n_iter_out[F.out] = iter;
        if (stats) {
            stats[(size_t)F.out * 3 + 0] = steps;
            stats[(size_t)F.out * 3 + 1] = shuffle_cycles;
            stats[(size_t)F.out * 3 + 2] = clock64() - t_begin;
        }
    }
}

// QD[r] = ||x_r||^2 + bias^2, summed in liblinear's order (features ascending, then the bias), one thread per row
template <typename TX>
__global__ void linsvr_qd_kernel(const TX *__restrict__ X, int n, int d, double bias, double *__restrict__ QD)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    double s = 0.0;
    for (int j = 0; j < d; j++) {
        const double v = (double)X[(size_t)r * d + j];
        s = __dadd_rn(s, __dmul_rn(v, v));
    }
    if (bias > 0) s = __dadd_rn(s, __dmul_rn(bias, bias));
    QD[r] = s;
}

// the first k outputs of std::mt19937(seed), drawn by WarpMt (one warp)
__global__ void linsvr_mt_kernel(uint32_t seed, int k, uint32_t *out)
{
    __shared__ uint32_t st[MT_N];
    const int lane = threadIdx.x & 31;
    WarpMt rng;
    rng.mt = st;
    rng.seed(seed, lane);
    for (int i0 = 0; i0 < k; i0 += 32) {
        rng.refill(lane);
        if (i0 + lane < k) out[i0 + lane] = rng.buf;
        rng.consume(32);
    }
}

struct SvrCol {            // per TRON column: its split and the fit's C and epsilon
    int fold;
    double C, p;
};

// l2r_l2_svr_fun between the two contractions (the file comment of linsvc.cu): fun mode: d = z - y, loss partials
// C_i (d + p)^2 for d < -p and C_i (d - p)^2 for d > p, residual C_i (d -/+ p) on that set, which becomes the spare mask;
// Hv mode: R = C_i (X s) on the current set.  Rows outside the split's training set or of zero weight take no part.
__global__ void linsvr_pointwise_kernel(const double *__restrict__ Zt, int64_t ldz, int n, const double *__restrict__ y,
                                        SplitMasks sm, const double *__restrict__ W, const TrState *__restrict__ St,
                                        const SvrCol *__restrict__ cols, unsigned char *__restrict__ mask, int64_t mask_stride,
                                        double *__restrict__ R, double *__restrict__ fpart)
{
    __shared__ double sh[256];
    const int c = blockIdx.y;
    const TrState &S = St[c];
    const int mode = S.mode;
    const SvrCol col = cols[c];
    const unsigned char *mcur = mask + (size_t)S.cur * mask_stride + (size_t)c * ldz;
    unsigned char *mnext = mask + (size_t)(S.cur ^ 1) * mask_stride + (size_t)c * ldz;
    double acc = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const size_t idx = (size_t)c * ldz + i;
        double res = 0.0;
        if (mode != M_DONE && split_train(sm, i, col.fold) && W[i] > 0) {
            const double Ci = __dmul_rn(col.C, W[i]);
            if (mode == M_FUN) {
                const double dz = __dsub_rn(Zt[idx], y[i]);
                bool act = false;
                if (dz < -col.p) {
                    const double e = __dadd_rn(dz, col.p);
                    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(Ci, e), e));
                    res = __dmul_rn(Ci, e);
                    act = true;
                } else if (dz > col.p) {
                    const double e = __dsub_rn(dz, col.p);
                    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(Ci, e), e));
                    res = __dmul_rn(Ci, e);
                    act = true;
                }
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

// final TRON weights (column c's w in Vec) -> row out[c] of the scoring submission V
__global__ void linsvr_scatter_w_kernel(const double *__restrict__ Vec, const int *__restrict__ out, int ncol, int nvp,
                                        double *__restrict__ V)
{
    const int c = blockIdx.x;
    if (c >= ncol) return;
    for (int j = threadIdx.x; j < nvp; j += blockDim.x) V[(size_t)out[c] * nvp + j] = Vec[(size_t)c * NVEC * nvp + j];
}

template <int NT, bool L1, typename TX>
cudaError_t launch_cd_t(const CdFit *fits, int nfits, const TX *X, int d, double bias, const int *order, const double *QD,
                        const double *y, const double *W, double *beta, int *index, int64_t idx_stride, int n, double eps,
                        int max_iter, double *V, int nvp, int *n_iter, long long *stats, cudaStream_t st)
{
    linsvr_cd_kernel<NT, L1, TX><<<(nfits + CD_WARPS - 1) / CD_WARPS, CD_WARPS * 32, 0, st>>>(
        fits, nfits, X, d, bias, order, QD, y, W, beta, index, idx_stride, n, eps, max_iter, V, nvp, n_iter, stats);
    return cudaGetLastError();
}

template <bool L1, typename TX>
cudaError_t launch_cd(int nt, const CdFit *fits, int nfits, const TX *X, int d, double bias, const int *order, const double *QD,
                      const double *y, const double *W, double *beta, int *index, int64_t idx_stride, int n, double eps,
                      int max_iter, double *V, int nvp, int *n_iter, long long *stats, cudaStream_t st)
{
#define CD_CASE(K) if (nt <= K) return launch_cd_t<K, L1, TX>(fits, nfits, X, d, bias, order, QD, y, W, beta, index, idx_stride, n, eps, max_iter, V, nvp, n_iter, stats, st)
    CD_CASE(1); CD_CASE(2); CD_CASE(3); CD_CASE(4); CD_CASE(6); CD_CASE(8); CD_CASE(12); CD_CASE(MAX_NT);
#undef CD_CASE
    return cudaErrorInvalidValue;
}

// solver[t] (t = c * ns + k): 11 TRON, 12 / 13 the dual CD.  refit: one fit on every row (ns = 1), coef_out [d + 1].
int linsvr_run(gs_handle *h, int n_cand, const double *Cv, const double *epsv, const int32_t *solver, const uint32_t *seed,
               double tol, int max_iter, int fit_intercept, double intercept_scaling, bool refit, double *test_scores,
               double *train_scores, int32_t *n_iter, double *coef_out, int64_t *cd_stats, float *ms_solve, float *ms_score)
{
    const char *who = refit ? "gs_linsvr_refit" : "gs_linsvr";
    auto fail = [&](int code, const std::string &msg) { gs_set_error(h, std::string(who) + ": " + msg); return code; };
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) return fail(GS_ERR_NO_DATA, "no dataset (call gs_set_data first)");
    if (h->classification) return fail(GS_ERR_ARG, "the dataset has class labels (LinearSVR needs a regression gs_set_data)");
    if (h->z64.empty()) return fail(GS_ERR_NO_DATA, "no float64 targets (call gs_set_targets_f64 after gs_set_data)");
    if (h->class_w_sets > 0) return fail(GS_ERR_ARG, "class weights do not apply to a regressor");
    if (n_cand <= 0 || !Cv || !epsv || !solver || !seed || !(tol > 0) || max_iter < 0) return fail(GS_ERR_ARG, "bad arguments");
    if (fit_intercept && !(intercept_scaling > 0 && std::isfinite(intercept_scaling)))
        return fail(GS_ERR_ARG, "intercept_scaling must be > 0 with an intercept");
    if (h->d > GS_LINSVR_MAX_FEATURES)
        return fail(GS_ERR_UNSUPPORTED, "more than " + std::to_string(GS_LINSVR_MAX_FEATURES) + " features");
    const int kind = refit ? GS_SCORE_DEFAULT : h->score_kind;
    if (int e = check_scorer(h, who, kind)) return e;
    const int ns = refit ? 1 : h->n_splits, nfit = n_cand * ns;
    for (int c = 0; c < n_cand; c++) {
        if (!(Cv[c] > 0) || !std::isfinite(Cv[c])) return fail(GS_ERR_ARG, "C must be > 0 and finite");
        if (!(epsv[c] >= 0) || !std::isfinite(epsv[c])) return fail(GS_ERR_ARG, "epsilon must be >= 0 and finite");
    }
    for (int t = 0; t < nfit; t++)
        if (solver[t] != 11 && solver[t] != 12 && solver[t] != 13) return fail(GS_ERR_ARG, "solver must be 11, 12 or 13");
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int n = (int)h->n, d = (int)h->d;
    const double bias = fit_intercept ? intercept_scaling : 0.0;
    const int nvar = d + (fit_intercept ? 1 : 0), nt = (nvar + 31) / 32;
    const int nvp = (int)round_up(d + 1, 64);
    const int64_t npad = round_up(n, 64);
    const bool has_sw = !h->sample_w.empty();

    // ---- every split's training rows in fit order (internal rows), zero-weight rows dropped in order ----
    std::vector<int> order, sp_off;
    const int lmax = train_rows(h, ns, refit, true, order, sp_off);
    if (lmax == 0) return fail(GS_ERR_UNSUPPORTED, "a split has no training row of positive weight");

    std::vector<CdFit> cd[2];                                  // [0] solver 12, [1] solver 13
    std::vector<int> tron_fit;
    for (int c = 0; c < n_cand; c++)
        for (int k = 0; k < ns; k++) {
            const int t = c * ns + k;
            if (solver[t] == 11) { tron_fit.push_back(t); continue; }
            cd[solver[t] == 13].push_back(CdFit{sp_off[k], sp_off[k + 1] - sp_off[k], t, seed[t], Cv[c], epsv[c]});
        }
    const int ncd = (int)(cd[0].size() + cd[1].size()), ntr = (int)tron_fit.size();
    const int mpad_all = (int)round_up(nfit, 64), mpad_t = (int)round_up(ntr, 64);

    h->evp.reset(); h->tt.reset();
    cudaEvent_t ev[3];
    for (auto &e : ev) e = h->evp.get();
    cudaEventRecord(ev[0], st);

    // ---- buffers ----
    DevBuf &bXa = h->dWork[0], &bZ = h->dWork[1], &bCd = h->dWork[7], &bOut = h->dWork[8];
    const size_t xa_elems = (size_t)npad * nvp;
    GS_CUDA(bXa.reserve((xa_elems * 2 + (size_t)n * 2) * 8));
    double *dXa = bXa.as<double>(), *dXat = dXa + xa_elems, *dW = dXat + xa_elems, *dQD = dW + n;
    GS_CUDA(bZ.reserve((size_t)std::max(mpad_all, mpad_t) * npad * 8));
    double *dZ = bZ.as<double>();
    GS_CUDA(bOut.reserve(((size_t)mpad_all * nvp + (size_t)nfit * 3) * 8 + (size_t)ntr * sizeof(SvrCol) + (size_t)(nfit + ntr) * 4));
    double *dV = bOut.as<double>();
    long long *dStats = reinterpret_cast<long long *>(dV + (size_t)mpad_all * nvp);
    SvrCol *dCols = reinterpret_cast<SvrCol *>(dStats + (size_t)nfit * 3);
    int *dIter = reinterpret_cast<int *>(dCols + ntr), *dOutRow = dIter + nfit;
    GS_CUDA(cudaMemsetAsync(dV, 0, (size_t)mpad_all * nvp * 8, st));
    GS_CUDA(cudaMemsetAsync(dStats, 0, (size_t)nfit * 3 * 8, st));
    {
        std::vector<double> W64(n, 1.0);
        if (has_sw) W64 = h->sample_w64;
        GS_CUDA(cudaMemcpyAsync(dW, W64.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    }
    const bool f64 = h->x_dtype == GS_F64;
    const float *X32 = h->dX.as<float>();
    const double *X64 = f64 ? h->dX64.as<double>() : nullptr;
    GS_CUDA(launch_build_xa64(f64 ? nullptr : X32, X64, n, d, bias, nvp, npad, dXa, dXat, st));
    int64_t launches = 1;
    std::vector<int> iters(nfit, 0);

    // ---- the dual CD fits: one warp each ----
    if (ncd > 0) {
        const size_t fit_bytes = (size_t)ncd * sizeof(CdFit);
        GS_CUDA(bCd.reserve(fit_bytes + order.size() * 4 + (size_t)ncd * n * 8 + (size_t)ncd * lmax * 4 + 256));
        unsigned char *base = bCd.as<unsigned char>();
        CdFit *dFits = reinterpret_cast<CdFit *>(base);
        double *dBeta = reinterpret_cast<double *>(base + round_up(fit_bytes, 256));
        int *dOrder = reinterpret_cast<int *>(dBeta + (size_t)ncd * n);
        int *dIndex = dOrder + order.size();
        std::vector<CdFit> all(cd[0]);
        all.insert(all.end(), cd[1].begin(), cd[1].end());
        GS_CUDA(cudaMemcpyAsync(dFits, all.data(), fit_bytes, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(dOrder, order.data(), order.size() * 4, cudaMemcpyHostToDevice, st));
        if (f64) linsvr_qd_kernel<double><<<(n + 255) / 256, 256, 0, st>>>(X64, n, d, bias, dQD);
        else linsvr_qd_kernel<float><<<(n + 255) / 256, 256, 0, st>>>(X32, n, d, bias, dQD);
        GS_CUDA(cudaGetLastError());
        launches++;
        const double *Wp = has_sw ? dW : nullptr;
        const double *Y = h->dZ64.as<double>();
        for (int loss = 0; loss < 2; loss++) {
            const int cnt = (int)cd[loss].size();
            if (!cnt) continue;
            const int first = loss ? (int)cd[0].size() : 0;
            cudaError_t e;
            if (loss == 1) e = f64 ? launch_cd<true>(nt, dFits + first, cnt, X64, d, bias, dOrder, dQD, Y, Wp, dBeta + (size_t)first * n, dIndex + (size_t)first * lmax, lmax, n, tol, max_iter, dV, nvp, dIter, dStats, st)
                                   : launch_cd<true>(nt, dFits + first, cnt, X32, d, bias, dOrder, dQD, Y, Wp, dBeta + (size_t)first * n, dIndex + (size_t)first * lmax, lmax, n, tol, max_iter, dV, nvp, dIter, dStats, st);
            else e = f64 ? launch_cd<false>(nt, dFits + first, cnt, X64, d, bias, dOrder, dQD, Y, Wp, dBeta + (size_t)first * n, dIndex + (size_t)first * lmax, lmax, n, tol, max_iter, dV, nvp, dIter, dStats, st)
                         : launch_cd<false>(nt, dFits + first, cnt, X32, d, bias, dOrder, dQD, Y, Wp, dBeta + (size_t)first * n, dIndex + (size_t)first * lmax, lmax, n, tol, max_iter, dV, nvp, dIter, dStats, st);
            GS_CUDA(e);
            launches++;
        }
    }

    // ---- the TRON fits (solver 11): linsvc.cu's rounds with the SVR element-wise pass ----
    TronRounds tr;
    if (ntr > 0) {
        if (int e = tr.reserve(h, ntr)) return e;
        std::vector<TrState> hs(ntr);
        std::vector<SvrCol> hc(ntr);
        for (int q = 0; q < ntr; q++) {
            const int t = tron_fit[q], c = t / ns, k = t % ns;
            TrState &S = hs[q];
            memset(&S, 0, sizeof S);
            S.mode = M_FUN; S.iter = 1; S.init = 1; S.fold = refit ? -100 : k;
            S.eps = tol;                                            // train_one, L2R_L2LOSS_SVR: TRON(eps) unscaled
            hc[q] = SvrCol{refit ? -100 : k, Cv[c], epsv[c]};
        }
        GS_CUDA(cudaMemcpyAsync(tr.St, hs.data(), (size_t)ntr * sizeof(TrState), cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(dCols, hc.data(), (size_t)ntr * sizeof(SvrCol), cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(dOutRow, tron_fit.data(), (size_t)ntr * 4, cudaMemcpyHostToDevice, st));
        const double *Y = h->dZ64.as<double>();
        auto pointwise = [&]() {
            linsvr_pointwise_kernel<<<dim3(PW_BLOCKS, ntr), 256, 0, st>>>(dZ, npad, n, Y, h->masks(), dW, tr.St, dCols, tr.mask,
                                                                          (int64_t)ntr * npad, tr.R, tr.F);
            return cudaGetLastError();
        };
        if (int e = tr.run(h, who, dXa, dXat, dZ, max_iter, pointwise, launches)) return e;
        linsvr_scatter_w_kernel<<<ntr, 128, 0, st>>>(tr.Vec, dOutRow, ntr, nvp, dV);
        GS_CUDA(cudaGetLastError());
        launches++;
        std::vector<TrState> fin(ntr);
        GS_CUDA(cudaMemcpyAsync(fin.data(), tr.St, (size_t)ntr * sizeof(TrState), cudaMemcpyDeviceToHost, st));
        GS_CUDA(cudaStreamSynchronize(st));
        for (int q = 0; q < ntr; q++) iters[tron_fit[q]] = fin[q].n_iter;
    }
    cudaEventRecord(ev[1], st);

    // ---- CD iteration counts and statistics ----
    std::vector<int> cd_iter(nfit, 0);
    std::vector<long long> stats((size_t)nfit * 3, 0);
    if (ncd > 0) {
        GS_CUDA(cudaMemcpyAsync(cd_iter.data(), dIter, (size_t)nfit * 4, cudaMemcpyDeviceToHost, st));
        GS_CUDA(cudaMemcpyAsync(stats.data(), dStats, stats.size() * 8, cudaMemcpyDeviceToHost, st));
    }
    std::vector<double> wraw;
    if (coef_out) {
        wraw.resize((size_t)nfit * nvp);
        GS_CUDA(cudaMemcpyAsync(wraw.data(), dV, wraw.size() * 8, cudaMemcpyDeviceToHost, st));
    }

    // ---- scoring: z = Xa w for every fit in one forward contraction, then the residual sums of squares ----
    if (!refit) {
        if (int e = score_linear_fits(h, dV, dXa, dZ, nfit, 1, ns, kind, test_scores, train_scores, ev[2], launches)) return e;
    } else {
        cudaEventRecord(ev[2], st);
        GS_CUDA(cudaStreamSynchronize(st));
    }
    for (const auto &v : cd) for (const CdFit &F : v) iters[F.out] = cd_iter[F.out];
    for (int t = 0; t < nfit; t++) {
        if (n_iter) n_iter[t] = iters[t];
        if (coef_out) {
            for (int j = 0; j <= d; j++) coef_out[(size_t)t * (d + 1) + j] = j < nvar ? wraw[(size_t)t * nvp + j] : 0.0;
        }
        if (cd_stats) for (int e = 0; e < 3; e++) cd_stats[(size_t)t * 3 + e] = stats[(size_t)t * 3 + e];
    }
    linear_profile(h, ev, launches, ms_solve, ms_score);
    int64_t total_steps = 0;
    for (int t = 0; t < nfit; t++) total_steps += stats[(size_t)t * 3];
    h->prof.smo_iterations = total_steps + tr.rounds;          // CD coordinate steps plus TRON rounds
    return GS_OK;
}

}  // namespace

extern "C" {

int gs_linsvr(gs_handle *h, int32_t n_cand, const double *C, const double *epsilon, const int32_t *solver, const uint32_t *seed,
              double tol, int32_t max_iter, int32_t fit_intercept, double intercept_scaling, uint32_t flags, double *test_scores,
              double *train_scores, int32_t *n_iter, float *fit_ms, float *score_ms, double *coef_out, int64_t *cd_stats)
{
    if (h && !test_scores) { gs_set_error(h, "gs_linsvr: test_scores is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    const int st = linsvr_run(h, n_cand, C, epsilon, solver, seed, tol, max_iter, fit_intercept, intercept_scaling, false, test_scores,
                              (flags & GS_RETURN_TRAIN) ? train_scores : nullptr, n_iter, coef_out, cd_stats, &a, &b);
    if (st) return st;
    spread_call_ms(n_cand * h->n_splits, a, b, fit_ms, score_ms);
    return GS_OK;
}

int gs_linsvr_refit(gs_handle *h, double C, double epsilon, int32_t solver, uint32_t seed, double tol, int32_t max_iter,
                    int32_t fit_intercept, double intercept_scaling, double *coef_out, int32_t *n_iter)
{
    if (h && !coef_out) { gs_set_error(h, "gs_linsvr_refit: coef_out is NULL"); return GS_ERR_ARG; }
    float a = 0, b = 0;
    return linsvr_run(h, 1, &C, &epsilon, &solver, &seed, tol, max_iter, fit_intercept, intercept_scaling, true, nullptr, nullptr,
                      n_iter, coef_out, nullptr, &a, &b);
}

int gs_debug_mt19937(gs_handle *h, uint32_t seed, int32_t k, uint32_t *out)
{
    if (!h) return GS_ERR_ARG;
    if (k <= 0 || !out) { gs_set_error(h, "gs_debug_mt19937: bad arguments"); return GS_ERR_ARG; }
    GS_CUDA(cudaSetDevice(h->device));
    GS_CUDA(h->dScore.reserve((size_t)k * 4));
    linsvr_mt_kernel<<<1, 32, 0, h->stream>>>(seed, k, h->dScore.as<uint32_t>());
    GS_CUDA(cudaGetLastError());
    GS_CUDA(cudaMemcpyAsync(out, h->dScore.p, (size_t)k * 4, cudaMemcpyDeviceToHost, h->stream));
    GS_CUDA(cudaStreamSynchronize(h->stream));
    return GS_OK;
}

}  // extern "C"
