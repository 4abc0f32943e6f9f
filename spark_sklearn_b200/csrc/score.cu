// score.cu -- SVC decision values for every (row, sub-model), one-vs-one voting / accuracy, the scorers' device counts, and
// the host side of scoring every search shares: the scorer check, the per-split score denominators and the score formulas.
//
// libsvm predicts with float64 kernel values (svm.cpp:2821-2904 svm_predict_values calls
// Kernel::k_function in double; the float32 rounding applies only to the training Q matrix), so the
// decision values are NOT formed from the float32 K matrix.  They are a float64 product
//      dec[c][r] = sum_j k64(r, j) * coef[c][j],   k64 = exp(-gamma*d2(r,j)), S_rj, or the poly / sigmoid of S_rj
// evaluated for ALL rows r at once (test rows give the test score, the other rows the train score)
// and for all sub-models c that share one (kernel, gamma): one pass over the float64 Gram per gamma,
// with the exp (or powi / tanh) fused into the operand load.  coef is zero outside a sub-model's training rows.
#include "common.cuh"
#include <algorithm>
#include <cmath>

namespace {

constexpr int TR = 64, TJ = 32;

// TC = columns per block (multiple of 8, the group's column count rounded up to 8 so no lane multiplies padding).  The float64 exp of a (row, SV) pair is the expensive part (n^2 of them per
// block row), so a block takes as many coefficient columns as the group has, up to 96 (static shared memory): the kernel values are computed once
// per group instead of once per 32 columns.  PS: the poly / sigmoid instance (gs_kernel_of_dot in the operand load); the
// linear / rbf instances are compiled without it, so their register use and occupancy -- and hence decision_chunks -- stay
// those of the two-kernel build.
template <int TC, bool PS>
__global__ void __launch_bounds__(256)
decision_kernel(const double *__restrict__ S, const double *__restrict__ xsq, int n, int kernel, double gamma,
                int degree, double coef0, const double *__restrict__ coef, int ncols, double *__restrict__ dec, int jlen)
{
    // blockIdx.z = chunk of the j (support-row) range: chunk z sums j in [z*jlen, (z+1)*jlen) into slab z of `dec`
    // (slab stride ncols*n); sum_slabs_kernel adds the slabs in ascending order.  One chunk per row block leaves one
    // 8-warp block per SM and a two-wave tail (157 blocks on 132 SMs at n = 10000).
    constexpr int CPT = TC / 8;                       // columns per thread
    __shared__ __align__(16) double E[TJ][TR + 2];
    __shared__ __align__(16) double Cf[TJ][TC + 2];
    const int tid = threadIdx.x;
    const int r0 = blockIdx.x * TR, c0 = blockIdx.y * TC;
    const int ty = tid >> 3, tx = tid & 7;          // rows ty*2..+1, cols tx + 8*b
    const int lj = tid & 31, lr = tid >> 5;         // loader mapping
    double acc[2][CPT];
#pragma unroll
    for (int b = 0; b < CPT; b++) { acc[0][b] = 0.0; acc[1][b] = 0.0; }
    const double ng = -gamma;

    const int jbeg = blockIdx.z * jlen, jend = min(n, jbeg + jlen);
    dec += (size_t)blockIdx.z * ncols * n;
    for (int j0 = jbeg; j0 < jend; j0 += TJ) {
        const int j = j0 + lj;
        const bool jok = j < jend;
        const double xj = jok ? xsq[j] : 0.0;
#pragma unroll
        for (int s = 0; s < TR / 8; s++) {
            const int r = r0 + lr + 8 * s;
            double v = 0.0;
            if (r < n && jok) {
                const double sv = S[(size_t)r * n + j];
                if (PS) {
                    v = gs_kernel_of_dot(kernel, sv, gamma, degree, coef0);
                } else if (kernel == GS_KERNEL_RBF) {
                    const double d2 = __dsub_rn(__dadd_rn(xsq[r], xj), __dmul_rn(2.0, sv));
                    v = exp(__dmul_rn(ng, d2));
                } else {
                    v = sv;
                }
            }
            E[lj][lr + 8 * s] = v;
        }
#pragma unroll
        for (int s = 0; s < TC / 8; s++) {
            const int c = c0 + lr + 8 * s;
            Cf[lj][lr + 8 * s] = (c < ncols && jok) ? coef[(size_t)c * n + j] : 0.0;
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < TJ; k++) {
            const double2 e = *reinterpret_cast<const double2 *>(&E[k][ty * 2]);
#pragma unroll
            for (int b = 0; b < CPT; b++) {
                const double cv = Cf[k][tx + 8 * b];
                acc[0][b] = fma(e.x, cv, acc[0][b]);
                acc[1][b] = fma(e.y, cv, acc[1][b]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 2; a++) {
        const int r = r0 + ty * 2 + a;
        if (r >= n) continue;
#pragma unroll
        for (int b = 0; b < CPT; b++) {
            const int c = c0 + tx + 8 * b;
            if (c < ncols) dec[(size_t)c * n + r] = acc[a][b];
        }
    }
}

// dec[i] = slab_0[i] + slab_1[i] + ... (ascending, deterministic)
__global__ void sum_slabs_kernel(const double *__restrict__ part, size_t count, int nslab, double *__restrict__ dec)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    double v = part[i];
    for (int z = 1; z < nslab; z++) v = __dadd_rn(v, part[(size_t)z * count + i]);
    dec[i] = v;
}

// One-vs-one vote (svm.cpp:2862-2892): dec - rho > 0 votes for the lower class of the pair, else the
// higher; first maximum wins.  Accuracy counts split by fold membership.
__global__ void __launch_bounds__(256)
vote_kernel(const double *__restrict__ dec, const double *__restrict__ rho, int n, int n_classes,
            const int *__restrict__ y, SplitMasks sm,
            const VoteTask *__restrict__ tasks, int *__restrict__ counts)
{
    const VoteTask T = tasks[blockIdx.y];
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    int c_te = 0, n_te = 0, c_tr = 0, n_tr = 0;
    if (r < n) {
        int pred;
        if (n_classes == 2) {
            const double dv = dec[(size_t)T.first_col * n + r] - rho[T.first_col];
            pred = dv > 0 ? 0 : 1;
        } else {
            int votes[32];
            for (int c = 0; c < n_classes; c++) votes[c] = 0;
            int p = T.first_col;
            for (int a = 0; a < n_classes; a++)
                for (int b = a + 1; b < n_classes; b++, p++) {
                    const double dv = dec[(size_t)p * n + r] - rho[p];
                    if (dv > 0) ++votes[a]; else ++votes[b];
                }
            pred = 0;
            for (int c = 1; c < n_classes; c++) if (votes[c] > votes[pred]) pred = c;
        }
        const bool ok = pred == y[r];
        if (split_test(sm, r, T.fold)) { n_te = 1; c_te = ok; }
        if (split_train(sm, r, T.fold)) { n_tr = 1; c_tr = ok; }
    }
    // block reduce the four counters
    __shared__ int sh[4][8];
#pragma unroll
    for (int m = 16; m; m >>= 1) {
        c_te += __shfl_xor_sync(0xffffffffu, c_te, m); n_te += __shfl_xor_sync(0xffffffffu, n_te, m);
        c_tr += __shfl_xor_sync(0xffffffffu, c_tr, m); n_tr += __shfl_xor_sync(0xffffffffu, n_tr, m);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { sh[0][w] = c_te; sh[1][w] = n_te; sh[2][w] = c_tr; sh[3][w] = n_tr; }
    __syncthreads();
    if (threadIdx.x < 4) {
        int s = 0;
        for (int i = 0; i < 8; i++) s += sh[threadIdx.x][i];
        if (s) atomicAdd(&counts[blockIdx.y * 4 + threadIdx.x], s);
    }
}

// Per-class counts for the count-based scorers (sklearn.metrics accuracy / balanced_accuracy / precision / recall / f1,
// metrics/_classification.py: everything they need is the multilabel confusion diagonal): for every task, split
// (0 test, 1 train) and class c:  support (y == c), tp (y == c and predicted c), predicted (predicted c).
// counts[task][split][class][3]; block-level shared-memory accumulation, one global atomic per non-zero cell.
__global__ void __launch_bounds__(256)
vote_classes_kernel(const double *__restrict__ dec, const double *__restrict__ rho, int n, int n_classes,
                    const int *__restrict__ y, SplitMasks sm,
                    const VoteTask *__restrict__ tasks, int *__restrict__ counts)
{
    __shared__ int sh[2 * 32 * 3];
    for (int i = threadIdx.x; i < 2 * n_classes * 3; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const VoteTask T = tasks[blockIdx.y];
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) {
        int pred;
        if (n_classes == 2) {
            const double dv = dec[(size_t)T.first_col * n + r] - rho[T.first_col];
            pred = dv > 0 ? 0 : 1;
        } else {
            int votes[32];
            for (int c = 0; c < n_classes; c++) votes[c] = 0;
            int p = T.first_col;
            for (int a = 0; a < n_classes; a++)
                for (int b = a + 1; b < n_classes; b++, p++) {
                    const double dv = dec[(size_t)p * n + r] - rho[p];
                    if (dv > 0) ++votes[a]; else ++votes[b];
                }
            pred = 0;
            for (int c = 1; c < n_classes; c++) if (votes[c] > votes[pred]) pred = c;
        }
        const int yc = y[r];
#pragma unroll
        for (int sp = 0; sp < 2; sp++) {
            if (sp == 0 ? split_test(sm, r, T.fold) : split_train(sm, r, T.fold)) {
                atomicAdd(&sh[(sp * n_classes + yc) * 3 + 0], 1);
                if (pred == yc) atomicAdd(&sh[(sp * n_classes + yc) * 3 + 1], 1);
                atomicAdd(&sh[(sp * n_classes + pred) * 3 + 2], 1);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * n_classes * 3; i += blockDim.x)
        if (sh[i]) atomicAdd(&counts[(size_t)blockIdx.y * 2 * n_classes * 3 + i], sh[i]);
}

// Area under the ROC curve of a binary task (sklearn.metrics.roc_auc_score == the Mann-Whitney statistic with ties counted
// one half): pairs (p, q) of a row p of the positive class (ids >= n_a in the class-sorted order) and a row q of the
// negative class whose scores satisfy s_p > s_q (wins) or s_p == s_q (ties), separately for the test rows of the task's
// fold and for its training rows.  out[task][4] = {test wins, test ties, train wins, train ties} (64-bit).
// SIGN: +1 when larger values mean the positive class (LogisticRegression z), -1 for libsvm's dec - rho (positive means
// the FIRST class, svm.cpp:2862; scikit-learn negates it for its binary decision_function).
template <typename T>
__global__ void __launch_bounds__(256)
auc_pairs_kernel(const T *__restrict__ score, int64_t ld, int n, int n_a, SplitMasks sm,
                 const int *__restrict__ col_of_task, const int *__restrict__ fold_of_task, int sign,
                 unsigned long long *__restrict__ out)
{
    __shared__ T s_a[256];
    __shared__ signed char f_a[256];
    __shared__ unsigned long long red[4];
    const int task = blockIdx.y, k = fold_of_task[task];
    const T *__restrict__ sc = score + (size_t)col_of_task[task] * ld;
    const int p = n_a + blockIdx.x * blockDim.x + threadIdx.x;
    const bool has = p < n;
    const T sp = has ? (sign > 0 ? sc[p] : -sc[p]) : T(0);
    const int p_st = !has ? 2 : (split_test(sm, p, k) ? 1 : (split_train(sm, p, k) ? 0 : 2));     // 1 test, 0 training, 2 neither
    unsigned w_te = 0, t_te = 0, w_tr = 0, t_tr = 0;
    if (threadIdx.x < 4) red[threadIdx.x] = 0ull;
    for (int q0 = 0; q0 < n_a; q0 += 256) {
        __syncthreads();
        const int q = q0 + threadIdx.x;
        s_a[threadIdx.x] = q < n_a ? (sign > 0 ? sc[q] : -sc[q]) : T(0);
        f_a[threadIdx.x] = q < n_a ? (split_test(sm, q, k) ? 1 : (split_train(sm, q, k) ? 0 : 2)) : (signed char)2;   // 2: no row / neither set
        __syncthreads();
        if (p_st != 2) {
            const int lim = min(256, n_a - q0);
            for (int j = 0; j < lim; j++) {
                if (f_a[j] == p_st) {                                                    // both test rows or both training rows
                    const unsigned win = sp > s_a[j], tie = sp == s_a[j];
                    if (p_st == 1) { w_te += win; t_te += tie; } else { w_tr += win; t_tr += tie; }
                }
            }
        }
    }
    __syncthreads();
    unsigned v[4] = {w_te, t_te, w_tr, t_tr};
#pragma unroll
    for (int e = 0; e < 4; e++) {
#pragma unroll
        for (int m = 16; m; m >>= 1) v[e] += __shfl_xor_sync(0xffffffffu, v[e], m);
        if ((threadIdx.x & 31) == 0 && v[e]) atomicAdd(&red[e], (unsigned long long)v[e]);
    }
    __syncthreads();
    if (threadIdx.x < 4 && red[threadIdx.x]) atomicAdd(&out[(size_t)task * 4 + threadIdx.x], red[threadIdx.x]);
}


// rss[task][0 / 1] = sum over test / training rows of the split of (z - (dec - rho))^2.  One block per task; every thread
// sums a fixed row stride, then a fixed shared-memory tree: the same bits every run.
constexpr int RSS_NT = 256;

__global__ void __launch_bounds__(RSS_NT)
rss_kernel(const double *__restrict__ dec, const double *__restrict__ rho, int n, const double *__restrict__ z, SplitMasks sm,
           const VoteTask *__restrict__ tasks, double *__restrict__ rss)
{
    __shared__ double red[2][RSS_NT];
    const VoteTask T = tasks[blockIdx.x];
    const double *__restrict__ dv = dec + (size_t)T.first_col * n;
    const double b = rho[T.first_col];
    double s_te = 0.0, s_tr = 0.0;
    for (int r = threadIdx.x; r < n; r += RSS_NT) {
        const bool te = split_test(sm, r, T.fold), tr = !te && split_train(sm, r, T.fold);
        if (te || tr) {
            const double e = __dsub_rn(z[r], __dsub_rn(dv[r], b));
            const double e2 = __dmul_rn(e, e);
            if (te) s_te = __dadd_rn(s_te, e2); else s_tr = __dadd_rn(s_tr, e2);
        }
    }
    red[0][threadIdx.x] = s_te; red[1][threadIdx.x] = s_tr;
    __syncthreads();
    for (int w = RSS_NT / 2; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) {
            red[0][threadIdx.x] = __dadd_rn(red[0][threadIdx.x], red[0][threadIdx.x + w]);
            red[1][threadIdx.x] = __dadd_rn(red[1][threadIdx.x], red[1][threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x < 2) rss[(size_t)blockIdx.x * 2 + threadIdx.x] = red[threadIdx.x][0];
}

}  // namespace

cudaError_t launch_vote_classes(const double *dec, const double *rho, int n, int n_classes, const int *y,
                                SplitMasks sm, const VoteTask *tasks, int n_tasks, int *counts, cudaStream_t st)
{
    if (n_tasks <= 0) return cudaSuccess;
    for (int t0 = 0; t0 < n_tasks; t0 += 32768) {                     // gridDim.y <= 65535
        const int nt = std::min(32768, n_tasks - t0);
        dim3 grid((n + 255) / 256, nt);
        vote_classes_kernel<<<grid, 256, 0, st>>>(dec, rho, n, n_classes, y, sm, tasks + t0, counts + (size_t)t0 * 2 * n_classes * 3);
    }
    return cudaGetLastError();
}

cudaError_t launch_auc_pairs_f64(const double *score, int64_t ld, int n, int n_a, SplitMasks sm, const int *col_of_task,
                                 const int *fold_of_task, int n_tasks, int sign, unsigned long long *out, cudaStream_t st)
{
    if (n_tasks <= 0 || n - n_a <= 0) return cudaSuccess;
    for (int t0 = 0; t0 < n_tasks; t0 += 32768) {
        const int nt = std::min(32768, n_tasks - t0);
        dim3 grid((n - n_a + 255) / 256, nt);
        auc_pairs_kernel<double><<<grid, 256, 0, st>>>(score, ld, n, n_a, sm, col_of_task + t0, fold_of_task + t0, sign, out + (size_t)t0 * 4);
    }
    return cudaGetLastError();
}

cudaError_t launch_auc_pairs_f32(const float *score, int64_t ld, int n, int n_a, SplitMasks sm, const int *col_of_task,
                                 const int *fold_of_task, int n_tasks, int sign, unsigned long long *out, cudaStream_t st)
{
    if (n_tasks <= 0 || n - n_a <= 0) return cudaSuccess;
    for (int t0 = 0; t0 < n_tasks; t0 += 32768) {
        const int nt = std::min(32768, n_tasks - t0);
        dim3 grid((n - n_a + 255) / 256, nt);
        auc_pairs_kernel<float><<<grid, 256, 0, st>>>(score, ld, n, n_a, sm, col_of_task + t0, fold_of_task + t0, sign, out + (size_t)t0 * 4);
    }
    return cudaGetLastError();
}

// resident CTAs per SM of the instance that serves `tc` columns (queried once per instance)
static int decision_ctas_per_sm(int tc)
{
    static int cache[13] = {0};
    const int slot = tc / 8;
    if (cache[slot] == 0) {
        int nb = 0;
#define GS_OCC(T) case T: cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, decision_kernel<T, false>, 256, 0); break;
        switch (tc) {
            GS_OCC(8) GS_OCC(16) GS_OCC(24) GS_OCC(32) GS_OCC(40) GS_OCC(48) GS_OCC(56) GS_OCC(64) GS_OCC(72) GS_OCC(80) GS_OCC(88)
            default: cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, decision_kernel<96, false>, 256, 0); break;
        }
#undef GS_OCC
        cache[slot] = nb > 0 ? nb : 1;
    }
    return cache[slot];
}

// part: workspace of at least jchunks * ncols * n doubles when jchunks > 1.
// The CTAs of a launch take the same time, so a launch costs ceil(CTAs / resident CTAs) rounds; the slab count with the
// fewest rounds per unit of work wins (config 2 on 132 SMs: 40 columns, 4 CTAs/SM -> 10 slabs instead of 4: 2.97 rounds of 1/10
// against 2 rounds of 1/4).  Short ranges are not split (each slab keeps >= 8 tiles of TJ support rows).
int decision_chunks(int n, int ncols, int sms)
{
    if (n < 4096 || ncols <= 0) return 1;
    const int tc = std::min(96, (ncols + 7) / 8 * 8);
    const long long slots = (long long)sms * decision_ctas_per_sm(tc);
    const long long base = (long long)((n + TR - 1) / TR) * ((ncols + tc - 1) / tc);
    int best = 1;
    double best_cost = 1e30;
    for (int jc = 1; jc <= 16 && n / jc >= 8 * TJ; jc++) {
        const double cost = (double)((base * jc + slots - 1) / slots) / jc;
        if (cost < best_cost - 1e-12) { best_cost = cost; best = jc; }
    }
    return best;
}

cudaError_t launch_decision(const double *S, const double *xsq, int n, int kernel, double gamma, int degree, double coef0,
                            const double *coef, int ncols, double *dec, double *part, int jchunks, cudaStream_t st)
{
    if (ncols <= 0) return cudaSuccess;
    const int tc = std::min(96, (ncols + 7) / 8 * 8);
    if (!part || jchunks < 1) jchunks = 1;
    const int jlen = ((n + jchunks - 1) / jchunks + TJ - 1) / TJ * TJ;
    dim3 grid((n + TR - 1) / TR, (ncols + tc - 1) / tc, jchunks);
    double *out = jchunks > 1 ? part : dec;
    const bool ps = kernel == GS_KERNEL_POLY || kernel == GS_KERNEL_SIGMOID;
#define GS_DEC(T) case T: if (ps) decision_kernel<T, true><<<grid, 256, 0, st>>>(S, xsq, n, kernel, gamma, degree, coef0, coef, ncols, out, jlen); \
                          else decision_kernel<T, false><<<grid, 256, 0, st>>>(S, xsq, n, kernel, gamma, degree, coef0, coef, ncols, out, jlen); break;
    switch (tc) {
        GS_DEC(8) GS_DEC(16) GS_DEC(24) GS_DEC(32) GS_DEC(40) GS_DEC(48) GS_DEC(56) GS_DEC(64) GS_DEC(72) GS_DEC(80) GS_DEC(88)
        default: GS_DEC(96)
    }
#undef GS_DEC
    if (jchunks > 1) {
        const size_t count = (size_t)ncols * n;
        sum_slabs_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(part, count, jchunks, dec);
    }
    return cudaGetLastError();
}

cudaError_t launch_vote(const double *dec, const double *rho, int n, int n_classes, const int *y,
                        SplitMasks sm, const VoteTask *tasks, int n_tasks, int *counts,
                        cudaStream_t st)
{
    if (n_tasks <= 0) return cudaSuccess;
    for (int t0 = 0; t0 < n_tasks; t0 += 32768) {                     // gridDim.y <= 65535
        const int nt = std::min(32768, n_tasks - t0);
        dim3 grid((n + 255) / 256, nt);
        vote_kernel<<<grid, 256, 0, st>>>(dec, rho, n, n_classes, y, sm, tasks + t0, counts + (size_t)t0 * 4);
    }
    return cudaGetLastError();
}

cudaError_t launch_rss(const double *dec, const double *rho, int n, const double *z, SplitMasks sm, const VoteTask *tasks,
                       int n_tasks, double *rss, cudaStream_t st)
{
    if (n_tasks <= 0) return cudaSuccess;
    rss_kernel<<<n_tasks, RSS_NT, 0, st>>>(dec, rho, n, z, sm, tasks, rss);
    return cudaGetLastError();
}

// scikit-learn's count-based scores (metrics/_classification.py) from cnt[class][3] = {support, tp, predicted}, float64.
// Undefined ratios follow zero_division="warn": 0.0.  accuracy_score :187; balanced_accuracy_score :2362 (mean recall over
// the classes present in y_true); precision_recall_fscore_support :1573 with beta = 1: f = 2 tp / (2 tp + fp + fn).
double gs_score_from_counts(int kind, int pos_class, int n_classes, const int *cnt)
{
    auto sup = [&](int c) { return (double)cnt[c * 3 + 0]; };
    auto tp = [&](int c) { return (double)cnt[c * 3 + 1]; };
    auto prd = [&](int c) { return (double)cnt[c * 3 + 2]; };
    auto f1c = [&](int c) { const double den = sup(c) + prd(c); return den > 0 ? 2.0 * tp(c) / den : 0.0; };   // 2tp + fp + fn = support + predicted
    double n = 0, correct = 0;
    for (int c = 0; c < n_classes; c++) { n += sup(c); correct += tp(c); }
    if (!(n > 0)) return NAN;
    switch (kind) {
    case GS_SCORE_DEFAULT: return correct / n;
    case GS_SCORE_BALANCED_ACCURACY: {
        double s = 0; int k = 0;
        for (int c = 0; c < n_classes; c++) if (sup(c) > 0) { s += tp(c) / sup(c); k++; }
        return k ? s / k : NAN;
    }
    case GS_SCORE_F1: return f1c(pos_class);
    case GS_SCORE_PRECISION: return prd(pos_class) > 0 ? tp(pos_class) / prd(pos_class) : 0.0;
    case GS_SCORE_RECALL: return sup(pos_class) > 0 ? tp(pos_class) / sup(pos_class) : 0.0;
    case GS_SCORE_F1_MACRO: {
        double s = 0;
        for (int c = 0; c < n_classes; c++) s += f1c(c);
        return s / n_classes;
    }
    case GS_SCORE_F1_MICRO: return correct / n;                         // single-label: micro f1 == accuracy
    case GS_SCORE_F1_WEIGHTED: {
        double s = 0;
        for (int c = 0; c < n_classes; c++) s += f1c(c) * sup(c);
        return s / n;
    }
    default: return NAN;
    }
}

int check_scorer(gs_handle *h, const char *who, int kind)
{
    const bool regression_kind = kind == GS_SCORE_NEG_MSE || kind == GS_SCORE_NEG_RMSE;
    const bool binary_kind = kind == GS_SCORE_ROC_AUC || kind == GS_SCORE_F1 || kind == GS_SCORE_PRECISION || kind == GS_SCORE_RECALL;
    const char *msg = nullptr;
    int code = GS_ERR_ARG;
    if (!h->classification) {
        if (kind != GS_SCORE_DEFAULT && !regression_kind) msg = "classification scorer on a regressor";
    } else if (regression_kind) {
        msg = "regression scorer on a classifier";
    } else if (binary_kind && h->n_classes != 2) {
        msg = "this scorer is defined for binary problems only";
        code = GS_ERR_UNSUPPORTED;
    } else if (kind != GS_SCORE_DEFAULT && h->score_pos >= h->n_classes) {
        msg = "positive class out of range";
    }
    if (!msg) return GS_OK;
    gs_set_error(h, std::string(who) + ": " + msg);
    return code;
}

SplitScoreStats::SplitScoreStats(const gs_handle *h, int ns, int kind_)
    : kind(kind_), pos_class(h->score_pos), n_classes(h->n_classes)
{
    const bool cls = h->classification;
    if (cls && kind != GS_SCORE_ROC_AUC) return;                         // the count-based scores carry their own totals
    const int n = (int)h->n;
    std::vector<int> by_orig(n);
    for (int r = 0; r < n; r++) by_orig[h->perm[r]] = r;
    rows.assign((size_t)ns * 2, 0.0); n_a.assign((size_t)ns * 2, 0.0); n_b.assign((size_t)ns * 2, 0.0); tss.assign((size_t)ns * 2, 0.0);
    for (int k = 0; k < ns; k++) {
        double sum[2] = {0, 0};
        for (int o = 0; o < n; o++) {
            const int r = by_orig[o];
            const int sp = h->is_test(r, k) ? 0 : (h->is_train(r, k) ? 1 : -1);
            if (sp < 0) continue;
            rows[(size_t)k * 2 + sp] += 1;
            if (cls) (r >= h->class_start[1] ? n_b : n_a)[(size_t)k * 2 + sp] += 1;    // rows are class-sorted
            else sum[sp] += h->z64[r];
        }
        if (cls) continue;
        for (int sp = 0; sp < 2; sp++) {
            // np.average then sum of squared deviations, ascending original row order as scikit-learn's y[test] / y[train]
            const double m = rows[(size_t)k * 2 + sp], mean = m > 0 ? sum[sp] / m : 0.0;
            double s = 0;
            for (int o = 0; o < n; o++) {
                const int r = by_orig[o];
                if (sp == 0 ? h->is_test(r, k) : (!h->is_test(r, k) && h->is_train(r, k))) { const double e = h->z64[r] - mean; s += e * e; }
            }
            tss[(size_t)k * 2 + sp] = s;
        }
    }
}

double SplitScoreStats::accuracy(const int *vote)
{
    return vote[1] > 0 ? (double)vote[0] / (double)vote[1] : NAN;
}

double SplitScoreStats::auc(int k, int sp, const unsigned long long *pairs) const
{
    const double np_ = n_a[(size_t)k * 2 + sp] * n_b[(size_t)k * 2 + sp];
    return np_ > 0 ? ((double)pairs[0] + 0.5 * (double)pairs[1]) / np_ : NAN;
}

double SplitScoreStats::counts(const int *cnt) const
{
    return gs_score_from_counts(kind, pos_class, n_classes, cnt);
}

double SplitScoreStats::regression(int k, int sp, double rss) const
{
    const double m = rows[(size_t)k * 2 + sp];
    if (!(m > 0)) return NAN;
    if (kind == GS_SCORE_NEG_MSE) return -(rss / m);                       // mean_squared_error
    if (kind == GS_SCORE_NEG_RMSE) return -std::sqrt(rss / m);             // root_mean_squared_error
    return gs_r2_score(rss, tss[(size_t)k * 2 + sp], m);
}
