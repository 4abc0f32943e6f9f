// knn.cu -- k-nearest-neighbour searches (gs_knn) and the neighbour-list test hook (gs_debug_knn_neighbors).
//
// A k-NN fit stores its training rows; all the work of a (candidate, split) task is in the neighbour queries of its scorer.
// For one split, the neighbours of a row depend only on the metric: n_neighbors and weights change how those neighbours vote.
// So a call computes, per metric present, the K_max = max n_neighbors nearest training rows of every evaluated row in every
// split once, and every candidate votes from those sorted lists:
//   1. distances, one row slab at a time (no n x n matrix is kept): Euclidean rows carry scikit-learn's brute-force ordering
//      key xsq[c] - 2 x_r.x_c (the row's own xsq is added back for the distance), Manhattan rows the float64 sum of the float32
//      (or float64) differences in feature order rounded to X's dtype, ManhattanDistance{32,64}.dist of
//      sklearn/metrics/_dist_metrics.pyx.tp;
//   2. selection: one CTA per row keeps, for every split the row is evaluated in, the K_max smallest (key, original row
//      index) of the split's training columns: exact ties go to the lower row index (deterministic; scikit-learn's
//      ArgKmin max-heap keeps the same rows except where its root replacement picks another of the tied entries);
//   3. votes: one thread per (row, candidate, split) -> per-class counts for the count scorers, predict_proba[:, 1] for
//      roc_auc, predictions for the residual sums of squares of the regressor.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <numeric>

namespace {

constexpr int DT = 64;              // distance tile: DT x DT outputs per CTA, 4 x 4 per thread
constexpr int DK = 16;              // features per shared-memory stage
constexpr int SEL_NT = 256;         // selection CTA: one row, columns in chunks of SEL_NT
constexpr int SEL_MAX_G = 32;       // splits served by one pass over a row's distances
constexpr int SEL_SMEM = 96 * 1024; // dynamic shared-memory budget of the selection kernel

// xsq[r] = sum_f x[r][f]^2 by the same fma chain as the distance tile's diagonal, so a row's distance to itself is 0
template <typename T>
__global__ void knn_sqnorm_kernel(const T *__restrict__ X, int n, int d, double *__restrict__ xsq)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    double acc = 0.0;
    for (int f = 0; f < d; f++) {
        const double v = (double)X[(size_t)r * d + f];
        acc = __fma_rn(v, v, acc);
    }
    xsq[r] = acc;
}

// D[i][c] for the slab rows r0 + i (i < rows) and every column c < n.  Euclidean (L1 == false): xsq[c] - 2 sum_f x_r,f x_c,f
// (float64 fma chain in feature order: float32 products are exact).  Manhattan: sum_f |x_r,f - x_c,f| with the difference
// rounded in T and the sum in float64, every operation rounded on its own, the result rounded to T.  Padding features are
// zeros and add nothing.
template <typename T, bool L1>
__global__ void __launch_bounds__(256)
knn_dist_kernel(const T *__restrict__ X, int n, int d, int r0, int rows, const double *__restrict__ xsq, double *__restrict__ D)
{
    __shared__ T As[DK][DT];
    __shared__ T Bs[DK][DT];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int i0 = blockIdx.y * DT, c0 = blockIdx.x * DT;
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.0;
    for (int k0 = 0; k0 < d; k0 += DK) {
        for (int e = threadIdx.x; e < DT * DK; e += 256) {
            const int rr = e / DK, kk = e % DK, f = k0 + kk;
            const int gi = i0 + rr, gc = c0 + rr;
            As[kk][rr] = (gi < rows && f < d) ? X[(size_t)(r0 + gi) * d + f] : T(0);
            Bs[kk][rr] = (gc < n && f < d) ? X[(size_t)gc * d + f] : T(0);
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < DK; kk++) {
            T a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) a[i] = As[kk][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < 4; j++) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    if (L1) {
                        if (sizeof(T) == 4) acc[i][j] = __dadd_rn(acc[i][j], (double)fabsf(__fsub_rn((float)a[i], (float)b[j])));
                        else acc[i][j] = __dadd_rn(acc[i][j], fabs(__dsub_rn((double)a[i], (double)b[j])));
                    } else {
                        acc[i][j] = __fma_rn((double)a[i], (double)b[j], acc[i][j]);
                    }
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int r = i0 + ty + 16 * i;
        if (r >= rows) continue;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = c0 + tx + 16 * j;
            if (c < n) {
                // ManhattanDistance32.dist returns its float64 sum as a float32: the key and the distance are that float32
                if (L1) D[(size_t)r * n + c] = sizeof(T) == 4 ? (double)__double2float_rn(acc[i][j]) : acc[i][j];
                else D[(size_t)r * n + c] = __dsub_rn(xsq[c], __dmul_rn(2.0, acc[i][j]));
            }
        }
    }
}

__device__ __forceinline__ bool key_less(double ka, int ia, double kb, int ib)
{
    return ka < kb || (ka == kb && ia < ib);
}

// One CTA per slab row r = r0 + blockIdx.x.  For the splits k_lo .. k_lo + G - 1 the row is evaluated in (mode 0: its test
// splits, 1: also the splits it trains, 2: every split), keeps the K smallest (key, original index) over the split's training
// columns as a sorted list in shared memory.  Each chunk of SEL_NT columns is read once for all G splits: a column enters a
// split's list when it trains that split and beats the list's last entry; the entrants of a chunk are merged by rank (keys
// with their indices are distinct, so the ranks are a permutation and the result does not depend on the entrants' order).
// Output: list of split k_lo + s of row r at ((k_lo + s - k_out0) * n + r) * K; entries past the training rows: -1 / +inf.
__global__ void __launch_bounds__(SEL_NT)
knn_select_kernel(const double *__restrict__ D, int n, int r0, const int *__restrict__ perm, SplitMasks sm, int k_lo, int G,
                  int K, int mode, int k_out0, int *__restrict__ out_idx, double *__restrict__ out_key)
{
    extern __shared__ __align__(16) unsigned char knn_smem[];
    double *Lk = (double *)knn_smem;                 // [G][K]
    double *Ck = Lk + (size_t)G * K;                 // [SEL_NT]
    int *Li = (int *)(Ck + SEL_NT);                  // [G][K]
    int *Ci = Li + (size_t)G * K;                    // [SEL_NT]
    int *Llen = Ci + SEL_NT;                         // [G]
    __shared__ int wcnt[SEL_NT / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int r = r0 + blockIdx.x;
    const double *__restrict__ drow = D + (size_t)blockIdx.x * n;
    unsigned active = 0;
    for (int s = 0; s < G; s++) {
        const int k = k_lo + s;
        if (mode == 2 || split_test(sm, r, k) || (mode == 1 && split_train(sm, r, k))) active |= 1u << s;
    }
    if (t < G) Llen[t] = 0;
    __syncthreads();
    for (int c0 = 0; c0 < n; c0 += SEL_NT) {
        const int c = c0 + t;
        const bool has = c < n;
        const double key = has ? drow[c] : 0.0;
        const int oi = has ? perm[c] : 0;
        const unsigned long long w0 = has ? sm.tr[(size_t)c * 2] : 0ull, w1 = has ? sm.tr[(size_t)c * 2 + 1] : 0ull;
        for (int s = 0; s < G; s++) {
            if (!((active >> s) & 1u)) continue;
            const int k = k_lo + s;
            double *LK = Lk + (size_t)s * K;
            int *LI = Li + (size_t)s * K;
            const int len = Llen[s];
            const bool member = has && (((k < 64 ? w0 >> k : w1 >> (k - 64)) & 1ull) != 0);
            const bool pass = member && (len < K || key_less(key, oi, LK[K - 1], LI[K - 1]));
            const unsigned bal = __ballot_sync(0xffffffffu, pass);
            if (lane == 0) wcnt[warp] = __popc(bal);
            const int cnt = __syncthreads_count(pass);
            if (cnt == 0) continue;
            if (pass) {
                int pos = __popc(bal & ((1u << lane) - 1u));
                for (int w = 0; w < warp; w++) pos += wcnt[w];
                Ck[pos] = key; Ci[pos] = oi;
            }
            __syncthreads();
            int posA = K, posB = K;
            double kA = 0.0, kB = 0.0;
            int iA = 0, iB = 0;
            if (t < len) {
                kA = LK[t]; iA = LI[t];
                int rank = 0;
                for (int j = 0; j < cnt; j++) rank += key_less(Ck[j], Ci[j], kA, iA);
                posA = t + rank;
            }
            if (t < cnt) {
                kB = Ck[t]; iB = Ci[t];
                int rank = 0;
                for (int j = 0; j < cnt; j++) rank += key_less(Ck[j], Ci[j], kB, iB);
                int lo = 0, hi = len;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (key_less(LK[mid], LI[mid], kB, iB)) lo = mid + 1; else hi = mid;
                }
                posB = lo + rank;
            }
            __syncthreads();
            if (posA < K) { LK[posA] = kA; LI[posA] = iA; }
            if (posB < K) { LK[posB] = kB; LI[posB] = iB; }
            if (t == 0) Llen[s] = min(K, len + cnt);
            __syncthreads();
        }
    }
    for (int s = 0; s < G; s++) {
        if (!((active >> s) & 1u)) continue;
        const size_t base = ((size_t)(k_lo + s - k_out0) * n + r) * K;
        const int len = Llen[s];
        for (int j = t; j < K; j += SEL_NT) {
            out_idx[base + j] = j < len ? Li[(size_t)s * K + j] : -1;
            out_key[base + j] = j < len ? Lk[(size_t)s * K + j] : INFINITY;
        }
    }
}

struct KnnTask {            // one (candidate, split) task of a vote launch
    int nn;                 // n_neighbors
    int weights;            // 0 uniform, 1 distance
    int k;                  // split
    int valid;              // 0: n_neighbors exceeds the split's training rows (no vote, the score is NaN)
};

// The distance of a list entry.  Euclidean: sqrt(max(surrogate + xsq[r], 0)); for float32 X scikit-learn's
// EuclideanDistance32._rdist_to_dist takes and returns float32, so the squared distance and its root are rounded to float32.
__device__ __forceinline__ double knn_dist(double key, double xsq_r, bool l1, bool f32)
{
    if (l1) return key;
    const double r = fmax(__dadd_rn(key, xsq_r), 0.0);
    return f32 ? (double)__double2float_rn(sqrt((double)__double2float_rn(r))) : sqrt(r);
}

// numpy's pairwise summation (np.add.reduce over a contiguous axis: 0 + pairwise_sum): below 8 terms in order, up to 128
// eight interleaved partial sums combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) then the remainder in
// order, beyond that the halves (the first a multiple of 8 long) summed separately.  term(j) gives the j-th term.
template <typename T, typename F>
__device__ __forceinline__ T pw_block(const F &term, int lo, int n)
{
    if (n < 8) {
        T res = T(0);
        for (int i = 0; i < n; i++) res = res + term(lo + i);
        return res;
    }
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = term(lo + j);
    int i = 8;
    for (; i < n - n % 8; i += 8)
#pragma unroll
        for (int j = 0; j < 8; j++) r[j] = r[j] + term(lo + i + j);
    T res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; i++) res = res + term(lo + i);
    return res;
}

template <typename T, int DEPTH, typename F>
__device__ __forceinline__ T pw_range(const F &term, int lo, int n)
{
    if (DEPTH == 0 || n <= 128) return pw_block<T>(term, lo, n);
    int n2 = n / 2;
    n2 -= n2 % 8;
    return pw_range<T, DEPTH == 0 ? 0 : DEPTH - 1>(term, lo, n2) + pw_range<T, DEPTH == 0 ? 0 : DEPTH - 1>(term, lo + n2, n - n2);
}

template <typename T, typename F>
__device__ __forceinline__ T pw_sum(const F &term, int n)      // n <= 256 needs two levels of halving
{
    return T(0) + pw_range<T, 3>(term, 0, n);
}

// One thread per (row r, task blockIdx.y): the row's vote from its list in the task's split (_get_weights: 1 / dist, or the
// indicator of zero distance when a neighbour is at distance 0; sums in neighbour order; prediction = first arg-max).
// Classifier: per-class {support, tp, predicted} of the task's test rows ([0]) and training rows ([1]) into
// counts[task][2][nc][3] (integer atomics: deterministic); proba (may be null) [task][n] = predict_proba[:, 1] (binary).
// Regressor (nc == 0): pred [task][n] = mean of the neighbours' z, or sum w z / sum w; y_f32: the uniform mean in float32
// (numpy keeps float32 y's dtype), the weighted one in float64.
template <bool CLS>
__global__ void __launch_bounds__(128, 1)
knn_vote_kernel(const int *__restrict__ li, const double *__restrict__ lk, int n, int K, int l1, const double *__restrict__ xsq,
                SplitMasks sm, int with_train, const KnnTask *__restrict__ tasks, const int *__restrict__ y_row,
                const int *__restrict__ y_orig, int nc, const double *__restrict__ z_orig, int y_f32, int x_f32,
                int *__restrict__ counts, double *__restrict__ out)
{
    extern __shared__ __align__(16) unsigned char vote_smem[];
    double *acc = (double *)vote_smem;                            // [nc][blockDim.x]
    int *sh = (int *)(acc + (size_t)nc * blockDim.x);             // [2][nc][3]
    const KnnTask T = tasks[blockIdx.y];
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    for (int i = threadIdx.x; i < 2 * nc * 3; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const bool te = r < n && split_test(sm, r, T.k);
    const bool tr = r < n && !te && with_train && split_train(sm, r, T.k);
    if ((te || tr) && T.valid) {
        const int *__restrict__ idx = li + ((size_t)T.k * n + r) * K;
        const double *__restrict__ key = lk + ((size_t)T.k * n + r) * K;
        const double xr = l1 ? 0.0 : xsq[r];
        bool zero = false;
        if (T.weights)
            for (int j = 0; j < T.nn; j++) zero |= knn_dist(key[j], xr, l1, x_f32) == 0.0;
        if (CLS) {
            for (int c = 0; c < nc; c++) acc[(size_t)c * blockDim.x + threadIdx.x] = 0.0;
            for (int j = 0; j < T.nn; j++) {
                double w = 1.0;
                if (T.weights) {
                    const double dj = knn_dist(key[j], xr, l1, x_f32);
                    w = zero ? (dj == 0.0 ? 1.0 : 0.0) : __drcp_rn(dj);
                }
                double &a = acc[(size_t)y_orig[idx[j]] * blockDim.x + threadIdx.x];
                a = __dadd_rn(a, w);
            }
            // prediction: uniform -> first arg-max of the counts (ArgKminClassMode); distance -> weighted_mode, whose class
            // sums are np.sum over the neighbours (pairwise), first arg-max among the classes present
            int pred = 0;
            double best = acc[threadIdx.x];
            if (T.weights) {
                best = -1.0;
                for (int c = 0; c < nc; c++) {
                    if (!(acc[(size_t)c * blockDim.x + threadIdx.x] > 0.0)) continue;
                    const double v = pw_sum<double>([=](int j) {
                        if (y_orig[idx[j]] != c) return 0.0;
                        const double dj = knn_dist(key[j], xr, l1, x_f32);
                        return zero ? (dj == 0.0 ? 1.0 : 0.0) : __drcp_rn(dj);
                    }, T.nn);
                    if (v > best) { best = v; pred = c; }
                }
            } else {
                for (int c = 1; c < nc; c++) {
                    const double v = acc[(size_t)c * blockDim.x + threadIdx.x];
                    if (v > best) { best = v; pred = c; }
                }
            }
            const int yc = y_row[r], sp = te ? 0 : 1;
            atomicAdd(&sh[(sp * nc + yc) * 3 + 0], 1);
            if (pred == yc) atomicAdd(&sh[(sp * nc + yc) * 3 + 1], 1);
            atomicAdd(&sh[(sp * nc + pred) * 3 + 2], 1);
            if (out && nc == 2) {
                const double a0 = acc[threadIdx.x], a1 = acc[blockDim.x + threadIdx.x];
                out[(size_t)blockIdx.y * n + r] = __ddiv_rn(a1, __dadd_rn(a0, a1));
            }
        } else {
            // np.mean(y[neigh], axis=1) (pairwise, in y's dtype), or np.sum(y w) / np.sum(w) (pairwise, float64)
            double p;
            if (!T.weights) {
                if (y_f32) p = (double)__fdiv_rn(pw_sum<float>([=](int j) { return (float)z_orig[idx[j]]; }, T.nn), (float)T.nn);
                else p = __ddiv_rn(pw_sum<double>([=](int j) { return z_orig[idx[j]]; }, T.nn), (double)T.nn);
            } else {
                auto w = [=](int j) {
                    const double dj = knn_dist(key[j], xr, l1, x_f32);
                    return zero ? (dj == 0.0 ? 1.0 : 0.0) : __drcp_rn(dj);
                };
                const double num = pw_sum<double>([=](int j) { return __dmul_rn(z_orig[idx[j]], w(j)); }, T.nn);
                const double den = pw_sum<double>(w, T.nn);
                p = __ddiv_rn(num, den);
            }
            out[(size_t)blockIdx.y * n + r] = p;
        }
    }
    if (CLS) {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * nc * 3; i += blockDim.x)
            if (sh[i]) atomicAdd(&counts[(size_t)blockIdx.y * 2 * nc * 3 + i], sh[i]);
    }
}

// scikit-learn r2_score (force_finite=True) from the residual and total sums of squares of m rows; NaN below two rows
double knn_r2(double rss, double tss, double m)
{
    if (m < 2) return NAN;
    if (tss != 0) return 1.0 - rss / tss;
    return rss == 0 ? 1.0 : 0.0;
}

// Slab rows per distance pass: the slab of float64 distances [rows][n] takes at most 1 GiB and a quarter of the free memory.
int slab_rows(int n, size_t free_bytes)
{
    const size_t cap = std::min<size_t>((size_t)1 << 30, free_bytes / 4);
    size_t rows = cap / ((size_t)n * 8);
    rows = std::max<size_t>(rows, 64);
    return (int)std::min<size_t>(rows, (size_t)n);
}

}  // namespace

// Neighbour lists of the splits [k_first, k_first + n_out) under one metric into d_idx / d_key ([n_out][n][K], rows in the
// handle's internal order, original indices in the lists).  Times: tag 0 distances, tag 1 selection.
static int knn_neighbors(gs_handle *h, int l1, int K, int k_first, int n_out, int mode, EvTimer &tm, int *d_idx, double *d_key)
{
    cudaStream_t st = h->stream;
    const int n = (int)h->n, d = (int)h->d;
    const bool f64 = h->x_dtype == GS_F64;
    const void *X = f64 ? h->dX64.p : h->dX.p;
    gs_profile &pf = h->prof;
    // xsq [n], perm [n] in dWork[0]; the distance slab in dWork[1]
    GS_CUDA(h->dWork[0].reserve((size_t)n * 12 + 64));
    double *d_xsq = h->dWork[0].as<double>();
    int *d_perm = (int *)(d_xsq + n);
    GS_CUDA(cudaMemcpyAsync(d_perm, h->perm.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    pf.h2d_bytes += (int64_t)n * 4;
    size_t fr = 0, tot = 0;
    GS_CUDA(cudaMemGetInfo(&fr, &tot));
    const int R = slab_rows(n, fr + h->dWork[1].cap);
    GS_CUDA(h->dWork[1].reserve((size_t)R * n * 8));
    double *D = h->dWork[1].as<double>();
    if (!l1) {
        if (f64) knn_sqnorm_kernel<double><<<(n + 255) / 256, 256, 0, st>>>((const double *)X, n, d, d_xsq);
        else knn_sqnorm_kernel<float><<<(n + 255) / 256, 256, 0, st>>>((const float *)X, n, d, d_xsq);
        GS_CUDA(cudaGetLastError());
        pf.launches++;
    }
    const size_t per_split = (size_t)K * 12 + 4;
    const int gmax = std::max(1, std::min(SEL_MAX_G, (int)((SEL_SMEM - SEL_NT * 12 - 64) / per_split)));
    GS_CUDA(cudaFuncSetAttribute(knn_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SEL_SMEM));
    for (int r0 = 0; r0 < n; r0 += R) {
        const int rows = std::min(R, n - r0);
        dim3 grid((n + DT - 1) / DT, (rows + DT - 1) / DT);
        tm.mark(-1);
        if (f64) {
            if (l1) knn_dist_kernel<double, true><<<grid, 256, 0, st>>>((const double *)X, n, d, r0, rows, d_xsq, D);
            else knn_dist_kernel<double, false><<<grid, 256, 0, st>>>((const double *)X, n, d, r0, rows, d_xsq, D);
        } else {
            if (l1) knn_dist_kernel<float, true><<<grid, 256, 0, st>>>((const float *)X, n, d, r0, rows, d_xsq, D);
            else knn_dist_kernel<float, false><<<grid, 256, 0, st>>>((const float *)X, n, d, r0, rows, d_xsq, D);
        }
        GS_CUDA(cudaGetLastError());
        pf.launches++;
        pf.gram_flops += 2.0 * rows * (double)n * d;
        pf.gram_bytes += (double)rows * n * 8;
        tm.mark(0);
        for (int g0 = 0; g0 < n_out; g0 += gmax) {
            const int G = std::min(gmax, n_out - g0);
            const size_t smem = (size_t)G * per_split + SEL_NT * 12;
            knn_select_kernel<<<rows, SEL_NT, smem, st>>>(D, n, r0, d_perm, h->masks(), k_first + g0, G, K, mode, k_first,
                                                         d_idx, d_key);
            GS_CUDA(cudaGetLastError());
            pf.launches++;
            pf.solve_bytes += (double)rows * n * 8 + (double)rows * G * K * 12;
        }
        tm.mark(1);
    }
    return GS_OK;
}

static int knn_run(gs_handle *h, int n_cand, const int32_t *nn, const int32_t *weights, const int32_t *metric, uint32_t flags,
                   double *test_scores, double *train_scores, float *fit_ms, float *score_ms)
{
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) { gs_set_error(h, "gs_knn: no dataset (call gs_set_data first)"); return GS_ERR_NO_DATA; }
    if (n_cand <= 0 || !nn || !weights || !metric || !test_scores) { gs_set_error(h, "gs_knn: bad arguments"); return GS_ERR_ARG; }
    if (!h->sample_w.empty() || h->class_w_sets > 0) { gs_set_error(h, "gs_knn: k-NN fits take no sample or class weights"); return GS_ERR_ARG; }
    const bool classif = h->classification;
    const int nc = classif ? h->n_classes : 0;
    if (classif && nc > 64) { gs_set_error(h, "gs_knn: more than 64 classes"); return GS_ERR_UNSUPPORTED; }
    if (!classif && h->z64.empty()) { gs_set_error(h, "gs_knn: no float64 targets (call gs_set_targets_f64 after gs_set_data)"); return GS_ERR_NO_DATA; }
    const int kind = h->score_kind;
    const bool reg_kind = kind == GS_SCORE_DEFAULT || kind == GS_SCORE_NEG_MSE || kind == GS_SCORE_NEG_RMSE;
    if (!classif && !reg_kind) { gs_set_error(h, "gs_knn: classification scorer on a regressor"); return GS_ERR_ARG; }
    if (classif && (kind == GS_SCORE_NEG_MSE || kind == GS_SCORE_NEG_RMSE)) { gs_set_error(h, "gs_knn: regression scorer on a classifier"); return GS_ERR_ARG; }
    if (classif && kind == GS_SCORE_ROC_AUC && nc != 2) { gs_set_error(h, "gs_knn: roc_auc needs two classes"); return GS_ERR_UNSUPPORTED; }
    for (int c = 0; c < n_cand; c++) {
        if (nn[c] < 1 || nn[c] > GS_KNN_MAX_NEIGHBORS) { gs_set_error(h, "gs_knn: n_neighbors must be in 1.." + std::to_string(GS_KNN_MAX_NEIGHBORS)); return GS_ERR_UNSUPPORTED; }
        if (weights[c] != GS_KNN_UNIFORM && weights[c] != GS_KNN_DISTANCE) { gs_set_error(h, "gs_knn: unknown weights code"); return GS_ERR_ARG; }
        if (metric[c] != GS_KNN_EUCLIDEAN && metric[c] != GS_KNN_MANHATTAN) { gs_set_error(h, "gs_knn: unknown metric code"); return GS_ERR_ARG; }
    }
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int n = (int)h->n, ns = h->n_splits;
    const bool with_train = (flags & GS_RETURN_TRAIN) && train_scores;
    const int n_tasks = n_cand * ns;

    // training rows of every split, and the sizes / r2 denominators of its test and training sets (original row order)
    std::vector<int> by_orig(n);
    for (int r = 0; r < n; r++) by_orig[h->perm[r]] = r;
    std::vector<double> m_train(ns, 0.0), cnt((size_t)ns * 2, 0.0), tss((size_t)ns * 2, 0.0);
    std::vector<double> na((size_t)ns * 2, 0.0), nb((size_t)ns * 2, 0.0);        // roc_auc: class-0 / class-1 rows per set
    for (int k = 0; k < ns; k++) {
        double sum[2] = {0, 0};
        for (int o = 0; o < n; o++) {
            const int r = by_orig[o];
            const bool te = h->is_test(r, k), tr = h->is_train(r, k);
            if (tr) m_train[k] += 1;
            const int sp = te ? 0 : (tr ? 1 : -1);
            if (sp < 0) continue;
            cnt[(size_t)k * 2 + sp] += 1;
            if (classif) ((h->yc[r] == 0 ? na : nb)[(size_t)k * 2 + sp]) += 1;
            else sum[sp] += h->z64[r];
        }
        if (!classif)
            for (int sp = 0; sp < 2; sp++) {
                const double m = cnt[(size_t)k * 2 + sp], mean = m > 0 ? sum[sp] / m : 0.0;
                double s = 0;
                for (int o = 0; o < n; o++) {
                    const int r = by_orig[o];
                    const bool te = h->is_test(r, k), tr = !te && h->is_train(r, k);
                    if (sp == 0 ? te : tr) { const double e = h->z64[r] - mean; s += e * e; }
                }
                tss[(size_t)k * 2 + sp] = s;
            }
    }

    gs_profile &pf = h->prof;
    const float keep_h2d = pf.ms_h2d;
    const int64_t keep_h2d_bytes = pf.h2d_bytes;
    memset(&pf, 0, sizeof pf);
    pf.ms_h2d = keep_h2d; pf.h2d_bytes = keep_h2d_bytes;
    h->evp.reset();
    EvTimer tm(st, h->evp);
    float acc[3] = {0, 0, 0};
    cudaEvent_t ev0 = h->evp.get(), ev1 = h->evp.get();
    cudaEventRecord(ev0, st);
    tm.mark(-1);

    // labels / targets by ORIGINAL row (the lists hold original indices), class of every internal row, zero intercepts
    GS_CUDA(h->dWork[5].reserve((size_t)n * 12 + (size_t)n_tasks * 8 + 256));
    int *d_yorig = h->dWork[5].as<int>();
    double *d_zorig = (double *)(h->dWork[5].as<unsigned char>() + (((size_t)n * 4 + 15) & ~(size_t)15));
    double *d_zero = d_zorig + n;
    GS_CUDA(cudaMemsetAsync(d_zero, 0, (size_t)n_tasks * 8, st));
    if (classif) {
        std::vector<int> yo(n);
        for (int r = 0; r < n; r++) yo[h->perm[r]] = h->yc[r];
        GS_CUDA(cudaMemcpyAsync(d_yorig, yo.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaStreamSynchronize(st));
    } else {
        std::vector<double> zo(n);
        for (int r = 0; r < n; r++) zo[h->perm[r]] = h->z64[r];
        GS_CUDA(cudaMemcpyAsync(d_zorig, zo.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaStreamSynchronize(st));
    }
    pf.h2d_bytes += (int64_t)n * (classif ? 4 : 8);

    std::vector<double> sc_test(n_tasks, NAN), sc_train(n_tasks, NAN);
    for (int met = 0; met < 2; met++) {
        std::vector<int> cands;
        int K = 0;
        for (int c = 0; c < n_cand; c++)
            if (metric[c] == met) { cands.push_back(c); K = std::max(K, (int)nn[c]); }
        if (cands.empty()) continue;
        // ---- 1 + 2. distances and neighbour lists [ns][n][K] ----
        const size_t list_bytes = (size_t)ns * n * K;
        size_t fr = 0, tot = 0;
        GS_CUDA(cudaMemGetInfo(&fr, &tot));
        const size_t have = h->dWork[2].cap + h->dWork[3].cap;
        if (list_bytes * 12 > have && list_bytes * 12 - have + ((size_t)64 << 20) > fr) {
            gs_set_error(h, "gs_knn: the neighbour lists (" + std::to_string(list_bytes * 12 >> 20) + " MiB) do not fit in free device memory");
            return GS_ERR_UNSUPPORTED;
        }
        GS_CUDA(h->dWork[2].reserve(list_bytes * 4));
        GS_CUDA(h->dWork[3].reserve(list_bytes * 8));
        int *d_idx = h->dWork[2].as<int>();
        double *d_key = h->dWork[3].as<double>();
        if (const int rc = knn_neighbors(h, met == GS_KNN_MANHATTAN, K, 0, ns, with_train ? 1 : 0, tm, d_idx, d_key)) return rc;
        const double *d_xsq = h->dWork[0].as<double>();

        // ---- 3. votes and scorers, candidates in batches whose per-row outputs take at most 512 MiB ----
        const bool need_out = !classif || kind == GS_SCORE_ROC_AUC;
        const int per = std::max(1, (int)std::min<size_t>(cands.size(), ((size_t)512 << 20) / ((size_t)ns * n * 8)));
        for (int b0 = 0; b0 < (int)cands.size(); b0 += per) {
            const int b1 = std::min((int)cands.size(), b0 + per);
            const int nt = (b1 - b0) * ns;
            std::vector<KnnTask> tasks(nt);
            std::vector<VoteTask> vt(nt);
            std::vector<int> col(nt), fold(nt);
            for (int i = b0; i < b1; i++)
                for (int k = 0; k < ns; k++) {
                    const int q = (i - b0) * ns + k, c = cands[i];
                    tasks[q] = KnnTask{(int)nn[c], (int)weights[c], k, nn[c] <= m_train[k] ? 1 : 0};
                    vt[q] = VoteTask{q, k};
                    col[q] = q; fold[q] = k;
                }
            const size_t cnt_bytes = classif ? (size_t)nt * 2 * nc * 3 * 4 : 0;
            const size_t meta = (size_t)nt * (sizeof(KnnTask) + sizeof(VoteTask) + 8);
            GS_CUDA(h->dWork[6].reserve(meta + 64));
            unsigned char *dm = h->dWork[6].as<unsigned char>();
            KnnTask *d_tasks = (KnnTask *)dm;
            VoteTask *d_vt = (VoteTask *)(dm + (size_t)nt * sizeof(KnnTask));
            int *d_col = (int *)(dm + (size_t)nt * (sizeof(KnnTask) + sizeof(VoteTask)));
            int *d_fold = d_col + nt;
            GS_CUDA(cudaMemcpyAsync(d_tasks, tasks.data(), (size_t)nt * sizeof(KnnTask), cudaMemcpyHostToDevice, st));
            GS_CUDA(cudaMemcpyAsync(d_vt, vt.data(), (size_t)nt * sizeof(VoteTask), cudaMemcpyHostToDevice, st));
            GS_CUDA(cudaMemcpyAsync(d_col, col.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, st));
            GS_CUDA(cudaMemcpyAsync(d_fold, fold.data(), (size_t)nt * 4, cudaMemcpyHostToDevice, st));
            pf.h2d_bytes += (int64_t)meta;
            double *d_out = nullptr;
            if (need_out) {
                GS_CUDA(h->dWork[4].reserve((size_t)nt * n * 8));
                d_out = h->dWork[4].as<double>();
                GS_CUDA(cudaMemsetAsync(d_out, 0, (size_t)nt * n * 8, st));
            }
            const size_t score_bytes = std::max(cnt_bytes, (size_t)nt * 4 * 8);
            GS_CUDA(h->dScore.reserve(score_bytes));
            GS_CUDA(cudaMemsetAsync(h->dScore.p, 0, score_bytes, st));
            const int vnt = nc > 32 ? 64 : 128;
            const size_t vsmem = (size_t)nc * vnt * 8 + (size_t)2 * nc * 3 * 4;
            for (int t0 = 0; t0 < nt; t0 += 32768) {                     // gridDim.y <= 65535
                const int tn = std::min(32768, nt - t0);
                dim3 grid((n + vnt - 1) / vnt, tn);
                auto vote = classif ? knn_vote_kernel<true> : knn_vote_kernel<false>;
                vote<<<grid, vnt, vsmem, st>>>(d_idx, d_key, n, K, met == GS_KNN_MANHATTAN, d_xsq, h->masks(), with_train ? 1 : 0,
                                               d_tasks + t0, h->dY.as<int>(), d_yorig, nc, d_zorig, (flags & GS_TARGET_F32) ? 1 : 0,
                                               h->x_dtype == GS_F32 ? 1 : 0, classif ? h->dScore.as<int>() + (size_t)t0 * 2 * nc * 3 : nullptr,
                                               d_out ? d_out + (size_t)t0 * n : nullptr);
                GS_CUDA(cudaGetLastError());
                pf.launches++;
            }
            if (classif && kind == GS_SCORE_ROC_AUC) {
                GS_CUDA(cudaMemsetAsync(h->dScore.p, 0, (size_t)nt * 4 * 8, st));
                GS_CUDA(launch_auc_pairs_f64(d_out, n, n, h->class_start[1], h->masks(), d_col, d_fold, nt, +1,
                                             h->dScore.as<unsigned long long>(), st));
                pf.launches++;
            } else if (!classif) {
                GS_CUDA(launch_rss(d_out, d_zero, n, h->dZ64.as<double>(), h->masks(), d_vt, nt, h->dScore.as<double>(), st));
                pf.launches++;
            }
            tm.mark(2);
            std::vector<unsigned char> host(score_bytes);
            GS_CUDA(cudaMemcpyAsync(host.data(), h->dScore.p, score_bytes, cudaMemcpyDeviceToHost, st));
            GS_CUDA(cudaStreamSynchronize(st));
            pf.d2h_bytes += (int64_t)score_bytes;
            for (int q = 0; q < nt; q++) {
                const int c = cands[b0 + q / ns], k = q % ns, t = c * ns + k;
                if (!tasks[q].valid) continue;
                for (int sp = 0; sp < 2; sp++) {
                    double s;
                    if (classif && kind == GS_SCORE_ROC_AUC) {
                        const unsigned long long *a = (const unsigned long long *)host.data() + (size_t)q * 4 + sp * 2;
                        const double pairs = na[(size_t)k * 2 + sp] * nb[(size_t)k * 2 + sp];
                        s = pairs > 0 ? ((double)a[0] + 0.5 * (double)a[1]) / pairs : NAN;
                    } else if (classif) {
                        s = gs_score_from_counts(kind, h->score_pos, nc, (const int *)host.data() + ((size_t)q * 2 + sp) * nc * 3);
                    } else {
                        const double rss = ((const double *)host.data())[(size_t)q * 2 + sp], m = cnt[(size_t)k * 2 + sp];
                        if (!(m > 0)) s = NAN;
                        else if (kind == GS_SCORE_NEG_MSE) s = -(rss / m);
                        else if (kind == GS_SCORE_NEG_RMSE) s = -std::sqrt(rss / m);
                        else s = knn_r2(rss, tss[(size_t)k * 2 + sp], m);
                    }
                    (sp == 0 ? sc_test : sc_train)[t] = s;
                }
            }
            tm.mark(-1);
        }
    }
    cudaEventRecord(ev1, st);
    GS_CUDA(cudaStreamSynchronize(st));
    tm.collect(acc, 3);
    cudaEventElapsedTime(&pf.ms_total, ev0, ev1);
    pf.ms_gram = acc[0]; pf.ms_solve = acc[1]; pf.ms_score = acc[2];
    for (int t = 0; t < n_tasks; t++) {
        test_scores[t] = sc_test[t];
        if (with_train) train_scores[t] = sc_train[t];
        if (fit_ms) fit_ms[t] = (pf.ms_gram + pf.ms_solve) / (float)n_tasks;
        if (score_ms) score_ms[t] = pf.ms_score / (float)n_tasks;
    }
    return GS_OK;
}

extern "C" {

int gs_knn(gs_handle *h, int32_t n_cand, const int32_t *n_neighbors, const int32_t *weights, const int32_t *metric,
           uint32_t flags, double *test_scores, double *train_scores, float *fit_ms, float *score_ms)
{
    return knn_run(h, n_cand, n_neighbors, weights, metric, flags, test_scores,
                   (flags & GS_RETURN_TRAIN) ? train_scores : nullptr, fit_ms, score_ms);
}

int gs_debug_knn_neighbors(gs_handle *h, int32_t metric, int32_t k, int32_t split, int32_t *idx_out, double *dist_out)
{
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) { gs_set_error(h, "gs_debug_knn_neighbors: no dataset (call gs_set_data first)"); return GS_ERR_NO_DATA; }
    if ((metric != GS_KNN_EUCLIDEAN && metric != GS_KNN_MANHATTAN) || k < 1 || k > GS_KNN_MAX_NEIGHBORS || split < 0 ||
        split >= h->n_splits) {
        gs_set_error(h, "gs_debug_knn_neighbors: bad arguments"); return GS_ERR_ARG;
    }
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int n = (int)h->n;
    h->evp.reset();
    EvTimer tm(st, h->evp);
    GS_CUDA(h->dWork[2].reserve((size_t)n * k * 4));
    GS_CUDA(h->dWork[3].reserve((size_t)n * k * 8));
    if (const int rc = knn_neighbors(h, metric == GS_KNN_MANHATTAN, k, split, 1, 2, tm, h->dWork[2].as<int>(), h->dWork[3].as<double>()))
        return rc;
    std::vector<int> idx((size_t)n * k);
    std::vector<double> key((size_t)n * k), xsq(n, 0.0);
    GS_CUDA(cudaMemcpyAsync(idx.data(), h->dWork[2].p, idx.size() * 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaMemcpyAsync(key.data(), h->dWork[3].p, key.size() * 8, cudaMemcpyDeviceToHost, st));
    if (metric == GS_KNN_EUCLIDEAN) GS_CUDA(cudaMemcpyAsync(xsq.data(), h->dWork[0].p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaStreamSynchronize(st));
    tm.collect(nullptr, 0);
    for (int r = 0; r < n; r++) {
        const int o = h->perm[r];
        for (int j = 0; j < k; j++) {
            const int i = idx[(size_t)r * k + j];
            const double kv = key[(size_t)r * k + j];
            if (idx_out) idx_out[(size_t)o * k + j] = i;
            if (dist_out)
                dist_out[(size_t)o * k + j] = i < 0 ? INFINITY : (metric == GS_KNN_MANHATTAN ? kv
                                  : h->x_dtype == GS_F32 ? (double)(float)std::sqrt((double)(float)std::max(kv + xsq[r], 0.0))
                                                         : std::sqrt(std::max(kv + xsq[r], 0.0)));
        }
    }
    return GS_OK;
}

}  // extern "C"
