// common.cuh -- shared declarations of the libb200gs.so translation units (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <cmath>
#include <cstring>
#include <functional>
#include <string>
#include <vector>
#include "../../include/b200gs.h"

inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

#define GS_CUDA(call)                                                                         \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess) {                                                              \
            gs_set_error(h, std::string(#call) + ": " + cudaGetErrorString(e_) + " @" +       \
                                __FILE__ + ":" + std::to_string(__LINE__));                   \
            return GS_ERR_CUDA;                                                               \
        }                                                                                     \
    } while (0)

// grow-only device buffer
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes)
    {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T *as() const { return (T *)p; }
};

// CUDA events owned by the handle: created on first use, reused by every later call, destroyed with the handle
// (no per-call cudaEventCreate / cudaEventDestroy, nothing to leak on an error return)
struct EventPool {
    std::vector<cudaEvent_t> ev;
    size_t used = 0;
    cudaEvent_t get()
    {
        if (used == ev.size()) { cudaEvent_t e = nullptr; cudaEventCreate(&e); ev.push_back(e); }
        return ev[used++];
    }
    void reset() { used = 0; }
    void release() { for (auto e : ev) cudaEventDestroy(e); ev.clear(); used = 0; }
};

// CUDA-event time and executed MMA flops of the tensor-core contraction launches of one call
struct TensorTimer {
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> spans;
    double flops = 0;
    cudaEvent_t open = nullptr;
    void reset() { spans.clear(); flops = 0; open = nullptr; }
    void begin(EventPool &p, cudaStream_t st) { open = p.get(); cudaEventRecord(open, st); }
    void end(EventPool &p, cudaStream_t st, double f)
    {
        cudaEvent_t e = p.get();
        cudaEventRecord(e, st);
        spans.emplace_back(open, e); flops += f;
    }
    float collect()                      // the stream must have been synchronised
    {
        float tot = 0;
        for (auto &s : spans) { float ms = 0; if (cudaEventElapsedTime(&ms, s.first, s.second) == cudaSuccess) tot += ms; }
        return tot;
    }
};

struct EvTimer {       // accumulates elapsed ms between consecutive marks on one stream (events from the handle's pool)
    cudaStream_t st;
    EventPool &pool;
    std::vector<cudaEvent_t> evs;
    std::vector<int> tag;
    EvTimer(cudaStream_t s, EventPool &p) : st(s), pool(p) {}
    void mark(int t)
    {
        cudaEvent_t e = pool.get();
        cudaEventRecord(e, st);
        evs.push_back(e); tag.push_back(t);
    }
    // after a stream sync: add the time between mark k-1 and mark k to acc[tag[k]]
    void collect(float *acc, int ntags)
    {
        for (size_t k = 1; k < evs.size(); k++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, evs[k - 1], evs[k]);
            if (tag[k] >= 0 && tag[k] < ntags) acc[tag[k]] += ms;
        }
        evs.clear(); tag.clear();
    }
};

// Membership of every row in the training / test set of every CV split: two 64-bit words per row and kind (splits 0..127).
// Replaces the per-task index arrays of the reference (base_search.py:81-82 islice(cv.split(...))): any splitter fits --
// overlapping test sets (RepeatedKFold), rows in neither set (ShuffleSplit), rows that only ever train (PredefinedSplit -1).
struct SplitMasks {
    const unsigned long long *te, *tr;
};
// scikit-learn r2_score (metrics/_regression.py, force_finite=True) from the residual and total sums of squares of m rows:
// NaN below two rows (UndefinedMetricWarning); a constant target (tss == 0) scores 1.0 when predicted exactly, else 0.0
__host__ __device__ inline double gs_r2_score(double rss, double tss, double m)
{
    if (m < 2) return NAN;
    if (tss != 0) return 1.0 - rss / tss;
    return rss == 0 ? 1.0 : 0.0;
}
#ifdef __CUDACC__
__device__ __forceinline__ bool split_test(const SplitMasks &m, int r, int k)      // k < 0 (refit): nobody is tested
{
    return k >= 0 && ((m.te[(size_t)r * 2 + (k >> 6)] >> (k & 63)) & 1ull);
}
__device__ __forceinline__ bool split_train(const SplitMasks &m, int r, int k)     // k < 0 (refit): every row trains
{
    return k < 0 || ((m.tr[(size_t)r * 2 + (k >> 6)] >> (k & 63)) & 1ull);
}
// libsvm's poly / sigmoid kernel of a dot product s (svm.cpp Kernel::kernel_poly, kernel_sigmoid, powi), every operation
// rounded on its own (no contraction): poly = powi(gamma*s + coef0, degree) by square-and-multiply, sigmoid = tanh(...)
__device__ __forceinline__ double gs_kernel_of_dot(int kernel, double s, double gamma, int degree, double coef0)
{
    const double a = __dadd_rn(__dmul_rn(gamma, s), coef0);
    if (kernel == GS_KERNEL_SIGMOID) return tanh(a);
    double tmp = a, ret = 1.0;
    for (int t = degree; t > 0; t /= 2) {
        if (t % 2 == 1) ret = __dmul_rn(ret, tmp);
        tmp = __dmul_rn(tmp, tmp);
    }
    return ret;
}
#endif

struct gs_handle {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaStream_t stream_hi = nullptr;   // second stream: the single-CTA SMO launch when a cluster launch runs beside it
    cudaStream_t stream_lo = nullptr;   // third stream: the shared-SM launch when cluster and exclusive-SM launches run beside it
    std::string err;
    // dataset (rows stored in INTERNAL order: sorted by class, then by original index)
    int64_t n = 0, d = 0;
    int n_splits = 0, n_classes = 0;
    bool classification = false;
    std::vector<int32_t> perm;        // internal row -> original row
    std::vector<int32_t> yc;          // [n] class ids, internal order
    std::vector<int8_t> fold;         // [n] fold ids, internal order (partition splitters; Ridge's fold blocks)
    std::vector<uint64_t> te_mask, tr_mask;   // [n][2] split membership, internal order
    bool partition = true;            // the splits are a partition into test folds whose complements train (gs_set_data's fold ids)
    bool is_test(int r, int k) const { return k >= 0 && ((te_mask[(size_t)r * 2 + (k >> 6)] >> (k & 63)) & 1ull); }
    bool is_train(int r, int k) const { return k < 0 || ((tr_mask[(size_t)r * 2 + (k >> 6)] >> (k & 63)) & 1ull); }
    SplitMasks masks() const { return SplitMasks{dTe.as<unsigned long long>(), dTr.as<unsigned long long>()}; }
    std::vector<int32_t> class_start; // [n_classes+1] internal row ranges per class
    DevBuf dX, dY, dFold, dYt;        // float X[n][d], int32 y[n], int8 fold[n], float yt[n]
    DevBuf dTe, dTr;                  // uint64 [n][2] test / training membership of every split
    DevBuf dX64;                      // double X[n][d] when the caller's matrix is float64
    int x_dtype = GS_F32;
    DevBuf dS, dXsq;                  // float64 Gram [n][n], squared norms [n]
    DevBuf dK;                        // float32 kernel matrices (batch)
    DevBuf dWork[9];                  // per-search scratch
    DevBuf dScore;                    // every search's scoring scratch: class counts, AUC pair counts, residual sums of squares
    int score_kind = 0, score_pos = 1;   // gs_set_scoring
    std::vector<double> class_w;         // gs_set_class_weight: [sets][n_classes]; empty = all ones
    int class_w_sets = 0;
    std::vector<float> sample_w;         // gs_set_sample_weight: [n] internal order; empty = all ones
    std::vector<double> sample_w64;      // the same weights in float64 (gs_linsvc; valid while sample_w is not empty)
    DevBuf dSw;                          // its device copy
    std::vector<int32_t> kp_degree;      // gs_set_kernel_params: per-candidate degree / coef0 of the next SVC call; empty = 3 / 0
    std::vector<double> kp_coef0;
    std::vector<double> z64;             // gs_set_targets_f64: [n] float64 regression targets, internal order; empty = not set
    DevBuf dZ64;                         // their device copy
    std::vector<int32_t> train_order;    // gs_set_train_order: training rows (original indices) of every split, in fit order;
    std::vector<int64_t> train_off;      // split k's are train_order[train_off[k] .. train_off[k + 1]); empty = ascending
    gs_profile prof;
    EventPool evp;                    // timing events of the current call
    TensorTimer tt;
};

void gs_set_error(gs_handle *h, const std::string &msg);

// ---- gram.cu ----
// S = X X^T in float64 from float32 X (exact products, float64 accumulation); xsq = diag(S).
cudaError_t launch_gram_f64(const void *X, int x_dtype, int n, int d, double *S, double *xsq, cudaStream_t st);
cudaError_t launch_widen_gram(const float *S32, int n, int64_t ld32, double *S, double *xsq, cudaStream_t st);
// K[r][c] = (float) k(x_r, x_c) from S: rbf exp(-gamma*(xsq_r + xsq_c - 2 S_rc)), linear S_rc, or libsvm's poly / sigmoid
// of S_rc (degree and coef0 are read by those two only).  qd (may be null): [n] float64 k(x_r, x_r), rows in S's order.
// *special (device int, pre-zeroed, may be null) is set when an entry is not a positive normal float.
cudaError_t launch_kernel_matrix(const double *S, const double *xsq, int n, int kernel, double gamma, int degree, double coef0,
                                 float *K, int64_t ldk, double *qd, int *special, cudaStream_t st);

// ---- smo.cu ----
struct SmoProblem {
    const float *K;       // float32 kernel matrix of this (kernel, gamma): [n][ldk]
    const double *qd;     // float64 diagonal by dataset row (linear, poly, sigmoid) or nullptr (rbf: QD == 1)
    const int *rows;      // [l] dataset rows in sub-problem order: n_pos rows of the +1 class first
    double *alpha;        // [l] workspace: alpha by position
    double *Gbar;         // [l] workspace
    int *scratch;         // [2*l + 64] workspace
    double *coef;         // [n] out: alpha*y scattered by dataset row (pre-zeroed)
    double *out_rho;      // out
    int *out_info;        // out: [0] n_iter [1] timed_out [2] n_sv [3] n_bounded_sv
    unsigned long long *out_ns;   // out: [0] start [1] end (globaltimer)
    // Device flag written by kernel_matrix_kernel: != 0 when K holds a zero, denormal or negative entry.  Both solver
    // instances are enqueued behind it; the branch-free (FAST) one returns at once when it is set, the general one when it
    // is clear -- the choice needs no host round trip in the middle of a search.  nullptr: run unconditionally.
    const int *guard;
    int64_t ldk;
    double C, Cn, eps;    // C of the +1 class (the pair's first class) and of the -1 class: C x class_weight
    int l, n_pos, max_iter, shrinking;
    // up to 4 column ranges (floats, multiples of 4) that cover this sub-problem's dataset rows: the single-CTA kernel
    // copies only these parts of a K row into shared memory (a fold's training rows are 2-3 contiguous runs of the
    // class-sorted dataset: 32 KB of a 40 KB row in config 2).  nseg == 0: copy the whole row.
    int nseg, seg_start[4], seg_len[4];
    int nslots;           // sum of seg_len: size of the slot space of smo_lean.cu (0 when nseg == 0)
};
int smo_max_rows();   // largest sub-problem the resident-state kernel supports
// epsilon-SVR data of one problem (parallel to SmoProblem; only the SVR instances read it)
struct SvrData {
    const double *z;      // [n] float64 targets by dataset row
    double eps;           // SVR epsilon (libsvm's p)
};
// nu-SVC / nu-SVR starting point of one problem (parallel to SmoProblem; only the nu instances read it): the sums that
// libsvm hands out greedily, min(C, remaining) in position order, to the +1 positions and to the -1 positions
struct NuData {
    double sum_pos, sum_neg;
};
// The position-owned kernel: solves problems order[0..n_prob) (one CTA each); lmax = max l selects the template instance,
// *why says why an lmax is not supported.  Parallel to d_probs, d_svr and d_nu (each may be null) select the model:
//   * neither: C-SVC;
//   * d_svr: epsilon-SVR: problem q has l = 2 x (training rows) positions, rows[] = the training rows (ascending original
//     index) twice, n_pos = l / 2; svr[q] holds its targets and epsilon.  coef gets alpha+ - alpha- by row;
//   * d_nu: libsvm's Solver_NU, nu-SVC (C = Cn = 1, coef = alpha y / r, rho / r), or with d_svr nu-SVR on the SVR layout
//     with svr[q].eps = 0 (linear term -/+ z).
cudaError_t launch_smo(const SmoProblem *d_probs, const SvrData *d_svr, const NuData *d_nu, const int *d_order, int n_prob,
                       int lmax, bool fast, int rowcap, cudaStream_t st, std::string *why);
// smo_lean.cu: the throughput instance (static slots = the problem's column runs, two or more sub-problems per SM).  Every
// problem of the launch needs a slot layout: nseg > 0, nslots <= smo_lean_max_slots(), l < 16383; alpha and Gbar hold nslots doubles.
int smo_lean_max_slots();
// exclusive: one sub-problem per SM (the launch asks for more than half of an SM's shared memory)
cudaError_t launch_smo_lean(const SmoProblem *d_probs, const int *d_order, int n_prob, int max_slots, bool fast, bool exclusive, cudaStream_t st);
// smo_colown.cu: the same solver with one sub-problem spread over a thread-block cluster of cl CTAs (DSMEM exchange)
int smo_colown_max_rows(int cl);
void launch_delay(unsigned ns, cudaStream_t st);      // one thread sleeping ns nanoseconds (stream-ordering aid)
cudaError_t launch_smo_colown(const SmoProblem *d_probs, const int *d_order, int n_prob, int lmax, int cl, bool fast, cudaStream_t st);

// ---- score.cu ----
// dec[c][r] = sum_j k64(r, j) * coef[c][j]  (float64 kernel values recomputed from S, not the
// float32-rounded K: svm.cpp:2821 svm_predict_values uses k_function in double).
// decision_chunks: into how many slabs the support-row range of one launch is split so that its CTAs fill the GPU in whole
// rounds (157 row blocks on 528 resident CTAs of 132 SMs: 4 slabs = 628 CTAs = two rounds for 1.19 rounds of work; 10 slabs = 2.97).
int decision_chunks(int n, int ncols, int sms);
cudaError_t launch_decision(const double *S, const double *xsq, int n, int kernel, double gamma, int degree, double coef0,
                            const double *coef, int ncols, double *dec, double *part, int jchunks, cudaStream_t st);
struct VoteTask {          // one (candidate, fold) task
    int first_col;         // first decision column of this task inside its group (n_pairs consecutive)
    int fold;              // test fold id
};
// counts[task][0..3] = {test correct, test total, train correct, train total}
cudaError_t launch_vote(const double *dec, const double *rho, int n, int n_classes, const int *y,
                        SplitMasks sm, const VoteTask *tasks, int n_tasks, int *counts,
                        cudaStream_t st);

// per-class counts for the count-based scorers: counts[task][split (0 test, 1 train)][class][3 = support, tp, predicted]
cudaError_t launch_vote_classes(const double *dec, const double *rho, int n, int n_classes, const int *y,
                                SplitMasks sm, const VoteTask *tasks, int n_tasks, int *counts, cudaStream_t st);
// ROC-AUC pair counts of binary tasks: out[task][4] = {test wins, test ties, train wins, train ties}; rows are class-sorted
// (negative class = rows [0, n_a)); score row of task t = score + col_of_task[t] * ld; sign -1 for libsvm decision values
cudaError_t launch_auc_pairs_f64(const double *score, int64_t ld, int n, int n_a, SplitMasks sm, const int *col_of_task,
                                 const int *fold_of_task, int n_tasks, int sign, unsigned long long *out, cudaStream_t st);
cudaError_t launch_auc_pairs_f32(const float *score, int64_t ld, int n, int n_a, SplitMasks sm, const int *col_of_task,
                                 const int *fold_of_task, int n_tasks, int sign, unsigned long long *out, cudaStream_t st);
// Residual sums of squares of regression tasks: rss[task][0 test, 1 train] = sum over the split's rows of
// (z_r - (dec[first_col][r] - rho[first_col]))^2, float64, fixed-order block reduction (deterministic, no atomics).
cudaError_t launch_rss(const double *dec, const double *rho, int n, const double *z, SplitMasks sm, const VoteTask *tasks,
                       int n_tasks, double *rss, cudaStream_t st);
// score of one (task, split) from the class counts cnt[class][3] (float64, scikit-learn's formulas); NaN when undefined
double gs_score_from_counts(int kind, int pos_class, int n_classes, const int *cnt);
// Rejects, with who in the message, a scorer the dataset cannot take: a classification scorer on a regressor or a
// regression scorer on a classifier (GS_ERR_ARG), f1 / precision / recall / roc_auc without exactly two classes
// (GS_ERR_UNSUPPORTED), a scorer other than the default whose positive class is not a class of the dataset (GS_ERR_ARG).
// Every search calls it before its device work; a refit does not score.
int check_scorer(gs_handle *h, const char *who, int kind);
// The score denominators of every split k and part sp (0 test, 1 train: its training rows that are not test rows), and the
// formulas that turn a search's device outputs into kind's score (float64, scikit-learn's; NaN when undefined).  One host
// pass over the rows, none for the count-based scorers, which carry their own totals.
struct SplitScoreStats {
    int kind, pos_class, n_classes;
    std::vector<double> rows, n_a, n_b;   // [ns][2]: rows; of those, rows of the first / second class (classifier)
    std::vector<double> tss;              // [ns][2], regressor: total sum of squares of the float64 targets about their mean,
                                          // in ascending original row order as scikit-learn's y[test] / y[train]
    SplitScoreStats(const gs_handle *h, int ns, int kind);
    static double accuracy(const int *vote);                         // {correct, total} of launch_vote
    double auc(int k, int sp, const unsigned long long *pairs) const;   // {wins, ties} of launch_auc_pairs_*
    double counts(const int *cnt) const;                               // cnt[class][3]: gs_score_from_counts
    double regression(int k, int sp, double rss) const;                // r2 / neg MSE / neg RMSE from a residual sum of squares
};

// ---- kernel_svm.cu: the batch loop of the SVC, NuSVC, SVR and NuSVR searches and refits (an int return is a GS_* status) ----
int build_gram(gs_handle *h, uint32_t flags, cudaStream_t st);   // S = X X^T -> h->dS, diag(S) -> h->dXsq
// One kernel matrix: the kernel and the parameters it reads.  Parameters a kernel ignores are stored as 0 (linear: all three,
// rbf: degree and coef0, sigmoid: degree), so candidates that differ only in them share the matrix.
struct KernelSpec {
    int kernel;
    double gamma;
    int degree;
    double coef0;
    KernelSpec(int k, double g, int deg, double c0)
        : kernel(k), gamma(k == GS_KERNEL_LINEAR ? 0.0 : g), degree(k == GS_KERNEL_POLY ? deg : 0),
          coef0(k == GS_KERNEL_POLY || k == GS_KERNEL_SIGMOID ? c0 : 0.0) {}
    bool has_qd() const { return kernel == GS_KERNEL_POLY || kernel == GS_KERNEL_SIGMOID; }   // a diagonal of its own
    bool operator<(const KernelSpec &o) const
    {
        if (kernel != o.kernel) return kernel < o.kernel;
        if (gamma != o.gamma) return gamma < o.gamma;
        if (degree != o.degree) return degree < o.degree;
        return coef0 < o.coef0;
    }
};
// The SMO problems of one batch on the host, in column order
struct SmoBatch {
    std::vector<SmoProblem> probs;
    std::vector<double> cost;                      // predicted solve cost of each problem: the costliest are launched first
    std::vector<SvrData> svr;                      // one per problem for SVR, else empty
    std::vector<NuData> nu;                        // one per problem for the nu models, else empty
};
// What one kernel-SVM model gives the batch loop.  Task t is candidate t / n_splits on split t % n_splits.
struct SvmModel {
    const char *who;                               // the C function, for error messages
    bool refit;
    int n_splits, kind;                            // kind: the scorer
    double tol;
    int max_iter;
    uint32_t flags;
    std::vector<int> rows;                         // the dataset rows of every problem
    int lmax;                                      // the most positions of a problem
    std::vector<char> skip;                        // per task, or empty: a task not solved scores NaN with n_iter -1
    // Appends task t's problems to b, made from base (its model-independent fields set, rows at the device copy of rows),
    // with their cost and, for SVR and nu, their SvrData / NuData.  ks: the task's kernel matrix.
    std::function<void(int t, const KernelSpec &ks, const SmoProblem &base, SmoBatch &b)> add_task;
};
struct SvmSearch {                                 // the state of one kernel-SVM search or refit
    gs_handle *h;
    cudaStream_t st;
    int n;
    int64_t ldk;                                   // row stride of the float32 kernel matrices in h->dK
    EvTimer tm;
    float acc[5] = {0, 0, 0, 0, 0};                // event time by phase: 0 gram, 1 kernel matrix, 2 solve, 3 score, 4 other
    cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
    std::vector<KernelSpec> groups;                // kernel and parameters of each kernel matrix, in order of first use
    std::vector<int> task_group;                   // task c * n_splits + k -> its group
    std::vector<std::vector<int>> group_tasks;     // group -> its tasks, ascending
    int per_batch = 0;                             // kernel matrices per batch
    double *d_qd = nullptr;                        // per_batch float64 diagonals [n] behind them in h->dK (poly / sigmoid)
    bool fast = false;                             // this batch enqueues the branch-free SMO instance before the general one,
    const int *d_guard = nullptr;                  // with this SmoProblem::guard
    double *d_rho = nullptr;                       // outputs of the batch's problems (h->dWork[5]): rho [np], info [np][4],
    int *d_info = nullptr;                         // ns [np][12], and their host copies; coef [np][n] only when asked for
    unsigned long long *d_ns = nullptr;
    std::vector<int> info;
    std::vector<unsigned long long> ns;
    std::vector<double> rho, coef;
    std::vector<unsigned long long> auc_pairs;     // host copies of the batch's ROC-AUC pair counts / class counts
    std::vector<int> class_counts;
    SvmSearch(gs_handle *h_, cudaStream_t st_) : h(h_), st(st_), n((int)h_->n), ldk(((int64_t)h_->n + 31) & ~31LL), tm(st_, h_->evp) {}
    // resets h->prof but gs_set_data's ms_h2d / h2d_bytes, records the begin event and enqueues the Gram
    int start(uint32_t flags);
    // groups the tasks by kernel matrix; rejects an rbf gamma that is not finite and > 0, a poly / sigmoid gamma that is not
    // finite and >= 0, with who in the message.  degree / coef0: per candidate, or null for scikit-learn's 3 / 0.
    int group(const char *who, int n_cand, int n_splits, const int32_t *kernel, const double *gamma, const int32_t *degree,
              const double *coef0);
    // Solves, scores and finishes every task in batches of kernel matrices, and writes the outputs (any may be null but a
    // search's test_scores).  A search writes per task; a refit writes rho, n_iter and coef ([n] by original row) per problem.
    int run(const SvmModel &m, double *test_scores, double *train_scores, int32_t *n_iter, int32_t *n_sv, float *fit_ms,
            float *score_ms, double *coef, double *rho_out);
    // the steps of run
    int plan_batches();                            // per_batch; reserves h->dK (and room for the diagonals when a group has one)
    int kernel_matrices(int g0, int g1);           // group g at h->dK + (g - g0) n ldk, its diagonal, the guard flag, fast
    const double *qd(int g, int g0) const;         // SmoProblem::qd of group g in the batch from g0
    int workspaces(std::vector<SmoProblem> &probs);   // alpha / Gbar / scratch / coef / outputs of every problem
    // enqueues the SMO launches of a batch in launch order d_order (its problems by cost, descending) and counts them in
    // h->prof.launches: C-SVC on the cluster / exclusive-SM / shared-SM tiers, nu and SVR on one position-owned launch.
    // *n_cl / *n_ex: how many went on clusters / exclusive SMs.
    int solve(const SmoBatch &b, const std::vector<int> &order, const SmoProblem *d_probs, const SvrData *d_svr,
              const NuData *d_nu, const int *d_order, int lmax, int *n_cl, int *n_ex);
    int decisions(int g0, int g1, const std::vector<int> &group_first);   // group g: columns from group_first[g - g0]
    // enqueues what kind's score of every vote task is computed from, from the decision values: a classifier's vote counts
    // or a regressor's residual sums of squares into d_votes (16 bytes per task), or AUC pair / class counts copied to
    // auc_pairs / class_counts (read after the next sync)
    int score(int kind, const std::vector<VoteTask> &vtasks, const VoteTask *d_vt, void *d_votes);
    int results(int np, bool with_coef);           // downloads the batch's outputs, syncs, collects its phase times
    int finish(int64_t smo_iterations, double solve_bytes);   // end event, sync, the profile's times and totals
};

// ---- linsvc.cu: liblinear's TRON, one column per fit (LinearSVC, and LinearSVR's primal solver in linsvr.cu) ----
enum { M_FUN = 0, M_HV = 1, M_DONE = 2 };
constexpr int PW_BLOCKS = 64;          // row blocks of the element-wise pass: the loss partials of a column, summed in order
constexpr int NVEC = 5;                // per-column vectors: w, g, s, r, d
struct TrState {                       // per column
    int mode, iter, cg_iter, init, cur, fold, pos, n_iter;
    double Cp, Cn, eps, f, delta, gnorm1, rTr, cgtol;
};
// One TRON step of every open column from the gradient contraction Gp ([nchunk] split-K partials) and the loss partials
// fpart[col][PW_BLOCKS]; the next submission goes to V[col]; *n_open counts the columns still running.
cudaError_t launch_tron_advance(TrState *St, double *Vec, double *V, const double *Gp, int nchunk, int64_t gp_stride,
                                const double *fpart, int ncol, int nvp, int max_iter, int *n_open, cudaStream_t st);
// Xa = [X | bias | 0 ...] in float64 ([npad][nvp], rows >= n zero) and its transpose [nvp][npad]
cudaError_t launch_build_xa64(const float *X32, const double *X64, int n, int d, double bias, int nvp, int64_t npad, double *Xa,
                              double *Xat, cudaStream_t st);
// Per-class counts of the predictions of nfit fits from their KC decision rows Zt[(f KC + k) ldz + row] (KC == 1: z > 0 ->
// class 1; else the first arg-max) on split fold_of_fit[f]: counts[f][split (0 test, 1 train)][class][3 = support, tp,
// predicted], pre-zeroed
cudaError_t launch_linsvc_count(const double *Zt, int64_t ldz, int n, int K, int KC, const int *y, SplitMasks sm,
                                const int *fold_of_fit, int nfit, int *counts, cudaStream_t st);

// ---- linear_search.cu: the host steps the primal linear searches share (LinearSVC, LinearSVR, SGD, SAG; an int return is
// a GS_* status).  The fits' weight rows are [mpad][nvp], nvp = round_up(d + 1, 64), mpad = round_up(rows, 64), row
// f K + q for fit f = candidate x ns + split and decision row q; Xa = [X | bias] is [round_up(n, 64)][nvp] (launch_build_xa64). ----
// Every split's training rows in fit order, as internal rows: gs_set_train_order's lists, else ascending original index; the
// refit (ns = 1) trains on every row.  positive_only: only rows of positive sample weight (liblinear's remove_zero_weight).
// Split k's rows are order[sp_off[k] .. sp_off[k + 1]).  Returns the longest split's row count, 0 when a split has none.
int train_rows(const gs_handle *h, int ns, bool refit, bool positive_only, std::vector<int> &order, std::vector<int> &sp_off);
// Rejects class weights given per split for another number of splits than ns
int check_class_weight_sets(gs_handle *h, const char *who, int ns);
// liblinear's TRON (tron.cpp) on ncol columns, one round for all open columns at a time: Z = V Xa^T (every column's
// submission), the caller's element-wise pass (Z, St -> R, F and the spare active set), Gp = R Xat^T split-K over rows, then
// tron_advance_kernel.  reserve() takes h->dWork[2..6] and zeroes V, Vec, R and the masks; the caller uploads St.
struct TronRounds {
    static constexpr int KCH = 2048;           // split-K chunk of the gradient contraction
    int ncol = 0, nvp = 0, mpad = 0, nchunk = 0;
    int64_t npad = 0;
    TrState *St = nullptr;                     // [ncol]
    double *V = nullptr, *Vec = nullptr;       // submissions [mpad][nvp]; w, g, s, r, d of every column [ncol][NVEC][nvp]
    double *R = nullptr, *F = nullptr;         // element-wise pass: [mpad][npad] and the loss partials [ncol][PW_BLOCKS]
    double *Gp = nullptr;                      // gradient partials [nchunk][mpad][nvp]
    unsigned char *mask = nullptr;             // active sets [2][ncol][npad], current one TrState::cur
    int *open = nullptr;                       // columns still running after a round
    int rounds = 0;
    int reserve(gs_handle *h, int ncol);
    // rounds until every column is done (GS_ERR_NUMERIC after 10^6, with who in the message); launches += 4 per round
    int run(gs_handle *h, const char *who, const double *Xa, const double *Xat, double *Z, int max_iter,
            const std::function<cudaError_t()> &pointwise, int64_t &launches);
};
// Scores nfit fits of K decision rows from their weight rows V: Z = V Xa^T in one FP64 contraction (timed by h->tt), then the
// class counts (and ROC-AUC pair counts) or the residual sums of squares; records ev_end, synchronises and writes
// test_scores / train_scores (train may be null) with kind's formula.  Z: [mpad][npad].  launches += its launches.
int score_linear_fits(gs_handle *h, const double *V, const double *Xa, double *Z, int nfit, int K, int ns, int kind,
                      double *test_scores, double *train_scores, cudaEvent_t ev_end, int64_t &launches);
void gs_profile_reset(gs_profile &pf);   // clears pf but gs_set_data's ms_h2d / h2d_bytes
// The profile of a call timed by ev[0] (start), ev[1] (fits done), ev[2] (scores done): reset, then the phase times (also
// into *ms_solve / *ms_score), their total, the launches and the tensor-core time and flops
void linear_profile(gs_handle *h, const cudaEvent_t ev[3], int64_t launches, float *ms_solve, float *ms_score);
// fit_ms / score_ms (either may be null) of the nt tasks of a search call: its solve and score times spread evenly
void spread_call_ms(int nt, float solve_ms, float score_ms, float *fit_ms, float *score_ms_out);

// ---- gemm_tc.cu: wgmma + TMA contraction  C[M][N] = sum_k A[M][k] B[N][k]  (3xTF32 split, fp32 accumulate) ----
struct alignas(64) TcMap { unsigned char bytes[128]; };            // CUtensorMap
struct TcBatch {                                                    // one GEMM of a batched launch (blockIdx.z)
    int a_row0, b_row0;   // first row of the A / B operand inside their tensor maps
    int k0, k1;           // contraction range [k0, k1) in elements; must be a multiple of 32 long (zero padded)
    float *c;             // output, row-major
    int64_t ldc;
};
cudaError_t tc_make_map(TcMap *out, const float *base, int64_t rows, int64_t cols, int64_t ld);
cudaError_t launch_split_tf32(const float *x, float *hi, float *lo, size_t n, cudaStream_t st);
constexpr int TC_KCHUNK = 512;   // longest accumulation chain kept inside the (not round-to-nearest) tensor-core accumulator
cudaError_t launch_sum_partials(const float *partial, int n_chunks, int64_t per, float *out, cudaStream_t st);
// symmetric: the A and B operands are the same matrix (M == N): tiles below the diagonal are not computed, their values are
// stored as transposes of the tiles above it (bitwise symmetric result)
cudaError_t launch_gemm_nt_tf32x3(const TcMap &a_hi, const TcMap &a_lo, const TcMap &b_hi, const TcMap &b_lo,
                                  const TcBatch *d_batches, int n_batches, int M, int N, cudaStream_t st, bool symmetric = false);

// ---- gemm_f64.cu: FP64 tensor-core (DMMA) contraction  C[M][N] = sum_k A[M][k] B[N][k], float64 throughout ----
// M, N multiples of 64; K and kchunk multiples of 16; every row read (A rows < M, B rows < N, k < K) must exist.
// Split-K: chunk z of [z*kchunk, min(K, (z+1)*kchunk)) writes C + z*c_chunk_stride.
cudaError_t launch_gemm_nt_f64(const double *A, int64_t lda, const double *B, int64_t ldb, double *C, int64_t ldc, int M, int N,
                               int K, int kchunk, int64_t c_chunk_stride, cudaStream_t st);
// out[i] = sum over q = 0, 1, ... of partial[q * per + i], in that order (out == partial is allowed)
cudaError_t launch_sum_partials_f64(const double *partial, int n_chunks, int64_t per, double *out, cudaStream_t st);
