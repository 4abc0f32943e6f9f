// svr.cu -- epsilon-SVR and nu-SVR searches and refits (gs_svr / gs_svr_refit, gs_nusvr / gs_nusvr_refit).
//
// An SVR fit on l training rows is libsvm's C-SVC Solver on 2l variables (svm.cpp solve_epsilon_svr): positions 0..l-1 are
// the rows with y = +1 and linear term eps - z, positions l..2l-1 the same rows with y = -1 and linear term eps + z.  The
// solve is the position-owned SMO kernel of smo.cu (its SVR instance), so the iterate sequence is libsvm's; everything
// around it -- float64 Gram, float32 kernel matrices per (kernel, gamma), float64 decision values -- is the host pipeline
// it shares with SVC (kernel_svm.cu).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>

// nu == false: epsilon-SVR, epsv[c] is epsilon.  nu == true: nu-SVR (svm.cpp solve_nu_svr on Solver_NU), epsv[c] is nu.
static int svr_run(gs_handle *h, int n_cand, const int32_t *kernel, const double *Cv, const double *epsv, const double *gamma,
                   double tol, int max_iter, uint32_t flags, bool refit, bool nu,
                   double *test_scores, double *train_scores, int32_t *n_iter, int32_t *n_sv, float *fit_ms, float *score_ms,
                   double *coef_out, double *rho_out)
{
    const char *who = nu ? "gs_nusvr" : "gs_svr";
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) { gs_set_error(h, std::string(who) + ": no dataset (call gs_set_data first)"); return GS_ERR_NO_DATA; }
    if (h->classification) { gs_set_error(h, std::string(who) + ": the dataset has class labels (SVR needs a regression gs_set_data)"); return GS_ERR_ARG; }
    if (h->z64.empty()) { gs_set_error(h, std::string(who) + ": no float64 targets (call gs_set_targets_f64 after gs_set_data)"); return GS_ERR_NO_DATA; }
    if (n_cand <= 0 || !kernel || !Cv || !epsv || !gamma) { gs_set_error(h, std::string(who) + ": bad arguments"); return GS_ERR_ARG; }
    if (!h->sample_w.empty()) { gs_set_error(h, std::string(who) + ": sample weights are not supported by the SVR kernels"); return GS_ERR_UNSUPPORTED; }
    if (h->class_w_sets > 0) { gs_set_error(h, std::string(who) + ": class weights do not apply to a regressor"); return GS_ERR_ARG; }
    const int kind = refit ? GS_SCORE_DEFAULT : h->score_kind;
    if (int e = check_scorer(h, who, kind)) return e;
    for (int c = 0; c < n_cand; c++) {
        if (kernel[c] != GS_KERNEL_LINEAR && kernel[c] != GS_KERNEL_RBF) { gs_set_error(h, std::string(who) + ": unsupported kernel id"); return GS_ERR_UNSUPPORTED; }
        if (!(Cv[c] > 0) || !std::isfinite(Cv[c])) { gs_set_error(h, std::string(who) + ": C must be > 0"); return GS_ERR_ARG; }
        if (nu && !(epsv[c] > 0 && epsv[c] <= 1)) { gs_set_error(h, "gs_nusvr: nu must be in (0, 1]"); return GS_ERR_ARG; }
        if (!(epsv[c] >= 0) || !std::isfinite(epsv[c])) { gs_set_error(h, std::string(who) + ": epsilon must be >= 0"); return GS_ERR_ARG; }
    }
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    const int n = (int)h->n;
    const int n_splits = refit ? 1 : h->n_splits;
    const int n_tasks = n_cand * n_splits;
    SvmSearch search(h, st);
    const int64_t ldk = search.ldk;

    // ---- training rows of every split, ascending ORIGINAL index (scikit-learn fits X[train]), validated before any launch ----
    std::vector<int> by_orig(n);
    for (int r = 0; r < n; r++) by_orig[h->perm[r]] = r;
    std::vector<int> rows_all;
    std::vector<int> sp_off(n_splits + 1, 0);
    int lmax = 0;
    for (int k = 0; k < n_splits; k++) {
        sp_off[k] = (int)rows_all.size();
        std::vector<int> rs;
        for (int o = 0; o < n; o++) {
            const int r = by_orig[o];
            if (refit || h->is_train(r, k)) rs.push_back(r);
        }
        const int l = (int)rs.size();
        if (l == 0) { gs_set_error(h, std::string(who) + ": a split has no training rows"); return GS_ERR_ARG; }
        if (2 * l > smo_max_rows()) {
            gs_set_error(h, std::string(who) + ": a fit on " + std::to_string(l) + " training rows exceeds the SVR kernel limit of " +
                                std::to_string(smo_max_rows() / 2));
            return GS_ERR_UNSUPPORTED;
        }
        rows_all.insert(rows_all.end(), rs.begin(), rs.end());                // +1 copies
        rows_all.insert(rows_all.end(), rs.begin(), rs.end());                // -1 copies
        lmax = std::max(lmax, 2 * l);
    }
    sp_off[n_splits] = (int)rows_all.size();
    if (const int rc = search.group(who, n_cand, n_splits, kernel, gamma, nullptr, nullptr)) return rc;   // groups by kernel matrix (kernel, gamma)

    gs_profile &pf = h->prof;
    search.begin();

    // ---- 1. Gram X X^T ----
    if (const int rc = build_gram(h, flags, st)) return rc;
    search.tm.mark(0);

    // ---- 2. kernel matrices in batches that fit in free HBM ----
    if (const int rc = search.plan_batches()) return rc;
    const int n_groups = (int)search.groups.size(), gpb = search.per_batch;
    GS_CUDA(h->dWork[0].reserve(rows_all.size() * 4));
    GS_CUDA(cudaMemcpyAsync(h->dWork[0].p, rows_all.data(), rows_all.size() * 4, cudaMemcpyHostToDevice, st));
    pf.h2d_bytes += rows_all.size() * 4;
    const int *d_rows = h->dWork[0].as<int>();

    std::vector<int> task_iter(n_tasks, 0), task_sv(n_tasks, 0);
    std::vector<double> task_fit_ms(n_tasks, 0.0), task_rss((size_t)n_tasks * 2, 0.0);
    std::vector<char> task_bad(n_tasks, 0);
    int64_t total_iter = 0;
    double solve_bytes = 0;

    for (int g0 = 0; g0 < n_groups; g0 += gpb) {
        const int g1 = std::min(n_groups, g0 + gpb);
        if (const int rc = search.kernel_matrices(g0, g1)) return rc;

        // ---- 3. one problem per (candidate, split), ordered by group: column index == problem index ----
        std::vector<SmoProblem> probs;
        std::vector<SvrData> svr;
        std::vector<NuData> nud;
        std::vector<int> prob_task, group_first(g1 - g0 + 1, 0);
        std::vector<VoteTask> vtasks;
        for (int g = g0; g < g1; g++) {
            group_first[g - g0] = (int)probs.size();
            for (int t : search.group_tasks[g]) {
                const int c = t / n_splits, k = t % n_splits;
                vtasks.push_back(VoteTask{(int)probs.size(), refit ? -100 : k});
                SmoProblem P;
                memset(&P, 0, sizeof P);
                P.K = h->dK.as<float>() + (size_t)(g - g0) * n * ldk;
                P.qd = search.qd(g, g0);
                P.rows = d_rows + sp_off[k];
                P.l = sp_off[k + 1] - sp_off[k];
                P.n_pos = P.l / 2;
                P.nseg = 0;                                   // bulk row copies take the whole row
                P.ldk = ldk; P.C = Cv[c]; P.Cn = Cv[c]; P.eps = tol; P.max_iter = max_iter;
                P.shrinking = (flags & GS_NO_SHRINKING) ? 0 : 1;
                P.guard = search.d_guard;
                probs.push_back(P);
                if (nu) {                                     // svm.cpp:1809-1815: linear term -/+ z, sum of C x nu in row order, halved
                    double sum = 0;
                    for (int r = 0; r < P.l / 2; r++) sum += Cv[c] * epsv[c];
                    sum /= 2;
                    nud.push_back(NuData{sum, sum});
                    svr.push_back(SvrData{h->dZ64.as<double>(), 0.0});
                } else svr.push_back(SvrData{h->dZ64.as<double>(), epsv[c]});
                prob_task.push_back(t);
            }
        }
        group_first[g1 - g0] = (int)probs.size();
        const int np = (int)probs.size();
        if (const int rc = search.workspaces(probs)) return rc;
        const size_t meta_bytes = (size_t)np * (sizeof(SmoProblem) + sizeof(SvrData) + sizeof(NuData) + 4) + vtasks.size() * sizeof(VoteTask) + 256;
        GS_CUDA(h->dWork[6].reserve(meta_bytes));
        GS_CUDA(h->dScore.reserve((size_t)np * 2 * 8));                   // rss[np][2]
        // ---- 4. launch order: longest predicted first.  There is no iteration model for SVR yet; C x l orders the
        // problems (larger C and more rows mean more iterations in the measured searches) until one is calibrated.
        std::vector<double> cost(np);
        for (int q = 0; q < np; q++) cost[q] = Cv[prob_task[q] / n_splits] * (double)probs[q].l;
        std::vector<int> order(np);
        std::iota(order.begin(), order.end(), 0);
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cost[a] > cost[b]; });
        unsigned char *dmeta = h->dWork[6].as<unsigned char>();
        SmoProblem *d_probs = (SmoProblem *)dmeta;
        size_t off = (size_t)np * sizeof(SmoProblem);
        SvrData *d_svr = (SvrData *)(dmeta + off);
        off += (size_t)np * sizeof(SvrData);
        int *d_order = (int *)(dmeta + off);
        off = (off + (size_t)np * 4 + 15) & ~(size_t)15;
        VoteTask *d_vt = (VoteTask *)(dmeta + off);
        off = (off + vtasks.size() * sizeof(VoteTask) + 15) & ~(size_t)15;
        NuData *d_nu = (NuData *)(dmeta + off);
        if (nu) {
            GS_CUDA(cudaMemcpyAsync(d_nu, nud.data(), nud.size() * sizeof(NuData), cudaMemcpyHostToDevice, st));
            pf.h2d_bytes += nud.size() * sizeof(NuData);
        }
        GS_CUDA(cudaMemcpyAsync(d_probs, probs.data(), (size_t)np * sizeof(SmoProblem), cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(d_svr, svr.data(), (size_t)np * sizeof(SvrData), cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(d_order, order.data(), (size_t)np * 4, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(d_vt, vtasks.data(), vtasks.size() * sizeof(VoteTask), cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemsetAsync(h->dWork[3].p, 0, (size_t)np * n * 8, st));
        pf.h2d_bytes += (size_t)np * (sizeof(SmoProblem) + sizeof(SvrData) + 4) + vtasks.size() * sizeof(VoteTask);
        search.tm.mark(4);
        // ---- 5. solve: one launch per instance (branch-free first, then the guarded general one) ----
        for (int inst = search.fast ? 1 : 0; inst >= 0; inst--) {
            std::string why;
            const cudaError_t ce = nu ? launch_smo_nu(d_probs, d_svr, d_nu, d_order, np, lmax, inst == 1, st, &why)
                                      : launch_smo_svr(d_probs, d_svr, d_order, np, lmax, inst == 1, (int)ldk, st, &why);
            if (ce != cudaSuccess) {
                gs_set_error(h, why.empty() ? std::string(nu ? "launch_smo_nu: " : "launch_smo_svr: ") + cudaGetErrorString(ce) : why);
                return why.empty() ? GS_ERR_CUDA : GS_ERR_UNSUPPORTED;
            }
            pf.launches++;
        }
        search.tm.mark(2);
        // ---- 6. decision values (float64 kernel, every row) and residual sums of squares ----
        if (!refit) {
            if (const int rc = search.decisions(g0, g1, group_first)) return rc;
            GS_CUDA(launch_rss(h->dWork[4].as<double>(), search.d_rho, n, h->dZ64.as<double>(), h->masks(), d_vt, (int)vtasks.size(),
                               h->dScore.as<double>(), st));
            pf.launches++;
        }
        search.tm.mark(3);
        // ---- results of this batch ----
        std::vector<double> rss((size_t)np * 2, 0.0);
        if (!refit) {
            GS_CUDA(cudaMemcpyAsync(rss.data(), h->dScore.p, rss.size() * 8, cudaMemcpyDeviceToHost, st));
            pf.d2h_bytes += rss.size() * 8;
        }
        if (const int rc = search.results(np, refit && coef_out)) return rc;
        const auto &info = search.info; const auto &ns = search.ns; const auto &rho = search.rho;
        for (int q = 0; q < np; q++) {
            const int t = prob_task[q];
            task_iter[t] = info[(size_t)q * 4]; task_sv[t] = info[(size_t)q * 4 + 2];
            task_fit_ms[t] = (double)(ns[(size_t)q * 12 + 1] - ns[(size_t)q * 12]) * 1e-6;
            task_rss[(size_t)t * 2] = rss[(size_t)q * 2]; task_rss[(size_t)t * 2 + 1] = rss[(size_t)q * 2 + 1];
            total_iter += info[(size_t)q * 4];
            // two gathered K rows per iteration, over the problem's l / 2 distinct columns
            solve_bytes += (double)info[(size_t)q * 4] * 2.0 * (probs[q].l / 2) * 4.0;
            if (!std::isfinite(rho[q])) { if (refit) { gs_set_error(h, std::string(who) + "_refit: non-finite intercept"); return GS_ERR_NUMERIC; } task_bad[t] = 1; }
        }
        if (refit) {
            if (rho_out) *rho_out = rho[0];
            if (n_iter) *n_iter = info[0];
            if (coef_out)
                for (int r = 0; r < n; r++) coef_out[h->perm[r]] = search.coef[r];
        }
    }
    if (const int rc = search.finish(total_iter, solve_bytes)) return rc;

    if (!refit) {
        const SplitScoreStats ss(h, n_splits, kind);
        for (int t = 0; t < n_tasks; t++) {
            const int k = t % n_splits;
            test_scores[t] = task_bad[t] ? NAN : ss.regression(k, 0, task_rss[(size_t)t * 2]);
            if (train_scores) train_scores[t] = task_bad[t] ? NAN : ss.regression(k, 1, task_rss[(size_t)t * 2 + 1]);
            if (n_iter) n_iter[t] = task_iter[t];
            if (n_sv) n_sv[t] = task_sv[t];
            if (fit_ms) fit_ms[t] = (float)task_fit_ms[t];
            if (score_ms) score_ms[t] = pf.ms_score / (float)n_tasks;
        }
    }
    return GS_OK;
}

extern "C" {

int gs_set_targets_f64(gs_handle *h, const double *y)
{
    if (!h) return GS_ERR_ARG;
    if (h->n == 0 || h->classification) { gs_set_error(h, "gs_set_targets_f64: no regression dataset (call gs_set_data first)"); return GS_ERR_NO_DATA; }
    if (!y) { gs_set_error(h, "gs_set_targets_f64: y is NULL"); return GS_ERR_ARG; }
    const int64_t n = h->n;
    std::vector<double> z((size_t)n);
    for (int64_t i = 0; i < n; i++) {
        z[i] = y[h->perm[i]];
        if (!std::isfinite(z[i])) { gs_set_error(h, "gs_set_targets_f64: targets must be finite"); return GS_ERR_ARG; }
    }
    GS_CUDA(cudaSetDevice(h->device));
    GS_CUDA(h->dZ64.reserve((size_t)n * 8));
    GS_CUDA(cudaMemcpyAsync(h->dZ64.p, z.data(), (size_t)n * 8, cudaMemcpyHostToDevice, h->stream));
    GS_CUDA(cudaStreamSynchronize(h->stream));
    h->z64.swap(z);
    h->prof.h2d_bytes += n * 8;
    return GS_OK;
}

int gs_svr(gs_handle *h, int32_t n_cand, const int32_t *kernel, const double *C, const double *epsilon, const double *gamma,
           double tol, int32_t max_iter, uint32_t flags, double *test_scores, double *train_scores, int32_t *n_iter,
           int32_t *n_sv, float *fit_ms, float *score_ms)
{
    if (h && !test_scores) { gs_set_error(h, "gs_svr: test_scores is NULL"); return GS_ERR_ARG; }
    return svr_run(h, n_cand, kernel, C, epsilon, gamma, tol, max_iter, flags, false, false, test_scores,
                   (flags & GS_RETURN_TRAIN) ? train_scores : nullptr, n_iter, n_sv, fit_ms, score_ms, nullptr, nullptr);
}

int gs_svr_refit(gs_handle *h, int32_t kernel, double C, double epsilon, double gamma, double tol, int32_t max_iter,
                 uint32_t flags, double *coef, double *rho, int32_t *n_iter)
{
    const int32_t k = kernel;
    return svr_run(h, 1, &k, &C, &epsilon, &gamma, tol, max_iter, flags, true, false, nullptr, nullptr, n_iter, nullptr, nullptr,
                   nullptr, coef, rho);
}

int gs_nusvr(gs_handle *h, int32_t n_cand, const int32_t *kernel, const double *C, const double *nu, const double *gamma,
             double tol, int32_t max_iter, uint32_t flags, double *test_scores, double *train_scores, int32_t *n_iter,
             int32_t *n_sv, float *fit_ms, float *score_ms)
{
    if (h && !test_scores) { gs_set_error(h, "gs_nusvr: test_scores is NULL"); return GS_ERR_ARG; }
    return svr_run(h, n_cand, kernel, C, nu, gamma, tol, max_iter, flags, false, true, test_scores,
                   (flags & GS_RETURN_TRAIN) ? train_scores : nullptr, n_iter, n_sv, fit_ms, score_ms, nullptr, nullptr);
}

int gs_nusvr_refit(gs_handle *h, int32_t kernel, double C, double nu, double gamma, double tol, int32_t max_iter,
                   uint32_t flags, double *coef, double *rho, int32_t *n_iter)
{
    const int32_t k = kernel;
    return svr_run(h, 1, &k, &C, &nu, &gamma, tol, max_iter, flags, true, true, nullptr, nullptr, n_iter, nullptr, nullptr,
                   nullptr, coef, rho);
}

}  // extern "C"
