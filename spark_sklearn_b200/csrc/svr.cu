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
    const int n = (int)h->n;
    const int n_splits = refit ? 1 : h->n_splits;
    SvmSearch search(h, h->stream);
    SvmModel m{who, refit, n_splits, kind, tol, max_iter, flags};

    // ---- training rows of every split, ascending ORIGINAL index (scikit-learn fits X[train]), validated before any launch ----
    std::vector<int> by_orig(n);
    for (int r = 0; r < n; r++) by_orig[h->perm[r]] = r;
    std::vector<int> &rows_all = m.rows;
    std::vector<int> sp_off(n_splits + 1, 0);
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
        m.lmax = std::max(m.lmax, 2 * l);
    }
    sp_off[n_splits] = (int)rows_all.size();
    if (const int rc = search.group(who, n_cand, n_splits, kernel, gamma, nullptr, nullptr)) return rc;   // groups by kernel matrix (kernel, gamma)
    if (const int rc = search.start(flags)) return rc;

    // ---- one problem per (candidate, split) ----
    m.add_task = [&](int t, const KernelSpec &, const SmoProblem &base, SmoBatch &batch) {
        const int c = t / n_splits, k = t % n_splits;
        SmoProblem P = base;
        P.rows += sp_off[k];
        P.l = sp_off[k + 1] - sp_off[k];
        P.n_pos = P.l / 2;                            // nseg == 0: bulk row copies take the whole row
        P.C = Cv[c]; P.Cn = Cv[c];
        if (nu) {                                     // svm.cpp:1809-1815: linear term -/+ z, sum of C x nu in row order, halved
            double sum = 0;
            for (int r = 0; r < P.l / 2; r++) sum += Cv[c] * epsv[c];
            sum /= 2;
            batch.nu.push_back(NuData{sum, sum});
            batch.svr.push_back(SvrData{h->dZ64.as<double>(), 0.0});
        } else batch.svr.push_back(SvrData{h->dZ64.as<double>(), epsv[c]});
        // There is no iteration model for SVR yet; C x l orders the problems (larger C and more rows mean more iterations
        // in the measured searches) until one is calibrated.
        batch.cost.push_back(Cv[c] * (double)P.l);
        batch.probs.push_back(P);
    };
    return search.run(m, test_scores, train_scores, n_iter, n_sv, fit_ms, score_ms, coef_out, rho_out);
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
