// linear_search.cu -- the host steps of a primal linear-model search that do not depend on the model (linsvc_run in
// linsvc.cu, linsvr_run in linsvr.cu, sgd_run in sgd.cu, sag_run in sag.cu): the training rows in fit order, the class
// weight check, TRON's round loop, the scoring of the final weights and the call's profile.  Host code only.
#include "common.cuh"
#include <algorithm>
#include <cstring>

int train_rows(const gs_handle *h, int ns, bool refit, bool positive_only, std::vector<int> &order, std::vector<int> &sp_off)
{
    const int n = (int)h->n;
    const bool drop = positive_only && !h->sample_w.empty();
    std::vector<int> by_orig(n);
    for (int r = 0; r < n; r++) by_orig[h->perm[r]] = r;
    order.clear();
    sp_off.assign(ns + 1, 0);
    int lmax = 0;
    for (int k = 0; k < ns; k++) {
        sp_off[k] = (int)order.size();
        auto take = [&](int o) {
            const int r = by_orig[o];
            if (!drop || h->sample_w64[r] > 0) order.push_back(r);
        };
        if (refit) for (int o = 0; o < n; o++) take(o);
        else if (!h->train_off.empty()) for (int64_t e = h->train_off[k]; e < h->train_off[k + 1]; e++) take(h->train_order[e]);
        else for (int o = 0; o < n; o++) if (h->is_train(by_orig[o], k)) take(o);
        const int l = (int)order.size() - sp_off[k];
        if (l == 0) return 0;
        lmax = std::max(lmax, l);
    }
    sp_off[ns] = (int)order.size();
    return lmax;
}

int check_class_weight_sets(gs_handle *h, const char *who, int ns)
{
    if (h->class_w_sets == 0 || h->class_w_sets == 1 || h->class_w_sets == ns) return GS_OK;
    gs_set_error(h, std::string(who) + ": gs_set_class_weight was given a weight set per split, but not for this number of splits");
    return GS_ERR_ARG;
}

int TronRounds::reserve(gs_handle *h, int ncol_)
{
    cudaStream_t st = h->stream;
    ncol = ncol_;
    nvp = (int)round_up(h->d + 1, 64);
    npad = round_up(h->n, 64);
    mpad = (int)round_up(ncol, 64);
    nchunk = (int)((npad + KCH - 1) / KCH);
    DevBuf &bR = h->dWork[2], &bG = h->dWork[3], &bV = h->dWork[4], &bS = h->dWork[5], &bM = h->dWork[6];
    const size_t v_elems = (size_t)mpad * nvp + (size_t)ncol * NVEC * nvp;
    GS_CUDA(bR.reserve((size_t)mpad * npad * 8));
    GS_CUDA(bG.reserve((size_t)nchunk * mpad * nvp * 8));
    GS_CUDA(bV.reserve(v_elems * 8));
    GS_CUDA(bS.reserve((size_t)ncol * sizeof(TrState) + (size_t)ncol * PW_BLOCKS * 8 + 64));
    GS_CUDA(bM.reserve((size_t)2 * ncol * npad));
    R = bR.as<double>(); Gp = bG.as<double>();
    V = bV.as<double>(); Vec = V + (size_t)mpad * nvp;
    St = bS.as<TrState>();
    F = reinterpret_cast<double *>(St + ncol);
    open = reinterpret_cast<int *>(F + (size_t)ncol * PW_BLOCKS);
    mask = bM.as<unsigned char>();
    GS_CUDA(cudaMemsetAsync(V, 0, v_elems * 8, st));                        // w0 = 0, the first trial point
    GS_CUDA(cudaMemsetAsync(mask, 0, (size_t)2 * ncol * npad, st));
    GS_CUDA(cudaMemsetAsync(R, 0, (size_t)mpad * npad * 8, st));            // rows >= ncol stay zero
    rounds = 0;
    return GS_OK;
}

int TronRounds::run(gs_handle *h, const char *who, const double *Xa, const double *Xat, double *Z, int max_iter,
                    const std::function<cudaError_t()> &pointwise, int64_t &launches)
{
    cudaStream_t st = h->stream;
    const double flops = 2.0 * mpad * (double)npad * nvp;
    int n_open = 1;
    while (n_open > 0) {
        if (++rounds > 1000000) { gs_set_error(h, std::string(who) + ": TRON did not terminate"); return GS_ERR_NUMERIC; }
        h->tt.begin(h->evp, st);
        GS_CUDA(launch_gemm_nt_f64(V, nvp, Xa, nvp, Z, npad, mpad, (int)npad, nvp, nvp, 0, st));
        h->tt.end(h->evp, st, flops);
        GS_CUDA(pointwise());
        h->tt.begin(h->evp, st);
        GS_CUDA(launch_gemm_nt_f64(R, npad, Xat, npad, Gp, nvp, mpad, nvp, (int)npad, KCH, (int64_t)mpad * nvp, st));
        h->tt.end(h->evp, st, flops);
        GS_CUDA(cudaMemsetAsync(open, 0, 4, st));
        GS_CUDA(launch_tron_advance(St, Vec, V, Gp, nchunk, (int64_t)mpad * nvp, F, ncol, nvp, max_iter, open, st));
        GS_CUDA(cudaMemcpyAsync(&n_open, open, 4, cudaMemcpyDeviceToHost, st));
        GS_CUDA(cudaStreamSynchronize(st));
        launches += 4;
    }
    return GS_OK;
}

int score_linear_fits(gs_handle *h, const double *V, const double *Xa, double *Z, int nfit, int K, int ns, int kind,
                      double *test_scores, double *train_scores, cudaEvent_t ev_end, int64_t &launches)
{
    cudaStream_t st = h->stream;
    const int n = (int)h->n, nc = h->n_classes, nvp = (int)round_up(h->d + 1, 64);
    const int64_t npad = round_up(n, 64);
    const int mpad = (int)round_up((int64_t)nfit * K, 64);
    const bool cls = h->classification;
    h->tt.begin(h->evp, st);
    GS_CUDA(launch_gemm_nt_f64(V, nvp, Xa, nvp, Z, npad, mpad, (int)npad, nvp, nvp, 0, st));
    h->tt.end(h->evp, st, 2.0 * mpad * (double)npad * nvp);
    launches++;

    const int per_fit = 6 * nc;
    std::vector<int> ccounts;
    std::vector<unsigned long long> araw;
    std::vector<double> rss;
    if (cls) {
        // h->dScore: AUC pair counts [nfit][4] | class counts [nfit][per_fit] | decision row, split of every fit [2][nfit]
        GS_CUDA(h->dScore.reserve((size_t)nfit * (32 + per_fit * 4 + 8)));
        unsigned long long *d_auc = h->dScore.as<unsigned long long>();
        int *d_cnt = reinterpret_cast<int *>(d_auc + (size_t)nfit * 4), *d_meta = d_cnt + (size_t)nfit * per_fit;
        std::vector<int> meta((size_t)nfit * 2);
        for (int f = 0; f < nfit; f++) { meta[f] = f; meta[nfit + f] = f % ns; }
        GS_CUDA(cudaMemcpyAsync(d_meta, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemsetAsync(d_auc, 0, (size_t)nfit * (32 + per_fit * 4), st));
        GS_CUDA(launch_linsvc_count(Z, npad, n, nc, K, h->dY.as<int>(), h->masks(), d_meta + nfit, nfit, d_cnt, st));
        ccounts.resize((size_t)nfit * per_fit);
        GS_CUDA(cudaMemcpyAsync(ccounts.data(), d_cnt, ccounts.size() * 4, cudaMemcpyDeviceToHost, st));
        launches++;
        if (kind == GS_SCORE_ROC_AUC) {
            GS_CUDA(launch_auc_pairs_f64(Z, npad, n, h->class_start[1], h->masks(), d_meta, d_meta + nfit, nfit, +1, d_auc, st));
            araw.resize((size_t)nfit * 4);
            GS_CUDA(cudaMemcpyAsync(araw.data(), d_auc, araw.size() * 8, cudaMemcpyDeviceToHost, st));
            launches++;
        }
    } else {
        // h->dScore: the decision rows at stride n (launch_rss reads rows of n) [nfit][n] | rss [nfit][2] | rho = 0 [nfit] | tasks
        GS_CUDA(h->dScore.reserve((size_t)nfit * ((size_t)n * 8 + 24 + sizeof(VoteTask))));
        double *d_zc = h->dScore.as<double>(), *d_rss = d_zc + (size_t)nfit * n, *d_rho = d_rss + (size_t)nfit * 2;
        VoteTask *d_vt = reinterpret_cast<VoteTask *>(d_rho + nfit);
        GS_CUDA(cudaMemcpy2DAsync(d_zc, (size_t)n * 8, Z, (size_t)npad * 8, (size_t)n * 8, nfit, cudaMemcpyDeviceToDevice, st));
        std::vector<VoteTask> vt(nfit);
        for (int f = 0; f < nfit; f++) vt[f] = VoteTask{f, f % ns};
        GS_CUDA(cudaMemcpyAsync(d_vt, vt.data(), (size_t)nfit * sizeof(VoteTask), cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemsetAsync(d_rho, 0, (size_t)nfit * 8, st));
        GS_CUDA(launch_rss(d_zc, d_rho, n, h->dZ64.as<double>(), h->masks(), d_vt, nfit, d_rss, st));
        rss.resize((size_t)nfit * 2);
        GS_CUDA(cudaMemcpyAsync(rss.data(), d_rss, rss.size() * 8, cudaMemcpyDeviceToHost, st));
        launches += 2;
    }
    cudaEventRecord(ev_end, st);
    GS_CUDA(cudaStreamSynchronize(st));

    const SplitScoreStats ss(h, ns, kind);
    for (int f = 0; f < nfit; f++) {
        const int k = f % ns;
        for (int sp = 0; sp < 2; sp++) {
            double *out = sp == 0 ? test_scores : train_scores;
            if (!out) continue;
            if (!cls) out[f] = ss.regression(k, sp, rss[(size_t)f * 2 + sp]);
            else if (kind == GS_SCORE_ROC_AUC) out[f] = ss.auc(k, sp, &araw[(size_t)f * 4 + sp * 2]);
            else out[f] = ss.counts(&ccounts[(size_t)f * per_fit + sp * 3 * nc]);
        }
    }
    return GS_OK;
}

void gs_profile_reset(gs_profile &pf)
{
    const float ms_h2d = pf.ms_h2d;
    const int64_t h2d_bytes = pf.h2d_bytes;
    memset(&pf, 0, sizeof pf);
    pf.ms_h2d = ms_h2d; pf.h2d_bytes = h2d_bytes;
}

void linear_profile(gs_handle *h, const cudaEvent_t ev[3], int64_t launches, float *ms_solve, float *ms_score)
{
    cudaEventElapsedTime(ms_solve, ev[0], ev[1]);
    cudaEventElapsedTime(ms_score, ev[1], ev[2]);
    gs_profile &pf = h->prof;
    gs_profile_reset(pf);
    pf.ms_total = *ms_solve + *ms_score; pf.ms_solve = *ms_solve; pf.ms_score = *ms_score;
    pf.launches = launches;
    pf.ms_tensor = h->tt.collect(); pf.tensor_flops = h->tt.flops;
}

void spread_call_ms(int nt, float solve_ms, float score_ms, float *fit_ms, float *score_ms_out)
{
    for (int i = 0; i < nt; i++) {
        if (fit_ms) fit_ms[i] = solve_ms / (float)nt;
        if (score_ms_out) score_ms_out[i] = score_ms / (float)nt;
    }
}

extern "C" {

int gs_set_train_order(gs_handle *h, const int32_t *rows, const int64_t *offsets, int32_t n_splits)
{
    if (!h) return GS_ERR_ARG;
    if (h->n == 0) { gs_set_error(h, "gs_set_train_order: no dataset (call gs_set_data first)"); return GS_ERR_NO_DATA; }
    if (!rows || !offsets) { h->train_order.clear(); h->train_off.clear(); return GS_OK; }
    if (n_splits != h->n_splits) { gs_set_error(h, "gs_set_train_order: n_splits differs from the dataset's splits"); return GS_ERR_ARG; }
    const int n = (int)h->n;
    std::vector<int> by_orig(n);
    for (int r = 0; r < n; r++) by_orig[h->perm[r]] = r;
    if (offsets[0] != 0) { gs_set_error(h, "gs_set_train_order: offsets[0] must be 0"); return GS_ERR_ARG; }
    std::vector<char> seen(n);
    for (int k = 0; k < n_splits; k++) {
        if (offsets[k + 1] < offsets[k]) { gs_set_error(h, "gs_set_train_order: offsets must not decrease"); return GS_ERR_ARG; }
        std::fill(seen.begin(), seen.end(), 0);
        int64_t want = 0;
        for (int r = 0; r < n; r++) want += h->is_train(r, k);
        if (offsets[k + 1] - offsets[k] != want) {
            gs_set_error(h, "gs_set_train_order: split " + std::to_string(k) + " lists a different number of rows than its training set");
            return GS_ERR_ARG;
        }
        for (int64_t e = offsets[k]; e < offsets[k + 1]; e++) {
            const int o = rows[e];
            if (o < 0 || o >= n || seen[o] || !h->is_train(by_orig[o], k)) {
                gs_set_error(h, "gs_set_train_order: split " + std::to_string(k) + " lists a row twice or a row outside its training set");
                return GS_ERR_ARG;
            }
            seen[o] = 1;
        }
    }
    h->train_order.assign(rows, rows + offsets[n_splits]);
    h->train_off.assign(offsets, offsets + n_splits + 1);
    return GS_OK;
}

}  // extern "C"
