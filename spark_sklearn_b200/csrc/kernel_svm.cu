// kernel_svm.cu -- the batch loop of the kernel-SVM searches and refits (SVC and NuSVC: api.cu, SVR and NuSVR: svr.cu) and
// the host steps it is made of; each model adds only its checks, its training rows and how a task becomes problems
// (SvmModel).  Host code only.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <numeric>

// Default: float64 on the FP64 pipe (libsvm-faithful, gram.cu).  GS_GRAM_TENSOR: wgmma tensor cores, 3xTF32 split,
// TMA-fed (gemm_tc.cu) -- fp32-faithful, so scores agree with scikit-learn to solver tolerance, not bit for bit.
int build_gram(gs_handle *h, uint32_t flags, cudaStream_t st)
{
    gs_profile &pf = h->prof;
    const int n = (int)h->n, d = (int)h->d;
    GS_CUDA(h->dS.reserve((size_t)n * n * 8));
    GS_CUDA(h->dXsq.reserve((size_t)n * 8));
    if (flags & GS_GRAM_TENSOR) {
        const int dpad = (d + 31) & ~31;
        const int64_t ld32 = ((int64_t)n + 3) & ~3LL;
        DevBuf &bx = h->dWork[1], &bs = h->dWork[2], &bb = h->dWork[6];
        GS_CUDA(bx.reserve((size_t)n * dpad * 4 * 3));
        GS_CUDA(bs.reserve((size_t)n * ld32 * 4));
        GS_CUDA(bb.reserve(sizeof(TcBatch) + 64));
        float *xp = bx.as<float>(), *xh = xp + (size_t)n * dpad, *xl = xh + (size_t)n * dpad;
        GS_CUDA(cudaMemsetAsync(xp, 0, (size_t)n * dpad * 4, st));
        GS_CUDA(cudaMemcpy2DAsync(xp, (size_t)dpad * 4, h->dX.p, (size_t)d * 4, (size_t)d * 4, n, cudaMemcpyDeviceToDevice, st));
        GS_CUDA(launch_split_tf32(xp, xh, xl, (size_t)n * dpad, st));
        TcMap mh, ml;
        GS_CUDA(tc_make_map(&mh, xh, n, dpad, dpad));
        GS_CUDA(tc_make_map(&ml, xl, n, dpad, dpad));
        TcBatch hb{0, 0, 0, dpad, bs.as<float>(), ld32};
        GS_CUDA(cudaMemcpyAsync(bb.p, &hb, sizeof hb, cudaMemcpyHostToDevice, st));
        h->tt.begin(h->evp, st);
        GS_CUDA(launch_gemm_nt_tf32x3(mh, ml, mh, ml, bb.as<TcBatch>(), 1, n, n, st, true));
        h->tt.end(h->evp, st, 3.0 * 2.0 * n * (double)n * dpad);
        GS_CUDA(launch_widen_gram(bs.as<float>(), n, ld32, h->dS.as<double>(), h->dXsq.as<double>(), st));
        pf.launches += 3;
    } else {
        GS_CUDA(launch_gram_f64(h->x_dtype == GS_F64 ? h->dX64.p : h->dX.p, h->x_dtype, n, d, h->dS.as<double>(), h->dXsq.as<double>(), st));
        pf.launches++;
    }
    pf.gram_flops = 2.0 * n * (double)n * d;
    pf.gram_bytes = (double)n * d * 4 + (double)n * n * ((flags & GS_GRAM_TENSOR) ? 4 : 8);
    return GS_OK;
}

int SvmSearch::start(uint32_t flags)
{
    gs_profile_reset(h->prof);
    h->evp.reset(); h->tt.reset();
    ev_begin = h->evp.get(); ev_end = h->evp.get();
    cudaEventRecord(ev_begin, st);
    tm.mark(-1);
    if (const int rc = build_gram(h, flags, st)) return rc;
    tm.mark(0);
    return GS_OK;
}

int SvmSearch::group(const char *who, int n_cand, int n_splits, const int32_t *kernel, const double *gamma,
                     const int32_t *degree, const double *coef0)
{
    std::map<KernelSpec, int> gmap;                                  // gamma: finite, > 0 for rbf, >= 0 for poly / sigmoid
    task_group.resize((size_t)n_cand * n_splits);
    for (int c = 0; c < n_cand; c++)
        for (int k = 0; k < n_splits; k++) {
            const KernelSpec key(kernel[c], gamma[(size_t)c * n_splits + k], degree ? degree[c] : 3, coef0 ? coef0[c] : 0.0);
            if (key.kernel == GS_KERNEL_RBF && !(key.gamma > 0 && std::isfinite(key.gamma))) {
                gs_set_error(h, std::string(who) + ": gamma must be finite and > 0"); return GS_ERR_ARG;
            }
            if (key.has_qd() && !(key.gamma >= 0 && std::isfinite(key.gamma))) {
                gs_set_error(h, std::string(who) + ": gamma must be finite and >= 0"); return GS_ERR_ARG;
            }
            auto it = gmap.find(key);
            if (it == gmap.end()) { it = gmap.emplace(key, (int)groups.size()).first; groups.push_back(key); }
            task_group[(size_t)c * n_splits + k] = it->second;
        }
    group_tasks.resize(groups.size());
    for (size_t t = 0; t < task_group.size(); t++) group_tasks[task_group[t]].push_back((int)t);
    return GS_OK;
}

int SvmSearch::plan_batches()
{
    // a poly / sigmoid group also needs its float64 diagonal: per_batch of them follow the kernel matrices in h->dK
    bool any_qd = false;
    for (const KernelSpec &g : groups) any_qd = any_qd || g.has_qd();
    const size_t kbytes = (size_t)n * ldk * 4, dbytes = any_qd ? (size_t)n * 8 : 0;
    per_batch = (int)groups.size();
    if (h->dK.cap < (kbytes + dbytes) * groups.size()) {
        // Ask the driver only when the buffer has to grow: cudaMemGetInfo takes anything from 0.1 to 100+ ms on a busy box
        // (it showed as outliers of this phase with the Gram already in flight), and a repeated search of the same
        // shape needs no new plan.
        size_t free_b = 0, total_b = 0;
        GS_CUDA(cudaMemGetInfo(&free_b, &total_b));
        free_b += h->dK.cap;
        const size_t budget = (size_t)(free_b * 0.6);
        per_batch = (int)std::max<size_t>(1, std::min<size_t>(groups.size(), budget / std::max<size_t>(kbytes + dbytes, 1)));
        GS_CUDA(h->dK.reserve((kbytes + dbytes) * per_batch));
    }
    d_qd = any_qd ? (double *)(h->dK.as<char>() + kbytes * per_batch) : nullptr;
    return GS_OK;
}

int SvmSearch::kernel_matrices(int g0, int g1)
{
    GS_CUDA(h->dWork[7].reserve(64));
    GS_CUDA(cudaMemsetAsync(h->dWork[7].p, 0, 4, st));
    fast = true;
    for (int g = g0; g < g1; g++) {
        const KernelSpec &ks = groups[g];
        GS_CUDA(launch_kernel_matrix(h->dS.as<double>(), h->dXsq.as<double>(), n, ks.kernel, ks.gamma, ks.degree, ks.coef0,
                                     h->dK.as<float>() + (size_t)(g - g0) * n * ldk, ldk,
                                     ks.has_qd() ? d_qd + (size_t)(g - g0) * n : nullptr, h->dWork[7].as<int>(), st));
        h->prof.launches++;
        fast = fast && ks.kernel == GS_KERNEL_RBF;
    }
    // The branch-free SMO instance needs rbf (QD == 1) and only positive normal floats in K.  The second condition is a
    // device flag the kernel-matrix kernels raise: both instances are enqueued and the wrong one returns at once
    // (SmoProblem::guard), so the host never waits in the middle of a search and everything it prepares next overlaps
    // the Gram and kernel-matrix kernels already in flight.
    d_guard = fast ? h->dWork[7].as<int>() : nullptr;
    tm.mark(1);
    return GS_OK;
}

const double *SvmSearch::qd(int g, int g0) const
{
    if (groups[g].kernel == GS_KERNEL_LINEAR) return h->dXsq.as<double>();   // k(x, x) = x.x
    if (groups[g].has_qd()) return d_qd + (size_t)(g - g0) * n;
    return nullptr;                                                           // rbf: QD == 1
}

int SvmSearch::workspaces(std::vector<SmoProblem> &probs)
{
    const int np = (int)probs.size();
    auto wlen = [](const SmoProblem &P) { return ((size_t)std::max(P.l, P.nslots) + 3) & ~(size_t)3; };   // 32-byte multiples
    size_t wl = 0, ws = 0;                                            // workspace doubles / ints
    for (const SmoProblem &P : probs) { wl += 2 * wlen(P); ws += 2 * (size_t)P.l + 64; }
    GS_CUDA(h->dWork[1].reserve(wl * 8));
    GS_CUDA(h->dWork[2].reserve(ws * 4));
    GS_CUDA(h->dWork[3].reserve((size_t)np * n * 8));                 // coef columns
    GS_CUDA(h->dWork[4].reserve((size_t)np * n * 8));                 // decision columns
    GS_CUDA(h->dWork[5].reserve((size_t)np * (8 + 16 + 96) + 64));    // rho, info[4], ns[12]
    d_rho = h->dWork[5].as<double>();
    d_info = (int *)(d_rho + np);
    d_ns = (unsigned long long *)(d_info + 4 * (size_t)np);
    GS_CUDA(cudaMemsetAsync(d_ns, 0, (size_t)np * 12 * 8, st));
    double *w = h->dWork[1].as<double>();
    int *s = h->dWork[2].as<int>();
    for (int q = 0; q < np; q++) {
        SmoProblem &P = probs[q];
        P.alpha = w; w += wlen(P);
        P.Gbar = w; w += wlen(P);
        P.scratch = s; s += 2 * (size_t)P.l + 64;
        P.coef = h->dWork[3].as<double>() + (size_t)q * n;
        P.out_rho = d_rho + q; P.out_info = d_info + 4 * (size_t)q; P.out_ns = d_ns + 12 * (size_t)q;
    }
    return GS_OK;
}

int SvmSearch::decisions(int g0, int g1, const std::vector<int> &group_first)
{
    size_t part_doubles = 0;                                          // partial sums of the j-slabs
    std::vector<int> jch(g1 - g0, 1);
    for (int g = g0; g < g1; g++) {
        const int cols = group_first[g - g0 + 1] - group_first[g - g0];
        jch[g - g0] = decision_chunks(n, cols, h->sm_count);
        if (jch[g - g0] > 1) part_doubles = std::max(part_doubles, (size_t)jch[g - g0] * cols * n);
    }
    if (part_doubles) GS_CUDA(h->dWork[8].reserve(part_doubles * 8));
    for (int g = g0; g < g1; g++) {
        const int c0 = group_first[g - g0], c1 = group_first[g - g0 + 1], jc = jch[g - g0];
        const KernelSpec &ks = groups[g];
        GS_CUDA(launch_decision(h->dS.as<double>(), h->dXsq.as<double>(), n, ks.kernel, ks.gamma, ks.degree, ks.coef0,
                                h->dWork[3].as<double>() + (size_t)c0 * n, c1 - c0,
                                h->dWork[4].as<double>() + (size_t)c0 * n, jc > 1 ? h->dWork[8].as<double>() : nullptr, jc, st));
        h->prof.launches += jc > 1 ? 2 : 1;
    }
    return GS_OK;
}

int SvmSearch::results(int np, bool with_coef)
{
    info.resize((size_t)np * 4); ns.resize((size_t)np * 12); rho.resize(np); coef.resize(with_coef ? (size_t)np * n : 0);
    GS_CUDA(cudaMemcpyAsync(info.data(), d_info, info.size() * 4, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaMemcpyAsync(ns.data(), d_ns, ns.size() * 8, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaMemcpyAsync(rho.data(), d_rho, rho.size() * 8, cudaMemcpyDeviceToHost, st));
    if (with_coef) GS_CUDA(cudaMemcpyAsync(coef.data(), h->dWork[3].p, coef.size() * 8, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaStreamSynchronize(st));
    h->prof.d2h_bytes += info.size() * 4 + ns.size() * 8 + rho.size() * 8 + coef.size() * 8;
    tm.collect(acc, 5);
    tm.mark(-1);
    return GS_OK;
}

int SvmSearch::finish(int64_t smo_iterations, double solve_bytes)
{
    gs_profile &pf = h->prof;
    cudaEventRecord(ev_end, st);
    GS_CUDA(cudaStreamSynchronize(st));
    tm.collect(acc, 5);
    cudaEventElapsedTime(&pf.ms_total, ev_begin, ev_end);
    pf.ms_tensor = h->tt.collect(); pf.tensor_flops = h->tt.flops;
    pf.ms_gram = acc[0]; pf.ms_kernel_matrix = acc[1]; pf.ms_solve = acc[2]; pf.ms_score = acc[3];
    pf.smo_iterations = smo_iterations;
    pf.solve_bytes = solve_bytes;
    return GS_OK;
}

// Development aids that leave results unchanged: B200GS_SMO_TIMELINE=1 prints when each solver tier of a batch starts and
// ends (globaltimer of the problems, ms after the first start), B200GS_SMO_PROF=1 the per-phase cycle counters of its
// longest problem (written by the PROF instances the same switch launches).
static void smo_diagnostics(const std::vector<int> &order, int n_cl, int n_ex, const std::vector<int> &info,
                            const std::vector<unsigned long long> &ns)
{
    const int np = (int)order.size();
    if (getenv("B200GS_SMO_TIMELINE") && atoi(getenv("B200GS_SMO_TIMELINE"))) {
        unsigned long long t0 = ~0ull;
        for (int q = 0; q < np; q++) if (ns[(size_t)q * 12]) t0 = std::min(t0, ns[(size_t)q * 12]);
        auto span = [&](int a, int b, const char *name) {
            if (b <= a) return;
            double s0 = 1e30, s1 = 0, e0 = 1e30, e1 = 0; long long it_max = 0;
            for (int i = a; i < b; i++) {
                const int q = order[i];
                const double st_ = (double)(ns[(size_t)q * 12] - t0) * 1e-6, en = (double)(ns[(size_t)q * 12 + 1] - t0) * 1e-6;
                s0 = std::min(s0, st_); s1 = std::max(s1, st_); e0 = std::min(e0, en); e1 = std::max(e1, en);
                it_max = std::max<long long>(it_max, info[(size_t)q * 4]);
            }
            fprintf(stderr, "[timeline] %-9s %4d problems: starts %.2f..%.2f ms, ends %.2f..%.2f ms, longest %lld iterations\n",
                    name, b - a, s0, s1, e0, e1, it_max);
        };
        span(0, n_cl, "cluster"); span(n_cl, n_cl + n_ex, "exclusive"); span(n_cl + n_ex, np, "shared");
        for (int i = 0; i < std::min(np, 16); i++) {
            const int q = order[i];
            fprintf(stderr, "[timeline]   #%d: %d iterations, %.2f -> %.2f ms (%.3f us/iteration)\n", i, info[(size_t)q * 4],
                    (double)(ns[(size_t)q * 12] - t0) * 1e-6, (double)(ns[(size_t)q * 12 + 1] - t0) * 1e-6,
                    (double)(ns[(size_t)q * 12 + 1] - ns[(size_t)q * 12]) * 1e-3 / std::max(1, info[(size_t)q * 4]));
        }
    }
    if (getenv("B200GS_SMO_PROF") && atoi(getenv("B200GS_SMO_PROF"))) {
        int qmax = 0;
        for (int q = 1; q < np; q++) if (info[(size_t)q * 4] > info[(size_t)qmax * 4]) qmax = q;
        const unsigned long long *pn = &ns[(size_t)qmax * 12];
        const double it = (double)info[(size_t)qmax * 4];
        // single-CTA kernel slots: scanA | bar1+redA | rowI+phaseB | bar2 | fetchJ+scalar | update
        // cluster kernel slots:    redA | xchg1 | rowI | phaseB | xchg2 | scalar | bar3 | rowJ | update
        fprintf(stderr, "[smo prof] longest problem: %d iters, %.1f ms (%.2f us/iter); cycles/iter by slot:", info[(size_t)qmax * 4],
                (double)(pn[1] - pn[0]) * 1e-6, (double)(pn[1] - pn[0]) * 1e-3 / it);
        for (int e = 0; e < 10; e++) fprintf(stderr, " %.0f", pn[2 + e] / it);
        fprintf(stderr, "\n");
    }
}

int SvmSearch::solve(const SmoBatch &b, const std::vector<int> &order, const SmoProblem *d_probs, const SvrData *d_svr,
                     const NuData *d_nu, const int *d_order, int lmax, int *n_cl_out, int *n_ex_out)
{
    gs_profile &pf = h->prof;
    const int np = (int)b.probs.size();
    const bool csvc = !d_svr && !d_nu;                  // nu and SVR problems take one position-owned launch
    std::string why;                                    // set by launch_smo for a problem size it does not support
    const char *what = d_nu ? "launch_smo_nu" : d_svr ? "launch_smo_svr" : "launch_smo";
    auto fail = [&](cudaError_t e) {
        gs_set_error(h, why.empty() ? std::string(what) + ": " + cudaGetErrorString(e) : why);
        return why.empty() ? GS_ERR_CUDA : GS_ERR_UNSUPPORTED;
    };
    // single-CTA launches go to the slot-layout kernel (smo_lean.cu) when every problem of the batch has one;
    // B200GS_SMO_LEAN=0 forces the position-owned kernel (smo.cu)
    int max_slots = 0;
    bool lean_ok = csvc && lmax < 16383 && !(getenv("B200GS_SMO_LEAN") && atoi(getenv("B200GS_SMO_LEAN")) == 0);
    for (int q = 0; q < np && lean_ok; q++) {
        lean_ok = b.probs[q].nseg > 0 && b.probs[q].nslots <= smo_lean_max_slots();
        max_slots = std::max(max_slots, b.probs[q].nslots);
    }
    auto launch_single = [&](const int *ord, int cnt, cudaStream_t s_, bool exclusive) -> cudaError_t {
        for (int inst = fast ? 1 : 0; inst >= 0; inst--) {              // branch-free instance, then the general one (guarded)
            const cudaError_t e = lean_ok ? launch_smo_lean(d_probs, ord, cnt, max_slots, inst == 1, exclusive, s_)
                                          : launch_smo(d_probs, d_svr, d_nu, ord, cnt, lmax, inst == 1, (int)ldk, s_, &why);
            if (e != cudaSuccess) return e;
            pf.launches++;
        }
        return cudaSuccess;
    };
    // C-SVC policy: clusters and exclusive SMs buy LATENCY for the critical path at the price of SM time
    // (gs_svc_schedule); a throughput-bound search (config 4) uses neither.  A 4-CTA cluster solves one problem in about
    // half the time per iteration of the single-CTA kernel, but costs twice the SM-time per iteration.
    //   * fewer problems than SMs: everything on the widest cluster that fits;
    //   * otherwise the three-tier schedule of the slot-layout kernel, or -- when a problem has no slot layout -- the
    //     two-tier schedule of the position-owned kernel (gs_svc_cluster_count): exactly the ten 66-68k-iteration
    //     problems of config 2 go on clusters (at 148 and 132 SMs).
    // B200GS_SMO_CLUSTER (0/2/4/8) and B200GS_SMO_CLUSTER_N force the cluster size and the number of clustered problems.
    int cl = 0, n_cl = 0, n_ex = 0;
    if (csvc) {
        if (lmax > 2048) {
            if (np * 8 <= h->sm_count) { cl = 8; n_cl = np; }
            else if (np * 4 <= h->sm_count) { cl = 4; n_cl = np; }
            else if (np * 2 <= h->sm_count) { cl = 2; n_cl = np; }
            else {
                std::vector<double> sorted_cost(np);
                for (int q = 0; q < np; q++) sorted_cost[q] = b.cost[order[q]];
                if (lean_ok) gs_svc_schedule(sorted_cost.data(), np, h->sm_count, &n_cl, &n_ex);
                else n_cl = gs_svc_cluster_count(sorted_cost.data(), np, h->sm_count);
                if (n_cl > 0) cl = 4;
            }
        }
        if (const char *e = getenv("B200GS_SMO_CLUSTER")) { cl = atoi(e); if (n_cl == 0) n_cl = std::max(1, np * 6 / 100); }
        if (const char *e = getenv("B200GS_SMO_CLUSTER_N")) n_cl = std::min(np, atoi(e));
        if (!(cl == 2 || cl == 4 || cl == 8) || lmax > smo_colown_max_rows(cl) || lmax <= 2048) n_cl = 0;
        n_ex = std::max(0, std::min(n_ex, np - n_cl));
    }
    *n_cl_out = n_cl; *n_ex_out = n_ex;
    if (n_cl == 0 && n_ex == 0) {
        if (const cudaError_t ce = launch_single(d_order, np, st, false)) return fail(ce);
        return GS_OK;
    }
    // The latency tiers must get their SMs before the shared-SM launch floods the GPU (a late start of the critical path
    // costs the makespan that much).  So the cluster kernel goes on the engine stream itself, in order behind the uploads;
    // the exclusive and the shared launches go on two more streams behind the same point plus a 30 / 60 us delay kernel
    // (each counted as a launch); the engine stream joins them afterwards.
    cudaEvent_t ready = h->evp.get();
    cudaEventRecord(ready, st);
    if (n_cl > 0) {
        cudaError_t ce = cudaSuccess;
        for (int inst = fast ? 1 : 0; inst >= 0 && ce == cudaSuccess; inst--) {
            ce = launch_smo_colown(d_probs, d_order, n_cl, lmax, cl, inst == 1, st);
            pf.launches++;
        }
        if (ce != cudaSuccess) { what = "launch_smo_colown"; return fail(ce); }
    }
    if (n_ex > 0) {
        cudaEvent_t done = h->evp.get();
        cudaStreamWaitEvent(h->stream_hi, ready, 0);
        launch_delay(30000, h->stream_hi);
        if (const cudaError_t ce = launch_single(d_order + n_cl, n_ex, h->stream_hi, true)) return fail(ce);
        pf.launches++;
        cudaEventRecord(done, h->stream_hi);
        cudaStreamWaitEvent(st, done, 0);
    }
    if (np - n_cl - n_ex > 0) {
        cudaStream_t s2 = n_ex > 0 ? h->stream_lo : h->stream_hi;
        cudaEvent_t done = h->evp.get();
        cudaStreamWaitEvent(s2, ready, 0);
        launch_delay(n_ex > 0 ? 60000 : 30000, s2);
        if (const cudaError_t ce = launch_single(d_order + n_cl + n_ex, np - n_cl - n_ex, s2, false)) return fail(ce);
        pf.launches++;
        cudaEventRecord(done, s2);
        cudaStreamWaitEvent(st, done, 0);
    }
    return GS_OK;
}

int SvmSearch::score(int kind, const std::vector<VoteTask> &vtasks, const VoteTask *d_vt, void *d_votes)
{
    const int nvt = (int)vtasks.size(), nc = h->n_classes;
    const double *dec = h->dWork[4].as<double>();
    if (!h->classification) {
        GS_CUDA(launch_rss(dec, d_rho, n, h->dZ64.as<double>(), h->masks(), d_vt, nvt, (double *)d_votes, st));
    } else if (kind == GS_SCORE_DEFAULT) {
        GS_CUDA(launch_vote(dec, d_rho, n, nc, h->dY.as<int>(), h->masks(), d_vt, nvt, (int *)d_votes, st));
    } else if (kind == GS_SCORE_ROC_AUC) {
        // rank statistic of the decision values already in HBM (scikit-learn: roc_auc_score(y, decision_function(X)))
        std::vector<int> meta((size_t)nvt * 2);
        for (int v = 0; v < nvt; v++) { meta[v] = vtasks[v].first_col; meta[nvt + v] = vtasks[v].fold; }
        GS_CUDA(h->dScore.reserve((size_t)nvt * (8 + 32)));
        unsigned long long *d_auc = h->dScore.as<unsigned long long>();
        int *d_meta = (int *)(d_auc + (size_t)nvt * 4);
        GS_CUDA(cudaMemcpyAsync(d_meta, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemsetAsync(d_auc, 0, (size_t)nvt * 32, st));
        GS_CUDA(launch_auc_pairs_f64(dec, n, n, h->class_start[1], h->masks(), d_meta, d_meta + nvt, nvt, -1, d_auc, st));
        auc_pairs.resize((size_t)nvt * 4);
        GS_CUDA(cudaMemcpyAsync(auc_pairs.data(), d_auc, (size_t)nvt * 32, cudaMemcpyDeviceToHost, st));
    } else {
        GS_CUDA(h->dScore.reserve((size_t)nvt * 2 * nc * 3 * 4));
        GS_CUDA(cudaMemsetAsync(h->dScore.p, 0, (size_t)nvt * 2 * nc * 3 * 4, st));
        GS_CUDA(launch_vote_classes(dec, d_rho, n, nc, h->dY.as<int>(), h->masks(), d_vt, nvt, h->dScore.as<int>(), st));
        class_counts.resize((size_t)nvt * 2 * nc * 3);
        GS_CUDA(cudaMemcpyAsync(class_counts.data(), h->dScore.p, class_counts.size() * 4, cudaMemcpyDeviceToHost, st));
    }
    h->prof.launches++;
    return GS_OK;
}

int SvmSearch::run(const SvmModel &m, double *test_scores, double *train_scores, int32_t *n_iter, int32_t *n_sv, float *fit_ms,
                   float *score_ms, double *coef_out, double *rho_out)
{
    gs_profile &pf = h->prof;
    const bool regression = !h->classification;
    const int n_tasks = (int)task_group.size(), n_groups = (int)groups.size(), nc = h->n_classes;
    const SplitScoreStats ss(h, m.n_splits, m.kind);
    if (const int rc = plan_batches()) return rc;
    GS_CUDA(h->dWork[0].reserve(m.rows.size() * 4));
    GS_CUDA(cudaMemcpyAsync(h->dWork[0].p, m.rows.data(), m.rows.size() * 4, cudaMemcpyHostToDevice, st));
    pf.h2d_bytes += m.rows.size() * 4;

    std::vector<int> task_iter(n_tasks, 0), task_sv(n_tasks, 0);
    std::vector<double> task_fit_ms(n_tasks, 0.0), task_score((size_t)n_tasks * 2, 0.0);   // test, train
    std::vector<char> task_bad(n_tasks, 0);
    int64_t total_iter = 0;
    double solve_bytes = 0;
    for (int g0 = 0; g0 < n_groups; g0 += per_batch) {
        const int g1 = std::min(n_groups, g0 + per_batch);
        if (const int rc = kernel_matrices(g0, g1)) return rc;
        // -- problems, ordered by (group, task, problem of the task): column index == problem index --
        SmoBatch b;
        std::vector<int> prob_task, vtask_id, group_first(g1 - g0 + 1, 0);
        std::vector<VoteTask> vtasks;
        for (int g = g0; g < g1; g++) {
            group_first[g - g0] = (int)b.probs.size();
            for (int t : group_tasks[g]) {
                if (!m.skip.empty() && m.skip[t]) continue;
                vtasks.push_back(VoteTask{(int)b.probs.size(), m.refit ? -100 : t % m.n_splits});
                vtask_id.push_back(t);
                SmoProblem P;
                memset(&P, 0, sizeof P);
                P.K = h->dK.as<float>() + (size_t)(g - g0) * n * ldk;
                P.qd = qd(g, g0);
                P.rows = h->dWork[0].as<int>();
                P.ldk = ldk; P.eps = m.tol; P.max_iter = m.max_iter;
                P.shrinking = (m.flags & GS_NO_SHRINKING) ? 0 : 1;
                P.guard = d_guard;
                m.add_task(t, groups[g], P, b);
                prob_task.resize(b.probs.size(), t);
            }
        }
        group_first[g1 - g0] = (int)b.probs.size();
        const int np = (int)b.probs.size(), nvt = (int)vtasks.size();
        if (np == 0) continue;                                // every task of the batch is skipped
        if (const int rc = workspaces(b.probs)) return rc;
        std::vector<int> order(np);                           // launch order: the costliest problems first
        std::iota(order.begin(), order.end(), 0);
        std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return b.cost[x] > b.cost[y]; });
        // -- batch metadata in h->dWork[6]: problems, SvrData, NuData, launch order, vote tasks, and 16 bytes per vote task
        // for its votes: vote counts {test correct, total, train correct, total} or residual sums of squares {test, train} --
        const size_t o_svr = (size_t)np * sizeof(SmoProblem), o_nu = o_svr + b.svr.size() * sizeof(SvrData),
                     o_order = o_nu + b.nu.size() * sizeof(NuData), o_vt = round_up(o_order + (size_t)np * 4, 16),
                     o_votes = round_up(o_vt + (size_t)nvt * sizeof(VoteTask), 16);
        GS_CUDA(h->dWork[6].reserve(o_votes + (size_t)nvt * 16));
        unsigned char *dm = h->dWork[6].as<unsigned char>();
        GS_CUDA(cudaMemcpyAsync(dm, b.probs.data(), o_svr, cudaMemcpyHostToDevice, st));
        if (!b.svr.empty()) GS_CUDA(cudaMemcpyAsync(dm + o_svr, b.svr.data(), o_nu - o_svr, cudaMemcpyHostToDevice, st));
        if (!b.nu.empty()) GS_CUDA(cudaMemcpyAsync(dm + o_nu, b.nu.data(), o_order - o_nu, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(dm + o_order, order.data(), (size_t)np * 4, cudaMemcpyHostToDevice, st));
        GS_CUDA(cudaMemcpyAsync(dm + o_vt, vtasks.data(), (size_t)nvt * sizeof(VoteTask), cudaMemcpyHostToDevice, st));
        if (!regression) GS_CUDA(cudaMemsetAsync(dm + o_votes, 0, (size_t)nvt * 16, st));   // the vote kernels add to it
        GS_CUDA(cudaMemsetAsync(h->dWork[3].p, 0, (size_t)np * n * 8, st));
        pf.h2d_bytes += o_order + (size_t)np * 4 + (size_t)nvt * sizeof(VoteTask);
        tm.mark(4);
        // -- solve --
        int n_cl = 0, n_ex = 0;
        if (const int rc = solve(b, order, (const SmoProblem *)dm, b.svr.empty() ? nullptr : (const SvrData *)(dm + o_svr),
                                 b.nu.empty() ? nullptr : (const NuData *)(dm + o_nu), (const int *)(dm + o_order), m.lmax, &n_cl, &n_ex))
            return rc;
        tm.mark(2);
        // -- score (a refit does not) --
        if (!m.refit) {
            if (const int rc = decisions(g0, g1, group_first)) return rc;
            if (const int rc = score(m.kind, vtasks, (const VoteTask *)(dm + o_vt), dm + o_votes)) return rc;
        }
        tm.mark(3);
        // -- results of this batch --
        std::vector<int> votes(regression ? 0 : (size_t)nvt * 4);           // a classifier's, also in a refit
        std::vector<double> rss(regression && !m.refit ? (size_t)nvt * 2 : 0);
        if (!votes.empty()) GS_CUDA(cudaMemcpyAsync(votes.data(), dm + o_votes, votes.size() * 4, cudaMemcpyDeviceToHost, st));
        if (!rss.empty()) GS_CUDA(cudaMemcpyAsync(rss.data(), dm + o_votes, rss.size() * 8, cudaMemcpyDeviceToHost, st));
        pf.d2h_bytes += votes.size() * 4 + rss.size() * 8;
        if (const int rc = results(np, m.refit && coef_out)) return rc;
        for (int q = 0; q < np; q++) {
            const int t = prob_task[q], it = info[(size_t)q * 4];
            task_iter[t] += it; task_sv[t] += info[(size_t)q * 4 + 2];
            task_fit_ms[t] += (double)(ns[(size_t)q * 12 + 1] - ns[(size_t)q * 12]) * 1e-6;
            total_iter += it;
            // two gathered K rows of the problem's (initially full) active set per iteration, over its distinct columns
            // (an SVR problem holds every training row twice)
            const int cols = b.svr.empty() ? b.probs[q].l : b.probs[q].l / 2;
            solve_bytes += (double)it * 2.0 * cols * 4.0;
            // a task whose solve went non-finite scores NaN; the caller applies error_score to THAT task only
            // (reference base_search.py:69,87: _fit_and_score(..., error_score) fills per task)
            if (!std::isfinite(rho[q])) {
                if (m.refit) { gs_set_error(h, std::string(m.who) + "_refit: non-finite intercept"); return GS_ERR_NUMERIC; }
                task_bad[t] = 1;
            }
        }
        smo_diagnostics(order, n_cl, n_ex, info, ns);
        if (m.refit) {
            for (int q = 0; q < np; q++) {
                if (rho_out) rho_out[q] = rho[q];
                if (n_iter) n_iter[q] = info[(size_t)q * 4];
                if (coef_out)
                    for (int r = 0; r < n; r++) coef_out[(size_t)q * n + h->perm[r]] = coef[(size_t)q * n + r];
            }
            continue;
        }
        for (int v = 0; v < nvt; v++)
            for (int sp = 0; sp < 2; sp++) {
                const int k = vtasks[v].fold;
                double &sc = task_score[(size_t)vtask_id[v] * 2 + sp];
                if (regression) sc = ss.regression(k, sp, rss[(size_t)v * 2 + sp]);
                else if (m.kind == GS_SCORE_DEFAULT) sc = SplitScoreStats::accuracy(&votes[(size_t)v * 4 + sp * 2]);
                else if (m.kind == GS_SCORE_ROC_AUC) sc = ss.auc(k, sp, &auc_pairs[(size_t)v * 4 + sp * 2]);
                else sc = ss.counts(&class_counts[((size_t)v * 2 + sp) * nc * 3]);
            }
    }
    if (const int rc = finish(total_iter, solve_bytes)) return rc;

    if (!m.refit)
        for (int t = 0; t < n_tasks; t++) {
            const bool skipped = !m.skip.empty() && m.skip[t], nan = skipped || task_bad[t];
            test_scores[t] = nan ? NAN : task_score[(size_t)t * 2];
            if (train_scores) train_scores[t] = nan ? NAN : task_score[(size_t)t * 2 + 1];
            if (n_iter) n_iter[t] = skipped ? -1 : task_iter[t];
            if (n_sv) n_sv[t] = task_sv[t];
            if (fit_ms) fit_ms[t] = (float)task_fit_ms[t];
            if (score_ms) score_ms[t] = pf.ms_score / (float)n_tasks;
        }
    return GS_OK;
}
