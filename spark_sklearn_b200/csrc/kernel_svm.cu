// kernel_svm.cu -- the host steps of a kernel-SVM search that do not depend on the model (svc_run in api.cu, svr_run in
// svr.cu).  Host code only.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <map>

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

void SvmSearch::begin()
{
    gs_profile_reset(h->prof);
    h->evp.reset(); h->tt.reset();
    ev_begin = h->evp.get(); ev_end = h->evp.get();
    cudaEventRecord(ev_begin, st);
    tm.mark(-1);
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
