// smo.cu -- batched C-SVC dual solver: one CTA per (candidate, fold, class-pair) sub-problem.
//
// Restates scikit-learn's libsvm Solver (svm.cpp:670-944 Solve, :946-1047 select_working_set,
// :1049-1129 do_shrinking, :629-668 reconstruct_gradient, :1131-1168 calculate_rho) as a
// block-parallel kernel that reproduces libsvm's ITERATE SEQUENCE, not just its fixed point:
//   * same WSS2 pair selection incl. tie-breaking ("last index wins" == (value, index) arg-reductions),
//   * same shrinking schedule and the same swap permutation (parallel two-pointer partition),
//   * same float64 arithmetic op-for-op: every multiply/add/divide is individually rounded
//     (__dmul_rn/__dadd_rn/__ddiv_rn are never contracted; libsvm's x86-64 build has no FMA),
//   * Q entries are the float32-rounded kernel values (Qfloat) read from the K matrix of gram.cu.
// Libsvm stops at a KKT gap of 1e-3; two solvers that merely agree on the optimum differ by ~1e-3 in
// decision values and flip test points near the margin -- more than the 1e-4 budget on
// mean_test_score.  Following the same trajectory removes that.
//
// Sign-free state ("m-domain").  With m_t = -y_t*G_t and mbar_t = -y_t*Gbar_t (negation is exact, so
// every rounding is mirrored bit for bit) all per-element sign handling of libsvm disappears:
//   select i:  argmax { m_t : t in I_up }                      (svm.cpp:964-978, both y branches)
//   select j:  gd = Gmax - m_t, quad = (QD_i+QD_t) - 2*K_it     (svm.cpp:986-1037, both y branches;
//              -2*y_i*Q_it == -2*K_it for y_t=+1 and +2*y_i*Q_it == -2*K_it for y_t=-1)
//   update:    m_t += fl(fl(K_it*a) + fl(K_jt*b)),  a = -y_i*dalpha_i, b = -y_j*dalpha_j   (:866-872)
//   G_bar:     mbar_t += fl(c*K_it),  c = -/+ y_i*C_i                                       (:876-905)
// where K is the UNSIGNED float32 kernel row.  Set membership is two precomputed flag bits.
//
// Throughput design (H100: 64 FP64 lanes/SM, 4 issue slots/clk/SM -- this kernel is FP64-pipe and
// issue bound, then latency bound; see DESIGN.md):
//   * the exact float64 division of WSS2 is evaluated only for elements that survive an approximate
//     filter (float32 arithmetic for rbf, a 20-bit reciprocal otherwise) with a provably safe band; the
//     winner is still chosen from exactly-rounded libsvm values, so the selection is bit-identical;
//   * float32->float64 widening of the K entries uses integer bit operations (ALU pipe) instead of
//     F2F (quarter-rate on the FP64 pipe);
//   * block arg-reductions run on REDUX.MAX over order-preserving 64-bit integer keys, not on
//     FP64 compares + shuffles;
//   * all solver state (m, mbar, alpha, column map, flags) of a sub-problem with <= 8192 rows is
//     resident in shared memory (27 B/row, 221 KB), the Q_i row of the owned positions in registers.
// Per iteration: two dependent gathers of a K row (HBM/L2), three CTA barriers.
#include "smo_common.cuh"
#include <cstdlib>

namespace {

using namespace smo;

// FAST: every problem of the launch is rbf (QD == 1) and its K matrix holds only positive normal floats,
// so the widening is three integer instructions and quad = 2 - 2K needs no diagonal lookups.
// ROWBUF: the two K rows of an iteration are brought into shared memory by ONE bulk asynchronous copy each
// (cp.async.bulk, mbarrier-signalled) and gathered from there.  A row gathered with per-thread LDGs is throttled by
// the SM's outstanding-miss capacity (~64 lines x ~900 cycles of DRAM latency = ~18 GB/s per SM, 2.5 us per 32 KB row,
// on the 148-SM GPU the kernels were first tuned on); the bulk copy streams the whole 40 KB row at the SM's full fill rate.  G_bar then lives in global memory.
template <int NT, int KPT, bool SMEM_STATE, bool FAST, bool PROF, bool ROWBUF>
__global__ void __launch_bounds__(NT, 1)
smo_kernel(const SmoProblem *__restrict__ probs, const int *__restrict__ order, int rowcap)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ Red red;
    constexpr int NW = NT / 32;
    constexpr int LCAP = NT * KPT;                                          // compile-time layout: no address math

    const SmoProblem *__restrict__ Pp = probs + order[blockIdx.x];
    if (Pp->guard != nullptr && (*Pp->guard != 0) == FAST) return;       // the other instance solves this launch (common.cuh)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int l = Pp->l;
    // ---- resident state ----
    double *const mG = reinterpret_cast<double *>(smem_raw);                // m_t = -y_t G_t
    double *mGbar, *alpha;
    unsigned short *col;                                                    // dataset row of each position
    if constexpr (ROWBUF) {
        alpha = mG + LCAP; mGbar = Pp->Gbar;
        col = reinterpret_cast<unsigned short *>(mG + 2 * LCAP);
    } else if constexpr (SMEM_STATE) {
        mGbar = mG + LCAP; alpha = mG + 2 * LCAP;
        col = reinterpret_cast<unsigned short *>(mG + 3 * LCAP);
    } else {
        mGbar = Pp->Gbar; alpha = Pp->alpha;
        col = reinterpret_cast<unsigned short *>(mG + LCAP);
    }
    unsigned char *const fl = reinterpret_cast<unsigned char *>(col + LCAP);
    // LCAP is a multiple of 128, so the row buffer starts 128-byte aligned; a pointer derived by plain arithmetic keeps
    // the shared address space (an integer round-up made every gather a generic LD instead of LDS)
    float *const rowbuf = reinterpret_cast<float *>(fl + LCAP);
    __shared__ unsigned long long rowbar;
    unsigned rowphase = 0;
    const float *__restrict__ const K = Pp->K;
    const int64_t ldk = Pp->ldk;
    const double eps = Pp->eps;
    const bool use_gbar = Pp->shrinking != 0;
    const double *__restrict__ const qd = FAST ? nullptr : Pp->qd;
    int *const scratch = Pp->scratch;

    unsigned long long t_start = 0;
    if (tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));

    // ---- initial point: alpha = 0, G = p = -1  =>  m_t = y_t (svm.cpp:1611-1626, :716-736) ----
    {
        const int n_pos = Pp->n_pos;
        const int *__restrict__ rows = Pp->rows;
        for (int t = tid; t < l; t += NT) {
            const bool yp = t < n_pos;
            mG[t] = yp ? 1.0 : -1.0;
            col[t] = (unsigned short)rows[t];
            fl[t] = (unsigned char)mkflags(yp, ST_LOWER);
            alpha[t] = 0.0;
            if (use_gbar) mGbar[t] = 0.0;
        }
        for (int t = l + tid; t < LCAP; t += NT) { mG[t] = 0.0; col[t] = 0; fl[t] = 0; }   // slots past l: inert
    }
    if constexpr (ROWBUF) {
        if (tid == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((unsigned)__cvta_generic_to_shared(&rowbar)));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
    }
    __syncthreads();

    // bulk fetch of dataset row `r` of K into rowbuf (issued by one thread) and the matching wait (all threads)
    // this thread's share of a row copy (threads 0..3): one of the problem's column ranges, or a quarter of the whole row
    unsigned cp_off = 0, cp_cnt = 0, cp_total = 0;
    if constexpr (ROWBUF) {
        const int nseg = Pp->nseg;
        if (nseg > 0) {
            for (int e = 0; e < nseg; e++) cp_total += (unsigned)Pp->seg_len[e];
            if (tid < nseg) { cp_off = (unsigned)Pp->seg_start[tid]; cp_cnt = (unsigned)Pp->seg_len[tid]; }
        } else {
            const unsigned part = ((unsigned)rowcap / 4u) & ~3u;            // floats per part, 16-byte multiple
            cp_total = (unsigned)rowcap;
            if (tid < 4) { cp_off = (unsigned)tid * part; cp_cnt = tid == 3 ? (unsigned)rowcap - 3u * part : part; }
        }
    }
    auto fetch_row = [&](int r) {
        if constexpr (ROWBUF) {
            // up to four bulk copies in flight at once (1.7k cycles from HBM for a 40 KB row instead of 2.05k for one copy,
            // on the 148-SM GPU the kernels were first tuned on), and only the column ranges this sub-problem reads
            const unsigned bar = (unsigned)__cvta_generic_to_shared(&rowbar);
            if (tid == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(cp_total * 4u) : "memory");
            if (cp_cnt)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"((unsigned)__cvta_generic_to_shared(rowbuf + cp_off)), "l"(K + (size_t)r * ldk + cp_off), "r"(cp_cnt * 4u), "r"(bar) : "memory");
        }
    };
    auto wait_row = [&]() {
        if constexpr (ROWBUF) {
            const unsigned bar = (unsigned)__cvta_generic_to_shared(&rowbar);
            unsigned done = 0;
            for (unsigned spin = 0; !done; ++spin) {
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(done) : "r"(bar), "r"(rowphase) : "memory");
                if (spin > (1u << 26)) __trap();
            }
            rowphase ^= 1u;
        }
    };

    int active = l, iter = 0, timed_out = 0;
    int counter = (l < 1000 ? l : 1000) + 1;
    bool unshrink = false;
    const int max_iter = Pp->max_iter == -1 ? SAFETY_MAX_ITER : Pp->max_iter;

    long long prof[6] = {0, 0, 0, 0, 0, 0};
    long long tprev = PROF ? clock64() : 0;
    auto tick = [&](int slot) {
        if constexpr (PROF) {
            const long long now = clock64();
            prof[slot] += now - tprev;
            tprev = now;
        }
    };

    float kvi[KPT];      // unsigned K_i row (float32 as stored) at the owned active positions t = k*NT + tid; widened on use

    auto QD = [&](int t) -> double {                                        // svm.cpp:1436-1437
        if constexpr (FAST) return 1.0;
        else return qd ? qd[col[t]] : 1.0;
    };
    auto widen = [&](float x) -> double {
        if constexpr (FAST) {
            const unsigned u = __float_as_uint(x);
            return __hiloint2double((int)((u >> 3) + 0x38000000u), (int)(u << 29));
        } else return f2d(x);
    };

    // ---------------- local scan: this thread's candidates for the next working-set selection -------
    // la/la_idx: arg-max m over its I_up positions (ties -> larger position); lm: min m over its I_low
    // positions (Gmax2 = max -m, svm.cpp:986-1031).  Normally produced for free by the update loop.
    double la = -CUDART_INF, lm = CUDART_INF;
    int la_idx = -1;
    auto local_scan = [&]() {
        la = -CUDART_INF; lm = CUDART_INF; la_idx = -1;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int t = k * NT + tid;
            if (t < active) {
                const int f = fl[t];
                const double m = mG[t];
                if ((f & F_UP) && m >= la) { la = m; la_idx = (t << IDX_SHIFT) | f; }
                if (f & F_LOW) lm = fmin(lm, m);
            }
        }
    };

    // ---------------- reconstruct_gradient (svm.cpp:629-668), m-domain ----------------
    // G_k = (Gbar_k + p_k) + sum_{free f, ascending} alpha_f Q_fk   <=>
    // m_k = (mbar_k + y_k) + sum_f fl((-y_f alpha_f) K_fk), same roundings mirrored.
    auto rebuild_gradient = [&]() {
        if (active == l) return;
        int nf = 0;
        for (int base = 0; base < active; base += NT) {
            const int t = base + tid;
            const bool isf = t < active && (fl[t] & 3) == ST_FREE;
            int tot;
            const int r = block_rank<NT>(isf, red.cnt, tot);
            if (isf) scratch[nf + r] = t;
            nf += tot;
        }
        __syncthreads();
        double g[KPT];
        int ck[KPT];
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int t = k * NT + tid;
            const bool in = t >= active && t < l;
            g[k] = in ? __dadd_rn(mGbar[t], (fl[t] & F_YPOS) ? 1.0 : -1.0) : 0.0;
            ck[k] = in ? (int)col[t] : -1;
        }
#pragma unroll 2
        for (int r = 0; r < nf; r++) {
            const int f = scratch[r];
            const float *__restrict__ Kf = K + (size_t)col[f] * ldk;
            const double af = (fl[f] & F_YPOS) ? -alpha[f] : alpha[f];      // -y_f alpha_f
#pragma unroll
            for (int k = 0; k < KPT; k++)
                if (ck[k] >= 0) g[k] = __dadd_rn(g[k], __dmul_rn(af, widen(__ldg(Kf + ck[k]))));
        }
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int t = k * NT + tid;
            if (t >= active && t < l) mG[t] = g[k];
        }
        __syncthreads();
    };

    // ---------------- select_working_set (svm.cpp:946-1047) ----------------
    int pi = -1, pj = -1;            // packed (position << 5 | flags)
    double gmax = 0, mg_j = 0, k_ij = 0, alpha_i = 0, alpha_j = 0;
    auto select = [&]() -> bool {
        // ---- phase A: i = argmax m_t over I_up; Gmax2 = max -m_t over I_low (both from the local scan) ----
        double gmax2;
        {
            const unsigned long long key = dkey(la);
            const KArg w = warp_argmax((unsigned)(key >> 32), (unsigned)key, la_idx);
            const unsigned long long km = warp_keymax(dkey(-lm));
            if (lane == 0) {
                red.a_hi[warp] = w.hi; red.a_lo[warp] = w.lo; red.a_idx[warp] = w.idx;
                red.m_hi[warp] = (unsigned)(km >> 32); red.m_lo[warp] = (unsigned)km;
            }
            tick(0);
            __syncthreads();                                                      // barrier 1
            tick(1);
            const bool v = lane < NW;
            const KArg a = warp_argmax(v ? red.a_hi[lane] : 0u, v ? red.a_lo[lane] : 0u, v ? red.a_idx[lane] : -1);
            const unsigned long long km2 =
                warp_keymax(v ? (((unsigned long long)red.m_hi[lane] << 32) | red.m_lo[lane]) : 0ull);
            pi = a.idx;
            gmax = dkey_inv(((unsigned long long)a.hi << 32) | a.lo);
            gmax2 = dkey_inv(km2);
        }
        if (pi < 0 || __dadd_rn(gmax, gmax2) < eps) return true;              // svm.cpp:1040-1041
        // ---- phase B: j = argmin -(gd^2)/quad over I_low with gd > 0 (svm.cpp:980-1037) ----
        // Approximate arg-max of gd^2/quad with a 20-bit reciprocal; it IS libsvm's choice unless the
        // runner-up lies within the error band, in which case the exact quotients decide (rare path).
        const int i = pi >> IDX_SHIFT;
        alpha_i = alpha[i];
        const double QDi = QD(i);
        const float *__restrict__ Ki = K + (size_t)col[i] * ldk;
        {
            if constexpr (ROWBUF) { fetch_row(col[i]); wait_row(); }
#pragma unroll
            for (int k = 0; k < KPT; k++) {                                  // issue the whole gather first
                const int t = k * NT + tid;
                if constexpr (ROWBUF) kvi[k] = t < active ? rowbuf[col[t]] : 0.f;
                else kvi[k] = t < active ? __ldg(Ki + col[t]) : 0.f;
            }
        }
        // Approximate gd^2/quad is tracked by a 32-bit order-preserving key; every near-tie (keys within BAND units) is
        // decided by the exact libsvm quotients below, so the choice stays bit-identical.
        //   FAST (rbf, 0 < K normal): the key is the bit pattern of a FLOAT32 evaluation (gd rounded to float, quad =
        //     2 - 2K exact-then-rounded, rcp.approx.f32, two products): relative error < 7 * 2^-24 < 2^-21 per candidate,
        //     one key unit >= 2^-24 relative, BAND = 64 units = 2^-18 > 2 * 2^-21.  Three FP64-pipe instructions per
        //     element instead of ten.  Below 2^-100 (flush-to-zero territory) every candidate goes to the exact path.
        //   otherwise: the HIGH WORD of a double evaluation with rcp.approx.f64 (2^-20-accurate), BAND = 514 units >= 2^-12.
        constexpr unsigned BAND = FAST ? 64u : 514u;
        constexpr unsigned KEY_TINY = 0x0D800000u;                          // float bits of 2^-100
        auto approx_key = [&](double gd, float kvf, int t) -> unsigned {
            if constexpr (FAST) {
                const float gdf = __double2float_rn(gd);
                const float quadf = __fmaf_rn(-2.f, kvf, 2.f);              // == fl32(2 - 2K): 2K is exact
                const float g2f = __fmul_rn(gdf, gdf);
                float r;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(quadf));
                const float apf = quadf > 0.f ? __fmul_rn(g2f, r) : __fmul_rn(g2f, 1e12f);
                return __float_as_uint(apf) + 1u;                           // +1: a valid candidate is never 0
            } else {
                const double q = widen(kvf);
                const double quad = __dsub_rn(__dadd_rn(QDi, QD(t)), __dmul_rn(2.0, q));
                const double g2 = __dmul_rn(gd, gd);
                const double ap = quad > 0 ? g2 * rcp_approx(quad) : g2 * 1e12;
                return (unsigned)__double2hiint(ap) + 1u;
            }
        };
        unsigned b1k = 0u, b2k = 0u;                    // keys of the best and second-best candidate (0 = none)
        int k1 = -1;
        double m1 = 0, q1 = 0;
        int idx1 = -1;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int t = k * NT + tid;
            if (t < active) {
                const int f = fl[t];
                const double m = mG[t];
                const double gd = __dsub_rn(gmax, m);
                if ((f & F_LOW) && gd > 0) {
                    const unsigned key = approx_key(gd, kvi[k], t);
                    const bool gt = key > b1k;
                    b2k = gt ? b1k : max(b2k, key);
                    b1k = gt ? key : b1k;
                    k1 = gt ? k : k1;
                }
            }
        }
        if (k1 >= 0) {
            const int t1 = k1 * NT + tid, s1 = t1;
            idx1 = (t1 << IDX_SHIFT) | fl[s1];
            m1 = mG[s1];
            float kq = kvi[0];
#pragma unroll
            for (int k = 1; k < KPT; k++) kq = k == k1 ? kvi[k] : kq;
            q1 = widen(kq);
        }
        unsigned top1k, top2k;
        {
            const unsigned w1 = __reduce_max_sync(0xffffffffu, b1k);
            const int widx = __reduce_max_sync(0xffffffffu, (b1k == w1) ? idx1 : -1);
            const unsigned w2 = __reduce_max_sync(0xffffffffu, (idx1 == widx) ? b2k : b1k);
            if (idx1 >= 0 && idx1 == widx) {                                   // this lane owns the warp's winner
                red.pl_mg[warp] = m1; red.pl_kv[warp] = q1; red.pl_alpha[warp] = alpha[idx1 >> IDX_SHIFT];
            }
            if (lane == 0) { red.b_hi[warp] = w1; red.b_idx[warp] = widx; red.t_hi[warp] = w2; }
            tick(2);
            __syncthreads();                                                      // barrier 2
            tick(3);
            const bool v = lane < NW;
            const unsigned bk = v ? red.b_hi[lane] : 0u;
            const int bi = v ? red.b_idx[lane] : -1;
            top1k = __reduce_max_sync(0xffffffffu, bk);
            pj = __reduce_max_sync(0xffffffffu, (bk == top1k) ? bi : -1);
            top2k = __reduce_max_sync(0xffffffffu, (v && bi == pj) ? red.t_hi[lane] : bk);
            if (pj < 0) return true;                                               // Gmin_idx == -1
        }
        if (top1k - top2k <= BAND || (FAST && top1k <= KEY_TINY)) {
            // ---- exact tie-break: libsvm's correctly rounded quotients for every element in the band ----
            const unsigned thrk = (top1k > BAND && !(FAST && top1k <= KEY_TINY)) ? top1k - BAND : 1u;
            double bestn = -CUDART_INF;
            int bidx = -1;
#pragma unroll
            for (int k = 0; k < KPT; k++) {
                const int t = k * NT + tid;
                if (t < active) {
                    const int f = fl[t];
                    const double m = mG[t];
                    const double gd = __dsub_rn(gmax, m);
                    if ((f & F_LOW) && gd > 0) {
                        if (approx_key(gd, kvi[k], t) >= thrk) {
                            const double q = widen(kvi[k]);
                            const double quad = __dsub_rn(__dadd_rn(QDi, QD(t)), __dmul_rn(2.0, q));
                            const double g2 = __dmul_rn(gd, gd);
                            const double nod = quad > 0 ? __ddiv_rn(g2, quad) : __ddiv_rn(g2, TAU);   // == -obj_diff
                            if (nod >= bestn) { bestn = nod; bidx = (t << IDX_SHIFT) | f; m1 = m; q1 = q; }
                        }
                    }
                }
            }
            const unsigned long long key = dkey(bestn);
            const KArg w = warp_argmax((unsigned)(key >> 32), (unsigned)key, bidx);
            if (bidx >= 0 && bidx == w.idx) {
                red.pl_mg[warp] = m1; red.pl_kv[warp] = q1; red.pl_alpha[warp] = alpha[bidx >> IDX_SHIFT];
            }
            if (lane == 0) { red.x_hi[warp] = w.hi; red.x_lo[warp] = w.lo; red.x_idx[warp] = w.idx; }
            __syncthreads();                                                      // rare barrier
            const bool v = lane < NW;
            const KArg b = warp_argmax(v ? red.x_hi[lane] : 0u, v ? red.x_lo[lane] : 0u, v ? red.x_idx[lane] : -1);
            pj = b.idx;
        }
        const int wj = ((pj >> IDX_SHIFT) % NT) >> 5;
        mg_j = red.pl_mg[wj]; k_ij = red.pl_kv[wj]; alpha_j = red.pl_alpha[wj];
        return false;
    };

    // ---------------- do_shrinking (svm.cpp:1070-1129), m-domain ----------------
    // Gmax1 = max{m_t : I_up}, Gmax2 = max{-m_t : I_low}; be_shrunk(t) = (!up && m_t > Gmax1) || (!low && -m_t > Gmax2)
    auto do_shrink = [&]() {
        double g1 = -CUDART_INF, g2 = -CUDART_INF;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int t = k * NT + tid;
            if (t < active) {
                const int f = fl[t];
                const double m = mG[t];
                if (f & F_UP) g1 = fmax(g1, m);
                if (f & F_LOW) g2 = fmax(g2, -m);
            }
        }
        g1 = block_max<NT>(g1, red.dm);
        g2 = block_max<NT>(g2, red.dm2);
        if (!unshrink && __dadd_rn(g1, g2) <= __dmul_rn(eps, 10.0)) {
            unshrink = true;
            rebuild_gradient();
            active = l;
        }
        int keep_local = 0;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int t = k * NT + tid;
            if (t < active) {
                const int f = fl[t] & 31;
                const double m = mG[t];
                const bool s = (!(f & F_UP) && m > g1) || (!(f & F_LOW) && -m > g2);
                fl[t] = (unsigned char)(f | (s ? F_MARK : 0));
                keep_local += s ? 0 : 1;
            }
        }
#pragma unroll
        for (int m = 16; m; m >>= 1) keep_local += __shfl_xor_sync(0xffffffffu, keep_local, m);
        __syncthreads();
        if (lane == 0) red.cnt[warp] = keep_local;
        __syncthreads();
        int na = 0;
#pragma unroll
        for (int w = 0; w < NW; w++) na += red.cnt[w];
        if (na != active) {
            // Two-pointer partition == pair the k-th marked position below na (ascending) with the k-th
            // unmarked position at/above na (descending).
            int *plist = scratch, *qlist = scratch + l;
            int np = 0, nq = 0;
            for (int base = 0; base < na; base += NT) {
                const int t = base + tid;
                const bool pr = t < na && (fl[t] & F_MARK);
                int tot;
                const int r = block_rank<NT>(pr, red.cnt, tot);
                if (pr) plist[np + r] = t;
                np += tot;
            }
            for (int base = na; base < active; base += NT) {
                const int t = base + tid;
                const bool pr = t < active && !(fl[t] & F_MARK);
                int tot;
                const int r = block_rank<NT>(pr, red.cnt, tot);
                if (pr) qlist[nq + r] = t;
                nq += tot;
            }
            __syncthreads();
            for (int r = tid; r < np; r += NT) {                 // np == nq; disjoint pairs
                const int p = plist[r], q = qlist[np - 1 - r];
                const double gp = mG[p]; mG[p] = mG[q]; mG[q] = gp;
                const unsigned short cp = col[p]; col[p] = col[q]; col[q] = cp;
                const unsigned char fp = fl[p]; fl[p] = fl[q]; fl[q] = fp;
                const double ap = alpha[p], aq = alpha[q]; alpha[p] = aq; alpha[q] = ap;
                const double bp = mGbar[p], bq = mGbar[q]; mGbar[p] = bq; mGbar[q] = bp;
            }
            active = na;
        }
        __syncthreads();
        for (int t = tid; t < l; t += NT) fl[t] &= 31;         // clear marks (owner-mapped)
        __syncthreads();
    };

    // ---------------- main loop (svm.cpp:742-907) ----------------
    bool scan_valid = false;
    for (;;) {
        if (iter >= max_iter) { timed_out = 1; break; }
        if (--counter == 0) {
            counter = l < 1000 ? l : 1000;
            if (use_gbar) { do_shrink(); scan_valid = false; }
            if constexpr (PROF) tprev = clock64();
        }
        if (!scan_valid) local_scan();
        if (select()) {
            rebuild_gradient();
            active = l;
            __syncthreads();                                     // selection scratch is rewritten below
            local_scan();
            if (select()) break;
            counter = 1;
        }
        ++iter;

        const int i = pi >> IDX_SHIFT, j = pj >> IDX_SHIFT;
        const float *__restrict__ Kj = K + (size_t)col[j] * ldk;
        float kvj[KPT];
        if constexpr (ROWBUF) fetch_row(col[j]);                 // everybody is past barrier 2: row i is no longer read
        else {
#pragma unroll
            for (int k = 0; k < KPT; k++) {                      // issue the Q_j gather before the scalar update
                const int t = k * NT + tid;
                kvj[k] = t < active ? __ldg(Kj + col[t]) : 0.f;
            }
        }
        if (warp == 0) {                                         // analytic 2-variable update, once per CTA
            const bool yi = (pi & F_YPOS) != 0, yj = (pj & F_YPOS) != 0;
            const double Ci = yi ? Pp->C : Pp->Cn, Cj = yj ? Pp->C : Pp->Cn;   // per-class C (class_weight, svm.cpp:1393-1396 get_C)
            const double Gi = yi ? -gmax : gmax;                 // G = -y m (exact)
            const double Gj = yj ? -mg_j : mg_j;
            const double QDi = QD(i), QDj = QD(j);
            const double Qij = (yi == yj) ? k_ij : -k_ij;        // signed Q_i[j]
            double ai = alpha_i, aj = alpha_j;
            if (yi != yj) {                                      // svm.cpp:772-815
                double quad = __dadd_rn(__dadd_rn(QDi, QDj), __dmul_rn(2.0, Qij));
                if (quad <= 0) quad = TAU;
                const double delta = __ddiv_rn(__dsub_rn(-Gi, Gj), quad);
                const double diff = __dsub_rn(ai, aj);
                ai = __dadd_rn(ai, delta); aj = __dadd_rn(aj, delta);
                if (diff > 0) { if (aj < 0) { aj = 0; ai = diff; } }
                else          { if (ai < 0) { ai = 0; aj = -diff; } }
                if (diff > __dsub_rn(Ci, Cj)) { if (ai > Ci) { ai = Ci; aj = __dsub_rn(Ci, diff); } }
                else                          { if (aj > Cj) { aj = Cj; ai = __dadd_rn(Cj, diff); } }
            } else {                                             // svm.cpp:816-862
                double quad = __dsub_rn(__dadd_rn(QDi, QDj), __dmul_rn(2.0, Qij));
                if (quad <= 0) quad = TAU;
                const double delta = __ddiv_rn(__dsub_rn(Gi, Gj), quad);
                const double sum = __dadd_rn(ai, aj);
                ai = __dsub_rn(ai, delta); aj = __dadd_rn(aj, delta);
                if (sum > Ci) { if (ai > Ci) { ai = Ci; aj = __dsub_rn(sum, Ci); } }
                else         { if (aj < 0) { aj = 0; ai = sum; } }
                if (sum > Cj) { if (aj > Cj) { aj = Cj; ai = __dsub_rn(sum, Cj); } }
                else         { if (ai < 0) { ai = 0; aj = sum; } }
            }
            if (lane == 0) {
                const double dai = __dsub_rn(ai, alpha_i), daj = __dsub_rn(aj, alpha_j);
                red.bc_d[0] = yi ? -dai : dai;                   // a = -y_i dalpha_i
                red.bc_d[1] = yj ? -daj : daj;                   // b = -y_j dalpha_j
                red.bc_d[2] = ai; red.bc_d[3] = aj;
                red.bc_i[0] = ai >= Ci ? ST_UPPER : (ai <= 0 ? ST_LOWER : ST_FREE);
                red.bc_i[1] = aj >= Cj ? ST_UPPER : (aj <= 0 ? ST_LOWER : ST_FREE);
            }
        }
        tick(4);
        __syncthreads();                                                          // barrier 3
        tick(1);
        if constexpr (ROWBUF) {
            wait_row();
#pragma unroll
            for (int k = 0; k < KPT; k++) {
                const int t = k * NT + tid;
                kvj[k] = t < active ? rowbuf[col[t]] : 0.f;
            }
        }
        const double a = red.bc_d[0], b = red.bc_d[1];
        const int sti = red.bc_i[0], stj = red.bc_i[1];
        // the owners of i and j publish alpha and status FIRST: the fused scan below must see the new sets
        if (tid == i % NT) { alpha[i] = red.bc_d[2]; fl[i] = (unsigned char)mkflags((pi & F_YPOS) != 0, sti); }
        if (tid == j % NT) { alpha[j] = red.bc_d[3]; fl[j] = (unsigned char)mkflags((pj & F_YPOS) != 0, stj); }

        // m update over the active set (svm.cpp:866-872), fused with the next iteration's local scan
        la = -CUDART_INF; lm = CUDART_INF; la_idx = -1;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int t = k * NT + tid;
            if (t < active) {
                const double m = __dadd_rn(mG[t], __dadd_rn(__dmul_rn(widen(kvi[k]), a), __dmul_rn(widen(kvj[k]), b)));
                mG[t] = m;
                const int f = fl[t];
                if ((f & F_UP) && m >= la) { la = m; la_idx = (t << IDX_SHIFT) | f; }
                if (f & F_LOW) lm = fmin(lm, m);
            }
        }
        scan_valid = true;
        // G_bar over all l when a bound status flips (svm.cpp:876-905): i first, then j
        const bool need_i = use_gbar && (((pi & 3) == ST_UPPER) != (sti == ST_UPPER));
        const bool need_j = use_gbar && (((pj & 3) == ST_UPPER) != (stj == ST_UPPER));
        if (need_i || need_j) {
            // Gbar -= C Q_i (was upper) / += C Q_i (became upper)  <=>  mbar += fl(c K_i), c = +/- y_i C
            const double Cmi = (pi & F_YPOS) ? Pp->C : Pp->Cn, Cmj = (pj & F_YPOS) ? Pp->C : Pp->Cn;
            const float *__restrict__ Ki = K + (size_t)col[i] * ldk;
            const double ci = (((pi & 3) == ST_UPPER) == ((pi & F_YPOS) != 0)) ? Cmi : -Cmi;
            const double cj = (((pj & 3) == ST_UPPER) == ((pj & F_YPOS) != 0)) ? Cmj : -Cmj;
#pragma unroll
            for (int k = 0; k < KPT; k++) {
                const int t = k * NT + tid;
                if (t < l) {
                    const bool act = t < active;
                    double gb = mGbar[t];
                    if (need_i) gb = __dadd_rn(gb, __dmul_rn(ci, widen(act ? kvi[k] : __ldg(Ki + col[t]))));
                    if (need_j) gb = __dadd_rn(gb, __dmul_rn(cj, widen(act ? kvj[k] : __ldg(Kj + col[t]))));
                    mGbar[t] = gb;
                }
            }
        }
        tick(5);
    }

    // ---------------- calculate_rho (svm.cpp:1131-1168): sequential float64 sum in libsvm's order ----
    __syncthreads();
    const double C = Pp->C, Cng = Pp->Cn;
    if (tid == 0) {
        int nfree = 0;
        double ub = CUDART_INF, lb = -CUDART_INF, sum = 0;
        for (int t = 0; t < active; t++) {
            const int f = fl[t];
            const double yG = -mG[t];                            // y_t G_t
            if ((f & 3) == ST_UPPER) { if (!(f & F_YPOS)) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
            else if ((f & 3) == ST_LOWER) { if (f & F_YPOS) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
            else { ++nfree; sum = __dadd_rn(sum, yG); }
        }
        *Pp->out_rho = nfree > 0 ? __ddiv_rn(sum, (double)nfree) : __ddiv_rn(__dadd_rn(ub, lb), 2.0);
    }
    // coefficients alpha_k*y_k scattered by dataset row (svm.cpp:922-925, :1641-1642); SV counts
    int nsv = 0, nbsv = 0;
    {
        double *__restrict__ coef = Pp->coef;
        for (int t = tid; t < l; t += NT) {
            const double av = alpha[t];
            coef[col[t]] = (fl[t] & F_YPOS) ? av : -av;
            nsv += av > 0;
            nbsv += av >= ((fl[t] & F_YPOS) ? C : Cng);
        }
    }
#pragma unroll
    for (int m = 16; m; m >>= 1) {
        nsv += __shfl_xor_sync(0xffffffffu, nsv, m);
        nbsv += __shfl_xor_sync(0xffffffffu, nbsv, m);
    }
    if (lane == 0) { red.cnt[warp] = nsv; red.a_idx[warp] = nbsv; }
    __syncthreads();
    if (tid == 0) {
        int s = 0, bs = 0;
        for (int w = 0; w < NW; w++) { s += red.cnt[w]; bs += red.a_idx[w]; }
        int *info = Pp->out_info;
        info[0] = iter; info[1] = timed_out; info[2] = s; info[3] = bs;
        unsigned long long t_end;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
        unsigned long long *ns = Pp->out_ns;
        ns[0] = t_start; ns[1] = t_end;
        if constexpr (PROF)
            for (int q = 0; q < 6; q++) ns[2 + q] = (unsigned long long)prof[q];
    }
}

template <int NT, int KPT, bool SMEM_STATE, bool FAST, bool PROF, bool ROWBUF>
cudaError_t launch_one(const SmoProblem *probs, const int *order, int n_prob, int rowcap, cudaStream_t st)
{
    constexpr int LCAP = NT * KPT;
    const size_t smem = ROWBUF ? (size_t)LCAP * (8 + 8 + 2 + 1) + 128 + (size_t)rowcap * 4
                               : (size_t)LCAP * (SMEM_STATE ? (8 + 8 + 8 + 2 + 1) : (8 + 2 + 1));
    auto kern = smo_kernel<NT, KPT, SMEM_STATE, FAST, PROF, ROWBUF>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<n_prob, NT, smem, st>>>(probs, order, rowcap);
    return cudaGetLastError();
}

template <int NT, int KPT, bool SMEM_STATE, bool ROWBUF = false>
cudaError_t launch_cfg(const SmoProblem *probs, const int *order, int n_prob, bool fast, bool prof, int rowcap, cudaStream_t st)
{
    if (prof) return fast ? launch_one<NT, KPT, SMEM_STATE, true, true, ROWBUF>(probs, order, n_prob, rowcap, st)
                          : launch_one<NT, KPT, SMEM_STATE, false, true, ROWBUF>(probs, order, n_prob, rowcap, st);
    return fast ? launch_one<NT, KPT, SMEM_STATE, true, false, ROWBUF>(probs, order, n_prob, rowcap, st)
                : launch_one<NT, KPT, SMEM_STATE, false, false, ROWBUF>(probs, order, n_prob, rowcap, st);
}

int env_int(const char *name, int dflt)
{
    const char *v = getenv(name);
    return v && *v ? atoi(v) : dflt;
}

}  // namespace

int smo_max_rows() { return 1024 * 16; }

// fast: every problem is rbf and every kernel matrix of the launch holds only positive normal floats
// rowcap: row length of the K matrices in floats (ldk); enables the bulk-copy row path when the row fits in shared memory
cudaError_t launch_smo(const SmoProblem *d_probs, const int *d_order, int n_prob, int lmax, bool fast, int rowcap, cudaStream_t st,
                       std::string *why)
{
    if (n_prob <= 0) return cudaSuccess;
    const bool prof = env_int("B200GS_SMO_PROF", 0) != 0;          // development switch: per-phase cycle counters
    if (env_int("B200GS_SMO_NOFAST", 0)) fast = false;
    if (lmax <= 512) return launch_cfg<128, 4, true>(d_probs, d_order, n_prob, fast, prof, 0, st);
    if (lmax <= 2048) return launch_cfg<256, 8, true>(d_probs, d_order, n_prob, fast, prof, 0, st);
    if (lmax <= 4096) return launch_cfg<512, 8, true>(d_probs, d_order, n_prob, fast, prof, 0, st);
    if (lmax <= 8192) {
        // 8192 rows of state without G_bar = 152 KB; the row buffer may use what is left of the 227 KB
        const bool rowbuf_fits = (size_t)8192 * 19 + 128 + (size_t)rowcap * 4 + 4096 <= 227 * 1024;
        if (rowbuf_fits && env_int("B200GS_SMO_ROWBUF", 1))
            return launch_cfg<1024, 8, true, true>(d_probs, d_order, n_prob, fast, prof, rowcap, st);
        return launch_cfg<1024, 8, true>(d_probs, d_order, n_prob, fast, prof, 0, st);
    }
    if (lmax <= 16384) return launch_cfg<1024, 16, false>(d_probs, d_order, n_prob, fast, prof, 0, st);
    if (why) *why = "SVC sub-problem larger than 16384 rows is not supported by the resident-state SMO kernel";
    return cudaErrorInvalidValue;
}
