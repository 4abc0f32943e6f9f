// smo_lean.cu -- batched C-SVC dual solver, throughput instance: one CTA per (candidate, fold, class-pair) sub-problem,
// TWO (or more) resident sub-problems per SM.
//
// Same algorithm and the same bit-exact iterate sequence as smo.cu (libsvm svm.cpp:629-1168 restated there; the m-domain,
// the approximate WSS2 filter with its exact tie-break and the REDUX arg-reductions are described in that file).  What
// differs is the data layout, chosen so that an SM never idles on one sub-problem's row fetch:
//
//   * SLOTS.  A sub-problem's training rows are <= 4 runs of columns of the (class-sorted) kernel matrix (api.cu:
//     SmoProblem::seg_*), each starting and ending on a multiple of 4 columns.  The runs are laid end to end into a slot
//     space; slot s <-> one fixed column for the whole solve (columns inside a run that are not training rows -- test-fold
//     rows inside a merged gap -- are inert slots).  Thread t owns the 4 consecutive slots of groups g*NT + t, g = 0..3:
//     a K row is read with FOUR coalesced, 16-byte-aligned LDG.128 per thread straight into registers -- no column
//     indirection, no staging buffer, no mbarrier.
//   * libsvm's positions (shrinking permutes them, and every tie-break is defined on them) are STATE, as in
//     smo_colown.cu: a 32-bit word per slot holds  position << 18 | slot << 4 | status | I_up | I_low.  Arg-reductions
//     compare (value, word); the winner's word carries its slot.  Elements outside the active set have I_up/I_low
//     cleared, so the hot loops need no active-set test; their m is updated along with the rest and overwritten by
//     reconstruct_gradient exactly as libsvm overwrites G (svm.cpp:633-636).
//   * Resident state per sub-problem: m (8 B) and the word (4 B) per slot in shared memory = 96 KB for 8192 slots; alpha
//     and G_bar (touched by two elements per iteration / on status flips) in global memory.  512 threads x 64 registers:
//     two sub-problems per SM, so one's row latency and barriers overlap the other's arithmetic.
//     m is stored in two planes (elements 0-1 and 2-3 of every group) so that a warp's 16-byte accesses are consecutive:
//     no bank conflicts (a plain [slot] array of doubles makes every LDS.128 / STS.128 a 2-way conflict, measured as the
//     limiter of both element loops).  The I_up / I_low bits of a thread's own slots are mirrored in ONE register
//     (2 bits per slot); the hot loops read no slot words -- only the winner's word is fetched after the loop.
//   * alpha_j and Q_ij travel with the warp records: each warp's phase-B winner lane loads its alpha before the barrier
//     (the latency hides in the barrier skew), so the two-variable update waits for no memory.
//   * The stopping test Gmax + Gmax2 < eps (svm.cpp:1040) is evaluated as "no I_low element has fl(Gmax - m_t) >= eps"
//     (rounding is monotone, so this is the same predicate) inside the j-selection loop and reduced by the barrier itself
//     (__syncthreads_or): the update loop carries one running arg-max instead of an arg-max and a min.
//     The float32 image of Gmax - m_t that the approximate WSS2 key needs anyway decides it: above / below fl32(eps) is
//     certain, exactly equal (one float in 2^23) is re-decided in float64.
//   * The running arg-max uses a strict compare and a tie flag; a thread whose flag is set re-scans its slots with the
//     full (value, position) order.  After the first iteration exact ties in m do not occur in practice.
//   * float32 -> float64 widening of a positive normal K entry is ONE integer multiply-add (u * 2^29 + 0x38 << 56).
#include "smo_common.cuh"
#include <algorithm>
#include <cstdlib>
#include <type_traits>

namespace {

using namespace smo;

constexpr unsigned LF_UP = 4u, LF_LOW = 8u;           // flag bits of the slot word (bits 0-1: status)
constexpr int POS_SHIFT = 18, SLOT_SHIFT = 4;
constexpr unsigned SLOT_MASK = 0x3fffu;
constexpr unsigned PF_INERT = 0xfffffff0u;            // position 0x3fff (never active), no flags

__device__ __forceinline__ unsigned lean_flags(bool ypos, int st)
{
    const bool up = ypos ? st != ST_UPPER : st != ST_LOWER;     // I_up  membership (svm.cpp:964-978)
    const bool low = ypos ? st != ST_LOWER : st != ST_UPPER;    // I_low membership (svm.cpp:986-1037)
    return (unsigned)st | (up ? LF_UP : 0u) | (low ? LF_LOW : 0u);
}

// compile-time unrolled loop: f(std::integral_constant<int, 0>) ... f(std::integral_constant<int, N - 1>)
template <int N, int I = 0, class F>
__device__ __forceinline__ void lean_loop(F &&f)
{
    if constexpr (I < N) { f(std::integral_constant<int, I>{}); lean_loop<N, I + 1>(f); }
}

struct UArg { unsigned hi, lo, idx; };
// warp arg-max over (64-bit key, word): largest key, ties -> largest word; word 0 = none.  3 REDUX.
__device__ __forceinline__ UArg warp_argmax_u(unsigned hi, unsigned lo, unsigned idx)
{
    UArg r;
    r.hi = __reduce_max_sync(0xffffffffu, idx ? hi : 0u);
    r.lo = __reduce_max_sync(0xffffffffu, (idx && hi == r.hi) ? lo : 0u);
    r.idx = __reduce_max_sync(0xffffffffu, (hi == r.hi && lo == r.lo) ? idx : 0u);
    return r;
}

// ---- per-slot bodies of the two hot loops, FAST instance (rbf, positive normal K), as straight PTX: the compiler's own
//      lowering of the same C++ kept the predicates in general registers and spilled (measured 20 instructions per slot and
//      loop); this is 17 and 13.  Rounding: every f64 operation carries .rn, which also forbids contraction.
// phase B: gd = Gmax - m; candidate iff I_low bit set and gd > 0; key = bits(fl32(gd)^2 * rcp(max(fl32(2 - 2K), 1e-12)))
template <int K>
__device__ __forceinline__ void lean_phase_b_slot(double gmax, double m, unsigned fm, float kv, unsigned &b1k, unsigned &b2k,
                                                  int &k1, float &kq1, float &gmxf)
{
    asm volatile("{\n\t"
                 ".reg .pred pc, pg;\n\t"
                 ".reg .f64 gd;\n\t"
                 ".reg .f32 gdf, qf, g2, r, ap;\n\t"
                 ".reg .b32 key, t;\n\t"
                 "sub.rn.f64 gd, %5, %6;\n\t"
                 "and.b32 t, %7, %8;\n\t"
                 "setp.ne.u32 pc, t, 0;\n\t"
                 "setp.gt.and.f64 pc, gd, 0d0000000000000000, pc;\n\t"
                 "cvt.rn.f32.f64 gdf, gd;\n\t"
                 "selp.f32 gdf, gdf, 0f00000000, pc;\n\t"
                 "max.f32 %4, %4, gdf;\n\t"
                 "fma.rn.f32 qf, %9, 0fC0000000, 0f40000000;\n\t"
                 "max.f32 qf, qf, 0f2B8CBCCC;\n\t"
                 "mul.rn.f32 g2, gdf, gdf;\n\t"
                 "rcp.approx.ftz.f32 r, qf;\n\t"
                 "mul.rn.f32 ap, g2, r;\n\t"
                 "mov.b32 key, ap;\n\t"
                 "setp.gt.u32 pg, key, %0;\n\t"
                 "min.u32 t, %0, key;\n\t"
                 "max.u32 %1, %1, t;\n\t"
                 "max.u32 %0, %0, key;\n\t"
                 "selp.b32 %2, %10, %2, pg;\n\t"
                 "selp.f32 %3, %9, %3, pg;\n\t"
                 "}"
                 : "+r"(b1k), "+r"(b2k), "+r"(k1), "+f"(kq1), "+f"(gmxf)
                 : "d"(gmax), "d"(m), "r"(fm), "n"(2u << (2 * K)), "f"(kv), "n"(K));
}
// update: m += fl(fl(K_i a) + fl(K_j b)); running arg-max over I_up with a strict compare, equal values raise `tie`
template <int K>
__device__ __forceinline__ void lean_update_slot(double &m, float kvi, float kvj, double a, double b, unsigned fm, double &la,
                                                 int &la_k, unsigned &tie)
{
    asm volatile("{\n\t"
                 ".reg .pred pu, pb, pe;\n\t"
                 ".reg .b64 wi, wj;\n\t"
                 ".reg .f64 fi, fj;\n\t"
                 ".reg .b32 t;\n\t"
                 "mad.wide.u32 wi, %4, 0x20000000, 0x3800000000000000;\n\t"
                 "mad.wide.u32 wj, %5, 0x20000000, 0x3800000000000000;\n\t"
                 "mov.b64 fi, wi;\n\t"
                 "mov.b64 fj, wj;\n\t"
                 "mul.rn.f64 fi, fi, %6;\n\t"
                 "mul.rn.f64 fj, fj, %7;\n\t"
                 "add.rn.f64 fi, fi, fj;\n\t"
                 "add.rn.f64 %0, %0, fi;\n\t"
                 "and.b32 t, %8, %9;\n\t"
                 "setp.ne.u32 pu, t, 0;\n\t"
                 "setp.gt.and.f64 pb, %0, %1, pu;\n\t"
                 "setp.eq.and.f64 pe, %0, %1, pu;\n\t"
                 "selp.f64 %1, %0, %1, pb;\n\t"
                 "selp.b32 %2, %10, %2, pb;\n\t"
                 "selp.b32 %3, 1, %3, pe;\n\t"
                 "}"
                 : "+d"(m), "+d"(la), "+r"(la_k), "+r"(tie)
                 : "r"(__float_as_uint(kvi)), "r"(__float_as_uint(kvj)), "d"(a), "d"(b), "r"(fm), "n"(1u << (2 * K)), "n"(K));
}

struct LeanRed {                                      // static shared scratch; NW <= 32 warps
    unsigned a_hi[32], a_lo[32], a_pf[32];            // phase A warp records (arg-max m over I_up)
    unsigned b_k1[32], b_pf[32], b_k2[32], b_fl[32];  // phase B warp records (approximate arg-max, stop-test bits)
    float b_kq[32]; double b_al[32], b_mg[32];        // ... the warp winner's K_i value, alpha and m
    double al_i;                                      // alpha_i (published by warp 0 before barrier 2)
    double bc_d[4]; int bc_i[2];                      // shared-SM instance: the two-variable update broadcast by warp 0
    unsigned x_hi[32], x_lo[32], x_pf[32];            // exact tie-break records (rare path)
    float x_kq[32]; double x_al[32], x_mg[32];
    double dm[32], dm2[32]; int cnt[32];              // cold-path reductions
    int seg_slot[5], seg_col[4];                      // slot -> column map
    int ysplit;                                       // first slot of the -1 class
};

// NT threads, G groups of 4 consecutive slots per thread: NT * G * 4 slots, NT * G * 48 bytes of shared memory
// SOLO: the sub-problem has its SM to itself (exclusive tier, or fewer problems than SMs): every warp evaluates the two-variable
// update (no third barrier: latency).  Otherwise two sub-problems share the SM and issue slots are the scarce resource: warp 0
// evaluates it once and the others wait at a third barrier, which the co-resident CTA fills.
template <int NT, int G, bool FAST, bool PROF, bool SOLO>
__global__ void __launch_bounds__(NT, (NT * G >= 4096 || NT >= 1024 ? 1 : 2048 / (NT * G / 2) > 8 ? 8 : 2048 / (NT * G / 2)))
smo_lean_kernel(const SmoProblem *__restrict__ probs, const int *__restrict__ order)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ LeanRed red;
    constexpr int NW = NT / 32;
    constexpr int KPT = G * 4;
    constexpr int LCAP = NT * KPT;

    const SmoProblem *__restrict__ Pp = probs + order[blockIdx.x];
    if (Pp->guard != nullptr && (*Pp->guard != 0) == FAST) return;       // the other instance solves this launch (common.cuh)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int l = Pp->l;
    const int nslots = Pp->nslots;
    double *const mG = reinterpret_cast<double *>(smem_raw);                // m = -y*G by slot
    unsigned *const pfS = reinterpret_cast<unsigned *>(mG + LCAP);          // slot word by slot
    double *const alpha_g = Pp->alpha;                                       // by slot (global)
    double *const gbar_g = Pp->Gbar;                                         // mbar = -y*G_bar by slot (global)
    int *const scratch = Pp->scratch;                                        // >= 2*l + 64 ints (global)
    const float *__restrict__ const K = Pp->K;
    const int64_t ldk = Pp->ldk;
    const double eps = Pp->eps;
    const double Cc = Pp->C, Cneg = Pp->Cn;                                   // C of the +1 / -1 class
    const bool use_gbar = Pp->shrinking != 0;
    const double *__restrict__ const qd = FAST ? nullptr : Pp->qd;

    unsigned long long t_start = 0;
    if (tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));

    // ---- slot -> column map ----
    if (tid == 0) {
        int s = 0;
        for (int e = 0; e < 4; e++) {
            red.seg_slot[e] = e < Pp->nseg ? s : 0x7fffffff;
            red.seg_col[e] = e < Pp->nseg ? Pp->seg_start[e] : 0;
            if (e < Pp->nseg) s += Pp->seg_len[e];
        }
        red.seg_slot[4] = 0x7fffffff;
    }
    __syncthreads();
    auto slot_col = [&](int slot) -> int {
        const int e = (slot >= red.seg_slot[1]) + (slot >= red.seg_slot[2]) + (slot >= red.seg_slot[3]);
        return red.seg_col[e] + (slot - red.seg_slot[e]);
    };
    int gcol[G];                                                             // column of the first slot of each owned group
#pragma unroll
    for (int g = 0; g < G; g++) {
        const int s4 = (g * NT + tid) * 4;
        gcol[g] = s4 < nslots ? slot_col(s4) : 0;                            // groups past the last slot read column 0 (valid memory)
    }

    // m of slot s lives at plane (s & 2), group s >> 2, element s & 1: a thread's group is two 16-byte pieces LCAP/2 doubles apart
    auto m_at = [&](int slot) -> double & { return mG[((slot >> 1) & 1) * (LCAP / 2) + (slot >> 2) * 2 + (slot & 1)]; };
    auto load_m4 = [&](int s4, double (&mv)[4]) {
        const double2 a = *reinterpret_cast<const double2 *>(mG + (s4 >> 1)), b = *reinterpret_cast<const double2 *>(mG + LCAP / 2 + (s4 >> 1));
        mv[0] = a.x; mv[1] = a.y; mv[2] = b.x; mv[3] = b.y;
    };
    auto store_m4 = [&](int s4, const double (&mv)[4]) {
        *reinterpret_cast<double2 *>(mG + (s4 >> 1)) = make_double2(mv[0], mv[1]);
        *reinterpret_cast<double2 *>(mG + LCAP / 2 + (s4 >> 1)) = make_double2(mv[2], mv[3]);
    };
    auto load_pf4 = [&](int s4, unsigned (&pv)[4]) {
        const uint4 p = *reinterpret_cast<const uint4 *>(pfS + s4);
        pv[0] = p.x; pv[1] = p.y; pv[2] = p.z; pv[3] = p.w;
    };

    // ---- initial point: alpha = 0, G = p = -1  =>  m = y (svm.cpp:1611-1626, :716-736) ----
    {
        const int n_pos = Pp->n_pos;
        const int *__restrict__ rows = Pp->rows;                            // ascending (class a rows, then class b rows)
        int ysp = 0x7fffffff;
#pragma unroll
        for (int g = 0; g < G; g++) {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const int s = (g * NT + tid) * 4 + q;
                unsigned w = PF_INERT;
                double mv = 0.0;
                if (s < nslots) {
                    const int c = gcol[g] + q;
                    int lo = 0, hi = l;                                      // first position with rows[p] >= c
                    while (lo < hi) { const int mid = (lo + hi) >> 1; if (rows[mid] < c) lo = mid + 1; else hi = mid; }
                    if (lo < l && rows[lo] == c) {
                        const bool yp = lo < n_pos;
                        w = ((unsigned)lo << POS_SHIFT) | ((unsigned)s << SLOT_SHIFT) | lean_flags(yp, ST_LOWER);
                        mv = yp ? 1.0 : -1.0;
                        if (lo == n_pos) ysp = s;
                    }
                    alpha_g[s] = 0.0;
                    if (use_gbar) gbar_g[s] = 0.0;
                }
                m_at(s) = mv; pfS[s] = w;
            }
        }
        if (ysp != 0x7fffffff) red.ysplit = ysp;                             // exactly one slot holds position n_pos
    }
    __syncthreads();
    const int ysplit = red.ysplit;

    int active = l, iter = 0, timed_out = 0;
    int counter = (l < 1000 ? l : 1000) + 1;
    bool unshrink = false;
    const int max_iter = Pp->max_iter == -1 ? SAFETY_MAX_ITER : Pp->max_iter;

    long long prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long tprev = PROF ? clock64() : 0;
    auto tick = [&](int slot) {
        if constexpr (PROF) {
            const long long now = clock64();
            prof[slot] += now - tprev;
            tprev = now;
        }
    };

    auto QDc = [&](int c) -> double {                                        // by column (svm.cpp:1436-1437)
        if constexpr (FAST) return 1.0;
        else return qd ? qd[c] : 1.0;
    };
    auto widen = [&](float x) -> double {
        if constexpr (FAST) {                                                // positive normal float: one IMAD.WIDE
            const unsigned long long r = (unsigned long long)__float_as_uint(x) * 0x20000000ull + 0x3800000000000000ull;
            return __longlong_as_double((long long)r);
        } else return f2d(x);
    };
    // one K row at this thread's 16 slots: four coalesced 16-byte loads, L1 left to alpha / G_bar
    auto load_row = [&](int col, float (&kv)[KPT]) {
        const float *__restrict__ Kr = K + (size_t)col * ldk;
#pragma unroll
        for (int g = 0; g < G; g++) {
            float4 v;
            asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                         : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(Kr + gcol[g]));
            kv[g * 4 + 0] = v.x; kv[g * 4 + 1] = v.y; kv[g * 4 + 2] = v.z; kv[g * 4 + 3] = v.w;
        }
    };

    // ---------------- local scan (normally fused into the update loop) ----------------
    // la / la_pf: arg-max of m over the owned I_up slots, ties -> larger position (libsvm's ascending ">=" scan)
    double la = -CUDART_INF;
    unsigned la_pf = 0u;
    unsigned fm = 0u;                   // I_up (bit 2k) and I_low (bit 2k+1) of the owned slot k = g*4 + q
    static_assert(G <= 4, "the flag mask holds 16 slots");
    auto slot_of = [&](int k) -> int { return ((k >> 2) * NT + tid) * 4 + (k & 3); };
    auto scan_exact = [&](double mv, unsigned w) {
        const bool better = ((w & LF_UP) != 0u) & ((mv > la) | ((mv == la) & (w > la_pf)));
        la = better ? mv : la;
        la_pf = better ? w : la_pf;
    };
    auto local_scan = [&]() {
        la = -CUDART_INF; la_pf = 0u;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const int s4 = (g * NT + tid) * 4;
            double mv[4]; unsigned pv[4];
            load_m4(s4, mv); load_pf4(s4, pv);
#pragma unroll
            for (int q = 0; q < 4; q++) scan_exact(mv[q], pv[q]);
        }
    };
    // I_up / I_low bits follow the active set: cleared for positions >= active, recomputed from status and label below it
    auto refresh_flags = [&]() {
        const unsigned act_lim = (unsigned)active << POS_SHIFT;
        fm = 0u;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const int s4 = (g * NT + tid) * 4;
            unsigned pv[4];
            load_pf4(s4, pv);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const unsigned w = pv[q];
                if (w < PF_INERT) {
                    const unsigned base = w & ~(LF_UP | LF_LOW);
                    pv[q] = w < act_lim ? (base & ~3u) | lean_flags(s4 + q < ysplit, (int)(w & 3u)) : base;
                }
                fm |= ((pv[q] >> 2) & 3u) << (2 * (g * 4 + q));
            }
            *reinterpret_cast<uint4 *>(pfS + s4) = make_uint4(pv[0], pv[1], pv[2], pv[3]);
        }
    };

    // ---------------- reconstruct_gradient (svm.cpp:629-668), m-domain ----------------
    // m_k = (mbar_k + y_k) + sum over free active f in ASCENDING POSITION of fl((-y_f alpha_f) K_fk), for inactive k
    auto rebuild_gradient = [&]() {
        if (active == l) return;
        const unsigned act_lim = (unsigned)active << POS_SHIFT;
        int *const slot_by_pos = scratch, *const lists = scratch + l;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const int s4 = (g * NT + tid) * 4;
            unsigned pv[4];
            load_pf4(s4, pv);
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (pv[q] < act_lim) slot_by_pos[pv[q] >> POS_SHIFT] = (pv[q] & 3u) == ST_FREE ? s4 + q : -1;
        }
        __syncthreads();
        int nf = 0;
        for (int base = 0; base < active; base += NT) {
            const int t = base + tid;
            const int sl = t < active ? __ldcg(slot_by_pos + t) : -1;
            int tot;
            const int r = block_rank<NT>(sl >= 0, red.cnt, tot);
            if (sl >= 0) lists[nf + r] = sl;
            nf += tot;
        }
        __syncthreads();
        // one group of 4 owned slots at a time (keeps the accumulators in registers); each element still adds its
        // terms in ascending position of f
#pragma unroll 1
        for (int g = 0; g < G; g++) {
            const int s4 = (g * NT + tid) * 4;
            unsigned pv[4];
            load_pf4(s4, pv);
            bool in[4];
            double gacc[4];
            bool any = false;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                in[q] = pv[q] >= act_lim && pv[q] < PF_INERT;
                any = any || in[q];
                gacc[q] = in[q] ? __dadd_rn(__ldcg(gbar_g + s4 + q), s4 + q < ysplit ? 1.0 : -1.0) : 0.0;
            }
            if (!any) continue;
            const int gc = gcol[g];
#pragma unroll 4
            for (int r = 0; r < nf; r++) {
                const int fs = __ldcg(lists + r);
                const double av = __ldcg(alpha_g + fs);
                const double af = fs < ysplit ? -av : av;                    // -y_f alpha_f
                const float4 v = __ldg(reinterpret_cast<const float4 *>(K + (size_t)slot_col(fs) * ldk + gc));
                const float kv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int q = 0; q < 4; q++)
                    if (in[q]) gacc[q] = __dadd_rn(gacc[q], __dmul_rn(af, widen(kv[q])));
            }
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (in[q]) m_at(s4 + q) = gacc[q];
        }
        __syncthreads();
    };

    // ---------------- select_working_set (svm.cpp:946-1047) ----------------
    unsigned pi = 0u, pj = 0u;           // slot words of i and j
    int col_i = 0, col_j = 0;
    double gmax = 0, mg_j = 0, k_ij = 0, alpha_i = 0, alpha_j = 0;
    float kvi[KPT];                      // K_i row at the owned slots (float32 as stored), alive until the update loop
    auto select = [&]() -> bool {
        // ---- phase A: i = argmax m_t over I_up (from the local scan) ----
        {
            const unsigned long long key = dkey(la);
            const UArg w = warp_argmax_u((unsigned)(key >> 32), (unsigned)key, la_pf);
            if (lane == 0) { red.a_hi[warp] = w.hi; red.a_lo[warp] = w.lo; red.a_pf[warp] = w.idx; }
            tick(0);
            __syncthreads();                                                      // barrier 1
            tick(1);
            const bool v = lane < NW;
            const UArg a = warp_argmax_u(v ? red.a_hi[lane] : 0u, v ? red.a_lo[lane] : 0u, v ? red.a_pf[lane] : 0u);
            pi = a.idx;
            gmax = dkey_inv(((unsigned long long)a.hi << 32) | a.lo);
        }
        if (pi == 0u) return true;                                                // I_up empty
        const int slot_i = (int)((pi >> SLOT_SHIFT) & SLOT_MASK);
        col_i = slot_col(slot_i);
        load_row(col_i, kvi);
        if (tid == 0) red.al_i = __ldcg(alpha_g + slot_i);                         // read by every warp after barrier 2
        const double QDi = QDc(col_i);
        // ---- phase B: j = argmin -(gd^2)/quad over I_low with gd > 0 (svm.cpp:980-1037); error analysis of the approximate
        //      key and of BAND: smo.cu.  A slot that is no candidate gets gd := 0 and with it key 0 (FAST) / is masked.
        constexpr unsigned BAND = FAST ? 64u : 514u;
        constexpr unsigned KEY_TINY = 0x0D800000u;                          // float bits of 2^-100
        const float epsf = __double2float_rn(eps);
        auto approx_key = [&](double gd, float gdf, float kvf, int c) -> unsigned {
            if constexpr (FAST) {
                const float quadf = fmaxf(__fmaf_rn(-2.f, kvf, 2.f), 1e-12f);       // fl32(2 - 2K) >= 2^-23 unless K == 1
                const float g2f = __fmul_rn(gdf, gdf);
                float r;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(quadf));
                return __float_as_uint(__fmul_rn(g2f, r));
            } else {
                const double quad = __dsub_rn(__dadd_rn(QDi, QDc(c)), __dmul_rn(2.0, widen(kvf)));
                const double g2 = __dmul_rn(gd, gd);
                const double ap = quad > 0 ? g2 * rcp_approx(quad) : g2 * 1e12;
                return (unsigned)__double2hiint(ap);
            }
        };
        unsigned b1k = 0u, b2k = 0u;                    // best / second-best key
        int k1 = 0;                                     // the best candidate's local slot number ...
        float kq1 = 0.f;                                // ... and its K_i value
        float gmxf = 0.f;                               // max over the candidates of fl32(Gmax - m_t)
        double mvb[4];
        if constexpr (FAST) {
            lean_loop<G * 4>([&](auto kc) {
                constexpr int k = decltype(kc)::value, g = k >> 2, q = k & 3;
                if constexpr (q == 0) load_m4((g * NT + tid) * 4, mvb);
                lean_phase_b_slot<k>(gmax, mvb[q], fm, kvi[k], b1k, b2k, k1, kq1, gmxf);
            });
        } else {
#pragma unroll
            for (int g = 0; g < G; g++) {
                const int s4 = (g * NT + tid) * 4;
                double mv[4];
                load_m4(s4, mv);
#pragma unroll
                for (int q = 0; q < 4; q++) {                                // branch-free: every slot evaluates a key
                    const int k = g * 4 + q;
                    const double gd = __dsub_rn(gmax, mv[q]);
                    const bool cand = ((fm & (2u << (2 * k))) != 0u) & (gd > 0);
                    const float gdf = cand ? __double2float_rn(gd) : 0.f;
                    gmxf = fmaxf(gmxf, gdf);
                    const unsigned key = cand ? approx_key(gd, gdf, kvi[k], gcol[g] + q) : 0u;
                    const bool gt = key > b1k;
                    b2k = max(b2k, min(b1k, key));
                    b1k = max(b1k, key);
                    k1 = gt ? k : k1;
                    kq1 = gt ? kvi[k] : kq1;
                }
            }
        }
        const unsigned idx1 = b1k ? pfS[slot_of(k1)] : 0u;                   // the best candidate's word
        unsigned top1k, top2k;
        {
            const unsigned w1 = __reduce_max_sync(0xffffffffu, b1k);
            const unsigned widx = __reduce_max_sync(0xffffffffu, (b1k == w1) ? idx1 : 0u);
            const unsigned w2 = __reduce_max_sync(0xffffffffu, (idx1 == widx) ? b2k : b1k);
            if (idx1 == widx && widx != 0u) {                                         // this lane owns the warp's winner
                red.b_kq[warp] = kq1;
                red.b_al[warp] = __ldcg(alpha_g + slot_of(k1));
                red.b_mg[warp] = m_at(slot_of(k1));
            }
            // stop-test bits: 1 = some candidate certainly has Gmax - m_t >= eps, 2 = undecided in float32, 4 = a candidate exists
            const unsigned fb = __reduce_or_sync(0xffffffffu, (gmxf > epsf ? 1u : 0u) | (gmxf == epsf ? 2u : 0u) | (gmxf > 0.f ? 4u : 0u));
            if (lane == 0) { red.b_k1[warp] = w1; red.b_pf[warp] = widx; red.b_k2[warp] = w2; red.b_fl[warp] = fb; }
            tick(2);
            __syncthreads();                                                          // barrier 2
            tick(3);
            const bool v = lane < NW;
            const unsigned bk = v ? red.b_k1[lane] : 0u;
            const unsigned bi = v ? red.b_pf[lane] : 0u;
            const unsigned fl = __reduce_or_sync(0xffffffffu, v ? red.b_fl[lane] : 0u);
            top1k = __reduce_max_sync(0xffffffffu, bk);
            pj = __reduce_max_sync(0xffffffffu, (bk == top1k) ? bi : 0u);
            top2k = __reduce_max_sync(0xffffffffu, (v && bi == pj) ? red.b_k2[lane] : bk);
            {
                const int wl = __ffs(__ballot_sync(0xffffffffu, v && bi == pj && pj != 0u)) - 1;
                if (wl >= 0) { k_ij = widen(red.b_kq[wl]); alpha_j = red.b_al[wl]; mg_j = red.b_mg[wl]; }
            }
            if (!(fl & 4u)) return true;                                              // no candidate: Gmin_idx == -1 (and Gmax + Gmax2 <= 0)
            if (!(fl & 1u)) {
                if (!(fl & 2u)) return true;                                          // every Gmax - m_t < eps: svm.cpp:1040-1041
                bool viol = false;                                                    // re-decide in float64 (rare)
#pragma unroll
                for (int g = 0; g < G; g++) {
                    const int s4 = (g * NT + tid) * 4;
                    double mv[4];
                    load_m4(s4, mv);
#pragma unroll
                    for (int q = 0; q < 4; q++) viol = viol | (((fm & (2u << (2 * (g * 4 + q)))) != 0u) & (__dsub_rn(gmax, mv[q]) >= eps));
                }
                if (!__syncthreads_or(viol ? 1 : 0)) return true;
            }
        }
        if (top1k - top2k <= BAND || top1k <= KEY_TINY) {
            // ---- exact tie-break: libsvm's correctly rounded quotients for every element in the band (rare) ----
            if constexpr (PROF) prof[7] += 1;                                     // how often: reported as slot 7
            const unsigned thrk = (top1k > BAND && top1k > KEY_TINY) ? top1k - BAND : 0u;
            double bestn = -CUDART_INF;
            unsigned bidx = 0u;
            float kqb = 0.f;
#pragma unroll
            for (int g = 0; g < G; g++) {
                const int s4 = (g * NT + tid) * 4;
                double mv[4]; unsigned pv[4];
                load_m4(s4, mv); load_pf4(s4, pv);
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const double gd = __dsub_rn(gmax, mv[q]);
                    if ((pv[q] & LF_LOW) && gd > 0) {
                        if (approx_key(gd, __double2float_rn(gd), kvi[g * 4 + q], gcol[g] + q) >= thrk) {
                            const double quad = __dsub_rn(__dadd_rn(QDi, QDc(gcol[g] + q)), __dmul_rn(2.0, widen(kvi[g * 4 + q])));
                            const double g2 = __dmul_rn(gd, gd);
                            const double nod = quad > 0 ? __ddiv_rn(g2, quad) : __ddiv_rn(g2, TAU);   // == -obj_diff
                            if (nod > bestn || (nod == bestn && pv[q] > bidx)) { bestn = nod; bidx = pv[q]; kqb = kvi[g * 4 + q]; }
                        }
                    }
                }
            }
            const unsigned long long key = dkey(bestn);
            const UArg w = warp_argmax_u((unsigned)(key >> 32), (unsigned)key, bidx);
            if (bidx == w.idx && w.idx != 0u) {
                red.x_kq[warp] = kqb;
                red.x_al[warp] = __ldcg(alpha_g + (int)((bidx >> SLOT_SHIFT) & SLOT_MASK));
                red.x_mg[warp] = m_at((int)((bidx >> SLOT_SHIFT) & SLOT_MASK));
            }
            if (lane == 0) { red.x_hi[warp] = w.hi; red.x_lo[warp] = w.lo; red.x_pf[warp] = w.idx; }
            __syncthreads();                                                      // rare barrier
            const bool v = lane < NW;
            const unsigned xi = v ? red.x_pf[lane] : 0u;
            const UArg b = warp_argmax_u(v ? red.x_hi[lane] : 0u, v ? red.x_lo[lane] : 0u, xi);
            pj = b.idx;                                                           // != 0: every candidate with a key >= thrk took part
            const int wl = __ffs(__ballot_sync(0xffffffffu, v && xi == pj)) - 1;
            k_ij = widen(red.x_kq[wl]); alpha_j = red.x_al[wl]; mg_j = red.x_mg[wl];
        }
        const int slot_j = (int)((pj >> SLOT_SHIFT) & SLOT_MASK);
        col_j = slot_col(slot_j);
        alpha_i = red.al_i;
        return false;
    };

    // ---------------- do_shrinking (svm.cpp:1070-1129), m-domain ----------------
    // Gmax1 = max{m : I_up}, Gmax2 = max{-m : I_low}; be_shrunk = (!up && m > Gmax1) || (!low && -m > Gmax2)
    auto do_shrink = [&]() {
        double g1 = -CUDART_INF, g2 = -CUDART_INF;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const int s4 = (g * NT + tid) * 4;
            double mv[4]; unsigned pv[4];
            load_m4(s4, mv); load_pf4(s4, pv);
#pragma unroll
            for (int q = 0; q < 4; q++) {                                    // I_up / I_low bits are set for active elements only
                if (pv[q] & LF_UP) g1 = fmax(g1, mv[q]);
                if (pv[q] & LF_LOW) g2 = fmax(g2, -mv[q]);
            }
        }
        g1 = block_max<NT>(g1, red.dm);
        g2 = block_max<NT>(g2, red.dm2);
        if (!unshrink && __dadd_rn(g1, g2) <= __dmul_rn(eps, 10.0)) {
            unshrink = true;
            rebuild_gradient();
            active = l;
            refresh_flags();
            __syncthreads();
        }
        const unsigned act_lim = (unsigned)active << POS_SHIFT;
        unsigned markmask = 0u;
        int keep_local = 0;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const int s4 = (g * NT + tid) * 4;
            double mv[4]; unsigned pv[4];
            load_m4(s4, mv); load_pf4(s4, pv);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                if (pv[q] < act_lim) {
                    const bool s = (!(pv[q] & LF_UP) && mv[q] > g1) || (!(pv[q] & LF_LOW) && -mv[q] > g2);
                    markmask |= s ? 1u << (g * 4 + q) : 0u;
                    keep_local += s ? 0 : 1;
                }
            }
        }
#pragma unroll
        for (int s = 16; s; s >>= 1) keep_local += __shfl_xor_sync(0xffffffffu, keep_local, s);
        __syncthreads();
        if (lane == 0) red.cnt[warp] = keep_local;
        __syncthreads();
        int na = 0;
#pragma unroll
        for (int w = 0; w < NW; w++) na += red.cnt[w];
        if (na != active) {
            // libsvm's two-pointer sweep pairs the k-th marked position below na (ascending) with the k-th unmarked
            // position at/above na (descending).  Marks are laid out by position in global scratch.
            const int lhalf = (l + 1) / 2;
            int *const plist = scratch, *const qlist = scratch + lhalf;
            unsigned short *const swapmap = reinterpret_cast<unsigned short *>(scratch + 2 * lhalf);           // l entries
            unsigned char *const mk = reinterpret_cast<unsigned char *>(swapmap + 2 * lhalf);                  // l entries
#pragma unroll
            for (int g = 0; g < G; g++) {
                const int s4 = (g * NT + tid) * 4;
                unsigned pv[4];
                load_pf4(s4, pv);
#pragma unroll
                for (int q = 0; q < 4; q++)
                    if (pv[q] < act_lim) mk[pv[q] >> POS_SHIFT] = (markmask >> (g * 4 + q)) & 1u;
            }
            __syncthreads();
            int np = 0, nq = 0;
            for (int base = 0; base < na; base += NT) {
                const int t = base + tid;
                const bool pr = t < na && __ldcg(mk + t);
                int tot;
                const int r = block_rank<NT>(pr, red.cnt, tot);
                if (pr) plist[np + r] = t;
                np += tot;
            }
            for (int base = na; base < active; base += NT) {
                const int t = base + tid;
                const bool pr = t < active && !__ldcg(mk + t);
                int tot;
                const int r = block_rank<NT>(pr, red.cnt, tot);
                if (pr) qlist[nq + r] = t;
                nq += tot;
            }
            __syncthreads();
            for (int r = tid; r < np; r += NT) {                 // np == nq; disjoint pairs
                const int p = __ldcg(plist + r), q = __ldcg(qlist + (np - 1 - r));
                swapmap[p] = (unsigned short)q; swapmap[q] = (unsigned short)p;
            }
            __syncthreads();
            const unsigned na_lim = (unsigned)na << POS_SHIFT;
#pragma unroll
            for (int g = 0; g < G; g++) {
                const int s4 = (g * NT + tid) * 4;
                unsigned pv[4];
                load_pf4(s4, pv);
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    if (pv[q] < act_lim) {
                        const bool marked = (markmask >> (g * 4 + q)) & 1u;
                        const bool moved = pv[q] < na_lim ? marked : !marked;
                        if (moved) {
                            const unsigned np_ = __ldcg(swapmap + (pv[q] >> POS_SHIFT));
                            pv[q] = (np_ << POS_SHIFT) | (pv[q] & ((1u << POS_SHIFT) - 1u));
                        }
                    }
                }
                *reinterpret_cast<uint4 *>(pfS + s4) = make_uint4(pv[0], pv[1], pv[2], pv[3]);
            }
            active = na;
        }
        refresh_flags();
        __syncthreads();
    };

    // ---------------- main loop (svm.cpp:742-907) ----------------
    refresh_flags();                                             // builds the register mirror of the I_up / I_low bits
    bool scan_valid = false, second = false;                     // second: the retry of svm.cpp:756-764 after un-shrinking
    for (;;) {
        if (!second) {
            if (iter >= max_iter) { timed_out = 1; break; }
            if (--counter == 0) {
                counter = l < 1000 ? l : 1000;
                if (use_gbar) { do_shrink(); scan_valid = false; }
                if constexpr (PROF) tprev = clock64();
            }
        }
        if (!scan_valid) local_scan();
        if (select()) {
            if (second) break;
            rebuild_gradient();                                  // reconstruct the whole gradient, retry on the full set
            active = l;
            refresh_flags();
            __syncthreads();                                     // flags and selection scratch are rewritten above / below
            scan_valid = false;
            second = true;
            continue;
        }
        if (second) { counter = 1; second = false; }
        ++iter;

        const int slot_i = (int)((pi >> SLOT_SHIFT) & SLOT_MASK), slot_j = (int)((pj >> SLOT_SHIFT) & SLOT_MASK);
        float kvj[KPT];
        load_row(col_j, kvj);                                    // in flight during the scalar update
        // analytic two-variable update.  SOLO: evaluated by EVERY warp (uniform) -- its ~250 dependent instructions run under
        // the row-j fetch that each warp waits for anyway and the CTA needs no third barrier (a single warp computing it kept
        // the other fifteen parked).  Shared SM: warp 0 alone (4000 fewer warp-instructions per iteration).
        double a = 0, b = 0, ai_new = 0, aj_new = 0;
        int sti = 0, stj = 0;
        const bool yi = slot_i < ysplit, yj = slot_j < ysplit;
        if (SOLO || warp == 0) {
            const double Ci = yi ? Cc : Cneg, Cj = yj ? Cc : Cneg;             // per-class C (class_weight, svm.cpp:1393-1396 get_C)
            const double Gi = yi ? -gmax : gmax;                 // G = -y m (exact)
            const double Gj = yj ? -mg_j : mg_j;
            const double QDi = QDc(col_i), QDj = QDc(col_j);
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
            const double dai = __dsub_rn(ai, alpha_i), daj = __dsub_rn(aj, alpha_j);
            sti = ai >= Ci ? ST_UPPER : (ai <= 0 ? ST_LOWER : ST_FREE);
            stj = aj >= Cj ? ST_UPPER : (aj <= 0 ? ST_LOWER : ST_FREE);
            a = yi ? -dai : dai;                                 // a = -y_i dalpha_i
            b = yj ? -daj : daj;                                 // b = -y_j dalpha_j
            ai_new = ai; aj_new = aj;
            if constexpr (!SOLO) {
                if (lane == 0) {
                    red.bc_d[0] = a; red.bc_d[1] = b; red.bc_d[2] = ai; red.bc_d[3] = aj;
                    red.bc_i[0] = sti; red.bc_i[1] = stj;
                }
            }
        }
        tick(4);
        if constexpr (!SOLO) {
            __syncthreads();                                                      // barrier 3
            a = red.bc_d[0]; b = red.bc_d[1]; ai_new = red.bc_d[2]; aj_new = red.bc_d[3];
            sti = red.bc_i[0]; stj = red.bc_i[1];
        }
        tick(5);
        {
            // the OWNERS of i and j store alpha and the slot word (new status and set membership) and patch their flag mask;
            // nobody else reads these before the next barrier
            auto own = [&](int s, unsigned w, bool y, int st, double av) {
                const int grp = s >> 2;
                if ((grp & (NT - 1)) == tid) {
                    const unsigned fl = lean_flags(y, st);
                    const int k = (grp / NT) * 4 + (s & 3);
                    alpha_g[s] = av;
                    pfS[s] = (w & ~15u) | fl;
                    fm = (fm & ~(3u << (2 * k))) | ((fl >> 2) << (2 * k));
                }
            };
            own(slot_i, pi, yi, sti, ai_new);
            own(slot_j, pj, yj, stj, aj_new);
        }

        // m update (svm.cpp:866-872) over every slot, fused with the next iteration's local scan: strict compare and a tie
        // flag here; a thread that met equal values redoes its scan with the full (value, position) order
        la = -CUDART_INF;
        int la_k = -1;
        unsigned la_tie = 0u;
        if constexpr (FAST) {
            double mvu[4];
            lean_loop<G * 4>([&](auto kc) {
                constexpr int k = decltype(kc)::value, g = k >> 2, q = k & 3;
                if constexpr (q == 0) load_m4((g * NT + tid) * 4, mvu);
                lean_update_slot<k>(mvu[q], kvi[k], kvj[k], a, b, fm, la, la_k, la_tie);
                if constexpr (q == 3) store_m4((g * NT + tid) * 4, mvu);
            });
        } else {
#pragma unroll
            for (int g = 0; g < G; g++) {
                const int s4 = (g * NT + tid) * 4;
                double mv[4];
                load_m4(s4, mv);
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int k = g * 4 + q;
                    mv[q] = __dadd_rn(mv[q], __dadd_rn(__dmul_rn(widen(kvi[k]), a), __dmul_rn(widen(kvj[k]), b)));
                    const bool up = (fm & (1u << (2 * k))) != 0u;
                    const bool better = up & (mv[q] > la);
                    la_tie |= (up & (mv[q] == la)) ? 1u : 0u;
                    la = better ? mv[q] : la;
                    la_k = better ? k : la_k;
                }
                store_m4(s4, mv);
            }
        }
        la_pf = la_k >= 0 ? pfS[slot_of(la_k)] : 0u;
        if (la_tie) local_scan();
        scan_valid = true;
        // G_bar over all l when a bound status flips (svm.cpp:876-905): i first, then j; K_i and K_j are still in registers
        const bool need_i = use_gbar && (((pi & 3u) == ST_UPPER) != (sti == ST_UPPER));
        const bool need_j = use_gbar && (((pj & 3u) == ST_UPPER) != (stj == ST_UPPER));
        if (need_i || need_j) {
            // Gbar -= C Q_i (was upper) / += C Q_i (became upper)  <=>  mbar += fl(c K_i), c = +/- y_i C
            const double Cmi = slot_i < ysplit ? Cc : Cneg, Cmj = slot_j < ysplit ? Cc : Cneg;
            const double ci = (((pi & 3u) == ST_UPPER) == (slot_i < ysplit)) ? Cmi : -Cmi;
            const double cj = (((pj & 3u) == ST_UPPER) == (slot_j < ysplit)) ? Cmj : -Cmj;
            // one group of 4 slots at a time, the next group's G_bar already in flight (all of it at once spills)
            double2 nx0 = make_double2(0, 0), nx1 = nx0;
            if (tid * 4 < nslots) { nx0 = *reinterpret_cast<const double2 *>(gbar_g + tid * 4); nx1 = *reinterpret_cast<const double2 *>(gbar_g + tid * 4 + 2); }
#pragma unroll
            for (int g = 0; g < G; g++) {
                const int s4 = (g * NT + tid) * 4;
                double gb[4] = {nx0.x, nx0.y, nx1.x, nx1.y};
                if (g + 1 < G) {
                    const int n4 = ((g + 1) * NT + tid) * 4;
                    if (n4 < nslots) { nx0 = *reinterpret_cast<const double2 *>(gbar_g + n4); nx1 = *reinterpret_cast<const double2 *>(gbar_g + n4 + 2); }
                }
                if (s4 < nslots) {
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        if (need_i) gb[q] = __dadd_rn(gb[q], __dmul_rn(ci, widen(kvi[g * 4 + q])));
                        if (need_j) gb[q] = __dadd_rn(gb[q], __dmul_rn(cj, widen(kvj[g * 4 + q])));
                    }
                    *reinterpret_cast<double2 *>(gbar_g + s4) = make_double2(gb[0], gb[1]);
                    *reinterpret_cast<double2 *>(gbar_g + s4 + 2) = make_double2(gb[2], gb[3]);
                }
            }
        }
        tick(6);
    }

    // ---------------- results ----------------
    __syncthreads();
    if (timed_out && active < l) {                               // svm.cpp:912-919: the gradient of the whole set before rho
        rebuild_gradient();
        active = l;
    }
    // coefficients alpha_k*y_k scattered by dataset row (svm.cpp:922-925, :1641-1642); SV counts; then y*G and the status
    // re-laid by POSITION for calculate_rho
    int nsv = 0, nbsv = 0;
    double yg[KPT];
    unsigned wv[KPT];
    {
        double *__restrict__ coef = Pp->coef;
#pragma unroll
        for (int g = 0; g < G; g++) {
            const int s4 = (g * NT + tid) * 4;
            double mv[4]; unsigned pv[4];
            load_m4(s4, mv); load_pf4(s4, pv);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                yg[g * 4 + q] = -mv[q]; wv[g * 4 + q] = pv[q];
                if (pv[q] < PF_INERT) {
                    const double av = __ldcg(alpha_g + s4 + q);
                    coef[gcol[g] + q] = s4 + q < ysplit ? av : -av;
                    nsv += av > 0;
                    nbsv += av >= (s4 + q < ysplit ? Cc : Cneg);
                }
            }
        }
    }
    __syncthreads();
    {
        const unsigned act_lim = (unsigned)active << POS_SHIFT;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            if (wv[k] < act_lim) {
                const int p = (int)(wv[k] >> POS_SHIFT);
                const int s = ((k >> 2) * NT + tid) * 4 + (k & 3);
                mG[p] = yg[k];
                pfS[p] = (wv[k] & 3u) | (s < ysplit ? 4u : 0u);
            }
        }
    }
    __syncthreads();
    // calculate_rho (svm.cpp:1131-1168): sequential float64 sum in ascending position
    if (tid == 0) {
        int nfree = 0;
        double ub = CUDART_INF, lb = -CUDART_INF, sum = 0;
        for (int t = 0; t < active; t++) {
            const unsigned f = pfS[t];
            const double yG = mG[t];
            if ((f & 3u) == ST_UPPER) { if (!(f & 4u)) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
            else if ((f & 3u) == ST_LOWER) { if (f & 4u) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
            else { ++nfree; sum = __dadd_rn(sum, yG); }
        }
        *Pp->out_rho = nfree > 0 ? __ddiv_rn(sum, (double)nfree) : __ddiv_rn(__dadd_rn(ub, lb), 2.0);
    }
#pragma unroll
    for (int s = 16; s; s >>= 1) {
        nsv += __shfl_xor_sync(0xffffffffu, nsv, s);
        nbsv += __shfl_xor_sync(0xffffffffu, nbsv, s);
    }
    if (lane == 0) { red.cnt[warp] = nsv; red.a_pf[warp] = (unsigned)nbsv; }
    __syncthreads();
    if (tid == 0) {
        int s = 0, bs = 0;
        for (int w = 0; w < NW; w++) { s += red.cnt[w]; bs += (int)red.a_pf[w]; }
        int *info = Pp->out_info;
        info[0] = iter; info[1] = timed_out; info[2] = s; info[3] = bs;
        unsigned long long t_end;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
        unsigned long long *ns = Pp->out_ns;
        ns[0] = t_start; ns[1] = t_end;
        if constexpr (PROF)
            for (int q = 0; q < 8; q++) ns[2 + q] = (unsigned long long)prof[q];
    }
}

template <int NT, int G, bool FAST, bool PROF, bool SOLO>
cudaError_t launch_lean_one(const SmoProblem *probs, const int *order, int n_prob, bool exclusive, cudaStream_t st)
{
    constexpr int LCAP = NT * G * 4;
    // exclusive: ask for more than half of the SM's 227 KB so that no second CTA (of this or of the shared launch) fits
    const size_t smem = exclusive ? std::max<size_t>((size_t)LCAP * 12, 132 * 1024) : (size_t)LCAP * 12;
    auto kern = smo_lean_kernel<NT, G, FAST, PROF, SOLO>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    kern<<<n_prob, NT, smem, st>>>(probs, order);
    return cudaGetLastError();
}

template <int NT, int G, bool SOLO>
cudaError_t launch_lean_cfg2(const SmoProblem *probs, const int *order, int n_prob, bool fast, bool prof, bool excl, cudaStream_t st)
{
    if (prof) return fast ? launch_lean_one<NT, G, true, true, SOLO>(probs, order, n_prob, excl, st) : launch_lean_one<NT, G, false, true, SOLO>(probs, order, n_prob, excl, st);
    return fast ? launch_lean_one<NT, G, true, false, SOLO>(probs, order, n_prob, excl, st) : launch_lean_one<NT, G, false, false, SOLO>(probs, order, n_prob, excl, st);
}

template <int NT, int G>
cudaError_t launch_lean_cfg(const SmoProblem *probs, const int *order, int n_prob, bool fast, bool prof, bool excl, bool solo, cudaStream_t st)
{
    return solo ? launch_lean_cfg2<NT, G, true>(probs, order, n_prob, fast, prof, excl, st) : launch_lean_cfg2<NT, G, false>(probs, order, n_prob, fast, prof, excl, st);
}

int env_int(const char *name, int dflt)
{
    const char *v = getenv(name);
    return v && *v ? atoi(v) : dflt;
}

}  // namespace

int smo_lean_max_slots() { return 16384; }

// Every problem of the launch must have a slot layout (nseg > 0, nslots <= max_slots <= 16384, l < 16383).
// Shapes: (threads) x 4 groups of 4 slots per thread = 16 slots per thread at 64 registers: two 8192-slot sub-problems per SM
// (32 slots per thread at 128 registers measured no faster and does not fit the one-register flag mask).
cudaError_t launch_smo_lean(const SmoProblem *d_probs, const int *d_order, int n_prob, int max_slots, bool fast, bool exclusive, cudaStream_t st)
{
    if (n_prob <= 0) return cudaSuccess;
    const bool prof = env_int("B200GS_SMO_PROF", 0) != 0;                    // development switch: per-phase cycle counters
    if (env_int("B200GS_SMO_NOFAST", 0)) fast = false;
    // Two instances of the two-variable update: warp 0 evaluates it behind a third barrier, or every warp evaluates it
    // redundantly (SOLO).  The barrier instance is the default: config 2's solve phase takes 331.8 ms with it and 342.2 ms with
    // SOLO (one H100 SXM capped at 400 W, B200GS_SMO_TIMELINE, same run).
    bool solo = false;
    if (const char *e = getenv("B200GS_LEAN_SOLO")) solo = atoi(e) != 0;      // development switch
    // A problem alone on its SM spreads over 1024 threads x 8 slots instead of 512 x 16 (bit-identical trajectories): config 2's
    // solve phase takes 331.8 ms with it and 352.6 ms without (same H100 run as above).  B200GS_LEAN_EXCL_WIDE=0: off.
    if (exclusive && max_slots > 4096 && max_slots <= 8192 && env_int("B200GS_LEAN_EXCL_WIDE", 1))
        return launch_lean_cfg<1024, 2>(d_probs, d_order, n_prob, fast, prof, exclusive, solo, st);
    if (max_slots <= 2048) return launch_lean_cfg<128, 4>(d_probs, d_order, n_prob, fast, prof, exclusive, solo, st);
    if (max_slots <= 4096) return launch_lean_cfg<256, 4>(d_probs, d_order, n_prob, fast, prof, exclusive, solo, st);
    if (max_slots <= 8192) return launch_lean_cfg<512, 4>(d_probs, d_order, n_prob, fast, prof, exclusive, solo, st);
    if (max_slots <= 16384) return launch_lean_cfg<1024, 4>(d_probs, d_order, n_prob, fast, prof, exclusive, solo, st);
    return cudaErrorInvalidValue;
}
