// smo_colown.cu -- cluster SMO solver with STATIC element ownership ("column owner") and register-resident state.
//
// Same algorithm and the same bit-exact trajectory as smo.cu (libsvm svm.cpp:629-1168 restated there), one sub-problem
// per thread-block cluster of CL CTAs.  What differs from a position-owned layout is WHERE an element lives:
//
//   * libsvm's shrinking permutes positions (swap_index, svm.cpp:616-627) and every tie-break and summation order is
//     defined on positions.  Here an element (one training row) never moves: thread (rank, tid, k) owns element
//     e = (k*CL + rank)*NT + tid for the whole solve and carries its CURRENT POSITION as state.  A libsvm swap of
//     positions p and q is an exchange of two integers; `pos < active` is the active-set test; arg-reductions compare
//     (value, position) exactly as libsvm's "last index wins" scans do.
//   * Because the element -> dataset-row map is fixed and the sub-problem's rows are ascending runs of the (class-sorted)
//     dataset, a K row is gathered with COALESCED loads: each CTA reads only its own 1/CL of the row, once, straight
//     into registers -- one DRAM round trip, no column indirection, no row staging.  (Position-owned layouts scatter a
//     CTA's columns over the whole row after the first shrink: every CTA then pulls all of it.)
//   * m = -y*G, the position, the flags and the K_i values of the owned elements live in REGISTERS; alpha and
//     mbar = -y*G_bar (touched by two elements per iteration / on status flips) in shared memory.
//
// The hot loop has no CTA-wide or cluster-wide barrier.  Each of the two arg-reductions
// of an iteration is two-level: a warp reduces its own elements (REDUX), its winner lane stores the warp's record in
// local shared memory and the warp arrives on a named barrier; the LEADER warp reduces the NW warp records, st.async-writes
// the CTA's record into every CTA's shared memory (bytes counted on each RECEIVER's mbarrier), reduces the CL CTA records
// and publishes the result through shared memory and a named barrier on which the worker warps are parked.  Only the
// leader executes the combines and the scalar two-variable update, so the workers' issue slots stay free.
// Cold paths keep CTA-level records (double-buffered by parity) behind __syncthreads.
//
// Cold paths (every 1000 iterations / at unshrink): do_shrinking builds libsvm's two-pointer partition from a
// position-indexed mark array (all-gathered through DSMEM), each CTA deriving the identical swap map; the gradient
// reconstruction and calculate_rho walk positions in ascending order through position-indexed global scratch.
#include "smo_common.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace {

using namespace smo;

constexpr int XW = 16;                       // words per exchange record
constexpr int NOPOS = 0x3fffffff;            // position of a slot that holds no element

template <int CL>
struct __align__(16) Xch {                   // double-buffered all-gather slots: [parity][source rank][word]
    unsigned w[2][CL][XW];
};

__device__ __forceinline__ unsigned lo32(double x) { return (unsigned)__double_as_longlong(x); }
__device__ __forceinline__ unsigned hi32(double x) { return (unsigned)((unsigned long long)__double_as_longlong(x) >> 32); }
__device__ __forceinline__ double mk64(unsigned lo, unsigned hi) { return __longlong_as_double((long long)(((unsigned long long)hi << 32) | lo)); }

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned mapa_u32(unsigned addr, unsigned cta)
{
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(cta));
    return r;
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Default (acquire, CTA scope) wait: shared-memory data delivered by st.async is made visible by the complete_tx that
// finishes the phase; a .cluster-scope acquire would add an L1 invalidate (CCTL.IVALL) to every wait.
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
    unsigned done = 0;
    for (unsigned spin = 0; !done; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1u << 26)) __trap();                                    // a lost signal must not hang the GPU
    }
}

template <int NT, int KPT, int CL, bool FAST, bool PROF>
__global__ void __launch_bounds__(NT, 1)
smo_colown_kernel(const SmoProblem *__restrict__ probs, const int *__restrict__ order)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ Red red;
    __shared__ Xch<CL> xch;
    __shared__ __align__(8) unsigned long long xbar[2];                      // cold paths: one mbarrier per exchange parity
    constexpr int NW = NT / 32;
    // hot-loop mailboxes: per-warp records (local), per-CTA records (written by every leader), results (leader -> workers)
    __shared__ struct __align__(16) {
        unsigned recA[NW][8];        // key hi lo | idx+flags | km hi | km lo | alpha lo hi | col
        unsigned recB[NW][12];       // b1 | idx | b2 | col | m lo hi | K_i lo hi | alpha lo hi | pad
        unsigned recX[NW][12];       // hi | idx | lo | col | m | K_i | alpha | pad          (exact tie-break)
        unsigned xA[CL][8], xB[CL][12], xX[CL][12];
        unsigned resA[4];            // i (packed; -1 = stop) | col_i | gmax lo hi
        unsigned resB1[4];           // j (packed) | col_j | mode | band threshold
        unsigned resB2[12];          // a | b | alpha_i' | alpha_j' | status_i | status_j
        unsigned resX[4];            // j (packed) | col_j
    } hot;
    enum { HB_XA = 0, HB_XB, HB_XX, HB_N };                                  // cross-CTA record arrival (mbarrier, tx bytes): leader only
    enum { NB_LA = 1, NB_RA, NB_LB, NB_RB1, NB_RB2, NB_LX, NB_RX };          // hardware named barriers (0 is __syncthreads)
    __shared__ __align__(8) unsigned long long hbar[HB_N];
    constexpr int LCAP = NT * KPT;                                          // elements owned by this CTA

    cg::cluster_group cluster = cg::this_cluster();
    const unsigned rank = cluster.block_rank();
    const SmoProblem *__restrict__ Pp = probs + order[blockIdx.x / CL];
    if (Pp->guard != nullptr && (*Pp->guard != 0) == FAST) return;       // the other instance solves this launch (common.cuh)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int l = Pp->l;
    const int lhalf = (l + 1) / 2;
    // ---- shared memory: per-element alpha / mbar, then the cold-path arrays indexed by POSITION ----
    double *const alpha = reinterpret_cast<double *>(smem_raw);             // [k*NT + tid]
    double *const mGbar = alpha + LCAP;
    int *const lists = reinterpret_cast<int *>(mGbar + LCAP);               // l ints: plist | qlist, or the free list
    unsigned short *const swapmap = reinterpret_cast<unsigned short *>(lists + l);   // l
    unsigned char *const mk = reinterpret_cast<unsigned char *>(swapmap + l);        // l
    const float *__restrict__ const K = Pp->K;
    const int64_t ldk = Pp->ldk;
    const double eps = Pp->eps;
    const double Cc = Pp->C, Cneg = Pp->Cn;                                   // C of the +1 / -1 class
    const bool use_gbar = Pp->shrinking != 0;
    const double *__restrict__ const qd = FAST ? nullptr : Pp->qd;
    int *const scratch = Pp->scratch;                                        // global ints, >= 2*l
    double *const gscratch = Pp->Gbar;                                       // global doubles, l (G_bar lives in shared memory here)

    unsigned long long t_start = 0;
    if (tid == 0 && rank == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));

    // ---- element state in registers ----
    double m[KPT];            // m = -y*G
    int pos[KPT];             // current libsvm position (NOPOS: empty slot)
    int fl[KPT];              // status | F_YPOS | F_UP | F_LOW
    int colr[KPT];            // dataset row == column of K
    // initial point: alpha = 0, G = -1  =>  m = y (svm.cpp:1611-1626, :716-736)
    {
        const int n_pos = Pp->n_pos;
        const int *__restrict__ rows = Pp->rows;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            const int e = (k * CL + (int)rank) * NT + tid, s = k * NT + tid;
            alpha[s] = 0.0; mGbar[s] = 0.0;
            if (e < l) {
                const bool yp = e < n_pos;
                m[k] = yp ? 1.0 : -1.0; pos[k] = e; fl[k] = mkflags(yp, ST_LOWER); colr[k] = rows[e];
            } else { m[k] = 0.0; pos[k] = NOPOS; fl[k] = 0; colr[k] = 0; }
        }
    }
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&xbar[0])));
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&xbar[1])));
        for (int q = 0; q < HB_N; q++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&hbar[q])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    cluster.sync();                                                         // every CTA's barriers exist before any remote signal

    long long prof[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    long long tprev = PROF ? clock64() : 0;
    auto tick = [&](int slot) {
        if constexpr (PROF) {
            const long long now = clock64();
            prof[slot] += now - tprev;
            tprev = now;
        }
    };

    int active = l, iter = 0, timed_out = 0;
    int counter = (l < 1000 ? l : 1000) + 1;
    bool unshrink = false;
    const int max_iter = Pp->max_iter == -1 ? SAFETY_MAX_ITER : Pp->max_iter;
    int par = 0;                                                            // exchange parity
    unsigned xphase = 0;                                                    // bit p: parity the next wait on xbar[p] uses

    float kvi[KPT];                                                         // unsigned K_i at the owned elements (float32 as stored)

    auto QDc = [&](int c) -> double {                                       // by dataset row (svm.cpp:1436-1437)
        if constexpr (FAST) return 1.0;
        else return qd ? qd[c] : 1.0;
    };
    auto widen = [&](float x) -> double {
        if constexpr (FAST) {
            const unsigned u = __float_as_uint(x);
            return __hiloint2double((int)((u >> 3) + 0x38000000u), (int)(u << 29));
        } else return f2d(x);
    };

    // all-gather of one record per CTA (v must be warp-uniform in warp 0: REDUX results and broadcast shared reads)
    auto exchange = [&](const unsigned (&v)[XW]) -> const unsigned (*)[XW] {
        const unsigned bar = smem_u32(&xbar[par]);
        if (warp == 0) {
            if (lane == 0) mbar_expect_tx(bar, CL * XW * 4);
            if (lane < CL * 4) {                                             // lane -> (destination CTA, 16-byte chunk)
                const int c = lane & 3;
                const unsigned dst = (unsigned)lane >> 2;
                const unsigned a0 = c == 0 ? v[0] : (c == 1 ? v[4] : (c == 2 ? v[8] : v[12]));
                const unsigned a1 = c == 0 ? v[1] : (c == 1 ? v[5] : (c == 2 ? v[9] : v[13]));
                const unsigned a2 = c == 0 ? v[2] : (c == 1 ? v[6] : (c == 2 ? v[10] : v[14]));
                const unsigned a3 = c == 0 ? v[3] : (c == 1 ? v[7] : (c == 2 ? v[11] : v[15]));
                const unsigned raddr = mapa_u32(smem_u32(&xch.w[par][rank][c * 4]), dst);
                const unsigned rbar = mapa_u32(bar, dst);
                asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
                             ::"r"(raddr), "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(rbar) : "memory");
            }
        }
        mbar_wait(bar, (xphase >> par) & 1u);
        xphase ^= 1u << par;
        const unsigned (*r)[XW] = xch.w[par];
        par ^= 1;
        return r;
    };

    // ---------------- local scan (normally fused into the update loop) ----------------
    // la: max m over the owned I_up elements, ties -> larger position (libsvm's ascending ">=" scan); lm: min m over I_low
    // (the winner's column / flags / slot are tracked as VALUES: selecting them later by a run-time k makes the compiler
    //  index the register arrays dynamically, which demotes them to local memory -- measured: 8 LDL per element loop)
    double la = -CUDART_INF, lm = CUDART_INF;
    int la_pos = -1, la_col = 0, la_fl = 0, la_slot = 0;
    auto scan_elem = [&](int k) {
        const int f = fl[k];
        const double mv = m[k];
        if ((f & F_UP) && (mv > la || (mv == la && pos[k] > la_pos))) { la = mv; la_pos = pos[k]; la_col = colr[k]; la_fl = f; la_slot = k * NT + tid; }
        if (f & F_LOW) lm = fmin(lm, mv);
    };
    auto local_scan = [&]() {
        la = -CUDART_INF; lm = CUDART_INF; la_pos = -1;
#pragma unroll
        for (int k = 0; k < KPT; k++)
            if (pos[k] < active) scan_elem(k);
    };

    // ---------------- reconstruct_gradient (svm.cpp:629-668) ----------------
    // m_k = (mbar_k + y_k) + sum over free active f in ASCENDING POSITION of fl((-y_f alpha_f) K_fk), for inactive k
    auto rebuild_gradient = [&]() {
        if (active == l) return;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            if (pos[k] < active) {
                const bool fr = (fl[k] & 3) == ST_FREE;
                scratch[pos[k]] = fr ? colr[k] : -1;
                if (fr) { const double av = alpha[k * NT + tid]; gscratch[pos[k]] = (fl[k] & F_YPOS) ? -av : av; }
            }
        }
        __threadfence();
        cluster.sync();
        int nf = 0;
        for (int base = 0; base < active; base += NT) {                     // every CTA compacts the same list
            const int t = base + tid;
            const bool isf = t < active && __ldcg(scratch + t) >= 0;
            int tot;
            const int r = block_rank<NT>(isf, red.cnt, tot);
            if (isf) lists[nf + r] = t;
            nf += tot;
        }
        __syncthreads();
        double g[KPT];
        bool in[KPT];
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            in[k] = pos[k] >= active && pos[k] != NOPOS;
            g[k] = in[k] ? __dadd_rn(mGbar[k * NT + tid], (fl[k] & F_YPOS) ? 1.0 : -1.0) : 0.0;
        }
#pragma unroll 2
        for (int r = 0; r < nf; r++) {
            const int p = lists[r];
            const float *__restrict__ Kf = K + (size_t)__ldcg(scratch + p) * ldk;
            const double af = __ldcg(gscratch + p);
#pragma unroll
            for (int k = 0; k < KPT; k++)
                if (in[k]) g[k] = __dadd_rn(g[k], __dmul_rn(af, widen(__ldg(Kf + colr[k]))));
        }
#pragma unroll
        for (int k = 0; k < KPT; k++)
            if (in[k]) m[k] = g[k];
        cluster.sync();                                                      // scratch is reused by the next cold path
    };

    // ---------------- select_working_set (svm.cpp:946-1047) ----------------
    // Two-level arg-reduction without CTA or cluster barriers.  Every warp reduces its own elements (REDUX); its winner
    // lane stores the warp's record in LOCAL shared memory and the warp arrives on a named barrier.  The leader warp
    // (warp 0) reduces the NW records, st.async-sends the CTA's record to every CTA of the cluster (bytes counted on each
    // receiver's mbarrier), reduces the CL CTA records, and publishes the result in shared memory + a named barrier the
    // workers are parked on.  Only the leader executes the combines and the scalar update: the other warps' issue slots stay free.
    // Slot reuse is safe without further synchronisation: a warp writes its stage-(n+1) record only after it consumed the
    // stage-n result, which the leader published after reading all stage-n records; a remote leader can send stage n+1
    // only after a full B (or X) stage in between, which needs this CTA's leader to have passed stage n.
    unsigned ph = 0;                                     // phase parity bit per hot mbarrier (index = HB_*)
    auto hb_wait = [&](int b) {
        mbar_wait(smem_u32(&hbar[b]), (ph >> b) & 1u);
        ph ^= 1u << b;
    };
    // worker <-> leader hand-offs inside the CTA use HARDWARE named barriers (waiting warps are parked, not polling:
    // fifteen warps spinning on an mbarrier starve the leader of issue slots -- 1.9k cycles per stage vs 0.6k on the 148-SM GPU the kernels were first tuned on)
    auto nb_arrive = [&](int id) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(NT) : "memory"); };
    auto nb_sync = [&](int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(NT) : "memory"); };
    // leader: send the CTA record (W words, uniform registers c[]) to slot [rank] of every CTA, then wait for all CL records
    auto leader_allgather = [&](unsigned slots_base, int W, const unsigned (&c)[12], int xb) {
        const unsigned bar = smem_u32(&hbar[xb]);
        const int chunks = W / 4;
        if (lane == 0) mbar_expect_tx(bar, (unsigned)(CL * W * 4));
        if (lane < CL * chunks) {
            const int dst = lane / chunks, ch = lane % chunks;
            const unsigned a0 = ch == 0 ? c[0] : (ch == 1 ? c[4] : c[8]);
            const unsigned a1 = ch == 0 ? c[1] : (ch == 1 ? c[5] : c[9]);
            const unsigned a2 = ch == 0 ? c[2] : (ch == 1 ? c[6] : c[10]);
            const unsigned a3 = ch == 0 ? c[3] : (ch == 1 ? c[7] : c[11]);
            const unsigned ra = mapa_u32(slots_base + (unsigned)((int)rank * W + ch * 4) * 4u, (unsigned)dst);
            const unsigned rb = mapa_u32(bar, (unsigned)dst);
            asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
                         ::"r"(ra), "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(rb) : "memory");
        }
        hb_wait(xb);
    };

    int pi = -1, pj = -1, col_i = 0, col_j = 0;          // packed (position << 5 | flags), dataset rows
    double gmax = 0, mg_j = 0, k_ij = 0, alpha_i = 0, alpha_j = 0;      // mg_j, k_ij, alpha_*: valid in the leader warp only
    auto select = [&]() -> bool {
        {   // ---- stage A: i = argmax m over I_up, Gmax2 = max -m over I_low ----
            const unsigned long long key = dkey(la);
            const int la_idx = la_pos >= 0 ? (la_pos << IDX_SHIFT) : -1;             // the winner lane adds the flags
            const KArg w = warp_argmax((unsigned)(key >> 32), (unsigned)key, la_idx);
            const unsigned long long km = warp_keymax(dkey(-lm));
            if (w.idx >= 0 ? la_idx == w.idx : lane == 0) {                          // exactly one lane per warp
                const int c = la_col, f = la_fl;
                const double av = w.idx >= 0 ? alpha[la_slot] : 0.0;
                *reinterpret_cast<uint4 *>(&hot.recA[warp][0]) =
                    make_uint4(w.hi, w.lo, w.idx >= 0 ? (unsigned)(w.idx | f) : 0xffffffffu, (unsigned)(km >> 32));
                *reinterpret_cast<uint4 *>(&hot.recA[warp][4]) = make_uint4((unsigned)km, lo32(av), hi32(av), (unsigned)c);
            }
            __syncwarp();
            tick(0);
            if (warp == 0) {
                nb_sync(NB_LA);
                const bool v = lane < NW;
                uint4 x0 = make_uint4(0u, 0u, 0xffffffffu, 0u), x1 = make_uint4(0u, 0u, 0u, 0u);
                if (v) { x0 = *reinterpret_cast<const uint4 *>(&hot.recA[lane][0]); x1 = *reinterpret_cast<const uint4 *>(&hot.recA[lane][4]); }
                const KArg a = warp_argmax(x0.x, x0.y, (int)x0.z);
                const unsigned long long km2 = warp_keymax(((unsigned long long)x0.w << 32) | x1.x);
                const int wl = a.idx >= 0 ? __ffs(__ballot_sync(0xffffffffu, (int)x0.z == a.idx)) - 1 : 0;
                unsigned c[12];
                c[0] = a.hi; c[1] = a.lo; c[2] = (unsigned)a.idx; c[3] = (unsigned)(km2 >> 32); c[4] = (unsigned)km2;
                c[5] = __shfl_sync(0xffffffffu, x1.y, wl); c[6] = __shfl_sync(0xffffffffu, x1.z, wl); c[7] = __shfl_sync(0xffffffffu, x1.w, wl);
                c[8] = c[9] = c[10] = c[11] = 0u;
                leader_allgather(smem_u32(&hot.xA[0][0]), 8, c, HB_XA);
                const bool vc = lane < CL;
                uint4 y0 = make_uint4(0u, 0u, 0xffffffffu, 0u), y1 = make_uint4(0u, 0u, 0u, 0u);
                if (vc) { y0 = *reinterpret_cast<const uint4 *>(&hot.xA[lane][0]); y1 = *reinterpret_cast<const uint4 *>(&hot.xA[lane][4]); }
                const KArg g = warp_argmax(y0.x, y0.y, (int)y0.z);
                const unsigned long long kg = warp_keymax(((unsigned long long)y0.w << 32) | y1.x);
                const int gl = g.idx >= 0 ? __ffs(__ballot_sync(0xffffffffu, (int)y0.z == g.idx)) - 1 : 0;
                alpha_i = mk64(__shfl_sync(0xffffffffu, y1.y, gl), __shfl_sync(0xffffffffu, y1.z, gl));
                const int ci = (int)__shfl_sync(0xffffffffu, y1.w, gl);
                const double gm = dkey_inv(((unsigned long long)g.hi << 32) | g.lo), gm2 = dkey_inv(kg);
                const bool stop = g.idx < 0 || __dadd_rn(gm, gm2) < eps;              // svm.cpp:1040-1041
                if (lane == 0)
                    *reinterpret_cast<uint4 *>(&hot.resA[0]) = make_uint4(stop ? 0xffffffffu : (unsigned)g.idx, (unsigned)ci, lo32(gm), hi32(gm));
                __syncwarp();
                nb_arrive(NB_RA);
            } else { nb_arrive(NB_LA); nb_sync(NB_RA); }
            const uint4 r = *reinterpret_cast<const uint4 *>(&hot.resA[0]);
            pi = (int)r.x; col_i = (int)r.y; gmax = mk64(r.z, r.w);
            tick(1);
        }
        if (pi < 0) return true;
        // ---- stage B: j = argmin -(gd^2)/quad over I_low with gd > 0 (svm.cpp:980-1037) ----
        const double QDi = QDc(col_i);
        const float *__restrict__ Ki = K + (size_t)col_i * ldk;
#pragma unroll
        for (int k = 0; k < KPT; k++) kvi[k] = pos[k] < active ? __ldg(Ki + colr[k]) : 0.f;    // coalesced: fixed columns
        tick(2);
        // Approximate gd^2/quad tracked by a 32-bit order-preserving key; every near-tie (keys within BAND units) is decided
        // by the exact libsvm quotients below, so the choice stays bit-identical (error analysis: smo.cu, same filter).
        constexpr unsigned BAND = FAST ? 64u : 514u;
        constexpr unsigned KEY_TINY = 0x0D800000u;                          // float bits of 2^-100
        auto approx_key = [&](double gd, float kvf, int c) -> unsigned {
            if constexpr (FAST) {
                const float gdf = __double2float_rn(gd);
                const float quadf = __fmaf_rn(-2.f, kvf, 2.f);              // == fl32(2 - 2K): 2K is exact
                const float g2f = __fmul_rn(gdf, gdf);
                float r;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(quadf));
                const float apf = quadf > 0.f ? __fmul_rn(g2f, r) : __fmul_rn(g2f, 1e12f);
                return __float_as_uint(apf) + 1u;                           // +1: a valid candidate is never 0
            } else {
                const double quad = __dsub_rn(__dadd_rn(QDi, QDc(c)), __dmul_rn(2.0, widen(kvf)));
                const double g2 = __dmul_rn(gd, gd);
                const double ap = quad > 0 ? g2 * rcp_approx(quad) : g2 * 1e12;
                return (unsigned)__double2hiint(ap) + 1u;
            }
        };
        unsigned b1k = 0u, b2k = 0u;                    // keys of the best and second-best candidate (0 = none)
        int idx1 = -1, c1v = 0, s1v = 0;                // the best candidate's packed index, column, state slot ...
        float kq1 = 0.f;                                // ... K_i value
        double m1v = 0.0;                               // ... and m
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            if (pos[k] < active) {
                const int f = fl[k];
                const double gd = __dsub_rn(gmax, m[k]);
                if ((f & F_LOW) && gd > 0) {
                    const unsigned key = approx_key(gd, kvi[k], colr[k]);
                    const bool gt = key > b1k;
                    b2k = gt ? b1k : max(b2k, key);
                    b1k = gt ? key : b1k;
                    if (gt) { idx1 = (pos[k] << IDX_SHIFT) | f; c1v = colr[k]; s1v = k * NT + tid; kq1 = kvi[k]; m1v = m[k]; }
                }
            }
        }
        // record of one candidate element: words 3.. = col | m | K_i (widened) | alpha
        auto store_record = [&](unsigned (*rec)[12], int cc, int slot, float kq, double mm, unsigned w0, unsigned w1, unsigned w2, bool has) {
            const double qq = widen(kq), av = has ? alpha[slot] : 0.0;
            *reinterpret_cast<uint4 *>(&rec[warp][0]) = make_uint4(w0, w1, w2, (unsigned)cc);
            *reinterpret_cast<uint4 *>(&rec[warp][4]) = make_uint4(lo32(mm), hi32(mm), lo32(qq), hi32(qq));
            *reinterpret_cast<uint2 *>(&rec[warp][8]) = make_uint2(lo32(av), hi32(av));
        };
        int mode;                                        // 0: j chosen; 1: exact tie-break needed; -1: no j (Gmin_idx == -1)
        unsigned thrk;
        {
            const unsigned w1 = __reduce_max_sync(0xffffffffu, b1k);
            const int widx = __reduce_max_sync(0xffffffffu, (b1k == w1) ? idx1 : -1);
            const unsigned w2 = __reduce_max_sync(0xffffffffu, (idx1 == widx) ? b2k : b1k);
            if (widx >= 0 ? idx1 == widx : lane == 0) {
                store_record(hot.recB, c1v, s1v, kq1, m1v, w1, (unsigned)widx, w2, widx >= 0);
            }
            __syncwarp();
            tick(3);
            if (warp == 0) {
                nb_sync(NB_LB);
                const bool v = lane < NW;
                uint4 x0 = make_uint4(0u, 0xffffffffu, 0u, 0u), x1 = make_uint4(0u, 0u, 0u, 0u);
                uint2 x2 = make_uint2(0u, 0u);
                if (v) {
                    x0 = *reinterpret_cast<const uint4 *>(&hot.recB[lane][0]); x1 = *reinterpret_cast<const uint4 *>(&hot.recB[lane][4]);
                    x2 = *reinterpret_cast<const uint2 *>(&hot.recB[lane][8]);
                }
                const unsigned c1 = __reduce_max_sync(0xffffffffu, (int)x0.y >= 0 ? x0.x : 0u);
                const int cidx = __reduce_max_sync(0xffffffffu, ((int)x0.y >= 0 && x0.x == c1) ? (int)x0.y : -1);
                const unsigned c2 = __reduce_max_sync(0xffffffffu, (int)x0.y == cidx ? x0.z : ((int)x0.y >= 0 ? x0.x : 0u));
                const int wl = cidx >= 0 ? __ffs(__ballot_sync(0xffffffffu, (int)x0.y == cidx)) - 1 : 0;
                unsigned c[12];
                c[0] = c1; c[1] = (unsigned)cidx; c[2] = c2; c[3] = __shfl_sync(0xffffffffu, x0.w, wl);
                c[4] = __shfl_sync(0xffffffffu, x1.x, wl); c[5] = __shfl_sync(0xffffffffu, x1.y, wl);
                c[6] = __shfl_sync(0xffffffffu, x1.z, wl); c[7] = __shfl_sync(0xffffffffu, x1.w, wl);
                c[8] = __shfl_sync(0xffffffffu, x2.x, wl); c[9] = __shfl_sync(0xffffffffu, x2.y, wl); c[10] = c[11] = 0u;
                leader_allgather(smem_u32(&hot.xB[0][0]), 12, c, HB_XB);
                const bool vc = lane < CL;
                uint4 y0 = make_uint4(0u, 0xffffffffu, 0u, 0u), y1 = make_uint4(0u, 0u, 0u, 0u);
                uint2 y2 = make_uint2(0u, 0u);
                if (vc) {
                    y0 = *reinterpret_cast<const uint4 *>(&hot.xB[lane][0]); y1 = *reinterpret_cast<const uint4 *>(&hot.xB[lane][4]);
                    y2 = *reinterpret_cast<const uint2 *>(&hot.xB[lane][8]);
                }
                const unsigned top1k = __reduce_max_sync(0xffffffffu, (int)y0.y >= 0 ? y0.x : 0u);
                const int gj = __reduce_max_sync(0xffffffffu, ((int)y0.y >= 0 && y0.x == top1k) ? (int)y0.y : -1);
                const unsigned top2k = __reduce_max_sync(0xffffffffu, (int)y0.y == gj ? y0.z : ((int)y0.y >= 0 ? y0.x : 0u));
                const int gl = gj >= 0 ? __ffs(__ballot_sync(0xffffffffu, (int)y0.y == gj)) - 1 : 0;
                const int cj = (int)__shfl_sync(0xffffffffu, y0.w, gl);
                mg_j = mk64(__shfl_sync(0xffffffffu, y1.x, gl), __shfl_sync(0xffffffffu, y1.y, gl));
                k_ij = mk64(__shfl_sync(0xffffffffu, y1.z, gl), __shfl_sync(0xffffffffu, y1.w, gl));
                alpha_j = mk64(__shfl_sync(0xffffffffu, y2.x, gl), __shfl_sync(0xffffffffu, y2.y, gl));
                const bool tiny = FAST && top1k <= KEY_TINY;
                const int md = gj < 0 ? -1 : ((top1k - top2k <= BAND || tiny) ? 1 : 0);
                const unsigned th = (top1k > BAND && !tiny) ? top1k - BAND : 1u;
                if (lane == 0)
                    *reinterpret_cast<uint4 *>(&hot.resB1[0]) = make_uint4((unsigned)gj, (unsigned)cj, (unsigned)md, th);
                __syncwarp();
                nb_arrive(NB_RB1);
            } else { nb_arrive(NB_LB); nb_sync(NB_RB1); }
            const uint4 r = *reinterpret_cast<const uint4 *>(&hot.resB1[0]);
            pj = (int)r.x; col_j = (int)r.y; mode = (int)r.z; thrk = r.w;
            tick(4);
        }
        if (mode < 0) return true;                                               // Gmin_idx == -1
        if (mode == 1) {
            // ---- exact tie-break: libsvm's correctly rounded quotients for every element in the band (rare) ----
            double bestn = -CUDART_INF, mbv = 0.0;
            int bidx = -1, cbv = 0, sbv = 0;
            float kqb = 0.f;
#pragma unroll
            for (int k = 0; k < KPT; k++) {
                if (pos[k] < active) {
                    const int f = fl[k];
                    const double gd = __dsub_rn(gmax, m[k]);
                    if ((f & F_LOW) && gd > 0) {
                        if (approx_key(gd, kvi[k], colr[k]) >= thrk) {
                            const double quad = __dsub_rn(__dadd_rn(QDi, QDc(colr[k])), __dmul_rn(2.0, widen(kvi[k])));
                            const double g2 = __dmul_rn(gd, gd);
                            const double nod = quad > 0 ? __ddiv_rn(g2, quad) : __ddiv_rn(g2, TAU);   // == -obj_diff
                            const int cand = (pos[k] << IDX_SHIFT) | f;
                            if (nod > bestn || (nod == bestn && cand > bidx)) { bestn = nod; bidx = cand; cbv = colr[k]; sbv = k * NT + tid; kqb = kvi[k]; mbv = m[k]; }
                        }
                    }
                }
            }
            const unsigned long long key = dkey(bestn);
            const KArg w = warp_argmax((unsigned)(key >> 32), (unsigned)key, bidx);
            if (w.idx >= 0 ? bidx == w.idx : lane == 0) {
                store_record(hot.recX, cbv, sbv, kqb, mbv, w.hi, (unsigned)w.idx, w.lo, w.idx >= 0);
            }
            __syncwarp();
            if (warp == 0) {
                nb_sync(NB_LX);
                const bool v = lane < NW;
                uint4 x0 = make_uint4(0u, 0xffffffffu, 0u, 0u), x1 = make_uint4(0u, 0u, 0u, 0u);
                uint2 x2 = make_uint2(0u, 0u);
                if (v) {
                    x0 = *reinterpret_cast<const uint4 *>(&hot.recX[lane][0]); x1 = *reinterpret_cast<const uint4 *>(&hot.recX[lane][4]);
                    x2 = *reinterpret_cast<const uint2 *>(&hot.recX[lane][8]);
                }
                const KArg a = warp_argmax(x0.x, x0.z, (int)x0.y);
                const int wl = a.idx >= 0 ? __ffs(__ballot_sync(0xffffffffu, (int)x0.y == a.idx)) - 1 : 0;
                unsigned c[12];
                c[0] = a.hi; c[1] = (unsigned)a.idx; c[2] = a.lo; c[3] = __shfl_sync(0xffffffffu, x0.w, wl);
                c[4] = __shfl_sync(0xffffffffu, x1.x, wl); c[5] = __shfl_sync(0xffffffffu, x1.y, wl);
                c[6] = __shfl_sync(0xffffffffu, x1.z, wl); c[7] = __shfl_sync(0xffffffffu, x1.w, wl);
                c[8] = __shfl_sync(0xffffffffu, x2.x, wl); c[9] = __shfl_sync(0xffffffffu, x2.y, wl); c[10] = c[11] = 0u;
                leader_allgather(smem_u32(&hot.xX[0][0]), 12, c, HB_XX);
                const bool vc = lane < CL;
                uint4 y0 = make_uint4(0u, 0xffffffffu, 0u, 0u), y1 = make_uint4(0u, 0u, 0u, 0u);
                uint2 y2 = make_uint2(0u, 0u);
                if (vc) {
                    y0 = *reinterpret_cast<const uint4 *>(&hot.xX[lane][0]); y1 = *reinterpret_cast<const uint4 *>(&hot.xX[lane][4]);
                    y2 = *reinterpret_cast<const uint2 *>(&hot.xX[lane][8]);
                }
                const KArg g = warp_argmax(y0.x, y0.z, (int)y0.y);
                const int gl = g.idx >= 0 ? __ffs(__ballot_sync(0xffffffffu, (int)y0.y == g.idx)) - 1 : 0;   // >= 0: the approximate winner is in the band
                const int cj = (int)__shfl_sync(0xffffffffu, y0.w, gl);
                mg_j = mk64(__shfl_sync(0xffffffffu, y1.x, gl), __shfl_sync(0xffffffffu, y1.y, gl));
                k_ij = mk64(__shfl_sync(0xffffffffu, y1.z, gl), __shfl_sync(0xffffffffu, y1.w, gl));
                alpha_j = mk64(__shfl_sync(0xffffffffu, y2.x, gl), __shfl_sync(0xffffffffu, y2.y, gl));
                if (lane == 0)
                    *reinterpret_cast<uint2 *>(&hot.resX[0]) = make_uint2((unsigned)g.idx, (unsigned)cj);
                __syncwarp();
                nb_arrive(NB_RX);
            } else { nb_arrive(NB_LX); nb_sync(NB_RX); }
            const uint2 r = *reinterpret_cast<const uint2 *>(&hot.resX[0]);
            pj = (int)r.x; col_j = (int)r.y;
        }
        return false;
    };

    // ---------------- do_shrinking (svm.cpp:1070-1129) ----------------
    // Gmax1 = max{m : I_up}, Gmax2 = max{-m : I_low}; be_shrunk = (!up && m > Gmax1) || (!low && -m > Gmax2)
    auto do_shrink = [&]() {
        double g1 = -CUDART_INF, g2 = -CUDART_INF;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            if (pos[k] < active) {
                if (fl[k] & F_UP) g1 = fmax(g1, m[k]);
                if (fl[k] & F_LOW) g2 = fmax(g2, -m[k]);
            }
        }
        g1 = block_max<NT>(g1, red.dm);
        g2 = block_max<NT>(g2, red.dm2);
        {
            unsigned v[XW] = {0};
            v[0] = lo32(g1); v[1] = hi32(g1); v[2] = lo32(g2); v[3] = hi32(g2);
            const unsigned (*r)[XW] = exchange(v);
#pragma unroll
            for (int c = 0; c < CL; c++) { g1 = fmax(g1, mk64(r[c][0], r[c][1])); g2 = fmax(g2, mk64(r[c][2], r[c][3])); }
        }
        if (!unshrink && __dadd_rn(g1, g2) <= __dmul_rn(eps, 10.0)) {
            unshrink = true;
            rebuild_gradient();
            active = l;
        }
        bool mark[KPT];
        int keep_local = 0;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            mark[k] = false;
            if (pos[k] < active) {
                const int f = fl[k];
                mark[k] = (!(f & F_UP) && m[k] > g1) || (!(f & F_LOW) && -m[k] > g2);
                keep_local += mark[k] ? 0 : 1;
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
        {
            unsigned v[XW] = {0};
            v[0] = (unsigned)na;
            const unsigned (*r)[XW] = exchange(v);
            na = 0;
#pragma unroll
            for (int c = 0; c < CL; c++) na += (int)r[c][0];
        }
        if (na != active) {
            // libsvm's two-pointer sweep pairs the k-th marked position below na (ascending) with the k-th unmarked
            // position at/above na (descending).  Marks are all-gathered by position; every CTA derives the same map.
#pragma unroll
            for (int k = 0; k < KPT; k++) {
                if (pos[k] < active) {
#pragma unroll
                    for (int c = 0; c < CL; c++) *cluster.map_shared_rank(mk + pos[k], c) = mark[k] ? 1 : 0;
                }
            }
            cluster.sync();
            int *plist = lists, *qlist = lists + lhalf;
            int np = 0, nq = 0;
            for (int base = 0; base < na; base += NT) {
                const int t = base + tid;
                const bool pr = t < na && mk[t];
                int tot;
                const int r = block_rank<NT>(pr, red.cnt, tot);
                if (pr) plist[np + r] = t;
                np += tot;
            }
            for (int base = na; base < active; base += NT) {
                const int t = base + tid;
                const bool pr = t < active && !mk[t];
                int tot;
                const int r = block_rank<NT>(pr, red.cnt, tot);
                if (pr) qlist[nq + r] = t;
                nq += tot;
            }
            __syncthreads();
            for (int r = tid; r < np; r += NT) {                 // np == nq; disjoint pairs
                const int p = plist[r], q = qlist[np - 1 - r];
                swapmap[p] = (unsigned short)q; swapmap[q] = (unsigned short)p;
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < KPT; k++) {
                if (pos[k] < active) {
                    const bool moved = pos[k] < na ? mark[k] : !mark[k];
                    if (moved) pos[k] = (int)swapmap[pos[k]];
                }
            }
            active = na;
            // mk / lists / swapmap are next written 1000 iterations (thousands of exchanges) later: no barrier needed here
        }
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
            local_scan();
            if (select()) break;
            counter = 1;
        }
        ++iter;

        const int i = pi >> IDX_SHIFT, j = pj >> IDX_SHIFT;
        const float *__restrict__ Kj = K + (size_t)col_j * ldk;
        float kvj[KPT];
#pragma unroll
        for (int k = 0; k < KPT; k++) kvj[k] = pos[k] < active ? __ldg(Kj + colr[k]) : 0.f;     // in flight during the scalar update
        if (warp == 0) {                                         // leader: analytic two-variable update, published to the workers
            const bool yi = (pi & F_YPOS) != 0, yj = (pj & F_YPOS) != 0;
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
            if (lane == 0) {
                const double dai = __dsub_rn(ai, alpha_i), daj = __dsub_rn(aj, alpha_j);
                const double av = yi ? -dai : dai, bv = yj ? -daj : daj;       // a = -y_i dalpha_i, b = -y_j dalpha_j
                const int si = ai >= Ci ? ST_UPPER : (ai <= 0 ? ST_LOWER : ST_FREE), sj = aj >= Cj ? ST_UPPER : (aj <= 0 ? ST_LOWER : ST_FREE);
                *reinterpret_cast<uint4 *>(&hot.resB2[0]) = make_uint4(lo32(av), hi32(av), lo32(bv), hi32(bv));
                *reinterpret_cast<uint4 *>(&hot.resB2[4]) = make_uint4(lo32(ai), hi32(ai), lo32(aj), hi32(aj));
                *reinterpret_cast<uint2 *>(&hot.resB2[8]) = make_uint2((unsigned)si, (unsigned)sj);
            }
            __syncwarp();
            nb_arrive(NB_RB2);
        } else nb_sync(NB_RB2);
        tick(5);
        const uint4 u0 = *reinterpret_cast<const uint4 *>(&hot.resB2[0]);
        const uint4 u1 = *reinterpret_cast<const uint4 *>(&hot.resB2[4]);
        const uint2 u2 = *reinterpret_cast<const uint2 *>(&hot.resB2[8]);
        const double a = mk64(u0.x, u0.y), b = mk64(u0.z, u0.w);
        const int sti = (int)u2.x, stj = (int)u2.y;
        tick(6);
        // the owners of i and j take the new alpha and status FIRST: the fused scan below must see the new sets
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            if (pos[k] == i) { alpha[k * NT + tid] = mk64(u1.x, u1.y); fl[k] = mkflags((pi & F_YPOS) != 0, sti); }
            if (pos[k] == j) { alpha[k * NT + tid] = mk64(u1.z, u1.w); fl[k] = mkflags((pj & F_YPOS) != 0, stj); }
        }
        // m update over the active set (svm.cpp:866-872), fused with the next iteration's local scan
        la = -CUDART_INF; lm = CUDART_INF; la_pos = -1;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            if (pos[k] < active) {
                m[k] = __dadd_rn(m[k], __dadd_rn(__dmul_rn(widen(kvi[k]), a), __dmul_rn(widen(kvj[k]), b)));
                scan_elem(k);
            }
        }
        scan_valid = true;
        tick(7);
        // G_bar over all l when a bound status flips (svm.cpp:876-905): i first, then j
        const bool need_i = use_gbar && (((pi & 3) == ST_UPPER) != (sti == ST_UPPER));
        const bool need_j = use_gbar && (((pj & 3) == ST_UPPER) != (stj == ST_UPPER));
        if (need_i || need_j) {
            // Gbar -= C Q_i (was upper) / += C Q_i (became upper)  <=>  mbar += fl(c K_i), c = +/- y_i C
            const float *__restrict__ Ki = K + (size_t)col_i * ldk;
            const double Cmi = (pi & F_YPOS) ? Cc : Cneg, Cmj = (pj & F_YPOS) ? Cc : Cneg;
            const double ci = (((pi & 3) == ST_UPPER) == ((pi & F_YPOS) != 0)) ? Cmi : -Cmi;
            const double cj = (((pj & 3) == ST_UPPER) == ((pj & F_YPOS) != 0)) ? Cmj : -Cmj;
#pragma unroll
            for (int k = 0; k < KPT; k++) {
                if (pos[k] != NOPOS) {
                    const bool act = pos[k] < active;
                    double gb = mGbar[k * NT + tid];
                    if (need_i) gb = __dadd_rn(gb, __dmul_rn(ci, widen(act ? kvi[k] : __ldg(Ki + colr[k]))));
                    if (need_j) gb = __dadd_rn(gb, __dmul_rn(cj, widen(act ? kvj[k] : __ldg(Kj + colr[k]))));
                    mGbar[k * NT + tid] = gb;
                }
            }
        }
        tick(8);
    }


    // ---------------- calculate_rho (svm.cpp:1131-1168): sequential float64 sum in ascending position ----------------
    cluster.sync();
#pragma unroll
    for (int k = 0; k < KPT; k++) {
        if (pos[k] < active) { gscratch[pos[k]] = -m[k]; scratch[pos[k]] = fl[k]; }     // y*G and flags, by position
    }
    __threadfence();
    cluster.sync();
    if (rank == 0 && tid == 0) {
        int nfree = 0;
        double ub = CUDART_INF, lb = -CUDART_INF, sum = 0;
#pragma unroll 8
        for (int t = 0; t < active; t++) {
            const int f = __ldcg(scratch + t);
            const double yG = __ldcg(gscratch + t);
            if ((f & 3) == ST_UPPER) { if (!(f & F_YPOS)) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
            else if ((f & 3) == ST_LOWER) { if (f & F_YPOS) ub = fmin(ub, yG); else lb = fmax(lb, yG); }
            else { ++nfree; sum = __dadd_rn(sum, yG); }
        }
        *Pp->out_rho = nfree > 0 ? __ddiv_rn(sum, (double)nfree) : __ddiv_rn(__dadd_rn(ub, lb), 2.0);
    }
    // coefficients alpha*y scattered by dataset row (svm.cpp:922-925, :1641-1642); SV counts
    int nsv = 0, nbsv = 0;
    {
        double *__restrict__ coef = Pp->coef;
#pragma unroll
        for (int k = 0; k < KPT; k++) {
            if (pos[k] != NOPOS) {
                const double av = alpha[k * NT + tid];
                coef[colr[k]] = (fl[k] & F_YPOS) ? av : -av;
                nsv += av > 0;
                nbsv += av >= ((fl[k] & F_YPOS) ? Cc : Cneg);
            }
        }
    }
#pragma unroll
    for (int s = 16; s; s >>= 1) {
        nsv += __shfl_xor_sync(0xffffffffu, nsv, s);
        nbsv += __shfl_xor_sync(0xffffffffu, nbsv, s);
    }
    __syncthreads();
    if (lane == 0) { red.cnt[warp] = nsv; red.a_idx[warp] = nbsv; }
    __syncthreads();
    {
        int s = 0, bs = 0;
        for (int w = 0; w < NW; w++) { s += red.cnt[w]; bs += red.a_idx[w]; }
        unsigned v[XW] = {0};
        v[0] = (unsigned)s; v[1] = (unsigned)bs;
        const unsigned (*r)[XW] = exchange(v);
        if (rank == 0 && tid == 0) {
            int ts = 0, tb = 0;
#pragma unroll
            for (int c = 0; c < CL; c++) { ts += (int)r[c][0]; tb += (int)r[c][1]; }
            int *info = Pp->out_info;
            info[0] = iter; info[1] = timed_out; info[2] = ts; info[3] = tb;
            unsigned long long t_end;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_end));
            unsigned long long *ns = Pp->out_ns;
            ns[0] = t_start; ns[1] = t_end;
            if constexpr (PROF)
                for (int q = 0; q < 10; q++) ns[2 + q] = (unsigned long long)prof[q];
        }
    }
    cluster.sync();                                              // no CTA may exit while a peer can still write its shared memory
}

template <int NT, int KPT, int CL, bool FAST, bool PROF>
cudaError_t launch_co(const SmoProblem *probs, const int *order, int n_prob, int lmax, cudaStream_t st)
{
    constexpr int LCAP = NT * KPT;
    // alpha + mbar per owned element, then 7 bytes per POSITION of cold-path scratch; padded to a whole SM's worth so a
    // cluster CTA never shares its SM (a resident small CTA would keep a full-SM single-CTA solver from being scheduled)
    size_t smem = (size_t)LCAP * 16 + (size_t)lmax * 7 + 64;
    if (smem < 160 * 1024) smem = 160 * 1024;
    auto kern = smo_colown_kernel<NT, KPT, CL, FAST, PROF>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(n_prob * CL));
    cfg.blockDim = dim3(NT);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, probs, order);
}

template <int NT, int KPT, int CL>
cudaError_t launch_co_f(const SmoProblem *p, const int *o, int n, int lmax, bool fast, cudaStream_t st)
{
    if (prof_enabled()) return fast ? launch_co<NT, KPT, CL, true, true>(p, o, n, lmax, st) : launch_co<NT, KPT, CL, false, true>(p, o, n, lmax, st);
    return fast ? launch_co<NT, KPT, CL, true, false>(p, o, n, lmax, st) : launch_co<NT, KPT, CL, false, false>(p, o, n, lmax, st);
}

}  // namespace

namespace {
__global__ void delay_kernel(unsigned ns)
{
    unsigned long long t0, t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    do { __nanosleep(1000); asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); } while (t - t0 < ns);
}
}  // namespace

void launch_delay(unsigned ns, cudaStream_t st) { delay_kernel<<<1, 1, 0, st>>>(ns); }

// Largest sub-problem a column-owner cluster launch of size cl supports (0: unsupported cluster size)
int smo_colown_max_rows(int cl) { return cl == 2 ? 8192 : ((cl == 4 || cl == 8) ? 16384 : 0); }

// Shape = (threads per CTA) x (elements per thread) x (CTAs per problem).
cudaError_t launch_smo_colown(const SmoProblem *d_probs, const int *d_order, int n_prob, int lmax, int cl, bool fast, cudaStream_t st)
{
    if (n_prob <= 0) return cudaSuccess;
    if (lmax > smo_colown_max_rows(cl)) return cudaErrorInvalidValue;
    // 512 threads at most: the register-resident state needs more than the 64 registers a 1024-thread CTA leaves a thread
    if (cl == 2) return launch_co_f<512, 8, 2>(d_probs, d_order, n_prob, lmax, fast, st);
    if (cl == 4) {
        if (lmax > 8192) return launch_co_f<512, 8, 4>(d_probs, d_order, n_prob, lmax, fast, st);
        return launch_co_f<512, 4, 4>(d_probs, d_order, n_prob, lmax, fast, st);
    }
    if (cl == 8) {
        if (lmax > 8192) return launch_co_f<512, 4, 8>(d_probs, d_order, n_prob, lmax, fast, st);
        return launch_co_f<256, 4, 8>(d_probs, d_order, n_prob, lmax, fast, st);
    }
    return cudaErrorInvalidValue;
}
