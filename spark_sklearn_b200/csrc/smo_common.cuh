// smo_common.cuh -- helpers shared by the position-owned (smo.cu), slot-layout (smo_lean.cu) and cluster (smo_colown.cu)
// SMO kernels.
#pragma once
#include "common.cuh"
#include <cstdlib>
#include <math_constants.h>

namespace smo {

constexpr double TAU = 1e-12;
constexpr int ST_LOWER = 0, ST_UPPER = 1, ST_FREE = 2;
constexpr int F_YPOS = 4, F_UP = 8, F_LOW = 16, F_MARK = 32;
constexpr int IDX_SHIFT = 5;                 // packed index = (position << 5) | (flags & 31)
constexpr int SAFETY_MAX_ITER = 10000000;    // max_iter=-1 is "no limit" in libsvm; bound a runaway solve

// B200GS_SMO_PROF=1 launches the PROF instances: per-phase cycle counters of every sub-problem in out_ns[2..] (a
// diagnostic: the iterates are the same)
inline bool prof_enabled()
{
    const char *e = getenv("B200GS_SMO_PROF");
    return e && atoi(e) != 0;
}

__device__ __forceinline__ int mkflags(bool ypos, int st)
{
    const bool up = ypos ? st != ST_UPPER : st != ST_LOWER;     // I_up  membership (svm.cpp:964-978)
    const bool low = ypos ? st != ST_LOWER : st != ST_UPPER;    // I_low membership (svm.cpp:986-1037)
    return st | (ypos ? F_YPOS : 0) | (up ? F_UP : 0) | (low ? F_LOW : 0);
}

// order-preserving map double -> uint64 (larger double <=> larger key) and back
__device__ __forceinline__ unsigned long long dkey(double x)
{
    const long long u = __double_as_longlong(x);
    return (unsigned long long)u ^ ((unsigned long long)(u >> 63) | 0x8000000000000000ull);
}
__device__ __forceinline__ double dkey_inv(unsigned long long k)
{
    return __longlong_as_double((long long)(k ^ ((k >> 63) ? 0x8000000000000000ull : ~0ull)));
}

// exact float -> double widening on the integer pipe; zero/denormal/inf/nan take the F2F path
__device__ __forceinline__ double f2d(float x)
{
    const unsigned u = __float_as_uint(x);
    const unsigned e = u & 0x7f800000u;
    if (__builtin_expect(e == 0u || e == 0x7f800000u, 0)) return (double)x;
    const unsigned hi = (u & 0x80000000u) | (((u & 0x7fffffffu) >> 3) + 0x38000000u);
    return __hiloint2double((int)hi, (int)(u << 29));
}

__device__ __forceinline__ double rcp_approx(double x)
{
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    return r;
}

struct KArg { unsigned hi, lo; int idx; };

// warp arg-max over (64-bit key, index): largest key, ties -> largest index.  3 REDUX.
__device__ __forceinline__ KArg warp_argmax(unsigned hi, unsigned lo, int idx)
{
    KArg r;
    r.hi = __reduce_max_sync(0xffffffffu, hi);
    r.lo = __reduce_max_sync(0xffffffffu, hi == r.hi ? lo : 0u);
    r.idx = __reduce_max_sync(0xffffffffu, (hi == r.hi && lo == r.lo) ? idx : -1);
    return r;
}
__device__ __forceinline__ unsigned long long warp_keymax(unsigned long long k)
{
    const unsigned hi = (unsigned)(k >> 32), lo = (unsigned)k;
    const unsigned mh = __reduce_max_sync(0xffffffffu, hi);
    const unsigned ml = __reduce_max_sync(0xffffffffu, hi == mh ? lo : 0u);
    return ((unsigned long long)mh << 32) | ml;
}

struct Red {            // static shared scratch; NW <= 32 warps
    unsigned a_hi[32], a_lo[32]; int a_idx[32];                 // phase A partials (arg-max m over I_up)
    unsigned m_hi[32], m_lo[32];                                // Gmax2 partials (max -m over I_low)
    unsigned b_hi[32], b_lo[32]; int b_idx[32];                 // phase B partials (approximate arg-max)
    unsigned t_hi[32], t_lo[32];                                // phase B runner-up partials
    unsigned x_hi[32], x_lo[32]; int x_idx[32];                 // exact tie-break partials (rare path)
    double pl_mg[32], pl_kv[32], pl_alpha[32];                  // payload of each warp's winner
    double bc_d[4]; int bc_i[4];                                // scalars broadcast by warp 0
    double dm[32], dm2[32]; int cnt[32];                        // cold-path reductions
};

template <int NT>
__device__ __forceinline__ double block_max(double v, double *buf)
{
#pragma unroll
    for (int m = 16; m; m >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, m));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) buf[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = -CUDART_INF;
#pragma unroll
    for (int w = 0; w < NT / 32; w++) r = fmax(r, buf[w]);
    return r;
}

// exclusive block scan of a predicate over the threads (position order); returns rank and total
template <int NT>
__device__ __forceinline__ int block_rank(bool pred, int *cnt, int &total)
{
    const unsigned b = __ballot_sync(0xffffffffu, pred);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) cnt[w] = __popc(b);
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < NT / 32; i++) {
        const int c = cnt[i];
        if (i < w) base += c;
        tot += c;
    }
    total = tot;
    return base + __popc(b & ((1u << lane) - 1u));
}


}  // namespace smo
