// sequential.cuh -- what the sample-by-sample solvers (sgd.cu, sag.cu) share: scikit-learn's xorshift32, the sum made in
// feature order, float32 rounding of a double, and the half-binomial gradient, each rounded operation by operation.
#pragma once
#include <stdint.h>

// a float operation made in double and rounded once gives the float result (53 >= 2 x 24 + 2)
template <typename T> __host__ __device__ __forceinline__ double rnd(double v);
template <> __host__ __device__ __forceinline__ double rnd<double>(double v) { return v; }
template <> __host__ __device__ __forceinline__ double rnd<float>(double v) { return (double)(float)v; }

// utils/_random.pxd our_rand_r: xorshift32 (a zero seed becomes DEFAULT_SEED = 1), reduced to [0, 2^31)
__host__ __device__ __forceinline__ uint32_t our_rand_r(uint32_t &s)
{
    if (s == 0) s = 1u;
    s ^= s << 13;
    s ^= s >> 17;
    s ^= s << 5;
    return s & 0x7fffffffu;
}

// v[0], v[stride], ... v[(n - 1) stride] summed in that order, the sum rounded to T after every addition (broadcast reads
// when every lane calls it)
template <typename T>
__device__ __forceinline__ double seq_sum(const double *v, int n, int stride)
{
    double a = 0.0;
#pragma unroll 8
    for (int j = 0; j < n; j++) a = rnd<T>(__dadd_rn(a, v[(size_t)j * stride]));
    return a;
}

// _loss.pyx.tp cgradient_half_binomial: expit(p) - y
__device__ __forceinline__ double grad_half_binomial(double y, double p)
{
    if (p > -37) { const double e = exp(-p); return __ddiv_rn(__dsub_rn(__dsub_rn(1.0, y), __dmul_rn(y, e)), __dadd_rn(1.0, e)); }
    return __dsub_rn(exp(p), y);
}
