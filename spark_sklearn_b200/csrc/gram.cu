// gram.cu -- float64 Gram matrix and float32 kernel-matrix materialisation (sm_90a).
//
// Why float64 here: libsvm (sklearn svm.cpp:336-347, 1439-1449) evaluates every kernel entry in
// float64 from float64 features and only then rounds to float32 (Qfloat).  X arrives as float32,
// so each product x_ik*x_jk is EXACT in float64 and a float64 accumulation differs from libsvm's
// BLAS ddot only in summation order (~1e-16 relative); after the exp and the float32 rounding the
// stored Q entries agree with libsvm's on all but ~2^-29 of the entries.  That is what lets the
// SMO kernel reproduce libsvm's iterate sequence, and therefore its scores, bit for bit.  A
// tensor-core (wgmma) Gram cannot do this: fp32 accumulation perturbs every entry by a few ulp.
//
// gram_f64_kernel: S = X X^T, 128x128 output tile per CTA, 8x8 float64 micro-tile per thread,
// upper-triangular tiles only (mirror-written), operands converted to float64 once when staged
// in shared memory (fp32->fp64 conversion runs at 1/4 of the DFMA rate, so never in the inner loop).
#include "common.cuh"

namespace {

constexpr int TM = 128;       // tile rows/cols
constexpr int TK = 16;        // k-slab
constexpr int PAD = 2;        // doubles of padding per smem row

template <typename T>
__global__ void __launch_bounds__(256, 1)
gram_f64_kernel(const T *__restrict__ X, int n, int d, double *__restrict__ S, double *__restrict__ xsq)
{
    __shared__ __align__(16) double As[TK][TM + PAD];
    __shared__ __align__(16) double Bs[TK][TM + PAD];

    // decode upper-triangular tile index -> (bi <= bj)
    const int NTILE = (n + TM - 1) / TM;
    int rem = blockIdx.x, bi = 0;
    while (rem >= NTILE - bi) { rem -= NTILE - bi; ++bi; }
    const int bj = bi + rem;
    const int i0 = bi * TM, j0 = bj * TM;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;

    double acc[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int c = 0; c < 8; c++) acc[r][c] = 0.0;

    // each thread stages 2x4 consecutive k-values of one row for A and for B
    const int lrow0 = tid >> 2, lk = (tid & 3) * 4;          // rows lrow0 and lrow0+64
    const bool vec = (d & 3) == 0 && sizeof(T) == 4;
    T pa[2][4], pb[2][4];

    auto fetch = [&](int k0) {
#pragma unroll
        for (int s = 0; s < 2; s++) {
            const int ra = i0 + lrow0 + 64 * s, rb = j0 + lrow0 + 64 * s, k = k0 + lk;
            if (vec && k + 3 < d) {
                float4 va = ra < n ? *reinterpret_cast<const float4 *>((const float *)X + (size_t)ra * d + k) : make_float4(0, 0, 0, 0);
                float4 vb = rb < n ? *reinterpret_cast<const float4 *>((const float *)X + (size_t)rb * d + k) : make_float4(0, 0, 0, 0);
                pa[s][0] = va.x; pa[s][1] = va.y; pa[s][2] = va.z; pa[s][3] = va.w;
                pb[s][0] = vb.x; pb[s][1] = vb.y; pb[s][2] = vb.z; pb[s][3] = vb.w;
            } else {
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    pa[s][e] = (ra < n && k + e < d) ? X[(size_t)ra * d + k + e] : T(0);
                    pb[s][e] = (rb < n && k + e < d) ? X[(size_t)rb * d + k + e] : T(0);
                }
            }
        }
    };

    fetch(0);
    for (int k0 = 0; k0 < d; k0 += TK) {
#pragma unroll
        for (int s = 0; s < 2; s++)
#pragma unroll
            for (int e = 0; e < 4; e++) {
                As[lk + e][lrow0 + 64 * s] = (double)pa[s][e];
                Bs[lk + e][lrow0 + 64 * s] = (double)pb[s][e];
            }
        __syncthreads();
        if (k0 + TK < d) fetch(k0 + TK);                      // register prefetch of the next slab
#pragma unroll
        for (int k = 0; k < TK; k++) {
            double a[8], b[8];
#pragma unroll
            for (int r = 0; r < 8; r += 2) {
                double2 v = *reinterpret_cast<const double2 *>(&As[k][ty * 8 + r]);
                a[r] = v.x; a[r + 1] = v.y;
                double2 w = *reinterpret_cast<const double2 *>(&Bs[k][tx * 8 + r]);
                b[r] = w.x; b[r + 1] = w.y;
            }
#pragma unroll
            for (int r = 0; r < 8; r++)
#pragma unroll
                for (int c = 0; c < 8; c++) acc[r][c] = fma(a[r], b[c], acc[r][c]);   // product exact
        }
        __syncthreads();
    }

#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int gi = i0 + ty * 8 + r;
        if (gi >= n) continue;
#pragma unroll
        for (int c = 0; c < 8; c++) {
            const int gj = j0 + tx * 8 + c;
            if (gj >= n) continue;
            S[(size_t)gi * n + gj] = acc[r][c];
            if (bi != bj) S[(size_t)gj * n + gi] = acc[r][c];
            else if (gi == gj) xsq[gi] = acc[r][c];
        }
    }
}

// K[r][c] = (float) kernel(r, c).  rbf: exp(-gamma*((xsq_r + xsq_c) - 2*S_rc)) -- the evaluation order
// of svm.cpp:344-347, each operation individually rounded (no contraction); linear: S_rc.
__global__ void __launch_bounds__(256)
kernel_matrix_kernel(const double *__restrict__ S, const double *__restrict__ xsq, int n, int kernel, double gamma,
                     float *__restrict__ K, int64_t ldk, int *__restrict__ special)
{
    bool odd = false;
    const int r = blockIdx.y;
    const double xr = xsq[r];
    const double ng = -gamma;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const double s = S[(size_t)r * n + c];
        double v;
        if (kernel == GS_KERNEL_RBF) {
            const double d2 = __dsub_rn(__dadd_rn(xr, xsq[c]), __dmul_rn(2.0, s));
            v = exp(__dmul_rn(ng, d2));
        } else {
            v = s;
        }
        const float kf = (float)v;
        K[(size_t)r * ldk + c] = kf;
        const unsigned e = __float_as_uint(kf) >> 23;           // sign + exponent: positive normal <=> 1..254
        odd |= (e == 0u || e >= 255u);
    }
    if (special && __any_sync(0xffffffffu, odd) && (threadIdx.x & 31) == 0) atomicOr(special, 1);
}

// tensor-core mode: widen the float32 Gram of gemm_tc.cu to the float64 layout the other kernels read, taking the
// diagonal as the squared norms; the two triangles of a tensor-core result can differ in the last bit, so the
// upper one is mirrored to keep K symmetric exactly as libsvm's is.
__global__ void widen_gram_kernel(const float *__restrict__ S32, int n, int64_t ld32, double *__restrict__ S, double *__restrict__ xsq)
{
    const int r = blockIdx.y;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
        const float v = r <= c ? S32[(size_t)r * ld32 + c] : S32[(size_t)c * ld32 + r];
        S[(size_t)r * n + c] = (double)v;
        if (r == c) xsq[r] = (double)v;
    }
}

}  // namespace

cudaError_t launch_widen_gram(const float *S32, int n, int64_t ld32, double *S, double *xsq, cudaStream_t st)
{
    dim3 grid((n + 1023) / 1024, n);
    widen_gram_kernel<<<grid, 256, 0, st>>>(S32, n, ld32, S, xsq);
    return cudaGetLastError();
}

cudaError_t launch_gram_f64(const void *X, int x_dtype, int n, int d, double *S, double *xsq, cudaStream_t st)
{
    const int T = (n + TM - 1) / TM;
    const int tiles = T * (T + 1) / 2;
    if (x_dtype == GS_F64) gram_f64_kernel<double><<<tiles, 256, 0, st>>>((const double *)X, n, d, S, xsq);
    else gram_f64_kernel<float><<<tiles, 256, 0, st>>>((const float *)X, n, d, S, xsq);
    return cudaGetLastError();
}

cudaError_t launch_kernel_matrix(const double *S, const double *xsq, int n, int kernel, double gamma,
                                 float *K, int64_t ldk, int *special, cudaStream_t st)
{
    dim3 grid((n + 1023) / 1024, n);
    if (grid.x < 1) grid.x = 1;
    kernel_matrix_kernel<<<grid, 256, 0, st>>>(S, xsq, n, kernel, gamma, K, ldk, special);
    return cudaGetLastError();
}
