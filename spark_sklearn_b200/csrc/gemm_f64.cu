// gemm_f64.cu -- batched float64 contraction C[M][N] = sum_k A[M][k] B[N][k] on the FP64 tensor cores (DMMA).
//
// liblinear's TRON solver works in float64 and scikit-learn upcasts X to float64, so the two products of every TRON round
// (linsvc.cu) cannot go through the 3xTF32 path of gemm_tc.cu, which is float32-faithful only: a margin moved by 1e-7
// relative moves rows across the hinge z < 1 and changes TRON's accept and stop tests.  Every product and every sum here
// is a float64 operation (mma.sync m8n8k4 .f64: fused multiply-add in float64), so the result differs from a sequential
// float64 dot product by the rounding of a reordered sum only.
//
// Tiling: a 64x64 block tile of C per CTA (4 warps, 32x32 each = 4x4 m8n8 fragments), K in steps of 16 staged through
// shared memory with a register prefetch of the next step.  Split-K: blockIdx.z takes the k range
// [z*kchunk, min(K, (z+1)*kchunk)) and writes its partial to C + z*c_chunk_stride; the caller sums the partials in a
// fixed order, so results are deterministic.
#include "common.cuh"
#include <algorithm>

namespace {

constexpr int BM = 64, BN = 64, BK = 16, SLD = BK + 1;   // odd shared-memory row stride: no bank conflicts on fragment loads

__device__ __forceinline__ void dmma(double &c0, double &c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(128) gemm_nt_f64_kernel(const double *__restrict__ A, int64_t lda, const double *__restrict__ B,
                                                          int64_t ldb, double *__restrict__ C, int64_t ldc, int K, int kchunk,
                                                          int64_t c_chunk_stride)
{
    __shared__ double As[BM * SLD], Bs[BN * SLD];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 1, wn = warp & 1;
    const int64_t m0 = (int64_t)blockIdx.y * BM, n0 = (int64_t)blockIdx.x * BN;
    const int k_begin = blockIdx.z * kchunk, k_end = min(K, k_begin + kchunk);
    C += (int64_t)blockIdx.z * c_chunk_stride;

    double acc[4][4][2];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j][0] = acc[i][j][1] = 0.0;

    // each thread stages 8 elements of each operand per K step: row (tid + 128 e) / 16, column (tid + 128 e) % 16
    double ra[8], rb[8];
    auto load = [&](int k0) {
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int idx = tid + 128 * e, r = idx >> 4, c = idx & 15;
            ra[e] = A[(m0 + r) * lda + k0 + c];
            rb[e] = B[(n0 + r) * ldb + k0 + c];
        }
    };
    if (k_begin < k_end) load(k_begin);
    for (int k0 = k_begin; k0 < k_end; k0 += BK) {
        __syncthreads();
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int idx = tid + 128 * e, r = idx >> 4, c = idx & 15;
            As[r * SLD + c] = ra[e];
            Bs[r * SLD + c] = rb[e];
        }
        __syncthreads();
        if (k0 + BK < k_end) load(k0 + BK);
#pragma unroll
        for (int kk = 0; kk < BK; kk += 4) {
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) a[i] = As[(wm * 32 + i * 8 + (lane >> 2)) * SLD + kk + (lane & 3)];
#pragma unroll
            for (int j = 0; j < 4; j++) b[j] = Bs[(wn * 32 + j * 8 + (lane >> 2)) * SLD + kk + (lane & 3)];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) dmma(acc[i][j][0], acc[i][j][1], a[i], b[j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int64_t row = m0 + wm * 32 + i * 8 + (lane >> 2), col = n0 + wn * 32 + j * 8 + (lane & 3) * 2;
            *reinterpret_cast<double2 *>(&C[row * ldc + col]) = make_double2(acc[i][j][0], acc[i][j][1]);
        }
}

}  // namespace

cudaError_t launch_gemm_nt_f64(const double *A, int64_t lda, const double *B, int64_t ldb, double *C, int64_t ldc, int M, int N,
                               int K, int kchunk, int64_t c_chunk_stride, cudaStream_t st)
{
    if (M % BM || N % BN || K % BK || kchunk % BK || kchunk <= 0 || ldc % 2) return cudaErrorInvalidValue;
    dim3 grid((unsigned)(N / BN), (unsigned)(M / BM), (unsigned)((K + kchunk - 1) / kchunk));
    gemm_nt_f64_kernel<<<grid, 128, 0, st>>>(A, lda, B, ldb, C, ldc, K, kchunk, c_chunk_stride);
    return cudaGetLastError();
}

extern "C" int gs_debug_gemm_f64(gs_handle *h, const double *A, int32_t M, const double *B, int32_t N, int32_t K, int32_t kchunk,
                                 double *C)
{
    if (!h) return GS_ERR_ARG;
    if (!A || !B || !C || M <= 0 || N <= 0 || K <= 0 || kchunk <= 0 || kchunk % BK) {
        gs_set_error(h, "gs_debug_gemm_f64: bad arguments (kchunk must be a positive multiple of 16)");
        return GS_ERR_ARG;
    }
    GS_CUDA(cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    // M, N padded to whole 64x64 tiles and K to whole 16-wide steps with zeros; split-K into kchunk-long chunks (the last one
    // ragged) and the fixed-order in-place sum of the partials, as the TRON gradient runs it
    const int Mp = (M + BM - 1) / BM * BM, Np = (N + BN - 1) / BN * BN, Kp = (K + BK - 1) / BK * BK;
    const int nchunk = (Kp + kchunk - 1) / kchunk;
    DevBuf a, b, c;
    GS_CUDA(a.reserve((size_t)Mp * Kp * 8)); GS_CUDA(b.reserve((size_t)Np * Kp * 8));
    GS_CUDA(c.reserve((size_t)nchunk * Mp * Np * 8));
    GS_CUDA(cudaMemsetAsync(a.p, 0, (size_t)Mp * Kp * 8, st));
    GS_CUDA(cudaMemsetAsync(b.p, 0, (size_t)Np * Kp * 8, st));
    GS_CUDA(cudaMemcpy2DAsync(a.p, (size_t)Kp * 8, A, (size_t)K * 8, (size_t)K * 8, M, cudaMemcpyHostToDevice, st));
    GS_CUDA(cudaMemcpy2DAsync(b.p, (size_t)Kp * 8, B, (size_t)K * 8, (size_t)K * 8, N, cudaMemcpyHostToDevice, st));
    GS_CUDA(launch_gemm_nt_f64(a.as<double>(), Kp, b.as<double>(), Kp, c.as<double>(), Np, Mp, Np, Kp, kchunk, (int64_t)Mp * Np, st));
    GS_CUDA(launch_sum_partials_f64(c.as<double>(), nchunk, (int64_t)Mp * Np, c.as<double>(), st));
    GS_CUDA(cudaMemcpy2DAsync(C, (size_t)N * 8, c.p, (size_t)Np * 8, (size_t)N * 8, M, cudaMemcpyDeviceToHost, st));
    GS_CUDA(cudaStreamSynchronize(st));
    a.release(); b.release(); c.release();
    return GS_OK;
}

namespace {
// out[i] = partial[0][i] + partial[1][i] + ... in chunk order (in place into partial[0] is allowed)
__global__ void sum_partials_f64_kernel(const double *partial, int n_chunks, int64_t per, double *out)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.x * blockDim.x) {
        double s = partial[i];
        for (int q = 1; q < n_chunks; q++) s += partial[(int64_t)q * per + i];
        out[i] = s;
    }
}
}  // namespace

cudaError_t launch_sum_partials_f64(const double *partial, int n_chunks, int64_t per, double *out, cudaStream_t st)
{
    const int64_t blocks = std::min<int64_t>((per + 255) / 256, 4096);
    sum_partials_f64_kernel<<<(unsigned)blocks, 256, 0, st>>>(partial, n_chunks, per, out);
    return cudaGetLastError();
}
