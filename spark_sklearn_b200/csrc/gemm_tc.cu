// gemm_tc.cu -- C[M][N] = sum_k A[M][k] * B[N][k]  ("NT", both operands K-major) on the Hopper tensor cores:
// wgmma.mma_async tf32 with the accumulator in registers, operands staged by TMA (cp.async.bulk.tensor,
// SWIZZLE_128B) through a 3-stage mbarrier pipeline.  sm_90a only.
//
// fp32-faithful on TF32 tensor cores ("3xTF32"): every fp32 operand is pre-split into
//   hi = x with the low 13 mantissa bits cleared (exactly a TF32 value),  lo = x - hi (exact in fp32)
// and each K-step issues hi*hi + hi*lo + lo*hi into the same fp32 accumulator.  The dropped
// lo*lo term and the truncation of lo to 11 bits are ~2^-22 relative, i.e. at the level of the fp32
// accumulation itself -- the precision scikit-learn's own fp32 BLAS calls have on this path
// (Ridge: sklearn/linear_model/_ridge.py:215-227 keeps float32 throughout).
//
// Replaces (reference path -> scikit-learn): safe_sparse_dot(X.T, X) of _solve_cholesky (_ridge.py:219),
// X @ w and X.T @ grad of the logistic objective (_linear_loss.py), and -- opt-in -- the libsvm kernel rows.
//
// The fp32 tensor-core accumulator does not round to nearest, so a long contraction drifts by ~sqrt(K)*2^-24 of sum|a||b| -- harmless
// for a Gram diagonal, ruinous for a heavily cancelled sum such as a gradient near its zero.  Callers therefore
// bound every accumulation chain to TC_KCHUNK terms (one TcBatch per K-chunk) and add the partial tiles in float64
// on the CUDA cores (launch_sum_partials).
//
// Tile: 128 x 128 x 32 (fp32) per stage.  PERSISTENT, warp-specialised CTAs (one per SM, 9 warps), tiles dealt round-robin:
//   warps 0-7 (two warpgroups): warpgroup g owns tile rows [64 g, 64 g + 64) in 64 fp32 registers per thread, issues 12
//              wgmma m64n128k8 per stage and stores straight from the accumulator fragment (float2 column pairs)
//   warp 8 / lane 0: TMA producer (3-stage ring over ALL tiles of the CTA: the next tile loads during the last one's stores)
// symmetric (A == B, M == N): only tiles on or above the diagonal are computed and their transposes stored too.
// Batched: per-batch row offsets into A and B, K range and output pointer.
#include "common.cuh"
#include <cuda.h>
#include <cstdio>
#include <algorithm>

namespace {

constexpr int BM = 128, BN = 128, BK = 32;            // BK fp32 = 128 B = one SWIZZLE_128B atom row
constexpr int STAGES = 3;
constexpr int TILE_BYTES = BM * BK * 4;               // 16 KB per operand tile
constexpr int STAGE_BYTES = 4 * TILE_BYTES;           // A_hi, A_lo, B_hi, B_lo
constexpr int CONSUMER_WARPS = 8, NTHREADS = (CONSUMER_WARPS + 1) * 32;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// bounded spin: a protocol bug traps the kernel instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t done = 0;
    for (uint32_t spin = 0; !done; ++spin) {
        asm volatile("{\n\t.reg .pred p;\n\t"
                     "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, int c0, int c1, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
// wgmma shared-memory matrix descriptor, K-major, SWIZZLE_128B: start>>4 @0, LBO (unused for swizzled K-major) = 1 @16,
// SBO = 8 rows * 128 B = 1024 B (>>4 = 64) @32, base offset 0 (every operand tile is 1024-byte aligned), layout 1 (128B) @62
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr)
{
    return (uint64_t)((saddr >> 4) & 0x3fff) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// d[64] += A[64 x 8] * B[128 x 8]^T, tf32 operands from shared memory; fragment of thread (warp w, lane l) of the
// warpgroup: d[4 j + 2 h + e] = row 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
                 "%23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, "
                 "%44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(adesc), "l"(bdesc), "r"(1));
}
// keeps the compiler from moving accumulator reads or writes across the asynchronous wgmma window
__device__ __forceinline__ void fence_acc(float (&d)[64])
{
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// tile t of the launch -> (batch, m-tile, n-tile); symmetric: n-tile >= m-tile only
__device__ __forceinline__ void decode_tile(int t, int tiles_m, int tiles_n, int symmetric, int &z, int &mi, int &ni)
{
    const int per = symmetric ? tiles_m * (tiles_m + 1) / 2 : tiles_m * tiles_n;
    z = t / per;
    int r = t - z * per;
    if (!symmetric) { mi = r / tiles_n; ni = r - mi * tiles_n; return; }
    mi = 0;
    while (r >= tiles_m - mi) { r -= tiles_m - mi; mi++; }
    ni = mi + r;
}

__device__ __forceinline__ void store_c(float *c, int64_t ldc, int row, int col, float v, int accumulate_c)
{
    float *dst = c + (size_t)row * ldc + col;
    *dst = accumulate_c ? *dst + v : v;
}

__global__ void __launch_bounds__(NTHREADS, 1)
gemm_nt_tf32x3_kernel(const __grid_constant__ CUtensorMap a_hi, const __grid_constant__ CUtensorMap a_lo,
                      const __grid_constant__ CUtensorMap b_hi, const __grid_constant__ CUtensorMap b_lo,
                      const TcBatch *__restrict__ batches, int n_batches, int M, int N, float alpha, int accumulate_c, int symmetric)
{
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_dyn + 1023) & ~(uintptr_t)1023);
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + STAGES * STAGE_BYTES);   // full[S], empty[S]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
    const int n_tiles = n_batches * (symmetric ? tiles_m * (tiles_m + 1) / 2 : tiles_m * tiles_n);
    const uint32_t b_full = smem_u32(&bars[0]), b_empty = smem_u32(&bars[STAGES]);

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(b_full + 8 * s, 1); mbar_init(b_empty + 8 * s, CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == CONSUMER_WARPS) {
        if (lane == 0) {
            // ---------------- TMA producer: one ring over all tiles of this CTA ----------------
            int it = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
                int z, mi, ni;
                decode_tile(t, tiles_m, tiles_n, symmetric, z, mi, ni);
                const TcBatch bt = batches[z];
                const int nkb = (bt.k1 - bt.k0 + BK - 1) / BK;
                for (int kb = 0; kb < nkb; kb++, it++) {
                    const int s = it % STAGES;
                    const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
                    mbar_wait(b_empty + 8 * s, ph ^ 1u);                        // slot free
                    const uint32_t full = b_full + 8 * s;
                    mbar_expect_tx(full, STAGE_BYTES);
                    const uint32_t base = smem_u32(smem + s * STAGE_BYTES);
                    const int kc = bt.k0 + kb * BK;
                    tma_load_2d(base, &a_hi, kc, bt.a_row0 + mi * BM, full);
                    tma_load_2d(base + TILE_BYTES, &a_lo, kc, bt.a_row0 + mi * BM, full);
                    tma_load_2d(base + 2 * TILE_BYTES, &b_hi, kc, bt.b_row0 + ni * BN, full);
                    tma_load_2d(base + 3 * TILE_BYTES, &b_lo, kc, bt.b_row0 + ni * BN, full);
                }
            }
        }
        return;
    }

    // ---------------- consumers: warpgroup wg computes and stores rows [64 wg, 64 wg + 64) of every tile ----------------
    const int wg = warp >> 2;
    const uint32_t a_off = (uint32_t)wg * 64 * BK * 4;                            // 8 KB: a multiple of the 1 KB swizzle atom
    float d[64];
    int it = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        int z, mi, ni;
        decode_tile(t, tiles_m, tiles_n, symmetric, z, mi, ni);
        const TcBatch bt = batches[z];
        const int nkb = (bt.k1 - bt.k0 + BK - 1) / BK;
#pragma unroll
        for (int i = 0; i < 64; i++) d[i] = 0.f;
        for (int kb = 0; kb < nkb; kb++, it++) {
            const int s = it % STAGES;
            mbar_wait(b_full + 8 * s, (uint32_t)(it / STAGES) & 1u);            // TMA bytes landed
            const uint32_t base = smem_u32(smem + s * STAGE_BYTES);
            const uint64_t dah = make_desc(base + a_off), dal = make_desc(base + TILE_BYTES + a_off);
            const uint64_t dbh = make_desc(base + 2 * TILE_BYTES), dbl = make_desc(base + 3 * TILE_BYTES);
            fence_acc(d);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int k = 0; k < BK / 8; k++) {                                   // K = 8 per tf32 wgmma: 32 B per step
                const uint64_t off = (uint64_t)(k * 32 >> 4);                    // advance inside the swizzle atom
                wgmma_tf32(d, dah + off, dbh + off);
                wgmma_tf32(d, dah + off, dbl + off);
                wgmma_tf32(d, dal + off, dbh + off);
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            // the previous stage's group has retired: its slot may be refilled while this one runs
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
            fence_acc(d);
            if (kb > 0 && lane == 0) mbar_arrive(b_empty + 8 * ((it - 1) % STAGES));
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        fence_acc(d);
        if (nkb > 0 && lane == 0) mbar_arrive(b_empty + 8 * ((it - 1) % STAGES));

        // ---------------- epilogue: straight from the accumulator fragment to global memory ----------------
        const int r0 = mi * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int c0 = ni * BN + 2 * (lane & 3);
        const bool diag = symmetric && mi == ni;       // diagonal tile: store j >= i, mirror the strict upper part (bitwise symmetric:
                                                       // the hi*lo and lo*hi products of C[i][j] and C[j][i] accumulate in swapped order)
        // columns col, col + 1 of a row are one float2 (4 lanes fill a 32-byte sector) except on diagonal tiles and odd ldc;
        // mirrored stores: 8 lanes write 8 consecutive floats of one row of C
        const bool vec = !diag && (bt.ldc & 1) == 0 && ((uintptr_t)bt.c & 7) == 0;
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int row = r0 + 8 * ((i >> 1) & 1), col = c0 + 8 * (i >> 2);
            if (row >= M || col >= N) continue;
            const float v0 = alpha * d[i], v1 = alpha * d[i + 1];
            const bool two = col + 1 < N;
            if (vec && two) {
                float2 *dst = reinterpret_cast<float2 *>(bt.c + (size_t)row * bt.ldc + col);
                float2 o = make_float2(v0, v1);
                if (accumulate_c) { const float2 p = *dst; o.x += p.x; o.y += p.y; }
                *dst = o;
            } else {
                if (!(diag && col < row)) store_c(bt.c, bt.ldc, row, col, v0, accumulate_c);
                if (two && !(diag && col + 1 < row)) store_c(bt.c, bt.ldc, row, col + 1, v1, accumulate_c);
            }
            if (symmetric) {                                                     // C[n][m] = C[m][n]
                if (!(diag && col <= row)) store_c(bt.c, bt.ldc, col, row, v0, accumulate_c);
                if (two && !(diag && col + 1 <= row)) store_c(bt.c, bt.ldc, col + 1, row, v1, accumulate_c);
            }
        }
    }
}

// hi = x with the low 13 mantissa bits cleared (a TF32 value), lo = x - hi (exact)
__global__ void split_tf32_kernel(const float *__restrict__ x, float *__restrict__ hi, float *__restrict__ lo, size_t n)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float v = x[i];
        const float h = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
        hi[i] = h;
        lo[i] = v - h;
    }
}

// out[i] = (float) sum_c partial[c][i] accumulated in float64 (round-to-nearest), i < per
__global__ void sum_partials_kernel(const float *__restrict__ partial, int n_chunks, int64_t per, float *__restrict__ out)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.x * blockDim.x) {
        double s = 0;
        for (int c = 0; c < n_chunks; c++) s += (double)partial[(size_t)c * per + i];
        out[i] = (float)s;
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

}  // namespace

// 2-D tensor map over a row-major fp32 matrix [rows][ld] exposing `cols` columns, box = BK x 128 rows, 128B swizzle
cudaError_t tc_make_map(TcMap *out, const float *base, int64_t rows, int64_t cols, int64_t ld)
{
    EncodeTiledFn fn = encode_fn();
    if (!fn) return cudaErrorNotSupported;
    if ((ld * 4) % 16 != 0 || ((uintptr_t)base & 15)) return cudaErrorInvalidValue;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(reinterpret_cast<CUtensorMap *>(out), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)base, dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

cudaError_t launch_sum_partials(const float *partial, int n_chunks, int64_t per, float *out, cudaStream_t st)
{
    sum_partials_kernel<<<(unsigned)std::min<int64_t>((per + 255) / 256, 1056), 256, 0, st>>>(partial, n_chunks, per, out);
    return cudaGetLastError();
}

cudaError_t launch_split_tf32(const float *x, float *hi, float *lo, size_t n, cudaStream_t st)
{
    split_tf32_kernel<<<528, 256, 0, st>>>(x, hi, lo, n);
    return cudaGetLastError();
}

cudaError_t launch_gemm_nt_tf32x3(const TcMap &a_hi, const TcMap &a_lo, const TcMap &b_hi, const TcMap &b_lo,
                                  const TcBatch *d_batches, int n_batches, int M, int N, float alpha, bool accumulate,
                                  cudaStream_t st, bool symmetric)
{
    // per device and per launch (cheap): a handle per GPU may launch this kernel from its own host thread
    cudaError_t e = cudaFuncSetAttribute(gemm_nt_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return e;
    if (symmetric && M != N) return cudaErrorInvalidValue;
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int tm = (M + BM - 1) / BM, tn = (N + BN - 1) / BN;
    const long long tiles = (long long)n_batches * (symmetric ? (long long)tm * (tm + 1) / 2 : (long long)tm * tn);
    if (tiles <= 0) return cudaSuccess;
    const int grid = (int)std::min<long long>(tiles, sms);
    gemm_nt_tf32x3_kernel<<<grid, NTHREADS, SMEM_BYTES, st>>>(*reinterpret_cast<const CUtensorMap *>(&a_hi),
                                                              *reinterpret_cast<const CUtensorMap *>(&a_lo),
                                                              *reinterpret_cast<const CUtensorMap *>(&b_hi),
                                                              *reinterpret_cast<const CUtensorMap *>(&b_lo), d_batches, n_batches, M, N, alpha,
                                                              accumulate ? 1 : 0, symmetric ? 1 : 0);
    return cudaGetLastError();
}
