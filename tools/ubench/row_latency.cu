// Development micro-benchmark: latency of bringing one 40 KB kernel-matrix row to an SM, cold (HBM) and warm (L2):
//   (a) one cp.async.bulk into shared memory   (b) N bulk copies of 1/N each   (c) coalesced LDG.128 by 1024 / 512 / 256 threads
//   (d) bulk copy after cp.async.bulk.prefetch.L2 issued `lead` cycles earlier
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o row_latency row_latency.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
    unsigned done = 0;
    while (!done)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
}

// mode 0: nsplit bulk copies; mode 1: LDG.128 by all threads (row floats/4 per thread strided); mode 2: prefetch.L2 then wait `lead` then bulk
__global__ void k(const float *K, size_t ldk, const int *rows, int nrows, int rowfloats, int mode, int nsplit, int lead, long long *out, float *sink)
{
    extern __shared__ __align__(128) float buf[];
    __shared__ __align__(8) unsigned long long bar;
    const int tid = threadIdx.x;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    unsigned phase = 0;
    float acc = 0.f;
    long long total = 0;
    for (int it = 0; it < nrows; it++) {
        const float *src = K + (size_t)rows[it] * ldk;
        __syncthreads();
        if (mode == 2 || mode == 3 || mode == 4) {
            if (mode == 4) { if (tid * 32 < rowfloats) asm volatile("prefetch.global.L2 [%0];" ::"l"(src + tid * 32) : "memory"); }
            else if (tid == 0) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(rowfloats * 4) : "memory");
            const long long t0 = clock64();
            while (clock64() - t0 < lead) { }
            __syncthreads();
        }
        const long long t0 = clock64();
        if (mode == 0 || mode == 2) {
            const unsigned b = smem_u32(&bar);
            if (tid == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(rowfloats * 4) : "memory");
            if (tid < nsplit) {
                const int part = rowfloats / nsplit;
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(buf + tid * part)), "l"(src + tid * part), "r"(part * 4), "r"(b) : "memory");
            }
            mbar_wait(b, phase);
            phase ^= 1;
            acc += buf[tid];
        } else {
            const float4 *s4 = reinterpret_cast<const float4 *>(src);
            float4 v[4];
            int n = 0;
            for (int q = tid; q < rowfloats / 4 && n < 4; q += blockDim.x) v[n++] = __ldg(s4 + q);
            for (int q = 0; q < n; q++) acc += v[q].x + v[q].y + v[q].z + v[q].w;
        }
        __syncthreads();
        total += clock64() - t0;
    }
    if (tid == 0) out[blockIdx.x] = total / nrows;
    if (acc == 123.456f) sink[0] = acc;
}

int main()
{
    const int n = 10000; const size_t ldk = 10016; const int NG = 8;          // 8 matrices of 400 MB: 3.2 GB, like config 2
    float *K; cudaMalloc(&K, (size_t)NG * n * ldk * 4); cudaMemset(K, 0, (size_t)NG * n * ldk * 4);
    const int nrows = 2000;
    std::vector<int> rows(nrows), same(nrows, 777), l2set(nrows), l2page(nrows);
    srand(1);
    for (auto &r : rows) r = rand() % (NG * n);
    for (int i = 0; i < nrows; i++) { l2set[i] = rows[i % 100]; l2page[i] = 5000 + (i % 40); }     // 100 rows (4 MB) cycled: L2 hits, L1 misses; 40 rows in one 2 MB page
    int *d_l2, *d_pg; cudaMalloc(&d_l2, nrows * 4); cudaMalloc(&d_pg, nrows * 4);
    cudaMemcpy(d_l2, l2set.data(), nrows * 4, cudaMemcpyHostToDevice); cudaMemcpy(d_pg, l2page.data(), nrows * 4, cudaMemcpyHostToDevice);
    int *d_rows, *d_same; cudaMalloc(&d_rows, nrows * 4); cudaMalloc(&d_same, nrows * 4);
    cudaMemcpy(d_rows, rows.data(), nrows * 4, cudaMemcpyHostToDevice); cudaMemcpy(d_same, same.data(), nrows * 4, cudaMemcpyHostToDevice);
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    long long *out; cudaMallocManaged(&out, (size_t)sms * 8); float *sink; cudaMalloc(&sink, 4);
    const int smem = 10016 * 4 + 256;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    auto run = [&](const char *name, int grid, int nt, const int *r, int mode, int nsplit, int lead) {
        k<<<grid, nt, smem>>>(K, ldk, r, nrows, 10016, mode, nsplit, lead, out, sink);
        cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(e)); exit(1); }
        long long s = 0; for (int i = 0; i < grid; i++) s += out[i];
        printf("%-44s grid %3d nt %4d : %6lld cycles/row\n", name, grid, nt, s / grid);
    };
    for (int grid : {1}) {
        run("bulk x1 L2set(100 rows cycled)", grid, 1024, d_l2, 0, 1, 0);
        run("ldg128 1024thr L2set", grid, 1024, d_l2, 1, 0, 0);
        run("ldg128 256thr L2set", grid, 256, d_l2, 1, 0, 0);
        run("bulk x1 one-page set (40 rows)", grid, 1024, d_pg, 0, 1, 0);
        run("ldg128 1024thr one-page set", grid, 1024, d_pg, 1, 0, 0);
        run("bulk x1 cold", grid, 1024, d_rows, 0, 1, 0);
        run("bulk x1 warm(L2)", grid, 1024, d_same, 0, 1, 0);
        run("bulk x2 cold", grid, 1024, d_rows, 0, 2, 0);
        run("bulk x4 cold", grid, 1024, d_rows, 0, 4, 0);
        run("bulk x8 cold", grid, 1024, d_rows, 0, 8, 0);
        run("bulk x8 warm", grid, 1024, d_same, 0, 8, 0);
        run("ldg128 1024thr cold", grid, 1024, d_rows, 1, 0, 0);
        run("ldg128 1024thr warm", grid, 1024, d_same, 1, 0, 0);
        run("ldg128 512thr cold (4/thread =32KB)", grid, 512, d_rows, 1, 0, 0);
        run("ldg128 256thr cold (4/thread =16KB)", grid, 256, d_rows, 1, 0, 0);
        run("ldg128 256thr warm", grid, 256, d_same, 1, 0, 0);
        run("bulk.prefetch.L2 lead 1000 + bulk x1", grid, 1024, d_rows, 2, 1, 1000);
        run("bulk.prefetch.L2 lead 3000 + bulk x1", grid, 1024, d_rows, 2, 1, 3000);
        run("bulk.prefetch.L2 lead 10000 + bulk x1", grid, 1024, d_rows, 2, 1, 10000);
        run("bulk.prefetch.L2 lead 500 + ldg128", grid, 1024, d_rows, 3, 0, 500);
        run("bulk.prefetch.L2 lead 1000 + ldg128", grid, 1024, d_rows, 3, 0, 1000);
        run("bulk.prefetch.L2 lead 1500 + ldg128", grid, 1024, d_rows, 3, 0, 1500);
        run("bulk.prefetch.L2 lead 3000 + ldg128", grid, 1024, d_rows, 3, 0, 3000);
        run("bulk.prefetch.L2 lead 10000 + ldg128", grid, 1024, d_rows, 3, 0, 10000);
        run("prefetch.global.L2/line lead 1500 + ldg128", grid, 1024, d_rows, 4, 0, 1500);
        run("prefetch.global.L2/line lead 3000 + ldg128", grid, 1024, d_rows, 4, 0, 3000);
    }
    return 0;
}
