// Micro-benchmark (diagnostics, not part of the library): what store pattern does NVLink want?
// One process, two devices; kernels on device 0 write into a buffer on device 1 (and, for reference, into local memory).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/p2p_write_bench tools/p2p_write_bench.cu && build/p2p_write_bench
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s failed: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

// every warp writes 256-byte segments; `shift` 8-byte elements of misalignment; `run` = consecutive segments before jumping
__global__ void stream_store(long long* dst, const long long* src, size_t n, int shift)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i + shift < n; i += stride) dst[i + shift] = src[i];
}
// scattered runs: element i goes to run-permuted place: blocks of `run` elements are permuted by a multiplicative hash
__global__ void run_store(long long* dst, const long long* src, size_t n, int run, int shift)
{
    size_t nblocks = n / run - 1;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < nblocks * run; i += stride) {
        size_t b = i / run, o = i % run;
        size_t pb = (b * 2654435761ull) % nblocks;
        dst[pb * run + o + shift] = src[i];
    }
}
// bulk (TMA) stores: each warp stages `bytes` in shared memory and issues one cp.async.bulk shared->global
template <int BYTES>
__global__ void bulk_store(char* dst, const char* src, size_t nbytes)
{
    extern __shared__ __align__(128) char sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    char* my = sm + (size_t)warp * BYTES;
    size_t tiles = nbytes / BYTES;
    for (size_t t = (size_t)blockIdx.x * nw + warp; t < tiles; t += (size_t)gridDim.x * nw) {
        const int4* s = (const int4*)(src + t * BYTES);
        for (int k = lane; k < BYTES / 16; k += 32) ((int4*)my)[k] = s[k];
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) {
            unsigned int sa = (unsigned int)__cvta_generic_to_shared(my);
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst + t * BYTES), "r"(sa), "r"(BYTES) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        }
        __syncwarp();
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

int main(int argc, char** argv)
{
    const int peer = argc > 1 ? atoi(argv[1]) : 1;
    const bool quick = argc > 2;
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    const size_t n = (size_t)512 << 20 >> 3;   // 512 MiB of int64
    long long *src, *local, *remote = nullptr;
    CK(cudaSetDevice(0));
    CK(cudaMalloc(&src, n * 8 + 4096));
    CK(cudaMalloc(&local, n * 8 + 4096));
    CK(cudaMemset(src, 1, n * 8));
    if (ndev > 1) {
        CK(cudaSetDevice(peer));
        CK(cudaMalloc(&remote, n * 8 + 4096));
        CK(cudaSetDevice(0));
        CK(cudaDeviceEnablePeerAccess(peer, 0));
    }
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    auto timeit = [&](const char* name, auto launch) {
        for (int w = 0; w < 2; w++) launch();
        CK(cudaEventRecord(e0));
        for (int r = 0; r < 5; r++) launch();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaGetLastError());
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        printf("%-44s %8.1f GB/s written\n", name, n * 8.0 * 5 / ms / 1e6);
    };
    const int grid = 132 * 8, bs = 256;      // 8 CTAs on each of an H100's 132 SMs
    for (int where = quick ? 1 : 0; where < (remote ? 2 : 1); where++) {
        long long* dst = where ? remote : local;
        printf("---- destination: %s (device %d)\n", where ? "peer GPU over NVLink" : "local HBM", where ? peer : 0);
        char name[128];
        timeit("cudaMemcpyAsync", [&] { CK(cudaMemcpyAsync(dst, src, n * 8, cudaMemcpyDefault)); });
        for (int shift : {0, 4, 8}) {
            if (quick && shift) continue;
            snprintf(name, sizeof name, "stream store, shift %d B", shift * 8);
            timeit(name, [&] { stream_store<<<grid, bs>>>(dst, src, n, shift); });
        }
        for (int run : {4, 16, 32, 128, 1024}) {
            if (quick && run != 32) continue;
            for (int shift : {0, 5}) {
                snprintf(name, sizeof name, "permuted runs of %d B, shift %d B", run * 8, shift * 8);
                timeit(name, [&] { run_store<<<grid, bs>>>(dst, src, n, run, shift); });
            }
        }
        if (quick) continue;
        timeit("bulk store 256 B per warp", [&] { bulk_store<256><<<grid, bs, 8 * 256>>>((char*)dst, (const char*)src, n * 8); });
        timeit("bulk store 2048 B per warp", [&] { bulk_store<2048><<<grid, bs, 8 * 2048>>>((char*)dst, (const char*)src, n * 8); });
        timeit("bulk store 8192 B per warp", [&] {
            cudaFuncSetAttribute(bulk_store<8192>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 8192);
            bulk_store<8192><<<grid, bs, 8 * 8192>>>((char*)dst, (const char*)src, n * 8);
        });
    }
    return 0;
}
