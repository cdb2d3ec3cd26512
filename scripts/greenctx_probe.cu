// greenctx_probe.cu — can this driver carve the GPU into two SM partitions (CUDA green contexts) and do kernels launched
// through a partition's stream stay on its SMs?  Diagnostics for the chain's modulator placement.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O2 -o scripts/_bin/greenctx_probe scripts/greenctx_probe.cu -lcuda
#include <cstdio>
#include <cstring>
#include <cuda.h>
#include <cuda_runtime.h>

#define CK(x) do { CUresult r_ = (x); if (r_ != CUDA_SUCCESS) { const char *s_; cuGetErrorString(r_, &s_); printf("%s -> %s\n", #x, s_); return 1; } } while (0)

__global__ void where(unsigned *hist, int spin)
{
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    if (threadIdx.x == 0) atomicAdd(&hist[smid], 1u);
    long long t0 = clock64();
    while (clock64() - t0 < spin) { }
}

int main()
{
    cudaFree(0);
    CUdevice dev; CK(cuDeviceGet(&dev, 0));
    CUdevResource sm; CK(cuDeviceGetDevResource(dev, &sm, CU_DEV_RESOURCE_TYPE_SM));
    printf("device SMs: %u\n", sm.sm.smCount);
    for (unsigned want : { 64u, 32u, 16u, 8u, 4u }) {
        CUdevResource part[1], rest; unsigned n = 1;
        CUresult r = cuDevSmResourceSplitByCount(part, &n, &sm, &rest, 0, want);
        if (r != CUDA_SUCCESS) { const char *s; cuGetErrorString(r, &s); printf("split %u -> %s\n", want, s); continue; }
        printf("split by %u: %u group(s) of %u SMs, remainder %u SMs\n", want, n, part[0].sm.smCount, rest.sm.smCount);
        CUdevResourceDesc d0, d1; CK(cuDevResourceGenerateDesc(&d0, &part[0], 1)); CK(cuDevResourceGenerateDesc(&d1, &rest, 1));
        CUgreenCtx g0, g1; CK(cuGreenCtxCreate(&g0, d0, dev, CU_GREEN_CTX_DEFAULT_STREAM)); CK(cuGreenCtxCreate(&g1, d1, dev, CU_GREEN_CTX_DEFAULT_STREAM));
        CUstream s0, s1; CK(cuGreenCtxStreamCreate(&s0, g0, CU_STREAM_NON_BLOCKING, 0)); CK(cuGreenCtxStreamCreate(&s1, g1, CU_STREAM_NON_BLOCKING, 0));
        unsigned *h0, *h1; cudaMalloc(&h0, 1024 * 4); cudaMalloc(&h1, 1024 * 4); cudaMemset(h0, 0, 4096); cudaMemset(h1, 0, 4096);
        cudaDeviceSynchronize();
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaEventRecord(e0, (cudaStream_t)s1);
        where<<<2000, 128, 0, (cudaStream_t)s0>>>(h0, 200000);
        where<<<2000, 128, 0, (cudaStream_t)s1>>>(h1, 200000);
        cudaEventRecord(e1, (cudaStream_t)s1);
        cudaError_t ce = cudaDeviceSynchronize();
        unsigned a[1024], b[1024]; cudaMemcpy(a, h0, 4096, cudaMemcpyDeviceToHost); cudaMemcpy(b, h1, 4096, cudaMemcpyDeviceToHost);
        int na = 0, nb = 0, both = 0;
        for (int i = 0; i < 1024; i++) { na += a[i] != 0; nb += b[i] != 0; both += (a[i] != 0 && b[i] != 0); }
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        printf("  launch status %s: partition kernel ran on %d SMs, remainder kernel on %d SMs, %d shared; remainder stream %.2f ms\n", cudaGetErrorString(ce), na, nb, both, ms);
        cudaFree(h0); cudaFree(h1);
        CK(cuStreamDestroy(s0)); CK(cuStreamDestroy(s1)); CK(cuGreenCtxDestroy(g0)); CK(cuGreenCtxDestroy(g1));
    }
    return 0;
}
