// q28_ubench.cu — cycles per band-sample of the RP2040 Q28 biquad (dsp_process_rp2040.S:263-365, fast_mul_q28
// dsp_pipeline.c:47-58) for two statements of the multiply, register-resident like eq_q28_kernel (10 bands, tile of 8):
//   V0  the three 32-bit partial products as the firmware writes them: 3 IMAD + 1 SHF per multiply
//   V1  one 64-bit sum  M = (c>>16) * x + (c&0xFFFF) * (x>>16)  and  r = low32(M >> 12): 2 IMAD.WIDE + 1 SHF.
//       Equal to V0 whenever the firmware's 32-bit `mid` does not wrap, which -2^30 <= c, x < 2^30 guarantees.
//   V2  V1 plus the range watch on every band input / output (what the kernel needs to fall back on wrap)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/_bin/q28_ubench scripts/q28_ubench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int NB = 10, SUB = 8;

struct C3 { int32_t hi; uint32_t lo; uint32_t hi16; };
struct C2 { int32_t hi; int32_t lo; };

__device__ __forceinline__ uint32_t mul3(const C3 &c, int32_t xh, uint32_t xl)
{
    const uint32_t mid = (uint32_t)c.hi * xl + c.lo * (uint32_t)xh;
    return c.hi16 * (uint32_t)xh + (uint32_t)((int32_t)mid >> 12);
}
__device__ __forceinline__ uint32_t mul2(const C2 &c, int32_t x, int32_t xh)
{
    int64_t m;
    asm("mul.wide.s32 %0, %1, %2;" : "=l"(m) : "r"(c.lo), "r"(xh));
    asm("mad.wide.s32 %0, %1, %2, %0;" : "+l"(m) : "r"(c.hi), "r"(x));
    return __funnelshift_r((uint32_t)m, (uint32_t)(m >> 32), 12);
}

template <int V, int MT>
__global__ void __launch_bounds__(MT, 1) k(const int32_t *__restrict__ coef, uint32_t *__restrict__ out, int iters, long long *clk)
{
    const int lane = threadIdx.x;
    C3 c3[NB][5];
    C2 c2[NB][5];
    uint32_t s1[NB], s2[NB];
#pragma unroll
    for (int b = 0; b < NB; b++) {
#pragma unroll
        for (int j = 0; j < 5; j++) {
            const int32_t c = coef[(b * 5 + j) * 32 + (lane & 31)];
            c3[b][j].hi = c >> 16; c3[b][j].lo = (uint32_t)c & 0xFFFFu; c3[b][j].hi16 = (uint32_t)(c >> 16) << 4;
            c2[b][j].hi = c >> 16; c2[b][j].lo = (int32_t)((uint32_t)c & 0xFFFFu);
        }
        s1[b] = 0; s2[b] = 0;
    }
    uint32_t x[SUB], rng = 0x9E3779B9u * (blockIdx.x * blockDim.x + threadIdx.x + 1), sum = 0, watch = 0;
    const long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < SUB; i++) { rng ^= rng << 13; rng ^= rng >> 17; rng ^= rng << 5; x[i] = (uint32_t)((int32_t)rng >> 4); }
#pragma unroll
        for (int b = 0; b < NB; b++) {
#pragma unroll
            for (int i = 0; i < SUB; i++) {
                if constexpr (V == 0) {
                    const int32_t xh = (int32_t)x[i] >> 16; const uint32_t xl = x[i] & 0xFFFFu;
                    const uint32_t y = mul3(c3[b][0], xh, xl) + s1[b];
                    const uint32_t t1 = mul3(c3[b][1], xh, xl), t3 = mul3(c3[b][2], xh, xl);
                    const int32_t yh = (int32_t)y >> 16; const uint32_t yl = y & 0xFFFFu;
                    const uint32_t t2 = mul3(c3[b][3], yh, yl), t4 = mul3(c3[b][4], yh, yl);
                    s1[b] = (t1 - t2) + s2[b]; s2[b] = t3 - t4; x[i] = y;
                } else {
                    const int32_t xv = (int32_t)x[i], xh = xv >> 16;
                    if (V == 2 && b == 0) watch |= x[i] + 0x40000000u;
                    const uint32_t y = mul2(c2[b][0], xv, xh) + s1[b];
                    const uint32_t t1 = mul2(c2[b][1], xv, xh), t3 = mul2(c2[b][2], xv, xh);
                    const int32_t yv = (int32_t)y, yh = yv >> 16;
                    if (V == 2) watch |= y + 0x40000000u;
                    const uint32_t t2 = mul2(c2[b][3], yv, yh), t4 = mul2(c2[b][4], yv, yh);
                    s1[b] = (t1 - t2) + s2[b]; s2[b] = t3 - t4; x[i] = y;
                }
            }
        }
#pragma unroll
        for (int i = 0; i < SUB; i++) sum += x[i];
    }
    const long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = sum + (watch >> 31);
    if (threadIdx.x == 0 && blockIdx.x == 0) *clk = t1 - t0;
}

template <int V, int MT>
double run(int warps_per_smsp, const int32_t *coef, uint32_t *out, long long *clk, uint32_t *checksum)
{
    const int iters = 2000, threads = warps_per_smsp * 128;
    k<V, MT><<<132, threads>>>(coef, out, 10, clk);
    cudaDeviceSynchronize();
    k<V, MT><<<132, threads>>>(coef, out, iters, clk);
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(cudaGetLastError())); return -1; }
    long long c; cudaMemcpy(&c, clk, 8, cudaMemcpyDeviceToHost);
    uint32_t h[256]; cudaMemcpy(h, out, sizeof h, cudaMemcpyDeviceToHost);
    uint32_t s = 0; for (int i = 0; i < 128; i++) s = s * 31 + h[i];       // first warp per SMSP only: same lanes in every config
    *checksum = s;
    return (double)c / ((double)iters * NB * SUB * warps_per_smsp);         // clocks per warp-level band-sample per SM sub-partition
}

int main()
{
    int32_t h[NB * 5 * 32];
    uint32_t r = 12345;
    for (int i = 0; i < NB * 5 * 32; i++) { r ^= r << 13; r ^= r >> 17; r ^= r << 5; h[i] = (int32_t)r >> 3; }   // |c| < 2^28 ... keeps the recursion bounded? no: wraps, which is fine for timing
    for (int b = 0; b < NB; b++) for (int l = 0; l < 32; l++) {                                                    // a stable-ish section so values stay in range for the equality check
        h[(b * 5 + 0) * 32 + l] = (1 << 28) / 4; h[(b * 5 + 1) * 32 + l] = (1 << 28) / 8; h[(b * 5 + 2) * 32 + l] = (1 << 28) / 16;
        h[(b * 5 + 3) * 32 + l] = -(1 << 28) / 4 + l * 4097; h[(b * 5 + 4) * 32 + l] = (1 << 28) / 8 - l * 523;
    }
    int32_t *coef; uint32_t *out; long long *clk;
    cudaMalloc(&coef, sizeof h); cudaMalloc(&out, 132 * 512 * 4); cudaMalloc(&clk, 8);
    cudaMemcpy(coef, h, sizeof h, cudaMemcpyHostToDevice);
    printf("clocks per band-sample (warp-level, per SM sub-partition); checksum of the first 128 lanes\n");
    for (int w = 1; w <= 4; w++) {
        uint32_t c0, c1, c2;
        double a, b, c;
        if (w <= 2) { a = run<0, 256>(w, coef, out, clk, &c0); b = run<1, 256>(w, coef, out, clk, &c1); c = run<2, 256>(w, coef, out, clk, &c2); }
        else if (w == 3) { a = run<0, 384>(w, coef, out, clk, &c0); b = run<1, 384>(w, coef, out, clk, &c1); c = run<2, 384>(w, coef, out, clk, &c2); }
        else { a = run<0, 512>(w, coef, out, clk, &c0); b = run<1, 512>(w, coef, out, clk, &c1); c = run<2, 512>(w, coef, out, clk, &c2); }
        printf("warps/SMSP %d:  V0 3xIMAD %.2f (%08x)   V1 2xIMAD.WIDE %.2f (%08x)   V2 +watch %.2f (%08x)\n", w, a, c0, b, c1, c, c2);
    }
    return 0;
}
