// pdm_ubench.cu — cycles per delta-sigma decision for several formulations of the inner loop of
// pdm_generator.c:372-378 (one warp per SM sub-partition, like chain_pdm_kernel at 8192 instances).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/_bin/pdm_ubench scripts/pdm_ubench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int V>
__device__ __forceinline__ uint32_t chunk(int32_t &err1, int32_t &err2, int32_t target, int32_t dither)
{
    uint32_t word = 0;
    if constexpr (V == 0) {                 // reference shape
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const int bit = (err2 + dither) >= 0;
            const int32_t fb = bit ? 65535 : 0;
            if (bit) word |= 1u << (31 - k);
            err1 += target - fb;
            err2 += err1 - fb;
        }
    } else if constexpr (V == 1) {          // mask form (round-1 kernel)
        int32_t s = err2 + dither;
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const int32_t m = s >> 31;
            const int32_t nfb = ~m & -65535;
            word = __funnelshift_l((uint32_t)~m, word, 1);
            err1 += target + nfb;
            s += err1 + nfb;
        }
        err2 = s - dither;
    } else if constexpr (V == 2) {          // two running sums, predicated corrections
        int32_t s = err2 + dither, g = err1 + target;
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const bool bit = s >= 0;
            int32_t t = s + g;
            g += target;
            if (bit) { t -= 131070; g -= 65535; word |= 1u << (31 - k); }
            s = t;
        }
        err2 = s - dither; err1 = g - target;
    } else if constexpr (V == 3) {          // two running sums, sign mask times constant on the FMA pipe
        int32_t s = err2 + dither, g = err1 + target;
        const int32_t tg = target - 65535;
        uint32_t acc = 0;
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const int32_t m = s >> 31;                    // 0 when the bit is 1, -1 when it is 0
            const int32_t t2 = s + g - 131070;
            const int32_t g2 = g + tg;
            s = m * -131070 + t2;
            g = m * -65535 + g2;
            acc = acc * 2u + (uint32_t)m;
        }
        word = acc - 1u;                                   // sum (bit-1) 2^(31-k) = W - (2^32-1)
        err2 = s - dither; err1 = g - target;
    } else if constexpr (V == 4) {          // select between the two candidate sums
        int32_t s = err2 + dither, g = err1 + target;
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const int32_t c0 = s + g, c1 = s + g - 131070;
            const int32_t g0 = g + target, g1 = g + target - 65535;
            const bool bit = s >= 0;
            s = bit ? c1 : c0;
            g = bit ? g1 : g0;
            word = word * 2u + (bit ? 1u : 0u);
        }
        err2 = s - dither; err1 = g - target;
    } else if constexpr (V == 5) {          // like 3 but the word is assembled from sign masks with one LOP3 per 2 bits
        int32_t s = err2 + dither, g = err1 + target;
        const int32_t tg = target - 65535;
        uint32_t inv = 0;
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const int32_t m = s >> 31;
            const int32_t t2 = s + g - 131070;
            const int32_t g2 = g + tg;
            s = m * -131070 + t2;
            g = m * -65535 + g2;
            inv |= (uint32_t)m & (1u << (31 - k));
        }
        word = ~inv;
        err2 = s - dither; err1 = g - target;
    } else if constexpr (V == 6) {          // fp32: every quantity is an integer below 2^24 in magnitude (guarded), so float adds and
                                            // fmas are exact; the comparator is one saturating add, the correction one fma: 2 dependent
                                            // 4-cycle FMA-pipe ops per decision.  Falls back to the integer form when the guard trips.
        const int32_t e1 = err1, e2 = err2;
        float s = (float)(err2 + dither), g = (float)(err1 + target);
        const float tf = (float)target;
        float hi = 0.0f, lo = 0.0f, ms = fabsf(s), mg = fabsf(g);
        bool ok = abs(err2 + dither) < (1 << 23) && abs(err1 + target) < (1 << 23);
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const float b = __saturatef(s + 1.0f);            // 1.0 when s >= 0 (s is an integer), else 0.0
            const float t2 = s + g;
            const float g2 = g + tf;
            s = fmaf(b, -131070.0f, t2);
            g = fmaf(b, -65535.0f, g2);
            if (k < 16) hi = fmaf(hi, 2.0f, b); else lo = fmaf(lo, 2.0f, b);
            ms = fmaxf(ms, fabsf(s));
            mg = fmaxf(mg, fabsf(g));
        }
        ok = ok && ms < 8000000.0f && mg < 8000000.0f;        // every intermediate (s + g, g + target) stayed below 2^24
        if (ok) {
            word = ((uint32_t)hi << 16) | (uint32_t)lo;
            err2 = (int32_t)s - dither; err1 = (int32_t)g - target;
        } else {
            err1 = e1; err2 = e2;
            word = chunk<5>(err1, err2, target, dither);
        }
    } else if constexpr (V == 7) {          // three running sums: the addends of all three IMADs depend on the PREVIOUS step only, so the
                                            // per-decision chain is IMAD -> SHF -> IMAD with no operand arriving late:
                                            //   t2 = s + g - 2K,  g2 = g + target - K;   m = s >> 31
                                            //   s' = m * -2K + t2;   t2' = m * -3K + (t2 + g2 - 2K);   g2' = m * -K + (g2 + target - K)
        int32_t sv = err2 + dither;
        const int32_t g0 = err1 + target, tg = target - 65535;
        int32_t t2 = sv + g0 - 131070, g2 = g0 + tg;
        uint32_t inv = 0;
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const int32_t m = sv >> 31;
            const int32_t a = t2 + g2 - 131070;
            const int32_t b = g2 + tg;
            inv |= (uint32_t)m & (1u << (31 - k));
            sv = m * -131070 + t2;
            t2 = m * -196605 + a;
            g2 = m * -65535 + b;
        }
        word = ~inv;
        err2 = sv - dither;
        err1 = g2 - tg - target;                               // g2 = g + tg, g = err1 + target
    } else if constexpr (V == 10) {
        // V7 with the sign mask taken on the FMA pipe too (mul.hi.s32 by 1 = s >> 31): no pipe crossing in the chain
        int32_t sv = err2 + dither;
        const int32_t g0 = err1 + target, tg = target - 65535;
        int32_t t2 = sv + g0 - 131070, g2 = g0 + tg;
        uint32_t inv = 0;
        int32_t one;
        asm volatile("mov.s32 %0, 1;" : "=r"(one));
#pragma unroll
        for (int k = 0; k < 32; k++) {
            int32_t m;
            asm("mul.hi.s32 %0, %1, %2;" : "=r"(m) : "r"(sv), "r"(one));
            const int32_t a = t2 + g2 - 131070;
            const int32_t b = g2 + tg;
            inv = __funnelshift_l((uint32_t)sv, inv, 1);
            sv = m * -131070 + t2;
            t2 = m * -196605 + a;
            g2 = m * -65535 + b;
        }
        word = ~inv;
        err2 = sv - dither;
        err1 = g2 - tg - target;
    } else if constexpr (V == 8 || V == 9) {
        // speculative two-step look-ahead on the three sums of V7 (z = -m, K = 65535):
        //   one step:  s' = t2 + 2K z;  t2' = (t2 + g2 - 2K) + 3K z;  g2' = (g2 + tg) + K z
        //   the second comparator sees s' = t2 (z0 = 0) or t2 + 2K (z0 = 1): both signs are taken BEFORE z0 is known and one LOP3 selects
        //   two steps: s'' = A + 3K z0 + 2K z1;  t2'' = B + 4K z0 + 3K z1;  g2'' = G + K z0 + K z1
        //              A = t2 + g2 - 2K,  B = t2 + 2 g2 + tg - 4K,  G = g2 + 2 tg
        // chain per PAIR of decisions: shift -> select -> IMAD (V9 carries u2 = t2 + 2K as a fourth sum so that its sign needs no add first)
        int32_t sv = err2 + dither;
        const int32_t g0 = err1 + target, tg = target - 65535;
        int32_t t2 = sv + g0 - 131070, g2 = g0 + tg, u2 = t2 + 131070;
        const int32_t cB = tg - 131070, tg2 = 2 * tg;
        uint32_t inv = 0;
#pragma unroll
        for (int k = 0; k < 32; k += 2) {
            const int32_t m0 = sv >> 31;
            const int32_t ma = t2 >> 31;
            const int32_t mb = (V == 9 ? u2 : t2 + 131070) >> 31;
            const int32_t A = t2 + g2 - 131070;
            const int32_t B = A + g2 + cB;
            const int32_t G = g2 + tg2;
            inv = __funnelshift_l((uint32_t)sv, inv, 1);
            const int32_t m1 = (m0 & mb) | (~m0 & ma);
            const int32_t pS = m0 * -196605 + A;
            const int32_t pT = m0 * -262140 + B;
            const int32_t pG = m0 * -65535 + G;
            inv = __funnelshift_l((uint32_t)m1, inv, 1);
            sv = m1 * -131070 + pS;
            t2 = m1 * -196605 + pT;
            g2 = m1 * -65535 + pG;
            if (V == 9) u2 = m1 * -196605 + (pT + 131070);
        }
        word = ~inv;
        err2 = sv - dither;
        err1 = g2 - tg - target;
    }
    return word;
}

// U chunks of 32 decisions unrolled per loop iteration: straight-line code size vs the instruction caches
// (chain_pdm.cuh unrolls a whole 256-bit frame = 8 chunks)
template <int U>
__global__ void ku(int32_t *st, uint32_t *out, long long *cyc, int iters)
{
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    int32_t err1 = st[tid * 2], err2 = st[tid * 2 + 1];
    const int32_t target = 32768 + (tid * 37 % 20000) - 10000;
    uint32_t h = 0;
    const long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < iters; it += U) {
#pragma unroll
        for (int c = 0; c < U; c++) {
            const int32_t dither = (int32_t)((h >> 7) & 255) - 128;
            h = h * 1664525u + chunk<5>(err1, err2, target, dither);
        }
        err1 -= err1 >> 16; err2 -= err2 >> 16;
    }
    const long long t1 = clock64();
    out[tid] = h ^ (uint32_t)err1 ^ (uint32_t)err2;
    if (threadIdx.x % 32 == 0) cyc[tid / 32] = t1 - t0;
}

template <int U>
void run_u(int32_t *st, uint32_t *out, long long *cyc)
{
    const int iters = 4096, nsm = 132, w = 4;
    ku<U><<<nsm, 32 * w>>>(st, out, cyc, iters);
    cudaDeviceSynchronize();
    ku<U><<<nsm, 32 * w>>>(st, out, cyc, iters);
    cudaDeviceSynchronize();
    static long long h_cyc[132 * 16];
    cudaMemcpy(h_cyc, cyc, sizeof(long long) * nsm * w, cudaMemcpyDeviceToHost);
    long long mx = 0;
    for (int i = 0; i < nsm * w; i++) mx = h_cyc[i] > mx ? h_cyc[i] : mx;
    printf("imad two-sum, %d chunks unrolled per iteration: cycles/bit %.2f (%s)\n", U, (double)mx / (iters * 32.0), cudaGetErrorString(cudaGetLastError()));
}

template <int V>
__global__ void k(int32_t *st, uint32_t *out, long long *cyc, int iters)
{
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    int32_t err1 = st[tid * 2], err2 = st[tid * 2 + 1];
    const int32_t target = 32768 + (tid * 37 % 20000) - 10000;
    uint32_t h = 0;
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        const int32_t dither = (int32_t)((h >> 7) & 255) - 128;
        h = h * 1664525u + chunk<V>(err1, err2, target, dither);
        if ((it & 7) == 7) { err1 -= err1 >> 16; err2 -= err2 >> 16; }
    }
    const long long t1 = clock64();
    out[tid] = h ^ (uint32_t)err1 ^ (uint32_t)err2;
    if (threadIdx.x % 32 == 0) cyc[tid / 32] = t1 - t0;
}

template <int V>
void run(const char *name, int32_t *st, uint32_t *out, long long *cyc, int warps_per_sm)
{
    const int iters = 4096, nsm = 132;
    k<V><<<nsm, 32 * warps_per_sm>>>(st, out, cyc, iters);
    cudaDeviceSynchronize();
    k<V><<<nsm, 32 * warps_per_sm>>>(st, out, cyc, iters);
    cudaDeviceSynchronize();
    static uint32_t h_out[132 * 512];
    static long long h_cyc[132 * 16];
    cudaMemcpy(h_out, out, sizeof(uint32_t) * nsm * 32 * warps_per_sm, cudaMemcpyDeviceToHost);
    cudaMemcpy(h_cyc, cyc, sizeof(long long) * nsm * warps_per_sm, cudaMemcpyDeviceToHost);
    long long mx = 0;
    for (int i = 0; i < nsm * warps_per_sm; i++) mx = h_cyc[i] > mx ? h_cyc[i] : mx;
    uint32_t x = 0;
    for (int i = 0; i < nsm * 32 * warps_per_sm; i++) x = x * 31 + h_out[i];
    printf("%-28s warps/SM %2d  cycles/bit %.2f  checksum %08x  (%s)\n", name, warps_per_sm, (double)mx / (iters * 32.0), x, cudaGetErrorString(cudaGetLastError()));
}

int main()
{
    int32_t *st; uint32_t *out; long long *cyc;
    cudaMalloc(&st, 132 * 512 * 8); cudaMalloc(&out, 132 * 512 * 4); cudaMalloc(&cyc, 132 * 16 * 8);
    cudaMemset(st, 0, 132 * 512 * 8);
    run_u<1>(st, out, cyc); run_u<2>(st, out, cyc); run_u<4>(st, out, cyc); run_u<8>(st, out, cyc); run_u<16>(st, out, cyc);
    for (int w : {4, 8, 16}) {
        run<0>("reference shape", st, out, cyc, w);
        run<1>("mask form (old)", st, out, cyc, w);
        run<2>("predicated two-sum", st, out, cyc, w);
        run<3>("imad two-sum", st, out, cyc, w);
        run<4>("select two-sum", st, out, cyc, w);
        run<5>("imad two-sum, lop3 word", st, out, cyc, w);
        run<6>("fp32 saturating-add two-sum", st, out, cyc, w);
        run<7>("imad three-sum", st, out, cyc, w);
        run<10>("three-sum, sign by IMAD.HI", st, out, cyc, w);
        run<8>("two-step look-ahead, 3 sums", st, out, cyc, w);
        run<9>("two-step look-ahead, 4 sums", st, out, cyc, w);
    }
    return 0;
}
