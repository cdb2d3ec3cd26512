// eq_q28.cu — K2: Q28 fixed-point 10-band TDF2 cascade (RP2040 arithmetic), bit-exact, sm_90a.
//
// Reference semantics: dsp_process_channel_block() in firmware/DSPi/dsp_process_rp2040.S:225-394;
// every multiply is fast_mul_q28() (dsp_pipeline.c:47-58):
//     mul(c, x) = ((c>>16)*(x>>16) << 4) + (((c>>16)*(x&0xFFFF) + (c&0xFFFF)*(x>>16)) >> 12)
// in 32-bit wrapping arithmetic with the lo*lo partial product dropped.
//
// Mapping: one channel per lane, one warp per group of 32 channels, all coefficients of the
// 10 bands pre-split into (c>>16, c&0xFFFF, (c>>16)<<4) and held in registers together with
// s1/s2; samples stream through the same per-warp TMA ring as the float kernel (eq_f32.cu).
// Per multiply: 3 IMAD + 1 SHF; the path is bound by the integer pipes, not by HBM.
#include <cstdlib>
#include "eq_kernels.cuh"

namespace dspi {
namespace {

constexpr int kTileT = 32;
constexpr int kStages = 3;
constexpr int kWarps = 8;
constexpr int kRows = 32;
constexpr uint32_t kStageBytes = kRows * kTileT * 4;
constexpr int kSlots = 20;      // per band: 5 x {hi, lo, hi<<4}, s1, s2, bypass, 2 pad

struct QCoef { int32_t hi; uint32_t lo; uint32_t hi16; };

// fast_mul_q28(c, x) with c pre-split and x given as (xh = x>>16, xl = x&0xFFFF)
__device__ __forceinline__ uint32_t mulq(const QCoef &c, int32_t xh, uint32_t xl)
{
    const uint32_t mid = (uint32_t)c.hi * xl + c.lo * (uint32_t)xh;          // mid1 + mid2 (wraps)
    return c.hi16 * (uint32_t)xh + (uint32_t)((int32_t)mid >> 12);            // (high << 4) + (mid >> 12)
}

// dsp_process_rp2040.S:263-365, one band over a register tile
template <int N>
__device__ __forceinline__ void q28_tile(uint32_t (&x)[N], const QCoef (&c)[5], uint32_t &s1, uint32_t &s2)
{
#pragma unroll
    for (int i = 0; i < N; i++) {
        const int32_t xh = (int32_t)x[i] >> 16;
        const uint32_t xl = x[i] & 0xFFFFu;
        const uint32_t y = mulq(c[0], xh, xl) + s1;                          // :273-285
        const uint32_t t1 = mulq(c[1], xh, xl);                              // :288-298
        const uint32_t t3 = mulq(c[2], xh, xl);                              // :301-312
        const int32_t yh = (int32_t)y >> 16;
        const uint32_t yl = y & 0xFFFFu;
        const uint32_t t2 = mulq(c[3], yh, yl);                              // :319-329
        const uint32_t t4 = mulq(c[4], yh, yl);                              // :338-348
        s1 = (t1 - t2) + s2;                                                 // :332-335
        s2 = t3 - t4;                                                        // :351-353
        x[i] = y;
    }
}

__device__ __noinline__ uint2 q28_slow_band(uint32_t *xs, int n, const int32_t *cf /*5 raw coefficients*/, uint32_t s1, uint32_t s2)
{
    QCoef c[5];
    for (int k = 0; k < 5; k++) { c[k].hi = cf[k] >> 16; c[k].lo = (uint32_t)cf[k] & 0xFFFFu; c[k].hi16 = (uint32_t)c[k].hi << 4; }
    for (int i = 0; i < n; i++) {
        const int32_t xh = (int32_t)xs[i] >> 16;
        const uint32_t xl = xs[i] & 0xFFFFu;
        const uint32_t y = mulq(c[0], xh, xl) + s1;
        const uint32_t t1 = mulq(c[1], xh, xl), t3 = mulq(c[2], xh, xl);
        const int32_t yh = (int32_t)y >> 16;
        const uint32_t yl = y & 0xFFFFu;
        const uint32_t t2 = mulq(c[3], yh, yl), t4 = mulq(c[4], yh, yl);
        s1 = (t1 - t2) + s2;
        s2 = t3 - t4;
        xs[i] = y;
    }
    return make_uint2(s1, s2);
}

template <int NB, int kSub>
__global__ void __launch_bounds__(kWarps * 32, 1)
eq_q28_kernel(const __grid_constant__ CUtensorMap tmap, int32_t *__restrict__ samples, uint32_t ld, int32_t *__restrict__ coef,
              uint32_t n_groups, uint32_t n_rows, uint32_t T, uint32_t nb_active, uint32_t use_tma, uint32_t no_plain)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ uint64_t bars[kWarps][kStages];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t g = blockIdx.x * kWarps + warp;
    if (g >= n_groups) return;

    uint8_t *my_smem = smem_raw + (size_t)warp * kStages * kStageBytes;
    uint64_t *full = bars[warp];
    if (lane == 0) {
        if (use_tma) prefetch_tmap(&tmap);
        for (int s = 0; s < kStages; s++) mbar_init(&full[s], 1);
        fence_mbar_init();
    }
    __syncwarp();

    const int c0 = g * kRows;
    const uint32_t ntiles = (T + kTileT - 1) / kTileT;
    auto issue_load = [&](uint32_t tile) {
        const uint32_t s = tile % kStages;
        mbar_arrive_expect_tx(&full[s], kStageBytes);
        tma_load_2d(my_smem + s * kStageBytes, &tmap, &full[s], tile * kTileT, c0);
    };
    if (use_tma && lane == 0)
        for (uint32_t s = 0; s + 1 < kStages && s < ntiles; s++) issue_load(s);

    QCoef c[NB][5];
    uint32_t s1[NB], s2[NB];
    uint32_t byp = 0;                                           // bit b: this lane's band b is bypassed
    int32_t *cg = coef + (size_t)g * kMaxBands * kSlots * 32;
#pragma unroll
    for (int b = 0; b < NB; b++) {
#pragma unroll
        for (int k = 0; k < 5; k++) {
            c[b][k].hi = cg[(b * kSlots + 3 * k + 0) * 32 + lane];
            c[b][k].lo = (uint32_t)cg[(b * kSlots + 3 * k + 1) * 32 + lane];
            c[b][k].hi16 = (uint32_t)cg[(b * kSlots + 3 * k + 2) * 32 + lane];
        }
        s1[b] = (uint32_t)cg[(b * kSlots + 15) * 32 + lane];
        s2[b] = (uint32_t)cg[(b * kSlots + 16) * 32 + lane];
        if (cg[(b * kSlots + 17) * 32 + lane]) byp |= 1u << b;
    }
    if (cg[18 * 32 + lane]) byp = (1u << NB) - 1u;              // whole row frozen (chain engines: eq_set_skip)
    uint32_t all_byp = 0, any_byp = 0;
#pragma unroll
    for (int b = 0; b < NB; b++) {
        if (__all_sync(0xffffffffu, (byp >> b) & 1u)) all_byp |= 1u << b;
        if (__any_sync(0xffffffffu, (byp >> b) & 1u)) any_byp |= 1u << b;
    }

    const uint32_t sw = (lane & 7) << 4;
    const bool straight = nb_active >= (uint32_t)NB && all_byp == 0 && !no_plain;
    for (uint32_t tile = 0; tile < ntiles; tile++) {
        const uint32_t s = tile % kStages;
        uint8_t *buf = my_smem + s * kStageBytes;
        if (use_tma) {
            mbar_wait(&full[s], (tile / kStages) & 1);
        } else {
            const uint32_t t = tile * kTileT + lane;
            for (int r = 0; r < kRows; r++) {
                const uint32_t ch = c0 + r;
                int32_t v = 0;
                if (t < T && ch < n_rows) v = samples[(size_t)ch * ld + t];
                *reinterpret_cast<int32_t *>(buf + r * 128 + ((((lane >> 2) << 4) ^ ((r & 7) << 4)) | ((lane & 3) << 2))) = v;
            }
            __syncwarp();
        }
        const int tile_valid = min((int)kTileT, (int)(T - tile * kTileT));
#pragma unroll 1
        for (int sub = 0; sub < kTileT / kSub; sub++) {
            const int nvalid = min(kSub, tile_valid - sub * kSub);
            if (nvalid <= 0) break;
            uint8_t *row = buf + lane * 128;
            uint32_t x[kSub];
#pragma unroll
            for (int h = 0; h < kSub / 4; h++) {                              // 16-byte chunks of this lane's row, chunk index XOR (row & 7)
                const uint4 q = *reinterpret_cast<const uint4 *>(row + ((((kSub / 4) * sub + h) << 4) ^ sw));
                x[4 * h] = q.x; x[4 * h + 1] = q.y; x[4 * h + 2] = q.z; x[4 * h + 3] = q.w;
            }
            // Warps in which no band can be skipped outright get ONE straight-line block over all bands, so that ptxas overlaps
            // band b+1's first samples with band b's last ones (the per-band branches below fence the scheduler).  Lanes with a
            // bypassed band keep their input and state through selects instead of a branch.
            if (straight && nvalid == kSub) {
                if (any_byp == 0) {
#pragma unroll
                    for (int b = 0; b < NB; b++) q28_tile(x, c[b], s1[b], s2[b]);
                } else {
#pragma unroll
                    for (int b = 0; b < NB; b++) {
                        uint32_t keep[kSub];
#pragma unroll
                        for (int i = 0; i < kSub; i++) keep[i] = x[i];
                        const uint32_t k1 = s1[b], k2 = s2[b];
                        q28_tile(x, c[b], s1[b], s2[b]);
                        const bool off = (byp >> b) & 1u;
#pragma unroll
                        for (int i = 0; i < kSub; i++) x[i] = off ? keep[i] : x[i];
                        s1[b] = off ? k1 : s1[b];
                        s2[b] = off ? k2 : s2[b];
                    }
                }
            } else
#pragma unroll
            for (int b = 0; b < NB; b++) {
                if (b >= (int)nb_active) break;
                if ((all_byp >> b) & 1u) continue;                           // bypass byte set: .S:246-248
                if (nvalid == kSub && !((any_byp >> b) & 1u)) {
                    q28_tile(x, c[b], s1[b], s2[b]);
                } else if (nvalid == kSub) {                                 // some lanes bypass this band
                    uint32_t keep[kSub];
#pragma unroll
                    for (int i = 0; i < kSub; i++) keep[i] = x[i];
                    const uint32_t k1 = s1[b], k2 = s2[b];
                    q28_tile(x, c[b], s1[b], s2[b]);
                    if ((byp >> b) & 1u) {
#pragma unroll
                        for (int i = 0; i < kSub; i++) x[i] = keep[i];
                        s1[b] = k1; s2[b] = k2;
                    }
                } else {                                                     // tail of the launch
                    uint32_t xs[kSub];
                    int32_t cf[5];
#pragma unroll
                    for (int i = 0; i < kSub; i++) xs[i] = x[i];
#pragma unroll
                    for (int k = 0; k < 5; k++) cf[k] = (int32_t)(((uint32_t)c[b][k].hi << 16) | c[b][k].lo);
                    if (!((byp >> b) & 1u)) {
                        const uint2 ns = q28_slow_band(xs, nvalid, cf, s1[b], s2[b]);
                        s1[b] = ns.x; s2[b] = ns.y;
                    }
#pragma unroll
                    for (int i = 0; i < kSub; i++) x[i] = xs[i];
                }
            }
#pragma unroll
            for (int h = 0; h < kSub / 4; h++)
                *reinterpret_cast<uint4 *>(row + ((((kSub / 4) * sub + h) << 4) ^ sw)) = make_uint4(x[4 * h], x[4 * h + 1], x[4 * h + 2], x[4 * h + 3]);
        }
        if (use_tma) {
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) {
                tma_store_2d(&tmap, buf, tile * kTileT, c0);
                tma_store_commit();
                const uint32_t nxt = tile + kStages - 1;
                if (nxt < ntiles) {
                    tma_store_wait_read<1>();
                    issue_load(nxt);
                }
            }
        } else {
            __syncwarp();
            const uint32_t t = tile * kTileT + lane;
            for (int r = 0; r < kRows; r++) {
                const uint32_t ch = c0 + r;
                const int32_t v = *reinterpret_cast<const int32_t *>(buf + r * 128 + ((((lane >> 2) << 4) ^ ((r & 7) << 4)) | ((lane & 3) << 2)));
                if (t < T && ch < n_rows) samples[(size_t)ch * ld + t] = v;
            }
            __syncwarp();
        }
    }
    if ((uint32_t)(c0 + lane) < n_rows) {                       // rows past the end of a range call are channels outside it
#pragma unroll
        for (int b = 0; b < NB; b++) {
            cg[(b * kSlots + 15) * 32 + lane] = (int32_t)s1[b];
            cg[(b * kSlots + 16) * 32 + lane] = (int32_t)s2[b];
        }
    }
    if (use_tma && lane == 0) tma_store_wait_all<0>();
}

template <int NB, int SUB>
cudaError_t launch_one(const EqLaunch &a, cudaStream_t stream)
{
    constexpr size_t smem = (size_t)kWarps * kStages * kStageBytes;
    auto kern = eq_q28_kernel<NB, SUB>;
    static PerDeviceOnce once;
    int dev = 0;
    if (once.needs(&dev)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        once.mark(dev);
    }
    const uint32_t grid = (a.n_groups + kWarps - 1) / kWarps;
    static const uint32_t no_plain = [] { const char *e = getenv("DSPI_K2_PLAIN"); return (e && atoi(e) == 0) ? 1u : 0u; }();
    kern<<<grid, kWarps * 32, smem, stream>>>(a.tmap, (int32_t *)a.samples, a.ld, (int32_t *)a.coef, a.n_groups, a.n_rows, a.T, a.n_bands, a.use_tma, no_plain);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_eq_q28(const EqLaunch &a, cudaStream_t stream)
{
    // register tile of 8 or 4 samples (DSPI_K2_SUB): the straight-line body is 10 bands x tile x ~27 instructions, 35 KB at 8.
    // Halving it shortens the body but leaves less independent work between dependent IMADs; 8 is the default.
    static const int sub = [] { const char *e = getenv("DSPI_K2_SUB"); return (e && atoi(e) == 8) ? 8 : ((e && atoi(e) == 4) ? 4 : 8); }();
    if (a.n_bands <= 10) return sub == 4 ? launch_one<10, 4>(a, stream) : launch_one<10, 8>(a, stream);
    return sub == 4 ? launch_one<12, 4>(a, stream) : launch_one<12, 8>(a, stream);
}

__global__ void pack_q28_kernel(const dspi_biquad_q28 *__restrict__ aos, uint32_t ch0, uint32_t n, int32_t *__restrict__ coef, RoleRange rr)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (rr.reject && rr.reject[i])) return;
    const uint32_t ch = ch0 + blockIdx.y * rr.stride + (rr.inst ? rr.inst[i] : i), g = ch / 32, lane = ch % 32;
    for (int b = 0; b < kMaxBands; b++) {
        const dspi_biquad_q28 &q = aos[(size_t)ch * kMaxBands + b];
        int32_t *dst = coef + ((size_t)g * kMaxBands + b) * kSlots * 32 + lane;
        const int32_t cf[5] = { q.b0, q.b1, q.b2, q.a1, q.a2 };
        for (int k = 0; k < 5; k++) {
            const int32_t hi = cf[k] >> 16;
            dst[(3 * k + 0) * 32] = hi;
            dst[(3 * k + 1) * 32] = (int32_t)((uint32_t)cf[k] & 0xFFFFu);
            dst[(3 * k + 2) * 32] = (int32_t)((uint32_t)hi << 4);
        }
        dst[15 * 32] = q.s1;
        dst[16 * 32] = q.s2;
        dst[17 * 32] = q.bypass ? 1 : 0;
    }
}

// row skip flags (chain engines): slot 18 of band 0
__global__ void skip_q28_kernel(int32_t *__restrict__ coef, const uint8_t *__restrict__ skip, uint32_t n)
{
    const uint32_t ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= n) return;
    coef[((size_t)(ch / 32) * kMaxBands * kSlots + 18) * 32 + ch % 32] = skip[ch] ? 1 : 0;
}
cudaError_t launch_skip_q28(int32_t *coef, const uint8_t *skip, uint32_t n, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    skip_q28_kernel<<<(n + 255) / 256, 256, 0, stream>>>(coef, skip, n);
    return cudaGetLastError();
}

__global__ void unpack_q28_kernel(dspi_biquad_q28 *__restrict__ aos, uint32_t ch0, uint32_t n, const int32_t *__restrict__ coef, RoleRange rr)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (rr.reject && rr.reject[i])) return;
    const uint32_t ch = ch0 + blockIdx.y * rr.stride + (rr.inst ? rr.inst[i] : i), g = ch / 32, lane = ch % 32;
    for (int b = 0; b < kMaxBands; b++) {
        dspi_biquad_q28 &q = aos[(size_t)ch * kMaxBands + b];
        const int32_t *src = coef + ((size_t)g * kMaxBands + b) * kSlots * 32 + lane;
        q.s1 = src[15 * 32];
        q.s2 = src[16 * 32];
    }
}

cudaError_t launch_pack_q28(const dspi_biquad_q28 *aos, uint32_t ch0, uint32_t n, int32_t *coef, cudaStream_t stream, const RoleRange &rr)
{
    if (n == 0) return cudaSuccess;
    pack_q28_kernel<<<dim3((n + 127) / 128, rr.roles), 128, 0, stream>>>(aos, ch0, n, coef, rr);
    return cudaGetLastError();
}
cudaError_t launch_unpack_q28(dspi_biquad_q28 *aos, uint32_t ch0, uint32_t n, const int32_t *coef, cudaStream_t stream, const RoleRange &rr)
{
    if (n == 0) return cudaSuccess;
    unpack_q28_kernel<<<dim3((n + 127) / 128, rr.roles), 128, 0, stream>>>(aos, ch0, n, coef, rr);
    return cudaGetLastError();
}

}  // namespace dspi
