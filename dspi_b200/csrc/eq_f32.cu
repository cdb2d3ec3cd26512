// eq_f32.cu — K1: float32 10-band EQ cascade (Cytomic SVF / TDF2 biquad hybrid) for
// thousands of independent channels, sm_90a.
//
// Reference semantics: dsp_process_channel_block(), firmware/DSPi/dsp_pipeline.c:281-365
// (band outer / sample inner, in place; the per-sample twin :256-279 yields the same values).
//
// Mapping
//   * one warp owns a GROUP of 32*CPL channels for the whole launch; lane L carries channel
//     L (and L+32 when CPL==2, held in the two halves of a 64-bit register pair) — the
//     serial sample recurrence and all coefficients/state of the 10 bands live in registers;
//   * samples are channel-major [C][T] in HBM; each warp streams its [32*CPL][64/CPL] tiles
//     through a private 3-stage shared-memory ring with TMA (cp.async.bulk.tensor, 128-byte
//     swizzle, mbarrier completion) and writes results back with TMA stores from the same
//     buffers — no block-wide synchronisation anywhere;
//   * CPL==1 (the default) moves 256 B of each row per transfer; CPL==2 (DSPI_F32_CPL=2)
//     moves 128 B but gives every lane two independent recurrences (two scalar FFMAs per
//     operation on sm_90).  Both fill 8 warps x 3 stages x 8 KB of shared memory per SM.
//
// Arithmetic is written with explicit-rounding intrinsics only, so nvcc can neither contract
// nor reassociate: FUSED follows GCC's -ffp-contract=fast pattern (what arm-none-eabi-gcc
// emits for the RP2350), !FUSED rounds every operation separately.  -ftz=true gives the
// firmware's FZ mode (main.c:593-600).  Negations are kept out of the inner loops (packed
// ops have no free negate): a1/a2 are stored negated, `a - b` is fma(b, -1, a) (exact), and
// the SVF state alternates sign every sample (see svf_tile() in eq_core.cuh).
#include "eq_kernels.cuh"
#include "eq_f32_kernel.cuh"

namespace dspi {
namespace {

using namespace core;
using k1::kStageBytes;
using k1::kStages;
using k1::kWarps;

template <typename V, bool FUSED, int NB, bool DYN>
__global__ void __launch_bounds__(kWarps * 32, 1)
eq_f32_kernel(const __grid_constant__ CUtensorMap tmap, float *__restrict__ samples, uint32_t ld, V *__restrict__ coef,
              const uint64_t *__restrict__ modes, uint32_t n_groups, uint32_t n_rows, uint32_t row_lo, uint32_t T, uint32_t nb_active, uint32_t use_tma,
              uint32_t dbg, unsigned long long nz_bits, uint32_t slice_tiles, uint32_t *__restrict__ sched)
{
    k1::eq_f32_body<V, FUSED, NB, DYN, k1::NoSig>(tmap, samples, ld, coef, modes, n_groups, n_rows, row_lo, T, nb_active, use_tma, dbg, nz_bits, slice_tiles, sched);
}

template <typename V, bool FUSED, int NB>
cudaError_t launch_one(const EqLaunch &a, cudaStream_t stream)
{
    constexpr int kTileT = k1::tile_t<V>();
    constexpr size_t smem = (size_t)kWarps * kStages * kStageBytes;
    auto kern = eq_f32_kernel<V, FUSED, NB, false>;
    auto kern_dyn = eq_f32_kernel<V, FUSED, NB, true>;
    static PerDeviceOnce once;                                  // per instantiation
    int dev = 0;
    if (once.needs(&dev)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kern_dyn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        once.mark(dev);
    }
    const uint32_t n_groups = a.n_groups;
    uint32_t grid = (n_groups + kWarps - 1) / kWarps;
    uint32_t slice_tiles = 0;
    uint32_t *sched = nullptr;
    const uint32_t ntiles = (a.T + kTileT - 1) / kTileT;
    // The dynamic schedule is opt-in (DSPI_DBG=8): a scheduler left with ONE resident warp runs it well
    // below half the two-warp rate, which eats the balance it buys (DESIGN.md, K1).
    if (a.sched && a.use_tma && a.T >= 1024 && (a.dbg & 8u)) {
        slice_tiles = 512 / kTileT;                             // time slices of 512 samples in either geometry
        sched = a.sched;
        if (grid > (uint32_t)a.n_sms) grid = a.n_sms;
        else if (grid < (uint32_t)a.n_sms && (uint32_t)a.n_sms * kWarps <= n_groups * ((ntiles + slice_tiles - 1) / slice_tiles)) grid = a.n_sms;
        cudaError_t e = cudaMemsetAsync(sched, 0, (size_t)(1 + n_groups) * sizeof(uint32_t), stream);
        if (e != cudaSuccess) return e;
    }
    if (sched)
        kern_dyn<<<grid, kWarps * 32, smem, stream>>>(a.tmap, (float *)a.samples, a.ld, (V *)a.coef, a.modes, n_groups, a.n_rows, a.row_lo, a.T, a.n_bands, a.use_tma,
                                                      a.dbg, 0x8000000080000000ull, slice_tiles, sched);
    else
        kern<<<grid, kWarps * 32, smem, stream>>>(a.tmap, (float *)a.samples, a.ld, (V *)a.coef, a.modes, n_groups, a.n_rows, a.row_lo, a.T, a.n_bands, a.use_tma,
                                                  a.dbg, 0x8000000080000000ull, 0u, nullptr);
    return cudaGetLastError();
}

template <typename V, bool FUSED>
cudaError_t launch_nb(const EqLaunch &a, cudaStream_t stream)
{
    if (a.n_bands <= 10) return launch_one<V, FUSED, 10>(a, stream);
    return launch_one<V, FUSED, 12>(a, stream);
}

}  // namespace

cudaError_t launch_eq_f32(const EqLaunch &a, bool fused, int cpl, cudaStream_t stream)
{
    if (cpl == 2) return fused ? launch_nb<P2, true>(a, stream) : launch_nb<P2, false>(a, stream);
    return fused ? launch_nb<float, true>(a, stream) : launch_nb<float, false>(a, stream);
}

// ---------------------------------------------------------------------------------------
// Biquad[n][12] (reference layout, AoS) <-> packed device store
// ---------------------------------------------------------------------------------------
__global__ void pack_f32_kernel(const dspi_biquad_f32 *__restrict__ aos, uint32_t ch0, uint32_t n, float *__restrict__ coef,
                                uint64_t *__restrict__ modes, int cpl, RoleRange rr)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (rr.reject && rr.reject[i])) return;
    const uint32_t ch = ch0 + blockIdx.y * rr.stride + (rr.inst ? rr.inst[i] : i);
    const uint32_t rows = 32 * cpl;
    const uint32_t g = ch / rows, r = ch % rows, lane = r & 31, h = r >> 5;
    uint64_t mw = 0;
    for (int b = 0; b < kMaxBands; b++) {
        const dspi_biquad_f32 &q = aos[(size_t)ch * kMaxBands + b];
        float v[8];
        uint32_t mode;
        if (q.bypass) mode = kModeBypass;
        else if (!q.use_svf) mode = kModeTdf2;
        else mode = q.svf_type == DSPI_FILTER_LOWPASS ? kModeSvfLP : q.svf_type == DSPI_FILTER_HIGHPASS ? kModeSvfHP
                  : q.svf_type == DSPI_FILTER_PEAKING ? kModeSvfPK : kModeSvfSH;
        if (q.use_svf && !q.bypass) {
            v[0] = q.sva1; v[1] = q.sva2; v[2] = q.sva3; v[3] = q.svm0; v[4] = q.svm1; v[5] = q.svm2;
            v[6] = q.svic1eq; v[7] = q.svic2eq;
        } else {
            v[0] = q.b0; v[1] = q.b1; v[2] = q.b2; v[3] = -q.a1; v[4] = -q.a2; v[5] = 0.0f;
            v[6] = q.s1; v[7] = q.s2;
        }
        mw |= (uint64_t)mode << (4 * b);
        for (int k = 0; k < 8; k++) coef[((((size_t)g * kMaxBands + b) * 8 + k) * 32 + lane) * cpl + h] = v[k];
    }
    modes[(size_t)g * rows + h * 32 + lane] = mw;
}

__global__ void unpack_f32_kernel(dspi_biquad_f32 *__restrict__ aos, uint32_t ch0, uint32_t n, const float *__restrict__ coef, int cpl, RoleRange rr)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (rr.reject && rr.reject[i])) return;
    const uint32_t ch = ch0 + blockIdx.y * rr.stride + (rr.inst ? rr.inst[i] : i);
    const uint32_t rows = 32 * cpl;
    const uint32_t g = ch / rows, r = ch % rows, lane = r & 31, h = r >> 5;
    for (int b = 0; b < kMaxBands; b++) {
        dspi_biquad_f32 &q = aos[(size_t)ch * kMaxBands + b];
        if (q.bypass) continue;
        const float s0 = coef[((((size_t)g * kMaxBands + b) * 8 + 6) * 32 + lane) * cpl + h];
        const float s1 = coef[((((size_t)g * kMaxBands + b) * 8 + 7) * 32 + lane) * cpl + h];
        if (q.use_svf) { q.svic1eq = s0; q.svic2eq = s1; }
        else { q.s1 = s0; q.s2 = s1; }
    }
}

cudaError_t launch_pack_f32(const dspi_biquad_f32 *aos, uint32_t ch0, uint32_t n, float *coef, uint64_t *modes, int cpl, cudaStream_t stream,
                            const RoleRange &rr)
{
    if (n == 0) return cudaSuccess;
    pack_f32_kernel<<<dim3((n + 127) / 128, rr.roles), 128, 0, stream>>>(aos, ch0, n, coef, modes, cpl, rr);
    return cudaGetLastError();
}
__global__ void mask_modes_kernel(const uint64_t *__restrict__ raw, const uint8_t *__restrict__ skip, uint64_t *__restrict__ eff, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) eff[i] = skip[i] ? 0ull : raw[i];
}
cudaError_t launch_mask_modes(const uint64_t *raw, const uint8_t *skip, uint64_t *eff, uint32_t n, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    mask_modes_kernel<<<(n + 255) / 256, 256, 0, stream>>>(raw, skip, eff, n);
    return cudaGetLastError();
}
cudaError_t launch_unpack_f32(dspi_biquad_f32 *aos, uint32_t ch0, uint32_t n, const float *coef, int cpl, cudaStream_t stream,
                              const RoleRange &rr)
{
    if (n == 0) return cudaSuccess;
    unpack_f32_kernel<<<dim3((n + 127) / 128, rr.roles), 128, 0, stream>>>(aos, ch0, n, coef, cpl, rr);
    return cudaGetLastError();
}

}  // namespace dspi
