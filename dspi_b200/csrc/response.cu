// response.cu — frequency response of EQ engine channels (dspi_eq_response_*), sm_90a.
//
// Reads the engine's reference-layout mirror (Biquad[c_pad][12]), which every coefficient upload and device-side
// generation writes before it packs: the response does not depend on the K1 stage geometry or the packed store, and it
// touches neither.  A CTA takes a tile of kTile channels: their active bands (b < n_bands, not bypassed) are turned into
// sections once, in shared memory; then every thread takes one frequency, evaluates w = e^{-j omega} once and runs the
// tile's cascades, accumulating numerator and denominator products with one complex division per channel.  Stores are
// float2 {re, im}, consecutive threads on consecutive frequencies of one channel row (coalesced).
#include "eq_kernels.cuh"
#include "response.cuh"

namespace dspi {
namespace {

constexpr int kTile = 16;                  // channels per CTA
constexpr int kThreads = 128;              // frequencies per CTA

template <typename Bq>
__global__ void __launch_bounds__(kThreads)
eq_response_kernel(const Bq *__restrict__ aos, uint32_t ch0, uint32_t n, uint32_t nb, const float *__restrict__ freqs, uint32_t nf, float fs,
                   float2 *__restrict__ out)
{
    __shared__ Sect sec[kTile][DSPI_MAX_BANDS];
    __shared__ int cnt[kTile];
    const uint32_t f = blockIdx.x * kThreads + threadIdx.x;
    const float fr = f < nf ? freqs[f] : 0.0f;
    const Trig t = trig_at(fr, fs);
    const uint32_t n_tiles = (n + kTile - 1) / kTile;
    for (uint32_t tile = blockIdx.y; tile < n_tiles; tile += gridDim.y) {
        const uint32_t c0 = tile * kTile;
        __syncthreads();
        if (threadIdx.x < kTile && c0 + threadIdx.x < n) {
            const Bq *row = aos + (size_t)(ch0 + c0 + threadIdx.x) * DSPI_MAX_BANDS;
            int k = 0;
            for (uint32_t b = 0; b < nb; b++) {
                Sect s;
                if (sect_band(row[b], s)) sec[threadIdx.x][k++] = s;
            }
            cnt[threadIdx.x] = k;
        }
        __syncthreads();
        if (f < nf) {
            const uint32_t m = min((uint32_t)kTile, n - c0);
            for (uint32_t c = 0; c < m; c++) out[(size_t)(c0 + c) * nf + f] = to_float2(cascade_eval(sec[c], cnt[c], t));
        }
    }
}

}  // namespace

cudaError_t launch_eq_response(bool q28, const void *aos, uint32_t ch0, uint32_t n, uint32_t nb, const float *d_freq, uint32_t nf, float fs,
                               void *d_out, cudaStream_t stream)
{
    const uint32_t n_tiles = (n + kTile - 1) / kTile;
    const dim3 grid((nf + kThreads - 1) / kThreads, n_tiles < 65535u ? n_tiles : 65535u);
    if (q28) eq_response_kernel<<<grid, kThreads, 0, stream>>>((const dspi_biquad_q28 *)aos, ch0, n, nb, d_freq, nf, fs, (float2 *)d_out);
    else eq_response_kernel<<<grid, kThreads, 0, stream>>>((const dspi_biquad_f32 *)aos, ch0, n, nb, d_freq, nf, fs, (float2 *)d_out);
    return cudaGetLastError();
}

}  // namespace dspi
