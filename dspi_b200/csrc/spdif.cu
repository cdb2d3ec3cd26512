// spdif.cu — S/PDIF (IEC 60958) subframe encoder for the chain's 24-bit word streams, sm_90a.
// The step right after the hot path (SURVEY.md §8 f-3): what the firmware does with every S/PDIF
// producer buffer before the PIO serialiser sees it.
//
// Reference (firmware/pico-extras/src/rp2_common/pico_audio_spdif_multi/):
//   spdif_update_subframe   include/pico/audio_spdif/sample_encoding.h:27-50   (3 table look-ups per sample)
//   table                   audio_spdif.c:141-153   (byte -> 16-bit biphase-mark word + parity)
//   preambles / channel status / validity-user-status-parity cells   audio_spdif.c:73-114, :372-388
//   caller                  sample_encoding.cpp:42-50 (stereo S32 producer: one update per subframe)
//
// One thread encodes one stereo frame: 8 bytes in (two 24-bit words), 16 bytes out (two subframes of
// {l, h}), both fully coalesced — 24 algorithmic bytes per frame, HBM-bound by design.  The encoding
// itself (table written out as arithmetic) is spdif_bmc.cuh, shared with the chain engines, which can
// also write subframes straight from their output stage (dspi_chain(q)_process_subframes_*).  This pass
// stays for words that come from elsewhere.
#include <cstdio>
#include <cstdarg>

#include "eq_kernels.cuh"
#include "spdif_bmc.cuh"

namespace dspi {
namespace {

int fail(int code, const char *fmt, ...)
{
    size_t cap = 0;
    char *buf = error_buffer(&cap);
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, cap, fmt, ap);
    va_end(ap);
    return code;
}

__global__ void __launch_bounds__(256)
spdif_encode_kernel(const int2 *__restrict__ words, uint4 *__restrict__ out, uint64_t n_streams, uint32_t frames, uint32_t pos0, uint64_t cs40)
{
    // grid.x walks the frames of a stream, grid.y the streams: no 64-bit division anywhere
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= frames) return;
    const uint32_t pos = (pos0 + n) % 192u;
    const uint32_t c = spdif_cs_bit(pos, cs40);
    const uint32_t pre_l = spdif_pre_left(pos);
    for (uint64_t s = blockIdx.y; s < n_streams; s += gridDim.y) {
        const uint64_t i = s * frames + n;
        const int2 w = words[i];
        out[i] = encode_frame(w, pre_l, c);
    }
}

}  // namespace
}  // namespace dspi

using dspi::fail;

#define CU_OK(expr)                                                                                         \
    do {                                                                                                    \
        cudaError_t err__ = (expr);                                                                         \
        if (err__ != cudaSuccess) return fail(DSPI_ECUDA, "%s -> %s (%s:%d)", #expr, cudaGetErrorString(err__), __FILE__, __LINE__); \
    } while (0)

extern "C" {

void dspi_spdif_lookup_table(uint32_t table[256])
{
    for (uint32_t i = 0; i < 256; i++) {                                     // audio_spdif.c:141-153
        uint32_t v = 0x5555, p = 0;
        for (uint32_t j = 0; j < 8; j++)
            if (i & (1u << j)) { p ^= 1; v |= 2u << (j * 2); }
        table[i] = v | (p << 16);
    }
}

static int spdif_check(int device, const void *a, const void *b, const uint8_t *cs, uint32_t frames)
{
    if (!a || !b || !cs) return fail(DSPI_EINVAL, "null argument");
    if (frames == 0) return fail(DSPI_EINVAL, "frames must be > 0");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(DSPI_ENODEV, "no CUDA device (there is no CPU fallback)"); }
    if (device < 0 || device >= ndev) return fail(DSPI_ENODEV, "device %d out of range (%d visible)", device, ndev);
    int major = 0;
    CU_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    if (major != 9) return fail(DSPI_ENODEV, "device %d is not sm_90", device);
    return DSPI_OK;
}

int dspi_spdif_encode_device(int device, const int32_t *d_words, uint64_t n_streams, uint32_t frames, uint32_t block_pos0,
                             const uint8_t channel_status[5], dspi_spdif_subframe *d_subframes, void *cuda_stream)
{
    int rc = spdif_check(device, d_words, d_subframes, channel_status, frames);
    if (rc) return rc;
    if (n_streams == 0) return DSPI_OK;
    if (((uintptr_t)d_words & 7) || ((uintptr_t)d_subframes & 15)) return fail(DSPI_EINVAL, "words must be 8-byte and subframes 16-byte aligned");
    CU_OK(cudaSetDevice(device));
    uint64_t cs40 = 0;
    for (int i = 0; i < 5; i++) cs40 |= (uint64_t)channel_status[i] << (8 * i);
    int n_sms = 0;
    CU_OK(cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, device));
    const uint32_t bx = (frames + 255) / 256;
    // enough CTAs for ~4 waves of 8 resident CTAs per SM; every CTA then loops over streams
    uint64_t by = ((uint64_t)n_sms * 8 * 4 + bx - 1) / bx;
    if (by > n_streams) by = n_streams;
    if (by > 65535) by = 65535;
    if (by == 0) by = 1;
    dspi::spdif_encode_kernel<<<dim3(bx, (unsigned)by), 256, 0, (cudaStream_t)cuda_stream>>>((const int2 *)d_words, (uint4 *)d_subframes, n_streams, frames,
                                                                                            block_pos0 % 192u, cs40);
    CU_OK(cudaGetLastError());
    return DSPI_OK;
}

int dspi_spdif_encode_host(int device, const int32_t *words, uint64_t n_streams, uint32_t frames, uint32_t block_pos0,
                           const uint8_t channel_status[5], dspi_spdif_subframe *subframes)
{
    int rc = spdif_check(device, words, subframes, channel_status, frames);
    if (rc) return rc;
    if (n_streams == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(device));
    const size_t in_bytes = (size_t)n_streams * frames * 8, out_bytes = in_bytes * 2;
    void *d_in = nullptr, *d_out = nullptr;
    cudaStream_t s = nullptr;
    cudaError_t e = cudaMalloc(&d_in, in_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&d_out, out_bytes);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_in, words, in_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        rc = dspi_spdif_encode_device(device, (const int32_t *)d_in, n_streams, frames, block_pos0, channel_status, (dspi_spdif_subframe *)d_out, s);
        if (rc == DSPI_OK) e = cudaMemcpyAsync(subframes, d_out, out_bytes, cudaMemcpyDeviceToHost, s);
        if (rc == DSPI_OK && e == cudaSuccess) e = cudaStreamSynchronize(s);
    }
    if (s) cudaStreamDestroy(s);
    if (d_in) cudaFree(d_in);
    if (d_out) cudaFree(d_out);
    if (rc) return rc;
    if (e != cudaSuccess) return fail(e == cudaErrorMemoryAllocation ? DSPI_ENOMEM : DSPI_ECUDA, "S/PDIF host path: %s", cudaGetErrorString(e));
    return DSPI_OK;
}

}  // extern "C"
