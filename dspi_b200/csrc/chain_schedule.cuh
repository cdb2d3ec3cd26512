// chain_schedule.cuh — the packet schedule of one chain process call, shared by the float and the Q28 chain engines.
//
// process_audio_packet() runs once per USB packet of whatever length the host sent (usb_audio.c:500), and three stages
// depend on that length: the leveller's block gain, the preset-mute envelope and the "last packet" meters.  A call
// carries n packets of packet_frames[p] frames each, the same for every instance of the call.  The kernels find packet
// p at frames off[p] .. off[p+1] of the call's rows; off lives in engine-owned device memory sized for the longest
// possible schedule (max_frames packets of one frame).
//
// The offsets reach the device as kernel parameters: schedule_kernel copies one chunk of up to kChunk offsets from its
// parameter block into d_off, on the engine stream.  The launch captures the parameters when it is issued, so no host
// buffer has to outlive the call and the host never waits for the device; everything issued on the stream before (the
// previous call's kernels included) has finished with d_off by the time the copy runs.  One launch covers every
// schedule of up to kChunk - 1 packets (7.9 s of audio in 96-frame packets at 96 kHz).
#pragma once
#include <cstdint>
#include <cstring>
#include <new>
#include <vector>
#include <cuda_runtime.h>
#include "dspi_b200.h"

namespace dspi {

constexpr uint32_t kChunk = 7936;                 // parameter block of schedule_kernel: 31.8 KB of the 32 KB sm_90 allows
struct OffChunk { uint32_t first, count, v[kChunk]; };

namespace {
__global__ void __launch_bounds__(256) schedule_kernel(uint32_t *__restrict__ d_off, const OffChunk chunk)
{
    for (uint32_t i = threadIdx.x; i < chunk.count; i += blockDim.x) d_off[chunk.first + i] = chunk.v[i];
}
}  // namespace

struct PacketSchedule {
    uint32_t cap = 0;                          // max_frames: the most packets (and frames) of one call
    uint32_t *d_off = nullptr;                 // [cap + 1] device: frame offsets of the current call's packets
    std::vector<uint32_t> off;                 // [cap + 1] host offsets of the current call (slice bounds)
    OffChunk *chunk = nullptr;                 // parameter block under construction
    uint32_t n_packets = 0, frames = 0, longest = 0;

    __noinline__ cudaError_t create(uint32_t max_frames)     // out of line: the library has always exported it
    {
        cap = max_frames;
        off.assign((size_t)cap + 1, 0u);
        chunk = new (std::nothrow) OffChunk;
        if (!chunk) return cudaErrorMemoryAllocation;
        return cudaMalloc((void **)&d_off, ((size_t)cap + 1) * sizeof(uint32_t));
    }

    void destroy()
    {
        if (d_off) { cudaFree(d_off); d_off = nullptr; }
        delete chunk;
        chunk = nullptr;
    }

    // Checks a caller's table: DSPI_EINVAL for a NULL table, no packets or a length outside 1..DSPI_PACKET_MAX,
    // DSPI_ERANGE when the frames add up to more than max_frames.  Sets n_packets, frames and longest.
    int check(uint32_t n, const uint16_t *packet_frames, const char **why)
    {
        if (!packet_frames) { *why = "packet_frames is NULL"; return DSPI_EINVAL; }
        if (n == 0) { *why = "n_packets must be > 0"; return DSPI_EINVAL; }
        uint64_t sum = 0;
        uint32_t mx = 0;
        for (uint32_t p = 0; p < n; p++) {
            const uint32_t k = packet_frames[p];
            if (k == 0 || k > DSPI_PACKET_MAX) { *why = "every packet length must be 1..192 frames"; return DSPI_EINVAL; }
            sum += k;
            if (k > mx) mx = k;
        }
        if (sum > cap) { *why = "the packets add up to more than max_frames"; return DSPI_ERANGE; }
        n_packets = n; frames = (uint32_t)sum; longest = mx;
        return DSPI_OK;
    }

    // After a successful check(): the offsets on the host, then into d_off on `stream`; *launches counts the copy kernels.
    cudaError_t upload(const uint16_t *packet_frames, cudaStream_t stream, uint64_t *launches)
    {
        off[0] = 0;
        for (uint32_t p = 0; p < n_packets; p++) off[p + 1] = off[p] + packet_frames[p];
        for (uint32_t first = 0; first <= n_packets; first += kChunk) {
            chunk->first = first;
            chunk->count = n_packets + 1 - first < kChunk ? n_packets + 1 - first : kChunk;
            memcpy(chunk->v, off.data() + first, (size_t)chunk->count * sizeof(uint32_t));
            schedule_kernel<<<1, 256, 0, stream>>>(d_off, *chunk);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return e;
            ++*launches;
        }
        return cudaSuccess;
    }
};

// Packet of frame T of the call: the last p <= hi with off[p] <= T (off[0] = 0).  A binary search over the offsets:
// it needs no per-frame table (nothing more to build or copy per call), and only envelope-mode instances ask for it,
// mostly for a T inside packet hi, which the first comparison settles.
__device__ __forceinline__ uint32_t packet_of(const uint32_t *__restrict__ off, uint32_t T, uint32_t hi)
{
    if (off[hi] <= T) return hi;
    uint32_t lo = 0;
    hi--;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (off[mid] <= T) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

}  // namespace dspi
