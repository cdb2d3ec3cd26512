// chain_streams.cuh — stream/event plumbing shared by the float and the Q28 chain engines.
//
// One process call is cut into packet slices and the three stages of a slice (front, outputs, PDM
// modulator) run on three streams chained by events: stage k of slice i+1 overlaps stage k+1 of slice i.
// Each stage is a set of serial recurrences with too few warps to fill the machine on its own (the
// modulator: one warp per 32 instances), so running them side by side is what fills it.  All state
// lives in HBM between slices and every slice touches its own frames of the intermediate buffers, so
// neither the slicing nor the overlap changes a bit.
//
// SM partition for the modulator.  The delta-sigma loop is ONE serial dependence chain per instance (two dependent
// integer operations per one-bit decision, 256 decisions per frame): it is latency-bound, wants one warp per SM
// sub-partition with nothing else competing for that scheduler's issue slots, and it is the longest stage of a call.
// Sharing SMs with the streaming stages slows exactly that chain down (their CTAs land on its SMs), and its resident
// CTAs keep K1 - which needs a whole SM's register file per CTA - off those SMs.  So the engine splits the GPU with CUDA
// green contexts: `pdm_sms` SMs run nothing but the modulator, every other kernel of the call runs on the rest
// (scripts/greenctx_probe.cu checks that a split is honoured, no SM shared).  The driver entry points are looked up at
// run time; without them (or with DSPI_PDM_SMS=0) the three priority streams of round 1 are used and results are the same.
#pragma once
#include <cstdlib>
#include <cuda.h>
#include <cuda_runtime.h>

namespace dspi {

struct GreenApi {
    decltype(&cuDeviceGetDevResource) DeviceGetDevResource = nullptr;
    decltype(&cuDevSmResourceSplitByCount) DevSmResourceSplitByCount = nullptr;
    decltype(&cuDevResourceGenerateDesc) DevResourceGenerateDesc = nullptr;
    decltype(&cuGreenCtxCreate) GreenCtxCreate = nullptr;
    decltype(&cuGreenCtxDestroy) GreenCtxDestroy = nullptr;
    decltype(&cuGreenCtxStreamCreate) GreenCtxStreamCreate = nullptr;
    bool ok = false;
    static const GreenApi &get()
    {
        static const GreenApi api = [] {
            GreenApi a;
            auto sym = [](const char *name) -> void * {
                void *p = nullptr;
                cudaDriverEntryPointQueryResult q;
                if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); return nullptr; }
                return p;
            };
            a.DeviceGetDevResource = (decltype(a.DeviceGetDevResource))sym("cuDeviceGetDevResource");
            a.DevSmResourceSplitByCount = (decltype(a.DevSmResourceSplitByCount))sym("cuDevSmResourceSplitByCount");
            a.DevResourceGenerateDesc = (decltype(a.DevResourceGenerateDesc))sym("cuDevResourceGenerateDesc");
            a.GreenCtxCreate = (decltype(a.GreenCtxCreate))sym("cuGreenCtxCreate");
            a.GreenCtxDestroy = (decltype(a.GreenCtxDestroy))sym("cuGreenCtxDestroy");
            a.GreenCtxStreamCreate = (decltype(a.GreenCtxStreamCreate))sym("cuGreenCtxStreamCreate");
            a.ok = a.DeviceGetDevResource && a.DevSmResourceSplitByCount && a.DevResourceGenerateDesc && a.GreenCtxCreate && a.GreenCtxDestroy &&
                   a.GreenCtxStreamCreate;
            return a;
        }();
        return api;
    }
};

// The engine's split of the GPU, made once per engine: every set of stage streams (the engine's own and each lane's,
// chain_host.cuh) is created in these two contexts with the same priorities, so that the modulator keeps its SMs to
// itself however many lanes run.
struct SmPartition {
    CUgreenCtx g_pdm = nullptr, g_rest = nullptr;
    unsigned pdm_sms = 0, rest_sms = 0;                       // 0: no partition (priority streams on the whole GPU)
    unsigned all_sms = 0;                                     // SM count of the device
    int prio_hi = 0, prio_mid = 0, prio_lo = 0;               // numerically lower = higher priority

    // SMs the streaming stages run on
    unsigned stream_sms() const { return rest_sms ? rest_sms : all_sms; }

    // modulator CTAs are 128 threads (one warp per sub-partition): ceil(instances / 128) SMs, in the partition granularity of 8,
    // at most 48.  On a 132-SM H100 SXM at 8192 instances, 48 modulator SMs beat 56 and 64 by 1-3 % per call (both chains)
    // and 72 or 80 lose 10-25 %: the other stages need the SMs more.
    static unsigned wanted_pdm_sms(unsigned n_instances)
    {
        if (const char *e = getenv("DSPI_PDM_SMS")) return (unsigned)atoi(e);
        unsigned want = ((n_instances + 127u) / 128u + 7u) / 8u * 8u;
        return want > 48u ? 48u : want;
    }

    bool create_partition(int device, unsigned want)
    {
        const GreenApi &ga = GreenApi::get();
        if (!ga.ok || want == 0) return false;
        CUdevResource sm, part, rest;
        unsigned groups = 1;
        if (ga.DeviceGetDevResource((CUdevice)device, &sm, CU_DEV_RESOURCE_TYPE_SM) != CUDA_SUCCESS) return false;
        if (want + 8 > sm.sm.smCount) return false;
        if (ga.DevSmResourceSplitByCount(&part, &groups, &sm, &rest, 0, want) != CUDA_SUCCESS || groups != 1 || rest.sm.smCount == 0) return false;
        CUdevResourceDesc d_part, d_rest;
        if (ga.DevResourceGenerateDesc(&d_part, &part, 1) != CUDA_SUCCESS || ga.DevResourceGenerateDesc(&d_rest, &rest, 1) != CUDA_SUCCESS) return false;
        if (ga.GreenCtxCreate(&g_pdm, d_part, (CUdevice)device, CU_GREEN_CTX_DEFAULT_STREAM) != CUDA_SUCCESS) { g_pdm = nullptr; return false; }
        if (ga.GreenCtxCreate(&g_rest, d_rest, (CUdevice)device, CU_GREEN_CTX_DEFAULT_STREAM) != CUDA_SUCCESS) { g_rest = nullptr; destroy(); return false; }
        pdm_sms = part.sm.smCount; rest_sms = rest.sm.smCount;
        return true;
    }

    // the priorities, the SM count and, for n_instances > 0, the split (none when the driver cannot make one)
    cudaError_t create(int device = 0, unsigned n_instances = 0)
    {
        int lo = 0, hi = 0;
        cudaError_t e = cudaDeviceGetStreamPriorityRange(&lo, &hi);
        int n_sms = 0;
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, device);
        all_sms = (unsigned)n_sms;
        // the modulator is the longest serial chain: its few CTAs are placed first whenever an SM frees a
        // slot; then the front; the many output CTAs fill what is left
        prio_hi = hi; prio_mid = hi < lo ? hi + 1 : lo; prio_lo = lo;
        if (e == cudaSuccess && n_instances && !create_partition(device, wanted_pdm_sms(n_instances))) cudaGetLastError();
        return e;
    }

    // a stream of priority `prio` in green context g (a plain priority stream when there is no partition)
    cudaError_t stream(CUgreenCtx g, cudaStream_t *s, int prio) const
    {
        if (!g) return cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, prio);
        CUstream cs = nullptr;
        if (GreenApi::get().GreenCtxStreamCreate(&cs, g, CU_STREAM_NON_BLOCKING, prio) != CUDA_SUCCESS) return cudaErrorUnknown;
        *s = (cudaStream_t)cs;
        return cudaSuccess;
    }

    void destroy()
    {
        const GreenApi &ga = GreenApi::get();
        if (g_pdm) { ga.GreenCtxDestroy(g_pdm); g_pdm = nullptr; }
        if (g_rest) { ga.GreenCtxDestroy(g_rest); g_rest = nullptr; }
        pdm_sms = rest_sms = 0;
    }
};

// The stage streams and events of one issue context (an engine's or a lane's).
struct ChainStreams {
    static constexpr int kMaxSlices = 16;

    // Packet slices of one call: bounds[0..n] (packet indices), returns n.  The modulator can only start once the first
    // slice has been through every other stage and it still has its last slice to do when the others are finished, so the
    // slices are short at both ends (1, 2, 4 packets ... 2, 1) and long (about 8 packets: launch overheads amortised, K1
    // tiles full) in the middle.  DSPI_UNIFORM_SLICES=1 restores the eight equal slices of round 1 for comparison.
    static int plan_slices(uint32_t n_packets, uint32_t *bounds)
    {
        int n = 0;
        bounds[0] = 0;
        const char *uni = getenv("DSPI_UNIFORM_SLICES");                // "1": eight equal slices; "n": n equal slices (<= 16)
        if (uni && uni[0] >= '1' && uni[0] <= '9') {
            uint32_t want = (uint32_t)atoi(uni);
            if (want == 1u) want = 8u;
            if (want > (uint32_t)kMaxSlices) want = (uint32_t)kMaxSlices;
            const uint32_t k = n_packets < want ? n_packets : want;
            for (uint32_t i = 1; i <= k; i++) bounds[i] = (uint32_t)((uint64_t)n_packets * i / k);
            return (int)k;
        }
        if (n_packets <= 8u) {
            for (uint32_t i = 1; i <= n_packets; i++) bounds[i] = i;
            return (int)n_packets;
        }
        const uint32_t head[3] = { 1, 2, 4 }, tail_rev[2] = { 1, 2 };      // the call ends ... 2, 1
        uint32_t used = 0;
        for (uint32_t h : head) if (used + h <= n_packets / 3) { used += h; bounds[++n] = used; }
        uint32_t tail_sum = 0, tail_n = 0;
        for (uint32_t t : tail_rev) if (used + tail_sum + t <= n_packets / 2) { tail_sum += t; tail_n++; }
        const uint32_t middle = n_packets - used - tail_sum;
        uint32_t m = (middle + 7) / 8;
        const uint32_t room = (uint32_t)kMaxSlices - (uint32_t)n - tail_n;
        if (m > room) m = room;
        if (m < 1) m = 1;
        for (uint32_t i = 1; i <= m; i++) bounds[++n] = used + (uint32_t)((uint64_t)middle * i / m);
        used += middle;
        for (uint32_t i = tail_n; i > 0; i--) { used += tail_rev[i - 1]; bounds[++n] = used; }
        return n;
    }
    cudaStream_t s_front = nullptr, s_out = nullptr, s_pdm = nullptr;
    cudaEvent_t ev_begin = nullptr, ev_done = nullptr, ev_aux = nullptr, ev_front[kMaxSlices] = {}, ev_out[kMaxSlices] = {};

    // the three stage streams in the partition's contexts (or priority streams without one), and the events.  This and
    // destroy() stay out of line: the library has always exported them.
    __noinline__ cudaError_t create(const SmPartition &p)
    {
        cudaError_t e = p.stream(p.g_pdm, &s_pdm, p.prio_hi);
        if (e == cudaSuccess) e = p.stream(p.g_rest, &s_front, p.prio_mid);
        if (e == cudaSuccess) e = p.stream(p.g_rest, &s_out, p.prio_lo);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_begin, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_done, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_aux, cudaEventDisableTiming);
        for (int i = 0; i < kMaxSlices && e == cudaSuccess; i++) {
            e = cudaEventCreateWithFlags(&ev_front[i], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_out[i], cudaEventDisableTiming);
        }
        return e;
    }

    __noinline__ void destroy()
    {
        for (cudaStream_t *s : { &s_front, &s_out, &s_pdm })
            if (*s) { cudaStreamSynchronize(*s); cudaStreamDestroy(*s); *s = nullptr; }
        for (cudaEvent_t *ev : { &ev_begin, &ev_done, &ev_aux })
            if (*ev) { cudaEventDestroy(*ev); *ev = nullptr; }
        for (int i = 0; i < kMaxSlices; i++) {
            if (ev_front[i]) { cudaEventDestroy(ev_front[i]); ev_front[i] = nullptr; }
            if (ev_out[i]) { cudaEventDestroy(ev_out[i]); ev_out[i] = nullptr; }
        }
    }
};

}  // namespace dspi
