// chain_host.cuh — the host half of the float and Q28 chain engines (chain_f32.cu, chain_q28.cu): engine record,
// lifetime, argument checks, parameter uploads, the stage pipeline over packet slices, host staging, S/PDIF transmitter
// state, checkpoints and the frequency response.  Host code, and the two record kernels of the lane getters; each engine
// file includes it after its kernels.
//
// Everything here is a template over the engine's arithmetic traits A, which supply what differs between the two
// engines: the types (A::Dev the device record, A::Biquad, A::Status, A::Params, A::Stores the device-side parameter
// stores), the constants (A::kOuts, A::kRoles, A::kMaxDelay, A::kLoudRows coefficient rows of the loudness shelves,
// A::kXs the post kernel's shared-memory column stride, A::kStateVersion of the blobs it writes), the kernels the host
// launches (A::scatter, A::dynamics, A::response, and per kernel set K of A::with_stages: K::pre, K::post, K::mix,
// K::outpost<SUBFRAMES>, K::ring, K::pdm, K::env, K::status) and the hooks
//   A::check_desc(desc)                       arithmetic, instance / frame counts and band count of a new engine
//   A::alloc_leveller(c)                      the leveller state arrays
//   A::leveller_arrays(c, v)                  their entries in the table of per-instance arrays, with their reset values
//   A::pack(params, i, n, rows)               volumes, preamp, loudness and matrix / output gains of one instance
// The code below never asks which arithmetic it serves.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <type_traits>
#include <utility>
#include <vector>

#include "bulk_ingest.cuh"
#include "chain_schedule.cuh"
#include "chain_streams.cuh"
#include "eq_kernels.cuh"
#include "instance_image.cuh"
#include "response.cuh"
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

#define CU_OK(expr)                                                                                         \
    do {                                                                                                    \
        cudaError_t err__ = (expr);                                                                         \
        if (err__ != cudaSuccess) return fail(DSPI_ECUDA, "%s -> %s (%s:%d)", #expr, cudaGetErrorString(err__), __FILE__, __LINE__); \
    } while (0)

// device copy of the instance lists of *_copy_instances (sources, then destinations); the engine's grows to the largest
// call, a lane's holds its whole window from its first copy as destination
struct IndexLists {
    uint32_t *d = nullptr;
    uint32_t cap = 0;                // pairs
    cudaError_t ensure(uint32_t n)
    {
        if (n <= cap) return cudaSuccess;
        cudaFree(d);
        d = nullptr; cap = 0;
        cudaError_t e = cudaMalloc((void **)&d, (size_t)2 * n * sizeof(uint32_t));
        if (e == cudaSuccess) cap = n;
        return e;
    }
    void destroy()
    {
        cudaFree(d);
        d = nullptr; cap = 0;
    }
};

// A lane's device staging of its host process calls (process_lane_host) and the two copy streams that move each packet
// slice in and out while the stage streams run.  Every buffer holds the whole window at max_frames, so that no later call
// grows it; each is allocated by the first call that needs it: PCM, status, streams and events by the first host call,
// PDM by the first one with PDM out, S/PDIF by the first one with words (8 bytes per pair frame) or subframes (16; a
// later subframe call after words replaces the words buffer once).  Freed when the lane closes.
struct HostStage {
    void *d_pcm = nullptr;                   // [n][max_frames] frames of up to 6 bytes
    void *d_status = nullptr;                // [n] status records
    uint32_t *d_pdm = nullptr;               // [n][max_frames][8]
    void *d_spdif = nullptr;                 // [n][pairs][max_frames] pair frames of spdif_frame bytes
    size_t spdif_frame = 0;
    cudaStream_t s_in = nullptr, s_back = nullptr;   // host to device (PCM), device to host (S/PDIF, PDM)
    cudaEvent_t ev_back = nullptr, ev_in[ChainStreams::kMaxSlices] = {}, ev_pdm[ChainStreams::kMaxSlices] = {};

    bool has(size_t sf, bool pdm) const { return s_in && (!pdm || d_pdm) && sf <= spdif_frame; }

    // a window of n instances of pairs S/PDIF pairs and status records of status_bytes; after has() was false, every
    // lane and the engine stream drained
    cudaError_t ensure(size_t n, size_t max_frames, size_t pairs, size_t status_bytes, size_t sf, bool pdm)
    {
        cudaError_t e = cudaSuccess;
        if (!s_in) {
            e = cudaStreamCreateWithFlags(&s_in, cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s_back, cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_back, cudaEventDisableTiming);
            for (int i = 0; i < ChainStreams::kMaxSlices && e == cudaSuccess; i++) {
                e = cudaEventCreateWithFlags(&ev_in[i], cudaEventDisableTiming);
                if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_pdm[i], cudaEventDisableTiming);
            }
            if (e == cudaSuccess) e = cudaMalloc(&d_pcm, n * max_frames * 6);
            if (e == cudaSuccess) e = cudaMalloc(&d_status, n * status_bytes);
            if (e != cudaSuccess) { destroy(); return e; }
        }
        if (pdm && !d_pdm) e = cudaMalloc((void **)&d_pdm, n * max_frames * 8 * 4);
        if (e == cudaSuccess && sf > spdif_frame) {
            cudaFree(d_spdif);
            d_spdif = nullptr; spdif_frame = 0;
            e = cudaMalloc(&d_spdif, n * pairs * max_frames * sf);
            if (e == cudaSuccess) spdif_frame = sf;
        }
        return e;
    }

    void destroy()
    {
        for (cudaStream_t *s : { &s_in, &s_back })
            if (*s) { cudaStreamSynchronize(*s); cudaStreamDestroy(*s); *s = nullptr; }
        for (void **p : { &d_pcm, &d_status, (void **)&d_pdm, &d_spdif }) { cudaFree(*p); *p = nullptr; }
        spdif_frame = 0;
        if (ev_back) { cudaEventDestroy(ev_back); ev_back = nullptr; }
        for (int i = 0; i < ChainStreams::kMaxSlices; i++) {
            if (ev_in[i]) { cudaEventDestroy(ev_in[i]); ev_in[i] = nullptr; }
            if (ev_pdm[i]) { cudaEventDestroy(ev_pdm[i]); ev_pdm[i] = nullptr; }
        }
    }
};

// An issue queue: the stream a call is issued on and where it ends, the stage streams and packet schedule of its process
// calls, the staging of its control calls, and the instance window [inst0, inst0 + n) its calls may touch.  The engine
// issues on one over every instance (ChainHost::q).  A lane (dspi_chain_lane_*) is another, over its window: its calls
// start behind the engine stream as it was when they were issued (ev_engine) and end with ev_last, which engine-level calls
// wait for (join_lanes).  The device staging is allocated by the queue's first call that needs it.
struct Queue {
    bool lane = false;
    uint32_t inst0 = 0, n = 0;
    cudaStream_t stream = nullptr;   // the engine stream callers see, or the lane's; stages run on st.* between ev_begin and ev_done
    ChainStreams st;
    PacketSchedule sched;            // packet lengths of the current call
    bulk::Stage bulk;                // device staging of the bulk applies, rate switches, collects and edits
    bulk::EditStage bulk_edit;
    bulk::PresetStage preset;        // device staging of the preset applies and collects
    bulk::HostRing ring;             // a lane's edits, packets, images, rates, slot indices, fade rows and transmitter rows on their way to the device
    ResponseBuffers resp;            // frequency table of the response calls; image staging of export and import (and, the engine's, of _response_host)
    IndexLists copy_lists;           // device instance lists of the copies issued on this queue (the destination's, for a lane)
    HostStage host;                  // a lane's staging and copy streams of its host process calls
    cudaEvent_t ev_engine = nullptr, ev_last = nullptr;   // a lane's

    // `lane` set first
    cudaError_t create(const SmPartition &p, uint32_t max_frames)
    {
        cudaError_t e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
        if (e == cudaSuccess && lane) e = cudaEventCreateWithFlags(&ev_engine, cudaEventDisableTiming);
        if (e == cudaSuccess && lane) e = cudaEventCreateWithFlags(&ev_last, cudaEventDisableTiming);
        if (e == cudaSuccess) e = st.create(p);
        return e == cudaSuccess ? sched.create(max_frames) : e;
    }

    // waits for the queue's calls; a lane's queue is closed after it (no stream)
    void destroy()
    {
        if (stream) cudaStreamSynchronize(stream);
        st.destroy();
        sched.destroy();
        bulk.destroy();
        bulk_edit.destroy();
        preset.destroy();
        ring.destroy();
        resp.destroy();
        copy_lists.destroy();
        host.destroy();
        for (cudaEvent_t *ev : { &ev_engine, &ev_last })
            if (*ev) { cudaEventDestroy(*ev); *ev = nullptr; }
        if (stream) { cudaStreamDestroy(stream); stream = nullptr; }
    }
};

// One engine: dspi_chain and dspi_chainq are this record for their arithmetic.
template <class A>
struct ChainHost {
    using Arith = A;
    dspi_chain_desc desc;
    typename A::Dev d;
    Queue q;                         // the engine's own issue queue, over every instance
    SmPartition part;                // the modulator's SMs and the rest, shared by the engine's and the lanes' stage streams
    typename A::Biquad *d_aos;       // [N_pad][roles][12] instance-major mirror of filters[][]
    dspi_eq *eq_m, *eq_o;            // EQ engines over the master rows (2 N_pad channels) and the output rows (kOuts N_pad)
    std::vector<void *> allocs;
    uint64_t launches;
    void *d_pcm; size_t pcm_bytes;   // host-path staging
    int32_t *d_spdif; size_t spdif_bytes;   // host-path staging of the S/PDIF output, words or subframes
    uint32_t *d_pdmout; size_t pdmout_bytes;
    typename A::Status *d_status;
    SpdifTx tx;                      // S/PDIF transmitter state; not part of the state blob (*_get/set_spdif_tx)
    uint32_t env_instances;          // instances in envelope mode (0: the envelope kernel and its table are not needed)
    std::vector<uint8_t> env_mode;   // [N] each instance's envelope-mode flag (env row 4 != 0), as the calls issued so far leave it
    uint32_t vmm_packets;            // capacity of d.vmm in packets
    bulk::Record rec;                // wire-visible configuration of every instance (*_collect_bulk_device); not part of the state blob
    Queue lanes[DSPI_CHAIN_MAX_LANES];   // open while it has a stream
    uint32_t open_lanes;
};

// Engine-level calls run after every lane call issued before them: the engine stream waits for each open lane's last
// call.  Every engine-level entry point passes its handle through here (chain_abi.inc).  After lane control calls
// re-packed EQ rows, the K1 kernel choice is stale (eq_choice_stale): the first engine-level call waits for that work and
// re-selects it.  With no lane open and no lane control call since the last such call it does nothing.
template <class H>
H *join_lanes(H *c)
{
    if (!c) return c;
    const bool stale = eq_choice_stale(c->eq_m) || eq_choice_stale(c->eq_o);
    if (!c->open_lanes && !stale) return c;
    cudaSetDevice(c->desc.device);
    for (Queue &l : c->lanes)
        if (l.stream && cudaStreamWaitEvent(c->q.stream, l.ev_last, 0) != cudaSuccess) {
            cudaGetLastError();
            cudaStreamSynchronize(l.stream);                                // the same order, from the host
        }
    if (stale && cudaStreamSynchronize(c->q.stream) == cudaSuccess) {       // a failed choice leaves the ahead-of-time kernels
        if (eq_choice_stale(c->eq_m)) eq_refresh_choice(c->eq_m);
        if (eq_choice_stale(c->eq_o)) eq_refresh_choice(c->eq_o);
    }
    cudaGetLastError();
    return c;
}

// everything issued so far, on the engine stream and on every lane, has finished (before engine-owned buffers that lane
// calls read are reallocated)
template <class A>
cudaError_t drain(ChainHost<A> *c)
{
    for (Queue &l : c->lanes)
        if (l.stream) {
            const cudaError_t e = cudaStreamSynchronize(l.stream);
            if (e != cudaSuccess) return e;
        }
    return cudaStreamSynchronize(c->q.stream);
}

// the queue of an engine-level call, or of an open lane; NULL with the error set
template <class A>
Queue *engine_queue(ChainHost<A> *c)
{
    if (!c) fail(DSPI_EINVAL, "null argument");
    return c ? &c->q : nullptr;
}

template <class A>
Queue *lane_queue(ChainHost<A> *c, uint32_t lane)
{
    if (!c) { fail(DSPI_EINVAL, "null argument"); return nullptr; }
    if (lane >= DSPI_CHAIN_MAX_LANES || !c->lanes[lane].stream) { fail(DSPI_EINVAL, "lane %u is not open", lane); return nullptr; }
    return &c->lanes[lane];
}

// Every call on a queue is issued between these two, and they are all that differs between the engine's queue and a
// lane's.  A lane's call starts behind the engine stream as it is now and ends by recording ev_last; it does not wait for
// the device.  An engine-level call starts behind every lane (join_lanes, at its entry point) and returns once its work
// is done, unless it is a process call (`wait` false).  `rc` is what issuing the call returned.
template <class A>
cudaError_t begin_call(ChainHost<A> *c, Queue &q)
{
    if (!q.lane) return cudaSuccess;
    const cudaError_t e = cudaEventRecord(q.ev_engine, c->q.stream);
    return e == cudaSuccess ? cudaStreamWaitEvent(q.stream, q.ev_engine, 0) : e;
}

inline int end_call(Queue &q, int rc, bool wait = true)
{
    CU_OK(q.lane ? cudaEventRecord(q.ev_last, q.stream) : wait && rc == DSPI_OK ? cudaStreamSynchronize(q.stream) : cudaSuccess);
    return rc;
}

template <class A, typename T>
cudaError_t dev_alloc(ChainHost<A> *c, T **p, size_t count, bool zero = true)
{
    void *m = nullptr;
    cudaError_t e = cudaMalloc(&m, count * sizeof(T));
    if (e != cudaSuccess) return e;
    c->allocs.push_back(m);
    *p = (T *)m;
    return zero ? cudaMemsetAsync(m, 0, count * sizeof(T), c->q.stream) : cudaSuccess;
}

// instances [inst0, inst0 + n) inside the window of q
int check_range(const Queue &q, uint32_t inst0, uint32_t n)
{
    if (inst0 < q.inst0 || (uint64_t)inst0 + n > (uint64_t)q.inst0 + q.n)
        return fail(DSPI_ERANGE, "instances [%u, %llu) outside the %s [%u, %u)", inst0, (unsigned long long)inst0 + n,
                    q.lane ? "lane's window" : "engine's instances", q.inst0, q.inst0 + q.n);
    return DSPI_OK;
}

// ---- the per-instance arrays -------------------------------------------------------------------------------------------
// One table of every per-instance array of an engine, read by the state blob (state_sections), the pipeline reset
// (reset_range) and the instance images (image_plan).  Entry: `rows` rows of N_pad elements of `elem` bytes, element
// (r, i) at p + (r * N_pad + i) * elem; `use` says who reads it; a reset writes `one` into the rows of the mask `one_rows`
// (4-byte elements) and 0 into every other row.
enum : uint32_t {
    kInBlob = 1,     // a section of the state blob, in table order
    kInImage = 2,    // part of an instance image
    kReset = 4,      // cleared by reset_state / _reset_instances
};
struct InstArray {
    void *p;
    uint32_t rows, elem, use, one_rows, one;
};
template <typename T>
InstArray inst_array(T *p, uint32_t rows, uint32_t use, uint32_t elem = sizeof(T), uint32_t one_rows = 0, uint32_t one = 0)
{
    return InstArray{ (void *)p, rows, elem, use, one_rows, one };
}

template <class A>
void instance_arrays(ChainHost<A> *c, std::vector<InstArray> &v)
{
    constexpr uint32_t all = kInBlob | kInImage | kReset, O = A::kOuts;
    auto &d = c->d;
    // the state blob's sections, in the order its format fixes
    v.push_back(inst_array(d.loud_st, 8, all));
    v.push_back(inst_array(d.xf, 7, kInBlob | kInImage));                 // crossfeed coefficients and state (CrossfeedState)
    A::leveller_arrays(c, v);
    v.push_back(inst_array(d.lev_idx, 1, all));
    v.push_back(inst_array(d.lev_la, 2 * DSPI_LA_SAMPLES, all));
    v.push_back(inst_array(d.dline, O, all, A::kMaxDelay * (uint32_t)sizeof(*d.dline)));   // one ring per (output, instance)
    v.push_back(inst_array(d.widx_in, 1, all));
    v.push_back(inst_array(d.pdm, 9, all, 4, 1u << 7, 123456789u));      // dither seed, pdm_generator.c:62
    v.push_back(inst_array(d.peaks, A::kRoles, all));
    v.push_back(inst_array(d.clip, 1, all));
    v.push_back(inst_array(d.env, 5, kInBlob | kInImage));                // preset-mute envelope state and mode
    // rewritten from widx_in by every call
    v.push_back(inst_array(d.widx_out, 1, kReset));
    // the parameter rows set_params, _set_dynamics_device and _apply_bulk_device write
    v.push_back(inst_array(d.preamp, 2, kInImage));
    v.push_back(inst_array(d.flags, 1, kInImage));
    v.push_back(inst_array(d.loud_c, A::kLoudRows, kInImage));
    v.push_back(inst_array(d.loud_byp, 1, kInImage));
    v.push_back(inst_array(d.lev_c, 9, kInImage));
    v.push_back(inst_array(d.o_gl, O, kInImage));
    v.push_back(inst_array(d.o_gr, O, kInImage));
    v.push_back(inst_array(d.o_gain, O, kInImage));
    v.push_back(inst_array(d.o_glin, O, kInImage));
    v.push_back(inst_array(d.o_flags, O, kInImage));
    v.push_back(inst_array(d.o_dly, O, kInImage));
    v.push_back(inst_array(d.vol_base, 1, kInImage));
    v.push_back(inst_array(d.vol_master, 1, kInImage));
    v.push_back(inst_array(d.pmg, 1, kInImage));
    v.push_back(inst_array(d.skip_m, 2, kInImage));
    v.push_back(inst_array(d.skip_o, O, kInImage));
    // S/PDIF transmitter and the wire configuration record
    v.push_back(inst_array(c->tx.bp, 1, kInImage));
    v.push_back(inst_array(c->tx.cs40, 1, kInImage));
    v.push_back(inst_array(c->rec.packets, 1, kInImage));
    v.push_back(inst_array(c->rec.host, 1, kInImage));
    v.push_back(inst_array(c->rec.mark, 1, kInImage));
}

// Instance images: a header, then the wide arrays (elements of 16 bytes or more: delay rings, the configuration packet,
// the 12 biquads of each EQ channel), then the scalar arrays by falling element size, so that every array is naturally
// aligned; each array holds its rows back to back.  The size is a multiple of 16.
struct ImageHeader { uint32_t magic, version, arith, n_bands; uint64_t bytes; uint32_t reserved[2]; };
static_assert(sizeof(ImageHeader) == image::kHeaderWords * 4, "image header");
constexpr uint32_t kImageMagic = 0x49505344u;             // "DSPI"
constexpr uint32_t kImageVersion = 1;

// The launch plan over the arrays of `use` (kInImage: with the biquads of the sub-engines' mirrors; kReset); returns the
// image size.
template <class A>
size_t image_plan(ChainHost<A> *c, uint32_t use, image::Plan &pl)
{
    using B = typename A::Biquad;
    std::vector<InstArray> t;
    instance_arrays(c, t);
    if (use == kInImage) {       // channel = role * N_pad + instance in both mirrors, [12] biquads each
        t.push_back(inst_array((B *)eq_aos_mirror(c->eq_m), 2, kInImage, DSPI_MAX_BANDS * (uint32_t)sizeof(B)));
        t.push_back(inst_array((B *)eq_aos_mirror(c->eq_o), A::kOuts, kInImage, DSPI_MAX_BANDS * (uint32_t)sizeof(B)));
    }
    memset(&pl, 0, sizeof(pl));
    pl.N_pad = c->d.N_pad;
    size_t off = sizeof(ImageHeader);
    for (uint32_t e : { 0u, 8u, 4u, 2u, 1u }) {               // 0: the wide arrays
        for (const InstArray &a : t) {
            if (!(a.use & use) || (e == 0 ? a.elem < 16 : a.elem != e)) continue;
            if (pl.n_fields == image::kMaxFields) return 0;
            const uint32_t fi = pl.n_fields++;
            pl.f[fi] = image::Field{ (char *)a.p, a.rows, a.elem, (uint32_t)off, a.one_rows, a.one };
            const uint32_t step = e == 0 ? 1 : image::kSlabRows, segs = e == 0 ? (a.elem + image::kSegBytes - 1) / image::kSegBytes : 1;
            for (uint32_t r = 0; r < a.rows; r += step)
                for (uint32_t s = 0; s < segs; s++) {
                    if (pl.n_tasks == image::kMaxTasks) return 0;
                    pl.t[pl.n_tasks++] = image::Task{ (uint8_t)fi, (uint8_t)(e == 0 ? s : (a.rows - r < step ? a.rows - r : step)), (uint16_t)r };
                }
            off += (size_t)a.rows * a.elem;
        }
    }
    pl.used = (uint32_t)off;
    pl.bytes = (uint32_t)((off + 15) & ~(size_t)15);
    const ImageHeader h = { kImageMagic, kImageVersion, c->desc.arith, c->desc.n_bands, pl.bytes, { 0, 0 } };
    memcpy(pl.header, &h, sizeof(h));
    return pl.bytes;
}

// the pipeline reset of instances [inst0, inst0 + n) on s
template <class A>
cudaError_t reset_range(ChainHost<A> *c, uint32_t inst0, uint32_t n, cudaStream_t s)
{
    image::Plan pl;
    if (!image_plan(c, kReset, pl)) return cudaErrorInvalidValue;
    image::instance_image_kernel<image::kReset><<<dim3((n + 31) / 32, pl.n_tasks), 256, 0, s>>>(pl, inst0, n, nullptr);
    c->launches++;
    return cudaGetLastError();
}

// every instance, padding included: what a new engine starts from and reset_state returns to
template <class A>
cudaError_t init_states(ChainHost<A> *c)
{
    cudaError_t e = reset_range(c, 0, c->d.N_pad, c->q.stream);
    return e == cudaSuccess ? cudaStreamSynchronize(c->q.stream) : e;
}

// a new engine's transmitters: block position 0, the channel status init_spdif_buffer() stamps (audio_spdif.c:82-88)
template <class A>
cudaError_t init_spdif_tx(ChainHost<A> *c)
{
    const std::vector<uint64_t> cs(c->d.N_pad, kSpdifDefaultCs40);
    cudaError_t e = cudaMemsetAsync(c->tx.bp, 0, (size_t)c->d.N_pad * 4, c->q.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(c->tx.cs40, cs.data(), (size_t)c->d.N_pad * 8, cudaMemcpyHostToDevice, c->q.stream);
    return e == cudaSuccess ? cudaStreamSynchronize(c->q.stream) : e;
}

// ---- lifetime ----------------------------------------------------------------------------------------------------------
template <class H>
int destroy(H *c)
{
    if (!c) return DSPI_OK;
    cudaSetDevice(c->desc.device);
    if (c->q.stream) cudaStreamSynchronize(c->q.stream);
    for (Queue &l : c->lanes) l.destroy();
    c->open_lanes = 0;
    c->q.destroy();
    c->part.destroy();
    if (c->eq_m) dspi_eq_destroy(c->eq_m);
    if (c->eq_o) dspi_eq_destroy(c->eq_o);
    for (void *p : c->allocs) cudaFree(p);
    if (c->d_pcm) cudaFree(c->d_pcm);
    if (c->d_spdif) cudaFree(c->d_spdif);
    if (c->d_pdmout) cudaFree(c->d_pdmout);
    if (c->d.vmm) cudaFree(c->d.vmm);
    delete c;
    cudaGetLastError();
    return DSPI_OK;
}

// H: the handle type (dspi_chain / dspi_chainq), a ChainHost<H::Arith>
template <class H>
int create(H **out, const dspi_chain_desc *desc)
{
    using A = typename H::Arith;
    if (!out || !desc) return fail(DSPI_EINVAL, "null argument");
    *out = nullptr;
    int rc = A::check_desc(*desc);
    if (rc) return rc;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(DSPI_ENODEV, "no CUDA device (there is no CPU fallback)"); }
    if (desc->device < 0 || desc->device >= ndev) return fail(DSPI_ENODEV, "device %d out of range", desc->device);
    int major = 0;
    CU_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, desc->device));
    if (major != 9) return fail(DSPI_ENODEV, "device %d is not sm_90", desc->device);
    CU_OK(cudaSetDevice(desc->device));
    H *c = new (std::nothrow) H();                                          // value-initialised: every pointer and count 0
    if (!c) return fail(DSPI_ENOMEM, "host allocation failed");
    c->desc = *desc;
    c->env_mode.assign(desc->n_instances, 0);
    auto &d = c->d;
    d.N = desc->n_instances;
    d.N_pad = (d.N + 31) / 32 * 32;
    d.nb = desc->n_bands;
    d.max_frames = desc->max_frames;
    d.ldF = (d.max_frames + 3u) & ~3u;
    const size_t Np = d.N_pad;
    {
        dspi_eq_desc ed;
        memset(&ed, 0, sizeof(ed));
        ed.arith = desc->arith; ed.n_bands = desc->n_bands; ed.device = desc->device;
        ed.n_channels = 2 * d.N_pad;
        rc = dspi_eq_create(&c->eq_m, &ed);
        ed.n_channels = A::kOuts * d.N_pad;
        if (rc == DSPI_OK) rc = dspi_eq_create(&c->eq_o, &ed);
        if (rc != DSPI_OK) { destroy(c); return rc; }
    }
    c->q.n = desc->n_instances;
    cudaError_t e = c->part.create(desc->device, desc->n_instances);
    if (e == cudaSuccess) e = c->q.create(c->part, d.max_frames);
    if (e != cudaSuccess && c->part.g_pdm) {                                // no streams in the partition: run without one
        cudaGetLastError();
        c->q.destroy();
        c->part.destroy();
        e = c->q.create(c->part, d.max_frames);
    }
#define TRY(x) if (e == cudaSuccess) e = (x)
    d.off = c->q.sched.d_off;
    TRY(dev_alloc(c, &c->d_aos, Np * A::kRoles * DSPI_MAX_BANDS));
    TRY(dev_alloc(c, &d.preamp, 2 * Np));
    TRY(dev_alloc(c, &d.flags, Np));
    TRY(dev_alloc(c, &d.loud_c, A::kLoudRows * Np));
    TRY(dev_alloc(c, &d.loud_st, 8 * Np));
    TRY(dev_alloc(c, &d.loud_byp, Np));
    TRY(dev_alloc(c, &d.xf, 7 * Np));
    TRY(dev_alloc(c, &d.lev_c, 9 * Np));
    TRY(A::alloc_leveller(c));
    TRY(dev_alloc(c, &d.lev_idx, Np));
    TRY(dev_alloc(c, &d.lev_la, (size_t)2 * DSPI_LA_SAMPLES * Np));
    TRY(dev_alloc(c, &d.o_gl, A::kOuts * Np));
    TRY(dev_alloc(c, &d.o_gr, A::kOuts * Np));
    TRY(dev_alloc(c, &d.o_gain, A::kOuts * Np));
    TRY(dev_alloc(c, &d.o_flags, A::kOuts * Np));
    TRY(dev_alloc(c, &d.o_dly, A::kOuts * Np));
    TRY(dev_alloc(c, &d.dline, (size_t)A::kOuts * A::kMaxDelay * Np));
    TRY(dev_alloc(c, &d.widx_in, Np));
    TRY(dev_alloc(c, &d.widx_out, Np));
    TRY(dev_alloc(c, &d.pdm, 9 * Np));
    TRY(dev_alloc(c, &d.peaks, A::kRoles * Np));
    TRY(dev_alloc(c, &d.clip, Np));
    TRY(dev_alloc(c, &d.mrow, (size_t)2 * Np * d.ldF));
    TRY(dev_alloc(c, &d.orow, (size_t)A::kOuts * Np * d.ldF));
    TRY(dev_alloc(c, &d.subq, (size_t)Np * d.ldF));
    TRY(dev_alloc(c, &d.skip_m, 2 * Np));
    TRY(dev_alloc(c, &d.skip_o, A::kOuts * Np));
    TRY(dev_alloc(c, &c->d_status, Np));
    TRY(dev_alloc(c, &d.env, 5 * Np));
    TRY(dev_alloc(c, &d.vol_base, Np));
    TRY(dev_alloc(c, &d.vol_master, Np));
    TRY(dev_alloc(c, &d.o_glin, A::kOuts * Np));
    TRY(dev_alloc(c, &d.pmg, Np));
    TRY(dev_alloc(c, &c->tx.bp, Np));
    TRY(dev_alloc(c, &c->tx.cs40, Np));
    TRY(dev_alloc(c, &c->rec.packets, Np));
    TRY(dev_alloc(c, &c->rec.host, Np));
    TRY(dev_alloc(c, &c->rec.mark, Np));
    TRY(cudaMemsetAsync(c->rec.mark, DSPI_BULK_UNSET, Np, c->q.stream));
    TRY(init_states(c));
    TRY(init_spdif_tx(c));
#undef TRY
    if (e != cudaSuccess) {
        rc = e == cudaErrorMemoryAllocation ? DSPI_ENOMEM : DSPI_ECUDA;
        fail(rc, "chain setup: %s", cudaGetErrorString(e));
        destroy(c);
        return rc;
    }
    *out = c;
    return DSPI_OK;
}

template <class A>
int reset_state(ChainHost<A> *c)
{
    if (!c) return fail(DSPI_EINVAL, "null argument");
    CU_OK(cudaSetDevice(c->desc.device));
    CU_OK(init_states(c));
    return DSPI_OK;
}

// ---- parameters --------------------------------------------------------------------------------------------------------
// host rows of set_params, [rows][n] each, typed like the device arrays they go to
template <class A>
struct ParamRows {
    template <typename P> using Rows = std::vector<std::remove_pointer_t<P>>;
    using D = typename A::Dev;
    Rows<decltype(D::preamp)> preamp;
    Rows<decltype(D::loud_c)> loud_c;
    Rows<decltype(D::xf)> xf;
    Rows<decltype(D::o_gl)> gl, gr;
    Rows<decltype(D::o_gain)> gain;
    Rows<decltype(D::vol_base)> vbase;
    Rows<decltype(D::vol_master)> vmaster;
    Rows<decltype(D::pmg)> pmg;
    Rows<decltype(D::lev_c)> lev_c;
    Rows<decltype(D::o_glin)> glin;
    Rows<decltype(D::o_dly)> dly;
    std::vector<uint8_t> flags, loud_byp, oflags, skip_m, skip_o;
    explicit ParamRows(uint32_t n)
        : preamp(2 * n), loud_c(A::kLoudRows * n), xf(7 * n), gl(A::kOuts * n), gr(A::kOuts * n), gain(A::kOuts * n), vbase(n), vmaster(n),
          pmg(n), lev_c(9 * n), glin(A::kOuts * n), dly(A::kOuts * n), flags(n), loud_byp(n), oflags(A::kOuts * n), skip_m(2 * n),
          skip_o(A::kOuts * n)
    {
    }
};

template <class A>
int set_params(ChainHost<A> *c, uint32_t inst0, uint32_t n, const typename A::Params *params)
{
    if (!c || !params) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(c->q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    const auto &d = c->d;
    const size_t Np = d.N_pad;
    constexpr int O = A::kOuts;
    ParamRows<A> r(n);
    decltype(r.xf) xf_cur(7 * n);
    CU_OK(cudaMemcpy2DAsync(xf_cur.data(), (size_t)n * 4, d.xf + inst0, Np * 4, (size_t)n * 4, 7, cudaMemcpyDeviceToHost, c->q.stream));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    for (uint32_t i = 0; i < n; i++) {
        const typename A::Params &p = params[i];
        A::pack(p, i, n, r);
        bool any_delay = false;
        for (int o = 0; o < O; o++) {
            const dspi_output_channel &oc = p.matrix.outputs[o];
            r.glin[o * n + i] = oc.gain_linear;
            const bool has_pair = o < O - 1;                                 // usb_audio.c:930-933
            r.oflags[o * n + i] = output_flags(oc.enabled, oc.mute, has_pair, has_pair && p.matrix.outputs[o ^ 1].enabled);
            r.skip_o[o * n + i] = A::Stores::output_eq_frozen(oc.enabled, oc.mute, p.bypass_master_eq) ? 1 : 0;   // :878-884: state frozen
            int32_t ds = oc.delay_samples;
            if (ds > A::kMaxDelay) ds = A::kMaxDelay;
            if (ds < 0) ds = 0;
            r.dly[o * n + i] = ds;
            if (ds > 0) any_delay = true;                                    // dsp_pipeline.c:237
        }
        r.flags[i] = chain_flags(p.bypass_master_eq, p.loudness_enabled, p.crossfeed_enabled, p.leveller_enabled, p.leveller_lookahead, any_delay,
                                 p.matrix.outputs[O - 1].enabled);
        r.skip_m[0 * n + i] = r.skip_m[1 * n + i] = p.bypass_master_eq ? 1 : 0;   // usb_audio.c:721-728
        r.loud_byp[i] = (p.loudness[0].bypass ? 1 : 0) | (p.loudness[1].bypass ? 2 : 0);
        const typename decltype(r.xf)::value_type xv[7] = { p.crossfeed.lp_a0, p.crossfeed.lp_b1, p.crossfeed.lp_state_L, p.crossfeed.lp_state_R,
                                                            p.crossfeed.ap_a, p.crossfeed.ap_state_L, p.crossfeed.ap_state_R };
        // crossfeed_compute_coefficients() is the only writer of crossfeed_state in the firmware and it clears the filter
        // state (crossfeed.c:35-127); a volume / mute / matrix update never touches it.  So the record's state rows are
        // taken only when its coefficients differ from the ones in force; otherwise the running state is kept.
        const bool xf_same = xv[0] == xf_cur[0 * n + i] && xv[1] == xf_cur[1 * n + i] && xv[4] == xf_cur[4 * n + i];
        for (int k = 0; k < 7; k++) {
            const bool is_state = k == 2 || k == 3 || k == 5 || k == 6;
            r.xf[k * n + i] = (is_state && xf_same) ? xf_cur[k * n + i] : xv[k];
        }
        const float *lv = &p.leveller.alpha_rms;
        for (int k = 0; k < 9; k++) r.lev_c[k * n + i] = lv[k];
    }
    auto put = [&](auto *dst_base, const auto &src, int rows) -> cudaError_t {
        const size_t elem = sizeof(*dst_base);
        return cudaMemcpy2DAsync((char *)dst_base + (size_t)inst0 * elem, Np * elem, src.data(), (size_t)n * elem, (size_t)n * elem, rows,
                                 cudaMemcpyHostToDevice, c->q.stream);
    };
    CU_OK(put(d.preamp, r.preamp, 2));
    CU_OK(put(d.flags, r.flags, 1));
    CU_OK(put(d.loud_c, r.loud_c, A::kLoudRows));
    CU_OK(put(d.loud_byp, r.loud_byp, 1));
    CU_OK(put(d.xf, r.xf, 7));
    CU_OK(put(d.lev_c, r.lev_c, 9));
    CU_OK(put(d.o_gl, r.gl, O));
    CU_OK(put(d.o_gr, r.gr, O));
    CU_OK(put(d.o_gain, r.gain, O));
    CU_OK(put(d.o_glin, r.glin, O));
    CU_OK(put(d.vol_base, r.vbase, 1));
    CU_OK(put(d.vol_master, r.vmaster, 1));
    CU_OK(put(d.pmg, r.pmg, 1));
    CU_OK(put(d.o_flags, r.oflags, O));
    CU_OK(put(d.o_dly, r.dly, O));
    CU_OK(put(d.skip_m, r.skip_m, 2));
    CU_OK(bulk::mark_stale(c->rec, inst0, n, c->q.stream));
    CU_OK(put(d.skip_o, r.skip_o, O));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    rc = eq_set_skip(c->eq_m, d.skip_m, c->q.stream);
    if (rc == DSPI_OK) rc = eq_set_skip(c->eq_o, d.skip_o, c->q.stream);
    return rc;
}

// The envelope rows [5][n] of instances [inst0, inst0+n) that states (or NULL: leave envelope mode) give; env_instances and
// the mode mirror follow.  Every writer of env row 4 is a call issued from the host (create, _set_preset_mute,
// _copy_instances, _import_instances, _state_import and their lane forms), so the mirror is exact at issue time.
template <class A>
void preset_rows(ChainHost<A> *c, uint32_t inst0, uint32_t n, const dspi_preset_mute *states, uint32_t sample_rate_hz, uint32_t *rows)
{
    memset(rows, 0, (size_t)5 * n * 4);
    for (uint32_t i = 0; i < n; i++) {
        uint8_t &on = c->env_mode[inst0 + i];
        if (on) c->env_instances--;
        on = states ? 1 : 0;
        if (states) {
            rows[0 * n + i] = states[i].loading ? 1u : 0u;
            rows[1 * n + i] = states[i].counter;
            memcpy(&rows[2 * n + i], &states[i].smooth_gain, 4);
            rows[3 * n + i] = sample_rate_hz;
            rows[4 * n + i] = 1u;
            c->env_instances++;
        }
    }
}

// preset-mute envelope of instances [inst0, inst0+n): states == NULL leaves envelope mode (the constant preset_mute_gain of
// set_params applies again); on queue q (the engine's or a lane's)
template <class A>
int set_preset_mute(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const dspi_preset_mute *states, uint32_t sample_rate_hz)
{
    if (!q) return DSPI_EINVAL;
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    unsigned char *buf = nullptr;
    CU_OK(q->ring.take((size_t)5 * n * 4, &buf));
    preset_rows(c, inst0, n, states, sample_rate_hz, (uint32_t *)buf);
    CU_OK(begin_call(c, *q));
    CU_OK(cudaMemcpy2DAsync(c->d.env + inst0, (size_t)c->d.N_pad * 4, buf, (size_t)n * 4, (size_t)n * 4, 5, cudaMemcpyHostToDevice, q->stream));
    CU_OK(q->ring.done(q->stream));
    return end_call(*q, DSPI_OK);
}

// dspi_preset_mute records of env rows 0-2 of n instances (row r of instance i at env[r * Np + i]), as get_preset_mute
// packs them on the host: loading in the low byte of the first word, the reserved bytes zero
__global__ void __launch_bounds__(128) preset_mute_records_kernel(const uint32_t *__restrict__ env, size_t Np, uint32_t n,
                                                                  dspi_preset_mute *__restrict__ out)
{
    static_assert(sizeof(dspi_preset_mute) == 12, "dspi_preset_mute");
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t *w = reinterpret_cast<uint32_t *>(out + i);
    w[0] = env[i] & 0xFFu;
    w[1] = env[Np + i];
    w[2] = env[2 * Np + i];
}

// dspi_spdif_tx records of n transmitters, as spdif_tx_pack makes them; bytewise, since the records are 1-byte aligned
__global__ void __launch_bounds__(128) spdif_tx_records_kernel(const uint32_t *__restrict__ bp, const uint64_t *__restrict__ cs40, uint32_t n,
                                                               dspi_spdif_tx *__restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t cs = cs40[i];
    uint8_t *o = reinterpret_cast<uint8_t *>(out + i);
    for (int b = 0; b < 5; b++) o[b] = (uint8_t)(cs >> (8 * b));
    o[5] = (uint8_t)bp[i];
    o[6] = o[7] = 0;
}

// on queue q: the engine's returns the records in host memory; a lane's writes them to device memory on its stream
template <class A>
int get_preset_mute(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, dspi_preset_mute *states)
{
    if (!q) return DSPI_EINVAL;
    if (!states) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    const size_t Np = c->d.N_pad;
    if (q->lane) {
        CU_OK(begin_call(c, *q));
        preset_mute_records_kernel<<<(n + 127) / 128, 128, 0, q->stream>>>(c->d.env + inst0, Np, n, states);
        c->launches++;
        return end_call(*q, cudaGetLastError() == cudaSuccess ? DSPI_OK : fail(DSPI_ECUDA, "preset-mute record kernel"));
    }
    std::vector<uint32_t> rows((size_t)3 * n);
    CU_OK(cudaMemcpy2DAsync(rows.data(), (size_t)n * 4, c->d.env + inst0, Np * 4, (size_t)n * 4, 3, cudaMemcpyDeviceToHost, c->q.stream));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    for (uint32_t i = 0; i < n; i++) {
        memset(&states[i], 0, sizeof(states[i]));
        states[i].loading = (uint8_t)rows[0 * n + i];
        states[i].counter = rows[1 * n + i];
        memcpy(&states[i].smooth_gain, &rows[2 * n + i], 4);
    }
    return DSPI_OK;
}

// crossfeed / leveller / loudness coefficients and the host volume of instances [inst0, inst0+n) generated ON THE GPU
template <class A>
int set_dynamics_device(ChainHost<A> *c, uint32_t inst0, uint32_t n, const dspi_dynamics_config *cfgs, float sample_rate)
{
    if (!c || !cfgs) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(c->q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    dspi_dynamics_config *d_cfg = nullptr;
    CU_OK(cudaMalloc((void **)&d_cfg, (size_t)n * sizeof(*cfgs)));
    cudaError_t e = cudaMemcpyAsync(d_cfg, cfgs, (size_t)n * sizeof(*cfgs), cudaMemcpyHostToDevice, c->q.stream);
    if (e == cudaSuccess) {
        A::dynamics<<<(n + 127) / 128, 128, 0, c->q.stream>>>(c->d, c->rec, inst0, n, d_cfg, sample_rate);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->q.stream);
    cudaFree(d_cfg);
    if (e != cudaSuccess) return fail(DSPI_ECUDA, "dynamics coefficient generation: %s", cudaGetErrorString(e));
    c->launches++;
    return DSPI_OK;
}

// Before a lane call that configures instances: a lane's first call that needs a staging it lacks (`staged` false)
// allocates it, and an engine whose skip rows were never set (no set_params, apply, import, copy or edit yet) remasks every
// row once; both first wait for every lane and the engine stream.  Nothing for the engine's queue.
template <class A>
int lane_prepare(ChainHost<A> *c, const Queue &q, bool staged)
{
    if (!q.lane) return DSPI_OK;
    const bool skip_set = eq_skip_set(c->eq_m) && eq_skip_set(c->eq_o);
    if (staged && skip_set) return DSPI_OK;
    CU_OK(drain(c));
    return skip_set ? DSPI_OK : bulk::finish_skip(c, c->q);
}

// Before a lane read that needs a staging or frequency table it lacks (`staged` false): wait for every lane and the
// engine stream, as lane_prepare does before an allocation.  Nothing for the engine's queue.
template <class A>
int lane_grow(ChainHost<A> *c, const Queue &q, bool staged)
{
    if (!q.lane || staged) return DSPI_OK;
    CU_OK(drain(c));
    return DSPI_OK;
}

// results: host memory for the engine's queue, device memory for a lane's
template <class A>
int apply_bulk_device(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const dspi_wire_bulk_params *packets, const dspi_bulk_host *host,
                      int exact_db, float sample_rate, int32_t *results)
{
    if (!q) return DSPI_EINVAL;
    if (!packets || !host || !results) return fail(DSPI_EINVAL, "null argument");
    if (!(sample_rate > 0.0f) || sample_rate > 3.4e38f) return fail(DSPI_EINVAL, "sample_rate must be positive and finite");
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_prepare(c, *q, q->bulk.results != nullptr)) != DSPI_OK) return rc;
    CU_OK(begin_call(c, *q));
    return end_call(*q, bulk::apply<typename A::Stores>(c, *q, inst0, n, packets, host, exact_db, sample_rate, results));
}

// results (may be NULL): host memory for the engine's queue, device memory for a lane's
template <class A>
int set_rate_device(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const float *sample_rates, int32_t *results)
{
    if (!q) return DSPI_EINVAL;
    if (!sample_rates) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(*q, inst0, n);                       // before the rates are read: n counts them
    if (rc) return rc;
    for (uint32_t i = 0; i < n; i++)
        if (!(sample_rates[i] > 0.0f) || sample_rates[i] > 3.4e38f) return fail(DSPI_EINVAL, "sample_rates[%u] must be positive and finite", i);
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_prepare(c, *q, q->bulk.results != nullptr)) != DSPI_OK) return rc;
    CU_OK(begin_call(c, *q));
    return end_call(*q, bulk::set_rate<typename A::Stores>(c, *q, inst0, n, sample_rates, results));
}

// the argument checks of *_edit_bulk_device on queue q: every edit well formed and naming an instance of the engine,
// then every instance inside q's window
template <class A>
int check_edits(ChainHost<A> *c, const Queue &q, uint32_t n_edits, const dspi_bulk_edit *edits, float sample_rate)
{
    if (!edits) return fail(DSPI_EINVAL, "null argument");
    if (!(sample_rate > 0.0f) || sample_rate > 3.4e38f) return fail(DSPI_EINVAL, "sample_rate must be positive and finite");
    // control-plane sections: the record keeps them zero and the collect kernel stamps them
    static const uint32_t kPlane[][2] = { { 0, 16 },
                                          { offsetof(dspi_wire_bulk_params, pins), offsetof(dspi_wire_bulk_params, eq) },
                                          { offsetof(dspi_wire_bulk_params, channel_names), offsetof(dspi_wire_bulk_params, leveller) } };
    for (uint32_t k = 0; k < n_edits; k++) {
        const dspi_bulk_edit &e = edits[k];
        const uint32_t lo = e.offset, hi = (uint32_t)e.offset + e.length;
        if (e.length == 0 || e.length > sizeof(e.bytes) || e.reserved)
            return fail(DSPI_EINVAL, "edit %u: length %u (1 .. 24) or reserved %u (0)", k, e.length, e.reserved);
        if (hi > bulk::kEditSpace) return fail(DSPI_EINVAL, "edit %u: bytes [%u, %u) past the %u-byte configuration", k, lo, hi, bulk::kEditSpace);
        for (const auto &p : kPlane)
            if (lo < p[1] && hi > p[0]) return fail(DSPI_EINVAL, "edit %u: bytes [%u, %u) touch a control-plane section", k, lo, hi);
        if (e.instance >= c->desc.n_instances) return fail(DSPI_ERANGE, "edit %u names instance %u, outside engine of %u", k, e.instance, c->desc.n_instances);
    }
    for (uint32_t k = 0; k < n_edits; k++)
        if (edits[k].instance < q.inst0 || edits[k].instance - q.inst0 >= q.n)
            return fail(DSPI_ERANGE, "edit %u names instance %u, outside the lane's window [%u, %u)", k, edits[k].instance, q.inst0, q.inst0 + q.n);
    return DSPI_OK;
}

// results: host memory for the engine's queue, device memory for a lane's (may be NULL)
template <class A>
int edit_bulk_device(ChainHost<A> *c, Queue *q, uint32_t n_edits, const dspi_bulk_edit *edits, int exact_db, float sample_rate, int32_t *results)
{
    if (!q) return DSPI_EINVAL;
    int rc = check_edits(c, *q, n_edits, edits, sample_rate);
    if (rc || n_edits == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_prepare(c, *q, q->bulk_edit.marks != nullptr)) != DSPI_OK) return rc;
    CU_OK(begin_call(c, *q));
    return end_call(*q, bulk::edit<typename A::Stores>(c, *q, n_edits, edits, exact_db, sample_rate, results));
}

// host, results (may be NULL): host memory for the engine's queue, device memory for a lane's, as packets
template <class A>
int collect_bulk_device(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, dspi_wire_bulk_params *packets, dspi_bulk_host *host,
                        int32_t *results)
{
    if (!q) return DSPI_EINVAL;
    if (!packets) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_grow(c, *q, !bulk::collect_staged(*q, packets) || q->bulk.results != nullptr)) != DSPI_OK) return rc;
    CU_OK(begin_call(c, *q));
    return end_call(*q, bulk::collect<typename A::Stores>(c, *q, inst0, n, packets, host, results));
}

// results: host memory for the engine's queue, device memory for a lane's
template <class A>
int apply_preset_device(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const void *images, size_t image_stride,
                        const dspi_preset_load *load, const dspi_bulk_host *host, float sample_rate, int32_t *results)
{
    constexpr size_t kSlot = sizeof(bulk::SlotOf<typename A::Stores>);
    if (!q) return DSPI_EINVAL;
    if (!images || !load || !host || !results) return fail(DSPI_EINVAL, "null argument");
    if (image_stride < kSlot) return fail(DSPI_EINVAL, "image_stride %zu below the slot size %zu", image_stride, kSlot);
    if (!(sample_rate > 0.0f) || sample_rate > 3.4e38f) return fail(DSPI_EINVAL, "sample_rate must be positive and finite");
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_prepare(c, *q, q->bulk.results && q->preset.results)) != DSPI_OK) return rc;
    CU_OK(begin_call(c, *q));
    return end_call(*q, bulk::apply_preset<typename A::Stores>(c, *q, inst0, n, images, image_stride, load, host, sample_rate, results));
}

// images, results (may be NULL): host memory for the engine's queue, device memory for a lane's
template <class A>
int collect_preset_device(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const uint8_t *slot_indices, void *images, size_t image_stride,
                          int32_t *results)
{
    constexpr size_t kSlot = sizeof(bulk::SlotOf<typename A::Stores>);
    if (!q) return DSPI_EINVAL;
    if (!slot_indices || !images) return fail(DSPI_EINVAL, "null argument");
    if (image_stride < kSlot) return fail(DSPI_EINVAL, "image_stride %zu below the slot size %zu", image_stride, kSlot);
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_grow(c, *q, q->preset.results != nullptr)) != DSPI_OK) return rc;
    CU_OK(begin_call(c, *q));
    return end_call(*q, bulk::collect_preset<typename A::Stores>(c, *q, inst0, n, slot_indices, images, image_stride, results));
}

template <class A>
int upload_biquads(ChainHost<A> *c, uint32_t inst0, uint32_t n, const typename A::Biquad *biquads)
{
    if (!c || !biquads) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(c->q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    using B = typename A::Biquad;
    const size_t row = (size_t)A::kRoles * DSPI_MAX_BANDS;
    CU_OK(cudaMemcpyAsync(c->d_aos + inst0 * row, biquads, n * row * sizeof(B), cudaMemcpyHostToDevice, c->q.stream));
    const uint32_t Np = c->d.N_pad, items = n * A::kRoles * DSPI_MAX_BANDS;
    A::scatter<<<(items + 255) / 256, 256, 0, c->q.stream>>>(c->d_aos, inst0, n, Np, (B *)eq_aos_mirror(c->eq_m), (B *)eq_aos_mirror(c->eq_o), 1);
    CU_OK(cudaGetLastError());
    c->launches++;
    for (int role = 0; role < A::kRoles; role++) {
        rc = role < 2 ? eq_pack_range(c->eq_m, role * Np + inst0, n, c->q.stream) : eq_pack_range(c->eq_o, (role - 2) * Np + inst0, n, c->q.stream);
        if (rc) return rc;
    }
    CU_OK(bulk::mark_stale(c->rec, inst0, n, c->q.stream));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    return DSPI_OK;
}

template <class A>
int set_eq_params_device(ChainHost<A> *c, uint32_t inst0, uint32_t n, dspi_eq_param *recipes, float sample_rate)
{
    if (!c || !recipes) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(c->q, inst0, n);
    if (rc || n == 0) return rc;
    // the sub-engines generate and pack on their own streams: everything issued on the engine stream so far (an
    // asynchronous process_device in particular) must have finished reading the coefficient stores first
    CU_OK(cudaSetDevice(c->desc.device));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    const uint32_t Np = c->d.N_pad;
    std::vector<dspi_eq_param> tmp((size_t)n * DSPI_MAX_BANDS);
    for (int role = 0; role < A::kRoles; role++) {                  // filter_recipes[role][band] of every instance -> one engine range per role
        for (uint32_t i = 0; i < n; i++)
            memcpy(&tmp[(size_t)i * DSPI_MAX_BANDS], &recipes[((size_t)i * A::kRoles + role) * DSPI_MAX_BANDS], DSPI_MAX_BANDS * sizeof(dspi_eq_param));
        rc = role < 2 ? dspi_eq_set_params_device(c->eq_m, role * Np + inst0, n, tmp.data(), sample_rate)
                      : dspi_eq_set_params_device(c->eq_o, (role - 2) * Np + inst0, n, tmp.data(), sample_rate);
        if (rc) return rc;
        for (uint32_t i = 0; i < n; i++)                            // the clamps, written back like the reference does
            memcpy(&recipes[((size_t)i * A::kRoles + role) * DSPI_MAX_BANDS], &tmp[(size_t)i * DSPI_MAX_BANDS], DSPI_MAX_BANDS * sizeof(dspi_eq_param));
    }
    return bulk::record_recipes<typename A::Stores>(c, inst0, n, recipes);
}

template <class A>
int download_biquads(ChainHost<A> *c, uint32_t inst0, uint32_t n, typename A::Biquad *biquads)
{
    if (!c || !biquads) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(c->q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    using B = typename A::Biquad;
    const uint32_t Np = c->d.N_pad, items = n * A::kRoles * DSPI_MAX_BANDS;
    for (int role = 0; role < A::kRoles; role++) {
        rc = role < 2 ? eq_unpack_range(c->eq_m, role * Np + inst0, n, c->q.stream) : eq_unpack_range(c->eq_o, (role - 2) * Np + inst0, n, c->q.stream);
        if (rc) return rc;
    }
    A::scatter<<<(items + 255) / 256, 256, 0, c->q.stream>>>(c->d_aos, inst0, n, Np, (B *)eq_aos_mirror(c->eq_m), (B *)eq_aos_mirror(c->eq_o), 0);
    CU_OK(cudaGetLastError());
    c->launches++;
    const size_t row = (size_t)A::kRoles * DSPI_MAX_BANDS;
    CU_OK(cudaMemcpyAsync(biquads, c->d_aos + inst0 * row, n * row * sizeof(B), cudaMemcpyDeviceToHost, c->q.stream));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    return DSPI_OK;
}

// ---- processing --------------------------------------------------------------------------------------------------------
template <class A>
int check_process(ChainHost<A> *c, const void *pcm, uint32_t bit_depth, uint32_t n_packets, uint32_t fpp)
{
    if (!c || !pcm) return fail(DSPI_EINVAL, "null argument");
    if (bit_depth != 16 && bit_depth != 24) return fail(DSPI_EINVAL, "bit_depth must be 16 or 24");
    if (fpp == 0 || fpp > DSPI_PACKET_MAX) return fail(DSPI_EINVAL, "frames_per_packet must be 1..%d", DSPI_PACKET_MAX);
    if (n_packets == 0) return fail(DSPI_EINVAL, "n_packets must be > 0");
    if ((uint64_t)n_packets * fpp > c->desc.max_frames) return fail(DSPI_ERANGE, "%u frames exceed max_frames %u", n_packets * fpp, c->desc.max_frames);
    return DSPI_OK;
}

template <class A>
int check_packets(ChainHost<A> *c, PacketSchedule &ps, const void *pcm, uint32_t bit_depth, uint32_t n_packets, const uint16_t *packet_frames)
{
    if (!pcm) return fail(DSPI_EINVAL, "null argument");
    if (bit_depth != 16 && bit_depth != 24) return fail(DSPI_EINVAL, "bit_depth must be 16 or 24");
    const char *why = "";
    const int rc = ps.check(n_packets, packet_frames, &why);
    if (rc == DSPI_ERANGE) return fail(rc, "%s %u", why, c->desc.max_frames);
    return rc ? fail(rc, "%s", why) : DSPI_OK;
}

// The EQ stage of one slice over the rows of `roles` roles (row = role * N_pad + instance) of instances [inst0, inst0 + n):
// one launch over every row for the whole engine, else one launch per role over that role's rows.
template <class A>
int eq_stage(ChainHost<A> *c, dspi_eq *eq, uint32_t roles, void *rows, uint32_t fb, uint32_t fe, uint32_t inst0, uint32_t n, cudaStream_t s)
{
    const auto &d = c->d;
    using T = std::remove_pointer_t<decltype(d.mrow)>;
    if (inst0 == 0 && n == d.N) return eq_process_on(eq, (T *)rows + fb, fe - fb, d.ldF, s);
    for (uint32_t r = 0; r < roles; r++) {
        const uint32_t ch0 = r * d.N_pad + inst0;
        const int rc = eq_process_range_on(eq, (T *)rows + (size_t)ch0 * d.ldF + fb, fe - fb, d.ldF, ch0, n, s);
        if (rc) return rc;
    }
    return DSPI_OK;
}

// The host buffers of a lane host call (process_lane_host), whose packet slices run_stages copies through the lane's
// staging hs on its copy streams: each slice's PCM in before its front stage, its S/PDIF rows out after its output stage
// and its PDM rows out after its modulator.  spdif / pdm NULL: that output is not copied.
struct HostCopies {
    HostStage *hs;
    const void *pcm;
    void *spdif;
    uint32_t *pdm;
    size_t pcm_frame, spdif_frame;   // bytes of one frame of a PCM row, of an S/PDIF row
    size_t spdif_rows;               // n * pairs
};

// frames [fb, fe) of `rows` rows of F frames of `frame` bytes, between two buffers of that layout
inline cudaError_t copy_frames(void *dst, const void *src, size_t rows, size_t F, size_t frame, uint32_t fb, uint32_t fe, cudaMemcpyKind kind,
                               cudaStream_t s)
{
    const size_t pitch = F * frame, off = (size_t)fb * frame;
    return cudaMemcpy2DAsync((char *)dst + off, pitch, (const char *)src + off, pitch, (size_t)(fe - fb) * frame, rows, kind, s);
}

// One call over instances [inst0, inst0 + n) and the schedule x.sched has checked, with the kernel set K, issued on the
// queue x: its offsets go to the device first, on x.stream, where the call also ends.  The caller's buffers hold rows for
// the n instances.  d_spdif: words, or subframes when `subframes` is set (either may be NULL).  With hc, the device
// buffers are the lane's staging and the slices are copied from and to the host as they go (HostCopies).
template <class A, class K>
int run_stages(ChainHost<A> *c, Queue &x, uint32_t inst0, uint32_t n, const void *d_pcm, uint32_t bit_depth, const uint16_t *packet_frames,
               void *d_spdif, bool subframes, uint32_t *d_pdm, typename A::Status *d_status, const HostCopies *hc = nullptr)
{
    PacketSchedule &ps = x.sched;
    const uint32_t n_packets = ps.n_packets, F = ps.frames;
    CU_OK(ps.upload(packet_frames, x.stream, &c->launches));
    const size_t post_smem = (size_t)4 * 2 * ps.longest * A::kXs * 4;      // 4 warps x (longest packet + look-ahead columns)
    static PerDeviceOnce once;                                              // per kernel set
    int dev = 0;
    if (once.needs(&dev)) {
        CU_OK(cudaFuncSetAttribute(K::post, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)4 * 2 * DSPI_PACKET_MAX * A::kXs * 4)));
        once.mark(dev);
    }
    // Stage pipeline over packet slices on three streams (chain_streams.cuh): front stages of slice
    // i+1 overlap the output stages of slice i and the modulator of slice i-1.
    ChainStreams &st = x.st;
    uint32_t slice_bounds[ChainStreams::kMaxSlices + 1];
    const uint32_t n_slices = (uint32_t)ChainStreams::plan_slices(n_packets, slice_bounds);
    if (c->env_instances && c->vmm_packets < n_packets) {                    // the table every context's calls read
        CU_OK(drain(c));
        if (c->d.vmm) CU_OK(cudaFree(c->d.vmm));
        c->d.vmm = nullptr; c->vmm_packets = 0;
        CU_OK(cudaMalloc((void **)&c->d.vmm, (size_t)n_packets * c->d.N_pad * sizeof(*c->d.vmm)));
        c->vmm_packets = n_packets;
    }
    typename A::Dev d = c->d;
    d.off = ps.d_off;
    if (c->env_instances) {                                                  // preset-mute envelope: this call's per-packet volumes
        K::env<<<(n + 127) / 128, 128, 0, x.stream>>>(d, inst0, n, n_packets);
        CU_OK(cudaGetLastError());
        c->launches++;
    }
    const uint32_t n_sms = c->part.stream_sms();
    static const uint32_t kStreamCtas = [] { const char *e = getenv("DSPI_CHAIN_CTAS"); const int v = e ? atoi(e) : 0; return (uint32_t)(v >= 1 && v <= 8 ? v : 8); }();   // streaming CTAs (256 threads) per SM
    auto stream_grid = [&](uint64_t units) {                                 // grid-stride kernels: no more CTAs than 8-warp units
        const uint64_t ctas = (units + 7) / 8;
        return (uint32_t)(ctas < (uint64_t)n_sms * kStreamCtas ? (ctas ? ctas : 1) : (uint64_t)n_sms * kStreamCtas);
    };
    const uint32_t n_warps16 = ((n + 31) & ~31u) / 16;                       // pre / post: 16 instances per warp
    CU_OK(cudaEventRecord(st.ev_begin, x.stream));
    CU_OK(cudaStreamWaitEvent(st.s_front, st.ev_begin, 0));
    HostStage *hs = hc ? hc->hs : nullptr;
    if (hs) {
        // the copy-in stream starts behind this call's beginning (earlier calls have read the PCM staging); the modulator
        // rows of instances without a sub go back as zeros, so the PDM staging is cleared before the first modulator
        CU_OK(cudaStreamWaitEvent(hs->s_in, st.ev_begin, 0));
        if (hc->pdm) {
            CU_OK(cudaStreamWaitEvent(st.s_pdm, st.ev_begin, 0));
            CU_OK(cudaMemsetAsync(d_pdm, 0, (size_t)n * F * 8 * 4, st.s_pdm));
        }
    }
    for (uint32_t sl = 0; sl < n_slices; sl++) {
        const uint32_t p0 = slice_bounds[sl], p1 = slice_bounds[sl + 1];
        const uint32_t fb = ps.off[p0], fe = ps.off[p1];
        int rc;
        if (hs) {                                                            // this slice's PCM frames, in before its front stage
            CU_OK(copy_frames((void *)d_pcm, hc->pcm, n, F, hc->pcm_frame, fb, fe, cudaMemcpyHostToDevice, hs->s_in));
            CU_OK(cudaEventRecord(hs->ev_in[sl], hs->s_in));
            CU_OK(cudaStreamWaitEvent(st.s_front, hs->ev_in[sl], 0));
        }
        // ---- front: unpack + loudness -> master EQ -> leveller + crossfeed
        K::pre<<<(n_warps16 + 1) / 2, 64, 0, st.s_front>>>(d, inst0, n, (const uint8_t *)d_pcm, bit_depth, fb, fe, F);
        CU_OK(cudaGetLastError());
        if ((rc = eq_stage(c, c->eq_m, 2, d.mrow, fb, fe, inst0, n, st.s_front)) != DSPI_OK) return rc;
        K::post<<<(n_warps16 + 3) / 4, 128, post_smem, st.s_front>>>(d, inst0, n, p0, p1 - p0, ps.longest);
        CU_OK(cudaGetLastError());
        CU_OK(cudaEventRecord(st.ev_front[sl], st.s_front));
        // ---- outputs: matrix -> per-output EQ -> gain / delay / metering / conversion
        CU_OK(cudaStreamWaitEvent(st.s_out, st.ev_front[sl], 0));
        K::mix<<<stream_grid((uint64_t)n * ((fe - fb + 127) / 128)), 256, 0, st.s_out>>>(d, inst0, n, fb, fe);
        CU_OK(cudaGetLastError());
        if ((rc = eq_stage(c, c->eq_o, A::kOuts, d.orow, fb, fe, inst0, n, st.s_out)) != DSPI_OK) return rc;
        const uint32_t out_grid = stream_grid((uint64_t)n * (p1 - p0));
        if (subframes && d_spdif)
            K::template outpost<true><<<out_grid, 256, 0, st.s_out>>>(d, inst0, n, p0, p1 - p0, F, (int32_t *)d_spdif, c->tx);
        else
            K::template outpost<false><<<out_grid, 256, 0, st.s_out>>>(d, inst0, n, p0, p1 - p0, F, (int32_t *)d_spdif, c->tx);
        CU_OK(cudaGetLastError());
        CU_OK(cudaEventRecord(st.ev_out[sl], st.s_out));
        if (hs && hc->spdif) {                                               // this slice's S/PDIF frames, out after its output stage
            CU_OK(cudaStreamWaitEvent(hs->s_back, st.ev_out[sl], 0));
            CU_OK(copy_frames(hc->spdif, d_spdif, hc->spdif_rows, F, hc->spdif_frame, fb, fe, cudaMemcpyDeviceToHost, hs->s_back));
        }
        // ---- modulator
        CU_OK(cudaStreamWaitEvent(st.s_pdm, st.ev_out[sl], 0));
        K::pdm<<<(n + 127) / 128, 128, 0, st.s_pdm>>>(d, inst0, n, fb, fe, F, d_pdm);
        CU_OK(cudaGetLastError());
        c->launches += 5;
        if (hs && hc->pdm) {                                                 // and its PDM frames, out after its modulator
            CU_OK(cudaEventRecord(hs->ev_pdm[sl], st.s_pdm));
            CU_OK(cudaStreamWaitEvent(hs->s_back, hs->ev_pdm[sl], 0));
            CU_OK(copy_frames(hc->pdm, d_pdm, n, F, 8 * 4, fb, fe, cudaMemcpyDeviceToHost, hs->s_back));
        }
    }
    if (hs) {                                                                // the call ends after its last copy out
        CU_OK(cudaEventRecord(hs->ev_back, hs->s_back));
        CU_OK(cudaStreamWaitEvent(x.stream, hs->ev_back, 0));
    }
    K::ring<<<stream_grid((uint64_t)n * A::kOuts), 256, 0, st.s_out>>>(d, inst0, n, F, n_packets, c->tx.bp);   // after the last outpost launch (stream order)
    CU_OK(cudaGetLastError());
    c->launches++;
    // The ring kernel wrote the advanced write index of the call's instances into widx_out (the outpost and ring kernels read
    // widx_in until the end of the call).  A whole-engine call swaps the two buffers; a range call copies its instances'
    // indices back, so that every other instance keeps the index it has in widx_in.
    if (inst0 == 0 && n == d.N) std::swap(c->d.widx_in, c->d.widx_out);
    else CU_OK(cudaMemcpyAsync(d.widx_in + inst0, d.widx_out + inst0, (size_t)n * sizeof(*d.widx_in), cudaMemcpyDeviceToDevice, st.s_out));
    CU_OK(cudaEventRecord(st.ev_aux, st.s_out));                             // ring update done
    CU_OK(cudaStreamWaitEvent(x.stream, st.ev_aux, 0));
    // the last modulator launch is ordered after every other stage launch of this call
    CU_OK(cudaEventRecord(st.ev_done, st.s_pdm));
    CU_OK(cudaStreamWaitEvent(x.stream, st.ev_done, 0));                     // later work on x.stream sees all outputs
    if (d_status) {
        K::status<<<(n + 127) / 128, 128, 0, x.stream>>>(c->d, inst0, n, d_status);
        CU_OK(cudaGetLastError());
        c->launches++;
    }
    return DSPI_OK;
}

// Instances [inst0, inst0 + n) of a call on queue q: inst0 on a 64-instance boundary, so that the pre and post stages'
// 16-instance warps and every vector access of the SoA arrays stay aligned.  Checked after the arguments check_packets covers.
int check_window(const Queue &q, uint32_t inst0, uint32_t n)
{
    if (inst0 % 64u) return fail(DSPI_EINVAL, "first instance %u is not a multiple of 64", inst0);
    return check_range(q, inst0, n);
}

// the window of a whole-engine call (a NULL handle is refused by the checks that follow)
template <class A>
uint32_t all_instances(const ChainHost<A> *c) { return c ? c->desc.n_instances : 0; }

// instances [inst0, inst0 + n) on queue q, every buffer laid out for the n instances (the whole engine: 0, n_instances)
template <class A>
int process_device(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const void *d_pcm, uint32_t bit_depth, uint32_t n_packets,
                   const uint16_t *packet_frames, void *d_spdif, bool subframes, uint32_t *d_pdm, typename A::Status *d_status)
{
    if (!q) return DSPI_EINVAL;
    int rc = check_packets(c, q->sched, d_pcm, bit_depth, n_packets, packet_frames);
    if (rc) return rc;
    if (subframes && ((uintptr_t)d_spdif & 15)) return fail(DSPI_EINVAL, "subframes must be 16-byte aligned");
    if ((rc = check_window(*q, inst0, n)) || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    CU_OK(begin_call(c, *q));
    rc = A::with_stages(c->desc, [&](auto k) {
        return run_stages<A, decltype(k)>(c, *q, inst0, n, d_pcm, bit_depth, packet_frames, d_spdif, subframes, d_pdm, d_status);
    });
    return end_call(*q, rc, false);
}

// host memory in and out, staged through the engine's device buffers
template <class A>
int process_host(ChainHost<A> *c, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth, uint32_t n_packets,
                 const uint16_t *packet_frames, void *spdif_out, bool subframes, uint32_t *pdm_out, typename A::Status *status)
{
    if (!c) return fail(DSPI_EINVAL, "null argument");
    int rc = check_packets(c, c->q.sched, pcm, bit_depth, n_packets, packet_frames);
    if (rc) return rc;
    if ((rc = check_window(c->q, inst0, n)) || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    const size_t N = n, F = c->q.sched.frames, pairs = (A::kOuts - 1) / 2;   // the sub output has no S/PDIF pair
    const size_t in_bytes = N * F * (bit_depth == 24 ? 6 : 4), sp_bytes = N * pairs * F * (subframes ? 16 : 8), pd_bytes = N * F * 8 * 4;
    if (in_bytes > c->pcm_bytes) { if (c->d_pcm) cudaFree(c->d_pcm); c->d_pcm = nullptr; c->pcm_bytes = 0; CU_OK(cudaMalloc(&c->d_pcm, in_bytes)); c->pcm_bytes = in_bytes; }
    if (spdif_out && sp_bytes > c->spdif_bytes) { if (c->d_spdif) cudaFree(c->d_spdif); c->d_spdif = nullptr; c->spdif_bytes = 0; CU_OK(cudaMalloc((void **)&c->d_spdif, sp_bytes)); c->spdif_bytes = sp_bytes; }
    if (pdm_out && pd_bytes > c->pdmout_bytes) { if (c->d_pdmout) cudaFree(c->d_pdmout); c->d_pdmout = nullptr; c->pdmout_bytes = 0; CU_OK(cudaMalloc((void **)&c->d_pdmout, pd_bytes)); c->pdmout_bytes = pd_bytes; }
    // the modulator writes the rows of instances with a sub only; the others go back to the caller as zeros, on every call
    // (an earlier call's bits would be there otherwise: a sub switched off since, or a longer call's [N][F][8] layout)
    if (pdm_out) CU_OK(cudaMemsetAsync(c->d_pdmout, 0, pd_bytes, c->q.stream));
    CU_OK(cudaMemcpyAsync(c->d_pcm, pcm, in_bytes, cudaMemcpyHostToDevice, c->q.stream));
    rc = process_device(c, &c->q, inst0, n, c->d_pcm, bit_depth, n_packets, packet_frames, spdif_out ? c->d_spdif : nullptr, subframes,
                        pdm_out ? c->d_pdmout : nullptr, status ? c->d_status : nullptr);
    if (rc) return rc;
    if (spdif_out) CU_OK(cudaMemcpyAsync(spdif_out, c->d_spdif, sp_bytes, cudaMemcpyDeviceToHost, c->q.stream));
    if (pdm_out) CU_OK(cudaMemcpyAsync(pdm_out, c->d_pdmout, pd_bytes, cudaMemcpyDeviceToHost, c->q.stream));
    if (status) CU_OK(cudaMemcpyAsync(status, c->d_status, N * sizeof(typename A::Status), cudaMemcpyDeviceToHost, c->q.stream));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    return DSPI_OK;
}

// a lane host call's buffer: NULL, or page-locked host memory (a copy from pageable memory would make the call wait)
inline bool page_locked(const void *p)
{
    if (!p) return true;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// process_host's layouts, checks and results on lane q, without waiting: every buffer page-locked, staged through the
// lane's own device buffers, each packet slice copied in and out on the lane's copy streams as the stages reach it
// (run_stages), the status after the call.  pcm is read and the outputs written on the lane's timeline.
template <class A>
int process_lane_host(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const void *pcm, uint32_t bit_depth, uint32_t n_packets,
                      const uint16_t *packet_frames, void *spdif_out, bool subframes, uint32_t *pdm_out, typename A::Status *status)
{
    if (!q) return DSPI_EINVAL;
    int rc = check_packets(c, q->sched, pcm, bit_depth, n_packets, packet_frames);
    if (rc) return rc;
    if ((rc = check_window(*q, inst0, n))) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    const void *bufs[4] = { pcm, spdif_out, pdm_out, status };
    static const char *const names[4] = { "pcm", "the S/PDIF output", "pdm_out", "status" };
    for (int k = 0; k < 4; k++)
        if (!page_locked(bufs[k])) return fail(DSPI_EINVAL, "%s is not page-locked host memory", names[k]);
    if (n == 0) return DSPI_OK;
    constexpr size_t pairs = (A::kOuts - 1) / 2;                            // the sub output has no S/PDIF pair
    const size_t sf = spdif_out ? (subframes ? 16 : 8) : 0;
    HostStage &hs = q->host;
    if ((rc = lane_grow(c, *q, hs.has(sf, pdm_out != nullptr))) != DSPI_OK) return rc;
    CU_OK(hs.ensure(q->n, c->desc.max_frames, pairs, sizeof(typename A::Status), sf, pdm_out != nullptr));
    CU_OK(begin_call(c, *q));
    const HostCopies hc = { &hs, pcm, spdif_out, pdm_out, (size_t)(bit_depth == 24 ? 6 : 4), sf, (size_t)n * pairs };
    typename A::Status *d_status = status ? (typename A::Status *)hs.d_status : nullptr;
    rc = A::with_stages(c->desc, [&](auto k) {
        return run_stages<A, decltype(k)>(c, *q, inst0, n, hs.d_pcm, bit_depth, packet_frames, spdif_out ? hs.d_spdif : nullptr, subframes,
                                          pdm_out ? hs.d_pdm : nullptr, d_status, &hc);
    });
    if (rc == DSPI_OK && status && cudaMemcpyAsync(status, d_status, (size_t)n * sizeof(*d_status), cudaMemcpyDeviceToHost, q->stream) != cudaSuccess)
        rc = fail(DSPI_ECUDA, "status copy: %s", cudaGetErrorString(cudaGetLastError()));
    return end_call(*q, rc, false);
}

// the uniform schedule: n_packets packets of fpp frames, from device (host == false) or host memory
template <class A>
int process_uniform(ChainHost<A> *c, const void *pcm, uint32_t bit_depth, uint32_t n_packets, uint32_t fpp, int32_t *spdif, uint32_t *pdm,
                    typename A::Status *status, bool host)
{
    int rc = check_process(c, pcm, bit_depth, n_packets, fpp);
    if (rc) return rc;
    const std::vector<uint16_t> table(n_packets, (uint16_t)fpp);
    const uint32_t n = c->desc.n_instances;
    return host ? process_host(c, 0, n, pcm, bit_depth, n_packets, table.data(), spdif, false, pdm, status)
                : process_device(c, &c->q, 0, n, pcm, bit_depth, n_packets, table.data(), spdif, false, pdm, status);
}

// ---- lanes: issue queues of one engine over disjoint instance windows, whose calls run concurrently -------------------
// A lane takes process calls and the control calls a running clock group needs (edits, fades, transmitter restamps,
// resets, applies, preset applies and rate switches): set_preset_mute, set_spdif_tx, reset_instances, edit_bulk_device,
// apply_bulk_device, apply_preset_device, set_rate_device, process_device and process_lane_host on its queue; the reads it needs
// (collect_bulk_device, collect_preset_device, export_instances, response, get_preset_mute, get_spdif_tx), into device
// memory; and the moves of devices into its window (import_instances, and copy_instances on the destination's queue,
// ordered against the source lane too).
template <class A>
int lane_open(ChainHost<A> *c, uint32_t inst0, uint32_t n, uint32_t *lane)
{
    if (!c || !lane) return fail(DSPI_EINVAL, "null argument");
    if (inst0 % 64u) return fail(DSPI_EINVAL, "first instance %u is not a multiple of 64", inst0);
    if (n == 0) return fail(DSPI_EINVAL, "a lane's window holds at least one instance");
    int rc = check_range(c->q, inst0, n);
    if (rc) return rc;
    for (const Queue &l : c->lanes)
        if (l.stream && inst0 < l.inst0 + l.n && l.inst0 < inst0 + n)
            return fail(DSPI_EINVAL, "window [%u, %u) overlaps the open lane window [%u, %u)", inst0, inst0 + n, l.inst0, l.inst0 + l.n);
    uint32_t id = 0;
    while (id < DSPI_CHAIN_MAX_LANES && c->lanes[id].stream) id++;
    if (id == DSPI_CHAIN_MAX_LANES) return fail(DSPI_ERANGE, "%d lanes are open already", DSPI_CHAIN_MAX_LANES);
    CU_OK(cudaSetDevice(c->desc.device));
    Queue &l = c->lanes[id];
    l.lane = true;
    l.inst0 = inst0;
    l.n = n;
    const cudaError_t e = l.create(c->part, c->desc.max_frames);
    if (e != cudaSuccess) {
        l.destroy();
        cudaGetLastError();
        return fail(e == cudaErrorMemoryAllocation ? DSPI_ENOMEM : DSPI_ECUDA, "lane setup: %s", cudaGetErrorString(e));
    }
    c->open_lanes++;
    *lane = id;
    return DSPI_OK;
}

template <class A>
int lane_close(ChainHost<A> *c, uint32_t lane)
{
    Queue *l = lane_queue(c, lane);
    if (!l) return DSPI_EINVAL;
    CU_OK(cudaSetDevice(c->desc.device));
    l->destroy();                                                           // waits for the lane's calls
    c->open_lanes--;
    return DSPI_OK;
}

template <class A>
void *lane_stream(ChainHost<A> *c, uint32_t lane)
{
    return c && lane < DSPI_CHAIN_MAX_LANES ? (void *)c->lanes[lane].stream : nullptr;
}

template <class A>
int lane_sync(ChainHost<A> *c, uint32_t lane)
{
    Queue *l = lane_queue(c, lane);
    if (!l) return DSPI_EINVAL;
    CU_OK(cudaSetDevice(c->desc.device));
    CU_OK(cudaStreamSynchronize(l->stream));
    return DSPI_OK;
}

// ---- S/PDIF transmitters -----------------------------------------------------------------------------------------------
// on queue q (the engine's or a lane's)
template <class A>
int set_spdif_tx(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const dspi_spdif_tx *tx)
{
    if (!q) return DSPI_EINVAL;
    if (!tx) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    unsigned char *buf = nullptr;
    CU_OK(q->ring.take((size_t)n * 12, &buf));
    uint64_t *cs = (uint64_t *)buf;                                          // channel status words, then block positions
    uint32_t *bp = (uint32_t *)(buf + (size_t)n * 8);
    if (!spdif_tx_unpack(tx, n, bp, cs)) return fail(DSPI_EINVAL, "block_pos must be 0..191");
    CU_OK(begin_call(c, *q));
    CU_OK(cudaMemcpyAsync(c->tx.bp + inst0, bp, (size_t)n * 4, cudaMemcpyHostToDevice, q->stream));   // behind earlier calls
    CU_OK(cudaMemcpyAsync(c->tx.cs40 + inst0, cs, (size_t)n * 8, cudaMemcpyHostToDevice, q->stream));
    CU_OK(q->ring.done(q->stream));
    return end_call(*q, DSPI_OK);
}

// on queue q: the engine's returns the records in host memory; a lane's writes them to device memory on its stream
template <class A>
int get_spdif_tx(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, dspi_spdif_tx *tx)
{
    if (!q) return DSPI_EINVAL;
    if (!tx) return fail(DSPI_EINVAL, "null argument");
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    if (q->lane) {
        CU_OK(cudaSetDevice(c->desc.device));
        CU_OK(begin_call(c, *q));
        spdif_tx_records_kernel<<<(n + 127) / 128, 128, 0, q->stream>>>(c->tx.bp + inst0, c->tx.cs40 + inst0, n, tx);
        c->launches++;
        return end_call(*q, cudaGetLastError() == cudaSuccess ? DSPI_OK : fail(DSPI_ECUDA, "transmitter record kernel"));
    }
    std::vector<uint32_t> bp(n);
    std::vector<uint64_t> cs(n);
    CU_OK(cudaSetDevice(c->desc.device));
    CU_OK(cudaMemcpyAsync(bp.data(), c->tx.bp + inst0, (size_t)n * 4, cudaMemcpyDeviceToHost, c->q.stream));
    CU_OK(cudaMemcpyAsync(cs.data(), c->tx.cs40 + inst0, (size_t)n * 8, cudaMemcpyDeviceToHost, c->q.stream));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    spdif_tx_pack(bp.data(), cs.data(), n, tx);
    return DSPI_OK;
}

// ---- checkpoint / resume: everything a later process call depends on besides the parameters ----------------------------
using Sections = std::vector<std::pair<void *, size_t>>;

template <class A>
void state_sections(ChainHost<A> *c, Sections &v, bool with_eq = true)
{
    std::vector<InstArray> t;
    instance_arrays(c, t);
    for (const InstArray &a : t)
        if (a.use & kInBlob) v.push_back({ a.p, (size_t)a.rows * c->d.N_pad * a.elem });
    if (!with_eq) return;
    eq_state_sections(c->eq_m, v);
    eq_state_sections(c->eq_o, v);
}

// Version 2 records the K1 geometry (channels per lane, DSPI_F32_CPL) that the two EQ engines' packed stores were laid out
// for, so that a blob resumes in an engine created under either geometry.  Version 1 blobs have no such fields and are read
// as one channel per lane.  An engine writes version A::kStateVersion and reads versions 1 .. A::kStateVersion.
struct StateHeader { uint32_t magic, version, arith, n_instances, n_bands, n_sections; uint64_t bytes; uint32_t cpl_m, cpl_o; };
constexpr uint32_t kStateMagic = 0x53505344u;             // "DSPS"
constexpr size_t kHeaderV1 = offsetof(StateHeader, cpl_m);
inline size_t header_bytes(uint32_t version) { return version == 1u ? kHeaderV1 : sizeof(StateHeader); }

// blob size for this engine's shape with header `hdr` bytes and EQ stores laid out for cpl_m / cpl_o channels per lane
template <class A>
size_t state_bytes(ChainHost<A> *c, size_t hdr, int cpl_m, int cpl_o)
{
    Sections v;
    state_sections(c, v, false);
    size_t n = hdr + eq_state_bytes(c->eq_m, cpl_m) + eq_state_bytes(c->eq_o, cpl_o);
    for (auto &s : v) n += s.second;
    return n;
}

template <class A>
size_t state_size(ChainHost<A> *c)
{
    if (!c) return 0;
    return state_bytes(c, header_bytes(A::kStateVersion), eq_geometry(c->eq_m), eq_geometry(c->eq_o));
}

template <class A>
int state_export(ChainHost<A> *c, void *blob, size_t cap)
{
    if (!c || !blob) return fail(DSPI_EINVAL, "null argument");
    const size_t need = state_size(c);
    if (cap < need) return fail(DSPI_ERANGE, "state blob needs %zu bytes, %zu given", need, cap);
    CU_OK(cudaSetDevice(c->desc.device));
    Sections v;
    state_sections(c, v);
    const StateHeader h = { kStateMagic, A::kStateVersion, c->desc.arith, c->desc.n_instances, c->desc.n_bands, (uint32_t)v.size(), (uint64_t)need,
                            (uint32_t)eq_geometry(c->eq_m), (uint32_t)eq_geometry(c->eq_o) };
    const size_t hdr = header_bytes(A::kStateVersion);
    memcpy(blob, &h, hdr);
    char *p = (char *)blob + hdr;
    for (auto &s : v) {
        CU_OK(cudaMemcpyAsync(p, s.first, s.second, cudaMemcpyDeviceToHost, c->q.stream));
        p += s.second;
    }
    CU_OK(cudaStreamSynchronize(c->q.stream));
    return DSPI_OK;
}

template <class A>
int state_import(ChainHost<A> *c, const void *blob, size_t len)
{
    if (!c || !blob) return fail(DSPI_EINVAL, "null argument");
    Sections v, all;
    state_sections(c, v, false);
    state_sections(c, all);
    StateHeader h;
    if (len < kHeaderV1) return fail(DSPI_EINVAL, "state blob too short");
    memcpy(&h, blob, kHeaderV1);
    h.cpl_m = h.cpl_o = 1;
    if (h.magic != kStateMagic || h.version < 1u || h.version > A::kStateVersion)
        return fail(DSPI_EINVAL, "not a dspi_b200 state blob (magic %08x version %u)", h.magic, h.version);
    const size_t hdr = header_bytes(h.version);
    if (len < hdr) return fail(DSPI_EINVAL, "state blob too short");
    memcpy(&h, blob, hdr);
    if ((h.cpl_m != 1 && h.cpl_m != 2) || (h.cpl_o != 1 && h.cpl_o != 2))
        return fail(DSPI_EINVAL, "state blob names an unknown K1 geometry (%u, %u channels per lane)", h.cpl_m, h.cpl_o);
    if (h.arith != c->desc.arith || h.n_instances != c->desc.n_instances || h.n_bands != c->desc.n_bands || h.n_sections != all.size() ||
        h.bytes != state_bytes(c, hdr, (int)h.cpl_m, (int)h.cpl_o) || len < h.bytes)
        return fail(DSPI_EINVAL, "state blob belongs to a different engine shape (%u instances, arith %u, %llu bytes)", h.n_instances, h.arith,
                    (unsigned long long)h.bytes);
    CU_OK(cudaSetDevice(c->desc.device));
    const char *p = (const char *)blob + hdr;
    for (auto &s : v) {
        CU_OK(cudaMemcpyAsync(s.first, p, s.second, cudaMemcpyHostToDevice, c->q.stream));
        p += s.second;
    }
    CU_OK(cudaStreamSynchronize(c->q.stream));
    int rc = eq_state_load(c->eq_m, p, (int)h.cpl_m, c->q.stream);
    p += eq_state_bytes(c->eq_m, (int)h.cpl_m);
    if (rc == DSPI_OK) rc = eq_state_load(c->eq_o, p, (int)h.cpl_o, c->q.stream);
    if (rc) return rc;
    rc = eq_state_imported(c->eq_m, c->q.stream);
    if (rc == DSPI_OK) rc = eq_state_imported(c->eq_o, c->q.stream);
    if (rc) return rc;
    std::vector<uint32_t> on(c->d.N);
    CU_OK(cudaMemcpyAsync(on.data(), c->d.env + (size_t)4 * c->d.N_pad, (size_t)c->d.N * 4, cudaMemcpyDeviceToHost, c->q.stream));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    c->env_instances = 0;
    for (uint32_t i = 0; i < c->d.N; i++) {
        c->env_mode[i] = on[i] ? 1 : 0;
        c->env_instances += on[i] ? 1u : 0u;
    }
    return DSPI_OK;
}

// ---- per-instance lifecycle: instance images and the pipeline reset of a range -------------------------------------------
template <class A>
size_t instance_image_size(ChainHost<A> *c)
{
    if (!c) return 0;
    image::Plan pl;
    return image_plan(c, kInImage, pl);
}

// arguments of the image calls; *plan filled, *size the image size
template <class A>
int check_images(ChainHost<A> *c, const Queue *q, uint32_t inst0, uint32_t n, const void *images, size_t stride, image::Plan *plan, size_t *size)
{
    if (!q) return DSPI_EINVAL;
    if (!images) return fail(DSPI_EINVAL, "null argument");
    *size = image_plan(c, kInImage, *plan);
    if (*size == 0) return fail(DSPI_EINVAL, "instance image plan exceeds its tables");
    if (stride < *size) return fail(DSPI_EINVAL, "image_stride %zu below the image size %zu", stride, *size);
    return check_range(*q, inst0, n);
}

// the EQ sub-engines' ranges of instances [inst0, inst0 + n): every role of the master / output engine in one launch
template <class A>
void role_ranges(ChainHost<A> *c, RoleRange &rm, RoleRange &ro)
{
    rm.roles = 2; ro.roles = A::kOuts;
    rm.stride = ro.stride = c->d.N_pad;
}

// On queue q with its staging: images is host memory for the engine's queue, device memory for a lane's.  A lane's staging
// holds chunks of its whole window (at most 32 MiB, kept until the lane closes), so that only its first export allocates
// it: a later growth would free device memory, which waits for the device.
template <class A>
int export_instances(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, void *images, size_t stride)
{
    image::Plan pl;
    size_t size = 0;
    int rc = check_images(c, q, inst0, n, images, stride, &pl, &size);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_grow(c, *q, q->resp.d_stage != nullptr)) != DSPI_OK) return rc;
    uint32_t chunk = 0;
    CU_OK(q->resp.stage(size, q->lane ? q->n : n, q->stream, &chunk));
    CU_OK(begin_call(c, *q));
    auto issue = [&]() -> int {
        RoleRange rm, ro;
        role_ranges(c, rm, ro);
        int rc = eq_unpack_range(c->eq_m, inst0, n, q->stream, rm);         // running EQ state into the mirrors, as download_biquads
        if (rc == DSPI_OK) rc = eq_unpack_range(c->eq_o, inst0, n, q->stream, ro);
        if (rc) return rc;
        unsigned char *stage = (unsigned char *)q->resp.d_stage;
        for (uint32_t i0 = 0; i0 < n; i0 += chunk) {
            const uint32_t nc = n - i0 < chunk ? n - i0 : chunk;
            image::instance_image_kernel<image::kExport><<<dim3((nc + 31) / 32, pl.n_tasks), 256, 0, q->stream>>>(pl, inst0 + i0, nc, stage);
            CU_OK(cudaGetLastError());
            c->launches++;
            CU_OK(cudaMemcpy2DAsync((char *)images + (size_t)i0 * stride, stride, stage, size, size, nc,
                                    q->lane ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, q->stream));
        }
        return DSPI_OK;
    };
    return end_call(*q, issue());
}

// Mirror rows -> packed stores of the instances ch0 .. of rm / ro (ranges or lists over the roles), then the skip masks: on
// the engine's queue every row, synchronising, as upload_biquads and set_params do; on a lane's the rows of its window only.
template <class A>
int pack_instances(ChainHost<A> *c, Queue &q, uint32_t ch0, uint32_t n, const RoleRange &rm, const RoleRange &ro)
{
    if (q.lane) {
        const int rc = eq_pack_rows(c->eq_m, ch0, n, q.stream, rm, q.inst0, q.n);
        return rc == DSPI_OK ? eq_pack_rows(c->eq_o, ch0, n, q.stream, ro, q.inst0, q.n) : rc;
    }
    int rc = eq_pack_range(c->eq_m, ch0, n, q.stream, rm);
    if (rc == DSPI_OK) rc = eq_pack_range(c->eq_o, ch0, n, q.stream, ro);
    return rc == DSPI_OK ? bulk::finish_skip(c, q) : rc;
}

// On queue q; images is host memory on both, so that every header is checked before anything is written and the envelope
// modes the images carry (env row 4) keep env_mode exact.  The engine's queue reads the range's modes before the call from
// the device and returns when the engine is updated.  A lane's takes them from env_mode, sends each chunk of images at the
// image size from a buffer of its ring into its image staging (which export shares) with one copy, and does not wait.
template <class A>
int import_instances(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const void *images, size_t stride)
{
    image::Plan pl;
    size_t size = 0;
    int rc = check_images(c, q, inst0, n, images, stride, &pl, &size);
    if (rc || n == 0) return rc;
    const char *img = (const char *)images;
    for (uint32_t i = 0; i < n; i++) {                                       // every header before anything is written
        ImageHeader h;
        memcpy(&h, img + (size_t)i * stride, sizeof(h));
        if (h.magic != kImageMagic || h.version != kImageVersion)
            return fail(DSPI_EINVAL, "image %u is not a dspi_b200 instance image (magic %08x version %u)", i, h.magic, h.version);
        if (h.arith != c->desc.arith || h.n_bands != c->desc.n_bands || h.bytes != size)
            return fail(DSPI_EINVAL, "image %u belongs to a different engine kind (arith %u, %u bands, %llu bytes)", i, h.arith, h.n_bands,
                        (unsigned long long)h.bytes);
    }
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_prepare(c, *q, q->resp.d_stage != nullptr)) != DSPI_OK) return rc;
    // envelope-mode instances: the range's modes before (behind earlier work) and in the images (env row 4)
    uint32_t env_off = 0;
    for (uint32_t k = 0; k < pl.n_fields; k++)
        if (pl.f[k].p == (char *)c->d.env) env_off = pl.f[k].off + 4 * 4;
    const size_t Np = c->d.N_pad;
    std::vector<uint32_t> cur(q->lane ? 0 : (size_t)n);
    if (!q->lane) {
        CU_OK(cudaMemcpyAsync(cur.data(), c->d.env + 4 * Np + inst0, (size_t)n * 4, cudaMemcpyDeviceToHost, q->stream));
        CU_OK(cudaStreamSynchronize(q->stream));
    }
    uint32_t before = 0, after = 0;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t on;
        memcpy(&on, img + (size_t)i * stride + env_off, 4);
        before += (q->lane ? c->env_mode[inst0 + i] : cur[i]) ? 1u : 0u;
        after += on ? 1u : 0u;
        c->env_mode[inst0 + i] = on ? 1 : 0;
    }
    uint32_t chunk = 0;
    CU_OK(q->resp.stage(size, q->lane ? q->n : n, q->stream, &chunk));
    CU_OK(begin_call(c, *q));
    auto issue = [&]() -> int {
        unsigned char *stage = (unsigned char *)q->resp.d_stage;
        for (uint32_t i0 = 0; i0 < n; i0 += chunk) {
            const uint32_t nc = n - i0 < chunk ? n - i0 : chunk;
            const char *src = img + (size_t)i0 * stride;
            if (q->lane)
                CU_OK(bulk::lane_upload(*q, stage, (size_t)nc * size, [&](unsigned char *b) {
                    for (uint32_t i = 0; i < nc; i++) memcpy(b + (size_t)i * size, src + (size_t)i * stride, size);
                }));
            else
                CU_OK(cudaMemcpy2DAsync(stage, size, src, stride, size, nc, cudaMemcpyHostToDevice, q->stream));
            image::instance_image_kernel<image::kImport><<<dim3((nc + 31) / 32, pl.n_tasks), 256, 0, q->stream>>>(pl, inst0 + i0, nc, stage);
            CU_OK(cudaGetLastError());
            c->launches++;
        }
        c->env_instances = c->env_instances - before + after;
        // mirrors -> packed stores of the range only (topology words, skip remask, K1 kernel choice), then the skip masks
        RoleRange rm, ro;
        role_ranges(c, rm, ro);
        return pack_instances(c, *q, inst0, n, rm, ro);
    };
    return end_call(*q, issue(), false);                                     // the engine's queue synchronised in pack_instances
}

// Instance src[k] becomes what export_instances(src[k], 1) then import_instances(dst[k], 1) would make of dst[k], with
// the data moving engine to engine: running EQ state of the sources into the mirrors, every array of the image plan
// (mirror rows included) from source to destination, then the destinations' mirror rows into the packed stores.  Issued on
// the destination's queue dst_q with its lists.  The engine's (src_q == dst_q) reads the modes of the instances named from
// the device and returns when the engine is updated.  On lanes every src[k] lies in src_q's window and every dst[k] in
// dst_q's; the copy runs after the source lane's calls issued before it and the source lane's later calls run after it,
// the envelope counts come from env_mode, and the call does not wait.
template <class A>
int copy_instances(ChainHost<A> *c, Queue *src_q, Queue *dst_q, uint32_t n, const uint32_t *src, const uint32_t *dst)
{
    if (!src_q || !dst_q) return DSPI_EINVAL;
    if (!src || !dst) return fail(DSPI_EINVAL, "null argument");
    const uint32_t N = c->desc.n_instances;
    uint32_t lo = N, hi = 0;                                                // span of every index named, for the envelope count
    for (uint32_t k = 0; k < n; k++) {
        if (src[k] >= N || dst[k] >= N)
            return fail(DSPI_ERANGE, "copy %u names instance %u, outside engine of %u", k, src[k] >= N ? src[k] : dst[k], N);
        const bool src_out = src[k] - src_q->inst0 >= src_q->n;              // never for the engine's queue
        if (src_out || dst[k] - dst_q->inst0 >= dst_q->n) {
            const Queue &w = src_out ? *src_q : *dst_q;
            return fail(DSPI_ERANGE, "copy %u names instance %u, outside its lane's window [%u, %u)", k, src_out ? src[k] : dst[k], w.inst0,
                        w.inst0 + w.n);
        }
        lo = std::min(lo, std::min(src[k], dst[k]));
        hi = std::max(hi, std::max(src[k], dst[k]));
    }
    if (n == 0) return DSPI_OK;
    std::vector<uint8_t> seen((size_t)hi - lo + 1, 0);                     // 1: a source, 2: a destination
    for (uint32_t k = 0; k < n; k++) seen[src[k] - lo] |= 1;
    for (uint32_t k = 0; k < n; k++) {
        uint8_t &s = seen[dst[k] - lo];
        if (s & 2) return fail(DSPI_EINVAL, "instance %u is a destination twice", dst[k]);
        if (s & 1) return fail(DSPI_EINVAL, "instance %u is both a source and a destination", dst[k]);
        s |= 2;
    }
    image::Plan pl;
    if (!image_plan(c, kInImage, pl)) return fail(DSPI_EINVAL, "instance image plan exceeds its tables");
    CU_OK(cudaSetDevice(c->desc.device));
    Queue &q = *dst_q;
    int rc = lane_prepare(c, q, q.copy_lists.d != nullptr);
    if (rc) return rc;
    CU_OK(q.copy_lists.ensure(q.lane ? q.n : n));                           // a lane's: n <= its window (dst distinct)
    const uint32_t *d_src = q.copy_lists.d, *d_dst = q.copy_lists.d + n;
    // envelope-mode instances: the modes (env row 4) of sources and destinations, behind earlier work
    uint32_t before = 0, after = 0;
    if (q.lane) {
        CU_OK(begin_call(c, q));
        if (src_q != dst_q) CU_OK(cudaStreamWaitEvent(q.stream, src_q->ev_last, 0));
        CU_OK(bulk::lane_upload(q, q.copy_lists.d, (size_t)2 * n * 4, [&](unsigned char *b) {
            memcpy(b, src, (size_t)n * 4);
            memcpy(b + (size_t)n * 4, dst, (size_t)n * 4);
        }));
        for (uint32_t k = 0; k < n; k++) {
            before += c->env_mode[dst[k]];
            after += c->env_mode[src[k]];
            c->env_mode[dst[k]] = c->env_mode[src[k]];
        }
    } else {
        std::vector<uint32_t> lists((size_t)2 * n);
        memcpy(lists.data(), src, (size_t)n * 4);
        memcpy(lists.data() + n, dst, (size_t)n * 4);
        CU_OK(cudaMemcpyAsync(q.copy_lists.d, lists.data(), (size_t)2 * n * 4, cudaMemcpyHostToDevice, q.stream));
        std::vector<uint32_t> mode((size_t)hi - lo + 1);
        CU_OK(cudaMemcpyAsync(mode.data(), c->d.env + (size_t)4 * c->d.N_pad + lo, mode.size() * 4, cudaMemcpyDeviceToHost, q.stream));
        CU_OK(cudaStreamSynchronize(q.stream));
        for (uint32_t k = 0; k < n; k++) {
            before += mode[dst[k] - lo] ? 1u : 0u;
            after += mode[src[k] - lo] ? 1u : 0u;
            c->env_mode[dst[k]] = mode[src[k] - lo] ? 1 : 0;
        }
    }
    auto issue = [&]() -> int {
        RoleRange rm, ro;
        role_ranges(c, rm, ro);
        rm.inst = ro.inst = d_src;
        int rc = eq_unpack_range(c->eq_m, 0, n, q.stream, rm);               // running EQ state into the mirrors, as export
        if (rc == DSPI_OK) rc = eq_unpack_range(c->eq_o, 0, n, q.stream, ro);
        if (rc) return rc;
        image::instance_copy_kernel<<<dim3((n + 31) / 32, pl.n_tasks), 256, 0, q.stream>>>(pl, n, d_src, d_dst);
        CU_OK(cudaGetLastError());
        c->launches++;
        c->env_instances = c->env_instances - before + after;
        // the destinations' mirror rows -> packed stores, then the skip masks, as import
        rm.inst = ro.inst = d_dst;
        return pack_instances(c, q, 0, n, rm, ro);
    };
    rc = end_call(q, issue(), false);                                       // the engine's queue synchronised in pack_instances
    if (src_q != dst_q) {                                                   // the source lane's next call, and join_lanes, wait for the copy
        CU_OK(cudaStreamWaitEvent(src_q->stream, q.ev_last, 0));
        CU_OK(cudaEventRecord(src_q->ev_last, src_q->stream));
    }
    return rc;
}

// on queue q (the engine's or a lane's)
template <class A>
int reset_instances(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n)
{
    if (!q) return DSPI_EINVAL;
    int rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    CU_OK(begin_call(c, *q));
    CU_OK(reset_range(c, inst0, n, q->stream));
    return end_call(*q, DSPI_OK);
}

// ---- queries -----------------------------------------------------------------------------------------------------------
// Frequency response of instances [inst0, inst0 + n) on queue q (the engine's, or an open lane's: a NULL q, which the
// lane entry point refuses before anything else, is a NULL engine here, reported after the arguments as it always was);
// out: device [n][kOuts][2][n_freqs] float2, or (the engine's queue only) host memory filled chunk by chunk through the
// staging buffer
template <class A>
int response(ChainHost<A> *c, Queue *q, uint32_t inst0, uint32_t n, const float *freqs, uint32_t n_freqs, float fs, float *out, bool host)
{
    const char *why = "";
    int rc = response_check_args(freqs, n_freqs, fs, out, &why);
    if (rc) return fail(rc, "%s", why);
    if (!q) return fail(DSPI_EINVAL, "null argument");
    if (q->lane && ((uintptr_t)out & 7u)) return fail(DSPI_EINVAL, "d_out must be 8-byte aligned (the kernel stores {re, im} pairs)");
    rc = check_range(*q, inst0, n);
    if (rc || n == 0) return rc;
    CU_OK(cudaSetDevice(c->desc.device));
    if ((rc = lane_grow(c, *q, q->resp.d_freq != nullptr)) != DSPI_OK) return rc;
    CU_OK(begin_call(c, *q));
    using B = typename A::Biquad;
    const B *m_aos = (const B *)eq_aos_mirror(c->eq_m), *o_aos = (const B *)eq_aos_mirror(c->eq_o);
    auto launch = [&](uint32_t i0, uint32_t m, void *dst) -> cudaError_t {
        const dim3 grid((n_freqs + 127) / 128, m < 65535u ? m : 65535u);
        A::response<<<grid, 128, 0, q->stream>>>(c->d, m_aos, o_aos, i0, m, q->resp.d_freq, n_freqs, fs, (float2 *)dst);
        c->launches++;
        return cudaGetLastError();
    };
    auto issue = [&]() -> int {
        CU_OK(q->resp.upload(freqs, n_freqs, q->stream, &c->launches));
        if (!host) {
            CU_OK(launch(inst0, n, out));
            return DSPI_OK;
        }
        const size_t row_bytes = (size_t)A::kOuts * 2 * n_freqs * 2 * sizeof(float);
        uint32_t rows = 0;
        CU_OK(q->resp.stage(row_bytes, n, q->stream, &rows));
        for (uint32_t i = 0; i < n; i += rows) {
            const uint32_t m = n - i < rows ? n - i : rows;
            CU_OK(launch(inst0 + i, m, q->resp.d_stage));
            CU_OK(cudaMemcpyAsync((char *)out + (size_t)i * row_bytes, q->resp.d_stage, (size_t)m * row_bytes, cudaMemcpyDeviceToHost, q->stream));
            CU_OK(cudaStreamSynchronize(q->stream));
        }
        return DSPI_OK;
    };
    return end_call(*q, issue(), host);
}

template <class A>
int sync(ChainHost<A> *c)
{
    if (!c) return fail(DSPI_EINVAL, "null argument");
    CU_OK(cudaSetDevice(c->desc.device));
    CU_OK(cudaStreamSynchronize(c->q.stream));
    return DSPI_OK;
}

template <class A>
void *stream(ChainHost<A> *c) { return c ? (void *)c->q.stream : nullptr; }

// SMs reserved for the modulator / left to every other stage (0, 0: no partition, see chain_streams.cuh)
template <class A>
int sm_partition(ChainHost<A> *c, uint32_t *pdm_sms, uint32_t *rest_sms)
{
    if (!c) return fail(DSPI_EINVAL, "null argument");
    if (pdm_sms) *pdm_sms = c->part.pdm_sms;
    if (rest_sms) *rest_sms = c->part.rest_sms;
    return DSPI_OK;
}

template <class A>
uint64_t launch_count(ChainHost<A> *c)
{
    return c ? c->launches + dspi_eq_launch_count(c->eq_m) + dspi_eq_launch_count(c->eq_o) : 0;
}

}  // namespace
}  // namespace dspi
