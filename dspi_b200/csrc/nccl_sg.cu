// nccl_sg.cu — frames that originate on ONE rank of a multi-process job: scatter, process, gather over NCCL, natively.
//
// SURVEY.md §8(e): instances / channels shard with no halo and no reduction, so the only communication a multi-GPU job can
// need is moving frames from the rank that has them to the ranks that own the channels and the results back - NCCL
// send / recv inside ncclGroupStart / ncclGroupEnd (NCCL has no scatter / gather), chunked and double-buffered so that the
// transfer of chunk j+1 overlaps the kernel of chunk j.  One process per GPU (torchrun); the communicator is created here
// from a unique id the caller distributes (dspi_b200/sharding.py broadcasts it over torch.distributed).
//
// Pipeline, step j = 0 .. K+L-1, all enqueued from the host without waiting (events order the streams):
//     comm stream     one NCCL group:  root  -> every peer  chunk j      (ncclSend / ncclRecv)
//                                      peers -> root        chunk j-L    (both NVLink directions busy in the same kernel)
//     compute streams K1 / K2 over the chunks that have arrived, chunk j on stream j mod S
// A cascade kernel runs as long as its rows are long however few rows it gets (parallel over channels, serial over time:
// ~1 ms for 6144 frames) but a chunk of a shard fills only a few SMs, so the kernels of consecutive chunks run CONCURRENTLY
// on several streams and a chunk travels back L steps after it arrived (L = kernel time / step time, rounded up, + 1).
// A peer keeps a ring of L + 2 chunk buffers; the root works in place on the caller's block.  Chunks are row ranges on
// 64-channel boundaries; sharding, chunking and the concurrency change no bit.
//
// libnccl is dlopen'ed (the copy torch already loaded when there is one), so the library has no link-time dependency on it
// and single-GPU users never touch it.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <dlfcn.h>
#include <new>
#include <vector>
#include <nccl.h>

#include "eq_kernels.cuh"

namespace {

int failn(int code, const char *fmt, ...)
{
    size_t cap = 0;
    char *buf = dspi::error_buffer(&cap);
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, cap, fmt, ap);
    va_end(ap);
    return code;
}

struct Nccl {
    void *so = nullptr;
    decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
    decltype(&ncclCommInitRank) CommInitRank = nullptr;
    decltype(&ncclCommDestroy) CommDestroy = nullptr;
    decltype(&ncclSend) Send = nullptr;
    decltype(&ncclRecv) Recv = nullptr;
    decltype(&ncclGroupStart) GroupStart = nullptr;
    decltype(&ncclGroupEnd) GroupEnd = nullptr;
    decltype(&ncclGetErrorString) GetErrorString = nullptr;
    bool ok = false;
};

const Nccl &nccl()
{
    static const Nccl n = [] {
        Nccl a;
        a.so = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);              // the copy already in the process (torch's), if any
        if (!a.so) a.so = dlopen("libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
        if (!a.so) a.so = dlopen("libnccl.so", RTLD_NOW | RTLD_LOCAL);
        if (!a.so) return a;
#define SYM(f) *(void **)(&a.f) = dlsym(a.so, "nccl" #f)
        SYM(GetUniqueId); SYM(CommInitRank); SYM(CommDestroy); SYM(Send); SYM(Recv); SYM(GroupStart); SYM(GroupEnd); SYM(GetErrorString);
#undef SYM
        a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.Send && a.Recv && a.GroupStart && a.GroupEnd && a.GetErrorString;
        return a;
    }();
    return n;
}

constexpr int kMaxLag = 30, kMaxRing = kMaxLag + 2, kStreams = 8;

}  // namespace

struct dspi_sg {
    dspi_eq *eng;
    int rank, world, root, device;
    ncclComm_t comm;
    cudaStream_t s_comm;
    cudaStream_t s_comp[kStreams];
    std::vector<cudaEvent_t> ev_recv, ev_done;     // per chunk
    void *ring[kMaxRing];
    int ring_slots;
    size_t ring_bytes;
    uint32_t rows;                                  // channels of this rank's shard == engine channels
};

#define CU_OKN(expr)                                                                                          \
    do {                                                                                                      \
        cudaError_t err__ = (expr);                                                                           \
        if (err__ != cudaSuccess) return failn(DSPI_ECUDA, "%s -> %s (%s:%d)", #expr, cudaGetErrorString(err__), __FILE__, __LINE__); \
    } while (0)
#define NC_OK(expr)                                                                                           \
    do {                                                                                                      \
        ncclResult_t r__ = (expr);                                                                            \
        if (r__ != ncclSuccess) return failn(DSPI_ECUDA, "%s -> %s (%s:%d)", #expr, nccl().GetErrorString(r__), __FILE__, __LINE__); \
    } while (0)

extern "C" {

int dspi_nccl_unique_id(void *id128)
{
    if (!id128) return failn(DSPI_EINVAL, "null argument");
    if (!nccl().ok) return failn(DSPI_ENODEV, "libnccl.so.2 not found");
    ncclUniqueId id;
    NC_OK(nccl().GetUniqueId(&id));
    static_assert(sizeof(id) == 128, "ncclUniqueId is 128 bytes");
    memcpy(id128, &id, 128);
    return DSPI_OK;
}

int dspi_sg_destroy(dspi_sg *g)
{
    if (!g) return DSPI_OK;
    cudaSetDevice(g->device);
    if (g->s_comm) cudaStreamSynchronize(g->s_comm);
    for (cudaEvent_t e : g->ev_recv) cudaEventDestroy(e);
    for (cudaEvent_t e : g->ev_done) cudaEventDestroy(e);
    for (int i = 0; i < kMaxRing; i++) if (g->ring[i]) cudaFree(g->ring[i]);
    if (g->comm) nccl().CommDestroy(g->comm);
    if (g->s_comm) cudaStreamDestroy(g->s_comm);
    for (int i = 0; i < kStreams; i++) if (g->s_comp[i]) { cudaStreamSynchronize(g->s_comp[i]); cudaStreamDestroy(g->s_comp[i]); }
    delete g;
    cudaGetLastError();
    return DSPI_OK;
}

int dspi_sg_create(dspi_sg **out, dspi_eq *engine, int device, const void *id128, int rank, int world, int root)
{
    if (!out || !engine || !id128) return failn(DSPI_EINVAL, "null argument");
    *out = nullptr;
    if (world < 1 || rank < 0 || rank >= world || root < 0 || root >= world) return failn(DSPI_EINVAL, "rank %d / world %d / root %d", rank, world, root);
    if (!nccl().ok) return failn(DSPI_ENODEV, "libnccl.so.2 not found");
    dspi_sg *g = new (std::nothrow) dspi_sg();
    if (!g) return failn(DSPI_ENOMEM, "host allocation failed");
    g->eng = engine; g->rank = rank; g->world = world; g->root = root; g->device = device;
    g->comm = nullptr; g->s_comm = nullptr; g->ring_bytes = 0; g->ring_slots = 0; g->rows = 0;
    for (int i = 0; i < kMaxRing; i++) g->ring[i] = nullptr;
    for (int i = 0; i < kStreams; i++) g->s_comp[i] = nullptr;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&g->s_comm, cudaStreamNonBlocking);
    for (int i = 0; i < kStreams && e == cudaSuccess; i++) e = cudaStreamCreateWithFlags(&g->s_comp[i], cudaStreamNonBlocking);
    if (e != cudaSuccess) { dspi_sg_destroy(g); return failn(DSPI_ECUDA, "stream: %s", cudaGetErrorString(e)); }
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    const ncclResult_t r = nccl().CommInitRank(&g->comm, world, id, rank);
    if (r != ncclSuccess) { g->comm = nullptr; dspi_sg_destroy(g); return failn(DSPI_ECUDA, "ncclCommInitRank: %s", nccl().GetErrorString(r)); }
    *out = g;
    return DSPI_OK;
}

/* Every rank calls this with the same total_channels / T / n_chunks; `d_full` ([total_channels][T], device memory of the
 * root) is read on the root only.  The engine of rank r must hold channels [lo_r, hi_r) of dspi_eqx_shard_range(total, world, r).
 * Returns when the block on the root is complete (all ranks return after their last transfer). */
int dspi_sg_process(dspi_sg *g, void *d_full, uint32_t total_channels, uint32_t T, uint32_t n_chunks)
{
    if (!g) return failn(DSPI_EINVAL, "null argument");
    if (T == 0 || total_channels == 0) return DSPI_OK;
    if (T % 4) return failn(DSPI_EINVAL, "T must be a multiple of 4 (dense rows feed the TMA path)");
    const bool is_root = g->rank == g->root;
    if (is_root && !d_full) return failn(DSPI_EINVAL, "the root needs the block");
    CU_OKN(cudaSetDevice(g->device));
    const int W = g->world;
    std::vector<uint32_t> lo(W), hi(W);
    for (int r = 0; r < W; r++) dspi_eqx_shard_range(total_channels, (uint32_t)W, (uint32_t)r, &lo[r], &hi[r]);
    // Transfer time of one direction: the root moves every peer's shard over its own links (estimated at 650 GB/s for
    // grouped ncclSend / ncclRecv); kernel time: ~0.17 us per frame (float; the Q28 cascade ~6x).  Both are estimates that
    // only set the chunk count, which changes no bit.
    const double t_dir = (double)(total_channels - (hi[g->root] - lo[g->root])) * T * 4.0 / 650e9;
    const double t_kernel = (double)T * 0.17e-6 * 1.1;
    if (n_chunks == 0) {                                                     // automatic: steps of about half a millisecond
        const double k = t_dir / 0.5e-3;
        n_chunks = k < 4.0 ? 4u : (k > 32.0 ? 32u : (uint32_t)k);
    }
    const uint32_t my_rows = hi[g->rank] - lo[g->rank];
    // chunk ranges of a shard: <= n_chunks pieces on 64-row boundaries; identical arithmetic on every rank
    auto chunk_rows = [&](uint32_t rows) { uint32_t per = (rows + n_chunks - 1) / n_chunks; per = (per + 63) / 64 * 64; return per ? per : 64u; };
    auto n_of = [&](uint32_t rows) { const uint32_t per = chunk_rows(rows); return (rows + per - 1) / per; };
    uint32_t K = 0;
    for (int r = 0; r < W; r++) { const uint32_t k = n_of(hi[r] - lo[r]); if (k > K) K = k; }
    cudaStream_t s_eng = (cudaStream_t)dspi_eq_stream(g->eng);
    if (g->ev_recv.size() < K) {
        const size_t old = g->ev_recv.size();
        g->ev_recv.resize(K); g->ev_done.resize(K);
        for (size_t i = old; i < K; i++) {
            CU_OKN(cudaEventCreateWithFlags(&g->ev_recv[i], cudaEventDisableTiming));
            CU_OKN(cudaEventCreateWithFlags(&g->ev_done[i], cudaEventDisableTiming));
        }
    }
    const uint32_t my_per = chunk_rows(my_rows), my_k = my_rows ? n_of(my_rows) : 0;
    // lag between a chunk's arrival and its return: its kernel must have finished, and kernels of consecutive chunks overlap
    uint32_t L = (uint32_t)(t_kernel / (t_dir / (double)K)) + 2u;
    if (L < 2u) L = 2u;
    if (L > (uint32_t)kMaxLag) L = (uint32_t)kMaxLag;
    const uint32_t R = L + 2u;                                               // ring slots of a peer
    if (!is_root) {
        const size_t need = (size_t)my_per * T * 4;
        if (need > g->ring_bytes || (int)R > g->ring_slots) {
            CU_OKN(cudaStreamSynchronize(g->s_comm));
            for (int i = 0; i < kStreams; i++) CU_OKN(cudaStreamSynchronize(g->s_comp[i]));
            for (int i = 0; i < kMaxRing; i++) { if (g->ring[i]) cudaFree(g->ring[i]); g->ring[i] = nullptr; }
            g->ring_bytes = 0; g->ring_slots = 0;
            for (uint32_t i = 0; i < R; i++) CU_OKN(cudaMalloc(&g->ring[i], need));
            g->ring_bytes = need; g->ring_slots = (int)R;
        }
    }
    // the root's own rows need no transfer: its kernel runs beside the transfers, in place
    if (is_root && my_rows) {
        const int rc = dspi_eq_process_device_range(g->eng, (char *)d_full + (size_t)lo[g->rank] * T * 4, T, T, 0, my_rows);
        if (rc) return rc;
    }
    if (W == 1) { CU_OKN(cudaStreamSynchronize(s_eng)); return DSPI_OK; }
    for (uint32_t j = 0; j < K + L; j++) {
        if (!is_root && j >= L && j - L < my_k) CU_OKN(cudaStreamWaitEvent(g->s_comm, g->ev_done[j - L], 0));      // results of chunk j-L are complete
        NC_OK(nccl().GroupStart());
        if (is_root) {
            for (int r = 0; r < W; r++) {
                if (r == g->root) continue;
                const uint32_t rows = hi[r] - lo[r], per = chunk_rows(rows), k = rows ? n_of(rows) : 0;
                if (j < k) {
                    const uint32_t a = j * per, b = (a + per < rows) ? a + per : rows;
                    NC_OK(nccl().Send((char *)d_full + ((size_t)lo[r] + a) * T * 4, (size_t)(b - a) * T, ncclFloat, r, g->comm, g->s_comm));
                }
                if (j >= L && j - L < k) {
                    const uint32_t a = (j - L) * per, b = (a + per < rows) ? a + per : rows;
                    NC_OK(nccl().Recv((char *)d_full + ((size_t)lo[r] + a) * T * 4, (size_t)(b - a) * T, ncclFloat, r, g->comm, g->s_comm));
                }
            }
        } else {
            if (j < my_k) {                                                  // slot j mod R was last sent from at step j - R + L < j: free
                const uint32_t a = j * my_per, b = (a + my_per < my_rows) ? a + my_per : my_rows;
                NC_OK(nccl().Recv(g->ring[j % R], (size_t)(b - a) * T, ncclFloat, g->root, g->comm, g->s_comm));
            }
            if (j >= L && j - L < my_k) {
                const uint32_t a = (j - L) * my_per, b = (a + my_per < my_rows) ? a + my_per : my_rows;
                NC_OK(nccl().Send(g->ring[(j - L) % R], (size_t)(b - a) * T, ncclFloat, g->root, g->comm, g->s_comm));
            }
        }
        NC_OK(nccl().GroupEnd());
        if (!is_root && j < my_k) {                                          // chunk j arrived: its kernel starts on its own stream
            cudaStream_t cs = g->s_comp[j % kStreams];
            CU_OKN(cudaEventRecord(g->ev_recv[j], g->s_comm));
            CU_OKN(cudaStreamWaitEvent(cs, g->ev_recv[j], 0));
            const uint32_t a = j * my_per, b = (a + my_per < my_rows) ? a + my_per : my_rows;
            const int rc = dspi::eq_process_range_on(g->eng, g->ring[j % R], T, T, a, b - a, cs);
            if (rc) return rc;
            CU_OKN(cudaEventRecord(g->ev_done[j], cs));
        }
    }
    for (int i = 0; i < kStreams; i++) CU_OKN(cudaStreamSynchronize(g->s_comp[i]));
    CU_OKN(cudaStreamSynchronize(g->s_comm));
    CU_OKN(cudaStreamSynchronize(s_eng));
    return DSPI_OK;
}

}  // extern "C"
