// engine.cu — the C-ABI of include/dspi_b200.h: EQ engine (K1 float / K2 Q28).
//
// No CPU fallback lives here: without an sm_90 device every create call fails with
// DSPI_ENODEV and nothing else can be reached.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <new>
#include <utility>
#include <vector>
#include <sched.h>
#include <unistd.h>
#include <sys/syscall.h>

#include "eq_kernels.cuh"
#include "eq_jit.h"
#include "response.cuh"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define CU_OK(expr)                                                                                         \
    do {                                                                                                    \
        cudaError_t err__ = (expr);                                                                         \
        if (err__ != cudaSuccess) return fail(DSPI_ECUDA, "%s -> %s (%s:%d)", #expr, cudaGetErrorString(err__), __FILE__, __LINE__); \
    } while (0)

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

constexpr int kHostBufs = 8;   // staging ring of the host / peer pipeline; each buffer has a kernel stream of its own

}  // namespace

namespace dspi {
char *error_buffer(size_t *cap)
{
    *cap = sizeof(g_err);
    return g_err;
}
}  // namespace dspi

struct dspi_eq {
    dspi_eq_desc desc;
    int cpl;                 // channels per lane (float: 1 or 2, which also fixes K1's stage geometry; Q28: 1)
    uint32_t rows;           // channels per group = 32 * cpl
    uint32_t n_groups;
    uint32_t c_pad;          // n_groups * rows
    cudaStream_t stream, s_h2d, s_d2h;
    cudaStream_t s_k[kHostBufs];   // chunk kernels of the staged pipeline (eq_process_remote_enqueue)
    cudaEvent_t ev_begin;
    void *d_aos;             // Biquad[c_pad][12] in the reference layout (device mirror)
    void *d_coef;            // packed coefficient + state store
    uint64_t *d_modes;       // float only: per-channel topology words as packed from the coefficient structs
    uint64_t *d_modes_eff;   // with the caller's skip mask applied (chain engines), else nullptr
    const uint8_t *d_skip;   // not owned
    uint32_t *d_sched;       // float only: dynamic scheduler words (sched_words)
    int n_sms;
    size_t aos_elem;
    uint64_t launches;
    // host-path staging
    void *d_stage[kHostBufs];
    size_t stage_bytes;
    cudaEvent_t ev_in[kHostBufs], ev_done[kHostBufs], ev_out[kHostBufs];
    // tensor-map cache
    CUtensorMap tmap;
    void *tm_ptr;
    uint32_t tm_T, tm_ld, tm_rows;
    // kernel choice (float engines): re-derived after every coefficient upload
    bool sig_dirty;
    bool sig_stale;          // rows re-packed by a lane control call since the last choice (eq_choice_stale)
    void *jit;               // run-time specialised K1 (eq_jit.cu) or nullptr = ahead-of-time kernels
    char kinfo[320];
    dspi::ResponseBuffers resp;   // frequency table and host staging of dspi_eq_response_*
};

// Scheduler words of K1's dynamic schedule (DSPI_DBG=8): a launch over groups [g0, g0 + ng) starting at row row_lo of g0
// uses 1 + ng words from word 2 h, h = (g0 * rows + row_lo) / 32 its first 32-row block.  A launch spans at least ng such
// blocks, so launches over disjoint channel ranges, which may share a 64-row group at their boundary, use disjoint words
// and may run concurrently; a whole-engine launch uses words 0 .. n_groups, as a single counter block would.
static size_t sched_words(const dspi_eq *e) { return 2 * (size_t)(e->c_pad / 32) + 1; }

extern "C" {

const char *dspi_last_error(void) { return g_err; }

int dspi_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    int ok = 0;
    for (int i = 0; i < n; i++) {
        int major = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess && major == 9) ok++;
    }
    return ok;
}

void *dspi_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void dspi_host_free(void *p) { if (p) cudaFreeHost(p); }

/* Pin the calling thread (and the pages it touches from now on) to the NUMA node the GPU's PCIe link hangs off, so
 * that pinned staging memory allocated afterwards is local to the link and host <-> device copies do not cross the
 * socket interconnect.  Linux sysfs only; returns the node (>= 0), or -1 when the topology is unknown (nothing changed). */
int dspi_bind_host_to_device(int device)
{
    char bus[32] = { 0 };
    if (cudaDeviceGetPCIBusId(bus, (int)sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char *p = bus; *p; p++) if (*p >= 'A' && *p <= 'F') *p = (char)(*p - 'A' + 'a');
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return -1;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return -1;
    cpu_set_t set;
    CPU_ZERO(&set);
    int lo = 0, hi = 0, n = 0;
    char sep = 0;
    while (fscanf(f, "%d", &lo) == 1) {                                     /* "0-31,64-95" */
        hi = lo;
        if (fscanf(f, "%c", &sep) == 1 && sep == '-') { if (fscanf(f, "%d", &hi) != 1) hi = lo; if (fscanf(f, "%c", &sep) != 1) sep = 0; }
        for (int c = lo; c <= hi && c < CPU_SETSIZE; c++) { CPU_SET(c, &set); n++; }
        if (sep != ',') break;
    }
    fclose(f);
    if (n == 0) return -1;
    cpu_set_t allowed;                                                       /* stay inside the cpuset this process was given */
    if (sched_getaffinity(0, sizeof(allowed), &allowed) == 0) {
        cpu_set_t both;
        CPU_AND(&both, &set, &allowed);
        if (CPU_COUNT(&both) == 0) return -1;
        set = both;
    }
    if (sched_setaffinity(0, sizeof(set), &set) != 0) return -1;
#ifdef SYS_set_mempolicy
    if (node < 1024) {                                                       /* MPOL_PREFERRED = 1: fall back to other nodes when full */
        unsigned long mask[16] = { 0 };
        mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
        syscall(SYS_set_mempolicy, 1, mask, (unsigned long)(sizeof(mask) * 8));
    }
#endif
    return node;
}

// Writes the record dsp_compute_coefficients() makes of a flat recipe (bypass set, b0 = 1, everything else zero) into every
// band of channels [0, c_pad) of the mirror: one row from the host, then doubling device-to-device copies.
static cudaError_t fill_default_records(dspi_eq *e)
{
    const bool q28 = e->desc.arith == DSPI_ARITH_Q28;
    const size_t row = (size_t)DSPI_MAX_BANDS * e->aos_elem;
    alignas(8) unsigned char rec[DSPI_MAX_BANDS * sizeof(dspi_biquad_f32)];
    memset(rec, 0, sizeof(rec));
    for (int b = 0; b < DSPI_MAX_BANDS; b++) {
        dspi_eq_param p;
        memset(&p, 0, sizeof(p));
        p.band = (uint8_t)b; p.type = DSPI_FILTER_FLAT; p.freq = 1000.0f; p.Q = 0.707f;
        if (q28) dspi_compute_coefficients_q28(&p, (dspi_biquad_q28 *)rec + b, 48000.0f);
        else dspi_compute_coefficients_f32(&p, (dspi_biquad_f32 *)rec + b, 48000.0f);
    }
    char *dst = (char *)e->d_aos;
    cudaError_t err = cudaMemcpyAsync(dst, rec, row, cudaMemcpyHostToDevice, e->stream);
    for (size_t k = 1; err == cudaSuccess && k < e->c_pad; k *= 2)
        err = cudaMemcpyAsync(dst + k * row, dst, std::min<size_t>(k, e->c_pad - k) * row, cudaMemcpyDeviceToDevice, e->stream);
    return err;
}

int dspi_eq_create(dspi_eq **out, const dspi_eq_desc *desc)
{
    if (!out || !desc) return fail(DSPI_EINVAL, "null argument");
    *out = nullptr;
    if (desc->arith > DSPI_ARITH_Q28) return fail(DSPI_EINVAL, "unknown arith %u", desc->arith);
    if (desc->n_channels == 0) return fail(DSPI_EINVAL, "n_channels must be > 0");
    if (desc->n_bands == 0 || desc->n_bands > DSPI_MAX_BANDS) return fail(DSPI_EINVAL, "n_bands must be 1..%d", DSPI_MAX_BANDS);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(DSPI_ENODEV, "no CUDA device (there is no CPU fallback)"); }
    if (desc->device < 0 || desc->device >= ndev) return fail(DSPI_ENODEV, "device %d out of range (%d visible)", desc->device, ndev);
    int major = 0;
    CU_OK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, desc->device));
    if (major != 9) return fail(DSPI_ENODEV, "device %d has compute capability %d.x; the kernels are built for sm_90a only", desc->device, major);
    if (!encode_fn()) return fail(DSPI_ENODEV, "driver does not export cuTensorMapEncodeTiled");
    CU_OK(cudaSetDevice(desc->device));

    dspi_eq *e = new (std::nothrow) dspi_eq();
    if (!e) return fail(DSPI_ENOMEM, "host allocation failed");
    memset(e, 0, sizeof(*e));
    e->desc = *desc;
    e->sig_dirty = true;
    const bool q28 = desc->arith == DSPI_ARITH_Q28;
    // K1 geometry: one channel per lane, 32 rows x 64 samples per stage (default), or a register pair per lane,
    // 64 rows x 32 samples per stage (DSPI_F32_CPL=2, for A/B measurement).  Fixed at create time: the packed
    // coefficient store is laid out by channels per lane.
    e->cpl = 1;
    if (const char *v = getenv("DSPI_F32_CPL")) e->cpl = atoi(v) == 2 ? 2 : 1;
    if (q28) e->cpl = 1;
    e->rows = 32u * e->cpl;
    e->n_groups = (desc->n_channels + e->rows - 1) / e->rows;
    e->c_pad = e->n_groups * e->rows;
    e->aos_elem = q28 ? sizeof(dspi_biquad_q28) : sizeof(dspi_biquad_f32);

    cudaError_t err;
    const size_t aos_bytes = (size_t)e->c_pad * DSPI_MAX_BANDS * e->aos_elem;
    const size_t coef_bytes = q28 ? (size_t)e->n_groups * DSPI_MAX_BANDS * 20 * 32 * 4 : (size_t)e->c_pad * DSPI_MAX_BANDS * 8 * 4;
    if ((err = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)) != cudaSuccess) goto cuda_fail;
    if ((err = cudaStreamCreateWithFlags(&e->s_h2d, cudaStreamNonBlocking)) != cudaSuccess) goto cuda_fail;
    if ((err = cudaStreamCreateWithFlags(&e->s_d2h, cudaStreamNonBlocking)) != cudaSuccess) goto cuda_fail;
    if ((err = cudaEventCreateWithFlags(&e->ev_begin, cudaEventDisableTiming)) != cudaSuccess) goto cuda_fail;
    for (int i = 0; i < kHostBufs; i++) {
        if ((err = cudaStreamCreateWithFlags(&e->s_k[i], cudaStreamNonBlocking)) != cudaSuccess) goto cuda_fail;
        if ((err = cudaEventCreateWithFlags(&e->ev_in[i], cudaEventDisableTiming)) != cudaSuccess) goto cuda_fail;
        if ((err = cudaEventCreateWithFlags(&e->ev_done[i], cudaEventDisableTiming)) != cudaSuccess) goto cuda_fail;
        if ((err = cudaEventCreateWithFlags(&e->ev_out[i], cudaEventDisableTiming)) != cudaSuccess) goto cuda_fail;
    }
    if ((err = cudaMalloc(&e->d_aos, aos_bytes)) != cudaSuccess) goto cuda_fail;
    if ((err = cudaMalloc(&e->d_coef, coef_bytes)) != cudaSuccess) goto cuda_fail;
    if ((err = cudaMemsetAsync(e->d_aos, 0, aos_bytes, e->stream)) != cudaSuccess) goto cuda_fail;
    if ((err = cudaMemsetAsync(e->d_coef, 0, coef_bytes, e->stream)) != cudaSuccess) goto cuda_fail;
    if (!q28) {
        if ((err = cudaMalloc(&e->d_modes, (size_t)e->c_pad * 8)) != cudaSuccess) goto cuda_fail;
        if ((err = cudaMalloc(&e->d_sched, sched_words(e) * 4)) != cudaSuccess) goto cuda_fail;
        if ((err = cudaDeviceGetAttribute(&e->n_sms, cudaDevAttrMultiProcessorCount, desc->device)) != cudaSuccess) goto cuda_fail;
        if ((err = cudaMemsetAsync(e->d_modes, 0, (size_t)e->c_pad * 8, e->stream)) != cudaSuccess) goto cuda_fail;
    }
    // every band of every (padding) channel starts bypassed, like dsp_init_default_filters() (dsp_pipeline.c:177-199)
    if ((err = fill_default_records(e)) != cudaSuccess) goto cuda_fail;
    err = q28 ? dspi::launch_pack_q28((const dspi_biquad_q28 *)e->d_aos, 0, e->c_pad, (int32_t *)e->d_coef, e->stream)
              : dspi::launch_pack_f32((const dspi_biquad_f32 *)e->d_aos, 0, e->c_pad, (float *)e->d_coef, e->d_modes, e->cpl, e->stream);
    if (err != cudaSuccess) goto cuda_fail;
    e->launches++;
    if ((err = cudaStreamSynchronize(e->stream)) != cudaSuccess) goto cuda_fail;
    *out = e;
    return DSPI_OK;

cuda_fail:
    fail(DSPI_ECUDA, "engine setup: %s", cudaGetErrorString(err));
    dspi_eq_destroy(e);
    return err == cudaErrorMemoryAllocation ? DSPI_ENOMEM : DSPI_ECUDA;
}

int dspi_eq_destroy(dspi_eq *e)
{
    if (!e) return DSPI_OK;
    cudaSetDevice(e->desc.device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->s_h2d) cudaStreamSynchronize(e->s_h2d);
    if (e->s_d2h) cudaStreamSynchronize(e->s_d2h);
    for (int i = 0; i < kHostBufs; i++) {
        if (e->s_k[i]) { cudaStreamSynchronize(e->s_k[i]); cudaStreamDestroy(e->s_k[i]); }
        if (e->d_stage[i]) cudaFree(e->d_stage[i]);
        if (e->ev_in[i]) cudaEventDestroy(e->ev_in[i]);
        if (e->ev_done[i]) cudaEventDestroy(e->ev_done[i]);
        if (e->ev_out[i]) cudaEventDestroy(e->ev_out[i]);
    }
    if (e->d_aos) cudaFree(e->d_aos);
    if (e->d_coef) cudaFree(e->d_coef);
    if (e->d_modes) cudaFree(e->d_modes);
    if (e->d_modes_eff) cudaFree(e->d_modes_eff);
    if (e->d_sched) cudaFree(e->d_sched);
    e->resp.destroy();
    if (e->stream) cudaStreamDestroy(e->stream);
    if (e->s_h2d) cudaStreamDestroy(e->s_h2d);
    if (e->s_d2h) cudaStreamDestroy(e->s_d2h);
    if (e->ev_begin) cudaEventDestroy(e->ev_begin);
    delete e;
    cudaGetLastError();
    return DSPI_OK;
}

static int check_range(dspi_eq *e, uint32_t ch0, uint32_t n, const void *p)
{
    if (!e || !p) return fail(DSPI_EINVAL, "null argument");
    if ((uint64_t)ch0 + n > e->desc.n_channels) return fail(DSPI_ERANGE, "channels [%u, %u) outside engine of %u", ch0, ch0 + n, e->desc.n_channels);
    return DSPI_OK;
}

int dspi_eq_upload_biquads(dspi_eq *e, uint32_t ch0, uint32_t n, const void *biquads)
{
    int rc = check_range(e, ch0, n, biquads);
    if (rc) return rc;
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    const size_t row = (size_t)DSPI_MAX_BANDS * e->aos_elem;
    CU_OK(cudaMemcpyAsync((char *)e->d_aos + ch0 * row, biquads, n * row, cudaMemcpyHostToDevice, e->stream));
    if (e->desc.arith == DSPI_ARITH_Q28)
        CU_OK(dspi::launch_pack_q28((const dspi_biquad_q28 *)e->d_aos, ch0, n, (int32_t *)e->d_coef, e->stream));
    else
        CU_OK(dspi::launch_pack_f32((const dspi_biquad_f32 *)e->d_aos, ch0, n, (float *)e->d_coef, e->d_modes, e->cpl, e->stream));
    e->launches++;
    e->sig_dirty = true;
    CU_OK(cudaStreamSynchronize(e->stream));     // the caller may reuse `biquads` immediately
    return DSPI_OK;
}

int dspi_eq_download_biquads(dspi_eq *e, uint32_t ch0, uint32_t n, void *biquads)
{
    int rc = check_range(e, ch0, n, biquads);
    if (rc) return rc;
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    if (e->desc.arith == DSPI_ARITH_Q28)
        CU_OK(dspi::launch_unpack_q28((dspi_biquad_q28 *)e->d_aos, ch0, n, (const int32_t *)e->d_coef, e->stream));
    else
        CU_OK(dspi::launch_unpack_f32((dspi_biquad_f32 *)e->d_aos, ch0, n, (const float *)e->d_coef, e->cpl, e->stream));
    e->launches++;
    const size_t row = (size_t)DSPI_MAX_BANDS * e->aos_elem;
    CU_OK(cudaMemcpyAsync(biquads, (char *)e->d_aos + ch0 * row, n * row, cudaMemcpyDeviceToHost, e->stream));
    CU_OK(cudaStreamSynchronize(e->stream));
    return DSPI_OK;
}

int dspi_eq_set_params_device(dspi_eq *e, uint32_t ch0, uint32_t n, dspi_eq_param *recipes, float sample_rate)
{
    int rc = check_range(e, ch0, n, recipes);
    if (rc) return rc;
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    const size_t bytes = (size_t)n * DSPI_MAX_BANDS * sizeof(dspi_eq_param);
    // the mirror must carry the CURRENT filter state before it is edited: dsp_compute_coefficients keeps state
    // unless the topology flips, and the pack kernel below writes the mirror's state back into the packed store
    rc = dspi::eq_unpack_range(e, ch0, n, e->stream);
    if (rc) return rc;
    dspi_eq_param *d_rec = nullptr;
    CU_OK(cudaMalloc((void **)&d_rec, bytes));
    cudaError_t err = cudaMemcpyAsync(d_rec, recipes, bytes, cudaMemcpyHostToDevice, e->stream);
    if (err == cudaSuccess) err = dspi::launch_coeffs(e->desc.arith == DSPI_ARITH_Q28, d_rec, e->d_aos, ch0, n, sample_rate, e->stream);
    if (err == cudaSuccess) err = cudaMemcpyAsync(recipes, d_rec, bytes, cudaMemcpyDeviceToHost, e->stream);   // the clamps, like the reference's write-back
    if (err == cudaSuccess) err = cudaStreamSynchronize(e->stream);
    cudaFree(d_rec);
    if (err != cudaSuccess) return fail(DSPI_ECUDA, "coefficient generation: %s", cudaGetErrorString(err));
    e->launches++;
    return dspi::eq_pack_range(e, ch0, n, e->stream);          // mirror -> packed store (and topology words)
}

int dspi_eq_set_param(dspi_eq *e, uint32_t channel, dspi_eq_param *p, float sample_rate)
{
    if (!e || !p) return fail(DSPI_EINVAL, "null argument");
    if (channel >= e->desc.n_channels) return fail(DSPI_ERANGE, "channel %u outside engine of %u", channel, e->desc.n_channels);
    if (p->band >= DSPI_MAX_BANDS) return fail(DSPI_ERANGE, "band %u >= %d", p->band, DSPI_MAX_BANDS);
    // main.c:826-857: between packets, recompute filters[ch][band] in place (state kept unless the topology flips)
    alignas(8) unsigned char rowbuf[DSPI_MAX_BANDS * sizeof(dspi_biquad_f32)];
    int rc = dspi_eq_download_biquads(e, channel, 1, rowbuf);
    if (rc) return rc;
    if (e->desc.arith == DSPI_ARITH_Q28)
        dspi_compute_coefficients_q28(p, &((dspi_biquad_q28 *)rowbuf)[p->band], sample_rate);
    else
        dspi_compute_coefficients_f32(p, &((dspi_biquad_f32 *)rowbuf)[p->band], sample_rate);
    return dspi_eq_upload_biquads(e, channel, 1, rowbuf);
}

static int make_tmap(dspi_eq *e, void *d_samples, uint32_t T, uint32_t ld, uint32_t n_rows, CUtensorMap *out)
{
    const cuuint64_t gdim[2] = { T, n_rows };
    const cuuint64_t gstride[1] = { (cuuint64_t)ld * 4 };
    const cuuint32_t box[2] = { 32, e->rows };
    const cuuint32_t estr[2] = { 1, 1 };
    const CUtensorMapDataType dt = e->desc.arith == DSPI_ARITH_Q28 ? CU_TENSOR_MAP_DATA_TYPE_INT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUresult r = encode_fn()(out, dt, 2, d_samples, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(DSPI_ECUDA, "cuTensorMapEncodeTiled failed (%d) for T=%u ld=%u rows=%u", (int)r, T, ld, n_rows);
    return DSPI_OK;
}

// Pick the K1 variant for the engine's current coefficient set: sample the per-channel topology words
// the pack kernel wrote, and if one vector dominates (and it is not the all-biquad vector the
// ahead-of-time kernel already runs straight-line) compile K1 for it.  Only speed depends on this.
static int refresh_kernel_choice(dspi_eq *e)
{
    e->sig_dirty = false;
    e->jit = nullptr;
    if (e->desc.arith == DSPI_ARITH_Q28) { snprintf(e->kinfo, sizeof(e->kinfo), "aot q28 cascade (K2)"); return DSPI_OK; }
    // the stage geometry closes every report, so that it shows which one ran
    const char *geo = e->cpl == 1 ? "tile 32 rows x 64 samples, 1 ch/lane" : "tile 64 rows x 32 samples, 2 ch/lane";
    const uint32_t C = e->desc.n_channels, nb = e->desc.n_bands;
    const int nbt = nb <= 10 ? 10 : 12;
    const uint32_t step = C > 2048 ? C / 2048 : 1;
    const uint32_t cnt = (C + step - 1) / step;
    std::vector<uint64_t> w(cnt);
    CU_OK(cudaMemcpy2DAsync(w.data(), 8, e->d_modes_eff ? e->d_modes_eff : e->d_modes, (size_t)step * 8, 8, cnt, cudaMemcpyDeviceToHost, e->stream));
    CU_OK(cudaStreamSynchronize(e->stream));
    const uint64_t mask = (1ull << (4 * nb)) - 1;                // nb <= 12
    for (auto &x : w) x &= mask;
    std::vector<uint64_t> sorted(w);
    std::sort(sorted.begin(), sorted.end());
    uint64_t best = 0;
    uint32_t best_n = 0;
    for (uint32_t i = 0; i < cnt;) {
        uint32_t j = i;
        while (j < cnt && sorted[j] == sorted[i]) j++;
        if (j - i > best_n) { best_n = j - i; best = sorted[i]; }
        i = j;
    }
    uint64_t tdf2 = 0;
    for (int b = 0; b < nbt; b++) tdf2 |= (uint64_t)dspi::kModeTdf2 << (4 * b);
    const unsigned pct = (unsigned)(100ull * best_n / cnt);
    if (best == tdf2 && (int)nb == nbt) {
        snprintf(e->kinfo, sizeof(e->kinfo), "aot straight-line biquad (%u%% of sampled channels are all-TDF2); %s", pct, geo);
        return DSPI_OK;
    }
    bool force = false;
    const bool on = dspi::jit::enabled_by_env(&force);
    const char *why = nullptr;
    if (!on) why = "DSPI_JIT=0";
    else if (best == 0) why = "all bands bypassed";
    else if (2 * best_n < cnt) why = "no dominant topology vector";
    else if (!force && C < 1024) why = "engine below 1024 channels (DSPI_JIT=force overrides)";
    if (why) {
        snprintf(e->kinfo, sizeof(e->kinfo), "aot generic column path (%s); %s", why, geo);
        return DSPI_OK;
    }
    char msg[256] = "";
    e->jit = dspi::jit::acquire(best, e->desc.arith == DSPI_ARITH_F32_FUSED, nbt, e->cpl, e->desc.device, msg, sizeof(msg));
    if (e->jit) snprintf(e->kinfo, sizeof(e->kinfo), "jit sig=0x%llx nb=%d (%u%% of sampled channels); %s", (unsigned long long)best, nbt, pct, geo);
    else snprintf(e->kinfo, sizeof(e->kinfo), "aot generic column path (jit unavailable: %.200s); %s", msg, geo);
    return DSPI_OK;
}

// launch over groups [g0, g0 + ng) of the engine on `stream`; d_samples points at row row_lo of group g0 (the first row
// of the launch) and holds `n_rows` valid rows
static int launch_eq(dspi_eq *e, void *d_samples, uint32_t T, uint32_t ld, uint32_t g0, uint32_t ng, uint32_t n_rows, cudaStream_t stream,
                     uint32_t row_lo = 0)
{
    dspi::EqLaunch a;
    memset(&a, 0, sizeof(a));
    const bool tma_ok = (ld % 4 == 0) && (((uintptr_t)d_samples & 15) == 0);
    if (tma_ok) {
        if (e->tm_ptr != d_samples || e->tm_T != T || e->tm_ld != ld || e->tm_rows != n_rows) {
            int rc = make_tmap(e, d_samples, T, ld, n_rows, &e->tmap);
            if (rc) return rc;
            e->tm_ptr = d_samples; e->tm_T = T; e->tm_ld = ld; e->tm_rows = n_rows;
        }
        a.tmap = e->tmap;
    }
    const bool q28 = e->desc.arith == DSPI_ARITH_Q28;
    a.samples = d_samples;
    a.ld = ld;
    a.coef = q28 ? (void *)((int32_t *)e->d_coef + (size_t)g0 * DSPI_MAX_BANDS * 20 * 32)
                 : (void *)((float *)e->d_coef + (size_t)g0 * DSPI_MAX_BANDS * 8 * 32 * e->cpl);
    const uint64_t *modes = e->d_modes_eff ? e->d_modes_eff : e->d_modes;
    a.modes = modes ? modes + (size_t)g0 * e->rows : nullptr;
    a.n_groups = ng;
    a.sched = e->d_sched + 2 * (((size_t)g0 * e->rows + row_lo) / 32);
    a.n_sms = e->n_sms;
    a.n_rows = n_rows;
    a.row_lo = row_lo;
    a.T = T;
    a.n_bands = e->desc.n_bands;
    a.use_tma = tma_ok ? 1u : 0u;
    if (const char *v = getenv("DSPI_DBG")) a.dbg = (uint32_t)atoi(v);
    cudaError_t err;
    if (e->sig_dirty) {
        int rc = refresh_kernel_choice(e);
        if (rc) return rc;
    }
    if (q28) err = dspi::launch_eq_q28(a, stream);
    else if (e->jit && !(a.dbg & 12u)) {
        char msg[200] = "";
        err = dspi::jit::launch(e->jit, a, stream, msg, sizeof(msg));
        if (err != cudaSuccess) return fail(DSPI_ECUDA, "%s", msg);
    } else err = dspi::launch_eq_f32(a, e->desc.arith == DSPI_ARITH_F32_FUSED, e->cpl, stream);
    if (err != cudaSuccess) return fail(DSPI_ECUDA, "EQ kernel launch: %s", cudaGetErrorString(err));
    e->launches++;
    return DSPI_OK;
}

}  // extern "C"

// ---- engine-internal interface (eq_kernels.cuh) ------------------------------------------------
namespace dspi {

// Range calls start on multiples of 64 channels for float engines whatever their group size (32 or 64 rows), so that
// callers' chunk boundaries do not depend on the geometry; Q28 engines keep their 32-channel groups.
static uint32_t range_unit(const dspi_eq *e) { return e->desc.arith == DSPI_ARITH_Q28 ? e->rows : 64u; }

void *eq_aos_mirror(dspi_eq *e) { return e->d_aos; }

static int remask(dspi_eq *e, cudaStream_t s)
{
    if (!e->d_skip) return DSPI_OK;
    if (e->desc.arith == DSPI_ARITH_Q28) {
        CU_OK(launch_skip_q28((int32_t *)e->d_coef, e->d_skip, e->desc.n_channels, s));
        e->launches++;
        return DSPI_OK;
    }
    if (!e->d_modes_eff) {
        CU_OK(cudaMalloc(&e->d_modes_eff, (size_t)e->c_pad * 8));
        CU_OK(cudaMemsetAsync(e->d_modes_eff, 0, (size_t)e->c_pad * 8, s));
    }
    CU_OK(launch_mask_modes(e->d_modes, e->d_skip, e->d_modes_eff, e->desc.n_channels, s));
    e->launches++;
    e->sig_dirty = true;
    return DSPI_OK;
}

int eq_pack_range(dspi_eq *e, uint32_t ch0, uint32_t n, cudaStream_t s, const RoleRange &rr)
{
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    if (e->desc.arith == DSPI_ARITH_Q28)
        CU_OK(launch_pack_q28((const dspi_biquad_q28 *)e->d_aos, ch0, n, (int32_t *)e->d_coef, s, rr));
    else
        CU_OK(launch_pack_f32((const dspi_biquad_f32 *)e->d_aos, ch0, n, (float *)e->d_coef, e->d_modes, e->cpl, s, rr));
    e->launches++;
    e->sig_dirty = true;
    int rc = remask(e, s);
    if (rc) return rc;
    CU_OK(cudaStreamSynchronize(s));
    return DSPI_OK;
}

int eq_unpack_range(dspi_eq *e, uint32_t ch0, uint32_t n, cudaStream_t s, const RoleRange &rr)
{
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    if (e->desc.arith == DSPI_ARITH_Q28)
        CU_OK(launch_unpack_q28((dspi_biquad_q28 *)e->d_aos, ch0, n, (const int32_t *)e->d_coef, s, rr));
    else
        CU_OK(launch_unpack_f32((dspi_biquad_f32 *)e->d_aos, ch0, n, (const float *)e->d_coef, e->cpl, s, rr));
    e->launches++;
    return DSPI_OK;
}

int eq_set_skip(dspi_eq *e, const uint8_t *d_skip, cudaStream_t s)
{
    CU_OK(cudaSetDevice(e->desc.device));
    e->d_skip = d_skip;
    int rc = remask(e, s);
    if (rc) return rc;
    CU_OK(cudaStreamSynchronize(s));
    return DSPI_OK;
}

// ---- lane control calls of the chain engines: one instance window's rows, never synchronising --------------------------
bool eq_skip_set(const dspi_eq *e) { return e->d_skip && (e->desc.arith == DSPI_ARITH_Q28 || e->d_modes_eff); }

int eq_remask_rows(dspi_eq *e, uint32_t ch0, uint32_t n, const RoleRange &rr, cudaStream_t s)
{
    if (n == 0 || !e->d_skip) return DSPI_OK;
    if (!eq_skip_set(e)) return fail(DSPI_EINVAL, "skip rows were never set on this engine");
    CU_OK(cudaSetDevice(e->desc.device));
    for (uint32_t r = 0; r < rr.roles; r++) {
        const size_t c = (size_t)ch0 + (size_t)r * rr.stride;
        if (e->desc.arith == DSPI_ARITH_Q28)         // groups of 32 channels; c is a multiple of 32
            CU_OK(launch_skip_q28((int32_t *)e->d_coef + c / 32 * DSPI_MAX_BANDS * 20 * 32, e->d_skip + c, n, s));
        else
            CU_OK(launch_mask_modes(e->d_modes + c, e->d_skip + c, e->d_modes_eff + c, n, s));
        e->launches++;
    }
    e->sig_stale = e->desc.arith != DSPI_ARITH_Q28;
    return DSPI_OK;
}

int eq_pack_rows(dspi_eq *e, uint32_t ch0, uint32_t n, cudaStream_t s, const RoleRange &rr, uint32_t win0, uint32_t win_n)
{
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    if (e->desc.arith == DSPI_ARITH_Q28)
        CU_OK(launch_pack_q28((const dspi_biquad_q28 *)e->d_aos, ch0, n, (int32_t *)e->d_coef, s, rr));
    else
        CU_OK(launch_pack_f32((const dspi_biquad_f32 *)e->d_aos, ch0, n, (float *)e->d_coef, e->d_modes, e->cpl, s, rr));
    e->launches++;
    e->sig_stale = e->desc.arith != DSPI_ARITH_Q28;
    RoleRange w;
    w.roles = rr.roles;
    w.stride = rr.stride;
    return eq_remask_rows(e, win0, win_n, w, s);
}

bool eq_choice_stale(const dspi_eq *e) { return e->sig_stale; }

int eq_refresh_choice(dspi_eq *e)
{
    e->sig_stale = false;
    CU_OK(cudaSetDevice(e->desc.device));
    return refresh_kernel_choice(e);
}

// the device arrays that make up an engine's coefficient + filter state (checkpointing by the chain engines)
void eq_state_sections(dspi_eq *e, std::vector<std::pair<void *, size_t>> &out)
{
    const bool q28 = e->desc.arith == DSPI_ARITH_Q28;
    const size_t coef_bytes = q28 ? (size_t)e->n_groups * DSPI_MAX_BANDS * 20 * 32 * 4 : (size_t)e->c_pad * DSPI_MAX_BANDS * 8 * 4;
    out.push_back({ e->d_coef, coef_bytes });
    if (e->d_modes) out.push_back({ e->d_modes, (size_t)e->c_pad * 8 });
    // the reference-layout mirror too: download / device-side coefficient edits start from it (its coefficients,
    // bypass and topology fields are not recoverable from the packed store alone)
    out.push_back({ e->d_aos, (size_t)e->c_pad * DSPI_MAX_BANDS * e->aos_elem });
}

// after the sections were overwritten: effective topology words and the kernel choice must be re-derived
int eq_state_imported(dspi_eq *e, cudaStream_t s)
{
    e->sig_dirty = true;
    return remask(e, s);
}

int eq_geometry(const dspi_eq *e) { return e->cpl; }

// channels of the packed store (and of the mirror) when laid out for `cpl` channels per lane
static size_t padded_channels(const dspi_eq *e, int cpl)
{
    const size_t rows = 32u * (size_t)cpl;
    return (e->desc.n_channels + rows - 1) / rows * rows;
}

size_t eq_state_bytes(const dspi_eq *e, int cpl)
{
    const size_t c_pad = padded_channels(e, cpl);
    if (e->desc.arith == DSPI_ARITH_Q28) return c_pad / 32 * DSPI_MAX_BANDS * 20 * 32 * 4 + c_pad * DSPI_MAX_BANDS * e->aos_elem;
    return c_pad * DSPI_MAX_BANDS * 8 * 4 + c_pad * 8 + c_pad * DSPI_MAX_BANDS * e->aos_elem;
}

int eq_state_load(dspi_eq *e, const void *src, int cpl, cudaStream_t s)
{
    CU_OK(cudaSetDevice(e->desc.device));
    if (cpl == e->cpl) {
        std::vector<std::pair<void *, size_t>> v;
        eq_state_sections(e, v);
        const char *p = (const char *)src;
        for (auto &sec : v) {
            CU_OK(cudaMemcpyAsync(sec.first, p, sec.second, cudaMemcpyHostToDevice, s));
            p += sec.second;
        }
        CU_OK(cudaStreamSynchronize(s));
        return DSPI_OK;
    }
    if (e->desc.arith == DSPI_ARITH_Q28 || (cpl != 1 && cpl != 2)) return fail(DSPI_EINVAL, "state saved for %d channels per lane", cpl);
    // Another geometry: the mirror's bytes do not depend on it.  Take the saved mirror, bring its state fields up to
    // date from the saved packed store (in the layout it was saved in), then rebuild this engine's packed store and
    // topology words from it, exactly as an upload would.
    const uint32_t n = e->desc.n_channels;
    const size_t c_pad = padded_channels(e, cpl);
    const size_t coef_bytes = c_pad * DSPI_MAX_BANDS * 8 * 4;
    const char *mirror = (const char *)src + coef_bytes + c_pad * 8;
    CU_OK(cudaMemcpyAsync(e->d_aos, mirror, (size_t)n * DSPI_MAX_BANDS * e->aos_elem, cudaMemcpyHostToDevice, s));
    float *saved = nullptr;
    CU_OK(cudaMalloc((void **)&saved, coef_bytes));
    cudaError_t err = cudaMemcpyAsync(saved, src, coef_bytes, cudaMemcpyHostToDevice, s);
    if (err == cudaSuccess) err = launch_unpack_f32((dspi_biquad_f32 *)e->d_aos, 0, n, saved, cpl, s);
    if (err == cudaSuccess) err = launch_pack_f32((const dspi_biquad_f32 *)e->d_aos, 0, n, (float *)e->d_coef, e->d_modes, e->cpl, s);
    if (err == cudaSuccess) err = cudaStreamSynchronize(s);
    cudaFree(saved);
    if (err != cudaSuccess) return fail(DSPI_ECUDA, "state conversion from %d to %d channels per lane: %s", cpl, e->cpl, cudaGetErrorString(err));
    e->launches += 2;
    return DSPI_OK;
}

int eq_process_on(dspi_eq *e, void *d_samples, uint32_t T, uint32_t ld, cudaStream_t s)
{
    if (T == 0) return DSPI_OK;
    return launch_eq(e, d_samples, T, ld, 0, e->n_groups, e->desc.n_channels, s);
}

// channels [ch0, ch0 + n) on a stream of the caller's choosing (launches over disjoint channel ranges may run concurrently:
// they touch disjoint parts of the coefficient / state store).  ch0 is a multiple of 32; in the 64-row geometry the range
// may begin half-way into a group, whose other rows K1 then leaves alone.
int eq_process_range_on(dspi_eq *e, void *d_rows, uint32_t T, uint32_t ld, uint32_t ch0, uint32_t n, cudaStream_t s)
{
    if (T == 0 || n == 0) return DSPI_OK;
    if (ch0 % 32u) return fail(DSPI_EINVAL, "first channel %u is not a multiple of 32", ch0);
    CU_OK(cudaSetDevice(e->desc.device));
    const uint32_t row_lo = ch0 % e->rows;
    return launch_eq(e, d_rows, T, ld, ch0 / e->rows, (row_lo + n + e->rows - 1) / e->rows, n, s, row_lo);
}

}  // namespace dspi

extern "C" {

int dspi_eq_kernel_info(dspi_eq *e, char *buf, size_t cap)
{
    if (!e || !buf || cap == 0) return fail(DSPI_EINVAL, "null argument");
    CU_OK(cudaSetDevice(e->desc.device));
    if (e->sig_dirty) {
        int rc = refresh_kernel_choice(e);
        if (rc) return rc;
    }
    snprintf(buf, cap, "%s", e->kinfo);
    return DSPI_OK;
}

int dspi_eq_process_device(dspi_eq *e, void *d_samples, uint32_t T, uint32_t ld)
{
    if (!e || !d_samples) return fail(DSPI_EINVAL, "null argument");
    if (T == 0) return DSPI_OK;
    if (ld < T) return fail(DSPI_EINVAL, "row stride %u < T %u", ld, T);
    CU_OK(cudaSetDevice(e->desc.device));
    return launch_eq(e, d_samples, T, ld, 0, e->n_groups, e->desc.n_channels, e->stream);
}

int dspi_eq_process_device_range(dspi_eq *e, void *d_rows, uint32_t T, uint32_t ld, uint32_t ch0, uint32_t n)
{
    if (!e || !d_rows) return fail(DSPI_EINVAL, "null argument");
    if (T == 0 || n == 0) return DSPI_OK;
    if (ld < T) return fail(DSPI_EINVAL, "row stride %u < T %u", ld, T);
    if ((uint64_t)ch0 + n > e->desc.n_channels) return fail(DSPI_ERANGE, "channels [%u, %u) outside engine of %u", ch0, ch0 + n, e->desc.n_channels);
    if (ch0 % dspi::range_unit(e)) return fail(DSPI_EINVAL, "first channel %u is not a multiple of %u", ch0, dspi::range_unit(e));
    CU_OK(cudaSetDevice(e->desc.device));
    return launch_eq(e, d_rows, T, ld, ch0 / e->rows, (n + e->rows - 1) / e->rows, n, e->stream);
}

}  // extern "C"

// The staged pipeline behind dspi_eq_process_host and the multi-device group (eqx.cu): rows [c0, c1) x T are contiguous in
// the caller's [C][T] array, so every copy is one large 1-D transfer at full link rate; copy-in, kernel and copy-out of
// consecutive chunks overlap, which also keeps BOTH directions of the link busy.  `remote` may be pinned host memory (PCIe)
// or memory of a peer GPU with peer access enabled (NVLink): cudaMemcpyDefault resolves either.
// A cascade kernel takes as long as its rows are long however few rows it gets (parallel over channels, serial over time:
// about a millisecond for 6144 frames) while a chunk fills only a few SMs, so every staging buffer has a kernel stream of its own and the
// kernels of consecutive chunks run side by side; one kernel stream would cap the pipeline at one chunk per kernel time, and
// the ring is deep enough to cover copy + kernel + copy (kHostBufs).  Channels are independent, so chunk order and size change
// no bit.  enqueue returns without waiting.
namespace dspi {
int eq_process_remote_enqueue(dspi_eq *e, void *remote, uint32_t T, uint32_t ch0, uint32_t n_ch)
{
    if (T == 0 || n_ch == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    const uint32_t ld = (T + 3) & ~3u;                                      // device rows padded for TMA
    // chunk bytes: from a peer GPU over NVLink a chunk should take about (kernel time) / (kHostBufs - 3) to copy: 128 MiB.  Over PCIe
    // 48 MiB chunks are used (smaller copies cost link efficiency faster than they shorten the ends of the pipeline).
    // DSPI_HOST_CHUNK_MB overrides both.
    static const size_t chunk_mb_env = [] { const char *v = getenv("DSPI_HOST_CHUNK_MB"); const long n = v ? atol(v) : 0; return (size_t)(n >= 1 && n <= 1024 ? n : 0); }();
    cudaPointerAttributes pa;
    const bool on_device = cudaPointerGetAttributes(&pa, remote) == cudaSuccess && pa.type == cudaMemoryTypeDevice;
    cudaGetLastError();
    const size_t chunk_mb = chunk_mb_env ? chunk_mb_env : (on_device ? 128 : 48);
    uint32_t cc = (uint32_t)((chunk_mb << 20) / ((size_t)ld * 4));
    cc = cc / e->rows * e->rows;
    if (cc < e->rows) cc = e->rows;
    if (cc > e->c_pad) cc = e->c_pad;
    const size_t need = (size_t)cc * ld * 4;
    if (need > e->stage_bytes) {
        CU_OK(cudaStreamSynchronize(e->s_d2h));
        for (int i = 0; i < kHostBufs; i++) {
            if (e->d_stage[i]) { cudaFree(e->d_stage[i]); e->d_stage[i] = nullptr; }
        }
        e->stage_bytes = 0;
        for (int i = 0; i < kHostBufs; i++) {
            if (cudaMalloc(&e->d_stage[i], need) != cudaSuccess) { cudaGetLastError(); return fail(DSPI_ENOMEM, "staging buffer of %zu bytes", need); }
        }
        e->stage_bytes = need;
    }
    const uint32_t nchunks = (n_ch + cc - 1) / cc;
    char *base = (char *)remote;
    CU_OK(cudaEventRecord(e->ev_begin, e->stream));                         // uploads / parameter changes queued on the engine stream come first
    for (uint32_t k = 0; k < nchunks; k++) {
        const int b = k % kHostBufs;
        const uint32_t c0 = k * cc, n = (n_ch - c0 < cc) ? (n_ch - c0) : cc;
        char *hp = base + (size_t)c0 * T * 4;
        CU_OK(cudaStreamWaitEvent(e->s_h2d, e->ev_out[b], 0));                                      // buffer drained (also by an earlier call)
        if (ld == T) CU_OK(cudaMemcpyAsync(e->d_stage[b], hp, (size_t)n * T * 4, cudaMemcpyDefault, e->s_h2d));
        else CU_OK(cudaMemcpy2DAsync(e->d_stage[b], (size_t)ld * 4, hp, (size_t)T * 4, (size_t)T * 4, n, cudaMemcpyDefault, e->s_h2d));
        CU_OK(cudaEventRecord(e->ev_in[b], e->s_h2d));
        if (k < (uint32_t)kHostBufs) CU_OK(cudaStreamWaitEvent(e->s_k[b], e->ev_begin, 0));
        CU_OK(cudaStreamWaitEvent(e->s_k[b], e->ev_in[b], 0));
        int rc = launch_eq(e, e->d_stage[b], T, ld, (ch0 + c0) / e->rows, (n + e->rows - 1) / e->rows, n, e->s_k[b]);
        if (rc) return rc;
        CU_OK(cudaEventRecord(e->ev_done[b], e->s_k[b]));
        CU_OK(cudaStreamWaitEvent(e->s_d2h, e->ev_done[b], 0));
        if (ld == T) CU_OK(cudaMemcpyAsync(hp, e->d_stage[b], (size_t)n * T * 4, cudaMemcpyDefault, e->s_d2h));
        else CU_OK(cudaMemcpy2DAsync(hp, (size_t)T * 4, e->d_stage[b], (size_t)ld * 4, (size_t)T * 4, n, cudaMemcpyDefault, e->s_d2h));
        CU_OK(cudaEventRecord(e->ev_out[b], e->s_d2h));
    }
    for (uint32_t b = 0; b < (uint32_t)kHostBufs && b < nchunks; b++)       // later work on the engine stream sees the new filter state
        CU_OK(cudaStreamWaitEvent(e->stream, e->ev_done[b], 0));
    return DSPI_OK;
}

int eq_process_remote_wait(dspi_eq *e)
{
    CU_OK(cudaSetDevice(e->desc.device));
    CU_OK(cudaStreamSynchronize(e->s_d2h));
    return DSPI_OK;
}
}  // namespace dspi

extern "C" {

int dspi_eq_process_host(dspi_eq *e, void *h_samples, uint32_t T)
{
    if (!e || !h_samples) return fail(DSPI_EINVAL, "null argument");
    if (T == 0) return DSPI_OK;
    int rc = dspi::eq_process_remote_enqueue(e, h_samples, T, 0, e->desc.n_channels);
    if (rc) return rc;
    return dspi::eq_process_remote_wait(e);
}

int dspi_eq_sync(dspi_eq *e)
{
    if (!e) return fail(DSPI_EINVAL, "null argument");
    CU_OK(cudaSetDevice(e->desc.device));
    CU_OK(cudaStreamSynchronize(e->stream));
    return DSPI_OK;
}

void *dspi_eq_stream(dspi_eq *e) { return e ? (void *)e->stream : nullptr; }

// Frequency response of channels [ch0, ch0 + n) from the mirror (response.cu), on the engine stream.  out: device memory
// [n][n_freqs] float2 (host = false), or host memory filled chunk by chunk through the staging buffer (host = true).
static int eq_response(dspi_eq *e, uint32_t ch0, uint32_t n, const float *freqs, uint32_t n_freqs, float fs, float *out, bool host)
{
    const char *why = "";
    int rc = dspi::response_check_args(freqs, n_freqs, fs, out, &why);
    if (rc) return fail(rc, "%s", why);
    if (!e) return fail(DSPI_EINVAL, "null argument");
    if ((uint64_t)ch0 + n > e->desc.n_channels) return fail(DSPI_ERANGE, "channels [%u, %llu) outside engine of %u", ch0, (unsigned long long)ch0 + n, e->desc.n_channels);
    if (n == 0) return DSPI_OK;
    CU_OK(cudaSetDevice(e->desc.device));
    CU_OK(e->resp.upload(freqs, n_freqs, e->stream, &e->launches));
    const bool q28 = e->desc.arith == DSPI_ARITH_Q28;
    if (!host) {
        CU_OK(dspi::launch_eq_response(q28, e->d_aos, ch0, n, e->desc.n_bands, e->resp.d_freq, n_freqs, fs, out, e->stream));
        e->launches++;
        return DSPI_OK;
    }
    const size_t row_bytes = (size_t)n_freqs * 2 * sizeof(float);
    uint32_t rows = 0;
    CU_OK(e->resp.stage(row_bytes, n, e->stream, &rows));
    for (uint32_t c = 0; c < n; c += rows) {
        const uint32_t m = n - c < rows ? n - c : rows;
        CU_OK(dspi::launch_eq_response(q28, e->d_aos, ch0 + c, m, e->desc.n_bands, e->resp.d_freq, n_freqs, fs, e->resp.d_stage, e->stream));
        e->launches++;
        CU_OK(cudaMemcpyAsync((char *)out + (size_t)c * row_bytes, e->resp.d_stage, (size_t)m * row_bytes, cudaMemcpyDeviceToHost, e->stream));
        CU_OK(cudaStreamSynchronize(e->stream));
    }
    return DSPI_OK;
}

int dspi_eq_response_host(dspi_eq *e, uint32_t ch0, uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *out)
{
    return eq_response(e, ch0, n, freqs_hz, n_freqs, sample_rate, out, true);
}

int dspi_eq_response_device(dspi_eq *e, uint32_t ch0, uint32_t n, const float *freqs_hz, uint32_t n_freqs, float sample_rate, float *d_out)
{
    return eq_response(e, ch0, n, freqs_hz, n_freqs, sample_rate, d_out, false);
}
uint64_t dspi_eq_launch_count(dspi_eq *e) { return e ? e->launches : 0; }

}  // extern "C"
