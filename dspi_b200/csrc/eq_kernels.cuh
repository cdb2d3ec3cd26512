// eq_kernels.cuh — declarations shared by the EQ kernels and the engine (C-ABI) code.
#pragma once
#include <utility>
#include <vector>

#include "eq_modes.cuh"
#include "dspi_b200.h"

namespace dspi {

static_assert(kMaxBands == DSPI_MAX_BANDS, "band stride");

struct EqLaunch {
    CUtensorMap tmap;      // [C rows][T] tiled map, box {32, rows-per-warp}, SWIZZLE_128B
    void *samples;         // device base (fallback path)
    uint32_t ld;           // row stride in elements
    void *coef;            // packed coefficient/state store
    const uint64_t *modes; // f32 only
    uint32_t n_groups;     // groups of (32 * channels-per-lane) channels
    uint32_t n_rows;       // valid channel rows in `samples`
    uint32_t row_lo;       // rows of the first group that lie before `samples` (K1 range launches half-way into a 64-row group; else 0)
    uint32_t T;
    uint32_t n_bands;
    uint32_t use_tma;
    uint32_t dbg;          // diagnostics only (env DSPI_DBG): 1 = skip arithmetic, 2 = skip HBM traffic, 4 = force column path, 8 = dynamic time-slice schedule
    uint32_t *sched;       // K1 dynamic scheduler words: [0] item counter, [1 + g] slices completed by group g (or nullptr)
    int n_sms;             // SM count of the device
};

// cudaFuncSetAttribute is per device: remembers, per kernel (one flag word per call site), which devices are done
struct PerDeviceOnce {
    unsigned long long done = 0;
    bool needs(int *device_out)
    {
        int dev = 0;
        cudaGetDevice(&dev);
        *device_out = dev;
        return dev < 0 || dev >= 64 || !((done >> dev) & 1ull);
    }
    void mark(int dev) { if (dev >= 0 && dev < 64) done |= 1ull << dev; }
};

// per-thread message buffer behind dspi_last_error() (engine.cu)
char *error_buffer(size_t *cap);

// One launch over the same channel range of several roles: role r covers channels [ch0 + r * stride, ch0 + r * stride + n).
// The chain engines keep role-major rows (channel = role * N_pad + instance), so an instance range is one such set.
// reject[i] != 0 (device memory, [n], or nullptr) leaves channel i of every role untouched.  fs (device memory, [n], or
// nullptr) gives channel i of every role its own sample rate in the coefficient kernels, in place of their scalar one.
// inst (device memory, [n], or nullptr) turns the range into a list: channel i of role r is ch0 + r * stride + inst[i]
// (pack / unpack and coefficient kernels; the chain engines' copy and edit of scattered instances).  band_mask (device
// memory, [roles][n], or nullptr): the coefficient kernels compute band b of channel i of role r only where bit b of
// band_mask[r * n + i] is set, and leave the other bands and their recipes alone.  The default is one plain range.
struct RoleRange {
    uint32_t roles = 1, stride = 0;
    const int32_t *reject = nullptr;
    const float *fs = nullptr;
    const uint32_t *inst = nullptr;
    const uint16_t *band_mask = nullptr;
};

// K1 — float cascade.  cpl: channels per lane (1, or 2 held in a register pair)
cudaError_t launch_eq_f32(const EqLaunch &a, bool fused, int cpl, cudaStream_t stream);
cudaError_t launch_pack_f32(const dspi_biquad_f32 *aos, uint32_t ch0, uint32_t n, float *coef, uint64_t *modes, int cpl, cudaStream_t stream,
                            const RoleRange &rr = RoleRange());
cudaError_t launch_unpack_f32(dspi_biquad_f32 *aos, uint32_t ch0, uint32_t n, const float *coef, int cpl, cudaStream_t stream,
                              const RoleRange &rr = RoleRange());

// K2 — Q28 cascade (1 channel per lane)
cudaError_t launch_eq_q28(const EqLaunch &a, cudaStream_t stream);
cudaError_t launch_pack_q28(const dspi_biquad_q28 *aos, uint32_t ch0, uint32_t n, int32_t *coef, cudaStream_t stream, const RoleRange &rr = RoleRange());
cudaError_t launch_unpack_q28(dspi_biquad_q28 *aos, uint32_t ch0, uint32_t n, const int32_t *coef, cudaStream_t stream,
                              const RoleRange &rr = RoleRange());

}  // namespace dspi

// ---- engine-internal interface (engine.cu), used by the chain engines which run their EQ rows
// through K1: same packed store, same kernels, on a stream of the caller's choosing -------------
struct dspi_eq;
namespace dspi {
void *eq_aos_mirror(dspi_eq *e);                                          // device Biquad[c_pad][12], reference layout
int eq_pack_range(dspi_eq *e, uint32_t ch0, uint32_t n, cudaStream_t s, const RoleRange &rr = RoleRange());   // mirror -> packed store (coefficients and state), synchronous
int eq_unpack_range(dspi_eq *e, uint32_t ch0, uint32_t n, cudaStream_t s, const RoleRange &rr = RoleRange()); // packed store -> mirror (state), asynchronous on s
// rows with skip[ch] != 0 keep their whole cascade frozen (all bands treated as bypassed, state untouched):
// usb_audio.c:721-728 (bypass_master_eq), :879-884 (muted / disabled outputs).  `d_skip` is [n_channels]
// device memory owned by the caller; call again after changing it.
int eq_set_skip(dspi_eq *e, const uint8_t *d_skip, cudaStream_t s);
// Lane control calls of the chain engines.  Other lanes' K1 / K2 launches may be in flight, so these touch the rows of one
// instance window only, row ch0 + r * rr.stride + i for r < rr.roles and i < n, and never synchronise:
//   eq_pack_rows    eq_pack_range's pack (any RoleRange), then the skip remask of the window rows [win0, win0 + win_n) per role
//   eq_remask_rows  the skip rows of the window into the effective modes (float) or the packed store (Q28); refused until
//                   eq_set_skip ran once (eq_skip_set), since the first remask covers every row
// Neither re-selects the K1 kernel: that reads every row's modes, synchronises and may load a module.  They mark the choice
// stale instead (eq_choice_stale), and the chain engine's next engine-level call re-selects it (eq_refresh_choice) once
// the lanes' work has finished.  Only speed depends on the choice: every K1 warp checks its own rows' topology.
bool eq_skip_set(const dspi_eq *e);
int eq_pack_rows(dspi_eq *e, uint32_t ch0, uint32_t n, cudaStream_t s, const RoleRange &rr, uint32_t win0, uint32_t win_n);
int eq_remask_rows(dspi_eq *e, uint32_t ch0, uint32_t n, const RoleRange &rr, cudaStream_t s);
bool eq_choice_stale(const dspi_eq *e);
int eq_refresh_choice(dspi_eq *e);
int eq_process_on(dspi_eq *e, void *d_samples, uint32_t T, uint32_t ld, cudaStream_t s);
int eq_process_range_on(dspi_eq *e, void *d_rows, uint32_t T, uint32_t ld, uint32_t ch0, uint32_t n, cudaStream_t s);
// staged copy-in / kernel / copy-out pipeline of channels [ch0, ch0 + n_ch) against `remote` rows [n_ch][T] (pinned host
// memory or a peer GPU's memory); enqueue does not block, wait returns when the results are back in `remote`
int eq_process_remote_enqueue(dspi_eq *e, void *remote, uint32_t T, uint32_t ch0, uint32_t n_ch);
int eq_process_remote_wait(dspi_eq *e);
void eq_state_sections(dspi_eq *e, std::vector<std::pair<void *, size_t>> &out);   // coefficient + state store (and topology words)
int eq_state_imported(dspi_eq *e, cudaStream_t s);
// checkpoints across K1 geometries: the packed store is laid out by channels per lane (1 or 2, DSPI_F32_CPL at create time;
// always 1 for Q28).  eq_state_bytes: size of eq_state_sections() for this engine's shape laid out for `cpl`.  eq_state_load:
// writes sections saved from an engine of the same shape laid out for `cpl` (host memory, in section order), converting them
// to this engine's layout when `cpl` differs; synchronous.
int eq_geometry(const dspi_eq *e);
size_t eq_state_bytes(const dspi_eq *e, int cpl);
int eq_state_load(dspi_eq *e, const void *src, int cpl, cudaStream_t s);
// coeff.cu: dsp_compute_coefficients() for channels [ch0, ch0 + n) of a mirror, recipes [n][12] on the device (clamped in place);
// with a RoleRange, recipes [roles][n][12]
cudaError_t launch_coeffs(bool q28, dspi_eq_param *d_recipes, void *d_aos, uint32_t ch0, uint32_t n, float fs, cudaStream_t stream,
                          const RoleRange &rr = RoleRange());
cudaError_t launch_skip_q28(int32_t *coef, const uint8_t *skip, uint32_t n, cudaStream_t stream);
cudaError_t launch_mask_modes(const uint64_t *raw, const uint8_t *skip, uint64_t *eff, uint32_t n, cudaStream_t stream);
// response.cu: frequency response of channels [ch0, ch0 + n) of a mirror (bands b < nb) at d_freq[nf] -> d_out [n][nf] float2
cudaError_t launch_eq_response(bool q28, const void *aos, uint32_t ch0, uint32_t n, uint32_t nb, const float *d_freq, uint32_t nf, float fs,
                               void *d_out, cudaStream_t stream);
}  // namespace dspi
