// bulk_ingest.cuh — parameter ingest on the device, from the wire packet (SURVEY.md §8 f-1): bulk_params_apply() and the
// main-loop work that follows it, for many instances of a chain engine at once, shared by chain_f32.cu and chain_q28.cu.
//
// Reference: bulk_params_apply() bulk_params.c:178-377 (validation :179-203, db_to_linear :49-56), dsp_update_delay_samples()
// dsp_pipeline.c:216-239, the pending-flag handlers main.c:868-900, audio_set_volume() usb_audio.c:410-440.
//
// bulk_ingest_kernel: one warp per instance, kWarps instances per CTA.  Lane 0 brings the 2896-byte packet into shared memory
// with one 1-D bulk copy on the warp's own mbarrier; every lane validates the header (the firmware returns before its first
// write, so a rejected packet writes nothing but its result code); then the lanes share the work:
//   lanes [0, 2 O)        crosspoint gains            lanes [2 O, 3 O)   output gains, flags, delay samples, skip rows
//   lanes 3 O, 3 O + 1    preamp L / R                lane 3 O + 2       master volume
//   lane 0 crossfeed, lane 1 leveller, lane 2 host volume + the loudness row it selects, then lane 0 the output gains
//   all lanes             the 12 x roles recipes, 16 bytes each, into the role-major recipe buffer [role][n][12]
// The recipes then go through the coefficient kernels of coeff.cu, one launch per sub-engine over all its roles (RoleRange).
//
// The way back (REQ_GET_ALL_PARAMS, bulk_params_collect() bulk_params.c:62-172): every instance has a Record, the body of the
// packet bulk_params_collect() would return for it.  The ingest warp rewrites its shared-memory copy of an accepted packet
// into that body (record_body) and sends it out with one bulk store; record_recipes_kernel then replaces the eq section by the
// recipes as the coefficient kernels left them (clamps written back, dsp_pipeline.c:78-81); the dynamics kernels edit their
// fields (record_dynamics).  bulk_collect_kernel, one warp per instance again, brings the record in with a bulk copy, stamps
// the constant header and pin count, and sends it to the staging buffer with a bulk store.
// The engine-specific stores (float or Q28 / Q15) are the engine's ParamStores, the same functions its dynamics kernel uses.
//
// A sample-rate switch (perform_rate_change(), main.c:132-171) starts from the record too: rate_kernel, one warp per
// instance, re-derives the rate-dependent rows of a current instance at its own rate and stages its recipes, and the
// ingest path's tail (recalculate_filters) recomputes the filters with a per-instance rate array in the RoleRange.
//
// Preset slot images (preset_load() / preset_save(), flash_storage.c:464-760) reuse that machinery.  preset_decode_kernel,
// one warp per instance, brings an image in with a bulk copy, checks magic, slot index and CRC-32 (one lane, four-table
// CRC over the words after the header) and writes a version-6 packet with the image's version gates and master-volume mode
// resolved, or for a rejected image a header the ingest kernel rejects; the packets then take the ingest path above with
// the flash gain conversion.  preset_collect_kernel maps a record to the image dspi_preset_slot_collect writes.
//
// Same arithmetic rules as coeff.cu / dynamics.cuh: every float operation is the reference's, rounded on its own
// (-fmad=false, divisions spelled __fdiv_rn), libm in double rounded once, float -> int32 stores saturate.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <type_traits>
#include <vector>

#include "dspi_common.cuh"
#include "dynamics.cuh"
#include "eq_kernels.cuh"
#include "preset_slot.h"

namespace dspi {

// per-instance and per-output flag rows of the chain engines
enum : uint8_t { F_BYPASS_MASTER = 1, F_LOUD = 2, F_XFEED = 4, F_LEV = 8, F_LOOKAHEAD = 16, F_ANY_DELAY = 32, F_SUB_ON = 64 };
enum : uint8_t { O_ENABLED = 1, O_MUTE = 2, O_PAIR_OFF = 4 };

// the derived flag words, one definition for dspi_chain(q)_set_params on the host and the ingest kernel on the device
__host__ __device__ inline uint8_t chain_flags(bool bypass_master_eq, bool loudness, bool crossfeed, bool leveller, bool lookahead, bool any_delay,
                                               bool sub_enabled)
{
    return (uint8_t)((bypass_master_eq ? F_BYPASS_MASTER : 0) | (loudness ? F_LOUD : 0) | (crossfeed ? F_XFEED : 0) | (leveller ? F_LEV : 0) |
                     (lookahead ? F_LOOKAHEAD : 0) | (any_delay ? F_ANY_DELAY : 0) | (sub_enabled ? F_SUB_ON : 0));
}
// `pair_partner_enabled`: outputs[o ^ 1].enabled; the last output (the sub) has no S/PDIF pair (usb_audio.c:930-933)
__host__ __device__ inline uint8_t output_flags(bool enabled, bool mute, bool has_pair, bool pair_partner_enabled)
{
    return (uint8_t)((enabled ? O_ENABLED : 0) | (mute ? O_MUTE : 0) | ((has_pair && !enabled && !pair_partner_enabled) ? O_PAIR_OFF : 0));
}

namespace bulk {

constexpr int kWarps = 4;                                  // instances per CTA: 4 x 2896 B of packets = 11.3 KB shared memory
constexpr uint32_t kChunk = 1024;                          // instances per staged chunk: 2.8 MB of packets, <= 2.1 MB of recipes
constexpr uint32_t kPacketBytes = sizeof(dspi_wire_bulk_params);
static_assert(kPacketBytes % 16 == 0, "the bulk copy moves multiples of 16 bytes");

#define DSPI_WIRE_OFF(member) ((uint32_t)offsetof(dspi_wire_bulk_params, member))

// The wire-visible configuration of every instance, in device memory for the life of the engine.  Not part of the state blob.
struct Record {
    dspi_wire_bulk_params *packets = nullptr;              // [N_pad] packet body; header and pins are stamped by the collect kernel
    dspi_bulk_host *host = nullptr;                        // [N_pad] the host volume and mute last given
    uint8_t *mark = nullptr;                               // [N_pad] DSPI_BULK_CURRENT / _STALE / _UNSET
};

// bulk_params.c:49-56 — the firmware's own conversion: 4-term Taylor series of exp(), clamped
__device__ inline float db_to_linear_fw(float db)
{
    if (db == 0.0f) return 1.0f;
    if (db < -60.0f) db = -60.0f;
    if (db > 20.0f) db = 20.0f;
    const float x = db * 0.1151292546f;
    const float linear = 1.0f + x + x * x * 0.5f + x * x * x * 0.1666667f + x * x * x * x * 0.0416667f;
    return (linear < 0.0f) ? 0.0f : linear;
}

// flash_storage.c:302-306 — the conversion of preset loads
__device__ inline float db_to_linear_flash(float db)
{
    if (db <= -120.0f) return 0.0f;
    if (db >= 80.0f) db = 80.0f;
    return dyn::pow_f(10.0f, dyn::fdiv(db, 20.0f));
}

// how the ingest kernel turns gains in dB into linear gains: the firmware's bulk_params.c, 10^(dB/20), flash_storage.c
enum GainMode : int { kGainTaylor = 0, kGainExact = 1, kGainFlash = 2 };

// bulk_params.c:179-203
__device__ inline int32_t validate(const unsigned char *w, int platform_id, int n_channels, int n_outputs)
{
    const uint32_t version = w[DSPI_WIRE_OFF(header.format_version)];
    if (version < 2 || version > DSPI_WIRE_FORMAT_VERSION) return -1;
    if (w[DSPI_WIRE_OFF(header.platform_id)] != platform_id) return -2;
    if (w[DSPI_WIRE_OFF(header.num_channels)] != n_channels) return -3;
    if (w[DSPI_WIRE_OFF(header.num_output_channels)] != n_outputs) return -3;
    const uint32_t len = *reinterpret_cast<const uint16_t *>(w + DSPI_WIRE_OFF(header.payload_length));
    const uint32_t v2_size = kPacketBytes - 16 - 16 - 16 - 16;
    if (len < v2_size || len > kPacketBytes) return -4;
    return 0;
}

// An accepted packet -> the body of the packet bulk_params_collect() returns once it is applied, in place in the warp's
// shared-memory copy `w`: flags as 0 / 1, the preamp fields from whichever the version makes valid (:206-215, :351-359),
// channel_delays_ms overwritten by the output delays (:242-244, :261), the leveller defaults below version 4 (:330-346),
// rows past NC channels / NO outputs, control-plane sections and reserved bytes zero.  `master_volume_bits` is the value in
// force after the apply.  Every word has one lane; the two cross-field copies are read before any lane writes.
template <int NC, int NO>
__device__ inline void record_body(unsigned char *w, int lane, uint32_t version, uint32_t master_volume_bits)
{
    static_assert(NC == NO + 2, "outputs are channels CH_OUT_1 = 2 onwards (config.h:310)");
    uint32_t *W = reinterpret_cast<uint32_t *>(w);
    constexpr uint32_t g = DSPI_WIRE_OFF(global) / 4, x = DSPI_WIRE_OFF(crossfeed) / 4, lg = DSPI_WIRE_OFF(legacy) / 4, dl = DSPI_WIRE_OFF(delays) / 4,
                       xp = DSPI_WIRE_OFF(crosspoints) / 4, out = DSPI_WIRE_OFF(outputs) / 4, eq = DSPI_WIRE_OFF(eq) / 4,
                       names = DSPI_WIRE_OFF(channel_names) / 4, lev = DSPI_WIRE_OFF(leveller) / 4, pre = DSPI_WIRE_OFF(preamp) / 4;
    const uint32_t pre0 = version >= 6 ? W[pre] : W[g], pre1 = version >= 6 ? W[pre + 1] : W[g];
    uint32_t delay = 0;
    if (lane < NC) delay = lane >= 2 ? W[out + (lane - 2) * 3 + 2] : W[dl + lane];
    __syncwarp();
    auto flag = [](uint32_t word, int byte) { return ((word >> (8 * byte)) & 0xFFu) ? 1u << (8 * byte) : 0u; };
    if (lane == 0) {
        W[0] = W[1] = W[2] = W[3] = 0;
        W[DSPI_WIRE_OFF(pins) / 4] = W[DSPI_WIRE_OFF(pins) / 4 + 1] = 0;
    } else if (lane == 1) {
        W[g] = pre0;
        W[g + 1] = flag(W[g + 1], 0) | flag(W[g + 1], 1);
    } else if (lane == 2) {
        W[x] = flag(W[x], 0) | (W[x] & 0xFF00u) | flag(W[x], 2);
        W[x + 3] = 0;
    } else if (lane == 3) {
        W[lg + 3] = flag(W[lg + 3], 0) | flag(W[lg + 3], 1) | flag(W[lg + 3], 2);
    } else if (lane == 4) {
        if (version >= 4) {
            W[lev] = flag(W[lev], 0) | (W[lev] & 0xFF00u) | flag(W[lev], 2);
        } else {
            W[lev] = 1u << 16;
            W[lev + 1] = __float_as_uint(50.0f);
            W[lev + 2] = __float_as_uint(15.0f);
            W[lev + 3] = __float_as_uint(-96.0f);
        }
    } else if (lane == 5) {
        W[pre] = pre0;
        W[pre + 1] = pre1;
        W[pre + 2] = W[pre + 3] = 0;
    } else if (lane == 6) {
        W[pre + 4] = master_volume_bits;
        W[pre + 5] = W[pre + 6] = W[pre + 7] = 0;
    }
    if (lane < DSPI_WIRE_MAX_CHANNELS) W[dl + lane] = delay;
    if (lane < 2 * DSPI_WIRE_MAX_OUTPUTS) {
        if (lane % DSPI_WIRE_MAX_OUTPUTS < NO) W[xp + lane * 2] &= 0xFFFFu;
        else W[xp + lane * 2] = W[xp + lane * 2 + 1] = 0;
    }
    if (lane < DSPI_WIRE_MAX_OUTPUTS) {
        if (lane < NO) W[out + lane * 3] &= 0xFFFFu;
        else W[out + lane * 3] = W[out + lane * 3 + 1] = W[out + lane * 3 + 2] = 0;
    }
    for (uint32_t r = lane; r < DSPI_WIRE_MAX_CHANNELS * kMaxBands; r += 32) {
        if (r / kMaxBands < NC) W[eq + r * 4] &= 0xFFu;
        else reinterpret_cast<uint4 *>(W + eq)[r] = make_uint4(0, 0, 0, 0);
    }
    for (uint32_t k = names + lane; k < lev; k += 32) W[k] = 0;                                    // channel names and the I2S section: control plane
}

// dsp_update_delay_samples() for output o of O at rate fs, dsp_pipeline.c:216-239: the sub adds SUB_ALIGN_SAMPLES
// (config.h:93-95), the result is clamped to [0, MAX]
template <class S>
__device__ __forceinline__ int32_t delay_samples(float delay_ms, uint32_t o, float fs)
{
    if (o == (uint32_t)S::kOuts - 1) delay_ms = delay_ms + dyn::fdiv(128.0f, fs) * 1000.0f;
    int32_t ds = dyn::f2i_sat(dyn::fdiv(delay_ms * fs, 1000.0f));
    if (ds > S::kMaxDelay) ds = S::kMaxDelay;
    if (ds < 0) ds = 0;
    return ds;
}

// recipe r = role * 12 + band (bulk_params.c:291-300) of instance i of n from the eq section of a packet or record in shared
// memory `w` -> the role-major recipe buffer [role][n][12] of the coefficient kernels
__device__ __forceinline__ void stage_recipe(const unsigned char *w, uint32_t r, uint32_t i, uint32_t n, dspi_eq_param *__restrict__ recipes)
{
    const uint32_t role = r / kMaxBands, b = r % kMaxBands;
    uint4 q = *reinterpret_cast<const uint4 *>(w + DSPI_WIRE_OFF(eq) + r * 16);                     // {type, reserved[3]}, freq, q, gain_db
    q.x = role | b << 8 | (q.x & 0xFFu) << 16;                                                     // {channel, band, type, reserved}
    reinterpret_cast<uint4 *>(recipes)[((size_t)role * n + i) * kMaxBands + b] = q;
}

// filter_recipes[][] of instance i of n, every role and band; all lanes of the warp
template <class S>
__device__ __forceinline__ void stage_recipes(const unsigned char *w, int lane, uint32_t i, uint32_t n, dspi_eq_param *__restrict__ recipes)
{
    for (uint32_t r = lane; r < (uint32_t)S::kRoles * kMaxBands; r += 32) stage_recipe(w, r, i, n, recipes);
}

// ---- lane bodies of the ingest, rate and edit kernels: each reads a packet or record in shared memory `w` ----
__device__ __forceinline__ float wire_f32(const unsigned char *w, uint32_t off) { return *reinterpret_cast<const float *>(w + off); }

// a crosspoint, output or preamp gain in dB -> linear (:206-215, :247-264) under the ingest's gain mode
__device__ __forceinline__ float gain_linear(float db, int gain_mode)
{
    if (gain_mode == kGainFlash) return db_to_linear_flash(db);
    return gain_mode == kGainExact ? dyn::pow_f(10.0f, dyn::fdiv(db, 20.0f)) : db_to_linear_fw(db);
}

// the master volume (:361-374): `db` made finite and clamped to [-128, 0] in place, then always the exact conversion
__device__ __forceinline__ float master_linear(float &db)
{
    if (isnan(db) || isinf(db)) db = 0.0f;
    if (db < -128.0f) db = -128.0f;
    if (db > 0.0f) db = 0.0f;
    return db <= -128.0f ? 0.0f : dyn::pow_f(10.0f, dyn::fdiv(db, 20.0f));
}

// output o's flag word (the S/PDIF pair-off bit reads its partner's enable) and its EQ skip row (usb_audio.c:878-884)
template <class S>
__device__ __forceinline__ void output_flag_rows(const typename S::Dev &d, const unsigned char *w, uint32_t inst, uint32_t o, bool bypass_master)
{
    const uint32_t Np = d.N_pad, off = DSPI_WIRE_OFF(outputs) + o * 12;
    const bool enabled = w[off] != 0, mute = w[off + 1] != 0;
    const bool partner = w[DSPI_WIRE_OFF(outputs) + (o ^ 1u) * 12] != 0;
    d.o_flags[o * Np + inst] = output_flags(enabled, mute, o < (uint32_t)S::kOuts - 1, partner);
    d.skip_o[o * Np + inst] = S::output_eq_frozen(enabled, mute, bypass_master) ? 1 : 0;
}

// output o's delay in samples at fs (dsp_update_delay_samples()); returns it
template <class S>
__device__ __forceinline__ int32_t output_delay_row(const typename S::Dev &d, const unsigned char *w, uint32_t inst, uint32_t o, float fs)
{
    const int32_t ds = delay_samples<S>(wire_f32(w, DSPI_WIRE_OFF(outputs) + o * 12 + 8), o, fs);
    d.o_dly[o * d.N_pad + inst] = ds;
    return ds;
}

// crossfeed_config (:225-230); S::crossfeed clears the filter state (crossfeed.c:110-126)
__device__ __forceinline__ dspi_crossfeed_config crossfeed_config(const unsigned char *w)
{
    dspi_crossfeed_config xf;
    xf.enabled = w[DSPI_WIRE_OFF(crossfeed.enabled)] != 0;
    xf.itd_enabled = w[DSPI_WIRE_OFF(crossfeed.itd_enabled)] != 0;
    xf.preset = w[DSPI_WIRE_OFF(crossfeed.preset)];
    xf.custom_fc = wire_f32(w, DSPI_WIRE_OFF(crossfeed.custom_fc));
    xf.custom_feed_db = wire_f32(w, DSPI_WIRE_OFF(crossfeed.custom_feed_db));
    return xf;
}

// leveller_config (:330-346): the fixed defaults below format version 4 (a record holds the version gates' result)
__device__ __forceinline__ dspi_leveller_config leveller_config(const unsigned char *w, uint32_t version)
{
    dspi_leveller_config lev;
    lev.enabled = version >= 4 ? (w[DSPI_WIRE_OFF(leveller.enabled)] != 0) : 0;
    lev.speed = version >= 4 ? w[DSPI_WIRE_OFF(leveller.speed)] : 0;
    lev.lookahead = version >= 4 ? (w[DSPI_WIRE_OFF(leveller.lookahead)] != 0) : 1;
    lev.amount = version >= 4 ? wire_f32(w, DSPI_WIRE_OFF(leveller.amount)) : 50.0f;
    lev.max_gain_db = version >= 4 ? wire_f32(w, DSPI_WIRE_OFF(leveller.max_gain_db)) : 15.0f;
    lev.gate_threshold_db = version >= 4 ? wire_f32(w, DSPI_WIRE_OFF(leveller.gate_threshold_db)) : -96.0f;
    return lev;
}

// the loudness row audio_set_volume() selected (`row`), at fs
template <class S>
__device__ __forceinline__ void loudness_row(const typename S::Dev &d, const unsigned char *w, uint32_t inst, uint32_t row, float fs)
{
    S::loudness(d, inst, row, wire_f32(w, DSPI_WIRE_OFF(global.loudness_ref_spl)), wire_f32(w, DSPI_WIRE_OFF(global.loudness_intensity_pct)), fs);
}

// the instance's flag word
template <class S>
__device__ __forceinline__ uint8_t instance_flags(const unsigned char *w, const dspi_leveller_config &lev, bool any_delay)
{
    return chain_flags(w[DSPI_WIRE_OFF(global.bypass)] != 0, w[DSPI_WIRE_OFF(global.loudness_enabled)] != 0, w[DSPI_WIRE_OFF(crossfeed.enabled)] != 0,
                       lev.enabled, lev.lookahead, any_delay, w[DSPI_WIRE_OFF(outputs) + (S::kOuts - 1) * 12] != 0);
}

template <class S>
__global__ void __launch_bounds__(kWarps * 32)
bulk_ingest_kernel(typename S::Dev d, Record rec, uint32_t inst0, uint32_t n, const dspi_wire_bulk_params *__restrict__ packets,
                   const dspi_bulk_host *__restrict__ host, int gain_mode, float fs, dspi_eq_param *__restrict__ recipes, int32_t *__restrict__ results)
{
    constexpr int O = S::kOuts, WO = DSPI_WIRE_MAX_OUTPUTS;
    static_assert(3 * O + 3 <= 32, "one lane per gain");
    __shared__ alignas(16) unsigned char pkt_s[kWarps][kPacketBytes];
    __shared__ uint64_t bar_s[kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t i = blockIdx.x * kWarps + warp;
    if (i >= n) return;
    const unsigned char *w = pkt_s[warp];
    uint64_t *bar = &bar_s[warp];
    if (lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar, kPacketBytes);
        bulk_load_1d(pkt_s[warp], packets + i, kPacketBytes, bar);
    }
    __syncwarp();
    mbar_wait(bar, 0);

    const int32_t rc = validate(w, S::kPlatformId, S::kRoles, O);
    if (lane == 0) results[i] = rc;
    if (rc != 0) return;

    const uint32_t inst = inst0 + i, Np = d.N_pad;
    const uint32_t version = w[DSPI_WIRE_OFF(header.format_version)];
    const bool bypass_master = w[DSPI_WIRE_OFF(global.bypass)] != 0;                               // :217

    // ---- one gain per lane (:206-215, :247-264, :351-375) ----
    const bool is_xp = lane < 2 * O, is_out = !is_xp && lane < 3 * O, is_pre = lane == 3 * O || lane == 3 * O + 1, is_mv = lane == 3 * O + 2;
    const uint32_t side = is_xp ? lane / O : (uint32_t)(lane - 3 * O), o = is_xp ? lane % O : (uint32_t)(lane - 2 * O);
    const uint32_t xp_off = DSPI_WIRE_OFF(crosspoints) + (side * WO + o) * 8, out_off = DSPI_WIRE_OFF(outputs) + o * 12;
    float db = 0.0f;
    if (is_xp) db = wire_f32(w, xp_off + 4);
    else if (is_out) db = wire_f32(w, out_off + 4);
    else if (is_pre) db = version >= 6 ? wire_f32(w, DSPI_WIRE_OFF(preamp.preamp_db) + side * 4) : wire_f32(w, DSPI_WIRE_OFF(global.preamp_gain_db));
    else if (is_mv) db = wire_f32(w, DSPI_WIRE_OFF(master_volume.master_volume_db));
    float lin = 0.0f;
    if (is_mv) lin = master_linear(db);
    else if (is_xp || is_out || is_pre) lin = gain_linear(db, gain_mode);
    bool delayed = false;
    if (is_xp) {
        S::crosspoint(d, inst, side, o, w[xp_off] != 0, w[xp_off + 1] != 0, lin);
    } else if (is_out) {
        d.o_glin[o * Np + inst] = lin;
        output_flag_rows<S>(d, w, inst, o, bypass_master);
        delayed = output_delay_row<S>(d, w, inst, o, fs) > 0;
    } else if (is_pre) {
        S::preamp(d, inst, side, lin);
    } else if (is_mv && version >= 6) {
        S::master_volume(d, inst, lin);
    }
    const bool any_delay = __ballot_sync(0xffffffffu, delayed) != 0;                               // dsp_pipeline.c:237

    // ---- the pending-flag handlers of the main loop (main.c:868-900), one generator per lane ----
    const dspi_leveller_config lev = leveller_config(w, version);
    const dspi_bulk_host hv = host[i];
    uint32_t row;
    const int16_t vol_mul = dyn::host_volume(hv.volume_8_8, row);
    if (lane == 0) {
        S::crossfeed(d, inst, crossfeed_config(w), fs);
        d.flags[inst] = instance_flags<S>(w, lev, any_delay);
        d.skip_m[inst] = d.skip_m[Np + inst] = bypass_master ? 1 : 0;                              // usb_audio.c:721-728
    } else if (lane == 1) {
        S::leveller(d, inst, lev, fs);
    } else if (lane == 2) {
        loudness_row<S>(d, w, inst, row, fs);
    }
    __syncwarp();                                          // the gain rows of this instance are written: audio_set_volume() reads them
    if (lane == 0) S::host_volume(d, inst, vol_mul, hv.host_mute != 0);

    // ---- filter_recipes[][] (:291-300), role-major for the coefficient kernels ----
    stage_recipes<S>(w, lane, i, n, recipes);

    // ---- the record: what bulk_params_collect() reads after this apply.  Below version 6 the master volume in force stays ----
    unsigned char *rp = reinterpret_cast<unsigned char *>(rec.packets + inst);
    const float mv_db = __shfl_sync(0xffffffffu, db, 3 * O + 2);                                   // finite, clamped to [-128, 0] (:361-368)
    const uint32_t mv_bits = version >= 6 ? __float_as_uint(mv_db) : *reinterpret_cast<const uint32_t *>(rp + DSPI_WIRE_OFF(master_volume));
    record_body<S::kRoles, O>(pkt_s[warp], lane, version, mv_bits);
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
        bulk_store_1d(rp, pkt_s[warp], kPacketBytes);
        tma_store_commit();
        rec.mark[inst] = DSPI_BULK_CURRENT;
        tma_store_wait_all<0>();
    } else if (lane == 1) {
        rec.host[inst] = hv;
    }
}

// perform_rate_change() (main.c:132-171) of instance inst0 + i at rate fs[i], from its record: one warp per instance.  Lane 0
// brings the record in with a bulk copy; the mark goes to results[i] and only a DSPI_BULK_CURRENT instance goes on (the
// derived records of a stale or unset one did not come from its record).  Output lanes: delay samples; lane 0 crossfeed
// (filter state cleared) and the any_delay bit of the flag word, lane 1 leveller, lane 2 the loudness row of the recorded
// host volume; all lanes: the recipes into the role-major buffer, for the coefficient kernels at fs[i].  No gain, no other
// flag or skip row and no other state is touched.
template <class S>
__global__ void __launch_bounds__(kWarps * 32)
rate_kernel(typename S::Dev d, Record rec, uint32_t inst0, uint32_t n, const float *__restrict__ rates, dspi_eq_param *__restrict__ recipes,
            int32_t *__restrict__ results)
{
    constexpr int O = S::kOuts;
    __shared__ alignas(16) unsigned char pkt_s[kWarps][kPacketBytes];
    __shared__ uint64_t bar_s[kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t i = blockIdx.x * kWarps + warp;
    if (i >= n) return;
    const uint32_t inst = inst0 + i, Np = d.N_pad;
    const unsigned char *w = pkt_s[warp];
    uint64_t *bar = &bar_s[warp];
    if (lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar, kPacketBytes);
        bulk_load_1d(pkt_s[warp], rec.packets + inst, kPacketBytes, bar);
    }
    const uint8_t mark = rec.mark[inst];
    const float fs = rates[i];
    __syncwarp();
    mbar_wait(bar, 0);
    if (lane == 0) results[i] = mark;
    if (mark != DSPI_BULK_CURRENT) return;

    bool delayed = false;
    if (lane < O) delayed = output_delay_row<S>(d, w, inst, lane, fs) > 0;                        // dsp_update_delay_samples()
    const bool any_delay = __ballot_sync(0xffffffffu, delayed) != 0;                               // dsp_pipeline.c:237
    if (lane == 0) {
        S::crossfeed(d, inst, crossfeed_config(w), fs);
        d.flags[inst] = (uint8_t)((d.flags[inst] & ~F_ANY_DELAY) | (any_delay ? F_ANY_DELAY : 0));
    } else if (lane == 1) {
        S::leveller(d, inst, leveller_config(w, DSPI_WIRE_FORMAT_VERSION), fs);                    // the record holds the version gates' result
    } else if (lane == 2) {
        uint32_t row;
        dyn::host_volume(rec.host[inst].volume_8_8, row);
        loudness_row<S>(d, w, inst, row, fs);
    }
    stage_recipes<S>(w, lane, i, n, recipes);
}

// One edit of dspi_chain(q)_edit_bulk_device, and the edit address space: the record, then the host record
constexpr uint32_t kEditSpace = kPacketBytes + (uint32_t)sizeof(dspi_bulk_host);
constexpr uint32_t kEditChunk = 65536;                     // edits per staged chunk: 2 MiB; at most kChunk distinct instances
static_assert(sizeof(dspi_bulk_edit) == 32, "dspi_bulk_edit");

// any byte of [off, off + len) written by an edit; len <= 32, `hit` one bit per byte of the edit space and a spare word
__device__ __forceinline__ bool touched(const uint32_t *hit, uint32_t off, uint32_t len)
{
    const uint64_t bits = (uint64_t)hit[off >> 5] | (uint64_t)hit[(off >> 5) + 1] << 32;
    return ((bits >> (off & 31)) & ((1ull << len) - 1)) != 0;
}

// Sparse edits of current instances (dspi_chain(q)_edit_bulk_device): one warp per distinct instance, segment s of the
// chunk, whose edits are edits[seg_off[s] .. seg_off[s + 1]) in list order.  Lane 0 brings the record in with a bulk copy
// and the host record beside it; the mark goes to marks[s] and only a DSPI_BULK_CURRENT instance goes on.  The edits are
// written over the shared-memory copy in order, each byte noting itself in a bitmap; the copy is normalised by record_body
// (version 6); then the lanes re-derive the rows of touched fields only, with the ingest kernel's lane bodies, and stage
// the touched bands' recipes with a per-(role, segment) band mask for the coefficient kernels.  reject[s] != 0 keeps the
// segment out of the filter recalculation (no touched band, or not current).
template <class S>
__global__ void __launch_bounds__(kWarps * 32)
edit_kernel(typename S::Dev d, Record rec, uint32_t nseg, const dspi_bulk_edit *__restrict__ edits, const uint32_t *__restrict__ seg_off,
            const uint32_t *__restrict__ seg_inst, int gain_mode, float fs, dspi_eq_param *__restrict__ recipes, uint16_t *__restrict__ band_mask,
            int32_t *__restrict__ reject, int32_t *__restrict__ marks)
{
    constexpr int O = S::kOuts, NC = S::kRoles, WO = DSPI_WIRE_MAX_OUTPUTS;
    constexpr uint32_t kHitWords = (kEditSpace + 31) / 32 + 1;
    static_assert(3 * O + 3 <= 32 && NC <= 32, "one lane per gain and per role");
    __shared__ alignas(16) unsigned char pkt_s[kWarps][kPacketBytes + 16];
    __shared__ uint32_t hit_s[kWarps][kHitWords];
    __shared__ uint64_t bar_s[kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t s = blockIdx.x * kWarps + warp;
    if (s >= nseg) return;
    const uint32_t inst = seg_inst[s], Np = d.N_pad;
    unsigned char *w = pkt_s[warp];
    uint32_t *hit = hit_s[warp];
    uint64_t *bar = &bar_s[warp];
    if (lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar, kPacketBytes);
        bulk_load_1d(w, rec.packets + inst, kPacketBytes, bar);
        *reinterpret_cast<dspi_bulk_host *>(w + kPacketBytes) = rec.host[inst];
    }
    for (uint32_t k = lane; k < kHitWords; k += 32) hit[k] = 0;
    const uint8_t mark = rec.mark[inst];
    __syncwarp();
    mbar_wait(bar, 0);
    if (lane == 0) marks[s] = mark;
    if (mark != DSPI_BULK_CURRENT) {
        if (lane < NC) band_mask[lane * nseg + s] = 0;
        if (lane == 0) reject[s] = 1;
        return;
    }

    // ---- the edits in list order: the last write to a byte wins ----
    for (uint32_t k = seg_off[s], end = seg_off[s + 1]; k < end; k++) {
        const uint32_t off = edits[k].offset, len = edits[k].length;
        if ((uint32_t)lane < len) {
            w[off + lane] = edits[k].bytes[lane];
            atomicOr(&hit[(off + lane) >> 5], 1u << ((off + lane) & 31));
        }
        __syncwarp();
    }

    // ---- normalised as the ingest leaves a record (version 6; the master volume made finite and clamped) ----
    float mv_db = wire_f32(w, DSPI_WIRE_OFF(master_volume.master_volume_db));
    const float mv_lin = master_linear(mv_db);
    __syncwarp();
    record_body<NC, O>(w, lane, DSPI_WIRE_FORMAT_VERSION, __float_as_uint(mv_db));
    __syncwarp();
    const dspi_bulk_host hv = *reinterpret_cast<const dspi_bulk_host *>(w + kPacketBytes);
    const bool bypass_master = w[DSPI_WIRE_OFF(global.bypass)] != 0;
    const bool bypass_t = touched(hit, DSPI_WIRE_OFF(global.bypass), 1), mv_t = touched(hit, DSPI_WIRE_OFF(master_volume.master_volume_db), 4);
    const bool vol_t = touched(hit, kPacketBytes, 2), host_t = touched(hit, kPacketBytes, 3);
    const bool xf_t = touched(hit, DSPI_WIRE_OFF(crossfeed), 16), lev_t = touched(hit, DSPI_WIRE_OFF(leveller), 16);
    const bool loud_t = touched(hit, DSPI_WIRE_OFF(global.loudness_enabled), 1) || touched(hit, DSPI_WIRE_OFF(global.loudness_ref_spl), 8);

    // ---- gains, output rows and delays: the ingest's lane layout ----
    const bool is_xp = lane < 2 * O, is_out = !is_xp && lane < 3 * O, is_pre = lane == 3 * O || lane == 3 * O + 1, is_mv = lane == 3 * O + 2;
    const uint32_t side = is_xp ? lane / O : (uint32_t)(lane - 3 * O), o = is_xp ? lane % O : (uint32_t)(lane - 2 * O);
    const uint32_t xp_off = DSPI_WIRE_OFF(crosspoints) + (side * WO + o) * 8, out_off = DSPI_WIRE_OFF(outputs) + o * 12;
    const bool out_en_t = is_out && touched(hit, out_off, 4), out_gain_t = is_out && touched(hit, out_off + 4, 4);
    const bool out_dly_t = is_out && touched(hit, out_off + 8, 4);
    const bool flags_t = __ballot_sync(0xffffffffu, out_en_t) != 0 || bypass_t;                   // every output: pair-off bits and skip rows
    const bool gains_t = __ballot_sync(0xffffffffu, out_en_t || out_gain_t) != 0 || mv_t || host_t;
    const bool dly_t = __ballot_sync(0xffffffffu, out_dly_t) != 0;
    if (is_xp) {
        if (touched(hit, xp_off, 8)) S::crosspoint(d, inst, side, o, w[xp_off] != 0, w[xp_off + 1] != 0, gain_linear(wire_f32(w, xp_off + 4), gain_mode));
    } else if (is_out) {
        if (out_gain_t) d.o_glin[o * Np + inst] = gain_linear(wire_f32(w, out_off + 4), gain_mode);
        if (flags_t) output_flag_rows<S>(d, w, inst, o, bypass_master);
        if (out_dly_t) output_delay_row<S>(d, w, inst, o, fs);
    } else if (is_pre) {
        if (touched(hit, DSPI_WIRE_OFF(preamp.preamp_db) + side * 4, 4)) S::preamp(d, inst, side, gain_linear(wire_f32(w, DSPI_WIRE_OFF(preamp.preamp_db) + side * 4), gain_mode));
    } else if (is_mv) {
        if (mv_t) S::master_volume(d, inst, mv_lin);
    }
    __syncwarp();
    const bool delayed = is_out && d.o_dly[o * Np + inst] > 0;                                     // the delays in force, touched or not
    const bool any_delay = __ballot_sync(0xffffffffu, delayed) != 0;

    // ---- the pending-flag handlers of the touched sections ----
    const dspi_leveller_config lev = leveller_config(w, DSPI_WIRE_FORMAT_VERSION);
    uint32_t row;
    const int16_t vol_mul = dyn::host_volume(hv.volume_8_8, row);
    if (lane == 0) {
        if (xf_t) S::crossfeed(d, inst, crossfeed_config(w), fs);
        if (flags_t || dly_t || xf_t || lev_t || loud_t) d.flags[inst] = instance_flags<S>(w, lev, any_delay);
        if (bypass_t) d.skip_m[inst] = d.skip_m[Np + inst] = bypass_master ? 1 : 0;
    } else if (lane == 1) {
        if (lev_t) S::leveller(d, inst, lev, fs);
    } else if (lane == 2) {
        if (loud_t || vol_t) loudness_row<S>(d, w, inst, row, fs);
    }
    __syncwarp();
    if (lane == 0 && gains_t) S::host_volume(d, inst, vol_mul, hv.host_mute != 0);

    // ---- the touched bands' recipes and their masks ----
    uint32_t m = 0;
    if (lane < NC)
        for (uint32_t b = 0; b < kMaxBands; b++)
            if (touched(hit, DSPI_WIRE_OFF(eq) + (lane * kMaxBands + b) * 16, 16)) m |= 1u << b;
    if (lane < NC) band_mask[lane * nseg + s] = (uint16_t)m;
    const bool any_band = __ballot_sync(0xffffffffu, m != 0) != 0;
    for (uint32_t r = lane; r < (uint32_t)NC * kMaxBands; r += 32)
        if (touched(hit, DSPI_WIRE_OFF(eq) + r * 16, 16)) stage_recipe(w, r, s, nseg, recipes);
    if (lane == 0) reject[s] = any_band ? 0 : 1;

    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
        bulk_store_1d(rec.packets + inst, w, kPacketBytes);
        tma_store_commit();
        tma_store_wait_all<0>();
    } else if (lane == 1) {
        rec.host[inst] = hv;
    }
}

// filter_recipes[][] of instances [inst0, inst0 + n) as dsp_compute_coefficients() left them -> the eq section of their records.
// Recipe (role, i, band) is recipes[role * role_stride + i * inst_stride + band]; reject, inst and band_mask as in RoleRange.
static __global__ void record_recipes_kernel(Record rec, uint32_t inst0, uint32_t n, uint32_t roles, const dspi_eq_param *__restrict__ recipes,
                                             size_t role_stride, size_t inst_stride, const int32_t *__restrict__ reject,
                                             const uint32_t *__restrict__ inst = nullptr, const uint16_t *__restrict__ band_mask = nullptr)
{
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * roles * kMaxBands) return;
    const uint32_t b = idx % kMaxBands, role = idx / kMaxBands % roles, i = idx / (kMaxBands * roles);
    if (reject && reject[i]) return;
    if (band_mask && !((band_mask[role * n + i] >> b) & 1u)) return;
    uint4 q = reinterpret_cast<const uint4 *>(recipes)[role * role_stride + i * inst_stride + b];
    q.x = (q.x >> 16) & 0xFFu;                                                                     // {channel, band, type, reserved} -> {type, reserved[3]}
    unsigned char *rp = reinterpret_cast<unsigned char *>(rec.packets + inst0 + (inst ? inst[i] : i));
    reinterpret_cast<uint4 *>(rp + DSPI_WIRE_OFF(eq))[role * kMaxBands + b] = q;
}

// dspi_chain(q)_set_params / _upload_biquads replaced records the packet does not describe any more
static __global__ void mark_stale_kernel(Record rec, uint32_t inst0, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && rec.mark[inst0 + i] == DSPI_BULK_CURRENT) rec.mark[inst0 + i] = DSPI_BULK_STALE;
}
inline cudaError_t mark_stale(const Record &rec, uint32_t inst0, uint32_t n, cudaStream_t s)
{
    mark_stale_kernel<<<(n + 255) / 256, 256, 0, s>>>(rec, inst0, n);
    return cudaGetLastError();
}

// What dspi_chain(q)_set_dynamics_device changes of the firmware's globals: crossfeed_config, leveller_config, the loudness
// settings and audio_state's volume and mute.  One instance per thread, from the engine's dynamics kernel.
__device__ inline void record_dynamics(const Record &rec, uint32_t inst, const dspi_dynamics_config &cfg)
{
    unsigned char *rp = reinterpret_cast<unsigned char *>(rec.packets + inst);
    auto put = [&](uint32_t off, uint32_t v) { *reinterpret_cast<uint32_t *>(rp + off) = v; };
    rp[DSPI_WIRE_OFF(global.loudness_enabled)] = cfg.loudness_enabled ? 1 : 0;
    put(DSPI_WIRE_OFF(global.loudness_ref_spl), __float_as_uint(cfg.loudness_ref_spl));
    put(DSPI_WIRE_OFF(global.loudness_intensity_pct), __float_as_uint(cfg.loudness_intensity_pct));
    put(DSPI_WIRE_OFF(crossfeed), (cfg.crossfeed.enabled ? 1u : 0u) | (uint32_t)cfg.crossfeed.preset << 8 | (cfg.crossfeed.itd_enabled ? 1u : 0u) << 16);
    put(DSPI_WIRE_OFF(crossfeed.custom_fc), __float_as_uint(cfg.crossfeed.custom_fc));
    put(DSPI_WIRE_OFF(crossfeed.custom_feed_db), __float_as_uint(cfg.crossfeed.custom_feed_db));
    put(DSPI_WIRE_OFF(leveller), (cfg.leveller.enabled ? 1u : 0u) | (uint32_t)cfg.leveller.speed << 8 | (cfg.leveller.lookahead ? 1u : 0u) << 16);
    put(DSPI_WIRE_OFF(leveller.amount), __float_as_uint(cfg.leveller.amount));
    put(DSPI_WIRE_OFF(leveller.max_gain_db), __float_as_uint(cfg.leveller.max_gain_db));
    put(DSPI_WIRE_OFF(leveller.gate_threshold_db), __float_as_uint(cfg.leveller.gate_threshold_db));
    rec.host[inst].volume_8_8 = cfg.volume_8_8;
    rec.host[inst].host_mute = cfg.host_mute;
}

// REQ_GET_ALL_PARAMS: record -> the packet bulk_params_collect() returns (:66-78 header, :123 pin count), one warp per instance.
// host and results may be null (a lane collect writes the caller's device memory, where both are optional).
template <class S>
__global__ void __launch_bounds__(kWarps * 32)
bulk_collect_kernel(Record rec, uint32_t inst0, uint32_t n, dspi_wire_bulk_params *__restrict__ packets, dspi_bulk_host *__restrict__ host,
                    int32_t *__restrict__ results)
{
    __shared__ alignas(16) unsigned char pkt_s[kWarps][kPacketBytes];
    __shared__ uint64_t bar_s[kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t i = blockIdx.x * kWarps + warp;
    if (i >= n) return;
    const uint32_t inst = inst0 + i;
    uint64_t *bar = &bar_s[warp];
    if (lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar, kPacketBytes);
        bulk_load_1d(pkt_s[warp], rec.packets + inst, kPacketBytes, bar);
    }
    __syncwarp();
    const uint8_t mark = rec.mark[inst];
    mbar_wait(bar, 0);
    uint32_t *W = reinterpret_cast<uint32_t *>(pkt_s[warp]);
    if (mark == DSPI_BULK_UNSET) {                         // whatever set_eq_params_device / set_dynamics_device noted: not a configuration yet
        for (uint32_t k = lane; k < kPacketBytes / 16; k += 32) reinterpret_cast<uint4 *>(W)[k] = make_uint4(0, 0, 0, 0);
    } else if (lane == 0) {
        W[0] = DSPI_WIRE_FORMAT_VERSION | (uint32_t)S::kPlatformId << 8 | (uint32_t)S::kRoles << 16 | (uint32_t)S::kOuts << 24;
        W[1] = 2u | (uint32_t)kMaxBands << 8 | kPacketBytes << 16;                                 // inputs, max_bands, payload_length
        W[2] = 1u | 1u << 16;                                                                      // firmware 1.1, config.h:273-274
        W[3] = 0;
        W[DSPI_WIRE_OFF(pins) / 4] = S::kPlatformId ? 5u : 3u;
        W[DSPI_WIRE_OFF(pins) / 4 + 1] = 0;
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
        bulk_store_1d(packets + i, pkt_s[warp], kPacketBytes);
        tma_store_commit();
        if (results) results[i] = mark;
        tma_store_wait_all<0>();
    } else if (lane == 1 && host) {
        host[i] = mark == DSPI_BULK_UNSET ? dspi_bulk_host{0, 0, 0} : rec.host[inst];
    }
}

// ---- preset slot images (PresetSlot v12, preset_slot.h) ----
template <class S>
using SlotOf = typename std::conditional<S::kPlatformId == DSPI_PLATFORM_RP2350, slot_rp2350, slot_rp2040>::type;
static_assert(sizeof(slot_rp2350) % 16 == 0 && sizeof(slot_rp2040) % 16 == 0, "the bulk copy moves multiples of 16 bytes");
constexpr uint32_t kSlotHeaderWords = 3;                   // magic, version | slot_index << 16, crc32; the CRC covers the rest

// crc32() of flash_storage.c:282-291 (reflected 0xEDB88320, as dspi_crc32), four tables for a word at a time
struct Crc32Tables {
    uint32_t t[4][256];
    constexpr Crc32Tables() : t{}
    {
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int j = 0; j < 8; j++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
            t[0][i] = c;
        }
        for (int k = 1; k < 4; k++)
            for (uint32_t i = 0; i < 256; i++) t[k][i] = (t[k - 1][i] >> 8) ^ t[0][t[k - 1][i] & 0xFFu];
    }
};
static __device__ const Crc32Tables kCrc32;

// the slot's CRC: words [kSlotHeaderWords, words) of an image in shared memory, on one lane
__device__ inline uint32_t slot_crc32(const uint32_t *W, uint32_t words)
{
    uint32_t crc = 0xFFFFFFFFu;
    for (uint32_t k = kSlotHeaderWords; k < words; k++) {
        crc ^= W[k];
        crc = __ldg(&kCrc32.t[3][crc & 0xFFu]) ^ __ldg(&kCrc32.t[2][(crc >> 8) & 0xFFu]) ^ __ldg(&kCrc32.t[1][(crc >> 16) & 0xFFu]) ^
              __ldg(&kCrc32.t[0][crc >> 24]);
    }
    return ~crc;
}

#define DSPI_SLOT_OFF(member) ((uint32_t)offsetof(T, member))

// preset_load(): image i of the chunk -> packet i of the chunk, and the preset result code.  validate_slot() (:750-760), then
// apply_slot_to_live() (:597-744) and apply_master_volume_from_mode() (:580-590) restated as the version-6 packet
// bulk_params_apply() gives the same fields from: the preamp per side from version 12 (the legacy field before), the leveller
// from version 10 (the fixed defaults before), the master volume the mode selects.  Gains stay in dB; the ingest kernel
// converts them.  A rejected image keeps the zero header, whose format version 0 the ingest kernel rejects.
template <class S>
__global__ void __launch_bounds__(kWarps * 32)
preset_decode_kernel(const unsigned char *__restrict__ images, const dspi_preset_load *__restrict__ load, uint32_t n,
                     dspi_wire_bulk_params *__restrict__ packets, int32_t *__restrict__ results)
{
    using T = SlotOf<S>;
    constexpr int NC = S::kRoles, NO = S::kOuts, WO = DSPI_WIRE_MAX_OUTPUTS;
    constexpr uint32_t kSlot = sizeof(T);
    static_assert(NC == NO + 2, "outputs are channels CH_OUT_1 = 2 onwards (config.h:310)");
    static_assert(DSPI_SLOT_OFF(filter_recipes) % 4 == 0 && DSPI_SLOT_OFF(preamp_db) % 4 == 0 && DSPI_SLOT_OFF(delays_ms) % 4 == 0 &&
                  DSPI_SLOT_OFF(channel_gain_db) % 4 == 0 && DSPI_SLOT_OFF(channel_mute) % 4 == 0 && DSPI_SLOT_OFF(loudness_enabled) % 4 == 0 &&
                  DSPI_SLOT_OFF(crossfeed_enabled) % 4 == 0 && DSPI_SLOT_OFF(matrix_crosspoints) % 4 == 0 && DSPI_SLOT_OFF(matrix_outputs) % 4 == 0 &&
                  DSPI_SLOT_OFF(leveller_enabled) % 4 == 0 && DSPI_SLOT_OFF(preamp_db_per_ch) % 4 == 0 && DSPI_SLOT_OFF(master_volume_db) % 4 == 0,
                  "the kernels move the image in 4-byte words");
    static_assert(DSPI_WIRE_OFF(eq) % 16 == 0, "16-byte recipe rows in the packet");
    __shared__ alignas(16) unsigned char img_s[kWarps][kSlot];
    __shared__ alignas(16) unsigned char pkt_s[kWarps][kPacketBytes];
    __shared__ uint64_t bar_s[kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t i = blockIdx.x * kWarps + warp;
    if (i >= n) return;
    uint64_t *bar = &bar_s[warp];
    if (lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar, kSlot);
        bulk_load_1d(img_s[warp], images + (size_t)i * kSlot, kSlot, bar);
    }
    uint32_t *P = reinterpret_cast<uint32_t *>(pkt_s[warp]);
    for (uint32_t k = lane; k < kPacketBytes / 16; k += 32) reinterpret_cast<uint4 *>(P)[k] = make_uint4(0, 0, 0, 0);
    const dspi_preset_load ld = load[i];
    __syncwarp();
    mbar_wait(bar, 0);
    const uint32_t *I = reinterpret_cast<const uint32_t *>(img_s[warp]);
    auto iw = [&](uint32_t off) { return I[off / 4]; };
    const uint32_t version = I[1] & 0xFFFFu;

    constexpr uint32_t g = DSPI_WIRE_OFF(global) / 4, x = DSPI_WIRE_OFF(crossfeed) / 4, lg = DSPI_WIRE_OFF(legacy) / 4, dl = DSPI_WIRE_OFF(delays) / 4,
                       xp = DSPI_WIRE_OFF(crosspoints) / 4, out = DSPI_WIRE_OFF(outputs) / 4, eq = DSPI_WIRE_OFF(eq) / 4,
                       lev = DSPI_WIRE_OFF(leveller) / 4, pre = DSPI_WIRE_OFF(preamp) / 4, mv = DSPI_WIRE_OFF(master_volume) / 4;
    if (lane == 0) {                                                                               // :602-620, :634-645
        P[g] = version >= 12 ? iw(DSPI_SLOT_OFF(preamp_db_per_ch)) : iw(DSPI_SLOT_OFF(preamp_db));
        P[g + 1] = (iw(DSPI_SLOT_OFF(bypass)) & 0xFFu) | (iw(DSPI_SLOT_OFF(loudness_enabled)) & 0xFFu) << 8;
        P[g + 2] = iw(DSPI_SLOT_OFF(loudness_ref_spl));
        P[g + 3] = iw(DSPI_SLOT_OFF(loudness_intensity_pct));
        P[x] = iw(DSPI_SLOT_OFF(crossfeed_enabled)) & 0xFFFFFFu;                                   // {enabled, preset, itd_enabled} on both sides
        P[x + 1] = iw(DSPI_SLOT_OFF(crossfeed_custom_fc));
        P[x + 2] = iw(DSPI_SLOT_OFF(crossfeed_custom_feed_db));
    } else if (lane == 1) {                                                                        // :626-631
        for (int k = 0; k < 3; k++) P[lg + k] = iw(DSPI_SLOT_OFF(channel_gain_db) + 4 * k);
        P[lg + 3] = iw(DSPI_SLOT_OFF(channel_mute)) & 0xFFFFFFu;
    } else if (lane == 2) {                                                                        // :724-741
        if (version >= 10) {
            P[lev] = iw(DSPI_SLOT_OFF(leveller_enabled)) & 0xFFFFFFu;                              // {enabled, speed, lookahead} on both sides
            for (int k = 1; k < 4; k++) P[lev + k] = iw(DSPI_SLOT_OFF(leveller_amount) + 4 * (k - 1));
        } else {
            P[lev] = 1u << 16;
            P[lev + 1] = __float_as_uint(50.0f);
            P[lev + 2] = __float_as_uint(15.0f);
            P[lev + 3] = __float_as_uint(-96.0f);
        }
    } else if (lane == 3) {                                                                        // :602-617, :580-590
        for (int k = 0; k < 2; k++) P[pre + k] = version >= 12 ? iw(DSPI_SLOT_OFF(preamp_db_per_ch) + 4 * k) : iw(DSPI_SLOT_OFF(preamp_db));
        P[mv] = (ld.master_volume_mode == 1 && version >= 12) ? iw(DSPI_SLOT_OFF(master_volume_db)) : __float_as_uint(ld.dir_master_volume_db);
    }
    if (lane < NC) P[dl + lane] = iw(DSPI_SLOT_OFF(delays_ms) + 4 * lane);                         // :623
    if (lane < 2 * NO) {                                                                           // :648-655
        const uint32_t side = lane / NO, o = lane % NO, s = DSPI_SLOT_OFF(matrix_crosspoints) / 4 + lane * 2, d = xp + (side * WO + o) * 2;
        P[d] = I[s] & 0xFFFFu;
        P[d + 1] = I[s + 1];
    } else if (lane < 3 * NO) {                                                                    // :656-663
        const uint32_t o = lane - 2 * NO, s = DSPI_SLOT_OFF(matrix_outputs) / 4 + o * 3;
        P[out + o * 3] = I[s] & 0xFFFFu;
        P[out + o * 3 + 1] = I[s + 1];
        P[out + o * 3 + 2] = I[s + 2];
    }
    for (uint32_t r = lane; r < (uint32_t)NC * kMaxBands; r += 32) {                               // :599, {channel, band, type, reserved} -> {type, reserved[3]}
        const uint32_t *q = I + DSPI_SLOT_OFF(filter_recipes) / 4 + r * 4;                         // 4-byte aligned only: the recipes start at byte 12
        reinterpret_cast<uint4 *>(P + eq)[r] = make_uint4((q[0] >> 16) & 0xFFu, q[1], q[2], q[3]);
    }
    __syncwarp();
    if (lane == 0) {
        const bool ok = I[0] == DSPI_PRESET_SLOT_MAGIC && (I[1] >> 16) == ld.slot_index && slot_crc32(I, kSlot / 4) == I[2];
        if (ok) {
            P[0] = 6u | (uint32_t)S::kPlatformId << 8 | (uint32_t)NC << 16 | (uint32_t)NO << 24;
            P[1] = 2u | (uint32_t)kMaxBands << 8 | kPacketBytes << 16;
        }
        results[i] = ok ? DSPI_PRESET_OK : DSPI_PRESET_ERR_CRC;
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
        bulk_store_1d(packets + i, pkt_s[warp], kPacketBytes);
        tma_store_commit();
        tma_store_wait_all<0>();
    }
}

// preset_save()'s state part for a record: what dspi_preset_slot_collect writes for the dspi_bulk_state
// dspi_bulk_params_apply(packet, exact_db = 1) leaves from dspi_bulk_state_defaults, where the packet is what
// bulk_collect_kernel returns.  An unset instance gives zero bytes.  One warp per instance.
template <class S>
__global__ void __launch_bounds__(kWarps * 32)
preset_collect_kernel(Record rec, uint32_t inst0, uint32_t n, const uint8_t *__restrict__ slots, unsigned char *__restrict__ images,
                      int32_t *__restrict__ results)
{
    using T = SlotOf<S>;
    constexpr int NC = S::kRoles, NO = S::kOuts, WO = DSPI_WIRE_MAX_OUTPUTS;
    constexpr uint32_t kSlot = sizeof(T);
    __shared__ alignas(16) unsigned char img_s[kWarps][kSlot];
    __shared__ alignas(16) unsigned char pkt_s[kWarps][kPacketBytes];
    __shared__ uint64_t bar_s[kWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t i = blockIdx.x * kWarps + warp;
    if (i >= n) return;
    const uint32_t inst = inst0 + i;
    uint64_t *bar = &bar_s[warp];
    if (lane == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(bar, kPacketBytes);
        bulk_load_1d(pkt_s[warp], rec.packets + inst, kPacketBytes, bar);
    }
    uint32_t *I = reinterpret_cast<uint32_t *>(img_s[warp]);
    for (uint32_t k = lane; k < kSlot / 16; k += 32) reinterpret_cast<uint4 *>(I)[k] = make_uint4(0, 0, 0, 0);
    const uint8_t mark = rec.mark[inst];
    __syncwarp();
    mbar_wait(bar, 0);
    if (mark != DSPI_BULK_UNSET) {
        const uint32_t *P = reinterpret_cast<const uint32_t *>(pkt_s[warp]);
        auto put = [&](uint32_t off, uint32_t v) { I[off / 4] = v; };
        auto flag = [](uint32_t word, int byte) { return ((word >> (8 * byte)) & 0xFFu) ? 1u << (8 * byte) : 0u; };
        constexpr uint32_t g = DSPI_WIRE_OFF(global) / 4, x = DSPI_WIRE_OFF(crossfeed) / 4, lg = DSPI_WIRE_OFF(legacy) / 4,
                           dl = DSPI_WIRE_OFF(delays) / 4, xp = DSPI_WIRE_OFF(crosspoints) / 4, out = DSPI_WIRE_OFF(outputs) / 4,
                           eq = DSPI_WIRE_OFF(eq) / 4, lev = DSPI_WIRE_OFF(leveller) / 4, pre = DSPI_WIRE_OFF(preamp) / 4,
                           mv = DSPI_WIRE_OFF(master_volume) / 4;
        if (lane == 0) {
            put(DSPI_SLOT_OFF(preamp_db), P[pre]);                                                 // preamp_db[0] after a version-6 apply
            put(DSPI_SLOT_OFF(bypass), flag(P[g + 1], 0));
            put(DSPI_SLOT_OFF(loudness_enabled), flag(P[g + 1], 1) >> 8);
            put(DSPI_SLOT_OFF(loudness_ref_spl), P[g + 2]);
            put(DSPI_SLOT_OFF(loudness_intensity_pct), P[g + 3]);
            put(DSPI_SLOT_OFF(crossfeed_enabled), flag(P[x], 0) | (P[x] & 0xFF00u) | flag(P[x], 2));
            put(DSPI_SLOT_OFF(crossfeed_custom_fc), P[x + 1]);
            put(DSPI_SLOT_OFF(crossfeed_custom_feed_db), P[x + 2]);
        } else if (lane == 1) {
            for (int k = 0; k < 3; k++) put(DSPI_SLOT_OFF(channel_gain_db) + 4 * k, P[lg + k]);
            put(DSPI_SLOT_OFF(channel_mute), flag(P[lg + 3], 0) | flag(P[lg + 3], 1) | flag(P[lg + 3], 2));
        } else if (lane == 2) {
            put(DSPI_SLOT_OFF(leveller_enabled), flag(P[lev], 0) | (P[lev] & 0xFF00u) | flag(P[lev], 2));
            for (int k = 0; k < 3; k++) put(DSPI_SLOT_OFF(leveller_amount) + 4 * k, P[lev + 1 + k]);
        } else if (lane == 3) {
            for (int k = 0; k < 2; k++) put(DSPI_SLOT_OFF(preamp_db_per_ch) + 4 * k, P[pre + k]);
            float db = __uint_as_float(P[mv]);                                                     // bulk_params.c:361-368
            if (isnan(db) || isinf(db)) db = 0.0f;
            if (db < -128.0f) db = -128.0f;
            if (db > 0.0f) db = 0.0f;
            put(DSPI_SLOT_OFF(master_volume_db), __float_as_uint(db));
        }
        if (lane < NC) put(DSPI_SLOT_OFF(delays_ms) + 4 * lane, lane < 2 ? P[dl + lane] : P[out + (lane - 2) * 3 + 2]);
        if (lane < 2 * NO) {
            const uint32_t side = lane / NO, o = lane % NO, d = DSPI_SLOT_OFF(matrix_crosspoints) / 4 + lane * 2, s = xp + (side * WO + o) * 2;
            I[d] = P[s] & 0xFFFFu;
            I[d + 1] = P[s + 1];
        } else if (lane < 3 * NO) {
            const uint32_t o = lane - 2 * NO, d = DSPI_SLOT_OFF(matrix_outputs) / 4 + o * 3;
            I[d] = P[out + o * 3] & 0xFFFFu;
            I[d + 1] = P[out + o * 3 + 1];
            I[d + 2] = P[out + o * 3 + 2];
        }
        for (uint32_t r = lane; r < (uint32_t)NC * kMaxBands; r += 32) {                           // {type, reserved[3]} -> {channel, band, type, 0}
            const uint4 q = reinterpret_cast<const uint4 *>(P + eq)[r];
            uint32_t *d = I + DSPI_SLOT_OFF(filter_recipes) / 4 + r * 4;                           // 4-byte aligned only: the recipes start at byte 12
            d[0] = r / kMaxBands | (r % kMaxBands) << 8 | (q.x & 0xFFu) << 16;
            d[1] = q.y;
            d[2] = q.z;
            d[3] = q.w;
        }
        __syncwarp();
        if (lane == 0) {
            I[0] = DSPI_PRESET_SLOT_MAGIC;
            I[1] = DSPI_PRESET_SLOT_VERSION | (uint32_t)slots[i] << 16;
            I[2] = slot_crc32(I, kSlot / 4);
        }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
        bulk_store_1d(images + (size_t)i * kSlot, img_s[warp], kSlot);
        tma_store_commit();
        results[i] = mark;
        tma_store_wait_all<0>();
    }
}
#undef DSPI_SLOT_OFF

// a queue's staging of one chunk: packets, host volumes, recipes, sample rates (rate switch) and result codes on the device.
// A lane's apply uploads a chunk's packets and host records in one copy: the host records follow the chunk's packets
// (lane_host), in room kept after the packets.
struct Stage {
    dspi_wire_bulk_params *packets = nullptr;
    dspi_bulk_host *host = nullptr;
    dspi_eq_param *recipes = nullptr;
    float *rates = nullptr;
    int32_t *results = nullptr;
    cudaError_t ensure(int roles)
    {
        if (results) return cudaSuccess;
        cudaError_t e = cudaMalloc((void **)&packets, (size_t)kChunk * (kPacketBytes + sizeof(dspi_bulk_host)));
        if (e == cudaSuccess) e = cudaMalloc((void **)&host, (size_t)kChunk * sizeof(dspi_bulk_host));
        if (e == cudaSuccess) e = cudaMalloc((void **)&recipes, (size_t)kChunk * roles * kMaxBands * sizeof(dspi_eq_param));
        if (e == cudaSuccess) e = cudaMalloc((void **)&rates, (size_t)kChunk * sizeof(float));
        if (e == cudaSuccess) e = cudaMalloc((void **)&results, (size_t)kChunk * sizeof(int32_t));
        if (e != cudaSuccess) destroy();
        return e;
    }
    void destroy()
    {
        cudaFree(packets); cudaFree(host); cudaFree(recipes); cudaFree(rates); cudaFree(results);
        packets = nullptr; host = nullptr; recipes = nullptr; rates = nullptr; results = nullptr;
    }
    dspi_bulk_host *lane_host(uint32_t nc) const { return reinterpret_cast<dspi_bulk_host *>(packets + nc); }
};

// a queue's staging of the preset calls, next to Stage.  A lane's preset apply uploads a chunk's images (packed at the slot
// size), load rows and host records in one copy into `images`, which keeps room for the two after the images.
struct PresetStage {
    unsigned char *images = nullptr;                       // [kChunk][slot size], packed; then room for [kChunk] load and host rows
    dspi_preset_load *load = nullptr;                      // [kChunk]; a collect call keeps its slot indices here, one byte each
    int32_t *results = nullptr;                            // [kChunk] preset result codes, or the marks of a collect
    cudaError_t ensure(size_t slot_bytes)
    {
        if (results) return cudaSuccess;
        cudaError_t e = cudaMalloc((void **)&images, (size_t)kChunk * (slot_bytes + sizeof(dspi_preset_load) + sizeof(dspi_bulk_host)));
        if (e == cudaSuccess) e = cudaMalloc((void **)&load, (size_t)kChunk * sizeof(dspi_preset_load));
        if (e == cudaSuccess) e = cudaMalloc((void **)&results, (size_t)kChunk * sizeof(int32_t));
        if (e != cudaSuccess) destroy();
        return e;
    }
    void destroy()
    {
        cudaFree(images); cudaFree(load); cudaFree(results);
        images = nullptr; load = nullptr; results = nullptr;
    }
};

// engine-owned staging of the edit calls, next to Stage: one chunk of edits grouped by instance with its segment table, as
// uploaded in one copy, and the band masks and marks of edit_kernel.  The host side keeps the upload image and, per
// instance, 1 + its segment in the chunk being grouped (0 outside it).
struct EditStage {
    unsigned char *d_in = nullptr;                         // [E] edits, [nseg + 1] segment offsets, [nseg] instances
    uint16_t *band_mask = nullptr;                         // [roles][kChunk]
    int32_t *marks = nullptr;                              // [kChunk]
    std::vector<unsigned char> h_in;
    std::vector<uint32_t> seg, last, count, inst;          // seg, last: per instance of the engine, or of a lane's window
    // with a lane edit's device results, each grouped edit's position in the call and its segment follow: [E] + [E]
    static constexpr size_t kInBytes = (size_t)kEditChunk * (sizeof(dspi_bulk_edit) + 2 * sizeof(uint32_t)) + (size_t)(2 * kChunk + 1) * sizeof(uint32_t);
    cudaError_t ensure(int roles, uint32_t n_instances)
    {
        if (seg.size() < n_instances) seg.assign(n_instances, 0);
        if (last.size() < n_instances) last.resize(n_instances);
        if (marks) return cudaSuccess;
        h_in.resize(kInBytes);
        count.resize(kChunk);
        inst.reserve(kChunk);
        cudaError_t e = cudaMalloc((void **)&d_in, kInBytes);
        if (e == cudaSuccess) e = cudaMalloc((void **)&band_mask, (size_t)roles * kChunk * sizeof(uint16_t));
        if (e == cudaSuccess) e = cudaMalloc((void **)&marks, (size_t)kChunk * sizeof(int32_t));
        if (e != cudaSuccess) destroy();
        return e;
    }
    void destroy()
    {
        cudaFree(d_in); cudaFree(band_mask); cudaFree(marks);
        d_in = nullptr; band_mask = nullptr; marks = nullptr;
    }
};

// Pinned host staging of a lane's control calls (edits, fade rows, transmitter rows): kSlots buffers taken in turn.  Each
// is guarded by an event recorded behind the copies that read it, so the host writes a buffer again only once those
// copies are done: with fewer than kSlots uploads in flight on the lane, taking one never waits.  A buffer grows to the
// largest upload it has carried; growing is a pinned allocation, which may wait for the device.
struct HostRing {
    static constexpr int kSlots = 8;
    unsigned char *buf[kSlots] = {};
    size_t cap[kSlots] = {};
    cudaEvent_t ev[kSlots] = {};
    int next = 0, cur = 0;
    cudaError_t take(size_t bytes, unsigned char **out)
    {
        const int k = next;
        cudaError_t e = ev[k] ? cudaEventSynchronize(ev[k]) : cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming);
        if (e == cudaSuccess && bytes > cap[k]) {
            cudaFreeHost(buf[k]);
            buf[k] = nullptr; cap[k] = 0;
            e = cudaHostAlloc((void **)&buf[k], bytes, cudaHostAllocDefault);
            if (e == cudaSuccess) cap[k] = bytes;
        }
        if (e != cudaSuccess) return e;
        next = (k + 1) % kSlots;
        cur = k;
        *out = buf[k];
        return cudaSuccess;
    }
    // the copies reading the buffer taken last are issued on s
    cudaError_t done(cudaStream_t s) { return cudaEventRecord(ev[cur], s); }
    void destroy()
    {
        for (int k = 0; k < kSlots; k++) {
            if (ev[k]) cudaEventSynchronize(ev[k]), cudaEventDestroy(ev[k]);
            cudaFreeHost(buf[k]);
            buf[k] = nullptr; cap[k] = 0; ev[k] = nullptr;
        }
        next = cur = 0;
    }
};

// A lane's upload of `bytes` to device memory `dst` on q's stream: fill(buf) packs them into a buffer taken from q's ring,
// which one copy sends; the buffer's event is recorded behind it.
template <class Queue, class Fill>
cudaError_t lane_upload(Queue &q, void *dst, size_t bytes, Fill &&fill)
{
    unsigned char *buf = nullptr;
    cudaError_t e = q.ring.take(bytes, &buf);
    if (e != cudaSuccess) return e;
    fill(buf);
    e = cudaMemcpyAsync(dst, buf, bytes, cudaMemcpyHostToDevice, q.stream);
    return e == cudaSuccess ? q.ring.done(q.stream) : e;
}

// d_results of a lane edit: grouped edit j of a chunk is edit pos[j] of the call, whose instance is segment seg[j]
static __global__ void edit_marks_kernel(const int32_t *__restrict__ marks, const uint32_t *__restrict__ pos, const uint32_t *__restrict__ seg,
                                         uint32_t n, int32_t *__restrict__ out)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) out[pos[j]] = marks[seg[j]];
}

inline int fail_cuda(cudaError_t e, const char *what)
{
    size_t cap = 0;
    char *buf = error_buffer(&cap);
    snprintf(buf, cap, "bulk ingest: %s -> %s", what, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? DSPI_ENOMEM : DSPI_ECUDA;
}

// dsp_recalculate_all_filters() for instances [first, first + nc) whose recipes are in stage.recipes and whose code in
// stage.results is 0 (the others are left alone): state into the mirrors, coefficients from the recipes at fs (or at
// rates[i] when rates is not null), the clamped recipes into the records, mirrors back into the packed stores.  With `inst`
// (device, [nc]) instance i is first + inst[i]; with `band_mask` (device, [roles][nc]) only the masked bands are computed.
// Issued on queue q (chain_host.cuh) with its staging; the engine's queue packs synchronously, a lane's packs and remasks its
// window's rows only.
template <class S, class Engine, class Queue>
int recalculate_filters(Engine *c, Queue &q, uint32_t first, uint32_t nc, float fs, const float *rates, const uint32_t *inst = nullptr,
                        const uint16_t *band_mask = nullptr)
{
    const cudaStream_t s = q.stream;
    const Stage &stage = q.bulk;
    RoleRange rm, ro;
    rm.roles = 2; ro.roles = S::kRoles - 2;
    rm.stride = ro.stride = c->d.N_pad;
    rm.reject = ro.reject = stage.results;
    rm.fs = ro.fs = rates;
    rm.inst = ro.inst = inst;
    rm.band_mask = band_mask;
    ro.band_mask = band_mask ? band_mask + (size_t)2 * nc : nullptr;
    int rc = eq_unpack_range(c->eq_m, first, nc, s, rm);
    if (rc == DSPI_OK) rc = eq_unpack_range(c->eq_o, first, nc, s, ro);
    if (rc != DSPI_OK) return rc;
    cudaError_t e = launch_coeffs(S::kQ28, stage.recipes, eq_aos_mirror(c->eq_m), first, nc, fs, s, rm);
    if (e == cudaSuccess) e = launch_coeffs(S::kQ28, stage.recipes + (size_t)2 * nc * kMaxBands, eq_aos_mirror(c->eq_o), first, nc, fs, s, ro);
    if (e != cudaSuccess) return fail_cuda(e, "coefficient kernels");
    record_recipes_kernel<<<(nc * S::kRoles * kMaxBands + 255) / 256, 256, 0, s>>>(c->rec, first, nc, S::kRoles, stage.recipes,
                                                                                   (size_t)nc * kMaxBands, kMaxBands, stage.results, inst, band_mask);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "recipe record kernel");
    c->launches += 3;
    if (q.lane) {
        rc = eq_pack_rows(c->eq_m, first, nc, s, rm, q.inst0, q.n);
        return rc == DSPI_OK ? eq_pack_rows(c->eq_o, first, nc, s, ro, q.inst0, q.n) : rc;
    }
    rc = eq_pack_range(c->eq_m, first, nc, s, rm);
    if (rc == DSPI_OK) rc = eq_pack_range(c->eq_o, first, nc, s, ro);
    return rc;
}

// The skip rows into the sub-engines' effective modes after the last chunk, on queue q: every row, synchronising (the
// engine's queue), or the rows of a lane's window (eq_skip_set must hold for both sub-engines).
template <class Engine, class Queue>
int finish_skip(Engine *c, Queue &q)
{
    if (q.lane) {
        RoleRange rm, ro;
        rm.roles = 2; ro.roles = Engine::Arith::kOuts;
        rm.stride = ro.stride = c->d.N_pad;
        const int rc = eq_remask_rows(c->eq_m, q.inst0, q.n, rm, q.stream);
        return rc == DSPI_OK ? eq_remask_rows(c->eq_o, q.inst0, q.n, ro, q.stream) : rc;
    }
    int rc = eq_set_skip(c->eq_m, c->d.skip_m, q.stream);
    if (rc == DSPI_OK) rc = eq_set_skip(c->eq_o, c->d.skip_o, q.stream);
    return rc;
}

// The ingest path for an engine (dspi_chain or dspi_chainq) whose arguments are checked, issued on queue q with its staging,
// behind earlier calls on it.  Per chunk, stage_inputs(i0, nc, &d_host) puts the packets of instances [i0, i0 + nc) of the
// call into stage.packets on q's stream; on a lane it uploads their host records with them and points d_host at them,
// otherwise ingest copies them to stage.host.  `codes` (device, [kChunk]) is what goes back to results, stage.results (the
// ingest kernel's codes) when it is null: host memory for the engine's queue, whose last step (eq_set_skip) synchronises
// it, device memory for a lane's, copied on the lane stream.
template <class S, class Engine, class Queue, class StageInputs>
int ingest(Engine *c, Queue &q, uint32_t inst0, uint32_t n, const dspi_bulk_host *host, int gain_mode, float fs, int32_t *results,
           const int32_t *codes, StageInputs &&stage_inputs)
{
    Stage &stage = q.bulk;
    cudaError_t e = stage.ensure(S::kRoles);
    if (e != cudaSuccess) return fail_cuda(e, "staging buffers");
    cudaStream_t s = q.stream;
    for (uint32_t i0 = 0; i0 < n; i0 += kChunk) {
        const uint32_t nc = n - i0 < kChunk ? n - i0 : kChunk, first = inst0 + i0;
        const dspi_bulk_host *d_host = stage.host;
        int rc = stage_inputs(i0, nc, &d_host);
        if (rc != DSPI_OK) return rc;
        if (!q.lane && (e = cudaMemcpyAsync(stage.host, host + i0, (size_t)nc * sizeof(dspi_bulk_host), cudaMemcpyHostToDevice, s)) != cudaSuccess)
            return fail_cuda(e, "packet copy");
        bulk_ingest_kernel<S><<<(nc + kWarps - 1) / kWarps, kWarps * 32, 0, s>>>(c->d, c->rec, first, nc, stage.packets, d_host, gain_mode, fs,
                                                                                 stage.recipes, stage.results);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "ingest kernel");
        c->launches++;
        if ((rc = recalculate_filters<S>(c, q, first, nc, fs, nullptr)) != DSPI_OK) return rc;
        if ((e = cudaMemcpyAsync(results + i0, codes ? codes : stage.results, (size_t)nc * sizeof(int32_t),
                                 q.lane ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s)) != cudaSuccess)
            return fail_cuda(e, "result copy");
    }
    return finish_skip(c, q);
}

// dspi_chain(q)_set_rate_device for checked arguments: per chunk the rates go to stage.rates, rate_kernel re-derives the
// rate-dependent rows of current instances and stages their recipes, and the filters are recalculated at each one's rate.
// results (may be null) gets the marks.  On queue q behind earlier work: the engine's returns when the engine is updated
// and results is host memory; a lane's uploads the rates through its ring and results is device memory.
template <class S, class Engine, class Queue>
int set_rate(Engine *c, Queue &q, uint32_t inst0, uint32_t n, const float *rates, int32_t *results)
{
    Stage &stage = q.bulk;
    cudaError_t e = stage.ensure(S::kRoles);
    if (e != cudaSuccess) return fail_cuda(e, "staging buffers");
    cudaStream_t s = q.stream;
    for (uint32_t i0 = 0; i0 < n; i0 += kChunk) {
        const uint32_t nc = n - i0 < kChunk ? n - i0 : kChunk, first = inst0 + i0;
        const size_t bytes = (size_t)nc * sizeof(float);
        e = q.lane ? lane_upload(q, stage.rates, bytes, [&](unsigned char *b) { memcpy(b, rates + i0, bytes); })
                   : cudaMemcpyAsync(stage.rates, rates + i0, bytes, cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return fail_cuda(e, "rate copy");
        rate_kernel<S><<<(nc + kWarps - 1) / kWarps, kWarps * 32, 0, s>>>(c->d, c->rec, first, nc, stage.rates, stage.recipes, stage.results);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "rate kernel");
        c->launches++;
        int rc = recalculate_filters<S>(c, q, first, nc, 0.0f, stage.rates);
        if (rc != DSPI_OK) return rc;
        if (results && (e = cudaMemcpyAsync(results + i0, stage.results, (size_t)nc * sizeof(int32_t),
                                            q.lane ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s)) != cudaSuccess)
            return fail_cuda(e, "result copy");
    }
    return finish_skip(c, q);
}

// dspi_chain(q)_edit_bulk_device for checked arguments.  Edits of different instances commute, so the list is cut into
// chunks by instance: a chunk takes the pending edits of the first kChunk instances it meets, at most kEditChunk edits, and
// leaves the others for later chunks; an instance's edits keep their list order within and across chunks.  Per chunk the
// edits are grouped by instance on the host - a stable counting pass, segments in order of first appearance - and uploaded
// with their segment table in one copy; edit_kernel applies them, and when an edit of the chunk lies in the eq section the
// touched bands go through the filter recalculation by instance list and band mask.  eq_set_skip at the end follows the
// skip rows and synchronises.  results (host, may be null) gets the mark of each edit's instance.
// Everything is issued on queue q with its staging, every instance inside its window.  A lane edit uploads through the
// lane's pinned ring, remasks its window's rows only and does not synchronise; results is device memory there.
template <class S, class Engine, class Queue>
int edit(Engine *c, Queue &q, uint32_t n_edits, const dspi_bulk_edit *edits, int exact_db, float fs, int32_t *results)
{
    const cudaStream_t s = q.stream;
    Stage &stage = q.bulk;
    EditStage &es = q.bulk_edit;
    int32_t *d_results = q.lane ? results : nullptr;
    if (q.lane) results = nullptr;
    const uint32_t base = q.inst0;                         // es.seg and es.last are indexed by instance - base
    cudaError_t e = stage.ensure(S::kRoles);
    if (e == cudaSuccess) e = es.ensure(S::kRoles, q.n);
    if (e != cudaSuccess) return fail_cuda(e, "staging buffers");
    constexpr uint32_t eq0 = DSPI_WIRE_OFF(eq), eq1 = DSPI_WIRE_OFF(eq) + S::kRoles * kMaxBands * 16;
    std::vector<int32_t> marks;                            // per segment of the call (never more than the edits)
    std::vector<uint32_t> seg_of(results ? n_edits : 0);   // per edit: its segment
    if (results) marks.reserve(n_edits);
    // per instance its last edit, so that a chunk holding kChunk instances stops scanning after their last edit
    for (uint32_t k = 0; k < n_edits; k++) es.last[edits[k].instance - base] = k;
    std::vector<uint32_t> pending(n_edits), taken, later;
    for (uint32_t k = 0; k < n_edits; k++) pending[k] = k;
    taken.reserve(n_edits < kEditChunk ? n_edits : kEditChunk);
    while (!pending.empty()) {
        // the chunk: in list order, every pending edit of the first kChunk instances met, at most kEditChunk edits; the
        // edits of other instances wait for a later chunk, so each instance's edits keep their order
        uint32_t nseg = 0, stop = 0;
        bool bands = false;
        es.inst.clear();
        taken.clear();
        later.clear();
        size_t p = 0;
        for (; p < pending.size(); p++) {
            const uint32_t k = pending[p];
            if (taken.size() == kEditChunk || (nseg == kChunk && k > stop)) break;
            const dspi_bulk_edit &ed = edits[k];
            uint32_t &sl = es.seg[ed.instance - base];
            if (!sl) {
                if (nseg == kChunk) {
                    later.push_back(k);
                    continue;
                }
                es.inst.push_back(ed.instance);
                es.count[nseg] = 0;
                sl = ++nseg;
                stop = std::max(stop, es.last[ed.instance - base]);
            }
            es.count[sl - 1]++;
            taken.push_back(k);
            bands |= ed.offset < eq1 && ed.offset + ed.length > eq0;
        }
        later.insert(later.end(), pending.begin() + p, pending.end());
        pending.swap(later);
        const uint32_t E = (uint32_t)taken.size();
        // upload image: edits grouped by segment, then the segment offsets, then the segments' instances (then, for
        // d_results, each grouped edit's position in the call and its segment)
        const size_t bytes = (size_t)E * sizeof(dspi_bulk_edit) + (size_t)(2 * nseg + 1) * sizeof(uint32_t) + (d_results ? (size_t)2 * E * sizeof(uint32_t) : 0);
        unsigned char *img = es.h_in.data();
        if (q.lane && (e = q.ring.take(bytes, &img)) != cudaSuccess) return fail_cuda(e, "edit staging");
        dspi_bulk_edit *ed_h = reinterpret_cast<dspi_bulk_edit *>(img);
        uint32_t *off_h = reinterpret_cast<uint32_t *>(img + (size_t)E * sizeof(dspi_bulk_edit));
        uint32_t *pos_h = off_h + 2 * nseg + 1;
        for (uint32_t g = 0, acc = 0; g <= nseg; g++) {
            off_h[g] = acc;
            if (g < nseg) acc += es.count[g];
        }
        memcpy(es.count.data(), off_h, (size_t)nseg * sizeof(uint32_t));                          // now each segment's write cursor
        const size_t done = marks.size();
        for (const uint32_t k : taken) {
            const uint32_t g = es.seg[edits[k].instance - base] - 1, j = es.count[g]++;
            ed_h[j] = edits[k];
            if (results) seg_of[k] = (uint32_t)done + g;
            if (d_results) { pos_h[j] = k; pos_h[E + j] = g; }
        }
        for (uint32_t g = 0; g < nseg; g++) es.seg[es.inst[g] - base] = 0;
        memcpy(off_h + nseg + 1, es.inst.data(), (size_t)nseg * sizeof(uint32_t));
        if ((e = cudaMemcpyAsync(es.d_in, img, bytes, cudaMemcpyHostToDevice, s)) != cudaSuccess) return fail_cuda(e, "edit copy");
        if (q.lane && (e = q.ring.done(s)) != cudaSuccess) return fail_cuda(e, "edit staging");
        const dspi_bulk_edit *d_edits = reinterpret_cast<const dspi_bulk_edit *>(es.d_in);
        const uint32_t *d_off = reinterpret_cast<const uint32_t *>(es.d_in + (size_t)E * sizeof(dspi_bulk_edit)), *d_inst = d_off + nseg + 1;
        edit_kernel<S><<<(nseg + kWarps - 1) / kWarps, kWarps * 32, 0, s>>>(c->d, c->rec, nseg, d_edits, d_off, d_inst, exact_db ? kGainExact : kGainTaylor,
                                                                           fs, stage.recipes, es.band_mask, stage.results, es.marks);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "edit kernel");
        c->launches++;
        if (d_results) {
            const uint32_t *d_pos = d_inst + nseg;
            edit_marks_kernel<<<(E + 255) / 256, 256, 0, s>>>(es.marks, d_pos, d_pos + E, E, d_results);
            if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "edit mark kernel");
            c->launches++;
        }
        if (bands) {
            const int rc = recalculate_filters<S>(c, q, 0, nseg, fs, nullptr, d_inst, es.band_mask);
            if (rc != DSPI_OK) return rc;
        }
        if (results) {
            marks.resize(done + nseg);
            if ((e = cudaMemcpyAsync(marks.data() + done, es.marks, (size_t)nseg * sizeof(int32_t), cudaMemcpyDeviceToHost, s)) != cudaSuccess)
                return fail_cuda(e, "mark copy");
        }
    }
    const int rc = finish_skip(c, q);
    if (rc != DSPI_OK) return rc;
    for (uint32_t k = 0; results && k < n_edits; k++) results[k] = marks[seg_of[k]];
    return DSPI_OK;
}

// dspi_chain(q)_apply_bulk_device for checked arguments, on queue q
template <class S, class Engine, class Queue>
int apply(Engine *c, Queue &q, uint32_t inst0, uint32_t n, const dspi_wire_bulk_params *packets, const dspi_bulk_host *host, int exact_db,
          float fs, int32_t *results)
{
    return ingest<S>(c, q, inst0, n, host, exact_db ? kGainExact : kGainTaylor, fs, results, nullptr,
                     [&](uint32_t i0, uint32_t nc, const dspi_bulk_host **d_host) -> int {
        const size_t pb = (size_t)nc * kPacketBytes, hb = (size_t)nc * sizeof(dspi_bulk_host);
        cudaError_t e;
        if (q.lane) {
            *d_host = q.bulk.lane_host(nc);
            e = lane_upload(q, q.bulk.packets, pb + hb, [&](unsigned char *b) {
                memcpy(b, packets + i0, pb);
                memcpy(b + pb, host + i0, hb);
            });
        } else {
            e = cudaMemcpyAsync(q.bulk.packets, packets + i0, pb, cudaMemcpyHostToDevice, q.stream);
        }
        return e == cudaSuccess ? DSPI_OK : fail_cuda(e, "packet copy");
    });
}

// dspi_chain(q)_apply_preset_device for checked arguments, on queue q with its preset staging: images -> packets by
// preset_decode_kernel, then the ingest path with the flash conversion; the preset result codes go back
template <class S, class Engine, class Queue>
int apply_preset(Engine *c, Queue &q, uint32_t inst0, uint32_t n, const void *images, size_t stride, const dspi_preset_load *load,
                 const dspi_bulk_host *host, float fs, int32_t *results)
{
    constexpr size_t kSlot = sizeof(SlotOf<S>);
    PresetStage &ps = q.preset;
    cudaError_t e = ps.ensure(kSlot);
    if (e != cudaSuccess) return fail_cuda(e, "preset staging buffers");
    return ingest<S>(c, q, inst0, n, host, kGainFlash, fs, results, ps.results, [&](uint32_t i0, uint32_t nc, const dspi_bulk_host **d_host) -> int {
        cudaStream_t s = q.stream;
        const unsigned char *src = static_cast<const unsigned char *>(images) + (size_t)i0 * stride;
        const dspi_preset_load *d_load = ps.load;
        cudaError_t e;
        if (q.lane) {
            const size_t ib = (size_t)nc * kSlot, lb = (size_t)nc * sizeof(dspi_preset_load), hb = (size_t)nc * sizeof(dspi_bulk_host);
            d_load = reinterpret_cast<const dspi_preset_load *>(ps.images + ib);
            *d_host = reinterpret_cast<const dspi_bulk_host *>(ps.images + ib + lb);
            e = lane_upload(q, ps.images, ib + lb + hb, [&](unsigned char *b) {
                for (uint32_t i = 0; i < nc; i++) memcpy(b + (size_t)i * kSlot, src + (size_t)i * stride, kSlot);
                memcpy(b + ib, load + i0, lb);
                memcpy(b + ib + lb, host + i0, hb);
            });
        } else {
            e = cudaMemcpy2DAsync(ps.images, kSlot, src, stride, kSlot, nc, cudaMemcpyHostToDevice, s);
            if (e == cudaSuccess) e = cudaMemcpyAsync(ps.load, load + i0, (size_t)nc * sizeof(dspi_preset_load), cudaMemcpyHostToDevice, s);
        }
        if (e != cudaSuccess) return fail_cuda(e, "image copy");
        preset_decode_kernel<S><<<(nc + kWarps - 1) / kWarps, kWarps * 32, 0, s>>>(ps.images, d_load, nc, q.bulk.packets, ps.results);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "preset decode kernel");
        c->launches++;
        return DSPI_OK;
    });
}

// The clamped recipes dspi_chain(q)_set_eq_params_device hands back ([n][roles][12], host memory) -> the records, on the
// engine stream; returns when they are there.
template <class S, class Engine>
int record_recipes(Engine *c, uint32_t inst0, uint32_t n, const dspi_eq_param *recipes)
{
    Stage &stage = c->q.bulk;
    cudaError_t e = stage.ensure(S::kRoles);
    if (e != cudaSuccess) return fail_cuda(e, "staging buffers");
    constexpr uint32_t per = S::kRoles * kMaxBands;
    for (uint32_t i0 = 0; i0 < n; i0 += kChunk) {
        const uint32_t nc = n - i0 < kChunk ? n - i0 : kChunk;
        e = cudaMemcpyAsync(stage.recipes, recipes + (size_t)i0 * per, (size_t)nc * per * sizeof(dspi_eq_param), cudaMemcpyHostToDevice, c->q.stream);
        if (e != cudaSuccess) return fail_cuda(e, "recipe copy");
        record_recipes_kernel<<<(nc * per + 255) / 256, 256, 0, c->q.stream>>>(c->rec, inst0 + i0, nc, S::kRoles, stage.recipes, kMaxBands, per, nullptr);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "recipe record kernel");
        c->launches++;
    }
    if ((e = cudaStreamSynchronize(c->q.stream)) != cudaSuccess) return fail_cuda(e, "recipe record");
    return DSPI_OK;
}

// Whether a collect into `packets` goes through q's staging.  bulk_collect_kernel stores whole packets with bulk copies,
// which need a 16-byte aligned destination, while a dspi_wire_bulk_params pointer may hold any address (the record is
// packed).  The engine's queue always stages (the caller's memory is on the host); a lane writes the caller's device
// memory directly when the packets are 16-byte aligned, and otherwise stages and copies device to device.
template <class Queue>
bool collect_staged(const Queue &q, const void *packets)
{
    return !q.lane || ((uintptr_t)packets & 15u) != 0;
}

// dspi_chain(q)_collect_bulk_device for checked arguments, on queue q behind everything issued before it; reads only.
// Staged (collect_staged): each chunk goes to q's staging, then to the caller's host memory (the engine's queue: the call's
// end synchronises) or device memory (a lane's).  Otherwise the kernel writes the caller's device memory directly.
template <class S, class Engine, class Queue>
int collect(Engine *c, Queue &q, uint32_t inst0, uint32_t n, dspi_wire_bulk_params *packets, dspi_bulk_host *host, int32_t *results)
{
    Stage &stage = q.bulk;
    const bool staged = collect_staged(q, packets);
    cudaError_t e = staged ? stage.ensure(S::kRoles) : cudaSuccess;
    if (e != cudaSuccess) return fail_cuda(e, "staging buffers");
    cudaStream_t s = q.stream;
    const cudaMemcpyKind back = q.lane ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    for (uint32_t i0 = 0; i0 < n; i0 += kChunk) {
        const uint32_t nc = n - i0 < kChunk ? n - i0 : kChunk;
        dspi_wire_bulk_params *to_p = staged ? stage.packets : packets + i0;
        dspi_bulk_host *to_h = staged ? stage.host : host ? host + i0 : nullptr;
        int32_t *to_r = staged ? stage.results : results ? results + i0 : nullptr;
        bulk_collect_kernel<S><<<(nc + kWarps - 1) / kWarps, kWarps * 32, 0, s>>>(c->rec, inst0 + i0, nc, to_p, to_h, to_r);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "collect kernel");
        c->launches++;
        if (!staged) continue;
        e = cudaMemcpyAsync(packets + i0, stage.packets, (size_t)nc * kPacketBytes, back, s);
        if (e == cudaSuccess && host) e = cudaMemcpyAsync(host + i0, stage.host, (size_t)nc * sizeof(dspi_bulk_host), back, s);
        if (e == cudaSuccess && results) e = cudaMemcpyAsync(results + i0, stage.results, (size_t)nc * sizeof(int32_t), back, s);
        if (e != cudaSuccess) return fail_cuda(e, "packet copy");
    }
    return DSPI_OK;
}

// dspi_chain(q)_collect_preset_device for checked arguments, on queue q with its preset staging, behind everything issued
// before it; reads only.  The slot indices go up with a copy (the engine's queue) or through the lane's ring; images and
// results come back to host memory (the engine's queue; the call's end synchronises) or to device memory (a lane's).
template <class S, class Engine, class Queue>
int collect_preset(Engine *c, Queue &q, uint32_t inst0, uint32_t n, const uint8_t *slot_indices, void *images, size_t stride, int32_t *results)
{
    constexpr size_t kSlot = sizeof(SlotOf<S>);
    PresetStage &ps = q.preset;
    cudaError_t e = ps.ensure(kSlot);
    if (e != cudaSuccess) return fail_cuda(e, "preset staging buffers");
    cudaStream_t s = q.stream;
    const cudaMemcpyKind back = q.lane ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    uint8_t *slots = reinterpret_cast<uint8_t *>(ps.load);
    for (uint32_t i0 = 0; i0 < n; i0 += kChunk) {
        const uint32_t nc = n - i0 < kChunk ? n - i0 : kChunk;
        e = q.lane ? lane_upload(q, slots, nc, [&](unsigned char *b) { memcpy(b, slot_indices + i0, nc); })
                   : cudaMemcpyAsync(slots, slot_indices + i0, nc, cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return fail_cuda(e, "slot index copy");
        preset_collect_kernel<S><<<(nc + kWarps - 1) / kWarps, kWarps * 32, 0, s>>>(c->rec, inst0 + i0, nc, slots, ps.images, ps.results);
        if ((e = cudaGetLastError()) != cudaSuccess) return fail_cuda(e, "preset collect kernel");
        c->launches++;
        e = cudaMemcpy2DAsync(static_cast<unsigned char *>(images) + (size_t)i0 * stride, stride, ps.images, kSlot, kSlot, nc, back, s);
        if (e == cudaSuccess && results) e = cudaMemcpyAsync(results + i0, ps.results, (size_t)nc * sizeof(int32_t), back, s);
        if (e != cudaSuccess) return fail_cuda(e, "image copy");
    }
    return DSPI_OK;
}

}  // namespace bulk
}  // namespace dspi
