// chain_f32.cu — the whole per-packet float signal chain of one DSPi device, for thousands of
// independent device instances, sm_90a.
//
// Reference: process_audio_packet(), firmware/DSPi/usb_audio.c:500-1317 — float pipeline :560-967,
// single-core branch :874-960; crossfeed.c:132-156; leveller.c:148-262; pdm_generator.c:351-397.
// Chain order (the code's, not the README's): preamp -> loudness -> master EQ -> leveller ->
// crossfeed (+ input peaks) -> matrix -> per-output EQ -> gain x volume -> delay -> peaks ->
// 24-bit words / delta-sigma PDM.
//
// The chain is feed-forward between stages (nothing downstream feeds an upstream stage), so a call is
// run stage by stage over whole slices of packets instead of packet by packet:
//
//   chain_pre_kernel      warp = 16 instances x {L, R}: PCM unpack, preamp, the two loudness shelves; results leave
//                         through a shared-memory transpose as ROWS [2 N][frames] (row = side * N + inst)
//   K1 (eq_f32_kernel.cuh) the 10-band master EQ over those rows — the same TMA-fed two-channels-per-lane kernel
//                         (and run-time specialisation) as the EQ engine, not a second implementation
//   chain_post_kernel     warp = 16 instances x {L, R}: per-packet leveller (stereo-linked, 480-sample
//                         look-ahead ring), input peaks, crossfeed; L <-> R exchange by __shfl_xor(.., 16)
//   chain_mix_kernel      lane = frame: the 2 x 9 matrix, writes output ROWS [9 N][frames]
//   K1                    per-output EQ over the 9 N rows (muted / disabled rows are masked out)
//   chain_outpost_kernel  lane = frame, warp = (instance, packet): gain, delay, peak/clip metering,
//                         float -> 24-bit S/PDIF pairs (coalesced 8-byte stores) or, in its SUBFRAMES
//                         instantiation, those pairs encoded straight into biphase-mark subframes at the
//                         instance's S/PDIF block position and channel status (spdif_bmc.cuh, 16-byte stores),
//                         Q28 for the modulator.  A delayed sample that lies inside the current call is read
//                         from the output rows; only older history comes from the delay ring in HBM.
//   chain_ring_kernel     once per call: the last <= 4096 post-gain samples go into the rings, every
//                         instance's S/PDIF block position advances by the call's frame count
//   chain_pdm_kernel      one instance per lane: 256x oversampled 2nd-order delta-sigma (chain_pdm.cuh)
//
// Everything with a serial recurrence but little arithmetic keeps lane = instance; everything without
// one runs lane = frame, fully coalesced; the EQ — 90 % of the arithmetic — runs in the kernel that is
// tuned against the roofline.  All per-instance parameters and states are SoA arrays with the instance
// index innermost.  The host side (engine record, launch order over the stages, staging, checkpoints) is chain_host.cuh.
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "eq_kernels.cuh"
#include "bulk_ingest.cuh"
#include "chain_pdm.cuh"
#include "chain_schedule.cuh"
#include "chain_streams.cuh"
#include "dynamics.cuh"
#include "response.cuh"
#include "spdif_bmc.cuh"

namespace dspi {
namespace {

constexpr int kOuts = DSPI_CHAIN_OUTPUTS;
constexpr int kRoles = DSPI_CHAIN_EQ_CHANNELS;
constexpr int kMaxDelay = DSPI_CHAIN_MAX_DELAY;
constexpr int kLa = DSPI_LA_SAMPLES;
constexpr int kXs = 33;                           // shared-memory column stride: conflict-free for lane = instance AND lane = frame

struct ChainDev {
    uint32_t N, N_pad, nb, max_frames, ldF;       // ldF: row stride of mrow / orow / subq (frames, multiple of 4)
    float *preamp;                                // [2][N_pad]
    uint8_t *flags;                               // [N_pad] F_*
    float *loud_c; float *loud_st; uint8_t *loud_byp;   // [2 j][6][N_pad], [2 side][2 j][2][N_pad], [N_pad] bit j
    float *xf;                                    // [7][N_pad] lp_a0 lp_b1 lp_L lp_R ap_a ap_L ap_R
    float *lev_c; float *lev_s; uint32_t *lev_idx; float *lev_la;   // [9][N_pad], [5][N_pad], [N_pad], [2][480][N_pad]
    float *o_gl, *o_gr, *o_gain; uint8_t *o_flags; int32_t *o_dly;  // [9][N_pad]
    float *dline; uint32_t *widx_in, *widx_out;   // [9][N_pad][4096], [N_pad]
    int32_t *pdm;                                 // [9][N_pad] err1 err2 x1 x2 y1 y2 err_acc rng fade_in_pos
    uint16_t *peaks; uint16_t *clip;              // [11][N_pad], [N_pad]
    float *mrow;                                  // [2 N_pad][ldF] master rows, row = side * N_pad + inst
    float *orow;                                  // [9 N_pad][ldF] output rows, row = o * N_pad + inst
    int32_t *subq;                                // [N_pad][ldF] Q28 sub samples for the modulator
    uint8_t *skip_m, *skip_o;                     // [2 N_pad], [9 N_pad]: rows whose EQ is frozen (K1 skip mask)
    // preset-mute envelope (usb_audio.c:456-498): per-instance state and the per-packet volume it produces
    uint32_t *env;                                // [5][N_pad] loading, counter, smooth gain (float bits), sample rate, envelope mode on
    float *vol_base, *vol_master, *o_glin;        // [N_pad] host volume (:569), [N_pad] master volume, [9][N_pad] outputs[o].gain_linear
    float *pmg;                                   // [N_pad] the constant preset_mute_gain of dspi_chain_set_params
    float *vmm;                                   // [packets of the call][N_pad] vol_mul_master (:571) of envelope-mode instances
    const uint32_t *off;                          // [packets of the call + 1] first frame of each packet (chain_schedule.cuh)
};

// a*b + c, c - a*b in the flavour's rounding (scalar: negation is free)
template <bool FUSED> __device__ __forceinline__ float fm(float a, float b, float c)
{
    if (FUSED) return __fmaf_rn(a, b, c);
    return __fadd_rn(__fmul_rn(a, b), c);
}
template <bool FUSED> __device__ __forceinline__ float fnm(float a, float b, float c)    // c - a*b
{
    if (FUSED) return __fmaf_rn(-a, b, c);
    return __fadd_rn(c, -__fmul_rn(a, b));
}

// leveller.c:124-139
__device__ __forceinline__ float gain_computer(float x_db, float threshold, float ratio, float knee)
{
    const float half_knee = __fmul_rn(knee, 0.5f);
    if (x_db > __fadd_rn(threshold, half_knee)) return 0.0f;
    if (x_db >= __fadd_rn(threshold, -half_knee)) {
        const float dd = __fadd_rn(__fadd_rn(threshold, half_knee), -x_db);
        const float k = __fadd_rn(1.0f, -__fdiv_rn(1.0f, ratio));
        return __fdiv_rn(__fmul_rn(__fmul_rn(k, dd), dd), __fmul_rn(2.0f, knee));
    }
    return __fmul_rn(__fadd_rn(threshold, -x_db), __fadd_rn(1.0f, -__fdiv_rn(1.0f, ratio)));
}

// ---------------------------------------------------------------------------------------------
// pre: PCM unpack + preamp (usb_audio.c:591-686), loudness shelves (:689-718) -> master rows
// ---------------------------------------------------------------------------------------------
template <bool FUSED>
__global__ void __launch_bounds__(64)
chain_pre_kernel(ChainDev d, uint32_t inst0, uint32_t n, const uint8_t *__restrict__ pcm, uint32_t bit_depth, uint32_t f_begin, uint32_t f_end,
                 uint32_t F)
{
    // warp = 16 instances x {L, R}: lane l handles side l >> 4 of instance inst16 + (l & 15).  The two sides of an
    // instance share nothing in this stage (separate shelf states, usb_audio.c:696 / :707), so splitting them over two
    // lanes halves the serial chain per lane and doubles the warps of a stage that is latency-bound on few warps.
    __shared__ float tile_s[2][32][kXs];                  // per warp: [frame][row = side * 16 + instance]
    __shared__ uint32_t pcm_s[2][2][16][49];              // per warp, double-buffered: 16 instances x 32 frames x <= 6 bytes (rows padded to 49 words)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // instances [inst0, inst0 + n) of the engine, PCM rows and warps counted from inst0; warps cover n rounded up to 32
    // instances, the lanes past n are not live and leave every state alone
    const uint32_t local16 = (blockIdx.x * 2 + warp) * 16;
    if (local16 >= ((n + 31) & ~31u)) return;
    const uint32_t side = lane >> 4, li = lane & 15;
    const uint32_t inst16 = inst0 + local16, inst = inst16 + li;
    const bool live = local16 + li < n;
    const uint32_t Np = d.N_pad;
    float (*tile)[kXs] = tile_s[warp];

    const bool loud_on = d.flags[inst] & F_LOUD;
    const uint8_t loud_byp = d.loud_byp[inst];
    float lc[2][6], ls[2][2];
#pragma unroll
    for (int j = 0; j < 2; j++) {
#pragma unroll
        for (int k = 0; k < 6; k++) lc[j][k] = d.loud_c[(j * 6 + k) * Np + inst];
        ls[j][0] = d.loud_st[((side * 2 + j) * 2 + 0) * Np + inst];
        ls[j][1] = d.loud_st[((side * 2 + j) * 2 + 1) * Np + inst];
    }
    const uint32_t bpf = bit_depth == 24 ? 6u : 4u;
    const float preamp = d.preamp[side * Np + inst];
    const float gain_in = bit_depth == 24 ? __fmul_rn(1.0f / 8388608.0f, preamp)        // usb_audio.c:601-603
                                          : __fmul_rn(1.0f / 32768.0f, preamp);          // :680-681
    // Each instance's packet stream is contiguous ([inst][F] frames of bpf bytes); when every tile starts on
    // a 4-byte boundary the warp fetches the 16 tiles of its instances with coalesced word loads into shared
    // memory and every lane then decodes its own side from there, otherwise lanes read their bytes directly.
    const bool words_ok = ((reinterpret_cast<uintptr_t>(pcm) | ((size_t)F * bpf) | ((size_t)f_begin * bpf)) & 3u) == 0;
    const uint8_t *my_pcm = pcm + (size_t)(local16 + li) * F * bpf;
    const uint32_t n_inst = min(16u, n > local16 ? n - local16 : 0u);
    // asynchronous fetch of the tile starting at frame f0 into buffer `buf` (one commit group per call).  A last
    // word may run <= 2 bytes past a ragged tile: still inside the PCM buffer, because the very end of the
    // buffer is word-aligned (F * bpf is) and so is every tile start.
    auto fetch = [&](uint32_t f0, int buf) {
        if (words_ok && f0 < f_end) {
            const uint32_t nwords = (min(32u, f_end - f0) * bpf + 3) / 4;
            for (uint32_t i = 0; i < n_inst; i++) {
                const uint32_t *src = reinterpret_cast<const uint32_t *>(pcm + ((size_t)(local16 + i) * F + f0) * bpf);
                for (uint32_t w = lane; w < nwords; w += 32) cp_async_4(&pcm_s[warp][buf][i][w], src + w);
            }
        }
        cp_async_commit();
    };
    fetch(f_begin, 0);

    int buf = 0;
    for (uint32_t f0 = f_begin; f0 < f_end; f0 += 32, buf ^= 1) {
        const uint32_t nv = min(32u, f_end - f0);
        const uint8_t *tile_bytes = my_pcm + (size_t)f0 * bpf;
        fetch(f0 + 32, buf ^ 1);                          // next tile streams in behind this tile's arithmetic
        if (words_ok) {
            cp_async_wait<1>();
            __syncwarp();
            tile_bytes = reinterpret_cast<const uint8_t *>(pcm_s[warp][buf][li]);
        }
        for (uint32_t t = 0; t < nv; t++) {
            const uint8_t *q = tile_bytes + (size_t)t * bpf;
            int32_t sm = 0;
            if (live) {
                if (bit_depth == 24) {
                    const uint8_t *b = q + side * 3;
                    sm = ((int32_t)((uint32_t)b[2] << 24 | (uint32_t)b[1] << 16 | (uint32_t)b[0] << 8)) >> 8;
                } else {
                    const uint8_t *b = q + side * 2;
                    sm = (int16_t)((uint16_t)b[0] | (uint16_t)b[1] << 8);
                }
            }
            float v = __fmul_rn((float)sm, gain_in);                         // :645-648 / :683-684
            if (loud_on) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    if ((loud_byp >> j) & 1) continue;
                    float &s0 = ls[j][0], &s1 = ls[j][1];
                    const float v3 = __fadd_rn(v, -s1);
                    const float pp = __fmul_rn(lc[j][1], v3);
                    float t2, v1, v2;
                    if (FUSED) {
                        t2 = __fmaf_rn(lc[j][1], s0, s1);
                        v1 = __fmaf_rn(lc[j][0], s0, pp);
                        v2 = __fmaf_rn(lc[j][2], v3, t2);
                    } else {
                        t2 = __fadd_rn(s1, __fmul_rn(lc[j][1], s0));
                        v1 = __fadd_rn(__fmul_rn(lc[j][0], s0), pp);
                        v2 = __fadd_rn(t2, __fmul_rn(lc[j][2], v3));
                    }
                    s0 = __fmaf_rn(2.0f, v1, -s0);
                    s1 = __fmaf_rn(2.0f, v2, -s1);
                    v = fm<FUSED>(lc[j][5], v2, fm<FUSED>(lc[j][3], v, __fmul_rn(lc[j][4], v1)));   // :702
                }
            }
            tile[t][lane] = v;
        }
        __syncwarp();
        // transpose out: lane = frame, one coalesced 128-byte store per (side, instance) row
        if ((uint32_t)lane < nv) {
#pragma unroll 8
            for (int r = 0; r < 32; r++)
                d.mrow[((size_t)(r >> 4) * Np + inst16 + (r & 15)) * d.ldF + f0 + lane] = tile[lane][r];
        }
        __syncwarp();
    }
    if (!live) return;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        d.loud_st[((side * 2 + j) * 2 + 0) * Np + inst] = ls[j][0];
        d.loud_st[((side * 2 + j) * 2 + 1) * Np + inst] = ls[j][1];
    }
}

// ---------------------------------------------------------------------------------------------
// post: leveller (leveller.c:148-262), input peaks, crossfeed (crossfeed.c:132-156), packet by packet
// ---------------------------------------------------------------------------------------------
template <bool FUSED>
__global__ void __launch_bounds__(128)
chain_post_kernel(ChainDev d, uint32_t inst0, uint32_t n, uint32_t p0, uint32_t n_packets, uint32_t longest)
{
    extern __shared__ float smem[];                       // per warp: packet columns [longest][33] + look-ahead reads [longest][33]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t side = lane >> 4;
    const uint32_t local16 = (blockIdx.x * (blockDim.x >> 5) + warp) * 16;      // instances [inst0, inst0 + n): see chain_pre_kernel
    if (local16 >= ((n + 31) & ~31u)) return;
    const uint32_t inst16 = inst0 + local16, inst = inst16 + (lane & 15);
    const bool live = local16 + (lane & 15) < n;
    const uint32_t Np = d.N_pad;
    float *xw = smem + (size_t)warp * 2 * longest * kXs;  // xw[t * 33 + r]: column r of this warp
    float *xs = xw + lane;                                // own column
    float *hs = xw + (size_t)longest * kXs + lane;        // held look-ahead samples, own column

    const uint8_t flags = live ? d.flags[inst] : 0;       // lanes past the range run with every stage off
    const bool lev_on = flags & F_LEV, xf_on = flags & F_XFEED, lookahead = flags & F_LOOKAHEAD;
    // crossfeed: this lane owns its side's lowpass / all-pass state
    const float xf_a0 = d.xf[0 * Np + inst], xf_b1 = d.xf[1 * Np + inst], xf_ap = d.xf[4 * Np + inst];
    float xf_lp = d.xf[(2 + side) * Np + inst], xf_as = d.xf[(5 + side) * Np + inst];
    float lvc[9];
#pragma unroll
    for (int k = 0; k < 9; k++) lvc[k] = d.lev_c[k * Np + inst];
    float env = d.lev_s[side * Np + inst];
    float smooth_db = d.lev_s[2 * Np + inst], gain_lin = d.lev_s[3 * Np + inst], gain_prev = d.lev_s[4 * Np + inst];
    uint32_t la_idx = d.lev_idx[inst];
    float *la_buf = d.lev_la + (size_t)side * kLa * Np + inst;

    float peak_in = 0.0f;
    uint16_t clip = 0;
    for (uint32_t p = p0; p < p0 + n_packets; p++) {
        const uint32_t f0 = d.off[p], count = d.off[p + 1] - f0;          // the leveller's block is this packet
        // The look-ahead ring is read one slot per sample, each read just before that slot is overwritten
        // (leveller.c:231-237), and a packet (<= 192 frames) never laps the 480-slot ring: all of this
        // packet's reads are issued now as asynchronous copies, together with the packet itself.
        if (lev_on && lookahead) {
            uint32_t idx = la_idx;
            for (uint32_t i = 0; i < count; i++) {
                cp_async_4(hs + i * kXs, la_buf + (size_t)idx * Np);
                if (++idx >= (uint32_t)kLa) idx = 0;
            }
        }
        // packet in: lane = frame, coalesced row reads, transposed into lane-private columns (asynchronous
        // copies again: 32 rows x count/32 independent requests in flight instead of one load-store pair at a time)
        for (int r = 0; r < 32; r++) {
            const float *row = d.mrow + ((size_t)(r >> 4) * Np + inst16 + (r & 15)) * d.ldF + f0;
            for (uint32_t t = lane; t < count; t += 32) cp_async_4(xw + t * kXs + r, row + t);
        }
        cp_async_commit();
        cp_async_wait_all();
        __syncwarp();

        // ---- PASS 3 for one sample: input peak, then crossfeed (usb_audio.c:741-749); every lane walks the same shuffle ----
        float pk = 0.0f;
        auto peak_and_crossfeed = [&](uint32_t i, float v) {
            const float a = fabsf(v);
            if (a > pk) pk = a;
            float lp = 0.0f, ap = 0.0f;
            if (xf_on) {
                lp = fm<FUSED>(xf_a0, v, __fmul_rn(xf_b1, xf_lp));           // crossfeed.c:137-138
                xf_lp = lp;
                ap = fm<FUSED>(xf_ap, lp, xf_as);                            // :146 / :148
                xf_as = fnm<FUSED>(xf_ap, ap, lp);                           // :147 / :149
            }
            const float ap_other = __shfl_xor_sync(0xffffffffu, ap, 16);
            if (xf_on) v = __fadd_rn(__fadd_rn(v, -lp), ap_other);           // :154-155
            xs[i * kXs] = v;
        };

        // ---- PASS 2.5: leveller ----
        if (__any_sync(0xffffffffu, lev_on)) {
            const float a_rms = lvc[0], one_minus = __fadd_rn(1.0f, -a_rms);
            float e = env;
            for (uint32_t i = 0; i < count; i++) {                             // leveller.c:161-166
                const float s = xs[i * kXs];
                e = fm<FUSED>(a_rms, e, __fmul_rn(one_minus, __fmul_rn(s, s)));
            }
            if (e < 1e-30f) e = 0.0f;                                        // :169-170
            const float e_other = __shfl_xor_sync(0xffffffffu, e, 16);
            const float env_l = side ? e_other : e, env_r = side ? e : e_other;
            const float rms_sq = (env_l > env_r) ? env_l : env_r;            // :177
            // per-block libm: evaluated in double and rounded once (DESIGN.md "libm policy")
            const float rms_db = __fmul_rn(10.0f, (float)log10((double)__fadd_rn(rms_sq, 1e-30f)));
            float gc_db;
            if (rms_db < lvc[7]) gc_db = 0.0f;
            else {
                gc_db = gain_computer(rms_db, lvc[3], lvc[4], lvc[5]);
                gc_db = __fadd_rn(gc_db, lvc[6]);
                if (gc_db > lvc[8]) gc_db = lvc[8];
            }
            const float alpha_s = (gc_db < smooth_db) ? lvc[1] : lvc[2];     // :198
            const float alpha = (float)pow((double)alpha_s, (double)(float)count);
            const float new_smooth = fm<FUSED>(alpha, smooth_db, __fmul_rn(__fadd_rn(1.0f, -alpha), gc_db));
            const float new_gain = (float)pow(10.0, (double)__fdiv_rn(new_smooth, 20.0f));
            // every lane walks the same shuffles; only instances with the leveller on commit results
            const float prev_for_ramp = gain_lin;
            float gain, gain_step;
            if (count == 1) { gain = new_gain; gain_step = 0.0f; }
            else { gain_step = __fdiv_rn(__fadd_rn(new_gain, -prev_for_ramp), (float)(count - 1)); gain = prev_for_ramp; }
            // the leveller's per-sample part and PASS 3 share one loop: ramp, look-ahead exchange and peak limit of sample
            // i+1 do not depend on the crossfeed recurrence of sample i, so the serial chains overlap
            for (uint32_t i = 0; i < count; i++) {                             // :228-259, then usb_audio.c:741-749
                const float x0 = xs[i * kXs];
                float o = x0;
                if (lev_on && lookahead) {
                    const float held = hs[i * kXs];
                    la_buf[(size_t)la_idx * Np] = o;
                    o = held;
                    la_idx++;
                    if (la_idx >= (uint32_t)kLa) la_idx = 0;
                }
                const float ao = fabsf(o);
                const float ao_other = __shfl_xor_sync(0xffffffffu, ao, 16);
                const float al = side ? ao_other : ao, ar = side ? ao : ao_other;
                float peak = al;
                if (ar > peak) peak = ar;
                float g = gain;
                if (peak > 0.0f && g > 1.0f) {
                    const float max_g = __fdiv_rn(0.70795f, peak);
                    if (max_g < g) g = (max_g > 1.0f) ? max_g : 1.0f;
                }
                gain = __fadd_rn(gain, gain_step);
                peak_and_crossfeed(i, lev_on ? __fmul_rn(o, g) : x0);
            }
            if (lev_on) {
                env = e;
                smooth_db = new_smooth;
                gain_prev = gain_lin;
                gain_lin = new_gain;
            }
        } else {
            for (uint32_t i = 0; i < count; i++) peak_and_crossfeed(i, xs[i * kXs]);
        }
        peak_in = pk;                                                        // peaks describe the last packet
        if (pk > 1.001f) clip |= (uint16_t)(1u << side);                     // config.h:53
        __syncwarp();
        // packet out: back into the same rows, coalesced
        for (uint32_t t = lane; t < count; t += 32) {
#pragma unroll 8
            for (int r = 0; r < 32; r++)
                d.mrow[((size_t)(r >> 4) * Np + inst16 + (r & 15)) * d.ldF + f0 + t] = xw[t * kXs + r];
        }
        __syncwarp();
    }

    // ---- state back ----
    const uint16_t clip_other = (uint16_t)__shfl_xor_sync(0xffffffffu, (uint32_t)clip, 16);
    if (!live) return;
    d.xf[(2 + side) * Np + inst] = xf_lp;
    d.xf[(5 + side) * Np + inst] = xf_as;
    d.lev_s[side * Np + inst] = env;
    if (side == 0) {
        d.lev_s[2 * Np + inst] = smooth_db;
        d.lev_s[3 * Np + inst] = gain_lin;
        d.lev_s[4 * Np + inst] = gain_prev;
        d.lev_idx[inst] = la_idx;
    }
    d.peaks[side * Np + inst] = (uint16_t)__fmul_rn(fminf(1.0f, peak_in), 32767.0f);    // usb_audio.c:963-964
    // clip_flags bits 0/1: the two sides of one instance sit in lanes l and l+16; two instances share a 32-bit word
    if (side == 0 && (clip | clip_other)) atomicOr(reinterpret_cast<unsigned int *>(d.clip + (inst & ~1u)), (unsigned int)(clip | clip_other) << (16 * (inst & 1)));
}

// ---------------------------------------------------------------------------------------------
// matrix mix (usb_audio.c:753-779): lane = frame
// ---------------------------------------------------------------------------------------------
template <bool FUSED>
__global__ void __launch_bounds__(256)
chain_mix_kernel(ChainDev d, uint32_t inst0, uint32_t n, uint32_t f_begin, uint32_t f_end)
{
    const int lane = threadIdx.x & 31;
    constexpr int kB = 4;                                  // frames per lane per unit: kB independent loads in flight
    const uint32_t n_tiles = (f_end - f_begin + 32 * kB - 1) / (32 * kB);
    const uint64_t units = (uint64_t)n * n_tiles;
    const uint32_t Np = d.N_pad;
    for (uint64_t u = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < units; u += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint32_t inst = inst0 + (uint32_t)(u / n_tiles), tile = (uint32_t)(u % n_tiles);
        const uint32_t fbase = f_begin + tile * 32 * kB + lane;
        float l[kB], r[kB];
#pragma unroll
        for (int j = 0; j < kB; j++) {
            const uint32_t f = fbase + 32 * j;
            l[j] = f < f_end ? d.mrow[(size_t)inst * d.ldF + f] : 0.0f;
            r[j] = f < f_end ? d.mrow[((size_t)Np + inst) * d.ldF + f] : 0.0f;
        }
#pragma unroll
        for (int o = 0; o < kOuts; o++) {
            const bool enabled = d.o_flags[o * Np + inst] & O_ENABLED;
            const float gl = d.o_gl[o * Np + inst], gr = d.o_gr[o * Np + inst];
            const int mixcase = !enabled ? 0 : (gl != 0.0f && gr != 0.0f) ? 3 : (gl != 0.0f) ? 1 : (gr != 0.0f) ? 2 : 0;   // :767-778
#pragma unroll
            for (int j = 0; j < kB; j++) {
                float v;
                if (mixcase == 3) v = fm<FUSED>(l[j], gl, __fmul_rn(r[j], gr));          // :769
                else if (mixcase == 1) v = __fmul_rn(l[j], gl);
                else if (mixcase == 2) v = __fmul_rn(r[j], gr);
                else v = 0.0f;
                const uint32_t f = fbase + 32 * j;
                if (f < f_end) d.orow[((size_t)o * Np + inst) * d.ldF + f] = v;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// outputs after the EQ: gain (:885-894), delay (:898-912), peaks (:914-923), 24-bit / Q28 (:925-959)
// ---------------------------------------------------------------------------------------------
// update_preset_mute_envelope() (usb_audio.c:466-498) for every packet of the call, one instance per thread, and the
// volume chain of :569-571 that depends on it: vmm[p] = (vol_base * g_p) * master_volume_linear.  Same operations, same
// order as dspi_preset_mute_step() on the host.
__global__ void chain_env_kernel(ChainDev d, uint32_t inst0, uint32_t n, uint32_t n_packets)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, inst = inst0 + i;
    const uint32_t Np = d.N_pad;
    if (i >= n || !d.env[4 * Np + inst]) return;
    uint32_t loading = d.env[0 * Np + inst], counter = d.env[1 * Np + inst];
    float g = __uint_as_float(d.env[2 * Np + inst]);
    const uint32_t fs = d.env[3 * Np + inst];
    unsigned long long ts = ((unsigned long long)fs * 8ull + 999ull) / 1000ull;          // :459-464
    if (ts < 1ull) ts = 1ull;
    if (ts > 0xFFFFFFFFull) ts = 0xFFFFFFFFull;
    const float vol_base = d.vol_base[inst], master = d.vol_master[inst];
    for (uint32_t p = 0; p < n_packets; p++) {
        const uint32_t count = d.off[p + 1] - d.off[p];                                  // sample_count of this packet
        float step = __fdiv_rn((float)count, (float)(uint32_t)ts);                       // :486
        if (step > 1.0f) step = 1.0f;
        const bool active = loading != 0;                                                // :469
        if (active) {
            if (counter > count) counter -= count;
            else { counter = 0; loading = 0; }
        }
        const float target = active ? 0.0f : 1.0f;
        if (g < target)      { g = __fadd_rn(g, step);  if (g > target) g = target; }
        else if (g > target) { g = __fadd_rn(g, -step); if (g < target) g = target; }
        d.vmm[(size_t)p * Np + inst] = __fmul_rn(__fmul_rn(vol_base, g), master);        // :570-571
    }
    d.env[0 * Np + inst] = loading;
    d.env[1 * Np + inst] = counter;
    d.env[2 * Np + inst] = __float_as_uint(g);
}

// The float stores of device-side parameter ingest, shared by chain_dynamics_kernel and the bulk ingest kernel
// (bulk_ingest.cuh): one instance per call, written straight into the engine's arrays.
struct ParamStores {
    using Dev = ChainDev;
    static constexpr int kRoles = dspi::kRoles, kOuts = dspi::kOuts, kMaxDelay = dspi::kMaxDelay, kPlatformId = 1;
    static constexpr bool kQ28 = false;
    // crossfeed_compute_coefficients(): coefficients and CLEARED filter state (crossfeed.c:110-126)
    static __device__ void crossfeed(const ChainDev &d, uint32_t inst, const dspi_crossfeed_config &cfg, float fs)
    {
        const uint32_t Np = d.N_pad;
        float a0, b1, ap;
        dyn::crossfeed_coeffs(cfg, fs, a0, b1, ap);
        d.xf[0 * Np + inst] = a0; d.xf[1 * Np + inst] = b1; d.xf[4 * Np + inst] = ap;
        d.xf[2 * Np + inst] = 0.0f; d.xf[3 * Np + inst] = 0.0f; d.xf[5 * Np + inst] = 0.0f; d.xf[6 * Np + inst] = 0.0f;
    }
    // leveller_compute_coefficients()
    static __device__ void leveller(const ChainDev &d, uint32_t inst, const dspi_leveller_config &cfg, float fs)
    {
        float lv[9];
        dyn::leveller_coeffs(cfg, fs, lv);
#pragma unroll
        for (int k = 0; k < 9; k++) d.lev_c[k * d.N_pad + inst] = lv[k];
    }
    // loudness_recompute_table() for the table row audio_set_volume() selected
    static __device__ void loudness(const ChainDev &d, uint32_t inst, uint32_t row, float ref_spl, float intensity_pct, float fs)
    {
        const uint32_t Np = d.N_pad;
        float lo_db, hi_db;
        dyn::loudness_row_gains((int)row, ref_spl, intensity_pct, lo_db, hi_db);
        float c[6];
        bool byp;
        uint8_t lb = 0;
        const float lfs = fs < 1.0f ? 48000.0f : fs;                         // loudness.c:171
        dyn::shelf_svf(200.0f, 0.707f, lo_db, false, lfs, c, byp);
        if (byp) lb |= 1;
#pragma unroll
        for (int k = 0; k < 6; k++) d.loud_c[(0 * 6 + k) * Np + inst] = c[k];
        dyn::shelf_svf(6000.0f, 0.707f, hi_db, true, lfs, c, byp);
        if (byp) lb |= 2;
#pragma unroll
        for (int k = 0; k < 6; k++) d.loud_c[(1 * 6 + k) * Np + inst] = c[k];
        d.loud_byp[inst] = lb;
    }
    // host volume -> output gains (usb_audio.c:569-571, 886-887), from the gain rows in force
    static __device__ void host_volume(const ChainDev &d, uint32_t inst, int16_t vol_mul, bool host_mute)
    {
        const uint32_t Np = d.N_pad;
        const float vol_base = host_mute ? 0.0f : __fmul_rn((float)vol_mul, 1.0f / 32768.0f);
        d.vol_base[inst] = vol_base;
        const float vmm = __fmul_rn(__fmul_rn(vol_base, d.pmg[inst]), d.vol_master[inst]);
        for (int o = 0; o < dspi::kOuts; o++)
            d.o_gain[o * Np + inst] = (d.o_flags[o * Np + inst] & O_MUTE) ? 0.0f : __fmul_rn(d.o_glin[o * Np + inst], vmm);
    }
    // what dspi_chain_set_params stores for the preamp, the master volume and one crosspoint (usb_audio.c:760-764)
    static __device__ void preamp(const ChainDev &d, uint32_t inst, uint32_t side, float linear) { d.preamp[side * d.N_pad + inst] = linear; }
    static __device__ void master_volume(const ChainDev &d, uint32_t inst, float linear) { d.vol_master[inst] = linear; }
    static __device__ void crosspoint(const ChainDev &d, uint32_t inst, uint32_t side, uint32_t o, bool enabled, bool invert, float linear)
    {
        (side ? d.o_gr : d.o_gl)[o * d.N_pad + inst] = enabled ? (invert ? -linear : linear) : 0.0f;
    }
    static __host__ __device__ bool output_eq_frozen(bool enabled, bool mute, bool) { return !enabled || mute; }   // :878-884
};

// Mass reconfiguration of the dynamics stages on the device (SURVEY f-1): what the main loop does for one instance when
// crossfeed_update_pending / leveller_update_pending / loudness_recompute_pending are set (main.c:868-895) plus
// audio_set_volume() (usb_audio.c:428-440), one instance per thread.
__global__ void chain_dynamics_kernel(ChainDev d, bulk::Record rec, uint32_t inst0, uint32_t n, const dspi_dynamics_config *__restrict__ cfgs, float fs)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t inst = inst0 + i;
    const dspi_dynamics_config cfg = cfgs[i];
    uint8_t flags = d.flags[inst] & (uint8_t)~(F_XFEED | F_LEV | F_LOOKAHEAD | F_LOUD);
    ParamStores::crossfeed(d, inst, cfg.crossfeed, fs);
    if (cfg.crossfeed.enabled) flags |= F_XFEED;                             // crossfeed_bypassed = !enabled, main.c:882
    ParamStores::leveller(d, inst, cfg.leveller, fs);                        // leveller_bypassed = !enabled, main.c:886-894
    if (cfg.leveller.enabled) flags |= F_LEV;
    if (cfg.leveller.lookahead) flags |= F_LOOKAHEAD;
    uint32_t row;
    const int16_t vol_mul = dyn::host_volume(cfg.volume_8_8, row);
    ParamStores::loudness(d, inst, row, cfg.loudness_ref_spl, cfg.loudness_intensity_pct, fs);
    if (cfg.loudness_enabled) flags |= F_LOUD;
    d.flags[inst] = flags;
    ParamStores::host_volume(d, inst, vol_mul, cfg.host_mute != 0);
    bulk::record_dynamics(rec, inst, cfg);
}

// post-gain sample of output row `o` (what the delay line stores)
__device__ __forceinline__ float out_gain(float v, bool enabled, float gain)
{
    if (enabled) {
        if (gain == 0.0f) v = 0.0f;
        else if (gain != 1.0f) v = __fmul_rn(v, gain);
    }
    return v;
}

struct OutCfg {
    bool enabled, pair_off, delay_on, mute;
    float gain;                        // constant gain of the call (no envelope)
    float glin;                        // outputs[o].gain_linear
    const float *vmm;                  // envelope mode: vol_mul_master per packet, stride N_pad; else nullptr
    const uint32_t *off;               // packet offsets of the call
    uint32_t Np;
    uint32_t dl;                       // delay & (MAX - 1): MAX aliases to 0 (SURVEY a-10)
    const float *row;                  // orow row of this (output, instance)
    const float *ring;
};

__device__ __forceinline__ OutCfg out_cfg(const ChainDev &d, uint32_t o, uint32_t inst, bool any_delay)
{
    OutCfg c;
    const uint32_t Np = d.N_pad;
    const uint8_t of = d.o_flags[o * Np + inst];
    const int32_t dly = d.o_dly[o * Np + inst];
    c.enabled = of & O_ENABLED;
    c.pair_off = of & O_PAIR_OFF;
    c.mute = of & O_MUTE;
    c.gain = d.o_gain[o * Np + inst];
    c.glin = d.o_glin[o * Np + inst];
    c.vmm = d.env[4 * Np + inst] ? d.vmm + inst : nullptr;
    c.off = d.off;
    c.Np = Np;
    c.delay_on = any_delay && dly > 0;                                       // usb_audio.c:898-901
    c.dl = (uint32_t)dly & (kMaxDelay - 1);
    c.row = d.orow + ((size_t)o * Np + inst) * d.ldF;
    c.ring = d.dline + ((size_t)o * Np + inst) * kMaxDelay;
    return c;
}

// output gain in force at frame T of the call (usb_audio.c:886-887): constant, or following the envelope packet by packet;
// p is the packet of T or a later one
__device__ __forceinline__ float gain_at(const OutCfg &c, uint32_t T, uint32_t p)
{
    if (!c.vmm) return c.gain;
    return c.mute ? 0.0f : __fmul_rn(c.glin, c.vmm[(size_t)packet_of(c.off, T, p) * c.Np]);
}

// the sample output `c` emits at frame T (in packet p) of this call (T counted from the start of the call):
// write-then-read per sample (:902-909) means frame T emits the post-gain sample of frame T - dl;
// inside the call that sample is still in the output rows, before it only the ring has it
__device__ __forceinline__ float out_sample(const OutCfg &c, uint32_t T, uint32_t p, uint32_t widx0)
{
    if (!c.delay_on) return out_gain(c.row[T], c.enabled, gain_at(c, T, p));
    if (T >= c.dl) return out_gain(c.row[T - c.dl], c.enabled, gain_at(c, T - c.dl, p));
    return c.ring[(widx0 + T - c.dl) & (kMaxDelay - 1)];
}

__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        const float o = __shfl_xor_sync(0xffffffffu, v, s);
        if (o > v) v = o;
    }
    return v;
}

// Instances [inst0, inst0 + n); the caller's rows are counted from inst0.
// SUBFRAMES = false: spdif_out is [n][4][F][2] int32 words.  SUBFRAMES = true: it is [n][4][F] uint4 subframe pairs
// {l, h, l, h}, each instance's frames encoded at its own block position and channel status (spdif_bmc.cuh) - what
// dspi_spdif_encode_* makes of the words, without the words buffer.
template <bool SUBFRAMES>
__global__ void __launch_bounds__(256)
chain_outpost_kernel(ChainDev d, uint32_t inst0, uint32_t n, uint32_t p0, uint32_t n_packets, uint32_t F, int32_t *__restrict__ spdif_out, SpdifTx tx)
{
    const int lane = threadIdx.x & 31;
    const uint64_t units = (uint64_t)(inst0 + n) * n_packets;              // units (instance, packet) of the range
    const uint32_t Np = d.N_pad;
    for (uint64_t u = (uint64_t)inst0 * n_packets + blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < units; u += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint32_t inst = (uint32_t)(u / n_packets), p = p0 + (uint32_t)(u % n_packets);
        const uint32_t f0 = d.off[p], count = d.off[p + 1] - f0;
        const bool last = p == p0 + n_packets - 1;
        const bool any_delay = d.flags[inst] & F_ANY_DELAY;
        const uint32_t widx0 = d.widx_in[inst];
        const uint32_t bp = SUBFRAMES ? tx.bp[inst] : 0u;
        const uint64_t cs40 = SUBFRAMES ? tx.cs40[inst] : 0ull;
        unsigned int clip = 0;
        for (int k = 0; k <= 4; k++) {                                        // four S/PDIF pairs, then the sub alone
            const bool is_sub = k == 4;
            const uint32_t oa = 2 * k, ob = is_sub ? oa : oa + 1;
            const OutCfg ca = out_cfg(d, oa, inst, any_delay), cb = out_cfg(d, ob, inst, any_delay);
            float pka = 0.0f, pkb = 0.0f;
            constexpr int kB = 4;                                            // independent loads in flight per lane
            for (uint32_t tb = lane; tb < count; tb += 32 * kB) {
                float xa[kB], xb[kB];
#pragma unroll
                for (int j = 0; j < kB; j++) {
                    const uint32_t t = tb + 32 * j;
                    xa[j] = t < count ? out_sample(ca, f0 + t, p, widx0) : 0.0f;
                    xb[j] = (!is_sub && t < count) ? out_sample(cb, f0 + t, p, widx0) : 0.0f;
                }
#pragma unroll
                for (int j = 0; j < kB; j++) {
                    const uint32_t t = tb + 32 * j, T = f0 + t;
                    if (t >= count) break;
                    const float aa = fabsf(xa[j]), ab = fabsf(xb[j]);
                    if (aa > pka) pka = aa;
                    if (ab > pkb) pkb = ab;
                    if (is_sub) {
                        if (ca.enabled) d.subq[(size_t)inst * d.ldF + T] = __float2int_rz(__fmul_rn(xa[j], 268435456.0f));   // :953 (saturating)
                    } else if (spdif_out) {
                        int2 w = make_int2(0, 0);
                        if (!ca.pair_off) {                                  // :930-939 (pair_off is a property of the pair)
                            w.x = __float2int_rz(__fmul_rn(fmaxf(-1.0f, fminf(1.0f, xa[j])), 8388607.0f));
                            w.y = __float2int_rz(__fmul_rn(fmaxf(-1.0f, fminf(1.0f, xb[j])), 8388607.0f));
                        }
                        if (SUBFRAMES) {                                      // 16 bytes per lane: 512 contiguous bytes per warp store
                            const uint32_t pos = (bp + T) % 192u;
                            reinterpret_cast<uint4 *>(spdif_out)[((size_t)(inst - inst0) * 4 + k) * F + T] = encode_frame(w, spdif_pre_left(pos), spdif_cs_bit(pos, cs40));
                        } else {
                            *reinterpret_cast<int2 *>(spdif_out + (((size_t)(inst - inst0) * 4 + k) * F + T) * 2) = w;
                        }
                    }
                }
            }
            pka = warp_max(pka);
            pkb = warp_max(pkb);
            if (lane == 0) {
                if (last) {
                    uint16_t pq = (uint16_t)__fmul_rn(fminf(1.0f, pka), 32767.0f);              // :921 / :950
                    if (is_sub && !ca.enabled) pq = 0;                                           // :957
                    d.peaks[(2 + oa) * Np + inst] = pq;
                    if (!is_sub) d.peaks[(2 + ob) * Np + inst] = (uint16_t)__fmul_rn(fminf(1.0f, pkb), 32767.0f);
                }
                if (pka > 1.001f && (!is_sub || ca.enabled)) clip |= 1u << (2 + oa);
                if (!is_sub && pkb > 1.001f) clip |= 1u << (2 + ob);
            }
        }
        if (lane == 0 && clip) atomicOr(reinterpret_cast<unsigned int *>(d.clip + (inst & ~1u)), clip << (16 * (inst & 1)));
    }
}

// once per call, after every outpost launch of the call: the delay rings of instances [inst0, inst0 + n) take the last
// <= 4096 post-gain samples (older writes of this call would have been overwritten anyway), the shared write index advances
// (into widx_out), and so does the S/PDIF block position - by all F frames whatever the call copied out (the transmitter
// sends every frame)
__global__ void __launch_bounds__(256)
chain_ring_kernel(ChainDev d, uint32_t inst0, uint32_t n, uint32_t F, uint32_t n_packets, uint32_t *__restrict__ spdif_bp)
{
    const int lane = threadIdx.x & 31;
    const uint64_t units = (uint64_t)n * kOuts;
    const uint32_t Np = d.N_pad;
    for (uint64_t u = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < units; u += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint32_t inst = inst0 + (uint32_t)(u / kOuts), o = (uint32_t)(u % kOuts);
        const bool any_delay = d.flags[inst] & F_ANY_DELAY;
        const uint32_t widx0 = d.widx_in[inst];
        const OutCfg c = out_cfg(d, o, inst, any_delay);
        if (c.delay_on) {                                                    // outputs without delay never touch their ring
            float *ring = d.dline + ((size_t)o * Np + inst) * kMaxDelay;
            for (uint32_t T = (F > (uint32_t)kMaxDelay ? F - kMaxDelay : 0u) + lane; T < F; T += 32)
                ring[(widx0 + T) & (kMaxDelay - 1)] = out_gain(c.row[T], c.enabled, gain_at(c, T, n_packets - 1));
        }
        if (o == 0 && lane == 0) {
            d.widx_out[inst] = any_delay ? (widx0 + F) & (kMaxDelay - 1) : widx0;   // :911, once per packet
            spdif_bp[inst] = (spdif_bp[inst] + F % 192u) % 192u;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// delta-sigma PDM (chain_pdm.cuh): one instance per lane
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
chain_pdm_kernel(ChainDev d, uint32_t inst0, uint32_t n, uint32_t f_begin, uint32_t f_end, uint32_t F, uint32_t *__restrict__ pdm_out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, inst = inst0 + i;
    if (i >= n) return;
    if (!(d.flags[inst] & F_SUB_ON)) return;                                 // usb_audio.c:944
    pdm_modulate_frames(d.pdm, d.subq + (size_t)inst * d.ldF, 1, d.N_pad, inst, f_begin, f_end, pdm_out ? pdm_out + (size_t)i * F * 8 : nullptr);
}

// filters[][] of n instances (instance-major AoS) <-> the mirrors of the two EQ engines (channel = role' * N_pad + inst)
__global__ void chain_scatter_kernel(const dspi_biquad_f32 *__restrict__ aos, uint32_t inst0, uint32_t n, uint32_t Np, dspi_biquad_f32 *__restrict__ m_aos,
                                     dspi_biquad_f32 *__restrict__ o_aos, int to_mirrors)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * kRoles * kMaxBands) return;
    const uint32_t b = i % kMaxBands, role = (i / kMaxBands) % kRoles, inst = inst0 + i / (kMaxBands * kRoles);
    dspi_biquad_f32 *chain_q = const_cast<dspi_biquad_f32 *>(aos) + ((size_t)inst * kRoles + role) * kMaxBands + b;
    dspi_biquad_f32 *eng_q = role < 2 ? m_aos + ((size_t)role * Np + inst) * kMaxBands + b : o_aos + ((size_t)(role - 2) * Np + inst) * kMaxBands + b;
    if (to_mirrors) *eng_q = *chain_q;
    else *chain_q = *eng_q;
}

__global__ void chain_status_kernel(ChainDev d, uint32_t inst0, uint32_t n, dspi_status *__restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, inst = inst0 + i;
    if (i >= n) return;
    dspi_status s;
    for (int r = 0; r < kRoles; r++) s.peaks[r] = d.peaks[r * d.N_pad + inst];
    s.cpu0_load = 0;
    s.cpu1_load = 0;
    s.clip_flags = d.clip[inst];
    out[i] = s;
}

// ---------------------------------------------------------------------------------------------
// frequency response (dspi_chain_response_*): the linear, time-invariant part of the path the next call applies, from the
// SoA parameters and the two EQ engines' mirrors (response.cuh).  CTA = one instance at a time, thread = one frequency:
// the instance's 11 filter rows and loudness shelves become sections in shared memory once, then every thread composes
// preamp -> loudness -> master EQ -> look-ahead delay -> crossfeed -> matrix -> output EQ -> gain -> delay for all 9 x 2
// (output, input) pairs of its frequency.  Nothing here reads or writes the packed stores or any state.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
chain_response_kernel(ChainDev d, const dspi_biquad_f32 *__restrict__ m_aos, const dspi_biquad_f32 *__restrict__ o_aos, uint32_t inst0,
                      uint32_t n, const float *__restrict__ freqs, uint32_t nf, float fs, float2 *__restrict__ out)
{
    __shared__ Sect sec[kRoles][kMaxBands];
    __shared__ Sect loud[2];
    __shared__ int cnt[kRoles], n_loud;
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    const float fr = f < nf ? freqs[f] : 0.0f;
    const Trig t = trig_at(fr, fs);
    const uint32_t Np = d.N_pad;
    for (uint32_t u = blockIdx.y; u < n; u += gridDim.y) {
        const uint32_t inst = inst0 + u;
        const uint8_t flags = d.flags[inst];
        __syncthreads();
        if (threadIdx.x < kRoles) {                                          // filters[role]: master L, R, Out1..9
            const uint32_t role = threadIdx.x;
            const dspi_biquad_f32 *row = role < 2 ? m_aos + ((size_t)role * Np + inst) * kMaxBands : o_aos + ((size_t)(role - 2) * Np + inst) * kMaxBands;
            int k = 0;
            for (uint32_t b = 0; b < d.nb; b++) {
                Sect s;
                if (sect_band(row[b], s)) sec[role][k++] = s;
            }
            cnt[role] = k;
        } else if (threadIdx.x == 32) {                                      // loudness shelves, general SVF mix (usb_audio.c:689-718)
            int k = 0;
            for (int j = 0; j < 2 && (flags & F_LOUD); j++) {
                if ((d.loud_byp[inst] >> j) & 1) continue;
                const float *c = d.loud_c + (size_t)j * 6 * Np + inst;
                loud[k++] = sect_svf(c[0], c[Np], c[2 * Np], c[3 * Np], c[4 * Np], c[5 * Np], 0u, true);
            }
            n_loud = k;
        }
        __syncthreads();
        if (f >= nf) continue;
        Cd pre = cascade_eval(loud, n_loud, t);
        if ((flags & F_LEV) && (flags & F_LOOKAHEAD)) pre = cmul(pre, delay_phase(fr, kLa, fs));   // leveller at 0 dB: its look-ahead delay
        Cd P[2];
#pragma unroll
        for (int s = 0; s < 2; s++) {
            P[s] = cscale(pre, d.preamp[s * Np + inst]);
            if (!(flags & F_BYPASS_MASTER)) P[s] = cmul(P[s], cascade_eval(sec[s], cnt[s], t));
        }
        // crossfeed.c:132-156: L' = (1 - LP) L + AP LP R, LP = a0 / (1 - b1 w), AP = (a + w) / (1 + a w)
        Cd direct = { 1.0, 0.0 }, cross = { 0.0, 0.0 };
        if (flags & F_XFEED) {
            const double a0 = d.xf[0 * Np + inst], b1 = d.xf[1 * Np + inst], ap = d.xf[4 * Np + inst];
            const Cd lp = cdiv({ a0, 0.0 }, { 1.0 - b1 * t.c1, -b1 * t.s1 });
            const Cd apd = { 1.0 + ap * t.c1, ap * t.s1 };                 // 0 only for a = +-1 at DC / Nyquist: AP = a there
            const Cd apv = (apd.re == 0.0 && apd.im == 0.0) ? Cd{ ap, 0.0 } : cdiv({ ap + t.c1, t.s1 }, apd);
            direct = { 1.0 - lp.re, -lp.im };
            cross = cmul(apv, lp);
        }
        const bool env = d.env[4 * Np + inst] != 0;                          // envelope mode: the gain reached so far
        const float vmm_env = __fmul_rn(__fmul_rn(d.vol_base[inst], __uint_as_float(d.env[2 * Np + inst])), d.vol_master[inst]);
        for (int o = 0; o < kOuts; o++) {
            const uint8_t of = d.o_flags[o * Np + inst];
            const float gain = !env ? d.o_gain[o * Np + inst] : ((of & O_MUTE) ? 0.0f : __fmul_rn(d.o_glin[o * Np + inst], vmm_env));
            Cd h[2] = { { 0.0, 0.0 }, { 0.0, 0.0 } };
            if ((of & O_ENABLED) && gain != 0.0f) {
                Cd g = cascade_eval(sec[2 + o], (of & O_MUTE) ? 0 : cnt[2 + o], t);
                g = cscale(g, gain);
                const int32_t dly = d.o_dly[o * Np + inst];
                if ((flags & F_ANY_DELAY) && dly > 0) g = cmul(g, delay_phase(fr, (uint32_t)dly & (kMaxDelay - 1), fs));   // MAX aliases to 0
                const double gl = d.o_gl[o * Np + inst], gr = d.o_gr[o * Np + inst];
                h[0] = cmul(g, cmul(cadd(cscale(direct, gl), cscale(cross, gr)), P[0]));
                h[1] = cmul(g, cmul(cadd(cscale(cross, gl), cscale(direct, gr)), P[1]));
            }
            out[(((size_t)u * kOuts + o) * 2 + 0) * nf + f] = to_float2(h[0]);
            out[(((size_t)u * kOuts + o) * 2 + 1) * nf + f] = to_float2(h[1]);
        }
    }
}

}  // namespace
}  // namespace dspi

#include "chain_host.cuh"

namespace dspi {
namespace {

// one kernel set per flavour: FUSED contracts a*b + c into one rounding (DSPI_ARITH_F32_FUSED), strict rounds twice
template <bool FUSED>
struct F32Stages {
    static constexpr auto pre = chain_pre_kernel<FUSED>;
    static constexpr auto post = chain_post_kernel<FUSED>;
    static constexpr auto mix = chain_mix_kernel<FUSED>;
    template <bool SUBFRAMES> static constexpr auto outpost = chain_outpost_kernel<SUBFRAMES>;
    static constexpr auto ring = chain_ring_kernel;
    static constexpr auto pdm = chain_pdm_kernel;
    static constexpr auto env = chain_env_kernel;
    static constexpr auto status = chain_status_kernel;
};

// what the float engine brings to the shared host code (chain_host.cuh)
struct F32 : ParamStores {
    using Biquad = dspi_biquad_f32;
    using Status = dspi_status;
    using Params = dspi_chain_params_f32;
    using Stores = ParamStores;
    static constexpr int kLoudRows = 12;                                     // [2 shelves][6] SVF coefficients
    static constexpr int kXs = dspi::kXs;
    static constexpr uint32_t kStateVersion = 2;
    static constexpr auto scatter = chain_scatter_kernel;
    static constexpr auto dynamics = chain_dynamics_kernel;
    static constexpr auto response = chain_response_kernel;

    template <class F>
    static int with_stages(const dspi_chain_desc &desc, F &&f)
    {
        return desc.arith == DSPI_ARITH_F32_FUSED ? f(F32Stages<true>()) : f(F32Stages<false>());
    }

    static int check_desc(const dspi_chain_desc &desc)
    {
        if (desc.arith != DSPI_ARITH_F32_FUSED && desc.arith != DSPI_ARITH_F32_STRICT) return fail(DSPI_EINVAL, "chain engines are float (arith 0 or 1)");
        if (desc.n_instances == 0 || desc.max_frames == 0) return fail(DSPI_EINVAL, "n_instances and max_frames must be > 0");
        if (desc.n_bands != 10) return fail(DSPI_EINVAL, "chain engines run channel_band_counts = 10");
        return DSPI_OK;
    }

    static cudaError_t alloc_leveller(ChainHost<F32> *c) { return dev_alloc(c, &c->d.lev_s, (size_t)5 * c->d.N_pad); }

    // leveller_reset_state(): envelopes and smoothed gain 0, gain_linear and gain_prev_linear (rows 3, 4) 1.0f
    static void leveller_arrays(ChainHost<F32> *c, std::vector<InstArray> &v)
    {
        v.push_back(inst_array(c->d.lev_s, 5, kInBlob | kInImage | kReset, 4, 1u << 3 | 1u << 4, 0x3f800000u));
    }

    // volumes, preamp, loudness shelves and matrix / output gains of instance i of a set_params call
    static void pack(const dspi_chain_params_f32 &p, uint32_t i, uint32_t n, ParamRows<F32> &r)
    {
        // usb_audio.c:569-571
        float vol_mul = p.host_mute ? 0.0f : (float)p.host_vol_mul * (1.0f / 32768.0f);
        r.vbase[i] = vol_mul;
        r.vmaster[i] = p.master_volume_linear;
        r.pmg[i] = p.preset_mute_gain;
        vol_mul *= p.preset_mute_gain;
        const float vol_mul_master = vol_mul * p.master_volume_linear;
        r.preamp[0 * n + i] = p.preamp_linear[0];
        r.preamp[1 * n + i] = p.preamp_linear[1];
        for (int o = 0; o < kOuts; o++) {
            const dspi_output_channel &oc = p.matrix.outputs[o];
            const dspi_matrix_crosspoint &xl = p.matrix.crosspoints[0][o], &xr = p.matrix.crosspoints[1][o];
            float a = 0.0f, b = 0.0f;                                        // :760-764
            if (xl.enabled) a = xl.phase_invert ? -xl.gain_linear : xl.gain_linear;
            if (xr.enabled) b = xr.phase_invert ? -xr.gain_linear : xr.gain_linear;
            r.gl[o * n + i] = a;
            r.gr[o * n + i] = b;
            r.gain[o * n + i] = oc.mute ? 0.0f : oc.gain_linear * vol_mul_master;    // :886-887
        }
        for (int j = 0; j < 2; j++) {
            const float v[6] = { p.loudness[j].sva1, p.loudness[j].sva2, p.loudness[j].sva3, p.loudness[j].svm0, p.loudness[j].svm1, p.loudness[j].svm2 };
            for (int k = 0; k < 6; k++) r.loud_c[(j * 6 + k) * n + i] = v[k];
        }
    }
};

}  // namespace
}  // namespace dspi

struct dspi_chain : dspi::ChainHost<dspi::F32> {};

extern "C" int32_t dspi_delay_samples(float delay_ms, float sample_rate, int is_last)
{
    if (is_last) delay_ms += (float)128 / sample_rate * 1000.0f;            // SUB_ALIGN_SAMPLES, config.h:93-95
    const float x = delay_ms * sample_rate / 1000.0f;
    int32_t s = (x != x) ? 0 : (x >= 2147483648.0f ? INT32_MAX : (x <= -2147483648.0f ? INT32_MIN : (int32_t)x));
    if (s > DSPI_CHAIN_MAX_DELAY) s = DSPI_CHAIN_MAX_DELAY;
    if (s < 0) s = 0;
    return s;
}

#define CHAIN dspi_chain
#define CHAIN_FN(name) dspi_chain_##name
#define CHAIN_PARAMS dspi_chain_params_f32
#define CHAIN_BIQUAD dspi_biquad_f32
#define CHAIN_STATUS dspi_status
#include "chain_abi.inc"
