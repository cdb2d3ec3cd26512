// chain_q28.cu — the whole per-packet signal chain in the RP2040's Q28 fixed-point arithmetic, for
// thousands of independent device instances (2 inputs -> 5 outputs each), bit-exact, sm_90a.
//
// Reference: process_audio_packet(), firmware/DSPi/usb_audio.c:968-1283 (single-core branch
// :1191-1276); fast_mul_q28 dsp_pipeline.c:47-58; fast_mul_q15 config.h:556-567; cascade
// dsp_process_rp2040.S:225-394; crossfeed.c:161-180; leveller.c:275-389; PDM pdm_generator.c:351-397.
//
// Same stage-wise decomposition as the float chain: pre (unpack, preamp, loudness) -> K2 over the master rows -> post
// (leveller, peaks, crossfeed) -> mix -> K2 over the output rows -> outpost (gain, delay, metering, 24-bit words or S/PDIF
// subframes) -> ring update -> modulator, run on three streams over packet slices by chain_host.cuh.  The EQ rows run through
// the Q28 cascade kernel of the EQ engine (eq_q28.cu: TMA ring, coefficients pre-split in registers);
// everything is integer-pipe bound (about 27 integer ops per band-sample).
#include <cstdarg>
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

constexpr int kOuts = DSPI_CHAINQ_OUTPUTS;
constexpr int kRoles = DSPI_CHAINQ_EQ_CHANNELS;
constexpr int kMaxDelay = DSPI_CHAINQ_MAX_DELAY;
constexpr int kLa = DSPI_LA_SAMPLES;
constexpr int kXs = 33;                                       // shared-memory column stride: conflict-free for lane = instance AND lane = frame
constexpr int32_t kUnity = 1 << 28;
constexpr int32_t kClipThresh = (1 << 28) + 268;              // config.h:54

struct ChainQ {
    uint32_t N, N_pad, nb, max_frames, ldF;        // ldF: row stride of mrow / orow / subq (frames, multiple of 4)
    int32_t *preamp;                               // [2][N_pad]
    uint8_t *flags;
    int32_t *loud_c; int32_t *loud_st; uint8_t *loud_byp;    // [2 j][5][N_pad], [2 side][2 j][2][N_pad], [N_pad]
    int32_t *xf;                                   // [7][N_pad]
    float *lev_c; int32_t *lev_i; float *lev_f; uint32_t *lev_idx; int32_t *lev_la;   // [9][Np], [4][Np] env_l env_r gain gain_prev, [Np] smooth_db, [Np], [2][480][Np]
    int32_t *o_gl, *o_gr, *o_gain; uint8_t *o_flags; int32_t *o_dly;                  // [5][N_pad]
    int32_t *dline; uint32_t *widx_in, *widx_out;  // [5][N_pad][2048], [N_pad]
    int32_t *pdm;                                  // [9][N_pad]
    uint16_t *peaks; uint16_t *clip;               // [7][N_pad], [N_pad]
    int32_t *mrow;                                 // [2 N_pad][ldF] master rows, row = side * N_pad + inst
    int32_t *orow;                                 // [5 N_pad][ldF] output rows, row = o * N_pad + inst
    int32_t *subq;                                 // [N_pad][ldF] Q28 sub samples for the modulator
    uint8_t *skip_m, *skip_o;                      // [2 N_pad], [5 N_pad]: rows whose EQ is frozen (K2 row skip)
    // preset-mute envelope (usb_audio.c:456-498, Q15 use :975-980)
    uint32_t *env;                                 // [5][N_pad] loading, counter, smooth gain (float bits), sample rate, envelope mode on
    int32_t *vol_base, *vol_master;                // [N_pad] host volume Q15 (:975), master_volume_q15
    float *o_glin;                                 // [5][N_pad] outputs[o].gain_linear
    int32_t *pmg;                                  // [N_pad] the constant preset_mute_gain of dspi_chainq_set_params, as Q15 (:976-978)
    int32_t *vmm;                                  // [packets of the call][N_pad] vol_mul_master (:980) of envelope-mode instances
    const uint32_t *off;                           // [packets of the call + 1] first frame of each packet (chain_schedule.cuh)
};

// fast_mul_q28(), dsp_pipeline.c:47-58: 32-bit wrapping, lo*lo partial product dropped
__device__ __forceinline__ int32_t mul_q28(int32_t a, int32_t b)
{
    const int32_t ah = a >> 16, bh = b >> 16;
    const uint32_t al = (uint32_t)a & 0xFFFFu, bl = (uint32_t)b & 0xFFFFu;
    const uint32_t high = (uint32_t)ah * (uint32_t)bh;
    const uint32_t mid = (uint32_t)ah * bl + al * (uint32_t)bh;
    return (int32_t)((high << 4) + (uint32_t)((int32_t)mid >> 12));
}
// fast_mul_q15(), config.h:556-567
__device__ __forceinline__ int32_t mul_q15(int32_t s, int32_t g)
{
    const int32_t sh = s >> 16, gh = g >> 16;
    const uint32_t sl = (uint32_t)s & 0xFFFFu, gl = (uint32_t)g & 0xFFFFu;
    const uint32_t hh = (uint32_t)sh * (uint32_t)gh;
    const uint32_t mid = (uint32_t)sh * gl + sl * (uint32_t)gh;
    const uint32_t ll = sl * gl;
    return (int32_t)((hh << 17) + (mid << 1) + (ll >> 15));
}

// leveller.c:124-139 (plain float, the RP2040's soft-float never fuses)
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
// pre: PCM unpack + preamp (usb_audio.c:997-1015), loudness TDF2 shelves (:1018-1047) -> master rows
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64)
chainq_pre_kernel(ChainQ d, uint32_t inst0, uint32_t n, const uint8_t *__restrict__ pcm, uint32_t bit_depth, uint32_t f_begin, uint32_t f_end,
                  uint32_t F)
{
    // warp = 16 instances x {L, R}, lane l = side l >> 4 of instance inst16 + (l & 15), instances [inst0, inst0 + n):
    // see chain_pre_kernel (chain_f32.cu)
    __shared__ int32_t tile_s[2][32][kXs];                // per warp: [frame][row = side * 16 + instance]
    __shared__ uint32_t pcm_s[2][2][16][49];              // per warp, double-buffered: 16 instances x 32 frames x <= 6 bytes (rows padded to 49 words)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t local16 = (blockIdx.x * 2 + warp) * 16;
    if (local16 >= ((n + 31) & ~31u)) return;
    const uint32_t side = lane >> 4, li = lane & 15;
    const uint32_t inst16 = inst0 + local16, inst = inst16 + li;
    const bool live = local16 + li < n;
    const size_t Np = d.N_pad;
    int32_t (*tile)[kXs] = tile_s[warp];

    const bool loud_on = d.flags[inst] & F_LOUD;
    const uint8_t loud_byp = d.loud_byp[inst];
    int32_t lc[2][5], ls[2][2];
#pragma unroll
    for (int j = 0; j < 2; j++) {
#pragma unroll
        for (int k = 0; k < 5; k++) lc[j][k] = d.loud_c[(j * 5 + k) * Np + inst];
        ls[j][0] = d.loud_st[((side * 2 + j) * 2 + 0) * Np + inst];
        ls[j][1] = d.loud_st[((side * 2 + j) * 2 + 1) * Np + inst];
    }
    const int32_t preamp = d.preamp[side * Np + inst];
    const uint32_t bpf = bit_depth == 24 ? 6u : 4u;
    const bool words_ok = ((reinterpret_cast<uintptr_t>(pcm) | ((size_t)F * bpf) | ((size_t)f_begin * bpf)) & 3u) == 0;
    const uint8_t *my_pcm = pcm + (size_t)(local16 + li) * F * bpf;
    const uint32_t n_inst = min(16u, n > local16 ? n - local16 : 0u);
    auto fetch = [&](uint32_t f0, int buf) {               // see chain_pre_kernel (chain_f32.cu)
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
        fetch(f0 + 32, buf ^ 1);
        if (words_ok) {
            cp_async_wait<1>();
            __syncwarp();
            tile_bytes = reinterpret_cast<const uint8_t *>(pcm_s[warp][buf][li]);
        }
        for (uint32_t t = 0; t < nv; t++) {
            const uint8_t *q = tile_bytes + (size_t)t * bpf;
            int32_t raw = 0;
            if (live) {
                if (bit_depth == 24) {
                    const uint8_t *b = q + side * 3;
                    raw = ((int32_t)((uint32_t)b[2] << 24 | (uint32_t)b[1] << 16 | (uint32_t)b[0] << 8)) >> 2;       // :1001
                } else {
                    const uint8_t *b = q + side * 2;
                    raw = (int32_t)((uint32_t)(int32_t)(int16_t)((uint16_t)b[0] | (uint16_t)b[1] << 8) << 14);       // :1010
                }
            }
            int32_t x = mul_q28(raw, preamp);
            if (loud_on) {
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    if ((loud_byp >> j) & 1) continue;
                    const int32_t result = mul_q28(lc[j][0], x) + ls[j][0];                                          // :1026
                    ls[j][0] = mul_q28(lc[j][1], x) - mul_q28(lc[j][3], result) + ls[j][1];
                    ls[j][1] = mul_q28(lc[j][2], x) - mul_q28(lc[j][4], result);
                    x = result;
                }
            }
            tile[t][lane] = x;
        }
        __syncwarp();
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
// post: Q28 leveller (leveller.c:275-389), input peaks, crossfeed (crossfeed.c:161-180), per packet
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
chainq_post_kernel(ChainQ d, uint32_t inst0, uint32_t n, uint32_t p0, uint32_t n_packets, uint32_t longest)
{
    extern __shared__ int32_t smem_q[];                    // per warp: packet columns [longest][33] + look-ahead reads [longest][33]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t side = lane >> 4;
    const uint32_t local16 = (blockIdx.x * (blockDim.x >> 5) + warp) * 16;      // instances [inst0, inst0 + n): see chain_pre_kernel
    if (local16 >= ((n + 31) & ~31u)) return;
    const uint32_t inst16 = inst0 + local16, inst = inst16 + (lane & 15);
    const bool live = local16 + (lane & 15) < n;
    const size_t Np = d.N_pad;
    int32_t *xw = smem_q + (size_t)warp * 2 * longest * kXs;
    int32_t *xs = xw + lane;
    int32_t *hs = xw + (size_t)longest * kXs + lane;

    const uint8_t flags = live ? d.flags[inst] : 0;       // lanes past the range run with every stage off
    const bool lev_on = flags & F_LEV, xf_on = flags & F_XFEED, lookahead = flags & F_LOOKAHEAD;
    const int32_t xf_a0 = d.xf[0 * Np + inst], xf_b1 = d.xf[1 * Np + inst], xf_ap = d.xf[4 * Np + inst];
    int32_t xf_lp = d.xf[(2 + side) * Np + inst], xf_as = d.xf[(5 + side) * Np + inst];
    float lvc[9];
#pragma unroll
    for (int k = 0; k < 9; k++) lvc[k] = d.lev_c[k * Np + inst];
    int32_t env = d.lev_i[side * Np + inst];
    int32_t gain_q = d.lev_i[2 * Np + inst], gain_prev_q = d.lev_i[3 * Np + inst];
    float smooth_db = d.lev_f[inst];
    uint32_t la_idx = d.lev_idx[inst];
    int32_t *la_buf = d.lev_la + (size_t)side * kLa * Np + inst;

    int32_t peak_last = 0;
    uint16_t clip = 0;
    for (uint32_t p = p0; p < p0 + n_packets; p++) {
        const uint32_t f0 = d.off[p], count = d.off[p + 1] - f0;          // the leveller's block is this packet
        if (lev_on && lookahead) {                                            // see chain_post_kernel (chain_f32.cu)
            uint32_t idx = la_idx;
            for (uint32_t i = 0; i < count; i++) {
                cp_async_4(hs + i * kXs, la_buf + (size_t)idx * Np);
                if (++idx >= (uint32_t)kLa) idx = 0;
            }
        }
        for (int r = 0; r < 32; r++) {
            const int32_t *row = d.mrow + ((size_t)(r >> 4) * Np + inst16 + (r & 15)) * d.ldF + f0;
            for (uint32_t t = lane; t < count; t += 32) cp_async_4(xw + t * kXs + r, row + t);
        }
        cp_async_commit();
        cp_async_wait_all();
        __syncwarp();

        // PASS 3 (:1065-1073) for one sample: input peak, crossfeed (every lane walks the same shuffle)
        int32_t pk = 0;
        auto peak_and_crossfeed = [&](uint32_t i, int32_t v) {
            const int32_t a = abs(v);
            if (a > pk) pk = a;
            int32_t lp = 0, ap = 0;
            if (xf_on) {
                lp = mul_q28(xf_a0, v) + mul_q28(xf_b1, xf_lp);                                           // crossfeed.c:166-167
                xf_lp = lp;
                ap = mul_q28(xf_ap, lp) + xf_as;                                                          // :172
                xf_as = lp - mul_q28(xf_ap, ap);                                                          // :173
            }
            const int32_t ap_other = __shfl_xor_sync(0xffffffffu, ap, 16);
            if (xf_on) v = (v - lp) + ap_other;                                                           // :178-179
            xs[i * kXs] = v;
        };

        // PASS 2.5: leveller (leveller.c:275-389); every lane walks the same shuffles
        if (__any_sync(0xffffffffu, lev_on)) {
            const int32_t a_rms = __float2int_rz(__fmul_rn(lvc[0], 268435456.0f));                       // :286
            const int32_t one_minus = kUnity - a_rms;
            int32_t e = env;
            for (uint32_t i = 0; i < count; i++) {                                                         // :292-299
                const int32_t s = xs[i * kXs];
                const int32_t sq = mul_q28(s, s);
                e = mul_q28(a_rms, e) + mul_q28(one_minus, sq);
            }
            const int32_t e_other = __shfl_xor_sync(0xffffffffu, e, 16);
            const float inv_q28 = 1.0f / 268435456.0f;
            const float el = __fmul_rn((float)(side ? e_other : e), inv_q28), er = __fmul_rn((float)(side ? e : e_other), inv_q28);
            const float rms_sq = (el > er) ? el : er;
            const float rms_db = __fmul_rn(10.0f, (float)log10((double)__fadd_rn(rms_sq, 1e-30f)));     // :311 (libm policy)
            float gc_db;
            if (rms_db < lvc[7]) gc_db = 0.0f;
            else {
                gc_db = gain_computer(rms_db, lvc[3], lvc[4], lvc[5]);
                gc_db = __fadd_rn(gc_db, lvc[6]);
                if (gc_db > lvc[8]) gc_db = lvc[8];
            }
            const float alpha_s = (gc_db < smooth_db) ? lvc[1] : lvc[2];
            const float alpha = (float)pow((double)alpha_s, (double)(float)count);                          // :327
            const float new_smooth = __fadd_rn(__fmul_rn(alpha, smooth_db), __fmul_rn(__fadd_rn(1.0f, -alpha), gc_db));   // :328-329
            const float gl = (float)pow(10.0, (double)__fdiv_rn(new_smooth, 20.0f));                      // :332
            const int32_t g_cur = __float2int_rz(__fmul_rn(gl, 268435456.0f));                            // :334 (saturating)
            const int32_t g_prev = gain_q;
            // :352 is gain = prev + (int32)((int64)(cur - prev) * i / (count - 1)) per sample (C division: towards zero).  With
            // diff = Q * D + R (D = count - 1, R with the sign of diff, |R| < D) the quotient is Q * i + trunc(R * i / D), both terms
            // of one sign, so it is carried incrementally: off += Q, acc += R, one correction when |acc| reaches D.  All in
            // 32-bit wrapping arithmetic, which is the int32 cast of :352; no 64-bit division in the per-sample loop.
            const int32_t g_diff = (int32_t)((uint32_t)g_cur - (uint32_t)g_prev);
            const int32_t den = count > 1 ? (int32_t)(count - 1) : 1;
            const int32_t ramp_q = g_diff / den, ramp_r = g_diff - ramp_q * den;
            uint32_t off = 0;
            int32_t acc = 0;
            // The leveller's per-sample part and PASS 3 share one loop: the ramp, the look-ahead exchange and the peak limit of
            // sample i+1 do not depend on the crossfeed recurrence of sample i, so the two serial chains overlap.
            for (uint32_t i = 0; i < count; i++) {                                                          // :347-386, :1065-1073
                int32_t gain = count == 1 ? g_cur : (int32_t)((uint32_t)g_prev + off);                      // :352
                off += (uint32_t)ramp_q;
                acc += ramp_r;
                if (acc >= den) { acc -= den; off++; }
                else if (acc <= -den) { acc += den; off--; }
                const int32_t x0 = xs[i * kXs];
                int32_t o = x0;
                if (lev_on && lookahead) {
                    const int32_t held = hs[i * kXs];
                    la_buf[(size_t)la_idx * Np] = o;
                    o = held;
                    la_idx++;
                    if (la_idx >= (uint32_t)kLa) la_idx = 0;
                }
                const int32_t o_other = __shfl_xor_sync(0xffffffffu, o, 16);
                if (gain > kUnity) {                                                                      // :370-379
                    const int32_t ol = side ? o_other : o, orr = side ? o : o_other;
                    float peak = fabsf(__fmul_rn((float)ol, inv_q28));
                    const float pr = fabsf(__fmul_rn((float)orr, inv_q28));
                    if (pr > peak) peak = pr;
                    if (peak > 0.0f) {
                        const float max_g_f = __fdiv_rn(0.70795f, peak);
                        const int32_t max_g = __float2int_rz(__fmul_rn(max_g_f, 268435456.0f));
                        if (max_g < gain) gain = (max_g > kUnity) ? max_g : kUnity;
                    }
                }
                peak_and_crossfeed(i, lev_on ? mul_q28(o, gain) : x0);
            }
            if (lev_on) {
                env = e;
                smooth_db = new_smooth;
                gain_prev_q = g_prev;
                gain_q = g_cur;
            }
        } else {
            for (uint32_t i = 0; i < count; i++) peak_and_crossfeed(i, xs[i * kXs]);
        }
        peak_last = pk;
        if (pk > kClipThresh) clip |= (uint16_t)(1u << side);
        __syncwarp();
        for (uint32_t t = lane; t < count; t += 32) {
#pragma unroll 8
            for (int r = 0; r < 32; r++)
                d.mrow[((size_t)(r >> 4) * Np + inst16 + (r & 15)) * d.ldF + f0 + t] = xw[t * kXs + r];
        }
        __syncwarp();
    }

    const uint16_t clip_other = (uint16_t)__shfl_xor_sync(0xffffffffu, (uint32_t)clip, 16);
    if (!live) return;
    d.xf[(2 + side) * Np + inst] = xf_lp;
    d.xf[(5 + side) * Np + inst] = xf_as;
    d.lev_i[side * Np + inst] = env;
    if (side == 0) {
        d.lev_i[2 * Np + inst] = gain_q;
        d.lev_i[3 * Np + inst] = gain_prev_q;
        d.lev_f[inst] = smooth_db;
        d.lev_idx[inst] = la_idx;
    }
    d.peaks[side * Np + inst] = (uint16_t)(peak_last >> 13);                                              // :1279-1280
    if (side == 0 && (clip | clip_other)) atomicOr(reinterpret_cast<unsigned int *>(d.clip + (inst & ~1u)), (unsigned int)(clip | clip_other) << (16 * (inst & 1)));
}

// ---------------------------------------------------------------------------------------------
// matrix mix in Q15 (usb_audio.c:1076-1100): lane = frame
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
chainq_mix_kernel(ChainQ d, uint32_t inst0, uint32_t n, uint32_t f_begin, uint32_t f_end)
{
    const int lane = threadIdx.x & 31;
    constexpr int kB = 4;
    const uint32_t n_tiles = (f_end - f_begin + 32 * kB - 1) / (32 * kB);
    const uint64_t units = (uint64_t)n * n_tiles;
    const size_t Np = d.N_pad;
    for (uint64_t u = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < units; u += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint32_t inst = inst0 + (uint32_t)(u / n_tiles), tile = (uint32_t)(u % n_tiles);
        const uint32_t fbase = f_begin + tile * 32 * kB + lane;
        int32_t l[kB], r[kB];
#pragma unroll
        for (int j = 0; j < kB; j++) {
            const uint32_t f = fbase + 32 * j;
            l[j] = f < f_end ? d.mrow[(size_t)inst * d.ldF + f] : 0;
            r[j] = f < f_end ? d.mrow[(Np + inst) * d.ldF + f] : 0;
        }
#pragma unroll
        for (int o = 0; o < kOuts; o++) {
            const bool enabled = d.o_flags[o * Np + inst] & O_ENABLED;
            const int32_t gl = d.o_gl[o * Np + inst], gr = d.o_gr[o * Np + inst];
#pragma unroll
            for (int j = 0; j < kB; j++) {
                int32_t v = 0;
                if (enabled) {
                    if (gl != 0 && gr != 0) v = mul_q15(l[j], gl) + mul_q15(r[j], gr);
                    else if (gl != 0) v = mul_q15(l[j], gl);
                    else if (gr != 0) v = mul_q15(r[j], gr);
                }
                const uint32_t f = fbase + 32 * j;
                if (f < f_end) d.orow[((size_t)o * Np + inst) * d.ldF + f] = v;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// outputs after the EQ: gain (:1203-1212), delay (:1216-1230), peaks (:1232-1241), 24-bit words (:1243-1257), sub (:1259-1275)
// ---------------------------------------------------------------------------------------------
// update_preset_mute_envelope() (usb_audio.c:466-498) for every packet of the call, one instance per thread, then the Q15
// volume chain of :976-980: pmg = (int32)(g * 32768 + 0.5) clamped, vmm[p] = mul_q15(mul_q15(vol_base, pmg), master_q15)
__global__ void chainq_env_kernel(ChainQ d, uint32_t inst0, uint32_t n, uint32_t n_packets)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, inst = inst0 + i;
    const size_t Np = d.N_pad;
    if (i >= n || !d.env[4 * Np + inst]) return;
    uint32_t loading = d.env[0 * Np + inst], counter = d.env[1 * Np + inst];
    float g = __uint_as_float(d.env[2 * Np + inst]);
    const uint32_t fs = d.env[3 * Np + inst];
    unsigned long long ts = ((unsigned long long)fs * 8ull + 999ull) / 1000ull;
    if (ts < 1ull) ts = 1ull;
    if (ts > 0xFFFFFFFFull) ts = 0xFFFFFFFFull;
    const int32_t vol_base = d.vol_base[inst], master = d.vol_master[inst];
    for (uint32_t p = 0; p < n_packets; p++) {
        const uint32_t count = d.off[p + 1] - d.off[p];                                  // sample_count of this packet
        float step = __fdiv_rn((float)count, (float)(uint32_t)ts);
        if (step > 1.0f) step = 1.0f;
        const bool active = loading != 0;
        if (active) {
            if (counter > count) counter -= count;
            else { counter = 0; loading = 0; }
        }
        const float target = active ? 0.0f : 1.0f;
        if (g < target)      { g = __fadd_rn(g, step);  if (g > target) g = target; }
        else if (g > target) { g = __fadd_rn(g, -step); if (g < target) g = target; }
        int32_t pmg = __float2int_rz(__fadd_rn(__fmul_rn(g, 32768.0f), 0.5f));          // :976-978
        if (pmg < 0) pmg = 0;
        if (pmg > 32768) pmg = 32768;
        d.vmm[(size_t)p * Np + inst] = mul_q15(mul_q15(vol_base, pmg), master);         // :979-980
    }
    d.env[0 * Np + inst] = loading;
    d.env[1 * Np + inst] = counter;
    d.env[2 * Np + inst] = __float_as_uint(g);
}

// The RP2040 stores (Q28 / Q15) of device-side parameter ingest, shared by chainq_dynamics_kernel and the bulk ingest kernel
// (bulk_ingest.cuh): see chain_f32.cu
struct ParamStores {
    using Dev = ChainQ;
    static constexpr int kRoles = dspi::kRoles, kOuts = dspi::kOuts, kMaxDelay = dspi::kMaxDelay, kPlatformId = 0;
    static constexpr bool kQ28 = true;
    static __device__ void crossfeed(const ChainQ &d, uint32_t inst, const dspi_crossfeed_config &cfg, float fs)
    {
        const size_t Np = d.N_pad;
        float a0, b1, ap;
        const bool xon = dyn::crossfeed_coeffs(cfg, fs, a0, b1, ap);
        const float scale = 268435456.0f;                                    // crossfeed.c:115-118
        d.xf[0 * Np + inst] = xon ? dyn::f2i_sat(__fmul_rn(a0, scale)) : 0;
        d.xf[1 * Np + inst] = xon ? dyn::f2i_sat(__fmul_rn(b1, scale)) : 0;
        d.xf[4 * Np + inst] = xon ? dyn::f2i_sat(__fmul_rn(ap, scale)) : 0;
        d.xf[2 * Np + inst] = 0; d.xf[3 * Np + inst] = 0; d.xf[5 * Np + inst] = 0; d.xf[6 * Np + inst] = 0;
    }
    static __device__ void leveller(const ChainQ &d, uint32_t inst, const dspi_leveller_config &cfg, float fs)
    {
        float lv[9];
        dyn::leveller_coeffs(cfg, fs, lv);
#pragma unroll
        for (int k = 0; k < 9; k++) d.lev_c[(size_t)k * d.N_pad + inst] = lv[k];
    }
    static __device__ void loudness(const ChainQ &d, uint32_t inst, uint32_t row, float ref_spl, float intensity_pct, float fs)
    {
        const size_t Np = d.N_pad;
        float lo_db, hi_db;
        dyn::loudness_row_gains((int)row, ref_spl, intensity_pct, lo_db, hi_db);
        int32_t c[5];
        bool byp;
        uint8_t lb = 0;
        const float lfs = fs < 1.0f ? 48000.0f : fs;
        dyn::shelf_q28(200.0f, 0.707f, lo_db, false, lfs, c, byp);
        if (byp) lb |= 1;
#pragma unroll
        for (int k = 0; k < 5; k++) d.loud_c[(0 * 5 + k) * Np + inst] = c[k];
        dyn::shelf_q28(6000.0f, 0.707f, hi_db, true, lfs, c, byp);
        if (byp) lb |= 2;
#pragma unroll
        for (int k = 0; k < 5; k++) d.loud_c[(1 * 5 + k) * Np + inst] = c[k];
        d.loud_byp[inst] = lb;
    }
    static __device__ void host_volume(const ChainQ &d, uint32_t inst, int16_t vol_mul, bool host_mute)
    {
        const size_t Np = d.N_pad;
        const int32_t vol_base = host_mute ? 0 : (int32_t)vol_mul;           // usb_audio.c:975
        d.vol_base[inst] = vol_base;
        const int32_t vmm = mul_q15(mul_q15(vol_base, d.pmg[inst]), d.vol_master[inst]);    // :979-980
        for (int o = 0; o < dspi::kOuts; o++)
            d.o_gain[o * Np + inst] = (d.o_flags[o * Np + inst] & O_MUTE) ? 0 : __float2int_rz(__fmul_rn(d.o_glin[o * Np + inst], (float)vmm));   // :1204-1205
    }
    // what dspi_chainq_set_params stores for the preamp (Q28), the master volume (Q15) and one crosspoint (Q15, :1084-1085)
    static __device__ void preamp(const ChainQ &d, uint32_t inst, uint32_t side, float linear)
    {
        d.preamp[(size_t)side * d.N_pad + inst] = dyn::f2i_sat(__fmul_rn(linear, 268435456.0f));
    }
    static __device__ void master_volume(const ChainQ &d, uint32_t inst, float linear) { d.vol_master[inst] = dyn::f2i_sat(__fmul_rn(linear, 32768.0f)); }
    static __device__ void crosspoint(const ChainQ &d, uint32_t inst, uint32_t side, uint32_t o, bool enabled, bool invert, float linear)
    {
        (side ? d.o_gr : d.o_gl)[(size_t)o * d.N_pad + inst] = enabled ? dyn::f2i_sat(__fmul_rn(invert ? -linear : linear, 32768.0f)) : 0;
    }
    // :1197-1201 (quirk: gated on bypass_master_eq too)
    static __host__ __device__ bool output_eq_frozen(bool enabled, bool mute, bool bypass_master_eq) { return !(enabled && !mute && !bypass_master_eq); }
};

// Mass reconfiguration of the dynamics stages on the device (SURVEY f-1), RP2040 stores: see chain_f32.cu
__global__ void chainq_dynamics_kernel(ChainQ d, bulk::Record rec, uint32_t inst0, uint32_t n, const dspi_dynamics_config *__restrict__ cfgs, float fs)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t inst = inst0 + i;
    const dspi_dynamics_config cfg = cfgs[i];
    uint8_t flags = d.flags[inst] & (uint8_t)~(F_XFEED | F_LEV | F_LOOKAHEAD | F_LOUD);
    ParamStores::crossfeed(d, inst, cfg.crossfeed, fs);
    if (cfg.crossfeed.enabled) flags |= F_XFEED;
    ParamStores::leveller(d, inst, cfg.leveller, fs);
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

__device__ __forceinline__ int32_t outq_gain(int32_t v, bool enabled, int32_t gain)
{
    if (enabled) v = (gain == 0) ? 0 : mul_q15(v, gain);
    return v;
}

struct OutCfgQ {
    bool enabled, pair_off, delay_on, mute;
    int32_t gain;                      // constant gain of the call (no envelope)
    float glin;                        // outputs[o].gain_linear
    const int32_t *vmm;                // envelope mode: vol_mul_master per packet, stride N_pad; else nullptr
    const uint32_t *off;               // packet offsets of the call
    size_t Np;
    uint32_t dl;                       // delay & (MAX - 1): MAX aliases to 0 (SURVEY a-10)
    const int32_t *row;
    const int32_t *ring;
};

__device__ __forceinline__ OutCfgQ outq_cfg(const ChainQ &d, uint32_t o, uint32_t inst, bool any_delay)
{
    OutCfgQ c;
    const size_t Np = d.N_pad;
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
    c.delay_on = any_delay && dly > 0;
    c.dl = (uint32_t)dly & (kMaxDelay - 1);
    c.row = d.orow + ((size_t)o * Np + inst) * d.ldF;
    c.ring = d.dline + ((size_t)o * Np + inst) * kMaxDelay;
    return c;
}

// output gain in force at frame T of the call (usb_audio.c:1204-1205): constant, or following the envelope packet by packet;
// p is the packet of T or a later one
__device__ __forceinline__ int32_t gainq_at(const OutCfgQ &c, uint32_t T, uint32_t p)
{
    if (!c.vmm) return c.gain;
    return c.mute ? 0 : __float2int_rz(__fmul_rn(c.glin, (float)c.vmm[(size_t)packet_of(c.off, T, p) * c.Np]));
}

// frame T (in packet p) of the call emits the post-gain sample of frame T - dl: inside the call from the output rows,
// before it from the ring (see chain_f32.cu)
__device__ __forceinline__ int32_t outq_sample(const OutCfgQ &c, uint32_t T, uint32_t p, uint32_t widx0)
{
    if (!c.delay_on) return outq_gain(c.row[T], c.enabled, gainq_at(c, T, p));
    if (T >= c.dl) return outq_gain(c.row[T - c.dl], c.enabled, gainq_at(c, T - c.dl, p));
    return c.ring[(widx0 + T - c.dl) & (kMaxDelay - 1)];
}

__device__ __forceinline__ int32_t clip_s24(int32_t w) { return w > 0x7FFFFF ? 0x7FFFFF : (w < -0x800000 ? -0x800000 : w); }   // config.h:547-551

// Instances [inst0, inst0 + n), the caller's rows counted from inst0.  SUBFRAMES = false: spdif_out is [n][2][F][2] int32
// words; true: [n][2][F] uint4 subframe pairs at each instance's block position and channel status (as chain_f32.cu)
template <bool SUBFRAMES>
__global__ void __launch_bounds__(256)
chainq_outpost_kernel(ChainQ d, uint32_t inst0, uint32_t n, uint32_t p0, uint32_t n_packets, uint32_t F, int32_t *__restrict__ spdif_out, SpdifTx tx)
{
    const int lane = threadIdx.x & 31;
    const uint64_t units = (uint64_t)n * n_packets;
    const size_t Np = d.N_pad;
    constexpr int kPairs = (kOuts - 1) / 2;
    for (uint64_t u = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < units; u += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint32_t local = (uint32_t)(u / n_packets), inst = inst0 + local, p = p0 + (uint32_t)(u % n_packets);
        const uint32_t f0 = d.off[p], count = d.off[p + 1] - f0;
        const bool last = p == p0 + n_packets - 1;
        const bool any_delay = d.flags[inst] & F_ANY_DELAY;
        const uint32_t widx0 = d.widx_in[inst];
        const uint32_t bp = SUBFRAMES ? tx.bp[inst] : 0u;
        const uint64_t cs40 = SUBFRAMES ? tx.cs40[inst] : 0ull;
        unsigned int clip = 0;
        for (int k = 0; k <= kPairs; k++) {                                   // the S/PDIF pairs, then the sub alone
            const bool is_sub = k == kPairs;
            const uint32_t oa = 2 * k, ob = is_sub ? oa : oa + 1;
            const OutCfgQ ca = outq_cfg(d, oa, inst, any_delay), cb = outq_cfg(d, ob, inst, any_delay);
            int32_t pka = 0, pkb = 0;
            constexpr int kB = 4;
            for (uint32_t tb = lane; tb < count; tb += 32 * kB) {
                int32_t xa[kB], xb[kB];
#pragma unroll
                for (int j = 0; j < kB; j++) {
                    const uint32_t t = tb + 32 * j;
                    xa[j] = t < count ? outq_sample(ca, f0 + t, p, widx0) : 0;
                    xb[j] = (!is_sub && t < count) ? outq_sample(cb, f0 + t, p, widx0) : 0;
                }
#pragma unroll
                for (int j = 0; j < kB; j++) {
                    const uint32_t t = tb + 32 * j, T = f0 + t;
                    if (t >= count) break;
                    const int32_t aa = abs(xa[j]), ab = abs(xb[j]);
                    if (aa > pka) pka = aa;
                    if (ab > pkb) pkb = ab;
                    if (is_sub) {
                        if (ca.enabled) d.subq[(size_t)inst * d.ldF + T] = xa[j];                          // :1270 pdm_push_sample(buf_out[pdm_out][i])
                    } else if (spdif_out) {
                        int2 w = make_int2(0, 0);
                        if (!ca.pair_off) { w.x = clip_s24((xa[j] + 32) >> 6); w.y = clip_s24((xb[j] + 32) >> 6); }   // :1254-1255
                        if (SUBFRAMES) {                                      // 16 bytes per lane: 512 contiguous bytes per warp store
                            const uint32_t pos = (bp + T) % 192u;
                            reinterpret_cast<uint4 *>(spdif_out)[((size_t)local * kPairs + k) * F + T] = encode_frame(w, spdif_pre_left(pos), spdif_cs_bit(pos, cs40));
                        } else {
                            *reinterpret_cast<int2 *>(spdif_out + (((size_t)local * kPairs + k) * F + T) * 2) = w;
                        }
                    }
                }
            }
            // the reference compares signed values (`if (a > pk)`), so INT_MIN from abs(INT_MIN) never wins: plain signed max
            pka = __reduce_max_sync(0xffffffffu, pka);
            pkb = __reduce_max_sync(0xffffffffu, pkb);
            if (lane == 0) {
                if (last) {
                    uint16_t pq = (uint16_t)(pka >> 13);                                                  // :1239 / :1267
                    if (is_sub && !ca.enabled) pq = 0;                                                    // :1273
                    d.peaks[(2 + oa) * Np + inst] = pq;
                    if (!is_sub) d.peaks[(2 + ob) * Np + inst] = (uint16_t)(pkb >> 13);
                }
                if (pka > kClipThresh && (!is_sub || ca.enabled)) clip |= 1u << (2 + oa);
                if (!is_sub && pkb > kClipThresh) clip |= 1u << (2 + ob);
            }
        }
        if (lane == 0 && clip) atomicOr(reinterpret_cast<unsigned int *>(d.clip + (inst & ~1u)), clip << (16 * (inst & 1)));
    }
}

__global__ void __launch_bounds__(256)
chainq_ring_kernel(ChainQ d, uint32_t inst0, uint32_t n, uint32_t F, uint32_t n_packets, uint32_t *__restrict__ spdif_bp)
{
    const int lane = threadIdx.x & 31;
    const uint64_t units = (uint64_t)n * kOuts;
    const size_t Np = d.N_pad;
    for (uint64_t u = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < units; u += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint32_t inst = inst0 + (uint32_t)(u / kOuts), o = (uint32_t)(u % kOuts);
        const bool any_delay = d.flags[inst] & F_ANY_DELAY;
        const uint32_t widx0 = d.widx_in[inst];
        const OutCfgQ c = outq_cfg(d, o, inst, any_delay);
        if (c.delay_on) {
            int32_t *ring = d.dline + ((size_t)o * Np + inst) * kMaxDelay;
            for (uint32_t T = (F > (uint32_t)kMaxDelay ? F - kMaxDelay : 0u) + lane; T < F; T += 32)
                ring[(widx0 + T) & (kMaxDelay - 1)] = outq_gain(c.row[T], c.enabled, gainq_at(c, T, n_packets - 1));
        }
        if (o == 0 && lane == 0) {
            d.widx_out[inst] = any_delay ? (widx0 + F) & (kMaxDelay - 1) : widx0;
            spdif_bp[inst] = (spdif_bp[inst] + F % 192u) % 192u;          // every frame of the call was sent
        }
    }
}

__global__ void __launch_bounds__(128)
chainq_pdm_kernel(ChainQ d, uint32_t inst0, uint32_t n, uint32_t f_begin, uint32_t f_end, uint32_t F, uint32_t *__restrict__ pdm_out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, inst = inst0 + i;
    if (i >= n) return;
    if (!(d.flags[inst] & F_SUB_ON)) return;                                                              // usb_audio.c:1261
    pdm_modulate_frames(d.pdm, d.subq + (size_t)inst * d.ldF, 1, d.N_pad, inst, f_begin, f_end, pdm_out ? pdm_out + (size_t)i * F * 8 : nullptr);
}

// filters[][] of n instances (instance-major AoS, 32-byte records) <-> the mirrors of the two EQ engines
__global__ void chainq_scatter_kernel(const dspi_biquad_q28 *__restrict__ aos, uint32_t inst0, uint32_t n, uint32_t Np, dspi_biquad_q28 *__restrict__ m_aos,
                                      dspi_biquad_q28 *__restrict__ o_aos, int to_mirrors)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * kRoles * DSPI_MAX_BANDS) return;
    const uint32_t b = i % DSPI_MAX_BANDS, role = (i / DSPI_MAX_BANDS) % kRoles, inst = inst0 + i / (DSPI_MAX_BANDS * kRoles);
    dspi_biquad_q28 *chain_q = const_cast<dspi_biquad_q28 *>(aos) + ((size_t)inst * kRoles + role) * DSPI_MAX_BANDS + b;
    dspi_biquad_q28 *eng_q = role < 2 ? m_aos + ((size_t)role * Np + inst) * DSPI_MAX_BANDS + b : o_aos + ((size_t)(role - 2) * Np + inst) * DSPI_MAX_BANDS + b;
    if (to_mirrors) *eng_q = *chain_q;
    else *chain_q = *eng_q;
}

__global__ void chainq_status_kernel(ChainQ d, uint32_t inst0, uint32_t n, dspi_status_q28 *__restrict__ out)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, inst = inst0 + i;
    if (i >= n) return;
    dspi_status_q28 s;
    for (int r = 0; r < kRoles; r++) s.peaks[r] = d.peaks[r * d.N_pad + inst];
    s.cpu0_load = 0;
    s.cpu1_load = 0;
    s.clip_flags = d.clip[inst];
    out[i] = s;
}

// ---------------------------------------------------------------------------------------------
// frequency response (dspi_chainq_response_*), as chain_f32.cu's chain_response_kernel in the RP2040's quantities: ratios of
// Q28 values (coefficients / 2^28), the matrix and output gains as the Q15 integers the packet loop uses (/ 32768), output EQs
// skipped while the master EQ is bypassed (quirk 3), MAX_DELAY 2048
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
chainq_response_kernel(ChainQ d, const dspi_biquad_q28 *__restrict__ m_aos, const dspi_biquad_q28 *__restrict__ o_aos, uint32_t inst0,
                       uint32_t n, const float *__restrict__ freqs, uint32_t nf, float fs, float2 *__restrict__ out)
{
    __shared__ Sect sec[kRoles][kMaxBands];
    __shared__ Sect loud[2];
    __shared__ int cnt[kRoles], n_loud;
    const double kQ28 = 1.0 / 268435456.0, kQ15 = 1.0 / 32768.0;
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    const float fr = f < nf ? freqs[f] : 0.0f;
    const Trig t = trig_at(fr, fs);
    const size_t Np = d.N_pad;
    for (uint32_t u = blockIdx.y; u < n; u += gridDim.y) {
        const uint32_t inst = inst0 + u;
        const uint8_t flags = d.flags[inst];
        __syncthreads();
        if (threadIdx.x < kRoles) {                                          // filters[role]: master L, R, Out1..4, sub
            const uint32_t role = threadIdx.x;
            const dspi_biquad_q28 *row = role < 2 ? m_aos + ((size_t)role * Np + inst) * kMaxBands : o_aos + ((size_t)(role - 2) * Np + inst) * kMaxBands;
            int k = 0;
            for (uint32_t b = 0; b < d.nb; b++) {
                Sect s;
                if (sect_band(row[b], s)) sec[role][k++] = s;
            }
            cnt[role] = k;
        } else if (threadIdx.x == 32) {                                      // loudness shelves, Q28 TDF2 (usb_audio.c:1018-1047)
            int k = 0;
            for (int j = 0; j < 2 && (flags & F_LOUD); j++) {
                if ((d.loud_byp[inst] >> j) & 1) continue;
                const int32_t *c = d.loud_c + (size_t)j * 5 * Np + inst;
                loud[k++] = sect_tdf2(c[0] * kQ28, c[Np] * kQ28, c[2 * Np] * kQ28, c[3 * Np] * kQ28, c[4 * Np] * kQ28);
            }
            n_loud = k;
        }
        __syncthreads();
        if (f >= nf) continue;
        Cd pre = cascade_eval(loud, n_loud, t);
        if ((flags & F_LEV) && (flags & F_LOOKAHEAD)) pre = cmul(pre, delay_phase(fr, kLa, fs));
        const bool master_on = !(flags & F_BYPASS_MASTER);
        Cd P[2];
#pragma unroll
        for (int s = 0; s < 2; s++) {
            P[s] = cscale(pre, d.preamp[s * Np + inst] * kQ28);
            if (master_on) P[s] = cmul(P[s], cascade_eval(sec[s], cnt[s], t));
        }
        Cd direct = { 1.0, 0.0 }, cross = { 0.0, 0.0 };                      // crossfeed.c:161-180
        if (flags & F_XFEED) {
            const double a0 = d.xf[0 * Np + inst] * kQ28, b1 = d.xf[1 * Np + inst] * kQ28, ap = d.xf[4 * Np + inst] * kQ28;
            const Cd lp = cdiv({ a0, 0.0 }, { 1.0 - b1 * t.c1, -b1 * t.s1 });
            const Cd apd = { 1.0 + ap * t.c1, ap * t.s1 };                 // 0 only for a = +-1 at DC / Nyquist: AP = a there
            const Cd apv = (apd.re == 0.0 && apd.im == 0.0) ? Cd{ ap, 0.0 } : cdiv({ ap + t.c1, t.s1 }, apd);
            direct = { 1.0 - lp.re, -lp.im };
            cross = cmul(apv, lp);
        }
        // envelope mode: the Q15 volume of the gain reached so far (usb_audio.c:976-980)
        const bool env = d.env[4 * Np + inst] != 0;
        int32_t pmg = __float2int_rz(__fadd_rn(__fmul_rn(__uint_as_float(d.env[2 * Np + inst]), 32768.0f), 0.5f));
        pmg = pmg < 0 ? 0 : (pmg > 32768 ? 32768 : pmg);
        const int32_t vmm_env = mul_q15(mul_q15(d.vol_base[inst], pmg), d.vol_master[inst]);
        for (int o = 0; o < kOuts; o++) {
            const uint8_t of = d.o_flags[o * Np + inst];
            const int32_t gain = !env ? d.o_gain[o * Np + inst] : ((of & O_MUTE) ? 0 : __float2int_rz(__fmul_rn(d.o_glin[o * Np + inst], (float)vmm_env)));
            Cd h[2] = { { 0.0, 0.0 }, { 0.0, 0.0 } };
            if ((of & O_ENABLED) && gain != 0) {
                Cd g = cascade_eval(sec[2 + o], ((of & O_MUTE) || !master_on) ? 0 : cnt[2 + o], t);
                g = cscale(g, gain * kQ15);
                const int32_t dly = d.o_dly[o * Np + inst];
                if ((flags & F_ANY_DELAY) && dly > 0) g = cmul(g, delay_phase(fr, (uint32_t)dly & (kMaxDelay - 1), fs));
                const double gl = d.o_gl[o * Np + inst] * kQ15, gr = d.o_gr[o * Np + inst] * kQ15;
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

// host copies of the firmware's integer helpers (per-packet scalars are folded on the host)
int32_t h_mul_q15(int32_t s, int32_t g)
{
    const int32_t sh = s >> 16, gh = g >> 16;
    const uint32_t sl = (uint32_t)s & 0xFFFFu, gl = (uint32_t)g & 0xFFFFu;
    const uint32_t hh = (uint32_t)sh * (uint32_t)gh, mid = (uint32_t)sh * gl + sl * (uint32_t)gh, ll = sl * gl;
    return (int32_t)((hh << 17) + (mid << 1) + (ll >> 15));
}
int32_t h_f2i_sat(float x)
{
    if (x != x) return 0;
    if (x >= 2147483648.0f) return INT32_MAX;
    if (x <= -2147483648.0f) return INT32_MIN;
    return (int32_t)x;
}

struct Q28Stages {
    static constexpr auto pre = chainq_pre_kernel;
    static constexpr auto post = chainq_post_kernel;
    static constexpr auto mix = chainq_mix_kernel;
    template <bool SUBFRAMES> static constexpr auto outpost = chainq_outpost_kernel<SUBFRAMES>;
    static constexpr auto ring = chainq_ring_kernel;
    static constexpr auto pdm = chainq_pdm_kernel;
    static constexpr auto env = chainq_env_kernel;
    static constexpr auto status = chainq_status_kernel;
};

// what the Q28 engine brings to the shared host code (chain_host.cuh)
struct Q28 : ParamStores {
    using Biquad = dspi_biquad_q28;
    using Status = dspi_status_q28;
    using Params = dspi_chain_params_q28;
    using Stores = ParamStores;
    static constexpr int kLoudRows = 10;                                     // [2 shelves][5] TDF2 coefficients
    static constexpr int kXs = dspi::kXs;
    static constexpr uint32_t kStateVersion = 1;
    static constexpr auto scatter = chainq_scatter_kernel;
    static constexpr auto dynamics = chainq_dynamics_kernel;
    static constexpr auto response = chainq_response_kernel;

    template <class F>
    static int with_stages(const dspi_chain_desc &, F &&f) { return f(Q28Stages()); }

    static int check_desc(const dspi_chain_desc &desc)
    {
        if (desc.arith != DSPI_ARITH_Q28) return fail(DSPI_EINVAL, "dspi_chainq engines are Q28 (arith 2)");
        if (desc.n_instances == 0 || desc.max_frames == 0) return fail(DSPI_EINVAL, "n_instances and max_frames must be > 0");
        if (desc.n_bands == 0 || desc.n_bands > DSPI_MAX_BANDS) return fail(DSPI_EINVAL, "n_bands must be 1..%d", DSPI_MAX_BANDS);
        return DSPI_OK;
    }

    static cudaError_t alloc_leveller(ChainHost<Q28> *c)
    {
        cudaError_t e = dev_alloc(c, &c->d.lev_i, (size_t)4 * c->d.N_pad);
        return e == cudaSuccess ? dev_alloc(c, &c->d.lev_f, (size_t)c->d.N_pad) : e;
    }

    // leveller_reset_state(): env_l, env_r 0, gain, gain_prev (rows 2, 3) unity (leveller.c:101-102), smooth_db 0
    static void leveller_arrays(ChainHost<Q28> *c, std::vector<InstArray> &v)
    {
        v.push_back(inst_array(c->d.lev_i, 4, kInBlob | kInImage | kReset, 4, 1u << 2 | 1u << 3, (uint32_t)kUnity));
        v.push_back(inst_array(c->d.lev_f, 1, kInBlob | kInImage | kReset));
    }

    // volumes, preamp, loudness shelves and matrix / output gains of instance i of a set_params call, folded to Q15 / Q28
    static void pack(const dspi_chain_params_q28 &p, uint32_t i, uint32_t n, ParamRows<Q28> &r)
    {
        int32_t vol_mul = p.host_mute ? 0 : (int32_t)p.host_vol_mul;                                    // usb_audio.c:975
        r.vbase[i] = vol_mul;
        r.vmaster[i] = p.master_volume_q15;
        int32_t pmg = (int32_t)(p.preset_mute_gain * 32768.0f + 0.5f);                                  // :976-978
        if (pmg < 0) pmg = 0;
        if (pmg > 32768) pmg = 32768;
        r.pmg[i] = pmg;
        vol_mul = h_mul_q15(vol_mul, pmg);                                                              // :979
        const int32_t vol_mul_master = h_mul_q15(vol_mul, p.master_volume_q15);                         // :980
        r.preamp[0 * n + i] = p.preamp_q28[0];
        r.preamp[1 * n + i] = p.preamp_q28[1];
        for (int o = 0; o < kOuts; o++) {
            const dspi_output_channel &oc = p.matrix.outputs[o];
            const dspi_matrix_crosspoint &xl = p.matrix.crosspoints[0][o], &xr = p.matrix.crosspoints[1][o];
            r.gl[o * n + i] = xl.enabled ? h_f2i_sat((xl.phase_invert ? -xl.gain_linear : xl.gain_linear) * 32768.0f) : 0;   // :1084-1085
            r.gr[o * n + i] = xr.enabled ? h_f2i_sat((xr.phase_invert ? -xr.gain_linear : xr.gain_linear) * 32768.0f) : 0;
            r.gain[o * n + i] = oc.mute ? 0 : h_f2i_sat(oc.gain_linear * (float)vol_mul_master);        // :1204-1205
        }
        for (int j = 0; j < 2; j++) {
            const int32_t v[5] = { p.loudness[j].b0, p.loudness[j].b1, p.loudness[j].b2, p.loudness[j].a1, p.loudness[j].a2 };
            for (int k = 0; k < 5; k++) r.loud_c[(j * 5 + k) * n + i] = v[k];
        }
    }
};

}  // namespace
}  // namespace dspi

struct dspi_chainq : dspi::ChainHost<dspi::Q28> {};

#define CHAIN dspi_chainq
#define CHAIN_FN(name) dspi_chainq_##name
#define CHAIN_PARAMS dspi_chain_params_q28
#define CHAIN_BIQUAD dspi_biquad_q28
#define CHAIN_STATUS dspi_status_q28
#include "chain_abi.inc"
