// chain_pdm.cuh — the 2nd-order error-feedback delta-sigma PDM modulator shared by the float and the
// Q28 chain (the firmware feeds it Q28 samples on both platforms: usb_audio.c:953 / :1270).
// Reference: pdm_generator.c:351-397 (steady-state branch: hardware running, a sample available, no
// fade-out), xorshift32 :62-68, noise-shaped TPDF dither :89-108, constants config.h:59-75.
#pragma once
#include <stdint.h>

namespace dspi {

// state words (SoA, [9][Np]): err1 err2 x1 x2 y1 y2 err_acc rng fade_in_pos.
// Modulates frames [f_begin, f_end) of instance `inst`: Q28 samples at subq[f * frame_stride] (the
// caller offsets `subq` to this instance), 8 words (256 bits, MSB first) per frame to
// pdm_out[f * 8 ..] (the caller offsets `pdm_out` to this instance's row).
__device__ __forceinline__ void pdm_modulate_frames(int32_t *__restrict__ pdm, const int32_t *__restrict__ subq, size_t frame_stride, uint32_t Np,
                                                    uint32_t inst, uint32_t f_begin, uint32_t f_end, uint32_t *__restrict__ pdm_out)
{
    int32_t err1 = pdm[0 * Np + inst], err2 = pdm[1 * Np + inst];
    int32_t x1 = pdm[2 * Np + inst], x2 = pdm[3 * Np + inst], y1 = pdm[4 * Np + inst], y2 = pdm[5 * Np + inst];
    int32_t err_acc = pdm[6 * Np + inst];
    uint32_t rng = (uint32_t)pdm[7 * Np + inst], fade = (uint32_t)pdm[8 * Np + inst];
    int32_t q_next = f_begin < f_end ? subq[(size_t)f_begin * frame_stride] : 0;
    for (uint32_t f = f_begin; f < f_end; f++) {
        int32_t pcm = q_next >> 14;                                          // :352
        if (f + 1 < f_end) q_next = subq[(size_t)(f + 1) * frame_stride];       // next frame's load overlaps this frame's 256 decisions
        pcm = max(-29500, min(29500, pcm));                                  // :353-354
        if (fade < 1024u) { pcm = (pcm * (int32_t)fade) >> 10; fade++; }     // :357-360
        const int32_t target = pcm + 32768;
        uint32_t words[8];
#pragma unroll
        for (int chunk = 0; chunk < 8; chunk++) {
            rng ^= rng << 13; rng ^= rng >> 17; rng ^= rng << 5;             // :63-68
            const int32_t raw = (int32_t)(rng & 0x1FFu) - 255;               // :368
            err_acc = ((err_acc * 248) >> 8) + ((err2 >> 8) >> 6);           // :92
            const int32_t in = raw - err_acc;
            const int32_t dither = (15778 * in - 31556 * x1 + 15778 * x2 + 31531 * y1 - 15580 * y2) >> 14;   // :98-99
            x2 = x1; x1 = in; y2 = y1; y1 = dither;
            // :372-378 restated on three running sums so that only TWO dependent integer ops separate consecutive
            // decisions and neither waits for a late operand (the loop is one serial chain per instance, its depth is the cost):
            //   s = err2 + dither (the comparator input)   g = err1 + target
            //   bit = s >= 0;   s' = s + g - 2*fb;   g' = g + target - fb        (fb = bit ? K : 0, K = 65535)
            // which is err1 += target - fb; err2 += err1 - fb with the substitutions above (all int32, wrapping like the
            // reference).  With m = s >> 31 (0 when the bit is 1, -1 when it is 0), t2 = s + g - 2K and g2 = g + target - K:
            //   s' = m * -2K + t2      t2' = s' + g' - 2K = m * -3K + (t2 + g2 - 2K)      g2' = g' + target - K = m * -K + (g2 + target - K)
            // Every addend on the right depends on the PREVIOUS step only, so a decision is one shift (ALU pipe) feeding
            // three independent IMADs (FMA pipe): the shortest dependence per decision of the forms scripts/pdm_ubench.cu
            // compares (two sums, an fp32 formulation, the mask form, predicated corrections, the reference's own order).
            uint32_t inv = 0;                                                // complement of the output word
            int32_t s = err2 + dither;
            const int32_t tg = target - 65535;
            int32_t g2 = err1 + target + tg;
            int32_t t2 = s + g2 - 65535 - target;                            // s + g - 2K with g = g2 - tg
#pragma unroll
            for (int k = 0; k < 32; k++) {
                const int32_t m = s >> 31;
                const int32_t a = t2 + g2 - 2 * 65535;
                const int32_t b = g2 + tg;
                inv = __funnelshift_l((uint32_t)s, inv, 1);                  // shift the sign in, MSB first (:375)
                s = m * (-2 * 65535) + t2;
                t2 = m * (-3 * 65535) + a;
                g2 = m * -65535 + b;
            }
            const uint32_t word = ~inv;
            err2 = s - dither;
            err1 = g2 - tg - target;
            words[chunk] = word;
        }
        err1 -= err1 >> 16;                                                  // :396-397
        err2 -= err2 >> 16;
        if (pdm_out) {
            uint4 *dst = reinterpret_cast<uint4 *>(pdm_out + (size_t)f * 8);
            dst[0] = make_uint4(words[0], words[1], words[2], words[3]);
            dst[1] = make_uint4(words[4], words[5], words[6], words[7]);
        }
    }
    pdm[0 * Np + inst] = err1; pdm[1 * Np + inst] = err2;
    pdm[2 * Np + inst] = x1; pdm[3 * Np + inst] = x2; pdm[4 * Np + inst] = y1; pdm[5 * Np + inst] = y2;
    pdm[6 * Np + inst] = err_acc; pdm[7 * Np + inst] = (int32_t)rng; pdm[8 * Np + inst] = (int32_t)fade;
}

}  // namespace dspi
