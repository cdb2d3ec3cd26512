// spdif_bmc.cuh — IEC 60958 biphase-mark subframe encoding, the one implementation shared by the standalone encoder
// (spdif.cu) and the chain engines' output stage (chain_f32.cu / chain_q28.cu).
//
// Reference (firmware/pico-extras/src/rp2_common/pico_audio_spdif_multi/):
//   spdif_update_subframe   include/pico/audio_spdif/sample_encoding.h:27-50   (3 table look-ups per sample)
//   table                   audio_spdif.c:141-153   (byte -> 16-bit biphase-mark word + parity)
//   preambles / channel status / validity-user-status-parity cells   audio_spdif.c:73-114, :372-388
//
// The table is replaced by arithmetic (no shared-memory bank conflicts, nothing to initialise): the biphase-mark word of
// k data bits is 0x55..5 with bit 2j+1 set where data bit j is set, i.e. a bit spread of the sample (four shift-or-mask
// steps per 12 bits).  A frame at block position `pos` (0..191) carries preamble Z (block start) or X on its left
// subframe, Y on its right one, and channel-status bit `pos` of the 5 consumer status bytes (zero past bit 39) in both.
#pragma once

#include <cstdint>

#include "dspi_b200.h"

namespace dspi {

// 12 data bits -> 24 bits with data bit j at position 2j
__device__ __forceinline__ uint32_t spread12(uint32_t t)
{
    t = (t | (t << 8)) & 0x00FF00FFu;
    t = (t | (t << 4)) & 0x0F0F0F0Fu;
    t = (t | (t << 2)) & 0x33333333u;
    t = (t | (t << 1)) & 0x55555555u;
    return t;
}

// one subframe (sample_encoding.h:27-50 with the table written out): `pre` = preamble byte,
// `c` = channel-status bit of this block position
__device__ __forceinline__ uint2 encode_subframe(int32_t sample, uint32_t pre, uint32_t c)
{
    const uint32_t x = (uint32_t)sample & 0x00FFFFFFu;
    const uint32_t lo = 0x00555555u | (spread12(x & 0xFFFu) << 1);          // cells of sample bits 0-11  -> l[31:8]
    const uint32_t hi = 0x00555555u | (spread12(x >> 12) << 1);             // cells of sample bits 12-23 -> h[23:0]
    const uint32_t p = (__popc(x) & 1u) ^ c;                                 // even parity over data + C (V = U = 0), :43-48
    uint2 r;
    r.x = pre | (lo << 8);
    r.y = hi | ((0x55u | (c << 5)) << 24) | (p << 31);                       // initial h = 0x55000000 | c << 29 (audio_spdif.c:106)
    return r;
}

// channel-status bit of block position `pos`; cs40 = the 5 status bytes, byte i in bits 8i..8i+7 (audio_spdif.c:91-94)
__device__ __forceinline__ uint32_t spdif_cs_bit(uint32_t pos, uint64_t cs40) { return pos < 40u ? (uint32_t)(cs40 >> pos) & 1u : 0u; }

// preamble of the left subframe: Z at block start, X elsewhere (:77-79, :104, :374)
__device__ __forceinline__ uint32_t spdif_pre_left(uint32_t pos) { return pos == 0 ? 0x39u : 0xC9u; }

constexpr uint32_t kSpdifPreY = 0x69u;                                       // preamble of the right subframe

// one stereo frame {l, h, l, h} from its two 24-bit words
__device__ __forceinline__ uint4 encode_frame(int2 w, uint32_t pre_l, uint32_t c)
{
    const uint2 a = encode_subframe(w.x, pre_l, c);
    const uint2 b = encode_subframe(w.y, kSpdifPreY, c);
    return make_uint4(a.x, a.y, b.x, b.y);
}

// ---- the chain engines' transmitter state --------------------------------------------------------------------------
// One S/PDIF transmitter per chain instance (audio_spdif.c:82-88, :372-388), shared by all its pairs (the firmware starts
// them together and feeds them the same frames): frame T of a call sits at block position (bp + T) % 192 on every pair.
// Only the outpost and ring kernels use it, so it travels as their last parameter instead of growing the engines' device
// structs, which every stage kernel takes by value.
struct SpdifTx {
    uint32_t *bp;                                 // [N_pad] block position of the next frame, 0..191
    uint64_t *cs40;                               // [N_pad] the 5 consumer channel-status bytes, byte i in bits 8i..8i+7
};

// the status bytes init_spdif_buffer() stamps (audio_spdif.c:82-88; byte 3, the sample-rate code, is left 0)
constexpr uint64_t kSpdifDefaultCs40 = 0x04ull | (0x0Bull << 32);

// records -> device rows; false (nothing written) when a block position is out of range
inline bool spdif_tx_unpack(const dspi_spdif_tx *tx, uint32_t n, uint32_t *bp, uint64_t *cs40)
{
    for (uint32_t i = 0; i < n; i++) {
        if (tx[i].block_pos >= 192) return false;
        uint64_t cs = 0;
        for (int b = 0; b < 5; b++) cs |= (uint64_t)tx[i].channel_status[b] << (8 * b);
        bp[i] = tx[i].block_pos;
        cs40[i] = cs;
    }
    return true;
}

inline void spdif_tx_pack(const uint32_t *bp, const uint64_t *cs40, uint32_t n, dspi_spdif_tx *tx)
{
    for (uint32_t i = 0; i < n; i++) {
        for (int b = 0; b < 5; b++) tx[i].channel_status[b] = (uint8_t)(cs40[i] >> (8 * b));
        tx[i].block_pos = (uint8_t)bp[i];
        tx[i].reserved[0] = tx[i].reserved[1] = 0;
    }
}

}  // namespace dspi
