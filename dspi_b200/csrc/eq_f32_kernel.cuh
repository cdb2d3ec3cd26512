// eq_f32_kernel.cuh — body of K1 (see eq_f32.cu for the design notes).  Kept in a header that is safe
// for runtime compilation: the ahead-of-time build instantiates it for arbitrary topologies, the
// runtime compiler (eq_jit.cu) for ONE topology vector as a template constant.
#pragma once
#include "eq_core.cuh"

namespace dspi {
namespace k1 {

using namespace core;

// Geometry.  A warp streams its 32*CPL channels (rows) through a private ring of kStages stages of
// 8 KB; a CTA is kWarps such warps (192 KB of shared memory, one CTA per SM).  The stage of a
// one-channel-per-lane warp is 32 rows x 64 samples, that of a channel-pair warp 64 rows x 32
// samples.  A stage is loaded and stored as 32-sample boxes of 128 B per row (the 128-byte swizzle
// span), placed one after the other: chunk k (16 B, 4 samples) of row r lives at
//   (k / 8) * (rows * 128) + r * 128 + ((k % 8) ^ (r % 8)) * 16.
// The wide stage moves 256 B of every row per transfer, both ways, so each DRAM page opened for a
// row serves twice the data it does for 128 B.
constexpr int kStages = 3;
constexpr int kWarps = 8;
constexpr uint32_t kStageBytes = 8192;
template <typename V> __host__ __device__ constexpr int tile_t() { return 64 / Lanes<V>::CPL; }     // samples per stage
template <typename V> __host__ __device__ constexpr int sub_t() { return tile_t<V>() / 4; }          // samples per register tile

__device__ __forceinline__ uint32_t chunk_off(int r, int k, uint32_t half_bytes)
{
    return (uint32_t)(k >> 3) * half_bytes + r * 128 + ((((k & 7) ^ (r & 7))) << 4);
}

// SIG::enabled: the launch is known to have ONE topology vector SIG::word for every channel
struct NoSig { static constexpr bool enabled = false; static constexpr unsigned long long word = 0; };
template <unsigned long long W> struct SigWord { static constexpr bool enabled = true; static constexpr unsigned long long word = W; };

template <typename V, bool FUSED, int NB, bool DYN, typename SIG>
__device__ __forceinline__ void eq_f32_body(const CUtensorMap &tmap, float *__restrict__ samples, uint32_t ld, V *__restrict__ coef,
              const uint64_t *__restrict__ modes, uint32_t n_groups, uint32_t n_rows, uint32_t row_lo, uint32_t T, uint32_t nb_active, uint32_t use_tma, uint32_t dbg, unsigned long long nz_bits, uint32_t slice_tiles, uint32_t *__restrict__ sched)
{
    constexpr int CPL = Lanes<V>::CPL;
    constexpr int kRows = 32 * CPL;
    constexpr int kTileT = tile_t<V>();
    constexpr int kSub = sub_t<V>();
    constexpr int kHalves = kTileT / 32;                        // 32-sample boxes per stage
    constexpr uint32_t kHalfBytes = kRows * 128;
    static_assert(kRows * kTileT * 4 == (int)kStageBytes, "every geometry fills the same 8 KB stage");

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ uint64_t bars[kWarps][kStages];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    uint8_t *my_smem = smem_raw + (size_t)warp * kStages * kStageBytes;
    uint64_t *full = bars[warp];
    if (lane == 0) {
        if (use_tma) prefetch_tmap(&tmap);
        for (int s = 0; s < kStages; s++) mbar_init(&full[s], 1);
        fence_mbar_init();
    }
    __syncwarp();

    const V nz = v_bits<V>(nz_bits);                            // (-0.0, -0.0): see mulx()
    const uint32_t ntiles = (T + kTileT - 1) / kTileT;
    const bool mem_on = !(dbg & 2u);                            // diagnostics: DSPI_DBG=2 runs the arithmetic without HBM traffic

    // ---- work distribution -------------------------------------------------------------------
    // A work item is (group g, time slice k): `slice_tiles` consecutive tiles of the 32*CPL channels
    // of group g.  Static mode (sched == nullptr): one item per warp = the whole launch of group
    // blockIdx.x * kWarps + warp.  Dynamic mode: a persistent grid pulls items from an atomic counter
    // in slice-major order; the filter state of a group travels from slice to slice through the
    // coefficient store, ordered by a per-group completion counter (release/acquire).  65536
    // channels are 1024 groups for 592 warp schedulers: no static split can load them evenly, the
    // time slices can.
    const uint32_t n_slices = DYN ? (ntiles + slice_tiles - 1) / slice_tiles : 1;
    const uint32_t n_items = DYN ? n_groups * n_slices : 0;
    uint32_t tcount = 0;                                        // tiles this warp has pushed through its ring (stage / parity bookkeeping)
    for (;;) {
        uint32_t g, tile_begin, tile_end, slice = 0;
        if constexpr (DYN) {
            uint32_t item = 0;
            if (lane == 0) item = atomicAdd(&sched[0], 1u);
            item = __shfl_sync(0xffffffffu, item, 0);
            if (item >= n_items) break;
            slice = item / n_groups;
            g = item - slice * n_groups;
            tile_begin = slice * slice_tiles;
            tile_end = min(ntiles, tile_begin + slice_tiles);
            if (slice > 0) {                                    // wait until the previous slice of this group has published its state
                if (lane == 0) {
                    const volatile uint32_t *flag = sched + 1 + g;
                    while (*flag < slice) __nanosleep(100);
                    __threadfence();
                }
                __syncwarp();
            }
        } else {
            g = blockIdx.x * kWarps + warp;
            if (g >= n_groups) break;                           // warps are fully independent
            tile_begin = 0;
            tile_end = ntiles;
        }
        // first channel (row) of this group, counted from `samples`: group 0 starts row_lo rows before it (a range that
        // begins half-way into a 64-row group).  Rows from n_rows on belong to other launches: TMA clips them (zero-filled
        // loads, dropped stores).  A group that starts below row 0 takes the plain path, which skips the rows outside the
        // launch both ways, so that a TMA box never starts at a negative row.  No state is stored for rows outside.
        const int c0 = (int)(g * kRows) - (int)row_lo;
        const bool tma = use_tma && c0 >= 0;
        const uint32_t tcount0 = tcount;

        // boxes of a tile that start inside the row (a box wholly past T is neither loaded nor stored)
        auto n_boxes = [&](uint32_t tile) { return kHalves == 1 || tile * kTileT + 32 < T ? kHalves : 1; };
        auto issue_load = [&](uint32_t tile, uint32_t seq) {    // lane 0 only; seq = position in this warp's ring sequence
            const uint32_t s = seq % kStages;
            const int nb = n_boxes(tile);
            mbar_arrive_expect_tx(&full[s], nb * kHalfBytes);
            for (int h = 0; h < nb; h++)                        // back to back: every row's boxes arrive together
                tma_load_2d(my_smem + s * kStageBytes + h * kHalfBytes, &tmap, &full[s], tile * kTileT + h * 32, c0);
        };
        if (use_tma && mem_on && lane == 0) {
            if constexpr (DYN) tma_store_wait_read<0>();        // ring buffers of the previous item are drained
            for (uint32_t j = 0; tma && j + 1 < kStages && tile_begin + j < tile_end; j++) issue_load(tile_begin + j, tcount + j);
        }

        // ---- coefficients, state and topology of every band -> registers ----------------------
        EqBank<V, FUSED, NB> bank;
        V *my_coef = coef + (size_t)g * kMaxBands * 8 * 32 + lane;
        {
            const uint64_t *mp[CPL];
#pragma unroll
            for (int h = 0; h < CPL; h++) mp[h] = modes + (size_t)g * kRows + h * 32 + lane;
            bank.load(my_coef, mp, nb_active, DYN);
        }
        // register-tile (straight-line) path: all-biquad warps in the ahead-of-time kernels; warps whose
        // channels all carry the compiled-in topology vector in a runtime-specialised kernel
        bool straight = bank.all_tdf2;
        if constexpr (SIG::enabled) straight = bank.template sig_match<SIG::word>();

        // ---- stream the tiles of this item --------------------------------------------------------
        for (uint32_t tile = tile_begin; tile < tile_end; tile++, tcount++) {
            const uint32_t s = tcount % kStages;
            uint8_t *buf = my_smem + s * kStageBytes;
            if (tma) {
                if (mem_on) mbar_wait(&full[s], (tcount / kStages) & 1);
            } else {                                                // plain-load fallback (odd strides / unaligned bases)
                for (int r = 0; r < kRows; r++) {
                    const uint32_t ch = c0 + r;                 // rows below the launch wrap past n_rows
                    for (int h = 0; h < kHalves; h++) {
                        const uint32_t t = tile * kTileT + h * 32 + lane;
                        float v = 0.0f;
                        if (t < T && ch < n_rows) v = samples[(size_t)ch * ld + t];
                        *reinterpret_cast<float *>(buf + chunk_off(r, h * 8 + (lane >> 2), kHalfBytes) + ((lane & 3) << 2)) = v;
                    }
                }
                __syncwarp();
            }

            const int tile_valid = min((int)kTileT, (int)(T - tile * kTileT));
            // a partial tile whose length is a whole number of register tiles (the 32-sample tail of a 96-frame
            // packet in a 64-sample stage) stays on the straight-line path
            if (straight && tile_valid % kSub == 0 && !(dbg & 4u)) {
                // ---- all-biquad warps: register tiles of kSub samples, straight-line over the 10 bands ----
    #pragma unroll 1
                for (int sub = 0; sub < tile_valid / kSub; sub++) {
                    // kSub / 4 16-byte chunks per row per sub-tile (LDS.128, conflict-free: chunk index XOR (row & 7))
                    constexpr int kQ = kSub / 4;
                    V x[kSub];
                    float4 q[CPL][kQ];
    #pragma unroll
                    for (int h = 0; h < CPL; h++)
    #pragma unroll
                        for (int j = 0; j < kQ; j++)
                            q[h][j] = *reinterpret_cast<const float4 *>(buf + chunk_off(lane + 32 * h, kQ * sub + j, kHalfBytes));
    #pragma unroll
                    for (int i = 0; i < kSub; i++) {
                        float part[CPL];
    #pragma unroll
                        for (int h = 0; h < CPL; h++) {
                            const float4 &qq = q[h][i >> 2];
                            part[h] = (i & 3) == 0 ? qq.x : (i & 3) == 1 ? qq.y : (i & 3) == 2 ? qq.z : qq.w;
                        }
                        v_make(x[i], part);
                    }
                    if (!(dbg & 1u)) {                                 // DSPI_DBG=1: data path only
                        if constexpr (SIG::enabled) bank.template run_sig<SIG::word>(x, nz);
                        else bank.run(x, kSub, nz);
                    }
    #pragma unroll
                    for (int h = 0; h < CPL; h++)
    #pragma unroll
                        for (int j = 0; j < kQ; j++)
                            *reinterpret_cast<float4 *>(buf + chunk_off(lane + 32 * h, kQ * sub + j, kHalfBytes)) =
                                make_float4(Lanes<V>::get(x[4 * j], h), Lanes<V>::get(x[4 * j + 1], h), Lanes<V>::get(x[4 * j + 2], h),
                                            Lanes<V>::get(x[4 * j + 3], h));
                }
            } else {
                // ---- any other topology: band-outer over the tile, re-laid out in place as lane-private
                //      columns of CPL-vectors (sample n of this lane at col[n * 32]) ----
                float4 q[CPL][kTileT / 4];
    #pragma unroll
                for (int h = 0; h < CPL; h++)
    #pragma unroll
                    for (int k = 0; k < kTileT / 4; k++) q[h][k] = *reinterpret_cast<const float4 *>(buf + chunk_off(lane + 32 * h, k, kHalfBytes));
                __syncwarp();                                       // every row is in registers before columns overwrite them
                V *col = reinterpret_cast<V *>(buf) + lane;
    #pragma unroll
                for (int n = 0; n < kTileT; n++) {
                    float part[CPL];
    #pragma unroll
                    for (int h = 0; h < CPL; h++) {
                        const float4 &qq = q[h][n >> 2];
                        part[h] = (n & 3) == 0 ? qq.x : (n & 3) == 1 ? qq.y : (n & 3) == 2 ? qq.z : qq.w;
                    }
                    V v;
                    v_make(v, part);
                    col[n * 32] = v;
                }
                if (!(dbg & 1u)) bank.run_columns(col, tile_valid, nz);
                float back[CPL][kTileT];
    #pragma unroll
                for (int n = 0; n < kTileT; n++) {
                    const V v = col[n * 32];
    #pragma unroll
                    for (int h = 0; h < CPL; h++) back[h][n] = Lanes<V>::get(v, h);
                }
                __syncwarp();
    #pragma unroll
                for (int h = 0; h < CPL; h++)
    #pragma unroll
                    for (int k = 0; k < kTileT / 4; k++)
                        *reinterpret_cast<float4 *>(buf + chunk_off(lane + 32 * h, k, kHalfBytes)) =
                            make_float4(back[h][4 * k], back[h][4 * k + 1], back[h][4 * k + 2], back[h][4 * k + 3]);
            }

            if (tma) {
                fence_proxy_async_smem();                           // my smem writes -> async proxy
                __syncwarp();
                if (lane == 0 && mem_on) {
                    const int nb = n_boxes(tile);
                    for (int h = 0; h < nb; h++) tma_store_2d(&tmap, buf + h * kHalfBytes, tile * kTileT + h * 32, c0);
                    tma_store_commit();                             // the stage leaves as one bulk group
                    const uint32_t nxt = tile + kStages - 1;        // refill the buffer stored one iteration ago
                    if (nxt < tile_end) {
                        tma_store_wait_read<1>();
                        issue_load(nxt, tcount + kStages - 1);
                    }
                }
            } else {
                __syncwarp();
                for (int r = 0; r < kRows; r++) {
                    const uint32_t ch = c0 + r;
                    for (int h = 0; h < kHalves; h++) {
                        const uint32_t t = tile * kTileT + h * 32 + lane;
                        const float v = *reinterpret_cast<const float *>(buf + chunk_off(r, h * 8 + (lane >> 2), kHalfBytes) + ((lane & 3) << 2));
                        if (t < T && ch < n_rows) samples[(size_t)ch * ld + t] = v;
                    }
                }
                __syncwarp();
            }
        }


        if (!tma) tcount = tcount0;                             // the TMA ring's stage / parity sequence only counts TMA tiles
        int h_lo = 0, h_hi = 0;                                 // this lane's channels lane + 32 h, h in [h_lo, h_hi), are in the launch
#pragma unroll
        for (int h = 0; h < CPL; h++) {
            if (c0 + 32 * h + lane < 0) h_lo = h + 1;
            if ((uint32_t)(c0 + 32 * h + lane) < n_rows) h_hi = h + 1;
        }
        bank.store(my_coef, h_lo, h_hi, DYN);                   // filter state back to the coefficient store
        if constexpr (!DYN) break;
        __threadfence();                                        // state visible before the slice counter moves
        __syncwarp();
        if (lane == 0) atomicExch(&sched[1 + g], slice + 1);
    }
    if (use_tma && lane == 0) tma_store_wait_all<0>();          // smem must outlive the bulk reads
}


}  // namespace k1
}  // namespace dspi
