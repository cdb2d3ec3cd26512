// eq_f32_jit_entry.cuh — translation unit compiled AT RUN TIME by eq_jit.cu (NVRTC) for one engine-wide
// topology vector: -DDSPI_JIT_SIG=<4 bits per band> -DDSPI_JIT_FUSED=<0|1> -DDSPI_JIT_CPL=<1|2>.  With the
// topology a template constant the whole 10-band cascade of K1 is one straight-line block for ANY mix of
// SVF / TDF2 bands (the ahead-of-time build only has that for all-biquad warps).  DSPI_JIT_CPL is the
// engine's channels per lane, which fixes the packed store layout and the stage geometry.
#include "eq_f32_kernel.cuh"

#ifndef DSPI_JIT_NB
#define DSPI_JIT_NB 10
#endif
#if DSPI_JIT_CPL == 2
typedef dspi::core::P2 JitV;
#else
typedef float JitV;
#endif

extern "C" __global__ void __launch_bounds__(dspi::k1::kWarps * 32, 1)
eq_f32_jit(const __grid_constant__ CUtensorMap tmap, float *__restrict__ samples, uint32_t ld, JitV *__restrict__ coef,
           const uint64_t *__restrict__ modes, uint32_t n_groups, uint32_t n_rows, uint32_t row_lo, uint32_t T, uint32_t nb_active, uint32_t use_tma, uint32_t dbg,
           unsigned long long nz_bits, uint32_t slice_tiles, uint32_t *__restrict__ sched)
{
    dspi::k1::eq_f32_body<JitV, (DSPI_JIT_FUSED) != 0, DSPI_JIT_NB, false, dspi::k1::SigWord<(DSPI_JIT_SIG)>>(
        tmap, samples, ld, coef, modes, n_groups, n_rows, row_lo, T, nb_active, use_tma, dbg, nz_bits, slice_tiles, sched);
}
