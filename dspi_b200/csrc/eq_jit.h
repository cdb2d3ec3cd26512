// eq_jit.h — run-time specialised K1 kernels (eq_jit.cu)
#pragma once
#include "eq_kernels.cuh"

namespace dspi {
namespace jit {

// DSPI_JIT=0 disables run-time specialisation; DSPI_JIT=force specialises engines of any size
bool enabled_by_env(bool *force);

// Compile (once per process and signature) K1 for the topology vector `sig` (4 bits per band, bands
// >= nb zero) and the engine's channels per lane `cpl`.  Returns an opaque handle, or nullptr with the
// reason in `msg`.
void *acquire(uint64_t sig, bool fused, int nb, int cpl, int device, char *msg, size_t cap);

cudaError_t launch(void *handle, const EqLaunch &a, cudaStream_t stream, char *msg, size_t cap);

}  // namespace jit
}  // namespace dspi
