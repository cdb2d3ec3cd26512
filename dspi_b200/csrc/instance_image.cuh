// instance_image.cuh — the one kernel behind dspi_chain(q)_export_instances / _import_instances / _reset_instances (and
// the engines' reset_state): it moves the per-instance arrays of an instance range between the engine and instance
// images in a device staging buffer, or writes their reset values.  Its sibling behind _copy_instances moves the same
// arrays from listed instances to listed instances of the same engine.  The host side (which arrays, the image layout,
// the staging and the EQ sub-engines' pack / unpack around it) is chain_host.cuh.
//
// Every array is `rows` rows of N_pad elements with the instance index innermost, element (r, i) at p + (r N_pad + i) elem:
//   scalar fields (elem 1, 2, 4 or 8): a CTA takes 32 instances x up to 32 rows, reads them lane = instance (coalesced)
//     into a shared-memory tile and writes them out instance-major (each image holds the rows of a field back to back);
//   wide fields (elem a multiple of 16: a delay ring, a configuration packet, the 12 biquads of one EQ channel in the
//     sub-engine's reference-layout mirror): each element is one contiguous run, copied by one warp in 16-byte vectors,
//     at most kSegBytes per task so that a chunk's rings spread over many CTAs.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace dspi {
namespace image {

constexpr int kMaxFields = 48, kMaxTasks = 160;
constexpr uint32_t kSlabRows = 32, kSegBytes = 4096, kHeaderWords = 8;

// One array of the engine and where its rows sit in an image (`off` bytes from the image start).  A reset writes `one`
// into the rows of the mask `one_rows` (4-byte scalars) and 0 everywhere else.
struct Field {
    char *p;
    uint32_t rows, elem, off, one_rows, one;
};

// One CTA row of the grid: rows [first, first + count) of a scalar field, or row `first`, segment `count` of a wide one.
struct Task {
    uint8_t field, count;
    uint16_t first;
};

// Everything a launch needs; a kernel parameter (the arrays move between calls: widx_in / widx_out swap every call).
struct Plan {
    Field f[kMaxFields];
    Task t[kMaxTasks];
    uint32_t header[kHeaderWords];   // written at the start of every exported image
    uint32_t N_pad, n_fields, n_tasks;
    uint32_t used, bytes;            // bytes of an image holding data / with the zero tail up to a multiple of 16
};

enum Op : int { kExport = 0, kImport = 1, kReset = 2 };

namespace {                                  // one copy of the kernel per engine object

__device__ __forceinline__ unsigned long long load_elem(const char *p, uint32_t elem)
{
    switch (elem) {
    case 1: return *reinterpret_cast<const uint8_t *>(p);
    case 2: return *reinterpret_cast<const uint16_t *>(p);
    case 4: return *reinterpret_cast<const uint32_t *>(p);
    default: return *reinterpret_cast<const unsigned long long *>(p);
    }
}

__device__ __forceinline__ void store_elem(char *p, uint32_t elem, unsigned long long v)
{
    switch (elem) {
    case 1: *reinterpret_cast<uint8_t *>(p) = (uint8_t)v; break;
    case 2: *reinterpret_cast<uint16_t *>(p) = (uint16_t)v; break;
    case 4: *reinterpret_cast<uint32_t *>(p) = (uint32_t)v; break;
    default: *reinterpret_cast<unsigned long long *>(p) = v; break;
    }
}

// Instances [inst0, inst0 + n) of the engine <-> images [n][plan.bytes] (OP kExport / kImport), or their reset values
// (kReset: `images` unused).  grid (ceil(n / 32), plan.n_tasks), 256 threads.
template <int OP>
__global__ void __launch_bounds__(256) instance_image_kernel(const __grid_constant__ Plan plan, uint32_t inst0, uint32_t n,
                                                             unsigned char *__restrict__ images)
{
    __shared__ unsigned long long tile[kSlabRows][33];
    const uint32_t g0 = blockIdx.x * 32, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const Task t = plan.t[blockIdx.y];
    const Field &f = plan.f[t.field];
    const size_t Np = plan.N_pad, isz = plan.bytes;
    if (OP == kExport && blockIdx.y == 0 && warp == 0 && g0 + lane < n) {          // header and zero tail of each image
        uint32_t *h = reinterpret_cast<uint32_t *>(images + (size_t)(g0 + lane) * isz);
        for (uint32_t k = 0; k < kHeaderWords; k++) h[k] = plan.header[k];
        for (uint32_t b = plan.used; b < plan.bytes; b++) images[(size_t)(g0 + lane) * isz + b] = 0;
    }
    if (f.elem >= 16) {
        const uint32_t seg = (uint32_t)t.count * kSegBytes, rest = f.elem - seg;
        const uint32_t nv = (rest < kSegBytes ? rest : kSegBytes) / 16;
        for (uint32_t k = warp; k < 32 && g0 + k < n; k += 8) {
            const uint32_t i = g0 + k;
            uint4 *dev = reinterpret_cast<uint4 *>(f.p + ((size_t)t.first * Np + inst0 + i) * f.elem + seg);
            uint4 *img = OP == kReset ? nullptr : reinterpret_cast<uint4 *>(images + (size_t)i * isz + f.off + (size_t)t.first * f.elem + seg);
            for (uint32_t w0 = 0; w0 < nv; w0 += 4 * 32) {                           // four 16-byte loads in flight per lane
                uint4 v[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t w = w0 + j * 32 + lane;
                    if (w < nv) v[j] = OP == kExport ? dev[w] : OP == kImport ? img[w] : make_uint4(0, 0, 0, 0);
                }
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t w = w0 + j * 32 + lane;
                    if (w < nv) { if (OP == kExport) img[w] = v[j]; else dev[w] = v[j]; }
                }
            }
        }
        return;
    }
    const uint32_t E = f.elem, r0 = t.first, S = t.count;
    auto dev_at = [&](uint32_t r, uint32_t i) { return f.p + ((size_t)(r0 + r) * Np + inst0 + i) * E; };
    auto img_at = [&](uint32_t r, uint32_t i) { return reinterpret_cast<char *>(images) + (size_t)i * isz + f.off + (size_t)(r0 + r) * E; };
    if (OP == kReset) {
        if (g0 + lane < n)
            for (uint32_t r = warp; r < S; r += 8)
                store_elem(dev_at(r, g0 + lane), E, (r0 + r < 32 && (f.one_rows >> (r0 + r) & 1u)) ? f.one : 0u);
        return;
    }
    if (OP == kExport) {
        if (g0 + lane < n)
            for (uint32_t r = warp; r < S; r += 8) tile[r][lane] = load_elem(dev_at(r, g0 + lane), E);
        __syncthreads();
        for (uint32_t k = threadIdx.x; k < 32 * S; k += 256) {                      // consecutive threads: consecutive rows of one image
            const uint32_t ii = k / S, r = k % S;
            if (g0 + ii < n) store_elem(img_at(r, g0 + ii), E, tile[r][ii]);
        }
    } else {
        for (uint32_t k = threadIdx.x; k < 32 * S; k += 256) {
            const uint32_t ii = k / S, r = k % S;
            if (g0 + ii < n) tile[r][ii] = load_elem(img_at(r, g0 + ii), E);
        }
        __syncthreads();
        if (g0 + lane < n)
            for (uint32_t r = warp; r < S; r += 8) store_elem(dev_at(r, g0 + lane), E, tile[r][lane]);
    }
}

// Instance src[k] -> instance dst[k] for k < n, engine to engine with no image in between (dspi_chain(q)_copy_instances):
// the same plan and grid as above, with the lists in place of (inst0, n).  No index of dst appears in src, so no copy
// reads an element another copy writes; src may repeat.  Scalar fields: one thread per (row, k), element (r, src[k]) to
// (r, dst[k]); wide fields: one warp per (k, segment) in 16-byte vectors.
__global__ void __launch_bounds__(256) instance_copy_kernel(const __grid_constant__ Plan plan, uint32_t n, const uint32_t *__restrict__ src,
                                                            const uint32_t *__restrict__ dst)
{
    const uint32_t g0 = blockIdx.x * 32, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const Task t = plan.t[blockIdx.y];
    const Field &f = plan.f[t.field];
    const size_t Np = plan.N_pad;
    if (f.elem >= 16) {
        const uint32_t seg = (uint32_t)t.count * kSegBytes, rest = f.elem - seg;
        const uint32_t nv = (rest < kSegBytes ? rest : kSegBytes) / 16;
        for (uint32_t k = warp; k < 32 && g0 + k < n; k += 8) {
            const size_t row = (size_t)t.first * Np;
            const uint4 *from = reinterpret_cast<const uint4 *>(f.p + (row + src[g0 + k]) * f.elem + seg);
            uint4 *to = reinterpret_cast<uint4 *>(f.p + (row + dst[g0 + k]) * f.elem + seg);
            for (uint32_t w0 = 0; w0 < nv; w0 += 4 * 32) {                           // four 16-byte loads in flight per lane
                uint4 v[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t w = w0 + j * 32 + lane;
                    if (w < nv) v[j] = from[w];
                }
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint32_t w = w0 + j * 32 + lane;
                    if (w < nv) to[w] = v[j];
                }
            }
        }
        return;
    }
    if (g0 + lane >= n) return;
    const size_t s = src[g0 + lane], d = dst[g0 + lane];
    for (uint32_t r = warp; r < t.count; r += 8) {
        const size_t row = (size_t)(t.first + r) * Np;
        store_elem(f.p + (row + d) * f.elem, f.elem, load_elem(f.p + (row + s) * f.elem, f.elem));
    }
}

}  // namespace
}  // namespace image
}  // namespace dspi
