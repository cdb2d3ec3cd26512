// response.cuh — frequency response of the engines' linear, time-invariant path, shared by the EQ engine
// (response.cu) and the two chain engines (chain_f32.cu, chain_q28.cu).
//
// Every filter stage is a recurrence with two state variables.  Its transfer function is that of the 2-state model
// s' = A s + B x, y = C s + D x:  H(w) = D + w C adj(I - w A) B / det(I - w A), w = z^-1, i.e. one rational section
// (n0 + n1 w + n2 w^2) / (1 + d1 w + d2 w^2).  The sections are formed from the engine's own device records in double and
// evaluated at w = e^{-j omega} in double; only the final value is rounded (once) to float.
//   - TDF2 band (dsp_pipeline.c:347-362, firmware signs: s1 = b1 x - a1 y + s2, s2 = b2 x - a2 y, y = b0 x + s1):
//     A = [[-a1, 1], [-a2, 0]], B = [b1 - a1 b0, b2 - a2 b0], C = [1, 0], D = b0, whose section is exactly
//     (b0, b1, b2, a1, a2) - taken as such, so no cancellation enters.
//   - SVF band (SVF_STEP, dsp_pipeline.c:301-306, state [ic1, ic2]):
//     A = [[2 a1 - 1, -2 a2], [2 a2, 1 - 2 a3]], B = [2 a2, 2 a3], v1 = [a1, -a2] s + a2 x, v2 = [a2, 1 - a3] s + a3 x,
//     y = v2 (low-pass), x + m1 v1 - v2 (high-pass), x + m1 v1 (peaking), m0 x + m1 v1 + m2 v2 (any other type).
//   - Q28 coefficients enter as value / 2^28.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <new>
#include <cuda_runtime.h>
#include "dspi_b200.h"

namespace dspi {

constexpr uint32_t kRespMaxFreqs = 65536;         // most frequencies of one response call
constexpr uint32_t kFreqChunk = 7936;             // parameter block of freq_table_kernel: 31.8 KB of the 32 KB sm_90 allows
struct FreqChunk { uint32_t first, count; float v[kFreqChunk]; };

struct Sect { double n0, n1, n2, d1, d2; };       // (n0 + n1 w + n2 w^2) / (1 + d1 w + d2 w^2)
struct Cd { double re, im; };

__host__ __device__ __forceinline__ Cd cmul(Cd a, Cd b) { return { a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re }; }
__host__ __device__ __forceinline__ Cd cscale(Cd a, double s) { return { a.re * s, a.im * s }; }
__host__ __device__ __forceinline__ Cd cadd(Cd a, Cd b) { return { a.re + b.re, a.im + b.im }; }
__host__ __device__ __forceinline__ Cd cdiv(Cd a, Cd b)
{
    const double r = 1.0 / (b.re * b.re + b.im * b.im);
    return { (a.re * b.re + a.im * b.im) * r, (a.im * b.re - a.re * b.im) * r };
}

__host__ __device__ __forceinline__ Sect sect_tdf2(double b0, double b1, double b2, double a1, double a2) { return { b0, b1, b2, a1, a2 }; }

// section of a 2-state model (see the file comment)
__host__ __device__ inline Sect sect_state(double A00, double A01, double A10, double A11, double B0, double B1, double C0, double C1, double D)
{
    const double tr = A00 + A11, det = A00 * A11 - A01 * A10;
    const double cb = C0 * B0 + C1 * B1;
    const double k2 = C0 * A01 * B1 + C1 * A10 * B0 - C0 * B0 * A11 - C1 * B1 * A00;
    return { D, cb - D * tr, D * det + k2, -tr, det };
}

// the SVF of SVF_STEP with the output mix of svf_type (DSPI_FILTER_*); general = true: the loudness shelves' mix (:702)
__host__ __device__ inline Sect sect_svf(double a1, double a2, double a3, double m0, double m1, double m2, uint32_t svf_type, bool general)
{
    const double v1c0 = a1, v1c1 = -a2, v1d = a2, v2c0 = a2, v2c1 = 1.0 - a3, v2d = a3;
    double C0, C1, D;
    if (!general && svf_type == DSPI_FILTER_LOWPASS) { C0 = v2c0; C1 = v2c1; D = v2d; }
    else if (!general && svf_type == DSPI_FILTER_HIGHPASS) { C0 = m1 * v1c0 - v2c0; C1 = m1 * v1c1 - v2c1; D = 1.0 + m1 * v1d - v2d; }
    else if (!general && svf_type == DSPI_FILTER_PEAKING) { C0 = m1 * v1c0; C1 = m1 * v1c1; D = 1.0 + m1 * v1d; }
    else { C0 = m1 * v1c0 + m2 * v2c0; C1 = m1 * v1c1 + m2 * v2c1; D = m0 + m1 * v1d + m2 * v2d; }
    return sect_state(2.0 * a1 - 1.0, -2.0 * a2, 2.0 * a2, 1.0 - 2.0 * a3, 2.0 * a2, 2.0 * a3, C0, C1, D);
}

// one band of filters[][] (float engines): false when it is bypassed
__host__ __device__ inline bool sect_band(const dspi_biquad_f32 &q, Sect &s)
{
    if (q.bypass) return false;
    if (q.use_svf) s = sect_svf(q.sva1, q.sva2, q.sva3, q.svm0, q.svm1, q.svm2, q.svf_type, false);
    else s = sect_tdf2(q.b0, q.b1, q.b2, q.a1, q.a2);
    return true;
}

__host__ __device__ inline bool sect_band(const dspi_biquad_q28 &q, Sect &s)
{
    if (q.bypass) return false;
    const double k = 1.0 / 268435456.0;
    s = sect_tdf2(q.b0 * k, q.b1 * k, q.b2 * k, q.a1 * k, q.a2 * k);
    return true;
}

// w = e^{-j omega} and w^2 at one frequency
struct Trig { double c1, s1, c2, s2; };

__device__ __forceinline__ Trig trig_at(float f, float fs)
{
    const double x = (double)f / (double)fs;     // cycles per sample, <= 0.5
    Trig t;
    sincospi(2.0 * x, &t.s1, &t.c1);
    sincospi(4.0 * x, &t.s2, &t.c2);
    t.s1 = -t.s1;
    t.s2 = -t.s2;
    return t;
}

__device__ __forceinline__ void sect_eval(const Sect &s, const Trig &t, Cd &num, Cd &den)
{
    const Cd n = { s.n0 + s.n1 * t.c1 + s.n2 * t.c2, s.n1 * t.s1 + s.n2 * t.s2 };
    const Cd d = { 1.0 + s.d1 * t.c1 + s.d2 * t.c2, s.d1 * t.s1 + s.d2 * t.s2 };
    num = cmul(num, n);
    den = cmul(den, d);
}

// H of a cascade of `count` sections
__device__ __forceinline__ Cd cascade_eval(const Sect *s, int count, const Trig &t)
{
    Cd num = { 1.0, 0.0 }, den = { 1.0, 0.0 };
    for (int i = 0; i < count; i++) sect_eval(s[i], t, num, den);
    return count ? cdiv(num, den) : num;
}

// e^{-j 2 pi f d / fs}: f * d is exact in double (24-bit f, d < 2^13), so the phase in cycles carries one rounding (the
// division) and is reduced to [-1/2, 1/2] exactly before sincospi - a 4096-sample delay near Nyquist keeps full precision
__device__ __forceinline__ Cd delay_phase(float f, uint32_t d, float fs)
{
    double t = (double)f * (double)d / (double)fs;
    t -= rint(t);
    Cd r;
    sincospi(2.0 * t, &r.im, &r.re);
    r.im = -r.im;
    return r;
}

__device__ __forceinline__ float2 to_float2(Cd h) { return make_float2(__double2float_rn(h.re), __double2float_rn(h.im)); }

namespace {
__global__ void __launch_bounds__(256) freq_table_kernel(float *__restrict__ d_freq, const FreqChunk chunk)
{
    for (uint32_t i = threadIdx.x; i < chunk.count; i += blockDim.x) d_freq[chunk.first + i] = chunk.v[i];
}
}  // namespace

// Argument checks shared by every response entry point (before the engine is looked at): *why names the fault.
inline int response_check_args(const float *freqs, uint32_t n_freqs, float fs, const void *out, const char **why)
{
    if (!freqs || !out) { *why = "null frequency table or output"; return DSPI_EINVAL; }
    if (n_freqs == 0 || n_freqs > kRespMaxFreqs) { *why = "n_freqs must be 1..65536"; return DSPI_EINVAL; }
    if (!(fs > 0.0f) || fs > 3.4e38f) { *why = "sample_rate must be positive and finite"; return DSPI_EINVAL; }
    for (uint32_t i = 0; i < n_freqs; i++)
        if (!(freqs[i] >= 0.0f && (double)freqs[i] <= 0.5 * (double)fs)) { *why = "every frequency must be 0 <= f <= sample_rate / 2"; return DSPI_EINVAL; }
    return DSPI_OK;
}

// Per-engine device buffers of the response calls: the frequency table (kRespMaxFreqs floats) and the bounded staging
// buffer of the _host forms; both allocated at first use.
struct ResponseBuffers {
    float *d_freq = nullptr;
    void *d_stage = nullptr;
    size_t stage_bytes = 0;
    FreqChunk *chunk = nullptr;

    void destroy()
    {
        if (d_freq) cudaFree(d_freq);
        if (d_stage) cudaFree(d_stage);
        delete chunk;
        d_freq = nullptr; d_stage = nullptr; stage_bytes = 0; chunk = nullptr;
    }

    // The table reaches the device as kernel parameters, like the packet schedule (chain_schedule.cuh): each launch
    // captures its chunk when it is issued, so the caller may reuse `freqs` as soon as the call returns, and the copy is
    // ordered on `stream` behind the earlier response kernels that read d_freq.
    cudaError_t upload(const float *freqs, uint32_t n, cudaStream_t stream, uint64_t *launches)
    {
        if (!d_freq) {
            cudaError_t e = cudaMalloc((void **)&d_freq, (size_t)kRespMaxFreqs * sizeof(float));
            if (e != cudaSuccess) { d_freq = nullptr; return e; }
        }
        if (!chunk && !(chunk = new (std::nothrow) FreqChunk)) return cudaErrorMemoryAllocation;
        for (uint32_t first = 0; first < n; first += kFreqChunk) {
            chunk->first = first;
            chunk->count = n - first < kFreqChunk ? n - first : kFreqChunk;
            memcpy(chunk->v, freqs + first, (size_t)chunk->count * sizeof(float));
            freq_table_kernel<<<1, 256, 0, stream>>>(d_freq, *chunk);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return e;
            ++*launches;
        }
        return cudaSuccess;
    }

    // rows per chunk of a _host call whose rows are `row_bytes` each (32 MiB chunks; DSPI_HOST_CHUNK_MB overrides, as for
    // dspi_eq_process_host), with the staging buffer grown to hold one chunk
    cudaError_t stage(size_t row_bytes, uint32_t n_rows, cudaStream_t stream, uint32_t *rows_per_chunk)
    {
        const char *v = getenv("DSPI_HOST_CHUNK_MB");
        const long mb = v ? atol(v) : 0;
        const size_t cap = (size_t)(mb >= 1 && mb <= 1024 ? mb : 32) << 20;
        size_t rows = cap / row_bytes;
        if (rows < 1) rows = 1;
        if (rows > n_rows) rows = n_rows;
        const size_t need = rows * row_bytes;
        if (need > stage_bytes) {
            cudaError_t e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) return e;
            if (d_stage) cudaFree(d_stage);
            d_stage = nullptr; stage_bytes = 0;
            if ((e = cudaMalloc(&d_stage, need)) != cudaSuccess) { d_stage = nullptr; return e; }
            stage_bytes = need;
        }
        *rows_per_chunk = (uint32_t)rows;
        return cudaSuccess;
    }
};

}  // namespace dspi
