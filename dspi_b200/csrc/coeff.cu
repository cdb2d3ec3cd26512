// coeff.cu — parameter ingest on the device (SURVEY.md §8 f-1): dsp_compute_coefficients() for many
// channels at once, written straight into an EQ engine's stores.
//
// Reference: dsp_compute_coefficients(), firmware/DSPi/dsp_pipeline.c:61-175 (is_filter_flat :6-17; clamps
// written back into the recipe :78-81; topology choice and state reset on a flip :87-92; Cytomic SVF :94-138;
// RBJ cookbook :145-156; float store through inv_a0 :160-165; Q28 store (int32)((b/a0)*2^28) :168-173).
//
// One thread per (channel, band).  Every arithmetic operation is the reference's float operation, rounded on
// its own (-fmad=false, explicit division / square root: IEEE).  The five libm calls (powf, tanf, sinf, cosf;
// sqrtf is exact everywhere) follow the library's libm policy (DESIGN.md §6): evaluated in double precision and
// rounded once to float, i.e. the correctly rounded float function — newlib on the firmware, glibc on a host
// and CUDA's float libm each differ from that, and from each other, in occasional last bits.  The oracle has
// the same definition behind orc_set_libm_f64(1).
#include "eq_kernels.cuh"

namespace dspi {
namespace {

constexpr float kPi = 3.1415926535f;                     // the reference's literal, dsp_pipeline.c:97,145

// nvcc rewrites `x / constant` into a multiplication by the rounded reciprocal even under -prec-div=true
// (seen in the PTX: gain_db / 40.0f became mul.rn by 0x3CCCCCCD): every division is spelled as the IEEE intrinsic
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ float pow10_f(float x) { return (float)pow(10.0, (double)x); }
__device__ __forceinline__ float sin_f(float x) { return (float)sin((double)x); }
__device__ __forceinline__ float cos_f(float x) { return (float)cos((double)x); }
__device__ __forceinline__ float tan_f(float x) { return (float)tan((double)x); }

__device__ __forceinline__ bool recipe_is_flat(const dspi_eq_param &p)                   // :6-17
{
    if (p.type == DSPI_FILTER_FLAT || p.freq <= 0.0f) return true;
    if (p.type == DSPI_FILTER_PEAKING || p.type == DSPI_FILTER_LOWSHELF || p.type == DSPI_FILTER_HIGHSHELF) return fabsf(p.gain_db) < 0.01f;
    return false;
}

__device__ __forceinline__ void recipe_clamp(dspi_eq_param &p, float fs)                // :78-81
{
    float q = p.Q, f = p.freq;
    if (q < 0.1f) q = 0.1f;
    if (q > 20.0f) q = 20.0f;
    if (f < 10.0f) f = 10.0f;
    if (f > fs * 0.45f) f = fs * 0.45f;
    p.Q = q;
    p.freq = f;
}

// un-normalised RBJ cookbook section, :145-156; n = {b0,b1,b2}, d = {a0,a1,a2}
__device__ void cookbook(const dspi_eq_param &p, float A, float fs, float (&n)[3], float (&d)[3])
{
    const float omega = fdiv(2.0f * kPi * p.freq, fs);
    const float sn = sin_f(omega), cs = cos_f(omega);
    const float alpha = fdiv(sn, 2.0f * p.Q);
    n[0] = 1.0f; n[1] = 0.0f; n[2] = 0.0f;
    d[0] = 1.0f; d[1] = 0.0f; d[2] = 0.0f;
    const float sA = fsqrt(A);
    switch (p.type) {
    case DSPI_FILTER_LOWPASS:
        n[0] = fdiv(1 - cs, 2.0f); n[1] = 1 - cs; n[2] = fdiv(1 - cs, 2.0f);
        d[0] = 1 + alpha; d[1] = -2 * cs; d[2] = 1 - alpha;
        break;
    case DSPI_FILTER_HIGHPASS:
        n[0] = fdiv(1 + cs, 2.0f); n[1] = -(1 + cs); n[2] = fdiv(1 + cs, 2.0f);
        d[0] = 1 + alpha; d[1] = -2 * cs; d[2] = 1 - alpha;
        break;
    case DSPI_FILTER_PEAKING:
        n[0] = 1 + alpha * A; n[1] = -2 * cs; n[2] = 1 - alpha * A;
        d[0] = 1 + fdiv(alpha, A); d[1] = -2 * cs; d[2] = 1 - fdiv(alpha, A);
        break;
    case DSPI_FILTER_LOWSHELF:
        n[0] = A * ((A + 1) - (A - 1) * cs + 2 * sA * alpha);
        n[1] = 2 * A * ((A - 1) - (A + 1) * cs);
        n[2] = A * ((A + 1) - (A - 1) * cs - 2 * sA * alpha);
        d[0] = (A + 1) + (A - 1) * cs + 2 * sA * alpha;
        d[1] = -2 * ((A - 1) + (A + 1) * cs);
        d[2] = (A + 1) + (A - 1) * cs - 2 * sA * alpha;
        break;
    case DSPI_FILTER_HIGHSHELF:
        n[0] = A * ((A + 1) + (A - 1) * cs + 2 * sA * alpha);
        n[1] = -2 * A * ((A - 1) + (A + 1) * cs);
        n[2] = A * ((A + 1) + (A - 1) * cs - 2 * sA * alpha);
        d[0] = (A + 1) - (A - 1) * cs + 2 * sA * alpha;
        d[1] = 2 * ((A - 1) - (A + 1) * cs);
        d[2] = (A + 1) - (A - 1) * cs - 2 * sA * alpha;
        break;
    default:
        break;
    }
}

// thread i = channel * 12 + band of role blockIdx.y: inside the range, not rejected, and in the band mask if there is one
__device__ __forceinline__ bool band_selected(uint32_t i, uint32_t n, const RoleRange &rr)
{
    if (i >= n * kMaxBands || (rr.reject && rr.reject[i / kMaxBands])) return false;
    return !rr.band_mask || ((rr.band_mask[(size_t)blockIdx.y * n + i / kMaxBands] >> (i % kMaxBands)) & 1u);
}
// its biquad in the role's rows: channel i / 12 of the range, or inst[i / 12] of a list
__device__ __forceinline__ size_t band_index(uint32_t i, const RoleRange &rr)
{
    return rr.inst ? (size_t)rr.inst[i / kMaxBands] * kMaxBands + i % kMaxBands : (size_t)i;
}

__global__ void __launch_bounds__(256)
coeff_f32_kernel(dspi_eq_param *__restrict__ recipes, dspi_biquad_f32 *__restrict__ aos, uint32_t ch0, uint32_t n, float fs, RoleRange rr)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!band_selected(i, n, rr)) return;
    if (rr.fs) fs = rr.fs[i / kMaxBands];
    recipes += (size_t)blockIdx.y * n * kMaxBands;
    aos += ((size_t)ch0 + (size_t)blockIdx.y * rr.stride) * kMaxBands;
    dspi_eq_param p = recipes[i];
    dspi_biquad_f32 &dst = aos[band_index(i, rr)];
    dspi_biquad_f32 bq = dst;
    if (recipe_is_flat(p) || fs == 0.0f) {                                   // :62-73
        bq.bypass = 1;
        bq.use_svf = 0;
        bq.b0 = 1.0f;
        bq.b1 = bq.b2 = bq.a1 = bq.a2 = 0.0f;
        bq.sva1 = bq.sva2 = bq.sva3 = 0.0f;
        bq.svm0 = bq.svm1 = bq.svm2 = 0.0f;
    } else {
        bq.bypass = 0;
        recipe_clamp(p, fs);
        const float A = pow10_f(fdiv(p.gain_db, 40.0f));                      // :83
        const uint8_t svf_now = (p.freq < fdiv(fs, 7.5f)) ? 1 : 0;               // :87-92
        if (svf_now != bq.use_svf) {
            bq.s1 = bq.s2 = 0.0f;
            bq.svic1eq = bq.svic2eq = 0.0f;
        }
        bq.use_svf = svf_now;
        if (svf_now) {                                                         // :94-138
            float g = tan_f(fdiv(kPi * p.freq, fs));
            float k = fdiv(1.0f, p.Q);
            if (p.type == DSPI_FILTER_PEAKING) k = fdiv(1.0f, p.Q * A);
            else if (p.type == DSPI_FILTER_LOWSHELF) g = fdiv(g, fsqrt(A));
            else if (p.type == DSPI_FILTER_HIGHSHELF) g = g * fsqrt(A);
            const float c1 = fdiv(1.0f, 1.0f + g * (g + k));
            const float c2 = g * c1;
            const float c3 = g * c2;
            float m0 = 0.0f, m1 = 0.0f, m2 = 0.0f;
            switch (p.type) {
            case DSPI_FILTER_LOWPASS: m2 = 1.0f; break;
            case DSPI_FILTER_HIGHPASS: m0 = 1.0f; m1 = -k; m2 = -1.0f; break;
            case DSPI_FILTER_PEAKING: m0 = 1.0f; m1 = k * (A * A - 1.0f); break;
            case DSPI_FILTER_LOWSHELF: m0 = 1.0f; m1 = k * (A - 1.0f); m2 = A * A - 1.0f; break;
            case DSPI_FILTER_HIGHSHELF: m0 = A * A; m1 = k * (1.0f - A) * A; m2 = 1.0f - A * A; break;
            default: break;
            }
            bq.sva1 = c1; bq.sva2 = c2; bq.sva3 = c3;
            bq.svm0 = m0; bq.svm1 = m1; bq.svm2 = m2;
            bq.svf_type = p.type;
            bq.b0 = 1.0f;
            bq.b1 = bq.b2 = bq.a1 = bq.a2 = 0.0f;
        } else {
            bq.sva1 = bq.sva2 = bq.sva3 = 0.0f;                               // :141-142
            bq.svm0 = bq.svm1 = bq.svm2 = 0.0f;
            float nn[3], dd[3];
            cookbook(p, A, fs, nn, dd);
            const float inv_a0 = fdiv(1.0f, dd[0]);                            // :160-165
            bq.b0 = nn[0] * inv_a0;
            bq.b1 = nn[1] * inv_a0;
            bq.b2 = nn[2] * inv_a0;
            bq.a1 = dd[1] * inv_a0;
            bq.a2 = dd[2] * inv_a0;
        }
    }
    recipes[i] = p;
    dst = bq;
}

// (int32_t) cast with the firmware's saturating semantics (:168-173 run on the RP2040's soft float)
__device__ __forceinline__ int32_t to_q28(float v)
{
    const float x = v * 268435456.0f;
    if (x != x) return 0;
    return __float2int_rz(x);                                                 // saturates
}

__global__ void __launch_bounds__(256)
coeff_q28_kernel(dspi_eq_param *__restrict__ recipes, dspi_biquad_q28 *__restrict__ aos, uint32_t ch0, uint32_t n, float fs, RoleRange rr)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!band_selected(i, n, rr)) return;
    if (rr.fs) fs = rr.fs[i / kMaxBands];
    recipes += (size_t)blockIdx.y * n * kMaxBands;
    aos += ((size_t)ch0 + (size_t)blockIdx.y * rr.stride) * kMaxBands;
    dspi_eq_param p = recipes[i];
    dspi_biquad_q28 &dst = aos[band_index(i, rr)];
    dspi_biquad_q28 bq = dst;
    if (recipe_is_flat(p) || fs == 0.0f) {
        bq.bypass = 1;
        bq.b0 = 1 << 28;
        bq.b1 = bq.b2 = bq.a1 = bq.a2 = 0;
    } else {
        bq.bypass = 0;
        recipe_clamp(p, fs);
        const float A = pow10_f(fdiv(p.gain_db, 40.0f));
        float nn[3], dd[3];
        cookbook(p, A, fs, nn, dd);
        bq.b0 = to_q28(fdiv(nn[0], dd[0]));                                        // :168-173 truncating store
        bq.b1 = to_q28(fdiv(nn[1], dd[0]));
        bq.b2 = to_q28(fdiv(nn[2], dd[0]));
        bq.a1 = to_q28(fdiv(dd[1], dd[0]));
        bq.a2 = to_q28(fdiv(dd[2], dd[0]));
    }
    recipes[i] = p;
    dst = bq;
}

}  // namespace

cudaError_t launch_coeffs(bool q28, dspi_eq_param *d_recipes, void *d_aos, uint32_t ch0, uint32_t n, float fs, cudaStream_t stream,
                          const RoleRange &rr)
{
    if (n == 0) return cudaSuccess;
    const dim3 grid((n * kMaxBands + 255) / 256, rr.roles);
    if (q28) coeff_q28_kernel<<<grid, 256, 0, stream>>>(d_recipes, (dspi_biquad_q28 *)d_aos, ch0, n, fs, rr);
    else coeff_f32_kernel<<<grid, 256, 0, stream>>>(d_recipes, (dspi_biquad_f32 *)d_aos, ch0, n, fs, rr);
    return cudaGetLastError();
}

}  // namespace dspi
