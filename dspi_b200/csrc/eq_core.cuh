// eq_core.cuh — arithmetic core of the float EQ cascade, shared by the EQ kernel (eq_f32.cu) and
// the full-chain kernels (chain_f32.cu): value types (scalar / register-pair f32x2), the per-band
// register-tile loops (TDF2 biquad, Cytomic SVF with its four output mixes) and EqBank, which
// holds all bands of one channel (or channel pair) in registers and runs a register tile of
// N samples through them.  Reference: dsp_process_channel_block(), dsp_pipeline.c:281-365.
#pragma once
#include "eq_modes.cuh"

namespace dspi {
namespace core {

// ---------------------------------------------------------------------------------------
// value types: float (1 channel / lane) or P2 (2 channels / lane, a register pair)
//
// P2 is an opaque 64-bit register pair driven with inline PTX.  sm_90 has no packed f32x2
// arithmetic, so each P2 operation is two scalar .rn.ftz instructions on the halves of the
// pair (the same roundings a packed instruction would apply); the pair gives every lane two
// independent recurrences to interleave.
// ---------------------------------------------------------------------------------------
struct P2 { unsigned long long v; };

__device__ __forceinline__ float v_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float v_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float v_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ P2 v_mul(P2 a, P2 b)
{
    P2 r;
    asm("{\n\t.reg .f32 a0, a1, b0, b1;\n\t"
        "mov.b64 {a0, a1}, %1;\n\tmov.b64 {b0, b1}, %2;\n\t"
        "mul.rn.ftz.f32 a0, a0, b0;\n\tmul.rn.ftz.f32 a1, a1, b1;\n\t"
        "mov.b64 %0, {a0, a1};\n\t}" : "=l"(r.v) : "l"(a.v), "l"(b.v));
    return r;
}
__device__ __forceinline__ P2 v_add(P2 a, P2 b)
{
    P2 r;
    asm("{\n\t.reg .f32 a0, a1, b0, b1;\n\t"
        "mov.b64 {a0, a1}, %1;\n\tmov.b64 {b0, b1}, %2;\n\t"
        "add.rn.ftz.f32 a0, a0, b0;\n\tadd.rn.ftz.f32 a1, a1, b1;\n\t"
        "mov.b64 %0, {a0, a1};\n\t}" : "=l"(r.v) : "l"(a.v), "l"(b.v));
    return r;
}
__device__ __forceinline__ P2 v_fma(P2 a, P2 b, P2 c)
{
    P2 r;
    asm("{\n\t.reg .f32 a0, a1, b0, b1, c0, c1;\n\t"
        "mov.b64 {a0, a1}, %1;\n\tmov.b64 {b0, b1}, %2;\n\tmov.b64 {c0, c1}, %3;\n\t"
        "fma.rn.ftz.f32 a0, a0, b0, c0;\n\tfma.rn.ftz.f32 a1, a1, b1, c1;\n\t"
        "mov.b64 %0, {a0, a1};\n\t}" : "=l"(r.v) : "l"(a.v), "l"(b.v), "l"(c.v));
    return r;
}
__device__ __forceinline__ P2 p2_pack(float lo, float hi)
{
    P2 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r.v) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void p2_unpack(P2 a, float &lo, float &hi)
{
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(a.v));
}

template <typename V> __device__ __forceinline__ V v_bits(unsigned long long b);
template <> __device__ __forceinline__ float v_bits<float>(unsigned long long b) { return __uint_as_float((unsigned)b); }
template <> __device__ __forceinline__ P2 v_bits<P2>(unsigned long long b) { P2 r; r.v = b; return r; }
template <typename V> __device__ __forceinline__ V v_set(float x);
template <> __device__ __forceinline__ float v_set<float>(float x) { return x; }
template <> __device__ __forceinline__ P2 v_set<P2>(float x) { return p2_pack(x, x); }

// sign flip on the integer pipe (exact; a flushed-denormal operand is flushed by the consumer)
__device__ __forceinline__ float v_neg(float a) { return __int_as_float(__float_as_int(a) ^ 0x80000000); }
__device__ __forceinline__ P2 v_neg(P2 a) { P2 r; r.v = a.v ^ 0x8000000080000000ull; return r; }

// The strict flavour forms pair products as fma(a, b, nz) where nz = (-0.0, -0.0) arrives as a
// KERNEL PARAMETER: an exact product rounding (x + -0 == x for every x, including both zeros)
// that the assembler cannot prove foldable.  The scalar mul.rn / add.rn that the pair operations
// issue on sm_90 are not contracted either, so this is not needed for correctness there; it stays
// because it guarantees the strict roundings whatever the assembler does with explicit-rounding
// arithmetic, and FFMA issues at the same rate as FMUL on the FMA pipe.
template <bool FUSED> __device__ __forceinline__ float mulx(float a, float b, float) { return __fmul_rn(a, b); }
template <bool FUSED> __device__ __forceinline__ P2 mulx(P2 a, P2 b, P2 nz)
{
    if constexpr (FUSED) return v_mul(a, b);
    else return v_fma(a, b, nz);
}

// a*b + c: one rounding (FUSED) or two (strict)
template <bool FUSED, typename V>
__device__ __forceinline__ V madd(V a, V b, V c, V nz)
{
    if constexpr (FUSED) return v_fma(a, b, c);
    else return v_add(mulx<false>(a, b, nz), c);
}
template <bool FUSED>
__device__ __forceinline__ float madd(float a, float b, float c)
{
    if constexpr (FUSED) return __fmaf_rn(a, b, c);
    else return __fadd_rn(__fmul_rn(a, b), c);
}

// ---------------------------------------------------------------------------------------
// per-band inner loops over a register tile x[N]
// ---------------------------------------------------------------------------------------

// TDF2 biquad, dsp_pipeline.c:354-360.  c = {b0, b1, b2, -a1, -a2}
//   out = b0*in + s1;  s1 = b1*in - a1*out + s2;  s2 = b2*in - a2*out
template <bool FUSED, int N, typename V>
__device__ __forceinline__ void tdf2_tile(const V (&x)[N], V (&y)[N], const V (&c)[6], V &s1, V &s2, const V nz)
{
#pragma unroll
    for (int i = 0; i < N; i++) {
        const V in = x[i];
        const V out = madd<FUSED>(c[0], in, s1, nz);
        const V m = mulx<FUSED>(c[3], out, nz);          // -(a1*out), exact negation of the reference's product
        s1 = v_add(madd<FUSED>(c[1], in, m, nz), s2);
        const V n = mulx<FUSED>(c[4], out, nz);
        s2 = madd<FUSED>(c[2], in, n, nz);
        y[i] = out;
    }
}

// Cytomic SVF, dsp_pipeline.c:299-342.  c = {a1, a2, a3, m0, m1, m2}
//   v3 = in - ic2;  v1 = a1*ic1 + a2*v3;  v2 = ic2 + a2*ic1 + a3*v3;
//   ic1 = 2*v1 - ic1;  ic2 = 2*v2 - ic2;  out = mix(in, v1, v2)
// The update `ic = 2v - ic` flips the sign the state enters with, so two samples are
// processed per step: the first with (ic1, ic2), leaving (-ic1', -ic2'); the second consumes
// the negated state and leaves it positive again.  Every rewritten operation is the
// reference's operation with operands negated in pairs, which commutes with rounding.
enum { kMixLP = 2, kMixHP = 3, kMixPK = 4, kMixSH = 5 };

template <bool FUSED, int MIX, int N, typename V>
__device__ __forceinline__ void svf_tile(const V (&x)[N], V (&y)[N], const V (&c)[6], V &ic1, V &ic2, const V nz)
{
    static_assert(N % 2 == 0, "SVF tile processes sample pairs");
    const V kN1 = v_set<V>(-1.0f), kN2 = v_set<V>(-2.0f), kP2 = v_set<V>(2.0f);
    const V na1 = v_neg(c[0]), na3 = v_neg(c[2]), nm2 = v_neg(c[5]);
#pragma unroll
    for (int i = 0; i < N; i += 2) {
        {   // ---- state positive on entry, negated on exit
            const V in = x[i];
            const V v3 = v_fma(ic2, kN1, in);                       // in - ic2 (exact product)
            const V p = mulx<FUSED>(c[1], v3, nz);
            V t, v1, v2;
            if constexpr (FUSED) {
                t = v_fma(c[1], ic1, ic2);                          // a2*ic1 + ic2
                v1 = v_fma(c[0], ic1, p);                           // a1*ic1 + a2*v3
                v2 = v_fma(c[2], v3, t);
            } else {
                t = v_add(ic2, mulx<FUSED>(c[1], ic1, nz));
                v1 = v_add(mulx<FUSED>(c[0], ic1, nz), p);
                v2 = v_add(t, mulx<FUSED>(c[2], v3, nz));
            }
            ic1 = v_fma(v1, kN2, ic1);                              // -(2*v1 - ic1)
            ic2 = v_fma(v2, kN2, ic2);
            if constexpr (MIX == kMixLP) y[i] = v2;
            else if constexpr (MIX == kMixPK) y[i] = madd<FUSED>(c[4], v1, in, nz);
            else if constexpr (MIX == kMixHP) y[i] = v_fma(v2, kN1, madd<FUSED>(c[4], v1, in, nz));
            else {
                const V q = mulx<FUSED>(c[4], v1, nz);
                y[i] = madd<FUSED>(c[5], v2, madd<FUSED>(c[3], in, q, nz), nz);
            }
        }
        {   // ---- state negated on entry (n1 = -ic1, n2 = -ic2), positive on exit
            const V in = x[i + 1];
            const V v3 = v_add(in, ic2);                            // in - ic2
            const V p = mulx<FUSED>(c[1], v3, nz);
            V nt, v1, nv2;
            if constexpr (FUSED) {
                nt = v_fma(c[1], ic1, ic2);                         // -(a2*ic1 + ic2)
                v1 = v_fma(na1, ic1, p);                            // a1*ic1 + a2*v3
                nv2 = v_fma(na3, v3, nt);                           // -v2
            } else {
                nt = v_add(ic2, mulx<FUSED>(c[1], ic1, nz));
                v1 = v_add(mulx<FUSED>(na1, ic1, nz), p);
                nv2 = v_add(nt, mulx<FUSED>(na3, v3, nz));
            }
            ic1 = v_fma(v1, kP2, ic1);                              // 2*v1 - ic1
            ic2 = v_fma(nv2, kN2, ic2);                             // 2*v2 - ic2
            if constexpr (MIX == kMixLP) y[i + 1] = mulx<FUSED>(nv2, kN1, nz);
            else if constexpr (MIX == kMixPK) y[i + 1] = madd<FUSED>(c[4], v1, in, nz);
            else if constexpr (MIX == kMixHP) y[i + 1] = v_add(madd<FUSED>(c[4], v1, in, nz), nv2);
            else {
                const V q = mulx<FUSED>(c[4], v1, nz);
                y[i + 1] = madd<FUSED>(nm2, nv2, madd<FUSED>(c[3], in, q, nz), nz);
            }
        }
    }
}

// Scalar, runtime-length, per-lane-mode version: used for warps whose channels do not share
// a band's topology and for the tail of a launch (T not a multiple of the register tile).
// Same operation sequences as above in their natural (reference) form.
template <bool FUSED>
__device__ __noinline__ float2 slow_band(float *xs, int n, uint32_t mode, float c0, float c1, float c2, float c3, float c4, float c5,
                                         float st0, float st1, int stride = 1)
{
    if (mode == kModeTdf2) {
        for (int i = 0; i < n; i++) {
            const float in = xs[i * stride];
            const float out = madd<FUSED>(c0, in, st0);
            const float m = __fmul_rn(c3, out);
            st0 = __fadd_rn(madd<FUSED>(c1, in, m), st1);
            const float nn = __fmul_rn(c4, out);
            st1 = madd<FUSED>(c2, in, nn);
            xs[i * stride] = out;
        }
    } else if (mode >= kModeSvfLP) {
        for (int i = 0; i < n; i++) {
            const float in = xs[i * stride];
            const float v3 = __fadd_rn(in, -st1);
            const float p = __fmul_rn(c1, v3);
            float t, v1, v2;
            if (FUSED) {
                t = __fmaf_rn(c1, st0, st1);
                v1 = __fmaf_rn(c0, st0, p);
                v2 = __fmaf_rn(c2, v3, t);
            } else {
                t = __fadd_rn(st1, __fmul_rn(c1, st0));
                v1 = __fadd_rn(__fmul_rn(c0, st0), p);
                v2 = __fadd_rn(t, __fmul_rn(c2, v3));
            }
            st0 = __fmaf_rn(2.0f, v1, -st0);
            st1 = __fmaf_rn(2.0f, v2, -st1);
            float y;
            if (mode == kModeSvfLP) y = v2;
            else if (mode == kModeSvfPK) y = madd<FUSED>(c4, v1, in);
            else if (mode == kModeSvfHP) y = __fadd_rn(madd<FUSED>(c4, v1, in), -v2);
            else y = madd<FUSED>(c5, v2, madd<FUSED>(c3, in, __fmul_rn(c4, v1)));
            xs[i * stride] = y;
        }
    }
    return make_float2(st0, st1);
}

// ---------------------------------------------------------------------------------------
// lane <-> register-tile plumbing
// ---------------------------------------------------------------------------------------
// L2-coherent accesses (bypass the per-SM L1) for words another SM may have written in this launch
__device__ __forceinline__ float ld_cg(const float *p) { return __ldcg(p); }
__device__ __forceinline__ P2 ld_cg(const P2 *p) { P2 r; r.v = __ldcg(&p->v); return r; }
__device__ __forceinline__ void st_cg(float *p, float v) { __stcg(p, v); }
__device__ __forceinline__ void st_cg(P2 *p, P2 v) { __stcg(&p->v, v.v); }

template <typename V> struct Lanes;
template <> struct Lanes<float> {
    static constexpr int CPL = 1;
    __device__ static __forceinline__ float get(float v, int) { return v; }
};
// build a value from per-half scalars (h = 0: channel `lane`, h = 1: channel `lane + 32`)
__device__ __forceinline__ void v_make(float &v, const float (&part)[1]) { v = part[0]; }
__device__ __forceinline__ void v_make(P2 &v, const float (&part)[2]) { v = p2_pack(part[0], part[1]); }
template <> struct Lanes<P2> {
    static constexpr int CPL = 2;
    __device__ static __forceinline__ float get(P2 v, int h) { float lo, hi; p2_unpack(v, lo, hi); return h ? hi : lo; }
};


// ---------------------------------------------------------------------------------------
// EqBank: every band of one channel (V = float) or channel pair (V = P2) in registers
// ---------------------------------------------------------------------------------------
// Packed store addressing: slot k of band b of this lane is base[(b * 8 + k) * 32] (V units):
//   k = 0..5 coefficients (TDF2: b0 b1 b2 -a1 -a2 0; SVF: a1 a2 a3 m0 m1 m2), k = 6,7 state.
template <typename V, bool FUSED, int NB>
struct EqBank {
    static constexpr int CPL = Lanes<V>::CPL;
    V c[NB][6], st[NB][2];
    uint64_t mode_h[CPL];       // this lane's 4-bit-per-band topology words
    uint64_t mode_w;            // lane 0's word: the warp-uniform candidate
    uint32_t uni;               // bit b: band b has one topology across the warp
    uint32_t nb_active;
    bool all_tdf2;

    // `shared_state`: the state words may have been written by another SM during this launch
    // (dynamic time slices): read them past the non-coherent L1
    __device__ __forceinline__ void load(const V *base, const uint64_t *const (&mode_ptr)[CPL], uint32_t nb, bool shared_state = false)
    {
        nb_active = nb;
#pragma unroll
        for (int b = 0; b < NB; b++) {
#pragma unroll
            for (int k = 0; k < 6; k++) c[b][k] = base[(b * 8 + k) * 32];
            if (shared_state) {
                st[b][0] = ld_cg(base + (b * 8 + 6) * 32);
                st[b][1] = ld_cg(base + (b * 8 + 7) * 32);
            } else {
                st[b][0] = base[(b * 8 + 6) * 32];
                st[b][1] = base[(b * 8 + 7) * 32];
            }
        }
#pragma unroll
        for (int h = 0; h < CPL; h++) {
            mode_h[h] = *mode_ptr[h];
            if (nb < 16) mode_h[h] &= (1ull << (4 * nb)) - 1;                 // bands >= nb are not processed
        }
        mode_w = __shfl_sync(0xffffffffu, mode_h[0], 0);
        uni = 0;
#pragma unroll
        for (int b = 0; b < NB; b++) {
            bool same = true;
#pragma unroll
            for (int h = 0; h < CPL; h++) same = same && (((mode_h[h] ^ mode_w) >> (4 * b)) & 15) == 0;
            if (__all_sync(0xffffffffu, same)) uni |= 1u << b;
        }
        uint64_t want = 0;
#pragma unroll
        for (int b = 0; b < NB; b++) want |= (uint64_t)kModeTdf2 << (4 * b);
        bool mine = nb == NB;
#pragma unroll
        for (int h = 0; h < CPL; h++) mine = mine && ((mode_h[h] & ((1ull << (4 * NB)) - 1)) == want);
        all_tdf2 = __all_sync(0xffffffffu, mine);
    }

    // This lane's channels lane + 32 h with h in [h_lo, h_hi) belong to the launch.  The others are rows outside a range
    // call (past its end, or below its start in a group it shares with another range): their state words are left as they are.
    __device__ __forceinline__ void store(V *base, int h_lo, int h_hi, bool shared_state = false) const
    {
        if (h_lo == 0 && h_hi >= CPL) {
#pragma unroll
            for (int b = 0; b < NB; b++) {
                if (shared_state) {
                    st_cg(base + (b * 8 + 6) * 32, st[b][0]);
                    st_cg(base + (b * 8 + 7) * 32, st[b][1]);
                } else {
                    base[(b * 8 + 6) * 32] = st[b][0];
                    base[(b * 8 + 7) * 32] = st[b][1];
                }
            }
        } else if constexpr (CPL == 2) {
#pragma unroll
            for (int h = 0; h < 2; h++) {                       // one float of each pair: channel lane (h = 0) or lane + 32
                if (h < h_lo || h >= h_hi) continue;
#pragma unroll
                for (int b = 0; b < NB; b++) {
                    float *s0 = reinterpret_cast<float *>(base + (b * 8 + 6) * 32) + h;
                    float *s1 = reinterpret_cast<float *>(base + (b * 8 + 7) * 32) + h;
                    if (shared_state) {
                        st_cg(s0, Lanes<V>::get(st[b][0], h));
                        st_cg(s1, Lanes<V>::get(st[b][1], h));
                    } else {
                        *s0 = Lanes<V>::get(st[b][0], h);
                        *s1 = Lanes<V>::get(st[b][1], h);
                    }
                }
            }
        }
    }

    // run x[0..nvalid) through all active bands, in place (x[nvalid..] is left unspecified)
    template <int N>
    __device__ __forceinline__ void run(V (&x)[N], int nvalid, const V nz)
    {
        if (all_tdf2 && nvalid == N) {
            // every band of every channel of this warp is a TDF2 biquad: one straight-line block,
            // no dispatch, the scheduler overlaps the bands (wavefront over band x sample)
            V y[N];
#pragma unroll
            for (int b = 0; b < NB; b += 2) {
                tdf2_tile<FUSED>(x, y, c[b], st[b][0], st[b][1], nz);
                tdf2_tile<FUSED>(y, x, c[b + 1], st[b + 1][0], st[b + 1][1], nz);
            }
            return;
        }
        V y[N];
#pragma unroll
        for (int b = 0; b < NB; b++) {
            // ping-pong between x and y so no case has to move its results back
            V(&in)[N] = (b & 1) ? y : x;
            V(&out)[N] = (b & 1) ? x : y;
            const uint32_t m = (b < (int)nb_active) ? ((uint32_t)(mode_w >> (4 * b)) & 15u) : kModeBypass;
            const bool fast = (((uni >> b) & 1u) || b >= (int)nb_active) && nvalid == N;
            if (fast) {
                if (m == kModeTdf2) tdf2_tile<FUSED>(in, out, c[b], st[b][0], st[b][1], nz);
                else if (m == kModeSvfPK) svf_tile<FUSED, kMixPK>(in, out, c[b], st[b][0], st[b][1], nz);
                else if (m == kModeSvfSH) svf_tile<FUSED, kMixSH>(in, out, c[b], st[b][0], st[b][1], nz);
                else if (m == kModeSvfLP) svf_tile<FUSED, kMixLP>(in, out, c[b], st[b][0], st[b][1], nz);
                else if (m == kModeSvfHP) svf_tile<FUSED, kMixHP>(in, out, c[b], st[b][0], st[b][1], nz);
                else {                                      // bypassed band: dsp_pipeline.c:288
#pragma unroll
                    for (int i = 0; i < N; i++) out[i] = in[i];
                }
            } else {
                float xs[CPL][N], ns0[CPL], ns1[CPL];
#pragma unroll
                for (int h = 0; h < CPL; h++) {
#pragma unroll
                    for (int i = 0; i < N; i++) xs[h][i] = Lanes<V>::get(in[i], h);
                    const uint32_t mh = (uint32_t)(mode_h[h] >> (4 * b)) & 15u;
                    const float2 ns = slow_band<FUSED>(xs[h], nvalid, mh, Lanes<V>::get(c[b][0], h), Lanes<V>::get(c[b][1], h),
                                                       Lanes<V>::get(c[b][2], h), Lanes<V>::get(c[b][3], h), Lanes<V>::get(c[b][4], h),
                                                       Lanes<V>::get(c[b][5], h), Lanes<V>::get(st[b][0], h), Lanes<V>::get(st[b][1], h));
                    ns0[h] = ns.x;
                    ns1[h] = ns.y;
                }
                v_make(st[b][0], ns0);
                v_make(st[b][1], ns1);
#pragma unroll
                for (int i = 0; i < N; i++) {
                    float part[CPL];
#pragma unroll
                    for (int h = 0; h < CPL; h++) part[h] = xs[h][i];
                    v_make(out[i], part);
                }
            }
        }
        static_assert(NB % 2 == 0, "results must land back in x");
    }

    // ---- compile-time signature: every band's topology is a template constant ------------------
    // (runtime-compiled kernels for engines whose channels all share one topology vector: the whole
    // cascade becomes one straight-line block like the all-biquad case, for any mix of SVF / TDF2)
    template <unsigned long long W, int B, bool IN_X, int N>
    __device__ __forceinline__ void sig_from(V (&x)[N], V (&y)[N], const V nz)
    {
        if constexpr (B < NB) {
            constexpr uint32_t m = (uint32_t)((W >> (4 * B)) & 15ull);
            V(&in)[N] = IN_X ? x : y;
            V(&out)[N] = IN_X ? y : x;
            if constexpr (m == kModeBypass) {
                sig_from<W, B + 1, IN_X>(x, y, nz);
            } else {
                if constexpr (m == kModeTdf2) tdf2_tile<FUSED>(in, out, c[B], st[B][0], st[B][1], nz);
                else svf_tile<FUSED, (int)m>(in, out, c[B], st[B][0], st[B][1], nz);
                sig_from<W, B + 1, !IN_X>(x, y, nz);
            }
        } else if constexpr (!IN_X) {
#pragma unroll
            for (int i = 0; i < N; i++) x[i] = y[i];
        }
    }
    // does every channel of this warp carry exactly the topology vector W (bands >= nb masked off)?
    template <unsigned long long W>
    __device__ __forceinline__ bool sig_match() const
    {
        bool mine = true;
#pragma unroll
        for (int h = 0; h < CPL; h++) mine = mine && mode_h[h] == W;
        return __all_sync(0xffffffffu, mine);
    }
    template <unsigned long long W, int N>
    __device__ __forceinline__ void run_sig(V (&x)[N], const V nz)
    {
        V y[N];
        sig_from<W, 0, true>(x, y, nz);
    }

    // one band over n samples (n % 4 == 0) stored as a lane-private column: sample i at col[i * 32]
    template <int MODE>
    __device__ __forceinline__ void band_loop(V *col, int n, const V (&cc)[6], V &s0, V &s1, const V nz)
    {
#pragma unroll 2
        for (int i = 0; i < n; i += 4) {
            V x[4], y[4];
#pragma unroll
            for (int j = 0; j < 4; j++) x[j] = col[(i + j) * 32];
            if constexpr (MODE == (int)kModeTdf2) tdf2_tile<FUSED>(x, y, cc, s0, s1, nz);
            else svf_tile<FUSED, MODE>(x, y, cc, s0, s1, nz);
#pragma unroll
            for (int j = 0; j < 4; j++) col[(i + j) * 32] = y[j];
        }
    }

    // two consecutive bands of the SAME topology in one pass: band b+1 of sample j only needs band b of
    // sample j, so inside the unrolled block the scheduler overlaps the two recurrences (a wavefront of
    // depth 2) and the tile travels through shared memory once instead of twice
    template <int MODE>
    __device__ __forceinline__ void band_loop2(V *col, int n, const V (&ca)[6], V &a0, V &a1, const V (&cb)[6], V &b0, V &b1, const V nz)
    {
#pragma unroll 2
        for (int i = 0; i < n; i += 4) {
            V x[4], y[4], z[4];
#pragma unroll
            for (int j = 0; j < 4; j++) x[j] = col[(i + j) * 32];
            if constexpr (MODE == (int)kModeTdf2) {
                tdf2_tile<FUSED>(x, y, ca, a0, a1, nz);
                tdf2_tile<FUSED>(y, z, cb, b0, b1, nz);
            } else {
                svf_tile<FUSED, MODE>(x, y, ca, a0, a1, nz);
                svf_tile<FUSED, MODE>(y, z, cb, b0, b1, nz);
            }
#pragma unroll
            for (int j = 0; j < 4; j++) col[(i + j) * 32] = z[j];
        }
    }

    // Band-outer pass over a shared-memory tile in column layout (the reference's own loop order,
    // dsp_pipeline.c:286-364): topology dispatch happens once per band per tile, each band is a
    // small rolled loop (stays in the instruction cache), samples travel LDS.64 -> registers ->
    // STS.64 between bands.  `col` already includes this lane's offset.
    __device__ __forceinline__ void run_columns(V *col, int n, const V nz)
    {
        bool fused_prev = false;                                // band b was already processed together with b-1
#pragma unroll
        for (int b = 0; b < NB; b++) {
            if (b >= (int)nb_active) break;
            if (fused_prev) { fused_prev = false; continue; }
            const uint32_t m = (uint32_t)(mode_w >> (4 * b)) & 15u;
            const bool fast = ((uni >> b) & 1u) && (n & 3) == 0;
            if (fast) {
                bool pair = false;
                if constexpr (true) {
                    if (b + 1 < NB) {
                        const uint32_t m1 = (uint32_t)(mode_w >> (4 * (b + 1))) & 15u;
                        pair = (b + 1 < (int)nb_active) && ((uni >> (b + 1)) & 1u) && m1 == m && m != kModeBypass;
                    }
                }
                if (pair) {
                    const int b1 = (b + 1 < NB) ? b + 1 : b;         // constant after unrolling
                    if (m == kModeTdf2) band_loop2<(int)kModeTdf2>(col, n, c[b], st[b][0], st[b][1], c[b1], st[b1][0], st[b1][1], nz);
                    else if (m == kModeSvfPK) band_loop2<kMixPK>(col, n, c[b], st[b][0], st[b][1], c[b1], st[b1][0], st[b1][1], nz);
                    else if (m == kModeSvfSH) band_loop2<kMixSH>(col, n, c[b], st[b][0], st[b][1], c[b1], st[b1][0], st[b1][1], nz);
                    else if (m == kModeSvfLP) band_loop2<kMixLP>(col, n, c[b], st[b][0], st[b][1], c[b1], st[b1][0], st[b1][1], nz);
                    else band_loop2<kMixHP>(col, n, c[b], st[b][0], st[b][1], c[b1], st[b1][0], st[b1][1], nz);
                    fused_prev = true;
                } else {
                    if (m == kModeTdf2) band_loop<(int)kModeTdf2>(col, n, c[b], st[b][0], st[b][1], nz);
                    else if (m == kModeSvfPK) band_loop<kMixPK>(col, n, c[b], st[b][0], st[b][1], nz);
                    else if (m == kModeSvfSH) band_loop<kMixSH>(col, n, c[b], st[b][0], st[b][1], nz);
                    else if (m == kModeSvfLP) band_loop<kMixLP>(col, n, c[b], st[b][0], st[b][1], nz);
                    else if (m == kModeSvfHP) band_loop<kMixHP>(col, n, c[b], st[b][0], st[b][1], nz);
                }
            } else {
                float ns0[CPL], ns1[CPL];
#pragma unroll
                for (int h = 0; h < CPL; h++) {
                    const uint32_t mh = (uint32_t)(mode_h[h] >> (4 * b)) & 15u;
                    const float2 ns = slow_band<FUSED>(reinterpret_cast<float *>(col) + h, n, mh, Lanes<V>::get(c[b][0], h), Lanes<V>::get(c[b][1], h),
                                                       Lanes<V>::get(c[b][2], h), Lanes<V>::get(c[b][3], h), Lanes<V>::get(c[b][4], h),
                                                       Lanes<V>::get(c[b][5], h), Lanes<V>::get(st[b][0], h), Lanes<V>::get(st[b][1], h), 32 * CPL);
                    ns0[h] = ns.x;
                    ns1[h] = ns.y;
                }
                v_make(st[b][0], ns0);
                v_make(st[b][1], ns1);
            }
        }
    }
};

}  // namespace core
}  // namespace dspi
