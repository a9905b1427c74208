/* kjb_numeric.h — the NUMERIC CONTRACT of the kajiya-b200 C-ABI.
 *
 * kajiya's shaders lean on driver-provided transcendental functions
 * (sin/cos/exp2/log2/pow/atan, f32<->f16) whose results differ from GPU to GPU.
 * Reservoir selection (`prob >= dart`, /root/reference assets/shaders/inc/reservoir.hlsl:47-59)
 * and every packed texel depend on them, so "bit-exact reservoir payloads" is only
 * meaningful once those functions are pinned.  This header pins them: every function below
 * is built exclusively from IEEE-754 binary32 +,-,*,/,sqrt, integer ops and comparisons,
 * evaluated in the written order (compile WITHOUT fp contraction: nvcc -fmad=false,
 * gcc -ffp-contract=off), so the CUDA kernels, the CPU oracle and any host that wants to
 * prepare bit-compatible inputs all get identical results.
 *
 * It is part of the public ABI (like a libm), not of the oracle and not of the kernels.
 * tests/test_numeric.py checks each function against libm to a stated ulp bound.
 */
#ifndef KJB_NUMERIC_H
#define KJB_NUMERIC_H

#include <stdint.h>
#include <string.h>
#include <math.h>
#if defined(__CUDACC__)
#include <cuda_fp16.h>
#endif

#if defined(__CUDACC__)
#define KJB_HD __host__ __device__ __forceinline__
#else
#define KJB_HD static inline
#endif

#define KJB_PI 3.14159265358979323846f
#define KJB_TAU 6.28318530717958647692f
#define KJB_FLT_MAX 3.402823466e+38f

KJB_HD uint32_t kjb_f2u(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
KJB_HD float kjb_u2f(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

/* ---- f32 <-> f16, round-to-nearest-even, IEEE (what DXC's f32tof16/f16tof32 and
 * R16G16B16A16_SFLOAT image stores do; pack_unpack.hlsl:90-100). Every NaN -> 0x7e00. ---- */
KJB_HD uint32_t kjb_f32_to_f16(float f) {
#if defined(__CUDA_ARCH__)
    /* cvt.rn.f16.f32 is the same IEEE RN-even conversion; only NaNs are canonicalised here, sign included: the GPU's 0/0 is
     * +NaN and x86's is -NaN, so a NaN a shader produces must not keep its sign to be stored the same on both */
    if (f != f) return 0x7e00u;
    return (uint32_t)__half_as_ushort(__float2half_rn(f));
#endif
    const uint32_t x = kjb_f2u(f);
    const uint32_t sign = (x >> 16) & 0x8000u;
    const uint32_t ax = x & 0x7fffffffu;
    if (ax >= 0x7f800000u) {                       /* inf / nan */
        return ax > 0x7f800000u ? 0x7e00u : (sign | 0x7c00u);
    }
    if (ax >= 0x477ff000u) {                       /* rounds to >= 65520 -> inf */
        return sign | 0x7c00u;
    }
    if (ax < 0x33000001u) {                        /* < 2^-25 (or == 2^-25, ties to even 0) */
        return sign;
    }
    uint32_t exp = ax >> 23;
    uint32_t man = ax & 0x7fffffu;
    if (exp < 113u) {                              /* subnormal half */
        man |= 0x800000u;
        const uint32_t shift = 126u - exp;         /* 14..24 */
        const uint32_t half_man = man >> shift;
        const uint32_t rem = man & ((1u << shift) - 1u);
        const uint32_t halfway = 1u << (shift - 1u);
        uint32_t r = half_man;
        if (rem > halfway || (rem == halfway && (half_man & 1u))) r += 1u;
        return sign | r;
    }
    uint32_t h = ((exp - 112u) << 10) | (man >> 13);
    const uint32_t rem = man & 0x1fffu;
    if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) h += 1u;   /* may carry into exponent: correct */
    return sign | h;
}

KJB_HD float kjb_f16_to_f32(uint32_t h) {
#if defined(__CUDA_ARCH__)
    return __half2float(__ushort_as_half((unsigned short)h));
#endif
    const uint32_t sign = (h & 0x8000u) << 16;
    const uint32_t exp = (h >> 10) & 0x1fu;
    uint32_t man = h & 0x3ffu;
    if (exp == 0u) {
        if (man == 0u) return kjb_u2f(sign);
        /* subnormal: value = man * 2^-24 (exact in f32) */
        const float v = (float)man * 5.9604644775390625e-08f;
        return kjb_u2f(kjb_f2u(v) | sign);
    }
    if (exp == 31u) return kjb_u2f(sign | 0x7f800000u | (man << 13));
    return kjb_u2f(sign | ((exp + 112u) << 23) | (man << 13));
}

/* ---- fused multiply-add: the ONLY place contraction happens.  Both sides compile with contraction off, so a*b+c written with
 * operators is two roundings everywhere; code that wants the fused form says so explicitly and gets it on the device (FFMA) and on
 * the host (vfmadd / libm fmaf) alike.  Used by dot / matrix-vector / lerp and the polynomial kernels below. ---- */
KJB_HD float kjb_fma(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
    return __fmaf_rn(a, b, c);
#else
    return __builtin_fmaf(a, b, c);
#endif
}

/* ---- elementary helpers with HLSL semantics ---- */
/* HLSL/DXIL FMin/FMax = IEEE minNum/maxNum: a NaN operand loses (the shaders rely on it, e.g. `max(0.0, dot(n, NaN_dir))`
 * for neighbours at depth 0 in restir_resolve.hlsl:112-114).  Signed zeros are ordered -0 < +0 and two NaNs give the canonical
 * 0x7fffffff (IEEE 754-2019 minimumNumber / maximumNumber): exactly what the single FMNMX instruction behind fminf/fmaxf returns on
 * sm_90a (probed: tools/probe_minmax.cu), spelled out for the host. */
KJB_HD float kjb_min(float a, float b) {
#if defined(__CUDA_ARCH__)
    return fminf(a, b);
#else
    if (a != a) return b == b ? b : kjb_u2f(0x7fffffffu);
    if (b != b) return a;
    if (a < b) return a;
    if (b < a) return b;
    return kjb_u2f(kjb_f2u(a) | kjb_f2u(b));   /* equal: identical bits, or +-0 where the sign bit (the smaller one) wins */
#endif
}
KJB_HD float kjb_max(float a, float b) {
#if defined(__CUDA_ARCH__)
    return fmaxf(a, b);
#else
    if (a != a) return b == b ? b : kjb_u2f(0x7fffffffu);
    if (b != b) return a;
    if (a > b) return a;
    if (b > a) return b;
    return kjb_u2f(kjb_f2u(a) & kjb_f2u(b));   /* equal: identical bits, or +-0 where +0 (the larger one) wins */
#endif
}
KJB_HD float kjb_clamp(float x, float lo, float hi) { return kjb_min(kjb_max(x, lo), hi); }
KJB_HD float kjb_saturate(float x) {
#if defined(__CUDA_ARCH__)
    return __saturatef(x);   /* one instruction; documented as clamp to [+0.0, 1.0] with NaN -> +0: exactly the expression below (-0 -> +0 too) */
#else
    return kjb_clamp(x, 0.0f, 1.0f);
#endif
}
KJB_HD float kjb_abs(float x) { return kjb_u2f(kjb_f2u(x) & 0x7fffffffu); }
KJB_HD float kjb_rcp(float x) { return 1.0f / x; }
KJB_HD float kjb_sqrt(float x) { return sqrtf(x); }                /* IEEE correctly rounded on both sides */
KJB_HD float kjb_rsqrt(float x) { return 1.0f / sqrtf(x); }
KJB_HD float kjb_floor(float x) { return floorf(x); }
KJB_HD float kjb_ceil(float x) { return ceilf(x); }
KJB_HD float kjb_trunc(float x) { return truncf(x); }
KJB_HD float kjb_frac(float x) { return x - floorf(x); }
/* x / d for a non-negative-or-integer x and a positive divisor d whose reciprocal is at hand (both well inside the normal range): reciprocal multiply plus one exact-residual correction
 * (q = x*(1/d); q + (x - d*q)*(1/d), both steps fused).  With 1/d correctly rounded this is the correctly rounded quotient — the same
 * bits as the IEEE division the oracle writes — in 3 instructions instead of the ~9 of a full-range division; tests/test_numeric.py
 * checks every numerator of every call site (texel decode: d = 127, 255, 1023, 2047, 32767, 65535) exhaustively. */
KJB_HD float kjb_div_int_const(float x, float d, float rcp_d) { const float q = x * rcp_d; return kjb_fma(kjb_fma(-d, q, x), rcp_d, q); }
#if defined(KJB_NO_DIV_INT_CONST)   /* A/B switch for tools/variant_bench.py */
#define KJB_DIV_INT_CONST(x, d) ((x) / (d))
#else
#define KJB_DIV_INT_CONST(x, d) kjb_div_int_const((x), (d), 1.0f / (d))
#endif

KJB_HD float kjb_lerp(float a, float b, float t) { return kjb_fma(b - a, t, a); }   /* HLSL lerp = a + t*(b-a) */
KJB_HD float kjb_step(float edge, float x) { return x >= edge ? 1.0f : 0.0f; }
KJB_HD float kjb_sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
KJB_HD float kjb_smoothstep(float a, float b, float x) {
    const float t = kjb_saturate((x - a) / (b - a));
    return t * t * kjb_fma(-2.0f, t, 3.0f);
}

/* float -> int conversions with the saturating semantics GPUs implement (HLSL leaves out-of-range
 * conversions undefined; restir_temporal.hlsl:216-238 does hit them at screen borders). NaN -> 0. */
KJB_HD int32_t kjb_cvt_i32(float x) {
#if defined(__CUDA_ARCH__)
    return __float2int_rz(x);
#else
    if (x != x) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return (int32_t)(-2147483647 - 1);
    return (int32_t)x;
#endif
}
KJB_HD uint32_t kjb_cvt_u32(float x) {
#if defined(__CUDA_ARCH__)
    return __float2uint_rz(x);
#else
    if (!(x > 0.0f)) return 0u;
    if (x >= 4294967296.0f) return 0xffffffffu;
    return (uint32_t)x;
#endif
}

/* ---- sin / cos: Cephes sinf/cosf scheme (octant reduction by pi/4 in three exact pieces) ---- */
KJB_HD void kjb_sincos(float xx, float *s_out, float *c_out) {
    const float FOPI = 1.27323954473516f;
    const float DP1 = 0.78515625f;
    const float DP2 = 2.4187564849853515625e-4f;
    const float DP3 = 3.77489497744594108e-8f;
    float x = kjb_abs(xx);
    const int neg = xx < 0.0f;
    if (!(x < 1.0e7f)) { *s_out = 0.0f; *c_out = 1.0f; return; }   /* outside the contract; also NaN */
    uint32_t j = (uint32_t)(FOPI * x);
    float y = (float)j;
    if (j & 1u) { j += 1u; y += 1.0f; }
    j &= 7u;
    x = kjb_fma(-y, DP3, kjb_fma(-y, DP2, kjb_fma(-y, DP1, x)));
    const float z = x * x;
    const float ps = kjb_fma(kjb_fma(kjb_fma(-1.9515295891e-4f, z, 8.3321608736e-3f), z, -1.6666654611e-1f) * z, x, x);
    const float pc = kjb_fma(kjb_fma(kjb_fma(2.443315711809948e-5f, z, -1.388731625493765e-3f), z, 4.166664568298827e-2f) * z, z, kjb_fma(-0.5f, z, 1.0f));
    float s, c;
    int ssign = neg, csign = 0;
    if (j > 3u) { ssign = !ssign; csign = !csign; j -= 4u; }
    if (j > 1u) csign = !csign;
    if (j == 1u || j == 2u) { s = pc; c = ps; } else { s = ps; c = pc; }
    *s_out = ssign ? -s : s;
    *c_out = csign ? -c : c;
}
KJB_HD float kjb_sin(float x) { float s, c; kjb_sincos(x, &s, &c); return s; }
KJB_HD float kjb_cos(float x) { float s, c; kjb_sincos(x, &s, &c); return c; }

/* ---- exp2 / log2 / pow / exp / log ---- */
KJB_HD float kjb_exp2(float x) {
    if (x != x) return x;
    if (x >= 128.0f) return kjb_u2f(0x7f800000u);
    if (x < -126.0f) return 0.0f;                 /* results below FLT_MIN flush to zero (documented) */
    const float fl = floorf(x + 0.5f);
    const float f = x - fl;                       /* [-0.5, 0.5] */
    const int n = (int)fl;
    /* 2^f, minimax-ish Taylor in f*ln2, degree 7 */
    const float t = f * 0.693147180559945f;
    float p = 1.984126984e-4f;
    p = kjb_fma(p, t, 1.388888889e-3f);
    p = kjb_fma(p, t, 8.333333333e-3f);
    p = kjb_fma(p, t, 4.166666667e-2f);
    p = kjb_fma(p, t, 1.666666667e-1f);
    p = kjb_fma(p, t, 0.5f);
    p = kjb_fma(p, t, 1.0f);
    p = kjb_fma(p, t, 1.0f);
    if (n > 127) return p * 2.0f * kjb_u2f((uint32_t)(127 + 127) << 23);
    return p * kjb_u2f((uint32_t)(n + 127) << 23);
}

KJB_HD float kjb_log2(float x) {
    if (x != x) return x;
    if (x < 0.0f) return kjb_u2f(0x7fc00000u);
    if (x == 0.0f) return kjb_u2f(0xff800000u);
    uint32_t ux = kjb_f2u(x);
    if (ux >= 0x7f800000u) return x;
    int e = 0;
    if (ux < 0x00800000u) { x = x * 16777216.0f; ux = kjb_f2u(x); e = -24; }
    e += (int)(ux >> 23) - 127;
    float m = kjb_u2f((ux & 0x007fffffu) | 0x3f800000u);   /* [1,2) */
    if (m > 1.41421356237f) { m = m * 0.5f; e += 1; }      /* [0.707,1.414) */
    const float f = m - 1.0f;
    /* ln(1+f) = 2 atanh(s), s = f/(2+f); odd series to s^11 */
    const float s = f / (2.0f + f);
    const float z = s * s;
    float p = 0.1818181818f;
    p = kjb_fma(p, z, 0.2222222222f);
    p = kjb_fma(p, z, 0.2857142857f);
    p = kjb_fma(p, z, 0.4f);
    p = kjb_fma(p, z, 0.6666666667f);
    p = kjb_fma(p, z, 2.0f);
    const float ln1pf = p * s;
    return kjb_fma(ln1pf, 1.44269504088896f, (float)e);
}

KJB_HD float kjb_pow(float x, float y) { return kjb_exp2(y * kjb_log2(x)); }   /* HLSL pow semantics */
KJB_HD float kjb_exp(float x) { return kjb_exp2(x * 1.44269504088896f); }
KJB_HD float kjb_log(float x) { return kjb_log2(x) * 0.693147180559945f; }

/* ---- atan / atan2 / acos (Cephes atanf scheme) ---- */
KJB_HD float kjb_atan(float xx) {
    float x = kjb_abs(xx);
    float y;
    if (x > 2.414213562373095f) { y = 1.5707963267948966f; x = -(1.0f / x); }
    else if (x > 0.4142135623730950f) { y = 0.7853981633974483f; x = (x - 1.0f) / (x + 1.0f); }
    else y = 0.0f;
    const float z = x * x;
    y = y + kjb_fma(kjb_fma(kjb_fma(kjb_fma(8.05374449538e-2f, z, -1.38776856032e-1f), z, 1.99777106478e-1f), z, -3.33329491539e-1f) * z, x, x);
    return xx < 0.0f ? -y : y;
}
KJB_HD float kjb_atan2(float y, float x) {
    if (x > 0.0f) return kjb_atan(y / x);
    if (x < 0.0f) return y >= 0.0f ? kjb_atan(y / x) + KJB_PI : kjb_atan(y / x) - KJB_PI;
    if (y > 0.0f) return 1.5707963267948966f;
    if (y < 0.0f) return -1.5707963267948966f;
    return 0.0f;
}
KJB_HD float kjb_acos(float x) {
    x = kjb_clamp(x, -1.0f, 1.0f);
    return kjb_atan2(sqrtf((1.0f - x) * (1.0f + x)), x);
}

/* ---- KJB_FAST: the price tag of the contract.  libkjb_fast.so is the SAME source compiled with -DKJB_FAST -use_fast_math: the
 * transcendentals below become the GPU's special-function-unit instructions (MUFU.SIN / COS / EX2 / LG2 / RCP / RSQ), division and square
 * root their approximate forms, and a*b+c contracts to FFMA — i.e. what a shader compiler makes of the reference's HLSL.  Results are then
 * close to, not equal to, the oracle's (tests/test_gpu_fast.py states how close); the product default stays the exact build. ---- */
#if defined(KJB_FAST) && defined(__CUDA_ARCH__)
#define kjb_sincos kjb_sincos_fast
#define kjb_sin kjb_sin_fast
#define kjb_cos kjb_cos_fast
#define kjb_exp2 kjb_exp2_fast
#define kjb_log2 kjb_log2_fast
#define kjb_pow kjb_pow_fast
#define kjb_exp kjb_exp_fast
#define kjb_log kjb_log_fast
#define kjb_atan kjb_atan_fast
#define kjb_atan2 kjb_atan2_fast
#define kjb_acos kjb_acos_fast
KJB_HD void kjb_sincos_fast(float x, float *s, float *c) { __sincosf(x, s, c); }
KJB_HD float kjb_sin_fast(float x) { return __sinf(x); }
KJB_HD float kjb_cos_fast(float x) { return __cosf(x); }
KJB_HD float kjb_exp2_fast(float x) { return exp2f(x); }
KJB_HD float kjb_log2_fast(float x) { return __log2f(x); }
KJB_HD float kjb_pow_fast(float x, float y) { return exp2f(y * __log2f(x)); }
KJB_HD float kjb_exp_fast(float x) { return __expf(x); }
KJB_HD float kjb_log_fast(float x) { return __logf(x); }
KJB_HD float kjb_atan_fast(float x) { return atanf(x); }
KJB_HD float kjb_atan2_fast(float y, float x) { return atan2f(y, x); }
KJB_HD float kjb_acos_fast(float x) { return acosf(fminf(fmaxf(x, -1.0f), 1.0f)); }
#endif

#endif /* KJB_NUMERIC_H */
