// Device-side numeric core of the H100 kernels: HLSL-style vector math, RNG, packing, reservoirs,
// view/ray context, BRDFs, sun/atmosphere, typed image access.
//
// Re-derived from kajiya's shader includes (paths relative to /root/reference/assets/shaders/inc/):
//   hash.hlsl:7-55, math.hlsl:21-91, uv.hlsl, pack_unpack.hlsl:1-164, reservoir.hlsl:6-98, gbuffer.hlsl:51-88,
//   frame_constants.hlsl:92-250, brdf.hlsl, brdf_lut.hlsl:10-77, layered_brdf.hlsl:11-169, sun.hlsl:21-42,
//   atmosphere.hlsl:7-24, atmosphere_felix.hlsl:50-243, blue_noise.hlsl:8-15, quasi_random.hlsl, lights/triangle.hlsl:36-80,
//   ray_cone.hlsl, color/srgb.hlsl:4-6, color/ycbcr.hlsl, working_color_space.hlsl:9-18, bilinear.hlsl.
// Arithmetic is written in the operation order of the numeric contract (include/kjb_numeric.h): no FMA contraction
// (nvcc -fmad=false), transcendentals from the contract, IEEE sqrt/div.  Everything here is __host__ __device__ only so
// that tests can run the very same kernel bodies through the CPU launch emulator (tests/emu) — the product never does.
#pragma once
#include "../../include/kjb_numeric.h"
#include "../../include/kjb.h"

#if defined(__CUDACC__)
#define KJB_DEV __host__ __device__ __forceinline__
#else
#define KJB_DEV inline
#endif

namespace kjb {

// ------------------------------------------------------------------------------------------------ vectors
KJB_DEV float2 f2(float x, float y) { float2 r; r.x = x; r.y = y; return r; }
KJB_DEV float2 f2(float a) { return f2(a, a); }
KJB_DEV float3 f3(float x, float y, float z) { float3 r; r.x = x; r.y = y; r.z = z; return r; }
KJB_DEV float3 f3(float a) { return f3(a, a, a); }
KJB_DEV float4 f4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
KJB_DEV float4 f4(float a) { return f4(a, a, a, a); }
KJB_DEV float4 f4(float3 v, float w) { return f4(v.x, v.y, v.z, w); }
KJB_DEV float3 xyz(float4 v) { return f3(v.x, v.y, v.z); }
KJB_DEV float2 xy(float4 v) { return f2(v.x, v.y); }
KJB_DEV float2 xy(float3 v) { return f2(v.x, v.y); }
KJB_DEV int2 i2(int x, int y) { int2 r; r.x = x; r.y = y; return r; }
KJB_DEV uint2 u2(uint32_t x, uint32_t y) { uint2 r; r.x = x; r.y = y; return r; }
KJB_DEV uint4 u4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }

#define KJB_OP2(op) \
    KJB_DEV float2 operator op(float2 a, float2 b) { return f2(a.x op b.x, a.y op b.y); } \
    KJB_DEV float2 operator op(float2 a, float b) { return f2(a.x op b, a.y op b); } \
    KJB_DEV float2 operator op(float a, float2 b) { return f2(a op b.x, a op b.y); }
#define KJB_OP3(op) \
    KJB_DEV float3 operator op(float3 a, float3 b) { return f3(a.x op b.x, a.y op b.y, a.z op b.z); } \
    KJB_DEV float3 operator op(float3 a, float b) { return f3(a.x op b, a.y op b, a.z op b); } \
    KJB_DEV float3 operator op(float a, float3 b) { return f3(a op b.x, a op b.y, a op b.z); }
#define KJB_OP4(op) \
    KJB_DEV float4 operator op(float4 a, float4 b) { return f4(a.x op b.x, a.y op b.y, a.z op b.z, a.w op b.w); } \
    KJB_DEV float4 operator op(float4 a, float b) { return f4(a.x op b, a.y op b, a.z op b, a.w op b); } \
    KJB_DEV float4 operator op(float a, float4 b) { return f4(a op b.x, a op b.y, a op b.z, a op b.w); }
KJB_OP2(+) KJB_OP2(-) KJB_OP2(*) KJB_OP2(/) KJB_OP3(+) KJB_OP3(-) KJB_OP3(*) KJB_OP3(/) KJB_OP4(+) KJB_OP4(-) KJB_OP4(*) KJB_OP4(/)
KJB_DEV float2 operator-(float2 a) { return f2(-a.x, -a.y); }
KJB_DEV float3 operator-(float3 a) { return f3(-a.x, -a.y, -a.z); }
KJB_DEV float4 operator-(float4 a) { return f4(-a.x, -a.y, -a.z, -a.w); }
KJB_DEV void operator+=(float2& a, float2 b) { a = a + b; }
KJB_DEV void operator+=(float3& a, float3 b) { a = a + b; }
KJB_DEV void operator+=(float4& a, float4 b) { a = a + b; }
KJB_DEV void operator*=(float3& a, float3 b) { a = a * b; }
KJB_DEV void operator*=(float3& a, float b) { a = a * b; }
KJB_DEV void operator/=(float3& a, float b) { a = a / b; }
KJB_DEV int2 operator+(int2 a, int2 b) { return i2(a.x + b.x, a.y + b.y); }
KJB_DEV int2 operator*(int2 a, int b) { return i2(a.x * b, a.y * b); }

KJB_DEV float fmin_(float a, float b) { return kjb_min(a, b); }
KJB_DEV float fmax_(float a, float b) { return kjb_max(a, b); }
KJB_DEV float2 vmin(float2 a, float2 b) { return f2(kjb_min(a.x, b.x), kjb_min(a.y, b.y)); }
KJB_DEV float2 vmax(float2 a, float2 b) { return f2(kjb_max(a.x, b.x), kjb_max(a.y, b.y)); }
KJB_DEV float3 vmin(float3 a, float3 b) { return f3(kjb_min(a.x, b.x), kjb_min(a.y, b.y), kjb_min(a.z, b.z)); }
KJB_DEV float3 vmax(float3 a, float3 b) { return f3(kjb_max(a.x, b.x), kjb_max(a.y, b.y), kjb_max(a.z, b.z)); }
KJB_DEV float4 vmin(float4 a, float4 b) { return f4(kjb_min(a.x, b.x), kjb_min(a.y, b.y), kjb_min(a.z, b.z), kjb_min(a.w, b.w)); }
KJB_DEV float4 vmax(float4 a, float4 b) { return f4(kjb_max(a.x, b.x), kjb_max(a.y, b.y), kjb_max(a.z, b.z), kjb_max(a.w, b.w)); }
KJB_DEV float2 vabs(float2 a) { return f2(kjb_abs(a.x), kjb_abs(a.y)); }
KJB_DEV float3 vabs(float3 a) { return f3(kjb_abs(a.x), kjb_abs(a.y), kjb_abs(a.z)); }
KJB_DEV float4 vabs(float4 a) { return f4(kjb_abs(a.x), kjb_abs(a.y), kjb_abs(a.z), kjb_abs(a.w)); }
KJB_DEV float3 vsqrt(float3 a) { return f3(kjb_sqrt(a.x), kjb_sqrt(a.y), kjb_sqrt(a.z)); }
KJB_DEV float4 vsqrt(float4 a) { return f4(kjb_sqrt(a.x), kjb_sqrt(a.y), kjb_sqrt(a.z), kjb_sqrt(a.w)); }
KJB_DEV float3 vexp(float3 a) { return f3(kjb_exp(a.x), kjb_exp(a.y), kjb_exp(a.z)); }
KJB_DEV float2 vfloor(float2 a) { return f2(kjb_floor(a.x), kjb_floor(a.y)); }
KJB_DEV float2 vfrac(float2 a) { return f2(kjb_frac(a.x), kjb_frac(a.y)); }
KJB_DEV float2 vsaturate(float2 a) { return f2(kjb_saturate(a.x), kjb_saturate(a.y)); }
KJB_DEV float3 vclamp(float3 v, float3 lo, float3 hi) { return vmin(vmax(v, lo), hi); }
// lerp, dot and matrix-vector products are FMA chains (numeric contract: the fused form is written out, kjb_numeric.h)
KJB_DEV float3 vlerp(float3 a, float3 b, float t) { return f3(kjb_lerp(a.x, b.x, t), kjb_lerp(a.y, b.y, t), kjb_lerp(a.z, b.z, t)); }
KJB_DEV float3 vlerp(float3 a, float3 b, float3 t) { return f3(kjb_lerp(a.x, b.x, t.x), kjb_lerp(a.y, b.y, t.y), kjb_lerp(a.z, b.z, t.z)); }
KJB_DEV float4 vlerp(float4 a, float4 b, float t) { return f4(kjb_lerp(a.x, b.x, t), kjb_lerp(a.y, b.y, t), kjb_lerp(a.z, b.z, t), kjb_lerp(a.w, b.w, t)); }
// HLSL mad(): a * s + c with ONE rounding per component — the weighted-sum taps of the filters (explicit, like every fused op of the contract)
KJB_DEV float  mad(float a, float s, float c) { return kjb_fma(a, s, c); }
KJB_DEV float2 mad(float2 a, float s, float2 c) { return f2(kjb_fma(a.x, s, c.x), kjb_fma(a.y, s, c.y)); }
KJB_DEV float3 mad(float3 a, float s, float3 c) { return f3(kjb_fma(a.x, s, c.x), kjb_fma(a.y, s, c.y), kjb_fma(a.z, s, c.z)); }
KJB_DEV float4 mad(float4 a, float s, float4 c) { return f4(kjb_fma(a.x, s, c.x), kjb_fma(a.y, s, c.y), kjb_fma(a.z, s, c.z), kjb_fma(a.w, s, c.w)); }
KJB_DEV float2 vlerp(float2 a, float2 b, float t) { return f2(kjb_lerp(a.x, b.x, t), kjb_lerp(a.y, b.y, t)); }
KJB_DEV float dot(float2 a, float2 b) { return kjb_fma(a.y, b.y, a.x * b.x); }
KJB_DEV float dot(float3 a, float3 b) { return kjb_fma(a.z, b.z, kjb_fma(a.y, b.y, a.x * b.x)); }
KJB_DEV float dot(float4 a, float4 b) { return kjb_fma(a.w, b.w, kjb_fma(a.z, b.z, kjb_fma(a.y, b.y, a.x * b.x))); }
KJB_DEV float3 cross(float3 a, float3 b) { return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
KJB_DEV float length(float2 a) { return kjb_sqrt(dot(a, a)); }
KJB_DEV float length(float3 a) { return kjb_sqrt(dot(a, a)); }
KJB_DEV float3 normalize(float3 a) { return a * kjb_rsqrt(dot(a, a)); }
KJB_DEV float3 reflect(float3 i, float3 n) { return i - 2.0f * dot(n, i) * n; }
KJB_DEV float max3(float x, float y, float z) { return kjb_max(x, kjb_max(y, z)); }
KJB_DEV float square(float x) { return x * x; }

// ------------------------------------------------------------------------------------------------ matrices
KJB_DEV float4 mul(const kjb_mat4& M, float4 v) {   // column-major glam Mat4, HLSL mul(M, v)
    const float* m = M.m;
    return f4(kjb_fma(m[12], v.w, kjb_fma(m[8], v.z, kjb_fma(m[4], v.y, m[0] * v.x))), kjb_fma(m[13], v.w, kjb_fma(m[9], v.z, kjb_fma(m[5], v.y, m[1] * v.x))),
              kjb_fma(m[14], v.w, kjb_fma(m[10], v.z, kjb_fma(m[6], v.y, m[2] * v.x))), kjb_fma(m[15], v.w, kjb_fma(m[11], v.z, kjb_fma(m[7], v.y, m[3] * v.x))));
}
struct float3x3 { float3 r0, r1, r2; };
KJB_DEV float3 mul(const float3x3& M, float3 v) { return f3(dot(M.r0, v), dot(M.r1, v), dot(M.r2, v)); }
KJB_DEV float3 mul(float3 v, const float3x3& M) {
    return f3(kjb_fma(v.z, M.r2.x, kjb_fma(v.y, M.r1.x, v.x * M.r0.x)), kjb_fma(v.z, M.r2.y, kjb_fma(v.y, M.r1.y, v.x * M.r0.y)), kjb_fma(v.z, M.r2.z, kjb_fma(v.y, M.r1.z, v.x * M.r0.z)));
}
KJB_DEV float3 xform_point(const float* m, float3 p) {   // row-major 3x4
    return f3(m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3], m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7], m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11]);
}
KJB_DEV float3 xform_dir(const float* m, float3 p) {
    return f3(m[0] * p.x + m[1] * p.y + m[2] * p.z, m[4] * p.x + m[5] * p.y + m[6] * p.z, m[8] * p.x + m[9] * p.y + m[10] * p.z);
}

#define KJB_PI_F 3.14159265358979323846f
#define KJB_TAU_F 6.28318530717958647692f
#define KJB_FRAC_1_PI 0.318309886183790671537767526745028724f
#define KJB_PLASTIC 1.32471795724474602596f
#define KJB_GOLDEN_ANGLE 2.39996323f

// ------------------------------------------------------------------------------------------------ RNG (u32, bit exact)
KJB_DEV uint32_t hash1(uint32_t x) { x += (x << 10u); x ^= (x >> 6u); x += (x << 3u); x ^= (x >> 11u); x += (x << 15u); return x; }
KJB_DEV uint32_t hash1_mut(uint32_t& h) { const uint32_t res = h; h = hash1(h); return res; }
KJB_DEV uint32_t hash_combine2(uint32_t x, uint32_t y) {
    uint32_t seed = (x * 1664525u + y + 1013904223u) * 1664525u;
    seed ^= (seed >> 11u); seed ^= (seed << 7u) & 0x9d2c5680u; seed ^= (seed << 15u) & 0xefc60000u; seed ^= (seed >> 18u);
    return seed;
}
KJB_DEV uint32_t hash2(uint32_t x, uint32_t y) { return hash_combine2(x, hash1(y)); }
KJB_DEV uint32_t hash3(uint32_t x, uint32_t y, uint32_t z) { return hash_combine2(x, hash2(y, z)); }
KJB_DEV float u01(uint32_t h) { return kjb_u2f((h & 0x007FFFFFu) | 0x3F800000u) - 1.0f; }
KJB_DEV float rand01(uint32_t& rng) { return u01(hash1_mut(rng)); }
KJB_DEV float interleaved_gradient_noise(uint32_t x, uint32_t y) { return kjb_frac(52.9829189f * kjb_frac(0.06711056f * float(x) + 0.00583715f * float(y))); }
KJB_DEV float radical_inverse_vdc(uint32_t bits) {
    bits = (bits << 16u) | (bits >> 16u);
    bits = ((bits & 0x55555555u) << 1u) | ((bits & 0xAAAAAAAAu) >> 1u);
    bits = ((bits & 0x33333333u) << 2u) | ((bits & 0xCCCCCCCCu) >> 2u);
    bits = ((bits & 0x0F0F0F0Fu) << 4u) | ((bits & 0xF0F0F0F0u) >> 4u);
    bits = ((bits & 0x00FF00FFu) << 8u) | ((bits & 0xFF00FF00u) >> 8u);
    return float(bits) * 2.3283064365386963e-10f;
}
KJB_DEV float2 hammersley(uint32_t i, uint32_t n) { return f2(float(i + 1) / float(n), radical_inverse_vdc(i + 1)); }
KJB_DEV float2 r2_sequence(uint32_t i) {
    const float a1 = 1.0f / KJB_PLASTIC, a2 = 1.0f / (KJB_PLASTIC * KJB_PLASTIC);
    return vfrac(f2(a1, a2) * float(i) + 0.5f);
}

// ------------------------------------------------------------------------------------------------ sampling helpers
KJB_DEV float3x3 build_orthonormal_basis(float3 n) {
    float3 b1, b2;
    if (n.z < 0.0f) {
        const float a = 1.0f / (1.0f - n.z), b = n.x * n.y * a;
        b1 = f3(1.0f - n.x * n.x * a, -b, n.x); b2 = f3(b, n.y * n.y * a - 1.0f, -n.y);
    } else {
        const float a = 1.0f / (1.0f + n.z), b = -n.x * n.y * a;
        b1 = f3(1.0f - n.x * n.x * a, b, -n.x); b2 = f3(b, 1.0f - n.y * n.y * a, -n.y);
    }
    float3x3 m; m.r0 = f3(b1.x, b2.x, n.x); m.r1 = f3(b1.y, b2.y, n.y); m.r2 = f3(b1.z, b2.z, n.z);
    return m;
}
KJB_DEV float3 uniform_sample_cone(float2 urand, float cos_theta_max) {
    const float cos_theta = (1.0f - urand.x) + urand.x * cos_theta_max;
    const float sin_theta = kjb_sqrt(kjb_saturate(1.0f - cos_theta * cos_theta));
    const float phi = urand.y * KJB_TAU_F;
    float s, c; kjb_sincos(phi, &s, &c);
    return f3(sin_theta * c, sin_theta * s, cos_theta);
}
KJB_DEV float3 uniform_sample_hemisphere(float2 urand) {
    const float phi = urand.y * KJB_TAU_F;
    const float cos_theta = 1.0f - urand.x;
    const float sin_theta = kjb_sqrt(1.0f - cos_theta * cos_theta);
    float s, c; kjb_sincos(phi, &s, &c);
    return f3(c * sin_theta, s * sin_theta, cos_theta);
}
KJB_DEV float inverse_depth_relative_diff(float primary_depth, float secondary_depth) {
    return kjb_abs(kjb_max(1e-20f, primary_depth) / kjb_max(1e-20f, secondary_depth) - 1.0f);
}
KJB_DEV float2 get_uv(int x, int y, const float* tex_size) { return f2((float(x) + 0.5f) * tex_size[2], (float(y) + 0.5f) * tex_size[3]); }
KJB_DEV float2 cs_to_uv(float2 cs) { return cs * f2(0.5f, -0.5f) + f2(0.5f, 0.5f); }
KJB_DEV float2 uv_to_cs(float2 uv) { return (uv - f2(0.5f)) * f2(2.0f, -2.0f); }

// ------------------------------------------------------------------------------------------------ packing
KJB_DEV float unpack_unorm(uint32_t p, uint32_t bits) { const uint32_t mx = (1u << bits) - 1u; return KJB_DIV_INT_CONST(float(p & mx), float(mx)); }   // == float(p & mx) / float(mx)
KJB_DEV uint32_t pack_unorm(float v, uint32_t bits) { const uint32_t mx = (1u << bits) - 1u; return uint32_t(kjb_clamp(v, 0.0f, 1.0f) * float(mx) + 0.5f); }
KJB_DEV uint32_t pack_normal_11_10_11(float3 n) {
    return pack_unorm(n.x * 0.5f + 0.5f, 11) + (pack_unorm(n.y * 0.5f + 0.5f, 10) << 11) + (pack_unorm(n.z * 0.5f + 0.5f, 11) << 21);
}
KJB_DEV float3 unpack_normal_11_10_11_no_normalize(uint32_t p) { return f3(unpack_unorm(p, 11), unpack_unorm(p >> 11, 10), unpack_unorm(p >> 21, 11)) * 2.0f - 1.0f; }
KJB_DEV float3 unpack_normal_11_10_11(uint32_t p) { return normalize(unpack_normal_11_10_11_no_normalize(p)); }
KJB_DEV uint32_t pack_color_888(float3 c) { c = vsqrt(c); return pack_unorm(c.x, 8) + (pack_unorm(c.y, 8) << 8) + (pack_unorm(c.z, 8) << 16); }
KJB_DEV float3 unpack_color_888(uint32_t p) { const float3 c = f3(unpack_unorm(p, 8), unpack_unorm(p >> 8, 8), unpack_unorm(p >> 16, 8)); return c * c; }
KJB_DEV uint32_t pack_2x16f(float a, float b) { return kjb_f32_to_f16(a) | (kjb_f32_to_f16(b) << 16u); }
KJB_DEV float2 unpack_2x16f(uint32_t u) { return f2(kjb_f16_to_f32(u & 0xffffu), kjb_f16_to_f32(u >> 16)); }
KJB_DEV uint32_t float3_to_rgb9e5(float3 rgb) {
    const float MAX_RGB9E5 = (511.0f / 512.0f) * 65536.0f;
    const float rc = kjb_clamp(rgb.x, 0.0f, MAX_RGB9E5), gc = kjb_clamp(rgb.y, 0.0f, MAX_RGB9E5), bc = kjb_clamp(rgb.z, 0.0f, MAX_RGB9E5);
    const float maxrgb = kjb_max(rc, kjb_max(gc, bc));
    const int fl = int((kjb_f2u(maxrgb) & 0x7F800000u) >> 23) - 127;
    int exp_shared = (fl > -16 ? fl : -16) + 1 + 15;
    float denom = kjb_exp2(float(exp_shared - 15 - 9));
    const int maxm = int(kjb_floor(maxrgb / denom + 0.5f));
    if (maxm == 512) { denom *= 2; exp_shared += 1; }
    const int rm = int(kjb_floor(rc / denom + 0.5f)), gm = int(kjb_floor(gc / denom + 0.5f)), bm = int(kjb_floor(bc / denom + 0.5f));
    return (uint32_t(rm) << 23) | (uint32_t(gm) << 14) | (uint32_t(bm) << 5) | uint32_t(exp_shared);
}
KJB_DEV float3 rgb9e5_to_float3(uint32_t v) {
    const float scale = kjb_exp2(float(int(v & 31u) - 15 - 9));
    return f3(float((v >> 23) & 511u) * scale, float((v >> 14) & 511u) * scale, float((v >> 5) & 511u) * scale);
}

struct GbufferData { float3 albedo, emissive, normal; float roughness, metalness; };
KJB_DEV uint4 gbuffer_pack(const GbufferData& g) {
    return u4(pack_color_888(g.albedo), pack_normal_11_10_11(g.normal), pack_2x16f(kjb_sqrt(g.roughness), g.metalness), float3_to_rgb9e5(g.emissive));
}
KJB_DEV GbufferData gbuffer_unpack(uint4 d) {
    GbufferData r;
    r.albedo = unpack_color_888(d.x);
    r.normal = unpack_normal_11_10_11(d.y);
    const float2 rm = unpack_2x16f(d.z);
    r.roughness = rm.x * rm.x; r.metalness = rm.y;
    r.emissive = rgb9e5_to_float3(d.w);
    return r;
}

// ------------------------------------------------------------------------------------------------ colour
KJB_DEV float luminance(float3 c) { return dot(c, f3(0.2126f, 0.7152f, 0.0722f)); }
KJB_DEV float3 rgb_to_ycbcr(float3 c) { return f3(dot(f3(0.2126f, 0.7152f, 0.0722f), c), dot(f3(-0.1146f, -0.3854f, 0.5f), c), dot(f3(0.5f, -0.4542f, -0.0458f), c)); }
KJB_DEV float3 ycbcr_to_rgb(float3 c) { return vmax(f3(0.0f), f3(dot(f3(1.0f, 0.0f, 1.5748f), c), dot(f3(1.0f, -0.1873f, -.4681f), c), dot(f3(1.0f, 1.8556f, 0.0f), c))); }
KJB_DEV float4 linear_to_working(float4 v) {          // linear_rgb_to_crunched_luma_chroma
    const float3 c = rgb_to_ycbcr(xyz(v));
    const float k = kjb_sqrt(c.x) / kjb_max(1e-8f, c.x);
    return f4(c * k, v.w);
}
KJB_DEV float4 working_to_linear(float4 v) {          // crunched_luma_chroma_to_linear_rgb
    return f4(ycbcr_to_rgb(xyz(v) * v.x), v.w);
}

// ------------------------------------------------------------------------------------------------ reservoirs
struct StreamState { float p_q_sel, M_sum; };
struct Reservoir {
    float w_sum; uint32_t payload; float M, W;
    KJB_DEV static Reservoir create() { Reservoir r; r.w_sum = 0; r.payload = 0; r.M = 0; r.W = 0; return r; }
    KJB_DEV static Reservoir from_raw(uint2 raw) { Reservoir r; r.w_sum = 0; r.payload = raw.x; const float2 mw = unpack_2x16f(raw.y); r.M = mw.x; r.W = mw.y; return r; }
    KJB_DEV uint2 as_raw() const { return u2(payload, pack_2x16f(M, kjb_max(0.0f, W))); }
    KJB_DEV bool update(float w, uint32_t sample_payload, uint32_t& rng) {
        w_sum += w; M += 1;
        const float dart = rand01(rng);
        const float prob = w / w_sum;
        if (prob >= dart) { payload = sample_payload; return true; }
        return false;
    }
    KJB_DEV bool update_with_stream(const Reservoir& r, float p_q, float weight, StreamState& st, uint32_t sample_payload, uint32_t& rng) {
        st.M_sum += r.M;
        if (update(p_q * weight * r.W * r.M, sample_payload, rng)) { st.p_q_sel = p_q; return true; }
        return false;
    }
    KJB_DEV void init_with_stream(float p_q, float weight, StreamState& st, uint32_t sample_payload) {
        payload = sample_payload; w_sum = p_q * weight; M = (weight != 0) ? 1.0f : 0.0f; W = weight;
        st.p_q_sel = p_q; st.M_sum = M;
    }
    KJB_DEV void finish_stream(const StreamState& st) { M = st.M_sum; W = w_sum / kjb_max(1e-8f, M * st.p_q_sel); }
};

// ------------------------------------------------------------------------------------------------ images
// Tightly packed row-major texels in the reference's Vulkan formats; out-of-range loads give 0, stores are dropped.
struct Img { const uint8_t* p; int w, h; };
struct ImgW { uint8_t* p; int w, h; };
KJB_DEV Img img_ro(const kjb_image& i) { Img r; r.p = (const uint8_t*)i.data; r.w = int(i.width); r.h = int(i.height); return r; }
KJB_DEV ImgW img_rw(const kjb_image& i) { ImgW r; r.p = (uint8_t*)i.data; r.w = int(i.width); r.h = int(i.height); return r; }
KJB_DEV Img as_ro(const ImgW& i) { Img r; r.p = i.p; r.w = i.w; r.h = i.h; return r; }
KJB_DEV bool inb(const Img& i, int x, int y) { return (unsigned)x < (unsigned)i.w && (unsigned)y < (unsigned)i.h; }
KJB_DEV bool inb(const ImgW& i, int x, int y) { return (unsigned)x < (unsigned)i.w && (unsigned)y < (unsigned)i.h; }
// texel index inside one layer in 32 bits (an image layer holds < 2^32 texels: one IMAD + one widening IMAD per access instead of 64-bit products)
KJB_DEV size_t texel_offset(int w, int h, int x, int y, int layer, size_t texel_bytes) {
    const uint32_t in_layer = uint32_t(y) * uint32_t(w) + uint32_t(x);
    return (layer == 0 ? size_t(in_layer) : size_t(layer) * size_t(uint32_t(h) * uint32_t(w)) + in_layer) * texel_bytes;
}
template <typename T> KJB_DEV T ld_raw(const Img& i, int x, int y, int layer = 0) { return *(const T*)(i.p + texel_offset(i.w, i.h, x, y, layer, sizeof(T))); }
template <typename T> KJB_DEV void st_raw(const ImgW& i, int x, int y, T v, int layer = 0) { *(T*)(i.p + texel_offset(i.w, i.h, x, y, layer, sizeof(T))) = v; }
KJB_DEV float4 half4_to_float4(uint2 v) { return f4(kjb_f16_to_f32(v.x & 0xffffu), kjb_f16_to_f32(v.x >> 16), kjb_f16_to_f32(v.y & 0xffffu), kjb_f16_to_f32(v.y >> 16)); }
KJB_DEV uint2 float4_to_half4(float4 v) { return u2(pack_2x16f(v.x, v.y), pack_2x16f(v.z, v.w)); }
KJB_DEV float snorm8(uint32_t b) { return kjb_max(KJB_DIV_INT_CONST(float(int(int8_t(b & 0xffu))), 127.0f), -1.0f); }
KJB_DEV float snorm16(uint32_t b) { return kjb_max(KJB_DIV_INT_CONST(float(int(int16_t(b & 0xffffu))), 32767.0f), -1.0f); }
KJB_DEV uint32_t enc_unorm(float v, float scale) { return uint32_t(kjb_clamp(v, 0.0f, 1.0f) * scale + 0.5f); }
KJB_DEV int enc_snorm(float v, float scale) { v = kjb_clamp(v, -1.0f, 1.0f) * scale; return v >= 0.0f ? int(v + 0.5f) : -int(-v + 0.5f); }

KJB_DEV float  ld_r32f(const Img& i, int x, int y) { return inb(i, x, y) ? ld_raw<float>(i, x, y) : 0.0f; }
KJB_DEV float4 ld_rgba32f(const Img& i, int x, int y) { return inb(i, x, y) ? ld_raw<float4>(i, x, y) : f4(0.0f); }
KJB_DEV uint4  ld_rgba32u(const Img& i, int x, int y) { return inb(i, x, y) ? ld_raw<uint4>(i, x, y) : u4(0, 0, 0, 0); }
KJB_DEV uint2  ld_rg32u(const Img& i, int x, int y) { return inb(i, x, y) ? ld_raw<uint2>(i, x, y) : u2(0, 0); }
KJB_DEV float4 ld_rgba16f(const Img& i, int x, int y, int layer = 0) { return inb(i, x, y) ? half4_to_float4(ld_raw<uint2>(i, x, y, layer)) : f4(0.0f); }
KJB_DEV float2 ld_rg16f(const Img& i, int x, int y) { return inb(i, x, y) ? unpack_2x16f(ld_raw<uint32_t>(i, x, y)) : f2(0.0f); }
KJB_DEV float4 ld_rgba8u(const Img& i, int x, int y) {
    if (!inb(i, x, y)) return f4(0.0f);
    const uint32_t v = ld_raw<uint32_t>(i, x, y);
    return f4(KJB_DIV_INT_CONST(float(v & 255u), 255.0f), KJB_DIV_INT_CONST(float((v >> 8) & 255u), 255.0f), KJB_DIV_INT_CONST(float((v >> 16) & 255u), 255.0f), KJB_DIV_INT_CONST(float(v >> 24), 255.0f));
}
KJB_DEV float4 ld_rgba8s(const Img& i, int x, int y) {
    if (!inb(i, x, y)) return f4(0.0f);
    const uint32_t v = ld_raw<uint32_t>(i, x, y);
    return f4(snorm8(v), snorm8(v >> 8), snorm8(v >> 16), snorm8(v >> 24));
}
KJB_DEV float ld_r8u(const Img& i, int x, int y) { return inb(i, x, y) ? KJB_DIV_INT_CONST(float(ld_raw<uint8_t>(i, x, y)), 255.0f) : 0.0f; }
KJB_DEV float ld_r8s(const Img& i, int x, int y) { return inb(i, x, y) ? snorm8(ld_raw<uint8_t>(i, x, y)) : 0.0f; }
KJB_DEV float4 ld_rgba16s(const Img& i, int x, int y) {
    if (!inb(i, x, y)) return f4(0.0f);
    const uint2 v = ld_raw<uint2>(i, x, y);
    return f4(snorm16(v.x), snorm16(v.x >> 16), snorm16(v.y), snorm16(v.y >> 16));
}
KJB_DEV float3 ld_a2r10g10b10(const Img& i, int x, int y) {
    if (!inb(i, x, y)) return f3(0.0f);
    const uint32_t v = ld_raw<uint32_t>(i, x, y);
    return f3(KJB_DIV_INT_CONST(float((v >> 20) & 1023u), 1023.0f), KJB_DIV_INT_CONST(float((v >> 10) & 1023u), 1023.0f), KJB_DIV_INT_CONST(float(v & 1023u), 1023.0f));
}
KJB_DEV void st_r32f(const ImgW& i, int x, int y, float v) { if (inb(i, x, y)) st_raw<float>(i, x, y, v); }
KJB_DEV void st_rgba32f(const ImgW& i, int x, int y, float4 v) { if (inb(i, x, y)) st_raw<float4>(i, x, y, v); }
KJB_DEV void st_rgba32u(const ImgW& i, int x, int y, uint4 v) { if (inb(i, x, y)) st_raw<uint4>(i, x, y, v); }
KJB_DEV void st_rg32u(const ImgW& i, int x, int y, uint2 v) { if (inb(i, x, y)) st_raw<uint2>(i, x, y, v); }
KJB_DEV void st_rgba16f(const ImgW& i, int x, int y, float4 v, int layer = 0) { if (inb(i, x, y)) st_raw<uint2>(i, x, y, float4_to_half4(v), layer); }
KJB_DEV void st_rg16f(const ImgW& i, int x, int y, float a, float b) { if (inb(i, x, y)) st_raw<uint32_t>(i, x, y, pack_2x16f(a, b)); }
KJB_DEV void st_rgba8u(const ImgW& i, int x, int y, float4 v) {
    if (inb(i, x, y)) st_raw<uint32_t>(i, x, y, enc_unorm(v.x, 255.0f) | (enc_unorm(v.y, 255.0f) << 8) | (enc_unorm(v.z, 255.0f) << 16) | (enc_unorm(v.w, 255.0f) << 24));
}
KJB_DEV void st_rgba8s(const ImgW& i, int x, int y, float4 v) {
    if (inb(i, x, y)) st_raw<uint32_t>(i, x, y, (uint32_t(enc_snorm(v.x, 127.0f)) & 255u) | ((uint32_t(enc_snorm(v.y, 127.0f)) & 255u) << 8)
                                                    | ((uint32_t(enc_snorm(v.z, 127.0f)) & 255u) << 16) | ((uint32_t(enc_snorm(v.w, 127.0f)) & 255u) << 24));
}
KJB_DEV void st_r8u(const ImgW& i, int x, int y, float v) { if (inb(i, x, y)) st_raw<uint8_t>(i, x, y, uint8_t(enc_unorm(v, 255.0f))); }
KJB_DEV void st_r8s(const ImgW& i, int x, int y, float v) { if (inb(i, x, y)) st_raw<uint8_t>(i, x, y, uint8_t(enc_snorm(v, 127.0f))); }
KJB_DEV void st_rgba16s(const ImgW& i, int x, int y, float4 v) {
    if (inb(i, x, y)) st_raw<uint2>(i, x, y, u2((uint32_t(enc_snorm(v.x, 32767.0f)) & 0xffffu) | (uint32_t(enc_snorm(v.y, 32767.0f)) << 16),
                                                 (uint32_t(enc_snorm(v.z, 32767.0f)) & 0xffffu) | (uint32_t(enc_snorm(v.w, 32767.0f)) << 16)));
}
KJB_DEV void st_a2r10g10b10(const ImgW& i, int x, int y, float3 v) {
    if (inb(i, x, y)) st_raw<uint32_t>(i, x, y, (enc_unorm(v.x, 1023.0f) << 20) | (enc_unorm(v.y, 1023.0f) << 10) | enc_unorm(v.z, 1023.0f));
}
// B10G11R11_UFLOAT: truncating float->ufloat conversion ("GPU will convert ... by trimming", pack_unpack.hlsl:166-177)
KJB_DEV uint32_t f32_to_uf(float v, int mant_bits) {
    if (!(v > 0.0f)) return 0u;
    const uint32_t u = kjb_f2u(v);
    const int e = int(u >> 23) - 127 + 15;
    const uint32_t m = (u & 0x7fffffu) >> (23 - mant_bits);
    if (e >= 31) return (30u << mant_bits) | ((1u << mant_bits) - 1u);
    if (e <= 0) {
        if (e < -mant_bits) return 0u;
        return ((u & 0x7fffffu) | 0x800000u) >> (23 - mant_bits + 1 - e);
    }
    return (uint32_t(e) << mant_bits) | m;
}
KJB_DEV float uf_to_f32(uint32_t v, int mant_bits) {
    const uint32_t e = v >> mant_bits, m = v & ((1u << mant_bits) - 1u);
    if (e == 0) return float(m) * kjb_exp2(float(-14 - mant_bits));
    if (e == 31) return kjb_u2f(0x7f800000u);
    return kjb_u2f(((e + 112u) << 23) | (m << (23 - mant_bits)));
}
KJB_DEV float3 ld_r11g11b10(const Img& i, int x, int y) {
    if (!inb(i, x, y)) return f3(0.0f);
    const uint32_t v = ld_raw<uint32_t>(i, x, y);
    return f3(uf_to_f32(v & 2047u, 6), uf_to_f32((v >> 11) & 2047u, 6), uf_to_f32(v >> 22, 5));
}
KJB_DEV void st_r11g11b10(const ImgW& i, int x, int y, float3 c) { if (inb(i, x, y)) st_raw<uint32_t>(i, x, y, f32_to_uf(c.x, 6) | (f32_to_uf(c.y, 6) << 11) | (f32_to_uf(c.z, 5) << 22)); }
KJB_DEV float ld_r16f(const Img& i, int x, int y) { return inb(i, x, y) ? kjb_f16_to_f32(ld_raw<uint16_t>(i, x, y)) : 0.0f; }
KJB_DEV void st_r16f(const ImgW& i, int x, int y, float v) { if (inb(i, x, y)) st_raw<uint16_t>(i, x, y, uint16_t(kjb_f32_to_f16(v))); }
KJB_DEV uint32_t ld_r32u(const Img& i, int x, int y) { return inb(i, x, y) ? ld_raw<uint32_t>(i, x, y) : 0u; }
KJB_DEV void st_r32u(const ImgW& i, int x, int y, uint32_t v) { if (inb(i, x, y)) st_raw<uint32_t>(i, x, y, v); }
KJB_DEV int clampi(int v, int n) { return v < 0 ? 0 : (v >= n ? n - 1 : v); }
// SampleLevel(sampler_nnc): nearest, clamp to edge
KJB_DEV int2 nearest_clamp_px(const Img& i, float2 uv) {
    return i2(clampi(kjb_cvt_i32(kjb_floor(uv.x * float(i.w))), i.w), clampi(kjb_cvt_i32(kjb_floor(uv.y * float(i.h))), i.h));
}
// SampleLevel(sampler_lnc): bilinear, clamp to edge.  Fetch is a functor (x, y) -> float4 so any format can be filtered.
template <typename F> KJB_DEV float4 bilinear_clamp(int w, int h, float2 uv, F fetch) {
    const float fx = uv.x * float(w) - 0.5f, fy = uv.y * float(h) - 0.5f;
    const float x0f = kjb_floor(fx), y0f = kjb_floor(fy);
    const float tx = fx - x0f, ty = fy - y0f;
    const int x0 = clampi(kjb_cvt_i32(x0f), w), x1 = clampi(kjb_cvt_i32(x0f) + 1, w), y0 = clampi(kjb_cvt_i32(y0f), h), y1 = clampi(kjb_cvt_i32(y0f) + 1, h);
    const float4 a = fetch(x0, y0), b = fetch(x1, y0), c = fetch(x0, y1), d = fetch(x1, y1);
    const float4 top = vlerp(a, b, tx), bot = vlerp(c, d, tx);
    return vlerp(top, bot, ty);
}
// TextureCube.SampleLevel(sampler_llr): Vulkan face selection, bilinear inside the face (no seamless edges; DESIGN.md)
KJB_DEV float4 sample_cube_rgba16f(const Img& cube, float3 dir) {
    const float ax = kjb_abs(dir.x), ay = kjb_abs(dir.y), az = kjb_abs(dir.z);
    int face; float sc, tc, ma;
    if (ax >= ay && ax >= az) { ma = ax; if (dir.x >= 0) { face = 0; sc = -dir.z; tc = -dir.y; } else { face = 1; sc = dir.z; tc = -dir.y; } }
    else if (ay >= az) { ma = ay; if (dir.y >= 0) { face = 2; sc = dir.x; tc = dir.z; } else { face = 3; sc = dir.x; tc = -dir.z; } }
    else { ma = az; if (dir.z >= 0) { face = 4; sc = dir.x; tc = -dir.y; } else { face = 5; sc = -dir.x; tc = -dir.y; } }
    const float2 uv = f2(0.5f * (sc / ma + 1.0f), 0.5f * (tc / ma + 1.0f));
    return bilinear_clamp(cube.w, cube.h, uv, [&](int x, int y) { return ld_rgba16f(cube, x, y, face); });
}

struct Rows { int y0, y1; };   // row range [y0, y1) of a pass's grid computed by one launch (tile-sharded frames)

// ------------------------------------------------------------------------------------------------ per-launch globals
// Passed BY VALUE to every kernel (lands in the constant bank: uniform, cached reads).  Stands in for descriptor
// sets 1-3: bindless LUTs + mesh data, FrameConstants + lights, acceleration structure.
struct BvhNode;      // kjb_bvh.h
struct BvhTri;
struct TriInfo;
struct SceneView {
    const BvhNode* nodes; const BvhTri* tris; const TriInfo* tri_info;
    const uint8_t* vertices; const kjb_gpu_mesh* meshes; const kjb_instance* instances;
    const uint8_t* tex_data; const uint4* tex_desc;   // per texture: byte offset, width, height, mip_count | (srgb << 16)
    uint32_t tex_count, tri_count;
    int32_t root;                       // HostBvh::root_child
    unsigned long long* ray_counters;   // [0] closest, [1] any-hit
};
struct Globals {
    kjb_frame_constants fc;
    float sun_color[4];                 // sun_color_in_direction(SUN_DIRECTION), a pure function of fc (computed once per frame on the host)
    const kjb_triangle_light* lights;
    Img brdf_fg_lut;                    // 64x64 RGBA16F
    Img blue_noise;                     // 256x256 RGBA8
    SceneView scene;
};

// ------------------------------------------------------------------------------------------------ view / ray context
struct ViewRayContext {
    float4 ray_dir_ws_h, ray_origin_ws_h, ray_hit_cs, ray_hit_vs_h, ray_hit_ws_h;
    KJB_DEV float3 ray_dir_ws() const { return normalize(xyz(ray_dir_ws_h)); }
    KJB_DEV float3 ray_origin_ws() const { return xyz(ray_origin_ws_h) / ray_origin_ws_h.w; }
    KJB_DEV float3 ray_hit_vs() const { return xyz(ray_hit_vs_h) / ray_hit_vs_h.w; }
    KJB_DEV float3 ray_hit_ws() const { return xyz(ray_hit_ws_h) / ray_hit_ws_h.w; }
    KJB_DEV float3 biased_secondary_ray_origin_ws() const { return ray_hit_ws() - ray_dir_ws() * (length(ray_hit_vs()) + length(ray_hit_ws())) * 1e-4f; }
    KJB_DEV float3 biased_secondary_ray_origin_ws_with_normal(float3 normal) const {
        const float3 hw = ray_hit_ws();
        const float3 ws_abs = vabs(hw);
        const float max_comp = kjb_max(kjb_max(ws_abs.x, ws_abs.y), kjb_max(ws_abs.z, -ray_hit_vs().z));
        return hw + (normal - ray_dir_ws()) * kjb_max(1e-4f, max_comp * 1e-6f);
    }
    KJB_DEV static ViewRayContext from_uv(const kjb_view_constants& vc, float2 uv) {
        ViewRayContext r;
        const float2 cs = uv_to_cs(uv);
        r.ray_dir_ws_h = mul(vc.view_to_world, mul(vc.sample_to_view, f4(cs.x, cs.y, 0.0f, 1.0f)));
        r.ray_origin_ws_h = mul(vc.view_to_world, mul(vc.sample_to_view, f4(cs.x, cs.y, 1.0f, 1.0f)));
        r.ray_hit_cs = f4(0.0f); r.ray_hit_vs_h = f4(0.0f); r.ray_hit_ws_h = f4(0.0f);
        return r;
    }
    KJB_DEV static ViewRayContext from_uv_and_depth(const kjb_view_constants& vc, float2 uv, float depth) {
        ViewRayContext r = from_uv(vc, uv);
        const float2 cs = uv_to_cs(uv);
        r.ray_hit_cs = f4(cs.x, cs.y, depth, 1.0f);
        r.ray_hit_vs_h = mul(vc.sample_to_view, r.ray_hit_cs);
        r.ray_hit_ws_h = mul(vc.view_to_world, r.ray_hit_vs_h);
        return r;
    }
    KJB_DEV static ViewRayContext from_uv_and_biased_depth(const kjb_view_constants& vc, float2 uv, float depth) {
        return from_uv_and_depth(vc, uv, kjb_min(1.0f, depth * kjb_u2f(0x3f800040u)));
    }
};
// cheaper variant when only the hit position is needed (restir spatial / resolve inner loops)
KJB_DEV float3 hit_ws_from_uv_depth(const kjb_view_constants& vc, float2 uv, float depth) {
    const float2 cs = uv_to_cs(uv);
    const float4 h = mul(vc.view_to_world, mul(vc.sample_to_view, f4(cs.x, cs.y, depth, 1.0f)));
    return xyz(h) / h.w;
}
KJB_DEV float3 hit_vs_from_uv_depth(const kjb_view_constants& vc, float2 uv, float depth) {
    const float2 cs = uv_to_cs(uv);
    const float4 h = mul(vc.sample_to_view, f4(cs.x, cs.y, depth, 1.0f));
    return xyz(h) / h.w;
}
KJB_DEV float3 get_eye_position(const kjb_view_constants& vc) { const float4 e = mul(vc.view_to_world, f4(0, 0, 0, 1)); return xyz(e) / e.w; }
KJB_DEV float3 direction_view_to_world(const kjb_view_constants& vc, float3 v) { return xyz(mul(vc.view_to_world, f4(v, 0))); }
KJB_DEV float3 direction_world_to_view(const kjb_view_constants& vc, float3 v) { return xyz(mul(vc.world_to_view, f4(v, 0))); }
KJB_DEV float3 position_world_to_clip(const kjb_view_constants& vc, float3 v) { const float4 p = mul(vc.view_to_clip, mul(vc.world_to_view, f4(v, 1))); return xyz(p) / p.w; }
KJB_DEV float3 position_world_to_sample(const kjb_view_constants& vc, float3 v) { const float4 p = mul(vc.view_to_sample, mul(vc.world_to_view, f4(v, 1))); return xyz(p) / p.w; }
KJB_DEV float pixel_cone_spread_angle_from_image_height(const kjb_view_constants& vc, float image_height) { return kjb_atan(2.0f * vc.clip_to_view.m[0] / image_height); }
KJB_DEV int2 halfres_subsample_offset(uint32_t frame_index) {
    const uint32_t i = frame_index & 3u;   // hi_px_subpixels = {(1,1),(1,0),(0,0),(0,1)}
    return i2(i < 2u ? 1 : 0, (i == 0u || i == 3u) ? 1 : 0);
}
struct RayCone { float width, spread_angle; };
KJB_DEV RayCone ray_cone_propagate(RayCone c, float surface_spread_angle, float hit_t) { RayCone r; r.width = c.spread_angle * hit_t + c.width; r.spread_angle = c.spread_angle + surface_spread_angle; return r; }

KJB_DEV float4 blue_noise_for_pixel(const Globals& g, uint32_t px, uint32_t py, uint32_t n) {
    const float2 r2 = r2_sequence(n);
    const uint32_t ox = kjb_cvt_u32(r2.x * 256.0f), oy = kjb_cvt_u32(r2.y * 256.0f);
    return ld_rgba8u(g.blue_noise, int((px + ox) & 255u), int((py + oy) & 255u)) * 255.0f / 256.0f + 0.5f / 256.0f;
}

// ------------------------------------------------------------------------------------------------ atmosphere & sun
KJB_DEV float2 atm_sphere_intersection(float3 ray_start, float3 ray_dir, float3 center, float radius) {
    ray_start = ray_start - center;
    const float a = dot(ray_dir, ray_dir);
    const float b = 2.0f * dot(ray_start, ray_dir);
    const float c = dot(ray_start, ray_start) - (radius * radius);
    float d = b * b - 4 * a * c;
    if (d < 0) return f2(-1.0f);
    d = kjb_sqrt(d);
    return f2(-b - d, -b + d) / (2 * a);
}
#define KJB_PLANET_RADIUS 6371000.0f
#define KJB_ATMOSPHERE_HEIGHT 100000.0f
KJB_DEV float3 atm_density(float3 pos_ws) {
    const float h = length(pos_ws - f3(0, -KJB_PLANET_RADIUS, 0)) - KJB_PLANET_RADIUS;
    return f3(kjb_exp(-kjb_max(0.0f, h / (KJB_ATMOSPHERE_HEIGHT * 0.08f))), kjb_exp(-kjb_max(0.0f, h / (KJB_ATMOSPHERE_HEIGHT * 0.012f))),
              kjb_max(0.0f, 1 - kjb_abs(h - 25000.0f) / 15000.0f));
}
KJB_DEV float3 atm_integrate_optical_depth(float3 ray_start, float3 ray_dir) {
    const float2 isect = atm_sphere_intersection(ray_start, ray_dir, f3(0, -KJB_PLANET_RADIUS, 0), KJB_PLANET_RADIUS + KJB_ATMOSPHERE_HEIGHT);
    const float step_size = isect.y / 8.0f;
    float3 od = f3(0.0f);
    for (int i = 0; i < 8; i++) od += atm_density(ray_start + ray_dir * (float(i) + 0.5f) * step_size) * step_size;
    return od;
}
KJB_DEV float3 atm_absorb(float3 od) {
    const float3 cr = f3(5.802f, 13.558f, 33.100f) * 1e-6f, cm = f3(3.996f, 3.996f, 3.996f) * 1e-6f, co = f3(0.650f, 1.881f, 0.085f) * 1e-6f;
    return vexp(-(od.x * cr + od.y * cm * 1.1f + od.z * co) * 1.0f);
}
KJB_DEV float3 atm_integrate_scattering(float3 ray_start, float3 ray_dir, float ray_length, float3 light_dir) {
    const float2 isect = atm_sphere_intersection(ray_start, ray_dir, f3(0, -KJB_PLANET_RADIUS, 0), KJB_PLANET_RADIUS + KJB_ATMOSPHERE_HEIGHT);
    ray_length = kjb_min(ray_length, isect.y);
    if (isect.x > 0) { ray_start = ray_start + ray_dir * isect.x; ray_length -= isect.x; }
    const float costh = dot(ray_dir, light_dir);
    const float phase_r = 3 * (1 + costh * costh) / (16 * 3.14159265359f);
    const float gk = 1.55f * 0.85f - 0.55f * 0.85f * 0.85f * 0.85f;
    const float kc = gk * costh;
    const float phase_m = (1 - gk * gk) / ((4 * 3.14159265359f) * (1 - kc) * (1 - kc));
    float3 od = f3(0.0f), rayleigh = f3(0.0f), mie = f3(0.0f);
    float prev_t = 0;
    for (int i = 1; i <= 16; i++) {
        const float t = kjb_pow(float(i) / 16.0f, 5.0f) * ray_length;
        const float step_size = t - prev_t;
        const float3 pos = ray_start + ray_dir * kjb_lerp(prev_t, t, 0.5f);
        const float3 dens = atm_density(pos);
        od += dens * step_size;
        const float3 view_tr = atm_absorb(od);
        const float3 light_tr = atm_absorb(atm_integrate_optical_depth(pos, light_dir));
        rayleigh += view_tr * light_tr * phase_r * dens.x * step_size;
        mie += view_tr * light_tr * phase_m * dens.y * step_size;
        prev_t = t;
    }
    const float3 cr = f3(5.802f, 13.558f, 33.100f) * 1e-6f, cm = f3(3.996f, 3.996f, 3.996f) * 1e-6f;
    return (rayleigh * cr + mie * cm) * f3(1.0f) * 20.0f;
}
KJB_DEV float3 sun_direction(const kjb_frame_constants& fc) { return f3(fc.sun_direction[0], fc.sun_direction[1], fc.sun_direction[2]); }
KJB_DEV float3 atmosphere_default(const kjb_frame_constants& fc, float3 wi, float3 light_dir) {
    const float3 amb = f3(fc.sky_ambient[0], fc.sky_ambient[1], fc.sky_ambient[2]), mult = f3(fc.sun_color_multiplier[0], fc.sun_color_multiplier[1], fc.sun_color_multiplier[2]);
    return (amb + mult * atm_integrate_scattering(f3(0.0f), wi, kjb_u2f(0x7f800000u), light_dir)) * fc.pre_exposure;
}
KJB_DEV float3 sun_color_in_direction(const kjb_frame_constants& fc, float3 dir) {
    const float3 mult = f3(fc.sun_color_multiplier[0], fc.sun_color_multiplier[1], fc.sun_color_multiplier[2]);
    return 20.0f * mult * fc.pre_exposure * atm_absorb(atm_integrate_optical_depth(f3(0.0f), dir));
}
KJB_DEV float3 sample_sun_direction(const kjb_frame_constants& fc, float2 urand, bool soft) {
    if (soft && fc.sun_angular_radius_cos < 1.0f) {
        const float3x3 basis = build_orthonormal_basis(normalize(sun_direction(fc)));
        return mul(basis, uniform_sample_cone(urand, fc.sun_angular_radius_cos));
    }
    return sun_direction(fc);
}

// ------------------------------------------------------------------------------------------------ BRDFs
struct BrdfValue { float3 value_over_pdf, value; float pdf; float3 transmission_fraction; };
struct BrdfSample { float3 value_over_pdf, value; float pdf; float3 transmission_fraction; float3 wi; float approx_roughness; };
KJB_DEV BrdfValue brdf_value_invalid() { BrdfValue r; r.value_over_pdf = f3(0.0f); r.value = f3(0.0f); r.pdf = 0; r.transmission_fraction = f3(0.0f); return r; }
KJB_DEV BrdfSample brdf_sample_invalid() { BrdfSample r; r.value_over_pdf = f3(0.0f); r.value = f3(0.0f); r.pdf = 0; r.transmission_fraction = f3(0.0f); r.wi = f3(0, 0, -1); r.approx_roughness = 0; return r; }
KJB_DEV float3 fresnel_schlick(float3 f0, float3 f90, float cos_theta) { return vlerp(f0, f90, kjb_pow(kjb_max(0.0f, 1.0f - cos_theta), 5.0f)); }
KJB_DEV float g_smith_ggx_correlated(float ndotv, float ndotl, float a2) {
    const float lv = ndotl * kjb_sqrt((-ndotv * a2 + ndotv) * ndotv + a2);
    const float ll = ndotv * kjb_sqrt((-ndotl * a2 + ndotl) * ndotl + a2);
    return 2.0f * ndotl * ndotv / (lv + ll);
}
KJB_DEV float g_smith_ggx1(float ndotv, float a2) { const float t2 = (1.0f - ndotv * ndotv) / (ndotv * ndotv); return 2.0f / (1.0f + kjb_sqrt(1.0f + a2 * t2)); }
KJB_DEV float ggx_ndf(float a2, float cos_theta) { const float ds = cos_theta * cos_theta * (a2 - 1.0f) + 1.0f; return a2 / (KJB_PI_F * ds * ds); }
KJB_DEV float pdf_ggx_vn(float a2, float3 wo, float3 h) { return g_smith_ggx1(wo.z, a2) * ggx_ndf(a2, h.z) * kjb_max(0.f, dot(wo, h)) / wo.z; }
struct SpecularBrdf { float roughness; float3 albedo; };
struct DiffuseBrdf { float3 albedo; };
KJB_DEV BrdfValue diffuse_evaluate(const DiffuseBrdf& b, float3 wi) {
    BrdfValue r; r.pdf = wi.z > 0.0f ? KJB_FRAC_1_PI : 0.0f; r.value_over_pdf = wi.z > 0.0f ? b.albedo : f3(0.0f);
    r.value = r.value_over_pdf * r.pdf; r.transmission_fraction = f3(0.0f); return r;
}
KJB_DEV BrdfSample diffuse_sample(const DiffuseBrdf& b, float2 urand) {
    const float phi = urand.x * KJB_TAU_F;
    const float cos_theta = kjb_sqrt(kjb_max(0.0f, 1.0f - urand.y));
    const float sin_theta = kjb_sqrt(kjb_max(0.0f, 1.0f - cos_theta * cos_theta));
    float sp, cp; kjb_sincos(phi, &sp, &cp);
    BrdfSample r; r.wi = f3(cp * sin_theta, sp * sin_theta, cos_theta); r.pdf = KJB_FRAC_1_PI; r.value_over_pdf = b.albedo; r.value = r.value_over_pdf * r.pdf;
    r.transmission_fraction = f3(0.0f); r.approx_roughness = 1.0f; return r;
}
KJB_DEV BrdfValue specular_evaluate(const SpecularBrdf& b, float3 wo, float3 wi) {
    if (wi.z <= 0.0f || wo.z <= 0.0f) return brdf_value_invalid();
    const float a2 = b.roughness * b.roughness;
    const float3 m = normalize(wo + wi);
    const float cos_theta = m.z;
    const float pdf_h = pdf_ggx_vn(a2, wo, m);
    const float jacobian = 1.0f / (4.0f * dot(wi, m));
    const float3 fresnel = fresnel_schlick(b.albedo, f3(1.0f), dot(m, wi));
    const float g = g_smith_ggx_correlated(wo.z, wi.z, a2);
    const float g_over_g1_wo = g / g_smith_ggx1(wo.z, a2);
    BrdfValue r; r.pdf = pdf_h * jacobian / wi.z; r.transmission_fraction = f3(1.0f) - fresnel;
    r.value_over_pdf = fresnel * g_over_g1_wo;
    r.value = fresnel * g * ggx_ndf(a2, cos_theta) / (4 * wo.z * wi.z);
    return r;
}
KJB_DEV BrdfSample specular_sample(const SpecularBrdf& b, float3 wo, float2 urand) {
    // sample_vndf (brdf.hlsl:186-214)
    const float alpha = b.roughness, a2 = alpha * alpha;
    const float3 Vh = normalize(f3(alpha * wo.x, alpha * wo.y, wo.z));
    const float3 T1 = (Vh.z < 0.9999f) ? normalize(cross(f3(0, 0, 1), Vh)) : f3(1, 0, 0);
    const float3 T2 = cross(Vh, T1);
    const float r = kjb_sqrt(urand.x);
    const float phi = (2.f * KJB_PI_F) * urand.y;
    float sp, cp; kjb_sincos(phi, &sp, &cp);
    const float t1 = r * cp;
    float t2 = r * sp;
    const float s = 0.5f * (1.f + Vh.z);
    t2 = (1.f - s) * kjb_sqrt(1.f - t1 * t1) + s * t2;
    const float3 Nh = t1 * T1 + t2 * T2 + kjb_sqrt(kjb_max(0.f, 1.f - t1 * t1 - t2 * t2)) * Vh;
    const float3 h = normalize(f3(alpha * Nh.x, alpha * Nh.y, kjb_max(0.f, Nh.z)));
    const float ndf_pdf = pdf_ggx_vn(a2, wo, h);
    const float3 wi = reflect(-wo, h);
    if (h.z <= 1e-5f || wi.z <= 1e-5f || wo.z <= 1e-5f) return brdf_sample_invalid();
    const float jacobian = 1.0f / (4.0f * dot(wi, h));
    const float3 fresnel = fresnel_schlick(b.albedo, f3(1.0f), dot(h, wi));
    const float g = g_smith_ggx_correlated(wo.z, wi.z, a2);
    const float g_over_g1_wo = g / g_smith_ggx1(wo.z, a2);
    BrdfSample res; res.pdf = ndf_pdf * jacobian / wi.z; res.wi = wi; res.transmission_fraction = f3(1.0f) - fresnel; res.approx_roughness = b.roughness;
    res.value_over_pdf = fresnel * g_over_g1_wo;
    res.value = fresnel * g * ggx_ndf(a2, h.z) / (4 * wo.z * wi.z);
    return res;
}
struct EnergyPreservation { float3 preintegrated_reflection, preintegrated_reflection_mult, preintegrated_transmission_fraction; float valid_sample_fraction; };
struct LayeredBrdf { SpecularBrdf specular_brdf; DiffuseBrdf diffuse_brdf; EnergyPreservation ep; };
struct Globals;
KJB_DEV EnergyPreservation energy_preservation_from_brdf_ndotv(const Globals& g, const SpecularBrdf& s, float ndotv);
KJB_DEV LayeredBrdf layered_brdf_from_gbuffer_ndotv(const Globals& g, const GbufferData& gb, float ndotv) {
    SpecularBrdf s; s.albedo = f3(0.04f); s.roughness = gb.roughness;
    DiffuseBrdf d; d.albedo = gb.albedo;
    {   // apply_metalness_to_brdfs + metalness_albedo_boost
        const float3 albedo = d.albedo; const float x = gb.metalness;
        s.albedo = vlerp(s.albedo, albedo, x);
        d.albedo = kjb_max(0.0f, 1.0f - x) * albedo;
        const float3 y3 = albedo * albedo * albedo;
        const float3 boost = 1.0f + (0.25f - (x - 0.5f) * (x - 0.5f)) * (1.749f + -1.61f * kjb_abs(x - 0.5f)) * (0.5555f * albedo + 0.8244f * y3);
        s.albedo = vmin(f3(1.0f), s.albedo * boost);
        d.albedo = vmin(f3(1.0f), d.albedo * boost);
    }
    LayeredBrdf r;
    r.ep = energy_preservation_from_brdf_ndotv(g, s, ndotv);
    r.specular_brdf = s; r.diffuse_brdf = d;
    return r;
}
// SpecularBrdfEnergyPreservation::from_brdf_ndotv (brdf_lut.hlsl:15-77, `#elif 1` branch)
KJB_DEV EnergyPreservation energy_preservation_from_brdf_ndotv(const Globals& g, const SpecularBrdf& s, float ndotv) {
    EnergyPreservation ep;
    const float2 uv = f2(ndotv, s.roughness) * f2((64.0f - 1.0f) / 64.0f) + f2(0.5f / 64.0f);
    const float4 fg = bilinear_clamp(64, 64, uv, [&](int x, int y) { return ld_rgba16f(g.brdf_fg_lut, x, y); });
    const float3 single_scatter = s.albedo * fg.x + fg.y;
    ep.valid_sample_fraction = fg.z;
    const float e_ss = fg.x + fg.y;
    const float3 f_ss = single_scatter / e_ss;
    const float3 f_ss_tail = vlerp(f_ss, f3(1.0f), 0.4f);
    const float3 bounce_radiance = (1.0f - e_ss) * f_ss_tail;
    const float3 mult = 1.0f + bounce_radiance / (1.0f - bounce_radiance);
    ep.preintegrated_reflection = single_scatter * mult;
    ep.preintegrated_reflection_mult = mult;
    ep.preintegrated_transmission_fraction = 1.0f - ep.preintegrated_reflection;
    return ep;
}
KJB_DEV float3 layered_evaluate(const LayeredBrdf& b, float3 wo, float3 wi) {
    if (wo.z <= 0 || wi.z <= 0) return f3(0.0f);
    const BrdfValue diff = diffuse_evaluate(b.diffuse_brdf, wi);
    const BrdfValue spec = specular_evaluate(b.specular_brdf, wo, wi);
    return spec.value * b.ep.preintegrated_reflection_mult + diff.value * spec.transmission_fraction;
}
KJB_DEV float3 layered_evaluate_directional_light(const LayeredBrdf& b, float3 wo, float3 wi) {
    if (wo.z <= 0 || wi.z <= 0) return f3(0.0f);
    const BrdfValue diff = diffuse_evaluate(b.diffuse_brdf, wi);
    const BrdfValue spec = specular_evaluate(b.specular_brdf, wo, wi);
    const float3 mult_dir = vlerp(f3(1.0f), b.ep.preintegrated_reflection_mult, kjb_sqrt(kjb_abs(wi.z)));
    return spec.value * mult_dir + diff.value * spec.transmission_fraction;
}
KJB_DEV BrdfSample layered_sample(const LayeredBrdf& b, float3 wo, float3 urand) {
    const float spec_wt = luminance(b.ep.preintegrated_reflection);
    const float diffuse_wt = luminance(b.ep.preintegrated_transmission_fraction * b.diffuse_brdf.albedo);
    const float transmission_p = diffuse_wt / (spec_wt + diffuse_wt);
    BrdfSample s;
    if (urand.z < transmission_p) {
        s = diffuse_sample(b.diffuse_brdf, f2(urand.x, urand.y));
        s.value_over_pdf = s.value_over_pdf / transmission_p; s.pdf *= transmission_p;
        s.value_over_pdf *= b.ep.preintegrated_transmission_fraction; s.value *= b.ep.preintegrated_transmission_fraction;
    } else {
        s = specular_sample(b.specular_brdf, wo, f2(urand.x, urand.y));
        const float lobe_pdf = 1.0f - transmission_p;
        s.value_over_pdf = s.value_over_pdf / lobe_pdf; s.pdf *= lobe_pdf;
        s.value_over_pdf *= b.ep.preintegrated_reflection_mult; s.value *= b.ep.preintegrated_reflection_mult;
    }
    return s;
}

struct LightSample { float3 pos, normal; float pdf; };
KJB_DEV LightSample sample_triangle_light(const kjb_triangle_light& tl, float2 urand) {
    const float3 v = f3(tl.verts[0][0], tl.verts[0][1], tl.verts[0][2]);
    const float3 e0 = f3(tl.verts[1][0], tl.verts[1][1], tl.verts[1][2]) - v, e1 = f3(tl.verts[2][0], tl.verts[2][1], tl.verts[2][2]) - v;
    const float3 perp = cross(e0, e1);
    const float perp_inv_len = kjb_rsqrt(dot(perp, perp));
    const float su0 = kjb_sqrt(urand.x);
    LightSample r; r.pos = v + (1.0f - su0) * e0 + (urand.y * su0) * e1; r.normal = perp * perp_inv_len; r.pdf = 2.0f * perp_inv_len;
    return r;
}

}  // namespace kjb
