// Ray traversal + hit shading for H100 SMs.
//
// The reference delegates traversal to VK_KHR_ray_tracing (TraceRay in inc/rt.hlsl:58-70,112-137) and shades hits in
// rt/gbuffer.rchit.hlsl:46-202.  Here both run in the calling kernel: a stack-based while-while BVH2 walk over 64-byte
// two-box nodes (kjb_bvh.h), Moeller-Trumbore in the operation order fixed by DESIGN.md "ray/triangle contract"
// (tmin < t < tmax, closest = min t, ties -> smallest global triangle id), then the closest-hit material fetch from
// kajiya's unified vertex buffer (inc/mesh.hlsl:10-68).  Node and triangle loads are 16-byte vector loads.
#pragma once
#include "kjb_device.cuh"
#include "kjb_bvh.h"

namespace kjb {

struct Ray { float3 origin, dir; float tmin, tmax; };
struct HitInfo { bool hit; float t, u, v; uint32_t gid; };

// child slot k of a node from the exact box b = (lo, hi): the slab test only culls, so the box is padded against its rounding.  The device
// build (kjb_bvh_build.cuh) and the refit (kjb_api.cu) both write every box through here.
KJB_DEV void write_padded_slot(BvhNode& nd, int k, const float* b) {
    float lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        const float pad = (b[3 + a] - b[a]) * 1e-5f + 1e-6f + 1e-6f * kjb_max(kjb_abs(b[a]), kjb_abs(b[3 + a]));
        lo[a] = b[a] - pad; hi[a] = b[3 + a] + pad;
    }
    float* nxy = k == 0 ? nd.n0 : nd.n1;
    nxy[0] = lo[0]; nxy[1] = hi[0]; nxy[2] = lo[1]; nxy[3] = hi[1];
    nd.n2[k * 2 + 0] = lo[2]; nd.n2[k * 2 + 1] = hi[2];
}

KJB_DEV float4 ldg4(const float* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(reinterpret_cast<const float4*>(p));
#else
    return f4(p[0], p[1], p[2], p[3]);
#endif
}

// intersection of one leaf's triangles; `best` updated in place
template <bool ANY_HIT>
KJB_DEV bool intersect_leaf(const BvhTri* tris, uint32_t first, uint32_t count, const Ray& r, bool cull_back, HitInfo& best) {
    for (uint32_t i = 0; i < count; ++i) {
        const float* tp = reinterpret_cast<const float*>(tris + first + i);
        const float4 a = ldg4(tp), b = ldg4(tp + 4), c = ldg4(tp + 8);
        const float3 v0 = f3(a.x, a.y, a.z), e1 = f3(b.x, b.y, b.z), e2 = f3(c.x, c.y, c.z);
        const float3 p = cross(r.dir, e2);
        const float det = dot(e1, p);
        if (det == 0.0f) continue;
        if (cull_back && det < 0.0f) continue;
        const float inv = 1.0f / det;
        const float3 tv = r.origin - v0;
        const float u = dot(tv, p) * inv;
        if (u < 0.0f || u > 1.0f) continue;
        const float3 q = cross(tv, e1);
        const float v = dot(r.dir, q) * inv;
        if (v < 0.0f || u + v > 1.0f) continue;
        const float t = dot(e2, q) * inv;
        if (!(t > r.tmin && t < r.tmax)) continue;
        if (ANY_HIT) return true;
        const uint32_t gid = kjb_f2u(a.w);
        if (!best.hit || t < best.t || (t == best.t && gid < best.gid)) { best.hit = true; best.t = t; best.u = u; best.v = v; best.gid = gid; }
    }
    return false;
}

// the slab test's min/max are kjb_min / kjb_max: one FMNMX each on the device (include/kjb_numeric.h)
#define KJB_SLAB_MIN kjb_min
#define KJB_SLAB_MAX kjb_max

// Culling slack: a child is kept when tn*(1 - s) <= min(tf, best.t)*(1 + s) (signs handled), s = KJB_SLAB_SLACK_K * 2^-24 = u * k.  Padding
// alone cannot keep culling conservative: the slab terms round relative to |plane - origin| (far origins), and the Moeller-Trumbore t of a
// triangle lying on its box's face (floors, walls: flat boxes) can come out below the computed box entry.  The bound, to first order in u:
//  * slab: c = (plane - o) * (1/d) is three roundings, min/max are exact, so the computed tn <= tn + 3u|tn| and tf >= tf - 3u|tf|;
//    the slack multiply is one more rounding;
//  * Moeller-Trumbore (kjb_device.cuh: cross without fma, dot with two fma): N = dot(e2, cross(o - v0, e1)) carries 6 roundings,
//    det = dot(e1, cross(d, e2)) 5, each at most 1.155 (= 2/sqrt 3, the largest |a||b||c|-normalised absolute triple product) of
//    u|a||b||c|; then 1/det and N*inv.  With S = |e1||e2| / |e1 x e2| (triangle shape), cos = the cosine between d and the normal and
//    rho = |o - v0| / (t|d|), the relative error of t is  delta <= (1.155 (6 rho + 5) S / |cos| + 2) u.
// A triangle whose exact hit lies in the box is therefore never culled while delta + 4u <= s, i.e. 1.155 (6 rho + 5) S / |cos| <= k - 6:
// with k = 2^14, S / |cos| <= 1290 for rho = 1 (origin far from the triangle) and <= 1010 for rho = 1.5.  Rays beyond that (grazing,
// slivers, origins close to a large triangle) may still lose a near-tie to topology; tests/test_ray_contract.py tags them ill-conditioned.
// Each bound is one FFMA with an |t| operand, rounded once: t - s|t|, t + s|t|.  An infinite tn = +inf or tf = -inf turns into NaN, which
// fails tn <= tf as the infinity would have.
#define KJB_SLAB_SLACK_K 16384.0f
KJB_DEV float slab_near(float t) { return kjb_fma(-KJB_SLAB_SLACK_K * 0x1p-24f, kjb_abs(t), t); }
KJB_DEV float slab_far(float t) { return kjb_fma(KJB_SLAB_SLACK_K * 0x1p-24f, kjb_abs(t), t); }
template <bool ANY_HIT>
KJB_DEV HitInfo trace(const SceneView& sc, const Ray& r, bool cull_back) {
    HitInfo best; best.hit = false; best.t = r.tmax; best.u = 0; best.v = 0; best.gid = 0xffffffffu;
    // A ray with a NaN anywhere can never pass the triangle test (every comparison on t/u/v is false), but the NaN-ignoring min/max of
    // the slab test would let it visit EVERY node.  Such rays are routine — the validation passes re-trace stored rays, and an empty
    // reservoir stores a zero-length one (normalize(0) = NaN).  Same result, no traversal.
    if (!(r.dir.x == r.dir.x && r.dir.y == r.dir.y && r.dir.z == r.dir.z && r.origin.x == r.origin.x && r.origin.y == r.origin.y && r.origin.z == r.origin.z
          && r.tmin == r.tmin && r.tmax == r.tmax)) return best;
    const float3 inv_dir = f3(1.0f / r.dir.x, 1.0f / r.dir.y, 1.0f / r.dir.z);
    int stack[64]; int sp = 0;
    int cur = sc.root;   // inner node index (>= 0) or an encoded leaf (< 0) when the whole scene is one leaf
    // "while-while" walk: every lane first descends through inner nodes until it holds a leaf (or runs out of work), then the lanes
    // that hold leaves intersect them together — fewer mixed node/leaf iterations per warp than a single interleaved loop.
    // The visiting order per ray is unchanged (near child first, far child pushed), hence so is the result.
    const int DONE = 0x7fffffff;
    for (;;) {
        while (cur >= 0 && cur != DONE) {
            const float* np = reinterpret_cast<const float*>(sc.nodes + cur);
            const float4 n0 = ldg4(np), n1 = ldg4(np + 4), n2 = ldg4(np + 8);
            const int2 ch = *reinterpret_cast<const int2*>(np + 12);
            // slab test on both children; (plane - origin) * inv_dir written as plane*inv_dir - origin*inv_dir is NOT used: keep
            // the subtraction first so that boxes padded on the host stay conservative
            const float c0lox = (n0.x - r.origin.x) * inv_dir.x, c0hix = (n0.y - r.origin.x) * inv_dir.x;
            const float c0loy = (n0.z - r.origin.y) * inv_dir.y, c0hiy = (n0.w - r.origin.y) * inv_dir.y;
            const float c0loz = (n2.x - r.origin.z) * inv_dir.z, c0hiz = (n2.y - r.origin.z) * inv_dir.z;
            const float c1lox = (n1.x - r.origin.x) * inv_dir.x, c1hix = (n1.y - r.origin.x) * inv_dir.x;
            const float c1loy = (n1.z - r.origin.y) * inv_dir.y, c1hiy = (n1.w - r.origin.y) * inv_dir.y;
            const float c1loz = (n2.z - r.origin.z) * inv_dir.z, c1hiz = (n2.w - r.origin.z) * inv_dir.z;
            const float tmax_cur = ANY_HIT ? r.tmax : best.t;
            const float t0n = slab_near(KJB_SLAB_MAX(KJB_SLAB_MAX(KJB_SLAB_MIN(c0lox, c0hix), KJB_SLAB_MIN(c0loy, c0hiy)), KJB_SLAB_MAX(KJB_SLAB_MIN(c0loz, c0hiz), r.tmin)));
            const float t0f = slab_far(KJB_SLAB_MIN(KJB_SLAB_MIN(KJB_SLAB_MAX(c0lox, c0hix), KJB_SLAB_MAX(c0loy, c0hiy)), KJB_SLAB_MIN(KJB_SLAB_MAX(c0loz, c0hiz), tmax_cur)));
            const float t1n = slab_near(KJB_SLAB_MAX(KJB_SLAB_MAX(KJB_SLAB_MIN(c1lox, c1hix), KJB_SLAB_MIN(c1loy, c1hiy)), KJB_SLAB_MAX(KJB_SLAB_MIN(c1loz, c1hiz), r.tmin)));
            const float t1f = slab_far(KJB_SLAB_MIN(KJB_SLAB_MIN(KJB_SLAB_MAX(c1lox, c1hix), KJB_SLAB_MAX(c1loy, c1hiy)), KJB_SLAB_MIN(KJB_SLAB_MAX(c1loz, c1hiz), tmax_cur)));
            const bool h0 = t0n <= t0f, h1 = t1n <= t1f;
            if (h0 && h1) {
                const bool near0 = t0n <= t1n;
                stack[sp++] = near0 ? ch.y : ch.x;
                cur = near0 ? ch.x : ch.y;
            } else if (h0) cur = ch.x;
            else if (h1) cur = ch.y;
            else cur = sp ? stack[--sp] : DONE;
        }
        if (cur == DONE) break;
        {
            const uint32_t enc = uint32_t(~cur);
            if (intersect_leaf<ANY_HIT>(sc.tris, enc >> 3, (enc & 7u) + 1u, r, cull_back, best)) { best.hit = true; return best; }
        }
        cur = sp ? stack[--sp] : DONE;
    }
    return best;
}

KJB_DEV void count_ray(const SceneView& sc, int which) {
#if defined(__CUDA_ARCH__)
    // one atomic per warp: ballot the active lanes, leader adds the popcount
    const unsigned m = __activemask();
    if ((threadIdx.x + threadIdx.y * blockDim.x) % 32 == __ffs(m) - 1) atomicAdd(sc.ray_counters + which, (unsigned long long)__popc(m));
#else
    __atomic_fetch_add(sc.ray_counters + which, 1ull, __ATOMIC_RELAXED);
#endif
}

// ---------------------------------------------------------------------------------------------- bindless texture fetch
KJB_DEV float srgb_eotf(float a) { return .04045f < a ? kjb_pow((a + .055f) / 1.055f, 2.4f) : a / 12.92f; }
KJB_DEV float4 tex_texel(const SceneView& sc, uint4 d, int mip, int x, int y) {
    const int w = int(d.y >> mip) > 1 ? int(d.y >> mip) : 1, h = int(d.z >> mip) > 1 ? int(d.z >> mip) : 1;
    x = ((x % w) + w) % w; y = ((y % h) + h) % h;
    size_t off = d.x;
    for (int m = 0; m < mip; ++m) { const size_t mw = (d.y >> m) > 1 ? (d.y >> m) : 1, mh = (d.z >> m) > 1 ? (d.z >> m) : 1; off += mw * mh * 4; }
    const uint8_t* p = sc.tex_data + off + (size_t(y) * w + x) * 4;
    float4 c = f4(float(p[0]) / 255.0f, float(p[1]) / 255.0f, float(p[2]) / 255.0f, float(p[3]) / 255.0f);
    if (d.w >> 16) { c.x = srgb_eotf(c.x); c.y = srgb_eotf(c.y); c.z = srgb_eotf(c.z); }
    return c;
}
KJB_DEV float4 tex_bilinear_repeat(const SceneView& sc, uint4 d, int mip, float2 uv) {
    const int w = int(d.y >> mip) > 1 ? int(d.y >> mip) : 1, h = int(d.z >> mip) > 1 ? int(d.z >> mip) : 1;
    const float fx = uv.x * float(w) - 0.5f, fy = uv.y * float(h) - 0.5f;
    const float x0f = kjb_floor(fx), y0f = kjb_floor(fy); const float tx = fx - x0f, ty = fy - y0f;
    const int x0 = kjb_cvt_i32(x0f), y0 = kjb_cvt_i32(y0f);
    const float4 a = tex_texel(sc, d, mip, x0, y0), b = tex_texel(sc, d, mip, x0 + 1, y0), c = tex_texel(sc, d, mip, x0, y0 + 1), e = tex_texel(sc, d, mip, x0 + 1, y0 + 1);
    const float4 top = a + (b - a) * tx, bot = c + (e - c) * tx;
    return top + (bot - top) * ty;
}
// SampleLevel(sampler_llr, uv, lod): trilinear, repeat
KJB_DEV float4 tex_sample_level(const SceneView& sc, uint32_t tex, float2 uv, float lod) {
    if (tex >= sc.tex_count) return f4(1.0f);
    const uint4 d = sc.tex_desc[tex];
    const int mips = int(d.w & 0xffffu);
    if (mips == 1 && d.y == 1u && d.z == 1u) return tex_texel(sc, d, 0, 0, 0);   // 1x1 placeholder maps: every filter tap is the same texel
    const float maxl = float(mips - 1);
    if (!(lod > 0.0f)) lod = 0.0f;
    if (lod > maxl) lod = maxl;
    const int l0 = kjb_cvt_i32(kjb_floor(lod)); const float f = lod - float(l0);
    const float4 a = tex_bilinear_repeat(sc, d, l0, uv);
    if (f == 0.0f || l0 + 1 >= mips) return a;
    const float4 b = tex_bilinear_repeat(sc, d, l0 + 1, uv);
    return a + (b - a) * f;
}
KJB_DEV float texture_lod(const SceneView& sc, uint32_t tex, float triangle_constant, float3 ray_direction, float3 surf_normal, float cone_width) {
    float2 wh = f2(1.0f);
    if (tex < sc.tex_count) { const uint4 d = sc.tex_desc[tex]; wh = f2(float(d.y), float(d.z)); }
    float lambda = triangle_constant;
    lambda += kjb_log2(kjb_abs(cone_width));
    lambda += 0.5f * kjb_log2(wh.x * wh.y);
    lambda -= kjb_log2(kjb_abs(dot(normalize(ray_direction), surf_normal)));
    return lambda;
}

KJB_DEV uint32_t vb_u32(const SceneView& sc, uint32_t off) { return *reinterpret_cast<const uint32_t*>(sc.vertices + off); }
KJB_DEV float vb_f32(const SceneView& sc, uint32_t off) { return *reinterpret_cast<const float*>(sc.vertices + off); }
KJB_DEV float3 unpack_unit_direction_11_10_11(uint32_t pck) {
    return f3(float(pck & ((1u << 11u) - 1u)) * (2.0f / float((1u << 11u) - 1u)) - 1.0f,
              float((pck >> 11u) & ((1u << 10u) - 1u)) * (2.0f / float((1u << 10u) - 1u)) - 1.0f,
              float((pck >> 21u)) * (2.0f / float((1u << 11u) - 1u)) - 1.0f);
}
KJB_DEV float2 transform_material_uv(const float* t, float2 uv, uint32_t map_idx) {
    const uint32_t xo = map_idx * 6;
    return f2(t[xo + 0] * uv.x + t[xo + 1] * uv.y, t[xo + 2] * uv.x + t[xo + 3] * uv.y) + f2(t[xo + 4], t[xo + 5]);
}

// closest-hit shader (rt/gbuffer.rchit.hlsl:46-202): returns the packed 16-byte G-buffer payload
KJB_DEV uint4 rchit_gbuffer(const Globals& g, const Ray& ray, const HitInfo& hit, RayCone ray_cone, uint32_t path_length, float3* geometric_normal_ws_out = nullptr) {
    const SceneView& sc = g.scene;
    const TriInfo ti = sc.tri_info[hit.gid];
    const kjb_instance& inst = sc.instances[ti.instance];
    const kjb_gpu_mesh mesh = sc.meshes[inst.mesh_index];
    const float* o2w = inst.transform;
    const float3 hit_point = ray.origin + ray.dir * hit.t;
    const float hit_dist = length(hit_point - ray.origin);
    const float3 bary = f3(1.0f - hit.u - hit.v, hit.u, hit.v);

    uint32_t ind[3];
    for (int k = 0; k < 3; ++k) ind[k] = vb_u32(sc, mesh.index_offset + (ti.prim * 3 + k) * 4);
    float3 vp[3], vn[3];
    for (int k = 0; k < 3; ++k) {
        const float4 v = *reinterpret_cast<const float4*>(sc.vertices + mesh.vertex_core_offset + ind[k] * 16);
        vp[k] = f3(v.x, v.y, v.z); vn[k] = unpack_unit_direction_11_10_11(kjb_f2u(v.w));
    }
    float3 normal = vn[0] * bary.x + vn[1] * bary.y + vn[2] * bary.z;
    const float3 surf_normal_os = normalize(cross(vp[1] - vp[0], vp[2] - vp[0]));
    const float3 surf_normal_ws = normalize(xform_dir(o2w, surf_normal_os));
    if (g.fc.render_override_flags & KJB_OVERRIDE_FORCE_FACE_NORMALS) normal = surf_normal_os;

    float4 v_color = f4(1.0f);
    if (mesh.vertex_aux_offset != 0) {
        float4 vc[3];
        for (int k = 0; k < 3; ++k) vc[k] = *reinterpret_cast<const float4*>(sc.vertices + mesh.vertex_aux_offset + ind[k] * 16);
        v_color = vc[0] * bary.x + vc[1] * bary.y + vc[2] * bary.z;
    }
    float2 uvs[3];
    for (int k = 0; k < 3; ++k) uvs[k] = *reinterpret_cast<const float2*>(sc.vertices + mesh.vertex_uv_offset + ind[k] * 8);
    const float2 uv = uvs[0] * bary.x + uvs[1] * bary.y + uvs[2] * bary.z;

    const uint32_t material_id = vb_u32(sc, mesh.vertex_mat_offset + ind[0] * 4);
    const kjb_mesh_material& material = *reinterpret_cast<const kjb_mesh_material*>(sc.vertices + mesh.mat_data_offset + material_id * (uint32_t)sizeof(kjb_mesh_material));

    // A map that is a single texel (kajiya's 1x1 placeholders for materials without that texture) returns the same value for every uv and lod
    // (tex_sample_level's first branch), so the ray-cone lod — four log2 per map plus the world-space triangle area — is evaluated only when a
    // map of this material actually has texels to filter.  Same result either way; untextured scenes skip ~350 instructions per hit.
#ifndef KJB_LOD_SKIP
#define KJB_LOD_SKIP 1
#endif
    auto flat = [&](uint32_t tex) { if (!KJB_LOD_SKIP) return false; if (tex >= sc.tex_count) return true; const uint4 d = sc.tex_desc[tex]; return (d.w & 0xffffu) == 1u && d.y == 1u && d.z == 1u; };
    const bool any_filtered = !flat(material.maps[2]) || !flat(material.maps[1]) || !flat(material.maps[3]);
    float cone_width = 0.0f, lod_triangle_constant = 0.0f;
    if (any_filtered) {
        cone_width = ray_cone.width + ray_cone.spread_angle * hit_dist;
        const float3 p0 = xform_point(o2w, vp[0]), p1 = xform_point(o2w, vp[1]), p2 = xform_point(o2w, vp[2]);
        const float twice_uv_area = kjb_abs((uvs[1].x - uvs[0].x) * (uvs[2].y - uvs[0].y) - (uvs[2].x - uvs[0].x) * (uvs[1].y - uvs[0].y));
        const float twice_triangle_area = length(cross(p1 - p0, p2 - p0));
        lod_triangle_constant = 0.5f * kjb_log2(twice_uv_area / twice_triangle_area);
    }
    auto sample_map = [&](uint32_t tex, uint32_t uv_slot) {
        if (flat(tex)) return tex_sample_level(sc, tex, f2(0.0f), 0.0f);
        return tex_sample_level(sc, tex, transform_material_uv(material.map_transforms, uv, uv_slot), texture_lod(sc, tex, lod_triangle_constant, ray.dir, surf_normal_ws, cone_width));
    };

    const float3 albedo = xyz(sample_map(material.maps[2], 0))
        * f3(material.base_color_mult[0], material.base_color_mult[1], material.base_color_mult[2]) * xyz(v_color);

    const float4 metalness_roughness = sample_map(material.maps[1], 2);
    const float perceptual_roughness = material.roughness_mult * metalness_roughness.x;
    float roughness = kjb_clamp(perceptual_roughness * perceptual_roughness, 1e-4f, 1.0f);
    float metalness = metalness_roughness.y * material.metalness_factor;
    if (g.fc.render_override_flags & KJB_OVERRIDE_NO_METAL) metalness = 0;
    const float rs = g.fc.render_override_material_roughness_scale;
    if (rs <= 1) roughness *= rs; else roughness = square(kjb_lerp(kjb_sqrt(roughness), 1.0f, 1.0f - 1.0f / rs));

    float3 emissive = f3(0.0f);
    if (0 == path_length || 0 == (material.flags & 1u)) {
        emissive = f3(1.0f) * xyz(sample_map(material.maps[3], 3))
            * f3(material.emissive[0], material.emissive[1], material.emissive[2]) * inst.emissive_multiplier * g.fc.pre_exposure;
    }
    GbufferData gb;
    gb.albedo = albedo;
    gb.normal = normalize(xform_dir(o2w, normal));
    gb.roughness = roughness; gb.metalness = metalness; gb.emissive = emissive;
    if (dot(ray.dir, gb.normal) > 0) gb.normal = gb.normal * -1.0f;
    if (geometric_normal_ws_out) *geometric_normal_ws_out = surf_normal_ws;
    return gbuffer_pack(gb);
}

struct GbufferPathVertex { bool is_hit; uint4 gbuffer_packed; float3 position; float ray_t; };
KJB_DEV GbufferPathVertex gbuffer_raytrace(const Globals& g, const Ray& ray, RayCone cone, uint32_t path_length, bool cull_back_faces) {
    count_ray(g.scene, 0);
    const HitInfo h = trace<false>(g.scene, ray, cull_back_faces);
    GbufferPathVertex r;
    if (h.hit) {
        r.is_hit = true; r.position = ray.origin + ray.dir * h.t; r.gbuffer_packed = rchit_gbuffer(g, ray, h, cone, path_length); r.ray_t = h.t;
    } else { r.is_hit = false; r.ray_t = KJB_FLT_MAX; r.gbuffer_packed = u4(0, 0, 0, 0); r.position = f3(0.0f); }
    return r;
}
KJB_DEV bool rt_is_shadowed(const Globals& g, float3 origin, float3 dir, float tmin, float tmax) {
    count_ray(g.scene, 1);
    Ray r; r.origin = origin; r.dir = dir; r.tmin = tmin; r.tmax = tmax;
    return trace<true>(g.scene, r, false).hit;
}

}  // namespace kjb
