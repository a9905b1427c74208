// ORACLE — TEST INFRASTRUCTURE ONLY (see kj_math.h header).
// Scene store + software ray tracing + the closest-hit "G-buffer" shader.
//
// The reference has NO BVH/intersection code (it calls VK_KHR_ray_tracing_pipeline;
// crates/lib/kajiya-backend/src/vulkan/ray_tracing.rs:96-260, inc/rt.hlsl:58-70,112-137), so the
// intersection CONTRACT is ours (DESIGN.md "ray/triangle contract") — PARITY UNPINNED for traversal:
//   * triangles are intersected in WORLD space: each vertex is transformed by the instance's 3x4
//     object-to-world matrix in fp32 (x' = m0*x + m1*y + m2*z + m3, left to right);
//   * Moeller-Trumbore in the written operation order below; a hit needs tmin < t < tmax;
//   * closest hit = smallest t, ties broken by the smallest global triangle id
//     (instance-major, then PrimitiveIndex) => independent of BVH topology;
//   * any-hit (shadow) = existence of a hit, also topology independent.
// The oracle's own BVH (median split) is validated against brute force in tests/test_oracle_bvh.py.
//
// Restates: rt/gbuffer.rchit.hlsl:46-202 (S1), inc/rt.hlsl (payloads, GbufferRaytrace), inc/mesh.hlsl.
#pragma once
#include "kj_shading.h"
#include <algorithm>
#include <atomic>

namespace kjo {

struct Texture {
    uint32_t width, height, mip_count, srgb;
    std::vector<std::vector<uint8_t>> mips;   // RGBA8 per mip
};

struct Ray { float3 origin, dir; float tmin, tmax; };

struct WorldTri { float3 v0, e1, e2; uint32_t instance, prim; };

struct BvhNode { float3 bmin, bmax; int left, right, first, count; };   // leaf if count > 0

struct Scene {
    std::vector<uint8_t> vertices;                 // kajiya's unified ByteAddressBuffer (world_renderer.rs:657-672)
    std::vector<kjb_gpu_mesh> meshes;
    std::vector<uint32_t> mesh_index_counts;
    std::vector<Texture> textures;
    std::vector<kjb_instance> instances;
    std::vector<WorldTri> tris;                    // world space, global id = index
    std::vector<BvhNode> nodes;
    std::vector<uint32_t> tri_order;               // leaf order -> global triangle id
    mutable std::atomic<uint64_t> n_closest{0}, n_any{0};

    uint32_t load_u32(uint32_t off) const { uint32_t v; memcpy(&v, &vertices[off], 4); return v; }
    float load_f32(uint32_t off) const { float v; memcpy(&v, &vertices[off], 4); return v; }
    float3 load_f3(uint32_t off) const { return float3(load_f32(off), load_f32(off + 4), load_f32(off + 8)); }

    static float3 xform_point(const float* m, float3 p) {
        return float3(m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3], m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7],
                      m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11]);
    }
    static float3 xform_dir(const float* m, float3 p) {
        return float3(m[0] * p.x + m[1] * p.y + m[2] * p.z, m[4] * p.x + m[5] * p.y + m[6] * p.z, m[8] * p.x + m[9] * p.y + m[10] * p.z);
    }

    void rebuild_tlas(const kjb_instance* inst, uint32_t n) {
        instances.assign(inst, inst + n);
        tris.clear();
        for (uint32_t i = 0; i < n; ++i) {
            const kjb_gpu_mesh& m = meshes[inst[i].mesh_index];
            const uint32_t ntri = mesh_index_counts[inst[i].mesh_index] / 3;
            for (uint32_t p = 0; p < ntri; ++p) {
                uint32_t i0 = load_u32(m.index_offset + (p * 3 + 0) * 4), i1 = load_u32(m.index_offset + (p * 3 + 1) * 4), i2 = load_u32(m.index_offset + (p * 3 + 2) * 4);
                float3 a = xform_point(inst[i].transform, load_f3(m.vertex_core_offset + i0 * 16));
                float3 b = xform_point(inst[i].transform, load_f3(m.vertex_core_offset + i1 * 16));
                float3 c = xform_point(inst[i].transform, load_f3(m.vertex_core_offset + i2 * 16));
                WorldTri t; t.v0 = a; t.e1 = b - a; t.e2 = c - a; t.instance = i; t.prim = p;
                tris.push_back(t);
            }
        }
        build_bvh();
    }

    // ---- median-split BVH (oracle-only; product uses its own SAH builder)
    void build_bvh() {
        nodes.clear(); tri_order.resize(tris.size());
        for (size_t i = 0; i < tris.size(); ++i) tri_order[i] = uint32_t(i);
        if (tris.empty()) return;
        nodes.reserve(tris.size() * 2);
        build_rec(0, int(tris.size()));
    }
    void tri_bounds(uint32_t id, float3& lo, float3& hi) const {
        const WorldTri& t = tris[id];
        float3 a = t.v0, b = t.v0 + t.e1, c = t.v0 + t.e2;
        lo = min(a, min(b, c)); hi = max(a, max(b, c));
    }
    int build_rec(int first, int count) {
        int idx = int(nodes.size()); nodes.push_back(BvhNode());
        float3 lo(FLT_MAX_F), hi(-FLT_MAX_F), clo(FLT_MAX_F), chi(-FLT_MAX_F);
        for (int i = first; i < first + count; ++i) {
            float3 a, b; tri_bounds(tri_order[i], a, b);
            lo = min(lo, a); hi = max(hi, b);
            float3 c = (a + b) * 0.5f; clo = min(clo, c); chi = max(chi, c);
        }
        // pad the box a little against the slab test's rounding (the product's padding: the |b| term keeps the pad above one ulp of the
        // box's own coordinates, so a flat box far from the origin stays a slab of non-zero width)
        float3 pad = (hi - lo) * 1e-5f + float3(1e-6f) + max(abs(lo), abs(hi)) * 1e-6f;
        nodes[idx].bmin = lo - pad; nodes[idx].bmax = hi + pad;
        if (count <= 4) { nodes[idx].first = first; nodes[idx].count = count; nodes[idx].left = nodes[idx].right = -1; return idx; }
        float3 ext = chi - clo;
        int axis = ext.x >= ext.y && ext.x >= ext.z ? 0 : (ext.y >= ext.z ? 1 : 2);
        int mid = first + count / 2;
        std::nth_element(tri_order.begin() + first, tri_order.begin() + mid, tri_order.begin() + first + count,
            [&](uint32_t a, uint32_t b) { float3 al, ah, bl, bh; tri_bounds(a, al, ah); tri_bounds(b, bl, bh); return (al[axis] + ah[axis]) < (bl[axis] + bh[axis]); });
        nodes[idx].count = 0; nodes[idx].first = 0;
        int l = build_rec(first, mid - first);
        int r = build_rec(mid, first + count - mid);
        nodes[idx].left = l; nodes[idx].right = r;
        return idx;
    }

    // ---- the ray/triangle contract
    static bool intersect_tri(const WorldTri& tr, const Ray& r, float tmax, bool cull_back, float& t_out, float& u_out, float& v_out) {
        const float3 p = cross(r.dir, tr.e2);
        const float det = dot(tr.e1, p);
        if (det == 0.0f) return false;
        if (cull_back && det < 0.0f) return false;     // RAY_FLAG_CULL_BACK_FACING_TRIANGLES (clockwise-front convention, see DESIGN.md)
        const float inv = 1.0f / det;
        const float3 tv = r.origin - tr.v0;
        const float u = dot(tv, p) * inv;
        if (u < 0.0f || u > 1.0f) return false;
        const float3 q = cross(tv, tr.e1);
        const float v = dot(r.dir, q) * inv;
        if (v < 0.0f || u + v > 1.0f) return false;
        const float t = dot(tr.e2, q) * inv;
        if (!(t > r.tmin && t < tmax)) return false;
        t_out = t; u_out = u; v_out = v;
        return true;
    }
    static bool ray_has_nan(const Ray& r) {
        return !(r.dir.x == r.dir.x && r.dir.y == r.dir.y && r.dir.z == r.dir.z && r.origin.x == r.origin.x && r.origin.y == r.origin.y && r.origin.z == r.origin.z && r.tmin == r.tmin && r.tmax == r.tmax);
    }
    // The culling slack of the product's walk (kajiya_b200/csrc/kjb_trace.cuh, where its error bound is written out): the interval is
    // widened by s = k * 2^-24 relative, so neither the slab's rounding nor the Moeller-Trumbore t of a triangle on its box's face can cull it.
    static constexpr float SLAB_SLACK = 16384.0f * 0x1p-24f;
    static bool slab(const BvhNode& n, const Ray& r, float3 inv_dir, float tmax) {
        float3 t0 = (n.bmin - r.origin) * inv_dir, t1 = (n.bmax - r.origin) * inv_dir;
        // a ray lying in a box plane (0 * inf = NaN, dropped by min/max) culls the box: the padding keeps every triangle strictly inside
        float3 a = min(t0, t1), b = max(t0, t1);
        float tn = max(max(a.x, a.y), max(a.z, r.tmin)), tf = min(min(b.x, b.y), min(b.z, tmax));
        tn = kjb_fma(-SLAB_SLACK, abs(tn), tn); tf = kjb_fma(SLAB_SLACK, abs(tf), tf);
        return tn <= tf;
    }
    struct HitInfo { bool hit; float t, u, v; uint32_t tri; };
    HitInfo closest(const Ray& r, bool cull_back) const {
        n_closest++;
        HitInfo h; h.hit = false; h.t = r.tmax; h.tri = 0xffffffffu; h.u = h.v = 0;
        if (nodes.empty() || ray_has_nan(r)) return h;   // a NaN ray cannot pass the triangle test; skip the (NaN-ignoring) slab walk
        float3 inv_dir = 1.0f / r.dir;
        int stack[64]; int sp = 0; stack[sp++] = 0;
        while (sp) {
            const BvhNode& n = nodes[stack[--sp]];
            if (!slab(n, r, inv_dir, h.t)) continue;
            if (n.count > 0) {
                for (int i = n.first; i < n.first + n.count; ++i) {
                    uint32_t id = tri_order[i]; float t, u, v;
                    // tmax for the test is the ORIGINAL tmax so that ties are seen; selection rule below
                    if (intersect_tri(tris[id], r, r.tmax, cull_back, t, u, v)) {
                        if (!h.hit || t < h.t || (t == h.t && id < h.tri)) { h.hit = true; h.t = t; h.u = u; h.v = v; h.tri = id; }
                    }
                }
            } else { stack[sp++] = n.left; stack[sp++] = n.right; }
        }
        return h;
    }
    HitInfo closest_brute(const Ray& r, bool cull_back) const {
        HitInfo h; h.hit = false; h.t = r.tmax; h.tri = 0xffffffffu; h.u = h.v = 0;
        for (uint32_t id = 0; id < tris.size(); ++id) { float t, u, v;
            if (intersect_tri(tris[id], r, r.tmax, cull_back, t, u, v)) if (!h.hit || t < h.t || (t == h.t && id < h.tri)) { h.hit = true; h.t = t; h.u = u; h.v = v; h.tri = id; } }
        return h;
    }
    bool any_hit(const Ray& r, bool cull_back = false) const {
        n_any++;
        if (nodes.empty() || ray_has_nan(r)) return false;
        float3 inv_dir = 1.0f / r.dir;
        int stack[64]; int sp = 0; stack[sp++] = 0;
        while (sp) {
            const BvhNode& n = nodes[stack[--sp]];
            if (!slab(n, r, inv_dir, r.tmax)) continue;
            if (n.count > 0) {
                for (int i = n.first; i < n.first + n.count; ++i) { float t, u, v; if (intersect_tri(tris[tri_order[i]], r, r.tmax, cull_back, t, u, v)) return true; }
            } else { stack[sp++] = n.left; stack[sp++] = n.right; }
        }
        return false;
    }

    // ---- bindless texture SampleLevel(sampler_llr, uv, lod): trilinear, repeat
    float4 texel(const Texture& tx, int mip, int x, int y) const {
        int w = std::max(1u, tx.width >> mip), h = std::max(1u, tx.height >> mip);
        x = ((x % w) + w) % w; y = ((y % h) + h) % h;
        const uint8_t* p = &tx.mips[mip][(size_t(y) * w + x) * 4];
        float4 c(p[0] / 255.0f, p[1] / 255.0f, p[2] / 255.0f, p[3] / 255.0f);
        if (tx.srgb) { auto eotf = [](float a) { return .04045f < a ? pow((a + .055f) / 1.055f, 2.4f) : a / 12.92f; };   // color/srgb.hlsl:37-39
            c.x = eotf(c.x); c.y = eotf(c.y); c.z = eotf(c.z); }
        return c;
    }
    float4 sample_bilinear_repeat(const Texture& tx, int mip, float2 uv) const {
        int w = std::max(1u, tx.width >> mip), h = std::max(1u, tx.height >> mip);
        float fx = uv.x * float(w) - 0.5f, fy = uv.y * float(h) - 0.5f;
        float x0f = floor(fx), y0f = floor(fy); float tx_ = fx - x0f, ty = fy - y0f;
        int x0 = int(x0f), y0 = int(y0f);
        float4 a = texel(tx, mip, x0, y0), b = texel(tx, mip, x0 + 1, y0), c = texel(tx, mip, x0, y0 + 1), d = texel(tx, mip, x0 + 1, y0 + 1);
        float4 top = a + (b - a) * tx_, bot = c + (d - c) * tx_;
        return top + (bot - top) * ty;
    }
    float4 sample_level(uint32_t tex_idx, float2 uv, float lod) const {
        if (tex_idx >= textures.size()) return float4(1.0f);
        const Texture& tx = textures[tex_idx];
        float maxl = float(tx.mip_count - 1);
        if (!(lod > 0.0f)) lod = 0.0f;      // also catches NaN / -inf (zero uv area)
        if (lod > maxl) lod = maxl;
        int l0 = int(floor(lod)); float f = lod - float(l0);
        float4 a = sample_bilinear_repeat(tx, l0, uv);
        if (f == 0.0f || l0 + 1 >= int(tx.mip_count)) return a;
        float4 b = sample_bilinear_repeat(tx, l0 + 1, uv);
        return a + (b - a) * f;
    }
    float2 texture_size(uint32_t tex_idx) const { if (tex_idx >= textures.size()) return float2(1.0f); return float2(float(textures[tex_idx].width), float(textures[tex_idx].height)); }
};

// ---------------------------------------------------------------- rt/gbuffer.rchit.hlsl
inline float3 unpack_unit_direction_11_10_11(uint pck) {   // mesh.hlsl:26-32
    return float3(float(pck & ((1u << 11u) - 1u)) * (2.0f / float((1u << 11u) - 1u)) - 1.0f,
                  float((pck >> 11u) & ((1u << 10u) - 1u)) * (2.0f / float((1u << 10u) - 1u)) - 1.0f,
                  float((pck >> 21u)) * (2.0f / float((1u << 11u) - 1u)) - 1.0f);
}
inline float2 transform_material_uv(const kjb_mesh_material& mat, float2 uv, uint map_idx) {   // mesh.hlsl:63-68
    uint xo = map_idx * 6;
    const float* t = mat.map_transforms;
    return float2(t[xo + 0] * uv.x + t[xo + 1] * uv.y, t[xo + 2] * uv.x + t[xo + 3] * uv.y) + float2(t[xo + 4], t[xo + 5]);
}
inline float compute_texture_lod(const Scene& sc, uint tex, float triangle_constant, float3 ray_direction, float3 surf_normal, float cone_width) {   // :29-44
    float2 wh = sc.texture_size(tex);
    float lambda = triangle_constant;
    lambda += log2(abs(cone_width));
    lambda += 0.5f * log2(wh.x * wh.y);
    lambda -= log2(abs(dot(normalize(ray_direction), surf_normal)));
    return lambda;
}

// closest-hit shader: returns the packed 16-byte G-buffer payload (gbuffer.rchit.hlsl:46-202)
inline uint4 rchit_gbuffer(const Scene& sc, const Globals& g, const Ray& ray, const Scene::HitInfo& hit, const RayCone& ray_cone, uint path_length) {
    const WorldTri& wt = sc.tris[hit.tri];
    const kjb_instance& inst = sc.instances[wt.instance];
    const kjb_gpu_mesh& mesh = sc.meshes[inst.mesh_index];
    const float* o2w = inst.transform;
    const float ray_t = hit.t;
    float3 hit_point = ray.origin + ray.dir * ray_t;
    const float hit_dist = length(hit_point - ray.origin);
    float3 bary(1.0f - hit.u - hit.v, hit.u, hit.v);

    uint ind[3] = { sc.load_u32(mesh.index_offset + (wt.prim * 3 + 0) * 4), sc.load_u32(mesh.index_offset + (wt.prim * 3 + 1) * 4), sc.load_u32(mesh.index_offset + (wt.prim * 3 + 2) * 4) };
    float3 vp[3], vn[3];
    for (int k = 0; k < 3; ++k) { vp[k] = sc.load_f3(mesh.vertex_core_offset + ind[k] * 16); vn[k] = unpack_unit_direction_11_10_11(sc.load_u32(mesh.vertex_core_offset + ind[k] * 16 + 12)); }
    float3 normal = vn[0] * bary.x + vn[1] * bary.y + vn[2] * bary.z;
    const float3 surf_normal_os = normalize(cross(vp[1] - vp[0], vp[2] - vp[0]));
    const float3 surf_normal_ws = normalize(Scene::xform_dir(o2w, surf_normal_os));
    if (g.fc.render_override_flags & KJB_OVERRIDE_FORCE_FACE_NORMALS) normal = surf_normal_os;

    float4 v_color(1.0f);
    if (mesh.vertex_aux_offset != 0) {
        float4 vc[3];
        for (int k = 0; k < 3; ++k) { uint o = mesh.vertex_aux_offset + ind[k] * 16; vc[k] = float4(sc.load_f32(o), sc.load_f32(o + 4), sc.load_f32(o + 8), sc.load_f32(o + 12)); }
        v_color = vc[0] * bary.x + vc[1] * bary.y + vc[2] * bary.z;
    }
    float2 uvs[3];
    for (int k = 0; k < 3; ++k) { uint o = mesh.vertex_uv_offset + ind[k] * 8; uvs[k] = float2(sc.load_f32(o), sc.load_f32(o + 4)); }
    float2 uv = uvs[0] * bary.x + uvs[1] * bary.y + uvs[2] * bary.z;

    const float cone_width = ray_cone.width_at_t(hit_dist);
    const float3 p0 = Scene::xform_point(o2w, vp[0]), p1 = Scene::xform_point(o2w, vp[1]), p2 = Scene::xform_point(o2w, vp[2]);
    const float twice_uv_area = abs((uvs[1].x - uvs[0].x) * (uvs[2].y - uvs[0].y) - (uvs[2].x - uvs[0].x) * (uvs[1].y - uvs[0].y));
    const float twice_triangle_area = length(cross(p1 - p0, p2 - p0));
    const float lod_triangle_constant = 0.5f * log2(twice_uv_area / twice_triangle_area);

    uint material_id = sc.load_u32(mesh.vertex_mat_offset + ind[0] * 4);
    kjb_mesh_material material; memcpy(&material, &sc.vertices[mesh.mat_data_offset + material_id * sizeof(kjb_mesh_material)], sizeof(material));

    float2 albedo_uv = transform_material_uv(material, uv, 0);
    float albedo_lod = compute_texture_lod(sc, material.maps[2], lod_triangle_constant, ray.dir, surf_normal_ws, cone_width);
    float3 albedo = sc.sample_level(material.maps[2], albedo_uv, albedo_lod).xyz()
        * float3(material.base_color_mult[0], material.base_color_mult[1], material.base_color_mult[2]) * v_color.xyz();

    float2 spec_uv = transform_material_uv(material, uv, 2);
    float spec_lod = compute_texture_lod(sc, material.maps[1], lod_triangle_constant, ray.dir, surf_normal_ws, cone_width);
    float4 metalness_roughness = sc.sample_level(material.maps[1], spec_uv, spec_lod);
    float perceptual_roughness = material.roughness_mult * metalness_roughness.x;
    float roughness = clamp(perceptual_roughness_to_roughness(perceptual_roughness), 1e-4f, 1.0f);
    float metalness = metalness_roughness.y * material.metalness_factor;
    if (g.fc.render_override_flags & KJB_OVERRIDE_NO_METAL) metalness = 0;
    const float rs = g.fc.render_override_material_roughness_scale;
    if (rs <= 1) roughness *= rs; else roughness = square(lerp(sqrt(roughness), 1.0f, 1.0f - 1.0f / rs));

    float2 emissive_uv = transform_material_uv(material, uv, 3);
    float emissive_lod = compute_texture_lod(sc, material.maps[3], lod_triangle_constant, ray.dir, surf_normal_ws, cone_width);
    float3 emissive(0.0f);
    if (0 == path_length || 0 == (material.flags & 1u)) {
        emissive = float3(1.0f) * sc.sample_level(material.maps[3], emissive_uv, emissive_lod).xyz()
            * float3(material.emissive[0], material.emissive[1], material.emissive[2]) * inst.emissive_multiplier * g.fc.pre_exposure;
    }
    GbufferData gb;
    gb.albedo = albedo;
    gb.normal = normalize(Scene::xform_dir(o2w, normal));
    gb.roughness = roughness; gb.metalness = metalness; gb.emissive = emissive;
    if (dot(ray.dir, gb.normal) > 0) gb.normal = gb.normal * -1.0f;   // force double-sided (:194-197)
    return gbuffer_pack(gb);
}

// inc/rt.hlsl:72-137
struct GbufferPathVertex { bool is_hit; uint4 gbuffer_packed; float3 position; float ray_t; };
inline GbufferPathVertex gbuffer_raytrace(const Scene& sc, const Globals& g, const Ray& ray, const RayCone& cone, uint path_length, bool cull_back_faces) {
    Scene::HitInfo h = sc.closest(ray, cull_back_faces);
    GbufferPathVertex res;
    if (h.hit) {
        res.is_hit = true;
        res.position = ray.origin + ray.dir * h.t;
        res.gbuffer_packed = rchit_gbuffer(sc, g, ray, h, cone, path_length);
        res.ray_t = h.t;
    } else { res.is_hit = false; res.ray_t = FLT_MAX_F; res.gbuffer_packed = uint4(0, 0, 0, 0); }
    return res;
}
inline bool rt_is_shadowed(const Scene& sc, float3 origin, float3 dir, float tmin, float tmax) {   // inc/rt.hlsl:58-70
    Ray r; r.origin = origin; r.dir = dir; r.tmin = tmin; r.tmax = tmax;
    return sc.any_hit(r);
}

}  // namespace kjo
