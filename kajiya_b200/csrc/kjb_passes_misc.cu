// Input producers and utility passes as sm_90a kernels (one thread per texel, 32x8 blocks => each warp touches one
// contiguous row segment: 128..512 B per request depending on the texel size).
#include "kjb_context.h"

using namespace kjb;

// ------------------------------------------------------------------ primary-visibility G-buffer by ray casting
// (stand-in for raster_simple_ps.hlsl:39-140; hit shading = rt/gbuffer.rchit.hlsl)
KJB_KERNEL(128) k_raster_gbuffer(const __grid_constant__ Globals g, ImgW gn, ImgW gb, ImgW dp, ImgW vel, const kjb_instance* prev_instances, uint32_t prev_instance_count, Rows kjb_rows) {
    KJB_PX; if (x >= gb.w || y >= gb.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float size[4] = {float(gb.w), float(gb.h), 1.0f / float(gb.w), 1.0f / float(gb.h)};
    const float2 uv = get_uv(x, y, size);
    const ViewRayContext vrc = ViewRayContext::from_uv(vc, uv);
    Ray r; r.origin = vrc.ray_origin_ws(); r.dir = vrc.ray_dir_ws(); r.tmin = 0; r.tmax = KJB_FLT_MAX;
    count_ray(g.scene, 0);
    const HitInfo h = trace<false>(g.scene, r, false);
    if (!h.hit) {
        st_raw<uint32_t>(gn, x, y, 0u); st_rgba32u(gb, x, y, u4(0, 0, 0, 0)); st_r32f(dp, x, y, 0.0f); st_rgba16f(vel, x, y, f4(0.0f));
        return;
    }
    RayCone cone; cone.width = 0; cone.spread_angle = pixel_cone_spread_angle_from_image_height(vc, float(gb.h));
    float3 surf_n_unused;
    const uint4 packed = rchit_gbuffer(g, r, h, cone, 0, &surf_n_unused);
    const float3 pos_ws = r.origin + r.dir * h.t;
    const float3 pos_cs = position_world_to_clip(vc, pos_ws);
    // geometric normal from the world-space triangle the contract intersected
    float3 e1, e2, prev_pos_ws = pos_ws;
    {   // find the leaf record again through the global id: tri_info -> instance/prim -> vertices (cheap: once per pixel)
        const TriInfo ti = g.scene.tri_info[h.gid];
        const kjb_instance& inst = g.scene.instances[ti.instance];
        const kjb_gpu_mesh mesh = g.scene.meshes[inst.mesh_index];
        float3 p[3], po[3];
        for (int k = 0; k < 3; ++k) {
            const uint32_t idx = vb_u32(g.scene, mesh.index_offset + (ti.prim * 3 + k) * 4);
            const float4 v = *reinterpret_cast<const float4*>(g.scene.vertices + mesh.vertex_core_offset + idx * 16);
            po[k] = f3(v.x, v.y, v.z);
            p[k] = xform_point(inst.transform, po[k]);
        }
        e1 = p[1] - p[0]; e2 = p[2] - p[0];
        if (prev_instances && ti.instance < prev_instance_count)   // object motion: the same surface point under last frame's transform
            prev_pos_ws = xform_point(prev_instances[ti.instance].transform, po[0] * (1.0f - h.u - h.v) + po[1] * h.u + po[2] * h.v);
    }
    float3 gnorm_ws = normalize(cross(e1, e2));
    if (dot(gnorm_ws, r.dir) > 0) gnorm_ws = -gnorm_ws;
    const float3 gnorm_vs = normalize(direction_world_to_view(vc, gnorm_ws));
    const float3 vs_pos = xyz(mul(vc.world_to_view, f4(pos_ws, 1)));
    const float3 prev_vs_pos = xyz(mul(vc.prev_world_to_prev_view, f4(prev_pos_ws, 1)));
    st_a2r10g10b10(gn, x, y, gnorm_vs * 0.5f + 0.5f);
    st_rgba32u(gb, x, y, packed);
    st_r32f(dp, x, y, pos_cs.z);
    st_rgba16f(vel, x, y, f4(prev_vs_pos - vs_pos, 0));
}

// ------------------------------------------------------------------ calculate_reprojection_map.hlsl:17-142
KJB_KERNEL(256) k_reprojection_map(const __grid_constant__ Globals g, Img depth_tex, Img geometric_normal_tex, Img prev_depth_tex, Img velocity_tex, ImgW output_tex, float4 output_tex_size, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float ots[4] = {output_tex_size.x, output_tex_size.y, output_tex_size.z, output_tex_size.w};
    const float2 uv = get_uv(x, y, ots);
    const float d0 = ld_r32f(depth_tex, x, y);
    if (d0 == 0.0f) {
        const float2 cs = uv_to_cs(uv);
        const float4 pos_vs = mul(vc.clip_to_view, f4(cs.x, cs.y, 0.0f, 1.0f));
        const float4 prev_pcs = mul(vc.clip_to_prev_clip, mul(vc.view_to_clip, pos_vs));
        const float2 uv_diff = cs_to_uv(xy(prev_pcs)) - uv;
        st_rgba16s(output_tex, x, y, f4(uv_diff.x, uv_diff.y, 0, 0));
        return;
    }
    float depth = 0.0f;
    if (d0 != 0.0f) depth = kjb_max(depth, d0);
    const float3 normal_vs = ld_a2r10g10b10(geometric_normal_tex, x, y) * 2.0f - 1.0f;
    const float3 normal_pvs = xyz(mul(vc.prev_clip_to_prev_view, mul(vc.clip_to_prev_clip, mul(vc.view_to_clip, f4(normal_vs, 0)))));
    const float2 cs = uv_to_cs(uv);
    const float4 pos_vs = mul(vc.clip_to_view, f4(cs.x, cs.y, depth, 1.0f));
    const float dist_to_point = -(pos_vs.z / pos_vs.w);
    float4 prev_vs = pos_vs / pos_vs.w;
    const float4 v = ld_rgba16f(velocity_tex, x, y);
    prev_vs.x += v.x; prev_vs.y += v.y; prev_vs.z += v.z;
    const float4 prev_pcs = mul(vc.clip_to_prev_clip, mul(vc.view_to_clip, prev_vs));
    float2 prev_uv = cs_to_uv(xy(prev_pcs) / prev_pcs.w);
    float2 uv_diff = prev_uv - uv;
    uv_diff = vfloor(uv_diff * 32767.0f + 0.5f) / 32767.0f;
    prev_uv = uv + uv_diff;
    float4 prev_pvs = mul(vc.prev_clip_to_prev_view, prev_pcs);
    prev_pvs = prev_pvs / prev_pvs.w;
    const float plane_dist_prev_dz = kjb_min(-0.2f, normal_vs.z);
    // get_bilinear_filter + GatherRed(...).wzxy at the quad whose top-left texel is `origin`
    const float2 bp = prev_uv * f2(output_tex_size.x, output_tex_size.y) - 0.5f;
    const int ox = kjb_cvt_i32(kjb_trunc(bp.x)), oy = kjb_cvt_i32(kjb_trunc(bp.y));
    const int W = output_tex.w, H = output_tex.h;
    const float4 prev_depth = f4(ld_r32f(prev_depth_tex, clampi(ox, W), clampi(oy, H)), ld_r32f(prev_depth_tex, clampi(ox + 1, W), clampi(oy, H)),
                                 ld_r32f(prev_depth_tex, clampi(ox, W), clampi(oy + 1, H)), ld_r32f(prev_depth_tex, clampi(ox + 1, W), clampi(oy + 1, H)));
    const float k43 = -vc.prev_clip_to_prev_view.m[2 * 4 + 3];
    const float4 prev_view_z = f4(kjb_rcp(prev_depth.x * k43), kjb_rcp(prev_depth.y * k43), kjb_rcp(prev_depth.z * k43), kjb_rcp(prev_depth.w * k43));
    const float4 quad_dists = vabs(plane_dist_prev_dz * (prev_view_z - prev_pvs.z));
    const float acceptance_threshold = 0.001f * (1080.0f / output_tex_size.y);
    const float3 pos_vs_norm = normalize(xyz(pos_vs) / pos_vs.w);
    const float ndotv = dot(normal_vs, pos_vs_norm);
    const float prev_ndotv = dot(normal_pvs, normalize(xyz(prev_pvs)));
    const float thr = acceptance_threshold * dist_to_point / -ndotv;
    float4 qv = f4(kjb_step(quad_dists.x, thr), kjb_step(quad_dists.y, thr), kjb_step(quad_dists.z, thr), kjb_step(quad_dists.w, thr));
    const int LW = int(kjb_cvt_u32(output_tex_size.x)), LH = int(kjb_cvt_u32(output_tex_size.y));
    qv.x *= (ox >= 0 && oy >= 0 && ox < LW && oy < LH) ? 1.0f : 0.0f;
    qv.y *= (ox + 1 >= 0 && oy >= 0 && ox + 1 < LW && oy < LH) ? 1.0f : 0.0f;
    qv.z *= (ox >= 0 && oy + 1 >= 0 && ox < LW && oy + 1 < LH) ? 1.0f : 0.0f;
    qv.w *= (ox + 1 >= 0 && oy + 1 >= 0 && ox + 1 < LW && oy + 1 < LH) ? 1.0f : 0.0f;
    const float validity = dot(qv, f4(1, 2, 4, 8)) / 15.0f;
    float accuracy = 1;
    accuracy *= kjb_smoothstep(0.8f, 0.95f, prev_ndotv / ndotv);
    const float2 sat = vsaturate(prev_uv);
    if (sat.x != prev_uv.x || sat.y != prev_uv.y) accuracy = -1;
    st_rgba16s(output_tex, x, y, f4(uv_diff.x, uv_diff.y, validity, accuracy));
}

// ------------------------------------------------------------------ sky/comp_cube.hlsl, convolve_cube.hlsl (inc/cube_map.hlsl rotations)
KJB_DEV float3 cube_dir(int face, float2 uv) {
    const float3 v = f3(uv.x * 2 - 1, uv.y * 2 - 1, -1.0f);
    float3 d;
    switch (face) {
        case 0: d = f3(-v.z, -v.y, -v.x); break;     // (0,0,-1; 0,-1,0; -1,0,0)
        case 1: d = f3(v.z, -v.y, v.x); break;       // (0,0,1; 0,-1,0; 1,0,0)
        case 2: d = f3(v.x, -v.z, v.y); break;       // (1,0,0; 0,0,-1; 0,1,0)
        case 3: d = f3(v.x, v.z, -v.y); break;       // (1,0,0; 0,0,1; 0,-1,0)
        case 4: d = f3(v.x, -v.y, -v.z); break;      // (1,0,0; 0,-1,0; 0,0,-1)
        default: d = f3(-v.x, -v.y, v.z); break;     // (-1,0,0; 0,-1,0; 0,0,1)
    }
    return normalize(d);
}
KJB_KERNEL(64) k_sky_cube(const __grid_constant__ Globals g, ImgW out, Rows kjb_rows) {
    KJB_PX; const int face = int(blockIdx.z); if (x >= out.w || y >= out.h) return;
    const float2 uv = (f2(float(x), float(y)) + 0.5f) / 64.0f;
    const float3 dir = cube_dir(face, uv);
    st_rgba16f(out, x, y, f4(atmosphere_default(g.fc, dir, sun_direction(g.fc)), 1), face);
}
KJB_KERNEL(64) k_convolve_sky(Img in, ImgW out, uint32_t face_width, Rows kjb_rows) {
    KJB_PX; const int face = int(blockIdx.z); if (x >= out.w || y >= out.h) return;
    const float2 uv = (f2(float(x), float(y)) + 0.5f) / float(face_width);
    const float3 output_dir = cube_dir(face, uv);
    const float3x3 basis = build_orthonormal_basis(output_dir);
    float4 result = f4(0.0f);
    for (uint32_t i = 0; i < 512u; ++i) {
        const float3 input_dir = mul(basis, uniform_sample_cone(hammersley(i, 512u), 0.99f));
        result += sample_cube_rgba16f(in, input_dir);
    }
    st_rgba16f(out, x, y, result / 512.0f, face);
}

// ------------------------------------------------------------------ lut/brdf_fg.hlsl:6-45
KJB_KERNEL(64) k_brdf_fg_lut(ImgW out, Rows kjb_rows) {
    KJB_PX; if (x >= 64 || y >= 64) return;
    const float ndotv = (float(x) / (64.0f - 1.0f)) * (1.0f - 1e-3f) + 1e-3f;
    const float roughness = kjb_max(1e-5f, float(y) / (64.0f - 1.0f));
    const float3 wo = f3(kjb_sqrt(1.0f - ndotv * ndotv), 0, ndotv);
    float a = 0, b = 0, valid = 0;
    SpecularBrdf brdf_a; brdf_a.roughness = roughness; brdf_a.albedo = f3(1.0f);
    SpecularBrdf brdf_b = brdf_a; brdf_b.albedo = f3(0.0f);
    for (uint32_t i = 0; i < 1024u; ++i) {
        const BrdfSample v_a = specular_sample(brdf_a, wo, hammersley(i, 1024u));
        if (v_a.wi.z > 1e-6f) {
            const BrdfValue v_b = specular_evaluate(brdf_b, wo, v_a.wi);
            a += (v_a.value_over_pdf.x - v_b.value_over_pdf.x);
            b += v_b.value_over_pdf.x;
            valid += 1;
        }
    }
    st_rgba16f(out, x, y, f4(f3(a, b, valid) / 1024.0f, 1.0f));
}

// ------------------------------------------------------------------ extract_half_res_*.hlsl
KJB_KERNEL(256) k_extract_half_depth(Img in, ImgW out, int2 off, Rows kjb_rows) {
    KJB_PX; if (x >= out.w || y >= out.h) return;
    st_r32f(out, x, y, ld_r32f(in, x * 2 + off.x, y * 2 + off.y));
}
KJB_KERNEL(256) k_extract_half_ssao(Img in, ImgW out, int2 off, Rows kjb_rows) {
    KJB_PX; if (x >= out.w || y >= out.h) return;
    st_r8s(out, x, y, ld_r8u(in, x * 2 + off.x, y * 2 + off.y));
}
KJB_KERNEL(256) k_extract_half_view_normal(const __grid_constant__ Globals g, Img in, ImgW out, int2 off, Rows kjb_rows) {
    KJB_PX; if (x >= out.w || y >= out.h) return;
    const uint4 gbt = ld_rgba32u(in, x * 2 + off.x, y * 2 + off.y);
    const float3 normal_ws = unpack_normal_11_10_11_no_normalize(gbt.y);
    const float3 normal_vs = normalize(xyz(mul(g.fc.view_constants.world_to_view, f4(normal_ws, 0))));
    st_rgba8s(out, x, y, f4(normal_vs, 1));
}
KJB_KERNEL(256) k_extract_half_fused(const __grid_constant__ Globals g, Img gbuffer, Img depth, Img ssao, ImgW out_normal, ImgW out_depth, ImgW out_ssao, int with_ssao, int2 off, float4* positions, float4 gts, Rows kjb_rows) {
    KJB_PX; if (x >= out_depth.w || y >= out_depth.h) return;
    const int sx = x * 2 + off.x, sy = y * 2 + off.y;
    const float d = ld_r32f(depth, sx, sy);
    st_r32f(out_depth, x, y, d);
    if (positions) {   // KJB_OPTION_HALF_RES_POSITION_CACHE: the same expression k_half_res_positions evaluates (kjb_passes_rtdgi.cu)
        const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
        positions[y * out_depth.w + x] = f4(hit_ws_from_uv_depth(g.fc.view_constants, get_uv(sx, sy, s4), d), 0.0f);
    }
    const uint4 gbt = ld_rgba32u(gbuffer, sx, sy);
    const float3 normal_ws = unpack_normal_11_10_11_no_normalize(gbt.y);
    const float3 normal_vs = normalize(xyz(mul(g.fc.view_constants.world_to_view, f4(normal_ws, 0))));
    st_rgba8s(out_normal, x, y, f4(normal_vs, 1));
    if (with_ssao) st_r8s(out_ssao, x, y, ld_r8u(ssao, sx, sy));
}

extern "C" {

int kjb_pass_raster_gbuffer(kjb_context* c, const kjb_raster_gbuffer_args* a) {
    const char* P = "raster simple";
    const uint32_t W = a->gbuffer_out.width, H = a->gbuffer_out.height;
    if (!check_img(c, a->gbuffer_out, KJB_FMT_RGBA32_FLOAT, P, "gbuffer_out") || !check_img(c, a->geometric_normal_out, KJB_FMT_A2R10G10B10_UNORM, P, "geometric_normal_out", W, H)
        || !check_img(c, a->depth_out, KJB_FMT_R32_FLOAT, P, "depth_out", W, H) || !check_img(c, a->velocity_out, KJB_FMT_RGBA16_FLOAT, P, "velocity_out", W, H)) return 1;
    const kjb_instance* d_prev = nullptr;
    if (a->prev_instances && a->prev_instance_count) {
        if (c->prev_instances_capacity < a->prev_instance_count) {
            dev_free(c->d_prev_instances); c->d_prev_instances = (kjb_instance*)dev_alloc(sizeof(kjb_instance) * a->prev_instance_count);
            if (!c->d_prev_instances) return c->fail("raster simple: out of memory");
            c->prev_instances_capacity = a->prev_instance_count;
        }
        c->h_prev_instances.assign(a->prev_instances, a->prev_instances + a->prev_instance_count);   // stable host copy for the async upload
        if (dev_h2d(c, c->d_prev_instances, c->h_prev_instances.data(), sizeof(kjb_instance) * a->prev_instance_count)) return c->fail("raster simple: upload failed");
        d_prev = c->d_prev_instances;
    }
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_raster_gbuffer, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, img_rw(a->geometric_normal_out), img_rw(a->gbuffer_out), img_rw(a->depth_out), img_rw(a->velocity_out), d_prev, d_prev ? a->prev_instance_count : 0u);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_reprojection_map(kjb_context* c, const kjb_reprojection_map_args* a) {
    const char* P = "reprojection map";
    const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    if (!check_img(c, a->output_tex, KJB_FMT_RGBA16_SNORM, P, "output_tex") || !check_img(c, a->depth_tex, KJB_FMT_R32_FLOAT, P, "depth_tex", W, H)
        || !check_img(c, a->geometric_normal_tex, KJB_FMT_A2R10G10B10_UNORM, P, "geometric_normal_tex", W, H) || !check_img(c, a->prev_depth_tex, KJB_FMT_R32_FLOAT, P, "prev_depth_tex", W, H)
        || !check_img(c, a->velocity_tex, KJB_FMT_RGBA16_FLOAT, P, "velocity_tex", W, H)) return 1;
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_reprojection_map, KJB_GRID2D(W, H, 32, 8), c->g, img_ro(a->depth_tex), img_ro(a->geometric_normal_tex), img_ro(a->prev_depth_tex), img_ro(a->velocity_tex),
               img_rw(a->output_tex), f4(a->output_tex_size[0], a->output_tex_size[1], a->output_tex_size[2], a->output_tex_size[3]));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_sky_cube(kjb_context* c, const kjb_sky_cube_args* a) {
    if (!check_img(c, a->output_tex, KJB_FMT_RGBA16_FLOAT, "sky cube", "output_tex", 64, 64) || a->output_tex.layers != 6) return c->fail("sky cube: output must be a 64x64x6 RGBA16F cube");
    const kjb::Rows kjb__rows = {0, 1 << 30};
    KJB_LAUNCH(c, k_sky_cube, KJB_DIMS(dim3(8, 8, 6), dim3(8, 8, 1)), c->g, img_rw(a->output_tex));
    KJB_PASS_EPILOGUE(c, "sky cube");
}
int kjb_pass_convolve_sky(kjb_context* c, const kjb_convolve_sky_args* a) {
    if (!check_img(c, a->input_tex, KJB_FMT_RGBA16_FLOAT, "convolve sky", "input_tex") || !check_img(c, a->output_tex, KJB_FMT_RGBA16_FLOAT, "convolve sky", "output_tex")) return 1;
    const uint32_t W = a->output_tex.width;
    const kjb::Rows kjb__rows = {0, 1 << 30};
    KJB_LAUNCH(c, k_convolve_sky, KJB_DIMS(dim3((W + 7) / 8, (W + 7) / 8, 6), dim3(8, 8, 1)), img_ro(a->input_tex), img_rw(a->output_tex), a->face_width);
    KJB_PASS_EPILOGUE(c, "convolve sky");
}
int kjb_pass_brdf_fg_lut(kjb_context* c, const kjb_brdf_fg_lut_args* a) {
    if (!check_img(c, a->output_tex, KJB_FMT_RGBA16_FLOAT, "brdf fg lut", "output_tex", 64, 64)) return 1;
    const kjb::Rows kjb__rows = {0, 1 << 30};
    KJB_LAUNCH(c, k_brdf_fg_lut, KJB_DIMS(dim3(8, 8, 1), dim3(8, 8, 1)), img_rw(a->output_tex));
    KJB_PASS_EPILOGUE(c, "brdf fg lut");
}
int kjb_pass_extract_half_res_depth(kjb_context* c, const kjb_extract_half_res_args* a) {
    c->epoch_a++;   // half_depth changes: the position cache built from it is stale
    if (!check_img(c, a->input_tex, KJB_FMT_R32_FLOAT, "extract half depth", "input_tex") || !check_img(c, a->output_tex, KJB_FMT_R32_FLOAT, "extract half depth", "output_tex")) return 1;
    KJB_ROWS(c, a->output_tex.height);
    KJB_LAUNCH(c, k_extract_half_depth, KJB_GRID2D(a->output_tex.width, a->output_tex.height, 32, 8), img_ro(a->input_tex), img_rw(a->output_tex), halfres_subsample_offset(c->g.fc.frame_index));
    KJB_PASS_EPILOGUE(c, "extract half depth");
}
int kjb_pass_extract_half_res_fused(kjb_context* c, const kjb_extract_half_res_fused_args* a) {
    const char* P = "extract half-res inputs";
    c->epoch_a++;   // half_depth changes: the position cache built from it is stale
    const uint32_t W = a->half_depth_out.width, H = a->half_depth_out.height;
    const bool with_ssao = a->ssao_tex.data != nullptr && a->half_ssao_out.data != nullptr;
    if (!check_img(c, a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, P, "gbuffer_tex") || !check_img(c, a->depth_tex, KJB_FMT_R32_FLOAT, P, "depth_tex") ||
        !check_img(c, a->half_depth_out, KJB_FMT_R32_FLOAT, P, "half_depth_out") || !check_img(c, a->half_view_normal_out, KJB_FMT_RGBA8_SNORM, P, "half_view_normal_out", W, H)) return 1;
    if (with_ssao && (!check_img(c, a->ssao_tex, KJB_FMT_R8_UNORM, P, "ssao_tex") || !check_img(c, a->half_ssao_out, KJB_FMT_R8_SNORM, P, "half_ssao_out", W, H))) return 1;
    KJB_ROWS(c, H);
    // the half-res world positions D7/D9 want (kjb_set_option) come for free here when the launch covers the whole image
    kjb_context::PosCache& pc = c->pos_a;
    const float gts[4] = {float(a->gbuffer_tex.width), float(a->gbuffer_tex.height), 1.0f / float(a->gbuffer_tex.width), 1.0f / float(a->gbuffer_tex.height)};
    float4* positions = nullptr;
    if (c->opt_position_cache && kjb__rows.y0 == 0 && kjb__rows.y1 == int(H)) {
        const size_t need = size_t(W) * H * sizeof(float4);
        if (pc.cap < need) { dev_sync(c); dev_free(pc.d); pc.d = (float4*)dev_alloc(need); pc.cap = pc.d ? need : 0; }
        positions = pc.d;
    }
    KJB_LAUNCH(c, k_extract_half_fused, KJB_GRID2D(W, H, 32, 8), c->g, img_ro(a->gbuffer_tex), img_ro(a->depth_tex), img_ro(with_ssao ? a->ssao_tex : a->depth_tex), img_rw(a->half_view_normal_out),
               img_rw(a->half_depth_out), img_rw(with_ssao ? a->half_ssao_out : a->half_depth_out), with_ssao ? 1 : 0, halfres_subsample_offset(c->g.fc.frame_index), positions, f4(gts[0], gts[1], gts[2], gts[3]));
    if (positions) { pc.epoch = c->epoch_a; pc.src = a->half_depth_out.data; pc.w = W; pc.h = H; memcpy(pc.gts, gts, 16); }
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_extract_half_res_ssao(kjb_context* c, const kjb_extract_half_res_args* a) {
    if (!check_img(c, a->input_tex, KJB_FMT_R8_UNORM, "extract ssao/2", "input_tex") || !check_img(c, a->output_tex, KJB_FMT_R8_SNORM, "extract ssao/2", "output_tex")) return 1;
    KJB_ROWS(c, a->output_tex.height);
    KJB_LAUNCH(c, k_extract_half_ssao, KJB_GRID2D(a->output_tex.width, a->output_tex.height, 32, 8), img_ro(a->input_tex), img_rw(a->output_tex), halfres_subsample_offset(c->g.fc.frame_index));
    KJB_PASS_EPILOGUE(c, "extract ssao/2");
}
int kjb_pass_extract_half_res_view_normal(kjb_context* c, const kjb_extract_half_res_args* a) {
    if (!check_img(c, a->input_tex, KJB_FMT_RGBA32_FLOAT, "extract view normal/2", "input_tex") || !check_img(c, a->output_tex, KJB_FMT_RGBA8_SNORM, "extract view normal/2", "output_tex")) return 1;
    KJB_ROWS(c, a->output_tex.height);
    KJB_LAUNCH(c, k_extract_half_view_normal, KJB_GRID2D(a->output_tex.width, a->output_tex.height, 32, 8), c->g, img_ro(a->input_tex), img_rw(a->output_tex), halfres_subsample_offset(c->g.fc.frame_index));
    KJB_PASS_EPILOGUE(c, "extract view normal/2");
}

}  // extern "C"
