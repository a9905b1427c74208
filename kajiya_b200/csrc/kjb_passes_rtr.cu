// Ray-traced specular reflections (rtr) as sm_90a kernels — one kernel per render-graph pass of
// crates/lib/kajiya/src/renderers/rtr.rs, shader sources under /root/reference/assets/shaders/rtr/ (settings frozen to rtr_settings.hlsl).
// Thread mapping as in kjb_passes_rtdgi.cu: 32x8 blocks on the pass's pixel grid, 8x16 for the two ray-tracing passes (a warp = an 8x4 pixel patch).
#include "kjb_context.h"
#include "kjb_ircache.cuh"

using namespace kjb;

#define SKY_DIST 1e4f
#define RTR_ROUGHNESS_CLAMP 6e-4f
#define RTR_RESTIR_TEMPORAL_M_CLAMP 8.0f
#define RTR_RESTIR_MAX_PDF_CLAMP 200.0f
#define RTR_NEIGHBOR_RAY_ORIGIN_CENTER_BIAS 0.5f
#define RTR_SAMPLING_BIAS 0.15f   /* reflection_trace_common.inc.hlsl:37-43, USE_HEAVY_BIAS */

KJB_DEV float3 get_prev_eye_position(const kjb_view_constants& vc) { const float4 e = mul(vc.prev_view_to_prev_world, f4(0, 0, 0, 1)); return xyz(e) / e.w; }
KJB_DEV float3 position_world_to_view(const kjb_view_constants& vc, float3 v) { return xyz(mul(vc.world_to_view, f4(v, 1))); }
KJB_DEV float depth_to_view_z(const kjb_view_constants& vc, float depth) { return kjb_rcp(depth * -vc.clip_to_view.m[2 * 4 + 3]); }   // clip_to_view._43
KJB_DEV float3 flip_wo(float3 wo) { if (wo.z < 0.0f) { wo.z *= -0.25f; wo = normalize(wo); } return wo; }
KJB_DEV float ggx_ndf_0_1(float a2, float cos_theta) { const float ds = cos_theta * cos_theta * (a2 - 1.0f) + 1.0f; return a2 * a2 / (ds * ds); }
KJB_DEV float exponential_squish(float len, float s) { return kjb_exp2(-kjb_clamp(s * len, 0.0f, 100.0f)); }
KJB_DEV float exponential_unsquish(float len, float s) { return kjb_max(0.0f, -1.0f / s * kjb_log2(1e-30f + len)); }
KJB_DEV float3 specular_dominant_direction(float3 n, float3 v, float roughness) {   // inc/brdf.hlsl:313-317
    const float3 r = reflect(-v, n);
    const float f = (1.0f - roughness) * (kjb_sqrt(1.0f - roughness) + roughness);
    return normalize(vlerp(n, r, f));
}
KJB_DEV float3 soft_color_clamp(float3 center, float3 history, float3 ex, float3 dev) {   // inc/soft_color_clamp.hlsl
    const float3 history_dist = vabs(history - ex) / vmax(vabs(history * 0.1f), dev);
    const float3 closest_pt = vclamp(history, center - dev, center + dev);
    return vlerp(history, closest_pt, f3(kjb_smoothstep(1.0f, 3.0f, history_dist.x), kjb_smoothstep(1.0f, 3.0f, history_dist.y), kjb_smoothstep(1.0f, 3.0f, history_dist.z)));
}
struct RtrRestirRayOrigin { float3 ray_origin_eye_offset_ws; float roughness; uint32_t frame_index_mod4; };   // rtr_restir_pack_unpack.inc.hlsl
KJB_DEV RtrRestirRayOrigin rtr_ray_origin_from_raw(float4 raw) {
    RtrRestirRayOrigin r; r.ray_origin_eye_offset_ws = xyz(raw);
    const float2 misc = unpack_2x16f(kjb_f2u(raw.w));
    r.roughness = misc.x; r.frame_index_mod4 = kjb_cvt_u32(misc.y) & 3u;
    return r;
}
KJB_DEV float4 rtr_ray_origin_to_raw(const RtrRestirRayOrigin& o) { return f4(o.ray_origin_eye_offset_ws, kjb_u2f(pack_2x16f(o.roughness, float(o.frame_index_mod4)))); }
KJB_DEV int2 hi_px_subpixel(uint32_t i) { return halfres_subsample_offset(i); }   // hi_px_subpixels[i & 3]

// inc/blue_noise.hlsl:28-56 (host-supplied Heitz/Belcour spp64 tables)
struct BlueNoiseSamplerTables { const uint32_t *ranking, *scrambling, *sobol; };
KJB_DEV float blue_noise_sampler(const BlueNoiseSamplerTables& t, int pixel_i, int pixel_j, int sampleIndex, int sampleDimension) {
    pixel_i &= 127; pixel_j &= 127; sampleIndex &= 255; sampleDimension &= 255;
    const int rankedSampleIndex = sampleIndex ^ int(t.ranking[sampleDimension + (pixel_i + pixel_j * 128) * 8]);
    int value = int(t.sobol[sampleDimension + rankedSampleIndex * 256]);
    value = value ^ int(t.scrambling[(sampleDimension % 8) + (pixel_i + pixel_j * 128) * 8]);
    return (0.5f + float(value)) / 256.0f;
}

struct RtrTraceResult { float3 total_radiance; float hit_t; float3 hit_normal_vs; };
// rtr/reflection_trace_common.inc.hlsl:49-257 (USE_WORLD_RADIANCE_CACHE 0, USE_HEAVY_BIAS 1)
KJB_DEV RtrTraceResult rtr_do_the_thing(const Globals& g, const Img& gbuffer_tex, const Img& depth_tex, const Img& rtdgi_tex, const Img& sky_cube_tex, float4 gts, const IrcacheBufs& ircache,
                                        float3 normal_ws, float roughness, uint32_t& rng, const Ray& outgoing_ray) {
    const kjb_view_constants& vc = g.fc.view_constants;
    const float roughness_bias = roughness;   // USE_AGGRESSIVE_SECONDARY_ROUGHNESS_BIAS
    RayCone cone; cone.width = 0; cone.spread_angle = pixel_cone_spread_angle_from_image_height(vc, gts.y);
    cone = ray_cone_propagate(cone, kjb_sqrt(roughness) * 0.05f, length(outgoing_ray.origin - get_eye_position(vc)));
    const GbufferPathVertex primary_hit = gbuffer_raytrace(g, outgoing_ray, cone, 1, false);
    RtrTraceResult result;
    if (primary_hit.is_hit) {
        GbufferData gbuffer = gbuffer_unpack(primary_hit.gbuffer_packed);
        gbuffer.roughness = kjb_lerp(gbuffer.roughness, 1.0f, roughness_bias);
        const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
        const float3 wo = mul(-outgoing_ray.dir, tangent_to_world);
        const LayeredBrdf brdf = layered_brdf_from_gbuffer_ndotv(g, gbuffer, wo.z);
        const float3 primary_hit_cs = position_world_to_sample(vc, primary_hit.position);
        const float2 primary_hit_uv = cs_to_uv(xy(primary_hit_cs));
        const int2 npx = nearest_clamp_px(depth_tex, primary_hit_uv);
        const float primary_hit_screen_depth = ld_r32f(depth_tex, npx.x, npx.y);
        const uint4 screen_gb = ld_rgba32u(gbuffer_tex, kjb_cvt_i32(primary_hit_uv.x * gts.x), kjb_cvt_i32(primary_hit_uv.y * gts.y));
        const float3 primary_hit_screen_normal_ws = unpack_normal_11_10_11(screen_gb.y);
        const bool is_on_screen = kjb_abs(primary_hit_cs.x) < 1.0f && kjb_abs(primary_hit_cs.y) < 1.0f
            && inverse_depth_relative_diff(primary_hit_cs.z, primary_hit_screen_depth) < 5e-3f
            && dot(primary_hit_screen_normal_ws, -outgoing_ray.dir) > 0.0f
            && dot(primary_hit_screen_normal_ws, gbuffer.normal) > 0.7f;
        float3 total_radiance = f3(0.0f);
        {   // sun
            float2 urand; urand.x = rand01(rng); urand.y = rand01(rng);
            const float3 to_light_norm = sample_sun_direction(g.fc, urand, true);
            const bool is_shadowed = rt_is_shadowed(g, primary_hit.position, to_light_norm, 1e-4f, SKY_DIST);
            const float3 wi = mul(to_light_norm, tangent_to_world);
            const float3 brdf_value = layered_evaluate(brdf, wo, wi) * kjb_max(0.0f, wi.z);
            const float3 light_radiance = is_shadowed ? f3(0.0f) : f3(g.sun_color[0], g.sun_color[1], g.sun_color[2]);
            total_radiance += brdf_value * light_radiance;
        }
        const float3 reflected_normal_vs = direction_world_to_view(vc, gbuffer.normal);
        total_radiance += gbuffer.emissive;
        if (is_on_screen) {   // USE_SCREEN_GI_REPROJECTION
            const int2 rp = nearest_clamp_px(rtdgi_tex, primary_hit_uv);
            const float3 reprojected_radiance = xyz(ld_rgba16f(rtdgi_tex, rp.x, rp.y)) * g.fc.pre_exposure_delta;
            total_radiance += reprojected_radiance * gbuffer.albedo;
        } else {
            float2 urand; urand.x = rand01(rng); urand.y = rand01(rng);
            for (uint32_t li = 0; li < g.fc.triangle_light_count; ++li) {
                const kjb_triangle_light tl = g.lights[li];
                const LightSample ls = sample_triangle_light(tl, urand);
                const float3 to_light_ws = ls.pos - primary_hit.position;
                const float dist_to_light2 = dot(to_light_ws, to_light_ws);
                const float3 to_light_norm_ws = to_light_ws * kjb_rsqrt(dist_to_light2);
                const float to_psa_metric = kjb_max(0.0f, dot(to_light_norm_ws, gbuffer.normal)) * kjb_max(0.0f, dot(to_light_norm_ws, -ls.normal)) / dist_to_light2;
                if (to_psa_metric > 0.0f) {
                    const bool is_shadowed = rt_is_shadowed(g, primary_hit.position, to_light_norm_ws, 1e-4f, kjb_sqrt(dist_to_light2) - 2e-4f);
                    const float3 bounce_albedo = vlerp(gbuffer.albedo, f3(1.0f), 0.04f);
                    const float3 brdf_value = bounce_albedo * to_psa_metric / KJB_PI_F;
                    total_radiance += !is_shadowed ? (f3(tl.radiance[0], tl.radiance[1], tl.radiance[2]) * brdf_value / ls.pdf) : f3(0.0f);
                }
            }
            const float cone_width = ray_cone_propagate(cone, 0.0f, primary_hit.ray_t).width;
            total_radiance += ircache_lookup<false>(g, ircache, outgoing_ray.origin, primary_hit.position, gbuffer.normal, 1, rng, cone_width < 0.1f) * gbuffer.albedo;
        }
        result.total_radiance = total_radiance; result.hit_t = primary_hit.ray_t; result.hit_normal_vs = reflected_normal_vs;
        return result;
    }
    result.total_radiance = xyz(sample_cube_rgba16f(sky_cube_tex, outgoing_ray.dir));
    result.hit_t = SKY_DIST;
    result.hit_normal_vs = -direction_world_to_view(vc, outgoing_ray.dir);
    return result;
}

// ------------------------------------------------------------------ R1 reflection.rgen.hlsl:41-169
struct RtrTraceImgs { Img gbuffer_tex, depth_tex, rtdgi_tex, sky_cube_tex; ImgW out0_tex, out1_tex, out2_tex, rng_out_tex; };
KJB_DEV void rtr_trace_px(const Globals& g, const RtrTraceImgs& t, const BlueNoiseSamplerTables& bn, float4 gts, uint32_t reuse_rtdgi_rays, const IrcacheBufs& ircache, int x, int y) {
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const int hx = x * 2 + hso.x, hy = y * 2 + hso.y;
    const float depth = ld_r32f(t.depth_tex, hx, hy);
    if (0.0f == depth) { st_rgba16f(t.out0_tex, x, y, f4(0, 0, 0, -SKY_DIST)); return; }
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float2 uv = get_uv(hx, hy, s4);
    GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, hx, hy));
    gbuffer.roughness = kjb_max(gbuffer.roughness, RTR_ROUGHNESS_CLAMP);
    if (reuse_rtdgi_rays && gbuffer.roughness > 0.6f) return;   // keep the diffuse candidates
    const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_biased_depth(vc, uv, depth);
    const float3 refl_ray_origin_ws = vrc.biased_secondary_ray_origin_ws_with_normal(gbuffer.normal);
    const float3 wo = flip_wo(mul(-vrc.ray_dir_ws(), tangent_to_world));
    SpecularBrdf specular_brdf; specular_brdf.albedo = vlerp(f3(0.04f), gbuffer.albedo, gbuffer.metalness); specular_brdf.roughness = gbuffer.roughness;
    const uint32_t noise_offset = g.fc.frame_index;   // USE_TEMPORAL_JITTER
    uint32_t rng = hash3(uint32_t(x), uint32_t(y), noise_offset);
    float2 urand;
    if (bn.ranking) { urand.x = blue_noise_sampler(bn, x, y, int(noise_offset), 0); urand.y = blue_noise_sampler(bn, x, y, int(noise_offset), 1); }
    else urand = xy(blue_noise_for_pixel(g, uint32_t(x), uint32_t(y), noise_offset));
    urand.x = kjb_lerp(urand.x, 0.0f, RTR_SAMPLING_BIAS);
    BrdfSample brdf_sample = specular_sample(specular_brdf, wo, urand);
    for (uint32_t retry_i = 0; retry_i < 4u && !(brdf_sample.wi.z > 1e-6f); ++retry_i) {
        urand.x = rand01(rng); urand.y = rand01(rng);
        urand.x = kjb_lerp(urand.x, 0.0f, RTR_SAMPLING_BIAS);
        brdf_sample = specular_sample(specular_brdf, wo, urand);
    }
    const float cos_theta = normalize(wo + brdf_sample.wi).z;
    if (brdf_sample.wi.z > 1e-6f) {   // is_valid
        Ray outgoing_ray; outgoing_ray.dir = mul(tangent_to_world, brdf_sample.wi); outgoing_ray.origin = refl_ray_origin_ws; outgoing_ray.tmin = 0; outgoing_ray.tmax = SKY_DIST;
        st_r32u(t.rng_out_tex, x, y, rng);
        const RtrTraceResult result = rtr_do_the_thing(g, t.gbuffer_tex, t.depth_tex, t.rtdgi_tex, t.sky_cube_tex, gts, ircache, gbuffer.normal, gbuffer.roughness, rng, outgoing_ray);
        const float3 hit_offset_ws = outgoing_ray.dir * result.hit_t;
        const EnergyPreservation brdf_lut = energy_preservation_from_brdf_ndotv(g, specular_brdf, wo.z);
        const float pdf = brdf_sample.pdf / brdf_lut.valid_sample_fraction;
        st_rgba16f(t.out0_tex, x, y, f4(result.total_radiance, 1 - cos_theta));
        st_rgba16f(t.out1_tex, x, y, f4(hit_offset_ws, pdf));
        st_rgba8s(t.out2_tex, x, y, f4(result.hit_normal_vs, 0));
    } else {
        st_rgba16f(t.out0_tex, x, y, f4(1, 0, 1, 0));
        st_rgba16f(t.out1_tex, x, y, f4(0.0f));
    }
}
#ifndef KJB_OCC_RTR_TRACE
#define KJB_OCC_RTR_TRACE 8   /* 80 -> 64 registers */
#endif
KJB_KERNEL_OCC(128, KJB_OCC_RTR_TRACE) k_rtr_trace(const __grid_constant__ Globals g, RtrTraceImgs t, BlueNoiseSamplerTables bn, float4 gts, uint32_t reuse_rtdgi_rays, IrcacheBufs ircache, Rows kjb_rows) {
    KJB_PX; if (x >= t.out0_tex.w || y >= t.out0_tex.h) return;
    rtr_trace_px(g, t, bn, gts, reuse_rtdgi_rays, ircache, x, y);
}
#define KJB_SERIAL_TILES(W, H, ...) do { if (blockIdx.x | blockIdx.y | threadIdx.x | threadIdx.y) return; \
        for (int by = kjb_rows.y0; by < kjb_rows.y1; by += KJB_RAY_BY) for (int bx = 0; bx < (W); bx += KJB_RAY_BX) \
            for (int y = by; y < by + KJB_RAY_BY && y < kjb_rows.y1 && y < (H); ++y) for (int x = bx; x < bx + KJB_RAY_BX && x < (W); ++x) { __VA_ARGS__; } } while (0)
KJB_KERNEL(32) k_rtr_trace_serial(const __grid_constant__ Globals g, RtrTraceImgs t, BlueNoiseSamplerTables bn, float4 gts, uint32_t reuse_rtdgi_rays, IrcacheBufs ircache, Rows kjb_rows) {
    KJB_SERIAL_TILES(t.out0_tex.w, t.out0_tex.h, rtr_trace_px(g, t, bn, gts, reuse_rtdgi_rays, ircache, x, y));
}

// ------------------------------------------------------------------ R2 reflection_validate.rgen.hlsl:42-146 (one thread per 2x2 quad of half-res pixels)
struct RtrValidateImgs { Img gbuffer_tex, depth_tex, rtdgi_tex, sky_cube_tex, ray_orig_history_tex, ray_history_tex, rng_history_tex; ImgW invalidity_tex, irradiance_history_tex, reservoir_history_tex; };
KJB_DEV void rtr_validate_quad(const Globals& g, const RtrValidateImgs& t, float4 gts, const IrcacheBufs& ircache, int qx, int qy) {
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const int x = qx * 2 + hso.x, y = qy * 2 + hso.y;
    const int hx = x * 2 + hso.x, hy = y * 2 + hso.y;
    const float depth = ld_r32f(t.depth_tex, hx, hy);
    if (0.0f == depth) { st_r8u(t.invalidity_tex, x, y, 1.0f); return; }
    GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, hx, hy));
    gbuffer.roughness = kjb_max(gbuffer.roughness, RTR_ROUGHNESS_CLAMP);
    const float3 ray_orig_ws = xyz(ld_rgba32f(t.ray_orig_history_tex, x, y)) + get_prev_eye_position(vc);
    const float3 ray_hit_ws = xyz(ld_rgba16f(t.ray_history_tex, x, y)) + ray_orig_ws;
    Ray outgoing_ray; outgoing_ray.dir = normalize(ray_hit_ws - ray_orig_ws); outgoing_ray.origin = ray_orig_ws; outgoing_ray.tmin = 0; outgoing_ray.tmax = SKY_DIST;
    uint32_t rng = ld_r32u(t.rng_history_tex, x, y);
    const RtrTraceResult result = rtr_do_the_thing(g, t.gbuffer_tex, t.depth_tex, t.rtdgi_tex, t.sky_cube_tex, gts, ircache, gbuffer.normal, gbuffer.roughness, rng, outgoing_ray);
    Reservoir r = Reservoir::from_raw(ld_rg32u(as_ro(t.reservoir_history_tex), x, y));
    const float ped = g.fc.pre_exposure_delta;
    const float4 prev_irradiance_packed = ld_rgba16f(as_ro(t.irradiance_history_tex), x, y);
    const float3 prev_irradiance = vmax(f3(0.0f), xyz(prev_irradiance_packed) * ped);
    const float3 check_radiance = vmax(f3(0.0f), result.total_radiance);
    const float rad_diff = length(vabs(prev_irradiance - check_radiance) / vmax(f3(1e-3f), prev_irradiance + check_radiance));
    const float invalidity = kjb_smoothstep(0.1f, 0.5f, rad_diff / length(f3(1.0f)));
    r.M *= 1 - invalidity;
    st_rgba16f(t.irradiance_history_tex, x, y, f4(check_radiance, prev_irradiance_packed.w));
    st_r8u(t.invalidity_tex, x, y, invalidity);
    st_rg32u(t.reservoir_history_tex, x, y, r.as_raw());
    for (uint32_t i = 1; i <= 3u; ++i) {   // also reduce M of the quad neighbours
        const int2 sp = hi_px_subpixel(g.fc.frame_index + i);
        const int nx = qx * 2 + sp.x, ny = qy * 2 + sp.y;
        const float4 neighbor_prev_irradiance_packed = ld_rgba16f(as_ro(t.irradiance_history_tex), nx, ny);
        {
            const float3 av = vmax(f3(0.0f), xyz(neighbor_prev_irradiance_packed) * ped), bv = prev_irradiance;
            const float neigh_rad_diff = length(vabs(av - bv) / vmax(f3(1e-8f), av + bv));
            if (neigh_rad_diff < 0.2f) st_rgba16f(t.irradiance_history_tex, nx, ny, f4(check_radiance, neighbor_prev_irradiance_packed.w));
        }
        st_r8u(t.invalidity_tex, nx, ny, invalidity);
        if (invalidity > 0) {
            Reservoir nr = Reservoir::from_raw(ld_rg32u(as_ro(t.reservoir_history_tex), nx, ny));
            nr.M *= 1 - invalidity;
            st_rg32u(t.reservoir_history_tex, nx, ny, nr.as_raw());
        }
    }
}
#ifndef KJB_OCC_RTR_VALIDATE
#define KJB_OCC_RTR_VALIDATE 8
#endif
KJB_KERNEL_OCC(128, KJB_OCC_RTR_VALIDATE) k_rtr_validate(const __grid_constant__ Globals g, RtrValidateImgs t, float4 gts, IrcacheBufs ircache, int QW, int QH, Rows kjb_rows) {
    KJB_PX; if (x >= QW || y >= QH) return;
    rtr_validate_quad(g, t, gts, ircache, x, y);
}
KJB_KERNEL(32) k_rtr_validate_serial(const __grid_constant__ Globals g, RtrValidateImgs t, float4 gts, IrcacheBufs ircache, int QW, int QH, Rows kjb_rows) {
    KJB_SERIAL_TILES(QW, QH, rtr_validate_quad(g, t, gts, ircache, x, y));
}

// ------------------------------------------------------------------ R3 rtr_restir_temporal.hlsl:148-533
struct RtrRestirTemporalImgs {
    Img gbuffer_tex, half_view_normal_tex, depth_tex, candidate0_tex, candidate1_tex, candidate2_tex, irradiance_history_tex, ray_orig_history_tex, ray_history_tex, rng_history_tex,
        reservoir_history_tex, reprojection_tex, hit_normal_history_tex;
    ImgW irradiance_out_tex, ray_orig_output_tex, ray_output_tex, rng_output_tex, hit_normal_output_tex, reservoir_out_tex;
};
// :103-146
KJB_DEV void find_best_reprojection_in_neighborhood(const Globals& g, const RtrRestirTemporalImgs& t, float4 gts, float3 eye, float3 prev_eye, float2 base_px, int2& best_px, float3 refl_ray_origin_ws, bool wide) {
    const kjb_view_constants& vc = g.fc.view_constants;
    float best_dist = 1e10f;
    const float2 clip_scale = f2(vc.clip_to_view.m[0], vc.clip_to_view.m[5]);
    const float2 offset_scale = f2(1, -1) * -2.0f * clip_scale * f2(gts.z, gts.w);
    const float3 look_direction = direction_view_to_world(vc, f3(0, 0, -1));
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    {
        const float z_offset = dot(look_direction, refl_ray_origin_ws - eye);
        const float2 o = f2(float(hso.x), float(hso.y)) * offset_scale * z_offset;
        refl_ray_origin_ws += direction_view_to_world(vc, f3(o.x, o.y, 0));
    }
    const int start_coord = wide ? -1 : 0;
    for (int y = start_coord; y <= 1; ++y) for (int x = start_coord; x <= 1; ++x) {
        const int sx = kjb_cvt_i32(kjb_floor(base_px.x + float(x))), sy = kjb_cvt_i32(kjb_floor(base_px.y + float(y)));
        const RtrRestirRayOrigin ray_orig = rtr_ray_origin_from_raw(ld_rgba32f(t.ray_orig_history_tex, sx, sy));
        float3 orig = ray_orig.ray_origin_eye_offset_ws + prev_eye;
        const int2 oj = hi_px_subpixel(ray_orig.frame_index_mod4);
        {
            const float z_offset = dot(look_direction, orig);
            const float2 o = f2(float(oj.x), float(oj.y)) * offset_scale * z_offset;
            orig += direction_view_to_world(vc, f3(o.x, o.y, 0));
        }
        const float d = length(orig - refl_ray_origin_ws);
        if (d < best_dist) { best_dist = d; best_px = i2(sx, sy); }
    }
}
#ifndef KJB_OCC_RTR_RESTIR_TEMPORAL
#define KJB_OCC_RTR_RESTIR_TEMPORAL 4   /* 107 -> 64 registers */
#endif
KJB_KERNEL_OCC(256, KJB_OCC_RTR_RESTIR_TEMPORAL) k_rtr_restir_temporal(const __grid_constant__ Globals g, RtrRestirTemporalImgs t, float4 gts, Rows kjb_rows) {
    KJB_PX; if (x >= t.irradiance_out_tex.w || y >= t.irradiance_out_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const int hx = x * 2 + hso.x, hy = y * 2 + hso.y;
    const float depth = ld_r32f(t.depth_tex, hx, hy);
    if (0.0f == depth) {
        st_rgba16f(t.irradiance_out_tex, x, y, f4(0, 0, 0, -SKY_DIST)); st_rgba16f(t.hit_normal_output_tex, x, y, f4(0.0f)); st_rg32u(t.reservoir_out_tex, x, y, u2(0, 0));
        return;
    }
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float2 uv = get_uv(hx, hy, s4);
    const float3 eye = get_eye_position(vc), prev_eye = get_prev_eye_position(vc);
    const float ped = g.fc.pre_exposure_delta;
    const float3 normal_vs = xyz(ld_rgba8s(t.half_view_normal_tex, x, y));
    const float3 normal_ws = direction_view_to_world(vc, normal_vs);
    float local_normal_flatness = 1;
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) local_normal_flatness *= kjb_saturate(dot(normal_vs, xyz(ld_rgba8s(t.half_view_normal_tex, x + xx, y + yy))));
    float reprojection_neighborhood_stability = 1;
    for (int yy = 0; yy <= 1; ++yy) for (int xx = 0; xx <= 1; ++xx) reprojection_neighborhood_stability *= ld_rgba16s(t.reprojection_tex, x * 2 + xx, y * 2 + yy).z;
    const ViewRayContext vrc = ViewRayContext::from_uv_and_biased_depth(vc, uv, depth);
    const float3 refl_ray_origin_ws = vrc.biased_secondary_ray_origin_ws_with_normal(normal_ws);
    const float3 refl_ray_origin_vs = position_world_to_view(vc, refl_ray_origin_ws);
    const float3x3 tangent_to_world = build_orthonormal_basis(normal_ws);
    float3 outgoing_dir = f3(0, 0, 1);
    uint32_t rng = hash3(uint32_t(x), uint32_t(y), g.fc.frame_index);
    const GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, hx, hy));
    const float a2 = kjb_max(RTR_ROUGHNESS_CLAMP, gbuffer.roughness) * kjb_max(RTR_ROUGHNESS_CLAMP, gbuffer.roughness);

    float pdf_sel = 0, cos_theta = 0;
    float3 irradiance_sel = f3(0.0f); float4 ray_orig_sel = f4(0.0f); float3 ray_hit_sel_ws = f3(1.0f), hit_normal_sel = f3(1.0f);
    uint32_t rng_sel = ld_r32u(as_ro(t.rng_output_tex), x, y);
    StreamState stream_state; stream_state.p_q_sel = 0; stream_state.M_sum = 0;
    Reservoir reservoir = Reservoir::create();
    const uint32_t reservoir_payload = uint32_t(x) | (uint32_t(y) << 16);
    reservoir.payload = reservoir_payload;
    {   // :68-83: the candidate
        const float4 hit0 = ld_rgba16f(t.candidate0_tex, x, y), hit1 = ld_rgba16f(t.candidate1_tex, x, y), hit2 = ld_rgba8s(t.candidate2_tex, x, y);
        const float r_pdf = kjb_min(hit1.w, RTR_RESTIR_MAX_PDF_CLAMP);
        if (r_pdf > 0) {
            outgoing_dir = normalize(xyz(hit1));
            const float p_q = 1 * kjb_max(1e-3f, luminance(xyz(hit0))) * r_pdf;
            const float inv_pdf_q = 1.0f / r_pdf;
            pdf_sel = r_pdf; cos_theta = 1 - hit0.w; irradiance_sel = xyz(hit0);
            RtrRestirRayOrigin ray_orig; ray_orig.ray_origin_eye_offset_ws = refl_ray_origin_ws; ray_orig.roughness = gbuffer.roughness; ray_orig.frame_index_mod4 = g.fc.frame_index & 3u;
            ray_orig_sel = rtr_ray_origin_to_raw(ray_orig);
            ray_hit_sel_ws = xyz(hit1) + refl_ray_origin_ws;
            hit_normal_sel = direction_view_to_world(vc, xyz(hit2));
            if (p_q * inv_pdf_q > 0) reservoir.init_with_stream(p_q, inv_pdf_q, stream_state, reservoir_payload);
        }
    }
    const float4 center_reproj = ld_rgba16s(t.reprojection_tex, hx, hy);
    {   // USE_RESAMPLING
        const float ang_offset = float(((g.fc.frame_index + 7u) * 11u) % 32u) * KJB_TAU_F;
        const uint32_t max_samples = center_reproj.z < 1.0f ? 5u : 1u;
        for (uint32_t sample_i = 0; sample_i < max_samples && stream_state.M_sum < RTR_RESTIR_TEMPORAL_M_CLAMP; ++sample_i) {
            const float ang = (float(sample_i) + ang_offset) * KJB_GOLDEN_ANGLE;
            const float rpx_offset_radius = kjb_sqrt(float(((sample_i - 1u) + g.fc.frame_index) & 3u) + 1.0f) * kjb_clamp(8.0f - stream_state.M_sum, 1.0f, 7.0f);
            float sn, cs; kjb_sincos(ang, &sn, &cs);
            const float2 reservoir_px_offset_base = f2(cs, sn) * rpx_offset_radius;
            const int ox = sample_i == 0 ? 0 : kjb_cvt_i32(reservoir_px_offset_base.x), oy = sample_i == 0 ? 0 : kjb_cvt_i32(reservoir_px_offset_base.y);
            const float4 reproj = ld_rgba16s(t.reprojection_tex, hx + ox * 2, hy + oy * 2);
            int2 reproj_px;
            {
                const float2 base_px = f2(float(x), float(y)) + f2(gts.x, gts.y) * xy(reproj) / 2.0f;
                int2 best_px = i2(kjb_cvt_i32(kjb_floor(base_px.x + 0.5f)), kjb_cvt_i32(kjb_floor(base_px.y + 0.5f)));
                if (reprojection_neighborhood_stability >= 1) {
                    if (kjb_abs(gts.x * reproj.x) > 0.1f || kjb_abs(gts.y * reproj.y) > 0.1f) find_best_reprojection_in_neighborhood(g, t, gts, eye, prev_eye, base_px, best_px, refl_ray_origin_ws, false);
                } else {
                    find_best_reprojection_in_neighborhood(g, t, gts, eye, prev_eye, base_px, best_px, refl_ray_origin_ws, true);
                }
                reproj_px = best_px;
            }
            const int rx = reproj_px.x + ox, ry = reproj_px.y + oy;
            Reservoir r = Reservoir::from_raw(ld_rg32u(t.reservoir_history_tex, rx, ry));
            const int spx_x = int(r.payload & 0xffffu), spx_y = int(r.payload >> 16);
            const float4 prev_ray_orig_and_roughness = ld_rgba32f(t.ray_orig_history_tex, spx_x, spx_y) + f4(prev_eye, 0);
            const float3 dro = refl_ray_origin_ws - xyz(prev_ray_orig_and_roughness);
            if (dot(dro, dro) > 0.05f * refl_ray_origin_vs.z * refl_ray_origin_vs.z) continue;   // disocclusion
            const float4 prev_irrad_and_cos_theta = ld_rgba16f(t.irradiance_history_tex, spx_x, spx_y) * f4(ped, ped, ped, 1);
            const float3 prev_irrad = xyz(prev_irrad_and_cos_theta);
            const float prev_cos_theta = 1 - prev_irrad_and_cos_theta.w;
            const float4 sample_hit_ws_and_pdf_packed = ld_rgba16f(t.ray_history_tex, spx_x, spx_y);
            const float prev_pdf = sample_hit_ws_and_pdf_packed.w;
            const float3 sample_hit_ws = xyz(sample_hit_ws_and_pdf_packed) + xyz(prev_ray_orig_and_roughness);
            const float prev_dist = length(xyz(sample_hit_ws_and_pdf_packed));
            const float4 hn = ld_rgba16f(t.hit_normal_history_tex, spx_x, spx_y);
            const float4 sample_hit_normal_ws_dot = f4(hn.x * 2 - 1, hn.y * 2 - 1, hn.z * 2 - 1, hn.w);
            const float3 dir_to_sample_hit_unnorm = sample_hit_ws - refl_ray_origin_ws;
            const float dist_to_sample_hit = length(dir_to_sample_hit_unnorm);
            const float3 dir_to_sample_hit = normalize(dir_to_sample_hit_unnorm);
            r.M = kjb_min(r.M, RTR_RESTIR_TEMPORAL_M_CLAMP);
            {   // USE_TRANSLATIONAL_CLAMP
                const float3 current_wo = normalize(vrc.ray_hit_ws() - eye);
                const float3 prev_wo = normalize(vrc.ray_hit_ws() - prev_eye);
                const float wo_dot = kjb_saturate(dot(current_wo, prev_wo));
                const float wo_similarity = kjb_pow(kjb_saturate(ggx_ndf_0_1(kjb_max(3e-5f, a2), wo_dot)), 64.0f);
                float mult = kjb_lerp(wo_similarity, 1.0f, kjb_smoothstep(0.05f, 0.5f, kjb_sqrt(gbuffer.roughness)));
                mult = kjb_lerp(1.0f, mult, local_normal_flatness);
                r.M *= mult;
            }
            float p_q = 1;
            p_q *= kjb_max(1e-3f, luminance(prev_irrad));
            p_q *= kjb_step(0.0f, dot(dir_to_sample_hit, normal_ws));   // RTR_RESTIR_BRDF_SAMPLING
            p_q *= prev_pdf;
            float jacobian = 1;
            jacobian *= kjb_clamp(prev_dist / dist_to_sample_hit, 1e-4f, 1e4f);
            jacobian *= jacobian;
            jacobian *= kjb_max(0.0f, -dot(xyz(sample_hit_normal_ws_dot), dir_to_sample_hit)) / kjb_max(1e-5f, sample_hit_normal_ws_dot.w);
            {   // USE_JACOBIAN_BASED_REJECTION
                const float JACOBIAN_REJECT_THRESHOLD = kjb_lerp(1.1f, 4.0f, gbuffer.roughness * gbuffer.roughness);
                if (!(jacobian < JACOBIAN_REJECT_THRESHOLD && jacobian > 1.0f / JACOBIAN_REJECT_THRESHOLD)) continue;
            }
            p_q *= jacobian;
            if (reservoir.update_with_stream(r, p_q, 1.0f, stream_state, reservoir_payload, rng)) {
                outgoing_dir = dir_to_sample_hit;
                pdf_sel = prev_pdf; cos_theta = prev_cos_theta; irradiance_sel = prev_irrad;
                ray_orig_sel = prev_ray_orig_and_roughness;
                ray_hit_sel_ws = sample_hit_ws;
                hit_normal_sel = xyz(sample_hit_normal_ws_dot);
                rng_sel = ld_r32u(t.rng_history_tex, spx_x, spx_y);
            }
        }
        reservoir.finish_stream(stream_state);
        reservoir.W = kjb_min(reservoir.W, 1e20f);   // RESTIR_RESERVOIR_W_CLAMP
    }
    const float4 hit_normal_ws_dot = f4(hit_normal_sel, -dot(hit_normal_sel, outgoing_dir));
    st_rgba16f(t.irradiance_out_tex, x, y, f4(irradiance_sel, 1 - cos_theta));
    st_rgba32f(t.ray_orig_output_tex, x, y, f4(xyz(ray_orig_sel) - eye, ray_orig_sel.w));
    st_rgba16f(t.hit_normal_output_tex, x, y, f4(hit_normal_ws_dot.x * 0.5f + 0.5f, hit_normal_ws_dot.y * 0.5f + 0.5f, hit_normal_ws_dot.z * 0.5f + 0.5f, hit_normal_ws_dot.w));
    st_rgba16f(t.ray_output_tex, x, y, f4(ray_hit_sel_ws - xyz(ray_orig_sel), pdf_sel));
    st_r32u(t.rng_output_tex, x, y, rng_sel);
    st_rg32u(t.reservoir_out_tex, x, y, reservoir.as_raw());
}

// ------------------------------------------------------------------ R4 resolve.hlsl:78-663 (USE_RESTIR, BORROW_SAMPLES, CUT_CORNERS_IN_MATH)
struct RtrResolveImgs { Img gbuffer_tex, depth_tex, hit1_tex, reprojection_tex, half_view_normal_tex, ray_len_history_tex, restir_irradiance_tex, restir_ray_tex, restir_reservoir_tex, restir_ray_orig_tex; ImgW output_tex, ray_len_output_tex; };
#ifndef KJB_OCC_RTR_RESOLVE
#define KJB_OCC_RTR_RESOLVE 4   /* 98 -> 64 registers, 4 blocks per SM */
#endif
// sin / cos of the tap angles `(sample_i + ang_offset) * GOLDEN_ANGLE + (px_idx_in_quad / 4) * TAU`: 4 quad slots x 8 taps = 32 distinct angles per FRAME
// (ang_offset depends on the frame index only), so the host evaluates them once with the contract's kjb_sincos and every pixel looks its eight up
struct ResolveTapAngles { float sn[32], cs[32]; };
KJB_KERNEL_OCC(256, KJB_OCC_RTR_RESOLVE) k_rtr_resolve(const __grid_constant__ Globals g, RtrResolveImgs t, float4 ots, float radius_sample_mult, const __grid_constant__ ResolveTapAngles ta, Rows kjb_rows) {
    KJB_PX; if (x >= t.output_tex.w || y >= t.output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const int hpx = x / 2, hpy = y / 2;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float depth = ld_r32f(t.depth_tex, x, y);
    if (0.0f == depth) { st_r11g11b10(t.output_tex, x, y, f3(0.0f)); return; }
    GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, x, y));
    const float3 eye = get_eye_position(vc);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_biased_depth(vc, uv, depth);
    const float3 refl_ray_origin_ws = vrc.biased_secondary_ray_origin_ws_with_normal(gbuffer.normal);
    const float3 refl_ray_origin_vs = position_world_to_view(vc, refl_ray_origin_ws);
    gbuffer.roughness = kjb_max(gbuffer.roughness, RTR_ROUGHNESS_CLAMP);
    const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
    const float3 view_dir = -normalize(vrc.ray_dir_ws());
    const float3 wo = flip_wo(mul(view_dir, tangent_to_world));
    const SpecularBrdf specular_brdf = layered_brdf_from_gbuffer_ndotv(g, gbuffer, wo.z).specular_brdf;
    const uint32_t px_idx_in_quad = (((uint32_t(x) & 1u) | (uint32_t(y) & 1u) * 2u) + g.fc.frame_index) & 3u;   // SHUFFLE_SUBPIXELS
    const float a2 = kjb_max(RTR_ROUGHNESS_CLAMP, gbuffer.roughness) * kjb_max(RTR_ROUGHNESS_CLAMP, gbuffer.roughness);
    const float surf_to_hit_dist = length(xyz(ld_rgba16f(t.hit1_tex, hpx, hpy)));
    const float eye_to_surf_dist = length(refl_ray_origin_vs);
    const float3 ray_dir_vs = normalize(xyz(mul(vc.sample_to_view, f4(uv_to_cs(uv).x, uv_to_cs(uv).y, 0.0f, 1.0f))));   // ViewRayContext::ray_dir_vs()
    const float eye_ray_z_scale = -ray_dir_vs.z;
    const float4 reprojection_params = ld_rgba16s(t.reprojection_tex, x, y);
    const float ray_squish_scale = 16.0f / kjb_max(1e-5f, eye_to_surf_dist);
    const Img& rlh = t.ray_len_history_tex;
    const float rl_hist_y = bilinear_clamp(rlh.w, rlh.h, uv + xy(reprojection_params), [&](int sx, int sy) { const float2 v = ld_rg16f(rlh, sx, sy); return f4(v.x, v.y, 0, 1); }).y;
    const float ray_len_avg = exponential_unsquish(kjb_lerp(exponential_squish(rl_hist_y, ray_squish_scale), exponential_squish(surf_to_hit_dist, ray_squish_scale), 0.1f), ray_squish_scale);
    float4 contrib_accum = f4(0.0f); float ray_len_accum = 0;
    const float3 normal_vs = direction_world_to_view(vc, gbuffer.normal);
    const float tan_theta = kjb_sqrt(gbuffer.roughness) * 0.25f;
    const float c2v11 = vc.clip_to_view.m[5];
    float kernel_size_ws;
    {
        const float clamped_ray_len_avg = kjb_max(ray_len_avg, eye_to_surf_dist / eye_ray_z_scale * c2v11 * 0.2f * kjb_smoothstep(0.0f, 0.05f * eye_to_surf_dist, ray_len_avg));
        const float kernel_size_vs = clamped_ray_len_avg / (clamped_ray_len_avg + eye_to_surf_dist);
        kernel_size_ws = kernel_size_vs * eye_to_surf_dist * eye_ray_z_scale;
        kernel_size_ws *= tan_theta;
    }
    {
        const float scale_factor = eye_to_surf_dist * eye_ray_z_scale * c2v11;
        kernel_size_ws = kjb_min(kernel_size_ws, 0.1f * scale_factor);
        kernel_size_ws = kjb_max(kernel_size_ws, ots.w * 4.0f * scale_factor);
    }
    float3 kernel_t1, kernel_t2;
    {   // get_specular_filter_kernel_basis (:69-76)
        const float3 dominant = specular_dominant_direction(gbuffer.normal, view_dir, gbuffer.roughness);
        const float3 reflected = reflect(-dominant, gbuffer.normal);
        kernel_t1 = normalize(cross(gbuffer.normal, reflected)) * kernel_size_ws;
        kernel_t2 = cross(reflected, kernel_t1);
    }
    const float4 blue = blue_noise_for_pixel(g, uint32_t(hpx) + 16u, uint32_t(hpy) + 16u, g.fc.frame_index);
    const float KERNEL_SHARPNESS = 0.666f;
    const float RADIUS_INC_ON_FAIL = 0.25f;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index); (void)hso;
    // per-pixel invariants of the tap loop
    const float origin_bias_lerp = kjb_lerp(1.0f, RTR_NEIGHBOR_RAY_ORIGIN_CENTER_BIAS, 0.4f * kjb_min(1.0f, 3 * kjb_sqrt(gbuffer.roughness)));
    const float pdf_lerp_t = kjb_smoothstep(0.4f, 0.7f, kjb_sqrt(gbuffer.roughness)) * kjb_smoothstep(0.0f, 0.1f, ray_len_avg / eye_to_surf_dist);
    const float depth_rej_scale = kjb_max(1e-10f, kernel_size_ws), depth_rej_nz = -kjb_max(0.3f, normal_vs.z);
    const float squished_surf_to_hit = exponential_squish(surf_to_hit_dist, ray_squish_scale);
    float sample_radius_accum = 1;
    for (int sample_i = 1; sample_i <= 8; ++sample_i, sample_radius_accum += RADIUS_INC_ON_FAIL) {
        const bool is_center_sample = sample_i == 8;
        int spx0, spy0;
        {
            float sample_i_with_jitter = sample_radius_accum;
            if (is_center_sample) sample_i_with_jitter = contrib_accum.w > 1e-8f ? blue.y : 0.0f;
            else sample_i_with_jitter += blue.y;
            const float radius = kjb_pow(sample_i_with_jitter, KERNEL_SHARPNESS) * radius_sample_mult;
            const float sn = ta.sn[px_idx_in_quad * 8u + uint32_t(sample_i - 1)], cs = ta.cs[px_idx_in_quad * 8u + uint32_t(sample_i - 1)];
            const float3 offset_ws = (cs * kernel_t1 + sn * kernel_t2) * radius;
            const float3 sample_cs = position_world_to_sample(vc, refl_ray_origin_ws + offset_ws);
            const float2 sample_uv = cs_to_uv(xy(sample_cs));
            const int sample_px_x = kjb_cvt_i32(kjb_floor(sample_uv.x * ots.x / 2.0f)), sample_px_y = kjb_cvt_i32(kjb_floor(sample_uv.y * ots.y / 2.0f));
            spx0 = hpx + (sample_px_x - hpx); spy0 = hpy + (sample_px_y - hpy);
        }
        float rejection_bias = 1;
        const float3 sample_normal_vs = xyz(ld_rgba8s(t.half_view_normal_tex, spx0, spy0));
        float pdf0_mult = 1, pdf1_mult = 1;
        const uint2 reservoir_raw = ld_rg32u(t.restir_reservoir_tex, spx0, spy0);
        const Reservoir r = Reservoir::from_raw(reservoir_raw);
        const int spx_x = int(r.payload & 0xffffu), spx_y = int(r.payload >> 16);
        const RtrRestirRayOrigin sample_origin = rtr_ray_origin_from_raw(ld_rgba32f(t.restir_ray_orig_tex, spx_x, spx_y));
        const float3 sample_origin_ws = sample_origin.ray_origin_eye_offset_ws + eye;
        if (reservoir_raw.x == 0 || sample_origin.roughness > gbuffer.roughness * 2) continue;
        const float4 restir_ray = ld_rgba16f(t.restir_ray_tex, spx_x, spx_y);
        const float3 sample_hit_ws = xyz(restir_ray) + sample_origin_ws;
        const float3 sample_origin_vs = position_world_to_view(vc, sample_origin_ws);
        const float4 restir_irr = ld_rgba16f(t.restir_irradiance_tex, spx_x, spx_y);
        const float3 sample_radiance = xyz(restir_irr);
        const float sample_ray_pdf = restir_ray.w;
        const float neighbor_sampling_pdf = 1.0f / r.W;
        const float3 sample_hit_vs = position_world_to_view(vc, sample_hit_ws);
        const float3 center_to_hit_vs = sample_hit_vs - vlerp(refl_ray_origin_vs, sample_origin_vs, RTR_NEIGHBOR_RAY_ORIGIN_CENTER_BIAS);
        const float sample_cos_theta = 1 - restir_irr.w;
        const float center_to_hit_dist = length(center_to_hit_vs);
        const float sample_to_hit_dist = length(sample_hit_ws - sample_origin_ws);
        {   // RTR_USE_BULLSHIT_TO_FIX_EDGE_HALOS
            const float wat = length(sample_hit_vs - vlerp(refl_ray_origin_vs, sample_origin_vs, origin_bias_lerp));
            pdf0_mult *= kjb_max(1e-5f, kjb_pow(wat / sample_to_hit_dist, 2.0f));
            pdf1_mult *= kjb_max(1.0f, kjb_pow(center_to_hit_dist / sample_to_hit_dist, 2.0f));
        }
        const float3 wi = normalize(mul(direction_view_to_world(vc, center_to_hit_vs), tangent_to_world));
        if (wi.z < 1e-5f) continue;
        rejection_bias *= dot(normal_vs, sample_normal_vs) > 0.7f ? 1.0f : 0.0f;
        {
            const float depth_diff = kjb_abs(refl_ray_origin_vs.z - sample_origin_vs.z) / depth_rej_scale;
            rejection_bias *= kjb_exp2(depth_rej_nz * depth_diff * depth_diff);
        }
        const float3 surface_offset = sample_origin_vs - refl_ray_origin_vs;
        if (dot(center_to_hit_vs, normal_vs) * 0.2f / length(center_to_hit_vs) < dot(surface_offset, normal_vs) / length(surface_offset)) rejection_bias *= is_center_sample ? 1.0f : 0.0f;   // USE_APPROXIMATE_SAMPLE_SHADOWING
        const BrdfValue spec = specular_evaluate(specular_brdf, wo, wi);
        const float spec_weight = spec.pdf * kjb_step(0.0f, wi.z);
        float contrib_wt = 0;
        {
            const float cos_theta = normalize(wo + wi).z;
            const float bent_cos_theta = kjb_min(sample_cos_theta, cos_theta * 1.25f);
            const float sample_ray_ndf = ggx_ndf(a2, bent_cos_theta), center_ndf = ggx_ndf(a2, cos_theta);
            const float bent_sample_pdf0 = spec.pdf * sample_ray_ndf / center_ndf;
            const float3 pdfs[2] = {f3(kjb_min(bent_sample_pdf0, RTR_RESTIR_MAX_PDF_CLAMP) * 1.0f, neighbor_sampling_pdf * pdf0_mult, 1 - pdf_lerp_t),
                                    f3(kjb_min(spec.pdf, RTR_RESTIR_MAX_PDF_CLAMP), neighbor_sampling_pdf * pdf1_mult, pdf_lerp_t)};
            for (uint32_t pdf_i = 0; pdf_i < 2u; ++pdf_i) {
                const float bent_sample_pdf = pdfs[pdf_i].x, nsp = pdfs[pdf_i].y, pdf_influence = pdfs[pdf_i].z;
                const float mis_weight = kjb_max(1e-4f, spec.pdf / (sample_ray_pdf + spec.pdf));
                contrib_wt = rejection_bias * mis_weight * kjb_max(1e-10f, spec_weight / bent_sample_pdf);
                contrib_accum += f4(sample_radiance * bent_sample_pdf / nsp * spec.value_over_pdf, 1) * contrib_wt * pdf_influence;
            }
        }
        ray_len_accum += squished_surf_to_hit * contrib_wt;
        sample_radius_accum += 1.0f - RADIUS_INC_ON_FAIL;
    }
    const float contrib_norm_factor = kjb_max(1e-14f, contrib_accum.w);
    float3 rgb = xyz(contrib_accum) / contrib_norm_factor;
    ray_len_accum /= contrib_norm_factor;
    const EnergyPreservation brdf_lut = energy_preservation_from_brdf_ndotv(g, specular_brdf, wo.z);
    rgb = rgb / brdf_lut.preintegrated_reflection;
    rgb = rgb * brdf_lut.preintegrated_reflection_mult;
    ray_len_accum = exponential_unsquish(ray_len_accum, ray_squish_scale);
    st_r11g11b10(t.output_tex, x, y, rgb);
    st_rg16f(t.ray_len_output_tex, x, y, ray_len_accum, ray_len_avg);
}

// ------------------------------------------------------------------ R5 temporal_filter.hlsl:36-259
struct RtrTemporalImgs { Img input_tex, history_tex, depth_tex, ray_len_tex, reprojection_tex, invalidity_tex, gbuffer_tex; ImgW output_tex; };
#ifndef KJB_OCC_RTR_TEMPORAL
#define KJB_OCC_RTR_TEMPORAL 4
#endif
// The block's (32+2)x(8+2) footprint of the resolved reflections (R11G11B10) and of the depth buffer is staged through the TMA engine (tile origin
// 4 texels left of the block: 16-byte aligned rows); the R11G11B10 decode and the conversion to the crunched luma-chroma working space run once per
// texel instead of once per tap of the 3x3 neighbourhood.
#define R5_TW 40
#define R5_AX 4
#define R5_LW 34
#define R5_TH 10
KJB_KERNEL_OCC(256, KJB_OCC_RTR_TEMPORAL) k_rtr_temporal(const __grid_constant__ TileSource ts_input, const __grid_constant__ TileSource ts_depth, int tile_mode_, Globals g, RtrTemporalImgs t, float4 ots, Rows kjb_rows) {
    constexpr int P4 = tile_pitch<4>(R5_TW);
    __shared__ __align__(128) uint32_t s_raw[P4 * R5_TH];
    __shared__ __align__(128) float s_depth[P4 * R5_TH];
    __shared__ float4 s_work[R5_LW * R5_TH];
    __shared__ __align__(8) uint64_t bar;
    const int tid = int(threadIdx.y) * 32 + int(threadIdx.x);
    const int bx0 = int(blockIdx.x) * 32, by0 = kjb_rows.y0 + int(blockIdx.y) * 8;
    tile_group_begin(&bar, 0, tile_mode_, tid);
    uint32_t staged = tile_issue<uint32_t, R5_TW, R5_TH>(s_raw, ts_input, t.input_tex, bx0 - R5_AX, by0 - 1, &bar, tile_mode_, tid, 256);
    staged += tile_issue<float, R5_TW, R5_TH>(s_depth, ts_depth, t.depth_tex, bx0 - R5_AX, by0 - 1, &bar, tile_mode_, tid, 256);
    tile_group_wait(&bar, 0, tile_mode_, staged, tid);
    for (int i = tid; i < R5_LW * R5_TH; i += 256) {
        const int lx = i % R5_LW, ly = i / R5_LW;
        const uint32_t v = s_raw[ly * P4 + lx + (R5_AX - 1)];
        // out-of-range taps read 0 from the R11G11B10 image with alpha 0, in-range ones alpha 1 (texel fetch of a 3-channel format) — as the oracle's load()
        const bool in_image = inb(t.input_tex, bx0 - 1 + lx, by0 - 1 + ly);
        s_work[i] = linear_to_working(in_image ? f4(f3(uf_to_f32(v & 2047u, 6), uf_to_f32((v >> 11) & 2047u, 6), uf_to_f32(v >> 22, 5)), 1) : f4(0.0f));
    }
    __syncthreads();
    const int x = bx0 + int(threadIdx.x), y = by0 + int(threadIdx.y);
    if (x >= t.output_tex.w || y >= t.output_tex.h || y >= kjb_rows.y1) return;
    const int tx = int(threadIdx.x) + 1, ty = int(threadIdx.y) + 1;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float ped = g.fc.pre_exposure_delta;
    const float4 history_mult = f4(ped, ped, ped, 1);
    const float3 eye = get_eye_position(vc), prev_eye = get_prev_eye_position(vc);
    const float4 center = s_work[ty * R5_LW + tx];
    const float refl_ray_length = kjb_clamp(ld_rg16f(t.ray_len_tex, x, y).x, 0.0f, 1e3f);
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float center_depth = s_depth[ty * P4 + tx + (R5_AX - 1)];
    const ViewRayContext vrc = ViewRayContext::from_uv_and_depth(vc, uv, center_depth);
    const float3 reflector_vs = vrc.ray_hit_vs();
    const float2 cs0 = uv_to_cs(uv);
    const float3 ray_dir_vs = normalize(xyz(mul(vc.sample_to_view, f4(cs0.x, cs0.y, 0.0f, 1.0f))));
    const float3 reflection_hit_vs = reflector_vs + ray_dir_vs * refl_ray_length;
    const float4 reflection_hit_cs = mul(vc.view_to_sample, f4(reflection_hit_vs, 1));
    const float4 prev_hit_cs = mul(vc.clip_to_prev_clip, reflection_hit_cs);
    float2 hit_prev_uv = cs_to_uv(f2(prev_hit_cs.x, prev_hit_cs.y) / prev_hit_cs.w);
    const float4 prev_reflector_cs = mul(vc.clip_to_prev_clip, vrc.ray_hit_cs);
    const float2 reflector_prev_uv = cs_to_uv(f2(prev_reflector_cs.x, prev_reflector_cs.y) / prev_reflector_cs.w);
    const float4 reproj = ld_rgba16s(t.reprojection_tex, x, y);
    const float reflector_move_rate = kjb_min(1.0f, length(xy(reproj)) / length(reflector_prev_uv - uv));
    hit_prev_uv = vlerp(uv, hit_prev_uv, reflector_move_rate);
    const uint32_t quad_reproj_valid_packed = kjb_cvt_u32(reproj.z * 15.0f + 0.5f);
    const Img& ht = t.history_tex;
    const float2 texSize = f2(ots.x, ots.y);
    float4 history0 = f4(0.0f); float history0_valid = 1;
    if (0u == quad_reproj_valid_packed) {
        history0_valid = 0;
    } else if (15u == quad_reproj_valid_packed) {   // image_sample_catmull_rom_5tap (inc/image.hlsl:85-170), sampler_lnc, identity remap
        auto smp = [&](float2 p) { return bilinear_clamp(ht.w, ht.h, p, [&](int sx, int sy) { return ld_rgba16f(ht, sx, sy); }); };
        const float2 samplePos = (uv + xy(reproj)) * texSize;
        const float2 texPos1 = vfloor(samplePos - 0.5f) + 0.5f;
        const float2 f = samplePos - texPos1;
        const float2 w0 = f * (-0.5f + f * (1.0f - 0.5f * f));
        const float2 w1 = 1.0f + f * f * (-2.5f + 1.5f * f);
        const float2 w2 = f * (0.5f + f * (2.0f - 1.5f * f));
        const float2 w3 = f * f * (-0.5f + 0.5f * f);
        const float2 w12 = w1 + w2;
        const float2 offset12 = w2 / (w1 + w2);
        const float2 texPos0 = (texPos1 - 1.0f) / texSize, texPos3 = (texPos1 + 2.0f) / texSize, texPos12 = (texPos1 + offset12) / texSize;
        float4 result = f4(0.0f);
        result += smp(f2(texPos12.x, texPos0.y)) * w12.x * w0.y;
        result += smp(f2(texPos0.x, texPos12.y)) * w0.x * w12.y;
        result += smp(f2(texPos12.x, texPos12.y)) * w12.x * w12.y;
        result += smp(f2(texPos3.x, texPos12.y)) * w3.x * w12.y;
        result += smp(f2(texPos12.x, texPos3.y)) * w12.x * w3.y;
        result = result / (w12.x * w0.y + w0.x * w12.y + w12.x * w12.y + w3.x * w12.y + w12.x * w3.y);
        history0 = vmax(f4(0.0f), result) * history_mult;
    } else {
        const float4 qv = f4((quad_reproj_valid_packed & 1u) ? 1.0f : 0.0f, (quad_reproj_valid_packed & 2u) ? 1.0f : 0.0f, (quad_reproj_valid_packed & 4u) ? 1.0f : 0.0f, (quad_reproj_valid_packed & 8u) ? 1.0f : 0.0f);
        const float2 bp = (uv + xy(reproj)) * texSize - 0.5f;
        const float2 bw = vfrac(bp);
        const int ox = kjb_cvt_i32(kjb_trunc(bp.x)), oy = kjb_cvt_i32(kjb_trunc(bp.y));
        const float4 s00 = ld_rgba16f(ht, ox, oy) * history_mult, s10 = ld_rgba16f(ht, ox + 1, oy) * history_mult, s01 = ld_rgba16f(ht, ox, oy + 1) * history_mult, s11 = ld_rgba16f(ht, ox + 1, oy + 1) * history_mult;
        const float4 wts = f4((1.0f - bw.x) * (1.0f - bw.y), bw.x * (1.0f - bw.y), (1.0f - bw.x) * bw.y, bw.x * bw.y) * qv;
        if (dot(wts, f4(1.0f)) > 1e-5f) { const float4 rr = s00 * wts.x + s10 * wts.y + s01 * wts.z + s11 * wts.w; history0 = rr * kjb_rcp(dot(wts, f4(1.0f))); }
        else history0 = (s00 + s10 + s01 + s11) / 4.0f;
    }
    history0 = linear_to_working(history0);
    const float4 history1 = linear_to_working(bilinear_clamp(ht.w, ht.h, hit_prev_uv, [&](int sx, int sy) { return ld_rgba16f(ht, sx, sy); }) * history_mult);
    const float history1_valid = quad_reproj_valid_packed == 15u ? 1.0f : 0.0f;
    float4 vsum = f4(0.0f), vsum2 = f4(0.0f); float wsum = 0;
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
        const float sample_depth = s_depth[(ty + yy) * P4 + (tx + xx) + (R5_AX - 1)];
        const float4 neigh = s_work[(ty + yy) * R5_LW + (tx + xx)];
        float w = 1;
        w *= kjb_exp2(-200.0f * kjb_abs(center_depth / sample_depth - 1.0f));
        vsum = mad(neigh, w, vsum); vsum2 = mad(neigh * neigh, w, vsum2); wsum += w;
    }
    const float4 ex = vsum / wsum, ex2 = vsum2 / wsum;
    const float4 dev = vsqrt(vmax(f4(0.0f), ex2 - ex * ex));
    const GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, x, y));
    const float restir_invalidity = ld_r8u(t.invalidity_tex, x / 2, y / 2);
    const float n_deviations = kjb_lerp(reproj.z > 0 ? 2.0f : 1.25f, 0.625f, restir_invalidity);
    float wo_similarity;
    {
        const float3 current_wo = normalize(vrc.ray_hit_ws() - eye), prev_wo = normalize(vrc.ray_hit_ws() - prev_eye);
        const float clamped_roughness = kjb_max(0.1f, gbuffer.roughness);
        wo_similarity = kjb_pow(kjb_saturate(ggx_ndf_0_1(clamped_roughness * clamped_roughness, dot(current_wo, prev_wo))), 32.0f);
    }
    const float h0diff = length((xyz(history0) - xyz(ex)) / xyz(dev));
    const float h1diff = length((xyz(history1) - xyz(ex)) / xyz(dev));
    const float sqrt_rough = kjb_sqrt(gbuffer.roughness);
    float h0_score = 1.0f * kjb_smoothstep(0.0f, 0.5f, sqrt_rough) * kjb_lerp(wo_similarity, 1.0f, sqrt_rough);
    float h1_score = (1 - h0_score) * kjb_lerp(1.0f, kjb_smoothstep(0.0f, 1.0f, h0diff - h1diff), kjb_smoothstep(0.0f, 0.15f, sqrt_rough));
    h0_score *= history0_valid; h1_score *= history1_valid;
    const float score_sum = h0_score + h1_score;
    h0_score /= score_sum;
    h1_score = 1 - h0_score;
    if (!(h0_score < 1.001f)) { h0_score = 1; h1_score = 0; }
    const float4 clamped_history0 = f4(soft_color_clamp(xyz(center), xyz(history0), xyz(ex), xyz(dev) * n_deviations), history0.w);
    const float4 clamped_history1 = f4(soft_color_clamp(xyz(center), xyz(history1), xyz(ex), xyz(dev) * n_deviations), history1.w);
    const float4 clamped_history = clamped_history0 * h0_score + clamped_history1 * h1_score;
    const float max_sample_count = 16;
    const float current_sample_count = clamped_history.w * kjb_saturate(h0_score * history0_valid + h1_score * history1_valid);
    float4 res = vlerp(clamped_history, center, 1.0f / (1.0f + kjb_min(max_sample_count, current_sample_count * kjb_lerp(wo_similarity, 1.0f, 0.5f))));
    res.w = kjb_min(current_sample_count, max_sample_count) + 1;
    res = working_to_linear(res);
    st_rgba16f(t.output_tex, x, y, vmax(f4(0.0f), res));
}

// ------------------------------------------------------------------ R6 spatial_cleanup.hlsl:19-65
KJB_KERNEL(256) k_rtr_cleanup(const __grid_constant__ Globals g, Img input_tex, Img depth_tex, Img geometric_normal_tex, ImgW output_tex, const int32_t* offs, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float4 center = ld_rgba16f(input_tex, x, y);
    const float center_depth = ld_r32f(depth_tex, x, y);
    const float center_sample_count = center.w;
    if (center_sample_count >= 8.0f || center_depth == 0.0f) { st_r11g11b10(output_tex, x, y, xyz(center)); return; }
    const float3 center_normal_vs = ld_a2r10g10b10(geometric_normal_tex, x, y) * 2.0f - 1.0f;
    const float filter_radius_ss = 0.5f * vc.view_to_clip.m[5] / -depth_to_view_z(vc, center_depth);
    const uint32_t filter_idx = kjb_cvt_u32(kjb_clamp(filter_radius_ss * 7.0f, 0.0f, 7.0f));
    float3 vsum = f3(0.0f); float wsum = 0;
    int sc = kjb_cvt_i32(8.0f - center_sample_count / 2.0f); sc = sc < 2 ? 2 : (sc > 8 ? 8 : sc);
    const int kernel_scale = center_sample_count < 4 ? 2 : 1;
    const uint32_t px_idx_in_quad = (((uint32_t(x) & 1u) | (uint32_t(y) & 1u) * 2u) + g.fc.frame_index) & 3u;
    for (uint32_t sample_i = 0; sample_i < uint32_t(sc); ++sample_i) {
        const int32_t* o = offs + 4 * ((px_idx_in_quad * 16u + sample_i) + 64u * filter_idx);
        const int sx = x + kernel_scale * o[0], sy = y + kernel_scale * o[1];
        const float3 neigh = vsqrt(xyz(ld_rgba16f(input_tex, sx, sy)));   // linear_rgb_to_crunched_rgb
        const float sample_depth = ld_r32f(depth_tex, sx, sy);
        const float3 sample_normal_vs = ld_a2r10g10b10(geometric_normal_tex, sx, sy) * 2.0f - 1.0f;
        float w = 1;
        w *= kjb_exp2(-50.0f * kjb_abs(center_normal_vs.z * (center_depth / sample_depth - 1.0f)));
        const float dp = kjb_saturate(dot(center_normal_vs, sample_normal_vs));
        w *= dp * dp * dp;
        vsum = mad(neigh, w, vsum); wsum += w;
    }
    const float3 v = vsum / wsum;
    st_r11g11b10(output_tex, x, y, v * v);   // crunched_rgb_to_linear_rgb
}

// ================================================================== entry points
#define F4A(a) f4((a)[0], (a)[1], (a)[2], (a)[3])
#define CHK(img, fmt, name) if (!check_img(c, (img), (fmt), P, name)) return 1
#define CHKE(img, fmt, name, w, h) if (!check_img(c, (img), (fmt), P, name, (w), (h))) return 1

static int check_ircache_bindings(kjb_context* c, const char* P, const kjb_ircache_bindings& b, IrcacheBufs& out) {
    out = IrcacheBufs{};
    if (!b.meta_buf.data) return 0;
    const uint64_t E = KJB_IRCACHE_MAX_ENTRIES;
    const bool ok = b.meta_buf.size_bytes >= 32 && b.grid_meta_buf.data && b.grid_meta_buf.size_bytes >= 8ull * KJB_IRCACHE_GRID_CELLS && b.entry_cell_buf.data && b.entry_cell_buf.size_bytes >= 4 * E
        && b.spatial_buf.data && b.spatial_buf.size_bytes >= 16 * E && b.irradiance_buf.data && b.irradiance_buf.size_bytes >= 48 * E && b.life_buf.data && b.life_buf.size_bytes >= 4 * E
        && b.pool_buf.data && b.pool_buf.size_bytes >= 4 * E && b.reposition_proposal_buf.data && b.reposition_proposal_buf.size_bytes >= 16 * E
        && b.reposition_proposal_count_buf.data && b.reposition_proposal_count_buf.size_bytes >= 4 * E;
    if (!ok) return c->fail(std::string(P) + ": irradiance cache bindings are incomplete or too small");
    out = ircache_bufs(b);
    ircache_attach_parallel(c, out);
    return 0;
}

extern "C" {

int kjb_pass_rtr_trace(kjb_context* c, const kjb_rtr_trace_args* a) {
    const char* P = "reflection trace"; const uint32_t W = a->out0_tex.width, H = a->out0_tex.height;
    CHK(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex"); CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex"); CHK(a->rtdgi_tex, KJB_FMT_RGBA16_FLOAT, "rtdgi_tex"); CHK(a->sky_cube_tex, KJB_FMT_RGBA16_FLOAT, "sky_cube_tex");
    CHK(a->out0_tex, KJB_FMT_RGBA16_FLOAT, "out0_tex"); CHKE(a->out1_tex, KJB_FMT_RGBA16_FLOAT, "out1_tex", W, H); CHKE(a->out2_tex, KJB_FMT_RGBA8_SNORM, "out2_tex", W, H); CHKE(a->rng_out_tex, KJB_FMT_R32_UINT, "rng_out_tex", W, H);
    if (!c->tlas_valid) return c->fail("reflection trace: no acceleration structure (call kjb_rebuild_tlas)");
    BlueNoiseSamplerTables bn; bn.ranking = (const uint32_t*)a->ranking_tile_buf.data; bn.scrambling = (const uint32_t*)a->scambling_tile_buf.data; bn.sobol = (const uint32_t*)a->sobol_buf.data;
    if (bn.ranking || bn.scrambling || bn.sobol) {
        if (!(bn.ranking && bn.scrambling && bn.sobol) || a->ranking_tile_buf.size_bytes < 4ull * 128 * 128 * 8 || a->scambling_tile_buf.size_bytes < 4ull * 128 * 128 * 8 || a->sobol_buf.size_bytes < 4ull * 256 * 256)
            return c->fail("reflection trace: blue-noise-sampler tables must be all NULL or all present (i32[131072], i32[131072], i32[65536])");
    }
    IrcacheBufs ircache; if (check_ircache_bindings(c, P, a->ircache, ircache)) return 1;
    RtrTraceImgs t{img_ro(a->gbuffer_tex), img_ro(a->depth_tex), img_ro(a->rtdgi_tex), img_ro(a->sky_cube_tex), img_rw(a->out0_tex), img_rw(a->out1_tex), img_rw(a->out2_tex), img_rw(a->rng_out_tex)};
    KJB_ROWS(c, H);
    if (ircache.bound() && c->debug_serial) KJB_LAUNCH(c, k_rtr_trace_serial, KJB_DIMS(dim3(1), dim3(32)), c->g, t, bn, F4A(a->gbuffer_tex_size), a->reuse_rtdgi_rays, ircache);
    else if (ircache.bound()) KJB_LAUNCH_ORDERED(c, k_rtr_trace, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, t, bn, F4A(a->gbuffer_tex_size), a->reuse_rtdgi_rays, ircache);
    else KJB_LAUNCH(c, k_rtr_trace, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, t, bn, F4A(a->gbuffer_tex_size), a->reuse_rtdgi_rays, ircache);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtr_validate(kjb_context* c, const kjb_rtr_validate_args* a) {
    const char* P = "reflection validate"; const uint32_t W = a->refl_restir_invalidity_tex.width, H = a->refl_restir_invalidity_tex.height;
    CHK(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex"); CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex"); CHK(a->rtdgi_tex, KJB_FMT_RGBA16_FLOAT, "rtdgi_tex"); CHK(a->sky_cube_tex, KJB_FMT_RGBA16_FLOAT, "sky_cube_tex");
    CHK(a->refl_restir_invalidity_tex, KJB_FMT_R8_UNORM, "refl_restir_invalidity_tex"); CHKE(a->ray_orig_history_tex, KJB_FMT_RGBA32_FLOAT, "ray_orig_history_tex", W, H);
    CHKE(a->ray_history_tex, KJB_FMT_RGBA16_FLOAT, "ray_history_tex", W, H); CHKE(a->rng_history_tex, KJB_FMT_R32_UINT, "rng_history_tex", W, H);
    CHKE(a->irradiance_history_tex, KJB_FMT_RGBA16_FLOAT, "irradiance_history_tex", W, H); CHKE(a->reservoir_history_tex, KJB_FMT_RG32_UINT, "reservoir_history_tex", W, H);
    if (!c->tlas_valid) return c->fail("reflection validate: no acceleration structure (call kjb_rebuild_tlas)");
    IrcacheBufs ircache; if (check_ircache_bindings(c, P, a->ircache, ircache)) return 1;
    RtrValidateImgs t{img_ro(a->gbuffer_tex), img_ro(a->depth_tex), img_ro(a->rtdgi_tex), img_ro(a->sky_cube_tex), img_ro(a->ray_orig_history_tex), img_ro(a->ray_history_tex), img_ro(a->rng_history_tex),
                      img_rw(a->refl_restir_invalidity_tex), img_rw(a->irradiance_history_tex), img_rw(a->reservoir_history_tex)};
    const int QW = int((W + 1) / 2), QH = int((H + 1) / 2);   // dispatched over half_res() of the half-res image (rtr.rs:229)
    kjb::Rows kjb__rows = c->rows_for(H); kjb__rows.y0 = kjb__rows.y0 / 2; kjb__rows.y1 = (kjb__rows.y1 + 1) / 2;   // scissor (half-res rows) -> quad rows
    if (ircache.bound() && c->debug_serial) KJB_LAUNCH(c, k_rtr_validate_serial, KJB_DIMS(dim3(1), dim3(32)), c->g, t, F4A(a->gbuffer_tex_size), ircache, QW, QH);
    else if (ircache.bound()) KJB_LAUNCH_ORDERED(c, k_rtr_validate, KJB_GRID2D(QW, QH, KJB_RAY_BX, KJB_RAY_BY), c->g, t, F4A(a->gbuffer_tex_size), ircache, QW, QH);
    else KJB_LAUNCH(c, k_rtr_validate, KJB_GRID2D(QW, QH, KJB_RAY_BX, KJB_RAY_BY), c->g, t, F4A(a->gbuffer_tex_size), ircache, QW, QH);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtr_restir_temporal(kjb_context* c, const kjb_rtr_restir_temporal_args* a) {
    const char* P = "rtr restir temporal"; const uint32_t W = a->irradiance_out_tex.width, H = a->irradiance_out_tex.height;
    CHK(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex"); CHKE(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex", W, H); CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex");
    CHKE(a->candidate0_tex, KJB_FMT_RGBA16_FLOAT, "candidate0_tex", W, H); CHKE(a->candidate1_tex, KJB_FMT_RGBA16_FLOAT, "candidate1_tex", W, H); CHKE(a->candidate2_tex, KJB_FMT_RGBA8_SNORM, "candidate2_tex", W, H);
    CHKE(a->irradiance_history_tex, KJB_FMT_RGBA16_FLOAT, "irradiance_history_tex", W, H); CHKE(a->ray_orig_history_tex, KJB_FMT_RGBA32_FLOAT, "ray_orig_history_tex", W, H);
    CHKE(a->ray_history_tex, KJB_FMT_RGBA16_FLOAT, "ray_history_tex", W, H); CHKE(a->rng_history_tex, KJB_FMT_R32_UINT, "rng_history_tex", W, H); CHKE(a->reservoir_history_tex, KJB_FMT_RG32_UINT, "reservoir_history_tex", W, H);
    CHK(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex"); CHKE(a->hit_normal_history_tex, KJB_FMT_RGBA16_FLOAT, "hit_normal_history_tex", W, H);
    CHK(a->irradiance_out_tex, KJB_FMT_RGBA16_FLOAT, "irradiance_out_tex"); CHKE(a->ray_orig_output_tex, KJB_FMT_RGBA32_FLOAT, "ray_orig_output_tex", W, H); CHKE(a->ray_output_tex, KJB_FMT_RGBA16_FLOAT, "ray_output_tex", W, H);
    CHKE(a->rng_output_tex, KJB_FMT_R32_UINT, "rng_output_tex", W, H); CHKE(a->hit_normal_output_tex, KJB_FMT_RGBA16_FLOAT, "hit_normal_output_tex", W, H); CHKE(a->reservoir_out_tex, KJB_FMT_RG32_UINT, "reservoir_out_tex", W, H);
    RtrRestirTemporalImgs t{img_ro(a->gbuffer_tex), img_ro(a->half_view_normal_tex), img_ro(a->depth_tex), img_ro(a->candidate0_tex), img_ro(a->candidate1_tex), img_ro(a->candidate2_tex), img_ro(a->irradiance_history_tex),
                            img_ro(a->ray_orig_history_tex), img_ro(a->ray_history_tex), img_ro(a->rng_history_tex), img_ro(a->reservoir_history_tex), img_ro(a->reprojection_tex), img_ro(a->hit_normal_history_tex),
                            img_rw(a->irradiance_out_tex), img_rw(a->ray_orig_output_tex), img_rw(a->ray_output_tex), img_rw(a->rng_output_tex), img_rw(a->hit_normal_output_tex), img_rw(a->reservoir_out_tex)};
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_rtr_restir_temporal, KJB_GRID2D(W, H, 32, 8), c->g, t, F4A(a->gbuffer_tex_size));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtr_resolve(kjb_context* c, const kjb_rtr_resolve_args* a) {
    const char* P = "reflection resolve"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHKE(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H); CHK(a->hit1_tex, KJB_FMT_RGBA16_FLOAT, "hit1_tex");
    CHKE(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex", W, H); CHK(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex"); CHKE(a->ray_len_history_tex, KJB_FMT_RG16_FLOAT, "ray_len_history_tex", W, H);
    CHK(a->restir_irradiance_tex, KJB_FMT_RGBA16_FLOAT, "restir_irradiance_tex"); CHK(a->restir_ray_tex, KJB_FMT_RGBA16_FLOAT, "restir_ray_tex"); CHK(a->restir_reservoir_tex, KJB_FMT_RG32_UINT, "restir_reservoir_tex");
    CHK(a->restir_ray_orig_tex, KJB_FMT_RGBA32_FLOAT, "restir_ray_orig_tex"); CHK(a->output_tex, KJB_FMT_R11G11B10_UFLOAT, "output_tex"); CHKE(a->ray_len_output_tex, KJB_FMT_RG16_FLOAT, "ray_len_output_tex", W, H);
    RtrResolveImgs t{img_ro(a->gbuffer_tex), img_ro(a->depth_tex), img_ro(a->hit1_tex), img_ro(a->reprojection_tex), img_ro(a->half_view_normal_tex), img_ro(a->ray_len_history_tex), img_ro(a->restir_irradiance_tex),
                     img_ro(a->restir_ray_tex), img_ro(a->restir_reservoir_tex), img_ro(a->restir_ray_orig_tex), img_rw(a->output_tex), img_rw(a->ray_len_output_tex)};
    const float radius_sample_mult = 1.0f / kjb_pow(8.0f, 0.666f);   // RADIUS_SAMPLE_MULT: const-folded in the shader
    KJB_ROWS(c, H);
    ResolveTapAngles ta;
    {
        const float ang_offset = float(c->g.fc.frame_index * 59u % 128u) * KJB_PLASTIC;
        for (uint32_t q = 0; q < 4u; ++q) for (int sample_i = 1; sample_i <= 8; ++sample_i) {
            const float ang = (float(sample_i) + ang_offset) * KJB_GOLDEN_ANGLE + (float(q) / 4.0f) * KJB_TAU_F;
            kjb_sincos(ang, &ta.sn[q * 8u + uint32_t(sample_i - 1)], &ta.cs[q * 8u + uint32_t(sample_i - 1)]);
        }
    }
    KJB_LAUNCH(c, k_rtr_resolve, KJB_GRID2D(W, H, 32, 8), c->g, t, F4A(a->output_tex_size), radius_sample_mult, ta);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtr_temporal(kjb_context* c, const kjb_rtr_temporal_args* a) {
    const char* P = "reflection temporal"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHKE(a->input_tex, KJB_FMT_R11G11B10_UFLOAT, "input_tex", W, H); CHKE(a->history_tex, KJB_FMT_RGBA16_FLOAT, "history_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H);
    CHKE(a->ray_len_tex, KJB_FMT_RG16_FLOAT, "ray_len_tex", W, H); CHKE(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex", W, H); CHK(a->refl_restir_invalidity_tex, KJB_FMT_R8_UNORM, "refl_restir_invalidity_tex");
    CHKE(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex", W, H); CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex");
    RtrTemporalImgs t{img_ro(a->input_tex), img_ro(a->history_tex), img_ro(a->depth_tex), img_ro(a->ray_len_tex), img_ro(a->reprojection_tex), img_ro(a->refl_restir_invalidity_tex), img_ro(a->gbuffer_tex), img_rw(a->output_tex)};
    KJB_ROWS(c, H);
    const TileSource ts_in = tile_source(c, a->input_tex, R5_TW, R5_TH), ts_depth = tile_source(c, a->depth_tex, R5_TW, R5_TH);
    KJB_LAUNCH_SYNC(c, k_rtr_temporal, KJB_GRID2D(W, H, 32, 8), ts_in, ts_depth, tile_mode({&ts_in, &ts_depth}), c->g, t, F4A(a->output_tex_size));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtr_cleanup(kjb_context* c, const kjb_rtr_cleanup_args* a) {
    const char* P = "reflection cleanup"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHKE(a->input_tex, KJB_FMT_RGBA16_FLOAT, "input_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H); CHKE(a->geometric_normal_tex, KJB_FMT_A2R10G10B10_UNORM, "geometric_normal_tex", W, H);
    CHK(a->output_tex, KJB_FMT_R11G11B10_UFLOAT, "output_tex");
    if (!a->spatial_resolve_offsets) return c->fail("reflection cleanup: spatial_resolve_offsets is null");
    // the constants tuple of the pass (rtr.rs:395): 8 KB, uploaded once per distinct table
    if (!c->d_resolve_offsets) { c->d_resolve_offsets = (int32_t*)dev_alloc(sizeof(int32_t) * 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT); if (!c->d_resolve_offsets) return c->fail("reflection cleanup: out of memory"); }
    if (c->h_resolve_offsets.size() != 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT || memcmp(c->h_resolve_offsets.data(), a->spatial_resolve_offsets, sizeof(int32_t) * 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT) != 0) {
        c->h_resolve_offsets.assign(a->spatial_resolve_offsets, a->spatial_resolve_offsets + 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT);
        if (dev_h2d(c, c->d_resolve_offsets, c->h_resolve_offsets.data(), sizeof(int32_t) * 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT)) return c->fail("reflection cleanup: upload failed");
    }
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_rtr_cleanup, KJB_GRID2D(W, H, 32, 8), c->g, img_ro(a->input_tex), img_ro(a->depth_tex), img_ro(a->geometric_normal_tex), img_rw(a->output_tex), (const int32_t*)c->d_resolve_offsets);
    KJB_PASS_EPILOGUE(c, P);
}

}  // extern "C"
