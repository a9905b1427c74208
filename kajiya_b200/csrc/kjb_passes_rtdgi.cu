// Ray-traced diffuse GI (rtdgi) as sm_90a kernels — one kernel per render-graph pass of
// crates/lib/kajiya/src/renderers/rtdgi.rs, shader sources under /root/reference/assets/shaders/rtdgi/.
// Thread mapping: 32x8 blocks on the pass's pixel grid (a warp = 32 consecutive pixels of one row, so the 4/8/16-byte
// texels of every bound image are fetched as 128/256/512-byte contiguous requests); the two ray-tracing passes use
// 16x8 blocks (register pressure of the traversal stack + BRDF state).  Neighbourhood taps go through L1/L2: the
// half-res working set at 1080p (~40 MB for all ReSTIR state) is largely L2-resident on H100 (50 MB).
#include "kjb_context.h"
#include "kjb_ircache.cuh"

using namespace kjb;

#define SKY_DIST 1e4f
#define RESTIR_TEMPORAL_M_CLAMP 20.0f
#define RESTIR_RESERVOIR_W_CLAMP 10.0f
#define SSGI_NEAR_FIELD_RADIUS 80.0f

KJB_DEV bool is_validation_frame(const Globals& g) { return g.fc.frame_index % 3u == 0u; }   // rtdgi_restir_settings.hlsl:40-46
KJB_DEV bool is_tracing_frame(const Globals& g) { return !is_validation_frame(g); }

struct TemporalReservoirOutput { float depth; float3 ray_hit_offset_ws; float luminance; float3 hit_normal_ws; };   // rtdgi_common.hlsl:12-39
KJB_DEV TemporalReservoirOutput tro_from_raw(uint4 raw) {
    const float2 a = unpack_2x16f(raw.y), b = unpack_2x16f(raw.z);
    TemporalReservoirOutput r; r.depth = kjb_u2f(raw.x); r.ray_hit_offset_ws = f3(a.x, a.y, b.x); r.luminance = b.y; r.hit_normal_ws = unpack_normal_11_10_11(raw.w);
    return r;
}

struct TraceResult { float3 out_value, hit_normal_ws; float hit_t, pdf; bool is_hit; };

// rtdgi/diffuse_trace_common.inc.hlsl:38-221
KJB_DEV TraceResult do_the_thing(const Globals& g, const Img& depth_tex, const Img& reprojected_gi_tex, const Img& sky_cube_tex, const float* gbuffer_tex_size,
                                 uint32_t px, uint32_t py, float3 normal_ws, uint32_t& rng, const Ray& outgoing_ray, const IrcacheBufs& ircache) {
    const kjb_view_constants& vc = g.fc.view_constants;
    float3 total_radiance = f3(0.0f);
    float3 hit_normal_ws = -outgoing_ray.dir;
    float hit_t = outgoing_ray.tmax;
    const float pdf = kjb_max(0.0f, 1.0f / (dot(normal_ws, outgoing_ray.dir) * 2 * KJB_PI_F));

    RayCone cone; cone.width = 0; cone.spread_angle = pixel_cone_spread_angle_from_image_height(vc, gbuffer_tex_size[1] * 0.5f);
    cone = ray_cone_propagate(cone, 0.03f, length(outgoing_ray.origin - get_eye_position(vc)));

    const GbufferPathVertex primary_hit = gbuffer_raytrace(g, outgoing_ray, cone, 1, false);
    if (primary_hit.is_hit) {
        hit_t = primary_hit.ray_t;
        GbufferData gbuffer = gbuffer_unpack(primary_hit.gbuffer_packed);
        hit_normal_ws = gbuffer.normal;

        const float3 primary_hit_cs = position_world_to_sample(vc, primary_hit.position);
        const float2 primary_hit_uv = cs_to_uv(xy(primary_hit_cs));
        const int2 dpx = nearest_clamp_px(depth_tex, primary_hit_uv);
        const float primary_hit_screen_depth = ld_r32f(depth_tex, dpx.x, dpx.y);
        bool is_on_screen = kjb_abs(primary_hit_cs.x) < 1.0f && kjb_abs(primary_hit_cs.y) < 1.0f
            && inverse_depth_relative_diff(primary_hit_cs.z, primary_hit_screen_depth) < 5e-3f;
        float4 reprojected_radiance = f4(0.0f);
        if (is_on_screen) {
            const int2 rpx = nearest_clamp_px(reprojected_gi_tex, primary_hit_uv);
            reprojected_radiance = ld_rgba16f(reprojected_gi_tex, rpx.x, rpx.y) * g.fc.pre_exposure_delta;
            is_on_screen = reprojected_radiance.w > 0;
        }
        gbuffer.roughness = kjb_lerp(gbuffer.roughness, 1.0f, 0.5f);
        const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
        const float3 wo = mul(-outgoing_ray.dir, tangent_to_world);
        const LayeredBrdf brdf = layered_brdf_from_gbuffer_ndotv(g, gbuffer, wo.z);

        const float3 sun_radiance = f3(g.sun_color[0], g.sun_color[1], g.sun_color[2]);
        if (sun_radiance.x != 0.0f || sun_radiance.y != 0.0f || sun_radiance.z != 0.0f) {
            const float3 to_light_norm = sample_sun_direction(g.fc, xy(blue_noise_for_pixel(g, px, py, rng)), false);
            const bool is_shadowed = rt_is_shadowed(g, primary_hit.position, to_light_norm, 1e-4f, SKY_DIST);
            const float3 wi = mul(to_light_norm, tangent_to_world);
            const float3 brdf_value = layered_evaluate(brdf, wo, wi) * kjb_max(0.0f, wi.z);
            const float3 light_radiance = is_shadowed ? f3(0.0f) : sun_radiance;
            total_radiance += brdf_value * light_radiance;
        }
        total_radiance += gbuffer.emissive;
        if (is_on_screen) {
            total_radiance += xyz(reprojected_radiance) * gbuffer.albedo;
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
                    const bool is_shadowed = rt_is_shadowed(g, primary_hit.position, to_light_norm_ws, 1e-3f, kjb_sqrt(dist_to_light2) - 2e-3f);
                    const float3 bounce_albedo = vlerp(gbuffer.albedo, f3(1.0f), 0.04f);
                    const float3 brdf_value = bounce_albedo * to_psa_metric / KJB_PI_F;
                    total_radiance += !is_shadowed ? (f3(tl.radiance[0], tl.radiance[1], tl.radiance[2]) * brdf_value / ls.pdf) : f3(0.0f);
                }
            }
            // USE_IRCACHE: the lookup contributes 0 when no cache is bound (kjb_ircache_bindings.meta_buf == NULL)
            total_radiance += ircache_lookup<false>(g, ircache, outgoing_ray.origin, primary_hit.position, gbuffer.normal, 1, rng) * gbuffer.albedo;
        }
    } else {
        total_radiance += xyz(sample_cube_rgba16f(sky_cube_tex, outgoing_ray.dir));
    }
    TraceResult r; r.out_value = total_radiance; r.hit_t = hit_t; r.hit_normal_ws = hit_normal_ws; r.pdf = pdf; r.is_hit = primary_hit.is_hit;
    return r;
}

// ------------------------------------------------------------------ D1 fullres_reproject.hlsl:29-77
KJB_DEV float4 cubic_hermite(float4 A, float4 B, float4 C, float4 D, float t) {   // inc/curve.hlsl:4-13
    const float t2 = t * t, t3 = t * t * t;
    const float4 a = -A / 2.0f + (3.0f * B) / 2.0f - (3.0f * C) / 2.0f + D / 2.0f;
    const float4 b = A - (5.0f * B) / 2.0f + 2.0f * C - D / 2.0f;
    const float4 c = -A / 2.0f + C / 2.0f;
    return a * t3 + b * t2 + c * t + B;
}
KJB_KERNEL(256) k_rtdgi_reproject(Img input_tex, Img reprojection_tex, ImgW output_tex, float4 ots, Rows kjb_rows) {
    KJB_PX; const int W = output_tex.w, H = output_tex.h; if (x >= W || y >= H) return;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float4 reproj = ld_rgba16s(reprojection_tex, x, y);
    const float2 prev_uv = uv + xy(reproj);
    const uint32_t quad_valid = uint32_t(reproj.z * 15.0f + 0.5f);
    float4 history = f4(0.0f);
    if (quad_valid == 15u) {
        // GatherBlue footprint of a bilinear fetch at uv + 0.5 * sign(prev_uv) * texel: all four must be fully valid
        const float2 guv = uv + 0.5f * f2(kjb_sign(prev_uv.x), kjb_sign(prev_uv.y)) * f2(ots.z, ots.w);
        const int gx0 = kjb_cvt_i32(kjb_floor(guv.x * float(W) - 0.5f)), gy0 = kjb_cvt_i32(kjb_floor(guv.y * float(H) - 0.5f));
        bool all_valid = true;
        for (int j = 0; j < 2; ++j) for (int i = 0; i < 2; ++i)
            if (uint32_t(ld_rgba16s(reprojection_tex, clampi(gx0 + i, W), clampi(gy0 + j, H)).z * 15.0f + 0.5f) != 15u) all_valid = false;
        if (all_valid) {   // image_sample_catmull_rom (inc/image.hlsl:42-79)
            const float2 pixel = prev_uv * f2(float(W), float(H)) + 0.5f;
            const float2 frc = vfrac(pixel);
            const int ix = kjb_cvt_i32(pixel.x) - 1, iy = kjb_cvt_i32(pixel.y) - 1;
            float4 rows[4];
            for (int j = 0; j < 4; ++j)
                rows[j] = cubic_hermite(ld_rgba16f(input_tex, ix - 1, iy - 1 + j), ld_rgba16f(input_tex, ix, iy - 1 + j), ld_rgba16f(input_tex, ix + 1, iy - 1 + j), ld_rgba16f(input_tex, ix + 2, iy - 1 + j), frc.x);
            history = vmax(f4(0.0f), cubic_hermite(rows[0], rows[1], rows[2], rows[3], frc.y));
        } else {
            history = bilinear_clamp(W, H, prev_uv, [&](int sx, int sy) { return ld_rgba16f(input_tex, sx, sy); });
        }
    } else if (quad_valid != 0u) {
        const float4 qv = f4((quad_valid & 1u) ? 1.0f : 0.0f, (quad_valid & 2u) ? 1.0f : 0.0f, (quad_valid & 4u) ? 1.0f : 0.0f, (quad_valid & 8u) ? 1.0f : 0.0f);
        const float2 bp = prev_uv * f2(ots.x, ots.y) - 0.5f;
        const float2 bw = vfrac(bp);
        const int ox = kjb_cvt_i32(kjb_trunc(bp.x)), oy = kjb_cvt_i32(kjb_trunc(bp.y));
        const float4 s00 = ld_rgba16f(input_tex, ox, oy), s10 = ld_rgba16f(input_tex, ox + 1, oy), s01 = ld_rgba16f(input_tex, ox, oy + 1), s11 = ld_rgba16f(input_tex, ox + 1, oy + 1);
        const float4 wts = f4((1.0f - bw.x) * (1.0f - bw.y), bw.x * (1.0f - bw.y), (1.0f - bw.x) * bw.y, bw.x * bw.y) * qv;
        if (dot(wts, f4(1.0f)) > 1e-5f) {
            const float4 r = s00 * wts.x + s10 * wts.y + s01 * wts.z + s11 * wts.w;
            history = r * kjb_rcp(dot(wts, f4(1.0f)));
        }
    }
    st_rgba16f(output_tex, x, y, history);
}

// ------------------------------------------------------------------ D3 diffuse_validate.rgen.hlsl:46-111
KJB_DEV void rtdgi_validate_px(const Globals& g, const Img& half_view_normal_tex, const Img& depth_tex, const Img& reprojected_gi_tex, const ImgW& reservoir_tex, const Img& reservoir_ray_history_tex,
                               const Img& sky_cube_tex, const ImgW& irradiance_history_tex, const Img& ray_orig_history_tex, const ImgW& out_tex, float4 gts, const IrcacheBufs& ircache, int x, int y) {
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    if (0.0f == ld_r32f(depth_tex, x * 2 + hso.x, y * 2 + hso.y)) { st_r8u(out_tex, x, y, 1.0f); return; }
    float invalidity = 0.0f;
    if (is_validation_frame(g)) {
        const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
        const float3 normal_ws = direction_view_to_world(vc, xyz(ld_rgba8s(half_view_normal_tex, x, y)));
        const float3 prev_ray_orig = xyz(ld_rgba32f(ray_orig_history_tex, x, y));
        const float3 prev_hit_pos = xyz(ld_rgba16f(reservoir_ray_history_tex, x, y)) + prev_ray_orig;
        const float4 prev_radiance_packed = ld_rgba16f(as_ro(irradiance_history_tex), x, y);
        const float3 prev_radiance = vmax(f3(0.0f), xyz(prev_radiance_packed));
        Ray prev_ray; prev_ray.dir = normalize(prev_hit_pos - prev_ray_orig); prev_ray.origin = prev_ray_orig; prev_ray.tmin = 0; prev_ray.tmax = SKY_DIST;
        uint32_t rng = hash3(uint32_t(x), uint32_t(y), 0u);
        const TraceResult result = do_the_thing(g, depth_tex, reprojected_gi_tex, sky_cube_tex, s4, uint32_t(x), uint32_t(y), normal_ws, rng, prev_ray, ircache);
        const float3 new_radiance = vmax(f3(0.0f), result.out_value);
        const float rad_diff = length(vabs(prev_radiance - new_radiance) / vmax(f3(1e-3f), prev_radiance + new_radiance));
        invalidity = kjb_smoothstep(0.1f, 0.5f, rad_diff / length(f3(1.0f)));
        const float prev_hit_dist = length(prev_hit_pos - prev_ray_orig);
        if (kjb_abs(result.hit_t - prev_hit_dist) / (prev_hit_dist + prev_hit_dist) < 0.2f) {
            st_rgba16f(irradiance_history_tex, x, y, f4(new_radiance, prev_radiance_packed.w));
            Reservoir r = Reservoir::from_raw(ld_rg32u(as_ro(reservoir_tex), x, y));
            const float lum_old = luminance(prev_radiance), lum_new = luminance(new_radiance);
            r.M *= kjb_clamp(lum_old / kjb_max(1e-8f, lum_new), 0.03f, 1.0f);
            r.W *= kjb_clamp(lum_old / kjb_max(1e-8f, lum_new) * 10.0f, 0.01f, 1.0f);
            st_rg32u(reservoir_tex, x, y, r.as_raw());
        }
    }
    st_r8u(out_tex, x, y, invalidity);
}
#ifndef KJB_OCC_VALIDATE
#define KJB_OCC_VALIDATE 8   /* 64 registers */
#endif
template <bool SERIAL>   // SERIAL: the serial schedule's form (KJB_PIXELS, kjb_context.h)
KJB_KERNEL_OCC(128, KJB_OCC_VALIDATE) k_rtdgi_validate(const __grid_constant__ Globals g, Img half_view_normal_tex, Img depth_tex, Img reprojected_gi_tex, ImgW reservoir_tex, Img reservoir_ray_history_tex,
                                 Img sky_cube_tex, ImgW irradiance_history_tex, Img ray_orig_history_tex, ImgW out_tex, float4 gts, IrcacheBufs ircache, Rows kjb_rows) {
    KJB_PIXELS(SERIAL, out_tex.w, out_tex.h, rtdgi_validate_px(g, half_view_normal_tex, depth_tex, reprojected_gi_tex, reservoir_tex, reservoir_ray_history_tex, sky_cube_tex, irradiance_history_tex,
                                                                ray_orig_history_tex, out_tex, gts, ircache, x, y));
}

// ------------------------------------------------------------------ D4 trace_diffuse.rgen.hlsl:49-120
KJB_DEV void rtdgi_trace_px(const Globals& g, const Img& half_view_normal_tex, const Img& depth_tex, const Img& reprojected_gi_tex, const Img& reprojection_tex, const Img& sky_cube_tex,
                            const ImgW& cand_irr, const ImgW& cand_normal, const ImgW& cand_hit, const Img& inv_in, const ImgW& inv_out, float4 gts, const IrcacheBufs& ircache, int x, int y) {
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const int hx = x * 2 + hso.x, hy = y * 2 + hso.y;
    const float depth = ld_r32f(depth_tex, hx, hy);
    if (0.0f == depth) {
        st_rgba16f(cand_irr, x, y, f4(0.0f)); st_rgba8s(cand_normal, x, y, f4(0, 0, 1, 0)); st_r8u(inv_out, x, y, 0.0f);
        return;
    }
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float2 uv = get_uv(hx, hy, s4);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_biased_depth(vc, uv, depth);
    const float NEAR_FIELD_FADE_OUT_END = -vrc.ray_hit_vs().z * (SSGI_NEAR_FIELD_RADIUS * gts.w * 0.5f);
    {
        const float3 normal_ws = direction_view_to_world(vc, xyz(ld_rgba8s(half_view_normal_tex, x, y)));
        const float3x3 tangent_to_world = build_orthonormal_basis(normal_ws);
        const float2 urand = xy(blue_noise_for_pixel(g, uint32_t(x), uint32_t(y), g.fc.frame_index));   // candidate_ray_dir.hlsl
        const float3 outgoing_dir = mul(tangent_to_world, uniform_sample_hemisphere(urand));
        Ray outgoing_ray; outgoing_ray.dir = outgoing_dir; outgoing_ray.origin = vrc.biased_secondary_ray_origin_ws_with_normal(normal_ws);
        outgoing_ray.tmin = 0; outgoing_ray.tmax = is_tracing_frame(g) ? SKY_DIST : NEAR_FIELD_FADE_OUT_END;
        uint32_t rng = hash3(uint32_t(x), uint32_t(y), g.fc.frame_index & 31u);
        TraceResult result = do_the_thing(g, depth_tex, reprojected_gi_tex, sky_cube_tex, s4, uint32_t(x), uint32_t(y), normal_ws, rng, outgoing_ray, ircache);
        if (!is_tracing_frame(g) && !result.is_hit) { result.out_value = f3(0.0f); result.hit_t = SKY_DIST; }
        const float3 hit_offset_ws = outgoing_ray.dir * result.hit_t;
        const float cos_theta = dot(normalize(outgoing_dir - vrc.ray_dir_ws()), normal_ws);
        st_rgba16f(cand_irr, x, y, f4(result.out_value, 1 - cos_theta));
        st_rgba16f(cand_hit, x, y, f4(hit_offset_ws, result.pdf * (is_tracing_frame(g) ? 1.0f : -1.0f)));
        st_rgba8s(cand_normal, x, y, f4(direction_world_to_view(vc, result.hit_normal_ws), 0));
    }
    const float4 reproj = ld_rgba16s(reprojection_tex, hx, hy);
    const int rx = kjb_cvt_i32(kjb_floor(float(x) + gts.x * reproj.x / 2 + 0.5f)), ry = kjb_cvt_i32(kjb_floor(float(y) + gts.y * reproj.y / 2 + 0.5f));
    st_r8u(inv_out, x, y, ld_r8u(inv_in, rx, ry));
}
#ifndef KJB_OCC_TRACE
#define KJB_OCC_TRACE 8   /* 64 registers */
#endif
template <bool SERIAL>
KJB_KERNEL_OCC(128, KJB_OCC_TRACE) k_rtdgi_trace(const __grid_constant__ Globals g, Img half_view_normal_tex, Img depth_tex, Img reprojected_gi_tex, Img reprojection_tex, Img sky_cube_tex,
                              ImgW cand_irr, ImgW cand_normal, ImgW cand_hit, Img inv_in, ImgW inv_out, float4 gts, IrcacheBufs ircache, Rows kjb_rows) {
    KJB_PIXELS(SERIAL, cand_irr.w, cand_irr.h, rtdgi_trace_px(g, half_view_normal_tex, depth_tex, reprojected_gi_tex, reprojection_tex, sky_cube_tex, cand_irr, cand_normal, cand_hit, inv_in, inv_out, gts, ircache, x, y));
}

// ------------------------------------------------------------------ D5 temporal_validity_integrate.hlsl:21-119
// The shader exchanges values between lanes of its 8x8 group (WaveReadLaneAt ^2, ^16, ^1, ^8; lane = x + 8*y in 32-wide waves):
// partners are pixels (x^2,y), (x,y^2), (x^1,y), (x,y^1).  Blocks are 8 x 32 threads whose rows start at a multiple of 4, so a warp is
// exactly the shader's wave — an 8x4 pixel patch with lane = x + 8*(y & 3) — and the four exchanges are warp shuffles (SHFL.BFLY 2, 16,
// 1, 8 and their combinations); every thread computes ITS pre-exchange blur / edge value first (threads past the image edge included,
// like the shader's out-of-range lanes).  The 5x5 blur reads the R8 input from a (8+4)x(32+4) tile decoded once per texel.
struct Weights25v { float w[25]; float w_sum; };   // w[(yy+2)*5+(xx+2)] = exp2(-0.1 r^2) and their float sum in tap order, host-evaluated
KJB_DEV float d5_edge(const Img& reprojection_tex, const Img& half_depth_tex, int x, int y) {
    const float center_depth = ld_r32f(half_depth_tex, x, y);
    float edge = 1;
    for (int yy = 0; yy <= 2; ++yy) for (int xx = 1; xx <= 2; ++xx) {
        const float4 reproj = ld_rgba16s(reprojection_tex, x * 2 + xx, y * 2 + yy);
        const float sample_depth = ld_r32f(half_depth_tex, x + xx / 2, y + yy / 2);
        if (reproj.w < 0 || inverse_depth_relative_diff(center_depth, sample_depth) > 0.1f) { edge = 0; break; }
        edge *= (reproj.z == 0 && sample_depth != 0) ? 1.0f : 0.0f;
    }
    return edge;
}
#define D5_BX 8
#define D5_BY 32
KJB_KERNEL(256) k_rtdgi_validity_integrate(const __grid_constant__ Globals g, Img input_tex, Img history_tex, Img reprojection_tex, Img half_depth_tex, ImgW output_tex, float4 gts, Weights25v wt, Rows kjb_rows) {
    __shared__ float in_tile[D5_BY + 4][D5_BX + 4];
    const int tx = int(threadIdx.x), ty = int(threadIdx.y);
    const int bx0 = int(blockIdx.x) * D5_BX, by0 = (kjb_rows.y0 & ~3) + int(blockIdx.y) * D5_BY;
    const int x = bx0 + tx, y = by0 + ty;
    for (int i = ty * D5_BX + tx; i < (D5_BY + 4) * (D5_BX + 4); i += D5_BX * D5_BY) {
        const int lx = i % (D5_BX + 4), ly = i / (D5_BX + 4);
        in_tile[ly][lx] = ld_r8u(input_tex, bx0 + lx - 2, by0 + ly - 2);
    }
    __syncthreads();
    float blur, edge;
    {
        float acc = 0.0f;
        for (int yy = 0; yy < 5; ++yy) for (int xx = 0; xx < 5; ++xx) acc = mad(in_tile[ty + yy][tx + xx], wt.w[yy * 5 + xx], acc);
        blur = acc / wt.w_sum;
        edge = d5_edge(reprojection_tex, half_depth_tex, x, y);
    }
    // lane = tx + 8 * (ty & 3): x^2 -> lane^2, y^2 -> lane^16, x^1 -> lane^1, y^1 -> lane^8
    const float b0 = kjb_lerp(blur, warp_xor(blur, 2), 0.5f);
    const float b1 = kjb_lerp(warp_xor(blur, 16), warp_xor(blur, 18), 0.5f);
    const float e0 = kjb_max(edge, warp_xor(edge, 1));
    const float e1 = kjb_max(warp_xor(edge, 8), warp_xor(edge, 9));
    if (x >= output_tex.w || y >= output_tex.h || y < kjb_rows.y0 || y >= kjb_rows.y1) return;
    float inv = kjb_lerp(b0, b1, 0.5f);
    inv = kjb_smoothstep(0.0f, 1.0f, inv);
    inv += kjb_max(e0, e1);
    inv = kjb_saturate(inv);
    const float4 reproj = ld_rgba16s(reprojection_tex, x * 2, y * 2);
    const float2 reproj_px = f2(float(x), float(y)) + f2(gts.x, gts.y) * xy(reproj) / 2.0f + 0.5f;
    float history = 0;
    const float ang_off = u01(hash3(uint32_t(x), uint32_t(y), g.fc.frame_index)) * KJB_PI_F * 2;
    for (uint32_t i = 0; i < 8u; ++i) {
        const float ang = (float(i) + ang_off) * KJB_GOLDEN_ANGLE;
        float s, c; kjb_sincos(ang, &s, &c);
        const float2 off = f2(c, s) * (float(i) * 1.0f);
        history += ld_rg16f(history_tex, kjb_cvt_i32(reproj_px.x + off.x), kjb_cvt_i32(reproj_px.y + off.y)).x;
    }
    history /= 8.0f;
    st_rg16f(output_tex, x, y, kjb_max(history * 0.75f, inv), in_tile[ty + 2][tx + 2]);
}

// ------------------------------------------------------------------ D6 restir_temporal.hlsl:83-422
struct RestirTemporalImgs {
    Img half_view_normal_tex, depth_tex, candidate_radiance_tex, candidate_normal_tex, candidate_hit_tex, radiance_history_tex, ray_orig_history_tex, ray_history_tex,
        reservoir_history_tex, reprojection_tex, hit_normal_history_tex, candidate_history_tex, rt_invalidity_tex;
    ImgW radiance_out_tex, ray_orig_output_tex, ray_output_tex, hit_normal_output_tex, reservoir_out_tex, candidate_out_tex, temporal_reservoir_packed_tex;
};
#ifndef KJB_OCC_RESTIR_TEMPORAL
#define KJB_OCC_RESTIR_TEMPORAL 4   /* 64 registers */
#endif
KJB_KERNEL_OCC(256, KJB_OCC_RESTIR_TEMPORAL) k_rtdgi_restir_temporal(const __grid_constant__ Globals g, RestirTemporalImgs t, float4 gts, float4* positions, Rows kjb_rows) {
    KJB_PX; if (x >= t.radiance_out_tex.w || y >= t.radiance_out_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const uint32_t frame_index = g.fc.frame_index;
    const int2 hso = halfres_subsample_offset(frame_index);
    const int hx = x * 2 + hso.x, hy = y * 2 + hso.y;
    const float depth = ld_r32f(t.depth_tex, hx, hy);
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float2 uv = get_uv(hx, hy, s4);
    if (0.0f == depth) {
        st_rgba16f(t.radiance_out_tex, x, y, f4(0, 0, 0, -SKY_DIST)); st_rgba8u(t.hit_normal_output_tex, x, y, f4(0.0f)); st_rg32u(t.reservoir_out_tex, x, y, u2(0, 0));
        // temporal_reservoir_packed_tex keeps its old texel here (as in the shader): the cached position is that of the old depth word
        if (positions) positions[y * t.radiance_out_tex.w + x] = f4(hit_ws_from_uv_depth(vc, uv, kjb_u2f(ld_rgba32u(as_ro(t.temporal_reservoir_packed_tex), x, y).x)), 0.0f);
        return;
    }
    // KJB_OPTION_HALF_RES_POSITION_CACHE: what k_half_res_positions would compute from the depth word written below
    if (positions) positions[y * t.radiance_out_tex.w + x] = f4(hit_ws_from_uv_depth(vc, uv, depth), 0.0f);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_biased_depth(vc, uv, depth);
    const float3 normal_vs = xyz(ld_rgba8s(t.half_view_normal_tex, x, y));
    const float3 normal_ws = direction_view_to_world(vc, normal_vs);
    const float3 refl_ray_origin_ws = vrc.biased_secondary_ray_origin_ws_with_normal(normal_ws);
    const float3 hit_offset_ws = xyz(ld_rgba16f(t.candidate_hit_tex, x, y));
    float3 outgoing_dir = normalize(hit_offset_ws);
    uint32_t rng = hash3(uint32_t(x), uint32_t(y), frame_index);

    float3 radiance_sel = f3(0.0f), ray_orig_sel_ws = f3(0.0f), ray_hit_sel_ws = f3(1.0f), hit_normal_sel = f3(1.0f);
    StreamState stream_state; stream_state.p_q_sel = 0; stream_state.M_sum = 0;
    Reservoir reservoir = Reservoir::create();
    const uint32_t reservoir_payload = uint32_t(x) | (uint32_t(y) << 16);

    if (is_tracing_frame(g)) {
        const float hit_t = length(hit_offset_ws);
        const float3 out_value = xyz(ld_rgba16f(t.candidate_radiance_tex, x, y));
        const float3 cand_hit_normal_ws = direction_view_to_world(vc, xyz(ld_rgba8s(t.candidate_normal_tex, x, y)));
        const float p_q = 1.0f * kjb_max(0.0f, luminance(out_value)) * kjb_step(0.0f, dot(outgoing_dir, normal_ws));
        radiance_sel = out_value; ray_orig_sel_ws = refl_ray_origin_ws; ray_hit_sel_ws = refl_ray_origin_ws + outgoing_dir * hit_t; hit_normal_sel = cand_hit_normal_ws;
        reservoir.init_with_stream(p_q, 1.0f, stream_state, reservoir_payload);
        const float rl = kjb_lerp(ld_rgba16f(t.candidate_history_tex, x, y).y, kjb_sqrt(hit_t), 0.05f);
        st_rgba16f(t.candidate_out_tex, x, y, f4(kjb_sqrt(hit_t), rl, 0, 0));
    }
    const float rt_invalidity = kjb_sqrt(kjb_saturate(ld_rg16f(t.rt_invalidity_tex, x, y).y));
    float center_M = 0;

    for (uint32_t sample_i = 0; sample_i < 5u && stream_state.M_sum < 1.25f * RESTIR_TEMPORAL_M_CLAMP; ++sample_i) {
        // get_rpx_offset (:64-81)
        int ox = 0, oy = 0;
        if (sample_i != 0) {
            const uint32_t ia = frame_index & 3u, ib = (sample_i + (frame_index ^ 1u)) & 3u;
            // offsets = {(-1,-1),(1,1),(-1,1),(1,-1)}
            ox = ((ia == 1u || ia == 3u) ? 1 : -1) + ((ib == 1u || ib == 3u) ? 1 : -1);
            oy = ((ia == 1u || ia == 2u) ? 1 : -1) + ((ib == 1u || ib == 2u) ? 1 : -1);
            if (ox == 0 && oy == 0) continue;
        }
        const float4 reproj = ld_rgba16s(t.reprojection_tex, hx + ox * 2, hy + oy * 2);
        // xor_seq = {(3,3),(2,1),(1,2),(3,3)}[frame & 3]
        const uint32_t fi = frame_index & 3u;
        const uint32_t xv = (fi == 1u) ? 2u : ((fi == 2u) ? 1u : 3u), yv = (fi == 1u) ? 1u : ((fi == 2u) ? 2u : 3u);
        const uint32_t perm_x = (uint32_t(x) + uint32_t(ox)) ^ xv, perm_y = (uint32_t(y) + uint32_t(oy)) ^ yv;
        const float base_x = sample_i == 0 ? float(uint32_t(x)) : float(perm_x), base_y = sample_i == 0 ? float(uint32_t(y)) : float(perm_y);
        const int prx = kjb_cvt_i32(kjb_floor(base_x + gts.x * reproj.x * 0.5f + 0.0f + 0.5f)), pry = kjb_cvt_i32(kjb_floor(base_y + gts.y * reproj.y * 0.5f + 0.0f + 0.5f));
        const int rpx_x = int(uint32_t(prx) + uint32_t(ox)), rpx_y = int(uint32_t(pry) + uint32_t(oy));
        const int pnx = kjb_cvt_i32(kjb_floor(base_x + 0.5f)), pny = kjb_cvt_i32(kjb_floor(base_y + 0.5f));
        const int npx = int(uint32_t(pnx) + uint32_t(ox)), npy = int(uint32_t(pny) + uint32_t(oy));
        const int nhx = int(uint32_t(npx) * 2u + uint32_t(hso.x)), nhy = int(uint32_t(npy) * 2u + uint32_t(hso.y));

        Reservoir r = Reservoir::from_raw(ld_rg32u(t.reservoir_history_tex, rpx_x, rpx_y));
        const int spx_x = int(r.payload & 0xffffu), spx_y = int(r.payload >> 16);
        float relevance = 1;
        const float sample_depth = ld_r32f(t.depth_tex, nhx, nhy);
        const float3 prev_ray_orig = xyz(ld_rgba32f(t.ray_orig_history_tex, spx_x, spx_y));
        if (length(prev_ray_orig - refl_ray_origin_ws) > 0.1f * -vrc.ray_hit_vs().z) continue;
        if (0 == sample_depth) continue;
        if (reproj.z == 0) continue;
        relevance *= 1 - kjb_smoothstep(0.0f, 0.1f, inverse_depth_relative_diff(depth, sample_depth));
        const float3 sample_normal_vs = xyz(ld_rgba8s(t.half_view_normal_tex, npx, npy));
        const float normal_similarity_dot = kjb_max(0.0f, dot(sample_normal_vs, normal_vs));
        if (sample_i != 0 && normal_similarity_dot < 0.2f) continue;
        relevance *= kjb_pow(normal_similarity_dot, 4.0f);

        const float4 sample_hit_ws_and_dist = ld_rgba16f(t.ray_history_tex, spx_x, spx_y) + f4(prev_ray_orig, 0.0f);
        const float3 sample_hit_ws = xyz(sample_hit_ws_and_dist);
        const float prev_dist = sample_hit_ws_and_dist.w;
        const float4 hn = ld_rgba8u(t.hit_normal_history_tex, spx_x, spx_y);
        const float4 sample_hit_normal_ws_dot = f4(hn.x * 2 - 1, hn.y * 2 - 1, hn.z * 2 - 1, hn.w);
        const float3 dir_to_sample_hit_unnorm = sample_hit_ws - refl_ray_origin_ws;
        const float dist_to_sample_hit = length(dir_to_sample_hit_unnorm);
        const float3 dir_to_sample_hit = normalize(dir_to_sample_hit_unnorm);
        const float center_to_hit_vis = -dot(xyz(sample_hit_normal_ws_dot), dir_to_sample_hit);
        const float ped = g.fc.pre_exposure_delta;
        const float4 prev_rad = ld_rgba16f(t.radiance_history_tex, spx_x, spx_y) * f4(ped, ped, ped, 1);
        r.M = kjb_max(0.0f, kjb_min(r.M, kjb_exp2(kjb_log2(RESTIR_TEMPORAL_M_CLAMP) * (1.0f - rt_invalidity))));
        const float p_q = 1 * kjb_max(0.0f, luminance(xyz(prev_rad))) * kjb_step(0.0f, dot(dir_to_sample_hit, normal_ws));
        float jacobian = 1;
        jacobian *= kjb_clamp(prev_dist / dist_to_sample_hit, 1e-4f, 1e4f);
        jacobian *= jacobian;
        jacobian *= kjb_clamp(center_to_hit_vis / sample_hit_normal_ws_dot.w, 0.0f, 1e4f);
        r.M *= relevance;
        if (0 == sample_i) center_M = r.M;
        if (reservoir.update_with_stream(r, p_q, jacobian * 1.0f, stream_state, reservoir_payload, rng)) {
            outgoing_dir = dir_to_sample_hit; radiance_sel = xyz(prev_rad); ray_orig_sel_ws = prev_ray_orig; ray_hit_sel_ws = sample_hit_ws;
            hit_normal_sel = xyz(sample_hit_normal_ws_dot);
        }
    }
    reservoir.finish_stream(stream_state);
    reservoir.W = kjb_min(reservoir.W, RESTIR_RESERVOIR_W_CLAMP);
    reservoir.M = center_M + 0.5f;

    const float4 hit_normal_ws_dot = f4(hit_normal_sel, -dot(hit_normal_sel, outgoing_dir));
    st_rgba16f(t.radiance_out_tex, x, y, f4(radiance_sel, dot(normal_ws, outgoing_dir)));
    st_rgba32f(t.ray_orig_output_tex, x, y, f4(ray_orig_sel_ws, 0.0f));
    st_rgba8u(t.hit_normal_output_tex, x, y, f4(hit_normal_ws_dot.x * 0.5f + 0.5f, hit_normal_ws_dot.y * 0.5f + 0.5f, hit_normal_ws_dot.z * 0.5f + 0.5f, hit_normal_ws_dot.w));
    st_rgba16f(t.ray_output_tex, x, y, f4(ray_hit_sel_ws - ray_orig_sel_ws, length(ray_hit_sel_ws - refl_ray_origin_ws)));
    st_rg32u(t.reservoir_out_tex, x, y, reservoir.as_raw());
    const float3 rho = ray_hit_sel_ws - vrc.ray_hit_ws();
    st_rgba32u(t.temporal_reservoir_packed_tex, x, y, u4(kjb_f2u(depth), pack_2x16f(rho.x, rho.y), pack_2x16f(rho.z, kjb_max(0.0f, luminance(radiance_sel))),
                                                         pack_normal_11_10_11(xyz(hit_normal_ws_dot))));
}

// ------------------------------------------------------------------ half-res world positions (KJB_OPTION_HALF_RES_POSITION_CACHE)
// D7 and D9 evaluate hit_ws_from_uv_depth(get_uv(p * 2 + hso), depth(p)) for 16 / 8 neighbours p of every pixel, with depth(p) taken from
// half_depth_tex or from the depth word of temporal_reservoir_packed_tex.  One small kernel evaluates it once per half-res pixel and
// source; the passes then load the 16-byte result (L2 hits) — the very same function of the very same inputs, hence the same bits.
struct PosView { const float4* p; int w, h; };
KJB_DEV float3 cached_or_hit_ws(const PosView& pv, const kjb_view_constants& vc, int px, int py, float2 uv, float depth) {
    if (pv.p && (unsigned)px < (unsigned)pv.w && (unsigned)py < (unsigned)pv.h) return xyz(pv.p[py * pv.w + px]);
    return hit_ws_from_uv_depth(vc, uv, depth);
}
KJB_KERNEL(256) k_half_res_positions(const __grid_constant__ Globals g, Img src, int packed, float4* out, float4 gts, Rows kjb_rows) {
    KJB_PX; if (x >= src.w || y >= src.h) return;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float depth = packed ? kjb_u2f(ld_rgba32u(src, x, y).x) : ld_r32f(src, x, y);
    out[y * src.w + x] = f4(hit_ws_from_uv_depth(g.fc.view_constants, get_uv(x * 2 + hso.x, y * 2 + hso.y, s4), depth), 0.0f);
}
static PosView ensure_positions(kjb_context* c, kjb_context::PosCache& pc, uint64_t epoch, const kjb_image& src, bool packed, const float* gts) {
    PosView none; none.p = nullptr; none.w = 0; none.h = 0;
    if (!c->opt_position_cache) return none;
    const bool fresh = pc.epoch == epoch && pc.src == src.data && pc.w == src.width && pc.h == src.height && memcmp(pc.gts, gts, 16) == 0;
    if (!fresh) {
        const size_t need = size_t(src.width) * src.height * sizeof(float4);
        if (pc.cap < need) { dev_sync(c); dev_free(pc.d); pc.d = (float4*)dev_alloc(need); pc.cap = pc.d ? need : 0; if (!pc.d) return none; }
        const kjb::Rows kjb__rows = {0, int(src.height)};
        KJB_LAUNCH(c, k_half_res_positions, KJB_GRID2D(src.width, src.height, 32, 8), c->g, img_ro(src), packed ? 1 : 0, pc.d, f4(gts[0], gts[1], gts[2], gts[3]));
        pc.epoch = epoch; pc.src = src.data; pc.w = src.width; pc.h = src.height; memcpy(pc.gts, gts, 16);
    }
    PosView v; v.p = pc.d; v.w = int(src.width); v.h = int(src.height);
    return v;
}

// ------------------------------------------------------------------ D7 restir_spatial.hlsl:48-372 + occlusion_raymarch.hlsl:69-146
KJB_DEV float normal_influence_nonlinearity(float x, float b) { return x < -b ? 0.0f : (x + b) * (x + b) / (4 * b); }
#ifndef KJB_OCC_RESTIR_SPATIAL
#define KJB_OCC_RESTIR_SPATIAL 1   /* 77 registers, uncapped */
#endif
KJB_KERNEL_OCC(256, KJB_OCC_RESTIR_SPATIAL) k_rtdgi_restir_spatial(const __grid_constant__ Globals g, Img reservoir_input_tex, Img half_view_normal_tex, Img half_depth_tex, Img half_ssao_tex, Img temporal_reservoir_packed_tex,
                                       ImgW reservoir_output_tex, float4 gts, float4 ots, uint32_t pass_idx, uint32_t perform_occlusion_raymarch, uint32_t importance_only, PosView pos_a, PosView pos_b, Rows kjb_rows) {
    // The tap angles `(sample_i + ang_offset) * GOLDEN_ANGLE` depend on the pixel only through its 8x8 (pass 0) / 4x4 (later passes) screen tile
    // (ang_offset = hash of the tile): a 32x8 block covers at most 4x2 / 8x3 such tiles, so the block evaluates each tile's 8 / 5 sin-cos pairs
    // once into shared memory (<= 120 kjb_sincos per block instead of 8 / 5 per pixel) and every pixel reads its tile's row.
    __shared__ float s_sn[24 * 8], s_cs[24 * 8];
    const uint32_t sample_count = pass_idx == 0 ? 8u : 5u;
    const int tshift = pass_idx == 0 ? 3 : 2;
    const int bx0 = int(blockIdx.x * blockDim.x), by0 = kjb_rows.y0 + int(blockIdx.y * blockDim.y);
    const int tiles_x = int(blockDim.x) >> tshift, tile_y0 = by0 >> tshift;
    {
        const int tiles_y = ((by0 + int(blockDim.y) - 1) >> tshift) - tile_y0 + 1;
        for (int i = int(threadIdx.y * blockDim.x + threadIdx.x); i < tiles_x * tiles_y * int(sample_count); i += int(blockDim.x * blockDim.y)) {
            const int sample_i = i % int(sample_count), tile = i / int(sample_count);
            const uint32_t tsx = uint32_t((bx0 >> tshift) + tile % tiles_x), tsy = uint32_t(tile_y0 + tile / tiles_x);
            const float ang_offset_t = u01(hash3(tsx, tsy, g.fc.frame_index * 2u + pass_idx)) * KJB_PI_F * 2;
            kjb_sincos((float(sample_i) + ang_offset_t) * KJB_GOLDEN_ANGLE, &s_sn[tile * 8 + sample_i], &s_cs[tile * 8 + sample_i]);
        }
        __syncthreads();
    }
    KJB_PX; if (x >= reservoir_output_tex.w || y >= reservoir_output_tex.h) return;
    const int my_tile = ((y >> tshift) - tile_y0) * tiles_x + ((x >> tshift) - (bx0 >> tshift));
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float depth = ld_r32f(half_depth_tex, x, y);
    uint32_t rng = hash3(uint32_t(x), uint32_t(y), g.fc.frame_index + pass_idx * 123u);
    const float2 uv = get_uv(x * 2 + hso.x, y * 2 + hso.y, s4);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_depth(vc, uv, depth);
    const float3 center_hit_ws = vrc.ray_hit_ws(), center_hit_vs = vrc.ray_hit_vs();
    const float3 center_normal_vs = xyz(ld_rgba8s(half_view_normal_tex, x, y));
    const float3 center_normal_ws = direction_view_to_world(vc, center_normal_vs);
    const float center_depth = depth;
    const float center_ssao = ld_r8s(half_ssao_tex, x, y);

    StreamState stream_state; stream_state.p_q_sel = 0; stream_state.M_sum = 0;
    Reservoir reservoir = Reservoir::create();
    const float sample_radius_offset = rand01(rng);
    const Reservoir center_r = Reservoir::from_raw(ld_rg32u(reservoir_input_tex, x, y));
    float kernel_tightness = 1.0f - center_ssao;
    const float MAX_INPUT_M_IN_PASS = pass_idx == 0 ? RESTIR_TEMPORAL_M_CLAMP : RESTIR_TEMPORAL_M_CLAMP * 8.0f;
    kernel_tightness = kjb_lerp(kernel_tightness, 1.0f, 0.5f * kjb_smoothstep(MAX_INPUT_M_IN_PASS * 0.5f, MAX_INPUT_M_IN_PASS, center_r.M));
    float max_kernel_radius = pass_idx == 0 ? kjb_lerp(32.0f, 12.0f, kernel_tightness) : kjb_lerp(16.0f, 6.0f, kernel_tightness);
    if (pass_idx >= 2) max_kernel_radius = 8;
    const float2 dist_to_edge_xy = vmin(f2(float(x), float(y)), f2(ots.x, ots.y) - f2(float(x), float(y)));
    const float allow_edge_overstep = center_r.M < 10 ? 100.0f : 1.25f;
    const float2 kernel_radius = vmin(f2(max_kernel_radius), dist_to_edge_xy * allow_edge_overstep);

    for (uint32_t sample_i = 0; sample_i < sample_count; ++sample_i) {
        const float2 radius = 0 == sample_i ? f2(0.0f) : (kjb_pow((float(sample_i) + sample_radius_offset) / float(sample_count), 0.5f) * kernel_radius);
        const float sn = s_sn[my_tile * 8 + int(sample_i)], cs = s_cs[my_tile * 8 + int(sample_i)];
        const float2 off_f = f2(cs, sn) * radius;
        const int rx = x + kjb_cvt_i32(off_f.x), ry = y + kjb_cvt_i32(off_f.y);
        const bool is_center_sample = sample_i == 0;
        const uint2 reservoir_raw = ld_rg32u(reservoir_input_tex, rx, ry);
        if (0 == reservoir_raw.x) continue;
        Reservoir r = Reservoir::from_raw(reservoir_raw);
        r.M = kjb_min(r.M, 500.0f);
        const int spx_x = int(r.payload & 0xffffu), spx_y = int(r.payload >> 16);
        const TemporalReservoirOutput spx_packed = tro_from_raw(ld_rgba32u(temporal_reservoir_packed_tex, spx_x, spx_y));
        const float reused_luminance = spx_packed.luminance;
        float visibility = 1, relevance = 1;
        const float3 sample_normal_vs = xyz(ld_rgba8s(half_view_normal_tex, rx, ry));
        const float normal_similarity_dot = dot(sample_normal_vs, center_normal_vs);
        relevance *= normal_influence_nonlinearity(normal_similarity_dot, 0.5f) / normal_influence_nonlinearity(1.0f, 0.5f);
        const float sample_ssao = ld_r8s(half_ssao_tex, rx, ry);
        relevance *= 1 - kjb_abs(sample_ssao - center_ssao);
        const float2 rpx_uv = get_uv(rx * 2 + hso.x, ry * 2 + hso.y, s4);
        const float rpx_depth = ld_r32f(half_depth_tex, rx, ry);
        if (rpx_depth == 0.0f) continue;
        const float3 rpx_hit_ws = cached_or_hit_ws(pos_a, vc, rx, ry, rpx_uv, rpx_depth);
        const float2 spx_uv = get_uv(spx_x * 2 + hso.x, spx_y * 2 + hso.y, s4);
        const float3 sample_hit_ws = spx_packed.ray_hit_offset_ws + cached_or_hit_ws(pos_b, vc, spx_x, spx_y, spx_uv, spx_packed.depth);
        const float3 reused_dir_unnorm = sample_hit_ws - rpx_hit_ws;
        const float reused_dist = length(reused_dir_unnorm);
        const float3 reused_dir_to_sample_hit_ws = reused_dir_unnorm / reused_dist;
        const float3 dir_to_sample_hit_unnorm = sample_hit_ws - center_hit_ws;
        const float dist_to_sample_hit = length(dir_to_sample_hit_unnorm);
        const float3 dir_to_sample_hit = normalize(dir_to_sample_hit_unnorm);
        if (!is_center_sample) {
            const float depth_diff = kjb_abs(kjb_max(0.3f, center_normal_vs.z) * (center_depth / rpx_depth - 1.0f));
            relevance *= 1 - kjb_smoothstep(0.0f, pass_idx == 0 ? 0.15f : 0.1f, depth_diff);
        }
        if (perform_occlusion_raymarch) {
            const float surface_offset_len = length(hit_vs_from_uv_depth(vc, spx_uv, depth) - center_hit_vs);
            const float3 raymarch_dir_unnorm_ws = sample_hit_ws - center_hit_ws;
            const float3 raymarch_end_ws = center_hit_ws + raymarch_dir_unnorm_ws * kjb_min(1.0f, 3.0f * surface_offset_len / length(raymarch_dir_unnorm_ws));
            const float3 raymarch_start_cs = xyz(vrc.ray_hit_cs);
            const float3 raymarch_end_cs = position_world_to_clip(vc, raymarch_end_ws);
            const float2 raymarch_len_px = (cs_to_uv(xy(raymarch_end_cs)) - uv) * f2(ots.x, ots.y);
            int k_count = kjb_cvt_i32(kjb_floor(length(raymarch_len_px) / 2.0f));
            if (k_count > 6) k_count = 6;
            const float depth_step_per_z = (raymarch_end_cs.z - raymarch_start_cs.z) / length(xy(raymarch_end_cs) - xy(raymarch_start_cs));
            const float t_step = 1.0f / float(k_count);
            const float rcp_gts_x = 1.0f / gts.x, rcp_gts_y = 1.0f / gts.y;
            float tt = 0.5f * t_step;
            for (int k = 0; k < k_count; ++k) {
                const float3 interp_pos_cs = vlerp(raymarch_start_cs, raymarch_end_cs, tt);
                const float2 uv_at_interp = cs_to_uv(xy(interp_pos_cs));
                const uint32_t pix = (kjb_cvt_u32(kjb_floor(uv_at_interp.x * gts.x - float(hso.x))) & ~1u) + uint32_t(hso.x);
                const uint32_t piy = (kjb_cvt_u32(kjb_floor(uv_at_interp.y * gts.y - float(hso.y))) & ~1u) + uint32_t(hso.y);
                const float depth_at_interp = ld_r32f(half_depth_tex, int(pix >> 1u), int(piy >> 1u));
                // (texel centre) / (texture size): positive finite numerators over a per-thread constant divisor, see kjb_div_int_const
                const float2 quantized_cs = uv_to_cs(f2(kjb_div_int_const(float(pix) + 0.5f, gts.x, rcp_gts_x), kjb_div_int_const(float(piy) + 0.5f, gts.y, rcp_gts_y)));
                const float biased_interp_z = raymarch_start_cs.z + depth_step_per_z * length(quantized_cs - xy(raymarch_start_cs));
                if (depth_at_interp > biased_interp_z) {
                    const float depth_diff = inverse_depth_relative_diff(interp_pos_cs.z, depth_at_interp);
                    visibility *= 1 - kjb_smoothstep(0.05f, 0.05f * 0.5f, depth_diff);
                }
                tt += t_step;
            }
        }
        const float center_to_hit_vis = -dot(spx_packed.hit_normal_ws, dir_to_sample_hit);
        const float reused_to_hit_vis = -dot(spx_packed.hit_normal_ws, reused_dir_to_sample_hit_ws);
        float p_q = 1;
        p_q *= reused_luminance;
        p_q *= kjb_max(0.0f, dot(dir_to_sample_hit, center_normal_ws));
        float jacobian = 1;
        jacobian *= reused_dist / dist_to_sample_hit;
        jacobian *= jacobian;
        jacobian *= kjb_clamp(center_to_hit_vis / reused_to_hit_vis, 0.0f, 1e4f);
        jacobian = kjb_sqrt(jacobian);
        if (is_center_sample) jacobian = 1;
        if (!(p_q >= 0)) continue;
        r.M *= relevance;
        if (importance_only) { p_q *= kjb_lerp(0.25f, 1.0f, visibility); visibility = 1; }
        reservoir.update_with_stream(r, p_q, visibility * jacobian, stream_state, r.payload, rng);
    }
    reservoir.finish_stream(stream_state);
    reservoir.W = kjb_min(reservoir.W, RESTIR_RESERVOIR_W_CLAMP);
    st_rg32u(reservoir_output_tex, x, y, reservoir.as_raw());
}

// ------------------------------------------------------------------ D8 restir_check.rgen.hlsl:21-66 (optional)
KJB_KERNEL(128) k_rtdgi_restir_check(const __grid_constant__ Globals g, Img half_depth_tex, Img temporal_reservoir_packed_tex, ImgW reservoir_input_tex, float4 gts, Rows kjb_rows) {
    KJB_PX; if (x >= reservoir_input_tex.w || y >= reservoir_input_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float depth = ld_r32f(half_depth_tex, x, y);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_biased_depth(vc, get_uv(x * 2 + hso.x, y * 2 + hso.y, s4), depth);
    Reservoir r = Reservoir::from_raw(ld_rg32u(as_ro(reservoir_input_tex), x, y));
    const int spx_x = int(r.payload & 0xffffu), spx_y = int(r.payload >> 16);
    const TemporalReservoirOutput spx_packed = tro_from_raw(ld_rgba32u(temporal_reservoir_packed_tex, spx_x, spx_y));
    const ViewRayContext spx_ctx = ViewRayContext::from_uv_and_depth(vc, get_uv(spx_x * 2 + hso.x, spx_y * 2 + hso.y, s4), spx_packed.depth);
    const float3 spx_pos_ws = spx_ctx.ray_hit_ws();
    const float3 hit_ws = spx_packed.ray_hit_offset_ws + spx_pos_ws;
    const float3 trace_origin_ws = vrc.biased_secondary_ray_origin_ws();
    const float3 trace_vec = hit_ws - trace_origin_ws;
    if (rt_is_shadowed(g, trace_origin_ws, normalize(trace_vec), 0.0f, kjb_min(5 * length(spx_pos_ws - trace_origin_ws), length(trace_vec) * 0.999f))) {
        r.W = 0;
        st_rg32u(reservoir_input_tex, x, y, r.as_raw());
    }
}

// ------------------------------------------------------------------ D9 restir_resolve.hlsl:42-205
KJB_DEV float ggx_ndf_unnorm(float a2, float cos_theta) { const float ds = cos_theta * cos_theta * (a2 - 1.0f) + 1.0f; return a2 / (ds * ds); }
struct ResolveImgs { Img radiance_tex, reservoir_input_tex, gbuffer_tex, depth_tex, half_view_normal_tex, half_depth_tex, ssao_tex, candidate_radiance_tex, candidate_hit_tex, temporal_reservoir_packed_tex; };
struct PowTable4 { float v[4]; };   // v[i] = pow(float(i), 0.666), host-evaluated
#ifndef KJB_OCC_RESTIR_RESOLVE
#define KJB_OCC_RESTIR_RESOLVE 5   /* 48 registers, 5 blocks/SM */
#endif
KJB_KERNEL_OCC(256, KJB_OCC_RESTIR_RESOLVE) k_rtdgi_restir_resolve(const __grid_constant__ Globals g, ResolveImgs t, ImgW irradiance_output_tex, float4 gts, float4 ots, PowTable4 pw, PosView pos_a, PosView pos_b, Rows kjb_rows) {
    KJB_PX; if (x >= irradiance_output_tex.w || y >= irradiance_output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float depth = ld_r32f(t.depth_tex, x, y);
    if (0 == depth) { st_rgba16f(irradiance_output_tex, x, y, f4(0.0f)); return; }
    const float2 uv = get_uv(x, y, s4);
    const float3 center_hit_ws = hit_ws_from_uv_depth(vc, uv, depth);
    const float center_hit_vs_z = hit_vs_from_uv_depth(vc, uv, depth).z;
    const GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, x, y));
    const float3 center_normal_ws = gbuffer.normal;
    const float3 center_normal_vs = direction_world_to_view(vc, center_normal_ws);
    const float center_depth = depth;
    const float center_ssao = ld_r8u(t.ssao_tex, x, y);
    const uint32_t frame_hash = hash1(g.fc.frame_index);
    const uint32_t px_idx_in_quad = (((uint32_t(x) & 1u) | (uint32_t(y) & 1u) * 2u) + frame_hash) & 3u;
    const float4 blue = blue_noise_for_pixel(g, uint32_t(x), uint32_t(y), g.fc.frame_index) * KJB_TAU_F;
    const float NEAR_FIELD_FADE_OUT_END = -center_hit_vs_z * (SSGI_NEAR_FIELD_RADIUS * ots.w * 0.5f);
    const float NEAR_FIELD_FADE_OUT_START = NEAR_FIELD_FADE_OUT_END * 0.5f;
    const float near_field_influence = center_ssao;

    // both tap loops use the same four angles: evaluate their sin/cos once
    float tap_sn[4], tap_cs[4];
    for (uint32_t i = 0; i < 4u; ++i) {
        const float ang = (float(i) + blue.x) * KJB_GOLDEN_ANGLE + (float(px_idx_in_quad) / 4.0f) * KJB_TAU_F;
        kjb_sincos(ang, &tap_sn[i], &tap_cs[i]);
    }
    float3 total_irradiance = f3(0.0f);
    bool sharpen_gi_kernel = false;
    {
        float w_sum = 0; float3 weighted_irradiance = f3(0.0f);
        for (uint32_t i = 0; i < 4u; ++i) {
            const float radius = pw.v[i] * 1.0f + 0.4f;
            const float sn = tap_sn[i], cs = tap_cs[i];
            const float2 off = f2(cs, sn) * radius;
            const int rx = kjb_cvt_i32(kjb_floor(float(x) * 0.5f + off.x)), ry = kjb_cvt_i32(kjb_floor(float(y) * 0.5f + off.y));
            const float2 rpx_uv = get_uv(rx * 2 + hso.x, ry * 2 + hso.y, s4);
            const float rpx_depth = ld_r32f(t.half_depth_tex, rx, ry);
            const float3 hit_ws = xyz(ld_rgba16f(t.candidate_hit_tex, rx, ry)) + cached_or_hit_ws(pos_a, vc, rx, ry, rpx_uv, rpx_depth);
            const float3 sample_offset = hit_ws - center_hit_ws;
            const float sample_dist = length(sample_offset);
            const float3 sample_dir = sample_offset / sample_dist;
            const float geometric_term = 2 * kjb_max(0.0f, dot(center_normal_ws, sample_dir));
            const float atten = kjb_smoothstep(NEAR_FIELD_FADE_OUT_END, NEAR_FIELD_FADE_OUT_START, sample_dist);
            sharpen_gi_kernel |= atten > 0.9f;
            float3 contribution = xyz(ld_rgba16f(t.candidate_radiance_tex, rx, ry)) * geometric_term;
            contribution *= kjb_lerp(0.0f, atten, near_field_influence);
            const float3 sample_normal_vs = xyz(ld_rgba8s(t.half_view_normal_tex, rx, ry));
            float w = 1;
            w *= ggx_ndf_unnorm(0.01f, kjb_saturate(dot(center_normal_vs, sample_normal_vs)));
            w *= kjb_exp2(-200.0f * kjb_abs(center_normal_vs.z * (center_depth / rpx_depth - 1.0f)));
            weighted_irradiance = mad(contribution, w, weighted_irradiance);
            w_sum += w;
        }
        total_irradiance += weighted_irradiance / kjb_max(1e-20f, w_sum);
    }
    {
        float w_sum = 0; float3 weighted_irradiance = f3(0.0f);
        const float kernel_scale = sharpen_gi_kernel ? 0.5f : 1.0f;
        for (uint32_t i = 0; i < 4u; ++i) {
            const float radius = pw.v[i] * 1.0f * kernel_scale + 0.4f * kernel_scale;
            const float sn = tap_sn[i], cs = tap_cs[i];
            const float2 off = f2(cs, sn) * radius;
            const int rx = kjb_cvt_i32(kjb_floor(float(x) * 0.5f + off.x)), ry = kjb_cvt_i32(kjb_floor(float(y) * 0.5f + off.y));
            const Reservoir r = Reservoir::from_raw(ld_rg32u(t.reservoir_input_tex, rx, ry));
            const int spx_x = int(r.payload & 0xffffu), spx_y = int(r.payload >> 16);
            const TemporalReservoirOutput spx_packed = tro_from_raw(ld_rgba32u(t.temporal_reservoir_packed_tex, spx_x, spx_y));
            const float2 spx_uv = get_uv(spx_x * 2 + hso.x, spx_y * 2 + hso.y, s4);
            const float rpx_depth = ld_r32f(t.half_depth_tex, rx, ry);
            const float3 hit_ws = spx_packed.ray_hit_offset_ws + cached_or_hit_ws(pos_b, vc, spx_x, spx_y, spx_uv, spx_packed.depth);
            const float3 sample_offset = hit_ws - center_hit_ws;
            const float sample_dist = length(sample_offset);
            const float3 sample_dir = sample_offset / sample_dist;
            const float geometric_term = 2 * kjb_max(0.0f, dot(center_normal_ws, sample_dir));
            float3 radiance = xyz(ld_rgba16f(t.radiance_tex, spx_x, spx_y));
            const float atten = kjb_smoothstep(NEAR_FIELD_FADE_OUT_START, NEAR_FIELD_FADE_OUT_END, sample_dist);
            radiance *= kjb_lerp(1.0f, atten, near_field_influence);
            const float3 contribution = radiance * geometric_term * r.W;
            const float3 sample_normal_vs = xyz(ld_rgba8s(t.half_view_normal_tex, spx_x, spx_y));
            const float sample_ssao = ld_r8u(t.ssao_tex, rx * 2 + hso.x, ry * 2 + hso.y);
            float w = 1;
            w *= ggx_ndf_unnorm(0.01f, kjb_saturate(dot(center_normal_vs, sample_normal_vs)));
            w *= kjb_exp2(-200.0f * kjb_abs(center_normal_vs.z * (center_depth / rpx_depth - 1.0f)));
            w *= kjb_exp2(-20.0f * kjb_abs(center_ssao - sample_ssao));
            weighted_irradiance = mad(contribution, w, weighted_irradiance);
            w_sum += w;
        }
        total_irradiance += weighted_irradiance / kjb_max(1e-20f, w_sum);
    }
    st_rgba16f(irradiance_output_tex, x, y, f4(total_irradiance, 1));
}

// ------------------------------------------------------------------ D10 temporal_filter.hlsl:39-252
// 5x5 moments over two images.  Each CTA stages its (32+4)x(16+4) footprint of BOTH images in shared memory already
// converted to the crunched luma-chroma working space (sRGB->YCbCr, sqrt, divide), so the conversion runs once per texel
// instead of once per tap (25x fewer), and the 50 taps per pixel become LDS instead of L1 requests.  The 25 Gaussian
// weights exp(-3 r^2 / 9) are evaluated once on the host with the contract's kjb_exp and arrive as a kernel parameter.
struct Weights25 { float w[25]; float w_sum; };   // w_sum: the float sum of w[] in tap order (what the shader's `wsum += w` arrives at), host-evaluated
#define D10_BX 32
#define D10_BY 16
#define D10_TW (D10_BX + 4)
#define D10_TH (D10_BY + 4)
KJB_KERNEL(512) k_rtdgi_temporal(int tile_mode_, Globals g, Img input_tex, Img history_tex,
                                 Img variance_history_tex, Img reprojection_tex, Img rt_history_invalidity_tex,
                                 ImgW output_tex, ImgW history_output_tex, ImgW variance_history_output_tex, float4 ots, Weights25 wt, Rows kjb_rows) {
    constexpr int PR = tile_pitch<8>(D10_TW);
    __shared__ __align__(128) uint2 s_raw_in[PR * D10_TH];      // the two RGBA16F footprints as the copy engine delivers them (tile origin x = 32k - 2: 16-byte aligned)
    __shared__ __align__(128) uint2 s_raw_hist[PR * D10_TH];
    __shared__ float4 s_in[D10_TH * D10_TW];
    __shared__ float s_hist_luma[D10_TH * D10_TW];
    __shared__ __align__(8) uint64_t bar;
    const int W = output_tex.w, H = output_tex.h;
    const int bx0 = int(blockIdx.x) * D10_BX - 2, by0 = kjb_rows.y0 + int(blockIdx.y) * D10_BY - 2;
    const float ped = g.fc.pre_exposure_delta;
    const float4 history_mult = f4(ped, ped, ped, 1);
    const int tid = int(threadIdx.y) * D10_BX + int(threadIdx.x);
    tile_group_begin(&bar, 0, tile_mode_, tid);
    uint32_t staged = tile_issue<uint2, D10_TW, D10_TH>(s_raw_in, input_tex, bx0, by0, &bar, tile_mode_, tid, D10_BX * D10_BY);
    staged += tile_issue<uint2, D10_TW, D10_TH>(s_raw_hist, history_tex, bx0, by0, &bar, tile_mode_, tid, D10_BX * D10_BY);
    tile_group_wait(&bar, 0, tile_mode_, staged, tid);
    for (int i = tid; i < D10_TW * D10_TH; i += D10_BX * D10_BY) {
        const int tx = i % D10_TW, ty = i / D10_TW;
        s_in[i] = linear_to_working(half4_to_float4(s_raw_in[ty * PR + tx]));
        s_hist_luma[i] = linear_to_working(half4_to_float4(s_raw_hist[ty * PR + tx]) * history_mult).x;
    }
    __syncthreads();
    const int x = int(blockIdx.x) * D10_BX + int(threadIdx.x), y = kjb_rows.y0 + int(blockIdx.y) * D10_BY + int(threadIdx.y);
    if (x >= W || y >= H || y >= kjb_rows.y1) return;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const int tcx = int(threadIdx.x) + 2, tcy = int(threadIdx.y) + 2;
    const float4 center = s_in[tcy * D10_TW + tcx];
    const float4 reproj = ld_rgba16s(reprojection_tex, x, y);
    const float4 history = linear_to_working(ld_rgba16f(history_tex, x, y) * history_mult);
    float4 vsum = f4(0.0f), vsum2 = f4(0.0f); const float wsum = wt.w_sum; float hist_vsum = 0, hist_vsum2 = 0;
    for (int yy = -2; yy <= 2; ++yy) for (int xx = -2; xx <= 2; ++xx) {
        const int ti = (tcy + yy) * D10_TW + (tcx + xx);
        const float4 neigh = s_in[ti];
        const float hist_luma = s_hist_luma[ti];
        const float w = wt.w[(yy + 2) * 5 + (xx + 2)];
        vsum = mad(neigh, w, vsum); vsum2 = mad(neigh * neigh, w, vsum2);
        hist_vsum = mad(hist_luma, w, hist_vsum); hist_vsum2 = mad(hist_luma * hist_luma, w, hist_vsum2);
    }
    const float4 ex = vsum / wsum, ex2 = vsum2 / wsum;
    const float4 dev = vsqrt(vmax(f4(0.0f), ex2 - ex * ex));
    hist_vsum /= wsum; hist_vsum2 /= wsum;
    const float4 mh = bilinear_clamp(W, H, uv + xy(reproj), [&](int sx, int sy) { const float2 v = ld_rg16f(variance_history_tex, sx, sy); return f4(v.x, v.y, 0, 0); });
    const float2 moments_history = f2(mh.x, mh.y) * f2(ped, ped * ped);
    const float center_luma = center.x + (hist_vsum - ex.x);
    const float2 current_moments = f2(center_luma, center_luma * center_luma);
    const float2 vout = vmax(f2(0.0f), vlerp(moments_history, current_moments, 0.25f));
    st_rg16f(variance_history_output_tex, x, y, vout.x, vout.y);
    const float center_temporal_dev = kjb_sqrt(kjb_max(0.0f, moments_history.y - moments_history.x * moments_history.x));
    const float temporal_change = kjb_abs(hist_vsum - ex.x) / kjb_max(1e-8f, hist_vsum + ex.x);
    const float rt_invalid = kjb_saturate(kjb_sqrt(ld_rg16f(rt_history_invalidity_tex, x / 2, y / 2).x) * 4);
    const float current_sample_count = history.w;
    float clamp_box_size = 1 * kjb_lerp(0.25f, 2.0f, 1.0f - rt_invalid) * kjb_lerp(0.333f, 1.0f, kjb_saturate(reproj.w)) * 2;
    clamp_box_size = kjb_max(clamp_box_size, 0.5f);
    const float4 nmin = center - dev * clamp_box_size, nmax = center + dev * clamp_box_size;
    const float3 clamped_history = vclamp(xyz(history), xyz(nmin), xyz(nmax));
    const float variance_adjusted_temporal_change = kjb_smoothstep(0.1f, 1.0f, 0.05f * temporal_change / center_temporal_dev);
    float max_sample_count = 32;
    max_sample_count = kjb_lerp(max_sample_count, 4.0f, variance_adjusted_temporal_change);
    max_sample_count *= kjb_lerp(1.0f, 0.5f, rt_invalid);
    const float3 res = vlerp(clamped_history, xyz(center), 1.0f / (1.0f + kjb_min(max_sample_count, current_sample_count)));
    const float output_sample_count = kjb_min(current_sample_count, max_sample_count) + 1;
    const float4 output = working_to_linear(f4(res, output_sample_count));
    st_rgba16f(history_output_tex, x, y, output);
    st_rgba16f(output_tex, x, y, f4(xyz(output), kjb_saturate(output_sample_count * kjb_lerp(1.0f, 0.5f, rt_invalid) * kjb_smoothstep(0.3f, 0.0f, temporal_change) / 32.0f)));
}

// ------------------------------------------------------------------ D11 spatial_filter.hlsl:33-101
KJB_DEV float3 crunch(float3 v) { return v * kjb_rcp(max3(v.x, v.y, v.z) + 1.0f); }
KJB_DEV float3 uncrunch(float3 v) { return v * kjb_rcp(1.0f - max3(v.x, v.y, v.z)); }
struct PowTable8 { float v[8]; };   // v[i] = pow(float(i), 0.666): compile-time constants in the shader ("must be constant, so the pow can be const-folded"), host-evaluated here
KJB_KERNEL(256) k_rtdgi_spatial(const __grid_constant__ Globals g, Img input_tex, Img depth_tex, Img ssao_tex, Img geometric_normal_tex, ImgW output_tex, PowTable8 pw, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    const float4 cin = ld_rgba16f(input_tex, x, y);
    const float center_validity = cin.w;
    const float3 center_value = xyz(cin);
    if (center_validity == 1) { st_rgba16f(output_tex, x, y, f4(center_value, 1.0f)); return; }
    const float center_depth = ld_r32f(depth_tex, x, y);
    const float center_ssao = ld_r8u(ssao_tex, x, y);
    const float3 center_normal_vs = ld_a2r10g10b10(geometric_normal_tex, x, y) * 2.0f - 1.0f;
    const float ang_off = float((g.fc.frame_index * 23u) % 32u) * KJB_TAU_F + interleaved_gradient_noise(uint32_t(x), uint32_t(y)) * KJB_PI_F;
    const float MAX_RADIUS_PX = kjb_sqrt(kjb_lerp(16.0f * 16.0f, 2.0f * 2.0f, center_validity));
    uint32_t sample_count = kjb_cvt_u32(kjb_exp2(4.0f * square(1.0f - center_validity)));
    sample_count = sample_count < 2u ? 2u : (sample_count > 8u ? 8u : sample_count);
    float4 sum = f4(crunch(center_value), 1);
    const float RADIUS_SAMPLE_MULT = MAX_RADIUS_PX / pw.v[7];
    for (uint32_t i = 1; i < sample_count; ++i) {   // the shader walks all 8 taps and masks i >= sample_count: no side effects, skip them
        const float ang = (float(i) + ang_off) * KJB_GOLDEN_ANGLE;
        const float radius = pw.v[i] * RADIUS_SAMPLE_MULT;
        float sn, cs; kjb_sincos(ang, &sn, &cs);
        const float2 off = f2(cs, sn) * radius;
        const int sx = kjb_cvt_i32(float(x) + off.x), sy = kjb_cvt_i32(float(y) + off.y);
        const float sample_depth = ld_r32f(depth_tex, sx, sy);
        if (sample_depth != 0) {
            const float3 sample_val = xyz(ld_rgba16f(input_tex, sx, sy));
            const float sample_ssao = ld_r8u(ssao_tex, sx, sy);
            float wt = 1;
            wt *= kjb_exp2(-100.0f * kjb_abs(center_normal_vs.z * (center_depth / sample_depth - 1.0f)));
            wt *= kjb_exp2(-20.0f * kjb_abs(sample_ssao - center_ssao));
            sum = mad(f4(crunch(sample_val), 1.0f), wt, sum);
        }
    }
    const float norm_factor = 1.0f / kjb_max(1e-5f, sum.w);
    st_rgba16f(output_tex, x, y, f4(uncrunch(xyz(sum) * norm_factor), 1.0f));
}

// ================================================================== entry points
#define F4A(a) f4((a)[0], (a)[1], (a)[2], (a)[3])
#define CHK(img, fmt, name) if (!check_img(c, (img), (fmt), P, name)) return 1
#define CHKE(img, fmt, name, w, h) if (!check_img(c, (img), (fmt), P, name, (w), (h))) return 1

// the irradiance-cache binding block of a pass: all-or-nothing (NULL meta_buf = unbound), sizes per ircache.rs:172-231
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

int kjb_pass_rtdgi_reproject(kjb_context* c, const kjb_rtdgi_reproject_args* a) {
    const char* P = "rtdgi reproject"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex"); CHKE(a->input_tex, KJB_FMT_RGBA16_FLOAT, "input_tex", W, H); CHKE(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex", W, H);
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_rtdgi_reproject, KJB_GRID2D(W, H, 32, 8), img_ro(a->input_tex), img_ro(a->reprojection_tex), img_rw(a->output_tex), F4A(a->output_tex_size));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_validate(kjb_context* c, const kjb_rtdgi_validate_args* a) {
    const char* P = "rtdgi validate"; const uint32_t W = a->rt_history_invalidity_out_tex.width, H = a->rt_history_invalidity_out_tex.height;
    CHK(a->rt_history_invalidity_out_tex, KJB_FMT_R8_UNORM, "rt_history_invalidity_out_tex"); CHKE(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex", W, H);
    CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex"); CHK(a->reprojected_gi_tex, KJB_FMT_RGBA16_FLOAT, "reprojected_gi_tex"); CHKE(a->reservoir_tex, KJB_FMT_RG32_UINT, "reservoir_tex", W, H);
    CHKE(a->reservoir_ray_history_tex, KJB_FMT_RGBA16_FLOAT, "reservoir_ray_history_tex", W, H); CHK(a->sky_cube_tex, KJB_FMT_RGBA16_FLOAT, "sky_cube_tex");
    CHKE(a->irradiance_history_tex, KJB_FMT_RGBA16_FLOAT, "irradiance_history_tex", W, H); CHKE(a->ray_orig_history_tex, KJB_FMT_RGBA32_FLOAT, "ray_orig_history_tex", W, H);
    IrcacheBufs ircache; if (check_ircache_bindings(c, P, a->ircache, ircache)) return 1;
    KJB_ROWS(c, H);
    KJB_LAUNCH_CACHE(c, ircache.bound(), k_rtdgi_validate, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, img_ro(a->half_view_normal_tex), img_ro(a->depth_tex), img_ro(a->reprojected_gi_tex),
                     img_rw(a->reservoir_tex), img_ro(a->reservoir_ray_history_tex), img_ro(a->sky_cube_tex), img_rw(a->irradiance_history_tex), img_ro(a->ray_orig_history_tex),
                     img_rw(a->rt_history_invalidity_out_tex), F4A(a->gbuffer_tex_size), ircache);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_trace(kjb_context* c, const kjb_rtdgi_trace_args* a) {
    const char* P = "rtdgi trace"; const uint32_t W = a->candidate_irradiance_out_tex.width, H = a->candidate_irradiance_out_tex.height;
    CHK(a->candidate_irradiance_out_tex, KJB_FMT_RGBA16_FLOAT, "candidate_irradiance_out_tex"); CHKE(a->candidate_normal_out_tex, KJB_FMT_RGBA8_SNORM, "candidate_normal_out_tex", W, H);
    CHKE(a->candidate_hit_out_tex, KJB_FMT_RGBA16_FLOAT, "candidate_hit_out_tex", W, H); CHKE(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex", W, H);
    CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex"); CHK(a->reprojected_gi_tex, KJB_FMT_RGBA16_FLOAT, "reprojected_gi_tex"); CHK(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex");
    CHK(a->sky_cube_tex, KJB_FMT_RGBA16_FLOAT, "sky_cube_tex"); CHKE(a->rt_history_invalidity_in_tex, KJB_FMT_R8_UNORM, "rt_history_invalidity_in_tex", W, H);
    CHKE(a->rt_history_invalidity_out_tex, KJB_FMT_R8_UNORM, "rt_history_invalidity_out_tex", W, H);
    IrcacheBufs ircache; if (check_ircache_bindings(c, P, a->ircache, ircache)) return 1;
    KJB_ROWS(c, H);
    KJB_LAUNCH_CACHE(c, ircache.bound(), k_rtdgi_trace, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, img_ro(a->half_view_normal_tex), img_ro(a->depth_tex), img_ro(a->reprojected_gi_tex),
                     img_ro(a->reprojection_tex), img_ro(a->sky_cube_tex), img_rw(a->candidate_irradiance_out_tex), img_rw(a->candidate_normal_out_tex), img_rw(a->candidate_hit_out_tex),
                     img_ro(a->rt_history_invalidity_in_tex), img_rw(a->rt_history_invalidity_out_tex), F4A(a->gbuffer_tex_size), ircache);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_validity_integrate(kjb_context* c, const kjb_rtdgi_validity_integrate_args* a) {
    const char* P = "validity integrate"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_RG16_FLOAT, "output_tex"); CHKE(a->input_tex, KJB_FMT_R8_UNORM, "input_tex", W, H); CHKE(a->history_tex, KJB_FMT_RG16_FLOAT, "history_tex", W, H);
    CHK(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex"); CHKE(a->half_depth_tex, KJB_FMT_R32_FLOAT, "half_depth_tex", W, H);
    Weights25v wt; wt.w_sum = 0.0f;
    for (int yy = -2; yy <= 2; ++yy) for (int xx = -2; xx <= 2; ++xx) { const float w = kjb_exp2(-0.1f * float(xx * xx + yy * yy)); wt.w[(yy + 2) * 5 + (xx + 2)] = w; wt.w_sum += w; }
    KJB_ROWS(c, H);
    // block rows start at a multiple of 4 so that the (y^1, y^2) exchange partners share the block
    KJB_LAUNCH_SYNC(c, k_rtdgi_validity_integrate, KJB_DIMS(dim3((W + D5_BX - 1) / D5_BX, unsigned(kjb__rows.y1 - (kjb__rows.y0 & ~3) + D5_BY - 1) / D5_BY, 1), dim3(D5_BX, D5_BY, 1)), c->g, img_ro(a->input_tex), img_ro(a->history_tex), img_ro(a->reprojection_tex), img_ro(a->half_depth_tex), img_rw(a->output_tex),
               F4A(a->gbuffer_tex_size), wt);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_restir_temporal(kjb_context* c, const kjb_rtdgi_restir_temporal_args* a) {
    c->epoch_b++;   // temporal_reservoir_packed_tex changes: the position cache built from it is stale
    const char* P = "restir temporal"; const uint32_t W = a->radiance_out_tex.width, H = a->radiance_out_tex.height;
    CHK(a->radiance_out_tex, KJB_FMT_RGBA16_FLOAT, "radiance_out_tex");
    CHKE(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex", W, H); CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex");
    CHKE(a->candidate_radiance_tex, KJB_FMT_RGBA16_FLOAT, "candidate_radiance_tex", W, H); CHKE(a->candidate_normal_tex, KJB_FMT_RGBA8_SNORM, "candidate_normal_tex", W, H);
    CHKE(a->candidate_hit_tex, KJB_FMT_RGBA16_FLOAT, "candidate_hit_tex", W, H); CHKE(a->radiance_history_tex, KJB_FMT_RGBA16_FLOAT, "radiance_history_tex", W, H);
    CHKE(a->ray_orig_history_tex, KJB_FMT_RGBA32_FLOAT, "ray_orig_history_tex", W, H); CHKE(a->ray_history_tex, KJB_FMT_RGBA16_FLOAT, "ray_history_tex", W, H);
    CHKE(a->reservoir_history_tex, KJB_FMT_RG32_UINT, "reservoir_history_tex", W, H); CHK(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex");
    CHKE(a->hit_normal_history_tex, KJB_FMT_RGBA8_UNORM, "hit_normal_history_tex", W, H); CHKE(a->candidate_history_tex, KJB_FMT_RGBA16_FLOAT, "candidate_history_tex", W, H);
    CHKE(a->rt_invalidity_tex, KJB_FMT_RG16_FLOAT, "rt_invalidity_tex", W, H); CHKE(a->ray_orig_output_tex, KJB_FMT_RGBA32_FLOAT, "ray_orig_output_tex", W, H);
    CHKE(a->ray_output_tex, KJB_FMT_RGBA16_FLOAT, "ray_output_tex", W, H); CHKE(a->hit_normal_output_tex, KJB_FMT_RGBA8_UNORM, "hit_normal_output_tex", W, H);
    CHKE(a->reservoir_out_tex, KJB_FMT_RG32_UINT, "reservoir_out_tex", W, H); CHKE(a->candidate_out_tex, KJB_FMT_RGBA16_FLOAT, "candidate_out_tex", W, H);
    CHKE(a->temporal_reservoir_packed_tex, KJB_FMT_RGBA32_UINT, "temporal_reservoir_packed_tex", W, H);
    RestirTemporalImgs t;
    t.half_view_normal_tex = img_ro(a->half_view_normal_tex); t.depth_tex = img_ro(a->depth_tex); t.candidate_radiance_tex = img_ro(a->candidate_radiance_tex);
    t.candidate_normal_tex = img_ro(a->candidate_normal_tex); t.candidate_hit_tex = img_ro(a->candidate_hit_tex); t.radiance_history_tex = img_ro(a->radiance_history_tex);
    t.ray_orig_history_tex = img_ro(a->ray_orig_history_tex); t.ray_history_tex = img_ro(a->ray_history_tex); t.reservoir_history_tex = img_ro(a->reservoir_history_tex);
    t.reprojection_tex = img_ro(a->reprojection_tex); t.hit_normal_history_tex = img_ro(a->hit_normal_history_tex); t.candidate_history_tex = img_ro(a->candidate_history_tex);
    t.rt_invalidity_tex = img_ro(a->rt_invalidity_tex); t.radiance_out_tex = img_rw(a->radiance_out_tex); t.ray_orig_output_tex = img_rw(a->ray_orig_output_tex);
    t.ray_output_tex = img_rw(a->ray_output_tex); t.hit_normal_output_tex = img_rw(a->hit_normal_output_tex); t.reservoir_out_tex = img_rw(a->reservoir_out_tex);
    t.candidate_out_tex = img_rw(a->candidate_out_tex); t.temporal_reservoir_packed_tex = img_rw(a->temporal_reservoir_packed_tex);
    KJB_ROWS(c, H);
    // the positions of the packed reservoirs' depth words (D7/D9 read them 8-16 times per pixel) ride along when the launch covers the whole image
    kjb_context::PosCache& pc = c->pos_b;
    float4* positions = nullptr;
    if (c->opt_position_cache && kjb__rows.y0 == 0 && kjb__rows.y1 == int(H)) {
        const size_t need = size_t(W) * H * sizeof(float4);
        if (pc.cap < need) { dev_sync(c); dev_free(pc.d); pc.d = (float4*)dev_alloc(need); pc.cap = pc.d ? need : 0; }
        positions = pc.d;
    }
    KJB_LAUNCH(c, k_rtdgi_restir_temporal, KJB_GRID2D(W, H, 32, 8), c->g, t, F4A(a->gbuffer_tex_size), positions);
    if (positions) { pc.epoch = c->epoch_b; pc.src = a->temporal_reservoir_packed_tex.data; pc.w = W; pc.h = H; memcpy(pc.gts, a->gbuffer_tex_size, 16); }
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_restir_spatial(kjb_context* c, const kjb_rtdgi_restir_spatial_args* a) {
    const char* P = "restir spatial"; const uint32_t W = a->reservoir_output_tex.width, H = a->reservoir_output_tex.height;
    CHK(a->reservoir_output_tex, KJB_FMT_RG32_UINT, "reservoir_output_tex"); CHKE(a->reservoir_input_tex, KJB_FMT_RG32_UINT, "reservoir_input_tex", W, H);
    CHKE(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex", W, H); CHKE(a->half_depth_tex, KJB_FMT_R32_FLOAT, "half_depth_tex", W, H);
    CHKE(a->half_ssao_tex, KJB_FMT_R8_SNORM, "half_ssao_tex", W, H); CHKE(a->temporal_reservoir_packed_tex, KJB_FMT_RGBA32_UINT, "temporal_reservoir_packed_tex", W, H);
    if (a->reservoir_input_tex.data == a->reservoir_output_tex.data) return c->fail("restir spatial: input and output reservoirs must differ");
    const PosView pos_a = ensure_positions(c, c->pos_a, c->epoch_a, a->half_depth_tex, false, a->gbuffer_tex_size);
    const PosView pos_b = ensure_positions(c, c->pos_b, c->epoch_b, a->temporal_reservoir_packed_tex, true, a->gbuffer_tex_size);
    KJB_ROWS(c, H);
    KJB_LAUNCH_SYNC(c, k_rtdgi_restir_spatial, KJB_GRID2D(W, H, 32, 8), c->g, img_ro(a->reservoir_input_tex), img_ro(a->half_view_normal_tex), img_ro(a->half_depth_tex), img_ro(a->half_ssao_tex),
               img_ro(a->temporal_reservoir_packed_tex), img_rw(a->reservoir_output_tex), F4A(a->gbuffer_tex_size), F4A(a->output_tex_size), a->spatial_reuse_pass_idx, a->perform_occlusion_raymarch,
               a->occlusion_raymarch_importance_only, pos_a, pos_b);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_restir_check(kjb_context* c, const kjb_rtdgi_restir_check_args* a) {
    const char* P = "restir check"; const uint32_t W = a->reservoir_input_tex.width, H = a->reservoir_input_tex.height;
    CHK(a->reservoir_input_tex, KJB_FMT_RG32_UINT, "reservoir_input_tex"); CHKE(a->half_depth_tex, KJB_FMT_R32_FLOAT, "half_depth_tex", W, H);
    CHKE(a->temporal_reservoir_packed_tex, KJB_FMT_RGBA32_UINT, "temporal_reservoir_packed_tex", W, H);
    if (!c->tlas_valid) return c->fail("restir check: no acceleration structure (call kjb_rebuild_tlas)");
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_rtdgi_restir_check, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, img_ro(a->half_depth_tex), img_ro(a->temporal_reservoir_packed_tex), img_rw(a->reservoir_input_tex), F4A(a->gbuffer_tex_size));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_restir_resolve(kjb_context* c, const kjb_rtdgi_restir_resolve_args* a) {
    const char* P = "restir resolve"; const uint32_t W = a->irradiance_output_tex.width, H = a->irradiance_output_tex.height;
    CHK(a->irradiance_output_tex, KJB_FMT_RGBA16_FLOAT, "irradiance_output_tex"); CHK(a->radiance_tex, KJB_FMT_RGBA16_FLOAT, "radiance_tex"); CHK(a->reservoir_input_tex, KJB_FMT_RG32_UINT, "reservoir_input_tex");
    CHKE(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H); CHK(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex");
    CHK(a->half_depth_tex, KJB_FMT_R32_FLOAT, "half_depth_tex"); CHKE(a->ssao_tex, KJB_FMT_R8_UNORM, "ssao_tex", W, H); CHK(a->candidate_radiance_tex, KJB_FMT_RGBA16_FLOAT, "candidate_radiance_tex");
    CHK(a->candidate_hit_tex, KJB_FMT_RGBA16_FLOAT, "candidate_hit_tex"); CHK(a->temporal_reservoir_packed_tex, KJB_FMT_RGBA32_UINT, "temporal_reservoir_packed_tex");
    ResolveImgs t;
    t.radiance_tex = img_ro(a->radiance_tex); t.reservoir_input_tex = img_ro(a->reservoir_input_tex); t.gbuffer_tex = img_ro(a->gbuffer_tex); t.depth_tex = img_ro(a->depth_tex);
    t.half_view_normal_tex = img_ro(a->half_view_normal_tex); t.half_depth_tex = img_ro(a->half_depth_tex); t.ssao_tex = img_ro(a->ssao_tex); t.candidate_radiance_tex = img_ro(a->candidate_radiance_tex);
    t.candidate_hit_tex = img_ro(a->candidate_hit_tex); t.temporal_reservoir_packed_tex = img_ro(a->temporal_reservoir_packed_tex);
    const PosView pos_a = ensure_positions(c, c->pos_a, c->epoch_a, a->half_depth_tex, false, a->gbuffer_tex_size);
    const PosView pos_b = ensure_positions(c, c->pos_b, c->epoch_b, a->temporal_reservoir_packed_tex, true, a->gbuffer_tex_size);
    KJB_ROWS(c, H);
    PowTable4 pw; for (int i = 0; i < 4; ++i) pw.v[i] = kjb_pow(float(i), 0.666f);
    KJB_LAUNCH(c, k_rtdgi_restir_resolve, KJB_GRID2D(W, H, 32, 8), c->g, t, img_rw(a->irradiance_output_tex), F4A(a->gbuffer_tex_size), F4A(a->output_tex_size), pw, pos_a, pos_b);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_temporal(kjb_context* c, const kjb_rtdgi_temporal_args* a) {
    const char* P = "rtdgi temporal"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex"); CHKE(a->input_tex, KJB_FMT_RGBA16_FLOAT, "input_tex", W, H); CHKE(a->history_tex, KJB_FMT_RGBA16_FLOAT, "history_tex", W, H);
    CHKE(a->variance_history_tex, KJB_FMT_RG16_FLOAT, "variance_history_tex", W, H); CHKE(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex", W, H);
    CHK(a->rt_history_invalidity_tex, KJB_FMT_RG16_FLOAT, "rt_history_invalidity_tex"); CHKE(a->history_output_tex, KJB_FMT_RGBA16_FLOAT, "history_output_tex", W, H);
    CHKE(a->variance_history_output_tex, KJB_FMT_RG16_FLOAT, "variance_history_output_tex", W, H);
    Weights25 wt;
    for (int yy = -2; yy <= 2; ++yy) for (int xx = -2; xx <= 2; ++xx) wt.w[(yy + 2) * 5 + (xx + 2)] = kjb_exp(-3.0f * float(xx * xx + yy * yy) / float((2 + 1.) * (2 + 1.)));
    wt.w_sum = 0; for (int i = 0; i < 25; ++i) wt.w_sum += wt.w[i];
    KJB_ROWS(c, H);
    KJB_LAUNCH_SYNC(c, k_rtdgi_temporal, KJB_GRID2D(W, H, D10_BX, D10_BY), tile_mode({&a->input_tex, &a->history_tex}), c->g, img_ro(a->input_tex), img_ro(a->history_tex), img_ro(a->variance_history_tex), img_ro(a->reprojection_tex), img_ro(a->rt_history_invalidity_tex),
               img_rw(a->output_tex), img_rw(a->history_output_tex), img_rw(a->variance_history_output_tex), F4A(a->output_tex_size), wt);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_rtdgi_spatial(kjb_context* c, const kjb_rtdgi_spatial_args* a) {
    const char* P = "rtdgi spatial"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex"); CHKE(a->input_tex, KJB_FMT_RGBA16_FLOAT, "input_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H);
    CHKE(a->ssao_tex, KJB_FMT_R8_UNORM, "ssao_tex", W, H); CHKE(a->geometric_normal_tex, KJB_FMT_A2R10G10B10_UNORM, "geometric_normal_tex", W, H);
    KJB_ROWS(c, H);
    PowTable8 pw; for (int i = 0; i < 8; ++i) pw.v[i] = kjb_pow(float(i), 0.666f);
    KJB_LAUNCH(c, k_rtdgi_spatial, KJB_GRID2D(W, H, 32, 8), c->g, img_ro(a->input_tex), img_ro(a->depth_tex), img_ro(a->ssao_tex), img_ro(a->geometric_normal_tex), img_rw(a->output_tex), pw);
    KJB_PASS_EPILOGUE(c, P);
}

}  // extern "C"
