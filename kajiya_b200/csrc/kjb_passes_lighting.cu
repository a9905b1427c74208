// Lighting composite (SURVEY §8f N4) as sm_90a kernels: "trace shadow mask" (renderers/shadows.rs:10-35,
// rt/trace_sun_shadow_mask.rgen.hlsl) and "light gbuffer" (renderers/deferred.rs:8-43, light_gbuffer.hlsl).
#include "kjb_context.h"

using namespace kjb;

// ------------------------------------------------------------------ rt/trace_sun_shadow_mask.rgen.hlsl:19-60
KJB_KERNEL(128) k_trace_sun_shadow_mask(const __grid_constant__ Globals g, Img depth_tex, Img geometric_normal_tex, ImgW output_tex, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float2 uv = (f2(float(x), float(y)) + 0.5f) / f2(float(output_tex.w), float(output_tex.h));
    const float z_over_w = ld_r32f(depth_tex, x, y);
    if (0.0f == z_over_w) { st_r8u(output_tex, x, y, 1.0f); return; }
    const float2 cs = uv_to_cs(uv);
    float4 pt_vs = mul(vc.sample_to_view, f4(cs.x, cs.y, z_over_w, 1.0f));
    float4 pt_ws = mul(vc.view_to_world, pt_vs);
    pt_ws = pt_ws / pt_ws.w; pt_vs = pt_vs / pt_vs.w;
    const float3 normal_vs = ld_a2r10g10b10(geometric_normal_tex, x, y) * 2.0f - 1.0f;
    const float3 normal_ws = xyz(mul(vc.view_to_world, f4(normal_vs, 0.0f)));
    const float bias_amount = (-pt_vs.z + length(xyz(pt_ws))) * 1e-5f;
    const float3 ray_origin = xyz(pt_ws) + normal_ws * bias_amount;
    const float4 bn = blue_noise_for_pixel(g, uint32_t(x), uint32_t(y), g.fc.frame_index);
    const bool is_shadowed = rt_is_shadowed(g, ray_origin, sample_sun_direction(g.fc, f2(bn.x, bn.y), true), 0.0f, KJB_FLT_MAX);
    st_r8u(output_tex, x, y, is_shadowed ? 0.0f : 1.0f);
}

// ------------------------------------------------------------------ light_gbuffer.hlsl:60-260 (debug_shading_mode 0, 2, 3, 4)
struct LightGbufferImgs { Img gbuffer_tex, depth_tex, shadow_mask_tex, rtr_tex, rtdgi_tex, unconvolved_sky_cube_tex; ImgW temporal_output_tex, output_tex; int shadow_is_rg16f; };
KJB_KERNEL(256) k_light_gbuffer(const __grid_constant__ Globals g, LightGbufferImgs t, float4 ots, uint32_t mode, float real_sun_radius_cos, Rows kjb_rows) {
    KJB_PX; if (x >= t.output_tex.w || y >= t.output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const ViewRayContext vrc = ViewRayContext::from_uv(vc, uv);
    const float3 ray_dir = vrc.ray_dir_ws();
    const float depth = ld_r32f(t.depth_tex, x, y);
    if (depth == 0.0f) {   // sky + sun disk
        const float real_sun_angular_radius = 0.53f * 0.5f * KJB_PI_F / 180.0f;
        const float sun_angular_radius_cos = kjb_min(real_sun_radius_cos, g.fc.sun_angular_radius_cos);
        const float current_sun_angular_radius = kjb_acos(sun_angular_radius_cos);
        const float sun_radius_ratio = real_sun_angular_radius / current_sun_angular_radius;
        float3 output = xyz(sample_cube_rgba16f(t.unconvolved_sky_cube_tex, ray_dir));
        if (dot(ray_dir, sun_direction(g.fc)) > sun_angular_radius_cos) output += 800.0f * sun_color_in_direction(g.fc, ray_dir) * sun_radius_ratio * sun_radius_ratio;
        st_rgba16f(t.temporal_output_tex, x, y, f4(output, 1)); st_rgba16f(t.output_tex, x, y, f4(output, 1));
        return;
    }
    const float3 to_light_norm = sun_direction(g.fc);
    float shadow_mask = t.shadow_is_rg16f ? ld_rg16f(t.shadow_mask_tex, x, y).x : ld_r8u(t.shadow_mask_tex, x, y);
    if (mode == 4u) shadow_mask = 1;
    const GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, x, y));
    const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
    const float3 wi = mul(to_light_norm, tangent_to_world);
    float3 wo = mul(-ray_dir, tangent_to_world);
    if (wo.z < 0.0f) { wo.z *= -0.25f; wo = normalize(wo); }
    const LayeredBrdf brdf = layered_brdf_from_gbuffer_ndotv(g, gbuffer, wo.z);
    const float3 brdf_value = layered_evaluate_directional_light(brdf, wo, wi) * kjb_max(0.0f, wi.z);
    const float3 light_radiance = shadow_mask * f3(g.sun_color[0], g.sun_color[1], g.sun_color[2]);
    float3 total_radiance = brdf_value * light_radiance;
    total_radiance += gbuffer.emissive;
    float3 gi_irradiance = f3(0.0f);
    if (mode != 4u) gi_irradiance = xyz(ld_rgba16f(t.rtdgi_tex, x, y));
    total_radiance += gi_irradiance * brdf.diffuse_brdf.albedo * brdf.ep.preintegrated_transmission_fraction;
    const float3 rtr = ld_r11g11b10(t.rtr_tex, x, y);
    if (mode != 4u) total_radiance += rtr * brdf.ep.preintegrated_reflection;   // !RTR_RENDER_SCALED_BY_FG
    st_rgba16f(t.temporal_output_tex, x, y, f4(total_radiance, 1.0f));
    float3 output = total_radiance;
    if (mode == 3u) { output = rtr * brdf.ep.preintegrated_reflection; output = output / brdf.ep.preintegrated_reflection; }
    if (mode == 2u) output = gi_irradiance;
    st_rgba16f(t.output_tex, x, y, f4(output, 1.0f));
}

// ------------------------------------------------------------------ shadow denoiser (renderers/shadow_denoise.rs; FidelityFX shadow denoiser as adapted upstream)
KJB_DEV uint32_t sd_rounded_divide(uint32_t v, uint32_t d) { return (v + d - 1u) / d; }                                        // ffx_denoiser_shadows_util.hlsl:26-29
KJB_DEV uint32_t sd_linear_tile_index(uint32_t tx, uint32_t ty, uint32_t screen_width) { return ty * sd_rounded_divide(screen_width, 8u) + tx; }   // :36-39
// WriteMask / ReadRaytracedShadowMask / Write- and ReadTileMetaData: linear index -> texel of the extent-sized R32_UINT image (0 outside)
KJB_DEV uint32_t sd_tile_read(const Img& img, uint32_t ext_x, uint32_t linear) { return ld_r32u(img, int(linear % ext_x), int(linear / ext_x)); }
KJB_DEV void sd_tile_write(const ImgW& img, uint32_t ext_x, uint32_t linear, uint32_t v) { st_r32u(img, int(linear % ext_x), int(linear / ext_x), v); }
struct ShadowKernelWeights { float k[9]; };   // FFX_DNSR_Shadows_KernelWeight(0..8), host-evaluated (tileclassification.hlsl:169-184)

// "shadow bitpack": one thread per 8x4 tile ORs its 32 lanes (prepare.hlsl:28-35; the shader's wave = the tile)
KJB_KERNEL(256) k_shadow_bitpack(Img input_tex, ImgW output_tex, uint32_t W, uint32_t ext_x, uint32_t tiles_x, uint32_t tiles_y, Rows kjb_rows) {
    KJB_PX; if (uint32_t(x) >= tiles_x || uint32_t(y) >= tiles_y) return;
    uint32_t mask = 0;
    for (uint32_t ly = 0; ly < 4u; ++ly) {
        const uint32_t py = uint32_t(y) * 4u + ly;
        for (uint32_t lx = 0; lx < 8u; ++lx) {
            const uint32_t px = uint32_t(x) * 8u + lx;
            if (ld_r8u(input_tex, int(px), int(py)) > 0.5f) mask |= 1u << ((py % 4u) * 8u + (px % 8u));
        }
    }
    sd_tile_write(output_tex, ext_x, sd_linear_tile_index(uint32_t(x), uint32_t(y), W), mask);
}

// FFX_DNSR_Shadows_HorizontalNeighborhood (tileclassification.hlsl:193-252): 17 taps of one row out of three bit masks
KJB_DEV float sd_horizontal_neighborhood(const Img& bitpacked, uint32_t ext_x, const ShadowKernelWeights& kw, int dx, int dy, uint32_t W, uint32_t H) {
    if (dy < 0 || dy >= int(H)) return 0.0f;
    const uint32_t tile_x = uint32_t(dx) / 8u, tile_y = uint32_t(dy) / 4u;
    const uint32_t lin = sd_linear_tile_index(tile_x, tile_y, W);
    const bool first = tile_x == 0u, last = tile_x == sd_rounded_divide(W, 8u) - 1u;
    uint32_t left_tile = 0; if (!first) left_tile = sd_tile_read(bitpacked, ext_x, uint32_t(int(lin) - 1));
    const uint32_t center_tile = sd_tile_read(bitpacked, ext_x, lin);
    uint32_t right_tile = 0; if (!last) right_tile = sd_tile_read(bitpacked, ext_x, uint32_t(int(lin) + 1));
    const uint32_t row_base = (uint32_t(dy) % 4u) * 8u;
    uint32_t neighborhood = ((left_tile >> row_base) & 0xFFu) | (((center_tile >> row_base) & 0xFFu) << 8) | (((right_tile >> row_base) & 0xFFu) << 16);
    neighborhood >>= (uint32_t(dx) % 8u);
    float moment = 0.0f;
    for (int i = 0; i < 8; ++i) moment += (neighborhood & (1u << i)) ? kw.k[8 - i] : 0.0f;
    moment += (neighborhood & (1u << 8)) ? kw.k[0] : 0.0f;
    for (int i = 1; i <= 8; ++i) moment += (neighborhood & (1u << (8 + i))) ? kw.k[i] : 0.0f;
    return moment;
}
KJB_DEV float4 sd_cubic_hermite(float4 A, float4 B, float4 C, float4 D, float t) {   // inc/curve.hlsl:4-13
    const float t2 = t * t, t3 = t * t * t;
    const float4 a = -A / 2.0f + (3.0f * B) / 2.0f - (3.0f * C) / 2.0f + D / 2.0f;
    const float4 b = A - (5.0f * B) / 2.0f + 2.0f * C - D / 2.0f;
    const float4 c = -A / 2.0f + C / 2.0f;
    return a * t3 + b * t2 + c * t + B;
}
template <typename F> KJB_DEV float4 sd_sample_catmull_rom(float2 size, float2 P, F fetch) {   // inc/image.hlsl:42-79, identity remap
    const float2 pixel = P * size + 0.5f;
    const float2 frc = vfrac(pixel);
    const int ix = kjb_cvt_i32(pixel.x) - 1, iy = kjb_cvt_i32(pixel.y) - 1;
    float4 rows[4];
    for (int j = 0; j < 4; ++j) rows[j] = sd_cubic_hermite(fetch(ix - 1, iy - 1 + j), fetch(ix, iy - 1 + j), fetch(ix + 1, iy - 1 + j), fetch(ix + 2, iy - 1 + j), frc.x);
    return sd_cubic_hermite(rows[0], rows[1], rows[2], rows[3], frc.y);
}
KJB_DEV float sd_soft_color_clamp(float center, float history, float ex, float dev) {   // inc/soft_color_clamp.hlsl:1-14, scalar
    const float history_dist = kjb_abs(history - ex) / kjb_max(kjb_abs(history * 0.1f), dev);
    const float closest_pt = kjb_clamp(history, center - dev, center + dev);
    return kjb_lerp(history, closest_pt, kjb_smoothstep(1.0f, 3.0f, history_dist));
}

// "shadow temporal": one 8x8 block per denoiser tile (megakernel.hlsl + ffx_denoiser_shadows_tileclassification.hlsl:316-461)
struct ShadowTemporalImgs { Img shadow_mask_tex, bitpacked_shadow_mask_tex, prev_moments_tex, prev_accum_tex, reprojection_tex; ImgW output_moments_tex, temporal_output_tex, meta_output_tex; };
KJB_KERNEL(64) k_shadow_temporal(const __grid_constant__ Globals g, ShadowTemporalImgs t, float4 its, uint32_t ext_x, ShadowKernelWeights kw, Rows kjb_rows) {
    __shared__ float s_neighborhood[8][24];
    const int lx = int(threadIdx.x), ly = int(threadIdx.y);
    const int gx = int(blockIdx.x), gy = kjb_rows.y0 / 8 + int(blockIdx.y);
    const int x = gx * 8 + lx, y = gy * 8 + ly;
    const uint32_t W = uint32_t(its.x), H = uint32_t(its.y);
    // FFX_DNSR_Shadows_SearchSpatialRegion (:48-86); IsShadowReciever is the constant true upstream, so this alone decides
    uint32_t combined_or = 0, combined_and = 0xFFFFFFFFu;
    for (int j = -2; j <= 3; ++j) for (int i = -1; i <= 1; ++i) {
        int tx = gx + i, ty = gy * 2 + j;
        const int mx = int(sd_rounded_divide(W, 8u)) - 1, my = int(sd_rounded_divide(H, 4u)) - 1;
        tx = tx < 0 ? 0 : (tx > mx ? mx : tx); ty = ty < 0 ? 0 : (ty > my ? my : ty);
        const uint32_t m = sd_tile_read(t.bitpacked_shadow_mask_tex, ext_x, sd_linear_tile_index(uint32_t(tx), uint32_t(ty), W));
        combined_or |= m; combined_and &= m;
    }
    const bool all_in_light = combined_and == 0xFFFFFFFFu, all_in_shadow = combined_or == 0u;
    const uint32_t meta_index = uint32_t(gy) * sd_rounded_divide(W, 8u) + uint32_t(gx);
    const bool in_rows = y < kjb_rows.y1;
    if (all_in_light || all_in_shadow) {   // FFX_DNSR_Shadows_ClearTargets (:300-313); uniform over the block
        const float shadow_value = all_in_light ? 1.0f : 0.0f;
        if (lx == 0 && ly == 0) sd_tile_write(t.meta_output_tex, ext_x, meta_index, (all_in_light ? 2u : 0u) | 1u);
        if (in_rows) { st_rg16f(t.temporal_output_tex, x, y, shadow_value, 0.0f); st_rgba16f(t.output_moments_tex, x, y, f4(shadow_value, 0.0f, 8.0f, shadow_value)); }
        return;
    }
    if (lx == 0 && ly == 0) sd_tile_write(t.meta_output_tex, ext_x, meta_index, 0u);
    const float4 reproj = ld_rgba16s(t.reprojection_tex, x, y);
    // FFX_DNSR_Shadows_ComputeLocalNeighborhood (:256-287)
    const float upper = sd_horizontal_neighborhood(t.bitpacked_shadow_mask_tex, ext_x, kw, x, y - 8, W, H);
    const float center = sd_horizontal_neighborhood(t.bitpacked_shadow_mask_tex, ext_x, kw, x, y, W, H);
    const float lower = sd_horizontal_neighborhood(t.bitpacked_shadow_mask_tex, ext_x, kw, x, y + 8, W, H);
    s_neighborhood[lx][ly] = upper; s_neighborhood[lx][ly + 8] = center; s_neighborhood[lx][ly + 16] = lower;
    __syncthreads();
    float local_neighborhood = 0;
    local_neighborhood = mad(center, kw.k[0], local_neighborhood);
    local_neighborhood = mad(upper, kw.k[8], local_neighborhood);
    local_neighborhood = mad(lower, kw.k[8], local_neighborhood);
    for (int i = 1; i < 8; ++i) {
        local_neighborhood = mad(s_neighborhood[lx][8 + ly - i], kw.k[i], local_neighborhood);
        local_neighborhood = mad(s_neighborhood[lx][8 + ly + i], kw.k[i], local_neighborhood);
    }
    const float2 uv = (f2(float(x), float(y)) + 0.5f) * f2(its.z, its.w);
    const float2 history_uv = uv + xy(reproj);
    const float shadow_current = ld_r8u(t.shadow_mask_tex, x, y);
    const uint32_t quad_reproj_valid_packed = kjb_cvt_u32(reproj.z * 15.0f + 0.5f);
    const bool is_disoccluded = (quad_reproj_valid_packed & 15u) != 15u;
    float4 previous_moments = f4(0.0f);
    if (!is_disoccluded) {
        previous_moments = sd_sample_catmull_rom(f2(its.x, its.y), history_uv, [&](int sx, int sy) { return ld_rgba16f(t.prev_moments_tex, sx, sy); });
        previous_moments.y = kjb_max(0.0f, previous_moments.y); previous_moments.z = kjb_max(0.0f, previous_moments.z);
    }
    const float old_m = previous_moments.x, old_s = previous_moments.y;
    const float sample_count = previous_moments.z + 1.0f;
    const float new_m = kjb_lerp(old_m, shadow_current, 1.0f / sample_count);
    const float new_s = kjb_lerp(old_s, (shadow_current - old_m) * (shadow_current - new_m), 1.0f / sample_count);
    float variance = new_s;
    float4 moments_current = f4(new_m, new_s, sample_count, local_neighborhood);
    const float mean = local_neighborhood;
    float spatial_variance = local_neighborhood;
    spatial_variance = kjb_max(spatial_variance - mean * mean, 0.0f);
    const float std_deviation = kjb_sqrt(spatial_variance);
    float shadow_previous = shadow_current;
    if (g.fc.frame_index != 0u) shadow_previous = sd_sample_catmull_rom(f2(its.x, its.y), history_uv, [&](int sx, int sy) { const float2 v = ld_rg16f(t.prev_accum_tex, sx, sy); return f4(v.x, v.y, 0.0f, inb(t.prev_accum_tex, sx, sy) ? 1.0f : 0.0f); }).x;
    const float sigma = 2.0f;
    const float temporal_discontinuity = (previous_moments.w - moments_current.w) / kjb_max(0.5f * std_deviation, 0.001f);
    const float sample_counter_damper = kjb_exp(-temporal_discontinuity * temporal_discontinuity / sigma);
    moments_current.z *= kjb_max(0.5f, sample_counter_damper);
    float shadow_clamped = sd_soft_color_clamp(shadow_current, shadow_previous, mean, std_deviation * 0.5f);
    if (moments_current.z < 16.0f) {
        const float variance_boost = kjb_max(16.0f - moments_current.z, 1.0f);
        variance = kjb_max(variance, spatial_variance);
        variance *= variance_boost;
    }
    shadow_clamped = kjb_lerp(shadow_clamped, shadow_current, 1.0f / kjb_max(1.0f, moments_current.z));
    if (in_rows) {
        st_rg16f(t.temporal_output_tex, x, y, shadow_clamped, variance);
        moments_current.z = kjb_min(moments_current.z, 32.0f);   // FFX_DNSR_Shadows_WriteMoments (megakernel.hlsl:93-99)
        st_rgba16f(t.output_moments_tex, x, y, moments_current);
    }
}

// "shadow spatial": 8x8 block, 16x16 group-shared tile with a 4 texel apron (ffx_denoiser_shadows_filter.hlsl)
struct ShadowSpatialImgs { Img input_tex, meta_tex, geometric_normal_tex, depth_tex; ImgW output_tex; };
KJB_KERNEL(64) k_shadow_spatial(ShadowSpatialImgs t, float4 its, uint32_t ext_x, int step, Rows kjb_rows) {
    __shared__ uint32_t s_input[16][16], s_normals_xy[16][16], s_normals_zw[16][16];
    __shared__ float s_depth[16][16];
    const int lx = int(threadIdx.x), ly = int(threadIdx.y);
    const int gx = int(blockIdx.x), gy = kjb_rows.y0 / 8 + int(blockIdx.y);
    const int x = gx * 8 + lx, y = gy * 8 + ly;
    const uint32_t W = uint32_t(its.x), H = uint32_t(its.y);
    const bool in_rows = y < kjb_rows.y1;
    const uint32_t m = sd_tile_read(t.meta_tex, ext_x, uint32_t(gy) * sd_rounded_divide(W, 8u) + uint32_t(gx));
    const bool is_cleared = (m & 1u) != 0u, all_in_light = (m & 2u) != 0u;
    if (is_cleared) {   // uniform over the block; pass index is the constant 0 upstream, so cleared tiles are written
        if (in_rows) st_rg16f(t.output_tex, x, y, kjb_max(0.0f, all_in_light ? 1.0f : 0.0f), kjb_max(0.0f, 0.0f));
        return;
    }
    // FFX_DNSR_Shadows_InitializeGroupSharedMemory (:93-132): four clamped loads per thread, normals and input through f32tof16
    for (int q = 0; q < 4; ++q) {
        const int ox = (q & 1) * 8, oy = (q >> 1) * 8;
        int px = x - 4 + ox, py = y - 4 + oy;
        px = px < 0 ? 0 : (px > int(W) - 1 ? int(W) - 1 : px); py = py < 0 ? 0 : (py > int(H) - 1 ? int(H) - 1 : py);
        const float3 n = ld_a2r10g10b10(t.geometric_normal_tex, px, py) * 2.0f - 1.0f;
        const float2 in = ld_rg16f(t.input_tex, px, py);
        s_input[ly + oy][lx + ox] = pack_2x16f(in.x, in.y);
        s_normals_xy[ly + oy][lx + ox] = pack_2x16f(n.x, n.y);
        s_normals_zw[ly + oy][lx + ox] = pack_2x16f(n.z, 0.0f);
        s_depth[ly + oy][lx + ox] = ld_r32f(t.depth_tex, px, py);
    }
    const float depth_here = ld_r32f(t.depth_tex, x, y);
    const bool needs_denoiser = depth_here != 0.0f;
    __syncthreads();
    float weight_sum = 1.0f; float2 shadow_sum = f2(0.0f);
    if (needs_denoiser) {   // FFX_DNSR_Shadows_DenoiseFromGroupSharedMemory (:155-214)
        const int cx = lx + 4, cy = ly + 4;
        const float2 shadow_center = unpack_2x16f(s_input[cy][cx]);
        const float3 normal_center = f3(unpack_2x16f(s_normals_xy[cy][cx]).x, unpack_2x16f(s_normals_xy[cy][cx]).y, unpack_2x16f(s_normals_zw[cy][cx]).x);
        weight_sum = 1.0f; shadow_sum = shadow_center;
        const float variance = shadow_center.y;
        const float std_deviation = kjb_sqrt(kjb_max(variance + 1e-9f, 0.0f));
        const float sharp = kjb_max(0.0f, 1.0f - 2.0f * std_deviation);
        const float kernel_sharpening = kjb_max(1e-10f, 1.0f - sharp * sharp);
        const float kernel[3] = {1.0f, kjb_exp2(-0.5849625007211563f / kernel_sharpening), kjb_exp2(-2.584962500721156f / kernel_sharpening)};
        for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
            const int tx = cx + xx * step, ty = cy + yy * step;
            const float depth_neigh = s_depth[ty][tx];
            const float3 normal_neigh = f3(unpack_2x16f(s_normals_xy[ty][tx]).x, unpack_2x16f(s_normals_xy[ty][tx]).y, unpack_2x16f(s_normals_zw[ty][tx]).x);
            const float2 shadow_neigh = unpack_2x16f(s_input[ty][tx]);
            const float sky_pixel_multiplier = ((xx == 0 && yy == 0) || depth_neigh >= 1.0f || depth_neigh <= 0.0f) ? 0.0f : 1.0f;
            float w = kernel[xx < 0 ? -xx : xx] * kernel[yy < 0 ? -yy : yy];
            w *= kjb_exp(-kjb_abs(shadow_center.x - shadow_neigh.x) / std_deviation);
            w *= kjb_exp2(-kjb_abs(1.0f - (depth_here / depth_neigh)) / 0.01f);
            w *= kjb_pow(kjb_saturate(dot(normal_center, normal_neigh)), 32.0f);
            w *= sky_pixel_multiplier;
            shadow_sum = shadow_sum + f2(w, w * w) * shadow_neigh;
            weight_sum += w;
        }
    }
    if (in_rows) st_rg16f(t.output_tex, x, y, kjb_max(0.0f, shadow_sum.x / weight_sum), kjb_max(0.0f, shadow_sum.y / (weight_sum * weight_sum)));
}

// ------------------------------------------------------------------ LightingRenderer::render_specular (renderers/lighting.rs:23-87)
// "sample lights" (lighting/sample_lights.rgen.hlsl:18-63): one light sample + shadow ray per half-res pixel
KJB_KERNEL(128) k_sample_lights(const __grid_constant__ Globals g, Img depth_tex, ImgW out0_tex, ImgW out1_tex, ImgW out2_tex, float4 gts, Rows kjb_rows) {
    KJB_PX; if (x >= out0_tex.w || y >= out0_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const int hx = x * 2 + hso.x, hy = y * 2 + hso.y;
    const float depth = ld_r32f(depth_tex, hx, hy);
    if (0.0f == depth) { st_rgba16f(out0_tex, x, y, f4(0.0f)); return; }
    const float s4[4] = {gts.x, gts.y, gts.z, gts.w};
    const float2 uv = get_uv(hx, hy, s4);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_depth(vc, uv, depth);
    const float3 shadow_ray_origin = vrc.biased_secondary_ray_origin_ws();
    const float4 urand4 = blue_noise_for_pixel(g, uint32_t(x), uint32_t(y), g.fc.frame_index);
    const uint32_t light_count = g.fc.triangle_light_count;
    const uint32_t light_idx = kjb_cvt_u32(urand4.z * float(light_count)) % light_count;
    const float light_choice_pmf = 1.0f / float(light_count);
    const kjb_triangle_light tl = g.lights[light_idx];
    const LightSample ls = sample_triangle_light(tl, f2(urand4.x, urand4.y));
    const float3 to_light_ws = ls.pos - shadow_ray_origin;
    const float dist_to_light = length(to_light_ws);
    const bool is_shadowed = rt_is_shadowed(g, shadow_ray_origin, to_light_ws / kjb_max(1e-8f, dist_to_light), 0.0f, dist_to_light - 1e-4f);
    st_rgba16f(out0_tex, x, y, f4(is_shadowed ? f3(0.0f) : f3(tl.radiance[0], tl.radiance[1], tl.radiance[2]), 1.0f));
    st_rgba32f(out1_tex, x, y, f4(vrc.ray_hit_vs() + direction_world_to_view(vc, to_light_ws), ls.pdf * light_choice_pmf));
    st_rgba8s(out2_tex, x, y, f4(direction_world_to_view(vc, ls.normal), 0.0f));
}

// "spatial reuse lights" (lighting/spatial_reuse_lights.hlsl:33-168): 8 borrowed half-res samples per pixel, added into the resolved reflections
struct ReuseLightsImgs { Img gbuffer_tex, depth_tex, hit0_tex, hit1_tex, hit2_tex, half_view_normal_tex, half_depth_tex; ImgW output_tex; };
KJB_KERNEL(256) k_spatial_reuse_lights(const __grid_constant__ Globals g, ReuseLightsImgs t, float4 ots, const int32_t* offs, Rows kjb_rows) {
    KJB_PX; if (x >= t.output_tex.w || y >= t.output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float depth = ld_r32f(t.depth_tex, x, y);
    if (0.0f == depth) return;
    const int2 hso = halfres_subsample_offset(g.fc.frame_index);
    const ViewRayContext vrc = ViewRayContext::from_uv_and_depth(vc, uv, depth);
    GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(t.gbuffer_tex, x, y));
    gbuffer.roughness = kjb_max(gbuffer.roughness, 3e-4f);
    const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
    float3 wo = mul(-normalize(vrc.ray_dir_ws()), tangent_to_world);
    if (wo.z < 0.0f) { wo.z *= -0.25f; wo = normalize(wo); }
    const LayeredBrdf layered_brdf = layered_brdf_from_gbuffer_ndotv(g, gbuffer, wo.z);
    const SpecularBrdf specular_brdf = layered_brdf.specular_brdf;
    const float3 energy_preservation_mult = layered_brdf.ep.preintegrated_reflection_mult;
    const uint32_t px_idx_in_quad = (((uint32_t(x) & 1u) | (uint32_t(y) & 1u) * 2u) + g.fc.frame_index) & 3u;
    float4 contrib_accum = f4(0.0f);
    const float3 normal_vs = direction_world_to_view(vc, gbuffer.normal);
    const float3 center_hit_vs = vrc.ray_hit_vs();
    for (uint32_t sample_i = 0; sample_i < 8u; ++sample_i) {
        const int32_t* o = offs + 4 * ((px_idx_in_quad * 16u + sample_i) + 64u * 3u);
        const int spx = x / 2 + o[0], spy = y / 2 + o[1];
        const float sample_depth = ld_r32f(t.half_depth_tex, spx, spy);
        const float4 packed0 = ld_rgba16f(t.hit0_tex, spx, spy);
        if (packed0.w != 0.0f && sample_depth != 0.0f) {
            const float2 sample_uv = get_uv(spx * 2 + hso.x, spy * 2 + hso.y, s4);
            const ViewRayContext sample_ray_ctx = ViewRayContext::from_uv_and_depth(vc, sample_uv, sample_depth);
            const float3 sample_origin_vs = sample_ray_ctx.ray_hit_vs();
            const float4 packed1 = ld_rgba32f(t.hit1_tex, spx, spy);
            float neighbor_sampling_pdf = packed1.w;
            const float3 sample_hit_normal_vs = xyz(ld_rgba8s(t.hit2_tex, spx, spy));
            const float3 center_to_hit_vs = xyz(packed1) - vlerp(center_hit_vs, sample_origin_vs, 0.5f);
            const float3 wi = normalize(mul(direction_view_to_world(vc, center_to_hit_vs), tangent_to_world));
            const float3 sample_normal_vs = xyz(ld_rgba8s(t.half_view_normal_tex, spx, spy));
            float rejection_bias = 1;
            rejection_bias *= kjb_saturate((dot(normal_vs, sample_normal_vs) - 0.9f) / (0.999f - 0.9f));
            rejection_bias *= kjb_exp2(-10.0f * kjb_abs(depth / sample_depth - 1.0f));
            {
                const float3 surface_offset = sample_origin_vs - center_hit_vs;
                const float fraction_of_normal_direction_as_offset = dot(surface_offset, normal_vs) / length(surface_offset);
                if (wi.z > 0.0f && wi.z * 0.2f < fraction_of_normal_direction_as_offset) rejection_bias *= sample_i == 0u ? 1.0f : 0.0f;
            }
            const BrdfValue spec = specular_evaluate(specular_brdf, wo, wi);
            const float center_to_hit_dist2 = dot(center_to_hit_vs, center_to_hit_vs);
            const float to_psa_metric = kjb_max(0.0f, wi.z) * kjb_max(0.0f, dot(sample_hit_normal_vs, -normalize(center_to_hit_vs))) / center_to_hit_dist2;
            neighbor_sampling_pdf /= to_psa_metric;
            const float3 contrib_rgb = xyz(packed0) * spec.value * energy_preservation_mult * kjb_step(0.0f, wi.z) * (neighbor_sampling_pdf > 0.0f ? (1 / neighbor_sampling_pdf) : 0.0f);
            contrib_accum = contrib_accum + f4(contrib_rgb, 1) * rejection_bias;
        }
    }
    const float contrib_norm_factor = kjb_max(1e-8f, contrib_accum.w);
    const float3 out_color = xyz(contrib_accum) / contrib_norm_factor;
    st_r11g11b10(t.output_tex, x, y, ld_r11g11b10(as_ro(t.output_tex), x, y) + out_color);   // RENDER_INTO_RTR: output_tex[px].rgb += out_color
}

#define F4A(a) f4((a)[0], (a)[1], (a)[2], (a)[3])
#define CHK(img, fmt, name) if (!check_img(c, (img), (fmt), P, name)) return 1
#define CHKE(img, fmt, name, w, h) if (!check_img(c, (img), (fmt), P, name, (w), (h))) return 1

extern "C" {

int kjb_pass_trace_sun_shadow_mask(kjb_context* c, const kjb_trace_sun_shadow_mask_args* a) {
    const char* P = "trace shadow mask"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R8_UNORM, "output_tex"); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H); CHKE(a->geometric_normal_tex, KJB_FMT_A2R10G10B10_UNORM, "geometric_normal_tex", W, H);
    if (!c->tlas_valid) return c->fail("trace shadow mask: no acceleration structure (call kjb_rebuild_tlas)");
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_trace_sun_shadow_mask, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, img_ro(a->depth_tex), img_ro(a->geometric_normal_tex), img_rw(a->output_tex));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_light_gbuffer(kjb_context* c, const kjb_light_gbuffer_args* a) {
    const char* P = "light gbuffer"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    if (a->debug_show_wrc || a->debug_shading_mode == 1 || a->debug_shading_mode > 4) return c->fail("light gbuffer: unsupported debug mode");
    CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex"); CHKE(a->temporal_output_tex, KJB_FMT_RGBA16_FLOAT, "temporal_output_tex", W, H); CHKE(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex", W, H);
    CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H); CHKE(a->shadow_mask_tex, a->shadow_mask_tex.format == KJB_FMT_RG16_FLOAT ? KJB_FMT_RG16_FLOAT : KJB_FMT_R8_UNORM, "shadow_mask_tex", W, H); CHKE(a->rtr_tex, KJB_FMT_R11G11B10_UFLOAT, "rtr_tex", W, H);
    CHKE(a->rtdgi_tex, KJB_FMT_RGBA16_FLOAT, "rtdgi_tex", W, H); CHK(a->unconvolved_sky_cube_tex, KJB_FMT_RGBA16_FLOAT, "unconvolved_sky_cube_tex");
    LightGbufferImgs t{img_ro(a->gbuffer_tex), img_ro(a->depth_tex), img_ro(a->shadow_mask_tex), img_ro(a->rtr_tex), img_ro(a->rtdgi_tex), img_ro(a->unconvolved_sky_cube_tex),
                       img_rw(a->temporal_output_tex), img_rw(a->output_tex), a->shadow_mask_tex.format == KJB_FMT_RG16_FLOAT ? 1 : 0};
    const float real_sun_radius_cos = kjb_cos(0.53f * 0.5f * KJB_PI_F / 180.0f);
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_light_gbuffer, KJB_GRID2D(W, H, 32, 8), c->g, t, f4(a->output_tex_size[0], a->output_tex_size[1], a->output_tex_size[2], a->output_tex_size[3]), a->debug_shading_mode, real_sun_radius_cos);
    KJB_PASS_EPILOGUE(c, P);
}

static ShadowKernelWeights shadow_kernel_weights() {   // FFX_DNSR_Shadows_KernelWeight (tileclassification.hlsl:169-184), KERNEL_RADIUS 8
    auto W = [](int i) { return kjb_exp(-3.0f * float(i * i) / ((8 + 1.0f) * (8 + 1.0f))); };
    float sum = 0; sum += W(0);
    for (int c = 1; c <= 8; ++c) sum += 2 * W(c);
    const float inv = kjb_rcp(sum);
    ShadowKernelWeights r; for (int i = 0; i <= 8; ++i) r.k[i] = W(i) * inv;
    return r;
}
static bool shadow_extent_ok(kjb_context* c, const char* P, const float* its, const uint32_t* ext, const kjb_image& tile_img) {
    const uint32_t W = uint32_t(its[0]), H = uint32_t(its[1]);
    if (ext[0] != (W + 7) / 8 || ext[1] != (H + 3) / 4 || tile_img.width != ext[0] || tile_img.height != ext[1]) { c->fail(std::string(P) + ": bitpacked_shadow_mask_extent must be ceil(W/8) x ceil(H/4) and match the tile image"); return false; }
    return true;
}
int kjb_pass_shadow_bitpack(kjb_context* c, const kjb_shadow_bitpack_args* a) {
    const char* P = "shadow bitpack"; const uint32_t W = uint32_t(a->input_tex_size[0]), H = uint32_t(a->input_tex_size[1]);
    CHKE(a->input_tex, KJB_FMT_R8_UNORM, "input_tex", W, H); CHK(a->output_tex, KJB_FMT_R32_UINT, "output_tex");
    if (!shadow_extent_ok(c, P, a->input_tex_size, a->bitpacked_shadow_mask_extent, a->output_tex)) return 1;
    const uint32_t tx = (W + 7) / 8, ty = (H + 3) / 4;
    KJB_ROWS(c, ty);
    KJB_LAUNCH(c, k_shadow_bitpack, KJB_GRID2D(tx, ty, 32, 8), img_ro(a->input_tex), img_rw(a->output_tex), W, a->bitpacked_shadow_mask_extent[0], tx, ty);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_shadow_temporal(kjb_context* c, const kjb_shadow_temporal_args* a) {
    const char* P = "shadow temporal"; const uint32_t W = uint32_t(a->input_tex_size[0]), H = uint32_t(a->input_tex_size[1]);
    CHKE(a->shadow_mask_tex, KJB_FMT_R8_UNORM, "shadow_mask_tex", W, H); CHK(a->bitpacked_shadow_mask_tex, KJB_FMT_R32_UINT, "bitpacked_shadow_mask_tex");
    CHKE(a->prev_moments_tex, KJB_FMT_RGBA16_FLOAT, "prev_moments_tex", W, H); CHKE(a->prev_accum_tex, KJB_FMT_RG16_FLOAT, "prev_accum_tex", W, H);
    CHKE(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex", W, H); CHKE(a->output_moments_tex, KJB_FMT_RGBA16_FLOAT, "output_moments_tex", W, H);
    CHKE(a->temporal_output_tex, KJB_FMT_RG16_FLOAT, "temporal_output_tex", W, H); CHK(a->meta_output_tex, KJB_FMT_R32_UINT, "meta_output_tex");
    if (!shadow_extent_ok(c, P, a->input_tex_size, a->bitpacked_shadow_mask_extent, a->bitpacked_shadow_mask_tex) || !shadow_extent_ok(c, P, a->input_tex_size, a->bitpacked_shadow_mask_extent, a->meta_output_tex)) return 1;
    ShadowTemporalImgs t{img_ro(a->shadow_mask_tex), img_ro(a->bitpacked_shadow_mask_tex), img_ro(a->prev_moments_tex), img_ro(a->prev_accum_tex), img_ro(a->reprojection_tex),
                         img_rw(a->output_moments_tex), img_rw(a->temporal_output_tex), img_rw(a->meta_output_tex)};
    KJB_ROWS(c, H);
    if (kjb__rows.y0 % 8) return c->fail("shadow temporal: the scissor must start on a multiple of 8 rows (8x8 denoiser tiles)");
    KJB_LAUNCH_SYNC(c, k_shadow_temporal, KJB_DIMS(dim3((W + 7) / 8, (uint32_t(kjb__rows.y1 - kjb__rows.y0) + 7) / 8), dim3(8, 8)), c->g, t, F4A(a->input_tex_size), a->bitpacked_shadow_mask_extent[0], shadow_kernel_weights());
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_shadow_spatial(kjb_context* c, const kjb_shadow_spatial_args* a) {
    const char* P = "shadow spatial"; const uint32_t W = uint32_t(a->input_tex_size[0]), H = uint32_t(a->input_tex_size[1]);
    CHKE(a->input_tex, KJB_FMT_RG16_FLOAT, "input_tex", W, H); CHK(a->meta_tex, KJB_FMT_R32_UINT, "meta_tex"); CHKE(a->geometric_normal_tex, KJB_FMT_A2R10G10B10_UNORM, "geometric_normal_tex", W, H);
    CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H); CHKE(a->output_tex, KJB_FMT_RG16_FLOAT, "output_tex", W, H);
    if (!shadow_extent_ok(c, P, a->input_tex_size, a->bitpacked_shadow_mask_extent, a->meta_tex)) return 1;
    if (a->step_size != 1 && a->step_size != 2 && a->step_size != 4) return c->fail("shadow spatial: step_size must be 1, 2 or 4 (the group-shared apron is 4 texels)");
    ShadowSpatialImgs t{img_ro(a->input_tex), img_ro(a->meta_tex), img_ro(a->geometric_normal_tex), img_ro(a->depth_tex), img_rw(a->output_tex)};
    KJB_ROWS(c, H);
    if (kjb__rows.y0 % 8) return c->fail("shadow spatial: the scissor must start on a multiple of 8 rows (8x8 denoiser tiles)");
    KJB_LAUNCH_SYNC(c, k_shadow_spatial, KJB_DIMS(dim3((W + 7) / 8, (uint32_t(kjb__rows.y1 - kjb__rows.y0) + 7) / 8), dim3(8, 8)), t, F4A(a->input_tex_size), a->bitpacked_shadow_mask_extent[0], int(a->step_size));
    KJB_PASS_EPILOGUE(c, P);
}

int kjb_pass_sample_lights(kjb_context* c, const kjb_sample_lights_args* a) {
    const char* P = "sample lights"; const uint32_t W = a->out0_tex.width, H = a->out0_tex.height;
    CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex"); CHK(a->out0_tex, KJB_FMT_RGBA16_FLOAT, "out0_tex"); CHKE(a->out1_tex, KJB_FMT_RGBA32_FLOAT, "out1_tex", W, H); CHKE(a->out2_tex, KJB_FMT_RGBA8_SNORM, "out2_tex", W, H);
    if (c->g.fc.triangle_light_count == 0) return c->fail("sample lights: the scene has no triangle lights");
    if (!c->tlas_valid) return c->fail("sample lights: no acceleration structure (call kjb_rebuild_tlas)");
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_sample_lights, KJB_GRID2D(W, H, KJB_RAY_BX, KJB_RAY_BY), c->g, img_ro(a->depth_tex), img_rw(a->out0_tex), img_rw(a->out1_tex), img_rw(a->out2_tex), F4A(a->gbuffer_tex_size));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_spatial_reuse_lights(kjb_context* c, const kjb_spatial_reuse_lights_args* a) {
    const char* P = "spatial reuse lights"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R11G11B10_UFLOAT, "output_tex"); CHKE(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H);
    const uint32_t HW = a->hit0_tex.width, HH = a->hit0_tex.height;
    CHK(a->hit0_tex, KJB_FMT_RGBA16_FLOAT, "hit0_tex"); CHKE(a->hit1_tex, KJB_FMT_RGBA32_FLOAT, "hit1_tex", HW, HH); CHKE(a->hit2_tex, KJB_FMT_RGBA8_SNORM, "hit2_tex", HW, HH);
    CHKE(a->half_view_normal_tex, KJB_FMT_RGBA8_SNORM, "half_view_normal_tex", HW, HH); CHKE(a->half_depth_tex, KJB_FMT_R32_FLOAT, "half_depth_tex", HW, HH);
    if (!a->spatial_resolve_offsets) return c->fail("spatial reuse lights: spatial_resolve_offsets is null");
    const size_t bytes = sizeof(int32_t) * 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT;
    if (!c->d_resolve_offsets) { c->d_resolve_offsets = (int32_t*)dev_alloc(bytes); if (!c->d_resolve_offsets) return c->fail("spatial reuse lights: out of device memory"); c->h_resolve_offsets.clear(); }
    if (c->h_resolve_offsets.size() != 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT || memcmp(c->h_resolve_offsets.data(), a->spatial_resolve_offsets, bytes) != 0) {
        c->h_resolve_offsets.assign(a->spatial_resolve_offsets, a->spatial_resolve_offsets + 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT);
        if (dev_h2d(c, c->d_resolve_offsets, c->h_resolve_offsets.data(), bytes)) return c->fail("spatial reuse lights: upload failed");
    }
    ReuseLightsImgs t{img_ro(a->gbuffer_tex), img_ro(a->depth_tex), img_ro(a->hit0_tex), img_ro(a->hit1_tex), img_ro(a->hit2_tex), img_ro(a->half_view_normal_tex), img_ro(a->half_depth_tex), img_rw(a->output_tex)};
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_spatial_reuse_lights, KJB_GRID2D(W, H, 32, 8), c->g, t, F4A(a->output_tex_size), (const int32_t*)c->d_resolve_offsets);
    KJB_PASS_EPILOGUE(c, P);
}

}  // extern "C"
