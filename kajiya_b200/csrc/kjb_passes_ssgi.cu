// Screen-space ambient occlusion guide (SURVEY §8f N3) as sm_90a kernels — the four passes of
// crates/lib/kajiya/src/renderers/ssgi.rs, shader sources under /root/reference/assets/shaders/ssgi/ (USE_AO_ONLY 1: the shader's
// lighting gather only feeds an accumulator the AO-only output never reads, so it is not evaluated).
#include "kjb_context.h"

using namespace kjb;

KJB_DEV float ssgi_fast_sqrt(float x) { return kjb_u2f(0x1fbd1df5u + (kjb_f2u(x) >> 1u)); }   // ssgi.hlsl:51-53
KJB_DEV float ssgi_fast_acos(float inX) {                                                     // :56-61
    const float x = kjb_abs(inX);
    float res = -0.156583f * x + 1.57079632679489661923f;
    res *= ssgi_fast_sqrt(1.0f - x);
    return (inX >= 0) ? res : KJB_PI_F - res;
}
KJB_DEV float ssgi_integrate_arc(float h1, float h2, float n) {                               // :103-107
    float s1, c1, s2, c2, sn, cn;
    kjb_sincos(2.0f * h1 - n, &s1, &c1); kjb_sincos(2.0f * h2 - n, &s2, &c2); kjb_sincos(n, &sn, &cn);
    const float a = -c1 + cn + 2.0f * h1 * sn;
    const float b = -c2 + cn + 2.0f * h2 * sn;
    return 0.25f * (a + b);
}
KJB_DEV float update_horizion_angle(float prev, float cur, float blend) { return cur > prev ? kjb_lerp(prev, cur, blend) : prev; }

struct SsaoFrameTables { float temporal_rotation, temporal_offset; };   // temporal_rotations[frame % 6], temporal_offsets[frame / 6 % 4]

// ------------------------------------------------------------------ "ssao": ssgi.hlsl:214-341 (half-res, 6 samples per half slice)
KJB_KERNEL(256) k_ssao(const __grid_constant__ Globals g, Img gbuffer_tex, Img depth_tex, ImgW output_tex, float4 its, float4 ots, SsaoFrameTables ft, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float depth = ld_r32f(depth_tex, x, y);
    if (0.0f == depth) { st_r16f(output_tex, x, y, 0.0f); return; }
    const GbufferData gbuffer = gbuffer_unpack(ld_rgba32u(gbuffer_tex, x * 2, y * 2));
    const float3 normal_vs = normalize(xyz(mul(vc.world_to_view, f4(gbuffer.normal, 0))));
    const ViewRayContext vrc = ViewRayContext::from_uv_and_depth(vc, uv, depth);
    const float2 cs0 = uv_to_cs(uv);
    const float3 v_vs = -normalize(normalize(xyz(mul(vc.sample_to_view, f4(cs0.x, cs0.y, 0.0f, 1.0f)))));   // -normalize(ray_dir_vs())
    const float4 ray_hit_cs = vrc.ray_hit_cs;
    const float3 ray_hit_vs = vrc.ray_hit_vs();
    const uint32_t ux = uint32_t(x), uy = uint32_t(y);
    const float spatial_direction_noise = 1.0f / 16.0f * float((((ux + uy) & 3u) << 2u) + (ux & 3u));
    const float temporal_direction_noise = ft.temporal_rotation / 360.0f;
    const float spatial_offset_noise = (1.0f / 4.0f) * float((uy - ux) & 3u);
    const float ss_angle = kjb_frac(spatial_direction_noise + temporal_direction_noise) * KJB_PI_F;
    const float rand_offset = kjb_frac(spatial_offset_noise + ft.temporal_offset);
    float sa, ca; kjb_sincos(ss_angle, &sa, &ca);
    float2 cs_slice_dir = f2(ca * its.y / its.x, sa);
    float kernel_radius_ws, kernel_radius_shrinkage;
    {
        const float ws_to_cs = 0.5f / -ray_hit_vs.z * vc.view_to_clip.m[5];
        const float cs_kernel_radius_scaled = 60.0f * ots.w;   // SSGI_KERNEL_RADIUS
        kernel_radius_ws = cs_kernel_radius_scaled / ws_to_cs;
        cs_slice_dir = cs_slice_dir * cs_kernel_radius_scaled;
        kernel_radius_shrinkage = kjb_min(1.0f, 0.4f / cs_kernel_radius_scaled);   // MAX_KERNEL_RADIUS_CS
    }
    cs_slice_dir = cs_slice_dir * kernel_radius_shrinkage;
    kernel_radius_ws *= kernel_radius_shrinkage;
    const float3 center_vs = ray_hit_vs;
    cs_slice_dir = cs_slice_dir * (1.0f / 6.0f);
    const float* m = vc.sample_to_view.m;   // mul(float4(cs_slice_dir, 0, 0), sample_to_view).xy: row vector times matrix
    const float2 vs_slice_dir = f2(kjb_fma(cs_slice_dir.y, m[1], cs_slice_dir.x * m[0]), kjb_fma(cs_slice_dir.y, m[5], cs_slice_dir.x * m[4]));
    const float3 slice_normal_vs = normalize(cross(v_vs, f3(vs_slice_dir.x, vs_slice_dir.y, 0)));
    float3 proj_normal_vs = normal_vs - slice_normal_vs * dot(slice_normal_vs, normal_vs);
    const float slice_contrib_weight = length(proj_normal_vs);
    proj_normal_vs = proj_normal_vs / slice_contrib_weight;
    const float n_angle = ssgi_fast_acos(kjb_clamp(dot(proj_normal_vs, v_vs), -1.0f, 1.0f)) * kjb_sign(dot(vs_slice_dir, f2(proj_normal_vs.x - v_vs.x, proj_normal_vs.y - v_vs.y)));
    const float FRAC_PI_2 = 1.57079632679489661923f;
    float theta_cos_max1 = kjb_cos(n_angle - FRAC_PI_2), theta_cos_max2 = kjb_cos(n_angle + FRAC_PI_2);
    int p0x = x, p0y = y, p1x = x, p1y = y;
    // process_sample (:121-206) restricted to what feeds the horizon angles
    auto process_sample = [&](float4 sample_cs, float theta_cos_max) {
        if (sample_cs.z > 0) {
            const float4 sv4 = mul(vc.sample_to_view, sample_cs);
            const float3 sample_vs_offset = xyz(sv4) / sv4.w - center_vs;
            const float len = length(sample_vs_offset);
            const float sample_theta_cos = dot(sample_vs_offset, v_vs) / len;
            const float dist_n = len / kernel_radius_ws;
            if (dist_n < 1.0f) theta_cos_max = update_horizion_angle(theta_cos_max, sample_theta_cos, kjb_smoothstep(1.0f, 0.0f, dist_n));
        } else {
            theta_cos_max = update_horizion_angle(theta_cos_max, -1.0f, 1.0f);
        }
        return theta_cos_max;
    };
    for (uint32_t i = 0; i < 6u; ++i) {
        {
            const float t = float(i) + rand_offset;
            float4 sample_cs = f4(ray_hit_cs.x - cs_slice_dir.x * t, ray_hit_cs.y - cs_slice_dir.y * t, 0, 1);
            const float2 suv = cs_to_uv(f2(sample_cs.x, sample_cs.y));
            const int sx = kjb_cvt_i32(ots.x * suv.x), sy = kjb_cvt_i32(ots.y * suv.y);
            if (sx != p0x || sy != p0y) { p0x = sx; p0y = sy; sample_cs.z = ld_r32f(depth_tex, sx, sy); theta_cos_max1 = process_sample(sample_cs, theta_cos_max1); }
        }
        {
            const float t = float(i) + (1.0f - rand_offset);
            float4 sample_cs = f4(ray_hit_cs.x + cs_slice_dir.x * t, ray_hit_cs.y + cs_slice_dir.y * t, 0, 1);
            const float2 suv = cs_to_uv(f2(sample_cs.x, sample_cs.y));
            const int sx = kjb_cvt_i32(ots.x * suv.x), sy = kjb_cvt_i32(ots.y * suv.y);
            if (sx != p1x || sy != p1y) { p1x = sx; p1y = sy; sample_cs.z = ld_r32f(depth_tex, sx, sy); theta_cos_max2 = process_sample(sample_cs, theta_cos_max2); }
        }
    }
    const float h1 = -ssgi_fast_acos(theta_cos_max1), h2 = +ssgi_fast_acos(theta_cos_max2);
    const float h1p = n_angle + kjb_max(h1 - n_angle, -FRAC_PI_2), h2p = n_angle + kjb_min(h2 - n_angle, FRAC_PI_2);
    const float inv_ao = ssgi_integrate_arc(h1p, h2p, n_angle);
    st_r16f(output_tex, x, y, kjb_max(0.0f, kjb_max(0.0f, inv_ao) * slice_contrib_weight));
}

// ------------------------------------------------------------------ "ssao spatial": spatial_filter.hlsl:35-73
KJB_KERNEL(256) k_ssao_spatial(Img ssgi_tex, Img depth_tex, Img normal_tex, ImgW output_tex, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    float result = 0.0f, w_sum = 0.0f;
    const float center_depth = ld_r32f(depth_tex, x, y);
    if (center_depth != 0.0f) {
        const float3 center_normal = xyz(ld_rgba8s(normal_tex, x, y));
        w_sum = 1.0f; result = ld_r16f(ssgi_tex, x, y);
        for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
            if (xx == 0 && yy == 0) continue;
            const float depth = ld_r32f(depth_tex, x + xx, y + yy);
            if (depth != 0.0f) {
                const float depth_factor = kjb_exp2(-200.0f * kjb_abs(1.0f - (center_depth / depth)));
                float normal_factor = kjb_max(0.0f, dot(xyz(ld_rgba8s(normal_tex, x + xx, y + yy)), center_normal));
                normal_factor *= normal_factor; normal_factor *= normal_factor;
                float w = 1; w *= depth_factor; w *= normal_factor;
                w_sum += w; result = mad(ld_r16f(ssgi_tex, x + xx, y + yy), w, result);
            }
        }
    }
    st_r16f(output_tex, x, y, result / kjb_max(w_sum, 1e-5f));
}

// ------------------------------------------------------------------ "ssao upsample": upsample.hlsl:38-75
struct W9e { float w[9]; };   // exp(-(x^2 + y^2)), host-evaluated
KJB_KERNEL(256) k_ssao_upsample(Img ssgi_tex, Img depth_tex, ImgW output_tex, W9e gw, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    float result = 0.0f, w_sum = 0.0f;
    const float center_depth = ld_r32f(depth_tex, x, y);
    if (center_depth != 0.0f) {
        for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
            const int spx = x / 2 + xx, spy = y / 2 + yy;
            const float depth = ld_r32f(depth_tex, spx * 2, spy * 2);
            if (depth != 0.0f) {
                float w = 1; w *= kjb_exp2(-200.0f * kjb_abs(1.0f - (center_depth / depth)));
                w *= gw.w[(yy + 1) * 3 + (xx + 1)];
                w_sum += w; result = mad(ld_r16f(ssgi_tex, spx, spy), w, result);
            }
        }
    }
    st_r16f(output_tex, x, y, w_sum > 1e-6f ? result / w_sum : ld_r16f(ssgi_tex, x / 2, y / 2));
}

// ------------------------------------------------------------------ "ssao temporal": temporal_filter.hlsl:19-61
struct W25e { float w[25]; };   // exp(-3 r^2 / 9), host-evaluated
KJB_KERNEL(256) k_ssao_temporal(Img input_tex, Img history_tex, Img reprojection_tex, ImgW final_output_tex, ImgW history_output_tex, float4 ots, W25e gw, Rows kjb_rows) {
    KJB_PX; if (x >= history_output_tex.w || y >= history_output_tex.h) return;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float center = ld_r16f(input_tex, x, y);
    const float4 reproj = ld_rgba16s(reprojection_tex, x, y);
    const float history = bilinear_clamp(history_tex.w, history_tex.h, uv + xy(reproj), [&](int sx, int sy) { return f4(ld_r16f(history_tex, sx, sy), 0, 0, 1); }).x;
    float vsum = 0.0f, vsum2 = 0.0f, wsum = 0.0f;
    for (int yy = -2; yy <= 2; ++yy) for (int xx = -2; xx <= 2; ++xx) {
        const float neigh = ld_r16f(input_tex, x + xx * 2, y + yy * 2);
        const float w = gw.w[(yy + 2) * 5 + (xx + 2)];
        vsum = mad(neigh, w, vsum); vsum2 = mad(neigh * neigh, w, vsum2); wsum += w;
    }
    const float ex = vsum / wsum, ex2 = vsum2 / wsum;
    const float dev = kjb_sqrt(kjb_max(0.0f, ex2 - ex * ex));
    const float box_size = 0.5f, n_deviations = 5.0f;
    const float mid = kjb_lerp(center, ex, box_size * box_size);
    const float nmin = mid - dev * box_size * n_deviations, nmax = mid + dev * box_size * n_deviations;
    const float clamped_history = kjb_min(kjb_max(history, nmin), nmax);
    const float res = kjb_lerp(clamped_history, center, 1.0f / 8.0f);
    st_r16f(history_output_tex, x, y, res);
    st_r8u(final_output_tex, x, y, res);
}

#define F4A(a) f4((a)[0], (a)[1], (a)[2], (a)[3])
#define CHK(img, fmt, name) if (!check_img(c, (img), (fmt), P, name)) return 1
#define CHKE(img, fmt, name, w, h) if (!check_img(c, (img), (fmt), P, name, (w), (h))) return 1

extern "C" {

int kjb_pass_ssao(kjb_context* c, const kjb_ssao_args* a) {
    const char* P = "ssao"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R16_FLOAT, "output_tex"); CHK(a->gbuffer_tex, KJB_FMT_RGBA32_FLOAT, "gbuffer_tex"); CHKE(a->half_depth_tex, KJB_FMT_R32_FLOAT, "half_depth_tex", W, H);
    static const float temporal_rotations[6] = {60.0f, 300.0f, 180.0f, 240.0f, 120.0f, 0.0f};
    static const float temporal_offsets[4] = {0.0f, 0.5f, 0.25f, 0.75f};
    SsaoFrameTables ft; ft.temporal_rotation = temporal_rotations[c->g.fc.frame_index % 6u]; ft.temporal_offset = temporal_offsets[c->g.fc.frame_index / 6u % 4u];
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_ssao, KJB_GRID2D(W, H, 32, 8), c->g, img_ro(a->gbuffer_tex), img_ro(a->half_depth_tex), img_rw(a->output_tex), F4A(a->input_tex_size), F4A(a->output_tex_size), ft);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ssao_spatial(kjb_context* c, const kjb_ssao_spatial_args* a) {
    const char* P = "ssao spatial"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R16_FLOAT, "output_tex"); CHKE(a->ssgi_tex, KJB_FMT_R16_FLOAT, "ssgi_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H);
    CHKE(a->normal_tex, KJB_FMT_RGBA8_SNORM, "normal_tex", W, H);
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_ssao_spatial, KJB_GRID2D(W, H, 32, 8), img_ro(a->ssgi_tex), img_ro(a->depth_tex), img_ro(a->normal_tex), img_rw(a->output_tex));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ssao_upsample(kjb_context* c, const kjb_ssao_upsample_args* a) {
    const char* P = "ssao upsample"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R16_FLOAT, "output_tex"); CHK(a->ssgi_tex, KJB_FMT_R16_FLOAT, "ssgi_tex"); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H);
    W9e gw; for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) gw.w[(yy + 1) * 3 + (xx + 1)] = kjb_exp(-kjb_fma(float(yy), float(yy), float(xx) * float(xx)));   // exp(-dot(soffset, soffset))
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_ssao_upsample, KJB_GRID2D(W, H, 32, 8), img_ro(a->ssgi_tex), img_ro(a->depth_tex), img_rw(a->output_tex), gw);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_ssao_temporal(kjb_context* c, const kjb_ssao_temporal_args* a) {
    const char* P = "ssao temporal"; const uint32_t W = a->history_output_tex.width, H = a->history_output_tex.height;
    CHK(a->history_output_tex, KJB_FMT_R16_FLOAT, "history_output_tex"); CHKE(a->final_output_tex, KJB_FMT_R8_UNORM, "final_output_tex", W, H); CHKE(a->input_tex, KJB_FMT_R16_FLOAT, "input_tex", W, H);
    CHKE(a->history_tex, KJB_FMT_R16_FLOAT, "history_tex", W, H); CHKE(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex", W, H);
    W25e gw; for (int yy = -2; yy <= 2; ++yy) for (int xx = -2; xx <= 2; ++xx) gw.w[(yy + 2) * 5 + (xx + 2)] = kjb_exp(-3.0f * float(xx * xx + yy * yy) / float((2 + 1.) * (2 + 1.)));
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_ssao_temporal, KJB_GRID2D(W, H, 32, 8), img_ro(a->input_tex), img_ro(a->history_tex), img_ro(a->reprojection_tex), img_rw(a->final_output_tex), img_rw(a->history_output_tex),
               F4A(a->output_tex_size), gw);
    KJB_PASS_EPILOGUE(c, P);
}

}  // extern "C"
