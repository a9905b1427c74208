// Temporal anti-aliasing / temporal super-resolution as sm_90a kernels — one per render-graph pass of
// crates/lib/kajiya/src/renderers/taa.rs:41-185 (shaders: /root/reference/assets/shaders/taa/, inc/unjitter_taa.hlsl, inc/image.hlsl).
// All seven passes are small-stencil screen-space filters: 32x8 thread blocks on the pass's grid, 8-byte RGBA16F texels =>
// 256 B per warp-row request; constant filter weights (exp(-r^2 ...)) are evaluated once on the host with the numeric
// contract and passed as kernel parameters.
#include "kjb_context.h"

using namespace kjb;

KJB_DEV float3 taa_decode_rgb(float3 v) { const float mc = max3(v.x, v.y, v.z); return v * kjb_sqrt(kjb_max(0.0f, mc)) / kjb_max(1e-20f, mc); }   // taa_common.hlsl:46-53
KJB_DEV float3 taa_encode_rgb(float3 v) { const float mc = max3(v.x, v.y, v.z); return v * (mc * mc) / kjb_max(1e-20f, mc); }                     // :55-62
KJB_DEV float3 taa_input_remap(float4 v) { return rgb_to_ycbcr(taa_decode_rgb(xyz(v))); }
struct W9 { float w[9]; };
struct W25t { float w[25]; };

// ------------------------------------------------------------------ T1 reproject_history.hlsl:38-129
KJB_DEV bool t1_should_dilate0(const Img& reprojection_tex, int x, int y, float2 irs, float4 its) {
    const int rx = int(kjb_cvt_u32((float(x) + 0.5f) * irs.x)), ry = int(kjb_cvt_u32((float(y) + 0.5f) * irs.y));
    float2 v = xy(ld_rgba16s(reprojection_tex, rx - 1, ry - 1)); float2 vel_min = v, vel_max = v;
    v = xy(ld_rgba16s(reprojection_tex, rx + 1, ry - 1)); vel_min = vmin(vel_min, v); vel_max = vmax(vel_max, v);
    v = xy(ld_rgba16s(reprojection_tex, rx - 1, ry + 1)); vel_min = vmin(vel_min, v); vel_max = vmax(vel_max, v);
    v = xy(ld_rgba16s(reprojection_tex, rx + 1, ry + 1)); vel_min = vmin(vel_min, v); vel_max = vmax(vel_max, v);
    const float2 d = vel_max - vel_min, thr = 0.1f * vmax(f2(its.z, its.w), vabs(vel_max + vel_min));
    return d.x > thr.x || d.y > thr.y;
}
// 8 x 32-thread blocks whose rows start at a multiple of 4: a warp is the shader's wave, an 8x4 pixel patch with lane = x + 8*(y & 3), and the
// WaveReadLaneAt(^2) / (^16) exchange of the dilation flag (reproject_history.hlsl:80-82) is two warp shuffles
#define T1_BX 8
#define T1_BY 32
KJB_KERNEL(256) k_taa_reproject(const __grid_constant__ Globals g, Img history_tex, Img reprojection_tex, Img depth_tex, ImgW output_tex, ImgW closest_velocity_output, float4 its, float4 ots, Rows kjb_rows) {
    const int x = int(blockIdx.x) * T1_BX + int(threadIdx.x), y = (kjb_rows.y0 & ~3) + int(blockIdx.y) * T1_BY + int(threadIdx.y);
    const int W = output_tex.w, H = output_tex.h;
    const float2 irs = f2(its.x, its.y) / f2(ots.x, ots.y);
    float dilate = t1_should_dilate0(reprojection_tex, x, y, irs, its) ? 1.0f : 0.0f;   // every lane, also those past the image edge (like the shader's)
    dilate = kjb_max(dilate, warp_xor(dilate, 2));     // (x^2, y)
    dilate = kjb_max(dilate, warp_xor(dilate, 16));    // (x, y^2) and, transitively, (x^2, y^2)
    if (x >= W || y >= H || y < kjb_rows.y0 || y >= kjb_rows.y1) return;
    const float ped = g.fc.pre_exposure_delta;
    const int rx = int(kjb_cvt_u32((float(x) + 0.5f) * irs.x)), ry = int(kjb_cvt_u32((float(y) + 0.5f) * irs.y));
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    int cx = rx, cy = ry;
    const bool should_dilate = dilate != 0.0f;
    if (should_dilate) {
        float reproj_depth = ld_r32f(depth_tex, rx, ry);
        for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
            const float d = ld_r32f(depth_tex, rx + xx, ry + yy);
            if (d > reproj_depth) { reproj_depth = d; cx = rx + xx; cy = ry + yy; }
        }
    }
    const float2 reproj_xy = xy(ld_rgba16s(reprojection_tex, cx, cy));
    st_rg16f(closest_velocity_output, x, y, reproj_xy.x, reproj_xy.y);
    const float2 history_uv = uv + reproj_xy;
    // image_sample_catmull_rom_5tap (inc/image.hlsl:85-162, no corner taps), bilinear taps with clamp addressing, HistoryRemap
    const Img& ht = history_tex;
    auto smp = [&](float2 p) {
        const float4 h = bilinear_clamp(ht.w, ht.h, p, [&](int sx, int sy) { return ld_rgba16f(ht, sx, sy); });
        return f4(taa_decode_rgb(xyz(h) * ped), h.w);
    };
    const float2 texSize = f2(ots.x, ots.y);
    const float2 samplePos = history_uv * texSize;
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
    st_rgba16f(output_tex, x, y, f4(xyz(result), kjb_max(0.0f, result.w)));
}

// ------------------------------------------------------------------ T2 filter_input.hlsl:32-89
// Tiled: the block's (32+2)x(8+2) footprint of input_tex and depth_tex arrives in shared memory through one TMA group; the per-texel
// decode (taa_input_remap: sqrt, three divisions, RGB->YCbCr) then runs once per texel instead of 18 times (two 3x3 passes), and the part
// of a tap's weight that does not depend on the luma cutoff (depth term x spatial weight) is evaluated once for both passes.  `pow(t, 8)`
// of t == 1 is exactly 1 under the numeric contract (kjb_log2(1) = 0, kjb_exp2(0) = 1), which is every tap of the first pass
// (cutoff 1e10): those skip the exp2/log2 pair.  Same operations in the same order per output value => the same bits as t2_inner.
// tile origins are 16-byte aligned in their image (row-wise bulk copies need it): 2 texels of left apron for the 8-byte RGBA16F texels, 4 for R32F depth
#define T2_TW 36
#define T2_AX 2
#define T2_DW 40
#define T2_DX 4
#define T2_LW 34   /* the logical (32+2)-wide footprint the decoded arrays hold */
#define T2_TH 10
KJB_DEVONLY float t2_pow8_sat(float luma_cutoff, float luma) { const float t = kjb_saturate(luma_cutoff / luma); return t == 1.0f ? 1.0f : kjb_pow(t, 8.0f); }
KJB_KERNEL(256) k_taa_filter_input_tiled(int tile_mode_, Img input_tex, Img depth_tex,
                                         ImgW output_tex, ImgW dev_output_tex, W9 dw, Rows kjb_rows) {
    constexpr int P8 = tile_pitch<8>(T2_TW), P4 = tile_pitch<4>(T2_DW);
    __shared__ __align__(128) uint2 s_raw[P8 * T2_TH];
    __shared__ __align__(128) float s_depth[P4 * T2_TH];
    __shared__ float s_y[T2_LW * T2_TH], s_cb[T2_LW * T2_TH], s_cr[T2_LW * T2_TH];
    __shared__ __align__(8) uint64_t bar;
    const int tid = int(threadIdx.y) * 32 + int(threadIdx.x);
    const int bx0 = int(blockIdx.x) * 32, by0 = kjb_rows.y0 + int(blockIdx.y) * 8 - 1;
    tile_group_begin(&bar, 0, tile_mode_, tid);
    uint32_t staged = tile_issue<uint2, T2_TW, T2_TH>(s_raw, input_tex, bx0 - T2_AX, by0, &bar, tile_mode_, tid, 256);
    staged += tile_issue<float, T2_DW, T2_TH>(s_depth, depth_tex, bx0 - T2_DX, by0, &bar, tile_mode_, tid, 256);
    tile_group_wait(&bar, 0, tile_mode_, staged, tid);
    for (int i = tid; i < T2_LW * T2_TH; i += 256) {
        const int lx = i % T2_LW, ly = i / T2_LW;
        const float3 c = taa_input_remap(half4_to_float4(s_raw[ly * P8 + lx + (T2_AX - 1)]));
        s_y[i] = c.x; s_cb[i] = c.y; s_cr[i] = c.z;
    }
    __syncthreads();
    const int x = int(blockIdx.x) * 32 + int(threadIdx.x), y = kjb_rows.y0 + int(blockIdx.y) * 8 + int(threadIdx.y);
    if (x >= output_tex.w || y >= output_tex.h || y >= kjb_rows.y1) return;
    const int tx = int(threadIdx.x) + 1, ty = int(threadIdx.y) + 1;
    const float center_depth = s_depth[ty * P4 + tx + (T2_DX - 1)];
    float wd[9];
    float3 iex = f3(0.0f), iex2 = f3(0.0f), clamped_iex = f3(0.0f); float iwsum = 0, clamped_iwsum = 0;
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
        const int k = (yy + 1) * 3 + (xx + 1), ti = (ty + yy) * T2_LW + (tx + xx);
        const float3 sv = f3(s_y[ti], s_cb[ti], s_cr[ti]);
        const float depth = s_depth[(ty + yy) * P4 + (tx + xx) + (T2_DX - 1)];
        float w = 1;
        w *= kjb_exp2(-kjb_min(16.0f, 200.0f * inverse_depth_relative_diff(center_depth, depth)));
        w *= dw.w[k];
        wd[k] = w;
        w *= t2_pow8_sat(1e10f, sv.x);
        clamped_iwsum += w; clamped_iex = mad(sv, w, clamped_iex);
        iwsum += 1; iex += sv; iex2 += sv * sv;
    }
    const float3 fi_clamped_ex = clamped_iex / clamped_iwsum;
    iex = iex / iwsum; iex2 = iex2 / iwsum;
    const float3 fi_var = vmax(f3(0.0f), iex2 - iex * iex);
    const float luma_cutoff = fi_clamped_ex.x * 1.001f;
    clamped_iex = f3(0.0f); clamped_iwsum = 0;
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
        const int k = (yy + 1) * 3 + (xx + 1), ti = (ty + yy) * T2_LW + (tx + xx);
        const float3 sv = f3(s_y[ti], s_cb[ti], s_cr[ti]);
        const float w = wd[k] * t2_pow8_sat(luma_cutoff, sv.x);
        clamped_iwsum += w; clamped_iex = mad(sv, w, clamped_iex);
    }
    st_rgba16f(output_tex, x, y, f4(clamped_iex / clamped_iwsum, 0));
    st_rgba16f(dev_output_tex, x, y, f4(vsqrt(fi_var), 0));
}

// ------------------------------------------------------------------ T3 filter_history.hlsl:15-62
KJB_DEV float3 t3_filter(const Img& input_tex, float2 uv, float4 its, float luma_cutoff, int k, const float* dw) {
    float3 iex = f3(0.0f); float iwsum = 0;
    const int sx = kjb_cvt_i32(kjb_floor(uv.x * its.x + 1e-3f)), sy = kjb_cvt_i32(kjb_floor(uv.y * its.y + 1e-3f));
    for (int y = -k; y <= k; ++y) for (int x = -k; x <= k; ++x) {
        const float3 s = rgb_to_ycbcr(xyz(ld_rgba16f(input_tex, sx + x, sy + y)));
        float w = 1;
        w *= dw[(y + 2) * 5 + (x + 2)];
        w *= kjb_pow(kjb_saturate(luma_cutoff / s.x), 8.0f);
        iwsum += w; iex = mad(s, w, iex);
    }
    return iex / iwsum;
}
KJB_KERNEL(256) k_taa_filter_history(Img input_tex, ImgW output_tex, float4 its, float4 ots, int k, W25t dw, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float filtered_luma = t3_filter(input_tex, uv, its, 1e10f, k, dw.w).x;
    st_rgba16f(output_tex, x, y, f4(t3_filter(input_tex, uv, its, filtered_luma * 1.001f, k, dw.w), 0));
}

// Tiled variant for the native-resolution case (input extent == output extent, k == 1: every tap lies in the block's 34x10 footprint):
// RGB->YCbCr once per texel, pow(1, 8) shortcut in the first pass as in T2.
KJB_KERNEL(256) k_taa_filter_history_tiled(int tile_mode_, Img input_tex, ImgW output_tex, float4 its, float4 ots, W25t dw, Rows kjb_rows) {
    constexpr int P8 = tile_pitch<8>(T2_TW);
    __shared__ __align__(128) uint2 s_raw[P8 * T2_TH];
    __shared__ float s_y[T2_LW * T2_TH], s_cb[T2_LW * T2_TH], s_cr[T2_LW * T2_TH];
    __shared__ __align__(8) uint64_t bar;
    const int tid = int(threadIdx.y) * 32 + int(threadIdx.x);
    const int bx0 = int(blockIdx.x) * 32 - 1, by0 = kjb_rows.y0 + int(blockIdx.y) * 8 - 1;   // logical footprint origin
    tile_group_begin(&bar, 0, tile_mode_, tid);
    const uint32_t staged = tile_issue<uint2, T2_TW, T2_TH>(s_raw, input_tex, bx0 + 1 - T2_AX, by0, &bar, tile_mode_, tid, 256);
    tile_group_wait(&bar, 0, tile_mode_, staged, tid);
    for (int i = tid; i < T2_LW * T2_TH; i += 256) {
        const int lx = i % T2_LW, ly = i / T2_LW;
        const float3 c = rgb_to_ycbcr(xyz(half4_to_float4(s_raw[ly * P8 + lx + (T2_AX - 1)])));
        s_y[i] = c.x; s_cb[i] = c.y; s_cr[i] = c.z;
    }
    __syncthreads();
    const int x = int(blockIdx.x) * 32 + int(threadIdx.x), y = kjb_rows.y0 + int(blockIdx.y) * 8 + int(threadIdx.y);
    if (x >= output_tex.w || y >= output_tex.h || y >= kjb_rows.y1) return;
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const int sx = kjb_cvt_i32(kjb_floor(uv.x * its.x + 1e-3f)), sy = kjb_cvt_i32(kjb_floor(uv.y * its.y + 1e-3f));
    const int tx = sx - bx0, ty = sy - by0;   // == threadIdx + 1 whenever the two extents are equal; a texel the tile does not hold falls back to global loads
    const bool in_tile = tx >= 1 && tx <= T2_LW - 2 && ty >= 1 && ty <= T2_TH - 2;
    float3 iex = f3(0.0f); float iwsum = 0; float3 taps[9];
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
        const int k = (yy + 1) * 3 + (xx + 1);
        taps[k] = in_tile ? f3(s_y[(ty + yy) * T2_LW + tx + xx], s_cb[(ty + yy) * T2_LW + tx + xx], s_cr[(ty + yy) * T2_LW + tx + xx]) : rgb_to_ycbcr(xyz(ld_rgba16f(input_tex, sx + xx, sy + yy)));
        float w = 1;
        w *= dw.w[(yy + 2) * 5 + (xx + 2)];
        w *= t2_pow8_sat(1e10f, taps[k].x);
        iwsum += w; iex = mad(taps[k], w, iex);
    }
    const float luma_cutoff = (iex / iwsum).x * 1.001f;
    iex = f3(0.0f); iwsum = 0;
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
        const int k = (yy + 1) * 3 + (xx + 1);
        float w = 1;
        w *= dw.w[(yy + 2) * 5 + (xx + 2)];
        w *= t2_pow8_sat(luma_cutoff, taps[k].x);
        iwsum += w; iex = mad(taps[k], w, iex);
    }
    st_rgba16f(output_tex, x, y, f4(iex / iwsum, 0));
}

// ------------------------------------------------------------------ T4 input_prob.hlsl:47-109
KJB_KERNEL(256) k_taa_input_prob(const __grid_constant__ Globals g, Img filtered_input_tex, Img filtered_input_dev_tex, Img filtered_history_tex, Img reprojection_tex, Img smooth_var_history_tex,
                                 Img velocity_history_tex, ImgW output_tex, float4 its, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    float input_prob = 0;
    float3 ivar = f3(0.0f);
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) ivar = vmax(ivar, xyz(ld_rgba16f(filtered_input_dev_tex, x + xx * 2, y + yy * 2)));
    ivar = ivar * ivar;
    const float2 sop = f2(g.fc.view_constants.sample_offset_pixels[0], g.fc.view_constants.sample_offset_pixels[1]);
    const float2 input_uv = (f2(float(x), float(y)) + sop) * f2(its.z, its.w);
    const int2 hp = nearest_clamp_px(filtered_history_tex, input_uv);
    const float3 closest_history = xyz(ld_rgba16f(filtered_history_tex, hp.x, hp.y));
    const float2 rxy = xy(ld_rgba16s(reprojection_tex, x, y));
    const Img& sv = smooth_var_history_tex; const Img& vh = velocity_history_tex;
    const float3 closest_smooth_var = xyz(bilinear_clamp(sv.w, sv.h, input_uv + rxy, [&](int sx, int sy) { return ld_rgba16f(sv, sx, sy); }));
    const float4 cv4 = bilinear_clamp(vh.w, vh.h, input_uv + rxy, [&](int sx, int sy) { const float2 v = ld_rg16f(vh, sx, sy); return f4(v.x, v.y, 0, 0); });
    const float2 closest_vel = f2(cv4.x, cv4.y) * g.fc.delta_time_seconds;
    const float3 combined_var = vmin(closest_smooth_var, ivar * 10.0f);
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) {
        const float3 s = xyz(ld_rgba16f(filtered_input_tex, x + xx, y + yy));
        const float3 idiff = s - closest_history;
        const float2 vel = xy(ld_rgba16s(reprojection_tex, x + xx, y + yy));
        const float vdiff = length((vel - closest_vel) / vmax(f2(1.0f), vabs(vel + closest_vel)));
        const float prob = kjb_exp2(-1.0f * length(idiff * idiff / vmax(f3(1e-6f), combined_var)) - 1000 * vdiff);
        input_prob = kjb_max(input_prob, prob);
    }
    st_raw<uint16_t>(output_tex, x, y, uint16_t(kjb_f32_to_f16(input_prob)));
}

// ------------------------------------------------------------------ T5 filter_prob.hlsl / T6 filter_prob2.hlsl
KJB_KERNEL(256) k_taa_prob_filter(Img input_tex, ImgW output_tex, Rows kjb_rows) {
    KJB_PX; if (x >= output_tex.w || y >= output_tex.h) return;
    float prob = ld_r16f(input_tex, x, y);
    for (int yy = -1; yy <= 1; ++yy) for (int xx = -1; xx <= 1; ++xx) prob = kjb_max(prob, ld_r16f(input_tex, x + xx, y + yy));
    st_raw<uint16_t>(output_tex, x, y, uint16_t(kjb_f32_to_f16(prob)));
}
// exponential_squish of a probability is a function of the texel alone, and each texel is a tap of 25 pixels: the block squishes its
// (32 + 8) x (8 + 8) footprint once into shared memory (640 exp2 instead of 6400) and every pixel sums its 25 taps in the reference's order.
KJB_KERNEL(256) k_taa_prob_filter2(Img input_tex, ImgW output_tex, Rows kjb_rows) {
    constexpr int TW = 32 + 8, TH = 8 + 8;
    __shared__ float s_sq[TW * TH];
    const int tid = int(threadIdx.y) * 32 + int(threadIdx.x);
    const int bx0 = int(blockIdx.x) * 32 - 4, by0 = kjb_rows.y0 + int(blockIdx.y) * 8 - 4;
    for (int i = tid; i < TW * TH; i += 256) {
        const float neighbor_prob = ld_r16f(input_tex, bx0 + i % TW, by0 + i / TW);
        s_sq[i] = kjb_exp2(-kjb_clamp(10.0f * neighbor_prob, 0.0f, 100.0f));     // exponential_squish
    }
    __syncthreads();
    const int x = int(blockIdx.x) * 32 + int(threadIdx.x), y = kjb_rows.y0 + int(blockIdx.y) * 8 + int(threadIdx.y);
    if (x >= output_tex.w || y >= output_tex.h || y >= kjb_rows.y1) return;
    float2 weighted_prob = f2(0.0f);
    for (int yy = -2; yy <= 2; ++yy) for (int xx = -2; xx <= 2; ++xx)
        weighted_prob += f2(s_sq[(int(threadIdx.y) + 4 + yy * 2) * TW + int(threadIdx.x) + 4 + xx * 2], 1);
    const float prob = kjb_max(0.0f, -1.0f / 10.0f * kjb_log2(1e-30f + weighted_prob.x / weighted_prob.y));   // exponential_unsquish
    st_raw<uint16_t>(output_tex, x, y, uint16_t(kjb_f32_to_f16(prob)));
}

// ------------------------------------------------------------------ T7 taa.hlsl:94-338 (+ inc/unjitter_taa.hlsl:58-125)
struct Unjittered { float4 color; float coverage; float3 ex, ex2; };
// sample_image_unjitter_taa for kernel_scale 1 (`u`: colour, coverage, moments) and 0.333 (`b`: colour and coverage, all taa.hlsl uses of it)
// in ONE walk over the 3x3 taps: the decoded tap colour is shared, every accumulator keeps its own tap order.  `fetch(x, y)` returns
// taa_input_remap of the input texel (bx + x, by + y).
template <typename F>
KJB_DEV void sample_image_unjitter_taa2(int img_w, int img_h, int ox, int oy, float2 output_tex_size, float2 sample_offset_pixels, F fetch, Unjittered& u, float4& b_color, float& b_coverage) {
    const float2 irs = f2(float(img_w), float(img_h)) / output_tex_size;
    const int bx = kjb_cvt_i32((float(ox) + 0.5f) * irs.x), by = kjb_cvt_i32((float(oy) + 0.5f) * irs.y);
    const float2 dst_sample_loc = f2(float(ox), float(oy)) + 0.5f;
    const float2 base_src_sample_loc = (f2(float(bx), float(by)) + 0.5f + sample_offset_pixels * f2(1, -1)) / irs;
    float4 res = f4(0.0f), bres = f4(0.0f); float3 ex = f3(0.0f), ex2 = f3(0.0f); float dev_wt_sum = 0.0f, wt_sum = 0.0f, bwt_sum = 0.0f;
    const float kdm = 1.0f * 1.0f, bkdm = 1.0f * 0.333f;
    for (int y = -1; y <= 1; ++y) for (int x = -1; x <= 1; ++x) {
        const float2 src_sample_loc = base_src_sample_loc + f2(float(x), float(y)) / irs;
        const float4 col = f4(fetch(bx, by, x, y), 1);
        {
            const float2 sco = (src_sample_loc - dst_sample_loc) * kdm;
            const float dist2 = dot(sco, sco);
            const float dev_wt = kjb_exp2(-dist2 * irs.x);
            const float wt = kjb_exp2(-10 * dist2 * irs.x);
            res = mad(col, wt, res); wt_sum += wt;
            ex = mad(xyz(col), dev_wt, ex); ex2 = mad(xyz(col) * xyz(col), dev_wt, ex2); dev_wt_sum += dev_wt;
        }
        {
            const float2 sco = (src_sample_loc - dst_sample_loc) * bkdm;
            const float dist2 = dot(sco, sco);
            const float wt = kjb_exp2(-10 * dist2 * irs.x);
            bres = mad(col, wt, bres); bwt_sum += wt;
        }
    }
    u.color = res; u.coverage = wt_sum; u.ex = ex / dev_wt_sum; u.ex2 = ex2 / dev_wt_sum;
    b_color = bres; b_coverage = bwt_sum;
}
struct TaaImgs { Img input_tex, history_tex, reprojection_tex, closest_velocity_tex, velocity_history_tex, smooth_var_history_tex, input_prob_tex;
                 ImgW temporal_output_tex, output_tex, smooth_var_output_tex, velocity_output_tex; };
// one output pixel of taa.hlsl:94-338; `hist(xx, yy)` = history texel (x + xx, y + yy) as float4, `inp(bx, by, dx, dy)` = taa_input_remap of input texel (bx + dx, by + dy)
template <typename FH, typename FI>
KJB_DEV void taa_px(const Globals& g, const TaaImgs& t, float4 its, float4 ots, const W25t& bw, int x, int y, FH hist, FI inp) {
    const float2 sop = f2(g.fc.view_constants.sample_offset_pixels[0], g.fc.view_constants.sample_offset_pixels[1]);
    const float dt = g.fc.delta_time_seconds;
    const float2 irf = f2(its.x, its.y) / f2(ots.x, ots.y);
    const int rx = int(kjb_cvt_u32((float(x) + 0.5f) * irf.x)), ry = int(kjb_cvt_u32((float(y) + 0.5f) * irf.y));
    const float s4[4] = {ots.x, ots.y, ots.z, ots.w};
    const float2 uv = get_uv(x, y, s4);
    const float4 history_packed = hist(0, 0);
    float3 history = xyz(history_packed);
    float history_coverage = kjb_max(0.0f, history_packed.w);
    float4 bhistory_packed;
    {   // fetch_blurred_history(px, 2, 1): w = exp(-r^2), host-evaluated table
        float4 csum = f4(0.0f); float wsum = 0;
        for (int yy = -2; yy <= 2; ++yy) for (int xx = -2; xx <= 2; ++xx) {
            const float w = bw.w[(yy + 2) * 5 + (xx + 2)];
            csum = mad(hist(xx, yy), w, csum); wsum += w;
        }
        bhistory_packed = csum / wsum;
    }
    float3 bhistory = xyz(bhistory_packed);
    const float3 bhistory_coverage = f3(bhistory_packed.w);
    history = rgb_to_ycbcr(history); bhistory = rgb_to_ycbcr(bhistory);
    const float4 reproj = ld_rgba16s(t.reprojection_tex, rx, ry);
    const float2 cvel = ld_rg16f(t.closest_velocity_tex, x, y);
    const float2 reproj_xy = cvel;
    Unjittered center_sample; float4 bcenter_color; float bcenter_coverage;
    sample_image_unjitter_taa2(t.input_tex.w, t.input_tex.h, x, y, f2(ots.x, ots.y), sop, inp, center_sample, bcenter_color, bcenter_coverage);
    float coverage = center_sample.coverage;
    float3 center = xyz(center_sample.color);
    const float3 bcenter = xyz(bcenter_color) / bcenter_coverage;
    history = vlerp(history, bcenter, kjb_saturate(1.0f - history_coverage));
    bhistory = vlerp(bhistory, bcenter, f3(kjb_saturate(1.0f - bhistory_coverage.x), kjb_saturate(1.0f - bhistory_coverage.y), kjb_saturate(1.0f - bhistory_coverage.z)));
    const float input_prob = ld_r16f(t.input_prob_tex, rx, ry);
    const float3 ex = center_sample.ex, ex2 = center_sample.ex2;
    const float3 var = vmax(f3(0.0f), ex2 - ex * ex);
    const Img& sv = t.smooth_var_history_tex; const Img& vh = t.velocity_history_tex;
    const float3 prev_var = f3(bilinear_clamp(sv.w, sv.h, uv + reproj_xy, [&](int sx, int sy) { return ld_rgba16f(sv, sx, sy); }).x);
    const float2 vel_now = cvel / dt;
    const float4 vp4 = bilinear_clamp(vh.w, vh.h, uv + cvel, [&](int sx, int sy) { const float2 v = ld_rg16f(vh, sx, sy); return f4(v.x, v.y, 0, 0); });
    const float2 vel_prev = f2(vp4.x, vp4.y);
    const float vel_diff = length((vel_now - vel_prev) / vmax(f2(1.0f), vabs(vel_now + vel_prev)));
    const float var_blend = kjb_saturate(0.3f + 0.7f * (1 - reproj.z) + vel_diff);
    float3 smooth_var = vmax(var, vlerp(prev_var, var, var_blend));
    smooth_var = vlerp(var, smooth_var, kjb_saturate(input_prob));
    const float3 input_dev = vsqrt(var);
    float3 clamped_history;
    {
        const float box_n_deviations = kjb_lerp(0.8f, 3.0f, input_prob);
        const float3 nmin = ex - input_dev * box_n_deviations, nmax = ex + input_dev * box_n_deviations;
        const float3 clamped_bhistory = vclamp(bhistory, nmin, nmax);
        const float clamping_event = length(vmax(f3(0.0f), vmax(bhistory - nmax, nmin - bhistory)) / vmax(f3(0.01f), ex));
        const float3 outlier3 = vmax(f3(0.0f), (vmax(nmin - history, history - nmax)) / (0.1f + vmax(vmax(vabs(history), vabs(ex)), f3(1e-5f))));
        const float3 boutlier3 = vmax(f3(0.0f), (vmax(nmin - bhistory, bhistory - nmax)) / (0.1f + vmax(vmax(vabs(bhistory), vabs(ex)), f3(1e-5f))));
        const float outlier = kjb_max(outlier3.x, kjb_max(outlier3.y, outlier3.z));
        const float boutlier = kjb_max(boutlier3.x, kjb_max(boutlier3.y, boutlier3.z));
        const float2 huv = uv + reproj_xy, hs = vsaturate(huv);
        if (huv.x == hs.x && huv.y == hs.y) {
            const float non_disoccluding_outliers = kjb_max(0.0f, outlier - boutlier) * 10;
            const float3 unclamped_history_detail = history - clamped_bhistory;
            const float temporal_clamping_detail = kjb_abs(unclamped_history_detail.x / kjb_max(1e-3f, input_dev.x)) * 0.05f;
            const float temporal_stability = kjb_saturate(1 - temporal_clamping_detail);
            const float allow_unclamped_detail = kjb_saturate(non_disoccluding_outliers) * temporal_stability;
            float3 history_detail = history - bhistory;
            history_detail = vlerp(history_detail, unclamped_history_detail, allow_unclamped_detail);
            const float initial_bclamp_amount = kjb_saturate(dot(clamped_bhistory - bhistory, bcenter - bhistory)
                / kjb_max(1e-5f, length(clamped_bhistory - bhistory) * length(bcenter - bhistory)));
            const float effective_clamp_amount = kjb_saturate(initial_bclamp_amount) * (1 - allow_unclamped_detail);
            const float keep_detail = 1 - effective_clamp_amount;
            history_detail *= keep_detail;
            clamped_history = clamped_bhistory + history_detail;
            if (irf.x < 1.0f) history_coverage *= kjb_lerp(kjb_lerp(0.0f, 0.9f, keep_detail), 1.0f, kjb_saturate(10 * clamping_event));
        } else {
            clamped_history = clamped_bhistory; coverage = 1; center = bcenter; history_coverage = 0;
        }
        clamped_history = vlerp(clamped_history, history, kjb_smoothstep(0.5f, 1.0f, input_prob));
    }
    float total_coverage = kjb_max(1e-5f, history_coverage + coverage);
    float3 temporal_result = (clamped_history * history_coverage + center) / total_coverage;
    const float max_coverage = kjb_max(2.0f, 8.0f / (irf.x * irf.y));
    total_coverage = kjb_min(max_coverage, total_coverage);
    coverage = total_coverage;
    st_rgba16f(t.smooth_var_output_tex, x, y, f4(smooth_var, 0));
    temporal_result = ycbcr_to_rgb(temporal_result);
    temporal_result = taa_encode_rgb(temporal_result);
    temporal_result = vmax(f3(0.0f), temporal_result);
    st_rgba16f(t.temporal_output_tex, x, y, f4(temporal_result, coverage));
    st_rgba16f(t.output_tex, x, y, f4(temporal_result, 0));
    const float2 vo = cvel / dt;
    st_rg16f(t.velocity_output_tex, x, y, vo.x, vo.y);
}
// Tiled variant: the history (32+4)x(8+4) footprint — and, at native resolution (NATIVE: input extent == output extent, so the input tap
// (bx + dx, by + dy) is (x + dx, y + dy)), the input (32+2)x(8+2) footprint — through one TMA group; f16 -> f32 of the history and taa_input_remap
// of the input run once per texel instead of once per tap (25 and 18 taps per pixel).  With temporal upsampling the input taps of a block do not form
// a fixed footprint and stay global loads; the history, which is always at output resolution, is still staged.
#define T7_HW 36
#define T7_HH 12
template <bool NATIVE>
KJB_DEVONLY void taa_tiled_block(int tile_mode_, const Globals& g, const TaaImgs& t, float4 its, float4 ots, const W25t& bw, const Rows& kjb_rows) {
    constexpr int PH = tile_pitch<8>(T7_HW), PI = tile_pitch<8>(T2_TW);
    __shared__ __align__(128) uint2 s_hraw[PH * T7_HH];
    __shared__ __align__(128) uint2 s_iraw[NATIVE ? PI * T2_TH : 2];
    __shared__ float4 s_hist[T7_HW * T7_HH];
    __shared__ float s_y[NATIVE ? T2_LW * T2_TH : 1], s_cb[NATIVE ? T2_LW * T2_TH : 1], s_cr[NATIVE ? T2_LW * T2_TH : 1];
    __shared__ __align__(8) uint64_t bar;
    const int tid = int(threadIdx.y) * 32 + int(threadIdx.x);
    const int bx0 = int(blockIdx.x) * 32, by0 = kjb_rows.y0 + int(blockIdx.y) * 8;
    tile_group_begin(&bar, 0, tile_mode_, tid);
    uint32_t staged = tile_issue<uint2, T7_HW, T7_HH>(s_hraw, t.history_tex, bx0 - 2, by0 - 2, &bar, tile_mode_, tid, 256);
    if (NATIVE) staged += tile_issue<uint2, T2_TW, T2_TH>(s_iraw, t.input_tex, bx0 - T2_AX, by0 - 1, &bar, tile_mode_, tid, 256);
    tile_group_wait(&bar, 0, tile_mode_, staged, tid);
    for (int i = tid; i < T7_HW * T7_HH; i += 256) s_hist[i] = half4_to_float4(s_hraw[(i / T7_HW) * PH + (i % T7_HW)]);
    if (NATIVE) for (int i = tid; i < T2_LW * T2_TH; i += 256) {
        const float3 c = taa_input_remap(half4_to_float4(s_iraw[(i / T2_LW) * PI + (i % T2_LW) + (T2_AX - 1)]));
        s_y[i] = c.x; s_cb[i] = c.y; s_cr[i] = c.z;
    }
    __syncthreads();
    const int x = bx0 + int(threadIdx.x), y = by0 + int(threadIdx.y);
    if (x >= t.temporal_output_tex.w || y >= t.temporal_output_tex.h || y >= kjb_rows.y1) return;
    const int tx = int(threadIdx.x), ty = int(threadIdx.y);
    auto hist = [&](int xx, int yy) { return s_hist[(ty + 2 + yy) * T7_HW + (tx + 2 + xx)]; };
    if (NATIVE) taa_px(g, t, its, ots, bw, x, y, hist, [&](int bx, int by, int dx, int dy) { const int ti = (by - by0 + 1 + dy) * T2_LW + (bx - bx0 + 1 + dx); return f3(s_y[ti], s_cb[ti], s_cr[ti]); });
    else taa_px(g, t, its, ots, bw, x, y, hist, [&](int bx, int by, int dx, int dy) { return taa_input_remap(ld_rgba16f(t.input_tex, bx + dx, by + dy)); });
}
KJB_KERNEL(256) k_taa_tiled(int tile_mode_, const __grid_constant__ Globals g, const __grid_constant__ TaaImgs t, float4 its, float4 ots, const __grid_constant__ W25t bw, Rows kjb_rows) {
    taa_tiled_block<true>(tile_mode_, g, t, its, ots, bw, kjb_rows);
}
KJB_KERNEL(256) k_taa_tiled_upsampling(int tile_mode_, const __grid_constant__ Globals g, const __grid_constant__ TaaImgs t, float4 its, float4 ots, const __grid_constant__ W25t bw, Rows kjb_rows) {
    taa_tiled_block<false>(tile_mode_, g, t, its, ots, bw, kjb_rows);
}

#define F4A(a) f4((a)[0], (a)[1], (a)[2], (a)[3])
#define CHK(img, fmt, name) if (!check_img(c, (img), (fmt), P, name)) return 1
#define CHKE(img, fmt, name, w, h) if (!check_img(c, (img), (fmt), P, name, (w), (h))) return 1

extern "C" {

int kjb_pass_taa_reproject(kjb_context* c, const kjb_taa_reproject_args* a) {
    const char* P = "reproject taa"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex"); CHKE(a->history_tex, KJB_FMT_RGBA16_FLOAT, "history_tex", W, H); CHK(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex");
    CHK(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex"); CHKE(a->closest_velocity_output, KJB_FMT_RG16_FLOAT, "closest_velocity_output", W, H);
    KJB_ROWS(c, H);
    KJB_LAUNCH_SYNC(c, k_taa_reproject, KJB_DIMS(dim3((W + T1_BX - 1) / T1_BX, unsigned(kjb__rows.y1 - (kjb__rows.y0 & ~3) + T1_BY - 1) / T1_BY, 1), dim3(T1_BX, T1_BY, 1)), c->g, img_ro(a->history_tex), img_ro(a->reprojection_tex), img_ro(a->depth_tex), img_rw(a->output_tex), img_rw(a->closest_velocity_output),
               F4A(a->input_tex_size), F4A(a->output_tex_size));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_taa_filter_input(kjb_context* c, const kjb_taa_filter_input_args* a) {
    const char* P = "taa filter input"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex"); CHKE(a->input_tex, KJB_FMT_RGBA16_FLOAT, "input_tex", W, H); CHKE(a->depth_tex, KJB_FMT_R32_FLOAT, "depth_tex", W, H);
    CHKE(a->dev_output_tex, KJB_FMT_RGBA16_FLOAT, "dev_output_tex", W, H);
    W9 dw; for (int y = -1; y <= 1; ++y) for (int x = -1; x <= 1; ++x) dw.w[(y + 1) * 3 + (x + 1)] = kjb_exp(-(0.8f / float(1 * 1)) * float(x * x + y * y));
    KJB_ROWS(c, H);
    KJB_LAUNCH_SYNC(c, k_taa_filter_input_tiled, KJB_GRID2D(W, H, 32, 8), tile_mode({&a->input_tex, &a->depth_tex}), img_ro(a->input_tex), img_ro(a->depth_tex), img_rw(a->output_tex), img_rw(a->dev_output_tex), dw);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_taa_filter_history(kjb_context* c, const kjb_taa_filter_history_args* a) {
    const char* P = "taa filter history"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex"); CHK(a->input_tex, KJB_FMT_RGBA16_FLOAT, "input_tex");
    const int k = (a->input_tex_size[0] / a->output_tex_size[0] > 1.75f) ? 2 : 1;
    W25t dw; for (int y = -2; y <= 2; ++y) for (int x = -2; x <= 2; ++x) dw.w[(y + 2) * 5 + (x + 2)] = kjb_exp(-(0.8f / float(k * k)) * float(x * x + y * y));
    KJB_ROWS(c, H);
    if (k == 1 && a->input_tex.width == W && a->input_tex.height == H)
        KJB_LAUNCH_SYNC(c, k_taa_filter_history_tiled, KJB_GRID2D(W, H, 32, 8), tile_mode({&a->input_tex}), img_ro(a->input_tex), img_rw(a->output_tex), F4A(a->input_tex_size), F4A(a->output_tex_size), dw);
    else
        KJB_LAUNCH(c, k_taa_filter_history, KJB_GRID2D(W, H, 32, 8), img_ro(a->input_tex), img_rw(a->output_tex), F4A(a->input_tex_size), F4A(a->output_tex_size), k, dw);
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_taa_input_prob(kjb_context* c, const kjb_taa_input_prob_args* a) {
    const char* P = "taa input prob"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R16_FLOAT, "output_tex"); CHKE(a->filtered_input_tex, KJB_FMT_RGBA16_FLOAT, "filtered_input_tex", W, H); CHKE(a->filtered_input_dev_tex, KJB_FMT_RGBA16_FLOAT, "filtered_input_dev_tex", W, H);
    CHKE(a->filtered_history_tex, KJB_FMT_RGBA16_FLOAT, "filtered_history_tex", W, H); CHKE(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex", W, H);
    CHK(a->smooth_var_history_tex, KJB_FMT_RGBA16_FLOAT, "smooth_var_history_tex"); CHK(a->velocity_history_tex, KJB_FMT_RG16_FLOAT, "velocity_history_tex");
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_taa_input_prob, KJB_GRID2D(W, H, 32, 8), c->g, img_ro(a->filtered_input_tex), img_ro(a->filtered_input_dev_tex), img_ro(a->filtered_history_tex), img_ro(a->reprojection_tex),
               img_ro(a->smooth_var_history_tex), img_ro(a->velocity_history_tex), img_rw(a->output_tex), F4A(a->input_tex_size));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_taa_prob_filter(kjb_context* c, const kjb_taa_prob_filter_args* a) {
    const char* P = "taa prob filter"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R16_FLOAT, "output_tex"); CHKE(a->input_tex, KJB_FMT_R16_FLOAT, "input_tex", W, H);
    KJB_ROWS(c, H);
    KJB_LAUNCH(c, k_taa_prob_filter, KJB_GRID2D(W, H, 32, 8), img_ro(a->input_tex), img_rw(a->output_tex));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_taa_prob_filter2(kjb_context* c, const kjb_taa_prob_filter_args* a) {
    const char* P = "taa prob filter2"; const uint32_t W = a->output_tex.width, H = a->output_tex.height;
    CHK(a->output_tex, KJB_FMT_R16_FLOAT, "output_tex"); CHKE(a->input_tex, KJB_FMT_R16_FLOAT, "input_tex", W, H);
    KJB_ROWS(c, H);
    KJB_LAUNCH_SYNC(c, k_taa_prob_filter2, KJB_GRID2D(W, H, 32, 8), img_ro(a->input_tex), img_rw(a->output_tex));
    KJB_PASS_EPILOGUE(c, P);
}
int kjb_pass_taa(kjb_context* c, const kjb_taa_args* a) {
    const char* P = "taa"; const uint32_t W = a->temporal_output_tex.width, H = a->temporal_output_tex.height;
    CHK(a->temporal_output_tex, KJB_FMT_RGBA16_FLOAT, "temporal_output_tex"); CHK(a->input_tex, KJB_FMT_RGBA16_FLOAT, "input_tex"); CHKE(a->history_tex, KJB_FMT_RGBA16_FLOAT, "history_tex", W, H);
    CHK(a->reprojection_tex, KJB_FMT_RGBA16_SNORM, "reprojection_tex"); CHKE(a->closest_velocity_tex, KJB_FMT_RG16_FLOAT, "closest_velocity_tex", W, H);
    CHKE(a->velocity_history_tex, KJB_FMT_RG16_FLOAT, "velocity_history_tex", W, H); CHKE(a->smooth_var_history_tex, KJB_FMT_RGBA16_FLOAT, "smooth_var_history_tex", W, H);
    CHK(a->input_prob_tex, KJB_FMT_R16_FLOAT, "input_prob_tex"); CHKE(a->output_tex, KJB_FMT_RGBA16_FLOAT, "output_tex", W, H);
    CHKE(a->smooth_var_output_tex, KJB_FMT_RGBA16_FLOAT, "smooth_var_output_tex", W, H); CHKE(a->velocity_output_tex, KJB_FMT_RG16_FLOAT, "velocity_output_tex", W, H);
    TaaImgs t;
    t.input_tex = img_ro(a->input_tex); t.history_tex = img_ro(a->history_tex); t.reprojection_tex = img_ro(a->reprojection_tex); t.closest_velocity_tex = img_ro(a->closest_velocity_tex);
    t.velocity_history_tex = img_ro(a->velocity_history_tex); t.smooth_var_history_tex = img_ro(a->smooth_var_history_tex); t.input_prob_tex = img_ro(a->input_prob_tex);
    t.temporal_output_tex = img_rw(a->temporal_output_tex); t.output_tex = img_rw(a->output_tex); t.smooth_var_output_tex = img_rw(a->smooth_var_output_tex); t.velocity_output_tex = img_rw(a->velocity_output_tex);
    W25t bw; for (int y = -2; y <= 2; ++y) for (int x = -2; x <= 2; ++x) { const float ox = float(x) * 1.0f, oy = float(y) * 1.0f; bw.w[(y + 2) * 5 + (x + 2)] = kjb_exp(-(ox * ox + oy * oy)); }
    KJB_ROWS(c, H);
    if (a->input_tex.width == W && a->input_tex.height == H)
        KJB_LAUNCH_SYNC(c, k_taa_tiled, KJB_GRID2D(W, H, 32, 8), tile_mode({&a->history_tex, &a->input_tex}), c->g, t, F4A(a->input_tex_size), F4A(a->output_tex_size), bw);
    else
        KJB_LAUNCH_SYNC(c, k_taa_tiled_upsampling, KJB_GRID2D(W, H, 32, 8), tile_mode({&a->history_tex}), c->g, t, F4A(a->input_tex_size), F4A(a->output_tex_size), bw);
    KJB_PASS_EPILOGUE(c, P);
}

}  // extern "C"
