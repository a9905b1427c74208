// "reference pt": kajiya's reference path tracer (rt/reference_path_trace.rgen.hlsl:75-377) as an sm_90a kernel.
// In the reference this IS a GPU pass (renderers/reference.rs:8-25); it doubles as the converged-image yardstick for rtdgi.
#include "kjb_context.h"

using namespace kjb;

KJB_DEV float remap_unorm_to_gaussian(float xin, float truncation) {   // :60-72
    const float x = xin * 2.0f - 1.0f;
    const float ALPHA = 0.14f, INV_ALPHA = 1.0f / ALPHA, K = 2.0f / (KJB_PI_F * ALPHA);
    const float y = kjb_log(kjb_max(truncation, 1.0f - x * x));
    const float z = K + 0.5f * y;
    return kjb_sqrt(kjb_max(0.0f, kjb_sqrt(z * z - y * INV_ALPHA) - z)) * kjb_sign(x);
}

KJB_KERNEL(128) k_reference_pt(const __grid_constant__ Globals g, ImgW output_tex, uint32_t indirect_only, Rows kjb_rows) {
    KJB_PX; const int W = output_tex.w, H = output_tex.h; if (x >= W || y >= H) return;
    const kjb_view_constants& vc = g.fc.view_constants;
    const float4 prev = ld_rgba32f(as_ro(output_tex), x, y);
    if (!(prev.w < 1000)) return;
    float4 acc = f4(0.0f);
    uint32_t rng = hash_combine2(hash_combine2(uint32_t(x), hash1(uint32_t(y))), g.fc.frame_index);
    {
        float px_off0 = 0.5f, px_off1 = 0.5f;
        px_off0 += 0.4f * remap_unorm_to_gaussian(rand01(rng), 1e-8f);
        px_off1 += 0.4f * remap_unorm_to_gaussian(rand01(rng), 1e-8f);
        const float2 uv = (f2(float(x), float(y)) + f2(px_off0, px_off1)) / f2(float(W), float(H));
        Ray ray;
        {
            const ViewRayContext vrc = ViewRayContext::from_uv(vc, uv);
            ray.origin = vrc.ray_origin_ws(); ray.dir = normalize(vrc.ray_dir_ws()); ray.tmin = 0.0f; ray.tmax = KJB_FLT_MAX;
        }
        float3 throughput = f3(1.0f), total_radiance = f3(0.0f);
        float roughness_bias = 0.0f;
        RayCone cone; cone.width = 0; cone.spread_angle = pixel_cone_spread_angle_from_image_height(vc, float(H));
        cone.spread_angle *= 0.3f;
        const float3 sun_color = f3(g.sun_color[0], g.sun_color[1], g.sun_color[2]);
        for (uint32_t path_length = 0; path_length < 16u; ++path_length) {
            if (path_length == 1) ray.tmax = KJB_FLT_MAX;
            const GbufferPathVertex hit = gbuffer_raytrace(g, ray, cone, path_length, false);
            if (hit.is_hit) {
                cone = ray_cone_propagate(cone, 0.0f, hit.ray_t);
                float2 su; su.x = rand01(rng); su.y = rand01(rng);
                const float3 to_light_norm = sample_sun_direction(g.fc, su, true);
                const bool is_shadowed = (indirect_only && path_length == 0) || rt_is_shadowed(g, hit.position, to_light_norm, 1e-4f, KJB_FLT_MAX);
                GbufferData gbuffer = gbuffer_unpack(hit.gbuffer_packed);
                if (dot(gbuffer.normal, ray.dir) >= 0.0f) { if (0 == path_length) gbuffer.normal = -gbuffer.normal; else break; }
                if (indirect_only && path_length == 0) { gbuffer.albedo = f3(1.0f); gbuffer.metalness = 0.0f; }
                const float3x3 tangent_to_world = build_orthonormal_basis(gbuffer.normal);
                const float3 wi = mul(to_light_norm, tangent_to_world);
                float3 wo = mul(-ray.dir, tangent_to_world);
                if (wo.z < 0.0f) { wo.z *= -0.25f; wo = normalize(wo); }
                LayeredBrdf brdf = layered_brdf_from_gbuffer_ndotv(g, gbuffer, wo.z);
                brdf.specular_brdf.roughness = kjb_lerp(brdf.specular_brdf.roughness, 1.0f, roughness_bias);
                {
                    const float3 brdf_value = layered_evaluate_directional_light(brdf, wo, wi);
                    const float3 light_radiance = is_shadowed ? f3(0.0f) : sun_color;
                    total_radiance += throughput * brdf_value * light_radiance * kjb_max(0.0f, wi.z);
                    total_radiance += gbuffer.emissive * throughput;
                    if (g.fc.triangle_light_count > 0) {
                        const float light_selection_pmf = 1.0f / float(g.fc.triangle_light_count);
                        const uint32_t light_idx = hash1_mut(rng) % g.fc.triangle_light_count;
                        float2 urand; urand.x = rand01(rng); urand.y = rand01(rng);
                        const kjb_triangle_light tl = g.lights[light_idx];
                        const LightSample ls = sample_triangle_light(tl, urand);
                        const float3 to_light_ws = ls.pos - hit.position;
                        const float dist_to_light2 = dot(to_light_ws, to_light_ws);
                        const float3 to_light_norm_ws = to_light_ws * kjb_rsqrt(dist_to_light2);
                        const float to_psa_metric = kjb_max(0.0f, dot(to_light_norm_ws, gbuffer.normal)) * kjb_max(0.0f, dot(to_light_norm_ws, -ls.normal)) / dist_to_light2;
                        if (to_psa_metric > 0.0f) {
                            const float3 wi2 = mul(to_light_norm_ws, tangent_to_world);
                            const bool sh = rt_is_shadowed(g, hit.position, to_light_norm_ws, 1e-3f, kjb_sqrt(dist_to_light2) - 2e-3f);
                            total_radiance += sh ? f3(0.0f) : throughput * f3(tl.radiance[0], tl.radiance[1], tl.radiance[2]) * layered_evaluate(brdf, wo, wi2) / ls.pdf * to_psa_metric / light_selection_pmf;
                        }
                    }
                }
                float3 urand; urand.x = rand01(rng); urand.y = rand01(rng); urand.z = rand01(rng);
                const BrdfSample bs = layered_sample(brdf, wo, urand);
                if (bs.wi.z > 1e-6f) {
                    roughness_bias = kjb_lerp(roughness_bias, 1.0f, 0.5f * bs.approx_roughness);
                    ray.origin = hit.position; ray.dir = mul(tangent_to_world, bs.wi); ray.tmin = 1e-4f;
                    throughput *= bs.value_over_pdf;
                } else break;
                if (path_length >= 3u) {
                    const float rr_coin = rand01(rng);
                    const float continue_p = kjb_max(gbuffer.albedo.x, kjb_max(gbuffer.albedo.y, gbuffer.albedo.z));
                    if (rr_coin > continue_p) break; else throughput /= continue_p;
                }
            } else {
                total_radiance += throughput * atmosphere_default(g.fc, ray.dir, sun_direction(g.fc));
                break;
            }
        }
        if (total_radiance.x >= 0.0f && total_radiance.y >= 0.0f && total_radiance.z >= 0.0f) acc += f4(total_radiance, 1.0f);
    }
    const float tsc = acc.w + prev.w;
    const float lrp = acc.w / kjb_max(1.0f, tsc);
    const float3 cur = xyz(acc) / kjb_max(1.0f, acc.w);
    st_rgba32f(output_tex, x, y, f4(vmax(f3(0.0f), vlerp(xyz(prev), cur, lrp)), kjb_max(1.0f, tsc)));
}

extern "C" int kjb_pass_reference_path_trace(kjb_context* c, const kjb_reference_pt_args* a) {
    if (!check_img(c, a->output_tex, KJB_FMT_RGBA32_FLOAT, "reference pt", "output_tex")) return 1;
    KJB_ROWS(c, a->output_tex.height);
    KJB_LAUNCH(c, k_reference_pt, KJB_GRID2D(a->output_tex.width, a->output_tex.height, KJB_RAY_BX, KJB_RAY_BY), c->g, img_rw(a->output_tex), a->indirect_only);
    KJB_PASS_EPILOGUE(c, "reference pt");
}
