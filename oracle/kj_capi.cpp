// ORACLE — TEST INFRASTRUCTURE ONLY (see kj_math.h header).
// The oracle exports the same C-ABI (include/kjb.h) as the CUDA library so the test harness and the
// host-side frame driver can run either behind identical calls.  "Device" memory is host memory here.
#include "kj_ctx.h"
#include <cstdlib>
#include <chrono>

namespace kjo {

extern "C" {

int kjb_abi_version(void) { return KJB_ABI_VERSION; }
const char* kjb_backend_name(void) { return "oracle-cpu"; }
int kjb_create(int, kjb_context** out) { *out = new kjb_context(); const char* e = getenv("KJO_THREADS"); if (e) (*out)->num_threads = atoi(e); return 0; }
void kjb_destroy(kjb_context* c) { delete c; }
int kjb_sync(kjb_context*) { return 0; }
const char* kjb_last_error(kjb_context* c) { return c ? c->last_error.c_str() : ""; }
uint64_t kjb_launch_count(kjb_context*) { return 0; }
void* kjb_stream(kjb_context*) { return nullptr; }
uint32_t kjb_format_texel_bytes(uint32_t f) { return format_texel_bytes(f); }

int kjb_image_alloc(kjb_context*, uint32_t w, uint32_t h, uint32_t layers, uint32_t fmt, kjb_image* out) {
    size_t bytes = size_t(w) * h * (layers ? layers : 1) * format_texel_bytes(fmt);
    out->data = calloc(bytes ? bytes : 1, 1); out->width = w; out->height = h; out->format = fmt; out->layers = layers ? layers : 1;
    return out->data ? 0 : 1;
}
int kjb_image_free(kjb_context*, kjb_image* img) { free(img->data); img->data = nullptr; return 0; }
static size_t img_bytes(const kjb_image* i) { return size_t(i->width) * i->height * i->layers * format_texel_bytes(i->format); }
int kjb_image_clear(kjb_context*, const kjb_image* img) { memset(img->data, 0, img_bytes(img)); return 0; }
int kjb_image_copy(kjb_context*, const kjb_image* dst, const kjb_image* src) { memcpy(dst->data, src->data, img_bytes(dst)); return 0; }
int kjb_image_fill_u8(kjb_context*, const kjb_image* img, uint32_t v) { memset(img->data, int(v), img_bytes(img)); return 0; }
int kjb_image_upload(kjb_context*, const kjb_image* dst, const void* src) { memcpy(dst->data, src, img_bytes(dst)); return 0; }
int kjb_image_download(kjb_context*, const kjb_image* src, void* dst) { memcpy(dst, src->data, img_bytes(src)); return 0; }
int kjb_buffer_alloc(kjb_context*, uint64_t n, kjb_buffer* out) { out->data = calloc(n ? n : 1, 1); out->size_bytes = n; return out->data ? 0 : 1; }
int kjb_buffer_free(kjb_context*, kjb_buffer* b) { free(b->data); b->data = nullptr; return 0; }
int kjb_buffer_upload(kjb_context*, const kjb_buffer* dst, uint64_t off, const void* src, uint64_t n) { memcpy((char*)dst->data + off, src, n); return 0; }
int kjb_buffer_download(kjb_context*, const kjb_buffer* src, uint64_t off, void* dst, uint64_t n) { memcpy(dst, (char*)src->data + off, n); return 0; }

int kjb_scene_set_geometry(kjb_context* c, const void* vb, uint64_t vb_bytes, const kjb_gpu_mesh* meshes, const uint32_t* counts, uint32_t n) {
    c->scene.vertices.assign((const uint8_t*)vb, (const uint8_t*)vb + vb_bytes);
    c->scene.meshes.assign(meshes, meshes + n);
    c->scene.mesh_index_counts.assign(counts, counts + n);
    return 0;
}
int kjb_scene_set_textures(kjb_context* c, const kjb_texture_desc* t, uint32_t n) {
    c->scene.textures.clear();
    for (uint32_t i = 0; i < n; ++i) {
        Texture tx; tx.width = t[i].width; tx.height = t[i].height; tx.mip_count = t[i].mip_count; tx.srgb = t[i].srgb;
        const uint8_t* p = t[i].texels;
        for (uint32_t m = 0; m < tx.mip_count; ++m) {
            size_t w = std::max(1u, tx.width >> m), h = std::max(1u, tx.height >> m);
            tx.mips.emplace_back(p, p + w * h * 4); p += w * h * 4;
        }
        c->scene.textures.push_back(std::move(tx));
    }
    return 0;
}
int kjb_rebuild_tlas(kjb_context* c, const kjb_instance* inst, uint32_t n) { c->scene.rebuild_tlas(inst, n); return 0; }
int kjb_set_frame_constants(kjb_context* c, const kjb_frame_constants* fc, const kjb_triangle_light* lights, uint32_t n) {
    c->g.fc = *fc; c->g.lights.assign(lights, lights + n);
    if (fc->triangle_light_count != n) { c->last_error = "triangle_light_count mismatch"; return 1; }
    return 0;
}
int kjb_comm_nccl_unique_id(void*) { return 1; }
int kjb_comm_init_nccl(kjb_context* c, const void*, uint32_t, uint32_t) { c->last_error = "oracle: no NCCL"; return 1; }
int kjb_comm_set_callback(kjb_context* c, kjb_allgather_fn fn, void* user, uint32_t rank, uint32_t nranks) { c->ag_fn = fn; c->ag_user = user; c->rank = rank; c->nranks = nranks; return 0; }
int kjb_comm_rank(kjb_context* c, uint32_t* r, uint32_t* n) { *r = c->rank; *n = c->nranks; return 0; }
int kjb_allgather(kjb_context* c, const void* send, void* recv, uint64_t bytes) {
    if (c->nranks <= 1) { memcpy(recv, send, bytes); return 0; }
    if (!c->ag_fn) { c->last_error = "kjb_allgather: no transport registered"; return 1; }
    return c->ag_fn(c->ag_user, send, recv, bytes);
}
int kjb_allgather_on(kjb_context* c, uint32_t, const void* send, void* recv, uint64_t bytes) { return kjb_allgather(c, send, recv, bytes); }
int kjb_memcpy_d2d(kjb_context*, void* dst, const void* src, uint64_t bytes) { memmove(dst, src, bytes); return 0; }
int kjb_memcpy_d2d_batch_on(kjb_context*, uint32_t, const kjb_copy_desc* c, uint32_t n) { for (uint32_t i = 0; i < n; ++i) if (c[i].bytes) memmove(c[i].dst, c[i].src, c[i].bytes); return 0; }
int kjb_memcpy_d2d_batch(kjb_context*, const kjb_copy_desc* c, uint32_t n) { for (uint32_t i = 0; i < n; ++i) if (c[i].bytes) memmove(c[i].dst, c[i].src, c[i].bytes); return 0; }
int kjb_set_scissor(kjb_context* c, uint32_t y0, uint32_t y1) { c->scissor_y0 = y0; c->scissor_y1 = y1; return 0; }
int kjb_graph_begin(kjb_context*) { return 0; }
int kjb_graph_end(kjb_context*) { return 0; }
int kjb_graph_select(kjb_context*, uint32_t) { return 0; }
int kjb_set_pass_queue(kjb_context*, uint32_t q) { return q == 0 ? 0 : 1; }
int kjb_async_passes_supported(kjb_context*) { return 0; }
int kjb_pass_ircache_export_requests(kjb_context*, const kjb_ircache_share_args*) { return 1; }   // tile-sharded frames run on the CUDA backend (and its emulator) only
int kjb_pass_ircache_merge_requests(kjb_context*, const kjb_ircache_share_args*) { return 1; }
int kjb_graph_stats(kjb_context*, uint64_t out[2]) { out[0] = out[1] = 0; return 0; }
int kjb_tlas_stats(kjb_context*, uint64_t out[2]) { out[0] = out[1] = 0; return 0; }   // the oracle rebuilds its median-split BVH whenever a transform changes
int kjb_set_debug_serial(kjb_context* c, uint32_t on) { c->cache_passes_parallel = on == 0; return 0; }   // default (never called): serial
int kjb_set_option(kjb_context*, uint32_t, uint32_t) { return 0; }   // performance options do not exist here
int kjb_image_upload_on(kjb_context* c, uint32_t, const kjb_image* dst, const void* src) { return kjb_image_upload(c, dst, src); }
int kjb_image_download_on(kjb_context* c, uint32_t, const kjb_image* src, void* dst) { return kjb_image_download(c, src, dst); }
int kjb_image_upload_rows_on(kjb_context*, uint32_t, const kjb_image* dst, const void* src, uint32_t r0, uint32_t n) {
    if (r0 + n > dst->height) return 1;
    const size_t rb = size_t(dst->width) * kjb_format_texel_bytes(dst->format); memcpy((char*)dst->data + rb * r0, (const char*)src + rb * r0, rb * n); return 0; }
int kjb_image_download_rows_on(kjb_context*, uint32_t, const kjb_image* src, void* dst, uint32_t r0, uint32_t n) {
    if (r0 + n > src->height) return 1;
    const size_t rb = size_t(src->width) * kjb_format_texel_bytes(src->format); memcpy((char*)dst + rb * r0, (const char*)src->data + rb * r0, rb * n); return 0; }
int kjb_event_record(kjb_context*, uint32_t, uint32_t) { return 0; }
int kjb_queue_wait_event(kjb_context*, uint32_t, uint32_t) { return 0; }
int kjb_event_synchronize(kjb_context*, uint32_t) { return 0; }   // the oracle's cache passes are always serial
int kjb_set_luts(kjb_context* c, const kjb_image* fg, const kjb_image* bn) { c->g.brdf_fg_lut = Img(*fg); c->g.blue_noise = Img(*bn); return 0; }
static std::chrono::steady_clock::time_point g_timer_slots[1024];
int kjb_timer_record(kjb_context*, uint32_t slot) { if (slot >= 1024) return 1; g_timer_slots[slot] = std::chrono::steady_clock::now(); return 0; }
int kjb_timer_elapsed_ms(kjb_context*, uint32_t a, uint32_t b, float* out) { if (a >= 1024 || b >= 1024) return 1; *out = std::chrono::duration<float, std::milli>(g_timer_slots[b] - g_timer_slots[a]).count(); return 0; }
int kjb_ray_counters(kjb_context* c, uint64_t out[2], int reset) {
    out[0] = c->scene.n_closest.load(); out[1] = c->scene.n_any.load();
    if (reset) { c->scene.n_closest = 0; c->scene.n_any = 0; }
    return 0;
}

// test-only known-answer hooks for the numeric core (tests/test_oracle_kat.py, vectors in tests/golden/kat_vectors.json)
uint32_t kjo_hash1(uint32_t x) { return hash1(x); }
uint32_t kjo_hash3(uint32_t x, uint32_t y, uint32_t z) { return hash3(x, y, z); }
uint32_t kjo_hash_combine2(uint32_t x, uint32_t y) { return hash_combine2(x, y); }
float kjo_u01(uint32_t h) { return uint_to_u01_float(h); }
uint32_t kjo_pack_normal_11_10_11(float x, float y, float z) { return asuint(pack_normal_11_10_11(float3(x, y, z))); }
void kjo_unpack_normal_11_10_11_no_normalize(uint32_t p, float* o) { float3 v = unpack_normal_11_10_11_no_normalize(asfloat(p)); o[0] = v.x; o[1] = v.y; o[2] = v.z; }
uint32_t kjo_float3_to_rgb9e5(float x, float y, float z) { return float3_to_rgb9e5(float3(x, y, z)); }
void kjo_rgb9e5_to_float3(uint32_t p, float* o) { float3 v = rgb9e5_to_float3(p); o[0] = v.x; o[1] = v.y; o[2] = v.z; }
uint32_t kjo_pack_color_888(float x, float y, float z) { return pack_color_888(float3(x, y, z)); }
uint32_t kjo_pack_2x16f(float a, float b) { return pack_2x16f_uint(float2(a, b)); }
// streams `n` (w, payload) candidates through Reservoir1spp::update with rng seed; returns payload, writes M, w_sum, rng
uint32_t kjo_reservoir_stream(uint32_t seed, const float* w, const uint32_t* payload, uint32_t n, float* out_m_wsum, uint32_t* out_rng) {
    Reservoir1spp r; uint32_t rng = seed;
    for (uint32_t i = 0; i < n; ++i) r.update(w[i], payload[i], rng);
    out_m_wsum[0] = r.M; out_m_wsum[1] = r.w_sum; *out_rng = rng;
    return r.payload;
}
void kjo_halfres_offset(uint32_t frame, int* o) { int2 v = halfres_subsample_offset(frame); o[0] = v.x; o[1] = v.y; }

// test-only helpers (not part of kjb.h): brute-force vs BVH closest hit for the traversal self-check
int kjo_trace_closest(kjb_context* c, const float* rays /* n x 8: o.xyz, tmin, d.xyz, tmax */, uint32_t n, int brute, float* out_t, uint32_t* out_tri) {
    for (uint32_t i = 0; i < n; ++i) {
        Ray r; r.origin = float3(rays[i * 8], rays[i * 8 + 1], rays[i * 8 + 2]); r.tmin = rays[i * 8 + 3];
        r.dir = float3(rays[i * 8 + 4], rays[i * 8 + 5], rays[i * 8 + 6]); r.tmax = rays[i * 8 + 7];
        Scene::HitInfo h = brute ? c->scene.closest_brute(r, false) : c->scene.closest(r, false);
        out_t[i] = h.hit ? h.t : -1.0f; out_tri[i] = h.tri;
    }
    return 0;
}
// The same with u, v, any-hit and back-face culling.  Rays and results as kjb_tlas_trace (include/kjb_tlas.h): n x 8 floats
// (o.xyz, tmin, d.xyz, tmax) in, n x 4 words (t, u, v bits, triangle id; 0, 0, 0, ~0 for a miss) out; with any_hit only word 3 counts (0 = hit).
int kjo_trace_rays(kjb_context* c, const float* rays, uint32_t n, int brute, int any_hit, int cull_back, uint32_t* out) {
    for (uint32_t i = 0; i < n; ++i) {
        Ray r; r.origin = float3(rays[i * 8], rays[i * 8 + 1], rays[i * 8 + 2]); r.tmin = rays[i * 8 + 3];
        r.dir = float3(rays[i * 8 + 4], rays[i * 8 + 5], rays[i * 8 + 6]); r.tmax = rays[i * 8 + 7];
        uint32_t* o = out + size_t(i) * 4;
        o[0] = o[1] = o[2] = 0; o[3] = 0xffffffffu;
        if (any_hit) {
            if (brute ? c->scene.closest_brute(r, cull_back != 0).hit : c->scene.any_hit(r, cull_back != 0)) o[3] = 0;
            continue;
        }
        Scene::HitInfo h = brute ? c->scene.closest_brute(r, cull_back != 0) : c->scene.closest(r, cull_back != 0);
        if (h.hit) { o[0] = asuint(h.t); o[1] = asuint(h.u); o[2] = asuint(h.v); o[3] = h.tri; }
    }
    return 0;
}

}  // extern "C"

}  // namespace kjo
