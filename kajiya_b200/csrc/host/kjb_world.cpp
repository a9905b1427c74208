// Host-side frame driver: C++ mirror of kajiya's Rust host for the ReSTIR-GI hot path.
//   WorldRenderer scene store / add_mesh        crates/lib/kajiya/src/world_renderer.rs:604-776
//   prepare_frame_constants                     world_renderer.rs:1001-1108
//   prepare_render_graph_standard (pass order)  crates/lib/kajiya/src/world_render_passes.rs:13-292
//   RtdgiRenderer::{reproject,render,temporal,spatial}   crates/lib/kajiya/src/renderers/rtdgi.rs
//   PingPongTemporalResource                    crates/lib/kajiya/src/renderers/mod.rs:73-103
//   camera / view constants                     crates/lib/kajiya/src/camera.rs, rust-shaders-shared/src/view_constants.rs
// It only calls the C-ABI in include/kjb.h (and, for tile-sharded frames with the cache, include/kjb_ircache_share.h).  No GPU, CUDA or oracle
// symbols are referenced directly.
#include "../../../include/kjb_world.h"
#include "../../../include/kjb_ircache_share.h"
#include <cmath>
#include <algorithm>
#include <cstring>
#include <cstdlib>
#include <map>
#include <string>
#include <vector>

namespace {

// ---------------------------------------------------------------- small column-major mat4 helpers (glam conventions)
struct M4 { float m[16]; };
M4 m4_identity() { M4 r{}; r.m[0] = r.m[5] = r.m[10] = r.m[15] = 1; return r; }
M4 m4_mul(const M4& a, const M4& b) {
    M4 r{};
    for (int c = 0; c < 4; ++c) for (int rr = 0; rr < 4; ++rr) {
        float s = 0; for (int k = 0; k < 4; ++k) s += a.m[k * 4 + rr] * b.m[c * 4 + k];
        r.m[c * 4 + rr] = s;
    }
    return r;
}
M4 m4_from_quat(const float q[4]) {   // glam Mat4::from_quat
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    const float x2 = x + x, y2 = y + y, z2 = z + z;
    const float xx = x * x2, xy = x * y2, xz = x * z2, yy = y * y2, yz = y * z2, zz = z * z2, wx = w * x2, wy = w * y2, wz = w * z2;
    M4 r = m4_identity();
    r.m[0] = 1 - (yy + zz); r.m[1] = xy + wz; r.m[2] = xz - wy;
    r.m[4] = xy - wz; r.m[5] = 1 - (xx + zz); r.m[6] = yz + wx;
    r.m[8] = xz + wy; r.m[9] = yz - wx; r.m[10] = 1 - (xx + yy);
    return r;
}
M4 m4_translation(float x, float y, float z) { M4 r = m4_identity(); r.m[12] = x; r.m[13] = y; r.m[14] = z; return r; }
void m4_store(kjb_mat4& d, const M4& s) { memcpy(d.m, s.m, sizeof(d.m)); }

struct CameraMatrices { M4 view_to_clip, clip_to_view, world_to_view, view_to_world; };

CameraMatrices camera_matrices(const kjb_world_frame& f, float aspect) {   // camera.rs:71-125
    CameraMatrices c;
    const float q[4] = {f.camera_rotation[0], f.camera_rotation[1], f.camera_rotation[2], f.camera_rotation[3]};
    const float qc[4] = {-q[0], -q[1], -q[2], q[3]};
    c.view_to_world = m4_mul(m4_translation(f.camera_position[0], f.camera_position[1], f.camera_position[2]), m4_from_quat(q));
    c.world_to_view = m4_mul(m4_from_quat(qc), m4_translation(-f.camera_position[0], -f.camera_position[1], -f.camera_position[2]));
    const float RADS_PER_DEG = 3.14159265358979323846f / 180.0f;   // f32::to_radians: self * (PI / 180), the constant folded in f32 (camera.rs:89)
    const float fov = (f.vertical_fov_deg > 0 ? f.vertical_fov_deg : 52.0f) * RADS_PER_DEG;
    const float znear = f.near_plane > 0 ? f.near_plane : 0.01f;
    const float h = std::cos(0.5f * fov) / std::sin(0.5f * fov);
    const float w = h / aspect;
    M4 v2c{}; v2c.m[0] = w; v2c.m[5] = h; v2c.m[11] = -1.0f; v2c.m[14] = znear;
    M4 c2v{}; c2v.m[0] = 1.0f / w; c2v.m[5] = 1.0f / h; c2v.m[11] = 1.0f / znear; c2v.m[14] = -1.0f;
    c.view_to_clip = v2c; c.clip_to_view = c2v;
    return c;
}

float radical_inverse(uint32_t n, uint32_t base) {   // world_renderer.rs:1116-1129
    float val = 0.0f; const float inv_base = 1.0f / float(base); float inv_bi = inv_base;
    while (n > 0) { uint32_t d = n % base; val += float(d) * inv_bi; n = uint32_t(float(n) * inv_base); inv_bi *= inv_base; }
    return val;
}

uint32_t pack_unit_direction_11_10_11(float x, float y, float z) {   // kajiya-asset/src/mesh.rs:452-458 (truncating!)
    auto cl = [](float v) { return v < -1.0f ? -1.0f : (v > 1.0f ? 1.0f : v); };
    uint32_t xi = uint32_t((cl(x) * 0.5f + 0.5f) * float((1u << 11) - 1u));
    uint32_t yi = uint32_t((cl(y) * 0.5f + 0.5f) * float((1u << 10) - 1u));
    uint32_t zi = uint32_t((cl(z) * 0.5f + 0.5f) * float((1u << 11) - 1u));
    return (zi << 21) | (yi << 11) | xi;
}

struct PingPong {   // renderers/mod.rs:73-103
    std::string output_key, history_key;
    explicit PingPong(const std::string& name) : output_key(name + ":0"), history_key(name + ":1") {}
};

}  // namespace

struct kjb_world {
    kjb_context* ctx = nullptr;
    kjb_world_desc desc{};
    uint32_t W = 0, H = 0, HW = 0, HH = 0;
    uint32_t frame_idx = 0;
    bool have_prev_camera = false;
    CameraMatrices prev_camera{};

    // scene (WorldRenderer fields)
    std::vector<uint8_t> vertex_buffer;
    std::vector<kjb_gpu_mesh> meshes;
    std::vector<uint32_t> mesh_index_counts;
    std::vector<std::vector<kjb_triangle_light>> mesh_lights;
    uint32_t frame_light_count = 0;   // triangle lights of the frame being rendered
    float sun_color_multiplier[3] = {1, 1, 1}, sky_ambient[3] = {0, 0, 0};   // world_renderer.rs:208-209,511-512
    uint32_t render_override_flags = 0; float render_override_material_roughness_scale = 1.0f;   // RenderOverrides (rust-shaders-shared frame_constants.rs)
    bool reset_reference_accumulation = false;   // world_renderer.rs:183
    uint32_t debug_shading_mode = 0;   // world_renderer.rs:201 (light_gbuffer.hlsl modes 0, 2, 3, 4)
    float sun_size_multiplier = 1.0f;  // WorldRenderer::sun_size_multiplier (world_renderer.rs:207,508): 1 = the sun as seen from Earth, 0 = point sun
    std::vector<uint32_t> instance_handles; std::map<uint32_t, uint32_t> instance_handle_to_index; uint32_t next_instance_handle = 0;   // world_renderer.rs:150-152
    std::vector<kjb_instance> instances, prev_instances;   // prev = transforms of the last rendered frame (retire_frame, world_renderer.rs:1110-1113)
    std::vector<std::vector<uint8_t>> texture_storage;
    std::vector<kjb_texture_desc> textures;
    bool geometry_dirty = true;

    std::map<std::string, kjb_image> images;
    std::string names_cache;
    std::string stop_after;
    bool stopped = false;
    uint64_t stats[4] = {0, 0, 0, 0};
    uint64_t launches_at_frame_start = 0;
    bool sky_valid = false; float sky_sun[3] = {0, 0, 0};
    bool lut_ready = false, noise_ready = false, ssao_filled = false;

    PingPong temporal_radiance_tex{"rtdgi.radiance"}, temporal_ray_orig_tex{"rtdgi.ray_orig"}, temporal_ray_tex{"rtdgi.ray"},
        temporal_reservoir_tex{"rtdgi.reservoir"}, temporal_candidate_tex{"rtdgi.candidate"}, temporal_invalidity_tex{"rtdgi.invalidity"},
        temporal2_tex{"rtdgi.temporal2"}, temporal2_variance_tex{"rtdgi.temporal2_var"}, temporal_hit_normal_tex{"rtdgi.hit_normal"};
    // RtrRenderer (rtr.rs:18-34, :55-72)
    PingPong rtr_temporal_tex{"rtr.temporal"}, rtr_ray_len_tex{"rtr.ray_len"}, rtr_temporal_irradiance_tex{"rtr.irradiance"}, rtr_temporal_ray_orig_tex{"rtr.ray_orig"},
        rtr_temporal_ray_tex{"rtr.ray"}, rtr_temporal_reservoir_tex{"rtr.reservoir"}, rtr_temporal_rng_tex{"rtr.rng"}, rtr_temporal_hit_normal_tex{"rtr.hit_normal"};
    bool rtr_reuse_rtdgi_rays = true;
    bool exchanged_this_frame = false, exchange_pending = false;   // tile exchange bookkeeping (tile_exchange_frame)
    uint32_t stream_frames = 0;   // streaming frames submitted (selects the input set / result stage)
    std::vector<int32_t> spatial_resolve_offsets;
    PingPong ssgi_tex{"ssgi"};   // SsgiRenderer (ssgi.rs:9-19)
    uint32_t half_normal_frame = 0xffffffffu, half_depth_frame = 0xffffffffu;   // GbufferDepth memoisation (renderers/mod.rs:54-70)
    PingPong shadow_denoise_accum{"shadow_denoise_accum"}, shadow_denoise_moments{"shadow_denoise_moments"};   // shadow_denoise.rs:5-17
    PingPong taa_temporal_tex{"taa"}, taa_temporal_velocity_tex{"taa.velocity"}, taa_temporal_smooth_var_tex{"taa.smooth_var"};   // taa.rs:19-27
    uint32_t OW = 0, OH = 0;   // temporal_upscale_extent

    // IrcacheRenderer (renderers/ircache.rs:92-100)
    bool ircache_initialized = false; uint32_t ircache_parity = 0;
    float ircache_grid_center[3] = {0, 0, 0}; int32_t ircache_cur_scroll[12][3] = {}, ircache_prev_scroll[12][3] = {};

    int err = 0;
    // ---- tile sharding (SURVEY §8e): this world owns half-res rows [ty0, ty1) of every frame
    bool tiled = false; uint32_t trank = 0, tcount = 1, ty0 = 0, ty1 = 0;
    kjb_buffer xchg_send[4]{}, xchg_recv[4]{}; uint64_t xchg_bytes_per_rank[4] = {0, 0, 0, 0};   // [0] end-of-frame history borders, [1] mid-frame GI bands (reflections on), [2] host-supplied inputs, [3] irradiance-cache requests
    kjb_ircache_bindings frame_cache{}; bool cache_share_pending = false;   // this frame's cache bindings (tile-sharded frames exchange the cache requests after the last user)
    void band(uint32_t r, uint32_t rows, uint32_t& b0, uint32_t& b1) const { b0 = uint32_t(uint64_t(rows) * r / tcount); b1 = uint32_t(uint64_t(rows) * (r + 1) / tcount); }
    // restrict the next pass to the owned band grown by `e` half-res rows; `scale` = 2 for full-res passes
    uint32_t cur_row0 = 0;   // first row of the scissor last set by rows()
    void rows(uint32_t e, uint32_t scale) {
        if (!tiled) return;
        const uint32_t a = ty0 > e ? ty0 - e : 0, b = ty1 + e;
        cur_row0 = a * scale;
        kjb_set_scissor(ctx, a * scale, b * scale);
    }
    void rows_all() { if (tiled) kjb_set_scissor(ctx, 0, 0); }
    void rows_span(int64_t a, int64_t b) { if (tiled) kjb_set_scissor(ctx, uint32_t(std::max<int64_t>(a, 0)), uint32_t(std::max<int64_t>(b, 1))); }   // rows [a, b) of the pass's grid
    // The row grids of a tile-sharded frame.  A band is half-res rows [b0, b1); its rows of a full-res image are [2·b0, 2·b1) clipped to H (odd
    // heights), and of the result image (RH rows: the TAA output, else the render-res result) the ONE ownership rule o(b) = ⌊RH·min(2b, H) / H⌋ at
    // each band boundary.  o(0) = 0, o(HH) = RH and o is monotone, so the ranks' result rows partition [0, RH) for any RH; without upsampling
    // o is the full-res rule.  kjb_world_result_rows reports them.
    enum Grid : uint32_t { GRID_HALF, GRID_FULL, GRID_OUT };
    uint32_t RH = 0;   // rows of the result image
    uint32_t grid_row(Grid g, uint32_t b) const {
        const uint32_t f = std::min(2 * b, H);
        return g == GRID_HALF ? b : g == GRID_FULL ? f : uint32_t(uint64_t(RH) * f / H);
    }
    void band_rows(Grid g, uint32_t r, uint32_t& y0, uint32_t& y1) const { uint32_t b0, b1; band(r, HH, b0, b1); y0 = grid_row(g, b0); y1 = grid_row(g, b1); }
    bool use_graph = true, graph_open = false;   // kjb_world_set_cuda_graph
    // Async compute (kjb_world_set_async_compute): the irradiance-cache chain of a frame (maintenance, cache rays, sum: ~10 small latency-bound launches)
    // runs on the async pass queue.  It needs nothing of this frame's screen-space inputs, only that the LAST frame's cache users are done, so it
    // executes under the reflection filters + TAA of the previous frame and under this frame's reprojection passes.
    bool use_async = true, async_ok = false, async_frame = false, cache_users_done_marked = false;   // async_ok: the two pass queues may run concurrently this frame
    bool profiling = false; uint32_t timer_next = 0;
    std::vector<std::pair<std::string, std::pair<uint32_t, uint32_t>>> timer_pending;   // label -> (slot_begin, slot_end) of this frame
    std::map<std::string, std::pair<uint32_t, double>> pass_ms;                          // label -> (calls, total ms)
    std::string timings_cache;
    void pass_begin(const char* label) {
        if (!profiling || timer_next + 2 > 1024) return;
        kjb_timer_record(ctx, timer_next);
        timer_pending.push_back({label, {timer_next, timer_next + 1}});
        timer_next += 2;
    }
    void pass_end() { if (profiling && !timer_pending.empty()) kjb_timer_record(ctx, timer_pending.back().second.second); }
    void flush_timers() {
        for (auto& t : timer_pending) {
            float ms = 0;
            if (kjb_timer_elapsed_ms(ctx, t.second.first, t.second.second, &ms) == 0) { auto& e = pass_ms[t.first]; e.first += 1; e.second += ms; }
        }
        timer_pending.clear(); timer_next = 0;
    }

    // rg.create / get_or_create_temporal: allocate once per name, zero-filled
    kjb_image& img(const std::string& name, uint32_t w, uint32_t h, uint32_t fmt, uint32_t layers = 1) {
        auto it = images.find(name);
        if (it != images.end()) return it->second;
        kjb_image i{};
        if (kjb_image_alloc(ctx, w, h, layers, fmt, &i)) err = 1;
        names_cache.clear();
        return images.emplace(name, i).first->second;
    }
    // temporal_storage_buffer (ircache.rs:80-90): buffers live in the same name table, viewed as 1024-wide images so that the
    // test harness can download and compare them like any other resource
    kjb_buffer buf(const std::string& name, uint64_t elems, uint32_t fmt, uint32_t elem_bytes) {
        const uint32_t wd = elems < 1024 ? uint32_t(elems) : 1024u, ht = uint32_t((elems + wd - 1) / wd);
        kjb_image& i = img(name, wd, ht, fmt);
        return kjb_buffer{i.data, uint64_t(wd) * ht * elem_bytes};
    }
    void get_output_and_history(PingPong& pp, uint32_t w, uint32_t h, uint32_t fmt, kjb_image*& out, kjb_image*& hist) {
        out = &img(pp.output_key, w, h, fmt);
        hist = &img(pp.history_key, w, h, fmt);
        std::swap(pp.output_key, pp.history_key);
    }
    // returns true if passes should keep running
    bool pass_done(const char* label, int rc) {
        if (rc) err = rc;
        stats[3]++;
        if (!stop_after.empty() && stop_after == label) stopped = true;
        return !stopped && !err;
    }
};

// tile mode: additionally run the pass on rows [0, top) when the main range starts below them (pixel (0,0) dependency)
#define RUN_TOP(label, call, top) do { if (w->tiled && !w->stopped && !w->err) { const uint32_t e__ = w->cur_row0; if (e__ > 0) { \
        kjb_set_scissor(w->ctx, 0, std::min<uint32_t>((top), e__)); int rc2__ = (call); if (rc2__) w->err = rc2__; } } } while (0)
#define RUN(label, call) do { if (w->stopped || w->err) break; w->pass_begin(label); int rc__ = (call); w->pass_end(); w->pass_done(label, rc__); } while (0)

static void size4(float out[4], const kjb_image& i) { out[0] = float(i.width); out[1] = float(i.height); out[2] = 1.0f / float(i.width); out[3] = 1.0f / float(i.height); }

extern "C" {

int kjb_world_create(kjb_context* ctx, const kjb_world_desc* desc, kjb_world** out) {
    if (!ctx || !desc || !out || desc->render_width == 0 || desc->render_height == 0) return 1;
    if (desc->tile_count > 1 && desc->tile_rank >= desc->tile_count) return 1;
    kjb_world* w = new kjb_world();
    w->ctx = ctx; w->desc = *desc;
    w->sun_size_multiplier = desc->hard_sun ? 0.0f : 1.0f;
    { const char* e = getenv("KJB_NO_GRAPH"); if (e && e[0] == '1') w->use_graph = false; }
    { const char* e = getenv("KJB_NO_ASYNC"); if (e && e[0] == '1') w->use_async = false; }
    kjb_set_option(ctx, KJB_OPTION_HALF_RES_POSITION_CACHE, 1);   // this driver only writes half_depth / the packed reservoirs through the passes the option tracks
    if (w->desc.spatial_reuse_pass_count == 0) w->desc.spatial_reuse_pass_count = 2;
    w->W = desc->render_width; w->H = desc->render_height;
    w->HW = (w->W + 1) / 2; w->HH = (w->H + 1) / 2;   // ImageDesc::half_res = div_up (image.rs:140-142)
    w->OW = desc->temporal_upscale_width ? desc->temporal_upscale_width : w->W; w->OH = desc->temporal_upscale_height ? desc->temporal_upscale_height : w->H;
    // Tiles + irradiance cache: every rank keeps its OWN replica of the cache, fed by the rays of its band and halos, and the replicas exchange
    // their requests after the frame's last cache user (ircache_share): exactly on the ordered schedule, so every replica stays the single-GPU
    // cache, statistically on the reference's atomics.  Tiles + lit composite: not yet.
    if (desc->tile_count > 1 && desc->enable_lighting) { delete w; return 1; }   // the lit composite (shadow denoiser history) does not shard yet
    w->RH = desc->enable_taa ? w->OH : w->H;
    if (desc->tile_count > 1) {
        w->tiled = true; w->trank = desc->tile_rank; w->tcount = desc->tile_count;
        w->band(w->trank, w->HH, w->ty0, w->ty1);
    }
    *out = w;
    return 0;
}
void kjb_world_destroy(kjb_world* w) {
    if (!w) return;
    kjb_sync(w->ctx);   // every queue: nothing of this world is in flight any more
    for (auto& kv : w->images) kjb_image_free(w->ctx, &kv.second);
    for (int k = 0; k < 4; ++k) { if (w->xchg_send[k].data) kjb_buffer_free(w->ctx, &w->xchg_send[k]); if (w->xchg_recv[k].data) kjb_buffer_free(w->ctx, &w->xchg_recv[k]); }
    delete w;
}

int kjb_world_add_mesh(kjb_world* w, const kjb_mesh_desc* mesh, uint32_t* out_handle) {
    // a malformed description is an error code, never an out-of-bounds access on the host or the device
    if (!w || !mesh || !mesh->positions || !mesh->normals || !mesh->indices || !mesh->material_ids || !mesh->materials) return 1;
    if (mesh->index_count % 3u != 0 || mesh->material_count == 0) return 1;
    for (uint32_t i = 0; i < mesh->index_count; ++i) if (mesh->indices[i] >= mesh->vertex_count) return 1;
    for (uint32_t i = 0; i < mesh->vertex_count; ++i) if (mesh->material_ids[i] >= mesh->material_count) return 1;
    if (mesh->map_count && !mesh->maps) return 1;
    for (uint32_t i = 0; i < mesh->map_count; ++i) if (!mesh->maps[i].texels || !mesh->maps[i].width || !mesh->maps[i].height || !mesh->maps[i].mip_count) return 1;
    // map ids index this mesh's own map list; a mesh without maps reads "no texture" (white) rather than whatever another mesh uploads later
    for (uint32_t i = 0; i < mesh->material_count; ++i) for (int k = 0; k < 4; ++k) if (mesh->map_count && mesh->materials[i].maps[k] >= mesh->map_count) return 1;
    const uint32_t mesh_idx = uint32_t(w->meshes.size());
    // bindless textures: one id per map of this mesh (add_mesh dedups identical assets; ids are per-upload here)
    const uint32_t tex_base = uint32_t(w->textures.size());
    for (uint32_t i = 0; i < mesh->map_count; ++i) {
        const kjb_texture_desc& t = mesh->maps[i];
        size_t bytes = 0; for (uint32_t m = 0; m < t.mip_count; ++m) bytes += size_t(std::max(1u, t.width >> m)) * std::max(1u, t.height >> m) * 4;
        w->texture_storage.emplace_back(t.texels, t.texels + bytes);
        kjb_texture_desc d = t; d.texels = nullptr; w->textures.push_back(d);
    }
    std::vector<kjb_mesh_material> materials(mesh->materials, mesh->materials + mesh->material_count);
    for (auto& mat : materials) {
        for (int k = 0; k < 4; ++k) mat.maps[k] = mesh->map_count ? tex_base + mat.maps[k] : 0xffffffffu;
        if (mesh->use_lights) mat.flags |= 1u;   // MESH_MATERIAL_FLAG_EMISSIVE_USED_AS_LIGHT (world_renderer.rs:649-654)
    }
    // BufferBuilder::append order (world_renderer.rs:657-672): indices, verts, uvs, material ids, colors, tangents, materials
    auto append = [&](const void* p, size_t bytes, size_t align) -> uint32_t {
        size_t off = (w->vertex_buffer.size() + align - 1) / align * align;
        w->vertex_buffer.resize(off + bytes);
        if (bytes) memcpy(&w->vertex_buffer[off], p, bytes);
        return uint32_t(off);
    };
    if (w->vertex_buffer.empty()) w->vertex_buffer.resize(16);   // keep offset 0 unused so `vertex_aux_offset != 0` stays meaningful
    kjb_gpu_mesh gm{};
    gm.index_offset = append(mesh->indices, size_t(mesh->index_count) * 4, 16);
    std::vector<float> verts(size_t(mesh->vertex_count) * 4);
    for (uint32_t i = 0; i < mesh->vertex_count; ++i) {
        verts[i * 4 + 0] = mesh->positions[i * 3 + 0]; verts[i * 4 + 1] = mesh->positions[i * 3 + 1]; verts[i * 4 + 2] = mesh->positions[i * 3 + 2];
        uint32_t pn = pack_unit_direction_11_10_11(mesh->normals[i * 3 + 0], mesh->normals[i * 3 + 1], mesh->normals[i * 3 + 2]);
        memcpy(&verts[i * 4 + 3], &pn, 4);
    }
    gm.vertex_core_offset = append(verts.data(), verts.size() * 4, 16);
    std::vector<float> uvs(size_t(mesh->vertex_count) * 2, 0.0f);
    if (mesh->uvs) memcpy(uvs.data(), mesh->uvs, uvs.size() * 4);
    gm.vertex_uv_offset = append(uvs.data(), uvs.size() * 4, 16);
    gm.vertex_mat_offset = append(mesh->material_ids, size_t(mesh->vertex_count) * 4, 16);
    std::vector<float> colors(size_t(mesh->vertex_count) * 4, 1.0f);
    if (mesh->colors) memcpy(colors.data(), mesh->colors, colors.size() * 4);
    gm.vertex_aux_offset = append(colors.data(), colors.size() * 4, 16);
    gm.vertex_tangent_offset = 0;   // tangents only feed the (disabled, `#if 0`) normal-map branch of gbuffer.rchit.hlsl:117-158
    gm.mat_data_offset = append(materials.data(), materials.size() * sizeof(kjb_mesh_material), 16);
    w->meshes.push_back(gm);
    w->mesh_index_counts.push_back(mesh->index_count);

    // triangle-light extraction (world_renderer.rs:741-769)
    std::vector<kjb_triangle_light> lights;
    if (mesh->use_lights) {
        for (uint32_t t = 0; t + 2 < mesh->index_count; t += 3) {
            const uint32_t i0 = mesh->indices[t], i1 = mesh->indices[t + 1], i2 = mesh->indices[t + 2];
            const kjb_mesh_material& mat = mesh->materials[mesh->material_ids[i0]];
            if (!(mat.emissive[0] > 0 || mat.emissive[1] > 0 || mat.emissive[2] > 0)) continue;
            kjb_triangle_light l{};
            const uint32_t ids[3] = {i0, i1, i2};
            for (int k = 0; k < 3; ++k) for (int c = 0; c < 3; ++c) l.verts[k][c] = mesh->positions[ids[k] * 3 + c];
            for (int c = 0; c < 3; ++c) l.radiance[c] = mat.emissive[c];
            lights.push_back(l);
        }
    }
    w->mesh_lights.push_back(lights);
    w->geometry_dirty = true;
    if (out_handle) *out_handle = mesh_idx;
    return 0;
}

int kjb_world_add_instance(kjb_world* w, uint32_t mesh, const float transform[12], uint32_t* out_handle) {
    if (mesh >= w->meshes.size()) return 1;
    kjb_instance i{}; memcpy(i.transform, transform, sizeof(i.transform)); i.mesh_index = mesh; i.emissive_multiplier = 1.0f;
    const uint32_t handle = w->next_instance_handle++;
    w->instance_handle_to_index[handle] = uint32_t(w->instances.size());
    w->instances.push_back(i); w->instance_handles.push_back(handle);
    w->prev_instances.push_back(i);   // a new instance starts with prev_transform = transform (world_renderer.rs:785-797)
    if (out_handle) *out_handle = handle;
    return 0;
}

// WorldRenderer::remove_instance (world_renderer.rs:800-813): swap_remove, so the last instance takes the freed slot (and its InstanceID)
int kjb_world_remove_instance(kjb_world* w, uint32_t handle) {
    auto it = w->instance_handle_to_index.find(handle);
    if (it == w->instance_handle_to_index.end()) return 1;   // upstream: expect("no such instance")
    const uint32_t index = it->second;
    w->instance_handle_to_index.erase(it);
    w->instances[index] = w->instances.back(); w->instances.pop_back();
    w->prev_instances[index] = w->prev_instances.back(); w->prev_instances.pop_back();   // prev_transform lives in the MeshInstance upstream: it moves with the swap_remove
    w->instance_handles[index] = w->instance_handles.back(); w->instance_handles.pop_back();
    if (index < w->instance_handles.size()) w->instance_handle_to_index[w->instance_handles[index]] = index;
    return 0;
}

int kjb_world_set_instance_transform(kjb_world* w, uint32_t handle, const float transform[12]) {
    auto it = w->instance_handle_to_index.find(handle);
    if (it == w->instance_handle_to_index.end()) return 1;
    memcpy(w->instances[it->second].transform, transform, sizeof(float) * 12);
    return 0;
}

// get_instance_dynamic_parameters_mut(inst).emissive_multiplier (world_renderer.rs:828-834, InstanceDynamicParameters :96-105)
int kjb_world_set_instance_emissive_multiplier(kjb_world* w, uint32_t handle, float emissive_multiplier) {
    auto it = w->instance_handle_to_index.find(handle);
    if (it == w->instance_handle_to_index.end()) return 1;
    w->instances[it->second].emissive_multiplier = emissive_multiplier;
    return 0;
}

int kjb_world_set_sun_color_multiplier(kjb_world* w, const float rgb[3]) { memcpy(w->sun_color_multiplier, rgb, 12); w->sky_valid = false; return 0; }   // the sky cube bakes it in
int kjb_world_set_sky_ambient(kjb_world* w, const float rgb[3]) { memcpy(w->sky_ambient, rgb, 12); w->sky_valid = false; return 0; }
int kjb_world_set_render_overrides(kjb_world* w, uint32_t flags, float material_roughness_scale) {
    if (flags & ~15u) return 1;
    w->render_override_flags = flags; w->render_override_material_roughness_scale = material_roughness_scale; return 0;
}
int kjb_world_reset_reference_accumulation(kjb_world* w) { w->reset_reference_accumulation = true; return 0; }
int kjb_world_set_debug_shading_mode(kjb_world* w, uint32_t mode) { if (mode == 1 || mode > 4) return 1; w->debug_shading_mode = mode; return 0; }
int kjb_world_set_sun_size_multiplier(kjb_world* w, float m) { if (!(m >= 0.0f)) return 1; w->sun_size_multiplier = m; return 0; }

int kjb_world_set_blue_noise(kjb_world* w, const uint8_t* rgba) {
    kjb_image& bn = w->img("lut.blue_noise", 256, 256, KJB_FMT_RGBA8_UNORM);
    int rc = kjb_image_upload(w->ctx, &bn, rgba);
    w->noise_ready = true;
    return rc | w->err;
}

uint32_t kjb_world_frame_index(kjb_world* w) { return w->frame_idx; }
int kjb_world_result_rows(kjb_world* w, uint32_t* y0, uint32_t* y1) {
    if (!w || !y0 || !y1) return 1;
    if (w->tiled) w->band_rows(kjb_world::GRID_OUT, w->trank, *y0, *y1);
    else { *y0 = 0; *y1 = w->RH; }
    return 0;
}
int kjb_world_set_spatial_resolve_offsets(kjb_world* w, const int32_t* t) {
    if (!t) return 1;
    w->spatial_resolve_offsets.assign(t, t + 4 * KJB_SPATIAL_RESOLVE_OFFSET_COUNT);
    return 0;
}
int kjb_world_get_image(kjb_world* w, const char* name, kjb_image* out) {
    auto it = w->images.find(name); if (it == w->images.end()) return 1; *out = it->second;
    // a caller that is about to read the image on the compute queue must see a finished border exchange (event slot 17 = EV_XCHG_DONE)
    if (w->exchange_pending) kjb_queue_wait_event(w->ctx, KJB_QUEUE_COMPUTE, 17);
    return 0;
}
const char* kjb_world_image_names(kjb_world* w) {
    if (w->names_cache.empty()) for (auto& kv : w->images) { w->names_cache += kv.first; w->names_cache += '\n'; }
    return w->names_cache.c_str();
}
// launches/passes of the last frame; rays traced since the previous call (reading the counters synchronises, so it is not done per frame)
int kjb_world_last_frame_stats(kjb_world* w, uint64_t out[4]) {
    uint64_t rays[2] = {0, 0};
    kjb_ray_counters(w->ctx, rays, 1);
    w->stats[1] = rays[0]; w->stats[2] = rays[1];
    memcpy(out, w->stats, sizeof(w->stats)); return 0;
}
int kjb_world_set_stop_after(kjb_world* w, const char* label) { w->stop_after = label ? label : ""; return 0; }
int kjb_world_set_cuda_graph(kjb_world* w, uint32_t on) { w->use_graph = on != 0; return 0; }
int kjb_world_set_async_compute(kjb_world* w, uint32_t on) { w->use_async = on != 0; return 0; }
int kjb_world_set_profiling(kjb_world* w, uint32_t on) { w->flush_timers(); w->profiling = on != 0; if (on) w->pass_ms.clear(); return 0; }
const char* kjb_world_pass_timings(kjb_world* w) {
    w->flush_timers();
    w->timings_cache.clear();
    for (auto& kv : w->pass_ms) w->timings_cache += kv.first + "\t" + std::to_string(kv.second.first) + "\t" + std::to_string(kv.second.second) + "\n";
    return w->timings_cache.c_str();
}

// ---------------------------------------------------------------- per-frame constants (world_renderer.rs:1001-1108)
static int begin_frame(kjb_world* w, const kjb_world_frame* f, kjb_frame_constants& fc, bool jitter) {
    kjb_context* ctx = w->ctx;
    w->stopped = false; w->stats[3] = 0; w->exchanged_this_frame = false;
    w->launches_at_frame_start = kjb_launch_count(ctx);
    if (w->geometry_dirty) {
        for (size_t i = 0; i < w->textures.size(); ++i) w->textures[i].texels = w->texture_storage[i].data();
        if (kjb_scene_set_geometry(ctx, w->vertex_buffer.data(), w->vertex_buffer.size(), w->meshes.data(), w->mesh_index_counts.data(), uint32_t(w->meshes.size()))) return 1;
        if (kjb_scene_set_textures(ctx, w->textures.data(), uint32_t(w->textures.size()))) return 1;
        w->geometry_dirty = false;
    }
    // "rebuild tlas" every frame (world_render_passes.rs:19); the library skips the rebuild when nothing moved
    if (kjb_rebuild_tlas(ctx, w->instances.data(), uint32_t(w->instances.size()))) return 1;

    const CameraMatrices cam = camera_matrices(*f, float(w->W) / float(w->H));
    const CameraMatrices prev = w->have_prev_camera ? w->prev_camera : cam;
    memset(&fc, 0, sizeof(fc));
    kjb_view_constants& vc = fc.view_constants;
    m4_store(vc.view_to_clip, cam.view_to_clip); m4_store(vc.clip_to_view, cam.clip_to_view);
    m4_store(vc.world_to_view, cam.world_to_view); m4_store(vc.view_to_world, cam.view_to_world);
    m4_store(vc.clip_to_prev_clip, m4_mul(m4_mul(m4_mul(prev.view_to_clip, prev.world_to_view), cam.view_to_world), cam.clip_to_view));
    m4_store(vc.prev_view_to_prev_clip, prev.view_to_clip); m4_store(vc.prev_clip_to_prev_view, prev.clip_to_view);
    m4_store(vc.prev_world_to_prev_view, prev.world_to_view); m4_store(vc.prev_view_to_prev_world, prev.view_to_world);
    // TAA jitter: Halton(2,3) - 0.5 over 128 frames (world_renderer.rs:425-428, :979-981); none for the reference path tracer (:989)
    float off[2] = {0, 0};
    if (jitter) { const uint32_t i = (w->frame_idx % 128u) + 1u; off[0] = radical_inverse(i, 2) - 0.5f; off[1] = radical_inverse(i, 3) - 0.5f; }
    vc.sample_offset_pixels[0] = off[0]; vc.sample_offset_pixels[1] = off[1];
    vc.sample_offset_clip[0] = (2.0f * off[0]) / float(w->W); vc.sample_offset_clip[1] = (2.0f * off[1]) / float(w->H);
    M4 jm = m4_identity(); jm.m[12] = -vc.sample_offset_clip[0]; jm.m[13] = -vc.sample_offset_clip[1];
    M4 jmi = m4_identity(); jmi.m[12] = vc.sample_offset_clip[0]; jmi.m[13] = vc.sample_offset_clip[1];
    m4_store(vc.view_to_sample, m4_mul(jm, cam.view_to_clip));
    m4_store(vc.sample_to_view, m4_mul(cam.clip_to_view, jmi));

    float sl = std::sqrt(f->sun_direction[0] * f->sun_direction[0] + f->sun_direction[1] * f->sun_direction[1] + f->sun_direction[2] * f->sun_direction[2]);
    for (int c = 0; c < 3; ++c) fc.sun_direction[c] = f->sun_direction[c] / sl;
    fc.frame_index = w->frame_idx;
    fc.delta_time_seconds = f->delta_time_seconds > 0 ? f->delta_time_seconds : 1.0f / 60.0f;
    // WorldRenderer::sun_size_multiplier (world_renderer.rs:207,508,1078): 1.0 = the sun as seen from Earth; hard_sun = 0
    fc.sun_angular_radius_cos = std::cos(w->sun_size_multiplier * ((0.53f * 3.14159265358979323846f / 180.0f) * 0.5f));
    for (int c = 0; c < 3; ++c) { fc.sun_color_multiplier[c] = w->sun_color_multiplier[c]; fc.sky_ambient[c] = w->sky_ambient[c]; }
    fc.pre_exposure = fc.pre_exposure_prev = fc.pre_exposure_delta = 1.0f;   // dynamic exposure lives in post (out of scope): EV 0
    fc.render_override_flags = w->render_override_flags; fc.render_override_material_roughness_scale = w->render_override_material_roughness_scale;

    if (w->desc.enable_ircache) {
        // IrcacheRenderer::update_eye_position + constants (ircache.rs:125-157, world_renderer.rs:1060-1092)
        const float IRCACHE_GRID_CELL_DIAMETER = 0.16f * 0.125f;
        for (int c = 0; c < 3; ++c) { w->ircache_grid_center[c] = f->camera_position[c]; fc.ircache_grid_center[c] = f->camera_position[c]; }
        fc.ircache_grid_center[3] = 1.0f;
        for (int cascade = 0; cascade < 12; ++cascade) {
            const float cell_diameter = IRCACHE_GRID_CELL_DIAMETER * float(1u << cascade);
            for (int c = 0; c < 3; ++c) {
                const int32_t cascade_center = int32_t(std::floor(f->camera_position[c] / cell_diameter));
                w->ircache_prev_scroll[cascade][c] = w->ircache_cur_scroll[cascade][c];
                w->ircache_cur_scroll[cascade][c] = cascade_center - 16;
                fc.ircache_cascades[cascade].origin[c] = w->ircache_cur_scroll[cascade][c];
                fc.ircache_cascades[cascade].voxels_scrolled_this_frame[c] = w->ircache_cur_scroll[cascade][c] - w->ircache_prev_scroll[cascade][c];
            }
        }
    }

    // triangle lights: instance-transformed copies of each mesh's light set (world_renderer.rs:1036-1056)
    std::vector<kjb_triangle_light> lights;
    for (const kjb_instance& inst : w->instances) for (kjb_triangle_light l : w->mesh_lights[inst.mesh_index]) {
        // to_scale_rotation_translation(): rotation = normalised columns, translation = last column; the scale is DROPPED (as upstream)
        float rot[9];
        for (int c = 0; c < 3; ++c) {
            float cx = inst.transform[0 * 4 + c], cy = inst.transform[1 * 4 + c], cz = inst.transform[2 * 4 + c];
            float len = std::sqrt(cx * cx + cy * cy + cz * cz); if (len == 0) len = 1;
            rot[0 * 3 + c] = cx / len; rot[1 * 3 + c] = cy / len; rot[2 * 3 + c] = cz / len;
        }
        for (int k = 0; k < 3; ++k) {
            float v[3] = {l.verts[k][0], l.verts[k][1], l.verts[k][2]};
            for (int r = 0; r < 3; ++r) l.verts[k][r] = rot[r * 3 + 0] * v[0] + rot[r * 3 + 1] * v[1] + rot[r * 3 + 2] * v[2] + inst.transform[r * 4 + 3];
        }
        for (int c = 0; c < 3; ++c) l.radiance[c] *= inst.emissive_multiplier;
        lights.push_back(l);
    }
    fc.triangle_light_count = uint32_t(lights.size());
    w->frame_light_count = fc.triangle_light_count;
    if (kjb_set_frame_constants(ctx, &fc, lights.data(), fc.triangle_light_count)) return 1;
    w->prev_camera = cam; w->have_prev_camera = true;

    // bindless LUTs (default_world_renderer.rs:22-51): BRDF FG LUT computed once, blue noise supplied by the caller
    kjb_image& fg = w->img("lut.brdf_fg", 64, 64, KJB_FMT_RGBA16_FLOAT);
    kjb_image& bn = w->img("lut.blue_noise", 256, 256, KJB_FMT_RGBA8_UNORM);
    if (!w->lut_ready) {
        kjb_brdf_fg_lut_args la{}; la.output_tex = fg;
        if (kjb_pass_brdf_fg_lut(ctx, &la)) return 1;
        w->lut_ready = true;
    }
    if (kjb_set_luts(ctx, &fg, &bn)) return 1;
    return w->err;
}

static void end_frame(kjb_world* w) {
    w->stats[0] = kjb_launch_count(w->ctx) - w->launches_at_frame_start;
    if (w->profiling) w->flush_timers();
    w->prev_instances = w->instances;
    w->frame_idx += 1;   // retire_frame (world_renderer.rs:1110-1113)
}


// ---------------------------------------------------------------- tile sharding: halos and the per-frame border exchange
// Half-res rows a pass must compute beyond the owned band so that every later pass of the SAME frame finds valid inputs
// (derived from the shaders' stencils: restir_spatial.hlsl:89-92 radii 32/16/8, payload indirection `spx`, resolve ~3,
// temporal filter 5x5, spatial filter <=16 px, taa 3x3..5x5).  History older than this frame comes from the exchange.
// Reflections (rtr.rs): the spatial cleanup reaches SPATIAL_RESOLVE_OFFSETS (|offset| <= 12, x2 at low sample counts) = 12 half-res rows, its
// temporal filter 3x3, the resolve's world-space footprint is clamped to 0.1 of the screen height (resolve.hlsl:201-207) = H/40 half-res
// rows (+ 8 % for the outermost tap + 2), the reservoir history is searched within 14 half-res px of the reprojected pixel
// (rtr_restir_temporal.hlsl rpx_offset_radius) and validated in 2x2 quads.
//
// TAA (taa.rs) runs on two row grids.  "reproject taa" and "taa" write the output grid (OW x OH); "taa filter input / history", "taa input prob" and
// "taa prob filter / filter2" the input grid (the render extent).  A band owns the output rows o(b0)..o(b1) (kjb_world::grid_row), and the input-grid
// passes run on the input rows under them, [i0, i1): output row y reads input row ry = ⌊(y + 0.5)·IH/OH⌋ as the unjittered 3x3's centre
// (unjitter_taa.hlsl:68, k_taa_tiled*: sample_image_unjitter_taa2), for its input probability and its reprojection texel (taa.hlsl:109,
// reproject_history.hlsl:45).  The host evaluates the kernels' float expression, so [i0, i1) is exact; with a ratio of 1 it is the full-res band.
// Halos on the input grid, consumer first (kjb_passes_taa.cu):
//   taa prob filter2  0   taa reads the probability at ry only;
//   taa prob filter   5   filter2 reads a 5x5 at stride 2 (:265-266) = ±4, + 1;
//   taa input prob    6   filter reads 3x3 (:247);
//   taa filter history 8  input prob reads the filtered history at the nearest texel of the jittered uv (:224) = ±1, + 1;
//   taa filter input 10   input prob reads the input deviation 3x3 at stride 2 (:220) = ±2;
//   the GI result (TAA's input) 11 = filter input's 3x3 (:120); the unjitter's 3x3 (:284) is inside.  tile_halos' `x` = 6 half-res rows holds it,
//   plus g = how far [i0, i1) reaches past the band's full-res rows (at most one row when upsampling), rounded up to half-res rows.
// "reproject taa" on the output grid: "taa filter history" at input row y reads output rows ⌊(y + 0.5)/IH·OH + 1e-3⌋ ± k (:150-151, k ≤ 2), and
// taa its 5x5 blurred history (:322-325) inside that range.  So reproject runs on the rows the filter reads from input rows [i0 - 8, i1 + 8),
// grown by 4: k plus two rows for the truncations of the float mapping (12 output rows at a ratio of 1, as without upsampling).
// The TAA histories (output grid) are read next frame by reproject's Catmull-Rom fetch (:62-77: rows texPos1 - 1 .. texPos1 + 2 through bilinear
// taps = ±3) and by input prob / taa bilinearly (±1) at the reprojected uv: the exchanged border is reproject's halo + 3 + the motion bound, one
// render row per frame = ⌈OH/H⌉ output rows (16 rows at a ratio of 1).
struct TaaRows { int64_t o0, o1, i0, i1, rep0, rep1; };
static TaaRows taa_rows(const kjb_world* w, uint32_t r) {
    TaaRows t{};
    uint32_t o0, o1; w->band_rows(kjb_world::GRID_OUT, r, o0, o1);
    const float irs = float(w->H) / float(w->RH), inv_ih = 1.0f / float(w->H), oh = float(w->RH);
    auto in_row = [&](int64_t y) { return int64_t(uint32_t((float(y) + 0.5f) * irs)); };                       // k_taa_tiled*, k_taa_reproject: rx, ry
    auto out_row = [&](int64_t y) { return int64_t(std::floor((float(y) + 0.5f) * inv_ih * oh + 1e-3f)); };   // t3_filter: sy
    t.o0 = o0; t.o1 = o1;
    t.i0 = in_row(o0); t.i1 = o1 > o0 ? in_row(o1 - 1) + 1 : t.i0;
    t.rep0 = out_row(t.i0 - 8) - 4; t.rep1 = out_row(t.i1 + 7) + 5;
    return t;
}
// the same for every rank (the exchange layout depends on it): the largest of the bands'
static void taa_reach(const kjb_world* w, uint32_t& g, uint32_t& border) {
    uint32_t e = 0; g = 0;
    for (uint32_t r = 0; r < w->tcount; ++r) {
        const TaaRows t = taa_rows(w, r);
        uint32_t f0, f1; w->band_rows(kjb_world::GRID_FULL, r, f0, f1);
        g = uint32_t(std::max<int64_t>({int64_t(g), int64_t(f0) - t.i0, t.i1 - int64_t(f1)}));
        e = uint32_t(std::max<int64_t>({int64_t(e), t.o0 - t.rep0, t.rep1 - t.o1}));
    }
    border = e + 3 + (w->RH + w->H - 1) / w->H;
}
struct TileHalos { uint32_t d11, d10, d9, spatial_last, d6, d5, d4, halo, border; uint32_t r_cleanup, r_temporal, r_resolve, r_rt, r_validate, r_border; uint32_t taa_border; };
static TileHalos tile_halos(const kjb_world* w) {
    TileHalos h{};
    uint32_t g = 0;
    if (w->tiled && w->desc.enable_taa) taa_reach(w, g, h.taa_border);
    const uint32_t x = w->desc.enable_taa ? 6u + (g + 1) / 2 : 0u;
    h.r_cleanup = x; h.r_temporal = x + 13; h.r_resolve = h.r_temporal + 1; h.r_rt = h.r_resolve + w->H / 36 + 4; h.r_validate = h.r_rt + 18; h.r_border = h.r_validate + 4;
    uint32_t sum_r = 0;
    for (uint32_t i = 0; i < w->desc.spatial_reuse_pass_count; ++i) sum_r += i == 0 ? 32u : (i == 1 ? 16u : 8u);
    h.d11 = x; h.d10 = x + 8; h.d9 = x + 9; h.spatial_last = x + 12;
    h.d6 = x + 12 + sum_r; h.d5 = h.d6; h.d4 = h.d6 + 4; h.halo = h.d6 + 8; h.border = h.halo + 4;
    if (w->desc.enable_rtr) h.d4 = std::max(h.d4, h.r_rt + 2);   // the diffuse candidates double as reflection candidates (rtr.rs:105-109)
    return h;
}
static uint32_t spatial_radius(uint32_t pass_idx) { return pass_idx == 0 ? 32u : (pass_idx == 1 ? 16u : 8u); }

static const uint32_t TILE_TOP_ROWS = 16;   // half-res rows at the top of the image kept valid on every rank (pixel (0,0) dependency)

struct XchgItem { kjb_image img; kjb_world::Grid grid; uint32_t border; };   // `grid`: which rows of the image a band owns; border in image rows, 0 = whole band

// ONE all-gather per frame: every rank contributes the top and bottom `border` rows of its band of each temporal image (its
// whole band for the full-res GI history, which the next frame's rays sample at arbitrary screen positions), and copies the
// strips it needs from the other ranks' contributions into its own images.  Row strips of row-major images are contiguous.
static int tile_exchange(kjb_world* w, const std::vector<XchgItem>& items_in, uint32_t queue, int set = 0) {
    kjb_context* ctx = w->ctx;
    const uint32_t n = w->tcount;
    // the fewest and the most rows a band owns of each item's image
    std::vector<uint32_t> rows_min(items_in.size(), 0xffffffffu), rows_max(items_in.size(), 0);
    for (size_t i = 0; i < items_in.size(); ++i) for (uint32_t r = 0; r < n; ++r) {
        uint32_t y0, y1; w->band_rows(items_in[i].grid, r, y0, y1);
        rows_min[i] = std::min(rows_min[i], y1 - y0); rows_max[i] = std::max(rows_max[i], y1 - y0);
    }
    // One whole-band image and equal bands (this frame's GI for the reflection rays at 2 / 4 GPUs): the image IS the concatenation of the ranks' bands, so the
    // all-gather runs in place on it — no staging buffers, no pack / unpack launches.
    if (items_in.size() == 1 && items_in[0].border == 0 && rows_max[0] == rows_min[0] && n > 1) {
        const kjb_image& img = items_in[0].img;
        const uint64_t band_bytes = uint64_t(img.width) * kjb_format_texel_bytes(img.format) * rows_max[0];
        if (band_bytes * n == uint64_t(img.width) * kjb_format_texel_bytes(img.format) * img.height)
            return kjb_allgather_on(ctx, queue, (const char*)img.data + band_bytes * w->trank, img.data, band_bytes);
    }
    // narrow bands (many ranks): when the two border strips of a band touch or overlap, send the band once instead of twice
    std::vector<XchgItem> items = items_in;
    for (size_t i = 0; i < items.size(); ++i) if (items[i].border && 2 * items[i].border >= rows_min[i]) items[i].border = 0;
    // layout of one rank's contribution
    std::vector<uint64_t> off(items.size()), strip_bytes(items.size());
    uint64_t total = 0;
    for (size_t i = 0; i < items.size(); ++i) {
        const uint64_t row_bytes = uint64_t(items[i].img.width) * kjb_format_texel_bytes(items[i].img.format);
        const uint32_t rows = items[i].border ? std::min(items[i].border, rows_max[i]) : rows_max[i];
        strip_bytes[i] = row_bytes * rows;
        off[i] = total; total += strip_bytes[i] * (items[i].border ? 2 : 1);
    }
    total = (total + 255) / 256 * 256;
    if (w->xchg_bytes_per_rank[set] != total) {
        if (w->xchg_send[set].data) { kjb_sync(ctx); kjb_buffer_free(ctx, &w->xchg_send[set]); kjb_buffer_free(ctx, &w->xchg_recv[set]); }
        if (kjb_buffer_alloc(ctx, total, &w->xchg_send[set]) || kjb_buffer_alloc(ctx, total * n, &w->xchg_recv[set])) return 1;
        w->xchg_bytes_per_rank[set] = total;
    }
    auto strips_of = [&](uint32_t r, const XchgItem& it, uint32_t out[2][2]) {   // [strip][row0,row1) in image rows
        uint32_t b0, b1; w->band_rows(it.grid, r, b0, b1);
        if (!it.border) { out[0][0] = b0; out[0][1] = b1; out[1][0] = out[1][1] = 0; return; }
        const uint32_t k = std::min(it.border, b1 - b0);
        out[0][0] = b0; out[0][1] = b0 + k; out[1][0] = b1 - k; out[1][1] = b1;
    };
    // pack (one batched launch)
    std::vector<kjb_copy_desc> copies;
    for (size_t i = 0; i < items.size(); ++i) {
        const uint64_t row_bytes = uint64_t(items[i].img.width) * kjb_format_texel_bytes(items[i].img.format);
        uint32_t st[2][2]; strips_of(w->trank, items[i], st);
        for (int k = 0; k < (items[i].border ? 2 : 1); ++k)
            copies.push_back({(char*)w->xchg_send[set].data + off[i] + strip_bytes[i] * k, (const char*)items[i].img.data + row_bytes * st[k][0], row_bytes * (st[k][1] - st[k][0])});
    }
    if (kjb_memcpy_d2d_batch_on(ctx, queue, copies.data(), uint32_t(copies.size()))) return 1;
    copies.clear();
    if (kjb_allgather_on(ctx, queue, w->xchg_send[set].data, w->xchg_recv[set].data, total)) return 1;
    // unpack what this rank reads next frame: its band grown by `border` rows (everything for whole-band items)
    for (uint32_t r = 0; r < n; ++r) {
        if (r == w->trank) continue;
        const char* base = (const char*)w->xchg_recv[set].data + total * r;
        for (size_t i = 0; i < items.size(); ++i) {
            const uint64_t row_bytes = uint64_t(items[i].img.width) * kjb_format_texel_bytes(items[i].img.format);
            uint32_t mine[2][2]; strips_of(w->trank, items[i], mine);
            const uint32_t my0 = mine[0][0], my1 = items[i].border ? mine[1][1] : mine[0][1];
            const uint32_t need0 = items[i].border ? (my0 > items[i].border ? my0 - items[i].border : 0) : 0;
            const uint32_t need1 = items[i].border ? my1 + items[i].border : 0xffffffffu;
            uint32_t st[2][2]; strips_of(r, items[i], st);
            // Reservoirs that never selected a sample keep payload 0 == pixel (0,0) (reservoir.hlsl:18-24), so restir_temporal /
            // restir_spatial / restir_resolve dereference the state of pixel (0,0) from anywhere on screen: the first rows of the
            // image are a global dependency and travel to every rank.
            const uint32_t top = items[i].border ? w->grid_row(items[i].grid, TILE_TOP_ROWS) : 0;
            const uint32_t iv[2][2] = {{need0, need1}, {0, need0 > top ? top : 0}};
            for (int k = 0; k < (items[i].border ? 2 : 1); ++k) for (int v = 0; v < 2; ++v) {
                uint32_t a = std::max(st[k][0], iv[v][0]), b = std::min(st[k][1], iv[v][1]);
                if (k == 1 && items[i].border) a = std::max(a, st[0][1]);   // rows already delivered by the top strip (band <= 2*border)
                if (a >= b) continue;
                copies.push_back({(char*)items[i].img.data + row_bytes * a, base + off[i] + strip_bytes[i] * k + row_bytes * (a - st[k][0]), row_bytes * (b - a)});
            }
        }
    }
    return kjb_memcpy_d2d_batch_on(ctx, queue, copies.data(), uint32_t(copies.size()));   // unpack (one batched launch per 96 strips)
}

// The frame's single collective: borders of every temporal image (what is history next frame) + this rank's band of the GI history.
// It runs on the COMM queue, fenced by two events, so that it overlaps whatever does not depend on it: the spatial filter of this
// frame when it is issued right after "rtdgi temporal" (no TAA), and the front of the next frame (reprojection map, extracts) up to
// "rtdgi reproject", the first consumer of exchanged history.  With per-pass profiling on it stays on the compute queue so that the
// timers see it.
static const uint32_t EV_XCHG_BEGIN = 16, EV_XCHG_DONE = 17;
static void tile_exchange_frame(kjb_world* w) {
    if (!w->tiled || w->err || w->stopped) return;
    kjb_context* ctx = w->ctx;
    const TileHalos th2 = tile_halos(w);
    std::vector<XchgItem> items;
    auto add = [&](const PingPong& pp, kjb_world::Grid grid, uint32_t border) { auto it = w->images.find(pp.history_key); if (it != w->images.end()) items.push_back({it->second, grid, border}); };
    const kjb_world::Grid HALF = kjb_world::GRID_HALF, FULL = kjb_world::GRID_FULL;
    add(w->temporal2_tex, FULL, 0);
    add(w->temporal2_variance_tex, FULL, 2 * (th2.d10 + 2));
    add(w->temporal_radiance_tex, HALF, th2.border); add(w->temporal_ray_orig_tex, HALF, th2.border); add(w->temporal_ray_tex, HALF, th2.border);
    add(w->temporal_reservoir_tex, HALF, th2.border); add(w->temporal_candidate_tex, HALF, th2.border); add(w->temporal_invalidity_tex, HALF, th2.border);
    add(w->temporal_hit_normal_tex, HALF, th2.border);
    if (w->desc.enable_taa) {   // output-grid histories (taa.rs:19-27)
        add(w->taa_temporal_tex, kjb_world::GRID_OUT, th2.taa_border); add(w->taa_temporal_velocity_tex, kjb_world::GRID_OUT, th2.taa_border);
        add(w->taa_temporal_smooth_var_tex, kjb_world::GRID_OUT, th2.taa_border);
    }
    if (w->desc.enable_rtr) {   // what RtrRenderer reads as history next frame
        add(w->rtr_temporal_irradiance_tex, HALF, th2.r_border); add(w->rtr_temporal_ray_orig_tex, HALF, th2.r_border); add(w->rtr_temporal_ray_tex, HALF, th2.r_border);
        add(w->rtr_temporal_reservoir_tex, HALF, th2.r_border); add(w->rtr_temporal_rng_tex, HALF, th2.r_border); add(w->rtr_temporal_hit_normal_tex, HALF, th2.r_border);
        add(w->rtr_temporal_tex, FULL, 2 * (th2.r_resolve + 4)); add(w->rtr_ray_len_tex, FULL, 2 * (th2.r_resolve + 4));
    }
    const uint32_t queue = w->profiling ? KJB_QUEUE_COMPUTE : KJB_QUEUE_COMM;
    w->pass_begin("tile border all-gather");
    int rc = 0;
    if (queue != KJB_QUEUE_COMPUTE) rc |= kjb_event_record(ctx, EV_XCHG_BEGIN, KJB_QUEUE_COMPUTE) | kjb_queue_wait_event(ctx, queue, EV_XCHG_BEGIN);
    rc |= tile_exchange(w, items, queue);
    if (queue != KJB_QUEUE_COMPUTE) { rc |= kjb_event_record(ctx, EV_XCHG_DONE, queue); w->exchange_pending = true; }
    if (rc) w->err = 1;
    w->pass_end();
    w->rows_all();
    w->exchanged_this_frame = true;
}

// Event slots of the async irradiance-cache chain; graph instances: 0..2 = the three recordings of an async frame, 3 = a whole frame.
static const uint32_t EV_CACHE_USERS_DONE = 18, EV_CACHE_READY = 19, EV_FORK = 20, EV_JOIN = 21;
static void graph_open_slot(kjb_world* w, uint32_t slot) {
    if (w->use_graph && !w->profiling && !w->tiled && w->frame_idx >= 4 && w->stop_after.empty() && !w->err && kjb_graph_select(w->ctx, slot) == 0 && kjb_graph_begin(w->ctx) == 0) w->graph_open = true;
}
static void graph_close(kjb_world* w) { if (w->graph_open) { w->graph_open = false; if (kjb_graph_end(w->ctx)) w->err = 1; } }
// Tile-sharded frames: the replicas of the irradiance cache exchange what this frame's rays asked of them (kjb.h), in one all-gather.  On the ordered
// schedule the exchange is exact (kjb_pass_ircache_export_pending: every replica stays the single-GPU cache, bit for bit); on the reference's atomics it is
// statistical (kjb_pass_ircache_export_requests: one small record per live entry, one merge launch per other rank).  With async compute it runs on the async
// queue — right in front of the next frame's cache chain, under the reflection filters and TAA of this frame.
// The CPU oracle links this driver too but renders no tile-sharded frames and has no ordered schedule: the entry points it lacks are weak references.
extern "C" int kjb_get_option(kjb_context*, uint32_t, uint32_t*) __attribute__((weak));
extern "C" int kjb_pass_ircache_export_pending(kjb_context*, const kjb_ircache_pending_args*) __attribute__((weak));
extern "C" int kjb_pass_ircache_merge_pending(kjb_context*, const kjb_ircache_pending_args*) __attribute__((weak));
static bool ircache_exact_share(kjb_world* w) {
    uint32_t ordered = 0;
    return kjb_get_option && kjb_pass_ircache_export_pending && kjb_pass_ircache_merge_pending &&
           kjb_get_option(w->ctx, KJB_OPTION_ORDERED_CACHE_SCHEDULE, &ordered) == 0 && ordered == 1;
}
static const uint32_t EV_CACHE_SHARED = 22, CACHE_SHARE_MAX_RECORDS = 32768;
static void ircache_share(kjb_world* w) {
    kjb_context* ctx = w->ctx;
    const uint32_t n = w->tcount;
    const bool exact = ircache_exact_share(w);
    const uint64_t block = exact ? uint64_t(KJB_IRCACHE_PENDING_BLOCK_BYTES) : (uint64_t(KJB_IRCACHE_SHARE_BLOCK_BYTES(CACHE_SHARE_MAX_RECORDS)) + 255) / 256 * 256;
    if (w->xchg_bytes_per_rank[3] != block) {
        if (w->xchg_send[3].data) { kjb_sync(ctx); kjb_buffer_free(ctx, &w->xchg_send[3]); kjb_buffer_free(ctx, &w->xchg_recv[3]); }
        if (kjb_buffer_alloc(ctx, block, &w->xchg_send[3]) || kjb_buffer_alloc(ctx, block * n, &w->xchg_recv[3])) { w->err = 1; return; }
        w->xchg_bytes_per_rank[3] = block;
    }
    const uint32_t queue = w->async_ok ? KJB_QUEUE_ASYNC : KJB_QUEUE_COMPUTE;
    int rc = 0;
    if (queue == KJB_QUEUE_ASYNC) rc |= kjb_queue_wait_event(ctx, KJB_QUEUE_ASYNC, EV_CACHE_USERS_DONE) | kjb_set_pass_queue(ctx, KJB_QUEUE_ASYNC);
    w->pass_begin("tile ircache all-gather");
    if (exact) {   // every rank's block, this rank's own included (merging it changes nothing), in one launch
        kjb_ircache_pending_args a{}; a.ircache = w->frame_cache; a.blocks = w->xchg_send[3]; a.block_count = 1;
        rc |= kjb_pass_ircache_export_pending(ctx, &a);
        rc |= kjb_allgather_on(ctx, queue, w->xchg_send[3].data, w->xchg_recv[3].data, block);
        a.blocks = w->xchg_recv[3]; a.block_count = n;
        if (!rc) rc |= kjb_pass_ircache_merge_pending(ctx, &a);
    } else {
        kjb_ircache_share_args a{}; a.ircache = w->frame_cache; a.max_records = CACHE_SHARE_MAX_RECORDS;
        a.block = w->xchg_send[3];
        rc |= kjb_pass_ircache_export_requests(ctx, &a);
        rc |= kjb_allgather_on(ctx, queue, w->xchg_send[3].data, w->xchg_recv[3].data, block);
        for (uint32_t r = 0; r < n && !rc; ++r) {
            if (r == w->trank) continue;
            a.block = kjb_buffer{(char*)w->xchg_recv[3].data + block * r, block}; a.seed = w->frame_idx * n + r;
            rc |= kjb_pass_ircache_merge_requests(ctx, &a);
        }
    }
    w->pass_end();
    if (queue == KJB_QUEUE_ASYNC) { rc |= kjb_event_record(ctx, EV_CACHE_SHARED, KJB_QUEUE_ASYNC) | kjb_set_pass_queue(ctx, KJB_QUEUE_COMPUTE); w->cache_share_pending = true; }
    if (rc) w->err = 1;
}
// Called after the last pass of the frame that reads or writes the irradiance cache: from here on the next frame's cache chain may run.  The event is
// recorded between two recordings (an event inside a recording is not visible to other queues).
static void cache_users_done(kjb_world* w) {
    if (w->cache_users_done_marked || w->err || w->stopped) return;
    w->cache_users_done_marked = true;
    static const bool no_share = [] { const char* e = getenv("KJB_NO_CACHE_SHARE"); return e && e[0] == '1'; }();   // A/B switch: independent replicas
    const bool share = w->tiled && w->desc.enable_ircache && w->frame_cache.meta_buf.data != nullptr && !no_share;
    if (!w->async_frame && !(share && w->async_ok)) { if (share) ircache_share(w); return; }   // (program order: the event is recorded at the end of the frame)
    const bool reopen = w->graph_open;
    graph_close(w);
    if (kjb_event_record(w->ctx, EV_CACHE_USERS_DONE, KJB_QUEUE_COMPUTE)) w->err = 1;
    if (share) ircache_share(w);
    if (reopen) graph_open_slot(w, 2);
}

// ---------------------------------------------------------------- RtdgiRenderer::render (rtdgi.rs:173-554)
// ---------------------------------------------------------------- IrcacheRenderer / IrcacheRenderState (renderers/ircache.rs)
struct IrcacheState {
    kjb_buffer meta_buf, grid_meta_buf, grid_meta_buf2, entry_cell_buf, spatial_buf, irradiance_buf, aux_buf, life_buf, pool_buf,
               entry_indirection_buf, reposition_proposal_buf, reposition_proposal_count_buf, trace_dispatch_args;
    bool bound = false;
    kjb_ircache_bindings bindings() const {   // bind_mut (ircache.rs:59-78)
        kjb_ircache_bindings b{};
        if (!bound) return b;
        b.meta_buf = meta_buf; b.grid_meta_buf = grid_meta_buf; b.entry_cell_buf = entry_cell_buf; b.spatial_buf = spatial_buf; b.irradiance_buf = irradiance_buf;
        b.life_buf = life_buf; b.pool_buf = pool_buf; b.reposition_proposal_buf = reposition_proposal_buf;
        b.reposition_proposal_count_buf = reposition_proposal_count_buf;
        return b;
    }
};

// IrcacheRenderer::prepare (ircache.rs:166-351)
static IrcacheState ircache_prepare(kjb_world* w) {
    kjb_context* ctx = w->ctx;
    const uint64_t MAX_ENTRIES = KJB_IRCACHE_MAX_ENTRIES, MAX_GRID_CELLS = KJB_IRCACHE_GRID_CELLS;
    IrcacheState st;
    st.meta_buf = w->buf("ircache.meta_buf", 8, KJB_FMT_R32_UINT, 4);
    st.grid_meta_buf = w->buf("ircache.grid_meta_buf", MAX_GRID_CELLS, KJB_FMT_RG32_UINT, 8);
    st.grid_meta_buf2 = w->buf("ircache.grid_meta_buf2", MAX_GRID_CELLS, KJB_FMT_RG32_UINT, 8);
    st.entry_cell_buf = w->buf("ircache.entry_cell_buf", MAX_ENTRIES, KJB_FMT_R32_UINT, 4);
    st.spatial_buf = w->buf("ircache.spatial_buf", MAX_ENTRIES, KJB_FMT_RGBA32_FLOAT, 16);
    st.irradiance_buf = w->buf("ircache.irradiance_buf", 3 * MAX_ENTRIES, KJB_FMT_RGBA32_FLOAT, 16);
    st.aux_buf = w->buf("ircache.aux_buf", 4 * 16 * MAX_ENTRIES, KJB_FMT_RGBA32_FLOAT, 16);
    st.life_buf = w->buf("ircache.life_buf", MAX_ENTRIES, KJB_FMT_R32_UINT, 4);
    st.pool_buf = w->buf("ircache.pool_buf", MAX_ENTRIES, KJB_FMT_R32_UINT, 4);
    st.entry_indirection_buf = w->buf("ircache.entry_indirection_buf", 1024 * 1024, KJB_FMT_R32_UINT, 4);
    st.reposition_proposal_buf = w->buf("ircache.reposition_proposal_buf", MAX_ENTRIES, KJB_FMT_RGBA32_FLOAT, 16);
    st.reposition_proposal_count_buf = w->buf("ircache.reposition_proposal_count_buf", MAX_ENTRIES, KJB_FMT_R32_UINT, 4);
    st.bound = true;
    if (1 == w->ircache_parity) std::swap(st.grid_meta_buf, st.grid_meta_buf2);

    if (!w->ircache_initialized) {
        kjb_ircache_clear_pool_args a{st.pool_buf, st.life_buf};
        RUN("clear ircache pool", kjb_pass_ircache_clear_pool(ctx, &a));
        w->ircache_initialized = true;
    } else {
        kjb_ircache_scroll_cascades_args a{st.grid_meta_buf, st.grid_meta_buf2, st.entry_cell_buf, st.irradiance_buf, st.life_buf, st.pool_buf, st.meta_buf};
        RUN("scroll cascades", kjb_pass_ircache_scroll_cascades(ctx, &a));
        std::swap(st.grid_meta_buf, st.grid_meta_buf2);
        w->ircache_parity = (w->ircache_parity + 1) % 2;
    }
    kjb_buffer age_args = w->buf("ircache.age_dispatch_args", 8, KJB_FMT_R32_UINT, 4);
    { kjb_ircache_dispatch_args_args a{st.meta_buf, age_args}; RUN("_ircache dispatch args", kjb_pass_ircache_prepare_age_dispatch_args(ctx, &a)); }
    kjb_buffer entry_occupancy_buf = w->buf("ircache.entry_occupancy_buf", MAX_ENTRIES, KJB_FMT_R32_UINT, 4);
    {
        kjb_ircache_age_args a{st.meta_buf, st.grid_meta_buf, st.entry_cell_buf, st.life_buf, st.pool_buf, st.spatial_buf, st.reposition_proposal_buf,
                               st.reposition_proposal_count_buf, st.irradiance_buf, entry_occupancy_buf};
        RUN("age ircache entries", kjb_pass_ircache_age_entries(ctx, &a));
    }
    { kjb_prefix_scan_args a{entry_occupancy_buf, uint32_t(MAX_ENTRIES)}; RUN("_prefix scan", kjb_pass_inclusive_prefix_scan_u32(ctx, &a)); }
    { kjb_ircache_compact_args a{st.meta_buf, st.life_buf, entry_occupancy_buf, st.entry_indirection_buf}; RUN("ircache compact", kjb_pass_ircache_compact(ctx, &a)); }
    return st;
}

// IrcacheRenderState::trace_irradiance (ircache.rs:360-487)
static void ircache_trace_irradiance(kjb_world* w, IrcacheState& st, kjb_image& sky_cube) {
    kjb_context* ctx = w->ctx;
    st.trace_dispatch_args = w->buf("ircache.trace_dispatch_args", 16, KJB_FMT_R32_UINT, 4);
    { kjb_ircache_dispatch_args_args a{st.meta_buf, st.trace_dispatch_args}; RUN("_ircache dispatch args", kjb_pass_ircache_prepare_trace_dispatch_args(ctx, &a)); }
    { kjb_ircache_reset_args a{st.life_buf, st.meta_buf, st.irradiance_buf, st.aux_buf, st.entry_indirection_buf}; RUN("ircache reset", kjb_pass_ircache_reset(ctx, &a)); }
    {
        kjb_ircache_trace_access_args a{st.spatial_buf, st.life_buf, st.reposition_proposal_buf, st.meta_buf, st.aux_buf, st.entry_indirection_buf};
        RUN("ircache trace access", kjb_pass_ircache_trace_access(ctx, &a));
    }
    kjb_ircache_trace_args t{};
    t.spatial_buf = st.spatial_buf; t.sky_cube_tex = sky_cube; t.grid_meta_buf = st.grid_meta_buf; t.life_buf = st.life_buf; t.reposition_proposal_buf = st.reposition_proposal_buf;
    t.reposition_proposal_count_buf = st.reposition_proposal_count_buf; t.meta_buf = st.meta_buf; t.aux_buf = st.aux_buf; t.pool_buf = st.pool_buf;
    t.entry_indirection_buf = st.entry_indirection_buf; t.entry_cell_buf = st.entry_cell_buf;
    RUN("ircache validate", kjb_pass_ircache_validate(ctx, &t));
    RUN("ircache trace", kjb_pass_ircache_trace(ctx, &t));
}

// IrcacheRenderState::sum_up_irradiance_for_sampling (ircache.rs:493-511)
static void ircache_sum_up_irradiance(kjb_world* w, IrcacheState& st) {
    kjb_ircache_sum_args a{st.life_buf, st.meta_buf, st.irradiance_buf, st.aux_buf, st.entry_indirection_buf};
    RUN("ircache sum", kjb_pass_ircache_sum(w->ctx, &a));
}

static void rtdgi_render(kjb_world* w, kjb_image& reprojected_history_tex, kjb_image& temporal_output_tex, kjb_image& gbuffer, kjb_image& depth,
                         kjb_image& geometric_normal, kjb_image& reprojection_map, kjb_image& sky_cube, kjb_image& ssao_tex, const kjb_ircache_bindings& ircache) {
    kjb_context* ctx = w->ctx;
    const uint32_t HW = w->HW, HH = w->HH, W = w->W, H = w->H;
    float gbuffer_size[4]; size4(gbuffer_size, gbuffer);
    const TileHalos th = tile_halos(w);
    w->rows_all();   // the half-res extracts are cheap and read at arbitrary screen positions (ray march): whole image

    kjb_image& half_ssao_tex = w->img("rtdgi.half_ssao", HW, HH, KJB_FMT_R8_SNORM);
    kjb_image& half_depth_tex = w->img("half_depth", HW, HH, KJB_FMT_R32_FLOAT);
    kjb_image& half_view_normal_tex = w->img("half_view_normal", HW, HH, KJB_FMT_RGBA8_SNORM);
    if (w->half_depth_frame != w->frame_idx && w->half_normal_frame != w->frame_idx) {   // nothing extracted yet this frame: the three reference passes in one launch
        kjb_extract_half_res_fused_args a{gbuffer, depth, ssao_tex, half_view_normal_tex, half_depth_tex, half_ssao_tex};
        RUN("extract half-res inputs", kjb_pass_extract_half_res_fused(ctx, &a));
        w->half_depth_frame = w->half_normal_frame = w->frame_idx;
    } else { kjb_extract_half_res_args a{ssao_tex, half_ssao_tex}; RUN("extract ssao/2", kjb_pass_extract_half_res_ssao(ctx, &a)); }

    kjb_image *hit_normal_output_tex, *hit_normal_history_tex; w->get_output_and_history(w->temporal_hit_normal_tex, HW, HH, KJB_FMT_RGBA8_UNORM, hit_normal_output_tex, hit_normal_history_tex);
    kjb_image *candidate_output_tex, *candidate_history_tex; w->get_output_and_history(w->temporal_candidate_tex, HW, HH, KJB_FMT_RGBA16_FLOAT, candidate_output_tex, candidate_history_tex);
    kjb_image& candidate_radiance_tex = w->img("rtdgi.candidate_radiance", HW, HH, KJB_FMT_RGBA16_FLOAT);
    kjb_image& candidate_normal_tex = w->img("rtdgi.candidate_normal", HW, HH, KJB_FMT_RGBA8_SNORM);
    kjb_image& candidate_hit_tex = w->img("rtdgi.candidate_hit", HW, HH, KJB_FMT_RGBA16_FLOAT);
    kjb_image& temporal_reservoir_packed_tex = w->img("rtdgi.temporal_reservoir_packed", HW, HH, KJB_FMT_RGBA32_UINT);

    if (w->half_depth_frame != w->frame_idx) { kjb_extract_half_res_args a{depth, half_depth_tex}; RUN("extract half depth", kjb_pass_extract_half_res_depth(ctx, &a)); w->half_depth_frame = w->frame_idx; }

    kjb_image *invalidity_output_tex, *invalidity_history_tex; w->get_output_and_history(w->temporal_invalidity_tex, HW, HH, KJB_FMT_RG16_FLOAT, invalidity_output_tex, invalidity_history_tex);
    kjb_image *radiance_output_tex, *radiance_history_tex; w->get_output_and_history(w->temporal_radiance_tex, HW, HH, KJB_FMT_RGBA16_FLOAT, radiance_output_tex, radiance_history_tex);
    kjb_image *ray_orig_output_tex, *ray_orig_history_tex; w->get_output_and_history(w->temporal_ray_orig_tex, HW, HH, KJB_FMT_RGBA32_FLOAT, ray_orig_output_tex, ray_orig_history_tex);
    kjb_image *ray_output_tex, *ray_history_tex; w->get_output_and_history(w->temporal_ray_tex, HW, HH, KJB_FMT_RGBA16_FLOAT, ray_output_tex, ray_history_tex);

    if (w->half_normal_frame != w->frame_idx) { kjb_extract_half_res_args a{gbuffer, half_view_normal_tex}; RUN("extract view normal/2", kjb_pass_extract_half_res_view_normal(ctx, &a)); w->half_normal_frame = w->frame_idx; }

    kjb_image& rt_history_validity_pre_input_tex = w->img("rtdgi.rt_history_validity_pre_input", HW, HH, KJB_FMT_R8_UNORM);
    kjb_image *reservoir_output_tex, *reservoir_history_tex; w->get_output_and_history(w->temporal_reservoir_tex, HW, HH, KJB_FMT_RG32_UINT, reservoir_output_tex, reservoir_history_tex);

    {   // "rtdgi validate" (rtdgi.rs:293-316)
        kjb_rtdgi_validate_args a{};
        a.half_view_normal_tex = half_view_normal_tex; a.depth_tex = depth; a.reprojected_gi_tex = reprojected_history_tex;
        a.reservoir_tex = *reservoir_history_tex; a.reservoir_ray_history_tex = *ray_history_tex; a.reprojection_tex = reprojection_map;
        a.ircache = ircache; a.sky_cube_tex = sky_cube; a.irradiance_history_tex = *radiance_history_tex; a.ray_orig_history_tex = *ray_orig_history_tex;
        a.rt_history_invalidity_out_tex = rt_history_validity_pre_input_tex; memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        w->rows(th.d4, 1);
        RUN("rtdgi validate", kjb_pass_rtdgi_validate(ctx, &a));
        RUN_TOP("rtdgi validate", kjb_pass_rtdgi_validate(ctx, &a), 12);
    }
    kjb_image& rt_history_validity_input_tex = w->img("rtdgi.rt_history_validity_input", HW, HH, KJB_FMT_R8_UNORM);
    {   // "rtdgi trace" (rtdgi.rs:321-345)
        kjb_rtdgi_trace_args a{};
        a.half_view_normal_tex = half_view_normal_tex; a.depth_tex = depth; a.reprojected_gi_tex = reprojected_history_tex; a.reprojection_tex = reprojection_map;
        a.ircache = ircache; a.sky_cube_tex = sky_cube; a.ray_orig_history_tex = *ray_orig_history_tex;
        a.candidate_irradiance_out_tex = candidate_radiance_tex; a.candidate_normal_out_tex = candidate_normal_tex; a.candidate_hit_out_tex = candidate_hit_tex;
        a.rt_history_invalidity_in_tex = rt_history_validity_pre_input_tex; a.rt_history_invalidity_out_tex = rt_history_validity_input_tex;
        memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        w->rows(th.d4, 1);
        RUN("rtdgi trace", kjb_pass_rtdgi_trace(ctx, &a));
        RUN_TOP("rtdgi trace", kjb_pass_rtdgi_trace(ctx, &a), 12);
    }
    {   // "validity integrate" (rtdgi.rs:347-361)
        kjb_rtdgi_validity_integrate_args a{};
        a.input_tex = rt_history_validity_input_tex; a.history_tex = *invalidity_history_tex; a.reprojection_tex = reprojection_map;
        a.half_view_normal_tex = half_view_normal_tex; a.half_depth_tex = half_depth_tex; a.output_tex = *invalidity_output_tex;
        memcpy(a.gbuffer_tex_size, gbuffer_size, 16); size4(a.output_tex_size, *invalidity_output_tex);
        w->rows(th.d5, 1);
        RUN("validity integrate", kjb_pass_rtdgi_validity_integrate(ctx, &a));
        RUN_TOP("validity integrate", kjb_pass_rtdgi_validity_integrate(ctx, &a), 8);
    }
    {   // "restir temporal" (rtdgi.rs:363-389)
        kjb_rtdgi_restir_temporal_args a{};
        a.half_view_normal_tex = half_view_normal_tex; a.depth_tex = depth; a.candidate_radiance_tex = candidate_radiance_tex; a.candidate_normal_tex = candidate_normal_tex;
        a.candidate_hit_tex = candidate_hit_tex; a.radiance_history_tex = *radiance_history_tex; a.ray_orig_history_tex = *ray_orig_history_tex; a.ray_history_tex = *ray_history_tex;
        a.reservoir_history_tex = *reservoir_history_tex; a.reprojection_tex = reprojection_map; a.hit_normal_history_tex = *hit_normal_history_tex;
        a.candidate_history_tex = *candidate_history_tex; a.rt_invalidity_tex = *invalidity_output_tex;
        a.radiance_out_tex = *radiance_output_tex; a.ray_orig_output_tex = *ray_orig_output_tex; a.ray_output_tex = *ray_output_tex; a.hit_normal_output_tex = *hit_normal_output_tex;
        a.reservoir_out_tex = *reservoir_output_tex; a.candidate_out_tex = *candidate_output_tex; a.temporal_reservoir_packed_tex = temporal_reservoir_packed_tex;
        memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        w->rows(th.d6, 1);
        RUN("restir temporal", kjb_pass_rtdgi_restir_temporal(ctx, &a));
        RUN_TOP("restir temporal", kjb_pass_rtdgi_restir_temporal(ctx, &a), 2);
    }
    kjb_image& radiance_tex = *radiance_output_tex;
    kjb_image* reservoir_input_tex = reservoir_output_tex;
    kjb_image* reservoir_output_tex0 = &w->img("rtdgi.reservoir_output0", HW, HH, KJB_FMT_RG32_UINT);
    kjb_image* reservoir_output_tex1 = &w->img("rtdgi.reservoir_output1", HW, HH, KJB_FMT_RG32_UINT);
    kjb_image none{};   // bounced radiance images only exist with RTDGI_RESTIR_SPATIAL_USE_RAYMARCH_COLOR_BOUNCE (off, rtdgi_restir_settings.hlsl:17)
    for (uint32_t pass_idx = 0; pass_idx < w->desc.spatial_reuse_pass_count; ++pass_idx) {   // rtdgi.rs:428-476
        kjb_rtdgi_restir_spatial_args a{};
        a.reservoir_input_tex = *reservoir_input_tex; a.bounced_radiance_input_tex = none; a.half_view_normal_tex = half_view_normal_tex; a.half_depth_tex = half_depth_tex;
        a.depth_tex = depth; a.half_ssao_tex = half_ssao_tex; a.temporal_reservoir_packed_tex = temporal_reservoir_packed_tex; a.reprojected_gi_tex = reprojected_history_tex;
        a.reservoir_output_tex = *reservoir_output_tex0; a.bounced_radiance_output_tex = none;
        memcpy(a.gbuffer_tex_size, gbuffer_size, 16); size4(a.output_tex_size, *reservoir_output_tex0);
        a.spatial_reuse_pass_idx = pass_idx;
        a.perform_occlusion_raymarch = (pass_idx + 1 == w->desc.spatial_reuse_pass_count) ? 1u : 0u;
        a.occlusion_raymarch_importance_only = w->desc.use_raytraced_reservoir_visibility ? 1u : 0u;
        { uint32_t e = th.spatial_last; for (uint32_t j = pass_idx + 1; j < w->desc.spatial_reuse_pass_count; ++j) e += spatial_radius(j); w->rows(e, 1); }
        RUN("restir spatial", kjb_pass_rtdgi_restir_spatial(ctx, &a));
        std::swap(reservoir_output_tex0, reservoir_output_tex1);
        reservoir_input_tex = reservoir_output_tex1;
    }
    if (w->desc.use_raytraced_reservoir_visibility) {   // "restir check" (rtdgi.rs:478-494)
        kjb_rtdgi_restir_check_args a{}; a.half_depth_tex = half_depth_tex; a.temporal_reservoir_packed_tex = temporal_reservoir_packed_tex; a.reservoir_input_tex = *reservoir_input_tex;
        memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        w->rows(th.spatial_last, 1);
        RUN("restir check", kjb_pass_rtdgi_restir_check(ctx, &a));
    }
    kjb_image& irradiance_output_tex = w->img("rtdgi.irradiance", W, H, KJB_FMT_RGBA16_FLOAT);
    {   // "restir resolve" (rtdgi.rs:502-523)
        kjb_rtdgi_restir_resolve_args a{};
        a.radiance_tex = radiance_tex; a.reservoir_input_tex = *reservoir_input_tex; a.gbuffer_tex = gbuffer; a.depth_tex = depth; a.half_view_normal_tex = half_view_normal_tex;
        a.half_depth_tex = half_depth_tex; a.ssao_tex = ssao_tex; a.candidate_radiance_tex = candidate_radiance_tex; a.candidate_hit_tex = candidate_hit_tex;
        a.temporal_reservoir_packed_tex = temporal_reservoir_packed_tex; a.bounced_radiance_input_tex = none; a.irradiance_output_tex = irradiance_output_tex;
        memcpy(a.gbuffer_tex_size, gbuffer_size, 16); size4(a.output_tex_size, irradiance_output_tex);
        w->rows(th.d9, 2);
        RUN("restir resolve", kjb_pass_rtdgi_restir_resolve(ctx, &a));
    }
    // RtdgiRenderer::temporal (rtdgi.rs:71-115)
    kjb_image *temporal_variance_output_tex, *variance_history_tex; w->get_output_and_history(w->temporal2_variance_tex, W, H, KJB_FMT_RG16_FLOAT, temporal_variance_output_tex, variance_history_tex);
    kjb_image& temporal_filtered_tex = w->img("rtdgi.temporal_filtered", W, H, KJB_FMT_RGBA16_FLOAT);
    {
        kjb_rtdgi_temporal_args a{};
        a.input_tex = irradiance_output_tex; a.history_tex = reprojected_history_tex; a.variance_history_tex = *variance_history_tex; a.reprojection_tex = reprojection_map;
        a.rt_history_invalidity_tex = *invalidity_output_tex; a.output_tex = temporal_filtered_tex; a.history_output_tex = temporal_output_tex;
        a.variance_history_output_tex = *temporal_variance_output_tex;
        size4(a.output_tex_size, temporal_output_tex); memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        w->rows(th.d10, 2);
        RUN("rtdgi temporal", kjb_pass_rtdgi_temporal(ctx, &a));
    }
    if (w->tiled && !w->desc.enable_taa && !w->desc.enable_rtr) tile_exchange_frame(w);   // everything that travels is final: overlap the collective with the spatial filter
    // RtdgiRenderer::spatial (rtdgi.rs:117-141)
    kjb_image& spatial_filtered_tex = w->img("rtdgi.spatial_filtered", W, H, KJB_FMT_RGBA16_FLOAT);
    {
        kjb_rtdgi_spatial_args a{};
        a.input_tex = temporal_filtered_tex; a.depth_tex = depth; a.ssao_tex = ssao_tex; a.geometric_normal_tex = geometric_normal; a.output_tex = spatial_filtered_tex;
        size4(a.output_tex_size, spatial_filtered_tex);
        w->rows(th.d11, 2);
        RUN("rtdgi spatial", kjb_pass_rtdgi_spatial(ctx, &a));
    }
}

// ---------------------------------------------------------------- TaaRenderer::render (taa.rs:41-185)
// ---------------------------------------------------------------- SsgiRenderer::render (ssgi.rs:23-181), USE_AO_ONLY
// The half-res depth / view-normal images are the memoised ones rtdgi uses (mod.rs:54-70); this renderer runs before rtdgi, so it
// produces them here (same kernels, same contents).
static kjb_image& ssgi_render(kjb_world* w, kjb_image& gbuffer, kjb_image& depth, kjb_image& reprojection_map) {
    kjb_context* ctx = w->ctx;
    const uint32_t HW = w->HW, HH = w->HH, W = w->W, H = w->H;
    w->rows_all();   // four small passes: every rank of a tiled frame computes the whole image
    kjb_image& half_view_normal_tex = w->img("half_view_normal", HW, HH, KJB_FMT_RGBA8_SNORM);
    kjb_image& half_depth_tex = w->img("half_depth", HW, HH, KJB_FMT_R32_FLOAT);
    if (w->half_depth_frame != w->frame_idx && w->half_normal_frame != w->frame_idx) {
        kjb_extract_half_res_fused_args a{gbuffer, depth, kjb_image{}, half_view_normal_tex, half_depth_tex, kjb_image{}};
        RUN("extract half-res inputs", kjb_pass_extract_half_res_fused(ctx, &a));
        w->half_depth_frame = w->half_normal_frame = w->frame_idx;
    }
    if (w->half_normal_frame != w->frame_idx) { kjb_extract_half_res_args a{gbuffer, half_view_normal_tex}; RUN("extract view normal/2", kjb_pass_extract_half_res_view_normal(ctx, &a)); w->half_normal_frame = w->frame_idx; }
    if (w->half_depth_frame != w->frame_idx) { kjb_extract_half_res_args a{depth, half_depth_tex}; RUN("extract half depth", kjb_pass_extract_half_res_depth(ctx, &a)); w->half_depth_frame = w->frame_idx; }
    kjb_image& raw = w->img("ssgi.raw", HW, HH, KJB_FMT_R16_FLOAT);
    {
        kjb_ssao_args a{}; a.gbuffer_tex = gbuffer; a.half_depth_tex = half_depth_tex; a.half_view_normal_tex = half_view_normal_tex; a.reprojection_tex = reprojection_map; a.output_tex = raw;
        size4(a.input_tex_size, gbuffer); size4(a.output_tex_size, raw);
        RUN("ssao", kjb_pass_ssao(ctx, &a));
    }
    kjb_image& spatially_filtered_tex = w->img("ssgi.spatial", HW, HH, KJB_FMT_R16_FLOAT);
    { kjb_ssao_spatial_args a{raw, half_depth_tex, half_view_normal_tex, spatially_filtered_tex}; RUN("ssao spatial", kjb_pass_ssao_spatial(ctx, &a)); }
    kjb_image& upsampled_tex = w->img("ssgi.upsampled", W, H, KJB_FMT_R16_FLOAT);
    { kjb_ssao_upsample_args a{spatially_filtered_tex, depth, gbuffer, upsampled_tex}; RUN("ssao upsample", kjb_pass_ssao_upsample(ctx, &a)); }
    kjb_image *history_output_tex, *history_tex; w->get_output_and_history(w->ssgi_tex, W, H, KJB_FMT_R16_FLOAT, history_output_tex, history_tex);
    kjb_image& filtered_output_tex = w->img("ssao", W, H, KJB_FMT_R8_UNORM);
    {
        kjb_ssao_temporal_args a{}; a.input_tex = upsampled_tex; a.history_tex = *history_tex; a.reprojection_tex = reprojection_map; a.final_output_tex = filtered_output_tex;
        a.history_output_tex = *history_output_tex; size4(a.output_tex_size, *history_output_tex);
        RUN("ssao temporal", kjb_pass_ssao_temporal(ctx, &a));
    }
    return filtered_output_tex;
}

// ---------------------------------------------------------------- RtrRenderer::trace + TracedRtr::filter_temporal (rtr.rs:90-399)
// `lighting.render_specular` (world_render_passes.rs:190-201), which adds triangle-light specular into the resolved image before the
// temporal filter, belongs to renderers/lighting.rs and is outside the hot path.
static kjb_image* rtr_render(kjb_world* w, kjb_image& gbuffer, kjb_image& depth, kjb_image& geometric_normal, kjb_image& reprojection_map, kjb_image& sky_cube,
                             kjb_image& rtdgi_irradiance, const kjb_ircache_bindings& ircache) {
    kjb_context* ctx = w->ctx;
    const uint32_t HW = w->HW, HH = w->HH, W = w->W, H = w->H;
    float gbuffer_size[4]; size4(gbuffer_size, gbuffer);
    if (w->spatial_resolve_offsets.empty()) { w->err = 1; return nullptr; }
    const TileHalos th = tile_halos(w);
    if (w->tiled && !w->err && !w->stopped) {
        // Reflection rays land anywhere on screen and read THIS frame's GI there (reflection_trace_common.inc.hlsl, USE_SCREEN_GI_REPROJECTION):
        // every rank contributes its band of the filtered GI and receives the others' — the frame's second (and last) collective.
        std::vector<XchgItem> gi; gi.push_back({rtdgi_irradiance, kjb_world::GRID_FULL, 0});
        w->pass_begin("tile gi all-gather");
        if (tile_exchange(w, gi, KJB_QUEUE_COMPUTE, 1)) w->err = 1;
        w->pass_end();
    }
    // RtdgiCandidates (rtr.rs:105-109): the diffuse candidate images double as the reflection candidates
    kjb_image& refl0_tex = w->img("rtdgi.candidate_radiance", HW, HH, KJB_FMT_RGBA16_FLOAT);
    kjb_image& refl1_tex = w->img("rtdgi.candidate_hit", HW, HH, KJB_FMT_RGBA16_FLOAT);
    kjb_image& refl2_tex = w->img("rtdgi.candidate_normal", HW, HH, KJB_FMT_RGBA8_SNORM);
    kjb_image *rng_output_tex, *rng_history_tex; w->get_output_and_history(w->rtr_temporal_rng_tex, HW, HH, KJB_FMT_R32_UINT, rng_output_tex, rng_history_tex);
    // "reflection trace" and "reflection validate" share no image (new candidates + rng vs the history reservoirs + invalidity mask; both only read the GI and
    // touch the racy cache): two latency-bound ray passes, the second a quarter of the first — with async compute they run side by side (fork here, join
    // after the second; inside a graph recording the fork becomes two branches of the graph).
    bool forked = false;
    if (w->async_ok && !w->err && !w->stopped) {
        if ((kjb_event_record(ctx, EV_FORK, KJB_QUEUE_COMPUTE) | kjb_queue_wait_event(ctx, KJB_QUEUE_ASYNC, EV_FORK)) == 0) forked = true; else w->err = 1;
    }
    {
        kjb_rtr_trace_args a{}; a.gbuffer_tex = gbuffer; a.depth_tex = depth; a.rtdgi_tex = rtdgi_irradiance; a.sky_cube_tex = sky_cube; a.ircache = ircache;
        a.out0_tex = refl0_tex; a.out1_tex = refl1_tex; a.out2_tex = refl2_tex; a.rng_out_tex = *rng_output_tex; memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        a.reuse_rtdgi_rays = w->rtr_reuse_rtdgi_rays ? 1u : 0u;
        w->rows(th.r_rt + 1, 1);
        RUN("reflection trace", kjb_pass_rtr_trace(ctx, &a));
    }
    kjb_image& half_view_normal_tex = w->img("half_view_normal", HW, HH, KJB_FMT_RGBA8_SNORM);   // memoised by rtdgi (mod.rs:54-70)
    kjb_image& half_depth_tex = w->img("half_depth", HW, HH, KJB_FMT_R32_FLOAT);
    kjb_image *ray_orig_output_tex, *ray_orig_history_tex; w->get_output_and_history(w->rtr_temporal_ray_orig_tex, HW, HH, KJB_FMT_RGBA32_FLOAT, ray_orig_output_tex, ray_orig_history_tex);
    kjb_image& refl_restir_invalidity_tex = w->img("rtr.restir_invalidity", HW, HH, KJB_FMT_R8_UNORM);
    kjb_image *hit_normal_output_tex, *hit_normal_history_tex; w->get_output_and_history(w->rtr_temporal_hit_normal_tex, HW, HH, KJB_FMT_RGBA16_FLOAT, hit_normal_output_tex, hit_normal_history_tex);
    kjb_image *irradiance_output_tex, *irradiance_history_tex; w->get_output_and_history(w->rtr_temporal_irradiance_tex, HW, HH, KJB_FMT_RGBA16_FLOAT, irradiance_output_tex, irradiance_history_tex);
    kjb_image *reservoir_output_tex, *reservoir_history_tex; w->get_output_and_history(w->rtr_temporal_reservoir_tex, HW, HH, KJB_FMT_RG32_UINT, reservoir_output_tex, reservoir_history_tex);
    kjb_image *ray_output_tex, *ray_history_tex; w->get_output_and_history(w->rtr_temporal_ray_tex, HW, HH, KJB_FMT_RGBA16_FLOAT, ray_output_tex, ray_history_tex);
    {
        kjb_rtr_validate_args a{}; a.gbuffer_tex = gbuffer; a.depth_tex = depth; a.rtdgi_tex = rtdgi_irradiance; a.sky_cube_tex = sky_cube; a.refl_restir_invalidity_tex = refl_restir_invalidity_tex;
        a.ircache = ircache; a.ray_orig_history_tex = *ray_orig_history_tex; a.ray_history_tex = *ray_history_tex; a.rng_history_tex = *rng_history_tex;
        a.irradiance_history_tex = *irradiance_history_tex; a.reservoir_history_tex = *reservoir_history_tex; memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        w->rows((th.r_validate + 1) & ~1u, 1);
        if (forked && kjb_set_pass_queue(ctx, KJB_QUEUE_ASYNC)) w->err = 1;
        RUN("reflection validate", kjb_pass_rtr_validate(ctx, &a));
        RUN_TOP("reflection validate", kjb_pass_rtr_validate(ctx, &a), 4);   // pixel (0,0): empty reservoirs (payload 0) dereference it from anywhere
        if (forked && (kjb_set_pass_queue(ctx, KJB_QUEUE_COMPUTE) | kjb_event_record(ctx, EV_JOIN, KJB_QUEUE_ASYNC) | kjb_queue_wait_event(ctx, KJB_QUEUE_COMPUTE, EV_JOIN))) w->err = 1;
    }
    cache_users_done(w);   // the reflection filters and everything after them leave the irradiance cache alone
    {
        kjb_rtr_restir_temporal_args a{}; a.gbuffer_tex = gbuffer; a.half_view_normal_tex = half_view_normal_tex; a.depth_tex = depth; a.candidate0_tex = refl0_tex; a.candidate1_tex = refl1_tex;
        a.candidate2_tex = refl2_tex; a.irradiance_history_tex = *irradiance_history_tex; a.ray_orig_history_tex = *ray_orig_history_tex; a.ray_history_tex = *ray_history_tex;
        a.rng_history_tex = *rng_history_tex; a.reservoir_history_tex = *reservoir_history_tex; a.reprojection_tex = reprojection_map; a.hit_normal_history_tex = *hit_normal_history_tex;
        a.irradiance_out_tex = *irradiance_output_tex; a.ray_orig_output_tex = *ray_orig_output_tex; a.ray_output_tex = *ray_output_tex; a.rng_output_tex = *rng_output_tex;
        a.hit_normal_output_tex = *hit_normal_output_tex; a.reservoir_out_tex = *reservoir_output_tex; memcpy(a.gbuffer_tex_size, gbuffer_size, 16);
        w->rows(th.r_rt, 1);
        RUN("rtr restir temporal", kjb_pass_rtr_restir_temporal(ctx, &a));
    }
    kjb_image& resolved_tex = w->img("rtr.resolved", W, H, KJB_FMT_R11G11B10_UFLOAT);
    kjb_image *temporal_output_tex, *history_tex; w->get_output_and_history(w->rtr_temporal_tex, W, H, KJB_FMT_RGBA16_FLOAT, temporal_output_tex, history_tex);
    kjb_image *ray_len_output_tex, *ray_len_history_tex; w->get_output_and_history(w->rtr_ray_len_tex, W, H, KJB_FMT_RG16_FLOAT, ray_len_output_tex, ray_len_history_tex);
    {
        kjb_rtr_resolve_args a{}; a.gbuffer_tex = gbuffer; a.depth_tex = depth; a.hit0_tex = refl0_tex; a.hit1_tex = refl1_tex; a.hit2_tex = refl2_tex; a.history_tex = *history_tex;
        a.reprojection_tex = reprojection_map; a.half_view_normal_tex = half_view_normal_tex; a.half_depth_tex = half_depth_tex; a.ray_len_history_tex = *ray_len_history_tex;
        a.restir_irradiance_tex = *irradiance_output_tex; a.restir_ray_tex = *ray_output_tex; a.restir_reservoir_tex = *reservoir_output_tex; a.restir_ray_orig_tex = *ray_orig_output_tex;
        a.restir_hit_normal_tex = *hit_normal_output_tex; a.output_tex = resolved_tex; a.ray_len_output_tex = *ray_len_output_tex; size4(a.output_tex_size, resolved_tex);
        a.spatial_resolve_offsets = w->spatial_resolve_offsets.data();
        w->rows(th.r_resolve, 2);
        RUN("reflection resolve", kjb_pass_rtr_resolve(ctx, &a));
    }
    if (w->frame_light_count > 0) {   // lighting.render_specular (world_render_passes.rs:190-201, lighting.rs:23-87): the triangle lights' specular, into the resolved reflections
        kjb_image& l0 = w->img("lighting.refl0", HW, HH, KJB_FMT_RGBA16_FLOAT);
        kjb_image& l1 = w->img("lighting.refl1", HW, HH, KJB_FMT_RGBA32_FLOAT);
        kjb_image& l2 = w->img("lighting.refl2", HW, HH, KJB_FMT_RGBA8_SNORM);
        { kjb_sample_lights_args a{}; a.depth_tex = depth; a.out0_tex = l0; a.out1_tex = l1; a.out2_tex = l2; size4(a.gbuffer_tex_size, gbuffer); RUN("sample lights", kjb_pass_sample_lights(ctx, &a)); }
        { kjb_spatial_reuse_lights_args a{}; a.gbuffer_tex = gbuffer; a.depth_tex = depth; a.hit0_tex = l0; a.hit1_tex = l1; a.hit2_tex = l2; a.half_view_normal_tex = half_view_normal_tex;
          a.half_depth_tex = half_depth_tex; a.output_tex = resolved_tex; size4(a.output_tex_size, resolved_tex); a.spatial_resolve_offsets = w->spatial_resolve_offsets.data();
          RUN("spatial reuse lights", kjb_pass_spatial_reuse_lights(ctx, &a)); }
    }
    {   // filter_temporal (rtr.rs:366-398)
        kjb_rtr_temporal_args a{}; a.input_tex = resolved_tex; a.history_tex = *history_tex; a.depth_tex = depth; a.ray_len_tex = *ray_len_output_tex; a.reprojection_tex = reprojection_map;
        a.refl_restir_invalidity_tex = refl_restir_invalidity_tex; a.gbuffer_tex = gbuffer; a.output_tex = *temporal_output_tex; size4(a.output_tex_size, *temporal_output_tex);
        w->rows(th.r_temporal, 2);
        RUN("reflection temporal", kjb_pass_rtr_temporal(ctx, &a));
    }
    {
        kjb_rtr_cleanup_args a{}; a.input_tex = *temporal_output_tex; a.depth_tex = depth; a.geometric_normal_tex = geometric_normal; a.output_tex = resolved_tex;
        a.spatial_resolve_offsets = w->spatial_resolve_offsets.data();
        w->rows(th.r_cleanup, 2);
        RUN("reflection cleanup", kjb_pass_rtr_cleanup(ctx, &a));
    }
    return &resolved_tex;
}

static kjb_image* taa_render(kjb_world* w, kjb_image& input_tex, kjb_image& reprojection_map, kjb_image& depth_tex) {
    kjb_context* ctx = w->ctx;
    const uint32_t OW = w->OW, OH = w->OH, IW = input_tex.width, IH = input_tex.height;
    const TaaRows tr = taa_rows(w, w->trank);   // tile-sharded frames: the band's output / input rows (tile_halos)
    kjb_image *temporal_output_tex, *history_tex; w->get_output_and_history(w->taa_temporal_tex, OW, OH, KJB_FMT_RGBA16_FLOAT, temporal_output_tex, history_tex);
    kjb_image *temporal_velocity_output_tex, *velocity_history_tex; w->get_output_and_history(w->taa_temporal_velocity_tex, OW, OH, KJB_FMT_RG16_FLOAT, temporal_velocity_output_tex, velocity_history_tex);
    kjb_image& reprojected_history_img = w->img("taa.reprojected_history", OW, OH, KJB_FMT_RGBA16_FLOAT);
    kjb_image& closest_velocity_img = w->img("taa.closest_velocity", OW, OH, KJB_FMT_RG16_FLOAT);
    {
        kjb_taa_reproject_args a{}; a.history_tex = *history_tex; a.reprojection_tex = reprojection_map; a.depth_tex = depth_tex; a.output_tex = reprojected_history_img;
        a.closest_velocity_output = closest_velocity_img; size4(a.input_tex_size, input_tex); size4(a.output_tex_size, reprojected_history_img);
        w->rows_span(tr.rep0, tr.rep1); RUN("reproject taa", kjb_pass_taa_reproject(ctx, &a));
    }
    kjb_image *smooth_var_output_tex, *smooth_var_history_tex; w->get_output_and_history(w->taa_temporal_smooth_var_tex, OW, OH, KJB_FMT_RGBA16_FLOAT, smooth_var_output_tex, smooth_var_history_tex);
    kjb_image& filtered_input_img = w->img("taa.filtered_input", IW, IH, KJB_FMT_RGBA16_FLOAT);
    kjb_image& filtered_input_deviation_img = w->img("taa.filtered_input_deviation", IW, IH, KJB_FMT_RGBA16_FLOAT);
    { kjb_taa_filter_input_args a{input_tex, depth_tex, filtered_input_img, filtered_input_deviation_img}; w->rows_span(tr.i0 - 10, tr.i1 + 10); RUN("taa filter input", kjb_pass_taa_filter_input(ctx, &a)); }
    kjb_image& filtered_history_img = w->img("taa.filtered_history", IW, IH, KJB_FMT_RGBA16_FLOAT);
    {
        kjb_taa_filter_history_args a{}; a.input_tex = reprojected_history_img; a.output_tex = filtered_history_img;
        size4(a.input_tex_size, reprojected_history_img); size4(a.output_tex_size, input_tex);
        w->rows_span(tr.i0 - 8, tr.i1 + 8); RUN("taa filter history", kjb_pass_taa_filter_history(ctx, &a));
    }
    kjb_image& input_prob_img = w->img("taa.input_prob", IW, IH, KJB_FMT_R16_FLOAT);
    {
        kjb_taa_input_prob_args a{}; a.input_tex = input_tex; a.filtered_input_tex = filtered_input_img; a.filtered_input_dev_tex = filtered_input_deviation_img;
        a.history_tex = reprojected_history_img; a.filtered_history_tex = filtered_history_img; a.reprojection_tex = reprojection_map; a.depth_tex = depth_tex;
        a.smooth_var_history_tex = *smooth_var_history_tex; a.velocity_history_tex = *velocity_history_tex; a.output_tex = input_prob_img; size4(a.input_tex_size, input_tex);
        w->rows_span(tr.i0 - 6, tr.i1 + 6); RUN("taa input prob", kjb_pass_taa_input_prob(ctx, &a));
    }
    kjb_image& prob_filtered1_img = w->img("taa.prob_filtered1", IW, IH, KJB_FMT_R16_FLOAT);
    { kjb_taa_prob_filter_args a{input_prob_img, prob_filtered1_img}; w->rows_span(tr.i0 - 5, tr.i1 + 5); RUN("taa prob filter", kjb_pass_taa_prob_filter(ctx, &a)); }
    kjb_image& prob_filtered2_img = w->img("taa.prob_filtered2", IW, IH, KJB_FMT_R16_FLOAT);
    { kjb_taa_prob_filter_args a{prob_filtered1_img, prob_filtered2_img}; w->rows_span(tr.i0, tr.i1); RUN("taa prob filter2", kjb_pass_taa_prob_filter2(ctx, &a)); }
    kjb_image& this_frame_output_img = w->img("taa.this_frame_out", OW, OH, KJB_FMT_RGBA16_FLOAT);
    {
        kjb_taa_args a{}; a.input_tex = input_tex; a.history_tex = reprojected_history_img; a.reprojection_tex = reprojection_map; a.closest_velocity_tex = closest_velocity_img;
        a.velocity_history_tex = *velocity_history_tex; a.depth_tex = depth_tex; a.smooth_var_history_tex = *smooth_var_history_tex; a.input_prob_tex = prob_filtered2_img;
        a.temporal_output_tex = *temporal_output_tex; a.output_tex = this_frame_output_img; a.smooth_var_output_tex = *smooth_var_output_tex; a.velocity_output_tex = *temporal_velocity_output_tex;
        size4(a.input_tex_size, input_tex); size4(a.output_tex_size, *temporal_output_tex);
        w->rows_span(tr.o0, tr.o1); RUN("taa", kjb_pass_taa(ctx, &a));
    }
    return &this_frame_output_img;
}

int kjb_world_render_frame(kjb_world* w, const kjb_world_frame* f) {
    kjb_context* ctx = w->ctx;
    kjb_frame_constants fc;
    uint64_t tlas_before[2] = {0, 0}, tlas_after[2] = {0, 0};
    kjb_tlas_stats(ctx, tlas_before);
    if (begin_frame(w, f, fc, true)) return 1;
    kjb_tlas_stats(ctx, tlas_after);
    // what the async cache chain reads besides the cache itself: the acceleration structure and the convolved sky.  A frame that rebuilt / refitted
    // the one or recomputes the other on the compute queue keeps the chain on the compute queue too (program order).
    bool frame_inputs_changed = tlas_before[0] != tlas_after[0] || tlas_before[1] != tlas_after[1];
    const uint32_t W = w->W, H = w->H;

    w->rows_all();
    // sky cube + convolved sky (world_render_passes.rs:33-38, renderers/sky.rs); recomputed only when the sun moves
    kjb_image& sky_cube = w->img("sky_cube", 64, 64, KJB_FMT_RGBA16_FLOAT, 6);
    kjb_image& convolved_sky_cube = w->img("convolved_sky_cube", 16, 16, KJB_FMT_RGBA16_FLOAT, 6);
    if (!w->sky_valid || memcmp(w->sky_sun, fc.sun_direction, 12) != 0) {
        { kjb_sky_cube_args a{sky_cube}; RUN("sky cube", kjb_pass_sky_cube(ctx, &a)); }
        { kjb_convolve_sky_args a{sky_cube, convolved_sky_cube, 16}; RUN("convolve sky", kjb_pass_convolve_sky(ctx, &a)); }
        w->sky_valid = true; memcpy(w->sky_sun, fc.sun_direction, 12);
        frame_inputs_changed = true;
    }

    // G-buffer + depth + geometric normal + velocity (world_render_passes.rs:40-82)
    // streaming mode: two input sets / two result stages so that the copy queues can run one frame ahead / behind the passes
    const bool streaming = f->streaming && f->host_gbuffer && f->host_result && !f->replay_slot;
    const uint32_t sset = w->stream_frames & 1u;
    const uint32_t EV_UP = 8 + sset, EV_DONE = 10 + sset, EV_DL = 12 + sset;   // kjb_event slots per set
    const std::string in_prefix = f->replay_slot ? "slot" + std::to_string(f->replay_slot) + "." : (streaming ? "in" + std::to_string(sset) + "." : "");
    kjb_image& geometric_normal = w->img(in_prefix + "geometric_normal", W, H, KJB_FMT_A2R10G10B10_UNORM);
    kjb_image& gbuffer = w->img(in_prefix + "gbuffer", W, H, KJB_FMT_RGBA32_FLOAT);
    kjb_image& depth = w->img(in_prefix + "depth", W, H, KJB_FMT_R32_FLOAT);
    kjb_image& velocity = w->img(in_prefix + "velocity", W, H, KJB_FMT_RGBA16_FLOAT);
    if (f->replay_slot) {
        // inputs already resident in HBM (captured earlier): nothing to produce
    } else if (f->host_gbuffer && w->tiled) {
        // Tile-sharded frame with host inputs: every rank needs the WHOLE G-buffer (rays land anywhere on screen), but pushing 32 B/px through every
        // rank's PCIe link multiplies the host traffic by N.  Each rank uploads its band only and the bands travel between the GPUs over NVLink
        // (one all-gather, ~17x the bandwidth of a PCIe link): N-fold less host traffic per frame.
        const uint32_t q = streaming ? KJB_QUEUE_UPLOAD : KJB_QUEUE_COMPUTE, r0 = w->grid_row(kjb_world::GRID_FULL, w->ty0), rn = w->grid_row(kjb_world::GRID_FULL, w->ty1) - r0;
        int rc = streaming ? kjb_queue_wait_event(ctx, KJB_QUEUE_UPLOAD, EV_DONE) : 0;
        rc |= kjb_image_upload_rows_on(ctx, q, &gbuffer, f->host_gbuffer, r0, rn) | kjb_image_upload_rows_on(ctx, q, &depth, f->host_depth, r0, rn)
            | kjb_image_upload_rows_on(ctx, q, &geometric_normal, f->host_geometric_normal, r0, rn) | kjb_image_upload_rows_on(ctx, q, &velocity, f->host_velocity, r0, rn);
        if (streaming) rc |= kjb_event_record(ctx, EV_UP, KJB_QUEUE_UPLOAD) | kjb_queue_wait_event(ctx, KJB_QUEUE_COMPUTE, EV_UP);
        if (rc) return rc;
        const kjb_world::Grid FULL = kjb_world::GRID_FULL;
        std::vector<XchgItem> in; in.push_back({gbuffer, FULL, 0}); in.push_back({depth, FULL, 0}); in.push_back({geometric_normal, FULL, 0}); in.push_back({velocity, FULL, 0});
        w->pass_begin("tile input all-gather");
        if (tile_exchange(w, in, KJB_QUEUE_COMPUTE, 2)) w->err = 1;
        w->pass_end();
    } else if (streaming) {
        // the upload queue may overwrite this input set once the passes of the frame that last used it are done
        int rc = kjb_queue_wait_event(ctx, KJB_QUEUE_UPLOAD, EV_DONE);
        rc |= kjb_image_upload_on(ctx, KJB_QUEUE_UPLOAD, &gbuffer, f->host_gbuffer) | kjb_image_upload_on(ctx, KJB_QUEUE_UPLOAD, &depth, f->host_depth)
            | kjb_image_upload_on(ctx, KJB_QUEUE_UPLOAD, &geometric_normal, f->host_geometric_normal) | kjb_image_upload_on(ctx, KJB_QUEUE_UPLOAD, &velocity, f->host_velocity);
        rc |= kjb_event_record(ctx, EV_UP, KJB_QUEUE_UPLOAD) | kjb_queue_wait_event(ctx, KJB_QUEUE_COMPUTE, EV_UP);
        if (rc) return rc;
    } else if (f->host_gbuffer) {
        int rc = kjb_image_upload(ctx, &gbuffer, f->host_gbuffer) | kjb_image_upload(ctx, &depth, f->host_depth)
               | kjb_image_upload(ctx, &geometric_normal, f->host_geometric_normal) | kjb_image_upload(ctx, &velocity, f->host_velocity);
        if (rc) return rc;
    } else {
        kjb_raster_gbuffer_args a{geometric_normal, gbuffer, depth, velocity, nullptr, 0};
        a.prev_instances = w->prev_instances.data(); a.prev_instance_count = uint32_t(w->prev_instances.size());   // slot-aligned with `instances` by construction
        RUN("raster simple", kjb_pass_raster_gbuffer(ctx, &a));
    }
    if (f->capture_slot && !f->replay_slot) {
        const std::string sp = "slot" + std::to_string(f->capture_slot) + ".";
        kjb_image_copy(ctx, &w->img(sp + "geometric_normal", W, H, KJB_FMT_A2R10G10B10_UNORM), &geometric_normal);
        kjb_image_copy(ctx, &w->img(sp + "gbuffer", W, H, KJB_FMT_RGBA32_FLOAT), &gbuffer);
        kjb_image_copy(ctx, &w->img(sp + "depth", W, H, KJB_FMT_R32_FLOAT), &depth);
        kjb_image_copy(ctx, &w->img(sp + "velocity", W, H, KJB_FMT_RGBA16_FLOAT), &velocity);
    }
    // From here to the end of the pass list everything runs on the compute queue: record it and submit the frame as one CUDA graph launch
    // (the inputs above may have come through the upload queue; the result download below goes through the download queue).
    w->cache_users_done_marked = false; w->frame_cache = kjb_ircache_bindings{};
    w->async_ok = w->use_async && !w->profiling && w->frame_idx >= 4 && w->stop_after.empty() && !w->err && kjb_async_passes_supported(ctx) == 1;   // tile-sharded frames too (direct launches)
    w->async_frame = w->async_ok && w->desc.enable_ircache && !frame_inputs_changed;
    graph_open_slot(w, w->async_frame ? 0 : 3);
    // reprojection map + copy depth (renderers/reprojection.rs:6-52)
    kjb_image& reprojection_map = w->img("reprojection_map", W, H, KJB_FMT_RGBA16_SNORM);
    kjb_image& prev_depth = w->img("reprojection.prev_depth", W, H, KJB_FMT_R32_FLOAT);
    {
        kjb_reprojection_map_args a{}; a.depth_tex = depth; a.geometric_normal_tex = geometric_normal; a.prev_depth_tex = prev_depth; a.velocity_tex = velocity; a.output_tex = reprojection_map;
        size4(a.output_tex_size, reprojection_map);
        RUN("reprojection map", kjb_pass_reprojection_map(ctx, &a));
        RUN("copy depth", kjb_image_copy(ctx, &prev_depth, &depth));
    }
    // SSAO guides the rtdgi kernels only; ssgi.rs is outside the hot path: constant 1.0 ("no occlusion"), SURVEY §8d input 2
    kjb_image& ssao_tex = w->img("ssao", W, H, KJB_FMT_R8_UNORM);
    if (w->desc.enable_ssao) ssgi_render(w, gbuffer, depth, reprojection_map);   // ssgi.render (world_render_passes.rs:90-96)
    else if (!w->ssao_filled) { kjb_image_fill_u8(ctx, &ssao_tex, 255); w->ssao_filled = true; }

    // ircache.prepare + trace_irradiance (world_render_passes.rs:99-122): cache rays use the convolved sky cube
    IrcacheState ircache_state;
    if (w->desc.enable_ircache) {
        if (w->cache_share_pending) { if (kjb_queue_wait_event(ctx, w->async_frame ? KJB_QUEUE_ASYNC : KJB_QUEUE_COMPUTE, EV_CACHE_SHARED)) w->err = 1; w->cache_share_pending = false; }
        if (w->async_frame && (kjb_queue_wait_event(ctx, KJB_QUEUE_ASYNC, EV_CACHE_USERS_DONE) | kjb_set_pass_queue(ctx, KJB_QUEUE_ASYNC))) w->err = 1;
        ircache_state = ircache_prepare(w); ircache_trace_irradiance(w, ircache_state, convolved_sky_cube);
        w->frame_cache = ircache_state.bindings();
        if (w->async_frame && kjb_set_pass_queue(ctx, KJB_QUEUE_COMPUTE)) w->err = 1;
    }

    // rtdgi.reproject (world_render_passes.rs:129, rtdgi.rs:143-171)
    kjb_image *temporal_output_tex, *history_tex; w->get_output_and_history(w->temporal2_tex, W, H, KJB_FMT_RGBA16_FLOAT, temporal_output_tex, history_tex);
    kjb_image& reprojected_history_tex = w->img("rtdgi.reprojected_history", W, H, KJB_FMT_RGBA16_FLOAT);
    {
        kjb_rtdgi_reproject_args a{}; a.input_tex = *history_tex; a.reprojection_tex = reprojection_map; a.output_tex = reprojected_history_tex;
        size4(a.output_tex_size, reprojected_history_tex);
        if (w->exchange_pending) { if (kjb_queue_wait_event(ctx, KJB_QUEUE_COMPUTE, EV_XCHG_DONE)) w->err = 1; w->exchange_pending = false; }   // first consumer of exchanged history
        RUN("rtdgi reproject", kjb_pass_rtdgi_reproject(ctx, &a));
    }
    if (w->desc.enable_ircache) {   // world_render_passes.rs:138-140
        if (w->async_frame && kjb_set_pass_queue(ctx, KJB_QUEUE_ASYNC)) w->err = 1;
        ircache_sum_up_irradiance(w, ircache_state);
        if (w->async_frame) {
            if (kjb_event_record(ctx, EV_CACHE_READY, KJB_QUEUE_ASYNC) | kjb_set_pass_queue(ctx, KJB_QUEUE_COMPUTE)) w->err = 1;
            // the cache's first user this frame ("rtdgi validate") waits for the chain: the wait sits between two recordings
            const bool reopen = w->graph_open;
            graph_close(w);
            if (kjb_queue_wait_event(ctx, KJB_QUEUE_COMPUTE, EV_CACHE_READY)) w->err = 1;
            if (reopen) graph_open_slot(w, 1);
        }
    }
    // rtdgi.render (world_render_passes.rs:146-160): diffuse rays use the convolved sky cube
    rtdgi_render(w, reprojected_history_tex, *temporal_output_tex, gbuffer, depth, geometric_normal, reprojection_map, convolved_sky_cube, ssao_tex, ircache_state.bindings());

    // rtr.trace + filter_temporal (world_render_passes.rs:171-205): reflection rays use the full sky cube
    if (w->desc.enable_rtr) {
        kjb_image gi{};
        if (kjb_world_get_image(w, "rtdgi.spatial_filtered", &gi) == 0) rtr_render(w, gbuffer, depth, geometric_normal, reprojection_map, sky_cube, gi, ircache_state.bindings());
    }
    cache_users_done(w);   // without reflections the diffuse GI passes were the last users

    // light_gbuffer + taa.render (world_render_passes.rs:215-263)
    const char* result_name = "rtdgi.spatial_filtered";
    if (w->desc.enable_lighting && !w->err && !w->stopped) {
        // "trace shadow mask" (+ the shadow denoiser under a soft sun) + "light gbuffer" (world_render_passes.rs:124-137,215-232)
        w->rows_all();
        kjb_image& sun_shadow_mask = w->img("sun_shadow_mask", W, H, KJB_FMT_R8_UNORM);
        { kjb_trace_sun_shadow_mask_args a{depth, geometric_normal, sun_shadow_mask}; RUN("trace shadow mask", kjb_pass_trace_sun_shadow_mask(ctx, &a)); }
        kjb_image gi{}; kjb_world_get_image(w, "rtdgi.spatial_filtered", &gi);
        kjb_image& rtr = w->img("rtr.resolved", W, H, KJB_FMT_R11G11B10_UFLOAT);   // zero image when rtr is off (create_dummy_output, rtr.rs:327-362)
        kjb_image& accum_img = w->img("accum", W, H, KJB_FMT_RGBA16_FLOAT);
        kjb_image& debug_out_tex = w->img("debug_out", W, H, KJB_FMT_RGBA16_FLOAT);
        // ShadowDenoiseRenderer::render (shadow_denoise.rs:19-120) whenever the sun is an area light (world_render_passes.rs:130-137)
        kjb_image* shadow_for_lighting = &sun_shadow_mask;
        if (w->sun_size_multiplier > 0.0f) {   // world_render_passes.rs:130
            uint32_t ext[2] = {(W + 7) / 8, (H + 3) / 4};
            float size[4]; size4(size, gbuffer);
            kjb_image& bitpacked = w->img("shadow_denoise.bitpacked", ext[0], ext[1], KJB_FMT_R32_UINT);
            { kjb_shadow_bitpack_args b{sun_shadow_mask, bitpacked, {size[0], size[1], size[2], size[3]}, {ext[0], ext[1]}}; RUN("shadow bitpack", kjb_pass_shadow_bitpack(ctx, &b)); }
            kjb_image *moments_image, *prev_moments_image; w->get_output_and_history(w->shadow_denoise_moments, W, H, KJB_FMT_RGBA16_FLOAT, moments_image, prev_moments_image);
            kjb_image *accum_image, *prev_accum_image; w->get_output_and_history(w->shadow_denoise_accum, W, H, KJB_FMT_RG16_FLOAT, accum_image, prev_accum_image);
            kjb_image& spatial_input_image = w->img("shadow_denoise.spatial_input", W, H, KJB_FMT_RG16_FLOAT);
            kjb_image& metadata_image = w->img("shadow_denoise.metadata", ext[0], ext[1], KJB_FMT_R32_UINT);
            { kjb_shadow_temporal_args b{sun_shadow_mask, bitpacked, *prev_moments_image, *prev_accum_image, reprojection_map, *moments_image, spatial_input_image, metadata_image,
                                         {size[0], size[1], size[2], size[3]}, {ext[0], ext[1]}};
              RUN("shadow temporal", kjb_pass_shadow_temporal(ctx, &b)); }
            kjb_image& temp = w->img("shadow_denoise.temp", W, H, KJB_FMT_RG16_FLOAT);
            auto filter_spatial = [&](uint32_t step, kjb_image& in, kjb_image& out) {
                kjb_shadow_spatial_args b{in, metadata_image, geometric_normal, depth, out, {size[0], size[1], size[2], size[3]}, {ext[0], ext[1]}, step};
                RUN("shadow spatial", kjb_pass_shadow_spatial(ctx, &b));
            };
            filter_spatial(1, spatial_input_image, *accum_image);
            filter_spatial(2, *accum_image, temp);
            filter_spatial(4, temp, spatial_input_image);
            shadow_for_lighting = &spatial_input_image;
        }
        kjb_light_gbuffer_args a{}; a.gbuffer_tex = gbuffer; a.depth_tex = depth; a.shadow_mask_tex = *shadow_for_lighting; a.rtr_tex = rtr; a.rtdgi_tex = gi;
        a.temporal_output_tex = accum_img; a.output_tex = debug_out_tex; a.unconvolved_sky_cube_tex = sky_cube; a.sky_cube_tex = convolved_sky_cube; size4(a.output_tex_size, gbuffer); a.debug_shading_mode = w->debug_shading_mode;
        RUN("light gbuffer", kjb_pass_light_gbuffer(ctx, &a));
        result_name = "debug_out";
    }
    if (w->desc.enable_taa) {
        // taa consumes the lit image when the lighting composite runs (world_render_passes.rs:253-263), else the GI result directly
        kjb_image taa_in{};
        if (kjb_world_get_image(w, result_name, &taa_in) == 0) { taa_render(w, taa_in, reprojection_map, depth); result_name = "taa.this_frame_out"; }
    }
    graph_close(w);
    if (!w->async_frame && w->desc.enable_ircache && kjb_event_record(ctx, EV_CACHE_USERS_DONE, KJB_QUEUE_COMPUTE)) w->err = 1;   // a later async frame orders its chain after this frame
    if (w->tiled && !w->exchanged_this_frame) tile_exchange_frame(w);   // with TAA its history images travel too: exchange at the end of the frame
    uint32_t res0 = 0, res1 = 0; kjb_world_result_rows(w, &res0, &res1);   // a rank delivers its rows of the result (kjb_world_result_rows)
    if (streaming && !w->err) {
        kjb_image result{};
        if (kjb_world_get_image(w, result_name, &result) == 0) {
            kjb_image& stage = w->img("result.stage" + std::to_string(sset), result.width, result.height, result.format);
            int rc = kjb_queue_wait_event(ctx, KJB_QUEUE_COMPUTE, EV_DL);          // the previous download from this stage has drained
            rc |= kjb_image_copy(ctx, &stage, &result) | kjb_event_record(ctx, EV_DONE, KJB_QUEUE_COMPUTE);
            rc |= kjb_queue_wait_event(ctx, KJB_QUEUE_DOWNLOAD, EV_DONE);
            rc |= w->tiled ? kjb_image_download_rows_on(ctx, KJB_QUEUE_DOWNLOAD, &stage, f->host_result, res0, res1 - res0)
                           : kjb_image_download_on(ctx, KJB_QUEUE_DOWNLOAD, &stage, f->host_result);
            rc |= kjb_event_record(ctx, EV_DL, KJB_QUEUE_DOWNLOAD);
            if (rc) w->err = rc;
        }
        w->stream_frames += 1;
    } else if (f->host_result && !w->err) {
        kjb_image result{};
        if (kjb_world_get_image(w, result_name, &result) == 0) {
            if (w->tiled) kjb_image_download_rows_on(ctx, KJB_QUEUE_COMPUTE, &result, f->host_result, res0, res1 - res0);
            else kjb_image_download(ctx, &result, f->host_result);
            kjb_sync(ctx);
        }
    }
    end_frame(w);
    return w->err;
}

int kjb_world_wait(kjb_world* w) {
    int rc = kjb_event_synchronize(w->ctx, 12) | kjb_event_synchronize(w->ctx, 13);
    return rc | kjb_sync(w->ctx);
}

int kjb_world_render_reference(kjb_world* w, const kjb_world_frame* f, uint32_t indirect_only) {
    kjb_frame_constants fc;
    if (begin_frame(w, f, fc, false)) return 1;
    kjb_image& accum = w->img("refpt.accum", w->W, w->H, KJB_FMT_RGBA32_FLOAT);
    if (w->reset_reference_accumulation) { w->reset_reference_accumulation = false; if (kjb_image_clear(w->ctx, &accum)) w->err = 1; }   // world_render_passes.rs:311-314
    kjb_reference_pt_args a{accum, indirect_only};
    RUN("reference pt", kjb_pass_reference_path_trace(w->ctx, &a));
    if (f->host_result && !w->err) { kjb_image_download(w->ctx, &accum, f->host_result); kjb_sync(w->ctx); }
    end_frame(w);
    return w->err;
}

}  // extern "C"
