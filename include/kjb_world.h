/* kjb_world.h — host-side frame driver above the per-pass C-ABI (kjb.h).
 *
 * kajiya's host for this path is Rust (not available here): `WorldRenderer`
 * (crates/lib/kajiya/src/world_renderer.rs), the per-frame pass list
 * `prepare_render_graph_standard` (crates/lib/kajiya/src/world_render_passes.rs:13-292) and the
 * per-effect modules `renderers/{rtdgi,ircache,rtr,taa}.rs`.  This is their C++ mirror: same scene
 * API (add_mesh / add_instance), same temporal resources and ping-pong keys, same pass order, same
 * constants tuples — it only ever talks to the GPU through the `kjb_pass_*` entry points, so a Rust
 * render-graph closure and this driver are interchangeable callers of the drop-in boundary.
 * The same source is linked into the CUDA library, the CPU-emulation test build and the oracle, so
 * frame sequences can be replayed against any of them.
 */
#ifndef KJB_WORLD_H
#define KJB_WORLD_H
#include "kjb.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct kjb_world kjb_world;

typedef struct kjb_world_desc {
    uint32_t render_width, render_height;         /* WorldFrameDesc::render_extent */
    uint32_t temporal_upscale_width, temporal_upscale_height;   /* TAA output extent; 0 = same as render */
    uint32_t spatial_reuse_pass_count;            /* RtdgiRenderer::spatial_reuse_pass_count (default 2) */
    uint32_t use_raytraced_reservoir_visibility;  /* RtdgiRenderer (default 0) */
    uint32_t enable_ircache, enable_rtr, enable_taa;
    /* Tile sharding (SURVEY §8e): this process renders half-res rows [tile_y0, tile_y1) plus a halo. 0,0 = whole frame. */
    uint32_t tile_y0, tile_y1;
    /* Tile sharding by rank: with tile_count > 1 this world renders the tile_rank-th of tile_count horizontal bands (balanced
     * split of the half-res rows) and exchanges band borders once per frame through kjb_allgather. Overrides tile_y0/y1. */
    uint32_t tile_rank, tile_count;
    uint32_t enable_ssao;   /* SsgiRenderer (ssgi.rs): real screen-space occlusion instead of the constant-1 guide */
    /* "trace shadow mask" + shadow denoiser + "light gbuffer" (world_render_passes.rs:124-137,215-232): the lit image ("debug_out"), which then is
     * what TAA consumes.  hard_sun = WorldRenderer::sun_size_multiplier 0: a point sun, for which upstream skips the denoiser (and so do we). */
    uint32_t enable_lighting, hard_sun;
} kjb_world_desc;

/* TriangleMesh as the asset pipeline hands it to add_mesh (kajiya-asset/src/mesh.rs:85-98) */
typedef struct kjb_mesh_desc {
    const float    *positions;      /* 3 per vertex */
    const float    *normals;        /* 3 per vertex */
    const float    *uvs;            /* 2 per vertex, may be NULL (zeros) */
    const float    *colors;         /* 4 per vertex, may be NULL (ones) */
    const uint32_t *material_ids;   /* 1 per vertex */
    const uint32_t *indices;
    uint32_t vertex_count, index_count;
    const kjb_mesh_material *materials;   /* `maps` index this mesh's own map list */
    uint32_t material_count;
    const kjb_texture_desc *maps;
    uint32_t map_count;
    uint32_t use_lights;            /* AddMeshOptions::use_lights */
} kjb_mesh_desc;

typedef struct kjb_world_frame {
    float camera_position[3];
    float camera_rotation[4];       /* quaternion xyzw */
    float vertical_fov_deg;         /* CameraLens (camera.rs:40-55): default 52 */
    float near_plane;               /* default 0.01 */
    float sun_direction[3];         /* direction TOWARDS the sun */
    float delta_time_seconds;
    /* Optional host-resident G-buffer inputs (pinned memory recommended).  When `host_gbuffer` is non-NULL the
     * raster stand-in is skipped and these are uploaded inside the call: gbuffer RGBA32F, depth R32F,
     * geometric normal A2R10G10B10, velocity RGBA16F — i.e. what kajiya's raster pass would hand over. */
    const void *host_gbuffer, *host_depth, *host_geometric_normal, *host_velocity;
    /* Optional host destination for the frame's result (rtdgi screen irradiance, RGBA16F full-res; the TAA
     * output RGBA16F when TAA is enabled).  Copied device->host inside the call when non-NULL.  A tile-sharded
     * world writes only its rows of it (kjb_world_result_rows). */
    void *host_result;
    /* Device-resident G-buffer ring for benchmarking with inputs already in HBM: capture_slot = k > 0 stores this frame's
     * G-buffer inputs (after the raster stand-in / upload) in ring slot k; replay_slot = k > 0 binds ring slot k as the
     * frame's G-buffer inputs (no raster pass, no copy). */
    uint32_t capture_slot, replay_slot;
    /* Streaming mode (host_gbuffer + host_result given, streaming != 0): the call returns as soon as the frame is enqueued.  Uploads,
     * passes and the result download run on three queues with two frames in flight, so the copies of neighbouring frames overlap the
     * passes.  The host input buffers of a frame and its host_result must stay untouched until kjb_world_wait() (or until two further
     * streaming frames have been submitted); consecutive frames must use different host_result buffers. */
    uint32_t streaming;
} kjb_world_frame;

int  kjb_world_create(kjb_context *ctx, const kjb_world_desc *desc, kjb_world **out);
void kjb_world_destroy(kjb_world *w);
/* WorldRenderer::add_mesh (world_renderer.rs:604-776) / add_instance (:778-). transform = row-major 3x4. */
int  kjb_world_add_mesh(kjb_world *w, const kjb_mesh_desc *mesh, uint32_t *out_mesh_handle);
int  kjb_world_add_instance(kjb_world *w, uint32_t mesh_handle, const float transform[12], uint32_t *out_instance_handle);
/* WorldRenderer::set_instance_transform (world_renderer.rs:815-818). The next frame re-flattens the acceleration structure.
 * (The primary-visibility stand-in that produces the G-buffer when the host supplies none uses last frame's transform for the velocity.) */
int  kjb_world_set_instance_transform(kjb_world *w, uint32_t instance_handle, const float transform[12]);
/* WorldRenderer::remove_instance (world_renderer.rs:800-813): swap_remove — the LAST instance moves into the freed slot (InstanceID order, hence ray tie-breaks, follow upstream) */
int  kjb_world_remove_instance(kjb_world *w, uint32_t instance_handle);
/* InstanceDynamicParameters::emissive_multiplier (world_renderer.rs:96-105,828-834): scales the instance's emissive in hit shading and its triangle lights */
int  kjb_world_set_instance_emissive_multiplier(kjb_world *w, uint32_t instance_handle, float emissive_multiplier);
/* WorldRenderer's public knobs that reach FrameConstants (world_renderer.rs:200-211,1066-1108): sun colour multiplier and sky ambient (baked into
 * the sky cubes, which are recomputed), RenderOverrides (KJB_OVERRIDE_* flags + material roughness scale, consumed by the closest-hit shader),
 * debug_shading_mode of the lit composite (0 default, 2 diffuse GI, 3 reflections, 4 "RTX off"). */
int  kjb_world_set_sun_color_multiplier(kjb_world *w, const float rgb[3]);
int  kjb_world_set_sky_ambient(kjb_world *w, const float rgb[3]);
int  kjb_world_set_render_overrides(kjb_world *w, uint32_t flags, float material_roughness_scale);
int  kjb_world_set_debug_shading_mode(kjb_world *w, uint32_t mode);
/* WorldRenderer::sun_size_multiplier (world_renderer.rs:207,1078): angular radius of the sun disk in units of the real one; 0 = point sun (no shadow
 * denoiser, world_render_passes.rs:130).  kjb_world_desc.hard_sun only picks the initial value (0 or 1). */
int  kjb_world_set_sun_size_multiplier(kjb_world *w, float multiplier);
/* the 256x256 RGBA8 blue-noise LUT (bindless slot 1; assets/images/bluenoise/256_256/LDR_RGBA_0.png in the reference) */
int  kjb_world_set_blue_noise(kjb_world *w, const uint8_t *rgba8_256x256);
/* SPATIAL_RESOLVE_OFFSETS (rtr.rs:402-915): the int4[512] constant table the reflection passes receive; required when enable_rtr */
int  kjb_world_set_spatial_resolve_offsets(kjb_world *w, const int32_t *int4x512);
/* one frame of prepare_render_graph_standard's hot-path passes; enqueues, does not sync (unless host_result is set) */
int  kjb_world_render_frame(kjb_world *w, const kjb_world_frame *frame);
/* one frame of prepare_render_graph_reference (world_render_passes.rs:294-330): the path tracer accumulating in place */
int  kjb_world_render_reference(kjb_world *w, const kjb_world_frame *frame, uint32_t indirect_only);
/* WorldRenderer::reset_reference_accumulation (world_renderer.rs:183): the next reference frame starts from a cleared accumulator (camera moved, scene edited) */
int  kjb_world_reset_reference_accumulation(kjb_world *w);
/* block until every streaming frame submitted so far has delivered its host_result */
int  kjb_world_wait(kjb_world *w);
uint32_t kjb_world_frame_index(kjb_world *w);
/* Rows [*y0, *y1) of the frame's result image (the TAA output, temporal_upscale_height rows; the render-res result without TAA) that this world
 * owns: what a tile-sharded frame writes into host_result, at the same rows of a whole-frame buffer.  Band boundary b (half-res rows) maps to
 * result row floor(RH * min(2b, render_height) / render_height), so the ranks' rows partition [0, RH) for any heights.  Untiled: [0, RH). */
int  kjb_world_result_rows(kjb_world *w, uint32_t *y0, uint32_t *y1);
/* Look up a live image by its reference resource name ("rtdgi.radiance:0", "gbuffer", "rtdgi.irradiance", ...). */
int  kjb_world_get_image(kjb_world *w, const char *name, kjb_image *out);
/* names of all live images, '\n' separated (test harness iterates them for per-pass parity) */
const char *kjb_world_image_names(kjb_world *w);
/* kernel launches / rays of the last frame */
int  kjb_world_last_frame_stats(kjb_world *w, uint64_t out[4]);   /* launches, closest rays, any-hit rays, passes */
/* Run frames only up to (and including) the pass with this rg label, for per-pass debugging ("" = all). */
int  kjb_world_set_stop_after(kjb_world *w, const char *pass_label);
/* Per-pass device timing: when on, every pass is bracketed by kjb_timer_record and accumulated per rg label. */
int  kjb_world_set_profiling(kjb_world *w, uint32_t on);
/* Submit each frame's passes as ONE CUDA graph launch (kjb_graph_begin / kjb_graph_end around the pass list).  On by default; it applies from the fifth
 * frame on (every lazily created resource exists by then), never while per-pass profiling is on or the frame is tile-sharded (its exchange lives on
 * another queue).  The environment variable KJB_NO_GRAPH=1 switches the default off (A/B timing). */
int  kjb_world_set_cuda_graph(kjb_world *w, uint32_t on);
/* Async compute (kjb_set_pass_queue, kjb.h): the irradiance-cache chain of a frame — cascade scroll, ageing, compaction, cache rays, sum — is ~10 small,
 * latency-bound launches that need nothing of the frame's screen-space inputs, only that the PREVIOUS frame's cache users ("rtdgi validate/trace",
 * "reflection trace/validate") are done.  With this on (default; CUDA backend, from the fifth frame, not while profiling / serialised, not in a
 * frame that rebuilt the acceleration structure or the sky) the chain is enqueued on the async queue: it runs under the previous frame's reflection
 * filters and TAA and under this frame's reprojection passes, and the frame is submitted as three recordings around the two ordering points.  The pass
 * call order (the reference's render-graph order) does not change.  KJB_NO_ASYNC=1 switches the default off (A/B timing). */
int  kjb_world_set_async_compute(kjb_world *w, uint32_t on);
/* "label\tcalls\ttotal_ms\n" per pass since profiling was switched on (synchronises). */
const char *kjb_world_pass_timings(kjb_world *w);

#ifdef __cplusplus
}
#endif
#endif
