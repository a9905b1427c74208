/* kjb.h — C-ABI of the H100-native kajiya ReSTIR-GI hot path.
 *
 * kajiya has no FFI: its extension point is the Rust closure handed to
 * `PassBuilder::render` (crates/lib/kajiya-rg/src/pass_builder.rs:325-337), normally built
 * with `SimpleRenderPass` (crates/lib/kajiya-rg/src/hl.rs:104-406).  Every entry point below
 * replaces the body of ONE such closure — the `vkCmdDispatch` / `vkCmdTraceRaysKHR` that
 * `SimpleRenderPass::{dispatch,trace_rays}` records (hl.rs:133-253) — and is named after the
 * render-graph pass label the reference gives it (`rg.add_pass("rtdgi trace")`, ...).
 * The fields of each `*_args` struct are the resources in the reference's BINDING ORDER
 * (binding index = call order of .read/.write/.constants, hl.rs:266,324,354-359) followed by the
 * constants tuple byte-for-byte.
 *
 * Conventions (SURVEY.md §8b):
 *   - plain pointers and sizes, no C++/torch types; all structs are POD;
 *   - every call returns 0 on success, non-zero on error (`kjb_last_error` gives the text);
 *     nothing unwinds across the boundary (the Rust closure maps non-zero to BackendError);
 *   - every call only ENQUEUES work on the context's CUDA stream, in call order (the reference
 *     records passes serially in declaration order, graph.rs:865-867); `kjb_sync` waits;
 *   - image memory is owned by whoever allocated it (`kjb_image_alloc` for the library's
 *     allocator); the library never frees caller-owned handles;
 *   - images are tightly packed row-major linear buffers of the texel formats below
 *     (the Vulkan formats the reference creates them with), temporal images are zero-filled
 *     at allocation (the reference leaves them undefined, temporal.rs:204-205).
 */
#ifndef KJB_H
#define KJB_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KJB_ABI_VERSION 1

/* ------------------------------------------------------------------ formats */
typedef enum kjb_format {
    KJB_FMT_UNKNOWN = 0,
    KJB_FMT_R32_FLOAT = 1,          /* depth (D32_SFLOAT), half depth                          4 B */
    KJB_FMT_RG32_UINT = 2,          /* reservoirs (rtdgi.rs:286)                                8 B */
    KJB_FMT_RGBA32_FLOAT = 3,       /* gbuffer, ray_orig (world_render_passes.rs:49, rtdgi.rs:261) 16 B */
    KJB_FMT_RGBA32_UINT = 4,        /* temporal_reservoir_packed (rtdgi.rs:232)                16 B */
    KJB_FMT_RGBA16_FLOAT = 5,       /* most colour targets                                      8 B */
    KJB_FMT_RG16_FLOAT = 6,         /* invalidity, variance                                     4 B */
    KJB_FMT_RGBA8_UNORM = 7,        /* hit_normal (rtdgi.rs:211)                                4 B */
    KJB_FMT_RGBA8_SNORM = 8,        /* half view normal, candidate normal                       4 B */
    KJB_FMT_R8_UNORM = 9,           /* rt_history_validity, ssao                                1 B */
    KJB_FMT_R8_SNORM = 10,          /* half ssao (rtdgi.rs:190)                                 1 B */
    KJB_FMT_RGBA16_SNORM = 11,      /* reprojection map (reprojection.rs)                       8 B */
    KJB_FMT_A2R10G10B10_UNORM = 12, /* geometric normal (world_render_passes.rs:44)             4 B */
    KJB_FMT_R11G11B10_UFLOAT = 13,  /* rtr resolve output                                       4 B */
    KJB_FMT_R32_UINT = 14,
    KJB_FMT_R16_FLOAT = 15,
    KJB_FMT_RG32_FLOAT = 16,
    KJB_FMT_COUNT_
} kjb_format;

/* A 2D image (or, with `layers` > 1, a 2D array / cube stored layer after layer). */
typedef struct kjb_image {
    void    *data;      /* device pointer (CUDA build) / host pointer (oracle, emulator) */
    uint32_t width;
    uint32_t height;
    uint32_t format;    /* kjb_format */
    uint32_t layers;    /* 1 for plain 2D, 6 for cubes */
} kjb_image;

typedef struct kjb_buffer {
    void    *data;
    uint64_t size_bytes;
} kjb_buffer;

/* ------------------------------------------------------------------ frame constants
 * Byte-identical to rust-shaders-shared: ViewConstants (view_constants.rs:4-23),
 * FrameConstants (frame_constants.rs:13-37), HLSL twin inc/frame_constants.hlsl:8-82.
 * Matrices are glam column-major: element (row r, col c) = m[c*4 + r].                */
typedef struct kjb_mat4 { float m[16]; } kjb_mat4;

typedef struct kjb_view_constants {
    kjb_mat4 view_to_clip, clip_to_view, view_to_sample, sample_to_view, world_to_view, view_to_world;
    kjb_mat4 clip_to_prev_clip;
    kjb_mat4 prev_view_to_prev_clip, prev_clip_to_prev_view, prev_world_to_prev_view, prev_view_to_prev_world;
    float sample_offset_pixels[2];
    float sample_offset_clip[2];
} kjb_view_constants;

#define KJB_IRCACHE_CASCADE_COUNT 12
typedef struct kjb_ircache_cascade_constants {
    int32_t origin[4];
    int32_t voxels_scrolled_this_frame[4];
} kjb_ircache_cascade_constants;

#define KJB_OVERRIDE_FORCE_FACE_NORMALS 1u
#define KJB_OVERRIDE_NO_NORMAL_MAPS 2u
#define KJB_OVERRIDE_FLIP_NORMAL_MAP_YZ 4u
#define KJB_OVERRIDE_NO_METAL 8u

typedef struct kjb_frame_constants {
    kjb_view_constants view_constants;
    float    sun_direction[4];
    uint32_t frame_index;
    float    delta_time_seconds;
    float    sun_angular_radius_cos;
    uint32_t triangle_light_count;
    float    sun_color_multiplier[4];
    float    sky_ambient[4];
    float    pre_exposure;
    float    pre_exposure_prev;
    float    pre_exposure_delta;
    float    pad0;
    uint32_t render_override_flags;
    float    render_override_material_roughness_scale;
    uint32_t render_override_pad0, render_override_pad1;
    float    ircache_grid_center[4];
    kjb_ircache_cascade_constants ircache_cascades[KJB_IRCACHE_CASCADE_COUNT];
} kjb_frame_constants;   /* 1216 bytes */

/* world_renderer.rs:107-136 / inc/lights/packed.hlsl */
typedef struct kjb_triangle_light { float verts[3][3]; float radiance[3]; } kjb_triangle_light;

/* ------------------------------------------------------------------ scene (bindless set 1 + TLAS set 3)
 * `GpuMesh` (world_renderer.rs:43-54, inc/mesh.hlsl:10-18): byte offsets into the unified vertex buffer. */
typedef struct kjb_gpu_mesh {
    uint32_t vertex_core_offset, vertex_uv_offset, vertex_mat_offset, vertex_aux_offset,
             vertex_tangent_offset, mat_data_offset, index_offset;
} kjb_gpu_mesh;

/* inc/mesh.hlsl:52-61, kajiya-asset/src/mesh.rs:73-84 — 152 bytes */
typedef struct kjb_mesh_material {
    float    base_color_mult[4];
    uint32_t maps[4];              /* normal, spec, albedo, emissive (bindless texture ids) */
    float    roughness_mult;
    float    metalness_factor;
    float    emissive[3];
    uint32_t flags;
    float    map_transforms[24];
} kjb_mesh_material;

/* RayTracingInstanceDesc (world_renderer.rs:843-851): 3x4 row-major object-to-world + mesh index */
typedef struct kjb_instance {
    float    transform[12];        /* row-major 3x4, like VkTransformMatrixKHR */
    uint32_t mesh_index;           /* InstanceID() in gbuffer.rchit.hlsl:54 */
    float    emissive_multiplier;  /* instance_dynamic_parameters_dyn (frame_constants.hlsl:86-90) */
} kjb_instance;

/* A bindless texture: RGBA8 texels already decoded to linear floats-in-bytes semantics
 * (sRGB decode done at import, see DESIGN.md), full mip chain stored mip after mip. */
typedef struct kjb_texture_desc {
    const uint8_t *texels;         /* host pointer at upload time */
    uint32_t width, height, mip_count;
    uint32_t srgb;                 /* 1: texels are sRGB-encoded, decode on fetch */
} kjb_texture_desc;

typedef struct kjb_context kjb_context;

/* ------------------------------------------------------------------ context / memory */
int  kjb_abi_version(void);
/* device < 0: the emulator/oracle builds ignore it; the CUDA build requires a valid ordinal. */
int  kjb_create(int device, kjb_context **out_ctx);
void kjb_destroy(kjb_context *ctx);
int  kjb_sync(kjb_context *ctx);
const char *kjb_last_error(kjb_context *ctx);
/* which implementation is behind the pointer: "cuda-sm90a", "emu-cpu", "oracle-cpu" */
const char *kjb_backend_name(void);
/* number of device kernels launched through this context so far (0 for the oracle) */
uint64_t kjb_launch_count(kjb_context *ctx);
/* the cudaStream_t all passes are enqueued on (NULL for CPU backends) */
void *kjb_stream(kjb_context *ctx);

uint32_t kjb_format_texel_bytes(uint32_t format);
int  kjb_image_alloc(kjb_context *ctx, uint32_t width, uint32_t height, uint32_t layers, uint32_t format, kjb_image *out);
int  kjb_image_free(kjb_context *ctx, kjb_image *img);
int  kjb_image_clear(kjb_context *ctx, const kjb_image *img);
int  kjb_image_copy(kjb_context *ctx, const kjb_image *dst, const kjb_image *src);       /* same extent+format ("copy depth", reprojection.rs:42-48) */
int  kjb_image_fill_u8(kjb_context *ctx, const kjb_image *img, uint32_t byte_value);     /* memset of every byte (constant ssao input) */
int  kjb_image_upload(kjb_context *ctx, const kjb_image *dst, const void *host_src);     /* async on the stream */
int  kjb_image_download(kjb_context *ctx, const kjb_image *src, void *host_dst);         /* async on the stream */
int  kjb_buffer_alloc(kjb_context *ctx, uint64_t size_bytes, kjb_buffer *out);           /* zero-filled (temporal.rs:270-275) */
int  kjb_buffer_free(kjb_context *ctx, kjb_buffer *buf);
int  kjb_buffer_upload(kjb_context *ctx, const kjb_buffer *dst, uint64_t dst_offset, const void *host_src, uint64_t size);
int  kjb_buffer_download(kjb_context *ctx, const kjb_buffer *src, uint64_t src_offset, void *host_dst, uint64_t size);

/* device-side stopwatch: record() drops an event on the context's stream; elapsed_ms() synchronises on `to_slot` and
 * returns the time between two recorded slots (CUDA events; wall-clock on the CPU test builds). slots 0..1023. */
int  kjb_timer_record(kjb_context *ctx, uint32_t slot);
int  kjb_timer_elapsed_ms(kjb_context *ctx, uint32_t from_slot, uint32_t to_slot, float *out_ms);

/* ------------------------------------------------------------------ scene upload
 * kjb_scene_set_geometry replaces WorldRenderer::add_mesh's buffer uploads + BLAS builds
 * (world_renderer.rs:604-776): the unified `vertices` byte buffer, the `meshes` table and, per mesh,
 * the index count (the BLAS geometry, ray_tracing.rs:96-170: OPAQUE triangles, u32 indices,
 * float3 positions at vertex_core_offset with 16-byte stride). */
int  kjb_scene_set_geometry(kjb_context *ctx, const void *vertex_buffer, uint64_t vertex_buffer_bytes,
                            const kjb_gpu_mesh *meshes, const uint32_t *mesh_index_counts, uint32_t mesh_count);
int  kjb_scene_set_textures(kjb_context *ctx, const kjb_texture_desc *textures, uint32_t texture_count);
/* "rebuild tlas" (world_renderer.rs:865-911): instance transforms -> TLAS, every frame in the reference. */
int  kjb_rebuild_tlas(kjb_context *ctx, const kjb_instance *instances, uint32_t instance_count);
/* how "rebuild tlas" was served so far: [0] full rebuilds (instances or meshes changed), [1] device refits (only transforms changed: the per-frame case) */
int  kjb_tlas_stats(kjb_context *ctx, uint64_t out_rebuilds_refits[2]);
/* set 2 of every pass (renderer.rs:45-78): FrameConstants + triangle lights. */
int  kjb_set_frame_constants(kjb_context *ctx, const kjb_frame_constants *fc,
                             const kjb_triangle_light *lights, uint32_t light_count);
/* bindless LUT slots 0 and 1 (inc/bindless_textures.hlsl:8-12): BRDF FG LUT 64x64 RGBA16F, blue noise 256x256 RGBA8 */
int  kjb_set_luts(kjb_context *ctx, const kjb_image *brdf_fg_lut, const kjb_image *blue_noise_rgba8);

/* ray statistics accumulated by tracing passes since the last reset: [0] closest-hit rays, [1] any-hit (shadow) rays */
int  kjb_ray_counters(kjb_context *ctx, uint64_t out_counts[2], int reset);

/* ------------------------------------------------------------------ multi-GPU plumbing for tile-sharded frames (SURVEY §8e)
 * One process per GPU.  The only data-path collective of a frame is ONE all-gather of packed row strips (tile borders of the
 * temporal ReSTIR/TAA state + each rank's band of the full-res GI history).  The CUDA build performs it with NCCL on the
 * context's stream (ncclAllGather; libnccl is dlopen'ed by kjb_comm_init_nccl, the unique id is distributed by the caller,
 * e.g. with torch.distributed); CPU test builds and custom transports register a callback instead. */
typedef int (*kjb_allgather_fn)(void *user, const void *send, void *recv, uint64_t bytes_per_rank);
int  kjb_comm_nccl_unique_id(void *out_128_bytes);
int  kjb_comm_init_nccl(kjb_context *ctx, const void *unique_id_128_bytes, uint32_t rank, uint32_t nranks);
int  kjb_comm_set_callback(kjb_context *ctx, kjb_allgather_fn fn, void *user, uint32_t rank, uint32_t nranks);
int  kjb_comm_rank(kjb_context *ctx, uint32_t *rank, uint32_t *nranks);
int  kjb_allgather(kjb_context *ctx, const void *send, void *recv, uint64_t bytes_per_rank);
int  kjb_allgather_on(kjb_context *ctx, uint32_t queue, const void *send, void *recv, uint64_t bytes_per_rank);   /* same, enqueued on `queue`; in place when send == recv + rank * bytes_per_rank */     /* enqueued on the stream */
int  kjb_memcpy_d2d(kjb_context *ctx, void *dst, const void *src, uint64_t bytes);
/* Many device-to-device copies in ONE launch (the pack / unpack of the tile border exchange is dozens of small row strips). */
typedef struct kjb_copy_desc { void *dst; const void *src; uint64_t bytes; } kjb_copy_desc;
int  kjb_memcpy_d2d_batch(kjb_context *ctx, const kjb_copy_desc *copies, uint32_t count);
int  kjb_memcpy_d2d_batch_on(kjb_context *ctx, uint32_t queue, const kjb_copy_desc *copies, uint32_t count);                /* enqueued on the stream */

/* Tile-sharded frames (SURVEY §8e): restrict the FOLLOWING passes to rows [y0, y1) of their own output grid
 * (each rank of a multi-GPU frame computes its band plus the halo a pass's consumers need).  (0, 0) = whole image. */
/* Copy queues: besides the compute queue every pass is enqueued on, a context owns an upload and a download queue (CUDA streams on
 * the copy engines) so that host<->device transfers of neighbouring frames overlap the passes.  Events order work between queues:
 * record on one queue, make another queue (or the host) wait.  Host memory must be page-locked for the copies to be asynchronous.
 * (An interop host that shares memory with Vulkan never needs these; the frame driver's streaming mode does, kjb_world.h.) */
#define KJB_QUEUE_COMPUTE  0u
#define KJB_QUEUE_UPLOAD   1u
#define KJB_QUEUE_DOWNLOAD 2u
#define KJB_QUEUE_COMM     3u   /* collectives of tile-sharded frames, so that they overlap passes that do not depend on them */
#define KJB_QUEUE_ASYNC    4u   /* a second, high-priority PASS queue ("async compute"): see kjb_set_pass_queue */
#define KJB_MAX_EVENTS 64u
int  kjb_image_upload_on(kjb_context *ctx, uint32_t queue, const kjb_image *dst, const void *host_src);
int  kjb_image_download_on(kjb_context *ctx, uint32_t queue, const kjb_image *src, void *host_dst);
/* the same for rows [row0, row0 + row_count) only; host pointers address the WHOLE image (tile-sharded frames move their band only) */
int  kjb_image_upload_rows_on(kjb_context *ctx, uint32_t queue, const kjb_image *dst, const void *host_src, uint32_t row0, uint32_t row_count);
int  kjb_image_download_rows_on(kjb_context *ctx, uint32_t queue, const kjb_image *src, void *host_dst, uint32_t row0, uint32_t row_count);
int  kjb_event_record(kjb_context *ctx, uint32_t event, uint32_t queue);
int  kjb_queue_wait_event(kjb_context *ctx, uint32_t queue, uint32_t event);   /* no-op if the event was never recorded */
int  kjb_event_synchronize(kjb_context *ctx, uint32_t event);                   /* host wait; no-op if never recorded */
/* Options (off unless set).
 * KJB_OPTION_HALF_RES_POSITION_CACHE: "restir spatial" and "restir resolve" unproject the same half-res pixels over and over (16 and 8
 * times per pixel); with this option the library keeps two scratch images of world positions — one from `half_depth_tex`, one from the
 * depth channel of `temporal_reservoir_packed_tex` — refreshes them when their sources change and lets the two passes load instead of
 * recompute (same values bit for bit).  "extract half-res inputs" and "restir temporal" write them as a by-product when they cover the whole
 * image; otherwise a small kernel refreshes them on demand.  The library sees every change made through its own entry points ("extract half depth",
 * "restir temporal", kjb_image_upload/clear/copy/fill, kjb_set_frame_constants); a host that writes those two images by other means
 * (interop) must leave the option off. */
#define KJB_OPTION_HALF_RES_POSITION_CACHE 1u
/* KJB_OPTION_ORDERED_CACHE_SCHEDULE (default 1 in the CUDA build, 0 in the CPU emulator): how the parallel kernels that touch the irradiance
 * cache resolve their conflicts.  1 = decisions that do not depend on the order the threads run in, so the same inputs give the same
 * frames on every run (claimed cells get entries at the next cache chain, votes go to the smallest hash; kjb_ircache.cuh).  0 = the
 * reference's atomics as they land (scheduling dependent on the GPU; in launch order, like the oracle, in the emulator).  Set it before the
 * first frame with the cache: it cannot change once the ordered schedule holds pending claims.
 * Tile-sharded frames exchange the cache's pending requests exactly on schedule 1 (kjb_pass_ircache_export_pending), so every replica stays
 * bit-identical to the single-GPU cache.  One buffer is left out of that equality: `reposition_proposal_count_buf`.  On schedule 1 no decision
 * reads it (ageing resets it), and the replicas carry the largest count of any rank, which is non-zero exactly where the single cache's is.
 * (include/kjb_ircache_share.h) */
#define KJB_OPTION_ORDERED_CACHE_SCHEDULE 2u
int  kjb_set_option(kjb_context *ctx, uint32_t option, uint32_t value);
/* CUDA Graph replay of a frame's passes (the reference records one command buffer per frame, graph.rs:865-867; ~40 kernel launches here):
 * every pass enqueued on the compute queue between the two calls is RECORDED instead of launched; kjb_graph_end turns the recording into
 * an executable graph on first use, afterwards only updates the kernel-node parameters of the instance it keeps (same pass list => same
 * topology), and submits the whole frame with ONE launch.  Calls that touch other queues or wait on the host must stay outside the pair. */
int  kjb_graph_begin(kjb_context *ctx);
int  kjb_graph_end(kjb_context *ctx);
/* A frame driver that splits its frame into several recordings (because it orders other queues against the middle of the frame) keeps one
 * instance per piece: the slot (0..3) selected here is the instance the following kjb_graph_begin / kjb_graph_end pairs update and launch. */
int  kjb_graph_select(kjb_context *ctx, uint32_t slot);
/* Async compute: the queue every FOLLOWING kjb_pass_* (and kjb_image_copy / clear helpers a pass driver issues) is enqueued on —
 * KJB_QUEUE_COMPUTE (default) or KJB_QUEUE_ASYNC.  The two queues run concurrently; the caller orders them with kjb_event_record /
 * kjb_queue_wait_event exactly like the copy queues.  Meant for small latency-bound pass chains that share no resource with what the
 * compute queue is doing (the frame driver runs the irradiance-cache maintenance + cache rays of frame N+1 under the reflection filters and
 * TAA of frame N, kjb_world.h).  Passes on the async queue are never part of a graph recording.  kjb_async_passes_supported: 1 when the two
 * queues really overlap (CUDA build, serialised debugging off), 0 for the single-queue backends (CPU oracle, emulator, recorder). */
int  kjb_set_pass_queue(kjb_context *ctx, uint32_t queue);
int  kjb_async_passes_supported(kjb_context *ctx);
int  kjb_graph_stats(kjb_context *ctx, uint64_t out_launches_instantiations[2]);
int  kjb_set_scissor(kjb_context *ctx, uint32_t y0, uint32_t y1);
/* Oracle schedule: while on, every pass that touches the irradiance cache runs on ONE device thread in the launch order of its
 * parallel kernel, with the reference's atomics — the oracle's schedule. Orders of magnitude slower; for bit-exact parity tests.
 * Like KJB_OPTION_ORDERED_CACHE_SCHEDULE, switch it on before the first frame with the cache. */
int  kjb_set_debug_serial(kjb_context *ctx, uint32_t on);

/* ------------------------------------------------------------------ input producers (SURVEY §8f N1/N2, needed to feed the path) */
typedef struct kjb_raster_gbuffer_args {   /* replaces "raster simple" (raster_simple_ps.hlsl:39-140) by primary-ray casting */
    kjb_image geometric_normal_out;        /* A2R10G10B10_UNORM, view-space normal *0.5+0.5 */
    kjb_image gbuffer_out;                 /* RGBA32_FLOAT (packed GbufferData) */
    kjb_image depth_out;                   /* R32_FLOAT reverse-Z, 0 = sky */
    kjb_image velocity_out;                /* RGBA16_FLOAT view-space motion: prev_view(prev_world_pos) - view(world_pos), raster_simple_vs.hlsl */
    /* last frame's instance list (HOST pointer, same order as the list given to kjb_rebuild_tlas) for the motion of moving objects;
     * NULL / 0 = objects are static (camera motion only) */
    const kjb_instance *prev_instances; uint32_t prev_instance_count;
} kjb_raster_gbuffer_args;
int kjb_pass_raster_gbuffer(kjb_context *ctx, const kjb_raster_gbuffer_args *a);

typedef struct kjb_reprojection_map_args { /* calculate_reprojection_map.hlsl:9-16 */
    kjb_image depth_tex, geometric_normal_tex, prev_depth_tex, velocity_tex, output_tex;
    float output_tex_size[4];
} kjb_reprojection_map_args;
int kjb_pass_reprojection_map(kjb_context *ctx, const kjb_reprojection_map_args *a);

typedef struct kjb_sky_cube_args { kjb_image output_tex; } kjb_sky_cube_args;            /* sky/comp_cube.hlsl */
int kjb_pass_sky_cube(kjb_context *ctx, const kjb_sky_cube_args *a);
typedef struct kjb_convolve_sky_args { kjb_image input_tex, output_tex; uint32_t face_width; } kjb_convolve_sky_args; /* convolve_cube.hlsl */
int kjb_pass_convolve_sky(kjb_context *ctx, const kjb_convolve_sky_args *a);
typedef struct kjb_brdf_fg_lut_args { kjb_image output_tex; } kjb_brdf_fg_lut_args;       /* lut/brdf_fg.hlsl */
int kjb_pass_brdf_fg_lut(kjb_context *ctx, const kjb_brdf_fg_lut_args *a);

/* ------------------------------------------------------------------ half-res extracts (renderers/half_res.rs, rtdgi.rs:185-202) */
typedef struct kjb_extract_half_res_args { kjb_image input_tex, output_tex; } kjb_extract_half_res_args;
int kjb_pass_extract_half_res_depth(kjb_context *ctx, const kjb_extract_half_res_args *a);        /* "extract half depth" */
int kjb_pass_extract_half_res_view_normal(kjb_context *ctx, const kjb_extract_half_res_args *a);  /* "extract view normal/2" */
int kjb_pass_extract_half_res_ssao(kjb_context *ctx, const kjb_extract_half_res_args *a);         /* "extract ssao/2" */
/* The three extracts above in ONE launch ("extract half-res inputs"): they read the same half-res pixel of three full-res images and each
 * one alone is launch-latency bound (3 x ~8 us -> ~9 us at 1080p).  Same outputs, texel for texel.  ssao_tex / half_ssao_out may be
 * null images (data == NULL): then only depth and view normal are produced (the SSAO guide is itself computed from those two). */
typedef struct kjb_extract_half_res_fused_args {
    kjb_image gbuffer_tex, depth_tex, ssao_tex;
    kjb_image half_view_normal_out, half_depth_out, half_ssao_out;
} kjb_extract_half_res_fused_args;
int kjb_pass_extract_half_res_fused(kjb_context *ctx, const kjb_extract_half_res_fused_args *a);

/* ------------------------------------------------------------------ ssao (renderers/ssgi.rs; shaders under assets/shaders/ssgi/, USE_AO_ONLY)
 * SURVEY §8f N3: the screen-space occlusion that guides the rtdgi kernels (half_ssao / ssao inputs of D7, D9, D11). */
typedef struct kjb_ssao_args {                        /* "ssao", ssgi.hlsl:10-21, ssgi.rs:61-73 */
    kjb_image gbuffer_tex, half_depth_tex, half_view_normal_tex, prev_radiance_tex, reprojection_tex;   /* prev_radiance: unused with USE_AO_ONLY, may be null */
    kjb_image output_tex;                             /* R16_FLOAT half-res */
    float input_tex_size[4], output_tex_size[4];
} kjb_ssao_args;
int kjb_pass_ssao(kjb_context *ctx, const kjb_ssao_args *a);
typedef struct kjb_ssao_spatial_args { kjb_image ssgi_tex, depth_tex, normal_tex, output_tex; } kjb_ssao_spatial_args;      /* "ssao spatial", spatial_filter.hlsl:4-7 */
int kjb_pass_ssao_spatial(kjb_context *ctx, const kjb_ssao_spatial_args *a);
typedef struct kjb_ssao_upsample_args { kjb_image ssgi_tex, depth_tex, gbuffer_tex, output_tex; } kjb_ssao_upsample_args;   /* "ssao upsample", upsample.hlsl:5-8 */
int kjb_pass_ssao_upsample(kjb_context *ctx, const kjb_ssao_upsample_args *a);
typedef struct kjb_ssao_temporal_args {               /* "ssao temporal", temporal_filter.hlsl:3-9 */
    kjb_image input_tex, history_tex, reprojection_tex, final_output_tex, history_output_tex;        /* final: R8_UNORM; history: R16_FLOAT */
    float output_tex_size[4];
} kjb_ssao_temporal_args;
int kjb_pass_ssao_temporal(kjb_context *ctx, const kjb_ssao_temporal_args *a);

/* ------------------------------------------------------------------ ircache binding block (ircache/bindings.hlsl, ircache.rs:59-78).
 * NULL `meta_buf.data` = irradiance cache not bound: lookups return 0 and allocate nothing. */
typedef struct kjb_ircache_bindings {
    /* IrcacheRenderState::bind_mut call order = DEFINE_IRCACHE_BINDINGS(b0..b8) (ircache.rs:67-75, ircache/bindings.hlsl:6-15).  The
     * per-entry reservoirs (`aux`) are NOT part of the block: only the cache's own passes bind them (IRCACHE_LOOKUP_PRECISE). */
    kjb_buffer meta_buf, pool_buf, reposition_proposal_buf, reposition_proposal_count_buf, grid_meta_buf, entry_cell_buf,
               spatial_buf, irradiance_buf, life_buf;
} kjb_ircache_bindings;

/* ------------------------------------------------------------------ ircache (renderers/ircache.rs, shaders under assets/shaders/ircache/)
 * Buffer sizes: ircache.rs:172-231 (MAX_ENTRIES 65536, 12 cascades x 32^3 cells).  Indirect dispatches of the reference
 * (dispatch_indirect / trace_rays_indirect) become fixed-size launches that early-out on the counters in meta_buf, exactly like
 * the reference's own fixed-size validate/trace dispatches (ircache.rs:438-447,471-476). */
#define KJB_IRCACHE_MAX_ENTRIES 65536u
#define KJB_IRCACHE_GRID_CELLS (32u * 32u * 32u * 12u)
typedef struct kjb_ircache_clear_pool_args { kjb_buffer pool_buf, life_buf; } kjb_ircache_clear_pool_args;            /* "clear ircache pool" */
int kjb_pass_ircache_clear_pool(kjb_context *ctx, const kjb_ircache_clear_pool_args *a);
typedef struct kjb_ircache_scroll_cascades_args {     /* "scroll cascades", scroll_cascades.hlsl:4-10 */
    kjb_buffer grid_meta_buf, grid_meta_buf2, entry_cell_buf, irradiance_buf, life_buf, pool_buf, meta_buf;
} kjb_ircache_scroll_cascades_args;
int kjb_pass_ircache_scroll_cascades(kjb_context *ctx, const kjb_ircache_scroll_cascades_args *a);
typedef struct kjb_ircache_dispatch_args_args { kjb_buffer meta_buf, dispatch_args; } kjb_ircache_dispatch_args_args;
int kjb_pass_ircache_prepare_age_dispatch_args(kjb_context *ctx, const kjb_ircache_dispatch_args_args *a);    /* "_ircache dispatch args" (prepare_age_dispatch_args.hlsl) */
int kjb_pass_ircache_prepare_trace_dispatch_args(kjb_context *ctx, const kjb_ircache_dispatch_args_args *a);  /* "_ircache dispatch args" (prepare_trace_dispatch_args.hlsl) */
typedef struct kjb_ircache_age_args {                 /* "age ircache entries", age_ircache_entries.hlsl:5-14 */
    kjb_buffer meta_buf, grid_meta_buf, entry_cell_buf, life_buf, pool_buf, spatial_buf, reposition_proposal_buf,
               reposition_proposal_count_buf, irradiance_buf, entry_occupancy_buf;
} kjb_ircache_age_args;
int kjb_pass_ircache_age_entries(kjb_context *ctx, const kjb_ircache_age_args *a);
typedef struct kjb_prefix_scan_args { kjb_buffer inout_buf; uint32_t element_count; } kjb_prefix_scan_args;   /* "_prefix scan 1/2/merge" (prefix_scan.rs:10-39): inclusive u32 scan */
int kjb_pass_inclusive_prefix_scan_u32(kjb_context *ctx, const kjb_prefix_scan_args *a);
typedef struct kjb_ircache_compact_args { kjb_buffer meta_buf, life_buf, entry_occupancy_buf, entry_indirection_buf; } kjb_ircache_compact_args;   /* "ircache compact" */
int kjb_pass_ircache_compact(kjb_context *ctx, const kjb_ircache_compact_args *a);
typedef struct kjb_ircache_reset_args { kjb_buffer life_buf, meta_buf, irradiance_buf, aux_buf, entry_indirection_buf; } kjb_ircache_reset_args;   /* "ircache reset" */
int kjb_pass_ircache_reset(kjb_context *ctx, const kjb_ircache_reset_args *a);
typedef struct kjb_ircache_trace_access_args {        /* "ircache trace access", trace_accessibility.rgen.hlsl:14-19 */
    kjb_buffer spatial_buf, life_buf, reposition_proposal_buf, meta_buf, aux_buf, entry_indirection_buf;
} kjb_ircache_trace_access_args;
int kjb_pass_ircache_trace_access(kjb_context *ctx, const kjb_ircache_trace_access_args *a);
typedef struct kjb_ircache_trace_args {               /* "ircache validate" / "ircache trace", trace_irradiance.rgen.hlsl:21-33 */
    kjb_buffer spatial_buf; kjb_image sky_cube_tex;
    kjb_buffer grid_meta_buf, life_buf, reposition_proposal_buf, reposition_proposal_count_buf, meta_buf, aux_buf, pool_buf,
               entry_indirection_buf, entry_cell_buf;   /* bindings 0-11 minus the (disabled) wrc block; IRCACHE_LOOKUP_PRECISE reads `aux`, never the SH */
} kjb_ircache_trace_args;
int kjb_pass_ircache_validate(kjb_context *ctx, const kjb_ircache_trace_args *a);
int kjb_pass_ircache_trace(kjb_context *ctx, const kjb_ircache_trace_args *a);
typedef struct kjb_ircache_sum_args { kjb_buffer life_buf, meta_buf, irradiance_buf, aux_buf, entry_indirection_buf; } kjb_ircache_sum_args;   /* "ircache sum" */
int kjb_pass_ircache_sum(kjb_context *ctx, const kjb_ircache_sum_args *a);
/* Multi-GPU (tile-sharded frames, SURVEY §8e): the irradiance cache is ONE global structure fed by every ray of the frame; a rank only traces the rays of
 * its band.  Every rank keeps a replica and, after the frame's last cache user, the ranks exchange what their rays asked of the cache: one 32-byte record per
 * live entry — (cell, life, this frame's vote count, the vote that won locally).  Merging a record keeps the cell alive (life = min), allocates it where the
 * local rays never went, and draws the surviving reposition vote with probability count_remote / (count_local + count_remote), i.e. the uniform vote over
 * the union of all ranks' rays (lookup.hlsl:268-309, IRCACHE_USE_UNIFORM_VOTING).  After the merge every replica holds the same set of live cells with the
 * positions the whole frame voted for, which is what the single-GPU cache holds.  Not a reference pass (kajiya is single-GPU). */
#define KJB_IRCACHE_SHARE_RECORD_BYTES 32u
#define KJB_IRCACHE_SHARE_BLOCK_BYTES(max_records) (16u + (max_records) * KJB_IRCACHE_SHARE_RECORD_BYTES)   /* header {count, 0, 0, 0} + records */
typedef struct kjb_ircache_share_args {
    kjb_ircache_bindings ircache;
    kjb_buffer block;            /* export: this rank's block (written).  merge: ONE other rank's block (read) */
    uint32_t max_records;        /* records beyond this stay local (the cache then degrades towards independent replicas) */
    uint32_t seed;               /* merge: frame index * rank count + source rank — decorrelates the vote draws */
} kjb_ircache_share_args;
int kjb_pass_ircache_export_requests(kjb_context *ctx, const kjb_ircache_share_args *a);
int kjb_pass_ircache_merge_requests(kjb_context *ctx, const kjb_ircache_share_args *a);
/* The exact exchange for the ordered schedule: include/kjb_ircache_share.h. */


/* ------------------------------------------------------------------ rtdgi (renderers/rtdgi.rs) */
typedef struct kjb_rtdgi_reproject_args {            /* "rtdgi reproject", fullres_reproject.hlsl:10-15, rtdgi.rs:156-164 */
    kjb_image input_tex, reprojection_tex, output_tex;
    float output_tex_size[4];
} kjb_rtdgi_reproject_args;
int kjb_pass_rtdgi_reproject(kjb_context *ctx, const kjb_rtdgi_reproject_args *a);

typedef struct kjb_rtdgi_validate_args {             /* "rtdgi validate", diffuse_validate.rgen.hlsl:20-39, rtdgi.rs:293-316 */
    kjb_image half_view_normal_tex, depth_tex, reprojected_gi_tex;
    kjb_image reservoir_tex;                          /* read-write: history reservoirs */
    kjb_image reservoir_ray_history_tex, reprojection_tex;
    kjb_ircache_bindings ircache;
    kjb_image sky_cube_tex;
    kjb_image irradiance_history_tex;                 /* read-write */
    kjb_image ray_orig_history_tex;
    kjb_image rt_history_invalidity_out_tex;
    float gbuffer_tex_size[4];
} kjb_rtdgi_validate_args;
int kjb_pass_rtdgi_validate(kjb_context *ctx, const kjb_rtdgi_validate_args *a);

typedef struct kjb_rtdgi_trace_args {                /* "rtdgi trace", trace_diffuse.rgen.hlsl:23-41, rtdgi.rs:321-345 */
    kjb_image half_view_normal_tex, depth_tex, reprojected_gi_tex, reprojection_tex;
    kjb_ircache_bindings ircache;
    kjb_image sky_cube_tex, ray_orig_history_tex;
    kjb_image candidate_irradiance_out_tex, candidate_normal_out_tex, candidate_hit_out_tex;
    kjb_image rt_history_invalidity_in_tex, rt_history_invalidity_out_tex;
    float gbuffer_tex_size[4];
} kjb_rtdgi_trace_args;
int kjb_pass_rtdgi_trace(kjb_context *ctx, const kjb_rtdgi_trace_args *a);

typedef struct kjb_rtdgi_validity_integrate_args {   /* "validity integrate", temporal_validity_integrate.hlsl:10-19 */
    kjb_image input_tex, history_tex, reprojection_tex, half_view_normal_tex, half_depth_tex, output_tex;
    float gbuffer_tex_size[4], output_tex_size[4];
} kjb_rtdgi_validity_integrate_args;
int kjb_pass_rtdgi_validity_integrate(kjb_context *ctx, const kjb_rtdgi_validity_integrate_args *a);

typedef struct kjb_rtdgi_restir_temporal_args {      /* "restir temporal", restir_temporal.hlsl:18-40, rtdgi.rs:363-389 */
    kjb_image half_view_normal_tex, depth_tex, candidate_radiance_tex, candidate_normal_tex, candidate_hit_tex,
              radiance_history_tex, ray_orig_history_tex, ray_history_tex, reservoir_history_tex, reprojection_tex,
              hit_normal_history_tex, candidate_history_tex, rt_invalidity_tex;
    kjb_image radiance_out_tex, ray_orig_output_tex, ray_output_tex, hit_normal_output_tex, reservoir_out_tex,
              candidate_out_tex, temporal_reservoir_packed_tex;
    float gbuffer_tex_size[4];
} kjb_rtdgi_restir_temporal_args;
int kjb_pass_rtdgi_restir_temporal(kjb_context *ctx, const kjb_rtdgi_restir_temporal_args *a);

typedef struct kjb_rtdgi_restir_spatial_args {       /* "restir spatial", restir_spatial.hlsl:15-32, rtdgi.rs:428-476 */
    kjb_image reservoir_input_tex, bounced_radiance_input_tex, half_view_normal_tex, half_depth_tex, depth_tex,
              half_ssao_tex, temporal_reservoir_packed_tex, reprojected_gi_tex;
    kjb_image reservoir_output_tex, bounced_radiance_output_tex;
    float gbuffer_tex_size[4], output_tex_size[4];
    uint32_t spatial_reuse_pass_idx, perform_occlusion_raymarch, occlusion_raymarch_importance_only;
} kjb_rtdgi_restir_spatial_args;
int kjb_pass_rtdgi_restir_spatial(kjb_context *ctx, const kjb_rtdgi_restir_spatial_args *a);

typedef struct kjb_rtdgi_restir_check_args {         /* "restir check" (optional: RtdgiRenderer::use_raytraced_reservoir_visibility), restir_check.rgen.hlsl:10-15, rtdgi.rs:478-494 */
    kjb_image half_depth_tex, temporal_reservoir_packed_tex, reservoir_input_tex;   /* reservoir_input_tex is read-write */
    float gbuffer_tex_size[4];
} kjb_rtdgi_restir_check_args;
int kjb_pass_rtdgi_restir_check(kjb_context *ctx, const kjb_rtdgi_restir_check_args *a);

typedef struct kjb_rtdgi_restir_resolve_args {       /* "restir resolve", restir_resolve.hlsl:16-31, rtdgi.rs:502-523 */
    kjb_image radiance_tex, reservoir_input_tex, gbuffer_tex, depth_tex, half_view_normal_tex, half_depth_tex,
              ssao_tex, candidate_radiance_tex, candidate_hit_tex, temporal_reservoir_packed_tex,
              bounced_radiance_input_tex;
    kjb_image irradiance_output_tex;
    float gbuffer_tex_size[4], output_tex_size[4];
} kjb_rtdgi_restir_resolve_args;
int kjb_pass_rtdgi_restir_resolve(kjb_context *ctx, const kjb_rtdgi_restir_resolve_args *a);

typedef struct kjb_rtdgi_temporal_args {             /* "rtdgi temporal", temporal_filter.hlsl:23-35, rtdgi.rs:96-112 */
    kjb_image input_tex, history_tex, variance_history_tex, reprojection_tex, rt_history_invalidity_tex;
    kjb_image output_tex, history_output_tex, variance_history_output_tex;
    float output_tex_size[4], gbuffer_tex_size[4];
} kjb_rtdgi_temporal_args;
int kjb_pass_rtdgi_temporal(kjb_context *ctx, const kjb_rtdgi_temporal_args *a);

typedef struct kjb_rtdgi_spatial_args {              /* "rtdgi spatial", spatial_filter.hlsl:10-17, rtdgi.rs:127-138 */
    kjb_image input_tex, depth_tex, ssao_tex, geometric_normal_tex, output_tex;
    float output_tex_size[4];
} kjb_rtdgi_spatial_args;
int kjb_pass_rtdgi_spatial(kjb_context *ctx, const kjb_rtdgi_spatial_args *a);

/* ------------------------------------------------------------------ rtr (renderers/rtr.rs; shaders under assets/shaders/rtr/)
 * Ray-traced specular reflections.  Half-res candidates go into the rtdgi candidate images (rtr.rs:105-109): radiance RGBA16F,
 * hit RGBA16F, normal RGBA8_SNORM.  Temporal images are RGBA16F (temporal_tex_desc, rtr.rs:87-90) unless stated. */
typedef struct kjb_rtr_trace_args {                  /* "reflection trace", reflection.rgen.hlsl:19-36, rtr.rs:132-156 */
    kjb_image gbuffer_tex, depth_tex;
    /* blue-noise-sampler spp64 tables (rtr.rs:66-68; crate blue-noise-sampler, not part of kajiya's tree): i32[128*128*8],
     * i32[128*128*8], i32[256*256].  All three NULL = the shader's own `blue_noise_for_pixel` alternative (reflection.rgen.hlsl:98-100). */
    kjb_buffer ranking_tile_buf, scambling_tile_buf, sobol_buf;
    kjb_image rtdgi_tex, sky_cube_tex;
    kjb_ircache_bindings ircache;
    kjb_image out0_tex, out1_tex, out2_tex, rng_out_tex;   /* rng: R32_UINT half-res */
    float gbuffer_tex_size[4];
    uint32_t reuse_rtdgi_rays;
} kjb_rtr_trace_args;
int kjb_pass_rtr_trace(kjb_context *ctx, const kjb_rtr_trace_args *a);

typedef struct kjb_rtr_validate_args {               /* "reflection validate", reflection_validate.rgen.hlsl:20-35, rtr.rs:208-231 */
    kjb_image gbuffer_tex, depth_tex, rtdgi_tex, sky_cube_tex, refl_restir_invalidity_tex;   /* invalidity: R8_UNORM half-res */
    kjb_ircache_bindings ircache;
    kjb_image ray_orig_history_tex, ray_history_tex, rng_history_tex, irradiance_history_tex, reservoir_history_tex;   /* ray_orig RGBA32F; reservoir RG32_UINT */
    float gbuffer_tex_size[4];
} kjb_rtr_validate_args;
int kjb_pass_rtr_validate(kjb_context *ctx, const kjb_rtr_validate_args *a);

typedef struct kjb_rtr_restir_temporal_args {        /* "rtr restir temporal", rtr_restir_temporal.hlsl:43-65, rtr.rs:234-261 */
    kjb_image gbuffer_tex, half_view_normal_tex, depth_tex, candidate0_tex, candidate1_tex, candidate2_tex, irradiance_history_tex, ray_orig_history_tex,
              ray_history_tex, rng_history_tex, reservoir_history_tex, reprojection_tex, hit_normal_history_tex;
    kjb_image irradiance_out_tex, ray_orig_output_tex, ray_output_tex, rng_output_tex, hit_normal_output_tex, reservoir_out_tex;
    float gbuffer_tex_size[4];
} kjb_rtr_restir_temporal_args;
int kjb_pass_rtr_restir_temporal(kjb_context *ctx, const kjb_rtr_restir_temporal_args *a);

#define KJB_SPATIAL_RESOLVE_OFFSET_COUNT (16 * 4 * 8)
typedef struct kjb_rtr_resolve_args {                /* "reflection resolve", resolve.hlsl:16-36, rtr.rs:290-316 */
    kjb_image gbuffer_tex, depth_tex, hit0_tex, hit1_tex, hit2_tex, history_tex, reprojection_tex, half_view_normal_tex, half_depth_tex, ray_len_history_tex,
              restir_irradiance_tex, restir_ray_tex, restir_reservoir_tex, restir_ray_orig_tex, restir_hit_normal_tex;
    kjb_image output_tex, ray_len_output_tex;        /* R11G11B10_UFLOAT full-res; RG16F full-res */
    float output_tex_size[4];
    const int32_t *spatial_resolve_offsets;          /* int4[512] pushed by the host (rtr.rs:402-915); not read by the shader's active path, may be NULL */
} kjb_rtr_resolve_args;
int kjb_pass_rtr_resolve(kjb_context *ctx, const kjb_rtr_resolve_args *a);

typedef struct kjb_rtr_temporal_args {               /* "reflection temporal", temporal_filter.hlsl:23-33, rtr.rs:372-385 */
    kjb_image input_tex, history_tex, depth_tex, ray_len_tex, reprojection_tex, refl_restir_invalidity_tex, gbuffer_tex, output_tex;
    float output_tex_size[4];
} kjb_rtr_temporal_args;
int kjb_pass_rtr_temporal(kjb_context *ctx, const kjb_rtr_temporal_args *a);

typedef struct kjb_rtr_cleanup_args {                /* "reflection cleanup", spatial_cleanup.hlsl:9-15, rtr.rs:387-396 */
    kjb_image input_tex, depth_tex, geometric_normal_tex, output_tex;
    const int32_t *spatial_resolve_offsets;          /* int4[512] HOST pointer (rtr.rs:402-915); copied inside the call */
} kjb_rtr_cleanup_args;
int kjb_pass_rtr_cleanup(kjb_context *ctx, const kjb_rtr_cleanup_args *a);

/* ------------------------------------------------------------------ lighting composite (SURVEY §8f N4)
 * "trace shadow mask" (renderers/shadows.rs:10-35, rt/trace_sun_shadow_mask.rgen.hlsl) and "light gbuffer" (renderers/deferred.rs:8-43,
 * light_gbuffer.hlsl): direct sun + emissive + rtdgi * albedo + rtr * FG; the sky with the sun disk where depth == 0. */
typedef struct kjb_trace_sun_shadow_mask_args { kjb_image depth_tex, geometric_normal_tex, output_tex; } kjb_trace_sun_shadow_mask_args;   /* output R8_UNORM */
int kjb_pass_trace_sun_shadow_mask(kjb_context *ctx, const kjb_trace_sun_shadow_mask_args *a);
/* ------------------------------------------------------------------ shadow denoiser (renderers/shadow_denoise.rs:19-149; shaders under
 * assets/shaders/shadow_denoise/, the FidelityFX shadow denoiser as kajiya adapted it).  Runs between "trace shadow mask" and "light gbuffer"
 * whenever the sun is an area light (WorldRenderer::sun_size_multiplier > 0, world_render_passes.rs:124-137). */
typedef struct kjb_shadow_bitpack_args {              /* "shadow bitpack", bitpack_shadow_mask.hlsl:1-30 */
    kjb_image input_tex;                              /* R8_UNORM ray-traced mask */
    kjb_image output_tex;                             /* R32_UINT, one texel per 8x4 pixel tile: bit (y%4)*8 + x%8 = lit */
    float input_tex_size[4]; uint32_t bitpacked_shadow_mask_extent[2];
} kjb_shadow_bitpack_args;
int kjb_pass_shadow_bitpack(kjb_context *ctx, const kjb_shadow_bitpack_args *a);
typedef struct kjb_shadow_temporal_args {             /* "shadow temporal", megakernel.hlsl:6-150 + ffx_denoiser_shadows_tileclassification.hlsl */
    kjb_image shadow_mask_tex, bitpacked_shadow_mask_tex, prev_moments_tex /* RGBA16F */, prev_accum_tex /* RG16F */, reprojection_tex;
    kjb_image output_moments_tex /* RGBA16F */, temporal_output_tex /* RG16F: shadow, variance */, meta_output_tex /* R32_UINT per 8x8 group */;
    float input_tex_size[4]; uint32_t bitpacked_shadow_mask_extent[2];
} kjb_shadow_temporal_args;
int kjb_pass_shadow_temporal(kjb_context *ctx, const kjb_shadow_temporal_args *a);
typedef struct kjb_shadow_spatial_args {              /* "shadow spatial", spatial_filter.hlsl:3-78 + ffx_denoiser_shadows_filter.hlsl; run with step 1, 2, 4 */
    kjb_image input_tex /* RG16F */, meta_tex, geometric_normal_tex, depth_tex, output_tex /* RG16F */;
    float input_tex_size[4]; uint32_t bitpacked_shadow_mask_extent[2]; uint32_t step_size;
} kjb_shadow_spatial_args;
int kjb_pass_shadow_spatial(kjb_context *ctx, const kjb_shadow_spatial_args *a);

/* ------------------------------------------------------------------ LightingRenderer::render_specular (renderers/lighting.rs:23-87): specular light of the
 * emissive-triangle lights, rendered INTO the resolved reflections before their temporal filter (world_render_passes.rs:190-201); only when
 * the scene has triangle lights (kjb_mesh_desc.use_lights). */
typedef struct kjb_sample_lights_args {               /* "sample lights", lighting/sample_lights.rgen.hlsl:10-63 */
    kjb_image depth_tex;
    kjb_image out0_tex, out1_tex, out2_tex;           /* half-res: RGBA16F radiance (w = 1 for a valid sample), RGBA32F view-space hit + area pdf, RGBA8_SNORM light normal */
    float gbuffer_tex_size[4];
} kjb_sample_lights_args;
int kjb_pass_sample_lights(kjb_context *ctx, const kjb_sample_lights_args *a);
typedef struct kjb_spatial_reuse_lights_args {        /* "spatial reuse lights", lighting/spatial_reuse_lights.hlsl:11-168 */
    kjb_image gbuffer_tex, depth_tex, hit0_tex, hit1_tex, hit2_tex, half_view_normal_tex, half_depth_tex;
    kjb_image output_tex;                             /* R11G11B10 resolved reflections: read, the light's specular is added, written back */
    float output_tex_size[4];
    const int32_t *spatial_resolve_offsets;           /* int4[512] HOST pointer (rtr.rs:402-915); copied inside the call */
} kjb_spatial_reuse_lights_args;
int kjb_pass_spatial_reuse_lights(kjb_context *ctx, const kjb_spatial_reuse_lights_args *a);

typedef struct kjb_light_gbuffer_args {              /* light_gbuffer.hlsl:27-44 */
    kjb_image gbuffer_tex, depth_tex, shadow_mask_tex, rtr_tex, rtdgi_tex;   /* shadow_mask_tex: R8_UNORM raw mask or RG16F denoiser output (.x); rtr_tex: R11G11B10 resolved reflections (a zero image when rtr is off) */
    kjb_ircache_bindings ircache;                     /* only read by debug_shading_mode 5, which is not supported */
    kjb_image temporal_output_tex, output_tex;        /* RGBA16F, RGBA16F */
    kjb_image unconvolved_sky_cube_tex, sky_cube_tex;
    float output_tex_size[4];
    uint32_t debug_shading_mode;                      /* 0 default, 2 diffuse GI, 3 reflections, 4 "RTX off"; 1 and 5 are refused */
    uint32_t debug_show_wrc;                          /* must be 0 (wrc is disabled upstream) */
} kjb_light_gbuffer_args;
int kjb_pass_light_gbuffer(kjb_context *ctx, const kjb_light_gbuffer_args *a);

/* ------------------------------------------------------------------ taa (renderers/taa.rs:41-185; shaders under assets/shaders/taa/) */
typedef struct kjb_taa_reproject_args {              /* "reproject taa", reproject_history.hlsl:8-16, taa.rs:66-79 */
    kjb_image history_tex, reprojection_tex, depth_tex, output_tex, closest_velocity_output;
    float input_tex_size[4], output_tex_size[4];
} kjb_taa_reproject_args;
int kjb_pass_taa_reproject(kjb_context *ctx, const kjb_taa_reproject_args *a);

typedef struct kjb_taa_filter_input_args {           /* "taa filter input", filter_input.hlsl:9-12, taa.rs:98-106 */
    kjb_image input_tex, depth_tex, output_tex, dev_output_tex;
} kjb_taa_filter_input_args;
int kjb_pass_taa_filter_input(kjb_context *ctx, const kjb_taa_filter_input_args *a);

typedef struct kjb_taa_filter_history_args {         /* "taa filter history", filter_history.hlsl:8-13, taa.rs:112-122 */
    kjb_image input_tex, output_tex;
    float input_tex_size[4], output_tex_size[4];      /* = (reprojected history extent, taa input extent), as the host pushes them */
} kjb_taa_filter_history_args;
int kjb_pass_taa_filter_history(kjb_context *ctx, const kjb_taa_filter_history_args *a);

typedef struct kjb_taa_input_prob_args {             /* "taa input prob", input_prob.hlsl:11-23, taa.rs:129-144 */
    kjb_image input_tex, filtered_input_tex, filtered_input_dev_tex, history_tex, filtered_history_tex, reprojection_tex, depth_tex,
              smooth_var_history_tex, velocity_history_tex, output_tex;
    float input_tex_size[4];
} kjb_taa_input_prob_args;
int kjb_pass_taa_input_prob(kjb_context *ctx, const kjb_taa_input_prob_args *a);

typedef struct kjb_taa_prob_filter_args { kjb_image input_tex, output_tex; } kjb_taa_prob_filter_args;
int kjb_pass_taa_prob_filter(kjb_context *ctx, const kjb_taa_prob_filter_args *a);    /* "taa prob filter", filter_prob.hlsl */
int kjb_pass_taa_prob_filter2(kjb_context *ctx, const kjb_taa_prob_filter_args *a);   /* "taa prob filter2", filter_prob2.hlsl */

typedef struct kjb_taa_args {                        /* "taa", taa.hlsl:10-26, taa.rs:168-185 */
    kjb_image input_tex, history_tex, reprojection_tex, closest_velocity_tex, velocity_history_tex, depth_tex, smooth_var_history_tex, input_prob_tex;
    kjb_image temporal_output_tex, output_tex, smooth_var_output_tex, velocity_output_tex;
    float input_tex_size[4], output_tex_size[4];
} kjb_taa_args;
int kjb_pass_taa(kjb_context *ctx, const kjb_taa_args *a);

/* ------------------------------------------------------------------ reference path tracer (the oracle's quantity, also a GPU pass)
 * "reference pt" (renderers/reference.rs:8-25, rt/reference_path_trace.rgen.hlsl:75-377): accumulates into RGBA32F. */
typedef struct kjb_reference_pt_args {
    kjb_image output_tex;          /* RGBA32_FLOAT, read-write accumulation */
    uint32_t indirect_only;        /* the shader's INDIRECT_ONLY compile-time switch (:33), runtime here */
} kjb_reference_pt_args;
int kjb_pass_reference_path_trace(kjb_context *ctx, const kjb_reference_pt_args *a);

#ifdef __cplusplus
}
#endif
#endif /* KJB_H */
