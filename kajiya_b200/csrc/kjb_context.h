// Library context + the thin device-runtime layer the entry points use.
// In the product this is the CUDA runtime on one stream of one H100.  When the translation unit is compiled by the
// test-only CPU launch emulator (KJB_EMU, tests/emu/), the same six calls map to libc — that build is never shipped,
// never loaded by kajiya_b200, and reports itself as "emu-cpu".
#pragma once
#include "kjb_trace.cuh"
#include "kjb_tile.cuh"
#include <map>
#include <tuple>
#include <initializer_list>
#include <string>
#include <vector>
#include <cstdio>
#include <cstring>
#include <cstdlib>

#if defined(KJB_EMU)
typedef void* kjb_stream_t;
#else
#include <cuda_runtime.h>
typedef cudaStream_t kjb_stream_t;
#endif

struct kjb_context {
    int device = 0;
    kjb_stream_t stream = nullptr;
    std::string last_error;
    uint64_t launches = 0;

    // scene
    uint8_t* d_vertices = nullptr; size_t vertices_bytes = 0;
    kjb_gpu_mesh* d_meshes = nullptr;
    std::vector<uint8_t> h_vertices; std::vector<kjb_gpu_mesh> h_meshes; std::vector<uint32_t> h_index_counts;
    kjb_instance* d_instances = nullptr; std::vector<kjb_instance> h_instances; bool tlas_valid = false;
    kjb::BvhNode* d_nodes = nullptr; kjb::BvhTri* d_tris = nullptr; kjb::TriInfo* d_tri_info = nullptr;
    // device refit of the acceleration structure when only instance transforms change ("rebuild tlas" every frame, kjb_api.cu)
    int32_t* d_node_parent = nullptr; uint32_t* d_refit_count = nullptr; float* d_slot_box = nullptr; float* d_tri_box = nullptr; uint32_t node_count = 0, slot_count = 0;
    uint64_t tlas_refits = 0, tlas_rebuilds = 0;
    // device build of the structure (kjb_bvh_build.cuh): grow-only capacities in triangles and instances, so that a rebuild with enough
    // room neither allocates nor synchronises; node_count above is then the capacity bound and d_node_count the built tree's count
    uint32_t bvh_tri_cap = 0, bvh_inst_cap = 0; void* d_bvh_scratch = nullptr; uint32_t* d_inst_prefix = nullptr; uint32_t* d_node_count = nullptr;
    uint64_t staging_seq = 0;   // slot of the pinned staging ring the next instance upload uses
    uint8_t* d_tex_data = nullptr; uint4* d_tex_desc = nullptr; uint32_t tex_count = 0;
    kjb_triangle_light* d_lights = nullptr; uint32_t lights_capacity = 0;
    unsigned long long* d_ray_counters = nullptr;
    void* pinned_staging = nullptr; size_t pinned_bytes = 0;
    kjb_instance* d_prev_instances = nullptr; uint32_t prev_instances_capacity = 0; std::vector<kjb_instance> h_prev_instances;   // raster stand-in: last frame's transforms
    int32_t* d_resolve_offsets = nullptr; std::vector<int32_t> h_resolve_offsets;   // SPATIAL_RESOLVE_OFFSETS as last pushed by the host
#if !defined(KJB_EMU)
    std::vector<cudaEvent_t> timer_events;
    cudaStream_t copy_streams[4] = {nullptr, nullptr, nullptr, nullptr};   // KJB_QUEUE_UPLOAD, _DOWNLOAD, _COMM, _ASYNC (created on first use)
    cudaStream_t compute_stream = nullptr;                    // KJB_QUEUE_COMPUTE; `stream` is the queue passes are enqueued on right now (kjb_set_pass_queue)
    cudaEvent_t queue_events[64] = {};                        // kjb_event_record slots
    cudaStream_t queue(uint32_t q) {
        if (q == 0) return compute_stream;
        if (q > 4) return nullptr;
        if (!copy_streams[q - 1]) {
            int lo = 0, hi = 0; cudaDeviceGetStreamPriorityRange(&lo, &hi);   // the async pass queue carries little, latency-bound work: let its blocks in first
            if (cudaStreamCreateWithPriority(&copy_streams[q - 1], cudaStreamNonBlocking, q == 4 ? hi : lo) != cudaSuccess) return nullptr;
        }
        return copy_streams[q - 1];
    }
#endif

#if !defined(KJB_EMU)
    // CUDA Graph replay of a frame (kjb_graph_begin / kjb_graph_end): the instance kept between frames, updated in place while the topology holds
    cudaGraphExec_t graph_execs[4] = {nullptr, nullptr, nullptr, nullptr}; uint32_t graph_slot = 0; bool graph_capturing = false;   // kjb_graph_select
#endif
    uint64_t graph_launches = 0, graph_instantiations = 0;
    kjb::Globals g;   // host copy, passed by value to every kernel
    // tensor maps of the images the tiled kernels stage through TMA, one per (image, box): built on first use, dropped when the image is freed
    std::map<std::tuple<const void*, uint32_t, uint32_t, uint32_t, uint32_t, uint32_t>, kjb::TileSource> tile_sources;
    // device scratch of the irradiance cache's ordered schedule (kjb_ircache.cuh), one set per cache, keyed by its life_buf; freed with that buffer
    struct IrcacheScratch { void* claim_rank; void* claim_vertex; void* life_pending; void* scan; void* claim_bits; void* aux_prev; void* entry_vertex; };
    std::map<const void*, IrcacheScratch> ircache_scratch;

    // multi-GPU transport (tile-sharded frames)
    kjb_allgather_fn ag_fn = nullptr; void* ag_user = nullptr; uint32_t rank = 0, nranks = 1; void* nccl_comm = nullptr;

    // Row scissor for tile-sharded frames (SURVEY §8e): the next pass only computes rows [scissor_y0, scissor_y1) of ITS output
    // grid (0,0 = whole image).  Set by kjb_set_scissor, consumed (and kept) by every kjb_pass_* launch.
    uint32_t scissor_y0 = 0, scissor_y1 = 0;
    // KJB_OPTION_HALF_RES_POSITION_CACHE: world positions of the half-res pixels, from half_depth (a) and from the packed reservoirs (b)
    struct PosCache { float4* d = nullptr; size_t cap = 0; const void* src = nullptr; uint32_t w = 0, h = 0; float gts[4] = {0, 0, 0, 0}; uint64_t epoch = ~0ull; };
    PosCache pos_a, pos_b; uint64_t epoch_a = 0, epoch_b = 0; bool opt_position_cache = false;
    void invalidate_positions() { epoch_a++; epoch_b++; }
    bool debug_serial = false;   // kjb_set_debug_serial: cache-touching passes run on one GPU thread in launch order
#if defined(KJB_EMU)
    bool ordered_cache = false;  // KJB_OPTION_ORDERED_CACHE_SCHEDULE: the emulator runs launches in order, like the oracle
#else
    bool ordered_cache = true;
#endif
    kjb::Rows rows_for(uint32_t H) const {
        kjb::Rows r; r.y0 = 0; r.y1 = int(H);
        if (scissor_y1 > scissor_y0) { r.y0 = int(scissor_y0 < H ? scissor_y0 : H); r.y1 = int(scissor_y1 < H ? scissor_y1 : H); }
        return r;
    }

    int fail(const std::string& msg) { last_error = msg; return 1; }
};

namespace kjb {

#if defined(KJB_EMU)
inline void* dev_alloc(size_t n) { return calloc(n ? n : 1, 1); }
inline void dev_free(void* p) { free(p); }
inline int dev_h2d(kjb_context*, void* d, const void* h, size_t n) { memcpy(d, h, n); return 0; }
inline int dev_d2h(kjb_context*, void* h, const void* d, size_t n) { memcpy(h, d, n); return 0; }
inline int dev_d2d(kjb_context*, void* d, const void* s, size_t n) { memcpy(d, s, n); return 0; }
inline int dev_memset(kjb_context*, void* d, int v, size_t n) { memset(d, v, n); return 0; }
inline int dev_sync(kjb_context*) { return 0; }
inline const char* dev_check(kjb_context*) { return nullptr; }
#else
// Zero-filled allocation.  cudaMemset runs on the legacy default stream, which does NOT order against the context's
// non-blocking stream: wait for it here (allocation is a set-up time operation), or a later async copy/kernel on the
// context stream could be overtaken by the memset.
inline void* dev_alloc(size_t n) {
    void* p = nullptr;
    if (cudaMalloc(&p, n ? n : 1) != cudaSuccess) return nullptr;
    // zero-fill on a stream of its own and wait for THAT stream only: allocation also happens lazily inside a frame that is being captured into
    // a CUDA graph (relaxed capture mode), where touching the legacy stream or synchronising the device would invalidate the capture
    static thread_local cudaStream_t setup = nullptr;
    if (!setup && cudaStreamCreateWithFlags(&setup, cudaStreamNonBlocking) != cudaSuccess) { setup = nullptr; cudaFree(p); return nullptr; }
    if (cudaMemsetAsync(p, 0, n ? n : 1, setup) != cudaSuccess || cudaStreamSynchronize(setup) != cudaSuccess) { cudaFree(p); return nullptr; }
    return p;
}
inline void dev_free(void* p) { if (p) cudaFree(p); }
inline int dev_h2d(kjb_context* c, void* d, const void* h, size_t n) { return cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, c->stream) != cudaSuccess; }
inline int dev_d2h(kjb_context* c, void* h, const void* d, size_t n) { return cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess; }
inline int dev_d2d(kjb_context* c, void* d, const void* s, size_t n) { return cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToDevice, c->stream) != cudaSuccess; }
inline int dev_memset(kjb_context* c, void* d, int v, size_t n) { return cudaMemsetAsync(d, v, n, c->stream) != cudaSuccess; }
inline int dev_sync(kjb_context* c) {   // every queue of the context
    int rc = cudaStreamSynchronize(c->compute_stream) != cudaSuccess;
    for (cudaStream_t st : c->copy_streams) if (st) rc |= cudaStreamSynchronize(st) != cudaSuccess;
    return rc;
}
inline const char* dev_check(kjb_context*) { cudaError_t e = cudaGetLastError(); return e == cudaSuccess ? nullptr : cudaGetErrorString(e); }
#endif

inline uint32_t texel_bytes(uint32_t f);
// TileSource of `img` for tiles of box_w x box_h texels (kjb_tile.cuh).  use_tma = 0 when the image cannot be described to the copy engine
// (row pitch or base not 16-byte aligned, driver entry point missing): the kernels then stage the same tile with guarded loads.
kjb::TileSource tile_source(kjb_context* c, const kjb_image& img, uint32_t box_w, uint32_t box_h);
// staging mode of one launch (KJB_TILE_*): what every source of the launch supports, under the process-wide preference KJB_TILE_MODE = rows | tensor | loads
int tile_mode(std::initializer_list<const kjb::TileSource*> sources);

inline uint32_t texel_bytes(uint32_t f) {
    switch (f) {
        case KJB_FMT_R32_FLOAT: case KJB_FMT_RG16_FLOAT: case KJB_FMT_RGBA8_UNORM: case KJB_FMT_RGBA8_SNORM:
        case KJB_FMT_A2R10G10B10_UNORM: case KJB_FMT_R11G11B10_UFLOAT: case KJB_FMT_R32_UINT: return 4;
        case KJB_FMT_RG32_UINT: case KJB_FMT_RGBA16_FLOAT: case KJB_FMT_RGBA16_SNORM: case KJB_FMT_RG32_FLOAT: return 8;
        case KJB_FMT_RGBA32_FLOAT: case KJB_FMT_RGBA32_UINT: return 16;
        case KJB_FMT_R8_UNORM: case KJB_FMT_R8_SNORM: return 1;
        case KJB_FMT_R16_FLOAT: return 2;
        default: return 0;
    }
}
inline size_t image_bytes(const kjb_image& i) { return size_t(i.width) * i.height * (i.layers ? i.layers : 1) * texel_bytes(i.format); }

// argument validation shared by all pass entry points: format + non-null + (optionally) extent
inline bool check_img(kjb_context* c, const kjb_image& i, uint32_t fmt, const char* pass, const char* name, uint32_t w = 0, uint32_t h = 0) {
    if (!i.data) { c->fail(std::string(pass) + ": image '" + name + "' is null"); return false; }
    if (i.format != fmt) { c->fail(std::string(pass) + ": image '" + name + "' has format " + std::to_string(i.format) + ", expected " + std::to_string(fmt)); return false; }
    if (w && (i.width != w || i.height != h)) { c->fail(std::string(pass) + ": image '" + name + "' has the wrong extent"); return false; }
    return true;
}

}  // namespace kjb

// ---- kernel launch: <<<>>> in the product; a serial block/thread loop under the test emulator
#if defined(KJB_EMU)
#define KJB_KERNEL(bounds) static void
#define KJB_KERNEL_OCC(bounds, min_blocks) static void
#define KJB_LAUNCH(ctx, kernel, dims, ...) do { if (kjb__rows.y1 > kjb__rows.y0) { kjb_emu::launch(dims, [&]() { kernel(__VA_ARGS__, kjb__rows); }); (ctx)->launches++; } } while (0)
#define KJB_LAUNCH_SYNC(ctx, kernel, dims, ...) do { if (kjb__rows.y1 > kjb__rows.y0) { kjb_emu::launch_sync(dims, [&]() { kernel(__VA_ARGS__, kjb__rows); }); (ctx)->launches++; } } while (0)
// kernels that touch the (racy by design) irradiance cache: the emulator runs their blocks one after another in launch order, which
// makes the test build deterministic and comparable with the oracle's serial schedule; on the GPU this is a plain launch
#define KJB_LAUNCH_ORDERED(ctx, kernel, dims, ...) do { if (kjb__rows.y1 > kjb__rows.y0) { kjb_emu::g_serial++; kjb_emu::launch(dims, [&]() { kernel(__VA_ARGS__, kjb__rows); }); kjb_emu::g_serial--; (ctx)->launches++; } } while (0)
#else
#define KJB_KERNEL(bounds) __global__ void __launch_bounds__(bounds)
// same, with a resident-blocks-per-SM target that caps the register allocation (occupancy tuning of the instruction-issue-bound filters)
#define KJB_KERNEL_OCC(bounds, min_blocks) __global__ void __launch_bounds__(bounds, min_blocks)
#define KJB_LAUNCH(ctx, kernel, dims, ...) do { if (kjb__rows.y1 > kjb__rows.y0) { kernel<<<dims, 0, (ctx)->stream>>>(__VA_ARGS__, kjb__rows); (ctx)->launches++; } } while (0)
#define KJB_LAUNCH_SYNC KJB_LAUNCH   /* kernels that use __syncthreads(): only the test emulator needs to know */
#define KJB_LAUNCH_ORDERED KJB_LAUNCH
#endif
#define KJB_DIMS(...) __VA_ARGS__
// Ray-tracing passes: 8 x 16 pixel blocks, so that a warp (32 consecutive threads) is an 8 x 4 pixel patch — compact footprints keep the
// lanes of a warp on neighbouring BVH nodes and make hit / miss shading branch together more often than 32 x 1 or 16 x 2 strips.  The
// serial twins (and the oracle's serial schedule, oracle/kj_ctx.h) walk the pixels in the same block order.
#ifndef KJB_RAY_BX
#define KJB_RAY_BX 8
#endif
#ifndef KJB_RAY_BY
#define KJB_RAY_BY 16
#endif
// every kernel's last parameter is `Rows kjb_rows`: the row range of its grid this launch covers (tile sharding)
#define KJB_ROWS(ctx, H) const kjb::Rows kjb__rows = (ctx)->rows_for(H)
#define KJB_GRID2D(W, H, BX, BY) dim3(((W) + (BX) - 1) / (BX), (unsigned(kjb__rows.y1 - kjb__rows.y0) + (BY) - 1) / (BY), 1), dim3((BX), (BY), 1)
#define KJB_PX int x = int(blockIdx.x * blockDim.x + threadIdx.x), y = kjb_rows.y0 + int(blockIdx.y * blockDim.y + threadIdx.y); if (y >= kjb_rows.y1) return

#define KJB_PASS_EPILOGUE(ctx, name) do { const char* e__ = kjb::dev_check(ctx); if (e__) return (ctx)->fail(std::string(name) + ": " + e__); return 0; } while (0)
