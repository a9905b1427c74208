// C-ABI entry points: context, memory, scene upload, "rebuild tlas", frame constants (include/kjb.h).
#include "kjb_context.h"
#include "kjb_ircache.cuh"
#include "kjb_bvh_build.cuh"   // the device build's kernels, compiled in this translation unit
#include "../../include/kjb_tlas.h"
#include <algorithm>

using namespace kjb;

// ---- "rebuild tlas" on the device.  The reference rebuilds its TLAS every frame (world_renderer.rs:865-911, ray_tracing.rs:455-520); here the
// acceleration structure is ONE flattened world-space BVH, so a transform change means new world-space triangles and new boxes.  When only
// transforms changed (same instances, same meshes) the topology is kept and two kernels redo the rest: (1) every leaf-order triangle record
// is re-derived from the unified vertex buffer and its instance's 3x4 matrix — the kernel that also fills the records of a full rebuild, so they
// are bit-identical to a full rebuild's; (2) boxes are refitted bottom-up (one thread per inner node fills its leaf slots, the second arriver
// at a node carries the union to the parent).  Hits do not depend on the topology (DESIGN.md "ray/triangle contract"), so a refitted
// structure returns exactly what a rebuilt one would.
KJB_DEV void box_of_tri(const float3 a, const float3 b, const float3 c, float* out6) {
    out6[0] = kjb_min(a.x, kjb_min(b.x, c.x)); out6[1] = kjb_min(a.y, kjb_min(b.y, c.y)); out6[2] = kjb_min(a.z, kjb_min(b.z, c.z));
    out6[3] = kjb_max(a.x, kjb_max(b.x, c.x)); out6[4] = kjb_max(a.y, kjb_max(b.y, c.y)); out6[5] = kjb_max(a.z, kjb_max(b.z, c.z));
}
KJB_KERNEL(256) k_refit_tris(SceneView sc, BvhTri* tris, float* tri_box, uint32_t slot_count, Rows kjb_rows) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slot_count) return;
    const uint32_t gid = tris[s].gid;
    if (gid >= sc.tri_count) return;
    const TriInfo ti = sc.tri_info[gid];
    const kjb_instance& inst = sc.instances[ti.instance];
    const kjb_gpu_mesh mesh = sc.meshes[inst.mesh_index];
    float3 wv[3];
    for (int k = 0; k < 3; ++k) {
        const uint32_t idx = vb_u32(sc, mesh.index_offset + (ti.prim * 3 + k) * 4);
        const float* v = reinterpret_cast<const float*>(sc.vertices + mesh.vertex_core_offset + size_t(idx) * 16);
        wv[k] = xform_point(inst.transform, f3(v[0], v[1], v[2]));
    }
    BvhTri t = tris[s];
    t.v0[0] = wv[0].x; t.v0[1] = wv[0].y; t.v0[2] = wv[0].z;
    t.e1[0] = wv[1].x - wv[0].x; t.e1[1] = wv[1].y - wv[0].y; t.e1[2] = wv[1].z - wv[0].z;
    t.e2[0] = wv[2].x - wv[0].x; t.e2[1] = wv[2].y - wv[0].y; t.e2[2] = wv[2].z - wv[0].z;
    tris[s] = t;
    box_of_tri(wv[0], wv[1], wv[2], tri_box + size_t(s) * 6);
}
// node_count: the built tree's inner-node count in device memory (the grid covers the capacity)
KJB_KERNEL(256) k_refit_nodes(BvhNode* nodes, const int32_t* parent, uint32_t* count, float* slot_box, const float* tri_box, const uint32_t* node_count, Rows kjb_rows) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *node_count) return;
    uint32_t leaves = 0;
    for (int k = 0; k < 2; ++k) {
        const int32_t ch = nodes[i].child[k];
        if (ch >= 0) continue;
        const uint32_t enc = uint32_t(~ch), first = enc >> 3, n = (enc & 7u) + 1u;
        float b[6] = {3.4e38f, 3.4e38f, 3.4e38f, -3.4e38f, -3.4e38f, -3.4e38f};
        for (uint32_t t = 0; t < n; ++t) for (int a = 0; a < 3; ++a) { b[a] = kjb_min(b[a], tri_box[size_t(first + t) * 6 + a]); b[3 + a] = kjb_max(b[3 + a], tri_box[size_t(first + t) * 6 + 3 + a]); }
        for (int a = 0; a < 6; ++a) slot_box[(size_t(i) * 2 + k) * 6 + a] = b[a];
        write_padded_slot(nodes[i], k, b);
        ++leaves;
    }
    if (leaves == 0) return;
    // climb: a node is complete once both of its slots hold this frame's boxes; the arrival that completes it carries the union upwards
    for (;;) {
#if defined(__CUDA_ARCH__)
        __threadfence();
#endif
        if (atom_add(&count[i], leaves) + leaves < 2u) return;
        const int32_t p = parent[i];
        if (p < 0) return;
        float u[6];
        for (int a = 0; a < 3; ++a) { u[a] = kjb_min(slot_box[(size_t(i) * 2) * 6 + a], slot_box[(size_t(i) * 2 + 1) * 6 + a]); u[3 + a] = kjb_max(slot_box[(size_t(i) * 2) * 6 + 3 + a], slot_box[(size_t(i) * 2 + 1) * 6 + 3 + a]); }
        const uint32_t pi = uint32_t(p >> 1); const int pk = p & 1;
        for (int a = 0; a < 6; ++a) slot_box[(size_t(pi) * 2 + pk) * 6 + a] = u[a];
        write_padded_slot(nodes[pi], pk, u);
        i = pi; leaves = 1;
    }
}

extern "C" {

int kjb_abi_version(void) { return KJB_ABI_VERSION; }
#if defined(KJB_EMU)
const char* kjb_backend_name(void) { return "emu-cpu"; }
#else
#if defined(KJB_FAST)
const char* kjb_backend_name(void) { return "cuda-sm90a-fast"; }   // approximate-math build (include/kjb_numeric.h, KJB_FAST): never the default
#else
const char* kjb_backend_name(void) { return "cuda-sm90a"; }
#endif
#endif

static thread_local std::string g_create_error;

int kjb_create(int device, kjb_context** out) {
    *out = nullptr;
#if !defined(KJB_EMU)
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { g_create_error = "kjb_create: no CUDA device (this library has no CPU fallback)"; return 1; }
    if (device < 0 || device >= n) { g_create_error = "kjb_create: invalid device ordinal"; return 1; }
    if (cudaSetDevice(device) != cudaSuccess) { g_create_error = "kjb_create: cudaSetDevice failed"; return 1; }
#endif
    kjb_context* c = new kjb_context();
    c->device = device;
#if !defined(KJB_EMU)
    if (cudaStreamCreateWithFlags(&c->compute_stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; g_create_error = "kjb_create: stream creation failed"; return 1; }
    c->stream = c->compute_stream;
#endif
    memset(&c->g, 0, sizeof(c->g));
    c->d_ray_counters = (unsigned long long*)dev_alloc(2 * sizeof(unsigned long long));
    c->g.scene.ray_counters = c->d_ray_counters;
    c->g.scene.root = ~int32_t(0);
    *out = c;
    return 0;
}
void kjb_destroy(kjb_context* c) {
    if (!c) return;
    dev_sync(c);
    dev_free(c->d_vertices); dev_free(c->d_meshes); dev_free(c->d_instances); dev_free(c->d_nodes); dev_free(c->d_tris); dev_free(c->d_tri_info);
    dev_free(c->d_node_parent); dev_free(c->d_refit_count); dev_free(c->d_slot_box); dev_free(c->d_tri_box); dev_free(c->d_bvh_scratch); dev_free(c->d_inst_prefix);
    dev_free(c->d_tex_data); dev_free(c->d_tex_desc); dev_free(c->d_lights); dev_free(c->d_ray_counters); dev_free(c->d_prev_instances); dev_free(c->d_resolve_offsets); dev_free(c->ag_scratch);
    for (auto& kv : c->ircache_scratch) { const auto& s = kv.second; dev_free(s.claim_rank); dev_free(s.claim_vertex); dev_free(s.life_pending); dev_free(s.scan); dev_free(s.claim_bits); dev_free(s.aux_prev); dev_free(s.entry_vertex); }
#if !defined(KJB_EMU)
    if (c->pinned_staging) cudaFreeHost(c->pinned_staging);
    for (auto& ge : c->graph_execs) if (ge) cudaGraphExecDestroy(ge);
    for (auto& ev : c->queue_events) if (ev) cudaEventDestroy(ev);
    for (auto& st : c->copy_streams) if (st) cudaStreamDestroy(st);
    if (c->compute_stream) cudaStreamDestroy(c->compute_stream);
#endif
    delete c;
}
int kjb_sync(kjb_context* c) {
    if (dev_sync(c)) return c->fail("kjb_sync: stream synchronize failed");
    const char* e = dev_check(c); if (e) return c->fail(std::string("kjb_sync: ") + e);
    return 0;
}
const char* kjb_last_error(kjb_context* c) { return c ? c->last_error.c_str() : g_create_error.c_str(); }
uint64_t kjb_launch_count(kjb_context* c) { return c->launches; }
#if defined(KJB_EMU)
void* kjb_stream(kjb_context* c) { return (void*)c->stream; }
#else
void* kjb_stream(kjb_context* c) { return (void*)c->compute_stream; }
#endif
uint32_t kjb_format_texel_bytes(uint32_t f) { return texel_bytes(f); }

int kjb_image_alloc(kjb_context* c, uint32_t w, uint32_t h, uint32_t layers, uint32_t fmt, kjb_image* out) {
    if (!texel_bytes(fmt) || !w || !h) return c->fail("kjb_image_alloc: bad format or extent");
    out->width = w; out->height = h; out->format = fmt; out->layers = layers ? layers : 1;
    out->data = dev_alloc(image_bytes(*out));   // zero-filled
    return out->data ? 0 : c->fail("kjb_image_alloc: out of device memory");
}
// the cache scratch of a freed life buffer goes with it: the address may be reused by a cache that must not inherit its pending claims
static void drop_ircache_scratch(kjb_context* c, const void* p) {
    auto it = c->ircache_scratch.find(p);
    if (it == c->ircache_scratch.end()) return;
    dev_sync(c);
    const auto& s = it->second; dev_free(s.claim_rank); dev_free(s.claim_vertex); dev_free(s.life_pending); dev_free(s.scan); dev_free(s.claim_bits); dev_free(s.aux_prev); dev_free(s.entry_vertex);
    c->ircache_scratch.erase(it);
}
int kjb_image_free(kjb_context* c, kjb_image* img) {
    drop_ircache_scratch(c, img->data);
    dev_free(img->data); img->data = nullptr; return 0;
}
int kjb_image_clear(kjb_context* c, const kjb_image* img) { c->invalidate_positions(); return dev_memset(c, img->data, 0, image_bytes(*img)); }
int kjb_image_fill_u8(kjb_context* c, const kjb_image* img, uint32_t v) { c->invalidate_positions(); return dev_memset(c, img->data, int(v), image_bytes(*img)); }
int kjb_image_copy(kjb_context* c, const kjb_image* dst, const kjb_image* src) { c->invalidate_positions();
    if (image_bytes(*dst) != image_bytes(*src) || dst->format != src->format) return c->fail("kjb_image_copy: extent/format mismatch");
    return dev_d2d(c, dst->data, src->data, image_bytes(*dst));
}
int kjb_image_upload(kjb_context* c, const kjb_image* dst, const void* src) { c->invalidate_positions(); return dev_h2d(c, dst->data, src, image_bytes(*dst)); }
int kjb_image_download(kjb_context* c, const kjb_image* src, void* dst) { return dev_d2h(c, dst, src->data, image_bytes(*src)); }
#if defined(KJB_EMU)
int kjb_image_upload_on(kjb_context* c, uint32_t, const kjb_image* dst, const void* src) { return kjb_image_upload(c, dst, src); }
int kjb_image_download_on(kjb_context* c, uint32_t, const kjb_image* src, void* dst) { return kjb_image_download(c, src, dst); }
int kjb_image_upload_rows_on(kjb_context* c, uint32_t, const kjb_image* dst, const void* src, uint32_t r0, uint32_t n) {
    if (r0 + n > dst->height) return c->fail("kjb_image_upload_rows_on: rows out of range");
    const size_t rb = size_t(dst->width) * texel_bytes(dst->format); c->invalidate_positions(); memcpy((char*)dst->data + rb * r0, (const char*)src + rb * r0, rb * n); return 0; }
int kjb_image_download_rows_on(kjb_context* c, uint32_t, const kjb_image* src, void* dst, uint32_t r0, uint32_t n) {
    if (r0 + n > src->height) return c->fail("kjb_image_download_rows_on: rows out of range");
    const size_t rb = size_t(src->width) * texel_bytes(src->format); memcpy((char*)dst + rb * r0, (const char*)src->data + rb * r0, rb * n); return 0; }
int kjb_event_record(kjb_context*, uint32_t, uint32_t) { return 0; }
int kjb_queue_wait_event(kjb_context*, uint32_t, uint32_t) { return 0; }
int kjb_event_synchronize(kjb_context*, uint32_t) { return 0; }
#else
int kjb_image_upload_on(kjb_context* c, uint32_t q, const kjb_image* dst, const void* src) {
    c->invalidate_positions();
    cudaStream_t st = c->queue(q); if (!st) return c->fail("kjb_image_upload_on: bad queue");
    return cudaMemcpyAsync(dst->data, src, image_bytes(*dst), cudaMemcpyHostToDevice, st) != cudaSuccess ? c->fail("kjb_image_upload_on: copy failed") : 0;
}
int kjb_image_upload_rows_on(kjb_context* c, uint32_t q, const kjb_image* dst, const void* src, uint32_t r0, uint32_t n) {
    if (r0 + n > dst->height || (dst->layers > 1)) return c->fail("kjb_image_upload_rows_on: rows out of range");
    c->invalidate_positions();
    cudaStream_t st = c->queue(q); if (!st) return c->fail("kjb_image_upload_rows_on: bad queue");
    const size_t rb = size_t(dst->width) * texel_bytes(dst->format);
    return cudaMemcpyAsync((char*)dst->data + rb * r0, (const char*)src + rb * r0, rb * n, cudaMemcpyHostToDevice, st) != cudaSuccess ? c->fail("kjb_image_upload_rows_on: copy failed") : 0;
}
int kjb_image_download_rows_on(kjb_context* c, uint32_t q, const kjb_image* src, void* dst, uint32_t r0, uint32_t n) {
    if (r0 + n > src->height || (src->layers > 1)) return c->fail("kjb_image_download_rows_on: rows out of range");
    cudaStream_t st = c->queue(q); if (!st) return c->fail("kjb_image_download_rows_on: bad queue");
    const size_t rb = size_t(src->width) * texel_bytes(src->format);
    return cudaMemcpyAsync((char*)dst + rb * r0, (const char*)src->data + rb * r0, rb * n, cudaMemcpyDeviceToHost, st) != cudaSuccess ? c->fail("kjb_image_download_rows_on: copy failed") : 0;
}
int kjb_image_download_on(kjb_context* c, uint32_t q, const kjb_image* src, void* dst) {
    cudaStream_t st = c->queue(q); if (!st) return c->fail("kjb_image_download_on: bad queue");
    return cudaMemcpyAsync(dst, src->data, image_bytes(*src), cudaMemcpyDeviceToHost, st) != cudaSuccess ? c->fail("kjb_image_download_on: copy failed") : 0;
}
int kjb_event_record(kjb_context* c, uint32_t e, uint32_t q) {
    cudaStream_t st = c->queue(q); if (!st || e >= KJB_MAX_EVENTS) return c->fail("kjb_event_record: bad queue or event");
    if (!c->queue_events[e] && cudaEventCreateWithFlags(&c->queue_events[e], cudaEventDisableTiming) != cudaSuccess) return c->fail("kjb_event_record: cudaEventCreate failed");
    return cudaEventRecord(c->queue_events[e], st) != cudaSuccess ? c->fail("kjb_event_record: record failed") : 0;
}
int kjb_queue_wait_event(kjb_context* c, uint32_t q, uint32_t e) {
    cudaStream_t st = c->queue(q); if (!st || e >= KJB_MAX_EVENTS) return c->fail("kjb_queue_wait_event: bad queue or event");
    if (!c->queue_events[e]) return 0;
    return cudaStreamWaitEvent(st, c->queue_events[e], 0) != cudaSuccess ? c->fail("kjb_queue_wait_event: wait failed") : 0;
}
int kjb_event_synchronize(kjb_context* c, uint32_t e) {
    if (e >= KJB_MAX_EVENTS) return c->fail("kjb_event_synchronize: bad event");
    if (!c->queue_events[e]) return 0;
    return cudaEventSynchronize(c->queue_events[e]) != cudaSuccess ? c->fail("kjb_event_synchronize: failed") : 0;
}
#endif
int kjb_buffer_alloc(kjb_context* c, uint64_t n, kjb_buffer* out) { out->data = dev_alloc(n); out->size_bytes = n; return out->data ? 0 : c->fail("kjb_buffer_alloc: out of device memory"); }
int kjb_buffer_free(kjb_context* c, kjb_buffer* b) { drop_ircache_scratch(c, b->data); dev_free(b->data); b->data = nullptr; return 0; }
int kjb_buffer_upload(kjb_context* c, const kjb_buffer* dst, uint64_t off, const void* src, uint64_t n) { return dev_h2d(c, (char*)dst->data + off, src, n); }
int kjb_buffer_download(kjb_context* c, const kjb_buffer* src, uint64_t off, void* dst, uint64_t n) { return dev_d2h(c, dst, (const char*)src->data + off, n); }

// ---------------------------------------------------------------------------------------------------------- scene
int kjb_scene_set_geometry(kjb_context* c, const void* vb, uint64_t vb_bytes, const kjb_gpu_mesh* meshes, const uint32_t* counts, uint32_t n) {
    dev_sync(c);
    dev_free(c->d_vertices); dev_free(c->d_meshes);
    c->h_vertices.assign((const uint8_t*)vb, (const uint8_t*)vb + vb_bytes);
    c->h_meshes.assign(meshes, meshes + n); c->h_index_counts.assign(counts, counts + n);
    c->d_vertices = (uint8_t*)dev_alloc(vb_bytes); c->d_meshes = (kjb_gpu_mesh*)dev_alloc(n * sizeof(kjb_gpu_mesh));
    if (!c->d_vertices || !c->d_meshes) return c->fail("kjb_scene_set_geometry: out of device memory");
    dev_h2d(c, c->d_vertices, c->h_vertices.data(), vb_bytes); dev_h2d(c, c->d_meshes, c->h_meshes.data(), n * sizeof(kjb_gpu_mesh));
    c->g.scene.vertices = c->d_vertices; c->g.scene.meshes = c->d_meshes;
    c->tlas_valid = false;
    return dev_sync(c);
}
int kjb_scene_set_textures(kjb_context* c, const kjb_texture_desc* t, uint32_t n) {
    dev_sync(c);
    dev_free(c->d_tex_data); dev_free(c->d_tex_desc); c->d_tex_data = nullptr; c->d_tex_desc = nullptr;
    std::vector<uint8_t> data; std::vector<uint4> desc(n);
    for (uint32_t i = 0; i < n; ++i) {
        size_t bytes = 0; for (uint32_t m = 0; m < t[i].mip_count; ++m) bytes += size_t(t[i].width >> m ? t[i].width >> m : 1) * (t[i].height >> m ? t[i].height >> m : 1) * 4;
        desc[i] = u4(uint32_t(data.size()), t[i].width, t[i].height, t[i].mip_count | (t[i].srgb << 16));
        data.insert(data.end(), t[i].texels, t[i].texels + bytes);
        while (data.size() & 15) data.push_back(0);
    }
    c->tex_count = n;
    if (n) {
        c->d_tex_data = (uint8_t*)dev_alloc(data.size()); c->d_tex_desc = (uint4*)dev_alloc(n * sizeof(uint4));
        if (!c->d_tex_data || !c->d_tex_desc) return c->fail("kjb_scene_set_textures: out of device memory");
        dev_h2d(c, c->d_tex_data, data.data(), data.size()); dev_h2d(c, c->d_tex_desc, desc.data(), n * sizeof(uint4));
    }
    c->g.scene.tex_data = c->d_tex_data; c->g.scene.tex_desc = c->d_tex_desc; c->g.scene.tex_count = n;
    return dev_sync(c);
}

// one slot of the pinned staging ring (4 slots): the caller's host array may change as soon as the upload is enqueued
static void* staging_slot(kjb_context* c, size_t bytes) {
    if (c->pinned_bytes < bytes) {
#if !defined(KJB_EMU)
        dev_sync(c); if (c->pinned_staging) cudaFreeHost(c->pinned_staging);
        if (cudaMallocHost(&c->pinned_staging, bytes * 4) != cudaSuccess) { c->pinned_staging = nullptr; c->pinned_bytes = 0; return nullptr; }
#else
        free(c->pinned_staging); c->pinned_staging = malloc(bytes * 4);
#endif
        c->pinned_bytes = bytes;
    }
    return (char*)c->pinned_staging + size_t(c->staging_seq++ & 3u) * c->pinned_bytes;
}
// grow-only device capacities of the structure and its build: past the first frames of a scene, a rebuild allocates nothing
static int reserve_tlas(kjb_context* c, uint32_t tris, uint32_t instances) {
    const bool grow_tris = tris > c->bvh_tri_cap || !c->d_bvh_scratch, grow_inst = instances + 1 > c->bvh_inst_cap || !c->d_instances;
    if (!grow_tris && !grow_inst) return 0;
    dev_sync(c);
    if (grow_inst) {
        const uint32_t cap = std::max(instances + 1, c->bvh_inst_cap * 2);
        dev_free(c->d_instances); dev_free(c->d_inst_prefix);
        c->d_instances = (kjb_instance*)dev_alloc(size_t(cap) * sizeof(kjb_instance)); c->d_inst_prefix = (uint32_t*)dev_alloc(size_t(cap + 1) * 4);
        c->bvh_inst_cap = cap;
        if (!c->d_instances || !c->d_inst_prefix) { c->bvh_inst_cap = 0; return c->fail("kjb_rebuild_tlas: out of device memory"); }
    }
    if (grow_tris) {
        const uint32_t cap = std::max(std::max(tris, 1u), c->bvh_tri_cap + c->bvh_tri_cap / 2);
        dev_free(c->d_nodes); dev_free(c->d_tris); dev_free(c->d_tri_info); dev_free(c->d_node_parent); dev_free(c->d_refit_count); dev_free(c->d_slot_box);
        dev_free(c->d_tri_box); dev_free(c->d_bvh_scratch);
        c->d_nodes = (BvhNode*)dev_alloc(size_t(cap) * sizeof(BvhNode)); c->d_tris = (BvhTri*)dev_alloc(size_t(cap) * sizeof(BvhTri));
        c->d_tri_info = (TriInfo*)dev_alloc(size_t(cap + 1) * sizeof(TriInfo)); c->d_node_parent = (int32_t*)dev_alloc(size_t(cap) * 4);
        c->d_refit_count = (uint32_t*)dev_alloc(size_t(cap) * 4); c->d_slot_box = (float*)dev_alloc(size_t(cap) * 12 * sizeof(float));
        c->d_tri_box = (float*)dev_alloc(size_t(cap) * 6 * sizeof(float)); c->d_bvh_scratch = dev_alloc(bvh_build_scratch_bytes(cap));
        c->bvh_tri_cap = cap;
        if (!c->d_nodes || !c->d_tris || !c->d_tri_info || !c->d_node_parent || !c->d_refit_count || !c->d_slot_box || !c->d_tri_box || !c->d_bvh_scratch) {
            c->bvh_tri_cap = 0; return c->fail("kjb_rebuild_tlas: out of device memory");
        }
        c->d_node_count = bvh_build_node_count(c);
    }
    return 0;
}

// "rebuild tlas": the instances' triangles in world space and the BVH over them, built on the device (kjb_bvh_build.cuh).  Skipped when the
// instance list is bit-identical to the previous call (static scenes), which is the steady state of every benchmark config.
int kjb_rebuild_tlas(kjb_context* c, const kjb_instance* inst, uint32_t n) {
    if (c->tlas_valid && c->h_instances.size() == n && (n == 0 || memcmp(c->h_instances.data(), inst, n * sizeof(kjb_instance)) == 0)) return 0;
    {   // same instances, same meshes, other transforms (the per-frame case of a moving scene): refit on the device, no host work, no sync
        bool same_topology = c->tlas_valid && c->h_instances.size() == n && n > 0 && c->node_count > 0 && c->d_node_parent;
        for (uint32_t i = 0; same_topology && i < n; ++i) same_topology = c->h_instances[i].mesh_index == inst[i].mesh_index;
        if (same_topology) {
            kjb_instance* stage = (kjb_instance*)staging_slot(c, n * sizeof(kjb_instance));
            if (!stage) return c->fail("kjb_rebuild_tlas: pinned staging allocation failed");
            memcpy(stage, inst, n * sizeof(kjb_instance));
            c->h_instances.assign(inst, inst + n);
            if (dev_h2d(c, c->d_instances, stage, n * sizeof(kjb_instance))) return c->fail("kjb_rebuild_tlas: instance upload failed");
            dev_memset(c, c->d_refit_count, 0, c->node_count * sizeof(uint32_t));
            const kjb::Rows kjb__rows = {0, 1};
            KJB_LAUNCH(c, k_refit_tris, KJB_DIMS(dim3((c->slot_count + 255) / 256), dim3(256)), c->g.scene, c->d_tris, c->d_tri_box, c->slot_count);
            KJB_LAUNCH(c, k_refit_nodes, KJB_DIMS(dim3((c->node_count + 255) / 256), dim3(256)), c->d_nodes, (const int32_t*)c->d_node_parent, c->d_refit_count, c->d_slot_box, (const float*)c->d_tri_box, (const uint32_t*)c->d_node_count);
            c->tlas_refits++;
            KJB_PASS_EPILOGUE(c, "rebuild tlas (refit)");
        }
    }
    // a new instance list: the triangle count and each instance's first triangle are known here, everything else is built on the device
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        if (inst[i].mesh_index >= c->h_meshes.size()) return c->fail("kjb_rebuild_tlas: instance references an unknown mesh");
        total += c->h_index_counts[inst[i].mesh_index] / 3;
    }
    if (total >= (1u << 28)) return c->fail("kjb_rebuild_tlas: more than 2^28 triangles (leaf references hold 28 bits of triangle slot)");
    const uint32_t ntri = uint32_t(total);
    if (reserve_tlas(c, ntri, n)) return 1;
    const size_t inst_bytes = size_t(n) * sizeof(kjb_instance), stage_bytes = inst_bytes + size_t(n + 1) * 4;
    uint8_t* stage = (uint8_t*)staging_slot(c, stage_bytes);
    if (!stage) return c->fail("kjb_rebuild_tlas: pinned staging allocation failed");
    memcpy(stage, inst, inst_bytes);
    uint32_t* prefix = (uint32_t*)(stage + inst_bytes);
    prefix[0] = 0;
    for (uint32_t i = 0; i < n; ++i) prefix[i + 1] = prefix[i] + c->h_index_counts[inst[i].mesh_index] / 3;
    if ((n && dev_h2d(c, c->d_instances, stage, inst_bytes)) || dev_h2d(c, c->d_inst_prefix, prefix, size_t(n + 1) * 4)) return c->fail("kjb_rebuild_tlas: instance upload failed");
    c->tlas_rebuilds++;
    c->h_instances.assign(inst, inst + n);
    c->g.scene.nodes = c->d_nodes; c->g.scene.tris = c->d_tris; c->g.scene.tri_info = c->d_tri_info; c->g.scene.instances = c->d_instances;
    c->g.scene.tri_count = ntri;
    // the root is known from the count alone: none (one all-zero triangle record that never hits), a single leaf, or inner node 0
    c->g.scene.root = ntri == 0 ? ~int32_t(0) : (ntri <= 4 ? ~int32_t(ntri - 1) : 0);
    c->slot_count = ntri ? ntri : 1;
    c->node_count = ntri > 4 ? ntri - 1 : 0;   // a bound: the refit reads the built count from d_node_count
    c->tlas_valid = true;
    if (ntri == 0) {
        if (dev_memset(c, c->d_tris, 0, sizeof(BvhTri))) return c->fail("kjb_rebuild_tlas: memset failed");
        KJB_PASS_EPILOGUE(c, "rebuild tlas");
    }
    if (bvh_build_on_device(c, n, ntri)) return 1;
    const kjb::Rows kjb__rows = {0, 1};
    KJB_LAUNCH(c, k_refit_tris, KJB_DIMS(dim3((ntri + 255) / 256), dim3(256)), c->g.scene, c->d_tris, c->d_tri_box, ntri);
    KJB_PASS_EPILOGUE(c, "rebuild tlas");
}

// Copies the structure to the host for inspection (synchronous; not for the frame loop).  Null arrays are skipped; the counts are always written.
int kjb_tlas_download(kjb_context* c, uint32_t out_counts[3], int32_t* out_root, void* nodes, void* tris, void* tri_info, int32_t* parent) {
    if (dev_sync(c)) return c->fail("kjb_tlas_download: sync failed");
    uint32_t nodes_n = 0;
    if (c->tlas_valid && c->node_count) dev_d2h(c, &nodes_n, c->d_node_count, 4);
    if (dev_sync(c)) return c->fail("kjb_tlas_download: sync failed");
    const uint32_t slots = c->tlas_valid ? c->slot_count : 0, infos = c->tlas_valid ? c->g.scene.tri_count : 0;
    out_counts[0] = nodes_n; out_counts[1] = slots; out_counts[2] = infos;
    if (out_root) *out_root = c->g.scene.root;
    if (nodes && nodes_n) dev_d2h(c, nodes, c->d_nodes, size_t(nodes_n) * sizeof(BvhNode));
    if (parent && nodes_n) dev_d2h(c, parent, c->d_node_parent, size_t(nodes_n) * 4);
    if (tris && slots) dev_d2h(c, tris, c->d_tris, size_t(slots) * sizeof(BvhTri));
    if (tri_info && infos) dev_d2h(c, tri_info, c->d_tri_info, size_t(infos) * sizeof(TriInfo));
    if (dev_sync(c)) return c->fail("kjb_tlas_download: sync failed");
    const char* e = dev_check(c); if (e) return c->fail(std::string("kjb_tlas_download: ") + e);
    return 0;
}

}  // extern "C"
// one thread per ray: the frame's walk (trace), or intersect_leaf over every triangle record, whose selection rule does not depend on the order
KJB_KERNEL(128) k_tlas_trace(SceneView sc, const float* rays, uint32_t n, uint32_t flags, uint32_t slots, uint32_t* out, Rows kjb_rows) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = rays + size_t(i) * 8;
    Ray r; r.origin = f3(p[0], p[1], p[2]); r.tmin = p[3]; r.dir = f3(p[4], p[5], p[6]); r.tmax = p[7];
    const bool any = flags & KJB_TLAS_TRACE_ANY_HIT, cull = flags & KJB_TLAS_TRACE_CULL_BACK;
    HitInfo h; h.hit = false; h.t = r.tmax; h.u = 0; h.v = 0; h.gid = 0xffffffffu;
    if (flags & KJB_TLAS_TRACE_BRUTE_FORCE) {
        if (any) h.hit = intersect_leaf<true>(sc.tris, 0, slots, r, cull, h);
        else intersect_leaf<false>(sc.tris, 0, slots, r, cull, h);
    } else {
        h = any ? trace<true>(sc, r, cull) : trace<false>(sc, r, cull);
    }
    uint32_t* o = out + size_t(i) * 4;
    if (!h.hit) { o[0] = 0; o[1] = 0; o[2] = 0; o[3] = 0xffffffffu; }
    else if (any) { o[0] = 0; o[1] = 0; o[2] = 0; o[3] = 0; }
    else { o[0] = kjb_f2u(h.t); o[1] = kjb_f2u(h.u); o[2] = kjb_f2u(h.v); o[3] = h.gid; }
}
extern "C" {

// Inspection call for tests (synchronous, allocates per call).
int kjb_tlas_trace(kjb_context* c, const float* rays, uint32_t n, uint32_t flags, float* out) {
    if (!c->tlas_valid) return c->fail("kjb_tlas_trace: no acceleration structure (render a frame or call kjb_rebuild_tlas first)");
    if (flags & ~(KJB_TLAS_TRACE_ANY_HIT | KJB_TLAS_TRACE_CULL_BACK | KJB_TLAS_TRACE_BRUTE_FORCE)) return c->fail("kjb_tlas_trace: unknown flags");
    if (n == 0) return 0;
    if (dev_sync(c)) return c->fail("kjb_tlas_trace: sync failed");
    float* d_rays = (float*)dev_alloc(size_t(n) * 8 * sizeof(float));
    uint32_t* d_out = (uint32_t*)dev_alloc(size_t(n) * 4 * sizeof(uint32_t));
    int rc = 0;
    if (!d_rays || !d_out) rc = c->fail("kjb_tlas_trace: out of device memory");
    if (!rc && dev_h2d(c, d_rays, rays, size_t(n) * 8 * sizeof(float))) rc = c->fail("kjb_tlas_trace: upload failed");
    if (!rc) {
        const kjb::Rows kjb__rows = {0, 1};
        KJB_LAUNCH(c, k_tlas_trace, KJB_DIMS(dim3((n + 127) / 128), dim3(128)), c->g.scene, (const float*)d_rays, n, flags, c->slot_count, d_out);
        if (dev_d2h(c, out, d_out, size_t(n) * 4 * sizeof(uint32_t))) rc = c->fail("kjb_tlas_trace: download failed");
    }
    if (dev_sync(c) && !rc) rc = c->fail("kjb_tlas_trace: sync failed");
    const char* e = dev_check(c);
    if (e && !rc) rc = c->fail(std::string("kjb_tlas_trace: ") + e);
    dev_free(d_rays); dev_free(d_out);
    return rc;
}

#if defined(KJB_EMU)
int kjb_graph_begin(kjb_context*) { return 0; }
int kjb_graph_end(kjb_context*) { return 0; }
int kjb_graph_select(kjb_context*, uint32_t slot) { return slot < 4 ? 0 : 1; }
int kjb_set_pass_queue(kjb_context* c, uint32_t q) { return q == KJB_QUEUE_COMPUTE ? 0 : c->fail("kjb_set_pass_queue: this backend has one pass queue"); }
int kjb_async_passes_supported(kjb_context*) { return 0; }
#else
// The recording always happens on the compute queue; passes enqueued on the async queue meanwhile (kjb_set_pass_queue) are launched, not recorded
// (relaxed capture mode: other streams of the thread stay usable).
int kjb_graph_begin(kjb_context* c) {
    if (c->graph_capturing) return c->fail("kjb_graph_begin: already recording");
    if (cudaStreamBeginCapture(c->compute_stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) { cudaGetLastError(); return c->fail("kjb_graph_begin: cudaStreamBeginCapture failed"); }
    c->graph_capturing = true;
    return 0;
}
int kjb_graph_end(kjb_context* c) {
    if (!c->graph_capturing) return c->fail("kjb_graph_end: not recording");
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(c->compute_stream, &g);
    c->graph_capturing = false;
    if (e != cudaSuccess || !g) { cudaGetLastError(); return c->fail(std::string("kjb_graph_end: the recording was invalidated (") + cudaGetErrorString(e) + "): a pass inside the pair synchronised or touched another queue"); }
    cudaGraphExec_t& exec = c->graph_execs[c->graph_slot];
    if (exec) {
        cudaGraphExecUpdateResultInfo info;
        if (cudaGraphExecUpdate(exec, g, &info) != cudaSuccess) { cudaGetLastError(); cudaGraphExecDestroy(exec); exec = nullptr; }   // other pass list: new instance
    }
    if (!exec) {
        if (cudaGraphInstantiate(&exec, g, 0) != cudaSuccess) { cudaGetLastError(); cudaGraphDestroy(g); exec = nullptr; return c->fail("kjb_graph_end: cudaGraphInstantiate failed"); }
        c->graph_instantiations++;
    }
    const cudaError_t le = cudaGraphLaunch(exec, c->compute_stream);
    cudaGraphDestroy(g);
    if (le != cudaSuccess) return c->fail(std::string("kjb_graph_end: cudaGraphLaunch failed: ") + cudaGetErrorString(le));
    c->graph_launches++;
    return 0;
}
int kjb_graph_select(kjb_context* c, uint32_t slot) {
    if (slot >= 4) return c->fail("kjb_graph_select: 4 instances are kept");
    if (c->graph_capturing) return c->fail("kjb_graph_select: a recording is open");
    c->graph_slot = slot; return 0;
}
int kjb_set_pass_queue(kjb_context* c, uint32_t q) {
    if (q != KJB_QUEUE_COMPUTE && q != KJB_QUEUE_ASYNC) return c->fail("kjb_set_pass_queue: passes run on the compute or the async queue");
    if (q == KJB_QUEUE_ASYNC && c->debug_serial) return c->fail("kjb_set_pass_queue: serialised debugging keeps every pass on the compute queue");
    cudaStream_t st = c->queue(q); if (!st) return c->fail("kjb_set_pass_queue: queue creation failed");
    c->stream = st; return 0;
}
int kjb_async_passes_supported(kjb_context* c) { return c->debug_serial ? 0 : 1; }
#endif
int kjb_graph_stats(kjb_context* c, uint64_t out[2]) { out[0] = c->graph_launches; out[1] = c->graph_instantiations; return 0; }
int kjb_tlas_stats(kjb_context* c, uint64_t out[2]) { out[0] = c->tlas_rebuilds; out[1] = c->tlas_refits; return 0; }
int kjb_set_frame_constants(kjb_context* c, const kjb_frame_constants* fc, const kjb_triangle_light* lights, uint32_t n) {
    if (fc->triangle_light_count != n) return c->fail("kjb_set_frame_constants: triangle_light_count mismatch");
    c->g.fc = *fc; c->invalidate_positions();
    // SUN_COLOR is a pure function of the frame constants (sun.hlsl:21-29): evaluate once here with the contract's math
    const float3 sc = sun_color_in_direction(*fc, sun_direction(*fc));
    c->g.sun_color[0] = sc.x; c->g.sun_color[1] = sc.y; c->g.sun_color[2] = sc.z; c->g.sun_color[3] = 0;
    if (n > c->lights_capacity) { dev_sync(c); dev_free(c->d_lights); c->d_lights = (kjb_triangle_light*)dev_alloc(n * sizeof(kjb_triangle_light)); c->lights_capacity = n; }
    if (n) {
        // lights change rarely; a synchronous small copy keeps the host buffer lifetime trivial
        dev_h2d(c, c->d_lights, lights, n * sizeof(kjb_triangle_light)); dev_sync(c);
    }
    c->g.lights = c->d_lights;
    return 0;
}
int kjb_set_scissor(kjb_context* c, uint32_t y0, uint32_t y1) { c->scissor_y0 = y0; c->scissor_y1 = y1; return 0; }
// the ordered cache schedule keeps claims pending until the next chain: another schedule would find cells flagged with no entry behind them
static bool ordered_cache_has_run(const kjb_context* c) { return !c->ircache_scratch.empty(); }
int kjb_set_debug_serial(kjb_context* c, uint32_t on) {
    if (on && !c->debug_serial && ordered_cache_has_run(c)) return c->fail("kjb_set_debug_serial: the irradiance cache already runs on the ordered schedule; switch before its first frame");
    c->debug_serial = on != 0; return 0;
}
int kjb_set_option(kjb_context* c, uint32_t option, uint32_t value) {
    if (option == KJB_OPTION_HALF_RES_POSITION_CACHE) { c->opt_position_cache = value != 0; c->invalidate_positions(); return 0; }
    if (option == KJB_OPTION_ORDERED_CACHE_SCHEDULE) {
        if (!value && c->ordered_cache && ordered_cache_has_run(c)) return c->fail("kjb_set_option: the irradiance cache already runs on the ordered schedule; switch before its first frame");
        c->ordered_cache = value != 0; return 0;
    }
    return c->fail("kjb_set_option: unknown option");
}
int kjb_set_luts(kjb_context* c, const kjb_image* fg, const kjb_image* bn) {
    if (!check_img(c, *fg, KJB_FMT_RGBA16_FLOAT, "kjb_set_luts", "brdf_fg_lut", 64, 64)) return 1;
    if (!check_img(c, *bn, KJB_FMT_RGBA8_UNORM, "kjb_set_luts", "blue_noise", 256, 256)) return 1;
    c->g.brdf_fg_lut = img_ro(*fg); c->g.blue_noise = img_ro(*bn);
    return 0;
}
#if defined(KJB_EMU)
}  // extern "C"
#include <chrono>
static std::chrono::steady_clock::time_point g_timer_slots[1024];
extern "C" {
int kjb_timer_record(kjb_context*, uint32_t slot) { if (slot >= 1024) return 1; g_timer_slots[slot] = std::chrono::steady_clock::now(); return 0; }
int kjb_timer_elapsed_ms(kjb_context*, uint32_t a, uint32_t b, float* out) { if (a >= 1024 || b >= 1024) return 1; *out = std::chrono::duration<float, std::milli>(g_timer_slots[b] - g_timer_slots[a]).count(); return 0; }
#else
int kjb_timer_record(kjb_context* c, uint32_t slot) {
    if (slot >= 1024) return c->fail("kjb_timer_record: slot out of range");
    if (c->timer_events.size() <= slot) c->timer_events.resize(slot + 1, nullptr);
    if (!c->timer_events[slot] && cudaEventCreate(&c->timer_events[slot]) != cudaSuccess) return c->fail("kjb_timer_record: cudaEventCreate failed");
    return cudaEventRecord(c->timer_events[slot], c->compute_stream) != cudaSuccess;
}
int kjb_timer_elapsed_ms(kjb_context* c, uint32_t a, uint32_t b, float* out) {
    if (a >= c->timer_events.size() || b >= c->timer_events.size() || !c->timer_events[a] || !c->timer_events[b]) return c->fail("kjb_timer_elapsed_ms: slot was never recorded");
    if (cudaEventSynchronize(c->timer_events[b]) != cudaSuccess) return c->fail("kjb_timer_elapsed_ms: event sync failed");
    return cudaEventElapsedTime(out, c->timer_events[a], c->timer_events[b]) != cudaSuccess;
}
#endif
int kjb_ray_counters(kjb_context* c, uint64_t out[2], int reset) {
    unsigned long long v[2] = {0, 0};
    dev_d2h(c, v, c->d_ray_counters, sizeof(v));
    if (dev_sync(c)) return c->fail("kjb_ray_counters: sync failed");
    out[0] = v[0]; out[1] = v[1];
    if (reset) dev_memset(c, c->d_ray_counters, 0, sizeof(v));
    return 0;
}

}  // extern "C"
