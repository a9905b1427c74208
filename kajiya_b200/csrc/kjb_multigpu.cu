// Multi-GPU transport for tile-sharded frames (SURVEY §8e): one ncclAllGather per frame on the context's stream.
// NCCL is dlopen'ed (no link-time dependency: the library must load in the GPU-less build container); the communicator is
// created from a unique id the caller distributes (bench.py uses torch.distributed for that plumbing only).
#include <vector>
#include "kjb_context.h"
#if !defined(KJB_EMU)
#include <dlfcn.h>
#endif

using namespace kjb;

namespace {
#if !defined(KJB_EMU)
struct NcclId { char b[128]; };   // ncclUniqueId
struct NcclApi {
    typedef NcclId Id;
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, NcclId /* by value */, int) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool load() {
        if (lib) return true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
        if (!lib) return false;
        GetUniqueId = (int (*)(void*))dlsym(lib, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
        AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
        CommDestroy = (int (*)(void*))dlsym(lib, "ncclCommDestroy");
        GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
        return GetUniqueId && CommInitRank && AllGather;
    }
} g_nccl;
#endif
}  // namespace

// ---- batched device-to-device copy: blockIdx.y selects the copy, gridDim.x CTAs stride over it with 16-byte accesses (four in flight per thread)
// when both ends and the size allow, bytes otherwise.  gridDim.x follows the largest copy of the batch: one CTA per 64 KiB, at most 256 — a whole band
// of a full-res image (8 MB) is then copied by the whole GPU instead of by 24 CTAs.
#define KJB_COPY_BATCH 96u
#define KJB_COPY_CTAS 24u
#define KJB_COPY_CTAS_MAX 256u
struct CopyBatch { kjb_copy_desc d[KJB_COPY_BATCH]; uint32_t count; };
KJB_KERNEL(256) k_copy_batch(CopyBatch b, kjb::Rows kjb_rows) {
    const kjb_copy_desc cd = b.d[blockIdx.y];
    const uint64_t tid = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x, nthreads = uint64_t(gridDim.x) * blockDim.x;
    if (((uintptr_t(cd.dst) | uintptr_t(cd.src) | cd.bytes) & 15u) == 0) {
        const uint4* s = reinterpret_cast<const uint4*>(cd.src); uint4* d = reinterpret_cast<uint4*>(cd.dst);
        const uint64_t n = cd.bytes / 16;
        uint64_t i = tid;
        for (; i + 3 * nthreads < n; i += 4 * nthreads) {
            const uint4 a0 = s[i], a1 = s[i + nthreads], a2 = s[i + 2 * nthreads], a3 = s[i + 3 * nthreads];
            d[i] = a0; d[i + nthreads] = a1; d[i + 2 * nthreads] = a2; d[i + 3 * nthreads] = a3;
        }
        for (; i < n; i += nthreads) d[i] = s[i];
    } else {
        const uint8_t* s = reinterpret_cast<const uint8_t*>(cd.src); uint8_t* d = reinterpret_cast<uint8_t*>(cd.dst);
        for (uint64_t i = tid; i < cd.bytes; i += nthreads) d[i] = s[i];
    }
}

extern "C" {

int kjb_comm_nccl_unique_id(void* out) {
#if defined(KJB_EMU)
    (void)out; return 1;
#else
    if (!g_nccl.load()) return 1;
    return g_nccl.GetUniqueId(out);
#endif
}
int kjb_comm_init_nccl(kjb_context* c, const void* id, uint32_t rank, uint32_t nranks) {
#if defined(KJB_EMU)
    (void)id; (void)rank; (void)nranks; return c->fail("emu: no NCCL");
#else
    if (!g_nccl.load()) return c->fail("kjb_comm_init_nccl: libnccl.so.2 not found");
    NcclApi::Id uid; memcpy(uid.b, id, 128);
    void* comm = nullptr;
    const int rc = g_nccl.CommInitRank(&comm, int(nranks), uid, int(rank));
    if (rc != 0) return c->fail(std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error"));
    c->nccl_comm = comm; c->rank = rank; c->nranks = nranks;
    return 0;
#endif
}
int kjb_comm_set_callback(kjb_context* c, kjb_allgather_fn fn, void* user, uint32_t rank, uint32_t nranks) { c->ag_fn = fn; c->ag_user = user; c->rank = rank; c->nranks = nranks; return 0; }
int kjb_comm_rank(kjb_context* c, uint32_t* r, uint32_t* n) { *r = c->rank; *n = c->nranks; return 0; }
int kjb_allgather_on(kjb_context* c, uint32_t queue, const void* send, void* recv, uint64_t bytes) {
#if !defined(KJB_EMU)
    cudaStream_t st = c->queue(queue); if (!st) return c->fail("kjb_allgather: bad queue");
    if (c->nranks <= 1) return cudaMemcpyAsync(recv, send, bytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess;
    if (c->nccl_comm) {
        const int rc = g_nccl.AllGather(send, recv, size_t(bytes), /* ncclInt8 */ 0, c->nccl_comm, st);
        return rc == 0 ? 0 : c->fail(std::string("ncclAllGather: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error"));
    }
#else
    if (c->nranks <= 1) return dev_d2d(c, recv, send, bytes);
#endif
    if (!c->ag_fn) return c->fail("kjb_allgather: no transport registered (kjb_comm_init_nccl / kjb_comm_set_callback)");
    if (dev_sync(c)) return c->fail("kjb_allgather: sync failed");
    if (send == (const char*)recv + uint64_t(c->rank) * bytes) {   // in place (this rank's part already sits in `recv`): the transport gets a separate copy of it
        if (c->ag_scratch_bytes < bytes) {
            dev_free(c->ag_scratch); c->ag_scratch_bytes = 0;
            c->ag_scratch = dev_alloc(bytes); if (!c->ag_scratch) return c->fail("kjb_allgather: out of device memory");
            c->ag_scratch_bytes = bytes;
        }
        if (dev_d2d(c, c->ag_scratch, send, bytes) || dev_sync(c)) return c->fail("kjb_allgather: staging copy failed");
        send = c->ag_scratch;
    }
    const int rc = c->ag_fn(c->ag_user, send, recv, bytes);
    // the callback may have left its copies into `recv` in flight on any queue of the context (an upload from pageable memory returns early)
    if (dev_sync(c)) return c->fail("kjb_allgather: sync failed");
    return rc;
}
int kjb_allgather(kjb_context* c, const void* send, void* recv, uint64_t bytes) { return kjb_allgather_on(c, KJB_QUEUE_COMPUTE, send, recv, bytes); }
int kjb_memcpy_d2d(kjb_context* c, void* dst, const void* src, uint64_t bytes) { c->invalidate_positions(); return dev_d2d(c, dst, src, bytes); }
int kjb_memcpy_d2d_batch_on(kjb_context* c, uint32_t queue, const kjb_copy_desc* copies, uint32_t count) {
    c->invalidate_positions();   // raw device writes may land in an image the position cache was built from
#if !defined(KJB_EMU)
    cudaStream_t st = c->queue(queue); if (!st) return c->fail("kjb_memcpy_d2d_batch: bad queue");
#endif
    for (uint32_t i0 = 0; i0 < count; i0 += KJB_COPY_BATCH) {
        CopyBatch b; b.count = count - i0 < KJB_COPY_BATCH ? count - i0 : KJB_COPY_BATCH;
        bool any = false; uint64_t largest = 0;
        for (uint32_t i = 0; i < b.count; ++i) { b.d[i] = copies[i0 + i]; any = any || copies[i0 + i].bytes; largest = largest > copies[i0 + i].bytes ? largest : copies[i0 + i].bytes; }
        if (!any) continue;
        uint32_t ctas = uint32_t((largest + 65535u) / 65536u); ctas = ctas < 1u ? 1u : (ctas > KJB_COPY_CTAS_MAX ? KJB_COPY_CTAS_MAX : ctas);
        if (ctas < KJB_COPY_CTAS && b.count < 16u) ctas = KJB_COPY_CTAS;   // few small copies: latency matters more than CTA count
        const kjb::Rows rows = {0, 1};
#if defined(KJB_EMU)
        kjb_emu::launch(dim3(ctas > 4u ? 4u : ctas, b.count), dim3(256), [&]() { k_copy_batch(b, rows); });
#else
        k_copy_batch<<<dim3(ctas, b.count), dim3(256), 0, st>>>(b, rows);
#endif
        c->launches++;
    }
    const char* e = dev_check(c); if (e) return c->fail(std::string("kjb_memcpy_d2d_batch: ") + e);
    return 0;
}
int kjb_memcpy_d2d_batch(kjb_context* c, const kjb_copy_desc* copies, uint32_t count) { return kjb_memcpy_d2d_batch_on(c, KJB_QUEUE_COMPUTE, copies, count); }

}  // extern "C"
