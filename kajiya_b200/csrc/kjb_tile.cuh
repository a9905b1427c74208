// Screen-space tile staging for the stencil / gather kernels: the (block + apron) footprint of an image arrives in shared memory as one
// bulk copy per tile row (cp.async.bulk, completion on an mbarrier) — the copy engine moves the rows and the lanes of warp 0 only issue
// them, instead of every thread a guarded LDG per texel; parts of the footprint outside the image are zero-filled, which is the ABI's
// "reads outside an image return 0".  Warp-level exchange helpers (SHFL) live here too.  Under the test-only CPU launch emulator
// (KJB_EMU) the same calls are plain loops / a shared scratch array.
//
// Bulk copies need 16-byte aligned rows: images whose base or row pitch is not a multiple of 16 bytes (odd test extents) are staged
// with cooperative guarded loads instead — same contents.  The host picks the form per launch (kjb::tile_mode, kjb_context.h).
#pragma once
#include "kjb_device.cuh"

#if defined(KJB_EMU)
#define KJB_DEVONLY inline
#else
#define KJB_DEVONLY __device__ __forceinline__
#endif

namespace kjb {

// number of texels of a tile row as staged in shared memory: the box width rounded up so that a row is a whole number of 16-byte units
template <int TEXEL_BYTES> constexpr int tile_pitch(int w) { return ((w * TEXEL_BYTES + 15) / 16 * 16) / TEXEL_BYTES; }

#if !defined(KJB_EMU)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "KJB_MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra KJB_MBAR_DONE;\n"
        "bra KJB_MBAR_WAIT;\n"
        "KJB_MBAR_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_load_row(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {   // 16-byte aligned on both sides, bytes % 16 == 0
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
#endif

// Staging protocol (every thread of the block executes all calls, uniform control flow):
//     tile_group_begin(bar, phase, mode, tid);                                       // first group of the block: initialises the mbarrier
//     bytes += tile_issue<T, TW, TH>(dst, img, x0, y0, bar, mode, tid, nthreads);        // once per tile: TW x TH texels whose top-left texel is (x0, y0)
//     tile_group_wait(bar, phase, mode, bytes, tid);                                 // arms the barrier with the group's byte count and waits: tiles visible
// `dst` has a row pitch of tile_pitch<sizeof(T)>(TW) texels and is 128-byte aligned; `phase` counts the groups this block has already pushed
// through `bar` (0 for the first).  `mode` is one value per launch, chosen by the host (tile_mode()):
//   KJB_TILE_ROWS   one cp.async.bulk per tile row issued by the lanes of warp 0 (SASS UBLKCP): x0 * sizeof(T) must be a multiple of 16;
//                   parts of the tile outside the image are zero-filled with ordinary stores
//   KJB_TILE_LOADS  guarded loads by every thread (rows not 16-byte aligned — odd test extents — and the CPU emulator)
#define KJB_TILE_LOADS 0
#define KJB_TILE_ROWS 1
template <typename T, int TW, int TH> constexpr uint32_t tile_bytes() { return uint32_t(tile_pitch<int(sizeof(T))>(TW) * TH * sizeof(T)); }

KJB_DEVONLY void tile_group_begin(uint64_t* bar, uint32_t phase, int mode, int tid) {
#if !defined(KJB_EMU)
    if (mode != KJB_TILE_LOADS && phase == 0) { if (tid == 0) mbar_init(bar, 1); __syncthreads(); }
#endif
}
template <typename T, int TW, int TH>
KJB_DEVONLY uint32_t tile_issue(T* dst, const Img& img, int x0, int y0, uint64_t* bar, int mode, int tid, int nthreads) {
    constexpr int PITCH = tile_pitch<int(sizeof(T))>(TW);
#if !defined(KJB_EMU)
    if (mode == KJB_TILE_ROWS) {
        const int xa = x0 < 0 ? 0 : x0, xb = x0 + PITCH < img.w ? x0 + PITCH : img.w;            // texel columns that exist
        const int ya = y0 < 0 ? 0 : y0, yb = y0 + TH < img.h ? y0 + TH : img.h;
        const bool any = xb > xa && yb > ya;
        if (tid < TH) {
            const int gy = y0 + tid;
            if (any && gy >= ya && gy < yb)
                bulk_load_row(dst + tid * PITCH + (xa - x0), img.p + (size_t(gy) * size_t(img.w) + size_t(xa)) * sizeof(T), uint32_t(xb - xa) * uint32_t(sizeof(T)), bar);
        }
        if (!any || xa != x0 || xb != x0 + PITCH || ya != y0 || yb != y0 + TH) {     // block at the image border: the rest of the tile reads as zero
            for (int i = tid; i < PITCH * TH; i += nthreads) {
                const int gx = x0 + i % PITCH, gy = y0 + i / PITCH;
                if (!(any && gx >= xa && gx < xb && gy >= ya && gy < yb)) { T v; memset(&v, 0, sizeof(T)); dst[i] = v; }
            }
        }
        return any ? uint32_t(xb - xa) * uint32_t(yb - ya) * uint32_t(sizeof(T)) : 0u;
    }
#endif
    for (int i = tid; i < PITCH * TH; i += nthreads) {
        const int lx = i % PITCH, ly = i / PITCH;
        T v; memset(&v, 0, sizeof(T));
        if (inb(img, x0 + lx, y0 + ly)) v = ld_raw<T>(img, x0 + lx, y0 + ly);
        dst[i] = v;
    }
    return 0u;
}
KJB_DEVONLY void tile_group_wait(uint64_t* bar, uint32_t phase, int mode, uint32_t bytes, int tid) {
#if !defined(KJB_EMU)
    if (mode != KJB_TILE_LOADS) {
        if (tid == 0) mbar_expect_tx(bar, bytes);     // the one arrival of the phase; copies that already landed have pre-decremented the count
        mbar_wait(bar, phase & 1u);
        __syncthreads();   // border zero-fill was done with ordinary stores
        return;
    }
#endif
    __syncthreads();
}

// ---- warp exchange: value of lane (lane ^ mask) of the same warp.  The blocks that use it are 32 threads wide, so a warp is one row of
// the block and lane == threadIdx.x.  Emulator: through a per-block scratch array with two barriers (all threads of the block take part).
KJB_DEVONLY float warp_xor(float v, int mask) {
#if !defined(KJB_EMU)
    return __shfl_xor_sync(0xffffffffu, v, mask);
#else
    static thread_local float scratch[1024];
    const int t = int(threadIdx.x + threadIdx.y * blockDim.x);
    scratch[t] = v; __syncthreads();
    const float r = scratch[(t & ~31) | ((t & 31) ^ mask)]; __syncthreads();
    return r;
#endif
}

}  // namespace kjb
