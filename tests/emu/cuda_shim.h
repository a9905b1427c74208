// TEST INFRASTRUCTURE ONLY — CPU launch emulator for the CUDA translation units in kajiya_b200/csrc.
//
// There is no GPU in the build container, so kernel LOGIC is debugged here: this header is force-included
// (g++ -x c++ -include cuda_shim.h -DKJB_EMU) in front of the unmodified .cu sources, supplies the handful of
// CUDA built-ins they use (vector types, threadIdx/blockIdx, dim3) and runs every launch as nested loops over
// blocks and threads (OpenMP over blocks).  The resulting libkjb_emu.so is loaded ONLY by tests/ ("emu-cpu" backend);
// the product package never builds, loads or falls back to it — kajiya_b200.lib() refuses anything but "cuda-sm90a".
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <atomic>
#include <thread>
#include <vector>

#define __host__
#define __device__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __restrict__
#define __grid_constant__
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static thread_local

struct float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct int2 { int x, y; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };

namespace kjb_emu {
struct Idx { unsigned x, y, z; };
}
extern thread_local kjb_emu::Idx threadIdx, blockIdx;
extern thread_local dim3 blockDim, gridDim;

namespace kjb_emu {
int num_workers();
extern int g_serial;   // > 0: run blocks one after another in launch order (KJB_LAUNCH_ORDERED)
template <typename F> inline void launch(dim3 grid, dim3 block, F body) {
    const long nblocks = long(grid.x) * grid.y * grid.z;
    std::atomic<long> next{0};
    auto worker = [&]() {
        for (;;) {
            const long b0 = next.fetch_add(4);
            if (b0 >= nblocks) break;
            for (long b = b0; b < b0 + 4 && b < nblocks; ++b) {
                gridDim = grid; blockDim = block;
                blockIdx.x = unsigned(b % grid.x); blockIdx.y = unsigned((b / grid.x) % grid.y); blockIdx.z = unsigned(b / (long(grid.x) * grid.y));
                for (unsigned tz = 0; tz < block.z; ++tz) for (unsigned ty = 0; ty < block.y; ++ty) for (unsigned tx = 0; tx < block.x; ++tx) {
                    threadIdx.x = tx; threadIdx.y = ty; threadIdx.z = tz;
                    body();
                }
            }
        }
    };
    const int n = (nblocks < 16 || g_serial > 0) ? 1 : num_workers();
    if (n <= 1) { worker(); return; }
    std::vector<std::thread> th;
    for (int i = 0; i < n; ++i) th.emplace_back(worker);
    for (auto& t : th) t.join();
}
// Kernels that use __syncthreads(): every thread of a block runs as a ucontext fiber; a barrier yields to the block
// scheduler, which resumes each unfinished fiber once per barrier phase.
void fiber_run_block(unsigned nthreads, dim3 block, void (*thread_body)(void*), void* arg);
void fiber_barrier();
template <typename F> inline void launch_sync(dim3 grid, dim3 block, F body) {
    const long nblocks = long(grid.x) * grid.y * grid.z;
    std::atomic<long> next{0};
    auto worker = [&]() {
        for (;;) {
            const long b = next.fetch_add(1);
            if (b >= nblocks) break;
            gridDim = grid; blockDim = block;
            blockIdx.x = unsigned(b % grid.x); blockIdx.y = unsigned((b / grid.x) % grid.y); blockIdx.z = unsigned(b / (long(grid.x) * grid.y));
            fiber_run_block(block.x * block.y * block.z, block, [](void* p) { (*static_cast<F*>(p))(); }, &body);
        }
    };
    const int n = nblocks < 4 ? 1 : num_workers();
    if (n <= 1) { worker(); return; }
    std::vector<std::thread> th;
    for (int i = 0; i < n; ++i) th.emplace_back(worker);
    for (auto& t : th) t.join();
}
}  // namespace kjb_emu
inline void __syncthreads() { kjb_emu::fiber_barrier(); }
