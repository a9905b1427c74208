// TEST INFRASTRUCTURE ONLY — CPU launch emulator for the CUDA translation units in kajiya_b200/csrc.
//
// There is no GPU in the build container, so kernel LOGIC is debugged here: this header is force-included
// (g++ -x c++ -include cuda_shim.h -DKJB_EMU) in front of the unmodified .cu sources, supplies the handful of
// CUDA built-ins they use (vector types, threadIdx/blockIdx, dim3) and runs every launch as nested loops over
// blocks and threads (blocks spread over worker threads).  The resulting libkjb_emu.so is loaded ONLY by tests/ ("emu-cpu" backend);
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

// Launch order (kjb_emu_set_launch_order): 0 = forward, 1 = reverse, 2 = a seeded permutation per launch.  The k-th block (thread) a
// launch runs is `order.at(k)`: the bijection k -> (a * k + c) mod n with gcd(a, n) = 1, so nothing is allocated per launch.  Kernels
// whose result may depend on the order their threads run in are bugs on the GPU; running them in another order here shows them.
struct Order {
    uint64_t a = 1, c = 0, n = 1;
    long at(long k) const { return long((a * uint64_t(k) + c) % n); }
};
Order launch_order(uint64_t n, uint64_t key);   // key: which launch / block / barrier phase (mode 2 mixes it into the seed)
uint64_t next_launch_key();
// runs worker(0) .. worker(n - 1) concurrently, worker(0) on the calling thread.  The other workers are threads that persist across launches:
// a thread per launch would pay thread creation, a fresh TLS block (every kernel's __shared__ arrays) and fresh fiber stacks every time.
void run_workers(int n, void (*worker)(void*), void* arg);
template <typename F> inline void launch(dim3 grid, dim3 block, F body) {
    const long nblocks = long(grid.x) * grid.y * grid.z;
    const unsigned nthreads = block.x * block.y * block.z;
    const uint64_t key = next_launch_key();
    const Order bo = launch_order(uint64_t(nblocks), key * 2), to = launch_order(nthreads, key * 2 + 1);
    std::atomic<long> next{0};
    auto worker = [&]() {
        for (;;) {
            const long b0 = next.fetch_add(4);
            if (b0 >= nblocks) break;
            for (long k = b0; k < b0 + 4 && k < nblocks; ++k) {
                const long b = bo.at(k);
                gridDim = grid; blockDim = block;
                blockIdx.x = unsigned(b % grid.x); blockIdx.y = unsigned((b / grid.x) % grid.y); blockIdx.z = unsigned(b / (long(grid.x) * grid.y));
                for (unsigned j = 0; j < nthreads; ++j) {
                    const unsigned t = unsigned(to.at(j));
                    threadIdx.x = t % block.x; threadIdx.y = (t / block.x) % block.y; threadIdx.z = t / (block.x * block.y);
                    body();
                }
            }
        }
    };
    const int n = (nblocks < 16 || g_serial > 0) ? 1 : num_workers();
    if (n <= 1) { worker(); return; }
    run_workers(n, [](void* w) { (*static_cast<decltype(worker)*>(w))(); }, &worker);
}
// Kernels that use __syncthreads(): every thread of a block runs as a ucontext fiber; a barrier yields to the block
// scheduler, which resumes each unfinished fiber once per barrier phase (in the launch order's sequence; `key` picks the phase's permutation).
void fiber_run_block(unsigned nthreads, dim3 block, void (*thread_body)(void*), void* arg, uint64_t key);
void fiber_barrier();
template <typename F> inline void launch_sync(dim3 grid, dim3 block, F body) {
    const long nblocks = long(grid.x) * grid.y * grid.z;
    const uint64_t key = next_launch_key();
    const Order bo = launch_order(uint64_t(nblocks), key * 2);
    std::atomic<long> next{0};
    auto worker = [&]() {
        for (;;) {
            const long k = next.fetch_add(1);
            if (k >= nblocks) break;
            const long b = bo.at(k);
            gridDim = grid; blockDim = block;
            blockIdx.x = unsigned(b % grid.x); blockIdx.y = unsigned((b / grid.x) % grid.y); blockIdx.z = unsigned(b / (long(grid.x) * grid.y));
            fiber_run_block(block.x * block.y * block.z, block, [](void* p) { (*static_cast<F*>(p))(); }, &body, (key << 24) ^ uint64_t(b));
        }
    };
    const int n = nblocks < 4 ? 1 : num_workers();
    if (n <= 1) { worker(); return; }
    run_workers(n, [](void* w) { (*static_cast<decltype(worker)*>(w))(); }, &worker);
}
}  // namespace kjb_emu
inline void __syncthreads() { kjb_emu::fiber_barrier(); }
