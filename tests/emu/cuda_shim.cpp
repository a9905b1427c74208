// TEST INFRASTRUCTURE ONLY (see cuda_shim.h)
#include "cuda_shim.h"
#include <condition_variable>
#include <mutex>
#include <pthread.h>
thread_local kjb_emu::Idx threadIdx, blockIdx;
thread_local dim3 blockDim, gridDim;
int kjb_emu::g_serial = 0;
int kjb_emu::num_workers() { static int n = [] { const char* e = getenv("KJB_EMU_THREADS"); int v = e ? atoi(e) : int(std::thread::hardware_concurrency()); return v < 1 ? 1 : v; }(); return n; }

namespace {
std::atomic<int> g_order_mode{0};
std::atomic<uint32_t> g_order_seed{0};
std::atomic<uint64_t> g_launches{0};
uint64_t mix64(uint64_t x) {   // splitmix64 finaliser
    x += 0x9e3779b97f4a7c15ull;
    x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull; x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
uint64_t gcd(uint64_t a, uint64_t b) { while (b) { const uint64_t t = a % b; a = b; b = t; } return a; }
struct WorkerPool {   // never destroyed: its threads wait for the next launch until the process ends
    std::mutex launch_m, m;
    std::condition_variable start, done;
    std::vector<std::thread> threads;
    void (*fn)(void*) = nullptr; void* arg = nullptr;
    int participants = 0, remaining = 0; uint64_t generation = 0;
    void loop(int idx) {
        for (uint64_t seen = 0;;) {
            void (*f)(void*); void* a;
            {
                std::unique_lock<std::mutex> l(m);
                start.wait(l, [&] { return generation != seen; });
                seen = generation;
                if (idx >= participants) continue;
                f = fn; a = arg;
            }
            f(a);
            std::lock_guard<std::mutex> l(m);
            if (--remaining == 0) done.notify_one();
        }
    }
    void run(int n, void (*f)(void*), void* a) {
        std::lock_guard<std::mutex> one_launch_at_a_time(launch_m);
        while (int(threads.size()) < n - 1) { const int idx = int(threads.size()) + 1; threads.emplace_back([this, idx] { loop(idx); }); threads.back().detach(); }
        { std::lock_guard<std::mutex> l(m); fn = f; arg = a; participants = n; remaining = n - 1; ++generation; }
        start.notify_all();
        f(a);
        std::unique_lock<std::mutex> l(m);
        done.wait(l, [&] { return remaining == 0; });
    }
};
WorkerPool* g_pool = [] {
    pthread_atfork(nullptr, nullptr, [] { g_pool = new WorkerPool; });   // a forked child has none of the parent's workers: start over
    return new WorkerPool;
}();
}
void kjb_emu::run_workers(int n, void (*worker)(void*), void* arg) { g_pool->run(n, worker, arg); }
uint64_t kjb_emu::next_launch_key() { return g_launches.fetch_add(1, std::memory_order_relaxed); }
kjb_emu::Order kjb_emu::launch_order(uint64_t n, uint64_t key) {
    Order o; o.n = n ? n : 1;
    const int mode = g_order_mode.load(std::memory_order_relaxed);
    if (o.n < 2 || mode == 0) return o;
    if (mode == 1) { o.a = o.n - 1; o.c = o.n - 1; return o; }   // (n-1) * k + n-1 = n-1-k (mod n)
    const uint64_t h = mix64(key ^ mix64(g_order_seed.load(std::memory_order_relaxed)));
    o.a = h % o.n;
    while (o.a == 0 || gcd(o.a, o.n) != 1) o.a = (o.a + 1) % o.n;
    o.c = mix64(h) % o.n;
    return o;
}
// mode: 0 = forward (the default), 1 = reverse, 2 = a permutation per launch, block and barrier phase derived from `seed` and a launch
// counter, which this call resets (the same mode and seed replay the same orders)
extern "C" void kjb_emu_set_launch_order(int mode, uint32_t seed) {
    g_order_mode.store(mode == 1 || mode == 2 ? mode : 0); g_order_seed.store(seed); g_launches.store(0);
}

#include <ucontext.h>
#include <memory>
namespace {
// Fiber switches.  swapcontext saves and restores the signal mask with a system call at every switch, and a frame switches millions of
// times; on hosts where system calls are slow that dominates the emulator.  A switch only has to keep the callee-saved registers, the
// stack pointer and the FP control words (SysV x86-64), which a dozen instructions do.  AddressSanitizer builds keep ucontext, which it
// knows how to follow.
#if defined(__SANITIZE_ADDRESS__)
using Ctx = ucontext_t;
void ctx_start(Ctx& c, char* stack, size_t size, void (*entry)()) {
    getcontext(&c); c.uc_stack.ss_sp = stack; c.uc_stack.ss_size = size; c.uc_link = nullptr; makecontext(&c, entry, 0);
}
void ctx_switch(Ctx& from, Ctx& to) { swapcontext(&from, &to); }
#else
struct Ctx { void* sp = nullptr; };
extern "C" void kjb_emu_fiber_switch(void** save_sp, void* to_sp);
asm(R"(
    .text
    .p2align 4
    .globl kjb_emu_fiber_switch
    .hidden kjb_emu_fiber_switch
    .type kjb_emu_fiber_switch, @function
kjb_emu_fiber_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    subq $8, %rsp
    stmxcsr (%rsp)
    fnstcw 4(%rsp)
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    ldmxcsr (%rsp)
    fldcw 4(%rsp)
    addq $8, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
    .size kjb_emu_fiber_switch, .-kjb_emu_fiber_switch
)");
void ctx_start(Ctx& c, char* stack, size_t size, void (*entry)()) {
    // the frame kjb_emu_fiber_switch pops: FP control words, six registers, then `entry` as the return address; `entry` starts with the
    // stack 8 bytes below a 16-byte boundary, as after a call
    uintptr_t top = (reinterpret_cast<uintptr_t>(stack) + size) & ~uintptr_t(15);
    uint64_t* p = reinterpret_cast<uint64_t*>(top);
    *--p = 0;                                      // the return address `entry` never uses
    *--p = reinterpret_cast<uint64_t>(entry);
    for (int i = 0; i < 6; ++i) *--p = 0;          // rbp rbx r12 r13 r14 r15
    *--p = uint64_t(0x1F80) | uint64_t(0x037F) << 32;   // MXCSR and x87 control word at their defaults
    c.sp = p;
}
void ctx_switch(Ctx& from, Ctx& to) { kjb_emu_fiber_switch(&from.sp, to.sp); }
#endif
struct Fiber { Ctx ctx; std::unique_ptr<char[]> stack; bool done = true; };
struct BlockState {
    std::vector<Fiber> fibers; Ctx sched; unsigned cur = 0;
    void (*body)(void*) = nullptr; void* arg = nullptr;
};
thread_local BlockState* g_block = nullptr;
const size_t STACK = 256 * 1024;
void trampoline() {
    BlockState* b = g_block;
    b->body(b->arg);
    b->fibers[b->cur].done = true;
    ctx_switch(b->fibers[b->cur].ctx, b->sched);
}
}
void kjb_emu::fiber_barrier() { BlockState* b = g_block; ctx_switch(b->fibers[b->cur].ctx, b->sched); }
void kjb_emu::fiber_run_block(unsigned nthreads, dim3 block, void (*thread_body)(void*), void* arg, uint64_t key) {
    static thread_local BlockState state;
    BlockState& b = state; g_block = &b; b.body = thread_body; b.arg = arg;
    if (b.fibers.size() < nthreads) { b.fibers.resize(nthreads); for (auto& f : b.fibers) if (!f.stack) f.stack.reset(new char[STACK]); }
    for (unsigned t = 0; t < nthreads; ++t) {
        Fiber& f = b.fibers[t];
        ctx_start(f.ctx, f.stack.get(), STACK, trampoline); f.done = false;
    }
    const uint64_t block_key = mix64(key);
    for (uint64_t phase = 0, any = 1; any; ++phase) {   // one round per barrier phase
        any = 0;
        const Order o = launch_order(nthreads, block_key + phase);
        for (unsigned j = 0; j < nthreads; ++j) {
            const unsigned t = unsigned(o.at(j));
            if (b.fibers[t].done) continue;
            any = 1; b.cur = t;
            threadIdx.x = t % block.x; threadIdx.y = (t / block.x) % block.y; threadIdx.z = t / (block.x * block.y);
            ctx_switch(b.sched, b.fibers[t].ctx);
        }
    }
}
