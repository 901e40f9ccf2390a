// tests/hostsim/cuda_sim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT (see cuda_sim.h).
#include "cuda_sim.h"

namespace sim {
State g;

// x86-64 SysV context switch: save callee-saved registers on the current stack, publish sp,
// adopt the target stack, restore, return into the target.
__asm__(R"(
.text
.globl sim_switch
.type sim_switch,@function
sim_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size sim_switch,.-sim_switch
)");

static const size_t kStack = 256 * 1024;
static std::vector<char*> stack_pool;

static bool runnable(int i) {
    Fiber& f = g.fibers[i];
    if (f.done) return false;
    if (f.wait_block) { if (g.gen == f.block_gen) return false; f.wait_block = false; }
    if (f.wait_warp) { if (g.warps[i >> 5].gen == f.warp_gen) return false; f.wait_warp = false; }
    return true;
}

void yield_to_next() {
    int from = g.cur;
    int n = g.nthreads;
    for (int k = 1; k <= n; ++k) {
        int i = from + k; if (i >= n) i -= n;
        if (runnable(i)) {
            if (i == from) return;
            g.cur = i; g.switches++;
            sim_switch(&g.fibers[from].sp, g.fibers[i].sp);
            return;
        }
    }
    if (g.live == 0) { sim_switch(&g.fibers[from].sp, g.sched_sp); return; }
    fprintf(stderr, "hostsim: deadlock in block %u (thread %d): %d live threads, barrier arrived %d\n",
            g.block_idx.x, from, g.live, g.arrived);
    abort();
}

static void trampoline() {
    g.body(g.body_arg);
    Fiber& f = g.fibers[g.cur];
    f.done = true;
    g.live--;
    Warp& w = g.warps[g.cur >> 5];
    w.live--;
    if (g.live > 0 && g.arrived == g.live) { g.arrived = 0; g.gen++; }
    if (w.live > 0 && w.arrived == w.live) { w.arrived = 0; w.gen++; }
    yield_to_next();
    abort();  // unreachable
}

void run_block(int nthreads) {
    if (nthreads % 32 != 0) { fprintf(stderr, "hostsim: blockDim must be a multiple of 32\n"); abort(); }
    g.nthreads = nthreads; g.live = nthreads; g.arrived = 0; g.gen = 0;
    g.fibers.assign(nthreads, Fiber());
    g.warps.assign(nthreads / 32, Warp());
    while ((int)stack_pool.size() < nthreads) stack_pool.push_back((char*)aligned_alloc(64, kStack));
    for (int i = 0; i < nthreads; ++i) {
        Fiber& f = g.fibers[i];
        f.tid = i; f.stack = stack_pool[i];
        g.warps[i >> 5].live++;
        uintptr_t top = (reinterpret_cast<uintptr_t>(f.stack) + kStack) & ~uintptr_t(15);
        void** sp = reinterpret_cast<void**>(top);
        *--sp = nullptr;                                   // fake return address of trampoline
        *--sp = reinterpret_cast<void*>(&trampoline);      // popped by `ret` in sim_switch
        for (int r = 0; r < 6; ++r) *--sp = nullptr;       // rbp rbx r12 r13 r14 r15
        f.sp = sp;
    }
    g.cur = 0;
    sim_switch(&g.sched_sp, g.fibers[0].sp);
}
}  // namespace sim

// the 16-bit conversions of cuda_sim.h, exported for tests/test_hostsim_reid.py (checked against NumPy / torch there)
extern "C" void b2t_sim_to16(const double* in, unsigned short* out, long long n, int bf16) {
    for (long long i = 0; i < n; ++i) out[i] = bf16 ? __double2bfloat16(in[i]).x : __double2half(in[i]).x;
}
extern "C" void b2t_sim_f32_to16(const float* in, unsigned short* out, long long n, int bf16) {
    for (long long i = 0; i < n; ++i) out[i] = bf16 ? __float2bfloat16_rn(in[i]).x : __float2half_rn(in[i]).x;
}
extern "C" void b2t_sim_from16(const unsigned short* in, float* out, long long n, int bf16) {
    for (long long i = 0; i < n; ++i) {
        if (bf16) { __nv_bfloat16 h; h.x = in[i]; out[i] = __bfloat162float(h); }
        else { __half h; h.x = in[i]; out[i] = __half2float(h); }
    }
}
