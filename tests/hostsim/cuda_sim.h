// tests/hostsim/cuda_sim.h -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// A single-OS-thread, fiber-per-CUDA-thread simulator for ONE thread block at a time.  It exists
// because the build container has no GPU: the tracker kernels (csrc/b2t_*.cuh) are compiled a
// second time with g++ against this header so that their control flow, barriers, warp shuffles
// and shared-memory indexing can be checked bit-for-bit against the oracle in the `not gpu` test
// tier.  The product (libb200track.so, built by nvcc) never includes this file and the Python
// package never loads the simulator library; GPU results are what the `-m gpu` tier checks.
//
// Supported: threadIdx/blockIdx/blockDim/gridDim (.x only), static + dynamic __shared__,
// __syncthreads, __syncwarp, full-mask __shfl*_sync / __ballot_sync / __any_sync / __all_sync /
// __match_any_sync, integer + fp atomics (fp64 included), software __half / __nv_bfloat16 conversions, and a handful of
// cudaMemcpy-style host calls.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>
#include <algorithm>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __constant__ static const
#define __align__(n) __attribute__((aligned(n)))

struct sim_dim3 { unsigned x, y, z; sim_dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
typedef sim_dim3 dim3;
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };

namespace sim {

struct Fiber {
    void* sp = nullptr;
    char* stack = nullptr;
    int tid = 0;
    bool done = false;
    bool wait_block = false; unsigned block_gen = 0;
    bool wait_warp = false;  unsigned warp_gen = 0;
};
struct Warp { uint64_t slot[32]; int arrived = 0; unsigned gen = 0; int live = 0; };

struct State {
    std::vector<Fiber> fibers;
    std::vector<Warp> warps;
    void* sched_sp = nullptr;
    int cur = 0;
    int nthreads = 0;
    int live = 0;
    int arrived = 0; unsigned gen = 0;
    sim_dim3 block_idx, block_dim, grid_dim;
    unsigned char* dyn_smem = nullptr;
    void (*body)(void*) = nullptr; void* body_arg = nullptr;
    unsigned long switches = 0;
};
extern State g;

extern "C" void sim_switch(void** from_sp, void* to_sp);
void run_block(int nthreads);
void yield_to_next();

inline Fiber& me() { return g.fibers[g.cur]; }
inline Warp& my_warp() { return g.warps[g.cur >> 5]; }

inline void warp_barrier() {
    Warp& w = my_warp();
    unsigned my_gen = w.gen;
    if (++w.arrived == w.live) { w.arrived = 0; w.gen++; return; }
    Fiber& f = me(); f.wait_warp = true; f.warp_gen = my_gen;
    yield_to_next();
}
inline void block_barrier() {
    unsigned my_gen = g.gen;
    if (++g.arrived == g.live) { g.arrived = 0; g.gen++; return; }
    Fiber& f = me(); f.wait_block = true; f.block_gen = my_gen;
    yield_to_next();
}
inline void check_mask(unsigned mask) {
    if (mask != 0xffffffffu) { fprintf(stderr, "hostsim: only full-mask warp collectives are supported\n"); abort(); }
}
template <class T> inline uint64_t to_bits(T v) { uint64_t b = 0; static_assert(sizeof(T) <= 8, ""); memcpy(&b, &v, sizeof(T)); return b; }
template <class T> inline T from_bits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }

template <class T> inline T shfl_from(unsigned mask, T v, int src_lane_abs) {
    check_mask(mask);
    Warp& w = my_warp();
    w.slot[g.cur & 31] = to_bits(v);
    warp_barrier();
    T r = from_bits<T>(w.slot[src_lane_abs & 31]);
    warp_barrier();
    return r;
}

template <class F> struct Thunk { static void call(void* p) { (*static_cast<F*>(p))(); } };

template <class F> inline void launch(sim_dim3 grid, sim_dim3 block, size_t smem, F&& f) {
    std::vector<unsigned char> dyn(smem + 1024);
    unsigned char* base = dyn.data();
    base += (1024 - (reinterpret_cast<uintptr_t>(base) & 1023)) & 1023;
    g.dyn_smem = base;
    g.grid_dim = grid; g.block_dim = block;
    typedef typename std::remove_reference<F>::type FT;
    g.body = &Thunk<FT>::call; g.body_arg = (void*)&f;
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                g.block_idx.x = bx; g.block_idx.y = by; g.block_idx.z = bz;
                memset(base, 0xCD, smem);   // poison: uninitialised shared memory reads show up
                run_block((int)block.x);
            }
}
}  // namespace sim

#define threadIdx (sim_dim3((unsigned)sim::g.cur, 0, 0))
#define blockIdx (sim::g.block_idx)
#define blockDim (sim::g.block_dim)
#define gridDim (sim::g.grid_dim)
#define warpSize 32

inline void __syncthreads() { sim::block_barrier(); }
inline void __syncwarp(unsigned mask = 0xffffffffu) { sim::check_mask(mask); sim::warp_barrier(); }
inline void __threadfence_block() {}
inline void __threadfence() {}

template <class T> inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    int lane = sim::g.cur & 31;
    int base = lane & ~(width - 1);
    return sim::shfl_from(mask, v, base + (src & (width - 1)));
}
template <class T> inline T __shfl_xor_sync(unsigned mask, T v, int lane_mask, int width = 32) {
    int lane = sim::g.cur & 31;
    int src = lane ^ lane_mask;
    if ((src & ~(width - 1)) != (lane & ~(width - 1))) src = lane;
    return sim::shfl_from(mask, v, src);
}
template <class T> inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    int lane = sim::g.cur & 31;
    int src = lane - (int)delta;
    if (src < (lane & ~(width - 1))) src = lane;
    return sim::shfl_from(mask, v, src);
}
template <class T> inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    int lane = sim::g.cur & 31;
    int src = lane + (int)delta;
    if (src > (lane | (width - 1))) src = lane;
    return sim::shfl_from(mask, v, src);
}
inline unsigned __ballot_sync(unsigned mask, int pred) {
    sim::check_mask(mask);
    sim::Warp& w = sim::my_warp();
    w.slot[sim::g.cur & 31] = pred ? 1 : 0;
    sim::warp_barrier();
    unsigned r = 0;
    for (int i = 0; i < 32; ++i) if (w.slot[i]) r |= 1u << i;
    sim::warp_barrier();
    return r;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) == 0xffffffffu; }
template <class T> inline unsigned __match_any_sync(unsigned mask, T v) {
    sim::check_mask(mask);
    sim::Warp& w = sim::my_warp();
    w.slot[sim::g.cur & 31] = sim::to_bits(v);
    sim::warp_barrier();
    unsigned r = 0; uint64_t mine = sim::to_bits(v);
    for (int i = 0; i < 32; ++i) if (w.slot[i] == mine) r |= 1u << i;
    sim::warp_barrier();
    return r;
}
inline unsigned __reduce_min_sync(unsigned mask, unsigned v) {
    sim::check_mask(mask);
    sim::Warp& w = sim::my_warp();
    w.slot[sim::g.cur & 31] = v;
    sim::warp_barrier();
    unsigned r = 0xffffffffu;
    for (int i = 0; i < 32; ++i) if ((unsigned)w.slot[i] < r) r = (unsigned)w.slot[i];
    sim::warp_barrier();
    return r;
}
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
template <class T> inline T __ldg(const T* p) { return *p; }

template <class T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T> inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <class T> inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> inline T atomicCAS(T* p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }

inline int __float2int_rn(float v) { return (int)lrintf(v); }      // round to nearest even (default FP environment)
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
struct float4 { float x, y, z, w; };
struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
inline float4 make_float4(float x, float y, float z, float w) { float4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
inline float __int_as_float(int v) { return sim::from_bits<float>((uint64_t)(uint32_t)v); }
inline int __float_as_int(float v) { return (int)(uint32_t)sim::to_bits(v); }

// ---- 16-bit floating point (cuda_fp16.h / cuda_bf16.h subset) in software: IEEE binary16 and bfloat16 bit patterns, conversions
// rounded to nearest even straight from the (exact) float / double value, subnormals and overflow to infinity included.
struct __half { unsigned short x; };
struct __nv_bfloat16 { unsigned short x; };
namespace sim {
// round |v| to a binary format with `mant` stored significand bits and `expb` exponent bits -> bit pattern (sign included)
inline unsigned short round16(double v, int mant, int expb) {
    const unsigned sign = std::signbit(v) ? 1u << (mant + expb) : 0u;
    const unsigned inf = ((1u << expb) - 1u) << mant;
    if (std::isnan(v)) return (unsigned short)(sign | inf | (1u << (mant - 1)));
    const double a = std::fabs(v);
    if (std::isinf(a)) return (unsigned short)(sign | inf);
    if (a == 0.0) return (unsigned short)sign;
    const int bias = (1 << (expb - 1)) - 1, emin = 1 - bias;
    int e;
    std::frexp(a, &e);
    int E = e - 1;                                          // a in [2^E, 2^(E+1))
    if (E < emin) E = emin;                                 // subnormal range: fixed quantum 2^(emin - mant)
    const double r = std::nearbyint(std::ldexp(a, mant - E)); // significand with `mant` fraction bits, rounded to nearest even
    // ((E + bias - 1) << mant) + r: a subnormal when E == emin and r < 2^mant, and a carry out of the significand bumps the exponent
    const double bits = std::ldexp((double)(E + bias - 1), mant) + r;
    if (bits >= (double)inf) return (unsigned short)(sign | inf);
    return (unsigned short)(sign | (unsigned)bits);
}
inline double widen16(unsigned short b, int mant, int expb) {
    const int bias = (1 << (expb - 1)) - 1;
    const unsigned m = b & ((1u << mant) - 1u), ex = (b >> mant) & ((1u << expb) - 1u);
    const double sgn = (b >> (mant + expb)) & 1u ? -1.0 : 1.0;
    if (ex == (1u << expb) - 1u) return m ? (double)NAN : sgn * (double)INFINITY;
    if (ex == 0) return sgn * std::ldexp((double)m, 1 - bias - mant);
    return sgn * std::ldexp((double)(m | (1u << mant)), (int)ex - bias - mant);
}
}  // namespace sim
inline __half __double2half(double v) { __half h; h.x = sim::round16(v, 10, 5); return h; }
inline __half __float2half_rn(float v) { return __double2half((double)v); }
inline float __half2float(__half h) { return (float)sim::widen16(h.x, 10, 5); }
inline __nv_bfloat16 __double2bfloat16(double v) { __nv_bfloat16 h; h.x = sim::round16(v, 7, 8); return h; }
inline __nv_bfloat16 __float2bfloat16_rn(float v) { return __double2bfloat16((double)v); }
inline float __bfloat162float(__nv_bfloat16 h) { return (float)sim::widen16(h.x, 7, 8); }

// ---- host runtime shims (device memory == host memory) ----
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = malloc(n ? n : 1); return *p ? 0 : 2; }
inline cudaError_t cudaFree(void* p) { free(p); return 0; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = 0) { memcpy(d, s, n); return 0; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return 0; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = 0) { memset(d, v, n); return 0; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
inline cudaError_t cudaDeviceSynchronize() { return 0; }
inline cudaError_t cudaGetLastError() { return 0; }
inline cudaError_t cudaPeekAtLastError() { return 0; }
inline const char* cudaGetErrorString(cudaError_t) { return "hostsim"; }
