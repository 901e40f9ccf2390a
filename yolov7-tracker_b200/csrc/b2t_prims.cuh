// b2t_prims.cuh -- warp / block building blocks shared by the tracker kernels.
#pragma once
#include <string.h>
#include "b2t_platform.cuh"

namespace b2t {

B2T_DEV int lane_id() { return (int)(threadIdx.x & 31u); }
B2T_DEV int warp_id() { return (int)(threadIdx.x >> 5); }
B2T_DEV int num_warps() { return (int)(blockDim.x >> 5); }
B2T_DEV unsigned lanemask_lt() { return (1u << lane_id()) - 1u; }

template <class T> B2T_DEV T shfl(T v, int src, int width = 32) { return __shfl_sync(B2T_FULL, v, src, width); }
template <class T> B2T_DEV T shfl_up(T v, int d) { return __shfl_up_sync(B2T_FULL, v, (unsigned)d); }
template <class T> B2T_DEV T shfl_xor(T v, int m, int width = 32) { return __shfl_xor_sync(B2T_FULL, v, m, width); }

template <class T> struct Inf;
template <> struct Inf<float> { B2T_DEV static float v() { return __int_as_float(0x7f800000); } };
template <> struct Inf<double> { B2T_DEV static double v() { return 1.0e300 * 1.0e300; } };

// Warp arg-min of (value, index) pairs; lanes without a candidate pass idx < 0.  Smallest value wins,
// ties go to the smaller index.  Values are mapped to order-preserving unsigned keys and reduced with
// __reduce_min_sync (REDUX): 2-3 reductions instead of a 5-step shuffle ladder of 64-bit values.
B2T_DEV unsigned int ordkey(float v) { unsigned int k; memcpy(&k, &v, 4); return (k & 0x80000000u) ? ~k : (k | 0x80000000u); }
B2T_DEV unsigned long long ordkey(double v) {
    unsigned long long k; memcpy(&k, &v, 8);
    return (k & 0x8000000000000000ull) ? ~k : (k | 0x8000000000000000ull);
}
B2T_DEV int warp_argmin(float v, int idx, float* vmin) {
    const unsigned key = idx >= 0 ? ordkey(v) : 0xffffffffu;
    const unsigned kmin = __reduce_min_sync(B2T_FULL, key);
    const unsigned imin = __reduce_min_sync(B2T_FULL, (idx >= 0 && key == kmin) ? (unsigned)idx : 0xffffffffu);
    if (imin == 0xffffffffu) return -1;
    const unsigned src = __ballot_sync(B2T_FULL, idx >= 0 && key == kmin && (unsigned)idx == imin);
    *vmin = __shfl_sync(B2T_FULL, v, __ffs((int)src) - 1);
    return (int)imin;
}
B2T_DEV int warp_argmin(double v, int idx, double* vmin) {
    const unsigned long long key = idx >= 0 ? ordkey(v) : ~0ull;
    const unsigned hi = (unsigned)(key >> 32), lo = (unsigned)key;
    const unsigned hmin = __reduce_min_sync(B2T_FULL, hi);
    const unsigned lmin = __reduce_min_sync(B2T_FULL, hi == hmin ? lo : 0xffffffffu);
    const bool best = idx >= 0 && hi == hmin && lo == lmin;
    const unsigned imin = __reduce_min_sync(B2T_FULL, best ? (unsigned)idx : 0xffffffffu);
    if (imin == 0xffffffffu) return -1;
    const unsigned src = __ballot_sync(B2T_FULL, best && (unsigned)idx == imin);
    *vmin = __shfl_sync(B2T_FULL, v, __ffs((int)src) - 1);
    return (int)imin;
}

// Bump allocator over the dynamic shared memory block.  Every thread performs the same
// arithmetic, so no synchronisation is involved.
struct Arena {
    unsigned char* base;
    size_t off;
    B2T_DEV Arena(unsigned char* b) : base(b), off(0) {}
    template <class T> B2T_DEV T* take(int n) {
        off = (off + 15) & ~size_t(15);
        T* p = reinterpret_cast<T*>(base + off);
        off += sizeof(T) * (size_t)(n > 0 ? n : 1);
        return p;
    }
};
// Arena over no memory, for sizing a launch: a carve run on it hands out Arena's offsets as pointers and leaves the total in off.
struct ArenaSize {
    size_t off = 0;
    template <class T> B2T_HD T* take(int n) {
        off = (off + 15) & ~size_t(15);
        T* p = reinterpret_cast<T*>(off);
        off += sizeof(T) * (size_t)(n > 0 ? n : 1);
        return p;
    }
};

// In-place exclusive scan of a[0..n) (shared memory), all threads of the CTA participate.
// scratch: >= 33 ints of shared memory.  Returns the total.
B2T_DEV int block_exscan(int* a, int n, int* scratch) {
    const int tid = (int)threadIdx.x, nt = (int)blockDim.x;
    const int per = (n + nt - 1) / nt;
    int s = tid * per, e = s + per;
    if (s > n) s = n;
    if (e > n) e = n;
    int sum = 0;
    for (int i = s; i < e; ++i) sum += a[i];
    int inc = sum;
    for (int d = 1; d < 32; d <<= 1) {
        int t = shfl_up(inc, d);
        if (lane_id() >= d) inc += t;
    }
    if (lane_id() == 31) scratch[warp_id()] = inc;
    __syncthreads();
    if (warp_id() == 0) {
        int w = lane_id() < num_warps() ? scratch[lane_id()] : 0;
        int winc = w;
        for (int d = 1; d < 32; d <<= 1) {
            int t = shfl_up(winc, d);
            if (lane_id() >= d) winc += t;
        }
        scratch[lane_id()] = winc - w;
        if (lane_id() == 31) scratch[32] = winc;
    }
    __syncthreads();
    int base = scratch[warp_id()] + inc - sum;
    for (int i = s; i < e; ++i) { int t = a[i]; a[i] = base; base += t; }
    int total = scratch[32];
    __syncthreads();
    return total;
}

// Order-preserving compaction: out[] receives every i in [0, n) with pred(i), ascending.
// All threads participate; scratch: >= 32 ints.  Returns the count (uniform).
template <class Pred> B2T_DEV int block_compact(int n, Pred pred, int* out, int* scratch) {
    const int tid = (int)threadIdx.x, nt = (int)blockDim.x;
    const int lane = lane_id(), wid = warp_id(), nw = num_warps();
    int base = 0;
    for (int c0 = 0; c0 < n; c0 += nt) {
        const int i = c0 + tid;
        const bool p = (i < n) && pred(i);
        const unsigned bal = __ballot_sync(B2T_FULL, p);
        if (lane == 0) scratch[wid] = __popc(bal);
        __syncthreads();
        // every warp scans the (<= 32) per-warp counts with shuffles
        const int cnt = lane < nw ? scratch[lane] : 0;
        int inc = cnt;
        for (int d = 1; d < 32; d <<= 1) { const int t = shfl_up(inc, d); if (lane >= d) inc += t; }
        const int woff = shfl(inc - cnt, wid);
        const int tot = shfl(inc, 31);
        if (p) out[base + woff + __popc(bal & lanemask_lt())] = i;
        base += tot;
        __syncthreads();
    }
    return base;
}

}  // namespace b2t
