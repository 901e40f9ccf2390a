// b2t_gallery.cu -- DeepSORT's appearance cost on the Hopper tensor cores (sm_90a, wgmma): matching.nearest_embedding_distance
// (matching.py:105-127 with cal_cosine_distance :165-178) for many tracks in one launch.  For each track (slot) t and detection j:
//     out[t][j] = min over the slot's gallery rows g of (1 - g^ . f^),   x^ = x / |x|.
// It is a GEMM (gallery rows x detection rows over the feature axis) with a min-reduction epilogue: the similarity matrix never
// leaves the CTA.
//
// Storage (b2t_gallery_pack): a feature row is normalised once, in float64, scaled by 2^8 and split into two fp16 rows,
//     v = 2^8 x / |x|,  hi = fp16(v),  lo = fp16(v - hi),
// stored as [hi (kpad halves) | lo (kpad halves)], kpad = feat_dim rounded up to 64, zero padded.  The scale keeps lo out of the
// fp16 subnormal range unless |x_i / |x|| < 2^-11 (see the bound below); |v| <= 2^8 cannot overflow fp16.
//
// Kernel: one CTA of two warpgroups per (slot, 128 detection rows).  The slot's gallery is walked in tiles of 128 rows, one m64 half
// per warpgroup, against an N = 128 tile of detection rows.  K is walked in chunks of 64 (one 128-byte swizzled shared-memory row),
// double-buffered with cp.async.  Each chunk is summed by 12 wgmma m64n128k16 (4 k16 steps x hi.hi + hi.lo + lo.hi) into a fresh fp32
// accumulator, and the chunk's sum is then added to a second fp32 register array.  The epilogue forms 1 - 2^-16 s in float64 and
// takes the minimum over the tile's rows (in-thread, across the quad's lanes, then across the 8 warps through shared memory).
//
// Error bound, against D_exact = min_g (1 - u_g . u_f) with u = x / |x| in exact arithmetic on the float32 input rows:
//   * packing: each v_i is within 2^-52 |v_i| of 2^8 u_i; |v_i - hi_i - lo_i| <= 2^-22 |v_i| + 2^-25 (the lo rounding, normal or
//     subnormal), and |lo_i| <= 2^-11 |v_i|.  The dropped lo.lo product and the residuals contribute at most
//     3 * 2^-22 + 2 * 2^-33 sqrt(feat_dim) + 2^-50 to the dot product of unit vectors.
//   * a k16 wgmma adds 16 exact fp16 products to the fp32 accumulator; modelling its alignment and normalisation as truncations
//     (products exact, every term aligned to the largest), one k16 step errs by at most 18 * 2^-23 * max(|acc|, |products|).
//     Within a chunk c every partial sum and product is at most |a_c| |b_c| (1 + 2^-9) in magnitude (Cauchy-Schwarz), so a chunk
//     errs by at most 12 * 18 * 2^-23 |a_c| |b_c| (1 + 2^-9), and the chunks together by 216 * 2^-23 (1 + 2^-9) (Cauchy-Schwarz over
//     chunks, |a| = |b| = 1).
//   * the chunk sums are added in fp32, round to nearest: at most ceil(feat_dim / 64) * 2^-24 (1 + 2^-9).
//   * 1 - 2^-16 s is exact in float64 up to 2^-53; the minimum adds nothing (|min a - min b| <= max |a - b|).
// Together: |out - D_exact| <= B(feat_dim) = (216 * 2^-23 + ceil(feat_dim / 64) * 2^-24) (1 + 2^-9) + 3 * 2^-22
//                                             + 2^-32 sqrt(feat_dim) + 2^-48,
// 2.7e-5 at feat_dim 512 and 2.9e-5 at 2048 (tests/gallery_ref.py restates it; the GPU tests hold the kernel to it).
#include <atomic>
#include <string>
#include <math.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include "b2t_wgmma.cuh"
#include "../../include/b200track.h"

namespace b2t { void set_tracker_error(const char* m); }

namespace {

constexpr int kRows = 128;                       // gallery rows per tile: two m64 warpgroups
constexpr int kCols = 128;                       // detection rows per CTA: the wgmma N
constexpr int kChunk = 64;                       // K chunk: one 128-byte swizzled row of fp16
constexpr int kThreads = 256;
constexpr int kTileBytes = kRows * kChunk * 2;   // 16 KB; the B tile has the same shape (kCols == kRows)
constexpr int kStageBytes = 4 * kTileBytes;      // A hi, A lo, B hi, B lo
constexpr int kSmemBytes = 1024 + 2 * kStageBytes + 8 * kCols * (int)sizeof(double);
constexpr double kScale = 256.0;                 // 2^8; the products carry 2^16

int gfail(int code, const char* m) { b2t::set_tracker_error(m); return code; }
int gcheck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { b2t::set_tracker_error((std::string(what) + ": " + cudaGetErrorString(e)).c_str()); return B2T_ECUDA; }
    return B2T_OK;
}
int kpad_of(int feat_dim) { return (feat_dim + kChunk - 1) / kChunk * kChunk; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int R> __device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// 16 bytes global -> shared, zero-filled when !valid (src-size 0 reads nothing)
__device__ __forceinline__ void cp16(void* dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// the minimum as NumPy's ndarray.min takes it: a NaN (a zero feature row packs to NaN, as the reference's 0 / 0) wins
__device__ __forceinline__ double nan_min(double a, double b) { return (a != a || a < b) ? a : b; }

// one warp per row: v = 2^8 x / |x| in float64 (each float32 square is exact in float64), then the fp16 hi / lo split
__global__ void __launch_bounds__(256) gallery_pack_kernel(const float* __restrict__ x, int n, int D, int kpad, __half* __restrict__ out) {
    const int lane = (int)threadIdx.x & 31;
    const int row = (int)blockIdx.x * 8 + ((int)threadIdx.x >> 5);
    if (row >= n) return;
    const float* xr = x + (size_t)row * D;
    double ss = 0.0;
    for (int k = lane; k < D; k += 32) { const double v = (double)xr[k]; ss += v * v; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const double nrm = sqrt(ss);
    __half* o = out + (size_t)row * 2 * kpad;
    for (int k = lane; k < kpad; k += 32) {
        const double v = k < D ? (double)xr[k] / nrm * kScale : 0.0;
        const __half h = __double2half(v);
        const __half l = __double2half(v - (double)__half2float(h));      // v - hi is exact in float64
        o[k] = h;
        o[kpad + k] = l;
    }
}

// one 128-row x 64-half operand tile (hi or lo part of `rows` packed rows from `src`, rows >= valid zero-filled) into the
// canonical K-major 128-byte-swizzled layout: 16-byte piece q of row r at r * 128 + ((q ^ (r & 7)) << 4) of a 1024-aligned tile
__device__ __forceinline__ void load_tile(uint8_t* tile, const __half* src, size_t row_halves, int valid, int tid) {
#pragma unroll
    for (int i = 0; i < kRows * 8 / kThreads; ++i) {
        const int piece = tid + i * kThreads, r = piece >> 3, q = piece & 7;
        const bool ok = r < valid;
        cp16(tile + r * 128 + ((q ^ (r & 7)) << 4), ok ? src + (size_t)r * row_halves + q * 8 : src, ok);
    }
}

__global__ void __launch_bounds__(kThreads, 1)
gallery_dist_kernel(const __half* __restrict__ gal, const int* __restrict__ counts, int budget, const __half* __restrict__ det, int m,
                    int kpad, double* __restrict__ out, int tiles_c) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    double* red = reinterpret_cast<double*>(smem + 2 * kStageBytes);           // [8 warps][kCols]
    const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
    const int slot = (int)blockIdx.x / tiles_c, c0 = ((int)blockIdx.x % tiles_c) * kCols;
    const int ncols = min(kCols, m - c0);
    int cnt = counts[slot];
    cnt = cnt < 0 ? 0 : (cnt > budget ? budget : cnt);
    const size_t rh = (size_t)2 * kpad;                                         // halves per packed row
    const __half* gslot = gal + (size_t)slot * budget * rh;
    const __half* dtile = det + (size_t)c0 * rh;
    const int chunks = kpad / kChunk;
    // descriptors: {lo: address >> 4 | LBO 1 << 16, hi: SBO 1024 B >> 4 | 128-byte swizzle << 30}; a k16 step is 32 bytes (+2)
    const uint32_t d_hi = (1024u >> 4) | (1u << 30);
    auto desc = [&](const uint8_t* p) { return ((uint64_t)d_hi << 32) | (((smem_u32(p) >> 4) & 0x3fffu) | (1u << 16)); };
    double best = INFINITY;                                                     // threads < kCols: column tid's running minimum
    const int rw = (warp & 3) * 16 + (lane >> 2);                               // first accumulator row of this thread in its m64 half
    for (int r0 = 0; r0 < cnt; r0 += kRows) {
        const int rows = min(kRows, cnt - r0);
        const bool active = 64 * wg < rows;                                     // uniform across the warpgroup
        float sum[kCols / 2], acc[kCols / 2];
#pragma unroll
        for (int i = 0; i < kCols / 2; ++i) sum[i] = 0.f;
        auto load_chunk = [&](int c, int st) {
            uint8_t* s = smem + st * kStageBytes;
            const __half* g = gslot + (size_t)r0 * rh + (size_t)c * kChunk;
            const __half* d = dtile + (size_t)c * kChunk;
            load_tile(s, g, rh, rows, tid);
            load_tile(s + kTileBytes, g + kpad, rh, rows, tid);
            load_tile(s + 2 * kTileBytes, d, rh, ncols, tid);
            load_tile(s + 3 * kTileBytes, d + kpad, rh, ncols, tid);
            cp_commit();
        };
        load_chunk(0, 0);
        for (int c = 0; c < chunks; ++c) {
            if (c + 1 < chunks) { load_chunk(c + 1, (c + 1) & 1); cp_wait<1>(); }
            else cp_wait<0>();
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // cp.async writes -> visible to the wgmma (async proxy)
            __syncthreads();
            if (active) {
                const uint8_t* s = smem + (c & 1) * kStageBytes;
                const uint8_t* a_hi = s + wg * 64 * 128;
                const uint8_t* a_lo = a_hi + kTileBytes;
                const uint8_t* b_hi = s + 2 * kTileBytes;
                const uint8_t* b_lo = s + 3 * kTileBytes;
                acc_fence(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kChunk / 16; ++k) {
                    const uint64_t k2 = 2u * (uint32_t)k;
                    wgmma_m64k16<kCols, true>(acc, desc(a_hi) + k2, desc(b_hi) + k2, k ? 1u : 0u);
                    wgmma_m64k16<kCols, true>(acc, desc(a_hi) + k2, desc(b_lo) + k2, 1u);
                    wgmma_m64k16<kCols, true>(acc, desc(a_lo) + k2, desc(b_hi) + k2, 1u);
                }
                wgmma_commit();
                wgmma_wait0();
                acc_fence(acc);
#pragma unroll
                for (int i = 0; i < kCols / 2; ++i) sum[i] = __fadd_rn(sum[i], acc[i]);
            }
            __syncthreads();                                                    // stage c & 1 is free for chunk c + 2
        }
        // epilogue: thread (warp w, lane l) holds rows rw and rw + 8 of its half, columns 8 j + 2 (l % 4) + e in sum[4 j + 2 h + e]
        const int ra = 64 * wg + rw;
#pragma unroll
        for (int j = 0; j < kCols / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                double v = INFINITY;
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    if (active && ra + 8 * h < rows) v = nan_min(v, 1.0 - (double)sum[4 * j + 2 * h + e] * (1.0 / (kScale * kScale)));
                v = nan_min(v, __shfl_xor_sync(0xffffffffu, v, 4));
                v = nan_min(v, __shfl_xor_sync(0xffffffffu, v, 8));
                v = nan_min(v, __shfl_xor_sync(0xffffffffu, v, 16));
                if (lane < 4) red[warp * kCols + 8 * j + 2 * lane + e] = v;
            }
        __syncthreads();
        if (tid < kCols)
#pragma unroll
            for (int w = 0; w < 8; ++w) best = nan_min(best, red[w * kCols + tid]);
        __syncthreads();
    }
    if (tid < ncols) out[(size_t)slot * m + c0 + tid] = best;
}

}  // namespace

extern "C" int b2t_gallery_row_halves(int feat_dim) { return feat_dim < 1 ? 0 : 2 * kpad_of(feat_dim); }

extern "C" int b2t_gallery_pack(const float* x, int n, int feat_dim, void* packed, void* stream) {
    if (n < 0 || feat_dim < 1 || (n && (!x || !packed)))
        return gfail(B2T_EINVAL, "b2t_gallery_pack: bad arguments");
    if (n == 0) return B2T_OK;
    gallery_pack_kernel<<<(n + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, n, feat_dim, kpad_of(feat_dim), (__half*)packed);
    return gcheck("gallery_pack");
}

extern "C" int b2t_gallery_distance(const void* gallery, const int* counts, int n_slots, int budget, const void* dets, int m, int feat_dim,
                                    double* out, void* stream) {
    if (n_slots < 0 || budget < 1 || m < 0 || feat_dim < 1 || (n_slots && m && (!gallery || !counts || !dets || !out)))
        return gfail(B2T_EINVAL, "b2t_gallery_distance: bad arguments");
    if (((uintptr_t)gallery | (uintptr_t)dets) & 15)
        return gfail(B2T_EINVAL, "b2t_gallery_distance: the packed rows must be 16-byte aligned");
    if (n_slots == 0 || m == 0) return B2T_OK;
    const int tiles_c = (m + kCols - 1) / kCols;
    if ((double)n_slots * tiles_c > 2147483647.0)
        return gfail(B2T_EINVAL, "b2t_gallery_distance: too many tiles for one launch");
    // the shared-memory opt-in is a per-device attribute: set once per device (setting it twice from two threads is harmless)
    static std::atomic<bool> attr_set[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return gcheck("gallery_distance (device)");
    if (dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        if (cudaFuncSetAttribute(gallery_dist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes) != cudaSuccess)
            return gcheck("gallery_distance (shared memory)");
        if (dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    gallery_dist_kernel<<<n_slots * tiles_c, kThreads, kSmemBytes, (cudaStream_t)stream>>>(
        (const __half*)gallery, counts, budget, (const __half*)dets, m, kpad_of(feat_dim), out, tiles_c);
    return gcheck("gallery_distance");
}
