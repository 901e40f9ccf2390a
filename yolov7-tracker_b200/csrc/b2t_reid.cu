// b2t_reid.cu -- glue kernels of the appearance branch (SURVEY.md section 8f row 3): everything of the reference's ReID extractor
// (tracker/reid_models/deepsort_reid.py:63-153) that is not a convolution.  The 3x3 / 1x1 convolutions (+ folded BatchNorm + ReLU) run on
// the wgmma kernel of b2t_conv.cu; these kernels are the byte / element-wise work around them -- HBM-bound, 16-byte vectors.
//   reid_crop_kernel       Extractor._preprocess :134-146: crop.astype(float32) / 255 -> cv2.resize to 64 x 128 (bilinear, float) ->
//                          ToTensor -> Normalize(mean, std); written as NHWC 16-bit with the 3 channels padded to 16 (tensor-core K granularity)
//   maxpool3x3s2_kernel    nn.MaxPool2d(3, 2, padding=1) :72
//   add_relu_kernel        BasicBlock.forward :49 F.relu(x.add(y))
//   avgpool_l2norm_kernel  nn.AvgPool2d((8, 4), 1) :83 + x.div(x.norm(p=2, dim=1)) :103-104 -> 512 floats per crop
// and, for many sequences in one extractor pass (TrackingPipeline with ReID):
//   reid_crop_list_kernel  botsort.py:339-346 per sequence: the det_high rows of the NMS output -> crop descriptors, segment offsets, row map
//   bn_*_seg_kernel        batch-statistics BatchNorm with the statistics of each sequence's crops only (each segment as bn_*_kernel alone)
//   avgpool_l2norm_rows_kernel  the pooled features of crop j straight into the tracker's [sequence][dmax][512] row rowmap[j]
#include <string>          // before b2t_platform.cuh (the simulator's __noinline__ macro must not reach libstdc++)
#include <math.h>
#include "b2t_platform.cuh"
#if !defined(B2T_HOSTSIM)
#include <cuda_fp16.h>                // the host simulator brings its own __half / __nv_bfloat16 (tests/hostsim/cuda_sim.h)
#include <cuda_bf16.h>
#endif
#include "../../include/b200track.h"

namespace b2t { void set_detect_error(const char* m); }

namespace {

int rfail(int code, const char* m) { b2t::set_detect_error(m); return code; }
int rcheck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { b2t::set_detect_error((std::string(what) + ": " + cudaGetErrorString(e)).c_str()); return B2T_ECUDA; }
    return B2T_OK;
}
int grid_for(long long total, int block) { long long g = (total + block - 1) / block; return (int)(g > 132 * 16 ? 132 * 16 : (g < 1 ? 1 : g)); }

__device__ __forceinline__ float load16(const unsigned short* p, int f16) {
    return f16 ? __half2float(*reinterpret_cast<const __half*>(p)) : __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(p));
}
__device__ __forceinline__ unsigned short store16(float v, int f16) {
    if (f16) { const __half h = __float2half_rn(v); return *reinterpret_cast<const unsigned short*>(&h); }
    const __nv_bfloat16 h = __float2bfloat16_rn(v); return *reinterpret_cast<const unsigned short*>(&h);
}

// cv2.resize(float32 image, (64, 128)), INTER_LINEAR: source coordinate (float)((d + 0.5) * scale - 0.5), left tap floor(), the
// weight zeroed and the tap clamped at both edges; value = (S[x0] * (1 - fx) + S[x1] * fx) per row, then rows blended the same way.
__device__ __forceinline__ void tap(int d, double scale, int src, int& s0, int& s1, float& f) {
    f = (float)((d + 0.5) * scale - 0.5);
    s0 = (int)floorf(f);
    f -= (float)s0;
    if (s0 < 0) { f = 0.f; s0 = 0; }
    if (s0 >= src - 1) { f = 0.f; s0 = src - 1; }
    s1 = s0 + 1 < src ? s0 + 1 : src - 1;
}

// crops[i] = {byte offset of the crop's first pixel in `pixels`, row pitch in bytes, height, width}
__global__ void reid_crop_kernel(const unsigned char* __restrict__ pixels, const long long* __restrict__ crops, int n, unsigned short* __restrict__ out, int f16) {
    const int total = n * 128 * 64;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int x = i & 63, y = (i >> 6) & 127, c = i >> 13;
        const long long* cr = crops + (size_t)c * 4;
        const unsigned char* img = pixels + cr[0];
        const int pitch = (int)cr[1], h = (int)cr[2], w = (int)cr[3];
        int x0, x1, y0, y1; float fx, fy;
        tap(x, 1.0 / (64.0 / (double)w), w, x0, x1, fx);
        tap(y, 1.0 / (128.0 / (double)h), h, y0, y1, fy);
        const unsigned char* r0 = img + (size_t)y0 * pitch;
        const unsigned char* r1 = img + (size_t)y1 * pitch;
        union { unsigned short o[16]; uint4 v[2]; } px;
        const float mean[3] = {0.485f, 0.456f, 0.406f}, sd[3] = {0.229f, 0.224f, 0.225f};
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const float a0 = (float)r0[x0 * 3 + ch] / 255.0f, a1 = (float)r0[x1 * 3 + ch] / 255.0f;
            const float b0 = (float)r1[x0 * 3 + ch] / 255.0f, b1 = (float)r1[x1 * 3 + ch] / 255.0f;
            const float top = a0 * (1.f - fx) + a1 * fx, bot = b0 * (1.f - fx) + b1 * fx;
            const float v = top * (1.f - fy) + bot * fy;
            px.o[ch] = store16((v - mean[ch]) / sd[ch], f16);          // Normalize on the channels in the order they arrive (B, G, R), like the reference
        }
#pragma unroll
        for (int ch = 3; ch < 16; ++ch) px.o[ch] = 0;
        uint4* dst = reinterpret_cast<uint4*>(out + (size_t)i * 16);
        dst[0] = px.v[0]; dst[1] = px.v[1];
    }
}

// NHWC, 8 channels (16 bytes) per thread
// k = 3: window -1 .. 1 (padding 1); k = 2: window 0 .. 1 (no padding)
__global__ void maxpool_s2_kernel(const unsigned short* __restrict__ in, unsigned short* __restrict__ out, int n, int h, int w, int c, int f16, int k) {
    const int ho = k == 3 ? (h + 1) / 2 : h / 2, wo = k == 3 ? (w + 1) / 2 : w / 2, cv = c / 8;
    const int d0 = k == 3 ? -1 : 0;
    const long long total = (long long)n * ho * wo * cv;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(i % cv), x = (int)((i / cv) % wo), y = (int)((i / ((long long)cv * wo)) % ho), b = (int)(i / ((long long)cv * wo * ho));
        float m[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) m[k] = -INFINITY;
        for (int dy = d0; dy <= 1; ++dy) {
            const int yy = 2 * y + dy;
            if (yy < 0 || yy >= h) continue;
            for (int dx = d0; dx <= 1; ++dx) {
                const int xx = 2 * x + dx;
                if (xx < 0 || xx >= w) continue;
                const uint4 q = *reinterpret_cast<const uint4*>(in + (((size_t)b * h + yy) * w + xx) * c + v * 8);
                const unsigned short* s = reinterpret_cast<const unsigned short*>(&q);
#pragma unroll
                for (int k = 0; k < 8; ++k) m[k] = fmaxf(m[k], load16(s + k, f16));
            }
        }
        union { unsigned short o[8]; uint4 q; } r;
#pragma unroll
        for (int k = 0; k < 8; ++k) r.o[k] = store16(m[k], f16);
        *reinterpret_cast<uint4*>(out + (((size_t)b * ho + y) * wo + x) * c + v * 8) = r.q;
    }
}

__global__ void add_relu_kernel(const unsigned short* __restrict__ a, const unsigned short* __restrict__ b, unsigned short* __restrict__ out, long long nvec, int f16) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        const uint4 qa = reinterpret_cast<const uint4*>(a)[i], qb = reinterpret_cast<const uint4*>(b)[i];
        const unsigned short* sa = reinterpret_cast<const unsigned short*>(&qa);
        const unsigned short* sb = reinterpret_cast<const unsigned short*>(&qb);
        union { unsigned short o[8]; uint4 q; } r;
#pragma unroll
        for (int k = 0; k < 8; ++k) r.o[k] = store16(fmaxf(load16(sa + k, f16) + load16(sb + k, f16), 0.f), f16);
        reinterpret_cast<uint4*>(out)[i] = r.q;
    }
}

// one block of 128 threads per crop: thread t owns channels 4t .. 4t+3 of the 512; mean over the hw positions, then the L2 norm
__device__ __forceinline__ void avgpool_l2norm_row(const unsigned short* __restrict__ in, float* __restrict__ out, int hw, int f16) {
    const int t = threadIdx.x;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int p = 0; p < hw; ++p) {
        const uint2 q = *reinterpret_cast<const uint2*>(in + (size_t)p * 512 + t * 4);
        const unsigned short* s = reinterpret_cast<const unsigned short*>(&q);
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k] += load16(s + k, f16);
    }
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) { acc[k] /= (float)hw; ss += acc[k] * acc[k]; }
    __shared__ float red[4];
    for (int d = 16; d >= 1; d >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, d);
    if ((t & 31) == 0) red[t >> 5] = ss;
    __syncthreads();
    const float nrm = sqrtf(red[0] + red[1] + red[2] + red[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) out[t * 4 + k] = acc[k] / nrm;
}

__global__ void avgpool_l2norm_kernel(const unsigned short* __restrict__ in, float* __restrict__ out, int hw, int f16) {
    avgpool_l2norm_row(in + (size_t)blockIdx.x * hw * 512, out + (size_t)blockIdx.x * 512, hw, f16);
}

// crop b -> row rowmap[b] of out [rows][512]; rowmap[b] < 0 (a padding crop): nothing written
__global__ void avgpool_l2norm_rows_kernel(const unsigned short* __restrict__ in, float* __restrict__ out, const int* __restrict__ rowmap, int hw, int f16) {
    const int r = rowmap[blockIdx.x];
    if (r < 0) return;
    avgpool_l2norm_row(in + (size_t)blockIdx.x * hw * 512, out + (size_t)r * 512, hw, f16);
}

// ---- BatchNorm with BATCH statistics.  The reference never calls net.eval() (deepsort_reid.py:112-121, :148-153): its BatchNorm layers
// normalise every call with the mean / biased variance of that call's crops.  x: [n_pix][c] 16-bit, c <= 512, c % 8 == 0, 256 % (c / 8) == 0.
// Three launches, all in a fixed summation order, so the result is bitwise reproducible from call to call:
//   bn_stats_kernel     block b: fp64 sums of (x - K) and (x - K)^2 per channel over its pixels, K = the channel's value at pixel 0 (a shift
//                       inside the data keeps the variance free of the E[x^2] - mean^2 cancellation); per-block partials -> ws
//   bn_finalize_kernel  per channel: the partials of all blocks in block order -> mean and gamma / sqrt(var + eps) (fp64) -> ws[0 .. 2c)
//   bn_apply_kernel     y = (x - mean) * scale + beta (+ ReLU) in fp64, rounded once to the 16-bit type
// ws layout (doubles): [0, c) mean, [c, 2c) scale, then [block][2][c] partials.
constexpr int kBnThreads = 256;
constexpr int kBnMaxBlocks = 132 * 8;
constexpr int kBnFinalWarps = 32;
// Segmented form (one segment = one sequence's crops, x [offsets[s] * pix_per_crop ..) [n_pix_s][c]): every segment gets exactly the
// launches above would give it alone -- bn_blocks(n_pix_s, c) stats blocks with the same grid-stride pattern, K from the segment's first
// pixel, the same tree, its partials added in block order -- so each segment's output is bitwise that of b2t_batchnorm_batch_stats on
// the segment.  The grid is an upper bound (bn_blocks(max_crops * pix_per_crop, c) x n_seg); blocks past their segment's count exit.
// ws layout (doubles): [n_seg][2][c] mean / scale, then [n_seg][bn_blocks(max)][2][c] partials.

__host__ __device__ inline int bn_blocks(long long n_pix, int c) {
    const long long ppb = kBnThreads / (c / 8);
    const long long g = (n_pix + ppb * 16 - 1) / (ppb * 16);
    return (int)(g < 1 ? 1 : (g > kBnMaxBlocks ? kBnMaxBlocks : g));
}

__device__ __forceinline__ unsigned short store16_d(double v, int f16) {
    if (f16) { const __half h = __double2half(v); return *reinterpret_cast<const unsigned short*>(&h); }
    const __nv_bfloat16 h = __double2bfloat16(v); return *reinterpret_cast<const unsigned short*>(&h);
}

// block bx of g over x [n_pix][c] -> part [2][c]
__device__ __forceinline__ void bn_stats_block(const unsigned short* __restrict__ x, long long n_pix, int c, double* __restrict__ part, int bx, int g, int f16) {
    // thread t handles the 8-channel vector (t % cv) of pixels t / cv, t / cv + stride ...
    const int cv = c / 8;
    const int vec = threadIdx.x % cv, lane_pix = threadIdx.x / cv, pix_per_block = blockDim.x / cv;
    double shift[8], s[8], q[8];
    {
        const uint4 v = *reinterpret_cast<const uint4*>(x + vec * 8);
        const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
#pragma unroll
        for (int k = 0; k < 8; ++k) { shift[k] = (double)load16(e + k, f16); s[k] = 0.0; q[k] = 0.0; }
    }
    for (long long p = (long long)bx * pix_per_block + lane_pix; p < n_pix; p += (long long)g * pix_per_block) {
        const uint4 v = *reinterpret_cast<const uint4*>(x + p * c + vec * 8);
        const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
#pragma unroll
        for (int k = 0; k < 8; ++k) { const double d = (double)load16(e + k, f16) - shift[k]; s[k] += d; q[k] += d * d; }
    }
    // fixed-order tree over the block's pixel lanes: lane l adds lane l + st for st = pix_per_block / 2 .. 1 (a power of two)
    __shared__ double sh[16][kBnThreads];
#pragma unroll
    for (int k = 0; k < 8; ++k) { sh[k][threadIdx.x] = s[k]; sh[8 + k][threadIdx.x] = q[k]; }
    __syncthreads();
    for (int st = pix_per_block / 2; st >= 1; st >>= 1) {
        if (lane_pix < st)
#pragma unroll
            for (int k = 0; k < 16; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + st * cv];
        __syncthreads();
    }
    if (lane_pix == 0) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { part[vec * 8 + k] = sh[k][threadIdx.x]; part[c + vec * 8 + k] = sh[8 + k][threadIdx.x]; }
    }
}

__global__ void bn_stats_kernel(const unsigned short* __restrict__ x, long long n_pix, int c, double* __restrict__ ws, int f16) {
    bn_stats_block(x, n_pix, c, ws + 2 * c + (size_t)blockIdx.x * 2 * c, blockIdx.x, gridDim.x, f16);
}

// block (bx, s): block bx of segment s, if the segment alone would have launched it
__global__ void bn_stats_seg_kernel(const unsigned short* __restrict__ x, const int* __restrict__ offsets, int pix_per_crop, int c, int gmax,
                                    double* __restrict__ ws, int f16) {
    const int sg = blockIdx.y, n_seg = gridDim.y;
    const long long n_pix = (long long)(offsets[sg + 1] - offsets[sg]) * pix_per_crop;
    if (n_pix <= 0 || (int)blockIdx.x >= bn_blocks(n_pix, c)) return;
    bn_stats_block(x + (size_t)offsets[sg] * pix_per_crop * c, n_pix, c, ws + (size_t)n_seg * 2 * c + ((size_t)sg * gmax + blockIdx.x) * 2 * c,
                   blockIdx.x, bn_blocks(n_pix, c), f16);
}

// block of kBnFinalWarps warps per 32 channels (channel block cb): lane = channel, warp w sums the partials of blocks w, w + 32, ... in
// order; then the warps' totals in warp order -> ms [2][c]
__device__ __forceinline__ void bn_finalize_block(const unsigned short* __restrict__ x, long long n_pix, int c, int blocks, const float* __restrict__ gamma,
                                                  float eps, const double* __restrict__ parts, double* __restrict__ ms, int cb, int f16) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ch = cb * 32 + lane;
    double s = 0.0, q = 0.0;
    if (ch < c)
        for (int b = warp; b < blocks; b += kBnFinalWarps) {
            const double* part = parts + (size_t)b * 2 * c;
            s += part[ch]; q += part[c + ch];
        }
    __shared__ double red[2][kBnFinalWarps][32];
    red[0][warp][lane] = s; red[1][warp][lane] = q;
    __syncthreads();
    if (warp == 0 && ch < c) {
        s = 0.0; q = 0.0;
        for (int w = 0; w < kBnFinalWarps; ++w) { s += red[0][w][lane]; q += red[1][w][lane]; }
        const double m = s / (double)n_pix;                                        // mean of x - K
        const double var = fmax(q / (double)n_pix - m * m, 0.0);                  // biased, like F.batch_norm in training mode
        ms[ch] = (double)load16(x + ch, f16) + m;
        ms[c + ch] = (double)gamma[ch] / sqrt(var + (double)eps);
    }
}

__global__ void bn_finalize_kernel(const unsigned short* __restrict__ x, long long n_pix, int c, int blocks, const float* __restrict__ gamma,
                                   float eps, double* __restrict__ ws, int f16) {
    bn_finalize_block(x, n_pix, c, blocks, gamma, eps, ws + 2 * c, ws, blockIdx.x, f16);
}

__global__ void bn_finalize_seg_kernel(const unsigned short* __restrict__ x, const int* __restrict__ offsets, int pix_per_crop, int c, int gmax,
                                       const float* __restrict__ gamma, float eps, double* __restrict__ ws, int f16) {
    const int sg = blockIdx.y, n_seg = gridDim.y;
    const long long n_pix = (long long)(offsets[sg + 1] - offsets[sg]) * pix_per_crop;
    if (n_pix <= 0) return;
    bn_finalize_block(x + (size_t)offsets[sg] * pix_per_crop * c, n_pix, c, bn_blocks(n_pix, c), gamma, eps,
                      ws + (size_t)n_seg * 2 * c + (size_t)sg * gmax * 2 * c, ws + (size_t)sg * 2 * c, blockIdx.x, f16);
}

// y = (x - mean) * scale + beta (+ ReLU) for the 8 channels of vector `vec`
__device__ __forceinline__ uint4 bn_apply_vec(uint4 v, int vec, int c, const double* __restrict__ ms, const float* __restrict__ beta, int relu, int f16) {
    const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
    union { unsigned short o[8]; uint4 q; } r;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int ch = vec * 8 + k;
        double f = ((double)load16(e + k, f16) - ms[ch]) * ms[c + ch] + (double)beta[ch];
        if (relu) f = fmax(f, 0.0);
        r.o[k] = store16_d(f, f16);
    }
    return r.q;
}

__global__ void bn_apply_kernel(const unsigned short* __restrict__ x, unsigned short* __restrict__ y, long long n_vec, int c,
                                const double* __restrict__ ws, const float* __restrict__ beta, int relu, int f16) {
    const int cv = c / 8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x)
        reinterpret_cast<uint4*>(y)[i] = bn_apply_vec(reinterpret_cast<const uint4*>(x)[i], (int)(i % cv), c, ws, beta, relu, f16);
}

// every vector of the crops [0, offsets[n_seg]) with its segment's statistics; the padding crops past offsets[n_seg] are not touched
__global__ void bn_apply_seg_kernel(const unsigned short* __restrict__ x, unsigned short* __restrict__ y, const int* __restrict__ offsets, int n_seg,
                                    int pix_per_crop, int c, const double* __restrict__ ws, const float* __restrict__ beta, int relu, int f16) {
    const int cv = c / 8;
    const long long per_crop = (long long)pix_per_crop * cv, n_vec = (long long)offsets[n_seg] * per_crop;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
        const long long crop = i / per_crop;
        int lo = 0, hi = n_seg;                 // the last segment starting at or before the crop: offsets[lo] <= crop < offsets[hi]
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (offsets[mid] <= crop) lo = mid; else hi = mid; }
        reinterpret_cast<uint4*>(y)[i] = bn_apply_vec(reinterpret_cast<const uint4*>(x)[i], (int)(i % cv), c, ws + (size_t)lo * 2 * c, beta, relu, f16);
    }
}

// ---- crop list of the sequences' det_high rows (botsort.py:339-346 per sequence; the crops of deepsort_reid.py:141-146).  One block walks
// the sequences in order; inside a sequence, rows in chunks of blockDim, compacted in row order with a ballot scan.
constexpr int kCropListThreads = 256;

__global__ void reid_crop_list_kernel(const float* __restrict__ dets, const int* __restrict__ det_count, int n_seq, int dmax, float det_thresh,
                                      int height, int width, int cap, long long* __restrict__ crops, int* __restrict__ offsets,
                                      int* __restrict__ rowmap, int* __restrict__ status) {
    __shared__ int warp_n[kCropListThreads / 32];
    __shared__ int seq_bits;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    const long long frame_bytes = (long long)height * width * 3;
    int total = 0;                                              // det_high rows so far, uncapped (same value in every thread)
    for (int s = 0; s < n_seq; ++s) {
        if (tid == 0) { offsets[s] = total < cap ? total : cap; seq_bits = 0; }
        __syncthreads();
        int bits = 0;
        const int nd = min(max(det_count[s], 0), dmax);
        for (int i0 = 0; i0 < nd; i0 += blockDim.x) {
            const int i = i0 + tid;
            const float* d = dets + ((size_t)s * dmax + i) * 6;
            const bool hi = i < nd && d[4] >= det_thresh;        // the tracker's det_high rows (b2t_step.cuh), has_area not applied
            const unsigned m = __ballot_sync(0xffffffffu, hi);
            if (lane == 0) warp_n[wid] = __popc(m);
            __syncthreads();
            int before = 0, chunk = 0;
            for (int w = 0; w < nw; ++w) { before += w < wid ? warp_n[w] : 0; chunk += warp_n[w]; }
            if (hi) {
                const int j = total + before + __popc(m & ((1u << lane) - 1u));
                // ori_img[int(y1):int(y2), int(x1):int(x2)]: int() truncates; the slice clips the right / bottom ends to the frame
                long long desc[4] = {(long long)s * frame_bytes, 3LL * width, 1, 1};       // a valid 1 x 1 crop for a refused row
                if (!(d[0] > -1.f && d[1] > -1.f && d[2] > -1.f && d[3] > -1.f)) {
                    bits |= B2T_REID_NEGATIVE;                  // int() < 0 (or NaN): the slice would wrap to the far side of the frame
                } else {
                    const int x1 = (int)fminf(d[0], (float)width), y1 = (int)fminf(d[1], (float)height);
                    const int x2 = (int)fminf(d[2], (float)width), y2 = (int)fminf(d[3], (float)height);
                    if (x2 - x1 < 1 || y2 - y1 < 1) bits |= B2T_REID_ZERO_SIZE;   // "size in bbox exists zero" (deepsort_reid.py:141-142)
                    else { desc[0] += ((long long)y1 * width + x1) * 3; desc[2] = y2 - y1; desc[3] = x2 - x1; }
                }
                if (j < cap) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) crops[(size_t)j * 4 + k] = desc[k];
                    rowmap[j] = s * dmax + i;
                } else {
                    bits |= B2T_REID_OVERFLOW;
                }
            }
            total += chunk;
            __syncthreads();                                    // warp_n is rewritten by the next chunk
        }
        if (bits) atomicOr(&seq_bits, bits);
        __syncthreads();
        if (tid == 0) status[s] = seq_bits;
    }
    const int used = total < cap ? total : cap;
    if (tid == 0) { offsets[n_seq] = used; status[n_seq] = total; }
    __syncthreads();                                            // crops[0] is visible to the whole block
    // padding rows [used, cap): a copy of crop 0 (a 1 x 1 crop of frame 0 when there is none), so the fixed-size crop kernel reads pixels
    for (int j = used + tid; j < cap; j += blockDim.x) {
#pragma unroll
        for (int k = 0; k < 4; ++k) crops[(size_t)j * 4 + k] = used ? crops[k] : (k == 0 ? 0LL : (k == 1 ? 3LL * width : 1LL));
        rowmap[j] = -1;
    }
}

}  // namespace

static int bn_args_ok(long long n_pix, int c) { return n_pix >= 1 && c >= 8 && c <= 512 && c % 8 == 0 && kBnThreads % (c / 8) == 0; }

extern "C" size_t b2t_batchnorm_workspace_bytes(long long n_pix, int c) {
    if (!bn_args_ok(n_pix, c)) return 0;
    return ((size_t)2 * c + (size_t)bn_blocks(n_pix, c) * 2 * c) * sizeof(double);
}

extern "C" int b2t_batchnorm_batch_stats(const void* x, void* y, long long n_pix, int c, const float* gamma, const float* beta, float eps, int relu,
                                         double* ws, int act_dtype, void* stream) {
    if (!x || !y || !gamma || !beta || !ws || n_pix < 1 || c < 8 || c > 512 || c % 8) return rfail(B2T_EINVAL, "b2t_batchnorm_batch_stats: bad arguments (8 <= c <= 512, c % 8 == 0)");
    if (!bn_args_ok(n_pix, c)) return rfail(B2T_EINVAL, "b2t_batchnorm_batch_stats: c / 8 must divide 256");
    cudaStream_t s = (cudaStream_t)stream;
    const int f16 = act_dtype == B2T_ACT_F16, g = bn_blocks(n_pix, c);
    const unsigned short* xs = (const unsigned short*)x;
    B2T_LAUNCH(bn_stats_kernel, g, kBnThreads, 0, s, xs, n_pix, c, ws, f16);
    B2T_LAUNCH(bn_finalize_kernel, (c + 31) / 32, kBnFinalWarps * 32, 0, s, xs, n_pix, c, g, gamma, eps, ws, f16);
    B2T_LAUNCH(bn_apply_kernel, grid_for(n_pix * (c / 8), 256), 256, 0, s, xs, (unsigned short*)y, n_pix * (c / 8), c, (const double*)ws, beta, relu, f16);
    return rcheck("batchnorm_batch_stats");
}

static int bn_seg_args_ok(int n_seg, int max_crops, int pix_per_crop, int c) {
    return n_seg >= 1 && n_seg <= 65535 && max_crops >= 1 && pix_per_crop >= 1 && (long long)max_crops * pix_per_crop <= (1LL << 40) && bn_args_ok(1, c);
}

extern "C" size_t b2t_batchnorm_segments_workspace_bytes(int n_seg, int max_crops, int pix_per_crop, int c) {
    if (!bn_seg_args_ok(n_seg, max_crops, pix_per_crop, c)) return 0;
    return ((size_t)n_seg * 2 * c + (size_t)n_seg * bn_blocks((long long)max_crops * pix_per_crop, c) * 2 * c) * sizeof(double);
}

extern "C" int b2t_batchnorm_batch_stats_segments(const void* x, void* y, const int* offsets, int n_seg, int max_crops, int pix_per_crop, int c,
                                                  const float* gamma, const float* beta, float eps, int relu, double* ws, int act_dtype, void* stream) {
    if (!x || !y || !offsets || !gamma || !beta || !ws || !bn_seg_args_ok(n_seg, max_crops, pix_per_crop, c))
        return rfail(B2T_EINVAL, "b2t_batchnorm_batch_stats_segments: bad arguments (1 <= n_seg <= 65535, max_crops >= 1, pix_per_crop >= 1, 8 <= c <= 512, c / 8 divides 256)");
    cudaStream_t s = (cudaStream_t)stream;
    const int f16 = act_dtype == B2T_ACT_F16;
    const long long max_pix = (long long)max_crops * pix_per_crop;
    const int gmax = bn_blocks(max_pix, c);
    const unsigned short* xs = (const unsigned short*)x;
    B2T_LAUNCH(bn_stats_seg_kernel, dim3(gmax, n_seg), kBnThreads, 0, s, xs, offsets, pix_per_crop, c, gmax, ws, f16);
    B2T_LAUNCH(bn_finalize_seg_kernel, dim3((c + 31) / 32, n_seg), kBnFinalWarps * 32, 0, s, xs, offsets, pix_per_crop, c, gmax, gamma, eps, ws, f16);
    B2T_LAUNCH(bn_apply_seg_kernel, grid_for(max_pix * (c / 8), 256), 256, 0, s, xs, (unsigned short*)y, offsets, n_seg, pix_per_crop, c,
               (const double*)ws, beta, relu, f16);
    return rcheck("batchnorm_batch_stats_segments");
}

extern "C" int b2t_reid_crops_from_dets(const float* dets, const int* det_count, int n_seq, int dmax, float det_thresh, int height, int width, int cap,
                                        long long* crops, int* offsets, int* rowmap, int* status, void* stream) {
    if (!dets || !det_count || !crops || !offsets || !rowmap || !status || n_seq < 1 || dmax < 1 || height < 1 || width < 1 || cap < 1)
        return rfail(B2T_EINVAL, "b2t_reid_crops_from_dets: bad arguments");
    B2T_LAUNCH(reid_crop_list_kernel, 1, kCropListThreads, 0, (cudaStream_t)stream, dets, det_count, n_seq, dmax, det_thresh, height, width, cap,
               crops, offsets, rowmap, status);
    return rcheck("reid_crops_from_dets");
}

extern "C" int b2t_reid_crops(const unsigned char* pixels, const long long* crops, int n, void* out_nhwc16, int act_dtype, void* stream) {
    if (!pixels || !crops || !out_nhwc16 || n < 1 || (act_dtype != B2T_ACT_BF16 && act_dtype != B2T_ACT_F16)) return rfail(B2T_EINVAL, "b2t_reid_crops: bad arguments");
    B2T_LAUNCH(reid_crop_kernel, grid_for((long long)n * 128 * 64, 256), 256, 0, (cudaStream_t)stream, pixels, crops, n, (unsigned short*)out_nhwc16, act_dtype == B2T_ACT_F16);
    return rcheck("reid_crops");
}

extern "C" int b2t_maxpool3x3s2(const void* in, void* out, int n, int h, int w, int c, int act_dtype, void* stream) {
    if (!in || !out || n < 1 || h < 1 || w < 1 || c < 8 || c % 8) return rfail(B2T_EINVAL, "b2t_maxpool3x3s2: bad arguments (channels must be a multiple of 8)");
    B2T_LAUNCH(maxpool_s2_kernel, grid_for((long long)n * ((h + 1) / 2) * ((w + 1) / 2) * (c / 8), 256), 256, 0, (cudaStream_t)stream,
               (const unsigned short*)in, (unsigned short*)out, n, h, w, c, act_dtype == B2T_ACT_F16, 3);
    return rcheck("maxpool3x3s2");
}

extern "C" int b2t_maxpool2x2s2(const void* in, void* out, int n, int h, int w, int c, int act_dtype, void* stream) {
    if (!in || !out || n < 1 || h < 2 || w < 2 || (h & 1) || (w & 1) || c < 8 || c % 8) return rfail(B2T_EINVAL, "b2t_maxpool2x2s2: bad arguments (even sides, channels a multiple of 8)");
    B2T_LAUNCH(maxpool_s2_kernel, grid_for((long long)n * (h / 2) * (w / 2) * (c / 8), 256), 256, 0, (cudaStream_t)stream,
               (const unsigned short*)in, (unsigned short*)out, n, h, w, c, act_dtype == B2T_ACT_F16, 2);
    return rcheck("maxpool2x2s2");
}

extern "C" int b2t_add_relu(const void* a, const void* b, void* out, long long n_elems, int act_dtype, void* stream) {
    if (!a || !b || !out || n_elems < 8 || n_elems % 8) return rfail(B2T_EINVAL, "b2t_add_relu: element count must be a multiple of 8");
    B2T_LAUNCH(add_relu_kernel, grid_for(n_elems / 8, 256), 256, 0, (cudaStream_t)stream, (const unsigned short*)a, (const unsigned short*)b, (unsigned short*)out,
               n_elems / 8, act_dtype == B2T_ACT_F16);
    return rcheck("add_relu");
}

extern "C" int b2t_avgpool_l2norm(const void* in, float* out, int n, int hw, int c, int act_dtype, void* stream) {
    if (!in || !out || n < 1 || hw < 1 || c != 512) return rfail(B2T_EINVAL, "b2t_avgpool_l2norm: 512 channels expected");
    B2T_LAUNCH(avgpool_l2norm_kernel, n, 128, 0, (cudaStream_t)stream, (const unsigned short*)in, out, hw, act_dtype == B2T_ACT_F16);
    return rcheck("avgpool_l2norm");
}

extern "C" int b2t_avgpool_l2norm_rows(const void* in, float* out, const int* rowmap, int n, int hw, int c, int act_dtype, void* stream) {
    if (!in || !out || !rowmap || n < 1 || hw < 1 || c != 512) return rfail(B2T_EINVAL, "b2t_avgpool_l2norm_rows: 512 channels expected");
    B2T_LAUNCH(avgpool_l2norm_rows_kernel, n, 128, 0, (cudaStream_t)stream, (const unsigned short*)in, out, rowmap, hw, act_dtype == B2T_ACT_F16);
    return rcheck("avgpool_l2norm_rows");
}
