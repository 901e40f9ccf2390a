// b2t_reid.cu -- glue kernels of the appearance branch (SURVEY.md section 8f row 3): everything of the reference's ReID extractor
// (tracker/reid_models/deepsort_reid.py:63-153) that is not a convolution.  The 3x3 / 1x1 convolutions (+ folded BatchNorm + ReLU) run on
// the wgmma kernel of b2t_conv.cu; these kernels are the byte / element-wise work around them -- HBM-bound, 16-byte vectors.
//   reid_crop_kernel       Extractor._preprocess :134-146: crop.astype(float32) / 255 -> cv2.resize to 64 x 128 (bilinear, float) ->
//                          ToTensor -> Normalize(mean, std); written as NHWC 16-bit with the 3 channels padded to 16 (tensor-core K granularity)
//   maxpool3x3s2_kernel    nn.MaxPool2d(3, 2, padding=1) :72
//   add_relu_kernel        BasicBlock.forward :49 F.relu(x.add(y))
//   avgpool_l2norm_kernel  nn.AvgPool2d((8, 4), 1) :83 + x.div(x.norm(p=2, dim=1)) :103-104 -> 512 floats per crop
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
__global__ void avgpool_l2norm_kernel(const unsigned short* __restrict__ in, float* __restrict__ out, int hw, int f16) {
    const int b = blockIdx.x, t = threadIdx.x;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int p = 0; p < hw; ++p) {
        const uint2 q = *reinterpret_cast<const uint2*>(in + ((size_t)b * hw + p) * 512 + t * 4);
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
    for (int k = 0; k < 4; ++k) out[(size_t)b * 512 + t * 4 + k] = acc[k] / nrm;
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

int bn_blocks(long long n_pix, int c) {
    const long long ppb = kBnThreads / (c / 8);
    const long long g = (n_pix + ppb * 16 - 1) / (ppb * 16);
    return (int)(g < 1 ? 1 : (g > kBnMaxBlocks ? kBnMaxBlocks : g));
}

__device__ __forceinline__ unsigned short store16_d(double v, int f16) {
    if (f16) { const __half h = __double2half(v); return *reinterpret_cast<const unsigned short*>(&h); }
    const __nv_bfloat16 h = __double2bfloat16(v); return *reinterpret_cast<const unsigned short*>(&h);
}

__global__ void bn_stats_kernel(const unsigned short* __restrict__ x, long long n_pix, int c, double* __restrict__ ws, int f16) {
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
    for (long long p = (long long)blockIdx.x * pix_per_block + lane_pix; p < n_pix; p += (long long)gridDim.x * pix_per_block) {
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
        double* part = ws + 2 * c + (size_t)blockIdx.x * 2 * c;
#pragma unroll
        for (int k = 0; k < 8; ++k) { part[vec * 8 + k] = sh[k][threadIdx.x]; part[c + vec * 8 + k] = sh[8 + k][threadIdx.x]; }
    }
}

// block of kBnFinalWarps warps per 32 channels: lane = channel, warp w sums the partials of blocks w, w + 32, ... in order; then the
// warps' totals in warp order
__global__ void bn_finalize_kernel(const unsigned short* __restrict__ x, long long n_pix, int c, int blocks, const float* __restrict__ gamma,
                                   float eps, double* __restrict__ ws, int f16) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ch = blockIdx.x * 32 + lane;
    double s = 0.0, q = 0.0;
    if (ch < c)
        for (int b = warp; b < blocks; b += kBnFinalWarps) {
            const double* part = ws + 2 * c + (size_t)b * 2 * c;
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
        ws[ch] = (double)load16(x + ch, f16) + m;
        ws[c + ch] = (double)gamma[ch] / sqrt(var + (double)eps);
    }
}

__global__ void bn_apply_kernel(const unsigned short* __restrict__ x, unsigned short* __restrict__ y, long long n_vec, int c,
                                const double* __restrict__ ws, const float* __restrict__ beta, int relu, int f16) {
    const int cv = c / 8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
        const int vec = (int)(i % cv);
        const uint4 v = reinterpret_cast<const uint4*>(x)[i];
        const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
        union { unsigned short o[8]; uint4 q; } r;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ch = vec * 8 + k;
            double f = ((double)load16(e + k, f16) - ws[ch]) * ws[c + ch] + (double)beta[ch];
            if (relu) f = fmax(f, 0.0);
            r.o[k] = store16_d(f, f16);
        }
        reinterpret_cast<uint4*>(y)[i] = r.q;
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
