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
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include "b2t_platform.cuh"
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
// normalise every call with the mean / biased variance of that call's crops.  Reproduced as two passes over the conv output:
// per-channel sums (fp32 partials per block, fp64 atomics), then scale / shift (+ ReLU).  x: [n_pix][c] 16-bit, c <= 512, c % 8 == 0.
__global__ void bn_stats_kernel(const unsigned short* __restrict__ x, long long n_pix, int c, double* __restrict__ sums, int f16) {
    // thread t handles the 8-channel vector (t % cv) of pixels t / cv, t / cv + stride ...
    const int cv = c / 8;
    const int vec = threadIdx.x % cv, lane_pix = threadIdx.x / cv, pix_per_block = blockDim.x / cv;
    float s[8], q[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { s[k] = 0.f; q[k] = 0.f; }
    if (lane_pix < pix_per_block)
        for (long long p = (long long)blockIdx.x * pix_per_block + lane_pix; p < n_pix; p += (long long)gridDim.x * pix_per_block) {
            const uint4 v = *reinterpret_cast<const uint4*>(x + p * c + vec * 8);
            const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
#pragma unroll
            for (int k = 0; k < 8; ++k) { const float f = load16(e + k, f16); s[k] += f; q[k] += f * f; }
        }
    __shared__ float sh[2][512];
    for (int i = threadIdx.x; i < 2 * 512; i += blockDim.x) (&sh[0][0])[i] = 0.f;
    __syncthreads();
    if (lane_pix < pix_per_block)
#pragma unroll
        for (int k = 0; k < 8; ++k) { atomicAdd(&sh[0][vec * 8 + k], s[k]); atomicAdd(&sh[1][vec * 8 + k], q[k]); }
    __syncthreads();
    for (int i = threadIdx.x; i < c; i += blockDim.x) { atomicAdd(&sums[i], (double)sh[0][i]); atomicAdd(&sums[512 + i], (double)sh[1][i]); }
}

// y = (x - mean) / sqrt(var + eps) * gamma + beta, optional ReLU; also clears the sums for the next use
__global__ void bn_apply_kernel(const unsigned short* __restrict__ x, unsigned short* __restrict__ y, long long n_vec, int c, long long n_pix,
                                const double* __restrict__ sums, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int relu, int f16) {
    const int cv = c / 8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
        const int vec = (int)(i % cv);
        const uint4 v = reinterpret_cast<const uint4*>(x)[i];
        const unsigned short* e = reinterpret_cast<const unsigned short*>(&v);
        union { unsigned short o[8]; uint4 q; } r;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ch = vec * 8 + k;
            const double mean = sums[ch] / (double)n_pix;
            const double var = fmax(sums[512 + ch] / (double)n_pix - mean * mean, 0.0);
            const float sc = gamma[ch] * (float)(1.0 / sqrt(var + (double)eps));
            float f = (load16(e + k, f16) - (float)mean) * sc + beta[ch];
            if (relu) f = fmaxf(f, 0.f);
            r.o[k] = store16(f, f16);
        }
        reinterpret_cast<uint4*>(y)[i] = r.q;
    }
}

}  // namespace

extern "C" int b2t_batchnorm_batch_stats(const void* x, void* y, long long n_pix, int c, const float* gamma, const float* beta, float eps, int relu,
                                         double* sums_ws, int act_dtype, void* stream) {
    if (!x || !y || !gamma || !beta || !sums_ws || n_pix < 1 || c < 8 || c > 512 || c % 8) return rfail(B2T_EINVAL, "b2t_batchnorm_batch_stats: bad arguments (8 <= c <= 512, c % 8 == 0)");
    cudaStream_t s = (cudaStream_t)stream;
    if (cudaMemsetAsync(sums_ws, 0, 1024 * sizeof(double), s) != cudaSuccess) return rfail(B2T_ECUDA, "b2t_batchnorm_batch_stats: memset failed");
    const int cv = c / 8, threads = 256;                  // cv is a power of two <= 64 for the extractor's widths: 256 % cv == 0
    if (threads % cv) return rfail(B2T_EINVAL, "b2t_batchnorm_batch_stats: c / 8 must divide 256");
    const long long ppb = threads / cv;
    long long g = (n_pix + ppb * 16 - 1) / (ppb * 16);
    g = g < 1 ? 1 : (g > 132 * 8 ? 132 * 8 : g);
    bn_stats_kernel<<<(int)g, threads, 0, s>>>((const unsigned short*)x, n_pix, c, sums_ws, act_dtype == B2T_ACT_F16);
    bn_apply_kernel<<<grid_for(n_pix * cv, 256), 256, 0, s>>>((const unsigned short*)x, (unsigned short*)y, n_pix * cv, c, n_pix, sums_ws, gamma, beta, eps, relu,
                                                           act_dtype == B2T_ACT_F16);
    return rcheck("batchnorm_batch_stats");
}

extern "C" int b2t_reid_crops(const unsigned char* pixels, const long long* crops, int n, void* out_nhwc16, int act_dtype, void* stream) {
    if (!pixels || !crops || !out_nhwc16 || n < 1 || (act_dtype != B2T_ACT_BF16 && act_dtype != B2T_ACT_F16)) return rfail(B2T_EINVAL, "b2t_reid_crops: bad arguments");
    reid_crop_kernel<<<grid_for((long long)n * 128 * 64, 256), 256, 0, (cudaStream_t)stream>>>(pixels, crops, n, (unsigned short*)out_nhwc16, act_dtype == B2T_ACT_F16);
    return rcheck("reid_crops");
}

extern "C" int b2t_maxpool3x3s2(const void* in, void* out, int n, int h, int w, int c, int act_dtype, void* stream) {
    if (!in || !out || n < 1 || h < 1 || w < 1 || c < 8 || c % 8) return rfail(B2T_EINVAL, "b2t_maxpool3x3s2: bad arguments (channels must be a multiple of 8)");
    maxpool_s2_kernel<<<grid_for((long long)n * ((h + 1) / 2) * ((w + 1) / 2) * (c / 8), 256), 256, 0, (cudaStream_t)stream>>>(
        (const unsigned short*)in, (unsigned short*)out, n, h, w, c, act_dtype == B2T_ACT_F16, 3);
    return rcheck("maxpool3x3s2");
}

extern "C" int b2t_maxpool2x2s2(const void* in, void* out, int n, int h, int w, int c, int act_dtype, void* stream) {
    if (!in || !out || n < 1 || h < 2 || w < 2 || (h & 1) || (w & 1) || c < 8 || c % 8) return rfail(B2T_EINVAL, "b2t_maxpool2x2s2: bad arguments (even sides, channels a multiple of 8)");
    maxpool_s2_kernel<<<grid_for((long long)n * (h / 2) * (w / 2) * (c / 8), 256), 256, 0, (cudaStream_t)stream>>>(
        (const unsigned short*)in, (unsigned short*)out, n, h, w, c, act_dtype == B2T_ACT_F16, 2);
    return rcheck("maxpool2x2s2");
}

extern "C" int b2t_add_relu(const void* a, const void* b, void* out, long long n_elems, int act_dtype, void* stream) {
    if (!a || !b || !out || n_elems < 8 || n_elems % 8) return rfail(B2T_EINVAL, "b2t_add_relu: element count must be a multiple of 8");
    add_relu_kernel<<<grid_for(n_elems / 8, 256), 256, 0, (cudaStream_t)stream>>>((const unsigned short*)a, (const unsigned short*)b, (unsigned short*)out, n_elems / 8,
                                                                                   act_dtype == B2T_ACT_F16);
    return rcheck("add_relu");
}

extern "C" int b2t_avgpool_l2norm(const void* in, float* out, int n, int hw, int c, int act_dtype, void* stream) {
    if (!in || !out || n < 1 || hw < 1 || c != 512) return rfail(B2T_EINVAL, "b2t_avgpool_l2norm: 512 channels expected");
    avgpool_l2norm_kernel<<<n, 128, 0, (cudaStream_t)stream>>>((const unsigned short*)in, out, hw, act_dtype == B2T_ACT_F16);
    return rcheck("avgpool_l2norm");
}
