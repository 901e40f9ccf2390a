// b2t_detect.cu -- the memory-bound glue around the convolutions of the YOLOv7 detector branch, and NMS.
//
//   image_reorg_kernel     ReOrg (models/common.py:48-53) + NCHW fp32 -> NHWC bf16 (+ zero pad to 16 ch)
//   upsample2x_kernel      nn.Upsample(None, 2, 'nearest'), written straight into the concat buffer
//   spp_pool_kernel        the three stride-1 max-pools (5/9/13) of SPPCSPC (models/common.py:271,278)
//   detect_decode_kernel   Detect.forward inference branch (models/yolo.py:44-55): sigmoid, grid / anchor decode
// (non_max_suppression and its fusion with the decode live in b2t_nms.cu.)
// All HBM-bound elementwise / scan work: coalesced along channels, 16-byte accesses where the layout allows.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string>
#include "../../include/b200track.h"
#include "b2t_decode.cuh"

namespace {
thread_local std::string g_det_err;
}
namespace b2t { void set_detect_error(const char* m) { g_det_err = m; } }     // shared with b2t_nms.cu
namespace {
int dfail(int code, const char* m) { g_det_err = m; return code; }
int dcheck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { g_det_err = std::string(what) + ": " + cudaGetErrorString(e); return B2T_ECUDA; }
    return B2T_OK;
}

// 16-bit activation types (B2T_ACT_BF16 / B2T_ACT_F16): conversion and packed max
template <typename T> struct Act16;
template <> struct Act16<__nv_bfloat16> {
    typedef __nv_bfloat162 T2;
    static __device__ __forceinline__ __nv_bfloat16 from_float(float f) { return __float2bfloat16_rn(f); }
    static __device__ __forceinline__ T2 lowest() { return __floats2bfloat162_rn(-3.0e38f, -3.0e38f); }
};
template <> struct Act16<__half> {
    typedef __half2 T2;
    static __device__ __forceinline__ __half from_float(float f) { return __float2half_rn(f); }
    static __device__ __forceinline__ T2 lowest() { return __floats2half2_rn(-65504.f, -65504.f); }
};
__device__ __forceinline__ __nv_bfloat162 bmax2(__nv_bfloat162 a, __nv_bfloat162 b) { return __hmax2(a, b); }
__device__ __forceinline__ __half2 bmax2(__half2 a, __half2 b) { return __hmax2(a, b); }

// ---------------------------------------------------------------- ReOrg + layout change
// out[b][y][x][phase*3 + c] = img[b][c][2y + dy][2x + dx], phase order (dy,dx) = (0,0),(1,0),(0,1),(1,1)
template <typename T>
__global__ void image_reorg_kernel(const float* __restrict__ img, T* __restrict__ out, int B, int H, int W, int row_pixels, int x0) {
    const int H2 = H / 2, W2 = W / 2;
    const long long total = (long long)B * H2 * W2;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(p % W2), y = (int)((p / W2) % H2), b = (int)(p / ((long long)W2 * H2));
        T v[16];
#pragma unroll
        for (int ph = 0; ph < 4; ++ph) {
            const int dy = ph & 1, dx = ph >> 1;
#pragma unroll
            for (int c = 0; c < 3; ++c)
                v[ph * 3 + c] = Act16<T>::from_float(img[(((long long)b * 3 + c) * H + 2 * y + dy) * W + 2 * x + dx]);
        }
        v[12] = v[13] = v[14] = v[15] = Act16<T>::from_float(0.f);
        uint4* o = reinterpret_cast<uint4*>(out + ((((long long)b * H2 + y) * row_pixels) + x0 + x) * 16);
        o[0] = *reinterpret_cast<uint4*>(&v[0]);
        o[1] = *reinterpret_cast<uint4*>(&v[8]);
    }
}

// NCHW fp32 -> NHWC 16-bit, 3 -> 16 channels (zero padded), no ReOrg: the first conv of YOLOv7-tiny reads the image itself
template <typename T>
__global__ void image_nhwc16_kernel(const float* __restrict__ img, T* __restrict__ out, int B, int H, int W) {
    const long long total = (long long)B * H * W, plane = (long long)H * W;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        const long long b = p / plane, r = p - b * plane;
        T v[16];
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = Act16<T>::from_float(img[(b * 3 + c) * plane + r]);
#pragma unroll
        for (int c = 3; c < 16; ++c) v[c] = Act16<T>::from_float(0.f);
        uint4* o = reinterpret_cast<uint4*>(out + p * 16);
        o[0] = *reinterpret_cast<uint4*>(&v[0]);
        o[1] = *reinterpret_cast<uint4*>(&v[8]);
    }
}

// ---------------------------------------------------------------- nearest x2 upsample, 8 channels (16 B) per thread
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ src, int sp, int sc, __nv_bfloat16* __restrict__ dst, int dp, int dc,
                                  int B, int H, int W, int C) {
    const int cv = C / 8;
    const long long total = (long long)B * (2 * H) * (2 * W) * cv;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % cv);
        long long p = i / cv;
        const int x = (int)(p % (2 * W)), y = (int)((p / (2 * W)) % (2 * H)), b = (int)(p / ((long long)4 * W * H));
        const uint4 v = *reinterpret_cast<const uint4*>(src + (((long long)b * H + y / 2) * W + x / 2) * sp + sc + c8 * 8);
        *reinterpret_cast<uint4*>(dst + p * dp + dc + c8 * 8) = v;
    }
}

// ---------------------------------------------------------------- SPP max-pools 5 / 9 / 13 (stride 1, pad k/2)
template <typename T>
__global__ void spp_pool_kernel(T* __restrict__ buf, int pitch, int C, int B, int H, int W) {
    typedef typename Act16<T>::T2 T2;
    const int cv = C / 2;
    const long long total = (long long)B * H * W * cv;
    const T2 ninf = Act16<T>::lowest();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c2 = (int)(i % cv);
        long long p = i / cv;
        const int x = (int)(p % W), y = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
        T2 m5 = ninf, m9 = ninf, m13 = ninf;
        for (int dy = -6; dy <= 6; ++dy) {
            const int yy = y + dy;
            if (yy < 0 || yy >= H) continue;
            for (int dx = -6; dx <= 6; ++dx) {
                const int xx = x + dx;
                if (xx < 0 || xx >= W) continue;
                const T2 v = *reinterpret_cast<const T2*>(buf + (((long long)b * H + yy) * W + xx) * pitch + c2 * 2);
                m13 = bmax2(m13, v);
                if (dy >= -4 && dy <= 4 && dx >= -4 && dx <= 4) m9 = bmax2(m9, v);
                if (dy >= -2 && dy <= 2 && dx >= -2 && dx <= 2) m5 = bmax2(m5, v);
            }
        }
        T* o = buf + p * pitch + c2 * 2;
        *reinterpret_cast<T2*>(o + C) = m5;
        *reinterpret_cast<T2*>(o + 2 * C) = m9;
        *reinterpret_cast<T2*>(o + 3 * C) = m13;
    }
}

// Small maps (the w6 SPP sees 20 x 20 at 1280 px): one CTA owns an (image, 8-channel) plane in shared memory and does the
// three pools separably -- 13 + 13 shared-memory reads per output instead of 169 global ones.  max is exact, so the result
// is identical to the direct kernel above (kept for planes that do not fit).
template <typename T>
__global__ void spp_pool_plane_kernel(T* __restrict__ buf, int pitch, int C, int H, int W) {
    typedef typename Act16<T>::T2 T2;
    extern __shared__ __align__(16) unsigned char spp_smem[];
    const int HW = H * W, cg = blockIdx.x, b = blockIdx.y;
    T2* in = reinterpret_cast<T2*>(spp_smem);
    T2* r5 = in + HW * 4;
    T2* r9 = r5 + HW * 4;
    T2* r13 = r9 + HW * 4;
    T* base = buf + (long long)b * HW * pitch + cg * 8;
    for (int px = threadIdx.x; px < HW; px += blockDim.x)
        reinterpret_cast<uint4*>(in)[px] = *reinterpret_cast<const uint4*>(base + (long long)px * pitch);
    __syncthreads();
    for (int i = threadIdx.x; i < HW * 4; i += blockDim.x) {              // along x
        const int c = i & 3, px = i >> 2, x = px % W;
        T2 m5 = in[i], m9 = m5, m13 = m5;
#pragma unroll
        for (int d = 1; d <= 6; ++d) {
            if (x - d >= 0) { const T2 v = in[(px - d) * 4 + c]; m13 = bmax2(m13, v); if (d <= 4) m9 = bmax2(m9, v); if (d <= 2) m5 = bmax2(m5, v); }
            if (x + d < W) { const T2 v = in[(px + d) * 4 + c]; m13 = bmax2(m13, v); if (d <= 4) m9 = bmax2(m9, v); if (d <= 2) m5 = bmax2(m5, v); }
        }
        r5[i] = m5; r9[i] = m9; r13[i] = m13;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < HW * 4; i += blockDim.x) {              // along y, then store
        const int c = i & 3, px = i >> 2, y = px / W;
        T2 m5 = r5[i], m9 = r9[i], m13 = r13[i];
#pragma unroll
        for (int d = 1; d <= 6; ++d) {
            if (y - d >= 0) { const int j = (px - d * W) * 4 + c; m13 = bmax2(m13, r13[j]); if (d <= 4) m9 = bmax2(m9, r9[j]); if (d <= 2) m5 = bmax2(m5, r5[j]); }
            if (y + d < H) { const int j = (px + d * W) * 4 + c; m13 = bmax2(m13, r13[j]); if (d <= 4) m9 = bmax2(m9, r9[j]); if (d <= 2) m5 = bmax2(m5, r5[j]); }
        }
        T* o = base + (long long)px * pitch + c * 2;
        *reinterpret_cast<T2*>(o + C) = m5;
        *reinterpret_cast<T2*>(o + 2 * C) = m9;
        *reinterpret_cast<T2*>(o + 3 * C) = m13;
    }
}

// ---------------------------------------------------------------- Detect decode
// raw [B][H][W][rp] fp32 (channel = a*no + o)  ->  pred [B][Ntot][no] rows level_off + (a*H + y)*W + x
__global__ void detect_decode_kernel(const float* __restrict__ raw, int rp, float* __restrict__ pred, int B, int H, int W, int na, int no,
                                     long long level_off, long long Ntot, float stride, float a0w, float a0h, float a1w, float a1h,
                                     float a2w, float a2h) {
    const long long total = (long long)B * H * W * na * no;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int o = (int)(i % no);
        long long t = i / no;
        const int x = (int)(t % W); t /= W;
        const int y = (int)(t % H); t /= H;
        const int a = (int)(t % na);
        const int b = (int)(t / na);
        const float r = raw[(((long long)b * H + y) * W + x) * rp + a * no + o];
        float s = b2t::det_sigmoid(r);
        if (o == 0) s = b2t::det_xy(s, (float)x, stride);
        else if (o == 1) s = b2t::det_xy(s, (float)y, stride);
        else if (o == 2) s = b2t::det_wh(s, a == 0 ? a0w : (a == 1 ? a1w : a2w));
        else if (o == 3) s = b2t::det_wh(s, a == 0 ? a0h : (a == 1 ? a1h : a2h));
        pred[((long long)b * Ntot + level_off + ((long long)a * H + y) * W + x) * no + o] = s;
    }
}

inline int grid_for(long long total, int block) { long long g = (total + block - 1) / block; return (int)(g > 132 * 32 ? 132 * 32 : (g < 1 ? 1 : g)); }
}  // namespace

extern "C" const char* b2t_detect_last_error(void) { return g_det_err.c_str(); }

extern "C" int b2t_image_reorg_padded(const float* img, void* out, int B, int H, int W, int row_pixels, int x0, int act_dtype, void* stream) {
    if (!img || !out || (H & 1) || (W & 1) || x0 < 0 || row_pixels < W / 2 + x0 || (act_dtype != B2T_ACT_BF16 && act_dtype != B2T_ACT_F16))
        return dfail(B2T_EINVAL, "b2t_image_reorg_padded: bad arguments");
    const long long total = (long long)B * (H / 2) * (W / 2);
    if (act_dtype == B2T_ACT_F16) image_reorg_kernel<__half><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(img, (__half*)out, B, H, W, row_pixels, x0);
    else image_reorg_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(img, (__nv_bfloat16*)out, B, H, W, row_pixels, x0);
    return dcheck("image_reorg_padded");
}

extern "C" int b2t_image_nhwc16(const float* img, void* out, int B, int H, int W, int act_dtype, void* stream) {
    if (!img || !out || B < 1 || H < 1 || W < 1 || (act_dtype != B2T_ACT_BF16 && act_dtype != B2T_ACT_F16)) return dfail(B2T_EINVAL, "b2t_image_nhwc16: bad arguments");
    const long long total = (long long)B * H * W;
    if (act_dtype == B2T_ACT_F16) image_nhwc16_kernel<__half><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(img, (__half*)out, B, H, W);
    else image_nhwc16_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(img, (__nv_bfloat16*)out, B, H, W);
    return dcheck("image_nhwc16");
}

extern "C" int b2t_image_reorg(const float* img, void* out, int B, int H, int W, int act_dtype, void* stream) {
    return b2t_image_reorg_padded(img, out, B, H, W, W / 2, 0, act_dtype, stream);
}

extern "C" int b2t_upsample2x(const void* src, int src_pitch, int src_coff, void* dst, int dst_pitch, int dst_coff, int B, int H, int W,
                              int C, void* stream) {
    if (!src || !dst || C % 8 || src_pitch % 8 || dst_pitch % 8 || src_coff % 8 || dst_coff % 8) return dfail(B2T_EINVAL, "b2t_upsample2x: channels / pitches must be multiples of 8");
    const long long total = (long long)B * 4 * H * W * (C / 8);
    upsample2x_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)src, src_pitch, src_coff, (__nv_bfloat16*)dst,
                                                                                 dst_pitch, dst_coff, B, H, W, C);
    return dcheck("upsample2x");
}

extern "C" int b2t_spp_pool(void* buf, int pitch, int C, int B, int H, int W, int act_dtype, void* stream) {
    if (!buf || C % 2 || pitch < 4 * C || (act_dtype != B2T_ACT_BF16 && act_dtype != B2T_ACT_F16)) return dfail(B2T_EINVAL, "b2t_spp_pool: bad arguments");
    const size_t plane_smem = (size_t)H * W * 16 * 4;
    const bool f16 = act_dtype == B2T_ACT_F16;
    if (C % 8 == 0 && pitch % 8 == 0 && ((uintptr_t)buf & 15) == 0 && plane_smem <= 48 * 1024) {
        if (f16) spp_pool_plane_kernel<__half><<<dim3(C / 8, B), 256, plane_smem, (cudaStream_t)stream>>>((__half*)buf, pitch, C, H, W);
        else spp_pool_plane_kernel<__nv_bfloat16><<<dim3(C / 8, B), 256, plane_smem, (cudaStream_t)stream>>>((__nv_bfloat16*)buf, pitch, C, H, W);
        return dcheck("spp_pool");
    }
    const long long total = (long long)B * H * W * (C / 2);
    if (f16) spp_pool_kernel<__half><<<grid_for(total, 128), 128, 0, (cudaStream_t)stream>>>((__half*)buf, pitch, C, B, H, W);
    else spp_pool_kernel<__nv_bfloat16><<<grid_for(total, 128), 128, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)buf, pitch, C, B, H, W);
    return dcheck("spp_pool");
}

extern "C" int b2t_detect_decode(const float* raw, int raw_pitch, float* pred, int B, int H, int W, int na, int no, long long level_off,
                                 long long n_total, float stride, const float* anchors_host, void* stream) {
    if (!raw || !pred || na != 3 || !anchors_host) return dfail(B2T_EINVAL, "b2t_detect_decode: bad arguments (na must be 3)");
    const long long total = (long long)B * H * W * na * no;
    detect_decode_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(raw, raw_pitch, pred, B, H, W, na, no, level_off, n_total, stride,
        anchors_host[0], anchors_host[1], anchors_host[2], anchors_host[3], anchors_host[4], anchors_host[5]);
    return dcheck("detect_decode");
}
