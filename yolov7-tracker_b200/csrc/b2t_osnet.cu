// b2t_osnet.cu -- StrongSORT's appearance network, OSNet x0.25 (tracker/strongsort.py:26-29, :47-89; tracker/reid_models/OSNet.py), on
// crops of any H x W that is a multiple of 16 (the reference's 128 x 256).  Eval-mode BatchNorm is folded into the weights on the host
// (b200track/osnet.py); every kernel reads NHWC 16-bit activations, accumulates in fp32 with fmaf in a fixed order and writes NHWC 16-bit:
//   osnet_crop_kernel       StrongSORT.reid_preprocess :47-64: / 255, cv2.resize(dsize=(out_w, out_h)) bilinear on float, Normalize;
//                           out [n][out_h][out_w][4] (B, G, R, 0)
//   osnet_stem_kernel       conv1 (7 x 7 / s2 / p3, 3 -> 16) + BN + ReLU and maxpool (3 x 3 / s2 / p1) on one tile: only the pooled map
//                           is written
//   osnet_pointwise_kernel  a 1 x 1 conv + BN (+ ReLU) over one or two inputs (block conv3 and the downsample branch share one
//                           accumulator), an optional residual before the ReLU, and the transition's AvgPool 2 x 2 fused
//   osnet_lightconv_kernel  LightConv3x3: 1 x 1 (no bias) -> depthwise 3 x 3 -> BN -> ReLU on a halo tile; the 1 x 1 output stays fp32 in
//                           shared memory (it has no bias, so the depthwise conv's zero padding is the 1 x 1 of zero input)
//   osnet_gate_sum_kernel   x2 = sum over the four streams of ChannelGate(stream): ONE gate (avg pool -> fc1 -> ReLU -> fc2 -> sigmoid)
//                           shared by the streams, each stream pooled on its own; one block per crop, written once
//   osnet_head_kernel       global average pool -> Linear -> BatchNorm1d -> ReLU -> (n, m) float32 (not normalised)
// The unit is compiled without FMA contraction (build.py), so its only fused multiply-adds are the explicit fmaf calls; the host
// simulator (tests/hostsim) computes the same expressions.
#include <string>          // before b2t_platform.cuh (the simulator's __noinline__ macro must not reach libstdc++)
#include <math.h>
#include "b2t_platform.cuh"
#if !defined(B2T_HOSTSIM)
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#endif
#include "../../include/b200track.h"

namespace b2t { void set_detect_error(const char* m); }

namespace {

int ofail(int code, const char* m) { b2t::set_detect_error(m); return code; }
int ocheck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { b2t::set_detect_error((std::string(what) + ": " + cudaGetErrorString(e)).c_str()); return B2T_ECUDA; }
    return B2T_OK;
}
int grid_cap(long long items, int per_block, int cap) {
    const long long g = (items + per_block - 1) / per_block;
    return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}
bool dtype_ok(int d) { return d == B2T_ACT_BF16 || d == B2T_ACT_F16; }

__device__ __forceinline__ float ld16(const unsigned short* p, int f16) {
    return f16 ? __half2float(*reinterpret_cast<const __half*>(p)) : __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(p));
}
__device__ __forceinline__ float cv16(unsigned short b, int f16) { return ld16(&b, f16); }
__device__ __forceinline__ unsigned short st16(float v, int f16) {
    if (f16) { const __half h = __float2half_rn(v); return *reinterpret_cast<const unsigned short*>(&h); }
    const __nv_bfloat16 h = __float2bfloat16_rn(v); return *reinterpret_cast<const unsigned short*>(&h);
}
// 8 consecutive 16-bit values -> fp32
// (vectors are reinterpreted through unions: g++ builds the host simulator with strict aliasing)
__device__ __forceinline__ void unpack8(const unsigned short* p, float* v, int f16) {
    union { uint4 q; unsigned short s[8]; } u;
    u.q = *reinterpret_cast<const uint4*>(p);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = cv16(u.s[k], f16);
}
__device__ __forceinline__ void pack8(unsigned short* p, const float* v, int f16) {
    union { unsigned short o[8]; uint4 q; } r;
#pragma unroll
    for (int k = 0; k < 8; ++k) r.o[k] = st16(v[k], f16);
    *reinterpret_cast<uint4*>(p) = r.q;
}

// ---------------------------------------------------------------- crops
// cv2.resize INTER_LINEAR on float32: source coordinate (float)((d + 0.5) * scale - 0.5), left tap floor(), weight zeroed and tap
// clamped at both edges (the rule of b2t_reid.cu's crop kernel)
__device__ __forceinline__ void tap(int d, double scale, int src, int& s0, int& s1, float& f) {
    f = (float)((d + 0.5) * scale - 0.5);
    s0 = (int)floorf(f);
    f -= (float)s0;
    if (s0 < 0) { f = 0.f; s0 = 0; }
    if (s0 >= src - 1) { f = 0.f; s0 = src - 1; }
    s1 = s0 + 1 < src ? s0 + 1 : src - 1;
}

// crops[i] = {byte offset of the crop's first pixel in `pixels`, row pitch in bytes, height, width}
__global__ void osnet_crop_kernel(const unsigned char* __restrict__ pixels, const long long* __restrict__ crops, int n, int oh, int ow,
                                  unsigned short* __restrict__ out, int f16) {
    const long long total = (long long)n * oh * ow;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % ow), y = (int)((i / ow) % oh);
        const long long c = i / ((long long)ow * oh);
        const long long* cr = crops + c * 4;
        const unsigned char* img = pixels + cr[0];
        const int pitch = (int)cr[1], h = (int)cr[2], w = (int)cr[3];
        int x0, x1, y0, y1; float fx, fy;
        tap(x, 1.0 / ((double)ow / (double)w), w, x0, x1, fx);
        tap(y, 1.0 / ((double)oh / (double)h), h, y0, y1, fy);
        const unsigned char* r0 = img + (size_t)y0 * pitch;
        const unsigned char* r1 = img + (size_t)y1 * pitch;
        const float mean[3] = {0.485f, 0.456f, 0.406f}, sd[3] = {0.229f, 0.224f, 0.225f};
        union { unsigned short o[4]; uint2 v; } px;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            const float a0 = (float)r0[x0 * 3 + ch] / 255.0f, a1 = (float)r0[x1 * 3 + ch] / 255.0f;
            const float b0 = (float)r1[x0 * 3 + ch] / 255.0f, b1 = (float)r1[x1 * 3 + ch] / 255.0f;
            const float top = a0 * (1.f - fx) + a1 * fx, bot = b0 * (1.f - fx) + b1 * fx;
            px.o[ch] = st16(((top * (1.f - fy) + bot * fy) - mean[ch]) / sd[ch], f16);      // channels as they arrive (B, G, R)
        }
        px.o[3] = 0;
        *reinterpret_cast<uint2*>(out + i * 4) = px.v;
    }
}

// ---------------------------------------------------------------- stem: conv 7 x 7 / s2 / p3 (3 -> 16) + bias + ReLU, max-pool 3 x 3 / s2 / p1
constexpr int kStemTY = 8, kStemTX = 16;                            // pooled outputs per block
constexpr int kStemCY = 2 * kStemTY + 1, kStemCX = 2 * kStemTX + 1;  // conv outputs the tile's pools read (17 x 33)
constexpr int kStemIY = 2 * kStemCY + 5, kStemIX = 2 * kStemCX + 5;  // input pixels those convs read (39 x 71)
constexpr int kStemC = 16;
constexpr size_t kStemSmem = (size_t)(kStemIY * kStemIX * 4 + kStemCY * kStemCX * kStemC + 147 * kStemC + kStemC) * sizeof(float);

// x [n][h][w][pitch] (channels 0..2 read), wt [(ky * 7 + kx) * 3 + ci][16], y [n][h/4][w/4][16]
__global__ void __launch_bounds__(256) osnet_stem_kernel(const unsigned short* __restrict__ x, int pitch, const float* __restrict__ wt, const float* __restrict__ bias,
                                                         int h, int w, int tiles_x, int tiles_y, unsigned short* __restrict__ y, int f16) {
    B2T_DYN_SMEM(smem);
    float* s_in = reinterpret_cast<float*>(smem);                   // [kStemIY][kStemIX][4]
    float* s_cv = s_in + kStemIY * kStemIX * 4;                     // [kStemCY * kStemCX][16], -inf outside the conv map
    float* s_w = s_cv + kStemCY * kStemCX * kStemC;                 // [147][16]
    float* s_b = s_w + 147 * kStemC;
    const int t = threadIdx.x;
    const int tile = blockIdx.x % (tiles_x * tiles_y), b = blockIdx.x / (tiles_x * tiles_y);
    const int py0 = (tile / tiles_x) * kStemTY, px0 = (tile % tiles_x) * kStemTX;
    const int hc = h / 2, wc = w / 2, hp = hc / 2, wp = wc / 2;
    const int cy0 = 2 * py0 - 1, cx0 = 2 * px0 - 1;                // first conv row / column of the tile
    const int iy0 = 2 * cy0 - 3, ix0 = 2 * cx0 - 3;                // first input row / column
    for (int i = t; i < 147 * kStemC; i += blockDim.x) s_w[i] = wt[i];
    if (t < kStemC) s_b[t] = bias[t];
    const unsigned short* xb = x + (size_t)b * h * w * pitch;
    for (int i = t; i < kStemIY * kStemIX; i += blockDim.x) {
        const int yy = iy0 + i / kStemIX, xx = ix0 + i % kStemIX;
        float v[4] = {0.f, 0.f, 0.f, 0.f};                          // zero padding
        if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
            union { uint2 q; unsigned short s[4]; } u;
            u.q = *reinterpret_cast<const uint2*>(xb + ((size_t)yy * w + xx) * pitch);
#pragma unroll
            for (int k = 0; k < 3; ++k) v[k] = cv16(u.s[k], f16);
        }
        *reinterpret_cast<float4*>(s_in + i * 4) = make_float4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();
    for (int i = t; i < kStemCY * kStemCX; i += blockDim.x) {
        const int ly = i / kStemCX, lx = i % kStemCX;
        const int cy = cy0 + ly, cx = cx0 + lx;
        float* dst = s_cv + i * kStemC;
        if (cy < 0 || cy >= hc || cx < 0 || cx >= wc) {              // the pool's padding: never the maximum
#pragma unroll
            for (int co = 0; co < kStemC; ++co) dst[co] = -INFINITY;
            continue;
        }
        float acc[kStemC];
#pragma unroll
        for (int co = 0; co < kStemC; ++co) acc[co] = 0.f;
        for (int ky = 0; ky < 7; ++ky) {
            const float* row = s_in + ((2 * ly + ky) * kStemIX + 2 * lx) * 4;
#pragma unroll
            for (int kx = 0; kx < 7; ++kx) {
                const float4 v = *reinterpret_cast<const float4*>(row + kx * 4);
                const float* wr = s_w + (ky * 7 + kx) * 3 * kStemC;
#pragma unroll
                for (int co = 0; co < kStemC; ++co) {
                    acc[co] = fmaf(v.x, wr[co], acc[co]);
                    acc[co] = fmaf(v.y, wr[kStemC + co], acc[co]);
                    acc[co] = fmaf(v.z, wr[2 * kStemC + co], acc[co]);
                }
            }
        }
#pragma unroll
        for (int co = 0; co < kStemC; ++co) dst[co] = fmaxf(acc[co] + s_b[co], 0.f);
    }
    __syncthreads();
    // pooled pixel t / 2, channels 8 (t & 1) .. +8: max of the 3 x 3 conv window, then one rounding (max and rounding commute)
    const int lp = t >> 1, half = t & 1;
    const int ly = lp / kStemTX, lx = lp % kStemTX;
    const int py = py0 + ly, px = px0 + lx;
    if (lp < kStemTY * kStemTX && py < hp && px < wp) {
        float m[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) m[k] = -INFINITY;
        for (int dy = 0; dy < 3; ++dy)
            for (int dx = 0; dx < 3; ++dx) {
                const float* s = s_cv + ((2 * ly + dy) * kStemCX + 2 * lx + dx) * kStemC + half * 8;
#pragma unroll
                for (int k = 0; k < 8; ++k) m[k] = fmaxf(m[k], s[k]);
            }
        pack8(y + (((size_t)b * hp + py) * wp + px) * kStemC + half * 8, m, f16);
    }
}

// ---------------------------------------------------------------- 1 x 1 conv (+ second input, residual, ReLU, 2 x 2 average pool)
// Thread item = (quad, 8 output channels).  quad: 4 consecutive pixels of the flat [n * h * w] map, or (pool) the 2 x 2 window of one
// output pixel.  y = act(sum_ci xa * wa + sum_ci xb * wb + bias (+ res)); pool: the mean of the window's four values after act.
// w [(ca + cb)][cout]: the rows of xa, then those of xb.
constexpr int kPwThreads = 256;

__global__ void __launch_bounds__(kPwThreads) osnet_pointwise_kernel(const unsigned short* __restrict__ xa, int ca, const unsigned short* __restrict__ xb, int cb,
                                                                     const float* __restrict__ wt, const float* __restrict__ bias,
                                                                     const unsigned short* __restrict__ res, unsigned short* __restrict__ y,
                                                                     int n, int h, int w, int cout, int relu, int pool, int f16) {
    B2T_DYN_SMEM(smem);
    float* s_w = reinterpret_cast<float*>(smem);
    float* s_b = s_w + (ca + cb) * cout;
    for (int i = threadIdx.x; i < (ca + cb) * cout; i += blockDim.x) s_w[i] = wt[i];
    for (int i = threadIdx.x; i < cout; i += blockDim.x) s_b[i] = bias[i];
    __syncthreads();
    const int ncg = cout / 8;
    const long long npix = (long long)n * h * w;
    const long long nquad = pool ? npix / 4 : (npix + 3) / 4;
    const int ho = h / 2, wo = w / 2;
    for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < nquad * ncg; it += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(it % ncg);
        const long long q = it / ncg;
        long long pix[4];
        if (pool) {
            const int ox = (int)(q % wo), oy = (int)((q / wo) % ho);
            const long long b = q / ((long long)wo * ho);
            const long long p0 = (b * h + 2 * oy) * w + 2 * ox;
            pix[0] = p0; pix[1] = p0 + 1; pix[2] = p0 + w; pix[3] = p0 + w + 1;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) pix[j] = 4 * q + j < npix ? 4 * q + j : -1;
        }
        float acc[4][8];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[j][k] = 0.f;
        for (int part = 0; part < 2; ++part) {
            const unsigned short* xs = part ? xb : xa;
            const int c = part ? cb : ca;
            const float* wbase = s_w + (part ? ca : 0) * cout + cg * 8;
            for (int c0 = 0; c0 < c; c0 += 8) {
                float xv[4][8];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (pix[j] >= 0) unpack8(xs + pix[j] * c + c0, xv[j], f16);
                    else
#pragma unroll
                        for (int k = 0; k < 8; ++k) xv[j][k] = 0.f;
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float4 w0 = *reinterpret_cast<const float4*>(wbase + (c0 + k) * cout);
                    const float4 w1 = *reinterpret_cast<const float4*>(wbase + (c0 + k) * cout + 4);
                    const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int o = 0; o < 8; ++o) acc[j][o] = fmaf(xv[j][k], wv[o], acc[j][o]);
                }
            }
        }
        float rv[8];
        if (pool) {
#pragma unroll
            for (int o = 0; o < 8; ++o) {
                float s = 0.f;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float v = acc[j][o] + s_b[cg * 8 + o];
                    if (relu) v = fmaxf(v, 0.f);
                    s += v;
                }
                rv[o] = s * 0.25f;
            }
            pack8(y + q * cout + cg * 8, rv, f16);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (pix[j] < 0) continue;
                float r[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
                if (res) unpack8(res + pix[j] * cout + cg * 8, r, f16);
#pragma unroll
                for (int o = 0; o < 8; ++o) {
                    float v = acc[j][o] + s_b[cg * 8 + o];
                    if (res) v += r[o];
                    rv[o] = relu ? fmaxf(v, 0.f) : v;
                }
                pack8(y + pix[j] * cout + cg * 8, rv, f16);
            }
        }
    }
}

// ---------------------------------------------------------------- LightConv3x3: 1 x 1 (c x c, no bias) -> depthwise 3 x 3 -> bias -> ReLU
constexpr int kLcTY = 8, kLcTX = 16, kLcHY = kLcTY + 2, kLcHX = kLcTX + 2;

// x, y [n][h][w][c]; w1 [ci][co]; dw [tap = dy * 3 + dx][c] (BN scale folded); bias [c]
__global__ void __launch_bounds__(256) osnet_lightconv_kernel(const unsigned short* __restrict__ x, const float* __restrict__ w1, const float* __restrict__ dw,
                                                              const float* __restrict__ bias, unsigned short* __restrict__ y, int h, int w, int c,
                                                              int tiles_x, int tiles_y, int f16) {
    B2T_DYN_SMEM(smem);
    float* s_t = reinterpret_cast<float*>(smem);                    // [kLcHY * kLcHX][c]: the 1 x 1 output on the halo tile, fp32
    float* s_w1 = s_t + kLcHY * kLcHX * c;                          // [c][c]
    float* s_dw = s_w1 + c * c;                                     // [9][c]
    float* s_b = s_dw + 9 * c;
    const int t = threadIdx.x, ncg = c / 8;
    const int tile = blockIdx.x % (tiles_x * tiles_y), b = blockIdx.x / (tiles_x * tiles_y);
    const int oy0 = (tile / tiles_x) * kLcTY, ox0 = (tile % tiles_x) * kLcTX;
    for (int i = t; i < c * c; i += blockDim.x) s_w1[i] = w1[i];
    for (int i = t; i < 9 * c; i += blockDim.x) s_dw[i] = dw[i];
    for (int i = t; i < c; i += blockDim.x) s_b[i] = bias[i];
    __syncthreads();
    const unsigned short* xb = x + (size_t)b * h * w * c;
    for (int i = t; i < kLcHY * kLcHX * ncg; i += blockDim.x) {
        const int hp = i / ncg, cg = i % ncg;
        const int yy = oy0 - 1 + hp / kLcHX, xx = ox0 - 1 + hp % kLcHX;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};    // outside the map: the depthwise conv's zero padding
        if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
            const unsigned short* px = xb + ((size_t)yy * w + xx) * c;
            for (int c0 = 0; c0 < c; c0 += 8) {
                float xv[8];
                unpack8(px + c0, xv, f16);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float4 a = *reinterpret_cast<const float4*>(s_w1 + (c0 + k) * c + cg * 8);
                    const float4 bq = *reinterpret_cast<const float4*>(s_w1 + (c0 + k) * c + cg * 8 + 4);
                    const float wv[8] = {a.x, a.y, a.z, a.w, bq.x, bq.y, bq.z, bq.w};
#pragma unroll
                    for (int o = 0; o < 8; ++o) acc[o] = fmaf(xv[k], wv[o], acc[o]);
                }
            }
        }
        float* dst = s_t + hp * c + cg * 8;
        *reinterpret_cast<float4*>(dst) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    __syncthreads();
    for (int i = t; i < kLcTY * kLcTX * ncg; i += blockDim.x) {
        const int op = i / ncg, cg = i % ncg;
        const int ly = op / kLcTX, lx = op % kLcTX;
        const int oy = oy0 + ly, ox = ox0 + lx;
        if (oy >= h || ox >= w) continue;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const float* s = s_t + ((ly + dy) * kLcHX + lx + dx) * c + cg * 8;
                const float* wd = s_dw + (dy * 3 + dx) * c + cg * 8;
#pragma unroll
                for (int o = 0; o < 8; ++o) acc[o] = fmaf(s[o], wd[o], acc[o]);
            }
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = fmaxf(acc[o] + s_b[cg * 8 + o], 0.f);
        pack8(y + (((size_t)b * h + oy) * w + ox) * c + cg * 8, acc, f16);
    }
}

// ---------------------------------------------------------------- shared ChannelGate over the four streams, summed
constexpr int kGateThreads = 256, kGateMaxC = 64, kGateMaxHidden = 16;

// s0..s3, y [n][hw][c]; fc1_w [hidden][c], fc1_b [hidden], fc2_w [c][hidden], fc2_b [c].  One block per crop.
__global__ void __launch_bounds__(kGateThreads) osnet_gate_sum_kernel(const unsigned short* __restrict__ s0, const unsigned short* __restrict__ s1,
                                                                      const unsigned short* __restrict__ s2, const unsigned short* __restrict__ s3,
                                                                      const float* __restrict__ fc1_w, const float* __restrict__ fc1_b,
                                                                      const float* __restrict__ fc2_w, const float* __restrict__ fc2_b,
                                                                      unsigned short* __restrict__ y, int hw, int c, int hidden, int f16) {
    __shared__ float part[4][kGateThreads][8];
    __shared__ float pooled[4][kGateMaxC];
    __shared__ float hid[4][kGateMaxHidden];
    __shared__ float gate[4][kGateMaxC];
    const int t = threadIdx.x, nv = c / 8, lanes = kGateThreads / nv;
    const size_t base = (size_t)blockIdx.x * hw * c;
    const unsigned short* src[4] = {s0 + base, s1 + base, s2 + base, s3 + base};
    // 1. per stream and channel: lane l sums pixels l, l + lanes, ...; then the lanes in order
    if (t < lanes * nv) {
        const int v = t % nv, lane = t / nv;
        float acc[4][8];
#pragma unroll
        for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[s][k] = 0.f;
        for (int p = lane; p < hw; p += lanes)
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                float xv[8];
                unpack8(src[s] + (size_t)p * c + v * 8, xv, f16);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[s][k] += xv[k];
            }
#pragma unroll
        for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int k = 0; k < 8; ++k) part[s][t][k] = acc[s][k];
    }
    __syncthreads();
    if (t < 4 * c) {
        const int s = t / c, ch = t % c;
        float sum = 0.f;
        for (int lane = 0; lane < lanes; ++lane) sum += part[s][lane * nv + ch / 8][ch % 8];
        pooled[s][ch] = sum / (float)hw;
    }
    __syncthreads();
    // 2. the one gate, applied to each stream's pooled vector
    if (t < 4 * hidden) {
        const int s = t / hidden, j = t % hidden;
        float a = 0.f;
        for (int ch = 0; ch < c; ++ch) a = fmaf(fc1_w[j * c + ch], pooled[s][ch], a);
        hid[s][j] = fmaxf(a + fc1_b[j], 0.f);
    }
    __syncthreads();
    if (t < 4 * c) {
        const int s = t / c, ch = t % c;
        float a = 0.f;
        for (int j = 0; j < hidden; ++j) a = fmaf(fc2_w[ch * hidden + j], hid[s][j], a);
        gate[s][ch] = 1.f / (1.f + expf(-(a + fc2_b[ch])));
    }
    __syncthreads();
    // 3. x2 = g0 * s0 + g1 * s1 + g2 * s2 + g3 * s3, in that order
    for (int i = t; i < hw * nv; i += blockDim.x) {
        const int p = i / nv, v = i % nv;
        float out[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            float xv[8];
            unpack8(src[s] + (size_t)p * c + v * 8, xv, f16);
#pragma unroll
            for (int k = 0; k < 8; ++k) out[k] += gate[s][v * 8 + k] * xv[k];
        }
        pack8(y + base + (size_t)p * c + v * 8, out, f16);
    }
}

// ---------------------------------------------------------------- head: global average pool -> Linear + BatchNorm1d (folded) -> ReLU
constexpr int kHeadThreads = 256, kHeadMaxC = 256;

// x [n][hw][c], wt [c][m], bias [m] -> out [n][m] float32.  One block per crop.
__global__ void __launch_bounds__(kHeadThreads) osnet_head_kernel(const unsigned short* __restrict__ x, const float* __restrict__ wt, const float* __restrict__ bias,
                                                                  float* __restrict__ out, int hw, int c, int m, int f16) {
    __shared__ float pooled[kHeadMaxC];
    const int t = threadIdx.x;
    const unsigned short* xb = x + (size_t)blockIdx.x * hw * c;
    if (t < c) {
        float s = 0.f;
        for (int p = 0; p < hw; ++p) s += ld16(xb + (size_t)p * c + t, f16);
        pooled[t] = s / (float)hw;
    }
    __syncthreads();
    for (int o = t; o < m; o += blockDim.x) {
        float a = 0.f;
        for (int ci = 0; ci < c; ++ci) a = fmaf(pooled[ci], wt[(size_t)ci * m + o], a);
        out[(size_t)blockIdx.x * m + o] = fmaxf(a + bias[o], 0.f);
    }
}

}  // namespace

extern "C" int b2t_osnet_crops(const unsigned char* pixels, const long long* crops, int n, int out_h, int out_w, void* out_nhwc4, int act_dtype,
                               void* stream) {
    if (!pixels || !crops || !out_nhwc4 || n < 1 || out_h < 1 || out_w < 1 || !dtype_ok(act_dtype))
        return ofail(B2T_EINVAL, "b2t_osnet_crops: bad arguments");
    B2T_LAUNCH(osnet_crop_kernel, grid_cap((long long)n * out_h * out_w, 256, 132 * 16), 256, 0, (cudaStream_t)stream, pixels, crops, n, out_h, out_w,
               (unsigned short*)out_nhwc4, act_dtype == B2T_ACT_F16);
    return ocheck("osnet_crops");
}

extern "C" int b2t_osnet_stem(const void* x, int pitch, const float* wt, const float* bias, int n, int height, int width, void* y, int act_dtype, void* stream) {
    if (!x || !wt || !bias || !y || pitch < 4 || pitch % 4 || n < 1 || height < 4 || width < 4 || height % 4 || width % 4 || !dtype_ok(act_dtype))
        return ofail(B2T_EINVAL, "b2t_osnet_stem: bad arguments (pitch a multiple of 4, height and width multiples of 4)");
    const int hp = height / 4, wp = width / 4;
    const int tx = (wp + kStemTX - 1) / kStemTX, ty = (hp + kStemTY - 1) / kStemTY;
    if ((long long)tx * ty * n > 0x7fffffffLL) return ofail(B2T_EINVAL, "b2t_osnet_stem: too many tiles");
    if (B2T_SET_SMEM(osnet_stem_kernel, kStemSmem) != 0) return ocheck("osnet_stem smem");
    B2T_LAUNCH(osnet_stem_kernel, tx * ty * n, 256, kStemSmem, (cudaStream_t)stream, (const unsigned short*)x, pitch, wt, bias, height, width, tx, ty,
               (unsigned short*)y, act_dtype == B2T_ACT_F16);
    return ocheck("osnet_stem");
}

extern "C" int b2t_osnet_pointwise(const void* xa, int ca, const void* xb, int cb, const float* wt, const float* bias, const void* res, void* y,
                                   int n, int height, int width, int cout, int relu, int pool, int act_dtype, void* stream) {
    if (!xa || !wt || !bias || !y || n < 1 || height < 1 || width < 1 || ca < 8 || ca % 8 || cb < 0 || cb % 8 || (cb > 0) != (xb != nullptr) ||
        cout < 8 || cout % 8 || (long long)(ca + cb) * cout > 24576 || !dtype_ok(act_dtype) || (pool && (res || height % 2 || width % 2)))
        return ofail(B2T_EINVAL, "b2t_osnet_pointwise: bad arguments (channels multiples of 8, (ca + cb) * cout <= 24576, pool: even sides, no residual)");
    const size_t smem = ((size_t)(ca + cb) * cout + cout) * sizeof(float);
    const long long npix = (long long)n * height * width;
    const long long items = (pool ? npix / 4 : (npix + 3) / 4) * (cout / 8);
    if (B2T_SET_SMEM(osnet_pointwise_kernel, smem) != 0) return ocheck("osnet_pointwise smem");
    B2T_LAUNCH(osnet_pointwise_kernel, grid_cap(items, kPwThreads, 132 * 4), kPwThreads, smem, (cudaStream_t)stream, (const unsigned short*)xa, ca,
               (const unsigned short*)xb, cb, wt, bias, (const unsigned short*)res, (unsigned short*)y, n, height, width, cout, relu ? 1 : 0, pool ? 1 : 0,
               act_dtype == B2T_ACT_F16);
    return ocheck("osnet_pointwise");
}

extern "C" int b2t_osnet_lightconv(const void* x, const float* w1, const float* dw, const float* bias, void* y, int n, int height, int width, int c,
                                   int act_dtype, void* stream) {
    if (!x || !w1 || !dw || !bias || !y || x == y || n < 1 || height < 1 || width < 1 || c < 8 || c % 8 || c > 64 || !dtype_ok(act_dtype))
        return ofail(B2T_EINVAL, "b2t_osnet_lightconv: bad arguments (8 <= c <= 64, c % 8 == 0, not in place)");
    const int tx = (width + kLcTX - 1) / kLcTX, ty = (height + kLcTY - 1) / kLcTY;
    if ((long long)tx * ty * n > 0x7fffffffLL) return ofail(B2T_EINVAL, "b2t_osnet_lightconv: too many tiles");
    const size_t smem = ((size_t)kLcHY * kLcHX * c + (size_t)c * c + 10 * (size_t)c) * sizeof(float);
    if (B2T_SET_SMEM(osnet_lightconv_kernel, smem) != 0) return ocheck("osnet_lightconv smem");
    B2T_LAUNCH(osnet_lightconv_kernel, tx * ty * n, 256, smem, (cudaStream_t)stream, (const unsigned short*)x, w1, dw, bias, (unsigned short*)y, height, width, c,
               tx, ty, act_dtype == B2T_ACT_F16);
    return ocheck("osnet_lightconv");
}

extern "C" int b2t_osnet_gate_sum(const void* s0, const void* s1, const void* s2, const void* s3, const float* fc1_w, const float* fc1_b,
                                  const float* fc2_w, const float* fc2_b, void* y, int n, int hw, int c, int hidden, int act_dtype, void* stream) {
    if (!s0 || !s1 || !s2 || !s3 || !fc1_w || !fc1_b || !fc2_w || !fc2_b || !y || n < 1 || hw < 1 || c < 8 || c % 8 || c > kGateMaxC ||
        hidden < 1 || hidden > kGateMaxHidden || !dtype_ok(act_dtype))
        return ofail(B2T_EINVAL, "b2t_osnet_gate_sum: bad arguments (8 <= c <= 64, c % 8 == 0, 1 <= hidden <= 16)");
    B2T_LAUNCH(osnet_gate_sum_kernel, n, kGateThreads, 0, (cudaStream_t)stream, (const unsigned short*)s0, (const unsigned short*)s1, (const unsigned short*)s2,
               (const unsigned short*)s3, fc1_w, fc1_b, fc2_w, fc2_b, (unsigned short*)y, hw, c, hidden, act_dtype == B2T_ACT_F16);
    return ocheck("osnet_gate_sum");
}

extern "C" int b2t_osnet_head(const void* x, const float* wt, const float* bias, float* out, int n, int hw, int c, int m, int act_dtype, void* stream) {
    if (!x || !wt || !bias || !out || n < 1 || hw < 1 || c < 1 || c > kHeadMaxC || m < 1 || !dtype_ok(act_dtype))
        return ofail(B2T_EINVAL, "b2t_osnet_head: bad arguments (1 <= c <= 256)");
    B2T_LAUNCH(osnet_head_kernel, n, kHeadThreads, 0, (cudaStream_t)stream, (const unsigned short*)x, wt, bias, out, hw, c, m, act_dtype == B2T_ACT_F16);
    return ocheck("osnet_head");
}
