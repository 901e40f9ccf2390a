// b2t_preproc.cu -- the reference's per-frame pre-processing as one kernel (SURVEY.md section 8f row 2).
//
// Replaces, for a uint8 BGR frame already in device memory (6 MB for 1080p instead of the 19.7 MB fp32 tensor the
// reference uploads):
//   TrackerLoader._letterbox   tracker/tracker_dataloader.py:100-130  cv2.resize(INTER_LINEAR) + copyMakeBorder(114)
//   TrackerLoader.__getitem__  :80-86                                 BGR -> RGB, HWC -> CHW, .float() / 255
// The geometry (new_unpad, top, left, output size) is computed on the host exactly as :105-126 do
// (b200track/preprocess.py) and passed in.
//
// cv2.resize on 8-bit images is integer arithmetic (OpenCV imgproc/resize.cpp, linear):
//   fx = (float)((dx + 0.5) * scale_x - 0.5), left tap floor(fx), weight clamped at the left / right edge;
//   weights saturate_cast<short>(w * 2048) (round half to even); horizontal pass S[sx]*a0 + S[sx+1]*a1 in int32;
//   vertical pass on rows clip(sy), clip(sy+1):  ((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
//   an exact 2 x 2 down-scale is INTER_AREA: (a + b + c + d + 2) >> 2.
// Reproduced bit for bit (oracle/preprocess.py is pinned against the real cv2 and against the reference's own output);
// the translation unit is compiled with --fmad=false so that (dx + 0.5) * scale - 0.5 rounds twice, as on the host.
// HBM-bound byte work: one thread per output pixel, three channels, 4 taps each; coalesced fp32 plane writes.
#include <string>          // before b2t_platform.cuh (the simulator's __noinline__ macro must not reach libstdc++)
#include "b2t_platform.cuh"
#include "../../include/b200track.h"

namespace b2t { void set_detect_error(const char* m); }

namespace {

struct LetterboxParams {
    int src_h, src_w, src_pitch;       // source rows of src_pitch bytes, 3 bytes per pixel (B, G, R)
    int unpad_w, unpad_h;              // size of the resized image
    int top, left;                     // where it sits inside the output
    int out_h, out_w;
    float pad;                         // border value / 255
    int mode;                          // 0 = copy (no resize), 1 = linear, 2 = exact 2 x 2 area
    double scale_x, scale_y;           // src / dst, as OpenCV computes them (double)
};

B2T_DEV void linear_tap(int d, double scale, int src, int& s, int& w0, int& w1, bool clamp_weight) {
    float f = (float)((d + 0.5) * scale - 0.5);
    s = (int)floorf(f);
    f -= (float)s;
    if (clamp_weight) {                // x axis: OpenCV zeroes the weight at the edges (resize.cpp, xofs / alpha tables)
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
    }
    w1 = __float2int_rn(f * 2048.f);                 // saturate_cast<short>: round half to even
    w0 = __float2int_rn((1.f - f) * 2048.f);
}

// value of canvas pixel (y, x) of image `img` for the three SOURCE channels (B, G, R), or false if it is border
B2T_DEV bool letterbox_pixel(const LetterboxParams& p, const unsigned char* __restrict__ img, int y, int x, int (&v)[3]) {
    const int dy = y - p.top, dx = x - p.left;
    if (dy < 0 || dy >= p.unpad_h || dx < 0 || dx >= p.unpad_w) return false;        // copyMakeBorder(value = 114)
    if (p.mode == 0) {
        const unsigned char* q = img + (long long)dy * p.src_pitch + dx * 3;
        v[0] = q[0]; v[1] = q[1]; v[2] = q[2];
    } else if (p.mode == 2) {
        const unsigned char* q0 = img + (long long)(2 * dy) * p.src_pitch + (2 * dx) * 3;
        const unsigned char* q1 = q0 + p.src_pitch;
        for (int c = 0; c < 3; ++c) v[c] = (q0[c] + q0[3 + c] + q1[c] + q1[3 + c] + 2) >> 2;
    } else {
        int sx, a0, a1, sy, b0, b1;
        linear_tap(dx, p.scale_x, p.src_w, sx, a0, a1, true);
        linear_tap(dy, p.scale_y, p.src_h, sy, b0, b1, false);
        const int sx1 = sx + 1 < p.src_w ? sx + 1 : p.src_w - 1;       // weight a1 is 0 whenever this clamps
        const int y0 = sy < 0 ? 0 : (sy > p.src_h - 1 ? p.src_h - 1 : sy);
        const int y1 = sy + 1 < 0 ? 0 : (sy + 1 > p.src_h - 1 ? p.src_h - 1 : sy + 1);
        const unsigned char* r0 = img + (long long)y0 * p.src_pitch;
        const unsigned char* r1 = img + (long long)y1 * p.src_pitch;
        for (int c = 0; c < 3; ++c) {
            const int h0 = r0[sx * 3 + c] * a0 + r0[sx1 * 3 + c] * a1;
            const int h1 = r1[sx * 3 + c] * a0 + r1[sx1 * 3 + c] * a1;
            v[c] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
            v[c] = v[c] < 0 ? 0 : (v[c] > 255 ? 255 : v[c]);
        }
    }
    return true;
}

__global__ void letterbox_kernel(const unsigned char* __restrict__ src, float* __restrict__ out, int B, LetterboxParams p) {
    const long long plane = (long long)p.out_h * p.out_w;
    const long long total = (long long)B * plane;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / plane);
        const long long r = i - (long long)b * plane;
        const int y = (int)(r / p.out_w), x = (int)(r - (long long)y * p.out_w);
        float* o = out + (long long)b * 3 * plane + r;
        int v[3];
        if (!letterbox_pixel(p, src + (long long)b * p.src_h * p.src_pitch, y, x, v)) {
            o[0] = p.pad; o[plane] = p.pad; o[2 * plane] = p.pad;
            continue;
        }
        // BGR -> RGB planes, float / 255 (IEEE division, like torch's img /= 255.0)
        o[0] = (float)v[2] / 255.0f;
        o[plane] = (float)v[1] / 255.0f;
        o[2 * plane] = (float)v[0] / 255.0f;
    }
}

// float -> bf16 bits, round to nearest even (== __float2bfloat16_rn for finite inputs; integer ops so that the host simulator
// runs the same code)
B2T_DEV unsigned short bf16_bits(float f) {
    const unsigned u = (unsigned)__float_as_int(f);
    return (unsigned short)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}

// float -> IEEE binary16 bits, round to nearest even (== __float2half_rn for the finite non-negative values a [0, 1] canvas holds;
// integer ops, like bf16_bits)
B2T_DEV unsigned short f16_bits(float f) {
    const unsigned u = (unsigned)__float_as_int(f);
    const unsigned sign = (u >> 16) & 0x8000u;
    const unsigned a = u & 0x7fffffffu;
    if (a >= 0x47800000u) return (unsigned short)(sign | (a > 0x7f800000u ? 0x7e00u : 0x7c00u));      // overflow / inf / nan
    if (a < 0x38800000u) {                          // below the smallest normal half: shift the 24-bit significand into place
        if (a < 0x33000000u) return (unsigned short)sign;
        const unsigned e = a >> 23, m = (a & 0x7fffffu) | 0x800000u;
        const unsigned shift = 126u - e;            // 14 .. 24
        const unsigned q = m >> shift, rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1u);
        return (unsigned short)(sign | (q + ((rem > half || (rem == half && (q & 1u))) ? 1u : 0u)));
    }
    const unsigned r = a - 0x38000000u;             // rebias the exponent (127 -> 15), keep 10 mantissa bits
    return (unsigned short)(sign | ((r + 0xfffu + ((r >> 13) & 1u)) >> 13));
}

// The same canvas, written directly in the detector's input layout: ReOrg (models/common.py:52-53, channel = phase * 3 + c with
// phases (dy, dx) = (0,0) (1,0) (0,1) (1,1)) + NHWC bf16 padded to 16 channels, rows of `row_pixels` pixels starting at pixel
// x0 -- what image_reorg_kernel (b2t_detect.cu) produces from the float tensor, without that tensor ever existing.
__global__ void letterbox_reorg_kernel(const unsigned char* __restrict__ src, unsigned short* __restrict__ out, int B, LetterboxParams p,
                                       int row_pixels, int x0, int f16) {
    const int H2 = p.out_h / 2, W2 = p.out_w / 2;
    const long long total = (long long)B * H2 * W2;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W2), y = (int)((i / W2) % H2), b = (int)(i / ((long long)W2 * H2));
        const unsigned char* img = src + (long long)b * p.src_h * p.src_pitch;
        // 16 channels x 2 bytes = two 16-byte stores per pixel (the row layout keeps every pixel 32-byte aligned)
        union { unsigned short o[16]; uint4 v[2]; } px;
        unsigned short* o = px.o;
        for (int ph = 0; ph < 4; ++ph) {
            int v[3];
            const bool in = letterbox_pixel(p, img, 2 * y + (ph & 1), 2 * x + (ph >> 1), v);
            for (int c = 0; c < 3; ++c)                                  // RGB order: channel c reads source channel 2 - c
            {
                const float val = in ? (float)v[2 - c] / 255.0f : p.pad;
                o[ph * 3 + c] = f16 ? f16_bits(val) : bf16_bits(val);
            }
        }
        o[12] = o[13] = o[14] = o[15] = 0;
        uint4* dst = reinterpret_cast<uint4*>(out + ((((long long)b * H2 + y) * row_pixels) + x0 + x) * 16);
        dst[0] = px.v[0];
        dst[1] = px.v[1];
    }
}

int pfail(int code, const char* m) { b2t::set_detect_error(m); return code; }

}  // namespace

namespace {
int make_params(const unsigned char* bgr, int B, int src_h, int src_w, int src_pitch, int unpad_w, int unpad_h, int top, int left, int out_h,
                int out_w, int pad_value, LetterboxParams* p) {
    if (!bgr || B < 1 || src_h < 1 || src_w < 1 || src_pitch < 3 * src_w || unpad_w < 1 || unpad_h < 1 || top < 0 || left < 0 ||
        out_h < top + unpad_h || out_w < left + unpad_w || pad_value < 0 || pad_value > 255)
        return B2T_EINVAL;
    p->src_h = src_h; p->src_w = src_w; p->src_pitch = src_pitch; p->unpad_w = unpad_w; p->unpad_h = unpad_h; p->top = top; p->left = left;
    p->out_h = out_h; p->out_w = out_w;
    p->pad = (float)pad_value / 255.0f;
    // cv::resize derives the scales from inv_scale = dsize / ssize in double: scale = 1. / inv_scale
    p->scale_x = 1.0 / ((double)unpad_w / (double)src_w);
    p->scale_y = 1.0 / ((double)unpad_h / (double)src_h);
    p->mode = (unpad_w == src_w && unpad_h == src_h) ? 0 : ((src_w == 2 * unpad_w && src_h == 2 * unpad_h) ? 2 : 1);
    return B2T_OK;
}
int launch_check(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { b2t::set_detect_error((std::string(what) + ": " + cudaGetErrorString(e)).c_str()); return B2T_ECUDA; }
    return B2T_OK;
}
int grid_of(long long total) { long long g = (total + 255) / 256; return (int)(g > 132 * 16 ? 132 * 16 : (g < 1 ? 1 : g)); }
}  // namespace

extern "C" int b2t_letterbox(const unsigned char* bgr, int B, int src_h, int src_w, int src_pitch, int unpad_w, int unpad_h, int top, int left,
                             int out_h, int out_w, int pad_value, float* out_chw, void* stream) {
    LetterboxParams p;
    if (!out_chw || make_params(bgr, B, src_h, src_w, src_pitch, unpad_w, unpad_h, top, left, out_h, out_w, pad_value, &p) != B2T_OK)
        return pfail(B2T_EINVAL, "b2t_letterbox: bad arguments");
    B2T_LAUNCH(letterbox_kernel, grid_of((long long)B * out_h * out_w), 256, 0, (cudaStream_t)stream, bgr, out_chw, B, p);
    return launch_check("letterbox");
}

extern "C" int b2t_letterbox_reorg(const unsigned char* bgr, int B, int src_h, int src_w, int src_pitch, int unpad_w, int unpad_h, int top,
                                   int left, int out_h, int out_w, int pad_value, void* out_nhwc16, int row_pixels, int x0, int act_dtype, void* stream) {
    LetterboxParams p;
    if (!out_nhwc16 || (out_h & 1) || (out_w & 1) || x0 < 0 || row_pixels < out_w / 2 + x0 || (act_dtype != B2T_ACT_BF16 && act_dtype != B2T_ACT_F16) ||
        make_params(bgr, B, src_h, src_w, src_pitch, unpad_w, unpad_h, top, left, out_h, out_w, pad_value, &p) != B2T_OK)
        return pfail(B2T_EINVAL, "b2t_letterbox_reorg: bad arguments");
    B2T_LAUNCH(letterbox_reorg_kernel, grid_of((long long)B * (out_h / 2) * (out_w / 2)), 256, 0, (cudaStream_t)stream, bgr,
               (unsigned short*)out_nhwc16, B, p, row_pixels, x0, act_dtype == B2T_ACT_F16 ? 1 : 0);
    return launch_check("letterbox_reorg");
}
