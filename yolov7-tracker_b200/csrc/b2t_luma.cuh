// b2t_luma.cuh -- the 8-bit luma and 8-bit INTER_LINEAR down-scale taps shared by the camera-motion estimators (b2t_gmc.cu: ORB,
// b2t_ecc.cu: ECC).  cv2.cvtColor(BGR2GRAY) on uint8 is 15-bit fixed point; cv2.resize(INTER_LINEAR) on uint8 uses 11-bit taps
// (b2t_preproc.cu), except at exactly 1/2 where it is the 2 x 2 mean (INTER_AREA).
#pragma once
#include "b2t_platform.cuh"

namespace {

B2T_DEV int gray_of(const unsigned char* q) { return (q[0] * 3735 + q[1] * 19235 + q[2] * 9798 + (1 << 14)) >> 15; }

B2T_DEV void lin_tap(int d, double scale, int src, int& s, int& w0, int& w1, bool clamp_weight) {     // cv2.resize, 8-bit linear (b2t_preproc.cu)
    float f = (float)((d + 0.5) * scale - 0.5);
    s = (int)floorf(f);
    f -= (float)s;
    if (clamp_weight) {
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
    }
    w1 = __float2int_rn(f * 2048.f);
    w0 = __float2int_rn((1.f - f) * 2048.f);
}

// one pixel (x, y) of cv2.resize(src, INTER_LINEAR) for 8-bit data; at(yy, xx) returns the source value (0 .. 255) at an
// in-range position.  scale_x / scale_y as cv::resize derives them: 1. / (dsize / ssize) in double.
template <class F>
B2T_DEV int resize_linear_px(F at, int x, int y, int src_h, int src_w, double scale_x, double scale_y) {
    int sx, a0, a1, sy, b0, b1;
    lin_tap(x, scale_x, src_w, sx, a0, a1, true);
    lin_tap(y, scale_y, src_h, sy, b0, b1, false);
    const int sx1 = sx + 1 < src_w ? sx + 1 : src_w - 1;
    const int y0 = sy < 0 ? 0 : (sy > src_h - 1 ? src_h - 1 : sy);
    const int y1 = sy + 1 < 0 ? 0 : (sy + 1 > src_h - 1 ? src_h - 1 : sy + 1);
    const int h0 = at(y0, sx) * a0 + at(y0, sx1) * a1;
    const int h1 = at(y1, sx) * a0 + at(y1, sx1) * a1;
    int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

}  // namespace
