// b2t_gmc.cu -- camera-motion estimation on the GPU (SURVEY.md section 8f row 1).
//
// Replaces GMC.applyFeaures, method 'orb' / downscale 2 -- what BoTSORT.__init__ builds -- of tracker/botsort.py:111-235, which
// costs the reference ~150 ms of host OpenCV per frame:
//   :114-121  cvtColor(BGR2GRAY) + resize to 1/downscale           gray_kernel          bit-exact (15-bit fixed point; 2x2 mean)
//   :123-130  mask: central 96 % of the frame minus detection boxes nms_flag_kernel      exact
//   :132      FastFeatureDetector_create(20).detect                 fast_score_kernel +  exact: same corners, same order
//                                                                    nms_flag / scan / compact
//   :135      ORB_create().compute (given key points: angle -1)     blur_kernel + describe_kernel   bit-exact up to rounding ties of
//                                                                    the float blur (a few pixels per million)
//   :149      BFMatcher(NORM_HAMMING).knnMatch(prev, cur, 2)        match_kernel         exact, ties -> lower train index
//   :158-198  ratio 0.9, |d| < size / 4, one-sided 2.5 sigma filter  filter_kernel       exact
//   :221      cv2.estimateAffinePartial2D(RANSAC)                    ransac_kernel + fit_kernel   same scheme (minimal samples of two pairs ->
//             similarity, inliers < 3 px, most inliers wins, least-squares refit on them -- what OpenCV's LM refinement converges
//             to), own sampling sequence: equal to OpenCV whenever both find the same inlier set, otherwise within its own
//             run-to-run spread (tests: 1e-3 on the linear part, 0.25 px on the translation)
// One call handles n_seq independent sequences (blockIdx.y); all state (previous key points + descriptors, frame counter) lives in
// the caller's workspace, nothing is allocated, nothing synchronises.  Byte / integer work, HBM- and latency-bound: no tensor
// cores.  The 256 ORB point pairs are a generated table (tools/extract_orb_pattern.py).
// Compiled with --fmad=false: the float blur and the double-precision fit round like the host code they are compared with.
#include <string>          // before b2t_platform.cuh (the simulator's __noinline__ macro must not reach libstdc++)
#include <math.h>
#include "b2t_platform.cuh"
#include "../../include/b200track.h"

namespace b2t { void set_detect_error(const char* m); }

namespace {

constexpr int kFastThreshold = 20;     // botsort.py:20
constexpr int kOrbEdge = 31;           // ORB_create() default edgeThreshold
constexpr int kSplit = 16;             // train-set slices of the matcher (blockIdx.z): enough blocks to hide the shared-memory latency
constexpr int kMaxBoxes = 256;         // detection boxes cached per image row by the mask test
constexpr int kHyp = 512;              // RANSAC hypotheses (oracle/gmc.py: RANSAC_HYPOTHESES)
constexpr int kHypBlocks = 16;         // blocks per sequence that score them
constexpr int kEstThreads = 1024;
constexpr int kStateWords = 16;

__constant__ signed char kOrbPairs[256][2][2] = {
#include "b2t_orb_pattern.inc"
};

struct GmcGeom {
    int n_seq, src_h, src_w, pitch, ds;
    int h, w;                          // working (down-scaled) size
    int wpr;                           // 32-bit flag words per row
    int max_kp;
    int mx0, mx1, my0, my1;            // central mask region (botsort.py:125)
    int slot;                          // plane set (blurred image, FAST scores) this call works on
    size_t plane;                      // bytes between the two plane sets
    // per-sequence workspace offsets (bytes)
    size_t o_state, o_gray, o_blur, o_score, o_flags, o_rowoff, o_kp, o_desc, o_match, o_pts, o_idx, o_hyp, stride;
};

size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

bool make_geom(int n_seq, int height, int width, int pitch, int ds, int max_kp, GmcGeom* g) {
    if (n_seq < 1 || height < 1 || width < 1 || ds < 1 || max_kp < 32 || max_kp > 65536) return false;
    g->n_seq = n_seq; g->src_h = height; g->src_w = width; g->pitch = pitch; g->ds = ds;
    g->h = height / ds; g->w = width / ds;
    if (g->h < 2 * kOrbEdge + 2 || g->w < 2 * kOrbEdge + 2 || g->h > 8192 || g->w > 8192) return false;
    g->wpr = (g->w + 31) / 32;
    g->max_kp = max_kp; g->slot = 0;
    g->my0 = (int)(0.02 * g->h); g->my1 = (int)(0.98 * g->h);
    g->mx0 = (int)(0.02 * g->w); g->mx1 = (int)(0.98 * g->w);
    const size_t px = (size_t)g->h * g->w;
    g->plane = align256(px);
    size_t o = 0;
    g->o_state = o; o += align256(kStateWords * sizeof(int));
    g->o_gray = o; o += align256(px);
    g->o_blur = o; o += 2 * align256(px);          // [2 plane sets]: a pipelined caller prepares frame t + 1 while frame t is being estimated
    g->o_score = o; o += 2 * align256(px);
    g->o_flags = o; o += align256((size_t)g->h * g->wpr * 4);
    g->o_rowoff = o; o += align256((size_t)(g->h + 1) * 4);
    g->o_kp = o; o += align256((size_t)2 * max_kp * 4);                  // [2][max_kp] x | y << 16
    g->o_desc = o; o += align256((size_t)2 * max_kp * 32);               // [2][max_kp][8] words
    g->o_match = o; o += align256((size_t)kSplit * max_kp * 16);         // [kSplit][max_kp] int4 (d1, i1, d2, i2)
    g->o_pts = o; o += align256((size_t)2 * max_kp * 16);                // [2][max_kp] float4 (src.x, src.y, dst.x, dst.y): after the ratio / after the sigma test
    g->o_idx = o; o += align256((size_t)2 * max_kp * 4);
    g->o_hyp = o; o += align256((size_t)kHypBlocks * 2 * 4);            // per RANSAC block: best inlier count, its hypothesis
    g->stride = o;
    return true;
}

template <class T> B2T_DEV T* wsp(unsigned char* ws, const GmcGeom& g, int seq, size_t off) {
    return reinterpret_cast<T*>(ws + (size_t)seq * g.stride + off);
}

// ---------------------------------------------------------------------------------------------- gray + 1/ds scale
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

__global__ void gray_kernel(const unsigned char* __restrict__ frames, unsigned char* ws, GmcGeom g, double scale_x, double scale_y) {
    const int seq = blockIdx.y;
    const unsigned char* img = frames + (size_t)seq * g.src_h * g.pitch;
    unsigned char* out = wsp<unsigned char>(ws, g, seq, g.o_gray);
    const int total = g.h * g.w;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int y = i / g.w, x = i - y * g.w;
        int v;
        if (g.ds == 1) {
            v = gray_of(img + (size_t)y * g.pitch + x * 3);
        } else if (g.ds == 2 && g.src_h == 2 * g.h && g.src_w == 2 * g.w) {           // INTER_LINEAR at exactly 1/2 == 2 x 2 INTER_AREA
            const unsigned char* q0 = img + (size_t)(2 * y) * g.pitch + (2 * x) * 3;
            const unsigned char* q1 = q0 + g.pitch;
            v = (gray_of(q0) + gray_of(q0 + 3) + gray_of(q1) + gray_of(q1 + 3) + 2) >> 2;
        } else {
            int sx, a0, a1, sy, b0, b1;
            lin_tap(x, scale_x, g.src_w, sx, a0, a1, true);
            lin_tap(y, scale_y, g.src_h, sy, b0, b1, false);
            const int sx1 = sx + 1 < g.src_w ? sx + 1 : g.src_w - 1;
            const int y0 = sy < 0 ? 0 : (sy > g.src_h - 1 ? g.src_h - 1 : sy);
            const int y1 = sy + 1 < 0 ? 0 : (sy + 1 > g.src_h - 1 ? g.src_h - 1 : sy + 1);
            const unsigned char* r0 = img + (size_t)y0 * g.pitch;
            const unsigned char* r1 = img + (size_t)y1 * g.pitch;
            const int h0 = gray_of(r0 + sx * 3) * a0 + gray_of(r0 + sx1 * 3) * a1;
            const int h1 = gray_of(r1 + sx * 3) * a0 + gray_of(r1 + sx1 * 3) * a1;
            v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
            v = v < 0 ? 0 : (v > 255 ? 255 : v);
        }
        out[i] = (unsigned char)v;
    }
}

// ---------------------------------------------------------------------------------------------- FAST-9/16 score
// score = max over the sixteen 9-arcs of min(v - p) and of min(p - v), minus 1 (OpenCV's cornerScore); 0 = not a corner.
__global__ void fast_score_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.y;
    const unsigned char* gray = wsp<unsigned char>(ws, g, seq, g.o_gray);
    unsigned char* score = wsp<unsigned char>(ws, g, seq, g.o_score + g.slot * g.plane);
    const int total = g.h * g.w;
    const int W = g.w;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int y = i / W, x = i - y * W;
        int sc = 0;
        if (y >= 3 && y < g.h - 3 && x >= 3 && x < W - 3) {
            const unsigned char* p = gray + i;
            const int v = p[0];
            int d[16];
            d[0] = v - p[3 * W]; d[1] = v - p[3 * W + 1]; d[2] = v - p[2 * W + 2]; d[3] = v - p[W + 3];
            d[4] = v - p[3]; d[5] = v - p[-W + 3]; d[6] = v - p[-2 * W + 2]; d[7] = v - p[-3 * W + 1];
            d[8] = v - p[-3 * W]; d[9] = v - p[-3 * W - 1]; d[10] = v - p[-2 * W - 2]; d[11] = v - p[-W - 3];
            d[12] = v - p[-3]; d[13] = v - p[W - 3]; d[14] = v - p[2 * W - 2]; d[15] = v - p[3 * W - 1];
            int nb = 0, nd = 0;
#pragma unroll
            for (int k = 0; k < 16; ++k) { nb += d[k] > kFastThreshold; nd += -d[k] > kFastThreshold; }
            if (nb >= 9 || nd >= 9) {
                // min over the arc k .. k+8 (cyclic) by doubling -- m2, m4, m8, then the ninth element -- once on d = v - p and
                // once on e = p - v.  (Deliberately NOT "-max(d)" for the dark arcs: nvcc 12.9 has been seen to fuse max(best, mn, -mx)
                // into a three-way VIMNMX3 and drop the negation, tools/gmc_debug.py.)
                int e[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) e[k] = -d[k];
                int a2[16], b2[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) { a2[k] = min(d[k], d[(k + 1) & 15]); b2[k] = min(e[k], e[(k + 1) & 15]); }
                int a4[16], b4[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) { a4[k] = min(a2[k], a2[(k + 2) & 15]); b4[k] = min(b2[k], b2[(k + 2) & 15]); }
                int best = -(1 << 20);
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    const int ma = min(min(a4[k], a4[(k + 4) & 15]), d[(k + 8) & 15]);       // brighter-centre arc: min of v - p
                    const int mb = min(min(b4[k], b4[(k + 4) & 15]), e[(k + 8) & 15]);       // darker-centre arc: min of p - v
                    best = max(best, ma);
                    best = max(best, mb);
                }
                if (best > kFastThreshold) sc = best - 1;
            }
        }
        score[i] = (unsigned char)sc;
    }
}

// ---------------------------------------------------------------------------------------------- ORB's smoothing
// 7 x 7 Gaussian, sigma 2, as OpenCV's float filter engine applies it to 8-bit data: symmetric taps paired before the multiply,
// rows then columns, float32, rounded half to even, BORDER_REFLECT_101.
B2T_DEV int refl(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

__global__ void blur_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.y;
    const unsigned char* gray = wsp<unsigned char>(ws, g, seq, g.o_gray);
    unsigned char* out = wsp<unsigned char>(ws, g, seq, g.o_blur + g.slot * g.plane);
    const float k0 = 0.07015932f, k1 = 0.13107488f, k2 = 0.19071282f, k3 = 0.21610594f;
    const int total = g.h * g.w;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int y = i / g.w, x = i - y * g.w;
        int xs[7];
#pragma unroll
        for (int j = 0; j < 7; ++j) xs[j] = refl(x + j - 3, g.w);
        float r[7];
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const unsigned char* row = gray + (size_t)refl(y + j - 3, g.h) * g.w;
            float hh = k3 * (float)(int)row[xs[3]];
            hh = hh + k2 * (float)((int)row[xs[4]] + (int)row[xs[2]]);
            hh = hh + k1 * (float)((int)row[xs[5]] + (int)row[xs[1]]);
            hh = hh + k0 * (float)((int)row[xs[6]] + (int)row[xs[0]]);
            r[j] = hh;
        }
        float v = k3 * r[3];
        v = v + k2 * (r[4] + r[2]);
        v = v + k1 * (r[5] + r[1]);
        v = v + k0 * (r[6] + r[0]);
        int q = __float2int_rn(v);
        out[i] = (unsigned char)(q < 0 ? 0 : (q > 255 ? 255 : q));
    }
}

// ---------------------------------------------------------------------------------------------- NMS + masks -> row-major key points
// A corner survives when its score is strictly greater than its eight neighbours' (FAST's non-maximum suppression), it lies in
// the central mask region and in no detection box (botsort.py:123-130), and ORB keeps it (>= 31 px from the border).
// One block per image row: flag words + the row's count.
__global__ void nms_flag_kernel(unsigned char* ws, GmcGeom g, const float* __restrict__ dets, const int* __restrict__ det_counts, int dmax,
                                float det_thresh) {
    const int seq = blockIdx.y, y = blockIdx.x;
    const unsigned char* score = wsp<unsigned char>(ws, g, seq, g.o_score + g.slot * g.plane);
    unsigned* flags = wsp<unsigned>(ws, g, seq, g.o_flags) + (size_t)y * g.wpr;
    int* rowoff = wsp<int>(ws, g, seq, g.o_rowoff);
    __shared__ int cnt, nbox;
    __shared__ int box_x0[kMaxBoxes], box_x1[kMaxBoxes];
    if (threadIdx.x == 0) { cnt = 0; nbox = 0; }
    __syncthreads();
    const int W = g.w;
    const int nd = dets ? (det_counts ? min(det_counts[seq], dmax) : dmax) : 0;
    const float* drow = dets ? dets + (size_t)seq * dmax * 6 : nullptr;
    const bool row_ok = y >= g.my0 && y < g.my1 && y >= kOrbEdge && y < g.h - kOrbEdge && y >= 3 && y < g.h - 3;
    // the x ranges of the boxes that cover this row: tlbr = (det[:4] / downscale).astype(int) -- float32 division, truncation;
    // negative corners clamp to 0 (the reference's NumPy slice would wrap around; detections are clipped to the image upstream)
    bool overflow = false;
    if (row_ok)
        for (int k = threadIdx.x; k < nd; k += (int)blockDim.x) {
            const float* d = drow + (size_t)k * 6;
            if (!(d[4] >= det_thresh)) continue;
            const int by0 = max((int)(d[1] / (float)g.ds), 0), by1 = max((int)(d[3] / (float)g.ds), 0);
            if (y < by0 || y >= by1) continue;
            const int slot = atomicAdd(&nbox, 1);
            if (slot < kMaxBoxes) { box_x0[slot] = max((int)(d[0] / (float)g.ds), 0); box_x1[slot] = max((int)(d[2] / (float)g.ds), 0); }
        }
    __syncthreads();
    const int nb = nbox;
    overflow = nb > kMaxBoxes;                            // more boxes on one row than the cache holds: test the detections directly
    for (int x0 = (int)(threadIdx.x & ~31u); x0 < g.wpr * 32; x0 += (int)blockDim.x) {
        const int x = x0 + (int)(threadIdx.x & 31u);
        bool keep = false;
        if (row_ok && x < W && x >= g.mx0 && x < g.mx1 && x >= kOrbEdge && x < W - kOrbEdge) {
            const unsigned char* p = score + (size_t)y * W + x;
            const int s = p[0];
            if (s > 0 && s > p[-1] && s > p[1] && s > p[-W - 1] && s > p[-W] && s > p[-W + 1] && s > p[W - 1] && s > p[W] && s > p[W + 1]) {
                keep = true;
                if (!overflow) {
                    for (int k = 0; k < nb && keep; ++k) keep = !(x >= box_x0[k] && x < box_x1[k]);
                } else {
                    for (int k = 0; k < nd && keep; ++k) {
                        const float* d = drow + (size_t)k * 6;
                        if (!(d[4] >= det_thresh)) continue;
                        const int bx0 = max((int)(d[0] / (float)g.ds), 0), by0 = max((int)(d[1] / (float)g.ds), 0);
                        const int bx1 = max((int)(d[2] / (float)g.ds), 0), by1 = max((int)(d[3] / (float)g.ds), 0);
                        if (x >= bx0 && x < bx1 && y >= by0 && y < by1) keep = false;
                    }
                }
            }
        }
        const unsigned bal = __ballot_sync(B2T_FULL, keep);
        if ((threadIdx.x & 31u) == 0) {
            flags[x0 >> 5] = bal;
            if (bal) atomicAdd(&cnt, __popc(bal));
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) rowoff[y] = cnt;
}

// exclusive scan of the row counts (one block per sequence); the frame counter selects the key-point buffer
__global__ void scan_rows_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.y;
    int* rowoff = wsp<int>(ws, g, seq, g.o_rowoff);
    int* state = wsp<int>(ws, g, seq, g.o_state);
    __shared__ int part[33];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int c0 = 0; c0 < g.h; c0 += (int)blockDim.x) {
        const int i = c0 + tid;
        const int v = i < g.h ? rowoff[i] : 0;
        int inc = v;
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(B2T_FULL, inc, (unsigned)d); if (lane >= d) inc += t; }
        if (lane == 31) part[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            const int w = lane < nw ? part[lane] : 0;
            int winc = w;
            for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(B2T_FULL, winc, (unsigned)d); if (lane >= d) winc += t; }
            part[lane] = winc - w;
            if (lane == 31) part[32] = winc;
        }
        __syncthreads();
        if (i < g.h) rowoff[i] = carry + part[wid] + inc - v;
        __syncthreads();
        if (tid == 0) carry += part[32];
        __syncthreads();
    }
    if (tid == 0) {
        rowoff[g.h] = carry;
        const int buf = state[0] & 1;
        state[1 + buf] = carry < g.max_kp ? carry : g.max_kp;
        state[3] = carry > g.max_kp ? 1 : 0;            // truncated (the reference has no cap: sticky flag in stat)
    }
}

// one warp per row writes its key points in x order at the row's offset
__global__ void compact_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.y;
    const int y = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (y >= g.h) return;
    const unsigned* flags = wsp<unsigned>(ws, g, seq, g.o_flags) + (size_t)y * g.wpr;
    const int* rowoff = wsp<int>(ws, g, seq, g.o_rowoff);
    const int* state = wsp<int>(ws, g, seq, g.o_state);
    unsigned* kp = wsp<unsigned>(ws, g, seq, g.o_kp) + (size_t)(state[0] & 1) * g.max_kp;
    int base = rowoff[y];
    if (rowoff[y + 1] == base) return;
    for (int w0 = 0; w0 < g.wpr; w0 += 32) {
        const unsigned word = (w0 + lane < g.wpr) ? flags[w0 + lane] : 0u;
        const int c = __popc(word);
        int inc = c;
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(B2T_FULL, inc, (unsigned)d); if (lane >= d) inc += t; }
        int o = base + inc - c;
        unsigned m = word;
        while (m) {
            const int b = __ffs((int)m) - 1;
            m &= m - 1;
            if (o < g.max_kp) kp[o] = (unsigned)((w0 + lane) * 32 + b) | ((unsigned)y << 16);
            ++o;
        }
        base += __shfl_sync(B2T_FULL, inc, 31);
    }
}

// ---------------------------------------------------------------------------------------------- descriptors: one warp per key point
__global__ void describe_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.y;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int* state = wsp<int>(ws, g, seq, g.o_state);
    const int buf = state[0] & 1;
    const int n = state[1 + buf];
    const unsigned* kp = wsp<unsigned>(ws, g, seq, g.o_kp) + (size_t)buf * g.max_kp;
    unsigned* desc = wsp<unsigned>(ws, g, seq, g.o_desc) + (size_t)buf * g.max_kp * 8;
    const unsigned char* img = wsp<unsigned char>(ws, g, seq, g.o_blur + g.slot * g.plane);
    const int wpb = blockDim.x >> 5;
    // the 27 x 27 patch (offsets -13 .. 13) is staged in shared memory row by row -- one coalesced 27-byte read per row instead of
    // sixteen scattered byte loads per lane (the kernel was LSU-bound: 512 sectors per key point) -- then the pairs read it there
    __shared__ unsigned char patch[8][27 * 32];
    int oa[8], ob[8];                                   // this lane's eight point pairs as patch offsets
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int i = lane * 8 + j;
        oa[j] = (kOrbPairs[i][0][0] + 13) * 32 + kOrbPairs[i][0][1] + 13;
        ob[j] = (kOrbPairs[i][1][0] + 13) * 32 + kOrbPairs[i][1][1] + 13;
    }
    unsigned char* pw = patch[wib];
    for (int k = blockIdx.x * wpb + wib; k < n; k += gridDim.x * wpb) {
        const unsigned xy = kp[k];
        const unsigned char* c = img + (size_t)((int)(xy >> 16) - 13) * g.w + ((int)(xy & 0xffffu) - 13);
        __syncwarp();
        if (lane < 27)
#pragma unroll 9
            for (int r = 0; r < 27; ++r) pw[r * 32 + lane] = c[(size_t)r * g.w + lane];
        __syncwarp();
        unsigned byte = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) byte |= (unsigned)((int)pw[oa[j]] < (int)pw[ob[j]]) << j;
        unsigned v = byte << (8 * (lane & 3));
        v |= __shfl_xor_sync(B2T_FULL, v, 1);
        v |= __shfl_xor_sync(B2T_FULL, v, 2);
        if ((lane & 3) == 0) desc[(size_t)k * 8 + (lane >> 2)] = v;
    }
}

// ---------------------------------------------------------------------------------------------- 2-NN Hamming matcher
// thread = query (previous frame's key point), the train descriptors (current frame) stream through shared memory in tiles;
// blockIdx.z = slice of the train set.  Strict '<' while walking in index order = BFMatcher's tie rule (lower index first).
__global__ void match_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.y, split = blockIdx.z;
    const int* state = wsp<int>(ws, g, seq, g.o_state);
    if (state[0] == 0) return;                                    // first frame: nothing to match against
    const int cur = state[0] & 1, prev = cur ^ 1;
    const int nq = state[1 + prev], nt = state[1 + cur];
    const unsigned* dq = wsp<unsigned>(ws, g, seq, g.o_desc) + (size_t)prev * g.max_kp * 8;
    const unsigned* dt = wsp<unsigned>(ws, g, seq, g.o_desc) + (size_t)cur * g.max_kp * 8;
    int* out = wsp<int>(ws, g, seq, g.o_match) + (size_t)split * g.max_kp * 4;
    const int per = (nt + kSplit - 1) / kSplit;
    const int t0 = split * per, t1 = min(nt, t0 + per);
    __shared__ uint4 tile4[128 * 2];                     // 128 train descriptors; read as two 16-byte broadcasts each (the kernel is
    unsigned* tile = reinterpret_cast<unsigned*>(tile4);   // POPC-bound -- 16 lanes / clk / SM -- once the loads are wide)
    for (int q0 = blockIdx.x * blockDim.x; q0 < nq; q0 += gridDim.x * blockDim.x) {
        const int q = q0 + (int)threadIdx.x;
        unsigned a[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = q < nq ? dq[(size_t)q * 8 + j] : 0u;
        int d1 = 1 << 20, i1 = -1, d2 = 1 << 20, i2 = -1;
        for (int tt = t0; tt < t1; tt += 128) {
            const int m = min(128, t1 - tt);
            __syncthreads();
            for (int e = threadIdx.x; e < m * 8; e += blockDim.x) tile[e] = dt[(size_t)tt * 8 + e];
            __syncthreads();
            for (int k = 0; k < m; ++k) {
                const uint4 t0 = tile4[2 * k], t1 = tile4[2 * k + 1];
                const int d = __popc(a[0] ^ t0.x) + __popc(a[1] ^ t0.y) + __popc(a[2] ^ t0.z) + __popc(a[3] ^ t0.w) +
                              __popc(a[4] ^ t1.x) + __popc(a[5] ^ t1.y) + __popc(a[6] ^ t1.z) + __popc(a[7] ^ t1.w);
                if (d < d1) { d2 = d1; i2 = i1; d1 = d; i1 = tt + k; }
                else if (d < d2) { d2 = d; i2 = tt + k; }
            }
        }
        if (q < nq) { int* o = out + (size_t)q * 4; o[0] = d1; o[1] = i1; o[2] = d2; o[3] = i2; }
    }
}

// ---------------------------------------------------------------------------------------------- filters + RANSAC + fit (one block per sequence)
B2T_DEV double block_sum(double v, double* red) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(B2T_FULL, v, d);
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    double t = 0.0;
    for (int i = 0; i < nw; ++i) t += red[i];
    return t;
}

// ordered compaction of the indices i in [0, n) with flag(i) into out[]; returns the count
template <class F> B2T_DEV int block_select(int n, F flag, int* out, int* scratch) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    int base = 0;
    for (int c0 = 0; c0 < n; c0 += (int)blockDim.x) {
        const int i = c0 + tid;
        const bool p = i < n && flag(i);
        const unsigned bal = __ballot_sync(B2T_FULL, p);
        __syncthreads();
        if (lane == 0) scratch[wid] = __popc(bal);
        __syncthreads();
        const int cnt = lane < nw ? scratch[lane] : 0;
        int inc = cnt;
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(B2T_FULL, inc, (unsigned)d); if (lane >= d) inc += t; }
        const int woff = __shfl_sync(B2T_FULL, inc - cnt, wid);
        const int tot = __shfl_sync(B2T_FULL, inc, 31);
        if (p) out[base + woff + __popc(bal & ((1u << lane) - 1u))] = i;
        base += tot;
    }
    __syncthreads();
    return base;
}

B2T_DEV void lcg_pair(unsigned t, unsigned n, int& i, int& j) {          // oracle/gmc.py: lcg_pair
    unsigned s = t * 2654435761u + 12345u;
    s = s * 1664525u + 1013904223u;
    i = (int)((s >> 8) % n);
    s = s * 1664525u + 1013904223u;
    j = (int)((s >> 8) % (n - 1u));
    if (j >= i) ++j;
}

// similarity (a, b, tx, ty) through the two correspondences of hypothesis t; false when the source points coincide
B2T_DEV bool pair_model(const float4* pts, int n, int t, double& ha, double& hb, double& htx, double& hty) {
    int i, j;
    lcg_pair((unsigned)t, (unsigned)n, i, j);
    const float4 p0 = pts[i], p1 = pts[j];
    const double dx = (double)p1.x - (double)p0.x, dy = (double)p1.y - (double)p0.y;
    const double den = dx * dx + dy * dy;
    if (den < 1e-12) return false;
    const double ux = (double)p1.z - (double)p0.z, uy = (double)p1.w - (double)p0.w;
    ha = (dx * ux + dy * uy) / den; hb = (dx * uy - dy * ux) / den;
    htx = (double)p0.z - (ha * (double)p0.x - hb * (double)p0.y);
    hty = (double)p0.w - (hb * (double)p0.x + ha * (double)p0.y);
    return true;
}
B2T_DEV bool is_inlier(const float4 p, double ha, double hb, double htx, double hty) {
    const double ex = ha * (double)p.x - hb * (double)p.y + htx - (double)p.z;
    const double ey = hb * (double)p.x + ha * (double)p.y + hty - (double)p.w;
    return ex * ex + ey * ey < 9.0;                       // reprojection error < 3 px (estimateAffinePartial2D's default)
}

// state words: [0] frames seen, [1], [2] key points of buffer 0 / 1, [3] truncated, [4] matches after ratio + spatial tests,
// [5] after the sigma test (the estimator's point set pts[max_kp ..]), [6] flags
// ---- E1: merge the matcher's slices, ratio + spatial tests, one-sided 2.5 sigma test (one block per sequence)
__global__ void __launch_bounds__(kEstThreads) filter_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.x;
    int* state = wsp<int>(ws, g, seq, g.o_state);
    const int frames_seen = state[0];
    const int cur = frames_seen & 1, prev = cur ^ 1;
    const int nq = frames_seen ? state[1 + prev] : 0, nt = state[1 + cur];
    const unsigned* kq = wsp<unsigned>(ws, g, seq, g.o_kp) + (size_t)prev * g.max_kp;
    const unsigned* kt = wsp<unsigned>(ws, g, seq, g.o_kp) + (size_t)cur * g.max_kp;
    const int* match = wsp<int>(ws, g, seq, g.o_match);
    float4* pts = wsp<float4>(ws, g, seq, g.o_pts);
    int* idx = wsp<int>(ws, g, seq, g.o_idx);               // [2][max_kp]: selected queries, then their best train index
    int* sel = idx + g.max_kp;
    const int tid = threadIdx.x;
    __shared__ double red[32];
    __shared__ int scratch[32];
    int n_ratio = 0, n_sigma = 0;
    if (frames_seen > 0 && nq > 0 && nt >= 2) {
        // lexicographic (distance, index) order over the slices = BFMatcher's sequential strict '<'
        const double max_dx = 0.25 * (double)g.w, max_dy = 0.25 * (double)g.h;
        for (int q = tid; q < nq; q += (int)blockDim.x) {
            int d1 = 1 << 20, i1 = -1, d2 = 1 << 20;
            for (int s = 0; s < kSplit; ++s) {
                const int* m = match + ((size_t)s * g.max_kp + q) * 4;
                for (int e = 0; e < 2; ++e) {
                    const int d = m[2 * e], i = m[2 * e + 1];
                    if (i < 0) continue;
                    if (d < d1) { d2 = d1; d1 = d; i1 = i; }          // slices come in index order: strict '<' keeps the lower index
                    else if (d < d2) d2 = d;
                }
            }
            bool ok = i1 >= 0 && (double)d1 < 0.9 * (double)d2;
            if (ok) {
                const unsigned pq = kq[q], pt = kt[i1];
                const double dx = (double)(int)(pq & 0xffffu) - (double)(int)(pt & 0xffffu);
                const double dy = (double)(int)(pq >> 16) - (double)(int)(pt >> 16);
                ok = fabs(dx) < max_dx && fabs(dy) < max_dy;
            }
            sel[q] = ok ? i1 : -1;
        }
        __syncthreads();
        n_ratio = block_select(nq, [&](int q) { return sel[q] >= 0; }, idx, scratch);
        if (n_ratio > 0) {                                   // botsort.py:187-190, population std like numpy
            double sx = 0.0, sy = 0.0;
            for (int k = tid; k < n_ratio; k += (int)blockDim.x) {
                const int q = idx[k];
                const unsigned pq = kq[q], pt = kt[sel[q]];
                const float4 p = make_float4((float)(pq & 0xffffu), (float)(pq >> 16), (float)(pt & 0xffffu), (float)(pt >> 16));
                pts[k] = p;
                sx += (double)p.x - (double)p.z; sy += (double)p.y - (double)p.w;
            }
            const double mx = block_sum(sx, red) / n_ratio;
            const double my = block_sum(sy, red) / n_ratio;
            double vx = 0.0, vy = 0.0;
            for (int k = tid; k < n_ratio; k += (int)blockDim.x) {
                const float4 p = pts[k];
                const double ex = ((double)p.x - (double)p.z) - mx, ey = ((double)p.y - (double)p.w) - my;
                vx += ex * ex; vy += ey * ey;
            }
            const double sdx = sqrt(block_sum(vx, red) / n_ratio), sdy = sqrt(block_sum(vy, red) / n_ratio);
            __syncthreads();
            n_sigma = block_select(n_ratio, [&](int k) {
                const float4 p = pts[k];
                return ((double)p.x - (double)p.z) - mx < 2.5 * sdx && ((double)p.y - (double)p.w) - my < 2.5 * sdy;
            }, sel, scratch);
            for (int k = tid; k < n_sigma; k += (int)blockDim.x) pts[g.max_kp + k] = pts[sel[k]];      // the estimator's point set, in order
        }
    }
    if (tid == 0) { state[4] = n_ratio; state[5] = n_sigma; }
}

// ---- E2: RANSAC over minimal samples of two correspondences; block b scores hypotheses [b * kHyp / kHypBlocks, ...)
__global__ void __launch_bounds__(256) ransac_kernel(unsigned char* ws, GmcGeom g) {
    const int seq = blockIdx.y;
    const int* state = wsp<int>(ws, g, seq, g.o_state);
    const int n = state[5];
    int* hyp = wsp<int>(ws, g, seq, g.o_hyp) + blockIdx.x * 2;
    const float4* pts = wsp<float4>(ws, g, seq, g.o_pts) + g.max_kp;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (int)blockDim.x >> 5;
    __shared__ int s_cnt[8], s_t[8];
    int wb_cnt = -1, wb_t = -1;
    if (n > 4) {
        const int per = kHyp / kHypBlocks, t0 = blockIdx.x * per;
        for (int t = t0 + wid; t < t0 + per; t += nw) {
            double ha, hb, htx, hty;
            if (!pair_model(pts, n, t, ha, hb, htx, hty)) continue;
            int c = 0;
            for (int k = lane; k < n; k += 32) c += is_inlier(pts[k], ha, hb, htx, hty) ? 1 : 0;
            for (int d = 16; d >= 1; d >>= 1) c += __shfl_xor_sync(B2T_FULL, c, d);
            if (c > wb_cnt) { wb_cnt = c; wb_t = t; }                  // ascending t within the warp: ties keep the lower t
        }
    }
    if (lane == 0) { s_cnt[wid] = wb_cnt; s_t[wid] = wb_t; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int bc = -1, bt = -1;
        for (int w = 0; w < nw; ++w)
            if (s_cnt[w] > bc || (s_cnt[w] == bc && s_t[w] >= 0 && s_t[w] < bt)) { bc = s_cnt[w]; bt = s_t[w]; }
        hyp[0] = bc; hyp[1] = bt;
    }
}

// ---- E3: best hypothesis (most inliers, then lowest index), least-squares similarity on its inliers, outputs
__global__ void __launch_bounds__(kEstThreads) fit_kernel(unsigned char* ws, GmcGeom g, double* __restrict__ warps, int* __restrict__ stat) {
    const int seq = blockIdx.x;
    int* state = wsp<int>(ws, g, seq, g.o_state);
    const int frames_seen = state[0];
    const int cur = frames_seen & 1, prev = cur ^ 1;
    const int nq = frames_seen ? state[1 + prev] : 0, nt = state[1 + cur];
    const int n_ratio = state[4], n_sigma = state[5];
    const int* hyp = wsp<int>(ws, g, seq, g.o_hyp);
    const float4* pts = wsp<float4>(ws, g, seq, g.o_pts) + g.max_kp;
    double* H = warps + (size_t)seq * 6;
    int* st = stat ? stat + (size_t)seq * B2T_GMC_STAT_WORDS : nullptr;
    const int tid = threadIdx.x;
    __shared__ double red[32];
    int best_cnt = -1, best_t = -1, flags = frames_seen == 0 ? B2T_GMC_FIRST_FRAME : 0;
    double a = 1.0, b = 0.0, tx = 0.0, ty = 0.0;
    if (n_sigma > 4) {
        for (int w = 0; w < kHypBlocks; ++w)                               // blocks hold ascending hypothesis ranges
            if (hyp[2 * w] > best_cnt) { best_cnt = hyp[2 * w]; best_t = hyp[2 * w + 1]; }
    }
    double ha = 1, hb = 0, htx = 0, hty = 0;
    if (best_cnt >= 2 && pair_model(pts, n_sigma, best_t, ha, hb, htx, hty)) {
        double sx = 0, sy = 0, su = 0, sv = 0;
        for (int k = tid; k < n_sigma; k += (int)blockDim.x) {
            const float4 p = pts[k];
            if (is_inlier(p, ha, hb, htx, hty)) { sx += p.x; sy += p.y; su += p.z; sv += p.w; }
        }
        const double msx = block_sum(sx, red) / best_cnt, msy = block_sum(sy, red) / best_cnt;
        const double mdx = block_sum(su, red) / best_cnt, mdy = block_sum(sv, red) / best_cnt;
        double num_a = 0, num_b = 0, den = 0;
        for (int k = tid; k < n_sigma; k += (int)blockDim.x) {
            const float4 p = pts[k];
            if (is_inlier(p, ha, hb, htx, hty)) {
                const double x = (double)p.x - msx, y = (double)p.y - msy, u = (double)p.z - mdx, v = (double)p.w - mdy;
                num_a += x * u + y * v; num_b += x * v - y * u; den += x * x + y * y;
            }
        }
        num_a = block_sum(num_a, red); num_b = block_sum(num_b, red); den = block_sum(den, red);
        a = num_a / den; b = num_b / den;
        tx = (mdx - (a * msx - b * msy)) * (double)g.ds;                   // botsort.py:224-226: translation back to full resolution
        ty = (mdy - (b * msx + a * msy)) * (double)g.ds;
    } else if (frames_seen > 0) flags |= B2T_GMC_FEW_POINTS;               // botsort.py:228 "not enough matching points"
    __syncthreads();
    if (tid == 0) {
        H[0] = a; H[1] = -b; H[2] = tx; H[3] = b; H[4] = a; H[5] = ty;
        if (state[3]) flags |= B2T_GMC_TRUNCATED;
        if (st) {
            st[0] = nt; st[1] = nq; st[2] = n_ratio; st[3] = n_sigma; st[4] = best_cnt > 0 ? best_cnt : 0; st[5] = flags; st[6] = best_t; st[7] = frames_seen;
        }
        state[0] = frames_seen + 1;                                         // the current buffers become the previous ones
    }
}

int gfail(int code, const char* m) { b2t::set_detect_error(m); return code; }
int gcheck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { b2t::set_detect_error((std::string(what) + ": " + cudaGetErrorString(e)).c_str()); return B2T_ECUDA; }
    return B2T_OK;
}

}  // namespace

extern "C" size_t b2t_gmc_workspace_bytes(int n_seq, int height, int width, int downscale, int max_kp) {
    GmcGeom g;
    if (!make_geom(n_seq, height, width, width * 3, downscale, max_kp, &g)) return 0;
    return g.stride * (size_t)n_seq;
}

extern "C" int b2t_gmc_workspace_layout(int n_seq, int height, int width, int downscale, int max_kp, size_t* out, int n) {
    GmcGeom g;
    if (!out || !make_geom(n_seq, height, width, width * 3, downscale, max_kp, &g)) return gfail(B2T_EINVAL, "b2t_gmc_workspace_layout: bad arguments");
    const size_t v[10] = {g.stride, g.o_state, g.o_gray, g.o_blur, g.o_score, g.o_kp, g.o_desc, (size_t)g.h, (size_t)g.w, g.o_pts};
    for (int i = 0; i < n && i < 10; ++i) out[i] = v[i];
    return B2T_OK;
}

extern "C" int b2t_gmc_reset(void* workspace, int n_seq, int height, int width, int downscale, int max_kp, void* stream) {
    GmcGeom g;
    if (!workspace || !make_geom(n_seq, height, width, width * 3, downscale, max_kp, &g)) return gfail(B2T_EINVAL, "b2t_gmc_reset: bad arguments");
    for (int s = 0; s < n_seq; ++s)
        if (cudaMemsetAsync((unsigned char*)workspace + (size_t)s * g.stride + g.o_state, 0, kStateWords * sizeof(int), (cudaStream_t)stream) != 0)
            return gfail(B2T_ECUDA, "b2t_gmc_reset: memset failed");
    return B2T_OK;
}

namespace {
int prepare(const unsigned char* frames_bgr, const GmcGeom& g, unsigned char* ws, cudaStream_t s) {
    const int px = g.h * g.w;
    const int gx = (px + 255) / 256 < 132 * 8 ? (px + 255) / 256 : 132 * 8;
    // cv::resize derives the scales from inv_scale = dsize / ssize in double: scale = 1. / inv_scale
    const double scale_x = 1.0 / ((double)g.w / (double)g.src_w), scale_y = 1.0 / ((double)g.h / (double)g.src_h);
    B2T_LAUNCH(gray_kernel, dim3(gx, g.n_seq), 256, 0, s, frames_bgr, ws, g, scale_x, scale_y);
    B2T_LAUNCH(fast_score_kernel, dim3(gx, g.n_seq), 256, 0, s, ws, g);
    B2T_LAUNCH(blur_kernel, dim3(gx, g.n_seq), 256, 0, s, ws, g);
    return gcheck("gmc_prepare");
}
int estimate(const GmcGeom& g, unsigned char* ws, const float* dets, const int* det_counts, int dmax, float det_thresh, double* warps_out, int* stat,
             cudaStream_t s) {
    B2T_LAUNCH(nms_flag_kernel, dim3(g.h, g.n_seq), 128, 0, s, ws, g, dets, det_counts, dmax, det_thresh);
    B2T_LAUNCH(scan_rows_kernel, dim3(1, g.n_seq), 1024, 0, s, ws, g);
    B2T_LAUNCH(compact_kernel, dim3((g.h + 3) / 4, g.n_seq), 128, 0, s, ws, g);
    const int kpb = (g.max_kp + 7) / 8 < 132 * 4 ? (g.max_kp + 7) / 8 : 132 * 4;
    B2T_LAUNCH(describe_kernel, dim3(kpb, g.n_seq), 256, 0, s, ws, g);
    B2T_LAUNCH(match_kernel, dim3((g.max_kp + 127) / 128, g.n_seq, kSplit), 128, 0, s, ws, g);
    B2T_LAUNCH(filter_kernel, dim3(g.n_seq), kEstThreads, 0, s, ws, g);
    B2T_LAUNCH(ransac_kernel, dim3(kHypBlocks, g.n_seq), 256, 0, s, ws, g);
    B2T_LAUNCH(fit_kernel, dim3(g.n_seq), kEstThreads, 0, s, ws, g, warps_out, stat);
    return gcheck("gmc_estimate");
}
}  // namespace

extern "C" int b2t_gmc_prepare(const unsigned char* frames_bgr, int n_seq, int height, int width, int pitch, int downscale, void* workspace, int max_kp,
                               int slot, void* stream) {
    GmcGeom g;
    if (!frames_bgr || !workspace || pitch < 3 * width || slot < 0 || slot > 1 || !make_geom(n_seq, height, width, pitch, downscale, max_kp, &g))
        return gfail(B2T_EINVAL, "b2t_gmc_prepare: bad arguments (frame at least 64 px per side after down-scaling, 32 <= max_kp <= 65536, slot 0 / 1)");
    g.slot = slot;
    return prepare(frames_bgr, g, (unsigned char*)workspace, (cudaStream_t)stream);
}

extern "C" int b2t_gmc_estimate_prepared(int n_seq, int height, int width, int downscale, const float* dets, const int* det_counts, int dmax,
                                         float det_thresh, void* workspace, int max_kp, int slot, double* warps_out, int* stat, void* stream) {
    GmcGeom g;
    if (!workspace || !warps_out || (dets && dmax < 1) || slot < 0 || slot > 1 || !make_geom(n_seq, height, width, 3 * width, downscale, max_kp, &g))
        return gfail(B2T_EINVAL, "b2t_gmc_estimate_prepared: bad arguments");
    g.slot = slot;
    return estimate(g, (unsigned char*)workspace, dets, det_counts, dmax, det_thresh, warps_out, stat, (cudaStream_t)stream);
}

extern "C" int b2t_gmc_estimate(const unsigned char* frames_bgr, int n_seq, int height, int width, int pitch, int downscale, const float* dets,
                                const int* det_counts, int dmax, float det_thresh, void* workspace, int max_kp, double* warps_out, int* stat,
                                void* stream) {
    GmcGeom g;
    if (!frames_bgr || !workspace || !warps_out || pitch < 3 * width || (dets && dmax < 1) || !make_geom(n_seq, height, width, pitch, downscale, max_kp, &g))
        return gfail(B2T_EINVAL, "b2t_gmc_estimate: bad arguments (frame at least 64 px per side after down-scaling, 32 <= max_kp <= 65536)");
    const int rc = prepare(frames_bgr, g, (unsigned char*)workspace, (cudaStream_t)stream);
    return rc != B2T_OK ? rc : estimate(g, (unsigned char*)workspace, dets, det_counts, dmax, det_thresh, warps_out, stat, (cudaStream_t)stream);
}
