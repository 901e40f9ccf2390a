// b2t_nms.cu -- non_max_suppression (utils/general.py:607-695) on the device, and its fusion with the Detect decode.
//
// The reference filters rows by objectness, multiplies the class scores, takes the best class, sorts by confidence,
// keeps max_nms rows, runs torchvision.ops.nms on class-offset boxes and truncates to max_det.  Here:
//
//   filter_pred_kernel / filter_raw_kernel   one thread per anchor row.  `filter_raw` reads the four raw head maps
//                        directly (Detect.forward's sigmoid / grid / anchor decode, models/yolo.py:44-55, is applied
//                        to the ~5 % of rows that pass the objectness test only), so the 278 MB `pred` tensor is never
//                        written or re-read on the detect() path.  Survivors are appended with an atomic cursor and
//                        counted into a 2048-bin histogram of their confidence bits.
//   bucket_scan_kernel   exclusive scan of the histogram, high confidence first      } a counting sort whose result
//   bucket_scatter_kernel  candidates grouped by bin (order inside a bin arbitrary)   } does not depend on the order
//   bucket_rank_kernel   exact rank inside the bin by (conf desc, row index asc)      } the atomics happened to run in
//   nms_greedy_kernel    one CTA per image walks the sorted list 64 candidates at a time: (a) the block against the
//                        boxes kept so far, (b) the block against itself (64 x 64 bits), (c) a one-thread bit scan
//                        that applies the greedy rule, until max_det rows are kept.  This evaluates ~max_det x (rows
//                        visited) IoUs instead of the full n x n suppression matrix (n ~ 5 000 rows per image at
//                        conf_thres = 0.01: 40x less work, and no 900 MB mask workspace), with the identical result:
//                        row i is kept iff no kept row of higher rank has IoU > thr with it.
//                        Output rows are [x1 y1 x2 y2 conf cls], after scale_coords / clip / round
//                        (utils/general.py:319-340, tracker/track.py:240) when post != 0.
//
// HBM-bound integer / compare work; written against b2t_platform.cuh so that tests/hostsim can run the same source
// on the CPU simulator (test infrastructure, see tests/hostsim/cuda_sim.h).
#include <string>          // before b2t_platform.cuh: the simulator's __noinline__ macro must not reach libstdc++
#include <string.h>
#include "b2t_platform.cuh"
#include "b2t_decode.cuh"
#include "../../include/b200track.h"

namespace b2t { void set_detect_error(const char* m); }

#if defined(B2T_HOSTSIM)
namespace { thread_local std::string g_sim_det_err; }
namespace b2t { void set_detect_error(const char* m) { g_sim_det_err = m; } }
extern "C" const char* b2t_detect_last_error(void) { return g_sim_det_err.c_str(); }
#endif

namespace {

constexpr int kBins = 2048;
constexpr int kGreedyThreads = 1024;

int nfail(int code, const char* m) { b2t::set_detect_error(m); return code; }
int ncheck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { b2t::set_detect_error((std::string(what) + ": " + cudaGetErrorString(e)).c_str()); return B2T_ECUDA; }
    return B2T_OK;
}

// candidate: corner box, best-class confidence, class, original row index, histogram bin (32 bytes)
struct Cand { float x1, y1, x2, y2, conf, cls; int idx; int bin; };
struct BKey { float conf; int idx; int slot; int bin; };

struct Binning { unsigned kmin; int shift; };

B2T_DEV int conf_bin(float conf, Binning bn) {
    const unsigned key = (unsigned)__float_as_int(conf);          // conf > conf_thres >= 0: the bit pattern is monotone
    const unsigned d = key > bn.kmin ? key - bn.kmin : 0u;
    const unsigned b = d >> bn.shift;
    return (kBins - 1) - (int)(b < (unsigned)kBins ? b : (unsigned)(kBins - 1));      // bin 0 = highest confidence
}

B2T_DEV void emit_candidate(float cx, float cy, float w, float h, float best, int cls, int row, int b, int maxc, Binning bn,
                            Cand* __restrict__ cand, int* __restrict__ count, int* __restrict__ hist) {
    const int slot = atomicAdd(&count[b], 1);
    if (slot >= maxc) return;
    Cand cd;
    cd.x1 = cx - w / 2; cd.y1 = cy - h / 2; cd.x2 = cx + w / 2; cd.y2 = cy + h / 2;                 // xywh2xyxy (:265-272)
    cd.conf = best; cd.cls = (float)cls; cd.idx = row; cd.bin = conf_bin(best, bn);
    cand[(long long)b * maxc + slot] = cd;
    atomicAdd(&hist[b * kBins + cd.bin], 1);
}

// ---- candidates from a materialised prediction tensor [B][N][no]
__global__ void filter_pred_kernel(const float* __restrict__ pred, int N, int no, float conf_thres, Binning bn, Cand* __restrict__ cand,
                                   int* __restrict__ count, int* __restrict__ hist, int maxc) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float* r = pred + ((long long)b * N + i) * no;
    const float obj = r[4];
    if (!(obj > conf_thres)) return;                                 // xc = prediction[..., 4] > conf_thres (:616)
    float best = -1.f; int bj = 0;
    for (int c = 5; c < no; ++c) { const float v = r[c] * obj; if (v > best) { best = v; bj = c - 5; } }   // (:648, :658)
    if (!(best > conf_thres)) return;
    emit_candidate(r[0], r[1], r[2], r[3], best, bj, i, b, maxc, bn, cand, count, hist);
}

// ---- candidates straight from the raw head maps: Detect decode fused with the filter
struct HeadLevels {
    const float* raw[4];
    int pitch[4], h[4], w[4];
    float stride[4];
    float anchors[4][6];
    long long level_off[4];      // first prediction row of the level
    long long first[4];          // first flat (pixel, anchor) index of the level inside one image
    int n_levels;
    long long per_image;         // sum of h*w*3
};

__global__ void filter_raw_kernel(HeadLevels L, int B, int no, float conf_thres, Binning bn, Cand* __restrict__ cand, int* __restrict__ count,
                                  int* __restrict__ hist, int maxc) {
    const long long total = (long long)B * L.per_image;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / L.per_image);
        long long t = i - (long long)b * L.per_image;
        int lv = 0;
        for (int k = 1; k < L.n_levels; ++k) if (t >= L.first[k]) lv = k;
        t -= L.first[lv];
        const int H = L.h[lv], W = L.w[lv];
        const int a = (int)(t % 3); t /= 3;
        const int x = (int)(t % W);
        const int y = (int)(t / W);
        const float* r = L.raw[lv] + (((long long)b * H + y) * W + x) * L.pitch[lv] + a * no;
        const float obj = b2t::det_sigmoid(r[4]);
        if (!(obj > conf_thres)) continue;
        float best = -1.f; int bj = 0;
        for (int c = 5; c < no; ++c) { const float v = b2t::det_sigmoid(r[c]) * obj; if (v > best) { best = v; bj = c - 5; } }
        if (!(best > conf_thres)) continue;
        const float cx = b2t::det_xy(b2t::det_sigmoid(r[0]), (float)x, L.stride[lv]);
        const float cy = b2t::det_xy(b2t::det_sigmoid(r[1]), (float)y, L.stride[lv]);
        const float bw = b2t::det_wh(b2t::det_sigmoid(r[2]), L.anchors[lv][2 * a]);
        const float bh = b2t::det_wh(b2t::det_sigmoid(r[3]), L.anchors[lv][2 * a + 1]);
        const int row = (int)(L.level_off[lv] + ((long long)a * H + y) * W + x);
        emit_candidate(cx, cy, bw, bh, best, bj, row, b, maxc, bn, cand, count, hist);
    }
}

// ---- exclusive scan of the 2048 bins of one image (1024 threads, 2 bins each); also clears the scatter cursors
__global__ void bucket_scan_kernel(const int* __restrict__ hist, int* __restrict__ base, int* __restrict__ cursor) {
    __shared__ int warp_tot[32];
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int h0 = hist[b * kBins + 2 * t], h1 = hist[b * kBins + 2 * t + 1];
    int v = h0 + h1;
    for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(B2T_FULL, v, d); if (lane >= d) v += u; }
    if (lane == 31) warp_tot[w] = v;
    __syncthreads();
    if (w == 0) {
        int s = warp_tot[lane];
        for (int d = 1; d < 32; d <<= 1) { const int u = __shfl_up_sync(B2T_FULL, s, d); if (lane >= d) s += u; }
        warp_tot[lane] = s;
    }
    __syncthreads();
    const int excl = v - (h0 + h1) + (w ? warp_tot[w - 1] : 0);
    base[b * kBins + 2 * t] = excl;
    base[b * kBins + 2 * t + 1] = excl + h0;
    cursor[b * kBins + 2 * t] = 0;
    cursor[b * kBins + 2 * t + 1] = 0;
}

__global__ void bucket_scatter_kernel(const Cand* __restrict__ cand, const int* __restrict__ count, int maxc, const int* __restrict__ base,
                                      int* __restrict__ cursor, BKey* __restrict__ keys) {
    const int b = blockIdx.y;
    const int n = min(count[b], maxc);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Cand* c = cand + (long long)b * maxc + i;
    BKey k; k.conf = c->conf; k.idx = c->idx; k.slot = i; k.bin = c->bin;
    const int pos = base[b * kBins + k.bin] + atomicAdd(&cursor[b * kBins + k.bin], 1);
    keys[(long long)b * maxc + pos] = k;
}

// rank = rows of higher confidence (earlier bins) + rows of the same bin that sort before this one.  The max_nms best are
// written in order (utils/general.py:673-674) together with their class-offset boxes (:677-678).
__global__ void bucket_rank_kernel(const Cand* __restrict__ cand, const BKey* __restrict__ keys, const int* __restrict__ count, int maxc,
                                   const int* __restrict__ base, const int* __restrict__ hist, int max_nms, float max_wh,
                                   float4* __restrict__ sbox, Cand* __restrict__ sorted) {
    const int b = blockIdx.y;
    const int n = min(count[b], maxc);
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const BKey* kb = keys + (long long)b * maxc;
    const BKey me = kb[p];
    const int lo = base[b * kBins + me.bin], hi = lo + hist[b * kBins + me.bin];
    int r = lo;
    for (int q = lo; q < hi; ++q) {
        const float c = kb[q].conf; const int id = kb[q].idx;
        r += (c > me.conf || (c == me.conf && id < me.idx)) ? 1 : 0;
    }
    if (r >= max_nms) return;
    const Cand cd = cand[(long long)b * maxc + me.slot];
    const float off = cd.cls * max_wh;
    sbox[(long long)b * max_nms + r] = make_float4(cd.x1 + off, cd.y1 + off, cd.x2 + off, cd.y2 + off);
    sorted[(long long)b * max_nms + r] = cd;
}

B2T_DEV bool iou_gt(const float4 a, const float4 b, float thr) {     // torchvision nms_kernel devIoU
    const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
    const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
    const float w = fmaxf(right - left, 0.f), h = fmaxf(bottom - top, 0.f);
    const float inter = w * h;
    const float sa = (a.z - a.x) * (a.w - a.y), sb = (b.z - b.x) * (b.w - b.y);
    return inter / (sa + sb - inter) > thr;
}

__global__ void __launch_bounds__(kGreedyThreads)
nms_greedy_kernel(const Cand* __restrict__ sorted, const float4* __restrict__ sbox, const int* __restrict__ count, int maxc, int max_nms,
                  int max_det, float thr, float* __restrict__ out, int* __restrict__ out_count, int post, float gain, float padw, float padh,
                  float img_w, float img_h) {
    B2T_DYN_SMEM(dyn);
    float4* kept = reinterpret_cast<float4*>(dyn);                   // class-offset boxes of the rows kept so far [max_det]
    __shared__ float4 blk[64];
    __shared__ int supp[64];
    __shared__ unsigned diag_lo[64], diag_hi[64];
    __shared__ int kept_rows[64];
    __shared__ int s_nk, s_keep;
    const int b = blockIdx.x, t = threadIdx.x;
    const int n = min(min(count[b], maxc), max_nms);
    const float4* sb = sbox + (long long)b * max_nms;
    const Cand* sc = sorted + (long long)b * max_nms;
    if (t == 0) s_keep = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += 64) {
        const int k0 = s_keep;
        if (k0 >= max_det) break;
        const int lim = min(64, n - i0);
        if (t < 64) { blk[t] = t < lim ? sb[i0 + t] : make_float4(0.f, 0.f, 0.f, 0.f); supp[t] = 0; }
        __syncthreads();
        // (a) block rows against the rows already kept
        for (int p = t; p < 64 * k0; p += kGreedyThreads) {
            const int q = p & 63, j = p >> 6;
            if (q < lim && iou_gt(kept[j], blk[q], thr)) supp[q] = 1;
        }
        // (b) block against itself: thread (q, sub) tests columns 4*sub .. 4*sub+3 of row q; bit r of diag[q] = "q suppresses r"
        {
            const int q = t >> 4, sub = t & 15;
            unsigned lo = 0, hi = 0;
            if (q < lim) {
                const float4 me = blk[q];
                for (int u = 0; u < 4; ++u) {
                    const int r = sub * 4 + u;
                    if (r > q && r < lim && iou_gt(me, blk[r], thr)) { if (r < 32) lo |= 1u << r; else hi |= 1u << (r - 32); }
                }
            }
            for (int d = 1; d < 16; d <<= 1) { lo |= __shfl_xor_sync(B2T_FULL, lo, d, 16); hi |= __shfl_xor_sync(B2T_FULL, hi, d, 16); }
            if (sub == 0) { diag_lo[q] = lo; diag_hi[q] = hi; }
        }
        __syncthreads();
        // (c) greedy rule inside the block, in rank order
        if (t == 0) {
            unsigned long long cur = 0;
            for (int q = 0; q < lim; ++q) if (supp[q]) cur |= 1ull << q;
            int nk = 0, k = k0;
            for (int q = 0; q < lim && k < max_det; ++q) {
                if ((cur >> q) & 1ull) continue;
                kept_rows[nk++] = q;
                cur |= ((unsigned long long)diag_hi[q] << 32) | (unsigned long long)diag_lo[q];
                ++k;
            }
            s_nk = nk;
        }
        __syncthreads();
        const int nk = s_nk;
        for (int q = t; q < nk; q += kGreedyThreads) {
            const int rq = kept_rows[q];
            kept[k0 + q] = blk[rq];
            const Cand cd = sc[i0 + rq];
            float x1 = cd.x1, y1 = cd.y1, x2 = cd.x2, y2 = cd.y2;
            if (post) {
                x1 = (x1 - padw) / gain; x2 = (x2 - padw) / gain; y1 = (y1 - padh) / gain; y2 = (y2 - padh) / gain;   // scale_coords
                x1 = fminf(fmaxf(x1, 0.f), img_w); x2 = fminf(fmaxf(x2, 0.f), img_w);                                  // clip_coords
                y1 = fminf(fmaxf(y1, 0.f), img_h); y2 = fminf(fmaxf(y2, 0.f), img_h);
                x1 = rintf(x1); y1 = rintf(y1); x2 = rintf(x2); y2 = rintf(y2);                                       // .round()
            }
            float* o = out + ((long long)b * max_det + k0 + q) * 6;
            o[0] = x1; o[1] = y1; o[2] = x2; o[3] = y2; o[4] = cd.conf; o[5] = cd.cls;
        }
        __syncthreads();
        if (t == 0) s_keep = k0 + nk;
        __syncthreads();
    }
    if (t == 0) out_count[b] = s_keep < max_det ? s_keep : max_det;
}

struct Workspace {
    int *count, *hist, *base, *cursor;
    Cand *cand, *sorted;
    BKey* keys;
    float4* sbox;
    size_t zero_bytes;
};

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

size_t carve(void* workspace, int B, int max_cand, int max_nms, Workspace* ws) {
    unsigned char* p0 = (unsigned char*)(((size_t)workspace + 255) / 256 * 256);
    unsigned char* p = p0;
    // count | hist | cursor are cleared together at the start of every call
    int* count = (int*)p;           p += align256((size_t)B * 4);
    int* hist = (int*)p;            p += align256((size_t)B * kBins * 4);
    const size_t zero_bytes = (size_t)(p - p0);
    int* cursor = (int*)p;          p += align256((size_t)B * kBins * 4);
    int* base = (int*)p;            p += align256((size_t)B * kBins * 4);
    Cand* cand = (Cand*)p;          p += align256((size_t)B * max_cand * sizeof(Cand));
    BKey* keys = (BKey*)p;          p += align256((size_t)B * max_cand * sizeof(BKey));
    Cand* sorted = (Cand*)p;        p += align256((size_t)B * max_nms * sizeof(Cand));
    float4* sbox = (float4*)p;      p += align256((size_t)B * max_nms * sizeof(float4));
    if (ws) { ws->count = count; ws->hist = hist; ws->base = base; ws->cursor = cursor; ws->cand = cand; ws->keys = keys; ws->sorted = sorted;
              ws->sbox = sbox; ws->zero_bytes = zero_bytes; }
    return (size_t)(p - p0) + 256;
}

Binning make_binning(float conf_thres) {
    Binning bn;
    float lo = conf_thres > 0.f ? conf_thres : 0.f;
    unsigned kmin; memcpy(&kmin, &lo, 4);
    const float one = 1.0f; unsigned kmax; memcpy(&kmax, &one, 4);
    bn.kmin = kmin; bn.shift = 0;
    if (kmax > kmin) while (((kmax - kmin) >> bn.shift) >= (unsigned)kBins) ++bn.shift;
    return bn;
}

int sort_and_select(const Workspace& ws, int B, float iou_thres, int max_det, int max_nms, int max_cand, int post, float gain, float padw,
                    float padh, float img_w, float img_h, float* out, int* out_count, cudaStream_t s) {
    B2T_LAUNCH(bucket_scan_kernel, B, kBins / 2, 0, s, ws.hist, ws.base, ws.cursor);
    B2T_LAUNCH(bucket_scatter_kernel, dim3((max_cand + 255) / 256, B), 256, 0, s, ws.cand, ws.count, max_cand, ws.base, ws.cursor, ws.keys);
    B2T_LAUNCH(bucket_rank_kernel, dim3((max_cand + 255) / 256, B), 256, 0, s, ws.cand, ws.keys, ws.count, max_cand, ws.base, ws.hist, max_nms,
               4096.f, ws.sbox, ws.sorted);
    B2T_LAUNCH(nms_greedy_kernel, B, kGreedyThreads, (size_t)max_det * sizeof(float4), s, ws.sorted, ws.sbox, ws.count, max_cand, max_nms, max_det,
               iou_thres, out, out_count, post, gain, padw, padh, img_w, img_h);
    return ncheck("nms");
}

}  // namespace

extern "C" size_t b2t_nms_workspace_bytes(int B, int max_cand, int max_nms) {
    if (B < 1 || max_cand < 1 || max_nms < 1) return 0;
    if (max_nms > max_cand) max_nms = max_cand;
    return carve(nullptr, B, max_cand, max_nms, nullptr);
}

extern "C" int b2t_nms(const float* pred, int B, int N, int no, float conf_thres, float iou_thres, int max_det, int max_nms, int max_cand,
                       int post, float gain, float padw, float padh, float img_w, float img_h, void* workspace, size_t workspace_bytes,
                       float* out, int* out_count, void* stream) {
    if (!pred || !workspace || !out || !out_count || B < 1 || N < 1 || no < 6 || max_det < 1 || max_nms < 1 || max_cand < 1)
        return nfail(B2T_EINVAL, "b2t_nms: bad arguments");
    if (max_det > 2048 || !(conf_thres >= 0.f)) return nfail(B2T_EINVAL, "b2t_nms: need max_det <= 2048 and conf_thres >= 0");
    if (max_nms > max_cand) max_nms = max_cand;
    if (workspace_bytes < b2t_nms_workspace_bytes(B, max_cand, max_nms)) return nfail(B2T_EINVAL, "b2t_nms: workspace too small");
    cudaStream_t s = (cudaStream_t)stream;
    Workspace ws;
    carve(workspace, B, max_cand, max_nms, &ws);
    const Binning bn = make_binning(conf_thres);
    cudaMemsetAsync(ws.count, 0, ws.zero_bytes, s);
    B2T_LAUNCH(filter_pred_kernel, dim3((N + 255) / 256, B), 256, 0, s, pred, N, no, conf_thres, bn, ws.cand, ws.count, ws.hist, max_cand);
    return sort_and_select(ws, B, iou_thres, max_det, max_nms, max_cand, post, gain, padw, padh, img_w, img_h, out, out_count, s);
}

extern "C" int b2t_detect_nms(const b2t_head_level* levels, int n_levels, int B, int no, float conf_thres, float iou_thres, int max_det,
                              int max_nms, int max_cand, int post, float gain, float padw, float padh, float img_w, float img_h,
                              void* workspace, size_t workspace_bytes, float* out, int* out_count, void* stream) {
    if (!levels || n_levels < 1 || n_levels > 4 || !workspace || !out || !out_count || B < 1 || no < 6 || max_det < 1 || max_nms < 1 || max_cand < 1)
        return nfail(B2T_EINVAL, "b2t_detect_nms: bad arguments");
    if (max_det > 2048 || !(conf_thres >= 0.f)) return nfail(B2T_EINVAL, "b2t_detect_nms: need max_det <= 2048 and conf_thres >= 0");
    if (max_nms > max_cand) max_nms = max_cand;
    if (workspace_bytes < b2t_nms_workspace_bytes(B, max_cand, max_nms)) return nfail(B2T_EINVAL, "b2t_detect_nms: workspace too small");
    HeadLevels L;
    memset(&L, 0, sizeof(L));
    L.n_levels = n_levels;
    long long first = 0;
    for (int k = 0; k < n_levels; ++k) {
        const b2t_head_level& lv = levels[k];
        if (!lv.raw || lv.h < 1 || lv.w < 1 || lv.raw_pitch < 3 * no) return nfail(B2T_EINVAL, "b2t_detect_nms: bad level");
        L.raw[k] = lv.raw; L.pitch[k] = lv.raw_pitch; L.h[k] = lv.h; L.w[k] = lv.w; L.stride[k] = lv.stride;
        for (int j = 0; j < 6; ++j) L.anchors[k][j] = lv.anchors[j];
        L.level_off[k] = lv.level_off; L.first[k] = first;
        first += (long long)lv.h * lv.w * 3;
    }
    L.per_image = first;
    cudaStream_t s = (cudaStream_t)stream;
    Workspace ws;
    carve(workspace, B, max_cand, max_nms, &ws);
    const Binning bn = make_binning(conf_thres);
    cudaMemsetAsync(ws.count, 0, ws.zero_bytes, s);
    const long long total = (long long)B * L.per_image;
    long long g = (total + 255) / 256;
    if (g > 132 * 16) g = 132 * 16;
    B2T_LAUNCH(filter_raw_kernel, (int)g, 256, 0, s, L, B, no, conf_thres, bn, ws.cand, ws.count, ws.hist, max_cand);
    return sort_and_select(ws, B, iou_thres, max_det, max_nms, max_cand, post, gain, padw, padh, img_w, img_h, out, out_count, s);
}
