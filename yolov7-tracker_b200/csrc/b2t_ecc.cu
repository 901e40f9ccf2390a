// b2t_ecc.cu -- ECC camera-motion estimation on the GPU: GMC(method='ecc') of tracker/botsort.py:78-109, which StrongSORT builds
// (tracker/strongsort.py:32) and which costs the reference 0.1 - 0.35 s of host OpenCV per frame.
//   :81-90   cvtColor -> GaussianBlur((3, 3), 1.5) -> resize to 1/ds   ecc_prepare_kernel   bit-exact (15-bit luma, fixed-point blur
//                                                                                             taps 79 / 98 / 79 in 1/256, 8-bit resize)
//   :93-100  the first frame becomes the template -- and stays it: every later frame is aligned to frame 1 (quirk q17)
//   :105     cv2.findTransformECC(MOTION_EUCLIDEAN, 100 iterations, eps 1e-5, no mask, gaussFiltSize 1)
//                                                                       ecc_iterate_kernel   per iteration: fixed-point bilinear warp of
//            the image and of its [-0.5, 0, 0.5] gradients (1/32 px source coordinates, as warpAffine), nearest-neighbour mask, 21 sums in
//            fp64, then the 3 x 3 Gauss-Newton step with OpenCV's fp32 roundings of the Hessian, its inverse and the projections
//   :104-109 on an exception (lambda_d <= 0, NaN rho) H is the map after the last completed update
// One thread-block cluster per sequence (blockIdx.y) runs all iterations in one launch: every CTA sums a fixed slice of the
// pixels, the per-CTA partials are combined over distributed shared memory in rank order, one thread solves the step, and two
// cluster barriers bracket it.  Fixed partition, fixed reduction tree: the result is bitwise the same from call to call and for
// any number of sequences per call.  The host simulator (tests/hostsim) runs one block at a time, so it instantiates cluster size
// 1; the DSMEM combine is exercised by the GPU tests only.
// Compiled with --fmad=false: the fp32 warp and Jacobian round like OpenCV's separate multiplies and adds.
#include <string>          // before b2t_platform.cuh (the simulator's __noinline__ macro must not reach libstdc++)
#include <math.h>
#include "b2t_platform.cuh"
#include "b2t_luma.cuh"
#include "../../include/b200track.h"
#if !defined(B2T_HOSTSIM)
#include <cooperative_groups.h>
#endif

namespace b2t { void set_detect_error(const char* m); }

namespace {

#if defined(B2T_HOSTSIM)
inline int __double2int_rn(double v) { return v >= 2147483647.0 ? 2147483647 : (v <= -2147483648.0 ? (-2147483647 - 1) : (int)lrint(v)); }
#endif

constexpr int kThreads = 512;              // per CTA
constexpr int kClusterGpu = 8;             // CTAs per sequence on the GPU (portable cluster size)
constexpr int kSums = 21;
constexpr int kStateWords = 64;            // [0] frames seen

struct EccGeom {
    int n_seq, src_h, src_w, pitch, ds;
    int h, w;                              // working (down-scaled) size
    size_t o_state, o_tmpl, o_cur, stride;
};

size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

bool make_geom(int n_seq, int height, int width, int pitch, int ds, EccGeom* g) {
    if (n_seq < 1 || height < 1 || width < 1 || ds < 1 || ds > 16 || pitch < 3 * width) return false;
    g->n_seq = n_seq; g->src_h = height; g->src_w = width; g->pitch = pitch; g->ds = ds;
    g->h = height / ds; g->w = width / ds;
    if (g->h < 8 || g->w < 8 || g->h > 8192 || g->w > 8192) return false;
    const size_t px = (size_t)g->h * g->w;
    size_t o = 0;
    g->o_state = o; o += align256(kStateWords * sizeof(int));
    g->o_tmpl = o; o += align256(px);
    g->o_cur = o; o += align256(px);
    g->stride = o;
    return true;
}

template <class T> B2T_DEV T* wsp(unsigned char* ws, const EccGeom& g, int seq, size_t off) {
    return reinterpret_cast<T*>(ws + (size_t)seq * g.stride + off);
}

// ---------------------------------------------------------------------------------------------- preparation
B2T_DEV int refl101(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// GaussianBlur((3, 3), 1.5) of the gray image at (y, x): rows then columns in 8-bit fixed point, (v + 2^15) >> 16
B2T_DEV int blur_at(const unsigned char* img, const EccGeom& g, int y, int x) {
    const int x0 = refl101(x - 1, g.src_w) * 3, x1 = x * 3, x2 = refl101(x + 1, g.src_w) * 3;
    int v = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const unsigned char* r = img + (size_t)refl101(y + i - 1, g.src_h) * g.pitch;
        const int row = 79 * gray_of(r + x0) + 98 * gray_of(r + x1) + 79 * gray_of(r + x2);
        v += (i == 1 ? 98 : 79) * row;
    }
    return (v + (1 << 15)) >> 16;
}

// BGR -> gray -> blur -> 1/ds into the template plane on a sequence's first frame, into the current plane afterwards
__global__ void ecc_prepare_kernel(const unsigned char* __restrict__ frames, unsigned char* ws, EccGeom g, double scale_x, double scale_y) {
    const int seq = blockIdx.y;
    const unsigned char* img = frames + (size_t)seq * g.src_h * g.pitch;
    const int* state = wsp<int>(ws, g, seq, g.o_state);
    unsigned char* out = wsp<unsigned char>(ws, g, seq, state[0] == 0 ? g.o_tmpl : g.o_cur);
    const int total = g.h * g.w;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int y = i / g.w, x = i - y * g.w;
        int v;
        if (g.ds == 1) {                                                   // botsort.py:86: no blur, no resize
            v = gray_of(img + (size_t)y * g.pitch + x * 3);
        } else if (g.ds == 2 && g.src_h == 2 * g.h && g.src_w == 2 * g.w) {  // INTER_LINEAR at exactly 1/2 == 2 x 2 INTER_AREA
            v = (blur_at(img, g, 2 * y, 2 * x) + blur_at(img, g, 2 * y, 2 * x + 1) + blur_at(img, g, 2 * y + 1, 2 * x) +
                 blur_at(img, g, 2 * y + 1, 2 * x + 1) + 2) >> 2;
        } else {
            v = resize_linear_px([&](int yy, int xx) { return blur_at(img, g, yy, xx); }, x, y, g.src_h, g.src_w, scale_x, scale_y);
        }
        out[i] = (unsigned char)v;
    }
}

// ---------------------------------------------------------------------------------------------- one pixel of the warped images
struct Map { float m00, m01, m02, m10, m11, m12; };

struct Warped { float I, gx, gy; bool mask; };

// warpAffine(INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT 0) of the plane and of its filter2D([-0.5, 0, 0.5]) gradients
// (BORDER_REFLECT_101: 0 in the first and last column / row) at destination (x, y), and warpAffine(ones, INTER_NEAREST) there.
// The source coordinate is OpenCV's fixed point: round-half-even of M * x * 2^10 per column and of (M * y + t) * 2^10 per row,
// + 2^4 and >> 5 for 1/32-px bilinear (+ 2^9, >> 10 for nearest); the tap weights are products of multiples of 1/32 (exact in
// fp32) and the four taps are summed in the order (0, 0), (0, 1), (1, 0), (1, 1), as warpAffine's remap does.
B2T_DEV Warped warp_px(const unsigned char* __restrict__ P, int h, int w, const Map& M, int x, int y) {
    const int ad = __double2int_rn((double)M.m00 * (double)x * 1024.0), bd = __double2int_rn((double)M.m10 * (double)x * 1024.0);
    const int X0 = __double2int_rn(((double)M.m01 * (double)y + (double)M.m02) * 1024.0);
    const int Y0 = __double2int_rn(((double)M.m11 * (double)y + (double)M.m12) * 1024.0);
    Warped r;
    {
        const int Xn = (X0 + 512 + ad) >> 10, Yn = (Y0 + 512 + bd) >> 10;
        r.mask = Xn >= 0 && Xn < w && Yn >= 0 && Yn < h;
    }
    const int X = (X0 + 16 + ad) >> 5, Y = (Y0 + 16 + bd) >> 5;
    const int sx = X >> 5, sy = Y >> 5;
    const float fx = (float)(X & 31) * (1.f / 32.f), fy = (float)(Y & 31) * (1.f / 32.f);
    const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
    float v[2][2], gx[2][2], gy[2][2];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int yy = sy + a, xx = sx + b;
            v[a][b] = gx[a][b] = gy[a][b] = 0.f;
            if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
                const unsigned char* p = P + (size_t)yy * w + xx;
                v[a][b] = (float)p[0];
                if (xx > 0 && xx < w - 1) gx[a][b] = 0.5f * (float)((int)p[1] - (int)p[-1]);
                if (yy > 0 && yy < h - 1) gy[a][b] = 0.5f * (float)((int)p[w] - (int)p[-w]);
            }
        }
    r.I = v[0][0] * w00 + v[0][1] * w01 + v[1][0] * w10 + v[1][1] * w11;
    r.gx = gx[0][0] * w00 + gx[0][1] * w01 + gx[1][0] * w10 + gx[1][1] * w11;
    r.gy = gy[0][0] * w00 + gy[0][1] * w01 + gy[1][0] * w10 + gy[1][1] * w11;
    return r;
}

// the same for a whole plane (tests: the warp stage against cv2.warpAffine)
__global__ void ecc_warp_kernel(const unsigned char* __restrict__ P, int h, int w, Map M, float* img, float* gx, float* gy, unsigned char* mask) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < h * w; i += gridDim.x * blockDim.x) {
        const int y = i / w, x = i - y * w;
        const Warped r = warp_px(P, h, w, M, x, y);
        img[i] = r.I; gx[i] = r.gx; gy[i] = r.gy; mask[i] = r.mask ? 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------------- cluster plumbing
#if defined(B2T_HOSTSIM)
template <int C> B2T_DEV void cluster_sync() { __syncthreads(); }
template <int C, class T> B2T_DEV T* cluster_map(T* p, int) { return p; }
#else
template <int C> B2T_DEV void cluster_sync() { cooperative_groups::this_cluster().sync(); }
template <int C, class T> B2T_DEV T* cluster_map(T* p, int rank) { return cooperative_groups::this_cluster().map_shared_rank(p, rank); }
#endif

B2T_DEV double f32(double v) { return (double)(float)v; }

struct Ctl {
    Map map;
    double rho, last_rho;
    int it, flags, stop;
};

// the Gauss-Newton step of findTransformECC from the 21 sums (one thread).  S: n, SI, SII, ST, STT, STI, SJI[3], SJ[3], SJT[3],
// SJJ[6] (00 01 02 11 12 22).  Returns 0 or the failure flag; on failure the map is left as it was.
B2T_DEV int ecc_step(const double* S, Map& M, double& rho) {
    const double n = S[0];
    const double im = S[1] / n, tm = S[3] / n;
    const double iv = S[2] / n - im * im, tv = S[4] / n - tm * tm;
    const double istd = sqrt(iv > 0.0 ? iv : 0.0), tstd = sqrt(tv > 0.0 ? tv : 0.0);
    const double imf = f32(im), tmf = f32(tm);                       // subtract(img, mean, ..., mask) with the mean as fp32
    const double tnorm = sqrt(n * tstd * tstd), inorm = sqrt(n * istd * istd);
    double Hm[3][3];                                                  // the Hessian is a CV_32F matrix
    Hm[0][0] = f32(S[15]); Hm[0][1] = Hm[1][0] = f32(S[16]); Hm[0][2] = Hm[2][0] = f32(S[17]);
    Hm[1][1] = f32(S[18]); Hm[1][2] = Hm[2][1] = f32(S[19]); Hm[2][2] = f32(S[20]);
    double Hi[3][3];                                                  // Mat::inv(): closed form in double, rounded to fp32
    {
        const double (&m)[3][3] = Hm;
        double d = m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
                   m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
        if (d != 0.0) {
            d = 1.0 / d;
            Hi[0][0] = f32((m[1][1] * m[2][2] - m[1][2] * m[2][1]) * d); Hi[0][1] = f32((m[0][2] * m[2][1] - m[0][1] * m[2][2]) * d);
            Hi[0][2] = f32((m[0][1] * m[1][2] - m[0][2] * m[1][1]) * d); Hi[1][0] = f32((m[1][2] * m[2][0] - m[1][0] * m[2][2]) * d);
            Hi[1][1] = f32((m[0][0] * m[2][2] - m[0][2] * m[2][0]) * d); Hi[1][2] = f32((m[0][2] * m[1][0] - m[0][0] * m[1][2]) * d);
            Hi[2][0] = f32((m[1][0] * m[2][1] - m[1][1] * m[2][0]) * d); Hi[2][1] = f32((m[0][1] * m[2][0] - m[0][0] * m[2][1]) * d);
            Hi[2][2] = f32((m[0][0] * m[1][1] - m[0][1] * m[1][0]) * d);
        } else {
            for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) Hi[a][b] = 0.0;
        }
    }
    const double corr = S[5] - imf * S[3] - tmf * S[1] + n * tmf * imf;
    rho = corr / (inorm * tnorm);
    double ip[3], tp[3], ipf[3], tpf[3];
    for (int k = 0; k < 3; ++k) {
        ip[k] = S[6 + k] - imf * S[9 + k];                            // J . (image - mean on the mask, raw elsewhere)
        tp[k] = S[12 + k] - tmf * S[9 + k];                           // J . (template - mean on the mask, 0 elsewhere)
        ipf[k] = f32(ip[k]); tpf[k] = f32(tp[k]);
    }
    double iph[3];
    for (int a = 0; a < 3; ++a) iph[a] = f32(Hi[a][0] * ipf[0] + Hi[a][1] * ipf[1] + Hi[a][2] * ipf[2]);
    const double lam_n = inorm * inorm - (ipf[0] * iph[0] + ipf[1] * iph[1] + ipf[2] * iph[2]);
    const double lam_d = corr - (tpf[0] * iph[0] + tpf[1] * iph[1] + tpf[2] * iph[2]);
    if (lam_d <= 0.0) return B2T_ECC_FAILED_LAMBDA;
    if (!(rho == rho)) return B2T_ECC_FAILED_NAN;                    // OpenCV 4.13 tests rho for NaN after lambda_d (oracle/ecc.py)
    const double lam = lam_n / lam_d;
    double ep[3], dp[3];
    for (int k = 0; k < 3; ++k) ep[k] = f32(lam * tp[k] - ip[k]);     // J . (lambda * templateZM - imageZM)
    for (int a = 0; a < 3; ++a) dp[a] = f32(Hi[a][0] * ep[0] + Hi[a][1] * ep[1] + Hi[a][2] * ep[2]);
    const double theta = dp[0] + asin((double)M.m10);                 // update_warping_matrix_ECC, MOTION_EUCLIDEAN
    M.m02 = M.m02 + (float)dp[1];
    M.m12 = M.m12 + (float)dp[2];
    M.m00 = M.m11 = (float)cos(theta);
    M.m10 = (float)sin(theta);
    M.m01 = -M.m10;
    return 0;
}

template <int C>
__global__ void __launch_bounds__(kThreads, 1) ecc_iterate_kernel(unsigned char* ws, EccGeom g, int max_iter, double eps, double* __restrict__ warps,
                                                                 int* __restrict__ stat) {
    const int seq = blockIdx.y, rank = blockIdx.x;                    // gridDim.x == C: the cluster is one sequence
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    int* state = wsp<int>(ws, g, seq, g.o_state);
    const int frames_seen = state[0];
    if (frames_seen == 0) {                                           // botsort.py:93-100: the template is stored, H = I
        cluster_sync<C>();                                            // every thread of the cluster has read the frame counter
        if (rank == 0 && tid == 0) {
            double* H = warps + (size_t)seq * 6;
            H[0] = 1; H[1] = 0; H[2] = 0; H[3] = 0; H[4] = 1; H[5] = 0;
            if (stat) {
                int* st = stat + (size_t)seq * B2T_GMC_STAT_WORDS;
                for (int k = 0; k < B2T_GMC_STAT_WORDS; ++k) st[k] = 0;
                st[5] = B2T_ECC_FIRST_FRAME;
            }
            state[0] = 1;
        }
        return;
    }
    const unsigned char* T = wsp<unsigned char>(ws, g, seq, g.o_tmpl);
    const unsigned char* P = wsp<unsigned char>(ws, g, seq, g.o_cur);
    __shared__ double s_warp[kThreads / 32][kSums];
    __shared__ double s_part[kSums];
    __shared__ double s_tot[kSums];
    __shared__ Ctl s_ctl;
    const int total = g.h * g.w;
    const int p0 = (int)((long long)total * rank / C), p1 = (int)((long long)total * (rank + 1) / C);
    Map M = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f};
    if (rank == 0 && tid == 0) { s_ctl.map = M; s_ctl.rho = -1.0; s_ctl.last_rho = -eps; s_ctl.it = 0; s_ctl.flags = 0; }
    bool stop = !(max_iter > 0 && fabs(-1.0 + eps) >= eps);
    while (!stop) {
        double acc[kSums];
#pragma unroll
        for (int k = 0; k < kSums; ++k) acc[k] = 0.0;
        const float c = M.m00, s = M.m10;
        for (int i = p0 + tid; i < p1; i += kThreads) {
            const int y = i / g.w, x = i - y * g.w;
            const Warped r = warp_px(P, g.h, g.w, M, x, y);
            const float xf = (float)x, yf = (float)y;
            const float hatX = -(xf * s) - (yf * c), hatY = xf * c - yf * s;   // image_jacobian_euclidean_ECC
            const double J[3] = {(double)(r.gx * hatX + r.gy * hatY), (double)r.gx, (double)r.gy};
            const double I = (double)r.I;
#pragma unroll
            for (int k = 0; k < 3; ++k) acc[6 + k] += J[k] * I;
            acc[15] += J[0] * J[0]; acc[16] += J[0] * J[1]; acc[17] += J[0] * J[2];
            acc[18] += J[1] * J[1]; acc[19] += J[1] * J[2]; acc[20] += J[2] * J[2];
            if (r.mask) {
                const double t = (double)T[i];
                acc[0] += 1.0; acc[1] += I; acc[2] += I * I; acc[3] += t; acc[4] += t * t; acc[5] += t * I;
#pragma unroll
                for (int k = 0; k < 3; ++k) { acc[9 + k] += J[k]; acc[12 + k] += J[k] * t; }
            }
        }
        // fixed reduction tree: butterfly in the warp, warps in order, CTAs in rank order
#pragma unroll
        for (int k = 0; k < kSums; ++k) {
            double v = acc[k];
            for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(B2T_FULL, v, d);
            if (lane == 0) s_warp[wid][k] = v;
        }
        __syncthreads();
        if (tid < kSums) {
            double v = 0.0;
            for (int q = 0; q < kThreads / 32; ++q) v += s_warp[q][tid];
            s_part[tid] = v;
        }
        cluster_sync<C>();                                            // every CTA's partial is in its shared memory
        if (rank == 0) {
            if (tid < kSums) {
                double v = 0.0;
                for (int q = 0; q < C; ++q) v += cluster_map<C>(s_part, q)[tid];
                s_tot[tid] = v;
            }
            __syncthreads();
            if (tid == 0) {
                Map m = s_ctl.map;
                double rho = 0.0;
                const int fail = ecc_step(s_tot, m, rho);
                s_ctl.it += 1;
                s_ctl.last_rho = s_ctl.rho;
                s_ctl.rho = rho;
                if (fail) {
                    s_ctl.flags = fail;
                    s_ctl.stop = 1;
                } else {
                    s_ctl.map = m;
                    const bool conv = fabs(s_ctl.rho - s_ctl.last_rho) < eps;
                    s_ctl.stop = conv || s_ctl.it >= max_iter;
                    s_ctl.flags = conv ? B2T_ECC_CONVERGED : (s_ctl.it >= max_iter ? B2T_ECC_ITER_CAP : 0);
                }
            }
        }
        cluster_sync<C>();                                            // the new map is in rank 0's shared memory
        const Ctl* ctl = cluster_map<C>(&s_ctl, 0);
        M = ctl->map;
        stop = ctl->stop != 0;
    }
    cluster_sync<C>();                                                // rank 0's shared memory stays alive until all have read it
    if (rank == 0 && tid == 0) {
        const Ctl& k = s_ctl;
        double* H = warps + (size_t)seq * 6;
        H[0] = k.map.m00; H[1] = k.map.m01; H[2] = k.map.m02; H[3] = k.map.m10; H[4] = k.map.m11; H[5] = k.map.m12;
        if (stat) {
            int* st = stat + (size_t)seq * B2T_GMC_STAT_WORDS;
            unsigned long long bits;
            memcpy(&bits, &k.rho, 8);
            st[0] = k.it; st[1] = (int)(unsigned)(bits & 0xffffffffull); st[2] = (int)(unsigned)(bits >> 32); st[3] = 0; st[4] = 0;
            st[5] = k.flags; st[6] = 0; st[7] = frames_seen;
        }
        state[0] = frames_seen + 1;
    }
}

int efail(int code, const char* m) { b2t::set_detect_error(m); return code; }
int echeck(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { b2t::set_detect_error((std::string(what) + ": " + cudaGetErrorString(e)).c_str()); return B2T_ECUDA; }
    return B2T_OK;
}

int launch_iterate(const EccGeom& g, unsigned char* ws, int max_iter, double eps, double* warps, int* stat, cudaStream_t s) {
#if defined(B2T_HOSTSIM)
    B2T_LAUNCH(ecc_iterate_kernel<1>, dim3(1, g.n_seq), kThreads, 0, s, ws, g, max_iter, eps, warps, stat);
    return B2T_OK;
#else
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(kClusterGpu, g.n_seq);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = kClusterGpu; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, ecc_iterate_kernel<kClusterGpu>, ws, g, max_iter, eps, warps, stat);
    if (e != cudaSuccess) return efail(B2T_ECUDA, (std::string("ecc_iterate_kernel: ") + cudaGetErrorString(e)).c_str());
    return B2T_OK;
#endif
}

}  // namespace

extern "C" size_t b2t_ecc_workspace_bytes(int n_seq, int height, int width, int downscale) {
    EccGeom g;
    if (!make_geom(n_seq, height, width, 3 * width, downscale, &g)) return 0;
    return g.stride * (size_t)n_seq;
}

extern "C" int b2t_ecc_workspace_layout(int n_seq, int height, int width, int downscale, size_t* out, int n) {
    EccGeom g;
    if (!out || !make_geom(n_seq, height, width, 3 * width, downscale, &g)) return efail(B2T_EINVAL, "b2t_ecc_workspace_layout: bad arguments");
    const size_t v[6] = {g.stride, g.o_state, g.o_tmpl, g.o_cur, (size_t)g.h, (size_t)g.w};
    for (int i = 0; i < n && i < 6; ++i) out[i] = v[i];
    return B2T_OK;
}

extern "C" int b2t_ecc_reset(void* workspace, int n_seq, int height, int width, int downscale, void* stream) {
    EccGeom g;
    if (!workspace || !make_geom(n_seq, height, width, 3 * width, downscale, &g)) return efail(B2T_EINVAL, "b2t_ecc_reset: bad arguments");
    for (int s = 0; s < n_seq; ++s)
        if (cudaMemsetAsync((unsigned char*)workspace + (size_t)s * g.stride + g.o_state, 0, kStateWords * sizeof(int), (cudaStream_t)stream) != 0)
            return efail(B2T_ECUDA, "b2t_ecc_reset: memset failed");
    return B2T_OK;
}

extern "C" int b2t_ecc_estimate(const unsigned char* frames_bgr, int n_seq, int height, int width, int pitch, int downscale, int max_iter, double eps,
                                void* workspace, double* warps_out, int* stat, void* stream) {
    EccGeom g;
    if (!frames_bgr || !workspace || !warps_out || max_iter < 1 || max_iter > 100000 || !(eps >= 0.0) || !make_geom(n_seq, height, width, pitch, downscale, &g))
        return efail(B2T_EINVAL, "b2t_ecc_estimate: bad arguments (at least 8 px per side after down-scaling, pitch >= 3 * width, 1 <= max_iter <= 100000, eps >= 0)");
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = (unsigned char*)workspace;
    const int px = g.h * g.w;
    const int gx = (px + 255) / 256 < 132 * 4 ? (px + 255) / 256 : 132 * 4;
    const double scale_x = 1.0 / ((double)g.w / (double)g.src_w), scale_y = 1.0 / ((double)g.h / (double)g.src_h);
    B2T_LAUNCH(ecc_prepare_kernel, dim3(gx, g.n_seq), 256, 0, s, frames_bgr, ws, g, scale_x, scale_y);
    int rc = echeck("ecc_prepare_kernel");
    if (rc != B2T_OK) return rc;
    rc = launch_iterate(g, ws, max_iter, eps, warps_out, stat, s);
    return rc != B2T_OK ? rc : echeck("ecc_iterate_kernel");
}

extern "C" int b2t_ecc_warp(const unsigned char* plane, int height, int width, const float* map_host, float* img, float* gx, float* gy, unsigned char* mask,
                            void* stream) {
    if (!plane || !map_host || !img || !gx || !gy || !mask || height < 2 || width < 2 || height > 8192 || width > 8192)
        return efail(B2T_EINVAL, "b2t_ecc_warp: bad arguments");
    const Map M = {map_host[0], map_host[1], map_host[2], map_host[3], map_host[4], map_host[5]};
    const int px = height * width;
    const int gx_ = (px + 255) / 256 < 132 * 4 ? (px + 255) / 256 : 132 * 4;
    B2T_LAUNCH(ecc_warp_kernel, dim3(gx_), 256, 0, (cudaStream_t)stream, plane, height, width, M, img, gx, gy, mask);
    return echeck("ecc_warp_kernel");
}
