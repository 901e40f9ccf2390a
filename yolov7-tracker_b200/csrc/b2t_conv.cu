// b2t_conv.cu -- conv2d + bias + SiLU as an implicit GEMM on the Hopper tensor cores (sm_90a: TMA + wgmma).
//
// Replaces ``Conv.fuseforward`` (models/common.py:110-111: act(conv(x)) with BN folded by
// utils/torch_utils.py:181-201) and the linear 1x1 head convs of ``Detect`` (models/yolo.py:44)
// for the YOLOv7-w6 / tiny graphs (k in {1,3}, s in {1,2}, pad k//2, groups 1).
//
//   D[pixel, cout] = sum_{kh,kw,cin} X[n, ho*s+kh-p, wo*s+kw-p, cin] * W[cout, kh, kw, cin]
//
// Layout: activations NHWC bf16 / fp16 (a tensor may be a channel slice of a wider concat buffer: pitch !=
// C), weights [Cout][KH][KW][Cin] (K-major), bias fp32, accumulation fp32 in registers.
//
// One CTA computes tiles of MT x 128 pixels x BLOCK_N channels:
//   * the 128 pixels of a sub-tile are a TH x TW spatial patch of one image (TH*TW = 128).  For filter tap
//     (kh,kw) and channel chunk kc the A operand is ONE TMA box {BK ch, TW, TH, 1} of the 4-D
//     tensor map (C, W, H, N) at coordinates (kc*BK, wo0*s+kw-p, ho0*s+kh-p, n): out-of-bounds
//     rows/cols are zero-filled by the TMA unit (that IS the padding), stride-2 convs use the tensor
//     map's element strides, and the box lands in shared memory as 128 rows of BK*2 bytes with the
//     128-/64-/32-byte swizzle -- exactly the canonical K-major wgmma operand layout.
//   * PIXEL RUNS (3x3, tile_w = 128): the 128 pixels of a sub-tile are instead 128 consecutive pixels of the flattened N*Ho*Wo output
//     axis, as in flat mode, so maps that no TH x TW patch divides (20 x 20, 40 x 40) compute no padding pixels.  For tap (kh,kw) and
//     chunk kc the A operand of the whole tile is ONE im2col box (cp.async.bulk.tensor.im2col, cuTensorMapEncodeIm2col) of 128*MT
//     pixels x BK channels: the TMA unit walks the output pixels through a bounding box of the input (corners -pad .. pad-(k-1), the
//     conv stride as traversal stride) in W, then H, then N order -- across rows and images -- and reads each at the tap's offset
//     (kw, kh), zero-filling outside the image.  It lands in the same 128-row swizzled layout as the tiled boxes, and the
//     epilogue stores through flat mode's 2-D (C, N*Ho*Wo) map.
//   * B operand: 2-D map (K, Cout), box {BK, BLOCK_N}.
//   * warps [0, 8 MT) are the consumers, issuing wgmma.mma_async m64 x BLOCK_N x k16 with the accumulators in registers, then
//     the epilogue from those registers: +bias -> SiLU (one tanh.approx on the SFU) -> fp16 / bf16 (or fp32) -> 128-byte-swizzled
//     staging tile -> TMA bulk tensor STORES straight into the consumer's concat buffer
//     (concat-by-address; partial tiles and the 255-channel head are clipped by the TMA unit).  Two schedules, fixed by (MT, BLOCK_N):
//       - PING-PONG (MT = 1, BLOCK_N <= 128): each of the two warpgroups owns WHOLE 128-pixel tiles (both m64 halves) and they take
//         alternate tiles; a turn barrier pair orders their MMA loops, so one warpgroup's epilogue runs under the other's MMAs.
//       - COOPERATIVE (MT = 2, or BLOCK_N = 256): two warpgroups per 128-pixel sub-tile, one m64 half each, epilogue together.
//     Both sum every output in the same K order, so the schedule changes the time, never a result bit.
//   * the warpgroup after the consumers is the producer warpgroup: 1 or 2 of its warps issue TMA copies, and it hands most of
//     its registers to the consumers (setmaxnreg), which is what lets a warpgroup hold 128 x 128 or 64 x 256 accumulators unspilled.
//   * PERSISTENT: the grid is (#SMs x CTAs/SM); a CTA draws every tile, the first one included, from a global
//     ticket counter (N tile fastest, so neighbouring CTAs share the A tile in L2); the first producer warp publishes every tile
//     index to the other warps through a small mbarrier-guarded ring in shared memory.  The operand ring (full/empty mbarriers)
//     keeps running across tile boundaries: the producers load the next tile's operands while the consumers run the epilogue.
//   * HALO mode (3x3, stride 1): one (TH+2) x (TW+2) input tile per K chunk instead of one tile per tap; the nine taps
//     are shifted windows of it (descriptor start + (kh*(TW+2) + kw) * BK*2 B, 8-row groups strided by the halo row pitch; BK = 16 / 32 use the 32- / 64-byte swizzle the same way).
//   * ROW-PACKED stem (Cin = 16): the three kw taps of a kernel row form one 64-wide K chunk through an
//     overlapping-stride tensor map on a zero-padded input buffer.
//   * Launched with programmatic stream serialization: griddepcontrol.launch_dependents / .wait bracket the CTA setup.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string>
#include <cstdio>
#include <cstdlib>
#include "../../include/b200track.h"
#include "b2t_wgmma.cuh"

namespace {

constexpr int kMaxStages = 8;
constexpr int kTileM = 128;        // pixels per sub-tile = rows of two m64 wgmma warpgroups
constexpr int kMaxHalo = 3;        // halo-tile buffers (halo mode)
constexpr int kRing = 4;           // tile-index ring depth (the producer runs at most a few tiles ahead)
constexpr int kMaxProducers = 2;   // warps [8 MT, 8 MT + P) of the producer warpgroup issue TMA copies; the others idle

// the consumer schedule is a function of the instantiation (see the header); the host sizes the staging boxes from it
__host__ __device__ constexpr bool ping_pong(int mt, int bn) { return mt == 1 && bn <= 128; }
// register budget: one CTA per SM.  ptxas sizes the launch allocation from __launch_bounds__ (65536 / threads, rounded down to 8
// per thread); the producer warpgroup lowers its limit with setmaxnreg.dec and the consumers raise theirs by what that freed inside
// the CTA: 168 -> 224 with 384 threads (MT = 1), 96 -> 104 with 640 (MT = 2).  48 is the least the producer code runs in unspilled.
__host__ __device__ constexpr int conv_threads(int mt) { return 256 * mt + 128; }
__host__ __device__ constexpr int launch_regs(int mt) { return 65536 / conv_threads(mt) / 8 * 8; }
constexpr int kProducerRegs = 48;
__host__ __device__ constexpr int consumer_regs(int mt) { return (launch_regs(mt) + (launch_regs(mt) - kProducerRegs) * 128 / (256 * mt)) / 8 * 8; }
static_assert(consumer_regs(1) == 224 && consumer_regs(2) == 104, "register hand-off");

struct ConvParams {
    int N, H, W, Cin;              // input geometry (Cin = channels of the slice read)
    int Ho, Wo, Cout;              // output geometry
    int KH, KW, stride, pad;       // pad = padding rows (kh/2)
    int pad_w;                     // padding columns applied through the A map's x coordinate (0 for row-packed layers)
    int halo;                      // 1 = halo-tile mode (3x3 / stride 1): one (TH+2) x (MT*TW+2) input tile per K chunk feeds all nine taps
    int halo_bytes;                // bytes of one halo buffer, rounded up to 1024
    int halo_bufs;                 // halo buffers in the A ring
    int kpair;                     // flat (1x1) mode: K chunks per ring stage (1 or 2): two chunks travel as ONE 3-D box per operand
    int tps;                       // halo mode: filter taps per weight-ring stage: 1, 3 (one kernel row = ONE 3-D TMA box) or 9 (b_res)
    int b_res;                     // halo mode, one K chunk, one N tile: the CTA's nine weight tiles are loaded once and stay resident
    int out_bufs;                  // epilogue staging boxes (128 pixels x 128 B each) per sub-tile: 1 or 2
    int MT;                        // sub-tiles of 128 pixels per tile (1 or 2): every weight tile that reaches shared memory feeds MT sub-tiles
    int sub_off;                   // bytes from sub-tile 0's A operand to sub-tile 1's inside a stage / halo buffer
    int TH, TW;                    // spatial extent of ONE sub-tile, TH*TW == 128
    int BK;                        // K chunk: 64 (SW128), 32 (SW64) or 16 (SW32) channels
    int BN;                        // output channels per CTA: 32, 64, 128 or 256 (the wgmma N)
    int tiles_w, tiles_h;          // tiles per image
    int out_pitch;                 // elements per output pixel (concat buffer width)
    int out_coff;                  // channel offset inside the output buffer
    int act;                       // 1 = SiLU, 0 = linear / ReLU (act_floor)
    float act_floor, act_slope;    // linear epilogue: max(max(v, floor), v * slope): (-inf, 1) = plain linear, (0, 1) = ReLU (the ReID extractor),
                                   // (-inf, 0.1) = LeakyReLU(0.1) (YOLOv7-tiny, cfg/deploy/yolov7-tiny.yaml:15)
    int out_f32;                   // 1 = fp32 output (head), 0 = 16-bit (bf16 or fp16)
    int f16;                       // 1 = operands (and 16-bit outputs) are IEEE fp16, 0 = bf16
    int flat;                      // 1 = pixels are the flattened N*Ho*Wo axis, TH/TW unused: 1x1/s1 (2-D A map) or pixel runs
    int im2col;                    // 1 = pixel runs (flat): the A operand of a tap is one im2col box of the tile's MT*128 output pixels
    int stages;                    // shared-memory ring depth (<= kMaxStages)
    int tiles_m, tiles_n;          // tile grid; tile t -> (m = t / tiles_n, n = t % tiles_n)
    int P;                         // TMA producer warps (1..2): a thread's bulk-tensor copies are served one after the other,
                                   // so two issuing threads fill the ring faster than one
    int splits;                    // split-K: work unit u = tile * splits + split; partial sums meet in `ws`
    int ksteps;                    // K steps of a whole tile: halo mode = channel chunks (9 taps each), otherwise taps x chunks
    long long total_pix;           // N*Ho*Wo (flat mode bound)
    float* ws;                     // split-K workspace [unit][MT][128][BN] fp32 (splits > 1)
    int* flags;                    // split-K arrival counters [tile][MT], self-resetting
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// im2col mode: the box is the run of output pixels that starts at bounding-box position (w, h, n), each read at (+ow, +oh)
__device__ __forceinline__ void tma_load_im2col_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c, int w, int h, int n, uint16_t ow, uint16_t oh) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(ow), "h"(oh) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
// one lane of a converged warp (elect.sync): the caller's control flow stays uniform up to this branch
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across wgmma fences / waits
template <int H, int R> __device__ __forceinline__ void acc_fence(float (&d)[H][R]) {
#pragma unroll
    for (int h = 0; h < H; ++h)
#pragma unroll
        for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[h][i])::"memory");
}
template <int N> struct Steps { static constexpr int value = N; };
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// SiLU with ONE SFU operation: x * sigmoid(x) = h + h * tanh(h), h = x / 2  (MUFU.TANH + 1 FMUL + 1 FFMA per element).
// max |error| 1.0e-5 on [-12, 12] -- below fp16 output rounding for |x| > 0.02 and far below bf16's.
__device__ __forceinline__ float silu(float v) {
    const float h = 0.5f * v;
    float t;
    asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
    return fmaf(h, t, h);
}

__device__ __forceinline__ uint32_t pack16(float a, float b, bool f16) {
    if (f16) { const __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<const uint32_t*>(&h); }
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b); return *reinterpret_cast<const uint32_t*>(&h);
}

// Staging box bx (128 pixel rows x 128 bytes = 64 halves / 32 floats of channels, 128-byte swizzle) of one sub-tile, the part this
// thread holds: wgmma's m64 fragment gives thread (warp w, lane l) of a warpgroup rows 16 w + l / 4 and + 8, and in every group of 8
// columns the two at 2 (l % 4).  r0 = the first of its two rows inside the sub-tile.  + bias -> activation -> 16-bit / fp32.
// (The column groups are walked at compile time and filtered by the box index, so the accumulator stays in registers.)
template <bool F32, bool F16, int BN>
__device__ __forceinline__ void stage_box(const float (&acc)[BN / 2], int bx, const float* __restrict__ bias_c, uint8_t* box, int r0, int lane,
                                          int act, float floor_v, float slope_v) {
    constexpr int cpb = F32 ? 32 : 64;
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        if ((8 * j) / cpb != bx) continue;
        const int col = 8 * j + cq;
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias_c + col));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
            float v0 = acc[4 * j + 2 * h] + b.x, v1 = acc[4 * j + 2 * h + 1] + b.y;
            if (act) { v0 = silu(v0); v1 = silu(v1); }
            else {        // linear: floor -inf, slope 1 (max(v, v)); ReLU: floor 0, slope 1; LeakyReLU(a): floor -inf, slope a
                v0 = fmaxf(fmaxf(v0, floor_v), v0 * slope_v); v1 = fmaxf(fmaxf(v1, floor_v), v1 * slope_v);
            }
            const int byte = (col - bx * cpb) * (F32 ? 4 : 2);
            uint8_t* dst = box + r * 128 + ((((byte >> 4) ^ (r & 7)) << 4) | (byte & 15));
            if (F32) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
            else *reinterpret_cast<uint32_t*>(dst) = pack16(v0, v1, F16);
        }
    }
}

template <bool F32, bool F16, int MT, int BN>
__global__ void __launch_bounds__(conv_threads(MT), 1)
conv_bias_act_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                     const __grid_constant__ CUtensorMap map_c, const float* __restrict__ bias, int* __restrict__ sched,
                     const ConvParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int kConsumerWarps = 8 * MT;
    constexpr bool kPingPong = ping_pong(MT, BN);
    constexpr int kSlots = kPingPong ? 2 : MT;          // epilogue groups: staging boxes, named barrier, split-K flag each
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int a_bytes = kTileM * p.BK * 2;             // one sub-tile's A operand (generic / flat mode)
    const int b_bytes = BN * p.BK * 2;
    // generic mode: a ring of (MT A sub-tiles + B tile) stages.  halo mode: p.halo_bufs halo tiles, then a ring of B tiles.
    const int stage_bytes = (((p.halo ? p.tps * b_bytes : (MT * a_bytes + b_bytes) * p.kpair) + 1023) / 1024) * 1024;
    // swizzled operand tiles need 1024-byte alignment in the shared window (slack is reserved by the host)
    uint8_t* tiles = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);
    uint8_t* ring = tiles + (p.halo ? p.halo_bufs * p.halo_bytes : 0);
    const int kStages = p.stages;
    constexpr int box_bytes = kTileM * 128;             // one staging box: 128 pixels x 128 B (64 halves / 32 floats of channels)
    const int staging_bytes = p.out_bufs * box_bytes;   // per sub-tile
    uint8_t* stage_out = ring + kStages * stage_bytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(stage_out + kSlots * staging_bytes);
    uint64_t* empty_bar = full_bar + kMaxStages;
    uint64_t* ring_full = empty_bar + kMaxStages;                             // [kRing] tile-index ring, producer -> everybody else
    uint64_t* ring_empty = ring_full + kRing;                                 // [kRing]
    uint64_t* a_full = ring_empty + kRing;                                    // [kMaxHalo] halo-tile ring (halo mode)
    uint64_t* a_empty = a_full + kMaxHalo;
    uint64_t* mma_turn = a_empty + kMaxHalo;                                  // [2] ping-pong: "warpgroup w may issue its MMAs"
    int* tile_ring = reinterpret_cast<int*>(mma_turn + 2);                    // [kRing]
    int* last_flag = tile_ring + kRing;                                       // [2] split-K: "this epilogue group reduces the tile"
    int* first_unit = last_flag + 2;                                          // the CTA's first work unit (ticket drawn at entry)

    // generic mode walks K channel-chunk-major (step kt = chunk kt / taps, tap kt % taps), the order the halo mode accumulates in:
    // every addressing variant of a layer sums each output in the same order, so the autotuner's choice cannot change a result bit
    const int ntaps = p.KH * p.KW;
    const int total_units = p.tiles_m * p.tiles_n * p.splits;
    const int P = p.P;
    const int pw = warp - kConsumerWarps;               // producer warp index (< 0: consumer)

    // Programmatic dependent launch: let the next layer's CTAs be scheduled as soon as every CTA of this grid is running;
    // they do their own setup (barriers, descriptor prefetch) in the shadow of this layer's tail and then block in
    // griddepcontrol.wait below until this grid has completed.  (No-ops when launched without the attribute.)
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    // EVERY work unit is a ticket, the first one included: a CTA that becomes resident late (another stream's kernel -- the tracker
    // step of the previous frame -- holds its SM) draws a ticket past the end and retires at once instead of owning a tile that
    // would then run after everybody else has finished.  The launch's counter pair is one of four rotating sets (b2t_conv_run), so
    // drawing before griddepcontrol.wait cannot meet the previous launch of the same plan.  The atomic's latency hides behind the setup.
    if (pw == 0 && lane == 0) {
        *first_unit = atomicAdd(sched, 1);
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c) : "memory");
        // operand stages and halo buffers are released by every warpgroup that reads them: the owner alone in ping-pong
        constexpr int readers = kPingPong ? 1 : 2 * MT;
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], readers); }
        for (int r = 0; r < kRing; ++r) { mbar_init(&ring_full[r], 1); mbar_init(&ring_empty[r], P - 1 + kConsumerWarps); }
        for (int h = 0; h < kMaxHalo; ++h) { mbar_init(&a_full[h], 1); mbar_init(&a_empty[h], readers); }
        for (int w = 0; w < 2; ++w) mbar_init(&mma_turn[w], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // griddepcontrol.wait (the previous kernel in the stream has completed, its writes are visible) is executed by the producer
    // warps only, AFTER they have requested the first weight tiles: weights do not depend on the previous layer, so their DRAM
    // latency and the first ring fill overlap its tail.  Every other global access of this kernel is ordered after a producer's
    // loads through the mbarrier chain (activation tiles -> MMAs -> epilogue stores, split-K workspace, tickets).

    // work unit u -> tile coordinates and K-step range [k0, k1)
    auto unit_coords = [&](int u, int& n0, int& img, int& ho0, int& wo0, long long& pix0, int& k0, int& k1) {
        int t = u;
        k0 = 0; k1 = p.ksteps;
        if (p.splits > 1) {
            t = u / p.splits;
            const int sp = u - t * p.splits;
            k0 = (p.ksteps * sp) / p.splits;
            k1 = (p.ksteps * (sp + 1)) / p.splits;
        }
        const int mt = t / p.tiles_n, nt = t % p.tiles_n;
        n0 = nt * BN; img = 0; ho0 = 0; wo0 = 0; pix0 = 0;
        if (p.flat) pix0 = (long long)mt * (kTileM * MT);
        else {
            const int per_img = p.tiles_w * p.tiles_h;
            img = mt / per_img;
            const int r = mt % per_img;
            // halo mode: the MT sub-tiles sit side by side (TH rows x MT*TW pixels); generic mode: stacked (MT*TH rows x TW pixels)
            ho0 = (r / p.tiles_w) * (p.halo ? p.TH : p.TH * MT);
            wo0 = (r % p.tiles_w) * (p.halo ? p.TW * MT : p.TW);
        }
    };

    if (pw >= 0) {
        setmaxnreg_dec<kProducerRegs>();    // the whole producer warpgroup, before any warp of it leaves
        if (pw >= P) return;
        // ===== TMA producers.  Producer 0 is also the tile scheduler: the first unit is the ticket drawn at entry, later ones are drawn from
        // the same global counter, so a CTA that starts late (or shares its SM with another stream's kernel) simply takes fewer tiles
        // instead of stretching the layer; every unit index (and the final -1) is published to the other producer and the consumer
        // warps through a small shared-memory ring.  The K steps of the operand ring are dealt round-robin
        // to the P producers (step c belongs to producer c % P): bulk-tensor copies issued by one thread are served one at a
        // time, so P issuing threads give P times the fill rate.  All producers run ahead of the consumers, across tile boundaries.
        // (whole warp, uniform control flow; one elected lane issues the copies)
        int stage = 0; uint32_t phase = 0;
        int hbuf = 0; uint32_t hphase = 0;
        int rslot = 0; uint32_t rphase = 0;
        int c = 0;                                  // operand-ring step counter: (c % P == pw) -> this producer loads it
        int u = *first_unit;
        // weight tile(s) of ring step `s` of a unit that starts at K step k0 (n0 = its first output channel)
        const int groups = p.halo ? 9 / p.tps : 1;         // halo mode: weight boxes per K chunk
        auto load_b = [&](int st, int n0, int k0, int s) {
            uint8_t* sb = ring + st * stage_bytes + (p.halo ? 0 : MT * a_bytes * p.kpair);
            if (p.halo) {
                const int kc = k0 + s / groups, tap = (s % groups) * p.tps;
                if (p.tps == 1) tma_load_2d(sb, &map_b, &full_bar[st], tap * p.Cin + kc * p.BK, n0);
                else tma_load_3d(sb, &map_b, &full_bar[st], kc * p.BK, n0, tap);     // one kernel row: taps tap .. tap + 2
            } else if (p.kpair == 2) {
                tma_load_3d(sb, &map_b, &full_bar[st], 0, n0, 2 * (k0 + s));
            } else {
                const int kt = k0 + s, kc = kt / ntaps, tap = kt % ntaps;
                tma_load_2d(sb, &map_b, &full_bar[st], tap * p.Cin + kc * p.BK, n0);
            }
        };
        const uint32_t stage_tx = (uint32_t)(p.halo ? p.tps * b_bytes : (MT * a_bytes + b_bytes) * p.kpair);
        int npre = 0;                               // ring steps of the FIRST unit whose weights were requested before the wait
        if (u < total_units) {
            int n0, img, ho0, wo0, k0, k1; long long pix0;
            unit_coords(u, n0, img, ho0, wo0, pix0, k0, k1);
            if (p.b_res) {
                if (pw == 0 && elect_one()) {
                    mbar_expect_tx(&full_bar[0], (uint32_t)(9 * b_bytes));
                    tma_load_3d(ring, &map_b, &full_bar[0], 0, n0, 0);
                }
            } else {
                const int nsteps = (k1 - k0) * groups;
                npre = nsteps < kStages ? nsteps : kStages;
                for (int s = pw; s < npre; s += P)
                    if (elect_one()) {
                        mbar_expect_tx(&full_bar[s], stage_tx);
                        load_b(s, n0, k0, s);
                    }
            }
            __syncwarp();
        }
        asm volatile("griddepcontrol.wait;" ::: "memory");
        for (;;) {
            if (pw == 0) {
                const bool live = u < total_units;
                mbar_wait(&ring_empty[rslot], rphase ^ 1);
                if (lane == 0) {
                    tile_ring[rslot] = live ? u : -1;
                    mbar_arrive(&ring_full[rslot]);
                }
                __syncwarp();
                if (++rslot == kRing) { rslot = 0; rphase ^= 1; }
                if (!live) break;
            } else {
                mbar_wait(&ring_full[rslot], rphase);
                u = tile_ring[rslot];
                __syncwarp();
                if (lane == 0) mbar_arrive(&ring_empty[rslot]);
                if (++rslot == kRing) { rslot = 0; rphase ^= 1; }
                if (u < 0) break;
            }
            // next unit: latency hidden behind this unit's loads
            int next = 0;
            if (pw == 0) {
                if (lane == 0) next = atomicAdd(sched, 1);
                next = __shfl_sync(0xffffffffu, next, 0);
            }
            int n0, img, ho0, wo0, k0, k1; long long pix0;
            unit_coords(u, n0, img, ho0, wo0, pix0, k0, k1);
            if (p.im2col) {             // the run's first output pixel -> its bounding-box position (the tap offsets are added per load)
                const int hw = p.Ho * p.Wo, q = (int)pix0;
                img = q / hw;
                const int r = q - img * hw;
                ho0 = r / p.Wo;
                wo0 = r - ho0 * p.Wo;
            }
            if (p.halo) {
                // one (TH+2) x (MT*TW+2) x BK-channel input tile per K chunk (zero-filled outside the image = the padding),
                // then the nine taps' weight tiles through the B ring
                const uint32_t halo_tx = (uint32_t)((p.TW * MT + 2) * (p.TH + 2) * p.BK * 2);
                auto load_halo = [&](int kc) {              // producer 0 only
                    mbar_wait(&a_empty[hbuf], hphase ^ 1);
                    if (elect_one()) {
                        mbar_expect_tx(&a_full[hbuf], halo_tx);
                        tma_load_4d(tiles + hbuf * p.halo_bytes, &map_a, &a_full[hbuf], kc * p.BK, wo0 - 1, ho0 - 1, img);
                    }
                    __syncwarp();
                    if (++hbuf == p.halo_bufs) { hbuf = 0; hphase ^= 1; }
                };
                // the input tile of chunk kc + 1 is requested BEFORE the weight tiles of chunk kc: the producer blocks on
                // the weight ring long before the consumers are done with chunk kc, and a late halo tile stalls nine taps
                if (pw == 0) load_halo(k0);
                for (int kc = k0; kc < k1; ++kc) {
                    if (pw == 0 && kc + 1 < k1) load_halo(kc + 1);
                    if (p.b_res) continue;        // the whole weight slice (nine taps of the single K chunk) landed once, before the wait
                    for (int g = 0; g < groups; ++g, ++c) {
                        if (c % P == pw && c >= npre) {      // (the first npre steps were requested before griddepcontrol.wait)
                            mbar_wait(&empty_bar[stage], phase ^ 1);
                            if (elect_one()) {
                                mbar_expect_tx(&full_bar[stage], stage_tx);
                                load_b(stage, n0, kc, g);
                            }
                            __syncwarp();
                        }
                        if (++stage == kStages) { stage = 0; phase ^= 1; }
                    }
                }
            } else
            for (int kt = k0; kt < k1; ++kt, ++c) {
                if (c % P == pw) {
                    const int kc = kt / ntaps, tap = kt % ntaps;
                    const int kh = tap / p.KW, kw = tap % p.KW;
                    const bool pre = c < npre;         // weights (and the byte count) of this step went out before the wait
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    if (elect_one()) {
                        uint8_t* sa = ring + stage * stage_bytes;
                        if (!pre) mbar_expect_tx(&full_bar[stage], stage_tx);
                        if (p.kpair == 2) tma_load_3d(sa, &map_a, &full_bar[stage], 0, (int)pix0, 2 * kt);      // chunks 2 kt, 2 kt + 1: one {64, rows, 2} box
                        else if (p.im2col) tma_load_im2col_4d(sa, &map_a, &full_bar[stage], kc * p.BK, wo0 * p.stride - p.pad, ho0 * p.stride - p.pad, img,
                                                              (uint16_t)kw, (uint16_t)kh);
                        else if (p.flat) tma_load_2d(sa, &map_a, &full_bar[stage], kc * p.BK, (int)pix0);
                        else tma_load_4d(sa, &map_a, &full_bar[stage], kc * p.BK, wo0 * p.stride + kw - p.pad_w, ho0 * p.stride + kh - p.pad, img);
                        if (!pre) load_b(stage, n0, kt, 0);
                    }
                    __syncwarp();
                }
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            u = next;
        }
        // every CTA draws exactly one ticket past the end; the last one to do so re-arms the counters for the next launch
        if (pw == 0 && lane == 0 && atomicAdd(sched + 1, 1) == (int)gridDim.x - 1) {
            sched[0] = 0; sched[1] = 0;
            __threadfence();
        }
    } else {
        // ===== consumers.  Ping-pong: warpgroup wg owns whole 128-pixel tiles (m64 halves 0 and 1) and takes ring entries wg, wg + 2, ...
        // Cooperative: sub-tile g = warps [8 g, 8 g + 8) = two warpgroups; warpgroup half hh owns pixel rows [64 hh, 64 hh + 64) of it.
        // Each warpgroup issues its own wgmma chain into its registers and releases a ring stage (one arrival per warpgroup) once the
        // wgmmas that read it have retired: wait_group 1 after each stage's batch, so the tensor core always has the next batch queued.
        setmaxnreg_inc<consumer_regs(MT)>();
        constexpr int kHalves = kPingPong ? 2 : 1;                 // m64 halves per warpgroup
        constexpr int kGroupThreads = kPingPong ? 128 : 256;      // threads that share an epilogue (one 128-pixel sub-tile)
        const int wg = warp >> 2;
        const int slot = kPingPong ? wg : warp >> 3;              // epilogue group: staging boxes, named barrier, split-K flag
        const int g = kPingPong ? 0 : warp >> 3;                  // sub-tile
        const int hh0 = kPingPong ? 0 : wg & 1;                   // first m64 half this warpgroup computes
        const int gtid = (int)threadIdx.x - slot * kGroupThreads; // thread index inside the epilogue group
        const int bar_id = 1 + slot;
        const bool wg_leader = (threadIdx.x & 127) == 0;
        const int rw = (warp & 3) * 16 + (lane >> 2);             // this thread's first accumulator row inside an m64 half (and rw + 8)
        // shared-memory matrix descriptor = {lo: (address >> 4) | LBO 1 << 16, hi: SBO >> 4 | swizzle mode << 30 (1 = 128 B, 2 = 64 B,
        // 3 = 32 B)}: K-major rows of BK*2 bytes, 8-row groups SBO bytes apart.  The swizzle is a function of the absolute shared-memory
        // address (the TMA unit writes the tiles the same way), so a start address shifted by whole rows and an SBO of any multiple of
        // the row size address a window of a larger tile -- what the halo windows rely on.  K advances by 32 bytes per k16 step.
        const int row_bytes = p.BK * 2;
        const int halo_w = p.TW * MT + 2;
        const uint32_t layout = row_bytes == 128 ? 1u : (row_bytes == 64 ? 2u : 3u);
        const uint32_t hi_b = (uint32_t)((8 * row_bytes) >> 4) | (layout << 30);
        const uint32_t hi_a = p.halo ? ((uint32_t)((halo_w * row_bytes) >> 4) | (layout << 30)) : hi_b;
        const uint32_t ring_lo = ((smem_u32(ring) >> 4) & 0x3fffu) | (1u << 16);
        const uint32_t tiles_lo = ((smem_u32(tiles) >> 4) & 0x3fffu) | (1u << 16);
        const uint32_t stage_step = (uint32_t)stage_bytes >> 4, halo_step = (uint32_t)p.halo_bytes >> 4;
        const uint32_t b_off = (uint32_t)(MT * a_bytes) >> 4, b_step = (uint32_t)b_bytes >> 4;
        const uint32_t row_step = (uint32_t)row_bytes >> 4;        // halo windows shift by whole pixel rows of the tile
        // the first half's rows: sub-tile g (sub_off), half hh0; the second half = 8 row groups further (8 tile rows of the halo tile, or 64 rows)
        const uint32_t half_step = p.halo ? 8u * (uint32_t)halo_w * row_step : 64u * row_step;
        const uint32_t a_off = (uint32_t)(g * p.sub_off) / 16u + (uint32_t)hh0 * half_step;
        auto desc = [](uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; };
        const int ksub = p.BK / 16;                       // k16 steps per K chunk: 4, 2 or 1
        bool b_ready = false;
        int stage = 0; uint32_t phase = 0;
        int hbuf = 0; uint32_t hphase = 0;
        int rslot = 0; uint32_t rphase = 0;
        constexpr int cols_per_box = F32 ? 32 : 64;
        constexpr int nboxes = (BN + cols_per_box - 1) / cols_per_box;
        int box_seq = 0;                                  // running box counter: staging buffer = box_seq & 1 when there are two
        int entry = 0;                                    // ping-pong: ring entries seen (entry % 2 == wg: this warpgroup's tile)
        int turns = 0;                                    // ping-pong: tiles this warpgroup has run
        // ring position after n more steps of a ring of `len` slots
        auto advance = [](int& pos, uint32_t& ph, int n, int len) { const int t = pos + n; ph ^= (uint32_t)((t / len) & 1); pos = t % len; };
        float acc[kHalves][BN / 2];
        for (;;) {
            mbar_wait(&ring_full[rslot], rphase);
            const int u = tile_ring[rslot];
            __syncwarp();
            if (lane == 0) mbar_arrive(&ring_empty[rslot]);
            if (++rslot == kRing) { rslot = 0; rphase ^= 1; }
            if (u < 0) break;
            int n0, img, ho0, wo0, k0, k1; long long pix0;
            unit_coords(u, n0, img, ho0, wo0, pix0, k0, k1);
            if (kPingPong && (entry++ & 1) != wg) {
                // the other warpgroup's tile: step over its operand stages and halo buffers in the shared rings
                if (p.halo) {
                    advance(hbuf, hphase, k1 - k0, p.halo_bufs);
                    if (!p.b_res) advance(stage, phase, (k1 - k0) * (9 / p.tps), kStages);
                } else {
                    advance(stage, phase, k1 - k0, kStages);
                }
                continue;
            }
            // ping-pong hand-off: warpgroup 0's tile j waits until warpgroup 1 has issued the MMAs of its tile j - 1, warpgroup 1's
            // tile j until warpgroup 0 has issued those of its tile j -- the MMA loops alternate, each epilogue runs under the other's MMAs
            if (kPingPong && (wg == 1 || turns > 0)) mbar_wait(&mma_turn[wg], (uint32_t)((wg == 0 ? turns - 1 : turns) & 1));
            // ring stage / halo buffer read by the most recent committed batch: released once a later wait_group shows it retired
            int pend_stage = -1, pend_halo = -1;
            auto release = [&](int st, int hb) {
                if (wg_leader) {
                    if (st >= 0) mbar_arrive(&empty_bar[st]);
                    if (hb >= 0) mbar_arrive(&a_empty[hb]);
                }
            };
            // after committing a batch that read (st, hb): keep it in flight behind the next one, or -- when the producer cannot deliver the
            // next batch's operands before these are back (a one-stage ring; the halo tile, whose successor's buffer is requested ahead of
            // the next chunk's weights) -- wait for everything and release at once
            auto retire = [&](int st, int hb, bool drain) {
                if (drain) {
                    wgmma_wait<0>();
                    acc_fence(acc);
                    release(pend_stage, pend_halo);
                    release(st, hb);
                    pend_stage = pend_halo = -1;
                } else {
                    wgmma_wait<1>();
                    acc_fence(acc);
                    release(pend_stage, pend_halo);
                    pend_stage = st; pend_halo = hb;
                }
            };
            uint32_t scale = 0;                             // the unit's first wgmma overwrites the accumulator
            // one K chunk = BK / 16 k16 steps x the warpgroup's m64 halves.  The step count is made a compile-time constant so the chunk is
            // ONE straight-line wgmma chain: in a runtime-count loop ptxas ends a wgmma group and injects a warpgroup.arrive every step.
            auto chain = [&](auto ksteps, uint32_t a_lo, uint32_t b_lo) {
#pragma unroll
                for (int k = 0; k < decltype(ksteps)::value; ++k) {
#pragma unroll
                    for (int h = 0; h < kHalves; ++h)
                        wgmma_m64k16<BN, F16>(acc[h], desc(a_lo + (uint32_t)h * half_step + 2u * k, hi_a), desc(b_lo + 2u * k, hi_b), scale);
                    scale = 1;
                }
            };
            auto mma_chunk = [&](uint32_t a_lo, uint32_t b_lo) {
                if (ksub == 4) chain(Steps<4>{}, a_lo, b_lo);
                else if (ksub == 2) chain(Steps<2>{}, a_lo, b_lo);
                else chain(Steps<1>{}, a_lo, b_lo);
            };
            if (p.halo) {
                for (int kc = k0; kc < k1; ++kc) {
                    mbar_wait(&a_full[hbuf], hphase);
                    const uint32_t a_buf = tiles_lo + (uint32_t)hbuf * halo_step + a_off;
                    for (int tap0 = 0; tap0 < 9; tap0 += p.tps) {
                        if (!p.b_res || !b_ready) {
                            mbar_wait(&full_bar[stage], phase);
                            b_ready = true;
                        }
                        const uint32_t b_stage = ring_lo + (uint32_t)stage * stage_step;
                        acc_fence(acc);
                        wgmma_fence();
                        for (int t = 0; t < p.tps; ++t) {
                            // A window of tap (kh, kw): the halo tile shifted by kh rows and kw pixels; the 8-row groups are the
                            // tile rows, strided by the halo row pitch
                            const int tap = tap0 + t, kh = tap / 3, kw = tap - 3 * kh;
                            const uint32_t a_lo = a_buf + (uint32_t)(kh * halo_w + kw) * row_step;
                            const uint32_t b_lo = b_stage + (uint32_t)t * b_step;
                            mma_chunk(a_lo, b_lo);
                        }
                        wgmma_commit();
                        const bool chunk_end = tap0 + p.tps >= 9;
                        retire(p.b_res ? -1 : stage, chunk_end ? hbuf : -1, chunk_end || kStages == 1);
                        if (!p.b_res && ++stage == kStages) { stage = 0; phase ^= 1; }
                    }
                    if (++hbuf == p.halo_bufs) { hbuf = 0; hphase ^= 1; }
                }
            } else
            for (int kt = k0; kt < k1; ++kt) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t a_st = ring_lo + (uint32_t)stage * stage_step;
                const uint32_t b_st = a_st + b_off * (uint32_t)p.kpair;
                acc_fence(acc);
                wgmma_fence();
                for (int j = 0; j < p.kpair; ++j) {       // K chunks of this stage: [chunk][sub-tile][128 rows] | [chunk][BN rows]
                    const uint32_t a_lo = a_st + (uint32_t)j * b_off + a_off, b_lo = b_st + (uint32_t)j * b_step;
                    mma_chunk(a_lo, b_lo);
                }
                wgmma_commit();
                retire(stage, -1, kStages == 1);
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            if (kPingPong) {                                // every MMA of this tile is issued: the other warpgroup's turn
                if (wg_leader) mbar_arrive(&mma_turn[wg ^ 1]);
                ++turns;
            }
            wgmma_wait<0>();
            acc_fence(acc);
            release(pend_stage, pend_halo);
            // this group's output window
            const long long gpix = pix0 + (long long)g * kTileM;
            const int gho = p.halo ? ho0 : ho0 + g * p.TH;
            const int gwo = p.halo ? wo0 + g * p.TW : wo0;
            const bool in_range = p.flat ? (gpix < p.total_pix) : (gho < p.Ho && gwo < p.Wo);
            bool reduce_here = true;
            if (p.splits > 1) {
                // ---- split-K: park the fp32 partial sums, count arrivals; the LAST split of a tile to arrive sums all of them in
                // split order (a fixed order: results do not depend on which CTA is last) and runs the normal epilogue
                const int cq = 2 * (lane & 3);
                float* wsub = p.ws + ((size_t)u * MT + g) * kTileM * BN;
#pragma unroll
                for (int hf = 0; hf < kHalves; ++hf) {
                    const int r0 = (hh0 + hf) * 64 + rw;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            __stcg(reinterpret_cast<float2*>(wsub + (size_t)(r0 + 8 * h) * BN + 8 * j + cq), make_float2(acc[hf][4 * j + 2 * h], acc[hf][4 * j + 2 * h + 1]));
                }
                __threadfence();
                asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "n"(kGroupThreads) : "memory");
                if (gtid == 0) {
                    const int t = u / p.splits;
                    const int old = atomicAdd(p.flags + t * MT + g, 1);
                    const int last = old == p.splits - 1;
                    if (last) p.flags[t * MT + g] = 0;              // re-armed for the next launch
                    last_flag[slot] = last;
                }
                asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "n"(kGroupThreads) : "memory");
                reduce_here = last_flag[slot] != 0;
                if (reduce_here) {
                    __threadfence();
                    const int t = u / p.splits;
#pragma unroll
                    for (int hf = 0; hf < kHalves; ++hf)
#pragma unroll
                        for (int i = 0; i < BN / 2; ++i) acc[hf][i] = 0.f;
                    for (int sp = 0; sp < p.splits; ++sp) {
                        const float* src = p.ws + (((size_t)t * p.splits + sp) * MT + g) * kTileM * BN;
#pragma unroll
                        for (int hf = 0; hf < kHalves; ++hf) {
                            const int r0 = (hh0 + hf) * 64 + rw;
#pragma unroll
                            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                                for (int h = 0; h < 2; ++h) {
                                    const float2 x = __ldcg(reinterpret_cast<const float2*>(src + (size_t)(r0 + 8 * h) * BN + 8 * j + cq));
                                    acc[hf][4 * j + 2 * h] += x.x; acc[hf][4 * j + 2 * h + 1] += x.y;
                                }
                        }
                    }
                }
            }
            // ---- one staging box (128 pixels x 128 B = 64 halves / 32 floats of channels) at a time: registers -> + bias ->
            // activation -> 16-bit -> swizzled shared memory -> TMA store, the store of box b overlapping the math of box b + 1
            if (reduce_here) {
                const float* bias_t = bias + n0;
#pragma unroll
                for (int bx = 0; bx < nboxes; ++bx, ++box_seq) {
                    uint8_t* stage_cur = stage_out + slot * staging_bytes + (p.out_bufs == 2 ? (box_seq & 1) * box_bytes : 0);
                    // the store that used this buffer (out_bufs boxes ago) must have finished READING it
                    if (gtid == 0) {
                        if (p.out_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    }
                    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "n"(kGroupThreads) : "memory");
                    if (in_range) {
#pragma unroll
                        for (int hf = 0; hf < kHalves; ++hf)
                            stage_box<F32, F16, BN>(acc[hf], bx, bias_t, stage_cur, (hh0 + hf) * 64 + rw, lane, p.act, p.act_floor, p.act_slope);
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy writes -> visible to the TMA unit
                    asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "n"(kGroupThreads) : "memory");   // the warps of this sub-tile
                    if (gtid == 0) {
                        const int cc = n0 + bx * cols_per_box;
                        if (in_range && cc < p.Cout) {
                            if (p.flat) tma_store_2d(&map_c, stage_cur, cc, (int)gpix);
                            else tma_store_4d(&map_c, stage_cur, cc, gwo, gho, img);
                        }
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");   // (possibly empty: keeps the wait_group arithmetic uniform)
                    }
                }
            }
        }
        // the staging boxes must outlive the stores' READS of them; the writes themselves are flushed by grid completion like any store
        if (gtid == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
}

// ------------------------------------------------------------------------------------------ host side
thread_local std::string g_conv_err;
int cfail(int code, const std::string& m) { g_conv_err = m; return code; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeIm2colFn get_encode_im2col() {
    static EncodeIm2colFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeIm2colFn>(p);
    }
    return fn;
}
CUtensorMapSwizzle swizzle_for(int bk) {
    return bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

}  // namespace

typedef void (*ConvKernelFn)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const float*, int*, const ConvParams);

struct b2t_conv_plan {
    ConvKernelFn kernel;           // the instantiation for (fp32 output, fp16, mt, BLOCK_N)
    CUtensorMap map_a, map_b, map_c;
    ConvParams p;
    float* bias_pad;               // plan-owned copy of the bias, zero-padded to whole 32-column epilogue blocks
    double flops;                  // algorithmic 2*pix*Cout*kh*kw*Cin of the layer as described by the caller
    int* sched;                    // [4][2] work-unit ticket counter, finished-CTA counter: self-resetting, four sets used in rotation by successive launches
    mutable unsigned launches;     // (programmatic dependent launch lets launch k + 1 of a plan draw tickets while launch k is still running)
    float* ws;                     // split-K partial sums (splits > 1)
    int* flags;                    // split-K arrival counters
    void* out;
    dim3 grid;
    int threads;
    size_t smem;
};

template <bool F32, bool F16>
ConvKernelFn kernel_for_bn(int mt, int bn) {
    if (mt == 1) {
        switch (bn) {
            case 32: return conv_bias_act_kernel<F32, F16, 1, 32>;
            case 64: return conv_bias_act_kernel<F32, F16, 1, 64>;
            case 128: return conv_bias_act_kernel<F32, F16, 1, 128>;
            case 256: return conv_bias_act_kernel<F32, F16, 1, 256>;
        }
    } else if (mt == 2) {           // four consumer warpgroups: BLOCK_N <= 128 keeps the accumulators within the register budget
        switch (bn) {
            case 32: return conv_bias_act_kernel<F32, F16, 2, 32>;
            case 64: return conv_bias_act_kernel<F32, F16, 2, 64>;
            case 128: return conv_bias_act_kernel<F32, F16, 2, 128>;
        }
    }
    return nullptr;
}
// nullptr: no instantiation for this (mt, BLOCK_N)
ConvKernelFn kernel_for(int f32, int f16, int mt, int bn) {
    if (f16) return f32 ? kernel_for_bn<true, true>(mt, bn) : kernel_for_bn<false, true>(mt, bn);
    return f32 ? kernel_for_bn<true, false>(mt, bn) : kernel_for_bn<false, false>(mt, bn);
}

extern "C" const char* b2t_conv_last_error(void) { return g_conv_err.c_str(); }

static void free_plan(b2t_conv_plan* pl) {
    if (!pl) return;
    if (pl->bias_pad) cudaFree(pl->bias_pad);
    if (pl->sched) cudaFree(pl->sched);
    if (pl->ws) cudaFree(pl->ws);
    if (pl->flags) cudaFree(pl->flags);
    delete pl;
}

extern "C" int b2t_conv_plan_create(const b2t_conv_desc* d, b2t_conv_plan** out_plan) {
    if (!d || !out_plan) return cfail(B2T_EINVAL, "b2t_conv_plan_create: null argument");
    if (d->io_dtype != B2T_ACT_BF16 && d->io_dtype != B2T_ACT_F16) return cfail(B2T_EINVAL, "b2t_conv_plan_create: io_dtype must be B2T_ACT_BF16 or B2T_ACT_F16");
    if (!(d->kh == d->kw && (d->kh == 1 || d->kh == 3)) || !(d->stride == 1 || d->stride == 2))
        return cfail(B2T_EINVAL, "b2t_conv_plan_create: only k in {1,3}, stride in {1,2}");
    const bool rowpack = d->rowpack != 0;
    if (rowpack && !(d->kh == 3 && d->stride == 1 && d->cin == 16 && d->in_row_pixels >= d->w + 3 && d->in_coff == 0 && d->in_pitch == 16))
        return cfail(B2T_EINVAL, "b2t_conv_plan_create: rowpack needs k=3, stride 1, cin = in_pitch = 16, in_coff 0, in_row_pixels >= w + 3");
    int bk = d->cin % 64 == 0 ? 64 : (d->cin % 32 == 0 ? 32 : (d->cin % 16 == 0 ? 16 : 0));
    if (!bk) return cfail(B2T_EINVAL, "b2t_conv_plan_create: Cin must be a multiple of 16");
    if (d->in_pitch % 8 || d->in_coff % 8 || d->out_coff % 8)
        return cfail(B2T_EINVAL, "b2t_conv_plan_create: pitches / offsets must keep 16-byte alignment");
    if (d->halo != 0 && d->halo != 1) return cfail(B2T_EINVAL, "b2t_conv_plan_create: halo must be 0 or 1 (the resident-weight variant of round 1 was removed: never faster)");
    const bool halo = d->halo == 1;
    if (halo && !(d->kh == 3 && d->stride == 1 && (d->cin % 64 == 0 || d->cin == 32 || d->cin == 16) && !rowpack))
        return cfail(B2T_EINVAL, "b2t_conv_plan_create: halo mode needs k=3, stride 1, cin = 16, 32 or a multiple of 64");
    const int MT = d->mt > 0 ? d->mt : 1;
    if (MT != 1 && MT != 2) return cfail(B2T_EINVAL, "b2t_conv_plan_create: mt must be 1 or 2");
    const int splits = d->splits > 0 ? d->splits : 1;
    const int P = d->producers > 0 ? d->producers : 2;
    if (P > kMaxProducers) return cfail(B2T_EINVAL, "b2t_conv_plan_create: at most 2 producer warps");
    const int row_pixels = d->in_row_pixels > 0 ? d->in_row_pixels : d->w;
    if (row_pixels < d->w) return cfail(B2T_EINVAL, "b2t_conv_plan_create: in_row_pixels < w");
    if (row_pixels != d->w && d->kh == 1 && d->stride == 1) return cfail(B2T_EINVAL, "b2t_conv_plan_create: padded rows are not supported for 1x1 layers");
    // pixel runs (tile_w = 128): 3x3 layers reading an unpadded NHWC map; 1x1 / stride 1 layers are flat already.  Every other
    // im2col limit holds for these geometries (4-D bounding-box corners -1 .. -1 within [-128, 127], 128 * mt <= 1024 pixels per
    // box, traversal stride <= 8, BK * 2 bytes <= the swizzle span).
    const bool runs = d->tile_w == 128;
    if (runs && !(d->kh == 3 && !halo && !rowpack && row_pixels == d->w))
        return cfail(B2T_EINVAL, "b2t_conv_plan_create: pixel runs (tile_w = 128) need a 3x3 layer without halo, row packing or padded input rows");
    EncodeTiledFn enc = get_encode();
    if (!enc) return cfail(B2T_ECUDA, "cuTensorMapEncodeTiled is not available from the driver");
    EncodeIm2colFn enc_im2col = runs ? get_encode_im2col() : nullptr;
    if (runs && !enc_im2col) return cfail(B2T_ECUDA, "cuTensorMapEncodeIm2col is not available from the driver");
    b2t_conv_plan* pl = new b2t_conv_plan();
    pl->kernel = nullptr; pl->bias_pad = nullptr; pl->sched = nullptr; pl->launches = 0; pl->ws = nullptr; pl->flags = nullptr; pl->out = d->y;
    ConvParams& p = pl->p;
    p.N = d->n; p.H = d->h; p.W = d->w; p.Cin = d->cin; p.Cout = d->cout;
    p.KH = d->kh; p.KW = d->kw; p.stride = d->stride; p.pad = d->kh / 2; p.pad_w = p.pad;
    p.Ho = (d->h + 2 * p.pad - d->kh) / d->stride + 1;
    p.Wo = (d->w + 2 * p.pad - d->kw) / d->stride + 1;
    pl->flops = 2.0 * (double)p.N * p.Ho * p.Wo * p.Cout * p.KH * p.KW * p.Cin;
    if (rowpack) {      // the kernel sees a 3x1 convolution over 64 "channels" = 4 consecutive pixels x 16
        p.KW = 1; p.Cin = 64; p.pad_w = 0; bk = 64;
    }
    p.BK = bk; p.MT = MT; p.splits = splits; p.P = P;
    const int cout_pad = (d->cout + 15) / 16 * 16;
    // default tile shape when the caller does not choose (DetectorW6 autotunes per layer)
    int bn = cout_pad;
    if (bn > 64) bn = (cout_pad % 128 == 0) ? 128 : 64;
    if (d->block_n > 0) bn = d->block_n;
    if (bn % 16 || bn > 256 || bn < 16) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: bad BLOCK_N"); }
    // the kernel is instantiated for BLOCK_N = 32, 64, 128 and 256 (the wgmma N and the accumulator registers are compile-time):
    // other widths round up, the extra weight rows are zero-filled by the TMA unit and the extra channels clipped on store
    { int b = 32; while (b < bn) b <<= 1; bn = b; }
    // a store box is 128 bytes of channels (64 halves / 32 floats): N tiles other than the last must be whole boxes,
    // otherwise a tile's last box would spill into its neighbour's channels (the LAST tile is clipped by the map)
    if (bn < cout_pad && bn % (d->out_f32 ? 32 : 64)) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: BLOCK_N must be a multiple of 64 (16-bit) / 32 (fp32) when the layer has several N tiles"); }
    p.BN = bn;
    if (MT * bn > 256) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: mt x BLOCK_N > 256: the accumulators of four consumer warpgroups exceed the register file"); }
    p.out_pitch = d->out_pitch; p.out_coff = d->out_coff; p.act = d->act == 1 ? 1 : 0; p.act_floor = d->act == 2 ? 0.0f : -INFINITY; p.act_slope = d->act == 3 ? 0.1f : 1.0f; p.out_f32 = d->out_f32; p.f16 = d->io_dtype == B2T_ACT_F16 ? 1 : 0;
    p.flat = (d->kh == 1 && d->stride == 1) || runs ? 1 : 0;
    p.im2col = runs ? 1 : 0;
    p.total_pix = (long long)p.N * p.Ho * p.Wo;
    p.halo = halo ? 1 : 0; p.halo_bytes = 0; p.halo_bufs = 0;
    if (p.flat) { p.TH = 1; p.TW = 128; p.tiles_w = p.tiles_h = 0; }
    else {
        int tw = 16;
        if (p.Wo % 16 != 0) { tw = (p.Wo % 8 == 0) ? 8 : 4; }
        if (d->tile_w > 0) tw = d->tile_w;
        if (halo) tw = 8;          // an 8-row MMA group = one tile row of 8 pixels, groups strided by the halo row pitch
        if (tw != 4 && tw != 8 && tw != 16) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: tile_w must be 4, 8 or 16"); }
        p.TW = tw; p.TH = 128 / tw;
        // a tile = MT sub-tiles: side by side in halo mode (TH rows x MT*TW pixels), stacked otherwise (MT*TH rows x TW pixels)
        const int tile_w_px = halo ? p.TW * MT : p.TW, tile_h_px = halo ? p.TH : p.TH * MT;
        if (tile_h_px * p.stride > 256) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: mt = 2 needs tile_w >= 8 for stride-2 layers (TMA box rows <= 256)"); }
        p.tiles_w = (p.Wo + tile_w_px - 1) / tile_w_px; p.tiles_h = (p.Ho + tile_h_px - 1) / tile_h_px;
    }
    // flat mode: two K chunks per ring stage when the layer has an even number of 64-channel chunks (bigger TMA boxes: a box
    // costs about the same whatever its size up to tens of KB, so small activation boxes alone cap the fill rate)
    p.kpair = (p.flat && !runs && bk == 64 && (p.Cin / bk) % 2 == 0 && d->kpair != 1) ? 2 : 1;
    if (d->kpair == 2 && p.kpair != 2) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: kpair = 2 needs a 1x1 / stride 1 layer with an even number of 64-channel chunks"); }
    p.sub_off = halo ? p.TW * bk * 2 : kTileM * bk * 2;
    p.ksteps = halo ? p.Cin / bk : p.KH * p.KW * (p.Cin / bk) / p.kpair;
    if (splits > p.ksteps) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: more K splits than K steps"); }
    // ---- tensor maps
    const CUtensorMapSwizzle sw = swizzle_for(bk);
    const CUtensorMapDataType dt16 = p.f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    char* a_base = reinterpret_cast<char*>(const_cast<void*>(d->x)) + (size_t)d->in_coff * 2;
    CUresult r;
    if (runs) {
        // bounding box of the output pixels in input coordinates: corner -pad, positions -pad + s j, Ho x Wo of them per image
        cuuint64_t dims[4] = {(cuuint64_t)p.Cin, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
        cuuint64_t strides[3] = {(cuuint64_t)d->in_pitch * 2, (cuuint64_t)d->in_pitch * 2 * p.W, (cuuint64_t)d->in_pitch * 2 * p.W * p.H};
        const int lower[2] = {-p.pad, -p.pad}, upper[2] = {p.pad - (p.KH - 1), p.pad - (p.KW - 1)};
        cuuint32_t es[4] = {1, (cuuint32_t)p.stride, (cuuint32_t)p.stride, 1};
        r = enc_im2col(&pl->map_a, dt16, 4, a_base, dims, strides, lower, upper, (cuuint32_t)bk, (cuuint32_t)(kTileM * MT), es,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else if (p.flat && p.kpair == 2) {
        // (channel within a chunk, pixel, chunk): lands as [chunk][pixel][64]
        cuuint64_t dims[3] = {64, (cuuint64_t)p.total_pix, (cuuint64_t)(p.Cin / 64)};
        cuuint64_t strides[2] = {(cuuint64_t)d->in_pitch * 2, 128};
        cuuint32_t box[3] = {64, (cuuint32_t)(kTileM * MT), 2};
        cuuint32_t es[3] = {1, 1, 1};
        r = enc(&pl->map_a, dt16, 3, a_base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else if (p.flat) {
        cuuint64_t dims[2] = {(cuuint64_t)p.Cin, (cuuint64_t)p.total_pix};
        cuuint64_t strides[1] = {(cuuint64_t)d->in_pitch * 2};
        cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)(kTileM * MT)};
        cuuint32_t es[2] = {1, 1};
        r = enc(&pl->map_a, dt16, 2, a_base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
        // row-packed: dim 0 spans 4 pixels (64 elements) while dim 1 still advances by ONE pixel -- overlapping boxes
        cuuint64_t dims[4] = {(cuuint64_t)p.Cin, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
        cuuint64_t strides[3] = {(cuuint64_t)d->in_pitch * 2, (cuuint64_t)d->in_pitch * 2 * row_pixels, (cuuint64_t)d->in_pitch * 2 * row_pixels * p.H};
        // with element strides the box extent is given in INPUT elements: TW outputs at stride s span TW*s inputs
        cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)(p.TW * p.stride), (cuuint32_t)(p.TH * MT * p.stride), 1};
        if (halo) { box[1] = (cuuint32_t)(p.TW * MT + 2); box[2] = (cuuint32_t)(p.TH + 2); }
        cuuint32_t es[4] = {1, (cuuint32_t)p.stride, (cuuint32_t)p.stride, 1};
        r = enc(&pl->map_a, dt16, 4, a_base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) { free_plan(pl); return cfail(B2T_ECUDA, std::string(runs ? "cuTensorMapEncodeIm2col" : "cuTensorMapEncodeTiled") + "(A) failed: " + std::to_string((int)r)); }
    // halo mode: how many filter taps travel in one weight box.  A bulk-tensor copy costs about the same whatever its size up to
    // tens of KB, so a kernel row of three taps per box fills the ring faster than one tap per box.
    const int kchunks_h = p.Cin / bk;
    const int tiles_n_pre = (cout_pad + bn - 1) / bn;
    int tps = 1;
    p.b_res = 0;
    if (halo) {
        tps = d->tps > 0 ? d->tps : (bn <= 128 ? 3 : 1);
        if (tps != 1 && tps != 3 && tps != 9) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: tps must be 1, 3 or 9"); }
        if ((d->tps == 0 || d->tps == 9) && kchunks_h == 1 && tiles_n_pre == 1 && splits == 1 && 9 * bn * bk * 2 <= 96 * 1024) { tps = 9; p.b_res = 1; }
        else if (tps == 9) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: tps = 9 (resident weights) needs one K chunk, one N tile and <= 96 KB of weights"); }
    }
    p.tps = tps;
    {
        const cuuint64_t K = (cuuint64_t)p.KH * p.KW * p.Cin;
        if (p.kpair == 2) {
            cuuint64_t dims[3] = {64, (cuuint64_t)d->cout_rows, (cuuint64_t)(p.Cin / 64)};
            cuuint64_t strides[2] = {K * 2, 128};
            cuuint32_t box[3] = {64, (cuuint32_t)bn, 2};
            cuuint32_t es[3] = {1, 1, 1};
            r = enc(&pl->map_b, dt16, 3, const_cast<void*>(d->w_packed), dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        } else if (tps > 1) {
            // (channel within the chunk, output row, tap): tap t of row n, chunk kc sits (t * Cin + kc * 64) elements into the row
            cuuint64_t dims[3] = {(cuuint64_t)p.Cin, (cuuint64_t)d->cout_rows, 9};
            cuuint64_t strides[2] = {K * 2, (cuuint64_t)p.Cin * 2};
            cuuint32_t box[3] = {(cuuint32_t)bk, (cuuint32_t)bn, (cuuint32_t)tps};
            cuuint32_t es[3] = {1, 1, 1};
            r = enc(&pl->map_b, dt16, 3, const_cast<void*>(d->w_packed), dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        } else {
            cuuint64_t dims[2] = {K, (cuuint64_t)d->cout_rows};
            cuuint64_t strides[1] = {K * 2};
            cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)bn};
            cuuint32_t es[2] = {1, 1};
            r = enc(&pl->map_b, dt16, 2, const_cast<void*>(d->w_packed), dims, strides, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        }
        if (r != CUDA_SUCCESS) { free_plan(pl); return cfail(B2T_ECUDA, "cuTensorMapEncodeTiled(B) failed: " + std::to_string((int)r)); }
    }
    {   // output map: dim0 = the layer's REAL channel count (TMA clips the padded tail), base = y + out_coff; one box = one sub-tile
        const int esize = p.out_f32 ? 4 : 2;
        const CUtensorMapDataType dt = p.out_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : dt16;
        char* c_base = reinterpret_cast<char*>(d->y) + (size_t)d->out_coff * esize;
        const cuuint32_t cb = 128 / esize;
        if (((uintptr_t)c_base & 15) || ((size_t)d->out_pitch * esize) % 16) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: output slice must be 16-byte aligned"); }
        if (p.flat) {
            cuuint64_t dims[2] = {(cuuint64_t)p.Cout, (cuuint64_t)p.total_pix};
            cuuint64_t strides[1] = {(cuuint64_t)d->out_pitch * esize};
            cuuint32_t box[2] = {cb, (cuuint32_t)kTileM};
            cuuint32_t es[2] = {1, 1};
            r = enc(&pl->map_c, dt, 2, c_base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        } else {
            cuuint64_t dims[4] = {(cuuint64_t)p.Cout, (cuuint64_t)p.Wo, (cuuint64_t)p.Ho, (cuuint64_t)p.N};
            cuuint64_t strides[3] = {(cuuint64_t)d->out_pitch * esize, (cuuint64_t)d->out_pitch * esize * p.Wo, (cuuint64_t)d->out_pitch * esize * p.Wo * p.Ho};
            cuuint32_t box[4] = {cb, (cuuint32_t)p.TW, (cuuint32_t)p.TH, 1};
            cuuint32_t es[4] = {1, 1, 1, 1};
            r = enc(&pl->map_c, dt, 4, c_base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        }
        if (r != CUDA_SUCCESS) { free_plan(pl); return cfail(B2T_ECUDA, "cuTensorMapEncodeTiled(C) failed: " + std::to_string((int)r)); }
    }
    // ---- shared memory: [halo buffers] [ring of stages] [one staging tile per sub-tile] [barriers]
    const int a_bytes = kTileM * bk * 2, b_bytes = bn * bk * 2;
    const int stage_bytes = (((halo ? tps * b_bytes : (MT * a_bytes + b_bytes) * p.kpair) + 1023) / 1024) * 1024;
    if (halo) { p.halo_bytes = ((p.TW * MT + 2) * (p.TH + 2) * bk * 2 + 1023) / 1024 * 1024; p.halo_bufs = 2; }
    const int box_bytes = kTileM * 128;                  // one staging box: 128 pixels x 64 halves / 32 floats
    p.out_bufs = d->out_bufs == 1 ? 1 : 2;
    const int slots = ping_pong(MT, bn) ? 2 : MT;        // epilogue groups with their own staging boxes: warpgroups (ping-pong) or sub-tiles
    auto smem_for = [&](int st) { return (size_t)p.halo_bufs * p.halo_bytes + (size_t)st * stage_bytes + (size_t)slots * p.out_bufs * box_bytes + 512 + 1024; };
    ConvKernelFn kfn = kernel_for(p.out_f32, p.f16, MT, bn);
    if (!kfn) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: no kernel for this mt / BLOCK_N"); }
    // the opt-in for > 48 KB of dynamic shared memory is per device and per kernel instantiation
    if (cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess) {
        free_plan(pl); return cfail(B2T_ECUDA, "cannot raise dynamic shared memory for conv kernel");
    }
    // Ring depth: what bounds a CTA is the data it keeps in flight, so by default the ring takes the shared memory that is left, up to
    // kMaxStages.  The register hand-off sizes every instantiation for one CTA per SM (its launch allocation is the whole register file).
    const int threads = conv_threads(MT);                // consumer warpgroups + the producer warpgroup, whatever P is
    int stages = d->stages > 0 ? (d->stages < kMaxStages ? d->stages : kMaxStages) : 0;
    if (p.b_res) stages = 1;
    const int min_stages = (halo || p.kpair == 2) ? 2 : 3;
    if (stages == 0) {
        for (int pass = 0; pass < 2 && stages == 0; ++pass) {
            int pick = 0;
            for (int st = kMaxStages; st >= 1 && !pick; --st) if (smem_for(st) <= 226 * 1024) pick = st;
            if (pick >= min_stages || p.out_bufs == 1 || d->out_bufs == 2) stages = pick;
            else p.out_bufs = 1;                          // a second staging box is worth less than a ring stage
        }
        if (stages < 1) stages = 1;
    }
    while (stages > 1 && smem_for(stages) > 226 * 1024) --stages;
    if (smem_for(stages) > 226 * 1024 && p.out_bufs == 2) p.out_bufs = 1;
    if (smem_for(stages) > 227 * 1024) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: tile does not fit in shared memory (reduce BLOCK_N, mt or tps)"); }
    if (halo && d->halo_bufs == 3 && smem_for(stages) + p.halo_bytes <= 226 * 1024) p.halo_bufs = 3;
    // a producer that skips the other producer's steps only checks the PARITY of its stage's barrier: with fewer stages than
    // producers it could run two phases ahead of a stage and alias it -- never more producers than stages
    const int P_eff = P > stages ? stages : P;
    p.P = P_eff;
    p.stages = stages;
    pl->smem = smem_for(stages);
    pl->threads = threads;
    int ctas_per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, kfn, threads, pl->smem) != cudaSuccess || ctas_per_sm < 1) ctas_per_sm = 1;
    p.tiles_m = p.flat ? (int)((p.total_pix + kTileM * MT - 1) / (kTileM * MT)) : p.N * p.tiles_w * p.tiles_h;
    p.tiles_n = (cout_pad + bn - 1) / bn;
    int n_sm = 132;
    { int devid = 0; cudaGetDevice(&devid); int v = 0; if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, devid) == cudaSuccess && v > 0) n_sm = v; }
    const long long total_units = (long long)p.tiles_m * p.tiles_n * splits;
    if (total_units > 0x7fffffff) { free_plan(pl); return cfail(B2T_EINVAL, "b2t_conv_plan_create: too many tiles"); }
    long long g = (long long)n_sm * ctas_per_sm;
    if (g > total_units) g = total_units;
    pl->grid = dim3((unsigned)g, 1, 1);
    pl->kernel = kfn;
    {   // the epilogue reads the bias in pairs without bounds checks: snapshot it into a zero-padded array
        const size_t nb = (size_t)p.tiles_n * bn + 64;
        if (cudaMalloc(&pl->bias_pad, nb * sizeof(float)) != cudaSuccess) { free_plan(pl); return cfail(B2T_ECUDA, "cudaMalloc(bias) failed"); }
        if (cudaMemset(pl->bias_pad, 0, nb * sizeof(float)) != cudaSuccess ||
            cudaMemcpy(pl->bias_pad, d->bias, (size_t)d->cout * sizeof(float), cudaMemcpyDeviceToDevice) != cudaSuccess) {
            free_plan(pl); return cfail(B2T_ECUDA, "bias snapshot failed");
        }
        if (cudaMalloc(&pl->sched, 8 * sizeof(int)) != cudaSuccess || cudaMemset(pl->sched, 0, 8 * sizeof(int)) != cudaSuccess) {
            free_plan(pl); return cfail(B2T_ECUDA, "cudaMalloc(tile counters) failed");
        }
    }
    if (splits > 1) {
        const size_t wsb = (size_t)total_units * MT * kTileM * bn * sizeof(float);
        const size_t nf = (size_t)p.tiles_m * p.tiles_n * MT * sizeof(int);
        if (cudaMalloc(&pl->ws, wsb) != cudaSuccess || cudaMalloc(&pl->flags, nf) != cudaSuccess || cudaMemset(pl->flags, 0, nf) != cudaSuccess) {
            free_plan(pl); return cfail(B2T_ECUDA, "cudaMalloc(split-K workspace) failed");
        }
    }
    p.ws = pl->ws; p.flags = pl->flags;
    *out_plan = pl;
    return B2T_OK;
}

extern "C" void b2t_conv_plan_destroy(b2t_conv_plan* pl) { free_plan(pl); }

extern "C" double b2t_conv_plan_flops(const b2t_conv_plan* pl) { return pl ? pl->flops : 0.0; }

extern "C" int b2t_conv_plan_info(const b2t_conv_plan* pl, int* out, int n) {
    if (!pl || !out) return cfail(B2T_EINVAL, "b2t_conv_plan_info: null argument");
    const ConvParams& p = pl->p;
    const int v[18] = {(int)pl->grid.x, pl->threads, (int)pl->smem, p.BN, p.stages, p.MT, p.splits, p.halo, p.halo_bufs, p.tiles_m, p.tiles_n,
                       p.BN / 2 * (ping_pong(p.MT, p.BN) ? 2 : 1), p.P, p.tps, p.b_res, p.out_bufs, p.kpair, ping_pong(p.MT, p.BN) ? 1 : 0};
    for (int i = 0; i < n && i < 18; ++i) out[i] = v[i];
    return B2T_OK;
}

extern "C" int b2t_conv_run(const b2t_conv_plan* pl, void* stream) {
    if (!pl) return cfail(B2T_EINVAL, "b2t_conv_run: null plan");
    static const bool use_pdl = [] { const char* v = getenv("B2T_CONV_PDL"); return !(v && v[0] == '0'); }();
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = pl->grid; cfg.blockDim = dim3(pl->threads); cfg.dynamicSmemBytes = pl->smem; cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = use_pdl ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, pl->kernel, pl->map_a, pl->map_b, pl->map_c, (const float*)pl->bias_pad,
                                       pl->sched + 2 * (pl->launches++ & 3u), pl->p);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return cfail(B2T_ECUDA, std::string("conv launch: ") + cudaGetErrorString(e));
    return B2T_OK;
}
