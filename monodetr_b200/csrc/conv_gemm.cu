// conv_gemm.cu -- wgmma / TMA implicit-GEMM kernel family for sm_90a (fp32 storage, error-compensated BF16x3 or
// TF32 tensor-core math, fp32 accumulate in registers).  One kernel template serves
//   * linear layers and 1x1 convolutions (a GEMM is a 1-tap convolution over a 1-row image),
//   * KxK convolutions, im2col-free: for every filter tap the TMA engine fetches the SHIFTED
//     NHWC activation box (out-of-bounds = zero fill = padding; element strides = conv stride),
//   * their data gradients (same kernel, B operand read MN-major straight from the packed weights),
//   * their weight gradients (both operands MN-major straight from dY / X, split-K with vector reds).
// It replaces the cuDNN / cuBLAS calls behind nn.Conv2d / nn.Linear on the reference path
// (lib/models/monodetr/backbone.py:100-102 torchvision ResNet-50 convs; monodetr.py:83-91 input_proj;
// depth_predictor/depth_predictor.py:29-47; ops/modules/ms_deform_attn.py:138-161 projections;
// depthaware_transformer.py:339-343,467-473 FFN / decoder linears).
//
// Layouts: activations NHWC fp32 [B][H][W][C]; packed weights [tap][Cout][Cin]; output NHWC.
// Tile: 128 output pixels (tw x th pixels of tb consecutive images) x BN output channels, K step = 32 fp32
// (one 128-byte swizzle span).  Persistent CTAs (one per SM) walk the tiles.  Warp roles: warps 0-7 = two consumer
// warpgroups (64 rows each: operand staging, wgmma, fused epilogue -- through a shared-memory staging tile and TMA
// stores for fprop / dgrad, straight from the accumulator registers otherwise), warpgroup 2 (warps 8-11) = TMA producer,
// which gives most of its registers to the consumers (setmaxnreg).  smem ring of STAGES stages, mbarrier full/empty pairs.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"
#include "tc_common.cuh"
#include "tma_host.cuh"

namespace {

using namespace mdb;

constexpr int BM = 128;
constexpr int BK = 32;                 // fp32 elements per k-block = 128 bytes
constexpr int kTileABytes = BM * 128;  // 16 KiB
constexpr int kChunkBytes = 32 * 128;  // one MN-major chunk: 32 reduction rows x 128 B
constexpr int kConsumerThreads = 256;  // two warpgroups
constexpr int kThreadsTC = kConsumerThreads + 128;   // + the producer warpgroup
// Registers per thread after reallocation: 128 x 40 + 256 x 232 = 64 512, what 384 threads at 168 start with.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
constexpr int kMaxTaps = 9;

struct TcParams {
    // ---- fprop / dgrad: decomposition of the M dimension into th x tw pixel rectangles ----------
    int tiles_x, tiles_y, tw, th, tb;   // an M tile = tw x th pixels of tb consecutive images (tw * th * tb == 128)
    int Ho, Wo;                      // logical output grid covered by tiles (bounds for rows)
    int out_sy, out_sx, out_oy, out_ox, out_H, out_W;   // real output pixel = (y*out_sy+out_oy, ...)
    int in_sy, in_sx;                // A-box origin = (y0*in_sy + dy[tap], x0*in_sx + dx[tap])
    int ntaps, cblocks;
    int tap_dy[kMaxTaps], tap_dx[kMaxTaps], tap_w[kMaxTaps];
    // ---- wgrad: reduction over pixel tiles of 32 (rth x rtw), split across blockIdx.z ----------
    int rtiles_x, rtiles_y, rtw, rth, n_img, red_per_split;
    // ---- fprop split-K (few tiles, very long reduction): slice z of the k-blocks writes its partial tile to out + z * slice_stride
    int kb_per_slice, slice_stride;  // 0 = off; a fixed-order reduction kernel sums the slices (deterministic, unlike atomics)
    int total_tiles, n_tiles_n, n_tiles_m;   // persistent tile walk: tile = (z * n_tiles_m + m) * n_tiles_n + n
    int w_sy, w_sx, wg_taps, wg_kw, wg_pad;   // X-box origin = (y0*w_sy + ky - pad, x0*w_sx + kx - pad); all taps in ONE launch
    // ---- epilogue -----------------------------------------------------------------------------
    int Mo_rows;                     // wgrad: number of valid output rows (Cout)
    int No, ldo;
    int relu, atomic_out, round_out;   // round_out: store round-to-nearest TF32 (next consumer is a tensor-core operand)
    // TMA epilogue (mapO / mapR): 0 = register epilogue.  epi_load: 1 = residual, 2 = ReLU mask fetched by TMA through mapR
    // into the staging tile.  Warpgroup 1's box starts half_{x,y,b} pixels / rows / images after warpgroup 0's.
    int epi_tma, epi_load, half_x, half_y, half_b;
    const float* bias;               // [No] or null
    const float* residual;           // same indexing as out, or null
    const float* relu_mask;          // same indexing as out: out *= (mask > 0), or null
    const float* rowscale;           // wgrad: [Mo_rows] or null
    float* out;
};

// Byte offset of fp32 element (row, k) of a TMA-delivered 128-byte-swizzled tile.  K-major: one 128-byte row per row
// index.  MN-major: 32-row chunks of [32 reduction rows][128 B], 4096 bytes apart.
template <bool MN>
__device__ __forceinline__ uint32_t raw_off(int row, int k) {
    if constexpr (MN) return (uint32_t)((row >> 5) * kChunkBytes + k * 128 + (((((row & 31) >> 2) ^ (k & 7))) << 4) + (row & 3) * 4);
    else return (uint32_t)(row * 128 + (((k >> 2) ^ (row & 7)) << 4) + (k & 3) * 4);
}

__device__ __forceinline__ float trunc_tf32(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// Shared memory of one kernel instance: the TMA ring, the epilogue staging tile of fprop / dgrad, the consumers' B operand
// tile(s) -- two sets, by k-block parity, so that one k-block's wgmmas can read one while the next k-block's B is written
// into the other --, barriers.  The staging tile is made of 32-channel boxes of 64 128-byte swizzled rows (8 KB), kBufs per
// warpgroup: all BN / 32 of a warpgroup's 64 x BN results when they fit beside the ring; for BN = 256 (a full staging tile
// is 128 KB) the largest power of two of them that fits, reused in turn as the stores drain (see the TMA epilogue).
template <int BN, int STAGES, int MODE, int PREC>
struct TcSmem {
    static constexpr bool kConvB = !(PREC == 2 && (MODE & 1) == 0);
    static constexpr int kRing = STAGES * (kTileABytes + BN * 128);
    static constexpr int kConvBuf = kConvB ? (PREC == 1 ? 2 : 1) * BN * 128 : 0;   // [hi | lo] operand tiles of one k-block
    static constexpr int kConv = 2 * kConvBuf;
    static constexpr int kFixed = kRing + kConv + 1024 /*align slack*/ + 256 /*barriers*/;
    static constexpr int kChunks = BN / 32;                        // 32-channel boxes per warpgroup and tile
    static constexpr int kRoom = (227 * 1024 - kFixed) / (2 * 8192);   // boxes per warpgroup that fit beside the ring
    static constexpr int kBufs = kRoom >= kChunks ? kChunks : BN < 256 ? 0 : kRoom >= 4 ? 4 : kRoom >= 2 ? 2 : kRoom;
    static constexpr int kStage = 2 * kBufs * 8192;
    static constexpr bool kTmaEpi = (MODE & 1) == 0 && kBufs > 0;
    static constexpr int kBytes = kFixed + (kTmaEpi ? kStage : 0);
};

// Persistent, warp-specialised kernel.  Each CTA walks tiles  tile = blockIdx.x + i * gridDim.x.
//   warps 8-11      producer warpgroup: one thread issues the TMA loads (smem ring of STAGES stages, full/empty mbarriers);
//                   the warpgroup shrinks to kProducerRegs registers so that the consumers can grow to kConsumerRegs
//   warps 0-7       two consumer warpgroups; warpgroup g owns rows [64g, 64g+64) of the 128-row tile.  Per k-block each
//                   thread loads its A fragments from the landed fp32 tile and splits them in registers; B is read by the
//                   tensor core from shared memory, either as delivered (pre-split bf16 weights) or after the consumers
//                   have rewritten it into a K-major operand tile (see CONVB).  The consumer loop is software-pipelined:
//                   k-block i's wgmmas run while the thread waits for k-block i+1's stage and loads it into the other of
//                   two fragment buffers (and B operand tiles); the stage of k-block i-1 is released once its wgmmas are
//                   known complete.  Every accumulator still sees the same wgmmas in the same k order.
// PREC (arithmetic):
//   2  bf16x3: x = hi + lo with hi = bf16(x), lo = bf16(x - hi); per k-block A_hi*B_hi + A_lo*B_hi + A_hi*B_lo as
//      m64nBNk16 bf16 wgmma (BN = 256 only here: 128 accumulators per consumer thread).  In fprop / dgrad the B operand
//      arrives PRE-SPLIT from global memory -- packed weights [tap][n][k-block][hi 32 | lo 32] bf16, one 128-byte swizzle
//      row per (n, k-block), written once per step by pack_gemm_weights_bf16x3.  Dropped terms are O(2^-17) per product.
//   1  3xTF32: hi = trunc_tf32(x), lo = x - hi; the same three products as m64nBNk8 tf32 wgmma.
//   0  single-pass TF32 (operands truncated by the tensor core; outputs optionally rounded for the next consumer).
// MODE 2 / 3 are the channel-banded twins of MODE 0 / 1 (grouped convolutions, see conv_grouped_check): the reduction of
// the tile at output channel n0 covers input channels [n0, n0 + BN) only, against a band-local weight [tap][C][BN].
// fprop / dgrad offset the A box's channel origin by n0; wgrad computes the diagonal (m0, m0) blocks only, reading the B
// operand's channels at m0.
template <int BN, int STAGES, int MODE /*0 fprop/dgrad, 1 wgrad, 2 / 3 banded*/, bool B_MN, int PREC>
__global__ void __launch_bounds__(kThreadsTC, 1)
tc_conv_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                    const __grid_constant__ CUtensorMap mapO, const __grid_constant__ CUtensorMap mapR,
                    const __grid_constant__ TcParams p) {
    constexpr bool WGRAD = (MODE & 1) != 0;
    constexpr bool BAND = MODE >= 2;
    constexpr bool A_MN = WGRAD;
    static_assert(!WGRAD || B_MN, "wgrad reads both operands MN-major");
    constexpr bool BF_B = (PREC == 2 && !WGRAD);                  // B arrives as pre-split bf16 rows
    static_assert(BN == 64 || BN == 128 || (BN == 256 && BF_B), "tile width");
    static_assert(!BF_B || !B_MN, "pre-split weights are K-major");
    constexpr bool CONVB = !BF_B;                                 // consumers rewrite B into the operand tile(s)
    constexpr int kTileBBytes = BN * 128;
    constexpr int kRawBytes = kTileABytes + kTileBBytes;          // what TMA delivers per stage
    using SM = TcSmem<BN, STAGES, MODE, PREC>;
    constexpr int NACC = BN / 2;

    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* stage_out = smem + STAGES * kRawBytes;               // epilogue staging tile (SM::kTmaEpi)
    uint8_t* bconv = stage_out + (SM::kTmaEpi ? SM::kStage : 0);  // [hi | lo] operand tiles of even / odd k-blocks (CONVB)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(bconv + SM::kConv);
    uint64_t* empty_bar = full_bar + STAGES;
    // TMA epilogue: the warpgroup's staging buffers are used in rounds of kRound boxes, kSlots rounds' worth at a time
    constexpr int kRound = SM::kBufs >= SM::kChunks ? SM::kChunks : 1;
    constexpr int kSlots = SM::kBufs / kRound > 0 ? SM::kBufs / kRound : 1;
    constexpr int kRounds = SM::kChunks / kRound;
    static_assert(kRounds % kSlots == 0, "every slot serves the same number of rounds per tile");
    uint64_t* epi_bar = empty_bar + STAGES;                       // [warpgroup][slot]: its residual / mask boxes have landed

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // ---- tile decode (identical in every role) -----------------------------------------------------
    struct Tile { int n0, img, y0, x0, m0, red_begin, iters, tap, slice; };
    auto decode = [&](int tix) {
        Tile t;
        t.n0 = (tix % p.n_tiles_n) * BN;
        int r = tix / p.n_tiles_n;
        t.img = t.y0 = t.x0 = t.m0 = t.red_begin = t.tap = t.slice = 0;
        if constexpr (!WGRAD) {
            const int per_img = p.tiles_x * p.tiles_y;
            t.iters = p.ntaps * p.cblocks;
            if (p.kb_per_slice > 0) {
                t.slice = r / p.n_tiles_m;
                r -= t.slice * p.n_tiles_m;
                t.red_begin = t.slice * p.kb_per_slice;
                t.iters = max(0, min(t.iters, t.red_begin + p.kb_per_slice) - t.red_begin);
            }
            const int grp = r / per_img;
            t.img = grp * p.tb;
            r -= grp * per_img;
            t.y0 = (r / p.tiles_x) * p.th;
            t.x0 = (r % p.tiles_x) * p.tw;
        } else {
            t.m0 = (r % p.n_tiles_m) * BM;
            r /= p.n_tiles_m;
            t.tap = r % p.wg_taps;
            const int z = r / p.wg_taps;
            const int total_red = p.n_img * p.rtiles_x * p.rtiles_y;
            t.red_begin = z * p.red_per_split;
            t.iters = max(0, min(total_red, t.red_begin + p.red_per_split) - t.red_begin);
        }
        return t;
    };

    if (threadIdx.x == 0) {
        if (smem_u32(smem) & 1023u) __trap();                     // SWIZZLE_128B tiles need 1024-byte aligned stages
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
        if (SM::kTmaEpi && p.epi_tma) {
            tma_prefetch_desc(&mapO);
            if (p.epi_load) tma_prefetch_desc(&mapR);
        }
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kConsumerThreads / 32);      // one arrival per consumer warp
        }
        for (int i = 0; i < 2 * kSlots; ++i) mbar_init(&epi_bar[i], 1);
        fence_mbar_init();
    }
    __syncthreads();
    // Programmatic dependent launch (launch_tc): everything above -- barrier init, tensor-map prefetch -- touches no global
    // data and may run while the previous kernel of the stream is still finishing; every thread waits here (before any
    // role reads or writes global memory, and before any thread can exit, so that completion of this grid implies
    // completion of its predecessors) until that kernel has completed and its writes are visible.  A no-op for a normal
    // launch.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    // ... and let the NEXT kernel of the stream (if it was launched as a programmatic dependent) start its own prologue now:
    // it waits at the same point for this grid to complete.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    if (warp >= kConsumerThreads / 32) {
        // ================================ TMA producer =============================================
        setmaxnreg_dec<kProducerRegs>();
        if (warp == kConsumerThreads / 32 && elect_one()) {
            int git = 0;                                          // ring position, continues across tiles
            for (int tix = blockIdx.x; tix < p.total_tiles; tix += gridDim.x) {
                const Tile t = decode(tix);
                for (int it = 0; it < t.iters; ++it, ++git) {
                    const int s = git % STAGES;
                    const uint32_t ph = (git / STAGES) & 1;
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t* a_dst = smem + s * kRawBytes;
                    uint8_t* b_dst = a_dst + kTileABytes;
                    mbar_arrive_expect_tx(&full_bar[s], kRawBytes);
                    if constexpr (!WGRAD) {
                        const int kit = t.red_begin + it;                 // (fprop split-K: this slice's first k-block)
                        const int tap = kit / p.cblocks;
                        const int cb = kit - tap * p.cblocks;
                        tma_load_4d(a_dst, &mapA, &full_bar[s], BAND ? t.n0 + cb * BK : cb * BK, t.x0 * p.in_sx + p.tap_dx[tap],
                                    t.y0 * p.in_sy + p.tap_dy[tap], t.img);
                        if constexpr (BF_B) {   // bf16 map: one 128-byte row = [hi 32 | lo 32] of k-block cb
                            tma_load_3d(b_dst, &mapB, &full_bar[s], cb * 64, t.n0, p.tap_w[tap]);
                        } else if constexpr (!B_MN) {
                            tma_load_3d(b_dst, &mapB, &full_bar[s], cb * BK, t.n0, p.tap_w[tap]);
                        } else {
#pragma unroll
                            for (int j = 0; j < BN / 32; ++j)
                                tma_load_3d(b_dst + j * kChunkBytes, &mapB, &full_bar[s], t.n0 + j * 32, cb * BK, p.tap_w[tap]);
                        }
                    } else {
                        int r = t.red_begin + it;
                        const int per_img = p.rtiles_x * p.rtiles_y;
                        const int ri = r / per_img;
                        r -= ri * per_img;
                        const int ry = (r / p.rtiles_x) * p.rth;
                        const int rx = (r % p.rtiles_x) * p.rtw;
#pragma unroll
                        for (int j = 0; j < BM / 32; ++j)
                            tma_load_4d(a_dst + j * kChunkBytes, &mapA, &full_bar[s], t.m0 + j * 32, rx, ry, ri);
#pragma unroll
                        for (int j = 0; j < BN / 32; ++j)
                            tma_load_4d(b_dst + j * kChunkBytes, &mapB, &full_bar[s], (BAND ? t.m0 : t.n0) + j * 32,
                                        rx * p.w_sx + (t.tap % p.wg_kw) - p.wg_pad, ry * p.w_sy + (t.tap / p.wg_kw) - p.wg_pad, ri);
                    }
                }
            }
        }
        return;
    }

    // ==================================== consumer warpgroups ==========================================
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2;
    const int g = lane >> 2, tig = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g;                 // this thread's tile rows: r0 and r0 + 8
    const int ctid = threadIdx.x;                                 // 0..255
    // TMA epilogue: warpgroup wg stages its 64 x BN results in its half of stage_out and thread 128 * wg (the leader, which
    // owns the warpgroup's bulk groups) stores them; the warpgroup goes on to the next tile while the store drains.
    const bool epi_tma = SM::kTmaEpi && p.epi_tma;
    const bool leader = (ctid & 127) == 0;
    uint8_t* my_stage = stage_out + wg * (SM::kStage / 2);
    uint64_t* my_epi_bar = epi_bar + wg * kSlots;
    uint32_t epi_use = 0;                                         // rounds each slot has served
    constexpr int KS = PREC == 2 ? 2 : 4;                         // k-steps per k-block: 16 bf16 or 8 tf32 each
    using Frag = uint32_t[KS][4];                                 // this thread's A fragments of one k-block (hi or lo)
    // Wait for ring k-block gi, rewrite its B into operand tile set `buf` (CONVB), then load this thread's A fragments of it
    // and split them into hi / lo.
    auto load_kblock = [&](int gi, int buf, Frag& hi, Frag& lo) {
        const int s = gi % STAGES;
        mbar_wait(&full_bar[s], (gi / STAGES) & 1);
        const uint8_t* a_raw = smem + s * kRawBytes;
        if constexpr (CONVB) {
            const uint8_t* b_raw = a_raw + kTileABytes;
            uint8_t* bc = bconv + buf * SM::kConvBuf;
            // Every consumer has waited for the wgmmas that last read this operand tile set (k-block gi - 2's, or the
            // previous tile's): it may be rewritten.
            named_bar_sync(1, kConsumerThreads);
            if constexpr (PREC == 2) {
                // B -> K-major bf16 rows [hi 32 | lo 32] (the packed-weight format): item = (n, 8-element k group c)
#pragma unroll
                for (int i = ctid; i < BN * 4; i += kConsumerThreads) {
                    const int n = i % BN, c = i / BN;
                    float x[8];
#pragma unroll
                    for (int e = 0; e < 8; ++e) x[e] = *reinterpret_cast<const float*>(b_raw + raw_off<B_MN>(n, 8 * c + e));
                    uint32_t hw[4], lw[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const uint32_t h = pack_bf16x2(x[2 * e], x[2 * e + 1]);
                        hw[e] = h;
                        lw[e] = pack_bf16x2(x[2 * e] - __uint_as_float(h << 16), x[2 * e + 1] - __uint_as_float(h & 0xFFFF0000u));
                    }
                    uint8_t* brow = bc + n * 128;
                    *reinterpret_cast<uint4*>(brow + ((c ^ (n & 7)) << 4)) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                    *reinterpret_cast<uint4*>(brow + (((4 + c) ^ (n & 7)) << 4)) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
                }
            } else {
                // B -> K-major tf32 hi tile (+ lo tile for 3xTF32): item = (n, 4-element k group c)
#pragma unroll 4
                for (int i = ctid; i < BN * 8; i += kConsumerThreads) {
                    const int n = i % BN, c = i / BN;
                    float4 x;
                    if constexpr (B_MN) {
                        x.x = *reinterpret_cast<const float*>(b_raw + raw_off<true>(n, 4 * c));
                        x.y = *reinterpret_cast<const float*>(b_raw + raw_off<true>(n, 4 * c + 1));
                        x.z = *reinterpret_cast<const float*>(b_raw + raw_off<true>(n, 4 * c + 2));
                        x.w = *reinterpret_cast<const float*>(b_raw + raw_off<true>(n, 4 * c + 3));
                    } else {
                        x = *reinterpret_cast<const float4*>(b_raw + raw_off<false>(n, 4 * c));
                    }
                    const float4 h = make_float4(trunc_tf32(x.x), trunc_tf32(x.y), trunc_tf32(x.z), trunc_tf32(x.w));
                    const uint32_t off = n * 128 + ((c ^ (n & 7)) << 4);
                    *reinterpret_cast<float4*>(bc + off) = h;
                    if constexpr (PREC == 1)
                        *reinterpret_cast<float4*>(bc + kTileBBytes + off) = make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
                }
            }
            fence_proxy_async_smem();      // generic-proxy writes -> visible to the tensor core's async-proxy reads
            named_bar_sync(1, kConsumerThreads);
        }
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int f = 0; f < 4; ++f) {
                const int row = r0 + (f & 1) * 8;
                if constexpr (PREC == 2) {
                    // fragment f: rows + 8 * (f & 1), k pair 2 * tig + 8 * (f >> 1) of this 16-wide step
                    const int k = ks * 16 + tig * 2 + (f >> 1) * 8;
                    float x0, x1;
                    if constexpr (A_MN) {
                        x0 = *reinterpret_cast<const float*>(a_raw + raw_off<true>(row, k));
                        x1 = *reinterpret_cast<const float*>(a_raw + raw_off<true>(row, k + 1));
                    } else {
                        const float2 v = *reinterpret_cast<const float2*>(a_raw + raw_off<false>(row, k));
                        x0 = v.x; x1 = v.y;
                    }
                    const uint32_t h = pack_bf16x2(x0, x1);
                    hi[ks][f] = h;
                    lo[ks][f] = pack_bf16x2(x0 - __uint_as_float(h << 16), x1 - __uint_as_float(h & 0xFFFF0000u));
                } else {
                    // fragment f: rows + 8 * (f & 1), k = tig + 4 * (f >> 1) of this 8-wide step
                    const int k = ks * 8 + tig + (f >> 1) * 4;
                    const float x = *reinterpret_cast<const float*>(a_raw + raw_off<A_MN>(row, k));
                    const float h = trunc_tf32(x);
                    hi[ks][f] = __float_as_uint(h);
                    lo[ks][f] = __float_as_uint(x - h);
                }
            }
        }
    };
    // Issue ring k-block gi's wgmmas (B from its stage, or from operand tile set `buf`) as one commit group.
    auto issue_kblock = [&](int gi, int buf, const Frag& hi, const Frag& lo, float (&acc)[NACC]) {
        const uint32_t b_addr = smem_u32(CONVB ? bconv + buf * SM::kConvBuf : smem + (gi % STAGES) * kRawBytes + kTileABytes);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            // B hi at byte 32 * ks of each 128-byte row; bf16 lo at 64 + 32 * ks, tf32 lo in the second tile
            const uint64_t bhi = make_wgmma_desc_sw128(b_addr + ks * 32);
            const uint64_t blo = make_wgmma_desc_sw128(b_addr + (PREC == 2 ? 64 : kTileBBytes) + ks * 32);
            if constexpr (PREC == 2) {
                if constexpr (BN == 256) {
                    wgmma_bf16_n256(acc, hi[ks], bhi, 1);
                    wgmma_bf16_n256(acc, lo[ks], bhi, 1);
                    wgmma_bf16_n256(acc, hi[ks], blo, 1);
                } else if constexpr (BN == 128) {
                    wgmma_bf16_n128(acc, hi[ks], bhi, 1);
                    wgmma_bf16_n128(acc, lo[ks], bhi, 1);
                    wgmma_bf16_n128(acc, hi[ks], blo, 1);
                } else {
                    wgmma_bf16_n64(acc, hi[ks], bhi, 1);
                    wgmma_bf16_n64(acc, lo[ks], bhi, 1);
                    wgmma_bf16_n64(acc, hi[ks], blo, 1);
                }
            } else {
                if constexpr (BN == 128) wgmma_tf32_n128(acc, hi[ks], bhi, 1);
                else wgmma_tf32_n64(acc, hi[ks], bhi, 1);
                if constexpr (PREC == 1) {
                    if constexpr (BN == 128) {
                        wgmma_tf32_n128(acc, lo[ks], bhi, 1);
                        wgmma_tf32_n128(acc, hi[ks], blo, 1);
                    } else {
                        wgmma_tf32_n64(acc, lo[ks], bhi, 1);
                        wgmma_tf32_n64(acc, hi[ks], blo, 1);
                    }
                }
            }
        }
        wgmma_commit();
    };
    int git = 0;
    for (int tix = blockIdx.x; tix < p.total_tiles; tix += gridDim.x) {
        const Tile t = decode(tix);
        if (p.atomic_out && t.iters == 0) continue;              // nothing to add
        // origin of this warpgroup's box: channel, then pixel x / y / image / split-K slice
        const int c1 = t.x0 + wg * p.half_x, c2 = t.y0 + wg * p.half_y, c3 = t.img + wg * p.half_b, c4 = t.slice;
        // Fetch round r's residual / mask boxes into slot r % kSlots of the staging buffers (its previous store has read it).
        auto fetch_round = [&](int r) {
            uint8_t* dst = my_stage + (r % kSlots) * (kRound * 8192);
            mbar_arrive_expect_tx(&my_epi_bar[r % kSlots], kRound * 8192);
#pragma unroll
            for (int c = 0; c < kRound; ++c)
                tma_load_5d(dst + c * 8192, &mapR, &my_epi_bar[r % kSlots], t.n0 + 32 * (r * kRound + c), c1, c2, c3, c4);
        };
        if (epi_tma && p.epi_load && leader) {
            // the previous tile's stores have read the staging buffers: fetch this tile's first rounds of residual / mask
            // into them now, while the k-blocks run
            bulk_wait_read_all();
#pragma unroll
            for (int r = 0; r < kSlots; ++r) fetch_round(r);
        }
        float acc[NACC];
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        if (t.iters > 0) {
            // Two fragment buffers (and operand tile sets) by k-block parity: k-block it's wgmmas run while k-block it + 1
            // is loaded into the other buffer.  A stage is released after the wait that retires its wgmmas.
            Frag ahi0, alo0, ahi1, alo1;
            auto step = [&](int it, const Frag& chi, const Frag& clo, Frag& nhi, Frag& nlo) {
                issue_kblock(git + it, it & 1, chi, clo, acc);
                wgmma_wait<1>();                                  // k-block it - 1's wgmmas have completed:
                wgmma_fence_operands(nhi);                        // its fragments may be overwritten
                wgmma_fence_operands(nlo);
                if (it > 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[(git + it - 1) % STAGES]);   // this warp is done with the stage
                }
                if (it + 1 < t.iters) load_kblock(git + it + 1, (it + 1) & 1, nhi, nlo);
            };
            load_kblock(git, 0, ahi0, alo0);
            for (int it = 0; it < t.iters; it += 2) {
                step(it, ahi0, alo0, ahi1, alo1);
                if (it + 1 < t.iters) step(it + 1, ahi1, alo1, ahi0, alo0);
            }
            wgmma_wait<0>();
            wgmma_fence_operands(acc);
            wgmma_fence_operands(ahi0);
            wgmma_fence_operands(alo0);
            wgmma_fence_operands(ahi1);
            wgmma_fence_operands(alo1);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[(git + t.iters - 1) % STAGES]);
            git += t.iters;
        }

        if (epi_tma) {
            // ---- TMA epilogue: the same operations in the same order as the register epilogue below, through the
            // staging tile (which holds the TMA-fetched residual or mask, read in place); the map clips the box at the
            // output's bounds, so rows and channels past them are computed but never stored.
            // Operands read from global memory (the bias; a mask beside a TMA-fetched residual) are loaded in batches with no
            // staging-tile store in between: a load placed after such a store is not moved above it (the compiler cannot
            // tell the two apart), which made every 8 columns one more global round trip.  The bias goes into the
            // accumulators first -- the same addition, in the same order, as below.
            if (p.bias) {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int n = t.n0 + j * 8 + tig * 2;         // No % 4 == 0: n < No implies n + 1 < No
                    if (n >= p.No) continue;
                    const float b0 = p.bias[n], b1 = p.bias[n + 1];
                    acc[4 * j] += b0; acc[4 * j + 1] += b1; acc[4 * j + 2] += b0; acc[4 * j + 3] += b1;
                }
            }
            // The staging buffers hold kRound boxes per slot and kSlots slots: BN = 64 / 128 stage the whole tile as one
            // round; BN = 256 stages one 32-channel box per round and alternates slots, so that a round is written
            // while the previous one's store still reads its slot.  With a residual / mask operand, the rounds past the
            // first kSlots are fetched as their slots drain, behind the tile's k-blocks no longer.
            constexpr int kMB = 8 < kRound * 4 ? 8 : kRound * 4;  // mask columns groups per batch (registers: 2 x kMB)
#pragma unroll
            for (int r = 0; r < kRounds; ++r) {                   // unrolled: the accumulators are indexed by r
                uint8_t* slot = my_stage + (r % kSlots) * (kRound * 8192);
                if (p.epi_load) {
                    mbar_wait(&my_epi_bar[r % kSlots], (epi_use + r / kSlots) & 1);
                } else {
                    if (leader) bulk_wait_read<kSlots - 1>();     // the store that last read this slot is done with it
                    named_bar_sync_diverged(2 + wg, 128);         // (the leader's lane may still be in its branch)
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = r0 + h * 8, rr = row - 64 * wg;
                    const float* gmask = nullptr;                 // mask beside a TMA-fetched residual: read from global
                    if (p.relu_mask && p.epi_load != 2) {
                        const int lyt = row / p.tw, lx = row - lyt * p.tw;
                        const int ib = lyt / p.th, ly = lyt - ib * p.th;
                        const int y = t.y0 + ly, x = t.x0 + lx, img = t.img + ib;
                        if ((y < p.Ho) && (x < p.Wo) && (img < p.n_img))
                            gmask = p.relu_mask + (size_t)((img * p.out_H + y * p.out_sy + p.out_oy) * p.out_W + x * p.out_sx + p.out_ox) * p.ldo;
                    }
#pragma unroll
                    for (int j0 = 0; j0 < kRound * 4; j0 += kMB) {
                        float2 mv[kMB];                           // 0 for rows past the output (computed, never stored)
#pragma unroll
                        for (int u = 0; u < kMB; ++u) {
                            const int n = t.n0 + (r * kRound * 4 + j0 + u) * 8 + tig * 2;
                            mv[u] = (gmask && n < p.No) ? *reinterpret_cast<const float2*>(gmask + n) : make_float2(0.f, 0.f);
                        }
#pragma unroll
                        for (int u = 0; u < kMB; ++u) {
                            const int jl = j0 + u, j = r * kRound * 4 + jl, n = t.n0 + j * 8 + tig * 2;
                            if (n >= p.No) continue;
                            float2* sp = reinterpret_cast<float2*>(slot + (jl >> 2) * 8192 + raw_off<false>(rr, (j & 3) * 8 + tig * 2));
                            float v[2] = {acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]};   // (+ bias; the register path's * 1.f: exact)
                            if (p.epi_load == 1) { const float2 e = *sp; v[0] += e.x; v[1] += e.y; }
                            if (p.relu) { v[0] = fmaxf(v[0], 0.f); v[1] = fmaxf(v[1], 0.f); }
                            if (p.relu_mask) {
                                const float2 m = p.epi_load == 2 ? *sp : mv[u];
                                v[0] = m.x > 0.f ? v[0] : 0.f; v[1] = m.y > 0.f ? v[1] : 0.f;
                            }
                            if (p.round_out) { v[0] = round_tf32(v[0]); v[1] = round_tf32(v[1]); }
                            *sp = make_float2(v[0], v[1]);
                        }
                    }
                }
                fence_proxy_async_smem();      // generic-proxy writes -> visible to the bulk copy's async-proxy reads
                named_bar_sync_diverged(2 + wg, 128);
                if (leader) {
#pragma unroll
                    for (int c = 0; c < kRound; ++c)
                        tma_store_5d(&mapO, slot + c * 8192, t.n0 + 32 * (r * kRound + c), c1, c2, c3, c4);
                    bulk_commit();
                    if (p.epi_load && r + kSlots < kRounds) {
                        bulk_wait_read_all();
                        fetch_round(r + kSlots);
                    }
                }
                __syncwarp();                  // the leader's lane rejoins its warp before the next round's barrier
            }
            epi_use += kRounds / kSlots;
            continue;
        }
        // ---- epilogue: accumulator registers -> fused bias / residual / ReLU / mask / row-scale -> global ------------
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + h * 8;
            bool ok;
            size_t roff;
            float rsc = 1.f;
            if constexpr (!WGRAD) {
                const int lyt = row / p.tw, lx = row - lyt * p.tw;
                const int ib = lyt / p.th, ly = lyt - ib * p.th;  // image within the tile, row within the image
                const int y = t.y0 + ly, x = t.x0 + lx, img = t.img + ib;
                ok = (y < p.Ho) && (x < p.Wo) && (img < p.n_img);
                const int oy = y * p.out_sy + p.out_oy, ox = x * p.out_sx + p.out_ox;
                roff = (size_t)((img * p.out_H + oy) * p.out_W + ox) * p.ldo + (size_t)t.slice * p.slice_stride;
            } else {
                ok = (t.m0 + row) < p.Mo_rows;
                if (ok && p.rowscale) rsc = p.rowscale[t.m0 + row];
                roff = (size_t)(t.tap * p.Mo_rows + t.m0 + row) * p.ldo;
            }
            if (!ok) continue;
            const bool vec = !(p.ldo & 1);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int n = t.n0 + j * 8 + tig * 2;
                if (n >= p.No) continue;
                float v[2] = {acc[4 * j + 2 * h] * rsc, acc[4 * j + 2 * h + 1] * rsc};
                const bool pair = vec && n + 1 < p.No;
                if (p.bias) { v[0] += p.bias[n]; if (pair) v[1] += p.bias[n + 1]; }
                if (p.residual) {
                    if (pair) { const float2 e = *reinterpret_cast<const float2*>(p.residual + roff + n); v[0] += e.x; v[1] += e.y; }
                    else v[0] += p.residual[roff + n];
                }
                if (p.relu) { v[0] = fmaxf(v[0], 0.f); v[1] = fmaxf(v[1], 0.f); }
                if (p.relu_mask) {
                    if (pair) {
                        const float2 m = *reinterpret_cast<const float2*>(p.relu_mask + roff + n);
                        v[0] = m.x > 0.f ? v[0] : 0.f; v[1] = m.y > 0.f ? v[1] : 0.f;
                    } else {
                        v[0] = p.relu_mask[roff + n] > 0.f ? v[0] : 0.f;
                    }
                }
                if (p.round_out) { v[0] = round_tf32(v[0]); v[1] = round_tf32(v[1]); }
                float* dst = p.out + roff + n;
                if (pair) {
                    if (p.atomic_out) red_add_v2_f32(dst, v[0], v[1]);
                    else *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
                } else {
                    for (int e = 0; e < 2 && n + e < p.No; ++e) {
                        // unpaired: odd ldo or the last column; recompute the second element's inputs scalar-wise
                        float x = e == 0 ? v[0] : acc[4 * j + 2 * h + 1] * rsc;
                        if (e == 1) {
                            if (p.bias) x += p.bias[n + 1];
                            if (p.residual) x += p.residual[roff + n + 1];
                            if (p.relu) x = fmaxf(x, 0.f);
                            if (p.relu_mask) x = p.relu_mask[roff + n + 1] > 0.f ? x : 0.f;
                            if (p.round_out) x = round_tf32(x);
                        }
                        if (p.atomic_out) atomicAdd(dst + e, x);
                        else dst[e] = x;
                    }
                }
            }
        }
    }
    // The grid's completion (which a programmatic dependent waits for) must imply that its bulk stores have landed.
    if (epi_tma && leader) bulk_wait_all();
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// Arithmetic mode: a process-wide numerical setting (like torch.backends.cuda.matmul.allow_tf32), not per-device state.
// 0 = single-pass TF32 (operands rounded to nearest), 1 = error-compensated 3xTF32, 2 = error-compensated BF16x3 for
// fprop / dgrad (pre-split weights) and wgrad -- the default.
int g_precision = 2;

// Everything that belongs to ONE device lives here, keyed by cudaGetDevice() (several devices per process: nn.DataParallel,
// tools/train_val.py:50-55): the split-K scratch registered by the caller.
constexpr int kMaxDevices = 64;
struct DeviceState {
    float* ws = nullptr;         // split-K scratch: owned by the CALLER (mdb_set_workspace), never freed / reallocated here
    size_t ws_bytes = 0;
};
DeviceState g_dev[kMaxDevices];

int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 0;
    return dev;
}

// `grid` carries the logical tile counts (x = column tiles, y = row tiles, z = split-K slices); the kernel is
// launched persistent with min(total_tiles, SMs) CTAs.
// `o` / `r` describe the output and the residual or mask operand for the TMA epilogue (p.epi_tma); an instance whose ring
// leaves no room for the staging tile runs the register epilogue whatever the launch asks.
template <int BN, int STAGES, int MODE, bool B_MN, int PREC>
int launch_tc(const CUtensorMap& a, const CUtensorMap& b, const CUtensorMap& o, const CUtensorMap& r, TcParams p, dim3 grid,
              cudaStream_t stream) {
    constexpr int smem = TcSmem<BN, STAGES, MODE, PREC>::kBytes;
    static_assert(smem <= 227 * 1024, "dynamic shared memory budget");
    if (!TcSmem<BN, STAGES, MODE, PREC>::kTmaEpi) p.epi_tma = p.epi_load = 0;
    auto kern = tc_conv_gemm_kernel<BN, STAGES, MODE, B_MN, PREC>;
    const cudaError_t e = set_max_dynamic_smem(kern, smem);
    if (e != cudaSuccess) return (int)e;
    p.n_tiles_n = (int)grid.x;
    p.n_tiles_m = (int)grid.y;
    p.total_tiles = (int)(grid.x * grid.y * grid.z);
    int ctas = num_sms();
    if (ctas > p.total_tiles) ctas = p.total_tiles;
    if (ctas < 1) return 0;
    // Launch as a PROGRAMMATIC DEPENDENT of the previous kernel in the stream (CUDA >= 11.8, graph capture >= 12.3; MDB_NO_PDL=1: plain launch): the
    // grid may be scheduled while that kernel drains, runs its prologue and then blocks in griddepcontrol.wait until the
    // predecessor has completed (see the kernel) -- the launch latency and the prologue of the ~470 GEMM launches of a training
    // step leave the critical path.  Other stream dependencies (events, memsets, copies) stay full dependencies.
    static const bool pdl = getenv("MDB_NO_PDL") == nullptr;
    if (pdl) {
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3((unsigned)ctas, 1, 1);
        cfg.blockDim = dim3((unsigned)kThreadsTC, 1, 1);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        return (int)cudaLaunchKernelEx(&cfg, kern, a, b, o, r, p);
    }
    kern<<<ctas, kThreadsTC, smem, stream>>>(a, b, o, r, p);
    return (int)cudaGetLastError();
}

// fprop split-K, second pass: y[i] = bias[i % N] + sum_z ws[z][i] in a fixed order.
__global__ void splitk_reduce_kernel(const float4* __restrict__ ws, const float4* __restrict__ bias, float4* __restrict__ y,
                                     long long n4, int N4, int slices, long long stride4) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 a = bias ? bias[i % N4] : make_float4(0.f, 0.f, 0.f, 0.f);
        for (int z = 0; z < slices; ++z) {
            const float4 v = ws[z * stride4 + i];
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
        y[i] = a;
    }
}

// Scratch for the split-K partial tiles.  The library never allocates: the caller registers a buffer for the current
// device (mdb_set_workspace; the Python side takes it from torch's caching allocator, which is CUDA-graph and
// multi-stream aware) after asking mdb_conv2d_forward_workspace_bytes.  Too small / missing -> MDB_EWORKSPACE.
int splitk_workspace(size_t bytes, float** out) {
    DeviceState& d = g_dev[current_device()];
    if (bytes > d.ws_bytes || !d.ws) return MDB_EWORKSPACE;
    *out = d.ws;
    return 0;
}

// choose a th x tw rectangle with th*tw == n_pix (128 for M tiles, 32 for wgrad reduction tiles)
void pick_tile(int W, int H, int n_pix, int* tw, int* th) {
    int best_tw = n_pix, best_waste = 1 << 30;
    for (int w = n_pix; w >= 1; w >>= 1) {
        const int h = n_pix / w;
        const int tx = (W + w - 1) / w, ty = (H + h - 1) / h;
        const int waste = tx * w * ty * h - W * H;
        if (waste < best_waste) { best_waste = waste; best_tw = w; }
    }
    *tw = best_tw;
    *th = n_pix / best_tw;
}

// M tile of fprop / dgrad: tw x th pixels of tb consecutive images, tw * th * tb == n_pix (128).  Spanning images keeps
// small feature maps dense (12 x 40 with 8 images: 8x4 pixels x 4 images = 30 full tiles instead of 40 tiles at 75 %).
void pick_tile3(int W, int H, int B, int n_pix, int* tw, int* th, int* tb) {
    long long best = -1;
    *tw = n_pix; *th = 1; *tb = 1;
    for (int b = 1; b <= n_pix; b <<= 1)
        for (int w = n_pix / b; w >= 1; w >>= 1) {
            const int h = n_pix / b / w;
            if (b > 1 && b >= 2 * B) continue;                    // never more padding images than real ones
            const long long cov = (long long)((W + w - 1) / w) * w * ((H + h - 1) / h) * h * ((B + b - 1) / b) * b;
            if (best < 0 || cov < best) { best = cov; *tw = w; *th = h; *tb = b; }   // ties: fewer images, wider rows
        }
}

bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; }

// TMA epilogue of a fprop / dgrad launch (p.epi_tma).  The output -- and the residual, else the ReLU mask, which share its
// indexing -- are 5-d tensor maps (C, W, H, B, split-K slice) over the launch's Wc x Hc x B pixel grid, starting `off`
// elements into each buffer, with pixel strides sx, sy, sb elements; the box is one consumer warpgroup's 64 rows of the
// tw x th x tb tile (the outermost tile dimension above 1 is halved).  Launches TMA cannot describe keep the register
// epilogue: a channel count or row pitch that is not a multiple of 4 (16-byte pitches), or a buffer that is not 16-byte
// aligned.
int setup_epi_px(TcParams& p, CUtensorMap* mo, CUtensorMap* mr, size_t off, int Wc, int Hc, int B, uint64_t sx, uint64_t sy,
                 uint64_t sb, int slices) {
    p.epi_tma = p.epi_load = p.half_x = p.half_y = p.half_b = 0;
    if (p.No % 4 || p.ldo % 4 || !aligned16(p.out + off) || (p.residual && !aligned16(p.residual + off)) ||
        (p.relu_mask && !aligned16(p.relu_mask + off)))
        return 0;
    uint32_t box[5] = {32, (uint32_t)p.tw, (uint32_t)p.th, (uint32_t)p.tb, 1};
    if (p.tb > 1) p.half_b = box[3] = p.tb / 2;
    else if (p.th > 1) p.half_y = box[2] = p.th / 2;
    else p.half_x = box[1] = p.tw / 2;
    if (box[1] > 256 || box[2] > 256 || box[3] > 256) return 0;
    uint64_t dims[5] = {(uint64_t)p.No, (uint64_t)Wc, (uint64_t)Hc, (uint64_t)B, (uint64_t)slices};
    uint64_t str[5] = {1, sx, sy, sb, slices > 1 ? (uint64_t)p.slice_stride : sb * B};
    int rc = make_map(mo, p.out + off, 5, dims, str, box, nullptr);
    if (rc) return rc;
    const float* opnd = p.residual ? p.residual : p.relu_mask;
    if (opnd) {
        rc = make_map(mr, opnd + off, 5, dims, str, box, nullptr);
        if (rc) return rc;
        p.epi_load = p.residual ? 1 : 2;
    }
    p.epi_tma = 1;
    return 0;
}

// Ring depth of the 128 x 256 BF16x3 tile: 4 stages of 48 KB leave 32 KB of staging (two 32-channel boxes per warpgroup).
constexpr int kWideStages = 4;

// Tile width of a BF16x3 fprop / dgrad launch with N output channels, `m_tiles` row tiles (per split-K slice, `slices`
// of them) and `kblocks` k-blocks per tile: 256 where N is a multiple of 256, the reduction is long and the wide tiles
// leave no CTA more work than the 128-wide ones do.  The wide tile's epilogue stages its 256 columns one 32-channel box
// at a time, so it costs more per tile than the 128-wide one's; only long reductions repay it (H100, 400 W: the 3x3
// 256 -> 256 convolution at 24 x 80, 72 k-blocks, 12 % faster; 1x1 layers with 2 - 32 k-blocks 2 - 15 % slower).  A wide
// tile costs per CTA what two 128-wide tiles cost, so it is taken when ceil(T256 / SMs) * 2 <= ceil(T128 / SMs) (3x3
// 512 -> 512 at 12 x 40, batch 8: 120 tiles at 128 on 132 SMs, one wave; 60 tiles at 256 would double it).  Every output
// element sees the same wgmmas in the same k order at either width, so the choice does not change the result.
constexpr int kWideMinKBlocks = 64;
int pick_bn(int N, int m_tiles, int slices, int kblocks) {
    const int base = N <= 64 ? 64 : 128;
    if (N % 256 || kblocks < kWideMinKBlocks) return base;
    const long long sms = num_sms(), t256 = (long long)m_tiles * (N / 256) * (slices > 0 ? slices : 1);
    const long long w256 = (t256 + sms - 1) / sms, w128 = (2 * t256 + sms - 1) / sms;
    return 2 * w256 <= w128 ? 256 : base;
}

// Launch the fprop / dgrad kernel (K-major B operand) for the arithmetic mode.
int launch_fwd(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr, const TcParams& p, dim3 grid, int bn, int precision, cudaStream_t stream) {
    if (precision == 2) {
        if (bn == 256) return launch_tc<256, kWideStages, 0, false, 2>(ma, mb, mo, mr, p, grid, stream);
        return bn == 64 ? launch_tc<64, 6, 0, false, 2>(ma, mb, mo, mr, p, grid, stream) : launch_tc<128, 5, 0, false, 2>(ma, mb, mo, mr, p, grid, stream);
    }
    if (precision == 1) return bn == 64 ? launch_tc<64, 5, 0, false, 1>(ma, mb, mo, mr, p, grid, stream) : launch_tc<128, 3, 0, false, 1>(ma, mb, mo, mr, p, grid, stream);
    return bn == 64 ? launch_tc<64, 6, 0, false, 0>(ma, mb, mo, mr, p, grid, stream) : launch_tc<128, 5, 0, false, 0>(ma, mb, mo, mr, p, grid, stream);
}

// Grouped convolutions (ResNeXt's 3x3 conv2: C channels in and out, `groups` groups of C / groups channels) as channel-banded
// GEMMs.  Every group lies inside one 128-channel band when C / groups divides 128, so the 128 output channels of a tile
// read only the 128 input channels of the same band: a tile walks taps x 4 k-blocks (MODE 2 / 3 instances) against a
// band-local weight [tap][C][128] that is zero outside the groups.  The tensor cores do 128 / (C / groups) times the
// grouped convolution's multiply-adds; the tile width stays 128, without the forward's split-K.
constexpr int kBand = 128;

// Launch the banded fprop / dgrad kernel (K-major band-local B operand) for the arithmetic mode.
int launch_band(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr, const TcParams& p, dim3 grid, int precision, cudaStream_t stream) {
    if (precision == 2) return launch_tc<kBand, 5, 2, false, 2>(ma, mb, mo, mr, p, grid, stream);
    if (precision == 1) return launch_tc<kBand, 3, 2, false, 1>(ma, mb, mo, mr, p, grid, stream);
    return launch_tc<kBand, 5, 2, false, 0>(ma, mb, mo, mr, p, grid, stream);
}

struct ConvGeom {
    int B, H, W, Cin, Cout, kh, kw, stride, pad, dil, Ho, Wo;
};

// Output size of a convolution (torch.nn.Conv2d's formula).
int conv_out(int n, int k, int stride, int pad, int dil) { return (n + 2 * pad - dil * (k - 1) - 1) / stride + 1; }

ConvGeom make_geom(int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dil) {
    return ConvGeom{B, H, W, Cin, Cout, kh, kw, stride, pad, dil, conv_out(H, kh, stride, pad, dil), conv_out(W, kw, stride, pad, dil)};
}

int check_geom(const ConvGeom& g, bool forward = false) {
    if (g.B <= 0 || g.H <= 0 || g.W <= 0 || g.Cin <= 0 || g.Cout <= 0) return MDB_EINVAL;
    if (g.kh != g.kw || (g.kh != 1 && g.kh != 3) || (g.stride != 1 && g.stride != 2)) return MDB_EUNSUPPORTED;
    // Dilation only changes the taps' box offsets; it is supported where ResNet's DC5 stage uses it: 3x3, stride 1.  (A
    // strided dilated dgrad would need per-parity tap sets of a different shape.)
    if (g.dil < 1 || (g.dil > 1 && (g.kh != 3 || g.stride != 1))) return MDB_EUNSUPPORTED;
    // TMA needs 16-byte row pitches on every operand it reads: Cin always; Cout only where dy / the output map is an
    // operand (dgrad, wgrad).  The forward epilogue writes ragged Cout with scalar stores.
    if (g.Cin % 4 || (!forward && g.Cout % 4)) return MDB_EUNSUPPORTED;
    return 0;
}

// Geometry of a grouped (banded) convolution: 3x3, Cin == Cout == C, C % 128 == 0, C / groups dividing 128, and the dense
// rules above (dilation > 1 only at stride 1; the weight gradient also needs pad % dilation == 0).
int conv_grouped_check(const ConvGeom& g, int groups, bool wgrad) {
    const int rc = check_geom(g);
    if (rc) return rc;
    if (groups <= 0) return MDB_EINVAL;
    if (g.kh != 3 || g.Cin != g.Cout || g.Cin % kBand || g.Cin % groups || kBand % (g.Cin / groups)) return MDB_EUNSUPPORTED;
    if (wgrad && g.pad % g.dil) return MDB_EUNSUPPORTED;
    return 0;
}

}  // namespace

extern "C" {

int mdb_set_precision(int mode) {
    if (mode < 0 || mode > 2) return MDB_EINVAL;
    g_precision = mode;
    return 0;
}
int mdb_get_precision(void) { return g_precision; }

}  // extern "C"

namespace {

// Split-K decision of the forward (shared by the launcher and mdb_conv2d_forward_workspace_bytes) for very long
// reductions (the 3x3 stride-2 2048->256 neck convolution: 16-32 tiles x 576 k-blocks kept a fifth of the SMs busy for
// 0.3 ms).  Returns the number of slices (0 = no split-K).  The decision deliberately ignores the tile count, which grows
// with the batch: it depends on the reduction length, Cout, the epilogue and (in the caller) the bias alignment, so an
// image is summed in the same order whatever batch it is in.  The one batch-dependent term is the 32-bit bound on the
// scratch size below.
int forward_splitk_slices(int precision, int kblocks, int bn, bool plain_epilogue, int Cout, long long out_elems) {
    const int kb_per_slice = 32;
    if (precision == 0 || bn != 128 || kblocks < 256 || !plain_epilogue || Cout % 4) return 0;
    const int slices = (kblocks + kb_per_slice - 1) / kb_per_slice;
    return (out_elems * slices < (1ll << 31)) ? slices : 0;
}

// y[B,Ho,Wo,Cout] = act( conv(x[B,H,W,Cin], w) + bias + residual );  w = fp32 packed [kh*kw][Cout][Cin] (bf == false)
// or the pre-split bf16 form [kh*kw][Cout][ceil(Cin/32)][hi 32 | lo 32] (bf == true, precision mode 2).
// band: the grouped form (conv_grouped_check), w = band-local [kh*kw][Cout][128] (fp32) or [kh*kw][Cout][4][hi 32 | lo 32].
int conv_forward_impl(const float* x, const void* w_packed, bool bf, const float* bias, const float* residual, float* y,
                      int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dil, int flags,
                      void* stream_, size_t* query_ws = nullptr /* non-null: only report the scratch bytes this call needs */,
                      bool band = false) {
    const int precision = bf ? 2 : (g_precision == 2 ? 1 : g_precision);   // fp32 weights in bf16x3 mode: 3xTF32
    ConvGeom g = make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dil);
    int rc = check_geom(g, true);
    if (rc) return rc;
    if (!query_ws && (!x || !w_packed || !y)) return MDB_EINVAL;
    if ((unsigned long long)B * g.Ho * g.Wo * Cout >= (1ull << 31)) return MDB_EUNSUPPORTED;   // the epilogue indexes with (signed) 32 bits
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (kh == 1 && stride == 1 && pad == 0) {     // pointwise: the batch of images is one long row of pixels (no tile waste)
        W = B * H * W; H = 1; B = 1;
        g = make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dil);
    }
    TcParams p;
    memset(&p, 0, sizeof(p));
    pick_tile3(g.Wo, g.Ho, B, BM, &p.tw, &p.th, &p.tb);
    p.tiles_x = (g.Wo + p.tw - 1) / p.tw;
    p.tiles_y = (g.Ho + p.th - 1) / p.th;
    p.n_img = B;
    const int n_groups = (B + p.tb - 1) / p.tb;
    p.Ho = g.Ho; p.Wo = g.Wo;
    p.out_sy = p.out_sx = 1; p.out_oy = p.out_ox = 0; p.out_H = g.Ho; p.out_W = g.Wo;
    p.in_sy = p.in_sx = stride;
    p.ntaps = kh * kw;
    p.cblocks = band ? kBand / BK : (Cin + BK - 1) / BK;
    for (int ky = 0; ky < kh; ++ky)
        for (int kx = 0; kx < kw; ++kx) {
            const int t = ky * kw + kx;
            p.tap_dy[t] = ky * dil - pad; p.tap_dx[t] = kx * dil - pad; p.tap_w[t] = t;
        }
    p.wg_taps = 1; p.wg_kw = 1;
    p.No = Cout; p.ldo = Cout; p.relu = flags & 1; p.round_out = (precision == 0) ? ((flags >> 1) & 1) : 0; p.atomic_out = 0;
    p.bias = bias; p.residual = residual; p.relu_mask = nullptr; p.rowscale = nullptr; p.out = y;

    const long long out_elems = (long long)B * g.Ho * g.Wo * Cout;
    const int slices = (!band && (reinterpret_cast<uintptr_t>(bias) & 15u) == 0)
                           ? forward_splitk_slices(precision, p.ntaps * p.cblocks, Cout <= 64 ? 64 : 128, !residual && !p.relu, Cout, out_elems)
                           : 0;
    if (query_ws) {
        *query_ws = sizeof(float) * (size_t)out_elems * slices;
        return 0;
    }
    const int m_tiles = n_groups * p.tiles_x * p.tiles_y;
    const int bn = band ? kBand
                   : precision == 2 ? pick_bn(Cout, m_tiles, slices, slices > 0 ? 32 : p.ntaps * p.cblocks) : (Cout <= 64 ? 64 : 128);
    dim3 grid((Cout + bn - 1) / bn, m_tiles, 1);

    CUtensorMap ma, mb;
    {   // A: x as (C, W, H, B), box (32, tw*s, th*s, 1), element strides (1, s, s, 1)
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
        uint64_t str[4] = {1, (uint64_t)Cin, (uint64_t)W * Cin, (uint64_t)H * W * Cin};
        uint32_t box[4] = {BK, (uint32_t)(p.tw * stride), (uint32_t)(p.th * stride), (uint32_t)p.tb};
        uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
        if (box[1] > 256 || box[2] > 256) return MDB_EUNSUPPORTED;
        rc = make_map(&ma, x, 4, dims, str, box, es);
        if (rc) return rc;
    }
    if (bf) {   // B: pre-split bf16 weights as (64 * k-blocks, Cout, taps), box (64 = one [hi 32 | lo 32] row, BN, 1)
        const uint64_t kb = (uint64_t)p.cblocks;
        uint64_t dims[3] = {64 * kb, (uint64_t)Cout, (uint64_t)(kh * kw)};
        uint64_t str[3] = {1, 64 * kb, (uint64_t)Cout * 64 * kb};
        uint32_t box[3] = {64, (uint32_t)bn, 1};
        rc = make_map(&mb, w_packed, 3, dims, str, box, nullptr, true);
        if (rc) return rc;
    } else {   // B: packed weights as (Cin, Cout, taps) (band: (128, Cout, taps)), box (32, BN, 1)
        const uint64_t K = band ? kBand : Cin;
        uint64_t dims[3] = {K, (uint64_t)Cout, (uint64_t)(kh * kw)};
        uint64_t str[3] = {1, K, (uint64_t)Cout * K};
        uint32_t box[3] = {BK, (uint32_t)bn, 1};
        rc = make_map(&mb, w_packed, 3, dims, str, box, nullptr);
        if (rc) return rc;
    }
    CUtensorMap mo, mr;   // TMA epilogue: y (or the split-K slices) and the residual, as (Cout, Wo, Ho, B, slice)
    memset(&mo, 0, sizeof(mo));
    memset(&mr, 0, sizeof(mr));
    const uint64_t pix_x = (uint64_t)Cout, pix_y = pix_x * g.Wo, pix_b = pix_y * g.Ho;
    // Split-K (see forward_splitk_slices): slices write partial tiles to the caller's scratch buffer and a second kernel adds
    // them in a fixed order (+ bias): bit-reproducible, unlike atomic accumulation.  Whether a shape splits and into how
    // many slices of a fixed length depends on the per-image problem only (up to the scratch bound in
    // forward_splitk_slices), so the summation order of an image does not depend on the batch size.
    {
        if (slices > 0) {
            float* ws = nullptr;
            rc = splitk_workspace(sizeof(float) * (size_t)out_elems * slices, &ws);
            if (rc) return rc;
            p.kb_per_slice = 32;
            p.slice_stride = (int)out_elems;
            p.out = ws; p.bias = nullptr;
            grid.z = slices;
            rc = setup_epi_px(p, &mo, &mr, 0, g.Wo, g.Ho, B, pix_x, pix_y, pix_b, slices);
            if (rc) return rc;
            rc = launch_fwd(ma, mb, mo, mr, p, grid, bn, precision, stream);
            if (rc) return rc;
            const long long n4 = out_elems / 4;
            splitk_reduce_kernel<<<grid_cap(n4, 256, num_sms() * 8), 256, 0, stream>>>(
                reinterpret_cast<const float4*>(ws), reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(y), n4, Cout / 4, slices, n4);
            return (int)cudaGetLastError();
        }
    }
    rc = setup_epi_px(p, &mo, &mr, 0, g.Wo, g.Ho, B, pix_x, pix_y, pix_b, 1);
    if (rc) return rc;
    return band ? launch_band(ma, mb, mo, mr, p, grid, precision, stream) : launch_fwd(ma, mb, mo, mr, p, grid, bn, precision, stream);
}

// dx[B,H,W,Cin] = (conv_transpose(dy[B,Ho,Wo,Cout], w) + residual) * (relu_mask > 0);  w = fp32 packed [taps][Cout][Cin]
// (read MN-major) or, bf == true, the pre-split TRANSPOSED bf16 form [taps][Cin][ceil(Cout/32)][hi 32 | lo 32] (K-major).
// band: the grouped form, w = the band-local transposed weight [taps][Cin][128] (fp32, K-major) or [taps][Cin][4][hi 32 | lo 32].
int conv_dgrad_impl(const float* dy, const void* w_packed, bool bf, const float* residual, const float* relu_mask,
                    float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dil,
                    int flags, void* stream_, bool band = false) {
    const int precision = bf ? 2 : (g_precision == 2 ? 1 : g_precision);
    ConvGeom g = make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dil);
    int rc = check_geom(g);
    if (rc) return rc;
    if (!dy || !w_packed || !dx) return MDB_EINVAL;
    if ((unsigned long long)B * H * W * Cin >= (1ull << 31)) return MDB_EUNSUPPORTED;           // the epilogue indexes with (signed) 32 bits
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (kh == 1 && stride == 1 && pad == 0) {     // pointwise: one long row of pixels
        W = B * H * W; H = 1; B = 1;
        g = make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dil);
    }
    // dx[y,x] = sum_{ky,kx} dy[(y+pad-ky*d)/s, (x+pad-kx*d)/s] * W[ky,kx]  where the division is exact.
    // Per output parity class (py,px) (only one class for s == 1) the contributing taps are fixed and the
    // dy access is a unit-stride shifted box: oy = (y + pad - ky*d)/s = j + (py + pad - ky*d)/s  for y = s*j + py.
    // (d > 1 only with s == 1: one class, tap offsets pad - ky*d.)
    for (int py = 0; py < stride; ++py)
        for (int px = 0; px < stride; ++px) {
            TcParams p;
            memset(&p, 0, sizeof(p));
            const int Hc = (H - py + stride - 1) / stride, Wc = (W - px + stride - 1) / stride;  // pixels in class
            if (Hc <= 0 || Wc <= 0) continue;
            pick_tile3(Wc, Hc, B, BM, &p.tw, &p.th, &p.tb);
            p.tiles_x = (Wc + p.tw - 1) / p.tw;
            p.tiles_y = (Hc + p.th - 1) / p.th;
            p.n_img = B;
            const int n_groups = (B + p.tb - 1) / p.tb;
            p.Ho = Hc; p.Wo = Wc;
            p.out_sy = p.out_sx = stride; p.out_oy = py; p.out_ox = px; p.out_H = H; p.out_W = W;
            p.in_sy = p.in_sx = 1;
            p.cblocks = band ? kBand / BK : (Cout + BK - 1) / BK;
            int nt = 0;
            for (int ky = 0; ky < kh; ++ky) {
                if ((py + pad - ky * dil) % stride) continue;
                for (int kx = 0; kx < kw; ++kx) {
                    if ((px + pad - kx * dil) % stride) continue;
                    // floor division is exact here (numerator divisible by stride; may be negative)
                    p.tap_dy[nt] = (py + pad - ky * dil) / stride;
                    p.tap_dx[nt] = (px + pad - kx * dil) / stride;
                    p.tap_w[nt] = ky * kw + kx;
                    ++nt;
                }
            }
            p.ntaps = nt;
            p.wg_taps = 1; p.wg_kw = 1;
            p.No = Cin; p.ldo = Cin; p.relu = 0; p.atomic_out = 0; p.round_out = (precision == 0) ? ((flags >> 1) & 1) : 0;
            p.bias = nullptr; p.residual = residual; p.relu_mask = relu_mask; p.rowscale = nullptr; p.out = dx;
            CUtensorMap ma, mb;
            {   // A: dy as (Cout, Wo, Ho, B), unit stride
                uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)g.Wo, (uint64_t)g.Ho, (uint64_t)B};
                uint64_t str[4] = {1, (uint64_t)Cout, (uint64_t)g.Wo * Cout, (uint64_t)g.Ho * g.Wo * Cout};
                uint32_t box[4] = {BK, (uint32_t)p.tw, (uint32_t)p.th, (uint32_t)p.tb};
                rc = make_map(&ma, dy, 4, dims, str, box, nullptr);
                if (rc) return rc;
            }
            const int bn = band ? kBand : bf ? pick_bn(Cin, n_groups * p.tiles_x * p.tiles_y, 0, nt * p.cblocks) : 128;
            if (bf) {   // B (K-major): transposed pre-split weights as (64 * k-blocks, Cin, taps); box (64, BN, 1)
                const uint64_t kb = (uint64_t)p.cblocks;
                uint64_t dims[3] = {64 * kb, (uint64_t)Cin, (uint64_t)(kh * kw)};
                uint64_t str[3] = {1, 64 * kb, (uint64_t)Cin * 64 * kb};
                uint32_t box[3] = {64, (uint32_t)bn, 1};
                rc = make_map(&mb, w_packed, 3, dims, str, box, nullptr, true);
                if (rc) return rc;
            } else if (band) {   // B (K-major): band-local transposed weights as (128, Cin, taps); box (32, BN, 1)
                uint64_t dims[3] = {(uint64_t)kBand, (uint64_t)Cin, (uint64_t)(kh * kw)};
                uint64_t str[3] = {1, (uint64_t)kBand, (uint64_t)Cin * kBand};
                uint32_t box[3] = {BK, (uint32_t)kBand, 1};
                rc = make_map(&mb, w_packed, 3, dims, str, box, nullptr);
                if (rc) return rc;
            } else {   // B (MN-major): packed weights as (Cin, Cout, taps); box = 32 output columns (Cin) x 32 reduction rows (Cout)
                uint64_t dims[3] = {(uint64_t)Cin, (uint64_t)Cout, (uint64_t)(kh * kw)};
                uint64_t str[3] = {1, (uint64_t)Cin, (uint64_t)Cout * Cin};
                uint32_t box[3] = {32, 32, 1};
                rc = make_map(&mb, w_packed, 3, dims, str, box, nullptr);
                if (rc) return rc;
            }
            dim3 grid((Cin + bn - 1) / bn, n_groups * p.tiles_x * p.tiles_y, 1);
            if (nt == 0) {   // no tap reaches this parity class (1x1 stride 2): result = (0 + residual) * mask
                p.ntaps = 0;
            }
            CUtensorMap mo, mr;   // TMA epilogue: the parity class of dx (and residual / mask) as (Cin, Wc, Hc, B, 1)
            memset(&mo, 0, sizeof(mo));
            memset(&mr, 0, sizeof(mr));
            rc = setup_epi_px(p, &mo, &mr, (size_t)(py * W + px) * Cin, Wc, Hc, B, (uint64_t)stride * Cin,
                              (uint64_t)stride * W * Cin, (uint64_t)H * W * Cin, 1);
            if (rc) return rc;
            if (band) rc = launch_band(ma, mb, mo, mr, p, grid, precision, stream);
            else if (bf) rc = launch_fwd(ma, mb, mo, mr, p, grid, bn, 2, stream);
            else rc = (precision == 1) ? launch_tc<128, 3, 0, true, 1>(ma, mb, mo, mr, p, grid, stream)
                                       : launch_tc<128, 5, 0, true, 0>(ma, mb, mo, mr, p, grid, stream);
            if (rc) return rc;
        }
    return 0;
}

}  // namespace

extern "C" {

int mdb_conv2d_forward_f32(const float* x, const float* w_packed, const float* bias, const float* residual, float* y,
                           int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int flags,
                           void* stream) {
    return conv_forward_impl(x, w_packed, false, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, 1, flags, stream);
}
int mdb_conv2d_forward_dilated_f32(const float* x, const float* w_packed, const float* bias, const float* residual, float* y,
                                   int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation,
                                   int flags, void* stream) {
    return conv_forward_impl(x, w_packed, false, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags, stream);
}
int mdb_conv2d_forward_bf16x3(const float* x, const void* w_split, const float* bias, const float* residual, float* y,
                              int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int flags,
                              void* stream) {
    return conv_forward_impl(x, w_split, true, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, 1, flags, stream);
}
int mdb_conv2d_forward_dilated_bf16x3(const float* x, const void* w_split, const float* bias, const float* residual, float* y,
                                      int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation,
                                      int flags, void* stream) {
    return conv_forward_impl(x, w_split, true, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags, stream);
}
long long mdb_conv2d_forward_workspace_bytes_dilated(int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                                     int dilation, int flags, int has_residual, int split_weights) {
    size_t bytes = 0;
    const float* res = has_residual ? reinterpret_cast<const float*>(16) : nullptr;
    const int rc = conv_forward_impl(nullptr, nullptr, split_weights != 0, nullptr, res, nullptr, B, H, W, Cin, Cout, kh, kw, stride,
                                     pad, dilation, flags, nullptr, &bytes);
    return rc ? (long long)rc : (long long)bytes;
}
long long mdb_conv2d_forward_workspace_bytes(int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                             int flags, int has_residual, int split_weights) {
    return mdb_conv2d_forward_workspace_bytes_dilated(B, H, W, Cin, Cout, kh, kw, stride, pad, 1, flags, has_residual, split_weights);
}
int mdb_set_workspace(void* buf, unsigned long long bytes) {
    DeviceState& d = g_dev[current_device()];
    d.ws = static_cast<float*>(buf);
    d.ws_bytes = buf ? (size_t)bytes : 0;
    return 0;
}
int mdb_conv2d_dgrad_f32(const float* dy, const float* w_packed, const float* residual, const float* relu_mask,
                         float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                         int flags, void* stream) {
    return conv_dgrad_impl(dy, w_packed, false, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, 1, flags, stream);
}
int mdb_conv2d_dgrad_dilated_f32(const float* dy, const float* w_packed, const float* residual, const float* relu_mask,
                                 float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                 int dilation, int flags, void* stream) {
    return conv_dgrad_impl(dy, w_packed, false, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags,
                           stream);
}
int mdb_conv2d_dgrad_bf16x3(const float* dy, const void* w_split_t, const float* residual, const float* relu_mask,
                            float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                            int flags, void* stream) {
    return conv_dgrad_impl(dy, w_split_t, true, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, 1, flags, stream);
}
int mdb_conv2d_dgrad_dilated_bf16x3(const float* dy, const void* w_split_t, const float* residual, const float* relu_mask,
                                    float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                    int dilation, int flags, void* stream) {
    return conv_dgrad_impl(dy, w_split_t, true, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags,
                           stream);
}

// dw_packed[tap][Cout][Cin] (+)= rowscale[co] * sum_{b,oy,ox} dy[b,oy,ox,co] * x[b, oy*s+ky-pad, ox*s+kx-pad, ci]
// dw_packed is zero-filled by the call unless accumulate != 0.
int mdb_conv2d_wgrad_f32(const float* dy, const float* x, const float* rowscale, float* dw_packed, int B, int H, int W,
                         int Cin, int Cout, int kh, int kw, int stride, int pad, int accumulate, void* stream_) {
    return mdb_conv2d_wgrad_bias_f32(dy, x, rowscale, dw_packed, nullptr, B, H, W, Cin, Cout, kh, kw, stride, pad, accumulate, stream_);
}

// Same, plus db[Cout] (+)= sum over pixels of dy (the bias gradient, by the column-sum kernel).
int mdb_conv2d_wgrad_bias_f32(const float* dy, const float* x, const float* rowscale, float* dw_packed, float* db, int B, int H,
                              int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int accumulate, void* stream_) {
    return mdb_conv2d_wgrad_bias_dilated_f32(dy, x, rowscale, dw_packed, db, B, H, W, Cin, Cout, kh, kw, stride, pad, 1, accumulate,
                                             stream_);
}

}  // extern "C"

namespace {

// One weight-gradient launch of an undilated convolution between dy, a Wo x Ho pixel grid with pixel strides (dsx, dsy, dsb)
// elements, and x, a W x H grid with pixel strides (xsx, xsy, xsb): the whole tensors, or one lattice class of a dilated
// convolution (below).  Accumulates into dw_packed (zero-filled by the caller) with the kernel's vector reds.  band: the
// grouped form, dw_packed = the band-local [taps][Cout][128], only the diagonal (Cout tile, Cin tile) blocks computed.
int wgrad_launch(const float* dy, const float* x, const float* rowscale, float* dw_packed, int B, int Cin, int Cout, int kh,
                 int kw, int stride, int pad, int Wo, int Ho, uint64_t dsx, uint64_t dsy, uint64_t dsb, int W, int H, uint64_t xsx,
                 uint64_t xsy, uint64_t xsb, cudaStream_t stream, bool band = false) {
    const int taps = kh * kw;
    TcParams p;
    memset(&p, 0, sizeof(p));
    pick_tile(Wo, Ho, 32, &p.rtw, &p.rth);
    p.rtiles_x = (Wo + p.rtw - 1) / p.rtw;
    p.rtiles_y = (Ho + p.rth - 1) / p.rth;
    p.n_img = B;
    const int total_red = B * p.rtiles_x * p.rtiles_y;
    const int bn = 128;
    const int n_tiles_n = band ? 1 : (Cin + bn - 1) / bn;
    const int tiles = ((Cout + BM - 1) / BM) * n_tiles_n * taps;
    // split-K over pixel tiles.  Large problems: ~2 waves of CTAs, but at least ~24 reduction steps per CTA so the
    // 128 x BN atomic epilogue stays a small fraction of the work.  Small problems (decoder / head linears, M = 4400 rows
    // = 138 steps): the launch is latency-bound, so spread it over up to one wave with >= 8 steps per CTA (measured
    // 23 us -> ~10 us per launch, ~200 such launches per step).
    const int sms = num_sms();
    int big = (2 * sms + tiles - 1) / tiles, small = sms / tiles;
    if (big > total_red / 24) big = total_red / 24;
    if (small > total_red / 8) small = total_red / 8;
    int splits = big > small ? big : small;
    if (splits < 1 || mdb_get_deterministic()) splits = 1;      // reproducible mode: exactly one accumulation per output element
    p.red_per_split = (total_red + splits - 1) / splits;
    splits = (total_red + p.red_per_split - 1) / p.red_per_split;
    p.w_sy = p.w_sx = stride;
    p.wg_taps = taps; p.wg_kw = kw; p.wg_pad = pad;
    p.Mo_rows = Cout; p.No = band ? kBand : Cin; p.ldo = p.No; p.relu = 0; p.atomic_out = 1;
    p.bias = nullptr; p.residual = nullptr; p.relu_mask = nullptr; p.rowscale = rowscale;
    p.out = dw_packed;

    CUtensorMap ma, mb;
    int rc;
    {   // A (MN-major): dy as (Cout, Wo, Ho, B); box = 32 channels x (rtw x rth) reduction pixels
        uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)B};
        uint64_t str[4] = {1, dsx, dsy, dsb};
        uint32_t box[4] = {32, (uint32_t)p.rtw, (uint32_t)p.rth, 1};
        rc = make_map(&ma, dy, 4, dims, str, box, nullptr);
        if (rc) return rc;
    }
    {   // B (MN-major): x as (Cin, W, H, B) with element strides s
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
        uint64_t str[4] = {1, xsx, xsy, xsb};
        uint32_t box[4] = {32, (uint32_t)(p.rtw * stride), (uint32_t)(p.rth * stride), 1};
        uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
        rc = make_map(&mb, x, 4, dims, str, box, es);
        if (rc) return rc;
    }
    // The split partial tiles are added by the register epilogue's vector reds: a bulk tensor reduction of the staged
    // tile (cp.reduce.async.bulk.tensor) measured slower on the H100 at the model's small-M shapes.
    CUtensorMap mo, mr;
    memset(&mo, 0, sizeof(mo));
    memset(&mr, 0, sizeof(mr));
    dim3 grid(n_tiles_n, (Cout + BM - 1) / BM, taps * splits);
    if (band)
        return g_precision == 2 ? launch_tc<kBand, 4, 3, true, 2>(ma, mb, mo, mr, p, grid, stream)
               : g_precision == 1 ? launch_tc<kBand, 4, 3, true, 1>(ma, mb, mo, mr, p, grid, stream)
                                  : launch_tc<kBand, 5, 3, true, 0>(ma, mb, mo, mr, p, grid, stream);
    return g_precision == 2 ? launch_tc<128, 4, 1, true, 2>(ma, mb, mo, mr, p, grid, stream)
           : g_precision == 1 ? launch_tc<128, 4, 1, true, 1>(ma, mb, mo, mr, p, grid, stream)
                              : launch_tc<128, 5, 1, true, 0>(ma, mb, mo, mr, p, grid, stream);
}

// Weight gradient with the taps `dilation` pixels apart: x[b, oy*s + ky*d - pad, ox*s + kx*d - pad, ci].  d > 1 (stride 1)
// also needs pad % d == 0: output pixel (d*j + py, d*i + px) then reads x at (d*(j + ky - pad/d) + py, d*(i + kx - pad/d) + px),
// so the dilated weight gradient is the sum over the d*d lattice classes (py, px) of UNDILATED ones with padding pad/d
// between the class's pixels of dy and of x (pixel strides d).  The classes are launched one after another into the same dw
// (the kernel adds its partial sums anyway; in reproducible mode each launch has one writer per element, in a fixed order),
// and the kernel is the undilated one.  band: the grouped form (dw = band-local [taps][Cout][128]).
int wgrad_impl(const float* dy, const float* x, const float* rowscale, float* dw_packed, float* db, int B, int H, int W, int Cin,
               int Cout, int kh, int kw, int stride, int pad, int dilation, int accumulate, void* stream_, bool band) {
    ConvGeom g = make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation);
    int rc = check_geom(g);
    if (rc) return rc;
    if (pad % dilation) return MDB_EUNSUPPORTED;
    if (!dy || !x || !dw_packed) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (kh == 1 && stride == 1 && pad == 0) {     // pointwise: one long row of pixels (full 32-pixel reduction tiles)
        W = B * H * W; H = 1; B = 1;
        g = make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation);
    }
    const int taps = kh * kw;
    if (!accumulate) {
        cudaError_t e = cudaMemsetAsync(dw_packed, 0, sizeof(float) * (size_t)taps * Cout * (band ? kBand : Cin), stream);
        if (e != cudaSuccess) return (int)e;
    }
    if (db) {
        rc = mdb_colsum_f32(dy, db, (long long)B * g.Ho * g.Wo, Cout, accumulate, stream_);
        if (rc) return rc;
    }
    const int d = dilation;
    for (int py = 0; py < d; ++py)
        for (int px = 0; px < d; ++px) {
            const int Hc = (g.Ho - py + d - 1) / d, Wc = (g.Wo - px + d - 1) / d;   // the class's dy pixels
            const int Hx = (H - py + d - 1) / d, Wx = (W - px + d - 1) / d;         // the class's x pixels
            if (Hc <= 0 || Wc <= 0) continue;
            rc = wgrad_launch(dy + (size_t)(py * g.Wo + px) * Cout, x + (size_t)(py * W + px) * Cin, rowscale, dw_packed, B, Cin, Cout,
                              kh, kw, stride, pad / d, Wc, Hc, (uint64_t)d * Cout, (uint64_t)d * g.Wo * Cout,
                              (uint64_t)g.Ho * g.Wo * Cout, Wx, Hx, (uint64_t)d * Cin, (uint64_t)d * W * Cin, (uint64_t)H * W * Cin,
                              stream, band);
            if (rc) return rc;
        }
    return 0;
}

// ---- grouped weight layouts ----------------------------------------------------------------------------------------------
// OIHW (C, C/groups, 3, 3) <-> band-local [tap][row][128]: row r's 128 k positions are the channels of r's 128-channel band,
// zero outside r's group.  wf (forward): row = output channel, k = input channel; wd (dgrad): row = input channel, k = output
// channel.  fp32 layout [tap][C][128]; bf16x3 layout [tap][C][4][hi 32 | lo 32] (the pre-split rows of
// mdb_pack_gemm_weights_bf16x3).  The FrozenBN scale of the output channel is folded in before the split / rounding.
constexpr int kMaxGrouped = 64;
constexpr int kGroupedTaps = 9;
struct GroupedTable {
    const float* src[kMaxGrouped];
    const float* scale[kMaxGrouped];
    void* wf[kMaxGrouped];
    void* wd[kMaxGrouped];
    int C[kMaxGrouped], gc[kMaxGrouped];   // channels, channels per group
};

// value of band-local element (t, row, k) of wf (transposed == false) or wd (transposed == true)
__device__ __forceinline__ float grouped_elem(const float* __restrict__ w, const float* __restrict__ scale, int gc, bool transposed,
                                              int t, int row, int k) {
    const int c = (row / kBand) * kBand + k;                      // the other channel: input (wf) or output (wd)
    if (c / gc != row / gc) return 0.f;
    const int o = transposed ? c : row, i = transposed ? row : c;
    const float v = w[((size_t)o * gc + (i - (o / gc) * gc)) * kGroupedTaps + t];
    return scale ? v * scale[o] : v;
}

// one thread per pair of k positions; blockIdx.y = tensor
__global__ void pack_grouped_kernel(const __grid_constant__ GroupedTable tb, int bf, int round_tf32_out) {
    const int j = blockIdx.y;
    const int C = tb.C[j], gc = tb.gc[j];
    const long long n = (long long)kGroupedTaps * C * (kBand / 2);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int kp = (int)(i % (kBand / 2));
        const long long r = i / (kBand / 2);
        const int row = (int)(r % C), t = (int)(r / C);
        for (int which = 0; which < 2; ++which) {
            void* dst = which ? tb.wd[j] : tb.wf[j];
            if (!dst) continue;
            const float a = grouped_elem(tb.src[j], tb.scale[j], gc, which, t, row, 2 * kp);
            const float b = grouped_elem(tb.src[j], tb.scale[j], gc, which, t, row, 2 * kp + 1);
            if (bf) {   // row (t, row, k-block kp / 16): 16 words of hi, then 16 of lo
                const uint32_t h = pack_bf16x2(a, b);
                const uint32_t l = pack_bf16x2(a - __uint_as_float(h << 16), b - __uint_as_float(h & 0xFFFF0000u));
                uint32_t* out = static_cast<uint32_t*>(dst) + (r * (kBand / 32) + kp / 16) * 32;
                out[kp % 16] = h;
                out[16 + kp % 16] = l;
            } else {
                float2* out = static_cast<float2*>(dst) + i;
                *out = round_tf32_out ? make_float2(round_tf32(a), round_tf32(b)) : make_float2(a, b);
            }
        }
    }
}

// dw_oihw[o][j][t] = dw_band[t][o][(o / gc) * gc + j - band(o)]: the in-group entries only
__global__ void unpack_grouped_kernel(const __grid_constant__ GroupedTable tb) {
    const int j = blockIdx.y;
    const int C = tb.C[j], gc = tb.gc[j];
    const float* __restrict__ src = tb.src[j];
    float* __restrict__ dst = static_cast<float*>(tb.wf[j]);
    const long long n = (long long)C * gc * kGroupedTaps;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % kGroupedTaps);
        const long long r = i / kGroupedTaps;
        const int ci = (int)(r % gc), o = (int)(r / gc);
        dst[i] = src[((size_t)t * C + o) * kBand + (o / gc) * gc + ci - (o / kBand) * kBand];
    }
}

int grouped_table(int n, int base, const float* const* src, const float* const* scale, void* const* wf, void* const* wd,
                  const int* C, const int* groups, GroupedTable* tb, int* m) {
    *m = n - base < kMaxGrouped ? n - base : kMaxGrouped;
    for (int k = 0; k < *m; ++k) {
        const int j = base + k;
        if (!src[j] || !wf[j] || C[j] <= 0 || groups[j] <= 0) return MDB_EINVAL;
        if (C[j] % kBand || C[j] % groups[j] || kBand % (C[j] / groups[j])) return MDB_EUNSUPPORTED;
        tb->src[k] = src[j]; tb->scale[k] = scale ? scale[j] : nullptr;
        tb->wf[k] = wf[j]; tb->wd[k] = wd ? wd[j] : nullptr;
        tb->C[k] = C[j]; tb->gc[k] = C[j] / groups[j];
    }
    return 0;
}

int pack_grouped(int n, const float* const* w, const float* const* scale, void* const* wf, void* const* wd, const int* C,
                 const int* groups, bool bf, void* stream) {
    if (n < 0 || (n > 0 && (!w || !wf || !C || !groups))) return MDB_EINVAL;
    for (int base = 0; base < n; base += kMaxGrouped) {
        GroupedTable tb;
        int m;
        const int rc = grouped_table(n, base, w, scale, wf, wd, C, groups, &tb, &m);
        if (rc) return rc;
        pack_grouped_kernel<<<dim3(64, m), 256, 0, static_cast<cudaStream_t>(stream)>>>(tb, bf, !bf && g_precision == 0);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

}  // namespace

extern "C" {

int mdb_conv2d_wgrad_bias_dilated_f32(const float* dy, const float* x, const float* rowscale, float* dw_packed, float* db, int B,
                                      int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation,
                                      int accumulate, void* stream_) {
    return wgrad_impl(dy, x, rowscale, dw_packed, db, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, accumulate, stream_, false);
}

int mdb_conv2d_forward_grouped_f32(const float* x, const float* w_band, const float* bias, const float* residual, float* y, int B,
                                   int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation, int groups,
                                   int flags, void* stream) {
    const int rc = conv_grouped_check(make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation), groups, false);
    if (rc) return rc;
    return conv_forward_impl(x, w_band, false, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags, stream,
                             nullptr, true);
}
int mdb_conv2d_forward_grouped_bf16x3(const float* x, const void* w_band, const float* bias, const float* residual, float* y,
                                      int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation,
                                      int groups, int flags, void* stream) {
    const int rc = conv_grouped_check(make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation), groups, false);
    if (rc) return rc;
    return conv_forward_impl(x, w_band, true, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags, stream,
                             nullptr, true);
}
int mdb_conv2d_dgrad_grouped_f32(const float* dy, const float* w_band_t, const float* residual, const float* relu_mask, float* dx,
                                 int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation, int groups,
                                 int flags, void* stream) {
    const int rc = conv_grouped_check(make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation), groups, false);
    if (rc) return rc;
    return conv_dgrad_impl(dy, w_band_t, false, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags,
                           stream, true);
}
int mdb_conv2d_dgrad_grouped_bf16x3(const float* dy, const void* w_band_t, const float* residual, const float* relu_mask,
                                    float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                    int dilation, int groups, int flags, void* stream) {
    const int rc = conv_grouped_check(make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation), groups, false);
    if (rc) return rc;
    return conv_dgrad_impl(dy, w_band_t, true, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags,
                           stream, true);
}
int mdb_conv2d_wgrad_grouped_f32(const float* dy, const float* x, const float* rowscale, float* dw_band, int B, int H, int W,
                                 int Cin, int Cout, int kh, int kw, int stride, int pad, int dilation, int groups, int accumulate,
                                 void* stream) {
    const int rc = conv_grouped_check(make_geom(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation), groups, true);
    if (rc) return rc;
    return wgrad_impl(dy, x, rowscale, dw_band, nullptr, B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, accumulate, stream, true);
}
int mdb_pack_conv_weights_grouped_multi_f32(int n, const float* const* w_oihw, const float* const* scale, float* const* wf,
                                            float* const* wd, const int* C, const int* groups, void* stream) {
    return pack_grouped(n, w_oihw, scale, reinterpret_cast<void* const*>(wf), reinterpret_cast<void* const*>(wd), C, groups, false,
                        stream);
}
int mdb_pack_conv_weights_grouped_multi_bf16x3(int n, const float* const* w_oihw, const float* const* scale, void* const* wf,
                                               void* const* wd, const int* C, const int* groups, void* stream) {
    return pack_grouped(n, w_oihw, scale, wf, wd, C, groups, true, stream);
}
int mdb_unpack_conv_wgrads_grouped_multi_f32(int n, const float* const* dw_band, float* const* dw_oihw, const int* C,
                                             const int* groups, void* stream) {
    if (n < 0 || (n > 0 && (!dw_band || !dw_oihw || !C || !groups))) return MDB_EINVAL;
    for (int base = 0; base < n; base += kMaxGrouped) {
        GroupedTable tb;
        int m;
        const int rc = grouped_table(n, base, dw_band, nullptr, reinterpret_cast<void* const*>(dw_oihw), nullptr, C, groups, &tb, &m);
        if (rc) return rc;
        unpack_grouped_kernel<<<dim3(64, m), 256, 0, static_cast<cudaStream_t>(stream)>>>(tb);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

}  // extern "C"
