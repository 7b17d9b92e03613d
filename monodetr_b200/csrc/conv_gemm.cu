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
// warpgroups (64 rows each: operand staging, wgmma, fused epilogue straight from the accumulator registers), warp 8 =
// TMA producer.  smem ring of STAGES stages, mbarrier full/empty pairs.
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
constexpr int kThreadsTC = kConsumerThreads + 32;
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

// Persistent, warp-specialised kernel.  Each CTA walks tiles  tile = blockIdx.x + i * gridDim.x.
//   warp 8          TMA producer (smem ring of STAGES stages, full/empty mbarriers)
//   warps 0-7       two consumer warpgroups; warpgroup g owns rows [64g, 64g+64) of the 128-row tile.  Per k-block each
//                   thread loads its A fragments from the landed fp32 tile and splits them in registers; B is read by the
//                   tensor core from shared memory, either as delivered (pre-split bf16 weights) or after the consumers
//                   have rewritten it into a K-major operand tile (see CONVB).
// PREC (arithmetic):
//   2  bf16x3: x = hi + lo with hi = bf16(x), lo = bf16(x - hi); per k-block A_hi*B_hi + A_lo*B_hi + A_hi*B_lo as
//      m64nBNk16 bf16 wgmma.  In fprop / dgrad the B operand arrives PRE-SPLIT from global memory -- packed weights
//      [tap][n][k-block][hi 32 | lo 32] bf16, one 128-byte swizzle row per (n, k-block), written once per step by
//      pack_gemm_weights_bf16x3.  Dropped terms are O(2^-17) per product.
//   1  3xTF32: hi = trunc_tf32(x), lo = x - hi; the same three products as m64nBNk8 tf32 wgmma.
//   0  single-pass TF32 (operands truncated by the tensor core; outputs optionally rounded for the next consumer).
template <int BN, int STAGES, int MODE /*0 fprop/dgrad, 1 wgrad*/, bool B_MN, int PREC>
__global__ void __launch_bounds__(kThreadsTC, 1)
tc_conv_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                    const __grid_constant__ TcParams p) {
    constexpr bool A_MN = (MODE == 1);
    static_assert(!(MODE == 1) || B_MN, "wgrad reads both operands MN-major");
    static_assert(BN == 64 || BN == 128, "tile width");
    constexpr bool BF_B = (PREC == 2 && MODE == 0);               // B arrives as pre-split bf16 rows
    static_assert(!BF_B || !B_MN, "pre-split weights are K-major");
    constexpr bool CONVB = !BF_B;                                 // consumers rewrite B into the operand tile(s)
    constexpr int kTileBBytes = BN * 128;
    constexpr int kRawBytes = kTileABytes + kTileBBytes;          // what TMA delivers per stage
    constexpr int kConvBytes = CONVB ? (PREC == 1 ? 2 : 1) * kTileBBytes : 0;
    constexpr int NACC = BN / 2;

    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* bconv = smem + STAGES * kRawBytes;                   // [hi | lo] operand tiles of the current k-block (CONVB)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(bconv + kConvBytes);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // ---- tile decode (identical in every role) -----------------------------------------------------
    struct Tile { int n0, img, y0, x0, m0, red_begin, iters, tap, slice; };
    auto decode = [&](int tix) {
        Tile t;
        t.n0 = (tix % p.n_tiles_n) * BN;
        int r = tix / p.n_tiles_n;
        t.img = t.y0 = t.x0 = t.m0 = t.red_begin = t.tap = t.slice = 0;
        if constexpr (MODE == 0) {
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
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kConsumerThreads / 32);      // one arrival per consumer warp
        }
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

    if (warp == kConsumerThreads / 32) {
        // ================================ TMA producer =============================================
        if (elect_one()) {
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
                    if constexpr (MODE == 0) {
                        const int kit = t.red_begin + it;                 // (fprop split-K: this slice's first k-block)
                        const int tap = kit / p.cblocks;
                        const int cb = kit - tap * p.cblocks;
                        tma_load_4d(a_dst, &mapA, &full_bar[s], cb * BK, t.x0 * p.in_sx + p.tap_dx[tap],
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
                            tma_load_4d(b_dst + j * kChunkBytes, &mapB, &full_bar[s], t.n0 + j * 32,
                                        rx * p.w_sx + (t.tap % p.wg_kw) - p.wg_pad, ry * p.w_sy + (t.tap / p.wg_kw) - p.wg_pad, ri);
                    }
                }
            }
        }
        return;
    }
    if (warp > kConsumerThreads / 32) return;

    // ==================================== consumer warpgroups ==========================================
    const int wg = warp >> 2;
    const int g = lane >> 2, tig = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g;                 // this thread's tile rows: r0 and r0 + 8
    const int ctid = threadIdx.x;                                 // 0..255
    int git = 0;
    for (int tix = blockIdx.x; tix < p.total_tiles; tix += gridDim.x) {
        const Tile t = decode(tix);
        if (p.atomic_out && t.iters == 0) continue;              // nothing to add
        float acc[NACC];
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        for (int it = 0; it < t.iters; ++it, ++git) {
            const int s = git % STAGES;
            const uint32_t ph = (git / STAGES) & 1;
            mbar_wait(&full_bar[s], ph);
            const uint8_t* a_raw = smem + s * kRawBytes;
            const uint8_t* b_raw = a_raw + kTileABytes;
            if constexpr (CONVB) {
                // Every consumer has waited for its MMAs of the previous k-block: the operand tile(s) may be rewritten.
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
                        uint8_t* brow = bconv + n * 128;
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
                        *reinterpret_cast<float4*>(bconv + off) = h;
                        if constexpr (PREC == 1)
                            *reinterpret_cast<float4*>(bconv + kTileBBytes + off) = make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
                    }
                }
                fence_proxy_async_smem();      // generic-proxy writes -> visible to the tensor core's async-proxy reads
                named_bar_sync(1, kConsumerThreads);
            }
            const uint32_t b_addr = smem_u32(CONVB ? bconv : b_raw);
            // All A fragments of the k-block are loaded and split before the first wgmma: registers an in-flight wgmma
            // reads must not be written until it completes.
            constexpr int KS = PREC == 2 ? 2 : 4;                 // k-steps per k-block: 16 bf16 or 8 tf32 each
            uint32_t ahi[KS][4], alo[KS][4];
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
                        ahi[ks][f] = h;
                        alo[ks][f] = pack_bf16x2(x0 - __uint_as_float(h << 16), x1 - __uint_as_float(h & 0xFFFF0000u));
                    } else {
                        // fragment f: rows + 8 * (f & 1), k = tig + 4 * (f >> 1) of this 8-wide step
                        const int k = ks * 8 + tig + (f >> 1) * 4;
                        const float x = *reinterpret_cast<const float*>(a_raw + raw_off<A_MN>(row, k));
                        const float h = trunc_tf32(x);
                        ahi[ks][f] = __float_as_uint(h);
                        alo[ks][f] = __float_as_uint(x - h);
                    }
                }
            }
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
                // B hi at byte 32 * ks of each 128-byte row; bf16 lo at 64 + 32 * ks, tf32 lo in the second tile
                const uint64_t bhi = make_wgmma_desc_sw128(b_addr + ks * 32);
                const uint64_t blo = make_wgmma_desc_sw128(b_addr + (PREC == 2 ? 64 : kTileBBytes) + ks * 32);
                if constexpr (PREC == 2) {
                    if constexpr (BN == 128) {
                        wgmma_bf16_n128(acc, ahi[ks], bhi, 1);
                        wgmma_bf16_n128(acc, alo[ks], bhi, 1);
                        wgmma_bf16_n128(acc, ahi[ks], blo, 1);
                    } else {
                        wgmma_bf16_n64(acc, ahi[ks], bhi, 1);
                        wgmma_bf16_n64(acc, alo[ks], bhi, 1);
                        wgmma_bf16_n64(acc, ahi[ks], blo, 1);
                    }
                } else {
                    if constexpr (BN == 128) wgmma_tf32_n128(acc, ahi[ks], bhi, 1);
                    else wgmma_tf32_n64(acc, ahi[ks], bhi, 1);
                    if constexpr (PREC == 1) {
                        if constexpr (BN == 128) {
                            wgmma_tf32_n128(acc, alo[ks], bhi, 1);
                            wgmma_tf32_n128(acc, ahi[ks], blo, 1);
                        } else {
                            wgmma_tf32_n64(acc, alo[ks], bhi, 1);
                            wgmma_tf32_n64(acc, ahi[ks], blo, 1);
                        }
                    }
                }
            }
            wgmma_commit();
            wgmma_wait_all();
            wgmma_fence_operands(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[s]);            // this warp is done with the stage
        }

        // ---- epilogue: accumulator registers -> fused bias / residual / ReLU / mask / row-scale -> global ------------
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + h * 8;
            bool ok;
            size_t roff;
            float rsc = 1.f;
            if constexpr (MODE == 0) {
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
template <int BN, int STAGES, int MODE, bool B_MN, int PREC>
int launch_tc(const CUtensorMap& a, const CUtensorMap& b, TcParams p, dim3 grid, cudaStream_t stream) {
    constexpr bool convb = !(PREC == 2 && MODE == 0);
    constexpr int smem = STAGES * (kTileABytes + BN * 128) + (convb ? (PREC == 1 ? 2 : 1) * BN * 128 : 0) +
                         1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(smem <= 227 * 1024, "dynamic shared memory budget");
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
        return (int)cudaLaunchKernelEx(&cfg, kern, a, b, p);
    }
    kern<<<ctas, kThreadsTC, smem, stream>>>(a, b, p);
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

// Launch the fprop / dgrad kernel (K-major B operand) for the arithmetic mode.
int launch_fwd(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& p, dim3 grid, int bn, int precision, cudaStream_t stream) {
    if (precision == 2) return bn == 64 ? launch_tc<64, 6, 0, false, 2>(ma, mb, p, grid, stream) : launch_tc<128, 5, 0, false, 2>(ma, mb, p, grid, stream);
    if (precision == 1) return bn == 64 ? launch_tc<64, 5, 0, false, 1>(ma, mb, p, grid, stream) : launch_tc<128, 4, 0, false, 1>(ma, mb, p, grid, stream);
    return bn == 64 ? launch_tc<64, 6, 0, false, 0>(ma, mb, p, grid, stream) : launch_tc<128, 5, 0, false, 0>(ma, mb, p, grid, stream);
}

struct ConvGeom {
    int B, H, W, Cin, Cout, kh, kw, stride, pad, Ho, Wo;
};

int check_geom(const ConvGeom& g, bool forward = false) {
    if (g.B <= 0 || g.H <= 0 || g.W <= 0 || g.Cin <= 0 || g.Cout <= 0) return MDB_EINVAL;
    if (g.kh != g.kw || (g.kh != 1 && g.kh != 3) || (g.stride != 1 && g.stride != 2)) return MDB_EUNSUPPORTED;
    // TMA needs 16-byte row pitches on every operand it reads: Cin always; Cout only where dy / the output map is an
    // operand (dgrad, wgrad).  The forward epilogue writes ragged Cout with scalar stores.
    if (g.Cin % 4 || (!forward && g.Cout % 4)) return MDB_EUNSUPPORTED;
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
int conv_forward_impl(const float* x, const void* w_packed, bool bf, const float* bias, const float* residual, float* y,
                      int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int flags,
                      void* stream_, size_t* query_ws = nullptr /* non-null: only report the scratch bytes this call needs */) {
    const int precision = bf ? 2 : (g_precision == 2 ? 1 : g_precision);   // fp32 weights in bf16x3 mode: 3xTF32
    ConvGeom g{B, H, W, Cin, Cout, kh, kw, stride, pad, (H + 2 * pad - kh) / stride + 1, (W + 2 * pad - kw) / stride + 1};
    int rc = check_geom(g, true);
    if (rc) return rc;
    if (!query_ws && (!x || !w_packed || !y)) return MDB_EINVAL;
    if ((unsigned long long)B * g.Ho * g.Wo * Cout >= (1ull << 31)) return MDB_EUNSUPPORTED;   // the epilogue indexes with (signed) 32 bits
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (kh == 1 && stride == 1 && pad == 0) {     // pointwise: the batch of images is one long row of pixels (no tile waste)
        W = B * H * W; H = 1; B = 1;
        g = ConvGeom{B, H, W, Cin, Cout, kh, kw, stride, pad, H, W};
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
    p.cblocks = (Cin + BK - 1) / BK;
    for (int ky = 0; ky < kh; ++ky)
        for (int kx = 0; kx < kw; ++kx) {
            const int t = ky * kw + kx;
            p.tap_dy[t] = ky - pad; p.tap_dx[t] = kx - pad; p.tap_w[t] = t;
        }
    p.wg_taps = 1; p.wg_kw = 1;
    p.No = Cout; p.ldo = Cout; p.relu = flags & 1; p.round_out = (precision == 0) ? ((flags >> 1) & 1) : 0; p.atomic_out = 0;
    p.bias = bias; p.residual = residual; p.relu_mask = nullptr; p.rowscale = nullptr; p.out = y;

    const int bn = Cout <= 64 ? 64 : 128;
    dim3 grid((Cout + bn - 1) / bn, n_groups * p.tiles_x * p.tiles_y, 1);
    const long long out_elems = (long long)B * g.Ho * g.Wo * Cout;
    const int slices = ((reinterpret_cast<uintptr_t>(bias) & 15u) == 0)
                           ? forward_splitk_slices(precision, p.ntaps * p.cblocks, bn, !residual && !p.relu, Cout, out_elems)
                           : 0;
    if (query_ws) {
        *query_ws = sizeof(float) * (size_t)out_elems * slices;
        return 0;
    }

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
    } else {   // B: packed weights as (Cin, Cout, taps), box (32, BN, 1)
        uint64_t dims[3] = {(uint64_t)Cin, (uint64_t)Cout, (uint64_t)(kh * kw)};
        uint64_t str[3] = {1, (uint64_t)Cin, (uint64_t)Cout * Cin};
        uint32_t box[3] = {BK, (uint32_t)bn, 1};
        rc = make_map(&mb, w_packed, 3, dims, str, box, nullptr);
        if (rc) return rc;
    }
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
            rc = launch_fwd(ma, mb, p, grid, 128, precision, stream);
            if (rc) return rc;
            const long long n4 = out_elems / 4;
            splitk_reduce_kernel<<<grid_cap(n4, 256, num_sms() * 8), 256, 0, stream>>>(
                reinterpret_cast<const float4*>(ws), reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(y), n4, Cout / 4, slices, n4);
            return (int)cudaGetLastError();
        }
    }
    return launch_fwd(ma, mb, p, grid, bn, precision, stream);
}

// dx[B,H,W,Cin] = (conv_transpose(dy[B,Ho,Wo,Cout], w) + residual) * (relu_mask > 0);  w = fp32 packed [taps][Cout][Cin]
// (read MN-major) or, bf == true, the pre-split TRANSPOSED bf16 form [taps][Cin][ceil(Cout/32)][hi 32 | lo 32] (K-major).
int conv_dgrad_impl(const float* dy, const void* w_packed, bool bf, const float* residual, const float* relu_mask,
                    float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                    int flags, void* stream_) {
    const int precision = bf ? 2 : (g_precision == 2 ? 1 : g_precision);
    ConvGeom g{B, H, W, Cin, Cout, kh, kw, stride, pad, (H + 2 * pad - kh) / stride + 1, (W + 2 * pad - kw) / stride + 1};
    int rc = check_geom(g);
    if (rc) return rc;
    if (!dy || !w_packed || !dx) return MDB_EINVAL;
    if ((unsigned long long)B * H * W * Cin >= (1ull << 31)) return MDB_EUNSUPPORTED;           // the epilogue indexes with (signed) 32 bits
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (kh == 1 && stride == 1 && pad == 0) {     // pointwise: one long row of pixels
        W = B * H * W; H = 1; B = 1;
        g = ConvGeom{B, H, W, Cin, Cout, kh, kw, stride, pad, H, W};
    }
    // dx[y,x] = sum_{ky,kx} dy[(y+pad-ky)/s, (x+pad-kx)/s] * W[ky,kx]  where the division is exact.
    // Per output parity class (py,px) (only one class for s == 1) the contributing taps are fixed and the
    // dy access is a unit-stride shifted box: oy = (y + pad - ky)/s = j + (py + pad - ky)/s  for y = s*j + py.
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
            p.cblocks = (Cout + BK - 1) / BK;
            int nt = 0;
            for (int ky = 0; ky < kh; ++ky) {
                if ((py + pad - ky) % stride) continue;
                for (int kx = 0; kx < kw; ++kx) {
                    if ((px + pad - kx) % stride) continue;
                    // floor division is exact here (numerator divisible by stride; may be negative)
                    p.tap_dy[nt] = (py + pad - ky) / stride;
                    p.tap_dx[nt] = (px + pad - kx) / stride;
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
            const int bn = (bf && Cin <= 64) ? 64 : 128;
            if (bf) {   // B (K-major): transposed pre-split weights as (64 * k-blocks, Cin, taps); box (64, BN, 1)
                const uint64_t kb = (uint64_t)p.cblocks;
                uint64_t dims[3] = {64 * kb, (uint64_t)Cin, (uint64_t)(kh * kw)};
                uint64_t str[3] = {1, 64 * kb, (uint64_t)Cin * 64 * kb};
                uint32_t box[3] = {64, (uint32_t)bn, 1};
                rc = make_map(&mb, w_packed, 3, dims, str, box, nullptr, true);
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
            if (bf) rc = launch_fwd(ma, mb, p, grid, bn, 2, stream);
            else rc = (precision == 1) ? launch_tc<128, 4, 0, true, 1>(ma, mb, p, grid, stream)
                                       : launch_tc<128, 5, 0, true, 0>(ma, mb, p, grid, stream);
            if (rc) return rc;
        }
    return 0;
}

}  // namespace

extern "C" {

int mdb_conv2d_forward_f32(const float* x, const float* w_packed, const float* bias, const float* residual, float* y,
                           int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int flags,
                           void* stream) {
    return conv_forward_impl(x, w_packed, false, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, flags, stream);
}
int mdb_conv2d_forward_bf16x3(const float* x, const void* w_split, const float* bias, const float* residual, float* y,
                              int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad, int flags,
                              void* stream) {
    return conv_forward_impl(x, w_split, true, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, flags, stream);
}
long long mdb_conv2d_forward_workspace_bytes(int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                                             int flags, int has_residual, int split_weights) {
    size_t bytes = 0;
    const float* res = has_residual ? reinterpret_cast<const float*>(16) : nullptr;
    const int rc = conv_forward_impl(nullptr, nullptr, split_weights != 0, nullptr, res, nullptr, B, H, W, Cin, Cout, kh, kw, stride,
                                     pad, flags, nullptr, &bytes);
    return rc ? (long long)rc : (long long)bytes;
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
    return conv_dgrad_impl(dy, w_packed, false, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, flags, stream);
}
int mdb_conv2d_dgrad_bf16x3(const float* dy, const void* w_split_t, const float* residual, const float* relu_mask,
                            float* dx, int B, int H, int W, int Cin, int Cout, int kh, int kw, int stride, int pad,
                            int flags, void* stream) {
    return conv_dgrad_impl(dy, w_split_t, true, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, flags, stream);
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
    ConvGeom g{B, H, W, Cin, Cout, kh, kw, stride, pad, (H + 2 * pad - kh) / stride + 1, (W + 2 * pad - kw) / stride + 1};
    int rc = check_geom(g);
    if (rc) return rc;
    if (!dy || !x || !dw_packed) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (kh == 1 && stride == 1 && pad == 0) {     // pointwise: one long row of pixels (full 32-pixel reduction tiles)
        W = B * H * W; H = 1; B = 1;
        g = ConvGeom{B, H, W, Cin, Cout, kh, kw, stride, pad, H, W};
    }
    const int taps = kh * kw;
    if (!accumulate) {
        cudaError_t e = cudaMemsetAsync(dw_packed, 0, sizeof(float) * (size_t)taps * Cout * Cin, stream);
        if (e != cudaSuccess) return (int)e;
    }
    if (db) {
        rc = mdb_colsum_f32(dy, db, (long long)B * g.Ho * g.Wo, Cout, accumulate, stream_);
        if (rc) return rc;
    }
    TcParams p;
    memset(&p, 0, sizeof(p));
    pick_tile(g.Wo, g.Ho, 32, &p.rtw, &p.rth);
    p.rtiles_x = (g.Wo + p.rtw - 1) / p.rtw;
    p.rtiles_y = (g.Ho + p.rth - 1) / p.rth;
    p.n_img = B;
    const int total_red = B * p.rtiles_x * p.rtiles_y;
    const int bn = 128;
    const int tiles = ((Cout + BM - 1) / BM) * ((Cin + bn - 1) / bn) * taps;
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
    p.Mo_rows = Cout; p.No = Cin; p.ldo = Cin; p.relu = 0; p.atomic_out = 1;
    p.bias = nullptr; p.residual = nullptr; p.relu_mask = nullptr; p.rowscale = rowscale;
    p.out = dw_packed;

    CUtensorMap ma, mb;
    {   // A (MN-major): dy as (Cout, Wo, Ho, B); box = 32 channels x (rtw x rth) reduction pixels
        uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)g.Wo, (uint64_t)g.Ho, (uint64_t)B};
        uint64_t str[4] = {1, (uint64_t)Cout, (uint64_t)g.Wo * Cout, (uint64_t)g.Ho * g.Wo * Cout};
        uint32_t box[4] = {32, (uint32_t)p.rtw, (uint32_t)p.rth, 1};
        rc = make_map(&ma, dy, 4, dims, str, box, nullptr);
        if (rc) return rc;
    }
    {   // B (MN-major): x as (Cin, W, H, B) with element strides s
        uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
        uint64_t str[4] = {1, (uint64_t)Cin, (uint64_t)W * Cin, (uint64_t)H * W * Cin};
        uint32_t box[4] = {32, (uint32_t)(p.rtw * stride), (uint32_t)(p.rth * stride), 1};
        uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
        rc = make_map(&mb, x, 4, dims, str, box, es);
        if (rc) return rc;
    }
    dim3 grid((Cin + bn - 1) / bn, (Cout + BM - 1) / BM, taps * splits);
    rc = g_precision == 2 ? launch_tc<128, 4, 1, true, 2>(ma, mb, p, grid, stream)
         : g_precision == 1 ? launch_tc<128, 4, 1, true, 1>(ma, mb, p, grid, stream)
                            : launch_tc<128, 5, 1, true, 0>(ma, mb, p, grid, stream);
    if (rc) return rc;
    return 0;
}

}  // extern "C"
