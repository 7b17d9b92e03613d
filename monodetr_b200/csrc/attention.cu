// attention.cu -- fused multi-head attention core (softmax(Q K^T / sqrt(d)) V, head dim 16, 32 or 64) for sm_90a,
// forward and backward, flash-style: the (Lq x Lk) probability matrix never touches HBM (the reference's
// nn.MultiheadAttention materialises it: 118 MB per image in the depth encoder, SURVEY.md 8a row a15).
// Replaces F.multi_head_attention_forward's core at depthaware_transformer.py:456-459 (depth cross-attn),
// :496 (group self-attn) and depth_predictor/transformer.py:59 (depth encoder).  The in/out projections
// are separate tensor-core GEMMs (conv_gemm.cu).
//
// Layout: q[b][i][h][HD] with token stride ldq floats (so a packed QKV buffer can be passed), same for
// k, v (ldk, ldv), out[b][i][h*HD] with token stride ldo.  The head width HD (16 / 32 / 64: nheads 16 / 8 / 4 at
// d_model 256) is a template parameter of every kernel; the entry points dispatch on head_dim.  key_padding_mask[b][j] (uint8, nonzero = ignore) or
// null.  Dropout on the probabilities uses a counter-based hash RNG keyed by (seed, site, b, h, i, j) so the backward
// pass regenerates the same mask.
//
// Mapping: warpgroup tensor-core tiles (wgmma m64nNk8 TF32, fp32 accumulate in registers).  A CTA is one warpgroup of
// 4 warps and owns 64 rows (queries, or keys in the dK/dV kernel); each warp owns 16 rows (its A fragments and
// accumulators have the m16n8k8 register layout) and the CTA streams 64-row tiles of the other operand through shared
// memory, stored in the 128-byte-swizzled K-major layouts the wgmma B descriptor reads (see unstage_tile).
// Scores (forward AND the recomputation in backward) use error-compensated 3xTF32 (hi/lo split in registers) so
// exp() sees fp32-accurate logits; P.V uses the same in the forward pass; the four gradient contractions of the
// backward pass are single-pass TF32 with round-to-nearest operands (measured 8e-4 of max|grad|).  The P (C-fragment) -> A-fragment hand-off needs no shuffles: the k index of the
// second GEMM is permuted (col t <-> key 2t, col t+4 <-> key 2t+1) and V/K/dO/Q rows are fetched in that order.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"
#include "rng.cuh"
#include "tc_common.cuh"

namespace {

using namespace mdb;

constexpr int BR = 64;             // rows per CTA (4 warps x 16)
constexpr int BC = 64;             // streamed tile rows
constexpr int ATT_THREADS = 128;
// One streamed operand tile in one wgmma layout, 1024-byte aligned: 8 KiB at head width 16 and 32, 16 KiB at 64.  At
// width 16 the NT layout keeps the 128-byte rows of width 32 with K zero-padded (the wgmmas read only its first 64
// bytes), so every width uses the one swizzle mode and descriptor.
template <int HD>
constexpr int kTileBytes = BC * (HD < 32 ? 32 : HD) * 4;

struct AttnParams {
    const float *q, *k, *v;
    const uint8_t* kpm;            // [B][Lk] or null
    float* out;
    float* lse;                    // [B][H][Lq]
    int B, H, Lq, Lk, ldq, ldk, ldv, ldo;
    float scale;                   // 1/sqrt(d)
    float drop_p;
    const unsigned long long* seed;
    unsigned long long site;
    const float *dout, *o;
    float* delta;                  // [B][H][Lq]
    float *dq, *dk, *dv;
    int lddq, lddk, lddv;
};

__device__ __forceinline__ uint32_t f2tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = f2tf32(x);
    lo = f2tf32(x - __uint_as_float(hi));
}
// A fragments (16 rows x HD cols) of a row-major global matrix: rows r0+g, r0+g+8; hi/lo split, optional scaling.
template <int HD>
struct AFrag {
    uint32_t hi[HD / 8][4];
    uint32_t lo[HD / 8][4];
};
template <int HD>
__device__ __forceinline__ void load_afrag(AFrag<HD>& f, const float* base, int ld, int r0, int nrows, int lane, float mul) {
    const int g = lane >> 2, t = lane & 3;
    const int ra = r0 + g, rb = r0 + g + 8;
    const float* pa = base + (size_t)min(ra, nrows - 1) * ld;
    const float* pb = base + (size_t)min(rb, nrows - 1) * ld;
    const float ma = ra < nrows ? mul : 0.f, mb = rb < nrows ? mul : 0.f;
#pragma unroll
    for (int ks = 0; ks < HD / 8; ++ks) {
        split_tf32(pa[ks * 8 + t] * ma, f.hi[ks][0], f.lo[ks][0]);
        split_tf32(pb[ks * 8 + t] * mb, f.hi[ks][1], f.lo[ks][1]);
        split_tf32(pa[ks * 8 + t + 4] * ma, f.hi[ks][2], f.lo[ks][2]);
        split_tf32(pb[ks * 8 + t + 4] * mb, f.hi[ks][3], f.lo[ks][3]);
    }
}

// Streamed tiles are stored PRE-SPLIT in shared memory (hi = rn_tf32(x), lo = rn_tf32(x - hi)) by the loader, once
// per element, in the layout(s) the tensor core reads them in:
//   NT  tile [64 rows][HD cols] as the K-major B operand of C = A . tile^T: row r = 128 bytes (32 cols), 16-byte chunk c
//       at c ^ (r & 7); at width 64 two such 8 KiB swizzle atoms along K (cols 0-31, then 32-63), at width 16 the
//       upper half of every row is padding that no wgmma reads
//   NN  tile as the K-major B operand of C = P . tile: tile^T, i.e. [HD cols][64 rows] as two halves of 32 rows (keys)
//       each (HD * 128 bytes), 128-byte rows, same swizzle; inside each 8-key step the keys are PERMUTED (k position
//       t <-> key 2t, t + 4 <-> key 2t + 1) so that P's accumulator fragments are A fragments as they stand (gemm_nn).
template <int HD>
__device__ __forceinline__ uint32_t nt_off(int r, int c) {
    if constexpr (HD == 64) return (uint32_t)((c >> 5) * (BC * 128)) + nt_off<32>(r, c & 31);
    else return (uint32_t)(r * 128 + ((((c >> 2) ^ (r & 7))) << 4) + (c & 3) * 4);
}
template <int HD>
__device__ __forceinline__ uint32_t nn_off(int r, int c) {
    const int kk = r & 31, q = kk & 7;
    const int kpos = (kk & ~7) + ((q & 1) ? 4 + (q >> 1) : (q >> 1));
    return (uint32_t)((r >> 5) * (HD * 128) + c * 128 + ((((kpos >> 2) ^ (c & 7))) << 4) + (kpos & 3) * 4);
}

// The m64nNk8 TF32 wgmma whose N is the accumulator's width (HD / 8 fragments of 4: N = HD).
__device__ __forceinline__ void wgmma_tf32(float (&d)[8], const uint32_t (&a)[4], uint64_t b, int sd) { wgmma_tf32_n16(d, a, b, sd); }
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], const uint32_t (&a)[4], uint64_t b, int sd) { wgmma_tf32_n32(d, a, b, sd); }
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], const uint32_t (&a)[4], uint64_t b, int sd) { wgmma_tf32_n64(d, a, b, sd); }

// C[64 x 64] = A[64 x HD] . T^T over the warpgroup (this warp: rows 16 w .. 16 w + 15), T = NT tile(s) at smem byte
// addresses th / tl.  NS = 3: error-compensated (A_lo T_hi + A_hi T_lo + A_hi T_hi).
template <int NS, int HD>
__device__ __forceinline__ void gemm_nt(float (&c)[8][4], const AFrag<HD>& a, uint32_t th, uint32_t tl) {
    float (&d)[32] = reinterpret_cast<float (&)[32]>(c);
#pragma unroll
    for (int i = 0; i < 32; ++i) d[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < HD / 8; ++ks) {
        const uint32_t off = (ks >> 2) * (BC * 128) + (ks & 3) * 32;    // swizzle atom along K, then 32 bytes per k-step
        const uint64_t bh = make_wgmma_desc_sw128(th + off);
        if (NS == 3) {
            const uint64_t bl = make_wgmma_desc_sw128(tl + off);
            wgmma_tf32_n64(d, a.lo[ks], bh, 1);
            wgmma_tf32_n64(d, a.hi[ks], bl, 1);
        }
        wgmma_tf32_n64(d, a.hi[ks], bh, 1);
    }
    wgmma_commit();
    wgmma_wait_all();
    wgmma_fence_operands(d);
}

// acc[64 x HD] += P[64 x 64] . T, P given as accumulator fragments (cols 2t, 2t+1 of each 8-wide block), T = NN tile(s).
// With the NN key permutation, A = (p0, p2, p1, p3) of each block.  The A fragments of four 8-key steps are split
// before their wgmmas are issued (registers an in-flight wgmma reads are not written).
template <int NS, int HD>
__device__ __forceinline__ void gemm_nn(float (&acc)[HD / 8][4], const float (&p)[8][4], uint32_t th, uint32_t tl) {
    float (&d)[HD / 2] = reinterpret_cast<float (&)[HD / 2]>(acc);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        uint32_t ah[4][4], al[4][4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int kt = half * 4 + u;
            split_tf32(p[kt][0], ah[u][0], al[u][0]);
            split_tf32(p[kt][2], ah[u][1], al[u][1]);
            split_tf32(p[kt][1], ah[u][2], al[u][2]);
            split_tf32(p[kt][3], ah[u][3], al[u][3]);
        }
        wgmma_fence();
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint32_t off = half * (HD * 128) + u * 32;      // keys 32 half + 8 u .. : half-tile, then 32 bytes per step
            const uint64_t bh = make_wgmma_desc_sw128(th + off);
            if (NS == 3) {
                const uint64_t bl = make_wgmma_desc_sw128(tl + off);
                wgmma_tf32(d, al[u], bh, 1);
                wgmma_tf32(d, ah[u], bl, 1);
            }
            wgmma_tf32(d, ah[u], bh, 1);
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_operands(d);
    }
}

// Streaming of a [64][HD] tile is software-pipelined with cp.async: stage_tile issues this thread's HD / 8 16-byte
// asynchronous copies of tile j+1 into a raw staging buffer right before the tensor-core work on tile j; after it,
// unstage_tile reads the same slots back (own copies only: cp.async.wait_all suffices, no barrier), splits them
// into hi (and lo) and writes the padded tiles.  The HBM/L2 latency hides behind the MMAs instead of stalling all
// four warps at the barrier (long-scoreboard was the top stall of the synchronous version)
// and no registers are held across the MMAs (a register-prefetch variant cost 57-80 registers and a CTA per SM).
template <int HD>
constexpr int STG = BC * HD;       // floats per staging buffer
template <int HD>
constexpr int kCopies = BC * HD / 4 / ATT_THREADS;   // 16-byte copies per thread and tile: 2 / 4 / 8
template <int HD>
constexpr int kRowShift = HD == 16 ? 2 : HD == 32 ? 3 : 4;       // log2(HD / 4): 16-byte chunks per tile row
template <int HD>
__device__ __forceinline__ void stage_tile(float* stg, const float* base, int ld, int r0, int nrows) {
#pragma unroll
    for (int u = 0; u < kCopies<HD>; ++u) {
        const int i = threadIdx.x + u * ATT_THREADS;
        const int r = i >> kRowShift<HD>, c = (i & (HD / 4 - 1)) * 4;
        const bool ok = r0 + r < nrows;
        const float* src = ok ? base + ((size_t)(r0 + r) * ld + c) : base;
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(stg) + (uint32_t)i * 16u;
        const int nbytes = ok ? 16 : 0;                              // 0 -> the 16 bytes are zero-filled
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(nbytes) : "memory");
    }
}
__device__ __forceinline__ void stage_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void stage_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// Split the staged fp32 tile into hi (and lo) and write it in the NT and / or NN layout; null pointers are skipped.  The
// caller orders these generic-proxy writes before the tensor core's reads (fence_proxy_async_smem + barrier).
template <int HD>
__device__ __forceinline__ void unstage_tile(uint8_t* nt_hi, uint8_t* nt_lo, uint8_t* nn_hi, uint8_t* nn_lo, const float* stg) {
#pragma unroll
    for (int u = 0; u < kCopies<HD>; ++u) {
        const int i = threadIdx.x + u * ATT_THREADS;
        const int r = i >> kRowShift<HD>, c = (i & (HD / 4 - 1)) * 4;
        const float4 v = *reinterpret_cast<const float4*>(stg + i * 4);
        uint32_t h[4], l[4];
        split_tf32(v.x, h[0], l[0]); split_tf32(v.y, h[1], l[1]); split_tf32(v.z, h[2], l[2]); split_tf32(v.w, h[3], l[3]);
        if (nt_hi) *reinterpret_cast<uint4*>(nt_hi + nt_off<HD>(r, c)) = make_uint4(h[0], h[1], h[2], h[3]);
        if (nt_lo) *reinterpret_cast<uint4*>(nt_lo + nt_off<HD>(r, c)) = make_uint4(l[0], l[1], l[2], l[3]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            if (nn_hi) *reinterpret_cast<uint32_t*>(nn_hi + nn_off<HD>(r, c + e)) = h[e];
            if (nn_lo) *reinterpret_cast<uint32_t*>(nn_lo + nn_off<HD>(r, c + e)) = l[e];
        }
    }
}
static_assert(BC * (16 / 4) == kCopies<16> * ATT_THREADS && BC * (32 / 4) == kCopies<32> * ATT_THREADS &&
              BC * (64 / 4) == kCopies<64> * ATT_THREADS, "tile loader mapping");

__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Dropout on the probabilities: keep(b, h, i, j) = fmix32-hash of (i * Lk + j) keyed per (seed, site, b, h); the
// same pure function in all three kernels.  Host check: Lq * Lk < 2^32.
struct DropCtx {
    uint32_t key, thr;
    float inv_keep;
    bool on;
};
__device__ __forceinline__ DropCtx make_drop(const AttnParams& p, int b, int h) {
    DropCtx d;
    d.on = p.drop_p > 0.f;
    d.inv_keep = 1.f / (1.f - p.drop_p);
    d.thr = mdb::rng_thr16(p.drop_p);
    d.key = 0u;
    if (d.on) d.key = mdb::rng_key32(*p.seed + p.site * 0x9E3779B97F4A7C15ull, (unsigned long long)(b * p.H + h));
    return d;
}
__device__ __forceinline__ float keep_scale(const DropCtx& d, uint32_t row_base, int j) {   // row_base = i * Lk
    return mdb::rng_keep16(d.key, row_base + (uint32_t)j, d.thr) ? d.inv_keep : 0.f;
}

// ---------------------------------------------------------------------------------------------------------
// dead-key flags of the streamed tile (key_padding_mask or past the end), fetched with the tile and read from smem
__device__ __forceinline__ uint32_t fetch_dead(const AttnParams& p, int b, int k0) {
    const int j = k0 + (int)threadIdx.x;
    if (threadIdx.x >= BC) return 0u;
    if (j >= p.Lk) return 1u;
    return (p.kpm && p.kpm[(size_t)b * p.Lk + j]) ? 1u : 0u;
}

// CTAs per SM the forward and dQ kernels are compiled for: 3 at widths 16 and 32.  At width 64 a CTA takes 96 KiB of
// shared memory, so no more than 2 fit on an SM anyway, and the register cap of 3 (168) would spill the 64-column
// Q (and dO) fragments.
template <int HD>
constexpr int kRowMinBlocks = HD == 64 ? 2 : 3;

template <int HD>
__global__ void __launch_bounds__(ATT_THREADS, kRowMinBlocks<HD>)
attn_fwd_kernel(const AttnParams p) {
    constexpr int TB = kTileBytes<HD>;
    extern __shared__ __align__(1024) uint8_t dyn_smem[];           // kFwdSmem bytes: 4 operand tiles, 2 staging buffers, flags
    uint8_t* sKh = dyn_smem;                                        // NT hi / lo
    uint8_t* sKl = sKh + TB;
    uint8_t* sVh = sKl + TB;                                        // NN hi / lo
    uint8_t* sVl = sVh + TB;
    float* gK = reinterpret_cast<float*>(sVl + TB);
    float* gV = gK + STG<HD>;
    uint8_t* sDead = reinterpret_cast<uint8_t*>(gV + STG<HD>);
    const int b = blockIdx.z, h = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = blockIdx.x * BR + warp * 16;
    const float* qb = p.q + (size_t)b * p.Lq * p.ldq + h * HD;
    const float* kb = p.k + (size_t)b * p.Lk * p.ldk + h * HD;
    const float* vb = p.v + (size_t)b * p.Lk * p.ldv + h * HD;
    const DropCtx drop = make_drop(p, b, h);
    stage_tile<HD>(gK, kb, p.ldk, 0, p.Lk);
    stage_tile<HD>(gV, vb, p.ldv, 0, p.Lk);
    stage_commit();
    uint32_t ndead = fetch_dead(p, b, 0);
    AFrag<HD> qa;
    load_afrag(qa, qb, p.ldq, r0, p.Lq, lane, p.scale);
    float acc[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;      // rows g and g+8
    const int qi0 = r0 + g, qi1 = r0 + g + 8;
    const uint32_t rb0 = (uint32_t)qi0 * (uint32_t)p.Lk, rb1 = (uint32_t)qi1 * (uint32_t)p.Lk;

    for (int k0 = 0; k0 < p.Lk; k0 += BC) {
        stage_wait();
        __syncthreads();                       // every warp is done with the previous tiles
        unstage_tile<HD>(sKh, sKl, nullptr, nullptr, gK);
        unstage_tile<HD>(nullptr, nullptr, sVh, sVl, gV);
        if (threadIdx.x < BC) sDead[threadIdx.x] = (uint8_t)ndead;
        mdb::fence_proxy_async_smem();
        __syncthreads();
        if (k0 + BC < p.Lk) {                  // next tile's copies fly during this tile's MMAs
            stage_tile<HD>(gK, kb, p.ldk, k0 + BC, p.Lk);
            stage_tile<HD>(gV, vb, p.ldv, k0 + BC, p.Lk);
            stage_commit();
            ndead = fetch_dead(p, b, k0 + BC);
        }
        float s[8][4];
        gemm_nt<3, HD>(s, qa, mdb::smem_u32(sKh), mdb::smem_u32(sKl));
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const uchar2 dd = *reinterpret_cast<const uchar2*>(&sDead[nt * 8 + 2 * t]);
            if (dd.x) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
            if (dd.y) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
            mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
            mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
        }
        const float mn0 = fmaxf(m0, quad_max(mx0)), mn1 = fmaxf(m1, quad_max(mx1));
        const float c0 = (mn0 == -INFINITY) ? 1.f : __expf(m0 - mn0), c1 = (mn1 == -INFINITY) ? 1.f : __expf(m1 - mn1);
        l0 *= c0; l1 *= c1;
#pragma unroll
        for (int dn = 0; dn < HD / 8; ++dn) { acc[dn][0] *= c0; acc[dn][1] *= c0; acc[dn][2] *= c1; acc[dn][3] *= c1; }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int j = k0 + nt * 8 + 2 * t + e;
                float p0 = (mn0 == -INFINITY) ? 0.f : __expf(s[nt][e] - mn0);
                float p1 = (mn1 == -INFINITY) ? 0.f : __expf(s[nt][2 + e] - mn1);
                l0 += p0; l1 += p1;
                if (drop.on) {
                    p0 *= keep_scale(drop, rb0, j);
                    p1 *= keep_scale(drop, rb1, j);
                }
                s[nt][e] = p0; s[nt][2 + e] = p1;
            }
        }
        m0 = mn0; m1 = mn1;
        gemm_nn<3, HD>(acc, s, mdb::smem_u32(sVh), mdb::smem_u32(sVl));
    }
    l0 = quad_sum(l0); l1 = quad_sum(l1);
    const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    float* ob = p.out + (size_t)b * p.Lq * p.ldo + h * HD;
#pragma unroll
    for (int dn = 0; dn < HD / 8; ++dn) {
        if (qi0 < p.Lq) *reinterpret_cast<float2*>(ob + (size_t)qi0 * p.ldo + dn * 8 + 2 * t) = make_float2(acc[dn][0] * i0, acc[dn][1] * i0);
        if (qi1 < p.Lq) *reinterpret_cast<float2*>(ob + (size_t)qi1 * p.ldo + dn * 8 + 2 * t) = make_float2(acc[dn][2] * i1, acc[dn][3] * i1);
    }
    if (t == 0) {
        float* lp = p.lse + ((size_t)b * p.H + h) * p.Lq;
        if (qi0 < p.Lq) lp[qi0] = l0 > 0.f ? m0 + __logf(l0) : -INFINITY;
        if (qi1 < p.Lq) lp[qi1] = l1 > 0.f ? m1 + __logf(l1) : -INFINITY;
    }
}

// delta[b][h][i] = dO_i . O_i
template <int HD>
__global__ void attn_delta_kernel(const AttnParams p) {
    const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;   // one thread per (b, i, h)
    const long long n = (long long)p.B * p.Lq * p.H;
    if (idx >= n) return;
    const int h = (int)(idx % p.H);
    const long long bi = idx / p.H;
    const int i = (int)(bi % p.Lq);
    const int b = (int)(bi / p.Lq);
    const float* a = p.dout + (size_t)bi * p.ldo + h * HD;
    const float* o = p.o + (size_t)bi * p.ldo + h * HD;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < HD; d += 4) {
        const float4 x = *reinterpret_cast<const float4*>(a + d);
        const float4 y = *reinterpret_cast<const float4*>(o + d);
        s += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
    }
    p.delta[((size_t)b * p.H + h) * p.Lq + i] = s;
}

// dQ: CTA = 64 queries, streams key/value tiles.
// At width 64 the Q and dO fragments are re-read from global memory (L1 / L2) for every key tile, as the dK / dV kernel
// does with K and V.  Held across the loop (as at widths 16 and 32), the compiled width-64 kernel reused the dO
// fragment's registers inside the loop and dQ came out wrong on an H100; with no loop-carried fragments it matches the
// float64 reference (tests/test_attention_heads_gpu.py).
template <int HD>
__global__ void __launch_bounds__(ATT_THREADS, kRowMinBlocks<HD>)
attn_bwd_dq_kernel(const AttnParams p) {
    constexpr int TB = kTileBytes<HD>;
    constexpr bool kReloadQG = HD == 64;
    extern __shared__ __align__(1024) uint8_t dyn_smem[];           // kDqSmem bytes
    uint8_t* sKh = dyn_smem;                                        // K: NT hi / lo, NN hi; V: NT hi
    uint8_t* sKl = sKh + TB;
    uint8_t* sKn = sKl + TB;
    uint8_t* sVh = sKn + TB;
    float* gK = reinterpret_cast<float*>(sVh + TB);
    float* gV = gK + STG<HD>;
    uint8_t* sDead = reinterpret_cast<uint8_t*>(gV + STG<HD>);
    const int b = blockIdx.z, h = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = blockIdx.x * BR + warp * 16;
    const float* qb = p.q + (size_t)b * p.Lq * p.ldq + h * HD;
    const float* gb = p.dout + (size_t)b * p.Lq * p.ldo + h * HD;
    const float* kb = p.k + (size_t)b * p.Lk * p.ldk + h * HD;
    const float* vb = p.v + (size_t)b * p.Lk * p.ldv + h * HD;
    const DropCtx drop = make_drop(p, b, h);
    stage_tile<HD>(gK, kb, p.ldk, 0, p.Lk);
    stage_tile<HD>(gV, vb, p.ldv, 0, p.Lk);
    stage_commit();
    uint32_t ndead = fetch_dead(p, b, 0);
    AFrag<HD> qa, ga;
    if constexpr (!kReloadQG) {
        load_afrag(qa, qb, p.ldq, r0, p.Lq, lane, p.scale);
        load_afrag(ga, gb, p.ldo, r0, p.Lq, lane, 1.f);
    }
    const int qi0 = r0 + g, qi1 = r0 + g + 8;
    const uint32_t rb0 = (uint32_t)qi0 * (uint32_t)p.Lk, rb1 = (uint32_t)qi1 * (uint32_t)p.Lk;
    const size_t st = ((size_t)b * p.H + h) * p.Lq;
    // lse = -inf (fully masked row) or a row past the end: +inf makes every p = exp(s - lse) exactly 0
    float lse0 = qi0 < p.Lq ? p.lse[st + qi0] : INFINITY, lse1 = qi1 < p.Lq ? p.lse[st + qi1] : INFINITY;
    if (lse0 == -INFINITY) lse0 = INFINITY;
    if (lse1 == -INFINITY) lse1 = INFINITY;
    const float dl0 = qi0 < p.Lq ? p.delta[st + qi0] : 0.f, dl1 = qi1 < p.Lq ? p.delta[st + qi1] : 0.f;
    float acc[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;

    for (int k0 = 0; k0 < p.Lk; k0 += BC) {
        stage_wait();
        __syncthreads();
        unstage_tile<HD>(sKh, sKl, sKn, nullptr, gK);
        unstage_tile<HD>(sVh, nullptr, nullptr, nullptr, gV);
        if (threadIdx.x < BC) sDead[threadIdx.x] = (uint8_t)ndead;
        mdb::fence_proxy_async_smem();
        __syncthreads();
        if (k0 + BC < p.Lk) {
            stage_tile<HD>(gK, kb, p.ldk, k0 + BC, p.Lk);
            stage_tile<HD>(gV, vb, p.ldv, k0 + BC, p.Lk);
            stage_commit();
            ndead = fetch_dead(p, b, k0 + BC);
        }
        if constexpr (kReloadQG) {
            load_afrag(qa, qb, p.ldq, r0, p.Lq, lane, p.scale);
            load_afrag(ga, gb, p.ldo, r0, p.Lq, lane, 1.f);
        }
        float s[8][4], dp[8][4];
        gemm_nt<3, HD>(s, qa, mdb::smem_u32(sKh), mdb::smem_u32(sKl));
        gemm_nt<1, HD>(dp, ga, mdb::smem_u32(sVh), 0u);   // gradients: single-pass TF32 with round-to-nearest operands
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const uchar2 dd = *reinterpret_cast<const uchar2*>(&sDead[nt * 8 + 2 * t]);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int j = k0 + nt * 8 + 2 * t + e;
                const bool dead = e ? dd.y : dd.x;
                float p0 = dead ? 0.f : __expf(s[nt][e] - lse0);
                float p1 = dead ? 0.f : __expf(s[nt][2 + e] - lse1);
                float d0 = dp[nt][e], d1 = dp[nt][2 + e];
                if (drop.on) {
                    d0 *= keep_scale(drop, rb0, j);
                    d1 *= keep_scale(drop, rb1, j);
                }
                s[nt][e] = p0 * (d0 - dl0);
                s[nt][2 + e] = p1 * (d1 - dl1);
            }
        }
        gemm_nn<1, HD>(acc, s, mdb::smem_u32(sKn), 0u);
    }
    float* ob = p.dq + (size_t)b * p.Lq * p.lddq + h * HD;
#pragma unroll
    for (int dn = 0; dn < HD / 8; ++dn) {
        if (qi0 < p.Lq) *reinterpret_cast<float2*>(ob + (size_t)qi0 * p.lddq + dn * 8 + 2 * t) = make_float2(acc[dn][0] * p.scale, acc[dn][1] * p.scale);
        if (qi1 < p.Lq) *reinterpret_cast<float2*>(ob + (size_t)qi1 * p.lddq + dn * 8 + 2 * t) = make_float2(acc[dn][2] * p.scale, acc[dn][3] * p.scale);
    }
}

// dK / dV: CTA = 64 keys, streams query tiles (Q, dO, lse, delta).  At width 64 the K and V fragments (96 registers)
// are re-read from global memory (L1 / L2) for every query tile rather than held across the loop: held, they would
// need more than the 255 registers a thread has beside the dK / dV accumulators and the S / dP tiles.
template <int HD>
__global__ void __launch_bounds__(ATT_THREADS, 2)
attn_bwd_dkv_kernel(const AttnParams p) {
    constexpr int TB = kTileBytes<HD>;
    constexpr bool kReloadKV = HD == 64;
    extern __shared__ __align__(1024) uint8_t dyn_smem[];           // kDkvSmem bytes
    uint8_t* sQh = dyn_smem;                                        // Q: NT hi / lo, NN hi; dO: NT hi, NN hi
    uint8_t* sQl = sQh + TB;
    uint8_t* sQn = sQl + TB;
    uint8_t* sGh = sQn + TB;
    uint8_t* sGn = sGh + TB;
    float* gQ = reinterpret_cast<float*>(sGn + TB);
    float* gG = gQ + STG<HD>;
    float* sL = gG + STG<HD>;
    float* sD = sL + BC;
    const int b = blockIdx.z, h = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = blockIdx.x * BR + warp * 16;                      // first key row of this warp
    const float* qb = p.q + (size_t)b * p.Lq * p.ldq + h * HD;
    const float* gb = p.dout + (size_t)b * p.Lq * p.ldo + h * HD;
    const float* kb = p.k + (size_t)b * p.Lk * p.ldk + h * HD;
    const float* vb = p.v + (size_t)b * p.Lk * p.ldv + h * HD;
    const DropCtx drop = make_drop(p, b, h);
    const size_t st = ((size_t)b * p.H + h) * p.Lq;
    // per-thread row statistics of the streamed query tile (threads 0..63): lse (+inf -> p = 0) and delta
    auto fetch_stats = [&](int q0, float& l, float& d) {
        const int i = q0 + (int)threadIdx.x;
        l = INFINITY; d = 0.f;
        if (threadIdx.x < BC && i < p.Lq) {
            l = p.lse[st + i];
            d = p.delta[st + i];
            if (l == -INFINITY) l = INFINITY;
        }
    };
    float nl, nd;
    stage_tile<HD>(gQ, qb, p.ldq, 0, p.Lq);
    stage_tile<HD>(gG, gb, p.ldo, 0, p.Lq);
    stage_commit();
    fetch_stats(0, nl, nd);
    AFrag<HD> ka, va;
    if constexpr (!kReloadKV) {
        load_afrag(ka, kb, p.ldk, r0, p.Lk, lane, p.scale);
        load_afrag(va, vb, p.ldv, r0, p.Lk, lane, 1.f);
    }
    const int kj0 = r0 + g, kj1 = r0 + g + 8;
    const bool dead0 = kj0 >= p.Lk || (p.kpm && p.kpm[(size_t)b * p.Lk + min(kj0, p.Lk - 1)]);
    const bool dead1 = kj1 >= p.Lk || (p.kpm && p.kpm[(size_t)b * p.Lk + min(kj1, p.Lk - 1)]);
    float dk[HD / 8][4], dv[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
        dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
        dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
    }

    for (int q0 = 0; q0 < p.Lq; q0 += BC) {
        stage_wait();
        __syncthreads();
        unstage_tile<HD>(sQh, sQl, sQn, nullptr, gQ);
        unstage_tile<HD>(sGh, nullptr, sGn, nullptr, gG);
        if (threadIdx.x < BC) { sL[threadIdx.x] = nl; sD[threadIdx.x] = nd; }
        mdb::fence_proxy_async_smem();
        __syncthreads();
        if (q0 + BC < p.Lq) {
            stage_tile<HD>(gQ, qb, p.ldq, q0 + BC, p.Lq);
            stage_tile<HD>(gG, gb, p.ldo, q0 + BC, p.Lq);
            stage_commit();
            fetch_stats(q0 + BC, nl, nd);
        }
        if constexpr (kReloadKV) {
            load_afrag(ka, kb, p.ldk, r0, p.Lk, lane, p.scale);
            load_afrag(va, vb, p.ldv, r0, p.Lk, lane, 1.f);
        }
        float s[8][4], dp[8][4];
        gemm_nt<3, HD>(s, ka, mdb::smem_u32(sQh), mdb::smem_u32(sQl));   // S^T[key][query] (already scaled through K)
        gemm_nt<1, HD>(dp, va, mdb::smem_u32(sGh), 0u);                  // dP^T[key][query] = V . dO^T
        float pd[8][4];                        // dropped probabilities for dV
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const float2 l2 = *reinterpret_cast<const float2*>(&sL[nt * 8 + 2 * t]);
            const float2 d2 = *reinterpret_cast<const float2*>(&sD[nt * 8 + 2 * t]);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int i = q0 + nt * 8 + 2 * t + e;
                const float lse = e ? l2.y : l2.x, dl = e ? d2.y : d2.x;
                float p0 = dead0 ? 0.f : __expf(s[nt][e] - lse);
                float p1 = dead1 ? 0.f : __expf(s[nt][2 + e] - lse);
                float d0 = dp[nt][e], d1 = dp[nt][2 + e];
                float w0 = p0, w1 = p1;
                if (drop.on) {
                    const uint32_t rb = (uint32_t)i * (uint32_t)p.Lk;
                    const float k0s = keep_scale(drop, rb, kj0), k1s = keep_scale(drop, rb, kj1);
                    w0 *= k0s; w1 *= k1s; d0 *= k0s; d1 *= k1s;
                }
                pd[nt][e] = w0; pd[nt][2 + e] = w1;
                s[nt][e] = p0 * (d0 - dl);
                s[nt][2 + e] = p1 * (d1 - dl);
            }
        }
        gemm_nn<1, HD>(dv, pd, mdb::smem_u32(sGn), 0u);   // dV += P^T_dropped . dO
        gemm_nn<1, HD>(dk, s, mdb::smem_u32(sQn), 0u);    // dK += dS^T . Q
    }
    float* dkb = p.dk + (size_t)b * p.Lk * p.lddk + h * HD;
    float* dvb = p.dv + (size_t)b * p.Lk * p.lddv + h * HD;
#pragma unroll
    for (int dn = 0; dn < HD / 8; ++dn) {
        if (kj0 < p.Lk) {
            *reinterpret_cast<float2*>(dkb + (size_t)kj0 * p.lddk + dn * 8 + 2 * t) = make_float2(dk[dn][0] * p.scale, dk[dn][1] * p.scale);
            *reinterpret_cast<float2*>(dvb + (size_t)kj0 * p.lddv + dn * 8 + 2 * t) = make_float2(dv[dn][0], dv[dn][1]);
        }
        if (kj1 < p.Lk) {
            *reinterpret_cast<float2*>(dkb + (size_t)kj1 * p.lddk + dn * 8 + 2 * t) = make_float2(dk[dn][2] * p.scale, dk[dn][3] * p.scale);
            *reinterpret_cast<float2*>(dvb + (size_t)kj1 * p.lddv + dn * 8 + 2 * t) = make_float2(dv[dn][2], dv[dn][3]);
        }
    }
}

template <int HD>
constexpr int kFwdSmem = 4 * kTileBytes<HD> + 2 * STG<HD> * 4 + BC;
template <int HD>
constexpr int kDqSmem = 4 * kTileBytes<HD> + 2 * STG<HD> * 4 + BC;
template <int HD>
constexpr int kDkvSmem = 5 * kTileBytes<HD> + 2 * STG<HD> * 4 + 2 * BC * 4;

int check(const AttnParams& p) {
    if (p.B <= 0 || p.H <= 0 || p.Lq <= 0 || p.Lk <= 0) return MDB_EINVAL;
    if ((p.ldq | p.ldk | p.ldv | p.ldo) % 4) return MDB_EINVAL;
    if (p.drop_p < 0.f || p.drop_p >= 1.f) return MDB_EINVAL;
    if (p.drop_p > 0.f && !p.seed) return MDB_EINVAL;
    if (p.H > 65535 || p.B > 65535) return MDB_EUNSUPPORTED;
    if ((unsigned long long)p.Lq * (unsigned long long)p.Lk >= (1ull << 32)) return MDB_EUNSUPPORTED;   // 32-bit mask index
    return 0;
}

template <int HD>
int launch_forward(const AttnParams& p, cudaStream_t stream) {
    dim3 grid((p.Lq + BR - 1) / BR, p.H, p.B);
    const cudaError_t e = set_max_dynamic_smem(attn_fwd_kernel<HD>, kFwdSmem<HD>);
    if (e != cudaSuccess) return (int)e;
    attn_fwd_kernel<HD><<<grid, ATT_THREADS, kFwdSmem<HD>, stream>>>(p);
    return (int)cudaGetLastError();
}

template <int HD>
int launch_backward(const AttnParams& p, cudaStream_t stream) {
    const long long n = (long long)p.B * p.Lq * p.H;
    attn_delta_kernel<HD><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p);
    cudaError_t e = set_max_dynamic_smem(attn_bwd_dq_kernel<HD>, kDqSmem<HD>);
    if (e == cudaSuccess) e = set_max_dynamic_smem(attn_bwd_dkv_kernel<HD>, kDkvSmem<HD>);
    if (e != cudaSuccess) return (int)e;
    attn_bwd_dq_kernel<HD><<<dim3((p.Lq + BR - 1) / BR, p.H, p.B), ATT_THREADS, kDqSmem<HD>, stream>>>(p);
    attn_bwd_dkv_kernel<HD><<<dim3((p.Lk + BR - 1) / BR, p.H, p.B), ATT_THREADS, kDkvSmem<HD>, stream>>>(p);
    return (int)cudaGetLastError();
}

bool supported_head_dim(int head_dim) { return head_dim == 16 || head_dim == 32 || head_dim == 64; }

}  // namespace

extern "C" {

int mdb_attention_forward_f32(const float* q, const float* k, const float* v, const unsigned char* key_padding_mask,
                              float* out, float* lse, int B, int H, int Lq, int Lk, int head_dim, int ldq, int ldk,
                              int ldv, int ldo, float drop_p, const unsigned long long* seed, unsigned long long site,
                              void* stream) {
    if (!supported_head_dim(head_dim)) return MDB_EUNSUPPORTED;
    if (!q || !k || !v || !out || !lse) return MDB_EINVAL;
    AttnParams p{};
    p.q = q; p.k = k; p.v = v; p.kpm = key_padding_mask; p.out = out; p.lse = lse;
    p.B = B; p.H = H; p.Lq = Lq; p.Lk = Lk; p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
    p.scale = 1.f / sqrtf((float)head_dim); p.drop_p = drop_p; p.seed = seed; p.site = site;
    int rc = check(p);
    if (rc) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (head_dim == 16) return launch_forward<16>(p, s);
    if (head_dim == 64) return launch_forward<64>(p, s);
    return launch_forward<32>(p, s);
}

int mdb_attention_backward_f32(const float* q, const float* k, const float* v, const unsigned char* key_padding_mask,
                               const float* out, const float* lse, const float* dout, float* delta_ws, float* dq,
                               float* dk, float* dv, int B, int H, int Lq, int Lk, int head_dim, int ldq, int ldk, int ldv,
                               int ldo, int lddq, int lddk, int lddv, float drop_p, const unsigned long long* seed,
                               unsigned long long site, void* stream_) {
    if (!supported_head_dim(head_dim)) return MDB_EUNSUPPORTED;
    if (!q || !k || !v || !out || !lse || !dout || !delta_ws || !dq || !dk || !dv) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    AttnParams p{};
    p.q = q; p.k = k; p.v = v; p.kpm = key_padding_mask; p.lse = const_cast<float*>(lse);
    p.B = B; p.H = H; p.Lq = Lq; p.Lk = Lk; p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
    p.scale = 1.f / sqrtf((float)head_dim); p.drop_p = drop_p; p.seed = seed; p.site = site;
    p.dout = dout; p.o = out; p.delta = delta_ws; p.dq = dq; p.dk = dk; p.dv = dv;
    p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
    int rc = check(p);
    if (rc) return rc;
    if ((lddq | lddk | lddv) % 4) return MDB_EINVAL;
    if (head_dim == 16) return launch_backward<16>(p, stream);
    if (head_dim == 64) return launch_backward<64>(p, stream);
    return launch_backward<32>(p, stream);
}

}  // extern "C"
