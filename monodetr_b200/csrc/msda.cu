// msda.cu -- multi-scale deformable attention gather (forward) and scatter (backward) for sm_90a.
//
// Replaces the reference kernels ms_deformable_im2col_gpu_kernel / ms_deformable_col2im_gpu_kernel_*
// (lib/models/monodetr/ops/src/cuda/ms_deform_im2col_cuda.cuh:237-299, 301-403) and their host
// launchers (ms_deform_attn_cuda.cu:20-153).  Math: SURVEY.md appendix A.
//
// Data layout (all contiguous, owned by the caller):
//   value  [B][S][M][D]      one (pixel, head) row is D floats = 128 B for D=32 -> one cache line
//   loc    [B][Lq][M][L][P][2], attn [B][Lq][M][L][P], out [B][Lq][M*D]
//
// Fast path (fp32, D in {16,32,64}, P in {2,4,8}, L <= 8): a "unit" is one (b, q, m).  D/4 lanes own a
// unit, each lane owns 4 channels, so every bilinear corner is ONE 16-byte load per lane and one
// fully coalesced 128-byte line per unit; a warp carries 32/(D/4) units = consecutive heads of one
// query, so its output store is one contiguous 512-byte run.  All 16 corner loads of a level are
// issued before use (ILP), sample coordinates are broadcast loads.
// The backward pass keeps the same mapping, re-gathers the corners, scatters w*g*A with vector
// reductions (red.global.add.v4.f32) and reduces d/dloc, d/dattn across the D/4 lanes with a
// butterfly transpose-reduction (42 shuffles per unit instead of 144).
//
// Generic path (any D/L/P, fp32 and fp64): one warp per unit, lanes stride over channels.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

using namespace mdb;

constexpr int kMaxLevels = 8;
constexpr int kThreads = 256;

struct LevelInfo {
    int H[kMaxLevels];
    int W[kMaxLevels];
    int start[kMaxLevels];
};

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d)
                 : "memory");
}

__device__ __forceinline__ float fma_t(float a, float b, float c) { return fmaf(a, b, c); }
__device__ __forceinline__ double fma_t(double a, double b, double c) { return fma(a, b, c); }
__device__ __forceinline__ float floor_t(float a) { return floorf(a); }
__device__ __forceinline__ double floor_t(double a) { return floor(a); }

// Coordinates and attention weights of N consecutive points (N = 2: one 16-byte and one 8-byte load; N = 4: three 16-byte
// loads).  lp / ap are 16- / 4N-byte aligned: the unit's rows are, and a level holds a multiple of N points.
template <int N>
__device__ __forceinline__ void load_points(const float* lp, const float* ap, float (&xs)[N], float (&ys)[N], float (&as)[N]) {
    if constexpr (N == 2) {
        const float4 xy = ldg4(lp);
        const float2 a2 = __ldg(reinterpret_cast<const float2*>(ap));
        xs[0] = xy.x; xs[1] = xy.z; ys[0] = xy.y; ys[1] = xy.w; as[0] = a2.x; as[1] = a2.y;
    } else {
        static_assert(N == 4, "2 or 4 points per load");
        const float4 xy01 = ldg4(lp);
        const float4 xy23 = ldg4(lp + 4);
        const float4 a4 = ldg4(ap);
        xs[0] = xy01.x; xs[1] = xy01.z; xs[2] = xy23.x; xs[3] = xy23.z;
        ys[0] = xy01.y; ys[1] = xy01.w; ys[2] = xy23.y; ys[3] = xy23.w;
        as[0] = a4.x; as[1] = a4.y; as[2] = a4.z; as[3] = a4.w;
    }
}

// ------------------------------------------------------------------------------------------------
// Fast forward: LPU lanes per unit, D = 4*LPU, P in {2, 4, 8} (the corners of up to 4 points in flight at a time).
// ------------------------------------------------------------------------------------------------
// Work distribution: every CTA owns one CONTIGUOUS range of units (= consecutive queries; in the encoder that is a
// strip of horizontally adjacent pixels), and its 8 warps walk it side by side, so that the bilinear footprints of
// neighbouring queries are re-read from the SM's L1 instead of L2 (an interleaved grid-stride walk spreads a strip over
// all SMs and gets ~35 % L1 hits; the contiguous walk reuses a line across ~8 neighbouring queries).
template <int LPU, int P>
__device__ __forceinline__ void
msda_fwd_vec(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const int64_t* __restrict__ lsi, const float* __restrict__ loc,
                    const float* __restrict__ attn, int S, int M, int L, int Lq, long long n_units,
                    long long units_per_block, float* __restrict__ out) {
    static_assert(P == 2 || P == 4 || P == 8, "fast path: 2, 4 or 8 points");
    constexpr int D = 4 * LPU;
    constexpr int UPW = 32 / LPU;
    constexpr int PG = P < 4 ? P : 4;      // points whose corners are in flight together (register budget)
    __shared__ LevelInfo lv;
    if (threadIdx.x < L) {
        lv.H[threadIdx.x] = (int)shapes[2 * threadIdx.x];
        lv.W[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
        lv.start[threadIdx.x] = (int)lsi[threadIdx.x];
    }
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const int sub = lane / LPU;
    const int cl = lane % LPU;
    const int wib = threadIdx.x >> 5;
    const int pix = M * D;  // floats between horizontally adjacent pixels
    const long long u_begin = (long long)blockIdx.x * units_per_block;
    const long long u_end = min(n_units, u_begin + units_per_block);

    for (long long unit = u_begin + wib * UPW + sub; unit < u_end; unit += (kThreads / 32) * UPW) {
        const int m = (int)(unit % M);
        const int b = (int)(unit / ((long long)Lq * M));
        const float* vb = value + ((size_t)b * S * M + m) * D + cl * 4;
        const float* lp = loc + (size_t)unit * L * P * 2;
        const float* ap = attn + (size_t)unit * L * P;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);

#pragma unroll
        for (int l = 0; l < kMaxLevels; ++l) {
            if (l >= L) break;
            const int H = lv.H[l], W = lv.W[l];
            const float fW = (float)W, fH = (float)H;
            const float* vl = vb + (size_t)lv.start[l] * pix;
#pragma unroll
            for (int p0 = 0; p0 < P; p0 += PG) {
                float xs[PG], ys[PG], as[PG];
                load_points<PG>(lp + l * 2 * P + 2 * p0, ap + l * P + p0, xs, ys, as);
                const int rowf = W * pix;           // floats between vertically adjacent pixels (fits int: host check)
                float4 v[PG][4];
                float w[PG][4];
#pragma unroll
                for (int p = 0; p < PG; ++p) {
                    const float x = fmaf(xs[p], fW, -0.5f);
                    const float y = fmaf(ys[p], fH, -0.5f);
                    const bool inside = (y > -1.f) && (x > -1.f) && (y < fH) && (x < fW);
                    const float xf = floorf(x), yf = floorf(y);
                    const int x0 = (int)xf, y0 = (int)yf;
                    // off the image the weights multiply zeros, so they must stay finite (x - floor(x) is NaN for x = +-inf, NaN)
                    const float lx = inside ? x - xf : 0.f, ly = inside ? y - yf : 0.f, hx = 1.f - lx, hy = 1.f - ly;
                    const bool top = inside && (y0 >= 0), bot = inside && (y0 + 1 <= H - 1);
                    const bool lef = (x0 >= 0), rig = (x0 + 1 <= W - 1);
                    const float* p00 = vl + (y0 * W + x0) * pix;      // only dereferenced when the predicate holds
                    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                    v[p][0] = (top && lef) ? ldg4(p00) : z;
                    v[p][1] = (top && rig) ? ldg4(p00 + pix) : z;
                    v[p][2] = (bot && lef) ? ldg4(p00 + rowf) : z;
                    v[p][3] = (bot && rig) ? ldg4(p00 + rowf + pix) : z;
                    const float a = as[p];
                    w[p][0] = a * (hy * hx);
                    w[p][1] = a * (hy * lx);
                    w[p][2] = a * (ly * hx);
                    w[p][3] = a * (ly * lx);
                }
#pragma unroll
                for (int p = 0; p < PG; ++p) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        acc.x = fmaf(w[p][k], v[p][k].x, acc.x);
                        acc.y = fmaf(w[p][k], v[p][k].y, acc.y);
                        acc.z = fmaf(w[p][k], v[p][k].z, acc.z);
                        acc.w = fmaf(w[p][k], v[p][k].w, acc.w);
                    }
                }
            }
        }
        *reinterpret_cast<float4*>(out + (size_t)unit * D + cl * 4) = acc;
    }
}

// ------------------------------------------------------------------------------------------------
// Forward, D = 32 (8 lanes per unit), L = 4, P in {2, 4, 8}: "distributed point set-up".  The L*P sample points of a unit
// need ~45 integer/float instructions each (coordinates, floor, clamping, 4 corner weights, offsets); doing that in
// all 8 lanes of the unit made the kernel issue-bound.  Here lane c of the unit prepares points c, c+8, ... (L*P/8 of them) and
// the 7 resulting words per point are broadcast inside the octet with width-8 shuffles; corners outside the image are
// redirected to a clamped (valid) address with weight 0, so no load is predicated and all 16 LDG.128 of a level
// stay in flight.
// ------------------------------------------------------------------------------------------------
struct PointSetup {
    int o00, dxo, dyo;      // float offset of corner (y0,x0) inside the (b, m) slice; +dxo -> x0+1, +dyo -> y0+1
    float w[4];             // attention * bilinear weight per corner, 0 for corners outside the image
};

__device__ __forceinline__ PointSetup setup_point(float lx_, float ly_, float a, int H, int W, int start, int pix) {
    PointSetup s;
    const float fW = (float)W, fH = (float)H;
    const float x = fmaf(lx_, fW, -0.5f), y = fmaf(ly_, fH, -0.5f);
    const bool inside = (y > -1.f) && (x > -1.f) && (y < fH) && (x < fW);
    const float xf = floorf(x), yf = floorf(y);
    const int x0 = inside ? (int)xf : 0, y0 = inside ? (int)yf : 0;
    const float lx = x - xf, ly = y - yf, hx = 1.f - lx, hy = 1.f - ly;
    const bool top = inside && (y0 >= 0), bot = inside && (y0 + 1 <= H - 1);
    const bool lef = (x0 >= 0), rig = (x0 + 1 <= W - 1);
    const int xc0 = max(x0, 0), yc0 = max(y0, 0);
    const int xc1 = min(x0 + 1, W - 1), yc1 = min(y0 + 1, H - 1);
    s.o00 = (start + yc0 * W + xc0) * pix;
    s.dxo = (max(xc1, xc0) - xc0) * pix;
    s.dyo = (max(yc1, yc0) - yc0) * W * pix;
    s.w[0] = (top && lef) ? a * (hy * hx) : 0.f;
    s.w[1] = (top && rig) ? a * (hy * lx) : 0.f;
    s.w[2] = (bot && lef) ? a * (ly * hx) : 0.f;
    s.w[3] = (bot && rig) ? a * (ly * lx) : 0.f;
    return s;
}

// FUSED: `loc` / `attn` are the RAW projections of the module (sampling offsets (.., L, P, 2) and attention logits (.., L*P)) and
// the pre-processing of ops/modules/ms_deform_attn.py:145-155 happens here: the softmax over the unit's L*P logits costs L*P/8
// exponentials per lane and six width-8 shuffles, the location arithmetic one divide / FMA per coordinate -- the separate
// pre-processing kernel and its 125 MB round trip through HBM (encoder call, B = 8, P = 4) disappear.
// P in {2, 4, 8}: lane c of the unit prepares points h * 8 + c (h < L*P/8), i.e. (level h*8/P + c/P, point c % P).
template <bool FUSED, int P>
__device__ __forceinline__ void
msda_fwd_d32(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const int64_t* __restrict__ lsi, const float* __restrict__ loc,
                    const float* __restrict__ attn, const float* __restrict__ ref, int ref_dim, int S, int M, int Lq,
                    long long n_units, long long units_per_block, float* __restrict__ out) {
    static_assert(P == 2 || P == 4 || P == 8, "2, 4 or 8 points");
    constexpr int L = 4, D = 32, UPW = 4;
    constexpr int NH = L * P / 8;          // points each lane prepares
    __shared__ LevelInfo lv;
    if (threadIdx.x < L) {
        lv.H[threadIdx.x] = (int)shapes[2 * threadIdx.x];
        lv.W[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
        lv.start[threadIdx.x] = (int)lsi[threadIdx.x];
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int sub = lane >> 3, cl = lane & 7;
    const int wib = threadIdx.x >> 5;
    const int pix = M * D;
    const long long u_begin = (long long)blockIdx.x * units_per_block;
    const long long u_end = min(((n_units + UPW - 1) / UPW) * UPW, u_begin + units_per_block);   // multiple of 4: warps stay converged
    // levels of this lane's first two points (P = 8: the level of point h is h, read from shared memory)
    const int lA = cl / P, lB = NH == 2 ? 8 / P + cl / P : lA;      // (lB is unused unless NH == 2)
    const int HA = lv.H[lA], WA = lv.W[lA], sA = lv.start[lA];
    const int HB = lv.H[lB], WB = lv.W[lB], sB = lv.start[lB];

    for (long long unit = u_begin + wib * UPW + sub; unit < u_end; unit += (kThreads / 32) * UPW) {
        const bool live = unit < n_units;
        const long long u = live ? unit : 0;
        const int m = (int)(u % M);
        const int b = (int)(u / ((long long)Lq * M));
        const float* vb = value + ((size_t)b * S * M + m) * D + cl * 4;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        [[maybe_unused]] float e[NH];
        if constexpr (FUSED) {                 // softmax over the unit's L*P logits: this lane holds logits h * 8 + cl
#pragma unroll
            for (int h = 0; h < NH; ++h) e[h] = __ldg(attn + (size_t)u * (L * P) + h * 8 + cl);
            float mx = e[0];
#pragma unroll
            for (int h = 1; h < NH; ++h) mx = fmaxf(mx, e[h]);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4, 8));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2, 8));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1, 8));
#pragma unroll
            for (int h = 0; h < NH; ++h) e[h] = expf(e[h] - mx);
            float sum = e[0];
#pragma unroll
            for (int h = 1; h < NH; ++h) sum += e[h];
            sum += __shfl_xor_sync(0xffffffffu, sum, 4, 8);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2, 8);
            sum += __shfl_xor_sync(0xffffffffu, sum, 1, 8);
            const float inv = 1.f / sum;
#pragma unroll
            for (int h = 0; h < NH; ++h) e[h] *= inv;
        }
#pragma unroll 1
        for (int half = 0; half < NH; ++half) {
            // this lane's point of this pass: h = half
            float2 xy = __ldg(reinterpret_cast<const float2*>(loc + (size_t)u * (L * P * 2)) + half * 8 + cl);
            // level of this pass's point: A / B in registers for the first two passes, shared memory beyond (P = 8)
            const bool inB = NH <= 2 && half;
            const int H = NH <= 2 ? (inB ? HB : HA) : lv.H[half], W = NH <= 2 ? (inB ? WB : WA) : lv.W[half];
            float a;
            if constexpr (FUSED) {
                a = e[0];
#pragma unroll
                for (int h = 1; h < NH; ++h) a = half == h ? e[h] : a;
                const int l = NH <= 2 ? (inB ? lB : lA) : half;
                const float* r = ref + ((size_t)(u / M) * L + l) * ref_dim;
                if (ref_dim == 2) {
                    xy.x = __ldg(r) + xy.x / (float)W;
                    xy.y = __ldg(r + 1) + xy.y / (float)H;
                } else {
                    xy.x = fmaf(xy.x, (__ldg(r + 2) + __ldg(r + 3)) * 0.5f / (float)P, __ldg(r));
                    xy.y = fmaf(xy.y, (__ldg(r + 4) + __ldg(r + 5)) * 0.5f / (float)P, __ldg(r + 1));
                }
            } else {
                a = __ldg(attn + (size_t)u * (L * P) + half * 8 + cl);
            }
            const PointSetup Sx = NH <= 2 ? (inB ? setup_point(xy.x, xy.y, a, HB, WB, sB, pix) : setup_point(xy.x, xy.y, a, HA, WA, sA, pix))
                                          : setup_point(xy.x, xy.y, a, H, W, lv.start[half], pix);
#pragma unroll
            for (int jg = 0; jg < 4; ++jg) {             // 2 points = 8 line loads in flight at a time (register budget: 64)
                float4 v[2][4];
                float w[2][4];
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                    const int j = jg * 2 + jj;
                    const int o00 = __shfl_sync(0xffffffffu, Sx.o00, j, 8);
                    const int dxo = __shfl_sync(0xffffffffu, Sx.dxo, j, 8);
                    const int dyo = __shfl_sync(0xffffffffu, Sx.dyo, j, 8);
#pragma unroll
                    for (int k = 0; k < 4; ++k) w[jj][k] = __shfl_sync(0xffffffffu, Sx.w[k], j, 8);
                    const float* p00 = vb + o00;
                    v[jj][0] = ldg4(p00);
                    v[jj][1] = ldg4(p00 + dxo);
                    v[jj][2] = ldg4(p00 + dyo);
                    v[jj][3] = ldg4(p00 + dyo + dxo);
                }
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        acc.x = fmaf(w[jj][k], v[jj][k].x, acc.x);
                        acc.y = fmaf(w[jj][k], v[jj][k].y, acc.y);
                        acc.z = fmaf(w[jj][k], v[jj][k].z, acc.z);
                        acc.w = fmaf(w[jj][k], v[jj][k].w, acc.w);
                    }
                }
            }
        }
        if (live) *reinterpret_cast<float4*>(out + (size_t)unit * D + cl * 4) = acc;
    }
}

// ------------------------------------------------------------------------------------------------
// Fast backward: LPU lanes per unit, D = 4*LPU, L = 4, P in {2, 4, 8}.
// ------------------------------------------------------------------------------------------------
// The unit's 3*L*P outputs (d loc x / y, d attn per point) are reduced across its LPU lanes by a butterfly transpose-reduce over
// CHUNKS of LC levels: the whole unit at P <= 4 (48 values at P = 4), one level at P = 8 (24 values instead of 96 in registers).
// A chunk's value count is padded with zeros to a multiple of LPU (P = 2 at LPU = 16: 24 -> 32).
// FUSED (LPU == 8 only): `loc` / `attn` are the raw sampling offsets / attention logits, `grad_loc` / `grad_attn` receive the
// gradients wrt THOSE (the softmax / location pre-processing and its backward, ms_deform_attn.py:145-155, run inside this kernel;
// the reference points are constants of this path -- the caller takes the unfused path when they need a gradient).
// REFGRAD (FUSED, 6-d boxes only): also writes, per unit and level, the box partials [sum d loc_x, sum d loc_y,
// sum d loc_x off_x, sum d loc_y off_y] over the level's points to ref_part (n_units, L, 4), from the lanes' d loc.
template <int LPU, int L, int P, bool FUSED, bool REFGRAD>
__device__ __forceinline__ void
msda_bwd_vec(const float* __restrict__ value, const int64_t* __restrict__ shapes,
             const int64_t* __restrict__ lsi, const float* __restrict__ loc,
             const float* __restrict__ attn, const float* __restrict__ grad_out, int S, int M,
             int Lq, long long n_units, long long units_per_block, float* __restrict__ grad_value,
             float* __restrict__ grad_loc, float* __restrict__ grad_attn, const float* __restrict__ ref,
             int ref_dim, float* __restrict__ ref_part) {
    static_assert(P == 2 || P == 4 || P == 8, "2, 4 or 8 points");
    static_assert(!FUSED || (LPU == 8 && L == 4), "fused pre-processing: D = 32, L = 4");
    static_assert(!REFGRAD || FUSED, "box partials: fused path only");
    constexpr int D = 4 * LPU;
    constexpr int UPW = 32 / LPU;
    constexpr int NLOC = 2 * L * P;      // grad_loc values per unit
    constexpr int LC = P <= 4 ? L : 1;   // levels per butterfly chunk
    constexpr int NLOCC = 2 * LC * P;    // grad_loc values per chunk
    constexpr int NVC = 3 * LC * P;      // + grad_attn values
    constexpr int NVP = (NVC + LPU - 1) / LPU * LPU;   // padded to the butterfly's width
    constexpr int PER = NVP / LPU;       // values a lane ends up owning
    constexpr int NH = L * P / 8;        // FUSED: points each lane prepares
    static_assert(L % LC == 0 && NLOCC % LPU == 0, "loc / attn split per butterfly row");
    __shared__ LevelInfo lv;
    if (threadIdx.x < L) {
        lv.H[threadIdx.x] = (int)shapes[2 * threadIdx.x];
        lv.W[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
        lv.start[threadIdx.x] = (int)lsi[threadIdx.x];
    }
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const int sub = lane / LPU;
    const int cl = lane % LPU;
    const int wib = threadIdx.x >> 5;
    const int pix = M * D;
    // contiguous unit range per CTA (L1 / L2-atomic locality, see the forward kernel); ranges are multiples of UPW so
    // the lanes of a warp stay converged for the shuffles.
    const long long u_begin = (long long)blockIdx.x * units_per_block;
    const long long u_end = min(((n_units + UPW - 1) / UPW) * UPW, u_begin + units_per_block);

    for (long long unit = u_begin + wib * UPW + sub; unit < u_end; unit += (kThreads / 32) * UPW) {
        const bool live = unit < n_units;
        const long long u = live ? unit : 0;
        const int m = (int)(u % M);
        const long long b = u / ((long long)Lq * M);
        const size_t vbase = ((size_t)b * S * M + m) * D + cl * 4;
        const float* lp = loc + (size_t)u * L * P * 2;
        const float* ap = attn + (size_t)u * L * P;
        float4 g = ldg4(grad_out + (size_t)u * D + cl * 4);
        if (!live) g = make_float4(0.f, 0.f, 0.f, 0.f);
        // FUSED: the pre-processing is DISTRIBUTED over the unit's 8 lanes like in the forward kernel -- lane cl prepares points
        // h * 8 + cl (h < NH: L*P/8 exponentials, locations) and the level loop fetches what it needs with width-8 shuffles.  (Every
        // lane preparing all 16 points at P = 4 cost 16 expf + 32 divides per lane and made this kernel 30 % slower than the
        // two-step path.)
        [[maybe_unused]] float pa[NH], px[NH], py[NH];
        [[maybe_unused]] float gA[NH];                             // FUSED: d out / d attn of this lane's points
        [[maybe_unused]] float sc[L][2];                           // FUSED: d loc / d offset per level (x, y)
        if constexpr (FUSED) {
#pragma unroll
            for (int h = 0; h < NH; ++h) pa[h] = __ldg(ap + h * 8 + cl);
            float mx = pa[0];
#pragma unroll
            for (int h = 1; h < NH; ++h) mx = fmaxf(mx, pa[h]);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4, 8));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2, 8));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1, 8));
#pragma unroll
            for (int h = 0; h < NH; ++h) pa[h] = expf(pa[h] - mx);
            float sum = pa[0];
#pragma unroll
            for (int h = 1; h < NH; ++h) sum += pa[h];
            sum += __shfl_xor_sync(0xffffffffu, sum, 4, 8);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2, 8);
            sum += __shfl_xor_sync(0xffffffffu, sum, 1, 8);
            const float inv = 1.f / sum;
#pragma unroll
            for (int h = 0; h < NH; ++h) pa[h] *= inv;
#pragma unroll
            for (int hf = 0; hf < NH; ++hf) {                      // point hf * 8 + cl = (level hf * 8 / P + cl / P, point cl % P)
                const int l = hf * 8 / P + cl / P;
                const float2 o = __ldg(reinterpret_cast<const float2*>(lp) + hf * 8 + cl);
                const float* r = ref + ((size_t)(u / M) * L + l) * ref_dim;
                if (ref_dim == 2) {
                    px[hf] = __ldg(r) + o.x / (float)lv.W[l];
                    py[hf] = __ldg(r + 1) + o.y / (float)lv.H[l];
                } else {
                    px[hf] = fmaf(o.x, (__ldg(r + 2) + __ldg(r + 3)) * 0.5f / (float)P, __ldg(r));
                    py[hf] = fmaf(o.y, (__ldg(r + 4) + __ldg(r + 5)) * 0.5f / (float)P, __ldg(r + 1));
                }
            }
        }

#pragma unroll
        for (int c = 0; c < L / LC; ++c) {
            // vals[] is stored pre-permuted so that after the butterfly lane `cl` owns the chunk's outputs
            // j = i*LPU + cl (i = 0..PER-1): output j lives at position (j % LPU) * PER + j / LPU.
            float vals[NVP];
#pragma unroll
            for (int j = NVC; j < NVP; ++j) vals[(j % LPU) * PER + j / LPU] = 0.f;
#pragma unroll
            for (int lc = 0; lc < LC; ++lc) {
                const int l = c * LC + lc;
                const int H = lv.H[l], W = lv.W[l];
                const size_t lbase = vbase + (size_t)lv.start[l] * pix;
#pragma unroll
                for (int p0 = 0; p0 < P; p0 += (P < 4 ? P : 4)) {
                    constexpr int PG = P < 4 ? P : 4;
                    float xs[PG], ys[PG], as[PG];
                    load_points<PG>(lp + l * 2 * P + 2 * p0, ap + l * P + p0, xs, ys, as);
                    if constexpr (FUSED) {
                        if (p0 == 0) {
                            if (ref_dim == 2) {
                                sc[l][0] = 1.f / (float)W; sc[l][1] = 1.f / (float)H;
                            } else {
                                const float* r = ref + ((size_t)(u / M) * L + l) * ref_dim;
                                sc[l][0] = (__ldg(r + 2) + __ldg(r + 3)) * 0.5f / (float)P;
                                sc[l][1] = (__ldg(r + 4) + __ldg(r + 5)) * 0.5f / (float)P;
                            }
                        }
#pragma unroll
                        for (int p = 0; p < PG; ++p) {             // point k = l * P + p0 + p lives in lane k % 8, slot k / 8
                            const int k = l * P + p0 + p;
                            xs[p] = __shfl_sync(0xffffffffu, px[k / 8], k % 8, 8);
                            ys[p] = __shfl_sync(0xffffffffu, py[k / 8], k % 8, 8);
                            as[p] = __shfl_sync(0xffffffffu, pa[k / 8], k % 8, 8);
                        }
                    }
#pragma unroll
                    for (int pp = 0; pp < PG; ++pp) {
                        const int p = p0 + pp;
                        const float x = fmaf(xs[pp], (float)W, -0.5f);
                        const float y = fmaf(ys[pp], (float)H, -0.5f);
                        const bool inside = live && (y > -1.f) && (x > -1.f) && (y < (float)H) && (x < (float)W);
                        const float xf = floorf(x), yf = floorf(y);
                        const int x0 = (int)xf, y0 = (int)yf;
                        // finite weights off the image: they multiply the zero corners in ga / gx / gy (see the forward kernel)
                        const float lx = inside ? x - xf : 0.f, ly = inside ? y - yf : 0.f, hx = 1.f - lx, hy = 1.f - ly;
                        const bool top = inside && (y0 >= 0), bot = inside && (y0 + 1 <= H - 1);
                        const bool lef = (x0 >= 0), rig = (x0 + 1 <= W - 1);
                        const long long o00 = (long long)lbase + ((long long)y0 * W + x0) * pix;
                        const long long o01 = o00 + pix, o10 = o00 + (long long)W * pix, o11 = o10 + pix;
                        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                        const float4 v1 = (top && lef) ? ldg4(value + o00) : z;
                        const float4 v2 = (top && rig) ? ldg4(value + o01) : z;
                        const float4 v3 = (bot && lef) ? ldg4(value + o10) : z;
                        const float4 v4 = (bot && rig) ? ldg4(value + o11) : z;
                        const float a = as[pp];
                        const float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
                        const float tx = g.x * a, ty = g.y * a, tz = g.z * a, tw = g.w * a;
                        if (top && lef) red_add_v4(grad_value + o00, w1 * tx, w1 * ty, w1 * tz, w1 * tw);
                        if (top && rig) red_add_v4(grad_value + o01, w2 * tx, w2 * ty, w2 * tz, w2 * tw);
                        if (bot && lef) red_add_v4(grad_value + o10, w3 * tx, w3 * ty, w3 * tz, w3 * tw);
                        if (bot && rig) red_add_v4(grad_value + o11, w4 * tx, w4 * ty, w4 * tz, w4 * tw);
                        // per-channel bilinear value and its x / y derivatives (cuh:123-158)
                        float ga = 0.f, gx = 0.f, gy = 0.f;
#define MDB_ACC(c)                                                                   \
    ga = fmaf(g.c, w1 * v1.c + w2 * v2.c + w3 * v3.c + w4 * v4.c, ga);               \
    gx = fmaf(g.c * a, hy * (v2.c - v1.c) + ly * (v4.c - v3.c), gx);                 \
    gy = fmaf(g.c * a, hx * (v3.c - v1.c) + lx * (v4.c - v2.c), gy);
                        MDB_ACC(x) MDB_ACC(y) MDB_ACC(z) MDB_ACC(w)
#undef MDB_ACC
                        const int jx = (lc * P + p) * 2, jy = jx + 1, ja = NLOCC + lc * P + p;
                        vals[(jx % LPU) * PER + jx / LPU] = gx * (float)W;
                        vals[(jy % LPU) * PER + jy / LPU] = gy * (float)H;
                        vals[(ja % LPU) * PER + ja / LPU] = ga;
                    }
                }
            }
            // butterfly transpose-reduce across the LPU lanes of the unit
            {
                int n = NVP;
#pragma unroll
                for (int off = LPU / 2; off >= 1; off >>= 1) {
                    n >>= 1;
                    const bool up = (cl & off) != 0;
#pragma unroll
                    for (int i = 0; i < NVP / 2; ++i) {
                        if (i < n) {
                            const float send = up ? vals[i] : vals[i + n];
                            const float keep = up ? vals[i + n] : vals[i];
                            vals[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
                        }
                    }
                }
            }
            if constexpr (FUSED) {
                // lane cl owns the chunk's d out / d loc entries j = 8 i + cl (i < NLOCC / 8; component cl & 1) and d out / d attn
                // of its own points of the chunk (rows NLOCC / 8 ..: slot c * LC * P / 8 + row)
#pragma unroll
                for (int i = NLOCC / 8; i < PER; ++i) gA[c * LC * P / 8 + i - NLOCC / 8] = vals[i];
                [[maybe_unused]] float dot = 0.f;
                if (c == L / LC - 1) {                 // the softmax backward needs every chunk's d attn: taken with the last one
                    dot = pa[0] * gA[0];
#pragma unroll
                    for (int h = 1; h < NH; ++h) dot += pa[h] * gA[h];
                    dot += __shfl_xor_sync(0xffffffffu, dot, 4, 8);
                    dot += __shfl_xor_sync(0xffffffffu, dot, 2, 8);
                    dot += __shfl_xor_sync(0xffffffffu, dot, 1, 8);
                }
                if (live) {
                    float* gl = grad_loc + (size_t)unit * NLOC + c * NLOCC;
#pragma unroll
                    for (int i = 0; i < NLOCC / 8; ++i) {
                        // entry 8 i + cl: point (8 i + cl) / 2 of the chunk, level c * LC + (8 i + cl) / (2 P)
                        float sx, sy;
                        if constexpr (P == 2) {
                            sx = (cl & 4) ? sc[2 * i + 1][0] : sc[2 * i][0];
                            sy = (cl & 4) ? sc[2 * i + 1][1] : sc[2 * i][1];
                        } else {
                            sx = sc[c * LC + i * 4 / P][0];
                            sy = sc[c * LC + i * 4 / P][1];
                        }
                        gl[i * 8 + cl] = vals[i] * ((cl & 1) ? sy : sx);
                    }
                    if (c == L / LC - 1) {
                        float* gat = grad_attn + (size_t)unit * (L * P);
#pragma unroll
                        for (int h = 0; h < NH; ++h) gat[h * 8 + cl] = pa[h] * (gA[h] - dot);
                    }
                }
                if constexpr (REFGRAD) {
                    // lane cl holds d loc of the chunk's entries 8 i + cl, whose raw offsets are lp[c * NLOCC + 8 i + cl]: the sum over
                    // a level's points runs over the lanes of equal parity (fixed butterfly) and, at P = 8, over its two rows i;
                    // lanes 0 / 1 (P = 2: also 4 / 5, the second level of a row) write x / y
                    float* rp = ref_part + (size_t)unit * (L * 4);
                    if constexpr (P == 2) {
#pragma unroll
                        for (int i = 0; i < NLOCC / 8; ++i) {
                            float s = vals[i], w = vals[i] * __ldg(lp + i * 8 + cl);
                            s += __shfl_xor_sync(0xffffffffu, s, 2, 8);
                            w += __shfl_xor_sync(0xffffffffu, w, 2, 8);
                            if (live && (cl & 2) == 0) {
                                const int l = 2 * i + (cl >> 2);
                                rp[l * 4 + (cl & 1)] = s;
                                rp[l * 4 + 2 + (cl & 1)] = w;
                            }
                        }
                    } else {
                        constexpr int R = P / 4;                   // butterfly rows per level
#pragma unroll
                        for (int lc = 0; lc < LC; ++lc) {
                            const int l = c * LC + lc;
                            float s = vals[lc * R], w = vals[lc * R] * __ldg(lp + l * 2 * P + cl);
#pragma unroll
                            for (int r = 1; r < R; ++r) {
                                s += vals[lc * R + r];
                                w += vals[lc * R + r] * __ldg(lp + l * 2 * P + r * 8 + cl);
                            }
                            s += __shfl_xor_sync(0xffffffffu, s, 2, 8);
                            w += __shfl_xor_sync(0xffffffffu, w, 2, 8);
                            s += __shfl_xor_sync(0xffffffffu, s, 4, 8);
                            w += __shfl_xor_sync(0xffffffffu, w, 4, 8);
                            if (live && cl < 2) {
                                rp[l * 4 + cl] = s;
                                rp[l * 4 + 2 + cl] = w;
                            }
                        }
                    }
                }
            } else if (live) {
                float* gl = grad_loc + (size_t)unit * NLOC + c * NLOCC;
                float* gat = grad_attn + (size_t)unit * (L * P) + c * LC * P;
#pragma unroll
                for (int i = 0; i < PER; ++i) {
                    const int j = i * LPU + cl;
                    if (i * LPU < NLOCC) gl[j] = vals[i];
                    else if (NVP == NVC || j < NVC) gat[j - NLOCC] = vals[i];
                }
            }
        }
    }
}



// ------------------------------------------------------------------------------------------------
// The sampling kernels.  The P = 4 instances keep the names they had before P became a parameter (profiles and the dispatch
// tests key on them); P = 2 / 8 are the *_pts_kernel instances.  fwd_vec_kernel<LPU, P>() etc. pick the one for P.
// ------------------------------------------------------------------------------------------------
#define MDB_FWD_VEC_ARGS                                                                                                   \
    const float* __restrict__ value, const int64_t* __restrict__ shapes, const int64_t* __restrict__ lsi,                 \
        const float* __restrict__ loc, const float* __restrict__ attn, int S, int M, int L, int Lq, long long n_units,    \
        long long units_per_block, float* __restrict__ out
#define MDB_FWD_D32_ARGS                                                                                                   \
    const float* __restrict__ value, const int64_t* __restrict__ shapes, const int64_t* __restrict__ lsi,                 \
        const float* __restrict__ loc, const float* __restrict__ attn, const float* __restrict__ ref, int ref_dim, int S,  \
        int M, int Lq, long long n_units, long long units_per_block, float* __restrict__ out
#define MDB_BWD_VEC_ARGS                                                                                                   \
    const float* __restrict__ value, const int64_t* __restrict__ shapes, const int64_t* __restrict__ lsi,                 \
        const float* __restrict__ loc, const float* __restrict__ attn, const float* __restrict__ grad_out, int S, int M,  \
        int Lq, long long n_units, long long units_per_block, float* __restrict__ grad_value, float* __restrict__ grad_loc, \
        float* __restrict__ grad_attn, const float* __restrict__ ref, int ref_dim, float* __restrict__ ref_part

// Register budgets of the P = 2 / 8 instances (CTAs per SM in __launch_bounds__).  Under the P = 4 budgets (4 CTAs: 64 registers;
// 2 CTAs: 128) the P = 8 fused forward and every P = 2 / 8 backward spill; with one CTA less they do not (the backward then takes
// 116-244 registers -- anything above 128 is one 256-thread CTA per SM).  The fused P = 2 forward spills 8-28 bytes at every budget
// tried (2, 3, 4 CTAs) and keeps the P = 4 one.  Timed in DESIGN.md (tools/bench_points.py).
template <int P> constexpr int kFwdD32PtsBlocks = P == 8 ? 3 : 4;
constexpr int kBwdPtsBlocks = 1;

template <int LPU>
__global__ void __launch_bounds__(kThreads) msda_fwd_vec_kernel(MDB_FWD_VEC_ARGS) {
    msda_fwd_vec<LPU, 4>(value, shapes, lsi, loc, attn, S, M, L, Lq, n_units, units_per_block, out);
}
template <int LPU, int P>
__global__ void __launch_bounds__(kThreads) msda_fwd_vec_pts_kernel(MDB_FWD_VEC_ARGS) {
    msda_fwd_vec<LPU, P>(value, shapes, lsi, loc, attn, S, M, L, Lq, n_units, units_per_block, out);
}
template <bool FUSED>
__global__ void __launch_bounds__(kThreads, 4) msda_fwd_d32_kernel(MDB_FWD_D32_ARGS) {
    msda_fwd_d32<FUSED, 4>(value, shapes, lsi, loc, attn, ref, ref_dim, S, M, Lq, n_units, units_per_block, out);
}
template <bool FUSED, int P>
__global__ void __launch_bounds__(kThreads, kFwdD32PtsBlocks<P>) msda_fwd_d32_pts_kernel(MDB_FWD_D32_ARGS) {
    msda_fwd_d32<FUSED, P>(value, shapes, lsi, loc, attn, ref, ref_dim, S, M, Lq, n_units, units_per_block, out);
}
template <int LPU, int L, bool FUSED = false, bool REFGRAD = false>
__global__ void __launch_bounds__(kThreads, 2) msda_bwd_vec_kernel(MDB_BWD_VEC_ARGS) {
    msda_bwd_vec<LPU, L, 4, FUSED, REFGRAD>(value, shapes, lsi, loc, attn, grad_out, S, M, Lq, n_units, units_per_block,
                                            grad_value, grad_loc, grad_attn, ref, ref_dim, ref_part);
}
template <int LPU, int L, int P, bool FUSED = false, bool REFGRAD = false>
__global__ void __launch_bounds__(kThreads, kBwdPtsBlocks) msda_bwd_vec_pts_kernel(MDB_BWD_VEC_ARGS) {
    msda_bwd_vec<LPU, L, P, FUSED, REFGRAD>(value, shapes, lsi, loc, attn, grad_out, S, M, Lq, n_units, units_per_block,
                                            grad_value, grad_loc, grad_attn, ref, ref_dim, ref_part);
}
#undef MDB_FWD_VEC_ARGS
#undef MDB_FWD_D32_ARGS
#undef MDB_BWD_VEC_ARGS

template <int LPU, int P>
constexpr auto fwd_vec_kernel() {
    if constexpr (P == 4) return &msda_fwd_vec_kernel<LPU>;
    else return &msda_fwd_vec_pts_kernel<LPU, P>;
}
template <bool FUSED, int P>
constexpr auto fwd_d32_kernel() {
    if constexpr (P == 4) return &msda_fwd_d32_kernel<FUSED>;
    else return &msda_fwd_d32_pts_kernel<FUSED, P>;
}
template <int LPU, int P, bool FUSED = false, bool REFGRAD = false>
constexpr auto bwd_vec_kernel() {
    if constexpr (P == 4) return &msda_bwd_vec_kernel<LPU, 4, FUSED, REFGRAD>;
    else return &msda_bwd_vec_pts_kernel<LPU, 4, P, FUSED, REFGRAD>;
}

// ------------------------------------------------------------------------------------------------
// Generic kernels: one warp per unit, lanes stride over channels; any D, L, P; float and double.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
msda_fwd_generic_kernel(const T* __restrict__ value, const int64_t* __restrict__ shapes,
                        const int64_t* __restrict__ lsi, const T* __restrict__ loc,
                        const T* __restrict__ attn, int S, int M, int D, int L, int Lq, int P,
                        long long n_units, T* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    const long long nwarps = (long long)gridDim.x * (kThreads / 32);
    const size_t pix = (size_t)M * D;
    for (long long unit = warp; unit < n_units; unit += nwarps) {
        const int m = (int)(unit % M);
        const long long b = unit / ((long long)Lq * M);
        for (int c0 = 0; c0 < D; c0 += 32) {
            const int c = c0 + lane;
            const bool cok = c < D;
            T acc = 0;
            for (int l = 0; l < L; ++l) {
                const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
                const T* vl = value + ((size_t)b * S + (size_t)lsi[l]) * pix + (size_t)m * D + (cok ? c : 0);
                for (int p = 0; p < P; ++p) {
                    const size_t pi = ((size_t)unit * L + l) * P + p;
                    const T a = attn[pi];
                    const T x = fma_t(loc[2 * pi], (T)W, (T)-0.5);
                    const T y = fma_t(loc[2 * pi + 1], (T)H, (T)-0.5);
                    if (!(y > (T)-1 && x > (T)-1 && y < (T)H && x < (T)W)) continue;
                    const T xf = floor_t(x), yf = floor_t(y);
                    const int x0 = (int)xf, y0 = (int)yf;
                    const T lx = x - xf, ly = y - yf, hx = (T)1 - lx, hy = (T)1 - ly;
                    const bool top = y0 >= 0, bot = y0 + 1 <= H - 1, lef = x0 >= 0, rig = x0 + 1 <= W - 1;
                    const long long o00 = ((long long)y0 * W + x0) * (long long)pix;
                    T v1 = 0, v2 = 0, v3 = 0, v4 = 0;
                    if (cok) {
                        if (top && lef) v1 = vl[o00];
                        if (top && rig) v2 = vl[o00 + (long long)pix];
                        if (bot && lef) v3 = vl[o00 + (long long)W * pix];
                        if (bot && rig) v4 = vl[o00 + (long long)W * pix + pix];
                    }
                    acc += a * ((hy * hx) * v1 + (hy * lx) * v2 + (ly * hx) * v3 + (ly * lx) * v4);
                }
            }
            if (cok) out[(size_t)unit * D + c] = acc;
        }
    }
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

template <typename T, bool SCATTER = true>
__global__ void __launch_bounds__(kThreads)
msda_bwd_generic_kernel(const T* __restrict__ value, const int64_t* __restrict__ shapes,
                        const int64_t* __restrict__ lsi, const T* __restrict__ loc,
                        const T* __restrict__ attn, const T* __restrict__ grad_out, int S, int M, int D,
                        int L, int Lq, int P, long long n_units, T* __restrict__ grad_value,
                        T* __restrict__ grad_loc, T* __restrict__ grad_attn) {
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    const long long nwarps = (long long)gridDim.x * (kThreads / 32);
    const size_t pix = (size_t)M * D;
    for (long long unit = warp; unit < n_units; unit += nwarps) {
        const int m = (int)(unit % M);
        const long long b = unit / ((long long)Lq * M);
        for (int l = 0; l < L; ++l) {
            const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
            const size_t lbase = ((size_t)b * S + (size_t)lsi[l]) * pix + (size_t)m * D;
            for (int p = 0; p < P; ++p) {
                const size_t pi = ((size_t)unit * L + l) * P + p;
                const T a = attn[pi];
                const T x = fma_t(loc[2 * pi], (T)W, (T)-0.5);
                const T y = fma_t(loc[2 * pi + 1], (T)H, (T)-0.5);
                T ga = 0, gx = 0, gy = 0;
                if (y > (T)-1 && x > (T)-1 && y < (T)H && x < (T)W) {   // warp-uniform
                    const T xf = floor_t(x), yf = floor_t(y);
                    const int x0 = (int)xf, y0 = (int)yf;
                    const T lx = x - xf, ly = y - yf, hx = (T)1 - lx, hy = (T)1 - ly;
                    const bool top = y0 >= 0, bot = y0 + 1 <= H - 1, lef = x0 >= 0, rig = x0 + 1 <= W - 1;
                    const long long o00 = (long long)lbase + ((long long)y0 * W + x0) * (long long)pix;
                    const long long o01 = o00 + (long long)pix, o10 = o00 + (long long)W * pix, o11 = o10 + pix;
                    for (int c = lane; c < D; c += 32) {
                        const T g = grad_out[(size_t)unit * D + c];
                        const T tg = g * a;
                        T v1 = 0, v2 = 0, v3 = 0, v4 = 0;
                        if (top && lef) { v1 = value[o00 + c]; if constexpr (SCATTER) atomicAdd(grad_value + o00 + c, (hy * hx) * tg); }
                        if (top && rig) { v2 = value[o01 + c]; if constexpr (SCATTER) atomicAdd(grad_value + o01 + c, (hy * lx) * tg); }
                        if (bot && lef) { v3 = value[o10 + c]; if constexpr (SCATTER) atomicAdd(grad_value + o10 + c, (ly * hx) * tg); }
                        if (bot && rig) { v4 = value[o11 + c]; if constexpr (SCATTER) atomicAdd(grad_value + o11 + c, (ly * lx) * tg); }
                        ga += g * ((hy * hx) * v1 + (hy * lx) * v2 + (ly * hx) * v3 + (ly * lx) * v4);
                        gx += tg * (hy * (v2 - v1) + ly * (v4 - v3));
                        gy += tg * (hx * (v3 - v1) + lx * (v4 - v2));
                    }
                }
                ga = warp_sum(ga);
                gx = warp_sum(gx);
                gy = warp_sum(gy);
                if (lane == 0) {
                    grad_attn[pi] = ga;
                    grad_loc[2 * pi] = (T)W * gx;
                    grad_loc[2 * pi + 1] = (T)H * gy;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Reproducible value gradient (mdb_set_deterministic(1)): CTA (b, m, l) owns grad_value[b, level l, head m, :]; thread c owns
// channels c, c + blockDim, ... and adds the contributions of every (query, point, corner) IN THAT ORDER with plain
// read-modify-writes -- no element is ever touched by two threads, so the result is bit-identical from run to run (and
// independent of the grid).  Same arithmetic as the scatter: contribution = (bilinear weight) * (grad_out * attention weight).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
msda_bwd_value_ordered_kernel(const int64_t* __restrict__ shapes, const int64_t* __restrict__ lsi, const T* __restrict__ loc,
                              const T* __restrict__ attn, const T* __restrict__ grad_out, int S, int M, int D, int L, int Lq,
                              int P, T* grad_value) {
    const int l = (int)(blockIdx.x % L);
    const int m = (int)((blockIdx.x / L) % M);
    const long long b = blockIdx.x / ((long long)L * M);
    const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
    const size_t pix = (size_t)M * D;
    const size_t lbase = ((size_t)b * S + (size_t)lsi[l]) * pix + (size_t)m * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        for (int q = 0; q < Lq; ++q) {
            const size_t unit = ((size_t)b * Lq + q) * M + m;
            const T g = grad_out[unit * D + c];
            for (int p = 0; p < P; ++p) {
                const size_t pi = (unit * L + l) * P + p;
                const T x = fma_t(loc[2 * pi], (T)W, (T)-0.5);
                const T y = fma_t(loc[2 * pi + 1], (T)H, (T)-0.5);
                if (!(y > (T)-1 && x > (T)-1 && y < (T)H && x < (T)W)) continue;
                const T tg = g * attn[pi];
                const T xf = floor_t(x), yf = floor_t(y);
                const int x0 = (int)xf, y0 = (int)yf;
                const T lx = x - xf, ly = y - yf, hx = (T)1 - lx, hy = (T)1 - ly;
                const bool top = y0 >= 0, bot = y0 + 1 <= H - 1, lef = x0 >= 0, rig = x0 + 1 <= W - 1;
                const long long o00 = (long long)lbase + ((long long)y0 * W + x0) * (long long)pix + c;
                const long long o01 = o00 + (long long)pix, o10 = o00 + (long long)W * pix, o11 = o10 + pix;
                if (top && lef) grad_value[o00] += (hy * hx) * tg;
                if (top && rig) grad_value[o01] += (hy * lx) * tg;
                if (bot && lef) grad_value[o10] += (ly * hx) * tg;
                if (bot && rig) grad_value[o11] += (ly * lx) * tg;
            }
        }
    }
}

int check_common(const void* a, const void* b, const void* c, const void* d, const void* e, int B, int S,
                 int M, int D, int L, int Lq, int P) {
    if (B < 0 || S < 0 || M < 0 || D < 0 || L < 0 || Lq < 0 || P < 0) return MDB_EINVAL;
    const long long n = (long long)B * Lq * M * D;
    if (n > 0 && L > 0 && P > 0 && (!a || !b || !c || !d || !e)) return MDB_EINVAL;
    return 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// point counts the fused kernels are compiled for
bool fused_points(int P) { return P == 2 || P == 4 || P == 8; }

// Fast fp32 paths (P in {2, 4, 8}, D in {16, 32, 64}, aligned rows): one instance per (D, P).
template <int P>
void launch_fwd_fast(const float* value, const int64_t* shapes, const int64_t* lsi, const float* loc, const float* attn, int S,
                     int M, int D, int L, int Lq, long long n_units, float* out, cudaStream_t stream) {
    const int lpu = D / 4, upw = 32 / lpu;
    const int grid = grid_cap((n_units + upw - 1) / upw, kThreads / 32, num_sms() * 8);
    const long long per = (kThreads / 32) * upw;                        // units one CTA pass covers
    const long long upb = ((n_units + grid - 1) / grid + per - 1) / per * per;
    if (P == 4 && lpu == 8 && L == 4)           // (P = 2 / 8: the spill-free msda_fwd_vec_pts_kernel<8, P> below)
        fwd_d32_kernel<false, 4>()<<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, nullptr, 0, S, M, Lq, n_units, upb, out);
    else if (lpu == 8)
        fwd_vec_kernel<8, P>()<<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, S, M, L, Lq, n_units, upb, out);
    else if (lpu == 4)
        fwd_vec_kernel<4, P>()<<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, S, M, L, Lq, n_units, upb, out);
    else
        fwd_vec_kernel<16, P>()<<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, S, M, L, Lq, n_units, upb, out);
}

template <int P>
void launch_bwd_fast(const float* value, const int64_t* shapes, const int64_t* lsi, const float* loc, const float* attn,
                     const float* grad_out, int S, int M, int D, int Lq, long long n_units, float* grad_value, float* grad_loc,
                     float* grad_attn, cudaStream_t stream) {
    const int lpu = D / 4, upw = 32 / lpu;
    const int grid = grid_cap((n_units + upw - 1) / upw, kThreads / 32, num_sms() * 6);
    const long long per = (kThreads / 32) * upw;
    const long long upb = ((n_units + grid - 1) / grid + per - 1) / per * per;
    if (lpu == 8)
        bwd_vec_kernel<8, P>()<<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, grad_out, S, M, Lq, n_units, upb, grad_value, grad_loc, grad_attn, nullptr, 0, nullptr);
    else if (lpu == 4)
        bwd_vec_kernel<4, P>()<<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, grad_out, S, M, Lq, n_units, upb, grad_value, grad_loc, grad_attn, nullptr, 0, nullptr);
    else
        bwd_vec_kernel<16, P>()<<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, grad_out, S, M, Lq, n_units, upb, grad_value, grad_loc, grad_attn, nullptr, 0, nullptr);
}

template <typename T>
int forward_impl(const T* value, const int64_t* shapes, const int64_t* lsi, const T* loc, const T* attn, int B,
                 int S, int M, int D, int L, int Lq, int P, T* out, void* stream_) {
    int rc = check_common(value, shapes, lsi, loc, attn, B, S, M, D, L, Lq, P);
    if (rc) return rc;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const long long n_units = (long long)B * Lq * M;
    if (n_units == 0 || D == 0) return 0;
    if (!out) return MDB_EINVAL;
    if (L == 0 || P == 0) {
        return (int)cudaMemsetAsync(out, 0, sizeof(T) * (size_t)n_units * D, stream);
    }
    if constexpr (sizeof(T) == 4) {
        const bool fast = (P == 2 || P == 4 || P == 8) && (L <= kMaxLevels) && (D == 16 || D == 32 || D == 64) &&
                          aligned16(value) && aligned16(loc) && aligned16(attn) && aligned16(out);
        if (fast) {
            if (P == 2) launch_fwd_fast<2>(value, shapes, lsi, loc, attn, S, M, D, L, Lq, n_units, out, stream);
            else if (P == 4) launch_fwd_fast<4>(value, shapes, lsi, loc, attn, S, M, D, L, Lq, n_units, out, stream);
            else launch_fwd_fast<8>(value, shapes, lsi, loc, attn, S, M, D, L, Lq, n_units, out, stream);
            return (int)cudaGetLastError();
        }
    }
    const int grid = grid_cap(n_units, kThreads / 32, num_sms() * 8);
    msda_fwd_generic_kernel<T><<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, S, M, D, L, Lq, P, n_units, out);
    return (int)cudaGetLastError();
}

template <typename T>
int backward_impl(const T* value, const int64_t* shapes, const int64_t* lsi, const T* loc, const T* attn,
                  const T* grad_out, int B, int S, int M, int D, int L, int Lq, int P, T* grad_value, T* grad_loc,
                  T* grad_attn, void* stream_) {
    int rc = check_common(value, shapes, lsi, loc, attn, B, S, M, D, L, Lq, P);
    if (rc) return rc;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const long long n_units = (long long)B * Lq * M;
    const size_t nv = (size_t)B * S * M * D;
    if (nv) {
        if (!grad_value) return MDB_EINVAL;
        cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(T) * nv, stream);
        if (e != cudaSuccess) return (int)e;
    }
    if (n_units == 0 || L == 0 || P == 0) return 0;
    if (!grad_loc || !grad_attn) return MDB_EINVAL;
    if (D == 0) {
        cudaError_t e = cudaMemsetAsync(grad_loc, 0, sizeof(T) * (size_t)n_units * L * P * 2, stream);
        if (e != cudaSuccess) return (int)e;
        return (int)cudaMemsetAsync(grad_attn, 0, sizeof(T) * (size_t)n_units * L * P, stream);
    }
    if (!grad_out) return MDB_EINVAL;
    if (mdb_get_deterministic()) {
        // grad_loc / grad_attn by the generic kernel (warp reductions, no atomics) with its scatter compiled out, then the
        // value gradient in a fixed accumulation order
        const int grid = grid_cap(n_units, kThreads / 32, num_sms() * 8);
        msda_bwd_generic_kernel<T, false><<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, grad_out, S, M, D, L, Lq, P, n_units, grad_value, grad_loc, grad_attn);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
        int threads = (D + 31) / 32 * 32;
        if (threads > kThreads) threads = kThreads;
        msda_bwd_value_ordered_kernel<T><<<(unsigned)((long long)B * M * L), threads, 0, stream>>>(shapes, lsi, loc, attn, grad_out, S, M, D, L, Lq, P, grad_value);
        return (int)cudaGetLastError();
    }
    if constexpr (sizeof(T) == 4) {
        const bool fast = (P == 2 || P == 4 || P == 8) && (L == 4) && (D == 16 || D == 32 || D == 64) && aligned16(value) &&
                          aligned16(loc) && aligned16(attn) && aligned16(grad_out) && aligned16(grad_value);
        if (fast) {
            // (Two variants were tried on another GPU and removed: a branch-free backward organised like msda_fwd_d32_kernel, and
            // the coarse levels' gradient rows privatised in shared memory.  Neither has been timed on an H100.)
            if (P == 2) launch_bwd_fast<2>(value, shapes, lsi, loc, attn, grad_out, S, M, D, Lq, n_units, grad_value, grad_loc, grad_attn, stream);
            else if (P == 4) launch_bwd_fast<4>(value, shapes, lsi, loc, attn, grad_out, S, M, D, Lq, n_units, grad_value, grad_loc, grad_attn, stream);
            else launch_bwd_fast<8>(value, shapes, lsi, loc, attn, grad_out, S, M, D, Lq, n_units, grad_value, grad_loc, grad_attn, stream);
            return (int)cudaGetLastError();
        }
    }
    const int grid = grid_cap(n_units, kThreads / 32, num_sms() * 8);
    msda_bwd_generic_kernel<T><<<grid, kThreads, 0, stream>>>(value, shapes, lsi, loc, attn, grad_out, S, M, D, L, Lq, P, n_units, grad_value, grad_loc, grad_attn);
    return (int)cudaGetLastError();
}

}  // namespace

extern "C" {

int mdb_msda_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                         const float* sampling_loc, const float* attn_weight, int B, int S, int M, int D, int L,
                         int Lq, int P, float* out, void* stream) {
    return forward_impl<float>(value, spatial_shapes, level_start, sampling_loc, attn_weight, B, S, M, D, L, Lq, P, out, stream);
}
int mdb_msda_forward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start,
                         const double* sampling_loc, const double* attn_weight, int B, int S, int M, int D, int L,
                         int Lq, int P, double* out, void* stream) {
    return forward_impl<double>(value, spatial_shapes, level_start, sampling_loc, attn_weight, B, S, M, D, L, Lq, P, out, stream);
}
int mdb_msda_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                          const float* sampling_loc, const float* attn_weight, const float* grad_out, int B, int S,
                          int M, int D, int L, int Lq, int P, float* grad_value, float* grad_loc, float* grad_attn,
                          void* stream) {
    return backward_impl<float>(value, spatial_shapes, level_start, sampling_loc, attn_weight, grad_out, B, S, M, D, L, Lq, P, grad_value, grad_loc, grad_attn, stream);
}
// Fused module path (MSDeformAttn.forward with constant reference points): pre-processing inside the sampling kernels.
// D = 32, L = 4, P in {2, 4, 8} only; anything else returns MDB_EUNSUPPORTED and the caller uses mdb_msda_prep_* + mdb_msda_*.
int mdb_msda_fused_forward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start, const float* offsets,
                               const float* logits, const float* ref, int B, int S, int M, int D, int L, int Lq, int P, int ref_dim,
                               float* out, void* stream_) {
    if (D != 32 || L != 4 || !fused_points(P) || (ref_dim != 2 && ref_dim != 6)) return MDB_EUNSUPPORTED;
    int rc = check_common(value, spatial_shapes, level_start, offsets, logits, B, S, M, D, L, Lq, P);
    if (rc) return rc;
    const long long n_units = (long long)B * Lq * M;
    if (n_units == 0) return 0;
    if (!ref || !out) return MDB_EINVAL;
    if (!aligned16(value) || !aligned16(offsets) || !aligned16(logits) || !aligned16(out)) return MDB_EUNSUPPORTED;
    const int grid = grid_cap((n_units + 3) / 4, kThreads / 32, num_sms() * 8);
    const long long per = (kThreads / 32) * 4;
    const long long upb = ((n_units + grid - 1) / grid + per - 1) / per * per;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (P == 2)
        fwd_d32_kernel<true, 2>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, ref, ref_dim, S, M, Lq, n_units, upb, out);
    else if (P == 4)
        fwd_d32_kernel<true, 4>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, ref, ref_dim, S, M, Lq, n_units, upb, out);
    else
        fwd_d32_kernel<true, 8>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, ref, ref_dim, S, M, Lq, n_units, upb, out);
    return (int)cudaGetLastError();
}
int mdb_msda_fused_backward_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start, const float* offsets,
                                const float* logits, const float* ref, const float* grad_out, int B, int S, int M, int D, int L, int Lq,
                                int P, int ref_dim, float* grad_value, float* grad_offsets, float* grad_logits, void* stream_) {
    if (D != 32 || L != 4 || !fused_points(P) || (ref_dim != 2 && ref_dim != 6)) return MDB_EUNSUPPORTED;
    if (mdb_get_deterministic()) return MDB_EUNSUPPORTED;      // ordered accumulation: mdb_msda_prep_* + mdb_msda_backward_*
    int rc = check_common(value, spatial_shapes, level_start, offsets, logits, B, S, M, D, L, Lq, P);
    if (rc) return rc;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const long long n_units = (long long)B * Lq * M;
    const size_t nv = (size_t)B * S * M * D;
    if (!aligned16(value) || !aligned16(offsets) || !aligned16(logits) || !aligned16(grad_out) || !aligned16(grad_value))
        return MDB_EUNSUPPORTED;
    if (nv) {
        if (!grad_value) return MDB_EINVAL;
        cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * nv, stream);
        if (e != cudaSuccess) return (int)e;
    }
    if (n_units == 0) return 0;
    if (!ref || !grad_out || !grad_offsets || !grad_logits) return MDB_EINVAL;
    const int grid = grid_cap((n_units + 3) / 4, kThreads / 32, num_sms() * 6);
    const long long per = (kThreads / 32) * 4;
    const long long upb = ((n_units + grid - 1) / grid + per - 1) / per * per;
    if (P == 2)
        bwd_vec_kernel<8, 2, true>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, grad_out, S, M, Lq,
                                                                          n_units, upb, grad_value, grad_offsets, grad_logits, ref, ref_dim, nullptr);
    else if (P == 4)
        bwd_vec_kernel<8, 4, true>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, grad_out, S, M, Lq,
                                                                          n_units, upb, grad_value, grad_offsets, grad_logits, ref, ref_dim, nullptr);
    else
        bwd_vec_kernel<8, 8, true>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, grad_out, S, M, Lq,
                                                                          n_units, upb, grad_value, grad_offsets, grad_logits, ref, ref_dim, nullptr);
    return (int)cudaGetLastError();
}
// mdb_msda_fused_backward_f32 for 6-d boxes that require grad, plus the box partials ref_part (B, Lq, M, L, 4) =
// [sum d loc_x, sum d loc_y, sum d loc_x off_x, sum d loc_y off_y] over each level's points (mdb_msda_ref_partials_reduce_f32
// turns them into the box gradient).
int mdb_msda_fused_backward_ref_f32(const float* value, const int64_t* spatial_shapes, const int64_t* level_start,
                                    const float* offsets, const float* logits, const float* ref, const float* grad_out, int B, int S,
                                    int M, int D, int L, int Lq, int P, int ref_dim, float* grad_value, float* grad_offsets,
                                    float* grad_logits, float* ref_part, void* stream_) {
    if (D != 32 || L != 4 || !fused_points(P) || ref_dim != 6) return MDB_EUNSUPPORTED;
    if (mdb_get_deterministic()) return MDB_EUNSUPPORTED;      // ordered accumulation: mdb_msda_prep_* + mdb_msda_backward_*
    int rc = check_common(value, spatial_shapes, level_start, offsets, logits, B, S, M, D, L, Lq, P);
    if (rc) return rc;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const long long n_units = (long long)B * Lq * M;
    const size_t nv = (size_t)B * S * M * D;
    if (!aligned16(value) || !aligned16(offsets) || !aligned16(logits) || !aligned16(grad_out) || !aligned16(grad_value))
        return MDB_EUNSUPPORTED;
    if (nv) {
        if (!grad_value) return MDB_EINVAL;
        cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * nv, stream);
        if (e != cudaSuccess) return (int)e;
    }
    if (n_units == 0) return 0;
    if (!ref || !grad_out || !grad_offsets || !grad_logits || !ref_part) return MDB_EINVAL;
    const int grid = grid_cap((n_units + 3) / 4, kThreads / 32, num_sms() * 6);
    const long long per = (kThreads / 32) * 4;
    const long long upb = ((n_units + grid - 1) / grid + per - 1) / per * per;
    if (P == 2)
        bwd_vec_kernel<8, 2, true, true>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, grad_out, S,
                                                                                M, Lq, n_units, upb, grad_value, grad_offsets, grad_logits, ref,
                                                                                ref_dim, ref_part);
    else if (P == 4)
        bwd_vec_kernel<8, 4, true, true>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, grad_out, S,
                                                                                M, Lq, n_units, upb, grad_value, grad_offsets, grad_logits, ref,
                                                                                ref_dim, ref_part);
    else
        bwd_vec_kernel<8, 8, true, true>()<<<grid, kThreads, 0, stream>>>(value, spatial_shapes, level_start, offsets, logits, grad_out, S,
                                                                                M, Lq, n_units, upb, grad_value, grad_offsets, grad_logits, ref,
                                                                                ref_dim, ref_part);
    return (int)cudaGetLastError();
}
int mdb_msda_backward_f64(const double* value, const int64_t* spatial_shapes, const int64_t* level_start,
                          const double* sampling_loc, const double* attn_weight, const double* grad_out, int B, int S,
                          int M, int D, int L, int Lq, int P, double* grad_value, double* grad_loc, double* grad_attn,
                          void* stream) {
    return backward_impl<double>(value, spatial_shapes, level_start, sampling_loc, attn_weight, grad_out, B, S, M, D, L, Lq, P, grad_value, grad_loc, grad_attn, stream);
}

}  // extern "C"

// =================================================================================================
// Fused pre-processing of the MSDeformAttn module (ops/modules/ms_deform_attn.py:145-155): from the raw
// projections  off = sampling_offsets(query) [.., M, L, P, 2]  and  logits = attention_weights(query) [.., M, L*P]
// produce  sampling_locations  and  softmax(logits)  in one pass (the reference runs ~6 elementwise kernels
// over these 83 MB tensors), and the matching backward.
//   ref_dim == 2:  loc = ref[b,q,l,:] + off / (W_l, H_l)
//   ref_dim == 6:  loc = ref_xy + off / P * (ref[2]+ref[3], ref[4]+ref[5]) * 0.5      (l+r, t+b)
// One thread per (b, q, m).  L*P <= 16 with P even: 16-byte loads and stores; any other L*P <= 32 (odd point counts, P = 8 at
// four levels): the scalar kernels below, with the same arithmetic in the same order.
// =================================================================================================
namespace {

constexpr int kPrepMaxLP = 16;

__global__ void __launch_bounds__(256)
msda_prep_fwd_kernel(const float* __restrict__ off, const float* __restrict__ logits, const float* __restrict__ ref,
                     const int64_t* __restrict__ shapes, int M, int L, int P, int ref_dim, long long n_units,
                     float* __restrict__ loc, float* __restrict__ attn) {
    const int LP = L * P;
    for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < n_units; u += (long long)gridDim.x * blockDim.x) {
        const long long bq = u / M;
        const float* o = off + u * LP * 2;
        const float* lg = logits + u * LP;
        float* lo = loc + u * LP * 2;
        float* at = attn + u * LP;
        float v[kPrepMaxLP];
        float mx = -INFINITY;
        for (int i = 0; i < LP; i += 4) {
            const float4 t = *reinterpret_cast<const float4*>(lg + i);
            v[i] = t.x; v[i + 1] = t.y; v[i + 2] = t.z; v[i + 3] = t.w;
            mx = fmaxf(mx, fmaxf(fmaxf(t.x, t.y), fmaxf(t.z, t.w)));
        }
        float sum = 0.f;
        for (int i = 0; i < LP; ++i) { v[i] = expf(v[i] - mx); sum += v[i]; }
        const float inv = 1.f / sum;
        for (int i = 0; i < LP; i += 4)
            *reinterpret_cast<float4*>(at + i) = make_float4(v[i] * inv, v[i + 1] * inv, v[i + 2] * inv, v[i + 3] * inv);
        for (int l = 0; l < L; ++l) {
            const float* r = ref + (bq * L + l) * ref_dim;
            float sx, sy;
            if (ref_dim == 2) {
                sx = 1.f / (float)shapes[2 * l + 1];
                sy = 1.f / (float)shapes[2 * l];
            } else {
                sx = (r[2] + r[3]) * 0.5f / (float)P;
                sy = (r[4] + r[5]) * 0.5f / (float)P;
            }
            const float rx = r[0], ry = r[1];
            for (int p = 0; p < P; p += 2) {
                const float4 t = *reinterpret_cast<const float4*>(o + (l * P + p) * 2);
                float4 w;
                if (ref_dim == 2) { w.x = rx + t.x / (float)shapes[2 * l + 1]; w.y = ry + t.y / (float)shapes[2 * l];
                                    w.z = rx + t.z / (float)shapes[2 * l + 1]; w.w = ry + t.w / (float)shapes[2 * l]; }
                else { w.x = fmaf(t.x, sx, rx); w.y = fmaf(t.y, sy, ry); w.z = fmaf(t.z, sx, rx); w.w = fmaf(t.w, sy, ry); }
                *reinterpret_cast<float4*>(lo + (l * P + p) * 2) = w;
            }
        }
    }
}

__global__ void __launch_bounds__(256)
msda_prep_bwd_kernel(const float* __restrict__ dloc, const float* __restrict__ dattn, const float* __restrict__ attn,
                     const float* __restrict__ ref, const int64_t* __restrict__ shapes, int M, int L, int P, int ref_dim,
                     long long n_units, float* __restrict__ doff, float* __restrict__ dlogits) {
    const int LP = L * P;
    for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < n_units; u += (long long)gridDim.x * blockDim.x) {
        const long long bq = u / M;
        float a[kPrepMaxLP], g[kPrepMaxLP];
        float dot = 0.f;
        for (int i = 0; i < LP; i += 4) {
            const float4 x = *reinterpret_cast<const float4*>(attn + u * LP + i);
            const float4 y = *reinterpret_cast<const float4*>(dattn + u * LP + i);
            a[i] = x.x; a[i + 1] = x.y; a[i + 2] = x.z; a[i + 3] = x.w;
            g[i] = y.x; g[i + 1] = y.y; g[i + 2] = y.z; g[i + 3] = y.w;
            dot += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
        }
        for (int i = 0; i < LP; i += 4)
            *reinterpret_cast<float4*>(dlogits + u * LP + i) = make_float4(a[i] * (g[i] - dot), a[i + 1] * (g[i + 1] - dot),
                                                                          a[i + 2] * (g[i + 2] - dot), a[i + 3] * (g[i + 3] - dot));
        for (int l = 0; l < L; ++l) {
            float sx, sy;
            if (ref_dim == 2) {
                sx = 1.f / (float)shapes[2 * l + 1];
                sy = 1.f / (float)shapes[2 * l];
            } else {
                const float* r = ref + (bq * L + l) * ref_dim;
                sx = (r[2] + r[3]) * 0.5f / (float)P;
                sy = (r[4] + r[5]) * 0.5f / (float)P;
            }
            for (int p = 0; p < P; p += 2) {
                const float4 t = *reinterpret_cast<const float4*>(dloc + (u * LP + l * P + p) * 2);
                float4 w;
                if (ref_dim == 2) { w.x = t.x / (float)shapes[2 * l + 1]; w.y = t.y / (float)shapes[2 * l];
                                    w.z = t.z / (float)shapes[2 * l + 1]; w.w = t.w / (float)shapes[2 * l]; }
                else { w.x = t.x * sx; w.y = t.y * sy; w.z = t.z * sx; w.w = t.w * sy; }
                *reinterpret_cast<float4*>(doff + (u * LP + l * P + p) * 2) = w;
            }
        }
    }
}

// Any L*P <= kPrepMaxLPAny, no alignment beyond 4 bytes: the logits are re-read instead of held in a register array.
constexpr int kPrepMaxLPAny = 32;

__device__ __forceinline__ void prep_scale(const float* __restrict__ ref, const int64_t* __restrict__ shapes, long long bq, int l,
                                           int L, int P, int ref_dim, float& sx, float& sy) {
    if (ref_dim == 2) {
        sx = 1.f / (float)shapes[2 * l + 1];
        sy = 1.f / (float)shapes[2 * l];
    } else {
        const float* r = ref + (bq * L + l) * ref_dim;
        sx = (r[2] + r[3]) * 0.5f / (float)P;
        sy = (r[4] + r[5]) * 0.5f / (float)P;
    }
}

__global__ void __launch_bounds__(256)
msda_prep_fwd_any_kernel(const float* __restrict__ off, const float* __restrict__ logits, const float* __restrict__ ref,
                         const int64_t* __restrict__ shapes, int M, int L, int P, int ref_dim, long long n_units,
                         float* __restrict__ loc, float* __restrict__ attn) {
    const int LP = L * P;
    for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < n_units; u += (long long)gridDim.x * blockDim.x) {
        const long long bq = u / M;
        const float* lg = logits + u * LP;
        float* at = attn + u * LP;
        float mx = -INFINITY;
        for (int i = 0; i < LP; ++i) mx = fmaxf(mx, lg[i]);
        float sum = 0.f;
        for (int i = 0; i < LP; ++i) sum += expf(lg[i] - mx);
        const float inv = 1.f / sum;
        for (int i = 0; i < LP; ++i) at[i] = expf(lg[i] - mx) * inv;
        for (int l = 0; l < L; ++l) {
            const float* r = ref + (bq * L + l) * ref_dim;
            float sx, sy;
            prep_scale(ref, shapes, bq, l, L, P, ref_dim, sx, sy);
            for (int p = 0; p < P; ++p) {
                const size_t i = (size_t)(u * LP + l * P + p) * 2;
                if (ref_dim == 2) {
                    loc[i] = r[0] + off[i] / (float)shapes[2 * l + 1];
                    loc[i + 1] = r[1] + off[i + 1] / (float)shapes[2 * l];
                } else {
                    loc[i] = fmaf(off[i], sx, r[0]);
                    loc[i + 1] = fmaf(off[i + 1], sy, r[1]);
                }
            }
        }
    }
}

__global__ void __launch_bounds__(256)
msda_prep_bwd_any_kernel(const float* __restrict__ dloc, const float* __restrict__ dattn, const float* __restrict__ attn,
                         const float* __restrict__ ref, const int64_t* __restrict__ shapes, int M, int L, int P, int ref_dim,
                         long long n_units, float* __restrict__ doff, float* __restrict__ dlogits) {
    const int LP = L * P;
    for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < n_units; u += (long long)gridDim.x * blockDim.x) {
        const long long bq = u / M;
        const float* a = attn + u * LP;
        const float* g = dattn + u * LP;
        float dot = 0.f;
        for (int i = 0; i < LP; ++i) dot += a[i] * g[i];
        for (int i = 0; i < LP; ++i) dlogits[u * LP + i] = a[i] * (g[i] - dot);
        for (int l = 0; l < L; ++l) {
            float sx, sy;
            prep_scale(ref, shapes, bq, l, L, P, ref_dim, sx, sy);
            for (int p = 0; p < P; ++p) {
                const size_t i = (size_t)(u * LP + l * P + p) * 2;
                if (ref_dim == 2) {
                    doff[i] = dloc[i] / (float)shapes[2 * l + 1];
                    doff[i + 1] = dloc[i + 1] / (float)shapes[2 * l];
                } else {
                    doff[i] = dloc[i] * sx;
                    doff[i + 1] = dloc[i + 1] * sy;
                }
            }
        }
    }
}

// the vectorised kernels' layout: L*P <= 16, whole float4 rows, pairs of points per float4
bool prep_vectorised(int L, int P) { return L * P <= kPrepMaxLP && (L * P) % 4 == 0 && P % 2 == 0; }

}  // namespace

extern "C" {

int mdb_msda_prep_forward_f32(const float* off, const float* logits, const float* ref, const int64_t* spatial_shapes,
                              int B, int Lq, int M, int L, int P, int ref_dim, float* loc, float* attn, void* stream) {
    if (!off || !logits || !ref || !spatial_shapes || !loc || !attn) return MDB_EINVAL;
    if (L <= 0 || P <= 0 || L * P > kPrepMaxLPAny || (ref_dim != 2 && ref_dim != 6)) return MDB_EUNSUPPORTED;
    const long long n = (long long)B * Lq * M;
    if (n == 0) return 0;
    const bool vec = prep_vectorised(L, P) && aligned16(off) && aligned16(logits) && aligned16(loc) && aligned16(attn);
    if (vec)
        msda_prep_fwd_kernel<<<grid_cap(n, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(off, logits, ref, spatial_shapes, M, L, P, ref_dim, n, loc, attn);
    else
        msda_prep_fwd_any_kernel<<<grid_cap(n, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(off, logits, ref, spatial_shapes, M, L, P, ref_dim, n, loc, attn);
    return (int)cudaGetLastError();
}

int mdb_msda_prep_backward_f32(const float* dloc, const float* dattn, const float* attn, const float* ref,
                               const int64_t* spatial_shapes, int B, int Lq, int M, int L, int P, int ref_dim,
                               float* doff, float* dlogits, void* stream) {
    if (!dloc || !dattn || !attn || !ref || !spatial_shapes || !doff || !dlogits) return MDB_EINVAL;
    if (L <= 0 || P <= 0 || L * P > kPrepMaxLPAny || (ref_dim != 2 && ref_dim != 6)) return MDB_EUNSUPPORTED;
    const long long n = (long long)B * Lq * M;
    if (n == 0) return 0;
    const bool vec = prep_vectorised(L, P) && aligned16(dloc) && aligned16(dattn) && aligned16(attn) && aligned16(doff) &&
                     aligned16(dlogits);
    if (vec)
        msda_prep_bwd_kernel<<<grid_cap(n, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(dloc, dattn, attn, ref, spatial_shapes, M, L, P, ref_dim, n, doff, dlogits);
    else
        msda_prep_bwd_any_kernel<<<grid_cap(n, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(dloc, dattn, attn, ref, spatial_shapes, M, L, P, ref_dim, n, doff, dlogits);
    return (int)cudaGetLastError();
}

}  // extern "C"
