// pos_embed.cu -- the learned position embedding (position_embedding: 'learned' / 'v3', position_encoding.py:59-86) for the
// all-False masks this path has: two (50, 128) tables, a row table indexed by y and a column table indexed by x, each read at
// the fractional coordinate i = x / w * 49 and interpolated linearly between rows floor(i) and min(floor(i) + 1, 49).
//   forward   (H*W, 256) channels-last table, channels 0..127 = column (x) embedding, 128..255 = row (y) embedding
//   backward  the (50, 128) gradients of both tables from the level's batch-summed (H*W, 256) gradient
// The forward spells every fp32 operation with an explicit round-to-nearest intrinsic, so that nvcc cannot contract a multiply
// and an add into an FMA: the table is then bit-identical to the reference's separately rounded torch operations.  The backward
// sums in a fixed order with no atomics, so the reproducible mode covers this branch without a separate path.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

using namespace mdb;

constexpr int kRows = 50;                  // nn.Embedding(50, num_pos_feats)
constexpr int kFeats = 128;                // num_pos_feats = hidden_dim / 2
constexpr int kOut = 2 * kFeats;

struct Lerp {
    int f, c;                              // floor and ceil rows
    float d;                               // i - floor(i), exact
};

// torch.arange(n) / n * 49 -> floor / clamped ceil / fraction, rounded as torch rounds each fp32 operation
__device__ __forceinline__ Lerp lerp_of(int x, int n) {
    const float i = __fmul_rn(__fdiv_rn((float)x, (float)n), (float)(kRows - 1));
    const float fl = floorf(i);
    Lerp l;
    l.f = (int)fl;
    l.c = min(l.f + 1, kRows - 1);
    l.d = __fsub_rn(i, fl);
    return l;
}

// table[f] * (1 - d) + table[c] * d, one float4 of features
__device__ __forceinline__ float4 lerp4(const float4 a, const float4 b, float d) {
    const float e = __fsub_rn(1.f, d);
    return make_float4(__fadd_rn(__fmul_rn(a.x, e), __fmul_rn(b.x, d)), __fadd_rn(__fmul_rn(a.y, e), __fmul_rn(b.y, d)),
                       __fadd_rn(__fmul_rn(a.z, e), __fmul_rn(b.z, d)), __fadd_rn(__fmul_rn(a.w, e), __fmul_rn(b.w, d)));
}

// One thread per float4 of the output: pixel p = t / 64, quad q = t % 64 (q < 32: column table at x, else row table at y).
__global__ void pos_learned_fwd_kernel(const float4* __restrict__ col, const float4* __restrict__ row, int H, int W,
                                       float4* __restrict__ out) {
    constexpr int kQuads = kOut / 4, kTabQuads = kFeats / 4;
    const long long n = (long long)H * W * kQuads;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const long long p = t / kQuads;
        const int q = (int)(t - p * kQuads);
        const bool is_col = q < kTabQuads;
        const int y = (int)(p / W), x = (int)(p - (long long)y * W);
        const Lerp l = is_col ? lerp_of(x, W) : lerp_of(y, H);
        const float4* tab = is_col ? col : row;
        const int k = is_col ? q : q - kTabQuads;
        out[t] = lerp4(tab[l.f * kTabQuads + k], tab[l.c * kTabQuads + k], l.d);
    }
}

// One CTA per (table, embedding row r), one thread per feature.  The coordinates whose floor or ceil is r are walked in ascending
// order; for each, the gradient is summed over the other axis in ascending order, weighted by (1 - d) for the floor and d for the
// ceil (both when they coincide at the clamp), and accumulated.  Rows no coordinate touches get zero.
__global__ void __launch_bounds__(kFeats) pos_learned_bwd_kernel(const float* __restrict__ dpos, int H, int W, float* __restrict__ dcol,
                                                                 float* __restrict__ drow) {
    const int r = blockIdx.x % kRows;
    const bool is_col = blockIdx.x < kRows;
    const int ch = threadIdx.x;
    const int n = is_col ? W : H;              // the interpolated axis
    const int m = is_col ? H : W;              // the summed axis
    // element (a, b) of the interpolated / summed axes: pixel (y, x) = (b, a) for the column table, (a, b) for the row table
    const long long sa = is_col ? kOut : (long long)W * kOut;
    const long long sb = is_col ? (long long)W * kOut : kOut;
    const float* g = dpos + (is_col ? 0 : kFeats) + ch;
    float acc = 0.f;
    for (int a = 0; a < n; ++a) {
        const Lerp l = lerp_of(a, n);
        if (l.f > r) break;                    // i is non-decreasing in a
        if (l.f != r && l.c != r) continue;
        const float* ga = g + a * sa;
        float s = 0.f;
        for (int b = 0; b < m; ++b) s = __fadd_rn(s, ga[b * sb]);
        if (l.f == r) acc = __fadd_rn(acc, __fmul_rn(s, __fsub_rn(1.f, l.d)));
        if (l.c == r) acc = __fadd_rn(acc, __fmul_rn(s, l.d));
    }
    (is_col ? dcol : drow)[r * kFeats + ch] = acc;
}

}  // namespace

extern "C" {

int mdb_pos_learned_forward_f32(const float* col, const float* row, int H, int W, float* out, void* stream) {
    if (H < 0 || W < 0) return MDB_EINVAL;
    if (H == 0 || W == 0) return 0;
    if (!col || !row || !out) return MDB_EINVAL;
    if (((uintptr_t)col | (uintptr_t)row | (uintptr_t)out) & 15) return MDB_EUNSUPPORTED;   // float4 loads and stores
    const long long n = (long long)H * W * (kOut / 4);
    pos_learned_fwd_kernel<<<grid_cap(n, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const float4*>(col), reinterpret_cast<const float4*>(row), H, W, reinterpret_cast<float4*>(out));
    return (int)cudaGetLastError();
}

int mdb_pos_learned_backward_f32(const float* dpos, int H, int W, float* dcol, float* drow, void* stream) {
    if (H <= 0 || W <= 0) return MDB_EINVAL;
    if (!dpos || !dcol || !drow) return MDB_EINVAL;
    pos_learned_bwd_kernel<<<2 * kRows, kFeats, 0, static_cast<cudaStream_t>(stream)>>>(dpos, H, W, dcol, drow);
    return (int)cudaGetLastError();
}

}  // extern "C"
