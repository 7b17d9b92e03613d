// dab.cu -- the anchor-box query branch of the decoder (use_dab, depthaware_transformer.py:29-65, :255-260, :557-599):
//   * sine embedding of 6-d boxes      gen_sineembed_for_position: (N, 6) -> (N, 768), layout [y | x | l | r | t | b]
//   * query-position product          query_pos = query_scale(output) * ref_point_head(sine), or the shared layer-0 rows
//   * box gradient of the sampling    d loc -> d (cx, cy, l, r, t, b) for 6-d boxes that require grad (layer 0's anchors)
//   * anchors                          sigmoid(refpoint_embed) and the fixed-order sum of its three gradient contributions
// Every reduction runs in a fixed order (no atomics), so the reproducible mode covers this branch without a separate path.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

using namespace mdb;

constexpr int kSineFeats = 128;        // per box component
constexpr int kSineOut = 6 * kSineFeats;

// Block j of the output embeds box component kSrc[j]: [y | x | l | r | t | b] (gen_sineembed_for_position, 6-d case).
__device__ __forceinline__ int sine_src(int j) { return j == 0 ? 1 : (j == 1 ? 0 : j); }

// dim_t[i] = 10000 ** (2 * (i // 2) / 128) in fp32, as torch evaluates it
__device__ __forceinline__ float sine_dim_t(int i) { return powf(10000.f, (float)(2 * (i >> 1)) / 128.f); }

__global__ void sine_embed_fwd_kernel(const float* __restrict__ box, float* __restrict__ out, long long n) {
    const float scale = 6.283185307179586f;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n * kSineOut; t += (long long)gridDim.x * blockDim.x) {
        const long long r = t / kSineOut;
        const int c = (int)(t - r * kSineOut);
        const int j = c / kSineFeats, i = c % kSineFeats;
        const float e = box[r * 6 + sine_src(j)] * scale;
        const float p = e / sine_dim_t(i);
        out[t] = (i & 1) ? cosf(p) : sinf(p);
    }
}

// One warp per (row, component): lane l owns features l, l + 32, l + 64, l + 96; then a fixed butterfly.
__global__ void sine_embed_bwd_kernel(const float* __restrict__ box, const float* __restrict__ dout, float* __restrict__ dbox,
                                      long long n) {
    const float scale = 6.283185307179586f;
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long w = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); w < n * 6; w += warps) {
        const long long r = w / 6;
        const int k = (int)(w - r * 6);                       // box component
        const int j = sine_src(k);                            // output block that embeds it (the map is its own inverse)
        const float e = box[r * 6 + k] * scale;
        const float* g = dout + r * kSineOut + j * kSineFeats;
        float acc = 0.f;
#pragma unroll
        for (int s = 0; s < kSineFeats / 32; ++s) {
            const int i = s * 32 + lane;
            const float d = sine_dim_t(i);
            const float p = e / d;
            const float dp = (i & 1) ? -sinf(p) : cosf(p);
            acc = fmaf(g[i], dp * (scale / d), acc);
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) dbox[w] = acc;
    }
}

// out[b][r][c] = (scale ? scale[b][r][c] : 1) * raw[shared ? r : b * rows + r][c]
__global__ void query_pos_fwd_kernel(const float* __restrict__ scale, const float* __restrict__ raw, float* __restrict__ out, int B,
                                     long long rows, int C, int shared) {
    const long long per = rows * C, n = (long long)B * per;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const float v = raw[shared ? t % per : t];
        out[t] = scale ? scale[t] * v : v;
    }
}

// dscale = dqp * raw; draw = dqp * scale, summed over b = 0..B-1 in order when raw is shared
__global__ void query_pos_bwd_kernel(const float* __restrict__ dqp, const float* __restrict__ scale, const float* __restrict__ raw,
                                     float* __restrict__ dscale, float* __restrict__ draw, int B, long long rows, int C, int shared) {
    const long long per = rows * C;
    const long long n = shared ? per : (long long)B * per;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        if (shared) {
            const float rv = raw[t];
            float acc = 0.f;
            for (int b = 0; b < B; ++b) {
                const long long u = (long long)b * per + t;
                const float g = dqp[u];
                if (dscale) dscale[u] = g * rv;
                acc = scale ? fmaf(g, scale[u], acc) : acc + g;         // explicit: the same rounding in every code path
            }
            if (draw) draw[t] = acc;
        } else {
            const float g = dqp[t];
            if (dscale) dscale[t] = g * raw[t];
            if (draw) draw[t] = scale ? g * scale[t] : g;
        }
    }
}

// loc = ref_xy + off / P * (l + r, t + b) / 2:  d(cx, cy) = sum d loc,  d l = d r = sum d loc_x off_x / (2P),
// d t = d b = sum d loc_y off_y / (2P), over (head, level, point) -- and over the batch when the boxes are shared.
// One warp per output row: lane l owns (head, level, point) indices l, l + 32, ...; batches in order, then a fixed butterfly.
__global__ void msda_ref_grad_kernel(const float* __restrict__ dloc, const float* __restrict__ off, int B, int Lq, int MLP, int P,
                                     int shared, float* __restrict__ dref) {
    const int lane = threadIdx.x & 31;
    const long long rows = shared ? Lq : (long long)B * Lq;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long w = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); w < rows; w += warps) {
        float cx = 0.f, cy = 0.f, wx = 0.f, wy = 0.f;
        const int nb = shared ? B : 1;
        for (int b = 0; b < nb; ++b) {
            const long long u = shared ? (long long)b * Lq + w : w;     // (b, q) row of dloc / off
            const float2* dl = reinterpret_cast<const float2*>(dloc) + u * MLP;
            const float2* of = reinterpret_cast<const float2*>(off) + u * MLP;
            for (int i = lane; i < MLP; i += 32) {
                const float2 g = dl[i], o = of[i];
                cx += g.x; cy += g.y;
                wx = fmaf(g.x, o.x, wx); wy = fmaf(g.y, o.y, wy);
            }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            cx += __shfl_xor_sync(0xffffffffu, cx, o);
            cy += __shfl_xor_sync(0xffffffffu, cy, o);
            wx += __shfl_xor_sync(0xffffffffu, wx, o);
            wy += __shfl_xor_sync(0xffffffffu, wy, o);
        }
        if (lane == 0) {
            const float h = 0.5f / (float)P;
            float* d = dref + w * 6;
            d[0] = cx; d[1] = cy;
            d[2] = d[3] = wx * h;
            d[4] = d[5] = wy * h;
        }
    }
}

// box gradient from the fused backward's partials part (B, Lq, ML, 4) = [sum dx, sum dy, sum dx off_x, sum dy off_y] per
// (head, level): one warp per output row, lane l owns (head, level) entries l, l + 32, ...; batches in order, fixed butterfly.
__global__ void ref_partials_reduce_kernel(const float4* __restrict__ part, int B, int Lq, int ML, int P, int shared,
                                           float* __restrict__ dref) {
    const int lane = threadIdx.x & 31;
    const long long rows = shared ? Lq : (long long)B * Lq;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long w = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); w < rows; w += warps) {
        float cx = 0.f, cy = 0.f, wx = 0.f, wy = 0.f;
        const int nb = shared ? B : 1;
        for (int b = 0; b < nb; ++b) {
            const long long u = shared ? (long long)b * Lq + w : w;
            for (int i = lane; i < ML; i += 32) {
                const float4 t = part[u * ML + i];
                cx += t.x; cy += t.y; wx += t.z; wy += t.w;
            }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            cx += __shfl_xor_sync(0xffffffffu, cx, o);
            cy += __shfl_xor_sync(0xffffffffu, cy, o);
            wx += __shfl_xor_sync(0xffffffffu, wx, o);
            wy += __shfl_xor_sync(0xffffffffu, wy, o);
        }
        if (lane == 0) {
            const float h = 0.5f / (float)P;
            float* d = dref + w * 6;
            d[0] = cx; d[1] = cy;
            d[2] = d[3] = wx * h;
            d[4] = d[5] = wy * h;
        }
    }
}

__global__ void anchor_fwd_kernel(const float* __restrict__ w, float* __restrict__ r, float* __restrict__ r2, float* __restrict__ rb, int B,
                                  long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const float s = 1.f / (1.f + expf(-w[t]));
        r[t] = s;
        r2[t] = s;
        for (int b = 0; b < B; ++b) rb[(long long)b * n + t] = s;
    }
}

// dw = (d_sine + d_msda + sum_b d_head[b]) * r (1 - r), in that order; a NULL contribution is zero
__global__ void anchor_bwd_kernel(const float* __restrict__ r, const float* __restrict__ d_sine, const float* __restrict__ d_msda,
                                  const float* __restrict__ d_head, int B, long long n, float* __restrict__ dw) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        float acc = d_sine ? d_sine[t] : 0.f;
        if (d_msda) acc += d_msda[t];
        if (d_head)
            for (int b = 0; b < B; ++b) acc += d_head[(long long)b * n + t];
        const float s = r[t];
        dw[t] = acc * (s * (1.f - s));
    }
}

}  // namespace

extern "C" {

int mdb_dab_sine_embed_forward_f32(const float* box, float* out, long long n, void* stream) {
    if (n < 0) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!box || !out) return MDB_EINVAL;
    sine_embed_fwd_kernel<<<grid_cap(n * kSineOut, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(box, out, n);
    return (int)cudaGetLastError();
}

int mdb_dab_sine_embed_backward_f32(const float* box, const float* dout, float* dbox, long long n, void* stream) {
    if (n < 0) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!box || !dout || !dbox) return MDB_EINVAL;
    sine_embed_bwd_kernel<<<grid_cap(n * 6, 256 / 32, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(box, dout, dbox, n);
    return (int)cudaGetLastError();
}

int mdb_dab_query_pos_forward_f32(const float* scale, const float* raw, float* out, int B, long long rows, int C, int shared,
                                  void* stream) {
    if (B < 0 || rows < 0 || C < 0) return MDB_EINVAL;
    const long long n = (long long)B * rows * C;
    if (n == 0) return 0;
    if (!raw || !out) return MDB_EINVAL;
    query_pos_fwd_kernel<<<grid_cap(n, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(scale, raw, out, B, rows, C,
                                                                                                         shared);
    return (int)cudaGetLastError();
}

int mdb_dab_query_pos_backward_f32(const float* dqp, const float* scale, const float* raw, float* dscale, float* draw, int B,
                                   long long rows, int C, int shared, void* stream) {
    if (B < 0 || rows < 0 || C < 0) return MDB_EINVAL;
    const long long n = (shared ? 1LL : (long long)B) * rows * C;
    if (n == 0 || B == 0) return 0;
    if (!dqp || !raw || (dscale && !scale)) return MDB_EINVAL;
    query_pos_bwd_kernel<<<grid_cap(n, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(dqp, scale, raw, dscale, draw, B,
                                                                                                         rows, C, shared);
    return (int)cudaGetLastError();
}

int mdb_msda_ref_grad_f32(const float* grad_loc, const float* offsets, int B, int Lq, int M, int L, int P, int shared, float* dref,
                          void* stream) {
    if (B < 0 || Lq < 0 || M <= 0 || L <= 0 || P <= 0) return MDB_EINVAL;
    const long long rows = shared ? (long long)Lq : (long long)B * Lq;
    if (rows == 0) return 0;
    if (!grad_loc || !offsets || !dref) return MDB_EINVAL;
    if (((uintptr_t)grad_loc | (uintptr_t)offsets) & 7) return MDB_EUNSUPPORTED;      // read as float2
    msda_ref_grad_kernel<<<grid_cap(rows, 256 / 32, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(grad_loc, offsets, B, Lq,
                                                                                                                 M * L * P, P, shared, dref);
    return (int)cudaGetLastError();
}

int mdb_msda_ref_partials_reduce_f32(const float* ref_part, int B, int Lq, int M, int L, int P, int shared, float* dref, void* stream) {
    if (B < 0 || Lq < 0 || M <= 0 || L <= 0 || P <= 0) return MDB_EINVAL;
    const long long rows = shared ? (long long)Lq : (long long)B * Lq;
    if (rows == 0) return 0;
    if (!ref_part || !dref) return MDB_EINVAL;
    if ((uintptr_t)ref_part & 15) return MDB_EUNSUPPORTED;                           // read as float4
    ref_partials_reduce_kernel<<<grid_cap(rows, 256 / 32, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const float4*>(ref_part), B, Lq, M * L, P, shared, dref);
    return (int)cudaGetLastError();
}

int mdb_dab_anchor_forward_f32(const float* w, float* r, float* r2, float* r_batch, int B, long long n, void* stream) {
    if (B < 0 || n < 0) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!w || !r || !r2 || (B > 0 && !r_batch)) return MDB_EINVAL;
    anchor_fwd_kernel<<<grid_cap(n, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(w, r, r2, r_batch, B, n);
    return (int)cudaGetLastError();
}

int mdb_dab_anchor_backward_f32(const float* r, const float* d_sine, const float* d_msda, const float* d_head, int B, long long n, float* dw,
                                void* stream) {
    if (B < 0 || n < 0) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!r || !dw) return MDB_EINVAL;
    anchor_bwd_kernel<<<grid_cap(n, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(r, d_sine, d_msda, d_head, B, n, dw);
    return (int)cudaGetLastError();
}

}  // extern "C"
