// heads.cu -- the small elementwise chains around the decoder / prediction heads and the depth predictor's tail, fused
// into one forward and one backward kernel each (the reference runs them as ~10-20 separate elementwise launches apiece,
// which under a CUDA graph still cost 3-7 us each: ~350 launches per training step).
//   * box refinement        depthaware_transformer.py:602-613   sigmoid(bbox_embed(out) + inverse_sigmoid(ref))
//   * depth of a query      monodetr.py:230-262                 mean of (regressed, geometric, depth-map) depth
//   * depth predictor tail  depth_predictor.py:74-104           softmax over the 81 bins -> expected depth -> embedding lerp
//   * mean of three maps    depth_predictor.py:66               (src_8 + src_16 + src_32) / 3
//   * sum_k mean(x_k^2)     the surrogate loss of SURVEY.md 8(d) (bench.py's training step), multi-tensor
// fp32, HBM- / latency-bound; parity against the plain PyTorch expressions in tests/test_heads_gpu.py.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

using namespace mdb;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---- box refinement ---------------------------------------------------------------------------------------------------
// y[i][k] = sigmoid(tmp[i][k] + (k < rd ? inverse_sigmoid(ref[i][k]) : 0)),  inverse_sigmoid of utils/misc.py:473-477
__global__ void box_refine_fwd_kernel(const float* __restrict__ tmp, const float* __restrict__ ref, float* __restrict__ y, long long n,
                                      int rd) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n * 6; i += (long long)gridDim.x * blockDim.x) {
        const long long q = i / 6;
        const int k = (int)(i - q * 6);
        float v = tmp[i];
        if (k < rd) {
            const float x = fminf(fmaxf(ref[q * rd + k], 0.f), 1.f);
            v += logf(fmaxf(x, 1e-5f) / fmaxf(1.f - x, 1e-5f));
        }
        y[i] = sigmoidf_(v);
    }
}
__global__ void box_refine_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ ref,
                                      float* __restrict__ dtmp, float* __restrict__ dref /* or null */, long long n, int rd) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n * 6; i += (long long)gridDim.x * blockDim.x) {
        const long long q = i / 6;
        const int k = (int)(i - q * 6);
        const float yy = y[i];
        const float g = dy[i] * yy * (1.f - yy);
        dtmp[i] = g;
        if (dref && k < rd) {
            const float r = ref[q * rd + k];
            float d = 0.f;
            if (r >= 0.f && r <= 1.f) {                            // clamp(min=0, max=1) passes the gradient inside [0, 1]
                if (r >= 1e-5f) d += 1.f / r;                      // clamp(min=eps) of x
                if (1.f - r >= 1e-5f) d += 1.f / (1.f - r);        // clamp(min=eps) of 1 - x
            }
            dref[q * rd + k] = g * d;
        }
    }
}

// ---- depth of a query ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bilinear_ac(float cx, float cy, int H, int W, int& x0, int& y0, float& lx, float& ly) {
    const float x = (cx + 1.f) * 0.5f * (float)(W - 1), y = (cy + 1.f) * 0.5f * (float)(H - 1);   // align_corners=True
    const float xf = floorf(x), yf = floorf(y);
    x0 = (int)xf; y0 = (int)yf; lx = x - xf; ly = y - yf;
}
__global__ void head_depth_fwd_kernel(const float* __restrict__ coord, const float* __restrict__ size3d, const float* __restrict__ reg,
                                      const float* __restrict__ wdepth, const float* __restrict__ calibs /*[B][3][4]*/,
                                      const float* __restrict__ img_sizes /*[B][2]*/, float* __restrict__ out, int B, int N, int H, int W) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * N) return;
    const int b = i / N;
    const float* c = coord + (size_t)i * 6;
    const float hn = c[4] + c[5];
    const float h = fmaxf(hn * img_sizes[2 * b + 1], 1.f);
    const float geo = size3d[(size_t)i * 3] / h * calibs[12 * b];
    int x0, y0; float lx, ly;
    bilinear_ac((c[0] - 0.5f) * 2.f, (c[1] - 0.5f) * 2.f, H, W, x0, y0, lx, ly);
    const float* d = wdepth + (size_t)b * H * W;
    auto tap = [&](int yy, int xx) { return (xx >= 0 && xx <= W - 1 && yy >= 0 && yy <= H - 1) ? d[yy * W + xx] : 0.f; };
    const float dm = tap(y0, x0) * (1.f - ly) * (1.f - lx) + tap(y0, x0 + 1) * (1.f - ly) * lx + tap(y0 + 1, x0) * ly * (1.f - lx) +
                     tap(y0 + 1, x0 + 1) * ly * lx;
    const float dr = 1.f / (sigmoidf_(reg[2 * i]) + 1e-6f) - 1.f;
    out[2 * i] = (dr + geo + dm) / 3.f;
    out[2 * i + 1] = reg[2 * i + 1];
}
// dwdepth must be zero-filled (or hold other contributions): accumulated with atomics
__global__ void head_depth_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ coord, const float* __restrict__ size3d,
                                      const float* __restrict__ reg, const float* __restrict__ calibs, const float* __restrict__ img_sizes,
                                      float* __restrict__ dcoord, float* __restrict__ dsize3d, float* __restrict__ dreg,
                                      float* __restrict__ dwdepth, int B, int N, int H, int W) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * N) return;
    const int b = i / N;
    const float* c = coord + (size_t)i * 6;
    const float g = dout[2 * i] / 3.f;
    const float ih = img_sizes[2 * b + 1], fu = calibs[12 * b];
    const float hn = c[4] + c[5];
    const float hraw = hn * ih;
    const float h = fmaxf(hraw, 1.f);
    const float s0 = size3d[(size_t)i * 3];
    const float dh = -g * s0 * fu / (h * h);
    const float dhn = (hraw >= 1.f) ? dh * ih : 0.f;
    float* dc = dcoord + (size_t)i * 6;
    dc[0] = dc[1] = dc[2] = dc[3] = 0.f;
    dc[4] = dc[5] = dhn;
    float* ds = dsize3d + (size_t)i * 3;
    ds[0] = g * fu / h; ds[1] = ds[2] = 0.f;
    const float sg = sigmoidf_(reg[2 * i]);
    const float den = sg + 1e-6f;
    dreg[2 * i] = -g * sg * (1.f - sg) / (den * den);
    dreg[2 * i + 1] = dout[2 * i + 1];
    int x0, y0; float lx, ly;
    bilinear_ac((c[0] - 0.5f) * 2.f, (c[1] - 0.5f) * 2.f, H, W, x0, y0, lx, ly);
    float* d = dwdepth + (size_t)b * H * W;
    auto put = [&](int yy, int xx, float w) { if (xx >= 0 && xx <= W - 1 && yy >= 0 && yy <= H - 1) atomicAdd(d + yy * W + xx, w * g); };
    put(y0, x0, (1.f - ly) * (1.f - lx)); put(y0, x0 + 1, (1.f - ly) * lx); put(y0 + 1, x0, ly * (1.f - lx)); put(y0 + 1, x0 + 1, ly * lx);
}

// ---- depth predictor tail ---------------------------------------------------------------------------------------------
// One warp per pixel: p = softmax(logits[81]); wd = sum p * bins; x = clamp(wd, 0, dmax); f = floor(x); c = min(f + 1, E - 1);
// ip[ch] = emb[f][ch] * (1 - (x - f)) + emb[c][ch] * (x - f)          (depth_predictor.py:74-77, 93-104)
constexpr int kMaxBins = 96;
__global__ void __launch_bounds__(256)
depth_tail_fwd_kernel(const float* __restrict__ logits, const float* __restrict__ bins, const float* __restrict__ emb,
                      float* __restrict__ wdepth, float* __restrict__ ip, long long npix, int nb, int E, int C, float dmax) {
    const int lane = threadIdx.x & 31;
    const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long px = warp; px < npix; px += nwarps) {
        const float* lg = logits + px * nb;
        float v[3], mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int j = lane + 32 * k;
            v[k] = j < nb ? lg[j] : -INFINITY;
            mx = fmaxf(mx, v[k]);
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float se = 0.f, sw = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int j = lane + 32 * k;
            const float e = j < nb ? expf(v[k] - mx) : 0.f;
            se += e;
            sw += j < nb ? e * bins[j] : 0.f;
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            se += __shfl_xor_sync(0xffffffffu, se, o);
            sw += __shfl_xor_sync(0xffffffffu, sw, o);
        }
        const float wd = sw / se;
        if (lane == 0) wdepth[px] = wd;
        const float x = fminf(fmaxf(wd, 0.f), dmax);
        const float f = floorf(x);
        const float delta = x - f;
        const int fi = (int)f, ci = min(fi + 1, E - 1);
        const float* e0 = emb + (size_t)fi * C;
        const float* e1 = emb + (size_t)ci * C;
        float* o = ip + px * C;
        for (int ch = lane * 4; ch < C; ch += 128) {
            const float4 a = *reinterpret_cast<const float4*>(e0 + ch), bb = *reinterpret_cast<const float4*>(e1 + ch);
            *reinterpret_cast<float4*>(o + ch) = make_float4(a.x * (1.f - delta) + bb.x * delta, a.y * (1.f - delta) + bb.y * delta,
                                                             a.z * (1.f - delta) + bb.z * delta, a.w * (1.f - delta) + bb.w * delta);
        }
    }
}
// backward: d_ip (npix, C), d_wd_ext (npix) = gradient reaching weighted_depth from elsewhere (the heads' depth-map lookup), or null.
// demb (E, C) accumulated through a per-CTA shared-memory copy (the 61 rows are hit by every pixel), dlogits (npix, nb) written.
__global__ void __launch_bounds__(256)
depth_tail_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ bins, const float* __restrict__ emb,
                      const float* __restrict__ d_ip, const float* __restrict__ d_wd_ext, float* __restrict__ dlogits,
                      float* __restrict__ demb, long long npix, int nb, int E, int C, float dmax) {
    extern __shared__ float sacc[];                                // [E][C]
    for (int i = threadIdx.x; i < E * C; i += blockDim.x) sacc[i] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    // Embedding gradient: neighbouring pixels mostly fall into the same depth bin, so every warp walks a CONTIGUOUS pixel range and
    // keeps the two rows it is adding to (floor, ceil) in registers (C <= 256: 8 channels per lane and row), spilling them to the CTA's
    // shared copy only when the bin changes.  (Plain shared-memory atomics per pixel serialise completely when the depth map is flat.)
    const long long per = (npix + nwarps - 1) / nwarps;
    const long long px_begin = warp * per, px_end = min(npix, px_begin + per);
    int cur_f = -1, cur_c = -1;
    float af[8], ac[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) af[k] = ac[k] = 0.f;
    auto flush = [&]() {
        if (cur_f < 0) return;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ch = (k >> 2) * 128 + lane * 4 + (k & 3);
            if (ch < C) {
                if (af[k] != 0.f) atomicAdd(sacc + cur_f * C + ch, af[k]);
                if (ac[k] != 0.f) atomicAdd(sacc + cur_c * C + ch, ac[k]);
            }
            af[k] = ac[k] = 0.f;
        }
    };
    for (long long px = px_begin; px < px_end; ++px) {
        const float* lg = logits + px * nb;
        float v[3], mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int j = lane + 32 * k;
            v[k] = j < nb ? lg[j] : -INFINITY;
            mx = fmaxf(mx, v[k]);
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float e[3], se = 0.f, sw = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int j = lane + 32 * k;
            e[k] = j < nb ? expf(v[k] - mx) : 0.f;
            se += e[k];
            sw += j < nb ? e[k] * bins[j] : 0.f;
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            se += __shfl_xor_sync(0xffffffffu, se, o);
            sw += __shfl_xor_sync(0xffffffffu, sw, o);
        }
        const float wd = sw / se;
        const float x = fminf(fmaxf(wd, 0.f), dmax);
        const float f = floorf(x);
        const float delta = x - f;
        const int fi = (int)f, ci = min(fi + 1, E - 1);
        if (fi != cur_f) {                                         // uniform across the warp
            flush();
            cur_f = fi; cur_c = ci;
        }
        const float* e0 = emb + (size_t)fi * C;
        const float* e1 = emb + (size_t)ci * C;
        const float* g = d_ip + px * C;
        float dd = 0.f;                                            // d loss / d delta = sum_ch g (e1 - e0)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int ch = hh * 128 + lane * 4;
            if (ch < C) {
                const float4 gg = *reinterpret_cast<const float4*>(g + ch);
                const float4 a = *reinterpret_cast<const float4*>(e0 + ch), bb = *reinterpret_cast<const float4*>(e1 + ch);
                dd += gg.x * (bb.x - a.x) + gg.y * (bb.y - a.y) + gg.z * (bb.z - a.z) + gg.w * (bb.w - a.w);
                af[hh * 4 + 0] += gg.x * (1.f - delta); af[hh * 4 + 1] += gg.y * (1.f - delta);
                af[hh * 4 + 2] += gg.z * (1.f - delta); af[hh * 4 + 3] += gg.w * (1.f - delta);
                ac[hh * 4 + 0] += gg.x * delta; ac[hh * 4 + 1] += gg.y * delta; ac[hh * 4 + 2] += gg.z * delta; ac[hh * 4 + 3] += gg.w * delta;
            }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) dd += __shfl_xor_sync(0xffffffffu, dd, o);
        // d delta / d wd = 1 inside the clamp (floor has zero gradient); clamp(min=0, max=dmax) passes the gradient on [0, dmax]
        float dwd = (wd >= 0.f && wd <= dmax) ? dd : 0.f;
        if (d_wd_ext) dwd += d_wd_ext[px];
        // wd = sum_j p_j bins_j  ->  dlogit_j = p_j (bins_j - wd) dwd
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int j = lane + 32 * k;
            if (j < nb) dlogits[px * nb + j] = e[k] / se * (bins[j] - wd) * dwd;
        }
    }
    flush();
    __syncthreads();
    for (int i = threadIdx.x; i < E * C; i += blockDim.x) {
        const float a = sacc[i];
        if (a != 0.f) atomicAdd(demb + i, a);
    }
}

// ---- mean of three maps, scale -------------------------------------------------------------------------------------------
__global__ void mean3_kernel(const float4* __restrict__ a, const float4* __restrict__ b, const float4* __restrict__ c,
                             float4* __restrict__ o, long long n4) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 x = a[i], y = b[i], z = c[i];
        o[i] = make_float4((x.x + y.x + z.x) / 3.f, (x.y + y.y + z.y) / 3.f, (x.z + y.z + z.z) / 3.f, (x.w + y.w + z.w) / 3.f);
    }
}
__global__ void scale_kernel(const float4* __restrict__ a, float4* __restrict__ o, long long n4, float s) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 x = a[i];
        o[i] = make_float4(x.x * s, x.y * s, x.z * s, x.w * s);
    }
}

// ---- sum_k mean(x_k^2): multi-tensor forward (one atomicAdd per block) and backward (grad_k = 2 x_k / n_k * dloss) ----
constexpr int kMaxLossTensors = 32;
struct LossTable {
    const float* x[kMaxLossTensors];
    float* g[kMaxLossTensors];
    long long n[kMaxLossTensors];
    int count;
};
__global__ void __launch_bounds__(256) sum_mean_sq_fwd_kernel(const __grid_constant__ LossTable tb, float* __restrict__ loss) {
    __shared__ float part[8];
    const int k = blockIdx.y;
    const float* __restrict__ x = tb.x[k];
    const long long n = tb.n[k];
    float acc = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) acc = fmaf(x[i], x[i], acc);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += part[w];
        atomicAdd(loss, s / (float)n);
    }
}
__global__ void __launch_bounds__(256) sum_mean_sq_bwd_kernel(const __grid_constant__ LossTable tb, const float* __restrict__ dloss) {
    const int k = blockIdx.y;
    const float* __restrict__ x = tb.x[k];
    float* __restrict__ g = tb.g[k];
    const long long n = tb.n[k];
    const float s = 2.f * (*dloss) / (float)n;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) g[i] = x[i] * s;
}

}  // namespace

extern "C" {

int mdb_box_refine_forward_f32(const float* tmp, const float* ref, float* y, long long n, int ref_dim, void* stream) {
    if (n < 0 || (ref_dim != 2 && ref_dim != 6)) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!tmp || !ref || !y) return MDB_EINVAL;
    box_refine_fwd_kernel<<<grid_cap(n * 6, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(tmp, ref, y, n, ref_dim);
    return (int)cudaGetLastError();
}
int mdb_box_refine_backward_f32(const float* dy, const float* y, const float* ref, float* dtmp, float* dref, long long n, int ref_dim,
                                void* stream) {
    if (n < 0 || (ref_dim != 2 && ref_dim != 6)) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!dy || !y || !ref || !dtmp) return MDB_EINVAL;
    box_refine_bwd_kernel<<<grid_cap(n * 6, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(dy, y, ref, dtmp, dref, n, ref_dim);
    return (int)cudaGetLastError();
}

int mdb_head_depth_forward_f32(const float* coord, const float* size3d, const float* depth_reg, const float* wdepth, const float* calibs,
                               const float* img_sizes, float* out, int B, int N, int H, int W, void* stream) {
    if (B <= 0 || N < 0 || H <= 0 || W <= 0) return MDB_EINVAL;
    if (N == 0) return 0;
    if (!coord || !size3d || !depth_reg || !wdepth || !calibs || !img_sizes || !out) return MDB_EINVAL;
    head_depth_fwd_kernel<<<(B * N + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(coord, size3d, depth_reg, wdepth, calibs,
                                                                                              img_sizes, out, B, N, H, W);
    return (int)cudaGetLastError();
}
int mdb_head_depth_backward_f32(const float* dout, const float* coord, const float* size3d, const float* depth_reg, const float* calibs,
                                const float* img_sizes, float* dcoord, float* dsize3d, float* dreg, float* dwdepth, int B, int N, int H,
                                int W, void* stream_) {
    if (B <= 0 || N < 0 || H <= 0 || W <= 0) return MDB_EINVAL;
    if (!dwdepth) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e = cudaMemsetAsync(dwdepth, 0, sizeof(float) * (size_t)B * H * W, stream);
    if (e != cudaSuccess) return (int)e;
    if (N == 0) return 0;
    if (!dout || !coord || !size3d || !depth_reg || !calibs || !img_sizes || !dcoord || !dsize3d || !dreg) return MDB_EINVAL;
    head_depth_bwd_kernel<<<(B * N + 127) / 128, 128, 0, stream>>>(dout, coord, size3d, depth_reg, calibs, img_sizes, dcoord, dsize3d, dreg,
                                                                   dwdepth, B, N, H, W);
    return (int)cudaGetLastError();
}

int mdb_depth_tail_forward_f32(const float* logits, const float* bins, const float* emb, float* wdepth, float* ip, long long npix, int nb,
                               int E, int C, float dmax, void* stream) {
    if (npix < 0 || nb <= 0 || nb > kMaxBins || E <= 0 || C <= 0 || C % 4 || C > 256) return MDB_EINVAL;
    if (npix == 0) return 0;
    if (!logits || !bins || !emb || !wdepth || !ip) return MDB_EINVAL;
    depth_tail_fwd_kernel<<<grid_cap(npix * 32, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(logits, bins, emb, wdepth, ip, npix, nb,
                                                                                                                  E, C, dmax);
    return (int)cudaGetLastError();
}
// demb (E x C) is zero-filled by the call.
int mdb_depth_tail_backward_f32(const float* logits, const float* bins, const float* emb, const float* d_ip, const float* d_wd_ext,
                                float* dlogits, float* demb, long long npix, int nb, int E, int C, float dmax, void* stream_) {
    if (npix < 0 || nb <= 0 || nb > kMaxBins || E <= 0 || C <= 0 || C % 4 || C > 256 || (size_t)E * C * 4 > 96 * 1024) return MDB_EINVAL;
    if (!demb) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e = cudaMemsetAsync(demb, 0, sizeof(float) * (size_t)E * C, stream);
    if (e != cudaSuccess) return (int)e;
    if (npix == 0) return 0;
    if (!logits || !bins || !emb || !d_ip || !dlogits) return MDB_EINVAL;
    const int smem = E * C * 4;
    e = set_max_dynamic_smem(depth_tail_bwd_kernel, 96 * 1024);
    if (e != cudaSuccess) return (int)e;
    depth_tail_bwd_kernel<<<grid_cap(npix * 32, 256, num_sms()), 256, smem, stream>>>(logits, bins, emb, d_ip, d_wd_ext, dlogits, demb, npix, nb, E, C,
                                                                                       dmax);
    return (int)cudaGetLastError();
}

int mdb_mean3_f32(const float* a, const float* b, const float* c, float* out, long long n, void* stream) {
    if (n < 0 || n % 4) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!a || !b || !c || !out) return MDB_EINVAL;
    mean3_kernel<<<grid_cap(n / 4, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const float4*>(a), reinterpret_cast<const float4*>(b), reinterpret_cast<const float4*>(c), reinterpret_cast<float4*>(out), n / 4);
    return (int)cudaGetLastError();
}
int mdb_scale_f32(const float* a, float* out, long long n, float s, void* stream) {
    if (n < 0 || n % 4) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!a || !out) return MDB_EINVAL;
    scale_kernel<<<grid_cap(n / 4, 256, num_sms() * 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const float4*>(a),
                                                                                         reinterpret_cast<float4*>(out), n / 4, s);
    return (int)cudaGetLastError();
}

// loss (1 float, zero-filled by the call) = sum_k mean(x_k^2); x / n are HOST arrays of `count` <= 32 entries
int mdb_sum_mean_squares_forward_f32(int count, const float* const* x, const long long* n, float* loss, void* stream_) {
    if (count < 0 || count > kMaxLossTensors || !loss) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), stream);
    if (e != cudaSuccess) return (int)e;
    if (count == 0) return 0;
    LossTable tb;
    tb.count = count;
    long long nmax = 0;
    for (int k = 0; k < count; ++k) {
        if (!x[k] || n[k] <= 0) return MDB_EINVAL;
        tb.x[k] = x[k]; tb.g[k] = nullptr; tb.n[k] = n[k];
        if (n[k] > nmax) nmax = n[k];
    }
    sum_mean_sq_fwd_kernel<<<dim3(grid_cap(nmax, 256 * 8, 64), count), 256, 0, stream>>>(tb, loss);
    return (int)cudaGetLastError();
}
int mdb_sum_mean_squares_backward_f32(int count, const float* const* x, float* const* g, const long long* n, const float* dloss,
                                      void* stream_) {
    if (count < 0 || count > kMaxLossTensors || !dloss) return MDB_EINVAL;
    if (count == 0) return 0;
    LossTable tb;
    tb.count = count;
    long long nmax = 0;
    for (int k = 0; k < count; ++k) {
        if (!x[k] || !g[k] || n[k] <= 0) return MDB_EINVAL;
        tb.x[k] = x[k]; tb.g[k] = g[k]; tb.n[k] = n[k];
        if (n[k] > nmax) nmax = n[k];
    }
    sum_mean_sq_bwd_kernel<<<dim3(grid_cap(nmax, 256 * 4, 128), count), 256, 0, static_cast<cudaStream_t>(stream_)>>>(tb, dloss);
    return (int)cudaGetLastError();
}

}  // extern "C"
