// norm.cu -- LayerNorm (fused with the residual add and dropout that precede it everywhere on the
// reference path: depthaware_transformer.py:348-349,341-343,461-462,502-503,509-510;
// depth_predictor/transformer.py:60-65) and GroupNorm(32, C) on NHWC activations (monodetr.py:83-91,
// depth_predictor.py:29-45, optionally fused with ReLU), forward and backward, for sm_90a.
// These are HBM-bound passes: one read of each input, one write of each output, fp32 statistics.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"
#include "rng.cuh"

namespace {

using namespace mdb;

constexpr int LN_THREADS = 256;      // 8 warps = 8 rows per CTA iteration
constexpr int LN_MAXV = 8;           // float4 vectors per lane -> C <= 1024

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// y = LN(x + drop(res)) * gamma + beta ; one warp per row, NV float4 per lane (C = 128*NV)
template <int NV>
__global__ void __launch_bounds__(LN_THREADS)
add_ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ res, const float* __restrict__ gamma,
                  const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ mean_out,
                  float* __restrict__ rstd_out, long long M, float eps, float drop_p,
                  const unsigned long long* __restrict__ seed_ptr, unsigned long long site) {
    constexpr int C = 128 * NV;
    const int lane = threadIdx.x & 31;
    const long long warp = (long long)blockIdx.x * (LN_THREADS / 32) + (threadIdx.x >> 5);
    const long long nwarps = (long long)gridDim.x * (LN_THREADS / 32);
    const unsigned long long seed = (drop_p > 0.f) ? (*seed_ptr + site * 0x9E3779B97F4A7C15ull) : 0ull;
    const float inv_keep = 1.f / (1.f - drop_p);
    float4 g[NV], b[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        g[i] = *reinterpret_cast<const float4*>(gamma + (i * 32 + lane) * 4);
        b[i] = *reinterpret_cast<const float4*>(beta + (i * 32 + lane) * 4);
    }
    for (long long row = warp; row < M; row += nwarps) {
        float4 z[NV];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const size_t off = (size_t)row * C + (i * 32 + lane) * 4;
            z[i] = *reinterpret_cast<const float4*>(x + off);
            if (res) {
                float4 r = *reinterpret_cast<const float4*>(res + off);
                if (drop_p > 0.f) {
                    float u[4];
                    mdb::rng_uniform4(seed, off >> 2, u);
                    r.x = u[0] >= drop_p ? r.x * inv_keep : 0.f;
                    r.y = u[1] >= drop_p ? r.y * inv_keep : 0.f;
                    r.z = u[2] >= drop_p ? r.z * inv_keep : 0.f;
                    r.w = u[3] >= drop_p ? r.w * inv_keep : 0.f;
                }
                z[i].x += r.x; z[i].y += r.y; z[i].z += r.z; z[i].w += r.w;
            }
            s += z[i].x + z[i].y + z[i].z + z[i].w;
        }
        const float mean = warp_sum(s) * (1.f / C);
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const float a0 = z[i].x - mean, a1 = z[i].y - mean, a2 = z[i].z - mean, a3 = z[i].w - mean;
            v += a0 * a0 + a1 * a1 + a2 * a2 + a3 * a3;
        }
        const float rstd = rsqrtf(warp_sum(v) * (1.f / C) + eps);
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            float4 o;
            o.x = (z[i].x - mean) * rstd * g[i].x + b[i].x;
            o.y = (z[i].y - mean) * rstd * g[i].y + b[i].y;
            o.z = (z[i].z - mean) * rstd * g[i].z + b[i].z;
            o.w = (z[i].w - mean) * rstd * g[i].w + b[i].w;
            *reinterpret_cast<float4*>(y + (size_t)row * C + (i * 32 + lane) * 4) = o;
        }
        if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
    }
}

// dz = LN backward wrt z = x + drop(res); dres = dz * mask/(1-p) (written only when dres != dz semantics needed)
template <int NV>
__global__ void __launch_bounds__(LN_THREADS)
add_ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ res,
                  const float* __restrict__ gamma, const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                  float* __restrict__ dx, float* __restrict__ dres, float* __restrict__ dgamma, float* __restrict__ dbeta,
                  long long M, float drop_p, const unsigned long long* __restrict__ seed_ptr, unsigned long long site) {
    constexpr int C = 128 * NV;
    __shared__ float s_dg[LN_THREADS / 32][C];
    __shared__ float s_db[LN_THREADS / 32][C];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long warp = (long long)blockIdx.x * (LN_THREADS / 32) + wid;
    const long long nwarps = (long long)gridDim.x * (LN_THREADS / 32);
    const unsigned long long seed = (drop_p > 0.f) ? (*seed_ptr + site * 0x9E3779B97F4A7C15ull) : 0ull;
    const float inv_keep = 1.f / (1.f - drop_p);
    float4 g[NV], adg[NV], adb[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        g[i] = *reinterpret_cast<const float4*>(gamma + (i * 32 + lane) * 4);
        adg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        adb[i] = adg[i];
    }
    for (long long row = warp; row < M; row += nwarps) {
        const float mean = mean_in[row], rstd = rstd_in[row];
        float4 xh[NV], gy[NV];
        float keepm[NV][4];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const size_t off = (size_t)row * C + (i * 32 + lane) * 4;
            float4 z = *reinterpret_cast<const float4*>(x + off);
            keepm[i][0] = keepm[i][1] = keepm[i][2] = keepm[i][3] = 1.f;
            if (res) {
                float4 r = *reinterpret_cast<const float4*>(res + off);
                if (drop_p > 0.f) {
                    float u[4];
                    mdb::rng_uniform4(seed, off >> 2, u);
#pragma unroll
                    for (int e = 0; e < 4; ++e) keepm[i][e] = u[e] >= drop_p ? inv_keep : 0.f;
                    r.x *= keepm[i][0]; r.y *= keepm[i][1]; r.z *= keepm[i][2]; r.w *= keepm[i][3];
                }
                z.x += r.x; z.y += r.y; z.z += r.z; z.w += r.w;
            }
            const float4 d = *reinterpret_cast<const float4*>(dy + off);
            xh[i] = make_float4((z.x - mean) * rstd, (z.y - mean) * rstd, (z.z - mean) * rstd, (z.w - mean) * rstd);
            gy[i] = make_float4(d.x * g[i].x, d.y * g[i].y, d.z * g[i].z, d.w * g[i].w);
            s1 += gy[i].x + gy[i].y + gy[i].z + gy[i].w;
            s2 += gy[i].x * xh[i].x + gy[i].y * xh[i].y + gy[i].z * xh[i].z + gy[i].w * xh[i].w;
            adg[i].x += d.x * xh[i].x; adg[i].y += d.y * xh[i].y; adg[i].z += d.z * xh[i].z; adg[i].w += d.w * xh[i].w;
            adb[i].x += d.x; adb[i].y += d.y; adb[i].z += d.z; adb[i].w += d.w;
        }
        s1 = warp_sum(s1) * (1.f / C);
        s2 = warp_sum(s2) * (1.f / C);
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const size_t off = (size_t)row * C + (i * 32 + lane) * 4;
            float4 dz;
            dz.x = rstd * (gy[i].x - s1 - xh[i].x * s2);
            dz.y = rstd * (gy[i].y - s1 - xh[i].y * s2);
            dz.z = rstd * (gy[i].z - s1 - xh[i].z * s2);
            dz.w = rstd * (gy[i].w - s1 - xh[i].w * s2);
            *reinterpret_cast<float4*>(dx + off) = dz;
            if (dres) {
                dz.x *= keepm[i][0]; dz.y *= keepm[i][1]; dz.z *= keepm[i][2]; dz.w *= keepm[i][3];
                *reinterpret_cast<float4*>(dres + off) = dz;
            }
        }
    }
    // reduce dgamma / dbeta over the 8 warps of the CTA, then one atomic per channel per CTA
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = (i * 32 + lane) * 4;
        s_dg[wid][c] = adg[i].x; s_dg[wid][c + 1] = adg[i].y; s_dg[wid][c + 2] = adg[i].z; s_dg[wid][c + 3] = adg[i].w;
        s_db[wid][c] = adb[i].x; s_db[wid][c + 1] = adb[i].y; s_db[wid][c + 2] = adb[i].z; s_db[wid][c + 3] = adb[i].w;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += LN_THREADS) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int w = 0; w < LN_THREADS / 32; ++w) { a += s_dg[w][c]; b += s_db[w][c]; }
        atomicAdd(dgamma + c, a);
        atomicAdd(dbeta + c, b);
    }
}

// ---------------------------------------------------------------------------------------------------
// GroupNorm on NHWC: x[B][HW][C], G groups of C/G = 8 channels.
// stats[b][g] = {sum, sumsq} in double (atomics), then a normalise pass.
// ---------------------------------------------------------------------------------------------------
constexpr int GN_THREADS = 256;

// thread t: channel quad cq = t % (C/4), pixel lane pl = t / (C/4); C/4 must divide 256 (C in {64,128,256,512,1024})
__global__ void __launch_bounds__(GN_THREADS)
gn_stats_kernel(const float* __restrict__ x, double* __restrict__ stats, int HW, int C, int G, int pix_per_block) {
    const int b = blockIdx.y;
    const int cq_n = C / 4;
    const int cq = threadIdx.x % cq_n, pl = threadIdx.x / cq_n, pls = GN_THREADS / cq_n;
    const int p0 = blockIdx.x * pix_per_block, p1 = min(HW, p0 + pix_per_block);
    float s = 0.f, ss = 0.f;
    for (int p = p0 + pl; p < p1; p += pls) {
        const float4 v = *reinterpret_cast<const float4*>(x + ((size_t)b * HW + p) * C + cq * 4);
        s += v.x + v.y + v.z + v.w;
        ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    // channels per group = C/G; quads per group = C/G/4 (2 for 8-channel groups)
    const int qpg = C / G / 4;
    __shared__ float sh[2][GN_THREADS];
    sh[0][threadIdx.x] = s;
    sh[1][threadIdx.x] = ss;
    __syncthreads();
    // one thread per group sums its quads over all pixel lanes
    if (threadIdx.x < G) {
        const int g = threadIdx.x;
        double a = 0.0, c = 0.0;
        for (int l = 0; l < pls; ++l)
            for (int k = 0; k < qpg; ++k) {
                a += sh[0][l * cq_n + g * qpg + k];
                c += sh[1][l * cq_n + g * qpg + k];
            }
        atomicAdd(stats + ((size_t)b * G + g) * 2, a);
        atomicAdd(stats + ((size_t)b * G + g) * 2 + 1, c);
    }
}

__global__ void __launch_bounds__(GN_THREADS)
gn_apply_kernel(const float* __restrict__ x, const double* __restrict__ stats, const float* __restrict__ gamma,
                const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ mean_out,
                float* __restrict__ rstd_out, int B, int HW, int C, int G, float eps, int relu) {
    const long long n4 = (long long)B * HW * C / 4;
    const int cpg = C / G;
    const double inv_n = 1.0 / ((double)HW * cpg);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const long long e = i * 4;
        const int c = (int)(e % C);
        const int b = (int)(e / ((long long)HW * C));
        const int g = c / cpg;
        const double su = stats[((size_t)b * G + g) * 2], sq = stats[((size_t)b * G + g) * 2 + 1];
        const double mu = su * inv_n;
        const float mean = (float)mu;
        const float rstd = rsqrtf((float)(sq * inv_n - mu * mu) + eps);
        const float4 v = *reinterpret_cast<const float4*>(x + e);
        const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
        const float4 be = *reinterpret_cast<const float4*>(beta + c);
        float4 o;
        o.x = (v.x - mean) * rstd * ga.x + be.x;
        o.y = (v.y - mean) * rstd * ga.y + be.y;
        o.z = (v.z - mean) * rstd * ga.z + be.z;
        o.w = (v.w - mean) * rstd * ga.w + be.w;
        if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
        *reinterpret_cast<float4*>(y + e) = o;
        if ((e % ((long long)HW * C)) < C && (c % cpg) == 0) {   // first pixel of the image: publish the statistics
            mean_out[(size_t)b * G + g] = mean;
            rstd_out[(size_t)b * G + g] = rstd;
        }
    }
}

// backward pass 1: per (b, g): s1 = sum dyg, s2 = sum dyg * xhat (double atomics); per channel dgamma/dbeta.
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_stats_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ y,
                    const float* __restrict__ gamma, const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                    double* __restrict__ stats, float* __restrict__ dgamma, float* __restrict__ dbeta, int HW, int C, int G,
                    int pix_per_block, int relu) {
    const int b = blockIdx.y;
    const int cq_n = C / 4, cpg = C / G;
    const int cq = threadIdx.x % cq_n, pl = threadIdx.x / cq_n, pls = GN_THREADS / cq_n;
    const int p0 = blockIdx.x * pix_per_block, p1 = min(HW, p0 + pix_per_block);
    const int c0 = cq * 4, g = c0 / cpg;
    const float mean = mean_in[(size_t)b * G + g], rstd = rstd_in[(size_t)b * G + g];
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c0);
    float s1 = 0.f, s2 = 0.f;
    float4 dg = make_float4(0.f, 0.f, 0.f, 0.f), db = dg;
    for (int p = p0 + pl; p < p1; p += pls) {
        const size_t off = ((size_t)b * HW + p) * C + c0;
        float4 d = *reinterpret_cast<const float4*>(dy + off);
        if (relu) {
            const float4 o = *reinterpret_cast<const float4*>(y + off);
            d.x = o.x > 0.f ? d.x : 0.f; d.y = o.y > 0.f ? d.y : 0.f; d.z = o.z > 0.f ? d.z : 0.f; d.w = o.w > 0.f ? d.w : 0.f;
        }
        const float4 v = *reinterpret_cast<const float4*>(x + off);
        const float4 xh = make_float4((v.x - mean) * rstd, (v.y - mean) * rstd, (v.z - mean) * rstd, (v.w - mean) * rstd);
        s1 += d.x * ga.x + d.y * ga.y + d.z * ga.z + d.w * ga.w;
        s2 += d.x * ga.x * xh.x + d.y * ga.y * xh.y + d.z * ga.z * xh.z + d.w * ga.w * xh.w;
        dg.x += d.x * xh.x; dg.y += d.y * xh.y; dg.z += d.z * xh.z; dg.w += d.w * xh.w;
        db.x += d.x; db.y += d.y; db.z += d.z; db.w += d.w;
    }
    __shared__ float sh[2][GN_THREADS];
    __shared__ float4 shg[GN_THREADS], shb[GN_THREADS];
    sh[0][threadIdx.x] = s1;
    sh[1][threadIdx.x] = s2;
    shg[threadIdx.x] = dg;
    shb[threadIdx.x] = db;
    __syncthreads();
    const int qpg = cpg / 4;
    if (threadIdx.x < G) {
        const int gg = threadIdx.x;
        double a = 0.0, c = 0.0;
        for (int l = 0; l < pls; ++l)
            for (int k = 0; k < qpg; ++k) {
                a += sh[0][l * cq_n + gg * qpg + k];
                c += sh[1][l * cq_n + gg * qpg + k];
            }
        atomicAdd(stats + ((size_t)b * G + gg) * 2, a);
        atomicAdd(stats + ((size_t)b * G + gg) * 2 + 1, c);
    }
    if (threadIdx.x < cq_n) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f), c = a;
        for (int l = 0; l < pls; ++l) {
            const float4 t = shg[l * cq_n + threadIdx.x], u = shb[l * cq_n + threadIdx.x];
            a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
            c.x += u.x; c.y += u.y; c.z += u.z; c.w += u.w;
        }
        const int cc = threadIdx.x * 4;
        atomicAdd(dgamma + cc, a.x); atomicAdd(dgamma + cc + 1, a.y); atomicAdd(dgamma + cc + 2, a.z); atomicAdd(dgamma + cc + 3, a.w);
        atomicAdd(dbeta + cc, c.x); atomicAdd(dbeta + cc + 1, c.y); atomicAdd(dbeta + cc + 2, c.z); atomicAdd(dbeta + cc + 3, c.w);
    }
}

__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ y,
                    const float* __restrict__ gamma, const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                    const double* __restrict__ stats, float* __restrict__ dx, int B, int HW, int C, int G, int relu) {
    const long long n4 = (long long)B * HW * C / 4;
    const int cpg = C / G;
    const float inv_n = 1.f / ((float)HW * cpg);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const long long e = i * 4;
        const int c = (int)(e % C);
        const int b = (int)(e / ((long long)HW * C));
        const int g = c / cpg;
        const float mean = mean_in[(size_t)b * G + g], rstd = rstd_in[(size_t)b * G + g];
        const float m1 = (float)stats[((size_t)b * G + g) * 2] * inv_n;
        const float m2 = (float)stats[((size_t)b * G + g) * 2 + 1] * inv_n;
        float4 d = *reinterpret_cast<const float4*>(dy + e);
        if (relu) {
            const float4 o = *reinterpret_cast<const float4*>(y + e);
            d.x = o.x > 0.f ? d.x : 0.f; d.y = o.y > 0.f ? d.y : 0.f; d.z = o.z > 0.f ? d.z : 0.f; d.w = o.w > 0.f ? d.w : 0.f;
        }
        const float4 v = *reinterpret_cast<const float4*>(x + e);
        const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
        float4 o;
        o.x = rstd * (d.x * ga.x - m1 - (v.x - mean) * rstd * m2);
        o.y = rstd * (d.y * ga.y - m1 - (v.y - mean) * rstd * m2);
        o.z = rstd * (d.z * ga.z - m1 - (v.z - mean) * rstd * m2);
        o.w = rstd * (d.w * ga.w - m1 - (v.w - mean) * rstd * m2);
        *reinterpret_cast<float4*>(dx + e) = o;
    }
}

}  // namespace

extern "C" {

int mdb_add_layernorm_forward_f32(const float* x, const float* res, const float* gamma, const float* beta, float* y,
                                  float* mean, float* rstd, long long M, int C, float eps, float drop_p,
                                  const unsigned long long* seed, unsigned long long site, void* stream_) {
    if (!x || !gamma || !beta || !y || !mean || !rstd || M < 0) return MDB_EINVAL;
    if (C % 128 || C > 128 * LN_MAXV) return MDB_EUNSUPPORTED;
    if (drop_p > 0.f && !seed) return MDB_EINVAL;
    if (M == 0) return 0;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int grid = grid_cap(M, LN_THREADS / 32, num_sms() * 16);
#define MDB_LN_FWD(NV) add_ln_fwd_kernel<NV><<<grid, LN_THREADS, 0, stream>>>(x, res, gamma, beta, y, mean, rstd, M, eps, drop_p, seed, site)
    switch (C / 128) {
        case 1: MDB_LN_FWD(1); break;
        case 2: MDB_LN_FWD(2); break;
        case 4: MDB_LN_FWD(4); break;
        case 8: MDB_LN_FWD(8); break;
        default: return MDB_EUNSUPPORTED;
    }
#undef MDB_LN_FWD
    return (int)cudaGetLastError();
}

// dgamma / dbeta are zero-filled by the call unless accumulate != 0.  dres may be NULL (then the caller uses dx
// for both branches, valid when drop_p == 0).
int mdb_add_layernorm_backward_f32(const float* dy, const float* x, const float* res, const float* gamma,
                                   const float* mean, const float* rstd, float* dx, float* dres, float* dgamma,
                                   float* dbeta, long long M, int C, float drop_p, const unsigned long long* seed,
                                   unsigned long long site, int accumulate, void* stream_) {
    if (!dy || !x || !gamma || !mean || !rstd || !dx || !dgamma || !dbeta || M < 0) return MDB_EINVAL;
    if (C % 128 || C > 512) return MDB_EUNSUPPORTED;   // smem staging of dgamma/dbeta: 8 warps x C x 2 floats
    if (drop_p > 0.f && (!seed || !dres)) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (!accumulate) {
        cudaMemsetAsync(dgamma, 0, sizeof(float) * C, stream);
        cudaMemsetAsync(dbeta, 0, sizeof(float) * C, stream);
    }
    if (M == 0) return 0;
    const int grid = grid_cap(M, LN_THREADS / 32, num_sms() * 4);
#define MDB_LN_BWD(NV) add_ln_bwd_kernel<NV><<<grid, LN_THREADS, 0, stream>>>(dy, x, res, gamma, mean, rstd, dx, dres, dgamma, dbeta, M, drop_p, seed, site)
    switch (C / 128) {
        case 1: MDB_LN_BWD(1); break;
        case 2: MDB_LN_BWD(2); break;
        case 4: MDB_LN_BWD(4); break;
        default: return MDB_EUNSUPPORTED;
    }
#undef MDB_LN_BWD
    return (int)cudaGetLastError();
}

// stats_ws: B*G*2 doubles of workspace (zero-filled by the call).
int mdb_groupnorm_forward_f32(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                              double* stats_ws, int B, int HW, int C, int G, float eps, int relu, void* stream_) {
    if (!x || !gamma || !beta || !y || !mean || !rstd || !stats_ws || B <= 0 || HW <= 0) return MDB_EINVAL;
    if (C % 4 || (GN_THREADS % (C / 4)) || C % G || (C / G) % 4 || G > GN_THREADS) return MDB_EUNSUPPORTED;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaMemsetAsync(stats_ws, 0, sizeof(double) * B * G * 2, stream);
    int blocks = (HW + 255) / 256;
    if (blocks > 64) blocks = 64;
    const int ppb = (HW + blocks - 1) / blocks;
    gn_stats_kernel<<<dim3((HW + ppb - 1) / ppb, B), GN_THREADS, 0, stream>>>(x, stats_ws, HW, C, G, ppb);
    gn_apply_kernel<<<grid_cap((long long)B * HW * C / 4, GN_THREADS, num_sms() * 16), GN_THREADS, 0, stream>>>(x, stats_ws, gamma, beta, y,
                                                                                                 mean, rstd, B, HW, C, G, eps, relu);
    return (int)cudaGetLastError();
}

// y is only read when relu != 0 (mask of the fused ReLU).  dgamma/dbeta zero-filled by the call.
int mdb_groupnorm_backward_f32(const float* dy, const float* x, const float* y, const float* gamma, const float* mean,
                               const float* rstd, float* dx, float* dgamma, float* dbeta, double* stats_ws, int B, int HW,
                               int C, int G, int relu, void* stream_) {
    if (!dy || !x || !gamma || !mean || !rstd || !dx || !dgamma || !dbeta || !stats_ws || B <= 0 || HW <= 0) return MDB_EINVAL;
    if (relu && !y) return MDB_EINVAL;
    if (C % 4 || (GN_THREADS % (C / 4)) || C % G || (C / G) % 4 || G > GN_THREADS) return MDB_EUNSUPPORTED;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaMemsetAsync(stats_ws, 0, sizeof(double) * B * G * 2, stream);
    cudaMemsetAsync(dgamma, 0, sizeof(float) * C, stream);
    cudaMemsetAsync(dbeta, 0, sizeof(float) * C, stream);
    int blocks = (HW + 255) / 256;
    if (blocks > 64) blocks = 64;
    const int ppb = (HW + blocks - 1) / blocks;
    gn_bwd_stats_kernel<<<dim3((HW + ppb - 1) / ppb, B), GN_THREADS, 0, stream>>>(dy, x, y, gamma, mean, rstd, stats_ws, dgamma,
                                                                                  dbeta, HW, C, G, ppb, relu);
    gn_bwd_apply_kernel<<<grid_cap((long long)B * HW * C / 4, GN_THREADS, num_sms() * 16), GN_THREADS, 0, stream>>>(dy, x, y, gamma, mean, rstd,
                                                                                                    stats_ws, dx, B, HW, C, G, relu);
    return (int)cudaGetLastError();
}

}  // extern "C"
