// elementwise.cu -- small HBM-bound helper kernels around the tensor-core convolutions:
// weight packing OIHW -> [tap][O][I] (with the FrozenBatchNorm scale folded in, backbone.py:54-64),
// the inverse for weight gradients, and column sums (bias gradients).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

using namespace mdb;

__global__ void pack_weight_kernel(const float* __restrict__ w, const float* __restrict__ scale, float* __restrict__ out,
                                   int O, int I, int taps, int round_tf32_out) {
    const long long n = (long long)O * I * taps;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        // i indexes the OUTPUT [tap][o][ci] so writes are coalesced
        const int ci = (int)(i % I);
        const long long r = i / I;
        const int o = (int)(r % O);
        const int t = (int)(r / O);
        float v = w[((size_t)o * I + ci) * taps + t];
        if (scale) v *= scale[o];
        if (round_tf32_out) {   // single-pass TF32 mode: round-to-nearest (the tensor core would truncate)
            uint32_t rb;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(rb) : "f"(v));
            v = __uint_as_float(rb);
        }
        out[i] = v;
    }
}

__global__ void unpack_wgrad_kernel(const float* __restrict__ dwp, float* __restrict__ dw, int O, int I, int taps,
                                    int accumulate) {
    const long long n = (long long)O * I * taps;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        // i indexes the OUTPUT [o][ci][tap]
        const int t = (int)(i % taps);
        const long long r = i / taps;
        const int ci = (int)(r % I);
        const int o = (int)(r / I);
        const float v = dwp[((size_t)t * O + o) * I + ci];
        dw[i] = accumulate ? dw[i] + v : v;
    }
}

// Multi-tensor variants: one launch re-lays-out up to kMaxMulti weight tensors (a ResNet-50 has 52 conv weights and the
// step is launch-count sensitive: ~5 us per tiny kernel).  blockIdx.y = tensor, the table travels as a kernel parameter.
constexpr int kMaxMulti = 64;
struct MultiTable {
    const float* src[kMaxMulti];
    const float* scale[kMaxMulti];
    float* dst[kMaxMulti];
    int O[kMaxMulti], I[kMaxMulti], taps[kMaxMulti];
};

__global__ void pack_weight_multi_kernel(const __grid_constant__ MultiTable tb, int round_tf32_out) {
    const int k = blockIdx.y;
    const float* __restrict__ w = tb.src[k];
    const float* __restrict__ scale = tb.scale[k];
    float* __restrict__ out = tb.dst[k];
    const int O = tb.O[k], I = tb.I[k], taps = tb.taps[k];
    const long long n = (long long)O * I * taps;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(i % I);
        const long long r = i / I;
        const int o = (int)(r % O);
        const int t = (int)(r / O);
        float v = w[((size_t)o * I + ci) * taps + t];
        if (scale) v *= scale[o];
        if (round_tf32_out) {
            uint32_t rb;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(rb) : "f"(v));
            v = __uint_as_float(rb);
        }
        out[i] = v;
    }
}

__global__ void unpack_wgrad_multi_kernel(const __grid_constant__ MultiTable tb) {
    const int k = blockIdx.y;
    const float* __restrict__ dwp = tb.src[k];
    float* __restrict__ dw = tb.dst[k];
    const int O = tb.O[k], I = tb.I[k], taps = tb.taps[k];
    const long long n = (long long)O * I * taps;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % taps);
        const long long r = i / taps;
        const int ci = (int)(r % I);
        const int o = (int)(r / I);
        dw[i] = dwp[((size_t)t * O + o) * I + ci];
    }
}


// ---- bf16x3 operand packing -----------------------------------------------------------------------------------------
// Weights of the tensor-core GEMMs, split ONCE per step into error-compensated bf16 pairs and laid out the way the
// kernels' B operand wants them (conv_gemm.cu, BF variant): for every (tap, row n, 32-wide k-block) one 128-byte row
// [hi(k0..k31) | lo(k0..k31)], hi = bf16_rn(v), lo = bf16_rn(v - hi), v = w * (scale ? scale[o] : 1).
//   wf[tap][o][ceil(I/32)][64]   rows = output channels, k = input channels   (fprop)
//   wd[tap][i][ceil(O/32)][64]   rows = input channels,  k = output channels  (dgrad: the transposed weight, K-major)
// Padding k positions (beyond I resp. O) are written as zeros.  One block = one 32(o) x 32(i) tile over all taps, staged in
// shared memory so that reads of the source and writes of both layouts are coalesced.
constexpr int kSplitMaxTaps = 9;
struct SplitTable {
    const float* src[kMaxMulti];
    const float* scale[kMaxMulti];
    uint32_t* wf[kMaxMulti];
    uint32_t* wd[kMaxMulti];
    int O[kMaxMulti], I[kMaxMulti], taps[kMaxMulti], tile_begin[kMaxMulti + 1];
    int n, packed_src;
};

__device__ __forceinline__ uint32_t bf16x2_rn(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

__global__ void __launch_bounds__(256) pack_split_bf16_kernel(const __grid_constant__ SplitTable tb) {
    __shared__ float tile[kSplitMaxTaps][32][33];
    int k = 0;
    while (k + 1 < tb.n && (int)blockIdx.x >= tb.tile_begin[k + 1]) ++k;
    const int O = tb.O[k], I = tb.I[k], taps = tb.taps[k];
    const int tiles_i = (I + 31) / 32;
    const int lt = blockIdx.x - tb.tile_begin[k];
    const int o0 = (lt / tiles_i) * 32, i0 = (lt % tiles_i) * 32;
    const float* __restrict__ w = tb.src[k];
    const float* __restrict__ scale = tb.scale[k];
    // element (o, i, t): OIHW source = w[(o*I + i)*taps + t]; packed source = w[(t*O + o)*I + i]
    for (int idx = threadIdx.x; idx < 32 * 32 * taps; idx += 256) {
        int o, i, t;
        if (tb.packed_src) { i = idx & 31; o = (idx >> 5) & 31; t = idx >> 10; }
        else { t = idx % taps; const int r = idx / taps; i = r & 31; o = r >> 5; }
        float v = 0.f;
        if (o0 + o < O && i0 + i < I) {
            v = tb.packed_src ? w[((size_t)t * O + o0 + o) * I + i0 + i] : w[((size_t)(o0 + o) * I + i0 + i) * taps + t];
            if (scale) v *= scale[o0 + o];
        }
        tile[t][o][i] = v;
    }
    __syncthreads();
    const int kbf = (I + 31) / 32, kbd = (O + 31) / 32;
    uint32_t* __restrict__ wf = tb.wf[k];
    uint32_t* __restrict__ wd = tb.wd[k];
    for (int idx = threadIdx.x; idx < taps * 32 * 16; idx += 256) {
        const int wq = idx & 15, r = (idx >> 4) & 31, t = idx >> 9;
        if (o0 + r < O) {      // wf row (t, o0 + r), k-block i0 / 32: 32-bit words, 16 hi then 16 lo
            const float a = tile[t][r][2 * wq], b = tile[t][r][2 * wq + 1];
            const uint32_t h = bf16x2_rn(a, b);
            const uint32_t l = bf16x2_rn(a - __uint_as_float(h << 16), b - __uint_as_float(h & 0xFFFF0000u));
            uint32_t* row = wf + (((size_t)t * O + o0 + r) * kbf + (i0 >> 5)) * 32;
            row[wq] = h;
            row[16 + wq] = l;
        }
        if (wd && i0 + r < I) {   // wd row (t, i0 + r), k-block o0 / 32
            const float a = tile[t][2 * wq][r], b = tile[t][2 * wq + 1][r];
            const uint32_t h = bf16x2_rn(a, b);
            const uint32_t l = bf16x2_rn(a - __uint_as_float(h << 16), b - __uint_as_float(h & 0xFFFF0000u));
            uint32_t* row = wd + (((size_t)t * I + i0 + r) * kbd + (o0 >> 5)) * 32;
            row[wq] = h;
            row[16 + wq] = l;
        }
    }
}

// out[n] += sum_m x[m][n]; grid.x covers column groups of 32, grid.y row slabs.
__global__ void colsum_kernel(const float* __restrict__ x, float* __restrict__ out, long long M, int N, int rows_per_block) {
    __shared__ float part[8][33];
    const int col = blockIdx.x * 32 + (threadIdx.x & 31);
    const int ty = threadIdx.x >> 5;   // 8 row lanes
    const long long r0 = (long long)blockIdx.y * rows_per_block;
    const long long r1 = min(M, r0 + rows_per_block);
    float acc = 0.f;
    if (col < N)
        for (long long r = r0 + ty; r < r1; r += 8) acc += x[r * N + col];
    part[ty][threadIdx.x & 31] = acc;
    __syncthreads();
    if (ty == 0 && col < N) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += part[k][threadIdx.x];
        atomicAdd(out + col, s);
    }
}

}  // namespace

extern "C" {

int mdb_get_precision(void);

int mdb_pack_conv_weight_f32(const float* w_oihw, const float* scale, float* w_packed, int O, int I, int taps,
                             void* stream) {
    if (!w_oihw || !w_packed || O <= 0 || I <= 0 || taps <= 0) return MDB_EINVAL;
    const long long n = (long long)O * I * taps;
    const int grid = grid_cap(n, 256, num_sms() * 16);
    pack_weight_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(w_oihw, scale, w_packed, O, I, taps,
                                                                             mdb_get_precision() == 0);
    return (int)cudaGetLastError();
}

int mdb_unpack_conv_wgrad_f32(const float* dw_packed, float* dw_oihw, int O, int I, int taps, int accumulate,
                              void* stream) {
    if (!dw_packed || !dw_oihw || O <= 0 || I <= 0 || taps <= 0) return MDB_EINVAL;
    const long long n = (long long)O * I * taps;
    const int grid = grid_cap(n, 256, num_sms() * 16);
    unpack_wgrad_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(dw_packed, dw_oihw, O, I, taps, accumulate);
    return (int)cudaGetLastError();
}

// n tensors per call (any n: the call is cut into launches of <= 64 tensors); array arguments are HOST arrays.
int mdb_pack_conv_weights_multi_f32(int n, const float* const* w_oihw, const float* const* scale, float* const* w_packed,
                                    const int* O, const int* I, const int* taps, void* stream) {
    if (n < 0 || (n > 0 && (!w_oihw || !w_packed || !O || !I || !taps))) return MDB_EINVAL;
    for (int base = 0; base < n; base += kMaxMulti) {
        MultiTable tb;
        const int m = n - base < kMaxMulti ? n - base : kMaxMulti;
        for (int k = 0; k < m; ++k) {
            const int j = base + k;
            if (!w_oihw[j] || !w_packed[j] || O[j] <= 0 || I[j] <= 0 || taps[j] <= 0) return MDB_EINVAL;
            tb.src[k] = w_oihw[j]; tb.scale[k] = scale ? scale[j] : nullptr; tb.dst[k] = w_packed[j];
            tb.O[k] = O[j]; tb.I[k] = I[j]; tb.taps[k] = taps[j];
        }
        pack_weight_multi_kernel<<<dim3(64, m), 256, 0, static_cast<cudaStream_t>(stream)>>>(tb, mdb_get_precision() == 0);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}


// Multi-tensor split-pack for precision mode 2 (see pack_split_bf16_kernel); array arguments are HOST arrays.  wd may be NULL
// (or hold NULL entries) when no data gradient will be taken.  src_packed: 0 = OIHW sources, 1 = [tap][O][I] sources.
int mdb_pack_gemm_weights_bf16x3(int n, const float* const* w, const float* const* scale, void* const* wf, void* const* wd,
                                 const int* O, const int* I, const int* taps, int src_packed, void* stream) {
    if (n < 0 || (n > 0 && (!w || !wf || !O || !I || !taps))) return MDB_EINVAL;
    for (int base = 0; base < n; base += kMaxMulti) {
        SplitTable tb;
        const int m = n - base < kMaxMulti ? n - base : kMaxMulti;
        int tiles = 0;
        for (int k = 0; k < m; ++k) {
            const int j = base + k;
            if (!w[j] || !wf[j] || O[j] <= 0 || I[j] <= 0 || taps[j] <= 0 || taps[j] > kSplitMaxTaps) return MDB_EINVAL;
            tb.src[k] = w[j]; tb.scale[k] = scale ? scale[j] : nullptr;
            tb.wf[k] = static_cast<uint32_t*>(wf[j]); tb.wd[k] = wd ? static_cast<uint32_t*>(wd[j]) : nullptr;
            tb.O[k] = O[j]; tb.I[k] = I[j]; tb.taps[k] = taps[j];
            tb.tile_begin[k] = tiles;
            tiles += ((O[j] + 31) / 32) * ((I[j] + 31) / 32);
        }
        tb.tile_begin[m] = tiles;
        tb.n = m; tb.packed_src = src_packed ? 1 : 0;
        pack_split_bf16_kernel<<<tiles, 256, 0, static_cast<cudaStream_t>(stream)>>>(tb);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

int mdb_unpack_conv_wgrads_multi_f32(int n, const float* const* dw_packed, float* const* dw_oihw, const int* O, const int* I,
                                     const int* taps, void* stream) {
    if (n < 0 || (n > 0 && (!dw_packed || !dw_oihw || !O || !I || !taps))) return MDB_EINVAL;
    for (int base = 0; base < n; base += kMaxMulti) {
        MultiTable tb;
        const int m = n - base < kMaxMulti ? n - base : kMaxMulti;
        for (int k = 0; k < m; ++k) {
            const int j = base + k;
            if (!dw_packed[j] || !dw_oihw[j] || O[j] <= 0 || I[j] <= 0 || taps[j] <= 0) return MDB_EINVAL;
            tb.src[k] = dw_packed[j]; tb.scale[k] = nullptr; tb.dst[k] = dw_oihw[j];
            tb.O[k] = O[j]; tb.I[k] = I[j]; tb.taps[k] = taps[j];
        }
        unpack_wgrad_multi_kernel<<<dim3(64, m), 256, 0, static_cast<cudaStream_t>(stream)>>>(tb);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

int mdb_colsum_f32(const float* x, float* out, long long M, int N, int accumulate, void* stream_) {
    if (!x || !out || M < 0 || N <= 0) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (!accumulate) {
        cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * N, stream);
        if (e != cudaSuccess) return (int)e;
    }
    if (M == 0) return 0;
    const int gx = (N + 31) / 32;
    int gy = (int)((M + 511) / 512);
    const int cap = (num_sms() * 8 + gx - 1) / gx;
    if (gy > cap) gy = cap;
    if (gy < 1 || mdb_get_deterministic()) gy = 1;      // reproducible mode: one accumulation per column
    const int rows = (int)((M + gy - 1) / gy);
    colsum_kernel<<<dim3(gx, gy), 256, 0, stream>>>(x, out, M, N, rows);
    return (int)cudaGetLastError();
}

}  // extern "C"

// =================================================================================================
// More HBM-bound helpers: ReLU backward mask, dropout (forward == backward kernel), TF32 rounding,
// and the frozen ResNet stem (conv 7x7/2 + FrozenBN + ReLU, max-pool 3x3/2) -- backbone.py:71-73 keeps
// conv1/layer1 frozen, so the stem only ever runs forward.
// =================================================================================================
#include "rng.cuh"

namespace {

__global__ void relu_bwd_kernel(const float4* __restrict__ dy, const float4* __restrict__ y, float4* __restrict__ out,
                                long long n4, float scale) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 d = dy[i], v = y[i];
        out[i] = make_float4(v.x > 0.f ? d.x * scale : 0.f, v.y > 0.f ? d.y * scale : 0.f, v.z > 0.f ? d.z * scale : 0.f,
                             v.w > 0.f ? d.w * scale : 0.f);
    }
}

__global__ void dropout_kernel(const float4* __restrict__ x, float4* __restrict__ out, long long n4, float p,
                               const unsigned long long* __restrict__ seed_ptr, unsigned long long site) {
    const unsigned long long seed = *seed_ptr + site * 0x9E3779B97F4A7C15ull;
    const float inv = 1.f / (1.f - p);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float u[4];
        mdb::rng_uniform4(seed, (unsigned long long)i, u);
        const float4 v = x[i];
        out[i] = make_float4(u[0] >= p ? v.x * inv : 0.f, u[1] >= p ? v.y * inv : 0.f, u[2] >= p ? v.z * inv : 0.f,
                             u[3] >= p ? v.w * inv : 0.f);
    }
}

__device__ __forceinline__ float round_tf32(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}

__global__ void round_tf32_kernel(const float* __restrict__ x, float* __restrict__ out, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = round_tf32(x[i]);
}

// ---- stem: y[b][oy][ox][64] = relu(scale[c] * conv7x7s2(x NCHW [b][3][H][W]) + bias[c]) ----------------
// CTA = 8 x 32 output pixels, 256 threads.  A thread owns TWO vertically adjacent pixels x 32 of the 64 channels
// (warp w: rows 2*(w>>1), +1; channel half w&1): a tap's 8 weight float4 (warp-broadcast LDS.128) feed 64 FMAs, so the
// loop is FMA-bound instead of LDS-bound (the one-pixel-per-thread version needed 16 weight loads per 64 FMAs).
constexpr int ST_TH = 8, ST_TW = 32, ST_C = 64, ST_K = 7;
constexpr int ST_IH = ST_TH * 2 + 5, ST_IW = ST_TW * 2 + 5;   // 21 x 69 input patch per channel

__global__ void __launch_bounds__(256)
stem_conv_kernel(const float* __restrict__ x, const float* __restrict__ w /*[64][3][7][7]*/, const float* __restrict__ scale,
                 const float* __restrict__ bias, float* __restrict__ y, int H, int W, int Ho, int Wo, int round_out) {
    extern __shared__ float sm[];
    float* s_w = sm;                          // [147][64]  (tap-major so a tap's 64 weights are contiguous)
    float* s_in = sm + 147 * ST_C;            // [3][21][69]
    const int b = blockIdx.z;
    const int oy0 = blockIdx.y * ST_TH, ox0 = blockIdx.x * ST_TW;
    for (int i = threadIdx.x; i < 147 * ST_C; i += 256) {
        const int c = i % ST_C, t = i / ST_C;
        s_w[i] = w[c * 147 + t];
    }
    const int iy0 = oy0 * 2 - 3, ix0 = ox0 * 2 - 3;
    for (int i = threadIdx.x; i < 3 * ST_IH * ST_IW; i += 256) {
        const int xx = i % ST_IW, r = i / ST_IW;
        const int yy = r % ST_IH, ch = r / ST_IH;
        const int gy = iy0 + yy, gx = ix0 + xx;
        s_in[i] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? x[(((size_t)b * 3 + ch) * H + gy) * W + gx] : 0.f;
    }
    __syncthreads();
    const int wrp = threadIdx.x >> 5, lx = threadIdx.x & 31;
    const int half = wrp & 1, ly = (wrp >> 1) * 2;            // pixels (ly, lx) and (ly + 1, lx)
    float acc0[ST_C / 2], acc1[ST_C / 2];
#pragma unroll
    for (int c = 0; c < ST_C / 2; ++c) acc0[c] = acc1[c] = 0.f;
    for (int ch = 0; ch < 3; ++ch)
        for (int ky = 0; ky < ST_K; ++ky) {
            const float* row0 = s_in + (ch * ST_IH + ly * 2 + ky) * ST_IW + lx * 2;
            const float* row1 = row0 + 2 * ST_IW;
#pragma unroll
            for (int kx = 0; kx < ST_K; ++kx) {
                const float v0 = row0[kx], v1 = row1[kx];
                const float4* wp = reinterpret_cast<const float4*>(s_w + ((ch * ST_K + ky) * ST_K + kx) * ST_C + half * (ST_C / 2));
#pragma unroll
                for (int c4 = 0; c4 < ST_C / 8; ++c4) {
                    const float4 ww = wp[c4];
                    acc0[c4 * 4] = fmaf(v0, ww.x, acc0[c4 * 4]);         acc1[c4 * 4] = fmaf(v1, ww.x, acc1[c4 * 4]);
                    acc0[c4 * 4 + 1] = fmaf(v0, ww.y, acc0[c4 * 4 + 1]); acc1[c4 * 4 + 1] = fmaf(v1, ww.y, acc1[c4 * 4 + 1]);
                    acc0[c4 * 4 + 2] = fmaf(v0, ww.z, acc0[c4 * 4 + 2]); acc1[c4 * 4 + 2] = fmaf(v1, ww.z, acc1[c4 * 4 + 2]);
                    acc0[c4 * 4 + 3] = fmaf(v0, ww.w, acc0[c4 * 4 + 3]); acc1[c4 * 4 + 3] = fmaf(v1, ww.w, acc1[c4 * 4 + 3]);
                }
            }
        }
    const int ox = ox0 + lx;
    if (ox < Wo) {
#pragma unroll
        for (int pxl = 0; pxl < 2; ++pxl) {
            const int oy = oy0 + ly + pxl;
            if (oy >= Ho) break;
            float* yp = y + (((size_t)b * Ho + oy) * Wo + ox) * ST_C + half * (ST_C / 2);
#pragma unroll
            for (int c4 = 0; c4 < ST_C / 8; ++c4) {
                const float4 s = *reinterpret_cast<const float4*>(scale + half * (ST_C / 2) + c4 * 4);
                const float4 bb = *reinterpret_cast<const float4*>(bias + half * (ST_C / 2) + c4 * 4);
                const float* a = pxl ? acc1 : acc0;
                float4 o;
                o.x = fmaxf(fmaf(a[c4 * 4], s.x, bb.x), 0.f);
                o.y = fmaxf(fmaf(a[c4 * 4 + 1], s.y, bb.y), 0.f);
                o.z = fmaxf(fmaf(a[c4 * 4 + 2], s.z, bb.z), 0.f);
                o.w = fmaxf(fmaf(a[c4 * 4 + 3], s.w, bb.w), 0.f);
                if (round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); o.z = round_tf32(o.z); o.w = round_tf32(o.w); }
                *reinterpret_cast<float4*>(yp + c4 * 4) = o;
            }
        }
    }
}

// NHWC max-pool 3x3 stride 2 pad 1
__global__ void maxpool3x3s2_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C, int Ho,
                                    int Wo) {
    const long long n4 = (long long)B * Ho * Wo * C / 4;
    const int c4n = C / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % c4n);
        long long r = i / c4n;
        const int ox = (int)(r % Wo); r /= Wo;
        const int oy = (int)(r % Ho);
        const int b = (int)(r / Ho);
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = oy * 2 - 1 + ky;
            if (iy < 0 || iy >= H) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ox * 2 - 1 + kx;
                if (ix < 0 || ix >= W) continue;
                const float4 v = *reinterpret_cast<const float4*>(x + (((size_t)b * H + iy) * W + ix) * C + c4 * 4);
                m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
            }
        }
        *reinterpret_cast<float4*>(y + i * 4) = m;
    }
}

}  // namespace

extern "C" {

// out = dy * (y > 0) * scale          (n % 4 == 0, 16-byte aligned)
int mdb_relu_backward_f32(const float* dy, const float* y, float* out, long long n, float scale, void* stream) {
    if (!dy || !y || !out || n < 0 || n % 4) return MDB_EINVAL;
    if (n == 0) return 0;
    relu_bwd_kernel<<<grid_cap(n / 4, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const float4*>(dy), reinterpret_cast<const float4*>(y), reinterpret_cast<float4*>(out), n / 4, scale);
    return (int)cudaGetLastError();
}

// out = x * keep(seed, site, index) / (1 - p): the same call regenerates the mask for the backward pass.
int mdb_dropout_f32(const float* x, float* out, long long n, float p, const unsigned long long* seed,
                    unsigned long long site, void* stream) {
    if (!x || !out || !seed || n < 0 || n % 4 || p < 0.f || p >= 1.f) return MDB_EINVAL;
    if (n == 0) return 0;
    dropout_kernel<<<grid_cap(n / 4, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(out), n / 4, p, seed, site);
    return (int)cudaGetLastError();
}

// out = round-to-nearest TF32 of x (operands of the tensor-core kernels; the tensor core truncates otherwise)
int mdb_round_tf32_f32(const float* x, float* out, long long n, void* stream) {
    if (!x || !out || n < 0) return MDB_EINVAL;
    if (n == 0) return 0;
    round_tf32_kernel<<<grid_cap(n, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, out, n);
    return (int)cudaGetLastError();
}

// ResNet stem, forward only: x NCHW [B][3][H][W] -> y NHWC [B][Ho][Wo][64], Ho = (H+6-7)/2+1.
int mdb_stem_conv7x7_bn_relu_f32(const float* x, const float* w, const float* scale, const float* bias, float* y, int B, int H,
                                 int W, void* stream_) {
    if (!x || !w || !scale || !bias || !y || B <= 0 || H <= 0 || W <= 0) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
    const int smem = (147 * ST_C + 3 * ST_IH * ST_IW) * (int)sizeof(float);
    const cudaError_t e = set_max_dynamic_smem(stem_conv_kernel, smem);
    if (e != cudaSuccess) return (int)e;
    dim3 grid((Wo + ST_TW - 1) / ST_TW, (Ho + ST_TH - 1) / ST_TH, B);
    // single-pass TF32 mode: the consumer is a tensor-core operand that expects round-to-nearest TF32 values
    stem_conv_kernel<<<grid, 256, smem, stream>>>(x, w, scale, bias, y, H, W, Ho, Wo, mdb_get_precision() == 0 ? 1 : 0);
    return (int)cudaGetLastError();
}

int mdb_maxpool3x3s2_nhwc_f32(const float* x, float* y, int B, int H, int W, int C, void* stream) {
    if (!x || !y || B <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 4) return MDB_EINVAL;
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long n4 = (long long)B * Ho * Wo * C / 4;
    maxpool3x3s2_kernel<<<grid_cap(n4, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, B, H, W, C, Ho, Wo);
    return (int)cudaGetLastError();
}

}  // extern "C"

// =================================================================================================
// Depth-map lookup of the detection head (monodetr.py:248-253): F.grid_sample(weighted_depth[:, None], centres,
// bilinear, zeros padding, align_corners=True) for N query centres per image, forward and backward wrt the map
// (the centres are detached in the reference).  One thread per (b, n).
// =================================================================================================
namespace {

__global__ void depth_sample_fwd_kernel(const float* __restrict__ depth, const float* __restrict__ xy, float* __restrict__ out,
                                        int B, int H, int W, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * N) return;
    const int b = i / N;
    const float x = (xy[2 * i] + 1.f) * 0.5f * (float)(W - 1), y = (xy[2 * i + 1] + 1.f) * 0.5f * (float)(H - 1);
    const float xf = floorf(x), yf = floorf(y);
    const int x0 = (int)xf, y0 = (int)yf;
    const float lx = x - xf, ly = y - yf;
    const float* d = depth + (size_t)b * H * W;
    auto tap = [&](int yy, int xx) { return (xx >= 0 && xx <= W - 1 && yy >= 0 && yy <= H - 1) ? d[yy * W + xx] : 0.f; };
    out[i] = tap(y0, x0) * (1.f - ly) * (1.f - lx) + tap(y0, x0 + 1) * (1.f - ly) * lx + tap(y0 + 1, x0) * ly * (1.f - lx) +
             tap(y0 + 1, x0 + 1) * ly * lx;
}

__global__ void depth_sample_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ xy, float* __restrict__ ddepth,
                                        int B, int H, int W, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * N) return;
    const int b = i / N;
    const float x = (xy[2 * i] + 1.f) * 0.5f * (float)(W - 1), y = (xy[2 * i + 1] + 1.f) * 0.5f * (float)(H - 1);
    const float xf = floorf(x), yf = floorf(y);
    const int x0 = (int)xf, y0 = (int)yf;
    const float lx = x - xf, ly = y - yf, g = dout[i];
    float* d = ddepth + (size_t)b * H * W;
    auto put = [&](int yy, int xx, float w) { if (xx >= 0 && xx <= W - 1 && yy >= 0 && yy <= H - 1) atomicAdd(d + yy * W + xx, w * g); };
    put(y0, x0, (1.f - ly) * (1.f - lx)); put(y0, x0 + 1, (1.f - ly) * lx); put(y0 + 1, x0, ly * (1.f - lx)); put(y0 + 1, x0 + 1, ly * lx);
}

// Reproducible mode: the map gradient in gather form -- one thread per map pixel walks the N centres of its image in order.
__global__ void depth_sample_bwd_gather_kernel(const float* __restrict__ dout, const float* __restrict__ xy, float* __restrict__ ddepth,
                                               int B, int H, int W, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * H * W) return;
    const int b = i / (H * W), py = (i / W) % H, px = i % W;
    float acc = 0.f;
    for (int q = b * N; q < (b + 1) * N; ++q) {
        const float x = (xy[2 * q] + 1.f) * 0.5f * (float)(W - 1), y = (xy[2 * q + 1] + 1.f) * 0.5f * (float)(H - 1);
        const float xf = floorf(x), yf = floorf(y);
        const int x0 = (int)xf, y0 = (int)yf;
        if ((y0 != py && y0 + 1 != py) || (x0 != px && x0 + 1 != px)) continue;
        const float lx = x - xf, ly = y - yf, g = dout[q];
        if (y0 == py && x0 == px) acc += ((1.f - ly) * (1.f - lx)) * g;
        if (y0 == py && x0 + 1 == px) acc += ((1.f - ly) * lx) * g;
        if (y0 + 1 == py && x0 == px) acc += (ly * (1.f - lx)) * g;
        if (y0 + 1 == py && x0 + 1 == px) acc += (ly * lx) * g;
    }
    ddepth[i] = acc;
}

// ---- bilinear resize of NHWC maps, F.interpolate(mode="bilinear", align_corners=False) without a scale factor ------------
// torch's source-index rule: src = (in / out) * (dst + 0.5) - 0.5, clamped below at 0; i0 = floor(src), i1 = i0 + (i0 < in - 1),
// lambda1 = src - i0, lambda0 = 1 - lambda1.
__device__ __forceinline__ void up_src(int o, float scale, int in, int& i0, int& i1, float& l0, float& l1) {
    float s = scale * ((float)o + 0.5f) - 0.5f;
    if (s < 0.f) s = 0.f;
    i0 = (int)s;
    i1 = i0 + (i0 < in - 1 ? 1 : 0);
    l1 = s - (float)i0;
    l0 = 1.f - l1;
}

// one thread per (b, oy, ox, channel quad)
__global__ void upsample_bilinear_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int Hi, int Wi, int Ho, int Wo,
                                             int C, float sh, float sw) {
    const int c4n = C / 4;
    const long long n4 = (long long)B * Ho * Wo * c4n;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % c4n) * 4;
        long long r = i / c4n;
        const int ox = (int)(r % Wo); r /= Wo;
        const int oy = (int)(r % Ho);
        const int b = (int)(r / Ho);
        int h0, h1, w0, w1; float hl0, hl1, wl0, wl1;
        up_src(oy, sh, Hi, h0, h1, hl0, hl1);
        up_src(ox, sw, Wi, w0, w1, wl0, wl1);
        const float* xb = x + (size_t)b * Hi * Wi * C + c;
        const float4 a = *reinterpret_cast<const float4*>(xb + ((size_t)h0 * Wi + w0) * C);
        const float4 bb = *reinterpret_cast<const float4*>(xb + ((size_t)h0 * Wi + w1) * C);
        const float4 cc = *reinterpret_cast<const float4*>(xb + ((size_t)h1 * Wi + w0) * C);
        const float4 d = *reinterpret_cast<const float4*>(xb + ((size_t)h1 * Wi + w1) * C);
        float4 o;
        o.x = hl0 * (wl0 * a.x + wl1 * bb.x) + hl1 * (wl0 * cc.x + wl1 * d.x);
        o.y = hl0 * (wl0 * a.y + wl1 * bb.y) + hl1 * (wl0 * cc.y + wl1 * d.y);
        o.z = hl0 * (wl0 * a.z + wl1 * bb.z) + hl1 * (wl0 * cc.z + wl1 * d.z);
        o.w = hl0 * (wl0 * a.w + wl1 * bb.w) + hl1 * (wl0 * cc.w + wl1 * d.w);
        *reinterpret_cast<float4*>(y + i * 4) = o;
    }
}

// Gather form of the backward (deterministic by construction): one thread per (b, h, w, channel quad) of the input walks the output
// rows / columns whose source window can contain it, in increasing order, and adds lambda_h * lambda_w * dy for each corner that is it.
__global__ void upsample_bilinear_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int B, int Hi, int Wi, int Ho, int Wo,
                                             int C, float sh, float sw) {
    const int c4n = C / 4;
    const long long n4 = (long long)B * Hi * Wi * c4n;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % c4n) * 4;
        long long r = i / c4n;
        const int w = (int)(r % Wi); r /= Wi;
        const int h = (int)(r % Hi);
        const int b = (int)(r / Hi);
        // outputs with src in [h - 1, h + 1): (dst + 0.5) * scale in [h - 0.5, h + 1.5), widened by 2 against rounding; the rows whose
        // src is clamped to 0 start at dst 0
        const int ylo = h <= 1 ? 0 : max(0, (int)floorf((h - 0.5f) / sh - 0.5f) - 2);
        const int yhi = min(Ho - 1, (int)ceilf((h + 1.5f) / sh - 0.5f) + 2);
        const int xlo = w <= 1 ? 0 : max(0, (int)floorf((w - 0.5f) / sw - 0.5f) - 2);
        const int xhi = min(Wo - 1, (int)ceilf((w + 1.5f) / sw - 0.5f) + 2);
        const float* gb = dy + (size_t)b * Ho * Wo * C + c;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int oy = ylo; oy <= yhi; ++oy) {
            int h0, h1; float hl0, hl1;
            up_src(oy, sh, Hi, h0, h1, hl0, hl1);
            if (h0 != h && h1 != h) continue;
            for (int ox = xlo; ox <= xhi; ++ox) {
                int w0, w1; float wl0, wl1;
                up_src(ox, sw, Wi, w0, w1, wl0, wl1);
                if (w0 != w && w1 != w) continue;
                const float4 g = *reinterpret_cast<const float4*>(gb + ((size_t)oy * Wo + ox) * C);
                float f[4] = {0.f, 0.f, 0.f, 0.f};
                int k = 0;
                if (h0 == h && w0 == w) f[k++] = hl0 * wl0;
                if (h0 == h && w1 == w) f[k++] = hl0 * wl1;
                if (h1 == h && w0 == w) f[k++] = hl1 * wl0;
                if (h1 == h && w1 == w) f[k++] = hl1 * wl1;
                for (int j = 0; j < k; ++j) {
                    acc.x += f[j] * g.x; acc.y += f[j] * g.y; acc.z += f[j] * g.z; acc.w += f[j] * g.w;
                }
            }
        }
        *reinterpret_cast<float4*>(dx + i * 4) = acc;
    }
}

}  // namespace

extern "C" {

int mdb_depth_sample_forward_f32(const float* depth, const float* xy, float* out, int B, int H, int W, int N, void* stream) {
    if (!depth || !xy || !out || B <= 0 || H <= 0 || W <= 0 || N < 0) return MDB_EINVAL;
    if (N == 0) return 0;
    depth_sample_fwd_kernel<<<(B * N + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(depth, xy, out, B, H, W, N);
    return (int)cudaGetLastError();
}

// ddepth (B,H,W) is zero-filled by the call, then accumulated.
int mdb_depth_sample_backward_f32(const float* dout, const float* xy, float* ddepth, int B, int H, int W, int N, void* stream_) {
    if (!dout || !xy || !ddepth || B <= 0 || H <= 0 || W <= 0 || N < 0) return MDB_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (mdb_get_deterministic()) {                   // reproducible mode: gather, every pixel written once
        depth_sample_bwd_gather_kernel<<<(B * H * W + 127) / 128, 128, 0, stream>>>(dout, xy, ddepth, B, H, W, N);
        return (int)cudaGetLastError();
    }
    cudaError_t e = cudaMemsetAsync(ddepth, 0, sizeof(float) * (size_t)B * H * W, stream);
    if (e != cudaSuccess) return (int)e;
    if (N == 0) return 0;
    depth_sample_bwd_kernel<<<(B * N + 127) / 128, 128, 0, stream>>>(dout, xy, ddepth, B, H, W, N);
    return (int)cudaGetLastError();
}

// x (B, Hi, Wi, C) -> y (B, Ho, Wo, C), NHWC contiguous, C % 4 == 0, 16-byte aligned.
int mdb_upsample_bilinear_nhwc_forward_f32(const float* x, float* y, int B, int Hi, int Wi, int Ho, int Wo, int C, void* stream) {
    if (!x || !y || B <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || C <= 0 || C % 4) return MDB_EINVAL;
    const long long n4 = (long long)B * Ho * Wo * C / 4;
    upsample_bilinear_fwd_kernel<<<grid_cap(n4, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, y, B, Hi, Wi, Ho, Wo, C, (float)Hi / (float)Ho, (float)Wi / (float)Wo);
    return (int)cudaGetLastError();
}
// dx (B, Hi, Wi, C) = gradient wrt x of the forward above for dy (B, Ho, Wo, C); fully written, no atomics.
int mdb_upsample_bilinear_nhwc_backward_f32(const float* dy, float* dx, int B, int Hi, int Wi, int Ho, int Wo, int C, void* stream) {
    if (!dy || !dx || B <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || C <= 0 || C % 4) return MDB_EINVAL;
    const long long n4 = (long long)B * Hi * Wi * C / 4;
    upsample_bilinear_bwd_kernel<<<grid_cap(n4, 256, num_sms() * 16), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        dy, dx, B, Hi, Wi, Ho, Wo, C, (float)Hi / (float)Ho, (float)Wi / (float)Wo);
    return (int)cudaGetLastError();
}

}  // extern "C"
