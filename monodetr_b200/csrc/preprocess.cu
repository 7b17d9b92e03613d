// preprocess.cu -- input pipeline on the device (SURVEY.md 8 f4): the step before the hot path.  The reference's dataset
// (lib/datasets/kitti/kitti_dataset.py:121-163) warps every image on a data-loader worker with PIL
// (`img.transform(resolution, Image.AFFINE, trans_inv, resample=Image.BILINEAR)`), converts to float, normalises and transposes
// to CHW with numpy.  Here the decoded 8-bit images are uploaded as they are (ragged sizes, 3 bytes per pixel) and ONE kernel
// produces the normalised NCHW fp32 batch the backbone reads: optional left-right flip (:140-142), inverse affine map of every
// output pixel centre, PIL's bilinear filter (clamped neighbours, zero fill outside, result truncated to 8 bits), /255,
// (x - mean) / std (:159-161).
// Arithmetic: coordinates and interpolation in fp64 in the order and with the roundings of PIL's C code (Geometry.c, built
// without FMA): xin = (a0*xc + a1*yc) + a2, then - 0.5, and v = a + (b - a) * d, every product rounded before its sum by an
// explicit _rn intrinsic, so that the floor of each coordinate and the 8-bit truncation are bit-identical to Pillow's for any
// affine map, sheared or not (tests/test_preprocess_edges_gpu.py); the float conversion in fp32 exactly as numpy's.
// HBM-bound: 12 bytes written per output pixel.
// Before it, when the dataset's `aug_pd` is on, a second kernel applies the reference's photometric distortion (:136-138,
// pd.py:376-397) to every source image with its own host-drawn parameters and writes the 8-bit result to a caller buffer that the
// warp then reads: pointwise, 3 bytes read and 3 written per source pixel.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

// Pillow's BILINEAR(v, a, b, d): a + (b - a) * d with the product rounded before the sum (nvcc would otherwise fuse it to a DFMA)
__device__ __forceinline__ double lerp_rn(double a, double b, double d) { return __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), d)); }

__global__ void __launch_bounds__(256) warp_affine_normalize_kernel(const unsigned char* const* __restrict__ src, const int* __restrict__ src_wh,
                                                                    const long long* __restrict__ src_pitch, const double* __restrict__ trans_inv,
                                                                    const unsigned char* __restrict__ flip, float* __restrict__ out, int Wo,
                                                                    int Ho, float3 mean, float3 stdv) {
    const int b = blockIdx.z;
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= Wo) return;
    const int W = src_wh[2 * b], H = src_wh[2 * b + 1];
    const double* a = trans_inv + 6 * b;
    const double xc = x + 0.5, yc = y + 0.5;
    double xin = __dadd_rn(__dadd_rn(__dmul_rn(a[0], xc), __dmul_rn(a[1], yc)), a[2]);
    double yin = __dadd_rn(__dadd_rn(__dmul_rn(a[3], xc), __dmul_rn(a[4], yc)), a[5]);
    float v[3] = {0.f, 0.f, 0.f};
    if (!(xin < 0.0 || xin >= (double)W || yin < 0.0 || yin >= (double)H)) {
        xin = __dsub_rn(xin, 0.5); yin = __dsub_rn(yin, 0.5);
        const int xf = (int)floor(xin), yf = (int)floor(yin);
        const double dx = __dsub_rn(xin, xf), dy = __dsub_rn(yin, yf);
        int x0 = min(max(xf, 0), W - 1), x1 = min(max(xf + 1, 0), W - 1);
        const int y0 = min(max(yf, 0), H - 1);
        const bool has_y1 = yf + 1 >= 0 && yf + 1 < H;
        if (flip && flip[b]) { x0 = W - 1 - x0; x1 = W - 1 - x1; }        // sampling the mirrored image
        const unsigned char* r0 = src[b] + (long long)y0 * src_pitch[b];
        const unsigned char* r1 = src[b] + (long long)(yf + 1) * src_pitch[b];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double p00 = r0[x0 * 3 + c], p01 = r0[x1 * 3 + c];
            const double v1 = lerp_rn(p00, p01, dx);
            double v2 = v1;
            if (has_y1) {
                const double p10 = r1[x0 * 3 + c], p11 = r1[x1 * 3 + c];
                v2 = lerp_rn(p10, p11, dx);
            }
            v[c] = (float)(unsigned char)lerp_rn(v1, v2, dy);
        }
    }
    const size_t plane = (size_t)Ho * Wo;
    float* o = out + (size_t)b * 3 * plane + (size_t)y * Wo + x;
    o[0] = __fdiv_rn(__fsub_rn(__fdiv_rn(v[0], 255.f), mean.x), stdv.x);
    o[plane] = __fdiv_rn(__fsub_rn(__fdiv_rn(v[1], 255.f), mean.y), stdv.y);
    o[2 * plane] = __fdiv_rn(__fsub_rn(__fdiv_rn(v[2], 255.f), mean.z), stdv.z);
}

// ---- photometric distortion (lib/datasets/kitti/pd.py:376-397 as called at kitti_dataset.py:136-138) ----------------------------
// cv2.cvtColor BGR<->HSV on float32 as the reference's cv2 runs it (AVX2 + FMA3): a vector loop over 8 pixels and a scalar loop
// over the last W % 8 pixels of each row, which round the hue differently.  Every operation is an explicit _rn intrinsic so that
// nvcc contracts nothing the reference does not.
constexpr int kHsvSimdWidth = 8;

__device__ __forceinline__ void bgr_to_hsv(float b, float g, float r, bool scalar_tail, float& h, float& s, float& v) {
    v = fmaxf(fmaxf(r, g), b);
    const float vmin = fminf(fminf(r, g), b);
    const float diff = __fsub_rn(v, vmin);
    s = __fdiv_rn(diff, __fadd_rn(fabsf(v), FLT_EPSILON));
    const float dd = __fadd_rn(diff, FLT_EPSILON);
    float num, off;
    if (r == v) { num = __fsub_rn(g, b); off = 0.f; }
    else if (g == v) { num = __fsub_rn(b, r); off = 120.f; }
    else { num = __fsub_rn(r, g); off = 240.f; }
    if (!scalar_tail) {                                   // vector loop: the +360 of a negative V == R hue is inside the FMA
        if (r == v && num < 0.f) off = 360.f;
        h = __fmaf_rn(num, __fdiv_rn(60.f, dd), off);
    } else {                                              // scalar loop: 60 / x in double, +360 afterwards
        h = __fmaf_rn(num, __double2float_rn(__ddiv_rn(60.0, (double)dd)), off);
        if (h < 0.f) h = __fadd_rn(h, 360.f);
    }
}

__device__ __forceinline__ void hsv_to_bgr(float h, float s, float v, float& b, float& g, float& r) {
    const float hs = __fmul_rn(h, 6.f / 360.f);
    const float pre = truncf(hs);
    const float f = __fsub_rn(hs, pre);
    int sector = (int)pre - 6 * (int)truncf(__fmul_rn(pre, 1.f / 6.f));
    if (sector < 0) sector += 6;
    const float t0 = v;
    const float t1 = __fmul_rn(v, __fsub_rn(1.f, s));
    const float t2 = __fmul_rn(v, __fmaf_rn(-s, f, 1.f));
    const float t3 = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.f, f), 1.f));
    switch (sector) {                                     // cv2's sector table {1,3,0} {1,0,2} {3,0,1} {0,2,1} {0,1,3} {2,1,0}
        case 0: b = t1; g = t3; r = t0; break;
        case 1: b = t1; g = t0; r = t2; break;
        case 2: b = t3; g = t0; r = t1; break;
        case 3: b = t0; g = t2; r = t1; break;
        case 4: b = t0; g = t1; r = t3; break;
        default: b = t2; g = t1; r = t0; break;
    }
}

// numpy's float32 -> uint8 cast on x86: truncate toward zero, keep the low 8 bits (290.3 -> 34, -5.7 -> 251)
__device__ __forceinline__ unsigned char to_u8_wrap(float x) { return (unsigned char)__float2int_rz(x); }

// grid (blocks per image, B): block x strides over the rows of image blockIdx.y, the threads over the pixels of a row
__global__ void __launch_bounds__(256) photometric_distort_kernel(const unsigned char* const* __restrict__ src,
                                                                  const int* __restrict__ src_wh,
                                                                  const long long* __restrict__ src_pitch,
                                                                  const mdb_photometric_params* __restrict__ params,
                                                                  unsigned char* const* __restrict__ dst,
                                                                  const long long* __restrict__ dst_pitch) {
    const int b = blockIdx.y;
    const int W = src_wh[2 * b], H = src_wh[2 * b + 1];
    const mdb_photometric_params p = params[b];
    if (W <= 0 || H <= 0 || (unsigned)p.perm > 5u || (unsigned)p.contrast_last > 1u) return;
    const int tail0 = W - W % kHsvSimdWidth;
    for (int y = blockIdx.x; y < H; y += gridDim.x) {
        const unsigned char* s_row = src[b] + (long long)y * src_pitch[b];
        unsigned char* d_row = dst[b] + (long long)y * dst_pitch[b];
        for (int x = threadIdx.x; x < W; x += blockDim.x) {
            float c[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                c[k] = __fadd_rn((float)s_row[3 * x + k], p.brightness);
                if (!p.contrast_last) c[k] = __fmul_rn(c[k], p.contrast);
            }
            float h, s, v;
            bgr_to_hsv(c[0], c[1], c[2], x >= tail0, h, s, v);
            s = __fmul_rn(s, p.saturation);
            h = __fadd_rn(h, p.hue);
            if (h > 360.f) h = __fsub_rn(h, 360.f);
            if (h < 0.f) h = __fadd_rn(h, 360.f);
            hsv_to_bgr(h, s, v, c[0], c[1], c[2]);
            if (p.contrast_last) {
#pragma unroll
                for (int k = 0; k < 3; ++k) c[k] = __fmul_rn(c[k], p.contrast);
            }
            float o0 = c[0], o1 = c[1], o2 = c[2];       // pd.py:143-145 perms: out[k] = c[perm[k]]
            switch (p.perm) {
                case 1: o1 = c[2]; o2 = c[1]; break;
                case 2: o0 = c[1]; o1 = c[0]; break;
                case 3: o0 = c[1]; o1 = c[2]; o2 = c[0]; break;
                case 4: o0 = c[2]; o1 = c[0]; o2 = c[1]; break;
                case 5: o0 = c[2]; o2 = c[0]; break;
                default: break;
            }
            d_row[3 * x] = to_u8_wrap(o0);
            d_row[3 * x + 1] = to_u8_wrap(o1);
            d_row[3 * x + 2] = to_u8_wrap(o2);
        }
    }
}

}  // namespace

extern "C" int mdb_photometric_distort_u8(const unsigned char* const* src, const int* src_wh, const long long* src_pitch,
                                          const mdb_photometric_params* params, unsigned char* const* dst,
                                          const long long* dst_pitch, int B, void* stream) {
    if (!src || !src_wh || !src_pitch || !params || !dst || !dst_pitch) return MDB_EINVAL;
    if (B <= 0 || B > 65535) return MDB_EINVAL;
    const int per_image = mdb::num_sms() * 8 / B;
    dim3 grid(per_image < 1 ? 1 : per_image, B);
    photometric_distort_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, src_wh, src_pitch, params, dst, dst_pitch);
    return (int)cudaGetLastError();
}

extern "C" int mdb_warp_affine_normalize_u8(const unsigned char* const* src, const int* src_wh, const long long* src_pitch,
                                            const double* trans_inv, const unsigned char* flip, int B, int out_w, int out_h,
                                            const float* mean3, const float* std3, float* out, void* stream) {
    if (!src || !src_wh || !src_pitch || !trans_inv || !mean3 || !std3 || !out) return MDB_EINVAL;
    if (B <= 0 || out_w <= 0 || out_h <= 0 || out_h > 65535 || B > 65535) return MDB_EINVAL;
    dim3 grid((out_w + 255) / 256, out_h, B);
    warp_affine_normalize_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, src_wh, src_pitch, trans_inv, flip, out, out_w, out_h,
                                                                         make_float3(mean3[0], mean3[1], mean3[2]),
                                                                         make_float3(std3[0], std3[1], std3[2]));
    return (int)cudaGetLastError();
}
