// kitti_eval.cu -- the KITTI object-detection metric (AP of 2-d boxes, bird's-eye-view boxes, 3-d boxes and AOS, 11- and
// 40-point) on the device: the reference's lib/datasets/kitti/kitti_eval_python/{eval.py, rotate_iou.py}, which runs JIT-compiled CPU
// loops and one JIT-compiled CUDA kernel.  Inputs are packed on the host in CSR form (per-image offsets into flat gt / detection
// tables, include/monodetr_b200.h).  Six kernels in two entry points, no host synchronisation, no device allocation:
//   * overlaps    eval.py:162-230, rotate_iou.py:17-330   one CTA per image: the dt x gt block of the image, 3 metrics
//   * clean       eval.py:30-82 (85-159 by distance)      one CTA per (class, difficulty or bin): ignored flags, valid-gt count
//   * pass 1      eval.py:233-350 (compute_fp=False)      one warp per (configuration, image): the matched TP scores
//   * thresholds  eval.py:9-27                            one CTA per configuration: bitonic sort, then the 41-point ranks
//   * pass 2      eval.py:365-412 (compute_fp=True)       one warp per (configuration, image, threshold): tp / fp / fn / AOS
//   * reduce                                              one thread per (configuration, threshold): the result table
// Arithmetic follows the reference operation by operation: the 2-d overlap and the statistics in fp64, the rotated intersection in
// fp32, with explicit _rn intrinsics wherever nvcc could contract a multiply and an add into an FMA (the reference's loops are plain
// IEEE operations, so a contraction would flip `overlap > min_overlap` decisions).  Counts are integers (atomics are exact in any
// order); the AOS similarity is summed in gt order per image and then in image order, so the result does not depend on scheduling.
// Parity: tests/test_kitti_eval_gpu.py against oracle/kitti_eval.py and the golden vectors generated from the reference;
// tests/test_kitti_eval_edges_gpu.py bit for bit where overlaps sit exactly at, or one or two ulps around, the thresholds.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"

namespace {

constexpr int kMaxBoxes = MDB_KITTI_MAX_BOXES;   // per image; a detection's "assigned" flag is one bit of a per-lane 32-bit mask
constexpr int kThr = MDB_KITTI_NUM_THRESH;       // eval.py:552  N_SAMPLE_PTS
constexpr int kGtCols = MDB_KITTI_GT_COLS, kDtCols = MDB_KITTI_DT_COLS;
constexpr int kWarps = 8;                        // warps per CTA of the two statistics passes
constexpr double kNoDetection = -10000000.0;     // eval.py:259

// ---------------------------------------------------------------------------------------------------------------------------
// Rotated-box intersection in fp32, rotate_iou.py:17-260 (the pair (query, box) of devRotateIoUEval).  Boxes are [x, z, l, w, ry].
// The reference computes cos / sin in double and rounds them to fp32; sqrt is the correctly rounded fp32 one.
__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }

__device__ void box_corners(const float* rb, float* c) {                                  // rotate_iou.py:204-228
    const float ac = (float)cos((double)rb[4]), as = (float)sin((double)rb[4]);
    const float hx = -rb[2] / 2.f, hy = -rb[3] / 2.f;
    const float cx[4] = {hx, hx, -hx, -hx}, cy[4] = {hy, -hy, -hy, hy};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        c[2 * i] = fa(fa(fm(ac, cx[i]), fm(as, cy[i])), rb[0]);
        c[2 * i + 1] = fa(fa(fm(-as, cx[i]), fm(ac, cy[i])), rb[1]);
    }
}

__device__ bool point_in_quad(float px, float py, const float* c) {                         // rotate_iou.py:161-177
    const float ab0 = fs(c[2], c[0]), ab1 = fs(c[3], c[1]), ad0 = fs(c[6], c[0]), ad1 = fs(c[7], c[1]);
    const float ap0 = fs(px, c[0]), ap1 = fs(py, c[1]);
    const float abab = fa(fm(ab0, ab0), fm(ab1, ab1)), abap = fa(fm(ab0, ap0), fm(ab1, ap1));
    const float adad = fa(fm(ad0, ad0), fm(ad1, ad1)), adap = fa(fm(ad0, ap0), fm(ad1, ap1));
    return abab >= abap && abap >= 0.f && adad >= adap && adap >= 0.f;
}

__device__ bool segment_intersection(const float* p1, const float* p2, int i, int j, float* out) {   // rotate_iou.py:73-116
    const float A0 = p1[2 * i], A1 = p1[2 * i + 1], B0 = p1[2 * ((i + 1) & 3)], B1 = p1[2 * ((i + 1) & 3) + 1];
    const float C0 = p2[2 * j], C1 = p2[2 * j + 1], D0 = p2[2 * ((j + 1) & 3)], D1 = p2[2 * ((j + 1) & 3) + 1];
    const float BA0 = fs(B0, A0), BA1 = fs(B1, A1), DA0 = fs(D0, A0), CA0 = fs(C0, A0), DA1 = fs(D1, A1), CA1 = fs(C1, A1);
    const bool acd = fm(DA1, CA0) > fm(CA1, DA0);
    const bool bcd = fm(fs(D1, B1), fs(C0, B0)) > fm(fs(C1, B1), fs(D0, B0));
    if (acd == bcd) return false;
    const bool abc = fm(CA1, BA0) > fm(BA1, CA0);
    const bool abd = fm(DA1, BA0) > fm(BA1, DA0);
    if (abc == abd) return false;
    const float DC0 = fs(D0, C0), DC1 = fs(D1, C1);
    const float ABBA = fs(fm(A0, B1), fm(B0, A1)), CDDC = fs(fm(C0, D1), fm(D0, C1));
    const float DH = fs(fm(BA1, DC0), fm(BA0, DC1));
    const float Dx = fs(fm(ABBA, DC0), fm(BA0, CDDC)), Dy = fs(fm(ABBA, DC1), fm(BA1, CDDC));
    out[0] = __fdiv_rn(Dx, DH);
    out[1] = __fdiv_rn(Dy, DH);
    return true;
}

// The intersection polygon of two convex quadrilaterals has at most 8 vertices; the 16-float array is the reference's
// (rotate_iou.py:235), and a degenerate input that would produce more points keeps the first 8 instead of writing past it.
__device__ float rotated_intersection(const float* rb1, const float* rb2) {                 // rotate_iou.py:231-245
    float c1[8], c2[8], pts[16], vs[8];
    box_corners(rb1, c1);
    box_corners(rb2, c2);
    int n = 0;
    for (int i = 0; i < 4; ++i) {                                                             // rotate_iou.py:180-201
        if (point_in_quad(c1[2 * i], c1[2 * i + 1], c2) && n < 8) { pts[2 * n] = c1[2 * i]; pts[2 * n + 1] = c1[2 * i + 1]; ++n; }
        if (point_in_quad(c2[2 * i], c2[2 * i + 1], c1) && n < 8) { pts[2 * n] = c2[2 * i]; pts[2 * n + 1] = c2[2 * i + 1]; ++n; }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float t[2];
            if (segment_intersection(c1, c2, i, j, t) && n < 8) { pts[2 * n] = t[0]; pts[2 * n + 1] = t[1]; ++n; }
        }
    if (n > 0) {                                                                              // rotate_iou.py:33-70
        float cx = 0.f, cy = 0.f;
        for (int i = 0; i < n; ++i) { cx = fa(cx, pts[2 * i]); cy = fa(cy, pts[2 * i + 1]); }
        cx = __fdiv_rn(cx, (float)n);
        cy = __fdiv_rn(cy, (float)n);
        for (int i = 0; i < n; ++i) {
            float v0 = fs(pts[2 * i], cx), v1 = fs(pts[2 * i + 1], cy);
            const float d = __fsqrt_rn(fa(fm(v0, v0), fm(v1, v1)));
            v0 = __fdiv_rn(v0, d);
            v1 = __fdiv_rn(v1, d);
            if (v1 < 0.f) v0 = fs(-2.f, v0);
            vs[i] = v0;
        }
        for (int i = 1; i < n; ++i) {
            if (vs[i - 1] > vs[i]) {
                const float tmp = vs[i], tx = pts[2 * i], ty = pts[2 * i + 1];
                int j = i;
                while (j > 0 && vs[j - 1] > tmp) {
                    vs[j] = vs[j - 1];
                    pts[2 * j] = pts[2 * j - 2];
                    pts[2 * j + 1] = pts[2 * j - 1];
                    --j;
                }
                vs[j] = tmp;
                pts[2 * j] = tx;
                pts[2 * j + 1] = ty;
            }
        }
    }
    float area = 0.f;                                                                         // rotate_iou.py:17-30
    for (int i = 0; i + 2 < n; ++i) {
        const float a0 = pts[0], a1 = pts[1], b0 = pts[2 * i + 2], b1 = pts[2 * i + 3], c0 = pts[2 * i + 4], c1v = pts[2 * i + 5];
        const float tri = fs(fm(fs(a0, c0), fs(b1, c1v)), fm(fs(a1, c1v), fs(b0, c0))) / 2.f;
        area = fa(area, fabsf(tri));
    }
    return area;
}

// 2-d overlap of eval.py:162-189 for one (box, query) pair; criterion -1 (IoU) or 0 (over the box's own area).
__device__ double image_overlap(const double* b, const double* q, int criterion) {
    const double iw = __dsub_rn(fmin(b[2], q[2]), fmax(b[0], q[0]));
    if (!(iw > 0.0)) return 0.0;
    const double ih = __dsub_rn(fmin(b[3], q[3]), fmax(b[1], q[1]));
    if (!(ih > 0.0)) return 0.0;
    const double barea = __dmul_rn(__dsub_rn(b[2], b[0]), __dsub_rn(b[3], b[1]));
    const double inter = __dmul_rn(iw, ih);
    double ua = barea;
    if (criterion == -1) {
        const double qarea = __dmul_rn(__dsub_rn(q[2], q[0]), __dsub_rn(q[3], q[1]));
        ua = __dsub_rn(__dadd_rn(barea, qarea), inter);
    }
    return __ddiv_rn(inter, ua);
}

// Overlaps of image b, all three metrics: block (n_dt, n_gt), detection-major, as calculate_iou_partly(dt_annos, gt_annos)
// returns it (eval.py:550).  bbox: image_box_overlap(dt, gt).  BEV: rotate_iou_gpu_eval(dt, gt) = devRotateIoUEval(gt, dt), fp32,
// criterion -1.  3d: the same fp32 intersection (criterion 2), then d3_box_overlap_kernel's fp64 height overlap and volumes, the
// result stored through the fp32 array the reference writes it into.
__global__ void __launch_bounds__(128) overlaps_kernel(const int* __restrict__ gt_off, const int* __restrict__ dt_off,
                                                       const long long* __restrict__ ov_off, long long n_ov,
                                                       const double* __restrict__ gt_f, const double* __restrict__ dt_f,
                                                       double* __restrict__ out) {
    const int b = blockIdx.x;
    const int g0 = gt_off[b], ng = gt_off[b + 1] - g0, d0 = dt_off[b], nd = dt_off[b + 1] - d0;
    if (ng > kMaxBoxes || nd > kMaxBoxes) return;
    double* o2 = out + ov_off[b];
    double* obev = o2 + n_ov;
    double* o3 = obev + n_ov;
    for (int p = threadIdx.x; p < ng * nd; p += blockDim.x) {
        const int j = p / ng, i = p - j * ng;
        const double* g = gt_f + (size_t)(g0 + i) * kGtCols;
        const double* d = dt_f + (size_t)(d0 + j) * kDtCols;
        o2[p] = image_overlap(d, g, -1);
        const float rg[5] = {(float)g[6], (float)g[8], (float)g[9], (float)g[11], (float)g[12]};   // x, z, l, w, ry
        const float rd[5] = {(float)d[6], (float)d[8], (float)d[9], (float)d[11], (float)d[12]};
        const float inter = rotated_intersection(rg, rd);
        const float area_g = fm(rg[2], rg[3]), area_d = fm(rd[2], rd[3]);
        obev[p] = (double)__fdiv_rn(inter, fs(fa(area_g, area_d), inter));
        float r3 = inter;                                                                     // eval.py:197-223
        if (inter > 0.f) {
            // columns 7 = y, 10 = h; boxes = detections, qboxes = gt
            const double iw = __dsub_rn(fmin(d[7], g[7]), fmax(__dsub_rn(d[7], d[10]), __dsub_rn(g[7], g[10])));
            if (iw > 0.0) {
                const double vd = __dmul_rn(__dmul_rn(d[9], d[10]), d[11]), vg = __dmul_rn(__dmul_rn(g[9], g[10]), g[11]);
                const double inc = __dmul_rn(iw, (double)inter);
                r3 = (float)__ddiv_rn(inc, __dsub_rn(__dadd_rn(vd, vg), inc));
            } else {
                r3 = 0.f;
            }
        }
        o3[p] = (double)r3;
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// clean_data (eval.py:30-82) for one (class m, difficulty l) per CTA: ignored_gt / ignored_dt in {-1, 0, 1} and num_valid_gt.
// BY_DISTANCE: clean_data_by_distance (eval.py:85-159, DISTANCE_COVER = False) for one (class m, distance bin l) per CTA.  Every
// bin takes the hard level's limits, and a gt is also ignored outside its bin of ||location||: (0, 30], (30, 50], (50, 70] m
// (the first bin has no lower edge).  The norm is fp64 x*x + y*y + z*z, left to right and correctly rounded.
template <bool BY_DISTANCE>
__global__ void __launch_bounds__(256) clean_kernel(const double* __restrict__ gt_f, const int* __restrict__ gt_i,
                                                    const double* __restrict__ dt_f, const int* __restrict__ dt_cls,
                                                    const int* __restrict__ classes, int n_gt, int n_dt, signed char* __restrict__ ign_gt,
                                                    signed char* __restrict__ ign_dt, int* __restrict__ n_valid) {
    const int ml = blockIdx.x, m = ml / 3, l = ml - m * 3;
    const int cls = classes[m];
    const int lv = BY_DISTANCE ? 2 : l;                                                   // the level whose limits apply
    const double min_height = lv == 0 ? 40.0 : 25.0, max_trunc = lv == 0 ? 0.15 : (lv == 1 ? 0.3 : 0.5);   // eval.py:32-34
    const int max_occ = lv;
    int mine = 0;
    for (int g = threadIdx.x; g < n_gt; g += blockDim.x) {
        const double* f = gt_f + (size_t)g * kGtCols;
        const int occ = gt_i[g * 3 + 0], code = gt_i[g * 3 + 1];
        const int valid = code == cls ? 1 : ((cls == 1 && code == 4) || (cls == 0 && code == 3)) ? 0 : -1;
        const double height = __dsub_rn(f[3], f[1]);
        bool ignore = occ > max_occ || f[5] > max_trunc || height <= min_height;
        if (BY_DISTANCE) {                                                                // eval.py:112, 121-133
            const double dis = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(f[6], f[6]), __dmul_rn(f[7], f[7])), __dmul_rn(f[8], f[8])));
            const double hi = l == 0 ? 30.0 : (l == 1 ? 50.0 : 70.0), lo = l == 1 ? 30.0 : 50.0;
            ignore = ignore || dis > hi || (l > 0 && dis <= lo);
        }
        signed char v;
        if (valid == 1 && !ignore) { v = 0; ++mine; }
        else if (valid == 0 || (ignore && valid == 1)) v = 1;
        else v = -1;
        ign_gt[(size_t)ml * n_gt + g] = v;
    }
    for (int d = threadIdx.x; d < n_dt; d += blockDim.x) {
        const double* f = dt_f + (size_t)d * kDtCols;
        const double height = fabs(__dsub_rn(f[3], f[1]));
        ign_dt[(size_t)ml * n_dt + d] = height < min_height ? 1 : (dt_cls[d] == cls ? 0 : -1);
    }
    __shared__ int s_count[8];
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0) s_count[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += s_count[w];
        n_valid[ml] = s;
    }
}

// Configuration index cfg = ((metric * n_cls + m) * 3 + difficulty) * 2 + k (k indexes the two overlap sets).
struct Cfg {
    int metric, m, l, k, ml;
};
__device__ __forceinline__ Cfg decode_cfg(int cfg, int n_cls) {
    Cfg c;
    c.k = cfg & 1;
    c.l = (cfg >> 1) % 3;
    c.m = ((cfg >> 1) / 3) % n_cls;
    c.metric = ((cfg >> 1) / 3) / n_cls;
    c.ml = c.m * 3 + c.l;
    return c;
}

struct Inputs {
    const int* gt_off;
    const int* dt_off;
    const long long* ov_off;
    long long n_ov;
    const double* gt_f;
    const int* gt_i;
    const double* dt_f;
    const double* overlaps;
    const double* min_overlaps;   // [2][3][n_cls]
    const signed char* ign_gt;
    const signed char* ign_dt;
    int n_img, n_gt, n_dt, n_cls;
};

// Warp-wide choice of the detection a gt takes.  Each lane owns detections lane + 32 q (q < 32) and scans them in increasing
// order, so a strict comparison keeps the lowest index; the shuffle reduction breaks ties by the lower index as well.
__device__ __forceinline__ void warp_best(double& key, int& idx) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double k2 = __shfl_xor_sync(0xffffffffu, key, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, idx, o);
        if (i2 >= 0 && (idx < 0 || k2 > key || (k2 == key && i2 < idx))) { key = k2; idx = i2; }
    }
}

__device__ __forceinline__ int warp_min(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Pass 1, compute_statistics_jit(compute_fp=False) (eval.py:233-317): every gt that is not ignored takes the highest-scoring
// free detection above the overlap, ignored detections included; a match of a valid gt with a valid detection is a TP whose
// score is written to scores[cfg][gt_off[b] + t] (t-th TP of the image); the other slots of the image get -inf.
__global__ void __launch_bounds__(kWarps * 32) pass1_kernel(Inputs in, double* __restrict__ scores, long long P) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * kWarps + (threadIdx.x >> 5), cfg = blockIdx.y;
    if (b >= in.n_img) return;
    const Cfg c = decode_cfg(cfg, in.n_cls);
    const double mo = in.min_overlaps[(c.k * 3 + c.metric) * in.n_cls + c.m];
    const int g0 = in.gt_off[b], ng = in.gt_off[b + 1] - g0, d0 = in.dt_off[b], nd = in.dt_off[b + 1] - d0;
    if (ng > kMaxBoxes || nd > kMaxBoxes) return;
    const double* ov = in.overlaps + c.metric * in.n_ov + in.ov_off[b];
    const signed char* igt = in.ign_gt + (size_t)c.ml * in.n_gt + g0;
    const signed char* idt = in.ign_dt + (size_t)c.ml * in.n_dt + d0;
    const double* dt = in.dt_f + (size_t)d0 * kDtCols;
    unsigned elig = 0, ign1 = 0, assigned = 0;
    for (int q = 0; lane + 32 * q < nd; ++q) {
        const int v = idt[lane + 32 * q];
        if (v != -1) elig |= 1u << q;
        if (v == 1) ign1 |= 1u << q;
    }
    double* out = scores + (long long)cfg * P + g0;
    int ntp = 0;
    for (int i = 0; i < ng; ++i) {
        const int gi = igt[i];
        if (gi == -1) continue;
        double best = kNoDetection;
        int bj = -1;
        for (unsigned free = elig & ~assigned; free; free &= free - 1) {
            const int j = lane + 32 * (__ffs(free) - 1);
            const double s = dt[(size_t)j * kDtCols + 5];
            if (ov[(size_t)j * ng + i] > mo && s > best) { best = s; bj = j; }
        }
        warp_best(best, bj);
        if (bj < 0) continue;
        const bool det_ignored = __shfl_sync(0xffffffffu, (int)((ign1 >> (bj >> 5)) & 1u), bj & 31) != 0;
        if (lane == (bj & 31)) assigned |= 1u << (bj >> 5);
        if (gi == 1 || det_ignored) continue;
        if (lane == 0) out[ntp] = dt[(size_t)bj * kDtCols + 5];
        ++ntp;
    }
    for (int t = ntp + lane; t < ng; t += 32) out[t] = -INFINITY;
}

// get_thresholds (eval.py:9-27) for one configuration per CTA.  The TP scores are sorted descending by a bitonic sort over
// scores[cfg][0, P) (P = a power of two >= n_gt, the slots past n_gt are filled with -inf first); which ranks are kept depends
// only on (number of TP scores, num_valid_gt) and is decided by one thread in the reference's fp64 order.  Also clears the
// configuration's pass-2 counters.
__global__ void __launch_bounds__(512) thresholds_kernel(double* __restrict__ scores, long long P, int n_gt, int n_cls,
                                                          const int* __restrict__ n_valid, double* __restrict__ thr,
                                                          int* __restrict__ n_thr, int* __restrict__ counts) {
    const int cfg = blockIdx.x;
    double* s = scores + (long long)cfg * P;
    for (long long i = n_gt + threadIdx.x; i < P; i += blockDim.x) s[i] = -INFINITY;
    for (int i = threadIdx.x; i < kThr * 3; i += blockDim.x) counts[cfg * kThr * 3 + i] = 0;
    __syncthreads();
    for (long long k = 2; k <= P; k <<= 1)
        for (long long j = k >> 1; j > 0; j >>= 1) {
            for (long long i = threadIdx.x; i < P; i += blockDim.x) {
                const long long p = i ^ j;
                if (p > i) {
                    const double a = s[i], bv = s[p];
                    const bool desc = (i & k) == 0;
                    if (desc ? a < bv : a > bv) { s[i] = bv; s[p] = a; }
                }
            }
            __syncthreads();
        }
    __shared__ int s_ntp[16];
    int mine = 0;
    for (long long i = threadIdx.x; i < P; i += blockDim.x) mine += s[i] > -INFINITY;
    mine = warp_sum(mine);
    if ((threadIdx.x & 31) == 0) s_ntp[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x != 0) return;
    int n = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) n += s_ntp[w];
    const Cfg c = decode_cfg(cfg, n_cls);
    const int num_gt = n_valid[c.ml];
    double current = 0.0;
    int count = 0;
    for (int i = 0; i < n; ++i) {
        const double l_recall = (double)(i + 1) / (double)num_gt;
        const double r_recall = i < n - 1 ? (double)(i + 2) / (double)num_gt : l_recall;
        if ((r_recall - current) < (current - l_recall) && i < n - 1) continue;
        if (count < kThr) thr[cfg * kThr + count] = s[i];
        ++count;
        current += 1.0 / (41 - 1.0);
    }
    n_thr[cfg] = count;
}

// Pass 2, compute_statistics_jit(compute_fp=True) for one (configuration, image, threshold) per warp (eval.py:233-350 as
// fused_compute_statistics calls it, :365-412).  A gt takes, among the free detections above the overlap whose score reaches the
// threshold, the non-ignored one of highest overlap (lowest index on ties), or failing that the first ignored one.  tp / fp / fn
// go to counts[cfg][t] by integer atomics; the image's AOS similarity (2-d metric only) to sim[cfg][t][b].
__global__ void __launch_bounds__(kWarps * 32) pass2_kernel(Inputs in, const double* __restrict__ thr, const int* __restrict__ n_thr,
                                                            int compute_aos, int* __restrict__ counts, double* __restrict__ sim) {
    const int lane = threadIdx.x & 31;
    const int w = blockIdx.x * kWarps + (threadIdx.x >> 5), cfg = blockIdx.y;
    const int b = w / kThr, t = w - b * kThr;
    if (b >= in.n_img || t >= n_thr[cfg]) return;
    const Cfg c = decode_cfg(cfg, in.n_cls);
    const bool aos = compute_aos && c.metric == 0;
    double* sim_out = aos ? sim + ((size_t)cfg * kThr + t) * in.n_img + b : nullptr;
    const double mo = in.min_overlaps[(c.k * 3 + c.metric) * in.n_cls + c.m];
    const double thresh = thr[cfg * kThr + t];
    const int g0 = in.gt_off[b], ng = in.gt_off[b + 1] - g0, d0 = in.dt_off[b], nd = in.dt_off[b + 1] - d0;
    if (ng > kMaxBoxes || nd > kMaxBoxes) return;
    const double* ov = in.overlaps + c.metric * in.n_ov + in.ov_off[b];
    const signed char* igt = in.ign_gt + (size_t)c.ml * in.n_gt + g0;
    const signed char* idt = in.ign_dt + (size_t)c.ml * in.n_dt + d0;
    const double* gt = in.gt_f + (size_t)g0 * kGtCols;
    const double* dt = in.dt_f + (size_t)d0 * kDtCols;
    unsigned elig = 0, ign1 = 0, assigned = 0;                  // elig: ignored_det != -1 and score >= thresh
    for (int q = 0; lane + 32 * q < nd; ++q) {
        const int j = lane + 32 * q, v = idt[j];
        if (v != -1 && !(dt[(size_t)j * kDtCols + 5] < thresh)) elig |= 1u << q;
        if (v == 1) ign1 |= 1u << q;
    }
    int tp = 0, fn = 0;
    double similarity = 0.0;
    for (int i = 0; i < ng; ++i) {
        const int gi = igt[i];
        if (gi == -1) continue;
        double best = -INFINITY;
        int bj = -1, first_ign = 0x7fffffff;
        for (unsigned free = elig & ~assigned; free; free &= free - 1) {
            const int q = __ffs(free) - 1, j = lane + 32 * q;
            const double o = ov[(size_t)j * ng + i];
            if (!(o > mo)) continue;
            if ((ign1 >> q) & 1u) first_ign = min(first_ign, j);
            else if (bj < 0 || o > best) { best = o; bj = j; }
        }
        warp_best(best, bj);
        first_ign = warp_min(first_ign);
        const int det = bj >= 0 ? bj : (first_ign != 0x7fffffff ? first_ign : -1);
        if (det < 0) {
            if (gi == 0) ++fn;
            continue;
        }
        if (lane == (det & 31)) assigned |= 1u << (det >> 5);
        const bool det_ignored = bj < 0;
        if (gi == 1 || det_ignored) continue;
        ++tp;
        if (aos) {
            const double delta = __dsub_rn(gt[(size_t)i * kGtCols + 4], dt[(size_t)det * kDtCols + 4]);
            similarity = __dadd_rn(similarity, __ddiv_rn(__dadd_rn(1.0, cos(delta)), 2.0));
        }
    }
    // fp: valid detections above the threshold left unassigned, minus those a DontCare region absorbs (2-d metric only)
    unsigned open = elig & ~ign1 & ~assigned;
    int fp = __popc(open), nstuff = 0;
    if (c.metric == 0) {
        for (; open; open &= open - 1) {
            const int j = lane + 32 * (__ffs(open) - 1);
            for (int i = 0; i < ng; ++i) {
                if (!in.gt_i[(size_t)(g0 + i) * 3 + 2]) continue;
                if (image_overlap(dt + (size_t)j * kDtCols, gt + (size_t)i * kGtCols, 0) > mo) { ++nstuff; break; }
            }
        }
    }
    fp = warp_sum(fp - nstuff);
    if (lane == 0) {
        int* cnt = counts + ((size_t)cfg * kThr + t) * 3;
        if (tp) atomicAdd(cnt + 0, tp);
        if (fp) atomicAdd(cnt + 1, fp);
        if (fn) atomicAdd(cnt + 2, fn);
        if (aos) *sim_out = similarity;
    }
}

// result[cfg] = [n_thr, (tp, fp, fn, similarity) x 41]; the similarity summed over images in image order.
__global__ void reduce_kernel(int n_cfg, int n_img, int compute_aos, int n_cls, const int* __restrict__ n_thr,
                              const int* __restrict__ counts, const double* __restrict__ sim, double* __restrict__ result) {
    const int id = blockIdx.x * blockDim.x + threadIdx.x;
    if (id >= n_cfg * kThr) return;
    const int cfg = id / kThr, t = id - cfg * kThr;
    double* r = result + (size_t)cfg * (1 + 4 * kThr);
    if (t == 0) r[0] = (double)n_thr[cfg];
    double* row = r + 1 + 4 * t;
    const int* cnt = counts + (size_t)id * 3;
    const bool used = t < n_thr[cfg];
    row[0] = used ? (double)cnt[0] : 0.0;
    row[1] = used ? (double)cnt[1] : 0.0;
    row[2] = used ? (double)cnt[2] : 0.0;
    double s = 0.0;
    if (used && compute_aos && decode_cfg(cfg, n_cls).metric == 0) {
        const double* p = sim + (size_t)id * n_img;
        for (int b = 0; b < n_img; ++b) s = __dadd_rn(s, p[b]);
    }
    row[3] = s;
}

// Workspace layout, 256-byte aligned pieces.
struct Workspace {
    size_t ign_gt, ign_dt, n_valid, scores, thr, n_thr, counts, sim, total;
    long long P;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

Workspace layout(int n_img, int n_gt, int n_dt, int n_cls, int compute_aos) {
    Workspace w;
    const int n_cfg = 3 * n_cls * 3 * 2;
    long long P = 1;
    while (P < n_gt) P <<= 1;
    w.P = P;
    size_t o = 0;
    w.ign_gt = o; o = align256(o + (size_t)n_cls * 3 * n_gt);
    w.ign_dt = o; o = align256(o + (size_t)n_cls * 3 * n_dt);
    w.n_valid = o; o = align256(o + sizeof(int) * n_cls * 3);
    w.scores = o; o = align256(o + sizeof(double) * (size_t)n_cfg * P);
    w.thr = o; o = align256(o + sizeof(double) * n_cfg * kThr);
    w.n_thr = o; o = align256(o + sizeof(int) * n_cfg);
    w.counts = o; o = align256(o + sizeof(int) * n_cfg * kThr * 3);
    w.sim = o; o = align256(o + (compute_aos ? sizeof(double) * (size_t)n_cfg * kThr * n_img : 0));
    w.total = o;
    return w;
}

int check_sizes(int n_img, int n_gt, int n_dt, int n_cls, int max_gt, int max_dt) {
    if (n_img < 1 || n_gt < 0 || n_dt < 0 || max_gt < 0 || max_dt < 0) return MDB_EINVAL;
    if (n_cls < 1 || n_cls > MDB_KITTI_MAX_CLASSES) return MDB_EUNSUPPORTED;
    if (max_gt > kMaxBoxes || max_dt > kMaxBoxes) return MDB_EUNSUPPORTED;
    if (n_gt > MDB_KITTI_MAX_TOTAL_GT || (long long)n_img * kThr > 0x7fffffffLL / 2) return MDB_EUNSUPPORTED;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// Detections of the validation pass, collected on the device (the path that replaced tester_helper.py:112-132 writing result
// files and kitti_common.py:294-347 reading them back).  A value goes through the text as '{:.2f}' of the float32 and float()
// of the text; for a float32 x that is rint(x * 100) / 100 in fp64: the product is exact (24 + 7 significant bits), rint rounds
// half to even as the formatting does, and the correctly rounded quotient is the double nearest the printed decimal.
constexpr int kRowCols = 14;                     // mdb_decode_dets_f32: cls, alpha, x0 y0 x1 y1, h w l, X Y Z, ry, score
constexpr int kCollectBatch = MDB_KITTI_COLLECT_MAX_BATCH;
__constant__ int kDtFromRow[kDtCols] = {2, 3, 4, 5, 1, 13, 9, 10, 11, 8, 6, 7, 12};   // dt_f column <- row column

__device__ __forceinline__ double text_round(float x) { return __ddiv_rn(rint(__dmul_rn((double)x, 100.0)), 100.0); }

struct CollectArgs {               // by value: the slots were range-checked on the host, no upload is needed
    int slot[kCollectBatch];
    int code[MDB_KITTI_COLLECT_MAX_CLASSES];
    int n_code;
};

// One CTA per batch image: its count leading rows go to slot slot[b] of the padded table; slot_info (3, n_img) records the count,
// how many times the slot was written, and whether the first detection's printed alpha differs from -10 (eval.py:745-751).
__global__ void __launch_bounds__(128) collect_kernel(const float* __restrict__ rows, const int* __restrict__ count, int topk,
                                                      int n_img, CollectArgs a, double* __restrict__ table_f,
                                                      int* __restrict__ table_cls, int* __restrict__ slot_info) {
    const int b = blockIdx.x, s = a.slot[b];
    const int n = min(max(count[b], 0), topk);
    const float* r = rows + (size_t)b * topk * kRowCols;
    double* f = table_f + (size_t)s * topk * kDtCols;
    for (int i = threadIdx.x; i < n * kDtCols; i += blockDim.x) {
        const int k = i / kDtCols, c = i - k * kDtCols;
        f[i] = text_round(r[k * kRowCols + kDtFromRow[c]]);
    }
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
        const int id = (int)r[k * kRowCols];                            // the tester's int(cls_id)
        table_cls[(size_t)s * topk + k] = id >= 0 && id < a.n_code ? a.code[id] : -1;
    }
    if (threadIdx.x == 0) {
        slot_info[s] = n;
        atomicAdd(slot_info + n_img + s, 1);
        slot_info[2 * n_img + s] = n > 0 && text_round(r[1]) != -10.0;
    }
}

// The padded table -> the CSR dt_f / dt_cls of mdb_kitti_eval, one CTA per slot.
__global__ void __launch_bounds__(128) compact_kernel(const int* __restrict__ dt_off, const double* __restrict__ table_f,
                                                      const int* __restrict__ table_cls, int topk, double* __restrict__ dt_f,
                                                      int* __restrict__ dt_cls) {
    const int s = blockIdx.x, d0 = dt_off[s], n = dt_off[s + 1] - d0;
    const double* f = table_f + (size_t)s * topk * kDtCols;
    for (int i = threadIdx.x; i < n * kDtCols; i += blockDim.x) dt_f[(size_t)d0 * kDtCols + i] = f[i];
    for (int k = threadIdx.x; k < n; k += blockDim.x) dt_cls[d0 + k] = table_cls[(size_t)s * topk + k];
}

}  // namespace

extern "C" int mdb_kitti_collect_dets_f32(const float* rows, const int* count, const int* slot, int B, int topk, int n_img,
                                          const int* cls_code, int n_code, double* table_f, int* table_cls, int* slot_info,
                                          void* stream) {
    if (!rows || !count || !slot || !table_f || !table_cls || !slot_info || (n_code > 0 && !cls_code)) return MDB_EINVAL;
    if (B < 0 || topk < 1 || n_img < 1 || n_code < 0) return MDB_EINVAL;
    if (topk > kMaxBoxes || n_code > MDB_KITTI_COLLECT_MAX_CLASSES) return MDB_EUNSUPPORTED;
    for (int b = 0; b < B; ++b)
        if (slot[b] < 0 || slot[b] >= n_img) return MDB_EINVAL;
    CollectArgs a;
    a.n_code = n_code;
    for (int c = 0; c < n_code; ++c) a.code[c] = cls_code[c];
    for (int b0 = 0; b0 < B; b0 += kCollectBatch) {
        const int nb = min(B - b0, kCollectBatch);
        for (int b = 0; b < nb; ++b) a.slot[b] = slot[b0 + b];
        collect_kernel<<<nb, 128, 0, (cudaStream_t)stream>>>(rows + (size_t)b0 * topk * kRowCols, count + b0, topk, n_img, a,
                                                             table_f, table_cls, slot_info);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return (int)e;
    }
    return 0;
}

extern "C" int mdb_kitti_compact_dets(const int* dt_off, const double* table_f, const int* table_cls, int n_img, int topk,
                                      double* dt_f, int* dt_cls, void* stream) {
    if (!dt_off || !table_f || !table_cls || !dt_f || !dt_cls || n_img < 0 || topk < 1) return MDB_EINVAL;
    if (topk > kMaxBoxes) return MDB_EUNSUPPORTED;
    if (n_img == 0) return 0;
    compact_kernel<<<n_img, 128, 0, (cudaStream_t)stream>>>(dt_off, table_f, table_cls, topk, dt_f, dt_cls);
    return (int)cudaGetLastError();
}

extern "C" int mdb_kitti_overlaps(const int* gt_off, const int* dt_off, const long long* ov_off, int n_img, int max_gt, int max_dt,
                                  long long n_ov, const double* gt_f, const double* dt_f, double* overlaps, void* stream) {
    if (!gt_off || !dt_off || !ov_off || (n_ov > 0 && (!gt_f || !dt_f || !overlaps))) return MDB_EINVAL;
    if (n_img < 0 || n_ov < 0 || max_gt < 0 || max_dt < 0) return MDB_EINVAL;
    if (max_gt > kMaxBoxes || max_dt > kMaxBoxes) return MDB_EUNSUPPORTED;
    if (n_img == 0 || n_ov == 0) return 0;
    overlaps_kernel<<<n_img, 128, 0, (cudaStream_t)stream>>>(gt_off, dt_off, ov_off, n_ov, gt_f, dt_f, overlaps);
    return (int)cudaGetLastError();
}

extern "C" long long mdb_kitti_eval_workspace_bytes(int n_img, int n_gt, int n_dt, int n_cls, int compute_aos) {
    const int rc = check_sizes(n_img, n_gt, n_dt, n_cls, 0, 0);
    if (rc) return rc;
    return (long long)layout(n_img, n_gt, n_dt, n_cls, compute_aos).total;
}

namespace {

// Both entry points: the configurations differ only in how clean_kernel assigns the third index (difficulty or distance bin).
int kitti_eval_impl(bool by_distance, const int* gt_off, const int* dt_off, const long long* ov_off, int n_img, int n_gt, int n_dt,
                    int max_gt, int max_dt, long long n_ov, const double* gt_f, const int* gt_i, const double* dt_f, const int* dt_cls,
                    const double* overlaps, const int* classes, const double* min_overlaps, int n_cls, int compute_aos,
                    void* workspace, long long workspace_bytes, double* result, void* stream) {
    if (!gt_off || !dt_off || !ov_off || !classes || !min_overlaps || !result) return MDB_EINVAL;
    if ((n_gt > 0 && (!gt_f || !gt_i)) || (n_dt > 0 && (!dt_f || !dt_cls)) || (n_ov > 0 && !overlaps) || n_ov < 0) return MDB_EINVAL;
    const int rc = check_sizes(n_img, n_gt, n_dt, n_cls, max_gt, max_dt);
    if (rc) return rc;
    const Workspace w = layout(n_img, n_gt, n_dt, n_cls, compute_aos);
    if (!workspace || workspace_bytes < (long long)w.total) return MDB_EWORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    char* ws = (char*)workspace;
    const int n_cfg = 3 * n_cls * 3 * 2;
    Inputs in{gt_off, dt_off, ov_off, n_ov, gt_f, gt_i, dt_f, overlaps, min_overlaps, (const signed char*)(ws + w.ign_gt),
              (const signed char*)(ws + w.ign_dt), n_img, n_gt, n_dt, n_cls};
    int* n_valid = (int*)(ws + w.n_valid);
    double* scores = (double*)(ws + w.scores);
    double* thr = (double*)(ws + w.thr);
    int* n_thr = (int*)(ws + w.n_thr);
    int* counts = (int*)(ws + w.counts);
    double* sim = (double*)(ws + w.sim);
    auto clean = by_distance ? clean_kernel<true> : clean_kernel<false>;
    clean<<<n_cls * 3, 256, 0, s>>>(gt_f, gt_i, dt_f, dt_cls, classes, n_gt, n_dt, (signed char*)(ws + w.ign_gt),
                                    (signed char*)(ws + w.ign_dt), n_valid);
    pass1_kernel<<<dim3((n_img + kWarps - 1) / kWarps, n_cfg), kWarps * 32, 0, s>>>(in, scores, w.P);
    thresholds_kernel<<<n_cfg, 512, 0, s>>>(scores, w.P, n_gt, n_cls, n_valid, thr, n_thr, counts);
    pass2_kernel<<<dim3((n_img * kThr + kWarps - 1) / kWarps, n_cfg), kWarps * 32, 0, s>>>(in, thr, n_thr, compute_aos, counts, sim);
    reduce_kernel<<<(n_cfg * kThr + 127) / 128, 128, 0, s>>>(n_cfg, n_img, compute_aos, n_cls, n_thr, counts, sim, result);
    return (int)cudaGetLastError();
}

}  // namespace

extern "C" int mdb_kitti_eval(const int* gt_off, const int* dt_off, const long long* ov_off, int n_img, int n_gt, int n_dt,
                              int max_gt, int max_dt, long long n_ov, const double* gt_f, const int* gt_i, const double* dt_f,
                              const int* dt_cls, const double* overlaps, const int* classes, const double* min_overlaps, int n_cls,
                              int compute_aos, void* workspace, long long workspace_bytes, double* result, void* stream) {
    return kitti_eval_impl(false, gt_off, dt_off, ov_off, n_img, n_gt, n_dt, max_gt, max_dt, n_ov, gt_f, gt_i, dt_f, dt_cls, overlaps,
                           classes, min_overlaps, n_cls, compute_aos, workspace, workspace_bytes, result, stream);
}

extern "C" int mdb_kitti_eval_distance(const int* gt_off, const int* dt_off, const long long* ov_off, int n_img, int n_gt, int n_dt,
                                       int max_gt, int max_dt, long long n_ov, const double* gt_f, const int* gt_i, const double* dt_f,
                                       const int* dt_cls, const double* overlaps, const int* classes, const double* min_overlaps,
                                       int n_cls, int compute_aos, void* workspace, long long workspace_bytes, double* result,
                                       void* stream) {
    return kitti_eval_impl(true, gt_off, dt_off, ov_off, n_img, n_gt, n_dt, max_gt, max_dt, n_ov, gt_f, gt_i, dt_f, dt_cls, overlaps,
                           classes, min_overlaps, n_cls, compute_aos, workspace, workspace_bytes, result, stream);
}
