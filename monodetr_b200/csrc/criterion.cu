// criterion.cu -- the training criterion on the device (SURVEY.md 8 f1): Hungarian matching + every loss term of the
// reference's SetCriterion without a single host synchronisation.  The reference moves the cost matrices to the host,
// solves 11 x B assignment problems per decoder layer with scipy and compacts the padded targets with boolean indexing
// (lib/models/monodetr/matcher.py:36-104, monodetr.py:297-532, lib/helpers/trainer_helper.py:175-186): ~40 host syncs a step.
//
//   prepare     compact list of the valid targets of every image from the loader's padded arrays + mask, counts, total
//   match       one warp per (decoder layer, image, query group): cost matrix in dynamic shared memory, sized by the launch's
//               queries per group and targets per image (matcher.py:57-84), and the rectangular linear-sum-assignment by
//               shortest augmenting paths -- the algorithm scipy.optimize.linear_sum_assignment implements (Crouse 2016) -- with
//               fp64 dual variables; writes the matched query of every target and the target class of every query
//   depth_map   per pixel: target depth bin from the ground-truth boxes (ddn_loss.py:43-101), 81-way softmax focal loss with
//               the one-hot + 1e-6 smoothing (focalloss.py:52-125) and the foreground / background balance (balancer.py:21-53);
//               gradient mode writes d loss / d logits
//   losses      one CTA per decoder layer, fixed-order reductions (deterministic): sigmoid focal loss over all (query, class)
//               (monodetr.py:316-345), cardinality error (:347-360), and over the matched pairs the 3-d centre / box L1 /
//               GIoU / depth (Laplacian aleatoric) / dimension / heading terms (:362-456), class_error
//   losses_backward   analytic gradients of the same terms; every element of the d pred_* buffers is written once (32 CTAs / layer)
// All fp32 (the matcher's dual variables fp64, like scipy).  Latency-bound: a few thousand pairs, 13 200 logits, 15 360 pixels.
// Parity: tests/test_criterion_gpu.py against oracle/criterion.py (autograd restatement, pinned to the unmodified reference by
// tests/golden/criterion.npz).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

constexpr int kMaxL = MDB_CRITERION_MAX_LAYERS;
constexpr int kNK = MDB_CRITERION_NUM_LOSSES;       // loss slots per layer (order documented in the header)
constexpr int kMaxTargets = 64;                     // targets per image the matcher accepts (so the rows' side is at most 64)
constexpr int kMaxQueries = 300;                    // queries per group the matcher accepts
constexpr int kBins = 12;                           // heading bins

struct LayerPtrs { const float* p[kMaxL]; };
struct LayerGradPtrs { float* p[kMaxL]; };

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// (cx, cy, l, r, t, b) -> x0 y0 x1 y1   utils/box_ops.py:20-24
__device__ __forceinline__ void to_xyxy(const float* b, float& x0, float& y0, float& x1, float& y1) {
    x0 = b[0] - b[2]; y0 = b[1] - b[4]; x1 = b[0] + b[3]; y1 = b[1] + b[5];
}
// utils/box_ops.py:35-72 for one pair
__device__ __forceinline__ float giou_pair(float ax0, float ay0, float ax1, float ay1, float bx0, float by0, float bx1, float by1) {
    const float area1 = (ax1 - ax0) * (ay1 - ay0), area2 = (bx1 - bx0) * (by1 - by0);
    const float iw = fmaxf(fminf(ax1, bx1) - fmaxf(ax0, bx0), 0.f), ih = fmaxf(fminf(ay1, by1) - fmaxf(ay0, by0), 0.f);
    const float inter = iw * ih, uni = area1 + area2 - inter;
    const float cw = fmaxf(fmaxf(ax1, bx1) - fminf(ax0, bx0), 0.f), ch = fmaxf(fmaxf(ay1, by1) - fminf(ay0, by0), 0.f);
    const float areac = cw * ch;
    return inter / uni - (areac - uni) / areac;
}

// ---- prepare ------------------------------------------------------------------------------------------------------------
__global__ void crit_prepare_kernel(const unsigned char* __restrict__ mask, int Gmax, int* __restrict__ tlist, int* __restrict__ count,
                                    float* __restrict__ total) {
    const int b = blockIdx.x;                       // one warp per image; order of the valid targets preserved
    int base = 0;
    for (int j0 = 0; j0 < Gmax; j0 += 32) {
        const int j = j0 + threadIdx.x;
        const bool v = j < Gmax && mask[b * Gmax + j] != 0;
        const unsigned m = __ballot_sync(0xffffffffu, v);
        if (v) tlist[b * Gmax + base + __popc(m & ((1u << threadIdx.x) - 1))] = j;
        base += __popc(m);
    }
    for (int j = base + threadIdx.x; j < Gmax; j += 32) tlist[b * Gmax + j] = -1;
    if (threadIdx.x == 0) { count[b] = base; atomicAdd(total, (float)base); }   // integers < 2^24: exact in any order
}

// ---- matcher ------------------------------------------------------------------------------------------------------------
// Dynamic shared memory of one matching with nq queries per group and at most Gmax targets (S = max(nq, Gmax) entries per side
// array; the rows are the smaller side, so R * Cn <= nq * Gmax):
//   double u[S], v[S], spc[S] | float cost[nq * Gmax] | int col4row[S], row4col[S], path[S], remaining[S] | uchar SR[S], SC[S]
// The cost entries are fp32 values widened to double where they are read, so storing them as float loses nothing; at
// 300 x 64 the matrix is 75 KB.
__host__ __device__ constexpr size_t match_smem_bytes(int nq, int Gmax) {
    return (size_t)(nq > Gmax ? nq : Gmax) * (3 * sizeof(double) + 4 * sizeof(int) + 2) + (size_t)nq * Gmax * sizeof(float);
}
constexpr int kMatchMaxSmem = (int)match_smem_bytes(kMaxQueries, kMaxTargets);

__global__ void __launch_bounds__(32) crit_match_kernel(LayerPtrs logits, LayerPtrs boxes, const int* __restrict__ labels,
                                                        const float* __restrict__ boxes3d, const int* __restrict__ tlist,
                                                        const int* __restrict__ count, int B, int Q, int C, int group, int Gmax,
                                                        float w_class, float w_center, float w_bbox, float w_giou,
                                                        int* __restrict__ match, int* __restrict__ tclass) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x;
    int p = blockIdx.x;
    const int g = p % group; p /= group;
    const int b = p % B;
    const int l = p / B;
    const int nq = Q / group, q0 = g * nq, nt = count[b];
    const int S = nq > Gmax ? nq : Gmax;
    double* u = reinterpret_cast<double*>(smem);
    double* v = u + S;
    double* spc = v + S;
    float* cost = reinterpret_cast<float*>(spc + S);
    int* col4row = reinterpret_cast<int*>(cost + (size_t)nq * Gmax);
    int* row4col = col4row + S;
    int* path = row4col + S;
    int* remaining = path + S;
    unsigned char* SR = reinterpret_cast<unsigned char*>(remaining + S);
    unsigned char* SC = SR + S;
    const float* lg = logits.p[l] + ((size_t)b * Q + q0) * C;
    const float* bx = boxes.p[l] + ((size_t)b * Q + q0) * 6;
    int* tc = tclass + ((size_t)l * B + b) * Q + q0;
    int* mt = match + (((size_t)l * B + b) * group + g) * Gmax;
    for (int i = lane; i < nq; i += 32) tc[i] = C;                  // "no object"
    for (int j = lane; j < Gmax; j += 32) mt[j] = -1;
    if (nt == 0) return;
    // rows = the smaller side: scipy transposes the (query x target) matrix only when it has more rows than columns
    const bool rows_are_targets = nt < nq;
    const int R = rows_are_targets ? nt : nq, Cn = rows_are_targets ? nq : nt;
    for (int e = lane; e < nq * nt; e += 32) {
        const int i = e / nt, j = e - i * nt;                        // query i, target j
        const int tj = tlist[b * Gmax + j];
        const float* tb = boxes3d + ((size_t)b * Gmax + tj) * 6;
        const float* qb = bx + (size_t)i * 6;
        const float prob = sigmoidf_(lg[(size_t)i * C + labels[b * Gmax + tj]]);
        const float neg = 0.75f * (prob * prob) * (-logf(1.f - prob + 1e-8f));               // matcher.py:64-68, alpha .25 gamma 2
        const float pos = 0.25f * ((1.f - prob) * (1.f - prob)) * (-logf(prob + 1e-8f));
        const float c_class = pos - neg;
        const float c_center = fabsf(qb[0] - tb[0]) + fabsf(qb[1] - tb[1]);
        const float c_bbox = fabsf(qb[2] - tb[2]) + fabsf(qb[3] - tb[3]) + fabsf(qb[4] - tb[4]) + fabsf(qb[5] - tb[5]);
        float ax0, ay0, ax1, ay1, bx0, by0, bx1, by1;
        to_xyxy(qb, ax0, ay0, ax1, ay1);
        to_xyxy(tb, bx0, by0, bx1, by1);
        const float c_giou = -giou_pair(ax0, ay0, ax1, ay1, bx0, by0, bx1, by1);
        const float c = w_bbox * c_bbox + w_center * c_center + w_class * c_class + w_giou * c_giou;   // matcher.py:87
        const int r = rows_are_targets ? j : i, cc = rows_are_targets ? i : j;
        cost[r * Cn + cc] = c;
    }
    for (int i = lane; i < S; i += 32) { u[i] = 0.0; v[i] = 0.0; col4row[i] = -1; row4col[i] = -1; }
    __syncwarp();
    const double kInf = 1e300;
    // Ties are broken as scipy's augmenting_path breaks them, so that equal-cost problems get scipy's assignment: the
    // unvisited columns are scanned in the order of `remaining` (reversed at first; a picked column is replaced by the last
    // entry), and a column of the same reduced cost displaces the current pick only if it is free.  The pick is therefore
    // the lowest reduced cost; among ties the last free column in scan order, or the first one if none is free.
    for (int cur = 0; cur < R; ++cur) {
        for (int i = lane; i < S; i += 32) { SR[i] = 0; SC[i] = 0; spc[i] = kInf; }
        for (int k = lane; k < Cn; k += 32) remaining[k] = Cn - 1 - k;
        __syncwarp();
        double minval = 0.0;
        int i = cur, sink = -1, nrem = Cn;
        while (sink < 0) {
            if (lane == 0) SR[i] = 1;
            double best = kInf;
            int bestk = -1, bestj = -1, bestfree = 0;
            for (int k = lane; k < nrem; k += 32) {                   // k rises along a lane's scan: scipy's rule applies as is
                const int j = remaining[k];
                const double r = minval + (double)cost[i * Cn + j] - u[i] - v[j];
                if (r < spc[j]) { spc[j] = r; path[j] = i; }
                const double s = spc[j];
                const int fr = row4col[j] < 0;
                if (s < best || (s == best && fr)) { best = s; bestk = k; bestj = j; bestfree = fr; }
            }
            // the lanes' picks ordered by (cost, free beats taken, free: later position first, taken: earlier position first)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int ok = __shfl_xor_sync(0xffffffffu, bestk, o), oj = __shfl_xor_sync(0xffffffffu, bestj, o);
                const int of = __shfl_xor_sync(0xffffffffu, bestfree, o);
                const bool tie_take = (of || bestfree) ? (of && (!bestfree || ok > bestk)) : ok < bestk;
                const bool take = ok >= 0 && (bestk < 0 || ob < best || (ob == best && tie_take));
                if (take) { best = ob; bestk = ok; bestj = oj; bestfree = of; }
            }
            if (bestk < 0 || !(best < kInf)) { sink = -2; break; }      // infeasible (NaN / inf costs): leave unmatched
            minval = best;
            if (lane == 0) { SC[bestj] = 1; remaining[bestk] = remaining[nrem - 1]; }
            --nrem;
            if (row4col[bestj] < 0) sink = bestj; else i = row4col[bestj];
            __syncwarp();
        }
        if (sink == -2) break;
        // dual update
        for (int r = lane; r < R; r += 32)
            if (SR[r]) u[r] += (r == cur) ? minval : minval - spc[col4row[r]];
        for (int j = lane; j < Cn; j += 32)
            if (SC[j]) v[j] -= minval - spc[j];
        __syncwarp();
        if (lane == 0) {                                              // augment along the path
            int j = sink;
            while (true) {
                const int r = path[j];
                row4col[j] = r;
                const int nj = col4row[r];
                col4row[r] = j;
                j = nj;
                if (r == cur) break;
            }
        }
        __syncwarp();
    }
    if (rows_are_targets) {
        for (int j = lane; j < nt; j += 32) {
            const int i = col4row[j];
            if (i >= 0) { mt[j] = q0 + i; tc[i] = labels[b * Gmax + tlist[b * Gmax + j]]; }
        }
    } else {
        for (int j = lane; j < nt; j += 32) {
            const int i = row4col[j];
            if (i >= 0) { mt[j] = q0 + i; tc[i] = labels[b * Gmax + tlist[b * Gmax + j]]; }
        }
    }
}

// ---- depth-map loss -------------------------------------------------------------------------------------------------------
// python slice semantics of `depth_maps[b, v1:v2, u1:u2]` (ddn_loss.py:64, balancer.py:79): negative bounds wrap once
__device__ __forceinline__ bool in_py_slice(int idx, long long start, long long stop, int n) {
    if (start < 0) { start += n; if (start < 0) start = 0; } else if (start > n) start = n;
    if (stop < 0) { stop += n; if (stop < 0) stop = 0; } else if (stop > n) stop = n;
    return idx >= start && idx < stop;
}

template <bool GRAD>
__global__ void crit_depth_map_kernel(const float* __restrict__ logits, long long sb, long long sp, long long sc, const float* __restrict__ boxes2d,
                                      const float* __restrict__ depth, const int* __restrict__ tlist, const int* __restrict__ count, int B, int H,
                                      int W, int nb, int Gmax, float sx, float sy, float dmin, float dmax, float alpha, float fg_w, float bg_w,
                                      float* __restrict__ pix_loss, const float* __restrict__ gw, float* __restrict__ dlogits) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int npix = B * H * W;
    if (warp >= npix) return;
    const int b = warp / (H * W), pix = warp - b * (H * W), y = pix / W, x = pix - y * W;
    // target depth of the pixel: boxes are painted far-to-near (ddn_loss.py:58-64), so the nearest covering box wins
    bool fg = false;
    float d = 0.f;
    const int nt = count[b];
    for (int k = lane; k < nt; k += 32) {
        const int t = tlist[b * Gmax + k];
        const float* bb = boxes2d + ((size_t)b * Gmax + t) * 4;
        // monodetr.py:462-463 rounds the scaled box before box_cxcywh_to_xyxy: the explicit roundings keep nvcc from
        // contracting bb[0] * sx into the subtraction, which moves a box edge that lies on a pixel boundary by one pixel
        const float cx = __fmul_rn(bb[0], sx), cy = __fmul_rn(bb[1], sy), hw = 0.5f * __fmul_rn(bb[2], sx), hh = 0.5f * __fmul_rn(bb[3], sy);
        const long long u1 = (long long)floorf(__fsub_rn(cx, hw)), v1 = (long long)floorf(__fsub_rn(cy, hh));
        const long long u2 = (long long)ceilf(__fadd_rn(cx, hw)), v2 = (long long)ceilf(__fadd_rn(cy, hh));
        if (in_py_slice(y, v1, v2, H) && in_py_slice(x, u1, u2, W)) {
            const float dk = depth[b * Gmax + t];
            d = fg ? fminf(d, dk) : dk;
            fg = true;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, d, o);
        const bool of = __shfl_xor_sync(0xffffffffu, (int)fg, o) != 0;
        if (of) { d = fg ? fminf(d, od) : od; fg = true; }
    }
    // LID bin (ddn_loss.py:84-98).  d - dmin, * 8, / bin_size, + 1 and sqrtf round one by one in the SASS; only
    // -0.5 + 0.5 * sqrt(...) is contracted into an FFMA, and 0.5 * sqrt(...) is exact, so (int)idxf sees the reference's value.
    const float bin_size = (float)(2.0 * ((double)dmax - (double)dmin) / ((double)nb * (1.0 + (double)nb)));
    const float idxf = -0.5f + 0.5f * sqrtf(1.f + 8.f * (d - dmin) / bin_size);
    int target = nb;
    if (idxf >= 0.f && idxf <= (float)nb && isfinite(idxf)) target = (int)idxf;
    // softmax over nb + 1 classes, 3 per lane (nb + 1 <= 96)
    const float* z = logits + (long long)b * sb + (long long)pix * sp;
    float zz[3], m = -INFINITY;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int c = lane + 32 * k;
        zz[k] = c <= nb ? z[(long long)c * sc] : -INFINITY;
        m = fmaxf(m, zz[k]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) s += (lane + 32 * k <= nb) ? expf(zz[k] - m) : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float logs = logf(s);
    const float wgt = fg ? fg_w : bg_w;
    float acc = 0.f, pk[3], fk[3];           // fk = t_c * f'(p_c) * p_c with f(p) = (1-p)^2 log p
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int c = lane + 32 * k;
        pk[k] = 0.f; fk[k] = 0.f;
        if (c <= nb) {
            const float lp = zz[k] - m - logs, pc = expf(lp), t = (c == target ? 1.f : 0.f) + 1e-6f, om = 1.f - pc;
            pk[k] = pc;
            acc += t * om * om * lp;
            fk[k] = t * (-2.f * om * pc * lp + om * om);
        }
    }
    if (!GRAD) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) pix_loss[warp] = -alpha * acc * wgt;
    } else {
        float fs = fk[0] + fk[1] + fk[2];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) fs += __shfl_xor_sync(0xffffffffu, fs, o);
        const float scale = -alpha * wgt * gw[0] / (float)npix;
        float* dz = dlogits + (long long)b * sb + (long long)pix * sp;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int c = lane + 32 * k;
            if (c <= nb) dz[(long long)c * sc] = scale * (fk[k] - pk[k] * fs);
        }
    }
}

// ---- per-layer losses -------------------------------------------------------------------------------------------------------
struct CritArgs {
    LayerPtrs logits, boxes, dim3, depth, angle;
    const int* labels; const float* boxes3d; const float* tdepth; const float* size3d; const int* hbin; const float* hres;
    const int* tlist; const int* count; const float* total; const int* match; const int* tclass;
    const float* pix_loss;
    int npix, B, Q, C, group, Gmax;
    float alpha, world;
};

constexpr int kThreads = 1024;

__device__ double block_sum(double v, double* red) {      // fixed order: deterministic
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    double t = 0.0;
    if (w == 0) {
        t = lane < (kThreads >> 5) ? red[lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) red[32] = t;
    }
    __syncthreads();
    return red[32];
}

__device__ __forceinline__ float num_boxes_of(const CritArgs& a) {
    return fmaxf(a.total[0] * (float)a.group / a.world, 1.f);      // monodetr.py:504-508 (`total` already summed over ranks)
}

struct PairTerms { float center, bbox, giou, depth, dim_abs, dim_rel, angle, correct; };

// matched pair `e` of layer l -> query / target rows; false if the slot is empty
__device__ __forceinline__ bool pair_of(const CritArgs& a, int l, int e, int& b, int& q, int& t) {
    const int j = e % a.Gmax;
    int r = e / a.Gmax;
    const int g = r % a.group;
    b = r / a.group;
    if (j >= a.count[b]) return false;
    q = a.match[(((size_t)l * a.B + b) * a.group + g) * a.Gmax + j];
    if (q < 0) return false;
    t = b * a.Gmax + a.tlist[b * a.Gmax + j];
    return true;
}

__global__ void __launch_bounds__(kThreads) crit_losses_kernel(CritArgs a, float* __restrict__ losses, float* __restrict__ aux) {
    __shared__ double red[33];
    __shared__ int card[1024];
    const int l = blockIdx.x, tid = threadIdx.x;
    const float nbx = num_boxes_of(a);
    const float* lg = a.logits.p[l];
    const int* tcl = a.tclass + (size_t)l * a.B * a.Q;
    // sigmoid focal loss over every (image, query, class)   dn_components.py:16-41, monodetr.py:337
    double ce = 0.0;
    for (int e = tid; e < a.B * a.Q * a.C; e += kThreads) {
        const int c = e % a.C, bq = e / a.C;
        const float x = lg[e], t = tcl[bq] == c ? 1.f : 0.f;
        const float prob = sigmoidf_(x);
        const float bce = fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
        const float pt = prob * t + (1.f - prob) * (1.f - t);
        const float at = a.alpha * t + (1.f - a.alpha) * (1.f - t);
        ce += (double)(at * bce * (1.f - pt) * (1.f - pt));
    }
    const double ce_sum = block_sum(ce, red);
    // cardinality error   monodetr.py:347-360 (argmax != last class, as written there)
    for (int i = tid; i < a.B; i += kThreads) card[i] = 0;
    __syncthreads();
    for (int bq = tid; bq < a.B * a.Q; bq += kThreads) {
        int am = 0;
        float best = lg[(size_t)bq * a.C];
        for (int c = 1; c < a.C; ++c) if (lg[(size_t)bq * a.C + c] > best) { best = lg[(size_t)bq * a.C + c]; am = c; }
        if (am != a.C - 1) atomicAdd(&card[bq / a.Q], 1);
    }
    __syncthreads();
    double cerr = 0.0;
    for (int i = tid; i < a.B; i += kThreads) cerr += fabs((double)card[i] - (double)a.count[i]);
    const double card_sum = block_sum(cerr, red);
    // matched pairs
    double s_center = 0, s_bbox = 0, s_giou = 0, s_depth = 0, s_dabs = 0, s_drel = 0, s_angle = 0, s_correct = 0, s_n = 0;
    const int npairs = a.B * a.group * a.Gmax;
    for (int e = tid; e < npairs; e += kThreads) {
        int b, q, t;
        if (!pair_of(a, l, e, b, q, t)) continue;
        const size_t bq = (size_t)b * a.Q + q;
        const float* sb = a.boxes.p[l] + bq * 6;
        const float* tb = a.boxes3d + (size_t)t * 6;
        s_center += (double)(fabsf(sb[0] - tb[0]) + fabsf(sb[1] - tb[1]));
        s_bbox += (double)(fabsf(sb[2] - tb[2]) + fabsf(sb[3] - tb[3]) + fabsf(sb[4] - tb[4]) + fabsf(sb[5] - tb[5]));
        float ax0, ay0, ax1, ay1, bx0, by0, bx1, by1;
        to_xyxy(sb, ax0, ay0, ax1, ay1);
        to_xyxy(tb, bx0, by0, bx1, by1);
        s_giou += (double)(1.f - giou_pair(ax0, ay0, ax1, ay1, bx0, by0, bx1, by1));
        const float* sd = a.depth.p[l] + bq * 2;
        s_depth += (double)(1.4142f * expf(-sd[1]) * fabsf(sd[0] - a.tdepth[t]) + sd[1]);       // monodetr.py:399-400
        const float* s3 = a.dim3.p[l] + bq * 3;
        const float* t3 = a.size3d + (size_t)t * 3;
        s_dabs += (double)(fabsf(s3[0] - t3[0]) + fabsf(s3[1] - t3[1]) + fabsf(s3[2] - t3[2]));   // == sum(|d|/t * comp), :411-418
        s_drel += (double)(fabsf(s3[0] - t3[0]) / t3[0] + fabsf(s3[1] - t3[1]) / t3[1] + fabsf(s3[2] - t3[2]) / t3[2]);
        const float* an = a.angle.p[l] + bq * (2 * kBins);
        const int hb = a.hbin[t];
        float m = an[0];
        for (int k = 1; k < kBins; ++k) m = fmaxf(m, an[k]);
        float se = 0.f;
        for (int k = 0; k < kBins; ++k) se += expf(an[k] - m);
        s_angle += (double)((m + logf(se) - an[hb]) + fabsf(an[kBins + hb] - a.hres[t]));        // :436-449
        int am = 0;
        float best = lg[bq * a.C];
        for (int c = 1; c < a.C; ++c) if (lg[bq * a.C + c] > best) { best = lg[bq * a.C + c]; am = c; }
        s_correct += (am == a.labels[t]) ? 1.0 : 0.0;
        s_n += 1.0;
    }
    const double r_center = block_sum(s_center, red), r_bbox = block_sum(s_bbox, red), r_giou = block_sum(s_giou, red);
    const double r_depth = block_sum(s_depth, red), r_dabs = block_sum(s_dabs, red), r_angle = block_sum(s_angle, red);
    const double r_correct = block_sum(s_correct, red), r_n = block_sum(s_n, red), r_drel = block_sum(s_drel, red);
    double dm = 0.0;
    if (l == 0 && a.pix_loss)
        for (int i = tid; i < a.npix; i += kThreads) dm += (double)a.pix_loss[i];
    const double r_dm = block_sum(dm, red);
    if (tid == 0) {
        float* o = losses + l * kNK;
        o[MDB_LOSS_CE] = (float)(ce_sum / nbx);
        o[MDB_LOSS_CLASS_ERROR] = r_n > 0 ? (float)(100.0 - 100.0 * r_correct / r_n) : 100.f;   // utils/misc.py:436-451
        o[MDB_LOSS_BBOX] = (float)(r_bbox / nbx);
        o[MDB_LOSS_GIOU] = (float)(r_giou / nbx);
        o[MDB_LOSS_CARDINALITY] = (float)(card_sum / a.B);
        o[MDB_LOSS_DEPTH] = (float)(r_depth / nbx);
        o[MDB_LOSS_DIM] = (float)(r_dabs / nbx);
        o[MDB_LOSS_ANGLE] = (float)(r_angle / nbx);
        o[MDB_LOSS_CENTER] = (float)(r_center / nbx);
        o[MDB_LOSS_DEPTH_MAP] = (l == 0 && a.pix_loss) ? (float)(r_dm / a.npix) : 0.f;
        // compensation weight of the dimension loss (no gradient through it, :414-416) = mean|d| / mean(|d| / t): kept for backward
        aux[l] = (float)(r_dabs / r_drel);
    }
}

constexpr int kBwdThreads = 256, kBwdBlocks = 32;     // per decoder layer

__global__ void __launch_bounds__(kBwdThreads) crit_losses_bwd_kernel(CritArgs a, const float* __restrict__ gw, const float* __restrict__ aux,
                                                                      LayerGradPtrs dlogits, LayerGradPtrs dboxes, LayerGradPtrs ddim3,
                                                                      LayerGradPtrs ddepth, LayerGradPtrs dangle) {
    // Pass 1, one thread per (image, query): the focal gradient of its C logits and, for UNMATCHED queries (tclass == C), zeros
    // in the box / size / depth / heading rows.  Pass 2, one thread per matched pair: the complete rows of the matched query.
    // Every output element is written exactly once, so the blocks need no ordering.
    const int l = blockIdx.y;
    const int tid = blockIdx.x * kBwdThreads + threadIdx.x, nth = kBwdBlocks * kBwdThreads;
    const float inv_nb = 1.f / num_boxes_of(a);
    const float* g = gw + l * kNK;
    const float* lg = a.logits.p[l];
    const int* tcl = a.tclass + (size_t)l * a.B * a.Q;
    const int nbq = a.B * a.Q;
    const float gce = g[MDB_LOSS_CE] * inv_nb;
    for (int bq = tid; bq < nbq; bq += nth) {
        for (int c = 0; c < a.C; ++c) {
            const int e = bq * a.C + c;
            const float x = lg[e], t = tcl[bq] == c ? 1.f : 0.f;
            const float prob = sigmoidf_(x);
            const float bce = fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
            const float pt = prob * t + (1.f - prob) * (1.f - t);
            const float at = a.alpha * t + (1.f - a.alpha) * (1.f - t);
            const float om = 1.f - pt;
            dlogits.p[l][e] = gce * at * (om * om * (prob - t) - 2.f * bce * om * prob * (1.f - prob) * (2.f * t - 1.f));
        }
        if (tcl[bq] != a.C) continue;                               // matched queries are written by the pair loop below
        for (int k = 0; k < 6; ++k) dboxes.p[l][(size_t)bq * 6 + k] = 0.f;
        for (int k = 0; k < 3; ++k) ddim3.p[l][(size_t)bq * 3 + k] = 0.f;
        for (int k = 0; k < 2; ++k) ddepth.p[l][(size_t)bq * 2 + k] = 0.f;
        for (int k = 0; k < 2 * kBins; ++k) dangle.p[l][(size_t)bq * 2 * kBins + k] = 0.f;
    }
    const float comp = aux[l];
    const int npairs = a.B * a.group * a.Gmax;
    for (int e = tid; e < npairs; e += nth) {
        int b, q, t;
        if (!pair_of(a, l, e, b, q, t)) continue;
        const size_t bq = (size_t)b * a.Q + q;
        const float* sb = a.boxes.p[l] + bq * 6;
        const float* tb = a.boxes3d + (size_t)t * 6;
        float db[6];
        const float gc = g[MDB_LOSS_CENTER] * inv_nb, gb = g[MDB_LOSS_BBOX] * inv_nb;
        for (int k = 0; k < 6; ++k) {
            const float d = sb[k] - tb[k];
            db[k] = (k < 2 ? gc : gb) * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f));
        }
        {   // GIoU: d(1 - giou) wrt the predicted corners, then to (cx, cy, l, r, t, b)
            float x0, y0, x1, y1, X0, Y0, X1, Y1;
            to_xyxy(sb, x0, y0, x1, y1);
            to_xyxy(tb, X0, Y0, X1, Y1);
            const float w = x1 - x0, h = y1 - y0, area1 = w * h, area2 = (X1 - X0) * (Y1 - Y0);
            const float iwr = fminf(x1, X1) - fmaxf(x0, X0), ihr = fminf(y1, Y1) - fmaxf(y0, Y0);
            const float iw = fmaxf(iwr, 0.f), ih = fmaxf(ihr, 0.f), inter = iw * ih, uni = area1 + area2 - inter;
            const float cwr = fmaxf(x1, X1) - fminf(x0, X0), chr = fmaxf(y1, Y1) - fminf(y0, Y0);
            const float cw = fmaxf(cwr, 0.f), ch = fmaxf(chr, 0.f), areac = cw * ch;
            // partial derivatives of inter / area1 / areac wrt x0 y0 x1 y1
            const float liv = iwr >= 0.f ? 1.f : 0.f, lih = ihr >= 0.f ? 1.f : 0.f, lcv = cwr >= 0.f ? 1.f : 0.f, lch = chr >= 0.f ? 1.f : 0.f;
            const float di[4] = {x0 > X0 ? -ih * liv : (x0 == X0 ? -0.5f * ih * liv : 0.f), y0 > Y0 ? -iw * lih : (y0 == Y0 ? -0.5f * iw * lih : 0.f),
                                 x1 < X1 ? ih * liv : (x1 == X1 ? 0.5f * ih * liv : 0.f), y1 < Y1 ? iw * lih : (y1 == Y1 ? 0.5f * iw * lih : 0.f)};
            const float da[4] = {-h, -w, h, w};
            const float dc[4] = {x0 < X0 ? -ch * lcv : (x0 == X0 ? -0.5f * ch * lcv : 0.f), y0 < Y0 ? -cw * lch : (y0 == Y0 ? -0.5f * cw * lch : 0.f),
                                 x1 > X1 ? ch * lcv : (x1 == X1 ? 0.5f * ch * lcv : 0.f), y1 > Y1 ? cw * lch : (y1 == Y1 ? 0.5f * cw * lch : 0.f)};
            const float gg = -g[MDB_LOSS_GIOU] * inv_nb;
            float dx[4];
            for (int k = 0; k < 4; ++k) {
                const float du = da[k] - di[k];
                const float dgiou = (di[k] * uni - inter * du) / (uni * uni) + (du * areac - uni * dc[k]) / (areac * areac);
                dx[k] = gg * dgiou;
            }
            db[0] += dx[0] + dx[2]; db[2] += -dx[0]; db[3] += dx[2];
            db[1] += dx[1] + dx[3]; db[4] += -dx[1]; db[5] += dx[3];
        }
        for (int k = 0; k < 6; ++k) dboxes.p[l][bq * 6 + k] = db[k];
        const float* sd = a.depth.p[l] + bq * 2;
        const float gd = g[MDB_LOSS_DEPTH] * inv_nb, dd = sd[0] - a.tdepth[t], ev = 1.4142f * expf(-sd[1]);
        ddepth.p[l][bq * 2 + 0] = gd * ev * (dd > 0.f ? 1.f : (dd < 0.f ? -1.f : 0.f));
        ddepth.p[l][bq * 2 + 1] = gd * (1.f - ev * fabsf(dd));
        const float* s3 = a.dim3.p[l] + bq * 3;
        const float* t3 = a.size3d + (size_t)t * 3;
        const float gdim = g[MDB_LOSS_DIM] * inv_nb * comp;
        for (int k = 0; k < 3; ++k) {
            const float d = s3[k] - t3[k];
            ddim3.p[l][bq * 3 + k] = gdim * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) / t3[k];
        }
        const float* an = a.angle.p[l] + bq * (2 * kBins);
        const int hb = a.hbin[t];
        const float ga = g[MDB_LOSS_ANGLE] * inv_nb;
        float m = an[0];
        for (int k = 1; k < kBins; ++k) m = fmaxf(m, an[k]);
        float se = 0.f;
        for (int k = 0; k < kBins; ++k) se += expf(an[k] - m);
        for (int k = 0; k < kBins; ++k) dangle.p[l][bq * 2 * kBins + k] = ga * (expf(an[k] - m) / se - (k == hb ? 1.f : 0.f));
        const float dr = an[kBins + hb] - a.hres[t];
        for (int k = 0; k < kBins; ++k)
            dangle.p[l][bq * 2 * kBins + kBins + k] = k == hb ? ga * (dr > 0.f ? 1.f : (dr < 0.f ? -1.f : 0.f)) : 0.f;
    }
}

int check_common(int L, int B, int Q, int C, int group, int Gmax) {
    if (L <= 0 || L > kMaxL || B <= 0 || Q <= 0 || C <= 0 || group <= 0 || Gmax <= 0 || Q % group) return MDB_EINVAL;
    if (Q / group > kMaxQueries || Gmax > kMaxTargets || B > 1024) return MDB_EUNSUPPORTED;
    return 0;
}

}  // namespace

extern "C" int mdb_criterion_prepare(const unsigned char* mask, int B, int Gmax, int* tlist, int* count, float* total, void* stream) {
    if (!mask || !tlist || !count || !total || B <= 0 || Gmax <= 0) return MDB_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(total, 0, sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    crit_prepare_kernel<<<B, 32, 0, st>>>(mask, Gmax, tlist, count, total);
    return (int)cudaGetLastError();
}

extern "C" int mdb_criterion_match_f32(int L, const float* const* logits, const float* const* boxes, const int* labels, const float* boxes3d,
                                       const int* tlist, const int* count, int B, int Q, int C, int group, int Gmax, float w_class,
                                       float w_center, float w_bbox, float w_giou, int* match, int* tclass, void* stream) {
    if (int rc = check_common(L, B, Q, C, group, Gmax)) return rc;
    if (!logits || !boxes || !labels || !boxes3d || !tlist || !count || !match || !tclass) return MDB_EINVAL;
    LayerPtrs lp{}, bp{};
    for (int l = 0; l < L; ++l) {
        if (!logits[l] || !boxes[l]) return MDB_EINVAL;
        lp.p[l] = logits[l]; bp.p[l] = boxes[l];
    }
    if (cudaError_t e = mdb::set_max_dynamic_smem(crit_match_kernel, kMatchMaxSmem)) return (int)e;
    crit_match_kernel<<<L * B * group, 32, match_smem_bytes(Q / group, Gmax), (cudaStream_t)stream>>>(
        lp, bp, labels, boxes3d, tlist, count, B, Q, C, group, Gmax, w_class, w_center, w_bbox, w_giou, match, tclass);
    return (int)cudaGetLastError();
}

extern "C" int mdb_criterion_depth_map_f32(const float* logits, long long stride_b, long long stride_pix, long long stride_c, const float* boxes2d,
                                           const float* depth, const int* tlist, const int* count, int B, int H, int W, int num_bins, int Gmax,
                                           float scale_x, float scale_y, float depth_min, float depth_max, float alpha, float fg_weight,
                                           float bg_weight, float* pix_loss, const float* grad_loss, float* dlogits, void* stream) {
    if (!logits || !boxes2d || !depth || !tlist || !count || B <= 0 || H <= 0 || W <= 0 || Gmax <= 0) return MDB_EINVAL;
    if (num_bins <= 0 || num_bins + 1 > 96) return MDB_EUNSUPPORTED;
    const bool grad = dlogits != nullptr;
    if (grad ? !grad_loss : !pix_loss) return MDB_EINVAL;
    const long long npix = (long long)B * H * W;
    if (npix > (1ll << 26)) return MDB_EUNSUPPORTED;
    const int blocks = (int)((npix * 32 + 255) / 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (grad)
        crit_depth_map_kernel<true><<<blocks, 256, 0, st>>>(logits, stride_b, stride_pix, stride_c, boxes2d, depth, tlist, count, B, H, W, num_bins,
                                                            Gmax, scale_x, scale_y, depth_min, depth_max, alpha, fg_weight, bg_weight, nullptr,
                                                            grad_loss, dlogits);
    else
        crit_depth_map_kernel<false><<<blocks, 256, 0, st>>>(logits, stride_b, stride_pix, stride_c, boxes2d, depth, tlist, count, B, H, W, num_bins,
                                                             Gmax, scale_x, scale_y, depth_min, depth_max, alpha, fg_weight, bg_weight, pix_loss,
                                                             nullptr, nullptr);
    return (int)cudaGetLastError();
}

static int fill_args(CritArgs& a, int L, const float* const* logits, const float* const* boxes, const float* const* dim3, const float* const* depth,
                     const float* const* angle, const int* labels, const float* boxes3d, const float* tdepth, const float* size3d,
                     const int* hbin, const float* hres, const int* tlist, const int* count, const float* total, const int* match,
                     const int* tclass, const float* pix_loss, int npix, int B, int Q, int C, int group, int Gmax, float alpha, float world) {
    if (int rc = check_common(L, B, Q, C, group, Gmax)) return rc;
    if (!logits || !boxes || !dim3 || !depth || !angle || !labels || !boxes3d || !tdepth || !size3d || !hbin || !hres || !tlist || !count ||
        !total || !match || !tclass || !(world > 0.f))
        return MDB_EINVAL;
    for (int l = 0; l < L; ++l) {
        if (!logits[l] || !boxes[l] || !dim3[l] || !depth[l] || !angle[l]) return MDB_EINVAL;
        a.logits.p[l] = logits[l]; a.boxes.p[l] = boxes[l]; a.dim3.p[l] = dim3[l]; a.depth.p[l] = depth[l]; a.angle.p[l] = angle[l];
    }
    a.labels = labels; a.boxes3d = boxes3d; a.tdepth = tdepth; a.size3d = size3d; a.hbin = hbin; a.hres = hres;
    a.tlist = tlist; a.count = count; a.total = total; a.match = match; a.tclass = tclass; a.pix_loss = pix_loss; a.npix = npix;
    a.B = B; a.Q = Q; a.C = C; a.group = group; a.Gmax = Gmax; a.alpha = alpha; a.world = world;
    return 0;
}

extern "C" int mdb_criterion_losses_f32(int L, const float* const* logits, const float* const* boxes, const float* const* dim3,
                                        const float* const* depth, const float* const* angle, const int* labels, const float* boxes3d,
                                        const float* tdepth, const float* size3d, const int* hbin, const float* hres, const int* tlist,
                                        const int* count, const float* total, const int* match, const int* tclass, const float* pix_loss, int npix,
                                        int B, int Q, int C, int group, int Gmax, float focal_alpha, float world_size, float* losses, float* aux,
                                        void* stream) {
    CritArgs a{};
    if (int rc = fill_args(a, L, logits, boxes, dim3, depth, angle, labels, boxes3d, tdepth, size3d, hbin, hres, tlist, count, total, match, tclass,
                           pix_loss, npix, B, Q, C, group, Gmax, focal_alpha, world_size))
        return rc;
    if (!losses || !aux) return MDB_EINVAL;
    crit_losses_kernel<<<L, kThreads, 0, (cudaStream_t)stream>>>(a, losses, aux);
    return (int)cudaGetLastError();
}

extern "C" int mdb_criterion_losses_backward_f32(int L, const float* const* logits, const float* const* boxes, const float* const* dim3,
                                                 const float* const* depth, const float* const* angle, const int* labels, const float* boxes3d,
                                                 const float* tdepth, const float* size3d, const int* hbin, const float* hres, const int* tlist,
                                                 const int* count, const float* total, const int* match, const int* tclass, int B, int Q, int C,
                                                 int group, int Gmax, float focal_alpha, float world_size, const float* grad_losses,
                                                 const float* aux, float* const* dlogits, float* const* dboxes, float* const* ddim3, float* const* ddepth,
                                                 float* const* dangle, void* stream) {
    CritArgs a{};
    if (int rc = fill_args(a, L, logits, boxes, dim3, depth, angle, labels, boxes3d, tdepth, size3d, hbin, hres, tlist, count, total, match, tclass,
                           nullptr, 0, B, Q, C, group, Gmax, focal_alpha, world_size))
        return rc;
    if (!grad_losses || !aux || !dlogits || !dboxes || !ddim3 || !ddepth || !dangle) return MDB_EINVAL;
    LayerGradPtrs gl{}, gb{}, g3{}, gd{}, ga{};
    for (int l = 0; l < L; ++l) {
        if (!dlogits[l] || !dboxes[l] || !ddim3[l] || !ddepth[l] || !dangle[l]) return MDB_EINVAL;
        gl.p[l] = dlogits[l]; gb.p[l] = dboxes[l]; g3.p[l] = ddim3[l]; gd.p[l] = ddepth[l]; ga.p[l] = dangle[l];
    }
    const ::dim3 grid(kBwdBlocks, L);        // (the parameter `dim3` shadows the type here)
    crit_losses_bwd_kernel<<<grid, kBwdThreads, 0, (cudaStream_t)stream>>>(a, grad_losses, aux, gl, gb, g3, gd, ga);
    return (int)cudaGetLastError();
}
