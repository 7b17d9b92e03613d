// labels.cu -- the label half of the reference dataset's __getitem__ (lib/datasets/kitti/kitti_dataset.py:173-330) for a whole
// batch in one launch: one thread per (image, target slot) reads label line `slot` of its image from the device-resident label
// bank and writes the padded targets.  Each step runs at the precision numpy 2 gives it in the reference (see the header and
// oracle/labels.py): fp64 steps as explicit _rn operations, float32 steps as float _rn intrinsics, so that nvcc contracts nothing
// the reference does not, and every value is rounded to float32 where the reference stores it into a float32 array.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"

namespace {

constexpr double kPi = 3.141592653589793;        // np.pi
constexpr int kHeadingBins = 12;                 // lib/datasets/utils.py num_heading_bin

struct LabelParams {
    double mean_size[9];
    int class_mask, clip_2d, depth_scale, max_objs;
    double res_w, res_h;
};

// Object3d.get_obj_level() == 'UnKnown' (kitti_utils.py:33-51): the height in fp64 from the float32 box
__device__ __forceinline__ bool level_unknown(float y1, float y2, double trunc, double occ) {
    const double height = __dadd_rn(__dsub_rn((double)y2, (double)y1), 1.0);
    if (trunc == -1.0) return false;
    if (height >= 40.0 && trunc <= 0.15 && occ <= 0.0) return false;
    if (height >= 25.0 && trunc <= 0.3 && occ <= 1.0) return false;
    return !(height >= 25.0 && trunc <= 0.5 && occ <= 2.0);
}

// affine_transform(): the point passes through a float32 array, the 2x3 product is fp64, summed left to right
__device__ __forceinline__ double affine_x(const double* t, float x, float y) {
    return __dadd_rn(__dadd_rn(__dmul_rn(t[0], (double)x), __dmul_rn(t[1], (double)y)), t[2]);
}
__device__ __forceinline__ double affine_y(const double* t, float x, float y) {
    return __dadd_rn(__dadd_rn(__dmul_rn(t[3], (double)x), __dmul_rn(t[4], (double)y)), t[5]);
}

// numpy's float32 `%` (npy_divmodf): fmod, then moved into the divisor's sign
__device__ __forceinline__ float mod_f32(float a, float b) {
    float m = fmodf(a, b);
    if (m != 0.f && ((m < 0.f) != (b < 0.f))) m = __fadd_rn(m, b);
    return m;
}

__global__ void __launch_bounds__(128) encode_targets_kernel(const long long* __restrict__ obj_off, const double* __restrict__ objects,
                                                             const float* __restrict__ P2s, int n_bank,
                                                             const mdb_label_image* __restrict__ images, int B, LabelParams cfg,
                                                             float* __restrict__ calibs, long long* __restrict__ indices,
                                                             signed char* __restrict__ labels, float* __restrict__ boxes,
                                                             float* __restrict__ boxes_3d, float* __restrict__ depth,
                                                             float* __restrict__ size_2d, float* __restrict__ size_3d,
                                                             float* __restrict__ src_size_3d, long long* __restrict__ heading_bin,
                                                             float* __restrict__ heading_res, unsigned char* __restrict__ mask_2d) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)B * cfg.max_objs) return;
    const int b = (int)(t / cfg.max_objs), slot = (int)(t % cfg.max_objs);

    // everything the slot holds when the reference leaves it untouched
    signed char lab = 0;
    bool mask = false;
    float s2d[2] = {0.f, 0.f}, bx[4] = {0.f, 0.f, 0.f, 0.f}, b3d[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float dep = 0.f, s3d[3] = {0.f, 0.f, 0.f}, src3d[3] = {0.f, 0.f, 0.f}, hres = 0.f;
    long long hbin = 0;
    const float* P2 = nullptr;
    bool kept = false;                                  // every target of the slot written, calibs included

    const mdb_label_image im = images[b];
    const int k = im.bank_index;
    const double* o = nullptr;
    if (k >= 0 && k < n_bank && slot < obj_off[k + 1] - obj_off[k]) o = objects + (obj_off[k] + slot) * MDB_LABEL_RECORD_WIDTH;
    do {
        if (!o) break;
        const int cls = (int)o[MDB_LABEL_CLS];
        if (cls < 0 || cls > 2 || !((cfg.class_mask >> cls) & 1)) break;                          // writelist
        const double trunc = o[MDB_LABEL_TRUNC], occ = o[MDB_LABEL_OCC];
        float x1 = (float)o[MDB_LABEL_BOX2D], y1 = (float)o[MDB_LABEL_BOX2D + 1];
        float x2 = (float)o[MDB_LABEL_BOX2D + 2], y2 = (float)o[MDB_LABEL_BOX2D + 3];
        const float pz = (float)o[MDB_LABEL_POS + 2];
        if (level_unknown(y1, y2, trunc, occ) || pz < 2.f || pz > 65.f) break;
        const double W_img = (double)im.img_w;
        double ry = o[MDB_LABEL_RY];
        if (im.flip) {                                                                              // :178-191
            const float nx1 = __double2float_rn(__dsub_rn(W_img, (double)x2));
            x2 = __double2float_rn(__dsub_rn(W_img, (double)x1));
            x1 = nx1;
            ry = __dsub_rn(kPi, ry);
            if (ry > kPi) ry = __dsub_rn(ry, 2.0 * kPi);
            if (ry < -kPi) ry = __dadd_rn(ry, 2.0 * kPi);
        }
        const float b0 = __double2float_rn(affine_x(im.trans, x1, y1)), b1 = __double2float_rn(affine_y(im.trans, x1, y1));
        const float b2 = __double2float_rn(affine_x(im.trans, x2, y2)), b3 = __double2float_rn(affine_y(im.trans, x2, y2));
        const float c2x = __fmul_rn(__fadd_rn(b0, b2), 0.5f), c2y = __fmul_rn(__fadd_rn(b1, b3), 0.5f);

        // projected 3-d centre: (pos + [0, -h/2, 0]) in fp64, rect_to_img divides the P2 rows by the rect z
        P2 = P2s + 12 * k;
        const double X = (double)(float)o[MDB_LABEL_POS], Y = __dadd_rn((double)(float)o[MDB_LABEL_POS + 1], -(o[MDB_LABEL_HWL] * 0.5));
        const double Z = (double)pz;
        double u = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)P2[0], X), __dmul_rn((double)P2[1], Y)), __dmul_rn((double)P2[2], Z)),
                             (double)P2[3]);
        double v = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)P2[4], X), __dmul_rn((double)P2[5], Y)), __dmul_rn((double)P2[6], Z)),
                             (double)P2[7]);
        u = __ddiv_rn(u, Z);
        v = __ddiv_rn(v, Z);
        if (im.flip) u = __dsub_rn(W_img, u);
        const float uf = __double2float_rn(u), vf = __double2float_rn(v);
        const double c3x = affine_x(im.trans, uf, vf), c3y = affine_y(im.trans, uf, vf);
        if (c3x < 0.0 || c3x >= cfg.res_w || c3y < 0.0 || c3y >= cfg.res_h) break;                   // :243-251

        lab = (signed char)cls;                                                                     // written before the l/r/t/b test
        const float w2 = __fsub_rn(b2, b0), h2 = __fsub_rn(b3, b1);
        s2d[0] = w2;
        s2d[1] = h2;
        const float cn0 = __double2float_rn(__ddiv_rn((double)b0, cfg.res_w)), cn1 = __double2float_rn(__ddiv_rn((double)b1, cfg.res_h));
        const float cn2 = __double2float_rn(__ddiv_rn((double)b2, cfg.res_w)), cn3 = __double2float_rn(__ddiv_rn((double)b3, cfg.res_h));
        const double c3nx = __ddiv_rn(c3x, cfg.res_w), c3ny = __ddiv_rn(c3y, cfg.res_h);
        double l = __dsub_rn(c3nx, (double)cn0), r = __dsub_rn((double)cn2, c3nx);
        double tt = __dsub_rn(c3ny, (double)cn1), bb = __dsub_rn((double)cn3, c3ny);
        if (l < 0.0 || r < 0.0 || tt < 0.0 || bb < 0.0) {
            if (!cfg.clip_2d) break;
            l = fmin(fmax(l, 0.0), 1.0);
            r = fmin(fmax(r, 0.0), 1.0);
            tt = fmin(fmax(tt, 0.0), 1.0);
            bb = fmin(fmax(bb, 0.0), 1.0);
        }
        bx[0] = __double2float_rn(__ddiv_rn((double)c2x, cfg.res_w));
        bx[1] = __double2float_rn(__ddiv_rn((double)c2y, cfg.res_h));
        bx[2] = __double2float_rn(__ddiv_rn((double)w2, cfg.res_w));
        bx[3] = __double2float_rn(__ddiv_rn((double)h2, cfg.res_h));
        b3d[0] = __double2float_rn(c3nx);
        b3d[1] = __double2float_rn(c3ny);
        b3d[2] = __double2float_rn(l);
        b3d[3] = __double2float_rn(r);
        b3d[4] = __double2float_rn(tt);
        b3d[5] = __double2float_rn(bb);
        dep = cfg.depth_scale == MDB_DEPTH_NORMAL    ? __double2float_rn(__dmul_rn((double)pz, im.crop_scale))
              : cfg.depth_scale == MDB_DEPTH_INVERSE ? __double2float_rn(__ddiv_rn((double)pz, im.crop_scale))
                                                     : pz;

        // ry2alpha on the flipped original box, then angle2class: float32 throughout (the Python floats are weak scalars)
        const float pi_f = (float)kPi, two_pi_f = (float)(2.0 * kPi);
        const float uc = __fmul_rn(__fadd_rn(x1, x2), 0.5f);
        const float at = __double2float_rn(atan2((double)__fsub_rn(uc, P2[2]), (double)P2[0]));
        float alpha = __fsub_rn(__double2float_rn(ry), at);
        for (int rep = 0; rep < 2; ++rep) {                                   // ry2alpha's range check, then :296-297 again
            if (alpha > pi_f) alpha = __fsub_rn(alpha, two_pi_f);
            if (alpha < -pi_f) alpha = __fadd_rn(alpha, two_pi_f);
        }
        const double apc = 2.0 * kPi / (double)kHeadingBins;
        const float a = mod_f32(alpha, two_pi_f);
        const float shifted = mod_f32(__fadd_rn(a, (float)(apc / 2.0)), two_pi_f);
        const int cid = (int)__fdiv_rn(shifted, (float)apc);
        hbin = cid;
        hres = __fsub_rn(shifted, __double2float_rn(__dadd_rn(__dmul_rn((double)cid, apc), apc / 2.0)));

#pragma unroll
        for (int j = 0; j < 3; ++j) {
            src3d[j] = (float)o[MDB_LABEL_HWL + j];
            s3d[j] = __double2float_rn(__dsub_rn((double)src3d[j], cfg.mean_size[3 * cls + j]));
        }
        mask = trunc <= 0.5 && occ <= 2.0;
        kept = true;
    } while (false);
    const long long s = t;
#pragma unroll
    for (int j = 0; j < 12; ++j) calibs[s * 12 + j] = kept ? P2[j] : 0.f;
    indices[s] = 0;
    labels[s] = lab;
#pragma unroll
    for (int j = 0; j < 4; ++j) boxes[s * 4 + j] = bx[j];
#pragma unroll
    for (int j = 0; j < 6; ++j) boxes_3d[s * 6 + j] = b3d[j];
    depth[s] = dep;
    size_2d[s * 2] = s2d[0];
    size_2d[s * 2 + 1] = s2d[1];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        size_3d[s * 3 + j] = s3d[j];
        src_size_3d[s * 3 + j] = src3d[j];
    }
    heading_bin[s] = hbin;
    heading_res[s] = hres;
    mask_2d[s] = mask ? 1 : 0;
}

}  // namespace

extern "C" int mdb_kitti_encode_targets(const long long* obj_off, const double* objects, const float* P2, int n_bank,
                                        const mdb_label_image* images, int B, const mdb_label_config* cfg, float* calibs,
                                        long long* indices, signed char* labels, float* boxes, float* boxes_3d, float* depth,
                                        float* size_2d, float* size_3d, float* src_size_3d, long long* heading_bin,
                                        float* heading_res, unsigned char* mask_2d, void* stream) {
    if (!obj_off || !objects || !P2 || !images || !cfg || !calibs || !indices || !labels || !boxes || !boxes_3d || !depth ||
        !size_2d || !size_3d || !src_size_3d || !heading_bin || !heading_res || !mask_2d)
        return MDB_EINVAL;
    if (B <= 0 || B > 65535 || n_bank < 1 || cfg->max_objs < 1 || cfg->max_objs > MDB_LABEL_MAX_OBJS || cfg->res_w <= 0 ||
        cfg->res_h <= 0 || cfg->depth_scale < MDB_DEPTH_NORMAL || cfg->depth_scale > MDB_DEPTH_NONE)
        return MDB_EINVAL;
    LabelParams p;
    for (int j = 0; j < 9; ++j) p.mean_size[j] = cfg->mean_size[j];
    p.class_mask = cfg->class_mask;
    p.clip_2d = cfg->clip_2d;
    p.depth_scale = cfg->depth_scale;
    p.max_objs = cfg->max_objs;
    p.res_w = (double)cfg->res_w;
    p.res_h = (double)cfg->res_h;
    const long long n = (long long)B * cfg->max_objs;
    encode_targets_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        obj_off, objects, P2, n_bank, images, B, p, calibs, indices, labels, boxes, boxes_3d, depth, size_2d, size_3d, src_size_3d,
        heading_bin, heading_res, mask_2d);
    return (int)cudaGetLastError();
}
