// optim.cu -- fused AdamW step over the FLAT parameter / gradient buffers (SURVEY.md 8f-2): the update of
// lib/helpers/optimizer_helper.py:69-129 (the reference's own AdamW class, configs/monodetr.yaml `optimizer: adamw`) for all
// parameters in ONE HBM-bound pass instead of ~10 small torch kernels per tensor x 313 tensors.
//
// Per element, exactly the reference's operation sequence in fp32 (optimizer_helper.py:104-127):
//   m = m * beta1 + (1 - beta1) * g                       exp_avg.mul_(beta1).add_(1 - beta1, grad)
//   v = v * beta2 + (1 - beta2) * g * g                   exp_avg_sq.mul_(beta2).addcmul_(1 - beta2, grad, grad)
//   denom = sqrt(v) + eps
//   p = p - step_size * (p * wd + m / denom)              p.data.add_(-step_size, mul(p, wd).addcdiv_(1, exp_avg, denom))
// with step_size = lr * sqrt(1 - beta2^t) / (1 - beta1^t) (note the reference multiplies the weight-decay term by
// step_size, not by lr).  wd applies to the first `n_decay` elements of the flat layout (parameters without 'bias' in
// their name, optimizer_helper.py:9-16), 0 to the rest.  Each multiply-add that torch's kernels contract into an FMA is
// written as an explicit fmaf, every other operation is kept separate (__fmul_rn / __fadd_rn), so the result does not
// depend on nvcc's own contraction choices.
// Algorithmic bytes: 7 x 4 B per parameter (read p, g, m, v; write p, m, v).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

__device__ __forceinline__ void adamw1(float& p, float g, float& m, float& v, float b1, float omb1, float b2, float omb2, float eps,
                                       float wd, float neg_step) {
    m = fmaf(omb1, g, __fmul_rn(m, b1));
    v = fmaf(omb2, __fmul_rn(g, g), __fmul_rn(v, b2));        // addcmul_: self + value * (t1 * t2)
    const float denom = __fadd_rn(sqrtf(v), eps);
    const float upd = __fadd_rn(__fmul_rn(p, wd), __fdiv_rn(m, denom));
    p = fmaf(neg_step, upd, p);
}

__global__ void __launch_bounds__(256)
adamw_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
                  long long n_decay, float b1, float omb1, float b2, float omb2, float eps, float wd, float step_size,
                  const float* __restrict__ step_size_dev) {
    const float neg_step = -(step_size_dev ? *step_size_dev : step_size);
    const long long n4 = n / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 pp = reinterpret_cast<float4*>(p)[i], mm = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
        const float4 gg = reinterpret_cast<const float4*>(g)[i];
        const long long e = 4 * i;
        adamw1(pp.x, gg.x, mm.x, vv.x, b1, omb1, b2, omb2, eps, e < n_decay ? wd : 0.f, neg_step);
        adamw1(pp.y, gg.y, mm.y, vv.y, b1, omb1, b2, omb2, eps, e + 1 < n_decay ? wd : 0.f, neg_step);
        adamw1(pp.z, gg.z, mm.z, vv.z, b1, omb1, b2, omb2, eps, e + 2 < n_decay ? wd : 0.f, neg_step);
        adamw1(pp.w, gg.w, mm.w, vv.w, b1, omb1, b2, omb2, eps, e + 3 < n_decay ? wd : 0.f, neg_step);
        reinterpret_cast<float4*>(p)[i] = pp;
        reinterpret_cast<float4*>(m)[i] = mm;
        reinterpret_cast<float4*>(v)[i] = vv;
    }
    // tail (n not a multiple of 4)
    for (long long e = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
        adamw1(p[e], g[e], m[e], v[e], b1, omb1, b2, omb2, eps, e < n_decay ? wd : 0.f, neg_step);
}

// One thread: t += 1 and the bias-corrected step size of that t.  Every operation is a separately rounded fp64 operation in
// the order of the host expression lr * sqrt(1 - beta2 ** t) / (1 - beta1 ** t); the result is rounded to fp32 once.
__global__ void adamw_advance_kernel(MdbAdamwHyper* h) {
    const double t = h->t + 1.0;
    const double bc2 = __dsub_rn(1.0, pow(h->beta2, t));
    const double bc1 = __dsub_rn(1.0, pow(h->beta1, t));
    h->t = t;
    h->step_size = (float)__ddiv_rn(__dmul_rn(h->lr, sqrt(bc2)), bc1);
}

}  // namespace

extern "C" int mdb_adamw_advance(MdbAdamwHyper* hyper, void* stream) {
    if (!hyper || (reinterpret_cast<uintptr_t>(hyper) & 7u)) return MDB_EINVAL;
    adamw_advance_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(hyper);
    return (int)cudaGetLastError();
}

extern "C" int mdb_adamw_step_f32(float* p, const float* g, float* m, float* v, long long n, long long n_decay, float beta1,
                                  float one_minus_beta1, float beta2, float one_minus_beta2, float eps, float weight_decay,
                                  float step_size, const float* step_size_dev, void* stream) {
    if (n < 0 || n_decay < 0 || n_decay > n) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!p || !g || !m || !v) return MDB_EINVAL;
    if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15u)
        return MDB_EINVAL;
    const int blocks = mdb::grid_cap(n / 4, 256, mdb::num_sms() * 8);
    adamw_flat_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(p, g, m, v, n, n_decay, beta1, one_minus_beta1, beta2,
                                                                                       one_minus_beta2, eps, weight_decay, step_size,
                                                                                       step_size_dev);
    return (int)cudaGetLastError();
}

// ---- SGD with momentum and Adam: torch.optim.SGD / torch.optim.Adam, the reference's other two `optimizer.type` values
// (lib/helpers/optimizer_helper.py:17-20), over the same flat layout.  The reference runs them on CUDA tensors, so the per-element
// operation order is that of torch's multi-tensor (`foreach`) branch, with each contraction torch's kernels make written as an
// explicit fmaf.  Weight decay is the L2 term torch adds to the gradient (`_foreach_add(grads, params, alpha=wd)`); torch skips
// that launch at wd == 0, so does the select below (fmaf(0, p, g) would turn g = -0 into +0).
namespace {

// torch/optim/sgd.py _multi_tensor_sgd, dampening 0, no Nesterov:
//   d = g + wd * p                      _foreach_add(grads, params, alpha=wd)                 fmaf
//   buf = d  (first step)               momentum_buffer = d.clone()
//   buf = buf * momentum + d            _foreach_mul_(bufs, momentum); _foreach_add_(bufs, d)
//   p = p + (-lr) * buf                 _foreach_add_(params, bufs, alpha=-lr)                 fmaf
// Algorithmic bytes: 5 x 4 B per parameter (read p, g, buf; write p, buf).
__device__ __forceinline__ void sgd1(float& p, float g, float& buf, float mom, float wd, float neg_lr, bool first) {
    const float d = wd != 0.f ? fmaf(wd, p, g) : g;
    buf = first ? d : __fadd_rn(__fmul_rn(buf, mom), d);
    p = fmaf(neg_lr, buf, p);
}

__global__ void __launch_bounds__(256)
sgd_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, long long n, long long n_decay,
                float mom, float wd, float lr, int first_step, const MdbSgdHyper* __restrict__ hyper) {
    const float neg_lr = -(hyper ? (float)hyper->lr : lr);
    const bool first = hyper ? hyper->t == 1.0 : first_step != 0;
    const long long n4 = n / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 pp = reinterpret_cast<float4*>(p)[i];
        float4 bb = first ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<float4*>(buf)[i];   // not read on the first step
        const float4 gg = reinterpret_cast<const float4*>(g)[i];
        const long long e = 4 * i;
        sgd1(pp.x, gg.x, bb.x, mom, e < n_decay ? wd : 0.f, neg_lr, first);
        sgd1(pp.y, gg.y, bb.y, mom, e + 1 < n_decay ? wd : 0.f, neg_lr, first);
        sgd1(pp.z, gg.z, bb.z, mom, e + 2 < n_decay ? wd : 0.f, neg_lr, first);
        sgd1(pp.w, gg.w, bb.w, mom, e + 3 < n_decay ? wd : 0.f, neg_lr, first);
        reinterpret_cast<float4*>(p)[i] = pp;
        reinterpret_cast<float4*>(buf)[i] = bb;
    }
    for (long long e = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        float b = first ? 0.f : buf[e];
        sgd1(p[e], g[e], b, mom, e < n_decay ? wd : 0.f, neg_lr, first);
        buf[e] = b;
    }
}

// torch/optim/adam.py _multi_tensor_adam (capturable=False), no amsgrad:
//   g' = g + wd * p                     _foreach_add(grads, params, alpha=wd)                 fmaf
//   m = lerp(m, g', w), w = 1 - beta1   _foreach_lerp_ (ATen/native/Lerp.h):
//                                         |w| < 0.5: m + w * (g' - m)                         fmaf
//                                         else:      g' - (g' - m) * (1 - w)                  fmaf
//   v = v * beta2 + (1 - beta2) * g'g'  _foreach_mul_; _foreach_addcmul_ (DeviceAddCmulCdiv.cuh: fma(value, g'*g', v), or
//                                       fma(g', g', v) when value == 1)
//   s = sqrt(v) / sqrt(bc2) + eps       _foreach_sqrt; _foreach_div_(scalar list); _foreach_add_
//   p = p + neg_step * (m / s)          _foreach_addcdiv_(params, m, s, neg_step)              fmaf
// with neg_step = (lr / bc1) * -1, bc1 = 1 - beta1^t, bc2 = 1 - beta2^t, computed in fp64 and rounded to fp32 once.
// Algorithmic bytes: 7 x 4 B per parameter (read p, g, m, v; write p, m, v).
__device__ __forceinline__ void adam1(float& p, float g, float& m, float& v, float w, float omw, float b2, float omb2, float eps,
                                      float wd, float neg_step, float bc2_sqrt) {
    const float gd = wd != 0.f ? fmaf(wd, p, g) : g;
    const float diff = __fsub_rn(gd, m);
    m = fabsf(w) < 0.5f ? fmaf(w, diff, m) : fmaf(-diff, omw, gd);
    const float v2 = __fmul_rn(v, b2);
    v = omb2 == 1.f ? fmaf(gd, gd, v2) : fmaf(omb2, __fmul_rn(gd, gd), v2);
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), bc2_sqrt), eps);
    p = fmaf(neg_step, __fdiv_rn(m, denom), p);
}

__global__ void __launch_bounds__(256)
adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
                 long long n_decay, float w, float b2, float omb2, float eps, float wd, float neg_step, float bc2_sqrt,
                 const MdbAdamHyper* __restrict__ hyper) {
    if (hyper) {
        neg_step = hyper->neg_step;
        bc2_sqrt = hyper->bc2_sqrt;
    }
    const float omw = __fsub_rn(1.f, w);
    const long long n4 = n / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 pp = reinterpret_cast<float4*>(p)[i], mm = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
        const float4 gg = reinterpret_cast<const float4*>(g)[i];
        const long long e = 4 * i;
        adam1(pp.x, gg.x, mm.x, vv.x, w, omw, b2, omb2, eps, e < n_decay ? wd : 0.f, neg_step, bc2_sqrt);
        adam1(pp.y, gg.y, mm.y, vv.y, w, omw, b2, omb2, eps, e + 1 < n_decay ? wd : 0.f, neg_step, bc2_sqrt);
        adam1(pp.z, gg.z, mm.z, vv.z, w, omw, b2, omb2, eps, e + 2 < n_decay ? wd : 0.f, neg_step, bc2_sqrt);
        adam1(pp.w, gg.w, mm.w, vv.w, w, omw, b2, omb2, eps, e + 3 < n_decay ? wd : 0.f, neg_step, bc2_sqrt);
        reinterpret_cast<float4*>(p)[i] = pp;
        reinterpret_cast<float4*>(m)[i] = mm;
        reinterpret_cast<float4*>(v)[i] = vv;
    }
    for (long long e = n4 * 4 + blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
        adam1(p[e], g[e], m[e], v[e], w, omw, b2, omb2, eps, e < n_decay ? wd : 0.f, neg_step, bc2_sqrt);
}

__global__ void sgd_advance_kernel(MdbSgdHyper* h) { h->t = h->t + 1.0; }

// One thread: t += 1 and torch's two step scalars for that t, every operation a separately rounded fp64 operation in the order of
// adam.py's Python floats: bc1 = 1 - beta1 ** t; bc2 = 1 - beta2 ** t; step_size = (lr / bc1) * -1; bc2 ** 0.5 (a correctly
// rounded square root here).
__global__ void adam_advance_kernel(MdbAdamHyper* h) {
    const double t = h->t + 1.0;
    const double bc1 = __dsub_rn(1.0, pow(h->beta1, t));
    const double bc2 = __dsub_rn(1.0, pow(h->beta2, t));
    h->t = t;
    h->neg_step = (float)(-__ddiv_rn(h->lr, bc1));
    h->bc2_sqrt = (float)sqrt(bc2);
}

bool misaligned16(const void* a, const void* b, const void* c, const void* d) {
    return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
             reinterpret_cast<uintptr_t>(d)) & 15u) != 0;
}

}  // namespace

extern "C" int mdb_sgd_advance(MdbSgdHyper* hyper, void* stream) {
    if (!hyper || (reinterpret_cast<uintptr_t>(hyper) & 7u)) return MDB_EINVAL;
    sgd_advance_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(hyper);
    return (int)cudaGetLastError();
}

extern "C" int mdb_sgd_step_f32(float* p, const float* g, float* buf, long long n, long long n_decay, float momentum,
                                float weight_decay, float lr, int first_step, const MdbSgdHyper* hyper_dev, void* stream) {
    if (n < 0 || n_decay < 0 || n_decay > n) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!p || !g || !buf) return MDB_EINVAL;
    if (misaligned16(p, g, buf, buf) || (reinterpret_cast<uintptr_t>(hyper_dev) & 7u)) return MDB_EINVAL;
    const int blocks = mdb::grid_cap(n / 4, 256, mdb::num_sms() * 8);
    sgd_flat_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(p, g, buf, n, n_decay, momentum, weight_decay, lr,
                                                                           first_step, hyper_dev);
    return (int)cudaGetLastError();
}

extern "C" int mdb_adam_advance(MdbAdamHyper* hyper, void* stream) {
    if (!hyper || (reinterpret_cast<uintptr_t>(hyper) & 7u)) return MDB_EINVAL;
    adam_advance_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(hyper);
    return (int)cudaGetLastError();
}

extern "C" int mdb_adam_step_f32(float* p, const float* g, float* m, float* v, long long n, long long n_decay, float one_minus_beta1,
                                 float beta2, float one_minus_beta2, float eps, float weight_decay, float neg_step, float bc2_sqrt,
                                 const MdbAdamHyper* hyper_dev, void* stream) {
    if (n < 0 || n_decay < 0 || n_decay > n) return MDB_EINVAL;
    if (n == 0) return 0;
    if (!p || !g || !m || !v) return MDB_EINVAL;
    if (misaligned16(p, g, m, v) || (reinterpret_cast<uintptr_t>(hyper_dev) & 7u)) return MDB_EINVAL;
    const int blocks = mdb::grid_cap(n / 4, 256, mdb::num_sms() * 8);
    adam_flat_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(p, g, m, v, n, n_decay, one_minus_beta1, beta2,
                                                                            one_minus_beta2, eps, weight_decay, neg_step, bc2_sqrt,
                                                                            hyper_dev);
    return (int)cudaGetLastError();
}
