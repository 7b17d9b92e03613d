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
