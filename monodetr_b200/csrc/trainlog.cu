// trainlog.cu -- the loss log of the training loop kept on the device.  The reference's trainer reads every weighted loss term
// with `.item()` on every step (lib/helpers/trainer_helper.py:145-152: 26 host synchronisations, printed or not).  Here the
// step appends the weighted terms to a ring in device memory; which record it writes is read from a device counter, so the
// launch can sit inside a captured CUDA graph, and the host copies a record out only for the steps it prints.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace {

__global__ void __launch_bounds__(256)
trainlog_push_kernel(const float* __restrict__ values, const float* __restrict__ weights, int n, float* ring, int slots, long long* counter) {
    float* rec = ring + (*counter % slots) * (long long)(n + 1);
    const int i = threadIdx.x;
    if (i < n) rec[i] = __fmul_rn(values[i], weights[i]);
    __syncthreads();                                   // every thread has read the counter and written its term
    if (i == 0) {
        float s = 0.f;
        for (int j = 0; j < n; ++j) s = __fadd_rn(s, rec[j]);
        rec[n] = s;
        *counter += 1;
    }
}

}  // namespace

extern "C" int mdb_trainlog_push_f32(const float* values, const float* weights, int n, float* ring, int slots, long long* counter,
                                     void* stream) {
    if (n < 1 || n > 255 || slots < 1) return MDB_EINVAL;
    if (!values || !weights || !ring || !counter || (reinterpret_cast<uintptr_t>(counter) & 7u)) return MDB_EINVAL;
    trainlog_push_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream)>>>(values, weights, n, ring, slots, counter);
    return (int)cudaGetLastError();
}
