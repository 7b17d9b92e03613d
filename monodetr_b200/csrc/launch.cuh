// launch.cuh -- host-side launch helpers shared by every kernel launcher of the library (definitions in capi.cu).
#pragma once
#include <cuda_runtime.h>

namespace mdb {

// Multiprocessor count of the current device, queried once per device.
int num_sms();

// Blocks of a grid-stride kernel: ceil(n / threads), at most `cap`, at least 1.
inline int grid_cap(long long n, int threads, int cap) {
    long long b = (n + threads - 1) / threads;
    if (b > cap) b = cap;
    return b < 1 ? 1 : (int)b;
}

// Sets cudaFuncAttributeMaxDynamicSharedMemorySize of `func` to `bytes` on the current device, once per (function, device).
// Safe to call from several host threads at once.
cudaError_t set_max_dynamic_smem(const void* func, int bytes);

template <typename Kernel>
cudaError_t set_max_dynamic_smem(Kernel* func, int bytes) {
    return set_max_dynamic_smem(reinterpret_cast<const void*>(func), bytes);
}

}  // namespace mdb
