// capi.cu -- ABI version and error strings of libmonodetr_b200.so (see include/monodetr_b200.h), and the per-device state of
// the launch helpers (launch.cuh).
#include <cuda_runtime.h>

#include <map>
#include <mutex>
#include <utility>

#include "../../include/monodetr_b200.h"
#include "launch.cuh"

namespace mdb {

namespace {
std::mutex g_launch_mutex;    // several host threads may launch at once (nn.DataParallel)
}

int num_sms() {
    constexpr int kFallback = 132;    // H100 SXM, if the device cannot be queried
    static std::map<int, int> sms;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return kFallback;
    std::lock_guard<std::mutex> lock(g_launch_mutex);
    int& n = sms[dev];
    if (n == 0 && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = kFallback;
    return n;
}

cudaError_t set_max_dynamic_smem(const void* func, int bytes) {
    static std::map<std::pair<const void*, int>, int> configured;    // the attribute is per (function, device)
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(g_launch_mutex);
    int& done = configured[{func, dev}];
    if (done == bytes) return cudaSuccess;
    e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done = bytes;
    return e;
}

}  // namespace mdb

extern "C" {

int mdb_abi_version(void) { return 2; }

// Reproducible-accumulation mode (process-wide, like the arithmetic mode): read by the two large scatter / accumulate sites,
// the MSDeformAttn value gradient (msda.cu) and the split-K weight gradient (conv_gemm.cu).
static int g_deterministic = 0;
int mdb_set_deterministic(int on) { g_deterministic = on ? 1 : 0; return 0; }
int mdb_get_deterministic(void) { return g_deterministic; }

const char* mdb_error_string(int code) {
    if (code == 0) return "ok";
    if (code == MDB_EINVAL) return "monodetr_b200: invalid argument (size, null or misaligned pointer)";
    if (code == MDB_EUNSUPPORTED) return "monodetr_b200: shape not supported by the sm_90a kernels";
    if (code == MDB_EWORKSPACE) return "monodetr_b200: scratch workspace missing or too small (mdb_set_workspace)";
    if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
    return "monodetr_b200: unknown error";
}

}  // extern "C"
