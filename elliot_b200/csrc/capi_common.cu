// capi_common.cu — error reporting and device queries for the C ABI.
#include <stdarg.h>

#include "common.cuh"

namespace eb {

thread_local char g_err[512] = "";

int set_err(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (!cached[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

}  // namespace eb

extern "C" const char *eb_last_error(void) { return eb::g_err; }

extern "C" int eb_version(void) { return 100; }

extern "C" int eb_device_info(int *sm_count, int *cc) {
    int dev = 0;
    EB_CUDA(cudaGetDevice(&dev));
    int n = 0, maj = 0, min = 0;
    EB_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    EB_CUDA(cudaDeviceGetAttribute(&maj, cudaDevAttrComputeCapabilityMajor, dev));
    EB_CUDA(cudaDeviceGetAttribute(&min, cudaDevAttrComputeCapabilityMinor, dev));
    if (sm_count) *sm_count = n;
    if (cc) *cc = maj * 10 + min;
    return EB_OK;
}
