// Library-level entry points: version, error string, device info.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace mub {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    // thread-local cache keyed by device id: no global mutable state shared across threads
    static thread_local int cached_dev = -1, cached_sms = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = 132;
        cached_dev = dev;
        cached_sms = n;
    }
    return cached_sms;
}

}  // namespace mub

extern "C" {

int mub_version(void) { return 109; /* 0.1.9: scOpen imputation (scopen) */ }

const char* mub_last_error(void) { return mub::g_err; }

int mub_device_info(int* sm_count, int* cc_major, int* cc_minor, int64_t* l2_bytes) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        mub::set_error("cudaGetDevice: %s", cudaGetErrorString(e));
        return -2;
    }
    int v = 0;
    if (sm_count) {
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        *sm_count = v;
    }
    if (cc_major) {
        cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev);
        *cc_major = v;
    }
    if (cc_minor) {
        cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev);
        *cc_minor = v;
    }
    if (l2_bytes) {
        cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev);
        *l2_bytes = v;
    }
    return 0;
}

}  // extern "C"
