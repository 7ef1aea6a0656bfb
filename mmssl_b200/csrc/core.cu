// Error reporting, ABI version and device check for libmmssl_b200.so.
#include <stdlib.h>

#include "common.cuh"
#include "../../include/mmssl_b200.h"

namespace mmssl {
static thread_local char g_err[512] = "";
char* last_error_buffer() { return g_err; }
int fail(const char* where, const char* what) {
    snprintf(g_err, sizeof(g_err), "%s: %s", where, what);
    return 1;
}
bool pdl_enabled() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("MMSSL_PDL"); v = (e == nullptr || e[0] != '0') ? 1 : 0; }
    return v == 1;
}
int fail_cuda(const char* where, cudaError_t e) {
    snprintf(g_err, sizeof(g_err), "%s: CUDA error %d (%s)", where, (int)e, cudaGetErrorString(e));
    return 2;
}
}  // namespace mmssl

extern "C" int mmssl_abi_version(void) { return MMSSL_ABI_VERSION; }
extern "C" const char* mmssl_last_error(void) { return mmssl::last_error_buffer(); }
extern "C" int mmssl_device_check(void) {
    int dev = 0;
    MMSSL_CUDA(cudaGetDevice(&dev));
    int major = 0;
    MMSSL_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    MMSSL_REQUIRE(major == 9, "libmmssl_b200 is built for sm_90a (H100) only; no other device and no CPU fallback");
    return 0;
}
