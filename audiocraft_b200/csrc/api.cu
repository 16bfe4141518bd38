// Library-wide pieces of the C-ABI: error string, version, device query.
#include "common.cuh"
#include <stdarg.h>
#include <stdio.h>

static thread_local char g_err[512] = "";

void acb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* acb_last_error(void) { return g_err; }
extern "C" int acb_version(void) { return 104; }

extern "C" int acb_device_sm_count(int device) {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    return sms;
}
