// api.cu -- version / error plumbing of the C ABI, and "not built yet" tensor-core entry points.
#include <stdarg.h>
#include "common.cuh"

static thread_local char g_err[512] = "";

void dz_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" int dz_version(void) { return 100; }                 // 0.1.0
extern "C" int dz_sm_arch(void) { return 90; }
extern "C" const char* dz_last_error_string(void) { return g_err; }
