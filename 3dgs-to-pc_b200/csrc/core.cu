// core.cu — version + thread-local error message for the C ABI.
#include <stdarg.h>
#include "common.cuh"

static thread_local char g_err[512] = "";

void g2pc_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" int g2pc_version(void) { return 113; }
extern "C" const char* g2pc_last_error(void) { return g_err; }
