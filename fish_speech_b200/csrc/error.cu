// Last-error storage for the C-ABI (one message per host thread).
#include <stdarg.h>

#include "common.cuh"

namespace fsb {

static thread_local char g_err[1024] = {0};
thread_local int g_launch_count = 0;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* get_error() { return g_err; }

}  // namespace fsb
