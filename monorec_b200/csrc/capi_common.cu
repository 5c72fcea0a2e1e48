// libmonorec_b200.so -- error text, version, launch counter (include/monorec_b200.h).
#include "mr_common.cuh"
#include <cstring>

namespace mr {

static thread_local char g_err[512] = "";
static thread_local long long g_launches = 0;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void count_launch(int n) { g_launches += n; }

}  // namespace mr

extern "C" int mr_version(void) { return (0 << 16) | (3 << 8) | 0; }

extern "C" const char* mr_last_error(void) { return mr::g_err; }

extern "C" long long mr_launch_count(int reset) {
    long long v = mr::g_launches;
    if (reset) mr::g_launches = 0;
    return v;
}
