// Library-level entry points of libfsdet.so.
#include <stdarg.h>

#include "common.cuh"

namespace fsdet {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace fsdet

extern "C" int fsdet_version(void) { return 100; }  // 0.1.0
extern "C" const char* fsdet_last_error(void) { return fsdet::g_err; }
extern "C" int fsdet_compiled_arch(void) { return 90; }   // sm_90a
extern "C" int fsdet_num_sms(void) { return fsdet::kNumSMs; }
