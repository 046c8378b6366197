#include <stdarg.h>

#include "common.cuh"

namespace psa {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace psa

extern "C" {
int psa_version(void) { return 100; /* 0.1.0 */ }
const char* psa_last_error(void) { return psa::g_err; }
int psa_sm_arch(void) { return 90; }
}
