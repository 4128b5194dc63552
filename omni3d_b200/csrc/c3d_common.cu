#include <stdarg.h>
#include <string.h>
#include "c3d_common.cuh"

namespace c3d {
static thread_local char g_err[512] = "";
char* last_error_buf() { return g_err; }
int32_t set_error(int32_t code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
}  // namespace c3d

extern "C" const char* c3d_last_error(void) { return c3d::last_error_buf(); }
extern "C" int32_t c3d_abi_version(void) { return 4; }
