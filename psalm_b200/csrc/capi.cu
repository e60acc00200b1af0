// C-ABI plumbing shared by all kernels: error string, version, arch.
#include "common.cuh"

namespace psalm {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace psalm

extern "C" int psalm_abi_version(void) { return PSALM_ABI_VERSION; }
extern "C" const char* psalm_last_error(void) { return psalm::g_err; }
extern "C" int psalm_compiled_arch(void) { return 90; }
