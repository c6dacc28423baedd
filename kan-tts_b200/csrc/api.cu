// Library-wide pieces of libkantts_b200.so (see include/kantts_b200.h): the error string and the library info.  Every other
// entry point is defined in the file that holds its kernels.
#include <stdarg.h>

#include "common.cuh"

namespace kt {

// thread-local: the ABI is re-entrant across forward / autograd threads
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* kt_last_error(void) { return g_err; }
extern "C" int kt_version(void) { return 9; }
extern "C" int kt_has_tc(void) { return 1; }

}  // namespace kt
