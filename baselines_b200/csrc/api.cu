// Error text and version of libb200rl; every other entry point of include/b200rl.h is defined in its kernel's file.
#include <stdarg.h>
#include <stdio.h>

#include "common.cuh"

namespace b200rl {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

}  // namespace b200rl

extern "C" const char* b200rl_last_error(void) { return b200rl::g_err; }
extern "C" int b200rl_version(void) { return 100; }
