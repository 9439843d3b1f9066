// C ABI of libddsp_b200.so - the library-wide entry points and the thread-local
// error and launch-count state.  Each kernel family's entry points (argument
// validation + kernel launches) live in its own unit: harmonic.cu, noise.cu,
// oscillators.cu, effects.cu, features.cu and losses.cu.  See
// include/ddsp_b200.h for the contract and the reference file:line each entry
// point replaces.
#include <stdarg.h>

#include "common.cuh"

namespace ddsp {

static thread_local char g_err[512] = "";
static thread_local uint64_t g_launches = 0;

void count_launch() { ++g_launches; }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

}  // namespace ddsp

using namespace ddsp;

extern "C" {

int ddsp_b200_version(void) { return DDSP_B200_VERSION; }

const char* ddsp_b200_last_error(void) { return g_err; }

uint64_t ddsp_b200_launch_count(void) { return g_launches; }

}  // extern "C"
