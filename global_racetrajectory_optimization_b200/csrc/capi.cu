// The library's own state: its version and the per-thread error message every entry point writes (capi.cuh).  The
// entry points themselves are defined beside their kernels; include/mincurv_b200.h declares them all.
#include "capi.cuh"

thread_local char mc::g_err[256] = "";

extern "C" {

int mc_version(void) { return 100; }
const char *mc_last_error(void) { return mc::g_err; }

}  // extern "C"
