// Helpers of the extern "C" entry points (include/mincurv_b200.h), which every kernel file defines beside the kernels
// they launch.  Errors go to one message buffer per thread for the whole library; mc_last_error (capi.cu) returns it.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <cuda_runtime.h>

#include "../../include/mincurv_b200.h"

namespace mc {
extern thread_local char g_err[256];
}

static inline int check_cuda(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        snprintf(mc::g_err, sizeof(mc::g_err), "%s: %s", what, cudaGetErrorString(e));
        return MC_ECUDA;
    }
    return MC_OK;
}
__attribute__((format(printf, 1, 2))) static inline int bad(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(mc::g_err, sizeof(mc::g_err), fmt, ap);
    va_end(ap);
    return MC_EINVAL;
}
static inline int small_workspace(const char *who) {
    snprintf(mc::g_err, sizeof(mc::g_err), "%s: workspace too small", who);
    return MC_EWORKSPACE;
}
static inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
