// Host-side plumbing shared by all entry points: last-error string, version, parameter count.
#include <stdarg.h>
#include <string.h>
#include "common.cuh"

namespace promp {
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return PROMP_OK;
    set_error("CUDA error in %s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
    return PROMP_ERR_CUDA;
}
}  // namespace promp

extern "C" const char* promp_last_error(void) { return promp::g_err; }
extern "C" int promp_version(void) { return 100; }
extern "C" int promp_num_params(int obs_dim, int act_dim, int hidden) {
    // the activations do not change the layout: (32 | 64) with PROMP_ACT_RELU and / or PROMP_OUT_TANH count as their width
    const int width = hidden & PROMP_HIDDEN_WIDTH_MASK, flags = hidden & ~PROMP_HIDDEN_WIDTH_MASK;
    if ((width == 32 || width == 64) && flags != 0 && (flags & ~(PROMP_ACT_RELU | PROMP_OUT_TANH)) == 0) hidden = width;
    return promp::num_params(obs_dim, act_dim, hidden);
}
