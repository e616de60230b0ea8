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
    // a depth field (1..3 hidden layers, PROMP_HIDDEN_DEPTH) counts its layers; no depth bits = two
    const int width = hidden & PROMP_HIDDEN_WIDTH_MASK, flags = hidden & ~PROMP_HIDDEN_WIDTH_MASK;
    if ((width == 32 || width == 64) && flags != 0 &&
        (flags & ~(PROMP_ACT_RELU | PROMP_OUT_TANH | PROMP_HIDDEN_DEPTH_MASK)) == 0) {
        const int field = (hidden & PROMP_HIDDEN_DEPTH_MASK) >> PROMP_HIDDEN_DEPTH_SHIFT;
        if (field > 3) return -1;
        return promp::num_params(obs_dim, act_dim, width, field == 0 ? 2 : field);
    }
    if (hidden > 0 && (hidden & PROMP_HIDDEN_DEPTH_MASK) != 0) return -1;     // deep policies are built for width 32 or 64
    return promp::num_params(obs_dim, act_dim, hidden);
}
