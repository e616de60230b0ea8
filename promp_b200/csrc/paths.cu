// Variable-length paths from fused early-termination rollouts (promp_rollout_early_term): the reference's sampling loop
// (samplers/meta_sampler.py:87-137) keeps stepping ALL envs until the COMPLETED paths hold >= M*E*H samples, appends a path
// to its task's list at the step it completes (env index order within a step) and drops unfinished ones.  The fused kernel
// has already stepped every env slot for a fixed timeline (>= 2H-1 steps always suffices: at step t every slot has at most
// H-1 samples in an unfinished path); these kernels apply the rule to the recorded `done` timelines, entirely on the device:
//   1. path_hist_kernel      hist[t] = samples of the paths completing at step t        (one thread per env slot)
//   2. path_cut_kernel       t* = first step with cumulative completed samples >= target (one CTA, scan)
//   3. path_table_kernel     per task: paths completing at steps <= t* in (step, env) order -> source (slot, start, length)
//                            and the prefix-sum table path_off / n_paths / n_valid      (one CTA per task, step-synchronous)
//   4. path_compact_kernel   timelines -> the ragged [M, Nmax] layout of promp_process_samples_ragged (one warp per path)
#include "common.cuh"

namespace promp {

__global__ void path_hist_kernel(int n_slots, int T, const uint8_t* __restrict__ done, int* __restrict__ hist) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    const uint8_t* d = done + (int64_t)s * T;
    int len = 0;
    for (int t = 0; t < T; ++t) {
        ++len;
        if (d[t]) {
            atomicAdd(hist + t, len);
            len = 0;
        }
    }
}

// cut[0] = t* (T-1 if the target is never reached), cut[1] = 1 if the target was reached.  clear == hist (the workspace
// histogram): all of hist[0..T-1] is cleared for the next call, including the chunks after the one that holds t*.
// clear == NULL (a caller's histogram, promp_paths_finalize_ex): hist is only read.
__global__ void __launch_bounds__(1024) path_cut_kernel(int T, int64_t target, const int* hist, int* clear, int* cut) {
    __shared__ long long s_carry;
    __shared__ int s_found;
    __shared__ long long s_scan[1024];
    const int tid = threadIdx.x;
    if (tid == 0) { s_carry = 0; s_found = -1; }
    __syncthreads();
    for (int t0 = 0; t0 < T; t0 += 1024) {
        const int t = t0 + tid;
        if (s_found >= 0) {                               // past the cut's chunk (s_found is block-uniform here): clear only
            if (!clear) break;
            if (t < T) clear[t] = 0;
            continue;
        }
        long long v = t < T ? hist[t] : 0;
        if (clear && t < T) clear[t] = 0;
        s_scan[tid] = v;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {          // Hillis-Steele inclusive scan
            const long long add = tid >= o ? s_scan[tid - o] : 0;
            __syncthreads();
            s_scan[tid] += add;
            __syncthreads();
        }
        const long long cum = s_carry + s_scan[tid];
        if (t < T && cum >= target && cum - v < target) s_found = t;      // exactly one thread: first crossing
        __syncthreads();
        if (tid == 0) s_carry += s_scan[1023];
        __syncthreads();
    }
    if (tid == 0) {
        cut[0] = s_found >= 0 ? s_found : T - 1;
        cut[1] = s_found >= 0 ? 1 : 0;
    }
}

// One CTA per task, thread e = env slot e (E <= 1024).  Walks the steps 0..t* together: at every step the finishing slots get
// consecutive path indices in env order (a block-wide exclusive scan), exactly the order of meta_sampler.py:116-125.
__global__ void __launch_bounds__(1024) path_table_kernel(int E, int T, int Pmax, const uint8_t* __restrict__ done,
                                                          const int* __restrict__ cut, int32_t* __restrict__ path_off,
                                                          int32_t* __restrict__ n_paths, int32_t* __restrict__ n_valid,
                                                          int32_t* __restrict__ src_slot, int32_t* __restrict__ src_start) {
    const int m = blockIdx.x, e = threadIdx.x, lane = e & 31, w = e >> 5;
    const int t_star = cut[0];
    __shared__ int s_wcnt[32], s_wlen[32];
    __shared__ int s_paths, s_samples, s_kept;        // s_kept: samples in the first Pmax paths, once a path Pmax-1 exists
    if (e == 0) { s_paths = 0; s_samples = 0; s_kept = 0; }
    __syncthreads();
    const uint8_t* d = done + ((int64_t)m * E + (e < E ? e : 0)) * T;
    int32_t* po = path_off + (int64_t)m * (Pmax + 1);
    int start = 0;
    for (int t = 0; t <= t_star; ++t) {
        const int fin = (e < E && d[t]) ? 1 : 0;
        const int len = fin ? t + 1 - start : 0;
        // block-wide exclusive scans of (fin, len)
        int c = fin, l = len;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int c2 = __shfl_up_sync(0xffffffffu, c, o), l2 = __shfl_up_sync(0xffffffffu, l, o);
            if (lane >= o) { c += c2; l += l2; }
        }
        if (lane == 31) { s_wcnt[w] = c; s_wlen[w] = l; }
        __syncthreads();
        int cb = 0, lb = 0, ctot = 0, ltot = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
            if (i < w) { cb += s_wcnt[i]; lb += s_wlen[i]; }
            ctot += s_wcnt[i];
            ltot += s_wlen[i];
        }
        if (fin) {
            const int k = s_paths + cb + c - 1;            // path index inside the task
            if (k < Pmax) {
                const int off = s_samples + lb + l - len;  // exclusive prefix of the lengths
                po[k] = off;
                src_slot[(int64_t)m * Pmax + k] = e;
                src_start[(int64_t)m * Pmax + k] = start;
                if (k == Pmax - 1) s_kept = off + len;
            }
            start = t + 1;
        }
        __syncthreads();
        if (e == 0) { s_paths += ctot; s_samples += ltot; }
        __syncthreads();
    }
    // more than Pmax paths: the table keeps the first Pmax of them, and the closing offset / n_valid count only those
    const int np = min(s_paths, Pmax);
    const int nv = s_paths > Pmax ? s_kept : s_samples;
    for (int k = np + e; k <= Pmax; k += blockDim.x) po[k] = nv;            // closing offset (and padding entries)
    if (e == 0) {
        n_paths[m] = np;
        n_valid[m] = nv;
    }
}

// One warp per (task, path): copies the path's samples from its slot's timeline into the ragged row of the task.
__global__ void __launch_bounds__(256) path_compact_kernel(int M, int E, int T, int Pmax, int Nmax, int Do, int Da,
                                                           const int32_t* __restrict__ path_off, const int32_t* __restrict__ n_paths,
                                                           const int32_t* __restrict__ src_slot, const int32_t* __restrict__ src_start,
                                                           const float* __restrict__ t_obs, const float* __restrict__ t_act,
                                                           const float* __restrict__ t_mean, const float* __restrict__ t_rew,
                                                           float* __restrict__ obs, float* __restrict__ act, float* __restrict__ mean,
                                                           float* __restrict__ rew, uint8_t* __restrict__ done) {
    const int m = blockIdx.y, lane = threadIdx.x & 31;
    const int np = n_paths[m];
    const int32_t* po = path_off + (int64_t)m * (Pmax + 1);
    for (int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < np; k += gridDim.x * (blockDim.x >> 5)) {
        const int off = po[k], len = po[k + 1] - off;
        const int64_t src = ((int64_t)m * E + src_slot[(int64_t)m * Pmax + k]) * T + src_start[(int64_t)m * Pmax + k];
        const int64_t dst = (int64_t)m * Nmax + off;
        for (int i = lane; i < len * Do; i += 32) obs[dst * Do + i] = t_obs[src * Do + i];
        for (int i = lane; i < len * Da; i += 32) {
            act[dst * Da + i] = t_act[src * Da + i];
            mean[dst * Da + i] = t_mean[src * Da + i];
        }
        for (int i = lane; i < len; i += 32) {
            rew[dst + i] = t_rew[src + i];
            done[dst + i] = (i == len - 1) ? 1 : 0;
        }
    }
}

}  // namespace promp

using namespace promp;

extern "C" int64_t promp_paths_workspace_bytes(int M, int E, int timeline_len) {
    (void)M; (void)E;
    return ((int64_t)timeline_len + 8) * 4;          // hist [T] (zero on entry, left zero) + cut [2]
}

extern "C" int promp_paths_histogram(int M, int E, int timeline_len, const uint8_t* t_done, int32_t* hist, void* stream) {
    PROMP_REQUIRE(M > 0 && E > 0 && timeline_len > 0, "promp_paths_histogram: sizes must be positive (got %d, %d, %d)", M, E,
                  timeline_len);
    PROMP_REQUIRE((int64_t)M * E <= INT32_MAX, "promp_paths_histogram: M * E = %lld env slots exceeds the int32 range",
                  (long long)M * E);
    PROMP_REQUIRE(t_done && hist, "promp_paths_histogram: null pointer argument");
    const int n_slots = M * E;
    path_hist_kernel<<<(n_slots + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n_slots, timeline_len, t_done, hist);
    PROMP_LAUNCH_CHECK("path_hist_kernel");
    return PROMP_OK;
}

static int paths_finalize(const char* fn, int M, int E, int timeline_len, int max_paths, int max_samples, int obs_dim,
                          int act_dim, int64_t target_samples, const int32_t* hist_in, const uint8_t* t_done, const float* t_obs,
                          const float* t_act, const float* t_mean, const float* t_rew, int32_t* path_off, int32_t* n_paths,
                          int32_t* n_valid, int32_t* src_slot, int32_t* src_start, float* obs, float* act, float* mean,
                          float* rew, uint8_t* done, int32_t* cut_out, void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(M > 0 && E > 0 && E <= 1024 && timeline_len > 0 && max_paths > 0 && max_samples > 0,
                  "%s: bad sizes (1 <= E <= 1024)", fn);
    PROMP_REQUIRE(M <= 65535, "%s: M=%d exceeds the grid.y limit 65535", fn, M);
    PROMP_REQUIRE(max_samples >= E * timeline_len, "%s: max_samples must cover E * timeline_len samples per task", fn);
    PROMP_REQUIRE(target_samples > 0, "%s: target_samples must be positive (got %lld)", fn, (long long)target_samples);
    PROMP_REQUIRE(t_done && t_obs && t_act && t_mean && t_rew && path_off && n_paths && n_valid && src_slot && src_start && obs &&
                      act && mean && rew && done && cut_out && workspace,
                  "%s: null pointer argument", fn);
    PROMP_REQUIRE(workspace_bytes >= promp_paths_workspace_bytes(M, E, timeline_len), "%s: workspace too small", fn);
    cudaStream_t st = (cudaStream_t)stream;
    if (hist_in) {        // counts summed over every shard of the task batch: scanned as given, left as given
        path_cut_kernel<<<1, 1024, 0, st>>>(timeline_len, target_samples, hist_in, nullptr, cut_out);
        PROMP_LAUNCH_CHECK("path_cut_kernel");
    } else {
        int* hist = (int*)workspace;
        const int n_slots = M * E;
        path_hist_kernel<<<(n_slots + 127) / 128, 128, 0, st>>>(n_slots, timeline_len, t_done, hist);
        PROMP_LAUNCH_CHECK("path_hist_kernel");
        path_cut_kernel<<<1, 1024, 0, st>>>(timeline_len, target_samples, hist, hist, cut_out);
        PROMP_LAUNCH_CHECK("path_cut_kernel");
    }
    const int threads = ((E + 31) / 32) * 32;
    path_table_kernel<<<M, threads, 0, st>>>(E, timeline_len, max_paths, t_done, cut_out, path_off, n_paths, n_valid, src_slot,
                                             src_start);
    PROMP_LAUNCH_CHECK("path_table_kernel");
    path_compact_kernel<<<dim3(32, M), 256, 0, st>>>(M, E, timeline_len, max_paths, max_samples, obs_dim, act_dim, path_off, n_paths,
                                                     src_slot, src_start, t_obs, t_act, t_mean, t_rew, obs, act, mean, rew, done);
    PROMP_LAUNCH_CHECK("path_compact_kernel");
    return PROMP_OK;
}

extern "C" int promp_paths_finalize(int M, int E, int timeline_len, int max_paths, int max_samples, int obs_dim, int act_dim,
                                    int64_t target_samples, const uint8_t* t_done, const float* t_obs, const float* t_act,
                                    const float* t_mean, const float* t_rew, int32_t* path_off, int32_t* n_paths, int32_t* n_valid,
                                    int32_t* src_slot, int32_t* src_start, float* obs, float* act, float* mean, float* rew,
                                    uint8_t* done, int32_t* cut_out, void* workspace, int64_t workspace_bytes, void* stream) {
    return paths_finalize("promp_paths_finalize", M, E, timeline_len, max_paths, max_samples, obs_dim, act_dim, target_samples,
                          nullptr, t_done, t_obs, t_act, t_mean, t_rew, path_off, n_paths, n_valid, src_slot, src_start, obs, act,
                          mean, rew, done, cut_out, workspace, workspace_bytes, stream);
}

extern "C" int promp_paths_finalize_ex(int M, int E, int timeline_len, int max_paths, int max_samples, int obs_dim, int act_dim,
                                       int64_t target_samples, const int32_t* hist_in, const uint8_t* t_done, const float* t_obs,
                                       const float* t_act, const float* t_mean, const float* t_rew, int32_t* path_off,
                                       int32_t* n_paths, int32_t* n_valid, int32_t* src_slot, int32_t* src_start, float* obs,
                                       float* act, float* mean, float* rew, uint8_t* done, int32_t* cut_out, void* workspace,
                                       int64_t workspace_bytes, void* stream) {
    return paths_finalize("promp_paths_finalize_ex", M, E, timeline_len, max_paths, max_samples, obs_dim, act_dim, target_samples,
                          hist_in, t_done, t_obs, t_act, t_mean, t_rew, path_off, n_paths, n_valid, src_slot, src_start, obs, act,
                          mean, rew, done, cut_out, workspace, workspace_bytes, stream);
}
