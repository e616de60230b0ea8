// Launch dispatch and C entry points of the fused rollout kernel and the single-step vec-env kernels (rollout_kernel.cuh).
// See include/promp_b200.h for the interface and the reference functions each entry point replaces.
#include <cstring>
#include <type_traits>

#include "rollout_kernel.cuh"

namespace promp {

template <class Env>
struct EnvTag {
    using type = Env;
};

// The one env_kind dispatch: calls f(EnvTag<Env>{}) with the environment type of env_kind.  A new environment is one type
// in envs.cuh plus one case here.
template <class F>
static int with_env(const char* fn, int env_kind, F&& f) {
    switch (env_kind) {
        case PointCorner::KIND: return f(EnvTag<PointCorner>{});
        case Point::KIND: return f(EnvTag<Point>{});
        case Cheetah::KIND: return f(EnvTag<Cheetah>{});
        case PointWalls::KIND: return f(EnvTag<PointWalls>{});
        case PointMomentum::KIND: return f(EnvTag<PointMomentum>{});
        case Walker::KIND: return f(EnvTag<Walker>{});
        case Swimmer::KIND: return f(EnvTag<Swimmer>{});
    }
    set_error("%s: unknown env_kind %d", fn, env_kind);
    return PROMP_ERR_INVALID_ARG;
}

// rollout_deep_kernel for a policy of depth 1 or 3: its hidden-to-hidden layers take dynamic shared memory beyond the
// 48 KB default, so the limit is raised once per instantiation
template <class Env, int HID, class Act, bool K>
static int launch_rollout_deep(const RolloutArgs& A, int nh, dim3 grid, cudaStream_t st) {
    static bool configured = false;
    constexpr auto kernel = rollout_deep_kernel<Env, HID, Act, K>;
    if (!configured) {
        PROMP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, rollout_deep_smem_bytes<HID>(2)));
        configured = true;
    }
    kernel<<<grid, RO_WARPS * 32, rollout_deep_smem_bytes<HID>(nh), st>>>(A, nh);
    return PROMP_OK;
}

template <class Env, bool K>
static int launch_rollout_deep_act(int width, bool relu, bool out_tanh, const RolloutArgs& A, int nh, dim3 grid,
                                   cudaStream_t st) {
    using OR = OutTanh<ActRelu>;
    using OT = OutTanh<ActTanh>;
    if (out_tanh) {
        if (relu) return width == 64 ? launch_rollout_deep<Env, 64, OR, K>(A, nh, grid, st) : launch_rollout_deep<Env, 32, OR, K>(A, nh, grid, st);
        return width == 64 ? launch_rollout_deep<Env, 64, OT, K>(A, nh, grid, st) : launch_rollout_deep<Env, 32, OT, K>(A, nh, grid, st);
    }
    if (relu)
        return width == 64 ? launch_rollout_deep<Env, 64, ActRelu, K>(A, nh, grid, st)
                           : launch_rollout_deep<Env, 32, ActRelu, K>(A, nh, grid, st);
    return width == 64 ? launch_rollout_deep<Env, 64, ActTanh, K>(A, nh, grid, st)
                       : launch_rollout_deep<Env, 32, ActTanh, K>(A, nh, grid, st);
}

// `hidden` as decode_hidden gives it: width 32 or 64, ReLU or tanh, identity or tanh output, 1 to 3 hidden layers
static int launch_rollout(const char* fn, int env_kind, int width, bool relu, bool out_tanh, int depth, const RolloutArgs& A,
                          cudaStream_t st) {
    const dim3 grid((A.E + RO_WARPS - 1) / RO_WARPS, A.M);
    return with_env(fn, env_kind, [&](auto env) -> int {
        using Env = typename decltype(env)::type;
        if (depth != 2) {
            const int rc = A.key_offset ? launch_rollout_deep_act<Env, true>(width, relu, out_tanh, A, depth - 1, grid, st)
                                        : launch_rollout_deep_act<Env, false>(width, relu, out_tanh, A, depth - 1, grid, st);
            if (rc != PROMP_OK) return rc;
            PROMP_LAUNCH_CHECK("rollout_deep_kernel");
            return PROMP_OK;
        }
        const auto go = [&](auto keyed) {
            constexpr bool K = decltype(keyed)::value;
            if (out_tanh) {
                using OR = OutTanh<ActRelu>;
                using OT = OutTanh<ActTanh>;
                if (relu) {
                    if (width == 64) rollout_kernel<Env, 64, OR, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
                    else rollout_kernel<Env, 32, OR, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
                } else {
                    if (width == 64) rollout_kernel<Env, 64, OT, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
                    else rollout_kernel<Env, 32, OT, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
                }
            } else if (relu) {
                if (width == 64) rollout_kernel<Env, 64, ActRelu, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
                else rollout_kernel<Env, 32, ActRelu, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
            } else {
                if (width == 64) rollout_kernel<Env, 64, ActTanh, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
                else rollout_kernel<Env, 32, ActTanh, K><<<grid, RO_WARPS * 32, 0, st>>>(A);
            }
        };
        if (A.key_offset) go(std::true_type{});
        else go(std::false_type{});
        PROMP_LAUNCH_CHECK("rollout_kernel");
        return PROMP_OK;
    });
}

}  // namespace promp

using namespace promp;

extern "C" int promp_env_state_dim(int env_kind) {
    return with_env("promp_env_state_dim", env_kind, [](auto env) { return decltype(env)::type::SD; });
}
extern "C" int promp_env_task_dim(int env_kind) {
    return with_env("promp_env_task_dim", env_kind, [](auto env) { return decltype(env)::type::TD; });
}

static int rollout_fixed(const char* fn, int env_kind, int reward_type, float sparse_radius, int normalize_actions, int M, int E,
                         int H, int hidden, const float* params, int64_t param_stride, const float* task_params,
                         const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                         const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs, float* act,
                         float* mean, float* rew, uint8_t* done, float* info, float* log_std_out, float* final_state,
                         void* stream, int task_offset) {
    PROMP_REQUIRE(M > 0 && E > 0 && H > 0, "%s: M, E, H must be positive (got %d, %d, %d)", fn, M, E, H);
    PROMP_REQUIRE(M <= 65535, "%s: M=%d exceeds the grid.y limit 65535", fn, M);
    if (check_task_offset(fn, task_offset, M, E) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(params && task_params && obs && act && mean && rew && done && log_std_out, "%s: null pointer argument", fn);
    int width, depth;
    bool relu, out_tanh;
    if (decode_hidden(fn, hidden, width, relu, out_tanh, depth) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(width == 64 || width == 32, "%s: hidden size %d unsupported (32 or 64)", fn, width);
    PROMP_REQUIRE(reward_type >= 0 && reward_type <= 2, "%s: bad reward_type %d", fn, reward_type);
    PROMP_REQUIRE(env_kind != PROMP_ENV_CHEETAH_DIR || info != nullptr,
                  "%s: cheetah needs the info buffer [2,M,E,H] ([3,M,E,H] for reward_type 1)", fn);
    PROMP_REQUIRE(env_kind != PROMP_ENV_CHEETAH_DIR || reward_type == 0 || reward_type == 1,
                  "%s: cheetah reward_type must be 0 (RandDirec) or 1 (RandVel)", fn);
    PROMP_REQUIRE(env_kind != PROMP_ENV_POINT_WALLS || reward_type == PROMP_REWARD_DENSE || reward_type == PROMP_REWARD_DENSE_SQUARED,
                  "%s: the walls env supports reward_type dense / dense_squared", fn);
    PROMP_REQUIRE(env_kind != PROMP_ENV_SWIMMER || info != nullptr, "%s: the swimmer needs the info buffer [2,M,E,H]", fn);
    PROMP_REQUIRE(env_kind != PROMP_ENV_SWIMMER || reward_type == 0, "%s: swimmer reward_type must be 0", fn);
    PROMP_REQUIRE(env_kind != PROMP_ENV_POINT, "%s: MetaPointEnv terminates early (variable-length paths); use the "
                                               "stepwise sampler (promp_env_step) for it", fn);
    RolloutArgs A{reward_type, sparse_radius, normalize_actions, M, E, H, params, param_stride, task_params, init_state, noise, seed,
                  stream_id, stream_id_dev, clip_reported_log_std, min_log_std, obs, act, mean, rew, done, info, log_std_out,
                  final_state, 0, H, (uint32_t)task_offset * (uint32_t)E};
    return launch_rollout(fn, env_kind, width, relu, out_tanh, depth, A, (cudaStream_t)stream);
}

extern "C" int promp_rollout(int env_kind, int reward_type, float sparse_radius, int normalize_actions, int M, int E, int H,
                             int hidden,
                             const float* params, int64_t param_stride, const float* task_params,
                             const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                             const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs, float* act, float* mean,
                             float* rew, uint8_t* done, float* info, float* log_std_out, float* final_state,
                             void* stream) {
    return rollout_fixed("promp_rollout", env_kind, reward_type, sparse_radius, normalize_actions, M, E, H, hidden, params,
                         param_stride, task_params, init_state, noise, seed, stream_id, stream_id_dev, clip_reported_log_std,
                         min_log_std, obs, act, mean, rew, done, info, log_std_out, final_state, stream, 0);
}

extern "C" int promp_rollout_ex(int env_kind, int reward_type, float sparse_radius, int normalize_actions, int M, int E, int H,
                                int hidden, const float* params, int64_t param_stride, const float* task_params,
                                const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                                const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs, float* act,
                                float* mean, float* rew, uint8_t* done, float* info, float* log_std_out, float* final_state,
                                void* stream, int task_offset) {
    return rollout_fixed("promp_rollout_ex", env_kind, reward_type, sparse_radius, normalize_actions, M, E, H, hidden, params,
                         param_stride, task_params, init_state, noise, seed, stream_id, stream_id_dev, clip_reported_log_std,
                         min_log_std, obs, act, mean, rew, done, info, log_std_out, final_state, stream, task_offset);
}

// MetaPointEnv (early `done`, point_env_2d.py:9-59) in the fused kernel: every env slot records a timeline of `timeline_len`
// steps; paths end on done / after `horizon` steps and the slot is reset in-kernel.  promp_paths_finalize then applies the
// reference's collect-until-enough rule (meta_sampler.py:87-137) to the timelines.
static int rollout_early_term(const char* fn, int env_kind, int normalize_actions, int M, int E, int timeline_len, int horizon,
                              int hidden, const float* params, int64_t param_stride, const float* task_params,
                              const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                              const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs, float* act,
                              float* mean, float* rew, uint8_t* done, float* log_std_out, void* stream, int task_offset) {
    PROMP_REQUIRE(env_kind == PROMP_ENV_POINT || env_kind == PROMP_ENV_WALKER,
                  "%s: implemented for MetaPointEnv and the walker (env_kind %d given)", fn, env_kind);
    PROMP_REQUIRE(M > 0 && E > 0 && timeline_len > 0 && horizon > 0, "%s: sizes must be positive", fn);
    PROMP_REQUIRE(M <= 65535, "%s: M=%d exceeds the grid.y limit 65535", fn, M);
    if (check_task_offset(fn, task_offset, M, E) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(params && task_params && obs && act && mean && rew && done && log_std_out, "%s: null pointer argument", fn);
    int width, depth;
    bool relu, out_tanh;
    if (decode_hidden(fn, hidden, width, relu, out_tanh, depth) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(width == 64 || width == 32, "%s: hidden size %d unsupported (32 or 64)", fn, width);
    RolloutArgs A{0, 0.f, normalize_actions, M, E, timeline_len, params, param_stride, task_params, init_state, noise, seed,
                  stream_id, stream_id_dev, clip_reported_log_std, min_log_std, obs, act, mean, rew, done, nullptr, log_std_out,
                  nullptr, 1, horizon, (uint32_t)task_offset * (uint32_t)E};
    return launch_rollout(fn, env_kind, width, relu, out_tanh, depth, A, (cudaStream_t)stream);
}

extern "C" int promp_rollout_early_term(int env_kind, int normalize_actions, int M, int E, int timeline_len, int horizon, int hidden,
                                        const float* params, int64_t param_stride, const float* task_params,
                                        const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                                        const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs,
                                        float* act, float* mean, float* rew, uint8_t* done, float* log_std_out, void* stream) {
    return rollout_early_term("promp_rollout_early_term", env_kind, normalize_actions, M, E, timeline_len, horizon, hidden, params,
                              param_stride, task_params, init_state, noise, seed, stream_id, stream_id_dev, clip_reported_log_std,
                              min_log_std, obs, act, mean, rew, done, log_std_out, stream, 0);
}

extern "C" int promp_rollout_early_term_ex(int env_kind, int normalize_actions, int M, int E, int timeline_len, int horizon,
                                           int hidden, const float* params, int64_t param_stride, const float* task_params,
                                           const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                                           const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std,
                                           float* obs, float* act, float* mean, float* rew, uint8_t* done, float* log_std_out,
                                           void* stream, int task_offset) {
    return rollout_early_term("promp_rollout_early_term_ex", env_kind, normalize_actions, M, E, timeline_len, horizon, hidden,
                              params, param_stride, task_params, init_state, noise, seed, stream_id, stream_id_dev,
                              clip_reported_log_std, min_log_std, obs, act, mean, rew, done, log_std_out, stream, task_offset);
}

__global__ void counter_add_kernel(uint64_t* c, uint64_t inc) { *c += inc; }
extern "C" int promp_counter_add(uint64_t* counter, uint64_t inc, void* stream) {
    PROMP_REQUIRE(counter != nullptr, "promp_counter_add: null counter");
    counter_add_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(counter, inc);
    PROMP_LAUNCH_CHECK("counter_add_kernel");
    return PROMP_OK;
}

// The task vectors travel inside the kernel's argument block, which the launch copies when it is enqueued: no host memory
// has to outlive the call and nothing waits for the stream.  A copy from pageable memory would wait for all work queued
// before it, and the device would then idle while the host enqueues what follows.  SET_TASKS_CHUNK floats per launch keep
// the block under the 4 KB kernel parameter limit.
constexpr int SET_TASKS_CHUNK = 960;
struct SetTasksArgs {
    float v[SET_TASKS_CHUNK];      // per-task values [c0, c0 + n) of the flat [M, task_dim] array
    int c0, n, task_dim, E;
    float* per_task;               // [M, task_dim]
    float* per_env;                // [M * E, task_dim] or NULL
};
__global__ void set_tasks_kernel(const __grid_constant__ SetTasksArgs A) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;        // (value, env of its task) pairs, value-major
    const int E = A.per_env ? A.E : 1;
    if (i >= A.n * E) return;
    const int j = i / E, k = i - j * E;
    const int f = A.c0 + j, m = f / A.task_dim, d = f - m * A.task_dim;
    if (k == 0) A.per_task[f] = A.v[j];
    if (A.per_env) A.per_env[((int64_t)m * A.E + k) * A.task_dim + d] = A.v[j];
}
extern "C" int promp_set_tasks(int M, int task_dim, int E, const float* host_vec, float* per_task, float* per_env,
                               void* stream) {
    PROMP_REQUIRE(M >= 0 && task_dim > 0 && E > 0, "promp_set_tasks: M >= 0, task_dim > 0 and E > 0 required");
    PROMP_REQUIRE(M == 0 || (host_vec && per_task), "promp_set_tasks: null host_vec or per_task");
    const int64_t total = (int64_t)M * task_dim;
    for (int64_t c0 = 0; c0 < total; c0 += SET_TASKS_CHUNK) {
        SetTasksArgs A;
        A.n = (int)(total - c0 < SET_TASKS_CHUNK ? total - c0 : SET_TASKS_CHUNK);
        A.c0 = (int)c0, A.task_dim = task_dim, A.E = E, A.per_task = per_task, A.per_env = per_env;
        memcpy(A.v, host_vec + c0, sizeof(float) * A.n);
        const int64_t threads = (int64_t)A.n * (per_env ? E : 1);
        set_tasks_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(A);
        PROMP_LAUNCH_CHECK("set_tasks_kernel");
    }
    return PROMP_OK;
}

extern "C" int promp_env_step(int env_kind, int reward_type, float sparse_radius, int normalize_actions, int n_env, int H,
                              float* state,
                              int32_t* ts, const float* actions, const float* task_params,
                              const float* reset_state, float* next_obs, float* rew, uint8_t* done, float* info,
                              void* stream) {
    PROMP_REQUIRE(n_env > 0 && H > 0, "promp_env_step: n_env and H must be positive");
    PROMP_REQUIRE(state && ts && actions && task_params && reset_state && next_obs && rew && done,
                  "promp_env_step: null pointer argument");
    const EnvCfg cfg{reward_type, sparse_radius, normalize_actions != 0};
    const int bs = 128, gs = (n_env + bs - 1) / bs;
    return with_env("promp_env_step", env_kind, [&](auto env) -> int {
        env_step_kernel<typename decltype(env)::type><<<gs, bs, 0, (cudaStream_t)stream>>>(
            cfg, n_env, H, state, ts, actions, task_params, reset_state, next_obs, rew, done, info);
        PROMP_LAUNCH_CHECK("env_step_kernel");
        return PROMP_OK;
    });
}

extern "C" int promp_env_observe(int env_kind, int n_env, const float* state, float* obs, void* stream) {
    PROMP_REQUIRE(n_env > 0 && state && obs, "promp_env_observe: bad arguments");
    const int bs = 128, gs = (n_env + bs - 1) / bs;
    return with_env("promp_env_observe", env_kind, [&](auto env) -> int {
        env_observe_kernel<typename decltype(env)::type><<<gs, bs, 0, (cudaStream_t)stream>>>(n_env, state, obs);
        PROMP_LAUNCH_CHECK("env_observe_kernel");
        return PROMP_OK;
    });
}

#ifdef PROMP_EXP_CLOCKS
extern "C" int promp_debug_rollout_clocks(unsigned long long* out16, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out16, promp::g_ro_clk, 16 * sizeof(unsigned long long));
    if (reset) {
        unsigned long long z[16] = {0};
        cudaMemcpyToSymbol(promp::g_ro_clk, z, sizeof(z));
    }
    return 0;
}
#endif
