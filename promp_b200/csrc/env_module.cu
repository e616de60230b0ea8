// Users' own environments: a cubin compiled at run time from a user's env struct (promp_b200/_jit.py, user_env.cuh) is
// loaded as a CUDA library, and these entry points launch its rollout / env-step / env-observe kernels with the same
// arguments and checks as the env_kind entry points of rollout.cu.  Runtime API only (cudaLibraryLoadData,
// cudaLibraryGetKernel, cudaLaunchKernel), so the launches are graph-capturable and nothing links libcuda.
#include "rollout_kernel.cuh"

namespace promp {

struct EnvModule {
    cudaLibrary_t lib;
    cudaKernel_t k[PROMP_ENV_MODULE_SLOTS];   // NULL: variant not compiled into this module
    int dims[PROMP_ENV_MODULE_NDIMS];
};

// slot of the rollout kernel of one `hidden` variant (decode_hidden), keyed (sharded launch) or not; depth 1 and 3 share the
// rollout_deep_kernel slots
static int rollout_slot(bool relu, bool out_tanh, int width, bool keyed, int depth) {
    const int v = ((relu ? 1 : 0) + (out_tanh ? 2 : 0)) * 2 + (width == 64 ? 1 : 0);
    return (depth == 2 ? PROMP_ENV_SLOT_ROLLOUT : PROMP_ENV_SLOT_ROLLOUT_DEEP) + 2 * v + (keyed ? 1 : 0);
}

static EnvModule* as_module(const char* fn, void* h) {
    if (!h) promp::set_error("%s: null env module handle", fn);
    return (EnvModule*)h;
}

static int launch(const char* fn, EnvModule* m, int slot, dim3 grid, dim3 block, void** args, int smem, cudaStream_t st) {
    PROMP_REQUIRE(m->k[slot] != nullptr, "%s: kernel slot %d was not compiled into this env module (the policy's hidden "
                                         "variant or the env kernels were not requested)", fn, slot);
    PROMP_CUDA(cudaLaunchKernel((const void*)m->k[slot], grid, block, args, smem, st));
    return PROMP_OK;
}

static int rollout_module(const char* fn, void* handle, int reward_type, float radius, int normalize_actions, int M, int E,
                          int T, int horizon, int early_term, int hidden, const float* params, int64_t param_stride,
                          const float* task_params, const float* init_state, const float* noise, uint64_t seed,
                          uint64_t stream_id, const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std,
                          float* obs, float* act, float* mean, float* rew, uint8_t* done, float* info, float* log_std_out,
                          float* final_state, void* stream, int task_offset) {
    EnvModule* m = as_module(fn, handle);
    if (!m) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(M > 0 && E > 0 && T > 0 && horizon > 0, "%s: sizes must be positive (got M=%d, E=%d, %d, %d)", fn, M, E, T,
                  horizon);
    PROMP_REQUIRE(M <= 65535, "%s: M=%d exceeds the grid.y limit 65535", fn, M);
    if (check_task_offset(fn, task_offset, M, E) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(params && task_params && obs && act && mean && rew && done && log_std_out, "%s: null pointer argument", fn);
    int width, depth;
    bool relu, out_tanh;
    if (decode_hidden(fn, hidden, width, relu, out_tanh, depth) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(width == 64 || width == 32, "%s: hidden size %d unsupported (32 or 64)", fn, width);
    PROMP_REQUIRE(reward_type >= 0 && reward_type <= 2, "%s: bad reward_type %d", fn, reward_type);
    const int ninfo = m->dims[4], ends_early = m->dims[5];
    PROMP_REQUIRE(early_term || ninfo == 0 || info != nullptr, "%s: the env writes %d info channels: info [%d,M,E,H] is required",
                  fn, ninfo, ninfo);
    PROMP_REQUIRE(!early_term || ends_early, "%s: the env does not end early (ENDS_EARLY = false); use promp_rollout_module",
                  fn);
    PROMP_REQUIRE(early_term || !ends_early, "%s: the env ends early (variable-length paths); use "
                                             "promp_rollout_early_term_module", fn);
    RolloutArgs A{reward_type, radius, normalize_actions, M, E, T, params, param_stride, task_params, init_state, noise, seed,
                  stream_id, stream_id_dev, clip_reported_log_std, min_log_std, obs, act, mean, rew, done,
                  early_term ? nullptr : info, log_std_out, early_term ? nullptr : final_state, early_term, horizon,
                  (uint32_t)task_offset * (uint32_t)E};
    int nh = depth - 1;
    void* args[] = {&A, &nh};
    const dim3 grid((E + RO_WARPS - 1) / RO_WARPS, M);
    const int smem = depth == 2 ? 0 : (width == 64 ? rollout_deep_smem_bytes<64>(nh) : rollout_deep_smem_bytes<32>(nh));
    return launch(fn, m, rollout_slot(relu, out_tanh, width, A.key_offset != 0, depth), grid, dim3(RO_WARPS * 32), args, smem,
                  (cudaStream_t)stream);
}

}  // namespace promp

using namespace promp;

extern "C" int promp_env_module_load(const void* image, int64_t bytes, const char* const* names, int n_names, const int* dims,
                                     void** handle_out) {
    const char* fn = "promp_env_module_load";
    PROMP_REQUIRE(image && bytes > 0 && names && dims && handle_out, "%s: bad arguments", fn);
    PROMP_REQUIRE(n_names == PROMP_ENV_MODULE_SLOTS, "%s: n_names must be %d (got %d)", fn, PROMP_ENV_MODULE_SLOTS, n_names);
    PROMP_REQUIRE(dims[0] >= 1 && dims[0] <= 19, "%s: observation size %d outside the policy range 1..19", fn, dims[0]);
    PROMP_REQUIRE(dims[1] >= 1 && dims[1] <= 8, "%s: action size %d outside the policy range 1..8", fn, dims[1]);
    PROMP_REQUIRE(dims[2] >= 1 && dims[3] >= 1, "%s: state and task sizes must be >= 1 (got %d, %d)", fn, dims[2], dims[3]);
    PROMP_REQUIRE(dims[4] >= 0 && dims[4] <= 3, "%s: %d info channels (0..3 supported)", fn, dims[4]);
    *handle_out = nullptr;
    EnvModule* m = new EnvModule();
    const cudaError_t e = cudaLibraryLoadData(&m->lib, image, nullptr, nullptr, 0, nullptr, nullptr, 0);
    if (e != cudaSuccess) {
        delete m;
        return check_cuda(e, "cudaLibraryLoadData");
    }
    for (int i = 0; i < PROMP_ENV_MODULE_NDIMS; ++i) m->dims[i] = dims[i];
    for (int i = 0; i < n_names; ++i) {
        if (!names[i] || !names[i][0]) continue;
        const cudaError_t ek = cudaLibraryGetKernel(&m->k[i], m->lib, names[i]);
        if (ek != cudaSuccess) {
            cudaLibraryUnload(m->lib);
            delete m;
            return check_cuda(ek, names[i]);
        }
        if (i >= PROMP_ENV_SLOT_ROLLOUT_DEEP) {      // rollout_deep_kernel: hidden layers in dynamic shared memory (> 48 KB)
            const int smem = ((i - PROMP_ENV_SLOT_ROLLOUT_DEEP) / 2) % 2 ? rollout_deep_smem_bytes<64>(2) : rollout_deep_smem_bytes<32>(2);
            const cudaError_t ea = cudaFuncSetAttribute((const void*)m->k[i], cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
            if (ea != cudaSuccess) {
                cudaLibraryUnload(m->lib);
                delete m;
                return check_cuda(ea, "cudaFuncSetAttribute (rollout_deep_kernel)");
            }
        }
    }
    *handle_out = m;
    return PROMP_OK;
}

extern "C" int promp_env_module_unload(void* handle) {
    EnvModule* m = as_module("promp_env_module_unload", handle);
    if (!m) return PROMP_ERR_INVALID_ARG;
    const cudaError_t e = cudaLibraryUnload(m->lib);
    delete m;
    return check_cuda(e, "cudaLibraryUnload");
}

extern "C" int promp_rollout_module(void* module, int reward_type, float sparse_radius, int normalize_actions, int M, int E, int H,
                                    int hidden, const float* params, int64_t param_stride, const float* task_params,
                                    const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                                    const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs,
                                    float* act, float* mean, float* rew, uint8_t* done, float* info, float* log_std_out,
                                    float* final_state, void* stream, int task_offset) {
    return rollout_module("promp_rollout_module", module, reward_type, sparse_radius, normalize_actions, M, E, H, H, 0, hidden,
                          params, param_stride, task_params, init_state, noise, seed, stream_id, stream_id_dev,
                          clip_reported_log_std, min_log_std, obs, act, mean, rew, done, info, log_std_out, final_state, stream,
                          task_offset);
}

extern "C" int promp_rollout_early_term_module(void* module, int normalize_actions, int M, int E, int timeline_len, int horizon,
                                               int hidden, const float* params, int64_t param_stride, const float* task_params,
                                               const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                                               const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std,
                                               float* obs, float* act, float* mean, float* rew, uint8_t* done,
                                               float* log_std_out, void* stream, int task_offset) {
    return rollout_module("promp_rollout_early_term_module", module, 0, 0.f, normalize_actions, M, E, timeline_len, horizon, 1,
                          hidden, params, param_stride, task_params, init_state, noise, seed, stream_id, stream_id_dev,
                          clip_reported_log_std, min_log_std, obs, act, mean, rew, done, nullptr, log_std_out, nullptr, stream,
                          task_offset);
}

extern "C" int promp_env_step_module(void* module, int reward_type, float sparse_radius, int normalize_actions, int n_env, int H,
                                     float* state, int32_t* ts, const float* actions, const float* task_params,
                                     const float* reset_state, float* next_obs, float* rew, uint8_t* done, float* info,
                                     void* stream) {
    const char* fn = "promp_env_step_module";
    EnvModule* m = as_module(fn, module);
    if (!m) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(n_env > 0 && H > 0, "%s: n_env and H must be positive", fn);
    PROMP_REQUIRE(state && ts && actions && task_params && reset_state && next_obs && rew && done, "%s: null pointer argument",
                  fn);
    EnvCfg cfg{reward_type, sparse_radius, normalize_actions != 0};
    void* args[] = {&cfg, &n_env, &H, &state, &ts, &actions, &task_params, &reset_state, &next_obs, &rew, &done, &info};
    const int bs = 128;
    return launch(fn, m, PROMP_ENV_SLOT_STEP, dim3((n_env + bs - 1) / bs), dim3(bs), args, 0, (cudaStream_t)stream);
}

extern "C" int promp_env_observe_module(void* module, int n_env, const float* state, float* obs, void* stream) {
    const char* fn = "promp_env_observe_module";
    EnvModule* m = as_module(fn, module);
    if (!m) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(n_env > 0 && state && obs, "%s: bad arguments", fn);
    void* args[] = {&n_env, &state, &obs};
    const int bs = 128;
    return launch(fn, m, PROMP_ENV_SLOT_OBSERVE, dim3((n_env + bs - 1) / bs), dim3(bs), args, 0, (cudaStream_t)stream);
}

extern "C" int promp_cuda_build_version(void) { return CUDART_VERSION; }
