/*
 * promp_b200 - C ABI of the H100-native (sm_90a) ProMP hot path.
 *
 * The reference (jonasrothfuss/ProMP @ 93ae339) is pure Python and has no FFI of its own: its
 * "operator interface" for this path is the set of Python methods that meta_trainer.py calls
 * (SURVEY.md section 8b).  Each entry point below replaces the body of one of those methods and
 * cites it (paths relative to the reference's meta_policy_search/).  promp_b200/_lib.py holds the
 * ctypes binding; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *  - Every pointer is a DEVICE pointer unless its name ends in _host.  The library never allocates,
 *    frees or retains memory: inputs, outputs and workspaces are owned by the caller.
 *  - All entry points are asynchronous on `stream` (a cudaStream_t passed as void*), re-entrant per
 *    stream, and return 0 on success or a negative promp_status; promp_last_error() gives the text.
 *  - Tensors are dense, row-major, float32 unless stated.  M = meta_batch_size (tasks), E = envs
 *    (rollouts) per task, H = max_path_length, N = E*H samples per task with the reference's index
 *    contract n = e*H + t (samplers/meta_sampler.py:117, samplers/base.py:165-173).
 *  - A policy parameter set is a flat vector of P floats in the reference's variable creation
 *    order (policies/gaussian_mlp_policy.py:55-80): W0[Do,Hd] b0[Hd] W1[Hd,Hd] b1[Hd] W2[Hd,Da]
 *    b2[Da] log_std[Da], kernels [in,out] row-major (policies/networks/mlp.py:100).
 *    `params` + `param_stride`: task m reads params + m*param_stride; stride 0 = one shared theta
 *    (pre-update policy), stride P = per-task theta_i' (post-update policy).
 */
#ifndef PROMP_B200_H
#define PROMP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    PROMP_OK = 0,
    PROMP_ERR_INVALID_ARG = -1,     /* bad dimension / unsupported combination / null pointer */
    PROMP_ERR_CUDA = -2,            /* a CUDA runtime call or kernel launch failed            */
    PROMP_ERR_WORKSPACE = -3        /* workspace too small                                     */
} promp_status;

/* env kinds (envs/point_envs/point_env_2d_corner.py, envs/point_envs/point_env_2d.py,
 * envs/mujoco_envs/half_cheetah_rand_direc.py [analytic surrogate]) */
enum {
    PROMP_ENV_POINT_CORNER = 0,
    PROMP_ENV_POINT = 1,
    PROMP_ENV_CHEETAH_DIR = 2,
    PROMP_ENV_POINT_WALLS = 3,     /* envs/point_envs/point_env_2d_walls.py: two circular walls with one gap each      */
    PROMP_ENV_POINT_MOMENTUM = 4,  /* envs/point_envs/point_env_2d_momentum.py: actions accelerate, obs = (pos, vel)   */
    PROMP_ENV_WALKER = 5,          /* envs/mujoco_envs/walker2d_rand_vel.py / walker2d_rand_direc.py [analytic surrogate,
                                      obs 17 / act 6, early done when the torso falls]                                  */
    PROMP_ENV_SWIMMER = 6          /* envs/mujoco_envs/swimmer_rand_vel.py [analytic surrogate, obs 8 / act 2]           */
};
/* MetaPointEnvCorner.reward_type (point_env_2d_corner.py:13-16) */
enum { PROMP_REWARD_SPARSE = 0, PROMP_REWARD_DENSE = 1, PROMP_REWARD_DENSE_SQUARED = 2 };
/* objective kinds of promp_policy_grad */
enum {
    PROMP_OBJ_RATIO = 0,   /* -mean(ratio*adv)                       meta_algos/pro_mp.py:59-65          */
    PROMP_OBJ_LOGLIK = 1,  /* -mean(logp*adv)                        meta_algos/trpo_maml.py:58-62       */
    PROMP_OBJ_CLIP = 2,    /* -mean(min(r*adv, clip(r,1-e,1+e)*adv)) meta_algos/pro_mp.py:135-141        */
    PROMP_OBJ_NONE = 3,    /* only the kl_coeff * mean KL(old||new) term                                 */
    PROMP_OBJ_EXPLORE = 4  /* -c_m * mean(logp): E-MAML exploration term, trpo_maml.py:137-144; `adv` is  */
                           /* the per-task coefficient c [M] (promp_emaml_coeff), gradient stages only    */
};
/* Hidden non-linearity of the policy (policies/networks/mlp.py: hidden_nonlinearity), carried in the `hidden` argument of
 * the policy and rollout entry points: hidden = width | flag, width 32 or 64 in the low byte.  No flag = tanh, so a plain
 * width keeps its meaning.  ReLU follows TensorFlow's gradient at 0 (sigma'(0) = 0).  Other bits are rejected.
 * promp_num_params, promp_policy_layout and the workspace sizes do not depend on the activation. */
#define PROMP_HIDDEN_WIDTH_MASK 0xFF
#define PROMP_ACT_RELU 0x100
/* Output non-linearity of the mean (policies/networks/mlp.py: output_nonlinearity), in the same `hidden` argument: no flag =
 * identity, PROMP_OUT_TANH = mean = tanh(h2 W2 + b2).  It combines with either hidden activation (width | PROMP_ACT_RELU |
 * PROMP_OUT_TANH), at width 32 or 64, and does not change the layout or the workspace sizes either.  Bits 0x200 - 0x800
 * stay unknown (rejected). */
#define PROMP_OUT_TANH 0x1000
/* Number of hidden layers (policies/networks/mlp.py: len(hidden_sizes)), in the same `hidden` argument: a 3-bit field at
 * PROMP_HIDDEN_DEPTH_SHIFT.  No depth bits = two hidden layers, so every value above keeps its meaning; PROMP_HIDDEN_DEPTH(1)
 * and PROMP_HIDDEN_DEPTH(3) select one and three hidden layers of the same width (32 or 64), with any activation flags.
 * Field values 4..7 are rejected.  The depth changes the layout: a depth-L parameter vector is
 *   W0[Do,Hd] b0[Hd] {W_l[Hd,Hd] b_l[Hd]}_{l=1..L-1} W_out[Hd,Da] b_out[Da] log_std[Da]
 * (the reference's creation order: hidden_0 .. hidden_{L-1}, output, log_std), and promp_num_params, promp_policy_layout and
 * the workspace sizes count it.  Policies of depth 1 and 3 run CUDA-core kernels of their own; the chain entry point runs
 * their stages as one launch each. */
#define PROMP_HIDDEN_DEPTH_SHIFT 14
#define PROMP_HIDDEN_DEPTH_MASK 0x1C000
#define PROMP_HIDDEN_DEPTH(layers) ((layers) << PROMP_HIDDEN_DEPTH_SHIFT)
/* baseline kinds of promp_process_samples.  LINEAR_TIME (baselines/linear_baseline.py:109-126) fits [t, t^2, t^3, 1],
 * t = step / 100, and never reads obs; its coefficients are [M,4].  GIVEN: the caller supplies the per-sample baseline
 * values (promp_process_samples_given); no fit, no coefficients. */
enum { PROMP_BASELINE_ZERO = 0, PROMP_BASELINE_LINEAR_FEATURE = 1, PROMP_BASELINE_LINEAR_TIME = 2, PROMP_BASELINE_GIVEN = 3 };

const char* promp_last_error(void);
int promp_version(void);

/* Number of policy parameters P for (obs_dim, act_dim, hidden,hidden), or for the depth the `hidden` argument carries. */
int promp_num_params(int obs_dim, int act_dim, int hidden);
/* State floats per env for init_state / final_state: 2 (point envs; 4 = pos, vel for the momentum env), 18 (cheetah, walker:
 * qpos[9] qvel[9]), 10 (swimmer: qpos[5] qvel[5]). */
int promp_env_state_dim(int env_kind);
/* Floats per task in task_params: 2 (point corner / momentum goal), 0 -> pass 1 dummy (point), 1 (cheetah: direction or goal
 * velocity), 6 (walls: goal, gap_1, gap_2), 2 (walker: direction or goal velocity, then the reward mode 0 = Walker2DRandDirec
 * [dir * forward_vel + 1], 1 = Walker2DRandVel [-|forward_vel - goal| + 15]; reward_type is not read), 1 (swimmer: goal
 * velocity). */
int promp_env_task_dim(int env_kind);

/*
 * Fused vectorised rollout: MetaSampler.obtain_samples (samplers/meta_sampler.py:59-137) with
 * MetaIterativeEnvExecutor.reset/step (samplers/vectorized_env_executor.py:25-75),
 * MetaGaussianMLPPolicy.get_actions (policies/meta_gaussian_mlp_policy.py:99-157),
 * NormalizedEnv.step (envs/normalized_env.py:109-123) and the env's step/reward, for all H steps of
 * all M*E envs in one launch.  One warp per env; weights live in registers; trajectory records are
 * staged in shared memory and flushed as coalesced float32 rows.
 *
 *   normalize_actions           1 = env wrapped by NormalizedEnv (affine map from [-10,10] + clip, envs/normalized_env.py:109-117),
 *                               0 = raw env (only the env's own action clip)
 *   task_params [M, task_dim]   goal (x,y) / direction
 *   init_state  [M, E, state_dim] or NULL  -> NULL draws the reset state in-kernel (Philox4x32-10)
 *   noise       [M, E, H, Da]    or NULL  -> NULL draws N(0,1) action noise in-kernel
 *   seed, stream_id             Philox key / sub-stream (use a fresh stream_id per sampling phase)
 *   stream_id_dev               optional device uint64 whose value is ADDED to stream_id; the host bumps it with
 *                               promp_counter_add after each launch, so a captured CUDA graph replays the same
 *                               launch with fresh noise / reset states every time
 *   clip_reported_log_std       1 = pre-update mode: reported log_std = max(log_std, min_log_std)
 *                               (policies/gaussian_mlp_policy.py:71); sampling always uses the raw one
 * outputs (all written):
 *   obs [M,E,H,Do]  act [M,E,H,Da]  mean [M,E,H,Da]  rew [M,E,H]  done [M,E,H] (uint8)
 *   info [2,M,E,H]  (cheetah: reward_run, reward_ctrl; others: untouched, may be NULL)
 *        [3,M,E,H]  for the cheetah with reward_type 1 = HalfCheetahRandVel (mujoco_envs/half_cheetah_rand_vel.py:30-40:
 *                   reward_run = -|forward_vel - task|, task = goal velocity): third channel = forward_vel;
 *                   reward_type 0 = HalfCheetahRandDirec (reward_run = task * forward_vel, task = direction)
 *        [2,M,E,H]  swimmer (mujoco_envs/swimmer_rand_vel.py:30-39, reward_type 0): reward_fwd, reward_ctrl
 *   The walker records fixed-horizon trajectories here (done only at t = H-1, its fall rule is not applied); its
 *   early-terminating sampler is promp_rollout_early_term.
 *   log_std_out [M,Da]  the per-task reported log_std (constant over the phase)
 *   final_state [M,E,state_dim] or NULL
 */
int promp_rollout(int env_kind, int reward_type, float sparse_radius, int normalize_actions,
                  int M, int E, int H, int hidden,
                  const float* params, int64_t param_stride,
                  const float* task_params, const float* init_state, const float* noise,
                  uint64_t seed, uint64_t stream_id, const uint64_t* stream_id_dev,
                  int clip_reported_log_std, float min_log_std,
                  float* obs, float* act, float* mean, float* rew, uint8_t* done, float* info,
                  float* log_std_out, float* final_state, void* stream);

/*
 * promp_rollout_ex / promp_rollout_early_term_ex: promp_rollout / promp_rollout_early_term for one rank's shard of a larger
 * task batch.  task_offset = global index of the shard's first task (rank * M).  It changes only the Philox key of every
 * env, (task_offset + m) * E + e instead of m * E + e, so action noise, in-kernel reset states and the walker's fall
 * redraws are the ones the shard's tasks get in one launch over the whole batch (the reference samples every task of the
 * meta-batch in one process, samplers/meta_sampler.py:59-137).  All buffers stay local ([M, E, ...]).  task_offset = 0 is
 * the base entry point, bit for bit (the same kernel code).  Rejected: task_offset < 0, (task_offset + M) * E > 2^32 (the
 * 32-bit env key).
 */
int promp_rollout_ex(int env_kind, int reward_type, float sparse_radius, int normalize_actions,
                     int M, int E, int H, int hidden,
                     const float* params, int64_t param_stride,
                     const float* task_params, const float* init_state, const float* noise,
                     uint64_t seed, uint64_t stream_id, const uint64_t* stream_id_dev,
                     int clip_reported_log_std, float min_log_std,
                     float* obs, float* act, float* mean, float* rew, uint8_t* done, float* info,
                     float* log_std_out, float* final_state, void* stream, int task_offset);

/* *counter += inc on the stream (device-side phase counter for graph-replayed rollouts). */
int promp_counter_add(uint64_t* counter, uint64_t inc, void* stream);

/*
 * Set the tasks of a sampling phase: per_task [M, task_dim] = host_vec (host memory, read during the call) and, when
 * per_env is not NULL, per_env [M * E, task_dim] = each task's row repeated for its E envs.  The values travel in the
 * kernel arguments (960 per launch), so the call never waits for work already queued on the stream and host_vec may be
 * reused as soon as it returns.
 */
int promp_set_tasks(int M, int task_dim, int E, const float* host_vec, float* per_task, float* per_env, void* stream);

/*
 * One vectorised env step (MetaIterativeEnvExecutor.step, samplers/vectorized_env_executor.py:25-52)
 * for policies that are not device-resident: state [n_env, state_dim] is updated in place.
 *   actions [n_env, Da] policy-space actions (NormalizedEnv rescale+clip applied inside when normalize_actions = 1)
 *   task_params [n_env, task_dim] (already expanded per env)
 *   ts [n_env] int32 step counters, incremented; when ts reaches H (or the env is done) the env is
 *   reset from reset_state [n_env, state_dim] (caller-provided fresh reset states) and ts = 0.
 *   next_obs [n_env, Do], rew [n_env], done [n_env] uint8, info [2, n_env] or NULL
 */
int promp_env_step(int env_kind, int reward_type, float sparse_radius, int normalize_actions, int n_env, int H,
                   float* state, int32_t* ts, const float* actions, const float* task_params,
                   const float* reset_state, float* next_obs, float* rew, uint8_t* done, float* info,
                   void* stream);

/* obs [n_env, Do] from state [n_env, state_dim] (env.reset observation). */
int promp_env_observe(int env_kind, int n_env, const float* state, float* obs, void* stream);

/*
 * Early-terminating envs in the fused rollout (MetaPointEnv, envs/point_envs/point_env_2d.py:9-59: done when the point is
 * within 0.01 of the origin; tests/test_integration.py) - replaces the reference's collect-until-enough loop
 * (samplers/meta_sampler.py:87-137 with vectorized_env_executor.py:25-52) without one host round trip per env step:
 *
 * promp_rollout_early_term: like promp_rollout, but every env slot records a TIMELINE of `timeline_len` steps
 *   (obs/act/mean [M,E,T,.], rew [M,E,T], done [M,E,T] u8); a path ends when the env reports done or after `horizon` steps;
 *   the slot is reset at once (U(-2,2)^2 from Philox keyed by (env, step) - the host numpy stream cannot be followed when the
 *   number of resets is data-dependent) and the next recorded observation is the reset state.  env_kind PROMP_ENV_POINT or
 *   PROMP_ENV_WALKER (walker2d_rand_*.py: done when the torso falls; reset = init_qpos + U(-.005,.005)^9, U(-.005,.005)^9
 *   from Philox keyed by (env, step, coordinate); task_params [M, 2] select the reward mode).  timeline_len >= 2*horizon - 1
 *   guarantees that promp_paths_finalize finds enough completed samples.
 * promp_paths_finalize: applies the reference's rule to the timelines: t* = first step at which the paths completed so far
 *   hold >= target_samples (= M*E*H, > 0) samples; task m keeps the paths completing at steps <= t*, in (step, env index)
 *   order (meta_sampler.py:116-125); unfinished paths are dropped.  Outputs the per-task path table of
 *   promp_process_samples_ragged (path_off [M, max_paths+1], n_paths [M], n_valid [M]; max_paths >= E*timeline_len is always
 *   enough; a task with more paths keeps its first max_paths in that order, and n_valid and the closing and padding offsets
 *   count only their samples, while cut_out still reports where the rule stopped) and the compacted ragged tensors
 *   obs/act/mean [M, max_samples, .], rew, done [M, max_samples]
 *   (max_samples >= E*timeline_len).  src_slot / src_start [M, max_paths]: where every path came from.  cut_out int32[2] =
 *   {t*, target reached}.  workspace: promp_paths_workspace_bytes, zero-filled before first use (left zero).
 */
int promp_rollout_early_term(int env_kind, int normalize_actions, int M, int E, int timeline_len, int horizon, int hidden,
                             const float* params, int64_t param_stride, const float* task_params, const float* init_state,
                             const float* noise, uint64_t seed, uint64_t stream_id, const uint64_t* stream_id_dev,
                             int clip_reported_log_std, float min_log_std, float* obs, float* act, float* mean, float* rew,
                             uint8_t* done, float* log_std_out, void* stream);
int64_t promp_paths_workspace_bytes(int M, int E, int timeline_len);
int promp_paths_finalize(int M, int E, int timeline_len, int max_paths, int max_samples, int obs_dim, int act_dim,
                         int64_t target_samples, const uint8_t* t_done, const float* t_obs, const float* t_act, const float* t_mean,
                         const float* t_rew, int32_t* path_off, int32_t* n_paths, int32_t* n_valid, int32_t* src_slot,
                         int32_t* src_start, float* obs, float* act, float* mean, float* rew, uint8_t* done, int32_t* cut_out,
                         void* workspace, int64_t workspace_bytes, void* stream);

/*
 * The cut over a task batch sharded across ranks.  The reference stops when the completed paths of ALL tasks of the
 * meta-batch hold meta_batch_size*E*H samples (samplers/meta_sampler.py:87-137), so t* is a property of the whole batch,
 * not of one shard:
 * promp_rollout_early_term_ex: the shard's timelines, keyed by global env index (see promp_rollout_ex).
 * promp_paths_histogram: hist[t] += samples of this shard's paths completing at step t (hist int32 [timeline_len], the
 *   caller zeroes it; the counts add, so the sum over shards - e.g. an all-reduce - is the histogram of the whole batch).
 * promp_paths_finalize_ex: promp_paths_finalize with hist_in.  hist_in != NULL: t* = first step at which the cumulative
 *   sum of hist_in reaches target_samples (the global target, world*M*E*H); hist_in is only read and the workspace is
 *   not touched.  The table and compaction are per task and take this shard's timelines.  hist_in == NULL: exactly
 *   promp_paths_finalize.
 */
int promp_rollout_early_term_ex(int env_kind, int normalize_actions, int M, int E, int timeline_len, int horizon, int hidden,
                                const float* params, int64_t param_stride, const float* task_params, const float* init_state,
                                const float* noise, uint64_t seed, uint64_t stream_id, const uint64_t* stream_id_dev,
                                int clip_reported_log_std, float min_log_std, float* obs, float* act, float* mean, float* rew,
                                uint8_t* done, float* log_std_out, void* stream, int task_offset);
int promp_paths_histogram(int M, int E, int timeline_len, const uint8_t* t_done, int32_t* hist, void* stream);

/*
 * Users' own environments (promp_b200.envs.CudaMetaEnv): an env struct compiled at run time by NVRTC into the same fused
 * rollout, env-step and env-observe kernels as the built-in envs (csrc/user_env.cuh, promp_b200/_jit.py).
 *
 * promp_env_module_load: loads the cubin `image` (`bytes` long) and resolves its kernels by their lowered names.
 *   names [PROMP_ENV_MODULE_SLOTS]: slot PROMP_ENV_SLOT_STEP = env_step_kernel, PROMP_ENV_SLOT_OBSERVE = env_observe_kernel,
 *   PROMP_ENV_SLOT_ROLLOUT + 2*v + keyed = rollout_kernel of `hidden` variant v = (relu + 2*out_tanh)*2 + (width == 64),
 *   keyed = the sharded (task_offset != 0) instantiation; PROMP_ENV_SLOT_ROLLOUT_DEEP + 2*v + keyed = rollout_deep_kernel, the
 *   same variants at depth 1 or 3 (PROMP_HIDDEN_DEPTH).  NULL or "" = not compiled; launching it returns
 *   PROMP_ERR_INVALID_ARG.  dims [PROMP_ENV_MODULE_NDIMS] = {obs, act, state, task sizes, info channels, ends early}; obs
 *   1..19, act 1..8 (the rollout policy's range), info 0..3.  *handle_out: the module, until promp_env_module_unload.
 *   There is no reference counterpart (the reference steps Python envs, envs/base.py:6-49).
 * promp_rollout_module: promp_rollout_ex (samplers/meta_sampler.py:59-137 with vectorized_env_executor.py:25-52) for the
 *   module's env.  info [NINFO, M, E, H] is required when the env writes info channels (channel c as the env wrote it).
 *   Rejects an env that ends early.
 * promp_rollout_early_term_module: promp_rollout_early_term_ex (the same reference loop with early `done`) for a module
 *   whose env ends early; in-kernel resets call the env's reset with Philox draws keyed by (env, step).  The timelines go
 *   to promp_paths_finalize / promp_paths_finalize_ex unchanged.
 * promp_env_step_module / promp_env_observe_module: promp_env_step / promp_env_observe (MetaIterativeEnvExecutor.step /
 *   reset, vectorized_env_executor.py:25-75) for the module's env; info [NINFO, n_env] or NULL.
 */
#define PROMP_ENV_MODULE_SLOTS 34
#define PROMP_ENV_MODULE_NDIMS 6
#define PROMP_ENV_SLOT_STEP 0
#define PROMP_ENV_SLOT_OBSERVE 1
#define PROMP_ENV_SLOT_ROLLOUT 2
#define PROMP_ENV_SLOT_ROLLOUT_DEEP 18
int promp_env_module_load(const void* image, int64_t bytes, const char* const* names, int n_names, const int* dims,
                          void** handle_out);
int promp_env_module_unload(void* handle);
int promp_rollout_module(void* module, int reward_type, float sparse_radius, int normalize_actions, int M, int E, int H,
                         int hidden, const float* params, int64_t param_stride, const float* task_params, const float* init_state,
                         const float* noise, uint64_t seed, uint64_t stream_id, const uint64_t* stream_id_dev,
                         int clip_reported_log_std, float min_log_std, float* obs, float* act, float* mean, float* rew,
                         uint8_t* done, float* info, float* log_std_out, float* final_state, void* stream, int task_offset);
int promp_rollout_early_term_module(void* module, int normalize_actions, int M, int E, int timeline_len, int horizon, int hidden,
                                    const float* params, int64_t param_stride, const float* task_params, const float* init_state,
                                    const float* noise, uint64_t seed, uint64_t stream_id, const uint64_t* stream_id_dev,
                                    int clip_reported_log_std, float min_log_std, float* obs, float* act, float* mean,
                                    float* rew, uint8_t* done, float* log_std_out, void* stream, int task_offset);
int promp_env_step_module(void* module, int reward_type, float sparse_radius, int normalize_actions, int n_env, int H,
                          float* state, int32_t* ts, const float* actions, const float* task_params, const float* reset_state,
                          float* next_obs, float* rew, uint8_t* done, float* info, void* stream);
int promp_env_observe_module(void* module, int n_env, const float* state, float* obs, void* stream);
/* CUDART_VERSION the library was built with (e.g. 12090): the JIT prefers an NVRTC of the same version, whose code for
 * the built-in env types is then the library's own. */
int promp_cuda_build_version(void);
int promp_paths_finalize_ex(int M, int E, int timeline_len, int max_paths, int max_samples, int obs_dim, int act_dim,
                            int64_t target_samples, const int32_t* hist_in, const uint8_t* t_done, const float* t_obs,
                            const float* t_act, const float* t_mean, const float* t_rew, int32_t* path_off, int32_t* n_paths,
                            int32_t* n_valid, int32_t* src_slot, int32_t* src_start, float* obs, float* act, float* mean,
                            float* rew, uint8_t* done, int32_t* cut_out, void* workspace, int64_t workspace_bytes,
                            void* stream);

/*
 * MetaSampleProcessor.process_samples (samplers/meta_sample_processor.py:8-49 ->
 * samplers/base.py:99-133): per task discounted returns (utils/utils.py:74-81), LinearFeatureBaseline
 * fit (baselines/linear_baseline.py:55-77, features :101-106) + predict (:17-33), GAE
 * (samplers/base.py:151-162), per-task advantage normalisation / positive shift
 * (utils/utils.py:59-71), path statistics (samplers/base.py:135-149).  One CTA per task; the Gram
 * matrix, solve, scans and moments run in float64 like the reference's numpy.
 *
 *   obs [M,E,H,Do]  rew [M,E,H]
 *   baseline_kind: PROMP_BASELINE_ZERO, _LINEAR_FEATURE or _LINEAR_TIME (LinearTimeBaseline, linear_baseline.py:109-126:
 *           the same fit and predict over the features [t, t^2, t^3, 1]; obs is not read)
 * outputs:
 *   returns [M,E,H]  adv [M,E,H]
 *   coeffs  [M,F] float64, F = 2*Do+4 (LINEAR_FEATURE) or 4 (LINEAR_TIME) (may be NULL)
 *   stats   [M,8] float64: sum R_0, sum G, sum G^2, max G, min G (G = undiscounted return per path),
 *           sum r, sum r^2, reg_coeff finally used            (may be NULL)
 *   workspace: scratch, >= promp_process_workspace_bytes(M,E,H,Do) bytes.  It must be ZERO-FILLED before its first
 *           use (per-task arrival tickets live at its start); every call leaves it ready for the next one.
 * One launch: grid (chunks of a task's trajectories, M); the last CTA of a task to arrive finishes the task
 * (fit / predict / GAE / normalisation).
 */
int64_t promp_process_workspace_bytes(int M, int E, int H, int obs_dim);
int promp_process_samples(int M, int E, int H, int obs_dim, const float* obs, const float* rew,
                          double discount, double gae_lambda, double reg_coeff, int baseline_kind,
                          int normalize_adv, int positive_adv,
                          float* returns, float* adv, double* coeffs, double* stats,
                          void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Variable-length paths (early termination: samplers/meta_sampler.py:116-125 appends a path whenever an env reports
 * `done`, envs/point_envs/point_env_2d.py:49-53): the same computation over a per-task PATH TABLE instead of E x H.
 * Task m owns n_paths[m] <= max_paths paths stored back to back; path e covers samples
 * [path_off[m][e], path_off[m][e+1]) of the task's row (path_off [M, max_paths+1] int32 prefix sums, path_off[m][0] = 0);
 * the baseline's time feature restarts at 0 in every path (baselines/linear_baseline.py:101-106).
 *   obs [M,max_samples,Do]  rew [M,max_samples]   (rows past path_off[m][n_paths[m]] are padding)
 *   returns / adv [M,max_samples]: padding rows of adv are written as 0
 *   stats as above (per-path sums run over n_paths[m] paths)
 */
int64_t promp_process_workspace_bytes_ragged(int M, int max_paths, int max_samples, int obs_dim);
int promp_process_samples_ragged(int M, int max_paths, int max_samples, int obs_dim, const float* obs, const float* rew,
                                 const int32_t* path_off, const int32_t* n_paths, double discount, double gae_lambda,
                                 double reg_coeff, int baseline_kind, int normalize_adv, int positive_adv,
                                 float* returns, float* adv, double* coeffs, double* stats,
                                 void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Any baseline object (samplers/base.py:99-108 accepts whatever has fit / predict): the caller fitted it and evaluated
 * predict(path) itself; the kernel takes those values and runs everything downstream of the reference's predict exactly
 * as above (discounted returns, GAE, normalisation / positive shift, stats).  PROMP_BASELINE_GIVEN.
 *   baseline_values [M,NS] float64 device memory in the phase's sample layout (NS = E*H, or max_samples on the ragged
 *   layout, where positions past path_off[m][n_paths[m]] are not read).  No coefficients are written; stats[m][7] = 0.
 *   The workspace is the one of promp_process_workspace_bytes / _ragged for the same shape.
 */
int promp_process_samples_given(int M, int E, int H, int obs_dim, const float* obs, const float* rew,
                                const double* baseline_values, double discount, double gae_lambda, int normalize_adv,
                                int positive_adv, float* returns, float* adv, double* stats,
                                void* workspace, int64_t workspace_bytes, void* stream);
int promp_process_samples_ragged_given(int M, int max_paths, int max_samples, int obs_dim, const float* obs, const float* rew,
                                       const int32_t* path_off, const int32_t* n_paths, const double* baseline_values,
                                       double discount, double gae_lambda, int normalize_adv, int positive_adv,
                                       float* returns, float* adv, double* stats,
                                       void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Launch geometry of the processing kernel for one shape, computed on the host (no CUDA call).  It replaces no reference
 * function: it exists so that tests can name the code path a shape exercises.  Fixed horizon (ragged = 0): max_paths = E,
 * NS = E*H, as in promp_process_samples.  Variable-length paths (ragged = 1): max_paths and NS = max_samples as in
 * promp_process_samples_ragged (promp_baseline_fit: M = 1, max_paths = n_paths, NS = n_samples); H is ignored.
 *   out [8] host int32: C (trajectory chunks per task), EPC (trajectories per chunk), chunk_cap, finish_cap (samples the
 *   front / finish stage stages in shared memory; 0 = float64 workspace), tt_cap (steps covered by the t/100 table),
 *   pred_tile, stage_f, stage_l (1 = that stage keeps its sample arrays in shared memory).
 */
int promp_process_launch_info(int M, int max_paths, int H, int obs_dim, int NS, int ragged, int32_t* out);

/*
 * Standalone LinearFeatureBaseline (baselines/linear_baseline.py): fit(paths, target_key) (:55-77) and predict(path)
 * (:17-33) for a flat list of n_paths paths stored back to back (path e = samples [path_off[e], path_off[e+1]), path_off
 * [n_paths+1] int32 device memory; the time feature restarts at 0 in every path, :101-106).
 *   fit:     obs [n_samples,Do] float32, target [n_samples] float64 (the caller's path[target_key]) ->
 *            coeffs [F] float64, F = 2*Do+4; *reg_used (device float64, may be NULL) = ridge finally used by the
 *            reference's x10-on-NaN retry rule.  workspace: zero-filled before first use, like promp_process_samples.
 *   predict: out [n_samples] float64 = features . coeffs
 */
int64_t promp_baseline_fit_workspace_bytes(int n_paths, int n_samples, int obs_dim);
int promp_baseline_fit(int n_paths, int n_samples, int obs_dim, const float* obs, const double* target,
                       const int32_t* path_off, double reg_coeff, double* coeffs, double* reg_used,
                       void* workspace, int64_t workspace_bytes, void* stream);
int promp_baseline_predict(int n_paths, int n_samples, int obs_dim, const float* obs, const int32_t* path_off,
                           const double* coeffs, double* out, void* stream);
/*
 * The same fit / predict for either linear baseline (baselines/linear_baseline.py:55-77, 17-33): kind =
 * PROMP_BASELINE_LINEAR_FEATURE (features :101-106, exactly promp_baseline_fit / _predict) or PROMP_BASELINE_LINEAR_TIME
 * (LinearTimeBaseline, features :122-126: [t, t^2, t^3, 1], coeffs [4]; obs is not read and may be NULL).  The workspace
 * is sized by promp_baseline_fit_workspace_bytes for both kinds.
 */
int promp_baseline_fit_ex(int kind, int n_paths, int n_samples, int obs_dim, const float* obs, const double* target,
                          const int32_t* path_off, double reg_coeff, double* coeffs, double* reg_used,
                          void* workspace, int64_t workspace_bytes, void* stream);
int promp_baseline_predict_ex(int kind, int n_paths, int n_samples, int obs_dim, const float* obs, const int32_t* path_off,
                              const double* coeffs, double* out, void* stream);

/*
 * Fused outer update of one Adam epoch (optimizers/maml_first_order_optimizer.py:82-115 with the task mean of
 * meta_algos/pro_mp.py:151-155 and, for world > 1, the all-reduce of SURVEY.md section 8e): per-task meta-gradients
 * task_grads [M, P] -> grad = scale * sum_m task_grads[m] (scale = 1 / (M * world)) -> rank-ordered sum over ranks through the
 * NVLink peer buffers of promp_comm_alloc -> TF1 Adam on theta / m / v with the device step counter (incremented once).
 * One launch of ceil(P / 256) CTAs; each CTA exchanges its own 256-parameter slice (no grid-wide barrier).  world == 1:
 * peers / epoch / error may be NULL.  `ticket_dev`: one zero-initialised uint32 of device memory (left zero).
 * grad_out (may be NULL) receives the reduced meta-gradient.  A missing peer (2 s time-out) sets *error_flag and poisons
 * the gradient with NaN.
 */
int promp_meta_update(int M, int P, const float* task_grads, float scale, float* grad_out, float* theta, float* m, float* v,
                      int32_t* step, float lr, float beta1, float beta2, float eps, int world, int rank, int capacity_floats,
                      void* const* peers_dev, uint32_t* epoch_dev, uint32_t* error_flag_dev, uint32_t* ticket_dev, void* stream);

/*
 * Meta-SGD (trainable per-parameter inner step sizes alpha [P], shared by all tasks and inner steps): the fused outer update
 * over the concatenated gradient [theta; alpha] (2P values).  Per element,
 *   grad_theta = scale * sum_m task_grads[m]                                (as promp_meta_update)
 *   grad_alpha = -scale * sum_m sum_s lam[s][m] * g[s][m]
 * where, for inner step s, lam[s] [M, P] is the direction that enters the Hessian-vector stage of step s and g[s] [M, P] is
 * the inner gradient of step s (theta_{s+1} = theta_s - alpha * g[s]); lam / g are HOST arrays of n_pairs (0..6) device
 * pointers.  Then ONE exchange of the 2P values over the peer buffers (world > 1, capacity >= 2P) and TF1 Adam on theta
 * (slots m, v) and alpha (slots m_alpha, v_alpha) with one step counter, incremented once.  grad_out [2P] or NULL.
 * grad_in [2P] non-NULL: the summed gradient is given (world must be 1; task_grads / lam / g are not read) and only Adam runs:
 * the NCCL path, after promp_reduce_tasks_sgd and an all-reduce.
 * promp_reduce_tasks_sgd: out [2P] = the local [grad_theta; grad_alpha] above; task_grads NULL: only out[P, 2P) (alpha).
 * n_pairs = 0 (no inner step) gives a zero alpha gradient.
 */
int promp_reduce_tasks_sgd(int M, int P, const float* task_grads, int n_pairs, const float* const* lam, const float* const* g,
                           float scale, float* out, void* stream);
int promp_meta_update_sgd(int M, int P, const float* task_grads, int n_pairs, const float* const* lam, const float* const* g,
                          const float* grad_in, float scale, float* grad_out, float* theta, float* alpha, float* m, float* v,
                          float* m_alpha, float* v_alpha, int32_t* step, float lr, float beta1, float beta2, float eps, int world,
                          int rank, int capacity_floats, void* const* peers_dev, uint32_t* epoch_dev, uint32_t* error_flag_dev,
                          uint32_t* ticket_dev, void* stream);

/* promp_meta_loss_terms with the sum over ranks fused in (world >= 2): local means -> peer exchange -> rank-ordered sum ->
 * KL penalty.  One launch instead of terms + all-reduce + elementwise glue. */
int promp_meta_loss_terms_p2p(int S, int M, const float* stats_all, float inv_m_global, const float* coeff, int n_out, float* out,
                              int world, int rank, int capacity_floats, void* const* peers_dev, uint32_t* epoch_dev,
                              uint32_t* error_flag_dev, void* stream);

/*
 * Device-resident ConjugateGradientOptimizer (optimizers/conjugate_gradient_optimizer.py:239-354) on flat float32 parameter
 * vectors [n]; one CTA each, dot products accumulated in float64 in a fixed order.  `scal` is a device float[4]:
 * [0] r.r  [1] converged flag  [2] beta  [3] beta-is-NaN flag.
 *   promp_vec_axpy    out = y + a*x                      (theta +- eps*p, theta - ratio^k*step; :73-82, :277-279)
 *   promp_cg_init     p = r = g, x = 0, r.r              (:325-331)
 *   promp_cg_step     z = (grad_plus - grad_minus)/two_eps + reg*p  (FiniteDifferenceHvp.Hx, :59-89, :101-104), then one
 *                     CG iteration (:337-349); a no-op once r.r < residual_tol (:350-351)
 *   promp_trpo_step   beta = sqrt(2*delta / (x.Hx(x) + 1e-8)), step = beta*x  (:262-269)
 *   promp_trpo_select verdict of the backtracking line search (:274-300) over candidates k0..k0+K-1 whose
 *                     [loss, ..., kl] rows (n_terms floats, promp_meta_loss_terms layout) are in `terms` and whose
 *                     parameter vectors are in `candidates` [K][n]: theta_out = accepted candidate, or theta_prev when the
 *                     step is rejected; untouched while undecided.
 *                     result float[8]: loss_before, kl_before, loss_after, kl_after, accepted k (-1), rejected, need_more, beta
 */
int promp_vec_axpy(int n, float a, const float* x, const float* y, float* out, void* stream);
int promp_cg_init(int n, const float* g, float* p, float* r, float* x, float* scal, void* stream);
int promp_cg_step(int n, const float* grad_plus, const float* grad_minus, float two_eps, float reg_coeff, float* p, float* r,
                  float* x, float* scal, float residual_tol, void* stream);
int promp_trpo_step(int n, const float* grad_plus, const float* grad_minus, float two_eps, float reg_coeff, const float* x,
                    float max_constraint, float* step, float* scal, void* stream);
int promp_trpo_select(int n, int n_candidates, int n_terms, int k0, int max_backtracks, const float* terms,
                      const float* base_terms, float max_constraint, const float* theta_prev, const float* candidates,
                      const float* scal, float* theta_out, float* result, void* stream);

/* adj_avg_rewards = (r - mean_all)/(std_all + 1e-8) (samplers/meta_sample_processor.py:40-44);
 * mean/std are passed by the caller (reduced over all tasks / ranks from `stats`). */
int promp_adj_avg_rewards(int64_t n, const float* rew, double mean, double std, float* out, void* stream);

/*
 * E-MAML coefficient (trpo_maml.py:137-144 with samplers/meta_sample_processor.py:40-44): the task mean of adj_avg_rewards,
 *   c_m = (mean_m r - mean_all) / (std_all + 1e-8),   mean / std over the rewards of every task (population std),
 * from the per-task sums stats[m][5] = sum r, stats[m][6] = sum r^2 of promp_process_samples(_ragged) ([M,8] float64).
 * Every mean covers a task's valid samples: n_m = n_valid[m] ([M] int32 device memory) or N when n_valid is NULL.
 * Totals are float64 sums in task order; c is written as float32 [M].  One launch, no host arithmetic (capturable).
 * Several ranks: promp_emaml_totals writes this rank's [sum r, sum r^2, sum n] (float64 [3]); sum them over ranks, then
 * promp_emaml_finish computes c from the summed totals.
 */
int promp_emaml_coeff(int M, const double* stats, const int32_t* n_valid, int N, float* coeff, void* stream);
int promp_emaml_totals(int M, const double* stats, const int32_t* n_valid, int N, double* totals, void* stream);
int promp_emaml_finish(int M, const double* stats, const int32_t* n_valid, int N, const double* totals, float* coeff,
                       void* stream);

/*
 * Per-task objective value, KL and gradient w.r.t. the task's parameter set, optionally fused with
 * the inner SGD step.  Covers
 *   - MAMLAlgo._adapt        (meta_algos/base.py:217-242, graph :158-215): obj RATIO|LOGLIK,
 *                            out_params = params - inner_lr * grad
 *   - the step-s surrogate / clipped outer objective and KL terms of ProMP.build_graph
 *                            (meta_algos/pro_mp.py:88-163) and TRPOMAML.build_graph
 *                            (meta_algos/trpo_maml.py:100-159)
 *   - DiagonalGaussian.log_likelihood_sym / likelihood_ratio_sym / kl_sym
 *                            (policies/distributions/diagonal_gaussian.py:16-109)
 *   - forward_mlp            (policies/networks/mlp.py:65-119)
 * Objective_m = obj_scale * surr_kind(m) + kl_coeff * mean_n KL(old || new)(m).
 * obj_kind PROMP_OBJ_EXPLORE: adv is [M], one weight per task (the E-MAML coefficient), and the objective is LOGLIK's.
 *
 *   obs [M,N,Do] act [M,N,Da] adv [M,N] old_mean [M,N,Da]
 *   old_log_std: [M,Da] if ls_per_sample == 0 else [M,N,Da]
 *   clip_log_std: 1 = evaluate with max(log_std, min_log_std) and mask its gradient (the
 *                 distribution_info_sym(params=None) path, policies/gaussian_mlp_policy.py:71,161)
 * outputs:
 *   grad       [M,P] or NULL (NULL = values only)
 *   out_params [M,P] or NULL: params_m - sgd_lr * grad_m      (needs grad != NULL)
 *   stats      [M,4]: surrogate value (unscaled), mean KL(old||new), mean ratio, unused
 *   workspace  >= promp_policy_workspace_bytes(M,N,Do,Da,hidden) bytes
 */
int64_t promp_policy_workspace_bytes(int M, int N, int obs_dim, int act_dim, int hidden);
int promp_policy_grad(int obs_dim, int act_dim, int hidden, int M, int N,
                      const float* params, int64_t param_stride,
                      const float* obs, const float* act, const float* adv,
                      const float* old_mean, const float* old_log_std, int ls_per_sample,
                      int obj_kind, float obj_scale, float clip_eps, float kl_coeff,
                      int clip_log_std, float min_log_std,
                      float* grad, float* out_params, float sgd_lr, float* stats,
                      void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Second-order term of the MAML meta-gradient for one inner step
 * (tf.gradients through _adapt_sym, meta_algos/base.py:192-215 with pro_mp.py:103,117):
 *   out_m = vec_m - inner_lr * H_m(params_m) vec_m + kl_coeff * grad_theta mean KL(old||new)(m)
 * where H_m is the Hessian of the inner surrogate (obj RATIO or LOGLIK) of task m on (obs, act, adv,
 * old dist) evaluated at params_m, computed exactly (forward-over-reverse through the tanh MLP and
 * the Gaussian log-likelihood), not by finite differences.
 *   vec [M,P], out [M,P] (may alias vec); stats [M,4] as in promp_policy_grad (surr, KL) or NULL
 */
int promp_policy_hvp(int obs_dim, int act_dim, int hidden, int M, int N,
                     const float* params, int64_t param_stride,
                     const float* obs, const float* act, const float* adv,
                     const float* old_mean, const float* old_log_std, int ls_per_sample,
                     int obj_kind, float inner_lr, float kl_coeff,
                     int clip_log_std, float min_log_std,
                     const float* vec, float* out, float* stats,
                     void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Variable-length paths: the same two kernels with a per-task valid-sample count.  Task m's rows [n_valid[m], N) of
 * obs / act / adv / old_mean are padding and contribute nothing; every per-task mean (objective, KL, gradients) is
 * taken over n_valid[m] samples, as tf.reduce_mean over the task's concatenated paths does in the reference
 * (meta_algos/pro_mp.py:59-65, 135-147; samplers/meta_sample_processor.py:36-47).  n_valid [M] int32, device memory.
 */
int promp_policy_grad_ragged(int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid,
                             const float* params, int64_t param_stride,
                             const float* obs, const float* act, const float* adv,
                             const float* old_mean, const float* old_log_std, int ls_per_sample,
                             int obj_kind, float obj_scale, float clip_eps, float kl_coeff,
                             int clip_log_std, float min_log_std,
                             float* grad, float* out_params, float sgd_lr, float* stats,
                             void* workspace, int64_t workspace_bytes, void* stream);

/*
 * promp_policy_grad_ragged plus launch re-use (n_valid may be NULL): the inner pass of the first Adam epoch of
 * optimize_policy repeats MAMLAlgo._adapt exactly - same theta, same phase-0 data - unless the reported-log_std clip of the
 * step-0 graph (policies/gaussian_mlp_policy.py:71) is active.
 *   producer (the _adapt launch): unclipped_out (device int32) = 1 iff every log_std component >= min_log_std;
 *                                 theta_copy_out [P] = the parameters the launch used.
 *   consumer (epoch-1 inner pass, SAME output buffers as the producer): if *skip_flag != 0 and params == skip_theta bit for bit
 *                                 the whole grid returns at once (its outputs are already correct); else it runs normally.
 * Both pairs may be NULL; only defined for param_stride == 0.
 */
int promp_policy_grad_ex(int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid, const float* params,
                         int64_t param_stride, const float* obs, const float* act, const float* adv, const float* old_mean,
                         const float* old_log_std, int ls_per_sample, int obj_kind, float obj_scale, float clip_eps,
                         float kl_coeff, int clip_log_std, float min_log_std, float* grad, float* out_params, float sgd_lr,
                         float* stats, const int32_t* skip_flag, const float* skip_theta, int32_t* unclipped_out,
                         float* theta_copy_out, void* workspace, int64_t workspace_bytes, void* stream);
/*
 * The gradient chain of one meta-objective evaluation in ONE launch (tf.gradients through the M per-task sub-graphs of
 * meta_algos/base.py:158-215 + the outer objective of pro_mp.py:88-163 / trpo_maml.py:69-159):
 *   stage 0..S-2  kind 0, inner objective, grad + out_params (theta_{s+1,m} = theta_{s,m} - sgd_lr * grad)     = promp_policy_grad
 *   stage S-1     kind 0, outer objective at the adapted parameters, grad = v (or NULL: values only)          = promp_policy_grad
 *   stage S..     kind 1, v <- v - inner_lr * H_s v + kl_coeff * grad KL_s   for s = S-2 .. 0                 = promp_policy_hvp
 * Stage k of task m depends on stage k-1 of the same task only (its params / vec may be the out_params / grad / out of the
 * previous stage); a persistent dataflow kernel pulls (stage, task, tiles) work items from a device-side queue and lets the
 * stages of different tasks overlap.  Each stage has the semantics and argument meaning of the stand-alone entry point named
 * above (per-task sums are taken in a different, still deterministic, order).  skip_flag / skip_theta: launch re-use for
 * stage 0, as in promp_policy_grad_ex.  Shapes without tensor-core kernels (hidden != 64) and promp_set_option("chain", 0)
 * run the stages as separate launches.  The workspace (>= promp_policy_chain_workspace_bytes) starts with control words
 * that must be zero before the first call and are left zero: allocate it zero-filled once and do not share it with other
 * entry points.  A call whose M differs from the previous call's on the same workspace clears the control words on the
 * stream first, so one workspace serves chains of any M and stage count, on either path (the record of the last M is kept
 * on the host: a workspace a captured CUDA graph uses is not used with another M outside that graph).  `stages` is a HOST
 * array (read during the call).
 */
typedef struct {
    int32_t kind;                  /* 0 = gradient stage, 1 = Hessian-vector stage */
    int32_t N;                     /* samples per task of this stage's phase */
    const int32_t* n_valid;        /* [M] or NULL (variable-length paths) */
    const float* params;
    int64_t param_stride;
    const float *obs, *act, *adv, *old_mean, *old_log_std;
    int32_t ls_per_sample, obj_kind;   /* PROMP_OBJ_EXPLORE: last stage only, param_stride 0, no out_params; its items
                                          wait for no other stage */
    float obj_scale, clip_eps, kl_coeff;
    int32_t clip_log_std;
    float* grad;                   /* gradient stage */
    float* out_params;
    float sgd_lr;
    float inner_lr;                /* HVP stage */
    const float* vec;
    float* out;
    float* stats;                  /* [M,4] or NULL */
    const float* kl_coeff_dev;     /* NULL, or a device float: the stage uses kl_coeff * (*kl_coeff_dev) (device-resident
                                      adaptive coefficient, see promp_adapt_kl_coeff) */
    const float* step_size;        /* NULL, or per-parameter inner step sizes alpha [P] (device; Meta-SGD,
                                      trainable_inner_step_size): a gradient stage writes out_params = params - alpha * grad
                                      (sgd_lr unused); an HVP stage computes vec - inner_lr * H (alpha * vec) + kl_coeff * grad KL
                                      (pass inner_lr = 1) */
} promp_policy_stage;
int64_t promp_policy_chain_workspace_bytes(int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                           const promp_policy_stage* stages);
/* kernels promp_policy_chain launches for these stages with the current options: 1 (dataflow kernel) or n_stages */
int promp_policy_chain_num_launches(int obs_dim, int act_dim, int hidden, int M, int n_stages, const promp_policy_stage* stages);
/*
 * The work-item plan of the dataflow kernel for these stages under the current chain_q / chain_taper options (reads only
 * `kind` and `N` of each stage; no device work).  out[0] = SMs the plan is made for, out[1] = items in all, then 15 ints per
 * stage: ntiles, item_base, n_items, n_regions, reg_m0[4], reg_q[3], reg_item0[3], kind.  Region r is tasks
 * [reg_m0[r], reg_m0[r+1]) at reg_q[r] tiles per item, its first item at stage-relative id reg_item0[r].  Whether the
 * dataflow kernel runs is promp_policy_chain_num_launches's answer.
 */
int promp_policy_chain_plan_info(int M, int n_stages, const promp_policy_stage* stages, int32_t* out);
int promp_policy_chain(int obs_dim, int act_dim, int hidden, int M, float min_log_std, int n_stages,
                       const promp_policy_stage* stages, const int32_t* skip_flag, const float* skip_theta,
                       void* workspace, int64_t workspace_bytes, void* stream);
int promp_policy_hvp_ragged(int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid,
                            const float* params, int64_t param_stride,
                            const float* obs, const float* act, const float* adv,
                            const float* old_mean, const float* old_log_std, int ls_per_sample,
                            int obj_kind, float inner_lr, float kl_coeff,
                            int clip_log_std, float min_log_std,
                            const float* vec, float* out, float* stats,
                            void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Scalars of one meta-objective evaluation (optimizers/maml_first_order_optimizer.py:146-163 compute_stats; the
 * objective of meta_algos/pro_mp.py:151-155) from the stats rows the policy kernels wrote:
 *   stats_all [S, M, 4]: row s < S-1 = inner step s (surr, KL, ...), row S-1 = outer objective (surr, KL, ...)
 *   out[0] = mean_m surr_{S-1,m} (+ mean_s coeff[s] * inner_kl_s if coeff != NULL), out[1..S-1] = mean inner KLs,
 *   out[S] = mean outer KL; means use inv_m_global = 1 / (M * world size); only the first n_out values are stored.
 */
int promp_meta_loss_terms(int S, int M, const float* stats_all, float inv_m_global, const float* coeff, int n_out,
                          float* out, void* stream);

/* out[P] = scale * sum_m in[m,P]   (mean over tasks of the meta objective, pro_mp.py:151-155). */
int promp_reduce_tasks(int M, int P, const float* in, float scale, float* out, void* stream);
/* out[P] = scale * sum_m a[m,P] + scale * sum_m b[m,P]: the meta-gradient plus the E-MAML exploration gradient, equal bit for
 * bit to promp_reduce_tasks on each and an add. */
int promp_reduce_tasks2(int M, int P, const float* a, const float* b, float scale, float* out, void* stream);

/*
 * Logged scalars without a host round trip per value (the Trainer reads ONE float64 vector back per iteration):
 *   promp_phase_log_terms : out7 = AverageDiscountedReturn, AverageReturn, NumTrajs, StdReturn, MaxReturn, MinReturn
 *                           (samplers/base.py:135-149, from the stats [M,8] of promp_process_samples; n_paths = total
 *                           number of paths of the phase) and AveragePolicyStd = mean exp(log_std [M,Da])
 *                           (policies/gaussian_mlp_policy.py:118-123).
 *   promp_promp_log_terms : out3 = LossBefore, LossAfter, KLInner (pro_mp.py:193-198) from the optimizer's device vector
 *                           [loss_before, loss_after, inner KLs (num_inner_steps), outer KL].
 */
int promp_phase_log_terms(int M, int act_dim, double n_paths, const double* stats, const float* log_std, double* out7, void* stream);
int promp_promp_log_terms(int num_inner_steps, const float* final_terms, double* out3, void* stream);
/* ProMP's adaptive inner-KL coefficient rule (meta_algos/pro_mp.py:201-214) applied on the device, so that an iteration with
 * adaptive_inner_kl_penalty=True (the reference class default) has no host decision and can be replayed as a CUDA graph:
 *   coeff_dev[s] /= 2 if KL_s < kl_target / 1.5;  *= 2 if KL_s > kl_target * 1.5     (KL_s = final_terms[2 + s]; adapt != 0)
 * out4 (device double[4], optional) = the four scalars ProMP logs (pro_mp.py:193-198): LossBefore, LossAfter, KLInner (as
 * promp_promp_log_terms) and KLCoeffInner = mean_s coeff_dev[s] after the update. */
int promp_adapt_kl_coeff(int num_inner_steps, const float* final_terms, double kl_target, int adapt, float* coeff_dev,
                         double* out4, void* stream);

/*
 * tf.train.AdamOptimizer step as used by MAMLFirstOrderOptimizer.optimize
 * (optimizers/maml_first_order_optimizer.py:48-64, 102-107):
 *   t += 1; lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m = b1*m+(1-b1)*g; v = b2*v+(1-b2)*g^2;
 *   theta -= lr_t*m/(sqrt(v)+eps).      step is a device int32 counter (persistent slot state).
 */
int promp_adam_tf1(int P, float* theta, const float* grad, float* m, float* v, int32_t* step,
                   float lr, float beta1, float beta2, float eps, void* stream);

/*
 * One-shot all-reduce (sum * scale) of a small float vector over NVLink peer memory, rank-ordered (bitwise identical
 * on every rank) and graph-capturable; replaces the single collective of the path, the all-reduce of the flat
 * meta-gradient (SURVEY.md section 8e).  Setup: every rank allocates a buffer of promp_comm_buffer_bytes() with
 * promp_comm_alloc (the one allocation the library performs: IPC export needs a whole cudaMalloc block), exchanges
 * promp_ipc_get_handle() blobs (64 bytes, e.g. via torch.distributed.all_gather_object), opens the peers' blobs with
 * promp_ipc_open_handle and passes the world-sized DEVICE array of buffer pointers (own buffer at index `rank`).
 *   epoch_dev, error_flag_dev, ticket_dev: device uint32, zero-initialised; error_flag becomes 1 (sticky) if a peer did not
 *   arrive in ~2 s, and the results of that and every later call are NaN.
 * Protocol (csrc/comm.cu): low-latency exchange - every element travels as one 8-byte {value, epoch} store into all ranks'
 * receive areas and is polled there; no flags, no system fences; ceil(n / 256) CTAs.
 */
int64_t promp_comm_buffer_bytes(int world, int capacity_floats);
int promp_comm_alloc(int64_t bytes, void** dev_ptr_host);
int promp_comm_free(void* dev_ptr);
int promp_ipc_get_handle(void* dev_ptr, void* handle64_host);
int promp_ipc_open_handle(const void* handle64_host, void** dev_ptr_host);
int promp_ipc_close_handle(void* dev_ptr);
int promp_allreduce_p2p(int world, int rank, int n, int capacity_floats, const float* in, float* out, float scale,
                        void* const* peers_dev, uint32_t* epoch_dev, uint32_t* error_flag_dev, uint32_t* ticket_dev,
                        void* stream);

/* Runtime options.
 *   "tensor_cores" = 1 (default): hidden-64 promp_policy_grad / promp_policy_hvp run their layer and weight-gradient GEMMs on
 *                    the tensor cores (wgmma / mma.sync tf32, 3xTF32 split), same results to fp32 round-off; 0 = CUDA cores.
 *   "tc_threads"   = 0 (default: 512 threads per CTA for obs_dim <= 4, else 256), or force 256 / 512. */
int promp_set_option(const char* name, int value);

/* Policy forward only (MetaGaussianMLPPolicy.get_actions without sampling / distribution_info_sym):
 * mean [M,N,Da] for obs [M,N,Do]. */
int promp_policy_forward(int obs_dim, int act_dim, int hidden, int M, int N,
                         const float* params, int64_t param_stride, const float* obs, float* mean,
                         void* stream);

/*
 * Padded policy kernels: any obs_dim in [1, 19], act_dim in [1, 8], hidden 32 or 64 (the policy of
 * policies/meta_gaussian_mlp_policy.py:9-157 / gaussian_mlp_policy.py:31-184 for any Box observation / action space of those
 * sizes).  The entry points above are built for the exact (obs_dim, act_dim) = (2,2), (4,2), (17,6) only and reject every
 * other shape; the *_padded siblings below run kernels instantiated at caps and take the logical sizes at run time.
 *
 * Layout.  promp_policy_layout gives out = (obs_cap, act_cap, hidden, P) with P = promp_num_params(obs_cap, act_cap, hidden)
 * (obs_cap = 8 for obs_dim <= 8, else 20; act_cap = 2 for act_dim <= 2, else 8; P % 4 == 0).  Every parameter-shaped vector
 * of the padded entries (params, grad, out_params, vec, out, skip_theta, theta_copy_out: [.., P]) is the flat layout of
 * promp_num_params at the caps, in the same order W0[obs_cap,H] b0[H] W1[H,H] b1[H] W2[H,act_cap] b2[act_cap]
 * log_std[act_cap], with the logical parameters in W0[:obs_dim, :], W2[:, :act_dim], b2[:act_dim], log_std[:act_dim].
 * Zero-pad invariant: every other entry (pad rows of W0, pad columns of W2, pad entries of b2 / log_std) must be 0 on input;
 * the kernels then return exactly 0 for them in every gradient and in the Hessian-vector product (out = vec there), so SGD,
 * Adam, CG / TRPO and the meta-update keep them at 0.
 * Data.  obs [M,N,obs_dim], act / old_mean / old_log_std / mean with act_dim columns: the logical sizes, as for the exact
 * entries.  promp_policy_layout is host-only; it returns PROMP_ERR_INVALID_ARG (and sets promp_last_error) out of range.
 * The *_padded siblings take the arguments of the entry named without the suffix and replace the same reference functions.
 * They always run the padded instantiations, also for shapes the exact table covers.
 */
int promp_policy_layout(int obs_dim, int act_dim, int hidden, int32_t out[4]);
int64_t promp_policy_workspace_bytes_padded(int M, int N, int obs_dim, int act_dim, int hidden);
int promp_policy_forward_padded(int obs_dim, int act_dim, int hidden, int M, int N,
                                const float* params, int64_t param_stride, const float* obs, float* mean,
                                void* stream);
int promp_policy_grad_ex_padded(int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid, const float* params,
                                int64_t param_stride, const float* obs, const float* act, const float* adv, const float* old_mean,
                                const float* old_log_std, int ls_per_sample, int obj_kind, float obj_scale, float clip_eps,
                                float kl_coeff, int clip_log_std, float min_log_std, float* grad, float* out_params, float sgd_lr,
                                float* stats, const int32_t* skip_flag, const float* skip_theta, int32_t* unclipped_out,
                                float* theta_copy_out, void* workspace, int64_t workspace_bytes, void* stream);
int promp_policy_hvp_ragged_padded(int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid,
                                   const float* params, int64_t param_stride,
                                   const float* obs, const float* act, const float* adv,
                                   const float* old_mean, const float* old_log_std, int ls_per_sample,
                                   int obj_kind, float inner_lr, float kl_coeff,
                                   int clip_log_std, float min_log_std,
                                   const float* vec, float* out, float* stats,
                                   void* workspace, int64_t workspace_bytes, void* stream);
int64_t promp_policy_chain_workspace_bytes_padded(int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                                  const promp_policy_stage* stages);
int promp_policy_chain_num_launches_padded(int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                           const promp_policy_stage* stages);
int promp_policy_chain_padded(int obs_dim, int act_dim, int hidden, int M, float min_log_std, int n_stages,
                              const promp_policy_stage* stages, const int32_t* skip_flag, const float* skip_theta,
                              void* workspace, int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PROMP_B200_H */
