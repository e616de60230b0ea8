// The fused rollout kernel and the single-step env kernels, templated over one environment type (see envs.cuh for the
// concept).  Included by rollout.cu, which instantiates them for the built-in environments, and by the source that
// promp_b200/_jit.py generates for a user's environment, which NVRTC compiles at run time.
//
// Design (sm_90a): the rollout is a strictly sequential H-step chain per env with ~9-11 kFLOP of
// MLP math and ~30-120 B of compulsory output per step, i.e. it is latency bound, not HBM bound.
// So: one warp owns one env for the whole horizon; each lane keeps its HID/32 columns of every
// weight matrix in REGISTERS (W1 alone is 2*64 registers/lane), activations are exchanged through
// a per-warp shared-memory line with __syncwarp only (no block barriers), the layer-2 reduction is
// a warp shuffle, the env state lives in registers, and the trajectory record is staged in shared
// memory for T_CH steps and flushed as coalesced 128-byte float32 rows.
#pragma once
#include "envs.cuh"

namespace promp {
constexpr int T_CH = 32;       // steps staged in shared memory between coalesced flushes
constexpr int RO_WARPS = 4;    // env-warps per CTA

struct RolloutArgs {
    int reward_type;
    float radius;
    int normalized;
    int M, E, H;
    const float* params;
    int64_t param_stride;
    const float* task_params;
    const float* init_state;
    const float* noise;
    uint64_t seed, stream_id;
    const uint64_t* stream_id_dev;
    int clip_reported;
    float min_log_std;
    float *obs, *act, *mean, *rew;
    uint8_t* done;
    float* info;
    float* log_std_out;
    float* final_state;
    // early-terminating envs (MetaPointEnv): the kernel records a TIMELINE of H steps per env slot; a path ends when the env
    // reports done or after `horizon` steps, the slot is reset in-kernel (Philox) and keeps stepping.  0: fixed-horizon mode.
    int early_term;
    int horizon;
    // task_offset * E, task_offset = global index of task 0 of this launch (a rank's shard of a larger task batch): added
    // to the env index of the Philox key only, so a shard draws the noise / reset states its tasks get in one launch over
    // the whole batch
    uint32_t key_offset;
};

// GENERIC_INFO = true (user envs, user_env.cuh): the rollout flushes env-info channels 0 .. NINFO-1 as the env wrote them.
// The built-in envs leave it undefined and keep their own channel layout (the cheetah's third channel for reward_type 1).
template <class Env, class = void>
struct generic_info {
    static constexpr bool value = false;
};
template <class Env>
struct generic_info<Env, decltype(void(Env::GENERIC_INFO))> {
    static constexpr bool value = Env::GENERIC_INFO;
};

template <class Env, int HID>
struct RolloutSmem {
    static constexpr int DOP = (Env::DO + 3) / 4 * 4;
    float obs[DOP];
    float h1[HID];
    float noise[T_CH * Env::DA];
    float st_obs[T_CH * Env::DO];
    float st_act[T_CH * Env::DA];
    float st_mean[T_CH * Env::DA];
    float st_rew[T_CH];
    float st_info[3 * T_CH];
    unsigned char st_done[T_CH];
};

#ifdef PROMP_EXP_CLOCKS
// experiment build only: per-phase clock64 totals of warp 0 of CTA (0,0) (tools/rollout_time.py)
__device__ unsigned long long g_ro_clk[16];
#define RCLK(i)                                                           \
    do {                                                                  \
        if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {     \
            const long long t_ = clock64();                               \
            ro_clk[i] += (unsigned long long)(t_ - ro_last);              \
            ro_last = t_;                                                 \
        }                                                                 \
    } while (0)
#else
#define RCLK(i)
#endif

// The parameter layout the policy keeps for an env's (DO, DA) (policies/meta_gaussian_mlp_policy.py EXACT_SHAPES): the
// shapes with policy kernels of their own are compact; every other shape is zero-padded to the caps of
// promp_policy_layout (obs 8 or 20, act 2 or 8).  The built-in envs' shapes are exact or equal their caps (swimmer 8, 2).
template <int DO, int DA>
struct PolicyCaps {
    static constexpr bool EXACT = (DO == 2 && DA == 2) || (DO == 4 && DA == 2) || (DO == 17 && DA == 6);
    static constexpr int OBS = EXACT ? DO : (DO <= 8 ? 8 : 20);
    static constexpr int ACT = EXACT ? DA : (DA <= 2 ? 2 : 8);
};

// KEYED: the launch is a shard of a larger task batch (key_offset != 0).  A separate instantiation, so that adding the
// offset leaves the code of the unsharded kernels as it was (ptxas schedules their step loop differently otherwise).
template <class Env, int HID, class Act, bool KEYED>
__global__ void __launch_bounds__(RO_WARPS * 32) rollout_kernel(RolloutArgs A) {
    constexpr int DO = Env::DO, DA = Env::DA, SD = Env::SD, TD = Env::TD;
    constexpr int NU = HID / 32;
    constexpr int DAP = PolicyCaps<DO, DA>::ACT;     // row stride of W2
    using L = PLayout<PolicyCaps<DO, DA>::OBS, DAP, HID>;
    static_assert(HID % 32 == 0, "hidden size must be a multiple of 32");

    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int m = blockIdx.y, e = blockIdx.x * RO_WARPS + w;
    if (e >= A.E) return;   // whole warp leaves; nothing below uses a block-wide barrier

    __shared__ __align__(16) RolloutSmem<Env, HID> smem_all[RO_WARPS];
    RolloutSmem<Env, HID>& S = smem_all[w];

#ifdef PROMP_EXP_CLOCKS
    unsigned long long ro_clk[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long ro_last = clock64();
#endif
    const float* th = A.params + (int64_t)m * A.param_stride;
    if (A.stream_id_dev) A.stream_id += *A.stream_id_dev;   // device-side phase counter (CUDA-graph replays)
    const int64_t env_id = (int64_t)m * A.E + e;     // env index in this launch's buffers
    const int64_t base = env_id * A.H;               // flat sample offset of this env (n = e*H + t)

    // ---- weights -> registers (lane owns hidden units j = lane + 32*u)
    float w0[DO][NU], b0[NU], w1[HID][NU], b1[NU], w2[NU][DA], b2[DA], sig[DA];
#pragma unroll
    for (int u = 0; u < NU; ++u) {
        const int j = lane + 32 * u;
#pragma unroll
        for (int i = 0; i < DO; ++i) w0[i][u] = __ldg(th + L::W0 + i * HID + j);
        b0[u] = __ldg(th + L::B0 + j);
#pragma unroll
        for (int k = 0; k < HID; ++k) w1[k][u] = __ldg(th + L::W1 + k * HID + j);
        b1[u] = __ldg(th + L::B1 + j);
#pragma unroll
        for (int d = 0; d < DA; ++d) w2[u][d] = __ldg(th + L::W2 + j * DAP + d);
    }
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        b2[d] = __ldg(th + L::B2 + d);
        float ls = __ldg(th + L::LS + d);
        sig[d] = expf(ls);   // sampling uses the raw log_std (gaussian_mlp_policy.py:74)
        if (e == 0 && lane == d)
            A.log_std_out[(int64_t)m * DA + d] = A.clip_reported ? fmaxf(ls, A.min_log_std) : ls;
    }

    // ---- task + initial state
    float task[TD];
#pragma unroll
    for (int i = 0; i < TD; ++i) task[i] = __ldg(A.task_params + (int64_t)m * TD + i);

    const EnvRng rng{KEYED ? (uint32_t)env_id + A.key_offset : (uint32_t)env_id, (uint32_t)A.stream_id,
                     (uint32_t)((A.stream_id >> 32) & 0xffffffu), A.seed};
    Env env;
    if (A.init_state) env.load(A.init_state + env_id * SD, lane);
    else env.reset(rng, 0u, 0x52000000u, lane, task);
    env.observe(S.obs, lane);
    __syncwarp();

    const EnvCfg cfg{A.reward_type, A.radius, A.normalized != 0};
    [[maybe_unused]] int path_ts = 0;   // steps taken in the current path (early-termination mode)

    RCLK(0);
    for (int t0 = 0; t0 < A.H; t0 += T_CH) {
        const int nt = min(T_CH, A.H - t0);
        // ---- action noise for this chunk -> shared memory
        if (A.noise) {
            const float* ng = A.noise + (base + t0) * DA;
            for (int i = lane; i < nt * DA; i += 32) S.noise[i] = __ldg(ng + i);   // coalesced
        } else if (lane < nt) {
            const int t = t0 + lane;
#pragma unroll
            for (int blk = 0; blk < (DA + 3) / 4; ++blk) {
                uint32_t r[4];
                rng.gen((uint32_t)t, (uint32_t)blk << 24, r);
                float z[4];
                box_muller(r[0], r[1], z[0], z[1]);
                box_muller(r[2], r[3], z[2], z[3]);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (blk * 4 + i < DA) S.noise[lane * DA + blk * 4 + i] = z[i];
            }
        }
        __syncwarp();
        RCLK(1);

        for (int tt = 0; tt < nt; ++tt) {
            // ---- layer 0: h1 = act(obs W0 + b0)            (policies/networks/mlp.py:96-117)
            float ob[DO];
#pragma unroll
            for (int i = 0; i < DO; ++i) ob[i] = S.obs[i];
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                float z = b0[u];
#pragma unroll
                for (int i = 0; i < DO; ++i) z = fmaf(ob[i], w0[i][u], z);
                S.h1[lane + 32 * u] = Act::f(z);
            }
            // stage obs_t (the observation the action is computed from)
            if (lane < DO) S.st_obs[tt * DO + lane] = S.obs[lane];
            __syncwarp();
            RCLK(2);
            // ---- layer 1: h2 = act(h1 W1 + b1); NACC accumulators per output for ILP (4 where the registers allow it)
            constexpr int NACC = Env::NACC;
            float acc[NU][NACC];
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                acc[u][0] = b1[u];
#pragma unroll
                for (int a = 1; a < NACC; ++a) acc[u][a] = 0.f;
            }
#pragma unroll
            for (int k4 = 0; k4 < HID / 4; ++k4) {
                const float4 h = *reinterpret_cast<const float4*>(&S.h1[4 * k4]);   // warp-broadcast LDS.128
#pragma unroll
                for (int u = 0; u < NU; ++u) {
                    acc[u][0 % NACC] = fmaf(h.x, w1[4 * k4 + 0][u], acc[u][0 % NACC]);
                    acc[u][1 % NACC] = fmaf(h.y, w1[4 * k4 + 1][u], acc[u][1 % NACC]);
                    acc[u][2 % NACC] = fmaf(h.z, w1[4 * k4 + 2][u], acc[u][2 % NACC]);
                    acc[u][3 % NACC] = fmaf(h.w, w1[4 * k4 + 3][u], acc[u][3 % NACC]);
                }
            }
            RCLK(3);
            // ---- layer 2: mean = h2 W2 + b2 (warp shuffle reduction over the hidden units)
            float mu[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = 0.f;
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                const float h2 = Act::f(NACC == 4 ? (acc[u][0] + acc[u][1]) + (acc[u][2 % NACC] + acc[u][3 % NACC]) : acc[u][0] + acc[u][1]);
#pragma unroll
                for (int d = 0; d < DA; ++d) mu[d] = fmaf(h2, w2[u][d], mu[d]);
            }
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = warp_sum(mu[d]) + b2[d];
            out_forward<Act, DA>(mu);      // tanh output layer: mean = tanh(h2 W2 + b2)

            RCLK(4);
            // ---- sample: a = mean + eps * exp(log_std)      (gaussian_mlp_policy.py:74)
            float a[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) a[d] = fmaf(S.noise[tt * DA + d], sig[d], mu[d]);
            if (lane < DA) {
                float al = 0.f, ml = 0.f;
#pragma unroll
                for (int d = 0; d < DA; ++d)
                    if (lane == d) al = a[d], ml = mu[d];
                S.st_act[tt * DA + lane] = al;
                S.st_mean[tt * DA + lane] = ml;
            }

            RCLK(5);
            // ---- env step (NormalizedEnv rescale + env dynamics + reward)
            bool dn = false;
            const float r = env.step(a, task, cfg, lane, S.st_info + tt, T_CH, dn);
            if constexpr (Env::ENDS_EARLY) {
                if (A.early_term) {
                    // executor semantics (vectorized_env_executor.py:44-52): ts += 1; done |= ts >= max_path_length; a done
                    // env is reset at once and the NEXT observation is the reset state, drawn here from Philox keyed by
                    // (env, step) instead of the host numpy stream.  `dn` is warp-uniform.
                    ++path_ts;
                    const bool fin = dn || path_ts >= A.horizon;
                    if (lane == 0) S.st_done[tt] = fin ? 1 : 0;
                    if (fin) {
                        env.reset(rng, (uint32_t)(t0 + tt), 0x53000000u, lane, task);
                        path_ts = 0;
                    }
                }
            }
            if (lane == 0) S.st_rew[tt] = r;
            RCLK(6);
            __syncwarp();      // all lanes are done reading S.obs / S.h1 of this step
            env.observe(S.obs, lane);
            __syncwarp();
            RCLK(7);
        }

        // ---- coalesced flush of the staged chunk: consecutive lanes -> consecutive floats
        {
            float* g;
            g = A.obs + (base + t0) * DO;
            for (int i = lane; i < nt * DO; i += 32) g[i] = S.st_obs[i];
            g = A.act + (base + t0) * DA;
            for (int i = lane; i < nt * DA; i += 32) g[i] = S.st_act[i];
            g = A.mean + (base + t0) * DA;
            for (int i = lane; i < nt * DA; i += 32) g[i] = S.st_mean[i];
            if (lane < nt) {
                A.rew[base + t0 + lane] = S.st_rew[lane];
                // horizon reset (vectorized_env_executor.py:46-50); early-termination mode: the recorded path ends
                A.done[base + t0 + lane] = A.early_term ? S.st_done[lane] : ((t0 + lane == A.H - 1) ? 1 : 0);
                if (Env::NINFO > 0 && A.info) {
                    const int64_t tot = (int64_t)A.M * A.E * A.H;
                    if constexpr (generic_info<Env>::value) {   // user envs: channels 0 .. NINFO-1
#pragma unroll
                        for (int c = 0; c < Env::NINFO; ++c) A.info[c * tot + base + t0 + lane] = S.st_info[c * T_CH + lane];
                    } else {
                        A.info[base + t0 + lane] = S.st_info[lane];
                        A.info[tot + base + t0 + lane] = S.st_info[T_CH + lane];
                        if (A.reward_type == 1) A.info[2 * tot + base + t0 + lane] = S.st_info[2 * T_CH + lane];   // RandVel: forward_vel
                    }
                }
            }
        }
        __syncwarp();
    }

#ifdef PROMP_EXP_CLOCKS
    RCLK(1);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0)
        for (int i = 0; i < 8; ++i) g_ro_clk[i] += ro_clk[i];
#endif
    if (A.final_state) env.store(A.final_state + env_id * SD, lane);
}

// ---------------------------------------------------------------------------- policies of depth 1 and 3
// rollout_kernel for a policy with nh = depth - 1 hidden-to-hidden layers (0 or 2, a kernel argument: one instantiation
// serves both depths).  A 64 x 64 matrix does not fit the registers of a warp next to the env (it alone is 128 registers per
// lane), so the hidden-to-hidden layers [W_1 b_1 W_2 b_2] live in dynamic shared memory, staged once per CTA: the RO_WARPS
// warps of a CTA step envs of the same task and share that copy.  Layer 0, the output layer and the env step are those of
// rollout_kernel; lane j reads row k of a hidden matrix at k * HID + j (conflict-free) and the activation as a broadcast.
template <int HID>
__host__ __device__ constexpr int rollout_deep_smem_bytes(int nh) {
    return nh * (HID * HID + HID) * (int)sizeof(float);
}

template <class Env, int HID, class Act, bool KEYED>
__global__ void __launch_bounds__(RO_WARPS * 32) rollout_deep_kernel(RolloutArgs A, int nh) {
    constexpr int DO = Env::DO, DA = Env::DA, SD = Env::SD, TD = Env::TD;
    constexpr int NU = HID / 32;
    constexpr int DAP = PolicyCaps<DO, DA>::ACT;
    const DeepLayout<PolicyCaps<DO, DA>::OBS, DAP, HID> L{nh};
    static_assert(HID % 32 == 0, "hidden size must be a multiple of 32");

    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int m = blockIdx.y, e = blockIdx.x * RO_WARPS + w;

    __shared__ __align__(16) RolloutSmem<Env, HID> smem_all[RO_WARPS];
    extern __shared__ __align__(16) float s_wh[];       // [nh][HID * HID + HID]: W_l then b_l, as in the parameter vector
    RolloutSmem<Env, HID>& S = smem_all[w];

    const float* th = A.params + (int64_t)m * A.param_stride;
    for (int i = threadIdx.x; i < nh * (HID * HID + HID); i += blockDim.x) s_wh[i] = __ldg(th + L.wh(0) + i);
    __syncthreads();
    if (e >= A.E) return;   // whole warp leaves; nothing below uses a block-wide barrier

    if (A.stream_id_dev) A.stream_id += *A.stream_id_dev;
    const int64_t env_id = (int64_t)m * A.E + e;
    const int64_t base = env_id * A.H;

    float w0[DO][NU], b0[NU], w2[NU][DA], b2[DA], sig[DA];
#pragma unroll
    for (int u = 0; u < NU; ++u) {
        const int j = lane + 32 * u;
#pragma unroll
        for (int i = 0; i < DO; ++i) w0[i][u] = __ldg(th + L.W0 + i * HID + j);
        b0[u] = __ldg(th + L.B0 + j);
#pragma unroll
        for (int d = 0; d < DA; ++d) w2[u][d] = __ldg(th + L.wo() + j * DAP + d);
    }
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        b2[d] = __ldg(th + L.bo() + d);
        float ls = __ldg(th + L.ls() + d);
        sig[d] = expf(ls);
        if (e == 0 && lane == d)
            A.log_std_out[(int64_t)m * DA + d] = A.clip_reported ? fmaxf(ls, A.min_log_std) : ls;
    }

    float task[TD];
#pragma unroll
    for (int i = 0; i < TD; ++i) task[i] = __ldg(A.task_params + (int64_t)m * TD + i);

    const EnvRng rng{KEYED ? (uint32_t)env_id + A.key_offset : (uint32_t)env_id, (uint32_t)A.stream_id,
                     (uint32_t)((A.stream_id >> 32) & 0xffffffu), A.seed};
    Env env;
    if (A.init_state) env.load(A.init_state + env_id * SD, lane);
    else env.reset(rng, 0u, 0x52000000u, lane, task);
    env.observe(S.obs, lane);
    __syncwarp();

    const EnvCfg cfg{A.reward_type, A.radius, A.normalized != 0};
    [[maybe_unused]] int path_ts = 0;

    for (int t0 = 0; t0 < A.H; t0 += T_CH) {
        const int nt = min(T_CH, A.H - t0);
        if (A.noise) {
            const float* ng = A.noise + (base + t0) * DA;
            for (int i = lane; i < nt * DA; i += 32) S.noise[i] = __ldg(ng + i);
        } else if (lane < nt) {
            const int t = t0 + lane;
#pragma unroll
            for (int blk = 0; blk < (DA + 3) / 4; ++blk) {
                uint32_t r[4];
                rng.gen((uint32_t)t, (uint32_t)blk << 24, r);
                float z[4];
                box_muller(r[0], r[1], z[0], z[1]);
                box_muller(r[2], r[3], z[2], z[3]);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (blk * 4 + i < DA) S.noise[lane * DA + blk * 4 + i] = z[i];
            }
        }
        __syncwarp();

        for (int tt = 0; tt < nt; ++tt) {
            // ---- layer 0: h = act(obs W0 + b0)            (policies/networks/mlp.py:96-117)
            float ob[DO], h[NU];
#pragma unroll
            for (int i = 0; i < DO; ++i) ob[i] = S.obs[i];
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                float z = b0[u];
#pragma unroll
                for (int i = 0; i < DO; ++i) z = fmaf(ob[i], w0[i][u], z);
                h[u] = Act::f(z);
                S.h1[lane + 32 * u] = h[u];
            }
            if (lane < DO) S.st_obs[tt * DO + lane] = S.obs[lane];
            __syncwarp();
            // ---- hidden layers: h = act(h W_l + b_l), weights from shared memory
            for (int l = 0; l < nh; ++l) {
                const float* Wl = s_wh + l * (HID * HID + HID);
                float acc[NU][4];
#pragma unroll
                for (int u = 0; u < NU; ++u) {
                    acc[u][0] = Wl[HID * HID + lane + 32 * u];
                    acc[u][1] = acc[u][2] = acc[u][3] = 0.f;
                }
#pragma unroll 4
                for (int k4 = 0; k4 < HID / 4; ++k4) {
                    const float4 hv = *reinterpret_cast<const float4*>(&S.h1[4 * k4]);
#pragma unroll
                    for (int u = 0; u < NU; ++u) {
                        const int j = lane + 32 * u;
                        acc[u][0] = fmaf(hv.x, Wl[(4 * k4 + 0) * HID + j], acc[u][0]);
                        acc[u][1] = fmaf(hv.y, Wl[(4 * k4 + 1) * HID + j], acc[u][1]);
                        acc[u][2] = fmaf(hv.z, Wl[(4 * k4 + 2) * HID + j], acc[u][2]);
                        acc[u][3] = fmaf(hv.w, Wl[(4 * k4 + 3) * HID + j], acc[u][3]);
                    }
                }
#pragma unroll
                for (int u = 0; u < NU; ++u) h[u] = Act::f((acc[u][0] + acc[u][1]) + (acc[u][2] + acc[u][3]));
                __syncwarp();      // every lane has read this layer's input
#pragma unroll
                for (int u = 0; u < NU; ++u) S.h1[lane + 32 * u] = h[u];
                __syncwarp();
            }
            // ---- output layer: mean = h W_out + b_out (warp shuffle reduction over the hidden units)
            float mu[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = 0.f;
#pragma unroll
            for (int u = 0; u < NU; ++u)
#pragma unroll
                for (int d = 0; d < DA; ++d) mu[d] = fmaf(h[u], w2[u][d], mu[d]);
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = warp_sum(mu[d]) + b2[d];
            out_forward<Act, DA>(mu);

            float a[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) a[d] = fmaf(S.noise[tt * DA + d], sig[d], mu[d]);
            if (lane < DA) {
                float al = 0.f, ml = 0.f;
#pragma unroll
                for (int d = 0; d < DA; ++d)
                    if (lane == d) al = a[d], ml = mu[d];
                S.st_act[tt * DA + lane] = al;
                S.st_mean[tt * DA + lane] = ml;
            }

            bool dn = false;
            const float r = env.step(a, task, cfg, lane, S.st_info + tt, T_CH, dn);
            if constexpr (Env::ENDS_EARLY) {
                if (A.early_term) {
                    ++path_ts;
                    const bool fin = dn || path_ts >= A.horizon;
                    if (lane == 0) S.st_done[tt] = fin ? 1 : 0;
                    if (fin) {
                        env.reset(rng, (uint32_t)(t0 + tt), 0x53000000u, lane, task);
                        path_ts = 0;
                    }
                }
            }
            if (lane == 0) S.st_rew[tt] = r;
            __syncwarp();
            env.observe(S.obs, lane);
            __syncwarp();
        }

        {
            float* g;
            g = A.obs + (base + t0) * DO;
            for (int i = lane; i < nt * DO; i += 32) g[i] = S.st_obs[i];
            g = A.act + (base + t0) * DA;
            for (int i = lane; i < nt * DA; i += 32) g[i] = S.st_act[i];
            g = A.mean + (base + t0) * DA;
            for (int i = lane; i < nt * DA; i += 32) g[i] = S.st_mean[i];
            if (lane < nt) {
                A.rew[base + t0 + lane] = S.st_rew[lane];
                A.done[base + t0 + lane] = A.early_term ? S.st_done[lane] : ((t0 + lane == A.H - 1) ? 1 : 0);
                if (Env::NINFO > 0 && A.info) {
                    const int64_t tot = (int64_t)A.M * A.E * A.H;
                    if constexpr (generic_info<Env>::value) {
#pragma unroll
                        for (int c = 0; c < Env::NINFO; ++c) A.info[c * tot + base + t0 + lane] = S.st_info[c * T_CH + lane];
                    } else {
                        A.info[base + t0 + lane] = S.st_info[lane];
                        A.info[tot + base + t0 + lane] = S.st_info[T_CH + lane];
                        if (A.reward_type == 1) A.info[2 * tot + base + t0 + lane] = S.st_info[2 * T_CH + lane];
                    }
                }
            }
        }
        __syncwarp();
    }
    if (A.final_state) env.store(A.final_state + env_id * SD, lane);
}

// ---------------------------------------------------------------------------- single-step kernels
template <class Env>
__global__ void env_step_kernel(EnvCfg cfg, int n_env, int H, float* state, int32_t* ts, const float* actions,
                                const float* task_params, const float* reset_state, float* next_obs, float* rew, uint8_t* done,
                                float* info) {
    constexpr int SD = Env::SD, DA = Env::DA;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_env) return;
    float st[SD], a[DA];
#pragma unroll
    for (int k = 0; k < SD; ++k) st[k] = state[(int64_t)i * SD + k];
#pragma unroll
    for (int k = 0; k < DA; ++k) a[k] = actions[(int64_t)i * DA + k];
    bool dn = false;
    const float r = Env::step_serial(st, a, task_params + (int64_t)i * Env::TD, cfg, info ? info + i : nullptr, n_env, dn);
    int t = ts[i] + 1;
    dn = dn || (t >= H);
    if (dn) {   // MetaIterativeEnvExecutor.step :46-50: a done env is reset and returns the reset obs
#pragma unroll
        for (int k = 0; k < SD; ++k) st[k] = reset_state[(int64_t)i * SD + k];
        t = 0;
    }
    ts[i] = t;
    rew[i] = r;
    done[i] = dn ? 1 : 0;
#pragma unroll
    for (int k = 0; k < SD; ++k) state[(int64_t)i * SD + k] = st[k];
    Env::observe_serial(st, next_obs + (int64_t)i * Env::DO);
}

template <class Env>
__global__ void env_observe_kernel(int n_env, const float* state, float* obs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_env) Env::observe_serial(state + (int64_t)i * Env::SD, obs + (int64_t)i * Env::DO);
}

}  // namespace promp
