// Fused vectorised rollout kernel (one warp per env, all H steps in one launch) and the
// single-step vec-env kernels.  See include/promp_b200.h for the interface and the reference
// functions each entry point replaces.
//
// Design (sm_90a): the rollout is a strictly sequential H-step chain per env with ~9-11 kFLOP of
// MLP math and ~30-120 B of compulsory output per step, i.e. it is latency bound, not HBM bound.
// So: one warp owns one env for the whole horizon; each lane keeps its HID/32 columns of every
// weight matrix in REGISTERS (W1 alone is 2*64 registers/lane), activations are exchanged through
// a per-warp shared-memory line with __syncwarp only (no block barriers), the layer-2 reduction is
// a warp shuffle, the env state lives in registers, and the trajectory record is staged in shared
// memory for T_CH steps and flushed as coalesced 128-byte float32 rows.
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
};

template <int KIND, int HID>
struct RolloutSmem {
    using T = EnvTraits<KIND>;
    static constexpr int DOP = (T::DO + 3) / 4 * 4;
    float obs[DOP];
    float h1[HID];
    float noise[T_CH * T::DA];
    float st_obs[T_CH * T::DO];
    float st_act[T_CH * T::DA];
    float st_mean[T_CH * T::DA];
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

// walker reset_model (walker2d_rand_*.py:47-52): qpos = init_qpos + U(-.005,.005)^9 (init_qpos z = 1.25, all else 0),
// qvel = U(-.005,.005)^9.  Lane i < 9 draws coordinate i from Philox counter (env, ctr + i); the result is spread over the
// warp like the cheetah's reset (root replicated, lane j < 6 keeps joint j).
__device__ __forceinline__ void walker_reset(const RolloutArgs& A, int64_t env_id, uint32_t ctr, uint32_t tag, int lane, float& q,
                                             float& qd, float (&root)[6]) {
    float pos = 0.f, vel = 0.f;
    if (lane < 9) {
        uint32_t r[4];
        Philox::gen((uint32_t)env_id, ctr + (uint32_t)lane, (uint32_t)A.stream_id, tag | (uint32_t)((A.stream_id >> 32) & 0xffffffu),
                    A.seed, r);
        pos = -0.005f + 0.01f * u01(r[0]);
        vel = -0.005f + 0.01f * u01(r[1]);
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        root[i] = __shfl_sync(0xffffffffu, pos, i);
        root[3 + i] = __shfl_sync(0xffffffffu, vel, i);
    }
    root[1] += 1.25f;
    const int jl = lane & 7;
    const float qq = __shfl_sync(0xffffffffu, pos, 3 + (jl < 6 ? jl : 0));
    const float qv = __shfl_sync(0xffffffffu, vel, 3 + (jl < 6 ? jl : 0));
    q = jl < 6 ? qq : 0.f;
    qd = jl < 6 ? qv : 0.f;
}

template <int KIND, int HID>
__global__ void __launch_bounds__(RO_WARPS * 32) rollout_kernel(RolloutArgs A) {
    using T = EnvTraits<KIND>;
    constexpr int DO = T::DO, DA = T::DA, SD = T::SD, TD = T::TD;
    constexpr int NU = HID / 32;
    using L = PLayout<DO, DA, HID>;
    static_assert(HID % 32 == 0, "hidden size must be a multiple of 32");

    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int m = blockIdx.y, e = blockIdx.x * RO_WARPS + w;
    if (e >= A.E) return;   // whole warp leaves; nothing below uses a block-wide barrier

    __shared__ __align__(16) RolloutSmem<KIND, HID> smem_all[RO_WARPS];
    RolloutSmem<KIND, HID>& S = smem_all[w];

#ifdef PROMP_EXP_CLOCKS
    unsigned long long ro_clk[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long ro_last = clock64();
#endif
    const float* th = A.params + (int64_t)m * A.param_stride;
    if (A.stream_id_dev) A.stream_id += *A.stream_id_dev;   // device-side phase counter (CUDA-graph replays)
    const int64_t env_id = (int64_t)m * A.E + e;     // global env index
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
        for (int d = 0; d < DA; ++d) w2[u][d] = __ldg(th + L::W2 + j * DA + d);
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

    // env state registers
    float sx = 0.f, sy = 0.f, vx = 0.f, vy = 0.f;   // point envs (vx, vy: momentum env)
    float q = 0.f, qd = 0.f, root[6] = {0, 0, 0, 0, 0, 0};   // cheetah / walker: lane's joint (lane&7) + replicated root
    cheetah::JointConst jc = cheetah::joint_const(lane & 7);
    walker::JointConst wjc = walker::joint_const(lane & 7);
    float sw[10];                                            // swimmer: qpos[5] ++ qvel[5], replicated in every lane
#pragma unroll
    for (int k = 0; k < 10; ++k) sw[k] = 0.f;

    if (KIND == PROMP_ENV_CHEETAH_DIR || KIND == PROMP_ENV_WALKER) {
        const int jl = lane & 7;
        if (A.init_state) {
            const float* s0 = A.init_state + env_id * SD;
            root[0] = s0[0]; root[1] = s0[1]; root[2] = s0[2];
            root[3] = s0[9]; root[4] = s0[10]; root[5] = s0[11];
            q = jl < 6 ? s0[3 + jl] : 0.f;
            qd = jl < 6 ? s0[12 + jl] : 0.f;
        } else if (KIND == PROMP_ENV_WALKER) {
            walker_reset(A, env_id, 0u, 0x52000000u, lane, q, qd, root);
        } else {
            // reset_model (half_cheetah_rand_direc.py:49-53): qpos = U(-.1,.1)^9, qvel = .1*N(0,1)^9
            float pos = 0.f, vel = 0.f;
            if (lane < 9) {
                uint32_t r[4];
                Philox::gen((uint32_t)env_id, (uint32_t)lane, (uint32_t)A.stream_id,
                            0x52000000u | (uint32_t)((A.stream_id >> 32) & 0xffffffu), A.seed, r);
                pos = -0.1f + 0.2f * u01(r[0]);
                float z0, z1;
                box_muller(r[1], r[2], z0, z1);
                vel = 0.1f * z0;
            }
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                root[i] = __shfl_sync(0xffffffffu, pos, i);
                root[3 + i] = __shfl_sync(0xffffffffu, vel, i);
            }
            float qq = __shfl_sync(0xffffffffu, pos, 3 + (jl < 6 ? jl : 0));
            float qv = __shfl_sync(0xffffffffu, vel, 3 + (jl < 6 ? jl : 0));
            q = jl < 6 ? qq : 0.f;
            qd = jl < 6 ? qv : 0.f;
        }
    } else if (KIND == PROMP_ENV_SWIMMER) {
        if (A.init_state) {
#pragma unroll
            for (int k = 0; k < 10; ++k) sw[k] = A.init_state[env_id * SD + k];
        } else {
            // reset_model (swimmer_rand_vel.py:41-46): qpos = U(-.1,.1)^5, qvel = U(-.1,.1)^5 (every lane draws the same)
#pragma unroll
            for (int blk = 0; blk < 3; ++blk) {
                uint32_t r[4];
                Philox::gen((uint32_t)env_id, (uint32_t)blk, (uint32_t)A.stream_id,
                            0x52000000u | (uint32_t)((A.stream_id >> 32) & 0xffffffu), A.seed, r);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (blk * 4 + i < 10) sw[blk * 4 + i] = -0.1f + 0.2f * u01(r[i]);
            }
        }
    } else {
        if (A.init_state) {
            sx = A.init_state[env_id * SD + 0];
            sy = A.init_state[env_id * SD + 1];
            if (KIND == PROMP_ENV_POINT_MOMENTUM) vx = A.init_state[env_id * SD + 2], vy = A.init_state[env_id * SD + 3];
        } else {
            uint32_t r[4];
            Philox::gen((uint32_t)env_id, 0u, (uint32_t)A.stream_id,
                        0x52000000u | (uint32_t)((A.stream_id >> 32) & 0xffffffu), A.seed, r);
            const float lim = (KIND == PROMP_ENV_POINT) ? 2.0f : 0.2f;   // reset ranges (point_env_2d_corner.py:50 / point_env_2d.py:34)
            sx = -lim + 2.f * lim * u01(r[0]);
            sy = -lim + 2.f * lim * u01(r[1]);
            if (KIND == PROMP_ENV_POINT_MOMENTUM) vx = -0.1f + 0.2f * u01(r[2]), vy = -0.1f + 0.2f * u01(r[3]);   // (:52)
        }
    }

    auto write_obs = [&]() {
        if (KIND == PROMP_ENV_CHEETAH_DIR) {
            // obs = qpos[1:] ++ qvel (half_cheetah_rand_direc.py:43-47)
            if (lane == 0) {
                S.obs[0] = root[1]; S.obs[1] = root[2];
                S.obs[8] = root[3]; S.obs[9] = root[4]; S.obs[10] = root[5];
            }
            if (lane < 6) {
                S.obs[2 + lane] = q;
                S.obs[11 + lane] = qd;
            }
        } else if (KIND == PROMP_ENV_WALKER) {
            // obs = qpos[1:] ++ clip(qvel, -10, 10) (walker2d_rand_*.py:42-45)
            if (lane == 0) {
                S.obs[0] = root[1]; S.obs[1] = root[2];
                S.obs[8] = walker::clip_vel(root[3]); S.obs[9] = walker::clip_vel(root[4]); S.obs[10] = walker::clip_vel(root[5]);
            }
            if (lane < 6) {
                S.obs[2 + lane] = q;
                S.obs[11 + lane] = walker::clip_vel(qd);
            }
        } else if (KIND == PROMP_ENV_SWIMMER) {
            // obs = qpos[2:] ++ qvel (swimmer_rand_vel.py:37-40)
            if (lane < 8) {
                float v = 0.f;
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (lane == k) v = sw[2 + k];
                S.obs[lane] = v;
            }
        } else if (lane == 0) {
            S.obs[0] = sx;
            S.obs[1] = sy;
            if (KIND == PROMP_ENV_POINT_MOMENTUM) S.obs[2] = vx, S.obs[3] = vy;
        }
    };
    write_obs();
    __syncwarp();

    const PointCornerCfg pcfg{A.reward_type, A.radius, A.normalized != 0};
    int path_ts = 0;       // steps taken in the current path (early-termination mode)

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
                Philox::gen((uint32_t)env_id, (uint32_t)t, (uint32_t)A.stream_id,
                            (uint32_t)blk << 24 | (uint32_t)((A.stream_id >> 32) & 0xffffffu), A.seed, r);
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
            // ---- layer 0: h1 = tanh(obs W0 + b0)           (policies/networks/mlp.py:96-117)
            float ob[DO];
#pragma unroll
            for (int i = 0; i < DO; ++i) ob[i] = S.obs[i];
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                float z = b0[u];
#pragma unroll
                for (int i = 0; i < DO; ++i) z = fmaf(ob[i], w0[i][u], z);
                S.h1[lane + 32 * u] = tanh_fast(z);
            }
            // stage obs_t (the observation the action is computed from)
            if (lane < DO) S.st_obs[tt * DO + lane] = S.obs[lane];
            __syncwarp();
            RCLK(2);
            // ---- layer 1: h2 = tanh(h1 W1 + b1); NACC accumulators per output for ILP (4 where the registers allow it)
            constexpr int NACC = (KIND == PROMP_ENV_CHEETAH_DIR || KIND == PROMP_ENV_WALKER) ? 2 : 4;
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
                const float h2 = tanh_fast(NACC == 4 ? (acc[u][0] + acc[u][1]) + (acc[u][2 % NACC] + acc[u][3 % NACC]) : acc[u][0] + acc[u][1]);
#pragma unroll
                for (int d = 0; d < DA; ++d) mu[d] = fmaf(h2, w2[u][d], mu[d]);
            }
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = warp_sum(mu[d]) + b2[d];

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
            float r;
            if (KIND == PROMP_ENV_POINT_CORNER) {
                r = point_corner_step(sx, sy, a[0], a[1], task[0], task[1], pcfg);
            } else if (KIND == PROMP_ENV_POINT) {
                bool dn;
                r = point_step(sx, sy, a[0], a[1], dn, A.normalized != 0);
                if (A.early_term) {
                    // executor semantics (vectorized_env_executor.py:44-52): ts += 1; done |= ts >= max_path_length; a done
                    // env is reset at once and the NEXT observation is the reset state (point_env_2d.py:28-36: U(-2,2)^2,
                    // drawn here from Philox keyed by (env, step) instead of the host numpy stream)
                    ++path_ts;
                    const bool fin = dn || path_ts >= A.horizon;
                    if (lane == 0) S.st_done[tt] = fin ? 1 : 0;
                    if (fin) {
                        uint32_t rr[4];
                        Philox::gen((uint32_t)env_id, (uint32_t)(t0 + tt), (uint32_t)A.stream_id,
                                    0x53000000u | (uint32_t)((A.stream_id >> 32) & 0xffffffu), A.seed, rr);
                        sx = -2.0f + 4.0f * u01(rr[0]);
                        sy = -2.0f + 4.0f * u01(rr[1]);
                        path_ts = 0;
                    }
                }
            } else if (KIND == PROMP_ENV_POINT_WALLS) {
                r = point_walls_step(sx, sy, a[0], a[1], task, A.reward_type, A.normalized != 0);
            } else if (KIND == PROMP_ENV_POINT_MOMENTUM) {
                r = point_momentum_step(sx, sy, vx, vy, a[0], a[1], task[0], task[1], pcfg);
            } else if (KIND == PROMP_ENV_WALKER) {
                float al = 0.f;
                const int jl = lane & 7;
#pragma unroll
                for (int d = 0; d < DA; ++d)
                    if (jl == d) al = a[d];
                const float u_l = jl < 6 ? (A.normalized ? normalized_action(al, -1.f, 1.f) : fminf(fmaxf(al, -1.f), 1.f)) : 0.f;
                float fwd_vel;
                walker::step_warp(wjc, u_l, q, qd, root, task[0], task[TD - 1] != 0.f, r, fwd_vel);
                if (A.early_term) {
                    // as MetaPointEnv above: the root is replicated, so the done decision is warp-uniform
                    ++path_ts;
                    const bool fin = walker::is_done(root[1], root[2]) || path_ts >= A.horizon;
                    if (lane == 0) S.st_done[tt] = fin ? 1 : 0;
                    if (fin) {
                        walker_reset(A, env_id, (uint32_t)(t0 + tt) << 4, 0x53000000u, lane, q, qd, root);
                        path_ts = 0;
                    }
                }
            } else if (KIND == PROMP_ENV_SWIMMER) {
                const float u0 = A.normalized ? normalized_action(a[0], -1.f, 1.f) : fminf(fmaxf(a[0], -1.f), 1.f);
                const float u1 = A.normalized ? normalized_action(a[1], -1.f, 1.f) : fminf(fmaxf(a[1], -1.f), 1.f);
                float r_fwd, r_ctrl;
                swimmer::step(sw, u0, u1, task[0], r, r_fwd, r_ctrl);
                if (lane == 0) {
                    S.st_info[tt] = r_fwd;
                    S.st_info[T_CH + tt] = r_ctrl;
                }
            } else {
                float al = 0.f;
                const int jl = lane & 7;
#pragma unroll
                for (int d = 0; d < DA; ++d)
                    if (jl == d) al = a[d];
                // raw MuJoCo env: ctrlrange clips the torque to [-1, 1] inside the simulator
                const float u_l = jl < 6 ? (A.normalized ? normalized_action(al, -1.f, 1.f) : fminf(fmaxf(al, -1.f), 1.f)) : 0.f;
                float r_run, r_ctrl, fwd_vel;
                cheetah::step_warp(jc, u_l, q, qd, root, task[0], A.reward_type, r, r_run, r_ctrl, fwd_vel);
                if (lane == 0) {
                    S.st_info[tt] = r_run;
                    S.st_info[T_CH + tt] = r_ctrl;
                    S.st_info[2 * T_CH + tt] = fwd_vel;
                }
            }
            if (lane == 0) S.st_rew[tt] = r;
            RCLK(6);
            __syncwarp();      // all lanes are done reading S.obs / S.h1 of this step
            write_obs();
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
                if (T::NINFO > 0 && A.info) {
                    const int64_t tot = (int64_t)A.M * A.E * A.H;
                    A.info[base + t0 + lane] = S.st_info[lane];
                    A.info[tot + base + t0 + lane] = S.st_info[T_CH + lane];
                    if (A.reward_type == 1) A.info[2 * tot + base + t0 + lane] = S.st_info[2 * T_CH + lane];   // RandVel: forward_vel
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
    if (A.final_state) {
        float* fs = A.final_state + env_id * SD;
        if (KIND == PROMP_ENV_CHEETAH_DIR || KIND == PROMP_ENV_WALKER) {
            if (lane == 0) {
                fs[0] = root[0]; fs[1] = root[1]; fs[2] = root[2];
                fs[9] = root[3]; fs[10] = root[4]; fs[11] = root[5];
            }
            if (lane < 6) {
                fs[3 + lane] = q;
                fs[12 + lane] = qd;
            }
        } else if (KIND == PROMP_ENV_SWIMMER) {
            if (lane == 0)
#pragma unroll
                for (int k = 0; k < 10; ++k) fs[k] = sw[k];
        } else if (lane == 0) {
            fs[0] = sx;
            fs[1] = sy;
            if (KIND == PROMP_ENV_POINT_MOMENTUM) fs[2] = vx, fs[3] = vy;
        }
    }
}

// ---------------------------------------------------------------------------- single-step kernels
template <int KIND>
__global__ void env_step_kernel(int reward_type, float radius, int normalized, int n_env, int H, float* state, int32_t* ts,
                                const float* actions, const float* task_params, const float* reset_state,
                                float* next_obs, float* rew, uint8_t* done, float* info) {
    using T = EnvTraits<KIND>;
    constexpr int DO = T::DO, DA = T::DA, SD = T::SD, TD = T::TD;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_env) return;
    float st[SD], a[DA];
#pragma unroll
    for (int k = 0; k < SD; ++k) st[k] = state[(int64_t)i * SD + k];
#pragma unroll
    for (int k = 0; k < DA; ++k) a[k] = actions[(int64_t)i * DA + k];
    float r;
    bool dn = false;
    if (KIND == PROMP_ENV_POINT_CORNER) {
        PointCornerCfg cfg{reward_type, radius, normalized != 0};
        r = point_corner_step(st[0], st[1], a[0], a[1], task_params[(int64_t)i * TD], task_params[(int64_t)i * TD + 1], cfg);
    } else if (KIND == PROMP_ENV_POINT) {
        r = point_step(st[0], st[1], a[0], a[1], dn, normalized != 0);
    } else if (KIND == PROMP_ENV_POINT_WALLS) {
        r = point_walls_step(st[0], st[1], a[0], a[1], task_params + (int64_t)i * TD, reward_type, normalized != 0);
    } else if (KIND == PROMP_ENV_POINT_MOMENTUM) {
        PointCornerCfg cfg{reward_type, radius, normalized != 0};
        r = point_momentum_step(st[0], st[1], st[SD > 2 ? 2 : 0], st[SD > 3 ? 3 : 1], a[0], a[1], task_params[(int64_t)i * TD],
                                task_params[(int64_t)i * TD + 1], cfg);
    } else if (KIND == PROMP_ENV_WALKER) {
        float u[DA], fv;
#pragma unroll
        for (int k = 0; k < DA; ++k) u[k] = normalized ? normalized_action(a[k], -1.f, 1.f) : fminf(fmaxf(a[k], -1.f), 1.f);
        walker::step_serial(st, u, task_params[(int64_t)i * TD], task_params[(int64_t)i * TD + TD - 1] != 0.f, r, fv);
        dn = walker::is_done(st[1], st[2]);
    } else if (KIND == PROMP_ENV_SWIMMER) {
        float s10[10], rf, rc;
#pragma unroll
        for (int k = 0; k < 10; ++k) s10[k] = st[k < SD ? k : 0];
        const float u0 = normalized ? normalized_action(a[0], -1.f, 1.f) : fminf(fmaxf(a[0], -1.f), 1.f);
        const float u1 = normalized ? normalized_action(a[DA > 1 ? 1 : 0], -1.f, 1.f) : fminf(fmaxf(a[DA > 1 ? 1 : 0], -1.f), 1.f);
        swimmer::step(s10, u0, u1, task_params[(int64_t)i * TD], r, rf, rc);
#pragma unroll
        for (int k = 0; k < SD; ++k) st[k] = s10[k < 10 ? k : 0];
        if (info) {
            info[i] = rf;
            info[n_env + i] = rc;
        }
    } else {
        float u[DA], rr, rc, fv;
#pragma unroll
        for (int k = 0; k < DA; ++k) u[k] = normalized ? normalized_action(a[k], -1.f, 1.f) : fminf(fmaxf(a[k], -1.f), 1.f);
        cheetah::step_serial(st, u, task_params[(int64_t)i * TD], reward_type, r, rr, rc, fv);
        if (info) {
            info[i] = rr;
            info[n_env + i] = rc;
            if (reward_type == 1) info[2 * n_env + i] = fv;
        }
    }
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
    if (KIND == PROMP_ENV_CHEETAH_DIR) {
#pragma unroll
        for (int k = 0; k < 8; ++k) next_obs[(int64_t)i * DO + k] = st[1 + k];
#pragma unroll
        for (int k = 0; k < 9; ++k) next_obs[(int64_t)i * DO + 8 + k] = st[9 + k];
    } else if (KIND == PROMP_ENV_WALKER) {
#pragma unroll
        for (int k = 0; k < 8; ++k) next_obs[(int64_t)i * DO + k] = st[1 + k];
#pragma unroll
        for (int k = 0; k < 9; ++k) next_obs[(int64_t)i * DO + 8 + k] = walker::clip_vel(st[9 + k]);
    } else if (KIND == PROMP_ENV_SWIMMER) {
#pragma unroll
        for (int k = 0; k < DO; ++k) next_obs[(int64_t)i * DO + k] = st[2 + k];
    } else {
#pragma unroll
        for (int k = 0; k < DO; ++k) next_obs[(int64_t)i * DO + k] = st[k];       // point envs: obs = state
    }
}

template <int KIND>
__global__ void env_observe_kernel(int n_env, const float* state, float* obs) {
    using T = EnvTraits<KIND>;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_env) return;
    if (KIND == PROMP_ENV_CHEETAH_DIR) {
        for (int k = 0; k < 8; ++k) obs[(int64_t)i * T::DO + k] = state[(int64_t)i * T::SD + 1 + k];
        for (int k = 0; k < 9; ++k) obs[(int64_t)i * T::DO + 8 + k] = state[(int64_t)i * T::SD + 9 + k];
    } else if (KIND == PROMP_ENV_WALKER) {
        for (int k = 0; k < 8; ++k) obs[(int64_t)i * T::DO + k] = state[(int64_t)i * T::SD + 1 + k];
        for (int k = 0; k < 9; ++k) obs[(int64_t)i * T::DO + 8 + k] = walker::clip_vel(state[(int64_t)i * T::SD + 9 + k]);
    } else if (KIND == PROMP_ENV_SWIMMER) {
        for (int k = 0; k < T::DO; ++k) obs[(int64_t)i * T::DO + k] = state[(int64_t)i * T::SD + 2 + k];
    } else {
        for (int k = 0; k < T::DO; ++k) obs[(int64_t)i * T::DO + k] = state[(int64_t)i * T::SD + k];
    }
}

template <int KIND, int HID>
static int launch_rollout(const RolloutArgs& A, cudaStream_t st) {
    dim3 grid((A.E + RO_WARPS - 1) / RO_WARPS, A.M);
    rollout_kernel<KIND, HID><<<grid, RO_WARPS * 32, 0, st>>>(A);
    PROMP_LAUNCH_CHECK("rollout_kernel");
    return PROMP_OK;
}

}  // namespace promp

using namespace promp;

extern "C" int promp_env_state_dim(int env_kind) {
    switch (env_kind) {
        case PROMP_ENV_POINT_CORNER: return 2;
        case PROMP_ENV_POINT: return 2;
        case PROMP_ENV_CHEETAH_DIR: return 18;
        case PROMP_ENV_POINT_WALLS: return 2;
        case PROMP_ENV_POINT_MOMENTUM: return 4;
        case PROMP_ENV_WALKER: return 18;
        case PROMP_ENV_SWIMMER: return 10;
    }
    return -1;
}
extern "C" int promp_env_task_dim(int env_kind) {
    switch (env_kind) {
        case PROMP_ENV_POINT_CORNER: return 2;
        case PROMP_ENV_POINT: return 1;
        case PROMP_ENV_CHEETAH_DIR: return 1;
        case PROMP_ENV_POINT_WALLS: return 6;
        case PROMP_ENV_POINT_MOMENTUM: return 2;
        case PROMP_ENV_WALKER: return 2;
        case PROMP_ENV_SWIMMER: return 1;
    }
    return -1;
}

extern "C" int promp_rollout(int env_kind, int reward_type, float sparse_radius, int normalize_actions, int M, int E, int H,
                             int hidden,
                             const float* params, int64_t param_stride, const float* task_params,
                             const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                             const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs, float* act, float* mean,
                             float* rew, uint8_t* done, float* info, float* log_std_out, float* final_state,
                             void* stream) {
    PROMP_REQUIRE(M > 0 && E > 0 && H > 0, "promp_rollout: M, E, H must be positive (got %d, %d, %d)", M, E, H);
    PROMP_REQUIRE(M <= 65535, "promp_rollout: M=%d exceeds the grid.y limit 65535", M);
    PROMP_REQUIRE(params && task_params && obs && act && mean && rew && done && log_std_out,
                  "promp_rollout: null pointer argument");
    PROMP_REQUIRE(hidden == 64 || hidden == 32, "promp_rollout: hidden size %d unsupported (32 or 64)", hidden);
    PROMP_REQUIRE(reward_type >= 0 && reward_type <= 2, "promp_rollout: bad reward_type %d", reward_type);
    RolloutArgs A{reward_type, sparse_radius, normalize_actions, M, E, H, params, param_stride, task_params, init_state, noise, seed,
                  stream_id, stream_id_dev, clip_reported_log_std, min_log_std, obs, act, mean, rew, done, info, log_std_out,
                  final_state, 0, H};
    cudaStream_t st = (cudaStream_t)stream;
    switch (env_kind) {
        case PROMP_ENV_POINT_CORNER:
            return hidden == 64 ? launch_rollout<PROMP_ENV_POINT_CORNER, 64>(A, st)
                                : launch_rollout<PROMP_ENV_POINT_CORNER, 32>(A, st);
        case PROMP_ENV_CHEETAH_DIR:
            PROMP_REQUIRE(info != nullptr, "promp_rollout: cheetah needs the info buffer [2,M,E,H] ([3,M,E,H] for reward_type 1)");
            PROMP_REQUIRE(reward_type == 0 || reward_type == 1, "promp_rollout: cheetah reward_type must be 0 (RandDirec) or 1 (RandVel)");
            return hidden == 64 ? launch_rollout<PROMP_ENV_CHEETAH_DIR, 64>(A, st)
                                : launch_rollout<PROMP_ENV_CHEETAH_DIR, 32>(A, st);
        case PROMP_ENV_POINT_WALLS:
            PROMP_REQUIRE(reward_type == PROMP_REWARD_DENSE || reward_type == PROMP_REWARD_DENSE_SQUARED,
                          "promp_rollout: the walls env supports reward_type dense / dense_squared");
            return hidden == 64 ? launch_rollout<PROMP_ENV_POINT_WALLS, 64>(A, st) : launch_rollout<PROMP_ENV_POINT_WALLS, 32>(A, st);
        case PROMP_ENV_POINT_MOMENTUM:
            return hidden == 64 ? launch_rollout<PROMP_ENV_POINT_MOMENTUM, 64>(A, st)
                                : launch_rollout<PROMP_ENV_POINT_MOMENTUM, 32>(A, st);
        case PROMP_ENV_WALKER:
            return hidden == 64 ? launch_rollout<PROMP_ENV_WALKER, 64>(A, st) : launch_rollout<PROMP_ENV_WALKER, 32>(A, st);
        case PROMP_ENV_SWIMMER:
            PROMP_REQUIRE(info != nullptr, "promp_rollout: the swimmer needs the info buffer [2,M,E,H]");
            PROMP_REQUIRE(reward_type == 0, "promp_rollout: swimmer reward_type must be 0");
            return hidden == 64 ? launch_rollout<PROMP_ENV_SWIMMER, 64>(A, st) : launch_rollout<PROMP_ENV_SWIMMER, 32>(A, st);
        case PROMP_ENV_POINT:
            set_error("promp_rollout: MetaPointEnv terminates early (variable-length paths); use the stepwise "
                      "sampler (promp_env_step) for it");
            return PROMP_ERR_INVALID_ARG;
    }
    set_error("promp_rollout: unknown env_kind %d", env_kind);
    return PROMP_ERR_INVALID_ARG;
}

// MetaPointEnv (early `done`, point_env_2d.py:9-59) in the fused kernel: every env slot records a timeline of `timeline_len`
// steps; paths end on done / after `horizon` steps and the slot is reset in-kernel.  promp_paths_finalize then applies the
// reference's collect-until-enough rule (meta_sampler.py:87-137) to the timelines.
extern "C" int promp_rollout_early_term(int env_kind, int normalize_actions, int M, int E, int timeline_len, int horizon, int hidden,
                                        const float* params, int64_t param_stride, const float* task_params,
                                        const float* init_state, const float* noise, uint64_t seed, uint64_t stream_id,
                                        const uint64_t* stream_id_dev, int clip_reported_log_std, float min_log_std, float* obs,
                                        float* act, float* mean, float* rew, uint8_t* done, float* log_std_out, void* stream) {
    PROMP_REQUIRE(env_kind == PROMP_ENV_POINT || env_kind == PROMP_ENV_WALKER,
                  "promp_rollout_early_term: implemented for MetaPointEnv and the walker (env_kind %d given)", env_kind);
    PROMP_REQUIRE(M > 0 && E > 0 && timeline_len > 0 && horizon > 0, "promp_rollout_early_term: sizes must be positive");
    PROMP_REQUIRE(M <= 65535, "promp_rollout_early_term: M=%d exceeds the grid.y limit 65535", M);
    PROMP_REQUIRE(params && task_params && obs && act && mean && rew && done && log_std_out,
                  "promp_rollout_early_term: null pointer argument");
    PROMP_REQUIRE(hidden == 64 || hidden == 32, "promp_rollout_early_term: hidden size %d unsupported (32 or 64)", hidden);
    RolloutArgs A{0, 0.f, normalize_actions, M, E, timeline_len, params, param_stride, task_params, init_state, noise, seed,
                  stream_id, stream_id_dev, clip_reported_log_std, min_log_std, obs, act, mean, rew, done, nullptr, log_std_out,
                  nullptr, 1, horizon};
    cudaStream_t st = (cudaStream_t)stream;
    if (env_kind == PROMP_ENV_WALKER)
        return hidden == 64 ? launch_rollout<PROMP_ENV_WALKER, 64>(A, st) : launch_rollout<PROMP_ENV_WALKER, 32>(A, st);
    return hidden == 64 ? launch_rollout<PROMP_ENV_POINT, 64>(A, st) : launch_rollout<PROMP_ENV_POINT, 32>(A, st);
}

__global__ void counter_add_kernel(uint64_t* c, uint64_t inc) { *c += inc; }
extern "C" int promp_counter_add(uint64_t* counter, uint64_t inc, void* stream) {
    PROMP_REQUIRE(counter != nullptr, "promp_counter_add: null counter");
    counter_add_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(counter, inc);
    PROMP_LAUNCH_CHECK("counter_add_kernel");
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
    cudaStream_t st = (cudaStream_t)stream;
    const int bs = 128, gs = (n_env + bs - 1) / bs;
    switch (env_kind) {
        case PROMP_ENV_POINT_CORNER:
            env_step_kernel<PROMP_ENV_POINT_CORNER><<<gs, bs, 0, st>>>(reward_type, sparse_radius, normalize_actions, n_env, H, state, ts,
                                                                       actions, task_params, reset_state, next_obs,
                                                                       rew, done, info);
            break;
        case PROMP_ENV_POINT:
            env_step_kernel<PROMP_ENV_POINT><<<gs, bs, 0, st>>>(reward_type, sparse_radius, normalize_actions, n_env, H, state, ts, actions,
                                                                task_params, reset_state, next_obs, rew, done, info);
            break;
        case PROMP_ENV_CHEETAH_DIR:
            env_step_kernel<PROMP_ENV_CHEETAH_DIR><<<gs, bs, 0, st>>>(reward_type, sparse_radius, normalize_actions, n_env, H, state, ts,
                                                                      actions, task_params, reset_state, next_obs, rew,
                                                                      done, info);
            break;
        case PROMP_ENV_POINT_WALLS:
            env_step_kernel<PROMP_ENV_POINT_WALLS><<<gs, bs, 0, st>>>(reward_type, sparse_radius, normalize_actions, n_env, H, state, ts,
                                                                      actions, task_params, reset_state, next_obs, rew, done, info);
            break;
        case PROMP_ENV_POINT_MOMENTUM:
            env_step_kernel<PROMP_ENV_POINT_MOMENTUM><<<gs, bs, 0, st>>>(reward_type, sparse_radius, normalize_actions, n_env, H, state,
                                                                         ts, actions, task_params, reset_state, next_obs, rew, done, info);
            break;
        case PROMP_ENV_WALKER:
            env_step_kernel<PROMP_ENV_WALKER><<<gs, bs, 0, st>>>(reward_type, sparse_radius, normalize_actions, n_env, H, state, ts,
                                                                 actions, task_params, reset_state, next_obs, rew, done, info);
            break;
        case PROMP_ENV_SWIMMER:
            env_step_kernel<PROMP_ENV_SWIMMER><<<gs, bs, 0, st>>>(reward_type, sparse_radius, normalize_actions, n_env, H, state, ts,
                                                                  actions, task_params, reset_state, next_obs, rew, done, info);
            break;
        default:
            set_error("promp_env_step: unknown env_kind %d", env_kind);
            return PROMP_ERR_INVALID_ARG;
    }
    PROMP_LAUNCH_CHECK("env_step_kernel");
    return PROMP_OK;
}

extern "C" int promp_env_observe(int env_kind, int n_env, const float* state, float* obs, void* stream) {
    PROMP_REQUIRE(n_env > 0 && state && obs, "promp_env_observe: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const int bs = 128, gs = (n_env + bs - 1) / bs;
    switch (env_kind) {
        case PROMP_ENV_POINT_CORNER: env_observe_kernel<PROMP_ENV_POINT_CORNER><<<gs, bs, 0, st>>>(n_env, state, obs); break;
        case PROMP_ENV_POINT: env_observe_kernel<PROMP_ENV_POINT><<<gs, bs, 0, st>>>(n_env, state, obs); break;
        case PROMP_ENV_CHEETAH_DIR: env_observe_kernel<PROMP_ENV_CHEETAH_DIR><<<gs, bs, 0, st>>>(n_env, state, obs); break;
        case PROMP_ENV_POINT_WALLS: env_observe_kernel<PROMP_ENV_POINT_WALLS><<<gs, bs, 0, st>>>(n_env, state, obs); break;
        case PROMP_ENV_POINT_MOMENTUM: env_observe_kernel<PROMP_ENV_POINT_MOMENTUM><<<gs, bs, 0, st>>>(n_env, state, obs); break;
        case PROMP_ENV_WALKER: env_observe_kernel<PROMP_ENV_WALKER><<<gs, bs, 0, st>>>(n_env, state, obs); break;
        case PROMP_ENV_SWIMMER: env_observe_kernel<PROMP_ENV_SWIMMER><<<gs, bs, 0, st>>>(n_env, state, obs); break;
        default:
            set_error("promp_env_observe: unknown env_kind %d", env_kind);
            return PROMP_ERR_INVALID_ARG;
    }
    PROMP_LAUNCH_CHECK("env_observe_kernel");
    return PROMP_OK;
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
