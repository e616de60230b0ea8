// Analytic environments of the ProMP hot path as device functions (float32).
//   point corner : ref envs/point_envs/point_env_2d_corner.py:22-81
//   point        : ref envs/point_envs/point_env_2d.py:9-59
//   cheetah      : MuJoCo-free HalfCheetahRandDirec surrogate; reward / obs / reset / task spec follow
//                  ref envs/mujoco_envs/half_cheetah_rand_direc.py:14-53, the dynamics are defined in
//                  DESIGN.md (restated on the CPU in oracle/cheetah_surrogate.py).
//   walker       : MuJoCo-free Walker2DRandVel / Walker2DRandDirec surrogate (ref envs/mujoco_envs/walker2d_rand_vel.py,
//                  walker2d_rand_direc.py), early `done` when the torso falls.
//   swimmer      : MuJoCo-free SwimmerRandVel surrogate (ref envs/mujoco_envs/swimmer_rand_vel.py).
//                  Both restated on the CPU in oracle/locomotion_surrogates.py.
//   NormalizedEnv: ref envs/normalized_env.py:109-117 (action affine map + clip; obs / reward
//                  normalisation are off by default, :23-24, and out of scope).
//
// Each environment is one type (PointCorner, Point, PointWalls, PointMomentum, Cheetah, Walker, Swimmer) with
//   KIND (PROMP_ENV_*), DO / DA (obs / action size), SD (floats of an init_state / final_state / reset_state row),
//   TD (floats per task), NINFO (env_infos channels), NACC (rollout layer-1 accumulators: 2 where the env's registers
//   leave no room for 4), ENDS_EARLY (the env reports `done` before the horizon);
//   warp-resident state for rollout_kernel, one warp per env:
//     load(init_state row, lane), reset(rng, step, tag, lane, task) (Philox draw), observe(shared obs line, lane),
//     step(a, task, cfg, lane, info, info_stride, done) -> reward, store(final_state row, lane);
//   one thread per env for env_step_kernel / env_observe_kernel:
//     step_serial(st[SD], a, task, cfg, info, info_stride, done) -> reward, observe_serial(st, obs).
// `info` is NULL or channel 0 of the env_infos record, channel c at info[c * info_stride].
#pragma once
#include "common.cuh"

namespace promp {

// step configuration every env receives
struct EnvCfg {
    int reward_type;
    float radius;       // sparse reward radius
    bool normalized;    // actions pass through the NormalizedEnv map
};

// Philox stream of one env slot: counter (env, ctr, stream_id low word, tag | stream_id bits 32-55), key = seed
struct EnvRng {
    uint32_t env, stream_lo, stream_hi;
    uint64_t seed;
    __device__ __forceinline__ void gen(uint32_t ctr, uint32_t tag, uint32_t (&r)[4]) const {
        Philox::gen(env, ctr, stream_lo, tag | stream_hi, seed, r);
    }
};

// NormalizedEnv.step action map, same evaluation order as the reference expression
//   lb + (a + scale) * (ub - lb) / (2*scale), then clip to [lb, ub]       (normalization_scale = 10)
__device__ __forceinline__ float normalized_action(float a, float lb, float ub) {
    float s = lb + ((a + 10.0f) * (ub - lb)) / 20.0f;
    return fminf(fmaxf(s, lb), ub);
}
// wrapped (normalize(env), every reference run script) or raw env (the reference's tests): the raw env receives the
// policy action unchanged and applies only its own clip to [-lim, lim] (point_env_2d_corner.py:37; the identity after
// the wrapper's clip)
__device__ __forceinline__ float env_action(float a, float lim, bool normalized) {
    const float e = normalized ? normalized_action(a, -lim, lim) : a;
    return fminf(fmaxf(e, -lim), lim);
}
// MuJoCo envs: the raw env's ctrlrange clips the torque to [-1, 1] inside the simulator
__device__ __forceinline__ float ctrl_action(float a, bool normalized) { return env_action(a, 1.f, normalized); }

// sqrt.approx (MUFU.RSQ-based, max relative error 2^-23 per the PTX ISA, i.e. within 1 ulp of sqrtf) without sqrtf's
// fix-up sequence and slow-path branch: the sparse reward needs five to six distances per env step and the branches
// serialised them (617 clk of a 1644 clk env step went here; tools/rollout_time.py).
__device__ __forceinline__ float sqrt_fast(float x) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float dist2d(float x, float y, float gx, float gy) {
    float dx = x - gx, dy = y - gy;
    return sqrt_fast(dx * dx + dy * dy);
}

// State that every lane of the env's warp holds and advances identically: the warp step is the serial step on that copy
// and lane 0 writes what leaves the warp.
template <class Env, int SD>
struct Replicated {
    float s[SD];
    __device__ __forceinline__ void load(const float* s0, int) {
#pragma unroll
        for (int k = 0; k < SD; ++k) s[k] = s0[k];
    }
    __device__ __forceinline__ void store(float* fs, int lane) const {
        if (lane == 0)
#pragma unroll
            for (int k = 0; k < SD; ++k) fs[k] = s[k];
    }
    __device__ __forceinline__ void observe(float* obs, int lane) const {
        if (lane == 0) Env::observe_serial(s, obs);
    }
    __device__ __forceinline__ float step(const float* a, const float* task, const EnvCfg& cfg, int lane, float* info,
                                          int info_stride, bool& done) {
        return Env::step_serial(s, a, task, cfg, lane == 0 ? info : nullptr, info_stride, done);
    }
};

// point envs: obs = state = position (++ velocity for the momentum env).  reset (point_env_2d_corner.py:50 /
// point_env_2d.py:34 / point_env_2d_momentum.py:52): position U(-RESET_LIM, RESET_LIM)^2, velocity U(-.1,.1)^2, from
// counter `step`.
template <class Env, int SD>
struct PointState : Replicated<Env, SD> {
    __device__ __forceinline__ void reset(const EnvRng& rng, uint32_t step, uint32_t tag, int, const float*) {
        uint32_t r[4];
        rng.gen(step, tag, r);
        const float lim = Env::RESET_LIM;
        this->s[0] = -lim + 2.f * lim * u01(r[0]);
        this->s[1] = -lim + 2.f * lim * u01(r[1]);
        if constexpr (SD == 4) this->s[2] = -0.1f + 0.2f * u01(r[2]), this->s[3] = -0.1f + 0.2f * u01(r[3]);
    }
    static __device__ __forceinline__ void observe_serial(const float* st, float* obs) {
#pragma unroll
        for (int k = 0; k < SD; ++k) obs[k] = st[k];
    }
};

// ------------------------------------------------------------------ point corner
struct PointCorner : PointState<PointCorner, 2> {
    static constexpr int KIND = PROMP_ENV_POINT_CORNER, DO = 2, DA = 2, SD = 2, TD = 2, NINFO = 0, NACC = 4;
    static constexpr bool ENDS_EARLY = false;
    static constexpr float RESET_LIM = 0.2f;
    // s (in/out): state; a: policy-space action; task: goal.  Returns reward.
    static __device__ __forceinline__ float step_serial(float (&s)[SD], const float* a, const float* task, const EnvCfg& cfg,
                                                        float*, int, bool&) {
        float &sx = s[0], &sy = s[1];
        const float gx = task[0], gy = task[1];
        const float ex = env_action(a[0], 0.2f, cfg.normalized), ey = env_action(a[1], 0.2f, cfg.normalized);
        float px = sx, py = sy;
        sx = px + ex;
        sy = py + ey;
        float r;
        if (cfg.reward_type == PROMP_REWARD_DENSE) {
            r = -dist2d(sx, sy, gx, gy);
        } else if (cfg.reward_type == PROMP_REWARD_DENSE_SQUARED) {
            float g = dist2d(sx, sy, gx, gy);
            r = -(g * g);
        } else {
            // sparse (:68-75): 0 inside the L1 radius; progress toward the goal iff the goal is the nearest corner
            float d0 = dist2d(sx, sy, -2.f, -2.f), d1 = dist2d(sx, sy, 2.f, -2.f);
            float d2 = dist2d(sx, sy, -2.f, 2.f), d3 = dist2d(sx, sy, 2.f, 2.f);
            float dmin = fminf(fminf(d0, d1), fminf(d2, d3));
            float g;   // take the goal distance from the same four values when the goal is a corner (exact ==)
            if (gx == -2.f && gy == -2.f) g = d0;
            else if (gx == 2.f && gy == -2.f) g = d1;
            else if (gx == -2.f && gy == 2.f) g = d2;
            else if (gx == 2.f && gy == 2.f) g = d3;
            else g = dist2d(sx, sy, gx, gy);
            r = 0.f;
            if (!(fabsf(sx) + fabsf(sy) < cfg.radius) && g == dmin) r = dist2d(px, py, gx, gy) - g;
        }
        return r;
    }
};

// ------------------------------------------------------------------ point (origin goal, early done)
struct Point : PointState<Point, 2> {
    static constexpr int KIND = PROMP_ENV_POINT, DO = 2, DA = 2, SD = 2, TD = 1, NINFO = 0, NACC = 4;
    static constexpr bool ENDS_EARLY = true;
    static constexpr float RESET_LIM = 2.0f;
    static __device__ __forceinline__ float step_serial(float (&s)[SD], const float* a, const float*, const EnvCfg& cfg, float*,
                                                        int, bool& done) {
        float &sx = s[0], &sy = s[1];
        const float ex = env_action(a[0], 0.1f, cfg.normalized), ey = env_action(a[1], 0.1f, cfg.normalized);
        sx += ex;
        sy += ey;
        done = (fabsf(sx) < 0.01f) && (fabsf(sy) < 0.01f);
        return -sqrt_fast(sx * sx + sy * sy);
    }
};

// ------------------------------------------------------------------ point walls (ref point_env_2d_walls.py:22-51)
// s' = s + clip(a, +-0.2); the reward is taken at s' BEFORE the wall logic (:37-39); crossing the unit circle outside
// gap_1 (distance > 1 from the gap centre) projects s' back to just inside radius 1, crossing the radius-2 circle
// outside gap_2 to just inside radius 2 (:40-49).  reward_type dense / dense_squared (the reference's 'sparse' branch
// returns None outside the radius and cannot be sampled).
struct PointWalls : PointState<PointWalls, 2> {
    static constexpr int KIND = PROMP_ENV_POINT_WALLS, DO = 2, DA = 2, SD = 2, TD = 6, NINFO = 0, NACC = 4;   // task = goal, gap_1, gap_2
    static constexpr bool ENDS_EARLY = false;
    static constexpr float RESET_LIM = 0.2f;
    static __device__ __forceinline__ float step_serial(float (&s)[SD], const float* a, const float* task, const EnvCfg& cfg,
                                                        float*, int, bool&) {
        float &sx = s[0], &sy = s[1];
        const float ex = env_action(a[0], 0.2f, cfg.normalized), ey = env_action(a[1], 0.2f, cfg.normalized);
        const float px = sx, py = sy;
        float nx = px + ex, ny = py + ey;
        const float g = dist2d(nx, ny, task[0], task[1]);
        const float r = (cfg.reward_type == PROMP_REWARD_DENSE_SQUARED) ? -(g * g) : -g;
        const float pn = sqrt_fast(px * px + py * py), nn = sqrt_fast(nx * nx + ny * ny);
        if (pn < 1.f && nn > 1.f) {
            if (dist2d(nx, ny, task[2], task[3]) > 1.f) {
                const float inv = 1.f / (nn + 1e-6f);
                nx *= inv, ny *= inv;
            }
        } else if (pn < 2.f && nn > 2.f) {
            if (dist2d(nx, ny, task[4], task[5]) > 1.f) {
                const float inv = 1.f / (nn * 0.5f + 1e-6f);
                nx *= inv, ny *= inv;
            }
        }
        sx = nx, sy = ny;
        return r;
    }
};

// ------------------------------------------------------------------ point momentum (ref point_env_2d_momentum.py:22-42, 58-68)
// v' = v + clip(a, +-0.1); s' = s + v'; obs = (s', v'); reward at s': sparse (default) = max(radius - |s' - goal|, 0)
struct PointMomentum : PointState<PointMomentum, 4> {
    static constexpr int KIND = PROMP_ENV_POINT_MOMENTUM, DO = 4, DA = 2, SD = 4, TD = 2, NINFO = 0, NACC = 4;   // state = (pos, vel)
    static constexpr bool ENDS_EARLY = false;
    static constexpr float RESET_LIM = 0.2f;
    static __device__ __forceinline__ float step_serial(float (&s)[SD], const float* a, const float* task, const EnvCfg& cfg,
                                                        float*, int, bool&) {
        float &sx = s[0], &sy = s[1], &vx = s[2], &vy = s[3];
        const float gx = task[0], gy = task[1];
        const float ex = env_action(a[0], 0.1f, cfg.normalized), ey = env_action(a[1], 0.1f, cfg.normalized);
        vx += ex, vy += ey;
        sx += vx, sy += vy;
        const float g = dist2d(sx, sy, gx, gy);
        if (cfg.reward_type == PROMP_REWARD_DENSE) return -g;
        if (cfg.reward_type == PROMP_REWARD_DENSE_SQUARED) return -(g * g);
        return fmaxf(cfg.radius - g, 0.f);
    }
};

// ------------------------------------------------------------------ planar 9-DoF state (cheetah, walker)
// state row = qpos[9] ++ qvel[9], qpos = root (x, z, pitch) ++ joint[6].  In the warp, lane j < 6 owns joint j (q, qd) and
// the six root floats (x, z, pitch, xd, zd, pd) are replicated in every lane.  obs = qpos[1:] ++ qvel
// (half_cheetah_rand_direc.py:43-47); CLIP_VEL: the walker's obs clips qvel to [-10, 10] (walker2d_rand_*.py:42-45).
template <bool CLIP_VEL>
struct Planar9 {
    float q, qd, root[6];

    static __device__ __forceinline__ float obs_vel(float v) { return CLIP_VEL ? fminf(fmaxf(v, -10.0f), 10.0f) : v; }

    __device__ __forceinline__ void load(const float* s0, int lane) {
        const int jl = lane & 7;
        root[0] = s0[0]; root[1] = s0[1]; root[2] = s0[2];
        root[3] = s0[9]; root[4] = s0[10]; root[5] = s0[11];
        q = jl < 6 ? s0[3 + jl] : 0.f;
        qd = jl < 6 ? s0[12 + jl] : 0.f;
    }
    __device__ __forceinline__ void store(float* fs, int lane) const {
        if (lane == 0) {
            fs[0] = root[0]; fs[1] = root[1]; fs[2] = root[2];
            fs[9] = root[3]; fs[10] = root[4]; fs[11] = root[5];
        }
        if (lane < 6) {
            fs[3 + lane] = q;
            fs[12 + lane] = qd;
        }
    }
    __device__ __forceinline__ void observe(float* obs, int lane) const {
        if (lane == 0) {
            obs[0] = root[1]; obs[1] = root[2];
            obs[8] = obs_vel(root[3]); obs[9] = obs_vel(root[4]); obs[10] = obs_vel(root[5]);
        }
        if (lane < 6) {
            obs[2 + lane] = q;
            obs[11 + lane] = obs_vel(qd);
        }
    }
    static __device__ __forceinline__ void observe_serial(const float* st, float* obs) {
#pragma unroll
        for (int k = 0; k < 8; ++k) obs[k] = st[1 + k];
#pragma unroll
        for (int k = 0; k < 9; ++k) obs[8 + k] = obs_vel(st[9 + k]);
    }
    // spreads a reset draw over the warp: lane i < 9 holds coordinate i of qpos (pos) and of qvel (vel)
    __device__ __forceinline__ void spread(float pos, float vel, int lane) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            root[i] = __shfl_sync(0xffffffffu, pos, i);
            root[3 + i] = __shfl_sync(0xffffffffu, vel, i);
        }
        const int jl = lane & 7;
        const float qq = __shfl_sync(0xffffffffu, pos, 3 + (jl < 6 ? jl : 0));
        const float qv = __shfl_sync(0xffffffffu, vel, 3 + (jl < 6 ? jl : 0));
        q = jl < 6 ? qq : 0.f;
        qd = jl < 6 ? qv : 0.f;
    }
    // this lane's joint torque: the clipped control of action lane & 7, 0 on lanes 6 and 7
    static __device__ __forceinline__ float joint_ctrl(const float* a, int lane, bool normalized) {
        float al = 0.f;
        const int jl = lane & 7;
#pragma unroll
        for (int d = 0; d < 6; ++d)
            if (jl == d) al = a[d];
        return jl < 6 ? ctrl_action(al, normalized) : 0.f;
    }
};

// ------------------------------------------------------------------ cheetah surrogate
namespace cheetah {
constexpr int NJ = 6;
constexpr float HS = 0.01f, DT = 0.05f;
constexpr int FRAME_SKIP = 5;
static __device__ __constant__ const float G[8] = {12.0f, 9.0f, 6.0f, 12.0f, 6.0f, 3.0f, 0.f, 0.f};
static __device__ __constant__ const float K[8] = {24.0f, 18.0f, 12.0f, 18.0f, 12.0f, 6.0f, 0.f, 0.f};
static __device__ __constant__ const float D[8] = {4.5f, 3.0f, 1.5f, 3.0f, 1.5f, 0.75f, 0.f, 0.f};
static __device__ __constant__ const float C[8] = {0.9f, 0.6f, 0.3f, -0.8f, -0.5f, -0.25f, 0.f, 0.f};
static __device__ __constant__ const float PH[8] = {0.3f, -0.4f, 0.8f, -0.3f, 0.5f, -0.9f, 0.f, 0.f};
static __device__ __constant__ const float P[8] = {0.6f, 0.4f, 0.2f, -0.6f, -0.4f, -0.2f, 0.f, 0.f};
constexpr float BX = 1.5f, LZ = 0.1f, KZ = 40.0f, DZ = 6.0f, KP = 30.0f, DP = 5.0f;

struct JointConst {
    float g, k, d, c, ph, p;
};
__device__ __forceinline__ JointConst joint_const(int j) {
    int i = j < NJ ? j : 7;
    return JointConst{G[i], K[i], D[i], C[i], PH[i], P[i]};
}

// root: x, z, pitch, xd, zd, pd
// Serial version (one thread per env): state = qpos[9] ++ qvel[9]; u[6] already rescaled+clipped.
// mode 0: HalfCheetahRandDirec, r_run = task * v (task = direction);  mode 1: HalfCheetahRandVel, r_run = -|v - task| (task = goal
// velocity; half_cheetah_rand_vel.py:30-40).  fwd_vel = (x_after - x_before) / dt.
__device__ inline void step_serial(float* st, const float* u, float task, int mode, float& reward, float& r_run, float& r_ctrl,
                                   float& fwd_vel) {
    float x0 = st[0];
    for (int s = 0; s < FRAME_SKIP; ++s) {
        float thrust = 0.f, lift = 0.f, twist = 0.f;
        float pitch = st[2];
        for (int j = 0; j < NJ; ++j) {
            float q = st[3 + j], qd = st[12 + j];
            float acc = G[j] * u[j] - K[j] * q - D[j] * qd;
            qd = qd + HS * acc;
            q = q + HS * qd;
            st[3 + j] = q;
            st[12 + j] = qd;
            float sn, cs;
            __sincosf(q + pitch + PH[j], &sn, &cs);   // |angle| stays O(1): fast path error ~5e-7
            thrust = thrust + C[j] * qd * sn;
            lift = lift + C[j] * qd * cs;
            twist = twist + P[j] * u[j];
        }
        float xd = st[9] + HS * (thrust - BX * st[9]);
        st[9] = xd;
        st[0] = st[0] + HS * xd;
        float zd = st[10] + HS * (LZ * lift - KZ * st[1] - DZ * st[10]);
        st[10] = zd;
        st[1] = st[1] + HS * zd;
        float pd = st[11] + HS * (twist - KP * st[2] - DP * st[11]);
        st[11] = pd;
        st[2] = st[2] + HS * pd;
    }
    float su = 0.f;
    for (int j = 0; j < NJ; ++j) su += u[j] * u[j];
    r_ctrl = -0.05f * su;
    fwd_vel = (st[0] - x0) / DT;
    r_run = mode ? -fabsf(fwd_vel - task) : task * fwd_vel;
    reward = r_ctrl + r_run;
}

// Warp version: lane j < 6 owns joint j (q, qd, torque u); the six root floats are replicated in
// every lane and stay bit-identical because the 8-lane xor reductions are symmetric.
__device__ __forceinline__ float sum8(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    return v;
}
__device__ __forceinline__ void step_warp(const JointConst& jc, float u, float& q, float& qd, float (&root)[6], float task, int mode,
                                          float& reward, float& r_run, float& r_ctrl, float& fwd_vel) {
    // The joints (q, qd) and the pitch (root[2], root[5]) evolve independently of the two quantities that need a
    // reduction over the joints (thrust -> x, lift -> z), and the x / z recurrences are LINEAR in thrust / lift.  So every
    // lane integrates the response of (xd, x, zd, z) to ITS OWN joint's thrust / lift from zero initial conditions, all
    // lanes integrate the homogeneous part from the real initial conditions, and one 8-lane reduction per env step (instead
    // of two per sub-step on the critical path: 1 790 -> ~600 clk per step, tools/rollout_time.py) adds them up.  Same
    // equations as step_serial / oracle/cheetah_surrogate.py; the summation order differs at float32 round-off.
    const float x0 = root[0];
    const float twist = sum8(jc.p * u);          // the torques are constant over the sub-steps
    const float su = sum8(u * u);
    float xdh = root[3], xh = root[0], zdh = root[4], zh = root[1];      // homogeneous parts
    float xdp = 0.f, xp = 0.f, zdp = 0.f, zp = 0.f;                      // this lane's driven parts
    float pitch = root[2], pd = root[5];
#pragma unroll
    for (int s = 0; s < FRAME_SKIP; ++s) {
        const float acc = jc.g * u - jc.k * q - jc.d * qd;
        qd = qd + HS * acc;
        q = q + HS * qd;
        float sn, cs;
        __sincosf(q + pitch + jc.ph, &sn, &cs);   // pitch of the START of the sub-step, as in step_serial
        const float t = jc.c * qd * sn, l = jc.c * qd * cs;
        xdp = xdp + HS * (t - BX * xdp);
        xp = xp + HS * xdp;
        zdp = zdp + HS * (LZ * l - KZ * zp - DZ * zdp);
        zp = zp + HS * zdp;
        xdh = xdh + HS * (0.f - BX * xdh);
        xh = xh + HS * xdh;
        zdh = zdh + HS * (0.f - KZ * zh - DZ * zdh);
        zh = zh + HS * zdh;
        pd = pd + HS * (twist - KP * pitch - DP * pd);
        pitch = pitch + HS * pd;
    }
    root[3] = xdh + sum8(xdp);
    root[0] = xh + sum8(xp);
    root[4] = zdh + sum8(zdp);
    root[1] = zh + sum8(zp);
    root[5] = pd;
    root[2] = pitch;
    r_ctrl = -0.05f * su;
    fwd_vel = (root[0] - x0) / DT;
    r_run = mode ? -fabsf(fwd_vel - task) : task * fwd_vel;
    reward = r_ctrl + r_run;
}
}  // namespace cheetah

// task = direction (reward_type 0, RandDirec) or goal velocity (reward_type 1, RandVel);
// info = reward_run, reward_ctrl (++ forward_vel for RandVel)
struct Cheetah : Planar9<false> {
    static constexpr int KIND = PROMP_ENV_CHEETAH_DIR, DO = 17, DA = 6, SD = 18, TD = 1, NINFO = 2, NACC = 2;
    static constexpr bool ENDS_EARLY = false;
    cheetah::JointConst jc = cheetah::joint_const(threadIdx.x & 7);   // this lane's joint (lane & 7)

    // reset_model (half_cheetah_rand_direc.py:49-53): qpos = U(-.1,.1)^9, qvel = .1*N(0,1)^9; lane i < 9 draws coordinate
    // i from counter (step << 4) + i
    __device__ __forceinline__ void reset(const EnvRng& rng, uint32_t step, uint32_t tag, int lane, const float*) {
        float pos = 0.f, vel = 0.f;
        if (lane < 9) {
            uint32_t r[4];
            rng.gen((step << 4) + (uint32_t)lane, tag, r);
            pos = -0.1f + 0.2f * u01(r[0]);
            float z0, z1;
            box_muller(r[1], r[2], z0, z1);
            vel = 0.1f * z0;
        }
        spread(pos, vel, lane);
    }
    __device__ __forceinline__ float step(const float* a, const float* task, const EnvCfg& cfg, int lane, float* info,
                                          int info_stride, bool&) {
        float r, r_run, r_ctrl, fwd_vel;
        cheetah::step_warp(jc, joint_ctrl(a, lane, cfg.normalized), q, qd, root, task[0], cfg.reward_type, r, r_run, r_ctrl,
                           fwd_vel);
        if (lane == 0) {
            info[0] = r_run;
            info[info_stride] = r_ctrl;
            info[2 * info_stride] = fwd_vel;
        }
        return r;
    }
    static __device__ __forceinline__ float step_serial(float (&st)[SD], const float* a, const float* task, const EnvCfg& cfg,
                                                        float* info, int info_stride, bool&) {
        float u[DA], r, r_run, r_ctrl, fwd_vel;
#pragma unroll
        for (int k = 0; k < DA; ++k) u[k] = ctrl_action(a[k], cfg.normalized);
        cheetah::step_serial(st, u, task[0], cfg.reward_type, r, r_run, r_ctrl, fwd_vel);
        if (info) {
            info[0] = r_run;
            info[info_stride] = r_ctrl;
            if (cfg.reward_type == 1) info[2 * info_stride] = fwd_vel;
        }
        return r;
    }
};

// ------------------------------------------------------------------ walker2d surrogate
// MuJoCo-free Walker2DRandVel / Walker2DRandDirec: obs / reward / done / reset follow ref envs/mujoco_envs/
// walker2d_rand_vel.py:32-55 and walker2d_rand_direc.py:32-55; the dynamics are defined in DESIGN.md §3.4 and restated
// on the CPU in oracle/locomotion_surrogates.py.  State = qpos[9] ++ qvel[9] with root (x, z, pitch) like the cheetah;
// the torso is an inverted pendulum, so a path ends (done) once it has fallen.
namespace walker {
constexpr int NJ = 6;
constexpr float HS = 0.002f, DT = 0.016f;
constexpr int FRAME_SKIP = 8;
static __device__ __constant__ const float G[8] = {6.0f, 5.0f, 3.0f, 6.0f, 5.0f, 3.0f, 0.f, 0.f};
static __device__ __constant__ const float K[8] = {20.0f, 16.0f, 10.0f, 20.0f, 16.0f, 10.0f, 0.f, 0.f};
static __device__ __constant__ const float D[8] = {3.0f, 2.5f, 1.5f, 3.0f, 2.5f, 1.5f, 0.f, 0.f};
static __device__ __constant__ const float C[8] = {0.8f, 0.6f, 0.3f, 0.8f, 0.6f, 0.3f, 0.f, 0.f};
static __device__ __constant__ const float PH[8] = {0.4f, -0.3f, 0.9f, -0.4f, 0.3f, -0.9f, 0.f, 0.f};
static __device__ __constant__ const float P[8] = {1.2f, -0.8f, 0.5f, -1.0f, 0.9f, -0.6f, 0.f, 0.f};
constexpr float BX = 1.0f, Z0 = 1.25f, KZ = 60.0f, DZ = 12.0f, LZ = 0.5f, AP = 5.0f, DP = 0.5f;

struct JointConst {
    float g, k, d, c, ph, p;
};
__device__ __forceinline__ JointConst joint_const(int j) {
    int i = j < NJ ? j : 7;
    return JointConst{G[i], K[i], D[i], C[i], PH[i], P[i]};
}

// walker2d_rand_*.py:36-37: done = not (0.8 < height < 2.0 and -1 < angle < 1)
__device__ __forceinline__ bool is_done(float z, float ang) {
    return !(z > 0.8f && z < 2.0f && ang > -1.0f && ang < 1.0f);
}

// mode 0: RandDirec, reward = dir * fwd_vel + 1 - 1e-3 |u|^2;  mode 1: RandVel, reward = -|fwd_vel - goal| + 15 - 1e-3 |u|^2
__device__ __forceinline__ float reward(float fwd_vel, float su, float task, int mode) {
    return (mode ? -fabsf(fwd_vel - task) + 15.0f : task * fwd_vel + 1.0f) - 1e-3f * su;
}

// Serial version (one thread per env): state = qpos[9] ++ qvel[9]; u[6] already clipped.
__device__ inline void step_serial(float* st, const float* u, float task, int mode, float& rew, float& fwd_vel) {
    const float x0 = st[0];
    float twist = 0.f, su = 0.f;
    for (int j = 0; j < NJ; ++j) twist = twist + P[j] * u[j];
    for (int s = 0; s < FRAME_SKIP; ++s) {
        float thrust = 0.f, lift = 0.f;
        const float pitch = st[2];
        for (int j = 0; j < NJ; ++j) {
            float q = st[3 + j], qd = st[12 + j];
            const float acc = G[j] * u[j] - K[j] * q - D[j] * qd;
            qd = qd + HS * acc;
            q = q + HS * qd;
            st[3 + j] = q;
            st[12 + j] = qd;
            float sn, cs;
            __sincosf(q + pitch + PH[j], &sn, &cs);
            thrust = thrust + C[j] * qd * sn;
            lift = lift + C[j] * qd * cs;
        }
        float psn, pcs;
        __sincosf(pitch, &psn, &pcs);
        const float xd = st[9] + HS * (thrust - BX * st[9]);
        st[9] = xd;
        st[0] = st[0] + HS * xd;
        const float zd = st[10] + HS * (KZ * (Z0 * pcs - st[1]) - DZ * st[10] + LZ * lift);
        st[10] = zd;
        st[1] = st[1] + HS * zd;
        const float pd = st[11] + HS * (AP * psn + twist - DP * st[11]);
        st[11] = pd;
        st[2] = pitch + HS * pd;
    }
    for (int j = 0; j < NJ; ++j) su += u[j] * u[j];
    fwd_vel = (st[0] - x0) / DT;
    rew = reward(fwd_vel, su, task, mode);
}

// Warp version, the cheetah's decomposition (cheetah::step_warp): lane j < 6 owns joint j, the root floats are
// replicated.  The pitch depends on the torques only (constant over the sub-steps), so every lane integrates it; x and z
// are LINEAR in the per-joint thrust / lift, so every lane integrates its own joint's driven response from zero and the
// homogeneous part (with the replicated Z0*cos(pitch) drive) from the real initial conditions; one 8-lane reduction per
// env step adds them up.
__device__ __forceinline__ void step_warp(const JointConst& jc, float u, float& q, float& qd, float (&root)[6], float task, int mode,
                                          float& rew, float& fwd_vel) {
    const float x0 = root[0];
    const float twist = cheetah::sum8(jc.p * u);
    const float su = cheetah::sum8(u * u);
    float xdh = root[3], xh = root[0], zdh = root[4], zh = root[1];
    float xdp = 0.f, xp = 0.f, zdp = 0.f, zp = 0.f;
    float pitch = root[2], pd = root[5];
#pragma unroll
    for (int s = 0; s < FRAME_SKIP; ++s) {
        const float acc = jc.g * u - jc.k * q - jc.d * qd;
        qd = qd + HS * acc;
        q = q + HS * qd;
        float sn, cs, psn, pcs;
        __sincosf(q + pitch + jc.ph, &sn, &cs);
        __sincosf(pitch, &psn, &pcs);
        const float t = jc.c * qd * sn, l = jc.c * qd * cs;
        xdp = xdp + HS * (t - BX * xdp);
        xp = xp + HS * xdp;
        zdp = zdp + HS * (LZ * l - KZ * zp - DZ * zdp);
        zp = zp + HS * zdp;
        xdh = xdh + HS * (0.f - BX * xdh);
        xh = xh + HS * xdh;
        zdh = zdh + HS * (KZ * (Z0 * pcs - zh) - DZ * zdh);
        zh = zh + HS * zdh;
        pd = pd + HS * (AP * psn + twist - DP * pd);
        pitch = pitch + HS * pd;
    }
    root[3] = xdh + cheetah::sum8(xdp);
    root[0] = xh + cheetah::sum8(xp);
    root[4] = zdh + cheetah::sum8(zdp);
    root[1] = zh + cheetah::sum8(zp);
    root[5] = pd;
    root[2] = pitch;
    fwd_vel = (root[0] - x0) / DT;
    rew = reward(fwd_vel, su, task, mode);
}
}  // namespace walker

// task = (direction | goal velocity, reward mode)
struct Walker : Planar9<true> {
    static constexpr int KIND = PROMP_ENV_WALKER, DO = 17, DA = 6, SD = 18, TD = 2, NINFO = 0, NACC = 2;
    static constexpr bool ENDS_EARLY = true;
    walker::JointConst jc = walker::joint_const(threadIdx.x & 7);     // this lane's joint (lane & 7)

    // reset_model (walker2d_rand_*.py:47-52): qpos = init_qpos + U(-.005,.005)^9 (init_qpos z = 1.25, all else 0),
    // qvel = U(-.005,.005)^9; lane i < 9 draws coordinate i from counter (step << 4) + i
    __device__ __forceinline__ void reset(const EnvRng& rng, uint32_t step, uint32_t tag, int lane, const float*) {
        float pos = 0.f, vel = 0.f;
        if (lane < 9) {
            uint32_t r[4];
            rng.gen((step << 4) + (uint32_t)lane, tag, r);
            pos = -0.005f + 0.01f * u01(r[0]);
            vel = -0.005f + 0.01f * u01(r[1]);
        }
        spread(pos, vel, lane);
        root[1] += 1.25f;
    }
    // the root is replicated, so `done` is warp-uniform
    __device__ __forceinline__ float step(const float* a, const float* task, const EnvCfg& cfg, int lane, float*, int,
                                          bool& done) {
        float r, fwd_vel;
        walker::step_warp(jc, joint_ctrl(a, lane, cfg.normalized), q, qd, root, task[0], task[TD - 1] != 0.f, r, fwd_vel);
        done = walker::is_done(root[1], root[2]);
        return r;
    }
    static __device__ __forceinline__ float step_serial(float (&st)[SD], const float* a, const float* task, const EnvCfg& cfg,
                                                        float*, int, bool& done) {
        float u[DA], r, fwd_vel;
#pragma unroll
        for (int k = 0; k < DA; ++k) u[k] = ctrl_action(a[k], cfg.normalized);
        walker::step_serial(st, u, task[0], task[TD - 1] != 0.f, r, fwd_vel);
        done = walker::is_done(st[1], st[2]);
        return r;
    }
};

// ------------------------------------------------------------------ swimmer surrogate
// MuJoCo-free SwimmerRandVel: obs / reward / reset follow ref envs/mujoco_envs/swimmer_rand_vel.py:30-50 (reward_fwd =
// |fwd_vel - goal| with the reference's sign), the dynamics are defined in DESIGN.md §3.4 (CPU: oracle/
// locomotion_surrogates.py).  State = qpos (x, y, rot, q0, q1) ++ qvel.  Two joints: the whole step is cheap enough to run
// replicated in every lane of the env's warp (no reductions), and the single-step kernel runs the same function.
namespace swimmer {
constexpr float HS = 0.01f, DT = 0.04f;
constexpr int FRAME_SKIP = 4;
constexpr float G0 = 10.0f, G1 = 10.0f, K0 = 4.0f, K1 = 4.0f, D0 = 1.0f, D1 = 1.0f, P0 = 0.5f, P1 = -0.5f;
constexpr float CS = 0.02f, DR = 2.0f, BV = 1.0f;

__device__ __forceinline__ void step(float (&st)[10], float u0, float u1, float goal, float& rew, float& r_fwd, float& r_ctrl) {
    const float x0 = st[0];
    const float twist = P0 * u0 + P1 * u1;
#pragma unroll
    for (int s = 0; s < FRAME_SKIP; ++s) {
        float qd0 = st[8] + HS * (G0 * u0 - K0 * st[3] - D0 * st[8]);
        const float q0 = st[3] + HS * qd0;
        float qd1 = st[9] + HS * (G1 * u1 - K1 * st[4] - D1 * st[9]);
        const float q1 = st[4] + HS * qd1;
        st[3] = q0, st[8] = qd0, st[4] = q1, st[9] = qd1;
        const float thrust = CS * (q0 * qd1 - q1 * qd0);
        const float rot = st[2];
        const float rd = st[7] + HS * (twist - DR * st[7]);
        float sn, cs;
        __sincosf(rot, &sn, &cs);
        const float xd = st[5] + HS * (thrust * cs - BV * st[5]);
        const float yd = st[6] + HS * (thrust * sn - BV * st[6]);
        st[5] = xd, st[6] = yd, st[7] = rd;
        st[0] = st[0] + HS * xd;
        st[1] = st[1] + HS * yd;
        st[2] = rot + HS * rd;
    }
    const float fwd_vel = (st[0] - x0) / DT;
    r_fwd = fabsf(fwd_vel - goal);
    r_ctrl = -1e-4f * (u0 * u0 + u1 * u1);
    rew = r_fwd + r_ctrl;
}
}  // namespace swimmer

// task = goal velocity; info = reward_fwd, reward_ctrl
struct Swimmer : Replicated<Swimmer, 10> {
    static constexpr int KIND = PROMP_ENV_SWIMMER, DO = 8, DA = 2, SD = 10, TD = 1, NINFO = 2, NACC = 4;
    static constexpr bool ENDS_EARLY = false;

    // reset_model (swimmer_rand_vel.py:41-46): qpos = U(-.1,.1)^5, qvel = U(-.1,.1)^5 from counters (step << 4) + 0..2
    __device__ __forceinline__ void reset(const EnvRng& rng, uint32_t step, uint32_t tag, int, const float*) {
#pragma unroll
        for (int blk = 0; blk < 3; ++blk) {
            uint32_t r[4];
            rng.gen((step << 4) + (uint32_t)blk, tag, r);
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (blk * 4 + i < SD) s[blk * 4 + i] = -0.1f + 0.2f * u01(r[i]);
        }
    }
    static __device__ __forceinline__ float step_serial(float (&st)[SD], const float* a, const float* task, const EnvCfg& cfg,
                                                        float* info, int info_stride, bool&) {
        const float u0 = ctrl_action(a[0], cfg.normalized), u1 = ctrl_action(a[1], cfg.normalized);
        float r, r_fwd, r_ctrl;
        swimmer::step(st, u0, u1, task[0], r, r_fwd, r_ctrl);
        if (info) {
            info[0] = r_fwd;
            info[info_stride] = r_ctrl;
        }
        return r;
    }
    // obs = qpos[2:] ++ qvel (swimmer_rand_vel.py:37-40)
    static __device__ __forceinline__ void observe_serial(const float* st, float* obs) {
#pragma unroll
        for (int k = 0; k < DO; ++k) obs[k] = st[2 + k];
    }
};

}  // namespace promp
