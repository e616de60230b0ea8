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
#pragma once
#include "common.cuh"

namespace promp {

template <int KIND> struct EnvTraits;
template <> struct EnvTraits<PROMP_ENV_POINT_CORNER> {
    static constexpr int DO = 2, DA = 2, SD = 2, TD = 2, NINFO = 0;
};
template <> struct EnvTraits<PROMP_ENV_POINT> {
    static constexpr int DO = 2, DA = 2, SD = 2, TD = 1, NINFO = 0;
};
template <> struct EnvTraits<PROMP_ENV_CHEETAH_DIR> {
    static constexpr int DO = 17, DA = 6, SD = 18, TD = 1, NINFO = 2;
};
template <> struct EnvTraits<PROMP_ENV_POINT_WALLS> {
    static constexpr int DO = 2, DA = 2, SD = 2, TD = 6, NINFO = 0;       // task = goal, gap_1, gap_2
};
template <> struct EnvTraits<PROMP_ENV_POINT_MOMENTUM> {
    static constexpr int DO = 4, DA = 2, SD = 4, TD = 2, NINFO = 0;       // state = obs = (pos, vel)
};
template <> struct EnvTraits<PROMP_ENV_WALKER> {
    static constexpr int DO = 17, DA = 6, SD = 18, TD = 2, NINFO = 0;     // task = (direction | goal velocity, mode)
};
template <> struct EnvTraits<PROMP_ENV_SWIMMER> {
    static constexpr int DO = 8, DA = 2, SD = 10, TD = 1, NINFO = 2;      // info = reward_fwd, reward_ctrl
};

// NormalizedEnv.step action map, same evaluation order as the reference expression
//   lb + (a + scale) * (ub - lb) / (2*scale), then clip to [lb, ub]       (normalization_scale = 10)
__device__ __forceinline__ float normalized_action(float a, float lb, float ub) {
    float s = lb + ((a + 10.0f) * (ub - lb)) / 20.0f;
    return fminf(fmaxf(s, lb), ub);
}
// wrapped (normalize(env), every reference run script) or raw env (the reference's tests): the raw env receives the
// policy action unchanged and applies only its own clip
__device__ __forceinline__ float env_action(float a, float lb, float ub, bool normalized) {
    return normalized ? normalized_action(a, lb, ub) : a;
}

// ------------------------------------------------------------------ point corner
struct PointCornerCfg {
    int reward_type;
    float radius;
    bool normalized;
};

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

// s (in/out): state; (ax, ay): policy-space action.  Returns reward.
__device__ __forceinline__ float point_corner_step(float& sx, float& sy, float ax, float ay, float gx, float gy,
                                                   const PointCornerCfg& cfg) {
    const float lim = 0.2f;
    float ex = env_action(ax, -lim, lim, cfg.normalized), ey = env_action(ay, -lim, lim, cfg.normalized);
    // env-side clip (point_env_2d_corner.py:37); the identity after the wrapper's clip
    ex = fminf(fmaxf(ex, -lim), lim);
    ey = fminf(fmaxf(ey, -lim), lim);
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

// ------------------------------------------------------------------ point (origin goal, early done)
__device__ __forceinline__ float point_step(float& sx, float& sy, float ax, float ay, bool& done, bool normalized) {
    const float lim = 0.1f;
    float ex = env_action(ax, -lim, lim, normalized), ey = env_action(ay, -lim, lim, normalized);
    ex = fminf(fmaxf(ex, -lim), lim);
    ey = fminf(fmaxf(ey, -lim), lim);
    sx += ex;
    sy += ey;
    done = (fabsf(sx) < 0.01f) && (fabsf(sy) < 0.01f);
    return -sqrt_fast(sx * sx + sy * sy);
}

// ------------------------------------------------------------------ point walls (ref point_env_2d_walls.py:22-51)
// s' = s + clip(a, +-0.2); the reward is taken at s' BEFORE the wall logic (:37-39); crossing the unit circle outside
// gap_1 (distance > 1 from the gap centre) projects s' back to just inside radius 1, crossing the radius-2 circle
// outside gap_2 to just inside radius 2 (:40-49).  reward_type dense / dense_squared (the reference's 'sparse' branch
// returns None outside the radius and cannot be sampled).
__device__ __forceinline__ float point_walls_step(float& sx, float& sy, float ax, float ay, const float* task, int reward_type,
                                                  bool normalized) {
    const float lim = 0.2f;
    float ex = env_action(ax, -lim, lim, normalized), ey = env_action(ay, -lim, lim, normalized);
    ex = fminf(fmaxf(ex, -lim), lim);
    ey = fminf(fmaxf(ey, -lim), lim);
    const float px = sx, py = sy;
    float nx = px + ex, ny = py + ey;
    const float g = dist2d(nx, ny, task[0], task[1]);
    const float r = (reward_type == PROMP_REWARD_DENSE_SQUARED) ? -(g * g) : -g;
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

// ------------------------------------------------------------------ point momentum (ref point_env_2d_momentum.py:22-42, 58-68)
// v' = v + clip(a, +-0.1); s' = s + v'; obs = (s', v'); reward at s': sparse (default) = max(radius - |s' - goal|, 0)
__device__ __forceinline__ float point_momentum_step(float& sx, float& sy, float& vx, float& vy, float ax, float ay, float gx,
                                                     float gy, const PointCornerCfg& cfg) {
    const float lim = 0.1f;
    float ex = env_action(ax, -lim, lim, cfg.normalized), ey = env_action(ay, -lim, lim, cfg.normalized);
    ex = fminf(fmaxf(ex, -lim), lim);
    ey = fminf(fmaxf(ey, -lim), lim);
    vx += ex, vy += ey;
    sx += vx, sy += vy;
    const float g = dist2d(sx, sy, gx, gy);
    if (cfg.reward_type == PROMP_REWARD_DENSE) return -g;
    if (cfg.reward_type == PROMP_REWARD_DENSE_SQUARED) return -(g * g);
    return fmaxf(cfg.radius - g, 0.f);
}

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
// obs clips qvel to [-10, 10] (walker2d_rand_*.py:42-45)
__device__ __forceinline__ float clip_vel(float v) { return fminf(fmaxf(v, -10.0f), 10.0f); }

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

}  // namespace promp
