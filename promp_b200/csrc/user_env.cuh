// Users' own environments in the fused rollout and single-step kernels (compiled at run time by promp_b200/_jit.py).
//
// The serial concept a user writes: one struct, one thread's view of one env,
//   static constexpr int DO, DA, SD, TD, NINFO (0..3);  static constexpr bool ENDS_EARLY;
//   static __device__ void  reset(float (&s)[SD], const float* task, promp::EnvDraw& rng);
//   static __device__ float step(float (&s)[SD], const float* a, const float* task, float* info, int info_stride, bool& done);
//   static __device__ void  observe(const float (&s)[SD], float* obs);
// `a` is the action the env receives: the NormalizedEnv map and clip to the action-space bounds are already applied when
// the env is wrapped by normalize(); the raw policy action otherwise.  step writes env-info channel c (c < NINFO) to
// info[c * info_stride] and sets `done` to end the path early (read only when ENDS_EARLY).
//
// SerialEnv<U, Bounds> wraps it in the warp concept of envs.cuh (Replicated: every lane of the env's warp holds and
// advances the same state, lane 0 writes).  A type that already has the warp concept (step_serial; the built-in envs,
// or a lane-parallel user env) is used as it is: UserEnvOf picks.
#pragma once
#include "rollout_kernel.cuh"

namespace promp {

// Reset draws of one env slot: uniform(i) in (0, 1] and normal(i) ~ N(0, 1), i = 0 .. 63, from the slot's Philox stream
// keyed like PointState::reset (env, step, stream) with counter (step << 4) + i / 4; the normals take their own tag.  A
// draw is a pure function of (seed, phase, env, step, i): asking twice for one i gives one value.
struct EnvDraw {
    const EnvRng& rng;
    uint32_t step, tag;
    __device__ __forceinline__ float uniform(int i) const {
        uint32_t r[4];
        rng.gen((step << 4) + (uint32_t)(i >> 2), tag, r);
        return u01(r[i & 3]);
    }
    __device__ __forceinline__ float normal(int i) const {
        uint32_t r[4];
        rng.gen((step << 4) + (uint32_t)(i >> 2), tag | 0x04000000u, r);
        float z[4];
        box_muller(r[0], r[1], z[0], z[1]);
        box_muller(r[2], r[3], z[2], z[3]);
        return z[i & 3];
    }
};

// Bounds: lb(d) / ub(d), the action-space bounds of the env (generated as constants).
template <class U, class Bounds>
struct SerialEnv : Replicated<SerialEnv<U, Bounds>, U::SD> {
    static constexpr int DO = U::DO, DA = U::DA, SD = U::SD, TD = U::TD, NINFO = U::NINFO;
    static constexpr int NACC = DO <= 8 ? 4 : 2;   // layer-1 accumulators of the rollout (the built-ins' choice by obs size)
    static constexpr bool ENDS_EARLY = U::ENDS_EARLY, GENERIC_INFO = true;
    static_assert(DO >= 1 && DO <= 19, "user env: DO must be 1..19 (the rollout policy's observation range)");
    static_assert(DA >= 1 && DA <= 8, "user env: DA must be 1..8 (the rollout policy's action range)");
    static_assert(SD >= 1 && TD >= 1, "user env: SD and TD must be >= 1");
    static_assert(NINFO >= 0 && NINFO <= 3, "user env: NINFO must be 0..3");

    __device__ __forceinline__ void reset(const EnvRng& rng, uint32_t step, uint32_t tag, int, const float* task) {
        EnvDraw d{rng, step, tag};
        U::reset(this->s, task, d);
    }
    static __device__ __forceinline__ float step_serial(float (&s)[SD], const float* a, const float* task, const EnvCfg& cfg,
                                                        float* info, int info_stride, bool& done) {
        float ea[DA];
#pragma unroll
        for (int d = 0; d < DA; ++d) ea[d] = cfg.normalized ? normalized_action(a[d], Bounds::lb(d), Bounds::ub(d)) : a[d];
        float inf[NINFO > 0 ? NINFO : 1];   // the env always has somewhere to write; only lane 0 / a real buffer keeps it
        bool dn = false;
        const float r = U::step(s, ea, task, inf, 1, dn);
        if (ENDS_EARLY) done = dn;
        if (info)
#pragma unroll
            for (int c = 0; c < NINFO; ++c) info[c * info_stride] = inf[c];
        return r;
    }
    static __device__ __forceinline__ void observe_serial(const float* st, float* obs) {
        U::observe(*reinterpret_cast<const float(*)[SD]>(st), obs);
    }
};

template <class U, class Bounds, class = void>
struct UserEnvOf {
    using type = SerialEnv<U, Bounds>;
};
template <class U, class Bounds>
struct UserEnvOf<U, Bounds, decltype(void(&U::step_serial))> {
    using type = U;
};

}  // namespace promp
