// Definitions shared by both families of Gaussian-MLP policy kernels (the CUDA-core kernels of policy.cu and the
// tensor-core kernels of policy_tc.cuh): the kernel arguments, the work schedule and its task-segment flush, the
// Gaussian head, and the SIMT tile machinery of the CUDA-core kernels.
//
// A CUDA-core CTA of 256 threads processes tiles of TB = 64 samples of ONE task.  All weight matrices of the
// task live in shared memory; activations are [TB][LD] row-major tiles (LD = HID + 4 keeps rows
// 16-byte aligned and spreads banks).  The 64 x HID x HID products are register-tiled SIMT fp32
// GEMMs (RM x 4 outputs per thread, float4 shared-memory loads): float32 FMA keeps the 1e-4 parity
// bar against the reference's float32 TF graph; tensor-core tf32/bf16 would not.
#pragma once
#include <stddef.h>
#include "common.cuh"

namespace promp {

constexpr int PT_THREADS = 256;
constexpr int TB = 64;   // samples per tile

template <int DO>
struct DOPad {
    static constexpr int V = (DO + 3) / 4 * 4;
};

constexpr int PSTAT = 4;   // per-partial trailing stats: sum obj, sum kl, sum ratio, unused

struct PolicyArgs {
    int M, N;
    const float* params;
    int64_t param_stride;
    const float *obs, *act, *adv, *old_mean, *old_ls;
    int ls_per_sample;
    int obj_kind;
    float obj_scale, clip_eps, kl_coeff;
    int clip_log_std;
    float min_log_std;
    int obs_dim;         // logical observation / action sizes; read only by the padded instantiations (IsBucket below).  Both
                         // sit in what was alignment padding.
    // grad kernel
    float* grad;
    float* out_params;
    float sgd_lr;
    int act_dim;
    // hvp kernel
    const float* vec;
    float* out;
    float inner_lr;
    int adv_per_task;    // PROMP_OBJ_EXPLORE: adv is a per-task [M] vector (the E-MAML coefficient), obj_kind is LOGLIK.  Read
                         // only by the *_explore instantiations; it sits in what was alignment padding, like obs_dim.
    float* stats;
    float* partial;      // [grid][kmax][P + PSTAT] per-(CTA, task-segment) partial sums
    int* counters;       // [M], zero on entry, left zero on exit
    int q;               // tiles per CTA
    int kmax;            // max task segments per CTA
    const int32_t* n_valid;   // [M] valid samples per task (rows >= n_valid[m] are padding) or nullptr = N everywhere
    // Re-use of an identical earlier launch (grad kernels only): the inner pass of the first Adam epoch repeats MAMLAlgo._adapt
    // (same theta, same phase-0 data, same outputs) unless the reported-log_std clip of the step-0 graph is active.
    //   producer side: unclipped_out = 1 iff every log_std component >= min_log_std, theta_copy_out = the parameters it used
    //   consumer side: the whole grid returns at once if *skip_flag != 0 and params == skip_theta bit for bit (its outputs
    //                  alias the producer's, which are then already correct)
    const int* skip_flag;
    const float* skip_theta;
    int* unclipped_out;
    float* theta_copy_out;
    // optional device-resident multiplier of kl_coeff (ProMP's adaptive inner-KL coefficient lives on the device so that an
    // iteration has no host decision: promp_adapt_kl_coeff updates it between launches)
    const float* kl_coeff_ptr;
    // optional per-parameter inner step sizes alpha [P] (Meta-SGD, trainable_inner_step_size): the gradient kernels' SGD step is
    // params - alpha * grad in place of params - sgd_lr * grad, and the HVP kernels stage the direction as alpha * vec (the
    // caller passes inner_lr = 1).  nullptr = the scalar forms.
    const float* step_size;
};
static_assert(sizeof(PolicyArgs) == 232 && offsetof(PolicyArgs, grad) == 96 && offsetof(PolicyArgs, vec) == 120 &&
                  offsetof(PolicyArgs, stats) == 144,
              "PolicyArgs layout");

// Where a kernel reads a sample's advantage: ADV_SAMPLE = adv[n] (every instantiation that existed before the E-MAML
// objective, unchanged), ADV_TASK = adv[m] (the stand-alone PROMP_OBJ_EXPLORE kernels), ADV_EITHER = per launch argument
// (the dataflow chain with an exploration stage, whose other stages read adv[n]).
constexpr int ADV_SAMPLE = 0, ADV_TASK = 1, ADV_EITHER = 2;
__device__ __forceinline__ float kl_coeff_eff(const PolicyArgs& A) {
    return A.kl_coeff_ptr ? A.kl_coeff * __ldcg(A.kl_coeff_ptr) : A.kl_coeff;
}

// Padded instantiations ("buckets"): compiled at the caps (DO, DA) of the zero-padded parameter layout of
// promp_policy_layout, they take the logical observation / action sizes from PolicyArgs at run time.  Observations are
// read with row stride obs_dim and zero-filled above it; action-side data (act, old_mean, old_log_std, mean) with row
// stride act_dim, entries d >= act_dim never touched; the Gaussian head masks d >= act_dim out of every sum and gradient.
// Pad rows of W0, pad columns of W2 and pad entries of b2 / log_std therefore get gradients and HVPs of exactly zero.
// Whether a (DO, DA) instantiation is a bucket is known at compile time, so the exact instantiations compile to the code
// they had.  The caps: obs_dim 1..8 -> 8, 9..19 -> 20; act_dim 1..2 -> 2, 3..8 -> 8 (even: P % 4 == 0).
template <int DO, int DA>
struct IsBucket {
    static constexpr bool value = (DO == 8 || DO == 20) && (DA == 2 || DA == 8);
};
template <int DO, int DA>
__device__ __forceinline__ int obs_dim_of(const PolicyArgs& A) {
    if constexpr (IsBucket<DO, DA>::value) return A.obs_dim;
    return DO;
}
template <int DO, int DA>
__device__ __forceinline__ int act_dim_of(const PolicyArgs& A) {
    if constexpr (IsBucket<DO, DA>::value) return A.act_dim;
    return DA;
}

// Consumer half of the launch re-use protocol above: true in every thread of the CTA if *skip_flag != 0 and the P
// parameters equal skip_theta bit for bit (the CTA must then exit).
template <int P>
__device__ __forceinline__ bool reuse_hit(const int* skip_flag, const float* params, const float* skip_theta) {
    if (!skip_flag) return false;
    bool same = *reinterpret_cast<const volatile int*>(skip_flag) != 0;
    for (int i = threadIdx.x; i < P && same; i += blockDim.x)
        same = __float_as_uint(__ldcg(params + i)) == __float_as_uint(__ldcg(skip_theta + i));
    return __syncthreads_and(same ? 1 : 0) != 0;
}
// Producer half: CTA 0 records whether the log_std clip is inactive and the parameters it used.
template <int P, int LS, int DA>
__device__ __forceinline__ void reuse_produce(const PolicyArgs& A) {
    if (A.unclipped_out && blockIdx.x == 0) {
        if (threadIdx.x == 0) {
            int ok = 1;
            for (int d = 0; d < DA; ++d)
                if (!(__ldcg(A.params + LS + d) >= A.min_log_std)) ok = 0;
            *A.unclipped_out = ok;
        }
        for (int i = threadIdx.x; i < P; i += blockDim.x) A.theta_copy_out[i] = __ldcg(A.params + i);
    }
}

// -------------------------------------------------------------------------------------------------------------
// Work decomposition seen by the tile loops.  Every tile loop is written against this interface:
//   [g_lo, g_hi)            the caller's range in the task-major tile list (ntiles tiles per task)
//   my_slot(m)              partial slot this range writes for task m
//   n_contrib / contrib_slot the slots of task m, in the fixed order in which its last arriver sums them
//   wait_task / publish_task dependency on / completion of task m (dataflow kernel only)
//   ldp                     parameter loads: read-only path (.nc) when nothing in this launch writes them, L2 (.cg) otherwise
// UniformSched = the stand-alone launches (CTA c owns tiles [c q, (c+1) q) of tb samples, kmax slots per CTA); ItemSched
// (policy_tc.cuh) = one work item of policy_chain_tc_kernel.
struct UniformSched {
    int ntiles, g_lo, g_hi, q, kmax;
    __device__ __forceinline__ UniformSched(int M, int N, int q_, int kmax_, int tb) {
        ntiles = (N + tb - 1) / tb;
        q = q_;
        kmax = kmax_;
        g_lo = blockIdx.x * q;
        g_hi = min(g_lo + q, M * ntiles);
    }
    __device__ __forceinline__ int first_task(int c) const { return (c * q) / ntiles; }
    __device__ __forceinline__ int cta_lo(int m) const { return (m * ntiles) / q; }
    __device__ __forceinline__ int cta_hi(int m) const { return ((m + 1) * ntiles - 1) / q; }
    __device__ __forceinline__ int my_slot(int m) const { return blockIdx.x * kmax + (m - first_task(blockIdx.x)); }
    __device__ __forceinline__ int n_contrib(int m) const { return cta_hi(m) - cta_lo(m) + 1; }
    __device__ __forceinline__ int contrib_slot(int m, int i) const {
        const int c = cta_lo(m) + i;
        return c * kmax + (m - first_task(c));
    }
    __device__ __forceinline__ void wait_task(int) const {}
    __device__ __forceinline__ void publish_task(int) const {}
    __device__ __forceinline__ void clk(int) const {}
    static __device__ __forceinline__ float ldp(const float* p) { return __ldg(p); }
    static __device__ __forceinline__ float4 ldp4(const float4* p) { return __ldg(p); }
};

// Sum one float4 column of a task's partial slots in contributor order, eight independent L2 loads in flight.
template <class Sched>
__device__ __forceinline__ float4 reduce_slots4(const float* partial, const Sched& sc, int pstride, int m, int n, int p) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i0 = 0; i0 < n; i0 += 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)
            v[u] = (i0 + u < n) ? __ldcg(reinterpret_cast<const float4*>(partial + (int64_t)sc.contrib_slot(m, i0 + u) * pstride + p))
                                : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < 8; ++u) s.x += v[u].x, s.y += v[u].y, s.z += v[u].z, s.w += v[u].w;
    }
    return s;
}

// The same sums for ALL of a thread's columns p = 4 tid + i * 4 * threads (i < NP) at once: NP x 4 independent 16-byte L2 loads
// in flight instead of one column at a time - the last arriver's reduction sits on the tail of the kernel and is pure L2
// latency.  Slots are added in contributor order, so the result is bit-identical to reduce_slots4.
template <int NP, class Sched>
__device__ __forceinline__ void reduce_slots4_wide(const float* partial, const Sched& sc, int pstride, int m, int n, int p0, int pstep,
                                                   int pend, float4 (&acc)[NP]) {
#pragma unroll
    for (int i = 0; i < NP; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c0 = 0; c0 < n; c0 += 4) {
        float4 v[NP][4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int64_t base = (c0 + u < n) ? (int64_t)sc.contrib_slot(m, c0 + u) * pstride : -1;
#pragma unroll
            for (int i = 0; i < NP; ++i) {
                const int p = p0 + i * pstep;
                v[i][u] = (base >= 0 && p < pend) ? __ldcg(reinterpret_cast<const float4*>(partial + base + p)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int i = 0; i < NP; ++i) acc[i].x += v[i][u].x, acc[i].y += v[i][u].y, acc[i].z += v[i][u].z, acc[i].w += v[i][u].w;
    }
}

template <int HID>
struct TileCfg {
    static constexpr int LD = HID + 4;
    static constexpr int TX = HID / 4;            // threads across the HID columns (4 columns each)
    static constexpr int TY = PT_THREADS / TX;    // thread rows
    static constexpr int RM = TB / TY;            // sample rows per thread          (64: 4, 32: 2)
    static constexpr int RK = HID / TY;           // weight-gradient rows per thread (64: 4, 32: 1)
    static_assert(HID == 64 || HID == 32, "hidden size must be 32 or 64");
};

// acc[i][c] += sum_k A[row0+i][k] * W[k][col0+c],  A: [TB][LDA] row-major, W: [K][LDW] row-major.
template <int K, int LDA, int LDW, int RM>
__device__ __forceinline__ void gemm_tile(const float* __restrict__ A, const float* __restrict__ W, int row0, int col0,
                                          float (&acc)[RM][4]) {
#pragma unroll 4
    for (int k = 0; k < K; k += 4) {
        float4 a[RM], w[4];
#pragma unroll
        for (int i = 0; i < RM; ++i) a[i] = *reinterpret_cast<const float4*>(A + (row0 + i) * LDA + k);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) w[kk] = *reinterpret_cast<const float4*>(W + (k + kk) * LDW + col0);
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            acc[i][0] = fmaf(a[i].x, w[0].x, acc[i][0]); acc[i][1] = fmaf(a[i].x, w[0].y, acc[i][1]);
            acc[i][2] = fmaf(a[i].x, w[0].z, acc[i][2]); acc[i][3] = fmaf(a[i].x, w[0].w, acc[i][3]);
            acc[i][0] = fmaf(a[i].y, w[1].x, acc[i][0]); acc[i][1] = fmaf(a[i].y, w[1].y, acc[i][1]);
            acc[i][2] = fmaf(a[i].y, w[1].z, acc[i][2]); acc[i][3] = fmaf(a[i].y, w[1].w, acc[i][3]);
            acc[i][0] = fmaf(a[i].z, w[2].x, acc[i][0]); acc[i][1] = fmaf(a[i].z, w[2].y, acc[i][1]);
            acc[i][2] = fmaf(a[i].z, w[2].z, acc[i][2]); acc[i][3] = fmaf(a[i].z, w[2].w, acc[i][3]);
            acc[i][0] = fmaf(a[i].w, w[3].x, acc[i][0]); acc[i][1] = fmaf(a[i].w, w[3].y, acc[i][1]);
            acc[i][2] = fmaf(a[i].w, w[3].z, acc[i][2]); acc[i][3] = fmaf(a[i].w, w[3].w, acc[i][3]);
        }
    }
}

// Small-K variant (layer 0: K = obs_dim, any value): scalar loads.
template <int K, int LDA, int LDW, int RM>
__device__ __forceinline__ void gemm_tile_smallk(const float* __restrict__ A, const float* __restrict__ W, int row0,
                                                 int col0, float (&acc)[RM][4]) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float4 w = *reinterpret_cast<const float4*>(W + k * LDW + col0);
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            const float a = A[(row0 + i) * LDA + k];
            acc[i][0] = fmaf(a, w.x, acc[i][0]); acc[i][1] = fmaf(a, w.y, acc[i][1]);
            acc[i][2] = fmaf(a, w.z, acc[i][2]); acc[i][3] = fmaf(a, w.w, acc[i][3]);
        }
    }
}

// Weight-gradient accumulation: g[r][c] += sum_b A[b][k0+r] * D[b][col0+c]  (A, D: [TB][LD] tiles).
template <int LD, int RK>
__device__ __forceinline__ void wgrad_tile(const float* __restrict__ A, const float* __restrict__ D, int k0, int col0,
                                           int nb, float (&g)[RK][4]) {
#pragma unroll 4
    for (int b = 0; b < nb; ++b) {
        const float4 d = *reinterpret_cast<const float4*>(D + b * LD + col0);
        float a[RK];
        if constexpr (RK == 4) {
            const float4 av = *reinterpret_cast<const float4*>(A + b * LD + k0);
            a[0] = av.x; a[1] = av.y; a[2] = av.z; a[3] = av.w;
        } else {
#pragma unroll
            for (int r = 0; r < RK; ++r) a[r] = A[b * LD + k0 + r];
        }
#pragma unroll
        for (int r = 0; r < RK; ++r) {
            g[r][0] = fmaf(a[r], d.x, g[r][0]); g[r][1] = fmaf(a[r], d.y, g[r][1]);
            g[r][2] = fmaf(a[r], d.z, g[r][2]); g[r][3] = fmaf(a[r], d.w, g[r][3]);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Diagonal-Gaussian head for one sample (ref: policies/distributions/diagonal_gaussian.py:16-109).
// Everything the objective kinds need, evaluated in float32 like the TF graph.
// Everything that depends only on the policy's log_std (a per-task constant) is computed ONCE per task
// (head_in_finish): the per-sample path multiplies by reciprocals instead of dividing - the head is a serial dependent
// chain executed by one thread per sample row, and its ~5 IEEE divisions + 1 expf per action dimension were most of it.
template <int DA>
struct HeadIn {
    float ls[DA];      // new log_std (after the optional clip)
    float sig[DA];     // exp(ls)
    float ls_mask[DA]; // 0 where the clip is active (gradient does not reach the variable), else 1
    float inv_sig[DA]; // 1 / sig
    float s2[DA];      // sig^2
    float inv_den[DA]; // 1 / (2 sig^2 + 1e-8)            (kl_sym denominator)
    float c1[DA];      // 1 - 2 sig^2 / den                d KL / d log_std = c1 - c2 * num
    float c2[DA];      // 4 sig^2 / den^2
    float sum_ls;      // sum_d ls
};
// da: the logical action size; dimensions d >= da are the zero padding of a padded instantiation (DA = its cap) and are
// left out of every sum, so that they contribute nothing and receive exactly zero gradient.
template <int DA>
__device__ __forceinline__ void head_in_finish(HeadIn<DA>& h, int da = DA) {
    h.sum_ls = 0.f;
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        h.inv_sig[d] = 1.f / h.sig[d];
        h.s2[d] = h.sig[d] * h.sig[d];
        const float den = 2.f * h.s2[d] + 1e-8f;
        h.inv_den[d] = 1.f / den;
        h.c1[d] = 1.f - 2.f * h.s2[d] / den;
        h.c2[d] = 4.f * h.s2[d] / (den * den);
        if (d < da) h.sum_ls += h.ls[d];
    }
}
// The old (sampling) distribution's log_std: per task when the phase stores one row per task, else per sample.
template <int DA>
struct HeadOld {
    float ls[DA];
    float so2[DA];     // exp(ls)^2
    float inv_so[DA];  // 1 / exp(ls)
    float sum_ls;
};
template <int DA>
__device__ __forceinline__ void head_old_from(const float* ls_old, HeadOld<DA>& ho, int da = DA) {
    ho.sum_ls = 0.f;
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        const float so = expf(ls_old[d]);
        ho.ls[d] = ls_old[d];
        ho.so2[d] = so * so;
        ho.inv_so[d] = 1.f / so;
        if (d < da) ho.sum_ls += ls_old[d];
    }
}

template <int DA>
struct HeadOut {
    float obj;        // per-sample surrogate term (unscaled, before the 1/N mean)
    float kl;         // KL(old || new)
    float ratio;
    float w;          // d obj / d logp_new
    float zeta[DA];   // (a - mu)/sigma
    float dkl_dmu[DA];
    float dkl_dls[DA];
};

constexpr float LOG_2PI = 1.8378770664093453f;

template <int DA>
__device__ __forceinline__ void gaussian_head(const HeadIn<DA>& hin, const HeadOld<DA>& ho, const float* mu, const float* a,
                                              const float* mu_old, float adv, int obj_kind, float clip_eps, HeadOut<DA>& o,
                                              int da = DA) {
    float sum_z2 = 0.f, sum_zo2 = 0.f, kl = 0.f;
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        if (d >= da) {          // padding of a padded instantiation: no term, no gradient
            o.zeta[d] = o.dkl_dmu[d] = o.dkl_dls[d] = 0.f;
            continue;
        }
        const float z = (a[d] - mu[d]) * hin.inv_sig[d];
        o.zeta[d] = z;
        sum_z2 += z * z;
        const float zo = (a[d] - mu_old[d]) * ho.inv_so[d];
        sum_zo2 += zo * zo;
        // kl_sym (:16-44): (dmu^2 + so^2 - sn^2) / (2 sn^2 + 1e-8) + ls_new - ls_old
        const float dm = mu_old[d] - mu[d];
        const float num = dm * dm + ho.so2[d] - hin.s2[d];
        kl += num * hin.inv_den[d] + hin.ls[d] - ho.ls[d];
        o.dkl_dmu[d] = -2.f * dm * hin.inv_den[d];
        o.dkl_dls[d] = hin.c1[d] - hin.c2[d] * num;
    }
    const float logp_new = -hin.sum_ls - 0.5f * sum_z2 - 0.5f * da * LOG_2PI;   // log_likelihood_sym (:89-109)
    const float logp_old = -ho.sum_ls - 0.5f * sum_zo2 - 0.5f * da * LOG_2PI;
    const float ratio = expf(logp_new - logp_old);                           // likelihood_ratio_sym (:71-87)
    o.ratio = ratio;
    o.kl = kl;
    if (obj_kind == PROMP_OBJ_RATIO) {
        o.obj = -ratio * adv;
        o.w = -adv * ratio;
    } else if (obj_kind == PROMP_OBJ_LOGLIK) {
        o.obj = -logp_new * adv;
        o.w = -adv;
    } else if (obj_kind == PROMP_OBJ_CLIP) {
        // -min(r*A, clip(r,1-e,1+e)*A); tf.minimum routes the gradient to r*A when r*A <= clipped,
        // and clip_by_value has zero gradient outside the range (pro_mp.py:135-141)
        const float x = ratio * adv;
        const float y = fminf(fmaxf(ratio, 1.f - clip_eps), 1.f + clip_eps) * adv;
        o.obj = -fminf(x, y);
        o.w = (x <= y) ? -adv * ratio : 0.f;
    } else {
        o.obj = 0.f;
        o.w = 0.f;
    }
}

// Per-task head constants from the policy's raw log_std (ls_raw[0 .. DA)): the optional clip and its gradient mask, sig,
// and head_in_finish.  With `hold` and a phase that stores one old log_std row per task, also task m's HeadOld.
template <int DA>
__device__ __forceinline__ void head_setup(const PolicyArgs& A, const float* ls_raw, int m, int dA, HeadIn<DA>& hin,
                                           HeadOld<DA>* hold) {
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        const float raw = ls_raw[d];
        const bool clipped = A.clip_log_std && (raw < A.min_log_std);      // tf.maximum: gradient goes to x when x >= y
        hin.ls[d] = clipped ? A.min_log_std : raw;
        hin.ls_mask[d] = (clipped || d >= dA) ? 0.f : 1.f;      // padding (d >= dA) gets no log_std gradient either
        hin.sig[d] = expf(hin.ls[d]);
    }
    head_in_finish<DA>(hin, dA);
    if (hold && !A.ls_per_sample) {
        float lso[DA];
#pragma unroll
        for (int d = 0; d < DA; ++d) lso[d] = d < dA ? __ldg(A.old_ls + (int64_t)m * dA + d) : 0.f;
        head_old_from<DA>(lso, *hold, dA);
    }
}

// act / old_mean of sample n (task m) and, if `with_ls`, its old log_std (the sample's, or task m's row when the phase stores
// one row per task), zero above the logical action size dA; returns the sample's advantage (see ADV_SAMPLE above).
template <int DA, int ADV = ADV_SAMPLE>
__device__ __forceinline__ float load_head_sample(const PolicyArgs& A, int64_t n, int m, int dA, bool with_ls, float (&a)[DA],
                                                  float (&mo)[DA], float (&lso)[DA]) {
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        a[d] = d < dA ? __ldg(A.act + n * dA + d) : 0.f;
        mo[d] = d < dA ? __ldg(A.old_mean + n * dA + d) : 0.f;
        // two loads and a select rather than one load from a selected address: the latter keeps the CUDA-core HVP kernels
        // from sharing z^2 between gaussian_head and hvp_signal, and ptxas then contracts both into FMAs (different bits)
        if (with_ls)
            lso[d] = d >= dA ? 0.f : A.ls_per_sample ? __ldg(A.old_ls + n * dA + d) : __ldg(A.old_ls + (int64_t)m * dA + d);
    }
    if constexpr (ADV == ADV_TASK) return __ldg(A.adv + m);
    if constexpr (ADV == ADV_EITHER) return A.adv_per_task ? __ldg(A.adv + m) : __ldg(A.adv + n);
    return __ldg(A.adv + n);
}

// Backprop signal of the gradient kernels at the head: d loss / d mu (dmu) and d loss / d log_std (dls) of one sample.
template <int DA>
__device__ __forceinline__ void grad_signal(const HeadIn<DA>& hin, const HeadOut<DA>& o, float obj_scale, float kl_eff, float invN,
                                            float (&dmu)[DA], float (&dls)[DA]) {
    const float wt = obj_scale * o.w * invN, kc = kl_eff * invN;
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        dmu[d] = wt * o.zeta[d] * hin.inv_sig[d] + kc * o.dkl_dmu[d];
        dls[d] = (wt * (o.zeta[d] * o.zeta[d] - 1.f) + kc * o.dkl_dls[d]) * hin.ls_mask[d];
    }
}

// Signals of the HVP kernels at the head for one sample, from the mean's tangent rmu and the (clipped) log_std's tangent rls:
// dmu = d loss / d mu, and the combined signals cmu / cls = ac * (tangent of d loss / d mu, log_std) + KL-penalty gradient.
template <int DA>
__device__ __forceinline__ void hvp_signal(const HeadIn<DA>& hin, const HeadOut<DA>& o, const float (&rmu)[DA], const float (&rls)[DA],
                                           int obj_kind, float kl_eff, float invN, float ac, int dA, float (&dmu)[DA],
                                           float (&cmu)[DA], float (&cls)[DA]) {
    const float wt = o.w * invN, kc = kl_eff * invN;
    // tangent of log p:  R l = sum_d (zeta/sig) R mu + (zeta^2 - 1) R ls
    float rl = 0.f;
#pragma unroll
    for (int d = 0; d < DA; ++d) rl += (o.zeta[d] * hin.inv_sig[d]) * rmu[d] + (o.zeta[d] * o.zeta[d] - 1.f) * rls[d];
    // d w / d logp: RATIO w = -A r -> R w = w R l ; LOGLIK w = -A -> 0
    const float rwt = (obj_kind == PROMP_OBJ_RATIO) ? wt * rl : 0.f;
#pragma unroll
    for (int d = 0; d < DA; ++d) {
        const float is = hin.inv_sig[d], z = o.zeta[d];
        const float rz = -rmu[d] * is - z * rls[d];
        dmu[d] = wt * z * is;
        const float rdmu = rwt * z * is + wt * (rz * is - z * rls[d] * is);
        const float rdls = rwt * (z * z - 1.f) + wt * 2.f * z * rz;
        cmu[d] = ac * rdmu + kc * o.dkl_dmu[d];
        cls[d] = (ac * rdls + kc * o.dkl_dls[d]) * hin.ls_mask[d];
        if (d >= dA) dmu[d] = cmu[d] = 0.f;      // padding: exactly zero whatever the direction's pad entries hold
    }
}

// -------------------------------------------------------------------------------------------------------------
// Last-arriver epilogues of the flush below: pre(p) is requested together with the slot loads, then out(p, pre, sum)
// stores float4 column p of the task's summed slots.
template <int P, class Sched>
struct GradEpilogue {      // grad = sum ; out_params = params - sgd_lr * grad   (meta_algos/base.py:209)
    const PolicyArgs& A;   // or params - alpha * grad with per-parameter step sizes (A.step_size)
    const float* th;
    int m;
    __device__ __forceinline__ float4 pre(int p) const {
        return A.out_params ? Sched::ldp4(reinterpret_cast<const float4*>(th + p)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __device__ __forceinline__ void out(int p, float4 t, float4 s) const {
        *reinterpret_cast<float4*>(A.grad + (int64_t)m * P + p) = s;
        if (A.out_params) {
            float4* o = reinterpret_cast<float4*>(A.out_params + (int64_t)m * P + p);
            if (A.step_size) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(A.step_size + p));
                *o = make_float4(t.x - a.x * s.x, t.y - a.y * s.y, t.z - a.z * s.z, t.w - a.w * s.w);
            } else {
                *o = make_float4(t.x - A.sgd_lr * s.x, t.y - A.sgd_lr * s.y, t.z - A.sgd_lr * s.z, t.w - A.sgd_lr * s.w);
            }
        }
    }
};
template <int P>
struct HvpEpilogue {       // out = vec + sum
    const PolicyArgs& A;
    const float* vg;       // task m's direction vector, written by the previous kernel or stage (L2 loads)
    int m;
    __device__ __forceinline__ float4 pre(int p) const { return __ldcg(reinterpret_cast<const float4*>(vg + p)); }
    __device__ __forceinline__ void out(int p, float4 v, float4 s) const {
        *reinterpret_cast<float4*>(A.out + (int64_t)m * P + p) = make_float4(v.x + s.x, v.y + s.y, v.z + s.z, v.w + s.w);
    }
};

// Task-segment flush, shared by the four tile loops.  The caller has stored the parts of its partial slot `part` that depend
// on its own register layout (W1, b1, b0, b2, log_std) and passed a barrier after its last use of `scr` (SCR floats of shared
// scratch, at least NPART x max(DO, DA) x HID).  This reduces the column-role W0 / W2 partials (unit tid % HID over sample slice
// tid / HID) over the NPART slices and the three head statistics (zero on threads without a sample row) over the warps, and
// takes task m's arrival ticket; the last arriver sums the task's slots in contributor order - the statistics ride in the
// trailing float4 - and hands every float4 column to `epi`.  want == false (values-only gradient): statistics only.  A thread
// reduces up to WIDE of its float4 columns at once (4 WIDE L2 loads in flight, ~20 WIDE registers).
template <int THREADS, int WIDE, int SCR, int DO, int DA, int HID, class Sched, class Epi>
__device__ __forceinline__ void flush_tail(const PolicyArgs& A, const Sched& sc, int m, float invN, bool want, float* part,
                                           float* scr, float* red, int& last, const float (&gW0p)[DO], const float (&gW2p)[DA],
                                           float s_obj, float s_kl, float s_ratio, const Epi& epi) {
    using L = PLayout<DO, DA, HID>;
    constexpr int NPART = THREADS / HID, NW = THREADS / 32, PSTRIDE = L::P + PSTAT;
    static_assert(NPART * DO * HID <= SCR && NPART * HID * DA <= SCR, "flush scratch too small");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cj = tid % HID, cp = tid / HID;
    if (want) {
#pragma unroll
        for (int i = 0; i < DO; ++i) scr[(cp * DO + i) * HID + cj] = gW0p[i];
        __syncthreads();
        for (int idx = tid; idx < DO * HID; idx += THREADS) {
            float s = 0.f;
            for (int p = 0; p < NPART; ++p) s += scr[p * DO * HID + idx];
            part[L::W0 + idx] = s;
        }
        __syncthreads();
#pragma unroll
        for (int d = 0; d < DA; ++d) scr[(cp * HID + cj) * DA + d] = gW2p[d];
        __syncthreads();
        for (int idx = tid; idx < HID * DA; idx += THREADS) {
            float s = 0.f;
            for (int p = 0; p < NPART; ++p) s += scr[p * HID * DA + idx];
            part[L::W2 + idx] = s;
        }
    }
    const float v0 = warp_sum(s_obj), v1 = warp_sum(s_kl), v2 = warp_sum(s_ratio);
    __syncthreads();
    if (lane == 0) red[warp] = v0, red[NW + warp] = v1, red[2 * NW + warp] = v2;
    __syncthreads();
    if (tid < 3) {
        float s = 0.f;
        for (int w = 0; w < NW; ++w) s += red[tid * NW + w];
        part[L::P + tid] = s;
    }
    __syncthreads();
    const int n_c = sc.n_contrib(m);
    if (tid == 0) {          // release by ONE thread: the barrier above orders the CTA's partial-slot writes before this fence
        __threadfence();
        last = (atomicAdd(A.counters + m, 1) == n_c - 1);
    }
    __syncthreads();
    sc.clk(4);
    if (last) {
        __threadfence();
        static_assert(L::P % 4 == 0 && PSTAT == 4, "stats ride on the float4 reduction");
        if (want) {
            constexpr int NPASS = (L::P + 4 + 4 * THREADS - 1) / (4 * THREADS);
            constexpr int NP = NPASS < WIDE ? NPASS : WIDE;
#pragma unroll 1
            for (int p0 = 4 * tid; p0 < L::P + 4; p0 += NP * 4 * THREADS) {
                float4 sum[NP], t4[NP];
#pragma unroll
                for (int i = 0; i < NP; ++i) {          // requested together with the slot loads below
                    const int p = p0 + i * 4 * THREADS;
                    t4[i] = p < L::P ? epi.pre(p) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                reduce_slots4_wide<NP>(A.partial, sc, PSTRIDE, m, n_c, p0, 4 * THREADS, L::P + 4, sum);
#pragma unroll
                for (int i = 0; i < NP; ++i) {
                    const int p = p0 + i * 4 * THREADS;
                    const float4 s = sum[i];
                    if (p == L::P) {
                        if (A.stats)
                            A.stats[(int64_t)m * 4 + 0] = s.x * invN, A.stats[(int64_t)m * 4 + 1] = s.y * invN,
                                                    A.stats[(int64_t)m * 4 + 2] = s.z * invN;
                    } else if (p < L::P) {
                        epi.out(p, t4[i], s);
                    }
                }
            }
        } else if (tid == 0 && A.stats) {
            const float4 s = reduce_slots4(A.partial, sc, PSTRIDE, m, n_c, L::P);
            A.stats[(int64_t)m * 4 + 0] = s.x * invN, A.stats[(int64_t)m * 4 + 1] = s.y * invN, A.stats[(int64_t)m * 4 + 2] = s.z * invN;
        }
        if (tid == 0) A.counters[m] = 0;
        sc.publish_task(m);
        sc.clk(5);
    }
    __syncthreads();
}

}  // namespace promp
