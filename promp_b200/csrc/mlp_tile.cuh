// Shared-memory tile machinery for the Gaussian-MLP policy kernels (policy_grad / policy_hvp).
//
// A CTA of 256 threads processes tiles of TB = 64 samples of ONE task.  All weight matrices of the
// task live in shared memory; activations are [TB][LD] row-major tiles (LD = HID + 4 keeps rows
// 16-byte aligned and spreads banks).  The 64 x HID x HID products are register-tiled SIMT fp32
// GEMMs (RM x 4 outputs per thread, float4 shared-memory loads): float32 FMA keeps the 1e-4 parity
// bar against the reference's float32 TF graph; tensor-core tf32/bf16 would not.
#pragma once
#include "common.cuh"

namespace promp {

constexpr int PT_THREADS = 256;
constexpr int TB = 64;   // samples per tile

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
#if defined(PROMP_EXP_NO_GEMM) || defined(PROMP_EXP_NO_LAYER_GEMM)   // kernel-time experiments only (tools/kernel_time.py)
    return;
#endif
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
#ifdef PROMP_EXP_NO_GEMM
    return;
#endif
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

}  // namespace promp
