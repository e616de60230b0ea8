// Gaussian-MLP policy kernels: per-task objective gradient (inner adapt step, outer surrogates, KL
// terms) and the exact Hessian-vector product that carries the MAML meta-gradient through the inner
// SGD step.  See include/promp_b200.h for the interface and the reference functions replaced.
//
// Work decomposition: persistent CTAs, one wave.  The M*ceil(N/64) sample tiles form one task-major
// list; CTA c owns the contiguous range [c*q, (c+1)*q) (q = ceil(T/grid), grid = SMs x resident
// CTAs), so every SM gets the same number of tiles whatever M and N are.  A CTA keeps the current
// task's weights in shared memory and its weight-gradient accumulators in registers; when its range
// crosses a task boundary (or ends) it flushes them to a per-(CTA,task) partial slot, and the last
// segment of each task to arrive (atomic ticket) reduces that task's slots in CTA order -> bitwise
// run-to-run deterministic sums.  These kernels are fp32-FMA bound (AI ~ 10^2..10^3 FLOP/B).
#include <string.h>
#include <type_traits>
#include "policy_tc.cuh"

// This file is compiled twice: as itself (tanh: every kernel, option, entry point) and through policy_relu.cu, which
// defines PROMP_POLICY_RELU_TU and compiles only the ReLU instantiations of the templated kernels and launchers
// (namespace promp::relu_tu below).  Separate translation units keep the tanh kernels' code exactly what it was before
// ReLU existed, and the two halves compile in parallel.  The tanh-output policies (OutTanh<ActTanh>, OutTanh<ActRelu>) are two
// more units of the same kind: policy_otanh.cu (PROMP_POLICY_OTANH_TU, namespace otanh_tu) and policy_relu_otanh.cu (both
// macros, namespace relu_otanh_tu).  PROMP_POLICY_EXTRA_TU marks every unit but this one.
#if defined(PROMP_POLICY_RELU_TU) || defined(PROMP_POLICY_OTANH_TU)
#define PROMP_POLICY_EXTRA_TU
#endif
#if defined(PROMP_POLICY_RELU_TU) && defined(PROMP_POLICY_OTANH_TU)
#define PROMP_POLICY_ACT OutTanh<ActRelu>
#define PROMP_ACT_NS relu_otanh_tu
#elif defined(PROMP_POLICY_OTANH_TU)
#define PROMP_POLICY_ACT OutTanh<ActTanh>
#define PROMP_ACT_NS otanh_tu
#elif defined(PROMP_POLICY_RELU_TU)
#define PROMP_POLICY_ACT ActRelu
#define PROMP_ACT_NS relu_tu
#else
#define PROMP_POLICY_ACT ActTanh
#define PROMP_ACT_NS tanh_tu
#endif

namespace promp {

// -------------------------------------------------------------------------------------------------
// Thread roles inside a 256-thread CTA working on a 64-sample tile:
//   GEMM role      (tx, ty): 4 (HID=64) or 2 (HID=32) rows x 4 columns of every [64 x HID] product
//   row role       (rb, rq): 4 threads per sample row, each owns a quarter of the hidden units (layer 2 + head)
//   column role    (cj, cp): thread owns hidden unit cj for the sample slice cp (small weight gradients)
// Small reductions (bias / W0 / W2 gradients) are accumulated per thread in registers across tiles and
// only combined through shared memory when the CTA flushes a task segment.
template <int HID>
struct RoleCfg {
    static constexpr int NPART = PT_THREADS / HID;    // sample slices for the column role (4 | 8)
    static constexpr int BPP = TB / NPART;            // samples per slice (16 | 8)
    static constexpr int QW = HID / 4;                // hidden units per row-role thread (16 | 8)
};

template <int DO, int DA, int HID>
struct GradSmem {
    using L = PLayout<DO, DA, HID>;
    using C = TileCfg<HID>;
    static constexpr int DOP = DOPad<DO>::V;
    static constexpr int PP = (L::P + 3) / 4 * 4;
    float P[PP];
    float W1T[HID * HID];
    float X[TB * DOP];
    float H1[TB * C::LD];     // also: flush scratch
    float H2[TB * C::LD];
    float DMU[TB * DA];
    float DLS[TB * DA];
    float red[3 * (PT_THREADS / 32)];
    int last;
};

template <int DO, int DA, int HID, class Act, int ADV = ADV_SAMPLE>
__device__ __forceinline__ void policy_grad_body(const PolicyArgs& A) {
    using L = PLayout<DO, DA, HID>;
    using C = TileCfg<HID>;
    using R = RoleCfg<HID>;
    using SM = GradSmem<DO, DA, HID>;
    constexpr int LD = C::LD, RM = C::RM, RK = C::RK, DOP = SM::DOP;
    constexpr int BPP = R::BPP, QW = R::QW;
    constexpr int PSTRIDE = L::P + PSTAT;
    constexpr int SCR = (int)((offsetof(SM, red) - offsetof(SM, X)) / sizeof(float));    // flush scratch: X .. DLS

    extern __shared__ __align__(16) unsigned char smem_raw[];
    SM& S = *reinterpret_cast<SM*>(smem_raw);

    const int tid = threadIdx.x;
    const int tx = tid % C::TX, ty = tid / C::TX;
    const int row0 = ty * RM, col0 = tx * 4;
    const int rb = tid >> 2, rq = tid & 3;           // row role
    const int cj = tid % HID, cp = tid / HID;        // column role
    const int dO = obs_dim_of<DO, DA>(A), dA = act_dim_of<DO, DA>(A);
    if (reuse_hit<L::P>(A.skip_flag, A.params, A.skip_theta)) return;
    reuse_produce<L::P, L::LS, DA>(A);
    const UniformSched sc(A.M, A.N, A.q, A.kmax, TB);
    const int N = A.N;
    const float kl_eff = kl_coeff_eff(A);
    float invN = 1.0f / (float)N;       // both re-set per task when A.n_valid is given (variable-length paths)
    int Nm = N;
    const bool want_grad = A.grad != nullptr;
    const float* th = nullptr;
    HeadIn<DA> hin;

    // register accumulators (per task segment)
    float gW1[RK][4];        // GEMM role: H1^T D2 block
    float gB1p[4], gB0p[4];  // GEMM role: column sums over this thread's rows
    float gW0p[DO], gW2p[DA];   // column role: X^T D1 / H2^T DMU for unit cj over sample slice cp
    float gB2 = 0.f, gLS = 0.f; // thread tid < DA
    float s_obj, s_kl, s_ratio; // row role, rq == 0
    auto zero_acc = [&]() {
#pragma unroll
        for (int r = 0; r < RK; ++r) gW1[r][0] = gW1[r][1] = gW1[r][2] = gW1[r][3] = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) gB1p[c] = gB0p[c] = 0.f;
#pragma unroll
        for (int i = 0; i < DO; ++i) gW0p[i] = 0.f;
#pragma unroll
        for (int d = 0; d < DA; ++d) gW2p[d] = 0.f;
        gB2 = gLS = 0.f;
        s_obj = s_kl = s_ratio = 0.f;
    };
    auto load_task = [&](int m, bool first) {
        if (A.n_valid) { Nm = __ldg(A.n_valid + m); invN = 1.0f / (float)max(Nm, 1); }
        th = A.params + (int64_t)m * A.param_stride;
        if (!first && A.param_stride == 0) return;       // shared theta: weights already resident
        __syncthreads();
        for (int i = tid; i < L::P; i += PT_THREADS) S.P[i] = __ldg(th + i);
        __syncthreads();
        for (int i = tid; i < HID * HID; i += PT_THREADS) {
            const int j = i / HID, k = i % HID;      // consecutive threads -> consecutive W1T addresses
            S.W1T[j * HID + k] = S.P[L::W1 + k * HID + j];
        }
        head_setup<DA>(A, S.P + L::LS, m, dA, hin, nullptr);
    };
    // write this CTA's partial sums for task m; the last segment of the task reduces them in CTA order
    auto flush = [&](int m) {
        float* part = A.partial + (int64_t)sc.my_slot(m) * PSTRIDE;
        float* scr = S.X;       // X .. DLS: free between tiles (H1 alone is too small for the W0 slices of <20, 2, 32>)
        __syncthreads();
        if (want_grad) {
#pragma unroll
            for (int r = 0; r < RK; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) part[L::W1 + (ty * RK + r) * HID + col0 + c] = gW1[r][c];
            // column sums: reduce the C::TY row groups
#pragma unroll
            for (int c = 0; c < 4; ++c) scr[ty * HID + col0 + c] = gB1p[c];
            __syncthreads();
            if (tid < HID) {
                float s = 0.f;
                for (int y = 0; y < C::TY; ++y) s += scr[y * HID + tid];
                part[L::B1 + tid] = s;
            }
            __syncthreads();
#pragma unroll
            for (int c = 0; c < 4; ++c) scr[ty * HID + col0 + c] = gB0p[c];
            __syncthreads();
            if (tid < HID) {
                float s = 0.f;
                for (int y = 0; y < C::TY; ++y) s += scr[y * HID + tid];
                part[L::B0 + tid] = s;
            }
            __syncthreads();
            if (tid < DA) part[L::B2 + tid] = gB2, part[L::LS + tid] = gLS;
        }
        flush_tail<PT_THREADS, 2, SCR, DO, DA, HID>(A, sc, m, invN, want_grad, part, scr, S.red, S.last, gW0p, gW2p, s_obj, s_kl, s_ratio,
                                               GradEpilogue<L::P, UniformSched>{A, th, m});
    };

    int cur_m = -1;
    for (int g = sc.g_lo; g < sc.g_hi; ++g) {
        const int m = g / sc.ntiles, tile = g - m * sc.ntiles;
        if (m != cur_m) {
            if (cur_m >= 0) flush(cur_m);
            load_task(m, cur_m < 0);
            zero_acc();
            cur_m = m;
        }
        const int n0 = tile * TB, nb = max(0, min(TB, Nm - n0));
        const int64_t g0 = (int64_t)m * N + n0;
        __syncthreads();
        for (int i = tid; i < TB * DOP; i += PT_THREADS) {
            const int b = i / DOP, c = i % DOP;
            S.X[i] = (b < nb && c < dO) ? __ldg(A.obs + (g0 + b) * dO + c) : 0.f;
        }
        __syncthreads();
        // ---- layer 0: H1 = act(X W0 + b0)                       (policies/networks/mlp.py:96-117)
        {
            float acc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.P + L::B0 + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
            gemm_tile_smallk<DO, DOP, HID, RM>(S.X, S.P + L::W0, row0, col0, acc);
#pragma unroll
            for (int i = 0; i < RM; ++i)
                *reinterpret_cast<float4*>(S.H1 + (row0 + i) * LD + col0) =
                    make_float4(Act::f(acc[i][0]), Act::f(acc[i][1]), Act::f(acc[i][2]), Act::f(acc[i][3]));
        }
        __syncthreads();
        // ---- layer 1: H2 = act(H1 W1 + b1)
        {
            float acc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.P + L::B1 + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
            gemm_tile<HID, LD, HID, RM>(S.H1, S.P + L::W1, row0, col0, acc);
#pragma unroll
            for (int i = 0; i < RM; ++i)
                *reinterpret_cast<float4*>(S.H2 + (row0 + i) * LD + col0) =
                    make_float4(Act::f(acc[i][0]), Act::f(acc[i][1]), Act::f(acc[i][2]), Act::f(acc[i][3]));
        }
        __syncthreads();
        // ---- layer 2 + Gaussian head: 4 threads per sample row, quarter dot products + 2 shuffles
        {
            float mu[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = 0.f;
#pragma unroll
            for (int k4 = 0; k4 < QW / 4; ++k4) {
                const int j = rq * QW + 4 * k4;
                const float4 h = *reinterpret_cast<const float4*>(S.H2 + rb * LD + j);
#pragma unroll
                for (int d = 0; d < DA; ++d) {
                    mu[d] = fmaf(h.x, S.P[L::W2 + (j + 0) * DA + d], mu[d]);
                    mu[d] = fmaf(h.y, S.P[L::W2 + (j + 1) * DA + d], mu[d]);
                    mu[d] = fmaf(h.z, S.P[L::W2 + (j + 2) * DA + d], mu[d]);
                    mu[d] = fmaf(h.w, S.P[L::W2 + (j + 3) * DA + d], mu[d]);
                }
            }
#pragma unroll
            for (int d = 0; d < DA; ++d) {
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 1);
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 2);
                mu[d] += S.P[L::B2 + d];
            }
            if (rq == 0) {
                float dmu[DA], dls[DA];
                if (rb < nb) {
                    float a[DA], mo[DA], lso[DA];
                    const float adv = load_head_sample<DA, ADV>(A, g0 + rb, m, dA, true, a, mo, lso);
                    HeadOut<DA> o;
                    HeadOld<DA> ho;
                    head_old_from<DA>(lso, ho, dA);
                    out_forward<Act, DA>(mu);
                    gaussian_head<DA>(hin, ho, mu, a, mo, adv, A.obj_kind, A.clip_eps, o, dA);
                    grad_signal<DA>(hin, o, A.obj_scale, kl_eff, invN, dmu, dls);
                    out_grad_back<Act, DA>(mu, dmu);
                    s_obj += o.obj;
                    s_kl += o.kl;
                    s_ratio += o.ratio;
                } else {
#pragma unroll
                    for (int d = 0; d < DA; ++d) dmu[d] = dls[d] = 0.f;
                }
#pragma unroll
                for (int d = 0; d < DA; ++d) S.DMU[rb * DA + d] = dmu[d], S.DLS[rb * DA + d] = dls[d];
            }
        }
        if (!want_grad) continue;
        __syncthreads();
        // ---- output layer gradients (column role): gW2[cj][d] += sum_{b in slice} H2[b][cj] * DMU[b][d]
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float h = S.H2[b * LD + cj];
#pragma unroll
                for (int d = 0; d < DA; ++d) gW2p[d] = fmaf(h, S.DMU[b * DA + d], gW2p[d]);
            }
            if (tid < DA) {
                float s1 = 0.f, s2 = 0.f;
                for (int b = 0; b < nb; ++b) s1 += S.DMU[b * DA + tid], s2 += S.DLS[b * DA + tid];
                gB2 += s1;
                gLS += s2;
            }
        }
        __syncthreads();
        // ---- D2 = (DMU W2^T) * act'(H2), in place over H2; bias gradient accumulates on the fly
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            const int b = row0 + i;
            float4 h = *reinterpret_cast<float4*>(S.H2 + b * LD + col0);
            float hv[4] = {h.x, h.y, h.z, h.w}, o4[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float dh = 0.f;
#pragma unroll
                for (int d = 0; d < DA; ++d) dh = fmaf(S.DMU[b * DA + d], S.P[L::W2 + (col0 + c) * DA + d], dh);
                o4[c] = dh * Act::d(hv[c]);
                gB1p[c] += o4[c];
            }
            *reinterpret_cast<float4*>(S.H2 + b * LD + col0) = make_float4(o4[0], o4[1], o4[2], o4[3]);
        }
        __syncthreads();
        // ---- gW1 += H1^T D2 ; dH1 = D2 W1^T
        wgrad_tile<LD, RK>(S.H1, S.H2, ty * RK, col0, nb, gW1);
        float acc[RM][4];
#pragma unroll
        for (int i = 0; i < RM; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
        gemm_tile<HID, LD, HID, RM>(S.H2, S.W1T, row0, col0, acc);
        __syncthreads();   // every read of H1 (wgrad) is done before it is overwritten
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            float4 h = *reinterpret_cast<float4*>(S.H1 + (row0 + i) * LD + col0);
            const float4 d1 = make_float4(acc[i][0] * Act::d(h.x), acc[i][1] * Act::d(h.y), acc[i][2] * Act::d(h.z),
                                          acc[i][3] * Act::d(h.w));
            gB0p[0] += d1.x; gB0p[1] += d1.y; gB0p[2] += d1.z; gB0p[3] += d1.w;
            *reinterpret_cast<float4*>(S.H1 + (row0 + i) * LD + col0) = d1;
        }
        __syncthreads();
        // ---- gW0 += X^T D1 (column role)
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float d1 = S.H1[b * LD + cj];
#pragma unroll
                for (int i = 0; i < DO; ++i) gW0p[i] = fmaf(S.X[b * DOP + i], d1, gW0p[i]);
            }
        }
    }
    if (cur_m >= 0) flush(cur_m);
}

// One kernel per activation (the tanh kernels keep their names): *_kernel = tanh, *_relu_kernel = ReLU
template <int DO, int DA, int HID>
__global__ void __launch_bounds__(PT_THREADS, 2) policy_grad_kernel(PolicyArgs A) { policy_grad_body<DO, DA, HID, ActTanh>(A); }
template <int DO, int DA, int HID>
__global__ void __launch_bounds__(PT_THREADS, 2) policy_grad_relu_kernel(PolicyArgs A) { policy_grad_body<DO, DA, HID, ActRelu>(A); }
// PROMP_OBJ_EXPLORE (E-MAML): the same kernel reading the per-task weight adv[m]; separate functions keep the kernels above
// exactly what they were
template <int DO, int DA, int HID>
__global__ void __launch_bounds__(PT_THREADS, 2) policy_grad_explore_kernel(PolicyArgs A) {
    policy_grad_body<DO, DA, HID, ActTanh, ADV_TASK>(A);
}
template <int DO, int DA, int HID>
__global__ void __launch_bounds__(PT_THREADS, 2) policy_grad_explore_relu_kernel(PolicyArgs A) {
    policy_grad_body<DO, DA, HID, ActRelu, ADV_TASK>(A);
}
// tanh output layer: *_otanh_kernel<..., Hid> for hidden activation Hid (ActTanh or ActRelu)
template <int DO, int DA, int HID, class Hid>
__global__ void __launch_bounds__(PT_THREADS, 2) policy_grad_otanh_kernel(PolicyArgs A) {
    policy_grad_body<DO, DA, HID, OutTanh<Hid>>(A);
}
template <int DO, int DA, int HID, class Hid>
__global__ void __launch_bounds__(PT_THREADS, 2) policy_grad_explore_otanh_kernel(PolicyArgs A) {
    policy_grad_body<DO, DA, HID, OutTanh<Hid>, ADV_TASK>(A);
}

// -------------------------------------------------------------------------------------------------
// Exact Hessian-vector product of the inner surrogate (R-operator: forward-mode tangent through the
// MLP + Gaussian log-likelihood, then the reverse sweep of the tangent), fused with the KL-penalty
// gradient:  out = vec - inner_lr * H vec + kl_coeff * grad KL.   Notation in the comments:
//   H1,H2 activations; R1,R2 their tangents; D* = backprop of the surrogate; C* = combined
//   (-inner_lr * tangent-of-backprop + kl-penalty backprop) signal that is accumulated into `out`.
template <int DO, int DA, int HID>
struct HvpSmem {
    using L = PLayout<DO, DA, HID>;
    using C = TileCfg<HID>;
    static constexpr int DOP = DOPad<DO>::V;
    static constexpr int PP = (L::P + 3) / 4 * 4;
    float P[PP];
    float V[PP];
    float W1T[HID * HID];
    float V1T[HID * HID];
    float X[TB * DOP];
    float H1[TB * C::LD];     // also: flush scratch
    float R1[TB * C::LD];
    float H2[TB * C::LD];
    float R2[TB * C::LD];
    float DMU[TB * DA];
    float CMU[TB * DA];
    float CLS[TB * DA];
    float red[3 * (PT_THREADS / 32)];
    int last;
};

template <int DO, int DA, int HID, class Act>
__device__ __forceinline__ void policy_hvp_body(const PolicyArgs& A) {
    using L = PLayout<DO, DA, HID>;
    using C = TileCfg<HID>;
    using R = RoleCfg<HID>;
    using SM = HvpSmem<DO, DA, HID>;
    constexpr int LD = C::LD, RM = C::RM, RK = C::RK, DOP = SM::DOP;
    constexpr int BPP = R::BPP, QW = R::QW;
    constexpr int PSTRIDE = L::P + PSTAT;
    constexpr int SCR = (int)((offsetof(SM, red) - offsetof(SM, H1)) / sizeof(float));   // flush scratch: H1 .. CLS

    extern __shared__ __align__(16) unsigned char smem_raw[];
    SM& S = *reinterpret_cast<SM*>(smem_raw);

    const int tid = threadIdx.x;
    const int tx = tid % C::TX, ty = tid / C::TX;
    const int row0 = ty * RM, col0 = tx * 4;
    const int rb = tid >> 2, rq = tid & 3;
    const int cj = tid % HID, cp = tid / HID;
    const int dO = obs_dim_of<DO, DA>(A), dA = act_dim_of<DO, DA>(A);
    const UniformSched sc(A.M, A.N, A.q, A.kmax, TB);
    const int N = A.N;
    const float kl_eff = kl_coeff_eff(A);
    float invN = 1.0f / (float)N;       // both re-set per task when A.n_valid is given (variable-length paths)
    int Nm = N;
    const float ac = -A.inner_lr;                 // coefficient of H vec in `out`
    const float* th = nullptr;
    const float* vg = nullptr;
    HeadIn<DA> hin;
    float rls[DA];     // tangent of the (clipped) log_std

    // accumulators: gW1c multiplies 1, gW1a multiplies `ac`
    float gW1c[RK][4], gW1a[RK][4], gB1p[4], gB0p[4], gW0p[DO], gW2p[DA];
    float gB2 = 0.f, gLS = 0.f;
    float s_obj, s_kl, s_ratio;
    auto zero_acc = [&]() {
#pragma unroll
        for (int r = 0; r < RK; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) gW1c[r][c] = gW1a[r][c] = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) gB1p[c] = gB0p[c] = 0.f;
#pragma unroll
        for (int i = 0; i < DO; ++i) gW0p[i] = 0.f;
#pragma unroll
        for (int d = 0; d < DA; ++d) gW2p[d] = 0.f;
        gB2 = gLS = 0.f;
        s_obj = s_kl = s_ratio = 0.f;
    };
    auto load_task = [&](int m, bool first) {
        if (A.n_valid) { Nm = __ldg(A.n_valid + m); invN = 1.0f / (float)max(Nm, 1); }
        th = A.params + (int64_t)m * A.param_stride;
        vg = A.vec + (int64_t)m * L::P;
        const bool reload_p = first || A.param_stride != 0;      // shared theta stays resident across tasks
        __syncthreads();
        for (int i = tid; i < L::P; i += PT_THREADS) {
            if (reload_p) S.P[i] = __ldg(th + i);
            const float v = __ldcg(vg + i);                      // written by the previous kernel on this stream
            S.V[i] = A.step_size ? __ldg(A.step_size + i) * v : v;       // the direction H is applied to: alpha * vec
        }
        __syncthreads();
        for (int i = tid; i < HID * HID; i += PT_THREADS) {
            const int j = i / HID, k = i % HID;      // consecutive threads -> consecutive addresses of the transposes
            if (reload_p) S.W1T[j * HID + k] = S.P[L::W1 + k * HID + j];
            S.V1T[j * HID + k] = S.V[L::W1 + k * HID + j];
        }
        head_setup<DA>(A, S.P + L::LS, m, dA, hin, nullptr);
#pragma unroll
        for (int d = 0; d < DA; ++d) rls[d] = S.V[L::LS + d] * hin.ls_mask[d];
    };
    auto flush = [&](int m) {
        float* part = A.partial + (int64_t)sc.my_slot(m) * PSTRIDE;
        float* scr = S.H1;      // H1 .. CLS: free between tiles
        __syncthreads();
#pragma unroll
        for (int r = 0; r < RK; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) part[L::W1 + (ty * RK + r) * HID + col0 + c] = gW1c[r][c] + ac * gW1a[r][c];
#pragma unroll
        for (int c = 0; c < 4; ++c) scr[ty * HID + col0 + c] = gB1p[c];
        __syncthreads();
        if (tid < HID) {
            float s = 0.f;
            for (int y = 0; y < C::TY; ++y) s += scr[y * HID + tid];
            part[L::B1 + tid] = s;
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < 4; ++c) scr[ty * HID + col0 + c] = gB0p[c];
        __syncthreads();
        if (tid < HID) {
            float s = 0.f;
            for (int y = 0; y < C::TY; ++y) s += scr[y * HID + tid];
            part[L::B0 + tid] = s;
        }
        __syncthreads();
        if (tid < DA) part[L::B2 + tid] = gB2, part[L::LS + tid] = gLS;
        flush_tail<PT_THREADS, 2, SCR, DO, DA, HID>(A, sc, m, invN, true, part, scr, S.red, S.last, gW0p, gW2p, s_obj, s_kl, s_ratio,
                                               HvpEpilogue<L::P>{A, vg, m});
    };

    int cur_m = -1;
    for (int g = sc.g_lo; g < sc.g_hi; ++g) {
        const int m = g / sc.ntiles, tile = g - m * sc.ntiles;
        if (m != cur_m) {
            if (cur_m >= 0) flush(cur_m);
            load_task(m, cur_m < 0);
            zero_acc();
            cur_m = m;
        }
        const int n0 = tile * TB, nb = max(0, min(TB, Nm - n0));
        const int64_t g0 = (int64_t)m * N + n0;
        __syncthreads();
        for (int i = tid; i < TB * DOP; i += PT_THREADS) {
            const int b = i / DOP, c = i % DOP;
            S.X[i] = (b < nb && c < dO) ? __ldg(A.obs + (g0 + b) * dO + c) : 0.f;
        }
        __syncthreads();
        // ---- layer 0 and its tangent: H1 = act(X W0 + b0); R1 = act'(H1) * (X V0 + vb0)
        {
            float acc[RM][4], racc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.P + L::B0 + col0);
            const float4 rv = *reinterpret_cast<const float4*>(S.V + L::B0 + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
                racc[i][0] = rv.x, racc[i][1] = rv.y, racc[i][2] = rv.z, racc[i][3] = rv.w;
            }
            gemm_tile_smallk<DO, DOP, HID, RM>(S.X, S.P + L::W0, row0, col0, acc);
            gemm_tile_smallk<DO, DOP, HID, RM>(S.X, S.V + L::W0, row0, col0, racc);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                float h[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) h[c] = Act::f(acc[i][c]);
                *reinterpret_cast<float4*>(S.H1 + (row0 + i) * LD + col0) = make_float4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<float4*>(S.R1 + (row0 + i) * LD + col0) =
                    make_float4(Act::d(h[0]) * racc[i][0], Act::d(h[1]) * racc[i][1], Act::d(h[2]) * racc[i][2],
                                Act::d(h[3]) * racc[i][3]);
            }
        }
        __syncthreads();
        // ---- layer 1 and its tangent: R2 = act'(H2) * (R1 W1 + H1 V1 + vb1)
        {
            float acc[RM][4], racc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.P + L::B1 + col0);
            const float4 rv = *reinterpret_cast<const float4*>(S.V + L::B1 + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
                racc[i][0] = rv.x, racc[i][1] = rv.y, racc[i][2] = rv.z, racc[i][3] = rv.w;
            }
            gemm_tile<HID, LD, HID, RM>(S.H1, S.P + L::W1, row0, col0, acc);
            gemm_tile<HID, LD, HID, RM>(S.R1, S.P + L::W1, row0, col0, racc);
            gemm_tile<HID, LD, HID, RM>(S.H1, S.V + L::W1, row0, col0, racc);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                float h[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) h[c] = Act::f(acc[i][c]);
                *reinterpret_cast<float4*>(S.H2 + (row0 + i) * LD + col0) = make_float4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<float4*>(S.R2 + (row0 + i) * LD + col0) =
                    make_float4(Act::d(h[0]) * racc[i][0], Act::d(h[1]) * racc[i][1], Act::d(h[2]) * racc[i][2],
                                Act::d(h[3]) * racc[i][3]);
            }
        }
        __syncthreads();
        // ---- layer 2, its tangent, and the Gaussian head with its tangent (row role)
        {
            float mu[DA], rmu[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = rmu[d] = 0.f;
#pragma unroll
            for (int k4 = 0; k4 < QW / 4; ++k4) {
                const int j = rq * QW + 4 * k4;
                const float4 h4 = *reinterpret_cast<const float4*>(S.H2 + rb * LD + j);
                const float4 r4 = *reinterpret_cast<const float4*>(S.R2 + rb * LD + j);
                const float hv[4] = {h4.x, h4.y, h4.z, h4.w}, rv[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int d = 0; d < DA; ++d) {
                        const float w2 = S.P[L::W2 + (j + e) * DA + d];
                        mu[d] = fmaf(hv[e], w2, mu[d]);
                        rmu[d] = fmaf(rv[e], w2, fmaf(hv[e], S.V[L::W2 + (j + e) * DA + d], rmu[d]));
                    }
            }
#pragma unroll
            for (int d = 0; d < DA; ++d) {
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 1);
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 2);
                rmu[d] += __shfl_xor_sync(0xffffffffu, rmu[d], 1);
                rmu[d] += __shfl_xor_sync(0xffffffffu, rmu[d], 2);
                mu[d] += S.P[L::B2 + d];
                rmu[d] += S.V[L::B2 + d];
            }
            if (rq == 0) {
                float dmu[DA], cmu[DA], cls[DA];
                if (rb < nb) {
                    float a[DA], mo[DA], lso[DA];
                    const float adv = load_head_sample<DA>(A, g0 + rb, m, dA, true, a, mo, lso);
                    HeadOut<DA> o;
                    HeadOld<DA> ho;
                    head_old_from<DA>(lso, ho, dA);
                    out_forward_tangent<Act, DA>(mu, rmu);
                    gaussian_head<DA>(hin, ho, mu, a, mo, adv, A.obj_kind, A.clip_eps, o, dA);
                    hvp_signal<DA>(hin, o, rmu, rls, A.obj_kind, kl_eff, invN, ac, dA, dmu, cmu, cls);
                    out_hvp_back<Act, DA>(mu, rmu, ac, dmu, cmu);
                    s_obj += o.obj;
                    s_kl += o.kl;
                    s_ratio += o.ratio;
                } else {
#pragma unroll
                    for (int d = 0; d < DA; ++d) dmu[d] = cmu[d] = cls[d] = 0.f;
                }
#pragma unroll
                for (int d = 0; d < DA; ++d)
                    S.DMU[rb * DA + d] = dmu[d], S.CMU[rb * DA + d] = cmu[d], S.CLS[rb * DA + d] = cls[d];
            }
        }
        __syncthreads();
        // ---- output layer (column role): out_W2 += H2^T CMU + ac * R2^T DMU ; out_b2 += colsum CMU ; out_ls += colsum CLS
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float h = S.H2[b * LD + cj], r = ac * S.R2[b * LD + cj];
#pragma unroll
                for (int d = 0; d < DA; ++d) gW2p[d] = fmaf(h, S.CMU[b * DA + d], fmaf(r, S.DMU[b * DA + d], gW2p[d]));
            }
            if (tid < DA) {
                float s1 = 0.f, s2 = 0.f;
                for (int b = 0; b < nb; ++b) s1 += S.CMU[b * DA + tid], s2 += S.CLS[b * DA + tid];
                gB2 += s1;
                gLS += s2;
            }
        }
        __syncthreads();
        // ---- D2 = dH2 * g2 -> H2 ; C2 = CdH2 * g2 + ac * dH2 * (act''/act')(H2) R2 -> R2 (g2 = act'(H2); tanh: act''/act' = -2 H2);
        //      out_b1 accumulates C2 on the fly
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            const int b = row0 + i;
            const float4 h4 = *reinterpret_cast<float4*>(S.H2 + b * LD + col0);
            const float4 r4 = *reinterpret_cast<float4*>(S.R2 + b * LD + col0);
            const float hv[4] = {h4.x, h4.y, h4.z, h4.w}, rv[4] = {r4.x, r4.y, r4.z, r4.w};
            float d2[4], c2[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float dh = 0.f, ch = 0.f;
#pragma unroll
                for (int d = 0; d < DA; ++d) {
                    const float w2 = S.P[L::W2 + (col0 + c) * DA + d], v2 = S.V[L::W2 + (col0 + c) * DA + d];
                    const float dm = S.DMU[b * DA + d];
                    dh = fmaf(dm, w2, dh);
                    ch = fmaf(S.CMU[b * DA + d], w2, fmaf(ac * dm, v2, ch));
                }
                d2[c] = dh * Act::d(hv[c]);
                c2[c] = act_hvp_back<Act>(ch, dh, hv[c], rv[c], ac);
                gB1p[c] += c2[c];
            }
            *reinterpret_cast<float4*>(S.H2 + b * LD + col0) = make_float4(d2[0], d2[1], d2[2], d2[3]);
            *reinterpret_cast<float4*>(S.R2 + b * LD + col0) = make_float4(c2[0], c2[1], c2[2], c2[3]);
        }
        __syncthreads();
        // ---- out_W1 += H1^T C2 + ac * R1^T D2
        wgrad_tile<LD, RK>(S.H1, S.R2, ty * RK, col0, nb, gW1c);
        wgrad_tile<LD, RK>(S.R1, S.H2, ty * RK, col0, nb, gW1a);
        // ---- dH1 = D2 W1^T ; CdH1 = C2 W1^T + ac * D2 V1^T
        float dh1[RM][4], ch1[RM][4];
#pragma unroll
        for (int i = 0; i < RM; ++i)
#pragma unroll
            for (int c = 0; c < 4; ++c) dh1[i][c] = ch1[i][c] = 0.f;
        gemm_tile<HID, LD, HID, RM>(S.H2, S.V1T, row0, col0, ch1);
#pragma unroll
        for (int i = 0; i < RM; ++i)
#pragma unroll
            for (int c = 0; c < 4; ++c) ch1[i][c] *= ac;
        gemm_tile<HID, LD, HID, RM>(S.R2, S.W1T, row0, col0, ch1);
        gemm_tile<HID, LD, HID, RM>(S.H2, S.W1T, row0, col0, dh1);
        __syncthreads();   // all reads of H1 / R1 by the weight-gradient loops are done
        // ---- C1 = CdH1 * g1 + ac * dH1 * (act''/act')(H1) R1 -> H1 ; out_b0 accumulates C1 on the fly
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            const float4 h4 = *reinterpret_cast<float4*>(S.H1 + (row0 + i) * LD + col0);
            const float4 r4 = *reinterpret_cast<float4*>(S.R1 + (row0 + i) * LD + col0);
            const float hv[4] = {h4.x, h4.y, h4.z, h4.w}, rv[4] = {r4.x, r4.y, r4.z, r4.w};
            float c1[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                c1[c] = act_hvp_back<Act>(ch1[i][c], dh1[i][c], hv[c], rv[c], ac);
                gB0p[c] += c1[c];
            }
            *reinterpret_cast<float4*>(S.H1 + (row0 + i) * LD + col0) = make_float4(c1[0], c1[1], c1[2], c1[3]);
        }
        __syncthreads();
        // ---- out_W0 += X^T C1 (column role)
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float c1 = S.H1[b * LD + cj];
#pragma unroll
                for (int i = 0; i < DO; ++i) gW0p[i] = fmaf(S.X[b * DOP + i], c1, gW0p[i]);
            }
        }
    }
    if (cur_m >= 0) flush(cur_m);
}

template <int DO, int DA, int HID>
__global__ void __launch_bounds__(PT_THREADS) policy_hvp_kernel(PolicyArgs A) { policy_hvp_body<DO, DA, HID, ActTanh>(A); }
template <int DO, int DA, int HID>
__global__ void __launch_bounds__(PT_THREADS) policy_hvp_relu_kernel(PolicyArgs A) { policy_hvp_body<DO, DA, HID, ActRelu>(A); }
template <int DO, int DA, int HID, class Hid>
__global__ void __launch_bounds__(PT_THREADS) policy_hvp_otanh_kernel(PolicyArgs A) { policy_hvp_body<DO, DA, HID, OutTanh<Hid>>(A); }

// -------------------------------------------------------------------------------------------------
// forward only: mean for arbitrary obs (distribution_info_sym / get_actions without sampling).  obs_dim / act_dim: the
// logical sizes, read only by the padded instantiations (IsBucket)
template <int DO, int DA, int HID, class Act>
__device__ __forceinline__ void policy_forward_body(int M, int N, const float* params, int64_t stride, const float* obs,
                                                    float* mean, int obs_dim, int act_dim) {
    using L = PLayout<DO, DA, HID>;
    constexpr bool BUCKET = IsBucket<DO, DA>::value;
    const int dO = BUCKET ? obs_dim : DO, dA = BUCKET ? act_dim : DA;
    constexpr int NU = HID / 32;
    __shared__ float sP[L::P];
    __shared__ float sh[4][HID];
    const int m = blockIdx.y, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const float* th = params + (int64_t)m * stride;
    for (int i = threadIdx.x; i < L::P; i += blockDim.x) sP[i] = __ldg(th + i);
    __syncthreads();
    for (int n = blockIdx.x * 4 + w; n < N; n += gridDim.x * 4) {
        const float* o = obs + ((int64_t)m * N + n) * dO;
#pragma unroll
        for (int u = 0; u < NU; ++u) {
            const int j = lane + 32 * u;
            float z = sP[L::B0 + j];
            for (int i = 0; i < dO; ++i) z = fmaf(__ldg(o + i), sP[L::W0 + i * HID + j], z);
            sh[w][j] = Act::f(z);
        }
        __syncwarp();
        float mu[DA];
#pragma unroll
        for (int d = 0; d < DA; ++d) mu[d] = 0.f;
#pragma unroll
        for (int u = 0; u < NU; ++u) {
            const int j = lane + 32 * u;
            float z = sP[L::B1 + j];
            for (int k = 0; k < HID; ++k) z = fmaf(sh[w][k], sP[L::W1 + k * HID + j], z);
            const float h2 = Act::f(z);
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = fmaf(h2, sP[L::W2 + j * DA + d], mu[d]);
        }
#pragma unroll
        for (int d = 0; d < DA; ++d) {
            float s = warp_sum(mu[d]) + sP[L::B2 + d];
            if constexpr (Act::OUT_TANH) s = ActTanh::f(s);
            if (lane == d && d < dA) mean[((int64_t)m * N + n) * dA + d] = s;
        }
        __syncwarp();
    }
}

template <int DO, int DA, int HID>
__global__ void __launch_bounds__(128) policy_forward_kernel(int M, int N, const float* params, int64_t stride, const float* obs,
                                                              float* mean, int obs_dim, int act_dim) {
    policy_forward_body<DO, DA, HID, ActTanh>(M, N, params, stride, obs, mean, obs_dim, act_dim);
}
template <int DO, int DA, int HID>
__global__ void __launch_bounds__(128) policy_forward_relu_kernel(int M, int N, const float* params, int64_t stride,
                                                                   const float* obs, float* mean, int obs_dim, int act_dim) {
    policy_forward_body<DO, DA, HID, ActRelu>(M, N, params, stride, obs, mean, obs_dim, act_dim);
}
template <int DO, int DA, int HID, class Hid>
__global__ void __launch_bounds__(128) policy_forward_otanh_kernel(int M, int N, const float* params, int64_t stride,
                                                                    const float* obs, float* mean, int obs_dim, int act_dim) {
    policy_forward_body<DO, DA, HID, OutTanh<Hid>>(M, N, params, stride, obs, mean, obs_dim, act_dim);
}

}  // namespace promp
#include "policy_deep.cuh"
namespace promp {

#ifndef PROMP_POLICY_EXTRA_TU
__global__ void reduce_tasks_kernel(int M, int P, const float* in, float scale, float* out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    float s = 0.f;
    for (int m = 0; m < M; ++m) s += in[(int64_t)m * P + p];
    out[p] = s * scale;
}
// out = scale * sum_m a[m] + scale * sum_m b[m]: each sum in the order of reduce_tasks_kernel, so the result equals two
// promp_reduce_tasks and an add bit for bit
__global__ void reduce_tasks2_kernel(int M, int P, const float* a, const float* b, float scale, float* out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    float sa = 0.f, sb = 0.f;
    for (int m = 0; m < M; ++m) sa += a[(int64_t)m * P + p];
    for (int m = 0; m < M; ++m) sb += b[(int64_t)m * P + p];
    out[p] = __fadd_rn(__fmul_rn(sa, scale), __fmul_rn(sb, scale));
}

__global__ void adam_tf1_kernel(int P, float* theta, const float* grad, float* mm, float* vv, int32_t* step, float lr,
                                float b1, float b2, float eps) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int t = *step + 1;
    // lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t)   (tf.train.AdamOptimizer)
    const float lr_t = lr * sqrtf(1.f - powf(b2, (float)t)) / (1.f - powf(b1, (float)t));
    if (p < P) {
        const float g = grad[p];
        const float mn = b1 * mm[p] + (1.f - b1) * g;
        const float vn = b2 * vv[p] + (1.f - b2) * g * g;
        mm[p] = mn;
        vv[p] = vn;
        theta[p] = theta[p] - lr_t * mn / (sqrtf(vn) + eps);
    }
}
__global__ void adam_step_inc_kernel(int32_t* step) { *step += 1; }

// [loss, inner_kl_0 .. inner_kl_{S-2}, outer_kl] of one meta-objective evaluation from the per-launch stats rows
// stats_all [S, M, 4] (row s < S-1: inner step s -> (surr, KL); row S-1: outer objective -> (surr, KL)):
//   loss = mean_m surr_{S-1,m} (+ mean_s coeff_s * inner_kl_s when coeff != NULL: pro_mp.py:151-155), means over M_global.
// One block, warp w reduces term w in a fixed order (deterministic).
__global__ void __launch_bounds__(256) meta_loss_terms_kernel(int S, int M, const float* __restrict__ stats_all, float inv_mg,
                                                               const float* __restrict__ coeff, int n_out, float* __restrict__ out) {
    __shared__ float terms[8];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (w < S + 1) {
        const int row = (w == 0 || w == S) ? S - 1 : w - 1;       // term 0: outer surr; 1..S-1: inner KLs; S: outer KL
        const int col = (w == 0) ? 0 : 1;
        float a = 0.f;
        for (int m = lane; m < M; m += 32) a += stats_all[((int64_t)row * M + m) * 4 + col];
        a = warp_sum(a) * inv_mg;
        if (lane == 0) terms[w] = a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float loss = terms[0];
        if (coeff && S > 1) {
            float pen = 0.f;
            for (int s = 0; s < S - 1; ++s) pen += coeff[s] * terms[1 + s];
            loss += pen / (float)(S - 1);
        }
        out[0] = loss;
        for (int i = 1; i < n_out && i < S + 1; ++i) out[i] = terms[i];
    }
}

// Logged scalars of one sampling phase as float64, straight into the vector the Trainer reads back once per iteration:
//   out[0..5] = AverageDiscountedReturn, AverageReturn, NumTrajs, StdReturn, MaxReturn, MinReturn (samplers/base.py:135-149)
//               from the per-task sums promp_process_samples left in stats [M, 8],
//   out[6]    = AveragePolicyStd = mean exp(log_std) (policies/gaussian_mlp_policy.py:118-123).
// One launch instead of ~15 reduce / elementwise / cat kernels per phase.
__global__ void __launch_bounds__(256) phase_log_terms_kernel(int M, int Da, double n_paths, const double* __restrict__ stats,
                                                               const float* __restrict__ log_std, double* __restrict__ out) {
    __shared__ double red[8][6];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    double v[6] = {0.0, 0.0, 0.0, -1e300, 1e300, 0.0};      // sum R0, sum G, sum G^2, max G, min G, sum exp(log_std)
    for (int m = tid; m < M; m += 256) {
        const double* st = stats + (int64_t)m * 8;
        v[0] += st[0]; v[1] += st[1]; v[2] += st[2];
        v[3] = fmax(v[3], st[3]);
        v[4] = fmin(v[4], st[4]);
    }
    for (int i = tid; i < M * Da; i += 256) v[5] += (double)expf(log_std[i]);
#pragma unroll
    for (int k = 0; k < 6; ++k) v[k] = k == 3 ? warp_max(v[k]) : k == 4 ? warp_min(v[k]) : warp_sum(v[k]);
    if (lane == 0)
        for (int k = 0; k < 6; ++k) red[w][k] = v[k];
    __syncthreads();
    if (tid == 0) {
        for (int i = 1; i < 8; ++i) {
            v[0] += red[i][0]; v[1] += red[i][1]; v[2] += red[i][2]; v[5] += red[i][5];
            v[3] = fmax(v[3], red[i][3]);
            v[4] = fmin(v[4], red[i][4]);
        }
        const double mean_g = v[1] / n_paths;
        out[0] = v[0] / n_paths;
        out[1] = mean_g;
        out[2] = n_paths;
        out[3] = sqrt(fmax(v[2] / n_paths - mean_g * mean_g, 0.0));
        out[4] = v[3];
        out[5] = v[4];
        out[6] = v[5] / (double)(M * Da);
    }
}

// ProMP's logged scalars (pro_mp.py:193-198) from the optimizer's device vector [loss_before, loss_after, inner KLs.., outer KL]
__global__ void promp_log_terms_kernel(int S1, const float* __restrict__ final_terms, double* __restrict__ out) {
    if (threadIdx.x == 0) {
        out[0] = (double)final_terms[0];
        out[1] = (double)final_terms[1];
        float s = 0.f;
        for (int i = 0; i < S1; ++i) s += final_terms[2 + i];
        out[2] = S1 > 0 ? (double)(s / (float)S1) : 0.0;
    }
}

// ProMP._adapt_kl_coeff (pro_mp.py:201-214) on the device: coeff_s /= 2 if KL_s < target / 1.5, *= 2 if KL_s > target * 1.5
// (comparisons in double like the reference's Python floats; halving / doubling is exact in float32).  out4 (optional):
// ProMP's four logged scalars [LossBefore, LossAfter, KLInner, KLCoeffInner (after the update)] (pro_mp.py:193-198).
__global__ void adapt_kl_coeff_kernel(int S1, const float* __restrict__ final_terms, double target, int adapt, float* __restrict__ coeff,
                                      double* __restrict__ out4) {
    if (threadIdx.x == 0) {
        if (out4) {
            out4[0] = (double)final_terms[0];
            out4[1] = (double)final_terms[1];
            float s = 0.f;
            for (int i = 0; i < S1; ++i) s += final_terms[2 + i];
            out4[2] = S1 > 0 ? (double)(s / (float)S1) : 0.0;
        }
        double* out_mean = out4 ? out4 + 3 : nullptr;
        double sum = 0.0;
        for (int i = 0; i < S1; ++i) {
            float c = coeff[i];
            if (adapt) {
                const double kl = (double)final_terms[2 + i];
                if (kl < target / 1.5) c *= 0.5f;
                else if (kl > target * 1.5) c *= 2.0f;
                coeff[i] = c;
            }
            sum += (double)c;
        }
        if (out_mean) *out_mean = S1 > 0 ? sum / (double)S1 : 0.0;
    }
}

#endif  // !PROMP_POLICY_EXTRA_TU

// -------------------------------------------------------------------------------------------------
// options of promp_set_option, defined by the tanh translation unit and read by both
#ifdef PROMP_POLICY_EXTRA_TU
#define PROMP_OPTION(name, init) extern int name
#else
#define PROMP_OPTION(name, init) int name = init
#endif
PROMP_OPTION(g_use_tc, 1);     // promp_set_option("tensor_cores", 0|1): HID = 64 policy kernels on the tensor cores, 3xTF32 (default) or CUDA cores

PROMP_OPTION(g_tc_threads, 0);  // promp_set_option("tc_threads", 0|256|512): 0 = per-shape default
// column groups of the TC kernels' thread mapping: 2 -> 256 threads (32 hidden units per thread), 4 -> 512 threads (16)
static int tc_column_groups(int obs_dim) {
    if (g_tc_threads == 256) return 2;
    if (g_tc_threads == 512) return 4;
    return obs_dim <= 4 ? 4 : 2;
}

struct TilePlan {
    int grid, q, kmax;
    int64_t partial_floats;
};
// One-wave persistent plan: `slots` resident CTAs share the T tiles as evenly as possible.
static TilePlan plan_tiles(int M, int N, int slots, int P, int tb = TB) {
    const int ntiles = (N + tb - 1) / tb;
    const int64_t T = (int64_t)M * ntiles;
    TilePlan p;
    int g = (int)(T < slots ? T : slots);
    if (g < 1) g = 1;
    p.q = (int)((T + g - 1) / g);
    p.grid = (int)((T + p.q - 1) / p.q);
    p.kmax = (p.q + ntiles - 1) / ntiles + 1;
    p.partial_floats = (int64_t)p.grid * p.kmax * (P + PSTAT);
    return p;
}
static int sm_count() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = 132;      // H100 SXM
    }
    return n;
}
static int64_t counters_bytes(int M) { return (((int64_t)M * sizeof(int) + 15) / 16) * 16; }
// Workspace of one launch over a P-parameter policy: an upper bound over the occupancies the kernels can have (1..4 CTAs per
// SM on this device's SMs, or on 160)
static int64_t policy_workspace_bytes(int M, int N, int P) {
    int64_t worst = 0;
    for (int occ = 1; occ <= 4; ++occ)
        for (int tb : {TB, TBT}) {            // CUDA-core kernels tile by 64 samples, the tensor-core kernels by 128
            const TilePlan p = plan_tiles(M, N, 160 * occ, P, tb);
            if (p.partial_floats > worst) worst = p.partial_floats;
            const TilePlan p2 = plan_tiles(M, N, sm_count() * occ, P, tb);
            if (p2.partial_floats > worst) worst = p2.partial_floats;
        }
    return counters_bytes(M) + worst * (int64_t)sizeof(float) + 16;
}

// One persistent launch over tb-sample tiles; `extra`: the kernel's arguments after A (nh for the kernels of policy_deep.cuh)
template <typename Kernel, typename... Extra>
static int launch_policy(Kernel kernel, int smem, int& occ_cache, PolicyArgs& A, int P, void* ws, int64_t ws_bytes,
                         cudaStream_t st, const char* name, int tb, int threads, Extra... extra) {
    if (occ_cache == 0) {
        PROMP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        int occ = 0;
        PROMP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem));
        occ_cache = occ < 1 ? 1 : occ;
    }
    const TilePlan p = plan_tiles(A.M, A.N, sm_count() * occ_cache, P, tb);
    const int64_t need = counters_bytes(A.M) + p.partial_floats * (int64_t)sizeof(float);
    if (ws_bytes < need) {
        set_error("policy workspace too small (%lld < %lld bytes)", (long long)ws_bytes, (long long)need);
        return PROMP_ERR_WORKSPACE;
    }
    A.counters = (int*)ws;
    A.partial = (float*)((char*)ws + counters_bytes(A.M));
    A.q = p.q;
    A.kmax = p.kmax;
    kernel<<<p.grid, threads, smem, st>>>(A, extra...);
    PROMP_LAUNCH_CHECK(name);
    return PROMP_OK;
}

// The kernel of each family for activation Act: policy_*_kernel (tanh) or policy_*_relu_kernel (ReLU).  `if constexpr`
// names only the selected one, so a tanh launcher instantiates exactly the kernels it did before ReLU existed.
template <class Act>
constexpr bool is_relu() { return std::is_same<Act, ActRelu>::value; }
// A tanh output layer selects policy_*_otanh_kernel<..., hidden activation>.
#define PROMP_ACT_KERNEL(Act, NAME, ...)                                                               \
    [] {                                                                                               \
        if constexpr (Act::OUT_TANH) return NAME##_otanh_kernel<__VA_ARGS__, typename Act::Hidden>;    \
        else if constexpr (is_relu<Act>()) return NAME##_relu_kernel<__VA_ARGS__>;                     \
        else return NAME##_kernel<__VA_ARGS__>;                                                        \
    }()

// nh = the number of hidden-to-hidden layers (depth - 1).  Two hidden layers run the tensor-core kernels (hidden 64) or the
// two-layer CUDA-core kernels above; one and three run the depth-generic CUDA-core kernels of policy_deep.cuh.
template <int DO, int DA, int HID, class Act>
static int launch_grad(PolicyArgs& A, int nh, void* ws, int64_t ws_bytes, cudaStream_t st) {
    if (nh != 1) {
        const int P = DeepLayout<DO, DA, HID>{nh}.P();
        constexpr int smem = (int)sizeof(DeepGradSmem<DO, DA, HID>);
        if (A.adv_per_task) {
            static int occ_x = 0;
            return launch_policy(policy_grad_deep_kernel<DO, DA, HID, Act, ADV_TASK>, smem, occ_x, A, P, ws, ws_bytes, st,
                                 "policy_grad_deep_kernel", TB, PT_THREADS, nh);
        }
        static int occ = 0;
        return launch_policy(policy_grad_deep_kernel<DO, DA, HID, Act, ADV_SAMPLE>, smem, occ, A, P, ws, ws_bytes, st,
                             "policy_grad_deep_kernel", TB, PT_THREADS, nh);
    }
    if (A.adv_per_task) {
        static int occ_x = 0;
        constexpr auto kx = PROMP_ACT_KERNEL(Act, policy_grad_explore, DO, DA, HID);
        return launch_policy(kx, (int)sizeof(GradSmem<DO, DA, HID>), occ_x, A, PLayout<DO, DA, HID>::P, ws, ws_bytes, st,
                             "policy_grad_explore_kernel", TB, PT_THREADS);
    }
    static int occ = 0;
    constexpr auto kernel = PROMP_ACT_KERNEL(Act, policy_grad, DO, DA, HID);
    return launch_policy(kernel, (int)sizeof(GradSmem<DO, DA, HID>), occ, A, PLayout<DO, DA, HID>::P, ws, ws_bytes, st,
                         "policy_grad_kernel", TB, PT_THREADS);
}

template <int DO, int DA, int HID, class Act>
static int launch_grad_any(PolicyArgs& A, int nh, void* ws, int64_t ws_bytes, cudaStream_t st) {
    if constexpr (HID == TC_HID) {
        if (g_use_tc && nh == 1 && A.adv_per_task) {
            static int occ2 = 0, occ4 = 0;
            constexpr auto k4 = PROMP_ACT_KERNEL(Act, policy_grad_tc_explore, DO, DA, 4);
            constexpr auto k2 = PROMP_ACT_KERNEL(Act, policy_grad_tc_explore, DO, DA, 2);
            if (tc_column_groups(DO) == 4)
                return launch_policy(k4, (int)sizeof(GradTcSmem<DO, DA, 4>), occ4, A,
                                     PLayout<DO, DA, HID>::P, ws, ws_bytes, st, "policy_grad_tc_explore_kernel", TBT, 512);
            return launch_policy(k2, (int)sizeof(GradTcSmem<DO, DA, 2>), occ2, A,
                                 PLayout<DO, DA, HID>::P, ws, ws_bytes, st, "policy_grad_tc_explore_kernel", TBT, 256);
        }
        if (g_use_tc && nh == 1) {
            static int occ2 = 0, occ4 = 0;
            constexpr auto k4 = PROMP_ACT_KERNEL(Act, policy_grad_tc, DO, DA, 4);
            constexpr auto k2 = PROMP_ACT_KERNEL(Act, policy_grad_tc, DO, DA, 2);
            if (tc_column_groups(DO) == 4)
                return launch_policy(k4, (int)sizeof(GradTcSmem<DO, DA, 4>), occ4, A,
                                     PLayout<DO, DA, HID>::P, ws, ws_bytes, st, "policy_grad_tc_kernel", TBT, 512);
            return launch_policy(k2, (int)sizeof(GradTcSmem<DO, DA, 2>), occ2, A,
                                 PLayout<DO, DA, HID>::P, ws, ws_bytes, st, "policy_grad_tc_kernel", TBT, 256);
        }
    }
    return launch_grad<DO, DA, HID, Act>(A, nh, ws, ws_bytes, st);
}

template <int DO, int DA, int HID, class Act>
static int launch_hvp(PolicyArgs& A, int nh, void* ws, int64_t ws_bytes, cudaStream_t st) {
    if (nh != 1) {
        static_assert(sizeof(DeepHvpSmem<DO, DA, HID>) <= 227 * 1024, "deep HVP tile exceeds the shared memory of one SM");
        static int occ = 0;
        return launch_policy(policy_hvp_deep_kernel<DO, DA, HID, Act>, (int)sizeof(DeepHvpSmem<DO, DA, HID>), occ, A,
                             DeepLayout<DO, DA, HID>{nh}.P(), ws, ws_bytes, st, "policy_hvp_deep_kernel", TB, PT_THREADS, nh);
    }
    if constexpr (HID == TC_HID && sizeof(HvpTcSmem<DO, DA, 2>) <= 227 * 1024) {     // fits the 227 KB of one SM
        if (g_use_tc) {
            static int occ2 = 0, occ4 = 0;
            constexpr auto k4 = PROMP_ACT_KERNEL(Act, policy_hvp_tc, DO, DA, 4);
            constexpr auto k2 = PROMP_ACT_KERNEL(Act, policy_hvp_tc, DO, DA, 2);
            if (tc_column_groups(DO) == 4)
                return launch_policy(k4, (int)sizeof(HvpTcSmem<DO, DA, 4>), occ4, A,
                                     PLayout<DO, DA, HID>::P, ws, ws_bytes, st, "policy_hvp_tc_kernel", TBT, 512);
            return launch_policy(k2, (int)sizeof(HvpTcSmem<DO, DA, 2>), occ2, A,
                                 PLayout<DO, DA, HID>::P, ws, ws_bytes, st, "policy_hvp_tc_kernel", TBT, 256);
        }
    }
    static int occ = 0;
    constexpr auto kernel = PROMP_ACT_KERNEL(Act, policy_hvp, DO, DA, HID);
    return launch_policy(kernel, (int)sizeof(HvpSmem<DO, DA, HID>), occ, A, PLayout<DO, DA, HID>::P, ws, ws_bytes, st,
                         "policy_hvp_kernel", TB, PT_THREADS);
}

// ---- dataflow chain (policy_chain_tc_kernel): work-item plan + launch ---------------------------------------------
PROMP_OPTION(g_chain, -1);         // promp_set_option("chain", -1|0|1): dataflow kernel always (1), never (0: one launch per stage),
                                   // or where it wins (-1, default; see chain_uses_dataflow)
PROMP_OPTION(g_chain_q, 0);        // promp_set_option("chain_q", q): tiles per work item (0 = automatic)
PROMP_OPTION(g_chain_taper, 1);    // promp_set_option("chain_taper", 0|1): last stage's items shrink to one tile towards the end

struct ChainPlan {
    ChainStageInfo info[CHAIN_MAX_STAGES];
    int n_items;
    int64_t ctrl_bytes, bytes;     // control words (zero on entry, left zero); whole workspace
};
static int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }
// Control words at the start of a chain workspace, the same whatever n_stages is (chains of different length share one
// workspace, and the words must stay zero between calls): work queue and finished-CTA count (4 ints), ready flags and
// arrival counters of the dataflow kernel ([CHAIN_MAX_STAGES][M] each), then, ending at chain_ctrl_bytes(M), the arrival
// counters of the one-launch-per-stage path.  Both paths put their partial slots after chain_ctrl_bytes(M), so neither
// writes scratch over the other's counters.
static int64_t chain_ctrl_bytes(int M) {
    return align_up(16 + (int64_t)2 * CHAIN_MAX_STAGES * M * sizeof(int) + counters_bytes(M), 128);
}
// Items are (stage, task, q consecutive tiles).  q = the largest of 4, 2, 1 that still gives every stage at least one item
// per SM; the last stage (nothing left to fill its tail with) uses q, q/2 and 1 on the first half, third quarter and last
// quarter of its tasks, so the final imbalance over the SMs is one tile.
static ChainPlan plan_chain(int n_stages, const int* kinds, const int* Ns, int M, int P) {
    ChainPlan pl;
    memset(&pl, 0, sizeof(pl));
    const int sms = sm_count();
    int base = 0;
    for (int s = 0; s < n_stages; ++s) {
        ChainStageInfo& I = pl.info[s];
        I.kind = kinds[s];
        I.ntiles = (Ns[s] + TBT - 1) / TBT;
        int q = 4;
        if (g_chain_q > 0) q = g_chain_q;
        else while (q > 1 && (int64_t)M * ((I.ntiles + q - 1) / q) < sms) q >>= 1;
        if (q > I.ntiles) q = I.ntiles;
        I.item_base = base;
        const bool taper = g_chain_taper && s == n_stages - 1 && q > 1 && M >= 4;
        if (!taper) {
            I.n_regions = 1;
            I.reg_m0[0] = 0, I.reg_m0[1] = M;
            I.reg_q[0] = q;
            I.reg_item0[0] = 0;
            I.n_items = M * ((I.ntiles + q - 1) / q);
        } else {
            const int q2 = q > 2 ? q / 2 : q;              // q = 2: three quarters at 2, the last quarter at 1
            const int mB = M - M / 4, mA = q2 < q ? M / 2 : mB;
            I.n_regions = 0;
            int items = 0;
            const int m0[4] = {0, mA, mB, M}, qs[3] = {q, q2, 1};
            for (int r = 0; r < 3; ++r) {
                if (m0[r + 1] <= m0[r]) continue;
                I.reg_m0[I.n_regions] = m0[r];
                I.reg_q[I.n_regions] = qs[r];
                I.reg_item0[I.n_regions] = items;
                items += (m0[r + 1] - m0[r]) * ((I.ntiles + qs[r] - 1) / qs[r]);
                ++I.n_regions;
            }
            I.reg_m0[I.n_regions] = M;
            I.n_items = items;
        }
        base += I.n_items;
    }
    pl.n_items = base;
    pl.ctrl_bytes = chain_ctrl_bytes(M);
    pl.bytes = pl.ctrl_bytes + (int64_t)pl.n_items * (P + PSTAT) * sizeof(float);
    return pl;
}

// the automatic choice: dataflow kernel for chains whose stages have one to three tiles per SM (where launch tails and the
// tile quantisation of every single launch dominate: measured wins of 2-10 %, profiles/r02_chain_time.txt), one launch per stage
// below (a stage is not even one wave: nothing to balance) and above (per-item flushes outweigh the gain)
static bool chain_uses_dataflow(const ChainPlan& pl, int n_stages, int M) {
    bool fits = true;
    for (int s = 0; s < n_stages; ++s) {
        const int64_t T = (int64_t)M * pl.info[s].ntiles;
        fits = fits && T >= sm_count() && T <= 3 * sm_count();
    }
    return g_use_tc && (g_chain == 1 || (g_chain < 0 && fits));
}

template <int DO, int DA, int HID>
static constexpr bool chain_tc_ok() {
    if constexpr (HID == TC_HID) return ChainSmem<DO, DA, 2>::SIZE <= 227 * 1024 && ChainSmem<DO, DA, 4>::SIZE <= 227 * 1024;
    return false;
}

template <int DO, int DA, int NQ, bool HAS_HVP, class Act, int ADV = ADV_SAMPLE>
static int launch_chain_nq(ChainArgs& C, cudaStream_t st) {
    static int configured = 0;
    constexpr int smem = ChainSmem<DO, DA, NQ>::SIZE;
    static_assert(std::is_same<Act, ChainAct>::value, "the chain kernel of this translation unit");
    constexpr auto kernel = PROMP_CHAIN_KERNEL<DO, DA, NQ, HAS_HVP, ADV>;
    if (!configured) {
        PROMP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = 1;
    }
    int grid = sm_count();
    if (grid > C.n_items) grid = C.n_items;
    kernel<<<grid, 128 * NQ, smem, st>>>(C);
    PROMP_LAUNCH_CHECK("policy_chain_tc_kernel");
    return PROMP_OK;
}

// kinds / Ns / A: the stages in order.  Falls back to one launch per stage (same results up to summation order) for the
// shapes and depths the tensor-core kernels do not cover (the dataflow kernel is built for two hidden layers) or when the
// "chain" option is off.
template <int DO, int DA, int HID, class Act>
static int launch_chain(int n_stages, const int* kinds, PolicyArgs* A, int nh, const int* skip_flag, const float* skip_theta,
                        void* ws, int64_t ws_bytes, cudaStream_t st) {
    int Ns[CHAIN_MAX_STAGES];
    for (int s = 0; s < n_stages; ++s) Ns[s] = A[s].N;
    const int M = A[0].M;
    const ChainPlan pl = plan_chain(n_stages, kinds, Ns, M, DeepLayout<DO, DA, HID>{nh}.P());
    if constexpr (chain_tc_ok<DO, DA, HID>()) {
        if (nh == 1 && chain_uses_dataflow(pl, n_stages, M)) {
            if (ws_bytes < pl.bytes) {
                set_error("policy chain workspace too small (%lld < %lld bytes)", (long long)ws_bytes, (long long)pl.bytes);
                return PROMP_ERR_WORKSPACE;
            }
            ChainArgs C;
            memset(&C, 0, sizeof(C));
            C.n_stages = n_stages, C.n_items = pl.n_items, C.M = M;
            C.ctrl = (int*)ws;
            C.ready = (int*)ws + 4;
            C.skip_flag = skip_flag, C.skip_theta = skip_theta;
            float* partial = (float*)((char*)ws + pl.ctrl_bytes);
            for (int s = 0; s < n_stages; ++s) {
                C.info[s] = pl.info[s];
                C.st[s] = A[s];
                C.st[s].counters = (int*)ws + 4 + (CHAIN_MAX_STAGES + s) * M;
                C.st[s].partial = partial;            // slots are numbered by global item id
            }
            bool has_hvp = false, has_explore = false;
            for (int s = 0; s < n_stages; ++s) has_hvp = has_hvp || kinds[s] == 1, has_explore = has_explore || A[s].adv_per_task;
            if (has_explore)      // one instantiation per shape: HAS_HVP = true runs chains without HVP stages as well
                return tc_column_groups(DO) == 4 ? launch_chain_nq<DO, DA, 4, true, Act, ADV_EITHER>(C, st)
                                                 : launch_chain_nq<DO, DA, 2, true, Act, ADV_EITHER>(C, st);
            if (tc_column_groups(DO) == 4)
                return has_hvp ? launch_chain_nq<DO, DA, 4, true, Act>(C, st) : launch_chain_nq<DO, DA, 4, false, Act>(C, st);
            return has_hvp ? launch_chain_nq<DO, DA, 2, true, Act>(C, st) : launch_chain_nq<DO, DA, 2, false, Act>(C, st);
        }
    }
    // one launch per stage: launch_policy's (counters, partial slots) workspace starts at the last control words, so its
    // partial slots start at pl.ctrl_bytes
    const int64_t off1 = pl.ctrl_bytes - counters_bytes(M);
    void* ws1 = (char*)ws + off1;
    const int64_t ws1_bytes = ws_bytes - off1;
    for (int s = 0; s < n_stages; ++s) {
        PolicyArgs a = A[s];
        if (s == 0) a.skip_flag = skip_flag, a.skip_theta = skip_theta;
        const int rc = kinds[s] == 0 ? launch_grad_any<DO, DA, HID, Act>(a, nh, ws1, ws1_bytes, st)
                                     : launch_hvp<DO, DA, HID, Act>(a, nh, ws1, ws1_bytes, st);
        if (rc != PROMP_OK) return rc;
    }
    return PROMP_OK;
}

// the activation does not change the plan: `Act` only keeps the dispatch uniform
template <int DO, int DA, int HID, class Act>
static int chain_num_launches(int n_stages, const int* kinds, const int* Ns, int M, int nh) {
    if constexpr (chain_tc_ok<DO, DA, HID>()) {
        const ChainPlan pl = plan_chain(n_stages, kinds, Ns, M, DeepLayout<DO, DA, HID>{nh}.P());
        if (nh == 1 && chain_uses_dataflow(pl, n_stages, M)) return 1;
    }
    return n_stages;
}

// The control words, then the workspace of the largest stand-alone launch; two hidden layers also reserve the dataflow
// kernel's partial slots
template <int DO, int DA, int HID, class Act>
static int64_t chain_ws_bytes(int n_stages, const int* kinds, const int* Ns, int M, int nh) {
    const int P = DeepLayout<DO, DA, HID>{nh}.P();
    const ChainPlan pl = plan_chain(n_stages, kinds, Ns, M, P);
    int nmax = 1;
    for (int s = 0; s < n_stages; ++s) nmax = Ns[s] > nmax ? Ns[s] : nmax;
    const int64_t single = pl.ctrl_bytes + policy_workspace_bytes(M, nmax, P);
    return nh == 1 && pl.bytes > single ? pl.bytes : single;
}

template <int DO, int DA, int HID, class Act>
static int launch_forward(int M, int N, const float* params, int64_t stride, const float* obs, float* mean, int obs_dim,
                          int act_dim, int nh, cudaStream_t st) {
    int gx = (N + 3) / 4;
    const int cap = (4 * sm_count() + M - 1) / M;
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    if (nh != 1) {
        policy_forward_deep_kernel<DO, DA, HID, Act><<<dim3(gx, M), 128, 0, st>>>(M, N, params, stride, obs, mean, obs_dim,
                                                                                   act_dim, nh);
        PROMP_LAUNCH_CHECK("policy_forward_deep_kernel");
        return PROMP_OK;
    }
    constexpr auto kernel = PROMP_ACT_KERNEL(Act, policy_forward, DO, DA, HID);
    kernel<<<dim3(gx, M), 128, 0, st>>>(M, N, params, stride, obs, mean, obs_dim, act_dim);
    PROMP_LAUNCH_CHECK("policy_forward_kernel");
    return PROMP_OK;
}

// the instantiation for this translation unit's activation; hid_ = the width decoded from `hidden`
#define PROMP_DISPATCH_ACT(FN, DO, DA, HID, ...) return FN<DO, DA, HID, PROMP_POLICY_ACT>(__VA_ARGS__);

// supported (obs_dim, act_dim, hidden) instantiations
#define PROMP_DISPATCH_DIMS(FN, ...)                                                                     \
    if (obs_dim == 2 && act_dim == 2 && hid_ == 64) PROMP_DISPATCH_ACT(FN, 2, 2, 64, __VA_ARGS__)         \
    if (obs_dim == 2 && act_dim == 2 && hid_ == 32) PROMP_DISPATCH_ACT(FN, 2, 2, 32, __VA_ARGS__)         \
    if (obs_dim == 17 && act_dim == 6 && hid_ == 64) PROMP_DISPATCH_ACT(FN, 17, 6, 64, __VA_ARGS__)       \
    if (obs_dim == 17 && act_dim == 6 && hid_ == 32) PROMP_DISPATCH_ACT(FN, 17, 6, 32, __VA_ARGS__)       \
    if (obs_dim == 4 && act_dim == 2 && hid_ == 64) PROMP_DISPATCH_ACT(FN, 4, 2, 64, __VA_ARGS__)         \
    if (obs_dim == 4 && act_dim == 2 && hid_ == 32) PROMP_DISPATCH_ACT(FN, 4, 2, 32, __VA_ARGS__)         \
    set_error("unsupported (obs_dim, act_dim, hidden) = (%d, %d, %d); built: (2,2,{32,64}), (4,2,{32,64}), (17,6,{32,64})", \
              obs_dim, act_dim, hidden);                                                                 \
    return PROMP_ERR_INVALID_ARG;

// the padded (bucket) instantiations, at the caps promp_policy_layout gives (obs, act, hidden)
#define PROMP_DISPATCH_BUCKETS(FN, ...)                                                                      \
    {                                                                                                        \
        int32_t lay_[4];                                                                                     \
        if (promp_policy_layout(obs_dim, act_dim, hidden, lay_) != PROMP_OK) return PROMP_ERR_INVALID_ARG;  \
        if (lay_[0] == 8 && lay_[1] == 2 && hid_ == 64) PROMP_DISPATCH_ACT(FN, 8, 2, 64, __VA_ARGS__)       \
        if (lay_[0] == 8 && lay_[1] == 2 && hid_ == 32) PROMP_DISPATCH_ACT(FN, 8, 2, 32, __VA_ARGS__)       \
        if (lay_[0] == 8 && lay_[1] == 8 && hid_ == 64) PROMP_DISPATCH_ACT(FN, 8, 8, 64, __VA_ARGS__)       \
        if (lay_[0] == 8 && lay_[1] == 8 && hid_ == 32) PROMP_DISPATCH_ACT(FN, 8, 8, 32, __VA_ARGS__)       \
        if (lay_[0] == 20 && lay_[1] == 2 && hid_ == 64) PROMP_DISPATCH_ACT(FN, 20, 2, 64, __VA_ARGS__)     \
        if (lay_[0] == 20 && lay_[1] == 2 && hid_ == 32) PROMP_DISPATCH_ACT(FN, 20, 2, 32, __VA_ARGS__)     \
        if (lay_[0] == 20 && lay_[1] == 8 && hid_ == 64) PROMP_DISPATCH_ACT(FN, 20, 8, 64, __VA_ARGS__)     \
        if (lay_[0] == 20 && lay_[1] == 8 && hid_ == 32) PROMP_DISPATCH_ACT(FN, 20, 8, 32, __VA_ARGS__)     \
        set_error("no padded instantiation for caps (%d, %d, %d)", lay_[0], lay_[1], hid_);                 \
        return PROMP_ERR_INVALID_ARG;                                                                        \
    }

// The (obs, act, hidden) dispatch of every entry point for this translation unit's activation: tanh_tu:: here, relu_tu:: in
// policy_relu.cu, otanh_tu:: and relu_otanh_tu:: in the tanh-output units.  `hidden` has been checked by decode_hidden;
// padded = the bucket table of the *_padded entry points.
namespace PROMP_ACT_NS {
#define PROMP_DISPATCH(FN, ...)                                                  \
    const int hid_ = hidden & PROMP_HIDDEN_WIDTH_MASK;                          \
    if (padded) PROMP_DISPATCH_BUCKETS(FN, __VA_ARGS__)                          \
    PROMP_DISPATCH_DIMS(FN, __VA_ARGS__)
int grad(bool padded, int obs_dim, int act_dim, int hidden, int nh, PolicyArgs& A, void* ws, int64_t ws_bytes, cudaStream_t s) {
    PROMP_DISPATCH(launch_grad_any, A, nh, ws, ws_bytes, s)
}
int hvp(bool padded, int obs_dim, int act_dim, int hidden, int nh, PolicyArgs& A, void* ws, int64_t ws_bytes, cudaStream_t s) {
    PROMP_DISPATCH(launch_hvp, A, nh, ws, ws_bytes, s)
}
int64_t chain_workspace_bytes(bool padded, int obs_dim, int act_dim, int hidden, int nh, int n_stages, const int* kinds,
                              const int* Ns, int M) {
    PROMP_DISPATCH(chain_ws_bytes, n_stages, kinds, Ns, M, nh)
}
int chain_launches(bool padded, int obs_dim, int act_dim, int hidden, int nh, int n_stages, const int* kinds, const int* Ns,
                   int M) {
    PROMP_DISPATCH(chain_num_launches, n_stages, kinds, Ns, M, nh)
}
int chain(bool padded, int obs_dim, int act_dim, int hidden, int nh, int n_stages, const int* kinds, PolicyArgs* A,
          const int* skip_flag, const float* skip_theta, void* ws, int64_t ws_bytes, cudaStream_t s) {
    PROMP_DISPATCH(launch_chain, n_stages, kinds, A, nh, skip_flag, skip_theta, ws, ws_bytes, s)
}
int forward(bool padded, int obs_dim, int act_dim, int hidden, int nh, int M, int N, const float* params, int64_t stride,
            const float* obs, float* mean, cudaStream_t s) {
    PROMP_DISPATCH(launch_forward, M, N, params, stride, obs, mean, obs_dim, act_dim, nh, s)
}
}  // namespace PROMP_ACT_NS

#ifndef PROMP_POLICY_EXTRA_TU
// the dispatch of the other units: relu_tu (policy_relu.cu), otanh_tu (policy_otanh.cu), relu_otanh_tu (policy_relu_otanh.cu)
#define PROMP_DECLARE_UNIT(NS)                                                                                                    \
    namespace NS {                                                                                                                \
    int grad(bool padded, int obs_dim, int act_dim, int hidden, int nh, PolicyArgs& A, void* ws, int64_t ws_bytes, cudaStream_t s);\
    int hvp(bool padded, int obs_dim, int act_dim, int hidden, int nh, PolicyArgs& A, void* ws, int64_t ws_bytes, cudaStream_t s); \
    int64_t chain_workspace_bytes(bool padded, int obs_dim, int act_dim, int hidden, int nh, int n_stages, const int* kinds,      \
                                  const int* Ns, int M);                                                                          \
    int chain_launches(bool padded, int obs_dim, int act_dim, int hidden, int nh, int n_stages, const int* kinds, const int* Ns,  \
                       int M);                                                                                                    \
    int chain(bool padded, int obs_dim, int act_dim, int hidden, int nh, int n_stages, const int* kinds, PolicyArgs* A,           \
              const int* skip_flag, const float* skip_theta, void* ws, int64_t ws_bytes, cudaStream_t s);                         \
    int forward(bool padded, int obs_dim, int act_dim, int hidden, int nh, int M, int N, const float* params, int64_t stride,     \
                const float* obs, float* mean, cudaStream_t s);                                                                   \
    }
PROMP_DECLARE_UNIT(relu_tu)
PROMP_DECLARE_UNIT(otanh_tu)
PROMP_DECLARE_UNIT(relu_otanh_tu)
#endif

// checks `hidden` (decode_hidden) and decodes its activations; returns from the caller on bad bits
#define PROMP_DECODE_HIDDEN(who)                                                                 \
    int hid_ = 0, depth_ = 2;                                                                    \
    bool relu_ = false, otanh_ = false;                                                          \
    if (decode_hidden(who, hidden, hid_, relu_, otanh_, depth_) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
// dispatch function FN of the unit that holds the decoded activations' kernels
#define PROMP_UNIT(FN) (otanh_ ? (relu_ ? relu_otanh_tu::FN : otanh_tu::FN) : (relu_ ? relu_tu::FN : tanh_tu::FN))

}  // namespace promp

#ifndef PROMP_POLICY_EXTRA_TU

using namespace promp;

extern "C" int64_t promp_policy_workspace_bytes(int M, int N, int obs_dim, int act_dim, int hidden) {
    return policy_workspace_bytes(M, N, promp_num_params(obs_dim, act_dim, hidden));
}

extern "C" int promp_policy_layout(int obs_dim, int act_dim, int hidden, int32_t out[4]) {
    PROMP_REQUIRE(out != nullptr, "promp_policy_layout: null output");
    int width, depth;    // the activations do not change the layout; the depth does
    bool relu, out_tanh;
    if (decode_hidden("promp_policy_layout", hidden, width, relu, out_tanh, depth) != PROMP_OK) return PROMP_ERR_INVALID_ARG;
    hidden = width;
    PROMP_REQUIRE(obs_dim >= 1 && obs_dim <= 19 && act_dim >= 1 && act_dim <= 8 && (hidden == 32 || hidden == 64),
                  "promp_policy_layout: padded policy kernels take obs_dim in [1, 19], act_dim in [1, 8] and hidden 32 or 64 "
                  "(got %d, %d, %d)", obs_dim, act_dim, hidden);
    out[0] = obs_dim <= 8 ? 8 : 20;
    out[1] = act_dim <= 2 ? 2 : 8;
    out[2] = hidden;
    out[3] = promp::num_params(out[0], out[1], hidden, depth);
    return PROMP_OK;
}

extern "C" int64_t promp_policy_workspace_bytes_padded(int M, int N, int obs_dim, int act_dim, int hidden) {
    int32_t lay[4];
    if (promp_policy_layout(obs_dim, act_dim, hidden, lay) != PROMP_OK) return -1;
    return promp_policy_workspace_bytes(M, N, lay[0], lay[1], hidden);
}

static int check_policy_args(const char* who, int M, int N, const void* params, const void* obs, const void* act,
                             const void* adv, const void* old_mean, const void* old_ls, const void* ws) {
    PROMP_REQUIRE(M > 0 && N > 0, "%s: M and N must be positive (got %d, %d)", who, M, N);
        PROMP_REQUIRE(params && obs && act && adv && old_mean && old_ls && ws, "%s: null pointer argument", who);
    return PROMP_OK;
}

// PROMP_OBJ_EXPLORE is the LOGLIK objective with the per-task weight adv[m]: the kernels see obj_kind LOGLIK and adv_per_task
static void explore_args(PolicyArgs& A) {
    if (A.obj_kind != PROMP_OBJ_EXPLORE) return;
    A.obj_kind = PROMP_OBJ_LOGLIK;
    A.adv_per_task = 1;
}

// padded: the bucket instantiations (promp_*_padded entry points), else the exact table
static int policy_grad_impl(bool padded, int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid,
                            const float* params, int64_t param_stride, const float* obs, const float* act,
                            const float* adv, const float* old_mean, const float* old_log_std, int ls_per_sample,
                            int obj_kind, float obj_scale, float clip_eps, float kl_coeff, int clip_log_std,
                            float min_log_std, float* grad, float* out_params, float sgd_lr, float* stats,
                            const int32_t* skip_flag, const float* skip_theta, int32_t* unclipped_out, float* theta_copy_out,
                            void* workspace, int64_t workspace_bytes, void* stream) {
    int st = check_policy_args(n_valid ? "promp_policy_grad_ragged" : "promp_policy_grad", M, N, params, obs, act, adv, old_mean, old_log_std, workspace);
    if (st != PROMP_OK) return st;
    PROMP_REQUIRE(obj_kind >= 0 && obj_kind <= PROMP_OBJ_EXPLORE, "promp_policy_grad: bad obj_kind %d", obj_kind);
    PROMP_REQUIRE(!(out_params && !grad), "promp_policy_grad: out_params needs grad");
    PROMP_REQUIRE((skip_flag == nullptr) == (skip_theta == nullptr) && (unclipped_out == nullptr) == (theta_copy_out == nullptr),
                  "promp_policy_grad_ex: skip_flag / skip_theta and unclipped_out / theta_copy_out come in pairs");
    PROMP_REQUIRE(!(skip_flag || unclipped_out) || param_stride == 0,
                  "promp_policy_grad_ex: launch re-use is defined for the shared pre-update parameters (param_stride 0)");
    PolicyArgs A{};
    A.M = M; A.N = N; A.params = params; A.param_stride = param_stride;
    A.obs = obs; A.act = act; A.adv = adv; A.old_mean = old_mean; A.old_ls = old_log_std;
    A.ls_per_sample = ls_per_sample; A.obj_kind = obj_kind; A.obj_scale = obj_scale; A.clip_eps = clip_eps;
    A.kl_coeff = kl_coeff; A.clip_log_std = clip_log_std; A.min_log_std = min_log_std;
    A.grad = grad; A.out_params = out_params; A.sgd_lr = sgd_lr; A.stats = stats; A.n_valid = n_valid;
    A.skip_flag = skip_flag; A.skip_theta = skip_theta; A.unclipped_out = unclipped_out; A.theta_copy_out = theta_copy_out;
    A.obs_dim = obs_dim; A.act_dim = act_dim;
    explore_args(A);
    cudaStream_t s = (cudaStream_t)stream;
    PROMP_DECODE_HIDDEN("promp_policy_grad")
    return PROMP_UNIT(grad)(padded, obs_dim, act_dim, hidden, depth_ - 1, A, workspace, workspace_bytes, s);
}

#define PROMP_GRAD_EX_PARAMS                                                                                               \
    int obs_dim, int act_dim, int hidden, int M, int N, const int32_t *n_valid, const float *params, int64_t param_stride, \
        const float *obs, const float *act, const float *adv, const float *old_mean, const float *old_log_std,             \
        int ls_per_sample, int obj_kind, float obj_scale, float clip_eps, float kl_coeff, int clip_log_std,                \
        float min_log_std, float *grad, float *out_params, float sgd_lr, float *stats, const int32_t *skip_flag,           \
        const float *skip_theta, int32_t *unclipped_out, float *theta_copy_out, void *workspace, int64_t workspace_bytes,  \
        void *stream
#define PROMP_GRAD_EX_ARGS                                                                                                 \
    obs_dim, act_dim, hidden, M, N, n_valid, params, param_stride, obs, act, adv, old_mean, old_log_std, ls_per_sample,    \
        obj_kind, obj_scale, clip_eps, kl_coeff, clip_log_std, min_log_std, grad, out_params, sgd_lr, stats, skip_flag,    \
        skip_theta, unclipped_out, theta_copy_out, workspace, workspace_bytes, stream
extern "C" int promp_policy_grad_ex(PROMP_GRAD_EX_PARAMS) { return policy_grad_impl(false, PROMP_GRAD_EX_ARGS); }
extern "C" int promp_policy_grad_ex_padded(PROMP_GRAD_EX_PARAMS) { return policy_grad_impl(true, PROMP_GRAD_EX_ARGS); }

extern "C" int promp_policy_grad_ragged(int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid,
                                        const float* params, int64_t param_stride, const float* obs, const float* act,
                                        const float* adv, const float* old_mean, const float* old_log_std, int ls_per_sample,
                                        int obj_kind, float obj_scale, float clip_eps, float kl_coeff, int clip_log_std,
                                        float min_log_std, float* grad, float* out_params, float sgd_lr, float* stats,
                                        void* workspace, int64_t workspace_bytes, void* stream) {
    return promp_policy_grad_ex(obs_dim, act_dim, hidden, M, N, n_valid, params, param_stride, obs, act, adv, old_mean, old_log_std,
                                ls_per_sample, obj_kind, obj_scale, clip_eps, kl_coeff, clip_log_std, min_log_std, grad, out_params,
                                sgd_lr, stats, nullptr, nullptr, nullptr, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int promp_policy_grad(int obs_dim, int act_dim, int hidden, int M, int N, const float* params,
                                 int64_t param_stride, const float* obs, const float* act, const float* adv,
                                 const float* old_mean, const float* old_log_std, int ls_per_sample, int obj_kind,
                                 float obj_scale, float clip_eps, float kl_coeff, int clip_log_std, float min_log_std,
                                 float* grad, float* out_params, float sgd_lr, float* stats, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
    return promp_policy_grad_ragged(obs_dim, act_dim, hidden, M, N, nullptr, params, param_stride, obs, act, adv, old_mean,
                                    old_log_std, ls_per_sample, obj_kind, obj_scale, clip_eps, kl_coeff, clip_log_std, min_log_std,
                                    grad, out_params, sgd_lr, stats, workspace, workspace_bytes, stream);
}

static int policy_hvp_impl(bool padded, int obs_dim, int act_dim, int hidden, int M, int N, const int32_t* n_valid,
                           const float* params, int64_t param_stride, const float* obs, const float* act,
                           const float* adv, const float* old_mean, const float* old_log_std, int ls_per_sample,
                           int obj_kind, float inner_lr, float kl_coeff, int clip_log_std, float min_log_std,
                           const float* vec, float* out, float* stats, void* workspace, int64_t workspace_bytes,
                           void* stream) {
    int st = check_policy_args(n_valid ? "promp_policy_hvp_ragged" : "promp_policy_hvp", M, N, params, obs, act, adv, old_mean, old_log_std, workspace);
    if (st != PROMP_OK) return st;
    PROMP_REQUIRE(obj_kind == PROMP_OBJ_RATIO || obj_kind == PROMP_OBJ_LOGLIK,
                  "promp_policy_hvp: inner objective must be RATIO or LOGLIK (got %d)", obj_kind);
    PROMP_REQUIRE(vec && out, "promp_policy_hvp: vec/out must not be null");
    PolicyArgs A{};
    A.M = M; A.N = N; A.params = params; A.param_stride = param_stride;
    A.obs = obs; A.act = act; A.adv = adv; A.old_mean = old_mean; A.old_ls = old_log_std;
    A.ls_per_sample = ls_per_sample; A.obj_kind = obj_kind; A.obj_scale = 1.f; A.clip_eps = 0.f;
    A.kl_coeff = kl_coeff; A.clip_log_std = clip_log_std; A.min_log_std = min_log_std;
    A.vec = vec; A.out = out; A.inner_lr = inner_lr; A.stats = stats; A.n_valid = n_valid;
    A.obs_dim = obs_dim; A.act_dim = act_dim;
    cudaStream_t s = (cudaStream_t)stream;
    PROMP_DECODE_HIDDEN("promp_policy_hvp")
    return PROMP_UNIT(hvp)(padded, obs_dim, act_dim, hidden, depth_ - 1, A, workspace, workspace_bytes, s);
}

#define PROMP_HVP_RAGGED_PARAMS                                                                                            \
    int obs_dim, int act_dim, int hidden, int M, int N, const int32_t *n_valid, const float *params, int64_t param_stride, \
        const float *obs, const float *act, const float *adv, const float *old_mean, const float *old_log_std,             \
        int ls_per_sample, int obj_kind, float inner_lr, float kl_coeff, int clip_log_std, float min_log_std,              \
        const float *vec, float *out, float *stats, void *workspace, int64_t workspace_bytes, void *stream
#define PROMP_HVP_RAGGED_ARGS                                                                                              \
    obs_dim, act_dim, hidden, M, N, n_valid, params, param_stride, obs, act, adv, old_mean, old_log_std, ls_per_sample,    \
        obj_kind, inner_lr, kl_coeff, clip_log_std, min_log_std, vec, out, stats, workspace, workspace_bytes, stream
extern "C" int promp_policy_hvp_ragged(PROMP_HVP_RAGGED_PARAMS) { return policy_hvp_impl(false, PROMP_HVP_RAGGED_ARGS); }
extern "C" int promp_policy_hvp_ragged_padded(PROMP_HVP_RAGGED_PARAMS) { return policy_hvp_impl(true, PROMP_HVP_RAGGED_ARGS); }

extern "C" int promp_policy_hvp(int obs_dim, int act_dim, int hidden, int M, int N, const float* params,
                                int64_t param_stride, const float* obs, const float* act, const float* adv,
                                const float* old_mean, const float* old_log_std, int ls_per_sample, int obj_kind,
                                float inner_lr, float kl_coeff, int clip_log_std, float min_log_std, const float* vec,
                                float* out, float* stats, void* workspace, int64_t workspace_bytes, void* stream) {
    return promp_policy_hvp_ragged(obs_dim, act_dim, hidden, M, N, nullptr, params, param_stride, obs, act, adv, old_mean,
                                   old_log_std, ls_per_sample, obj_kind, inner_lr, kl_coeff, clip_log_std, min_log_std, vec, out,
                                   stats, workspace, workspace_bytes, stream);
}

static int chain_stage_args(const promp_policy_stage* stages, int n_stages, int M, float min_log_std, PolicyArgs* A, int* kinds, int* Ns) {
    PROMP_REQUIRE(stages != nullptr && n_stages >= 1 && n_stages <= CHAIN_MAX_STAGES,
                  "promp_policy_chain: 1..%d stages (got %d)", CHAIN_MAX_STAGES, n_stages);
    for (int s = 0; s < n_stages; ++s) {
        const promp_policy_stage& g = stages[s];
        PROMP_REQUIRE(g.kind == 0 || g.kind == 1, "promp_policy_chain: stage %d has kind %d (0 = gradient, 1 = HVP)", s, g.kind);
        PROMP_REQUIRE(g.N > 0 && g.params && g.obs && g.act && g.adv && g.old_mean && g.old_log_std,
                      "promp_policy_chain: stage %d: null pointer / non-positive N", s);
        PolicyArgs& a = A[s];
        memset(&a, 0, sizeof(a));
        a.M = M; a.N = g.N; a.params = g.params; a.param_stride = g.param_stride;
        a.obs = g.obs; a.act = g.act; a.adv = g.adv; a.old_mean = g.old_mean; a.old_ls = g.old_log_std;
        a.ls_per_sample = g.ls_per_sample; a.obj_kind = g.obj_kind; a.kl_coeff = g.kl_coeff;
        a.clip_log_std = g.clip_log_std; a.min_log_std = min_log_std; a.stats = g.stats; a.n_valid = g.n_valid;
        a.kl_coeff_ptr = g.kl_coeff_dev;
        a.step_size = g.step_size;
        if (g.kind == 0) {
            PROMP_REQUIRE(g.obj_kind >= 0 && g.obj_kind <= PROMP_OBJ_EXPLORE, "promp_policy_chain: stage %d: bad obj_kind %d", s,
                          g.obj_kind);
            PROMP_REQUIRE(!(g.out_params && !g.grad), "promp_policy_chain: stage %d: out_params needs grad", s);
            // the exploration stage depends on no other stage and no stage depends on it: the dataflow kernel takes it last
            PROMP_REQUIRE(g.obj_kind != PROMP_OBJ_EXPLORE || (s == n_stages - 1 && g.param_stride == 0 && !g.out_params),
                          "promp_policy_chain: stage %d: an EXPLORE stage must be the last stage, at shared parameters "
                          "(param_stride 0) and without out_params", s);
            a.obj_scale = g.obj_scale; a.clip_eps = g.clip_eps; a.grad = g.grad; a.out_params = g.out_params; a.sgd_lr = g.sgd_lr;
            explore_args(a);
        } else {
            PROMP_REQUIRE(g.obj_kind == PROMP_OBJ_RATIO || g.obj_kind == PROMP_OBJ_LOGLIK,
                          "promp_policy_chain: stage %d: HVP inner objective must be RATIO or LOGLIK (got %d)", s, g.obj_kind);
            PROMP_REQUIRE(g.vec && g.out, "promp_policy_chain: stage %d: vec / out must not be null", s);
            a.obj_scale = 1.f; a.vec = g.vec; a.out = g.out; a.inner_lr = g.inner_lr;
        }
        kinds[s] = g.kind;
        Ns[s] = g.N;
    }
    return PROMP_OK;
}

// the argument check of the chain's size queries; sets last_error
static bool chain_query_args_ok(const char* who, int M, int n_stages, const promp_policy_stage* stages) {
    if (stages != nullptr && n_stages >= 1 && n_stages <= CHAIN_MAX_STAGES && M >= 1) return true;
    set_error("%s: needs M >= 1 and 1..%d stages (got M=%d, %d stages%s)", who, CHAIN_MAX_STAGES, M, n_stages,
              stages ? "" : ", null stages");
    return false;
}

extern "C" int promp_policy_chain_plan_info(int M, int n_stages, const promp_policy_stage* stages, int32_t* out) {
    if (!chain_query_args_ok("promp_policy_chain_plan_info", M, n_stages, stages)) return PROMP_ERR_INVALID_ARG;
    PROMP_REQUIRE(out != nullptr, "promp_policy_chain_plan_info: null out");
    int kinds[CHAIN_MAX_STAGES], Ns[CHAIN_MAX_STAGES];
    for (int s = 0; s < n_stages; ++s) kinds[s] = stages[s].kind, Ns[s] = stages[s].N > 0 ? stages[s].N : 1;
    const ChainPlan pl = plan_chain(n_stages, kinds, Ns, M, 0);
    out[0] = sm_count();
    out[1] = pl.n_items;
    for (int s = 0; s < n_stages; ++s) {
        const ChainStageInfo& I = pl.info[s];
        int32_t* o = out + 2 + 15 * s;
        o[0] = I.ntiles, o[1] = I.item_base, o[2] = I.n_items, o[3] = I.n_regions;
        for (int r = 0; r <= CHAIN_MAX_REGIONS; ++r) o[4 + r] = I.reg_m0[r];
        for (int r = 0; r < CHAIN_MAX_REGIONS; ++r) o[8 + r] = I.reg_q[r], o[11 + r] = I.reg_item0[r];
        o[14] = I.kind;
    }
    return PROMP_OK;
}

static int64_t policy_chain_workspace_bytes_impl(bool padded, int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                                 const promp_policy_stage* stages) {
    if (!chain_query_args_ok("promp_policy_chain_workspace_bytes", M, n_stages, stages)) return -1;
    int kinds[CHAIN_MAX_STAGES], Ns[CHAIN_MAX_STAGES];
    for (int s = 0; s < n_stages; ++s) kinds[s] = stages[s].kind, Ns[s] = stages[s].N > 0 ? stages[s].N : 1;
    PROMP_DECODE_HIDDEN("promp_policy_chain_workspace_bytes")
    return PROMP_UNIT(chain_workspace_bytes)(padded, obs_dim, act_dim, hidden, depth_ - 1, n_stages, kinds, Ns, M);
}
extern "C" int64_t promp_policy_chain_workspace_bytes(int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                                      const promp_policy_stage* stages) {
    return policy_chain_workspace_bytes_impl(false, obs_dim, act_dim, hidden, M, n_stages, stages);
}
extern "C" int64_t promp_policy_chain_workspace_bytes_padded(int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                                             const promp_policy_stage* stages) {
    return policy_chain_workspace_bytes_impl(true, obs_dim, act_dim, hidden, M, n_stages, stages);
}

static int policy_chain_num_launches_impl(bool padded, int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                          const promp_policy_stage* stages) {
    if (!chain_query_args_ok("promp_policy_chain_num_launches", M, n_stages, stages)) return -1;
    int kinds[CHAIN_MAX_STAGES], Ns[CHAIN_MAX_STAGES];
    for (int s = 0; s < n_stages; ++s) kinds[s] = stages[s].kind, Ns[s] = stages[s].N > 0 ? stages[s].N : 1;
    PROMP_DECODE_HIDDEN("promp_policy_chain_num_launches")
    return PROMP_UNIT(chain_launches)(padded, obs_dim, act_dim, hidden, depth_ - 1, n_stages, kinds, Ns, M);
}
extern "C" int promp_policy_chain_num_launches(int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                               const promp_policy_stage* stages) {
    return policy_chain_num_launches_impl(false, obs_dim, act_dim, hidden, M, n_stages, stages);
}
extern "C" int promp_policy_chain_num_launches_padded(int obs_dim, int act_dim, int hidden, int M, int n_stages,
                                                      const promp_policy_stage* stages) {
    return policy_chain_num_launches_impl(true, obs_dim, act_dim, hidden, M, n_stages, stages);
}

// The control words grow with M: a call with a larger M finds them where a call with a smaller M left partial slots (its
// arrival counters would start non-zero, no CTA would be a task's last arriver).  So when M changes on a workspace, clear
// them on the stream first.  An algorithm keeps one M per workspace, so the steady state (and a captured CUDA graph) has no
// extra node.  Workspaces this record has not seen are cleared once: a fresh one is zero anyway, and one pushed out of the
// record may have served another M.
static int chain_clear_on_new_m(void* ws, int M, cudaStream_t st) {
    static struct { void* ws; int M; } seen[16];
    static int next = 0;
    int i = 0;
    while (i < 16 && seen[i].ws != ws) ++i;
    if (i < 16 && seen[i].M == M) return PROMP_OK;
    if (i == 16) i = next, next = (next + 1) % 16;
    seen[i].ws = ws, seen[i].M = M;
    PROMP_CUDA(cudaMemsetAsync(ws, 0, chain_ctrl_bytes(M), st));
    return PROMP_OK;
}

static int policy_chain_impl(bool padded, int obs_dim, int act_dim, int hidden, int M, float min_log_std, int n_stages,
                             const promp_policy_stage* stages, const int32_t* skip_flag, const float* skip_theta,
                             void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(M > 0 && workspace != nullptr, "promp_policy_chain: M must be positive and workspace non-null");
    PROMP_REQUIRE((skip_flag == nullptr) == (skip_theta == nullptr), "promp_policy_chain: skip_flag / skip_theta come as a pair");
    PolicyArgs A[CHAIN_MAX_STAGES];
    int kinds[CHAIN_MAX_STAGES], Ns[CHAIN_MAX_STAGES];
    const int rc = chain_stage_args(stages, n_stages, M, min_log_std, A, kinds, Ns);
    if (rc != PROMP_OK) return rc;
    PROMP_REQUIRE(!skip_flag || (kinds[0] == 0 && A[0].param_stride == 0 && !A[0].adv_per_task),
                  "promp_policy_chain: launch re-use is defined for a gradient stage 0 on shared parameters (param_stride 0)");
    for (int k = 0; k < n_stages; ++k) A[k].obs_dim = obs_dim, A[k].act_dim = act_dim;
    cudaStream_t s = (cudaStream_t)stream;
    PROMP_DECODE_HIDDEN("promp_policy_chain")
    if (workspace_bytes < chain_ctrl_bytes(M)) {
        set_error("policy chain workspace too small (%lld < %lld bytes of control words)", (long long)workspace_bytes,
                  (long long)chain_ctrl_bytes(M));
        return PROMP_ERR_WORKSPACE;
    }
    const int rc_clear = chain_clear_on_new_m(workspace, M, s);
    if (rc_clear != PROMP_OK) return rc_clear;
    return PROMP_UNIT(chain)(padded, obs_dim, act_dim, hidden, depth_ - 1, n_stages, kinds, A, skip_flag, skip_theta, workspace,
                             workspace_bytes, s);
}
extern "C" int promp_policy_chain(int obs_dim, int act_dim, int hidden, int M, float min_log_std, int n_stages,
                                  const promp_policy_stage* stages, const int32_t* skip_flag, const float* skip_theta,
                                  void* workspace, int64_t workspace_bytes, void* stream) {
    return policy_chain_impl(false, obs_dim, act_dim, hidden, M, min_log_std, n_stages, stages, skip_flag, skip_theta, workspace,
                             workspace_bytes, stream);
}
extern "C" int promp_policy_chain_padded(int obs_dim, int act_dim, int hidden, int M, float min_log_std, int n_stages,
                                         const promp_policy_stage* stages, const int32_t* skip_flag, const float* skip_theta,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
    return policy_chain_impl(true, obs_dim, act_dim, hidden, M, min_log_std, n_stages, stages, skip_flag, skip_theta, workspace,
                             workspace_bytes, stream);
}

extern "C" int promp_set_option(const char* name, int value) {
    PROMP_REQUIRE(name != nullptr, "promp_set_option: null name");
    if (strcmp(name, "tensor_cores") == 0) {
        g_use_tc = value ? 1 : 0;
        return PROMP_OK;
    }
    if (strcmp(name, "chain") == 0) {          // promp_policy_chain: dataflow kernel (1), one launch per stage (0), automatic (-1)
        g_chain = value < 0 ? -1 : (value ? 1 : 0);
        return PROMP_OK;
    }
    if (strcmp(name, "chain_q") == 0) {        // tiles per work item of the dataflow kernel (0 = automatic)
        PROMP_REQUIRE(value >= 0 && value <= 64, "promp_set_option: chain_q must be in [0, 64]");
        g_chain_q = value;
        return PROMP_OK;
    }
    if (strcmp(name, "chain_taper") == 0) {    // shrinking items at the end of the last stage (1, default) or uniform (0)
        g_chain_taper = value ? 1 : 0;
        return PROMP_OK;
    }
    if (strcmp(name, "tc_threads") == 0) {
        PROMP_REQUIRE(value == 0 || value == 256 || value == 512, "promp_set_option: tc_threads must be 0, 256 or 512");
        g_tc_threads = value;
        return PROMP_OK;
    }
    set_error("promp_set_option: unknown option '%s'", name);
    return PROMP_ERR_INVALID_ARG;
}

static int policy_forward_impl(bool padded, int obs_dim, int act_dim, int hidden, int M, int N, const float* params,
                               int64_t param_stride, const float* obs, float* mean, void* stream) {
    PROMP_REQUIRE(M > 0 && N > 0 && params && obs && mean, "promp_policy_forward: bad arguments");
    PROMP_REQUIRE(M <= 65535, "promp_policy_forward: M=%d exceeds the grid.y limit", M);
    cudaStream_t s = (cudaStream_t)stream;
    PROMP_DECODE_HIDDEN("promp_policy_forward")
    return PROMP_UNIT(forward)(padded, obs_dim, act_dim, hidden, depth_ - 1, M, N, params, param_stride, obs, mean, s);
}
extern "C" int promp_policy_forward(int obs_dim, int act_dim, int hidden, int M, int N, const float* params,
                                    int64_t param_stride, const float* obs, float* mean, void* stream) {
    return policy_forward_impl(false, obs_dim, act_dim, hidden, M, N, params, param_stride, obs, mean, stream);
}
extern "C" int promp_policy_forward_padded(int obs_dim, int act_dim, int hidden, int M, int N, const float* params,
                                           int64_t param_stride, const float* obs, float* mean, void* stream) {
    return policy_forward_impl(true, obs_dim, act_dim, hidden, M, N, params, param_stride, obs, mean, stream);
}

extern "C" int promp_reduce_tasks(int M, int P, const float* in, float scale, float* out, void* stream) {
    PROMP_REQUIRE(M > 0 && P > 0 && in && out, "promp_reduce_tasks: bad arguments");
    reduce_tasks_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(M, P, in, scale, out);
    PROMP_LAUNCH_CHECK("reduce_tasks_kernel");
    return PROMP_OK;
}

extern "C" int promp_reduce_tasks2(int M, int P, const float* a, const float* b, float scale, float* out, void* stream) {
    PROMP_REQUIRE(M > 0 && P > 0 && a && b && out, "promp_reduce_tasks2: bad arguments");
    reduce_tasks2_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(M, P, a, b, scale, out);
    PROMP_LAUNCH_CHECK("reduce_tasks2_kernel");
    return PROMP_OK;
}

extern "C" int promp_meta_loss_terms(int S, int M, const float* stats_all, float inv_m_global, const float* coeff, int n_out,
                                     float* out, void* stream) {
    PROMP_REQUIRE(S >= 1 && S <= 7 && M > 0 && stats_all && out && n_out >= 1 && n_out <= S + 1,
                  "promp_meta_loss_terms: bad arguments (1 <= S <= 7 sampling phases, 1 <= n_out <= S+1)");
    meta_loss_terms_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(S, M, stats_all, inv_m_global, coeff, n_out, out);
    PROMP_LAUNCH_CHECK("meta_loss_terms_kernel");
    return PROMP_OK;
}

extern "C" int promp_phase_log_terms(int M, int act_dim, double n_paths, const double* stats, const float* log_std, double* out7,
                                     void* stream) {
    PROMP_REQUIRE(M > 0 && act_dim > 0 && n_paths > 0 && stats && log_std && out7, "promp_phase_log_terms: bad arguments");
    phase_log_terms_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(M, act_dim, n_paths, stats, log_std, out7);
    PROMP_LAUNCH_CHECK("phase_log_terms_kernel");
    return PROMP_OK;
}

extern "C" int promp_promp_log_terms(int num_inner_steps, const float* final_terms, double* out3, void* stream) {
    PROMP_REQUIRE(num_inner_steps >= 0 && final_terms && out3, "promp_promp_log_terms: bad arguments");
    promp_log_terms_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(num_inner_steps, final_terms, out3);
    PROMP_LAUNCH_CHECK("promp_log_terms_kernel");
    return PROMP_OK;
}

extern "C" int promp_adapt_kl_coeff(int num_inner_steps, const float* final_terms, double kl_target, int adapt, float* coeff_dev,
                                    double* out4, void* stream) {
    PROMP_REQUIRE(num_inner_steps >= 0 && num_inner_steps <= 7 && final_terms && (coeff_dev || num_inner_steps == 0),
                  "promp_adapt_kl_coeff: bad arguments");
    adapt_kl_coeff_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(num_inner_steps, final_terms, kl_target, adapt, coeff_dev, out4);
    PROMP_LAUNCH_CHECK("adapt_kl_coeff_kernel");
    return PROMP_OK;
}

extern "C" int promp_adam_tf1(int P, float* theta, const float* grad, float* m, float* v, int32_t* step, float lr,
                              float beta1, float beta2, float eps, void* stream) {
    PROMP_REQUIRE(P > 0 && theta && grad && m && v && step, "promp_adam_tf1: bad arguments");
    cudaStream_t s = (cudaStream_t)stream;
    adam_tf1_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, theta, grad, m, v, step, lr, beta1, beta2, eps);
    adam_step_inc_kernel<<<1, 1, 0, s>>>(step);
    PROMP_LAUNCH_CHECK("adam_tf1_kernel");
    return PROMP_OK;
}

#ifdef PROMP_EXP_CLOCKS
extern "C" int promp_debug_chain_clocks(unsigned long long* out16, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out16, promp::g_chain_clk, 16 * sizeof(unsigned long long));
    if (reset) {
        unsigned long long z[16] = {0};
        cudaMemcpyToSymbol(promp::g_chain_clk, z, sizeof(z));
    }
    return 0;
}
extern "C" int promp_debug_phase_clocks(unsigned long long* out16, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out16, promp::g_phase_clk, 16 * sizeof(unsigned long long));
    if (reset) {
        unsigned long long z[16] = {0};
        cudaMemcpyToSymbol(promp::g_phase_clk, z, sizeof(z));
    }
    return 0;
}
#endif
#endif  // !PROMP_POLICY_EXTRA_TU
