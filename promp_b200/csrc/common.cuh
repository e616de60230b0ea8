// Shared device/host helpers for the promp_b200 kernels (sm_90a).
// The device parts also compile under NVRTC (__CUDACC_RTC__: user environments, promp_b200/_jit.py); the host-only parts
// (error plumbing, argument decoding) are left out there.
#pragma once
#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>
#include <stdio.h>
#endif
#include <stdint.h>
#include "../../include/promp_b200.h"

namespace promp {

// SM count of the target GPU (H100 SXM) for the launch-size heuristics that are fixed at compile time
constexpr int PROMP_NUM_SMS = 132;

#ifndef __CUDACC_RTC__
// ---------------------------------------------------------------- error plumbing (host)
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);

#define PROMP_REQUIRE(cond, ...)                                   \
    do {                                                           \
        if (!(cond)) {                                             \
            promp::set_error(__VA_ARGS__);                         \
            return PROMP_ERR_INVALID_ARG;                          \
        }                                                          \
    } while (0)

#define PROMP_CUDA(call)                                           \
    do {                                                           \
        int _st = promp::check_cuda((call), #call);                \
        if (_st != PROMP_OK) return _st;                           \
    } while (0)

#define PROMP_LAUNCH_CHECK(name)                                   \
    do {                                                           \
        int _st = promp::check_cuda(cudaGetLastError(), name);     \
        if (_st != PROMP_OK) return _st;                           \
    } while (0)
#endif

// ---------------------------------------------------------------- parameter layout
// Flat parameter vector in the reference's creation order
// (ref: policies/gaussian_mlp_policy.py:55-80, policies/networks/mlp.py:100):
//   W0[Do,Hd] b0[Hd] W1[Hd,Hd] b1[Hd] W2[Hd,Da] b2[Da] log_std[Da]
template <int DO, int DA, int HID>
struct PLayout {
    static constexpr int W0 = 0;
    static constexpr int B0 = W0 + DO * HID;
    static constexpr int W1 = B0 + HID;
    static constexpr int B1 = W1 + HID * HID;
    static constexpr int W2 = B1 + HID;
    static constexpr int B2 = W2 + HID * DA;
    static constexpr int LS = B2 + DA;
    static constexpr int P = LS + DA;
};

__host__ __device__ inline int num_params(int Do, int Da, int Hd) {
    return Do * Hd + Hd + Hd * Hd + Hd + Hd * Da + Da + Da;
}
// Any depth (1..3 hidden layers): W0[Do,Hd] b0[Hd] {W_l[Hd,Hd] b_l[Hd]}_{l=1..depth-1} W_out[Hd,Da] b_out[Da] log_std[Da]
__host__ __device__ inline int num_params(int Do, int Da, int Hd, int depth) {
    return Do * Hd + Hd + (depth - 1) * (Hd * Hd + Hd) + Hd * Da + Da + Da;
}
// The same layout with the number of hidden-to-hidden layers nh = depth - 1 known at run time (the kernels of depth 1 and 3)
template <int DO, int DA, int HID>
struct DeepLayout {
    int nh;
    static constexpr int W0 = 0, B0 = DO * HID;
    __host__ __device__ int wh(int l) const { return B0 + HID + l * (HID * HID + HID); }   // W_{l+1}, l < nh
    __host__ __device__ int bh(int l) const { return wh(l) + HID * HID; }
    __host__ __device__ int wo() const { return wh(nh); }
    __host__ __device__ int bo() const { return wo() + HID * DA; }
    __host__ __device__ int ls() const { return bo() + DA; }
    __host__ __device__ int P() const { return ls() + DA; }
};

// ---------------------------------------------------------------- math
// tanh via one ex2.approx + one fast division: |abs error| <= ~2e-7 over the whole range (saturates to +-1
// exactly for |x| > 10), ~4x fewer instructions than tanhf.  MUFU.TANH (tanh.approx) is only 2^-11 accurate
// and would break the 1e-4 parity bar on gradients.
// Five instructions (FMUL, MUFU.EX2, FADD, MUFU.RCP, FFMA): the .ftz forms drop the denormal / huge-operand guard sequences of
// __expf / __fdividef (7-8 extra instructions per call, ~10 % of all instructions of the policy kernels), whose cases end in
// the same saturated values here (e -> 0: 1 - 2 = -1; e -> inf: 1 - 0 = 1).  2 * log2(e) is folded into one constant:
// (2 x) * c and x * (2 c) are the same real number, so the rounded product is bit-identical.
__device__ __forceinline__ float tanh_fast(float x) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * 2.8853900817779268f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
    return fmaf(-2.0f, r, 1.0f);
}

// ---------------------------------------------------------------- hidden-layer activations
// Every policy kernel takes its hidden non-linearity as a template parameter.  The kernels keep the activation OUTPUT h,
// so the derivatives are written in terms of h:
//   f(z)     = sigma(z)
//   d(h)     = sigma'(z)
//   dd_d(h)  = sigma''(z) / sigma'(z).  The Hessian-vector kernels carry the tangent r = sigma'(z) * zdot of h, and their
//              second-derivative term sigma''(z) * zdot is dd_d(h) * r (tanh: -2 h r).
// CURVED = false says sigma'' = 0 everywhere the kernels evaluate it (ReLU): the Hessian-vector kernels drop the
// second-derivative terms at compile time.
// OUT_TANH = false: the trait's policy has the identity output layer (see OutTanh below).
struct ActTanh {
    static constexpr bool CURVED = true;
    static constexpr bool OUT_TANH = false;
    __device__ __forceinline__ static float f(float z) { return tanh_fast(z); }
    __device__ __forceinline__ static float d(float h) { return 1.f - h * h; }
    __device__ __forceinline__ static float dd_d(float h) { return -2.f * h; }
};
// sigma'(0) = 0, as TensorFlow's ReluGrad (the gradient flows only where the output is positive)
struct ActRelu {
    static constexpr bool CURVED = false;
    static constexpr bool OUT_TANH = false;
    __device__ __forceinline__ static float f(float z) { return fmaxf(z, 0.f); }
    __device__ __forceinline__ static float d(float h) { return h > 0.f ? 1.f : 0.f; }
};
// The same hidden activation with a tanh output layer: mean = tanh(h2 W2 + b2) (policies/networks/mlp.py:53-56, 93-113,
// output_nonlinearity=tf.tanh).  The policy kernels take the pair as their one activation parameter; the out_* helpers
// below are no-ops for the identity output, so the kernels of ActTanh / ActRelu keep their code.
template <class Hid>
struct OutTanh : Hid {
    using Hidden = Hid;
    static constexpr bool OUT_TANH = true;
};

// Backward step of the Hessian-vector product through one hidden layer:  c * sigma'(z) + ac * dh * sigma''(z) * zdot,
// with h = sigma(z) and r = sigma'(z) * zdot.
template <class Act>
__device__ __forceinline__ float act_hvp_back(float c, float dh, float h, float r, float ac) {
    if constexpr (Act::CURVED) return c * Act::d(h) + ac * dh * (Act::dd_d(h) * r);
    else return c * Act::d(h);
}

// ---- output layer of the mean, for DA action dimensions.  mu holds z = h2 W2 + b2 on entry, the mean on exit.
template <class Act, int DA>
__device__ __forceinline__ void out_forward(float (&mu)[DA]) {
    if constexpr (Act::OUT_TANH) {
#pragma unroll
        for (int d = 0; d < DA; ++d) mu[d] = ActTanh::f(mu[d]);
    }
}
// ... and the tangent: rmu holds zdot on entry, the mean's tangent (1 - mu^2) zdot on exit
template <class Act, int DA>
__device__ __forceinline__ void out_forward_tangent(float (&mu)[DA], float (&rmu)[DA]) {
    if constexpr (Act::OUT_TANH) {
#pragma unroll
        for (int d = 0; d < DA; ++d) {
            mu[d] = ActTanh::f(mu[d]);
            rmu[d] *= ActTanh::d(mu[d]);
        }
    }
}
// Gradient: the head's d loss / d mu -> d loss / d z
template <class Act, int DA>
__device__ __forceinline__ void out_grad_back(const float (&mu)[DA], float (&dmu)[DA]) {
    if constexpr (Act::OUT_TANH) {
#pragma unroll
        for (int d = 0; d < DA; ++d) dmu[d] *= ActTanh::d(mu[d]);
    }
}
// Hessian-vector product: the head's signals at mu (dmu, cmu; rmu = the mean's tangent) -> their values at z.  The same
// step as a hidden layer's (act_hvp_back), with the mean in place of h:  C_z = (1 - mu^2) cmu + ac dmu (-2 mu) rmu.
template <class Act, int DA>
__device__ __forceinline__ void out_hvp_back(const float (&mu)[DA], const float (&rmu)[DA], float ac, float (&dmu)[DA],
                                             float (&cmu)[DA]) {
    if constexpr (Act::OUT_TANH) {
#pragma unroll
        for (int d = 0; d < DA; ++d) {
            cmu[d] = act_hvp_back<ActTanh>(cmu[d], dmu[d], mu[d], rmu[d], ac);
            dmu[d] *= ActTanh::d(mu[d]);
        }
    }
}

#ifndef __CUDACC_RTC__
// The `hidden` argument of the policy and rollout entry points: the width (32 or 64) in the low byte, PROMP_ACT_RELU and
// PROMP_OUT_TANH above it, the number of hidden layers in the PROMP_HIDDEN_DEPTH_MASK field (no bits = 2).  A plain width
// selects two tanh hidden layers and the identity output.
inline int decode_hidden(const char* who, int hidden, int& width, bool& relu, bool& out_tanh, int& depth) {
    constexpr int known = PROMP_HIDDEN_WIDTH_MASK | PROMP_ACT_RELU | PROMP_OUT_TANH | PROMP_HIDDEN_DEPTH_MASK;
    PROMP_REQUIRE((hidden & ~known) == 0,
                  "%s: unknown flag bits 0x%x in hidden (%d); known: PROMP_ACT_RELU = 0x%x, PROMP_OUT_TANH = 0x%x, "
                  "PROMP_HIDDEN_DEPTH_MASK = 0x%x", who, hidden & ~known, hidden, PROMP_ACT_RELU, PROMP_OUT_TANH,
                  PROMP_HIDDEN_DEPTH_MASK);
    width = hidden & PROMP_HIDDEN_WIDTH_MASK;
    relu = (hidden & PROMP_ACT_RELU) != 0;
    out_tanh = (hidden & PROMP_OUT_TANH) != 0;
    const int field = (hidden & PROMP_HIDDEN_DEPTH_MASK) >> PROMP_HIDDEN_DEPTH_SHIFT;
    depth = field == 0 ? 2 : field;
    PROMP_REQUIRE(!relu || width == 32 || width == 64, "%s: ReLU policies are built for hidden 32 or 64 (got %d)", who, width);
    PROMP_REQUIRE(!out_tanh || width == 32 || width == 64, "%s: tanh-output policies are built for hidden 32 or 64 (got %d)",
                  who, width);
    PROMP_REQUIRE(depth <= 3, "%s: policies have 1 to 3 hidden layers (depth field %d in hidden 0x%x)", who, depth, hidden);
    PROMP_REQUIRE(field == 0 || width == 32 || width == 64,
                  "%s: policies of depth 1 or 3 are built for hidden 32 or 64 (got %d)", who, width);
    return PROMP_OK;
}

// The Philox key of an env is its global index (task_offset + m) * E + e, a 32-bit word (rollout entry points)
inline int check_task_offset(const char* fn, int task_offset, int M, int E) {
    PROMP_REQUIRE(task_offset >= 0, "%s: task_offset must be >= 0 (got %d)", fn, task_offset);
    PROMP_REQUIRE(((int64_t)task_offset + M) * E <= ((int64_t)1 << 32),
                  "%s: (task_offset + M) * E = (%d + %d) * %d exceeds the 32-bit Philox env key", fn, task_offset, M, E);
    return PROMP_OK;
}
#endif

// ---------------------------------------------------------------- warp helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------- TMA bulk copies (cp.async.bulk, 1-D) + mbarriers
// Contiguous global -> shared copies issued by ONE thread and completed on an mbarrier (SASS: UBLKCP).  Source, destination
// and size must be multiples of 16 bytes.
__device__ __forceinline__ uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tma_mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_addr_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void tma_mbar_fence_init() {     // make the initialised barriers visible to the async proxy
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
__device__ __forceinline__ void tma_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}\n" ::"r"(smem_addr_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_addr_u32(bar)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                     smem_addr_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_addr_u32(bar))
                 : "memory");
}

// ---------------------------------------------------------------- Philox4x32-10
struct Philox {
    static constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    __host__ __device__ static inline void round(uint32_t c[4], uint32_t k0, uint32_t k1) {
        uint64_t p0 = (uint64_t)M0 * c[0], p1 = (uint64_t)M1 * c[2];
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    }
    // counter = (c0,c1,c2,c3), key = seed
    __host__ __device__ static inline void gen(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint64_t seed,
                                               uint32_t out[4]) {
        uint32_t c[4] = {c0, c1, c2, c3};
        uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
        for (int i = 0; i < 10; ++i) {
            round(c, k0, k1);
            k0 += W0;
            k1 += W1;
        }
        out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
    }
};
// uniform in (0,1]: never 0 so log() is finite
__host__ __device__ inline float u01(uint32_t x) { return ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f); }
// two N(0,1) from two uint32 (Box-Muller)
__device__ inline void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
    float r = sqrtf(-2.0f * logf(u01(a)));
    float s, c;
    sincospif(2.0f * u01(b), &s, &c);
    z0 = r * c;
    z1 = r * s;
}

}  // namespace promp
