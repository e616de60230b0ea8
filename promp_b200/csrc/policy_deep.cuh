// CUDA-core kernels of the policies with one or three hidden layers (hidden_sizes of length 1 or 3, PROMP_HIDDEN_DEPTH):
// gradient (with the E-MAML exploration variant), Hessian-vector product and forward.  Included by policy.cu after its
// two-layer kernels, so that every activation unit (tanh_tu, relu_tu, otanh_tu, relu_otanh_tu) instantiates them for its
// own activation; policy.cu's launchers pick them for every depth but two.
//
// One instantiation per (obs, act, hidden width, activation) serves both depths: the number of hidden-to-hidden layers
// nh = depth - 1 (0 or 2) is a kernel argument, the per-layer loops are unrolled to DEEP_NH and predicated on it.  The tile
// schedule, thread roles, Gaussian head and task-segment flush are those of the two-layer CUDA-core kernels (64-sample tiles,
// 256 threads); what differs:
//   - the weights are staged per layer (DeepW): hidden-to-hidden matrices with rows padded to HID + 4 floats, so that the
//     forward GEMM reads them row-major and the backward GEMM (dH = D W^T, gemm_tile_t) reads their rows without bank
//     conflicts and without a transposed copy;
//   - every layer's activation tile H_l (and, in the HVP, its tangent R_l) stays in shared memory for the backward pass, and
//     the backward signals overwrite them in place;
//   - the elementwise backward steps own the strided columns tx + TX c of gemm_tile_t (bias sums follow that mapping);
//   - the layout offsets (DeepLayout) and P are run-time values, so the flush and epilogues take them as arguments.
namespace promp {

constexpr int DEEP_NH = 2;      // hidden-to-hidden layers of the deepest supported policy (three hidden layers)

template <int DO, int DA, int HID>
struct DeepW {
    static constexpr int LDW = HID + 4, DAP = (DA + 3) / 4 * 4;
    float W0[DO * HID];
    float B0[HID];
    float WH[DEEP_NH][HID * LDW];
    float BH[DEEP_NH][HID];
    float WO[HID * DA];
    float BO[DAP];
    float LS[DAP];
};

// Stage one parameter set (DeepLayout order) into shared memory; get(i) = its i-th value.
template <int DO, int DA, int HID, class Get>
__device__ __forceinline__ void deep_stage(DeepW<DO, DA, HID>& W, const DeepLayout<DO, DA, HID>& L, Get get) {
    constexpr int LDW = DeepW<DO, DA, HID>::LDW;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < DO * HID + HID; i += nt) {
        const float v = get(i);
        if (i < DO * HID) W.W0[i] = v;
        else W.B0[i - DO * HID] = v;
    }
    for (int l = 0; l < L.nh; ++l) {
        for (int i = tid; i < HID * HID; i += nt) W.WH[l][(i / HID) * LDW + i % HID] = get(L.wh(l) + i);
        for (int i = tid; i < HID; i += nt) W.BH[l][i] = get(L.bh(l) + i);
    }
    for (int i = tid; i < HID * DA + 2 * DA; i += nt) {
        const float v = get(L.wo() + i);
        if (i < HID * DA) W.WO[i] = v;
        else if (i < HID * DA + DA) W.BO[i - HID * DA] = v;
        else W.LS[i - HID * DA - DA] = v;
    }
}

// acc[i][c] += sum_k A[row0+i][k] * W[col0 + c*CS][k]: the product with W^T for W [HID][LDW] row-major.  The thread's
// output columns are col0 + c*CS, CS threads apart: the 8 threads of a quarter-warp read 8 consecutive W rows, which
// LDW % 32 == 4 spreads over all 32 banks.
template <int K, int LDA, int LDW, int CS, int RM>
__device__ __forceinline__ void gemm_tile_t(const float* __restrict__ A, const float* __restrict__ W, int row0, int col0,
                                            float (&acc)[RM][4]) {
#pragma unroll 4
    for (int k = 0; k < K; k += 4) {
        float4 a[RM], w[4];
#pragma unroll
        for (int i = 0; i < RM; ++i) a[i] = *reinterpret_cast<const float4*>(A + (row0 + i) * LDA + k);
#pragma unroll
        for (int c = 0; c < 4; ++c) w[c] = *reinterpret_cast<const float4*>(W + (col0 + c * CS) * LDW + k);
#pragma unroll
        for (int i = 0; i < RM; ++i)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                acc[i][c] = fmaf(a[i].x, w[c].x, acc[i][c]);
                acc[i][c] = fmaf(a[i].y, w[c].y, acc[i][c]);
                acc[i][c] = fmaf(a[i].z, w[c].z, acc[i][c]);
                acc[i][c] = fmaf(a[i].w, w[c].w, acc[i][c]);
            }
    }
}

// Launch re-use (promp_policy_grad_ex) with the run-time P: see reuse_hit / reuse_produce
__device__ __forceinline__ bool deep_reuse_hit(const PolicyArgs& A, int P) {
    if (!A.skip_flag) return false;
    bool same = *reinterpret_cast<const volatile int*>(A.skip_flag) != 0;
    for (int i = threadIdx.x; i < P && same; i += blockDim.x)
        same = __float_as_uint(__ldcg(A.params + i)) == __float_as_uint(__ldcg(A.skip_theta + i));
    return __syncthreads_and(same ? 1 : 0) != 0;
}
template <int DA>
__device__ __forceinline__ void deep_reuse_produce(const PolicyArgs& A, int P, int ls) {
    if (A.unclipped_out && blockIdx.x == 0) {
        if (threadIdx.x == 0) {
            int ok = 1;
            for (int d = 0; d < DA; ++d)
                if (!(__ldcg(A.params + ls + d) >= A.min_log_std)) ok = 0;
            *A.unclipped_out = ok;
        }
        for (int i = threadIdx.x; i < P; i += blockDim.x) A.theta_copy_out[i] = __ldcg(A.params + i);
    }
}

// GradEpilogue / HvpEpilogue with the run-time P
struct DeepGradEpilogue {
    const PolicyArgs& A;
    const float* th;
    int m, P;
    __device__ __forceinline__ float4 pre(int p) const {
        return A.out_params ? __ldg(reinterpret_cast<const float4*>(th + p)) : make_float4(0.f, 0.f, 0.f, 0.f);
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
struct DeepHvpEpilogue {
    const PolicyArgs& A;
    const float* vg;
    int m, P;
    __device__ __forceinline__ float4 pre(int p) const { return __ldcg(reinterpret_cast<const float4*>(vg + p)); }
    __device__ __forceinline__ void out(int p, float4 v, float4 s) const {
        *reinterpret_cast<float4*>(A.out + (int64_t)m * P + p) = make_float4(v.x + s.x, v.y + s.y, v.z + s.z, v.w + s.w);
    }
};

// flush_tail with the run-time P and output-kernel offset wo (W0 starts at 0)
template <int DO, int DA, int HID, class Epi>
__device__ __forceinline__ void deep_flush_tail(const PolicyArgs& A, const UniformSched& sc, int P, int wo, int m, float invN,
                                                bool want, float* part, float* scr, float* red, int& last,
                                                const float (&gW0p)[DO], const float (&gW2p)[DA], float s_obj, float s_kl,
                                                float s_ratio, const Epi& epi) {
    constexpr int THREADS = PT_THREADS, NPART = THREADS / HID, NW = THREADS / 32, NP = 2;
    const int PSTRIDE = P + PSTAT;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cj = tid % HID, cp = tid / HID;
    if (want) {
#pragma unroll
        for (int i = 0; i < DO; ++i) scr[(cp * DO + i) * HID + cj] = gW0p[i];
        __syncthreads();
        for (int idx = tid; idx < DO * HID; idx += THREADS) {
            float s = 0.f;
            for (int p = 0; p < NPART; ++p) s += scr[p * DO * HID + idx];
            part[idx] = s;
        }
        __syncthreads();
#pragma unroll
        for (int d = 0; d < DA; ++d) scr[(cp * HID + cj) * DA + d] = gW2p[d];
        __syncthreads();
        for (int idx = tid; idx < HID * DA; idx += THREADS) {
            float s = 0.f;
            for (int p = 0; p < NPART; ++p) s += scr[p * HID * DA + idx];
            part[wo + idx] = s;
        }
    }
    const float v0 = warp_sum(s_obj), v1 = warp_sum(s_kl), v2 = warp_sum(s_ratio);
    __syncthreads();
    if (lane == 0) red[warp] = v0, red[NW + warp] = v1, red[2 * NW + warp] = v2;
    __syncthreads();
    if (tid < 3) {
        float s = 0.f;
        for (int w = 0; w < NW; ++w) s += red[tid * NW + w];
        part[P + tid] = s;
    }
    __syncthreads();
    const int n_c = sc.n_contrib(m);
    if (tid == 0) {
        __threadfence();
        last = (atomicAdd(A.counters + m, 1) == n_c - 1);
    }
    __syncthreads();
    if (last) {
        __threadfence();
        if (want) {
#pragma unroll 1
            for (int p0 = 4 * tid; p0 < P + 4; p0 += NP * 4 * THREADS) {
                float4 sum[NP], t4[NP];
#pragma unroll
                for (int i = 0; i < NP; ++i) {
                    const int p = p0 + i * 4 * THREADS;
                    t4[i] = p < P ? epi.pre(p) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                reduce_slots4_wide<NP>(A.partial, sc, PSTRIDE, m, n_c, p0, 4 * THREADS, P + 4, sum);
#pragma unroll
                for (int i = 0; i < NP; ++i) {
                    const int p = p0 + i * 4 * THREADS;
                    const float4 s = sum[i];
                    if (p == P) {
                        if (A.stats)
                            A.stats[(int64_t)m * 4 + 0] = s.x * invN, A.stats[(int64_t)m * 4 + 1] = s.y * invN,
                                                    A.stats[(int64_t)m * 4 + 2] = s.z * invN;
                    } else if (p < P) {
                        epi.out(p, t4[i], s);
                    }
                }
            }
        } else if (tid == 0 && A.stats) {
            const float4 s = reduce_slots4(A.partial, sc, PSTRIDE, m, n_c, P);
            A.stats[(int64_t)m * 4 + 0] = s.x * invN, A.stats[(int64_t)m * 4 + 1] = s.y * invN, A.stats[(int64_t)m * 4 + 2] = s.z * invN;
        }
        if (tid == 0) A.counters[m] = 0;
    }
    __syncthreads();
}

// Bias partials of every layer l <= nh: gB[l][c] belongs to unit tx + TX c (the strided columns); reduce the TY row groups.
template <int HID>
__device__ __forceinline__ void deep_flush_biases(float* part, float* scr, int nh, int b0_off, int bh0_off,
                                                  const float (&gB)[DEEP_NH + 1][4]) {
    using C = TileCfg<HID>;
    const int tid = threadIdx.x, tx = tid % C::TX, ty = tid / C::TX;
#pragma unroll
    for (int l = 0; l <= DEEP_NH; ++l) {
        if (l > nh) break;
#pragma unroll
        for (int c = 0; c < 4; ++c) scr[ty * HID + tx + C::TX * c] = gB[l][c];
        __syncthreads();
        if (tid < HID) {
            float s = 0.f;
            for (int y = 0; y < C::TY; ++y) s += scr[y * HID + tid];
            part[(l == 0 ? b0_off : bh0_off + (l - 1) * (HID * HID + HID)) + tid] = s;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------ gradient
template <int DO, int DA, int HID>
struct DeepGradSmem {
    static constexpr int DOP = DOPad<DO>::V, LD = TileCfg<HID>::LD;
    DeepW<DO, DA, HID> W;
    float H[DEEP_NH + 1][TB * LD];     // activations of every hidden layer, then their backprop signals; also flush scratch
    float X[TB * DOP];
    float DMU[TB * DA];
    float DLS[TB * DA];
    float red[3 * (PT_THREADS / 32)];
    int last;
};

template <int DO, int DA, int HID, class Act, int ADV>
__device__ __forceinline__ void deep_grad_body(const PolicyArgs& A, int nh) {
    using C = TileCfg<HID>;
    using R = RoleCfg<HID>;
    using SM = DeepGradSmem<DO, DA, HID>;
    constexpr int LD = C::LD, RM = C::RM, RK = C::RK, TX = C::TX, DOP = SM::DOP, LDW = DeepW<DO, DA, HID>::LDW;
    constexpr int BPP = R::BPP, QW = R::QW;
    static_assert(R::NPART * DO * HID <= (DEEP_NH + 1) * TB * LD && R::NPART * HID * DA <= (DEEP_NH + 1) * TB * LD,
                  "flush scratch too small");
    const DeepLayout<DO, DA, HID> L{nh};
    const int P = L.P();

    extern __shared__ __align__(16) unsigned char smem_raw[];
    SM& S = *reinterpret_cast<SM*>(smem_raw);

    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int row0 = ty * RM, col0 = tx * 4;
    const int rb = tid >> 2, rq = tid & 3;
    const int cj = tid % HID, cp = tid / HID;
    const int dO = obs_dim_of<DO, DA>(A), dA = act_dim_of<DO, DA>(A);
    if (deep_reuse_hit(A, P)) return;
    deep_reuse_produce<DA>(A, P, L.ls());
    const UniformSched sc(A.M, A.N, A.q, A.kmax, TB);
    const int N = A.N;
    const float kl_eff = kl_coeff_eff(A);
    float invN = 1.0f / (float)N;
    int Nm = N;
    const bool want_grad = A.grad != nullptr;
    const float* th = nullptr;
    HeadIn<DA> hin;
    float* HL = S.H[nh];      // the last hidden layer

    float gW[DEEP_NH][RK][4];       // GEMM role: H_l^T D_{l+1}
    float gB[DEEP_NH + 1][4];       // strided columns: bias sums of layer l (0 = b0)
    float gW0p[DO], gW2p[DA];
    float gB2 = 0.f, gLS = 0.f;
    float s_obj, s_kl, s_ratio;
    auto zero_acc = [&]() {
#pragma unroll
        for (int l = 0; l < DEEP_NH; ++l)
#pragma unroll
            for (int r = 0; r < RK; ++r) gW[l][r][0] = gW[l][r][1] = gW[l][r][2] = gW[l][r][3] = 0.f;
#pragma unroll
        for (int l = 0; l <= DEEP_NH; ++l) gB[l][0] = gB[l][1] = gB[l][2] = gB[l][3] = 0.f;
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
        if (!first && A.param_stride == 0) return;
        __syncthreads();
        deep_stage(S.W, L, [&](int i) { return __ldg(th + i); });
        __syncthreads();
        head_setup<DA>(A, S.W.LS, m, dA, hin, nullptr);
    };
    auto flush = [&](int m) {
        float* part = A.partial + (int64_t)sc.my_slot(m) * (P + PSTAT);
        float* scr = S.H[0];
        __syncthreads();
        if (want_grad) {
#pragma unroll
            for (int l = 0; l < DEEP_NH; ++l)
                if (l < nh)
#pragma unroll
                    for (int r = 0; r < RK; ++r)
#pragma unroll
                        for (int c = 0; c < 4; ++c) part[L.wh(l) + (ty * RK + r) * HID + col0 + c] = gW[l][r][c];
            deep_flush_biases<HID>(part, scr, nh, L.B0, L.bh(0), gB);
            if (tid < DA) part[L.bo() + tid] = gB2, part[L.ls() + tid] = gLS;
        }
        deep_flush_tail<DO, DA, HID>(A, sc, P, L.wo(), m, invN, want_grad, part, scr, S.red, S.last, gW0p, gW2p, s_obj, s_kl,
                                     s_ratio, DeepGradEpilogue{A, th, m, P});
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
        // ---- layer 0: H_0 = act(X W0 + b0)                       (policies/networks/mlp.py:96-117)
        {
            float acc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.W.B0 + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
            gemm_tile_smallk<DO, DOP, HID, RM>(S.X, S.W.W0, row0, col0, acc);
#pragma unroll
            for (int i = 0; i < RM; ++i)
                *reinterpret_cast<float4*>(S.H[0] + (row0 + i) * LD + col0) =
                    make_float4(Act::f(acc[i][0]), Act::f(acc[i][1]), Act::f(acc[i][2]), Act::f(acc[i][3]));
        }
        // ---- hidden layers: H_{l+1} = act(H_l W_{l+1} + b_{l+1})
#pragma unroll
        for (int l = 0; l < DEEP_NH; ++l) {
            if (l >= nh) break;
            __syncthreads();
            float acc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.W.BH[l] + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
            gemm_tile<HID, LD, LDW, RM>(S.H[l], S.W.WH[l], row0, col0, acc);
#pragma unroll
            for (int i = 0; i < RM; ++i)
                *reinterpret_cast<float4*>(S.H[l + 1] + (row0 + i) * LD + col0) =
                    make_float4(Act::f(acc[i][0]), Act::f(acc[i][1]), Act::f(acc[i][2]), Act::f(acc[i][3]));
        }
        __syncthreads();
        // ---- output layer + Gaussian head: 4 threads per sample row
        {
            float mu[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = 0.f;
#pragma unroll
            for (int k4 = 0; k4 < QW / 4; ++k4) {
                const int j = rq * QW + 4 * k4;
                const float4 h = *reinterpret_cast<const float4*>(HL + rb * LD + j);
#pragma unroll
                for (int d = 0; d < DA; ++d) {
                    mu[d] = fmaf(h.x, S.W.WO[(j + 0) * DA + d], mu[d]);
                    mu[d] = fmaf(h.y, S.W.WO[(j + 1) * DA + d], mu[d]);
                    mu[d] = fmaf(h.z, S.W.WO[(j + 2) * DA + d], mu[d]);
                    mu[d] = fmaf(h.w, S.W.WO[(j + 3) * DA + d], mu[d]);
                }
            }
#pragma unroll
            for (int d = 0; d < DA; ++d) {
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 1);
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 2);
                mu[d] += S.W.BO[d];
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
        // ---- output-layer gradients (column role)
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float h = HL[b * LD + cj];
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
        // ---- D_last = (DMU W_out^T) * act'(H_last), in place; strided columns
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            const int b = row0 + i;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int j = tx + TX * c;
                float dh = 0.f;
#pragma unroll
                for (int d = 0; d < DA; ++d) dh = fmaf(S.DMU[b * DA + d], S.W.WO[j * DA + d], dh);
                const float o = dh * Act::d(HL[b * LD + j]);
#pragma unroll
                for (int l = 0; l <= DEEP_NH; ++l)
                    if (l == nh) gB[l][c] += o;
                HL[b * LD + j] = o;
            }
        }
        // ---- hidden layers, top down: gW_l += H_l^T D_{l+1};  D_l = (D_{l+1} W_{l+1}^T) * act'(H_l)
#pragma unroll
        for (int l = DEEP_NH - 1; l >= 0; --l) {
            if (l >= nh) continue;
            __syncthreads();
            wgrad_tile<LD, RK>(S.H[l], S.H[l + 1], ty * RK, col0, nb, gW[l]);
            float acc[RM][4];
#pragma unroll
            for (int i = 0; i < RM; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
            gemm_tile_t<HID, LD, LDW, TX, RM>(S.H[l + 1], S.W.WH[l], row0, tx, acc);
            __syncthreads();   // every read of H_l is done before it is overwritten
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                const int b = row0 + i;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int j = tx + TX * c;
                    const float o = acc[i][c] * Act::d(S.H[l][b * LD + j]);
                    gB[l][c] += o;
                    S.H[l][b * LD + j] = o;
                }
            }
        }
        __syncthreads();
        // ---- gW0 += X^T D_0 (column role)
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float d1 = S.H[0][b * LD + cj];
#pragma unroll
                for (int i = 0; i < DO; ++i) gW0p[i] = fmaf(S.X[b * DOP + i], d1, gW0p[i]);
            }
        }
    }
    if (cur_m >= 0) flush(cur_m);
}

template <int DO, int DA, int HID, class Act, int ADV>
__global__ void __launch_bounds__(PT_THREADS) policy_grad_deep_kernel(PolicyArgs A, int nh) {
    deep_grad_body<DO, DA, HID, Act, ADV>(A, nh);
}

// ------------------------------------------------------------------------------------------------- Hessian-vector product
// out = vec - inner_lr * H vec + kl_coeff * grad KL, as policy_hvp_body: R_l = tangent of H_l; D_l / C_l = backprop of the
// surrogate / combined signal, written over H_l / R_l.
template <int DO, int DA, int HID>
struct DeepHvpSmem {
    static constexpr int DOP = DOPad<DO>::V, LD = TileCfg<HID>::LD;
    DeepW<DO, DA, HID> W, V;
    float H[DEEP_NH + 1][TB * LD];     // also flush scratch (with R)
    float R[DEEP_NH + 1][TB * LD];
    float X[TB * DOP];
    float DMU[TB * DA];
    float CMU[TB * DA];
    float CLS[TB * DA];
    float red[3 * (PT_THREADS / 32)];
    int last;
};

template <int DO, int DA, int HID, class Act>
__device__ __forceinline__ void deep_hvp_body(const PolicyArgs& A, int nh) {
    using C = TileCfg<HID>;
    using R = RoleCfg<HID>;
    using SM = DeepHvpSmem<DO, DA, HID>;
    constexpr int LD = C::LD, RM = C::RM, RK = C::RK, TX = C::TX, DOP = SM::DOP, LDW = DeepW<DO, DA, HID>::LDW;
    constexpr int BPP = R::BPP, QW = R::QW;
    const DeepLayout<DO, DA, HID> L{nh};
    const int P = L.P();

    extern __shared__ __align__(16) unsigned char smem_raw[];
    SM& S = *reinterpret_cast<SM*>(smem_raw);

    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int row0 = ty * RM, col0 = tx * 4;
    const int rb = tid >> 2, rq = tid & 3;
    const int cj = tid % HID, cp = tid / HID;
    const int dO = obs_dim_of<DO, DA>(A), dA = act_dim_of<DO, DA>(A);
    const UniformSched sc(A.M, A.N, A.q, A.kmax, TB);
    const int N = A.N;
    const float kl_eff = kl_coeff_eff(A);
    float invN = 1.0f / (float)N;
    int Nm = N;
    const float ac = -A.inner_lr;
    const float* th = nullptr;
    const float* vg = nullptr;
    HeadIn<DA> hin;
    float rls[DA];
    float* HL = S.H[nh];
    float* RL = S.R[nh];

    float gWc[DEEP_NH][RK][4], gWa[DEEP_NH][RK][4], gB[DEEP_NH + 1][4], gW0p[DO], gW2p[DA];
    float gB2 = 0.f, gLS = 0.f;
    float s_obj, s_kl, s_ratio;
    auto zero_acc = [&]() {
#pragma unroll
        for (int l = 0; l < DEEP_NH; ++l)
#pragma unroll
            for (int r = 0; r < RK; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) gWc[l][r][c] = gWa[l][r][c] = 0.f;
#pragma unroll
        for (int l = 0; l <= DEEP_NH; ++l) gB[l][0] = gB[l][1] = gB[l][2] = gB[l][3] = 0.f;
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
        vg = A.vec + (int64_t)m * P;
        __syncthreads();
        if (first || A.param_stride != 0) deep_stage(S.W, L, [&](int i) { return __ldg(th + i); });
        deep_stage(S.V, L, [&](int i) {       // the direction H is applied to: alpha * vec with per-parameter step sizes
            const float v = __ldcg(vg + i);
            return A.step_size ? __ldg(A.step_size + i) * v : v;
        });
        __syncthreads();
        head_setup<DA>(A, S.W.LS, m, dA, hin, nullptr);
#pragma unroll
        for (int d = 0; d < DA; ++d) rls[d] = S.V.LS[d] * hin.ls_mask[d];
    };
    auto flush = [&](int m) {
        float* part = A.partial + (int64_t)sc.my_slot(m) * (P + PSTAT);
        float* scr = S.H[0];
        __syncthreads();
#pragma unroll
        for (int l = 0; l < DEEP_NH; ++l)
            if (l < nh)
#pragma unroll
                for (int r = 0; r < RK; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        part[L.wh(l) + (ty * RK + r) * HID + col0 + c] = gWc[l][r][c] + ac * gWa[l][r][c];
        deep_flush_biases<HID>(part, scr, nh, L.B0, L.bh(0), gB);
        if (tid < DA) part[L.bo() + tid] = gB2, part[L.ls() + tid] = gLS;
        deep_flush_tail<DO, DA, HID>(A, sc, P, L.wo(), m, invN, true, part, scr, S.red, S.last, gW0p, gW2p, s_obj, s_kl, s_ratio,
                                     DeepHvpEpilogue{A, vg, m, P});
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
        // ---- layer 0 and its tangent: H_0 = act(X W0 + b0); R_0 = act'(H_0) * (X V0 + vb0)
        {
            float acc[RM][4], racc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.W.B0 + col0);
            const float4 rv = *reinterpret_cast<const float4*>(S.V.B0 + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
                racc[i][0] = rv.x, racc[i][1] = rv.y, racc[i][2] = rv.z, racc[i][3] = rv.w;
            }
            gemm_tile_smallk<DO, DOP, HID, RM>(S.X, S.W.W0, row0, col0, acc);
            gemm_tile_smallk<DO, DOP, HID, RM>(S.X, S.V.W0, row0, col0, racc);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                float h[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) h[c] = Act::f(acc[i][c]);
                *reinterpret_cast<float4*>(S.H[0] + (row0 + i) * LD + col0) = make_float4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<float4*>(S.R[0] + (row0 + i) * LD + col0) =
                    make_float4(Act::d(h[0]) * racc[i][0], Act::d(h[1]) * racc[i][1], Act::d(h[2]) * racc[i][2],
                                Act::d(h[3]) * racc[i][3]);
            }
        }
        // ---- hidden layers and tangents: R_{l+1} = act'(H_{l+1}) * (R_l W + H_l V + vb)
#pragma unroll
        for (int l = 0; l < DEEP_NH; ++l) {
            if (l >= nh) break;
            __syncthreads();
            float acc[RM][4], racc[RM][4];
            const float4 bv = *reinterpret_cast<const float4*>(S.W.BH[l] + col0);
            const float4 rv = *reinterpret_cast<const float4*>(S.V.BH[l] + col0);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                acc[i][0] = bv.x, acc[i][1] = bv.y, acc[i][2] = bv.z, acc[i][3] = bv.w;
                racc[i][0] = rv.x, racc[i][1] = rv.y, racc[i][2] = rv.z, racc[i][3] = rv.w;
            }
            gemm_tile<HID, LD, LDW, RM>(S.H[l], S.W.WH[l], row0, col0, acc);
            gemm_tile<HID, LD, LDW, RM>(S.R[l], S.W.WH[l], row0, col0, racc);
            gemm_tile<HID, LD, LDW, RM>(S.H[l], S.V.WH[l], row0, col0, racc);
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                float h[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) h[c] = Act::f(acc[i][c]);
                *reinterpret_cast<float4*>(S.H[l + 1] + (row0 + i) * LD + col0) = make_float4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<float4*>(S.R[l + 1] + (row0 + i) * LD + col0) =
                    make_float4(Act::d(h[0]) * racc[i][0], Act::d(h[1]) * racc[i][1], Act::d(h[2]) * racc[i][2],
                                Act::d(h[3]) * racc[i][3]);
            }
        }
        __syncthreads();
        // ---- output layer, its tangent, and the Gaussian head with its tangent (row role)
        {
            float mu[DA], rmu[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = rmu[d] = 0.f;
#pragma unroll
            for (int k4 = 0; k4 < QW / 4; ++k4) {
                const int j = rq * QW + 4 * k4;
                const float4 h4 = *reinterpret_cast<const float4*>(HL + rb * LD + j);
                const float4 r4 = *reinterpret_cast<const float4*>(RL + rb * LD + j);
                const float hv[4] = {h4.x, h4.y, h4.z, h4.w}, rv[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int d = 0; d < DA; ++d) {
                        const float w2 = S.W.WO[(j + e) * DA + d];
                        mu[d] = fmaf(hv[e], w2, mu[d]);
                        rmu[d] = fmaf(rv[e], w2, fmaf(hv[e], S.V.WO[(j + e) * DA + d], rmu[d]));
                    }
            }
#pragma unroll
            for (int d = 0; d < DA; ++d) {
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 1);
                mu[d] += __shfl_xor_sync(0xffffffffu, mu[d], 2);
                rmu[d] += __shfl_xor_sync(0xffffffffu, rmu[d], 1);
                rmu[d] += __shfl_xor_sync(0xffffffffu, rmu[d], 2);
                mu[d] += S.W.BO[d];
                rmu[d] += S.V.BO[d];
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
        // ---- output layer (column role): out_Wout += H_last^T CMU + ac * R_last^T DMU ; out_bout, out_ls
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float h = HL[b * LD + cj], r = ac * RL[b * LD + cj];
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
        // ---- D_last -> H_last, C_last -> R_last (strided columns)
#pragma unroll
        for (int i = 0; i < RM; ++i) {
            const int b = row0 + i;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int j = tx + TX * c;
                float dh = 0.f, ch = 0.f;
#pragma unroll
                for (int d = 0; d < DA; ++d) {
                    const float w2 = S.W.WO[j * DA + d], v2 = S.V.WO[j * DA + d];
                    const float dm = S.DMU[b * DA + d];
                    dh = fmaf(dm, w2, dh);
                    ch = fmaf(S.CMU[b * DA + d], w2, fmaf(ac * dm, v2, ch));
                }
                const float h = HL[b * LD + j], r = RL[b * LD + j];
                const float c2 = act_hvp_back<Act>(ch, dh, h, r, ac);
#pragma unroll
                for (int l = 0; l <= DEEP_NH; ++l)
                    if (l == nh) gB[l][c] += c2;
                HL[b * LD + j] = dh * Act::d(h);
                RL[b * LD + j] = c2;
            }
        }
        // ---- hidden layers, top down: out_W += H_l^T C_{l+1} + ac * R_l^T D_{l+1};
        //      dH_l = D_{l+1} W^T ; CdH_l = C_{l+1} W^T + ac * D_{l+1} V^T ; D_l, C_l -> H_l, R_l
#pragma unroll
        for (int l = DEEP_NH - 1; l >= 0; --l) {
            if (l >= nh) continue;
            __syncthreads();
            wgrad_tile<LD, RK>(S.H[l], S.R[l + 1], ty * RK, col0, nb, gWc[l]);
            wgrad_tile<LD, RK>(S.R[l], S.H[l + 1], ty * RK, col0, nb, gWa[l]);
            float dh[RM][4], ch[RM][4];
#pragma unroll
            for (int i = 0; i < RM; ++i)
#pragma unroll
                for (int c = 0; c < 4; ++c) dh[i][c] = ch[i][c] = 0.f;
            gemm_tile_t<HID, LD, LDW, TX, RM>(S.H[l + 1], S.V.WH[l], row0, tx, ch);
#pragma unroll
            for (int i = 0; i < RM; ++i)
#pragma unroll
                for (int c = 0; c < 4; ++c) ch[i][c] *= ac;
            gemm_tile_t<HID, LD, LDW, TX, RM>(S.R[l + 1], S.W.WH[l], row0, tx, ch);
            gemm_tile_t<HID, LD, LDW, TX, RM>(S.H[l + 1], S.W.WH[l], row0, tx, dh);
            __syncthreads();   // all reads of H_l / R_l are done
#pragma unroll
            for (int i = 0; i < RM; ++i) {
                const int b = row0 + i;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int j = tx + TX * c;
                    const float h = S.H[l][b * LD + j], r = S.R[l][b * LD + j];
                    const float c1 = act_hvp_back<Act>(ch[i][c], dh[i][c], h, r, ac);
                    gB[l][c] += c1;
                    S.H[l][b * LD + j] = dh[i][c] * Act::d(h);
                    S.R[l][b * LD + j] = c1;
                }
            }
        }
        __syncthreads();
        // ---- out_W0 += X^T C_0 (column role)
        {
            const int b0 = cp * BPP;
#pragma unroll 4
            for (int bb = 0; bb < BPP; ++bb) {
                const int b = b0 + bb;
                const float c1 = S.R[0][b * LD + cj];
#pragma unroll
                for (int i = 0; i < DO; ++i) gW0p[i] = fmaf(S.X[b * DOP + i], c1, gW0p[i]);
            }
        }
    }
    if (cur_m >= 0) flush(cur_m);
}

template <int DO, int DA, int HID, class Act>
__global__ void __launch_bounds__(PT_THREADS) policy_hvp_deep_kernel(PolicyArgs A, int nh) {
    deep_hvp_body<DO, DA, HID, Act>(A, nh);
}

// ------------------------------------------------------------------------------------------------------------- forward
// mean for arbitrary obs: one warp per sample, lane owns hidden units lane + 32 u, activations exchanged through a
// per-warp double buffer
template <int DO, int DA, int HID, class Act>
__global__ void __launch_bounds__(128) policy_forward_deep_kernel(int M, int N, const float* params, int64_t stride,
                                                                   const float* obs, float* mean, int obs_dim, int act_dim,
                                                                   int nh) {
    constexpr bool BUCKET = IsBucket<DO, DA>::value;
    constexpr int NU = HID / 32;
    constexpr int PMAX = DO * HID + HID + DEEP_NH * (HID * HID + HID) + HID * DA + 2 * DA;
    const DeepLayout<DO, DA, HID> L{nh};
    const int dO = BUCKET ? obs_dim : DO, dA = BUCKET ? act_dim : DA;
    __shared__ float sP[PMAX];
    __shared__ float sh[4][2][HID];
    const int m = blockIdx.y, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const float* th = params + (int64_t)m * stride;
    for (int i = threadIdx.x; i < L.P(); i += blockDim.x) sP[i] = __ldg(th + i);
    __syncthreads();
    for (int n = blockIdx.x * 4 + w; n < N; n += gridDim.x * 4) {
        const float* o = obs + ((int64_t)m * N + n) * dO;
        float h[NU];
#pragma unroll
        for (int u = 0; u < NU; ++u) {
            const int j = lane + 32 * u;
            float z = sP[L.B0 + j];
            for (int i = 0; i < dO; ++i) z = fmaf(__ldg(o + i), sP[L.W0 + i * HID + j], z);
            h[u] = Act::f(z);
            sh[w][0][j] = h[u];
        }
        __syncwarp();
        for (int l = 0; l < nh; ++l) {
            const float* hin = sh[w][l & 1];
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                const int j = lane + 32 * u;
                float z = sP[L.bh(l) + j];
                for (int k = 0; k < HID; ++k) z = fmaf(hin[k], sP[L.wh(l) + k * HID + j], z);
                h[u] = Act::f(z);
            }
#pragma unroll
            for (int u = 0; u < NU; ++u) sh[w][(l + 1) & 1][lane + 32 * u] = h[u];
            __syncwarp();
        }
        float mu[DA];
#pragma unroll
        for (int d = 0; d < DA; ++d) mu[d] = 0.f;
#pragma unroll
        for (int u = 0; u < NU; ++u)
#pragma unroll
            for (int d = 0; d < DA; ++d) mu[d] = fmaf(h[u], sP[L.wo() + (lane + 32 * u) * DA + d], mu[d]);
#pragma unroll
        for (int d = 0; d < DA; ++d) {
            float s = warp_sum(mu[d]) + sP[L.bo() + d];
            if constexpr (Act::OUT_TANH) s = ActTanh::f(s);
            if (lane == d && d < dA) mean[((int64_t)m * N + n) * dA + d] = s;
        }
        __syncwarp();
    }
}

}  // namespace promp
