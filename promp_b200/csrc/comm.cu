// Small-vector collectives over NVLink peer memory (the meta-gradient is 18-23 KB: pure latency).
//
// Every rank owns one IPC-exported buffer with a low-latency receive area [2 slots][world senders][cap] of 64-bit words
// {float value, uint32 epoch}.  A call (epoch e, slot e & 1): every thread stores its element - value and epoch in ONE
// 8-byte store - into all ranks' receive areas (remote stores over NVLink), then polls its own receive words until they
// carry epoch e and sums them in RANK ORDER -> every rank gets the bitwise identical result.  No flags, no system fences,
// no grid-wide barrier; the cost is one one-way NVLink latency.  Plain kernel launches, so - unlike an NCCL call in this
// PyTorch build - they sit inside the CUDA graph of a meta-iteration; the epoch counter lives in device memory and advances
// on every replay.  Two slots are enough: a rank can only start epoch e+2 after every peer has sent e+1, i.e. has finished
// reading epoch e.  A peer that does not show up within ~2 s sets a sticky error word and the result is NaN-poisoned.
#include <string.h>
#include "common.cuh"

namespace promp {

constexpr int COMM_MAX_SLICES = 64;      // CTAs of the fused meta-update kernel (256 parameters each: P <= 16384)

struct CommLayout {
    __host__ __device__ static int64_t data_off(int slot, int cap) { return (int64_t)slot * cap; }
    __host__ __device__ static int64_t flag_off(int slot, int cap, int world) { return 2 * (int64_t)cap + (int64_t)slot * world; }
    // per-slice arrival flags of the fused kernels: [slot][rank][slice], behind the one-shot all-reduce's flags
    __host__ __device__ static int64_t slice_flag_off(int slot, int cap, int world, int rank, int slice) {
        return 2 * (int64_t)cap + 2 * (int64_t)world + ((int64_t)slot * world + rank) * COMM_MAX_SLICES + slice;
    }
    // low-latency receive area of the fused kernels: [slot][sender rank][cap] 64-bit words {float value, uint32 epoch}
    // (float offset of word (slot, rank, i); the region starts 8-byte aligned behind the flag arrays)
    __host__ __device__ static int64_t ll_base(int cap, int world) {
        const int64_t o = 2 * (int64_t)cap + 2 * (int64_t)world + 2 * (int64_t)world * COMM_MAX_SLICES;
        return (o + 1) & ~(int64_t)1;
    }
    __host__ __device__ static int64_t ll_word(int slot, int cap, int world, int rank, int i) {
        return ((int64_t)slot * world + rank) * cap + i;
    }
};

// One value of the low-latency exchange: the payload and the epoch travel in ONE 8-byte store (atomic over NVLink), so the
// receiver polls the data words themselves - no flags, no __threadfence_system, one one-way NVLink latency per exchange.
// A rank can only be one epoch ahead of the slowest reader (it needs everybody's epoch e+1 data to finish e+1, and a rank
// sends e+1 only after consuming e), so two slots suffice.
__device__ __forceinline__ void ll_send(float* const* peers, int world, int rank, int cap, int slot, int i, float v, uint32_t epoch) {
    const unsigned long long w = ((unsigned long long)epoch << 32) | (unsigned long long)__float_as_uint(v);
    for (int r = 0; r < world; ++r) {
        volatile unsigned long long* dst =
            reinterpret_cast<volatile unsigned long long*>(peers[r] + CommLayout::ll_base(cap, world)) +
            CommLayout::ll_word(slot, cap, world, rank, i);
        *dst = w;
    }
}
// rank-ordered sum of everybody's value i; false (and *error_flag = 1) if a peer does not show up within ~2 s
__device__ __forceinline__ bool ll_recv_sum(float* const* peers, int world, int rank, int cap, int slot, int i, uint32_t epoch,
                                            uint32_t* error_flag, float* out) {
    const volatile unsigned long long* base =
        reinterpret_cast<const volatile unsigned long long*>(peers[rank] + CommLayout::ll_base(cap, world));
    float s = 0.f;
    const long long t0 = clock64();
    for (int r = 0; r < world; ++r) {
        const volatile unsigned long long* src = base + CommLayout::ll_word(slot, cap, world, r, i);
        unsigned long long w = *src;
        while ((uint32_t)(w >> 32) != epoch) {
            if (clock64() - t0 > 4000000000LL) {
                *error_flag = 1;
                return false;
            }
            w = *src;
        }
        s += __uint_as_float((uint32_t)w);
    }
    *out = s;
    return true;
}

// Generic small all-reduce (TRPO gradients / scalars, misc): one element per thread through the low-latency exchange.
__global__ void __launch_bounds__(256) allreduce_ll_kernel(int world, int rank, int n, int cap, const float* in, float* out,
                                                            float scale, float* const* peers, uint32_t* epoch_ptr,
                                                            uint32_t* error_flag, unsigned int* ticket) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    const uint32_t epoch = *epoch_ptr + 1;
    const int slot = epoch & 1;
    if (i < n) {
        ll_send(peers, world, rank, cap, slot, i, in[i], epoch);
        float s;
        const bool ok = *reinterpret_cast<volatile uint32_t*>(error_flag) == 0 &&
                        ll_recv_sum(peers, world, rank, cap, slot, i, epoch, error_flag, &s);
        out[i] = ok ? s * scale : __int_as_float(0x7fc00000);     // a missing peer poisons the result (P2PComm.check raises)
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned int old = atomicAdd(ticket, 1u);
        if (old == gridDim.x - 1) {          // every CTA has read the epoch before taking its ticket
            *epoch_ptr = epoch;
            *ticket = 0u;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused outer update of one PPO / Adam epoch: per-task meta-gradients v [M, P] -> mean over this rank's tasks -> sum over
// ranks through NVLink peer memory -> TF1 Adam on theta, ONE launch (was: reduce_tasks + all-reduce + adam + step
// increment = 4 launches, the all-reduce on a single CTA).  CTA b owns parameters [256 b, 256 b + 256): slices are
// independent: every THREAD pushes its element to all ranks and polls its own receive words (low-latency protocol below:
// no flags, no fences, no grid- or block-wide barrier), so the exchange of one slice overlaps the task reduction of the next.  Rank-ordered sums: every rank computes bitwise identical gradients and
// parameters.  `step` and the exchange epoch are read by every CTA before it takes its completion ticket; the last ticket
// holder publishes the incremented values, so no CTA can observe them half-way.
struct MetaUpdateArgs {
    int M, P;
    const float* v;          // [M, P] per-task gradients (local tasks)
    float scale;             // 1 / (M * world)
    float* grad_out;         // [P] reduced meta-gradient (may be NULL)
    float* theta; float* mm; float* vv; int32_t* step;
    float lr, b1, b2, eps;
    int world, rank, cap;
    float* const* peers; uint32_t* epoch_ptr; uint32_t* error_flag;
    unsigned int* ticket;
};

// task sum of column `col` of an [M, P] array in task order (bit-identical to promp_reduce_tasks), 16 independent L2 loads in
// flight per round trip
__device__ __forceinline__ float task_sum(const float* col, int M, int P) {
    float g = 0.f;
    int m = 0;
    for (; m + 16 <= M; m += 16) {
        float x[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) x[u] = __ldcg(col + (int64_t)(m + u) * P);
#pragma unroll
        for (int u = 0; u < 16; ++u) g += x[u];
    }
    {
        float x[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) x[u] = (m + u < M) ? __ldcg(col + (int64_t)(m + u) * P) : 0.f;
#pragma unroll
        for (int u = 0; u < 16; ++u)
            if (m + u < M) g += x[u];
    }
    return g;
}

__global__ void __launch_bounds__(256) meta_update_kernel(MetaUpdateArgs A) {
    const int tid = threadIdx.x, b = blockIdx.x, p = b * 256 + tid;
    const int t = *A.step + 1;
    float g = 0.f;
    if (p < A.P) g = task_sum(A.v + p, A.M, A.P) * A.scale;
    uint32_t epoch = 0;
    if (A.world > 1) {
        epoch = *A.epoch_ptr + 1;
        const int slot = epoch & 1;
        if (p < A.P) {
            ll_send(A.peers, A.world, A.rank, A.cap, slot, p, g, epoch);
            float s;
            // a failed exchange poisons the gradient: a partial sum must never reach Adam silently (P2PComm.check raises)
            g = (*reinterpret_cast<volatile uint32_t*>(A.error_flag) == 0 &&
                 ll_recv_sum(A.peers, A.world, A.rank, A.cap, slot, p, epoch, A.error_flag, &s)) ? s : __int_as_float(0x7fc00000);
        }
    }
    if (p < A.P) {
        if (A.grad_out) A.grad_out[p] = g;
        // tf.train.AdamOptimizer: lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t)
        const float lr_t = A.lr * sqrtf(1.f - powf(A.b2, (float)t)) / (1.f - powf(A.b1, (float)t));
        const float mn = A.b1 * A.mm[p] + (1.f - A.b1) * g;
        const float vn = A.b2 * A.vv[p] + (1.f - A.b2) * g * g;
        A.mm[p] = mn;
        A.vv[p] = vn;
        A.theta[p] = A.theta[p] - lr_t * mn / (sqrtf(vn) + A.eps);
    }
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        const unsigned int old = atomicAdd(A.ticket, 1u);
        if (old == gridDim.x - 1) {          // every CTA has read step / epoch before taking its ticket
            *A.step = t;
            if (A.world > 1) *A.epoch_ptr = epoch;
            *A.ticket = 0u;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Meta-SGD (trainable per-parameter inner step sizes alpha): the same fused outer update over the concatenated gradient
// [theta; alpha] (2P values), one Adam step counter for both.  Element e < P is theta's task mean, as in meta_update_kernel;
// element P + i is alpha's gradient
//   dJ/dalpha_i = -scale * sum_m sum_s lam_s[m, i] * g_s[m, i]
// (lam_s = the direction entering HVP stage s, g_s = the inner gradient of stage s: theta_{s+1} = theta_s - alpha * g_s).
// With grad_in set, the summed [2P] gradient is given (the NCCL path: promp_reduce_tasks_sgd + all-reduce) and only Adam runs.
constexpr int SGD_MAX_PAIRS = 6;
struct MetaUpdateSgdArgs {
    int M, P, n_pairs;
    const float* v;                        // [M, P] per-task theta gradients (local tasks)
    const float* lam[SGD_MAX_PAIRS];       // [M, P] each
    const float* gs[SGD_MAX_PAIRS];        // [M, P] each
    const float* grad_in;                  // [2P] or NULL
    float scale;                           // 1 / (M * world)
    float* grad_out;                       // [2P] or NULL
    float* prm[2]; float* mm[2]; float* vv[2];     // theta / alpha and their Adam slots
    int32_t* step;
    float lr, b1, b2, eps;
    int world, rank, cap;
    float* const* peers; uint32_t* epoch_ptr; uint32_t* error_flag;
    unsigned int* ticket;
};

// element e of the local [theta; alpha] gradient (scaled, not yet summed over ranks)
__device__ __forceinline__ float sgd_local_grad(const MetaUpdateSgdArgs& A, int e) {
    if (e < A.P) return task_sum(A.v + e, A.M, A.P) * A.scale;
    // per task the sum over inner steps, then the tasks in task order; 4 tasks' loads in flight per round trip
    constexpr int U = 4;
    const int i = e - A.P;
    float g = 0.f;
#pragma unroll 1
    for (int m0 = 0; m0 < A.M; m0 += U) {
        float t[U];
#pragma unroll
        for (int u = 0; u < U; ++u) t[u] = 0.f;
#pragma unroll
        for (int s = 0; s < SGD_MAX_PAIRS; ++s) {
            if (s >= A.n_pairs) break;
            float l[U], x[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int64_t o = (int64_t)(m0 + u) * A.P + i;
                l[u] = m0 + u < A.M ? __ldcg(A.lam[s] + o) : 0.f;
                x[u] = m0 + u < A.M ? __ldcg(A.gs[s] + o) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < U; ++u) t[u] = fmaf(l[u], x[u], t[u]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (m0 + u < A.M) g += t[u];
    }
    return -g * A.scale;
}

__global__ void __launch_bounds__(256) reduce_tasks_sgd_kernel(MetaUpdateSgdArgs A, int e0) {
    const int e = e0 + blockIdx.x * 256 + threadIdx.x;
    if (e < 2 * A.P) A.grad_out[e] = sgd_local_grad(A, e);
}

__global__ void __launch_bounds__(256) meta_update_sgd_kernel(MetaUpdateSgdArgs A) {
    const int tid = threadIdx.x, e = blockIdx.x * 256 + tid;
    const int t = *A.step + 1;
    const int n = 2 * A.P;
    float g = 0.f;
    if (e < n) g = A.grad_in ? A.grad_in[e] : sgd_local_grad(A, e);
    uint32_t epoch = 0;
    if (A.world > 1) {          // one exchange of the whole [theta; alpha] vector per Adam epoch
        epoch = *A.epoch_ptr + 1;
        const int slot = epoch & 1;
        if (e < n) {
            ll_send(A.peers, A.world, A.rank, A.cap, slot, e, g, epoch);
            float s;
            g = (*reinterpret_cast<volatile uint32_t*>(A.error_flag) == 0 &&
                 ll_recv_sum(A.peers, A.world, A.rank, A.cap, slot, e, epoch, A.error_flag, &s)) ? s : __int_as_float(0x7fc00000);
        }
    }
    if (e < n) {
        if (A.grad_out) A.grad_out[e] = g;
        const int h = e >= A.P, p = e - h * A.P;
        float* const th = A.prm[h];
        float* const mm = A.mm[h];
        float* const vv = A.vv[h];
        const float lr_t = A.lr * sqrtf(1.f - powf(A.b2, (float)t)) / (1.f - powf(A.b1, (float)t));
        const float mn = A.b1 * mm[p] + (1.f - A.b1) * g;
        const float vn = A.b2 * vv[p] + (1.f - A.b2) * g * g;
        mm[p] = mn;
        vv[p] = vn;
        th[p] = th[p] - lr_t * mn / (sqrtf(vn) + A.eps);
    }
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        const unsigned int old = atomicAdd(A.ticket, 1u);
        if (old == gridDim.x - 1) {
            *A.step = t;
            if (A.world > 1) *A.epoch_ptr = epoch;
            *A.ticket = 0u;
        }
    }
}

// [loss, inner KLs.., outer KL] (promp_meta_loss_terms) with the sum over ranks fused in: local means (already scaled by
// 1 / M_global) -> peer-memory exchange -> rank-ordered sum -> KL penalty added to the loss.  One CTA.
__global__ void __launch_bounds__(256) meta_loss_terms_p2p_kernel(int S, int M, const float* __restrict__ stats_all, float inv_mg,
                                                                   const float* __restrict__ coeff, int n_out, float* __restrict__ out,
                                                                   int world, int rank, int cap, float* const* peers,
                                                                   uint32_t* epoch_ptr, uint32_t* error_flag) {
    __shared__ float terms[8];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
    if (w < S + 1) {
        const int row = (w == 0 || w == S) ? S - 1 : w - 1;       // term 0: outer surr; 1..S-1: inner KLs; S: outer KL
        const int col = (w == 0) ? 0 : 1;
        float a = 0.f;
        for (int m = lane; m < M; m += 32) a += stats_all[((int64_t)row * M + m) * 4 + col];
        a = warp_sum(a) * inv_mg;
        if (lane == 0) terms[w] = a;
    }
    __syncthreads();
    const uint32_t epoch = *epoch_ptr + 1;
    const int slot = epoch & 1;
    if (tid < S + 1) {
        ll_send(peers, world, rank, cap, slot, tid, terms[tid], epoch);
        float s;
        terms[tid] = (*reinterpret_cast<volatile uint32_t*>(error_flag) == 0 &&
                      ll_recv_sum(peers, world, rank, cap, slot, tid, epoch, error_flag, &s)) ? s : __int_as_float(0x7fc00000);
    }
    __syncthreads();
    if (tid == 0) {
        float loss = terms[0];
        if (coeff && S > 1) {
            float pen = 0.f;
            for (int s = 0; s < S - 1; ++s) pen += coeff[s] * terms[1 + s];
            loss += pen / (float)(S - 1);
        }
        out[0] = loss;
        for (int i = 1; i < n_out && i < S + 1; ++i) out[i] = terms[i];
        *epoch_ptr = epoch;
    }
}

}  // namespace promp

using namespace promp;

extern "C" int64_t promp_comm_buffer_bytes(int world, int capacity_floats) {
    // [2 data slots | one-shot flags | per-slice flags | low-latency receive area 2 x world x cap 64-bit words]
    return CommLayout::ll_base(capacity_floats, world) * 4 + 2 * (int64_t)world * capacity_floats * 8;
}

// The ONE place the library allocates: communication buffers must be whole cudaMalloc allocations to be IPC-exportable.
extern "C" int promp_comm_alloc(int64_t bytes, void** dev_ptr_host) {
    PROMP_REQUIRE(bytes > 0 && dev_ptr_host, "promp_comm_alloc: bad arguments");
    PROMP_CUDA(cudaMalloc(dev_ptr_host, (size_t)bytes));
    PROMP_CUDA(cudaMemset(*dev_ptr_host, 0, (size_t)bytes));
    return PROMP_OK;
}
extern "C" int promp_comm_free(void* dev_ptr) {
    PROMP_CUDA(cudaFree(dev_ptr));
    return PROMP_OK;
}
extern "C" int promp_ipc_get_handle(void* dev_ptr, void* handle64_host) {
    PROMP_REQUIRE(dev_ptr && handle64_host, "promp_ipc_get_handle: bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    PROMP_CUDA(cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle64_host), dev_ptr));
    return PROMP_OK;
}
extern "C" int promp_ipc_open_handle(const void* handle64_host, void** dev_ptr_host) {
    PROMP_REQUIRE(handle64_host && dev_ptr_host, "promp_ipc_open_handle: bad arguments");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64_host, sizeof(h));
    PROMP_CUDA(cudaIpcOpenMemHandle(dev_ptr_host, h, cudaIpcMemLazyEnablePeerAccess));
    return PROMP_OK;
}
extern "C" int promp_ipc_close_handle(void* dev_ptr) {
    PROMP_CUDA(cudaIpcCloseMemHandle(dev_ptr));
    return PROMP_OK;
}

extern "C" int promp_allreduce_p2p(int world, int rank, int n, int capacity_floats, const float* in, float* out, float scale,
                                   void* const* peers_dev, uint32_t* epoch_dev, uint32_t* error_flag_dev, uint32_t* ticket_dev,
                                   void* stream) {
    PROMP_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world, "promp_allreduce_p2p: bad world/rank");
    PROMP_REQUIRE(n > 0 && n <= capacity_floats, "promp_allreduce_p2p: n=%d exceeds the buffer capacity %d", n, capacity_floats);
    PROMP_REQUIRE(in && out && peers_dev && epoch_dev && error_flag_dev && ticket_dev, "promp_allreduce_p2p: null pointer argument");
    allreduce_ll_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(world, rank, n, capacity_floats, in, out, scale,
                                                                         reinterpret_cast<float* const*>(peers_dev), epoch_dev,
                                                                         error_flag_dev, ticket_dev);
    PROMP_LAUNCH_CHECK("allreduce_ll_kernel");
    return PROMP_OK;
}

extern "C" int promp_meta_update(int M, int P, const float* task_grads, float scale, float* grad_out, float* theta, float* m,
                                 float* v, int32_t* step, float lr, float beta1, float beta2, float eps, int world, int rank,
                                 int capacity_floats, void* const* peers_dev, uint32_t* epoch_dev, uint32_t* error_flag_dev,
                                 uint32_t* ticket_dev, void* stream) {
    PROMP_REQUIRE(M > 0 && P > 0 && task_grads && theta && m && v && step && ticket_dev, "promp_meta_update: bad arguments");
    PROMP_REQUIRE(P <= 256 * COMM_MAX_SLICES, "promp_meta_update: P=%d exceeds %d parameters", P, 256 * COMM_MAX_SLICES);
    PROMP_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world, "promp_meta_update: bad world/rank");
    if (world > 1) {
        PROMP_REQUIRE(peers_dev && epoch_dev && error_flag_dev && P <= capacity_floats,
                      "promp_meta_update: multi-rank call needs the peer table, epoch / error words and capacity >= P");
    }
    MetaUpdateArgs A{M, P, task_grads, scale, grad_out, theta, m, v, step, lr, beta1, beta2, eps, world, rank, capacity_floats,
                     reinterpret_cast<float* const*>(peers_dev), epoch_dev, error_flag_dev, ticket_dev};
    meta_update_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(A);
    PROMP_LAUNCH_CHECK("meta_update_kernel");
    return PROMP_OK;
}

static int sgd_pairs(MetaUpdateSgdArgs& A, const char* who, int M, int P, const float* task_grads, int n_pairs,
                     const float* const* lam, const float* const* g) {
    PROMP_REQUIRE(M > 0 && P > 0 && n_pairs >= 0 && n_pairs <= SGD_MAX_PAIRS && (n_pairs == 0 || (lam && g)),
                  "%s: bad arguments (0 <= n_pairs <= %d)", who, SGD_MAX_PAIRS);
    A.M = M; A.P = P; A.n_pairs = n_pairs; A.v = task_grads;
    for (int s = 0; s < n_pairs; ++s) {
        PROMP_REQUIRE(lam[s] && g[s], "%s: pair %d has a null pointer", who, s);
        A.lam[s] = lam[s];
        A.gs[s] = g[s];
    }
    return PROMP_OK;
}

// task_grads NULL: only the alpha half out[P, 2P) is written (the theta half comes from promp_reduce_tasks / _tasks2)
extern "C" int promp_reduce_tasks_sgd(int M, int P, const float* task_grads, int n_pairs, const float* const* lam,
                                      const float* const* g, float scale, float* out, void* stream) {
    MetaUpdateSgdArgs A{};
    const int st = sgd_pairs(A, "promp_reduce_tasks_sgd", M, P, task_grads, n_pairs, lam, g);
    if (st != PROMP_OK) return st;
    PROMP_REQUIRE(out, "promp_reduce_tasks_sgd: null output");
    A.scale = scale; A.grad_out = out;
    const int e0 = task_grads ? 0 : P;
    reduce_tasks_sgd_kernel<<<(2 * P - e0 + 255) / 256, 256, 0, (cudaStream_t)stream>>>(A, e0);
    PROMP_LAUNCH_CHECK("reduce_tasks_sgd_kernel");
    return PROMP_OK;
}

extern "C" int promp_meta_update_sgd(int M, int P, const float* task_grads, int n_pairs, const float* const* lam,
                                     const float* const* g, const float* grad_in, float scale, float* grad_out, float* theta,
                                     float* alpha, float* m, float* v, float* m_alpha, float* v_alpha, int32_t* step, float lr,
                                     float beta1, float beta2, float eps, int world, int rank, int capacity_floats,
                                     void* const* peers_dev, uint32_t* epoch_dev, uint32_t* error_flag_dev, uint32_t* ticket_dev,
                                     void* stream) {
    MetaUpdateSgdArgs A{};
    if (grad_in) {
        PROMP_REQUIRE(P > 0 && world == 1, "promp_meta_update_sgd: a given gradient needs P > 0 and world == 1");
        A.P = P; A.grad_in = grad_in;
    } else {
        const int st = sgd_pairs(A, "promp_meta_update_sgd", M, P, task_grads, n_pairs, lam, g);
        if (st != PROMP_OK) return st;
    }
    PROMP_REQUIRE(theta && alpha && m && v && m_alpha && v_alpha && step && ticket_dev, "promp_meta_update_sgd: null pointer argument");
    PROMP_REQUIRE(2 * P <= 256 * COMM_MAX_SLICES, "promp_meta_update_sgd: 2P=%d exceeds %d values", 2 * P, 256 * COMM_MAX_SLICES);
    PROMP_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world, "promp_meta_update_sgd: bad world/rank");
    if (world > 1) {
        PROMP_REQUIRE(peers_dev && epoch_dev && error_flag_dev && 2 * P <= capacity_floats,
                      "promp_meta_update_sgd: multi-rank call needs the peer table, epoch / error words and capacity >= 2P");
    }
    A.scale = scale; A.grad_out = grad_out;
    A.prm[0] = theta; A.prm[1] = alpha; A.mm[0] = m; A.mm[1] = m_alpha; A.vv[0] = v; A.vv[1] = v_alpha;
    A.step = step; A.lr = lr; A.b1 = beta1; A.b2 = beta2; A.eps = eps;
    A.world = world; A.rank = rank; A.cap = capacity_floats;
    A.peers = reinterpret_cast<float* const*>(peers_dev); A.epoch_ptr = epoch_dev; A.error_flag = error_flag_dev;
    A.ticket = ticket_dev;
    meta_update_sgd_kernel<<<(2 * P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(A);
    PROMP_LAUNCH_CHECK("meta_update_sgd_kernel");
    return PROMP_OK;
}

extern "C" int promp_meta_loss_terms_p2p(int S, int M, const float* stats_all, float inv_m_global, const float* coeff, int n_out,
                                         float* out, int world, int rank, int capacity_floats, void* const* peers_dev,
                                         uint32_t* epoch_dev, uint32_t* error_flag_dev, void* stream) {
    PROMP_REQUIRE(S >= 1 && S <= 7 && M > 0 && stats_all && out && n_out >= 1 && n_out <= S + 1,
                  "promp_meta_loss_terms_p2p: bad arguments (1 <= S <= 7 sampling phases, 1 <= n_out <= S+1)");
    PROMP_REQUIRE(world >= 2 && world <= 64 && rank >= 0 && rank < world && peers_dev && epoch_dev && error_flag_dev &&
                      capacity_floats >= 8,
                  "promp_meta_loss_terms_p2p: bad communicator arguments");
    meta_loss_terms_p2p_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(S, M, stats_all, inv_m_global, coeff, n_out, out, world, rank,
                                                                    capacity_floats, reinterpret_cast<float* const*>(peers_dev),
                                                                    epoch_dev, error_flag_dev);
    PROMP_LAUNCH_CHECK("meta_loss_terms_p2p_kernel");
    return PROMP_OK;
}
