// Tensor-core variant of policy_grad_kernel for HID = 64.
//
// The two [128 x 64] x [64 x 64] layer GEMMs of a tile (forward H1.W1 and backward D2.W1^T) run on the tensor cores as
// warpgroup MMAs (wgmma.mma_async m64nNk8 tf32) with the 3-term split  a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo  (a_hi =
// trunc_tf32(a), a_lo = a - a_hi), i.e. fp32-level accuracy at 3 MMAs per product.  Every warp of the CTA takes part:
// warp w computes rows [16 (w % 8), +16) and 64 / (NW / 8) of the 64 output columns, accumulating in registers.  The A
// operand (activations) is split into hi / lo while its fragments are loaded into registers; the B operand (weights) is
// stored once per task as hi + lo tiles that the tensor cores read from shared memory.  Activation and weight tiles sit
// in shared memory in a K-major core-matrix layout: 8x4-float core matrices (128 contiguous bytes, rows 16 B apart),
// next 8 rows at +128 B, next 4 columns at +S_c.  S_c = rows*16 + 16 bytes: the extra 16 B make the row-wise 16-byte
// stores of the epilogue, the column-wise scalar reads of the SIMT reductions and the fragment loads of the MMAs
// bank-conflict free, and the same bytes stay readable as a plain fp32 tile.  A forward result is staged through a dead
// [128 x 64] tile so that the epilogue gets one sample row per thread (64 / NQ columns each; NQ = 2 or 4 column groups =
// 256 or 512 threads per CTA); a backward result is consumed element-wise straight from the accumulator fragments.  The
// weight-gradient GEMM H1^T.D2 contracts over samples and runs on warp-level mma.sync with fragments loaded from the
// same tiles (wgrad_mma_tile below).
#pragma once
#include "mlp_tile.cuh"

namespace promp {

constexpr int TBT = 128;                      // samples per tile
constexpr int TC_HID = 64;
constexpr int SCA = TBT * 16 + 16;            // bytes between 4-column chunks of a [128 x 64] activation tile
constexpr int SCW = TC_HID * 16 + 16;         // ... of a [64 x 64] weight tile
constexpr int TILE_A_BYTES = 16 * SCA;        // 33 024
constexpr int TILE_W_BYTES = 16 * SCW;        // 16 640

__device__ __forceinline__ int core_off(int r, int c, int sc) {      // byte offset of element (r, c)
    return (c >> 2) * sc + (r >> 3) * 128 + (r & 7) * 16 + ((c & 3) << 2);
}
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }

template <int DO, int DA>
struct SmallLayout {      // the parameters other than W1, compact
    static constexpr int W0 = 0;
    static constexpr int B0 = W0 + DO * TC_HID;
    static constexpr int B1 = B0 + TC_HID;
    static constexpr int W2 = B1 + TC_HID;
    static constexpr int B2 = W2 + TC_HID * DA;
    static constexpr int LS = B2 + DA;
    static constexpr int SIZE = (LS + DA + 3) / 4 * 4;
};

template <int DO, int DA, int NQ>
struct GradTcSmem {
    static constexpr int DOP = DOPad<DO>::V;
    alignas(16) unsigned char W1T_hi[TILE_W_BYTES];   // B of the forward GEMM: rows n = output unit, K = k
    alignas(16) unsigned char W1T_lo[TILE_W_BYTES];
    alignas(16) unsigned char W1_hi[TILE_W_BYTES];    // B of the backward GEMM: rows n = k', K = j
    alignas(16) unsigned char W1_lo[TILE_W_BYTES];
    alignas(16) unsigned char A0[TILE_A_BYTES];       // H1 -> D1
    alignas(16) unsigned char A1[TILE_A_BYTES];       // H2 -> D2
    alignas(16) unsigned char LO[TILE_A_BYTES];       // Z2 (forward GEMM result) ; flush scratch
    alignas(16) float Ps[SmallLayout<DO, DA>::SIZE];
    alignas(16) float X[TBT * DOP];
    float MUP[NQ * TBT * DA];
    float DMU[TBT * DA];
    float red[3 * 4 * NQ];
    HeadIn<DA> hin;           // per-task constants of the Gaussian head (written by thread 0 in load_task)
    HeadOld<DA> hold;         // ... of the old distribution when the phase stores one log_std row per task
    int last;
};


// -------------------------------------------------------------------------------------------------------------
// Weight-gradient GEMM  acc[k][j] += sum_b A[b][k] * (scale * D[b][j])  over the 128 rows of two fp32 tiles in the
// K-major core-matrix layout, on the warp-level tensor-core path (mma.sync m16n8k8 tf32, 3xTF32 split).  This GEMM
// contracts over SAMPLES, i.e. both operands are MN-major in these tiles.  The CUDA-core version
// was bound by shared-memory wavefronts (every LDS.128 costs 4, 8 per sample row per warp for 16 FFMA); the fragment
// loads below are 12 conflict-free LDS.32 per 8 sample rows and the math leaves the FP32 pipe.
//   warp w owns the 16 x 8NT block  k in [16 (w&3), +16), j in [8NT (w>>2), +8NT)  as NT n-tiles of m16n8
//   (NT = 4 with 8 warps, 2 with 16 warps).
//   fragment column t (t+4) <-> sample 8s+2t (8s+2t+1): with the 16-byte chunk padding this makes every fragment
//   load hit 32 distinct banks (bank = 4 (g>>2) + (g&3) + 8 t).
__device__ __forceinline__ void mma_tf32_16n8k8(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(x) & 0xffffe000u;
    lo = __float_as_uint(x - __uint_as_float(hi));
}
// COLSUM: also accumulate the column sums of D (unscaled) from the B fragments: csum[nt] holds, per lane, the partial
// over this lane's sample rows for column 32 (warp>>2) + 8 nt + (lane>>2); reduce over lane&3 at flush time.
template <bool COLSUM, int NT, bool UNIT = false>
__device__ __forceinline__ void wgrad_mma_tile(const unsigned char* __restrict__ At, const unsigned char* __restrict__ Dt,
                                               float scale, int warp, int lane, float (&acc)[NT][4], float (&csum)[NT]) {
    const int g = lane >> 2, t = lane & 3;
    const int k0 = 16 * (warp & 3) + g, j0 = 8 * NT * (warp >> 2) + g;
    const unsigned char* ap = At + (k0 >> 2) * SCA + (k0 & 3) * 4 + t * 32;     // rows k0 (and k0+8: two chunks further)
    const unsigned char* dp = Dt + (j0 >> 2) * SCA + (j0 & 3) * 4 + t * 32;     // n-tile nt: two chunks further each
#pragma unroll 2
    for (int s = 0; s < TBT / 8; ++s) {
        uint32_t ah[4], al[4], bh[NT][2], bl[NT][2];
        split_tf32(*reinterpret_cast<const float*>(ap + s * 128), ah[0], al[0]);
        split_tf32(*reinterpret_cast<const float*>(ap + s * 128 + 2 * SCA), ah[1], al[1]);
        split_tf32(*reinterpret_cast<const float*>(ap + s * 128 + 16), ah[2], al[2]);
        split_tf32(*reinterpret_cast<const float*>(ap + s * 128 + 2 * SCA + 16), ah[3], al[3]);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const float d0 = *reinterpret_cast<const float*>(dp + nt * 2 * SCA + s * 128);
            const float d1 = *reinterpret_cast<const float*>(dp + nt * 2 * SCA + s * 128 + 16);
            if (COLSUM) csum[nt] += d0 + d1;
            split_tf32(UNIT ? d0 : scale * d0, bh[nt][0], bl[nt][0]);      // UNIT: scale == 1 (no multiply)
            split_tf32(UNIT ? d1 : scale * d1, bh[nt][1], bl[nt][1]);
        }
        // term-major order: consecutive MMAs hit different accumulators (no back-to-back dependent issue)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_tf32_16n8k8(acc[nt], al, bh[nt]);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_tf32_16n8k8(acc[nt], ah, bl[nt]);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) mma_tf32_16n8k8(acc[nt], ah, bh[nt]);
    }
}
// accumulator element (nt, i) of wgrad_mma_tile -> flat index into the [HID, HID] weight (row k, column j)
template <int NT>
__device__ __forceinline__ int wgrad_mma_index(int warp, int lane, int nt, int i) {
    const int g = lane >> 2, t = lane & 3;
    return (16 * (warp & 3) + g + 8 * (i >> 1)) * TC_HID + 8 * NT * (warp >> 2) + 8 * nt + 2 * t + (i & 1);
}

// -------------------------------------------------------------------------------------------------------------
// Layer GEMM  acc += A[128 x 64] . B^T  with B [64(N) x 64(K)] given as hi + lo tiles (K-major, stride SCW), A as one
// fp32 tile (K-major, stride SCA) split into hi / lo at fragment load, on Hopper's asynchronous warpgroup MMA
// (wgmma.mma_async m64nNk8 tf32, 3xTF32 split).  Warpgroup q = w >> 2 owns rows [64 (q & 1), +64) and columns
// [8 LNT (q >> 1), +8 LNT) (LNT = 8 with 8 warps: m64n64; 4 with 16 warps: m64n32), so warp w still owns rows
// [16 (w & 7), +16) and the n8 tiles [LNT (w >> 3), +LNT), and its accumulator registers have the m16n8 fragment layout
// (frag_off).  A comes from registers (conflict-free fragment loads, bank = 4 g + t); B is read by the tensor cores from
// shared memory through a no-swizzle K-major descriptor: core matrices of 8 rows x 16 B, the K-adjacent one at
// +SCW (leading byte offset), the next 8 rows at +128 B (stride byte offset).  Terms per k-step: lo.hi, hi.lo, then
// hi.hi.  The hi weight tiles hold tf32-truncated values (the tensor cores ignore the low 13 bits of a tf32 operand
// either way).
//
// layer_gemm_issue issues the MMAs as one commit group per k-step in a rolled loop and waits for each group before the
// next k-step's fragment loads overwrite the A registers it reads, so only one k-step of A fragments is live.  Keeping
// more k-steps in flight (to overlap the weight-gradient GEMM) needs distinct registers per k-step, which spilled in the
// 512-thread kernels and in the dataflow kernel.  The caller still waits (wg_wait) before it reads acc.  The weight tiles must have
// been made visible to the async proxy (wg_fence_weights, then a barrier) after their generic stores.
__device__ __forceinline__ uint64_t wg_desc(const unsigned char* p) {
    const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
    return (uint64_t)((a & 0x3ffff) >> 4) | ((uint64_t)(SCW >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);   // layout 0: no swizzle
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory"); }
constexpr int WG_DEPTH = 0;      // k-step groups left in flight: 0, as the rolled loop reuses the A registers
__device__ __forceinline__ void wg_wait_depth() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(WG_DEPTH) : "memory"); }
__device__ __forceinline__ void wg_fence_weights() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
// pins the accumulator registers at this point of the program (no use of them is moved across an issue or a wait)
template <int LNT>
__device__ __forceinline__ void wg_pin(float (&acc)[LNT][4]) {
#pragma unroll
    for (int nt = 0; nt < LNT; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) asm volatile("" : "+f"(acc[nt][i])::"memory");
}

template <int LNT>
__device__ __forceinline__ void wgmma_tf32(float (&d)[LNT][4], const uint32_t (&a)[4], uint64_t desc);
template <>
__device__ __forceinline__ void wgmma_tf32<4>(float (&d)[4][4], const uint32_t (&a)[4], uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, 1, 1, 1;\n"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<8>(float (&d)[8][4], const uint32_t (&a)[4], uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, 1, 1, 1;\n"
        : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]), "+f"(d[1][3]),
          "+f"(d[2][0]), "+f"(d[2][1]), "+f"(d[2][2]), "+f"(d[2][3]), "+f"(d[3][0]), "+f"(d[3][1]), "+f"(d[3][2]), "+f"(d[3][3]),
          "+f"(d[4][0]), "+f"(d[4][1]), "+f"(d[4][2]), "+f"(d[4][3]), "+f"(d[5][0]), "+f"(d[5][1]), "+f"(d[5][2]), "+f"(d[5][3]),
          "+f"(d[6][0]), "+f"(d[6][1]), "+f"(d[6][2]), "+f"(d[6][3]), "+f"(d[7][0]), "+f"(d[7][1]), "+f"(d[7][2]), "+f"(d[7][3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <int LNT>
__device__ __forceinline__ void layer_gemm_issue(float (&acc)[LNT][4], const unsigned char* __restrict__ a,
                                                 const unsigned char* __restrict__ b_hi, const unsigned char* __restrict__ b_lo,
                                                 int warp, int lane) {
    const int g = lane >> 2, t = lane & 3;
    const unsigned char* ap = a + (warp & 7) * 256 + g * 16 + t * 4;
    const int bo = (warp >> 3) * LNT * 128;
#pragma unroll 1      // a rolled loop keeps the fragment loads of later k-steps from being hoisted (register pressure)
    for (int s = 0; s < TC_HID / 8; ++s) {
        const uint64_t dh = wg_desc(b_hi + bo + 2 * s * SCW), dl = wg_desc(b_lo + bo + 2 * s * SCW);      // k-step s
        uint32_t ah[4], al[4];
        const unsigned char* as = ap + 2 * s * SCA;
        split_tf32(*reinterpret_cast<const float*>(as), ah[0], al[0]);
        split_tf32(*reinterpret_cast<const float*>(as + 128), ah[1], al[1]);
        split_tf32(*reinterpret_cast<const float*>(as + SCA), ah[2], al[2]);
        split_tf32(*reinterpret_cast<const float*>(as + SCA + 128), ah[3], al[3]);
        wg_fence();                                              // the A fragments were just written
        wgmma_tf32<LNT>(acc, al, dh);
        wgmma_tf32<LNT>(acc, ah, dl);
        wgmma_tf32<LNT>(acc, ah, dh);
        wg_commit();
        wg_wait_depth();
    }
}
template <int LNT>
__device__ __forceinline__ void zero_frag(float (&acc)[LNT][4]) {
#pragma unroll
    for (int nt = 0; nt < LNT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
}
// byte offset (in a [128 x 64] activation tile) of the accumulator pair acc[nt][2h], acc[nt][2h + 1] of layer_gemm_issue
template <int LNT>
__device__ __forceinline__ int frag_off(int warp, int lane, int nt, int h) {
    return core_off(16 * (warp & 7) + (lane >> 2) + 8 * h, 8 * (LNT * (warp >> 3) + nt) + 2 * (lane & 3), SCA);
}
template <int LNT>
__device__ __forceinline__ void store_frag(const float (&acc)[LNT][4], unsigned char* tile, int warp, int lane) {
#pragma unroll
    for (int nt = 0; nt < LNT; ++nt)
#pragma unroll
        for (int h = 0; h < 2; ++h)
            *reinterpret_cast<float2*>(tile + frag_off<LNT>(warp, lane, nt, h)) = make_float2(acc[nt][2 * h], acc[nt][2 * h + 1]);
}
// row r, columns [c0, c0 + CW) of an activation tile -> registers (16-byte loads)
template <int CW>
__device__ __forceinline__ void load_row(const unsigned char* tile, int r, int c0, float (&v)[CW]) {
#pragma unroll
    for (int c4 = 0; c4 < CW / 4; ++c4) {
        const float4 x = *reinterpret_cast<const float4*>(tile + core_off(r, c0 + 4 * c4, SCA));
        v[4 * c4] = x.x, v[4 * c4 + 1] = x.y, v[4 * c4 + 2] = x.z, v[4 * c4 + 3] = x.w;
    }
}

// -------------------------------------------------------------------------------------------------------------
#ifdef PROMP_EXP_CLOCKS
// experiment build only: clock64 totals over ALL CTAs of policy_chain_tc_kernel (thread 0 of each CTA):
// 0 queue pop + decode, 1 dependency wait, 2 parameter / weight load, 3 tiles, 4 flush up to the ticket, 5 last-arriver
// reduction + publish, 6 items, 7 last arrivals, 8 whole kernel (sum over CTAs), 9 CTAs
__device__ unsigned long long g_chain_clk[16];
__device__ long long g_chain_last[1024];
#define CCLK(i)                                                                                  \
    do {                                                                                         \
        if (threadIdx.x == 0) {                                                                  \
            const long long t_ = clock64();                                                      \
            atomicAdd(&g_chain_clk[i], (unsigned long long)(t_ - g_chain_last[blockIdx.x]));     \
            g_chain_last[blockIdx.x] = t_;                                                       \
        }                                                                                        \
    } while (0)
#define CCNT(i)                                            \
    do {                                                   \
        if (threadIdx.x == 0) atomicAdd(&g_chain_clk[i], 1ull); \
    } while (0)
#else
#define CCLK(i)
#define CCNT(i)
#endif
// ItemSched: the schedule (see UniformSched in mlp_tile.cuh) of one work item of policy_chain_tc_kernel: tiles
// [g_lo, g_hi) of ONE task; slots are numbered by item id.
struct ItemSched {
    int ntiles, g_lo, g_hi;
    int item, first_item, n_items;        // this item's id; the ids of its task's items in this stage
    const int* ready_prev;                // [M] flags of the previous stage (nullptr: no dependency)
    int* ready_mine;                      // [M] flags of this stage
    __device__ __forceinline__ int my_slot(int) const { return item; }
    __device__ __forceinline__ int n_contrib(int) const { return n_items; }
    __device__ __forceinline__ int contrib_slot(int, int i) const { return first_item + i; }
    __device__ __forceinline__ void clk(int i) const { CCLK(i); }
    __device__ __forceinline__ void wait_task(int m) const {       // called by every thread of the CTA
        if (ready_prev == nullptr) return;
        if (threadIdx.x == 0) {
            int v;
            unsigned spins = 0;
            long long t0 = 0;
            do {
                asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(ready_prev + m) : "memory");
                if (v == 0 && (++spins & 0xfffu) == 0) {          // safety net: a producer that never arrives is a bug, not a wait
                    const long long t = clock64();
                    if (t0 == 0) t0 = t;
                    else if (t - t0 > 8000000000ll) {              // ~4 s
                        // no printf here: a call anywhere in the kernel makes ptxas serialize every wgmma of it
                        __trap();
                    }
                }
            } while (v == 0);
        }
        __syncthreads();
        CCLK(1);
    }
    __device__ __forceinline__ void publish_task(int m) const {    // called by every thread of the task's last arriver
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) asm volatile("st.release.gpu.global.s32 [%0], %1;\n" ::"l"(ready_mine + m), "r"(1) : "memory");
        CCNT(7);
    }
    static __device__ __forceinline__ float ldp(const float* p) { return __ldcg(p); }
    static __device__ __forceinline__ float4 ldp4(const float4* p) { return __ldcg(p); }
};

#ifdef PROMP_EXP_CLOCKS
// experiment build only: per-phase clock64 totals of CTA 0 (tools/kernel_time.py --clocks)
__device__ unsigned long long g_phase_clk[16];
#define PCLK(i)                                                   \
    do {                                                          \
        if (blockIdx.x == 0 && threadIdx.x == 0) {                \
            const long long t_ = clock64();                       \
            s_clk[i] += (unsigned long long)(t_ - s_last);        \
            s_last = t_;                                          \
        }                                                         \
    } while (0)
#else
#define PCLK(i)
#endif
// The tile loop of the gradient kernel over the range `sc` describes.  `cached_th` = the parameter vector whose weights
// the shared-memory tiles currently hold (nullptr: none) - kept across calls by the dataflow kernel.
template <int DO, int DA, int NQ, class Act, class Sched, int ADV = ADV_SAMPLE>
__device__ __forceinline__ void grad_tc_tiles(const PolicyArgs& A, GradTcSmem<DO, DA, NQ>& S, const Sched& sc,
                                              const float*& cached_th) {
    constexpr int HID = TC_HID;
    using L = PLayout<DO, DA, HID>;
    using SL = SmallLayout<DO, DA>;
    using SM = GradTcSmem<DO, DA, NQ>;
    constexpr int TCT = 128 * NQ, CW = TC_HID / NQ, NW = TCT / 32, NT = 8 / NQ;   // threads, columns per thread, warps, wgrad n-tiles per warp
    constexpr int LNT = 64 / NW;                                                 // layer-GEMM n-tiles per warp
    constexpr int DOP = SM::DOP;
    constexpr int PSTRIDE = L::P + PSTAT;
    constexpr int NPART = TCT / HID, BPP = TBT / NPART;     // column role: 4 slices of 32 rows

#ifdef PROMP_EXP_CLOCKS
    __shared__ unsigned long long s_clk[16];
    __shared__ long long s_last;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 16; ++i) s_clk[i] = 0;
        s_last = clock64();
    }
#endif

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int qd = warp & 3, cq = warp >> 2;               // row quadrant, column group
    const int r = qd * 32 + lane, c0 = CW * cq;          // row / column-group role: sample row r, hidden units [c0, c0+32)
    const int cj = tid & (HID - 1), cp = tid / HID;        // column role
    const int dO = obs_dim_of<DO, DA>(A), dA = act_dim_of<DO, DA>(A);      // logical sizes (padded instantiations)
    const int N = A.N;
    const float kl_eff = kl_coeff_eff(A);      // kl_coeff, times the device-resident multiplier when there is one
    float invN = 1.0f / (float)N;       // both re-set per task when A.n_valid is given (variable-length paths)
    int Nm = N;
    const bool want_grad = A.grad != nullptr;
    const float* th = nullptr;
    HeadIn<DA>& hin = S.hin;

    float gW1[NT][4], gB1f[NT], gW0p[DO], gW2p[DA], gB0c, gB2w[DA], gLSw[DA];   // gB2w/gLSw: per-thread partials (cq == 0 rows)
    float s_obj, s_kl, s_ratio;
    auto zero_acc = [&]() {
#pragma unroll
        for (int a = 0; a < NT; ++a) gW1[a][0] = gW1[a][1] = gW1[a][2] = gW1[a][3] = gB1f[a] = 0.f;
#pragma unroll
        for (int i = 0; i < DO; ++i) gW0p[i] = 0.f;
#pragma unroll
        for (int d = 0; d < DA; ++d) gW2p[d] = 0.f;
#pragma unroll
        for (int d = 0; d < DA; ++d) gB2w[d] = gLSw[d] = 0.f;
        gB0c = 0.f;
        s_obj = s_kl = s_ratio = 0.f;
    };
    auto load_task = [&](int m) {
        sc.wait_task(m);
        if (A.n_valid) { Nm = __ldg(A.n_valid + m); invN = 1.0f / (float)max(Nm, 1); }
        th = A.params + (int64_t)m * A.param_stride;
        const bool reload = th != cached_th;      // CTA-uniform: do the shared-memory tiles already hold these weights?
        cached_th = th;
        if (reload) __syncthreads();
        for (int i = tid; reload && i < DO * HID + HID; i += TCT) S.Ps[SL::W0 + i] = Sched::ldp(th + L::W0 + i);          // W0, b0
        for (int i = tid; reload && i < HID; i += TCT) S.Ps[SL::B1 + i] = Sched::ldp(th + L::B1 + i);
        for (int i = tid; reload && i < HID * DA + 2 * DA; i += TCT) S.Ps[SL::W2 + i] = Sched::ldp(th + L::W2 + i);       // W2, b2, ls
        // W1 in both operand layouts, 4 elements (one 16-byte shared-memory store, conflict-free) per thread and buffer
        for (int u = tid; reload && u < HID * HID / 4; u += TCT) {
            float4 w, wl;
            {       // backward operand: tile row = k, K = j; one 16-byte load of W1[k][4 jg ..]
                const int jg = u % (HID / 4), k = u / (HID / 4);
                w = Sched::ldp4(reinterpret_cast<const float4*>(th + L::W1 + k * HID + 4 * jg));
                wl = make_float4(w.x - tf32_trunc(w.x), w.y - tf32_trunc(w.y), w.z - tf32_trunc(w.z), w.w - tf32_trunc(w.w));
                const int off = jg * SCW + (k >> 3) * 128 + (k & 7) * 16;
                *reinterpret_cast<float4*>(S.W1_hi + off) = make_float4(tf32_trunc(w.x), tf32_trunc(w.y), tf32_trunc(w.z), tf32_trunc(w.w));
                *reinterpret_cast<float4*>(S.W1_lo + off) = wl;
            }
            {       // forward operand: tile row = j, K = k; W1[4 kg .. 4 kg + 3][j], lanes run over j
                const int j = u % HID, kg = u / HID;
                const float* src = th + L::W1 + 4 * kg * HID + j;
                w = make_float4(Sched::ldp(src), Sched::ldp(src + HID), Sched::ldp(src + 2 * HID), Sched::ldp(src + 3 * HID));
                wl = make_float4(w.x - tf32_trunc(w.x), w.y - tf32_trunc(w.y), w.z - tf32_trunc(w.z), w.w - tf32_trunc(w.w));
                const int off = kg * SCW + (j >> 3) * 128 + (j & 7) * 16;
                *reinterpret_cast<float4*>(S.W1T_hi + off) = make_float4(tf32_trunc(w.x), tf32_trunc(w.y), tf32_trunc(w.z), tf32_trunc(w.w));
                *reinterpret_cast<float4*>(S.W1T_lo + off) = wl;
            }
        }
        if (reload) wg_fence_weights();      // the weight tiles are read by the wgmma (async) proxy after the barrier
        __syncthreads();          // Ps is in place; every reader of the previous task's hin / hold is done
        if (tid == 0) head_setup<DA>(A, S.Ps + SL::LS, m, dA, hin, &S.hold);
        __syncthreads();
    };
    auto flush = [&](int m) {
        sc.clk(3);
        float* part = A.partial + (int64_t)sc.my_slot(m) * PSTRIDE;
        float* scr = reinterpret_cast<float*>(S.A1);      // A1 + LO (contiguous, 2 tiles): free between tiles (all MMAs have completed)
        __syncthreads();
        if (want_grad) {
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) part[L::W1 + wgrad_mma_index<NT>(warp, lane, nt, i)] = gW1[nt][i];
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {            // b1 gradient: fragment column sums, reduced over the 4 lanes of a column
                float c = gB1f[nt];
                c += __shfl_xor_sync(0xffffffffu, c, 1);
                c += __shfl_xor_sync(0xffffffffu, c, 2);
                if ((lane & 3) == 0 && (warp & 3) == 0) part[L::B1 + 8 * NT * (warp >> 2) + 8 * nt + (lane >> 2)] = c;
            }
            scr[cp * HID + cj] = gB0c;
            __syncthreads();
            if (tid < HID) {
                float s = 0.f;
                for (int p = 0; p < NPART; ++p) s += scr[p * HID + tid];
                part[L::B0 + tid] = s;
            }
            __syncthreads();
#pragma unroll
            for (int d = 0; d < DA; ++d) {                 // (uniform over the CTA: every warp takes part in the shuffles)
                const float s1 = warp_sum(gB2w[d]), s2 = warp_sum(gLSw[d]);
                if (cq == 0 && lane == 0) scr[qd * 2 * DA + d] = s1, scr[qd * 2 * DA + DA + d] = s2;
            }
            __syncthreads();
            if (tid < 2 * DA) part[L::B2 + tid] = scr[tid] + scr[2 * DA + tid] + scr[4 * DA + tid] + scr[6 * DA + tid];   // b2 then log_std
            __syncthreads();
        }
        PCLK(14);
        flush_tail<TCT, 8, 2 * TILE_A_BYTES / 4, DO, DA, HID>(A, sc, m, invN, want_grad, part, scr, S.red, S.last, gW0p, gW2p, s_obj, s_kl, s_ratio,
                                        GradEpilogue<L::P, Sched>{A, th, m});
        PCLK(15);
    };

    // observation prefetch (small observation / action spaces: one or two elements per thread, registers to spare)
    constexpr int XR = (TBT * DOP) / TCT;
    constexpr bool XPRE = (TBT * DOP) % TCT == 0 && XR >= 1 && XR <= 2 && DA <= 2;
    float xq[XPRE ? XR : 1], ha[DA], hmo[DA], hlso[DA], hadv = 0.f;
    auto fetch_x = [&](int g_, float (&dst)[XPRE ? XR : 1]) {
        const int m_ = g_ / sc.ntiles, n0_ = (g_ - m_ * sc.ntiles) * TBT;
        const int nb_ = max(0, min(TBT, (A.n_valid ? __ldg(A.n_valid + m_) : N) - n0_));
#pragma unroll
        for (int e = 0; e < (XPRE ? XR : 1); ++e) {
            const int i = tid + e * TCT, b = i / DOP, c = i % DOP;
            dst[e] = (b < nb_ && c < dO) ? __ldg(A.obs + ((int64_t)m_ * N + n0_ + b) * dO + c) : 0.f;
        }
    };
    int cur_m = -1;
    for (int g = sc.g_lo; g < sc.g_hi; ++g) {
        const int m = g / sc.ntiles, tile = g - m * sc.ntiles;
        PCLK(10);
        if (m != cur_m) {
            if (cur_m >= 0) flush(cur_m);
            PCLK(11);
            load_task(m);
            sc.clk(2);
            zero_acc();
            cur_m = m;
            PCLK(12);
        }
        const int n0 = tile * TBT, nb = max(0, min(TBT, Nm - n0));
        const int64_t g0 = (int64_t)m * N + n0;
        __syncthreads();
        if constexpr (XPRE) {
            // software pipeline: this tile's observations were fetched while the previous tile was processed; the next
            // tile's are fetched now, and the Gaussian head's per-sample inputs are requested ~10 k cycles before their use
            if (g == sc.g_lo) fetch_x(g, xq);
#pragma unroll
            for (int e = 0; e < XR; ++e) S.X[tid + e * TCT] = xq[e];
            if (g + 1 < sc.g_hi) fetch_x(g + 1, xq);
            if (cq == 0 && r < nb) hadv = load_head_sample<DA, ADV>(A, g0 + r, m, dA, A.ls_per_sample, ha, hmo, hlso);
        } else {
            for (int i = tid; i < TBT * DOP; i += TCT) {
                const int b = i / DOP, c = i % DOP;
                S.X[i] = (b < nb && c < dO) ? __ldg(A.obs + (g0 + b) * dO + c) : 0.f;
            }
        }
        __syncthreads();
        PCLK(0);
        // ---- layer 0 (CUDA cores, row / column-group role): H1 = act(X W0 + b0) -> A0
        {
            float x[DO];
#pragma unroll
            for (int i = 0; i < DO; ++i) x[i] = S.X[r * DOP + i];
#pragma unroll
            for (int c4 = 0; c4 < CW / 4; ++c4) {
                float h[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = c0 + 4 * c4 + e;
                    float z = S.Ps[SL::B0 + c];
#pragma unroll
                    for (int i = 0; i < DO; ++i) z = fmaf(x[i], S.Ps[SL::W0 + i * HID + c], z);
                    h[e] = Act::f(z);
                }
                *reinterpret_cast<float4*>(S.A0 + core_off(r, c0 + 4 * c4, SCA)) = make_float4(h[0], h[1], h[2], h[3]);
            }
        }
        PCLK(1);
        // ---- layer 1 on the tensor cores: Z2 = H1 W1 -> LO (staged for the row-per-thread epilogue)
        __syncthreads();
        {
            float acc[LNT][4];
            zero_frag<LNT>(acc);
            layer_gemm_issue<LNT>(acc, S.A0, S.W1T_hi, S.W1T_lo, warp, lane);
            wg_wait();
            wg_pin<LNT>(acc);
            store_frag<LNT>(acc, S.LO, warp, lane);
        }
        __syncthreads();
        PCLK(2);
        float h2[CW];
        load_row<CW>(S.LO, r, c0, h2);
        float mup[DA];
#pragma unroll
        for (int d = 0; d < DA; ++d) mup[d] = 0.f;
#pragma unroll
        for (int c4 = 0; c4 < CW / 4; ++c4) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int c = 4 * c4 + e;
                h2[c] = Act::f(h2[c] + S.Ps[SL::B1 + c0 + c]);
#pragma unroll
                for (int d = 0; d < DA; ++d) mup[d] = fmaf(h2[c], S.Ps[SL::W2 + (c0 + c) * DA + d], mup[d]);
            }
            *reinterpret_cast<float4*>(S.A1 + core_off(r, c0 + 4 * c4, SCA)) =
                make_float4(h2[4 * c4], h2[4 * c4 + 1], h2[4 * c4 + 2], h2[4 * c4 + 3]);
        }
#pragma unroll
        for (int d = 0; d < DA; ++d) S.MUP[(cq * TBT + r) * DA + d] = mup[d];
        __syncthreads();
        PCLK(3);
        // ---- Gaussian head: one thread per sample row (cq == 0)
        if (cq == 0) {
            float dmu[DA], dls[DA];
            if (r < nb) {
                float mu[DA];
#pragma unroll
                for (int d = 0; d < DA; ++d) {
                    float sm = S.Ps[SL::B2 + d];
#pragma unroll
                    for (int q = 0; q < NQ; ++q) sm += S.MUP[(q * TBT + r) * DA + d];
                    mu[d] = sm;
                }
                float a[DA], mo[DA], lso[DA], adv;
                if constexpr (XPRE) {
#pragma unroll
                    for (int d = 0; d < DA; ++d) a[d] = ha[d], mo[d] = hmo[d], lso[d] = hlso[d];
                    adv = hadv;
                } else {
                    adv = load_head_sample<DA, ADV>(A, g0 + r, m, dA, A.ls_per_sample, a, mo, lso);
                }
                HeadOut<DA> o;
                out_forward<Act, DA>(mu);
                if (A.ls_per_sample) {
                    HeadOld<DA> ho;
                    head_old_from<DA>(lso, ho, dA);
                    gaussian_head<DA>(hin, ho, mu, a, mo, adv, A.obj_kind, A.clip_eps, o, dA);
                } else {
                    gaussian_head<DA>(hin, S.hold, mu, a, mo, adv, A.obj_kind, A.clip_eps, o, dA);
                }
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
            for (int d = 0; d < DA; ++d) {
                S.DMU[r * DA + d] = dmu[d];
                gB2w[d] += dmu[d], gLSw[d] += dls[d];      // gB2 / g_log_std: per-thread partials, reduced over the warp at flush
            }
        }
        if (!want_grad) continue;
        __syncthreads();
        PCLK(4);
        // ---- output-layer gradients (column role) from the fp32 H2 tile
        {
            const int b0 = cp * BPP;
            // b0 is a multiple of 8: row b0 + bb of column cj sits at a compile-time offset from row b0 (fully unrolled)
            const unsigned char* colp = S.A1 + core_off(b0, cj, SCA);
            const float* dmu0 = S.DMU + b0 * DA;
#pragma unroll(BPP <= 16 ? 2 : 1)
            for (int b8 = 0; b8 < BPP; b8 += 8)
#pragma unroll
            for (int b1 = 0; b1 < 8; ++b1) {
                const int bb = b8 + b1;
                const float h = *reinterpret_cast<const float*>(colp + (bb >> 3) * 128 + (bb & 7) * 16);
#pragma unroll
                for (int d = 0; d < DA; ++d) gW2p[d] = fmaf(h, dmu0[bb * DA + d], gW2p[d]);
            }
        }
        __syncthreads();
        PCLK(5);
        // ---- D2 = (DMU W2^T) * act'(H2) from the h2 registers -> A1
        {
            float dm[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) dm[d] = S.DMU[r * DA + d];
#pragma unroll
            for (int c4 = 0; c4 < CW / 4; ++c4) {
                float v[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = 4 * c4 + e;
                    float dh = 0.f;
#pragma unroll
                    for (int d = 0; d < DA; ++d) dh = fmaf(dm[d], S.Ps[SL::W2 + (c0 + c) * DA + d], dh);
                    v[e] = dh * Act::d(h2[c]);
                }
                *reinterpret_cast<float4*>(S.A1 + core_off(r, c0 + 4 * c4, SCA)) = make_float4(v[0], v[1], v[2], v[3]);
            }
        }
        __syncthreads();
        PCLK(6);
        // ---- weight gradient gW1 += H1^T D2 (mma.sync 3xTF32) and the bias column sums
        wgrad_mma_tile<true, NT, true>(S.A0, S.A1, 1.f, warp, lane, gW1, gB1f);
        PCLK(7);
        // ---- backward GEMM on the tensor cores: dH1 = D2 W1^T (registers), then D1 = dH1 * act'(H1) -> A0 in place
        {
            float acc[LNT][4];
            zero_frag<LNT>(acc);
            layer_gemm_issue<LNT>(acc, S.A1, S.W1_hi, S.W1_lo, warp, lane);
            wg_wait();
            wg_pin<LNT>(acc);
            __syncthreads();       // every read of H1 (weight gradient) is done before A0 is overwritten
            PCLK(8);
#pragma unroll
            for (int nt = 0; nt < LNT; ++nt)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float2* p = reinterpret_cast<float2*>(S.A0 + frag_off<LNT>(warp, lane, nt, h));
                    const float2 hv = *p;
                    *p = make_float2(acc[nt][2 * h] * Act::d(hv.x), acc[nt][2 * h + 1] * Act::d(hv.y));
                }
        }
        __syncthreads();
        PCLK(9);
        // ---- gW0 += X^T D1, gB0 += colsum(D1) (column role)
        {
            const int b0 = cp * BPP;
            const unsigned char* colp = S.A0 + core_off(b0, cj, SCA);
            const float* x0 = S.X + b0 * DOP;
#pragma unroll(BPP <= 16 ? 2 : 1)
            for (int b8 = 0; b8 < BPP; b8 += 8)
#pragma unroll
            for (int b1 = 0; b1 < 8; ++b1) {
                const int bb = b8 + b1;
                const float d1 = *reinterpret_cast<const float*>(colp + (bb >> 3) * 128 + (bb & 7) * 16);
                gB0c += d1;
#pragma unroll
                for (int i = 0; i < DO; ++i) gW0p[i] = fmaf(x0[bb * DOP + i], d1, gW0p[i]);
            }
        }
    }
    PCLK(10);
    if (cur_m >= 0) flush(cur_m);
    PCLK(11);
#ifdef PROMP_EXP_CLOCKS
    if (blockIdx.x == 0 && threadIdx.x == 0)
        for (int i = 0; i < 16; ++i) g_phase_clk[i] += s_clk[i];
#endif
}

template <int DO, int DA, int NQ, class Act, int ADV = ADV_SAMPLE>
__device__ __forceinline__ void policy_grad_tc_body(const PolicyArgs& A) {
    using SM = GradTcSmem<DO, DA, NQ>;
    using L = PLayout<DO, DA, TC_HID>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SM& S = *reinterpret_cast<SM*>(smem_raw);
    if (reuse_hit<L::P>(A.skip_flag, A.params, A.skip_theta)) return;
    reuse_produce<L::P, L::LS, DA>(A);
    const UniformSched sc(A.M, A.N, A.q, A.kmax, TBT);
    const float* cached_th = nullptr;
    grad_tc_tiles<DO, DA, NQ, Act, UniformSched, ADV>(A, S, sc, cached_th);
}
// one kernel per activation, as in policy.cu: *_kernel = tanh, *_relu_kernel = ReLU
template <int DO, int DA, int NQ>
__global__ void __launch_bounds__(128 * NQ, 1) policy_grad_tc_kernel(PolicyArgs A) { policy_grad_tc_body<DO, DA, NQ, ActTanh>(A); }
template <int DO, int DA, int NQ>
__global__ void __launch_bounds__(128 * NQ, 1) policy_grad_tc_relu_kernel(PolicyArgs A) { policy_grad_tc_body<DO, DA, NQ, ActRelu>(A); }
// PROMP_OBJ_EXPLORE: per-task weight adv[m] (see policy_grad_explore_kernel)
template <int DO, int DA, int NQ>
__global__ void __launch_bounds__(128 * NQ, 1) policy_grad_tc_explore_kernel(PolicyArgs A) {
    policy_grad_tc_body<DO, DA, NQ, ActTanh, ADV_TASK>(A);
}
template <int DO, int DA, int NQ>
__global__ void __launch_bounds__(128 * NQ, 1) policy_grad_tc_explore_relu_kernel(PolicyArgs A) {
    policy_grad_tc_body<DO, DA, NQ, ActRelu, ADV_TASK>(A);
}
// tanh output layer, for hidden activation Hid
template <int DO, int DA, int NQ, class Hid>
__global__ void __launch_bounds__(128 * NQ, 1) policy_grad_tc_otanh_kernel(PolicyArgs A) {
    policy_grad_tc_body<DO, DA, NQ, OutTanh<Hid>>(A);
}
template <int DO, int DA, int NQ, class Hid>
__global__ void __launch_bounds__(128 * NQ, 1) policy_grad_tc_explore_otanh_kernel(PolicyArgs A) {
    policy_grad_tc_body<DO, DA, NQ, OutTanh<Hid>, ADV_TASK>(A);
}


// =================================================================================================================
// Tensor-core variant of policy_hvp_kernel (HID = 64).  All six layer GEMMs of the exact Hessian-vector product
//   forward :  Z2 = H1 W1            RZ2 = R1 W1 + H1 V1
//   backward:  dH1 = D2 W1^T         CdH1 = C2 W1^T + D2 (ac V1)^T
// run as layer_gemm_issue (wgmma 3xTF32, A split into hi / lo at fragment load).  Shared memory cannot hold four
// activation tiles next to hi+lo copies of four weight tiles, so the B (weight) buffer is time-multiplexed:
// [W1^T, V1^T] for the forward MMAs, re-filled with [W1, ac V1] for the backward MMAs (66 KB from L2 twice per 128-row
// tile).  The forward results Z2 / RZ2 are staged in T2a / T2b (the thread that reads an element back writes H2 / R2
// over it); the backward results are consumed element-wise from the accumulators.  The two weight-gradient GEMMs
// (H1^T C2, R1^T D2) contract over samples and run as wgrad_mma_tile.
template <int DO, int DA, int NQ>
struct HvpTcSmem {
    static constexpr int DOP = DOPad<DO>::V;
    alignas(16) unsigned char WB[4][TILE_W_BYTES];    // fwd: W1T_hi, W1T_lo, V1T_hi, V1T_lo ; bwd: W1_hi, W1_lo, aV1_hi, aV1_lo
    alignas(16) unsigned char H1[TILE_A_BYTES];       // H1 -> C1
    alignas(16) unsigned char R1[TILE_A_BYTES];
    alignas(16) unsigned char T2a[TILE_A_BYTES];      // Z2 -> H2 -> D2
    alignas(16) unsigned char T2b[TILE_A_BYTES];      // RZ2 -> R2 -> C2 ; flush scratch
    alignas(16) float Ps[SmallLayout<DO, DA>::SIZE];
    alignas(16) float Vs[SmallLayout<DO, DA>::SIZE];
    // X (observations) aliases T2a (needed only before H2 is written and, re-read from L2, after D2 is dead);
    // MUP (per-column-group partial means) aliases WB[0..1] between the forward MMAs and the backward weight re-fill.
    float DMU[TBT * DA];
    float CMU[TBT * DA];
    float red[3 * 4 * NQ];
    HeadIn<DA> hin;           // per-task constants of the Gaussian head (written by thread 0 in load_task)
    HeadOld<DA> hold;         // ... of the old distribution when the phase stores one log_std row per task
    int last;
};

// Tile loop of the HVP kernel; same calling convention as grad_tc_tiles.
template <int DO, int DA, int NQ, class Act, class Sched>
__device__ __forceinline__ void hvp_tc_tiles(const PolicyArgs& A, HvpTcSmem<DO, DA, NQ>& S, const Sched& sc,
                                             const float*& cached_th) {
    constexpr int HID = TC_HID;
    using L = PLayout<DO, DA, HID>;
    using SL = SmallLayout<DO, DA>;
    using SM = HvpTcSmem<DO, DA, NQ>;
    constexpr int TCT = 128 * NQ, CW = TC_HID / NQ, NW = TCT / 32, NT = 8 / NQ;
    constexpr int LNT = 64 / NW;
    constexpr int DOP = SM::DOP;
    constexpr int PSTRIDE = L::P + PSTAT;
    constexpr int NPART = TCT / HID, BPP = TBT / NPART;

    float* const sX = reinterpret_cast<float*>(S.T2a);
    float* const sMUP = reinterpret_cast<float*>(S.WB[0]);
    static_assert(TBT * DOP * 4 <= TILE_A_BYTES && NQ * TBT * 2 * DA * 4 <= 2 * TILE_W_BYTES, "aliased buffers must fit");

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int qd = warp & 3, cq = warp >> 2;               // row quadrant, column group
    const int r = qd * 32 + lane, c0 = CW * cq;
    const int cj = tid & (HID - 1), cp = tid / HID;
    const int dO = obs_dim_of<DO, DA>(A), dA = act_dim_of<DO, DA>(A);
    const int N = A.N;
    const float kl_eff = kl_coeff_eff(A);      // kl_coeff, times the device-resident multiplier when there is one
    float invN = 1.0f / (float)N;       // both re-set per task when A.n_valid is given (variable-length paths)
    int Nm = N;
    const float ac = -A.inner_lr;
    const float* th = nullptr;
    const float* vg = nullptr;
    HeadIn<DA>& hin = S.hin;
    float rls[DA];

    float gW1[NT][4], gB1f[NT], gW0p[DO], gW2p[DA], gB0c, gB2w[DA], gLSw[DA];
    float s_obj, s_kl, s_ratio;
    auto zero_acc = [&]() {
#pragma unroll
        for (int a = 0; a < NT; ++a) gW1[a][0] = gW1[a][1] = gW1[a][2] = gW1[a][3] = gB1f[a] = 0.f;
#pragma unroll
        for (int i = 0; i < DO; ++i) gW0p[i] = 0.f;
#pragma unroll
        for (int d = 0; d < DA; ++d) gW2p[d] = 0.f;
#pragma unroll
        for (int d = 0; d < DA; ++d) gB2w[d] = gLSw[d] = 0.f;
        gB0c = 0.f;
        s_obj = s_kl = s_ratio = 0.f;
    };
    // The direction vector may be read through the read-only path only if nothing in this launch writes it: out != vec (the
    // in-place form v <- v - alpha H v rewrites task m's slice at its flush) and no producer stage in the same launch.
    const bool vec_ro = A.out != A.vec;
    // Per-parameter step sizes (A.step_size): H is applied to alpha * vec, so every staged direction element i - both the
    // shared-memory copy and the W1 weight buffers - is scaled by alpha[i]; the epilogue's vec stays unscaled.
    const float* const al = A.step_size;
    auto ldv = [&](const float* p) {
        const float v = vec_ro ? Sched::ldp(p) : __ldcg(p);
        return al ? __ldg(al + (p - vg)) * v : v;
    };
    auto ldv4 = [&](const float4* p) {
        const float4 v = vec_ro ? Sched::ldp4(p) : __ldcg(p);
        if (!al) return v;
        const float4 a = __ldg(reinterpret_cast<const float4*>(al + (reinterpret_cast<const float*>(p) - vg)));
        return make_float4(a.x * v.x, a.y * v.y, a.z * v.z, a.w * v.w);
    };
    auto load_task = [&](int m) {
        sc.wait_task(m);
        if (A.n_valid) { Nm = __ldg(A.n_valid + m); invN = 1.0f / (float)max(Nm, 1); }
        th = A.params + (int64_t)m * A.param_stride;
        vg = A.vec + (int64_t)m * L::P;
        __syncthreads();
        const bool reload_p = th != cached_th;      // CTA-uniform: S.Ps already holds these parameters
        cached_th = th;
        for (int i = tid; i < DO * HID + HID; i += TCT) {
            if (reload_p) S.Ps[SL::W0 + i] = Sched::ldp(th + L::W0 + i);
            S.Vs[SL::W0 + i] = ldv(vg + L::W0 + i);
        }
        for (int i = tid; i < HID; i += TCT) {
            if (reload_p) S.Ps[SL::B1 + i] = Sched::ldp(th + L::B1 + i);
            S.Vs[SL::B1 + i] = ldv(vg + L::B1 + i);
        }
        for (int i = tid; i < HID * DA + 2 * DA; i += TCT) {
            if (reload_p) S.Ps[SL::W2 + i] = Sched::ldp(th + L::W2 + i);
            S.Vs[SL::W2 + i] = ldv(vg + L::W2 + i);
        }
        __syncthreads();
        if (tid == 0) head_setup<DA>(A, S.Ps + SL::LS, m, dA, hin, &S.hold);
        __syncthreads();
#pragma unroll
        for (int d = 0; d < DA; ++d) rls[d] = S.Vs[SL::LS + d] * hin.ls_mask[d];
    };
    // (re)fill the weight buffer from L2: forward = [W1^T, V1^T], backward = [W1, ac*V1], each as hi (tf32-truncated) + lo
    // 4 elements per thread and buffer: one conflict-free 16-byte shared-memory store each (the element-wise version paid a
    // 4-way bank conflict on every forward-layout store: 1.0 M of the kernel's 1.2 M conflicts in the round-1 profile)
    auto load_weights = [&](bool fwd) {
        for (int u = tid; u < HID * HID / 4; u += TCT) {
            float4 w, v;
            int off;
            if (fwd) {      // tile row = j, K = k: W1[4 kg .. 4 kg + 3][j], lanes run over j (coalesced 4-byte loads)
                const int j = u % HID, kg = u / HID;
                const float* sw = th + L::W1 + 4 * kg * HID + j;
                const float* sv = vg + L::W1 + 4 * kg * HID + j;
                w = make_float4(Sched::ldp(sw), Sched::ldp(sw + HID), Sched::ldp(sw + 2 * HID), Sched::ldp(sw + 3 * HID));
                v = make_float4(ldv(sv), ldv(sv + HID), ldv(sv + 2 * HID), ldv(sv + 3 * HID));
                off = kg * SCW + (j >> 3) * 128 + (j & 7) * 16;
            } else {        // tile row = k, K = j: one 16-byte load of W1[k][4 jg ..]
                const int jg = u % (HID / 4), k = u / (HID / 4);
                w = Sched::ldp4(reinterpret_cast<const float4*>(th + L::W1 + k * HID + 4 * jg));
                v = ldv4(reinterpret_cast<const float4*>(vg + L::W1 + k * HID + 4 * jg));
                v = make_float4(ac * v.x, ac * v.y, ac * v.z, ac * v.w);
                off = jg * SCW + (k >> 3) * 128 + (k & 7) * 16;
            }
            *reinterpret_cast<float4*>(S.WB[0] + off) = make_float4(tf32_trunc(w.x), tf32_trunc(w.y), tf32_trunc(w.z), tf32_trunc(w.w));
            *reinterpret_cast<float4*>(S.WB[1] + off) =
                make_float4(w.x - tf32_trunc(w.x), w.y - tf32_trunc(w.y), w.z - tf32_trunc(w.z), w.w - tf32_trunc(w.w));
            *reinterpret_cast<float4*>(S.WB[2] + off) = make_float4(tf32_trunc(v.x), tf32_trunc(v.y), tf32_trunc(v.z), tf32_trunc(v.w));
            *reinterpret_cast<float4*>(S.WB[3] + off) =
                make_float4(v.x - tf32_trunc(v.x), v.y - tf32_trunc(v.y), v.z - tf32_trunc(v.z), v.w - tf32_trunc(v.w));
        }
        wg_fence_weights();      // read by the wgmma (async) proxy after the caller's next barrier
    };
    auto flush = [&](int m) {
        sc.clk(3);
        float* part = A.partial + (int64_t)sc.my_slot(m) * PSTRIDE;
        float* scr = reinterpret_cast<float*>(S.T2a);     // T2a + T2b (contiguous, 2 tiles)
        __syncthreads();
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) part[L::W1 + wgrad_mma_index<NT>(warp, lane, nt, i)] = gW1[nt][i];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            float c = gB1f[nt];
            c += __shfl_xor_sync(0xffffffffu, c, 1);
            c += __shfl_xor_sync(0xffffffffu, c, 2);
            if ((lane & 3) == 0 && (warp & 3) == 0) part[L::B1 + 8 * NT * (warp >> 2) + 8 * nt + (lane >> 2)] = c;
        }
        scr[cp * HID + cj] = gB0c;
        __syncthreads();
        if (tid < HID) {
            float s = 0.f;
            for (int p = 0; p < NPART; ++p) s += scr[p * HID + tid];
            part[L::B0 + tid] = s;
        }
        __syncthreads();
#pragma unroll
        for (int d = 0; d < DA; ++d) {                     // (uniform over the CTA: every warp takes part in the shuffles)
            const float s1 = warp_sum(gB2w[d]), s2 = warp_sum(gLSw[d]);
            if (cq == 0 && lane == 0) scr[qd * 2 * DA + d] = s1, scr[qd * 2 * DA + DA + d] = s2;
        }
        __syncthreads();
        if (tid < 2 * DA) part[L::B2 + tid] = scr[tid] + scr[2 * DA + tid] + scr[4 * DA + tid] + scr[6 * DA + tid];   // b2 then log_std
        __syncthreads();
        flush_tail<TCT, 8, 2 * TILE_A_BYTES / 4, DO, DA, HID>(A, sc, m, invN, true, part, scr, S.red, S.last, gW0p, gW2p, s_obj, s_kl, s_ratio,
                                        HvpEpilogue<L::P>{A, vg, m});
    };

    constexpr int XR = (TBT * DOP) / TCT;
    constexpr bool XPRE = (TBT * DOP) % TCT == 0 && XR >= 1 && XR <= 2 && DA <= 2;
    float xq[XPRE ? XR : 1], xc[XPRE ? XR : 1], ha[DA], hmo[DA], hlso[DA], hadv = 0.f;
    auto fetch_x = [&](int g_, float (&dst)[XPRE ? XR : 1]) {
        const int m_ = g_ / sc.ntiles, n0_ = (g_ - m_ * sc.ntiles) * TBT;
        const int nb_ = max(0, min(TBT, (A.n_valid ? __ldg(A.n_valid + m_) : N) - n0_));
#pragma unroll
        for (int e = 0; e < (XPRE ? XR : 1); ++e) {
            const int i = tid + e * TCT, b = i / DOP, c = i % DOP;
            dst[e] = (b < nb_ && c < dO) ? __ldg(A.obs + ((int64_t)m_ * N + n0_ + b) * dO + c) : 0.f;
        }
    };
    int cur_m = -1;
    for (int g = sc.g_lo; g < sc.g_hi; ++g) {
        const int m = g / sc.ntiles, tile = g - m * sc.ntiles;
        if (m != cur_m) {
            if (cur_m >= 0) flush(cur_m);
            load_task(m);
            sc.clk(2);
            zero_acc();
            cur_m = m;
        }
        const int n0 = tile * TBT, nb = max(0, min(TBT, Nm - n0));
        const int64_t g0 = (int64_t)m * N + n0;
        __syncthreads();
        auto load_x = [&]() {
            for (int i = tid; i < TBT * DOP; i += TCT) {
                const int b = i / DOP, c = i % DOP;
                sX[i] = (b < nb && c < dO) ? __ldg(A.obs + (g0 + b) * dO + c) : 0.f;
            }
        };
        if constexpr (XPRE) {      // software pipeline, as in grad_tc_tiles; xc keeps this tile's elements for the second use below
            if (g == sc.g_lo) fetch_x(g, xq);
#pragma unroll
            for (int e = 0; e < XR; ++e) xc[e] = xq[e], sX[tid + e * TCT] = xc[e];
            if (g + 1 < sc.g_hi) fetch_x(g + 1, xq);
            if (cq == 0 && r < nb) hadv = load_head_sample<DA>(A, g0 + r, m, dA, A.ls_per_sample, ha, hmo, hlso);
        } else {
            load_x();
        }
        load_weights(true);
        __syncthreads();
        // ---- layer 0 and its tangent (CUDA cores, row / column-group role)
        {
            float x[DO];
#pragma unroll
            for (int i = 0; i < DO; ++i) x[i] = sX[r * DOP + i];
#pragma unroll
            for (int c4 = 0; c4 < CW / 4; ++c4) {
                float h[4], r1[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = c0 + 4 * c4 + e;
                    float z = S.Ps[SL::B0 + c], rz = S.Vs[SL::B0 + c];
#pragma unroll
                    for (int i = 0; i < DO; ++i) {
                        z = fmaf(x[i], S.Ps[SL::W0 + i * HID + c], z);
                        rz = fmaf(x[i], S.Vs[SL::W0 + i * HID + c], rz);
                    }
                    h[e] = Act::f(z);
                    r1[e] = Act::d(h[e]) * rz;
                }
                const int off = core_off(r, c0 + 4 * c4, SCA);
                *reinterpret_cast<float4*>(S.H1 + off) = make_float4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<float4*>(S.R1 + off) = make_float4(r1[0], r1[1], r1[2], r1[3]);
            }
        }
        // ---- forward MMAs: Z2 = H1 W1 -> T2a ; RZ2 = R1 W1 + H1 V1 -> T2b (X, aliasing T2a, has been read above)
        __syncthreads();
        {
            float acc[LNT][4];
            zero_frag<LNT>(acc);
            layer_gemm_issue<LNT>(acc, S.H1, S.WB[0], S.WB[1], warp, lane);
            wg_wait();
            wg_pin<LNT>(acc);
            store_frag<LNT>(acc, S.T2a, warp, lane);
            zero_frag<LNT>(acc);
            layer_gemm_issue<LNT>(acc, S.R1, S.WB[0], S.WB[1], warp, lane);
            layer_gemm_issue<LNT>(acc, S.H1, S.WB[2], S.WB[3], warp, lane);
            wg_wait();
            wg_pin<LNT>(acc);
            store_frag<LNT>(acc, S.T2b, warp, lane);
        }
        __syncthreads();       // also: every MMA read of WB has completed before MUP (aliasing WB[0..1]) is written
        float h2[CW], r2[CW];
        load_row<CW>(S.T2a, r, c0, h2);
        load_row<CW>(S.T2b, r, c0, r2);
        {
            float mup[DA], rmup[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) mup[d] = rmup[d] = 0.f;
#pragma unroll
            for (int c4 = 0; c4 < CW / 4; ++c4) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = 4 * c4 + e;
                    h2[c] = Act::f(h2[c] + S.Ps[SL::B1 + c0 + c]);
                    r2[c] = Act::d(h2[c]) * (r2[c] + S.Vs[SL::B1 + c0 + c]);
#pragma unroll
                    for (int d = 0; d < DA; ++d) {
                        const float w2 = S.Ps[SL::W2 + (c0 + c) * DA + d];
                        mup[d] = fmaf(h2[c], w2, mup[d]);
                        rmup[d] = fmaf(r2[c], w2, fmaf(h2[c], S.Vs[SL::W2 + (c0 + c) * DA + d], rmup[d]));
                    }
                }
                const int off = core_off(r, c0 + 4 * c4, SCA);
                *reinterpret_cast<float4*>(S.T2a + off) = make_float4(h2[4 * c4], h2[4 * c4 + 1], h2[4 * c4 + 2], h2[4 * c4 + 3]);
                *reinterpret_cast<float4*>(S.T2b + off) = make_float4(r2[4 * c4], r2[4 * c4 + 1], r2[4 * c4 + 2], r2[4 * c4 + 3]);
            }
#pragma unroll
            for (int d = 0; d < DA; ++d) {
                sMUP[((cq * TBT + r) * 2 + 0) * DA + d] = mup[d];
                sMUP[((cq * TBT + r) * 2 + 1) * DA + d] = rmup[d];
            }
        }
        __syncthreads();
        // ---- Gaussian head and its tangent: one thread per sample row (cq == 0)
        if (cq == 0) {
            float dmu[DA], cmu[DA], cls[DA];
            if (r < nb) {
                float mu[DA], rmu[DA];
#pragma unroll
                for (int d = 0; d < DA; ++d) {
                    float sm = S.Ps[SL::B2 + d], sr = S.Vs[SL::B2 + d];
#pragma unroll
                    for (int q = 0; q < NQ; ++q) sm += sMUP[((q * TBT + r) * 2 + 0) * DA + d], sr += sMUP[((q * TBT + r) * 2 + 1) * DA + d];
                    mu[d] = sm;
                    rmu[d] = sr;
                }
                float a[DA], mo[DA], lso[DA], adv;
                if constexpr (XPRE) {
#pragma unroll
                    for (int d = 0; d < DA; ++d) a[d] = ha[d], mo[d] = hmo[d], lso[d] = hlso[d];
                    adv = hadv;
                } else {
                    adv = load_head_sample<DA>(A, g0 + r, m, dA, A.ls_per_sample, a, mo, lso);
                }
                HeadOut<DA> o;
                out_forward_tangent<Act, DA>(mu, rmu);
                if (A.ls_per_sample) {
                    HeadOld<DA> ho;
                    head_old_from<DA>(lso, ho, dA);
                    gaussian_head<DA>(hin, ho, mu, a, mo, adv, A.obj_kind, A.clip_eps, o, dA);
                } else {
                    gaussian_head<DA>(hin, S.hold, mu, a, mo, adv, A.obj_kind, A.clip_eps, o, dA);
                }
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
            for (int d = 0; d < DA; ++d) {
                S.DMU[r * DA + d] = dmu[d], S.CMU[r * DA + d] = cmu[d];
                gB2w[d] += cmu[d], gLSw[d] += cls[d];      // per-thread partials, reduced over the warp at flush
            }
        }
        __syncthreads();
        // the forward MMAs are complete and MUP is consumed: re-fill the weight buffer for the backward MMAs
        load_weights(false);
        // ---- output layer (column role): out_W2 += H2^T CMU + ac R2^T DMU ; out_b2 += colsum CMU ; out_ls += colsum CLS
        {
            const int b0 = cp * BPP;
            const int off0 = core_off(b0, cj, SCA);      // rows b0 + bb at compile-time offsets (b0 is a multiple of 8)
            const float* cmu0 = S.CMU + b0 * DA;
            const float* dmu0 = S.DMU + b0 * DA;
#pragma unroll(BPP <= 16 ? 2 : 1)
            for (int b8 = 0; b8 < BPP; b8 += 8)
#pragma unroll
            for (int b1 = 0; b1 < 8; ++b1) {
                const int bb = b8 + b1;
                const int off = off0 + (bb >> 3) * 128 + (bb & 7) * 16;
                const float h = *reinterpret_cast<const float*>(S.T2a + off);
                const float rr = ac * *reinterpret_cast<const float*>(S.T2b + off);
#pragma unroll
                for (int d = 0; d < DA; ++d) gW2p[d] = fmaf(h, cmu0[bb * DA + d], fmaf(rr, dmu0[bb * DA + d], gW2p[d]));
            }
        }
        __syncthreads();
        // ---- D2 = dH2 g2 -> T2a ; C2 = CdH2 g2 + ac dH2 (act''/act')(H2) R2 -> T2b   (g2 = act'(H2); tanh: act''/act' = -2 H2)
        {
            float dm[DA], cm[DA];
#pragma unroll
            for (int d = 0; d < DA; ++d) dm[d] = S.DMU[r * DA + d], cm[d] = S.CMU[r * DA + d];
#pragma unroll
            for (int c4 = 0; c4 < CW / 4; ++c4) {
                float d2[4], c2[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = 4 * c4 + e;
                    float dh = 0.f, ch = 0.f;
#pragma unroll
                    for (int d = 0; d < DA; ++d) {
                        const float w2 = S.Ps[SL::W2 + (c0 + c) * DA + d], v2 = S.Vs[SL::W2 + (c0 + c) * DA + d];
                        dh = fmaf(dm[d], w2, dh);
                        ch = fmaf(cm[d], w2, fmaf(ac * dm[d], v2, ch));
                    }
                    d2[e] = dh * Act::d(h2[c]);
                    c2[e] = act_hvp_back<Act>(ch, dh, h2[c], r2[c], ac);
                }
                const int off = core_off(r, c0 + 4 * c4, SCA);
                *reinterpret_cast<float4*>(S.T2a + off) = make_float4(d2[0], d2[1], d2[2], d2[3]);
                *reinterpret_cast<float4*>(S.T2b + off) = make_float4(c2[0], c2[1], c2[2], c2[3]);
            }
        }
        __syncthreads();
        // ---- weight gradients out_W1 += H1^T C2 + R1^T (ac D2) (mma.sync 3xTF32) and colsum(C2)
        {
            float unused[NT] = {};
            wgrad_mma_tile<true, NT, true>(S.H1, S.T2b, 1.f, warp, lane, gW1, gB1f);
            wgrad_mma_tile<false, NT>(S.R1, S.T2a, ac, warp, lane, gW1, unused);
        }
        // ---- backward MMAs: dH1 = D2 W1^T ; CdH1 = C2 W1^T + D2 (ac V1)^T (registers), then
        //      C1 = CdH1 g1 + ac dH1 (act''/act')(H1) R1 -> H1 in place
        {
            float dacc[LNT][4], cacc[LNT][4];
            zero_frag<LNT>(dacc);
            zero_frag<LNT>(cacc);
            layer_gemm_issue<LNT>(dacc, S.T2a, S.WB[0], S.WB[1], warp, lane);
            layer_gemm_issue<LNT>(cacc, S.T2b, S.WB[0], S.WB[1], warp, lane);
            layer_gemm_issue<LNT>(cacc, S.T2a, S.WB[2], S.WB[3], warp, lane);
            wg_wait();
            wg_pin<LNT>(dacc);
            wg_pin<LNT>(cacc);
            __syncthreads();       // all reads of H1 / R1 / T2a are done before H1 and X (aliasing T2a) are overwritten
#pragma unroll
            for (int nt = 0; nt < LNT; ++nt)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int off = frag_off<LNT>(warp, lane, nt, h);
                    float2* p = reinterpret_cast<float2*>(S.H1 + off);
                    const float2 hv = *p;
                    const float2 rv = *reinterpret_cast<const float2*>(S.R1 + off);
                    const float dx = dacc[nt][2 * h], dy = dacc[nt][2 * h + 1];
                    *p = make_float2(act_hvp_back<Act>(cacc[nt][2 * h], dx, hv.x, rv.x, ac),
                                     act_hvp_back<Act>(cacc[nt][2 * h + 1], dy, hv.y, rv.y, ac));
                }
        }
        if constexpr (XPRE) {  // D2 (T2a) is dead: bring the observations back for the input-layer gradient
#pragma unroll
            for (int e = 0; e < XR; ++e) sX[tid + e * TCT] = xc[e];
        } else {
            load_x();
        }
        __syncthreads();
        // ---- out_W0 += X^T C1 ; out_b0 += colsum C1 (column role)
        {
            const int b0 = cp * BPP;
            const unsigned char* colp = S.H1 + core_off(b0, cj, SCA);
            const float* x0 = sX + b0 * DOP;
#pragma unroll(BPP <= 16 ? 2 : 1)
            for (int b8 = 0; b8 < BPP; b8 += 8)
#pragma unroll
            for (int b1 = 0; b1 < 8; ++b1) {
                const int bb = b8 + b1;
                const float c1 = *reinterpret_cast<const float*>(colp + (bb >> 3) * 128 + (bb & 7) * 16);
                gB0c += c1;
#pragma unroll
                for (int i = 0; i < DO; ++i) gW0p[i] = fmaf(x0[bb * DOP + i], c1, gW0p[i]);
            }
        }
    }
    if (cur_m >= 0) flush(cur_m);
}

template <int DO, int DA, int NQ, class Act>
__device__ __forceinline__ void policy_hvp_tc_body(const PolicyArgs& A) {
    using SM = HvpTcSmem<DO, DA, NQ>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SM& S = *reinterpret_cast<SM*>(smem_raw);
    const UniformSched sc(A.M, A.N, A.q, A.kmax, TBT);
    const float* cached_th = nullptr;
    hvp_tc_tiles<DO, DA, NQ, Act>(A, S, sc, cached_th);
}
template <int DO, int DA, int NQ>
__global__ void __launch_bounds__(128 * NQ, 1) policy_hvp_tc_kernel(PolicyArgs A) { policy_hvp_tc_body<DO, DA, NQ, ActTanh>(A); }
template <int DO, int DA, int NQ>
__global__ void __launch_bounds__(128 * NQ, 1) policy_hvp_tc_relu_kernel(PolicyArgs A) { policy_hvp_tc_body<DO, DA, NQ, ActRelu>(A); }
template <int DO, int DA, int NQ, class Hid>
__global__ void __launch_bounds__(128 * NQ, 1) policy_hvp_tc_otanh_kernel(PolicyArgs A) {
    policy_hvp_tc_body<DO, DA, NQ, OutTanh<Hid>>(A);
}

// =================================================================================================================
// Dataflow kernel: the whole gradient chain of one meta-objective evaluation in ONE persistent launch
//   stage 0..S-2   inner gradients + SGD step (theta_{s+1,m} = theta_{s,m} - alpha grad)        grad_tc_tiles
//   stage S-1      outer gradient v_m at the adapted parameters                                  grad_tc_tiles
//   stage S..      backward chain v_m <- v_m - alpha H v_m + c grad KL                           hvp_tc_tiles
// Stage k of task m only depends on stage k-1 of the SAME task, so the stages of different tasks overlap: CTAs pull work
// items (a few consecutive tiles of one task in one stage; ids ordered by stage, then task) from a device-side queue,
// the last arriver of a (stage, task) reduces its partial slots in item order (deterministic) and raises that task's
// ready flag, and an item of stage k+1 spins on the flag of its task before it reads the parameters / direction vector
// the previous stage produced.  Every id below the one a CTA holds has been taken by a CTA that is already running, so
// the spin always terminates whatever the residency.  Versus three launches this removes the tile-quantisation loss of
// each launch (640 tiles on 132 SMs = 5 rounds for 4.8), two launch tails and the idle time between them; the items of
// the last stage get smaller towards the end so the final imbalance is one tile.
// Control words (queue, finished-CTA count, ready flags, arrival counters) are zero on entry and left zero by the last
// CTA to finish.
constexpr int CHAIN_MAX_STAGES = 6;
constexpr int CHAIN_MAX_REGIONS = 3;
struct ChainStageInfo {
    int kind;                              // 0 = gradient stage, 1 = HVP stage
    int ntiles;                            // 128-sample tiles per task
    int item_base, n_items;                // global ids of the stage's items: [item_base, item_base + n_items)
    int n_regions;
    int reg_m0[CHAIN_MAX_REGIONS + 1];     // region r = tasks [reg_m0[r], reg_m0[r+1])
    int reg_q[CHAIN_MAX_REGIONS];          // tiles per item in region r
    int reg_item0[CHAIN_MAX_REGIONS];      // stage-relative id of the region's first item
};
struct ChainArgs {
    int n_stages, n_items, M;
    int* ctrl;                             // [0] work queue, [1] finished CTAs
    int* ready;                            // [n_stages][M]
    const int* skip_flag;                  // launch re-use of stage 0 (see PolicyArgs): both null or both set
    const float* skip_theta;
    ChainStageInfo info[CHAIN_MAX_STAGES];
    PolicyArgs st[CHAIN_MAX_STAGES];
};

template <int DO, int DA, int NQ>
struct ChainSmem {
    static constexpr int BODY = (int)((sizeof(GradTcSmem<DO, DA, NQ>) > sizeof(HvpTcSmem<DO, DA, NQ>) ? sizeof(GradTcSmem<DO, DA, NQ>)
                                                                                                    : sizeof(HvpTcSmem<DO, DA, NQ>)) + 15) / 16 * 16;
    static constexpr int SIZE = BODY + 16;     // + current item
};

// One chain kernel per translation unit (policy.cu / policy_relu.cu / policy_otanh.cu / policy_relu_otanh.cu), for that unit's
// activation: policy_chain_tc_kernel (tanh), policy_chain_tc_relu_kernel (ReLU), policy_chain_tc_otanh_kernel (tanh, tanh
// output) or policy_chain_tc_relu_otanh_kernel (ReLU, tanh output).  The body is written in the kernel itself: passed on to a
// device function by reference, the __grid_constant__ argument changed the tanh kernels' code.
#if defined(PROMP_POLICY_RELU_TU) && defined(PROMP_POLICY_OTANH_TU)
#define PROMP_CHAIN_KERNEL policy_chain_tc_relu_otanh_kernel
using ChainAct = OutTanh<ActRelu>;
#elif defined(PROMP_POLICY_OTANH_TU)
#define PROMP_CHAIN_KERNEL policy_chain_tc_otanh_kernel
using ChainAct = OutTanh<ActTanh>;
#elif defined(PROMP_POLICY_RELU_TU)
#define PROMP_CHAIN_KERNEL policy_chain_tc_relu_kernel
using ChainAct = ActRelu;
#else
#define PROMP_CHAIN_KERNEL policy_chain_tc_kernel
using ChainAct = ActTanh;
#endif
// ADV = ADV_EITHER: the chain has an exploration stage (PROMP_OBJ_EXPLORE, the last stage): its items read the per-task weight
// adv[m] and wait for no other stage.
template <int DO, int DA, int NQ, bool HAS_HVP = true, int ADV = ADV_SAMPLE>
__global__ void __launch_bounds__(128 * NQ, 1) PROMP_CHAIN_KERNEL(const __grid_constant__ ChainArgs C) {
    using Act = ChainAct;
    using GS = GradTcSmem<DO, DA, NQ>;
    using HS = HvpTcSmem<DO, DA, NQ>;
    using L = PLayout<DO, DA, TC_HID>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GS& G = *reinterpret_cast<GS*>(smem_raw);              // the two layouts time-share the same bytes
    HS& H = *reinterpret_cast<HS*>(smem_raw);
    int* cur_item = reinterpret_cast<int*>(smem_raw + ChainSmem<DO, DA, NQ>::BODY);
    const int tid = threadIdx.x;

    // launch re-use: stage 0 repeats an earlier stand-alone launch whose outputs are still in place (see promp_policy_grad_ex)
    const bool skip0 = reuse_hit<L::P>(C.skip_flag, C.st[0].params, C.skip_theta);
#ifdef PROMP_EXP_CLOCKS
    if (tid == 0) g_chain_last[blockIdx.x] = clock64();
    const long long t_begin = clock64();
#endif
    const float* cached_g = nullptr;
    const float* cached_h = nullptr;
    for (;;) {
        __syncthreads();                                   // everybody is done with the previous item (and its *cur_item)
        if (tid == 0) *cur_item = atomicAdd(C.ctrl, 1);
        __syncthreads();
        const int it = *cur_item;
        if (it >= C.n_items) break;
        CCNT(6);
        int s = 0;
        while (s + 1 < C.n_stages && it >= C.info[s + 1].item_base) ++s;
        if (s == 0 && skip0) continue;
        const ChainStageInfo& I = C.info[s];
        const int j = it - I.item_base;
        int r = 0;
        while (r + 1 < I.n_regions && j >= I.reg_item0[r + 1]) ++r;
        const int q = I.reg_q[r], per_task = (I.ntiles + q - 1) / q;
        const int jr = j - I.reg_item0[r];
        const int mr = jr / per_task, k = jr - mr * per_task;
        const int m = I.reg_m0[r] + mr;
        ItemSched sc;
        sc.ntiles = I.ntiles;
        sc.g_lo = m * I.ntiles + k * q;
        sc.g_hi = m * I.ntiles + min(k * q + q, I.ntiles);
        sc.item = it;
        sc.first_item = I.item_base + I.reg_item0[r] + mr * per_task;
        sc.n_items = per_task;
        sc.ready_prev = (s > 0 && !(s == 1 && skip0)) ? C.ready + (s - 1) * C.M : nullptr;
        if constexpr (ADV == ADV_EITHER)
            if (C.st[s].adv_per_task) sc.ready_prev = nullptr;
        sc.ready_mine = C.ready + s * C.M;
        CCLK(0);
        if (!HAS_HVP || I.kind == 0) {
            cached_h = nullptr;
            grad_tc_tiles<DO, DA, NQ, Act, ItemSched, ADV>(C.st[s], G, sc, cached_g);
        } else if constexpr (HAS_HVP) {
            cached_g = nullptr;
            hvp_tc_tiles<DO, DA, NQ, Act>(C.st[s], H, sc, cached_h);
        }
    }
#ifdef PROMP_EXP_CLOCKS
    if (tid == 0) {
        atomicAdd(&g_chain_clk[8], (unsigned long long)(clock64() - t_begin));
        atomicAdd(&g_chain_clk[9], 1ull);
    }
#endif
    if (tid == 0) {
        __threadfence();
        if (atomicAdd(C.ctrl + 1, 1) == (int)gridDim.x - 1) {       // every CTA has left the loop: nobody reads the flags any more
            for (int i = 0; i < C.n_stages * C.M; ++i) C.ready[i] = 0;
            C.ctrl[0] = 0;
            C.ctrl[1] = 0;
            __threadfence();
        }
    }
}

}  // namespace promp
