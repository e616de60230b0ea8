// Sample processing: returns -> linear-feature baseline fit/predict -> GAE -> normalisation -> stats, ONE launch.
// Tasks are independent (the reference re-fits the shared baseline inside its task loop,
// samplers/meta_sample_processor.py:31-34).  Grid (C, M): CTA (c, m) owns a chunk of task m's trajectories:
//   front stage  rewards -> shared memory (one coalesced round trip), discounted-return scans out of shared memory,
//                returns written back coalesced, path statistics, and the chunk's slice of the Gram matrix
//                Phi^T [Phi | y] in float64 (4x4 register blocks over 32-sample feature tiles);
//   ticket       the chunk's partials go to the workspace, then one atomic ticket per task; the LAST CTA of a task
//   finish stage reduces the partials in fixed chunk order (deterministic), solves the ridge system (Crout Cholesky over
//                the whole CTA, the reference's x10 ridge / NaN retry rule), predicts, runs the GAE scans out of shared
//                memory, and writes normalised advantages.
// The scans, Gram matrix, solve and moments run in float64 like the reference's numpy/LAPACK path; inputs/outputs are
// float32.  HBM-bound stage (AI < 1 FLOP/B): per env-step it reads obs (4*Do B) twice + rew (4 B) twice and writes
// returns + advantages (8 B).
// Round-1 version (two launches, per-trajectory scans walking global memory in a load->fma->store chain, finish stage on
// M CTAs re-reading float64 intermediates from L2): 74 us at 40x20x100 / 285 us at 40x20x200x(17,6).
#include "common.cuh"

namespace promp {

constexpr int PS_THREADS = 256;
constexpr int PS_WARPS = PS_THREADS / 32;
constexpr int PS_TS = 32;           // samples per Gram tile
constexpr int PS_MAXCOL = 44;       // NC = F+1 <= 44  (obs_dim <= 19)
constexpr int PS_MAXBLK = 66;       // 4x4 blocks of the upper triangle, nb = 11
constexpr int PS_GP = PS_MAXBLK * 16;   // doubles per partial Gram
constexpr int PS_SMEM_SAMPLES_BYTES = 12;   // per staged sample: float64 value + float32 reward
constexpr int PS_RING = 4;          // TMA stages of the Gram loop (observation tiles in flight)
constexpr int PS_SMEM_BUDGET = 160 * 1024;  // above this the sample arrays stay in the (L2-resident) workspace

enum { PS_MODE_PROCESS = 0, PS_MODE_FIT_ONLY = 1 };
// Baseline kind as a template argument of process_fused_kernel.  PS_KIND_RUNTIME: ZERO or LINEAR_FEATURE, chosen by
// A.baseline_kind at run time (the kernels this file always had).  LINEAR_TIME and GIVEN are instantiations of their own,
// so the code the two runtime kinds run is compiled exactly as before.
constexpr int PS_KIND_RUNTIME = -1;

#ifdef PROMP_EXP_CLOCKS
__device__ unsigned long long g_proc_clk[16];
#define PCLK(i) do { __syncthreads(); if (threadIdx.x == 0 && blockIdx.y == 0 && (i >= 8 || blockIdx.x == 0)) { const long long t_ = clock64(); g_proc_clk[i] += (unsigned long long)(t_ - t_prev); t_prev = t_; } } while (0)
#else
#define PCLK(i) do { } while (0)
#endif

struct ProcArgs {
    int M, E, H, Do;
    const float* __restrict__ obs;
    const float* __restrict__ rew;
    double discount, gae_lambda, reg_coeff;
    int baseline_kind, normalize_adv, positive_adv;
    float* __restrict__ returns;
    float* __restrict__ adv;
    double* coeffs;
    double* stats;
    // workspace
    unsigned int* counters;   // [M] tickets, zero on entry, left zero
    double* gram_p;           // [M][C][PS_GP] partial Gram blocks
    double* stat_p;           // [M][C][8] partial path statistics
    double* ws64;             // [M][2][NS] float64 (returns | baseline->advantages): only used when the arrays do not fit smem
    int C, EPC;               // trajectory chunks per task, trajectories per chunk
    // variable-length paths (early termination, meta_sampler.py:116-125); path_off == nullptr: E paths of H steps each
    const int32_t* __restrict__ path_off;   // [M][Pmax+1] prefix sums, E := Pmax
    const int32_t* __restrict__ n_paths;    // [M]
    int NS;                   // sample stride between tasks (E*H, or Nmax for variable-length paths)
    int32_t* tpos;            // [M][NS] time index of every sample inside its path (variable-length only)
    // standalone LinearFeatureBaseline.fit: targets given by the caller instead of the return scan
    const double* __restrict__ target;      // [M][NS] or nullptr
    int mode;
    int chunk_cap;            // samples a front-stage CTA can stage in shared memory (0: use ws64)
    int finish_cap;           // samples the finish stage can stage in shared memory (0: use ws64)
    int tt_cap;               // entries of the shared-memory time-feature table t/100 (covers every step of fixed-horizon paths)
    int pred_tile;            // samples per TMA tile of the predict stage (0: no TMA ring there)
    const double* __restrict__ given;       // [M][NS] caller's baseline values (PROMP_BASELINE_GIVEN only)
};
__device__ __forceinline__ int n_paths_of(const ProcArgs& A, int m) { return (A.path_off && A.n_paths) ? __ldg(A.n_paths + m) : A.E; }
__device__ __forceinline__ int path_begin(const ProcArgs& A, int m, int e) {
    return A.path_off ? __ldg(A.path_off + (int64_t)m * (A.E + 1) + e) : e * A.H;
}

// block-wide reductions of K values at once: warp shuffles, one smem exchange
template <int K>
__device__ __forceinline__ void block_reduce(double (&v)[K], const int (&op)[K], double* red /* [PS_WARPS][K] */) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = op[k] == 0 ? warp_sum(v[k]) : op[k] == 1 ? warp_max(v[k]) : warp_min(v[k]);
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) red[w * K + k] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double t = red[k];
#pragma unroll
        for (int i = 1; i < PS_WARPS; ++i) {
            const double x = red[i * K + k];
            t = op[k] == 0 ? t + x : op[k] == 1 ? fmax(t, x) : fmin(t, x);
        }
        v[k] = t;
    }
}

// LinearFeatureBaseline._features (baselines/linear_baseline.py:101-106), column `col` of one sample, float64:
//   [clip(o,-10,10), clip(o)^2, t, t^2, t^3, 1] with t = step/100
__device__ __forceinline__ double feature_col(const float* __restrict__ o, int Do, int step, int col) {
    if (col < 2 * Do) {
        const double c = fmin(fmax((double)__ldg(o + (col < Do ? col : col - Do)), -10.0), 10.0);
        return col < Do ? c : c * c;
    }
    const double tt = (double)step / 100.0;
    const int k = col - 2 * Do;
    return k == 0 ? tt : k == 1 ? tt * tt : k == 2 ? tt * tt * tt : 1.0;
}

// shared-memory carve-up (dynamic): [tile | red | (front: val, rewf) or (finish: A, L, w, bval, rall)]

// ---------------------------------------------------------------------------------------------------------------
// Sum `cnt` values spaced `stride` doubles apart in chunk order, with the (independent) L2 loads issued 8 at a time so
// that a reduction over C partials costs ceil(C/8) memory round trips instead of C.
__device__ __forceinline__ double ordered_sum_ldcg(const double* p, int cnt, int64_t stride) {
    double v = 0.0;
    for (int c0 = 0; c0 < cnt; c0 += 8) {
        double x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] = (c0 + k < cnt) ? __ldcg(p + (int64_t)(c0 + k) * stride) : 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) v += x[k];
    }
    return v;
}

// One launch.  STAGE_F / STAGE_L: the front / finish stage keeps its sample arrays in shared memory.
// Latency notes (clock64 phase counters of tools/process_time.py): fp64 divide / sqrt cost 200-400 clk each and a
// dependent shared-memory load -> DFMA -> store step ~75 clk, so (i) the time features t/100 come from a per-CTA table
// (one divide per table entry, exact like the reference), (ii) the serial scans run in blocks of 4 steps whose loads are
// issued before the dependent DFMA chain, (iii) the Cholesky uses one rsqrt per column and multiplies by stored inverse
// pivots, (iv) partials written by other CTAs are fetched with batched independent loads.
// KIND (see PS_KIND_RUNTIME): LINEAR_TIME fits the 4 time features only (LinearTimeBaseline, linear_baseline.py:109-126):
// no observation is read, the chunk partials are its 5 x 5 Gram matrix [Phi | y]^T [Phi | y] (padded into the same 4x4
// block layout), and the prediction is the per-step table alone.  GIVEN reads the baseline values from A.given.
template <bool STAGE_F, bool STAGE_L, int KIND = PS_KIND_RUNTIME>
__global__ void __launch_bounds__(PS_THREADS, 3) process_fused_kernel(ProcArgs A) {
    constexpr bool TIME = KIND == PROMP_BASELINE_LINEAR_TIME, GIVEN = KIND == PROMP_BASELINE_GIVEN;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int c = blockIdx.x, m = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
    const int E = n_paths_of(A, m), H = A.H, Do = A.Do, NS = A.NS;
    const int F = TIME ? 4 : 2 * Do + 4, NC = F + 1, nb = (NC + 3) >> 2, NCP = nb * 4, nblk = nb * (nb + 1) / 2;
    const int T0 = TIME ? 0 : 2 * Do;                  // first time feature among the coefficients
    const bool linear = !GIVEN && (TIME || A.baseline_kind == PROMP_BASELINE_LINEAR_FEATURE);
    const int e_lo = min(E, c * A.EPC), e_hi = min(E, e_lo + A.EPC);
    const float* __restrict__ obs = A.obs + (int64_t)m * NS * Do;
    const float* __restrict__ rew = A.rew ? A.rew + (int64_t)m * NS : nullptr;
    int32_t* tpos = A.tpos ? A.tpos + (int64_t)m * NS : nullptr;

    __shared__ unsigned char blk_i[PS_MAXBLK], blk_j[PS_MAXBLK];
    __shared__ int s_last, s_flag;
    __shared__ double s_piv, s_reg;
    __shared__ unsigned char s_def[PS_MAXCOL];
    __shared__ double s_inv[PS_MAXCOL];

    // dynamic shared memory: [tt_s | U | rest].  U is a union of the two feature-tile buffers (Gram loop) and the 256 x 8
    // reduction scratch (used before / after the loop, and by the moments at the very end); front rest = [val | rewf | obs
    // ring], finish rest = [A | L | w | bval | rall]; the predict stage re-uses U..L as its observation ring and turns the
    // time-feature table into the time part of the prediction in place.
    double* tt_s = reinterpret_cast<double*>(smem_raw);     // A.tt_cap (even) time features t/100
    double* tile = tt_s + A.tt_cap;                          // 2 x (PS_TS x NCP) feature rows, double-buffered
    double* red = tile;                                      // 256 x 8: Gram group reduction / block_reduce scratch
    double* rest = tile + max(2 * PS_TS * NCP, PS_THREADS * 8);
    __shared__ __align__(8) uint64_t s_bar_g[PS_RING], s_bar_p[2];

#ifdef PROMP_EXP_CLOCKS
    long long t_prev = clock64();
#endif
    if (tid < nblk) {      // packed (bi <= bj) block index tables
        int i = 0, rem = tid;
        while (rem >= nb - i) { rem -= nb - i; ++i; }
        blk_i[tid] = (unsigned char)i;
        blk_j[tid] = (unsigned char)(i + rem);
    }
    for (int t = tid; t < A.tt_cap; t += PS_THREADS) tt_s[t] = (double)t / 100.0;      // exact divide, once per table entry
    if (tid == 0) {
        for (int i = 0; i < PS_RING; ++i) tma_mbar_init(&s_bar_g[i], 1);
        tma_mbar_init(&s_bar_p[0], 1);
        tma_mbar_init(&s_bar_p[1], 1);
        tma_mbar_fence_init();
    }

    // ================================================================================================ front stage
    const int n_lo = path_begin(A, m, e_lo), n_hi = path_begin(A, m, e_hi), ns = n_hi - n_lo;
    double* val = STAGE_F ? rest : A.ws64 + (int64_t)m * 2 * NS + n_lo;          // returns / targets of this chunk, float64
    float* rewf = STAGE_F ? reinterpret_cast<float*>(rest + A.chunk_cap) : nullptr;      // then the TMA ring (16-byte aligned)
    if (A.target) {
        const double* __restrict__ tg = A.target + (int64_t)m * NS + n_lo;
        for (int i = tid; i < ns; i += PS_THREADS) val[i] = tg[i];
    } else if (STAGE_F) {
        for (int i = tid; i < ns; i += PS_THREADS) rewf[i] = __ldg(rew + n_lo + i);
    }
    __syncthreads();
    PCLK(0);
    {
        // ---- discounted returns R_t = r_t + g R_{t+1}  (utils/utils.py:74-81) + path statistics; one thread per path,
        //      walking shared memory in blocks of 4 steps (loads first, then the dependent DFMA chain)
        double st[7] = {0, 0, 0, -1e300, 1e300, 0, 0};   // sum R0, sum G, sum G^2, max G, min G, sum r, sum r^2
        const double g = A.discount;
        for (int e = e_lo + tid; e < e_hi; e += PS_THREADS) {
            const int o = path_begin(A, m, e) - n_lo, L = path_begin(A, m, e + 1) - n_lo - o;
            if (A.target) {
                if (tpos) for (int t = 0; t < L; ++t) tpos[n_lo + o + t] = t;
                continue;
            }
            double R = 0.0, G = 0.0, sr2 = 0.0;
            int t = L - 1;
            for (; t >= 3; t -= 4) {
                double r[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) r[k] = (double)(STAGE_F ? rewf[o + t - k] : __ldg(rew + n_lo + o + t - k));
                double Rk[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) { R = fma(g, R, r[k]); Rk[k] = R; }
#pragma unroll
                for (int k = 0; k < 4; ++k) { val[o + t - k] = Rk[k]; G += r[k]; sr2 = fma(r[k], r[k], sr2); }
            }
            for (; t >= 0; --t) {
                const double r = (double)(STAGE_F ? rewf[o + t] : __ldg(rew + n_lo + o + t));
                R = fma(g, R, r);
                val[o + t] = R;
                G += r;
                sr2 = fma(r, r, sr2);
            }
            if (tpos) for (int k = 0; k < L; ++k) tpos[n_lo + o + k] = k;
            st[0] += R; st[1] += G; st[2] += G * G; st[3] = fmax(st[3], G); st[4] = fmin(st[4], G); st[5] += G; st[6] += sr2;
        }
        PCLK(1);
        if (!A.target) {
            const int op[7] = {0, 0, 0, 1, 2, 0, 0};
            if (A.EPC <= 32) {            // only warp 0 holds paths: no block-wide exchange needed
                if (tid < 32) {
#pragma unroll
                    for (int k = 0; k < 7; ++k) st[k] = op[k] == 0 ? warp_sum(st[k]) : op[k] == 1 ? warp_max(st[k]) : warp_min(st[k]);
                    if (lane == 0) {
#pragma unroll
                        for (int k = 0; k < 7; ++k) A.stat_p[((int64_t)m * A.C + c) * 8 + k] = st[k];
                    }
                }
            } else {
                block_reduce<7>(st, op, red);
                if (tid < 7) A.stat_p[((int64_t)m * A.C + c) * 8 + tid] = st[tid];
            }
        }
        __syncthreads();
        if (A.returns && !A.target)
            for (int i = tid; i < ns; i += PS_THREADS) A.returns[(int64_t)m * NS + n_lo + i] = (float)val[i];
    }

    PCLK(2);
    if constexpr (TIME) {
        // ---- time features only: thread-strided sums of f_a f_b (a <= b) and f_a y over the chunk, f = [t, t^2, t^3, 1]
        double s[14];
#pragma unroll
        for (int k = 0; k < 14; ++k) s[k] = 0.0;
        for (int i = tid; i < ns; i += PS_THREADS) {
            const int n = n_lo + i;
            const int step = tpos ? tpos[n] : n % H;
            const double tt = step < A.tt_cap ? tt_s[step] : (double)step / 100.0;
            const double f[4] = {tt, tt * tt, tt * tt * tt, 1.0}, y = val[i];
            int k = 0;
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = a; b < 4; ++b) s[k++] += f[a] * f[b];
#pragma unroll
            for (int a = 0; a < 4; ++a) s[10 + a] += f[a] * y;
        }
        const int op[14] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
        block_reduce<14>(s, op, red);
        double* gp = A.gram_p + ((int64_t)m * A.C + c) * PS_GP;
        if (tid == 0) {
#pragma unroll
            for (int idx = 0; idx < 48; ++idx) {           // blocks (0,0), (0,1), (1,1) of the 8 x 8 layout (nb = 2)
                const int b = idx >> 4, i = 4 * (b == 2) + ((idx >> 2) & 3), j = 4 * (b != 0) + (idx & 3);
                const int lo = min(i, j), hi = max(i, j);
                gp[idx] = hi < 4 ? s[lo * 4 - lo * (lo - 1) / 2 + (hi - lo)] : (hi == 4 && lo < 4) ? s[10 + lo] : 0.0;
            }
        }
    } else if (linear) {
    // ---- partial Gram matrix over this chunk's samples (baselines/linear_baseline.py:66-73): thread = (4x4 block, group)
        const int G = max(1, min(PS_THREADS / nblk, 8));
        const int blk = tid % nblk, g = tid / nblk;
        const bool active = g < G;
        const int bi = blk_i[active ? blk : 0], bj = blk_j[active ? blk : 0];
        double acc[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = 0.0;
        const int s_row = tid >> 3, part = tid & 7;          // feature rows: thread (sample s_row, column part)
        // generic tile builder (no TMA: unaligned sources, partial last tile): feature rows straight from global memory
        auto build = [&](int n0, double* dst) {
            const int tn = min(PS_TS, ns - n0);
            if (s_row < tn) {
                const int n = n_lo + n0 + s_row;
                const int step = tpos ? tpos[n] : n % H;
                const double tt = step < A.tt_cap ? tt_s[step] : (double)step / 100.0;
                const float* o = obs + (int64_t)n * Do;
                for (int col = part; col < NCP; col += 8) {
                    double v;
                    if (col < 2 * Do) {
                        const double cl = fmin(fmax((double)__ldg(o + (col < Do ? col : col - Do)), -10.0), 10.0);
                        v = col < Do ? cl : cl * cl;
                    } else {
                        const int kk = col - 2 * Do;      // t, t^2, t^3, 1, target, zero padding
                        v = kk == 0 ? tt : kk == 1 ? tt * tt : kk == 2 ? tt * tt * tt : kk == 3 ? 1.0 : kk == 4 ? val[n0 + s_row] : 0.0;
                    }
                    dst[s_row * NCP + col] = v;
                }
            }
        };
        double* tile2 = tile + PS_TS * NCP;                  // second tile buffer
        // Observation tiles (PS_TS consecutive samples = one contiguous block of PS_TS*Do floats) stream through a ring of
        // PS_RING shared-memory stages filled by 1-D TMA bulk copies (one elected thread, mbarrier completion): the L2 / HBM
        // latency of a tile is paid PS_RING-1 tiles ahead of its use.  Needs 16-byte aligned sources; otherwise (and for
        // the last partial tile) the rows are fetched with plain loads.
        float* ring = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(rest) +
                                               ((size_t)A.chunk_cap * PS_SMEM_SAMPLES_BYTES + 15) / 16 * 16);
        const float* obs_chunk = obs + (int64_t)n_lo * Do;
        const int tile_floats = PS_TS * Do;
        const int full_tiles = ns / PS_TS;
        const bool use_tma = STAGE_F && full_tiles > 0 && ((reinterpret_cast<uintptr_t>(obs_chunk) & 15) == 0);
        auto issue = [&](int t) {       // thread 0 only
            tma_load_1d(ring + (t % PS_RING) * tile_floats, obs_chunk + (int64_t)t * tile_floats, (uint32_t)tile_floats * 4u,
                        &s_bar_g[t % PS_RING]);
        };
        auto build_from_ring = [&](int t, double* dst) {
            const float* src = ring + (t % PS_RING) * tile_floats + s_row * Do;
            const int n = n_lo + t * PS_TS + s_row;
            const int step = tpos ? tpos[n] : n % H;
            const double tt = step < A.tt_cap ? tt_s[step] : (double)step / 100.0;
            for (int col = part; col < NCP; col += 8) {
                double v;
                if (col < 2 * Do) {
                    const double cl = fmin(fmax((double)src[col < Do ? col : col - Do], -10.0), 10.0);
                    v = col < Do ? cl : cl * cl;
                } else {
                    const int kk = col - 2 * Do;
                    v = kk == 0 ? tt : kk == 1 ? tt * tt : kk == 2 ? tt * tt * tt : kk == 3 ? 1.0 : kk == 4 ? val[t * PS_TS + s_row] : 0.0;
                }
                dst[s_row * NCP + col] = v;
            }
        };
        auto multiply = [&](const double* tb, int tn) {
            if (active) {
                for (int s = g; s < tn; s += G) {
                    const double2* ra = reinterpret_cast<const double2*>(tb + s * NCP + 4 * bi);
                    const double2* rb = reinterpret_cast<const double2*>(tb + s * NCP + 4 * bj);
                    const double2 a01 = ra[0], a23 = ra[1], b01 = rb[0], b23 = rb[1];
                    const double a[4] = {a01.x, a01.y, a23.x, a23.y}, b[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int q = 0; q < 4; ++q) acc[r * 4 + q] = fma(a[r], b[q], acc[r * 4 + q]);
                }
            }
        };
        int cur = 0;
        int done_tiles = 0;
        if (use_tma) {
            if (tid == 0)
                for (int t = 0; t < min(PS_RING - 1, full_tiles); ++t) issue(t);
            for (int t = 0; t < full_tiles; ++t) {
                tma_mbar_wait(&s_bar_g[t % PS_RING], (uint32_t)((t / PS_RING) & 1));
                build_from_ring(t, cur ? tile2 : tile);
                __syncthreads();                  // tile t complete; stage (t-1) % PS_RING is free (its tile was built before the previous barrier)
                if (tid == 0 && t + PS_RING - 1 < full_tiles) issue(t + PS_RING - 1);
                multiply(cur ? tile2 : tile, PS_TS);
                cur ^= 1;
            }
            done_tiles = full_tiles;
        }
        // remaining samples (everything when TMA is not usable): plain loads
        for (int n0 = done_tiles * PS_TS; n0 < ns; n0 += PS_TS) {
            __syncthreads();
            build(n0, tile);
            __syncthreads();
            multiply(tile, min(PS_TS, ns - n0));
        }
        PCLK(3);
        // deterministic group reduction (groups added in order g = 0..G-1), two halves of 8 accumulators
        double* gp = A.gram_p + ((int64_t)m * A.C + c) * PS_GP;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            __syncthreads();
            if (active) {
#pragma unroll
                for (int i = 0; i < 8; ++i) red[tid * 8 + i] = acc[half * 8 + i];
            }
            __syncthreads();
            for (int idx = tid; idx < nblk * 8; idx += PS_THREADS) {
                const int b = idx >> 3, i = idx & 7;
                double sum = 0.0;
                for (int gg = 0; gg < G; ++gg) sum += red[(gg * nblk + b) * 8 + i];
                gp[b * 16 + half * 8 + i] = sum;
            }
        }
    }

    PCLK(4);
    // ================================================================================================ ticket
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const unsigned int old = atomicAdd(A.counters + m, 1u);
        s_last = (old == (unsigned int)(A.C - 1));
        if (s_last) A.counters[m] = 0u;        // self-cleaning: the workspace is left ready for the next launch
    }
    __syncthreads();
    PCLK(5);
    if (!s_last) return;
    __threadfence();

    // ================================================================================================ finish stage
    const int N = path_begin(A, m, E);                 // valid samples of this task
    double* Afull = rest;                              // [NCP][NCP]
    const int LD = F | 1;
    double* Lm = Afull + NCP * NCP;                    // [F][LD] lower triangle
    double* wv = Lm + F * LD + (F * LD & 1);           // [PS_MAXCOL], 16-byte aligned
    double* bval = STAGE_L ? wv + PS_MAXCOL + 4 : A.ws64 + (int64_t)m * 2 * NS + NS;   // baseline -> advantages, float64
    float* rall = STAGE_L ? reinterpret_cast<float*>(bval + A.finish_cap) : nullptr;

    if (tid < 8 && A.mode == PS_MODE_PROCESS) {   // path statistics: sums for 0,1,2,5,6; max for 3; min for 4
        const double* sp = A.stat_p + (int64_t)m * A.C * 8 + tid;
        double v;
        if (tid == 3 || tid == 4) {
            v = __ldcg(sp);
            for (int cc = 1; cc < A.C; ++cc) {
                const double x = __ldcg(sp + cc * 8);
                v = (tid == 3) ? fmax(v, x) : fmin(v, x);
            }
        } else {
            v = ordered_sum_ldcg(sp, A.C, 8);
        }
        if (A.stats && tid < 7) A.stats[(int64_t)m * 8 + tid] = v;
    }
    if (STAGE_L && A.mode == PS_MODE_PROCESS)
        for (int n = tid; n < N; n += PS_THREADS) rall[n] = __ldg(rew + n);

    double reg_used = 0.0;
    if (linear) {
        for (int idx = tid; idx < nblk * 16; idx += PS_THREADS) {   // reduce the chunk partials in chunk order
            const double v = ordered_sum_ldcg(A.gram_p + (int64_t)m * A.C * PS_GP + idx, A.C, PS_GP);
            const int b = idx >> 4, r = (idx >> 2) & 3, q = idx & 3;
            const int i = 4 * blk_i[b] + r, j = 4 * blk_j[b] + q;
            Afull[i * NCP + j] = v;
            Afull[j * NCP + i] = v;
        }
        if (tid == 0) { s_reg = A.reg_coeff; s_flag = 0; }
        __syncthreads();
        PCLK(8);
        // ---- solve (Phi^T Phi + reg I) w = Phi^T y; retry with 10x reg on NaN, up to 5 tries (:68-77).
        //      Crout Cholesky, 4 lanes per row, one rsqrt per column (L_jj = d * rsqrt(d), inverse pivot kept for the
        //      solves).  A pivot that vanishes relative to its diagonal entry (only possible with reg_coeff = 0 and collinear
        //      features) marks the column rank-deficient: w_j = 0, which gives the same fitted values as the reference's
        //      minimum-norm lstsq solution (least-squares fits are unique in Phi w).
        const int ti = tid >> 4, tk = tid & 15;             // trailing-update role: rows ti, ti+16, .. x columns tk, tk+16, ..
        for (int attempt = 0; attempt < 5; ++attempt) {
            const double reg = s_reg;
            for (int idx = tid; idx < F * F; idx += PS_THREADS) {
                const int i = idx / F, j = idx - i * F;
                if (j <= i) Lm[i * LD + j] = Afull[i * NCP + j] + (i == j ? reg : 0.0);
            }
            __syncthreads();
            // Right-looking Cholesky over the whole CTA: after column j is scaled, all 256 threads apply its outer product
            // to the trailing triangle, so the critical path per column is one rsqrt + two barriers (every thread derives
            // the pivot itself from shared memory: no broadcast round; the diagonal keeps d, the solves multiply by 1/sqrt(d)).
            bool bad = false;
            for (int j = 0; j < F; ++j) {
                const double d = Lm[j * LD + j], a_orig = Afull[j * NCP + j] + reg;      // d stays in place: the solves use s_inv
                const bool deficient = d <= 1e-14 * fabs(a_orig) && d == d && isfinite(a_orig);
                const double inv = deficient ? 0.0 : rsqrt(d);      // d < 0 or NaN input -> NaN -> retry with a larger ridge
                if (!deficient && (!(inv > 0.0) || !isfinite(inv))) bad = true;
                if (tid == j) {
                    s_inv[j] = inv;
                    s_def[j] = deficient ? 1 : 0;
                } else if (tid > j && tid < F) {
                    Lm[tid * LD + j] *= inv;                          // rank-deficient column -> 0
                }
                __syncthreads();                                     // column j scaled
                for (int i = j + 1 + ti; i < F; i += 16) {
                    const double lij = Lm[i * LD + j];
                    for (int k = j + 1 + tk; k <= i; k += 16) Lm[i * LD + k] = fma(-lij, Lm[k * LD + j], Lm[i * LD + k]);
                }
                __syncthreads();                                     // trailing triangle updated: next pivot is final
            }
            // forward L z = b, backward L^T w = z on one warp: lane l owns rows l and l+32   (b = Gram column F)
            if (tid < 32) {
                double b0 = lane < F ? Afull[lane * NCP + F] : 0.0, b1 = lane + 32 < F ? Afull[(lane + 32) * NCP + F] : 0.0;
                for (int k = 0; k < F; ++k) {
                    const double mine = (k < 32 ? b0 : b1) * s_inv[k];         // s_inv = 0 for rank-deficient columns
                    const double zk = __shfl_sync(0xffffffffu, mine, k & 31);
                    if (lane == (k & 31)) { if (k < 32) b0 = zk; else b1 = zk; }
                    if (lane > k && lane < F) b0 = fma(-Lm[lane * LD + k], zk, b0);
                    if (lane + 32 > k && lane + 32 < F) b1 = fma(-Lm[(lane + 32) * LD + k], zk, b1);
                }
                for (int k = F - 1; k >= 0; --k) {
                    const double mine = (k < 32 ? b0 : b1) * s_inv[k];
                    const double wk = __shfl_sync(0xffffffffu, mine, k & 31);
                    if (lane == (k & 31)) { if (k < 32) b0 = wk; else b1 = wk; }
                    if (lane < k) b0 = fma(-Lm[k * LD + lane], wk, b0);
                    if (lane + 32 < k) b1 = fma(-Lm[k * LD + lane + 32], wk, b1);
                }
                if (lane < F) wv[lane] = b0;
                if (lane + 32 < F) wv[lane + 32] = b1;
                bool nf = (lane < F && !isfinite(b0)) || (lane + 32 < F && !isfinite(b1));
                nf = __any_sync(0xffffffffu, nf) || bad;
                if (lane == 0) {
                    s_flag = nf ? 0 : 1;
                    if (nf) s_reg = reg * 10.0;
                }
            }
            __syncthreads();
            reg_used = reg;
            if (s_flag) break;
        }
        PCLK(9);
        if (A.coeffs)
            for (int i = tid; i < F; i += PS_THREADS) A.coeffs[(int64_t)m * F + i] = wv[i];
        if (A.mode == PS_MODE_FIT_ONLY) {
            if (A.stats && tid == 0) A.stats[(int64_t)m * 8 + 7] = reg_used;
            return;
        }
        // ---- predict b_n = phi_n . w (baselines/linear_baseline.py:17-33): the time part of the dot product comes from a
        //      per-step table (overwriting the t/100 table in place), the observation part is 2*Do FMAs per sample
        double* tw = tt_s;                                  // [tt_cap] t*w_t + t^2*w_t2 + t^3*w_t3 + w_1, in place over t/100
        __syncthreads();                                    // every thread is done with A / L before they become the ring
        for (int t = tid; t < A.tt_cap; t += PS_THREADS) {
            const double tt = tt_s[t];
            tw[t] = fma(tt, wv[T0], fma(tt * tt, wv[T0 + 1], fma(tt * tt * tt, wv[T0 + 2], wv[T0 + 3])));
        }
        __syncthreads();
        auto time_part = [&](int n) {
            const int step = tpos ? tpos[n] : n % H;
            if (step < A.tt_cap) return tw[step];
            const double tt = (double)step / 100.0;          // beyond the table (very long variable-length paths)
            return fma(tt, wv[T0], fma(tt * tt, wv[T0 + 1], fma(tt * tt * tt, wv[T0 + 2], wv[T0 + 3])));
        };
        if constexpr (TIME) {
            for (int n = tid; n < N; n += PS_THREADS) bval[n] = time_part(n);
        } else {
            // Observations of the whole task stream through a 2-stage TMA ring of A.pred_tile samples (re-using the tile / A / L
            // area, which is dead by now): thread = one sample of the tile, row stride Do floats.
            int n_done = 0;
            const int PT = A.pred_tile;
            if (STAGE_L && PT > 0 && N >= PT && ((reinterpret_cast<uintptr_t>(obs) & 15) == 0)) {
                float* pring = reinterpret_cast<float*>(tile);
                const int ptiles = N / PT, pfloats = PT * Do;
                if (tid == 0) {
                    tma_load_1d(pring, obs, (uint32_t)pfloats * 4u, &s_bar_p[0]);
                    if (ptiles > 1) tma_load_1d(pring + pfloats, obs + pfloats, (uint32_t)pfloats * 4u, &s_bar_p[1]);
                }
                for (int t = 0; t < ptiles; ++t) {
                    tma_mbar_wait(&s_bar_p[t & 1], (uint32_t)((t >> 1) & 1));
                    if (tid < PT) {
                        const float* src = pring + (t & 1) * pfloats + tid * Do;
                        const int n = t * PT + tid;
                        double b = time_part(n), b2 = 0.0, b3 = 0.0, b4 = 0.0;      // four chains: the fp64 FMA latency, not its
                        int i = 0;                                                    // throughput, limits this loop
                        for (; i + 1 < Do; i += 2) {
                            const double c0 = fmin(fmax((double)src[i], -10.0), 10.0), c1 = fmin(fmax((double)src[i + 1], -10.0), 10.0);
                            b = fma(c0, wv[i], b);
                            b2 = fma(c0 * c0, wv[Do + i], b2);
                            b3 = fma(c1, wv[i + 1], b3);
                            b4 = fma(c1 * c1, wv[Do + i + 1], b4);
                        }
                        if (i < Do) {
                            const double c0 = fmin(fmax((double)src[i], -10.0), 10.0);
                            b = fma(c0, wv[i], b);
                            b2 = fma(c0 * c0, wv[Do + i], b2);
                        }
                        bval[n] = (b + b2) + (b3 + b4);
                    }
                    __syncthreads();                  // stage (t & 1) consumed
                    if (tid == 0 && t + 2 < ptiles)
                        tma_load_1d(pring + (t & 1) * pfloats, obs + (int64_t)(t + 2) * pfloats, (uint32_t)pfloats * 4u, &s_bar_p[t & 1]);
                }
                n_done = ptiles * PT;
            }
            for (int n = n_done + tid; n < N; n += PS_THREADS) {      // rest (tail / no TMA): straight from global memory
                const float* o = obs + (int64_t)n * Do;
                double b = time_part(n);
                for (int i = 0; i < Do; ++i) {
                    const double cl = fmin(fmax((double)__ldg(o + i), -10.0), 10.0);
                    b = fma(cl, wv[i], b);
                    b = fma(cl * cl, wv[Do + i], b);
                }
                bval[n] = b;
            }
        }
    } else {
        if (A.mode == PS_MODE_FIT_ONLY) return;
        for (int n = tid; n < N; n += PS_THREADS)                  // ZeroBaseline.predict, or the caller's values
            bval[n] = GIVEN ? __ldg(A.given + (int64_t)m * NS + n) : 0.0;
    }
    __syncthreads();
    PCLK(10);

    // ---- GAE: delta_t = r_t + g b_{t+1} - b_t (b_H = 0); A_t = delta_t + g*lam A_{t+1}  (samplers/base.py:151-162);
    //      blocks of 4 steps: loads and deltas first, then the dependent chain of 4 DFMAs
    const double gl = A.discount * A.gae_lambda, gd = A.discount;
    double mom[2] = {0.0, 0.0};
    for (int e = tid; e < E; e += PS_THREADS) {
        double b_next = 0.0, a_next = 0.0;
        const int o = path_begin(A, m, e), L = path_begin(A, m, e + 1) - o;
        int t = L - 1;
        for (; t >= 3; t -= 4) {
            double b[4], d[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) b[k] = bval[o + t - k];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const double r = (double)(STAGE_L ? rall[o + t - k] : __ldg(rew + o + t - k));
                d[k] = (r + gd * (k == 0 ? b_next : b[k - 1])) - b[k];
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) { a_next = d[k] + gl * a_next; d[k] = a_next; }
#pragma unroll
            for (int k = 0; k < 4; ++k) { bval[o + t - k] = d[k]; mom[0] += d[k]; }
            b_next = b[3];
        }
        for (; t >= 0; --t) {
            const double b = bval[o + t];
            const double r = (double)(STAGE_L ? rall[o + t] : __ldg(rew + o + t));
            const double a = (r + gd * b_next - b) + gl * a_next;
            bval[o + t] = a;
            mom[0] += a;
            a_next = a;
            b_next = b;
        }
    }
    __syncthreads();
    PCLK(11);

    // ---- per-task normalisation / positive shift (utils/utils.py:59-71; population std)
    double mean = 0.0, inv = 1.0;
    if (A.normalize_adv) {
        {
            double v[1] = {mom[0]};
            const int op[1] = {0};
            block_reduce<1>(v, op, red);
            mean = v[0] / (double)N;
        }
        double v[1] = {0.0};
        for (int n = tid; n < N; n += PS_THREADS) {
            const double d = bval[n] - mean;
            v[0] += d * d;
        }
        const int op[1] = {0};
        block_reduce<1>(v, op, red);
        inv = 1.0 / (sqrt(v[0] / (double)N) + 1e-8);
    }
    double mn = 0.0;
    if (A.positive_adv) {
        double v[1] = {1e300};
        for (int n = tid; n < N; n += PS_THREADS) v[0] = fmin(v[0], (bval[n] - mean) * inv);
        const int op[1] = {2};
        block_reduce<1>(v, op, red);
        mn = v[0];
    }
    for (int n = tid; n < N; n += PS_THREADS) {
        double a = (bval[n] - mean) * inv;
        if (A.positive_adv) a = (a - mn) + 1e-8;
        A.adv[(int64_t)m * NS + n] = (float)a;
    }
    for (int n = N + tid; n < NS; n += PS_THREADS) A.adv[(int64_t)m * NS + n] = 0.f;      // padding rows (variable-length paths)
    if (A.stats && tid == 0) A.stats[(int64_t)m * 8 + 7] = reg_used;
    PCLK(12);
}

__global__ void adj_avg_rewards_kernel(int64_t n, const float* rew, double mean, double inv, float* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)(((double)rew[i] - mean) * inv);
}

// E-MAML coefficient c_m = (mean_m r - mean_all) / (std_all + 1e-8) from the per-task reward sums stats[m][5..6]
// (samplers/meta_sample_processor.py:40-44 averaged over task m; trpo_maml.py:137-144).  n_m = n_valid[m] or N.  One warp;
// lane 0 sums the totals in task order in float64.  totals_out (may be NULL): [sum r, sum r^2, sum n] of these tasks.
// coeff (may be NULL): c_m, from totals_in when given (the totals of every rank), else from this launch's totals.  Every
// operation is rounded on its own (no contraction), in the order of the eager torch expression it replaces.
__global__ void emaml_coeff_kernel(int M, const double* __restrict__ stats, const int32_t* __restrict__ n_valid, int N,
                                   const double* __restrict__ totals_in, double* __restrict__ totals_out, float* __restrict__ coeff) {
    __shared__ double tot[3];
    const int lane = threadIdx.x;
    if (lane == 0) {
        double s = 0.0, q = 0.0, n = 0.0;
        for (int m = 0; m < M; ++m) {
            s = __dadd_rn(s, stats[(int64_t)m * 8 + 5]);
            q = __dadd_rn(q, stats[(int64_t)m * 8 + 6]);
            n = __dadd_rn(n, (double)(n_valid ? n_valid[m] : N));
        }
        if (totals_out) totals_out[0] = s, totals_out[1] = q, totals_out[2] = n;
        tot[0] = totals_in ? totals_in[0] : s;
        tot[1] = totals_in ? totals_in[1] : q;
        tot[2] = totals_in ? totals_in[2] : n;
    }
    __syncwarp();
    if (!coeff) return;
    const double mean = __ddiv_rn(tot[0], tot[2]);
    const double var = fmax(__dsub_rn(__ddiv_rn(tot[1], tot[2]), __dmul_rn(mean, mean)), 0.0);
    const double den = __dadd_rn(__dsqrt_rn(var), 1e-8);
    for (int m = lane; m < M; m += 32) {
        const int nm = n_valid ? n_valid[m] : N;
        coeff[m] = nm > 0 ? __double2float_rn(__ddiv_rn(__dsub_rn(__ddiv_rn(stats[(int64_t)m * 8 + 5], (double)nm), mean), den))
                          : 0.f;
    }
}

// LinearFeatureBaseline / LinearTimeBaseline (KIND) .predict (baselines/linear_baseline.py:17-33) for a flat list of paths
template <int KIND>
__global__ void baseline_predict_kernel(int n_paths, const int32_t* __restrict__ path_off, int Do, const float* __restrict__ obs,
                                        const double* __restrict__ coeffs, double* __restrict__ out) {
    constexpr bool TIME = KIND == PROMP_BASELINE_LINEAR_TIME;
    const int T0 = TIME ? 0 : 2 * Do;
    const int n_total = __ldg(path_off + n_paths);
    for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < n_total; n += gridDim.x * blockDim.x) {
        int lo = 0, hi = n_paths;           // path containing sample n: path_off[lo] <= n < path_off[lo+1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(path_off + mid) <= n) lo = mid; else hi = mid;
        }
        const int step = n - __ldg(path_off + lo);
        double b = 0.0;
        if constexpr (!TIME) {
            const float* o = obs + (int64_t)n * Do;
            for (int i = 0; i < Do; ++i) {
                const double cl = fmin(fmax((double)__ldg(o + i), -10.0), 10.0);
                b = fma(cl, coeffs[i], b);
                b = fma(cl * cl, coeffs[Do + i], b);
            }
        }
        const double tt = (double)step / 100.0;
        b = fma(tt, coeffs[T0], b);
        b = fma(tt * tt, coeffs[T0 + 1], b);
        b = fma(tt * tt * tt, coeffs[T0 + 2], b);
        out[n] = b + coeffs[T0 + 3];
    }
}

}  // namespace promp

using namespace promp;

// ---- launch geometry ------------------------------------------------------------------------------------------------
static int proc_tt_cap(int H, int NS, bool ragged) {
    const int n = ragged ? NS : H;
    return ((n < 1024 ? n : 1024) + 1) & ~1;      // even: keeps the areas behind the table 16-byte aligned
}
// F: the kind's feature count (proc_features); kinds 0 and 1 size for 2*Do+4 as they always have
static int proc_features(int Do, int kind) { return kind == PROMP_BASELINE_LINEAR_TIME ? 4 : 2 * Do + 4; }
static size_t proc_smem_fixed(int F, int tt_cap) {
    const int NC = F + 1, NCP = (NC + 3) / 4 * 4;
    const int u = 2 * PS_TS * NCP > PS_THREADS * 8 ? 2 * PS_TS * NCP : PS_THREADS * 8;      // tiles and scratch share one area
    return (size_t)(u + tt_cap) * 8;
}
static size_t proc_smem_finish_fixed(int F) {
    const int NC = F + 1, NCP = (NC + 3) / 4 * 4, LD = F | 1;
    return (size_t)(NCP * NCP + F * LD + (F * LD & 1) + PS_MAXCOL + 4) * 8;
}
struct ProcGeom {
    int C, EPC, chunk_cap, finish_cap, tt_cap, pred_tile;
    bool stage_f, stage_l;
    size_t smem;
};
// Shared memory of one CTA when a chunk holds `EPC` paths (front stage: the chunk's rewards + returns; finish stage: the
// task's rewards + baseline; whichever is larger, because any CTA may turn out to be the finisher).
// Invariant: !stage_f implies !stage_l.  front - fin = round16(chunk_samples*12) + ring - proc_smem_finish_fixed(Do) - NS*12
// with chunk_samples <= NS, and the Gram loop's TMA ring (PS_RING*PS_TS*Do*4 B) plus the 12 B of rounding is smaller than
// the finish stage's fixed arrays for every obs_dim 1..19, so front < fin: when the front stage does not fit, neither does
// the finish stage.  launch_process therefore has no <false, true> kernel.  The time kind reads no observations: no ring
// in either stage (and its finish stage's fixed arrays, 1056 B, still exceed the 12 B of rounding).
static ProcGeom proc_geom_for(int EPC, int E, int H, int Do, int NS, bool ragged, int kind) {
    ProcGeom g;
    const bool reads_obs = kind != PROMP_BASELINE_LINEAR_TIME;
    const int F = proc_features(Do, kind);
    g.EPC = EPC;
    g.C = (E + EPC - 1) / EPC;
    g.tt_cap = proc_tt_cap(H, NS, ragged);
    const int chunk_samples = ragged ? NS : EPC * H;
    const size_t fixed = proc_smem_fixed(F, g.tt_cap);
    const size_t ring = reads_obs ? (size_t)PS_RING * PS_TS * Do * 4 : 0;   // TMA stages of the Gram loop
    size_t front = fixed + ((size_t)chunk_samples * PS_SMEM_SAMPLES_BYTES + 15) / 16 * 16 + ring;
    size_t fin = fixed + proc_smem_finish_fixed(F) + (size_t)NS * PS_SMEM_SAMPLES_BYTES;
    // predict ring: 2 stages of pred_tile samples inside the (dead) tile / A / L area
    g.pred_tile = 0;
    if (reads_obs) {
        const int NC = F + 1, NCP = (NC + 3) / 4 * 4;
        const int LD = F | 1;
        const size_t avail = (size_t)(2 * PS_TS * NCP + NCP * NCP + F * LD) * 8;
        for (int pt = 256; pt >= 32; pt >>= 1)
            if ((size_t)2 * pt * Do * 4 <= avail) { g.pred_tile = pt; break; }
    }
    g.stage_f = front <= (size_t)PS_SMEM_BUDGET;
    g.stage_l = fin <= (size_t)PS_SMEM_BUDGET;
    if (!g.stage_f) front = fixed;
    if (!g.stage_l) fin = fixed + proc_smem_finish_fixed(F);
    g.chunk_cap = g.stage_f ? chunk_samples : 0;
    g.finish_cap = g.stage_l ? NS : 0;
    g.smem = (front > fin ? front : fin) + 16;
    return g;
}
// Chunking: ~4 CTAs per SM worth of chunks (the front stage is issue / latency-bound at 8-16 resident warps per SM, so
// short chunks on many CTAs beat one exact wave of longer ones: measured 33 vs 38 us at 40x20x100), never more than one
// CTA per path.
static ProcGeom proc_geom(int M, int E, int H, int Do, int NS, bool ragged, int kind) {
    int target = (4 * PROMP_NUM_SMS + M - 1) / M;
    if (target > E) target = E;
    if (target < 1) target = 1;
    const int EPC = (E + target - 1) / target;
    return proc_geom_for(EPC, E, H, Do, NS, ragged, kind);
}

struct ProcLayout {
    ProcGeom g;
    int64_t off_gram, off_stat, off_ws64, off_tpos, total;
};
// The offsets depend on C only, which no kind changes: one workspace size serves every kind.
static ProcLayout proc_layout(int M, int E, int H, int Do, int NS, bool ragged, int kind) {
    ProcLayout L;
    L.g = proc_geom(M, E, H, Do, NS, ragged, kind);
    // arrival tickets: a FIXED-size header (grid.y <= 65535 tasks), so a workspace shared by launches of different
    // shapes never finds stale partials where a later layout expects zeroed tickets
    int64_t o = 65536 * 4;
    L.off_gram = o;  o += (int64_t)M * L.g.C * PS_GP * 8;
    L.off_stat = o;  o += (int64_t)M * L.g.C * 8 * 8;
    L.off_ws64 = o;  o += (int64_t)M * 2 * NS * 8;
    L.off_tpos = o;  if (ragged) o += ((int64_t)M * NS * 4 + 7) / 8 * 8;
    L.total = o;
    return L;
}

template <int KIND>
static void (*proc_kernel(const ProcGeom& g))(ProcArgs) {
    return g.stage_f ? (g.stage_l ? process_fused_kernel<true, true, KIND> : process_fused_kernel<true, false, KIND>)
                     : process_fused_kernel<false, false, KIND>;
}

static int launch_process(ProcArgs& A, const ProcGeom& g, cudaStream_t stream) {
    A.C = g.C; A.EPC = g.EPC; A.chunk_cap = g.chunk_cap; A.finish_cap = g.finish_cap; A.tt_cap = g.tt_cap;
    A.pred_tile = g.pred_tile;
    PROMP_REQUIRE(g.stage_f || !g.stage_l, "process_fused_kernel: finish stage staged without a staged front stage "
                  "(M=%d E=%d Do=%d NS=%d); proc_geom_for's invariant is broken", A.M, A.E, A.Do, A.NS);
    const int slot = A.baseline_kind == PROMP_BASELINE_LINEAR_TIME ? 1 : A.baseline_kind == PROMP_BASELINE_GIVEN ? 2 : 0;
    auto kern = slot == 1 ? proc_kernel<PROMP_BASELINE_LINEAR_TIME>(g)
              : slot == 2 ? proc_kernel<PROMP_BASELINE_GIVEN>(g) : proc_kernel<PS_KIND_RUNTIME>(g);
    static size_t configured[3][3] = {};
    const int which = g.stage_f ? (g.stage_l ? 2 : 1) : 0;
    if (g.smem > configured[slot][which]) {
        PROMP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem));
        configured[slot][which] = g.smem;
    }
    kern<<<dim3(A.C, A.M), PS_THREADS, g.smem, stream>>>(A);
    PROMP_LAUNCH_CHECK("process_fused_kernel");
    return PROMP_OK;
}

extern "C" int promp_process_launch_info(int M, int max_paths, int H, int obs_dim, int NS, int ragged, int32_t* out) {
    PROMP_REQUIRE(M > 0 && max_paths > 0 && obs_dim > 0 && NS > 0 && out, "promp_process_launch_info: bad arguments");
    PROMP_REQUIRE(2 * obs_dim + 5 <= PS_MAXCOL, "promp_process_launch_info: obs_dim %d too large (max %d)", obs_dim,
                  (PS_MAXCOL - 5) / 2);
    PROMP_REQUIRE(ragged || (H > 0 && NS == max_paths * H), "promp_process_launch_info: fixed horizon needs NS = E*H");
    const ProcGeom g = proc_geom(M, max_paths, ragged ? 0 : H, obs_dim, NS, ragged != 0, PROMP_BASELINE_LINEAR_FEATURE);
    const int32_t v[8] = {g.C, g.EPC, g.chunk_cap, g.finish_cap, g.tt_cap, g.pred_tile, g.stage_f ? 1 : 0, g.stage_l ? 1 : 0};
    for (int i = 0; i < 8; ++i) out[i] = v[i];
    return PROMP_OK;
}

extern "C" int64_t promp_process_workspace_bytes(int M, int E, int H, int obs_dim) {
    return proc_layout(M, E, H, obs_dim, E * H, false, PROMP_BASELINE_LINEAR_FEATURE).total;
}

// kind: ZERO, LINEAR_FEATURE, LINEAR_TIME, or GIVEN with `given` set (obs is not read by the last two)
static int process_fixed(const char* who, int M, int E, int H, int obs_dim, const float* obs, const float* rew,
                         const double* given, double discount, double gae_lambda, double reg_coeff, int baseline_kind,
                         int normalize_adv, int positive_adv, float* returns, float* adv, double* coeffs, double* stats,
                         void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(M > 0 && E > 0 && H > 0 && obs_dim > 0, "%s: dimensions must be positive", who);
    PROMP_REQUIRE(M <= 65535, "%s: M=%d exceeds the grid.y limit", who, M);
    PROMP_REQUIRE(2 * obs_dim + 5 <= PS_MAXCOL, "%s: obs_dim %d too large (max %d)", who, obs_dim, (PS_MAXCOL - 5) / 2);
    PROMP_REQUIRE(obs && rew && returns && adv && workspace, "%s: null pointer argument", who);
    PROMP_REQUIRE(discount >= 0.0 && discount <= 1.0 && gae_lambda >= 0.0 && gae_lambda <= 1.0,
                  "%s: discount and gae_lambda must be in [0,1]", who);   // samplers/base.py:56-57
    const ProcLayout L = proc_layout(M, E, H, obs_dim, E * H, false, baseline_kind);
    if (workspace_bytes < L.total) {
        set_error("%s: workspace too small (%lld < %lld bytes)", who, (long long)workspace_bytes, (long long)L.total);
        return PROMP_ERR_WORKSPACE;
    }
    unsigned char* w = (unsigned char*)workspace;
    ProcArgs A{};
    A.M = M; A.E = E; A.H = H; A.Do = obs_dim; A.obs = obs; A.rew = rew;
    A.discount = discount; A.gae_lambda = gae_lambda; A.reg_coeff = reg_coeff;
    A.baseline_kind = baseline_kind; A.normalize_adv = normalize_adv; A.positive_adv = positive_adv;
    A.returns = returns; A.adv = adv; A.coeffs = coeffs; A.stats = stats;
    A.counters = (unsigned int*)w; A.gram_p = (double*)(w + L.off_gram); A.stat_p = (double*)(w + L.off_stat);
    A.ws64 = (double*)(w + L.off_ws64);
    A.path_off = nullptr; A.n_paths = nullptr; A.NS = E * H; A.tpos = nullptr;
    A.target = nullptr; A.mode = PS_MODE_PROCESS; A.given = given;
    return launch_process(A, L.g, (cudaStream_t)stream);
}

extern "C" int promp_process_samples(int M, int E, int H, int obs_dim, const float* obs, const float* rew,
                                     double discount, double gae_lambda, double reg_coeff, int baseline_kind,
                                     int normalize_adv, int positive_adv, float* returns, float* adv, double* coeffs,
                                     double* stats, void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(baseline_kind == PROMP_BASELINE_ZERO || baseline_kind == PROMP_BASELINE_LINEAR_FEATURE ||
                  baseline_kind == PROMP_BASELINE_LINEAR_TIME, "promp_process_samples: unknown baseline kind %d", baseline_kind);
    return process_fixed("promp_process_samples", M, E, H, obs_dim, obs, rew, nullptr, discount, gae_lambda, reg_coeff,
                         baseline_kind, normalize_adv, positive_adv, returns, adv, coeffs, stats, workspace, workspace_bytes,
                         stream);
}

// MetaSampleProcessor with a host baseline object (samplers/base.py:99-108): the caller's predict(path) values, GAE onwards
extern "C" int promp_process_samples_given(int M, int E, int H, int obs_dim, const float* obs, const float* rew,
                                           const double* baseline_values, double discount, double gae_lambda, int normalize_adv,
                                           int positive_adv, float* returns, float* adv, double* stats,
                                           void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(baseline_values, "promp_process_samples_given: null baseline_values");
    return process_fixed("promp_process_samples_given", M, E, H, obs_dim, obs, rew, baseline_values, discount, gae_lambda,
                         0.0, PROMP_BASELINE_GIVEN, normalize_adv, positive_adv, returns, adv, nullptr, stats, workspace,
                         workspace_bytes, stream);
}

extern "C" int promp_adj_avg_rewards(int64_t n, const float* rew, double mean, double std, float* out, void* stream) {
    PROMP_REQUIRE(n > 0 && rew && out, "promp_adj_avg_rewards: bad arguments");
    const int bs = 256;
    adj_avg_rewards_kernel<<<(unsigned)((n + bs - 1) / bs), bs, 0, (cudaStream_t)stream>>>(n, rew, mean,
                                                                                         1.0 / (std + 1e-8), out);
    PROMP_LAUNCH_CHECK("adj_avg_rewards_kernel");
    return PROMP_OK;
}

static int emaml_launch(const char* who, int M, const double* stats, const int32_t* n_valid, int N, const double* totals_in,
                        double* totals_out, float* coeff, void* stream) {
    PROMP_REQUIRE(M > 0 && stats && (n_valid || N > 0), "%s: bad arguments (M = %d, N = %d)", who, M, N);
    emaml_coeff_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(M, stats, n_valid, N, totals_in, totals_out, coeff);
    PROMP_LAUNCH_CHECK("emaml_coeff_kernel");
    return PROMP_OK;
}
extern "C" int promp_emaml_coeff(int M, const double* stats, const int32_t* n_valid, int N, float* coeff, void* stream) {
    PROMP_REQUIRE(coeff, "promp_emaml_coeff: null coeff");
    return emaml_launch("promp_emaml_coeff", M, stats, n_valid, N, nullptr, nullptr, coeff, stream);
}
extern "C" int promp_emaml_totals(int M, const double* stats, const int32_t* n_valid, int N, double* totals, void* stream) {
    PROMP_REQUIRE(totals, "promp_emaml_totals: null totals");
    return emaml_launch("promp_emaml_totals", M, stats, n_valid, N, nullptr, totals, nullptr, stream);
}
extern "C" int promp_emaml_finish(int M, const double* stats, const int32_t* n_valid, int N, const double* totals, float* coeff,
                                  void* stream) {
    PROMP_REQUIRE(totals && coeff, "promp_emaml_finish: null totals / coeff");
    return emaml_launch("promp_emaml_finish", M, stats, n_valid, N, totals, nullptr, coeff, stream);
}

// ---- variable-length paths: same kernel driven by a per-task path table ------------------------------------------
extern "C" int64_t promp_process_workspace_bytes_ragged(int M, int max_paths, int max_samples, int obs_dim) {
    return proc_layout(M, max_paths, 0, obs_dim, max_samples, true, PROMP_BASELINE_LINEAR_FEATURE).total;
}

static int process_ragged(const char* who, int M, int max_paths, int max_samples, int obs_dim, const float* obs,
                          const float* rew, const int32_t* path_off, const int32_t* n_paths, const double* given,
                          double discount, double gae_lambda, double reg_coeff, int baseline_kind, int normalize_adv,
                          int positive_adv, float* returns, float* adv, double* coeffs, double* stats,
                          void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(M > 0 && max_paths > 0 && max_samples > 0 && obs_dim > 0, "%s: dimensions must be positive", who);
    PROMP_REQUIRE(M <= 65535, "%s: M=%d exceeds the grid.y limit", who, M);
    PROMP_REQUIRE(2 * obs_dim + 5 <= PS_MAXCOL, "%s: obs_dim %d too large (max %d)", who, obs_dim, (PS_MAXCOL - 5) / 2);
    PROMP_REQUIRE(obs && rew && returns && adv && workspace && path_off && n_paths, "%s: null pointer argument", who);
    PROMP_REQUIRE(discount >= 0.0 && discount <= 1.0 && gae_lambda >= 0.0 && gae_lambda <= 1.0,
                  "%s: discount and gae_lambda must be in [0,1]", who);
    const ProcLayout L = proc_layout(M, max_paths, 0, obs_dim, max_samples, true, baseline_kind);
    if (workspace_bytes < L.total) {
        set_error("%s: workspace too small (%lld < %lld bytes)", who, (long long)workspace_bytes, (long long)L.total);
        return PROMP_ERR_WORKSPACE;
    }
    unsigned char* w = (unsigned char*)workspace;
    ProcArgs A{};
    A.M = M; A.E = max_paths; A.H = 0; A.Do = obs_dim; A.obs = obs; A.rew = rew;
    A.discount = discount; A.gae_lambda = gae_lambda; A.reg_coeff = reg_coeff;
    A.baseline_kind = baseline_kind; A.normalize_adv = normalize_adv; A.positive_adv = positive_adv;
    A.returns = returns; A.adv = adv; A.coeffs = coeffs; A.stats = stats;
    A.counters = (unsigned int*)w; A.gram_p = (double*)(w + L.off_gram); A.stat_p = (double*)(w + L.off_stat);
    A.ws64 = (double*)(w + L.off_ws64);
    A.path_off = path_off; A.n_paths = n_paths; A.NS = max_samples;
    A.tpos = (int32_t*)(w + L.off_tpos);
    A.target = nullptr; A.mode = PS_MODE_PROCESS; A.given = given;
    return launch_process(A, L.g, (cudaStream_t)stream);
}

extern "C" int promp_process_samples_ragged(int M, int max_paths, int max_samples, int obs_dim, const float* obs,
                                            const float* rew, const int32_t* path_off, const int32_t* n_paths, double discount,
                                            double gae_lambda, double reg_coeff, int baseline_kind, int normalize_adv,
                                            int positive_adv, float* returns, float* adv, double* coeffs, double* stats,
                                            void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(baseline_kind == PROMP_BASELINE_ZERO || baseline_kind == PROMP_BASELINE_LINEAR_FEATURE ||
                  baseline_kind == PROMP_BASELINE_LINEAR_TIME, "promp_process_samples_ragged: unknown baseline kind %d",
                  baseline_kind);
    return process_ragged("promp_process_samples_ragged", M, max_paths, max_samples, obs_dim, obs, rew, path_off, n_paths,
                          nullptr, discount, gae_lambda, reg_coeff, baseline_kind, normalize_adv, positive_adv, returns, adv,
                          coeffs, stats, workspace, workspace_bytes, stream);
}

extern "C" int promp_process_samples_ragged_given(int M, int max_paths, int max_samples, int obs_dim, const float* obs,
                                                  const float* rew, const int32_t* path_off, const int32_t* n_paths,
                                                  const double* baseline_values, double discount, double gae_lambda,
                                                  int normalize_adv, int positive_adv, float* returns, float* adv,
                                                  double* stats, void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(baseline_values, "promp_process_samples_ragged_given: null baseline_values");
    return process_ragged("promp_process_samples_ragged_given", M, max_paths, max_samples, obs_dim, obs, rew, path_off,
                          n_paths, baseline_values, discount, gae_lambda, 0.0, PROMP_BASELINE_GIVEN, normalize_adv,
                          positive_adv, returns, adv, nullptr, stats, workspace, workspace_bytes, stream);
}

// ---- standalone LinearFeatureBaseline / LinearTimeBaseline .fit / predict (baselines/linear_baseline.py:55-77, 17-33) ---
extern "C" int64_t promp_baseline_fit_workspace_bytes(int n_paths, int n_samples, int obs_dim) {
    return proc_layout(1, n_paths, 0, obs_dim, n_samples, true, PROMP_BASELINE_LINEAR_FEATURE).total;
}

// kind: LINEAR_FEATURE or LINEAR_TIME (LinearTimeBaseline, linear_baseline.py:109-126; obs is not read and may be NULL)
extern "C" int promp_baseline_fit_ex(int kind, int n_paths, int n_samples, int obs_dim, const float* obs, const double* target,
                                     const int32_t* path_off, double reg_coeff, double* coeffs, double* reg_used,
                                     void* workspace, int64_t workspace_bytes, void* stream) {
    PROMP_REQUIRE(kind == PROMP_BASELINE_LINEAR_FEATURE || kind == PROMP_BASELINE_LINEAR_TIME,
                  "promp_baseline_fit: unknown baseline kind %d", kind);
    PROMP_REQUIRE(n_paths > 0 && n_samples > 0 && obs_dim > 0, "promp_baseline_fit: dimensions must be positive");
    PROMP_REQUIRE(2 * obs_dim + 5 <= PS_MAXCOL, "promp_baseline_fit: obs_dim %d too large (max %d)", obs_dim, (PS_MAXCOL - 5) / 2);
    PROMP_REQUIRE((obs || kind == PROMP_BASELINE_LINEAR_TIME) && target && path_off && coeffs && workspace,
                  "promp_baseline_fit: null pointer argument");
    const ProcLayout L = proc_layout(1, n_paths, 0, obs_dim, n_samples, true, kind);
    if (workspace_bytes < L.total) {
        set_error("promp_baseline_fit: workspace too small (%lld < %lld bytes)", (long long)workspace_bytes, (long long)L.total);
        return PROMP_ERR_WORKSPACE;
    }
    unsigned char* w = (unsigned char*)workspace;
    // n_paths lives on the host here; the kernel reads it through the path table of its single task
    ProcArgs A{};
    A.M = 1; A.E = n_paths; A.H = 0; A.Do = obs_dim; A.obs = obs; A.rew = nullptr;
    A.discount = 0.0; A.gae_lambda = 0.0; A.reg_coeff = reg_coeff;
    A.baseline_kind = kind; A.normalize_adv = 0; A.positive_adv = 0;
    A.returns = nullptr; A.adv = nullptr; A.coeffs = coeffs; A.stats = nullptr;
    A.counters = (unsigned int*)w; A.gram_p = (double*)(w + L.off_gram); A.stat_p = (double*)(w + L.off_stat);
    A.ws64 = (double*)(w + L.off_ws64);
    A.path_off = path_off; A.n_paths = nullptr; A.NS = n_samples;
    A.tpos = (int32_t*)(w + L.off_tpos);
    A.target = target; A.mode = PS_MODE_FIT_ONLY;
    // reg_used is reported through an 8-double stats row when requested
    A.stats = reg_used ? reg_used - 7 : nullptr;
    return launch_process(A, L.g, (cudaStream_t)stream);
}

extern "C" int promp_baseline_fit(int n_paths, int n_samples, int obs_dim, const float* obs, const double* target,
                                  const int32_t* path_off, double reg_coeff, double* coeffs, double* reg_used,
                                  void* workspace, int64_t workspace_bytes, void* stream) {
    return promp_baseline_fit_ex(PROMP_BASELINE_LINEAR_FEATURE, n_paths, n_samples, obs_dim, obs, target, path_off, reg_coeff,
                                 coeffs, reg_used, workspace, workspace_bytes, stream);
}

extern "C" int promp_baseline_predict_ex(int kind, int n_paths, int n_samples, int obs_dim, const float* obs,
                                         const int32_t* path_off, const double* coeffs, double* out, void* stream) {
    PROMP_REQUIRE(kind == PROMP_BASELINE_LINEAR_FEATURE || kind == PROMP_BASELINE_LINEAR_TIME,
                  "promp_baseline_predict: unknown baseline kind %d", kind);
    PROMP_REQUIRE(n_paths > 0 && n_samples > 0 && obs_dim > 0, "promp_baseline_predict: dimensions must be positive");
    PROMP_REQUIRE((obs || kind == PROMP_BASELINE_LINEAR_TIME) && path_off && coeffs && out,
                  "promp_baseline_predict: null pointer argument");
    const int bs = 256;
    int grid = (n_samples + bs - 1) / bs;
    if (grid > PROMP_NUM_SMS * 8) grid = PROMP_NUM_SMS * 8;
    auto kern = kind == PROMP_BASELINE_LINEAR_TIME ? baseline_predict_kernel<PROMP_BASELINE_LINEAR_TIME>
                                                   : baseline_predict_kernel<PROMP_BASELINE_LINEAR_FEATURE>;
    kern<<<grid, bs, 0, (cudaStream_t)stream>>>(n_paths, path_off, obs_dim, obs, coeffs, out);
    PROMP_LAUNCH_CHECK("baseline_predict_kernel");
    return PROMP_OK;
}

extern "C" int promp_baseline_predict(int n_paths, int n_samples, int obs_dim, const float* obs, const int32_t* path_off,
                                      const double* coeffs, double* out, void* stream) {
    return promp_baseline_predict_ex(PROMP_BASELINE_LINEAR_FEATURE, n_paths, n_samples, obs_dim, obs, path_off, coeffs, out,
                                     stream);
}

#ifdef PROMP_EXP_CLOCKS
extern "C" int promp_debug_proc_clocks(unsigned long long* out16, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out16, promp::g_proc_clk, 16 * sizeof(unsigned long long));
    if (reset) {
        unsigned long long z[16] = {0};
        cudaMemcpyToSymbol(promp::g_proc_clk, z, sizeof(z));
    }
    return 0;
}
#endif
