// softmax_rows.cuh -- streaming row-softmax building blocks for the (T,B,N) / (B,N) logits tensors
// of V-trace, UPGO and PPO.
//
// The reference spends one 256-thread block per row and five block-wide reductions
// (include/hpc/rll/cuda/rl_utils/vtrace_kernel.h:11-112, upgo_kernel.h:40-81,
// ppo_kernel.h:12-112) and materialises three (T,B,N) gradient buffers in the forward pass.
// Here a row lives in the registers of a sub-warp group of G lanes (G = 1..32, a power of two chosen
// so that every lane owns up to four 128-bit chunks: N=16 -> one lane per row, N=128 -> 8 lanes),
// is loaded once with 128-bit loads, reduced with shuffles only when G > 1, and needs ONE exp per
// element:
//     m = max x,  e_i = exp(x_i - m),  s = sum e_i,  t = sum e_i (x_i - m)
//     log p_i = x_i - (m + log s),  p_i = e_i / s,  H = -sum p log p = log s - t / s
// The backward recomputes the softmax from the logits instead of reading saved (T,B,N) buffers:
//     d/dx_k = c1*(1[k=a] - p_k) + c2*(-p_k*(log p_k + H))            (SURVEY.md A.3)
// HBM bytes per row: forward 4N (+8 action, +4 per per-row scalar), backward 4N in + 4N out.
#pragma once
#include "common.cuh"
#include "reduce.cuh"

namespace hpcrll {

// geometry of the row -> lane mapping, decided on the host
struct RowGeom {
    int G;      // lanes per row (power of two <= 32)
    int kmax;   // register chunks per lane, exact: 1..8 (0 = N too large for registers: looping kernel)
    int width;  // floats per chunk: 4 (N % 4 == 0, 16B-aligned bases), 2 (N even, 8B-aligned: Atari's 6 / 18), 1
};

// p0 / p1: the tensors the kernel reads or writes row-wise (p1 may be null)
inline RowGeom row_geom(int64_t N, const void* p0, const void* p1 = nullptr) {
    RowGeom g;
    const bool a16 = aligned16(p0) && (!p1 || aligned16(p1)), a8 = aligned8(p0) && (!p1 || aligned8(p1));
    g.width = (a16 && N % 4 == 0) ? 4 : ((a8 && N % 2 == 0) ? 2 : 1);
    const int64_t chunks = N / g.width;  // chunk = one load per lane
    // lanes per row: the smallest power of two that leaves <= 4 float4 (or <= 8 narrower) chunks per lane; the
    // chunk count per lane is EXACT (kernels are instantiated for 1..8), so N=6 is one lane x 3 float2, N=18 two
    // lanes x 5 float2, N=24 two lanes x 3 float4 -- the row kernels are issue-bound, idle register slots cost
    const int64_t cap = g.width == 4 ? 4 : 8;
    int G = 1;
    while (G < 32 && chunks > static_cast<int64_t>(G) * cap) G <<= 1;
    g.G = G;
    const int64_t per_lane = (chunks + G - 1) / G;
    g.kmax = per_lane <= 8 ? static_cast<int>(per_lane) : 0;
    return g;
}

#ifdef __CUDACC__

// stands in for -inf in masked register slots and clamps (x - m): finite, so 0 * it stays 0 -- the
// same guard torch.distributions.Categorical.entropy applies (clamp to finfo.min) for -inf logits
constexpr float kNegBig = -3.0e38f;

// e^d for the N-wide softmax terms (d = x - max <= 0, or a log-probability): FMUL + MUFU.EX2 instead of
// expf's 9 instructions -- the row kernels are issue-bound at small N.
// Error budget: ex2.approx is good to 2 ulp; rounding d*log2(e) adds a relative |d| * 6e-8, so a term e^d
// is off by at most |d| e^d * 6e-8 <= 2.2e-8 of the row's largest term -- far inside the 1e-5 parity bar
// (SURVEY.md 8c).  Per-row scalars (importance ratios) keep expf.  exp_term(-3e38) = 0 like expf.
__device__ __forceinline__ float exp_term(float d) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(d * 1.4426950408889634f));
    return r;
}

__device__ __forceinline__ float group_max(float v, int G) {
    for (int o = G >> 1; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float group_sum(float v, int G) {
    for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One row held across a group of G lanes.  Element index of x[j*W+q] is ((j*G + lig)*W + q).
template <int KMAX, int WIDTH>
struct RowRegs {
    static_assert(WIDTH == 1 || WIDTH == 2 || WIDTH == 4, "chunk width");
    static constexpr int W = WIDTH;
    static constexpr int NE = KMAX * W;
    float x[NE];

    __device__ __forceinline__ int index(int j, int q, int G, int lig) const { return (j * G + lig) * W + q; }

    // default-cached (L1-allocating) loads: with G < 8 a 128-byte line is shared by several chunk
    // indices j, so later j hit in L1 instead of re-fetching sectors from L2
    __device__ __forceinline__ void load(const float* __restrict__ row, int N, int G, int lig, bool active) {
#pragma unroll
        for (int j = 0; j < KMAX; ++j) {
            const int e0 = (j * G + lig) * W;
            if (W == 4) {
                float4 v = make_float4(kNegBig, kNegBig, kNegBig, kNegBig);
                if (active && e0 < N) v = __ldg(reinterpret_cast<const float4*>(row + e0));
                x[j * W + 0] = v.x;
                x[j * W + (W > 1 ? 1 : 0)] = v.y;
                x[j * W + (W > 2 ? 2 : 0)] = v.z;
                x[j * W + (W > 3 ? 3 : 0)] = v.w;
            } else if (W == 2) {
                float2 v = make_float2(kNegBig, kNegBig);
                if (active && e0 < N) v = __ldg(reinterpret_cast<const float2*>(row + e0));
                x[j * W + 0] = v.x;
                x[j * W + (W > 1 ? 1 : 0)] = v.y;
            } else {
                x[j] = (active && e0 < N) ? __ldg(row + e0) : kNegBig;
            }
        }
    }

    __device__ __forceinline__ float row_max(int G) const {
        float mm = x[0];
#pragma unroll
        for (int i = 1; i < NE; ++i) mm = fmaxf(mm, x[i]);
        return group_max(mm, G);
    }

    // one pass: s = sum exp(x-m), t = sum exp(x-m)*(x-m)  (group-wide); optionally keeps e_i
    template <bool WANT_T, bool KEEP_E>
    __device__ __forceinline__ void stats(int G, float m, float& s, float& t, float (&e)[NE]) const {
        float ss = 0.f, tt = 0.f;
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            const float d = fmaxf(x[i] - m, kNegBig);
            const float ei = exp_term(d);  // masked slots: exp(-3e38) = 0
            ss += ei;
            if (WANT_T) tt = fmaf(ei, d, tt);
            if (KEEP_E) e[i] = ei;
        }
        s = group_sum(ss, G);
        t = WANT_T ? group_sum(tt, G) : 0.f;
    }

    // x[index == a] (0 if this lane does not hold it); sum over the group afterwards
    __device__ __forceinline__ float select(int a, int G, int lig) const {
        float sel = 0.f;
#pragma unroll
        for (int j = 0; j < KMAX; ++j)
#pragma unroll
            for (int q = 0; q < W; ++q)
                if (index(j, q, G, lig) == a) sel = x[j * W + q];
        return sel;
    }
};

// Per-row log-prob in the two normalisations origin uses:
//   CATEGORICAL: logp = x - (m + log s)          torch.distributions.Categorical (vtrace.py:74, ppo.py:54)
//   otherwise  : logp = (x - m) - log s          F.cross_entropy / log_softmax   (upgo.py:16)
template <bool CATEGORICAL>
__device__ __forceinline__ float row_logp(float x, float m, float logs) {
    return CATEGORICAL ? x - (m + logs) : (x - m) - logs;
}

// ---------------------------------------------------------------------------------------------------
// Staged rows: action counts that are not a multiple of 4 (Atari's 6 / 9 / 18 ...) cannot use 128-bit
// row chunks, and scalar per-lane chunks waste lanes and shuffles.  For N <= 32 such tensors are instead
// read as a FLAT contiguous stream: a CTA copies kStageRows consecutive rows (kStageRows*N floats, 128-bit
// coalesced, row boundaries ignored) into shared memory with an odd pitch, then every thread owns ONE row
// (bank-conflict-free column walk, no shuffles, all lanes busy).  Gradients go back the same way.
// ---------------------------------------------------------------------------------------------------
constexpr int kStageRows = 256;
inline int stage_pitch(int N) { return N | 1; }
// for N <= 8 the per-lane scalar chunks are as fast or faster; from N = 9 the staged path wins.  Rows that can be read in 64-bit or
// 128-bit chunks (`width` > 1) stay on the register path.
inline bool use_staged_rows(int64_t N, int width) { return N > 8 && N <= 32 && width == 1; }
inline size_t stage_bytes(int N, int tiles) { return static_cast<size_t>(tiles) * kStageRows * stage_pitch(N) * sizeof(float); }

// copy rows [row0, row0 + kStageRows) of a contiguous (R, N) tensor into tile[r * P + c]
__device__ __forceinline__ void stage_rows(const float* __restrict__ g, int64_t R, int N, int P, int64_t row0,
                                           float* __restrict__ tile, bool aligned) {
    const int64_t rows = min(static_cast<int64_t>(kStageRows), R - row0);
    const int cnt = static_cast<int>(rows) * N;  // <= 256 * 32
    const float* __restrict__ src = g + row0 * N;
    const float invN = 1.f / static_cast<float>(N);
    if (aligned) {  // (row0 * N) % 4 == 0 because row0 is a multiple of kStageRows
        for (int i = threadIdx.x * 4; i < cnt; i += kStageRows * 4) {
            const int r = __float2int_rd((static_cast<float>(i) + 0.5f) * invN);  // exact for i < 2^13, N <= 32
            int c = i - r * N;
            int idx = r * P + c;  // running shared-memory index: +1 per element, +(P-N) more at a row end
            if (i + 3 < cnt) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(src + i));
                const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    tile[idx++] = e[q];
                    if (++c == N) c = 0, idx += P - N;
                }
            } else {
                for (int q = 0; i + q < cnt; ++q) {
                    tile[idx++] = __ldg(src + i + q);
                    if (++c == N) c = 0, idx += P - N;
                }
            }
        }
    } else {
        for (int i = threadIdx.x; i < cnt; i += kStageRows) {
            const int r = __float2int_rd((static_cast<float>(i) + 0.5f) * invN);
            tile[r * P + (i - r * N)] = __ldg(src + i);
        }
    }
}

// inverse: write tile rows back to a contiguous (R, N) tensor
__device__ __forceinline__ void unstage_rows(float* __restrict__ g, int64_t R, int N, int P, int64_t row0,
                                             const float* __restrict__ tile, bool aligned) {
    const int64_t rows = min(static_cast<int64_t>(kStageRows), R - row0);
    const int cnt = static_cast<int>(rows) * N;
    float* __restrict__ dst = g + row0 * N;
    const float invN = 1.f / static_cast<float>(N);
    if (aligned) {
        for (int i = threadIdx.x * 4; i < cnt; i += kStageRows * 4) {
            const int r = __float2int_rd((static_cast<float>(i) + 0.5f) * invN);
            int c = i - r * N;
            int idx = r * P + c;
            float e[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (i + q < cnt) e[q] = tile[idx];
                ++idx;
                if (++c == N) c = 0, idx += P - N;
            }
            if (i + 3 < cnt) {
                st_stream4(reinterpret_cast<float4*>(dst + i), make_float4(e[0], e[1], e[2], e[3]));
            } else {
                for (int q = 0; i + q < cnt; ++q) dst[i + q] = e[q];
            }
        }
    } else {
        for (int i = threadIdx.x; i < cnt; i += kStageRows) {
            const int r = __float2int_rd((static_cast<float>(i) + 0.5f) * invN);
            dst[i] = tile[r * P + (i - r * N)];
        }
    }
}

// statistics of one row sitting in shared memory (one thread per row)
template <bool WANT_T>
__device__ __forceinline__ void staged_stats(const float* __restrict__ x, int N, float& m, float& s, float& t) {
    float mm = x[0];
    for (int k = 1; k < N; ++k) mm = fmaxf(mm, x[k]);
    float ss = 0.f, tt = 0.f;
    for (int k = 0; k < N; ++k) {
        const float d = fmaxf(x[k] - mm, kNegBig);
        const float e = exp_term(d);
        ss += e;
        if (WANT_T) tt = fmaf(e, d, tt);
    }
    m = mm;
    s = ss;
    t = tt;
}

// ---------------------------------------------------------------------------------------------------
// Forward row drivers.  V-trace, UPGO and PPO reduce each logits row to (max, log-sum, entropy, the chosen action's
// log-prob) and differ only in what they do with it.  One driver per row layout walks the rows of the logits tensors
// l0 and l1 (l1: null when the op has one); the op says what a row is made of and what is done with the result:
//   kTensors       logits tensors per row (1 or 2), of the same row length N
//   kEntropy       tensor 0 needs the entropy H (the moment t of the row statistics); H is 0 otherwise
//   kCat           the log-prob form of row_logp
//   Scalars scalars(r, ok, lig, args...)          the per-row scalars of row r, `.a` the action (-1 when !ok); lig:
//                                                 the lane's index in the row's group
//   emit(row, sc, H, lp0, lp1, args...)           run by one lane per row; lp0 / lp1: the action's log-prob in
//                                                 tensor 0 / 1
// args...: the kernel's remaining arguments, passed through as function arguments.  The op struct holds no pointers,
// only accumulators and per-call constants: a pointer read from a struct member, or values kept in an array, change
// the register kernels' machine code, so the drivers also name the two tensors' values (x0 / x1, m0 / m1, ...)
// instead of indexing arrays.
// ---------------------------------------------------------------------------------------------------

// Register layout: a row in the registers of a group of G lanes, grid-stride over blocks of (32 / G) * 8 rows.
// G1: one lane per row (G == 1, N == KMAX * WIDTH exactly) known at compile time -- the group loops, the `e0 < N`
// predicates and the element-index arithmetic of the row helpers fold away (the kernels are bound by instruction issue
// at small N).  The walk is a macro expanded in the kernel, not a function: behind any call boundary, even a
// force-inlined one, the 128-bit kernels compile to different machine code.  It expects the kernel's template
// parameters KMAX, WIDTH, G1 and its arguments R, N_, G_, log2G_ in scope.
#define HPC_ROWS_FWD_REGS(op, l0, l1, ...)                                                                        \
    do {                                                                                                          \
        using Op = decltype(op);                                                                                  \
        using Row = RowRegs<KMAX, WIDTH>;                                                                         \
        constexpr bool TWO = Op::kTensors == 2;                                                                   \
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;                                               \
        const int N = G1 ? KMAX * WIDTH : N_, G = G1 ? 1 : G_, log2G = G1 ? 0 : log2G_;                           \
        const int lig = G1 ? 0 : (lane & (G - 1)), gw = lane >> log2G;                                            \
        const int rows_per_warp = 32 >> log2G;                                                                    \
        const int rows_per_block = rows_per_warp * 8;                                                             \
        /* software pipeline (small rows only): the next row block's loads are issued before this one is reduced */ \
        constexpr bool PF = Row::NE <= 8;                                                                         \
        Row x0, x1, n0, n1;                                                                                       \
        typename Op::Scalars cur, nxt;                                                                            \
        /* row index and row pointers advance by increments (no 64-bit multiply per row) */                       \
        const int64_t stride = static_cast<int64_t>(gridDim.x) * rows_per_block;                                 \
        int64_t base = static_cast<int64_t>(blockIdx.x) * rows_per_block;                                         \
        int64_t row = base + warp * rows_per_warp + gw;                                                           \
        const float* p0 = (l0) + row * N;                                                                         \
        [[maybe_unused]] const float* p1 = TWO ? static_cast<const float*>(l1) + row * N : nullptr;               \
        const int64_t pstep = stride * N;                                                                         \
        x0.load(p0, N, G, lig, row < R);                                                                          \
        if constexpr (TWO) x1.load(p1, N, G, lig, row < R);                                                       \
        cur = op.scalars(row, row < R, lig, __VA_ARGS__);                                                         \
        for (; base < R; base += stride, row += stride) { /* block-uniform trip count */                          \
            const bool active = row < R;                                                                          \
            const int64_t nrow = row + stride;                                                                    \
            p0 += pstep;                                                                                          \
            if constexpr (TWO) p1 += pstep;                                                                       \
            if (PF) {                                                                                             \
                n0.load(p0, N, G, lig, nrow < R);                                                                 \
                if constexpr (TWO) n1.load(p1, N, G, lig, nrow < R);                                              \
            }                                                                                                     \
            if (PF) nxt = op.scalars(nrow, nrow < R, lig, __VA_ARGS__);                                        \
            const int a = cur.a;                                                                                  \
            [[maybe_unused]] float m1 = 0.f, s0, t0, s1, t1, none[Row::NE], ls0 = 0.f, ls1 = 0.f, lp1 = 0.f;      \
            const float m0 = x0.row_max(G);                                                                       \
            if constexpr (TWO) m1 = x1.row_max(G);                                                                \
            x0.template stats<Op::kEntropy, false>(G, m0, s0, t0, none);                                          \
            if constexpr (TWO) x1.template stats<false, false>(G, m1, s1, t1, none);                              \
            if constexpr (Op::kEntropy) ls0 = logf(s0);                                                           \
            if constexpr (TWO) ls1 = logf(s1);                                                                    \
            const float H = Op::kEntropy ? ls0 - t0 / s0 : 0.f;                                                   \
            /* exactly one lane of the group holds the action's logit */                                          \
            /* (log s after the selection when nothing else needs it: the order the UPGO kernels were tuned in) */ \
            const float lp0 = row_logp<Op::kCat>(group_sum(x0.select(a, G, lig), G), m0, Op::kEntropy ? ls0 : logf(s0)); \
            if constexpr (TWO) lp1 = row_logp<Op::kCat>(group_sum(x1.select(a, G, lig), G), m1, ls1);             \
            if (active && lig == 0) op.emit(row, cur, H, lp0, lp1, __VA_ARGS__);                                  \
            if (PF) {                                                                                             \
                x0 = n0;                                                                                          \
                if constexpr (TWO) x1 = n1;                                                                       \
            } else {                                                                                              \
                x0.load(p0, N, G, lig, nrow < R);                                                                 \
                if constexpr (TWO) x1.load(p1, N, G, lig, nrow < R);                                              \
            }                                                                                                     \
            if (PF) cur = nxt;                                                                                    \
            else cur = op.scalars(nrow, nrow < R, lig, __VA_ARGS__);                                              \
        }                                                                                                         \
    } while (0)

// Staged layout (N <= 32, not 128-bit eligible, see "Staged rows" above): kTensors tiles of kStageRows rows in dynamic
// shared memory, one thread per row.
template <class Op, class... A>
__device__ __forceinline__ void rows_fwd_staged(Op& op, int64_t R, int N, int P, int aligned, const float* l0,
                                                const float* l1, A... args) {
    constexpr bool TWO = Op::kTensors == 2;
    extern __shared__ float tiles[];
    float* tile0 = tiles;
    float* tile1 = tiles + kStageRows * P;
    const int64_t ntiles = (R + kStageRows - 1) / kStageRows;
    for (int64_t tix = blockIdx.x; tix < ntiles; tix += gridDim.x) {
        const int64_t row0 = tix * kStageRows, row = row0 + threadIdx.x;
        __syncthreads();  // every thread is done with the previous tiles
        stage_rows(l0, R, N, P, row0, tile0, aligned != 0);
        if constexpr (TWO) stage_rows(l1, R, N, P, row0, tile1, aligned != 0);
        __syncthreads();
        if (row < R) {
            const float* x0 = tile0 + threadIdx.x * P;
            const float* x1 = tile1 + threadIdx.x * P;
            float m0, s0, t0, m1 = 0.f, s1 = 0.f, t1, ls1 = 0.f, lp1 = 0.f;
            staged_stats<Op::kEntropy>(x0, N, m0, s0, t0);
            if constexpr (TWO) staged_stats<false>(x1, N, m1, s1, t1);
            const float ls0 = logf(s0);
            if constexpr (TWO) ls1 = logf(s1);
            const float H = Op::kEntropy ? ls0 - t0 / s0 : 0.f;
            const typename Op::Scalars sc = op.scalars(row, true, 0, args...);
            const float lp0 = row_logp<Op::kCat>(x0[sc.a], m0, ls0);
            if constexpr (TWO) lp1 = row_logp<Op::kCat>(x1[sc.a], m1, ls1);
            op.emit(row, sc, H, lp0, lp1, args...);
        }
    }
}

// Looping layout (N too large for registers): one warp per row, strided passes over the row.
template <class Op, class... A>
__device__ __forceinline__ void rows_fwd_loop(Op& op, int64_t R, int N, const float* l0, const float* l1, A... args) {
    constexpr bool TWO = Op::kTensors == 2;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + warp; row < R; row += static_cast<int64_t>(gridDim.x) * 8) {
        const float* x0 = l0 + row * N;
        const float* x1 = l1 + row * N;
        float m0 = -INFINITY, m1 = -INFINITY;
        for (int k = lane; k < N; k += 32) {
            m0 = fmaxf(m0, x0[k]);
            if constexpr (TWO) m1 = fmaxf(m1, x1[k]);
        }
        m0 = warp_max(m0);
        if constexpr (TWO) m1 = warp_max(m1);
        float s0 = 0.f, s1 = 0.f;
        for (int k = lane; k < N; k += 32) {
            s0 += exp_term(x0[k] - m0);
            if constexpr (TWO) s1 += exp_term(x1[k] - m1);
        }
        s0 = warp_sum(s0);
        if constexpr (TWO) s1 = warp_sum(s1);
        float ls1 = 0.f, lp1 = 0.f, H = 0.f;
        const float ls0 = logf(s0);
        if constexpr (TWO) ls1 = logf(s1);
        if constexpr (Op::kEntropy) {
            float h = 0.f;
            for (int k = lane; k < N; k += 32) {
                const float lp = fmaxf(row_logp<Op::kCat>(x0[k], m0, ls0), kNegBig);  // -inf logits: 0 * -3e38, not NaN
                h += exp_term(lp) * lp;
            }
            H = -warp_sum(h);
        }
        if (lane == 0) {
            const typename Op::Scalars sc = op.scalars(row, true, 0, args...);
            const float lp0 = row_logp<Op::kCat>(x0[sc.a], m0, ls0);
            if constexpr (TWO) lp1 = row_logp<Op::kCat>(x1[sc.a], m1, ls1);
            op.emit(row, sc, H, lp0, lp1, args...);
        }
    }
}

// one fp64 partial per CTA and term: partials[k * gridDim.x + blockIdx.x]
template <int K>
__device__ __forceinline__ void flush_partials(double (&acc)[K], double* __restrict__ partials) {
    __shared__ double red[K * 32];
    block_sum<K>(acc, red);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < K; ++k) partials[static_cast<size_t>(k) * gridDim.x + blockIdx.x] = acc[k];
    }
}

#endif  // __CUDACC__

// ---- shared backward: grad[r,k] = (g1*c1[r])*(1[k=a_r]-p_k) + (g2*w_r*inv_n)*(-p_k(logp_k+H)) ----------
// g1, g2: device scalars (upstream gradients); g2 == nullptr skips the entropy term; w == nullptr -> 1.
// Categorical log-probs (see row_logp).
int launch_softmax_grad_rows(const float* logits, const int64_t* action, const float* c1, const float* w,
                             const float* g1, const float* g2, double inv_n, float* grad, int64_t R, int64_t N,
                             cudaStream_t stream);

// *out = the library's device constants {+1, -1} on the current device: the fixed upstream scale g1 of a
// launch_softmax_grad_rows call.  The address is looked up once per device and cached, so a call made once eagerly
// leaves nothing to resolve while a stream is being captured.
int unit_scalars(const float** out);

// grid size for a row-streaming kernel: enough CTAs to fill the machine, grid-stride over row blocks
inline unsigned rows_grid(int64_t R, int rows_per_block) {
    int64_t blocks = (R + rows_per_block - 1) / rows_per_block;
    const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return static_cast<unsigned>(blocks);
}

// launch-time descriptor for finalize_terms: term k sums partials[off[k] .. off[k]+cnt[k]) * scale[k]
struct FinSpec {
    int off[5];
    int cnt[5];
    double scale[5];
};
int launch_finalize_terms(const double* partials, const FinSpec& spec, int nterms, float* out, cudaStream_t stream);

// The register layouts (WIDTH, G1, KMAX) row_geom and use_staged_rows can select, and the only ones built: with G == 1
// every KMAX up to the lane's chunk cap (4 float4, 8 narrower); G > 1 only when the row has more chunks than that cap,
// so more than half of it per lane; width 1 with 9 <= N <= 32 is staged.  tests/test_row_layouts_cpu.py checks this
// table against the built library and the dispatch mirror of tests/row_paths.py.
#define HPC_ROW_LAYOUTS(X)                                                                               \
    X(4, true, 1) X(4, true, 2) X(4, true, 3) X(4, true, 4)                                              \
    X(2, true, 1) X(2, true, 2) X(2, true, 3) X(2, true, 4) X(2, true, 5) X(2, true, 6) X(2, true, 7) X(2, true, 8) \
    X(1, true, 1) X(1, true, 2) X(1, true, 3) X(1, true, 4) X(1, true, 5) X(1, true, 6) X(1, true, 7) X(1, true, 8) \
    X(4, false, 3) X(4, false, 4) X(4, false, 5) X(4, false, 6) X(4, false, 7) X(4, false, 8)            \
    X(2, false, 5) X(2, false, 6) X(2, false, 7) X(2, false, 8)                                          \
    X(1, false, 5) X(1, false, 6) X(1, false, 7) X(1, false, 8)

constexpr int row_layout_key(int width, bool g1, int kmax) { return (width * 2 + (g1 ? 1 : 0)) * 16 + kmax; }

#ifdef __CUDACC__
// Launches the row kernel of one family that row_geom / use_staged_rows pick for rows of N floats.  p0, p1: the row
// tensors whose alignment decides the layout (p1 may be null).  Rows::reg<KMAX, WIDTH, G1>(), Rows::staged() and
// Rows::loop() return the family's kernels, which take args... followed by (R, N, G, log2G), (R, N, pitch, aligned)
// and (R, N); the staged kernel holds Rows::kStagedTiles tiles.  *grid: the CTA count (the caller's partial count).
template <class Rows, class... Args>
int launch_rows(unsigned* grid, int64_t R, int64_t N, const void* p0, const void* p1, cudaStream_t stream,
                Args... args) {
    const RowGeom ge = row_geom(N, p0, p1);
    const int n = static_cast<int>(N);
    if (use_staged_rows(N, ge.width)) {
        const int max_bytes = static_cast<int>(stage_bytes(32, Rows::kStagedTiles));  // largest pitch (N=32 -> 33)
        if (max_bytes > 48 * 1024) {
            static SmemOptIn opt;
            if (int rc = opt.ensure(Rows::staged(), max_bytes)) return rc;
        }
        *grid = rows_grid(R, kStageRows);
        Rows::staged()<<<*grid, kStageRows, stage_bytes(n, Rows::kStagedTiles), stream>>>(
            args..., R, n, stage_pitch(n), aligned16(p0) && (!p1 || aligned16(p1)) ? 1 : 0);
    } else if (ge.kmax == 0) {
        *grid = rows_grid(R, 8);
        Rows::loop()<<<*grid, 256, 0, stream>>>(args..., R, n);
    } else {
        int log2G = 0;
        while ((1 << log2G) < ge.G) ++log2G;
        *grid = rows_grid(R, (32 / ge.G) * 8);
        decltype(Rows::template reg<1, 1, true>()) kernel;
        switch (row_layout_key(ge.width, ge.G == 1, ge.kmax)) {
#define HPC_ROW_CASE(W, G1, K) \
    case row_layout_key(W, G1, K): kernel = Rows::template reg<K, W, G1>(); break;
            HPC_ROW_LAYOUTS(HPC_ROW_CASE)
#undef HPC_ROW_CASE
            default:
                return set_error(HPC_RLL_ENOSUP, "row kernels: no register layout for width %d, G %d, kmax %d", ge.width,
                                 ge.G, ge.kmax);
        }
        kernel<<<*grid, 256, 0, stream>>>(args..., R, n, ge.G, log2G);
    }
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}
#endif  // __CUDACC__

}  // namespace hpcrll
