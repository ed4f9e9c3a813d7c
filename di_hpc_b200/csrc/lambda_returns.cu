// lambda_returns.cu -- λ-returns with per-step γ/λ and `done` masks, forward and adjoint, for sm_90a.
//
// Semantics: DI-engine's `generalized_lambda_returns` / `multistep_forward_view` over a (T,B) segment.  V_t is the
// bootstrap value of step t (bootstrap_values[t+1] of a (T+1,B) tensor, or bootstrap_values[t] of a (T,B) one).
// With d_t = γ_t·λ_t, e_t = γ_t − d_t and m_t = 0 where done_t is set, 1 elsewhere:
//     done absent:  R_{T-1} = r + γ·V              R_t = (r_t + d_t·R_{t+1}) + e_t·V_t
//     done given:   R_{T-1} = r + (m·γ)·V          R_t = r_t + m_t·(d_t·R_{t+1} + e_t·V_t)
// Adjoint (G = dL/dR), a forward-in-time scan from u_0 = G_0:
//     done absent:  u_t = G_t + u_{t-1}·d_{t-1}            grad_V_t = u_t·e_t,  grad_V_{T-1} = u_{T-1}·γ_{T-1}
//     done given:   u_t = G_t + (u_{t-1}·m_{t-1})·d_{t-1}  grad_V_t = (u_t·m_t)·e_t,  grad_V_{T-1} = u_{T-1}·(m·γ)
//     grad_rewards = u
// γ and λ are each a (T,B) fp32 tensor or a scalar; a scalar is fp32(γ), and with both scalar d and e are formed once
// on the host.  Every operation is one round-to-nearest fp32 op in the order above (explicit __f*_rn, no FMA
// contraction), so the wide and generic kernels are bit-identical to eager PyTorch of the formula on the CPU.  Masks
// enter as products with m, so a non-finite V or carry propagates as it does there.
//
// Regimes (hpc_rll_debug_set_config(HPC_RLL_OP_LAMBDA_RETURNS, id) / HPC_RLL_CFG_LAMBDA_RETURNS force one):
//   33 wide   ScanPipe (scan_pipe.cuh), templated on <GT, LT, DONE> so that every operand combination streams only the
//             bytes it needs: fp32 boxes of V, r (G backward) and the γ/λ tensors, a byte box of `done`; outputs
//             TMA-stored (backward: grad_rewards and grad_V in one pass).  Needs 16-byte aligned pointers and
//             B % 4 == 0, and B % 16 == 0 with `done` (a uint8 tensor map needs a 16-byte row stride).
//   21 look-back  single-launch T-split (scan_lookback.cuh) with the per-element coefficient m_t·d_t (CONSTA = false),
//             automatic for B <= 2048 and T >= 512.  V, r / G are staged; γ, λ and the mask are read per step.
//   99 generic the wide bodies driven by scan_column (scan_pipe.cuh), one column per thread, 64-bit indexing: ragged B,
//             misaligned pointers, short T.
// HBM traffic = algorithmic, each direction: 12 B per element with scalar γ/λ and no mask, up to 21 B with both tensors
// and a mask.  No atomics except the look-back tickets and counters.
#include <cstdint>
#include <initializer_list>

#include "scan_lookback.cuh"
#include "scan_pipe.cuh"

namespace hpcrll {

// the scalar forms of γ and λ, and d = γ·λ, e = γ − d formed from them in fp32
struct LrScal {
    float g, l, d, e;
};

namespace {

// m_t as a factor: 0 when the byte is set, 1 otherwise
__device__ __forceinline__ float keep(unsigned m) { return m != 0u ? 0.f : 1.f; }

struct Disc {
    float g, d, e;
};

// γ_t, d_t, e_t of one step from the tensor values xg / xl (ignored where the operand is a scalar)
template <bool GT, bool LT>
__device__ __forceinline__ Disc disc(float xg, float xl, const LrScal& s) {
    if constexpr (!GT && !LT) {
        return Disc{s.g, s.d, s.e};
    } else {
        const float g = GT ? xg : s.g, l = LT ? xl : s.l;
        const float d = __fmul_rn(g, l);
        return Disc{g, d, __fsub_rn(g, d)};
    }
}

// one forward step: `carry` = R_{t+1} on entry (ignored on the last row), R_t on exit.  Returns the coefficient of
// R_{t+1} in R_t, which the look-back folds.
template <bool DN>
__device__ __forceinline__ float fwd_step(float v, float r, const Disc& c, unsigned done, bool last, float& carry) {
    if constexpr (DN) {
        const float k = keep(done);
        carry = last ? __fadd_rn(r, __fmul_rn(__fmul_rn(k, c.g), v))
                     : __fadd_rn(r, __fmul_rn(k, __fadd_rn(__fmul_rn(c.d, carry), __fmul_rn(c.e, v))));
        return last ? 0.f : __fmul_rn(k, c.d);
    } else {
        carry = last ? __fadd_rn(r, __fmul_rn(c.g, v))
                     : __fadd_rn(__fadd_rn(r, __fmul_rn(c.d, carry)), __fmul_rn(c.e, v));
        return last ? 0.f : c.d;
    }
}

// one backward step: `carry` = (u_{t-1}·m_{t-1})·d_{t-1} on entry (-0 before row 0), the same of row t on exit.
// Returns u_t; `gv` = grad_V_t, `coef` = the coefficient of the entry carry in the exit carry.
template <bool DN>
__device__ __forceinline__ float bwd_step(float G, const Disc& c, unsigned done, bool last, float& carry, float& gv,
                                          float& coef) {
    const float u = __fadd_rn(G, carry);
    if constexpr (DN) {
        const float k = keep(done);
        const float um = __fmul_rn(u, k);
        gv = last ? __fmul_rn(u, __fmul_rn(k, c.g)) : __fmul_rn(um, c.e);
        carry = __fmul_rn(um, c.d);
        coef = __fmul_rn(k, c.d);
    } else {
        gv = last ? __fmul_rn(u, c.g) : __fmul_rn(u, c.e);
        carry = __fmul_rn(u, c.d);
        coef = c.d;
    }
    return u;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// wide-path bodies (ScanPipe), also driven by scan_column on the generic path.
// forward inputs x = {V, r, [γ], [λ]}, byte input {done}; output {R}
// backward inputs x = {G, [γ], [λ]}, byte input {done}; outputs {grad_V, grad_r}
// ------------------------------------------------------------------------------------------------
template <bool GT, bool LT, bool DN>
struct LrFwdBody {
    static constexpr int NF = 2 + GT + LT;
    float carry;
    LrScal s;
    int last;
    __device__ __forceinline__ void step(int t, const float (&x)[NF], const float (&)[1], const unsigned (&m)[1],
                                         float (&o)[1]) {
        const Disc c = disc<GT, LT>(x[GT ? 2 : 0], x[LT ? 2 + GT : 0], s);
        fwd_step<DN>(x[0], x[1], c, m[0], t == last, carry);
        o[0] = carry;
    }
};

template <bool GT, bool LT, bool DN>
struct LrBwdBody {
    static constexpr int NF = 1 + GT + LT;
    float carry;
    LrScal s;
    int last;
    __device__ __forceinline__ void step(int t, const float (&x)[NF], const float (&)[1], const unsigned (&m)[1],
                                         float (&o)[2]) {
        const Disc c = disc<GT, LT>(x[GT ? 1 : 0], x[LT ? 1 + GT : 0], s);
        float coef;
        o[1] = bwd_step<DN>(x[0], c, m[0], t == last, carry, o[0], coef);
    }
};

template <bool GT, bool LT, bool DN, int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) lambda_ret_fwd_tma(const __grid_constant__ TmapPack<2 + GT + LT + DN> maps,
                                                               const __grid_constant__ TmapPack<1> omaps, int T,
                                                               LrScal s) {
    using Pipe = ScanPipe<2 + GT + LT, DN, 1, BT, TT, ST, 0>;
    LrFwdBody<GT, LT, DN> body{-0.f, s, T - 1};
    Pipe::template run<true>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
}

template <bool GT, bool LT, bool DN, int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) lambda_ret_bwd_tma(const __grid_constant__ TmapPack<1 + GT + LT + DN> maps,
                                                               const __grid_constant__ TmapPack<2> omaps, int T,
                                                               LrScal s) {
    using Pipe = ScanPipe<1 + GT + LT, DN, 2, BT, TT, ST, 0>;
    LrBwdBody<GT, LT, DN> body{-0.f, s, T - 1};
    Pipe::template run<false>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
}

// ------------------------------------------------------------------------------------------------
// generic path: the same bodies driven by scan_column, one column per thread
// ------------------------------------------------------------------------------------------------
template <bool GT, bool LT, bool DN>
__global__ void __launch_bounds__(128) lambda_ret_fwd_generic(const float* __restrict__ v, const float* __restrict__ r,
                                                               const float* __restrict__ g,
                                                               const float* __restrict__ l,
                                                               const uint8_t* __restrict__ done,
                                                               float* __restrict__ ret, int64_t T, int64_t B,
                                                               LrScal s) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    constexpr int NF = LrFwdBody<GT, LT, DN>::NF;
    ColOp<const float*> in[NF];
    in[0] = {v, B};
    in[1] = {r, B};
    if constexpr (GT) in[2] = {g, B};
    if constexpr (LT) in[2 + GT] = {l, B};
    LrFwdBody<GT, LT, DN> body{-0.f, s, static_cast<int>(T - 1)};
    scan_column<NF, DN ? 1 : 0, 1, 0, true>(in, {{done, B}}, nullptr, {{ret, B}}, T, col, body);
}

template <bool GT, bool LT, bool DN>
__global__ void __launch_bounds__(128) lambda_ret_bwd_generic(const float* __restrict__ grad_ret,
                                                               const float* __restrict__ g,
                                                               const float* __restrict__ l,
                                                               const uint8_t* __restrict__ done,
                                                               float* __restrict__ gv, float* __restrict__ gr,
                                                               int64_t T, int64_t B, LrScal s) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    constexpr int NF = LrBwdBody<GT, LT, DN>::NF;
    ColOp<const float*> in[NF];
    in[0] = {grad_ret, B};
    if constexpr (GT) in[1] = {g, B};
    if constexpr (LT) in[1 + GT] = {l, B};
    LrBwdBody<GT, LT, DN> body{-0.f, s, static_cast<int>(T - 1)};
    scan_column<NF, DN ? 1 : 0, 2, 0, false>(in, {{done, B}}, nullptr, {{gv, B}, {gr, B}}, T, col, body);
}

// ------------------------------------------------------------------------------------------------
// small-batch path: single-launch T-split with look-back (scan_lookback.cuh).  V and r (G backward) are staged in
// shared memory by lb_segment; γ, λ and the mask byte of a step are read by the Fac from global memory (their loads do
// not depend on the carry, so they issue ahead of the chain like the staged ones).  A NULL γ / λ is the scalar, a NULL
// mask selects the done-absent formula.
// ------------------------------------------------------------------------------------------------
struct LrLbBody {
    float carry, coef;
    bool store;
};

struct LrLbOps {
    const float* g;
    const float* l;
    const uint8_t* done;
    int64_t B;
    int col;
    bool valid;
    int last;
    LrScal s;
    __device__ __forceinline__ Disc disc_at(int64_t i) const {
        if (g == nullptr && l == nullptr) return Disc{s.g, s.d, s.e};
        const float gg = g != nullptr && valid ? __ldg(g + i) : s.g;
        const float ll = l != nullptr && valid ? __ldg(l + i) : s.l;
        const float d = __fmul_rn(gg, ll);
        return Disc{gg, d, __fsub_rn(gg, d)};
    }
};

struct LrFwdLbFac {
    LrLbOps op;
    float* ret;
    using Body = LrLbBody;
    __device__ __forceinline__ Body make(int pass, int, float carry) const {
        return Body{carry, 1.f, op.valid && pass == 1};
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[2]) const {
        const int64_t i = static_cast<int64_t>(t) * op.B + op.col;
        const Disc c = op.disc_at(i);
        const bool last = t == op.last;
        if (op.done != nullptr)
            b.coef = fwd_step<true>(x[0], x[1], c, op.valid ? ld_mask(op.done, i) : 0u, last, b.carry);
        else
            b.coef = fwd_step<false>(x[0], x[1], c, 0u, last, b.carry);
        if (b.store) st_stream(ret + i, b.carry);
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.carry; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.coef; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) lambda_ret_fwd_lookback(const float* __restrict__ v,
                                                                    const float* __restrict__ r,
                                                                    const float* __restrict__ g,
                                                                    const float* __restrict__ l,
                                                                    const uint8_t* __restrict__ done,
                                                                    float* __restrict__ ret, int T, int B, LrScal s,
                                                                    int S, int L, int tiles, LbCtl* ctl,
                                                                    unsigned long long* words) {
    __shared__ float smem[2 * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;  // backward in time: the last segment goes first
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const LrFwdLbFac fac{{g, l, done, B, col, col < B, T - 1, s}, ret};
    const float* const in[2] = {v, r};
    const int64_t ld[2] = {B, B};
    lb_segment<2, true, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

struct LrBwdLbFac {
    LrLbOps op;
    float *gv, *gr;
    using Body = LrLbBody;
    __device__ __forceinline__ Body make(int pass, int, float carry) const {
        return Body{carry, 1.f, op.valid && pass == 1};
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[1]) const {
        const int64_t i = static_cast<int64_t>(t) * op.B + op.col;
        const Disc c = op.disc_at(i);
        const bool last = t == op.last;
        float gvt, u;
        if (op.done != nullptr)
            u = bwd_step<true>(x[0], c, op.valid ? ld_mask(op.done, i) : 0u, last, b.carry, gvt, b.coef);
        else
            u = bwd_step<false>(x[0], c, 0u, last, b.carry, gvt, b.coef);
        if (b.store) {
            st_stream(gv + i, gvt);
            st_stream(gr + i, u);
        }
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.carry; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.coef; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) lambda_ret_bwd_lookback(const float* __restrict__ grad_ret,
                                                                    const float* __restrict__ g,
                                                                    const float* __restrict__ l,
                                                                    const uint8_t* __restrict__ done,
                                                                    float* __restrict__ gv, float* __restrict__ gr,
                                                                    int T, int B, LrScal s, int S, int L, int tiles,
                                                                    LbCtl* ctl, unsigned long long* words) {
    __shared__ float smem[kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int t0 = lt.k * L, t1 = min(T, t0 + L);  // forward in time
    const int col = lt.tile * kLbCols + threadIdx.x;
    const LrBwdLbFac fac{{g, l, done, B, col, col < B, T - 1, s}, gv, gr};
    const float* const in[1] = {grad_ret};
    const int64_t ld[1] = {B};
    lb_segment<1, false, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

// ------------------------------------------------------------------------------------------------
// launchers and dispatch
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int kCfgWide = 33, kCfgLookback = 21, kCfgGeneric = 99;

// the wide path's tile: <BT, TT, ST> = columns per CTA, rows per box, ring stages (sweep in DESIGN.md §4.14)
constexpr int kFwdBT = 256, kFwdTT = 4, kFwdST = 5;
constexpr int kBwdBT = 256, kBwdTT = 4, kBwdST = 6;

// one (T,B) problem: the fp32 operands in the order the kernels read them, NULL for a scalar γ / λ or an absent mask
struct Problem {
    const float* g;
    const float* l;
    const uint8_t* done;
    int64_t T, B;
    LrScal s;
};

// every operand TMA-describable: fp32 (T,B) needs B % 4 == 0, a uint8 (T,B) map B % 16 == 0
bool wide_ok(std::initializer_list<const void*> f32, const Problem& p) {
    for (const void* q : f32)
        if (q != nullptr && !tma_ok_2d(q, p.B, p.B)) return false;
    return p.done == nullptr || (p.B % 16 == 0 && aligned16(p.done));
}

int pick(int64_t T, int64_t B, LbGeom* lg) {
    if (lookback_geometry(HPC_RLL_OP_LAMBDA_RETURNS, T, B, lg)) return kCfgLookback;
    const int forced = tuning_config(HPC_RLL_OP_LAMBDA_RETURNS);
    return forced == kCfgGeneric ? kCfgGeneric : kCfgWide;  // 21 on a shape that does not split: automatic
}

// calls L::run<GT, LT, DN>() for the operand combination of `p`
template <class L>
int dispatch(const L& launch, const Problem& p) {
    switch ((p.g ? 4 : 0) | (p.l ? 2 : 0) | (p.done ? 1 : 0)) {
        case 0: return launch.template run<false, false, false>();
        case 1: return launch.template run<false, false, true>();
        case 2: return launch.template run<false, true, false>();
        case 3: return launch.template run<false, true, true>();
        case 4: return launch.template run<true, false, false>();
        case 5: return launch.template run<true, false, true>();
        case 6: return launch.template run<true, true, false>();
        default: return launch.template run<true, true, true>();
    }
}

// fp32 tensor maps for the inputs `first..` followed by the γ / λ tensors that are present, then the mask
template <int N>
int input_maps(TmapPack<N>* maps, std::initializer_list<const float*> first, const Problem& p, int TT, int BT) {
    int k = 0;
    for (const float* q : first)
        if (int rc = make_tmap_2d(&maps->m[k++], q, p.T, p.B, p.B, TT, BT)) return rc;
    for (const float* q : {p.g, p.l})
        if (q != nullptr)
            if (int rc = make_tmap_2d(&maps->m[k++], q, p.T, p.B, p.B, TT, BT)) return rc;
    if (p.done != nullptr)
        if (int rc = make_tmap_2d_u8(&maps->m[k++], p.done, p.T, p.B, p.B, TT, BT)) return rc;
    return HPC_RLL_OK;
}

struct FwdWide {
    const Problem& p;
    const float *v, *r;
    float* ret;
    cudaStream_t stream;
    template <bool GT, bool LT, bool DN>
    int run() const {
        constexpr int BT = kFwdBT, TT = kFwdTT;
        TmapPack<2 + GT + LT + DN> maps;
        TmapPack<1> omaps;
        if (int rc = input_maps(&maps, {v, r}, p, TT, BT)) return rc;
        if (int rc = make_tmap_2d(&omaps.m[0], ret, p.T, p.B, p.B, TT, BT)) return rc;
        const unsigned grid = static_cast<unsigned>((p.B + BT - 1) / BT);
        return launch_scan<ScanPipe<2 + GT + LT, DN, 1, BT, TT, kFwdST, 0>,
                           lambda_ret_fwd_tma<GT, LT, DN, BT, TT, kFwdST>>(grid, stream, maps, omaps,
                                                                           static_cast<int>(p.T), p.s);
    }
};

struct BwdWide {
    const Problem& p;
    const float* grad_ret;
    float *gv, *gr;
    cudaStream_t stream;
    template <bool GT, bool LT, bool DN>
    int run() const {
        constexpr int BT = kBwdBT, TT = kBwdTT;
        TmapPack<1 + GT + LT + DN> maps;
        TmapPack<2> omaps;
        if (int rc = input_maps(&maps, {grad_ret}, p, TT, BT)) return rc;
        if (int rc = make_tmap_2d(&omaps.m[0], gv, p.T, p.B, p.B, TT, BT)) return rc;
        if (int rc = make_tmap_2d(&omaps.m[1], gr, p.T, p.B, p.B, TT, BT)) return rc;
        const unsigned grid = static_cast<unsigned>((p.B + BT - 1) / BT);
        return launch_scan<ScanPipe<1 + GT + LT, DN, 2, BT, TT, kBwdST, 0>,
                           lambda_ret_bwd_tma<GT, LT, DN, BT, TT, kBwdST>>(grid, stream, maps, omaps,
                                                                           static_cast<int>(p.T), p.s);
    }
};

struct FwdGeneric {
    const Problem& p;
    const float *v, *r;
    float* ret;
    cudaStream_t stream;
    template <bool GT, bool LT, bool DN>
    int run() const {
        lambda_ret_fwd_generic<GT, LT, DN><<<static_cast<unsigned>((p.B + 127) / 128), 128, 0, stream>>>(
            v, r, p.g, p.l, p.done, ret, p.T, p.B, p.s);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
};

struct BwdGeneric {
    const Problem& p;
    const float* grad_ret;
    float *gv, *gr;
    cudaStream_t stream;
    template <bool GT, bool LT, bool DN>
    int run() const {
        lambda_ret_bwd_generic<GT, LT, DN><<<static_cast<unsigned>((p.B + 127) / 128), 128, 0, stream>>>(
            grad_ret, p.g, p.l, p.done, gv, gr, p.T, p.B, p.s);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
};

int check_args(const char* what, int64_t T, int64_t B, int64_t offset) {
    HPC_REQUIRE(T >= 0 && B >= 0, "%s: negative size T=%lld B=%lld", what, (long long)T, (long long)B);
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512, "%s: T/B exceed 2^31", what);
    HPC_REQUIRE(offset == 0 || offset == 1, "%s: bootstrap_offset must be 0 or 1, got %lld", what, (long long)offset);
    return HPC_RLL_OK;
}

Problem make_problem(const float* g, const float* l, const uint8_t* done, int64_t T, int64_t B, double gamma,
                     double lambda) {
    LrScal s;
    s.g = static_cast<float>(gamma);
    s.l = static_cast<float>(lambda);
    s.d = s.g * s.l;  // fp32 products, as γ·ones_like(r) * λ·ones_like(r) would round them
    s.e = s.g - s.d;
    return Problem{g, l, done, T, B, s};
}

}  // namespace

static int lambda_returns_forward_impl(const float* bootstrap, const float* rewards, const float* gammas,
                                       const float* lambdas, const uint8_t* done, float* ret, int64_t T, int64_t B,
                                       int64_t offset, double gamma, double lambda, cudaStream_t stream) {
    if (int rc = check_args("lambda_returns_forward", T, B, offset)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(bootstrap && rewards && ret,
                "lambda_returns_forward: null bootstrap_values, rewards or returns pointer");
    const Problem p = make_problem(gammas, lambdas, done, T, B, gamma, lambda);
    const float* v = bootstrap + offset * B;
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        lambda_ret_fwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            v, rewards, gammas, lambdas, done, ret, static_cast<int>(T), static_cast<int>(B), p.s, lg.S, lg.L,
            lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
    if (cfg == kCfgWide && wide_ok({v, rewards, gammas, lambdas, ret}, p))
        return dispatch(FwdWide{p, v, rewards, ret, stream}, p);
    return dispatch(FwdGeneric{p, v, rewards, ret, stream}, p);
}

static int lambda_returns_backward_impl(const float* grad_ret, const float* gammas, const float* lambdas,
                                        const uint8_t* done, float* grad_bootstrap, float* grad_rewards, int64_t T,
                                        int64_t B, int64_t offset, double gamma, double lambda, cudaStream_t stream) {
    if (int rc = check_args("lambda_returns_backward", T, B, offset)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(grad_ret && grad_bootstrap && grad_rewards,
                "lambda_returns_backward: null grad_returns, grad_bootstrap_values or grad_rewards pointer");
    const Problem p = make_problem(gammas, lambdas, done, T, B, gamma, lambda);
    // the row of bootstrap_values no return reads gets a zero gradient
    if (offset > 0)
        HPC_CUDA(cudaMemsetAsync(grad_bootstrap, 0, static_cast<size_t>(offset * B) * sizeof(float), stream));
    float* gv = grad_bootstrap + offset * B;
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        lambda_ret_bwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            grad_ret, gammas, lambdas, done, gv, grad_rewards, static_cast<int>(T), static_cast<int>(B), p.s, lg.S,
            lg.L, lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
    if (cfg == kCfgWide && wide_ok({grad_ret, gammas, lambdas, gv, grad_rewards}, p))
        return dispatch(BwdWide{p, grad_ret, gv, grad_rewards, stream}, p);
    return dispatch(BwdGeneric{p, grad_ret, gv, grad_rewards, stream}, p);
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_lambda_returns_forward(const float* bootstrap_values, const float* rewards, const float* gammas,
                                   const float* lambdas, const uint8_t* done_u8, float* returns, int64_t T, int64_t B,
                                   int64_t bootstrap_offset, double gamma, double lambda, void* stream) {
    HPC_NVTX("lambda_returns_forward");
    return hpcrll::lambda_returns_forward_impl(bootstrap_values, rewards, gammas, lambdas, done_u8, returns, T, B,
                                               bootstrap_offset, gamma, lambda, hpcrll::as_stream(stream));
}

int hpc_rll_lambda_returns_backward(const float* grad_returns, const float* gammas, const float* lambdas,
                                    const uint8_t* done_u8, float* grad_bootstrap_values, float* grad_rewards,
                                    int64_t T, int64_t B, int64_t bootstrap_offset, double gamma, double lambda,
                                    void* stream) {
    HPC_NVTX("lambda_returns_backward");
    return hpcrll::lambda_returns_backward_impl(grad_returns, gammas, lambdas, done_u8, grad_bootstrap_values,
                                                grad_rewards, T, B, bootstrap_offset, gamma, lambda,
                                                hpcrll::as_stream(stream));
}

}  // extern "C"
