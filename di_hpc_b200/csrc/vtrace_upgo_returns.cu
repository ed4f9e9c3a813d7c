// vtrace_upgo_returns.cu -- the V-trace target (`vtrace_nstep_return`) and the UPGO return (`upgo_returns`) as
// standalone ops, forward and adjoint, for sm_90a.
//
// Semantics: hpc_rll/origin/vtrace.py:5-13 and hpc_rll/origin/upgo.py:21-38.  T = reward rows, V_t =
// bootstrap_values[t] for t = 0..T ((T+1,B)), G = dL/dR.  Every operation is one round-to-nearest fp32 op in the order
// written (explicit __f*_rn, no FMA contraction), which is origin's order:
//   V-trace, g = fp32(γ), f = fp32(γ·λ) (the product taken in double):
//     a_t = (r_t + g·V_{t+1}) − V_t    item_T = +0    item_t = ρ_t·a_t + (f·c_t)·item_{t+1}    R_t = V_t + item_t
//     adjoint, forward in time:  w_0 = G_0,  w_t = G_t + (f·c_{t−1})·w_{t−1},  p_t = w_t·ρ_t
//     grad_reward = p,  grad_V_t = (G_t − p_t) + g·p_{t−1}  (grad_V_0 = G_0 − p_0),  grad_V_T = g·p_{T−1}
//   UPGO, ℓ_t = [r_{t+1} + V_{t+2} >= V_{t+1}] for t < T−1 (a NaN compares false), ℓ_{T−1} := 0:
//     R_{T−1} = r_{T−1} + V_T          R_t = (r_t + ℓ_t·R_{t+1}) + (1 − ℓ_t)·V_{t+1}
//     adjoint:  u_0 = G_0,  u_t = G_t + ℓ_{t−1}·u_{t−1};  grad_r = u,  grad_V_{t+1} = u_t·(1 − ℓ_t),  grad_V_0 = +0
//   The forward can save ℓ as a (T,B) byte mask (1 = set, row T−1 = 0); the backward streams G and that mask only.
//
// The bodies here are new rather than VtraceBody / UpgoBody (vtrace.cu, upgo.cu): those carry the loss terms, and
// giving them a returns-only mode would change their kernels' machine code.
//
// Regimes (hpc_rll_debug_set_config(HPC_RLL_OP_LAMBDA_RETURNS, id) / HPC_RLL_CFG_LAMBDA_RETURNS force one; both ops
// are members of the λ-return family and share its switch):
//   33 wide   ScanPipe (scan_pipe.cuh), outputs TMA-stored.  V-trace forward streams V, r, ρ, c and stores R;
//             backward streams G, ρ, c and stores grad_V, grad_r (row T of grad_V by a plain store).  UPGO forward
//             streams V, r and stores R (the ℓ bytes by plain stores); backward streams G and the ℓ box and stores
//             grad_V (rows 1..T: its tensor map starts one row in) and grad_r.  Needs 16-byte aligned pointers and
//             B % 4 == 0, and B % 16 == 0 for the ℓ box.
//   21 look-back  single-launch T-split (scan_lookback.cuh) with the per-element coefficient f·c_t (V-trace) or ℓ_t
//             (UPGO) (CONSTA = false), automatic for B <= 2048 and T >= 512.
//   99 generic the wide bodies driven by scan_column, one column per thread, 64-bit indexing.
// HBM traffic, bytes per element: V-trace 20 forward, 20 backward; UPGO 12 forward (13 with ℓ saved), 13 backward.
// No atomics except the look-back tickets and counters.
#include <cstdint>
#include <initializer_list>

#include "scan_lookback.cuh"
#include "scan_pipe.cuh"

namespace hpcrll {

// V-trace scalars: g = fp32(γ), f = fp32(γ·λ)
struct VrScal {
    float g, f;
};

namespace {

// one V-trace forward step at row t: `item` = item_{t+1} on entry, item_t on exit; `v1` = V_{t+1} on entry, V_t on
// exit.  Returns f·c_t, the coefficient of item_{t+1} in item_t.
__device__ __forceinline__ float vr_fwd_step(float v, float r, float rho, float c, const VrScal& s, float& item,
                                             float& v1) {
    const float a = __fsub_rn(__fadd_rn(r, __fmul_rn(s.g, v1)), v);
    const float fc = __fmul_rn(s.f, c);
    item = __fadd_rn(__fmul_rn(rho, a), __fmul_rn(fc, item));
    v1 = v;
    return fc;
}

// the V-trace adjoint's state after row t−1: w_{t−1}, f·c_{t−1} and g·p_{t−1}.  Before row 0 it is {−0, 0, −0}, so
// that w_0 = G_0 + 0·(−0) = G_0 and grad_V_0 = (G_0 − p_0) + (−0) = G_0 − p_0 exactly.
struct VrAdj {
    float w, fc, gp;
};

// one V-trace backward step at row t: writes grad_V_t and grad_r_t, returns f·c_{t−1}, the coefficient of w_{t−1} in w_t
__device__ __forceinline__ float vr_bwd_step(float G, float rho, float c, const VrScal& s, VrAdj& a, float& gv,
                                             float& gr) {
    const float coef = a.fc;
    a.w = __fadd_rn(G, __fmul_rn(coef, a.w));
    const float p = __fmul_rn(a.w, rho);
    gv = __fadd_rn(__fsub_rn(G, p), a.gp);
    gr = p;
    a.gp = __fmul_rn(s.g, p);
    a.fc = __fmul_rn(s.f, c);
    return coef;
}

// the UPGO forward's history at row t: V_{t+1}, V_{t+2}, r_{t+1}
struct UrHist {
    float v1, v2, r1;
};

// one UPGO forward step at row t: `ret` = R_{t+1} on entry (ignored on the last row), R_t on exit.  Returns ℓ_t
// (0 on the last row), the coefficient of R_{t+1} in R_t.
__device__ __forceinline__ float ur_fwd_step(float v, float r, bool last, UrHist& h, float& ret) {
    float l = 0.f;
    if (last) {
        ret = __fadd_rn(r, h.v1);
    } else {
        l = __fadd_rn(h.r1, h.v2) >= h.v1 ? 1.f : 0.f;
        ret = __fadd_rn(__fadd_rn(r, __fmul_rn(l, ret)), __fmul_rn(__fsub_rn(1.f, l), h.v1));
    }
    h.v2 = h.v1;
    h.v1 = v;
    h.r1 = r;
    return l;
}

// one UPGO backward step at row t: `carry` = ℓ_{t−1}·u_{t−1} on entry (−0 before row 0), ℓ_t·u_t on exit.  Returns
// u_t = grad_r_t; `gv` = grad_V_{t+1}.
__device__ __forceinline__ float ur_bwd_step(float G, unsigned m, float& carry, float& gv) {
    const float l = m != 0u ? 1.f : 0.f;
    const float u = __fadd_rn(G, carry);
    gv = __fmul_rn(u, __fsub_rn(1.f, l));
    carry = __fmul_rn(l, u);
    return u;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// wide-path bodies (ScanPipe), also driven by scan_column on the generic path
// ------------------------------------------------------------------------------------------------
// inputs {V, r, ρ, c}, output {R}
struct VrFwdBody {
    float item, v1;
    VrScal s;
    __device__ __forceinline__ void step(int, const float (&x)[4], const float (&)[1], const unsigned (&)[1],
                                         float (&o)[1]) {
        vr_fwd_step(x[0], x[1], x[2], x[3], s, item, v1);
        o[0] = __fadd_rn(x[0], item);
    }
};

// inputs {G, ρ, c}, outputs {grad_V, grad_r}
struct VrBwdBody {
    VrAdj a;
    VrScal s;
    __device__ __forceinline__ void step(int, const float (&x)[3], const float (&)[1], const unsigned (&)[1],
                                         float (&o)[2]) {
        vr_bwd_step(x[0], x[1], x[2], s, a, o[0], o[1]);
    }
};

// inputs {V, r}, output {R}; `mask` = this column's ℓ byte of row 0, or NULL (not saved, or no such column)
struct UrFwdBody {
    float ret;
    UrHist h;
    int last;
    uint8_t* mask;
    int64_t B;
    __device__ __forceinline__ void step(int t, const float (&x)[2], const float (&)[1], const unsigned (&)[1],
                                         float (&o)[1]) {
        const float l = ur_fwd_step(x[0], x[1], t == last, h, ret);
        o[0] = ret;
        if (mask != nullptr) mask[static_cast<int64_t>(t) * B] = l != 0.f ? 1 : 0;
    }
};

// input {G}, byte input {ℓ}, outputs {grad_V of the next row, grad_r}
struct UrBwdBody {
    float carry;
    __device__ __forceinline__ void step(int, const float (&x)[1], const float (&)[1], const unsigned (&m)[1],
                                         float (&o)[2]) {
        o[1] = ur_bwd_step(x[0], m[0], carry, o[0]);
    }
};

// V_T of column `col`, the row no streamed box holds (0 outside the tensor)
__device__ __forceinline__ float last_value(const float* __restrict__ v, int64_t T, int64_t B, int64_t col, bool ok) {
    return ok ? __ldg(v + T * B + col) : 0.f;
}

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) vtrace_ret_fwd_tma(const __grid_constant__ TmapPack<4> maps,
                                                              const __grid_constant__ TmapPack<1> omaps,
                                                              const float* __restrict__ v, int T, int B, VrScal s) {
    using Pipe = ScanPipe<4, 0, 1, BT, TT, ST, 0>;
    const int col = blockIdx.x * BT + threadIdx.x;
    VrFwdBody body{0.f, last_value(v, T, B, col, threadIdx.x < BT && col < B), s};
    Pipe::template run<true>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
}

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) vtrace_ret_bwd_tma(const __grid_constant__ TmapPack<3> maps,
                                                              const __grid_constant__ TmapPack<2> omaps,
                                                              float* __restrict__ gv, int T, int B, VrScal s) {
    using Pipe = ScanPipe<3, 0, 2, BT, TT, ST, 0>;
    const int col = blockIdx.x * BT + threadIdx.x;
    VrBwdBody body{{-0.f, 0.f, -0.f}, s};
    Pipe::template run<false>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
    if (threadIdx.x < BT && col < B) gv[static_cast<int64_t>(T) * B + col] = body.a.gp;  // grad_V_T = g·p_{T−1}
}

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) upgo_ret_fwd_tma(const __grid_constant__ TmapPack<2> maps,
                                                            const __grid_constant__ TmapPack<1> omaps,
                                                            const float* __restrict__ v, uint8_t* __restrict__ mask,
                                                            int T, int B) {
    using Pipe = ScanPipe<2, 0, 1, BT, TT, ST, 0>;
    const int col = blockIdx.x * BT + threadIdx.x;
    const bool ok = threadIdx.x < BT && col < B;
    UrFwdBody body{0.f, {last_value(v, T, B, col, ok), 0.f, 0.f}, T - 1, ok && mask ? mask + col : nullptr, B};
    Pipe::template run<true>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
}

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) upgo_ret_bwd_tma(const __grid_constant__ TmapPack<2> maps,
                                                            const __grid_constant__ TmapPack<2> omaps, int T) {
    using Pipe = ScanPipe<1, 1, 2, BT, TT, ST, 0>;
    UrBwdBody body{-0.f};
    Pipe::template run<false>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
}

// ------------------------------------------------------------------------------------------------
// generic path: the same bodies driven by scan_column, one column per thread
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) vtrace_ret_fwd_generic(const float* __restrict__ v, const float* __restrict__ r,
                                                              const float* __restrict__ rho,
                                                              const float* __restrict__ c, float* __restrict__ ret,
                                                              int64_t T, int64_t B, VrScal s) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    VrFwdBody body{0.f, last_value(v, T, B, col, true), s};
    scan_column<4, 0, 1, 0, true>({{v, B}, {r, B}, {rho, B}, {c, B}}, {{nullptr, B}}, nullptr, {{ret, B}}, T, col,
                                  body);
}

__global__ void __launch_bounds__(128) vtrace_ret_bwd_generic(const float* __restrict__ grad_ret,
                                                              const float* __restrict__ rho,
                                                              const float* __restrict__ c, float* __restrict__ gv,
                                                              float* __restrict__ gr, int64_t T, int64_t B, VrScal s) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    VrBwdBody body{{-0.f, 0.f, -0.f}, s};
    scan_column<3, 0, 2, 0, false>({{grad_ret, B}, {rho, B}, {c, B}}, {{nullptr, B}}, nullptr, {{gv, B}, {gr, B}}, T,
                                   col, body);
    gv[T * B + col] = body.a.gp;
}

__global__ void __launch_bounds__(128) upgo_ret_fwd_generic(const float* __restrict__ v, const float* __restrict__ r,
                                                            float* __restrict__ ret, uint8_t* __restrict__ mask,
                                                            int64_t T, int64_t B) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    UrFwdBody body{0.f, {last_value(v, T, B, col, true), 0.f, 0.f}, static_cast<int>(T - 1),
                   mask ? mask + col : nullptr, B};
    scan_column<2, 0, 1, 0, true>({{v, B}, {r, B}}, {{nullptr, B}}, nullptr, {{ret, B}}, T, col, body);
}

// gv1: grad_bootstrap_values + B, the row of V_1
__global__ void __launch_bounds__(128) upgo_ret_bwd_generic(const float* __restrict__ grad_ret,
                                                            const uint8_t* __restrict__ mask, float* __restrict__ gv1,
                                                            float* __restrict__ gr, int64_t T, int64_t B) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    UrBwdBody body{-0.f};
    scan_column<1, 1, 2, 0, false>({{grad_ret, B}}, {{mask, B}}, nullptr, {{gv1, B}, {gr, B}}, T, col, body);
}

// ------------------------------------------------------------------------------------------------
// small-batch path: single-launch T-split with look-back (scan_lookback.cuh).  The streamed operands are staged in
// shared memory by lb_segment; what a segment needs from beyond its edge (V-trace: V_{t1}, or ρ, c of row t0−1;
// UPGO: V_{t1}, V_{t1+1}, r_{t1}) is loaded by the Fac, and the UPGO mask byte of a step by the step.
// ------------------------------------------------------------------------------------------------
struct VrFwdLbFac {
    const float* v;
    float* ret;
    int64_t B;
    int col;
    bool valid;
    VrScal s;
    struct Body {
        float item, v1, coef;
        bool store;
    };
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {
        return Body{carry, last_value(v, t_edge, B, col, valid), 1.f, valid && pass == 1};
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[4]) const {
        b.coef = vr_fwd_step(x[0], x[1], x[2], x[3], s, b.item, b.v1);
        if (b.store) st_stream(ret + static_cast<int64_t>(t) * B + col, __fadd_rn(x[0], b.item));
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.item; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.coef; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) vtrace_ret_fwd_lookback(const float* __restrict__ v,
                                                                   const float* __restrict__ r,
                                                                   const float* __restrict__ rho,
                                                                   const float* __restrict__ c,
                                                                   float* __restrict__ ret, int T, int B, VrScal s,
                                                                   int S, int L, int tiles, LbCtl* ctl,
                                                                   unsigned long long* words) {
    __shared__ float smem[4 * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;  // backward in time: the last segment goes first
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const VrFwdLbFac fac{v, ret, B, col, col < B, s};
    const float* const in[4] = {v, r, rho, c};
    const int64_t ld[4] = {B, B, B, B};
    lb_segment<4, true, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

// The state carried across segments is w (not f·c·w, which would lose p_{t0−1}): a segment starting at t0 > 0 rebuilds
// f·c_{t0−1} and g·p_{t0−1} from the carry-in w_{t0−1} and row t0−1 of ρ and c.
struct VrBwdLbFac {
    const float* rho;
    const float* c;
    float *gv, *gr;
    int64_t B;
    int col, T;
    bool valid;
    VrScal s;
    struct Body {
        VrAdj a;
        float coef;
        bool store;
    };
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {
        Body b{{-0.f, 0.f, -0.f}, 1.f, valid && pass == 1};
        if (t_edge > 0) {
            const int64_t i = static_cast<int64_t>(t_edge - 1) * B + col;
            const float rr = valid ? __ldg(rho + i) : 0.f, cc = valid ? __ldg(c + i) : 0.f;
            b.a = VrAdj{carry, __fmul_rn(s.f, cc), __fmul_rn(s.g, __fmul_rn(carry, rr))};
        }
        return b;
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[3]) const {
        float gvt, grt;
        b.coef = vr_bwd_step(x[0], x[1], x[2], s, b.a, gvt, grt);
        if (b.store) {
            const int64_t i = static_cast<int64_t>(t) * B + col;
            st_stream(gv + i, gvt);
            st_stream(gr + i, grt);
        }
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.a.w; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.coef; }
    __device__ __forceinline__ void finish(Body& b, int, int t1) const {
        if (b.store && t1 == T) gv[static_cast<int64_t>(T) * B + col] = b.a.gp;
    }
};

__global__ void __launch_bounds__(kLbCols) vtrace_ret_bwd_lookback(const float* __restrict__ grad_ret,
                                                                   const float* __restrict__ rho,
                                                                   const float* __restrict__ c,
                                                                   float* __restrict__ gv, float* __restrict__ gr,
                                                                   int T, int B, VrScal s, int S, int L, int tiles,
                                                                   LbCtl* ctl, unsigned long long* words) {
    __shared__ float smem[3 * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int t0 = lt.k * L, t1 = min(T, t0 + L);  // forward in time
    const int col = lt.tile * kLbCols + threadIdx.x;
    const VrBwdLbFac fac{rho, c, gv, gr, B, col, T, col < B, s};
    const float* const in[3] = {grad_ret, rho, c};
    const int64_t ld[3] = {B, B, B};
    lb_segment<3, false, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

struct UrFwdLbFac {
    const float* v;
    const float* r;
    float* ret;
    uint8_t* mask;
    int64_t B;
    int col, T;
    bool valid;
    struct Body {
        float ret, coef;
        UrHist h;
        bool store;
    };
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {
        const bool in = valid && t_edge < T;  // rows t_edge+1 of V and t_edge of r exist
        const UrHist h{last_value(v, t_edge, B, col, valid), last_value(v, t_edge + 1, B, col, in),
                       last_value(r, t_edge, B, col, in)};
        return Body{carry, 1.f, h, valid && pass == 1};
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[2]) const {
        b.coef = ur_fwd_step(x[0], x[1], t == T - 1, b.h, b.ret);
        if (b.store) {
            const int64_t i = static_cast<int64_t>(t) * B + col;
            st_stream(ret + i, b.ret);
            if (mask != nullptr) mask[i] = b.coef != 0.f ? 1 : 0;
        }
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.ret; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.coef; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) upgo_ret_fwd_lookback(const float* __restrict__ v,
                                                                 const float* __restrict__ r, float* __restrict__ ret,
                                                                 uint8_t* __restrict__ mask, int T, int B, int S,
                                                                 int L, int tiles, LbCtl* ctl,
                                                                 unsigned long long* words) {
    __shared__ float smem[2 * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const UrFwdLbFac fac{v, r, ret, mask, B, col, T, col < B};
    const float* const in[2] = {v, r};
    const int64_t ld[2] = {B, B};
    lb_segment<2, true, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

struct UrBwdLbFac {
    const uint8_t* mask;
    float *gv1, *gr;
    int64_t B;
    int col;
    bool valid;
    struct Body {
        float carry, coef;
        bool store;
    };
    __device__ __forceinline__ Body make(int pass, int, float carry) const {
        return Body{carry, 1.f, valid && pass == 1};
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[1]) const {
        const int64_t i = static_cast<int64_t>(t) * B + col;
        const unsigned m = valid ? ld_mask(mask, i) : 0u;
        float gvt;
        const float u = ur_bwd_step(x[0], m, b.carry, gvt);
        b.coef = m != 0u ? 1.f : 0.f;
        if (b.store) {
            st_stream(gv1 + i, gvt);
            st_stream(gr + i, u);
        }
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.carry; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.coef; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) upgo_ret_bwd_lookback(const float* __restrict__ grad_ret,
                                                                 const uint8_t* __restrict__ mask,
                                                                 float* __restrict__ gv1, float* __restrict__ gr,
                                                                 int T, int B, int S, int L, int tiles, LbCtl* ctl,
                                                                 unsigned long long* words) {
    __shared__ float smem[kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int t0 = lt.k * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const UrBwdLbFac fac{mask, gv1, gr, B, col, col < B};
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

// the wide path's tile <BT, TT, ST>: λ-returns' (DESIGN.md §4.15)
constexpr int kFwdBT = 256, kFwdTT = 4, kFwdST = 5;
constexpr int kBwdBT = 256, kBwdTT = 4, kBwdST = 6;

int pick(int64_t T, int64_t B, LbGeom* lg) {
    if (lookback_geometry(HPC_RLL_OP_LAMBDA_RETURNS, T, B, lg)) return kCfgLookback;
    const int forced = tuning_config(HPC_RLL_OP_LAMBDA_RETURNS);
    return forced == kCfgGeneric ? kCfgGeneric : kCfgWide;  // 21 on a shape that does not split: automatic
}

// every fp32 (T,B) operand TMA-describable: 16-byte aligned, B % 4 == 0
bool wide_ok(std::initializer_list<const void*> f32, int64_t B) {
    for (const void* q : f32)
        if (!tma_ok_2d(q, B, B)) return false;
    return true;
}

template <int N>
int f32_maps(TmapPack<N>* maps, std::initializer_list<const float*> ops, int64_t T, int64_t B, int TT, int BT) {
    int k = 0;
    for (const float* q : ops)
        if (int rc = make_tmap_2d(&maps->m[k++], q, T, B, B, TT, BT)) return rc;
    return HPC_RLL_OK;
}

unsigned grid_of(int64_t B, int BT) { return static_cast<unsigned>((B + BT - 1) / BT); }

int launched() {
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

int check_args(const char* what, int64_t T, int64_t B) {
    HPC_REQUIRE(T >= 0 && B >= 0, "%s: negative size T=%lld B=%lld", what, (long long)T, (long long)B);
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512, "%s: T/B exceed 2^31", what);
    return HPC_RLL_OK;
}

VrScal vr_scalars(double gamma, double lambda) {
    return VrScal{static_cast<float>(gamma), static_cast<float>(gamma * lambda)};  // γ·λ in double, as origin's Python
}

}  // namespace

static int vtrace_return_forward_impl(const float* rhos, const float* cs, const float* reward, const float* bootstrap,
                                      float* ret, int64_t T, int64_t B, double gamma, double lambda,
                                      cudaStream_t stream) {
    if (int rc = check_args("vtrace_return_forward", T, B)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(rhos && cs && reward && bootstrap && ret,
                "vtrace_return_forward: null rhos, cs, reward, bootstrap_values or returns pointer");
    const VrScal s = vr_scalars(gamma, lambda);
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        vtrace_ret_fwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            bootstrap, reward, rhos, cs, ret, static_cast<int>(T), static_cast<int>(B), s, lg.S, lg.L, lg.tiles,
            sc.ctl, sc.words);
        return launched();
    }
    if (cfg == kCfgWide && wide_ok({bootstrap, reward, rhos, cs, ret}, B)) {
        constexpr int BT = kFwdBT, TT = kFwdTT;
        TmapPack<4> maps;
        TmapPack<1> omaps;
        if (int rc = f32_maps(&maps, {bootstrap, reward, rhos, cs}, T, B, TT, BT)) return rc;
        if (int rc = f32_maps(&omaps, {ret}, T, B, TT, BT)) return rc;
        return launch_scan<ScanPipe<4, 0, 1, BT, TT, kFwdST, 0>, vtrace_ret_fwd_tma<BT, TT, kFwdST>>(
            grid_of(B, BT), stream, maps, omaps, bootstrap, static_cast<int>(T), static_cast<int>(B), s);
    }
    vtrace_ret_fwd_generic<<<grid_of(B, 128), 128, 0, stream>>>(bootstrap, reward, rhos, cs, ret, T, B, s);
    return launched();
}

static int vtrace_return_backward_impl(const float* grad_ret, const float* rhos, const float* cs, float* grad_reward,
                                       float* grad_bootstrap, int64_t T, int64_t B, double gamma, double lambda,
                                       cudaStream_t stream) {
    if (int rc = check_args("vtrace_return_backward", T, B)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(grad_ret && rhos && cs && grad_reward && grad_bootstrap,
                "vtrace_return_backward: null grad_returns, rhos, cs, grad_reward or grad_bootstrap_values pointer");
    const VrScal s = vr_scalars(gamma, lambda);
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        vtrace_ret_bwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            grad_ret, rhos, cs, grad_bootstrap, grad_reward, static_cast<int>(T), static_cast<int>(B), s, lg.S, lg.L,
            lg.tiles, sc.ctl, sc.words);
        return launched();
    }
    if (cfg == kCfgWide && wide_ok({grad_ret, rhos, cs, grad_reward, grad_bootstrap}, B)) {
        constexpr int BT = kBwdBT, TT = kBwdTT;
        TmapPack<3> maps;
        TmapPack<2> omaps;
        if (int rc = f32_maps(&maps, {grad_ret, rhos, cs}, T, B, TT, BT)) return rc;
        if (int rc = f32_maps(&omaps, {grad_bootstrap, grad_reward}, T, B, TT, BT)) return rc;
        return launch_scan<ScanPipe<3, 0, 2, BT, TT, kBwdST, 0>, vtrace_ret_bwd_tma<BT, TT, kBwdST>>(
            grid_of(B, BT), stream, maps, omaps, grad_bootstrap, static_cast<int>(T), static_cast<int>(B), s);
    }
    vtrace_ret_bwd_generic<<<grid_of(B, 128), 128, 0, stream>>>(grad_ret, rhos, cs, grad_bootstrap, grad_reward, T, B,
                                                                s);
    return launched();
}

static int upgo_returns_forward_impl(const float* rewards, const float* bootstrap, float* ret, uint8_t* mask,
                                     int64_t T, int64_t B, cudaStream_t stream) {
    if (int rc = check_args("upgo_returns_forward", T, B)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(rewards && bootstrap && ret, "upgo_returns_forward: null rewards, bootstrap_values or returns pointer");
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        upgo_ret_fwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            bootstrap, rewards, ret, mask, static_cast<int>(T), static_cast<int>(B), lg.S, lg.L, lg.tiles, sc.ctl,
            sc.words);
        return launched();
    }
    if (cfg == kCfgWide && wide_ok({bootstrap, rewards, ret}, B)) {  // the ℓ bytes are plain stores
        constexpr int BT = kFwdBT, TT = kFwdTT;
        TmapPack<2> maps;
        TmapPack<1> omaps;
        if (int rc = f32_maps(&maps, {bootstrap, rewards}, T, B, TT, BT)) return rc;
        if (int rc = f32_maps(&omaps, {ret}, T, B, TT, BT)) return rc;
        return launch_scan<ScanPipe<2, 0, 1, BT, TT, kFwdST, 0>, upgo_ret_fwd_tma<BT, TT, kFwdST>>(
            grid_of(B, BT), stream, maps, omaps, bootstrap, mask, static_cast<int>(T), static_cast<int>(B));
    }
    upgo_ret_fwd_generic<<<grid_of(B, 128), 128, 0, stream>>>(bootstrap, rewards, ret, mask, T, B);
    return launched();
}

static int upgo_returns_backward_impl(const float* grad_ret, const uint8_t* mask, float* grad_rewards,
                                      float* grad_bootstrap, int64_t T, int64_t B, cudaStream_t stream) {
    if (int rc = check_args("upgo_returns_backward", T, B)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(grad_ret && mask && grad_rewards && grad_bootstrap,
                "upgo_returns_backward: null grad_returns, lambda_mask, grad_rewards or grad_bootstrap_values pointer");
    // no return reads V_0: its gradient is +0
    HPC_CUDA(cudaMemsetAsync(grad_bootstrap, 0, static_cast<size_t>(B) * sizeof(float), stream));
    float* gv1 = grad_bootstrap + B;
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        upgo_ret_bwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            grad_ret, mask, gv1, grad_rewards, static_cast<int>(T), static_cast<int>(B), lg.S, lg.L, lg.tiles, sc.ctl,
            sc.words);
        return launched();
    }
    if (cfg == kCfgWide && wide_ok({grad_ret, gv1, grad_rewards}, B) && B % 16 == 0 && aligned16(mask)) {
        constexpr int BT = kBwdBT, TT = kBwdTT;
        TmapPack<2> maps;
        TmapPack<2> omaps;
        if (int rc = f32_maps(&maps, {grad_ret}, T, B, TT, BT)) return rc;
        if (int rc = make_tmap_2d_u8(&maps.m[1], mask, T, B, B, TT, BT)) return rc;
        if (int rc = f32_maps(&omaps, {gv1, grad_rewards}, T, B, TT, BT)) return rc;
        return launch_scan<ScanPipe<1, 1, 2, BT, TT, kBwdST, 0>, upgo_ret_bwd_tma<BT, TT, kBwdST>>(
            grid_of(B, BT), stream, maps, omaps, static_cast<int>(T));
    }
    upgo_ret_bwd_generic<<<grid_of(B, 128), 128, 0, stream>>>(grad_ret, mask, gv1, grad_rewards, T, B);
    return launched();
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_vtrace_return_forward(const float* rhos, const float* cs, const float* reward,
                                  const float* bootstrap_values, float* returns, int64_t T, int64_t B, double gamma,
                                  double lambda, void* stream) {
    HPC_NVTX("vtrace_return_forward");
    return hpcrll::vtrace_return_forward_impl(rhos, cs, reward, bootstrap_values, returns, T, B, gamma, lambda,
                                              hpcrll::as_stream(stream));
}

int hpc_rll_vtrace_return_backward(const float* grad_returns, const float* rhos, const float* cs, float* grad_reward,
                                   float* grad_bootstrap_values, int64_t T, int64_t B, double gamma, double lambda,
                                   void* stream) {
    HPC_NVTX("vtrace_return_backward");
    return hpcrll::vtrace_return_backward_impl(grad_returns, rhos, cs, grad_reward, grad_bootstrap_values, T, B, gamma,
                                               lambda, hpcrll::as_stream(stream));
}

int hpc_rll_upgo_returns_forward(const float* rewards, const float* bootstrap_values, float* returns,
                                 uint8_t* lambda_mask, int64_t T, int64_t B, void* stream) {
    HPC_NVTX("upgo_returns_forward");
    return hpcrll::upgo_returns_forward_impl(rewards, bootstrap_values, returns, lambda_mask, T, B,
                                             hpcrll::as_stream(stream));
}

int hpc_rll_upgo_returns_backward(const float* grad_returns, const uint8_t* lambda_mask, float* grad_rewards,
                                  float* grad_bootstrap_values, int64_t T, int64_t B, void* stream) {
    HPC_NVTX("upgo_returns_backward");
    return hpcrll::upgo_returns_backward_impl(grad_returns, lambda_mask, grad_rewards, grad_bootstrap_values, T, B,
                                              hpcrll::as_stream(stream));
}

}  // extern "C"
