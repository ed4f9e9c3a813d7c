// gae_episodic.cu -- episode-aware (un-normalised) GAE, forward and adjoint, for sm_90a.
//
// Semantics: DI-engine's functional `gae(gae_data(value, next_value, reward, done, traj_flag), gamma, lambda_)`,
// i.e. standard GAE over a (T,B) segment whose columns may hold several episodes:
//     nv_t    = next_value_t * (1 - done_t)
//     delta_t = (reward_t + g * nv_t) - value_t                 g  = fp32(gamma)
//     f_t     = gl * (1 - traj_t)                               gl = fp32(gamma * lambda), product in double
//     adv_t   = delta_t + f_t * adv_{t+1},   adv_{T-1} = delta_{T-1}
// Adjoint (G = dL/dadv), a forward-in-time scan:
//     u_0 = G_0,  u_t = G_t + f_{t-1} * u_{t-1}
//     grad_reward = u, grad_value = -u, grad_next_value = (g * u) * (1 - done)
// Masks are bytes (non-zero = set; NULL = all zero) and enter as multiplications by (1 - mask), so a non-finite
// next_value or carry propagates exactly as in eager PyTorch.  Every operation is one round-to-nearest fp32 op in the
// order above (explicit __f*_rn, no FMA contraction): the wide and generic kernels are bit-identical to eager PyTorch
// of the formula on the CPU.  The scans carry adv_{t+1} (forward) and f_t * u_t (backward) starting from -0, the
// additive identity, so the first row is delta_{T-1} / G_0 exactly, signed zeros included (for gamma*lambda >= 0).
//
// Regimes (hpc_rll_debug_set_config(HPC_RLL_OP_GAE_EPISODIC, id) / HPC_RLL_CFG_GAE_EPISODIC force one):
//   33 wide   ScanPipe (scan_pipe.cuh): value/next_value/reward and the two masks TMA-staged in (TT x BT) boxes,
//             outputs TMA-stored.  Needs 16-byte aligned pointers and B % 16 == 0 with masks (a uint8 tensor map
//             needs a 16-byte row stride), B % 4 == 0 without.
//   21 look-back  single-launch T-split (scan_lookback.cuh), automatic for B <= 2048 and T >= 512.  The recurrence
//             has a per-element coefficient (CONSTA = false): each segment publishes A = prod f_t.
//   99 generic the wide bodies driven by scan_column (scan_pipe.cuh), one column per thread: ragged B, misaligned
//             pointers, short T.
// HBM traffic = algorithmic: forward 3 fp32 + 2 byte reads + 1 fp32 write = 18 B per element, backward 1 fp32 +
// 2 byte reads + 3 fp32 writes = 18 B per element.  No atomics except the look-back tickets and counters.
#include <cstdint>
#include <initializer_list>

#include "scan_lookback.cuh"
#include "scan_pipe.cuh"

namespace hpcrll {

namespace {

// 1 - mask as a factor: 0 when the byte is set, 1 otherwise
__device__ __forceinline__ float keep(unsigned m) { return m != 0u ? 0.f : 1.f; }

// one forward step: `carry` = adv_{t+1} on entry (-0 before the last row), adv_t on exit; `f` = f_t
__device__ __forceinline__ float fwd_step(float value, float next_value, float reward, unsigned done, unsigned traj,
                                          float g, float gl, float& carry, float& f) {
    const float nv = __fmul_rn(next_value, keep(done));
    const float delta = __fsub_rn(__fadd_rn(reward, __fmul_rn(g, nv)), value);
    f = __fmul_rn(gl, keep(traj));
    carry = __fadd_rn(delta, __fmul_rn(f, carry));
    return carry;
}

// one backward step: `c` = f_{t-1} * u_{t-1} on entry, f_t * u_t on exit
struct BwdOut {
    float gv, gnv, gr;
};
__device__ __forceinline__ BwdOut bwd_step(float G, unsigned done, unsigned traj, float g, float gl, float& c,
                                           float& f) {
    const float u = __fadd_rn(G, c);
    f = __fmul_rn(gl, keep(traj));
    c = __fmul_rn(f, u);
    return BwdOut{-u, __fmul_rn(__fmul_rn(g, u), keep(done)), u};
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// wide path: ScanPipe with byte boxes.  NB = 2 reads both masks (a NULL one is replaced by the other's map and ignored
// through has_done / has_traj), NB = 0 reads none.
// ------------------------------------------------------------------------------------------------
template <int NB>
struct EpiFwdBody {
    float carry, g, gl;
    int has_done, has_traj;
    __device__ __forceinline__ void step(int, const float (&x)[3], const float (&)[1],
                                         const unsigned (&m)[NB > 0 ? NB : 1], float (&o)[1]) {
        const unsigned d = NB > 0 && has_done ? m[0] : 0u;
        const unsigned tr = NB > 0 && has_traj ? m[NB > 1 ? 1 : 0] : 0u;
        float f;
        o[0] = fwd_step(x[0], x[1], x[2], d, tr, g, gl, carry, f);
    }
};

template <int NB, int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) gae_episodic_fwd_tma(const __grid_constant__ TmapPack<3 + NB> maps,
                                                                 const __grid_constant__ TmapPack<1> omaps, int T,
                                                                 float g, float gl, int has_done, int has_traj) {
    using Pipe = ScanPipe<3, NB, 1, BT, TT, ST, 0>;
    EpiFwdBody<NB> body{-0.f, g, gl, has_done, has_traj};
    Pipe::template run<true>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
}

template <int NB>
struct EpiBwdBody {
    float c, g, gl;
    int has_done, has_traj;
    __device__ __forceinline__ void step(int, const float (&x)[1], const float (&)[1],
                                         const unsigned (&m)[NB > 0 ? NB : 1], float (&o)[3]) {
        const unsigned d = NB > 0 && has_done ? m[0] : 0u;
        const unsigned tr = NB > 0 && has_traj ? m[NB > 1 ? 1 : 0] : 0u;
        float f;
        const BwdOut r = bwd_step(x[0], d, tr, g, gl, c, f);
        o[0] = r.gv;
        o[1] = r.gnv;
        o[2] = r.gr;
    }
};

template <int NB, int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) gae_episodic_bwd_tma(const __grid_constant__ TmapPack<1 + NB> maps,
                                                                 const __grid_constant__ TmapPack<3> omaps, int T,
                                                                 float g, float gl, int has_done, int has_traj) {
    using Pipe = ScanPipe<1, NB, 3, BT, TT, ST, 0>;
    EpiBwdBody<NB> body{-0.f, g, gl, has_done, has_traj};
    Pipe::template run<false>(maps, omaps, nullptr, T, blockIdx.x * BT, body);
}

// ------------------------------------------------------------------------------------------------
// generic path: the wide bodies driven by scan_column (scan_pipe.cuh); a NULL mask reads as 0
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) gae_episodic_fwd_generic(const float* __restrict__ value,
                                                                 const float* __restrict__ next_value,
                                                                 const float* __restrict__ reward,
                                                                 const uint8_t* __restrict__ done,
                                                                 const uint8_t* __restrict__ traj,
                                                                 float* __restrict__ adv, int64_t T, int64_t B,
                                                                 float g, float gl) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    EpiFwdBody<2> body{-0.f, g, gl, 1, 1};
    scan_column<3, 2, 1, 0, true>({{value, B}, {next_value, B}, {reward, B}}, {{done, B}, {traj, B}}, nullptr,
                                  {{adv, B}}, T, col, body);
}

__global__ void __launch_bounds__(128) gae_episodic_bwd_generic(const float* __restrict__ grad_adv,
                                                                 const uint8_t* __restrict__ done,
                                                                 const uint8_t* __restrict__ traj,
                                                                 float* __restrict__ gv, float* __restrict__ gnv,
                                                                 float* __restrict__ gr, int64_t T, int64_t B,
                                                                 float g, float gl) {
    const int64_t col = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (col >= B) return;
    EpiBwdBody<2> body{-0.f, g, gl, 1, 1};
    scan_column<1, 2, 3, 0, false>({{grad_adv, B}}, {{done, B}, {traj, B}}, nullptr, {{gv, B}, {gnv, B}, {gr, B}}, T,
                                   col, body);
}

// ------------------------------------------------------------------------------------------------
// small-batch path: single-launch T-split with look-back (scan_lookback.cuh).  lb_segment stages the fp32 operands
// in shared memory; the mask bytes of a step are read by the Fac straight from global memory (a warp's 32 bytes of a
// row are one sector, and the loads do not depend on the carry, so they issue ahead of the chain like the staged
// ones), which leaves lb_segment and lb_stage -- and the code of every existing look-back kernel -- unchanged.
// ------------------------------------------------------------------------------------------------
struct EpiLbBody {
    float carry, f;
    float* out0;
    bool store;
};

struct EpiFwdLbFac {
    const uint8_t* done;
    const uint8_t* traj;
    float* adv;
    int64_t B;
    int col;
    bool valid;
    float g, gl;
    using Body = EpiLbBody;
    __device__ __forceinline__ Body make(int pass, int, float carry) const {
        return Body{carry, 1.f, adv, valid && pass == 1};
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[3]) const {
        const int64_t i = static_cast<int64_t>(t) * B + col;
        const unsigned d = valid ? ld_mask(done, i) : 0u, tr = valid ? ld_mask(traj, i) : 0u;
        const float a = fwd_step(x[0], x[1], x[2], d, tr, g, gl, b.carry, b.f);
        if (b.store) st_stream(b.out0 + i, a);
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.carry; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.f; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) gae_episodic_fwd_lookback(const float* __restrict__ value,
                                                                      const float* __restrict__ next_value,
                                                                      const float* __restrict__ reward,
                                                                      const uint8_t* __restrict__ done,
                                                                      const uint8_t* __restrict__ traj,
                                                                      float* __restrict__ adv, int T, int B, float g,
                                                                      float gl, int S, int L, int tiles, LbCtl* ctl,
                                                                      unsigned long long* words) {
    __shared__ float smem[3 * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;  // backward in time: the last segment goes first
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const EpiFwdLbFac fac{done, traj, adv, B, col, col < B, g, gl};
    const float* const in[3] = {value, next_value, reward};
    const int64_t ld[3] = {B, B, B};
    lb_segment<3, true, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

struct EpiBwdLbFac {
    const uint8_t* done;
    const uint8_t* traj;
    float *gv, *gnv, *gr;
    int64_t B;
    int col;
    bool valid;
    float g, gl;
    using Body = EpiLbBody;
    __device__ __forceinline__ Body make(int pass, int, float carry) const {
        return Body{carry, 1.f, nullptr, valid && pass == 1};
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[1]) const {
        const int64_t i = static_cast<int64_t>(t) * B + col;
        const unsigned d = valid ? ld_mask(done, i) : 0u, tr = valid ? ld_mask(traj, i) : 0u;
        const BwdOut o = bwd_step(x[0], d, tr, g, gl, b.carry, b.f);
        if (b.store) {
            st_stream(gv + i, o.gv);
            st_stream(gnv + i, o.gnv);
            st_stream(gr + i, o.gr);
        }
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.carry; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.f; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) gae_episodic_bwd_lookback(const float* __restrict__ grad_adv,
                                                                      const uint8_t* __restrict__ done,
                                                                      const uint8_t* __restrict__ traj,
                                                                      float* __restrict__ gv, float* __restrict__ gnv,
                                                                      float* __restrict__ gr, int T, int B, float g,
                                                                      float gl, int S, int L, int tiles, LbCtl* ctl,
                                                                      unsigned long long* words) {
    __shared__ float smem[kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int t0 = lt.k * L, t1 = min(T, t0 + L);  // forward in time
    const int col = lt.tile * kLbCols + threadIdx.x;
    const EpiBwdLbFac fac{done, traj, gv, gnv, gr, B, col, col < B, g, gl};
    const float* const in[1] = {grad_adv};
    const int64_t ld[1] = {B};
    lb_segment<1, false, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

// ------------------------------------------------------------------------------------------------
// launchers and dispatch
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int kCfgWide = 33, kCfgLookback = 21, kCfgGeneric = 99;

// the wide path's tile: <BT, TT, ST> = columns per CTA, rows per box, ring stages.  On H100 at T=1024, B=65536 this
// pair was the fastest or tied among <256,4,5|6> <128,8,4> <256,8,3> <128,4,8> <256,4,8> (sweep in DESIGN.md §4.13)
constexpr int kFwdBT = 256, kFwdTT = 4, kFwdST = 5;
constexpr int kBwdBT = 256, kBwdTT = 4, kBwdST = 6;

struct Masks {
    const uint8_t* done;
    const uint8_t* traj;
    bool any() const { return done != nullptr || traj != nullptr; }
};

// every operand TMA-describable: fp32 (T,B) needs B % 4 == 0, a uint8 (T,B) map B % 16 == 0
bool wide_ok(std::initializer_list<const void*> f32, const Masks& mk, int64_t B) {
    for (const void* p : f32)
        if (!tma_ok_2d(p, B, B)) return false;
    if (!mk.any()) return true;
    if (B % 16 != 0) return false;
    return (mk.done == nullptr || aligned16(mk.done)) && (mk.traj == nullptr || aligned16(mk.traj));
}

int pick(int64_t T, int64_t B, LbGeom* lg) {
    if (lookback_geometry(HPC_RLL_OP_GAE_EPISODIC, T, B, lg)) return kCfgLookback;
    const int forced = tuning_config(HPC_RLL_OP_GAE_EPISODIC);
    return forced == kCfgGeneric ? kCfgGeneric : kCfgWide;  // 21 on a shape that does not split: automatic
}

template <int NB>
int launch_fwd_tma(const float* value, const float* next_value, const float* reward, const Masks& mk, float* adv,
                   int64_t T, int64_t B, float g, float gl, cudaStream_t stream) {
    constexpr int BT = kFwdBT, TT = kFwdTT;
    TmapPack<3 + NB> maps;
    TmapPack<1> omaps;
    const float* in[3] = {value, next_value, reward};
    for (int k = 0; k < 3; ++k)
        if (int rc = make_tmap_2d(&maps.m[k], in[k], T, B, B, TT, BT)) return rc;
    if (NB > 0) {
        const uint8_t* d = mk.done ? mk.done : mk.traj;
        const uint8_t* tr = mk.traj ? mk.traj : mk.done;
        if (int rc = make_tmap_2d_u8(&maps.m[3], d, T, B, B, TT, BT)) return rc;
        if (int rc = make_tmap_2d_u8(&maps.m[3 + NB - 1], tr, T, B, B, TT, BT)) return rc;
    }
    if (int rc = make_tmap_2d(&omaps.m[0], adv, T, B, B, TT, BT)) return rc;
    const unsigned grid = static_cast<unsigned>((B + BT - 1) / BT);
    return launch_scan<ScanPipe<3, NB, 1, BT, TT, kFwdST, 0>, gae_episodic_fwd_tma<NB, BT, TT, kFwdST>>(
        grid, stream, maps, omaps, static_cast<int>(T), g, gl, mk.done != nullptr, mk.traj != nullptr);
}

template <int NB>
int launch_bwd_tma(const float* grad_adv, const Masks& mk, float* gv, float* gnv, float* gr, int64_t T, int64_t B,
                   float g, float gl, cudaStream_t stream) {
    constexpr int BT = kBwdBT, TT = kBwdTT;
    TmapPack<1 + NB> maps;
    TmapPack<3> omaps;
    if (int rc = make_tmap_2d(&maps.m[0], grad_adv, T, B, B, TT, BT)) return rc;
    if (NB > 0) {
        const uint8_t* d = mk.done ? mk.done : mk.traj;
        const uint8_t* tr = mk.traj ? mk.traj : mk.done;
        if (int rc = make_tmap_2d_u8(&maps.m[1], d, T, B, B, TT, BT)) return rc;
        if (int rc = make_tmap_2d_u8(&maps.m[1 + NB - 1], tr, T, B, B, TT, BT)) return rc;
    }
    float* out[3] = {gv, gnv, gr};
    for (int k = 0; k < 3; ++k)
        if (int rc = make_tmap_2d(&omaps.m[k], out[k], T, B, B, TT, BT)) return rc;
    const unsigned grid = static_cast<unsigned>((B + BT - 1) / BT);
    return launch_scan<ScanPipe<1, NB, 3, BT, TT, kBwdST, 0>, gae_episodic_bwd_tma<NB, BT, TT, kBwdST>>(
        grid, stream, maps, omaps, static_cast<int>(T), g, gl, mk.done != nullptr, mk.traj != nullptr);
}

int check_sizes(const char* what, int64_t T, int64_t B) {
    HPC_REQUIRE(T >= 0 && B >= 0, "%s: negative size T=%lld B=%lld", what, (long long)T, (long long)B);
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512, "%s: T/B exceed 2^31", what);
    return HPC_RLL_OK;
}

}  // namespace

static int gae_episodic_forward_impl(const float* value, const float* next_value, const float* reward,
                                     const uint8_t* done, const uint8_t* traj, float* adv, int64_t T, int64_t B,
                                     double gamma, double lambda, cudaStream_t stream) {
    if (int rc = check_sizes("gae_episodic_forward", T, B)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(value && next_value && reward && adv,
                "gae_episodic_forward: null value, next_value, reward or adv pointer");
    const float g = static_cast<float>(gamma), gl = static_cast<float>(gamma * lambda);
    const Masks mk{done, traj};
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        gae_episodic_fwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            value, next_value, reward, done, traj, adv, static_cast<int>(T), static_cast<int>(B), g, gl, lg.S, lg.L,
            lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
    if (cfg == kCfgWide && wide_ok({value, next_value, reward, adv}, mk, B)) {
        if (mk.any()) return launch_fwd_tma<2>(value, next_value, reward, mk, adv, T, B, g, gl, stream);
        return launch_fwd_tma<0>(value, next_value, reward, mk, adv, T, B, g, gl, stream);
    }
    gae_episodic_fwd_generic<<<static_cast<unsigned>((B + 127) / 128), 128, 0, stream>>>(value, next_value, reward,
                                                                                         done, traj, adv, T, B, g, gl);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

static int gae_episodic_backward_impl(const float* grad_adv, const uint8_t* done, const uint8_t* traj, float* gv,
                                      float* gnv, float* gr, int64_t T, int64_t B, double gamma, double lambda,
                                      cudaStream_t stream) {
    if (int rc = check_sizes("gae_episodic_backward", T, B)) return rc;
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(grad_adv && gv && gnv && gr,
                "gae_episodic_backward: null grad_adv, grad_value, grad_next_value or grad_reward pointer");
    const float g = static_cast<float>(gamma), gl = static_cast<float>(gamma * lambda);
    const Masks mk{done, traj};
    LbGeom lg;
    const int cfg = pick(T, B, &lg);
    if (cfg == kCfgLookback) {
        LbScratch sc;
        if (int rc = lookback_scratch(lg, B, stream, &sc)) return rc;
        gae_episodic_bwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            grad_adv, done, traj, gv, gnv, gr, static_cast<int>(T), static_cast<int>(B), g, gl, lg.S, lg.L, lg.tiles,
            sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
    if (cfg == kCfgWide && wide_ok({grad_adv, gv, gnv, gr}, mk, B)) {
        if (mk.any()) return launch_bwd_tma<2>(grad_adv, mk, gv, gnv, gr, T, B, g, gl, stream);
        return launch_bwd_tma<0>(grad_adv, mk, gv, gnv, gr, T, B, g, gl, stream);
    }
    gae_episodic_bwd_generic<<<static_cast<unsigned>((B + 127) / 128), 128, 0, stream>>>(grad_adv, done, traj, gv, gnv,
                                                                                         gr, T, B, g, gl);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_gae_episodic_forward(const float* value, const float* next_value, const float* reward,
                                 const uint8_t* done_u8, const uint8_t* traj_u8, float* adv, int64_t T, int64_t B,
                                 double gamma, double lambda, void* stream) {
    HPC_NVTX("gae_episodic_forward");
    return hpcrll::gae_episodic_forward_impl(value, next_value, reward, done_u8, traj_u8, adv, T, B, gamma, lambda,
                                             hpcrll::as_stream(stream));
}

int hpc_rll_gae_episodic_backward(const float* grad_adv, const uint8_t* done_u8, const uint8_t* traj_u8,
                                  float* grad_value, float* grad_next_value, float* grad_reward, int64_t T, int64_t B,
                                  double gamma, double lambda, void* stream) {
    HPC_NVTX("gae_episodic_backward");
    return hpcrll::gae_episodic_backward_impl(grad_adv, done_u8, traj_u8, grad_value, grad_next_value, grad_reward, T,
                                              B, gamma, lambda, hpcrll::as_stream(stream));
}

}  // extern "C"
