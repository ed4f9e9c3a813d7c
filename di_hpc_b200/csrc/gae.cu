// gae.cu -- Generalized Advantage Estimation, forward and adjoint, for sm_90a.
//
// Semantics: hpc_rll/origin/gae.py:28-37 (normalised GAE):
//     delta_t = r_t + gamma*v_{t+1} - v_t
//     d_t     = 1 + lambda*d_{t+1}            (d_T = 0; a Python double in origin)
//     g_t     = d_t*delta_t + gamma*lambda*g_{t+1}
//     adv_t   = g_t / d_t
// Replaces the reference's GaeForward (src/rl_utils/gae.cu:8-28) and gaeForwardKernel
// (include/hpc/rll/cuda/rl_utils/gae_kernel.h:10-29: one thread per column, <<<B/32,32>>>,
// three dependent scalar loads per step).  The reference has NO backward
// (hpc_rll/rl_utils/gae.py:16-18 returns None); gae_bwd here is the exact adjoint
// (SURVEY.md A.1), a forward-in-time scan:
//     ghat_t = G_t/d_t + gamma*lambda*ghat_{t-1};  dd_t = d_t*ghat_t
//     grad_reward_t = dd_t;   grad_value_t = gamma*dd_{t-1} - dd_t  (dd_{-1}=0, dd_T=0)
//
// Design: ScanPipe (scan_pipe.cuh) -- (TT x BT) boxes of value/reward (fwd) or grad_adv (bwd)
// plus the d_t slice are TMA-staged through a shared-memory ring; BT consumer threads own one
// column each, carry (g, v_{t+1}) in registers and stream results out with evict-first stores.
// From 256 columns per SM up the OUTPUT is TMA-staged as well (NOUT > 0: results collected in shared-memory
// boxes and written with cp.async.bulk.tensor stores; gae_*_tma_st, config 33) -- the fastest backward at the
// headline shape (see pick_cfg).
// HBM traffic = algorithmic: fwd 12 B/step, bwd 12 B/step (+ one extra value row).
//
// Arithmetic uses explicit round-to-nearest intrinsics in origin's operation order (no FMA
// contraction), so forward results are bit-identical to origin fp32 on CPU / oracle_f32.
// The division by d_t uses the table's correctly rounded reciprocal r_t = RN(1/d_t) and one FMA
// residual step (q0 = x*r; q = fma(fma(-d,q0,x), r, q0)) -- by Markstein's theorem this is the
// correctly rounded quotient for every normal-range x (brute-forced on 1.5e8 cases, see
// DESIGN.md); it costs 3 instructions instead of the ~14 of the generic IEEE division sequence.
// Non-finite x yields NaN (IEEE division would give +-inf for x = +-inf).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "reduce.cuh"
#include "scan_lookback.cuh"
#include "scan_pipe.cuh"

namespace hpcrll {

// ------------------------------------------------------------------------------------------------
// d_t table (device, fp32, cached per (device, T, lambda)).  Built on the host in double exactly as
// origin does (`denom = 1 + lambda_*denom` on Python floats, gae.py:34) and rounded once to fp32.
// Stored as interleaved pairs (d_t, RN(1/d_t)); padded with (1,1) to a multiple of 64 rows so every
// ring stage can bulk-copy a full slice.
// ------------------------------------------------------------------------------------------------
namespace {
struct DtabKey {
    int dev;
    int64_t T;
    uint64_t lam_bits;
    bool operator<(const DtabKey& o) const {
        if (dev != o.dev) return dev < o.dev;
        if (T != o.T) return T < o.T;
        return lam_bits < o.lam_bits;
    }
};
std::mutex g_dtab_mu;
struct DtabEntry {
    float* ptr;
    uint64_t last_use;
};
std::map<DtabKey, DtabEntry> g_dtab;
uint64_t g_dtab_tick = 0;
constexpr int kDtabPad = 64;
constexpr size_t kDtabMaxPerDevice = 1024;  // tables are 8*(T+128) bytes each
}  // namespace

static bool stream_capturing(cudaStream_t stream) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    return cudaStreamIsCapturing(stream, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone;
}

// Cache policy (ADVICE r1): bounded PER DEVICE; when a device's share is full the least recently used table OF
// THAT DEVICE is dropped after synchronising that device (the current one -- other devices' tables and streams
// are never touched).  Nothing is freed while `stream` is being captured (a synchronise would invalidate the
// capture); a table pointer baked into an instantiated graph stays valid as long as its (T, lambda) is among the
// 1024 most recently used on that device.
static int get_dtab(int64_t T, double lambda, cudaStream_t stream, const float** out) {
    int dev = 0;
    HPC_CUDA(cudaGetDevice(&dev));
    DtabKey key{dev, T, 0};
    std::memcpy(&key.lam_bits, &lambda, sizeof(double));
    std::lock_guard<std::mutex> lk(g_dtab_mu);
    auto it = g_dtab.find(key);
    if (it != g_dtab.end()) {
        it->second.last_use = ++g_dtab_tick;
        *out = it->second.ptr;
        return HPC_RLL_OK;
    }
    size_t mine = 0;
    auto lru = g_dtab.end();
    for (auto i = g_dtab.begin(); i != g_dtab.end(); ++i) {
        if (i->first.dev != dev) continue;
        ++mine;
        if (lru == g_dtab.end() || i->second.last_use < lru->second.last_use) lru = i;
    }
    if (mine >= kDtabMaxPerDevice && lru != g_dtab.end() && !stream_capturing(stream)) {
        HPC_CUDA(cudaDeviceSynchronize());  // this device only; its kernels may still read the table
        cudaFree(lru->second.ptr);
        g_dtab.erase(lru);
    }
    const int64_t padded = ((T + kDtabPad - 1) / kDtabPad) * kDtabPad + kDtabPad;
    std::vector<float> h(static_cast<size_t>(padded) * 2, 1.0f);
    double den = 0.0;
    for (int64_t t = T - 1; t >= 0; --t) {
        den = 1.0 + lambda * den;
        const float df = static_cast<float>(den);
        h[static_cast<size_t>(t) * 2] = df;
        h[static_cast<size_t>(t) * 2 + 1] = 1.0f / df;  // host fp32 division: correctly rounded
    }
    float* d = nullptr;
    HPC_CUDA(cudaMalloc(&d, sizeof(float) * h.size()));
    // blocking copy: the table is valid for every stream once this returns (first use per (T,lambda)
    // only; do one warm-up call before CUDA-graph capture)
    cudaError_t e = cudaMemcpy(d, h.data(), sizeof(float) * h.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(d);
        return set_error(HPC_RLL_ECUDA, "gae: uploading d_t table failed: %s", cudaGetErrorString(e));
    }
    g_dtab[key] = DtabEntry{d, ++g_dtab_tick};
    *out = d;
    return HPC_RLL_OK;
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
// correctly rounded x/d given r = RN(1/d) (see file header)
__device__ __forceinline__ float div_by_table(float x, float d, float r) {
    const float q0 = __fmul_rn(x, r);
    return __fmaf_rn(__fmaf_rn(-d, q0, x), r, q0);
}

namespace {

// one forward step: x = (v_t, r_t), dt = (d_t, 1/d_t), v1 = v_{t+1}; `g` = g_{t+1} on entry, g_t on exit.
// Returns adv_t.
__device__ __forceinline__ float fwd_step(const float (&x)[2], const float (&dt)[2], float v1, float gamma,
                                          float factor, float& g) {
    const float delta = __fsub_rn(__fadd_rn(x[1], __fmul_rn(gamma, v1)), x[0]);
    g = __fadd_rn(__fmul_rn(dt[0], delta), __fmul_rn(factor, g));
    return div_by_table(g, dt[0], dt[1]);
}

// one backward step: G = grad_adv_t, dt = (d_t, 1/d_t); `gh` = ghat_{t-1} on entry, ghat_t on exit; `prev` =
// dd_{t-1} on entry, dd_t on exit.  Returns (grad_value_t, grad_reward_t) = (gamma*dd_{t-1} - dd_t, dd_t).
struct BwdOut {
    float gv, gr;
};
__device__ __forceinline__ BwdOut bwd_step(float G, const float (&dt)[2], float gamma, float factor, float& gh,
                                           float& prev) {
    gh = __fadd_rn(div_by_table(G, dt[0], dt[1]), __fmul_rn(factor, gh));
    const float dd = __fmul_rn(dt[0], gh);
    const BwdOut o{__fsub_rn(__fmul_rn(gamma, prev), dd), dd};
    prev = dd;
    return o;
}

}  // namespace

// MOM: also accumulate sum(adv) and sum(adv^2) in fp64 (hpc_rll_gae_forward_moments)
template <bool MOM = false>
struct GaeFwdBody {
    float g, v1, gamma, factor;
    float* adv;  // running pointer: &adv[t][col] of the NEXT step (steps arrive with t descending)
    int64_t ld;
    bool valid;
    double m1, m2;
    float p1, p2;  // fp32 partial moments of the current 16-row run, folded into m1/m2 at t % 16 == 0
    // state at a segment edge: steps run from row t_edge-1 down, with g = g_{t_edge} (the carry) and
    // v1 = v_row[col] (value row t_edge); `valid`: column col exists
    static __device__ __forceinline__ GaeFwdBody at(int t_edge, float carry, const float* v_row, float* adv,
                                                    int64_t ld, int col, float gamma, float factor, bool valid) {
        GaeFwdBody b;
        b.valid = valid;
        b.g = carry;
        b.gamma = gamma;
        b.factor = factor;
        b.ld = ld;
        b.m1 = b.m2 = 0.0;
        b.p1 = b.p2 = 0.f;
        b.adv = adv + static_cast<int64_t>(t_edge - 1) * ld + col;
        b.v1 = valid ? __ldg(v_row + col) : 0.f;
        return b;
    }
    __device__ __forceinline__ void step(int t, const float (&x)[2], const float (&dt)[2]) {
        const float a = fwd_step(x, dt, v1, gamma, factor, g);
        if (valid) st_stream(adv, a);
        if (MOM) {  // t descends to 0, so the last run is always flushed
            p1 += a;
            p2 = fmaf(a, a, p2);
            if ((t & 15) == 0) {
                m1 += static_cast<double>(p1);
                m2 += static_cast<double>(p2);
                p1 = 0.f;
                p2 = 0.f;
            }
        }
        adv -= ld;
        v1 = x[0];
    }
};

// per-CTA moment partials -> partials[blockIdx.x] (sum) and partials[gridDim.x + blockIdx.x] (sum of squares)
template <bool MOM>
__device__ __forceinline__ void gae_store_moments(const GaeFwdBody<MOM>& body, double* __restrict__ partials,
                                                  double* red) {
    if (MOM) {
        double v[2] = {body.valid ? body.m1 : 0.0, body.valid ? body.m2 : 0.0};
        block_sum<2>(v, red);
        if (threadIdx.x == 0) {
            partials[blockIdx.x] = v[0];
            partials[gridDim.x + blockIdx.x] = v[1];
        }
    }
}

template <int BT, int TT, int ST, bool MOM>
__global__ void __launch_bounds__(BT + 32) gae_fwd_tma(const __grid_constant__ TmapPack<2> maps,
                                                        const float* __restrict__ dtab,
                                                        const float* __restrict__ v_next, float* __restrict__ carry,
                                                        float* __restrict__ adv, int64_t ld_adv, int T, int B,
                                                        float gamma, float factor, double* __restrict__ partials) {
    // v_next: the value row that follows the last row of this launch (value[T], or the carried row of a T-chunk);
    // carry (nullable): (2,B) scan state of a T-chunked run -- g in/out, value row out (see gae_forward_chunk)
    using Pipe = ScanPipe<2, 0, 0, BT, TT, ST, 2>;
    const int col0 = blockIdx.x * BT;
    const int col = col0 + threadIdx.x;
    const bool valid = threadIdx.x < BT && col < B;
    GaeFwdBody<MOM> body = GaeFwdBody<MOM>::at(T, 0.f, v_next, adv, ld_adv, col, gamma, factor, valid);
    if (carry != nullptr && valid) body.g = carry[col];  // after at(): loading it first reorders the machine code
    Pipe::template run<true>(maps, {}, dtab, T, col0, body);
    if (carry != nullptr && body.valid) {
        carry[col] = body.g;
        carry[B + col] = body.v1;
    }
    if constexpr (MOM) {
        __shared__ double red[64];
        gae_store_moments<MOM>(body, partials, red);
    }
}

struct GaeBwdBody {
    float gh, prev, gamma, factor;
    float* gv;
    float* gr;
    int64_t ld_gv, ld_gr;
    bool valid;
    // gv / gr are running pointers (&grad[t][col] of the next step; t ascending)
    // state at a segment edge: steps run from row t_edge up, with (gh, prev) = (ghat, dd) of row t_edge-1 (the carry)
    static __device__ __forceinline__ GaeBwdBody at(int t_edge, float gh, float prev, float* gv, int64_t ld_gv,
                                                    float* gr, int64_t ld_gr, int col, float gamma, float factor,
                                                    bool valid) {
        GaeBwdBody b;
        b.valid = valid;
        b.gh = gh;
        b.prev = prev;
        b.gamma = gamma;
        b.factor = factor;
        b.gv = gv + static_cast<int64_t>(t_edge) * ld_gv + col;
        b.gr = gr + static_cast<int64_t>(t_edge) * ld_gr + col;
        b.ld_gv = ld_gv;
        b.ld_gr = ld_gr;
        return b;
    }
    __device__ __forceinline__ void step(int /*t*/, const float (&x)[1], const float (&dt)[2]) {
        const BwdOut o = bwd_step(x[0], dt, gamma, factor, gh, prev);
        if (valid) {
            st_stream(gr, o.gr);
            st_stream(gv, o.gv);
        }
        gr += ld_gr;
        gv += ld_gv;
    }
};

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) gae_bwd_tma(const __grid_constant__ TmapPack<1> maps,
                                                        const float* __restrict__ dtab,
                                                        float* __restrict__ grad_value, int64_t ld_gv,
                                                        float* __restrict__ grad_reward, int64_t ld_gr, int T, int B,
                                                        float gamma, float factor, float* __restrict__ carry,
                                                        int write_last) {
    // carry (nullable): (2,B) = (ghat, dd of the previous row) of a T-chunked run; write_last: this launch ends at the
    // global row T-1, so row T of grad_value (= gamma*dd_{T-1}) is written as well
    using Pipe = ScanPipe<1, 0, 0, BT, TT, ST, 2>;
    const int col0 = blockIdx.x * BT;
    const int col = col0 + threadIdx.x;
    const bool valid = threadIdx.x < BT && col < B;
    GaeBwdBody body = GaeBwdBody::at(0, 0.f, 0.f, grad_value, ld_gv, grad_reward, ld_gr, col, gamma, factor, valid);
    if (carry != nullptr && valid) {  // after at(): loading it first reorders the machine code
        body.gh = carry[col];
        body.prev = carry[B + col];
    }
    Pipe::template run<false>(maps, {}, dtab, T, col0, body);
    if (body.valid && write_last) st_stream(body.gv, __fmul_rn(gamma, body.prev));  // row T
    if (carry != nullptr && body.valid) {
        carry[col] = body.gh;
        carry[B + col] = body.prev;
    }
}

// ---- variants with TMA-staged OUTPUT (NOUT > 0): same arithmetic, results leave as (TT x BT) bulk stores ----
struct GaeFwdBodyO {
    float g, v1, gamma, factor;
    __device__ __forceinline__ void step(int /*t*/, const float (&x)[2], const float (&dt)[2],
                                         const unsigned (&)[1], float (&o)[1]) {
        o[0] = fwd_step(x, dt, v1, gamma, factor, g);
        v1 = x[0];
    }
};

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) gae_fwd_tma_st(const __grid_constant__ TmapPack<2> maps,
                                                           const __grid_constant__ TmapPack<1> omaps,
                                                           const float* __restrict__ dtab,
                                                           const float* __restrict__ v_next,
                                                           float* __restrict__ carry, int T, int B, float gamma,
                                                           float factor) {
    using Pipe = ScanPipe<2, 0, 1, BT, TT, ST, 2>;
    const int col0 = blockIdx.x * BT;
    const int col = col0 + threadIdx.x;
    const bool valid = threadIdx.x < BT && col < B;
    GaeFwdBodyO body;
    body.g = (carry != nullptr && valid) ? carry[col] : 0.f;
    body.gamma = gamma;
    body.factor = factor;
    body.v1 = valid ? v_next[col] : 0.f;
    Pipe::template run<true>(maps, omaps, dtab, T, col0, body);
    if (carry != nullptr && valid) {
        carry[col] = body.g;
        carry[B + col] = body.v1;
    }
}

struct GaeBwdBodyO {
    float gh, prev, gamma, factor;
    __device__ __forceinline__ void step(int /*t*/, const float (&x)[1], const float (&dt)[2],
                                         const unsigned (&)[1], float (&o)[2]) {
        const BwdOut r = bwd_step(x[0], dt, gamma, factor, gh, prev);
        o[0] = r.gv;
        o[1] = r.gr;
    }
};

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) gae_bwd_tma_st(const __grid_constant__ TmapPack<1> maps,
                                                           const __grid_constant__ TmapPack<2> omaps,
                                                           const float* __restrict__ dtab,
                                                           float* __restrict__ grad_value, int64_t ld_gv, int T, int B,
                                                           float gamma, float factor, float* __restrict__ carry,
                                                           int write_last) {
    using Pipe = ScanPipe<1, 0, 2, BT, TT, ST, 2>;
    const int col0 = blockIdx.x * BT;
    const int col = col0 + threadIdx.x;
    const bool valid = threadIdx.x < BT && col < B;
    GaeBwdBodyO body;
    body.gh = (carry != nullptr && valid) ? carry[col] : 0.f;
    body.prev = (carry != nullptr && valid) ? carry[B + col] : 0.f;
    body.gamma = gamma;
    body.factor = factor;
    Pipe::template run<false>(maps, omaps, dtab, T, col0, body);
    // row T of grad_value is outside the output tensor map (T rows): one plain store per column
    if (valid && write_last) st_stream(grad_value + static_cast<int64_t>(T) * ld_gv + col, __fmul_rn(gamma, body.prev));
    if (carry != nullptr && valid) {
        carry[col] = body.gh;
        carry[B + col] = body.prev;
    }
}

// Generic (no alignment requirements) variants: the same bodies driven by scan_column (scan_pipe.cuh), one thread per
// column.  Used when a pointer / pitch is not 16-byte aligned so TMA cannot describe the tensor.
template <bool MOM>
__global__ void __launch_bounds__(128) gae_fwd_generic(const float* __restrict__ value, int64_t ld_value,
                                                        const float* __restrict__ reward, int64_t ld_reward,
                                                        const float* __restrict__ dtab, float* __restrict__ adv,
                                                        int64_t ld_adv, int T, int B, float gamma, float factor,
                                                        double* __restrict__ partials,
                                                        const float* __restrict__ v_next, float* __restrict__ carry) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = col < B;
    if (!MOM && !valid) return;
    GaeFwdBody<MOM> body = GaeFwdBody<MOM>::at(T, carry != nullptr && valid ? carry[col] : 0.f, v_next, adv,
                                               ld_adv, col, gamma, factor, valid);
    if (valid) {
        scan_column<2, 0, 0, 2, true>({{value, ld_value}, {reward, ld_reward}}, {}, dtab, {}, T, col, body);
        if (carry != nullptr) {
            carry[col] = body.g;
            carry[B + col] = body.v1;
        }
    }
    if constexpr (MOM) {
        __shared__ double red[64];
        gae_store_moments<MOM>(body, partials, red);
    }
}

__global__ void __launch_bounds__(128) gae_bwd_generic(const float* __restrict__ grad_adv, int64_t ld_ga,
                                                        const float* __restrict__ dtab,
                                                        float* __restrict__ grad_value, int64_t ld_gv,
                                                        float* __restrict__ grad_reward, int64_t ld_gr, int T, int B,
                                                        float gamma, float factor, float* __restrict__ carry,
                                                        int write_last) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= B) return;
    GaeBwdBody body = GaeBwdBody::at(0, carry != nullptr ? carry[col] : 0.f, carry != nullptr ? carry[B + col] : 0.f,
                                     grad_value, ld_gv, grad_reward, ld_gr, col, gamma, factor, true);
    scan_column<1, 0, 0, 2, false>({{grad_adv, ld_ga}}, {}, dtab, {}, T, col, body);
    if (write_last) *body.gv = __fmul_rn(gamma, body.prev);  // row T
    if (carry != nullptr) {
        carry[col] = body.gh;
        carry[B + col] = body.prev;
    }
}

// ------------------------------------------------------------------------------------------------
// Small-batch regime (few columns, long T: e.g. the reference's own test shape T=1024, B=64,
// tests/test_gae.py:10-11): single-launch T-split with look-back, scan_lookback.cuh.  One warp per
// (segment, 32-column tile); the GAE recurrences have the constant coefficient gamma*lambda, so a segment
// publishes only its zero-carry result and successors fold it with a^L.
// ------------------------------------------------------------------------------------------------
struct GaeFwdLbFac {
    const float* value;
    int64_t ldv;
    const float* dtab;
    float* adv;
    int64_t lda;
    int col;
    bool valid;
    float gamma, factor;
    using Body = GaeFwdBody<false>;
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {  // t_edge = row after the segment
        const bool store = valid && pass == 1;
        Body b = Body::at(t_edge, carry, value + static_cast<int64_t>(t_edge) * ldv, adv, lda, col, gamma, factor, valid);
        b.valid = store;
        return b;
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[2]) const {
        const float2 d = __ldg(reinterpret_cast<const float2*>(dtab) + t);
        const float dt[2] = {d.x, d.y};
        b.step(t, x, dt);
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.g; }
    static __device__ __forceinline__ float coef(const Body&) { return 0.f; }
    __device__ __forceinline__ void finish(Body&, int, int) const {}
};

__global__ void __launch_bounds__(kLbCols) gae_fwd_lookback(const float* __restrict__ value, int64_t ldv,
                                                            const float* __restrict__ reward, int64_t ldr,
                                                            const float* __restrict__ dtab, float* __restrict__ adv,
                                                            int64_t lda, int T, int B, float gamma, float factor,
                                                            float AL, int S, int L, int tiles, LbCtl* ctl,
                                                            unsigned long long* words) {
    __shared__ float smem[2 * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;  // the scan runs backward in time: the last segment goes first
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const GaeFwdLbFac fac{value, ldv, dtab, adv, lda, col, col < B, gamma, factor};
    const float* const in[2] = {value, reward};
    const int64_t ld[2] = {ldv, ldr};
    lb_segment<2, true, true>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, AL, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

struct GaeBwdLbFac {
    const float* dtab;
    float* gv;
    int64_t ldgv;
    float* gr;
    int64_t ldgr;
    int col, T;
    bool valid;
    float gamma, factor;
    using Body = GaeBwdBody;
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {  // t_edge = first row of the segment
        // dd of the previous row, exactly as the serial scan forms it: d_{t-1} * ghat_{t-1}
        const float prev = t_edge > 0 ? __fmul_rn(__ldg(dtab + 2 * (t_edge - 1)), carry) : 0.f;
        return Body::at(t_edge, carry, prev, gv, ldgv, gr, ldgr, col, gamma, factor, valid && pass == 1);
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[1]) const {
        const float2 d = __ldg(reinterpret_cast<const float2*>(dtab) + t);
        const float dt[2] = {d.x, d.y};
        b.step(t, x, dt);
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.gh; }
    static __device__ __forceinline__ float coef(const Body&) { return 0.f; }
    __device__ __forceinline__ void finish(Body& b, int, int t1) const {
        if (t1 == T && valid) st_stream(b.gv, __fmul_rn(gamma, b.prev));  // row T
    }
};

__global__ void __launch_bounds__(kLbCols) gae_bwd_lookback(const float* __restrict__ grad_adv, int64_t ldg,
                                                            const float* __restrict__ dtab, float* __restrict__ gv,
                                                            int64_t ldgv, float* __restrict__ gr, int64_t ldgr, int T,
                                                            int B, float gamma, float factor, float AL, int S, int L,
                                                            int tiles, LbCtl* ctl, unsigned long long* words) {
    __shared__ float smem[kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int t0 = lt.k * L, t1 = min(T, t0 + L);  // forward in time
    const int col = lt.tile * kLbCols + threadIdx.x;
    const GaeBwdLbFac fac{dtab, gv, ldgv, gr, ldgr, col, T, col < B, gamma, factor};
    const float* const in[1] = {grad_adv};
    const int64_t ld[1] = {ldg};
    lb_segment<1, false, true>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, AL, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------

template <int BT, int TT, int ST, bool MOM = false>
static int launch_fwd_tma(const float* value, int64_t ldv, const float* reward, int64_t ldr, const float* dtab,
                          float* adv, int64_t lda, int64_t T, int64_t B, float gamma, float factor,
                          cudaStream_t stream, double* partials = nullptr, int* nblocks = nullptr,
                          const float* v_next = nullptr, float* carry = nullptr) {
    TmapPack<2> maps;
    int rc = make_tmap_2d(&maps.m[0], value, T + 1, B, ldv, TT, BT);
    if (rc) return rc;
    rc = make_tmap_2d(&maps.m[1], reward, T, B, ldr, TT, BT);
    if (rc) return rc;
    const unsigned grid = static_cast<unsigned>((B + BT - 1) / BT);
    if (nblocks) *nblocks = static_cast<int>(grid);
    if (v_next == nullptr) v_next = value + T * ldv;
    return launch_scan<ScanPipe<2, 0, 0, BT, TT, ST, 2>, gae_fwd_tma<BT, TT, ST, MOM>>(
        grid, stream, maps, dtab, v_next, carry, adv, lda, static_cast<int>(T), static_cast<int>(B), gamma, factor,
        partials);
}

template <int BT, int TT, int ST>
static int launch_bwd_tma(const float* grad_adv, int64_t ldg, const float* dtab, float* gv, int64_t ldgv, float* gr,
                          int64_t ldgr, int64_t T, int64_t B, float gamma, float factor, cudaStream_t stream,
                          float* carry = nullptr, int write_last = 1) {
    TmapPack<1> maps;
    int rc = make_tmap_2d(&maps.m[0], grad_adv, T, B, ldg, TT, BT);
    if (rc) return rc;
    const unsigned grid = static_cast<unsigned>((B + BT - 1) / BT);
    return launch_scan<ScanPipe<1, 0, 0, BT, TT, ST, 2>, gae_bwd_tma<BT, TT, ST>>(
        grid, stream, maps, dtab, gv, ldgv, gr, ldgr, static_cast<int>(T), static_cast<int>(B), gamma, factor, carry,
        write_last);
}

template <int BT, int TT, int ST>
static int launch_fwd_tma_st(const float* value, int64_t ldv, const float* reward, int64_t ldr, const float* dtab,
                             float* adv, int64_t lda, int64_t T, int64_t B, float gamma, float factor,
                             cudaStream_t stream, const float* v_next = nullptr, float* carry = nullptr) {
    TmapPack<2> maps;
    TmapPack<1> omaps;
    int rc = make_tmap_2d(&maps.m[0], value, T + 1, B, ldv, TT, BT);
    if (rc) return rc;
    rc = make_tmap_2d(&maps.m[1], reward, T, B, ldr, TT, BT);
    if (rc) return rc;
    rc = make_tmap_2d(&omaps.m[0], adv, T, B, lda, TT, BT);
    if (rc) return rc;
    const unsigned grid = static_cast<unsigned>((B + BT - 1) / BT);
    if (v_next == nullptr) v_next = value + T * ldv;
    return launch_scan<ScanPipe<2, 0, 1, BT, TT, ST, 2>, gae_fwd_tma_st<BT, TT, ST>>(
        grid, stream, maps, omaps, dtab, v_next, carry, static_cast<int>(T), static_cast<int>(B), gamma, factor);
}

template <int BT, int TT, int ST>
static int launch_bwd_tma_st(const float* grad_adv, int64_t ldg, const float* dtab, float* gv, int64_t ldgv, float* gr,
                             int64_t ldgr, int64_t T, int64_t B, float gamma, float factor, cudaStream_t stream,
                             float* carry = nullptr, int write_last = 1) {
    TmapPack<1> maps;
    TmapPack<2> omaps;
    int rc = make_tmap_2d(&maps.m[0], grad_adv, T, B, ldg, TT, BT);
    if (rc) return rc;
    rc = make_tmap_2d(&omaps.m[0], gv, T, B, ldgv, TT, BT);  // rows 0..T-1; row T is written by the kernel tail
    if (rc) return rc;
    rc = make_tmap_2d(&omaps.m[1], gr, T, B, ldgr, TT, BT);
    if (rc) return rc;
    const unsigned grid = static_cast<unsigned>((B + BT - 1) / BT);
    return launch_scan<ScanPipe<1, 0, 2, BT, TT, ST, 2>, gae_bwd_tma_st<BT, TT, ST>>(
        grid, stream, maps, omaps, dtab, gv, ldgv, static_cast<int>(T), static_cast<int>(B), gamma, factor, carry,
        write_last);
}

// Kernel regimes; hpc_rll_debug_set_config(HPC_RLL_OP_GAE, id) forces one, -1 picks by B.  <BT,TT,ST> = columns per
// CTA, rows per TMA box, ring stages (a TMA box dimension is limited to 256 elements, so BT <= 256).
//   33 wide (B >= 256*SMs, all operands TMA-describable): fwd gae_fwd_tma_st<256,4,5>, bwd gae_bwd_tma_st<256,4,6>
//    7 wide, an output not TMA-describable:               gae_fwd_tma / gae_bwd_tma <256,8,4>
//    5 mid (32*SMs <= B < 256*SMs):                        gae_fwd_tma / gae_bwd_tma <64,8,6>
//   13 narrow (B < 32*SMs):                                gae_fwd_tma / gae_bwd_tma <32,64,6>
//   21 single-launch T-split with look-back (automatic for B <= 2048, T >= 512; see lookback_geometry)
//   99 generic (non-TMA) kernels, used when an input is not TMA-describable
// gae_forward_moments runs gae_fwd_tma<...,true> with <256,8,4> (33, 7), <64,16,3> (5), <32,64,6> (13).
static int pick_cfg(int64_t B) {
    const int forced = tuning_config(HPC_RLL_OP_GAE);
    if (forced >= 0) return forced;
    const int64_t sms = sm_count();
    // tools/tune_gae.py on H100 at T=1024, B=65536 (median of 20 single calls): the bulk-store output kernels with
    // shallow boxes give the fastest backward (0.295 ms against 0.300-0.31 for per-thread stores) and a forward within
    // 1 % of the fastest
    if (B >= 256 * sms) return 33;
    // mid-size batches, same sweep at B = 8192 ... 32768: <64,8,6> (a deep row pipeline on narrow tiles) is the
    // fastest or within 5 % of it everywhere, fwd+bwd 0.091 ms at B=8192 against 0.113 for <32,32,3> and 0.229 ms at
    // B=24576 against 0.238 for <128,16,3>
    if (B >= 32 * sms) return 5;
    return 13;  // few column tiles: deeper row pipeline per CTA
}

// One launch of the forward scan over `T` consecutive rows.  A whole problem has chunk == nullptr; a T-chunk of a
// longer trajectory (rows [t0, t0+T) of T_total) passes its carry: (2,B) floats = g_{t0+T} and value row t0+T on
// entry, g_{t0} and value row t0 on exit (chunks are processed from the LAST one to the first).
struct GaeChunk {
    int64_t T_total;
    int64_t t0;
    float* carry;
};

static int gae_forward_impl(const float* value, int64_t ldv, const float* reward, int64_t ldr, float* adv,
                            int64_t lda, int64_t T, int64_t B, double gamma, double lambda, cudaStream_t stream,
                            const GaeChunk* chunk = nullptr) {
    HPC_REQUIRE(T >= 0 && B >= 0, "gae_forward: negative size T=%lld B=%lld", (long long)T, (long long)B);
    if (T == 0 || B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(value && reward && adv, "gae_forward: null pointer");
    HPC_REQUIRE(ldv >= B && ldr >= B && lda >= B, "gae_forward: row pitch smaller than B");
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512, "gae_forward: T/B exceed 2^31");
    const float* dtab = nullptr;
    int rc = get_dtab(chunk ? chunk->T_total : T, lambda, stream, &dtab);
    if (rc) return rc;
    float* carry = chunk ? chunk->carry : nullptr;
    const float* v_next = chunk ? chunk->carry + B : value + T * ldv;
    if (chunk) dtab += 2 * chunk->t0;
    const float g = static_cast<float>(gamma), f = static_cast<float>(gamma * lambda);
    LbGeom lg;
    if (!chunk && lookback_geometry(HPC_RLL_OP_GAE, T, B, &lg)) {  // small batch: single-launch T-split
        LbScratch sc;
        rc = lookback_scratch(lg, B, stream, &sc);
        if (rc) return rc;
        const float AL = static_cast<float>(std::pow(gamma * lambda, static_cast<double>(lg.L)));
        gae_fwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            value, ldv, reward, ldr, dtab, adv, lda, static_cast<int>(T), static_cast<int>(B), g, f, AL, lg.S, lg.L,
            lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
    int cfg = pick_cfg(B);
    if (cfg == 21) cfg = 13;
    // the d_t slice of a stage is a 16-byte-aligned bulk copy: a chunk must start on an even row
    const bool tma = tma_ok_2d(value, B, ldv) && tma_ok_2d(reward, B, ldr) && aligned16(dtab);
    if (!tma) cfg = 99;
    if (cfg == 33 && !tma_ok_2d(adv, B, lda)) cfg = 7;  // output not TMA-describable: per-thread stores
#define HPC_FWD(BT_, TT_, ST_) \
    return launch_fwd_tma<BT_, TT_, ST_>(value, ldv, reward, ldr, dtab, adv, lda, T, B, g, f, stream, nullptr, nullptr, \
                                         v_next, carry)
    switch (cfg) {
        case 5: HPC_FWD(64, 8, 6);
        case 7: HPC_FWD(256, 8, 4);
        case 13: HPC_FWD(32, 64, 6);
        case 33:
            return launch_fwd_tma_st<256, 4, 5>(value, ldv, reward, ldr, dtab, adv, lda, T, B, g, f, stream, v_next, carry);
        default: break;
    }
#undef HPC_FWD
    const unsigned grid = static_cast<unsigned>((B + 127) / 128);
    gae_fwd_generic<false><<<grid, 128, 0, stream>>>(value, ldv, reward, ldr, dtab, adv, lda, static_cast<int>(T),
                                                     static_cast<int>(B), g, f, nullptr, v_next, carry);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

// sum / sum-of-squares of the per-CTA partials, fixed order -> moments[0..1] (fp64)
__global__ void __launch_bounds__(256) gae_finalize_moments(const double* __restrict__ partials, int n,
                                                             double* __restrict__ moments) {
    __shared__ double scratch[64];
    double v[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += 256) {
        v[0] += partials[i];
        v[1] += partials[n + i];
    }
    block_sum<2>(v, scratch);
    if (threadIdx.x == 0) {
        moments[0] = v[0];
        moments[1] = v[1];
    }
}

// stats[0] = mean, stats[1] = unbiased std + 1e-8 (fp32 add, as `adv.std() + 1e-8` on an fp32 tensor)
__global__ void adv_stats_kernel(const double* __restrict__ moments, double count, float* __restrict__ stats) {
    const double s1 = moments[0], s2 = moments[1];
    if (count <= 0.0) count = moments[2];  // count carried (and all-reduced) next to the sums
    const double mean = s1 / count;
    const double var = (s2 - s1 * mean) / (count - 1.0);  // count == 1 -> NaN like torch.std
    const float sd = static_cast<float>(sqrt(var > 0.0 ? var : (var == var ? 0.0 : var)));
    stats[0] = static_cast<float>(mean);
    stats[1] = __fadd_rn(sd, 1e-8f);
}

size_t gae_moments_workspace_bytes(int64_t B) { return 2 * sizeof(double) * static_cast<size_t>((B + 31) / 32 + 8); }

static int gae_forward_moments_impl(const float* value, const float* reward, float* adv, double* moments, int64_t T,
                                    int64_t B, double gamma, double lambda, double* partials, cudaStream_t stream) {
    const float* dtab = nullptr;
    int rc = get_dtab(T, lambda, stream, &dtab);
    if (rc) return rc;
    const float g = static_cast<float>(gamma), f = static_cast<float>(gamma * lambda);
    int cfg = pick_cfg(B);
    if (!(tma_ok_2d(value, B, B) && tma_ok_2d(reward, B, B))) cfg = 99;
    int nblocks = 0;
    switch (cfg) {
        case 7: case 33:
            rc = launch_fwd_tma<256, 8, 4, true>(value, B, reward, B, dtab, adv, B, T, B, g, f, stream, partials, &nblocks);
            break;
        case 5:
            rc = launch_fwd_tma<64, 16, 3, true>(value, B, reward, B, dtab, adv, B, T, B, g, f, stream, partials, &nblocks);
            break;
        case 13:
            rc = launch_fwd_tma<32, 64, 6, true>(value, B, reward, B, dtab, adv, B, T, B, g, f, stream, partials, &nblocks);
            break;
        default: {
            const unsigned grid = static_cast<unsigned>((B + 127) / 128);
            nblocks = static_cast<int>(grid);
            gae_fwd_generic<true><<<grid, 128, 0, stream>>>(value, B, reward, B, dtab, adv, B, static_cast<int>(T),
                                                            static_cast<int>(B), g, f, partials, value + T * B, nullptr);
            count_launch();
            HPC_LAUNCH_CHECK();
        }
    }
    if (rc) return rc;
    gae_finalize_moments<<<1, 256, 0, stream>>>(partials, nblocks, moments);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

// Backward scan over `T` consecutive rows; chunk as above with carry = (ghat, dd of the previous row), chunks processed
// from the FIRST one to the last.  Row T_total of grad_value is written by the launch that ends at the last row.
static int gae_backward_impl(const float* grad_adv, int64_t ldg, float* gv, int64_t ldgv, float* gr, int64_t ldgr,
                             int64_t T, int64_t B, double gamma, double lambda, cudaStream_t stream,
                             const GaeChunk* chunk = nullptr) {
    HPC_REQUIRE(T >= 0 && B >= 0, "gae_backward: negative size T=%lld B=%lld", (long long)T, (long long)B);
    if (B == 0) return HPC_RLL_OK;
    HPC_REQUIRE(gv != nullptr, "gae_backward: null grad_value");
    if (T == 0) {  // value is (1,B): no advantage depends on it
        if (!chunk) HPC_CUDA(cudaMemsetAsync(gv, 0, sizeof(float) * static_cast<size_t>(B), stream));
        return HPC_RLL_OK;
    }
    HPC_REQUIRE(grad_adv && gr, "gae_backward: null pointer");
    HPC_REQUIRE(ldg >= B && ldgv >= B && ldgr >= B, "gae_backward: row pitch smaller than B");
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512, "gae_backward: T/B exceed 2^31");
    const float* dtab = nullptr;
    int rc = get_dtab(chunk ? chunk->T_total : T, lambda, stream, &dtab);
    if (rc) return rc;
    float* carry = chunk ? chunk->carry : nullptr;
    const int write_last = (!chunk || chunk->t0 + T == chunk->T_total) ? 1 : 0;
    if (chunk) dtab += 2 * chunk->t0;
    const float g = static_cast<float>(gamma), f = static_cast<float>(gamma * lambda);
    LbGeom lg;
    if (!chunk && lookback_geometry(HPC_RLL_OP_GAE, T, B, &lg)) {
        LbScratch sc;
        rc = lookback_scratch(lg, B, stream, &sc);
        if (rc) return rc;
        const float AL = static_cast<float>(std::pow(gamma * lambda, static_cast<double>(lg.L)));
        gae_bwd_lookback<<<static_cast<unsigned>(lg.S * lg.tiles), kLbCols, 0, stream>>>(
            grad_adv, ldg, dtab, gv, ldgv, gr, ldgr, static_cast<int>(T), static_cast<int>(B), g, f, AL, lg.S, lg.L,
            lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
        return HPC_RLL_OK;
    }
    int cfg = pick_cfg(B);
    if (cfg == 21) cfg = 13;
    if (!(tma_ok_2d(grad_adv, B, ldg) && aligned16(dtab))) cfg = 99;
    if (cfg == 33 && !(tma_ok_2d(gv, B, ldgv) && tma_ok_2d(gr, B, ldgr))) cfg = 7;
#define HPC_BWD(BT_, TT_, ST_) \
    return launch_bwd_tma<BT_, TT_, ST_>(grad_adv, ldg, dtab, gv, ldgv, gr, ldgr, T, B, g, f, stream, carry, write_last)
    switch (cfg) {
        case 5: HPC_BWD(64, 8, 6);
        case 7: HPC_BWD(256, 8, 4);
        case 13: HPC_BWD(32, 64, 6);
        case 33:
            return launch_bwd_tma_st<256, 4, 6>(grad_adv, ldg, dtab, gv, ldgv, gr, ldgr, T, B, g, f, stream, carry,
                                                write_last);
        default: break;
    }
#undef HPC_BWD
    const unsigned grid = static_cast<unsigned>((B + 127) / 128);
    gae_bwd_generic<<<grid, 128, 0, stream>>>(grad_adv, ldg, dtab, gv, ldgv, gr, ldgr, static_cast<int>(T),
                                              static_cast<int>(B), g, f, carry, write_last);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

// ------------------------------------------------------------------------------------------------
// host-buffer end-to-end path: T-CHUNKED carry pipeline (round 2; replaces the column-block pipeline)
//
// The scan state between two row ranges is two floats per column, so a (T,B) problem whose operands live in host
// memory is streamed as contiguous ROW RANGES: every copy is one 1-D DMA of rows*B*4 bytes (full 256 KB rows at
// B=65536) in both directions, and every kernel launch is full width (the TMA-store kernels of the resident
// path).  Forward walks the chunks from the last to the first (carry g, v), backward from the first to the
// last (carry ghat, dd); stage i handles forward chunk nC-1-i and backward chunk i, so the host->device engine
// streams value/reward/grad_adv rows while the device->host engine drains adv/grad_value/grad_reward rows of
// earlier stages.  Three streams (H2D, compute, D2H) + per-slot events; kSlots stages in flight.
// ------------------------------------------------------------------------------------------------
namespace {
struct HostPipe {
    static constexpr int kSlots = 4;
    int dev = -1;
    bool busy = false;
    cudaStream_t s_h2d = nullptr, s_k = nullptr, s_d2h = nullptr;
    cudaEvent_t ev_h[kSlots] = {}, ev_k[kSlots] = {}, ev_d[kSlots] = {};
    cudaEvent_t done = nullptr;
    float* buf = nullptr;
    size_t cap = 0;  // floats
};
std::mutex g_hp_mu;
std::vector<HostPipe*> g_hp_pool;

// every concurrent host-entry caller gets its own pipe (streams, events, staging memory); pipes are pooled per device
struct HostPipeLease {
    HostPipe* p = nullptr;
    ~HostPipeLease() {
        if (p) {
            std::lock_guard<std::mutex> lk(g_hp_mu);
            p->busy = false;
        }
    }
};

int host_pipe_acquire(int dev, size_t floats, HostPipeLease* lease) {
    HostPipe* hp = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_hp_mu);
        for (HostPipe* c : g_hp_pool)
            if (!c->busy && c->dev == dev) {
                hp = c;
                break;
            }
        if (!hp) {
            hp = new HostPipe();
            hp->dev = dev;
            g_hp_pool.push_back(hp);
        }
        hp->busy = true;
    }
    lease->p = hp;
    if (!hp->s_h2d) {
        HPC_CUDA(cudaStreamCreateWithFlags(&hp->s_h2d, cudaStreamNonBlocking));
        HPC_CUDA(cudaStreamCreateWithFlags(&hp->s_k, cudaStreamNonBlocking));
        HPC_CUDA(cudaStreamCreateWithFlags(&hp->s_d2h, cudaStreamNonBlocking));
        for (int i = 0; i < HostPipe::kSlots; ++i) {
            HPC_CUDA(cudaEventCreateWithFlags(&hp->ev_h[i], cudaEventDisableTiming));
            HPC_CUDA(cudaEventCreateWithFlags(&hp->ev_k[i], cudaEventDisableTiming));
            HPC_CUDA(cudaEventCreateWithFlags(&hp->ev_d[i], cudaEventDisableTiming));
        }
        // the final wait sleeps instead of spinning: with one rank per GPU the host cores are shared
        HPC_CUDA(cudaEventCreateWithFlags(&hp->done, cudaEventDisableTiming | cudaEventBlockingSync));
    }
    if (hp->cap < floats) {
        if (hp->buf) {
            HPC_CUDA(cudaStreamSynchronize(hp->s_d2h));
            cudaFree(hp->buf);
            hp->buf = nullptr;
            hp->cap = 0;
        }
        HPC_CUDA(cudaMalloc(&hp->buf, floats * sizeof(float)));
        hp->cap = floats;
    }
    return HPC_RLL_OK;
}

// Stage heights of the T-chunked pipeline.  In duplex the two copy engines run concurrently, every copy costs some
// microseconds of set-up, and the first stage's H2D plus the last stage's D2H overlap with nothing.  Stages are uniform,
// 16 MB per tensor (64 rows at B=65536: 16 stages), the best of {2..64 MB} when the pipeline was tuned; ramped heights
// (short first / last stages) were slower: the D2H engine falls behind during the tall middle stages and drains alone
// at the end.  On H100 this schedule runs at 94-95 % of the duplex copy rate measured alongside it (bench.py e2e).
// The generator still takes
// "r0:rmax" for experiments (HPC_RLL_HOST_CHUNK_ROWS); one number = uniform.  Rows are multiples of 4 (whole TMA
// boxes, 16-byte aligned d_t slices); T % 4 extra rows ride in the stage that touches row T.  The list is a
// palindrome: the backward walks it from row 0 up, the forward from row T down.
std::vector<int64_t> host_schedule(int64_t T, int64_t B) {
    static const std::pair<long long, long long> forced = [] {
        const char* e = getenv("HPC_RLL_HOST_CHUNK_ROWS");
        if (!e) return std::make_pair(0LL, 0LL);
        const long long a = atoll(e);
        const char* c = strchr(e, ':');
        return std::make_pair(a, c ? atoll(c + 1) : a);
    }();
    const int64_t row_bytes = 4 * (B > 0 ? B : 1);
    auto round4 = [](int64_t r) { return r < 4 ? int64_t(4) : (r / 4) * 4; };
    int64_t r0 = round4(forced.first >= 4 ? forced.first : (int64_t(16) << 20) / row_bytes);
    int64_t rmax = round4(forced.second >= 4 ? forced.second : r0);
    if (rmax < r0) rmax = r0;
    const int64_t T4 = (T / 4) * 4, rem = T - T4;
    std::vector<int64_t> sizes;
    if (T4 < 2 * r0) {
        sizes.push_back(T);
        return sizes;
    }
    std::vector<int64_t> up;  // r0, r0, 2 r0, 4 r0, ... while both ramps still fit
    int64_t used = 0;
    for (int64_t r = r0, k = 0; r <= rmax; ++k) {
        if (2 * (used + r) > T4) break;
        up.push_back(r);
        used += r;
        if (k >= 1) r *= 2;
    }
    int64_t middle = T4 - 2 * used;
    const int64_t top = up.empty() ? r0 : up.back();
    sizes = up;
    while (middle >= 2 * top) {
        sizes.push_back(top);
        middle -= top;
    }
    if (middle > 0) sizes.push_back(middle);  // multiple of 4 by construction
    for (size_t i = up.size(); i-- > 0;) sizes.push_back(up[i]);
    sizes.back() += rem;  // the stage that ends at row T (backward order); the forward sees it first
    return sizes;
}
}  // namespace

static int gae_host_impl(const float* h_value, const float* h_reward, const float* h_gadv, float* h_adv,
                         float* h_gvalue, float* h_greward, int64_t T, int64_t B, double gamma, double lambda) {
    HPC_REQUIRE(T > 0 && B > 0, "gae_fwd_bwd_host: T and B must be positive");
    HPC_REQUIRE(h_value && h_reward && h_adv, "gae_fwd_bwd_host: null forward buffer");
    const bool bwd = h_gadv != nullptr;
    HPC_REQUIRE(!bwd || (h_gvalue && h_greward), "gae_fwd_bwd_host: backward needs grad_value and grad_reward");
    int dev = 0;
    HPC_CUDA(cudaGetDevice(&dev));
    // stage heights; backward stage i = rows [off[i], off[i+1]) ascending, forward stage i = the mirrored range
    const std::vector<int64_t> sizes = host_schedule(T, B);
    const int64_t nC = static_cast<int64_t>(sizes.size());
    std::vector<int64_t> off(nC + 1, 0);
    int64_t R = 0;
    for (int64_t i = 0; i < nC; ++i) {
        off[i + 1] = off[i] + sizes[i];
        if (sizes[i] > R) R = sizes[i];
    }
    const size_t Bs = static_cast<size_t>(B);
    const size_t chunk = static_cast<size_t>(R) * Bs;           // floats per staged tensor
    const size_t slot = 6 * chunk + Bs;                          // + row T of grad_value in the last backward chunk
    HostPipeLease lease;
    int rc = host_pipe_acquire(dev, HostPipe::kSlots * slot + 4 * Bs, &lease);
    if (rc) return rc;
    HostPipe& hp = *lease.p;
    float* carry_f = hp.buf + HostPipe::kSlots * slot;  // (2,B): g, value row
    float* carry_b = carry_f + 2 * Bs;                  // (2,B): ghat, dd
    // initial scan state: g = 0, v_next = value[T]; ghat = dd = 0
    HPC_CUDA(cudaMemsetAsync(carry_f, 0, Bs * sizeof(float), hp.s_h2d));
    HPC_CUDA(cudaMemcpyAsync(carry_f + Bs, h_value + static_cast<size_t>(T) * Bs, Bs * sizeof(float),
                             cudaMemcpyHostToDevice, hp.s_h2d));
    HPC_CUDA(cudaMemsetAsync(carry_b, 0, 2 * Bs * sizeof(float), hp.s_h2d));
    // HPC_RLL_HOST_TRACE=1: per-stage timeline (ms since the first copy) on stderr -- a diagnosis aid, off by default
    static const bool trace = [] {
        const char* e = getenv("HPC_RLL_HOST_TRACE");
        return e && atoi(e) != 0;
    }();
    static const int debug_skip = [] {  // bit0: no kernels, bit1: no D2H, bit2: no H2D (timing experiments only)
        const char* e = getenv("HPC_RLL_HOST_DEBUG_SKIP");
        return e ? atoi(e) : 0;
    }();
    std::vector<cudaEvent_t> tev;
    if (trace) {
        tev.resize(static_cast<size_t>(nC) * 4 + 1);
        for (auto& e : tev) HPC_CUDA(cudaEventCreate(&e));
        HPC_CUDA(cudaEventRecord(tev[nC * 4], hp.s_h2d));
    }
    for (int64_t i = 0; i < nC; ++i) {
        const int s = static_cast<int>(i % HostPipe::kSlots);
        float* d_value = hp.buf + s * slot;
        float* d_reward = d_value + chunk;
        float* d_adv = d_reward + chunk;
        float* d_gadv = d_adv + chunk;
        float* d_greward = d_gadv + chunk;
        float* d_gvalue = d_greward + chunk;  // last: may hold one extra row
        // the palindrome read from the other end: forward stage i covers the rows the backward covers in stage nC-1-i
        const int64_t f0 = off[nC - 1 - i], frows = sizes[nC - 1 - i];
        const int64_t b0 = off[i], brows = sizes[i];
        const size_t fbytes = static_cast<size_t>(frows) * Bs * sizeof(float);
        const size_t bbytes = static_cast<size_t>(brows) * Bs * sizeof(float);
        // ---- host -> device (waits until the kernels of the stage that used this slot before have read it)
        if (i >= HostPipe::kSlots) HPC_CUDA(cudaStreamWaitEvent(hp.s_h2d, hp.ev_k[s], 0));
        if (trace) HPC_CUDA(cudaEventRecord(tev[i * 4 + 0], hp.s_h2d));
        if (!(debug_skip & 4)) {
        HPC_CUDA(cudaMemcpyAsync(d_value, h_value + static_cast<size_t>(f0) * Bs, fbytes, cudaMemcpyHostToDevice, hp.s_h2d));
        HPC_CUDA(cudaMemcpyAsync(d_reward, h_reward + static_cast<size_t>(f0) * Bs, fbytes, cudaMemcpyHostToDevice, hp.s_h2d));
        if (bwd)
            HPC_CUDA(cudaMemcpyAsync(d_gadv, h_gadv + static_cast<size_t>(b0) * Bs, bbytes, cudaMemcpyHostToDevice, hp.s_h2d));
        }
        HPC_CUDA(cudaEventRecord(hp.ev_h[s], hp.s_h2d));
        if (trace) HPC_CUDA(cudaEventRecord(tev[i * 4 + 1], hp.s_h2d));
        // ---- kernels (wait for the inputs, and for the D2H copies that drained this slot's outputs)
        HPC_CUDA(cudaStreamWaitEvent(hp.s_k, hp.ev_h[s], 0));
        if (i >= HostPipe::kSlots) HPC_CUDA(cudaStreamWaitEvent(hp.s_k, hp.ev_d[s], 0));
        GaeChunk cf{T, f0, carry_f};
        if (!(debug_skip & 1)) {
        rc = gae_forward_impl(d_value, B, d_reward, B, d_adv, B, frows, B, gamma, lambda, hp.s_k, &cf);
        if (rc) return rc;
        if (bwd) {
            GaeChunk cb{T, b0, carry_b};
            rc = gae_backward_impl(d_gadv, B, d_gvalue, B, d_greward, B, brows, B, gamma, lambda, hp.s_k, &cb);
            if (rc) return rc;
        }
        }
        HPC_CUDA(cudaEventRecord(hp.ev_k[s], hp.s_k));
        if (trace) HPC_CUDA(cudaEventRecord(tev[i * 4 + 2], hp.s_k));
        // ---- device -> host
        HPC_CUDA(cudaStreamWaitEvent(hp.s_d2h, hp.ev_k[s], 0));
        if (!(debug_skip & 2))
        HPC_CUDA(cudaMemcpyAsync(h_adv + static_cast<size_t>(f0) * Bs, d_adv, fbytes, cudaMemcpyDeviceToHost, hp.s_d2h));
        if (bwd && !(debug_skip & 2)) {
            const size_t gvbytes = bbytes + (b0 + brows == T ? Bs * sizeof(float) : 0);  // + row T at the end
            HPC_CUDA(cudaMemcpyAsync(h_gvalue + static_cast<size_t>(b0) * Bs, d_gvalue, gvbytes, cudaMemcpyDeviceToHost, hp.s_d2h));
            HPC_CUDA(cudaMemcpyAsync(h_greward + static_cast<size_t>(b0) * Bs, d_greward, bbytes, cudaMemcpyDeviceToHost, hp.s_d2h));
        }
        HPC_CUDA(cudaEventRecord(hp.ev_d[s], hp.s_d2h));
        if (trace) HPC_CUDA(cudaEventRecord(tev[i * 4 + 3], hp.s_d2h));
    }
    HPC_CUDA(cudaEventRecord(hp.done, hp.s_d2h));
    HPC_CUDA(cudaEventSynchronize(hp.done));
    if (trace) {
        fprintf(stderr, "stage rows  h2d_begin  h2d_end  kernels_end  d2h_end   (ms)\n");
        for (int64_t i = 0; i < nC; ++i) {
            float t[4];
            for (int k = 0; k < 4; ++k) cudaEventElapsedTime(&t[k], tev[nC * 4], tev[i * 4 + k]);
            fprintf(stderr, "%5lld %4lld  %8.3f %8.3f %8.3f %8.3f\n", (long long)i, (long long)sizes[i], t[0], t[1], t[2], t[3]);
        }
        for (auto& e : tev) cudaEventDestroy(e);
    }
    return HPC_RLL_OK;
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_gae_forward(const float* value, const float* reward, float* adv, int64_t T, int64_t B, double gamma,
                        double lambda, void* stream) {
    HPC_NVTX("gae_forward");
    return hpcrll::gae_forward_impl(value, B, reward, B, adv, B, T, B, gamma, lambda, hpcrll::as_stream(stream));
}

int hpc_rll_gae_forward_moments(const float* value, const float* reward, float* adv, double* moments, int64_t T,
                                int64_t B, double gamma, double lambda, void* workspace, size_t workspace_bytes,
                                void* stream) {
    HPC_NVTX("gae_forward_moments");
    using namespace hpcrll;
    HPC_REQUIRE(T > 0 && B > 0, "gae_forward_moments: T and B must be positive (T=%lld B=%lld)", (long long)T,
                (long long)B);
    HPC_REQUIRE(value && reward && adv && moments && workspace, "gae_forward_moments: null pointer");
    HPC_REQUIRE(workspace_bytes >= gae_moments_workspace_bytes(B), "gae_forward_moments: workspace too small");
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512, "gae_forward_moments: T/B exceed 2^31");
    return gae_forward_moments_impl(value, reward, adv, moments, T, B, gamma, lambda, static_cast<double*>(workspace),
                                    as_stream(stream));
}

int hpc_rll_adv_stats(const double* moments, int64_t count, float* stats, void* stream) {
    HPC_NVTX("adv_stats");
    using namespace hpcrll;
    HPC_REQUIRE(moments && stats, "adv_stats: null pointer");
    adv_stats_kernel<<<1, 1, 0, as_stream(stream)>>>(moments, static_cast<double>(count), stats);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

int hpc_rll_gae_backward(const float* grad_adv, float* grad_value, float* grad_reward, int64_t T, int64_t B,
                         double gamma, double lambda, void* stream) {
    HPC_NVTX("gae_backward");
    return hpcrll::gae_backward_impl(grad_adv, B, grad_value, B, grad_reward, B, T, B, gamma, lambda,
                                     hpcrll::as_stream(stream));
}

int hpc_rll_gae_forward_ld(const float* value, int64_t ld_value, const float* reward, int64_t ld_reward,
                           float* adv, int64_t ld_adv, int64_t T, int64_t B, double gamma, double lambda,
                           void* stream) {
    HPC_NVTX("gae_forward_ld");
    return hpcrll::gae_forward_impl(value, ld_value, reward, ld_reward, adv, ld_adv, T, B, gamma, lambda,
                                    hpcrll::as_stream(stream));
}

int hpc_rll_gae_backward_ld(const float* grad_adv, int64_t ld_grad_adv, float* grad_value, int64_t ld_grad_value,
                            float* grad_reward, int64_t ld_grad_reward, int64_t T, int64_t B, double gamma,
                            double lambda, void* stream) {
    HPC_NVTX("gae_backward_ld");
    return hpcrll::gae_backward_impl(grad_adv, ld_grad_adv, grad_value, ld_grad_value, grad_reward, ld_grad_reward,
                                     T, B, gamma, lambda, hpcrll::as_stream(stream));
}

int hpc_rll_gae_forward_chunk(const float* value, const float* reward, float* adv, float* carry, int64_t T_total,
                              int64_t t0, int64_t rows, int64_t B, double gamma, double lambda, void* stream) {
    HPC_NVTX("gae_forward_chunk");
    using namespace hpcrll;
    HPC_REQUIRE(carry != nullptr, "gae_forward_chunk: null carry");
    HPC_REQUIRE(t0 >= 0 && rows >= 0 && t0 + rows <= T_total, "gae_forward_chunk: rows [%lld, %lld) outside T=%lld",
                (long long)t0, (long long)(t0 + rows), (long long)T_total);
    GaeChunk c{T_total, t0, carry};
    return gae_forward_impl(value, B, reward, B, adv, B, rows, B, gamma, lambda, as_stream(stream), &c);
}

int hpc_rll_gae_backward_chunk(const float* grad_adv, float* grad_value, float* grad_reward, float* carry,
                               int64_t T_total, int64_t t0, int64_t rows, int64_t B, double gamma, double lambda,
                               void* stream) {
    HPC_NVTX("gae_backward_chunk");
    using namespace hpcrll;
    HPC_REQUIRE(carry != nullptr, "gae_backward_chunk: null carry");
    HPC_REQUIRE(t0 >= 0 && rows >= 0 && t0 + rows <= T_total, "gae_backward_chunk: rows [%lld, %lld) outside T=%lld",
                (long long)t0, (long long)(t0 + rows), (long long)T_total);
    GaeChunk c{T_total, t0, carry};
    return gae_backward_impl(grad_adv, B, grad_value, B, grad_reward, B, rows, B, gamma, lambda, as_stream(stream), &c);
}

int64_t hpc_rll_debug_host_schedule(int64_t T, int64_t B, int64_t* rows, int64_t cap) {
    const std::vector<int64_t> v = hpcrll::host_schedule(T, B);
    for (size_t i = 0; i < v.size() && static_cast<int64_t>(i) < cap; ++i) rows[i] = v[i];
    return static_cast<int64_t>(v.size());
}

int hpc_rll_gae_fwd_bwd_host(const float* h_value, const float* h_reward, const float* h_grad_adv, float* h_adv,
                             float* h_grad_value, float* h_grad_reward, int64_t T, int64_t B, double gamma,
                             double lambda) {
    HPC_NVTX("gae_fwd_bwd_host");
    return hpcrll::gae_host_impl(h_value, h_reward, h_grad_adv, h_adv, h_grad_value, h_grad_reward, T, B, gamma,
                                 lambda);
}

}  // extern "C"
