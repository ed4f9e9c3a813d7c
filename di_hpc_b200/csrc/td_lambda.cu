// td_lambda.cu -- TD(lambda) loss, forward and backward, for sm_90a.
//
// Semantics: hpc_rll/origin/td.py:148-176 (td_lambda_error) with the lambda-return of
// td.py:207-244 (multistep_forward_view):
//     ret_{T-1} = r_{T-1} + gamma*v_T
//     ret_t     = r_t + (gamma*lambda)*ret_{t+1} + (gamma - gamma*lambda)*v_{t+1}     (no_grad)
//     loss      = 0.5 * mean_{T*B}( w * (ret - v[:-1])^2 )
//     dloss/dv_t = -w_t (ret_t - v_t)/(T*B) for t < T, 0 for t = T
// Replaces TdLambdaForward/Backward (src/rl_utils/td_lambda.cu:8-52) and the kernels of
// include/hpc/rll/cuda/rl_utils/td_lambda_kernel.h:11-51.
//
// Forward = ONE pass: ScanPipe streams value/reward(/weight) boxes by TMA, each column thread walks
// T backward carrying ret, accumulates the loss term in fp64 and writes grad_buf = dloss/dv
// (without the upstream gradient).  Backward = scale by the upstream gradient (device scalar).
// Bytes/step: fwd 8 (+4 weight) in + 4 out, bwd 4 in + 4 out.
#include "reduce.cuh"
#include "scan_lookback.cuh"
#include "scan_pipe.cuh"

namespace hpcrll {

template <int NIN>
struct TdLambdaBody {
    float ret, v1, gamma, disc, gmd, neg_inv_n;
    double acc;
    float* gbuf;  // running pointer, t descending
    int64_t ld;
    int t_last;
    bool valid;
    // state at a segment edge: steps run from row t_edge-1 down, with ret = ret_{t_edge} (the carry; unused when
    // t_edge = T) and v1 = value[t_edge]; `valid`: column col exists
    static __device__ __forceinline__ TdLambdaBody at(int t_edge, float carry, const float* value, float* grad_buf,
                                                      int B, int T, int col, float gamma, float disc, float gmd,
                                                      float neg_inv_n, bool valid) {
        TdLambdaBody b;
        b.valid = valid;
        b.ret = carry;
        b.gamma = gamma;
        b.disc = disc;
        b.gmd = gmd;
        b.neg_inv_n = neg_inv_n;
        b.acc = 0.0;
        b.ld = B;
        b.t_last = T - 1;
        b.gbuf = grad_buf + static_cast<int64_t>(t_edge - 1) * B + col;
        b.v1 = valid ? __ldg(value + static_cast<int64_t>(t_edge) * B + col) : 0.f;
        return b;
    }
    __device__ __forceinline__ void step(int t, const float (&x)[NIN], const float (&)[1]) {
        // x[0] = v_t, x[1] = r_t, x[2] = w_t (if NIN == 3)
        if (t == t_last)
            ret = __fadd_rn(x[1], __fmul_rn(gamma, v1));
        else
            ret = __fadd_rn(__fadd_rn(x[1], __fmul_rn(disc, ret)), __fmul_rn(gmd, v1));
        const float w = NIN == 3 ? x[2] : 1.f;
        const float diff = __fsub_rn(ret, x[0]);
        const float wd = __fmul_rn(w, diff);
        acc += static_cast<double>(__fmul_rn(wd, diff));
        if (valid) st_stream(gbuf, __fmul_rn(neg_inv_n, wd));
        gbuf -= ld;
        v1 = x[0];
    }
};

template <int NIN, int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) td_lambda_fwd_tma(const __grid_constant__ TmapPack<NIN> maps,
                                                              const float* __restrict__ value,
                                                              float* __restrict__ grad_buf,
                                                              double* __restrict__ partials, int T, int B,
                                                              float gamma, float disc, float gmd, float neg_inv_n) {
    using Pipe = ScanPipe<NIN, 0, 0, BT, TT, ST, 0>;
    __shared__ double red[32];
    const int col0 = blockIdx.x * BT;
    const int col = col0 + threadIdx.x;
    TdLambdaBody<NIN> body = TdLambdaBody<NIN>::at(T, 0.f, value, grad_buf, B, T, col, gamma, disc, gmd, neg_inv_n,
                                                   threadIdx.x < BT && col < B);
    Pipe::template run<true>(maps, {}, nullptr, T, col0, body);
    double v[1] = {body.valid ? body.acc : 0.0};
    block_sum<1>(v, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = v[0];
}

// small batches: single-launch T-split with look-back (scan_lookback.cuh); constant coefficient gamma*lambda (the
// reset at t = T-1 sits in the first segment scanned, which has no predecessor)
template <int NIN>
struct TdlLbFac {
    const float* value;
    float* grad_buf;
    int B, T, col;
    bool valid;
    float gamma, disc, gmd, neg_inv_n;
    double* partial;  // this CTA's slot
    using Body = TdLambdaBody<NIN>;
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {
        const bool store = valid && pass == 1;
        Body b = Body::at(t_edge, carry, value, grad_buf, B, T, col, gamma, disc, gmd, neg_inv_n, valid);
        b.valid = store;
        return b;
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[NIN]) const {
        const float none[1] = {0.f};
        b.step(t, x, none);
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.ret; }
    static __device__ __forceinline__ float coef(const Body&) { return 0.f; }
    __device__ __forceinline__ void finish(Body& b, int, int) const {
        double v = valid ? b.acc : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0) *partial = v;
    }
};

template <int NIN>
__global__ void __launch_bounds__(kLbCols) td_lambda_fwd_lookback(const float* __restrict__ value,
                                                                  const float* __restrict__ reward,
                                                                  const float* __restrict__ weight,
                                                                  float* __restrict__ grad_buf,
                                                                  double* __restrict__ partials, int T, int B, float gamma,
                                                                  float disc, float gmd, float neg_inv_n, float AL, int S,
                                                                  int L, int tiles, LbCtl* ctl, unsigned long long* words) {
    __shared__ float smem[NIN * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const TdlLbFac<NIN> fac{value, grad_buf, B, T, col, col < B, gamma, disc, gmd, neg_inv_n, partials + lt.vid};
    const float* in[NIN];
    int64_t ld[NIN];
    in[0] = value;
    in[1] = reward;
    if (NIN == 3) in[NIN - 1] = weight;
#pragma unroll
    for (int k = 0; k < NIN; ++k) ld[k] = B;
    lb_segment<NIN, true, true>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, AL, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

// generic fallback (no TMA alignment requirements): the same body driven by scan_column, one thread per column
template <bool HAS_W>
__global__ void __launch_bounds__(128) td_lambda_fwd_generic(const float* __restrict__ value,
                                                              const float* __restrict__ reward,
                                                              const float* __restrict__ weight,
                                                              float* __restrict__ grad_buf,
                                                              double* __restrict__ partials, int T, int B,
                                                              float gamma, float disc, float gmd, float neg_inv_n) {
    constexpr int NIN = HAS_W ? 3 : 2;
    __shared__ double red[32];
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    TdLambdaBody<NIN> body = TdLambdaBody<NIN>::at(T, 0.f, value, grad_buf, B, T, col, gamma, disc, gmd, neg_inv_n, col < B);
    if (body.valid) {
        if constexpr (HAS_W)
            scan_column<3, 0, 0, 0, true>({{value, B}, {reward, B}, {weight, B}}, {}, nullptr, {}, T, col, body);
        else
            scan_column<2, 0, 0, 0, true>({{value, B}, {reward, B}}, {}, nullptr, {}, T, col, body);
    }
    double v[1] = {body.valid ? body.acc : 0.0};
    block_sum<1>(v, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = v[0];
}

template <int NIN, int BT, int TT, int ST>
static int launch_tdl_tma(const float* value, const float* reward, const float* weight, float* grad_buf,
                          double* partials, int64_t T, int64_t B, float g, float disc, float gmd, float nin,
                          cudaStream_t stream, int* nblocks) {
    TmapPack<NIN> maps;
    int rc = make_tmap_2d(&maps.m[0], value, T + 1, B, B, TT, BT);
    if (rc) return rc;
    rc = make_tmap_2d(&maps.m[1], reward, T, B, B, TT, BT);
    if (rc) return rc;
    if (NIN == 3) {
        rc = make_tmap_2d(&maps.m[NIN - 1], weight, T, B, B, TT, BT);
        if (rc) return rc;
    }
    const unsigned grid = static_cast<unsigned>((B + BT - 1) / BT);
    *nblocks = static_cast<int>(grid);
    return launch_scan<ScanPipe<NIN, 0, 0, BT, TT, ST, 0>, td_lambda_fwd_tma<NIN, BT, TT, ST>>(
        grid, stream, maps, value, grad_buf, partials, static_cast<int>(T), static_cast<int>(B), g, disc, gmd, nin);
}

// per-CTA loss partials: one per column tile, or one per (segment, tile) of the small-batch T-split (<= 4*SMs + tiles)
size_t td_lambda_workspace_bytes(int64_t B) {
    return sizeof(double) * static_cast<size_t>((B + 31) / 32 + 4 * sm_count() + 72);
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_td_lambda_forward(const float* value, const float* reward, const float* weight, float* loss,
                              float* grad_buf, int64_t T, int64_t B, double gamma, double lambda,
                              int64_t global_B, void* workspace, size_t workspace_bytes, void* stream_) {
    HPC_NVTX("td_lambda_forward");
    using namespace hpcrll;
    cudaStream_t stream = as_stream(stream_);
    HPC_REQUIRE(T > 0 && B > 0, "td_lambda_forward: T and B must be positive (T=%lld B=%lld)", (long long)T,
                (long long)B);
    HPC_REQUIRE(value && reward && loss && grad_buf && workspace, "td_lambda_forward: null pointer");
    HPC_REQUIRE(workspace_bytes >= td_lambda_workspace_bytes(B), "td_lambda_forward: workspace too small");
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512, "td_lambda_forward: T/B exceed 2^31");
    if (global_B <= 0) global_B = B;
    // origin builds gammas/lambdas as fp32 tensors and multiplies them (td.py:196-199,239)
    const float g = static_cast<float>(gamma), l = static_cast<float>(lambda);
    const float disc = g * l;
    const float gmd = g - disc;
    const double inv_n = 1.0 / (static_cast<double>(T) * static_cast<double>(global_B));
    const float nin = static_cast<float>(-inv_n);
    double* partials = static_cast<double*>(workspace);
    int nblocks = 0;
    const bool tma = tma_ok_2d(value, B, B) && tma_ok_2d(reward, B, B) && (!weight || tma_ok_2d(weight, B, B));
    int cfg = tuning_config(HPC_RLL_OP_TD_LAMBDA);
    LbGeom lg;
    const bool lookback = lookback_geometry(HPC_RLL_OP_TD_LAMBDA, T, B, &lg);
    if (!tma) cfg = 99;
    if (cfg < 0 || cfg == 21) cfg = B >= 128 * static_cast<int64_t>(sm_count()) ? 1 : (B >= 4096 ? 0 : 2);
    int rc = HPC_RLL_OK;
    if (lookback) {
        LbScratch sc;
        rc = lookback_scratch(lg, B, stream, &sc);
        if (rc) return rc;
        nblocks = lg.S * lg.tiles;
        const float AL = powf(disc, static_cast<float>(lg.L));
        if (weight)
            td_lambda_fwd_lookback<3><<<static_cast<unsigned>(nblocks), kLbCols, 0, stream>>>(
                value, reward, weight, grad_buf, partials, static_cast<int>(T), static_cast<int>(B), g, disc, gmd, nin, AL,
                lg.S, lg.L, lg.tiles, sc.ctl, sc.words);
        else
            td_lambda_fwd_lookback<2><<<static_cast<unsigned>(nblocks), kLbCols, 0, stream>>>(
                value, reward, weight, grad_buf, partials, static_cast<int>(T), static_cast<int>(B), g, disc, gmd, nin, AL,
                lg.S, lg.L, lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
    } else if (cfg == 99) {
        const unsigned grid = static_cast<unsigned>((B + 127) / 128);
        nblocks = static_cast<int>(grid);
        if (weight)
            td_lambda_fwd_generic<true><<<grid, 128, 0, stream>>>(value, reward, weight, grad_buf, partials,
                                                                  static_cast<int>(T), static_cast<int>(B), g, disc,
                                                                  gmd, nin);
        else
            td_lambda_fwd_generic<false><<<grid, 128, 0, stream>>>(value, reward, weight, grad_buf, partials,
                                                                   static_cast<int>(T), static_cast<int>(B), g, disc,
                                                                   gmd, nin);
        count_launch();
        HPC_LAUNCH_CHECK();
    } else if (weight) {
        switch (cfg) {
            case 0: rc = launch_tdl_tma<3, 64, 16, 3>(value, reward, weight, grad_buf, partials, T, B, g, disc, gmd, nin, stream, &nblocks); break;
            case 1: rc = launch_tdl_tma<3, 256, 8, 4>(value, reward, weight, grad_buf, partials, T, B, g, disc, gmd, nin, stream, &nblocks); break;
            default: rc = launch_tdl_tma<3, 32, 32, 3>(value, reward, weight, grad_buf, partials, T, B, g, disc, gmd, nin, stream, &nblocks); break;
        }
    } else {
        switch (cfg) {
            case 0: rc = launch_tdl_tma<2, 64, 16, 3>(value, reward, weight, grad_buf, partials, T, B, g, disc, gmd, nin, stream, &nblocks); break;
            case 1: rc = launch_tdl_tma<2, 256, 8, 4>(value, reward, weight, grad_buf, partials, T, B, g, disc, gmd, nin, stream, &nblocks); break;
            default: rc = launch_tdl_tma<2, 32, 32, 3>(value, reward, weight, grad_buf, partials, T, B, g, disc, gmd, nin, stream, &nblocks); break;
        }
    }
    if (rc) return rc;
    finalize_sums<1><<<1, 256, 0, stream>>>(partials, nblocks, nullptr, 0.5 * inv_n, 0, 0, 0, 0, loss);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

int hpc_rll_td_lambda_backward(const float* grad_loss, const float* grad_buf, float* grad_value, int64_t T,
                               int64_t B, void* stream_) {
    HPC_NVTX("td_lambda_backward");
    using namespace hpcrll;
    HPC_REQUIRE(T > 0 && B > 0, "td_lambda_backward: T and B must be positive");
    HPC_REQUIRE(grad_loss && grad_buf && grad_value, "td_lambda_backward: null pointer");
    // rows 0..T-1 scaled by the upstream gradient, row T (bootstrap value) gets exactly 0
    return launch_scale_copy(grad_buf, grad_loss, grad_value, T * B, B, as_stream(stream_));
}

}  // extern "C"
