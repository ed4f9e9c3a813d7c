// upgo.cu -- UPGO loss, forward and backward, for sm_90a.
//
// Semantics: hpc_rll/origin/upgo.py:21-38 (upgo_returns), 40-70 (upgo_loss), 7-18 (tb_cross_entropy):
//     l_t   = [r_{t+1} + v_{t+2} >= v_{t+1}]  (t < T-1)
//     ret_{T-1} = r_{T-1} + v_T;   ret_t = r_t + l_t*ret_{t+1} + (1-l_t)*v_{t+1}
//     adv = rho*(ret - v[:-1])  (no_grad);   loss = -mean(adv * log_softmax(logits)[a])
//     dloss/dlogits = -(adv/(T*B)) * (onehot(a) - softmax)
// Replaces UpgoForward/UpgoBackward (src/rl_utils/upgo.cu:8-69) and the 4 kernels of
// include/hpc/rll/cuda/rl_utils/upgo_kernel.h:11-108 (block-per-row cross entropy writing a (T,B,N)
// grad buffer that the backward re-reads).
//
// Forward = upgo_rows_fwd (streaming log-softmax gather -> metric (T,B)) + upgo_scan (ScanPipe over
// value/reward/rho/metric with the {0,1} coefficient carried in registers; emits coef = -adv/n and the
// loss partials) + finaliser.  Backward = shared softmax-gradient row kernel (recompute from logits).
#include "scan_lookback.cuh"
#include "scan_pipe.cuh"
#include "softmax_rows.cuh"

namespace hpcrll {

// one logits row -> the log-softmax of the chosen action (`metric`); args: (action, metric)
struct UpgoRowOp {
    static constexpr int kTensors = 1;
    static constexpr bool kEntropy = false, kCat = false;
    struct Scalars {
        int a;
    };
    __device__ __forceinline__ Scalars scalars(int64_t r, bool ok, int, const int64_t* __restrict__ action,
                                               float*) const {
        return {ok ? static_cast<int>(action[r]) : -1};
    }
    __device__ __forceinline__ void emit(int64_t row, const Scalars&, float, float lp0, float, const int64_t*,
                                         float* __restrict__ metric) const {
        metric[row] = lp0;
    }
};

template <int KMAX, int WIDTH, bool G1>
__global__ void __launch_bounds__(256) upgo_rows_fwd(const float* __restrict__ logits,
                                                      const int64_t* __restrict__ action,
                                                      float* __restrict__ metric, int64_t R, int N_, int G_,
                                                      int log2G_) {
    UpgoRowOp op;
    HPC_ROWS_FWD_REGS(op, logits, nullptr, action, metric);
}

__global__ void __launch_bounds__(kStageRows) upgo_rows_fwd_staged(const float* __restrict__ logits,
                                                                    const int64_t* __restrict__ action,
                                                                    float* __restrict__ metric, int64_t R, int N, int P,
                                                                    int aligned) {
    UpgoRowOp op;
    rows_fwd_staged(op, R, N, P, aligned, logits, nullptr, action, metric);
}

__global__ void __launch_bounds__(256) upgo_rows_fwd_loop(const float* __restrict__ logits,
                                                           const int64_t* __restrict__ action,
                                                           float* __restrict__ metric, int64_t R, int N) {
    UpgoRowOp op;
    rows_fwd_loop(op, R, N, logits, nullptr, action, metric);
}

struct UpgoRows {
    template <int K, int W, bool G1>
    static auto reg() { return upgo_rows_fwd<K, W, G1>; }
    static auto staged() { return upgo_rows_fwd_staged; }
    static auto loop() { return upgo_rows_fwd_loop; }
    static constexpr int kStagedTiles = 1;
};

struct UpgoBody {
    float ret, v1, v2, r1, neg_inv_n;
    float a_last;  // coefficient of the last step (0 or 1): used by the T-split look-back
    double acc;
    float* coef;  // running pointer, t descending
    int64_t ld;
    int t_last;
    bool valid;
    // state at a segment edge: steps run from row t_edge-1 down, with ret = ret_{t_edge} (the carry; unused when
    // t_edge = T), v1 = value[t_edge] and the history the first step looks at, r_{t_edge} and v_{t_edge+1} (rows that
    // exist whenever t_edge < T; `reward` is not read at t_edge = T); `valid`: column col exists
    static __device__ __forceinline__ UpgoBody at(int t_edge, float carry, const float* value, const float* reward,
                                                  float* coef, int B, int T, int col, float neg_inv_n, bool valid) {
        UpgoBody b;
        b.valid = valid;
        b.ret = carry;
        b.neg_inv_n = neg_inv_n;
        b.a_last = 1.f;
        b.acc = 0.0;
        b.ld = B;
        b.t_last = T - 1;
        b.coef = coef + static_cast<int64_t>(t_edge - 1) * B + col;
        b.v1 = valid ? __ldg(value + static_cast<int64_t>(t_edge) * B + col) : 0.f;
        b.v2 = (valid && t_edge < T) ? __ldg(value + static_cast<int64_t>(t_edge + 1) * B + col) : 0.f;
        b.r1 = (valid && t_edge < T) ? __ldg(reward + static_cast<int64_t>(t_edge) * B + col) : 0.f;
        return b;
    }
    __device__ __forceinline__ void step(int t, const float (&x)[4], const float (&)[1]) {
        // x[0]=v_t x[1]=r_t x[2]=rho_t x[3]=metric_t
        const float v0 = x[0], r = x[1];
        if (t == t_last) {
            ret = __fadd_rn(r, v1);
            a_last = 0.f;
        } else {
            const float l = __fadd_rn(r1, v2) >= v1 ? 1.f : 0.f;
            a_last = l;
            ret = __fadd_rn(__fadd_rn(r, __fmul_rn(l, ret)), __fmul_rn(1.f - l, v1));
        }
        const float adv = __fmul_rn(x[2], __fsub_rn(ret, v0));
        acc += static_cast<double>(__fmul_rn(adv, x[3]));
        if (valid) st_stream(coef, adv * neg_inv_n);
        coef -= ld;
        v2 = v1;
        v1 = v0;
        r1 = r;
    }
};

template <int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) upgo_scan_tma(const __grid_constant__ TmapPack<4> maps,
                                                          const float* __restrict__ value, float* __restrict__ coef,
                                                          double* __restrict__ partials, int T, int B,
                                                          float neg_inv_n) {
    using Pipe = ScanPipe<4, 0, 0, BT, TT, ST, 0>;
    __shared__ double red[32];
    const int col0 = blockIdx.x * BT;
    const int col = col0 + threadIdx.x;
    UpgoBody body = UpgoBody::at(T, 0.f, value, nullptr, coef, B, T, col, neg_inv_n, threadIdx.x < BT && col < B);
    Pipe::template run<true>(maps, {}, nullptr, T, col0, body);
    double v[1] = {body.valid ? body.acc : 0.0};
    block_sum<1>(v, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = v[0];
}

// small batches: single-launch T-split with look-back (scan_lookback.cuh).  The coefficient is the 0/1 "keep following
// the trajectory" flag, so a segment publishes (prod a_t, zero-carry return); with a_t in {0,1} the composition is exact.
struct UpgoLbFac {
    const float* value;
    const float* reward;
    float* coef_out;
    int B, T, col;
    bool valid;
    float neg_inv_n;
    double* partial;
    using Body = UpgoBody;
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {
        const bool store = valid && pass == 1;
        Body b = Body::at(t_edge, carry, value, reward, coef_out, B, T, col, neg_inv_n, valid);
        b.valid = store;
        return b;
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[4]) const {
        const float none[1] = {0.f};
        b.step(t, x, none);
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.ret; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.a_last; }
    __device__ __forceinline__ void finish(Body& b, int, int) const {
        double v = valid ? b.acc : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0) *partial = v;
    }
};

__global__ void __launch_bounds__(kLbCols) upgo_scan_lookback(const float* __restrict__ value,
                                                              const float* __restrict__ reward,
                                                              const float* __restrict__ rho,
                                                              const float* __restrict__ metric, float* __restrict__ coef,
                                                              double* __restrict__ partials, int T, int B, float neg_inv_n,
                                                              int S, int L, int tiles, LbCtl* ctl,
                                                              unsigned long long* words) {
    __shared__ float smem[4 * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const UpgoLbFac fac{value, reward, coef, B, T, col, col < B, neg_inv_n, partials + lt.vid};
    const float* const in[4] = {value, reward, rho, metric};
    const int64_t ld[4] = {B, B, B, B};
    lb_segment<4, true, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

__global__ void __launch_bounds__(128) upgo_scan_generic(const float* __restrict__ value,
                                                          const float* __restrict__ reward,
                                                          const float* __restrict__ rho,
                                                          const float* __restrict__ metric, float* __restrict__ coef,
                                                          double* __restrict__ partials, int T, int B,
                                                          float neg_inv_n) {
    __shared__ double red[32];
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    UpgoBody body = UpgoBody::at(T, 0.f, value, nullptr, coef, B, T, col, neg_inv_n, col < B);
    if (body.valid)
        scan_column<4, 0, 0, 0, true>({{value, B}, {reward, B}, {rho, B}, {metric, B}}, {}, nullptr, {}, T, col, body);
    double v[1] = {body.valid ? body.acc : 0.0};
    block_sum<1>(v, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = v[0];
}

template <int BT, int TT, int ST>
static int launch_upgo_scan(const float* value, const float* reward, const float* rho, const float* metric,
                            float* coef, double* partials, int64_t T, int64_t B, float nin, cudaStream_t stream,
                            int* nblocks) {
    TmapPack<4> maps;
    const float* srcs[4] = {value, reward, rho, metric};
    for (int k = 0; k < 4; ++k) {
        int rc1 = make_tmap_2d(&maps.m[k], srcs[k], k == 0 ? T + 1 : T, B, B, TT, BT);
        if (rc1) return rc1;
    }
    *nblocks = static_cast<int>((B + BT - 1) / BT);
    return launch_scan<ScanPipe<4, 0, 0, BT, TT, ST, 0>, upgo_scan_tma<BT, TT, ST>>(
        static_cast<unsigned>(*nblocks), stream, maps, value, coef, partials, static_cast<int>(T), static_cast<int>(B),
        nin);
}

static inline int64_t align_up_(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// workspace: [metric (T*B f32) | partials]
size_t upgo_workspace_bytes(int64_t T, int64_t B) {
    // partials: one per scan CTA -- column tiles, or (segment, tile) pairs of the small-batch T-split
    return static_cast<size_t>(align_up_(T * B * 4, 256) + ((B + 31) / 32 + 4 * sm_count() + 80) * 8 + 256);
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_upgo_forward(const float* target_output, const float* rhos, const int64_t* action,
                         const float* rewards, const float* bootstrap_values, float* loss, float* coef, int64_t T,
                         int64_t B, int64_t N, int64_t global_B, void* workspace, size_t workspace_bytes,
                         void* stream_) {
    HPC_NVTX("upgo_forward");
    using namespace hpcrll;
    cudaStream_t stream = as_stream(stream_);
    HPC_REQUIRE(T > 0 && B > 0 && N > 0, "upgo_forward: sizes must be positive (T=%lld B=%lld N=%lld)", (long long)T,
                (long long)B, (long long)N);
    HPC_REQUIRE(target_output && rhos && action && rewards && bootstrap_values && loss && coef && workspace,
                "upgo_forward: null pointer");
    HPC_REQUIRE(workspace_bytes >= upgo_workspace_bytes(T, B), "upgo_forward: workspace too small");
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512 && N < (int64_t(1) << 30),
                "upgo_forward: sizes exceed 2^31");
    if (global_B <= 0) global_B = B;
    const int64_t R = T * B;
    char* ws = static_cast<char*>(workspace);
    float* metric = reinterpret_cast<float*>(ws);
    double* partials = reinterpret_cast<double*>(ws + align_up_(R * 4, 256));
    const double inv_n = 1.0 / (static_cast<double>(T) * static_cast<double>(global_B));

    unsigned grid1;
    if (int rc1 = launch_rows<UpgoRows>(&grid1, R, N, target_output, nullptr, stream, target_output, action, metric))
        return rc1;

    const float nin = static_cast<float>(-inv_n);
    const bool tma = tma_ok_2d(bootstrap_values, B, B) && tma_ok_2d(rewards, B, B) && tma_ok_2d(rhos, B, B);
    int cfg = tuning_config(HPC_RLL_OP_UPGO);
    LbGeom lg;
    const bool lookback = lookback_geometry(HPC_RLL_OP_UPGO, T, B, &lg);
    if (!tma) cfg = 99;
    if (cfg < 0 || cfg == 21) cfg = B >= 64 * static_cast<int64_t>(sm_count()) ? 0 : 2;
    int nblocks = 0, rc = HPC_RLL_OK;
    if (lookback) {
        LbScratch sc;
        rc = lookback_scratch(lg, B, stream, &sc);
        if (rc) return rc;
        nblocks = lg.S * lg.tiles;
        upgo_scan_lookback<<<static_cast<unsigned>(nblocks), kLbCols, 0, stream>>>(
            bootstrap_values, rewards, rhos, metric, coef, partials, static_cast<int>(T), static_cast<int>(B), nin, lg.S,
            lg.L, lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
    } else if (cfg == 99) {
        nblocks = static_cast<int>((B + 127) / 128);
        upgo_scan_generic<<<nblocks, 128, 0, stream>>>(bootstrap_values, rewards, rhos, metric, coef, partials,
                                                       static_cast<int>(T), static_cast<int>(B), nin);
        count_launch();
        HPC_LAUNCH_CHECK();
    } else if (cfg == 0) {
        rc = launch_upgo_scan<64, 8, 4>(bootstrap_values, rewards, rhos, metric, coef, partials, T, B, nin, stream, &nblocks);
    } else {
        rc = launch_upgo_scan<32, 16, 3>(bootstrap_values, rewards, rhos, metric, coef, partials, T, B, nin, stream, &nblocks);
    }
    if (rc) return rc;
    FinSpec spec;
    for (int k = 0; k < 5; ++k) spec.off[k] = spec.cnt[k] = 0, spec.scale[k] = 0.0;
    spec.cnt[0] = nblocks;
    spec.scale[0] = -inv_n;
    return launch_finalize_terms(partials, spec, 1, loss, stream);
}

int hpc_rll_upgo_backward(const float* grad_loss, const float* target_output, const int64_t* action,
                          const float* coef, float* grad_target_output, int64_t T, int64_t B, int64_t N,
                          void* stream_) {
    HPC_NVTX("upgo_backward");
    using namespace hpcrll;
    HPC_REQUIRE(T > 0 && B > 0 && N > 0, "upgo_backward: sizes must be positive");
    HPC_REQUIRE(grad_loss && target_output && action && coef && grad_target_output, "upgo_backward: null pointer");
    return launch_softmax_grad_rows(target_output, action, coef, nullptr, grad_loss, nullptr, 0.0,
                                    grad_target_output, T * B, N, as_stream(stream_));
}

// tb_cross_entropy (hpc_rll/origin/upgo.py:7-18): UPGO's `metric` as a standalone op, through the same row kernels
int hpc_rll_tb_cross_entropy_forward(const float* logit, const int64_t* label, float* out, int64_t R, int64_t N,
                                     void* stream_) {
    HPC_NVTX("tb_cross_entropy_forward");
    using namespace hpcrll;
    HPC_REQUIRE(R >= 0, "tb_cross_entropy_forward: negative row count R=%lld", (long long)R);
    HPC_REQUIRE(N > 0 && N < (int64_t(1) << 30), "tb_cross_entropy_forward: the row length N must be in [1, 2^30), "
                "got %lld", (long long)N);
    if (R == 0) return HPC_RLL_OK;
    HPC_REQUIRE(logit && label && out, "tb_cross_entropy_forward: null logit, label or out pointer");
    unsigned grid;
    return launch_rows<UpgoRows>(&grid, R, N, logit, nullptr, as_stream(stream_), logit, label, out);
}

int hpc_rll_tb_cross_entropy_backward(const float* grad_out, const float* logit, const int64_t* label,
                                      float* grad_logit, int64_t R, int64_t N, void* stream_) {
    HPC_NVTX("tb_cross_entropy_backward");
    using namespace hpcrll;
    HPC_REQUIRE(R >= 0, "tb_cross_entropy_backward: negative row count R=%lld", (long long)R);
    HPC_REQUIRE(N > 0 && N < (int64_t(1) << 30), "tb_cross_entropy_backward: the row length N must be in [1, 2^30), "
                "got %lld", (long long)N);
    if (R == 0) return HPC_RLL_OK;
    HPC_REQUIRE(grad_out && logit && label && grad_logit,
                "tb_cross_entropy_backward: null grad_out, logit, label or grad_logit pointer");
    const float* one;  // {+1, -1}: the upstream gradient is the per-row c1, scaled by +1
    if (int rc = unit_scalars(&one)) return rc;
    return launch_softmax_grad_rows(logit, label, grad_out, nullptr, one, nullptr, 0.0, grad_logit, R, N,
                                    as_stream(stream_));
}

}  // extern "C"
