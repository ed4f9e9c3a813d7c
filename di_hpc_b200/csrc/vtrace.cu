// vtrace.cu -- V-trace (IMPALA) losses, forward and backward, for sm_90a.
//
// Semantics: hpc_rll/origin/vtrace.py:63-79 (vtrace_error), 5-13 (vtrace_nstep_return),
// 16-17 (vtrace_advantage), 81-111 (compute_importance_weights):
//     IS = exp(logp_target[a] - logp_behaviour[a]);  rho=min(IS,rho_bar) c=min(IS,c_bar) rpg=min(IS,rho_pg)
//     item_t = rho_t(r_t + gamma v_{t+1} - v_t) + gamma*lambda*c_t*item_{t+1};  ret_t = v_t + item_t
//     adv_t  = rpg_t (r_t + gamma ret_{t+1} - v_t),  ret_T := v_T                  (all no_grad)
//     pg = -mean(logp[a]*adv*w)   value = mean((v-ret)^2 w)   entropy = mean(H w)
// Replaces VTraceForward/VTraceBackward (src/rl_utils/vtrace.cu:8-130) and the 8 kernels of
// include/hpc/rll/cuda/rl_utils/vtrace_kernel.h (6 forward launches + 3 memsets, three (T,B,N)
// scratch tensors written and re-read, float atomics).
//
// Forward here = 2 kernels + finaliser:
//   vtrace_rows_fwd : one streaming pass over both logits tensors -> IS (T,B), logp (T,B),
//                     entropy-loss partial sums (row-in-registers softmax, see softmax_rows.cuh)
//   vtrace_scan     : ScanPipe over (value, reward, IS, logp[, weight]) walking T backward with the
//                     data-dependent coefficient gamma*lambda*c_t; emits the two per-step coefficients
//                     the backward needs (pg_coef = -adv*w/n, gv_buf = 2(v-ret)w/n) and loss partials
// Backward = softmax-gradient row kernel (recomputes softmax from logits) + scale of gv_buf.
#include "scan_lookback.cuh"
#include "scan_pipe.cuh"
#include "softmax_rows.cuh"

namespace hpcrll {

// ------------------------------------------------------------------------------------------------
// forward stage 1: rows
// ------------------------------------------------------------------------------------------------
// one (target, behaviour) row pair -> IS and the target's log-prob of the chosen action, and the entropy partial;
// args: (action, weight, is_out, logp_out)
struct VtraceRowOp {
    static constexpr int kTensors = 2;
    static constexpr bool kEntropy = true, kCat = true;
    struct Scalars {
        int a;
    };
    double acc[1] = {0.0};
    __device__ __forceinline__ Scalars scalars(int64_t r, bool ok, int, const int64_t* __restrict__ action,
                                               const float*, float*, float*) const {
        return {ok ? static_cast<int>(action[r]) : -1};
    }
    __device__ __forceinline__ void emit(int64_t row, const Scalars&, float H, float lp0, float lp1, const int64_t*,
                                         const float* __restrict__ weight, float* __restrict__ is_out,
                                         float* __restrict__ logp_out) {
        is_out[row] = expf(lp0 - lp1);
        logp_out[row] = lp0;
        acc[0] += static_cast<double>(H * (weight ? weight[row] : 1.f));
    }
};

template <int KMAX, int WIDTH, bool G1>
__global__ void __launch_bounds__(256) vtrace_rows_fwd(const float* __restrict__ target,
                                                        const float* __restrict__ behaviour,
                                                        const int64_t* __restrict__ action,
                                                        const float* __restrict__ weight, float* __restrict__ is_out,
                                                        float* __restrict__ logp_out, double* __restrict__ partials,
                                                        int64_t R, int N_, int G_, int log2G_) {
    VtraceRowOp op;
    HPC_ROWS_FWD_REGS(op, target, behaviour, action, weight, is_out, logp_out);
    flush_partials(op.acc, partials);
}

__global__ void __launch_bounds__(kStageRows) vtrace_rows_fwd_staged(const float* __restrict__ target,
                                                                      const float* __restrict__ behaviour,
                                                                      const int64_t* __restrict__ action,
                                                                      const float* __restrict__ weight,
                                                                      float* __restrict__ is_out,
                                                                      float* __restrict__ logp_out,
                                                                      double* __restrict__ partials, int64_t R, int N,
                                                                      int P, int aligned) {
    VtraceRowOp op;
    rows_fwd_staged(op, R, N, P, aligned, target, behaviour, action, weight, is_out, logp_out);
    flush_partials(op.acc, partials);
}

__global__ void __launch_bounds__(256) vtrace_rows_fwd_loop(const float* __restrict__ target,
                                                             const float* __restrict__ behaviour,
                                                             const int64_t* __restrict__ action,
                                                             const float* __restrict__ weight,
                                                             float* __restrict__ is_out, float* __restrict__ logp_out,
                                                             double* __restrict__ partials, int64_t R, int N) {
    VtraceRowOp op;
    rows_fwd_loop(op, R, N, target, behaviour, action, weight, is_out, logp_out);
    flush_partials(op.acc, partials);
}

struct VtraceRows {
    template <int K, int W, bool G1>
    static auto reg() { return vtrace_rows_fwd<K, W, G1>; }
    static auto staged() { return vtrace_rows_fwd_staged; }
    static auto loop() { return vtrace_rows_fwd_loop; }
    static constexpr int kStagedTiles = 2;
};

// ------------------------------------------------------------------------------------------------
// forward stage 2: scan
// ------------------------------------------------------------------------------------------------
template <int NIN>
struct VtraceBody {
    float item, v1, ret_next, gamma, factor, rc, cc, pc, inv_n;
    float a_last;  // coefficient of the last step (gamma*lambda*c_t): the T-split look-back multiplies these up
    double acc_pg, acc_v;
    float* pg_coef;  // running pointers, t descending
    float* gv_buf;
    int64_t ld;
    bool valid;
    // state at a segment edge: steps run from row t_edge-1 down, with item = item_{t_edge} (the carry), v1 = value[t_edge]
    // and ret_next = v1 + item (ret_T := v_T, vtrace.py:70); `valid`: column col exists
    static __device__ __forceinline__ VtraceBody at(int t_edge, float carry, const float* value, float* pg_coef,
                                                    float* gv_buf, int B, int T, int col, float gamma, float factor,
                                                    float rc, float cc, float pc, float inv_n, bool valid) {
        VtraceBody b;
        b.valid = valid;
        b.item = carry;
        b.gamma = gamma;
        b.factor = factor;
        b.rc = rc;
        b.cc = cc;
        b.pc = pc;
        b.inv_n = inv_n;
        b.a_last = 1.f;
        b.acc_pg = b.acc_v = 0.0;
        b.ld = B;
        b.pg_coef = pg_coef + static_cast<int64_t>(t_edge - 1) * B + col;
        b.gv_buf = gv_buf + static_cast<int64_t>(t_edge - 1) * B + col;
        b.v1 = valid ? __ldg(value + static_cast<int64_t>(t_edge) * B + col) : 0.f;
        b.ret_next = t_edge < T ? __fadd_rn(b.v1, carry) : b.v1;
        return b;
    }
    __device__ __forceinline__ void step(int /*t*/, const float (&x)[NIN], const float (&)[1]) {
        // x[0]=v_t x[1]=r_t x[2]=IS_t x[3]=logp_t x[4]=w_t
        const float is = x[2];
        const float rho = fminf(is, rc), c = fminf(is, cc), rpg = fminf(is, pc);
        const float v0 = x[0], r = x[1];
        const float delta = __fmul_rn(rho, __fsub_rn(__fadd_rn(r, __fmul_rn(gamma, v1)), v0));
        a_last = __fmul_rn(factor, c);
        item = __fadd_rn(delta, __fmul_rn(a_last, item));
        const float ret = __fadd_rn(v0, item);
        const float adv = __fmul_rn(rpg, __fsub_rn(__fadd_rn(r, __fmul_rn(gamma, ret_next)), v0));
        ret_next = ret;
        const float w = NIN == 5 ? x[NIN - 1] : 1.f;
        acc_pg += static_cast<double>(__fmul_rn(__fmul_rn(x[3], adv), w));
        const float dv = __fsub_rn(v0, ret);
        acc_v += static_cast<double>(__fmul_rn(__fmul_rn(dv, dv), w));
        if (valid) {
            st_stream(pg_coef, -(adv * w) * inv_n);
            st_stream(gv_buf, 2.f * (dv * w) * inv_n);
        }
        pg_coef -= ld;
        gv_buf -= ld;
        v1 = v0;
    }
};

template <int NIN, int BT, int TT, int ST>
__global__ void __launch_bounds__(BT + 32) vtrace_scan_tma(const __grid_constant__ TmapPack<NIN> maps,
                                                            const float* __restrict__ value,
                                                            float* __restrict__ pg_coef, float* __restrict__ gv_buf,
                                                            double* __restrict__ partials, int nblocks, int T, int B,
                                                            float gamma, float factor, float rc, float cc, float pc,
                                                            float inv_n) {
    using Pipe = ScanPipe<NIN, 0, 0, BT, TT, ST, 0>;
    __shared__ double red[64];
    const int col0 = blockIdx.x * BT;
    const int col = col0 + threadIdx.x;
    VtraceBody<NIN> body = VtraceBody<NIN>::at(T, 0.f, value, pg_coef, gv_buf, B, T, col, gamma, factor, rc, cc, pc,
                                               inv_n, threadIdx.x < BT && col < B);
    Pipe::template run<true>(maps, {}, nullptr, T, col0, body);
    double v[2] = {body.valid ? body.acc_pg : 0.0, body.valid ? body.acc_v : 0.0};
    block_sum<2>(v, red);
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = v[0];
        partials[nblocks + blockIdx.x] = v[1];
    }
}

// small batches: single-launch T-split with look-back (scan_lookback.cuh).  The coefficient gamma*lambda*min(IS, c_bar)
// is data dependent, so a segment publishes (prod a_t, zero-carry item); ret_{t+1} at a boundary is v_{t+1} + item_{t+1}
// formed with the same single rounding as in the serial scan.
template <int NIN>
struct VtraceLbFac {
    const float* value;
    float* pg_coef;
    float* gv_buf;
    int B, col;
    bool valid;
    float gamma, factor, rc, cc, pc, inv_n;
    double* partial_pg;
    double* partial_v;
    using Body = VtraceBody<NIN>;
    // not VtraceBody::at: its t_edge < T test for ret_next changes this kernel's machine code.  The carry is 0 at
    // t_edge = T, so v1 + carry here equals at()'s v1 up to the sign of a zero.
    __device__ __forceinline__ Body make(int pass, int t_edge, float carry) const {
        Body b;
        b.valid = valid && pass == 1;
        b.item = carry;
        b.gamma = gamma;
        b.factor = factor;
        b.rc = rc;
        b.cc = cc;
        b.pc = pc;
        b.inv_n = inv_n;
        b.a_last = 1.f;
        b.acc_pg = b.acc_v = 0.0;
        b.ld = B;
        b.pg_coef = pg_coef + static_cast<int64_t>(t_edge - 1) * B + col;
        b.gv_buf = gv_buf + static_cast<int64_t>(t_edge - 1) * B + col;
        b.v1 = valid ? __ldg(value + static_cast<int64_t>(t_edge) * B + col) : 0.f;
        b.ret_next = __fadd_rn(b.v1, carry);  // ret_T := v_T (carry is 0 there, vtrace.py:70)
        return b;
    }
    __device__ __forceinline__ void step(Body& b, int t, const float (&x)[NIN]) const {
        const float none[1] = {0.f};
        b.step(t, x, none);
    }
    static __device__ __forceinline__ float state(const Body& b) { return b.item; }
    static __device__ __forceinline__ float coef(const Body& b) { return b.a_last; }
    __device__ __forceinline__ void finish(Body& b, int, int) const {
        double v0 = valid ? b.acc_pg : 0.0, v1 = valid ? b.acc_v : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            v0 += __shfl_xor_sync(0xffffffffu, v0, o);
            v1 += __shfl_xor_sync(0xffffffffu, v1, o);
        }
        if (threadIdx.x == 0) {
            *partial_pg = v0;
            *partial_v = v1;
        }
    }
};

template <int NIN>
__global__ void __launch_bounds__(kLbCols) vtrace_scan_lookback(const float* __restrict__ value,
                                                                const float* __restrict__ reward,
                                                                const float* __restrict__ is_in,
                                                                const float* __restrict__ logp_in,
                                                                const float* __restrict__ weight,
                                                                float* __restrict__ pg_coef, float* __restrict__ gv_buf,
                                                                double* __restrict__ partials, int nblocks, int T, int B,
                                                                float gamma, float factor, float rc, float cc, float pc,
                                                                float inv_n, int S, int L, int tiles, LbCtl* ctl,
                                                                unsigned long long* words) {
    __shared__ float smem[NIN * kLbChunkRows * kLbCols];
    const LbTile lt = lb_begin(ctl, tiles);
    const int seg = S - 1 - lt.k;
    const int t0 = seg * L, t1 = min(T, t0 + L);
    const int col = lt.tile * kLbCols + threadIdx.x;
    const VtraceLbFac<NIN> fac{value, pg_coef, gv_buf, B,  col,           col < B, gamma, factor, rc, cc, pc, inv_n,
                               partials + lt.vid, partials + nblocks + lt.vid};
    const float* in[NIN];
    int64_t ld[NIN];
    in[0] = value;
    in[1] = reward;
    in[2] = is_in;
    in[3] = logp_in;
    if (NIN == 5) in[NIN - 1] = weight;
#pragma unroll
    for (int k = 0; k < NIN; ++k) ld[k] = B;
    lb_segment<NIN, true, false>(fac, in, ld, t0, t1, col, col < B, lt, words, tiles * kLbCols, 1.f, smem);
    lb_end(ctl, S * tiles, lt.epoch);
}

template <bool HAS_W>
__global__ void __launch_bounds__(128) vtrace_scan_generic(const float* __restrict__ value,
                                                            const float* __restrict__ reward,
                                                            const float* __restrict__ is_in,
                                                            const float* __restrict__ logp_in,
                                                            const float* __restrict__ weight,
                                                            float* __restrict__ pg_coef, float* __restrict__ gv_buf,
                                                            double* __restrict__ partials, int nblocks, int T, int B,
                                                            float gamma, float factor, float rc, float cc, float pc,
                                                            float inv_n) {
    __shared__ double red[64];
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    VtraceBody<HAS_W ? 5 : 4> body = VtraceBody<HAS_W ? 5 : 4>::at(T, 0.f, value, pg_coef, gv_buf, B, T, col, gamma,
                                                                   factor, rc, cc, pc, inv_n, col < B);
    if (body.valid) {
        if constexpr (HAS_W)
            scan_column<5, 0, 0, 0, true>({{value, B}, {reward, B}, {is_in, B}, {logp_in, B}, {weight, B}}, {}, nullptr,
                                          {}, T, col, body);
        else
            scan_column<4, 0, 0, 0, true>({{value, B}, {reward, B}, {is_in, B}, {logp_in, B}}, {}, nullptr, {}, T, col,
                                          body);
    }
    double v[2] = {body.valid ? body.acc_pg : 0.0, body.valid ? body.acc_v : 0.0};
    block_sum<2>(v, red);
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = v[0];
        partials[nblocks + blockIdx.x] = v[1];
    }
}

template <int NIN, int BT, int TT, int ST>
static int launch_vtrace_scan(const float* value, const float* reward, const float* is_in, const float* logp_in,
                              const float* weight, float* pg_coef, float* gv_buf, double* partials, int64_t T,
                              int64_t B, float g, float f, float rc, float cc, float pc, float inv_n,
                              cudaStream_t stream, int nblocks) {
    TmapPack<NIN> maps;
    const float* srcs[5] = {value, reward, is_in, logp_in, weight};
    for (int k = 0; k < NIN; ++k) {
        int rc1 = make_tmap_2d(&maps.m[k], srcs[k], k == 0 ? T + 1 : T, B, B, TT, BT);
        if (rc1) return rc1;
    }
    return launch_scan<ScanPipe<NIN, 0, 0, BT, TT, ST, 0>, vtrace_scan_tma<NIN, BT, TT, ST>>(
        static_cast<unsigned>(nblocks), stream, maps, value, pg_coef, gv_buf, partials, nblocks, static_cast<int>(T),
        static_cast<int>(B), g, f, rc, cc, pc, inv_n);
}

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// workspace layout: [IS (T*B f32) | logp (T*B f32) | partials (doubles)]
// rows-kernel partials (<= 16 per SM) + two per scan CTA: column tiles, or (segment, tile) pairs of the small-batch
// T-split (<= 4*SMs + tiles of them)
static int64_t vtrace_partials_cap(int64_t B) { return static_cast<int64_t>(sm_count()) * 24 + 4 * ((B + 31) / 32) + 160; }
size_t vtrace_workspace_bytes(int64_t T, int64_t B) {
    return static_cast<size_t>(align_up(T * B * 4, 256) * 2 + vtrace_partials_cap(B) * 8 + 256);
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_vtrace_forward(const float* target_output, const float* behaviour_output, const int64_t* action,
                           const float* value, const float* reward, const float* weight, float* losses,
                           float* pg_coef, float* gv_buf, int64_t T, int64_t B, int64_t N, double gamma,
                           double lambda, double rho_clip_ratio, double c_clip_ratio, double rho_pg_clip_ratio,
                           int64_t global_B, void* workspace, size_t workspace_bytes, void* stream_) {
    HPC_NVTX("vtrace_forward");
    using namespace hpcrll;
    cudaStream_t stream = as_stream(stream_);
    HPC_REQUIRE(T > 0 && B > 0 && N > 0, "vtrace_forward: sizes must be positive (T=%lld B=%lld N=%lld)",
                (long long)T, (long long)B, (long long)N);
    HPC_REQUIRE(target_output && behaviour_output && action && value && reward && losses && pg_coef && gv_buf &&
                    workspace,
                "vtrace_forward: null pointer");
    HPC_REQUIRE(workspace_bytes >= vtrace_workspace_bytes(T, B), "vtrace_forward: workspace too small");
    HPC_REQUIRE(T < (int64_t(1) << 31) - 64 && B < (int64_t(1) << 31) - 512 && N < (int64_t(1) << 30),
                "vtrace_forward: sizes exceed 2^31");
    if (global_B <= 0) global_B = B;
    const int64_t R = T * B;
    char* ws = static_cast<char*>(workspace);
    float* is_buf = reinterpret_cast<float*>(ws);
    float* logp_buf = reinterpret_cast<float*>(ws + align_up(R * 4, 256));
    double* partials = reinterpret_cast<double*>(ws + 2 * align_up(R * 4, 256));
    const double inv_n = 1.0 / (static_cast<double>(T) * static_cast<double>(global_B));

    // ---- stage 1: rows ----
    unsigned grid1;
    if (int rc1 = launch_rows<VtraceRows>(&grid1, R, N, target_output, behaviour_output, stream, target_output,
                                          behaviour_output, action, weight, is_buf, logp_buf, partials))
        return rc1;

    // ---- stage 2: scan ----
    const float g = static_cast<float>(gamma), f = static_cast<float>(gamma * lambda);
    const float rc = static_cast<float>(rho_clip_ratio), cc = static_cast<float>(c_clip_ratio),
                pc = static_cast<float>(rho_pg_clip_ratio);
    double* part2 = partials + grid1;
    const bool tma = tma_ok_2d(value, B, B) && tma_ok_2d(reward, B, B) && (!weight || tma_ok_2d(weight, B, B));
    int cfg = tuning_config(HPC_RLL_OP_VTRACE);
    LbGeom lg;
    const bool lookback = lookback_geometry(HPC_RLL_OP_VTRACE, T, B, &lg);
    if (!tma) cfg = 99;
    if (cfg < 0 || cfg == 21) cfg = B >= 64 * static_cast<int64_t>(sm_count()) ? 0 : 2;
    int nblocks2;
    int rc2 = HPC_RLL_OK;
    const float in = static_cast<float>(inv_n);
    if (lookback) {
        LbScratch sc;
        rc2 = lookback_scratch(lg, B, stream, &sc);
        if (rc2) return rc2;
        nblocks2 = lg.S * lg.tiles;
        if (weight)
            vtrace_scan_lookback<5><<<static_cast<unsigned>(nblocks2), kLbCols, 0, stream>>>(
                value, reward, is_buf, logp_buf, weight, pg_coef, gv_buf, part2, nblocks2, static_cast<int>(T),
                static_cast<int>(B), g, f, rc, cc, pc, in, lg.S, lg.L, lg.tiles, sc.ctl, sc.words);
        else
            vtrace_scan_lookback<4><<<static_cast<unsigned>(nblocks2), kLbCols, 0, stream>>>(
                value, reward, is_buf, logp_buf, weight, pg_coef, gv_buf, part2, nblocks2, static_cast<int>(T),
                static_cast<int>(B), g, f, rc, cc, pc, in, lg.S, lg.L, lg.tiles, sc.ctl, sc.words);
        count_launch();
        HPC_LAUNCH_CHECK();
    } else if (cfg == 99) {
        nblocks2 = static_cast<int>((B + 127) / 128);
        if (weight)
            vtrace_scan_generic<true><<<nblocks2, 128, 0, stream>>>(value, reward, is_buf, logp_buf, weight, pg_coef,
                                                                    gv_buf, part2, nblocks2, static_cast<int>(T),
                                                                    static_cast<int>(B), g, f, rc, cc, pc, in);
        else
            vtrace_scan_generic<false><<<nblocks2, 128, 0, stream>>>(value, reward, is_buf, logp_buf, weight, pg_coef,
                                                                     gv_buf, part2, nblocks2, static_cast<int>(T),
                                                                     static_cast<int>(B), g, f, rc, cc, pc, in);
        count_launch();
        HPC_LAUNCH_CHECK();
    } else if (cfg == 0) {
        nblocks2 = static_cast<int>((B + 63) / 64);
        rc2 = weight ? launch_vtrace_scan<5, 64, 8, 4>(value, reward, is_buf, logp_buf, weight, pg_coef, gv_buf, part2,
                                                       T, B, g, f, rc, cc, pc, in, stream, nblocks2)
                     : launch_vtrace_scan<4, 64, 8, 4>(value, reward, is_buf, logp_buf, weight, pg_coef, gv_buf, part2,
                                                       T, B, g, f, rc, cc, pc, in, stream, nblocks2);
    } else {
        nblocks2 = static_cast<int>((B + 31) / 32);
        rc2 = weight ? launch_vtrace_scan<5, 32, 16, 3>(value, reward, is_buf, logp_buf, weight, pg_coef, gv_buf,
                                                        part2, T, B, g, f, rc, cc, pc, in, stream, nblocks2)
                     : launch_vtrace_scan<4, 32, 16, 3>(value, reward, is_buf, logp_buf, weight, pg_coef, gv_buf,
                                                        part2, T, B, g, f, rc, cc, pc, in, stream, nblocks2);
    }
    if (rc2) return rc2;

    // ---- finalise: {policy, value, entropy} ----
    FinSpec spec;
    spec.off[0] = static_cast<int>(grid1);
    spec.cnt[0] = nblocks2;
    spec.scale[0] = -inv_n;
    spec.off[1] = static_cast<int>(grid1) + nblocks2;
    spec.cnt[1] = nblocks2;
    spec.scale[1] = inv_n;
    spec.off[2] = 0;
    spec.cnt[2] = static_cast<int>(grid1);
    spec.scale[2] = inv_n;
    for (int k = 3; k < 5; ++k) spec.off[k] = spec.cnt[k] = 0, spec.scale[k] = 0.0;
    return launch_finalize_terms(partials, spec, 3, losses, stream);
}

int hpc_rll_vtrace_backward(const float* grad_policy_loss, const float* grad_value_loss,
                            const float* grad_entropy_loss, const float* target_output, const int64_t* action,
                            const float* weight, const float* pg_coef, const float* gv_buf, float* grad_target_output,
                            float* grad_value, int64_t T, int64_t B, int64_t N, int64_t global_B, void* stream_) {
    HPC_NVTX("vtrace_backward");
    using namespace hpcrll;
    cudaStream_t stream = as_stream(stream_);
    HPC_REQUIRE(T > 0 && B > 0 && N > 0, "vtrace_backward: sizes must be positive");
    HPC_REQUIRE(grad_policy_loss && grad_value_loss && grad_entropy_loss && target_output && action && pg_coef &&
                    gv_buf && grad_target_output && grad_value,
                "vtrace_backward: null pointer");
    if (global_B <= 0) global_B = B;
    const double inv_n = 1.0 / (static_cast<double>(T) * static_cast<double>(global_B));
    int rc = launch_softmax_grad_rows(target_output, action, pg_coef, weight, grad_policy_loss, grad_entropy_loss,
                                      inv_n, grad_target_output, T * B, N, stream);
    if (rc) return rc;
    return launch_scale_copy(gv_buf, grad_value_loss, grad_value, T * B, B, stream);
}

}  // extern "C"
