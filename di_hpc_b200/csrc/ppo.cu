// ppo.cu -- PPO clipped-surrogate losses, forward and backward, for sm_90a.
//
// Semantics: hpc_rll/origin/ppo.py:51-80 (ppo_error): policy loss with clip and optional dual clip,
// clipped value loss, entropy, approx_kl, clipfrac.  No T axis, no recurrence: one streaming pass.
// Tie rules follow autograd (torch.min/max split the gradient on exact ties, clamp passes it on the
// closed interval) -- SURVEY.md A.5, restated in oracle/oracle.c orc_ppo.
// Replaces PPOForward/PPOBackward (src/rl_utils/ppo.cu:8-111) and the 5 kernels of
// include/hpc/rll/cuda/rl_utils/ppo_kernel.h:12-283 (block-per-row softmax x2, 5 atomics, three
// (B,N) gradient buffers written by the forward, two host syncs for the info scalars).
//
// Forward = ONE kernel: both logits rows of a sample live in the registers of a sub-warp group;
// lane 0 of the group evaluates the scalar loss terms, stores the two per-sample coefficients the
// backward needs (pol_coef = dpolicy/dlogp_new[a], val_coef = dvalue_loss/dvalue_new) and feeds the
// 5 fixed-order reductions.  Backward = shared softmax-gradient row kernel + scale of val_coef.
#include "softmax_rows.cuh"

namespace hpcrll {

struct PpoParams {
    float lo, hi, eps, dual;  // 1-clip, 1+clip, clip, dual_clip (<=0: off)
    int use_value_clip;
    float inv_n;
    const float* adv_stats;  // {mean, std + 1e-8} on the device, or nullptr (adv already normalised)
};

// (adv - mean) / (std + 1e-8) with the statistics of hpc_rll_adv_stats; identity when there are none
struct AdvNorm {
    float mean, denom;
    bool has;
    __device__ __forceinline__ explicit AdvNorm(const PpoParams& P)
        : mean(P.adv_stats ? __ldg(P.adv_stats) : 0.f), denom(P.adv_stats ? __ldg(P.adv_stats + 1) : 1.f),
          has(P.adv_stats != nullptr) {}
    // (no statistics: (a - 0) / 1 == a exactly, so the IEEE division is skipped -- a block-uniform branch)
    __device__ __forceinline__ float operator()(float a) const {
        return has ? __fdiv_rn(__fsub_rn(a, mean), denom) : a;
    }
};

// scalar part for one sample; returns the five loss terms' contributions and the two coefficients
__device__ __forceinline__ void ppo_sample(const PpoParams& P, float lpn, float lpo, float H, float ad, float vn,
                                           float vo, float rt, float w, double (&acc)[5], float& pol_coef,
                                           float& val_coef) {
    const float ratio = expf(lpn - lpo);
    const float s1 = ratio * ad;
    const float rcl = fminf(fmaxf(ratio, P.lo), P.hi);
    const float s2 = rcl * ad;
    const float m = fminf(s1, s2);
    const float in_range = (ratio >= P.lo && ratio <= P.hi) ? 1.f : 0.f;
    const float g1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
    float dm = g1 * ad + (1.f - g1) * ad * in_range;
    float pol = m;
    if (P.dual > 0.f) {
        const float d = P.dual * ad;
        const float gm = m > d ? 1.f : (m == d ? 0.5f : 0.f);
        pol = fmaxf(m, d);
        dm *= gm;
    }
    const float e1 = rt - vn;
    const float v1 = e1 * e1;
    float vl, dval;
    if (P.use_value_clip) {
        const float dvv = vn - vo;
        const float cl = fminf(fmaxf(dvv, -P.eps), P.eps);
        const float e2 = rt - (vo + cl);
        const float v2 = e2 * e2;
        const float inr = (dvv >= -P.eps && dvv <= P.eps) ? 1.f : 0.f;
        const float k1 = v1 > v2 ? 1.f : (v1 == v2 ? 0.5f : 0.f);
        vl = fmaxf(v1, v2);
        dval = k1 * (-2.f * e1) + (1.f - k1) * (-2.f * e2) * inr;
    } else {
        vl = v1;
        dval = -2.f * e1;
    }
    acc[0] += static_cast<double>(-pol * w);
    acc[1] += static_cast<double>(vl * w);
    acc[2] += static_cast<double>(H * w);
    acc[3] += static_cast<double>(lpo - lpn);
    acc[4] += (ratio > P.hi || ratio < P.lo) ? 1.0 : 0.0;
    pol_coef = -(dm * ratio) * w * P.inv_n;
    val_coef = 0.5f * dval * w * P.inv_n;
}

// resident CTAs per SM the register budget is tuned for: two rows (+ their prefetched successors when the row is
// small) live in registers
constexpr int ppo_min_blocks(int kmax, int width) {
    const int ne = kmax * width;
    return ne >= 32 ? 1 : ((ne >= 20 || (ne == 8 && kmax >= 4)) ? 2 : 3);
}

// staged and looping layouts: one (new, old) logits row pair and the sample's scalars -> the five loss terms and the
// two backward coefficients; args: (action, value_new, value_old, adv, ret, weight, pol_coef, val_coef, &P)
struct PpoRowOp {
    static constexpr int kTensors = 2;
    static constexpr bool kEntropy = true, kCat = true;
    struct Scalars {
        float adv, vn, vo, ret, w;
        int a;
    };
    double acc[5];
    const AdvNorm norm;
    __device__ __forceinline__ Scalars scalars(int64_t r, bool, int, const int64_t* __restrict__ action,
                                               const float* __restrict__ value_new,
                                               const float* __restrict__ value_old, const float* __restrict__ adv,
                                               const float* __restrict__ ret, const float* __restrict__ weight, float*,
                                               float*, const PpoParams*) const {
        Scalars sc;
        sc.a = static_cast<int>(action[r]);
        sc.adv = adv[r];
        sc.vn = value_new[r];
        sc.vo = value_old[r];
        sc.ret = ret[r];
        sc.w = weight ? weight[r] : 1.f;
        return sc;
    }
    __device__ __forceinline__ void emit(int64_t row, const Scalars& sc, float H, float lp0, float lp1, const int64_t*,
                                         const float*, const float*, const float*, const float*, const float*,
                                         float* __restrict__ pol_coef, float* __restrict__ val_coef,
                                         const PpoParams* P) {
        float pc, vc;
        ppo_sample(*P, lp0, lp1, H, norm(sc.adv), sc.vn, sc.vo, sc.ret, sc.w, acc, pc, vc);
        pol_coef[row] = pc;
        val_coef[row] = vc;
    }
};

// The register layout keeps its own walk rather than HPC_ROWS_FWD_REGS: through the shared walk this kernel's machine
// code changes (register assignment in every layout, register counts and spills in some), whatever the shape of the op.
// G1: see HPC_ROWS_FWD_REGS.
template <int KMAX, int WIDTH, bool G1>
__global__ void __launch_bounds__(256, ppo_min_blocks(KMAX, WIDTH)) ppo_rows_fwd(const float* __restrict__ logits_new,
                                                     const float* __restrict__ logits_old,
                                                     const int64_t* __restrict__ action,
                                                     const float* __restrict__ value_new,
                                                     const float* __restrict__ value_old,
                                                     const float* __restrict__ adv, const float* __restrict__ ret,
                                                     const float* __restrict__ weight, float* __restrict__ pol_coef,
                                                     float* __restrict__ val_coef, double* __restrict__ partials,
                                                     const PpoParams P, int64_t R, int N_, int G_, int log2G_) {
    using Row = RowRegs<KMAX, WIDTH>;
    __shared__ double red[5 * 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = G1 ? KMAX * WIDTH : N_, G = G1 ? 1 : G_, log2G = G1 ? 0 : log2G_;
    const int lig = G1 ? 0 : (lane & (G - 1)), gw = lane >> log2G;
    const int rows_per_warp = 32 >> log2G;
    const int rows_per_block = rows_per_warp * 8;
    double acc[5] = {0, 0, 0, 0, 0};
    const AdvNorm norm(P);
    constexpr bool PF = Row::NE <= 8;  // software pipeline (see HPC_ROWS_FWD_REGS)
    Row rn, ro, nn, no;
    // per-sample scalars travel with the row loads (one iteration ahead), so that their latency is not exposed a
    // second time after the row statistics (ncu: this kernel was long-scoreboard-bound, 5.8 of 10 stall cycles)
    struct Scal {
        float adv, vn, vo, ret, w;
        int a;
    };
    auto load_scal = [&](int64_t r) {
        Scal sc;
        const bool ok = r < R;
        sc.a = ok ? static_cast<int>(__ldg(action + r)) : -1;
        const bool mine = ok && lig == 0;
        sc.adv = mine ? __ldg(adv + r) : 0.f;
        sc.vn = mine ? __ldg(value_new + r) : 0.f;
        sc.vo = mine ? __ldg(value_old + r) : 0.f;
        sc.ret = mine ? __ldg(ret + r) : 0.f;
        sc.w = (mine && weight) ? __ldg(weight + r) : 1.f;
        return sc;
    };
    Scal cur, nxt;
    // row index and row pointers advance by increments (no 64-bit multiply per row)
    const int64_t stride = static_cast<int64_t>(gridDim.x) * rows_per_block;
    int64_t base = static_cast<int64_t>(blockIdx.x) * rows_per_block;
    int64_t row = base + warp * rows_per_warp + gw;
    const float* pn = logits_new + row * N;
    const float* po = logits_old + row * N;
    const int64_t pstep = stride * N;
    rn.load(pn, N, G, lig, row < R);
    ro.load(po, N, G, lig, row < R);
    cur = load_scal(row);
    for (; base < R; base += stride, row += stride) {  // block-uniform trip count
        const bool active = row < R;
        const int64_t nrow = row + stride;
        pn += pstep;
        po += pstep;
        if (PF) {
            nn.load(pn, N, G, lig, nrow < R);
            no.load(po, N, G, lig, nrow < R);
        }
        nxt = load_scal(nrow);
        const int a = cur.a;
        const float mn = rn.row_max(G), mo = ro.row_max(G);
        float sn, tn, so, to, none[Row::NE];
        rn.template stats<true, false>(G, mn, sn, tn, none);
        ro.template stats<false, false>(G, mo, so, to, none);
        const float lsn = logf(sn), lso = logf(so);
        const float H = lsn - tn / sn;
        const float seln = row_logp<true>(group_sum(rn.select(a, G, lig), G), mn, lsn);
        const float selo = row_logp<true>(group_sum(ro.select(a, G, lig), G), mo, lso);
        if (active && lig == 0) {
            float pc, vc;
            ppo_sample(P, seln, selo, H, norm(cur.adv), cur.vn, cur.vo, cur.ret, cur.w, acc, pc, vc);
            pol_coef[row] = pc;
            val_coef[row] = vc;
        }
        if (PF) {
            rn = nn;
            ro = no;
        } else {
            rn.load(pn, N, G, lig, nrow < R);
            ro.load(po, N, G, lig, nrow < R);
        }
        cur = nxt;
    }
    block_sum<5>(acc, red);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < 5; ++k) partials[static_cast<size_t>(k) * gridDim.x + blockIdx.x] = acc[k];
    }
}

__global__ void __launch_bounds__(kStageRows) ppo_rows_fwd_staged(
    const float* __restrict__ logits_new, const float* __restrict__ logits_old, const int64_t* __restrict__ action,
    const float* __restrict__ value_new, const float* __restrict__ value_old, const float* __restrict__ adv,
    const float* __restrict__ ret, const float* __restrict__ weight, float* __restrict__ pol_coef,
    float* __restrict__ val_coef, double* __restrict__ partials, const PpoParams P, int64_t R, int N, int pitch,
    int aligned) {
    PpoRowOp op{{0, 0, 0, 0, 0}, AdvNorm(P)};
    rows_fwd_staged(op, R, N, pitch, aligned, logits_new, logits_old, action, value_new, value_old, adv, ret, weight,
                    pol_coef, val_coef, &P);
    flush_partials(op.acc, partials);
}

__global__ void __launch_bounds__(256) ppo_rows_fwd_loop(const float* __restrict__ logits_new,
                                                          const float* __restrict__ logits_old,
                                                          const int64_t* __restrict__ action,
                                                          const float* __restrict__ value_new,
                                                          const float* __restrict__ value_old,
                                                          const float* __restrict__ adv, const float* __restrict__ ret,
                                                          const float* __restrict__ weight,
                                                          float* __restrict__ pol_coef, float* __restrict__ val_coef,
                                                          double* __restrict__ partials, const PpoParams P, int64_t R,
                                                          int N) {
    PpoRowOp op{{0, 0, 0, 0, 0}, AdvNorm(P)};
    rows_fwd_loop(op, R, N, logits_new, logits_old, action, value_new, value_old, adv, ret, weight, pol_coef, val_coef,
                  &P);
    flush_partials(op.acc, partials);
}

struct PpoRows {
    template <int K, int W, bool G1>
    static auto reg() { return ppo_rows_fwd<K, W, G1>; }
    static auto staged() { return ppo_rows_fwd_staged; }
    static auto loop() { return ppo_rows_fwd_loop; }
    static constexpr int kStagedTiles = 2;
};

size_t ppo_workspace_bytes() { return static_cast<size_t>(sm_count()) * 16 * 5 * 8 + 256; }

static int ppo_forward_impl(const float* logits_new, const float* logits_old, const int64_t* action,
                            const float* value_new, const float* value_old, const float* adv, const float* return_,
                            const float* weight, const float* adv_stats, float* out5, float* pol_coef,
                            float* val_coef, int64_t B, int64_t N, double clip_ratio, int use_value_clip,
                            double dual_clip, int64_t global_B, void* workspace, size_t workspace_bytes,
                            void* stream_) {
    cudaStream_t stream = as_stream(stream_);
    HPC_REQUIRE(B > 0 && N > 0, "ppo_forward: sizes must be positive (B=%lld N=%lld)", (long long)B, (long long)N);
    HPC_REQUIRE(logits_new && logits_old && action && value_new && value_old && adv && return_ && out5 && pol_coef &&
                    val_coef && workspace,
                "ppo_forward: null pointer");
    HPC_REQUIRE(workspace_bytes >= ppo_workspace_bytes(), "ppo_forward: workspace too small");
    HPC_REQUIRE(N < (int64_t(1) << 30), "ppo_forward: N too large");
    HPC_REQUIRE(dual_clip <= 0.0 || dual_clip > 1.0, "ppo_forward: dual_clip must be > 1.0 (or <= 0 for None)");
    if (global_B <= 0) global_B = B;
    const double inv_n = 1.0 / static_cast<double>(global_B);
    PpoParams P;
    P.lo = static_cast<float>(1.0 - clip_ratio);
    P.hi = static_cast<float>(1.0 + clip_ratio);
    P.eps = static_cast<float>(clip_ratio);
    P.dual = dual_clip > 0.0 ? static_cast<float>(dual_clip) : 0.f;
    P.use_value_clip = use_value_clip;
    P.inv_n = static_cast<float>(inv_n);
    P.adv_stats = adv_stats;
    double* partials = static_cast<double*>(workspace);
    unsigned grid;
    if (int rc = launch_rows<PpoRows>(&grid, B, N, logits_new, logits_old, stream, logits_new, logits_old, action,
                                      value_new, value_old, adv, return_, weight, pol_coef, val_coef, partials, P))
        return rc;
    FinSpec spec;
    const double sc[5] = {inv_n, 0.5 * inv_n, inv_n, inv_n, inv_n};
    for (int k = 0; k < 5; ++k) {
        spec.off[k] = k * static_cast<int>(grid);
        spec.cnt[k] = static_cast<int>(grid);
        spec.scale[k] = sc[k];
    }
    return launch_finalize_terms(partials, spec, 5, out5, stream);
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_ppo_forward(const float* logits_new, const float* logits_old, const int64_t* action,
                        const float* value_new, const float* value_old, const float* adv, const float* return_,
                        const float* weight, float* out5, float* pol_coef, float* val_coef, int64_t B, int64_t N,
                        double clip_ratio, int use_value_clip, double dual_clip, int64_t global_B, void* workspace,
                        size_t workspace_bytes, void* stream) {
    HPC_NVTX("ppo_forward");
    return hpcrll::ppo_forward_impl(logits_new, logits_old, action, value_new, value_old, adv, return_, weight, nullptr,
                                    out5, pol_coef, val_coef, B, N, clip_ratio, use_value_clip, dual_clip, global_B,
                                    workspace, workspace_bytes, stream);
}

int hpc_rll_ppo_forward_norm(const float* logits_new, const float* logits_old, const int64_t* action,
                             const float* value_new, const float* value_old, const float* adv, const float* return_,
                             const float* weight, const float* adv_stats, float* out5, float* pol_coef,
                             float* val_coef, int64_t B, int64_t N, double clip_ratio, int use_value_clip,
                             double dual_clip, int64_t global_B, void* workspace, size_t workspace_bytes,
                             void* stream) {
    HPC_NVTX("ppo_forward_norm");
    using namespace hpcrll;
    HPC_REQUIRE(adv_stats, "ppo_forward_norm: adv_stats is null (use hpc_rll_ppo_forward for pre-normalised adv)");
    return ppo_forward_impl(logits_new, logits_old, action, value_new, value_old, adv, return_, weight, adv_stats, out5,
                            pol_coef, val_coef, B, N, clip_ratio, use_value_clip, dual_clip, global_B, workspace,
                            workspace_bytes, stream);
}

int hpc_rll_ppo_backward(const float* grad_policy_loss, const float* grad_value_loss, const float* grad_entropy_loss,
                         const float* logits_new, const int64_t* action, const float* weight, const float* pol_coef,
                         const float* val_coef, float* grad_logits_new, float* grad_value_new, int64_t B, int64_t N,
                         int64_t global_B, void* stream_) {
    HPC_NVTX("ppo_backward");
    using namespace hpcrll;
    cudaStream_t stream = as_stream(stream_);
    HPC_REQUIRE(B > 0 && N > 0, "ppo_backward: sizes must be positive");
    HPC_REQUIRE(grad_policy_loss && grad_value_loss && grad_entropy_loss && logits_new && action && pol_coef &&
                    val_coef && grad_logits_new && grad_value_new,
                "ppo_backward: null pointer");
    if (global_B <= 0) global_B = B;
    const double inv_n = 1.0 / static_cast<double>(global_B);
    int rc = launch_softmax_grad_rows(logits_new, action, pol_coef, weight, grad_policy_loss, grad_entropy_loss, inv_n,
                                      grad_logits_new, B, N, stream);
    if (rc) return rc;
    return launch_scale_copy(val_coef, grad_value_loss, grad_value_new, B, 0, stream);
}

}  // extern "C"
