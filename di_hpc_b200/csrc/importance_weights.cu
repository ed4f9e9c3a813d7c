// importance_weights.cu -- V-trace's importance ratios as a standalone op, forward and backward, for sm_90a.
//
// Semantics: hpc_rll/origin/vtrace.py:81-111 (compute_importance_weights):
//     rho = exp(logp_target[a] - logp_behaviour[a]),  logp = x - (m + log s)  (torch.distributions.Categorical)
//     d rho / d target[k]    =  c * (1[k=a] - p_target[k])
//     d rho / d behaviour[k] = -c * (1[k=a] - p_behaviour[k]),   c = G * rho  (one rounded fp32 multiply)
// The reference has no kernel for it: V-trace computes the ratios inside its loss (vtrace_rows_fwd writes them to its
// workspace), and callers that need them alone fall back to two torch Categorical distributions.
//
// Forward = importance_rows_fwd: one streaming pass over both logits tensors (row-in-registers softmax, see
// softmax_rows.cuh), 8N + 12 bytes per row.  The row statistics and log-probs are formed exactly as in vtrace_rows_fwd,
// so rho is bit-identical to the `is_out` of the fused V-trace forward.
// Backward = importance_grad_coef (c = G * rho into the workspace) + the shared softmax-gradient row kernel once per
// logits tensor that needs a gradient, with the upstream scale +1 (target) or -1 (behaviour).
#include "softmax_rows.cuh"

namespace hpcrll {

// one (target, behaviour) row pair -> the importance ratio of the chosen action; args: (action, rho)
struct ImportanceRowOp {
    static constexpr int kTensors = 2;
    static constexpr bool kEntropy = false, kCat = true;
    struct Scalars {
        int a;
    };
    __device__ __forceinline__ Scalars scalars(int64_t r, bool ok, int, const int64_t* __restrict__ action,
                                               float*) const {
        return {ok ? static_cast<int>(action[r]) : -1};
    }
    __device__ __forceinline__ void emit(int64_t row, const Scalars&, float, float lp0, float lp1, const int64_t*,
                                         float* __restrict__ rho) const {
        rho[row] = expf(lp0 - lp1);  // VtraceRowOp's is_out
    }
};

template <int KMAX, int WIDTH, bool G1>
__global__ void __launch_bounds__(256) importance_rows_fwd(const float* __restrict__ target,
                                                            const float* __restrict__ behaviour,
                                                            const int64_t* __restrict__ action,
                                                            float* __restrict__ rho, int64_t R, int N_, int G_,
                                                            int log2G_) {
    ImportanceRowOp op;
    HPC_ROWS_FWD_REGS(op, target, behaviour, action, rho);
}

__global__ void __launch_bounds__(kStageRows) importance_rows_fwd_staged(const float* __restrict__ target,
                                                                          const float* __restrict__ behaviour,
                                                                          const int64_t* __restrict__ action,
                                                                          float* __restrict__ rho, int64_t R, int N,
                                                                          int P, int aligned) {
    ImportanceRowOp op;
    rows_fwd_staged(op, R, N, P, aligned, target, behaviour, action, rho);
}

__global__ void __launch_bounds__(256) importance_rows_fwd_loop(const float* __restrict__ target,
                                                                 const float* __restrict__ behaviour,
                                                                 const int64_t* __restrict__ action,
                                                                 float* __restrict__ rho, int64_t R, int N) {
    ImportanceRowOp op;
    rows_fwd_loop(op, R, N, target, behaviour, action, rho);
}

struct ImportanceRows {
    template <int K, int W, bool G1>
    static auto reg() { return importance_rows_fwd<K, W, G1>; }
    static auto staged() { return importance_rows_fwd_staged; }
    static auto loop() { return importance_rows_fwd_loop; }
    static constexpr int kStagedTiles = 2;
};

// c[r] = G[r] * rho[r]: the coefficient autograd's exp backward forms, one rounded multiply
__global__ void __launch_bounds__(256) importance_grad_coef(const float* __restrict__ grad_rho,
                                                             const float* __restrict__ rho, float* __restrict__ c,
                                                             int64_t R) {
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < R;
         i += static_cast<int64_t>(gridDim.x) * blockDim.x)
        c[i] = __fmul_rn(__ldg(grad_rho + i), __ldg(rho + i));
}

static inline int64_t align_up_iw(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// workspace: [c (R f32)]
size_t importance_weights_workspace_bytes(int64_t R) {
    return static_cast<size_t>(align_up_iw((R > 0 ? R : 0) * 4, 256) + 256);
}

static int check_sizes(const char* what, int64_t R, int64_t N) {
    HPC_REQUIRE(R >= 0, "%s: negative row count R=%lld", what, (long long)R);
    HPC_REQUIRE(N > 0, "%s: the row length N must be positive, got %lld", what, (long long)N);
    HPC_REQUIRE(N < (int64_t(1) << 30), "%s: N too large (%lld)", what, (long long)N);
    return HPC_RLL_OK;
}

}  // namespace hpcrll

extern "C" {

int hpc_rll_importance_weights_forward(const float* target_output, const float* behaviour_output,
                                       const int64_t* action, float* rho, int64_t R, int64_t N, void* stream_) {
    HPC_NVTX("importance_weights_forward");
    using namespace hpcrll;
    if (int rc = check_sizes("importance_weights_forward", R, N)) return rc;
    if (R == 0) return HPC_RLL_OK;
    HPC_REQUIRE(target_output && behaviour_output && action && rho,
                "importance_weights_forward: null target_output, behaviour_output, action or rho pointer");
    unsigned grid;
    return launch_rows<ImportanceRows>(&grid, R, N, target_output, behaviour_output, as_stream(stream_), target_output,
                                       behaviour_output, action, rho);
}

int hpc_rll_importance_weights_backward(const float* grad_rho, const float* target_output,
                                        const float* behaviour_output, const int64_t* action, const float* rho,
                                        float* grad_target_output, float* grad_behaviour_output, int64_t R, int64_t N,
                                        void* workspace, size_t workspace_bytes, void* stream_) {
    HPC_NVTX("importance_weights_backward");
    using namespace hpcrll;
    if (int rc = check_sizes("importance_weights_backward", R, N)) return rc;
    if (R == 0 || (!grad_target_output && !grad_behaviour_output)) return HPC_RLL_OK;
    HPC_REQUIRE(grad_rho && action && rho && workspace, "importance_weights_backward: null grad_rho, action, rho or "
                                                        "workspace pointer");
    HPC_REQUIRE(!grad_target_output || target_output,
                "importance_weights_backward: null target_output pointer with grad_target_output");
    HPC_REQUIRE(!grad_behaviour_output || behaviour_output,
                "importance_weights_backward: null behaviour_output pointer with grad_behaviour_output");
    HPC_REQUIRE(workspace_bytes >= importance_weights_workspace_bytes(R),
                "importance_weights_backward: workspace too small");
    const float* sign;  // {+1, -1}
    if (int rc = unit_scalars(&sign)) return rc;
    cudaStream_t stream = as_stream(stream_);
    float* c = static_cast<float*>(workspace);
    importance_grad_coef<<<rows_grid(R, 256), 256, 0, stream>>>(grad_rho, rho, c, R);
    count_launch();
    HPC_LAUNCH_CHECK();
    if (grad_target_output)
        if (int rc = launch_softmax_grad_rows(target_output, action, c, nullptr, sign, nullptr, 0.0,
                                              grad_target_output, R, N, stream))
            return rc;
    if (grad_behaviour_output)
        return launch_softmax_grad_rows(behaviour_output, action, c, nullptr, sign + 1, nullptr, 0.0,
                                        grad_behaviour_output, R, N, stream);
    return HPC_RLL_OK;
}

}  // extern "C"
