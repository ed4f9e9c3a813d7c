// softmax_rows.cu -- the softmax-gradient row kernel shared by V-trace, UPGO and PPO backward, and
// the fixed-order loss finaliser.  See softmax_rows.cuh for the design.
//
// Replaces vtraceBackwardTargetOutput (include/hpc/rll/cuda/rl_utils/vtrace_kernel.h:235-273),
// upgoBackwardKernel (upgo_kernel.h:96-108) and ppoBackwardLogitsNew (ppo_kernel.h:252-283), which
// re-read (T,B,N) buffers saved by the forward; here the softmax is recomputed from the logits.
#include <atomic>

#include "softmax_rows.cuh"

namespace hpcrll {

// The backward writes a whole row where the forwards reduce it to scalars, so it keeps its own three kernels.  They
// always carry the entropy term; a caller without one passes a zero coefficient (launch_softmax_grad_rows).

// G1: one lane per row known at compile time (G == 1, N == KMAX * WIDTH): see HPC_ROWS_FWD_REGS
template <int KMAX, int WIDTH, bool G1>
__global__ void __launch_bounds__(256) softmax_grad_rows_kernel(const float* __restrict__ logits,
                                                                 const int64_t* __restrict__ action,
                                                                 const float* __restrict__ c1,
                                                                 const float* __restrict__ w,
                                                                 const float* __restrict__ g1,
                                                                 const float* __restrict__ g2, float inv_n,
                                                                 float* __restrict__ grad, int64_t R, int N_, int G_,
                                                                 int log2G_) {
    using Row = RowRegs<KMAX, WIDTH>;
    constexpr int W = Row::W;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = G1 ? KMAX * WIDTH : N_, G = G1 ? 1 : G_, log2G = G1 ? 0 : log2G_;
    const int lig = G1 ? 0 : (lane & (G - 1)), gw = lane >> log2G;
    const int rows_per_warp = 32 >> log2G;
    const int rows_per_block = rows_per_warp * 8;
    const float s1 = __ldg(g1);
    const float s2 = __ldg(g2) * inv_n;
    // software pipeline (small rows only): the next row block's loads fly while this one is reduced
    constexpr bool PF = Row::NE <= 8;
    Row rr, nx;
    // row index and row pointers advance by increments (no 64-bit multiply per row)
    const int64_t stride = static_cast<int64_t>(gridDim.x) * rows_per_block;
    int64_t base = static_cast<int64_t>(blockIdx.x) * rows_per_block;
    int64_t row = base + warp * rows_per_warp + gw;
    const float* pl = logits + row * N;
    float* pg = grad + row * N;
    const int64_t pstep = stride * N;
    rr.load(pl, N, G, lig, row < R);
    for (; base < R; base += stride, row += stride, pg += pstep) {  // block-uniform trip count
        const bool active = row < R;
        const int64_t nrow = row + stride;
        pl += pstep;
        if (PF) nx.load(pl, N, G, lig, nrow < R);
        const int a = active ? static_cast<int>(action[row]) : -1;
        const float c = active ? s1 * c1[row] : 0.f;
        const float e2 = s2 * ((w && active) ? w[row] : 1.f);
        const float m = rr.row_max(G);
        float s, t, e[Row::NE];
        rr.template stats<true, true>(G, m, s, t, e);
        const float logs = logf(s), inv_s = 1.f / s;
        const float H = logs - t * inv_s;  // = -sum p log p
#pragma unroll
        for (int j = 0; j < KMAX; ++j) {
            float o[W];
#pragma unroll
            for (int q = 0; q < W; ++q) {
                const int i = j * W + q;
                const int idx = rr.index(j, q, G, lig);
                const float p = e[i] * inv_s;
                float gq = c * ((idx == a ? 1.f : 0.f) - p);
                gq += e2 * (-p * (fmaxf(row_logp<true>(rr.x[i], m, logs), kNegBig) + H));
                o[q] = gq;
            }
            const int e0 = rr.index(j, 0, G, lig);
            if (active && e0 < N) {
                if (W == 4)
                    st_stream4(reinterpret_cast<float4*>(pg + e0),
                               make_float4(o[0], o[W > 1 ? 1 : 0], o[W > 2 ? 2 : 0], o[W > 3 ? 3 : 0]));
                else if (W == 2)
                    st_stream2(reinterpret_cast<float2*>(pg + e0), make_float2(o[0], o[W > 1 ? 1 : 0]));
                else
                    st_stream(pg + e0, o[0]);
            }
        }
        if (PF) rr = nx;
        else rr.load(pl, N, G, lig, nrow < R);
    }
}

// Staged variant (N <= 32, not 128-bit eligible): see softmax_rows.cuh "Staged rows".
__global__ void __launch_bounds__(kStageRows) softmax_grad_rows_staged_kernel(
    const float* __restrict__ logits, const int64_t* __restrict__ action, const float* __restrict__ c1,
    const float* __restrict__ w, const float* __restrict__ g1, const float* __restrict__ g2, float inv_n,
    float* __restrict__ grad, int64_t R, int N, int P, int aligned) {
    extern __shared__ float tile[];
    const float s1 = __ldg(g1);
    const float s2 = __ldg(g2) * inv_n;
    const int64_t ntiles = (R + kStageRows - 1) / kStageRows;
    for (int64_t tix = blockIdx.x; tix < ntiles; tix += gridDim.x) {
        const int64_t row0 = tix * kStageRows, row = row0 + threadIdx.x;
        __syncthreads();  // the previous tile has been written back
        stage_rows(logits, R, N, P, row0, tile, aligned != 0);
        __syncthreads();
        if (row < R) {
            float* x = tile + threadIdx.x * P;
            float m, s, t;
            staged_stats<true>(x, N, m, s, t);
            const float logs = logf(s), inv_s = 1.f / s;
            const float H = logs - t * inv_s;
            const int a = static_cast<int>(action[row]);
            const float c = s1 * c1[row];
            const float e2 = s2 * (w ? w[row] : 1.f);
            for (int k = 0; k < N; ++k) {
                const float xv = x[k];
                const float p = exp_term(fmaxf(xv - m, kNegBig)) * inv_s;
                float gq = c * ((k == a ? 1.f : 0.f) - p);
                gq += e2 * (-p * (fmaxf(row_logp<true>(xv, m, logs), kNegBig) + H));
                x[k] = gq;
            }
        }
        __syncthreads();
        unstage_rows(grad, R, N, P, row0, tile, aligned != 0);
    }
}

// N too large for the register-resident path: one warp per row, strided passes over the row.
__global__ void __launch_bounds__(256) softmax_grad_rows_loop_kernel(const float* __restrict__ logits,
                                                                      const int64_t* __restrict__ action,
                                                                      const float* __restrict__ c1,
                                                                      const float* __restrict__ w,
                                                                      const float* __restrict__ g1,
                                                                      const float* __restrict__ g2, float inv_n,
                                                                      float* __restrict__ grad, int64_t R, int N) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float s1 = __ldg(g1);
    const float s2 = __ldg(g2) * inv_n;
    for (int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + warp; row < R; row += static_cast<int64_t>(gridDim.x) * 8) {
        const float* x = logits + row * N;
        float m = -INFINITY;
        for (int k = lane; k < N; k += 32) m = fmaxf(m, x[k]);
        m = warp_max(m);
        float s = 0.f;
        for (int k = lane; k < N; k += 32) s += exp_term(x[k] - m);
        s = warp_sum(s);
        const float logs = logf(s);
        float H = 0.f;
        {
            float h = 0.f;
            for (int k = lane; k < N; k += 32) {
                const float l = fmaxf(row_logp<true>(x[k], m, logs), kNegBig);  // -inf logits: 0 * -3e38, not NaN
                h += exp_term(l) * l;
            }
            H = -warp_sum(h);
        }
        const int a = static_cast<int>(action[row]);
        const float c = s1 * c1[row];
        const float e2 = s2 * (w ? w[row] : 1.f);
        for (int k = lane; k < N; k += 32) {
            const float l = fmaxf(row_logp<true>(x[k], m, logs), kNegBig);  // p = 0 and a finite l for -inf logits
            const float p = exp_term(l);
            float gq = c * ((k == a ? 1.f : 0.f) - p);
            gq += e2 * (-p * (l + H));
            grad[row * N + k] = gq;
        }
    }
}

struct GradRows {
    template <int K, int W, bool G1>
    static auto reg() { return softmax_grad_rows_kernel<K, W, G1>; }
    static auto staged() { return softmax_grad_rows_staged_kernel; }
    static auto loop() { return softmax_grad_rows_loop_kernel; }
    static constexpr int kStagedTiles = 1;
};

int launch_softmax_grad_rows(const float* logits, const int64_t* action, const float* c1, const float* w,
                             const float* g1, const float* g2, double inv_n, float* grad, int64_t R, int64_t N,
                             cudaStream_t stream) {
    if (R <= 0 || N <= 0) return HPC_RLL_OK;
    HPC_REQUIRE(N < (int64_t(1) << 30), "softmax rows: N too large");
    unsigned grid;
    if (g2 != nullptr)
        return launch_rows<GradRows>(&grid, R, N, logits, grad, stream, logits, action, c1, w, g1, g2,
                                     static_cast<float>(inv_n), grad);
    // The no-entropy gradient (UPGO backward) runs through the same kernels with a zero entropy coefficient
    // (g2 := g1, inv_n := 0  =>  s2 = 0, every entropy term is 0 * finite): a lighter kernel without the entropy term was
    // measured SLOWER on the same traffic: the extra arithmetic spaces the loads and stores of a row out.  Results are
    // bit-identical.
    return launch_rows<GradRows>(&grid, R, N, logits, grad, stream, logits, action, c1, static_cast<const float*>(nullptr),
                                 g1, g1, 0.f, grad);
}

__device__ float g_unit_scalars[2] = {1.f, -1.f};

int unit_scalars(const float** out) {
    constexpr int kMaxDevices = 64;
    static std::atomic<const float*> cache[kMaxDevices] = {};
    int dev = 0;
    HPC_CUDA(cudaGetDevice(&dev));
    if (dev < kMaxDevices && (*out = cache[dev].load(std::memory_order_acquire)) != nullptr) return HPC_RLL_OK;
    void* p = nullptr;
    HPC_CUDA(cudaGetSymbolAddress(&p, g_unit_scalars));
    *out = static_cast<const float*>(p);
    if (dev < kMaxDevices) cache[dev].store(*out, std::memory_order_release);
    return HPC_RLL_OK;
}

// ---- fixed-order finaliser for several loss terms with different partial counts ---------------------
__global__ void __launch_bounds__(256) finalize_terms_kernel(const double* __restrict__ partials,
                                                              const __grid_constant__ FinSpec spec, int nterms,
                                                              float* __restrict__ out) {
    // One CTA per TERM (this kernel sits on the critical path of every loss op, and a single CTA walking up to five
    // lists of ~2400 partials with dependent loads took 13.9 us in the serialised ncu list).  Per term the summation
    // order is unchanged -- thread t adds i = t, t+256, ... in order, then the same shuffle tree -- so results are
    // bit-identical to the single-CTA version.
    __shared__ double scratch[32];
    const int k = blockIdx.x;
    if (k >= nterms) return;
    const double* p = partials + spec.off[k];
    const int n = spec.cnt[k];
    double a = 0.0;
    for (int i0 = threadIdx.x; i0 < n; i0 += 256 * 4) {  // four loads in flight, adds in the original order
        double x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) x[u] = __ldcg(p + min(i0 + u * 256, n - 1));  // clamped index: no predicate
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (i0 + u * 256 < n) a += x[u];
    }
    double v[1] = {a};
    block_sum<1>(v, scratch);
    if (threadIdx.x == 0) out[k] = static_cast<float>(v[0] * spec.scale[k]);
}

int launch_finalize_terms(const double* partials, const FinSpec& spec, int nterms, float* out,
                          cudaStream_t stream) {
    finalize_terms_kernel<<<nterms, 256, 0, stream>>>(partials, spec, nterms, out);
    count_launch();
    HPC_LAUNCH_CHECK();
    return HPC_RLL_OK;
}

}  // namespace hpcrll
