// legacy.cpp -- the reference's native boundary: the 19 hot-path entry points of the pybind module `hpc_rl_utils`
// and the two ScatterConnection entry points of `hpc_torch_utils_network` (in the submodule `_torch_utils_network`)
// (/root/reference/src/rl_utils/entry.cpp:20-38, declared in include/hpc/rll/cuda/rl_utils/entry.h:62-165), with the
// SAME names, the same `(inputs: List[Tensor], outputs: List[Tensor], float...)` shape and the same positional tensor
// order as each reference launcher (src/rl_utils/*.cu, `index++` unpacking), implemented on top of the C ABI.
// With this module importable as `hpc_rl_utils` the UNMODIFIED reference wrappers (hpc_rll/rl_utils/*.py) run on these
// kernels: tests/test_legacy_shim_*.py call every name in the reference's argument layout and compare with the oracle.
//
// The reference kernels communicate between Forward and Backward through module-owned scratch tensors that the Python
// wrapper merely hands back (e.g. vtrace.py:25-28: `bp_inputs = [value, action, weight, returns, advantages,
// target_output_grad_logits, target_output_grad_prob, target_output_grad_entropy]`).  Those buffers are opaque to the
// wrapper, so the shim keeps their SHAPES and stores what its own backward needs in them:
//   V-trace  `target_output_grad_logits` (T,B,N) <- copy of the logits (our backward recomputes the softmax);
//            `advantages` (T,B) <- pg_coef = -adv*w/n;  `returns` (T,B) <- gv_buf = 2(v-ret)w/n
//   UPGO     `grad_buf` (T,B,N) <- d loss / d logits at upstream gradient 1 (backward = scale by grad_loss);
//            `advantage` (T,B) <- -adv/n
//   PPO      `logits_new_grad_prob` (B,N) <- d policy_loss / d logits,  `logits_new_grad_entropy` (B,N) <- d entropy_loss /
//            d logits, `grad_value_loss_buf` (B) <- d value_loss / d value  (backward = linear combination, hpc_rll_axpby)
//   C51      `buf` (B + B*n_atom): our (B,n_atom) grad_buf sits in its tail, where the reference keeps the projection
//   IQN      `grad_buf` (B,tau',tau): our (tau,B) grad_buf occupies its first tau*B floats
// Everything else the reference lists as output (probabilities, importance weights, bellman / huber scratch) is
// accepted and left untouched.  Reference defects are not reproduced (SURVEY.md 0.4 #5-7): B is not limited to 65535,
// the QR-DQN (B,tau) grad_buf is not overrun, and TD-lambda's default (B,) weight is broadcast instead of read out of
// bounds.
#include "common.h"

namespace hpcrl {
namespace {

using TL = std::vector<Tensor>;

void need(const TL& v, size_t n, const char* what) {
    TORCH_CHECK(v.size() >= n, what, ": expected at least ", n, " tensors, got ", v.size());
}

// dense fp32 view of a caller-owned OUTPUT tensor (the reference writes through raw pointers; outputs are module buffers)
float* outp(Tensor& t, const char* name, int64_t min_numel) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == torch::kFloat32 && t.is_contiguous(), name,
                " must be a contiguous float32 CUDA tensor");
    TORCH_CHECK(t.numel() >= min_numel, name, " holds ", t.numel(), " elements, needs ", min_numel);
    return t.data_ptr<float>();
}

Tensor weight_or_none(const Tensor& w, int64_t numel) {  // reference passes ones when the caller gave None
    if (!w.defined() || w.numel() == 0) return Tensor();
    Tensor c = f32(w, "weight");
    TORCH_CHECK(c.numel() == numel, "weight holds ", c.numel(), " elements, expected ", numel);
    return c;
}

Tensor one_like(const Tensor& like) { return torch::ones({1}, like.options().dtype(torch::kFloat32)); }

// ---- gae (gae.cu:8-28) -----------------------------------------------------------------------------------------
void GaeForward(const TL& in, TL& out, float gamma, float lambda) {
    need(in, 2, "GaeForward inputs");
    need(out, 1, "GaeForward outputs");
    const Tensor value = f32(in[0], "value"), reward = f32(in[1], "reward");
    const int64_t T = reward.size(0), B = reward.size(1);
    c10::cuda::CUDAGuard guard(reward.device());
    ck(hpc_rll_gae_forward(fp(value), fp(reward), outp(out[0], "adv", T * B), T, B, gamma, lambda, cur_stream()),
       "hpc_rll_gae_forward");
}

// ---- td_lambda (td_lambda.cu:8-52) -----------------------------------------------------------------------------
void TdLambdaForward(const TL& in, TL& out, float gamma, float lambda) {
    need(in, 3, "TdLambdaForward inputs");
    need(out, 2, "TdLambdaForward outputs");
    const Tensor value = f32(in[0], "value"), reward = f32(in[1], "reward");
    const int64_t T = reward.size(0), B = reward.size(1);
    Tensor weight = f32(in[2], "weight");
    if (weight.numel() == B && T != 1) weight = weight.reshape({1, B}).expand({T, B}).contiguous();  // rl_utils/td.py:160
    TORCH_CHECK(weight.numel() == T * B, "weight must be (T, B) or (B,)");
    c10::cuda::CUDAGuard guard(reward.device());
    Tensor ws = workspace(HPC_RLL_OP_TD_LAMBDA, T, B, 0, reward);
    ck(hpc_rll_td_lambda_forward(fp(value), fp(reward), fp(weight), outp(out[0], "loss", 1),
                                 outp(out[1], "grad_buf", T * B), T, B, gamma, lambda, 0, ws.data_ptr(), ws.numel(),
                                 cur_stream()),
       "hpc_rll_td_lambda_forward");
}

void TdLambdaBackward(const TL& in, TL& out) {
    need(in, 2, "TdLambdaBackward inputs");
    need(out, 1, "TdLambdaBackward outputs");
    const Tensor gbuf = f32(in[1], "grad_buf");
    const int64_t T = gbuf.size(0), B = gbuf.size(1);
    c10::cuda::CUDAGuard guard(gbuf.device());
    const Tensor g = gscalar(in[0], gbuf);
    ck(hpc_rll_td_lambda_backward(fp(g), fp(gbuf), outp(out[0], "grad_value", (T + 1) * B), T, B, cur_stream()),
       "hpc_rll_td_lambda_backward");
}

// ---- q_nstep_td / rescale (q_nstep_td.cu:8-64) -----------------------------------------------------------------
void q_forward(const TL& in, TL& out, float gamma, int rescale) {
    need(in, 7, "QNStepTdForward inputs");
    need(out, 3, "QNStepTdForward outputs");
    const Tensor q = f32(in[0], "q"), nq = f32(in[1], "next_n_q"), a = i64(in[2], "action"), na = i64(in[3], "next_n_action");
    const Tensor reward = f32(in[4], "reward"), done = f32(in[5], "done");
    const int64_t B = q.size(0), N = q.size(1), T = reward.size(0);
    const Tensor w = weight_or_none(in[6], B);
    c10::cuda::CUDAGuard guard(q.device());
    Tensor ws = workspace(HPC_RLL_OP_Q_NSTEP_TD, T, B, N, q);
    ck(hpc_rll_q_nstep_td_forward(fp(q), fp(nq), ip(a), ip(na), fp(reward), fp(done), fp(w), outp(out[1], "loss", 1),
                                  outp(out[0], "td_err", B), outp(out[2], "grad_buf", B), T, B, N, gamma, rescale, 0,
                                  ws.data_ptr(), ws.numel(), cur_stream()),
       "hpc_rll_q_nstep_td_forward");
}
void QNStepTdForward(const TL& in, TL& out, float gamma) { q_forward(in, out, gamma, 0); }
void QNStepTdRescaleForward(const TL& in, TL& out, float gamma) { q_forward(in, out, gamma, 1); }

void QNStepTdBackward(const TL& in, TL& out) {
    need(in, 3, "QNStepTdBackward inputs");
    need(out, 1, "QNStepTdBackward outputs");
    const Tensor gbuf = f32(in[1], "grad_buf"), a = i64(in[2], "action");
    const int64_t B = a.size(0);
    TORCH_CHECK(out[0].dim() == 2 && out[0].size(0) == B, "grad_q must be (B, N)");
    const int64_t N = out[0].size(1);
    c10::cuda::CUDAGuard guard(gbuf.device());
    const Tensor g = gscalar(in[0], gbuf);
    ck(hpc_rll_q_nstep_td_backward(fp(g), fp(gbuf), ip(a), outp(out[0], "grad_q", B * N), B, N, cur_stream()),
       "hpc_rll_q_nstep_td_backward");
}

// ---- dist_nstep_td (dist_nstep_td.cu:8-98) ---------------------------------------------------------------------
void DistNStepTdForward(const TL& in, TL& out, float gamma, float v_min, float v_max) {
    need(in, 7, "DistNStepTdForward inputs");
    need(out, 3, "DistNStepTdForward outputs");
    const Tensor dist = f32(in[0], "dist"), ndist = f32(in[1], "next_n_dist"), a = i64(in[2], "action");
    const Tensor na = i64(in[3], "next_n_action"), reward = f32(in[4], "reward"), done = f32(in[5], "done");
    const int64_t B = dist.size(0), N = dist.size(1), n_atom = dist.size(2), T = reward.size(0);
    const Tensor w = weight_or_none(in[6], B);
    c10::cuda::CUDAGuard guard(dist.device());
    float* buf = outp(out[2], "buf", B + B * n_atom);  // [0,B): n-step reward in the reference; [B, ...): projection / grad
    Tensor ws = workspace(HPC_RLL_OP_DIST_NSTEP_TD, T, B, N, dist);
    ck(hpc_rll_dist_nstep_td_forward(fp(dist), fp(ndist), ip(a), ip(na), fp(reward), fp(done), fp(w),
                                     outp(out[1], "loss", 1), outp(out[0], "td_err", B), buf + B, T, B, N, n_atom, gamma,
                                     v_min, v_max, 0, ws.data_ptr(), ws.numel(), cur_stream()),
       "hpc_rll_dist_nstep_td_forward");
}

void DistNStepTdBackward(const TL& in, TL& out) {
    need(in, 3, "DistNStepTdBackward inputs");
    need(out, 1, "DistNStepTdBackward outputs");
    const Tensor buf = f32(in[1], "buf"), a = i64(in[2], "action");
    TORCH_CHECK(out[0].dim() == 3, "grad_dist must be (B, N, n_atom)");
    const int64_t B = out[0].size(0), N = out[0].size(1), n_atom = out[0].size(2);
    TORCH_CHECK(buf.numel() >= B + B * n_atom, "buf too small");
    c10::cuda::CUDAGuard guard(buf.device());
    const Tensor g = gscalar(in[0], buf);
    ck(hpc_rll_dist_nstep_td_backward(fp(g), fp(buf) + B, ip(a), outp(out[0], "grad_dist", B * N * n_atom), B, N, n_atom,
                                      cur_stream()),
       "hpc_rll_dist_nstep_td_backward");
}

// ---- qrdqn_nstep_td_error (qrdqn_nstep_td_error.cu:8-95) -------------------------------------------------------
void QRDQNNStepTDErrorForward(const TL& in, TL& out, float gamma) {
    need(in, 8, "QRDQNNStepTDErrorForward inputs");
    need(out, 5, "QRDQNNStepTDErrorForward outputs");
    const Tensor q = f32(in[0], "q"), nq = f32(in[1], "next_n_q"), a = i64(in[2], "action"), na = i64(in[3], "next_n_action");
    const Tensor reward = f32(in[4], "reward"), done = f32(in[5], "done"), vg = f32(in[7], "value_gamma");
    const int64_t B = q.size(0), N = q.size(1), tau = q.size(2), T = reward.size(0);
    const Tensor w = weight_or_none(in[6], B);
    c10::cuda::CUDAGuard guard(q.device());
    Tensor ws = workspace(HPC_RLL_OP_QRDQN_NSTEP_TD, T, B, N, q);
    ck(hpc_rll_qrdqn_nstep_td_forward(fp(q), fp(nq), ip(a), ip(na), fp(reward), fp(done), fp(w), fp(vg),
                                      outp(out[0], "loss", 1), outp(out[1], "td_err", B), outp(out[4], "grad_buf", B * tau),
                                      tau, T, B, N, gamma, 0, ws.data_ptr(), ws.numel(), cur_stream()),
       "hpc_rll_qrdqn_nstep_td_forward");
}

void QRDQNNStepTDErrorBackward(const TL& in, TL& out) {
    need(in, 4, "QRDQNNStepTDErrorBackward inputs");  // grad_loss, grad_buf, weight (already folded in), action
    need(out, 1, "QRDQNNStepTDErrorBackward outputs");
    const Tensor gbuf = f32(in[1], "grad_buf"), a = i64(in[3], "action");
    TORCH_CHECK(out[0].dim() == 3, "grad_q must be (B, N, tau)");
    const int64_t B = out[0].size(0), N = out[0].size(1), tau = out[0].size(2);
    c10::cuda::CUDAGuard guard(gbuf.device());
    const Tensor g = gscalar(in[0], gbuf);
    ck(hpc_rll_qrdqn_nstep_td_backward(fp(g), fp(gbuf), ip(a), outp(out[0], "grad_q", B * N * tau), tau, B, N,
                                       cur_stream()),
       "hpc_rll_qrdqn_nstep_td_backward");
}

// ---- iqn_nstep_td_error (iqn_nstep_td_error.cu:8-100) ----------------------------------------------------------
void IQNNStepTDErrorForward(const TL& in, TL& out, float gamma, float kappa) {
    need(in, 9, "IQNNStepTDErrorForward inputs");
    need(out, 5, "IQNNStepTDErrorForward outputs");
    const Tensor q = f32(in[0], "q"), nq = f32(in[1], "next_n_q"), a = i64(in[2], "action"), na = i64(in[3], "next_n_action");
    const Tensor reward = f32(in[4], "reward"), done = f32(in[5], "done"), rq = f32(in[6], "replay_quantiles");
    const Tensor vg = f32(in[8], "value_gamma");
    const int64_t tau = q.size(0), B = q.size(1), N = q.size(2), tau_p = nq.size(0), T = reward.size(0);
    const Tensor w = weight_or_none(in[7], B);
    c10::cuda::CUDAGuard guard(q.device());
    Tensor ws = workspace(HPC_RLL_OP_IQN_NSTEP_TD, T, B, N, q);
    ck(hpc_rll_iqn_nstep_td_forward(fp(q), fp(nq), ip(a), ip(na), fp(reward), fp(done), fp(rq), fp(w), fp(vg),
                                    outp(out[0], "loss", 1), outp(out[1], "td_err", B), outp(out[4], "grad_buf", tau * B),
                                    tau, tau_p, T, B, N, gamma, kappa, 0, ws.data_ptr(), ws.numel(), cur_stream()),
       "hpc_rll_iqn_nstep_td_forward");
}

void IQNNStepTDErrorBackward(const TL& in, TL& out) {
    need(in, 4, "IQNNStepTDErrorBackward inputs");
    need(out, 1, "IQNNStepTDErrorBackward outputs");
    const Tensor gbuf = f32(in[1], "grad_buf"), a = i64(in[3], "action");
    TORCH_CHECK(out[0].dim() == 3, "grad_q must be (tau, B, N)");
    const int64_t tau = out[0].size(0), B = out[0].size(1), N = out[0].size(2);
    c10::cuda::CUDAGuard guard(gbuf.device());
    const Tensor g = gscalar(in[0], gbuf);
    ck(hpc_rll_iqn_nstep_td_backward(fp(g), fp(gbuf), ip(a), outp(out[0], "grad_q", tau * B * N), tau, B, N, cur_stream()),
       "hpc_rll_iqn_nstep_td_backward");
}

// ---- upgo (upgo.cu:8-69) ---------------------------------------------------------------------------------------
void UpgoForward(const TL& in, TL& out) {
    need(in, 5, "UpgoForward inputs");
    need(out, 4, "UpgoForward outputs");  // advantage, metric (untouched), loss, grad_buf
    const Tensor target = f32(in[0], "target_output"), rho = f32(in[1], "rho"), a = i64(in[2], "action");
    const Tensor reward = f32(in[3], "reward"), value = f32(in[4], "value");
    const int64_t T = target.size(0), B = target.size(1), N = target.size(2);
    c10::cuda::CUDAGuard guard(target.device());
    float* coef = outp(out[0], "advantage", T * B);
    Tensor ws = workspace(HPC_RLL_OP_UPGO, T, B, N, reward);
    ck(hpc_rll_upgo_forward(fp(target), fp(rho), ip(a), fp(reward), fp(value), outp(out[2], "loss", 1), coef, T, B, N, 0,
                            ws.data_ptr(), ws.numel(), cur_stream()),
       "hpc_rll_upgo_forward");
    const Tensor one = one_like(reward);
    ck(hpc_rll_upgo_backward(fp(one), fp(target), ip(a), coef, outp(out[3], "grad_buf", T * B * N), T, B, N, cur_stream()),
       "hpc_rll_upgo_backward (unit gradient)");
}

void UpgoBackward(const TL& in, TL& out) {
    need(in, 3, "UpgoBackward inputs");  // grad_loss, grad_buf, advantage
    need(out, 1, "UpgoBackward outputs");
    const Tensor gbuf = f32(in[1], "grad_buf");
    c10::cuda::CUDAGuard guard(gbuf.device());
    const Tensor g = gscalar(in[0], gbuf);
    ck(hpc_rll_axpby(fp(g), fp(gbuf), nullptr, nullptr, outp(out[0], "grad_target_output", gbuf.numel()), gbuf.numel(),
                     cur_stream()),
       "hpc_rll_axpby");
}

// ---- vtrace (vtrace.cu:8-130) ----------------------------------------------------------------------------------
void VTraceForward(const TL& in, TL& out, float gamma, float lambda, float rho_clip, float c_clip, float rho_pg_clip) {
    need(in, 6, "VTraceForward inputs");
    need(out, 12, "VTraceForward outputs");
    const Tensor target = f32(in[0], "target_output"), behaviour = f32(in[1], "behaviour_output"), a = i64(in[2], "action");
    const Tensor value = f32(in[3], "value"), reward = f32(in[4], "reward");
    const int64_t T = target.size(0), B = target.size(1), N = target.size(2);
    const Tensor w = weight_or_none(in[5], T * B);
    c10::cuda::CUDAGuard guard(target.device());
    Tensor losses = torch::empty({3}, reward.options());
    Tensor ws = workspace(HPC_RLL_OP_VTRACE, T, B, N, reward);
    ck(hpc_rll_vtrace_forward(fp(target), fp(behaviour), ip(a), fp(value), fp(reward), fp(w), fpm(losses),
                              outp(out[8], "advantages", T * B), outp(out[7], "returns", T * B), T, B, N, gamma, lambda,
                              rho_clip, c_clip, rho_pg_clip, 0, ws.data_ptr(), ws.numel(), cur_stream()),
       "hpc_rll_vtrace_forward");
    outp(out[2], "target_output_grad_logits", T * B * N);
    out[2].view({T, B, N}).copy_(target);  // the logits, for the softmax recomputation in VTraceBackward
    for (int k = 0; k < 3; ++k) {
        outp(out[9 + k], "loss", 1);
        out[9 + k].view({1}).copy_(losses.slice(0, k, k + 1));
    }
}

void VTraceBackward(const TL& in, TL& out) {
    need(in, 11, "VTraceBackward inputs");
    need(out, 2, "VTraceBackward outputs");  // grad_value, grad_target_output
    const Tensor a = i64(in[4], "action"), gv_buf = f32(in[6], "returns"), pg_coef = f32(in[7], "advantages");
    const Tensor logits = f32(in[8], "target_output_grad_logits");
    TORCH_CHECK(logits.dim() == 3, "target_output_grad_logits must be (T, B, N)");
    const int64_t T = logits.size(0), B = logits.size(1), N = logits.size(2);
    const Tensor w = weight_or_none(in[5], T * B);
    c10::cuda::CUDAGuard guard(logits.device());
    const Tensor g0 = gscalar(in[0], pg_coef), g1 = gscalar(in[1], pg_coef), g2 = gscalar(in[2], pg_coef);
    ck(hpc_rll_vtrace_backward(fp(g0), fp(g1), fp(g2), fp(logits), ip(a), fp(w), fp(pg_coef), fp(gv_buf),
                               outp(out[1], "grad_target_output", T * B * N), outp(out[0], "grad_value", (T + 1) * B), T, B,
                               N, 0, cur_stream()),
       "hpc_rll_vtrace_backward");
}

// ---- ppo (ppo.cu:8-111) ----------------------------------------------------------------------------------------
void PPOForward(const TL& in, TL& out, bool use_value_clip, float clip_ratio, float dual_clip) {
    need(in, 8, "PPOForward inputs");
    need(out, 14, "PPOForward outputs");
    const Tensor ln = f32(in[0], "logits_new"), lo = f32(in[1], "logits_old"), a = i64(in[2], "action");
    const Tensor vn = f32(in[3], "value_new"), vo = f32(in[4], "value_old"), adv = f32(in[5], "adv"), ret = f32(in[6], "return_");
    const int64_t B = ln.size(0), N = ln.size(1);
    const Tensor w = weight_or_none(in[7], B);
    c10::cuda::CUDAGuard guard(ln.device());
    Tensor out5 = torch::empty({5}, adv.options());
    Tensor pol_coef = torch::empty({B}, adv.options()), val_coef = torch::empty({B}, adv.options());
    Tensor ws = workspace(HPC_RLL_OP_PPO, 0, B, N, adv);
    // the reference wrapper passes dual_clip = 0.0 for None and the kernel tests `dual_clip < 1` (rl_utils/ppo.py:136-137)
    ck(hpc_rll_ppo_forward(fp(ln), fp(lo), ip(a), fp(vn), fp(vo), fp(adv), fp(ret), fp(w), fpm(out5), fpm(pol_coef),
                           fpm(val_coef), B, N, clip_ratio, use_value_clip ? 1 : 0, dual_clip < 1.f ? -1.0 : dual_clip, 0,
                           ws.data_ptr(), ws.numel(), cur_stream()),
       "hpc_rll_ppo_forward");
    for (int k = 0; k < 5; ++k) {
        outp(out[9 + k], "loss/info scalar", 1);
        out[9 + k].view({1}).copy_(out5.slice(0, k, k + 1));
    }
    // gradients at unit upstream gradients: (1,1,0) -> d policy / d logits, d value / d value;  (0,0,1) -> d entropy / d logits
    const Tensor one = one_like(adv), zero = torch::zeros({1}, adv.options());
    Tensor scratch = torch::empty({B}, adv.options());
    ck(hpc_rll_ppo_backward(fp(one), fp(one), fp(zero), fp(ln), ip(a), fp(w), fp(pol_coef), fp(val_coef),
                            outp(out[3], "logits_new_grad_prob", B * N), outp(out[7], "grad_value_loss_buf", B), B, N, 0,
                            cur_stream()),
       "hpc_rll_ppo_backward (policy/value unit gradient)");
    ck(hpc_rll_ppo_backward(fp(zero), fp(zero), fp(one), fp(ln), ip(a), fp(w), fp(pol_coef), fp(val_coef),
                            outp(out[4], "logits_new_grad_entropy", B * N), fpm(scratch), B, N, 0, cur_stream()),
       "hpc_rll_ppo_backward (entropy unit gradient)");
}

void PPOBackward(const TL& in, TL& out) {
    need(in, 9, "PPOBackward inputs");
    need(out, 2, "PPOBackward outputs");  // grad_value, grad_logits_new
    const Tensor gvbuf = f32(in[4], "grad_value_loss_buf"), A = f32(in[7], "logits_new_grad_prob");
    const Tensor E = f32(in[8], "logits_new_grad_entropy");
    c10::cuda::CUDAGuard guard(A.device());
    const Tensor g0 = gscalar(in[0], A), g1 = gscalar(in[1], A), g2 = gscalar(in[2], A);
    ck(hpc_rll_axpby(fp(g0), fp(A), fp(g2), fp(E), outp(out[1], "grad_logits_new", A.numel()), A.numel(), cur_stream()),
       "hpc_rll_axpby");
    ck(hpc_rll_axpby(fp(g1), fp(gvbuf), nullptr, nullptr, outp(out[0], "grad_value", gvbuf.numel()), gvbuf.numel(),
                     cur_stream()),
       "hpc_rll_axpby");
}

// ---- scatter_connection (src/torch_utils/network/scatter_connection.cu) --------------------------------------------
// inputs {x (B,M,N), location (B,M,2)}, outputs {out (B,N,H,W)}: H and W come from the caller's output tensor
void ScatterConnectionForward(const TL& in, TL& out, const std::string& scatter_type) {
    need(in, 2, "ScatterConnectionForward inputs");
    need(out, 1, "ScatterConnectionForward outputs");
    TORCH_CHECK(scatter_type == "cover" || scatter_type == "add", "scatter_type must be 'cover' or 'add'");
    const Tensor x = f32(in[0], "input"), loc = i64(in[1], "location");
    TORCH_CHECK(x.dim() == 3 && out[0].dim() == 4, "input must be (B, M, N) and output (B, N, H, W)");
    const int64_t B = x.size(0), M = x.size(1), N = x.size(2), H = out[0].size(2), W = out[0].size(3);
    TORCH_CHECK(out[0].size(0) == B && out[0].size(1) == N, "output must be (B, N, H, W)=(", B, ", ", N, ", H, W)");
    TORCH_CHECK(loc.numel() == B * M * 2, "location must be (B, M, 2)");
    c10::cuda::CUDAGuard guard(x.device());
    ck(hpc_rll_scatter_connection_forward(fp(x), ip(loc), outp(out[0], "output", B * N * H * W), B, M, N, H, W,
                                          scatter_type == "add" ? HPC_RLL_SCATTER_ADD : HPC_RLL_SCATTER_COVER,
                                          cur_stream()),
       "hpc_rll_scatter_connection_forward");
}

// inputs {grad_out (B,N,H,W), location (B,M,2)}, outputs {grad_in (B,M,N)}
void ScatterConnectionBackward(const TL& in, TL& out) {
    need(in, 2, "ScatterConnectionBackward inputs");
    need(out, 1, "ScatterConnectionBackward outputs");
    const Tensor g = f32(in[0], "grad_out"), loc = i64(in[1], "location");
    TORCH_CHECK(g.dim() == 4 && out[0].dim() == 3, "grad_out must be (B, N, H, W) and grad_in (B, M, N)");
    const int64_t B = out[0].size(0), M = out[0].size(1), N = out[0].size(2), H = g.size(2), W = g.size(3);
    TORCH_CHECK(g.size(0) == B && g.size(1) == N, "grad_out must be (B, N, H, W)=(", B, ", ", N, ", H, W)");
    TORCH_CHECK(loc.numel() == B * M * 2, "location must be (B, M, 2)");
    c10::cuda::CUDAGuard guard(g.device());
    ck(hpc_rll_scatter_connection_backward(fp(g), ip(loc), outp(out[0], "grad_in", B * M * N), B, M, N, H, W,
                                           cur_stream()),
       "hpc_rll_scatter_connection_backward");
}

}  // namespace

void register_legacy(pybind11::module& m) {
    m.def("DistNStepTdForward", &DistNStepTdForward, "dist_nstep_td forward (CUDA)");
    m.def("DistNStepTdBackward", &DistNStepTdBackward, "dist_nstep_td backward (CUDA)");
    m.def("GaeForward", &GaeForward, "gae forward (CUDA)");
    m.def("PPOForward", &PPOForward, "ppo forward (CUDA)");
    m.def("PPOBackward", &PPOBackward, "ppo backward (CUDA)");
    m.def("QNStepTdForward", &QNStepTdForward, "q_nstep_td forward (CUDA)");
    m.def("QNStepTdBackward", &QNStepTdBackward, "q_nstep_td backward (CUDA)");
    m.def("QNStepTdRescaleForward", &QNStepTdRescaleForward, "q_nstep_td_with_rescale forward (CUDA)");
    m.def("QNStepTdRescaleBackward", &QNStepTdBackward, "q_nstep_td_with_rescale backward (CUDA)");
    m.def("TdLambdaForward", &TdLambdaForward, "td_lambda forward (CUDA)");
    m.def("TdLambdaBackward", &TdLambdaBackward, "td_lambda backward (CUDA)");
    m.def("UpgoForward", &UpgoForward, "upgo forward (CUDA)");
    m.def("UpgoBackward", &UpgoBackward, "upgo backward (CUDA)");
    m.def("VTraceForward", &VTraceForward, "vtrace forward (CUDA)");
    m.def("VTraceBackward", &VTraceBackward, "vtrace backward (CUDA)");
    m.def("IQNNStepTDErrorForward", &IQNNStepTDErrorForward, "iqn_nstep_td_error forward (CUDA)");
    m.def("IQNNStepTDErrorBackward", &IQNNStepTDErrorBackward, "iqn_nstep_td_error backward (CUDA)");
    m.def("QRDQNNStepTDErrorForward", &QRDQNNStepTDErrorForward, "qrdqn_nstep_td_error forward (CUDA)");
    m.def("QRDQNNStepTDErrorBackward", &QRDQNNStepTDErrorBackward, "qrdqn_nstep_td_error backward (CUDA)");
    // the reference's second native module, `hpc_torch_utils_network` (src/torch_utils/network/entry.cpp), as a
    // submodule so that `hpc_rl_utils` keeps exactly its own names; LstmForward / LstmBackward are not provided
    auto net = m.def_submodule("_torch_utils_network", "the reference's hpc_torch_utils_network binding names");
    net.def("ScatterConnectionForward", &ScatterConnectionForward, "scatter_connection forward (CUDA)");
    net.def("ScatterConnectionBackward", &ScatterConnectionBackward, "scatter_connection backward (CUDA)");
}

}  // namespace hpcrl
