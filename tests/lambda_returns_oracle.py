"""Oracle of the λ-returns (``hpc_rll.rl_utils.td.generalized_lambda_returns`` / ``multistep_forward_view``): a numpy
restatement of the formula, forward and adjoint.

With dtype=np.float32 every operation is one rounded fp32 numpy operation in the order below, which is what eager
PyTorch does with the formula on the CPU (tests/test_lambda_returns_cpu.py pins the two to each other bit for bit, and
the done-free form to the reference's origin through tests/golden/lambda_*.npz).

    V_t = bootstrap_values[t + offset]      offset 1: generalized_lambda_returns, 0: multistep_forward_view
    γ_t, λ_t = the (T,B) tensors, or dtype(scalar) everywhere
    d_t = γ_t·λ_t;  e_t = γ_t − d_t;  m_t = 0 where done_t != 0, else 1
    done None:  R_{T-1} = r + γ·V               R_t = (r_t + d_t·R_{t+1}) + e_t·V_t
    done given: R_{T-1} = r + (m·γ)·V           R_t = r_t + m_t·(d_t·R_{t+1} + e_t·V_t)
adjoint, G = dL/dR, from u_0 = G_0:
    done None:  u_t = G_t + u_{t-1}·d_{t-1}            grad_V_t = u_t·e_t,      grad_V_{T-1} = u_{T-1}·γ_{T-1}
    done given: u_t = G_t + (u_{t-1}·m_{t-1})·d_{t-1}  grad_V_t = (u_t·m_t)·e_t, grad_V_{T-1} = u_{T-1}·(m·γ)
    grad_rewards = u;  rows of bootstrap_values before `offset` get +0
"""
import numpy as np


def _terms(gammas, lambda_, done, shape, dtype):
    g = np.asarray(gammas, dtype=dtype) if np.ndim(gammas) else np.full(shape, dtype(gammas), dtype)
    lam = np.asarray(lambda_, dtype=dtype) if np.ndim(lambda_) else np.full(shape, dtype(lambda_), dtype)
    d = g * lam
    e = g - d
    m = None if done is None else (dtype(1) - (np.asarray(done) != 0).astype(dtype))
    return g, d, e, m


def forward(bootstrap_values, rewards, gammas, lambda_, done=None, offset=1, dtype=np.float32):
    r = np.asarray(rewards, dtype=dtype)
    V = np.asarray(bootstrap_values, dtype=dtype)[offset:]
    T = r.shape[0]
    g, d, e, m = _terms(gammas, lambda_, done, r.shape, dtype)
    R = np.empty_like(r)
    if T == 0:
        return R
    if m is None:
        R[T - 1] = r[T - 1] + g[T - 1] * V[T - 1]
        for t in range(T - 2, -1, -1):
            R[t] = (r[t] + d[t] * R[t + 1]) + e[t] * V[t]
    else:
        R[T - 1] = r[T - 1] + (m[T - 1] * g[T - 1]) * V[T - 1]
        for t in range(T - 2, -1, -1):
            R[t] = r[t] + m[t] * (d[t] * R[t + 1] + e[t] * V[t])
    return R


def backward(grad_returns, gammas, lambda_, done=None, offset=1, dtype=np.float32):
    """-> dict(bootstrap_values=..., rewards=...), the gradients of sum(grad_returns * R)"""
    G = np.asarray(grad_returns, dtype=dtype)
    T, B = G.shape
    g, d, e, m = _terms(gammas, lambda_, done, G.shape, dtype)
    u = np.empty_like(G)
    gv = np.empty_like(G)
    if T > 0:
        u[0] = G[0]
        for t in range(1, T):
            u[t] = G[t] + (u[t - 1] * d[t - 1] if m is None else (u[t - 1] * m[t - 1]) * d[t - 1])
        if m is None:
            gv[:T - 1] = u[:T - 1] * e[:T - 1]
            gv[T - 1] = u[T - 1] * g[T - 1]
        else:
            gv[:T - 1] = (u[:T - 1] * m[:T - 1]) * e[:T - 1]
            gv[T - 1] = u[T - 1] * (m[T - 1] * g[T - 1])
    gb = np.concatenate([np.zeros((offset, B), dtype), gv], axis=0)
    return {"bootstrap_values": gb, "rewards": u}
