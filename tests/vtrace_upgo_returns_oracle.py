"""Oracle of the V-trace target and the UPGO return (``hpc_rll.rl_utils.vtrace.vtrace_nstep_return`` /
``hpc_rll.rl_utils.upgo.upgo_returns``): a numpy restatement of the formulas, forward and adjoint.

With dtype=np.float32 every operation is one rounded fp32 numpy operation in the order below, which is the order of the
reference's origin (tests/test_vtrace_upgo_returns_cpu.py pins the two to each other through
tests/golden/returns_*.npz).  V_t = bootstrap_values[t], t = 0..T; G = dL/dR.

V-trace, g = dtype(γ), f = dtype(γ·λ) with the product taken in double:
    a_t = (r_t + g·V_{t+1}) − V_t     item_T = +0     item_t = ρ_t·a_t + (f·c_t)·item_{t+1}     R_t = V_t + item_t
    adjoint: w_0 = G_0, w_t = G_t + (f·c_{t−1})·w_{t−1}, p_t = w_t·ρ_t
             grad_reward = p, grad_V_0 = G_0 − p_0, grad_V_t = (G_t − p_t) + g·p_{t−1}, grad_V_T = g·p_{T−1}
UPGO, ℓ_t = [r_{t+1} + V_{t+2} >= V_{t+1}] for t < T−1 (NaN compares false), ℓ_{T−1} = 0:
    R_{T−1} = r_{T−1} + V_T           R_t = (r_t + ℓ_t·R_{t+1}) + (1 − ℓ_t)·V_{t+1}
    adjoint: u_0 = G_0, u_t = G_t + ℓ_{t−1}·u_{t−1}; grad_rewards = u, grad_V_{t+1} = u_t·(1 − ℓ_t), grad_V_0 = +0
"""
import numpy as np


def vtrace_forward(clipped_rhos, clipped_cs, reward, bootstrap_values, gamma=0.99, lambda_=0.95, dtype=np.float32):
    rho, c = np.asarray(clipped_rhos, dtype), np.asarray(clipped_cs, dtype)
    r, V = np.asarray(reward, dtype), np.asarray(bootstrap_values, dtype)
    g, f = dtype(gamma), dtype(gamma * lambda_)
    R = np.empty_like(r)
    item = np.zeros(r.shape[1:], dtype)
    with np.errstate(all="ignore"):
        for t in range(r.shape[0] - 1, -1, -1):
            item = rho[t] * ((r[t] + g * V[t + 1]) - V[t]) + (f * c[t]) * item
            R[t] = V[t] + item
    return R


def vtrace_backward(grad_returns, clipped_rhos, clipped_cs, gamma=0.99, lambda_=0.95, dtype=np.float32):
    """-> dict(reward=..., bootstrap_values=...), the gradients of sum(grad_returns * R)"""
    G = np.asarray(grad_returns, dtype)
    rho, c = np.asarray(clipped_rhos, dtype), np.asarray(clipped_cs, dtype)
    g, f = dtype(gamma), dtype(gamma * lambda_)
    T, B = G.shape
    p = np.empty_like(G)
    gv = np.zeros((T + 1, B), dtype)
    with np.errstate(all="ignore"):
        w = None
        for t in range(T):
            w = G[t] if t == 0 else G[t] + (f * c[t - 1]) * w
            p[t] = w * rho[t]
        if T > 0:
            gv[0] = G[0] - p[0]
            gv[1:T] = (G[1:] - p[1:]) + g * p[:-1]
            gv[T] = g * p[T - 1]
    return {"reward": p, "bootstrap_values": gv}


def upgo_mask(rewards, bootstrap_values, dtype=np.float32):
    """ℓ as 0/1 of `dtype`, (T, B), last row 0"""
    r, V = np.asarray(rewards, dtype), np.asarray(bootstrap_values, dtype)
    lam = np.zeros_like(r)
    with np.errstate(all="ignore"):
        lam[:-1] = ((r[1:] + V[2:]) >= V[1:-1]).astype(dtype)
    return lam


def upgo_forward(rewards, bootstrap_values, dtype=np.float32):
    r, V = np.asarray(rewards, dtype), np.asarray(bootstrap_values, dtype)
    lam = upgo_mask(r, V, dtype)
    T = r.shape[0]
    R = np.empty_like(r)
    if T == 0:
        return R
    with np.errstate(all="ignore"):
        R[T - 1] = r[T - 1] + V[T]
        for t in range(T - 2, -1, -1):
            R[t] = (r[t] + lam[t] * R[t + 1]) + (dtype(1) - lam[t]) * V[t + 1]
    return R


def upgo_backward(grad_returns, lam, dtype=np.float32):
    """`lam`: the mask of upgo_mask -> dict(rewards=..., bootstrap_values=...)"""
    G = np.asarray(grad_returns, dtype)
    lam = (np.asarray(lam) != 0).astype(dtype)
    T, B = G.shape
    u = np.empty_like(G)
    gv = np.zeros((T + 1, B), dtype)
    with np.errstate(all="ignore"):
        for t in range(T):
            u[t] = G[t] if t == 0 else G[t] + lam[t - 1] * u[t - 1]
        gv[1:] = u * (dtype(1) - lam)
    return {"rewards": u, "bootstrap_values": gv}
