"""Oracle of episode-aware GAE (``hpc_rll.rl_utils.gae.gae``): a numpy restatement of the formula, forward and adjoint.

The reference's ``origin`` has no such op, so this file is the reference.  With dtype=np.float32 every operation is
one rounded fp32 numpy operation in the order below, which is what eager PyTorch does with the formula on the CPU
(tests/test_gae_episodic_cpu.py pins the two to each other bit for bit); dtype=np.float64 gives the exact-arithmetic
reference the fp32 results are compared against.

    g  = dtype(gamma);  gl = dtype(gamma * lambda_)   (the product taken in double, then rounded once)
    nv_t    = next_value_t * (1 - done_t)
    delta_t = (reward_t + g * nv_t) - value_t
    f_t     = gl * (1 - traj_flag_t)
    adv_{T-1} = delta_{T-1};   adv_t = delta_t + f_t * adv_{t+1}
adjoint, G = dL/dadv:
    u_0 = G_0;   u_t = G_t + f_{t-1} * u_{t-1}
    grad_reward = u;  grad_value = -u;  grad_next_value = (g * u) * (1 - done)
Masks: non-zero = set, None = all zero; traj_flag None means traj_flag = done.
"""
import numpy as np


def _masks(done, traj_flag, shape, dtype):
    one = dtype(1)
    keep_d = np.full(shape, one, dtype) if done is None else (one - (np.asarray(done) != 0).astype(dtype))
    if traj_flag is None:
        traj_flag = done
    keep_t = np.full(shape, one, dtype) if traj_flag is None else (one - (np.asarray(traj_flag) != 0).astype(dtype))
    return keep_d, keep_t


def forward(value, next_value, reward, done=None, traj_flag=None, gamma=0.99, lambda_=0.97, dtype=np.float32):
    value, next_value, reward = (np.asarray(x, dtype=dtype) for x in (value, next_value, reward))
    T = reward.shape[0]
    g, gl = dtype(gamma), dtype(gamma * lambda_)
    keep_d, keep_t = _masks(done, traj_flag, reward.shape, dtype)
    nv = next_value * keep_d
    delta = (reward + g * nv) - value
    f = gl * keep_t
    adv = np.empty_like(delta)
    if T == 0:
        return adv
    adv[T - 1] = delta[T - 1]
    for t in range(T - 2, -1, -1):
        adv[t] = delta[t] + f[t] * adv[t + 1]
    return adv


def backward(grad_adv, done=None, traj_flag=None, gamma=0.99, lambda_=0.97, dtype=np.float32):
    """-> dict(value=..., next_value=..., reward=...), the gradients of sum(grad_adv * adv)"""
    G = np.asarray(grad_adv, dtype=dtype)
    T = G.shape[0]
    g, gl = dtype(gamma), dtype(gamma * lambda_)
    keep_d, keep_t = _masks(done, traj_flag, G.shape, dtype)
    f = gl * keep_t
    u = np.empty_like(G)
    if T > 0:
        u[0] = G[0]
        for t in range(1, T):
            u[t] = G[t] + f[t - 1] * u[t - 1]
    return {"value": -u, "next_value": (g * u) * keep_d, "reward": u}
