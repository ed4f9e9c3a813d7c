"""Oracle of the importance weights and the time-batch cross entropy (``hpc_rll.rl_utils.vtrace.compute_importance_weights``
/ ``hpc_rll.rl_utils.upgo.tb_cross_entropy``): a numpy restatement of the formulas in fp64, forward and adjoint.
tests/test_importance_weights_cpu.py pins it to the reference's origin through tests/golden/importance_*.npz.

Per row x of N logits with chosen action a, m = max x, s = Σ exp(x − m), p = exp(x − m) / s; -inf logits give p = 0:
    log-prob       lp = x[a] − m − log s
    importance     ρ = exp(lp_target − lp_behaviour)
                   ∂/∂target[k] = G·ρ·(1[k=a] − p_target[k]),   ∂/∂behaviour[k] = −G·ρ·(1[k=a] − p_behaviour[k])
    cross entropy  out = lp,   ∂/∂x[k] = G·(1[k=a] − p[k])
Inputs are (*, N) logits and (*) actions; G has the shape of the output.
"""
import numpy as np


def _rows(logits, action):
    x = np.asarray(logits, np.float64)
    N = x.shape[-1]
    x = x.reshape(-1, N)
    a = np.asarray(action).reshape(-1)
    m = x.max(axis=1, keepdims=True)
    e = np.exp(x - m)  # exp(-inf) = 0
    s = e.sum(axis=1, keepdims=True)
    p = e / s
    lp = x[np.arange(x.shape[0]), a] - m[:, 0] - np.log(s[:, 0])
    onehot = np.zeros_like(x)
    onehot[np.arange(x.shape[0]), a] = 1.0
    return lp, onehot - p


def log_prob(logits, action):
    """the chosen action's log-softmax, shape of `action`"""
    return _rows(logits, action)[0].reshape(np.shape(action))


def importance_weights(target_output, behaviour_output, action, grad=None):
    """-> dict(out, and with `grad`: grad_target_output, grad_behaviour_output)"""
    lt, dt = _rows(target_output, action)
    lb, db = _rows(behaviour_output, action)
    rho = np.exp(lt - lb)
    out = dict(out=rho.reshape(np.shape(action)))
    if grad is not None:
        c = (np.asarray(grad, np.float64).reshape(-1) * rho)[:, None]
        out["grad_target_output"] = (c * dt).reshape(np.shape(target_output))
        out["grad_behaviour_output"] = (-c * db).reshape(np.shape(behaviour_output))
    return out


def tb_cross_entropy(logit, label, grad=None):
    """-> dict(out, and with `grad`: grad_logit); `logit` holds label.size rows of N"""
    lp, d = _rows(logit, label)
    out = dict(out=lp.reshape(np.shape(label)))
    if grad is not None:
        out["grad_logit"] = (np.asarray(grad, np.float64).reshape(-1, 1) * d).reshape(np.shape(logit))
    return out
