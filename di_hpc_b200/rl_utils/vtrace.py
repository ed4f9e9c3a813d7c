"""V-trace -- drop-in for /root/reference/hpc_rll/rl_utils/vtrace.py (VTrace, VtraceFunction,
hpc_vtrace_loss).  Same constructor ``VTrace(T, B, N)`` and forward signature (vtrace.py:83-133).
The three losses are shape-(1,) tensors as in the reference (vtrace.py:77-79)."""
from collections import namedtuple

import torch

from .. import _ext

hpc_vtrace_loss = namedtuple('hpc_vtrace_loss', ['policy_loss', 'value_loss', 'entropy_loss'])


@_ext.reference_function
def VtraceFunction(target_output, behaviour_output, action, value, reward, weight, gamma, lambda_, rho_clip_ratio,
                   c_clip_ratio, rho_pg_clip_ratio, global_B):
    return tuple(_ext.require().vtrace(target_output, behaviour_output, action, value, reward, weight, float(gamma),
                                       float(lambda_), float(rho_clip_ratio), float(c_clip_ratio),
                                       float(rho_pg_clip_ratio), int(global_B)))


class VTrace(torch.nn.Module):
    """
    Overview:
        V-trace losses (IMPALA, arXiv:1802.01561), hpc_rll/origin/vtrace.py:24-79.

    Interface:
        __init__, forward
    """

    def __init__(self, T, B, N):
        r"""
        Arguments:
            - T (:obj:`int`): trajectory length
            - B (:obj:`int`): batch size
            - N (:obj:`int`): number of output
        """
        super().__init__()
        self.T, self.B, self.N = T, B, N
        self.global_B = 0

    def forward(self, target_output, behaviour_output, action, value, reward, weight=None, gamma: float = 0.99,
                lambda_: float = 0.95, rho_clip_ratio: float = 1.0, c_clip_ratio: float = 1.0,
                rho_pg_clip_ratio: float = 1.0):
        """
        Arguments:
            - target_output (:obj:`torch.Tensor`): :math:`(T, B, N)` logits of the current policy
            - behaviour_output (:obj:`torch.Tensor`): :math:`(T, B, N)` logits of the behaviour policy
            - action (:obj:`torch.Tensor`): :math:`(T, B)` int64
            - value (:obj:`torch.Tensor`): :math:`(T + 1, B)`
            - reward (:obj:`torch.Tensor`): :math:`(T, B)`
            - weight (:obj:`torch.Tensor` or None): :math:`(T, B)`
        Returns:
            - trace_loss (:obj:`hpc_vtrace_loss`): policy_loss, value_loss, entropy_loss -- shape (1,) each
        """
        assert (target_output.is_cuda)
        assert (behaviour_output.is_cuda)
        assert (action.is_cuda)
        assert (value.is_cuda)
        assert (reward.is_cuda)
        if weight is not None:
            assert (weight.is_cuda)
        return hpc_vtrace_loss(*VtraceFunction.apply(target_output, behaviour_output, action, value, reward, weight,
                                                     gamma, lambda_, rho_clip_ratio, c_clip_ratio, rho_pg_clip_ratio,
                                                     self.global_B))


def vtrace_nstep_return(clipped_rhos, clipped_cs, reward, bootstrap_values, gamma=0.99, lambda_=0.95):
    r"""
    Overview:
        The V-trace target :math:`v_s` of a ``(T, B)`` rollout segment, as DI-engine's ``vtrace_nstep_return``
        (hpc_rll/origin/vtrace.py:5-13).  With ``V_t = bootstrap_values[t]``, ``g = fp32(γ)`` and ``f = fp32(γ·λ)``
        (the product taken in double)::

            a_t = (r_t + g·V_{t+1}) − V_t     item_T = +0     item_t = ρ_t·a_t + (f·c_t)·item_{t+1}
            R_t = V_t + item_t

        Every product is one rounded fp32 operation in this order, so the result matches origin bit for bit; long,
        narrow batches (B <= 2048, T >= 512) are scanned in parallel pieces and agree to ~1e-7 relative instead.
        Differentiable in ``reward`` and ``bootstrap_values``; the ratios are constants (IMPALA computes the target
        under ``no_grad``).
    Arguments:
        - clipped_rhos (:obj:`torch.FloatTensor`): :math:`(T, B)`, the clipped importance ratios ρ; must not require
          grad
        - clipped_cs (:obj:`torch.FloatTensor`): :math:`(T, B)`, the clipped trace ratios c; must not require grad
        - reward (:obj:`torch.FloatTensor`): :math:`(T, B)`
        - bootstrap_values (:obj:`torch.FloatTensor`): :math:`(T + 1, B)`, the value estimates of steps 0 to T
        - gamma (:obj:`float`): discount factor, defaults to 0.99
        - lambda_ (:obj:`float`): trace decay, defaults to 0.95
    Returns:
        - return (:obj:`torch.FloatTensor`): :math:`(T, B)`
    """
    for x, name in ((clipped_rhos, "clipped_rhos"), (clipped_cs, "clipped_cs")):
        if isinstance(x, torch.Tensor) and x.requires_grad:
            raise ValueError("%s requires grad, but vtrace_nstep_return is differentiable in reward and "
                             "bootstrap_values only; pass %s.detach()" % (name, name))
    return _ext.require().vtrace_nstep_return(clipped_rhos, clipped_cs, reward, bootstrap_values, float(gamma),
                                              float(lambda_))


def compute_importance_weights(target_output, behaviour_output, action, requires_grad=False):
    r"""
    Overview:
        The importance-sampling ratios :math:`ρ = π(a) / μ(a)` of the chosen actions under the target and the
        behaviour policy, as DI-engine's ``compute_importance_weights`` (hpc_rll/origin/vtrace.py:81-111).  Per row of
        ``N`` logits, with ``m = max x`` and ``s = Σ exp(x − m)`` (the log-prob of ``torch.distributions.Categorical``)::

            lp = x[a] − (m + log s)     per tensor        ρ = exp(lp_target − lp_behaviour)

        One pass over both logits tensors; ρ is bit-identical to the ratios the fused ``VTrace`` loss forms for the
        same rows.  Unlike ``Categorical`` with its default argument validation, nothing is checked on the host, so
        the call never synchronises and can be captured in a CUDA graph.  ``-inf`` (masked) logits are allowed and
        get a gradient of exactly 0; an action outside ``[0, N)`` or on a masked entry is a precondition.
    Arguments:
        - target_output (:obj:`torch.FloatTensor`): :math:`(*, N)`, logits of the target (current) policy, e.g.
          :math:`(T, B, N)`
        - behaviour_output (:obj:`torch.FloatTensor`): :math:`(*, N)`, logits of the behaviour policy, same shape
        - action (:obj:`torch.LongTensor`): :math:`(*)`, the chosen actions
        - requires_grad (:obj:`bool`): False (default) runs under ``torch.no_grad()`` and the result never requires
          grad; True runs under ``torch.enable_grad()``, even inside an outer ``no_grad``, and gradients flow to
          whichever logits tensor requires grad: :math:`∂ρ/∂x_t[k] = ρ·(1[k=a] − p_t[k])`,
          :math:`∂ρ/∂x_b[k] = −ρ·(1[k=a] − p_b[k])`
    Returns:
        - rhos (:obj:`torch.FloatTensor`): :math:`(*)`
    """
    grad_context = torch.enable_grad() if requires_grad else torch.no_grad()
    assert isinstance(action, torch.Tensor)
    with grad_context:
        return _ext.require().importance_weights(target_output, behaviour_output, action)
