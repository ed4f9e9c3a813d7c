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
