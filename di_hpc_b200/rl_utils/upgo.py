"""UPGO -- drop-in for /root/reference/hpc_rll/rl_utils/upgo.py (UPGO, UpgoFunction).
Same constructor ``UPGO(T, B, N)`` and ``forward(target_output, rhos, action, rewards,
bootstrap_values)`` (upgo.py:46-79); the loss is a shape-(1,) tensor."""
import torch

from .. import _ext


@_ext.reference_function
def UpgoFunction(target_output, rho, action, reward, value, global_B):
    return _ext.require().upgo(target_output, rho, action, reward, value, int(global_B))


class UPGO(torch.nn.Module):
    """
    Overview:
        UPGO loss (hpc_rll/origin/upgo.py:40-70).

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

    def forward(self, target_output, rhos, action, rewards, bootstrap_values):
        """
        Arguments:
            - target_output (:obj:`torch.Tensor`): :math:`(T, B, N)`
            - rhos (:obj:`torch.Tensor`): :math:`(T, B)` importance sampling ratio
            - action (:obj:`torch.Tensor`): :math:`(T, B)` int64
            - rewards (:obj:`torch.Tensor`): :math:`(T, B)`
            - bootstrap_values (:obj:`torch.Tensor`): :math:`(T + 1, B)`
        Returns:
            - loss (:obj:`torch.Tensor`): shape :math:`(1,)`
        """
        assert (target_output.is_cuda)
        assert (rhos.is_cuda)
        assert (action.is_cuda)
        assert (rewards.is_cuda)
        assert (bootstrap_values.is_cuda)
        return UpgoFunction.apply(target_output, rhos, action, rewards, bootstrap_values, self.global_B)
