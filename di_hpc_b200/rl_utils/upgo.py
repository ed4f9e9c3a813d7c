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


def upgo_returns(rewards, bootstrap_values):
    r"""
    Overview:
        UPGO return targets of a ``(T, B)`` rollout segment, as DI-engine's ``upgo_returns``
        (hpc_rll/origin/upgo.py:21-38): a λ-return with γ = 1 whose trace continues (``ℓ_t = 1``) while the next step
        did at least as well as its value estimate.  With ``V_t = bootstrap_values[t]``::

            ℓ_t = [r_{t+1} + V_{t+2} >= V_{t+1}]   (t < T−1; a NaN compares false)
            R_{T−1} = r_{T−1} + V_T                R_t = (r_t + ℓ_t·R_{t+1}) + (1 − ℓ_t)·V_{t+1}

        Every operation is one rounded fp32 operation in this order, so the result and its gradients match origin bit
        for bit; long, narrow batches (B <= 2048, T >= 512) are scanned in parallel pieces and agree to ~1e-7 relative
        instead.  Differentiable in ``rewards`` and ``bootstrap_values`` (ℓ is not differentiated, and the gradient of
        ``bootstrap_values[0]`` is +0).  When a gradient may be asked for, the call keeps ℓ as one byte per element
        for the backward.
    Arguments:
        - rewards (:obj:`torch.FloatTensor`): :math:`(T, B)`
        - bootstrap_values (:obj:`torch.FloatTensor`): :math:`(T + 1, B)`, the value estimates of steps 0 to T
    Returns:
        - return (:obj:`torch.FloatTensor`): :math:`(T, B)`
    """
    save_mask = torch.is_grad_enabled() and any(isinstance(x, torch.Tensor) and x.requires_grad
                                                for x in (rewards, bootstrap_values))
    return _ext.require().upgo_returns(rewards, bootstrap_values, save_mask)


def tb_cross_entropy(logit, label, mask=None):
    r"""
    Overview:
        The log-probability of the labelled action for every step of a ``(T, B)`` segment, as DI-engine's
        ``tb_cross_entropy`` (hpc_rll/origin/upgo.py:7-18), i.e. ``-F.cross_entropy(logit, label, reduction='none')``
        and UPGO's ``metric``.  Per row of ``N`` logits, with ``m = max x`` and ``s = Σ exp(x − m)``::

            out = (x[a] − m) − log s

        Differentiable in ``logit``: :math:`∂out/∂x[k] = 1[k=a] − p[k]`.  ``-inf`` (masked) logits are allowed and get
        a gradient of exactly 0; a label outside ``[0, N)`` (PyTorch's ``ignore_index = −100`` included) or on a
        masked entry is a precondition.  As in origin, only the 2-D label and ``mask=None`` are supported.
    Arguments:
        - logit (:obj:`torch.FloatTensor`): :math:`T·B` rows of :math:`N` logits, e.g. :math:`(T, B, N)`
        - label (:obj:`torch.LongTensor`): :math:`(T, B)`
        - mask: must be None
    Returns:
        - metric (:obj:`torch.FloatTensor`): :math:`(T, B)`
    """
    assert (len(label.shape) >= 2)
    assert len(label.shape) == 2
    assert mask is None
    return _ext.require().tb_cross_entropy(logit, label)
