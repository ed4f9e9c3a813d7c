"""GAE -- drop-in for /root/reference/hpc_rll/rl_utils/gae.py (class GAE, GAEFunction).

Same constructor ``GAE(T, B)`` and ``forward(value, reward, gamma=0.99, lambda_=0.97)`` as the
reference (gae.py:20-61).  Differences, all deliberate (DESIGN.md "Deviations"):
  * the backward is a real adjoint (the reference's ``GAEFunction.backward`` returns None for every
    input, gae.py:16-18, while hpc_rll/origin/gae.py is differentiable);
  * the result is a fresh tensor sized from the inputs, not the module-owned ``adv`` buffer returned
    by alias (gae.py:39,61) -- T and B of the constructor are kept only for API compatibility;
  * kernels run on PyTorch's current stream, with argument checks.

``gae(gae_data(value, next_value, reward, done, traj_flag))`` is the episode-aware, un-normalised GAE of DI-engine's
functional ``ding.rl_utils.gae``, for rollouts whose columns hold several episodes.  The reference has no counterpart.
"""
from collections import namedtuple

import torch

from .. import _abi, _ext

gae_data = namedtuple('gae_data', ['value', 'next_value', 'reward', 'done', 'traj_flag'])


@_ext.reference_function
def GAEFunction(value, reward, gamma, lambda_):
    return _ext.require().gae(value, reward, float(gamma), float(lambda_))


def gae(data, gamma: float = 0.99, lambda_: float = 0.97) -> torch.Tensor:
    """
    Overview:
        Standard (un-normalised) Generalized Advantage Estimation over a ``(T, B)`` rollout segment in which episodes
        may end anywhere, as DI-engine's ``ding.rl_utils.gae``.  This is NOT the normalised variant that ``GAE``
        computes (no ``denom``).  With ``g = float32(gamma)`` and ``gl = float32(gamma * lambda_)``::

            delta_t = (reward_t + g * next_value_t * (1 - done_t)) - value_t
            adv_t   = delta_t + gl * (1 - traj_flag_t) * adv_{t+1},    adv_{T-1} = delta_{T-1}

        Every step is one rounded fp32 operation in this order, so the result (and its gradients) match eager
        PyTorch of the formula bit for bit; segments of long, narrow batches (B <= 2048, T >= 512) are scanned in
        parallel pieces and agree to ~1e-7 relative instead.  Differentiable in ``value``, ``next_value`` and
        ``reward``.
    Arguments:
        - data (:obj:`gae_data` or any 5-tuple): ``(value, next_value, reward, done, traj_flag)``
            - value, next_value, reward (:obj:`torch.FloatTensor`): :math:`(T, B)`, ``next_value_t`` is the value of
              the state after step t (the bootstrap value at an episode's end)
            - done (:obj:`torch.Tensor` or None): :math:`(T, B)`; a set entry masks the bootstrap of that step.
              None: no step ends an episode.
            - traj_flag (:obj:`torch.Tensor` or None): :math:`(T, B)`; a set entry cuts the recursion after that step.
              None: ``traj_flag = done``.
            Masks may be bool or uint8 (read in place, non-zero = set); any other dtype is converted with
            ``mask != 0``, so a fractional float mask counts as set.
        - gamma (:obj:`float`): discount factor, defaults to 0.99
        - lambda_ (:obj:`float`): GAE lambda, defaults to 0.97
    Returns:
        - adv (:obj:`torch.FloatTensor`): :math:`(T, B)`
    """
    value, next_value, reward, done, traj_flag = data
    if value.dim() != 2:
        raise ValueError("gae: value must be (T, B), got %s; multi-agent (T, B, A) values are not supported"
                         % (tuple(value.shape), ))
    return _ext.require().gae_episodic(value, next_value, reward, done, traj_flag, float(gamma), float(lambda_))


def gae_with_adv_stats(value, reward, gamma: float = 0.99, lambda_: float = 0.97, group=None):
    """
    Overview:
        GAE forward fused with the statistics of the advantage normalisation
        ``(adv - adv.mean()) / (adv.std() + 1e-8)`` that precedes ``ppo_error``
        (hpc_rll/origin/ppo.py:43-47): the scan kernel accumulates sum(adv) and sum(adv^2) in fp64 while it
        writes ``adv``, so mean/std cost no extra pass over HBM.  Hand ``adv_stats`` to ``PPO.forward(...,
        adv_stats=adv_stats)`` and the normalisation itself happens inside the PPO kernel.  No autograd
        (advantages are targets; the reference's GAE has no backward at all, rl_utils/gae.py:16-18).
    Arguments:
        - value (:obj:`torch.FloatTensor`): :math:`(T + 1, B)`; reward :math:`(T, B)`
        - group: ``torch.distributed`` group over which the batch axis is sharded (moments are all-reduced)
    Returns:
        - adv (:obj:`torch.FloatTensor`): :math:`(T, B)`, NOT normalised
        - adv_stats (:obj:`torch.FloatTensor`): :math:`(2,)` = ``[mean, std + 1e-8]`` of the (global) advantages
    """
    from ..sharding import all_reduce_moments
    value = _abi.require_f32_cuda("value", value.detach())
    reward = _abi.require_f32_cuda("reward", reward.detach())
    T, B = reward.shape
    if value.shape != (T + 1, B):
        raise ValueError("value must be (T+1, B)=(%d, %d), got %s" % (T + 1, B, tuple(value.shape)))
    if T == 0 or B == 0:
        raise ValueError("gae_with_adv_stats needs a non-empty batch")
    dev = reward.device
    adv = torch.empty_like(reward)
    moments = torch.empty(3, dtype=torch.float64, device=dev)
    moments[2] = T * B
    stats = torch.empty(2, dtype=torch.float32, device=dev)
    ws = _abi.workspace(_abi.OP_GAE_MOMENTS, T, B, 0, dev)
    with _abi.on_device(dev):
        _abi.check(
            _abi.lib().hpc_rll_gae_forward_moments(_abi.ptr(value), _abi.ptr(reward), _abi.ptr(adv),
                                                   _abi.ptr(moments), T, B, float(gamma), float(lambda_),
                                                   _abi.ptr(ws), ws.numel(), _abi.stream_of(reward)),
            "hpc_rll_gae_forward_moments")
        all_reduce_moments(moments, group)
        _abi.check(_abi.lib().hpc_rll_adv_stats(_abi.ptr(moments), 0, _abi.ptr(stats), _abi.stream_of(reward)),
                   "hpc_rll_adv_stats")
    return adv, stats


class GAE(torch.nn.Module):
    """
    Overview:
        Generalized Advantage Estimator (arXiv:1506.02438), normalised variant of
        hpc_rll/origin/gae.py:28-37.

    Interface:
        __init__, forward
    """

    def __init__(self, T, B):
        r"""
        Arguments:
            - T (:obj:`int`): trajectory length
            - B (:obj:`int`): batch size
        """
        super().__init__()
        self.T, self.B = T, B

    def forward(self, value, reward, gamma: float = 0.99, lambda_: float = 0.97) -> torch.FloatTensor:
        """
        Arguments:
            - value (:obj:`torch.FloatTensor`): :math:`(T + 1, B)`
            - reward (:obj:`torch.FloatTensor`): :math:`(T, B)`
            - gamma (:obj:`float`): discount factor, defaults to 0.99
            - lambda_ (:obj:`float`): GAE lambda, defaults to 0.97
        Returns:
            - adv (:obj:`torch.FloatTensor`): :math:`(T, B)`
        """
        assert (value.is_cuda)
        assert (reward.is_cuda)
        return GAEFunction.apply(value, reward, gamma, lambda_)
