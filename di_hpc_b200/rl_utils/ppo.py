"""PPO -- drop-in for /root/reference/hpc_rll/rl_utils/ppo.py (PPO, PPOFunction, hpc_ppo_loss,
hpc_ppo_info).  Same constructor ``PPO(B, N)`` and forward signature (ppo.py:90-148).  approx_kl and
clipfrac are returned as Python floats like the reference, but fetched with ONE device->host copy
(the reference issues two ``.item()`` syncs, ppo.py:148)."""
import os
from collections import namedtuple
from typing import Optional

import torch

from .. import _ext

hpc_ppo_loss = namedtuple('hpc_ppo_loss', ['policy_loss', 'value_loss', 'entropy_loss'])
hpc_ppo_info = namedtuple('hpc_ppo_info', ['approx_kl', 'clipfrac'])


class LazyScalar:
    """A device-computed scalar that is only brought to the host when somebody reads it.

    ``PPO.forward`` returns ``approx_kl`` / ``clipfrac`` as Python floats like the reference (rl_utils/ppo.py:148,
    two ``.item()`` syncs there, one D2H copy here) -- which still blocks the host once per call.  With
    ``PPO.lazy_info = True`` the two values come back as ``LazyScalar``: the 8-byte device->host copy is queued on the
    current stream into pinned memory next to an event, and the host waits for it only in ``float(x)`` / formatting /
    arithmetic / comparison.  A training loop that logs the info every k steps never stalls the launch queue."""
    __slots__ = ("_host", "_idx", "_event", "_value")

    def __init__(self, host, idx, event):
        self._host, self._idx, self._event, self._value = host, idx, event, None

    def item(self) -> float:
        if self._value is None:
            self._event.synchronize()
            self._value = float(self._host[self._idx])
        return self._value

    __float__ = item

    def ready(self) -> bool:
        return self._value is not None or self._event.query()

    def __repr__(self):
        return repr(self.item())

    def __format__(self, spec):
        return format(self.item(), spec)

    def __bool__(self):
        return bool(self.item())

    def __eq__(self, o):
        return self.item() == float(o)

    def __lt__(self, o):
        return self.item() < float(o)

    def __le__(self, o):
        return self.item() <= float(o)

    def __gt__(self, o):
        return self.item() > float(o)

    def __ge__(self, o):
        return self.item() >= float(o)

    def __hash__(self):
        return hash(self.item())

    def __add__(self, o):
        return self.item() + float(o)

    __radd__ = __add__

    def __sub__(self, o):
        return self.item() - float(o)

    def __rsub__(self, o):
        return float(o) - self.item()

    def __mul__(self, o):
        return self.item() * float(o)

    __rmul__ = __mul__

    def __truediv__(self, o):
        return self.item() / float(o)

    def __rtruediv__(self, o):
        return float(o) / self.item()

    def __neg__(self):
        return -self.item()

    def __abs__(self):
        return abs(self.item())


def _lazy_info(info):
    host = torch.empty(2, dtype=torch.float32, pin_memory=True)  # caching host allocator: no cudaHostAlloc per call
    host.copy_(info, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(info.device))
    return hpc_ppo_info(LazyScalar(host, 0, ev), LazyScalar(host, 1, ev))


@_ext.reference_function
def PPOFunction(logits_new, logits_old, action, value_new, value_old, adv, return_, weight, clip_ratio, use_value_clip,
                dual_clip, global_B, adv_stats=None):
    return tuple(_ext.require().ppo(logits_new, logits_old, action, value_new, value_old, adv, return_, weight,
                                    float(clip_ratio), bool(use_value_clip),
                                    -1.0 if dual_clip is None else float(dual_clip), int(global_B), adv_stats))


class PPO(torch.nn.Module):
    """
    Overview:
        Proximal Policy Optimization losses with value clip and dual clip (hpc_rll/origin/ppo.py:13-80).

    Interface:
        __init__, forward
    """

    def __init__(self, B, N):
        r"""
        Arguments:
            - B (:obj:`int`): batch size
            - N (:obj:`int`): number of output
        """
        super().__init__()
        self.B, self.N = B, N
        self.global_B = 0
        # False: approx_kl / clipfrac are Python floats as in the reference (one blocking D2H copy per call);
        # True: LazyScalar objects that synchronise only when read
        self.lazy_info = os.environ.get("HPC_RLL_PPO_LAZY_INFO", "0") == "1"

    def forward(self, logits_new, logits_old, action, value_new, value_old, adv, return_, weight=None,
                clip_ratio: float = 0.2, use_value_clip: bool = True, dual_clip: Optional[float] = None,
                *, adv_stats: Optional[torch.Tensor] = None):
        """
        Arguments:
            - logits_new, logits_old (:obj:`torch.FloatTensor`): :math:`(B, N)`
            - action (:obj:`torch.LongTensor`): :math:`(B, )`
            - value_new, value_old, adv, return_ (:obj:`torch.FloatTensor`): :math:`(B, )`
            - weight (:obj:`torch.FloatTensor` or :obj:`None`): :math:`(B, )`
            - clip_ratio (:obj:`float`): defaults to 0.2
            - use_value_clip (:obj:`bool`)
            - dual_clip (:obj:`float` or None): must be > 1.0 when given
            - adv_stats (:obj:`torch.FloatTensor` or None): extension -- :math:`(2,)` ``[mean, std + 1e-8]`` from
              ``gae_with_adv_stats``; ``adv`` is then normalised inside the kernel (origin/ppo.py:43-47 leaves
              that step to the caller)
        Returns:
            - ppo_loss (:obj:`hpc_ppo_loss`): shape-(1,) tensors
            - ppo_info (:obj:`hpc_ppo_info`): Python floats
        """
        assert (logits_new.is_cuda)
        assert (logits_old.is_cuda)
        assert (action.is_cuda)
        assert (value_new.is_cuda)
        assert (value_old.is_cuda)
        assert (adv.is_cuda)
        assert (return_.is_cuda)
        if weight is not None:
            assert (weight.is_cuda)
        assert dual_clip is None or dual_clip > 1.0, \
            "dual_clip value must be greater than 1.0, but get value: {}".format(dual_clip)
        policy_loss, value_loss, entropy_loss, info = PPOFunction.apply(logits_new, logits_old, action, value_new,
                                                                        value_old, adv, return_, weight, clip_ratio,
                                                                        use_value_clip, dual_clip, self.global_B,
                                                                        adv_stats)
        if self.lazy_info:
            return hpc_ppo_loss(policy_loss, value_loss, entropy_loss), _lazy_info(info)
        approx_kl, clipfrac = info.tolist()  # one device->host copy
        return hpc_ppo_loss(policy_loss, value_loss, entropy_loss), hpc_ppo_info(approx_kl, clipfrac)
