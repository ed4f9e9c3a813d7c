"""TD-error family -- drop-in for /root/reference/hpc_rll/rl_utils/td.py.

Classes (same names, constructor arguments and forward signatures as the reference):
    DistNStepTD(T, B, N, n_atom)        td.py:33-108
    TDLambda(T, B)                      td.py:140-187
    QNStepTD(T, B, N)                   td.py:213-277
    QNStepTDRescale(T, B, N)            td.py:303-371
    IQNNStepTDError(tau, tauPrime, T, B, N)   td.py:397-485
    QRDQNNStepTDError(tau, T, B, N)     td.py:513-592

Functions (DI-engine's ``ding.rl_utils.td``; the reference computes them in Python only, origin/td.py:179-244):
    generalized_lambda_returns(bootstrap_values, rewards, gammas, lambda_, done=None)
    multistep_forward_view(bootstrap_values, rewards, gammas, lambda_, done=None)

Common deviations from the reference wrapper (DESIGN.md "Deviations"): results are fresh tensors
(the reference returns module-owned buffers by alias), scratch lives in a per-call workspace rather
than in registered buffers that pollute ``state_dict``, shapes come from the inputs (constructor
sizes are kept for API compatibility), saved state goes through ``save_for_backward``.
Scalars keep the reference's shape ``(1,)`` (register_buffer('loss', torch.zeros(1)), td.py:161).
"""
import numbers
from typing import Optional

import torch

from .. import _ext


@_ext.reference_function
def TDLambdaFunction(value, reward, weight, gamma, lambda_, global_B):
    return _ext.require().td_lambda(value, reward, weight, float(gamma), float(lambda_), int(global_B))


class TDLambda(torch.nn.Module):
    """
    Overview:
        TD(lambda) loss with constant gamma and lambda (hpc_rll/origin/td.py:148-176).

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
        self.global_B = 0  # set >0 when B is one shard of a data-parallel batch (see di_hpc_b200.sharding)

    def forward(self, value, reward, weight=None, gamma: float = 0.9, lambda_: float = 0.8) -> torch.Tensor:
        """
        Arguments:
            - value (:obj:`torch.FloatTensor`): :math:`(T + 1, B)`
            - reward (:obj:`torch.FloatTensor`): :math:`(T, B)`
            - weight (:obj:`torch.FloatTensor` or None): :math:`(T, B)` (or :math:`(B,)`, broadcast)
            - gamma (:obj:`float`): discount factor, defaults to 0.9
            - lambda_ (:obj:`float`): lambda, defaults to 0.8
        Returns:
            - loss (:obj:`torch.Tensor`): shape :math:`(1,)`
        """
        assert (value.is_cuda)
        assert (reward.is_cuda)
        if weight is not None:
            assert (weight.is_cuda)
        return TDLambdaFunction.apply(value, reward, weight, gamma, lambda_, self.global_B)


# ------------------------------------------------------------------------------------------- lambda-returns
def _per_step(x, name):
    """-> (tensor or None, scalar) for a discount argument that is a number or a (T, B) tensor"""
    if isinstance(x, torch.Tensor):
        if x.requires_grad:
            raise ValueError("%s requires grad, but lambda-returns are differentiable in bootstrap_values and rewards "
                             "only; pass %s.detach()" % (name, name))
        return x, 0.0
    if isinstance(x, numbers.Real):
        return None, float(x)
    raise TypeError("%s must be a number or a (T, B) float32 tensor, got %s" % (name, type(x).__name__))


def _lambda_returns(bootstrap_values, rewards, gammas, lambda_, done, offset):
    g_t, g = _per_step(gammas, "gammas")
    l_t, lam = _per_step(lambda_, "lambda_")
    return _ext.require().lambda_returns(bootstrap_values, rewards, g_t, l_t, done, g, lam, offset)


def generalized_lambda_returns(bootstrap_values, rewards, gammas, lambda_, done=None) -> torch.Tensor:
    r"""
    Overview:
        λ-returns of a ``(T, B)`` rollout segment, as DI-engine's ``generalized_lambda_returns``, with per-step
        discounts and episode ends.  With ``V_t = bootstrap_values[t+1]``, ``d_t = γ_t·λ_t``, ``e_t = γ_t − d_t`` and
        ``m_t = 0`` where ``done_t`` is set, 1 elsewhere::

            done=None:  R_{T-1} = r + γ·V               R_t = (r_t + d_t·R_{t+1}) + e_t·V_t
            done given: R_{T-1} = r + (m·γ)·V           R_t = r_t + m_t·(d_t·R_{t+1} + e_t·V_t)

        Every product is one rounded fp32 operation in this order, so the result and its gradients match eager
        PyTorch of the formula bit for bit; long, narrow batches (B <= 2048, T >= 512) are scanned in parallel pieces
        and agree to ~1e-7 relative instead.  Differentiable in ``bootstrap_values`` and ``rewards`` (the gradient of
        ``bootstrap_values[0]``, which no return reads, is +0).
    Arguments:
        - bootstrap_values (:obj:`torch.FloatTensor`): :math:`(T + 1, B)`, the value estimates of steps 0 to T
        - rewards (:obj:`torch.FloatTensor`): :math:`(T, B)`
        - gammas, lambda_ (:obj:`float` or :obj:`torch.FloatTensor`): a number, or a :math:`(T, B)` tensor that does
          not require grad
        - done (:obj:`torch.Tensor` or None): :math:`(T, B)`; a set entry ends the episode at that step.  Bool or
          uint8 masks are read in place (non-zero = set); any other dtype is converted with ``done != 0``, so a
          fractional float counts as set.
    Returns:
        - return (:obj:`torch.FloatTensor`): :math:`(T, B)`
    """
    return _lambda_returns(bootstrap_values, rewards, gammas, lambda_, done, 1)


def multistep_forward_view(bootstrap_values, rewards, gammas, lambda_, done=None) -> torch.Tensor:
    r"""
    Overview:
        The λ-return recursion of ``generalized_lambda_returns`` with ``V_t = bootstrap_values[t]``: DI-engine's
        ``multistep_forward_view`` (Sutton & Barto (12.18)), where ``bootstrap_values`` holds the value estimates of
        steps 1 to T.  Same formula, operation order, arguments and gradients otherwise.
    Arguments:
        - bootstrap_values (:obj:`torch.FloatTensor`): :math:`(T, B)`
        - rewards, gammas, lambda_, done: as in ``generalized_lambda_returns``
    Returns:
        - return (:obj:`torch.FloatTensor`): :math:`(T, B)`
    """
    return _lambda_returns(bootstrap_values, rewards, gammas, lambda_, done, 0)


# ------------------------------------------------------------------------------------------- q n-step
@_ext.reference_function
def QNStepTDFunction(q, next_n_q, action, next_n_action, reward, done, weight, gamma, global_B):
    return tuple(_ext.require().q_nstep_td(q, next_n_q, action, next_n_action, reward, done, weight, float(gamma),
                                           False, int(global_B)))


@_ext.reference_function
def QNStepTDRescaleFunction(q, next_n_q, action, next_n_action, reward, done, weight, gamma, global_B):
    return tuple(_ext.require().q_nstep_td(q, next_n_q, action, next_n_action, reward, done, weight, float(gamma),
                                           True, int(global_B)))


class QNStepTD(torch.nn.Module):
    """
    Overview:
        Multistep (1 step or n step) td_error for q-learning based algorithm
        (hpc_rll/origin/td.py:252-291; criterion = MSELoss as in the reference, td.py:266-268).

    Interface:
        __init__, forward
    """
    _fn = QNStepTDFunction

    def __init__(self, T, B, N):
        r"""
        Arguments:
            - T (:obj:`int`): nstep
            - B (:obj:`int`): batch size
            - N (:obj:`int`): action dim
        """
        super().__init__()
        self.T, self.B, self.N = T, B, N
        self.global_B = 0

    def forward(self, q, next_n_q, action, next_n_action, reward, done, weight, gamma: float) -> torch.Tensor:
        """
        Arguments:
            - q, next_n_q (:obj:`torch.FloatTensor`): :math:`(B, N)`
            - action, next_n_action (:obj:`torch.LongTensor`): :math:`(B, )`
            - reward (:obj:`torch.FloatTensor`): :math:`(T, B)`
            - done (:obj:`torch.FloatTensor`): :math:`(B, )` 0/1
            - weight (:obj:`torch.FloatTensor` or None): :math:`(B, )`
            - gamma (:obj:`float`): discount factor
        Returns:
            - loss (:obj:`torch.Tensor`): shape :math:`(1,)`
            - td_error_per_sample (:obj:`torch.Tensor`): :math:`(B, )`
        """
        for t in (q, next_n_q, action, next_n_action, reward, done):
            assert (t.is_cuda)
        if weight is not None:
            assert (weight.is_cuda)
        return self._fn.apply(q, next_n_q, action, next_n_action, reward, done, weight, gamma, self.global_B)


class QNStepTDRescale(QNStepTD):
    """
    Overview:
        n-step td_error with value rescaling (hpc_rll/origin/td.py:294-340), same interface as QNStepTD.
    """
    _fn = QNStepTDRescaleFunction


# ------------------------------------------------------------------------------------------- C51
@_ext.reference_function
def DistNStepTDFunction(dist, next_n_dist, action, next_n_action, reward, done, weight, gamma, v_min, v_max, global_B):
    return tuple(_ext.require().dist_nstep_td(dist, next_n_dist, action, next_n_action, reward, done, weight,
                                              float(gamma), float(v_min), float(v_max), int(global_B)))


class DistNStepTD(torch.nn.Module):
    """
    Overview:
        Multistep td_error for distributional (C51) q-learning (hpc_rll/origin/td.py:29-143).

    Interface:
        __init__, forward
    """

    def __init__(self, T, B, N, n_atom):
        r"""
        Arguments:
            - T (:obj:`int`): nstep
            - B (:obj:`int`): batch size
            - N (:obj:`int`): action dim
            - n_atom (:obj:`int`): number of atoms
        """
        super().__init__()
        self.T, self.B, self.N, self.n_atom = T, B, N, n_atom
        self.global_B = 0
        # the reference asserts dist[range, action] > 0 on the host every call (td.py:101-103), which forces
        # a device sync; keep the check available but off the hot path
        self.check_positive = False

    def forward(self, dist, next_n_dist, action, next_n_action, reward, done, weight, gamma: float, v_min: float,
                v_max: float) -> torch.Tensor:
        """
        Arguments:
            - dist, next_n_dist (:obj:`torch.FloatTensor`): :math:`(B, N, n_atom)`
            - action, next_n_action (:obj:`torch.LongTensor`): :math:`(B, )`
            - reward (:obj:`torch.FloatTensor`): :math:`(T, B)`
            - done (:obj:`torch.FloatTensor`): :math:`(B, )`
            - weight (:obj:`torch.FloatTensor` or None): :math:`(B, )`
            - gamma, v_min, v_max (:obj:`float`)
        Returns:
            - loss (:obj:`torch.Tensor`): shape :math:`(1,)`
            - td_error_per_sample (:obj:`torch.Tensor`): :math:`(B, )`
        """
        for t in (dist, next_n_dist, action, next_n_action, reward, done):
            assert (t.is_cuda)
        if weight is not None:
            assert (weight.is_cuda)
        if self.check_positive:
            batch_range = torch.arange(action.shape[0], device=action.device)
            assert (dist[batch_range, action] > 0.0).all(), ("dist act", dist[batch_range, action], "dist:", dist)
        return DistNStepTDFunction.apply(dist, next_n_dist, action, next_n_action, reward, done, weight, gamma, v_min,
                                         v_max, self.global_B)


# ------------------------------------------------------------------------------------------- QR-DQN
@_ext.reference_function
def QRDQNNStepTDErrorFunction(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma, gamma, global_B):
    return tuple(_ext.require().qrdqn_nstep_td(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma,
                                               float(gamma), int(global_B)))


class QRDQNNStepTDError(torch.nn.Module):
    """
    Overview:
        Multistep td_error in QR-DQN (hpc_rll/origin/td.py:455-517).  As in the reference wrapper, the
        quantile weight uses the integer quantile COUNT ``tau`` (hpc_rll/rl_utils/td.py:538,
        qrdqn_nstep_td_error_kernel.h:60), not a tensor of fractions.

    Interface:
        __init__, forward
    """

    def __init__(self, tau, T, B, N):
        r"""
        Arguments:
            - tau (:obj:`int`): num of quantiles
            - T (:obj:`int`): nstep
            - B (:obj:`int`): batch size
            - N (:obj:`int`): action dim
        """
        super().__init__()
        self.tau, self.T, self.B, self.N = tau, T, B, N
        self.global_B = 0

    def forward(self, q, next_n_q, action, next_n_action, reward, done, gamma: float,
                weight: Optional[torch.Tensor] = None, value_gamma: Optional[torch.Tensor] = None) -> torch.Tensor:
        """
        Arguments:
            - q, next_n_q (:obj:`torch.FloatTensor`): :math:`(B, N, tau)`
            - action, next_n_action (:obj:`torch.LongTensor`): :math:`(B, )`
            - reward (:obj:`torch.FloatTensor`): :math:`(T, B)`
            - done (:obj:`torch.FloatTensor`): :math:`(B, )`
            - gamma (:obj:`float`)
            - weight, value_gamma (:obj:`torch.FloatTensor` or None): :math:`(B, )`
        Returns:
            - loss (:obj:`torch.Tensor`): shape :math:`(1,)`;  td_error_per_sample :math:`(B, )`
        """
        for t in (q, next_n_q, action, next_n_action, reward, done):
            assert (t.is_cuda)
        if weight is not None:
            assert (weight.is_cuda)
        if value_gamma is not None:
            assert (value_gamma.is_cuda)
        return QRDQNNStepTDErrorFunction.apply(q, next_n_q, action, next_n_action, reward, done, weight, value_gamma,
                                               gamma, self.global_B)


# ------------------------------------------------------------------------------------------- IQN
@_ext.reference_function
def IQNNStepTDErrorFunction(q, next_n_q, action, next_n_action, reward, done, replay_quantiles, weight, value_gamma,
                            gamma, kappa, global_B):
    return tuple(_ext.require().iqn_nstep_td(q, next_n_q, action, next_n_action, reward, done, replay_quantiles,
                                             weight, value_gamma, float(gamma), float(kappa), int(global_B)))


class IQNNStepTDError(torch.nn.Module):
    """
    Overview:
        Multistep td_error in IQN (arXiv:1806.06923), hpc_rll/origin/td.py:361-448.

    Interface:
        __init__, forward
    """

    def __init__(self, tau, tauPrime, T, B, N):
        r"""
        Arguments:
            - tau (:obj:`int`): num of quantiles
            - tauPrime (:obj:`int`): num of target quantiles
            - T (:obj:`int`): nstep
            - B (:obj:`int`): batch size
            - N (:obj:`int`): action dim
        """
        super().__init__()
        self.tau, self.tauPrime, self.T, self.B, self.N = tau, tauPrime, T, B, N
        self.global_B = 0

    def forward(self, q, next_n_q, action, next_n_action, reward, done, replay_quantiles, gamma: float,
                kappa: float = 1.0, weight: Optional[torch.Tensor] = None,
                value_gamma: Optional[torch.Tensor] = None) -> torch.Tensor:
        """
        Arguments:
            - q (:obj:`torch.FloatTensor`): :math:`(tau, B, N)`
            - next_n_q (:obj:`torch.FloatTensor`): :math:`(tau', B, N)`
            - action, next_n_action (:obj:`torch.LongTensor`): :math:`(B, )`
            - reward (:obj:`torch.FloatTensor`): :math:`(T, B)`
            - done (:obj:`torch.FloatTensor`): :math:`(B, )`
            - replay_quantiles (:obj:`torch.FloatTensor`): :math:`(tau, B)`
            - gamma, kappa (:obj:`float`)
            - weight, value_gamma (:obj:`torch.FloatTensor` or None): :math:`(B, )`
        Returns:
            - loss (:obj:`torch.Tensor`): shape :math:`(1,)`;  td_error_per_sample :math:`(B, )`
        """
        for t in (q, next_n_q, action, next_n_action, reward, done, replay_quantiles):
            assert (t.is_cuda)
        if weight is not None:
            assert (weight.is_cuda)
        if value_gamma is not None:
            assert (value_gamma.is_cuda)
        return IQNNStepTDErrorFunction.apply(q, next_n_q, action, next_n_action, reward, done, replay_quantiles,
                                             weight, value_gamma, gamma, kappa, self.global_B)
