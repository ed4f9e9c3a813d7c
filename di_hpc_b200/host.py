"""Host-side entry of the trajectory-return path: operands in (pinned) HOST memory, results in host memory.

The reference has no host data path (its wrappers assert ``is_cuda``, hpc_rll/rl_utils/gae.py:58-59); a collector that
keeps trajectories in host RAM would `.cuda()` three tensors, call ``GAE``, and `.cpu()` three results -- six serial
copies around two kernels.  ``gae_fwd_bwd_host`` is that whole round trip as ONE call into the C ABI
(``hpc_rll_gae_fwd_bwd_host``): a T-chunked carry pipeline in which contiguous row ranges stream over the H2D copy
engine, full-width TMA kernels, and the D2H engine at the same time (di_hpc_b200/csrc/gae.cu, "host-buffer path").

``bind_to_device`` / ``pinned_empty`` place the calling process and its page-locked buffers on the GPU's NUMA node
(csrc/host_numa.cu): with one rank per GPU this is what keeps eight ranks from funnelling their DMA traffic through one
socket.  This is what bench.py times as ``e2e``.
"""
import ctypes
import weakref

import torch

from . import _abi


def device_numa_node(device: int = None) -> int:
    """NUMA node of a CUDA device (-1 if the platform does not say)."""
    if device is None:
        device = torch.cuda.current_device()
    return int(_abi.lib().hpc_rll_device_numa_node(int(device)))


def bind_to_device(device: int = None) -> int:
    """Pin the calling thread (and the threads it starts afterwards) to the CPUs of the GPU's NUMA node and prefer that
    node for its allocations.  Returns the node, or -1 when nothing was changed."""
    if device is None:
        device = torch.cuda.current_device()
    return int(_abi.lib().hpc_rll_bind_thread_to_device(int(device)))


def unbind() -> None:
    """Undo ``bind_to_device``: the CPU affinity from before the first bind and the default memory policy."""
    _abi.lib().hpc_rll_bind_thread_to_device(-1)


def pinned_empty(shape, device: int = None) -> torch.Tensor:
    """A page-locked fp32 host tensor whose pages sit on the NUMA node of ``device`` (zero-filled by the first touch).
    The memory is owned by the library and released when the tensor's storage dies."""
    if device is None:
        device = torch.cuda.current_device()
    shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list, torch.Size)) else (shape, )))
    n = 1
    for s in shape:
        n *= s
    L = _abi.lib()
    p = L.hpc_rll_host_alloc(max(n, 1) * 4, int(device))
    if not p:
        msg = L.hpc_rll_last_error()
        raise _abi.HpcRllError("hpc_rll_host_alloc failed: %s" % (msg.decode() if msg else "?"))
    buf = (ctypes.c_float * max(n, 1)).from_address(p)
    t = torch.frombuffer(buf, dtype=torch.float32, count=n).reshape(shape)
    weakref.finalize(t.untyped_storage(), L.hpc_rll_host_free, p)
    t._hpc_rll_keepalive = buf
    return t


def gae_fwd_bwd_host(value, reward, grad_adv=None, gamma: float = 0.99, lambda_: float = 0.97, out=None):
    """
    Overview:
        GAE forward (+ adjoint when ``grad_adv`` is given) on HOST tensors, pipelined through the current CUDA device.
        Semantics of ``GAE.forward`` and its backward (hpc_rll/origin/gae.py:28-37), bit-identical to the
        device-resident path.
    Arguments:
        - value (:obj:`torch.FloatTensor`): :math:`(T + 1, B)` CPU, contiguous (pinned memory for full copy speed)
        - reward (:obj:`torch.FloatTensor`): :math:`(T, B)` CPU
        - grad_adv (:obj:`torch.FloatTensor` or None): :math:`(T, B)` CPU upstream gradient of ``adv``
        - out: optional tuple of preallocated CPU result tensors ``(adv, grad_value, grad_reward)``
    Returns:
        - adv :math:`(T, B)`; and ``grad_value`` :math:`(T + 1, B)``, ``grad_reward`` :math:`(T, B)`` when ``grad_adv`` is given
    """
    def chk(name, t, shape):
        if t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != shape:
            raise ValueError("%s must be a contiguous float32 CPU tensor of shape %s" % (name, shape))

    T, B = reward.shape
    chk("value", value, (T + 1, B))
    chk("reward", reward, (T, B))
    if grad_adv is not None:
        chk("grad_adv", grad_adv, (T, B))
    if out is None:
        adv = torch.empty((T, B), dtype=torch.float32).pin_memory()
        gv = torch.empty((T + 1, B), dtype=torch.float32).pin_memory() if grad_adv is not None else None
        gr = torch.empty((T, B), dtype=torch.float32).pin_memory() if grad_adv is not None else None
    else:
        adv, gv, gr = out
        chk("out adv", adv, (T, B))
        if grad_adv is not None:
            chk("out grad_value", gv, (T + 1, B))
            chk("out grad_reward", gr, (T, B))
    _abi.check(
        _abi.lib().hpc_rll_gae_fwd_bwd_host(value.data_ptr(), reward.data_ptr(),
                                            None if grad_adv is None else grad_adv.data_ptr(), adv.data_ptr(),
                                            None if grad_adv is None else gv.data_ptr(),
                                            None if grad_adv is None else gr.data_ptr(), T, B, float(gamma),
                                            float(lambda_)), "hpc_rll_gae_fwd_bwd_host")
    return adv if grad_adv is None else (adv, gv, gr)
