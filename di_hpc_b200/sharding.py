"""Batch-axis sharding of the trajectory-return path across the GPUs of one box.

Every op of the path is independent per column/sample; the only cross-sample coupling is the final
``mean`` of the loss ops (and the 1/count in their gradients).  So the batch axis B shards trivially:
one process per GPU (``torch.distributed``, NCCL over NVLink/NVSwitch), rank r owns columns
``[r*B/W, (r+1)*B/W)``, kernels normalise by the GLOBAL element count (``module.global_B``) and the
only collective is one all-reduce(SUM) of the few loss scalars.  GAE has no collective at all.
The reference has no multi-GPU story (SURVEY.md 2.3); this module is the whole of ours.
"""
import ctypes
from typing import Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from . import _abi, _ext


def shard_columns(B: int, rank: int, world: int, align: int = 4) -> Tuple[int, int]:
    """Column range [b0, b1) of ``rank``.  Shard starts are multiples of ``align`` columns (16 bytes of
    fp32) so every shard of a (T,B) tensor can be described by a TMA tensor map."""
    if world <= 0 or not (0 <= rank < world):
        raise ValueError("bad rank/world %d/%d" % (rank, world))
    per = -(-B // world)
    per = -(-per // align) * align
    b0 = min(B, rank * per)
    b1 = min(B, b0 + per)
    return b0, b1


def local_shard(x: torch.Tensor, rank: int, world: int, dim: int = -1) -> torch.Tensor:
    """Contiguous copy of this rank's column block of a global tensor (time-major tensors are
    B-innermost, so a column block of a global tensor is strided; real data-parallel jobs already hold
    their own contiguous shard and never call this)."""
    b0, b1 = shard_columns(x.shape[dim], rank, world)
    return x.narrow(dim, b0, b1 - b0).contiguous()


class _AllReduceSum(torch.autograd.Function):
    """loss_global = sum over ranks of loss_local; d loss_global / d loss_local = 1 on every rank."""

    @staticmethod
    def forward(ctx, x, group):
        y = x.clone()
        dist.all_reduce(y, op=dist.ReduceOp.SUM, group=group)
        return y

    @staticmethod
    def backward(ctx, g):
        return g, None


class P2PScalarAllReduce:
    """all-reduce(SUM) of <= 16 fp32 scalars over NVLink peer memory (csrc/p2p.cu) -- the path's only collective without
    NCCL: one 32-thread kernel per rank stores its epoch-tagged scalars into every peer's (CUDA-IPC mapped) buffer, waits
    for all ranks' words in its own buffer and adds them in rank order.  Cheaper than an NCCL call, bit-identical on every rank, capturable in CUDA graphs.  Single node, <= 64 ranks; set up once
    per process group (the IPC handles travel through ``torch.distributed``)."""

    def __init__(self, group=None):
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        L = _abi.lib()
        local, handle = ctypes.c_void_p(), (ctypes.c_ubyte * 64)()
        _abi.check(L.hpc_rll_p2p_alloc(ctypes.byref(local), handle), "hpc_rll_p2p_alloc")
        self._local = local.value
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle), group=group)
        self._bufs = (ctypes.c_void_p * self.world)()
        self._peers = []
        for r, h in enumerate(handles):
            if r == self.rank:
                self._bufs[r] = self._local
                continue
            p, raw = ctypes.c_void_p(), (ctypes.c_ubyte * 64).from_buffer_copy(h)
            _abi.check(L.hpc_rll_p2p_open(raw, ctypes.byref(p)), "hpc_rll_p2p_open")
            self._bufs[r] = p.value
            self._peers.append(p.value)
        dist.barrier(group=group)  # nobody stores into a buffer that is not mapped everywhere yet

    def __call__(self, t: torch.Tensor) -> torch.Tensor:
        """in place on the current stream; ``t``: contiguous fp32 CUDA tensor with <= 16 elements"""
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and 1 <= t.numel() <= 16):
            raise ValueError("P2PScalarAllReduce takes a contiguous float32 CUDA tensor of 1..16 elements")
        with _abi.on_device(t.device):
            _abi.check(
                _abi.lib().hpc_rll_allreduce_scalars_p2p(t.data_ptr(), t.numel(), self._bufs, self.rank, self.world,
                                                         _abi.stream_of(t)), "hpc_rll_allreduce_scalars_p2p")
        return t

    def close(self):
        L = _abi.lib()
        torch.cuda.synchronize()
        if dist.is_initialized():
            dist.barrier(group=self.group)  # peers may still be polling words we have not written yet
        for p in self._peers:
            L.hpc_rll_p2p_close(p)
        self._peers = []
        if self._local:
            L.hpc_rll_p2p_free(self._local)
            self._local = None


_default_comm: Optional[P2PScalarAllReduce] = None


def enable_p2p_allreduce(group=None) -> P2PScalarAllReduce:
    """Route ``all_reduce_losses`` through the NVLink peer-memory kernel from now on (call on every rank)."""
    global _default_comm
    _default_comm = P2PScalarAllReduce(group)
    return _default_comm


def all_reduce_losses(losses: Sequence[torch.Tensor], group=None, comm: Optional[P2PScalarAllReduce] = None):
    """Sum per-rank partial losses (already divided by the global count) into the global losses.
    Differentiable: gradients flow back to the local losses unchanged.  Packs the scalars into one
    tensor so a step costs a single latency-bound collective: the NVLink peer-memory kernel when a
    ``P2PScalarAllReduce`` is given (or enabled with ``enable_p2p_allreduce``), else one NCCL call."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return list(losses)
    flat = losses[0].reshape(-1) if len(losses) == 1 else torch.cat([l.reshape(-1) for l in losses])
    comm = comm if comm is not None else _default_comm
    if comm is not None and flat.is_cuda and flat.numel() <= 16:
        red = _ext.require().allreduce_scalars_p2p(flat, ctypes.addressof(comm._bufs), comm.rank, comm.world)
    else:
        red = _AllReduceSum.apply(flat, group)
    out, o = [], 0
    for l in losses:
        n = l.numel()
        out.append(red[o:o + n].reshape(l.shape))
        o += n
    return out


def all_reduce_moments(moments: torch.Tensor, group=None) -> torch.Tensor:
    """In-place all-reduce(SUM) of ``[sum(adv), sum(adv^2), count]`` (fp64) over the ranks that shard the
    batch: the element count rides in the same tensor, so the global mean/std need one latency-bound
    collective and no device->host read."""
    if moments.dtype != torch.float64 or moments.numel() != 3:
        raise TypeError("moments must be 3 float64 values [sum, sum of squares, count]")
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(moments, op=dist.ReduceOp.SUM, group=group)
    return moments


def set_global_batch(module: torch.nn.Module, global_B: int) -> torch.nn.Module:
    """Tell a loss module that its batch is one shard of ``global_B`` columns/samples."""
    if not hasattr(module, "global_B"):
        raise TypeError("%s has no global_B (GAE needs none)" % type(module).__name__)
    module.global_B = int(global_B)
    return module
