"""Padding -- drop-in for /root/reference/hpc_rll/rl_utils/padding.py: ``Padding{1,2,3}D`` /
``UnPadding{1,2,3}D`` over lists of ragged CUDA tensors (same signatures and return structure:
``new_x, mask, shapes``; in group mode ``[tuple(new_x), tuple(mask), tuple(shapes)]`` with per-group flat
shape lists, padding.py:39-41,93-95,155-157).  ``mask`` is int32 (1 inside, ``value`` outside), as the
reference's CUDA path returns it.

One CUDA launch pads every tensor of every group: the per-tensor descriptors travel in kernel parameter
space (di_hpc_b200/csrc/padding.cu), so a call performs no cudaMalloc / cudaMemcpy (the reference does up
to 7 of each per call, src/rl_utils/padding.cu:118-131,172-199).  UnPadding writes all outputs into one
allocation and returns views of it (origin's default ``deepcopy=False`` also returns views).
"""
from functools import reduce
from typing import List, Union

import torch

from .. import _ext


def cum(t) -> int:
    return reduce(lambda x, y: x * y, t, 1)


def _padding(inputs, ndim, mode, value, group, group_mode):
    assert mode in ['constant'], mode
    assert group_mode in ['sample', 'oracle'], group_mode
    assert group >= 1, group
    assert len(inputs) > 0, "empty input list"
    assert inputs[0].is_cuda, "hpc version only supports cuda"
    ext = _ext.require()  # list handling in C++ (csrc_torch/ext.cpp)
    try:
        if group > 1:
            return ext.group_pad_nd(list(inputs), ndim, group, 1 if group_mode == 'oracle' else 0, int(value))
        new_x, mask, shapes = ext.pad_nd(list(inputs), ndim, int(value))
        return new_x, mask, shapes
    except RuntimeError as e:  # ext.cpp's checks raise RuntimeError, which its Pad*Forward bindings keep
        msg = str(e)
        if "float32" in msg:
            raise TypeError(msg) from None
        if "-D tensors" in msg or "one CUDA device" in msg:
            raise ValueError(msg) from None
        raise


def _unpad_one(x, shapes, ndim):
    assert x.is_cuda, "hpc version only supports cuda"
    return _ext.require().unpad_nd(x, [int(v) for v in shapes], ndim)


def _unpadding(x, shapes, ndim):
    if isinstance(x, torch.Tensor):
        return _unpad_one(x, shapes, ndim)
    ret = []
    for t, s in zip(x, shapes):
        ret.extend(_unpad_one(t, s, ndim))
    return ret


def Padding1D(inputs: List[torch.Tensor], mode='constant', value: int = 0, group: int = 1, group_mode='sample'):
    return _padding(inputs, 1, mode, value, group, group_mode)


def UnPadding1D(x: Union[torch.Tensor, List[torch.Tensor]], shapes: Union[List, List[List]]) -> List[torch.Tensor]:
    return _unpadding(x, shapes, 1)


def Padding2D(inputs: List[torch.Tensor], mode='constant', value: int = 0, group: int = 1, group_mode='sample'):
    return _padding(inputs, 2, mode, value, group, group_mode)


def UnPadding2D(x: Union[torch.Tensor, List[torch.Tensor]], shapes: Union[List, List[List]]) -> List[torch.Tensor]:
    return _unpadding(x, shapes, 2)


def Padding3D(inputs: List[torch.Tensor], mode='constant', value: int = 0, group: int = 1, group_mode='sample'):
    return _padding(inputs, 3, mode, value, group, group_mode)


def UnPadding3D(x: Union[torch.Tensor, List[torch.Tensor]], shapes: Union[List, List[List]]) -> List[torch.Tensor]:
    return _unpadding(x, shapes, 3)
