"""Padding / UnPadding on the GPU (one CUDA launch through the C ABI) vs the oracle and the origin-generated
fixtures.  Pure data movement: everything must be BIT-EXACT.  Mirrors the assertions of the reference's
tests/test_padding.py (shapes, group counts, round trip against the size-sorted inputs)."""
import os

import numpy as np
import pytest
import torch

from oracle import padding_oracle as po
from tests._golden import GOLDEN_DIR, names
from tests._gpu import host, need_cuda

pytestmark = pytest.mark.gpu


def mods():
    import hpc_rll.rl_utils.padding as H
    return {1: (H.Padding1D, H.UnPadding1D), 2: (H.Padding2D, H.UnPadding2D), 3: (H.Padding3D, H.UnPadding3D)}


@pytest.mark.parametrize("name", names("padding"))
def test_padding_vs_golden(name):
    need_cuda()
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    n, ndim, value = int(z["n"]), int(z["ndim"]), int(z["value"])
    xs = [z["x%d" % i] for i in range(n)]
    pad, unpad = mods()[ndim]
    new_x, mask, shapes = pad([torch.from_numpy(x).cuda() for x in xs], value=value)
    torch.cuda.synchronize()
    assert new_x.dtype == torch.float32 and mask.dtype == torch.int32
    assert np.array_equal(host(new_x), z["new_x"])
    assert np.array_equal(host(mask).astype(np.float32), z["mask"])
    assert shapes == [int(v) for s in xs for v in s.shape]
    for a, b in zip(unpad(new_x, shapes), xs):
        assert np.array_equal(host(a), b)


RANGES = {1: [(32, 128)], 2: [(48, 80), (32, 64)], 3: [(24, 32), (24, 32), (32, 40)]}  # tests/test_padding.py:10-13


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_reference_test_shapes_and_group_modes(ndim):
    need_cuda()
    B = 64
    rng = np.random.default_rng(ndim)
    shapes = [tuple(int(rng.integers(lo, hi)) for lo, hi in RANGES[ndim]) for _ in range(B)]
    data = [torch.randn(*s).cuda() for s in shapes]
    pad, unpad = mods()[ndim]
    max_shape = tuple(max(s[d] for s in shapes) for d in range(ndim))
    x, m, ori = pad(data)
    assert x.shape == (B, ) + max_shape and m.shape == (B, ) + max_shape
    ox, om, _ = po.pad([host(d) for d in data])
    assert np.array_equal(host(x), ox) and np.array_equal(host(m), om)
    for item, new_item in zip(data, unpad(x, ori)):
        assert item.eq(new_item).all()
    sorted_data = sorted(data, key=lambda t: po.cum(t.shape))
    for mode in ("sample", "oracle"):
        px, pm, ps = pad(data, group=4, group_mode=mode)
        assert len(px) <= 4 and len(pm) <= 4 and len(ps) <= 4
        assert sum(len(i) for i in px) == B and sum(len(i) for i in pm) == B
        if mode == "oracle":
            assert len(px) == 4
        out = unpad(px, ps)
        assert len(out) == B
        for item, new_item in zip(sorted_data, out):
            assert item.eq(new_item).all()
        # every group is padded to its own max and masks count the real elements
        k = 0
        for gx, gm in zip(px, pm):
            cnt = gx.shape[0]
            grp = sorted_data[k:k + cnt]
            assert tuple(gx.shape[1:]) == tuple(max(t.shape[d] for t in grp) for d in range(ndim))
            assert int(gm.sum()) == sum(t.numel() for t in grp)
            k += cnt
    same = [torch.randn(*([32] * ndim if ndim < 3 else [8, 8, 8])).cuda() for _ in range(B)]
    sx, _, _ = pad(same, group=4)
    assert len(sx) == 1 and sx[0].shape[0] == B


def test_padding_value_large_and_empty_rows():
    need_cuda()
    pad, unpad = mods()[2]
    rng = np.random.default_rng(9)
    # large items (many CTAs per item), a non-zero pad value, and a tensor with a zero-length dim
    data = [torch.randn(700, 900).cuda(), torch.randn(1024, 333).cuda(), torch.randn(0, 5).cuda(),
            torch.randn(1, 1).cuda()]
    x, m, shp = pad(data, value=7)
    ox, om, _ = po.pad([host(d) for d in data], 7)
    assert np.array_equal(host(x), ox) and np.array_equal(host(m), om)
    back = unpad(x, shp)
    for a, b in zip(back, data):
        assert a.shape == b.shape and a.eq(b).all()
    # more tensors than one parameter-space batch holds (512)
    many = [torch.full((int(rng.integers(1, 6)), ), float(i)).cuda() for i in range(1300)]
    p1, m1, s1 = mods()[1][0](many)
    o1, om1, _ = po.pad([host(d) for d in many])
    assert np.array_equal(host(p1), o1) and np.array_equal(host(m1), om1)
    for a, b in zip(mods()[1][1](p1, s1), many):
        assert a.eq(b).all()


def test_padding_argument_errors():
    need_cuda()
    pad, _ = mods()[2]
    with pytest.raises(ValueError):
        pad([torch.zeros(3).cuda()])
    with pytest.raises(TypeError):
        pad([torch.zeros(3, 3, dtype=torch.float64).cuda()])
    with pytest.raises(AssertionError):
        pad([torch.zeros(3, 3)])


def test_reference_named_pybind_bindings():
    """The thin torch/pybind layer exports the reference's 11 padding bindings (src/rl_utils/entry.cpp:9-20)
    with the same call conventions as hpc_rll/rl_utils/padding.py uses them."""
    need_cuda()
    from di_hpc_b200 import _ext
    E = _ext.require()
    assert E is not None, "hpc_rl_utils_b200 extension missing (python -m di_hpc_b200.build_torch_ext)"
    rng = np.random.default_rng(3)
    shapes = [(int(rng.integers(3, 9)), int(rng.integers(2, 7))) for _ in range(20)]
    data = [torch.randn(*s).cuda() for s in shapes]
    x, m = E.Pad2DForward(data, 0)
    ox, om, _ = po.pad([host(d) for d in data])
    assert np.array_equal(host(x), ox) and np.array_equal(host(m), om)
    flat = [int(v) for s in shapes for v in s]
    for a, b in zip(E.Unpad2DForward(x, flat), data):
        assert a.eq(b).all()
    srt = sorted(data, key=lambda t: t.numel())
    res = E.oracle_split_group(srt, 3)
    group_shape, group_idx = res[:-1], res[-1]
    assert len(group_idx) == len(group_shape) + 1 == 4 and group_idx[0] == 0 and group_idx[-1] == len(srt)
    for g, shp in enumerate(group_shape):
        grp = srt[group_idx[g]:group_idx[g + 1]]
        assert list(shp) == [max(t.shape[0] for t in grp), max(t.shape[1] for t in grp)]
    res_s = E.sample_split_group(srt, 4)
    assert res_s[-1][0] == 0 and res_s[-1][-1] == len(srt) and len(res_s) - 1 <= 4
    cnt = [group_idx[i + 1] - group_idx[i] for i in range(3)]
    mx = [v for s in group_shape for v in s]
    gid = [g for g in range(3) for _ in range(cnt[g])]
    gx, gm = E.GroupPad2DForward(srt, cnt, mx, gid, group_idx, 0)
    assert len(gx) == 3 and [t.shape[0] for t in gx] == cnt
    k = 0
    for g in range(3):
        ogx, ogm, _ = po.pad([host(t) for t in srt[k:k + cnt[g]]])
        assert np.array_equal(host(gx[g]), ogx) and np.array_equal(host(gm[g]), ogm)
        k += cnt[g]
