"""CPU oracle of ScatterConnection (numpy).  TEST INFRASTRUCTURE ONLY: the product never imports it.

It restates hpc_rll/origin/scatter_connection.py in origin's order.  Origin zero-fills the map and runs torch's CPU
scatter_ / scatter_add_ over the entities in (b, m) order.  So a cell holds the LAST entity's row (cover), or the
sequential fp32 sum starting from +0.0 in increasing m (add).  The loop below walks m in increasing order and updates
every sample at once.  Within one m each sample touches one cell, so no element is updated twice in one step, and each
update is one IEEE fp32 addition or copy in the input dtype.  The committed origin fixtures (tests/golden/scatter_*.npz)
pin it bit for bit (tests/test_scatter_connection_cpu.py).

Deliberate deviation from origin: an entity with y outside [0,H) or x outside [0,W) is dropped.  Origin flattens
b*H*W + y*W + x without a check.  Backward: grad_x[b,m,:] = grad_out[b,:,y,x], 0 for dropped entities.
"""
import numpy as np


def _cells(location, H, W):
    """(B, M) flat cell index of every entity, -1 where the location is outside the map."""
    loc = np.asarray(location, dtype=np.int64)
    y, x = loc[..., 0], loc[..., 1]
    valid = (y >= 0) & (y < H) & (x >= 0) & (x < W)
    return np.where(valid, y * W + x, -1)


def scatter_connection_forward(x, location, H, W, scatter_type="cover"):
    """x (B,M,N), location (B,M,2) int64 (y, x) -> out (B,N,H,W) ('cover' or 'add'; out-of-range entities dropped)."""
    assert scatter_type in ("cover", "add")
    x = np.ascontiguousarray(x)
    B, M, N = x.shape
    cells = _cells(location, H, W)
    assert cells.shape == (B, M)
    out = np.zeros((B, N, H * W), dtype=x.dtype)
    for m in range(M):
        b = np.nonzero(cells[:, m] >= 0)[0]
        c = cells[b, m]
        if scatter_type == "add":
            out[b, :, c] = out[b, :, c] + x[b, m, :]
        else:
            out[b, :, c] = x[b, m, :]
    return out.reshape(B, N, H, W)


def scatter_connection_backward(grad_out, location):
    """grad_out (B,N,H,W), location (B,M,2) -> grad_x (B,M,N) = grad_out[b, :, y_m, x_m] (0 for dropped entities)."""
    g = np.ascontiguousarray(grad_out)
    B, N, H, W = g.shape
    cells = _cells(location, H, W)
    gt = g.reshape(B, N, H * W).transpose(0, 2, 1)  # (B, HW, N)
    gx = gt[np.arange(B)[:, None], np.maximum(cells, 0)]  # (B, M, N)
    gx[cells < 0] = 0
    return np.ascontiguousarray(gx, dtype=g.dtype)
