#!/usr/bin/env python
"""Generate the ScatterConnection fixtures (tests/golden/scatter_*.npz) by RUNNING THE REFERENCE.

Runs ``/root/reference/hpc_rll/origin/scatter_connection.py`` (imported read-only; nothing is copied) on the CPU with
seeded inputs.  Each fixture stores the inputs, the forward output, and grad_x = autograd of sum(out * G) for a random
upstream G.  Locations are all in range: origin does not check them, and the library drops out-of-range entities.
Re-run only where the reference is available; it rewrites only the scatter_*.npz files:

    python tests/golden/make_scatter_golden.py
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_origin  # noqa: E402


def load_origin():
    spec = importlib.util.spec_from_file_location(
        "ref_origin_scatter", os.path.join(_ref_origin.REF_ROOT, "hpc_rll", "origin", "scatter_connection.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def case_scatter(S, name, B, M, N, H, W, scatter_type, seed, one_cell=False, exponents=False):
    g = torch.Generator().manual_seed(seed)
    if exponents:  # magnitudes over ~2^-20 .. 2^20 with both signs: the order of an fp32 sum changes its bits
        x = torch.randn(B, M, N, generator=g) * torch.pow(2.0, torch.randint(-20, 21, (B, M, N), generator=g).float())
    else:
        x = torch.randn(B, M, N, generator=g)
    if one_cell:
        loc = torch.zeros(B, M, 2, dtype=torch.int64)
        loc[..., 0] = H - 1
        loc[..., 1] = W // 2
    else:
        loc = torch.stack([torch.randint(0, H, (B, M), generator=g), torch.randint(0, W, (B, M), generator=g)], dim=2)
    G = torch.randn(B, N, H, W, generator=g)
    xr = x.clone().requires_grad_(True)
    out = S.ScatterConnection(scatter_type)(xr, (H, W), loc)
    (grad_x,) = torch.autograd.grad((out * G).sum(), [xr])
    blob = {"in_x": x.numpy(), "in_location": loc.numpy(), "in_G": G.numpy(), "out": out.detach().numpy(),
            "grad_x": grad_x.numpy(), "H": np.asarray(H), "W": np.asarray(W), "scatter_type": np.asarray(scatter_type)}
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **blob)


def main():
    S = load_origin()
    s = 777
    for k, mode in enumerate(("cover", "add")):
        case_scatter(S, "scatter_%s_collide_b2_m300_n5_h5w6" % mode, 2, 300, 5, 5, 6, mode, s + 10 * k + 1)
        case_scatter(S, "scatter_%s_onecell_b3_m17_n4_h3w3" % mode, 3, 17, 4, 3, 3, mode, s + 10 * k + 2,
                     one_cell=True)
        case_scatter(S, "scatter_%s_n1_b3_m40_h4w4" % mode, 3, 40, 1, 4, 4, mode, s + 10 * k + 3)
        case_scatter(S, "scatter_%s_odd_b2_m50_n7_h3w5" % mode, 2, 50, 7, 3, 5, mode, s + 10 * k + 4)
        case_scatter(S, "scatter_%s_exp_b2_m200_n3_h2w4" % mode, 2, 200, 3, 2, 4, mode, s + 10 * k + 5,
                     exponents=True)


if __name__ == "__main__":
    main()
