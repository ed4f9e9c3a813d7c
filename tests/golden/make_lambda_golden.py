#!/usr/bin/env python
"""Generate the λ-return fixtures (tests/golden/lambda_*.npz) by RUNNING THE REFERENCE.

Runs ``generalized_lambda_returns`` and ``multistep_forward_view`` of ``/root/reference/hpc_rll/origin/td.py``
(imported read-only through _ref_origin; nothing is copied) on the CPU in fp32 with seeded inputs, done=None.  Each
fixture stores the inputs, the returns, and the autograd gradients of sum(ret * G) for bootstrap_values and rewards.
A scalar γ / λ is stored as a 0-d array; origin's multistep_forward_view indexes its discounts, so it is handed
``γ * ones_like(rewards)``, which is what the scalar means.  Re-run only where the reference is available; it rewrites
only the lambda_*.npz files:

    python tests/golden/make_lambda_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_origin  # noqa: E402


def case(O, fn, form, T, B, seed):
    g = torch.Generator().manual_seed(seed)
    offset = 1 if fn == "gen" else 0
    boot = torch.randn(T + offset, B, generator=g)
    rewards = torch.randn(T, B, generator=g)
    G = torch.randn(T, B, generator=g)
    if form == "tensor":
        gammas = 0.5 + 0.5 * torch.rand(T, B, generator=g)
        lam = torch.rand(T, B, generator=g)
    else:
        gammas, lam = 0.99, 0.95
    bt, rt = boot.clone().requires_grad_(True), rewards.clone().requires_grad_(True)
    if fn == "gen":
        ret = O.td.generalized_lambda_returns(bt, rt, gammas, lam)
    else:
        full = (lambda x: x * torch.ones_like(rewards)) if form == "scalar" else (lambda x: x)
        ret = O.td.multistep_forward_view(bt, rt, full(gammas), full(lam))
    gb, gr = torch.autograd.grad((ret * G).sum(), [bt, rt])
    as_np = (lambda x: np.asarray(x, np.float64)) if form == "scalar" else (lambda x: x.numpy())
    blob = {"in_bootstrap_values": boot.numpy(), "in_rewards": rewards.numpy(), "in_gammas": as_np(gammas),
            "in_lambda_": as_np(lam), "in_grad": G.numpy(), "out": ret.detach().numpy(),
            "grad_bootstrap_values": gb.numpy(), "grad_rewards": gr.numpy(), "offset": np.asarray(offset)}
    np.savez_compressed(os.path.join(HERE, "lambda_%s_%s_t%d_b%d.npz" % (fn, form, T, B)), **blob)


def main():
    O = _ref_origin.load()
    seed = 4242
    for T, B in ((1, 5), (2, 4), (37, 3), (64, 6)):
        for fn in ("gen", "msv"):
            for form in ("scalar", "tensor"):
                seed += 1
                case(O, fn, form, T, B, seed)


if __name__ == "__main__":
    main()
