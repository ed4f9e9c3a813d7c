#!/usr/bin/env python
"""Generate the V-trace / UPGO return fixtures (tests/golden/returns_{vtrace,upgo}_*.npz) by RUNNING THE REFERENCE.

Runs ``vtrace_nstep_return`` and ``upgo_returns`` of ``/root/reference/hpc_rll/origin`` (imported read-only through
_ref_origin; nothing is copied) on the CPU in fp32 with seeded inputs.  Each fixture stores the inputs, the returns,
and the autograd gradients of sum(ret * G) for the rewards and bootstrap_values.  The V-trace ratios are clipped at 1,
and a quarter of them sit exactly on the clip; the `tie` UPGO cases use small integers, so that r_{t+1} + V_{t+2} ==
V_{t+1} happens often.  Re-run only where the reference is available; it rewrites only the returns_*.npz files:

    python tests/golden/make_returns_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_origin  # noqa: E402

GAMMA, LAMBDA = 0.99, 0.95


def save(name, **blob):
    np.savez_compressed(os.path.join(HERE, "returns_%s.npz" % name), **{k: np.asarray(v) for k, v in blob.items()})


def vtrace_case(O, T, B, seed):
    g = torch.Generator().manual_seed(seed)
    boot = torch.randn(T + 1, B, generator=g)
    reward = torch.randn(T, B, generator=g)
    G = torch.randn(T, B, generator=g)
    ratio = torch.exp(0.5 * torch.randn(T, B, generator=g))
    ratio[torch.rand(T, B, generator=g) < 0.25] = 1.0  # exactly at the clip value
    rhos, cs = ratio.clamp(max=1.0), (0.8 * ratio).clamp(max=1.0)
    bt, rt = boot.clone().requires_grad_(True), reward.clone().requires_grad_(True)
    ret = O.vtrace.vtrace_nstep_return(rhos, cs, rt, bt, GAMMA, LAMBDA)
    gr, gb = torch.autograd.grad((ret * G).sum(), [rt, bt])
    save("vtrace_t%d_b%d" % (T, B), in_clipped_rhos=rhos.numpy(), in_clipped_cs=cs.numpy(), in_reward=reward.numpy(),
         in_bootstrap_values=boot.numpy(), in_grad=G.numpy(), attr_gamma=GAMMA, attr_lambda_=LAMBDA,
         out=ret.detach().numpy(), grad_reward=gr.numpy(), grad_bootstrap_values=gb.numpy())


def upgo_case(O, T, B, seed, tie):
    g = torch.Generator().manual_seed(seed)
    if tie:
        boot = torch.randint(-2, 3, (T + 1, B), generator=g).float()
        rewards = torch.randint(-2, 3, (T, B), generator=g).float()
    else:
        boot = torch.randn(T + 1, B, generator=g)
        rewards = torch.randn(T, B, generator=g)
    G = torch.randn(T, B, generator=g)
    bt, rt = boot.clone().requires_grad_(True), rewards.clone().requires_grad_(True)
    ret = O.upgo.upgo_returns(rt, bt)
    gr, gb = torch.autograd.grad((ret * G).sum(), [rt, bt])
    save("upgo_%st%d_b%d" % ("tie_" if tie else "", T, B), in_rewards=rewards.numpy(),
         in_bootstrap_values=boot.numpy(), in_grad=G.numpy(), out=ret.detach().numpy(), grad_rewards=gr.numpy(),
         grad_bootstrap_values=gb.numpy())


def main():
    O = _ref_origin.load()
    seed = 5150
    for T, B in ((1, 5), (2, 4), (37, 3), (64, 6)):
        seed += 1
        vtrace_case(O, T, B, seed)
        for tie in (False, True):
            seed += 1
            upgo_case(O, T, B, seed, tie)


if __name__ == "__main__":
    main()
