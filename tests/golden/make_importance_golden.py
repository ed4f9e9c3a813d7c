#!/usr/bin/env python
"""Generate the importance-weight and time-batch cross-entropy fixtures (tests/golden/importance_{is,ce}_*.npz) by
RUNNING THE REFERENCE.

Runs ``compute_importance_weights`` (with ``requires_grad=True``) and ``tb_cross_entropy`` of
``/root/reference/hpc_rll/origin`` (imported read-only through _ref_origin; nothing is copied) on the CPU in fp32 with
seeded inputs.  Each fixture stores the inputs, the output, and the autograd gradients of sum(out * G) for every logits
tensor.  Cases: (T, B, N) in {(1,5,3), (2,4,6), (37,3,18), (64,6,16)}, one (B, N) case (importance weights only: the
cross entropy takes a 2-D label), one N = 1 case, one case with -inf-masked entries (never the chosen action; the
behaviour policy has its own mask) and one with identical target and behaviour rows, where every ratio is exactly 1.
Re-run only where the reference is available; it rewrites only the importance_*.npz files:

    python tests/golden/make_importance_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _ref_origin  # noqa: E402


def save(name, **blob):
    np.savez_compressed(os.path.join(HERE, "importance_%s.npz" % name), **{k: np.asarray(v) for k, v in blob.items()})


def inputs(shape, N, seed, masked=False, same=False):
    g = torch.Generator().manual_seed(seed)
    target = 1.5 * torch.randn(*shape, N, generator=g)
    behaviour = target.clone() if same else target + 0.5 * torch.randn(*shape, N, generator=g)
    action = torch.randint(0, N, shape, generator=g)
    G = torch.randn(*shape, generator=g)
    if masked:
        for x in (target, behaviour):
            m = torch.rand(*shape, N, generator=g) < 0.4
            m.scatter_(-1, action.unsqueeze(-1), False)
            x[m] = -float("inf")
    return target, behaviour, action, G


def is_case(O, name, shape, N, seed, **kw):
    target, behaviour, action, G = inputs(shape, N, seed, **kw)
    t, b = target.clone().requires_grad_(True), behaviour.clone().requires_grad_(True)
    rho = O.vtrace.compute_importance_weights(t, b, action, requires_grad=True)
    gt, gb = torch.autograd.grad((rho * G).sum(), [t, b])
    if kw.get("same"):
        assert (rho == 1).all()
    save("is_" + name, in_target_output=target.numpy(), in_behaviour_output=behaviour.numpy(),
         in_action=action.numpy(), in_grad=G.numpy(), out=rho.detach().numpy(), grad_target_output=gt.numpy(),
         grad_behaviour_output=gb.numpy())


def ce_case(O, name, shape, N, seed, **kw):
    logit, _, label, G = inputs(shape, N, seed, **kw)
    x = logit.clone().requires_grad_(True)
    out = O.upgo.tb_cross_entropy(x, label)
    (gl, ) = torch.autograd.grad((out * G).sum(), [x])
    save("ce_" + name, in_logit=logit.numpy(), in_label=label.numpy(), in_grad=G.numpy(), out=out.detach().numpy(),
         grad_logit=gl.numpy())


def main():
    O = _ref_origin.load()
    seed = 8080
    cases = [("t%d_b%d_n%d" % (T, B, N), (T, B), N, {}) for T, B, N in ((1, 5, 3), (2, 4, 6), (37, 3, 18), (64, 6, 16))]
    cases += [("n1_t3_b4", (3, 4), 1, {}), ("masked_t9_b7_n13", (9, 7), 13, dict(masked=True)),
              ("same_t5_b6_n10", (5, 6), 10, dict(same=True))]
    for name, shape, N, kw in cases:
        seed += 1
        is_case(O, name, shape, N, seed, **kw)
        if not kw.get("same"):
            ce_case(O, name, shape, N, seed, **kw)
    is_case(O, "bn_b11_n7", (11, ), 7, seed + 1)


if __name__ == "__main__":
    main()
