#!/usr/bin/env python
"""Time the V-trace target and the UPGO return (hpc_rll.rl_utils.vtrace.vtrace_nstep_return,
hpc_rll.rl_utils.upgo.upgo_returns) against the eager PyTorch loops of their formulas.

    python tools/bench_vtrace_upgo_returns.py [--iters 200] [--warmup 20] [--out profiles/bench_vtrace_upgo_returns_h100.json]

Cases (each selects one kernel regime, see csrc/vtrace_upgo_returns.cu)
  wide      T=1024, B=65536   TMA pipeline
  lookback  T=1024, B=64      single-launch T-split with look-back
  generic   T=128,  B=1000    one column per thread (UPGO's backward: B % 16 != 0; V-trace: forced with config 99)
For every case and op, warm, with CUDA events around back-to-back calls (median of 3 windows):
  new_fwd / new_fwdbwd       the op on inputs that need no gradient / + torch.autograd.grad to rewards and bootstrap
  eager_fwd / eager_fwdbwd   the formula as a Python loop over T (fewer calls: it is 10^3 times slower)
Algorithmic bytes per element: V-trace reads V, r, ρ, c and writes R forward (20 B), reads G, ρ, c and writes grad_V,
grad_r backward (20 B); UPGO reads V, r and writes R forward (12 B, 13 B with the ℓ byte saved for a backward), reads G
and ℓ and writes grad_V, grad_r backward (13 B).  Rates are bytes over time; the share of the H100 SXM data-sheet HBM3
bandwidth (3.35 TB/s) is given beside them.  The card's name and power limit are read in the same run.
Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_lambda_returns import HBM_PEAK, card, time_ms  # noqa: E402

CASES = {"wide": (1024, 65536, -1), "lookback": (1024, 64, -1), "generic": (128, 1000, 99)}
GAMMA, LAMBDA = 0.99, 0.95
OP_LAMBDA_RETURNS = 11
# bytes per element: forward, forward+backward (the forward that feeds a backward also writes the ℓ byte)
BYTES = {"vtrace": (20, 40), "upgo": (12, 26)}


def eager_vtrace(rho, c, reward, boot):
    """vtrace_nstep_return in eager PyTorch: one op per term, a Python loop over T."""
    deltas = rho * (reward + GAMMA * boot[1:] - boot[:-1])
    factor = GAMMA * LAMBDA
    item = 0.
    out = [None] * reward.shape[0]
    for t in reversed(range(reward.shape[0])):
        item = deltas[t] + factor * c[t] * item
        out[t] = boot[t] + item
    return torch.stack(out)


def eager_upgo(rewards, boot):
    """upgo_returns in eager PyTorch: ℓ from three tensor ops, then the γ = 1 λ-return loop."""
    lam = (rewards + boot[1:]) >= boot[:-1]
    lam = torch.cat([lam[1:], torch.ones_like(lam[-1:])], dim=0).float()
    T = rewards.shape[0]
    out = [None] * T
    out[T - 1] = rewards[T - 1] + boot[T]
    for t in range(T - 2, -1, -1):
        out[t] = rewards[t] + lam[t] * out[t + 1] + (1 - lam[t]) * boot[t + 1]
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--eager-iters", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from di_hpc_b200 import _abi
    from hpc_rll.rl_utils.upgo import upgo_returns
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    res = {"card": card(), "hbm_peak_Bps": HBM_PEAK, "iters": args.iters, "eager_iters": args.eager_iters,
           "gamma": GAMMA, "lambda": LAMBDA, "rows": []}
    print(json.dumps(res["card"]))
    for case, (T, B, cfg) in CASES.items():
        gen = torch.Generator(device="cuda").manual_seed(0)
        boot = torch.randn(T + 1, B, device="cuda", generator=gen)
        r, G = (torch.randn(T, B, device="cuda", generator=gen) for _ in range(2))
        ratio = torch.exp(0.5 * torch.randn(T, B, device="cuda", generator=gen))
        rho, c = ratio.clamp(max=1.0), (0.8 * ratio).clamp(max=1.0)
        bg, rg = boot.clone().requires_grad_(True), r.clone().requires_grad_(True)
        ops = {"vtrace": (lambda b, x: vtrace_nstep_return(rho, c, x, b, GAMMA, LAMBDA),
                          lambda b, x: eager_vtrace(rho, c, x, b)),
               "upgo": (lambda b, x: upgo_returns(x, b), lambda b, x: eager_upgo(x, b))}
        _abi.set_config(OP_LAMBDA_RETURNS, cfg)
        try:
            for op, (new, eager) in ops.items():
                def new_fwdbwd():
                    torch.autograd.grad(new(bg, rg), (bg, rg), G)

                def eager_fwdbwd():
                    torch.autograd.grad(eager(bg, rg), (bg, rg), G)

                it, ei = args.iters, args.eager_iters
                row = {"op": op, "case": case, "T": T, "B": B, "config": cfg,
                       "new_fwd_ms": time_ms(lambda: new(boot, r), it, args.warmup),
                       "new_fwdbwd_ms": time_ms(new_fwdbwd, it, args.warmup),
                       "eager_fwd_ms": time_ms(lambda: eager(boot, r), ei, 1),
                       "eager_fwdbwd_ms": time_ms(eager_fwdbwd, ei, 1)}
                fb, fbb = BYTES[op]
                row["fwd_bytes"], row["fwdbwd_bytes"] = fb * T * B, fbb * T * B
                for k, nb in (("new_fwd", "fwd_bytes"), ("new_fwdbwd", "fwdbwd_bytes")):
                    row[k + "_GBps"] = row[nb] / (row[k + "_ms"] * 1e-3) / 1e9
                    row[k + "_frac_of_peak"] = row[k + "_GBps"] * 1e9 / HBM_PEAK
                row["fwd_speedup_vs_eager"] = row["eager_fwd_ms"] / row["new_fwd_ms"]
                row["fwdbwd_speedup_vs_eager"] = row["eager_fwdbwd_ms"] / row["new_fwdbwd_ms"]
                row["max_abs_diff_vs_eager"] = float((new(boot, r) - eager(boot, r)).abs().max())
                res["rows"].append(row)
                print(json.dumps(row))
        finally:
            _abi.set_config(OP_LAMBDA_RETURNS, -1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
