#!/usr/bin/env python
"""Time the λ-returns (hpc_rll.rl_utils.td.generalized_lambda_returns) against the eager PyTorch loop of their formula.

    python tools/bench_lambda_returns.py [--iters 200] [--warmup 20] [--out profiles/bench_lambda_returns_h100.json]

Cases (each selects one kernel regime, see csrc/lambda_returns.cu)
  wide_scalar   T=1024, B=65536  scalar γ / λ, no done   TMA pipeline, 12 B per element each way
  wide_tensor   T=1024, B=65536  (T,B) γ and λ, done     TMA pipeline, 21 B per element each way
  lookback      T=1024, B=64     (T,B) γ and λ, done     single-launch T-split with look-back
  generic       T=128,  B=1000   (T,B) γ and λ, done     one column per thread (B % 16 != 0)
`done` is a bool mask with 1 % of entries set.  For every case, warm, with CUDA events around back-to-back calls
(median of 3 windows):
  new_fwd / new_fwdbwd       the op on inputs that need no gradient / + torch.autograd.grad to bootstrap and rewards
  eager_fwd / eager_fwdbwd   the formula as a Python loop over T (fewer calls: it is 10^3 times slower)
Algorithmic bytes per element, each direction: forward reads V, r (+ γ, λ as fp32, + done as a byte) and writes R;
backward reads G (+ γ, λ, done) and writes grad_V and grad_r.  Rates are bytes over time; the share of the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s) is given beside them.  The card's name and power limit are read in the same run.
Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
CASES = {"wide_scalar": (1024, 65536, False), "wide_tensor": (1024, 65536, True), "lookback": (1024, 64, True),
         "generic": (128, 1000, True)}
GAMMA, LAMBDA = 0.99, 0.95


def eager_returns(bootstrap, rewards, gammas, lambda_, done):
    """generalized_lambda_returns in eager PyTorch: one op per term, a Python loop over T."""
    if not isinstance(gammas, torch.Tensor):
        gammas = gammas * torch.ones_like(rewards)
    if not isinstance(lambda_, torch.Tensor):
        lambda_ = lambda_ * torch.ones_like(rewards)
    V = bootstrap[1:]
    d = gammas * lambda_
    e = gammas - d
    T = rewards.shape[0]
    R = [None] * T
    if done is None:
        R[T - 1] = rewards[T - 1] + gammas[T - 1] * V[T - 1]
        for t in range(T - 2, -1, -1):
            R[t] = rewards[t] + d[t] * R[t + 1] + e[t] * V[t]
    else:
        m = 1 - done.float()
        R[T - 1] = rewards[T - 1] + (m[T - 1] * gammas[T - 1]) * V[T - 1]
        for t in range(T - 2, -1, -1):
            R[t] = rewards[t] + m[t] * (d[t] * R[t + 1] + e[t] * V[t])
    return torch.stack(R)


def time_ms(fn, iters, warmup, windows=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / iters)
    return sorted(out)[len(out) // 2]


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = r.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--eager-iters", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from hpc_rll.rl_utils.td import generalized_lambda_returns as glr
    res = {"card": card(), "hbm_peak_Bps": HBM_PEAK, "iters": args.iters, "eager_iters": args.eager_iters,
           "gamma": GAMMA, "lambda": LAMBDA, "done_density": 0.01, "rows": []}
    print(json.dumps(res["card"]))
    for case, (T, B, tensors) in CASES.items():
        gen = torch.Generator(device="cuda").manual_seed(0)
        boot = torch.randn(T + 1, B, device="cuda", generator=gen)
        r, G = (torch.randn(T, B, device="cuda", generator=gen) for _ in range(2))
        if tensors:
            gam = 0.9 + 0.1 * torch.rand(T, B, device="cuda", generator=gen)
            lam = torch.rand(T, B, device="cuda", generator=gen)
            done = torch.rand(T, B, device="cuda", generator=gen) < 0.01
        else:
            gam, lam, done = GAMMA, LAMBDA, None
        bg, rg = boot.clone().requires_grad_(True), r.clone().requires_grad_(True)

        def new_fwdbwd():
            torch.autograd.grad(glr(bg, rg, gam, lam, done), (bg, rg), G)

        def eager_fwdbwd():
            torch.autograd.grad(eager_returns(bg, rg, gam, lam, done), (bg, rg), G)

        it, ei = args.iters, args.eager_iters
        row = {"case": case, "T": T, "B": B, "tensor_gamma_lambda_done": tensors,
               "new_fwd_ms": time_ms(lambda: glr(boot, r, gam, lam, done), it, args.warmup),
               "new_fwdbwd_ms": time_ms(new_fwdbwd, it, args.warmup),
               "eager_fwd_ms": time_ms(lambda: eager_returns(boot, r, gam, lam, done), ei, 1),
               "eager_fwdbwd_ms": time_ms(eager_fwdbwd, ei, 1)}
        per_elem = 12 + (9 if tensors else 0)
        row["fwd_bytes"], row["fwdbwd_bytes"] = per_elem * T * B, 2 * per_elem * T * B
        for k, nb in (("new_fwd", "fwd_bytes"), ("new_fwdbwd", "fwdbwd_bytes")):
            row[k + "_GBps"] = row[nb] / (row[k + "_ms"] * 1e-3) / 1e9
            row[k + "_frac_of_peak"] = row[k + "_GBps"] * 1e9 / HBM_PEAK
        row["fwd_speedup_vs_eager"] = row["eager_fwd_ms"] / row["new_fwd_ms"]
        row["fwdbwd_speedup_vs_eager"] = row["eager_fwdbwd_ms"] / row["new_fwdbwd_ms"]
        row["max_abs_diff_vs_eager"] = float((glr(boot, r, gam, lam, done) -
                                              eager_returns(boot, r, gam, lam, done)).abs().max())
        res["rows"].append(row)
        print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
