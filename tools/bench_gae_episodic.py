#!/usr/bin/env python
"""Time episode-aware GAE (hpc_rll.rl_utils.gae.gae) against the eager PyTorch loop of its formula, with the existing
normalised GAE module at the same shape as a bandwidth yardstick.

    python tools/bench_gae_episodic.py [--iters 200] [--warmup 20] [--out profiles/bench_gae_episodic_h100.json]

Shapes (each selects one kernel regime, see csrc/gae_episodic.cu)
  wide      T=1024, B=65536   TMA pipeline (ScanPipe with uint8 mask boxes)
  lookback  T=1024, B=64      single-launch T-split with look-back
  generic   T=128,  B=1000    one column per thread (B % 16 != 0)
Inputs: fp32 value / next_value / reward, a bool `done` with 1 % of entries set, traj_flag=None (= done).
For every shape, warm, with CUDA events around back-to-back calls (median of 3 windows):
  new_fwd       gae(...) on inputs that need no gradient
  new_fwdbwd    gae(...) + torch.autograd.grad(adv, (value, next_value, reward), G)
  eager_fwd / eager_fwdbwd   the formula as a Python loop over T (fewer calls: it is 10^3 times slower)
  gae_fwd / gae_fwdbwd       the existing GAE module, value (T+1,B), reward (T,B)
Algorithmic bytes: new op 18 B per element in each direction (3 fp32 + 2 byte reads + 1 fp32 write forward; 1 fp32 +
2 byte reads + 3 fp32 writes backward); existing GAE 12 B per element forward (value, reward, adv) and 12 backward
(grad_adv, grad_value, grad_reward).  Rates are bytes over time; the share of the H100 SXM data-sheet HBM3 bandwidth
(3.35 TB/s) is given beside them.  The card's name and power limit are read in the same run.  Needs a CUDA device.
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
SHAPES = {"wide": (1024, 65536), "lookback": (1024, 64), "generic": (128, 1000)}
GAMMA, LAMBDA = 0.99, 0.95


def eager_gae(value, next_value, reward, done, traj_flag, gamma, lambda_):
    """The formula in eager PyTorch: one op per term, a Python loop over T."""
    if traj_flag is None:
        traj_flag = done
    g = torch.tensor(gamma, dtype=torch.float64).float().to(reward.device)
    gl = torch.tensor(gamma * lambda_, dtype=torch.float64).float().to(reward.device)
    nv = next_value * (1 - done.float())
    delta = (reward + g * nv) - value
    f = gl * (1 - traj_flag.float())
    T = reward.shape[0]
    adv = [None] * T
    adv[T - 1] = delta[T - 1]
    for t in range(T - 2, -1, -1):
        adv[t] = delta[t] + f[t] * adv[t + 1]
    return torch.stack(adv)


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
    from hpc_rll.rl_utils.gae import GAE, gae, gae_data
    res = {"card": card(), "hbm_peak_Bps": HBM_PEAK, "iters": args.iters, "eager_iters": args.eager_iters,
           "gamma": GAMMA, "lambda": LAMBDA, "done_density": 0.01, "rows": []}
    print(json.dumps(res["card"]))
    for regime, (T, B) in SHAPES.items():
        gen = torch.Generator(device="cuda").manual_seed(0)
        v, nv, r, G = (torch.randn(T, B, device="cuda", generator=gen) for _ in range(4))
        done = torch.rand(T, B, device="cuda", generator=gen) < 0.01
        vg, nvg, rg = (t.clone().requires_grad_(True) for t in (v, nv, r))
        value1 = torch.randn(T + 1, B, device="cuda", generator=gen)
        value1g, rg1 = value1.clone().requires_grad_(True), r.clone().requires_grad_(True)
        mod = GAE(T, B)

        def new_fwdbwd():
            adv = gae(gae_data(vg, nvg, rg, done, None), GAMMA, LAMBDA)
            torch.autograd.grad(adv, (vg, nvg, rg), G)

        def eager_fwdbwd():
            adv = eager_gae(vg, nvg, rg, done, None, GAMMA, LAMBDA)
            torch.autograd.grad(adv, (vg, nvg, rg), G)

        def gae_fwdbwd():
            adv = mod(value1g, rg1, GAMMA, LAMBDA)
            torch.autograd.grad(adv, (value1g, rg1), G)

        it, ei = args.iters, args.eager_iters
        row = {"regime": regime, "T": T, "B": B,
               "new_fwd_ms": time_ms(lambda: gae(gae_data(v, nv, r, done, None), GAMMA, LAMBDA), it, args.warmup),
               "new_fwdbwd_ms": time_ms(new_fwdbwd, it, args.warmup),
               "eager_fwd_ms": time_ms(lambda: eager_gae(v, nv, r, done, None, GAMMA, LAMBDA), ei, 1),
               "eager_fwdbwd_ms": time_ms(eager_fwdbwd, ei, 1),
               "gae_fwd_ms": time_ms(lambda: mod(value1, r, GAMMA, LAMBDA), it, args.warmup),
               "gae_fwdbwd_ms": time_ms(gae_fwdbwd, it, args.warmup)}
        n = T * B
        row["new_fwd_bytes"], row["new_fwdbwd_bytes"] = 18 * n, 36 * n
        row["gae_fwd_bytes"], row["gae_fwdbwd_bytes"] = 12 * n, 24 * n
        for k in ("new_fwd", "new_fwdbwd", "gae_fwd", "gae_fwdbwd"):
            row[k + "_GBps"] = row[k + "_bytes"] / (row[k + "_ms"] * 1e-3) / 1e9
            row[k + "_frac_of_peak"] = row[k + "_GBps"] * 1e9 / HBM_PEAK
        row["new_fwd_bw_vs_gae_fwd"] = row["new_fwd_GBps"] / row["gae_fwd_GBps"]
        row["fwd_speedup_vs_eager"] = row["eager_fwd_ms"] / row["new_fwd_ms"]
        row["fwdbwd_speedup_vs_eager"] = row["eager_fwdbwd_ms"] / row["new_fwdbwd_ms"]
        row["max_abs_diff_vs_eager"] = float((gae(gae_data(v, nv, r, done, None), GAMMA, LAMBDA) -
                                              eager_gae(v, nv, r, done, None, GAMMA, LAMBDA)).abs().max())
        res["rows"].append(row)
        print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
