#!/usr/bin/env python
"""Time ScatterConnection (hpc_rll.torch_utils.network.scatter_connection) against an eager-torch expression of the same op.

    python tools/bench_scatter_connection.py [--iters 200] [--warmup 20] [--out results.json]

Shapes
  S1  B=M=N=256, H=W=16     the reference's test shape: dense, many entities per cell
  S2  B=64, M=512, N=32, H=W=128   a sparse large map (almost every cell empty)
For each shape and mode ('cover', 'add') it times, warm, with CUDA events around `--iters` back-to-back calls:
  forward   module(x, location)                          (x requires grad, as in training)
  backward  torch.autograd.grad(out, x, G, retain_graph=True)
for the module and for `eager_scatter` below.  Algorithmic bytes (formulas in `fwd_bytes` / `bwd_bytes`) over the
measured time give a rate, reported as a fraction of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  Which
backward kernel ran is read from a separate torch.profiler pass.  The card's name and power limit are read in the same
run.  Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
SHAPES = {"S1": (256, 256, 256, 16, 16), "S2": (64, 512, 32, 128, 128)}


def fwd_bytes(B, M, N, H, W):
    """read x (B*M*N fp32) and location (B*M*2 int64), write out (B*N*H*W fp32) once"""
    return 4 * B * M * N + 16 * B * M + 4 * B * N * H * W


def bwd_bytes(B, M, N, H, W):
    """read location, write grad_x once, and read the cheaper of: the whole grad_out planes (B*N*H*W fp32), or one
    32-byte sector per (entity, channel)"""
    return 16 * B * M + 4 * B * M * N + min(4 * B * N * H * W, 32 * B * M * N)


def eager_scatter(x, location, H, W, mode):
    """The same op in eager torch (all locations in range): scatter into a (B, H*W, N) map, then lay it out
    (B, N, H, W).  Autograd gives the gather backward."""
    B, M, N = x.shape
    cell = (location[..., 0] * W + location[..., 1]).unsqueeze(-1).expand(B, M, N)
    out = x.new_zeros(B, H * W, N)
    out = out.scatter_add(1, cell, x) if mode == "add" else out.scatter(1, cell, x)
    return out.view(B, H, W, N).permute(0, 3, 1, 2).contiguous()


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = r.stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def backward_kernel(mod, x, loc, G):
    out = mod(x, loc)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.autograd.grad(out, x, G)
        torch.cuda.synchronize()
    ks = sorted({k for e in prof.events() for k in re.findall(r"scatter_conn_bwd_\w+", e.name)})
    return ",".join(ks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from hpc_rll.torch_utils.network.scatter_connection import ScatterConnection
    res = {"card": card(), "hbm_peak_Bps": HBM_PEAK, "iters": args.iters, "rows": []}
    print(json.dumps(res["card"]))
    for sname, (B, M, N, H, W) in SHAPES.items():
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(B, M, N, device="cuda", generator=g).requires_grad_(True)
        loc = torch.stack([torch.randint(0, H, (B, M), device="cuda", generator=g),
                           torch.randint(0, W, (B, M), device="cuda", generator=g)], 2)
        G = torch.randn(B, N, H, W, device="cuda", generator=g)
        fb, bb = fwd_bytes(B, M, N, H, W), bwd_bytes(B, M, N, H, W)
        for mode in ("cover", "add"):
            mod = ScatterConnection(B, M, N, H, W, mode)
            impls = {"module": lambda x_, m=mod: m(x_, loc), "eager": lambda x_, m=mode: eager_scatter(x_, loc, H, W, m)}
            row = {"shape": sname, "B": B, "M": M, "N": N, "H": H, "W": W, "mode": mode, "fwd_bytes": fb,
                   "bwd_bytes": bb, "bwd_kernel": backward_kernel(mod, x, loc, G)}
            for name, f in impls.items():
                out = f(x)
                row[name + "_fwd_ms"] = time_ms(lambda: f(x), args.iters, args.warmup)
                row[name + "_bwd_ms"] = time_ms(lambda: torch.autograd.grad(out, x, G, retain_graph=True), args.iters,
                                                args.warmup)
            ref = impls["eager"](x).detach()
            row["max_abs_diff_vs_eager"] = float((impls["module"](x).detach() - ref).abs().max())
            for k in ("fwd", "bwd"):
                t = row["module_%s_ms" % k] * 1e-3
                row["module_%s_frac_of_peak" % k] = (fb if k == "fwd" else bb) / t / HBM_PEAK
                row["%s_speedup_vs_eager" % k] = row["eager_%s_ms" % k] / row["module_%s_ms" % k]
            res["rows"].append(row)
            print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
