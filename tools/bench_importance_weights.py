#!/usr/bin/env python
"""Time the importance weights and the time-batch cross entropy (hpc_rll.rl_utils.vtrace.compute_importance_weights,
hpc_rll.rl_utils.upgo.tb_cross_entropy) against origin's formulas in eager PyTorch.

    python tools/bench_importance_weights.py [--iters 100] [--warmup 10] [--out profiles/bench_importance_weights_h100.json]

Cases (each selects one row-kernel path, see csrc/softmax_rows.cuh)
  n16    T=512, B=32768, N=16     register rows, 128-bit chunks (width 4)
  n18    T=512, B=32768, N=18     register rows, 64-bit chunks (width 2, two lanes per row)
  n9     T=512, B=32768, N=9      rows staged through shared memory
  n1000  T=512, B=2048,  N=1000   one warp per row (looping kernel); each logits tensor is 4.2 GB
For every case and op, warm, with CUDA events around back-to-back calls (median of 3 windows):
  new_fwd / new_fwdbwd     the op on inputs that need no gradient / + torch.autograd.grad to every logits tensor
  eager_*                  origin's formula: two torch.distributions.Categorical with default argument validation (as
                           DI-engine runs it; each distribution and log_prob checks its arguments on the host) and with
                           validate_args=False; the cross entropy is -F.cross_entropy, which validates nothing
Algorithmic bytes per row, from the shapes: the importance-weights forward reads two logits rows, the action and writes
ρ (8N + 12); its backward reads G and ρ and writes c (12), then per logits tensor reads the row, the action and c and
writes the gradient row (8N + 12 each).  The cross-entropy forward reads one row and the label and writes the output
(4N + 12); its backward reads the row, the label and G and writes the gradient row (8N + 12).  Rates are bytes over
time; the share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s) is given beside them.  The card's name and power
limit are read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_lambda_returns import HBM_PEAK, card, time_ms  # noqa: E402

CASES = {"n16": (512, 32768, 16), "n18": (512, 32768, 18), "n9": (512, 32768, 9), "n1000": (512, 2048, 1000)}


def bytes_per_row(op, N):
    """(forward, forward + backward) algorithmic bytes per row"""
    if op == "importance_weights":
        fwd = 8 * N + 12
        return fwd, fwd + 12 + 2 * (8 * N + 12)
    fwd = 4 * N + 12
    return fwd, fwd + 8 * N + 12


def eager_is(t, b, a, validate):
    """origin's compute_importance_weights body; validate=None: torch's default argument validation"""
    dt = torch.distributions.Categorical(logits=t, validate_args=validate)
    db = torch.distributions.Categorical(logits=b, validate_args=validate)
    return torch.exp(dt.log_prob(a) - db.log_prob(a))


def eager_ce(x, label):
    """origin's tb_cross_entropy body (2-D label, no mask)"""
    T, B = label.shape
    return -F.cross_entropy(x.reshape(-1, x.shape[-1]), label.reshape(-1), reduction='none').reshape(T, B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--eager-iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from hpc_rll.rl_utils.upgo import tb_cross_entropy
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    res = {"card": card(), "hbm_peak_Bps": HBM_PEAK, "iters": args.iters, "eager_iters": args.eager_iters, "rows": []}
    print(json.dumps(res["card"]))
    for case, (T, B, N) in CASES.items():
        gen = torch.Generator(device="cuda").manual_seed(0)
        t = 1.5 * torch.randn(T, B, N, device="cuda", generator=gen)
        b = t + 0.5 * torch.randn(T, B, N, device="cuda", generator=gen)
        a = torch.randint(0, N, (T, B), device="cuda", generator=gen)
        G = torch.randn(T, B, device="cuda", generator=gen)
        tg, bg = t.clone().requires_grad_(True), b.clone().requires_grad_(True)
        ops = {
            "importance_weights": (
                lambda x, y: compute_importance_weights(x, y, a, requires_grad=x.requires_grad),
                {"eager_validate": lambda x, y: eager_is(x, y, a, None),
                 "eager_novalidate": lambda x, y: eager_is(x, y, a, False)}, (tg, bg)),
            "tb_cross_entropy": (lambda x, y: tb_cross_entropy(x, a), {"eager": lambda x, y: eager_ce(x, a)}, (tg, )),
        }
        for op, (new, eagers, wrt) in ops.items():
            it, ei, w = args.iters, args.eager_iters, args.warmup
            row = {"op": op, "case": case, "T": T, "B": B, "N": N,
                   "new_fwd_ms": time_ms(lambda: new(t, b), it, w),
                   "new_fwdbwd_ms": time_ms(lambda: torch.autograd.grad(new(tg, bg), wrt, G), it, w)}
            for name, fn in eagers.items():
                row[name + "_fwd_ms"] = time_ms(lambda: fn(t, b), ei, 2)
                row[name + "_fwdbwd_ms"] = time_ms(lambda: torch.autograd.grad(fn(tg, bg), wrt, G), ei, 2)
                row[name + "_fwd_speedup"] = row[name + "_fwd_ms"] / row["new_fwd_ms"]
                row[name + "_fwdbwd_speedup"] = row[name + "_fwdbwd_ms"] / row["new_fwdbwd_ms"]
            fb, fbb = bytes_per_row(op, N)
            row["fwd_bytes"], row["fwdbwd_bytes"] = fb * T * B, fbb * T * B
            for k, nb in (("new_fwd", "fwd_bytes"), ("new_fwdbwd", "fwdbwd_bytes")):
                row[k + "_GBps"] = row[nb] / (row[k + "_ms"] * 1e-3) / 1e9
                row[k + "_frac_of_peak"] = row[k + "_GBps"] * 1e9 / HBM_PEAK
            with torch.no_grad():
                ref = next(iter(eagers.values()))(t, b)
                row["max_abs_diff_vs_eager"] = float((new(t, b) - ref).abs().max())
            res["rows"].append(row)
            print(json.dumps(row))
        del t, b, a, G, tg, bg
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
