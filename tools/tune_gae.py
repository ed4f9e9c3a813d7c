"""Time the GAE kernel regimes on the GPU (gae.cu:pick_cfg): per-regime fwd / bwd time (CUDA events) and GB/s."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from di_hpc_b200 import _abi  # noqa: E402


def time_fn(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in evs:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in evs)
    return ts[len(ts) // 2], ts[0]


def main():
    T = int(os.environ.get("T", 1024))
    B = int(os.environ.get("B", 65536))
    cfgs = [int(c) for c in os.environ.get("CFGS", "5,7,13,21,33,99").split(",")]
    L = _abi.lib()
    v = torch.randn(T + 1, B, device="cuda")
    r = torch.randn(T, B, device="cuda")
    G = torch.randn(T, B, device="cuda")
    adv = torch.empty(T, B, device="cuda")
    gv = torch.empty(T + 1, B, device="cuda")
    gr = torch.empty(T, B, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    fwd_bytes = 12 * T * B + 4 * B
    bwd_bytes = 12 * T * B + 4 * B
    out = []
    for c in cfgs:
        _abi.set_config(0, c)
        f = lambda: _abi.check(L.hpc_rll_gae_forward(v.data_ptr(), r.data_ptr(), adv.data_ptr(), T, B, 0.99, 0.97, st), "f")
        b = lambda: _abi.check(L.hpc_rll_gae_backward(G.data_ptr(), gv.data_ptr(), gr.data_ptr(), T, B, 0.99, 0.97, st), "b")
        fm, fb = time_fn(f)
        bm, bb = time_fn(b)
        rec = dict(cfg=c, T=T, B=B, fwd_ms=fm, fwd_best_ms=fb, fwd_gbs=fwd_bytes / fm / 1e6, bwd_ms=bm, bwd_best_ms=bb,
                   bwd_gbs=bwd_bytes / bm / 1e6)
        print(json.dumps(rec), flush=True)
        out.append(rec)
    _abi.set_config(0, -1)
    # plain copy for reference (same bytes as one direction)
    x = torch.empty(3 * T * B // 2, device="cuda")
    y = torch.empty_like(x)
    cm, cb = time_fn(lambda: y.copy_(x))
    print(json.dumps(dict(copy_ms=cm, copy_gbs=2 * x.numel() * 4 / cm / 1e6)))


if __name__ == "__main__":
    main()
