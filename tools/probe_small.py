"""Small-batch regime (the reference's own test shapes, T=1024 B=64 ...): device time of GAE forward+backward per kernel
configuration -- column scan (5, 13) vs the single-launch T-split with look-back (21, the automatic choice for B <= 4096)
-- measured three ways: raw C-ABI calls between events, CUDA-graph replay of fwd+bwd (what a captured training step
sees), and the module API (GAE.forward + autograd) per call.

    python tools/probe_small.py [--shapes 1024x64,1024x512,...]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from di_hpc_b200 import _abi  # noqa: E402
from hpc_rll.rl_utils.gae import GAE  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1024x64,1024x256,1024x1024,1024x4096,128x128,256x2048")
    a = ap.parse_args()
    L = _abi.lib()
    for shp in a.shapes.split(","):
        T, B = (int(x) for x in shp.split("x"))
        v = torch.randn(T + 1, B, device="cuda", requires_grad=True)
        r = torch.randn(T, B, device="cuda", requires_grad=True)
        g = torch.randn(T, B, device="cuda")
        adv, gv, gr = torch.empty(T, B, device="cuda"), torch.empty(T + 1, B, device="cuda"), torch.empty(T, B, device="cuda")
        m = GAE(T, B)
        side = torch.cuda.Stream()
        for cfg in (5, 13, 21, -1):
            _abi.set_config(0, cfg)

            def raw(st):
                _abi.check(L.hpc_rll_gae_forward(v.data_ptr(), r.data_ptr(), adv.data_ptr(), T, B, 0.99, 0.97, st), "f")
                _abi.check(L.hpc_rll_gae_backward(g.data_ptr(), gv.data_ptr(), gr.data_ptr(), T, B, 0.99, 0.97, st), "b")

            with torch.cuda.stream(side):
                for _ in range(3):
                    raw(side.cuda_stream)
            side.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=side):
                raw(torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(5):
                graph.replay()
            torch.cuda.synchronize()
            n = 200
            e0.record()
            for _ in range(n):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            graph_us = e0.elapsed_time(e1) / n * 1e3
            st = torch.cuda.current_stream().cuda_stream
            for _ in range(3):
                raw(st)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(n):
                raw(st)
            e1.record()
            torch.cuda.synchronize()
            raw_us = e0.elapsed_time(e1) / n * 1e3
            for _ in range(3):
                torch.autograd.grad(m(v, r), [v, r], grad_outputs=g)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(n):
                torch.autograd.grad(m(v, r), [v, r], grad_outputs=g)
            e1.record()
            torch.cuda.synchronize()
            mod_us = e0.elapsed_time(e1) / n * 1e3
            print(json.dumps({"T": T, "B": B, "cfg": cfg, "graph_replay_us": round(graph_us, 2),
                              "raw_abi_queued_us": round(raw_us, 2), "module_queued_us": round(mod_us, 2)}), flush=True)
        _abi.set_config(0, -1)


if __name__ == "__main__":
    main()
