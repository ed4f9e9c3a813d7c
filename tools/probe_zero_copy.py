"""Can the scan kernels read and write PINNED HOST memory directly (TMA over PCIe, no staging copies)?
Runs hpc_rll_gae_forward / _backward with host pointers (UVA), checks the bits against the device-resident
result, and times forward alone, backward alone, and both concurrently on two streams.  Also times plain chunked
copy-engine traffic (duplex) per chunk size, to separate per-copy overhead from pipeline structure."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from di_hpc_b200 import _abi  # noqa: E402
from di_hpc_b200 import host as hp  # noqa: E402


def main():
    T, B = 1024, 65536
    L = _abi.lib()
    hp.bind_to_device()
    hv, hr, hg = hp.pinned_empty((T + 1, B)), hp.pinned_empty((T, B)), hp.pinned_empty((T, B))
    ha, hgv, hgr = hp.pinned_empty((T, B)), hp.pinned_empty((T + 1, B)), hp.pinned_empty((T, B))
    for t in (hv, hr, hg):
        t.normal_()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def fwd(st):
        _abi.check(L.hpc_rll_gae_forward(hv.data_ptr(), hr.data_ptr(), ha.data_ptr(), T, B, 0.99, 0.97, st), "fwd")

    def bwd(st):
        _abi.check(L.hpc_rll_gae_backward(hg.data_ptr(), hgv.data_ptr(), hgr.data_ptr(), T, B, 0.99, 0.97, st), "bwd")

    def timeit(fn, n=5):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(n):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return sorted(ts)[len(ts) // 2] * 1e3

    res = {}
    try:
        res["zero_copy_fwd_ms"] = timeit(lambda: fwd(s1.cuda_stream))
        res["zero_copy_bwd_ms"] = timeit(lambda: bwd(s2.cuda_stream))

        def both():
            fwd(s1.cuda_stream)
            bwd(s2.cuda_stream)

        res["zero_copy_both_ms"] = timeit(both)
        # correctness vs the device-resident path
        dv, dr, dg = hv.cuda(), hr.cuda(), hg.cuda()
        da, dgv, dgr = torch.empty_like(dr), torch.empty_like(dv), torch.empty_like(dr)
        st = torch.cuda.current_stream().cuda_stream
        _abi.check(L.hpc_rll_gae_forward(dv.data_ptr(), dr.data_ptr(), da.data_ptr(), T, B, 0.99, 0.97, st), "f")
        _abi.check(L.hpc_rll_gae_backward(dg.data_ptr(), dgv.data_ptr(), dgr.data_ptr(), T, B, 0.99, 0.97, st), "b")
        torch.cuda.synchronize()
        res["zero_copy_bit_exact"] = bool(torch.equal(da.cpu(), ha) and torch.equal(dgv.cpu(), hgv)
                                          and torch.equal(dgr.cpu(), hgr))
        for cfg in (5, 7, 13, 33):
            _abi.set_config(0, cfg)
            res["zero_copy_both_ms_cfg%d" % cfg] = timeit(both, 3)
        _abi.set_config(0, -1)
    except Exception as e:  # noqa: BLE001
        res["zero_copy_error"] = repr(e)
    print(json.dumps(res), flush=True)

    # chunked duplex copies, no kernels
    d_in, d_out = torch.empty(T, B, device="cuda"), torch.empty(T, B, device="cuda")
    for rows in (8, 16, 32, 64, 128, 1024):
        def run():
            for t0 in range(0, T, rows):
                with torch.cuda.stream(s1):
                    d_in[t0:t0 + rows].copy_(hv[t0:t0 + rows], non_blocking=True)
                with torch.cuda.stream(s2):
                    ha[t0:t0 + rows].copy_(d_out[t0:t0 + rows], non_blocking=True)
        ms = timeit(run, 3)
        print(json.dumps({"chunked_duplex_rows": rows, "ms": ms, "gbs_each": T * B * 4 / ms / 1e6}), flush=True)


if __name__ == "__main__":
    main()
