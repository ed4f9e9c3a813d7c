"""One small forward+backward of every op (and the padding path) -- the workload for
`compute-sanitizer --tool memcheck|racecheck|synccheck python tools/sanitize_smoke.py`."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hpc_rll.rl_utils.gae import GAE, gae_with_adv_stats  # noqa: E402
from hpc_rll.rl_utils.padding import Padding2D, UnPadding2D  # noqa: E402
from hpc_rll.rl_utils.ppo import PPO  # noqa: E402
from hpc_rll.rl_utils.td import (DistNStepTD, IQNNStepTDError, QNStepTD, QNStepTDRescale, QRDQNNStepTDError,  # noqa: E402
                                 TDLambda)
from hpc_rll.rl_utils.upgo import UPGO  # noqa: E402
from hpc_rll.rl_utils.vtrace import VTrace  # noqa: E402
from di_hpc_b200 import _abi  # noqa: E402

D = "cuda"
ONE = torch.ones(1, device=D)


def r(*s):
    return torch.randn(*s, device=D)


def wide_and_fused():
    """kernels added late in round 1: TMA-staged output (ScanPipe with NOUT > 0, config 33 = the default for wide batches),
    GAE with moments + PPO with fused normalisation, 64-bit / staged row paths (N = 18 / 9)"""
    T, B = 7, 40000
    v, rew = r(T + 1, B).requires_grad_(True), r(T, B).requires_grad_(True)
    for cfg in (-1, 7, 33):
        _abi.set_config(0, cfg)
        torch.autograd.grad(GAE(T, B)(v, rew), [v, rew], grad_outputs=r(T, B))
    _abi.set_config(0, -1)
    adv, st = gae_with_adv_stats(v, rew)
    R, N = T * B, 6
    ln, vn = r(R, N).requires_grad_(True), r(R).requires_grad_(True)
    l, _ = PPO(R, N)(ln, r(R, N), torch.randint(0, N, (R, ), device=D), vn, r(R), adv.reshape(-1), r(R), None, 0.2, True,
                     None, adv_stats=st)
    torch.autograd.grad(l.policy_loss + l.value_loss + l.entropy_loss, [ln, vn], grad_outputs=ONE)
    for T, B, N in ((5, 300, 18), (5, 300, 9)):
        t = r(T, B, N).requires_grad_(True)
        a = torch.randint(0, N, (T, B), device=D)
        v = r(T + 1, B).requires_grad_(True)
        l = VTrace(T, B, N)(t, r(T, B, N), a, v, r(T, B), torch.rand(T, B, device=D))
        torch.autograd.grad(l.policy_loss + l.value_loss + l.entropy_loss, [t, v], grad_outputs=ONE)
        torch.autograd.grad(UPGO(T, B, N)(t, torch.rand(T, B, device=D), a, r(T, B), v.detach()), [t], grad_outputs=ONE)


def chunked_and_host():
    """round 2: T-chunked scan with a carried state (incl. the TMA-store kernels on a chunk) and the host-buffer
    pipeline (three streams, per-slot events, pooled staging memory)"""
    from di_hpc_b200 import host as hp
    L = _abi.lib()
    st = torch.cuda.current_stream().cuda_stream
    for T, B, rows in ((23, 40000, 8), (23, 516, 4), (10, 133, 4)):
        v, rew, ga = r(T + 1, B), r(T, B), r(T, B)
        adv, gv, gr = torch.empty(T, B, device=D), torch.empty(T + 1, B, device=D), torch.empty(T, B, device=D)
        cf, cb = torch.zeros(2, B, device=D), torch.zeros(2, B, device=D)
        cf[1] = v[T]
        nC = (T + rows - 1) // rows
        for k in reversed(range(nC)):
            t0, n = k * rows, min(rows, T - k * rows)
            _abi.check(L.hpc_rll_gae_forward_chunk(v[t0].data_ptr(), rew[t0].data_ptr(), adv[t0].data_ptr(),
                                                   cf.data_ptr(), T, t0, n, B, 0.99, 0.97, st), "fwd_chunk")
        for k in range(nC):
            t0, n = k * rows, min(rows, T - k * rows)
            _abi.check(L.hpc_rll_gae_backward_chunk(ga[t0].data_ptr(), gv[t0].data_ptr(), gr[t0].data_ptr(),
                                                    cb.data_ptr(), T, t0, n, B, 0.99, 0.97, st), "bwd_chunk")
    T, B = 40, 40000
    hv, hr, hg = torch.randn(T + 1, B).pin_memory(), torch.randn(T, B).pin_memory(), torch.randn(T, B).pin_memory()
    hp.gae_fwd_bwd_host(hv, hr, hg)
    hp.gae_fwd_bwd_host(hv, hr, None)


def small_batch_tsplit():
    """round 2: the automatic small-batch path (T >= 512, B <= 2048) of all four scans, incl. a ragged last segment and
    a column count that is not a multiple of the 32-column tile"""
    for T, B, N in ((600, 70, 5), (1024, 64, 3)):
        v, rew = r(T + 1, B).requires_grad_(True), r(T, B).requires_grad_(True)
        torch.autograd.grad(GAE(T, B)(v, rew), [v, rew], grad_outputs=r(T, B))
        torch.autograd.grad(TDLambda(T, B)(v, rew.detach(), torch.rand(T, B, device=D)), [v], grad_outputs=ONE)
        t = r(T, B, N).requires_grad_(True)
        a = torch.randint(0, N, (T, B), device=D)
        l = VTrace(T, B, N)(t, r(T, B, N), a, v, rew.detach())
        torch.autograd.grad(l.policy_loss + l.value_loss + l.entropy_loss, [t, v], grad_outputs=ONE)
        torch.autograd.grad(UPGO(T, B, N)(t, torch.rand(T, B, device=D), a, rew.detach(), v.detach()), [t], grad_outputs=ONE)


def main():
    wide_and_fused()
    chunked_and_host()
    small_batch_tsplit()
    for T, B, N in ((37, 132, 6), (16, 260, 16), (9, 64, 40)):
        v, rew = r(T + 1, B).requires_grad_(True), r(T, B).requires_grad_(True)
        for cfg in (-1, 5, 13, 21, 99):
            _abi.set_config(0, cfg)
            torch.autograd.grad(GAE(T, B)(v, rew), [v, rew], grad_outputs=r(T, B))
        _abi.set_config(0, -1)
        w = torch.rand(T, B, device=D)
        for cfg in (-1, 21, 99):  # 21 = single-launch T-split with look-back
            _abi.set_config(1, cfg)
            torch.autograd.grad(TDLambda(T, B)(v, rew.detach(), w), [v], grad_outputs=ONE)
        _abi.set_config(1, -1)
        t = r(T, B, N).requires_grad_(True)
        a = torch.randint(0, N, (T, B), device=D)
        for cfg in (-1, 21, 99):
            _abi.set_config(2, cfg)
            _abi.set_config(3, cfg)
            l = VTrace(T, B, N)(t, r(T, B, N), a, v, rew.detach(), w)
            torch.autograd.grad(l.policy_loss + l.value_loss + l.entropy_loss, [t, v], grad_outputs=ONE)
            torch.autograd.grad(UPGO(T, B, N)(t, torch.rand(T, B, device=D), a, rew.detach(), v.detach()), [t],
                                grad_outputs=ONE)
        _abi.set_config(2, -1)
        _abi.set_config(3, -1)
        ln = r(B, N).requires_grad_(True)
        vn = r(B).requires_grad_(True)
        l, _ = PPO(B, N)(ln, r(B, N), a[0], vn, r(B), r(B), r(B), torch.rand(B, device=D), 0.2, True, 3.0)
        torch.autograd.grad(l.policy_loss + l.value_loss + l.entropy_loss, [ln, vn], grad_outputs=ONE)
        q = r(B, N).requires_grad_(True)
        act, nact = a[0], torch.randint(0, N, (B, ), device=D)
        done = (torch.rand(B, device=D) < 0.3).float()
        for dcfg in (1, 2):  # lane-per-sample (TMA-gathered rows) and warp-per-sample C51 kernels
            _abi.set_config(6, dcfg)
            dd = torch.softmax(r(B, N, 21), -1).requires_grad_(True)
            torch.autograd.grad(DistNStepTD(T, B, N, 21)(dd, torch.softmax(r(B, N, 21), -1), act, nact, rew.detach(), done, None, 0.9, -3., 3.)[0], [dd], grad_outputs=ONE)
        _abi.set_config(6, -1)
        for cls in (QNStepTD, QNStepTDRescale):
            torch.autograd.grad(cls(T, B, N)(q, r(B, N), act, nact, rew.detach(), done, None, 0.95)[0], [q],
                                grad_outputs=ONE)
        d0 = torch.softmax(r(B, N, 51), -1).requires_grad_(True)
        torch.autograd.grad(
            DistNStepTD(T, B, N, 51)(d0, torch.softmax(r(B, N, 51), -1), act, nact, rew.detach(), done, None, 0.95, -10.,
                                     10.)[0], [d0], grad_outputs=ONE)
        for tau in (8, 39, 64):
            qq = r(B, N, tau).requires_grad_(True)
            torch.autograd.grad(QRDQNNStepTDError(tau, T, B, N)(qq, r(B, N, tau), act, nact, rew.detach(), done, 0.95)[0],
                                [qq], grad_outputs=ONE)
            qi = r(tau, B, N).requires_grad_(True)
            torch.autograd.grad(
                IQNNStepTDError(tau, tau + 1, T, B, N)(qi, r(tau + 1, B, N), act, nact, rew.detach(), done,
                                                       torch.rand(tau, B, device=D), 0.95, 0.9)[0], [qi], grad_outputs=ONE)
    # round 2: the backward scatter from shared-memory images (taken from 1 MB of output on), one case per mapping
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    from tests.test_scatter_gpu import run as scatter_case
    for case in (("q", 40003, 8, 1, 1), ("q", 9001, 40, 1, 1), ("iqn", 5003, 8, 1, 13), ("dist", 9001, 4, 7, 1),
                 ("dist", 3001, 8, 51, 1), ("qrdqn", 2003, 8, 64, 1), ("qrdqn", 1203, 5, 130, 1)):
        scatter_case(*case)
    data = [r(int(torch.randint(3, 20, (1, ))), int(torch.randint(2, 17, (1, )))) for _ in range(40)]
    x, m, s = Padding2D(data)
    UnPadding2D(x, s)
    gx, gm, gs = Padding2D(data, group=4, group_mode='oracle')
    UnPadding2D(gx, gs)
    torch.cuda.synchronize()
    print("sanitize_smoke done, kernel launches:", _abi.launch_count())


if __name__ == "__main__":
    main()
