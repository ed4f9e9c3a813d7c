"""V-trace and UPGO returns on the GPU (``hpc_rll.rl_utils.vtrace.vtrace_nstep_return`` /
``hpc_rll.rl_utils.upgo.upgo_returns``) against the oracle (tests/vtrace_upgo_returns_oracle.py), the reference's origin
(tests/golden/returns_*.npz) and the eager PyTorch formula.

The wide (TMA) and generic kernels evaluate the formulas in the oracle's exact fp32 operation order and must be
BIT-EXACT, forward and backward.  The small-batch look-back kernels (config 21; automatic for B <= 2048, T >= 512)
re-associate the recurrence at segment boundaries: 2e-6 norm-relative there."""
import os

import numpy as np
import pytest
import torch

from tests import vtrace_upgo_returns_oracle as orc
from tests._golden import GOLDEN_DIR, names, rel_err
from tests._gpu import dev, host, need_cuda, rng

pytestmark = pytest.mark.gpu

OP = 11  # HPC_RLL_OP_LAMBDA_RETURNS: both ops are members of the λ-return family
SHAPES = [(1, 5), (2, 4), (37, 3), (128, 1000), (96, 1002), (1024, 64), (1024, 65536)]
CONFIGS = [-1, 33, 21, 99]
GAMMA, LAMBDA = 0.99, 0.95


def uses_split(T, B, cfg):
    """mirror of lookback_geometry (csrc/scan_lookback.cu) for T <= 2048: 32-row segments, at least two of them"""
    if cfg == 21:
        return T > 32
    return cfg == -1 and B <= 2048 and T >= 512


class forced:
    def __init__(self, cfg):
        self.cfg = cfg

    def __enter__(self):
        from di_hpc_b200 import _abi
        _abi.set_config(OP, self.cfg)

    def __exit__(self, *exc):
        from di_hpc_b200 import _abi
        _abi.set_config(OP, -1)
        return False


def vtrace_inputs(T, B, seed):
    g = rng(seed)
    boot = g.standard_normal((T + 1, B), dtype=np.float32)
    reward, G = (g.standard_normal((T, B), dtype=np.float32) for _ in range(2))
    ratio = np.exp(0.5 * g.standard_normal((T, B))).astype(np.float32)
    ratio[g.random((T, B)) < 0.25] = 1.0
    return np.minimum(ratio, 1.0), np.minimum(0.8 * ratio, 1.0).astype(np.float32), reward, boot, G


def upgo_inputs(T, B, seed, tie=False):
    g = rng(seed)
    if tie:
        boot = g.integers(-2, 3, (T + 1, B)).astype(np.float32)
        rewards = g.integers(-2, 3, (T, B)).astype(np.float32)
    else:
        boot = g.standard_normal((T + 1, B), dtype=np.float32)
        rewards = g.standard_normal((T, B), dtype=np.float32)
    return rewards, boot, g.standard_normal((T, B), dtype=np.float32)


def run_vtrace(rho, c, reward, boot, G):
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    r, b = dev(reward).requires_grad_(True), dev(boot).requires_grad_(True)
    ret = vtrace_nstep_return(dev(rho), dev(c), r, b, GAMMA, LAMBDA)
    ret.backward(dev(G))
    torch.cuda.synchronize()
    return host(ret), host(r.grad), host(b.grad)


def want_vtrace(rho, c, reward, boot, G):
    wb = orc.vtrace_backward(G, rho, c, GAMMA, LAMBDA)
    return orc.vtrace_forward(rho, c, reward, boot, GAMMA, LAMBDA), wb["reward"], wb["bootstrap_values"]


def run_upgo(rewards, boot, G):
    from hpc_rll.rl_utils.upgo import upgo_returns
    r, b = dev(rewards).requires_grad_(True), dev(boot).requires_grad_(True)
    ret = upgo_returns(r, b)
    ret.backward(dev(G))
    torch.cuda.synchronize()
    return host(ret), host(r.grad), host(b.grad)


def want_upgo(rewards, boot, G):
    wb = orc.upgo_backward(G, orc.upgo_mask(rewards, boot))
    return orc.upgo_forward(rewards, boot), wb["rewards"], wb["bootstrap_values"]


def same(got, ref, exact, what):
    for g, w, name in zip(got, ref, ("returns", "grad_rewards", "grad_bootstrap_values")):
        if exact:
            assert np.array_equal(g, w), "%s %s not bit-exact (max diff %g)" % (what, name, np.max(np.abs(g - w)))
        else:
            assert rel_err(g, w) <= 2e-6, (what, name, rel_err(g, w))


@pytest.mark.parametrize("T,B", SHAPES)
def test_vtrace_vs_oracle(T, B):
    need_cuda()
    x = vtrace_inputs(T, B, T * 7919 + B)
    ref = want_vtrace(*x)
    for cfg in CONFIGS:
        with forced(cfg):
            got = run_vtrace(*x)
        same(got, ref, not uses_split(T, B, cfg), ("vtrace", T, B, cfg))


@pytest.mark.parametrize("T,B", SHAPES)
def test_upgo_vs_oracle(T, B):
    need_cuda()
    for tie in (False, True):
        x = upgo_inputs(T, B, T * 7919 + B + tie, tie)
        ref = want_upgo(*x)
        for cfg in CONFIGS:
            with forced(cfg):
                got = run_upgo(*x)
            same(got, ref, not uses_split(T, B, cfg), ("upgo", T, B, cfg, tie))
            assert not np.signbit(got[2][0]).any() and not got[2][0].any()


@pytest.mark.parametrize("cfg", [-1, 33, 99])
def test_origin_fixtures(cfg):
    need_cuda()
    for name in names("returns_vtrace"):
        z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        with forced(cfg):
            ret, gr, gb = run_vtrace(z["in_clipped_rhos"], z["in_clipped_cs"], z["in_reward"],
                                     z["in_bootstrap_values"], z["in_grad"])
        assert np.array_equal(ret, z["out"]) and np.array_equal(gr, z["grad_reward"]), name
        want = z["grad_bootstrap_values"]
        assert np.allclose(gb, want, rtol=1e-6, atol=1e-6 * max(1.0, np.abs(want).max())), name
    for name in names("returns_upgo"):
        z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
        with forced(cfg):
            got = run_upgo(z["in_rewards"], z["in_bootstrap_values"], z["in_grad"])
        same(got, (z["out"], z["grad_rewards"], z["grad_bootstrap_values"]), True, name)


def shifted(a):
    """a contiguous view one element into a buffer: not 16-byte aligned"""
    t = dev(a)
    buf = torch.empty(a.size + 1, dtype=t.dtype, device="cuda")
    view = buf[1:].view(a.shape)
    view.copy_(t)
    return view


def test_ragged_batches_and_offset_views():
    """B % 4 != 0 (no fp32 tensor map), B % 16 != 0 (no byte map for the UPGO backward) and views one element into a
    buffer (not 16-byte aligned) fall back to the generic kernels: bit-exact under every forced config"""
    need_cuda()
    from hpc_rll.rl_utils.upgo import upgo_returns
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    T = 96
    for B in (4098, 4100):
        x, y = vtrace_inputs(T, B, B), upgo_inputs(T, B, B, tie=True)
        for cfg in (-1, 33):
            with forced(cfg):
                same(run_vtrace(*x), want_vtrace(*x), True, ("vtrace", B, cfg))
                same(run_upgo(*y), want_upgo(*y), True, ("upgo", B, cfg))
    B = 4096
    x, y = vtrace_inputs(T, B, 1), upgo_inputs(T, B, 2, tie=True)
    for cfg in (-1, 33):
        with forced(cfg):
            r, b = shifted(x[2]).requires_grad_(True), shifted(x[3]).requires_grad_(True)
            ret = vtrace_nstep_return(shifted(x[0]), shifted(x[1]), r, b, GAMMA, LAMBDA)
            ret.backward(shifted(x[4]))
            same((host(ret), host(r.grad), host(b.grad)), want_vtrace(*x), True, ("vtrace offset view", cfg))
            r, b = shifted(y[0]).requires_grad_(True), shifted(y[1]).requires_grad_(True)
            ret = upgo_returns(r, b)
            ret.backward(shifted(y[2]))
            same((host(ret), host(r.grad), host(b.grad)), want_upgo(*y), True, ("upgo offset view", cfg))


def test_requires_grad_subsets():
    need_cuda()
    from hpc_rll.rl_utils.upgo import upgo_returns
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    rho, c, reward, boot, G = vtrace_inputs(250, 4096, 3)
    ref = want_vtrace(rho, c, reward, boot, G)
    r = dev(reward).requires_grad_(True)
    ret = vtrace_nstep_return(dev(rho), dev(c), r, dev(boot), GAMMA, LAMBDA)
    ret.backward(dev(G))
    assert np.array_equal(host(r.grad), ref[1])
    ret = vtrace_nstep_return(dev(rho), dev(c), dev(reward), dev(boot), GAMMA, LAMBDA)
    assert not ret.requires_grad and np.array_equal(host(ret), ref[0])
    for which in ("clipped_rhos", "clipped_cs"):
        args = {"clipped_rhos": dev(rho), "clipped_cs": dev(c)}
        args[which].requires_grad_(True)
        with pytest.raises(ValueError, match=which):
            vtrace_nstep_return(args["clipped_rhos"], args["clipped_cs"], dev(reward), dev(boot))
    with pytest.raises(ValueError, match="clipped_cs"):  # wrong shape
        vtrace_nstep_return(dev(rho), dev(c[:-1]), dev(reward), dev(boot))
    with pytest.raises(ValueError, match="bootstrap_values"):
        vtrace_nstep_return(dev(rho), dev(c), dev(reward), dev(boot[:-1]))
    with pytest.raises(TypeError, match="reward"):  # wrong dtype
        vtrace_nstep_return(dev(rho), dev(c), dev(reward).double(), dev(boot))
    rewards, boot, G = upgo_inputs(250, 4096, 4)
    ref = want_upgo(rewards, boot, G)
    b = dev(boot).requires_grad_(True)
    ret = upgo_returns(dev(rewards), b)
    ret.backward(dev(G))
    assert np.array_equal(host(b.grad), ref[2])
    with torch.no_grad():
        ret = upgo_returns(dev(rewards), dev(boot).requires_grad_(True))
    assert not ret.requires_grad and np.array_equal(host(ret), ref[0])
    with pytest.raises(ValueError, match="bootstrap_values"):
        upgo_returns(dev(rewards), dev(boot[1:]))


@pytest.mark.parametrize("T,B", [(1024, 64), (64, 65536), (128, 1000)])
def test_run_to_run_identical(T, B):
    need_cuda()
    x = vtrace_inputs(T, B, 17)
    y = upgo_inputs(T, B, 18)
    for fn, args in ((run_vtrace, x), (run_upgo, y)):
        a, b = fn(*args), fn(*args)
        for p, q in zip(a, b):
            assert np.array_equal(p.view(np.uint32), q.view(np.uint32))


@pytest.mark.parametrize("T,B", [(1024, 64), (64, 65536), (128, 1000)])
def test_cuda_graph_replay(T, B):
    need_cuda()
    from hpc_rll.rl_utils.upgo import upgo_returns
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    x0, y0 = vtrace_inputs(T, B, 23), upgo_inputs(T, B, 24, tie=True)
    rho, c, r, b, g = (dev(a) for a in x0)
    ur, ub, ug = (dev(a) for a in y0)
    r.requires_grad_(True)
    b.requires_grad_(True)
    ur.requires_grad_(True)
    ub.requires_grad_(True)

    def step():
        ret = vtrace_nstep_return(rho, c, r, b, GAMMA, LAMBDA)
        ret.backward(g)
        uret = upgo_returns(ur, ub)
        uret.backward(ug)
        return ret, uret

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    for t in (r, b, ur, ub):
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ret, uret = step()
    x1, y1 = vtrace_inputs(T, B, 29), upgo_inputs(T, B, 30, tie=True)
    with torch.no_grad():
        for t, a in zip((rho, c, r, b, g, ur, ub, ug), x1 + y1):
            t.copy_(dev(a))
    graph.replay()
    torch.cuda.synchronize()
    for p, q in zip((host(ret), host(r.grad), host(b.grad)), run_vtrace(*x1)):
        assert np.array_equal(p, q)
    for p, q in zip((host(uret), host(ur.grad), host(ub.grad)), run_upgo(*y1)):
        assert np.array_equal(p, q)


def eager_vtrace(rho, c, reward, boot, gamma=GAMMA, lambda_=LAMBDA):
    """the V-trace target as a user would write it in PyTorch: a Python loop over T"""
    deltas = rho * (reward + gamma * boot[1:] - boot[:-1])
    factor = gamma * lambda_
    item = 0.
    out = [None] * reward.shape[0]
    for t in reversed(range(reward.shape[0])):
        item = deltas[t] + factor * c[t] * item
        out[t] = boot[t] + item
    return torch.stack(out)


def eager_upgo(rewards, boot):
    """the UPGO return in PyTorch: ℓ from the comparisons, then the γ = 1 λ-return loop"""
    lam = (rewards + boot[1:]) >= boot[:-1]
    lam = torch.cat([lam[1:], torch.ones_like(lam[-1:])], dim=0).float()
    T = rewards.shape[0]
    out = [None] * T
    out[T - 1] = rewards[T - 1] + boot[T]
    for t in range(T - 2, -1, -1):
        out[t] = rewards[t] + lam[t] * out[t + 1] + (1 - lam[t]) * boot[t + 1]
    return torch.stack(out)


@pytest.mark.parametrize("cfg", [33, 99])
def test_non_finite_values(cfg):
    """inf V behind ℓ = 0 and NaN ties (UPGO), inf / NaN values and ratios (V-trace): as the eager formula"""
    need_cuda()
    T, B = 16, 64
    rewards, boot, G = upgo_inputs(T, B, 31, tie=True)
    boot[5, :8] = np.inf  # V_5 = inf with r_5 + V_6 < V_5: ℓ_4 = 0, R_4 bootstraps from inf
    boot[6, :8] = 0.0
    rewards[5, :8] = 0.0
    boot[9, 8:16] = np.nan  # NaN comparisons: ℓ = 0 around row 9
    rewards[12, 16:24] = np.nan
    boot[T, 24:32] = -np.inf
    with forced(cfg):
        got = run_upgo(rewards, boot, G)
    ref = want_upgo(rewards, boot, G)
    for g, w in zip(got, ref):
        assert np.array_equal(g, w, equal_nan=True)
    e = eager_upgo(torch.from_numpy(rewards), torch.from_numpy(boot))
    assert np.array_equal(got[0], e.numpy(), equal_nan=True)
    assert (orc.upgo_mask(rewards, boot)[4, :8] == 0).all() and np.isinf(got[0][4, :8]).all()

    rho, c, reward, boot, G = vtrace_inputs(T, B, 32)
    boot[3, :8] = np.inf
    boot[T, 8:16] = -np.inf
    boot[7, 16:24] = np.nan
    c[10, 24:32] = np.inf
    rho[12, 32:40] = np.nan
    with forced(cfg):
        got = run_vtrace(rho, c, reward, boot, G)
    ref = want_vtrace(rho, c, reward, boot, G)
    for g, w in zip(got, ref):
        assert np.array_equal(g, w, equal_nan=True)
    e = eager_vtrace(*(torch.from_numpy(a) for a in (rho, c, reward, boot)))
    assert np.array_equal(got[0], e.numpy(), equal_nan=True)


def test_empty():
    need_cuda()
    from hpc_rll.rl_utils.upgo import upgo_returns
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    for T, B in ((0, 5), (5, 0), (0, 0)):
        b = torch.randn(T + 1, B, device="cuda", requires_grad=True)
        r = torch.zeros(T, B, device="cuda", requires_grad=True)
        ones = torch.ones(T, B, device="cuda")
        for ret in (vtrace_nstep_return(ones, ones, r, b), upgo_returns(r, b)):
            assert ret.shape == (T, B)
            b.grad = r.grad = None
            ret.sum().backward()
            assert b.grad.shape == (T + 1, B) and r.grad.shape == (T, B)
            assert not b.grad.any() and not r.grad.any()


def test_more_than_2_31_elements():
    """One forward of each op over T*B > 2^31 elements (about 43 GB of device memory for V-trace), checked column-wise
    against the oracle."""
    need_cuda()
    from hpc_rll.rl_utils.upgo import upgo_returns
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    T, B = 32800, 65536
    n = T * B
    if torch.cuda.mem_get_info()[0] < n * 5 * 4 + (1 << 30):
        pytest.skip("needs %.1f GB of free device memory" % ((n * 5 * 4 + (1 << 30)) / 1e9))
    cols = [0, 1, 777, 40001, B - 1]
    gen = torch.Generator(device="cuda").manual_seed(0)
    boot = torch.randn(T + 1, B, device="cuda", generator=gen)
    reward = torch.randn(T, B, device="cuda", generator=gen)
    rho = torch.rand(T, B, device="cuda", generator=gen)
    c = torch.rand(T, B, device="cuda", generator=gen)
    ret = vtrace_nstep_return(rho, c, reward, boot)
    torch.cuda.synchronize()
    w = orc.vtrace_forward(host(rho[:, cols]), host(c[:, cols]), host(reward[:, cols]), host(boot[:, cols]))
    assert np.array_equal(host(ret[:, cols]), w)
    del rho, c, ret
    ret = upgo_returns(reward, boot)
    torch.cuda.synchronize()
    assert np.array_equal(host(ret[:, cols]), orc.upgo_forward(host(reward[:, cols]), host(boot[:, cols])))
    del boot, reward, ret
    torch.cuda.empty_cache()
