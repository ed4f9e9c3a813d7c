"""λ-returns on the GPU (``hpc_rll.rl_utils.td.generalized_lambda_returns`` / ``multistep_forward_view``) against the
oracle (tests/lambda_returns_oracle.py), the reference's origin (tests/golden/lambda_*.npz) and TD(lambda).

The wide (TMA) and generic kernels evaluate the formula in the oracle's exact fp32 operation order and must be
BIT-EXACT, forward and backward.  The small-batch look-back kernels (config 21; automatic for B <= 2048, T >= 512)
re-associate the recurrence at segment boundaries: 2e-6 norm-relative there."""
import os

import numpy as np
import pytest
import torch

from tests import lambda_returns_oracle as orc
from tests._golden import GOLDEN_DIR, names, rel_err
from tests._gpu import dev, host, need_cuda, rng

pytestmark = pytest.mark.gpu

OP = 11  # HPC_RLL_OP_LAMBDA_RETURNS
SHAPES = [(1, 8), (2, 16), (37, 3), (64, 1000), (128, 4096), (600, 16), (1024, 64), (1024, 2048)]
CONFIGS = [-1, 33, 21, 99]
COMBOS = [(gt, lt, dn) for gt in (False, True) for lt in (False, True) for dn in (False, True)]
FNS = {"generalized_lambda_returns": 1, "multistep_forward_view": 0}
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


def inputs(T, B, gt, lt, dn, offset, seed, density=0.1):
    g = rng(seed)
    boot = g.standard_normal((T + offset, B), dtype=np.float32)
    rewards, G = (g.standard_normal((T, B), dtype=np.float32) for _ in range(2))
    gammas = (0.5 + 0.5 * g.random((T, B))).astype(np.float32) if gt else GAMMA
    lam = g.random((T, B)).astype(np.float32) if lt else LAMBDA
    done = (g.random((T, B)) < density) if dn else None
    return boot, rewards, G, gammas, lam, done


def fn_of(offset):
    import hpc_rll.rl_utils.td as td
    return td.generalized_lambda_returns if offset == 1 else td.multistep_forward_view


def run(boot, rewards, G, gammas, lam, done, offset, mask_dtype=torch.bool):
    b, r = dev(boot).requires_grad_(True), dev(rewards).requires_grad_(True)
    as_t = (lambda x: dev(x) if isinstance(x, np.ndarray) else x)
    d = None if done is None else dev(done).to(mask_dtype)
    ret = fn_of(offset)(b, r, as_t(gammas), as_t(lam), d)
    ret.backward(dev(G))
    torch.cuda.synchronize()
    return host(ret), host(b.grad), host(r.grad)


def want(boot, rewards, G, gammas, lam, done, offset):
    wb = orc.backward(G, gammas, lam, done, offset)
    return orc.forward(boot, rewards, gammas, lam, done, offset), wb["bootstrap_values"], wb["rewards"]


def same(got, ref, exact, what):
    for g, w, name in zip(got, ref, ("returns", "grad_bootstrap_values", "grad_rewards")):
        if exact:
            assert np.array_equal(g, w), "%s %s not bit-exact (max diff %g)" % (what, name, np.max(np.abs(g - w)))
        else:
            assert rel_err(g, w) <= 2e-6, (what, name, rel_err(g, w))


@pytest.mark.parametrize("fn", list(FNS))
@pytest.mark.parametrize("T,B", SHAPES)
def test_vs_oracle(T, B, fn):
    need_cuda()
    offset = FNS[fn]
    for i, (gt, lt, dn) in enumerate(COMBOS):
        x = inputs(T, B, gt, lt, dn, offset, T * 7919 + B * 13 + i)
        ref = want(*x, offset)
        for cfg in CONFIGS:
            with forced(cfg):
                got = run(*x, offset)
            same(got, ref, not uses_split(T, B, cfg), (T, B, fn, cfg, gt, lt, dn))
            assert not np.signbit(got[1][:offset]).any() and not got[1][:offset].any()


@pytest.mark.parametrize("name", names("lambda"))
@pytest.mark.parametrize("cfg", [-1, 99])
def test_origin_fixtures(name, cfg):
    need_cuda()
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    gam, lam = z["in_gammas"], z["in_lambda_"]
    gam = float(gam) if gam.ndim == 0 else gam
    lam = float(lam) if lam.ndim == 0 else lam
    with forced(cfg):
        got = run(z["in_bootstrap_values"], z["in_rewards"], z["in_grad"], gam, lam, None, int(z["offset"]))
    same(got, (z["out"], z["grad_bootstrap_values"], z["grad_rewards"]), True, name)


@pytest.mark.parametrize("name", names("tdlambda"))
def test_td_lambda_fixtures_and_loss(name):
    """the returns inside TD(lambda): bit-exact against the fixtures' returns, and the loss built from them agrees with
    the TDLambda module"""
    need_cuda()
    from hpc_rll.rl_utils.td import TDLambda, generalized_lambda_returns
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    g, lam = float(z["attr_gamma"]), float(z["attr_lambda_"])
    v, r = dev(z["in_value"]), dev(z["in_reward"])
    w = dev(z["in_weight"]) if "in_weight" in z.files else torch.ones_like(r)
    R = generalized_lambda_returns(v, r, g, lam)
    assert np.array_equal(host(R), z["out32_ret"])
    loss = 0.5 * ((R - v[:-1]) ** 2 * w).mean()
    T, B = r.shape
    ref = TDLambda(T, B)(v, r, w, g, lam)
    assert abs(float(loss) - float(ref)) <= 1e-6 * max(1.0, abs(float(ref)))


@pytest.mark.parametrize("T,B", [(64, 4096), (1024, 64), (100, 260)])
def test_mask_dtypes(T, B):
    need_cuda()
    x = inputs(T, B, True, False, True, 1, 5, density=0.3)
    ref = run(*x, 1, mask_dtype=torch.bool)
    for dt in (torch.uint8, torch.float32):
        got = run(*x, 1, mask_dtype=dt)
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), dt


def kernels_run(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def test_ragged_and_offset_views_take_the_generic_path():
    need_cuda()
    T, B = 96, 4104  # B % 16 == 8: no uint8 tensor map
    x = inputs(T, B, True, True, True, 1, 11, density=0.3)
    ref = want(*x, 1)
    names_ = kernels_run(lambda: same(run(*x, 1), ref, True, "ragged"))
    assert "lambda_ret_fwd_generic" in names_ and "lambda_ret_bwd_generic" in names_, names_
    assert "_tma" not in names_, names_
    boot, rewards, G, gammas, lam, done = x

    def shifted(a, dtype=None):  # contiguous views one element into a buffer: not 16-byte aligned
        t = dev(a) if dtype is None else dev(a).to(dtype)
        buf = torch.empty(a.size + 1, dtype=t.dtype, device="cuda")
        view = buf[1:].view(a.shape)
        view.copy_(t)
        return view

    def go():
        b, r = shifted(boot).requires_grad_(True), shifted(rewards).requires_grad_(True)
        ret = fn_of(1)(b, r, shifted(gammas), shifted(lam), shifted(done, torch.bool))
        ret.backward(shifted(G))
        same((host(ret), host(b.grad), host(r.grad)), ref, True, "offset view")
    names_ = kernels_run(go)
    assert "lambda_ret_fwd_generic" in names_ and "_tma" not in names_, names_
    # an aligned B % 16 == 0 problem of the same rows takes the wide kernels
    x = inputs(T, 4096, True, True, True, 1, 12, density=0.3)
    names_ = kernels_run(lambda: same(run(*x, 1), want(*x, 1), True, "wide"))
    assert "lambda_ret_fwd_tma" in names_ and "lambda_ret_bwd_tma" in names_, names_


def test_requires_grad_subset_and_discount_gradients():
    need_cuda()
    import hpc_rll.rl_utils.td as td
    boot, rewards, G, gammas, lam, done = inputs(250, 4096, True, True, True, 1, 3)
    ref = want(boot, rewards, G, gammas, lam, done, 1)
    b, r = dev(boot), dev(rewards).requires_grad_(True)
    ret = td.generalized_lambda_returns(b, r, dev(gammas), dev(lam), dev(done))
    ret.backward(dev(G))
    assert b.grad is None and np.array_equal(host(r.grad), ref[2])
    b, r = dev(boot).requires_grad_(True), dev(rewards)
    ret = td.generalized_lambda_returns(b, r, dev(gammas), dev(lam), dev(done))
    ret.backward(dev(G))
    assert np.array_equal(host(b.grad), ref[1])
    ret = td.generalized_lambda_returns(dev(boot), dev(rewards), dev(gammas), dev(lam), dev(done))
    assert not ret.requires_grad and np.array_equal(host(ret), ref[0])
    for kw in ("gammas", "lambda_"):
        args = {"gammas": dev(gammas), "lambda_": dev(lam)}
        args[kw] = args[kw].requires_grad_(True)
        with pytest.raises(ValueError, match=kw):
            td.generalized_lambda_returns(dev(boot), dev(rewards), args["gammas"], args["lambda_"], dev(done))
    with pytest.raises(ValueError, match="gammas"):  # wrong shape
        td.multistep_forward_view(dev(boot[1:]), dev(rewards), dev(gammas[:-1]), LAMBDA)
    with pytest.raises(TypeError, match="lambda_"):  # wrong dtype
        td.multistep_forward_view(dev(boot[1:]), dev(rewards), GAMMA, dev(lam).double())


@pytest.mark.parametrize("T,B", [(1024, 64), (64, 65536), (128, 1000)])
def test_run_to_run_identical(T, B):
    need_cuda()
    x = inputs(T, B, True, True, True, 1, 17)
    a, b = run(*x, 1), run(*x, 1)
    for p, q in zip(a, b):
        assert np.array_equal(p.view(np.uint32), q.view(np.uint32))


@pytest.mark.parametrize("T,B", [(1024, 64), (64, 65536), (128, 1000)])
def test_cuda_graph_replay(T, B):
    need_cuda()
    import hpc_rll.rl_utils.td as td
    x0 = inputs(T, B, True, False, True, 1, 23)
    b, r = dev(x0[0]).requires_grad_(True), dev(x0[1]).requires_grad_(True)
    g, gam, d = dev(x0[2]), dev(x0[3]), dev(x0[5])

    def step():
        ret = td.generalized_lambda_returns(b, r, gam, LAMBDA, d)
        ret.backward(g)
        return ret

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    b.grad = None
    r.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ret = step()
    x1 = inputs(T, B, True, False, True, 1, 29)
    with torch.no_grad():
        for t, a in zip((b, r, g, gam), x1[:4]):
            t.copy_(dev(a))
        d.copy_(dev(x1[5]))
    graph.replay()
    torch.cuda.synchronize()
    got = (host(ret), host(b.grad), host(r.grad))
    for p, q in zip(got, run(*x1, 1)):
        assert np.array_equal(p, q)


@pytest.mark.parametrize("cfg", [33, 99])
def test_non_finite_values_under_done(cfg):
    """inf / nan in V where done is set and where it is not: products with m, as in eager PyTorch"""
    need_cuda()
    T, B = 16, 64
    boot, rewards, G, gammas, lam, done = inputs(T, B, False, False, True, 1, 31, density=0.5)
    boot[3, :8] = np.inf
    boot[7, 8:16] = -np.inf
    boot[11, 16:24] = np.nan
    boot[T, 24:32] = np.inf  # the last row's bootstrap
    with np.errstate(all="ignore"):
        ref = want(boot, rewards, G, gammas, lam, done, 1)
    with forced(cfg):
        got = run(boot, rewards, G, gammas, lam, done, 1)
    for g, w in zip(got, ref):
        assert np.array_equal(g, w, equal_nan=True)
    # the eager formula on the CPU agrees too
    from tests.test_lambda_returns_cpu import eager
    e = eager(torch.from_numpy(boot), torch.from_numpy(rewards), gammas, lam, torch.from_numpy(done), 1)
    assert np.array_equal(got[0], e.numpy(), equal_nan=True)


def test_empty():
    need_cuda()
    import hpc_rll.rl_utils.td as td
    for T, B in ((0, 5), (5, 0), (0, 0)):
        for fn, off in FNS.items():
            b = torch.randn(T + off, B, device="cuda", requires_grad=True)
            r = torch.zeros(T, B, device="cuda", requires_grad=True)
            d = torch.zeros(T, B, dtype=torch.bool, device="cuda")
            ret = getattr(td, fn)(b, r, torch.full((T, B), GAMMA, device="cuda"), LAMBDA, d)
            assert ret.shape == (T, B)
            ret.sum().backward()
            assert b.grad.shape == (T + off, B) and r.grad.shape == (T, B)
            assert not b.grad.any()


def test_more_than_2_31_elements():
    """One forward over T*B > 2^31 elements (about 30 GB of device memory), checked column-wise against the oracle."""
    need_cuda()
    T, B = 32800, 65536
    n = T * B
    need = n * (3 * 4 + 1) + (1 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    import hpc_rll.rl_utils.td as td
    gen = torch.Generator(device="cuda").manual_seed(0)
    boot = torch.randn(T + 1, B, device="cuda", generator=gen)
    rewards = torch.randn(T, B, device="cuda", generator=gen)
    done = torch.rand(T, B, device="cuda", generator=gen) < 0.01
    ret = td.generalized_lambda_returns(boot, rewards, GAMMA, LAMBDA, done)
    torch.cuda.synchronize()
    cols = [0, 1, 777, 40001, B - 1]
    w = orc.forward(host(boot[:, cols]), host(rewards[:, cols]), GAMMA, LAMBDA, host(done[:, cols]), 1)
    assert np.array_equal(host(ret[:, cols]), w)
    del boot, rewards, done, ret
    torch.cuda.empty_cache()
