"""Episode-aware GAE on the GPU (``hpc_rll.rl_utils.gae.gae``) against the oracle (tests/gae_episodic_oracle.py).

The wide (TMA) and generic kernels evaluate the formula in the oracle's exact fp32 operation order and must be
BIT-EXACT, forward and backward.  The small-batch look-back kernels (config 21; automatic for B <= 2048, T >= 512)
re-associate the recurrence at segment boundaries: 2e-6 norm-relative there, and the same shapes forced through the
generic kernel (config 99) are bit-exact."""
import numpy as np
import pytest
import torch

from tests import gae_episodic_oracle as orc
from tests._golden import rel_err
from tests._gpu import dev, host, need_cuda, rng

pytestmark = pytest.mark.gpu

OP = 10  # HPC_RLL_OP_GAE_EPISODIC
SHAPES = [(1, 5), (37, 3), (1000, 7), (128, 1000), (513, 100), (1024, 64), (100, 260), (250, 4096), (64, 65536),
          (7, 40000)]
CONFIGS = [-1, 33, 21, 99]
MASKS = [(d, m) for d in (0.0, 0.01, 0.3, 1.0) for m in ("other", "none")]
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


def inputs(T, B, density, traj_mode, seed):
    g = rng(seed)
    value, next_value, reward, gadv = (g.standard_normal((T, B), dtype=np.float32) for _ in range(4))
    done = g.random((T, B)) < density
    traj = None if traj_mode == "none" else g.random((T, B)) < max(density, 0.2)
    return value, next_value, reward, gadv, done, traj


def run(value, next_value, reward, gadv, done, traj, gamma=GAMMA, lambda_=LAMBDA, mask_dtype=torch.bool):
    from hpc_rll.rl_utils.gae import gae, gae_data
    v, nv, r = (dev(x).requires_grad_(True) for x in (value, next_value, reward))
    d = None if done is None else dev(done).to(mask_dtype)
    tr = None if traj is None else dev(traj).to(mask_dtype)
    adv = gae(gae_data(v, nv, r, d, tr), gamma, lambda_)
    adv.backward(dev(gadv))
    torch.cuda.synchronize()
    return host(adv), host(v.grad), host(nv.grad), host(r.grad)


def want(value, next_value, reward, gadv, done, traj, gamma=GAMMA, lambda_=LAMBDA):
    wb = orc.backward(gadv, done, traj, gamma, lambda_)
    return orc.forward(value, next_value, reward, done, traj, gamma, lambda_), wb["value"], wb["next_value"], \
        wb["reward"]


def same(got, ref, exact, what):
    for g, w, name in zip(got, ref, ("adv", "grad_value", "grad_next_value", "grad_reward")):
        if exact:
            assert np.array_equal(g, w), "%s %s not bit-exact (max diff %g)" % (what, name, np.max(np.abs(g - w)))
        else:
            assert rel_err(g, w) <= 2e-6, (what, name, rel_err(g, w))


@pytest.mark.parametrize("cfg", CONFIGS)
@pytest.mark.parametrize("T,B", SHAPES)
def test_vs_oracle(T, B, cfg):
    need_cuda()
    exact = not uses_split(T, B, cfg)
    with forced(cfg):
        for i, (density, traj_mode) in enumerate(MASKS):
            x = inputs(T, B, density, traj_mode, T * 7919 + B * 13 + i)
            same(run(*x), want(*x), exact, (T, B, cfg, density, traj_mode))


def test_no_masks():
    need_cuda()
    for T, B, cfg in ((64, 65536, -1), (64, 65532, -1), (1024, 64, -1), (37, 3, -1), (100, 260, 99)):
        x = inputs(T, B, 0.0, "none", T + B)[:4] + (None, None)
        with forced(cfg):
            same(run(*x), want(*x), not uses_split(T, B, cfg), (T, B, cfg))


@pytest.mark.parametrize("T,B", [(64, 4096), (1024, 64), (100, 260)])
def test_mask_dtypes(T, B):
    need_cuda()
    value, next_value, reward, gadv, done, traj = inputs(T, B, 0.3, "other", 5)
    ref = run(value, next_value, reward, gadv, done, traj, mask_dtype=torch.bool)
    for dt in (torch.uint8, torch.float32, torch.int64):
        got = run(value, next_value, reward, gadv, done, traj, mask_dtype=dt)
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), dt
    # a fractional float mask counts as set, as does any non-zero byte
    from hpc_rll.rl_utils.gae import gae, gae_data
    v, nv, r = dev(value), dev(next_value), dev(reward)
    half = dev(done.astype(np.float32) * 0.5)
    bytes_ = dev(done.astype(np.uint8) * 7)
    a = gae(gae_data(v, nv, r, half, None), GAMMA, LAMBDA)
    b = gae(gae_data(v, nv, r, bytes_, None), GAMMA, LAMBDA)
    c = gae(gae_data(v, nv, r, dev(done), None), GAMMA, LAMBDA)
    assert torch.equal(a, c) and torch.equal(b, c)


def kernels_run(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " ".join(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def test_ragged_and_misaligned_fall_to_generic():
    need_cuda()
    from hpc_rll.rl_utils.gae import gae, gae_data
    T, B = 96, 4104  # B % 16 == 8: no uint8 tensor map
    x = inputs(T, B, 0.3, "other", 11)
    ref = want(*x)
    names = kernels_run(lambda: same(run(*x), ref, True, "ragged"))
    assert "gae_episodic_fwd_generic" in names and "gae_episodic_bwd_generic" in names, names
    # contiguous views whose data pointers are not 16-byte aligned
    value, next_value, reward, gadv, done, traj = x

    def shifted(a, dtype=None):
        t = dev(a) if dtype is None else dev(a).to(dtype)
        buf = torch.empty(a.size + 1, dtype=t.dtype, device="cuda")
        view = buf[1:].view(a.shape)
        view.copy_(t)
        return view

    def go():
        v, nv, r = (shifted(a).requires_grad_(True) for a in (value, next_value, reward))
        adv = gae(gae_data(v, nv, r, shifted(done, torch.bool), shifted(traj, torch.bool)), GAMMA, LAMBDA)
        adv.backward(dev(gadv))
        same((host(adv), host(v.grad), host(nv.grad), host(r.grad)), ref, True, "misaligned")
    names = kernels_run(go)
    assert "gae_episodic_fwd_generic" in names, names
    # column slices of wider tensors (not contiguous: the torch layer copies them)
    def col_slice(a):
        return dev(np.concatenate([np.zeros((T, 1), a.dtype), a], axis=1))[:, 1:]
    v, nv, r = (col_slice(a).requires_grad_(True) for a in (value, next_value, reward))
    adv = gae(gae_data(v, nv, r, col_slice(done), col_slice(traj)), GAMMA, LAMBDA)
    adv.backward(dev(gadv))
    same((host(adv), host(v.grad), host(nv.grad), host(r.grad)), ref, True, "column slice")


def test_requires_grad_subset():
    need_cuda()
    from hpc_rll.rl_utils.gae import gae, gae_data
    value, next_value, reward, gadv, done, traj = inputs(250, 4096, 0.3, "other", 3)
    ref = want(value, next_value, reward, gadv, done, traj)
    v, nv = dev(value), dev(next_value)
    r = dev(reward).requires_grad_(True)
    adv = gae(gae_data(v, nv, r, dev(done), dev(traj)), GAMMA, LAMBDA)
    adv.backward(dev(gadv))
    assert v.grad is None and nv.grad is None
    assert np.array_equal(host(r.grad), ref[3])
    nv = dev(next_value).requires_grad_(True)
    adv = gae(gae_data(dev(value), nv, dev(reward), dev(done), None), GAMMA, LAMBDA)
    adv.backward(dev(gadv))
    assert np.array_equal(host(nv.grad), orc.backward(gadv, done, None, GAMMA, LAMBDA)["next_value"])
    # no input requires grad: a plain forward
    adv = gae(gae_data(dev(value), dev(next_value), dev(reward), dev(done), dev(traj)), GAMMA, LAMBDA)
    assert not adv.requires_grad and np.array_equal(host(adv), ref[0])


@pytest.mark.parametrize("T,B", [(1024, 64), (64, 65536), (128, 1000)])
def test_run_to_run_identical(T, B):
    need_cuda()
    x = inputs(T, B, 0.3, "other", 17)
    a, b = run(*x), run(*x)
    for p, q in zip(a, b):
        assert np.array_equal(p.view(np.uint32), q.view(np.uint32))


@pytest.mark.parametrize("T,B", [(1024, 64), (64, 65536), (128, 1000)])
def test_cuda_graph_replay(T, B):
    need_cuda()
    from hpc_rll.rl_utils.gae import gae, gae_data
    x0 = inputs(T, B, 0.3, "other", 23)
    v, nv, r = (dev(a).requires_grad_(True) for a in x0[:3])
    g, d, tr = dev(x0[3]), dev(x0[4]), dev(x0[5])

    def step():
        adv = gae(gae_data(v, nv, r, d, tr), GAMMA, LAMBDA)
        adv.backward(g)
        return adv

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    for t in (v, nv, r):
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        adv = step()
    x1 = inputs(T, B, 0.1, "other", 29)
    with torch.no_grad():
        for t, a in zip((v, nv, r, g), x1[:4]):
            t.copy_(dev(a))
        d.copy_(dev(x1[4]))
        tr.copy_(dev(x1[5]))
    graph.replay()
    torch.cuda.synchronize()
    got = (host(adv), host(v.grad), host(nv.grad), host(r.grad))
    eager = run(*x1)
    for p, q in zip(got, eager):
        assert np.array_equal(p, q)


def test_empty():
    need_cuda()
    from hpc_rll.rl_utils.gae import gae, gae_data
    for T, B in ((0, 5), (5, 0), (0, 0)):
        v, nv, r = (torch.zeros(T, B, device="cuda", requires_grad=True) for _ in range(3))
        d = torch.zeros(T, B, dtype=torch.bool, device="cuda")
        adv = gae(gae_data(v, nv, r, d, None))
        assert adv.shape == (T, B)
        adv.sum().backward()
        assert v.grad.shape == (T, B) and nv.grad.shape == (T, B) and r.grad.shape == (T, B)


def test_more_than_2_31_elements():
    """One forward over T*B > 2^31 elements (about 40 GB of device memory), checked column-wise against the oracle."""
    need_cuda()
    T, B = 32800, 65536
    n = T * B
    need = n * (4 * 4 + 1) + (1 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    from hpc_rll.rl_utils.gae import gae, gae_data
    gen = torch.Generator(device="cuda").manual_seed(0)
    value, next_value, reward = (torch.randn(T, B, device="cuda", generator=gen) for _ in range(3))
    done = torch.rand(T, B, device="cuda", generator=gen) < 0.01
    adv = gae(gae_data(value, next_value, reward, done, None), GAMMA, LAMBDA)
    torch.cuda.synchronize()
    cols = [0, 1, 777, 40001, B - 1]
    w = orc.forward(host(value[:, cols]), host(next_value[:, cols]), host(reward[:, cols]), host(done[:, cols]), None,
                    GAMMA, LAMBDA)
    assert np.array_equal(host(adv[:, cols]), w)
    del value, next_value, reward, done, adv
    torch.cuda.empty_cache()
