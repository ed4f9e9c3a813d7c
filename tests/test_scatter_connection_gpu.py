"""ScatterConnection on the GPU: forward (cover, add) and backward bit-exact against the oracle and against origin's
fixtures, at the reference test shape, a large sparse map and edge shapes; both backward regimes; out-of-range
locations with guard bands; run-to-run and layout invariance; the legacy names; CUDA-graph replay; > 2^31 elements."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests._golden import GOLDEN_DIR, names

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")


def bits(t):
    a = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


def inputs(B, M, N, H, W, seed, one_cell=False, spread=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, M, N, generator=g)
    if spread:  # magnitudes over ~2^-20 .. 2^20: the order of an fp32 sum shows in its bits
        x = x * torch.pow(2.0, torch.randint(-20, 21, (B, M, N), generator=g).float())
    if one_cell:
        loc = torch.zeros(B, M, 2, dtype=torch.int64)
        loc[..., 0], loc[..., 1] = H // 2, W - 1
    else:
        loc = torch.stack([torch.randint(0, H, (B, M), generator=g), torch.randint(0, W, (B, M), generator=g)], 2)
    G = torch.randn(B, N, H, W, generator=g)
    return x, loc, G


def module_run(x, loc, G, H, W, mode):
    from hpc_rll.torch_utils.network.scatter_connection import ScatterConnection
    B, M, N = x.shape
    xd = x.cuda().requires_grad_(True)
    out = ScatterConnection(B, M, N, H, W, mode).cuda()(xd, loc.cuda())
    out.backward(G.cuda())
    torch.cuda.synchronize()
    return out.detach(), xd.grad


def check_vs_oracle(B, M, N, H, W, seed, modes=("cover", "add"), **kw):
    from tests import scatter_oracle as orc
    x, loc, G = inputs(B, M, N, H, W, seed, **kw)
    want_gx = orc.scatter_connection_backward(G.numpy(), loc.numpy())
    for mode in modes:
        out, gx = module_run(x, loc, G, H, W, mode)
        assert out.shape == (B, N, H, W) and gx.shape == (B, M, N)
        assert same(out, orc.scatter_connection_forward(x.numpy(), loc.numpy(), H, W, mode)), (mode, B, M, N, H, W)
        assert same(gx, want_gx), ("grad", mode, B, M, N, H, W)


def test_reference_test_shape():  # S1: dense, many collisions; dense backward regime
    check_vs_oracle(256, 256, 256, 16, 16, 1)


def test_large_sparse_map():  # S2: sparse, sector-gather backward regime
    check_vs_oracle(64, 512, 32, 128, 128, 2, spread=True)


@pytest.mark.parametrize("B,M,N,H,W,kw", [
    (1, 37, 8, 6, 6, {}),
    (5, 1, 16, 9, 7, {}),
    (3, 5000, 12, 10, 10, {"spread": True}),    # several 1024-entity passes, heavy collisions
    (2, 5000, 4, 64, 96, {}),                   # several passes over a tiled map
    (4, 300, 1, 12, 12, {}),
    (4, 300, 3, 7, 9, {"spread": True}),        # odd N, odd H*W
    (2, 300, 33, 5, 13, {}),                    # odd H*W: scalar stores
    (2, 2000, 33, 16, 16, {}),                  # N not a multiple of the channel chunk
    (3, 64, 5, 4, 4, {"one_cell": True, "spread": True}),
    (2, 1100, 8, 3, 3, {"one_cell": True}),     # one cell, more than one pass
    (2, 100, 7, 300, 301, {}),                  # many tiles, almost every cell empty
])
def test_edge_shapes(B, M, N, H, W, kw):
    check_vs_oracle(B, M, N, H, W, B * 131 + M + N + H * W, **kw)


def backward_kernels(B, M, N, H, W):
    """Names of the backward kernels one module call launches.  Profiled in a fresh process: late in a long GPU run in
    one process, torch.profiler sessions have come back with no CUDA events at all."""
    code = "\n".join([
        "import torch",
        "from tests.test_scatter_connection_gpu import inputs, module_run",
        "x, loc, G = inputs(%d, %d, %d, %d, %d, 5)" % (B, M, N, H, W),
        "with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:",
        "    module_run(x, loc, G, %d, %d, 'add')" % (H, W),
        "print('\\n'.join({e.name for e in prof.events() if 'scatter_conn_bwd' in e.name}))"])
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return set(r.stdout.splitlines())


@pytest.mark.parametrize("M,dense", [(64, True), (8, False)])
def test_both_backward_regimes(M, dense):
    B, N, H, W = 4, 33, 16, 16  # 8*M >= H*W picks the staged-plane kernel
    ks = backward_kernels(B, M, N, H, W)
    assert len(ks) == 1 and ("dense" in next(iter(ks))) == dense, ks
    check_vs_oracle(B, M, N, H, W, M)


@pytest.mark.parametrize("name", names("scatter"))
def test_bit_exact_against_origin(name):
    z = np.load("%s/%s.npz" % (GOLDEN_DIR, name))
    out, gx = module_run(torch.from_numpy(z["in_x"]), torch.from_numpy(z["in_location"]),
                         torch.from_numpy(z["in_G"]), int(z["H"]), int(z["W"]), str(z["scatter_type"]))
    assert same(out, z["out"]) and same(gx, z["grad_x"]), name


@pytest.mark.parametrize("guard", [7, 16])  # 7: unaligned output -> scalar stores; 16: float4 stores
@pytest.mark.parametrize("mode", ["cover", "add"])
def test_out_of_range_locations_are_dropped(guard, mode):
    from di_hpc_b200 import _abi
    from tests import scatter_oracle as orc
    B, M, N, H, W = 3, 200, 6, 8, 12
    x, loc, G = inputs(B, M, N, H, W, 11)
    g = torch.Generator().manual_seed(12)
    bad = torch.randint(0, 4, (B, M), generator=g)  # 0: keep, 1: y<0 or y>=H, 2: x<0 or x>=W, 3: both
    big = torch.randint(0, 2, (B, M), generator=g).bool()
    loc[..., 0] = torch.where(bad % 2 == 1, torch.where(big, H + loc[..., 0], -1 - loc[..., 0]), loc[..., 0])
    loc[..., 1] = torch.where(bad >= 2, torch.where(big, W + loc[..., 1], -3 - loc[..., 1]), loc[..., 1])
    no, nx = B * N * H * W, B * M * N
    store_o = torch.full((no + 2 * guard,), float("nan"), device="cuda")
    store_x = torch.full((nx + 2 * guard,), float("nan"), device="cuda")
    out, gx = store_o[guard:guard + no], store_x[guard:guard + nx]
    xd, ld, Gd = x.cuda(), loc.cuda(), G.cuda()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    L, s = _abi.lib(), _abi.stream_of(xd)
    _abi.check(L.hpc_rll_scatter_connection_forward(p(xd), p(ld), p(out), B, M, N, H, W,
                                                    _abi.SCATTER_ADD if mode == "add" else _abi.SCATTER_COVER, s), "fwd")
    _abi.check(L.hpc_rll_scatter_connection_backward(p(Gd), p(ld), p(gx), B, M, N, H, W, s), "bwd")
    torch.cuda.synchronize()
    assert same(out.view(B, N, H, W), orc.scatter_connection_forward(x.numpy(), loc.numpy(), H, W, mode))
    want = orc.scatter_connection_backward(G.numpy(), loc.numpy())
    assert same(gx.view(B, M, N), want)
    assert not want[(bad != 0).numpy()].any() and (bad != 0).any()
    for st in (store_o, store_x):
        assert torch.isnan(st[:guard]).all() and torch.isnan(st[-guard:]).all()


def test_add_is_run_to_run_identical():
    x, loc, G = inputs(16, 4000, 32, 4, 4, 21, spread=True)
    a = module_run(x, loc, G, 4, 4, "add")
    b = module_run(x, loc, G, 4, 4, "add")
    assert same(a[0], b[0]) and same(a[1], b[1])


@pytest.mark.parametrize("mode", ["cover", "add"])
def test_non_contiguous_x(mode):
    from hpc_rll.torch_utils.network.scatter_connection import ScatterConnection
    B, M, N, H, W = 4, 300, 24, 10, 10
    x, loc, _ = inputs(B, M, N, H, W, 31)
    base = x.transpose(1, 2).contiguous().cuda()  # (B, N, M)
    xt = base.transpose(1, 2)
    assert not xt.is_contiguous()
    m = ScatterConnection(B, M, N, H, W, mode)
    assert same(m(xt, loc.cuda()), m(x.cuda(), loc.cuda()))


@pytest.mark.parametrize("mode", ["cover", "add"])
def test_legacy_names_write_into_the_callers_tensors(mode):
    import hpc_torch_utils_network as net
    B, M, N, H, W = 3, 150, 20, 9, 8
    x, loc, G = inputs(B, M, N, H, W, 41)
    want_out, want_gx = module_run(x, loc, G, H, W, mode)
    out = torch.full((B, N, H, W), float("nan"), device="cuda")
    gin = torch.full((B, M, N), float("nan"), device="cuda")
    net.ScatterConnectionForward([x.cuda(), loc.cuda()], [out], mode)
    net.ScatterConnectionBackward([G.cuda(), loc.cuda()], [gin])
    torch.cuda.synchronize()
    assert same(out, want_out) and same(gin, want_gx)


def test_cuda_graph_replay():
    from hpc_rll.torch_utils.network.scatter_connection import ScatterConnection
    B, M, N, H, W = 8, 256, 32, 16, 16
    x, loc, G = inputs(B, M, N, H, W, 51)
    want = {mode: module_run(x, loc, G, H, W, mode) for mode in ("cover", "add")}
    for mode in ("cover", "add"):
        m = ScatterConnection(B, M, N, H, W, mode)
        xd = x.cuda().requires_grad_(True)
        ld, Gd = loc.cuda(), G.cuda()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):  # warm-up outside the capture
            m(xd, ld).backward(Gd)
        torch.cuda.current_stream().wait_stream(s)
        xd.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m(xd, ld)
            (gx,) = torch.autograd.grad(out, xd, Gd)
        for _ in range(2):
            out.zero_()
            gx.zero_()
            graph.replay()
            torch.cuda.synchronize()
            assert same(out, want[mode][0]) and same(gx, want[mode][1]), mode


def test_more_than_2_31_output_elements():
    """out and grad_out hold B*N*H*W = 2^31 + 2^25 elements (8.6 GB each in fp32); sampled (b, n) planes and entity
    rows are checked against the oracle run on those planes alone."""
    import hpc_torch_utils_network as net
    from di_hpc_b200 import _ext
    from tests import scatter_oracle as orc
    B, M, N, H, W = 2, 96, 16, 8192, 8448
    assert B * N * H * W > 2**31
    if torch.cuda.get_device_properties(0).total_memory < 24 * 2**30:
        pytest.skip("needs 24 GB of device memory")
    x, loc, _ = inputs(B, M, N, 4, 4, 61)  # small draw; locations spread over the whole map below
    g = torch.Generator().manual_seed(62)
    loc = torch.stack([torch.randint(0, H, (B, M), generator=g), torch.randint(0, W, (B, M), generator=g)], 2)
    loc[:, :4] = torch.tensor([[H - 1, W - 1], [H - 1, W - 1], [0, 0], [H - 1, 0]])  # collisions at the far end
    xd, ld = x.cuda(), loc.cuda()
    out = _ext.require().scatter_connection(xd, ld, H, W, "add")
    gin = torch.empty(B, M, N, device="cuda")
    net.ScatterConnectionBackward([out, ld], [gin])  # grad_out = out: the gather reads the far planes back
    torch.cuda.synchronize()
    gin = gin.cpu().numpy()
    for b, n in [(0, 0), (1, N - 1), (1, 7)]:
        plane = orc.scatter_connection_forward(x[b:b + 1, :, n:n + 1].numpy(), loc[b:b + 1].numpy(), H, W, "add")
        assert same(out[b, n], plane[0, 0]), (b, n)
        assert same(gin[b, :, n], orc.scatter_connection_backward(plane, loc[b:b + 1].numpy())[0, :, 0]), (b, n)
        del plane
