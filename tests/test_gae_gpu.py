"""GAE parity on the GPU: CUDA kernels (through libhpc_rll_b200.so) vs the oracle / golden fixtures.

Tolerances: forward and backward are element-wise chains evaluated in the oracle's exact fp32
operation order, so the column-scan kernels must be BIT-EXACT against oracle_f32 (and the forward
against origin's own fp32 output in the golden fixtures).  Small batches (B <= 2048, T >= 512) automatically take the
single-launch T-split with look-back (scan_lookback.cuh, config 21; automatic for T >= 512), which re-associates the recurrence across
segment boundaries: 2e-6 norm-relative there, and the same shape forced through the column scan is bit-exact.
Gradients vs origin autograd (different summation structure): 1e-5 norm-relative (north_star)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests._golden import Case, names, rel_err
from tests._gpu import dev, host, need_cuda, rng

pytestmark = pytest.mark.gpu

SHAPES = [(1024, 64), (128, 128), (1, 5), (37, 3), (100, 260), (17, 1028), (64, 1), (33, 4), (250, 4096),
          (16, 128), (15, 132), (1000, 7), (129, 2048), (513, 100), (2048, 36), (1024, 4096), (3000, 33), (40, 70), (31, 64),
          (64, 65536), (7, 40000)]  # wide batches: the TMA-staged-output kernels (ragged T and column tiles)


def uses_split(T, B):
    """mirror of lookback_geometry (csrc/scan_lookback.cu): automatic for B <= 2048 and T >= 512"""
    return B <= 2048 and T >= 512


def same(got, want, exact):
    if exact:
        assert np.array_equal(got, want)
    else:
        assert rel_err(got, want) <= 2e-6, rel_err(got, want)


def _run(value, reward, grad_adv, gamma, lam):
    from di_hpc_b200.rl_utils.gae import GAE
    v = dev(value).requires_grad_(True)
    r = dev(reward).requires_grad_(True)
    adv = GAE(*reward.shape)(v, r, gamma, lam)
    adv.backward(dev(grad_adv))
    torch.cuda.synchronize()
    return host(adv), host(v.grad), host(r.grad)


@pytest.mark.parametrize("T,B", SHAPES)
def test_gae_vs_oracle_bitexact(T, B):
    need_cuda()
    g = rng(T * 100003 + B)
    value = g.standard_normal((T + 1, B), dtype=np.float32)
    reward = g.standard_normal((T, B), dtype=np.float32)
    gadv = g.standard_normal((T, B), dtype=np.float32)
    adv, gv, gr = _run(value, reward, gadv, 0.99, 0.97)
    exact = not uses_split(T, B)
    ob = orc.gae_backward(gadv, 0.99, 0.97)
    same(adv, orc.gae_forward(value, reward, 0.99, 0.97), exact)
    same(gv, ob["value"], exact)
    same(gr, ob["reward"], exact)
    if not exact:  # the same shape through the column-scan kernel is bit-exact
        from di_hpc_b200 import _abi
        try:
            _abi.set_config(0, 13)
            adv, gv, gr = _run(value, reward, gadv, 0.99, 0.97)
        finally:
            _abi.set_config(0, -1)
        same(adv, orc.gae_forward(value, reward, 0.99, 0.97), True)
        same(gv, ob["value"], True)
        same(gr, ob["reward"], True)


@pytest.mark.parametrize("name", names("gae"))
def test_gae_vs_golden(name):
    need_cuda()
    c = Case(name)
    adv, gv, gr = _run(c.inp("value"), c.inp("reward"), c.inp("grad_adv"), c.attr("gamma"), c.attr("lambda_"))
    T, B = c.inp("reward").shape
    same(adv, c.out("adv", 32), not uses_split(T, B))  # bit-exact vs origin fp32 on the column-scan path
    assert rel_err(gv, c.grad("value", 32)) <= 1e-5
    assert rel_err(gr, c.grad("reward", 32)) <= 1e-5
    assert rel_err(gv, c.grad("value", 64)) <= 1e-5
    assert rel_err(gr, c.grad("reward", 64)) <= 1e-5


@pytest.mark.parametrize("cfg", [5, 7, 13, 21, 33, 99])
def test_gae_every_kernel_config(cfg):
    """Every kernel regime (and the non-TMA kernel) must give identical bits; 21 = T-split with look-back.  The
    moments forward (gae_with_adv_stats) runs its own kernel for each regime and is bit-exact for all of them."""
    need_cuda()
    from di_hpc_b200 import _abi
    from di_hpc_b200.rl_utils.gae import gae_with_adv_stats
    g = rng(77 + cfg)
    T, B = 203, 1300
    value = g.standard_normal((T + 1, B), dtype=np.float32)
    reward = g.standard_normal((T, B), dtype=np.float32)
    gadv = g.standard_normal((T, B), dtype=np.float32)
    try:
        _abi.set_config(0, cfg)
        adv, gv, gr = _run(value, reward, gadv, 0.95, 0.9)
        adv_m, _ = gae_with_adv_stats(dev(value), dev(reward), 0.95, 0.9)
        adv_m = host(adv_m)
    finally:
        _abi.set_config(0, -1)
    ob = orc.gae_backward(gadv, 0.95, 0.9)
    want = orc.gae_forward(value, reward, 0.95, 0.9)
    same(adv, want, cfg != 21)
    same(gv, ob["value"], cfg != 21)
    same(gr, ob["reward"], cfg != 21)
    same(adv_m, want, True)


def test_gae_strided_views():
    """_ld entry points: operate on column slices of wider buffers without copying."""
    need_cuda()
    from di_hpc_b200 import _abi
    g = rng(5)
    T, B, LD, C0 = 50, 96, 256, 64
    big_v = dev(g.standard_normal((T + 1, LD), dtype=np.float32))
    big_r = dev(g.standard_normal((T, LD), dtype=np.float32))
    big_a = torch.zeros((T, LD), device="cuda")
    L = _abi.lib()
    st = torch.cuda.current_stream().cuda_stream
    _abi.check(L.hpc_rll_gae_forward_ld(big_v[:, C0:].data_ptr(), LD, big_r[:, C0:].data_ptr(), LD,
                                        big_a[:, C0:].data_ptr(), LD, T, B, 0.99, 0.97, st), "fwd_ld")
    torch.cuda.synchronize()
    want = orc.gae_forward(host(big_v[:, C0:C0 + B]).copy(), host(big_r[:, C0:C0 + B]).copy(), 0.99, 0.97)
    assert np.array_equal(host(big_a[:, C0:C0 + B]), want)
    assert float(big_a[:, :C0].abs().max()) == 0.0 and float(big_a[:, C0 + B:].abs().max()) == 0.0


def test_gae_full_size_properties():
    """BASELINE C1 size (T=1024, B=65536): adjoint identity <adv(v,r),G> == <v,gv>+<r,gr> (GAE is linear),
    and exact agreement with the oracle on column slabs (columns are independent)."""
    need_cuda()
    from di_hpc_b200.rl_utils.gae import GAE
    T, B = 1024, 65536
    # drawn on the host so that every GPU sees the same data (torch's CUDA generator depends on the SM count)
    g = rng(1234)
    v = dev(g.standard_normal((T + 1, B), dtype=np.float32)).requires_grad_(True)
    r = dev(g.standard_normal((T, B), dtype=np.float32)).requires_grad_(True)
    G = dev(g.standard_normal((T, B), dtype=np.float32))
    adv = GAE(T, B)(v, r)
    adv.backward(G)
    terms = [adv.detach().double() * G.double(), v.detach().double() * v.grad.double(),
             r.detach().double() * r.grad.double()]
    lhs, rhs = terms[0].sum().item(), terms[1].sum().item() + terms[2].sum().item()
    # fp32 rounding leaves errors of ~eps*|term| in each of the ~2e8 terms, so |lhs - rhs| ~ eps * ||terms||_2 (0.35-2.6x
    # that over five seeds through the oracle, which the kernels match bit for bit); the bar is 8x.  Unlike |lhs| it does
    # not shrink when the sum cancels, and one wrong gradient entry (error ~|term| ~ 1) exceeds it many times over.
    noise = float(np.finfo(np.float32).eps) * sum(float((t * t).sum().item()) for t in terms) ** 0.5
    assert abs(lhs - rhs) <= 8.0 * noise, (lhs, rhs, noise)
    del terms
    for sl in (slice(0, 192), slice(32700, 32900), slice(B - 130, B)):
        vs, rs, gs = host(v[:, sl]).copy(), host(r[:, sl]).copy(), host(G[:, sl]).copy()
        assert np.array_equal(host(adv[:, sl]), orc.gae_forward(vs, rs))
        ob = orc.gae_backward(gs)
        assert np.array_equal(host(v.grad[:, sl]), ob["value"])
        assert np.array_equal(host(r.grad[:, sl]), ob["reward"])


@pytest.mark.parametrize("T,B,rows", [(1024, 4096, 32), (203, 1300, 16), (203, 1300, 60), (37, 516, 4), (37, 516, 5), (64, 1301, 8),
                                      (50, 40000, 12), (9, 70000, 4)])
def test_gae_chunked_scan_is_bit_identical(T, B, rows):
    """hpc_rll_gae_forward_chunk / _backward_chunk: the scan cut into row ranges with the state carried in a (2,B)
    buffer gives the same BITS as the monolithic call and the oracle (incl. a ragged last chunk, B % 4 != 0 ->
    generic kernel, wide B -> TMA-store kernels)."""
    need_cuda()
    from di_hpc_b200 import _abi
    g = rng(T * 7 + B + rows)
    value = g.standard_normal((T + 1, B), dtype=np.float32)
    reward = g.standard_normal((T, B), dtype=np.float32)
    gadv = g.standard_normal((T, B), dtype=np.float32)
    v, r, ga = dev(value), dev(reward), dev(gadv)
    adv, gv, gr = torch.full((T, B), 7.0, device="cuda"), torch.full((T + 1, B), 7.0, device="cuda"), \
        torch.full((T, B), 7.0, device="cuda")
    L = _abi.lib()
    st = torch.cuda.current_stream().cuda_stream
    nC = (T + rows - 1) // rows
    cf = torch.zeros(2, B, device="cuda")
    cf[1] = v[T]
    for k in reversed(range(nC)):
        t0, n = k * rows, min(rows, T - k * rows)
        _abi.check(L.hpc_rll_gae_forward_chunk(v[t0].data_ptr(), r[t0].data_ptr(), adv[t0].data_ptr(), cf.data_ptr(),
                                               T, t0, n, B, 0.95, 0.9, st), "fwd_chunk")
    cb = torch.zeros(2, B, device="cuda")
    for k in range(nC):
        t0, n = k * rows, min(rows, T - k * rows)
        _abi.check(L.hpc_rll_gae_backward_chunk(ga[t0].data_ptr(), gv[t0].data_ptr(), gr[t0].data_ptr(),
                                                cb.data_ptr(), T, t0, n, B, 0.95, 0.9, st), "bwd_chunk")
    torch.cuda.synchronize()
    ob = orc.gae_backward(gadv, 0.95, 0.9)
    assert np.array_equal(host(adv), orc.gae_forward(value, reward, 0.95, 0.9))
    assert np.array_equal(host(gv), ob["value"])
    assert np.array_equal(host(gr), ob["reward"])
    rc = L.hpc_rll_gae_forward_chunk(v.data_ptr(), r.data_ptr(), adv.data_ptr(), cf.data_ptr(), T, T - 1, 4, B, 0.95,
                                     0.9, st)
    assert rc == 1 and b"outside" in L.hpc_rll_last_error()


@pytest.mark.parametrize("T,B,numa", [(257, 9000, False), (1024, 65536, True), (100, 1301, False), (5, 64, True)])
def test_gae_host_entry_matches_oracle(T, B, numa):
    """di_hpc_b200.host.gae_fwd_bwd_host -> hpc_rll_gae_fwd_bwd_host: host buffers in, host buffers out through the
    T-chunked H2D / kernel / D2H pipeline; bit-exact vs the oracle (chunking does not re-associate the scan).
    numa=True uses the library's NUMA-local page-locked allocator, otherwise torch's pin_memory."""
    need_cuda()
    from di_hpc_b200 import host as hp
    g = rng(11 + T + B)
    if numa:
        value, reward, gadv = hp.pinned_empty((T + 1, B)), hp.pinned_empty((T, B)), hp.pinned_empty((T, B))
        out = (hp.pinned_empty((T, B)), hp.pinned_empty((T + 1, B)), hp.pinned_empty((T, B)))
        value.copy_(torch.from_numpy(g.standard_normal((T + 1, B), dtype=np.float32)))
        reward.copy_(torch.from_numpy(g.standard_normal((T, B), dtype=np.float32)))
        gadv.copy_(torch.from_numpy(g.standard_normal((T, B), dtype=np.float32)))
    else:
        value = torch.from_numpy(g.standard_normal((T + 1, B), dtype=np.float32)).pin_memory()
        reward = torch.from_numpy(g.standard_normal((T, B), dtype=np.float32)).pin_memory()
        gadv = torch.from_numpy(g.standard_normal((T, B), dtype=np.float32)).pin_memory()
        out = None
    for _ in range(2):  # second call reuses the pooled pipe
        adv, gv, gr = hp.gae_fwd_bwd_host(value, reward, gadv, 0.99, 0.97, out=out)
    if T * B <= 1 << 22:
        ob = orc.gae_backward(gadv.numpy())
        assert np.array_equal(adv.numpy(), orc.gae_forward(value.numpy(), reward.numpy()))
        assert np.array_equal(gv.numpy(), ob["value"])
        assert np.array_equal(gr.numpy(), ob["reward"])
    else:  # full C1 size: column slabs through the oracle + the device-resident path for everything
        from di_hpc_b200.rl_utils.gae import GAE
        for sl in (slice(0, 130), slice(B - 70, B)):
            assert np.array_equal(adv[:, sl].numpy(), orc.gae_forward(value[:, sl].numpy().copy(),
                                                                      reward[:, sl].numpy().copy()))
            ob = orc.gae_backward(gadv[:, sl].numpy().copy())
            assert np.array_equal(gv[:, sl].numpy(), ob["value"]) and np.array_equal(gr[:, sl].numpy(), ob["reward"])
        v = value.cuda().requires_grad_(True)
        r = reward.cuda().requires_grad_(True)
        a = GAE(T, B)(v, r)
        a.backward(gadv.cuda())
        assert torch.equal(a.detach().cpu(), adv) and torch.equal(v.grad.cpu(), gv) and torch.equal(r.grad.cpu(), gr)
    fwd_only = hp.gae_fwd_bwd_host(value, reward, None, 0.99, 0.97)
    assert torch.equal(fwd_only, adv)


def test_host_numa_helpers():
    need_cuda()
    from di_hpc_b200 import host as hp
    node = hp.device_numa_node(0)
    assert node >= -1
    t = hp.pinned_empty((3, 1000))
    assert t.shape == (3, 1000) and t.is_pinned() and float(t.abs().sum()) == 0.0
    t.fill_(2.0)
    assert float(t.cuda().sum().item()) == 6000.0
    del t


def test_gae_argument_errors():
    need_cuda()
    from di_hpc_b200 import _abi
    from di_hpc_b200.rl_utils.gae import GAE
    with pytest.raises(ValueError):
        GAE(4, 4)(torch.zeros(4, 4, device="cuda"), torch.zeros(4, 4, device="cuda"))
    with pytest.raises(TypeError):
        GAE(4, 4)(torch.zeros(5, 4, device="cuda", dtype=torch.float64), torch.zeros(4, 4, device="cuda"))
    rc = _abi.lib().hpc_rll_gae_forward(None, None, None, 4, 4, 0.99, 0.97, None)
    assert rc == 1 and b"null" in _abi.lib().hpc_rll_last_error()
