"""Importance weights and the time-batch cross entropy on the GPU (``hpc_rll.rl_utils.vtrace.compute_importance_weights``
/ ``hpc_rll.rl_utils.upgo.tb_cross_entropy``) against the reference's origin (tests/golden/importance_*.npz) and the
fp64 oracle (tests/importance_weights_oracle.py), on every row-softmax path of tests/row_paths.py.

The importance-weights forward reads target and behaviour logits, so it takes the V-trace forward's path; the cross
entropy reads one logits tensor, UPGO's forward path; both backwards run the shared softmax-gradient kernels.  Outputs
and gradients must agree with the oracle to 1e-5 (rel_err for outputs, grad_err for gradients), masked entries must get
a gradient of exactly 0, -inf / finfo.min / -1e9 masks must give the same bits, and two identical calls must too.  The
ratios must be bit-identical to the ones the fused V-trace forward forms for the same rows."""
import ctypes
import zlib

import numpy as np
import pytest
import torch

from tests import importance_weights_oracle as orc
from tests import row_paths as rp
from tests._golden import GOLDEN_DIR, grad_err, names, rel_err
from tests._gpu import dev, host, need_cuda, rng

pytestmark = pytest.mark.gpu
TOL = 1e-5
MASK_VALUE = {rp.NEG_INF: -np.inf, rp.FINFO_MIN: float(np.finfo(np.float32).min), rp.NEG_1E9: -1e9}


def n_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def load(name):
    return np.load("%s/%s.npz" % (GOLDEN_DIR, name))


def check_close(name, got, want, grad=False):
    e = (grad_err if grad else rel_err)(got, want)
    assert np.isfinite(got).all() and e <= TOL, "%s: err %.3e" % (name, e)


# ------------------------------------------------------------------------------------------------- runs
def run_is(t, b, a, G, want_t=True, want_b=True):
    """ρ and the gradients of sum(ρ·G) through the public function; None for a gradient not asked for"""
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    t = t.detach().requires_grad_(want_t)
    b = b.detach().requires_grad_(want_b)
    rho = compute_importance_weights(t, b, a, requires_grad=True)
    rho.backward(G)
    torch.cuda.synchronize()
    return dict(out=host(rho), grad_target_output=None if t.grad is None else host(t.grad),
                grad_behaviour_output=None if b.grad is None else host(b.grad))


def run_ce(x, label, G):
    from hpc_rll.rl_utils.upgo import tb_cross_entropy
    x = x.detach().requires_grad_(True)
    out = tb_cross_entropy(x, label)
    out.backward(G)
    torch.cuda.synchronize()
    return dict(out=host(out), grad_logit=host(x.grad))


def fused_vtrace_ratios(t, b, a):
    """the ratios hpc_rll_vtrace_forward writes to the head of its workspace, for the (T, B, N) logits t, b"""
    from di_hpc_b200 import _abi
    L = _abi.lib()
    T, B, N = t.shape
    value, reward = torch.zeros(T + 1, B, device="cuda"), torch.zeros(T, B, device="cuda")
    losses, pg, gv = torch.empty(3, device="cuda"), torch.empty(T, B, device="cuda"), torch.empty(T, B, device="cuda")
    ws = _abi.workspace(_abi.OP_VTRACE, T, B, N, "cuda")
    _abi.check(L.hpc_rll_vtrace_forward(t.data_ptr(), b.data_ptr(), a.data_ptr(), value.data_ptr(), reward.data_ptr(),
                                        None, losses.data_ptr(), pg.data_ptr(), gv.data_ptr(), T, B, N, 0.99, 0.95,
                                        1.0, 1.0, 1.0, 0, ws.data_ptr(), ctypes.c_size_t(ws.numel()),
                                        _abi.stream_of(t)), "hpc_rll_vtrace_forward")
    torch.cuda.synchronize()
    return host(ws[:T * B * 4].view(torch.float32)).reshape(T, B)


# ------------------------------------------------------------------------------------------------- fixtures
@pytest.mark.parametrize("name", names("importance_is"))
def test_importance_weights_vs_origin_fixtures(name):
    need_cuda()
    z = load(name)
    got = run_is(dev(z["in_target_output"]), dev(z["in_behaviour_output"]), dev(z["in_action"]), dev(z["in_grad"]))
    ref = orc.importance_weights(z["in_target_output"], z["in_behaviour_output"], z["in_action"], z["in_grad"])
    for k in ("out", "grad_target_output", "grad_behaviour_output"):
        assert got[k].shape == z[k].shape, k
        check_close(k + " vs origin", got[k], z[k], grad=k != "out")
        check_close(k + " vs oracle", got[k], ref[k], grad=k != "out")
        if k != "out":
            assert (got[k][np.isinf(z["in_" + k[5:]])] == 0).all(), k
    if "same" in name or "_n1_" in name:  # identical rows, or one action: ρ = 1 exactly
        assert (got["out"] == 1).all()


@pytest.mark.parametrize("name", names("importance_ce"))
def test_tb_cross_entropy_vs_origin_fixtures(name):
    need_cuda()
    z = load(name)
    got = run_ce(dev(z["in_logit"]), dev(z["in_label"]), dev(z["in_grad"]))
    ref = orc.tb_cross_entropy(z["in_logit"], z["in_label"], z["in_grad"])
    for k in ("out", "grad_logit"):
        assert got[k].shape == z[k].shape, k
        check_close(k + " vs origin", got[k], z[k], grad=k != "out")
        check_close(k + " vs oracle", got[k], ref[k], grad=k != "out")
    assert (got["grad_logit"][np.isinf(z["in_logit"])] == 0).all()


# ------------------------------------------------------------------------------------------------- row paths
# op "is": V-trace forward geometry (two logits tensors at one offset); op "ce": UPGO forward geometry
FWD_GEOMETRY = {"is": "vtrace", "ce": "upgo"}
WRAPPED = (("is", 8, 0), ("is", 9, 0), ("is", 257, 0), ("ce", 6, 1), ("ce", 300, 1))


def cases():
    out = []
    for op in ("is", "ce"):
        for N, off in rp.MASKED_GEOMS:
            vals = rp.ALL_MASK_VALUES if (N, off) in rp.ALL_VALUE_GEOMS else (rp.NEG_INF, )
            out.append(rp.Case(op, N, off, rp.small_rows("vtrace"), True, vals, False))
        for N, off in rp.OFFSET_GEOMS:
            out.append(rp.Case(op, N, off, rp.small_rows("vtrace"), False, (), False))
    for N, off in ((33, 0), (300, 1), (9, 0), (16, 0)):  # the behaviour policy has its own legal set
        out.append(rp.Case("is", N, off, rp.small_rows("vtrace"), True, (rp.NEG_INF, ), True))
    for op, N, off in WRAPPED:
        out.append(rp.Case(op, N, off, None, True, (rp.NEG_INF, ), False))
    return out


def make_inputs(case, shape, kind):
    from tests.test_masked_rows_gpu import edge_actions, make_mask
    g = np.random.default_rng(zlib.crc32(("importance-" + rp.case_id(case)).encode()))
    R, N = int(np.prod(shape)), case.N
    action = g.integers(0, N, R)
    d = dict(action=action, logits=(g.standard_normal((R, N)) * 1.5).astype(np.float32),
             G=g.standard_normal(R).astype(np.float32))
    if case.op == "is":
        d["logits2"] = (d["logits"] + 0.5 * g.standard_normal((R, N))).astype(np.float32)
    if case.masked:
        edge_actions(g, action, N)
        d["mask"] = make_mask(g, R, N, action, kind)
        if "logits2" in d:
            d["mask2"] = make_mask(g, R, N, action, kind) if case.differ else d["mask"]
    return d


def filled(d, fill):
    out = {}
    for k, mk in (("logits", "mask"), ("logits2", "mask2")):
        if k in d:
            x = d[k].copy()
            if mk in d:
                x[d[mk]] = fill
            out[k] = x
    return out


def offset_view(a, off):
    store = torch.empty(a.size + 4, dtype=torch.float32, device="cuda")
    x = store[off:off + a.size].view(a.shape)
    x.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    assert x.data_ptr() % 16 == 4 * off, (x.data_ptr(), off)
    return x


def run_case(case, shape, d, fill):
    lg = filled(d, fill)
    N = case.N
    a = dev(d["action"].reshape(shape))
    G = dev(d["G"].reshape(shape))
    t = offset_view(lg["logits"].reshape(shape + (N, )), case.off)
    if case.op == "ce":
        return run_ce(t, a, G)
    b = offset_view(lg["logits2"].reshape(shape + (N, )), case.off)
    out = run_is(t, b, a, G)
    out["fused_vtrace_rho"] = fused_vtrace_ratios(t, b, a)
    return out


def bits(out):
    return {k: np.asarray(v).tobytes() for k, v in out.items()}


@pytest.mark.parametrize("case", cases(), ids=rp.case_id)
def test_row_path(case):
    need_cuda()
    sms = n_sms()
    shape = rp.case_shape(rp.Case("vtrace", *case[1:]), rp.case_rows(case, sms))
    R = int(np.prod(shape))
    paths = dict(fwd=rp.row_path(FWD_GEOMETRY[case.op], "fwd", case.N, case.off, R, sms),
                 bwd=rp.row_path(FWD_GEOMETRY[case.op], "bwd", case.N, case.off, R, sms))
    if case.rows is None:
        assert all(p.passes >= 2 for p in paths.values()), paths
    where = "%s N=%d off=%d R=%d paths=%s" % (case.op, case.N, case.off, R, paths)
    d = make_inputs(case, shape, paths["fwd"].kind)
    lg = filled(d, -np.inf)
    if case.op == "is":
        ref = orc.importance_weights(lg["logits"], lg["logits2"], d["action"], d["G"])
        grads = ("grad_target_output", "grad_behaviour_output")
        masks = (d.get("mask"), d.get("mask2"))
    else:
        ref = orc.tb_cross_entropy(lg["logits"], d["action"], d["G"])
        grads, masks = ("grad_logit", ), (d.get("mask"), )
    results = {}
    for value in case.mask_values or ("none", ):
        out = run_case(case, shape, d, MASK_VALUE.get(value, 0.0))
        check_close("%s mask=%s: out" % (where, value), out["out"].reshape(-1), ref["out"])
        for k, m in zip(grads, masks):
            got = out[k].reshape(R, case.N)
            check_close("%s mask=%s: %s" % (where, value, k), got, ref[k].reshape(R, case.N), grad=True)
            if m is not None:
                assert (got[m] == 0).all(), "%s mask=%s: %s non-zero at a masked entry" % (where, value, k)
                only = m.sum(axis=1) == case.N - 1
                assert only.any() and (got[only] == 0).all(), "%s: %s non-zero in a one-legal-action row" % (where, k)
        if case.op == "is":
            assert np.array_equal(out["out"].reshape(-1).view(np.uint32),
                                  out["fused_vtrace_rho"].reshape(-1).view(np.uint32)), \
                "%s mask=%s: ratios differ from the fused V-trace forward's" % (where, value)
        again = bits(run_case(case, shape, d, MASK_VALUE.get(value, 0.0)))
        for k, v in bits(out).items():
            assert v == again[k], "%s mask=%s: %s differs between two identical calls" % (where, value, k)
        results[value] = out
    first = (case.mask_values or ("none", ))[0]
    for value, out in results.items():
        for k, v in out.items():
            assert np.array_equal(v, results[first][k]), "%s: %s with mask=%s differs from mask=%s" % (where, k, value,
                                                                                                    first)


# ------------------------------------------------------------------------------------------------- requires_grad
def test_requires_grad_semantics():
    need_cuda()
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    g = rng(7)
    T, B, N = 5, 6, 7
    tn = (g.standard_normal((T, B, N)) * 1.5).astype(np.float32)
    bn = (tn + 0.5 * g.standard_normal((T, B, N))).astype(np.float32)
    an, Gn = g.integers(0, N, (T, B)), g.standard_normal((T, B)).astype(np.float32)
    a, G = dev(an), dev(Gn)
    t, b = dev(tn).requires_grad_(True), dev(bn).requires_grad_(True)
    ref = orc.importance_weights(tn, bn, an, Gn)
    # False (the default): no graph, even when the inputs require grad
    rho = compute_importance_weights(t, b, a)
    assert not rho.requires_grad and rho.grad_fn is None
    check_close("out", host(rho), ref["out"])
    # True inside an outer no_grad: the op still builds a graph
    with torch.no_grad():
        rho2 = compute_importance_weights(t, b, a, requires_grad=True)
    assert rho2.requires_grad and rho2.grad_fn is not None
    assert np.array_equal(host(rho), host(rho2))
    rho2.backward(G)
    check_close("grad_target_output", host(t.grad), ref["grad_target_output"], grad=True)
    check_close("grad_behaviour_output", host(b.grad), ref["grad_behaviour_output"], grad=True)
    # only the tensors that require grad receive gradients
    for want_t, want_b in ((True, False), (False, True)):
        out = run_is(dev(tn), dev(bn), a, G, want_t, want_b)
        assert (out["grad_target_output"] is None) != want_t and (out["grad_behaviour_output"] is None) != want_b
        k = "grad_target_output" if want_t else "grad_behaviour_output"
        check_close(k, out[k], ref[k], grad=True)
        assert np.array_equal(out[k], host(t.grad if want_t else b.grad))  # the same bits as with both wanted
    # neither requires grad: nothing to differentiate
    rho3 = compute_importance_weights(dev(tn), dev(bn), a, requires_grad=True)
    assert not rho3.requires_grad
    # N = 1: ρ = 1 exactly and zero gradients
    one = run_is(dev(tn[..., :1]), dev(bn[..., :1]), torch.zeros_like(a), G)
    assert (one["out"] == 1).all()
    assert not one["grad_target_output"].any() and not one["grad_behaviour_output"].any()


def test_bn_and_flat_shapes():
    """(B, N) logits give (B,) ratios, as Categorical does; the cross entropy accepts T*B rows of N in any shape"""
    need_cuda()
    from hpc_rll.rl_utils.upgo import tb_cross_entropy
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    g = rng(8)
    B, N = 37, 12
    t, b = (g.standard_normal((B, N)).astype(np.float32) for _ in range(2))
    a = g.integers(0, N, B)
    rho = compute_importance_weights(dev(t), dev(b), dev(a))
    assert rho.shape == (B, )
    check_close("out", host(rho), orc.importance_weights(t, b, a)["out"])
    T, B = 4, 9
    x = g.standard_normal((T * B, N)).astype(np.float32)
    lab = g.integers(0, N, (T, B))
    out = tb_cross_entropy(dev(x), dev(lab))
    assert out.shape == (T, B)
    assert np.array_equal(host(out), host(tb_cross_entropy(dev(x.reshape(T, B, N)), dev(lab))))
    check_close("out", host(out), orc.tb_cross_entropy(x, lab)["out"])


# ------------------------------------------------------------------------------------------------- composition
def test_composes_to_the_vtrace_value_loss():
    need_cuda()
    from hpc_rll.rl_utils.vtrace import VTrace, compute_importance_weights, vtrace_nstep_return
    g = rng(9)
    T, B, N = 32, 64, 18
    hp = dict(gamma=0.9, lambda_=0.8, rho_clip_ratio=1.2, c_clip_ratio=0.9, rho_pg_clip_ratio=1.5)
    t = dev((g.standard_normal((T, B, N)) * 1.5).astype(np.float32))
    b = dev((host(t) + 0.5 * g.standard_normal((T, B, N))).astype(np.float32))
    a = dev(g.integers(0, N, (T, B)))
    v, r, w = dev(g.standard_normal((T + 1, B)).astype(np.float32)), dev(g.standard_normal((T, B)).astype(
        np.float32)), dev(g.random((T, B)).astype(np.float32))
    rho = compute_importance_weights(t, b, a)
    ret = vtrace_nstep_return(rho.clamp(max=hp["rho_clip_ratio"]), rho.clamp(max=hp["c_clip_ratio"]), r, v,
                              hp["gamma"], hp["lambda_"])
    value_loss = ((v[:-1] - ret)**2 * w).mean()
    fused = VTrace(T, B, N)(t, b, a, v, r, w, **hp).value_loss
    assert rel_err(value_loss.item(), fused.item()) <= TOL


def test_composes_to_the_upgo_loss_and_gradient():
    need_cuda()
    from hpc_rll.rl_utils.upgo import UPGO, tb_cross_entropy, upgo_returns
    g = rng(10)
    T, B, N = 32, 64, 9
    tn = (g.standard_normal((T, B, N)) * 1.5).astype(np.float32)
    rho_in, a = dev(g.random((T, B)).astype(np.float32) * 2), dev(g.integers(0, N, (T, B)))
    r, v = dev(g.standard_normal((T, B)).astype(np.float32)), dev(g.standard_normal((T + 1, B)).astype(np.float32))
    t1 = dev(tn).requires_grad_(True)
    with torch.no_grad():
        adv = rho_in * (upgo_returns(r, v) - v[:-1])
    loss = -(adv * tb_cross_entropy(t1, a)).mean()
    loss.backward()
    t2 = dev(tn).requires_grad_(True)
    fused = UPGO(T, B, N)(t2, rho_in, a, r, v)
    fused.sum().backward()
    assert rel_err(loss.item(), fused.item()) <= TOL
    assert grad_err(host(t1.grad), host(t2.grad)) <= TOL


# ------------------------------------------------------------------------------------------------- other checks
@pytest.mark.parametrize("N", [16, 18, 9, 1000])
def test_run_to_run_identical(N):
    need_cuda()
    g = rng(11 + N)
    T, B = 16, 4096 if N < 1000 else 64
    t, b = (dev((g.standard_normal((T, B, N)) * 1.5).astype(np.float32)) for _ in range(2))
    a, G = dev(g.integers(0, N, (T, B))), dev(g.standard_normal((T, B)).astype(np.float32))
    x = [run_is(t, b, a, G), run_ce(t, a, G)]
    y = [run_is(t, b, a, G), run_ce(t, a, G)]
    for p, q in zip(x, y):
        assert bits(p) == bits(q)


def test_cuda_graph_replay():
    need_cuda()
    from hpc_rll.rl_utils.upgo import tb_cross_entropy
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    T, B, N = 32, 256, 18

    def inputs(seed):
        g = rng(seed)
        tn = (g.standard_normal((T, B, N)) * 1.5).astype(np.float32)
        return (tn, (tn + 0.5 * g.standard_normal((T, B, N))).astype(np.float32), g.integers(0, N, (T, B)),
                g.standard_normal((T, B)).astype(np.float32))

    t, b, a, G = (dev(x) for x in inputs(12))
    t.requires_grad_(True)
    b.requires_grad_(True)

    def step():
        rho = compute_importance_weights(t, b, a, requires_grad=True)
        rho.backward(G)
        ce = tb_cross_entropy(t, a)
        ce.backward(G)
        return rho, ce

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    t.grad = b.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        rho, ce = step()
    x1 = inputs(13)
    with torch.no_grad():
        for dst, src in zip((t, b, a, G), x1):
            dst.copy_(dev(src))
    graph.replay()
    torch.cuda.synchronize()
    tn, bn, an, Gn = x1
    want_is = run_is(dev(tn), dev(bn), dev(an), dev(Gn))
    want_ce = run_ce(dev(tn), dev(an), dev(Gn))
    assert np.array_equal(host(rho), want_is["out"]) and np.array_equal(host(ce), want_ce["out"])
    # t.grad accumulates both ops' gradients, in the same order as eagerly
    assert np.array_equal(host(t.grad), want_is["grad_target_output"] + want_ce["grad_logit"])
    assert np.array_equal(host(b.grad), want_is["grad_behaviour_output"])


def test_empty():
    need_cuda()
    from hpc_rll.rl_utils.upgo import tb_cross_entropy
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    for T, B in ((0, 5), (5, 0), (0, 0)):
        t = torch.randn(T, B, 6, device="cuda", requires_grad=True)
        b = torch.randn(T, B, 6, device="cuda", requires_grad=True)
        a = torch.zeros(T, B, dtype=torch.long, device="cuda")
        rho = compute_importance_weights(t, b, a, requires_grad=True)
        ce = tb_cross_entropy(t, a)
        assert rho.shape == ce.shape == (T, B)
        (rho.sum() + ce.sum()).backward()
        assert t.grad.shape == b.grad.shape == (T, B, 6)


def test_more_than_2_31_logits_elements():
    """One forward of each op over logits of more than 2^31 elements (about 19 GB of device memory), checked at
    sampled rows against the oracle"""
    need_cuda()
    from hpc_rll.rl_utils.upgo import tb_cross_entropy
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    N = 16
    T, B = 2, (1 << 30) // N + 4099
    R = T * B
    assert R * N > 1 << 31
    need = 2 * R * N * 4 + R * 8 + R * 4 + (1 << 30)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("needs %.1f GB of free device memory" % (need / 1e9))
    gen = torch.Generator(device="cuda").manual_seed(0)
    t = torch.randn(T, B, N, device="cuda", generator=gen)
    b = torch.randn(T, B, N, device="cuda", generator=gen)
    a = torch.randint(0, N, (T, B), device="cuda", generator=gen)
    rows = np.array([0, 1, B - 1, B, R // 2 + 3, (1 << 31) // N + 1, R - 2, R - 1])  # past 2^31 elements
    tf, bf, af = t.view(R, N), b.view(R, N), a.view(R)
    idx = torch.from_numpy(rows).cuda()
    tr, br, ar = host(tf[idx]), host(bf[idx]), host(af[idx])
    rho = compute_importance_weights(t, b, a)
    got = host(rho.view(R)[idx])
    check_close("rho", got, orc.importance_weights(tr, br, ar)["out"])
    del rho, b
    ce = tb_cross_entropy(t, a)
    check_close("ce", host(ce.view(R)[idx]), orc.tb_cross_entropy(tr, ar.reshape(-1, 1))["out"].reshape(-1))
    del t, a, ce
    torch.cuda.empty_cache()
