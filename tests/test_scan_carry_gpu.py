"""The scan carries of GAE, TD(lambda), V-trace, UPGO and episodic GAE on the GPU, in every kernel regime, with the
probes of tests/scan_probes.py (certified by tests/test_scan_carry_cpu.py).

Each op runs through its C ABI forward (and backward, for the two GAE ops) with a forced tuning config and with the
automatic dispatch.  The outputs compared are what the scan kernels write: advantages and adjoints for the GAE ops, and
the per-element buffers that V-trace, UPGO and TD(lambda) save for their backward (-(adv*w)/n, 2(v-ret)w/n, -adv/n,
-w(ret-v)/n).  The backward kernels of those three only scale these buffers.

- exact probes (coefficient exactly 1 or 0, small integers): every regime, the look-back T-split included, equals the
  fp32 oracle bit for bit.  The look-back path re-associates the recurrence, but it cannot change an exact result.
- undamped random data (coefficient 1): no regime is further from the fp64 oracle than 4x the serial fp32 oracle's
  own error plus 8 fp32 ulps of the output's scale.
- the losses: within 2 fp32 ulps of the oracle on exact probes, and within the same bound on random data.
- the regime the config asks for actually ran, read from the random probe's bits: a column scan reproduces the serial
  fp32 oracle exactly, and the look-back path (three or more segments) cannot.  Kernel names from torch.profiler were
  not used because sessions on a busy run now and then come back empty."""
import functools

import numpy as np
import pytest
import torch

from tests import scan_probes as sp
from tests._gpu import dev, host, need_cuda

pytestmark = pytest.mark.gpu

EPS32 = float(np.finfo(np.float32).eps)

class forced:
    def __init__(self, op, cfg):
        self.op, self.cfg = sp.OP_ID[op], cfg

    def __enter__(self):
        from di_hpc_b200 import _abi
        _abi.set_config(self.op, self.cfg)

    def __exit__(self, *exc):
        from di_hpc_b200 import _abi
        _abi.set_config(self.op, -1)
        return False


# ------------------------------------------------------------------------------------------------ runners (C ABI)
def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")  # an element no kernel writes stays NaN


def _opt(x):
    return None if x is None else dev(x)


def run(p):
    """-> (outputs keyed like scan_probes.reference's `out`, losses)"""
    from di_hpc_b200 import _abi
    L = _abi.lib()
    st = torch.cuda.current_stream().cuda_stream
    x, hp, T, B = p.inputs, p.params, p.T, p.B
    ptr = _abi.ptr
    if p.op == "gae":
        from di_hpc_b200.rl_utils.gae import gae_with_adv_stats
        v, r, ga = dev(x["value"]), dev(x["reward"]), dev(x["grad_adv"])
        adv, gv, gr = _nan(T, B), _nan(T + 1, B), _nan(T, B)
        _abi.check(L.hpc_rll_gae_forward(ptr(v), ptr(r), ptr(adv), T, B, hp["gamma"], hp["lambda_"], st), "gae fwd")
        _abi.check(L.hpc_rll_gae_backward(ptr(ga), ptr(gv), ptr(gr), T, B, hp["gamma"], hp["lambda_"], st), "gae bwd")
        adv_m, _ = gae_with_adv_stats(v, r, hp["gamma"], hp["lambda_"])
        return dict(adv=host(adv), grad_value=host(gv), grad_reward=host(gr), adv_moments=host(adv_m)), {}
    if p.op == "td_lambda":
        v, r, w = dev(x["value"]), dev(x["reward"]), _opt(x["weight"])
        loss, gbuf = _nan(1), _nan(T, B)
        ws = _abi.workspace(_abi.OP_TD_LAMBDA, T, B, 0, "cuda")
        _abi.check(L.hpc_rll_td_lambda_forward(ptr(v), ptr(r), ptr(w), ptr(loss), ptr(gbuf), T, B, hp["gamma"],
                                               hp["lambda_"], 0, ptr(ws), ws.numel(), st), "td_lambda fwd")
        return dict(grad_buf=host(gbuf)), dict(loss=float(loss.item()))
    if p.op == "vtrace":
        N = x["target_output"].shape[2]
        t, bo, a = dev(x["target_output"]), dev(x["behaviour_output"]), dev(x["action"])
        v, r, w = dev(x["value"]), dev(x["reward"]), _opt(x["weight"])
        losses, pg, gvb = _nan(3), _nan(T, B), _nan(T, B)
        ws = _abi.workspace(_abi.OP_VTRACE, T, B, N, "cuda")
        _abi.check(L.hpc_rll_vtrace_forward(ptr(t), ptr(bo), ptr(a), ptr(v), ptr(r), ptr(w), ptr(losses), ptr(pg),
                                            ptr(gvb), T, B, N, hp["gamma"], hp["lambda_"], hp["rho_clip_ratio"],
                                            hp["c_clip_ratio"], hp["rho_pg_clip_ratio"], 0, ptr(ws), ws.numel(), st),
                   "vtrace fwd")
        lv = host(losses)
        return dict(pg_coef=host(pg), gv_buf=host(gvb)), dict(policy_loss=float(lv[0]), value_loss=float(lv[1]),
                                                              entropy_loss=float(lv[2]))
    if p.op == "upgo":
        N = x["target_output"].shape[2]
        t, rho, a = dev(x["target_output"]), dev(x["rhos"]), dev(x["action"])
        r, bv = dev(x["rewards"]), dev(x["bootstrap_values"])
        loss, coef = _nan(1), _nan(T, B)
        ws = _abi.workspace(_abi.OP_UPGO, T, B, N, "cuda")
        _abi.check(L.hpc_rll_upgo_forward(ptr(t), ptr(rho), ptr(a), ptr(r), ptr(bv), ptr(loss), ptr(coef), T, B, N,
                                          0, ptr(ws), ws.numel(), st), "upgo fwd")
        return dict(coef=host(coef)), dict(loss=float(loss.item()))
    if p.op == "gae_episodic":
        v, nv, r, ga = (dev(x[k]) for k in ("value", "next_value", "reward", "grad_adv"))
        d, tr = dev(x["done"].astype(np.uint8)), dev(x["traj_flag"].astype(np.uint8))
        adv, gv, gnv, gr = _nan(T, B), _nan(T, B), _nan(T, B), _nan(T, B)
        _abi.check(L.hpc_rll_gae_episodic_forward(ptr(v), ptr(nv), ptr(r), ptr(d), ptr(tr), ptr(adv), T, B,
                                                  hp["gamma"], hp["lambda_"], st), "episodic fwd")
        _abi.check(L.hpc_rll_gae_episodic_backward(ptr(ga), ptr(d), ptr(tr), ptr(gv), ptr(gnv), ptr(gr), T, B,
                                                   hp["gamma"], hp["lambda_"], st), "episodic bwd")
        return dict(adv=host(adv), grad_value=host(gv), grad_next_value=host(gnv), grad_reward=host(gr)), {}
    raise ValueError(p.op)


# ------------------------------------------------------------------------------------------------ checks
@functools.lru_cache(maxsize=8)
def probe_and_refs(op, family, T, B):
    p = sp.make_probe(op, family, T, B)
    return p, sp.reference(p, np.float32), sp.reference(p, np.float64)


def where(p, cfg, name, t, b):
    g = sp.lb_geom(p.T, p.B, cfg)
    seg = "segment %d of %d (L=%d, t - segment start = %d)" % (t // g.L, g.S, g.L, t % g.L) if g.split else \
        "column scan"
    return "%s cfg=%d (T=%d, B=%d) %s probe, %s first wrong at (t=%d, b=%d), %s; column %d's %s rows: %s" % (
        p.op, cfg, p.T, p.B, p.family, name, t, b, seg, b, "break" if p.family == "break" else "impulse",
        p.marks[b] if p.marks[b] else "none")


def check_exact(p, cfg, got, want):
    for name, w in want.items():
        gk = got[name]
        assert gk.shape == w.shape, (name, gk.shape, w.shape)
        bad = np.argwhere(~(gk == w))
        if bad.size:
            t, b = (int(i) for i in bad[0])
            pytest.fail("%s: kernel %r, fp32 oracle %r; %d of %d elements differ" % (
                where(p, cfg, name, t, b), gk[t, b], w[t, b], len(bad), w.size))


def check_bound(p, cfg, got, o32, o64):
    for name, w64 in o64.items():
        gk = got[name].astype(np.float64)
        assert np.all(np.isfinite(gk)), where(p, cfg, name, *np.argwhere(~np.isfinite(gk))[0])
        serial = float(np.max(np.abs(o32[name].astype(np.float64) - w64)))
        bound = 4.0 * serial + 8.0 * EPS32 * float(np.max(np.abs(w64)))
        err = np.abs(gk - w64)
        if float(err.max()) > bound:
            t, b = (int(i) for i in np.unravel_index(np.argmax(err), err.shape))
            pytest.fail("%s: |kernel - fp64| = %.3g > bound %.3g (serial fp32 oracle %.3g)" % (
                where(p, cfg, name, t, b), float(err.max()), bound, serial))


def check_losses(p, cfg, got, l32, l64, o64):
    # a policy loss sums terms of both signs in fp64, in an order that differs between the kernels and the oracle's
    # OpenMP reduction: when it cancels, the order shows at ~1e-16 of the largest term (|log p| * max|adv|)
    floor = 1e-12 * max(1.0, max(float(np.max(np.abs(o))) for o in o64.values()) * p.T * p.B)
    for name, k in got.items():
        if p.exact:
            ok = abs(k - l32[name]) <= 2.0 * EPS32 * abs(l32[name]) + floor
        else:
            ok = abs(k - l64[name]) <= 4.0 * abs(l32[name] - l64[name]) + 8.0 * EPS32 * abs(l64[name]) + floor
        assert ok, "%s cfg=%d (T=%d, B=%d) %s probe: %s = %r, oracle fp32 %r, fp64 %r" % (
            p.op, cfg, p.T, p.B, p.family, name, k, l32[name], l64[name])


CASES = sorted({(op, T, B, cfg) for op in sp.OPS for cfg in (-1,) + sp.CONFIGS[op] for T, B in sp.shapes_for(cfg)},
               key=lambda c: (sp.OPS.index(c[0]), c[1] * c[2], c[1], c[3]))


@pytest.mark.parametrize("op,T,B,cfg", CASES, ids=["%s-T%d-B%d-cfg%d" % c for c in CASES])
def test_scan_carry(op, T, B, cfg):
    need_cuda()
    geom = sp.lb_geom(T, B, cfg)
    for family in sp.FAMILIES[op]:
        p, (_, o32, l32), (_, o64, l64) = probe_and_refs(op, family, T, B)
        with forced(op, cfg):
            got, losses = run(p)
        if family == "random":  # which regime ran, read from the bits of the random probe
            serial = all(np.array_equal(got[k], o32[k]) for k in o32)
            if geom.split and geom.S >= 3:
                # segments past the second fold their carry by one fused multiply-add per predecessor, which rounds
                # differently from the serial chain somewhere in a random column: bit-identical results mean the
                # look-back kernel did not run
                assert not serial, "%s cfg=%d (T=%d, B=%d): results bit-identical to the serial scan; the look-back " \
                    "path did not run" % (op, cfg, T, B)
            elif not geom.split:
                assert serial, "%s cfg=%d (T=%d, B=%d): a column scan must reproduce the serial fp32 oracle bit for " \
                    "bit" % (op, cfg, T, B)
        if op == "gae":  # gae_with_adv_stats runs its own forward kernels (never the look-back one)
            moments = dict(adv=got.pop("adv_moments"))
            if p.exact:
                check_exact(p, cfg, moments, dict(adv=o32["adv"]))
            else:
                check_bound(p, cfg, moments, dict(adv=o32["adv"]), dict(adv=o64["adv"]))
        if p.exact:
            check_exact(p, cfg, got, o32)
        else:
            check_bound(p, cfg, got, o32, o64)
        check_losses(p, cfg, losses, l32, l64, o64)


@pytest.mark.parametrize("family", ["impulse", "zero", "random"])
@pytest.mark.parametrize("T,B,rows", [(1025, 64, 32), (2049, 36, 40), (4100, 33, 72), (1025, 64, 33)])
def test_gae_chunk_abi_carries(T, B, rows, family):
    """hpc_rll_gae_forward_chunk / _backward_chunk cut at the look-back segment length, so every chunk edge sits on
    impulse rows (rows = 33 puts the edges at odd rows: the generic kernel).  Chunks carry the serial state, so even
    the random probe is bit-exact against the fp32 oracle."""
    need_cuda()
    from di_hpc_b200 import _abi
    p, (_, o32, _), _ = probe_and_refs("gae", family, T, B)
    L = _abi.lib()
    st = torch.cuda.current_stream().cuda_stream
    gm, lm = p.params["gamma"], p.params["lambda_"]
    v, r, ga = dev(p.inputs["value"]), dev(p.inputs["reward"]), dev(p.inputs["grad_adv"])
    adv, gv, gr = _nan(T, B), _nan(T + 1, B), _nan(T, B)
    nC = (T + rows - 1) // rows
    cf = torch.zeros(2, B, device="cuda")
    cf[1] = v[T]
    for k in reversed(range(nC)):
        t0, n = k * rows, min(rows, T - k * rows)
        _abi.check(L.hpc_rll_gae_forward_chunk(v[t0].data_ptr(), r[t0].data_ptr(), adv[t0].data_ptr(), cf.data_ptr(),
                                               T, t0, n, B, gm, lm, st), "fwd_chunk")
    cb = torch.zeros(2, B, device="cuda")
    for k in range(nC):
        t0, n = k * rows, min(rows, T - k * rows)
        _abi.check(L.hpc_rll_gae_backward_chunk(ga[t0].data_ptr(), gv[t0].data_ptr(), gr[t0].data_ptr(),
                                                cb.data_ptr(), T, t0, n, B, gm, lm, st), "bwd_chunk")
    torch.cuda.synchronize()
    check_exact(p, -1, dict(adv=host(adv), grad_value=host(gv), grad_reward=host(gr)), o32)
