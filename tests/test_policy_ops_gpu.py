"""V-trace, UPGO and PPO parity on the GPU (CUDA through the C ABI) vs the oracle and the
origin-generated golden fixtures.  Tolerance: 1e-5 norm-relative (north_star) for every loss and
gradient tensor; the gradient's exact-zero structure is checked where the op defines one."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests._golden import Case, grad_err, names, rel_err
from tests._gpu import dev, host, need_cuda, rng

pytestmark = pytest.mark.gpu
TOL = 1e-5


def close(got, want, what):
    e = rel_err(got, want)
    assert e <= TOL, "%s: rel err %.3e" % (what, e)


def close_grad(got, want, what):
    """gradients: relative to their own largest entry (they carry 1/n, see tests/_golden.grad_err)"""
    e = grad_err(got, want)
    assert e <= TOL, "%s: err / max|grad| = %.3e" % (what, e)


# ----------------------------------------------------------------------------------------- vtrace
def run_vtrace(inp, hp, coef):
    from hpc_rll.rl_utils.vtrace import VTrace
    t = dev(inp["target_output"]).requires_grad_(True)
    v = dev(inp["value"]).requires_grad_(True)
    w = None if inp.get("weight") is None else dev(inp["weight"])
    T, B, N = inp["target_output"].shape
    l = VTrace(T, B, N)(t, dev(inp["behaviour_output"]), dev(inp["action"]), v, dev(inp["reward"]), w, **hp)
    assert all(x.shape == (1, ) for x in l)
    (coef[0] * l.policy_loss + coef[1] * l.value_loss + coef[2] * l.entropy_loss).sum().backward()
    torch.cuda.synchronize()
    return [float(x.item()) for x in l], host(t.grad), host(v.grad)


def vtrace_inputs(g, T, B, N, use_w):
    return dict(target_output=(g.standard_normal((T, B, N)) * 1.5).astype(np.float32),
                behaviour_output=(g.standard_normal((T, B, N)) * 1.5).astype(np.float32),
                action=g.integers(0, N, (T, B)).astype(np.int64),
                value=g.standard_normal((T + 1, B), dtype=np.float32),
                reward=g.standard_normal((T, B), dtype=np.float32),
                weight=g.random((T, B), dtype=np.float32) if use_w else None)


HP1 = dict(gamma=0.99, lambda_=0.95, rho_clip_ratio=1.0, c_clip_ratio=1.0, rho_pg_clip_ratio=1.0)
HP2 = dict(gamma=0.9, lambda_=0.8, rho_clip_ratio=1.5, c_clip_ratio=0.9, rho_pg_clip_ratio=2.0)


@pytest.mark.parametrize("T,B,N,use_w,hp", [(128, 128, 128, False, HP1), (16, 256, 16, True, HP2), (5, 7, 3, True, HP1),
                                             (1, 2, 1, False, HP1), (33, 132, 6, True, HP2), (9, 260, 40, False, HP1),
                                             (4, 64, 300, True, HP1), (12, 1024, 8, True, HP2), (6, 36, 1100, False, HP2),
                                             (50, 4100, 4, False, HP1),
                                             # staged-rows path (9 <= N <= 32, N % 4 != 0), partial last tile
                                             (7, 300, 18, True, HP2), (3, 1000, 9, False, HP1), (2, 129, 31, True, HP1),
                                             (11, 77, 13, False, HP2)])
def test_vtrace_vs_oracle(T, B, N, use_w, hp):
    need_cuda()
    inp = vtrace_inputs(rng(T * 131 + B * 7 + N), T, B, N, use_w)
    coef = [1.0, 0.5, -0.25]
    losses, gt, gv = run_vtrace(inp, hp, coef)
    o = orc.vtrace(inp["target_output"], inp["behaviour_output"], inp["action"], inp["value"], inp["reward"],
                   inp["weight"], coef=coef, **hp)
    for k, name in enumerate(("policy_loss", "value_loss", "entropy_loss")):
        close(losses[k], o[name], name)
    close_grad(gt, o["grad_target_output"], "grad_target_output")
    close_grad(gv, o["grad_value"], "grad_value")
    assert np.all(gv[-1] == 0)


@pytest.mark.parametrize("name", names("vtrace"))
def test_vtrace_vs_golden(name):
    need_cuda()
    c = Case(name)
    inp = {k: c.inp(k) for k in ("target_output", "behaviour_output", "action", "value", "reward", "weight")}
    hp = {k: c.attr(k) for k in HP1}
    coef = [c.attr("coef_policy"), c.attr("coef_value"), c.attr("coef_entropy")]
    losses, gt, gv = run_vtrace(inp, hp, coef)
    for prec in (32, 64):
        for k, nm in enumerate(("policy_loss", "value_loss", "entropy_loss")):
            close(losses[k], c.out(nm, prec), nm)
        close_grad(gt, c.grad("target_output", prec), "grad_target_output")
        close_grad(gv, c.grad("value", prec), "grad_value")


@pytest.mark.parametrize("cfg", [0, 2, 99])
def test_vtrace_scan_configs(cfg):
    need_cuda()
    from di_hpc_b200 import _abi
    inp = vtrace_inputs(rng(cfg + 50), 21, 520, 8, True)
    upgo_inp = dict(target_output=inp["target_output"], rhos=2 * inp["weight"], action=inp["action"],
                    rewards=inp["reward"], bootstrap_values=inp["value"])
    coef = [1.0, 1.0, 1.0]
    runs = {}
    try:
        for c in (cfg, 99):
            _abi.set_config(_abi.OP_VTRACE, c)
            _abi.set_config(_abi.OP_UPGO, c)
            runs[c] = run_vtrace(inp, HP2, coef), run_upgo(upgo_inp, -0.7)
    finally:
        _abi.set_config(_abi.OP_VTRACE, -1)
        _abi.set_config(_abi.OP_UPGO, -1)
    (losses, gt, gv), (upgo_loss, upgo_gt) = runs[cfg]
    o = orc.vtrace(inp["target_output"], inp["behaviour_output"], inp["action"], inp["value"], inp["reward"],
                   inp["weight"], coef=coef, **HP2)
    close(losses[0], o["policy_loss"], "pg")
    close(losses[1], o["value_loss"], "v")
    close_grad(gt, o["grad_target_output"], "gt")
    close_grad(gv, o["grad_value"], "gv")
    ou = orc.upgo(upgo_inp["target_output"], upgo_inp["rhos"], upgo_inp["action"], upgo_inp["rewards"],
                  upgo_inp["bootstrap_values"], -0.7)
    close(upgo_loss, ou["loss"], "upgo loss")
    close_grad(upgo_gt, ou["grad_target_output"], "upgo gt")
    # the column scan and the generic kernel drive the same bodies: per-element gradients agree bit for bit (losses
    # are summed per CTA, and CTA sizes differ between the two)
    (_, gt99, gv99), (_, upgo_gt99) = runs[99]
    assert np.array_equal(gt, gt99) and np.array_equal(gv, gv99) and np.array_equal(upgo_gt, upgo_gt99)


# ----------------------------------------------------------------------------------------- upgo
def run_upgo(inp, coef):
    from hpc_rll.rl_utils.upgo import UPGO
    t = dev(inp["target_output"]).requires_grad_(True)
    T, B, N = inp["target_output"].shape
    loss = UPGO(T, B, N)(t, dev(inp["rhos"]), dev(inp["action"]), dev(inp["rewards"]), dev(inp["bootstrap_values"]))
    assert loss.shape == (1, )
    (coef * loss).sum().backward()
    torch.cuda.synchronize()
    return float(loss.item()), host(t.grad)


@pytest.mark.parametrize("T,B,N", [(256, 256, 256), (16, 256, 16), (5, 7, 3), (1, 4, 3), (2, 4, 16), (33, 132, 6),
                                   (20, 3, 33), (8, 1024, 8), (3, 40, 1100), (40, 4100, 4), (7, 300, 18), (3, 1000, 9),
                                   (2, 129, 31), (11, 77, 13)])
def test_upgo_vs_oracle(T, B, N):
    need_cuda()
    g = rng(T * 17 + B * 3 + N)
    inp = dict(target_output=(g.standard_normal((T, B, N)) * 1.5).astype(np.float32),
               rhos=(g.random((T, B)) * 2).astype(np.float32), action=g.integers(0, N, (T, B)).astype(np.int64),
               rewards=g.standard_normal((T, B), dtype=np.float32),
               bootstrap_values=g.standard_normal((T + 1, B), dtype=np.float32))
    loss, gt = run_upgo(inp, -0.7)
    o = orc.upgo(inp["target_output"], inp["rhos"], inp["action"], inp["rewards"], inp["bootstrap_values"], -0.7)
    close(loss, o["loss"], "loss")
    close_grad(gt, o["grad_target_output"], "grad_target_output")


@pytest.mark.parametrize("name", names("upgo"))
def test_upgo_vs_golden(name):
    need_cuda()
    c = Case(name)
    inp = {k: c.inp(k) for k in ("target_output", "rhos", "action", "rewards", "bootstrap_values")}
    loss, gt = run_upgo(inp, c.attr("coef_loss"))
    for prec in (32, 64):
        close(loss, c.out("loss", prec), "loss")
        close_grad(gt, c.grad("target_output", prec), "grad_target_output")


# ----------------------------------------------------------------------------------------- ppo
def run_ppo(inp, clip_ratio, use_value_clip, dual_clip, coef):
    from hpc_rll.rl_utils.ppo import PPO
    ln = dev(inp["logits_new"]).requires_grad_(True)
    vn = dev(inp["value_new"]).requires_grad_(True)
    w = None if inp.get("weight") is None else dev(inp["weight"])
    B, N = inp["logits_new"].shape
    loss, info = PPO(B, N)(ln, dev(inp["logits_old"]), dev(inp["action"]), vn, dev(inp["value_old"]), dev(inp["adv"]),
                           dev(inp["return_"]), w, clip_ratio, use_value_clip, dual_clip)
    assert isinstance(info.approx_kl, float) and isinstance(info.clipfrac, float)
    (coef[0] * loss.policy_loss + coef[1] * loss.value_loss + coef[2] * loss.entropy_loss).sum().backward()
    torch.cuda.synchronize()
    return [float(x.item()) for x in loss] + [info.approx_kl, info.clipfrac], host(ln.grad), host(vn.grad)


def ppo_inputs(g, B, N, use_w):
    lo = g.standard_normal((B, N)).astype(np.float32)
    return dict(logits_new=(lo + 0.3 * g.standard_normal((B, N))).astype(np.float32), logits_old=lo,
                action=g.integers(0, N, (B, )).astype(np.int64), value_new=g.standard_normal(B).astype(np.float32),
                value_old=g.standard_normal(B).astype(np.float32), adv=g.standard_normal(B).astype(np.float32),
                return_=g.standard_normal(B).astype(np.float32),
                weight=g.random(B).astype(np.float32) if use_w else None)


@pytest.mark.parametrize("B,N,use_w,clip,vclip,dual", [(128, 128, False, 0.2, True, None), (4096, 6, True, 0.2, True, 3.0),
                                                         (17, 16, True, 0.1, False, None), (5, 1, False, 0.2, True, 2.0),
                                                         (1000, 37, False, 0.3, False, 1.5), (300, 260, True, 0.2, True, None),
                                                         (64, 1100, True, 0.2, True, 5.0), (70000, 8, True, 0.2, True, None),
                                                         (3000, 18, True, 0.2, True, None), (257, 9, False, 0.2, False, 2.0),
                                                         (1000, 31, True, 0.1, True, None)])
def test_ppo_vs_oracle(B, N, use_w, clip, vclip, dual):
    need_cuda()
    inp = ppo_inputs(rng(B * 13 + N), B, N, use_w)
    coef = [1.0, 0.5, -0.01]
    outs, gl, gv = run_ppo(inp, clip, vclip, dual, coef)
    o = orc.ppo(inp["logits_new"], inp["logits_old"], inp["action"], inp["value_new"], inp["value_old"], inp["adv"],
                inp["return_"], inp["weight"], clip, vclip, dual, coef)
    for k, nm in enumerate(("policy_loss", "value_loss", "entropy_loss", "approx_kl", "clipfrac")):
        close(outs[k], o[nm], nm)
    close_grad(gl, o["grad_logits_new"], "grad_logits_new")
    close_grad(gv, o["grad_value_new"], "grad_value_new")


@pytest.mark.parametrize("name", names("ppo"))
def test_ppo_vs_golden(name):
    need_cuda()
    c = Case(name)
    inp = {k: c.inp(k) for k in ("logits_new", "logits_old", "action", "value_new", "value_old", "adv", "return_",
                                 "weight")}
    coef = [c.attr("coef_policy"), c.attr("coef_value"), c.attr("coef_entropy")]
    outs, gl, gv = run_ppo(inp, c.attr("clip_ratio"), bool(c.attr("use_value_clip")), c.attr("dual_clip"), coef)
    for prec in (32, 64):
        for k, nm in enumerate(("policy_loss", "value_loss", "entropy_loss")):
            close(outs[k], c.out(nm, prec), nm)
        close_grad(gl, c.grad("logits_new", prec), "grad_logits_new")
        close_grad(gv, c.grad("value_new", prec), "grad_value_new")
    close(outs[3], c.out("approx_kl", 32), "approx_kl")
    close(outs[4], c.out("clipfrac", 32), "clipfrac")


def test_ppo_dual_clip_must_exceed_one():
    need_cuda()
    from hpc_rll.rl_utils.ppo import PPO
    inp = ppo_inputs(rng(1), 8, 4, False)
    with pytest.raises(AssertionError):
        PPO(8, 4)(*[dev(inp[k]) for k in ("logits_new", "logits_old", "action", "value_new", "value_old", "adv",
                                          "return_")], None, 0.2, True, 0.5)


def test_masked_actions_with_minus_inf_logits():
    """Illegal-action masking puts -inf into logits.  The row statistics must stay finite (the same guard
    torch.distributions.Categorical applies, clamping to finfo.min) and equal the result of simply removing
    the masked action: compare an N-action problem with one -inf column against the (N-1)-action oracle."""
    need_cuda()
    g = rng(77)
    T, B, N = 6, 40, 9
    inp = vtrace_inputs(g, T, B, N - 1, True)
    coef = [1.0, 0.5, -0.25]
    o = orc.vtrace(inp["target_output"], inp["behaviour_output"], inp["action"], inp["value"], inp["reward"],
                   inp["weight"], coef=coef, **HP2)
    k = 4  # masked column inserted at index k; actions >= k shift by one
    big = dict(inp)
    for name in ("target_output", "behaviour_output"):
        big[name] = np.insert(inp[name], k, -np.inf, axis=2).astype(np.float32)
    big["action"] = np.where(inp["action"] >= k, inp["action"] + 1, inp["action"]).astype(np.int64)
    losses, gt, gv = run_vtrace(big, HP2, coef)
    assert np.all(np.isfinite(losses)) and np.all(np.isfinite(gt)) and np.all(np.isfinite(gv))
    for i, name in enumerate(("policy_loss", "value_loss", "entropy_loss")):
        close(losses[i], o[name], name)
    assert np.all(gt[:, :, k] == 0)
    close(np.delete(gt, k, axis=2), o["grad_target_output"], "grad_target_output")
    close_grad(gv, o["grad_value"], "grad_value")


# ----------------------------------------------------------------------------------------- row geometry sweep
SWEEP_N = list(range(1, 41)) + [44, 48, 52, 60, 66, 100, 132, 250, 255, 257]


@pytest.mark.parametrize("N", SWEEP_N)
def test_row_geometry_sweep(N):
    """Every (chunk width, lanes per row, chunks per lane) combination `row_geom` can pick -- 128-bit / 64-bit /
    scalar chunks with 1..8 chunks per lane, staged rows for odd 9 <= N <= 31, the looping kernel beyond -- on all
    three ops that share the row machinery, ragged row counts included."""
    need_cuda()
    g = rng(1000 + N)
    T, B = 3, 45
    inp = vtrace_inputs(g, T, B, N, True)
    coef = [1.0, 0.5, -0.25]
    losses, gt, gv = run_vtrace(inp, HP2, coef)
    o = orc.vtrace(inp["target_output"], inp["behaviour_output"], inp["action"], inp["value"], inp["reward"],
                   inp["weight"], coef=coef, **HP2)
    for i, name in enumerate(("policy_loss", "value_loss", "entropy_loss")):
        close(losses[i], o[name], "vtrace " + name)
    close_grad(gt, o["grad_target_output"], "vtrace grad_target_output")
    close_grad(gv, o["grad_value"], "vtrace grad_value")

    up = dict(target_output=inp["target_output"], rhos=(g.random((T, B)) * 2).astype(np.float32), action=inp["action"],
              rewards=inp["reward"], bootstrap_values=inp["value"])
    loss, gt = run_upgo(up, -0.7)
    o = orc.upgo(up["target_output"], up["rhos"], up["action"], up["rewards"], up["bootstrap_values"], -0.7)
    close(loss, o["loss"], "upgo loss")
    close_grad(gt, o["grad_target_output"], "upgo grad_target_output")

    pp = ppo_inputs(g, 131, N, True)
    c3 = [1.0, 0.5, -0.01]
    outs, gl, gvn = run_ppo(pp, 0.2, True, None, c3)
    o = orc.ppo(pp["logits_new"], pp["logits_old"], pp["action"], pp["value_new"], pp["value_old"], pp["adv"],
                pp["return_"], pp["weight"], 0.2, True, None, c3)
    for k, nm in enumerate(("policy_loss", "value_loss", "entropy_loss", "approx_kl")):
        close(outs[k], o[nm], "ppo " + nm)
    assert abs(outs[4] - o["clipfrac"]) <= 2.0 / 131 + 1e-6
    close_grad(gl, o["grad_logits_new"], "ppo grad_logits_new")
    close_grad(gvn, o["grad_value_new"], "ppo grad_value_new")


@pytest.mark.parametrize("T,B,N,use_w", [(1024, 64, 6, True), (100, 33, 16, False), (64, 4096, 4, True), (517, 130, 9, True)])
def test_small_batch_tsplit_agrees_with_column_scan(T, B, N, use_w):
    """V-trace / UPGO scans: the single-launch T-split with look-back (config 21, automatic for B <= 4096) against the
    column-scan kernels (config 2) and the oracle on the same inputs; data-dependent coefficients (gamma*lambda*c_t,
    the 0/1 UPGO flag) are multiplied up across segments.  Also run-to-run bit reproducibility of the T-split."""
    need_cuda()
    from di_hpc_b200 import _abi
    g = rng(T + 31 * B + N)
    inp = vtrace_inputs(g, T, B, N, use_w)
    coef = [1.0, 0.5, -0.25]
    up = dict(target_output=inp["target_output"], rhos=(g.random((T, B)) * 2).astype(np.float32), action=inp["action"],
              rewards=inp["reward"], bootstrap_values=inp["value"])
    res = {}
    try:
        for cfg in (21, 2, 21):
            _abi.set_config(_abi.OP_VTRACE, cfg)
            _abi.set_config(_abi.OP_UPGO, cfg)
            res.setdefault(cfg, []).append((run_vtrace(inp, HP2, coef), run_upgo(up, -0.7)))
    finally:
        _abi.set_config(_abi.OP_VTRACE, -1)
        _abi.set_config(_abi.OP_UPGO, -1)
    o = orc.vtrace(inp["target_output"], inp["behaviour_output"], inp["action"], inp["value"], inp["reward"],
                   inp["weight"], coef=coef, **HP2)
    ou = orc.upgo(up["target_output"], up["rhos"], up["action"], up["rewards"], up["bootstrap_values"], -0.7)
    for cfg in (21, 2):
        (losses, gt, gv), (ul, ugt) = res[cfg][0]
        for i, name in enumerate(("policy_loss", "value_loss", "entropy_loss")):
            close(losses[i], o[name], "cfg %d vtrace %s" % (cfg, name))
        close_grad(gt, o["grad_target_output"], "cfg %d vtrace grad_target_output" % cfg)
        close_grad(gv, o["grad_value"], "cfg %d vtrace grad_value" % cfg)
        close(ul, ou["loss"], "cfg %d upgo loss" % cfg)
        close_grad(ugt, ou["grad_target_output"], "cfg %d upgo grad" % cfg)
    a, b = res[21]
    assert a[0][0] == b[0][0] and np.array_equal(a[0][1], b[0][1]) and np.array_equal(a[0][2], b[0][2])
    assert a[1][0] == b[1][0] and np.array_equal(a[1][1], b[1][1])
    # UPGO's coefficient is 0/1: composing segments is exact, the T-split must give the column scan's bits
    assert np.array_equal(res[21][0][1][1], res[2][0][1][1])


def test_ppo_lazy_info_matches_eager_floats():
    """PPO.lazy_info: approx_kl / clipfrac as LazyScalars (8-byte D2H copy queued next to an event, host waits only when the
    value is read) must equal the reference-style Python floats of the default mode."""
    need_cuda()
    from hpc_rll.rl_utils.ppo import PPO, LazyScalar
    inp = ppo_inputs(rng(5), 777, 6, True)
    args = [dev(inp[k]) for k in ("logits_new", "logits_old", "action", "value_new", "value_old", "adv", "return_", "weight")]
    eager = PPO(777, 6)
    lazy = PPO(777, 6)
    lazy.lazy_info = True
    _, info_e = eager(*args, 0.2, True, None)
    loss_l, info_l = lazy(*args, 0.2, True, None)
    assert isinstance(info_e.approx_kl, float) and isinstance(info_l.approx_kl, LazyScalar)
    assert float(info_l.approx_kl) == info_e.approx_kl and float(info_l.clipfrac) == info_e.clipfrac
    assert info_l.clipfrac.ready() and (info_l.clipfrac + 1.0) == info_e.clipfrac + 1.0 and info_l.approx_kl < 10.0
    assert "%.4f" % info_l.approx_kl == "%.4f" % info_e.approx_kl
