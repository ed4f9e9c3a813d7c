"""n-step TD-error family parity on the GPU vs the oracle and origin-generated golden fixtures.
Values: 1e-5 norm-relative.  Integer paths: the gradient's zero pattern (which (b, action) slot
receives gradient) must match the oracle EXACTLY."""
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


def same_zero_pattern(got, want):
    assert np.array_equal(got != 0, want != 0), "gradient zero pattern (action gather) differs"


def base_inputs(g, T, B, N, use_w):
    return dict(action=g.integers(0, N, (B, )).astype(np.int64), next_n_action=g.integers(0, N, (B, )).astype(np.int64),
                reward=g.standard_normal((T, B), dtype=np.float32), done=(g.random(B) < 0.3).astype(np.float32),
                weight=g.random(B).astype(np.float32) if use_w else None)


# ----------------------------------------------------------------------------------------- q n-step
def run_q(inp, gamma, rescale, coef):
    from hpc_rll.rl_utils.td import QNStepTD, QNStepTDRescale
    q = dev(inp["q"]).requires_grad_(True)
    T, B = inp["reward"].shape
    N = inp["q"].shape[1]
    cls = QNStepTDRescale if rescale else QNStepTD
    w = None if inp["weight"] is None else dev(inp["weight"])
    loss, td = cls(T, B, N)(q, dev(inp["next_n_q"]), dev(inp["action"]), dev(inp["next_n_action"]),
                            dev(inp["reward"]), dev(inp["done"]), w, gamma)
    assert loss.shape == (1, ) and td.shape == (B, )
    (coef * loss).sum().backward()
    torch.cuda.synchronize()
    return float(loss.item()), host(td), host(q.grad)


@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("T,B,N,use_w", [(1024, 64, 64, False), (5, 4096, 6, True), (1, 7, 3, True), (30, 4, 1, True),
                                          (3, 70001, 18, True), (5, 1000, 7, False), (2, 9, 2048, False)])
def test_q_nstep_vs_oracle(T, B, N, use_w, rescale):
    need_cuda()
    g = rng(T + B + N + int(rescale))
    inp = base_inputs(g, T, B, N, use_w)
    sc = 3.0 if rescale else 1.0
    inp["q"] = (g.standard_normal((B, N)) * sc).astype(np.float32)
    inp["next_n_q"] = (g.standard_normal((B, N)) * sc).astype(np.float32)
    loss, td, gq = run_q(inp, 0.95, rescale, 1.3)
    o = orc.q_nstep_td(inp["q"], inp["next_n_q"], inp["action"], inp["next_n_action"], inp["reward"], inp["done"],
                       inp["weight"], 0.95, rescale, 1.3)
    close(loss, o["loss"], "loss")
    close(td, o["td_error_per_sample"], "td")
    close_grad(gq, o["grad_q"], "grad_q")
    same_zero_pattern(gq, o["grad_q"])


@pytest.mark.parametrize("name", names("qnstep"))
def test_q_nstep_vs_golden(name):
    need_cuda()
    c = Case(name)
    inp = {k: c.inp(k) for k in ("q", "next_n_q", "action", "next_n_action", "reward", "done", "weight")}
    loss, td, gq = run_q(inp, c.attr("gamma"), "rescale" in name, c.attr("coef_loss"))
    for prec in (32, 64):
        close(loss, c.out("loss", prec), "loss")
        close(td, c.out("td_error_per_sample", prec), "td")
        close_grad(gq, c.grad("q", prec), "grad_q")
    same_zero_pattern(gq, c.grad("q", 32))


# ----------------------------------------------------------------------------------------- C51
def run_dist(inp, gamma, v_min, v_max, coef):
    from hpc_rll.rl_utils.td import DistNStepTD
    d = dev(inp["dist"]).requires_grad_(True)
    T, B = inp["reward"].shape
    _, N, n_atom = inp["dist"].shape
    w = None if inp["weight"] is None else dev(inp["weight"])
    loss, td = DistNStepTD(T, B, N, n_atom)(d, dev(inp["next_n_dist"]), dev(inp["action"]), dev(inp["next_n_action"]),
                                           dev(inp["reward"]), dev(inp["done"]), w, gamma, v_min, v_max)
    (coef * loss).sum().backward()
    torch.cuda.synchronize()
    return float(loss.item()), host(td), host(d.grad)


def softmax(x):
    e = np.exp(x - x.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32)


# n_atom 1536: exactly 48 KB of dynamic shared memory, over the limit with the warp kernel's static shared memory
@pytest.mark.parametrize("T,B,N,n_atom,use_w,vr", [(128, 128, 128, 51, False, (-10.0, 10.0)), (5, 1000, 4, 51, True, (-10.0, 10.0)),
                                                    (3, 6, 3, 21, True, (-5.0, 5.0)), (1, 4, 2, 5, True, (0.0, 4.0)),
                                                    (2, 300, 2, 200, False, (-1.0, 3.0)), (4, 33, 5, 2, True, (-2.0, 2.0)),
                                                    (3, 9, 2, 1536, True, (-10.0, 10.0))])
def test_dist_nstep_vs_oracle(T, B, N, n_atom, use_w, vr):
    need_cuda()
    g = rng(T + B + N + n_atom)
    inp = base_inputs(g, T, B, N, use_w)
    inp["reward"] = (inp["reward"] * 2).astype(np.float32)
    inp["dist"] = softmax(g.standard_normal((B, N, n_atom)))
    inp["next_n_dist"] = softmax(g.standard_normal((B, N, n_atom)))
    loss, td, gd = run_dist(inp, 0.95, vr[0], vr[1], 0.9)
    o = orc.dist_nstep_td(inp["dist"], inp["next_n_dist"], inp["action"], inp["next_n_action"], inp["reward"],
                          inp["done"], inp["weight"], 0.95, vr[0], vr[1], 0.9)
    close(loss, o["loss"], "loss")
    close(td, o["td_error_per_sample"], "td")
    close_grad(gd, o["grad_dist"], "grad_dist")
    # rows of non-selected actions are exactly zero
    mask = np.ones((B, N), dtype=bool)
    mask[np.arange(B), inp["action"]] = False
    assert np.all(gd[mask] == 0)


@pytest.mark.parametrize("name", names("dist"))
def test_dist_nstep_vs_golden(name):
    need_cuda()
    c = Case(name)
    inp = {k: c.inp(k) for k in ("dist", "next_n_dist", "action", "next_n_action", "reward", "done", "weight")}
    loss, td, gd = run_dist(inp, c.attr("gamma"), c.attr("v_min"), c.attr("v_max"), c.attr("coef_loss"))
    for prec in (32, 64):
        close(loss, c.out("loss", prec), "loss")
        close(td, c.out("td_error_per_sample", prec), "td")
        close_grad(gd, c.grad("dist", prec), "grad_dist")


# ----------------------------------------------------------------------------------------- QR-DQN
def run_qrdqn(inp, gamma, coef):
    from hpc_rll.rl_utils.td import QRDQNNStepTDError
    q = dev(inp["q"]).requires_grad_(True)
    T, B = inp["reward"].shape
    _, N, tau = inp["q"].shape
    w = None if inp["weight"] is None else dev(inp["weight"])
    vg = None if inp.get("value_gamma") is None else dev(inp["value_gamma"])
    loss, td = QRDQNNStepTDError(tau, T, B, N)(q, dev(inp["next_n_q"]), dev(inp["action"]), dev(inp["next_n_action"]),
                                               dev(inp["reward"]), dev(inp["done"]), gamma, w, vg)
    (coef * loss).sum().backward()
    torch.cuda.synchronize()
    return float(loss.item()), host(td), host(q.grad)


# tau 1536: exactly 48 KB of dynamic shared memory, over the limit with the pairwise kernel's static shared memory
@pytest.mark.parametrize("tau,T,B,N,use_w,use_vg", [(39, 10, 89, 67, False, True), (64, 5, 2000, 8, True, False),
                                                     (8, 5, 6, 4, False, False), (1, 1, 4, 1, True, False),
                                                     (32, 3, 100, 3, True, True), (33, 3, 50, 2, False, False),
                                                     (130, 2, 40, 2, True, False), (200, 1, 9, 1, False, True),
                                                     (64, 2, 33, 20, False, False), (1536, 1, 5, 2, True, False)])
def test_qrdqn_vs_oracle(tau, T, B, N, use_w, use_vg):
    need_cuda()
    g = rng(tau * 3 + T + B + N)
    inp = base_inputs(g, T, B, N, use_w)
    inp["q"] = g.standard_normal((B, N, tau), dtype=np.float32)
    inp["next_n_q"] = g.standard_normal((B, N, tau), dtype=np.float32)
    inp["value_gamma"] = g.random(B).astype(np.float32) if use_vg else None
    loss, td, gq = run_qrdqn(inp, 0.95, 1.1)
    o = orc.qrdqn_nstep_td(inp["q"], inp["next_n_q"], inp["action"], inp["next_n_action"], inp["reward"], inp["done"],
                           inp["weight"], inp["value_gamma"], 0.95, 1.1)
    close(loss, o["loss"], "loss")
    close(td, o["td_error_per_sample"], "td")
    close_grad(gq, o["grad_q"], "grad_q")
    mask = np.ones((B, N), dtype=bool)
    mask[np.arange(B), inp["action"]] = False
    assert np.all(gq[mask] == 0)


@pytest.mark.parametrize("name", names("qrdqn"))
def test_qrdqn_vs_golden(name):
    need_cuda()
    c = Case(name)
    inp = {k: c.inp(k) for k in ("q", "next_n_q", "action", "next_n_action", "reward", "done", "weight",
                                 "value_gamma")}
    loss, td, gq = run_qrdqn(inp, c.attr("gamma"), c.attr("coef_loss"))
    for prec in (32, 64):
        close(loss, c.out("loss", prec), "loss")
        close(td, c.out("td_error_per_sample", prec), "td")
        close_grad(gq, c.grad("q", prec), "grad_q")


# ----------------------------------------------------------------------------------------- IQN
def run_iqn(inp, gamma, kappa, coef):
    from hpc_rll.rl_utils.td import IQNNStepTDError
    q = dev(inp["q"]).requires_grad_(True)
    T, B = inp["reward"].shape
    tau, _, N = inp["q"].shape
    tau_p = inp["next_n_q"].shape[0]
    w = None if inp["weight"] is None else dev(inp["weight"])
    vg = None if inp.get("value_gamma") is None else dev(inp["value_gamma"])
    loss, td = IQNNStepTDError(tau, tau_p, T, B, N)(q, dev(inp["next_n_q"]), dev(inp["action"]),
                                                    dev(inp["next_n_action"]), dev(inp["reward"]), dev(inp["done"]),
                                                    dev(inp["replay_quantiles"]), gamma, kappa, w, vg)
    (coef * loss).sum().backward()
    torch.cuda.synchronize()
    return float(loss.item()), host(td), host(q.grad)


# (128, 28) and (127, 128): dynamic shared memory that fits the default limit only without the static shared memory
# of the sorted (12.5 KB) and the pairwise kernel
@pytest.mark.parametrize("tau,tau_p,T,B,N,kappa,use_w,use_vg", [(33, 34, 10, 64, 8, 0.9, False, True),
                                                                 (64, 64, 5, 2000, 8, 1.0, True, False),
                                                                 (8, 9, 5, 6, 4, 1.0, False, False),
                                                                 (1, 1, 1, 4, 1, 0.5, True, False),
                                                                 (32, 16, 3, 100, 3, 2.0, True, True),
                                                                 (70, 40, 2, 45, 2, 1.0, False, False),
                                                                 (5, 130, 2, 33, 5, 1.0, True, False),
                                                                 (128, 28, 3, 37, 2, 1.0, True, True),
                                                                 (127, 128, 2, 33, 2, 1.0, False, False)])
def test_iqn_vs_oracle(tau, tau_p, T, B, N, kappa, use_w, use_vg):
    need_cuda()
    g = rng(tau * 3 + tau_p + T + B + N)
    inp = base_inputs(g, T, B, N, use_w)
    inp["q"] = g.standard_normal((tau, B, N), dtype=np.float32)
    inp["next_n_q"] = g.standard_normal((tau_p, B, N), dtype=np.float32)
    inp["replay_quantiles"] = g.random((tau, B)).astype(np.float32)
    inp["value_gamma"] = g.random(B).astype(np.float32) if use_vg else None
    loss, td, gq = run_iqn(inp, 0.95, kappa, 0.8)
    o = orc.iqn_nstep_td(inp["q"], inp["next_n_q"], inp["action"], inp["next_n_action"], inp["reward"], inp["done"],
                         inp["replay_quantiles"], inp["weight"], inp["value_gamma"], 0.95, kappa, 0.8)
    close(loss, o["loss"], "loss")
    close(td, o["td_error_per_sample"], "td")
    close_grad(gq, o["grad_q"], "grad_q")
    mask = np.ones((B, N), dtype=bool)
    mask[np.arange(B), inp["action"]] = False
    assert np.all(gq[:, mask] == 0)


@pytest.mark.parametrize("name", names("iqn"))
def test_iqn_vs_golden(name):
    need_cuda()
    c = Case(name)
    inp = {k: c.inp(k) for k in ("q", "next_n_q", "action", "next_n_action", "reward", "done", "replay_quantiles",
                                 "weight", "value_gamma")}
    loss, td, gq = run_iqn(inp, c.attr("gamma"), c.attr("kappa"), c.attr("coef_loss"))
    for prec in (32, 64):
        close(loss, c.out("loss", prec), "loss")
        close(td, c.out("td_error_per_sample", prec), "td")
        close_grad(gq, c.grad("q", prec), "grad_q")


@pytest.mark.parametrize("n_atom", [2, 3, 4, 5, 31, 32, 33, 61, 62, 63, 64, 65, 114, 115, 116, 127, 128, 129, 200])
def test_dist_atom_counts(n_atom):
    """every row length around the 32-atom segment / 4-float group boundaries of the TMA-gather kernel (rows start at
    any of the four 16-byte phases: N * n_atom and the actions vary), a batch with a partial warp, the hand-over to
    the warp-per-sample kernel above 128 atoms, and 114-116 atoms, whose dynamic shared memory fits 48 KB but not
    together with the kernel's static shared memory"""
    need_cuda()
    g = rng(4000 + n_atom)
    T, B, N = 3, 77, 3
    inp = base_inputs(g, T, B, N, True)
    inp["reward"] = (inp["reward"] * 3).astype(np.float32)
    inp["dist"] = softmax(g.standard_normal((B, N, n_atom)))
    inp["next_n_dist"] = softmax(g.standard_normal((B, N, n_atom)))
    loss, td, gd = run_dist(inp, 0.97, -4.0, 6.0, 1.0)
    o = orc.dist_nstep_td(inp["dist"], inp["next_n_dist"], inp["action"], inp["next_n_action"], inp["reward"],
                          inp["done"], inp["weight"], 0.97, -4.0, 6.0, 1.0)
    close(loss, o["loss"], "loss")
    close(td, o["td_error_per_sample"], "td")
    close_grad(gd, o["grad_dist"], "grad_dist")


def test_dist_many_samples_short_rows():
    """short rows make the lane kernel's CTAs small enough for > 16 per SM: the grid (and with it the number of loss
    partials in the workspace) must stay within what the workspace holds"""
    need_cuda()
    g = rng(4242)
    T, B, N, n_atom = 2, 300001, 2, 5
    inp = base_inputs(g, T, B, N, False)
    inp["dist"] = softmax(g.standard_normal((B, N, n_atom)))
    inp["next_n_dist"] = softmax(g.standard_normal((B, N, n_atom)))
    loss, td, gd = run_dist(inp, 0.9, -1.0, 2.0, 1.0)
    o = orc.dist_nstep_td(inp["dist"], inp["next_n_dist"], inp["action"], inp["next_n_action"], inp["reward"],
                          inp["done"], inp["weight"], 0.9, -1.0, 2.0, 1.0)
    close(loss, o["loss"], "loss")
    close(td, o["td_error_per_sample"], "td")
    close_grad(gd, o["grad_dist"], "grad_dist")


@pytest.mark.parametrize("cfg", [1, 2])
def test_dist_kernel_variants(cfg):
    """lane-per-sample (1) and warp-per-sample (2) C51 kernels against the oracle, incl. done=1 rows whose whole
    mass lands on one atom and a batch that is not a multiple of the sample tile."""
    need_cuda()
    from di_hpc_b200 import _abi
    g = rng(cfg + 900)
    T, B, N, n_atom = 3, 300, 5, 51
    inp = base_inputs(g, T, B, N, True)
    inp["reward"] = (inp["reward"] * 4).astype(np.float32)
    inp["dist"] = softmax(g.standard_normal((B, N, n_atom)))
    inp["next_n_dist"] = softmax(g.standard_normal((B, N, n_atom)))
    try:
        _abi.set_config(_abi.OP_DIST_NSTEP_TD, cfg)
        loss, td, gd = run_dist(inp, 0.99, -10.0, 10.0, 1.0)
        loss_b, td_b, gd_b = run_dist(inp, 0.99, -10.0, 10.0, 1.0)
    finally:
        _abi.set_config(_abi.OP_DIST_NSTEP_TD, -1)
    o = orc.dist_nstep_td(inp["dist"], inp["next_n_dist"], inp["action"], inp["next_n_action"], inp["reward"],
                          inp["done"], inp["weight"], 0.99, -10.0, 10.0, 1.0)
    close(loss, o["loss"], "loss")
    close(td, o["td_error_per_sample"], "td")
    close_grad(gd, o["grad_dist"], "grad_dist")
    assert loss == loss_b and np.array_equal(td, td_b) and np.array_equal(gd, gd_b)  # run-to-run reproducible
