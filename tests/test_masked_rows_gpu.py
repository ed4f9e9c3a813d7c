"""V-trace, UPGO and PPO on every row-softmax path (tests/row_paths.py) with illegal-action masks, logits that start 4, 8
or 12 bytes past a 16-byte boundary, and grids that every CTA wraps around more than once.

Masked logits hold -inf (on a few paths also float32's finfo.min and -1e9, which must give the same result).  The
reference is the CPU oracle on the same inputs with the masked entries set to -1e30, which tests/test_row_paths_cpu.py
shows equals deleting those actions.  Each case checks, forward and backward:
- losses and gradients within the 1e-5 bar of tests/test_policy_ops_gpu.py (rel_err for losses, grad_err for
  gradients), and all finite;
- a gradient of exactly 0 at masked entries, and an all-zero gradient row where only the chosen action is legal;
- two identical calls give identical bits.
Precondition of the masked result: the chosen action is legal and every row has a legal action."""
import zlib

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests import row_paths as rp
from tests._golden import grad_err, rel_err
from tests._gpu import dev, host, need_cuda

pytestmark = pytest.mark.gpu
TOL = 1e-5
MASK_VALUE = {rp.NEG_INF: -np.inf, rp.FINFO_MIN: float(np.finfo(np.float32).min), rp.NEG_1E9: -1e9}
REF_FILL = np.float32(-1e30)
VT_HP = dict(gamma=0.9, lambda_=0.8, rho_clip_ratio=1.5, c_clip_ratio=0.9, rho_pg_clip_ratio=2.0)
VT_COEF = [1.0, 0.5, -0.25]
PPO_COEF = [1.0, 0.5, -0.5]
UPGO_COEF = -0.7


def n_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ------------------------------------------------------------------------------------------------- inputs
def edge_actions(g, action, N):
    """the rows that mask elements 0 and N-1 choose an action between them"""
    if N >= 3:
        R = action.size
        action[[1, R - 3]] = g.integers(1, N - 1, 2)


def make_mask(g, R, N, action, kind):
    """per-row illegal-action masks, 30-60 % of each row, never the chosen action.  Rows 0-3 and the last four are
    edge rows: only the action legal; elements 0 and N-1 masked; the entries on either side of every 4-float chunk
    edge masked; every element owned by one lane of the row's group masked (register rows with G > 1)."""
    mask = g.random((R, N)) < g.uniform(0.3, 0.6, (R, 1))
    mask[[0, R - 4]] = True
    if N >= 3:
        mask[[1, R - 3], 0] = True
        mask[[1, R - 3], N - 1] = True
    e = np.arange(N)
    for r in (2, R - 2):
        mask[r, (e % 4 == 0) | (e % 4 == 3)] = True
    if kind[0] == "reg" and kind[2] > 1:
        _, W, G, _ = kind
        lane = (e // W) % G
        for r in (3, R - 1):
            mask[r, lane == (lane[action[r]] + 1) % G] = True
    mask[np.arange(R), action] = False
    return mask


def make_inputs(case, shape, kind):
    g = np.random.default_rng(zlib.crc32(rp.case_id(case).encode()))
    R, N = int(np.prod(shape)), case.N
    action = g.integers(0, N, R)
    d = dict(action=action, logits=(g.standard_normal((R, N)) * 1.5).astype(np.float32))
    if case.op != "upgo":  # the behaviour / old policy, near the target one
        d["logits2"] = (d["logits"] + 0.5 * g.standard_normal((R, N))).astype(np.float32)
    if case.masked:
        edge_actions(g, action, N)
        d["mask"] = make_mask(g, R, N, action, kind)
        if "logits2" in d:
            d["mask2"] = make_mask(g, R, N, action, kind) if case.differ else d["mask"]
    if case.op == "ppo":
        for k in ("value_new", "value_old", "adv", "return_"):
            d[k] = g.standard_normal(R).astype(np.float32)
        d["weight"] = g.random(R).astype(np.float32)
    else:
        T, B = shape
        d["value"] = g.standard_normal((T + 1, B)).astype(np.float32)
        d["reward"] = g.standard_normal((T, B)).astype(np.float32)
        d["weight"] = g.random((T, B)).astype(np.float32)
        d["rhos"] = (g.random((T, B)) * 2).astype(np.float32)
    return d


def masked_logits(d, fill):
    out = {}
    for k, mk in (("logits", "mask"), ("logits2", "mask2")):
        if k in d:
            x = d[k].copy()
            if mk in d:
                x[d[mk]] = fill
            out[k] = x
    return out


def offset_view(a, off):
    """a copy of `a` on the GPU whose first element lies `off` floats past a 16-byte boundary"""
    store = torch.empty(a.size + 4, dtype=torch.float32, device="cuda")
    x = store[off:off + a.size].view(a.shape)
    x.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    assert x.data_ptr() % 16 == 4 * off, (x.data_ptr(), off)
    return x


# ------------------------------------------------------------------------------------------------- runs
def run_gpu(case, shape, d, fill):
    """losses and gradients of one forward + backward; logits are offset views at case.off"""
    lg = masked_logits(d, fill)
    N = case.N
    t = offset_view(lg["logits"].reshape(shape + (N, )), case.off).requires_grad_(True)
    if case.op == "vtrace":
        from hpc_rll.rl_utils.vtrace import VTrace
        T, B = shape
        v = dev(d["value"]).requires_grad_(True)
        b = offset_view(lg["logits2"].reshape(T, B, N), case.off)
        l = VTrace(T, B, N)(t, b, dev(d["action"].reshape(T, B)), v, dev(d["reward"]), dev(d["weight"]), **VT_HP)
        (VT_COEF[0] * l.policy_loss + VT_COEF[1] * l.value_loss + VT_COEF[2] * l.entropy_loss).sum().backward()
        torch.cuda.synchronize()
        return dict(policy_loss=l.policy_loss.item(), value_loss=l.value_loss.item(),
                    entropy_loss=l.entropy_loss.item(), grad_target_output=host(t.grad), grad_value=host(v.grad))
    if case.op == "upgo":
        from hpc_rll.rl_utils.upgo import UPGO
        T, B = shape
        loss = UPGO(T, B, N)(t, dev(d["rhos"]), dev(d["action"].reshape(T, B)), dev(d["reward"]), dev(d["value"]))
        (UPGO_COEF * loss).sum().backward()
        torch.cuda.synchronize()
        return dict(loss=loss.item(), grad_target_output=host(t.grad))
    from hpc_rll.rl_utils.ppo import PPO
    (B, ) = shape
    vn = dev(d["value_new"]).requires_grad_(True)
    o = offset_view(lg["logits2"], case.off)
    clip = 10.0 if case.rows is None else 0.2  # a million rows: no ratio near a clip edge, where fp32 rounding decides
    loss, info = PPO(B, N)(t, o, dev(d["action"]), vn, dev(d["value_old"]), dev(d["adv"]), dev(d["return_"]),
                           dev(d["weight"]), clip, True, None)
    (PPO_COEF[0] * loss.policy_loss + PPO_COEF[1] * loss.value_loss + PPO_COEF[2] * loss.entropy_loss).sum().backward()
    torch.cuda.synchronize()
    return dict(policy_loss=loss.policy_loss.item(), value_loss=loss.value_loss.item(),
                entropy_loss=loss.entropy_loss.item(), approx_kl=float(info.approx_kl), clipfrac=float(info.clipfrac),
                grad_logits_new=host(t.grad), grad_value_new=host(vn.grad))


def run_oracle(case, shape, d):
    lg = masked_logits(d, REF_FILL)
    N = case.N
    if case.op == "vtrace":
        T, B = shape
        o = orc.vtrace(lg["logits"].reshape(T, B, N), lg["logits2"].reshape(T, B, N), d["action"].reshape(T, B),
                       d["value"], d["reward"], d["weight"], coef=VT_COEF, **VT_HP)
        return {k: o[k] for k in ("policy_loss", "value_loss", "entropy_loss", "grad_target_output", "grad_value")}
    if case.op == "upgo":
        T, B = shape
        o = orc.upgo(lg["logits"].reshape(T, B, N), d["rhos"], d["action"].reshape(T, B), d["reward"], d["value"],
                     UPGO_COEF)
        return dict(loss=o["loss"], grad_target_output=o["grad_target_output"])
    clip = 10.0 if case.rows is None else 0.2
    o = orc.ppo(lg["logits"], lg["logits2"], d["action"], d["value_new"], d["value_old"], d["adv"], d["return_"],
                d["weight"], clip, True, None, PPO_COEF)
    return {k: o[k] for k in ("policy_loss", "value_loss", "entropy_loss", "approx_kl", "clipfrac", "grad_logits_new",
                              "grad_value_new")}


LOGIT_GRADS = ("grad_target_output", "grad_logits_new")


# ------------------------------------------------------------------------------------------------- checks
class Ctx:
    def __init__(self, case, R, paths, value):
        self.case, self.R, self.paths, self.value = case, R, paths, value

    def __call__(self, name, msg):
        direction = "bwd" if name.startswith("grad") else "fwd"
        p = self.paths[direction]
        return "%s %s path=%s (N=%d, off=%d, R=%d, passes=%d) mask=%s: %s %s" % (
            self.case.op, direction, p.kind, self.case.N, self.case.off, self.R, p.passes, self.value, name, msg)


def first_bad(bad, mask, N):
    """where the first flagged entry is: (row, k) of a logits-shaped array (N > 0) and whether it is masked"""
    i = int(np.flatnonzero(bad.reshape(-1))[0])
    if not N:
        return "index %d" % i
    row, k = divmod(i, N)
    return "(row, k) = (%d, %d)%s" % (row, k, "" if mask is None else (", masked" if mask[row, k] else ", legal"))


def check(out, ref, d, ctx):
    """every output against the oracle; the failure lists every output that is wrong, not only the first"""
    mask = d.get("mask")
    errors = []
    for name, want in ref.items():
        got = np.asarray(out[name], dtype=np.float64)
        want = np.asarray(want, dtype=np.float64)
        N = ctx.case.N if name in LOGIT_GRADS else 0
        fin = np.isfinite(got)
        if not fin.all():
            errors.append(ctx(name, "not finite, first at %s" % first_bad(~fin, mask, N)))
            continue
        if name == "clipfrac":  # a fraction of rows: one ratio rounded across a clip edge moves it by 1/B
            if abs(got - want) > 2.0 / d["action"].size + 1e-6:
                errors.append(ctx(name, "%r vs %r" % (float(got), float(want))))
        elif not name.startswith("grad"):
            e = rel_err(got, want)
            if e > TOL:
                errors.append(ctx(name, "rel err %.3e (%r vs %r)" % (e, float(got), float(want))))
        else:
            e = grad_err(got, want)
            if e > TOL:
                bad = np.abs(got - want) > TOL * np.max(np.abs(want))
                errors.append(ctx(name, "err / max|grad| = %.3e, first bad %s" % (e, first_bad(bad, mask, N))))
        if N and mask is not None:
            g2 = got.reshape(-1, N)
            z = (g2 != 0) & mask
            if z.any():
                errors.append(ctx(name, "non-zero at a masked entry, first at %s" % first_bad(z, mask, N)))
            only = mask.sum(axis=1) == N - 1  # only the chosen action legal: p = 1, H = 0
            nz = (g2 != 0) & only[:, None]
            assert only.any(), "make_mask leaves a one-legal-action row"
            if nz.any():
                errors.append(ctx(name, "non-zero in a one-legal-action row, first at %s" % first_bad(nz, mask, N)))
    assert not errors, "\n".join(errors)


def bits(out):
    return {k: np.asarray(v).tobytes() for k, v in out.items()}


@pytest.mark.parametrize("case", rp.cases(), ids=rp.case_id)
def test_row_path(case):
    need_cuda()
    sms = n_sms()
    shape = rp.case_shape(case, rp.case_rows(case, sms))
    R = int(np.prod(shape))
    paths = {dd: rp.row_path(case.op, dd, case.N, case.off, R, sms) for dd in rp.DIRECTIONS}
    if case.rows is None:
        assert all(p.passes >= 2 for p in paths.values()), paths
    d = make_inputs(case, shape, paths["fwd"].kind)
    ref = run_oracle(case, shape, d)
    results = {}
    for value in case.mask_values or ("none", ):
        ctx = Ctx(case, R, paths, value)
        fill = MASK_VALUE.get(value, 0.0)
        out = run_gpu(case, shape, d, fill)
        check(out, ref, d, ctx)
        again = bits(run_gpu(case, shape, d, fill))
        for k, v in bits(out).items():
            assert v == again[k], ctx(k, "differs between two identical calls")
        results[value] = out
    first = case.mask_values[0] if case.mask_values else "none"
    for value, out in results.items():
        for k, v in out.items():
            assert np.array_equal(v, results[first][k]), Ctx(case, R, paths, value)(k, "differs from mask=%s" % first)


def test_masked_column_equals_deleted_column_on_looping_kernel():
    """one -inf column inserted into an N-1 action V-trace problem on the looping kernel gives the N-1 action oracle's
    losses and gradients, and a zero gradient in that column"""
    need_cuda()
    T, B, N, k = 4, 50, 301, 137
    sms = n_sms()
    assert rp.row_path("vtrace", "fwd", N, 0, T * B, sms).kind == ("loop", )
    g = np.random.default_rng(301)
    inp = dict(target_output=(g.standard_normal((T, B, N - 1)) * 1.5).astype(np.float32),
               behaviour_output=(g.standard_normal((T, B, N - 1)) * 1.5).astype(np.float32),
               action=g.integers(0, N - 1, (T, B)), value=g.standard_normal((T + 1, B)).astype(np.float32),
               reward=g.standard_normal((T, B)).astype(np.float32), weight=g.random((T, B)).astype(np.float32))
    o = orc.vtrace(**inp, coef=VT_COEF, **VT_HP)
    from hpc_rll.rl_utils.vtrace import VTrace
    t = dev(np.insert(inp["target_output"], k, -np.inf, axis=2)).requires_grad_(True)
    b = dev(np.insert(inp["behaviour_output"], k, -np.inf, axis=2))
    a = dev(np.where(inp["action"] >= k, inp["action"] + 1, inp["action"]))
    v = dev(inp["value"]).requires_grad_(True)
    l = VTrace(T, B, N)(t, b, a, v, dev(inp["reward"]), dev(inp["weight"]), **VT_HP)
    (VT_COEF[0] * l.policy_loss + VT_COEF[1] * l.value_loss + VT_COEF[2] * l.entropy_loss).sum().backward()
    gt = host(t.grad)
    for name, x in (("policy_loss", l.policy_loss), ("value_loss", l.value_loss), ("entropy_loss", l.entropy_loss)):
        assert rel_err(x.item(), o[name]) <= TOL, name
    assert np.all(np.isfinite(gt)) and np.all(gt[:, :, k] == 0)
    assert grad_err(np.delete(gt, k, axis=2), o["grad_target_output"]) <= TOL
    assert grad_err(host(v.grad), o["grad_value"]) <= TOL
