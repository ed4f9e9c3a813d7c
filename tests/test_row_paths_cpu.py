"""The row-path mirror of tests/row_paths.py, pinned to known dispatch results; the GPU case list of
tests/test_masked_rows_gpu.py checked to reach every kernel path; and the masked reference that GPU test relies on:
the CPU oracle with masked logits set to -1e30 equals the oracle of the problem without those actions."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import row_paths as rp

SMS = (132, 114, 78, 1)  # H100 SXM, H100 PCIe, a small part, and the degenerate one-SM grid


@pytest.mark.parametrize("N,off,kind", [
    (8, 0, ("reg", 4, 1, 2)), (8, 1, ("reg", 1, 1, 8)), (16, 2, ("reg", 2, 1, 8)), (16, 1, ("staged", 0)),
    (18, 0, ("reg", 2, 2, 5)), (33, 0, ("reg", 1, 8, 5)), (255, 0, ("reg", 1, 32, 8)), (257, 0, ("loop", )),
    (300, 1, ("loop", )), (514, 0, ("loop", )), (1028, 0, ("loop", )), (9, 0, ("staged", 1)), (9, 3, ("staged", 0)),
    (8, 2, ("reg", 2, 1, 4)), (64, 2, ("reg", 2, 4, 8)), (1024, 0, ("reg", 4, 32, 8)), (256, 0, ("reg", 4, 16, 4)),
    (512, 2, ("reg", 2, 32, 8)), (6, 0, ("reg", 2, 1, 3)),
    (32, 0, ("reg", 4, 2, 4)), (32, 2, ("reg", 2, 2, 8)), (32, 1, ("staged", 0)), (36, 1, ("reg", 1, 8, 5)),
])
def test_mirror_matches_known_dispatch(N, off, kind):
    for op in rp.OPS:
        for d in rp.DIRECTIONS:
            assert rp.row_path(op, d, N, off, 1000, 132).kind == kind, (op, d, N, off)


def test_looping_kernel_thresholds():
    """the first N on the looping kernel, per base alignment (a 4-byte aligned base takes it from N = 257 on)"""
    def first_loop(off, step, start):
        N = start
        while rp.row_path("vtrace", "fwd", N, off, 10, 132).kind != ("loop", ):
            N += step
        return N
    assert first_loop(0, 2, 1) == 257           # odd N
    assert first_loop(0, 4, 2) == 514           # N = 2 mod 4
    assert first_loop(0, 4, 4) == 1028          # N = 0 mod 4
    for off in (1, 3):
        assert first_loop(off, 1, 1) == 257


def test_backward_alignment_follows_the_logits():
    """the gradient is allocated fresh (16-byte aligned), so every backward takes the forward's path"""
    for N in list(range(1, 41)) + [64, 255, 256, 257, 300, 514, 1028]:
        for off in range(4):
            fw = {op: rp.row_path(op, "fwd", N, off, 500, 132).kind for op in rp.OPS}
            assert len(set(fw.values())) == 1, (N, off, fw)
            assert rp.row_path("ppo", "bwd", N, off, 500, 132).kind == fw["ppo"], (N, off)


@pytest.mark.parametrize("sms", SMS)
def test_grid_passes(sms):
    cap = 16 * sms
    p = rp.row_path("ppo", "fwd", 8, 0, cap * 256, sms)
    assert (p.grid, p.passes) == (cap, 1)
    # one row more: only CTA 0 wraps; the last CTA still makes one pass
    assert rp.row_path("ppo", "fwd", 8, 0, cap * 256 + 1, sms).passes == 1
    assert rp.row_path("ppo", "fwd", 8, 0, (2 * cap - 1) * 256, sms).passes == 1
    assert rp.row_path("ppo", "fwd", 8, 0, (2 * cap - 1) * 256 + 1, sms).passes == 2
    for N, off in ((8, 0), (9, 0), (16, 1), (257, 0), (300, 1), (64, 0), (33, 0)):
        R = rp.wrap_rows(N, off, sms)
        for op in rp.OPS:
            for d in rp.DIRECTIONS:
                assert rp.row_path(op, d, N, off, R, sms).passes >= 2, (op, d, N, off, sms)


REQUIRED = {("reg", 4, "G1"), ("reg", 4, "G>1"), ("reg", 2, "G1"), ("reg", 2, "G>1"), ("reg", 1, "G1"),
            ("reg", 1, "G>1"), ("staged", 1), ("staged", 0), ("loop", )} | {("kmax", k) for k in range(1, 9)}


def features(kind):
    if kind[0] == "reg":
        _, width, G, kmax = kind
        return {("reg", width, "G1" if G == 1 else "G>1"), ("kmax", kmax)}
    return {kind}


@pytest.mark.parametrize("sms", SMS[:3])
def test_gpu_cases_reach_every_path(sms):
    cases = rp.cases()
    for op in rp.OPS:
        for d in rp.DIRECTIONS:
            masked, offset_views = set(), set()
            for c in cases:
                if c.op != op:
                    continue
                kind = rp.row_path(op, d, c.N, c.off, rp.case_rows(c, sms), sms).kind
                (masked if c.masked else offset_views).update(features(kind))
            assert REQUIRED <= masked, (op, d, sorted(REQUIRED - masked, key=str))
            # the unmasked offset views reach the branches nothing aligned reaches
            assert {("staged", 0), ("reg", 2, "G1"), ("reg", 2, "G>1"), ("reg", 1, "G1"), ("reg", 1, "G>1")} <= \
                offset_views, (op, d)
        staged_even = [c for c in cases if c.op == op and c.N % 2 == 0 and
                       rp.row_path(op, "fwd", c.N, c.off, 100, sms).kind == ("staged", 0)]
        assert any(c.masked for c in staged_even) and any(not c.masked for c in staged_even), op
        narrow_mult4 = {rp.row_path(op, "fwd", c.N, c.off, 100, sms).kind[1] for c in cases
                        if c.op == op and not c.masked and c.N % 4 == 0 and c.N not in range(9, 33)}
        assert {1, 2} <= narrow_mult4, op
        # every mask value runs on a register, a staged and the looping path
        kinds = {rp.row_path(op, "fwd", c.N, c.off, 100, sms).kind[0] for c in cases
                 if c.op == op and c.mask_values == rp.ALL_MASK_VALUES}
        assert kinds == {"reg", "staged", "loop"}, op
    for op in ("vtrace", "ppo"):
        kinds = {rp.row_path(op, "fwd", c.N, c.off, 100, sms).kind[0] for c in cases if c.op == op and c.differ}
        assert {"reg", "loop"} <= kinds, op
    wrapped = set()
    for c in cases:
        if c.rows is None:
            assert c.masked
            for d in rp.DIRECTIONS:
                p = rp.row_path(c.op, d, c.N, c.off, int(np.prod(rp.case_shape(c, rp.case_rows(c, sms)))), sms)
                assert p.passes >= 2, (c, d, p)
                wrapped.add((c.op, d, p.kind if p.kind[0] != "staged" else ("staged", )))
    for d in rp.DIRECTIONS:
        assert ("ppo", d, ("reg", 4, 1, 2)) in wrapped
        assert any(k == ("staged", ) for op, dd, k in wrapped if dd == d)
        assert ("vtrace", d, ("loop", )) in wrapped and ("upgo", d, ("loop", )) in wrapped


def test_case_ids_are_unique():
    ids = [rp.case_id(c) for c in rp.cases()]
    assert len(ids) == len(set(ids))


# ------------------------------------------------------------------------------------- the masked reference
BIG = -1e30


def _vtrace_problem(g, T, B, N):
    return dict(target_output=g.standard_normal((T, B, N)) * 1.5, behaviour_output=g.standard_normal((T, B, N)) * 1.5,
                action=g.integers(0, N, (T, B)), value=g.standard_normal((T + 1, B)), reward=g.standard_normal((T, B)),
                weight=g.random((T, B)))


HP = dict(gamma=0.9, lambda_=0.8, rho_clip_ratio=1.5, c_clip_ratio=0.9, rho_pg_clip_ratio=2.0)


def _insert(inp, keys, k, fill):
    big = dict(inp)
    for name in keys:
        big[name] = np.insert(inp[name], k, fill, axis=-1)
    big["action"] = np.where(inp["action"] >= k, inp["action"] + 1, inp["action"])
    return big


def _agree(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.all(np.isfinite(got)), what
    err = np.max(np.abs(got - want)) / max(1.0, np.max(np.abs(want)))
    assert err <= 1e-12, "%s: %.3e" % (what, err)


@pytest.mark.parametrize("N,k", [(2, 0), (9, 4), (9, 8), (300, 0), (300, 151), (300, 299)])
def test_masked_reference_equals_column_deletion(N, k):
    """fp64 oracle: a column of -1e30 inserted at k gives the losses and gradients of the problem without it, and an
    exactly zero gradient in that column.  With -inf the oracle itself returns NaN (logp * prob = -inf * 0), which is
    why the GPU tests feed it -1e30 where the kernels get -inf."""
    g = np.random.default_rng(N * 7 + k)
    T, B = 3, 11
    keys = ("target_output", "behaviour_output")
    inp = _vtrace_problem(g, T, B, N - 1 if N > 1 else 1)
    o = orc.vtrace(**inp, coef=[1.0, 0.5, -0.25], **HP)
    m = orc.vtrace(**_insert(inp, keys, k, BIG), coef=[1.0, 0.5, -0.25], **HP)
    for name in ("policy_loss", "value_loss", "entropy_loss", "grad_value"):
        _agree(m[name], o[name], "vtrace " + name)
    assert np.all(m["grad_target_output"][..., k] == 0)
    _agree(np.delete(m["grad_target_output"], k, axis=-1), o["grad_target_output"], "vtrace grad_target_output")
    nan = orc.vtrace(**_insert(inp, keys, k, -np.inf), coef=[1.0, 0.5, -0.25], **HP)
    assert np.isnan(nan["entropy_loss"])

    up = dict(target_output=inp["target_output"], rhos=g.random((T, B)) * 2, action=inp["action"],
              rewards=inp["reward"], bootstrap_values=inp["value"])
    o = orc.upgo(**up, coef_loss=-0.7)
    m = orc.upgo(**_insert(up, ("target_output", ), k, BIG), coef_loss=-0.7)
    _agree(m["loss"], o["loss"], "upgo loss")
    assert np.all(m["grad_target_output"][..., k] == 0)
    _agree(np.delete(m["grad_target_output"], k, axis=-1), o["grad_target_output"], "upgo grad_target_output")

    Bp = 37
    lo = g.standard_normal((Bp, N - 1))
    pp = dict(logits_new=lo + 0.3 * g.standard_normal((Bp, N - 1)), logits_old=lo, action=g.integers(0, N - 1, Bp),
              value_new=g.standard_normal(Bp), value_old=g.standard_normal(Bp), adv=g.standard_normal(Bp),
              return_=g.standard_normal(Bp), weight=g.random(Bp))
    args = dict(clip_ratio=0.2, use_value_clip=True, dual_clip=None, coef=[1.0, 0.5, -0.01])
    o = orc.ppo(**pp, **args)
    m = orc.ppo(**_insert(pp, ("logits_new", "logits_old"), k, BIG), **args)
    for name in ("policy_loss", "value_loss", "entropy_loss", "approx_kl", "clipfrac", "grad_value_new"):
        _agree(m[name], o[name], "ppo " + name)
    assert np.all(m["grad_logits_new"][..., k] == 0)
    _agree(np.delete(m["grad_logits_new"], k, axis=-1), o["grad_logits_new"], "ppo grad_logits_new")
    nan = orc.ppo(**_insert(pp, ("logits_new", "logits_old"), k, -np.inf), **args)
    assert np.isnan(nan["entropy_loss"])
