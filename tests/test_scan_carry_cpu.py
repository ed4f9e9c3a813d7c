"""Certifies the scan-carry probes of tests/scan_probes.py on the CPU, before tests/test_scan_carry_gpu.py holds the
kernels to them bit for bit.

- Every probe that claims to be exact is: the fp32 oracle equals the fp64 oracle rounded to fp32 on every carry-bearing
  quantity, at every shape the GPU test runs.
- The look-back shapes reach every geometry property that has its own code path, for every op with a look-back kernel.
- Every segment edge (and the rows next to it) carries an impulse in some column."""
import numpy as np
import pytest

from tests import scan_probes as sp

EXACT_CASES = sorted({(op, fam, T, B) for op in sp.OPS for fam in sp.FAMILIES[op] if fam != "random"
                      for cfg in (-1,) + sp.CONFIGS[op] for T, B in sp.shapes_for(cfg)})


@pytest.mark.parametrize("op,family,T,B", EXACT_CASES)
def test_exact_probe_is_exact_in_fp32(op, family, T, B):
    p = sp.make_probe(op, family, T, B)
    assert p.exact
    s32, o32, _ = sp.reference(p, np.float32)
    s64, _, _ = sp.reference(p, np.float64)
    for name, a in s32.items():
        want = s64[name].astype(np.float32)
        bad = np.argwhere(a != want)
        assert bad.size == 0, "%s %s (T=%d, B=%d): %s not exact in fp32, first at (t, b) = %s (%r vs %r)" % (
            op, family, T, B, name, tuple(bad[0]), a[tuple(bad[0])], want[tuple(bad[0])])
        # below 2^24: every partial sum of the chain is an exact fp32 integer or a correctly rounded quotient
        assert np.max(np.abs(s64[name])) < 2.0 ** 24, (op, family, name)
    for name, a in o32.items():
        assert a.dtype == np.float32 and np.all(np.isfinite(a)), (op, family, name)


@pytest.mark.parametrize("op", sp.OPS)
def test_probes_carry_through_every_segment(op):
    """with coefficient 1 an impulse reaches every row behind it in scan order: the impulse probe's outputs are non-zero
    almost everywhere, so a dropped carry changes them by O(1)"""
    p = sp.make_probe(op, "impulse", 1025, 33)
    s32, _, _ = sp.reference(p, np.float32)
    for name, a in s32.items():
        if name in ("grad_next_value",):
            continue
        assert np.count_nonzero(a) >= 0.9 * a.size, (op, name, np.count_nonzero(a) / a.size)


@pytest.mark.parametrize("op", sp.OPS)
def test_lookback_shapes_reach_every_geometry(op):
    geoms = {(T, B): sp.lb_geom(T, B, 21) for T, B in sp.shapes_for(21)}
    assert all(g.split for g in geoms.values()), geoms
    # the segment at the end of T is partial: it is the first one scanned by the reverse-time scans (forwards of
    # all five ops) and the last one scanned by the forward-time scans (the GAE and episodic GAE adjoints)
    props = {
        "partial segment at the end of T": lambda g, T, B: g.partial < g.L,
        "L > 32 (multi-chunk segments)": lambda g, T, B: g.L > sp.LB_CHUNK_ROWS and g.chunks > 1,
        "three chunks per segment": lambda g, T, B: g.chunks >= 3,
        "two fold rounds (S > 33)": lambda g, T, B: g.fold_rounds >= 2 and g.S > 33,
        "S = 64": lambda g, T, B: g.S == sp.LB_MAX_SEG,
        "ticket-ordered grid": lambda g, T, B: g.ticketed,
        "blockIdx-ordered grid": lambda g, T, B: not g.ticketed,
        "ticket-ordered with multi-chunk segments": lambda g, T, B: g.ticketed and g.L > sp.LB_CHUNK_ROWS,
        "B % 32 != 0": lambda g, T, B: B % 32 != 0,
        "B = 1": lambda g, T, B: B == 1,
        "several column tiles": lambda g, T, B: g.tiles > 1,
    }
    for name, fn in props.items():
        assert any(fn(g, T, B) for (T, B), g in geoms.items()), "%s: no look-back shape has %s" % (op, name)
    # the automatic rule takes the look-back path at some shapes and the column scan at the others
    auto = [sp.lb_geom(T, B, -1).split for T, B in sp.shapes_for(-1)]
    assert any(auto) and not all(auto)


def test_lb_geom_mirrors_the_geometry_rule():
    # (T, B) -> (S, L, tiles, ticketed, chunks, fold rounds, partial rows)
    want = {(33, 1): (2, 32, 1, False, 1, 1, 1), (1024, 64): (32, 32, 2, False, 1, 1, 32),
            (1025, 33): (33, 32, 2, False, 1, 1, 1), (2048, 1): (64, 32, 1, False, 1, 2, 32),
            (2049, 64): (52, 40, 2, False, 2, 2, 9), (4096, 33): (64, 64, 2, False, 2, 2, 64),
            (4100, 640): (57, 72, 20, True, 3, 2, 68), (1024, 2048): (32, 32, 64, True, 1, 1, 32)}
    for (T, B), w in want.items():
        g = sp.lb_geom(T, B, 21)
        assert (g.S, g.L, g.tiles, g.ticketed, g.chunks, g.fold_rounds, g.partial) == w, (T, B, g)
    assert not sp.lb_geom(31, 64, 21).split and not sp.lb_geom(32, 64, 21).split  # one segment: no split
    assert not sp.lb_geom(1024, 64, 13).split  # any other forced config disables the look-back path
    assert sp.lb_geom(512, 2048, -1).split and not sp.lb_geom(511, 64, -1).split and not sp.lb_geom(1024, 2049, -1).split


@pytest.mark.parametrize("T,B", sorted({s for cfg in (-1, 21, 0) for s in sp.shapes_for(cfg)}))
def test_every_segment_edge_carries_an_impulse(T, B):
    p = sp.make_probe("gae", "impulse", T, B)
    hit = set(r for rows in p.marks for r in rows)
    g = sp.lb_geom(T, B, 21)
    if g.split:
        for k in range(1, g.S):
            for r in (k * g.L - 1, k * g.L, k * g.L + 1):
                if r < T:
                    assert r in hit, (T, B, k, r)
        p0 = (g.S - 1) * g.L
        assert {p0 - 1, p0}.issubset(hit)
    assert {0, T - 1}.issubset(hit)
    # the same rows in every op's impulse probe
    for op in sp.OPS:
        assert sp.make_probe(op, "impulse", T, B).marks == p.marks
