"""Mirror of the host-side dispatch of the row-softmax kernels shared by V-trace, UPGO and PPO, and the case list that
tests/test_masked_rows_gpu.py runs through them.  Pure Python: tests/test_row_paths_cpu.py pins the mirror to known
cases and checks that the case list reaches every kernel path.

Per call, `row_geom` / `use_staged_rows` (csrc/softmax_rows.cuh) pick one of three kernel families:
  ("reg", width, G, kmax)  -- a row in the registers of G lanes, kmax chunks of `width` floats per lane
  ("staged", aligned)      -- 9 <= N <= 32 read as scalars: rows staged through shared memory; `aligned` selects the
                              128-bit branch of stage_rows / unstage_rows, 0 the scalar one
  ("loop",)                -- one warp per row, N too large for registers
and `rows_grid` caps the grid at 16 CTAs per SM, so large row counts make every CTA stride over the rows more than once.

Which pointers the choice looks at (the base offset of each, in floats, decides its 16- and 8-byte alignment):
  V-trace forward: target_output, behaviour_output     PPO forward: logits_new, logits_old
  UPGO forward: target_output                           every backward: the logits and the freshly allocated gradient
"""
import collections

OPS = ("vtrace", "upgo", "ppo")
DIRECTIONS = ("fwd", "bwd")

STAGE_ROWS = 256   # kStageRows
CTAS_PER_SM = 16   # rows_grid


def row_geom(N, offs):
    """(width, G, kmax) of `row_geom` for row length N and the float offsets `offs` of the tensors it looks at
    (kmax 0: too large for registers, the looping kernel)"""
    a16 = all(o % 4 == 0 for o in offs)
    a8 = all(o % 2 == 0 for o in offs)
    width = 4 if (a16 and N % 4 == 0) else (2 if (a8 and N % 2 == 0) else 1)
    chunks = N // width
    cap = 4 if width == 4 else 8
    G = 1
    while G < 32 and chunks > G * cap:
        G <<= 1
    per_lane = (chunks + G - 1) // G
    return width, G, (per_lane if per_lane <= 8 else 0)


def use_staged_rows(N, width):
    return 8 < N <= 32 and width == 1


def rows_grid(R, rows_per_block, sms):
    return max(1, min((R + rows_per_block - 1) // rows_per_block, sms * CTAS_PER_SM))


def geometry_offsets(op, direction, off):
    """float offsets of the pointers the dispatch of (op, direction) looks at, when every logits tensor of the call
    starts `off` floats past a 16-byte boundary (the gradient is allocated fresh, so its offset is 0)"""
    assert op in OPS and direction in DIRECTIONS
    if direction == "bwd":
        return (off, 0)
    return (off, ) if op == "upgo" else (off, off)


Path = collections.namedtuple("Path", "kind rows_per_block grid passes")


def row_path(op, direction, N, off, R, sms):
    """the kernel (op, direction) runs for N actions, logits at float offset `off`, R rows on `sms` SMs.

    kind: ("reg", width, G, kmax) | ("staged", aligned) | ("loop",).  passes: the number of grid-stride passes of the
    CTA with the fewest (the last one); >= 2 means every CTA wraps around the grid at least once."""
    offs = geometry_offsets(op, direction, off)
    width, G, kmax = row_geom(N, offs)
    if use_staged_rows(N, width):
        kind, rpb = ("staged", int(all(o % 4 == 0 for o in offs))), STAGE_ROWS
    elif kmax == 0:
        kind, rpb = ("loop", ), 8
    else:
        kind, rpb = ("reg", width, G, kmax), (32 // G) * 8
    grid = rows_grid(R, rpb, sms)
    stride = grid * rpb
    last = R - (grid - 1) * rpb  # rows from the last CTA's first row on
    return Path(kind, rpb, grid, max(1, (last + stride - 1) // stride))


def row_layouts():
    """every row kernel the dispatch can select: (family, width, G1, kmax) for a register layout (G1: one lane per row),
    (family, "staged") and (family, "loop"); family: the op of a forward, "grad" for the backward all three share.  N runs
    past the three looping thresholds (257, 514, 1028) at every float offset of the logits"""
    out = set()
    for op in OPS:
        for direction in DIRECTIONS:
            family = op if direction == "fwd" else "grad"
            for N in range(1, 1101):
                for off in range(4):
                    kind = row_path(op, direction, N, off, 1000, 132).kind
                    out.add((family, kind[1], kind[2] == 1, kind[3]) if kind[0] == "reg" else (family, kind[0]))
    return out


def wrap_rows(N, off, sms):
    """a ragged row count at which every CTA of the (N, off) path makes at least two grid-stride passes"""
    p = row_path("upgo", "fwd", N, off, 1, sms)
    rpb = p.rows_per_block
    return (2 * CTAS_PER_SM * sms - 1) * rpb + rpb // 2 + 3


# ----------------------------------------------------------------------------------------------------- GPU case list
# Case.rows: R, the number of logits rows (T*B for V-trace and UPGO, B for PPO); None: wrap_rows() at the device's SM
# count.  masked: per-row illegal-action masks; mask_values: the values masked entries hold (each runs separately and
# must give the same result); differ: the second logits tensor (behaviour / old policy) has its own legal set.
Case = collections.namedtuple("Case", "op N off rows masked mask_values differ")

NEG_INF, FINFO_MIN, NEG_1E9 = "-inf", "finfo.min", "-1e9"
ALL_MASK_VALUES = (NEG_INF, FINFO_MIN, NEG_1E9)

# (N, off) reaching, for every op: each register width with G = 1 and G > 1, kmax 1..8, staged aligned and unaligned
# (an even N, so the shared-memory pitch N|1 differs from N), and the looping kernel from every entry of its table
MASKED_GEOMS = (
    (4, 0), (8, 0), (12, 0), (16, 0), (64, 0), (1000, 0),      # width 4: k1 k2 k3 k4, G4 k4, G32 k8
    (6, 0), (10, 0), (12, 2), (14, 0), (16, 2), (18, 0),       # width 2: k3 k5 k6 k7 k8, G2 k5
    (7, 0), (6, 1), (8, 1), (33, 0), (255, 0),                 # width 1: k7 k6 k8, G8 k5, G32 k8
    (9, 0), (31, 0), (16, 1), (18, 3),                         # staged: aligned, unaligned
    (257, 0), (300, 1), (514, 0), (1028, 0),                   # looping kernel
)
# run with every mask value
ALL_VALUE_GEOMS = ((16, 0), (33, 0), (9, 0), (16, 1), (257, 0))
# unmasked offset views on the branches nothing else runs: staged unaligned, widths 2 and 1 at N % 4 == 0
OFFSET_GEOMS = ((16, 1), (9, 3), (18, 1), (10, 3), (8, 2), (16, 2), (64, 2), (8, 1), (4, 3), (64, 1), (36, 3))
# every CTA makes two or more passes: PPO's register kernel at G = 1 (per-row scalars prefetched a pass ahead), a
# staged kernel, and the looping kernels of V-trace and UPGO
WRAPPED = (("ppo", 8, 0), ("ppo", 9, 0), ("vtrace", 257, 0), ("upgo", 300, 1))


def small_rows(op):
    return 131 if op == "ppo" else 3 * 45


def cases():
    out = []
    for op in OPS:
        for N, off in MASKED_GEOMS:
            vals = ALL_MASK_VALUES if (N, off) in ALL_VALUE_GEOMS else (NEG_INF, )
            out.append(Case(op, N, off, small_rows(op), True, vals, False))
        if op != "upgo":
            out.append(Case(op, 33, 0, small_rows(op), True, (NEG_INF, ), True))
            out.append(Case(op, 300, 1, small_rows(op), True, (NEG_INF, ), True))
        for N, off in OFFSET_GEOMS:
            out.append(Case(op, N, off, small_rows(op), False, (), False))
    for op, N, off in WRAPPED:
        out.append(Case(op, N, off, None, True, (NEG_INF, ), False))
    return out


def case_id(c):
    return "%s-N%d-off%d-%s%s%s" % (c.op, c.N, c.off, "wrap" if c.rows is None else "R%d" % c.rows,
                                   "-masked" if c.masked else "", "-differ" if c.differ else "")


def case_rows(c, sms):
    return wrap_rows(c.N, c.off, sms) if c.rows is None else c.rows


def case_shape(c, R):
    """(T, B) for V-trace and UPGO (T = 3; B rounded up so that T*B >= R), (B,) for PPO"""
    return (R, ) if c.op == "ppo" else (3, (R + 2) // 3)
