"""Probe inputs for the first-order affine scans (GAE, TD(lambda), V-trace, UPGO, episodic GAE) and a mirror of the
look-back geometry.  numpy only: tests/test_scan_carry_cpu.py certifies the probes on the CPU and
tests/test_scan_carry_gpu.py runs them through every kernel regime.

Every scan of these ops is x_t = a_t * x_{t+-1} + b_t.  The look-back T-split (csrc/scan_lookback.cuh) cuts T into
segments and carries (A = prod a_t, B = zero-carry result) from one segment to the next.  Random data with a damped
coefficient (gamma*lambda < 1) multiplies any carry error below the tolerances within about one segment, so the probes
here keep the coefficient at exactly 1 (or exactly 0, or break the chain at one chosen row):

- ``impulse``: zeros except small integers at chosen rows of each column.  The rows run over every segment edge
  (kL-1, kL, kL+1), the partial segment, rows 0 and T-1 and TMA box edges.  With a coefficient of 1 every step of a
  column's chain carries the impulse, and small integers keep the recurrence exact in fp32.
- ``zero``: coefficient 0 everywhere, dense small integers.  Every step is the one-step formula.
- ``break``: dense small integers, coefficient 1, except on segment-edge rows (one per column, several when B is
  smaller than the number of edges), where an episode ends (episodic GAE) or UPGO stops following the trajectory.
- ``random``: standard-normal data with coefficient 1.  Not exact; used for an error bound against fp64.

``reference(probe, dtype)`` evaluates an op with the CPU oracle and returns three dicts:
  scan -- the carry-bearing quantities (returns, advantages, adjoints); an exact probe has them exact in fp32;
  out  -- what the kernel writes, formed from ``scan`` in the kernel's own fp32 operation order (float32), or in exact
          arithmetic (float64);
  loss -- scalar losses.
"""
import collections

import numpy as np

from oracle import oracle as orc
from tests import gae_episodic_oracle as epi

OPS = ("gae", "td_lambda", "vtrace", "upgo", "gae_episodic")
OP_ID = {"gae": 0, "td_lambda": 1, "vtrace": 2, "upgo": 3, "gae_episodic": 10}  # _abi.OP_*
# families per op; "_w" runs the same probe with an all-ones weight (the weighted kernel instantiation)
FAMILIES = {
    "gae": ("impulse", "zero", "random"),
    "td_lambda": ("impulse", "impulse_w", "zero", "random"),
    "vtrace": ("impulse", "impulse_w", "zero", "random"),
    "upgo": ("impulse", "zero", "break", "random"),
    "gae_episodic": ("impulse", "zero", "break", "random"),
}
N_ACT = 4  # actions of the policy ops (their logits only feed the losses, not the carries)

# forced tuning configs per op (hpc_rll_debug_set_config); -1 (automatic) runs as well
CONFIGS = {
    "gae": (5, 7, 13, 21, 33, 99),
    "td_lambda": (0, 1, 2, 21, 99),
    "vtrace": (0, 2, 21, 99),
    "upgo": (0, 2, 21, 99),
    "gae_episodic": (33, 21, 99),
}
# look-back shapes: partial segments, B = 1, B % 32 != 0, L > 32 (T > 2048), two fold rounds (S > 33), S = 64 and
# ticket-ordered grids (S * tiles > 1024: (4100, 640) and (1024, 2048)); tests/test_scan_carry_cpu.py checks the list
LB_SHAPES = ((33, 1), (63, 31), (64, 33), (1024, 64), (1025, 33), (2048, 1), (2049, 64), (4096, 33), (4100, 640),
             (1024, 2048))
# forced column scans: B % 4 != 0 (generic kernel), and TMA-describable shapes with partial column tiles
COL_SHAPES = ((63, 31), (1025, 64), (2048, 36))
# automatic dispatch at a wide batch: the widest column-scan regime of every op (B >= 256 SMs on a 132-SM H100)
WIDE_SHAPES = ((40, 33792),)


def shapes_for(cfg):
    if cfg == 21:
        return LB_SHAPES
    if cfg < 0:
        return LB_SHAPES + WIDE_SHAPES
    return COL_SHAPES

# mirror of csrc/scan_lookback.cuh / scan_lookback.cu
LB_COLS = 32
LB_CHUNK_ROWS = 32
LB_MAX_SEG = 64
LB_RESIDENT_CTAS = 1024
LB_FOLD_BATCH = 32  # predecessors folded per round in lb_fold

Geom = collections.namedtuple("Geom", "split S L tiles grid ticketed chunks fold_rounds partial")


def lb_geom(T, B, cfg):
    """``lookback_geometry`` (csrc/scan_lookback.cu) for any T.  cfg is the forced tuning config (-1 = automatic).
    Returns split=False when the look-back path does not run; otherwise S segments of L rows (the last one
    ``partial`` rows long), ``tiles`` 32-column tiles, the grid, whether CTAs take atomic tickets (grid > 1024),
    shared-memory chunks per segment and the fold rounds of the last segment in scan order."""
    no = Geom(False, 1, 0, 0, 0, False, 0, 0, 0)
    if cfg >= 0 and cfg != 21:
        return no
    if cfg < 0 and (B > 2048 or T < 512):
        return no
    if T < 32 or B <= 0:
        return no
    tiles = (B + LB_COLS - 1) // LB_COLS
    L = LB_CHUNK_ROWS
    S = (T + L - 1) // L
    if S > LB_MAX_SEG:
        L = ((T + LB_MAX_SEG - 1) // LB_MAX_SEG + 7) // 8 * 8
        S = (T + L - 1) // L
    if S < 2:
        return no
    grid = S * tiles
    return Geom(True, S, L, tiles, grid, grid > LB_RESIDENT_CTAS, (L + LB_CHUNK_ROWS - 1) // LB_CHUNK_ROWS,
                (S - 1 + LB_FOLD_BATCH - 1) // LB_FOLD_BATCH, T - (S - 1) * L)


def segment_edges(T, B):
    """rows kL-1, kL, kL+1 of every inner segment boundary of the forced look-back geometry"""
    g = lb_geom(T, B, 21)
    if not g.split:
        return []
    rows = set()
    for k in range(1, g.S):
        rows.update((k * g.L - 1, k * g.L, k * g.L + 1))
    return sorted(r for r in rows if 0 <= r < T)


def impulse_rows(T, B):
    """every row an impulse probe of (T, B) puts an impulse on"""
    g = lb_geom(T, B, 21)
    rows = set(segment_edges(T, B)) | {0, 1, T - 2, T - 1}
    if g.split:
        p0 = (g.S - 1) * g.L  # first row of the partial (last) segment
        rows.update((p0 - 1, p0, p0 + 1, p0 + g.partial // 2))
    for box in (4, 8, 16, 64):  # TMA box heights of the column scans, at both ends of T
        rows.update((box - 1, box, box + 1, T - box - 1, T - box, T - box + 1))
    return sorted(r for r in rows if 0 <= r < T)


def column_rows(rows, B):
    """deal ``rows`` to the B columns: one row per column when B >= len(rows) (cycling), else several per column"""
    n = len(rows)
    if B >= n:
        return [[rows[b % n]] for b in range(B)]
    return [rows[b::B] for b in range(B)]


Probe = collections.namedtuple("Probe", "op family T B inputs params exact marks")


def _marks_to_mask(marks, T, B):
    m = np.zeros((T, B), dtype=bool)
    for b, rows in enumerate(marks):
        m[rows, b] = True
    return m


def _gae_d(T, lam):
    """GAE's per-row denominators d_t (oracle.c gae_denoms), rounded to fp32"""
    d = np.empty(T, dtype=np.float64)
    den = 0.0
    for t in range(T - 1, -1, -1):
        den = 1.0 + lam * den
        d[t] = den
    return d.astype(np.float32)


def make_probe(op, family, T, B, seed=0):
    """the inputs of one probe; ``marks[b]`` lists column b's impulse or break rows (for failure messages)"""
    g = np.random.default_rng(seed * 1000003 + T * 7919 + B)
    f32 = np.float32
    exact = family != "random"
    base = family[:-2] if family.endswith("_w") else family
    marks = [[] for _ in range(B)]
    if base == "impulse":
        marks = column_rows(impulse_rows(T, B), B)
    elif base == "break":
        # one edge row per column; a batch narrower than the edge list gets several, so that even B = 1 has breaks
        # in segments whose aggregate A a successor reads (row L-1 alone zeroes the A of segment 0, which is the
        # last one the reverse-time scans reach)
        marks = column_rows(segment_edges(T, B) or [T // 2], B)
    hit = _marks_to_mask(marks, T, B)

    def dense(lo, hi, shape=(T, B)):
        return g.integers(lo, hi + 1, shape).astype(f32)

    def spikes(v):
        return np.where(hit, f32(v), f32(0))

    def value_rows(inner):  # (T+1, B): `inner` on rows 0..T-1, row T chosen per family
        last = {"impulse": np.full((1, B), 2, f32), "random": g.standard_normal((1, B), dtype=f32)}.get(
            base, dense(-3, 3, (1, B)))
        return np.concatenate([inner, last], axis=0)

    inputs, params = {}, {}
    if op in ("gae", "td_lambda", "vtrace"):
        if base == "impulse":
            reward, value = spikes(3), value_rows(spikes(-1))
        elif base == "random":
            reward, value = g.standard_normal((T, B), dtype=f32), value_rows(g.standard_normal((T, B), dtype=f32))
        else:
            reward, value = dense(-3, 3), value_rows(dense(-3, 3))
        inputs.update(value=value, reward=reward)
    if op == "gae":
        lam = 0.0 if base == "zero" else 1.0
        params.update(gamma=1.0, lambda_=lam)
        d = _gae_d(T, lam)[:, None]
        if base == "impulse":
            gadv = np.where(hit, d, f32(0)).astype(f32)  # G_p = d_p: G/d is exactly 1
        elif base == "random":
            gadv = g.standard_normal((T, B), dtype=f32)
        else:
            gadv = dense(-3, 3)
        inputs.update(grad_adv=gadv)
    elif op == "td_lambda":
        params.update(gamma=0.0 if base == "zero" else 1.0, lambda_=1.0)
        inputs.update(weight=np.ones((T, B), f32) if family.endswith("_w") or base == "random" else None)
    elif op == "vtrace":
        params.update(gamma=1.0, lambda_=0.0 if base == "zero" else 1.0, rho_clip_ratio=1.0, c_clip_ratio=1.0,
                      rho_pg_clip_ratio=1.0)
        action = g.integers(0, N_ACT, (T, B)).astype(np.int64)
        target = np.zeros((T, B, N_ACT), f32)
        behaviour = target.copy()
        # the behaviour logit of the taken action 3 below the target's: every importance ratio is about 11, so the
        # clipped ratios (and the coefficient gamma*lambda*min(c_bar, rho)) are exactly the clip constants
        np.put_along_axis(behaviour, action[..., None], f32(-3), axis=2)
        inputs.update(target_output=target, behaviour_output=behaviour, action=action,
                      weight=np.ones((T, B), f32) if family.endswith("_w") or base == "random" else None)
    elif op == "upgo":
        # bootstrap values 0: the flag of step t is [r_{t+1} >= 0]
        if base == "impulse":
            rewards = spikes(3)
        elif base == "random":
            rewards = np.abs(g.standard_normal((T, B), dtype=f32))
        elif base == "zero":
            rewards = -dense(1, 3)  # every r_{t+1} < 0: every flag 0
        else:
            rewards = dense(0, 3)
            for b, rows in enumerate(marks):  # flag 0 exactly at the break row
                for r in rows:
                    if r + 1 < T:
                        rewards[r + 1, b] = -1
        action = g.integers(0, N_ACT, (T, B)).astype(np.int64)
        inputs.update(target_output=np.zeros((T, B, N_ACT), f32), rhos=np.ones((T, B), f32), action=action,
                      rewards=rewards, bootstrap_values=np.zeros((T + 1, B), f32))
    elif op == "gae_episodic":
        params.update(gamma=1.0, lambda_=1.0)
        if base == "impulse":
            value, next_value, reward, gadv = spikes(-1), spikes(2), spikes(3), spikes(1)
        elif base == "random":
            value, next_value, reward, gadv = (g.standard_normal((T, B), dtype=f32) for _ in range(4))
        else:
            value, next_value, reward, gadv = (dense(-3, 3) for _ in range(4))
        done = np.zeros((T, B), bool)
        traj = np.zeros((T, B), bool)
        if base == "zero":
            traj[:] = True
        elif base == "break":
            done = hit.copy()
            traj = hit.copy()
        inputs.update(value=value, next_value=next_value, reward=reward, grad_adv=gadv, done=done, traj_flag=traj)
    return Probe(op, family, T, B, inputs, params, exact, marks)


def reference(p, dtype):
    """-> (scan, out, loss) of probe ``p`` through the CPU oracle in ``dtype`` (see the module docstring)"""
    dt = np.dtype(dtype).type
    x = {k: (v.astype(dt) if isinstance(v, np.ndarray) and v.dtype.kind == "f" else v) for k, v in p.inputs.items()}
    T, B, hp = p.T, p.B, p.params
    n = float(T) * float(B)
    f32 = dt is np.float32
    scan, out, loss = {}, {}, {}
    if p.op == "gae":
        adv = orc.gae_forward(x["value"], x["reward"], hp["gamma"], hp["lambda_"])
        ob = orc.gae_backward(x["grad_adv"], hp["gamma"], hp["lambda_"])
        scan = dict(adv=adv, grad_value=ob["value"], grad_reward=ob["reward"])
        out = dict(scan)
    elif p.op == "td_lambda":
        o = orc.td_lambda(x["value"], x["reward"], x["weight"], hp["gamma"], hp["lambda_"], 1.0)
        w = dt(1) if x["weight"] is None else x["weight"]
        scan = dict(ret=o["ret"])
        # kernel: grad_buf = float(-1/n) * (w * (ret - v))
        wd = w * (o["ret"] - x["value"][:T])
        out = dict(grad_buf=(np.float32(-1.0 / n) * wd) if f32 else -wd / n)
        loss = dict(loss=float(o["loss"]))
    elif p.op == "vtrace":
        o = orc.vtrace(x["target_output"], x["behaviour_output"], x["action"], x["value"], x["reward"], x["weight"],
                       want_grad=False, **hp)
        w = dt(1) if x["weight"] is None else x["weight"]
        scan = dict(ret=o["ret"], adv=o["adv"])
        inv_n = np.float32(1.0 / n) if f32 else 1.0 / n
        # kernel: pg_coef = -(adv * w) * inv_n;  gv_buf = 2 * ((v - ret) * w) * inv_n
        out = dict(pg_coef=-(o["adv"] * w) * inv_n, gv_buf=(dt(2) * ((x["value"][:T] - o["ret"]) * w)) * inv_n)
        loss = dict(policy_loss=float(o["policy_loss"]), value_loss=float(o["value_loss"]),
                    entropy_loss=float(o["entropy_loss"]))
    elif p.op == "upgo":
        o = orc.upgo(x["target_output"], x["rhos"], x["action"], x["rewards"], x["bootstrap_values"], 1.0,
                     want_grad=False)
        scan = dict(ret=o["ret"])
        adv = x["rhos"] * (o["ret"] - x["bootstrap_values"][:T])
        out = dict(coef=adv * np.float32(-1.0 / n) if f32 else -adv / n)  # kernel: coef = adv * float(-1/n)
        loss = dict(loss=float(o["loss"]))
    elif p.op == "gae_episodic":
        adv = epi.forward(x["value"], x["next_value"], x["reward"], x["done"], x["traj_flag"], hp["gamma"],
                          hp["lambda_"], dtype=dt)
        ob = epi.backward(x["grad_adv"], x["done"], x["traj_flag"], hp["gamma"], hp["lambda_"], dtype=dt)
        scan = dict(adv=adv, grad_value=ob["value"], grad_next_value=ob["next_value"], grad_reward=ob["reward"])
        out = dict(scan)
    else:
        raise ValueError(p.op)
    return scan, out, loss
