"""V-trace and UPGO returns without a GPU: the numpy oracle pinned to the reference's origin
(tests/golden/returns_*.npz) and to the returns stored in the UPGO loss fixtures; the C-ABI argument errors, the public
API surface, the ValueError for ratios that require grad, and what the compiler made of the kernels."""
import inspect
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from tests import vtrace_upgo_returns_oracle as orc
from tests._golden import GOLDEN_DIR, names

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GAMMA, LAMBDA = 0.99, 0.95


def load(name):
    return np.load(os.path.join(GOLDEN_DIR, name + ".npz"))


@pytest.mark.parametrize("name", names("returns_vtrace"))
def test_vtrace_oracle_matches_origin_fixtures(name):
    """forward and grad_reward bit for bit; grad_V to 1e-6 relative, because autograd does not fix the order in which
    it adds V_t's three contributions"""
    z = load(name)
    g, lam = float(z["attr_gamma"]), float(z["attr_lambda_"])
    rho, c = z["in_clipped_rhos"], z["in_clipped_cs"]
    assert (rho == 1.0).any() and (rho < 1.0).any()  # ratios on and below the clip
    R = orc.vtrace_forward(rho, c, z["in_reward"], z["in_bootstrap_values"], g, lam)
    assert R.dtype == np.float32 and np.array_equal(R, z["out"])
    wb = orc.vtrace_backward(z["in_grad"], rho, c, g, lam)
    assert np.array_equal(wb["reward"], z["grad_reward"])
    want = z["grad_bootstrap_values"]
    assert np.allclose(wb["bootstrap_values"], want, rtol=1e-6, atol=1e-6 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("name", names("returns_upgo"))
def test_upgo_oracle_matches_origin_fixtures(name):
    z = load(name)
    r, V = z["in_rewards"], z["in_bootstrap_values"]
    assert np.array_equal(orc.upgo_forward(r, V), z["out"])
    wb = orc.upgo_backward(z["in_grad"], orc.upgo_mask(r, V))
    assert np.array_equal(wb["rewards"], z["grad_rewards"])
    assert np.array_equal(wb["bootstrap_values"], z["grad_bootstrap_values"])
    assert not np.signbit(wb["bootstrap_values"][0]).any()
    if "tie" in name and r.shape[0] > 2:  # the fixture exercises r_{t+1} + V_{t+2} == V_{t+1}
        assert ((r[1:] + V[2:]) == V[1:-1]).any()


@pytest.mark.parametrize("name", names("upgo"))
def test_upgo_oracle_matches_upgo_loss_fixtures(name):
    z = load(name)
    assert np.array_equal(orc.upgo_forward(z["in_rewards"], z["in_bootstrap_values"]), z["out32_ret"])


def test_oracle_semantics_by_hand():
    V = np.array([[0.0], [10.0], [20.0], [30.0]])
    r = np.array([[1.0], [2.0], [3.0]])
    # V-trace with ρ = c = 1 is the λ-return of the TD errors
    one = np.ones_like(r)
    g, lam = 0.5, 0.5
    d = [(r[t, 0] + g * V[t + 1, 0]) - V[t, 0] for t in range(3)]
    item2 = d[2]
    item1 = d[1] + g * lam * item2
    item0 = d[0] + g * lam * item1
    R = orc.vtrace_forward(one, one, r, V, g, lam, dtype=np.float64)
    assert np.allclose(R[:, 0], [item0, item1 + 10, item2 + 20])
    # UPGO: ℓ_0 = [r_1 + V_2 >= V_1] = [22 >= 10] = 1, ℓ_1 = [r_2 + V_3 >= V_2] = [33 >= 20] = 1
    R = orc.upgo_forward(r, V, dtype=np.float64)
    assert np.allclose(R[:, 0], [1 + 2 + 3 + 30, 2 + 3 + 30, 3 + 30])
    V2 = np.array([[0.0], [50.0], [20.0], [30.0]])  # ℓ_0 = [22 >= 50] = 0: R_0 bootstraps from V_1
    R = orc.upgo_forward(r, V2, dtype=np.float64)
    assert np.allclose(R[:, 0], [1 + 50, 2 + 3 + 30, 3 + 30])
    nan = V2.copy()
    nan[2, 0] = np.nan  # a NaN comparison gives ℓ = 0
    assert orc.upgo_mask(r, nan, np.float64)[:, 0].tolist() == [0.0, 0.0, 0.0]


def test_abi_argument_errors():
    from di_hpc_b200 import _abi
    L = _abi.lib()
    vf, vb = L.hpc_rll_vtrace_return_forward, L.hpc_rll_vtrace_return_backward
    uf, ub = L.hpc_rll_upgo_returns_forward, L.hpc_rll_upgo_returns_backward
    assert vf(None, None, None, None, None, 4, 4, GAMMA, LAMBDA, None) == 1
    assert b"null" in L.hpc_rll_last_error()
    assert vf(None, None, None, None, None, -1, 4, GAMMA, LAMBDA, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    assert vb(None, None, None, None, None, 4, 4, GAMMA, LAMBDA, None) == 1
    assert b"null" in L.hpc_rll_last_error()
    assert vb(None, None, None, None, None, 4, -2, GAMMA, LAMBDA, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    assert uf(None, None, None, None, 4, 4, None) == 1
    msg = L.hpc_rll_last_error()
    assert b"null" in msg and b"lambda_mask" not in msg  # the mask may be NULL: not saved
    assert uf(None, None, None, None, -3, 4, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    assert ub(None, None, None, None, 4, 4, None) == 1
    assert b"lambda_mask" in L.hpc_rll_last_error()  # the backward needs it
    assert ub(None, None, None, None, 4, -1, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    # empty problems: nothing to launch, NULL pointers accepted
    for T, B in ((0, 4), (4, 0), (0, 0)):
        assert vf(None, None, None, None, None, T, B, GAMMA, LAMBDA, None) == 0
        assert vb(None, None, None, None, None, T, B, GAMMA, LAMBDA, None) == 0
        assert uf(None, None, None, None, T, B, None) == 0
        assert ub(None, None, None, None, T, B, None) == 0
    assert L.hpc_rll_launch_count() == 0


def test_api_surface():
    import hpc_rll.rl_utils.upgo as upgo
    import hpc_rll.rl_utils.vtrace as vtrace
    from di_hpc_b200.rl_utils import upgo as upgo_impl
    from di_hpc_b200.rl_utils import vtrace as vtrace_impl
    assert vtrace.vtrace_nstep_return is vtrace_impl.vtrace_nstep_return
    assert upgo.upgo_returns is upgo_impl.upgo_returns
    params = inspect.signature(vtrace.vtrace_nstep_return).parameters
    assert list(params) == ["clipped_rhos", "clipped_cs", "reward", "bootstrap_values", "gamma", "lambda_"]
    assert params["gamma"].default == 0.99 and params["lambda_"].default == 0.95
    assert all(params[p].default is inspect.Parameter.empty for p in list(params)[:4])
    params = inspect.signature(upgo.upgo_returns).parameters
    assert list(params) == ["rewards", "bootstrap_values"]
    assert all(p.default is inspect.Parameter.empty for p in params.values())


@pytest.mark.parametrize("which", ["clipped_rhos", "clipped_cs"])
def test_ratios_that_require_grad_are_refused_before_any_call(which):
    from hpc_rll.rl_utils.vtrace import vtrace_nstep_return
    args = {"clipped_rhos": torch.ones(3, 2), "clipped_cs": torch.ones(3, 2)}
    args[which] = args[which].requires_grad_(True)
    with pytest.raises(ValueError, match=which):
        vtrace_nstep_return(args["clipped_rhos"], args["clipped_cs"], torch.zeros(3, 2), torch.zeros(4, 2))


@pytest.fixture(scope="module")
def sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    sys.path.insert(0, ROOT)
    from di_hpc_b200 import build
    from tools import sass_opcodes
    kernels, atomics, _ = sass_opcodes.parse(build.build())
    return kernels, atomics


def test_kernels_are_what_the_design_says(sass):
    kernels, atomics = sass
    from tools import sass_opcodes
    mine = {k: c for k, c in kernels.items() if "vtrace_ret_" in k or "upgo_ret_" in k}
    readable = dict(zip(sass_opcodes.demangle(list(mine)), mine))
    want = set()
    for op in ("vtrace_ret", "upgo_ret"):
        want |= {op + "_fwd_lookback", op + "_bwd_lookback", op + "_fwd_generic", op + "_bwd_generic",
                 op + "_fwd_tma<256, 4, 5>", op + "_bwd_tma<256, 4, 6>"}
    assert set(readable) == want, set(readable) ^ want
    for name, k in readable.items():
        c = mine[k]
        if "_tma" in name:  # TMA-staged inputs and outputs
            assert c["UTMALDG"] > 0 and c["UTMASTG"] > 0 and c["SYNCS"] > 0, (name, dict(c))
        if k in atomics:
            assert "lookback" in name and not any(".F" in op for op in atomics[k]), (name, atomics[k])
