"""Importance weights and the time-batch cross entropy without a GPU: the fp64 numpy oracle pinned to the reference's
origin (tests/golden/importance_*.npz), the C-ABI argument errors, the tuning configs op 12 refuses, the public API
surface with origin's asserts, and the row kernels built for the importance-weights forward."""
import inspect
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from tests import importance_weights_oracle as orc
from tests import row_paths as rp
from tests._golden import GOLDEN_DIR, grad_err, names, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-6  # fp32 origin against the fp64 oracle


def load(name):
    return np.load(os.path.join(GOLDEN_DIR, name + ".npz"))


@pytest.mark.parametrize("name", names("importance_is"))
def test_importance_oracle_matches_origin_fixtures(name):
    z = load(name)
    o = orc.importance_weights(z["in_target_output"], z["in_behaviour_output"], z["in_action"], z["in_grad"])
    assert o["out"].shape == z["out"].shape == z["in_action"].shape
    assert rel_err(o["out"], z["out"]) <= TOL
    for k in ("grad_target_output", "grad_behaviour_output"):
        assert grad_err(o[k], z[k]) <= TOL, k
        masked = np.isinf(z["in_" + k[5:]])
        assert (z[k][masked] == 0).all() and (o[k][masked] == 0).all(), k
    if "same" in name:
        assert (z["out"] == 1).all() and (o["out"] == 1).all()
    if "_n1_" in name:
        assert (z["out"] == 1).all() and not z["grad_target_output"].any() and not o["grad_target_output"].any()
    if "masked" in name:
        assert np.isinf(z["in_target_output"]).any() and np.isinf(z["in_behaviour_output"]).any()


@pytest.mark.parametrize("name", names("importance_ce"))
def test_cross_entropy_oracle_matches_origin_fixtures(name):
    z = load(name)
    o = orc.tb_cross_entropy(z["in_logit"], z["in_label"], z["in_grad"])
    assert o["out"].shape == z["out"].shape == z["in_label"].shape
    assert rel_err(o["out"], z["out"]) <= TOL
    assert grad_err(o["grad_logit"], z["grad_logit"]) <= TOL
    masked = np.isinf(z["in_logit"])
    assert (z["grad_logit"][masked] == 0).all() and (o["grad_logit"][masked] == 0).all()


def test_oracle_by_hand():
    t = np.array([[0.0, np.log(3.0)]])  # p = (1/4, 3/4)
    b = np.array([[0.0, 0.0]])  # p = (1/2, 1/2)
    o = orc.importance_weights(t, b, np.array([1]), np.array([2.0]))
    assert np.isclose(o["out"][0], 1.5)
    assert np.allclose(o["grad_target_output"], 2.0 * 1.5 * np.array([[-0.25, 0.25]]))
    assert np.allclose(o["grad_behaviour_output"], -2.0 * 1.5 * np.array([[-0.5, 0.5]]))
    o = orc.tb_cross_entropy(t, np.array([[0]]), np.array([[1.0]]))
    assert np.isclose(o["out"][0, 0], np.log(0.25)) and np.allclose(o["grad_logit"], [[0.75, -0.75]])


def test_abi_argument_errors():
    from di_hpc_b200 import _abi
    L = _abi.lib()
    f, b = L.hpc_rll_importance_weights_forward, L.hpc_rll_importance_weights_backward
    cf, cb = L.hpc_rll_tb_cross_entropy_forward, L.hpc_rll_tb_cross_entropy_backward
    P = 256  # a non-null stand-in: every check below fails before a pointer is read
    assert f(None, None, None, None, 4, 3, None) == 1
    assert b"null" in L.hpc_rll_last_error()
    assert f(P, P, P, P, -1, 3, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    for N in (0, -2, 1 << 30):
        assert f(P, P, P, P, 4, N, None) == 1
        assert b"N" in L.hpc_rll_last_error()
        assert b(P, P, P, P, P, P, P, 4, N, P, 1 << 20, None) == 1
        assert cf(P, P, P, 4, N, None) == 1
        assert cb(P, P, P, P, 4, N, None) == 1
    assert b(None, P, P, P, P, P, None, 4, 3, P, 1 << 20, None) == 1
    assert b"null" in L.hpc_rll_last_error()
    assert b(P, None, P, P, P, P, None, 4, 3, P, 1 << 20, None) == 1  # target_output needed for its gradient
    assert b"target_output" in L.hpc_rll_last_error()
    assert b(P, P, None, P, P, None, P, 4, 3, P, 1 << 20, None) == 1
    assert b"behaviour_output" in L.hpc_rll_last_error()
    assert b(P, P, P, P, P, P, P, -3, 3, P, 1 << 20, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    need = L.hpc_rll_workspace_bytes(_abi.OP_IMPORTANCE_WEIGHTS, 1000, 1, 7)
    assert need >= 1000 * 4
    assert b(P, P, P, P, P, P, P, 1000, 7, P, need - 1, None) == 1
    assert b"workspace" in L.hpc_rll_last_error()
    assert cf(None, P, P, 4, 3, None) == 1 and b"null" in L.hpc_rll_last_error()
    assert cf(P, P, P, -4, 3, None) == 1 and b"negative" in L.hpc_rll_last_error()
    assert cb(P, P, None, P, 4, 3, None) == 1 and b"null" in L.hpc_rll_last_error()
    assert cb(P, P, P, P, -4, 3, None) == 1 and b"negative" in L.hpc_rll_last_error()
    # nothing to do: no rows, or (backward) no gradient wanted; NULL pointers accepted
    assert f(None, None, None, None, 0, 3, None) == 0
    assert b(None, None, None, None, None, None, None, 0, 3, None, 0, None) == 0
    assert b(None, None, None, None, None, None, None, 4, 3, None, 0, None) == 0
    assert cf(None, None, None, 0, 3, None) == 0
    assert cb(None, None, None, None, 0, 3, None) == 0
    assert L.hpc_rll_launch_count() == 0


def test_debug_set_config_refuses_every_config():
    """op 12 sizes a workspace only: no config can be forced for it, automatic included"""
    from di_hpc_b200 import _abi
    L = _abi.lib()
    assert _abi.OP_IMPORTANCE_WEIGHTS == 12
    for cfg in (-1, 0, 1, 2, 21, 33, 99, -2):
        assert L.hpc_rll_debug_set_config(_abi.OP_IMPORTANCE_WEIGHTS, cfg) == 1
        assert b"unknown config" in L.hpc_rll_last_error()
    assert L.hpc_rll_debug_set_config(13, -1) == 1  # HPC_RLL_OP_COUNT


def test_api_surface():
    import hpc_rll.rl_utils.upgo as upgo
    import hpc_rll.rl_utils.vtrace as vtrace
    from di_hpc_b200.rl_utils import upgo as upgo_impl
    from di_hpc_b200.rl_utils import vtrace as vtrace_impl
    assert vtrace.compute_importance_weights is vtrace_impl.compute_importance_weights
    assert upgo.tb_cross_entropy is upgo_impl.tb_cross_entropy
    params = inspect.signature(vtrace.compute_importance_weights).parameters
    assert list(params) == ["target_output", "behaviour_output", "action", "requires_grad"]
    assert params["requires_grad"].default is False
    assert all(params[p].default is inspect.Parameter.empty for p in list(params)[:3])
    params = inspect.signature(upgo.tb_cross_entropy).parameters
    assert list(params) == ["logit", "label", "mask"]
    assert params["mask"].default is None
    assert all(params[p].default is inspect.Parameter.empty for p in ("logit", "label"))


def test_origin_asserts():
    from hpc_rll.rl_utils.upgo import tb_cross_entropy
    from hpc_rll.rl_utils.vtrace import compute_importance_weights
    x = torch.zeros(3, 2, 4)
    with pytest.raises(AssertionError):
        compute_importance_weights(x, x, [[0, 1], [1, 0], [0, 0]])  # action must be a tensor
    with pytest.raises(AssertionError):
        tb_cross_entropy(x.reshape(6, 4), torch.zeros(6, dtype=torch.long))  # 1-D label
    with pytest.raises(AssertionError):
        tb_cross_entropy(x.reshape(3, 2, 1, 4), torch.zeros(3, 2, 1, dtype=torch.long))  # 3-D label
    with pytest.raises(AssertionError):
        tb_cross_entropy(x, torch.zeros(3, 2, dtype=torch.long), mask=torch.ones(3, 2))


def test_built_importance_kernels_are_the_vtrace_forward_layouts():
    """the importance-weights forward reads the same two pointers as the V-trace forward, so the dispatch selects the
    same layouts: 34 register layouts, the staged and the looping kernel"""
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not on PATH")
    import re
    sys.path.insert(0, ROOT)
    from di_hpc_b200 import build
    from tools import sass_opcodes
    kernel = re.compile(r"importance_rows_fwd(?:_(staged|loop))?(?:<(\d+), (\d+), (true|false)>)?$")
    built = []
    names_ = sass_opcodes.demangle(list(sass_opcodes.listing(build.build())))
    for name in names_:
        m = kernel.match(name)
        if m:
            path, kmax, width, g1 = m.groups()
            built.append(("vtrace", path) if path else ("vtrace", int(width), g1 == "true", int(kmax)))
    assert len(built) == len(set(built)) == 36
    want = {k for k in rp.row_layouts() if k[0] == "vtrace"}
    assert set(built) == want, (sorted(set(built) - want, key=str), sorted(want - set(built), key=str))
    assert "importance_grad_coef" in names_
    assert not [n for n in names_ if n.startswith("importance_") and n != "importance_grad_coef"
                and not kernel.match(n)]
