"""Episode-aware GAE without a GPU: the numpy oracle pinned bit for bit to eager PyTorch of the formula (forward and
autograd), the C-ABI argument errors, the public API surface, and what the compiler made of the kernels."""
import inspect
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from tests import gae_episodic_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DENSITIES = [0.0, 0.01, 0.3, 1.0]
SHAPES = [(1, 1), (1, 7), (2, 3), (9, 5), (33, 4), (64, 17)]


def eager(value, next_value, reward, done, traj_flag, gamma, lambda_, dtype=torch.float32):
    """The formula as a user would write it in PyTorch: one op per term, a Python loop over T."""
    g = torch.tensor(gamma, dtype=torch.float64).to(dtype)
    gl = torch.tensor(gamma * lambda_, dtype=torch.float64).to(dtype)
    if traj_flag is None:
        traj_flag = done
    d = torch.zeros_like(reward) if done is None else (done != 0).to(dtype)
    tr = torch.zeros_like(reward) if traj_flag is None else (traj_flag != 0).to(dtype)
    nv = next_value * (1 - d)
    delta = (reward + g * nv) - value
    f = gl * (1 - tr)
    T = reward.shape[0]
    adv = [None] * T
    adv[T - 1] = delta[T - 1]
    for t in range(T - 2, -1, -1):
        adv[t] = delta[t] + f[t] * adv[t + 1]
    return torch.stack(adv)


def make(T, B, density, traj_mode, seed, dtype=np.float32):
    g = np.random.default_rng(seed)
    value, next_value, reward, gadv = (g.standard_normal((T, B)).astype(dtype) for _ in range(4))
    done = g.random((T, B)) < density
    traj = {"same": done, "none": None, "other": g.random((T, B)) < max(density, 0.2)}[traj_mode]
    return value, next_value, reward, gadv, done, traj


def run_eager(value, next_value, reward, gadv, done, traj, gamma, lambda_, dtype):
    v, nv, r = (torch.from_numpy(x).requires_grad_(True) for x in (value, next_value, reward))
    d = torch.from_numpy(done)
    tr = None if traj is None else torch.from_numpy(traj)
    adv = eager(v, nv, r, d, tr, gamma, lambda_, dtype)
    adv.backward(torch.from_numpy(gadv))
    return adv.detach().numpy(), v.grad.numpy(), nv.grad.numpy(), r.grad.numpy()


@pytest.mark.parametrize("T,B", SHAPES)
@pytest.mark.parametrize("density", DENSITIES)
@pytest.mark.parametrize("traj_mode", ["same", "none", "other"])
def test_oracle_pinned_to_eager_torch(T, B, density, traj_mode):
    value, next_value, reward, gadv, done, traj = make(T, B, density, traj_mode, T * 1000 + B)
    gamma, lambda_ = 0.99, 0.95
    adv, gv, gnv, gr = run_eager(value, next_value, reward, gadv, done, traj, gamma, lambda_, torch.float32)
    want = orc.forward(value, next_value, reward, done, traj, gamma, lambda_)
    wb = orc.backward(gadv, done, traj, gamma, lambda_)
    assert want.dtype == np.float32 and np.array_equal(adv, want)
    assert np.array_equal(gv, wb["value"])
    assert np.array_equal(gnv, wb["next_value"])
    assert np.array_equal(gr, wb["reward"])
    # the fp64 restatement against eager fp64
    v64, nv64, r64, g64 = (x.astype(np.float64) for x in (value, next_value, reward, gadv))
    adv, gv, gnv, gr = run_eager(v64, nv64, r64, g64, done, traj, gamma, lambda_, torch.float64)
    want = orc.forward(v64, nv64, r64, done, traj, gamma, lambda_, dtype=np.float64)
    wb = orc.backward(g64, done, traj, gamma, lambda_, dtype=np.float64)
    scale = max(1.0, float(np.abs(want).max()))
    assert np.abs(adv - want).max() <= 1e-12 * scale
    for got, k in ((gv, "value"), (gnv, "next_value"), (gr, "reward")):
        assert np.abs(got - wb[k]).max() <= 1e-12 * max(1.0, float(np.abs(wb[k]).max()))


def test_oracle_semantics_by_hand():
    """done masks the bootstrap of its own step, traj_flag cuts the recursion after its step."""
    value = np.array([[1.0], [2.0], [3.0]], np.float32)
    next_value = np.array([[10.0], [20.0], [30.0]], np.float32)
    reward = np.zeros((3, 1), np.float32)
    done = np.array([[0], [1], [0]], np.uint8)
    g, lam = 0.5, 0.5
    adv = orc.forward(value, next_value, reward, done, None, g, lam, dtype=np.float64)
    d2 = 0.5 * 30 - 3
    d1 = 0.0 - 2  # done: no bootstrap, and (traj_flag = done) no carry from row 2
    d0 = 0.5 * 10 - 1
    assert np.allclose(adv[:, 0], [d0 + 0.25 * d1, d1, d2])
    adv = orc.forward(value, next_value, reward, done, np.zeros_like(done), g, lam, dtype=np.float64)
    assert np.allclose(adv[:, 0], [d0 + 0.25 * (d1 + 0.25 * d2), d1 + 0.25 * d2, d2])
    # a fractional float mask counts as set
    half = done.astype(np.float32) * 0.5
    assert np.array_equal(orc.forward(value, next_value, reward, half, None, g, lam),
                          orc.forward(value, next_value, reward, done, None, g, lam))


def test_abi_argument_errors():
    from di_hpc_b200 import _abi
    L = _abi.lib()
    fwd, bwd = L.hpc_rll_gae_episodic_forward, L.hpc_rll_gae_episodic_backward
    assert fwd(None, None, None, None, None, None, 4, 4, 0.99, 0.97, None) == 1
    msg = L.hpc_rll_last_error()
    assert b"null" in msg and b"done" not in msg and b"traj" not in msg  # masks may be NULL
    assert fwd(None, None, None, None, None, None, -1, 4, 0.99, 0.97, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    assert fwd(None, None, None, None, None, None, 4, -1, 0.99, 0.97, None) == 1
    assert bwd(None, None, None, None, None, None, 4, 4, 0.99, 0.97, None) == 1
    msg = L.hpc_rll_last_error()
    assert b"null" in msg and b"done" not in msg and b"traj" not in msg
    assert bwd(None, None, None, None, None, None, -3, 4, 0.99, 0.97, None) == 1
    assert bwd(None, None, None, None, None, None, 4, -3, 0.99, 0.97, None) == 1
    # empty problems: nothing to launch, NULL masks and data accepted
    for T, B in ((0, 4), (4, 0), (0, 0)):
        assert fwd(None, None, None, None, None, None, T, B, 0.99, 0.97, None) == 0
        assert bwd(None, None, None, None, None, None, T, B, 0.99, 0.97, None) == 0
    assert _abi.OP_GAE_EPISODIC == 10
    assert L.hpc_rll_debug_set_config(_abi.OP_GAE_EPISODIC, -1) == 0
    assert L.hpc_rll_debug_set_config(11, 0) == 1


def test_api_surface():
    import hpc_rll.rl_utils.gae as mod
    from di_hpc_b200.rl_utils import gae as impl
    assert mod.gae is impl.gae and mod.gae_data is impl.gae_data
    params = inspect.signature(mod.gae).parameters
    assert list(params) == ["data", "gamma", "lambda_"]
    assert params["gamma"].default == 0.99 and params["lambda_"].default == 0.97
    assert mod.gae_data._fields == ("value", "next_value", "reward", "done", "traj_flag")
    # the normalised GAE module keeps its exact reference signature
    assert [p for p in inspect.signature(mod.GAE.forward).parameters if p != "self"] == \
        ["value", "reward", "gamma", "lambda_"]


def test_multi_agent_value_is_rejected():
    from hpc_rll.rl_utils.gae import gae, gae_data
    z = torch.zeros(4, 3, 2)
    with pytest.raises(ValueError, match="multi-agent"):
        gae(gae_data(z, z, torch.zeros(4, 3), None, None))


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
    mine = {k: c for k, c in kernels.items() if "gae_episodic" in k}
    wide = [k for k in mine if "_tma" in k]
    assert len([k for k in wide if "fwd" in k]) >= 1 and len([k for k in wide if "bwd" in k]) >= 1
    for k in wide:  # TMA-staged inputs and outputs
        assert mine[k]["UTMALDG"] > 0 and mine[k]["UTMASTG"] > 0 and mine[k]["SYNCS"] > 0, (k, dict(mine[k]))
    lookback = [k for k in mine if "lookback" in k]
    assert any("fwd" in k for k in lookback) and any("bwd" in k for k in lookback)
    for k in mine:
        if k in atomics:
            assert "lookback" in k and not any(".F" in op for op in atomics[k]), (k, atomics[k])
