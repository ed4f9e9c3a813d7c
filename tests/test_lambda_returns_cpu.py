"""λ-returns without a GPU: the numpy oracle pinned bit for bit to eager PyTorch of the formula (forward and autograd,
all eight γ / λ / done combinations), to the reference's origin (tests/golden/lambda_*.npz) and to the TD(lambda)
fixtures' returns; the C-ABI argument errors, the public API surface, and what the compiler made of the kernels."""
import inspect
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from tests import lambda_returns_oracle as orc
from tests._golden import GOLDEN_DIR, names

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

COMBOS = [(gt, lt, dn) for gt in (False, True) for lt in (False, True) for dn in (False, True)]
SHAPES = [(1, 1), (1, 6), (2, 3), (9, 5), (33, 4), (64, 17)]
GAMMA, LAMBDA = 0.99, 0.95


def eager(bootstrap, rewards, gammas, lambda_, done, offset):
    """The formula as a user would write it in PyTorch: one op per term, a Python loop over T."""
    if not isinstance(gammas, torch.Tensor):
        gammas = gammas * torch.ones_like(rewards)
    if not isinstance(lambda_, torch.Tensor):
        lambda_ = lambda_ * torch.ones_like(rewards)
    V = bootstrap[offset:]
    d = gammas * lambda_
    e = gammas - d
    T = rewards.shape[0]
    R = [None] * T
    if done is None:
        R[T - 1] = rewards[T - 1] + gammas[T - 1] * V[T - 1]
        for t in range(T - 2, -1, -1):
            R[t] = rewards[t] + d[t] * R[t + 1] + e[t] * V[t]
    else:
        m = 1 - (done != 0).float()
        R[T - 1] = rewards[T - 1] + (m[T - 1] * gammas[T - 1]) * V[T - 1]
        for t in range(T - 2, -1, -1):
            R[t] = rewards[t] + m[t] * (d[t] * R[t + 1] + e[t] * V[t])
    return torch.stack(R)


def make(T, B, gt, lt, dn, offset, seed, density=0.3):
    g = np.random.default_rng(seed)
    boot = g.standard_normal((T + offset, B)).astype(np.float32)
    rewards, G = (g.standard_normal((T, B)).astype(np.float32) for _ in range(2))
    gammas = (0.5 + 0.5 * g.random((T, B))).astype(np.float32) if gt else GAMMA
    lam = g.random((T, B)).astype(np.float32) if lt else LAMBDA
    done = (g.random((T, B)) < density) if dn else None
    return boot, rewards, G, gammas, lam, done


@pytest.mark.parametrize("T,B", SHAPES)
@pytest.mark.parametrize("gt,lt,dn", COMBOS)
@pytest.mark.parametrize("offset", [1, 0])
def test_oracle_pinned_to_eager_torch(T, B, gt, lt, dn, offset):
    boot, rewards, G, gammas, lam, done = make(T, B, gt, lt, dn, offset, T * 1000 + B)
    bt, rt = torch.from_numpy(boot).requires_grad_(True), torch.from_numpy(rewards).requires_grad_(True)
    as_t = (lambda x: torch.from_numpy(x) if isinstance(x, np.ndarray) else x)
    ret = eager(bt, rt, as_t(gammas), as_t(lam), None if done is None else torch.from_numpy(done), offset)
    ret.backward(torch.from_numpy(G))
    want = orc.forward(boot, rewards, gammas, lam, done, offset)
    wb = orc.backward(G, gammas, lam, done, offset)
    assert want.dtype == np.float32 and np.array_equal(ret.detach().numpy(), want)
    assert np.array_equal(bt.grad.numpy(), wb["bootstrap_values"])
    assert np.array_equal(rt.grad.numpy(), wb["rewards"])
    if offset == 1:  # the unread row gets +0, not -0
        assert not np.signbit(wb["bootstrap_values"][0]).any()


def test_oracle_semantics_by_hand():
    """done cuts both the bootstrap of its step and the recursion behind it; an all-zero mask is the done-free result
    up to association."""
    boot = np.array([[0.0], [10.0], [20.0], [30.0]], np.float32)
    rewards = np.array([[1.0], [2.0], [3.0]], np.float32)
    g, lam = 0.5, 0.5  # d = 0.25, e = 0.25
    R = orc.forward(boot, rewards, g, lam, None, 1, dtype=np.float64)
    r2 = 3 + 0.5 * 30
    r1 = 2 + 0.25 * r2 + 0.25 * 20
    assert np.allclose(R[:, 0], [1 + 0.25 * r1 + 0.25 * 10, r1, r2])
    done = np.array([[0], [1], [0]], np.uint8)
    R = orc.forward(boot, rewards, g, lam, done, 1, dtype=np.float64)
    assert np.allclose(R[:, 0], [1 + 0.25 * 2 + 0.25 * 10, 2, r2])
    zero = np.zeros_like(done)
    assert np.allclose(orc.forward(boot, rewards, g, lam, zero, 1), orc.forward(boot, rewards, g, lam, None, 1))
    # a fractional float mask counts as set
    half = done.astype(np.float32) * 0.5
    assert np.array_equal(orc.forward(boot, rewards, g, lam, half, 1), orc.forward(boot, rewards, g, lam, done, 1))


@pytest.mark.parametrize("name", names("lambda"))
def test_oracle_matches_origin_fixtures(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    off = int(z["offset"])
    gam, lam = z["in_gammas"], z["in_lambda_"]
    gam = float(gam) if gam.ndim == 0 else gam
    lam = float(lam) if lam.ndim == 0 else lam
    assert np.array_equal(orc.forward(z["in_bootstrap_values"], z["in_rewards"], gam, lam, None, off), z["out"])
    wb = orc.backward(z["in_grad"], gam, lam, None, off)
    assert np.array_equal(wb["bootstrap_values"], z["grad_bootstrap_values"])
    assert np.array_equal(wb["rewards"], z["grad_rewards"])


@pytest.mark.parametrize("name", names("tdlambda"))
def test_oracle_matches_td_lambda_returns(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    R = orc.forward(z["in_value"], z["in_reward"], float(z["attr_gamma"]), float(z["attr_lambda_"]), None, 1)
    assert np.array_equal(R, z["out32_ret"])


def test_abi_argument_errors():
    from di_hpc_b200 import _abi
    L = _abi.lib()
    fwd, bwd = L.hpc_rll_lambda_returns_forward, L.hpc_rll_lambda_returns_backward
    assert fwd(None, None, None, None, None, None, 4, 4, 1, GAMMA, LAMBDA, None) == 1
    msg = L.hpc_rll_last_error()
    assert b"null" in msg and b"gamma" not in msg and b"done" not in msg  # gammas / lambdas / done may be NULL
    assert fwd(None, None, None, None, None, None, -1, 4, 1, GAMMA, LAMBDA, None) == 1
    assert b"negative" in L.hpc_rll_last_error()
    assert fwd(None, None, None, None, None, None, 4, -1, 0, GAMMA, LAMBDA, None) == 1
    assert fwd(None, None, None, None, None, None, 4, 4, 2, GAMMA, LAMBDA, None) == 1
    assert b"bootstrap_offset" in L.hpc_rll_last_error()
    assert bwd(None, None, None, None, None, None, 4, 4, 0, GAMMA, LAMBDA, None) == 1
    msg = L.hpc_rll_last_error()
    assert b"null" in msg and b"gamma" not in msg and b"done" not in msg
    assert bwd(None, None, None, None, None, None, -3, 4, 1, GAMMA, LAMBDA, None) == 1
    assert bwd(None, None, None, None, None, None, 4, -3, 1, GAMMA, LAMBDA, None) == 1
    # empty problems: nothing to launch, NULL pointers accepted
    for T, B in ((0, 4), (4, 0), (0, 0)):
        for off in (0, 1):
            assert fwd(None, None, None, None, None, None, T, B, off, GAMMA, LAMBDA, None) == 0
            assert bwd(None, None, None, None, None, None, T, B, off, GAMMA, LAMBDA, None) == 0
    assert _abi.OP_LAMBDA_RETURNS == 11
    for cfg in (-1, 21, 33, 99):
        assert L.hpc_rll_debug_set_config(_abi.OP_LAMBDA_RETURNS, cfg) == 0
    assert L.hpc_rll_debug_set_config(_abi.OP_LAMBDA_RETURNS, 7) == 1
    assert b"unknown config" in L.hpc_rll_last_error()
    assert L.hpc_rll_debug_set_config(_abi.OP_LAMBDA_RETURNS, -1) == 0
    assert L.hpc_rll_debug_set_config(12, -1) == 1


def test_api_surface():
    import hpc_rll.rl_utils.td as mod
    from di_hpc_b200.rl_utils import td as impl
    for fn in ("generalized_lambda_returns", "multistep_forward_view"):
        assert getattr(mod, fn) is getattr(impl, fn)
        params = inspect.signature(getattr(mod, fn)).parameters
        assert list(params) == ["bootstrap_values", "rewards", "gammas", "lambda_", "done"]
        assert params["done"].default is None
        assert all(params[p].default is inspect.Parameter.empty for p in list(params)[:4])


@pytest.mark.parametrize("fn", ["generalized_lambda_returns", "multistep_forward_view"])
def test_discount_arguments_are_checked_before_any_call(fn):
    import hpc_rll.rl_utils.td as mod
    f = getattr(mod, fn)
    r = torch.zeros(3, 2)
    v = torch.zeros(4 if fn == "generalized_lambda_returns" else 3, 2)
    with pytest.raises(ValueError, match="gammas"):
        f(v, r, torch.ones(3, 2, requires_grad=True), 0.9)
    with pytest.raises(ValueError, match="lambda_"):
        f(v, r, 0.9, torch.ones(3, 2, requires_grad=True))
    with pytest.raises(TypeError, match="gammas"):
        f(v, r, "0.9", 0.9)
    with pytest.raises(TypeError, match="lambda_"):
        f(v, r, 0.9, [0.9])


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
    mine = {k: c for k, c in kernels.items() if "lambda_ret_" in k}
    readable = dict(zip(sass_opcodes.demangle(list(mine)), mine))
    flags = ["<%s, %s, %s" % c for c in (tuple(str(x).lower() for x in combo) for combo in COMBOS)]
    want = {"lambda_ret_fwd_lookback", "lambda_ret_bwd_lookback"}
    for f in flags:
        want |= {"lambda_ret_fwd_generic%s>" % f, "lambda_ret_bwd_generic%s>" % f,
                 "lambda_ret_fwd_tma%s, 256, 4, 5>" % f, "lambda_ret_bwd_tma%s, 256, 4, 6>" % f}
    assert set(readable) == want, set(readable) ^ want
    for name, k in readable.items():
        if "_tma" in name:  # TMA-staged inputs and outputs
            c = mine[k]
            assert c["UTMALDG"] > 0 and c["UTMASTG"] > 0 and c["SYNCS"] > 0, (name, dict(c))
        if k in atomics:
            assert "lookback" in name and not any(".F" in op for op in atomics[k]), (name, atomics[k])
