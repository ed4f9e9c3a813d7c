"""ScatterConnection without a GPU: the fp32 oracle against origin's CPU output on the committed fixtures (bit-exact,
forward and grad_x), the C ABI's argument errors, and the Python surface of the drop-in module and the legacy names."""
import ctypes
import importlib
import inspect
import os

import numpy as np
import pytest
import torch

from tests._golden import GOLDEN_DIR, names

CASES = names("scatter")


def load(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return z, int(z["H"]), int(z["W"]), str(z["scatter_type"])


def test_fixtures_cover_both_modes_and_stay_small():
    assert {load(n)[3] for n in CASES} == {"cover", "add"}
    assert sum(os.path.getsize(os.path.join(GOLDEN_DIR, n + ".npz")) for n in CASES) < 1 << 20


@pytest.mark.parametrize("name", CASES)
def test_oracle_is_bit_exact_against_origin(name):
    from tests import scatter_oracle as orc
    z, H, W, mode = load(name)
    out = orc.scatter_connection_forward(z["in_x"], z["in_location"], H, W, mode)
    assert out.dtype == np.float32 and np.array_equal(out.view(np.uint32), z["out"].view(np.uint32)), name
    gx = orc.scatter_connection_backward(z["in_G"], z["in_location"])
    assert np.array_equal(gx.view(np.uint32), z["grad_x"].view(np.uint32)), name


def test_oracle_drops_out_of_range_entities():
    from tests import scatter_oracle as orc
    x = np.arange(1, 7, dtype=np.float32).reshape(1, 3, 2)
    loc = np.array([[[0, 1], [2, 0], [-1, 1]]], dtype=np.int64)  # H=2: the 2nd and 3rd entities are dropped
    out = orc.scatter_connection_forward(x, loc, 2, 2, "add")
    want = np.zeros((1, 2, 2, 2), np.float32)
    want[0, :, 0, 1] = x[0, 0]
    assert np.array_equal(out, want)
    g = np.random.default_rng(0).standard_normal((1, 2, 2, 2)).astype(np.float32)
    gx = orc.scatter_connection_backward(g, loc)
    assert np.array_equal(gx[0, 0], g[0, :, 0, 1]) and not gx[0, 1:].any()


def test_abi_argument_errors_without_a_gpu():
    from di_hpc_b200 import _abi
    L = _abi.lib()
    fwd, bwd = L.hpc_rll_scatter_connection_forward, L.hpc_rll_scatter_connection_backward
    buf = (ctypes.c_float * 64)()
    loc = (ctypes.c_int64 * 8)()
    p, q = ctypes.addressof(buf), ctypes.addressof(loc)
    assert fwd(None, q, p, 1, 4, 2, 2, 2, 0, None) == 1 and b"null" in L.hpc_rll_last_error()
    assert fwd(p, None, p, 1, 4, 2, 2, 2, 0, None) == 1
    assert fwd(p, q, None, 1, 4, 2, 2, 2, 1, None) == 1
    assert fwd(p, q, p, 1, -4, 2, 2, 2, 0, None) == 1 and b"negative" in L.hpc_rll_last_error()
    assert fwd(p, q, p, 1, 4, 2, 2, -2, 0, None) == 1
    assert fwd(p, q, p, 1, 4, 2, 2, 2, 2, None) == 1 and b"mode" in L.hpc_rll_last_error()
    assert fwd(p, q, p, 1, 4, 2, 2, 2, -1, None) == 1
    assert bwd(None, q, p, 1, 4, 2, 2, 2, None) == 1
    assert bwd(p, q, None, 1, 4, 2, 2, 2, None) == 1
    assert bwd(p, q, p, -1, 4, 2, 2, 2, None) == 1
    assert bwd(p, q, p, 1, 4, 2, 2**40, 2**40, None) == 1 and b"overflow" in L.hpc_rll_last_error()
    assert _abi.SCATTER_COVER == 0 and _abi.SCATTER_ADD == 1
    assert L.hpc_rll_launch_count() == 0


def test_module_api_surface():
    from hpc_rll.torch_utils.network.scatter_connection import ScatterConnection, ScatterConnectionFunction
    assert list(inspect.signature(ScatterConnection.__init__).parameters)[1:] == ["B", "M", "N", "H", "W",
                                                                                  "scatter_type"]
    assert list(inspect.signature(ScatterConnection.forward).parameters)[1:] == ["x", "location"]
    assert list(inspect.signature(ScatterConnectionFunction.apply).parameters) == ["input", "location", "output",
                                                                                   "grad_in", "scatter_type"]
    for bad in ("sum", "Cover", None):
        with pytest.raises(AssertionError):
            ScatterConnection(2, 3, 4, 5, 6, bad)
    m = ScatterConnection(256, 256, 256, 16, 16, "add").cuda()  # no buffers: .cuda() needs no device
    assert isinstance(m, torch.nn.Module) and (m.H, m.W) == (16, 16)
    with pytest.raises(AssertionError):
        m(torch.zeros(1, 2, 3), torch.zeros(1, 2, 2, dtype=torch.int64))  # CPU tensors: hpc version only supports cuda


def test_no_python_autograd_function_and_no_rnn():
    for dirpath, _, files in os.walk(os.path.join(os.path.dirname(GOLDEN_DIR), "..", "di_hpc_b200", "torch_utils")):
        for f in files:
            if f.endswith(".py"):
                rel = os.path.relpath(os.path.join(dirpath, f), os.path.join(GOLDEN_DIR, "..", ".."))
                mod = importlib.import_module(rel[:-3].replace(os.sep, "."))
                twins = [n for n, c in inspect.getmembers(mod, inspect.isclass)
                         if issubclass(c, torch.autograd.Function)]
                assert not twins, (mod.__name__, twins)
    with pytest.raises(ModuleNotFoundError):
        importlib.import_module("hpc_rll.torch_utils.network.rnn")


def test_legacy_native_names():
    import hpc_rl_utils
    import hpc_torch_utils_network
    for name in ("ScatterConnectionForward", "ScatterConnectionBackward"):
        assert callable(getattr(hpc_torch_utils_network, name)), name
        assert not hasattr(hpc_rl_utils, name), name
    assert "Sequence[torch.Tensor]" in hpc_torch_utils_network.ScatterConnectionForward.__doc__.splitlines()[0]
    assert not hasattr(hpc_torch_utils_network, "LstmForward")
