"""The drop-in modules reach the CUDA library through one binding, the C++ extension: no Python autograd functions and
no switch that selects another binding.  Without the extension the package still imports and the modules construct;
calling into them then fails with the reason the extension did not load."""
import importlib
import inspect
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RL_UTILS = ("gae", "td", "vtrace", "upgo", "ppo", "padding")


def test_one_binding_behind_the_modules():
    for name in RL_UTILS:
        mod = importlib.import_module("di_hpc_b200.rl_utils." + name)
        twins = [n for n, c in inspect.getmembers(mod, inspect.isclass) if issubclass(c, torch.autograd.Function)]
        assert not twins, "%s defines Python autograd functions %s" % (mod.__name__, twins)
    for pkg in ("di_hpc_b200", "hpc_rll"):
        for dirpath, dirs, files in os.walk(os.path.join(ROOT, pkg)):
            dirs[:] = [d for d in dirs if d not in ("__pycache__", "_lib")]  # build products
            for f in files:
                path = os.path.join(dirpath, f)
                with open(path, "rb") as fh:
                    assert b"HPC_RLL_BINDING" not in fh.read(), "%s mentions HPC_RLL_BINDING" % path


def test_missing_extension_is_reported_at_call_time(monkeypatch):
    from di_hpc_b200 import _ext
    from di_hpc_b200._abi import HpcRllError
    import tests.test_abi_cpu as abi_tests
    monkeypatch.setattr(_ext, "_mod", None)
    monkeypatch.setattr(_ext, "_err", "ImportError: built against another torch")
    with pytest.raises(HpcRllError, match="built against another torch"):
        _ext.require()
    monkeypatch.delitem(sys.modules, "di_hpc_b200.rl_utils.padding", raising=False)
    padding = importlib.import_module("di_hpc_b200.rl_utils.padding")
    with pytest.raises(AssertionError):
        padding.Padding1D([])
    with pytest.raises(AssertionError):
        padding.Padding1D([torch.zeros(3)])
    abi_tests.test_di_engine_hpc_wrapper_lookup()
