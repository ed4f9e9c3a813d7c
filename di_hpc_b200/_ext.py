"""Loader of the torch/pybind layer ``_lib/hpc_rl_utils_b200*.so`` (csrc_torch/: C++ autograd functions behind the
nn.Modules, the reference's 30 ``hpc_rl_utils`` binding names, the padding list handling).

The nn.Modules of ``rl_utils`` and the padding functions reach libhpc_rll_b200.so only through this extension; when it
cannot be loaded, ``require()`` raises with the reason.
"""
import glob
import importlib.util
import os
import sys

from ._abi import LIB_PATH, HpcRllError

_NAME = "hpc_rl_utils_b200"
_mod = None
_err = None


def load():
    """The extension module, or None (reason in ``why_missing()``)."""
    global _mod, _err
    if _mod is not None or _err is not None:
        return _mod
    if _NAME in sys.modules:
        _mod = sys.modules[_NAME]
        return _mod
    cands = glob.glob(os.path.join(os.path.dirname(LIB_PATH), _NAME + "*.so"))
    if not cands:
        _err = "not built (run `python -m di_hpc_b200.build_torch_ext` or __graft_entry__.build())"
        return None
    try:
        import torch  # noqa: F401  (the extension links against libtorch)
        spec = importlib.util.spec_from_file_location(_NAME, cands[0])
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        sys.modules[_NAME] = mod
        _mod = mod
    except Exception as e:  # noqa: BLE001  e.g. built against another torch: require() reports it
        _err = "%s: %s" % (type(e).__name__, e)
    return _mod


def why_missing():
    return _err


def fast():
    return load()  # kept for bench.py, which reports whether the extension loaded


def require():
    m = load()
    if m is None:
        raise HpcRllError("torch extension %s unavailable: %s" % (_NAME, _err))
    return m


def reference_function(apply):
    """Decorator: a plain class named like ``apply`` whose static ``apply`` is the function, i.e. the reference's
    ``*Function.apply`` entry point.  The autograd function behind it is the extension's C++ one (fast_ops.cpp)."""
    return type(apply.__name__, (), {"apply": staticmethod(apply), "__module__": apply.__module__,
                                     "__doc__": apply.__doc__})
