"""`hpc_torch_utils_network` -- the reference's second NATIVE module name (src/torch_utils/network/entry.cpp), re-exporting
`ScatterConnectionForward(inputs, outputs, scatter_type)` and `ScatterConnectionBackward(inputs, outputs)` with the
reference's tensor-list signatures, implemented on libhpc_rll_b200.so (di_hpc_b200/csrc_torch/legacy.cpp).  The
reference's `LstmForward` / `LstmBackward` are not provided (INTEGRATION.md)."""
from di_hpc_b200 import _ext as _loader

_m = _loader.require()._torch_utils_network
ScatterConnectionForward = _m.ScatterConnectionForward
ScatterConnectionBackward = _m.ScatterConnectionBackward
__all__ = ["ScatterConnectionForward", "ScatterConnectionBackward"]
