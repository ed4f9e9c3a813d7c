"""di_hpc_b200 -- H100-native (sm_90a) re-implementation of DI-hpc's trajectory-return hot path.

The package holds only what that path needs:
  csrc/       hand-written CUDA kernels + the C ABI (include/hpc_rll_b200.h)
  csrc_torch/ torch/pybind extension over that library: one C++ autograd function per op, which the
              rl_utils modules call (loaded by _ext.py), the padding list handling and the reference's
              binding names
  _abi.py     ctypes binding of libhpc_rll_b200.so for the calls without autograd (fails loudly if the
              library is missing)
  rl_utils/   host-side mirror of the reference's `hpc_rll.rl_utils` modules (same class names,
              constructor arguments and forward signatures); `hpc_rll/` at the repo root re-exports it
              under the reference's import paths so DI-engine can swap it in unchanged.
  torch_utils/ the same for `hpc_rll.torch_utils.network.scatter_connection` (ScatterConnection; no LSTM).
There is no CPU fallback and no multi-backend dispatch.
"""
__version__ = "0.1.0"
