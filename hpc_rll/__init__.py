"""`hpc_rll` -- the reference's package name, re-exporting the H100-native implementation.

DI-engine imports `hpc_rll.rl_utils.{gae,td,upgo,vtrace,ppo}` and `hpc_rll.torch_utils.network.scatter_connection`
(see SURVEY.md 3.5); those module paths resolve to `di_hpc_b200.rl_utils.*` and `di_hpc_b200.torch_utils.network.*`.
`hpc_rll.origin` (the reference's PyTorch oracle) and `hpc_rll.torch_utils.network.rnn` (the LSTM) are intentionally
absent: out of scope (DESIGN.md section 8).
"""
