"""Host-side mirror of the reference package `hpc_rll.torch_utils.network`: `scatter_connection` only (no `rnn`)."""
