from di_hpc_b200.rl_utils.gae import GAE, GAEFunction, gae, gae_data, gae_with_adv_stats  # noqa: F401
