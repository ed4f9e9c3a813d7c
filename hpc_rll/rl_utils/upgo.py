from di_hpc_b200.rl_utils.upgo import *  # noqa: F401,F403
from di_hpc_b200.rl_utils.upgo import UPGO, UpgoFunction, tb_cross_entropy, upgo_returns  # noqa: F401
