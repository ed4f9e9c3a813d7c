from di_hpc_b200.rl_utils.vtrace import *  # noqa: F401,F403
from di_hpc_b200.rl_utils.vtrace import (VTrace, VtraceFunction, compute_importance_weights, hpc_vtrace_loss,  # noqa: F401
                                         vtrace_nstep_return)
