from di_hpc_b200.rl_utils.vtrace import *  # noqa: F401,F403
from di_hpc_b200.rl_utils.vtrace import VTrace, VtraceFunction, hpc_vtrace_loss, vtrace_nstep_return  # noqa: F401
