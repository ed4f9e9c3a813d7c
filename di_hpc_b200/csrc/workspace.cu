// workspace.cu -- scratch sizing for hpc_rll_workspace_bytes().  One place so that the Python
// binding and the C launchers agree; each launcher re-checks the size it is handed.
#include "common.cuh"

namespace hpcrll {

size_t td_lambda_workspace_bytes(int64_t B);
size_t gae_moments_workspace_bytes(int64_t B);
size_t vtrace_workspace_bytes(int64_t T, int64_t B);
size_t upgo_workspace_bytes(int64_t T, int64_t B);
size_t ppo_workspace_bytes();
size_t nstep_workspace_bytes();
size_t importance_weights_workspace_bytes(int64_t R);

size_t workspace_bytes(int op, int64_t T, int64_t B, int64_t N) {
    (void)T;
    (void)B;
    (void)N;
    switch (op) {
        case HPC_RLL_OP_GAE:
            return 0;
        case HPC_RLL_OP_GAE_MOMENTS:
            return gae_moments_workspace_bytes(B);
        case HPC_RLL_OP_TD_LAMBDA:
            return td_lambda_workspace_bytes(B);
        case HPC_RLL_OP_VTRACE:
            return vtrace_workspace_bytes(T, B);
        case HPC_RLL_OP_UPGO:
            return upgo_workspace_bytes(T, B);
        case HPC_RLL_OP_PPO:
            return ppo_workspace_bytes();
        case HPC_RLL_OP_Q_NSTEP_TD:
        case HPC_RLL_OP_DIST_NSTEP_TD:
        case HPC_RLL_OP_QRDQN_NSTEP_TD:
        case HPC_RLL_OP_IQN_NSTEP_TD:
            return nstep_workspace_bytes();
        case HPC_RLL_OP_IMPORTANCE_WEIGHTS:
            return importance_weights_workspace_bytes(T * B);
        default:
            return 0;
    }
}

}  // namespace hpcrll
