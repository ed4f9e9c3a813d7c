from di_hpc_b200.rl_utils.td import (DistNStepTD, DistNStepTDFunction, IQNNStepTDError,  # noqa: F401
                                      IQNNStepTDErrorFunction, QNStepTD, QNStepTDFunction, QNStepTDRescale,
                                      QNStepTDRescaleFunction, QRDQNNStepTDError, QRDQNNStepTDErrorFunction,
                                      TDLambda, TDLambdaFunction, generalized_lambda_returns,
                                      multistep_forward_view)
