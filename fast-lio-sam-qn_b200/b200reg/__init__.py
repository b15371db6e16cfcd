"""b200reg -- H100-native loop-closure registration engine (Nano-GICP + Quatro path of FAST-LIO-SAM-QN).

Python here is plumbing only (ctypes over the C ABI in include/b200reg.h, synthetic inputs,
torch.distributed sharding); the product is csrc/*.cu.
"""
from . import synth  # noqa: F401
from .native import (B200RegError, Batch, Context, comm_unique_id, GicpParams, QuatroInfo, QuatroParams, Result, default_params,  # noqa: F401
                     default_quatro_params, Keyframes, LoopConfig, LoopFactor, default_loop_config,
                     loop_factor_from_poses, LM_TRIAL_DTYPE, LmTrial, CLOUD_SOURCE, CLOUD_TARGET, CLOUD_COARSE, CLOUD_FINAL,
                     fitness_score)
