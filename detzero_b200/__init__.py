"""detzero_b200 -- Hopper-native (sm_90a) implementation of the DetZero point-cloud hot path.

csrc/            hand-written CUDA kernels + the C ABI (include/detzero_b200.h) -> libdetzero_b200.so
_lib.py / ops.py ctypes binding and torch-tensor wrappers (torch = device memory + streams only)
spconv/          ``spconv.pytorch`` / ``spconv.utils``-shaped API the reference's modules are written against
det/             CenterPoint template, module registry, VFE / backbones / CenterHead mirrors, data processor
refine/          GRM / PRM / CRM transformer modules
config.py        YAML + ``--set`` config semantics of detzero_utils.config_utils
dist.py          frame sharding + per-sequence NCCL box gather
"""
__version__ = '0.1.0'
