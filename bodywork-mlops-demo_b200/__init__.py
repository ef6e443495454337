"""H100-native (sm_90a) retrain hot path of AlexIoannides/bodywork-mlops-demo (stage_1's least-squares fit).

Import name: ``bodywork_mlops_demo_b200`` (a shim package that points here -- the directory name
``bodywork-mlops-demo_b200`` is not a valid Python identifier).

    native      ctypes binding of libb2gram.so (include/b2gram.h)
    Context     one GPU: Gram accumulation, solve, scoring, synthetic rows, NCCL all-reduce
    B200LinearRegression   estimator-protocol mirror of sklearn's LinearRegression as stage_1 uses it
    stage_1_train_model    drop-in for mlops_simulation/stage_1_train_model.py
"""
from . import _native as native
from ._native import (BF16, F32, KERNEL_AUTO, KERNEL_NARROW, KERNEL_SIMT, KERNEL_TCGEN05, PRECISION_BF16, PRECISION_SPLIT, Context,
                      DeviceArray, PinnedArray)
from .estimator import B200LinearRegression, default_context
from . import sharding, tranche_io  # noqa: F401

__all__ = ["native", "Context", "DeviceArray", "PinnedArray", "B200LinearRegression", "default_context",
           "F32", "BF16", "KERNEL_AUTO", "KERNEL_SIMT", "KERNEL_TCGEN05", "KERNEL_NARROW", "PRECISION_SPLIT", "PRECISION_BF16"]
__version__ = "0.1.0"
