"""lfm_quant_b200: GPU-native (H100, sm_90a) training / inference step for the lfm_quant recurrent forecaster.

Only what the hot path needs lives here: ``csrc/`` (CUDA kernels + the C-ABI of include/lfmq.h),
``_native`` (ctypes binding), ``engine`` (device-memory owner) and ``scripts/`` (the host-side mirror of
the reference's scripts/ interface: configs, Dataset, model classes, Train, Predict, CLI).
"""
__version__ = '0.1.0'
