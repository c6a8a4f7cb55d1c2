"""dynamo_b200 -- Hopper-native (sm_90a) KV-block transfer path behind Dynamo's KVBM surface.

Only what the prefill->decode KV hand-off needs:
  csrc/kernels   CUDA kernels + the C ABI of libkvbm_kernels.so (include/kvbm_kernels.h)
  csrc/host      C++ restatement of the kvbm-physical host half (layouts, validation, strategy,
                 TransferManager) behind the C ABI of libkvbm_physical.so (include/kvbm_physical.h)
  kernels.py     thin ctypes mirror of lib/kvbm-kernels/src/tensor_kernels.rs
  physical.py    thin ctypes mirror of lib/kvbm-physical (LayoutConfig, PhysicalLayout, TransferManager)
The package never falls back to a CPU copy: a missing or unloadable native library raises.
"""
__version__ = "0.1.0"
