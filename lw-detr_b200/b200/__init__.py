"""Host-side glue of the CUDA-native (H100, sm_90a) LW-DETR path (ctypes binding, configs, synthetic weights)."""
