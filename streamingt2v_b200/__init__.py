"""b200-streamingsvd: Hopper-native (sm_90a) denoiser hot path for the StreamingSVD pipeline.

Python host code over a C-ABI CUDA library (streamingt2v_b200/libb200svd.so, include/b200svd.h).
"""
__version__ = "0.1.0"
