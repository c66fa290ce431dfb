"""anyv2v_b200 — H100-native (sm_90a) hot path of AnyV2V (DDIM inversion + PnP edit over the I2VGen-XL UNet).

Python host code over PyTorch tensors calling hand-written sm_90a kernels through a C ABI
(include/anyv2v_b200.h).  No CPU fallback: importing is cheap, every op raises if the extension is missing.
"""
__version__ = "0.1.0"
