"""H100-native (sm_90a) implementation of the animate-anything latent-video denoising hot path.

Host side: Python/PyTorch mirror of the reference's diffusers-style classes (same constructor configs, state_dict keys
and call signatures as /root/reference `models/unet_3d_condition_mask.py`, `models/unet_3d_blocks.py`,
`models/pipeline.py` + diffusers' AutoencoderKL / schedulers).  Device side: hand-written CUDA (wgmma / TMA / mbarrier)
behind the C-ABI in include/aab200.h, loaded with ctypes from libaab200.so.  No CPU fallback.
"""
__version__ = "0.1.0"
