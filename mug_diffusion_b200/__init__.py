"""mug_diffusion_b200 -- H100-native (sm_90a) denoising sampler for Mug-Diffusion.

Only the hot path lives here: DDIM loop -> U-Net eval -> first-stage decode, as hand-written CUDA kernels
behind the C ABI declared in include/mugd.h, plus the Python host mirror of the reference call surface
(``DDIMSampler(model).sample(...)``, ``model.model.decode(z)``).
"""
__version__ = "0.1.0"
