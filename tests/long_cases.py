"""Golden cases for long songs (z_length past 1568, where the S4 convolution streams its operands), shared by
tools/make_long_goldens.py (which runs the UNMODIFIED reference on the CPU and writes tests/golden/) and the tests that replay
them against oracle/ and the CUDA path.  Inputs come from the seeds of mug_diffusion_b200.synth; only outputs are stored."""

# whole-network evaluations: z_length, batch, timesteps, and the z_length the S4 `L` buffers were persisted at (None = the
# request's own length: a fresh model).  From 512 every S4 layer doubles twice, the case a trained checkpoint (L buffers
# 512 / 256 / 128 / 64) meets at z_length 2048.
LONG_UNET_CASES = {
    "unet_L2048_B1": dict(L=2048, B=1, t=[333], persisted=None),
    "unet_L2048_from512": dict(L=2048, B=1, t=[611], persisted=512),
}

# DDIM trajectories: 1600 is the first z_length whose level-0 S4 layers do not fit the resident kernel
LONG_DDIM_CASES = {
    "ddim_L1600_B1_S4_cfg5": dict(L=1600, B=1, S=4, scale=5.0),
}
