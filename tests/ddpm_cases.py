"""The DDPM golden cases shared by tools/make_ddpm_goldens.py (which runs the UNMODIFIED reference ``DDPM.log_beatmap`` and writes
tests/golden/ddpm_*.npz) and the tests that replay them.  The U-Net weights and inputs come from the seeds of
mug_diffusion_b200.synth, as for the DDIM goldens; x_T and the step noise come from torch's CPU generator after
``torch.manual_seed(seed)``, in the reference's order (x_T first, diffusion.py:234, then one draw per step, :274)."""

# DDPM trajectories: (z_length, batch, num_timesteps, log_every_t, seed)
DDPM_CASES = {
    "ddpm_L96_B1_T1000": dict(L=96, B=1, T=1000, log_every_t=100, seed=2024),
    "ddpm_L96_B2_T50":   dict(L=96, B=2, T=50, log_every_t=10, seed=77),
}

# the reference's float32 schedule buffers stored with each golden as sched_<name> (diffusion.py:152-176)
SCHEDULE_KEYS = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod", "sqrt_one_minus_alphas_cumprod",
                 "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_variance",
                 "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2")


def logged_steps(T: int, log_every_t: int) -> list:
    """the timesteps i whose x diffusion.py:279 records, in loop order"""
    return [i for i in reversed(range(T)) if i % log_every_t == 0 or i == T - 1]


def cpu_noise(seed: int, shape, T: int):
    """(x_T, [noise of the step at i = T-1, ..., 0]): the reference's CPU draws after torch.manual_seed(seed), from a private
    generator seeded the same way (same values; the global generator is left alone)"""
    import torch
    g = torch.Generator().manual_seed(seed)
    x_T = torch.randn(shape, generator=g)
    return x_T, [torch.randn(shape, generator=g) for _ in range(T)]
