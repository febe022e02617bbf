"""CPU oracle of the DDPM ancestral sampler (DDPM.log_beatmap, mug/diffusion/diffusion.py) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-fp32 restatement over oracle/mug_oracle.py's U-Net, citing diffusion.py line by line.  tests/test_ddpm.py pins it to outputs
of the UNMODIFIED reference (tests/golden/ddpm_*.npz, tools/make_ddpm_goldens.py)."""
from typing import Optional, Sequence

import numpy as np
import torch

from oracle import mug_oracle as orc


def register_schedule(timesteps: int = 1000, linear_start: float = 1e-4, linear_end: float = 2e-2, v_posterior: float = 0.) -> dict:
    """DDPM.register_schedule -- diffusion.py:131-176 (make_beta_schedule "linear", utils.py:16-21): float64 numpy, cast to float32"""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=torch.float64) ** 2).numpy()
    alphas = 1. - betas                                                      # :139
    alphas_cumprod = np.cumprod(alphas, axis=0)                              # :140
    alphas_cumprod_prev = np.append(1., alphas_cumprod[:-1])                 # :141
    f32 = lambda a: torch.tensor(a, dtype=torch.float32)                     # :150
    posterior_variance = (1 - v_posterior) * betas * (1. - alphas_cumprod_prev) / (1. - alphas_cumprod) + v_posterior * betas  # :166
    return dict(
        betas=f32(betas), alphas_cumprod=f32(alphas_cumprod), alphas_cumprod_prev=f32(alphas_cumprod_prev),        # :152-154
        sqrt_alphas_cumprod=f32(np.sqrt(alphas_cumprod)), sqrt_one_minus_alphas_cumprod=f32(np.sqrt(1. - alphas_cumprod)),  # :157-159
        log_one_minus_alphas_cumprod=f32(np.log(1. - alphas_cumprod)),                                             # :160
        sqrt_recip_alphas_cumprod=f32(np.sqrt(1. / alphas_cumprod)),                                               # :161
        sqrt_recipm1_alphas_cumprod=f32(np.sqrt(1. / alphas_cumprod - 1)),                                         # :162-163
        posterior_variance=f32(posterior_variance),                                                                # :169
        posterior_log_variance_clipped=f32(np.log(np.maximum(posterior_variance, 1e-20))),                        # :171-172
        posterior_mean_coef1=f32(betas * np.sqrt(alphas_cumprod_prev) / (1. - alphas_cumprod)),                   # :173-174
        posterior_mean_coef2=f32((1. - alphas_cumprod_prev) * np.sqrt(alphas) / (1. - alphas_cumprod)))           # :175-176


def extract(a: torch.Tensor, t: torch.Tensor, x_shape) -> torch.Tensor:
    """extract_into_tensor: a.gather(-1, t) reshaped to [b, 1, 1]"""
    return a.gather(-1, t).reshape(t.shape[0], *((1,) * (len(x_shape) - 1)))


def ddpm_sample(p: orc.Params, T: int, c: torch.Tensor, w: Sequence[torch.Tensor], seed: Optional[int] = None,
                x_T: Optional[torch.Tensor] = None, noise_seq: Optional[Sequence[torch.Tensor]] = None, log_every_t: int = 100,
                clip_denoised: bool = True, scale: float = 1.0, uc: Optional[torch.Tensor] = None, z_length: Optional[int] = None,
                cfg: dict = orc.DEFAULT_UNET, schedule: Optional[dict] = None):
    """DDPM.log_beatmap's loop -- diffusion.py:234-282, parameterization "eps".  Returns (x, {'x_inter': [...], 'pred_x0': [...]}),
    x_T first, then x and x_recon of every logged step.
    x_T and the step noise: by default the CPU generator's draws after manual_seed(seed) (x_T first, :234, then one randn per
    step, :274), from a private generator; ``x_T`` / ``noise_seq[k]`` (the noise of the k-th iteration) replace them.
    ``scale`` / ``uc``: classifier-free guidance, an extension the reference loop does not have, combined as ddim.py:170-175."""
    sch = schedule or register_schedule(T)
    B = c.shape[0]
    g = torch.Generator().manual_seed(seed) if seed is not None else None
    if x_T is None:
        x_T = torch.randn((B, 16, z_length), generator=g)                 # :234
    x = x_T
    intermediates = {'x_inter': [x], 'pred_x0': [x]}

    def model_out(x, t):                                                 # :259 (+ the CFG extension)
        if uc is None or scale == 1.0:
            return orc.unet_forward(p, x, t, c, w, cfg)
        e = orc.unet_forward(p, torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c]), [torch.cat([wi, wi]) for wi in w], cfg)
        e_u, e_c = e.chunk(2)
        return e_u + scale * (e_c - e_u)

    for k, i in enumerate(reversed(range(0, T))):                        # :255
        t = torch.full((B,), i, dtype=torch.long)                       # :257
        e = model_out(x, t)
        x_recon = (extract(sch["sqrt_recip_alphas_cumprod"], t, x.shape) * x -
                   extract(sch["sqrt_recipm1_alphas_cumprod"], t, x.shape) * e)          # :261, predict_start_from_noise :211-215
        if clip_denoised:                                                # :266-267
            x_recon.clamp_(-10., 10.)
        model_mean = (extract(sch["posterior_mean_coef1"], t, x.shape) * x_recon +
                      extract(sch["posterior_mean_coef2"], t, x.shape) * x)              # :268-271
        model_log_variance = extract(sch["posterior_log_variance_clipped"], t, x.shape)  # :272-273
        noise = noise_seq[k] if noise_seq is not None else torch.randn(x.shape, generator=g)   # :274, noise_like
        nonzero_mask = (1 - (t == 0).float()).reshape(B, *((1,) * (len(x.shape) - 1)))     # :276
        x = model_mean + nonzero_mask * (0.5 * model_log_variance).exp() * noise            # :277
        if i % log_every_t == 0 or i == T - 1:                           # :279
            intermediates['x_inter'].append(x)
            intermediates['pred_x0'].append(x_recon)
    return x, intermediates
