"""CPU oracle of the PLMS sampler (mug/diffusion/plms.py) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-fp32 restatement over oracle/mug_oracle.py's U-Net and schedule, citing plms.py line by line (the inpainting mask branch
included).  tests/test_plms.py pins it to outputs of the UNMODIFIED reference (tests/golden/plms_*.npz, tools/make_plms_goldens.py);
on them it is bit-identical (max-abs error 0.0)."""
from typing import Optional, Sequence

import numpy as np
import torch

from oracle import mug_oracle as orc


def plms_sample(p: orc.Params, S: int, c: torch.Tensor, w: Sequence[torch.Tensor], x_T: torch.Tensor,
                scale: float = 1.0, uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET, log_every_t: int = 100,
                mask: Optional[torch.Tensor] = None, x0: Optional[torch.Tensor] = None,
                q_noise_seq: Optional[Sequence[torch.Tensor]] = None):
    """PLMSSampler.plms_sampling + p_sample_plms  -- mug/diffusion/plms.py:115-236, at eta = 0 (:25-26).
    Returns (x, {'x_inter': [...], 'pred_x0': [...]}).  ``mask`` / ``x0``: the blend of :147-150 with ``DDPM.q_sample``
    (diffusion.py:327-333); ``q_noise_seq[i]`` replaces the ``randn_like(x0)`` it draws in iteration i.
    The reference's coefficients are [b, 1, 1, 1] tensors (:201-204), which broadcast a [B, C, L] x to [B, B, C, L] whose B copies
    are equal; this restatement keeps [B, C, L] (the same operations on the same values).  Its step noise is sigma_t * randn * T
    with sigma_t = 0 (:212); it is left out."""
    sch = orc.make_schedule(S)                                               # make_schedule, :24-55 (ddim_eta = 0)
    ts = sch["timesteps"]
    B = x_T.shape[0]
    total = ts.shape[0]
    time_range = np.flip(ts)                                             # :135
    x = x_T
    intermediates = {'x_inter': [x], 'pred_x0': [x]}                     # :134
    old_eps = []

    def model_output(x, t):                                              # :178-192
        if uc is None or scale == 1.0:
            return orc.unet_forward(p, x, t, c, w, cfg)
        e = orc.unet_forward(p, torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c]), [torch.cat([wi, wi]) for wi in w], cfg)
        e_u, e_c = e.chunk(2)
        return e_u + scale * (e_c - e_u)

    def x_prev_and_pred_x0(x, e_t, index):                               # :199-216
        a_t = torch.full((B, 1, 1), float(sch["alphas"][index]))
        a_prev = torch.full((B, 1, 1), float(sch["alphas_prev"][index]))
        sigma_t = torch.full((B, 1, 1), float(sch["sigmas"][index]))
        s1m = torch.full((B, 1, 1), float(sch["sqrt_one_minus_alphas"][index]))
        pred_x0 = (x - s1m * e_t) / a_t.sqrt()                           # :207
        dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e_t               # :211
        return a_prev.sqrt() * pred_x0 + dir_xt, pred_x0                  # :215

    for i, step in enumerate(time_range):                                # :142
        index = total - i - 1                                            # :143
        t = torch.full((B,), int(step), dtype=torch.long)                # :144
        t_next = torch.full((B,), int(time_range[min(i + 1, len(time_range) - 1)]), dtype=torch.long)   # :145
        if mask is not None:                                             # :147-150
            assert x0 is not None
            qn = q_noise_seq[i] if q_noise_seq is not None else torch.randn(x0.shape)
            x_orig = sch["sqrt_alphas_cumprod"][t].view(-1, 1, 1) * x0 + sch["sqrt_one_minus_alphas_cumprod"][t].view(-1, 1, 1) * qn
            x = x_orig * mask + (1. - mask) * x
        e_t = model_output(x, t)                                         # :218
        if len(old_eps) == 0:                                            # :219-223 pseudo improved Euler
            x_prev, _ = x_prev_and_pred_x0(x, e_t, index)
            e_t_next = model_output(x_prev, t_next)
            e_t_prime = (e_t + e_t_next) / 2
        elif len(old_eps) == 1:                                          # :224-226
            e_t_prime = (3 * e_t - old_eps[-1]) / 2
        elif len(old_eps) == 2:                                          # :227-229
            e_t_prime = (23 * e_t - 16 * old_eps[-1] + 5 * old_eps[-2]) / 12
        else:                                                            # :230-232
            e_t_prime = (55 * e_t - 59 * old_eps[-1] + 37 * old_eps[-2] - 9 * old_eps[-3]) / 24
        x, pred_x0 = x_prev_and_pred_x0(x, e_t_prime, index)             # :234
        old_eps.append(e_t)                                              # :160-162
        if len(old_eps) >= 4:
            old_eps.pop(0)
        if index % log_every_t == 0 or index == total - 1:               # :166-168
            intermediates['x_inter'].append(x)
            intermediates['pred_x0'].append(pred_x0)
    return x, intermediates
