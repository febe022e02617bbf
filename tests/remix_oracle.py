"""CPU oracle of the remix path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-fp32 restatement over oracle/mug_oracle.py's U-Net and schedule of
  * DDIMSampler.ddim_sampling with ``timesteps=k`` (mug/diffusion/ddim.py:110-159, the subset of :123-127) from a given x_T;
  * PLMSSampler.plms_sampling with ``timesteps=k`` (mug/diffusion/plms.py:115-170, the subset of :128-132);
  * Stable Diffusion's DDIMSampler.decode with Mug's (c, w) conditioning, with a scalar start or one start per chart (chart b joins
    the loop of m = max(t_start) iterations at iteration m - t_start[b], its latent held until then).
All at eta = 0.  tests/test_remix.py pins the truncated runs to outputs of the UNMODIFIED reference (tests/golden/remix_*.npz,
tools/make_remix_goldens.py)."""
from typing import Optional, Sequence

import numpy as np
import torch

from oracle import mug_oracle as orc
from remix_cases import subset_end


def _eps(p, x, t, c, w, scale, uc, cfg):
    """e_t of p_sample_ddim / get_model_output (ddim.py:167-175, plms.py:178-192)"""
    if uc is None or scale == 1.0:
        return orc.unet_forward(p, x, t, c, w, cfg)
    e = orc.unet_forward(p, torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c]), [torch.cat([wi, wi]) for wi in w], cfg)
    e_u, e_c = e.chunk(2)
    return e_u + scale * (e_c - e_u)


def _x_prev(sch, x, e_t, index):
    """x_prev and pred_x0 of DDIM index ``index`` at sigma = 0 (ddim.py:178-196, plms.py:199-216)"""
    B = x.shape[0]
    a_t = torch.full((B, 1, 1), float(sch["alphas"][index]))
    a_prev = torch.full((B, 1, 1), float(sch["alphas_prev"][index]))
    sigma_t = torch.full((B, 1, 1), float(sch["sigmas"][index]))
    s1m = torch.full((B, 1, 1), float(sch["sqrt_one_minus_alphas"][index]))
    pred_x0 = (x - s1m * e_t) / a_t.sqrt()
    dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e_t
    return a_prev.sqrt() * pred_x0 + dir_xt, pred_x0


def subset(S: int, timesteps) -> np.ndarray:
    """the DDIM timesteps a request with ``timesteps`` runs (ddim.py:123-127)"""
    ts = orc.make_schedule(S)["timesteps"]
    return ts if timesteps is None else ts[:subset_end(timesteps, ts.shape[0])]


def _ddim_loop(p, sch, ts, c, w, x, scale, uc, log_every_t, cfg, x_latent=None, joins=None):
    total = ts.shape[0]
    B = x.shape[0]
    intermediates = {'x_inter': [x], 'pred_x0': [x]}                          # :129
    for i, step in enumerate(np.flip(ts)):                                    # :130, :137
        index = total - i - 1                                                 # :138
        if joins is not None:
            hold = torch.tensor([i <= j for j in joins])[:, None, None]       # charts that have not joined yet keep their latent
            x = torch.where(hold, x_latent, x)
        t = torch.full((B,), int(step), dtype=torch.long)
        x, pred_x0 = _x_prev(sch, x, _eps(p, x, t, c, w, scale, uc, cfg), index)
        if index % log_every_t == 0 or index == total - 1:                    # :155-157
            intermediates['x_inter'].append(x)
            intermediates['pred_x0'].append(pred_x0)
    return x, intermediates


def ddim_sampling(p: orc.Params, S: int, c: torch.Tensor, w: Sequence[torch.Tensor], x_T: torch.Tensor, scale: float = 1.0,
                  uc: Optional[torch.Tensor] = None, timesteps=None, log_every_t: int = 100, cfg: dict = orc.DEFAULT_UNET):
    """DDIMSampler.ddim_sampling(w, c, shape, x_T=x_T, timesteps=timesteps, ...) after make_schedule(S, eta=0).  Returns
    (x, {'x_inter', 'pred_x0'})."""
    sch = orc.make_schedule(S)
    return _ddim_loop(p, sch, subset(S, timesteps), c, w, x_T, scale, uc, log_every_t, cfg)


def decode(p: orc.Params, S: int, x_latent: torch.Tensor, c: torch.Tensor, w: Sequence[torch.Tensor], t_start, scale: float = 1.0,
           uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET) -> torch.Tensor:
    """decode(x_latent, c, w, t_start) after make_schedule(S, eta=0): SD's loop over ddim_timesteps[:t_start] flipped at index
    t_start - i - 1; with one start per chart, m = max(t_start) iterations and chart b held at x_latent[b] while i <= m - t_start[b];
    charts with t_start[b] = 0 come back as x_latent[b]."""
    sch = orc.make_schedule(S)
    B = x_latent.shape[0]
    starts = [int(t_start)] * B if isinstance(t_start, int) else [int(s) for s in t_start]
    m = max(starts)
    if m == 0:
        return x_latent
    joins = None if len(set(starts)) == 1 else [m - s for s in starts]
    x, _ = _ddim_loop(p, sch, sch["timesteps"][:m], c, w, x_latent, scale, uc, 100, cfg, x_latent, joins)
    idle = [b for b, s in enumerate(starts) if s == 0]
    if idle:
        x = x.clone()
        x[idle] = x_latent[idle]
    return x


def plms_sampling(p: orc.Params, S: int, c: torch.Tensor, w: Sequence[torch.Tensor], x_T: torch.Tensor, scale: float = 1.0,
                  uc: Optional[torch.Tensor] = None, timesteps=None, log_every_t: int = 100, cfg: dict = orc.DEFAULT_UNET):
    """PLMSSampler.plms_sampling(cond, shape, x_T=x_T, timesteps=timesteps, ...) after make_schedule(S, eta=0), as
    tests/plms_oracle.py restates it, over the subset: t_next (:145) and the warm-up follow the truncated range."""
    sch = orc.make_schedule(S)
    ts = subset(S, timesteps)
    B = x_T.shape[0]
    total = ts.shape[0]
    time_range = np.flip(ts)
    x = x_T
    intermediates = {'x_inter': [x], 'pred_x0': [x]}
    old_eps = []
    for i, step in enumerate(time_range):
        index = total - i - 1
        t = torch.full((B,), int(step), dtype=torch.long)
        t_next = torch.full((B,), int(time_range[min(i + 1, len(time_range) - 1)]), dtype=torch.long)
        e_t = _eps(p, x, t, c, w, scale, uc, cfg)
        if len(old_eps) == 0:                                                 # :219-223 pseudo improved Euler
            x_prev, _ = _x_prev(sch, x, e_t, index)
            e_t_prime = (e_t + _eps(p, x_prev, t_next, c, w, scale, uc, cfg)) / 2
        elif len(old_eps) == 1:
            e_t_prime = (3 * e_t - old_eps[-1]) / 2
        elif len(old_eps) == 2:
            e_t_prime = (23 * e_t - 16 * old_eps[-1] + 5 * old_eps[-2]) / 12
        else:
            e_t_prime = (55 * e_t - 59 * old_eps[-1] + 37 * old_eps[-2] - 9 * old_eps[-3]) / 24
        x, pred_x0 = _x_prev(sch, x, e_t_prime, index)
        old_eps.append(e_t)
        if len(old_eps) >= 4:
            old_eps.pop(0)
        if index % log_every_t == 0 or index == total - 1:
            intermediates['x_inter'].append(x)
            intermediates['pred_x0'].append(pred_x0)
    return x, intermediates
