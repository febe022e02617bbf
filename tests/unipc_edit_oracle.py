"""CPU oracle of UniPC inpainting, remix and inversion -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The D-form loop of tests/unipc_oracle.py (``d_form_step``, every step's coefficients solved in float64, the latents in torch fp32 over
oracle/mug_oracle.py's U-Net), with
  * inpainting: before the evaluation of iteration i, x~_i <- (alpha_i x0 + sigma_i eps_i) * mask + (1 - mask) * x~_i with the schedule's
    (alpha_i, sigma_i) in float32 and the given per-step noise eps_i; the corrector's previous latent is not blended;
  * remix (decode): chart b runs iterations f_b = S - t_start[b] .. S - 1 from x_latent[b] with its own history, predictor order
    min(orders[i], i - f_b + 1) and its corrector only for i > f_b, at order min(orders[i - 1], i - f_b); held charts keep their latent;
  * inversion: the same loop on the reversed grid of ``unipc.inversion_schedule`` (orders min(j + 1, order), the corrector on every
    j >= 1 when the request has one), chart b stopping after t_enc[b] iterations.
It steps the D-form, not the expanded rows or their row forms, so it checks the tables, the kernels' forms and the loops."""
from typing import Optional, Sequence

import torch

from dpm_remix_oracle import _eps
from mug_diffusion_b200 import unipc as U
from oracle import mug_oracle as orc
from unipc_oracle import d_form_step


def _loop(p, t_grid, ns, variant, model_times, x, firsts, stops, kp, kc, c, w, scale, uc, cfg, blend=None):
    """iterations min(firsts) .. max(stops) - 1 on ``t_grid``; chart b runs iterations firsts[b] .. stops[b] - 1 with predictor order
    kp(b, i) and corrector order kc(b, i) (0: no corrector).  ``blend(i, x)`` runs in front of each evaluation."""
    alpha, sigma, lam = ns.marginal_alpha(t_grid), ns.marginal_std(t_grid), ns.marginal_lambda(t_grid)
    B = x.shape[0]
    xc, ms = [None] * B, [[] for _ in range(B)]
    for i in range(min(firsts), max(stops)):
        if blend is not None:
            x = blend(i, x)
        t = torch.full((B,), float(model_times[i]), dtype=torch.float32)
        e = _eps(p, x, t, c, w, scale, uc, cfg)
        out = []
        for b in range(B):
            xb = x[b:b + 1]
            if i < firsts[b] or i >= stops[b]:
                out.append(xb)
                continue
            m = (xb - float(sigma[i]) * e[b:b + 1]) / float(alpha[i])
            k = kc(b, i)
            xi = d_form_step(xc[b], ms[b], i, k, alpha, sigma, lam, variant, m_new=m) if k else xb
            ms[b] = [m] + ms[b][:2]
            out.append(d_form_step(xi, ms[b], i + 1, kp(b, i), alpha, sigma, lam, variant))
            xc[b] = xi
        x = torch.cat(out)
    return x


def inpaint(p: orc.Params, sched: U.UniPCSchedule, c: torch.Tensor, w: Sequence[torch.Tensor], x_T: torch.Tensor, mask: torch.Tensor,
            x0: torch.Tensor, q_noise: Sequence[torch.Tensor], scale: float = 1.0, uc: Optional[torch.Tensor] = None,
            cfg: dict = orc.DEFAULT_UNET) -> torch.Tensor:
    """the S iterations of UniPCSampler.inpaint from x_T with q_noise[i] the blend noise of iteration i; returns x~_S"""
    q = torch.from_numpy(sched.q_coef_f32())
    B, S = x_T.shape[0], sched.S

    def blend(i, x):
        return (q[i, 0] * x0 + q[i, 1] * q_noise[i]) * mask + (1. - mask) * x

    return _loop(p, sched.t, sched.ns, sched.variant, sched.model_times, x_T, [0] * B, [S] * B, lambda b, i: int(sched.orders[i]),
                 lambda b, i: int(sched.orders[i - 1]) if sched.corrector[i] else 0, c, w, scale, uc, cfg, blend)


def decode(p: orc.Params, sched: U.UniPCSchedule, x_latent: torch.Tensor, c: torch.Tensor, w: Sequence[torch.Tensor], t_start,
           scale: float = 1.0, uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET) -> torch.Tensor:
    """UniPCSampler.decode: chart b from iteration S - t_start[b] on, warming up with its own history"""
    B, S = x_latent.shape[0], sched.S
    starts = [int(t_start)] * B if isinstance(t_start, int) else [int(s) for s in t_start]
    if max(starts) == 0:
        return x_latent
    kp, kc = U.chart_orders(sched, starts)
    return _loop(p, sched.t, sched.ns, sched.variant, sched.model_times, x_latent, [S - s for s in starts], [S] * B,
                 lambda b, i: int(kp[b, i]), lambda b, i: int(kc[b, i]), c, w, scale, uc, cfg)


def invert(p: orc.Params, sched: U.UniPCSchedule, x0: torch.Tensor, c: torch.Tensor, w: Sequence[torch.Tensor], t_enc,
           scale: float = 1.0, uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET) -> torch.Tensor:
    """UniPCSampler.invert: chart b runs t_enc[b] iterations of ``unipc.inversion_schedule(sched)`` from x0[b]"""
    inv = U.inversion_schedule(sched)
    B = x0.shape[0]
    stops = [int(t_enc)] * B if isinstance(t_enc, int) else [int(s) for s in t_enc]
    if max(stops) == 0:
        return x0
    return _loop(p, inv.t, inv.ns, inv.variant, inv.model_times, x0, [0] * B, stops, lambda b, i: int(inv.orders[i]),
                 lambda b, i: int(inv.orders[i - 1]) if inv.corrector[i] else 0, c, w, scale, uc, cfg)
