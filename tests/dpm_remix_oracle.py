"""CPU oracle of DPM-Solver++ inpainting and remix -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-fp32 restatement over oracle/mug_oracle.py's U-Net, in the update kernel's order, of
  * inpainting: before the evaluation of step i, x <- (alpha_i x0 + sigma_i eps_i) * mask + (1 - mask) * x with the schedule's
    (alpha_i, sigma_i) in float32 and the given per-step noise eps_i;
  * remix (decode): chart b runs steps S - t_start[b] .. S - 1 from x_latent[b], at step i with order
    min(orders[i], i - (S - t_start[b]) + 1) and that order's coefficient row of the per-order table; held charts keep their latent.
The rows come from mug_diffusion_b200.dpm_solver, whose D-form tests/test_dpm_solver.py and tests/test_dpm_remix.py check in float64."""
from typing import Optional, Sequence

import torch

from mug_diffusion_b200 import dpm_solver as D
from oracle import mug_oracle as orc


def _eps(p, x, t, c, w, scale, uc, cfg):
    if uc is None or scale == 1.0:
        return orc.unet_forward(p, x, t, c, w, cfg)
    eo = orc.unet_forward(p, torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c]), [torch.cat([wi, wi]) for wi in w], cfg)
    e_u, e_c = eo.chunk(2)
    return e_u + scale * (e_c - e_u)


def _update(r, x, e, hist, k):
    """one row of the per-step update: m0 = (x - sigma e) / alpha, x = ((A x + c0 m0) + c1 m1) + c2 m2 (terms up to order k)"""
    m0 = (x - r[D.ROW_SIGMA] * e) / r[D.ROW_ALPHA]
    xn = r[D.ROW_A] * x + r[D.ROW_C0] * m0
    if k >= 2:
        xn = xn + r[D.ROW_C1] * hist[-1]
    if k >= 3:
        xn = xn + r[D.ROW_C2] * hist[-2]
    return xn, m0


def inpaint(p: orc.Params, sched: D.DPMSchedule, c: torch.Tensor, w: Sequence[torch.Tensor], x_T: torch.Tensor, mask: torch.Tensor,
            x0: torch.Tensor, q_noise: Sequence[torch.Tensor], scale: float = 1.0, uc: Optional[torch.Tensor] = None,
            cfg: dict = orc.DEFAULT_UNET):
    """the S steps of DPMSolverSampler.inpaint from x_T with q_noise[i] the blend noise of step i; returns the final x"""
    rows = torch.from_numpy(sched.rows_f32())
    B = x_T.shape[0]
    x, hist = x_T, []
    for i in range(sched.S):
        r = rows[i]
        x_orig = r[D.ROW_ALPHA] * x0 + r[D.ROW_SIGMA] * q_noise[i]
        x = x_orig * mask + (1. - mask) * x
        t = torch.full((B,), float(sched.model_times[i]), dtype=torch.float32)
        x, m0 = _update(r, x, _eps(p, x, t, c, w, scale, uc, cfg), hist, int(r[D.ROW_ORDER]))
        hist = (hist + [m0])[-2:]
    return x


def decode(p: orc.Params, sched: D.DPMSchedule, x_latent: torch.Tensor, c: torch.Tensor, w: Sequence[torch.Tensor], t_start,
           scale: float = 1.0, uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET) -> torch.Tensor:
    """DPMSolverSampler.decode: one loop of m = max(t_start) iterations from step S - m, every chart at its own order"""
    S = sched.S
    B = x_latent.shape[0]
    starts = [int(t_start)] * B if isinstance(t_start, int) else [int(s) for s in t_start]
    m = max(starts)
    if m == 0:
        return x_latent
    orders = D.chart_orders(sched, starts)
    by_order = torch.from_numpy(sched.order_rows_f32())
    x, hist = x_latent, []
    for i in range(S - m, S):
        t = torch.full((B,), float(sched.model_times[i]), dtype=torch.float32)
        e = _eps(p, x, t, c, w, scale, uc, cfg)
        xs, ms = [], []
        for b in range(B):
            k = int(orders[b, i])
            if k == 0:                                                   # held: the latent stays, no prediction is formed
                xs.append(x[b:b + 1])
                ms.append(torch.full_like(x[b:b + 1], float("nan")))
                continue
            xb, mb = _update(by_order[i, k - 1], x[b:b + 1], e[b:b + 1], [h[b:b + 1] for h in hist], k)
            xs.append(xb)
            ms.append(mb)
        x = torch.cat(xs)
        hist = (hist + [torch.cat(ms)])[-2:]
    return x
