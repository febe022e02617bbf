"""CPU oracle of the DPM-Solver++ multistep sampler -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-fp32 restatement over oracle/mug_oracle.py's U-Net: each step evaluates the U-Net at the schedule's float model time, forms
the CFG-combined eps and the data prediction m = (x - sigma * e) / alpha, and applies the step's coefficient row
x = ((A x + c0 m0) + c1 m1) + c2 m2 in the update kernel's order.  The rows come from mug_diffusion_b200.dpm_solver, whose D-form
tests/test_dpm_solver.py checks in float64."""
from typing import Optional, Sequence

import torch

from mug_diffusion_b200 import dpm_solver
from oracle import mug_oracle as orc


def dpm_sample(p: orc.Params, sched: dpm_solver.DPMSchedule, c: torch.Tensor, w: Sequence[torch.Tensor], x_T: torch.Tensor,
               scale: float = 1.0, uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET, log_every_t: int = 100):
    """Returns (x, {'x_inter': [...], 'pred_x0': [...]}) with DDIM's logging rule over the S steps."""
    rows = torch.from_numpy(sched.rows_f32())
    B = x_T.shape[0]
    S = sched.S
    x = x_T
    intermediates = {'x_inter': [x], 'pred_x0': [x]}
    hist = []                                                            # m of the previous steps, newest last
    for i in range(S):
        t = torch.full((B,), float(sched.model_times[i]), dtype=torch.float32)
        if uc is None or scale == 1.0:
            e = orc.unet_forward(p, x, t, c, w, cfg)
        else:
            eo = orc.unet_forward(p, torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c]), [torch.cat([wi, wi]) for wi in w], cfg)
            e_u, e_c = eo.chunk(2)
            e = e_u + scale * (e_c - e_u)
        r = rows[i]
        m0 = (x - r[dpm_solver.ROW_SIGMA] * e) / r[dpm_solver.ROW_ALPHA]
        k = int(r[dpm_solver.ROW_ORDER])
        xn = r[dpm_solver.ROW_A] * x + r[dpm_solver.ROW_C0] * m0
        if k >= 2:
            xn = xn + r[dpm_solver.ROW_C1] * hist[-1]
        if k >= 3:
            xn = xn + r[dpm_solver.ROW_C2] * hist[-2]
        x = xn
        hist = (hist + [m0])[-2:]
        index = S - i - 1
        if index % log_every_t == 0 or index == S - 1:
            intermediates['x_inter'].append(x)
            intermediates['pred_x0'].append(m0)
    return x, intermediates
