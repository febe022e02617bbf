"""CPU oracle of DPM-Solver++ / DDIM inversion -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A torch-fp32 restatement over oracle/mug_oracle.py's U-Net, in the stop-aware update kernel's order, of ``invert``: chart b runs
steps 0 .. t_enc[b] - 1 of an inversion schedule from x0[b]; step j evaluates the U-Net at model_times[j] and applies row j, in DDIM's
form x = alpha_j+1 m0 + sigma_j+1 e when the row's ROW_FORM is set, otherwise in the expanded form of dpm_remix_oracle's ``_update``.
A chart that has run its steps keeps its latent.  The rows come from mug_diffusion_b200.dpm_solver.inversion_schedule, whose D-form
tests/test_dpm_invert.py checks in float64."""
from typing import Optional, Sequence

import torch

from dpm_remix_oracle import _eps, _update
from mug_diffusion_b200 import dpm_solver as D
from oracle import mug_oracle as orc


def step_row(r, x, e, hist, k):
    """one inversion row: (x, m0) of DDIM's form for a FORM_EPS row, else the expanded form up to order k"""
    if float(r[D.ROW_FORM]) != D.FORM_EXPANDED:
        m0 = (x - r[D.ROW_SIGMA] * e) / r[D.ROW_ALPHA]
        return r[D.ROW_C1] * m0 + r[D.ROW_C2] * e, m0
    return _update(r, x, e, hist, k)


def invert(p: orc.Params, inv: D.DPMSchedule, x0: torch.Tensor, c: torch.Tensor, w: Sequence[torch.Tensor], t_enc,
           scale: float = 1.0, uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET) -> torch.Tensor:
    """invert over the rows of ``inv`` (an inversion_schedule): one loop of m = max(t_enc) iterations, every chart from step 0"""
    B = x0.shape[0]
    stops = [int(t_enc)] * B if isinstance(t_enc, int) else [int(s) for s in t_enc]
    rows = torch.from_numpy(inv.rows_f32())
    x, hist = x0, []
    for j in range(max(stops)):
        t = torch.full((B,), float(inv.model_times[j]), dtype=torch.float32)
        e = _eps(p, x, t, c, w, scale, uc, cfg)
        xn, m0 = step_row(rows[j], x, e, hist, int(inv.orders[j]))
        run = torch.tensor([j < s for s in stops]).view(B, 1, 1)
        x = torch.where(run, xn, x)
        hist = (hist + [m0])[-2:]
    return x
