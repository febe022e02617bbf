"""CPU oracle of the UniPC sampler -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

UniPC's data-prediction bh update (Zhao et al., 2023; the official ``multistep_uni_pc_bh_update`` with predict_x0=True) stepped in its
D-form, not through the expanded coefficient rows of mug_diffusion_b200.unipc: ``d_form_step`` works on numpy float64 arrays and on
torch tensors, and ``unipc_sample`` runs the predictor / evaluation / corrector loop in torch fp32 over oracle/mug_oracle.py's U-Net,
with every step's coefficients solved in float64.
``d_form`` computes b, R and rho by the same published formulas as ``unipc.coefficients`` (they are the contract), so it is not an
independent statement of them: what this oracle checks is the expansion into rows, the kernel's order and the loop.  The formulas
themselves are pinned by tests/test_unipc.py's slopes on the analytic Gaussian model and by the exact agreements with DPM-Solver++ 2M
(UniP-2 bh2) and DDIM (order 1 without corrector)."""
from typing import Optional, Sequence

import numpy as np
import torch

from dpm_remix_oracle import _eps
from oracle import mug_oracle as orc


def d_form(lam, j, k, variant):
    """(phi, B_h, rk [k - 1], rho_p [k - 1], rho_c [k]) of the order-k step j from t_j-1 to t_j on a grid with these lambdas"""
    h = lam[j] - lam[j - 1]
    hh = -h
    phi = np.expm1(hh)
    rks = np.array([(lam[j - 1 - m] - lam[j - 1]) / h for m in range(1, k)] + [1.])
    B_h = hh if variant == "bh1" else phi
    h_phi_k, factorial, R, b = phi / hh - 1., 1., [], []
    for i in range(1, k + 1):
        R.append(rks ** (i - 1))
        b.append(h_phi_k * factorial / B_h)
        factorial *= i + 1
        h_phi_k = h_phi_k / hh - 1. / factorial
    R, b = np.stack(R), np.array(b)
    rho_p = np.zeros(0) if k == 1 else np.array([0.5]) if k == 2 else np.linalg.solve(R[:-1, :-1], b[:-1])
    rho_c = np.array([0.5]) if k == 1 else np.linalg.solve(R, b)
    return phi, B_h, rks[:-1], rho_p, rho_c


def d_form_step(x_prev, ms, j, k, alpha, sigma, lam, variant, m_new=None):
    """step j of order k from x_prev = x_j-1 with ms = [m_j-1, m_j-2, ...] (newest first): UniP's x~_j, or with ``m_new`` = m_j UniC's
    x_j = base - alpha_j B_h (sum_m rho_c,m D_m + rho_c,k (m_j - m_j-1)), D_m = (m_j-1-m - m_j-1) / rk_m"""
    phi, B_h, rk, rho_p, rho_c = d_form(lam, j, k, variant)
    base = float(sigma[j] / sigma[j - 1]) * x_prev - float(alpha[j] * phi) * ms[0]
    D = [(ms[m] - ms[0]) / float(rk[m - 1]) for m in range(1, k)]
    rho = rho_p if m_new is None else rho_c
    res = 0. * ms[0]
    for m in range(k - 1):
        res = res + float(rho[m]) * D[m]
    if m_new is not None:
        res = res + float(rho_c[-1]) * (m_new - ms[0])
    return base - float(alpha[j] * B_h) * res


def unipc_sample(p: orc.Params, sched, c: torch.Tensor, w: Sequence[torch.Tensor], x_T: torch.Tensor, scale: float = 1.0,
                 uc: Optional[torch.Tensor] = None, cfg: dict = orc.DEFAULT_UNET, log_every_t: int = 100):
    """The S iterations of a UniPC request of ``sched`` (a UniPCSchedule: its grid, orders, corrector steps and variant): iteration i
    evaluates the U-Net on x~_i at model_times[i], forms m_i, corrects step i (when its corrector runs) and predicts x~_i+1.  Returns
    (x~_S, {'x_inter': [...], 'pred_x0': [...]}) with DDIM's logging rule: x~_i+1 and m_i after iteration i."""
    ns = sched.ns
    alpha, sigma, lam = ns.marginal_alpha(sched.t), ns.marginal_std(sched.t), ns.marginal_lambda(sched.t)
    B, S = x_T.shape[0], sched.S
    x = xt = x_T
    ms = []
    intermediates = {'x_inter': [x_T], 'pred_x0': [x_T]}
    for i in range(S):
        t = torch.full((B,), float(sched.model_times[i]), dtype=torch.float32)
        e = _eps(p, xt, t, c, w, scale, uc, cfg)
        m = (xt - float(sigma[i]) * e) / float(alpha[i])
        x = d_form_step(x, ms, i, int(sched.orders[i - 1]), alpha, sigma, lam, sched.variant, m_new=m) if sched.corrector[i] else xt
        ms = [m] + ms[:2]
        xt = d_form_step(x, ms, i + 1, int(sched.orders[i]), alpha, sigma, lam, sched.variant)
        index = S - i - 1
        if index % log_every_t == 0 or index == S - 1:
            intermediates['x_inter'].append(xt)
            intermediates['pred_x0'].append(m)
    return xt, intermediates
