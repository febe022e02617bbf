"""UniPC multistep (Zhao et al., 2023, "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling of Diffusion Models"), the
data-prediction form with the B(h) variants bh1 / bh2: host math only.

Pure numpy in float64; nothing here needs a GPU.  The noise schedule, the grids and the model times are DPM-Solver++'s
(``dpm_solver``).  Evaluation i (i = 0 .. S-1) runs at model_time(t_i) on the latent x~_i (x~_0 = x_T) and gives the data prediction
m_i = (x~_i - sigma_i e_i) / alpha_i.  Step j (j = 1 .. S) goes from t_j-1 to t_j with order k_j and, with h = lambda_j - lambda_j-1,
hh = -h, phi = expm1(hh):

    rk_m = (lambda_j-1-m - lambda_j-1) / h  (m = 1 .. k-1), rk_k = 1        D_m = (m_j-1-m - m_j-1) / rk_m
    B_h  = hh (bh1) or phi (bh2)         b_i = g f / B_h for i = 1 .. k, from g = phi / hh - 1, f = 1, then f *= i + 1, g = g / hh - 1 / f
    R    = [rk^0; rk^1; ..; rk^(k-1)]     base = (sigma_j / sigma_j-1) x_j-1 - alpha_j phi m_j-1
    UniP (predictor)  x~_j = base - alpha_j B_h sum_m rhop_m D_m                      rhop = [0.5] (k = 2), R[:-1, :-1]^-1 b[:-1] (k = 3)
    UniC (corrector)  x_j  = base - alpha_j B_h (sum_m rhoc_m D_m + rhoc_k (m_j - m_j-1))   rhoc = [0.5] (k = 1), R^-1 b (k >= 2)

The corrector needs m_j, which evaluation j computes anyway for the next step, so a step costs one U-Net evaluation.  It is off on
step S and on the steps of ``disable_corrector``; where it is off, x_j = x~_j.  This is the official ``multistep_uni_pc_bh_update``
with predict_x0=True.  Each step is expanded into two coefficient rows, applied by the update kernel (csrc/dpm.cu) in iteration i:

    corrector row i  (A', dn, d0, d1, d2, k_i, on, 0):      x_i    = A' x_i-1 + dn m_i + d0 m_i-1 + d1 m_i-2 + d2 m_i-3   (if on)
    predictor row i  (alpha_i, sigma_i, A, c0, c1, c2, k_i+1, 0):  x~_i+1 = A x_i + c0 m_i + c1 m_i-1 + c2 m_i-2

The predictor row has dpm_solver's row layout (ROW_*), so the kernels share its arithmetic.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import dpm_solver
from .dpm_solver import MAX_STEPS, ROW_WIDTH, NoiseScheduleVP

VARIANTS = ("bh1", "bh2")
ORDERS = (1, 2, 3)
# columns of a corrector row (the kernel's second [S][8] table; column 7 is padding)
CORR_A, CORR_DN, CORR_D0, CORR_D1, CORR_D2, CORR_ORDER, CORR_ON = range(7)


def step_orders(S: int, order: int, lower_order_final: bool) -> np.ndarray:
    """[S] the order k_j of step j = 1 .. S (index j - 1): min(j, order), and with lower_order_final min(k_j, S + 1 - j) at every S.
    This is UniPC's rule; DPM-Solver++ (``dpm_solver.step_orders``) lowers the final orders only when S < 15."""
    j = np.arange(1, S + 1)
    k = np.minimum(j, order)
    if lower_order_final:
        k = np.minimum(k, S + 1 - j)
    return k.astype(np.int64)


def coefficients(j: int, k: int, lam, variant: str):
    """(h, phi, B_h, rk [k], b [k], R [k, k]) of the order-k step j on a grid with these lambdas (float64)"""
    h = lam[j] - lam[j - 1]
    hh = -h
    phi = np.expm1(hh)
    rk = np.array([(lam[j - 1 - m] - lam[j - 1]) / h for m in range(1, k)] + [1.])
    B_h = hh if variant == "bh1" else phi
    b, g, f = [], phi / hh - 1., 1.
    for i in range(1, k + 1):
        b.append(g * f / B_h)
        f *= i + 1
        g = g / hh - 1. / f
    R = np.stack([rk ** (i - 1) for i in range(1, k + 1)])
    return h, phi, B_h, rk, np.array(b), R


def rho_predictor(k: int, R, b) -> np.ndarray:
    if k == 1:
        return np.zeros(0)
    if k == 2:
        return np.array([0.5])
    return np.linalg.solve(R[:-1, :-1], b[:-1])


def rho_corrector(k: int, R, b) -> np.ndarray:
    return np.array([0.5]) if k == 1 else np.linalg.solve(R, b)


def predictor_row(j: int, k: int, alpha, sigma, lam, variant: str) -> np.ndarray:
    """predictor row j - 1 (alpha_j-1, sigma_j-1, A, c0, c1, c2, k, 0): x~_j = A x_j-1 + c0 m_j-1 + c1 m_j-2 + c2 m_j-3, the UniP
    update of step j expanded from its D-form"""
    h, phi, B_h, rk, b, R = coefficients(j, k, lam, variant)
    rho = rho_predictor(k, R, b)
    w = alpha[j] * B_h
    c = np.zeros(3)
    c[0] = -alpha[j] * phi
    for m in range(1, k):                                         # - w rho_m (m_j-1-m - m_j-1) / rk_m
        c[m] -= w * rho[m - 1] / rk[m - 1]
        c[0] += w * rho[m - 1] / rk[m - 1]
    return np.array([alpha[j - 1], sigma[j - 1], sigma[j] / sigma[j - 1], c[0], c[1], c[2], k, 0.])


def corrector_row(j: int, k: int, alpha, sigma, lam, variant: str) -> np.ndarray:
    """corrector row j (A', dn, d0, d1, d2, k, 1, 0): x_j = A' x_j-1 + dn m_j + d0 m_j-1 + d1 m_j-2 + d2 m_j-3, the UniC update of
    step j expanded from its D-form"""
    h, phi, B_h, rk, b, R = coefficients(j, k, lam, variant)
    rho = rho_corrector(k, R, b)
    w = alpha[j] * B_h
    d = np.zeros(3)
    d[0] = -alpha[j] * phi + w * rho[k - 1]                       # - w rho_k (m_j - m_j-1)
    dn = -w * rho[k - 1]
    for m in range(1, k):                                         # - w rho_m (m_j-1-m - m_j-1) / rk_m
        d[m] -= w * rho[m - 1] / rk[m - 1]
        d[0] += w * rho[m - 1] / rk[m - 1]
    return np.array([sigma[j] / sigma[j - 1], dn, d[0], d[1], d[2], k, 1., 0.])


@dataclass
class UniPCSchedule:
    """One request's tables: ``model_times`` [S] float32 (evaluation i runs at model_times[i]), the predictor ``rows`` [S, 8] (row i is
    step i + 1) and the corrector rows ``corr_rows`` [S, 8] (row i is step i; row 0 and the steps without corrector are off: all zero
    but the order column) in float64, the continuous grid ``t`` [S + 1], each step's order ``orders`` [S] (orders[i] = k_i+1) and
    whether step j's corrector runs, ``corrector`` [S] (index j; corrector[0] is False)."""
    t: np.ndarray
    model_times: np.ndarray
    rows: np.ndarray
    corr_rows: np.ndarray
    orders: np.ndarray
    corrector: np.ndarray
    order: int
    variant: str
    ns: NoiseScheduleVP

    @property
    def S(self) -> int:
        return int(self.rows.shape[0])

    def rows_f32(self) -> np.ndarray:
        """the predictor rows rounded once to float32, as the kernel reads them"""
        return np.ascontiguousarray(self.rows, dtype=np.float32)

    def corr_rows_f32(self) -> np.ndarray:
        """the corrector rows rounded once to float32, as the kernel reads them"""
        return np.ascontiguousarray(self.corr_rows, dtype=np.float32)


def multistep_schedule(alphas_cumprod, S: int, order: int = 2, skip_type: str = "time_uniform", variant: str = "bh2",
                       lower_order_final: bool = True, use_corrector: bool = True, disable_corrector: Sequence[int] = (),
                       t_grid: Optional[np.ndarray] = None) -> UniPCSchedule:
    """The coefficient rows of an S-step UniPC request of ``order`` (1..3) on ``skip_type``'s grid, or on ``t_grid`` (S + 1
    decreasing times from 1 to 1/N, e.g. ``dpm_solver.ddim_grid``).  ``disable_corrector``: steps j in [1, S - 1] that run the
    predictor alone; ``use_corrector=False`` turns the corrector off everywhere (UniP alone).  ValueError for malformed arguments."""
    if isinstance(order, bool) or not isinstance(order, (int, np.integer)) or order not in ORDERS:
        raise ValueError(f"order={order!r}: UniPC runs order 1, 2 or 3")
    if isinstance(S, bool) or not isinstance(S, (int, np.integer)) or not 0 < S <= MAX_STEPS:
        raise ValueError(f"S={S!r}: the number of steps must be an integer in [1, {MAX_STEPS}]")
    if S < order:
        raise ValueError(f"S={S}: order {order} needs at least {order} steps")
    if variant not in VARIANTS:
        raise ValueError(f"variant={variant!r}: one of {VARIANTS}")
    if t_grid is None and skip_type not in dpm_solver.SKIP_TYPES:
        raise ValueError(f"skip_type={skip_type!r}: one of {dpm_solver.SKIP_TYPES}")
    for name, v in (("lower_order_final", lower_order_final), ("use_corrector", use_corrector)):
        if v not in (True, False):
            raise ValueError(f"{name}={v!r} must be True or False")
    try:
        off = sorted({int(j) for j in disable_corrector if not isinstance(j, bool) and int(j) == j})
        bad = len(off) != len(set(disable_corrector)) or any(j < 1 or j > S - 1 for j in off)
    except (TypeError, ValueError):
        bad = True
    if bad:
        raise ValueError(f"disable_corrector={disable_corrector!r}: steps in [1, S - 1 = {S - 1}]")
    S, order = int(S), int(order)
    ns = NoiseScheduleVP(alphas_cumprod)
    t = dpm_solver.request_grid(ns, skip_type, S, t_grid)
    alpha, sigma, lam = ns.marginal_alpha(t), ns.marginal_std(t), ns.marginal_lambda(t)
    orders = step_orders(S, order, bool(lower_order_final))
    rows = np.stack([predictor_row(j, int(orders[j - 1]), alpha, sigma, lam, variant) for j in range(1, S + 1)])
    corrector = np.zeros(S, dtype=bool)
    if use_corrector:
        corrector[1:] = True
        corrector[off] = False
    corr = np.zeros((S, ROW_WIDTH))
    for j in range(1, S):
        corr[j, CORR_ORDER] = orders[j - 1]
        if corrector[j]:
            corr[j] = corrector_row(j, int(orders[j - 1]), alpha, sigma, lam, variant)
    return UniPCSchedule(t=t, model_times=dpm_solver.model_time(ns, t[:-1]), rows=rows, corr_rows=corr, orders=orders,
                         corrector=corrector, order=order, variant=variant, ns=ns)

