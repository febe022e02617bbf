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

A chart that joins a request late (remix: ``chart_orders``) warms up like a fresh request: at iteration i, from its first iteration f,
its predictor takes order min(orders[i], i - f + 1) and its corrector runs only for i > f (there is no earlier evaluation at f), at
order min(orders[i - 1], i - f).  ``order_rows`` / ``order_corr`` hold those rows per order.  ``inversion_schedule`` runs the
request's ODE backwards on the reversed grid.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import dpm_solver
from .dpm_solver import FORM_EPS, MAX_STEPS, ROW_C1, ROW_C2, ROW_FORM, ROW_WIDTH, GridTables, NoiseScheduleVP

VARIANTS = ("bh1", "bh2")
ORDERS = (1, 2, 3)
# columns of a corrector row (the kernel's second [S][8] table; column 7 is padding, except in inversion rows: CORR_FORM)
CORR_A, CORR_DN, CORR_D0, CORR_D1, CORR_D2, CORR_ORDER, CORR_ON, CORR_FORM = range(8)
# an inversion corrector row with CORR_FORM = FORM_DIFF is taken in the correction form (``correction_row``), which never multiplies
# the previous corrected latent by A'
FORM_DIFF = 1.


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


def correction_row(j: int, k: int, alpha, sigma, lam, variant: str) -> np.ndarray:
    """corrector row j in the correction form (A', dn, d0, e1, e2, k, 1, FORM_DIFF): UniC minus UniP of step j,
        x_j = x~_j + ((dn (m_j - m_j-1) + e1 (m_j-2 - m_j-1)) + e2 (m_j-3 - m_j-1))       (the e1 term for k >= 2, e2 for k = 3)
    with e_m = -alpha_j B_h (rhoc_m - rhop_m) / rk_m; A' and d0 are the expanded row's (not read in this form).  It holds where x~_j is
    the predictor's own output, which an inversion never blends."""
    h, phi, B_h, rk, b, R = coefficients(j, k, lam, variant)
    rc, rp = rho_corrector(k, R, b), rho_predictor(k, R, b)
    w = alpha[j] * B_h
    row = corrector_row(j, k, alpha, sigma, lam, variant)
    row[CORR_D1] = row[CORR_D2] = 0.
    for m in range(1, k):
        row[CORR_D0 + m] = -w * (rc[m - 1] - rp[m - 1]) / rk[m - 1]
    row[CORR_FORM] = FORM_DIFF
    return row


@dataclass
class UniPCSchedule(GridTables):
    """One request's tables: ``model_times`` [S] float32 (evaluation i runs at model_times[i]), the predictor ``rows`` [S, 8] (row i is
    step i + 1) and the corrector rows ``corr_rows`` [S, 8] (row i is step i; row 0 and the steps without corrector are off: all zero
    but the order column) in float64, the continuous grid ``t`` [S + 1], each step's order ``orders`` [S] (orders[i] = k_i+1) and
    whether step j's corrector runs, ``corrector`` [S] (index j; corrector[0] is False).  ``order_rows`` / ``order_corr`` [S, 3, 8]
    (float64) hold the rows a late-joining chart takes (``chart_orders``): row (i, k - 1) is the order-k predictor of iteration i
    (k <= orders[i]) and the order-k corrector of iteration i (k <= orders[i - 1], where the corrector runs), NaN where no chart can
    read; row (i, orders[i] - 1) equals rows[i] and, where the corrector runs, row (i, orders[i - 1] - 1) equals corr_rows[i].  They
    are None in an ``inversion_schedule``.  ``use_corrector``: whether the request asked for a corrector at all."""
    t: np.ndarray
    model_times: np.ndarray
    rows: np.ndarray
    corr_rows: np.ndarray
    orders: np.ndarray
    corrector: np.ndarray
    order: int
    variant: str
    ns: NoiseScheduleVP
    order_rows: Optional[np.ndarray] = None
    order_corr: Optional[np.ndarray] = None
    use_corrector: bool = True

    @property
    def S(self) -> int:
        return int(self.rows.shape[0])

    def rows_f32(self) -> np.ndarray:
        """the predictor rows rounded once to float32, as the kernel reads them"""
        return np.ascontiguousarray(self.rows, dtype=np.float32)

    def corr_rows_f32(self) -> np.ndarray:
        """the corrector rows rounded once to float32, as the kernel reads them"""
        return np.ascontiguousarray(self.corr_rows, dtype=np.float32)

    def order_rows_f32(self) -> np.ndarray:
        """``order_rows`` rounded once to float32, as the per-chart update kernel reads them"""
        return np.ascontiguousarray(self.order_rows, dtype=np.float32)

    def order_corr_f32(self) -> np.ndarray:
        """``order_corr`` rounded once to float32, as the per-chart update kernel reads them"""
        return np.ascontiguousarray(self.order_corr, dtype=np.float32)


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
    by_order = np.full((S, 3, ROW_WIDTH), np.nan)
    corr_by_order = np.full((S, 3, ROW_WIDTH), np.nan)
    for i in range(S):
        for k in range(1, int(orders[i]) + 1):
            by_order[i, k - 1] = predictor_row(i + 1, k, alpha, sigma, lam, variant)
        if corrector[i]:
            for k in range(1, int(orders[i - 1]) + 1):
                corr_by_order[i, k - 1] = corrector_row(i, k, alpha, sigma, lam, variant)
    return UniPCSchedule(t=t, model_times=dpm_solver.model_time(ns, t[:-1]), rows=rows, corr_rows=corr, orders=orders,
                         corrector=corrector, order=order, variant=variant, ns=ns, order_rows=by_order, order_corr=corr_by_order,
                         use_corrector=bool(use_corrector))


def chart_orders(sched: UniPCSchedule, starts):
    """([B, S], [B, S]) the predictor and corrector orders each chart takes at each iteration when chart b runs iterations
    f_b = S - starts[b] .. S - 1: predictor min(orders[i], i - f_b + 1) from f_b on; corrector min(orders[i - 1], i - f_b) where the
    request's corrector runs and i > f_b.  0 while the chart is held, and 0 where its corrector does not run."""
    S = sched.S
    i = np.arange(S)[None, :]
    first = S - np.asarray(starts, dtype=np.int64)[:, None]
    kp = np.where(i >= first, np.minimum(sched.orders[None, :], i - first + 1), 0)
    prev = np.concatenate([[0], sched.orders[:-1]])[None, :]
    kc = np.where(sched.corrector[None, :] & (i > first), np.minimum(prev, i - first), 0)
    return kp, kc


def inversion_schedule(sched: UniPCSchedule) -> UniPCSchedule:
    """The tables of the inversion of ``sched`` (a ``multistep_schedule``): UniPC run backwards on the reversed grid u_j = t_S-j,
    j = 0 .. S.  Iteration j evaluates the U-Net at model_time(u_j); its predictor has order min(j + 1, order) (no lower_order_final:
    charts stop at different steps) and its corrector runs on every j >= 1 when ``sched`` asked for a corrector (its
    ``disable_corrector`` steps do not carry over).  After s iterations a chart sits at t_S-s, where a remix over the last s steps of
    ``sched`` starts.  Two forms keep every step within 1e-6 of max |x| in float32 (the first steps leave u_0 = 1/N, where sigma is
    about 0.01, so sigma_1 / sigma_0 reaches 17 on the time-uniform grid at S = 10):
      - every corrector row is in the correction form (``correction_row``, CORR_FORM = FORM_DIFF), which never multiplies the previous
        corrected latent by A';
      - every order-1 predictor row also carries DDIM's form (ROW_FORM = FORM_EPS, alpha_j+1 / sigma_j+1 in the c1 / c2 columns), as
        ``dpm_solver.inversion_schedule``'s rows do: x~_j+1 = (alpha_j+1 m_j + sigma_j+1 e) + A c, where e is the eps of x~_j and c the
        correction x_j - x~_j of this iteration (no term where the corrector does not run), which equals A x_j + c0 m_j."""
    if not isinstance(sched, UniPCSchedule) or sched.ns is None or sched.order not in ORDERS:
        raise ValueError("sched must be a UniPCSchedule from multistep_schedule")
    ns, S, variant = sched.ns, sched.S, sched.variant
    u = np.ascontiguousarray(sched.t[::-1], dtype=np.float64)
    alpha, sigma, lam = ns.marginal_alpha(u), ns.marginal_std(u), ns.marginal_lambda(u)
    orders = np.minimum(np.arange(S) + 1, sched.order).astype(np.int64)
    rows = np.stack([predictor_row(j + 1, int(orders[j]), alpha, sigma, lam, variant) for j in range(S)])
    corrector = np.zeros(S, dtype=bool)
    corrector[1:] = bool(sched.use_corrector)
    corr = np.zeros((S, ROW_WIDTH))
    for j in range(1, S):
        corr[j, CORR_ORDER] = orders[j - 1]
        if corrector[j]:
            corr[j] = correction_row(j, int(orders[j - 1]), alpha, sigma, lam, variant)
    eps = orders == 1
    rows[eps, ROW_C1], rows[eps, ROW_C2], rows[eps, ROW_FORM] = alpha[1:][eps], sigma[1:][eps], FORM_EPS
    return UniPCSchedule(t=u, model_times=dpm_solver.model_time(ns, u[:-1]), rows=rows, corr_rows=corr, orders=orders,
                         corrector=corrector, order=sched.order, variant=variant, ns=ns, use_corrector=bool(sched.use_corrector))

