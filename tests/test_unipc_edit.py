"""UniPC inpainting, remix and inversion, CPU side: the per-order predictor and corrector rows against the float64 D-form, the NaN of
rows no chart can read, the chart_orders rule, the inversion rows against D-form stepping on the reversed grid, the float32 conditioning
of every inversion step, analytic-Gaussian error slopes of a remix and of the invert -> decode round trip, order 1 on DDIM's grid
against the reference's remix goldens through the oracle, the C entry points' argument checks and the sampler's refusals before any
GPU work."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

import golden_cases as gc
import remix_cases as rc
import unipc_edit_oracle as ueo
from mug_diffusion_b200 import dpm_solver as D
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth
from mug_diffusion_b200 import unipc as U
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.sampler import UniPCSampler, ddim_timesteps_uniform, register_schedule
from test_unipc import ACP, NS, data_prediction, gaussian_exact, gaussian_run
from unipc_oracle import d_form_step

GRIDS = ("time_uniform", "logSNR", "time_quadratic")


def grid(t):
    return NS.marginal_alpha(t), NS.marginal_std(t), NS.marginal_lambda(t)


def close(got, want):
    return np.abs(got - want).max() < 1e-12 * max(1., np.abs(want).max())


def apply_predictor(row, k, x, ms):
    out = row[D.ROW_A] * x + row[D.ROW_C0] * ms[0]
    out = out + row[D.ROW_C1] * ms[1] if k >= 2 else out
    return out + row[D.ROW_C2] * ms[2] if k >= 3 else out


def apply_corrector(q, k, xc, mn, ms):
    out = q[U.CORR_A] * xc + q[U.CORR_DN] * mn + q[U.CORR_D0] * ms[0]
    out = out + q[U.CORR_D1] * ms[1] if k >= 2 else out
    return out + q[U.CORR_D2] * ms[2] if k >= 3 else out


# ---- the per-order tables ----------------------------------------------------------------------------------------------------------
CASES = [(o, v, sk, lof, S) for o in U.ORDERS for v in U.VARIANTS for sk in GRIDS for lof in (True, False) for S in (3, 5, 10, 20)
         if S >= o]


@pytest.mark.parametrize("order,variant,skip,lof,S", CASES)
def test_order_tables_equal_the_d_form(order, variant, skip, lof, S):
    sched = U.multistep_schedule(ACP, S, order, skip, variant, lof)
    alpha, sigma, lam = grid(sched.t)
    rng = np.random.default_rng(S * 7 + order)
    for i in range(S):
        for k in range(1, 4):
            row = sched.order_rows[i, k - 1]
            if k > sched.orders[i]:
                assert np.isnan(row).all(), (i, k)                       # no chart can take it
                continue
            assert row[D.ROW_ORDER] == k and row[D.ROW_ALPHA] == alpha[i] and row[D.ROW_SIGMA] == sigma[i]
            x, ms = rng.standard_normal(32), [rng.standard_normal(32) for _ in range(3)]
            assert close(apply_predictor(row, k, x, ms), d_form_step(x, ms, i + 1, k, alpha, sigma, lam, variant)), (i, k)
        assert np.array_equal(sched.order_rows[i, sched.orders[i] - 1], sched.rows[i])
        for k in range(1, 4):
            q = sched.order_corr[i, k - 1]
            if not sched.corrector[i] or k > sched.orders[i - 1]:
                assert np.isnan(q).all(), (i, k)
                continue
            assert q[U.CORR_ORDER] == k and q[U.CORR_ON] == 1
            xc, mn, ms = rng.standard_normal(32), rng.standard_normal(32), [rng.standard_normal(32) for _ in range(3)]
            assert close(apply_corrector(q, k, xc, mn, ms), d_form_step(xc, ms, i, k, alpha, sigma, lam, variant, m_new=mn)), (i, k)
        if sched.corrector[i]:
            assert np.array_equal(sched.order_corr[i, sched.orders[i - 1] - 1], sched.corr_rows[i])


def test_chart_orders():
    """warm-up from each chart's first iteration, lower_order_final kept, and no corrector at a chart's first iteration"""
    sched = U.multistep_schedule(ACP, 6, 3, disable_corrector=[4])
    assert sched.orders.tolist() == [1, 2, 3, 3, 2, 1]
    kp, kc = U.chart_orders(sched, [6, 4, 1, 0])
    assert kp.tolist() == [[1, 2, 3, 3, 2, 1], [0, 0, 1, 2, 2, 1], [0, 0, 0, 0, 0, 1], [0] * 6]
    assert kc.tolist() == [[0, 1, 2, 3, 0, 2], [0, 0, 0, 1, 0, 2], [0] * 6, [0] * 6]


# ---- inversion rows ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [3, 10])
@pytest.mark.parametrize("skip", GRIDS)
@pytest.mark.parametrize("variant", U.VARIANTS)
@pytest.mark.parametrize("order", U.ORDERS)
def test_inversion_rows_equal_the_d_form_on_the_reversed_grid(order, variant, skip, S):
    sched = U.multistep_schedule(ACP, S, order, skip, variant, True, True, disable_corrector=[1] if S > 2 else ())
    inv = U.inversion_schedule(sched)
    assert np.array_equal(inv.t, sched.t[::-1]) and np.array_equal(inv.model_times, D.model_time(NS, inv.t[:-1]))
    assert inv.orders.tolist() == [min(j + 1, order) for j in range(S)]
    assert inv.corrector.tolist() == [False] + [True] * (S - 1)                      # disable_corrector does not carry over
    assert inv.order_rows is None and inv.order_corr is None
    alpha, sigma, lam = grid(inv.t)
    rng = np.random.default_rng(S + order)
    for j in range(S):
        row, k = inv.rows[j], int(inv.orders[j])
        x, ms = rng.standard_normal(32), [rng.standard_normal(32) for _ in range(3)]
        want = d_form_step(x, ms, j + 1, k, alpha, sigma, lam, variant)
        assert close(apply_predictor(row, k, x, ms), want), j
        if k == 1:
            assert row[D.ROW_FORM] == D.FORM_EPS and row[D.ROW_C1] == alpha[j + 1] and row[D.ROW_C2] == sigma[j + 1]
            e = (x - alpha[j] * ms[0]) / sigma[j]
            assert close(row[D.ROW_C1] * ms[0] + row[D.ROW_C2] * e, want), j
        else:
            assert row[D.ROW_FORM] == D.FORM_EXPANDED
        if j >= 1:
            q, kc = inv.corr_rows[j], int(inv.orders[j - 1])
            assert q[U.CORR_FORM] == U.FORM_DIFF and q[U.CORR_ORDER] == kc
            xc, mn = rng.standard_normal(32), rng.standard_normal(32)
            want_c = d_form_step(xc, ms, j, kc, alpha, sigma, lam, variant, m_new=mn)
            xt = d_form_step(xc, ms, j, kc, alpha, sigma, lam, variant)             # the predictor's x~_j from the same xc
            c = q[U.CORR_DN] * (mn - ms[0])
            c = c + q[U.CORR_D1] * (ms[1] - ms[0]) if kc >= 2 else c
            c = c + q[U.CORR_D2] * (ms[2] - ms[0]) if kc >= 3 else c
            assert close(xt + c, want_c), j


def test_inversion_without_corrector_and_refusals():
    inv = U.inversion_schedule(U.multistep_schedule(ACP, 6, 2, use_corrector=False))
    assert not inv.corrector.any() and not inv.corr_rows[:, U.CORR_ON].any()
    for bad in (None, D.multistep_schedule(ACP, 6, 2)):
        with pytest.raises(ValueError, match="sched must be a UniPCSchedule from multistep_schedule"):
            U.inversion_schedule(bad)


# ---- float32 conditioning of every inversion step ----------------------------------------------------------------------------------
F = np.float32


def f32_predictor_error(row, rng, n=1 << 14):
    """test_dpm_invert's measurement: max |float32 kernel arithmetic - float64| / max |x| over random x, e, m1, m2 (m0 from x and e)
    and, for a DDIM-form row, a random correction c of this iteration (x = x~ + c in float64)"""
    r32 = row.astype(F)
    x, e, m1, m2, c = (rng.standard_normal(n).astype(F) for _ in range(5))
    k = int(row[D.ROW_ORDER])
    X = lambda a: a.astype(np.float64)  # noqa: E731
    m0 = (x - r32[1] * e) / r32[0]
    m64 = (X(x) - row[1] * X(e)) / row[0]
    if row[D.ROW_FORM] != D.FORM_EXPANDED:
        got = r32[4] * m0 + r32[5] * e + r32[2] * c
        want = row[2] * (X(x) + X(c)) + row[3] * m64
    else:
        got, want = r32[2] * x + r32[3] * m0, row[2] * X(x) + row[3] * m64
        if k >= 2:
            got, want = got + r32[4] * m1, want + row[4] * X(m1)
        if k >= 3:
            got, want = got + r32[5] * m2, want + row[5] * X(m2)
    return float(np.abs(got - want).max() / max(np.abs(X(x)).max(), np.abs(want).max()))


def f32_corrector_error(inv, j, q, rng, n=1 << 14):
    """the same measurement for corrector row ``q`` of iteration j: random xc (x_j-1), e, e', m_j-2, m_j-3; m_j-1 the data prediction of
    xc at u_j-1 (so A' xc and d0 m_j-1 cancel as they do on a trajectory), x~_j the predictor of iteration j - 1 and m_j its prediction"""
    k = int(q[U.CORR_ORDER])
    X = lambda a: a.astype(np.float64)  # noqa: E731
    xc, ep, e, m2, m3 = (X(rng.standard_normal(n).astype(F)) for _ in range(5))
    P, R = inv.rows[j - 1], inv.rows[j]
    m1 = X(((xc - P[1] * ep) / P[0]).astype(F))
    kp = int(P[D.ROW_ORDER])
    xt = X((P[2] * xc + P[3] * m1 + (P[4] * m2 if kp >= 2 else 0.) + (P[5] * m3 if kp >= 3 else 0.)).astype(F))
    m0 = X(((xt - R[1] * e) / R[0]).astype(F))
    q32, f = q.astype(F), lambda a: a.astype(F)  # noqa: E731
    want = q[0] * xc + q[1] * m0 + q[2] * m1 + (q[3] * m2 if k >= 2 else 0.) + (q[4] * m3 if k >= 3 else 0.)
    if q[U.CORR_FORM] == U.FORM_DIFF:
        c = q32[1] * (f(m0) - f(m1))
        c = c + q32[3] * (f(m2) - f(m1)) if k >= 2 else c
        c = c + q32[4] * (f(m3) - f(m1)) if k >= 3 else c
        got = f(xt) + c
        want = xt + q[1] * (m0 - m1) + (q[3] * (m2 - m1) if k >= 2 else 0.) + (q[4] * (m3 - m1) if k >= 3 else 0.)
    else:
        got = q32[0] * f(xc) + q32[1] * f(m0) + q32[2] * f(m1)
        got = got + q32[3] * f(m2) if k >= 2 else got
        got = got + q32[4] * f(m3) if k >= 3 else got
    return float(np.abs(X(got) - want).max() / max(np.abs(xc).max(), np.abs(xt).max(), np.abs(want).max()))


def forward(grid_name, S, order, variant, use_corrector=True):
    if grid_name == "ddim":
        ts = ddim_timesteps_uniform(S, 1000)
        return U.multistep_schedule(ACP, len(ts), order, variant=variant, use_corrector=use_corrector, t_grid=D.ddim_grid(NS, ts))
    return U.multistep_schedule(ACP, S, order, grid_name, variant, use_corrector=use_corrector)


@pytest.mark.parametrize("variant", U.VARIANTS)
@pytest.mark.parametrize("order", U.ORDERS)
@pytest.mark.parametrize("S", [10, 20, 50])
@pytest.mark.parametrize("grid_name", GRIDS + ("ddim",))
def test_every_inversion_step_is_well_conditioned_in_float32(grid_name, S, order, variant):
    """every predictor and corrector row within 1e-6 of max |x| (measured at most 3.1e-7 and 2.4e-7)"""
    for use_corrector in (True, False):
        inv = U.inversion_schedule(forward(grid_name, S, order, variant, use_corrector))
        rng = np.random.default_rng(S)
        worst_p = max(f32_predictor_error(inv.rows[j], rng) for j in range(inv.S))
        worst_c = max([f32_corrector_error(inv, j, inv.corr_rows[j], rng) for j in range(1, inv.S) if inv.corrector[j]] or [0.])
        assert worst_p < 1e-6 and worst_c < 1e-6, (use_corrector, worst_p, worst_c)


def test_the_expanded_corrector_of_the_first_step_is_the_hazard():
    """on the reversed time-uniform grid at S = 10, step 1's corrector has A' = sigma_1 / sigma_0 near 17, and its expanded form loses
    1.35e-6 of max |x| (bh1); the correction form of the same step stays near 1e-7"""
    inv = U.inversion_schedule(U.multistep_schedule(ACP, 10, 2, variant="bh1"))
    alpha, sigma, lam = grid(inv.t)
    q = U.corrector_row(1, 1, alpha, sigma, lam, "bh1")
    assert q[U.CORR_A] > 15
    assert f32_corrector_error(inv, 1, q, np.random.default_rng(10)) > 1e-6
    assert f32_corrector_error(inv, 1, inv.corr_rows[1], np.random.default_rng(10)) < 2e-7


# ---- the analytic Gaussian model ---------------------------------------------------------------------------------------------------
def gaussian_remix(sched, x, s, use_order_tables=True):
    """the per-chart loop of a chart that runs the last s iterations of ``sched`` from x, on the exact data prediction, through the
    per-order rows in the kernel's order"""
    S = sched.S
    kp, kc = U.chart_orders(sched, [s])
    xc, xt, hist = x.copy(), x.copy(), []
    for i in range(S - s, S):
        r = sched.order_rows[i, kp[0, i] - 1]
        m = data_prediction(xt, r[0], r[1])
        xi = apply_corrector(sched.order_corr[i, kc[0, i] - 1], kc[0, i], xc, m, hist[::-1]) if kc[0, i] else xt
        hist = (hist + [m])[-3:]
        xc, xt = xi, apply_predictor(r, kp[0, i], xi, hist[::-1])
    return xt


def gaussian_invert(inv, x0, steps=None):
    """the inversion rows on the exact data prediction in float64, each row in its own form"""
    xc, xt, hist = x0.copy(), x0.copy(), []
    for j in range(inv.S if steps is None else steps):
        r, q = inv.rows[j], inv.corr_rows[j]
        m = data_prediction(xt, r[0], r[1])
        c = 0.
        if q[U.CORR_ON]:
            k = int(q[U.CORR_ORDER])
            ms = hist[::-1]
            c = q[U.CORR_DN] * (m - ms[0]) + (q[U.CORR_D1] * (ms[1] - ms[0]) if k >= 2 else 0.) + \
                (q[U.CORR_D2] * (ms[2] - ms[0]) if k >= 3 else 0.)
        xi = xt + c
        hist = (hist + [m])[-3:]
        if r[D.ROW_FORM] != D.FORM_EXPANDED:
            e = (xt - r[0] * m) / r[1]
            xn = r[D.ROW_C1] * m + r[D.ROW_C2] * e + r[D.ROW_A] * c
        else:
            xn = apply_predictor(r, int(r[D.ROW_ORDER]), xi, hist[::-1])
        xc, xt = xi, xn
    return xt


X_T = np.random.default_rng(0).standard_normal(64)
X0 = gaussian_exact(np.random.default_rng(3).standard_normal(64), 1e-3)            # a sample of the data marginal at t = 1/N
STEPS = [20, 40, 80, 160]


def slope(errs, steps=STEPS):
    return float(-np.polyfit(np.log(steps), np.log(errs), 1)[0])


def test_full_strength_remix_is_the_request():
    for sched in (U.multistep_schedule(ACP, 10, 3, "logSNR"), U.multistep_schedule(ACP, 7, 2, disable_corrector=[3])):
        assert close(gaussian_remix(sched, X_T, sched.S), gaussian_run(sched, X_T))


# half-strength remix from the exact marginal at t_S/2 to t = 1/N on logSNR (bh2, no lower_order_final), measured over S = 20 .. 160:
# order 1 0.98 -> 1.98 with the corrector, order 2 1.63 -> 2.83.  Without the corrector order 2 is still pre-asymptotic here (the
# chart's first step is order 1 and its lambda step is the largest), as DPM-Solver++ 2M's remix is.
@pytest.mark.parametrize("order,corrector,lo,hi", [(1, False, 0.85, 1.15), (1, True, 1.85, 2.15), (2, False, 1.5, 1.8),
                                                   (2, True, 2.7, 3.0)])
def test_remix_global_error_slope(order, corrector, lo, hi):
    errs = []
    for S in STEPS:
        sched = U.multistep_schedule(ACP, S, order, "logSNR", "bh2", False, corrector)
        s = S // 2
        x = gaussian_exact(X_T, sched.t[S - s])
        errs.append(float(np.abs(gaussian_remix(sched, x, s) - gaussian_exact(X_T, sched.t[-1])).max()))
    assert all(a > b for a, b in zip(errs, errs[1:])), errs
    assert lo <= slope(errs) <= hi, (slope(errs), errs)


# the invert -> decode round trip on logSNR, measured over S = 20 .. 160: order 1 0.96 -> 2.25 with the corrector, order 2 2.74 -> 2.97
# (at order 2 the errors of the two directions partly cancel at these S, as they do for DPM-Solver++ 2M's round trip)
@pytest.mark.parametrize("order,corrector,lo,hi", [(1, False, 0.85, 1.1), (1, True, 2.1, 2.4), (2, False, 2.6, 2.9),
                                                   (2, True, 2.85, 3.1)])
def test_round_trip_global_error_slope(order, corrector, lo, hi):
    errs = []
    for S in STEPS:
        sched = U.multistep_schedule(ACP, S, order, "logSNR", "bh2", False, corrector)
        errs.append(float(np.abs(gaussian_remix(sched, gaussian_invert(U.inversion_schedule(sched), X0), S) - X0).max()))
    assert all(a > b for a, b in zip(errs, errs[1:])), errs
    assert lo <= slope(errs) <= hi, (slope(errs), errs)


# ---- order 1 without corrector on DDIM's grid: the reference's DDIM remix goldens through the oracle ---------------------------------
@pytest.mark.parametrize("name", [n for n, cse in rc.REMIX_CASES.items() if cse["sampler"] == "ddim" and cse["S"] == 10][:2])
def test_order_one_remix_on_the_ddim_grid_matches_the_reference(name, golden_dir):
    case = rc.REMIX_CASES[name]
    L, B = case["L"], case["B"]
    ts = ddim_timesteps_uniform(case["S"], 1000)
    sched = U.multistep_schedule(ACP, len(ts), 1, use_corrector=False, t_grid=D.ddim_grid(NS, ts))
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    inp = synth.synthetic_inputs(B, L)
    sd = synth.synthetic_state_dict(L)
    with torch.no_grad():
        z = ueo.decode(sd, sched, rc.intermediates(g, "x_inter")[0], inp["c"], inp["w"], rc.subset_end(case["k"], sched.S),
                       case["scale"], inp["uc"] if case["scale"] != 1.0 else None)
    err = float((z - torch.as_tensor(g["z"])).abs().max() / torch.as_tensor(g["z"]).abs().max())
    assert err < 1e-3, err


# ---- C ABI -------------------------------------------------------------------------------------------------------------------------
def test_library_exports_the_unipc_edit_entry_points_at_abi_13():
    lib = L_.load()
    assert lib.mugd_abi_version() == L_.ABI_VERSION == 13
    for sym in ("mugd_sample_unipc_ex", "mugd_unipc_ex_update", "mugd_sample_unipc_stop", "mugd_unipc_stop_update"):
        assert sym in L_.EXPORTED_SYMBOLS and hasattr(lib, sym)
    with open(os.path.join(os.path.dirname(L_.HERE), "include", "mugd.h")) as f:
        h = f.read()
    assert ("int  mugd_sample_unipc_ex(mugd_plan* eval_plan, const mugd_unipc_ex* e, int32_t first_step, int32_t n_steps, "
            "void* stream);") in h
    assert ("int  mugd_sample_unipc_stop(mugd_plan* eval_plan, const mugd_unipc_stop* e, int32_t first_step, int32_t n_steps, "
            "void* stream);") in h
    assert C.sizeof(L_.UnipcEx) == C.sizeof(L_.Unipc) + 4 * 8 + 2 * 4
    assert C.sizeof(L_.UnipcStop) == C.sizeof(L_.Unipc) + 8 + 2 * 4


N, S_ = 2 * 16 * 8, 6


def _unipc():
    """a well-formed descriptor over fake (never dereferenced) device addresses"""
    u = L_.Unipc()
    d = u.dpm
    d.x, d.x_dup, d.eps, d.pred_x0, d.ring, d.coef, d.step = 0x1000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000, 0x70000
    d.n, d.S, d.cfg, d.scale = N, S_, 1, 5.0
    u.xc, u.corr = 0x80000, 0x90000
    return u


STAGE = L_.Stage()


def _ex(kind="start"):
    e = L_.UnipcEx()
    e.unipc = _unipc()
    if kind == "start":
        e.start, e.order_coef, e.order_corr, e.B = 0xa0000, 0xb0000, 0xc0000, 2
    else:
        s = STAGE
        s.x, s.x_dup, s.x0, s.mask, s.q_noise, s.q_coef = e.unipc.dpm.x, e.unipc.dpm.x_dup, 0xd0000, 0xe0000, 0xf0000, _QCOEF.ctypes.data
        s.noise, s.noise_rows, s.B, s.C, s.L = None, None, 2, 16, 8
        e.stage = C.addressof(s)
    return e


_QCOEF = np.ones((8, 2), np.float32)


def _stop():
    e = L_.UnipcStop()
    e.unipc, e.stop, e.B = _unipc(), 0xa0000, 2
    return e


def _malformed_ex():
    out = []
    e = _ex(); e.unipc.xc = None; out.append((e, "xc and corr must be given"))
    e = _ex(); e.unipc.xc = e.unipc.dpm.x + 4; out.append((e, "xc overlaps x, x_dup or the ring"))
    e = _ex(); e.unipc.dpm.S = 0; out.append((e, "S=0 outside"))
    e = _ex(); e.stage = _ex("stage").stage; out.append((e, "cannot be combined"))
    e = _ex(); e.order_corr = None; out.append((e, "start, order_coef and order_corr go together"))
    e = _ex(); e.start = None; out.append((e, "start, order_coef and order_corr go together"))
    e = _ex(); e.B = 3; out.append((e, "B=3 does not divide n=256"))
    e = _ex(); e.reserved_ = 1; out.append((e, "reserved_=1 must be 0"))
    e = _ex("stage"); STAGE.x0 = STAGE.mask = STAGE.q_noise = STAGE.q_coef = None
    out.append((e, "the stage has no x0 (a UniPC stage is the inpainting blend)"))
    return out


def _malformed_stop():
    out = []
    e = _stop(); e.unipc.corr = None; out.append((e, "xc and corr must be given"))
    e = _stop(); e.unipc.dpm.cfg = 0; out.append((e, "x_dup must be given exactly when cfg = 1"))
    e = _stop(); e.stop = None; out.append((e, "stop must be given"))
    e = _stop(); e.B = 0; out.append((e, "B=0 does not divide"))
    e = _stop(); e.reserved_ = 2; out.append((e, "reserved_=2 must be 0"))
    return out


@pytest.mark.parametrize("case", range(9))
@pytest.mark.parametrize("entry", ["update", "loop"])
def test_unipc_ex_entry_points_check_their_arguments_without_a_device(case, entry):
    e, msg = _malformed_ex()[case]
    lib = L_.load()
    rc_ = lib.mugd_unipc_ex_update(C.byref(e), None) if entry == "update" else lib.mugd_sample_unipc_ex(None, C.byref(e), 0, 2, None)
    assert rc_ == 1 and msg in lib.mugd_last_error().decode()


def test_unipc_ex_stage_checks():
    lib = L_.load()
    for change, msg in ((dict(noise=0x1), "stages step noise; UniPC draws none"), (dict(x=0x2000000), "blends other rows"),
                        (dict(L=9), "the update's n=256")):
        e = _ex("stage")
        for k, v in change.items():
            setattr(STAGE, k, v)
        if "noise" in change:
            STAGE.noise_rows = 0x3000000
        assert lib.mugd_sample_unipc_ex(None, C.byref(e), 0, 2, None) == 1
        assert msg in lib.mugd_last_error().decode(), lib.mugd_last_error()
    e = _ex("stage")
    assert lib.mugd_sample_unipc_ex(None, C.byref(e), 0, 2, None) == 1
    assert "must be captured" in lib.mugd_last_error().decode()


@pytest.mark.parametrize("case", range(5))
@pytest.mark.parametrize("entry", ["update", "loop"])
def test_unipc_stop_entry_points_check_their_arguments_without_a_device(case, entry):
    e, msg = _malformed_stop()[case]
    lib = L_.load()
    rc_ = lib.mugd_unipc_stop_update(C.byref(e), None) if entry == "update" else lib.mugd_sample_unipc_stop(None, C.byref(e), 0, 2, None)
    assert rc_ == 1 and msg in lib.mugd_last_error().decode()


def test_loops_check_the_step_range_before_the_plan():
    lib = L_.load()
    for fn, e in ((lib.mugd_sample_unipc_ex, _ex()), (lib.mugd_sample_unipc_stop, _stop())):
        for first, n in ((0, S_ + 1), (S_, 1), (-1, 1), (2, -1)):
            assert fn(None, C.byref(e), first, n, None) == 1
            assert "outside the S=6 steps" in lib.mugd_last_error().decode()
        assert fn(None, C.byref(e), 1, S_ - 1, None) == 1 and "must be captured" in lib.mugd_last_error().decode()
        assert fn(None, None, 0, 1, None) == 1 and "null descriptor" in lib.mugd_last_error().decode()
    assert lib.mugd_unipc_ex_update(None, None) == 1 and "null argument" in lib.mugd_last_error().decode()
    assert lib.mugd_unipc_stop_update(None, None) == 1 and "null argument" in lib.mugd_last_error().decode()


# ---- the sampler refuses before any GPU work ---------------------------------------------------------------------------------------
def _cpu_sampler(L=96):
    s = UniPCSampler.__new__(UniPCSampler)
    sch = register_schedule()
    s.model = types.SimpleNamespace(z_channels=16, z_length=L, num_timesteps=1000, alphas_cumprod=sch["alphas_cumprod"],
                                    cfg=ModelConfig())
    s.ddpm_num_timesteps, s.device = 1000, torch.device("cpu")
    return s


SCHED = U.multistep_schedule(ACP, 10, 2)
X0_T = torch.zeros(2, 16, 96)


def _guided(**kw):
    inp = synth.synthetic_inputs(2, 96)
    out = dict(c=inp["c"], w=inp["w"], unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"])
    out.update(kw)
    return out


BAD_INPAINT = [
    (dict(mask=None), ValueError, "needs the mask and x0 as tensors"),
    (dict(x0=torch.zeros(2, 16, 64)), ValueError, "inpainting needs x0 of shape"),
    (dict(mask=torch.ones(2, 3, 96)), ValueError, "does not broadcast"),
    (dict(S=1, order=2), ValueError, "order 2 needs at least 2 steps"),
    (dict(variant="bh3"), ValueError, "variant="),
    (dict(c=None), TypeError, "needs the conditioning"),
    (dict(unconditional_guidance_scale=float("inf")), ValueError, "finite number"),
    (dict(log_every_t=0), ValueError, "log_every_t"),
]


@pytest.mark.parametrize("kw,exc,msg", BAD_INPAINT, ids=[f"bad{i}" for i in range(len(BAD_INPAINT))])
def test_inpaint_refuses_before_any_gpu_work(kw, exc, msg):
    args = _guided(S=10, batch_size=2, shape=(16, 96), verbose=False, mask=torch.ones(2, 1, 96), x0=X0_T)
    args.update(kw)
    with pytest.raises(exc, match=msg):
        _cpu_sampler().inpaint(**args)


def test_sample_still_refuses_inpainting():
    with pytest.raises(ValueError, match="mask="):
        _cpu_sampler().sample(**_guided(S=10, batch_size=2, shape=(16, 96), verbose=False, mask=torch.ones(2, 1, 96), x0=X0_T))


@pytest.mark.parametrize("kw,msg", [(dict(sched=None), "sched must be a UniPCSchedule"),
                                    (dict(sched=U.inversion_schedule(SCHED)), "sched must be a UniPCSchedule"),
                                    (dict(t_enc=11), r"every start must lie in \[0, 10\]"),
                                    (dict(x0=np.zeros((2, 16, 96), np.float32)), "x0 must be"),
                                    (dict(noise=torch.zeros(2, 16, 95)), "noise must be")])
def test_stochastic_encode_refuses_before_any_gpu_work(kw, msg):
    args = dict(x0=X0_T, t_enc=3, sched=SCHED)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        _cpu_sampler().stochastic_encode(**args)


@pytest.mark.parametrize("kw,msg", [(dict(sched=D.multistep_schedule(ACP, 10, 2)), "sched must be a UniPCSchedule"),
                                    (dict(x_latent=torch.zeros(16, 96)), "x_latent must be"),
                                    (dict(t_start=[1, 2, 3]), "t_start has 3 entries"),
                                    (dict(t_start=-1), r"every start must lie in \[0, 10\]"),
                                    (dict(c=None), "needs the conditioning"),
                                    (dict(unconditional_guidance_scale=float("nan")), "finite number")])
def test_decode_refuses_before_any_gpu_work(kw, msg):
    args = _guided(x_latent=X0_T, t_start=[3, 10], sched=SCHED)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        _cpu_sampler().decode(**args)


@pytest.mark.parametrize("kw,exc,msg", [(dict(sched=None), ValueError, "sched must be a UniPCSchedule"),
                                        (dict(x0=torch.zeros(2, 16, 64)), ValueError, "x0 must be a float32"),
                                        (dict(t_enc=[1.0, 2.0]), ValueError, "must be integers"),
                                        (dict(w=None), ValueError, "needs the conditioning c and the audio features w"),
                                        (dict(mask=torch.ones(2, 1, 96)), ValueError, "has no mask"),
                                        (dict(eta=0.5), ValueError, "eta=0.5"),
                                        (dict(x_T=X0_T), TypeError, r"UniPCSampler\.invert got unexpected arguments")])
def test_invert_refuses_before_any_gpu_work(kw, exc, msg):
    args = _guided(x0=X0_T, t_enc=[3, 10], sched=SCHED, verbose=False)
    args.update(kw)
    with pytest.raises(exc, match=msg):
        _cpu_sampler().invert(**args)


def test_zero_steps_return_the_latent_without_gpu_work():
    s = _cpu_sampler()
    assert s.decode(**_guided(x_latent=X0_T, t_start=0, sched=SCHED)) is X0_T
    assert s.invert(**_guided(x0=X0_T, t_enc=[0, 0], sched=SCHED, verbose=False)) is X0_T
    assert s.last_intermediates["x_inter"] == [X0_T]


def test_valid_requests_reach_the_engine():
    s = _cpu_sampler()
    for call in (lambda: s.decode(**_guided(x_latent=X0_T, t_start=[3, 10], sched=SCHED)),
                 lambda: s.invert(**_guided(x0=X0_T, t_enc=[3, 10], sched=SCHED, verbose=False)),
                 lambda: s.inpaint(**_guided(S=10, batch_size=2, shape=(16, 96), verbose=False, mask=torch.ones(2, 1, 96), x0=X0_T))):
        with pytest.raises(AttributeError, match="engine"):
            call()
