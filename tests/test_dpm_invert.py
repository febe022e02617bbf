"""DPM-Solver++ and DDIM inversion, CPU side: the inversion rows against the solver's D-form on the reversed grid in float64, the
float32 conditioning of every step, the analytic Gaussian model (inversion against the exact probability-flow map, the round trip
sample(invert(x0)) against x0, on the DPM-Solver grids and on DDIM's), the C entry points' argument checks and the samplers' refusals
before any GPU work."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from mug_diffusion_b200 import dpm_solver as D
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.sampler import DDIMSampler, ddim_timesteps_uniform, register_schedule
from test_dpm_solver import ACP, MU, NS, SD, _cpu_sampler, _request, d_form_step, gaussian_run

GRIDS = ("time_uniform", "logSNR", "time_quadratic")


# ---- the inversion rows ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [5, 20])
@pytest.mark.parametrize("skip", GRIDS)
@pytest.mark.parametrize("solver_type", D.SOLVER_TYPES)
@pytest.mark.parametrize("order", D.ORDERS)
def test_inversion_rows_equal_the_d_form_on_the_reversed_grid(order, solver_type, skip, S):
    sched = D.multistep_schedule(ACP, S, order, skip, solver_type, True)
    inv = D.inversion_schedule(sched)
    u = inv.t
    assert np.array_equal(u, sched.t[::-1]) and u[0] == sched.t[-1] and u[-1] == sched.t[0]
    assert inv.orders.tolist() == [min(j + 1, order) for j in range(S)]               # no lower_order_final
    assert np.array_equal(inv.model_times, D.model_time(NS, u[:-1])) and inv.model_times.dtype == np.float32
    lam, alpha, sigma = NS.marginal_lambda(u), NS.marginal_alpha(u), NS.marginal_std(u)
    assert np.all(np.diff(lam) < 0)                                                    # h < 0 on every step
    rng = np.random.default_rng(S * 10 + order)
    for j in range(S):
        row, k = inv.rows[j], int(inv.orders[j])
        assert row[D.ROW_ORDER] == k and row[D.ROW_ALPHA] == alpha[j] and row[D.ROW_SIGMA] == sigma[j]
        x, ms = rng.standard_normal(64), [rng.standard_normal(64) for _ in range(3)]
        want = d_form_step(j, k, lam, alpha, sigma, x, ms, solver_type)
        A, c0, c1, c2 = row[D.ROW_A:D.ROW_C2 + 1]
        if k == 1:
            # DDIM's form, with e = (x - alpha_j m0) / sigma_j; the expanded columns A / c0 are kept as well
            assert row[D.ROW_FORM] == D.FORM_EPS and c1 == alpha[j + 1] and c2 == sigma[j + 1]
            got = c1 * ms[0] + c2 * (x - alpha[j] * ms[0]) / sigma[j]
            assert np.abs(got - want).max() < 1e-12 * max(1., np.abs(want).max()), j
            got = A * x + c0 * ms[0]
        else:
            assert row[D.ROW_FORM] == D.FORM_EXPANDED and (k >= 3 or c2 == 0)
            got = A * x + c0 * ms[0] + c1 * ms[1] + c2 * ms[2]
        assert np.abs(got - want).max() < 1e-12 * max(1., np.abs(want).max()), j
    assert inv.order_rows is None


def test_inversion_schedule_needs_a_multistep_schedule():
    sched = D.multistep_schedule(ACP, 6, 2)
    with pytest.raises(ValueError, match="sched must be a DPMSchedule from multistep_schedule"):
        D.inversion_schedule(D.DPMSchedule(sched.t, sched.model_times, sched.rows, sched.orders))
    with pytest.raises(ValueError, match="decreasing"):                               # multistep_schedule still refuses increasing grids
        D.multistep_schedule(ACP, 6, 2, t_grid=sched.t[::-1])


def ddim_schedule(S):
    ts = ddim_timesteps_uniform(S, 1000)
    return D.multistep_schedule(ACP, len(ts), 1, t_grid=D.ddim_grid(NS, ts))


def test_inversion_on_the_ddim_grid_evaluates_at_ddim_timesteps():
    """step j runs at timestep 0 (j = 0) and ddim_timesteps[j - 1] after that, so after s steps a chart is at ddim_timesteps[s - 1]"""
    ts = ddim_timesteps_uniform(10, 1000)
    inv = D.inversion_schedule(ddim_schedule(10))
    assert np.array_equal(inv.model_times, np.append(0, ts[:-1]).astype(np.float32))
    assert np.array_equal(D.model_time(NS, inv.t[1:]), ts.astype(np.float32))


# ---- float32 conditioning ------------------------------------------------------------------------------------------------------------
def f32_step_error(row, rng, n=1 << 14):
    """max |kernel arithmetic in float32 - the same row in float64| / max |x| over random x, e, m1, m2 of one step"""
    r32 = row.astype(np.float32)
    x, e, m1, m2 = (rng.standard_normal(n).astype(np.float32) for _ in range(4))
    k = int(row[D.ROW_ORDER])
    m0 = (x - r32[1] * e) / r32[0]
    x64, e64 = x.astype(np.float64), e.astype(np.float64)
    m64 = (x64 - row[1] * e64) / row[0]
    if row[D.ROW_FORM] != D.FORM_EXPANDED:
        got, want = r32[4] * m0 + r32[5] * e, row[4] * m64 + row[5] * e64
    else:
        got, want = r32[2] * x + r32[3] * m0, row[2] * x64 + row[3] * m64
        if k >= 2:
            got, want = got + r32[4] * m1, want + row[4] * m1
        if k >= 3:
            got, want = got + r32[5] * m2, want + row[5] * m2
    return float(np.abs(got - want).max() / max(np.abs(x64).max(), np.abs(want).max()))


@pytest.mark.parametrize("S", [10, 20, 50])
@pytest.mark.parametrize("grid,order", [("time_uniform", 1), ("time_uniform", 2), ("time_uniform", 3), ("logSNR", 1), ("logSNR", 2),
                                        ("logSNR", 3), ("ddim", 1)])
def test_every_inversion_step_is_well_conditioned_in_float32(grid, order, S):
    """A = sigma_j+1 / sigma_j reaches 17 on the first step away from t = 1/N (time_uniform, S = 10), where A x + c0 m0 loses
    1.9e-6 of max |x|; the order-1 rows take DDIM's form, which keeps every step within 1e-6"""
    sched = ddim_schedule(S) if grid == "ddim" else D.multistep_schedule(ACP, S, order, grid)
    inv = D.inversion_schedule(sched)
    rng = np.random.default_rng(S)
    worst = max(f32_step_error(inv.rows[j], rng) for j in range(inv.S))
    assert worst < 1e-6, worst


def test_the_expanded_form_of_the_first_step_is_the_hazard():
    """the same first step in the expanded form loses more than 1e-6 of max |x| (the figure DESIGN records)"""
    row = D.inversion_schedule(D.multistep_schedule(ACP, 10, 2)).rows[0].copy()
    assert row[D.ROW_A] > 15
    row[D.ROW_C1] = row[D.ROW_C2] = row[D.ROW_FORM] = 0.
    assert f32_step_error(row, np.random.default_rng(0)) > 1e-6


# ---- the analytic Gaussian model ------------------------------------------------------------------------------------------------------
def gaussian_map(x, t_from, t_to):
    """the probability-flow ODE of N(MU, SD^2) data from t_from to t_to: it keeps the z-score of N(alpha MU, alpha^2 SD^2 + sigma^2)"""
    a0, s0, a1, s1 = NS.marginal_alpha(t_from), NS.marginal_std(t_from), NS.marginal_alpha(t_to), NS.marginal_std(t_to)
    return a1 * MU + (x - a0 * MU) / np.sqrt(a0 ** 2 * SD ** 2 + s0 ** 2) * np.sqrt(a1 ** 2 * SD ** 2 + s1 ** 2)


def gaussian_invert(inv, x0, steps=None):
    """the inversion rows on the exact eps, in float64, each row in its own form"""
    x, hist = x0.copy(), []
    for j in range(inv.S if steps is None else steps):
        a, s, A, c0, c1, c2, k, form = inv.rows[j]
        e = s * (x - a * MU) / (a * a * SD * SD + s * s)
        m0 = (x - s * e) / a
        if form != D.FORM_EXPANDED:
            xn = c1 * m0 + c2 * e
        else:
            xn = A * x + c0 * m0 + (c1 * hist[-1] if k >= 2 else 0.) + (c2 * hist[-2] if k >= 3 else 0.)
        x, hist = xn, (hist + [m0])[-2:]
    return x


X0 = gaussian_map(np.random.default_rng(3).standard_normal(64), 1., 1e-3)      # a sample of the data marginal at t = 1/N
STEPS = [20, 40, 80, 160]


def slope(steps, errs):
    return float(-np.polyfit(np.log(steps), np.log(errs), 1)[0])


# slopes over S in STEPS, measured: inversion 0.97 / 1.42 (time_uniform, orders 1 / 2) and 0.98 / 1.98 (logSNR); round trip 0.94 / 2.07
# and 0.96 / 2.74.  The first inversion step leaves t = 1/N at order 1 (there is no history yet); on the time-uniform grid its lambda
# step is about -0.5 log(1 + N/S), which shrinks only logarithmically, so it holds order 2 at 1.42 (1.56 over S = 160 .. 1000).  On
# the logSNR grid the errors of the two directions partly cancel at small S; over S = 160 .. 1000 the round trip's slope is 2.03.
@pytest.mark.parametrize("skip,order,lo,hi", [("time_uniform", 1, 0.8, 1.2), ("logSNR", 1, 0.8, 1.2), ("time_uniform", 2, 1.3, 1.7),
                                              ("logSNR", 2, 1.7, 2.3)])
def test_inversion_global_error_slope(skip, order, lo, hi):
    errs = []
    for S in STEPS:
        inv = D.inversion_schedule(D.multistep_schedule(ACP, S, order, skip))
        errs.append(float(np.abs(gaussian_invert(inv, X0) - gaussian_map(X0, 1e-3, 1.)).max()))
    assert all(a > b for a, b in zip(errs, errs[1:])), errs
    assert lo <= slope(STEPS, errs) <= hi, errs


@pytest.mark.parametrize("skip,order,steps,lo,hi", [("time_uniform", 1, STEPS, 0.8, 1.2), ("logSNR", 1, STEPS, 0.8, 1.2),
                                                    ("time_uniform", 2, STEPS, 1.7, 2.3), ("logSNR", 2, STEPS, 2.3, 3.0),
                                                    ("logSNR", 2, [160, 320, 640, 1000], 1.7, 2.3)])
def test_round_trip_global_error_slope(skip, order, steps, lo, hi):
    """sample(invert(x0)) with the same schedule returns x0, its error falling at least like the solver's order"""
    errs = []
    for S in steps:
        sched = D.multistep_schedule(ACP, S, order, skip)
        errs.append(float(np.abs(gaussian_run(sched, gaussian_invert(D.inversion_schedule(sched), X0)) - X0).max()))
    assert all(a > b for a, b in zip(errs, errs[1:])), errs
    assert lo <= slope(steps, errs) <= hi, errs


@pytest.mark.parametrize("order,bound", [(1, 0.06), (2, 0.01)])
def test_partial_inversion_pairs_with_the_remix_of_the_same_steps(order, bound):
    """s inversion steps end at t_S-s, where a remix over the last s steps starts: at S = 80 the pair returns x0 within the full
    round trip's error (measured 5.7e-2 at order 1, 9.6e-3 at order 2 for s = 1, where both steps are order 1)"""
    from test_dpm_remix import gaussian_remix
    S = 80
    sched = D.multistep_schedule(ACP, S, order)
    inv = D.inversion_schedule(sched)
    for s in (1, 2, 20, 40, 79, 80):
        assert np.abs(gaussian_remix(sched, gaussian_invert(inv, X0, s), s) - X0).max() < bound, s


def ddim_step(x, a, ap):
    """DDIM's eta = 0 update from alphas_cumprod a to ap on the exact eps"""
    e = np.sqrt(1 - a) * (x - np.sqrt(a) * MU) / (a * SD * SD + (1 - a))
    return np.sqrt(ap) * (x - np.sqrt(1 - a) * e) / np.sqrt(a) + np.sqrt(1 - ap) * e


def test_round_trip_on_the_ddim_grid_converges_at_order_one():
    """order-1 inversion on DDIM's grid, then DDIM's own update over the same timesteps"""
    n_steps, errs = [], []
    for S in STEPS:
        ts = ddim_timesteps_uniform(S, 1000)
        inv = D.inversion_schedule(ddim_schedule(S))
        a_seq = np.append(ACP[np.flip(ts)], ACP[0])
        x = gaussian_invert(inv, X0)
        for i in range(len(ts)):
            x = ddim_step(x, a_seq[i], a_seq[i + 1])
        n_steps.append(len(ts))
        errs.append(float(np.abs(x - X0).max()))
    assert all(a > b for a, b in zip(errs, errs[1:])), errs
    assert 0.8 <= slope(n_steps, errs) <= 1.2, errs


# ---- C ABI -------------------------------------------------------------------------------------------------------------------------
def test_library_exports_the_dpm_stop_entry_points_at_abi_13():
    lib = L_.load()
    assert lib.mugd_abi_version() == L_.ABI_VERSION == 13
    for sym in ("mugd_sample_dpm_stop", "mugd_dpm_stop_update"):
        assert sym in L_.EXPORTED_SYMBOLS and hasattr(lib, sym)
    with open(os.path.join(os.path.dirname(L_.HERE), "include", "mugd.h")) as f:
        h = f.read()
    assert ("int  mugd_sample_dpm_stop(mugd_plan* eval_plan, const mugd_dpm_stop* e, int32_t first_step, int32_t n_steps, "
            "void* stream);") in h
    assert "int  mugd_dpm_stop_update(const mugd_dpm_stop* e, void* stream);" in h
    assert C.sizeof(L_.DpmStop) == C.sizeof(L_.Dpm) + 8 + 2 * 4


N, S_ = 2 * 16 * 8, 6


def _stop():
    """a well-formed descriptor over fake (never dereferenced) device addresses"""
    d = L_.Dpm()
    d.x, d.x_dup, d.eps, d.pred_x0, d.ring, d.coef, d.step = 0x1000, 0x2000, 0x3000, 0x4000, 0x5000, 0x6000, 0x7000
    d.n, d.S, d.cfg, d.scale = N, S_, 1, 5.0
    e = L_.DpmStop()
    e.dpm, e.stop, e.B = d, 0x8000, 2
    return e


def _malformed_stop():
    out = []
    e = _stop(); e.dpm.coef = None; out.append((e, "must be given"))
    e = _stop(); e.dpm.S = 0; out.append((e, "S=0 outside"))
    e = _stop(); e.dpm.cfg = 0; out.append((e, "x_dup must be given exactly when cfg = 1"))
    e = _stop(); e.dpm.scale = float("nan"); out.append((e, "scale is not finite"))
    e = _stop(); e.stop = None; out.append((e, "stop must be given"))
    e = _stop(); e.B = 3; out.append((e, "B=3 does not divide n=256"))
    e = _stop(); e.B = 0; out.append((e, "B=0 does not divide"))
    e = _stop(); e.reserved_ = 1; out.append((e, "reserved_=1 must be 0"))
    return out


@pytest.mark.parametrize("case", range(len(_malformed_stop())))
@pytest.mark.parametrize("entry", ["update", "loop"])
def test_dpm_stop_entry_points_check_their_arguments_without_a_device(case, entry):
    e, msg = _malformed_stop()[case]
    lib = L_.load()
    rc_ = lib.mugd_dpm_stop_update(C.byref(e), None) if entry == "update" else lib.mugd_sample_dpm_stop(None, C.byref(e), 0, 2, None)
    assert rc_ == 1
    assert msg in lib.mugd_last_error().decode()


def test_sample_dpm_stop_checks_the_step_range_before_the_plan():
    lib = L_.load()
    e = _stop()
    for first, n in ((0, S_ + 1), (S_, 1), (-1, 1), (2, -1)):
        assert lib.mugd_sample_dpm_stop(None, C.byref(e), first, n, None) == 1
        assert "outside the S=6 steps" in lib.mugd_last_error().decode()
    assert lib.mugd_sample_dpm_stop(None, C.byref(e), 1, S_ - 1, None) == 1
    assert "must be captured" in lib.mugd_last_error().decode()
    assert lib.mugd_sample_dpm_stop(None, None, 0, 1, None) == 1 and "null descriptor" in lib.mugd_last_error().decode()
    assert lib.mugd_dpm_stop_update(None, None) == 1 and "null argument" in lib.mugd_last_error().decode()


# ---- the samplers refuse before any GPU work -----------------------------------------------------------------------------------------
SCHED = D.multistep_schedule(ACP, 10, 2)
X0_T = torch.zeros(2, 16, 96)


def _ddim_sampler(eta=0.):
    s = DDIMSampler.__new__(DDIMSampler)
    s.model = types.SimpleNamespace(z_channels=16, z_length=96, num_timesteps=1000, alphas_cumprod=register_schedule()["alphas_cumprod"],
                                    cfg=ModelConfig())
    s.ddpm_num_timesteps, s.device = 1000, torch.device("cpu")
    s.make_schedule(10, ddim_eta=eta, verbose=False)
    return s


def _invert_args(**kw):
    r = _request()
    args = dict(x0=X0_T, c=r["c"], w=r["w"], t_enc=[3, 10], unconditional_guidance_scale=5.0,
                unconditional_conditioning=r["unconditional_conditioning"], verbose=False)
    args.update(kw)
    return args


BAD_INVERT = [
    (dict(x0=torch.zeros(2, 16, 96, dtype=torch.float64)), ValueError, r"x0 must be a float32 \[B, 16, 96\] tensor"),
    (dict(x0=torch.zeros(16, 96)), ValueError, "x0 must be a float32"),
    (dict(x0=torch.zeros(2, 16, 64)), ValueError, "x0 must be a float32"),
    (dict(x0=torch.zeros(2, 8, 96)), ValueError, "x0 must be a float32"),
    (dict(x0=torch.zeros(0, 16, 96)), ValueError, "x0 must be a float32"),
    (dict(x0=np.zeros((2, 16, 96), np.float32)), ValueError, "x0 must be a float32"),
    (dict(t_enc=11), ValueError, r"every start must lie in \[0, 10\] \(S = 10\)"),
    (dict(t_enc=-1), ValueError, r"every start must lie in \[0, 10\]"),
    (dict(t_enc=[1, 2, 3]), ValueError, "t_enc has 3 entries for 2 charts"),
    (dict(t_enc=[1.0, 2.0]), ValueError, "must be integers"),
    (dict(t_enc=None), ValueError, "must be an integer or one integer per chart"),
    (dict(c=torch.zeros(3, 128, 21)), ValueError, "c must be"),
    (dict(c=None), ValueError, "needs the conditioning c and the audio features w"),
    (dict(w=None), ValueError, "needs the conditioning c and the audio features w"),
    (dict(unconditional_guidance_scale=float("inf")), ValueError, "must be a finite number"),
    (dict(unconditional_conditioning=torch.zeros(1, 128, 21)), ValueError, "unconditional_conditioning must be"),
    (dict(log_every_t=0), ValueError, "log_every_t"),
    (dict(mask=torch.ones(2, 1, 96)), ValueError, "has no mask"),
    (dict(eta=0.5), ValueError, "eta=0.5"),
    (dict(temperature=0.9), ValueError, "temperature=0.9"),
    (dict(noise_dropout=0.1), ValueError, "noise_dropout=0.1"),
    (dict(x_T=torch.zeros(2, 16, 96)), TypeError, r"\.invert got unexpected arguments \['x_T'\]"),
]


@pytest.mark.parametrize("kw,exc,msg", BAD_INVERT, ids=[f"bad{i}" for i in range(len(BAD_INVERT))])
@pytest.mark.parametrize("which", ["dpm", "ddim"])
def test_invert_refuses_before_any_gpu_work(which, kw, exc, msg):
    with pytest.raises(exc, match=msg):
        if which == "dpm":
            _cpu_sampler().invert(sched=SCHED, **_invert_args(**kw))
        else:
            _ddim_sampler().invert(**_invert_args(**kw))


def test_invert_refuses_malformed_schedules():
    with pytest.raises(ValueError, match="sched must be a DPMSchedule"):
        _cpu_sampler().invert(sched=None, **_invert_args())
    with pytest.raises(ValueError, match="sched must be a DPMSchedule"):
        _cpu_sampler().invert(sched=D.DPMSchedule(SCHED.t, SCHED.model_times, SCHED.rows, SCHED.orders), **_invert_args())
    with pytest.raises(ValueError, match="eta = 0"):
        _ddim_sampler(eta=0.5).invert(**_invert_args())
    s = _ddim_sampler()
    s.ddim_timesteps = None
    with pytest.raises(ValueError, match="call make_schedule"):
        s.invert(**_invert_args())


def test_invert_of_zero_steps_returns_x0_without_gpu_work():
    for s, kw in ((_cpu_sampler(), dict(sched=SCHED)), (_ddim_sampler(), {})):
        out = s.invert(**_invert_args(t_enc=0, **kw))
        assert out is X0_T
        assert s.last_intermediates["x_inter"] == [X0_T]
        assert s.invert(**_invert_args(t_enc=[0, 0], unconditional_guidance_scale=1.0, **kw)) is X0_T


def test_a_valid_inversion_reaches_the_engine():
    for s, kw in ((_cpu_sampler(), dict(sched=SCHED)), (_ddim_sampler(), {})):
        with pytest.raises(AttributeError, match="engine"):
            s.invert(**_invert_args(**kw))
