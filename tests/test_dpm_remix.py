"""DPM-Solver++ inpainting and remix, CPU side: the per-order coefficient rows against the solver's D-form in float64, the per-chart
order rule, the per-chart warm-up's accuracy on the analytic Gaussian model, the oracle's order-1 remix on DDIM's grid against the
UNMODIFIED reference's DDIM remix goldens, the C entry points' argument checks, the sampler's refusals before any GPU work, and the
exact C-call and random-number sequence of an inpainting request on a recording stand-in for the engine."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

import golden_cases as gc
import remix_cases as rc
from dpm_remix_oracle import decode as oracle_decode
from mug_diffusion_b200 import dpm_solver as D
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import sampler as sampler_mod
from mug_diffusion_b200 import synth
from mug_diffusion_b200.sampler import ddim_timesteps_uniform
from oracle import mug_oracle as orc
from test_dpm_solver import ACP, MU, NS, SD, X_T, _cpu_sampler, _request, d_form_step, gaussian_exact, rel_err
from test_request_loop import PLAN_LAUNCHES, SHAPE, SMALL_CAP, STEP_BYTES, _Bar, _logged, _Recorder, _stretches


# ---- per-order rows ----------------------------------------------------------------------------------------------------------------
ROW_CASES = [(o, st, sk, S) for o in D.ORDERS for st in D.SOLVER_TYPES for sk in D.SKIP_TYPES for S in (5, 14, 15, 20)]


@pytest.mark.parametrize("order,solver_type,skip,S", ROW_CASES)
def test_order_rows_equal_the_d_form(order, solver_type, skip, S):
    sched = D.multistep_schedule(ACP, S, order, skip, solver_type, True)
    t = sched.t
    lam, alpha, sigma = NS.marginal_lambda(t), NS.marginal_alpha(t), NS.marginal_std(t)
    R = sched.order_rows
    assert R.shape == (S, 3, 8)
    rng = np.random.default_rng(S * 10 + order)
    for i in range(S):
        for k in (1, 2, 3):
            if k > i + 1:
                assert np.isnan(R[i, k - 1]).all(), (i, k)                  # no chart can take this update: a read shows up as NaN
                continue
            row = R[i, k - 1]
            assert row[D.ROW_ORDER] == k and row[7] == 0 and row[D.ROW_ALPHA] == alpha[i] and row[D.ROW_SIGMA] == sigma[i]
            A, c0, c1, c2 = row[D.ROW_A:D.ROW_C2 + 1]
            assert (k >= 2 or c1 == 0) and (k >= 3 or c2 == 0)
            x, ms = rng.standard_normal(64), [rng.standard_normal(64) for _ in range(3)]
            want = d_form_step(i, k, lam, alpha, sigma, x, ms, solver_type)
            got = A * x + c0 * ms[0] + c1 * ms[1] + c2 * ms[2]
            assert np.abs(got - want).max() < 1e-12 * max(1., np.abs(want).max()), (i, k)
    f32 = sched.order_rows_f32()
    rows = sched.rows_f32()
    for i in range(S):
        assert np.array_equal(f32[i, int(sched.orders[i]) - 1], rows[i]), i          # the request's own row, bit for bit


def test_chart_orders():
    sched = D.multistep_schedule(ACP, 8, 3, lower_order_final=True)               # S < 15: the final steps drop to order 2, 1
    assert sched.orders.tolist() == [1, 2, 3, 3, 3, 3, 2, 1]
    got = D.chart_orders(sched, [8, 6, 3, 1, 0, 2])
    assert got.tolist() == [[1, 2, 3, 3, 3, 3, 2, 1],
                            [0, 0, 1, 2, 3, 3, 2, 1],
                            [0, 0, 0, 0, 0, 1, 2, 1],
                            [0, 0, 0, 0, 0, 0, 0, 1],
                            [0] * 8,
                            [0, 0, 0, 0, 0, 0, 1, 1]]
    sched = D.multistep_schedule(ACP, 16, 2, lower_order_final=True)              # S >= 15: no lower-order final steps
    assert D.chart_orders(sched, [16, 5]).tolist() == [[1] + [2] * 15, [0] * 11 + [1, 2, 2, 2, 2]]
    sched = D.multistep_schedule(ACP, 6, 3, lower_order_final=False)
    assert D.chart_orders(sched, [6, 4, 2]).tolist() == [[1, 2, 3, 3, 3, 3], [0, 0, 1, 2, 3, 3], [0, 0, 0, 0, 1, 2]]


def test_encode_tables_index_the_remaining_steps():
    sched = D.multistep_schedule(ACP, 7, 2, "logSNR")
    a, s = sched.encode_tables_f32()
    assert a.dtype == s.dtype == np.float32 and a.shape == s.shape == (8,)
    assert a[0] == 1 and s[0] == 0
    for k in range(1, 8):
        assert a[k] == np.float32(NS.marginal_alpha(sched.t[7 - k])) and s[k] == np.float32(NS.marginal_std(sched.t[7 - k]))
    assert np.array_equal(sched.q_coef_f32(), sched.rows_f32()[:, :2])


# ---- the per-chart warm-up on the analytic Gaussian model --------------------------------------------------------------------------
def gaussian_remix(sched, x_start, s):
    """the last s steps of ``sched`` from x_start at t_S-s on the exact eps of N(MU, SD^2) data, each step with its per-chart order"""
    S = sched.S
    k_of = D.chart_orders(sched, [s])[0]
    x, hist = x_start.copy(), []
    for i in range(S - s, S):
        k = int(k_of[i])
        a, sg, A, c0, c1, c2, kk, _ = sched.order_rows[i, k - 1]
        assert kk == k
        e = sg * (x - a * MU) / (a * a * SD * SD + sg * sg)
        m0 = (x - sg * e) / a
        xn = A * x + c0 * m0
        if k >= 2:
            xn = xn + c1 * hist[-1]
        if k >= 3:
            xn = xn + c2 * hist[-2]
        x, hist = xn, (hist + [m0])[-2:]
    return x


STEPS = [40, 80, 160, 320]                      # at S = 20 a half-strength 2M remix on the logSNR grid is still pre-asymptotic (1.63)


@pytest.mark.parametrize("strength", [2, 3])
@pytest.mark.parametrize("skip", ["time_uniform", "logSNR"])
@pytest.mark.parametrize("order,lo,hi", [(1, 0.8, 1.2), (2, 1.7, 2.3)])
def test_remix_global_error_slope(order, lo, hi, skip, strength):
    """remixes over the last s = strength / 4 * S steps started from the exact marginal at t_S-s: the per-chart warm-up (a first
    step of order 1) keeps the solver's order"""
    errs = []
    for S in STEPS:
        sched = D.multistep_schedule(ACP, S, order, skip)
        s = S * strength // 4
        x_start = gaussian_exact(X_T, sched.t[S - s])
        errs.append(float(np.abs(gaussian_remix(sched, x_start, s) - gaussian_exact(X_T, 1e-3)).max()))
    got = -np.polyfit(np.log(STEPS), np.log(errs), 1)[0]
    assert lo <= got <= hi, errs


def test_full_strength_remix_is_the_request():
    """t_start = S reads exactly the request's own rows"""
    sched = D.multistep_schedule(ACP, 12, 3, "logSNR")
    assert np.array_equal(D.chart_orders(sched, [12])[0], sched.orders)


# ---- the oracle against the reference's DDIM remix goldens ------------------------------------------------------------------------
DDIM_REMIX = [n for n, cse in rc.REMIX_CASES.items() if cse["sampler"] == "ddim"]


@pytest.mark.parametrize("name", DDIM_REMIX)
def test_order_one_remix_on_the_ddim_grid_matches_the_reference(name, golden_dir):
    """decode(x_T, s = subset_end(k, n)) of order 1 on DDIM's grid is the reference's ddim_sampling(x_T, timesteps=k)"""
    case = rc.REMIX_CASES[name]
    ts = ddim_timesteps_uniform(case["S"], 1000)
    n = len(ts)
    sched = D.multistep_schedule(ACP, n, 1, t_grid=D.ddim_grid(NS, ts))
    s = rc.subset_end(case["k"], n)
    sd = synth.synthetic_state_dict(case["L"])
    inp = synth.synthetic_inputs(case["B"], case["L"])
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    x_start = rc.intermediates(g, "x_inter")[0]
    assert torch.equal(x_start, inp["x_T"])
    with torch.no_grad():
        z = oracle_decode(sd, sched, x_start, inp["c"], inp["w"], s, scale=case["scale"], uc=inp["uc"])
        logits = orc.decoder_forward(sd, z)
    if s == 0:
        assert z is x_start
    assert rel_err(z, g["z"]) < 1e-3
    assert rel_err(logits, g["logits"]) < 1e-3


# ---- C ABI -------------------------------------------------------------------------------------------------------------------------
def test_library_exports_the_dpm_ex_entry_points_at_abi_13():
    lib = L_.load()
    assert lib.mugd_abi_version() == L_.ABI_VERSION == 13
    for sym in ("mugd_sample_dpm_ex", "mugd_dpm_ex_update"):
        assert sym in L_.EXPORTED_SYMBOLS and hasattr(lib, sym)
    with open(os.path.join(os.path.dirname(L_.HERE), "include", "mugd.h")) as f:
        h = f.read()
    assert "int  mugd_sample_dpm_ex(mugd_plan* eval_plan, const mugd_dpm_ex* e, int32_t first_step, int32_t n_steps, void* stream);" in h
    assert "int  mugd_dpm_ex_update(const mugd_dpm_ex* e, void* stream);" in h
    assert C.sizeof(L_.DpmEx) == C.sizeof(L_.Dpm) + 3 * 8 + 2 * 4


N, S_ = 2 * 16 * 8, 6
_QCOEF = np.ones((S_, 2), np.float32)


def _ex(kind):
    """a well-formed descriptor over fake (never dereferenced) device addresses: kind "stage" (inpainting) or "start" (remix)"""
    d = L_.Dpm()
    d.x, d.x_dup, d.eps, d.pred_x0, d.ring, d.coef, d.step = 0x1000, 0x2000, 0x3000, 0x4000, 0x5000, 0x6000, 0x7000
    d.n, d.S, d.cfg, d.scale = N, S_, 1, 5.0
    e = L_.DpmEx()
    e.dpm = d
    st = L_.Stage()
    st.x, st.x_dup, st.x0, st.mask, st.q_noise, st.q_coef = 0x1000, 0x2000, 0x8000, 0x9000, 0xa000, _QCOEF.ctypes.data
    st.B, st.C, st.L = 2, 16, 8
    if kind == "stage":
        e.stage = C.addressof(st)
    else:
        e.start, e.order_coef, e.B = 0xb000, 0xc000, 2
    return e, st


def _malformed_ex():
    out = []
    e, st = _ex("start"); e.dpm.ring = None; out.append((e, st, "must be given"))
    e, st = _ex("start"); e.order_coef = None; out.append((e, st, "start and order_coef go together"))
    e, st = _ex("start"); e.start = None; out.append((e, st, "start and order_coef go together"))
    e, st = _ex("start"); e.B = 3; out.append((e, st, "B=3 does not divide n=256"))
    e, st = _ex("start"); e.B = 0; out.append((e, st, "B=0 does not divide"))
    e, st = _ex("stage"); e.start, e.order_coef, e.B = 0xb000, 0xc000, 2; out.append((e, st, "cannot be combined"))
    e, st = _ex("stage"); st.x0, st.mask, st.q_noise, st.q_coef = None, None, None, None; out.append((e, st, "has no x0"))
    e, st = _ex("stage"); st.mask = None; out.append((e, st, "x0 needs mask"))
    e, st = _ex("stage"); st.noise, st.noise_rows = 0xd000, 0xe000; out.append((e, st, "DPM-Solver++ draws none"))
    e, st = _ex("stage"); st.x = 0xf000; out.append((e, st, "other rows"))
    e, st = _ex("stage"); st.x_dup = None; out.append((e, st, "other rows"))
    e, st = _ex("stage"); st.L = 4; out.append((e, st, "the update's n=256"))
    return out


@pytest.mark.parametrize("case", range(len(_malformed_ex())))
@pytest.mark.parametrize("entry", ["update", "loop"])
def test_dpm_ex_entry_points_check_their_arguments_without_a_device(case, entry):
    e, st, msg = _malformed_ex()[case]
    lib = L_.load()
    rc_ = lib.mugd_dpm_ex_update(C.byref(e), None) if entry == "update" else lib.mugd_sample_dpm_ex(None, C.byref(e), 0, 2, None)
    assert rc_ == 1
    assert msg in lib.mugd_last_error().decode()


def test_sample_dpm_ex_checks_the_stage_table_and_the_step_range_before_the_plan():
    lib = L_.load()
    e, st = _ex("stage")
    bad = _QCOEF.copy()
    bad[3, 1] = np.inf
    st.q_coef = bad.ctypes.data
    assert lib.mugd_sample_dpm_ex(None, C.byref(e), 0, 3, None) == 1                           # rows 0..2 are finite: the plan is next
    assert "must be captured" in lib.mugd_last_error().decode()
    assert lib.mugd_sample_dpm_ex(None, C.byref(e), 0, 4, None) == 1
    assert "q_coef[3][1] = inf is not finite" in lib.mugd_last_error().decode()
    for kind in ("stage", "start"):
        e, st = _ex(kind)
        for first, n in ((0, S_ + 1), (S_, 1), (-1, 1), (2, -1)):
            assert lib.mugd_sample_dpm_ex(None, C.byref(e), first, n, None) == 1
            assert "outside the S=6 steps" in lib.mugd_last_error().decode()
        assert lib.mugd_sample_dpm_ex(None, C.byref(e), 1, S_ - 1, None) == 1
        assert "must be captured" in lib.mugd_last_error().decode()
    assert lib.mugd_sample_dpm_ex(None, None, 0, 1, None) == 1 and "null descriptor" in lib.mugd_last_error().decode()
    assert lib.mugd_dpm_ex_update(None, None) == 1 and "null argument" in lib.mugd_last_error().decode()



# ---- the sampler refuses before any GPU work -------------------------------------------------------------------------------------
def _inpaint_request(B=2, L=96, **kw):
    base = _request(B, L)
    base.update(mask=torch.ones(B, 1, L), x0=torch.zeros(B, 16, L))
    base.update(kw)
    return base


BAD_INPAINT = [
    (dict(mask=None), ValueError, "mask and x0 as tensors"),
    (dict(x0=None), ValueError, "mask and x0 as tensors"),
    (dict(x0=np.zeros((2, 16, 96), np.float32)), ValueError, "mask and x0 as tensors"),
    (dict(x0=torch.zeros(2, 16, 64)), ValueError, "inpainting needs x0 of shape"),
    (dict(mask=torch.ones(3, 1, 96)), ValueError, "does not broadcast"),
    (dict(S=1, order=2), ValueError, "order 2 needs at least 2 steps"),
    (dict(S=0), ValueError, "number of steps"),
    (dict(order=4), ValueError, "order=4"),
    (dict(skip_type="uniform"), ValueError, "skip_type='uniform'"),
    (dict(solver_type="dpm_solver"), ValueError, "solver_type='dpm_solver'"),
    (dict(lower_order_final=None), ValueError, "lower_order_final=None"),
    (dict(unconditional_guidance_scale=float("nan")), ValueError, "must be a finite number"),
    (dict(batch_size=0), ValueError, "batch_size"),
    (dict(log_every_t=0), ValueError, "log_every_t"),
    (dict(x_T=torch.zeros(2, 16, 64)), ValueError, "x_T has shape"),
    (dict(c=torch.zeros(3, 128, 21)), ValueError, "c must be"),
    (dict(c=None), TypeError, "needs the conditioning"),
    (dict(w=None), TypeError, "audio features"),
    (dict(conditioning=torch.zeros(2, 128, 21)), TypeError, "not both"),
    (dict(eta=0.5), TypeError, "eta"),
    (dict(noise_dropout=0.1), TypeError, "noise_dropout"),
    (dict(temperature=0.9), TypeError, "temperature"),
]


def _match(msg):
    return msg.replace("(", r"\(").replace(")", r"\)").replace(".", r"\.")


@pytest.mark.parametrize("kw,exc,msg", BAD_INPAINT, ids=[f"bad{i}" for i in range(len(BAD_INPAINT))])
def test_inpaint_refuses_before_any_gpu_work(kw, exc, msg):
    with pytest.raises(exc, match=_match(msg)):
        _cpu_sampler().inpaint(**_inpaint_request(**kw))


def test_a_valid_inpainting_request_reaches_the_engine():
    for kw in (_inpaint_request(order=3, skip_type="logSNR"), _inpaint_request(S=1, order=1, mask=torch.ones(16, 96))):
        kw["conditioning"] = kw.pop("c")
        with pytest.raises(AttributeError, match="engine"):
            _cpu_sampler().inpaint(**kw)


SCHED = D.multistep_schedule(ACP, 10, 2)
X0 = torch.zeros(2, 16, 96)
BAD_ENCODE = [
    (dict(sched=None), "sched must be a DPMSchedule"),
    (dict(x0=torch.zeros(2, 16, 96, dtype=torch.float64)), "x0 must be a float32"),
    (dict(x0=torch.zeros(16, 96)), "x0 must be a float32"),
    (dict(t_enc=11), r"every start must lie in \[0, 10\] \(S = sched\.S\)"),
    (dict(t_enc=-1), r"every start must lie in \[0, 10\]"),
    (dict(t_enc=[1, 2, 3]), "t_enc has 3 entries for 2 charts"),
    (dict(t_enc=[1.0, 2.0]), "must be integers"),
    (dict(t_enc=2.0), "must be an integer or one integer per chart"),
    (dict(t_enc=True), "must be an integer or one integer per chart"),
    (dict(noise=torch.zeros(2, 16, 64)), "noise must be a float32 tensor"),
]


@pytest.mark.parametrize("kw,msg", BAD_ENCODE, ids=[f"bad{i}" for i in range(len(BAD_ENCODE))])
def test_stochastic_encode_refuses_before_any_gpu_work(kw, msg):
    args = dict(x0=X0, t_enc=[3, 10], sched=SCHED, noise=None)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        _cpu_sampler().stochastic_encode(**args)


BAD_DECODE = [
    (dict(sched=D.DPMSchedule(SCHED.t, SCHED.model_times, SCHED.rows, SCHED.orders)), "sched must be a DPMSchedule"),
    (dict(x_latent=torch.zeros(2, 8, 96)), r"x_latent must be a \[B, 16, L\] tensor"),
    (dict(x_latent=torch.zeros(0, 16, 96)), r"x_latent must be a \[B, 16, L\] tensor"),
    (dict(t_start=11), r"every start must lie in \[0, 10\]"),
    (dict(t_start=[4, 11]), r"every start must lie in \[0, 10\]"),
    (dict(t_start=[4]), "t_start has 1 entries for 2 charts"),
    (dict(t_start=torch.tensor([1.0, 2.0])), "must be integers"),
    (dict(t_start=None), "must be an integer or one integer per chart"),
    (dict(c=torch.zeros(3, 128, 21)), "c must be"),
    (dict(c=None), "needs the conditioning c and the audio features w"),
    (dict(w=None), "needs the conditioning c and the audio features w"),
    (dict(unconditional_guidance_scale=float("inf")), "must be a finite number"),
    (dict(unconditional_conditioning=torch.zeros(1, 128, 21)), "unconditional_conditioning must be"),
]


@pytest.mark.parametrize("kw,msg", BAD_DECODE, ids=[f"bad{i}" for i in range(len(BAD_DECODE))])
def test_decode_refuses_before_any_gpu_work(kw, msg):
    r = _request()
    args = dict(x_latent=torch.zeros(2, 16, 96), c=r["c"], w=r["w"], t_start=[3, 10], sched=SCHED, unconditional_guidance_scale=5.0,
                unconditional_conditioning=r["unconditional_conditioning"])
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        _cpu_sampler().decode(**args)


def test_decode_of_zero_steps_returns_the_latent_without_gpu_work():
    r = _request()
    z = torch.zeros(2, 16, 96)
    assert _cpu_sampler().decode(z, r["c"], r["w"], 0, SCHED) is z
    assert _cpu_sampler().decode(z, r["c"], r["w"], [0, 0], SCHED, 5.0, r["unconditional_conditioning"]) is z


def test_sample_still_refuses_inpainting():
    with pytest.raises(ValueError, match="mask="):
        _cpu_sampler().sample(**_request(mask=torch.ones(2, 1, 96), x0=torch.zeros(2, 16, 96)))


# ---- inpainting's request loop on a recording stand-in ------------------------------------------------------------------------------
class _InpaintRecorder(_Recorder):
    def __init__(self):
        super().__init__()
        self.ex = []

    def dpm_ex(self, dpm, stage=None, **kw):
        assert stage is not None and not kw
        self.stage = stage
        return L_.DpmEx()

    def launch_dpm_ex(self, ex, first, n):
        self.q_rows.append(self.stage.q_coef)
        self._device("dpm_ex", first, n)


def _run_inpaint(monkeypatch, total, log_every_t, cap, callback):
    rec = _InpaintRecorder()
    monkeypatch.setattr(sampler_mod, "STAGE_TABLE_BYTES", cap * STEP_BYTES + 5)

    def draw(steps, shape, x0, q_table, draw_noise, noise_table, noise_dropout, device):
        assert tuple(shape) == SHAPE and steps >= 1 and q_table.shape[0] >= steps and x0 is x0_in
        rec.trace.append(("draw", steps, not draw_noise, noise_table is None, noise_dropout))

    monkeypatch.setattr(sampler_mod, "draw_step_noise", draw)
    real_randn_like = torch.randn_like
    monkeypatch.setattr(torch, "randn_like", lambda t, **k: (rec.trace.append(("randn_like", tuple(t.shape))), real_randn_like(t, **k))[1])
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    model = types.SimpleNamespace(engine=rec, z_channels=SHAPE[1], z_length=SHAPE[2], num_timesteps=1000)
    s = object.__new__(sampler_mod.DPMSolverSampler)
    s.model, s.ddpm_num_timesteps, s.device, s.last_launches_per_step = model, 1000, "cpu", 0
    x = torch.zeros(SHAPE)
    monkeypatch.setattr(s, "_load_session", lambda w, c, shape, x_T, scale, uc, time_range: (x, False, rec, time_range))
    ticks = []
    kw = dict(tqdm_class=lambda it, desc, total: _Bar(it, desc, total, ticks, rec), log_every_t=log_every_t)
    if callback:
        kw["callback"] = lambda i: rec.trace.append(("callback", i))
    x0_in = torch.zeros(SHAPE)
    sched = D.multistep_schedule(ACP, total, min(2, total))
    z, inter = s.dpm_sampling([], None, SHAPE, sched, mask=torch.ones(1, 1, SHAPE[2]), x0=x0_in, **kw)
    return rec, z, inter, ticks, s, sched


@pytest.mark.parametrize("cap", [1 << 20, SMALL_CAP])
@pytest.mark.parametrize("log_every_t", [1, 7, 100])
@pytest.mark.parametrize("total", [1, 2, 10, 25])
def test_inpaint_device_loop(monkeypatch, total, log_every_t, cap):
    """per stretch between logged steps, calls of at most STAGE_TABLE_BYTES' steps, each drawing its blend noise up front (no step
    noise) and pointing the stage at its rows of the (alpha_i, sigma_i) table; DDIM staged's launches per step"""
    rec, z, inter, ticks, s, sched = _run_inpaint(monkeypatch, total, log_every_t, cap, False)
    want, firsts = [], []
    for first, n in _stretches(total, log_every_t):
        for k in range(first, first + n, cap):
            m = min(cap, first + n - k)
            want += [("draw", m, True, True, 0.0), ("dpm_ex", k, m)]
            firsts.append(k)
    assert rec.trace == want
    assert [q - rec.q_rows[0] for q in rec.q_rows] == [8 * k for k in firsts]
    assert s.last_launches_per_step == PLAN_LAUNCHES + 3
    ends = [f + n for f, n in _stretches(total, log_every_t)]
    assert [float(t.flatten()[0]) for t in inter["x_inter"]] == [0.0] + [float(e) for e in ends]
    assert len(ticks) == total


@pytest.mark.parametrize("log_every_t", [1, 7])
@pytest.mark.parametrize("total", [1, 2, 10])
def test_inpaint_per_step_loop(monkeypatch, total, log_every_t):
    """per step: one randn_like(x0) for the blend, the blended x loaded, the evaluation, the update and the advance"""
    rec, z, inter, ticks, s, sched = _run_inpaint(monkeypatch, total, log_every_t, SMALL_CAP, True)
    want = []
    for i in range(total):
        want += [("randn_like", SHAPE), ("load_x",), ("eval", i), ("dpm_update",), ("ops", L_.OP_STEP_ADVANCE), ("callback", i)]
    assert rec.trace == want
    assert s.last_launches_per_step == PLAN_LAUNCHES + 2
    assert len(inter["x_inter"]) == 1 + sum(_logged(i, total, log_every_t) for i in range(total))
