"""Remixing an existing chart, CPU side: the reference's ``timesteps=`` subset rule over every schedule length, the oracle's truncated
DDIM / PLMS runs against the UNMODIFIED reference (tests/golden/remix_*.npz), the oracle's decode against its truncated sampling and
its per-chart joins against scalar runs, the argument checks of ddim_sampling / plms_sampling / stochastic_encode / decode before any
GPU work, and the exported entry points checking their arguments without a device."""
import ctypes as C
import os
import threading
import types

import numpy as np
import pytest
import torch

import golden_cases as gc
import remix_cases as rc
import remix_oracle as ro
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth
from mug_diffusion_b200.sampler import (DDIMSampler, PLMSSampler, ddim_parameters, ddim_subset_end, ddim_timesteps_uniform,
                                        register_schedule, takes_device_loop)
from oracle import mug_oracle as orc


def rel_err(a, b):
    b = torch.as_tensor(b)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ---- the subset rule ------------------------------------------------------------------------------------------------------------
def _reference_subset(ddim_timesteps, timesteps):
    """ddim.py:126-131 verbatim (the ddim_use_original_steps=False branch)"""
    subset_end = int(min(timesteps / ddim_timesteps.shape[0], 1) * ddim_timesteps.shape[0]) - 1
    timesteps = ddim_timesteps[:subset_end]
    return np.flip(timesteps), timesteps.shape[0]


class _NoGpu:
    lock = threading.RLock()

    def __getattr__(self, name):
        raise AssertionError(f"GPU work started: engine.{name}")


def _sampler(cls=DDIMSampler, S=10, eta=0.0):
    """a sampler over a stand-in model whose engine raises on any use, with make_schedule's tables (from the model's schedule)"""
    sch = register_schedule()
    model = types.SimpleNamespace(engine=_NoGpu(), z_channels=16, z_length=96, num_timesteps=1000, **sch)
    s = object.__new__(cls)
    s.model, s.ddpm_num_timesteps, s.device, s.last_launches_per_step = model, 1000, "cpu", 0
    s.make_schedule(S, ddim_eta=eta, verbose=False)
    return s


def test_subset_rule_equals_the_reference_expression_for_every_schedule():
    s = object.__new__(DDIMSampler)
    lengths, pulled_down = set(), set()
    for S in range(1, 1001):
        ts = ddim_timesteps_uniform(S, 1000)
        n = ts.shape[0]
        lengths.add(n)
        s.ddim_timesteps = ts
        for k in range(0, n + 3):
            want_range, want_total = _reference_subset(ts, k)
            got = s._schedule_subset(k, False)
            assert got.shape[0] == want_total and np.array_equal(np.flip(got), want_range), (S, k)
            assert ddim_subset_end(k, n) == rc.subset_end(k, n)
            if 1 <= k <= n and want_total != k - 1:
                pulled_down.add((k, n))                                          # the float product rounded down
    assert ddim_timesteps_uniform(30, 1000).shape[0] == 31
    s.ddim_timesteps = ddim_timesteps_uniform(50, 1000)
    assert s._schedule_subset(29, False).shape[0] == 27                      # int(28.999999999999996) - 1
    assert s._schedule_subset(1, False).shape[0] == 0
    assert s._schedule_subset(51, False).shape[0] == 49
    assert (29, 50) in pulled_down and len(pulled_down) == 66 and len(lengths) == 57


# ---- the oracle against the reference -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(rc.REMIX_CASES))
def test_oracle_equals_the_reference_truncated_runs(name, golden_dir):
    case = rc.REMIX_CASES[name]
    sd = synth.synthetic_state_dict(case["L"])
    inp = synth.synthetic_inputs(case["B"], case["L"])
    run = ro.ddim_sampling if case["sampler"] == "ddim" else ro.plms_sampling
    with torch.no_grad():
        z, inter = run(sd, case["S"], inp["c"], inp["w"], inp["x_T"], scale=case["scale"], uc=inp["uc"], timesteps=case["k"],
                       log_every_t=rc.LOG_EVERY_T)
        logits = orc.decoder_forward(sd, z)
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    assert rel_err(z, g["z"]) <= 2e-5
    assert rel_err(logits, g["logits"]) <= 2e-5
    steps = ro.subset(case["S"], case["k"]).shape[0]
    for key in ("x_inter", "pred_x0"):
        ref = rc.intermediates(g, key)
        assert len(inter[key]) == len(ref) == 1 + sum(1 for i in range(steps) if (steps - i - 1) % rc.LOG_EVERY_T == 0 or i == 0)
        for a, b in zip(inter[key], ref):
            assert rel_err(a, b) <= 2e-5, key
    if steps == 0:
        assert torch.equal(z, inp["x_T"]) and inter == {'x_inter': [inp["x_T"]], 'pred_x0': [inp["x_T"]]}


def test_oracle_decode_equals_its_truncated_sampling():
    """decode(z, s) == ddim_sampling(x_T=z, timesteps=s + 1) bit for bit wherever the subset gives s steps; s = n runs the whole
    schedule, s = 0 returns the latent"""
    L, B, S = 96, 1, 10
    sd = synth.synthetic_state_dict(L)
    inp = synth.synthetic_inputs(B, L)
    n = orc.make_schedule(S)["timesteps"].shape[0]
    with torch.no_grad():
        for s in (1, 4, n - 1):
            assert ro.subset(S, s + 1).shape[0] == s
            want, _ = ro.ddim_sampling(sd, S, inp["c"], inp["w"], inp["x_T"], timesteps=s + 1)
            assert torch.equal(ro.decode(sd, S, inp["x_T"], inp["c"], inp["w"], s), want), s
        full, _ = ro.ddim_sampling(sd, S, inp["c"], inp["w"], inp["x_T"])
        assert torch.equal(ro.decode(sd, S, inp["x_T"], inp["c"], inp["w"], n), full)
        assert ro.decode(sd, S, inp["x_T"], inp["c"], inp["w"], 0) is inp["x_T"]


def test_oracle_per_chart_starts_follow_their_own_scalar_runs():
    L, B, S = 96, 3, 10
    sd = synth.synthetic_state_dict(L)
    inp = synth.synthetic_inputs(B, L)
    starts = [0, 2, 5]
    with torch.no_grad():
        z = ro.decode(sd, S, inp["x_T"], inp["c"], inp["w"], starts, scale=5.0, uc=inp["uc"])
        assert torch.equal(z[0], inp["x_T"][0])
        for b in (1, 2):
            one = ro.decode(sd, S, inp["x_T"][b:b + 1], inp["c"][b:b + 1], [wi[b:b + 1] for wi in inp["w"]], starts[b], scale=5.0,
                            uc=inp["uc"][b:b + 1])
            assert rel_err(z[b:b + 1], one) <= 1e-5, b


# ---- argument checks before any GPU work ----------------------------------------------------------------------------------------
def test_original_steps_raise_before_any_gpu_work():
    for cls, run in ((DDIMSampler, "ddim_sampling"), (PLMSSampler, "plms_sampling")):
        s = _sampler(cls)
        with pytest.raises(ValueError, match="ddim_sigmas_for_original_num_steps"):
            getattr(s, run)([], None, (1, 16, 96), ddim_use_original_steps=True)
        with pytest.raises(ValueError, match="finite number"):
            getattr(s, run)([], None, (1, 16, 96), timesteps=float("nan"))
        with pytest.raises(ValueError, match="finite number"):
            getattr(s, run)([], None, (1, 16, 96), timesteps=True)


@pytest.mark.parametrize("cls", [DDIMSampler, PLMSSampler])
def test_empty_subset_returns_x_T_without_gpu_work(cls):
    s = _sampler(cls)
    x_T = torch.randn(2, 16, 96)
    z, inter = getattr(s, "ddim_sampling" if cls is DDIMSampler else "plms_sampling")([], None, (2, 16, 96), x_T=x_T, timesteps=1)
    assert z is x_T and inter == {'x_inter': [x_T], 'pred_x0': [x_T]}


@pytest.mark.parametrize("mask,eta", [(False, 0.0), (True, 0.0), (False, 1.0), (True, 1.0)])
def test_subset_requests_reach_the_device_loop(monkeypatch, mask, eta):
    """timesteps= changes only the timesteps the request loads: with and without mask / eta the request reaches _load_request with
    the subset, and the routing rule (which does not look at timesteps) sends it to the device loop"""
    s = _sampler(S=10, eta=eta)
    shape = (2, 16, 96)
    seen = {}

    def stop(w, c, shp, x_T, scale, uc, ts=None):
        seen["ts"] = ts
        raise RuntimeError("stop")

    monkeypatch.setattr(s, "_load_request", stop)
    x0 = torch.zeros(shape) if mask else None
    m = torch.ones(shape) if mask else None
    with pytest.raises(RuntimeError, match="stop"):
        s.ddim_sampling([], None, shape, x_T=torch.zeros(shape), timesteps=5, mask=m, x0=x0)
    assert np.array_equal(seen["ts"], s.ddim_timesteps[:4])
    assert takes_device_loop(shape, "cpu", m, x0)


def _decode_args(B=2, L=96):
    return dict(x_latent=torch.zeros(B, 16, L), c=torch.zeros(B, 128, 21), w=[torch.zeros(B, 4, L)], t_start=3)


@pytest.mark.parametrize("change,msg", [
    (dict(x_latent=torch.zeros(2, 8, 96)), "x_latent must be"),
    (dict(x_latent=torch.zeros(16, 96)), "x_latent must be"),
    (dict(x_latent=None), "x_latent must be"),
    (dict(t_start=11), r"lie in \[0, 10\]"),
    (dict(t_start=-1), r"lie in \[0, 10\]"),
    (dict(t_start=[1, 2, 3]), "3 entries for 2 charts"),
    (dict(t_start=[1, 11]), r"lie in \[0, 10\]"),
    (dict(t_start=[1, 2.0]), "must be integers"),
    (dict(t_start=2.0), "must be an integer"),
    (dict(t_start=True), "must be an integer"),
    (dict(c=torch.zeros(3, 128, 21)), "c must be"),
    (dict(use_original_steps=True), "ddim_sigmas_for_original_num_steps"),
    (dict(unconditional_guidance_scale=5.0, unconditional_conditioning=torch.zeros(1, 128, 21)), "unconditional_conditioning must be"),
])
def test_decode_refuses_before_any_gpu_work(change, msg):
    kw = _decode_args()
    kw.update(change)
    with pytest.raises(ValueError, match=msg):
        _sampler().decode(**kw)


def test_decode_needs_an_eta_0_schedule_and_returns_s_0_untouched():
    with pytest.raises(ValueError, match="eta = 0"):
        _sampler(eta=1.0).decode(**_decode_args())
    s = object.__new__(DDIMSampler)
    s.model, s.device = types.SimpleNamespace(engine=_NoGpu(), z_channels=16), "cpu"
    with pytest.raises(ValueError, match="make_schedule"):
        s.decode(**_decode_args())
    kw = _decode_args()
    kw["t_start"] = [0, 0]
    assert _sampler().decode(**kw) is kw["x_latent"]


@pytest.mark.parametrize("t,msg", [([0, 10], r"lie in \[0, 9\]"), ([-1, 0], r"lie in \[0, 9\]"), ([0], "one per chart"),
                                   ([0.0, 1.0], "integer table indices"), (torch.tensor([[0, 1]]), "one per chart")])
def test_stochastic_encode_refuses_before_any_gpu_work(t, msg):
    s = _sampler(S=10)
    torch.manual_seed(3)
    with pytest.raises(ValueError, match=msg):
        s.stochastic_encode(torch.zeros(2, 16, 96), t)
    after = torch.randn(3)
    torch.manual_seed(3)
    assert torch.equal(after, torch.randn(3))                                   # no noise was drawn


def test_stochastic_encode_checks_the_original_steps_table_range():
    s = _sampler(S=10)
    with pytest.raises(ValueError, match=r"lie in \[0, 999\]"):
        s.stochastic_encode(torch.zeros(1, 16, 96), [1000], use_original_steps=True)
    with pytest.raises(ValueError, match="noise must be"):
        s.stochastic_encode(torch.zeros(1, 16, 96), [3], noise=torch.zeros(1, 16, 95))


def test_make_schedule_tables_are_the_encode_tables():
    """stochastic_encode's default tables are make_schedule's: sqrt(ddim_alphas) (torch's float32 sqrt) and
    ddim_sqrt_one_minus_alphas, both float32"""
    s = _sampler(S=50)
    _, alphas, _ = ddim_parameters(s.model.alphas_cumprod, s.ddim_timesteps, 0.0)
    assert torch.equal(torch.as_tensor(s.ddim_alphas), alphas)
    assert torch.as_tensor(s.ddim_sqrt_one_minus_alphas).dtype == torch.float32


# ---- the library --------------------------------------------------------------------------------------------------------------
def test_library_exports_the_remix_entry_points_at_abi_13():
    lib = L_.load()
    assert lib.mugd_abi_version() == L_.ABI_VERSION == 13
    for sym in ("mugd_stochastic_encode", "mugd_sample_join"):
        assert sym in L_.EXPORTED_SYMBOLS and hasattr(lib, sym)
    with open(os.path.join(os.path.dirname(L_.HERE), "include", "mugd.h")) as f:
        h = f.read()
    assert "int  mugd_stochastic_encode(const mugd_q_encode* d, void* stream);" in h
    assert "int  mugd_sample_join(mugd_plan* eval_plan, const mugd_join* join, const mugd_op* tail, int32_t n_tail, int32_t first_step," in h
    assert C.sizeof(L_.QEncode) == 6 * 8 + 4 * 4 and C.sizeof(L_.Join) == 4 * 8 + 4 * 4


def _q_encode():
    d = L_.QEncode()
    d.x0, d.noise, d.t, d.sqrt_a, d.sqrt_1ma, d.out = 0x1000, 0x2000, 0x3000, 0x4000, 0x5000, 0x6000
    d.B, d.C, d.L, d.n = 2, 16, 96, 10
    return d


def _encode_malformed():
    out = []
    for f in ("x0", "noise", "t", "sqrt_a", "sqrt_1ma", "out"):
        d = _q_encode(); setattr(d, f, None); out.append((d, "must be given"))
    d = _q_encode(); d.B = 0; out.append((d, "bad shape"))
    d = _q_encode(); d.L = -1; out.append((d, "bad shape"))
    d = _q_encode(); d.n = 0; out.append((d, "n=0 rows"))
    return out


@pytest.mark.parametrize("case", range(len(_encode_malformed())))
def test_stochastic_encode_entry_checks_its_arguments_without_a_device(case):
    d, msg = _encode_malformed()[case]
    lib = L_.load()
    assert lib.mugd_stochastic_encode(C.byref(d), None) == 1
    assert msg in lib.mugd_last_error().decode()
    assert lib.mugd_stochastic_encode(None, None) == 1
    assert "null argument" in lib.mugd_last_error().decode()


def test_sample_join_needs_a_captured_plan_and_a_descriptor():
    lib = L_.load()
    j = L_.Join()
    assert lib.mugd_sample_join(None, C.byref(j), None, 0, 0, 1, None) == 1
    assert "must be captured" in lib.mugd_last_error().decode()
