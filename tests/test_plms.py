"""PLMS sampler, CPU side: the oracle restatement equals the UNMODIFIED reference plms.py (tests/golden/plms_*.npz), requests the
device path cannot take are refused before any GPU work, and libmugd exports the PLMS entry points at ABI 13, checking their
arguments before anything is launched."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

import golden_cases as gc
import plms_cases as pc
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth
from mug_diffusion_b200.sampler import PLMSSampler, register_schedule
from oracle import mug_oracle as orc
from plms_oracle import plms_sample


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("name", list(pc.PLMS_CASES))
def test_oracle_equals_the_reference_plms(name, golden_dir):
    case = pc.PLMS_CASES[name]
    sd = synth.synthetic_state_dict(case["L"])
    inp = synth.synthetic_inputs(case["B"], case["L"])
    with torch.no_grad():
        z, inter = plms_sample(sd, case["S"], inp["c"], inp["w"], inp["x_T"], scale=case["scale"], uc=inp["uc"],
                                   log_every_t=pc.LOG_EVERY_T)
        logits = orc.decoder_forward(sd, z)
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    assert rel_err(z, g["z"]) <= 2e-5
    assert rel_err(logits, g["logits"]) <= 2e-5
    for key in ("x_inter", "pred_x0"):
        ref = pc.intermediates(g, key)
        assert len(inter[key]) == len(ref) == pc.n_logged(case["S"], pc.LOG_EVERY_T)
        for a, b in zip(inter[key], ref):
            assert rel_err(a, b) <= 2e-5, key
    assert not torch.equal(inter["x_inter"][1], inter["x_inter"][2])             # the trajectory moves


def test_plms_differs_from_ddim_on_the_same_request(golden_dir):
    """the PLMS golden is not the DDIM golden of the same inputs: the multistep combine changed the trajectory"""
    p, d = (gc.load_golden(os.path.join(golden_dir, n + ".npz")) for n in ("plms_L96_B2_S10_cfg5", "ddim_L96_B2_S10_cfg5"))
    assert rel_err(p["z"], d["z"]) > 1e-3


def _cpu_sampler(L=96):
    """a PLMSSampler over a stand-in model: enough for the checks that run before any GPU work"""
    s = PLMSSampler.__new__(PLMSSampler)
    sch = register_schedule()
    s.model = types.SimpleNamespace(z_channels=16, z_length=L, num_timesteps=1000, alphas_cumprod=sch["alphas_cumprod"])
    s.ddpm_num_timesteps, s.device = 1000, torch.device("cpu")
    return s


def _request(B=2, L=96, **kw):
    inp = synth.synthetic_inputs(B, L)
    base = dict(S=10, c=inp["c"], w=inp["w"], batch_size=B, shape=(16, L), verbose=False, x_T=inp["x_T"],
                unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"])
    base.update(kw)
    return base


BAD = [
    (dict(eta=0.5), ValueError, "ddim_eta must be 0 for PLMS"),
    (dict(eta=1.0, S=0), ValueError, "ddim_eta must be 0 for PLMS"),
    (dict(S=0), ValueError, "number of steps"),
    (dict(S=1001), ValueError, "number of steps"),
    (dict(S=2.5), ValueError, "number of steps"),
    (dict(S=3), ValueError, "reaches timestep 1000"),
    (dict(batch_size=0), ValueError, "batch_size"),
    (dict(log_every_t=0), ValueError, "log_every_t"),
    (dict(shape=(16, 96, 1)), ValueError, "(channels, length)"),
    (dict(shape=(8, 96)), ValueError, "16 channels"),
    (dict(x_T=torch.zeros(2, 16, 64)), ValueError, "x_T has shape"),
    (dict(c=torch.zeros(3, 128, 21)), ValueError, "c must be"),
    (dict(unconditional_conditioning=torch.zeros(1, 128, 21)), ValueError, "unconditional_conditioning must be"),
    (dict(c=None), TypeError, "needs the conditioning"),
    (dict(w=None), TypeError, "audio features"),
    (dict(conditioning=torch.zeros(2, 128, 21)), TypeError, "not both"),
    (dict(mask=torch.ones(2, 1, 96)), ValueError, "needs x0"),
    (dict(mask=torch.ones(2, 1, 96), x0=torch.zeros(2, 16, 48)), ValueError, "needs x0"),
    (dict(mask=torch.ones(3, 1, 96), x0=torch.zeros(2, 16, 96)), ValueError, "does not broadcast"),
]


@pytest.mark.parametrize("kw,exc,msg", BAD, ids=[f"bad{i}" for i in range(len(BAD))])
def test_sample_refuses_before_any_gpu_work(kw, exc, msg):
    with pytest.raises(exc, match=msg.replace("(", r"\(").replace(")", r"\)")):
        _cpu_sampler().sample(**_request(**kw))


def test_make_schedule_refuses_eta():
    s = _cpu_sampler()
    with pytest.raises(ValueError, match="ddim_eta must be 0 for PLMS"):
        s.make_schedule(10, ddim_eta=0.1, verbose=False)
    s.make_schedule(10, verbose=False)
    assert len(s.ddim_timesteps) == 10 and float(np.abs(np.asarray(s.ddim_sigmas, dtype=np.float64)).max()) == 0.0


def test_conditioning_is_accepted_under_the_reference_name():
    """``conditioning=`` (plms.py:62) passes the checks like ``c=``; the run then needs the engine, which this stand-in lacks"""
    kw = _request()
    kw["conditioning"] = kw.pop("c")
    with pytest.raises(AttributeError, match="engine"):
        _cpu_sampler().sample(**kw)


def test_library_exports_plms_at_abi_13():
    lib = L_.load()
    assert lib.mugd_abi_version() == L_.ABI_VERSION == 13
    for sym in ("mugd_sample_plms", "mugd_plms_combine"):
        assert sym in L_.EXPORTED_SYMBOLS and hasattr(lib, sym)
    with open(os.path.join(os.path.dirname(L_.HERE), "include", "mugd.h")) as f:
        h = f.read()
    assert "int  mugd_sample_plms(mugd_plan* eval_plan, const mugd_plms* p, int32_t first_step, int32_t n_steps, void* stream);" in h


def _plms(n=64, S=10):
    """a well-formed descriptor over fake (never dereferenced) addresses"""
    p = L_.Plms()
    u = p.update
    u.x, u.x_dup, u.pred_x0, u.coef, u.step = 0x1000, 0x2000, 0x3000, 0x4000, 0x5000
    u.eps, u.noise, u.S, u.n, u.cfg = 0x6000, None, S, n, 0
    p.eps, p.e_prime, p.hist, p.x_stash, p.cfg, p.scale = 0x7000, 0x6000, 0x8000, 0x9000, 1, 5.0
    return p


def _malformed():
    out = []
    p = _plms(); p.hist = None; out.append((p, 0, 0, "must be given"))
    p = _plms(); p.update.step = None; out.append((p, 0, 0, "must be given"))
    p = _plms(); p.update.eps = 0x7000; out.append((p, 0, 0, "update.eps must be e_prime"))
    p = _plms(); p.update.cfg = 1; out.append((p, 0, 0, "update.cfg must be 0"))
    p = _plms(); p.update.noise = 0xa000; out.append((p, 0, 0, "update.noise must be NULL"))
    p = _plms(); p.update.n = 0; out.append((p, 0, 0, "bad update"))
    p = _plms(); p.cfg = 2; out.append((p, 0, 0, "cfg=2"))
    p = _plms(); p.scale = float("nan"); out.append((p, 0, 0, "scale is not finite"))
    p = _plms(); out.append((p, 10, 0, "step=10 outside"))
    p = _plms(); out.append((p, 1, 1, "Heun mode is step 0's"))
    return out


@pytest.mark.parametrize("case", range(len(_malformed())))
def test_plms_combine_checks_its_arguments_without_a_device(case):
    p, step, heun, msg = _malformed()[case]
    lib = L_.load()
    assert lib.mugd_plms_combine(C.byref(p), step, heun, None) == 1
    assert msg in lib.mugd_last_error().decode()


def test_sample_plms_needs_a_captured_plan_and_a_descriptor():
    lib = L_.load()
    assert lib.mugd_sample_plms(None, C.byref(_plms()), 0, 1, None) == 1
    assert "must be captured" in lib.mugd_last_error().decode()
    assert lib.mugd_plms_combine(None, 0, 0, None) == 1
    assert "null argument" in lib.mugd_last_error().decode()
