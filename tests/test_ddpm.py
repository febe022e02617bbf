"""DDPM sampler, CPU side: the oracle restatement equals the UNMODIFIED reference DDPM.log_beatmap (tests/golden/ddpm_*.npz), the host
schedule equals the reference's buffers bit for bit, requests the device path cannot take are refused before any GPU work, and
libmugd exports the DDPM entry points at ABI 13, checking their arguments before anything is launched."""
import ctypes as C
import gzip
import json
import os
import types

import numpy as np
import pytest
import torch

import ddpm_cases as dc
import golden_cases as gc
from ddpm_oracle import ddpm_sample, register_schedule as oracle_schedule
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.sampler import DDPMSampler, MugDiffusionB200, register_schedule
from oracle import mug_oracle as orc


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _golden(golden_dir, name):
    return gc.load_golden(os.path.join(golden_dir, name + ".npz"))


@pytest.mark.parametrize("name", list(dc.DDPM_CASES))
def test_oracle_equals_the_reference_ddpm(name, golden_dir):
    case = dc.DDPM_CASES[name]
    sd = synth.synthetic_state_dict(case["L"])
    inp = synth.synthetic_inputs(case["B"], case["L"])
    g = _golden(golden_dir, name)
    with torch.no_grad():
        z, inter = ddpm_sample(sd, case["T"], inp["c"], inp["w"], seed=case["seed"], z_length=case["L"],
                               log_every_t=case["log_every_t"])
        logits = orc.decoder_forward(sd, z)
    assert torch.equal(inter["x_inter"][0], g["x_T"])
    assert rel_err(z, g["z"]) <= 2e-5
    assert rel_err(logits, g["logits"]) <= 2e-5
    n = len(dc.logged_steps(case["T"], case["log_every_t"]))
    assert len(inter["x_inter"]) == n + 1
    for k in range(n):
        assert rel_err(inter["x_inter"][k + 1], g[f"x_inter_{k}"]) <= 2e-5, k
    assert not torch.equal(inter["x_inter"][1], inter["x_inter"][2])             # the trajectory moves


@pytest.mark.parametrize("name", list(dc.DDPM_CASES))
def test_register_schedule_equals_the_reference_buffers(name, golden_dir):
    """sampler.register_schedule (and the oracle's restatement) give the reference's float32 buffers bit for bit"""
    g = _golden(golden_dir, name)
    T = dc.DDPM_CASES[name]["T"]
    for sch in (register_schedule(T), oracle_schedule(T)):
        for key in dc.SCHEDULE_KEYS:
            assert sch[key].dtype == torch.float32 and torch.equal(sch[key], g["sched_" + key]), key


def test_register_schedule_v_posterior():
    """v_posterior mixes beta into the posterior variance (diffusion.py:166-167); the other tables do not depend on it"""
    a, b = register_schedule(1000, v_posterior=0.0), register_schedule(1000, v_posterior=0.3)
    assert torch.equal(b["posterior_variance"], oracle_schedule(1000, v_posterior=0.3)["posterior_variance"])
    assert not torch.equal(a["posterior_variance"], b["posterior_variance"])
    assert torch.equal(a["posterior_mean_coef1"], b["posterior_mean_coef1"])
    assert float(a["posterior_variance"][0]) == 0.0 and float(a["posterior_log_variance_clipped"][0]) == pytest.approx(np.log(1e-20))


def _cpu_sampler(L=96, T=1000):
    """a DDPMSampler over a stand-in model: enough for the checks that run before any GPU work"""
    s = DDPMSampler.__new__(DDPMSampler)
    s.model = types.SimpleNamespace(z_channels=16, z_length=L, num_timesteps=T, clip_denoised=True)
    s.ddpm_num_timesteps, s.device = T, torch.device("cpu")
    return s


def _request(B=2, L=96, **kw):
    inp = synth.synthetic_inputs(B, L)
    base = dict(c=inp["c"], w=inp["w"], batch_size=B, shape=(16, L), verbose=False, x_T=inp["x_T"],
                unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"])
    base.update(kw)
    return base


BAD = [
    (dict(S=50), ValueError, "runs all T=1000 steps"),
    (dict(S=True), ValueError, "runs all T=1000 steps"),
    (dict(mask=torch.ones(2, 1, 96)), ValueError, "no mask"),
    (dict(x0=torch.zeros(2, 16, 96)), ValueError, "no x0"),
    (dict(eta=1.0), ValueError, "no eta"),
    (dict(temperature=0.5), ValueError, "no temperature"),
    (dict(noise_dropout=0.1), ValueError, "no noise_dropout"),
    (dict(eta=False), ValueError, "no eta"),
    (dict(quantize_denoised=True), TypeError, "unexpected arguments"),
    (dict(c=None), TypeError, "needs the conditioning"),
    (dict(w=None), TypeError, "audio features"),
    (dict(clip_denoised=2), ValueError, "clip_denoised"),
    (dict(unconditional_guidance_scale=float("nan")), ValueError, "finite number"),
    (dict(batch_size=0), ValueError, "batch_size"),
    (dict(log_every_t=0), ValueError, "log_every_t"),
    (dict(shape=(16, 96, 1)), ValueError, "(channels, length)"),
    (dict(shape=(8, 96)), ValueError, "16 channels"),
    (dict(x_T=torch.zeros(2, 16, 64)), ValueError, "x_T has shape"),
    (dict(c=torch.zeros(3, 128, 21)), ValueError, "c must be"),
    (dict(unconditional_conditioning=torch.zeros(1, 128, 21)), ValueError, "unconditional_conditioning must be"),
]


@pytest.mark.parametrize("kw,exc,msg", BAD, ids=[f"bad{i}" for i in range(len(BAD))])
def test_sample_refuses_before_any_gpu_work(kw, exc, msg):
    with pytest.raises(exc, match=msg.replace("(", r"\(").replace(")", r"\)")):
        _cpu_sampler().sample(**_request(**kw))


@pytest.mark.parametrize("kw", [dict(), dict(S=1000, eta=0, temperature=1, noise_dropout=0., mask=None, x0=None),
                                dict(clip_denoised=False, unconditional_guidance_scale=1.0, log_every_t=7)])
def test_well_formed_requests_pass_the_checks(kw):
    """arguments that mean "not used" pass; the run then needs the engine, which this stand-in lacks"""
    with pytest.raises(AttributeError, match="engine"):
        _cpu_sampler().sample(**_request(**kw))


def _standin(**ddpm_attrs):
    from test_from_reference import _standin_ddpm
    with gzip.open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ddpm_surface.json.gz"), "rt") as f:
        m = _standin_ddpm(json.load(f))
    for k, v in ddpm_attrs.items():
        setattr(m, k, v)
    return m


def test_config_from_reference_reads_the_ddpm_settings():
    _, cfg = MugDiffusionB200.config_from_reference(_standin())
    assert (cfg.clip_denoised, cfg.v_posterior, cfg.parameterization) == (True, 0.0, "eps")
    _, cfg = MugDiffusionB200.config_from_reference(_standin(clip_denoised=False, v_posterior=0.25, parameterization="eps"))
    assert (cfg.clip_denoised, cfg.v_posterior, cfg.parameterization) == (False, 0.25, "eps")


@pytest.mark.parametrize("p", ["x0", "recon"])
def test_only_eps_models_are_built(p):
    with pytest.raises(L_.MugdError, match=f'parameterization "{p}"'):
        MugDiffusionB200.config_from_reference(_standin(parameterization=p))
    with pytest.raises(L_.MugdError, match=f'parameterization "{p}"'):
        MugDiffusionB200({}, ModelConfig(parameterization=p), z_length=96)


def test_library_exports_ddpm_at_abi_13():
    lib = L_.load()
    assert lib.mugd_abi_version() == L_.ABI_VERSION == 13
    for sym in ("mugd_sample_ddpm", "mugd_ddpm_update"):
        assert sym in L_.EXPORTED_SYMBOLS and hasattr(lib, sym)
    with open(os.path.join(os.path.dirname(L_.HERE), "include", "mugd.h")) as f:
        h = f.read()
    assert "int  mugd_sample_ddpm(mugd_plan* eval_plan, const mugd_ddpm* d, int32_t first_step, int32_t n_steps, void* stream);" in h
    assert "int  mugd_ddpm_update(const mugd_ddpm* d, void* stream);" in h
    assert C.sizeof(L_.Ddpm) == 7 * 8 + 8 * 4


def _ddpm(B=2, L=96, T=1000, cfg=1):
    """a well-formed descriptor over fake (never dereferenced) addresses"""
    d = L_.Ddpm()
    d.x, d.x_dup, d.eps, d.pred_x0, d.noise, d.coef, d.step = 0x1000, 0x2000 if cfg else None, 0x3000, 0x4000, 0x5000, 0x6000, 0x7000
    d.T, d.B, d.C, d.L, d.cfg, d.scale, d.clip = T, B, 16, L, cfg, 5.0, 1
    return d


def _malformed():
    out = []
    for f in ("x", "eps", "noise", "coef", "step"):
        d = _ddpm(); setattr(d, f, None); out.append((d, "must be given"))
    d = _ddpm(); d.B = 0; out.append((d, "bad shape"))
    d = _ddpm(); d.C = -16; out.append((d, "bad shape"))
    d = _ddpm(); d.B, d.L = 65536, 65536; out.append((d, "bad shape"))
    d = _ddpm(); d.B, d.L = 65536, 1; out.append((d, "too large for one launch"))
    d = _ddpm(); d.T = 0; out.append((d, "T=0 outside"))
    d = _ddpm(); d.T = 1001; out.append((d, "T=1001 outside"))
    d = _ddpm(); d.cfg = 2; out.append((d, "cfg=2"))
    d = _ddpm(); d.clip = -1; out.append((d, "clip=-1"))
    d = _ddpm(); d.scale = float("inf"); out.append((d, "scale is not finite"))
    d = _ddpm(); d.x_dup = None; out.append((d, "x_dup must be given exactly when cfg = 1"))
    d = _ddpm(cfg=0); d.x_dup = 0x2000; out.append((d, "x_dup must be given exactly when cfg = 1"))
    return out


@pytest.mark.parametrize("case", range(len(_malformed())))
def test_ddpm_update_checks_its_arguments_without_a_device(case):
    d, msg = _malformed()[case]
    lib = L_.load()
    assert lib.mugd_ddpm_update(C.byref(d), None) == 1
    assert msg in lib.mugd_last_error().decode()


def test_sample_ddpm_needs_a_captured_plan_and_a_descriptor():
    lib = L_.load()
    assert lib.mugd_sample_ddpm(None, C.byref(_ddpm()), 0, 1, None) == 1
    assert "must be captured" in lib.mugd_last_error().decode()
    assert lib.mugd_ddpm_update(None, None) == 1
    assert "null argument" in lib.mugd_last_error().decode()
