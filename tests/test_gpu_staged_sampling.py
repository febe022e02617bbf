"""Inpainting and eta > 0 requests in the device loop (mugd_sample_staged): the result equals the per-step loop bit for bit -- the
final z, every recorded intermediate and the CUDA generator afterwards -- and a host without Python runs such a request from a bundle.
The per-step loop is forced with a callback; it is the referee."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import encoder_cases as ec  # noqa: E402
from gpu_util import rel_err  # noqa: E402
from mug_diffusion_b200 import sampler as sampler_mod  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.runtime import Plan, Session  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_DIR = os.path.join(ROOT, "examples", "host_c")

_models = {}


def model_for(L, encoder=False):
    key = (L, encoder)
    if key not in _models:
        _models.clear()
        sd = synth.synthetic_state_dict(L)
        if encoder:
            sd = {**sd, **synth.synthetic_encoder_state_dict(seed=ec.ENCODER_SEED)}
        _models[key] = MugDiffusionB200.from_state_dict(sd, z_length=L)
    return _models[key]


def make_mask(kind, B, L):
    shape, soft = kind
    dims = {"B16L": (B, 16, L), "11L": (1, 1, L), "B1L": (B, 1, L)}[shape]
    m = torch.zeros(dims)
    m[..., :L // 2] = 1.0
    if soft:
        m[..., L // 2:L // 2 + L // 8] = 0.5
        if dims[0] == B and B > 1:
            m[1, ..., L // 4:L // 2] = 0.25
    return m.cuda()


def both_paths(sampler, seed, **kw):
    """(z, intermediates, generator probe) of the device loop, then of the per-step loop, from the same seed"""
    out = []
    for cb in (None, lambda i: None):
        torch.cuda.manual_seed(seed)
        z, inter = sampler.sample(callback=cb, **kw)
        out.append((z, inter, torch.randn(4, device="cuda")))
    return out


def assert_same(dev, ref):
    (z1, i1, g1), (z2, i2, g2) = dev, ref
    assert torch.equal(z1, z2)
    for key in ("x_inter", "pred_x0"):
        assert len(i1[key]) == len(i2[key])
        for a, b in zip(i1[key], i2[key]):
            assert torch.equal(a, b), key
    assert torch.equal(g1, g2)


# (mask shape or None, soft, eta, noise_dropout, CFG, log_every_t, table cap in steps or None, match_reference_rng)
CASES = [
    (("B16L", False), 0.0, 0.0, True, 100, None, False),
    (("B16L", True), 1.0, 0.0, True, 2, None, False),
    (("B16L", True), 1.0, 0.25, False, 2, 2, False),
    (("11L", True), 1.0, 0.25, False, 100, 2, False),
    (("11L", False), 0.0, 0.25, True, 100, 2, False),
    (("B1L", False), 1.0, 0.25, True, 2, 2, False),
    (("B1L", True), 0.0, 0.0, False, 2, None, False),
    (("B16L", False), 0.0, 0.0, True, 2, None, True),
    (None, 1.0, 0.0, True, 100, None, False),
    (None, 1.0, 0.25, False, 2, 2, False),
    (None, 0.0, 0.25, True, 2, None, True),
]


@pytest.mark.parametrize("mask_kind,eta,dropout,cfg,log_every_t,cap,match_rng", CASES)
def test_device_loop_equals_the_per_step_loop(mask_kind, eta, dropout, cfg, log_every_t, cap, match_rng, monkeypatch):
    L, B, S = 96, 2, 6                                                  # S = 6 gives 7 DDIM steps
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    if cap is not None:
        monkeypatch.setattr(sampler_mod, "STAGE_TABLE_BYTES", cap * 4 * B * 16 * L)
    kw = dict(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
              eta=eta, shape=(16, L), temperature=0.8, noise_dropout=dropout, log_every_t=log_every_t, match_reference_rng=match_rng)
    if cfg:
        kw.update(unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    if mask_kind is not None:
        kw.update(mask=make_mask(mask_kind, B, L), x0=synth._gauss(synth._rng(31, "x0"), (B, 16, L)).cuda())
    sampler = DDIMSampler(m)
    dev, ref = both_paths(sampler, 77, **kw)
    assert_same(dev, ref)
    assert len(dev[1]["x_inter"]) == (5 if log_every_t == 2 else 3)
    if mask_kind is not None:
        z_plain, _ = sampler.sample(**{k: v for k, v in kw.items() if k not in ("mask", "x0")})
        assert rel_err(z_plain, dev[0]) > 1e-2                          # the mask really steered the trajectory


def test_device_loop_is_taken(monkeypatch):
    """no Session.eval per step: the request runs from mugd_sample_staged calls, one stage kernel + the two tail ops per step"""
    L, B = 96, 2
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    calls = []
    orig = Session.eval
    monkeypatch.setattr(Session, "eval", lambda self, graph=True: (calls.append(1), orig(self, graph))[1])
    sampler = DDIMSampler(m)
    sampler.sample(S=6, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), eta=1.0,
                   shape=(16, L), mask=make_mask(("B1L", True), B, L), x0=torch.zeros(B, 16, L, device="cuda"),
                   unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    assert calls == []
    sess = m.engine.session(2 * B, L, per_sample_t=False)
    assert sampler.last_launches_per_step == sess.plan.launches + 3
    sampler.sample(S=6, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), eta=1.0,
                   shape=(16, L), callback=lambda i: None, unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    assert len(calls) == 7                                              # the per-step loop, for comparison


def test_inpainting_an_encoded_chart_at_the_headline_shape():
    """keep the first half of four real charts (encode_hit_objects -> mode()), L = 512, B = 4, CFG 5, 20 steps: both loops give the
    same bits"""
    L, B, S = 512, 4, 20
    m = model_for(L, encoder=True)
    g = ec.golden_charts()
    charts = (g["ddim_L512_B1_S50_cfg5"] + g["ddim_L96_B2_S10_cfg5"] + g["synthetic"])[:B]
    x0 = m.model.encode_hit_objects(charts, g["frame_ms"]).mode()
    assert x0.shape == (B, 16, L)
    mask = torch.zeros(B, 1, L, device="cuda")
    mask[:, :, :L // 2] = 1.0
    inp = synth.synthetic_inputs(B, L, seed=77)
    kw = dict(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), eta=0.0,
              shape=(16, L), unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda(), mask=mask, x0=x0)
    dev, ref = both_paths(DDIMSampler(m), 5, **kw)
    assert_same(dev, ref)


def test_sample_staged_rejects_malformed_arguments_before_any_launch():
    L, B = 96, 2
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    DDIMSampler(m).sample(S=2, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
                          shape=(16, L))                                # captures the B = 2 evaluation plan
    eng = m.engine
    sess = eng.session(B, L, per_sample_t=False)
    noise_rows = torch.zeros(B * L * 16, device="cuda")
    tail = sess.ddim_tail(B, 2, False, 1.0, 1.0, 0, noise_rows.data_ptr())
    x0, mask = torch.zeros(B, 16, L, device="cuda"), torch.ones(B, 16, L, device="cuda")
    qn, nz = torch.zeros(2, B, 16, L, device="cuda"), torch.zeros(2, B, 16, L, device="cuda")
    coef = np.ones((2, 2), dtype=np.float32)

    def good():
        s = sess.ddim_stage(B, False, noise_rows.data_ptr())
        s.x0, s.mask, s.q_noise, s.q_coef, s.noise = x0.data_ptr(), mask.data_ptr(), qn.data_ptr(), coef.ctypes.data, nz.data_ptr()
        return s

    def call(plan, stage, n_steps=2):
        return eng.lib.mugd_sample_staged(plan.handle, C.byref(stage) if stage is not None else None, tail.array(), len(tail.ops),
                                          n_steps, torch.cuda.current_stream().cuda_stream)

    eng.attach_workspace(tail)
    before = sess.read_rows(sess.xin.r(0, B * L), B, 16, L)
    step0 = sess.step.clone()
    cases = []
    s = good(); s.x = None; cases.append((sess.plan, s, 2, "stage.x is NULL"))
    s = good(); s.L = L - 1; cases.append((sess.plan, s, 2, "updates n="))
    s = good(); s.x = s.x + 4; cases.append((sess.plan, s, 2, "other rows"))
    s = good(); s.x0 = s.mask = s.q_noise = None; cases.append((sess.plan, s, 2, "q_coef given without a q-noise table"))
    s = good(); s.noise_rows = None; cases.append((sess.plan, s, 2, "noise and noise_rows go together"))
    coef_nan = np.array([[1.0, np.nan], [1.0, 1.0]], dtype=np.float32)
    s = good(); s.q_coef = coef_nan.ctypes.data; cases.append((sess.plan, s, 2, "not finite"))
    cases.append((sess.plan, good(), -1, "n_steps=-1"))
    cases.append((sess.plan, None, 2, "null stage"))
    cases.append((Plan(eng, tail), good(), 2, "must be captured"))
    for plan, stage, n, msg in cases:
        assert call(plan, stage, n) == 1, msg
        assert msg in eng.lib.mugd_last_error().decode()
    torch.cuda.synchronize()
    assert torch.equal(sess.read_rows(sess.xin.r(0, B * L), B, 16, L), before) and torch.equal(sess.step, step0)
    assert call(sess.plan, good(), 0) == 0                              # zero steps: valid, nothing runs
    torch.cuda.synchronize()
    assert torch.equal(sess.read_rows(sess.xin.r(0, B * L), B, 16, L), before)


def test_c_host_runs_an_inpainting_eta1_request(tmp_path):
    """bundle --inpaint --eta 1: the Python run of the bundle's plans equals sampler.sample with the same seed, and the C host reproduces
    z and the logits from one mugd_sample_staged call"""
    from mug_diffusion_b200.bundle import export_bundle
    L, B, S = 96, 2, 10
    m = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    x0, mask = synth.synthetic_inpainting(B, L)
    out = str(tmp_path / "bundle")
    torch.cuda.manual_seed(3)
    res = export_bundle(m, inp, S, 5.0, out, eta=1.0, inpaint=(x0, mask))
    torch.cuda.manual_seed(3)
    z, _ = DDIMSampler(m).sample(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False,
                                 x_T=inp["x_T"].cuda(), eta=1.0, shape=(16, L), mask=mask.cuda(), x0=x0.cuda(),
                                 unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    logits = m.model.decode(z)
    assert rel_err(res["z"], z) < 1e-5
    assert rel_err(res["logits"], logits) < 1e-5
    manifest = open(os.path.join(out, "manifest.txt")).read()
    assert "staged eval.plan tail.plan 10 stage_coef.bin" in manifest and "sample eval.plan" not in manifest
    _models.clear()
    del m
    torch.cuda.empty_cache()
    subprocess.run(["make", "-C", HOST_DIR], check=True, capture_output=True)
    r = subprocess.run([os.path.join(HOST_DIR, "sample_host"), out], capture_output=True, text=True, timeout=600)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count(" OK") == 2 and "sampled 10 DDIM steps" in r.stdout and "staged: inpainting" in r.stdout
