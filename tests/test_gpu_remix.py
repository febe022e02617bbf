"""Remixing an existing chart on the GPU.  ``timesteps=k`` DDIM and PLMS runs match the UNMODIFIED reference (goldens) and the device
loop equals the per-step loop bit for bit; the stochastic_encode kernel equals torch's CUDA expressions bit for bit and leaves the
generator where randn_like leaves it; decode with a scalar start equals the truncated ddim_sampling bit for bit; per-chart starts run
in one mugd_sample_join loop that equals a per-step host loop doing the same holds bit for bit; an encoded golden chart is remixed
at the headline shape within the config-2 tolerance of the live CPU oracle; malformed join arguments launch nothing."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import encoder_cases as ec  # noqa: E402
import golden_cases as gc  # noqa: E402
import remix_cases as rc  # noqa: E402
import remix_oracle as ro  # noqa: E402
from gpu_util import rel_err  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402
from mug_diffusion_b200.runtime import _ptr  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200, PLMSSampler  # noqa: E402
from oracle import mug_oracle as orc  # noqa: E402

_models = {}


def model_for(L, encoder=False):
    key = (L, encoder)
    if key not in _models:
        _models.clear()
        sd = synth.synthetic_state_dict(L)
        if encoder:
            sd = {**sd, **synth.synthetic_encoder_state_dict(seed=ec.ENCODER_SEED)}
        _models[key] = (MugDiffusionB200.from_state_dict(sd, z_length=L), sd)
    return _models[key]


def request(B, L, cfg, seed=1234):
    inp = synth.synthetic_inputs(B, L, seed=seed)
    kw = dict(w=[w.cuda() for w in inp["w"]], c=inp["c"].cuda())
    if cfg:
        kw.update(unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    return inp, kw


# ---- timesteps= against the reference and the per-step loop -----------------------------------------------------------------------
@pytest.mark.parametrize("name", list(rc.REMIX_CASES))
def test_truncated_runs_match_the_reference_and_the_per_step_loop(name, golden_dir):
    case = rc.REMIX_CASES[name]
    m, _ = model_for(case["L"])
    inp, kw = request(case["B"], case["L"], case["scale"] != 1.0)
    cls = DDIMSampler if case["sampler"] == "ddim" else PLMSSampler
    sampler = cls(m)
    sampler.make_schedule(case["S"], ddim_eta=0.0, verbose=False)
    run = sampler.ddim_sampling if cls is DDIMSampler else sampler.plms_sampling
    shape = (case["B"], 16, case["L"])
    out = [run(shape=shape, x_T=inp["x_T"].cuda(), timesteps=case["k"], log_every_t=rc.LOG_EVERY_T, callback=cb, **kw)
           for cb in (None, lambda i: None)]
    (z, inter), (z2, inter2) = out
    assert torch.equal(z, z2)
    for key in ("x_inter", "pred_x0"):
        assert len(inter[key]) == len(inter2[key]) and all(torch.equal(a, b) for a, b in zip(inter[key], inter2[key])), key
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    logits = m.model.decode(z)
    assert rel_err(z, g["z"]) < 1e-3 and rel_err(logits, g["logits"]) < 1e-3
    for key in ("x_inter", "pred_x0"):
        ref = rc.intermediates(g, key)
        assert len(inter[key]) == len(ref)
        for a, b in zip(inter[key], ref):
            assert rel_err(a, b) < 1e-3, key


def test_truncated_inpainting_and_eta_take_the_device_loop(monkeypatch):
    """mask / eta > 0 with timesteps= run from mugd_sample_staged as without it: no Session.eval per step, same bits as the per-step
    loop, the generator left in the same place"""
    from mug_diffusion_b200.runtime import Session
    L, B = 96, 2
    m, _ = model_for(L)
    inp, kw = request(B, L, True)
    x0, mask = synth.synthetic_inpainting(B, L)
    sampler = DDIMSampler(m)
    sampler.make_schedule(10, ddim_eta=1.0, verbose=False)
    calls = []
    orig = Session.eval
    monkeypatch.setattr(Session, "eval", lambda self, graph=True: (calls.append(1), orig(self, graph))[1])
    res = []
    for cb in (None, lambda i: None):
        torch.cuda.manual_seed(21)
        z, inter = sampler.ddim_sampling(shape=(B, 16, L), x_T=inp["x_T"].cuda(), timesteps=6, mask=mask.cuda(), x0=x0.cuda(),
                                         callback=cb, log_every_t=2, **kw)
        res.append((z, inter, torch.randn(4, device="cuda")))
        if cb is None:
            assert calls == []
    assert len(calls) == 5                                                       # timesteps=6: 5 steps
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][2], res[1][2])
    for key in ("x_inter", "pred_x0"):
        assert all(torch.equal(a, b) for a, b in zip(res[0][1][key], res[1][1][key]))


# ---- stochastic_encode --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("original", [False, True])
@pytest.mark.parametrize("given", [False, True])
def test_stochastic_encode_equals_the_torch_expressions(original, given):
    m, _ = model_for(96)
    sampler = DDIMSampler(m)
    sampler.make_schedule(50, verbose=False)
    B = 5
    x0 = torch.randn(B, 16, 96, device="cuda") * 3
    t = torch.tensor([0, 7, 25, 49, 13] if not original else [0, 1, 500, 999, 250], device="cuda")
    noise = torch.randn_like(x0) if given else None
    torch.cuda.manual_seed(8)
    got = sampler.stochastic_encode(x0, t, use_original_steps=original, noise=noise)
    after = torch.randn(4, device="cuda")
    torch.cuda.manual_seed(8)
    nz = noise if given else torch.randn_like(x0)
    want_after = torch.randn(4, device="cuda")
    if original:
        sa, s1m = m.sqrt_alphas_cumprod, m.sqrt_one_minus_alphas_cumprod
    else:
        sa = torch.sqrt(torch.as_tensor(sampler.ddim_alphas).cuda())
        s1m = torch.as_tensor(sampler.ddim_sqrt_one_minus_alphas).cuda()
    want = sa.gather(-1, t).reshape(B, 1, 1) * x0 + s1m.gather(-1, t).reshape(B, 1, 1) * nz
    assert torch.equal(got, want)
    assert torch.equal(after, want_after)


def test_stochastic_encode_entry_writes_nan_for_an_index_outside_the_table():
    """the host refuses such indices; the entry point itself never reads past the tables"""
    x0 = torch.ones(2, 16, 40, device="cuda")
    t = torch.tensor([3, 10], device="cuda")
    tab = torch.arange(10, dtype=torch.float32, device="cuda")
    out = torch.zeros_like(x0)
    d = L_.QEncode()
    d.x0, d.noise, d.t, d.sqrt_a, d.sqrt_1ma, d.out = _ptr(x0), _ptr(x0), _ptr(t), _ptr(tab), _ptr(tab), _ptr(out)
    d.B, d.C, d.L, d.n = 2, 16, 40, 10
    L_.check(L_.load().mugd_stochastic_encode(C.byref(d), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.equal(out[0], torch.full_like(out[0], 6.0)) and torch.isnan(out[1]).all()


# ---- decode -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [False, True])
def test_scalar_decode_equals_the_truncated_sampling(cfg):
    L, B, S = 96, 2, 10
    m, _ = model_for(L)
    inp, kw = request(B, L, cfg)
    sampler = DDIMSampler(m)
    sampler.make_schedule(S, verbose=False)
    n = len(sampler.ddim_timesteps)
    z0 = inp["x_T"].cuda()
    scale, uc = kw.get("unconditional_guidance_scale", 1.0), kw.get("unconditional_conditioning")
    for s in range(1, n):
        if ro.subset(S, s + 1).shape[0] != s:
            continue
        got = sampler.decode(z0, kw["c"], kw["w"], s, scale, uc)
        assert sampler.last_launches_per_step == m.engine.session((2 if cfg else 1) * B, L).plan.launches + 2
        want, _ = sampler.ddim_sampling(kw["w"], kw["c"], (B, 16, L), x_T=z0, timesteps=s + 1, unconditional_guidance_scale=scale,
                                        unconditional_conditioning=uc)
        assert torch.equal(got, want), s
    full, _ = sampler.ddim_sampling(kw["w"], kw["c"], (B, 16, L), x_T=z0, unconditional_guidance_scale=scale, unconditional_conditioning=uc)
    assert torch.equal(sampler.decode(z0, kw["c"], kw["w"], n, scale, uc), full)
    assert sampler.decode(z0, kw["c"], kw["w"], 0, scale, uc) is z0


def host_join_loop(sampler, z0, c, w, starts, scale, uc):
    """the per-chart decode as a per-step host loop: before each step, the rows of every chart that has not joined are set to its
    latent with transposes, then the evaluation and the DDIM tail run one by one"""
    eng = sampler.model.engine
    B, Cz, Lz = z0.shape
    m = max(starts)
    joins = [m - s for s in starts]
    x, cfg_on, sess, _ = sampler._load_request(w, c, (B, Cz, Lz), z0, scale, uc, sampler.ddim_timesteps[:m])
    pred = torch.empty(B * Lz, Cz, device="cuda")
    tail = sess.ddim_tail(B, m, cfg_on, scale, 1.0, _ptr(pred))
    for i in range(m):
        ops = OpList()
        for b in range(B):
            if i <= joins[b]:
                for h in ((0, B) if cfg_on else (0,)):
                    rows = sess.xin.r((h + b) * Lz, (h + b + 1) * Lz)
                    ops.transpose(_ptr(x[b]), rows.ptr, 0, rows.ld, 1, Cz, Lz, True)
        eng.run_ops(ops)
        sess.eval(graph=True)
        eng.run_ops(tail)
    z = sess.read_rows(sess.xin.r(0, B * Lz), B, Cz, Lz)
    for b, s in enumerate(starts):
        if s == 0:
            z[b] = x[b]
    return z


def join_device_loop(sampler, z0, c, w, starts, scale, uc):
    """the mugd_sample_join loop straight from the session (decode takes the plain loop when every start is equal)"""
    B, Cz, Lz = z0.shape
    m = max(starts)
    x, cfg_on, sess, _ = sampler._load_request(w, c, (B, Cz, Lz), z0, scale, uc, sampler.ddim_timesteps[:m])
    pred = torch.empty(B * Lz, Cz, device="cuda")
    tail = sess.ddim_tail(B, m, cfg_on, scale, 1.0, _ptr(pred))
    joins = torch.tensor([m - s for s in starts], dtype=torch.int32, device="cuda")
    sess.plan.launch_join(sess.join(B, cfg_on, _ptr(x), _ptr(joins)), tail, 0, m)
    return sess.read_rows(sess.xin.r(0, B * Lz), B, Cz, Lz)


@pytest.mark.parametrize("cfg", [False, True])
@pytest.mark.parametrize("B", [1, 4])
def test_join_device_loop_equals_the_per_step_host_loop(B, cfg):
    L, S = 96, 10
    m, _ = model_for(L)
    inp, kw = request(B, L, cfg)
    sampler = DDIMSampler(m)
    sampler.make_schedule(S, verbose=False)
    scale, uc = kw.get("unconditional_guidance_scale", 1.0), kw.get("unconditional_conditioning")
    z0 = inp["x_T"].cuda()
    starts = [7] if B == 1 else [0, 3, 10, 6]
    ref = host_join_loop(sampler, z0, kw["c"], kw["w"], starts, scale, uc)
    if B == 1:
        assert torch.equal(join_device_loop(sampler, z0, kw["c"], kw["w"], starts, scale, uc), ref)
        assert torch.equal(sampler.decode(z0, kw["c"], kw["w"], starts, scale, uc), ref)
        return
    got = sampler.decode(z0, kw["c"], kw["w"], starts, scale, uc)
    assert torch.equal(got, ref)
    assert sampler.last_launches_per_step == m.engine.session((2 if cfg else 1) * B, L).plan.launches + 3
    assert torch.equal(got[0], z0[0])
    # each chart against its own scalar run at B = 1 (another batch composition: the GEMM K-split may differ)
    worst = 0.0
    for b, s in enumerate(starts):
        if s == 0:
            continue
        one = sampler.decode(z0[b:b + 1], kw["c"][b:b + 1], [wi[b:b + 1] for wi in kw["w"]], s, scale,
                             None if uc is None else uc[b:b + 1])
        worst = max(worst, rel_err(got[b:b + 1], one))
    print(f"per-chart starts vs scalar runs (B={B}, cfg={cfg}): max rel err {worst:.2e}")
    assert worst <= 1e-5


def test_remix_an_encoded_chart_at_the_headline_shape_vs_the_live_oracle():
    """four copies of a golden chart -> encode_hit_objects -> mode() -> stochastic_encode at per-chart t_enc -> decode with
    t_start = [3, 5, 8, 10], S = 10, L = 512, CFG 5, against the CPU oracle fed the same noised latent"""
    L, B, S = 512, 4, 10
    m, sd = model_for(L, encoder=True)
    g = ec.golden_charts()
    x0 = m.model.encode_hit_objects([g["ddim_L512_B1_S50_cfg5"][0]] * B, g["frame_ms"]).mode()
    sampler = DDIMSampler(m)
    sampler.make_schedule(S, verbose=False)
    n = len(sampler.ddim_timesteps)
    starts = [3, 5, 8, 10]
    torch.cuda.manual_seed(31)
    z_enc = sampler.stochastic_encode(x0, torch.tensor([min(s, n - 1) for s in starts], device="cuda"))
    inp, kw = request(B, L, True, seed=404)
    z = sampler.decode(z_enc, kw["c"], kw["w"], starts, 5.0, kw["unconditional_conditioning"])
    logits = m.model.decode(z)
    with torch.no_grad():
        z_ref = ro.decode(sd, S, z_enc.cpu(), inp["c"], inp["w"], starts, scale=5.0, uc=inp["uc"])
        l_ref = orc.decoder_forward(sd, z_ref)
    ez, el = rel_err(z, z_ref), rel_err(logits, l_ref)
    print(f"remix at the headline shape: z {ez:.2e} logits {el:.2e}")
    assert ez < 1e-3 and el < 1e-3
    assert not torch.equal(z, z_enc)
    lines = m.model.decode_to_hit_objects(z, g["frame_ms"])
    assert len(lines) == B


# ---- malformed join arguments -------------------------------------------------------------------------------------------------
def test_sample_join_rejects_malformed_arguments_before_any_launch():
    L, B = 96, 2
    m, _ = model_for(L)
    inp, kw = request(B, L, False)
    sampler = DDIMSampler(m)
    sampler.make_schedule(4, verbose=False)
    z0 = inp["x_T"].cuda()
    sampler.decode(z0, kw["c"], kw["w"], [1, 2])                                  # captures the B = 2 plan
    sess = m.engine.session(B, L)
    lib = L_.load()
    pred = torch.zeros(B * L * 16, device="cuda")
    joins = torch.zeros(B, dtype=torch.int32, device="cuda")

    def good():
        tail = sess.ddim_tail(B, 4, False, 1.0, 1.0, _ptr(pred))
        return sess.join(B, False, _ptr(z0), _ptr(joins)), tail

    cases = []
    j, t = good(); j.x_latent = None; cases.append((j, t, 0, 1, "x, x_latent and join must be given"))
    j, t = good(); j.join = None; cases.append((j, t, 0, 1, "x, x_latent and join must be given"))
    j, t = good(); j.B = 0; cases.append((j, t, 0, 1, "bad shape"))
    j, t = good(); j.B = 3; cases.append((j, t, 0, 1, "the join B*C*L"))
    j, t = good(); j.x = _ptr(pred); cases.append((j, t, 0, 1, "updates other rows"))
    j, t = good(); j.x_dup = _ptr(pred); cases.append((j, t, 0, 1, "updates other rows"))
    j, t = good(); t.ops[0].u.ddim.step = None; cases.append((j, t, 0, 1, "no device step counter"))
    j, t = good(); t.ops = t.ops[1:]; cases.append((j, t, 0, 1, "no DDIM update"))
    j, t = good(); t.ops = [t.ops[0], t.ops[0], t.ops[1]]; cases.append((j, t, 0, 1, "more than one DDIM update"))
    j, t = good(); cases.append((j, t, 2, 3, "outside the S=4 steps"))
    j, t = good(); cases.append((j, t, -1, 1, "outside the S=4 steps"))
    before, step0 = sess.read_rows(sess.xin.r(0, B * L), B, 16, L), sess.step.clone()
    for j, t, first, n, msg in cases:
        m.engine.attach_workspace(t)
        rc_ = lib.mugd_sample_join(sess.plan.handle, C.byref(j), t.array(), len(t.ops), first, n,
                                   torch.cuda.current_stream().cuda_stream)
        assert rc_ == 1 and msg in lib.mugd_last_error().decode(), msg
    torch.cuda.synchronize()
    assert torch.equal(sess.read_rows(sess.xin.r(0, B * L), B, 16, L), before) and torch.equal(sess.step, step0)
