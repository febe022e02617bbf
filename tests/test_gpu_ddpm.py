"""DDPMSampler on the GPU.  The update kernel equals torch's CUDA expressions of diffusion.py:260-277 bit for bit at every timestep;
the device loop (mugd_sample_ddpm) equals the per-step loop (forced with a callback) bit for bit: z, every recorded intermediate and
the CUDA generator afterwards.  Trajectories match the UNMODIFIED reference (goldens, fed the reference's own CPU noise) and the
oracle fed the GPU's noise within DESIGN §2's DDPM tolerances."""
import ctypes as C
import itertools
import os
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

import ddpm_cases as dc  # noqa: E402
import golden_cases as gc  # noqa: E402
from ddpm_oracle import ddpm_sample  # noqa: E402
from gpu_util import ncl, nlc, rel_err  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import sampler as sampler_mod  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.config import ModelConfig  # noqa: E402
from mug_diffusion_b200.runtime import Session, _ptr  # noqa: E402
from mug_diffusion_b200.sampler import DDPMSampler, MugDiffusionB200, register_schedule  # noqa: E402

_models = {}


def model_for(L, T):
    if (L, T) not in _models:
        _models.clear()
        sd = synth.synthetic_state_dict(L)
        _models[(L, T)] = (MugDiffusionB200.from_state_dict(sd, cfg=ModelConfig(timesteps=T), z_length=L), sd)
    return _models[(L, T)]


def request(B, L, cfg, **kw):
    inp = synth.synthetic_inputs(B, L)
    out = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), shape=(16, L))
    if cfg:
        out.update(unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    out.update(kw)
    return out


def both_loops(sampler, seed, **kw):
    out = []
    for cb in (None, lambda i: None):
        torch.cuda.manual_seed(seed)
        z, inter = sampler.sample(callback=cb, **kw)
        out.append((z, inter, torch.randn(4, device="cuda")))
    return out


def assert_same_runs(runs, n_logged):
    (z1, i1, g1), (z2, i2, g2) = runs
    assert torch.equal(z1, z2)
    for key in ("x_inter", "pred_x0"):
        assert len(i1[key]) == len(i2[key]) == n_logged + 1
        for a, b in zip(i1[key], i2[key]):
            assert torch.equal(a, b), key
    assert torch.equal(g1, g2)


MATRIX = list(itertools.product((1000, 50, 2), (False, True), (1, 4), (1, 7, 100)))


@pytest.mark.parametrize("T,cfg,B,log_every_t", MATRIX)
def test_device_loop_equals_the_per_step_loop(T, cfg, B, log_every_t):
    L = 96
    m, _ = model_for(L, T)
    kw = request(B, L, cfg, log_every_t=log_every_t)
    sampler = DDPMSampler(m)
    runs = both_loops(sampler, 11, **kw)
    assert_same_runs(runs, len(dc.logged_steps(T, log_every_t)))
    # one randn(shape) per step (x_T was given), as the reference's noise_like
    torch.cuda.manual_seed(11)
    for _ in range(T):
        torch.randn(B, 16, L, device="cuda")
    assert torch.equal(torch.randn(4, device="cuda"), runs[0][2])
    z = runs[0][0]
    assert torch.isfinite(z).all() and not torch.equal(z, kw["x_T"])


def test_split_stretches_and_drawn_x_T(monkeypatch):
    """noise tables capped at 3 steps (stretches of 7 split into 3 + 3 + 1), x_T drawn by the sampler: still the per-step loop's bits
    and generator state (x_T, then one draw per step)"""
    L, B, T = 96, 2, 50
    m, _ = model_for(L, T)
    monkeypatch.setattr(sampler_mod, "STAGE_TABLE_BYTES", 3 * 4 * B * 16 * L + 5)
    kw = request(B, L, True, log_every_t=7)
    kw.pop("x_T")
    runs = both_loops(DDPMSampler(m), 5, **kw)
    assert_same_runs(runs, len(dc.logged_steps(T, 7)))
    torch.cuda.manual_seed(5)
    assert torch.equal(torch.randn(B, 16, L, device="cuda"), runs[0][1]["x_inter"][0])
    for _ in range(T):
        torch.randn(B, 16, L, device="cuda")
    assert torch.equal(torch.randn(4, device="cuda"), runs[0][2])


def _schedule_holder(T):
    """the model attributes ddpm_coef_table / predict_start_from_noise / q_posterior read, on the device"""
    ns = types.SimpleNamespace(num_timesteps=T, device=torch.device("cuda"), _ddpm_coef=None)
    for k, v in register_schedule(T).items():
        setattr(ns, k, v.cuda())
    return ns


@pytest.mark.parametrize("cfg,clip", list(itertools.product((False, True), (True, False))))
def test_update_kernel_equals_the_torch_expressions(cfg, clip):
    """every timestep of the shipped schedule (0, 1 and T-1 included), x_recon well beyond +-10, a NaN and an inf in eps"""
    T, B, L, scale = 1000, 2, 40, 5.0
    ns = _schedule_holder(T)
    coef = MugDiffusionB200.ddpm_coef_table(ns)
    g = torch.Generator(device="cuda").manual_seed(3)
    x_ncl = torch.randn(B, 16, L, device="cuda", generator=g) * 30
    eps_ncl = torch.randn((2 if cfg else 1) * B, 16, L, device="cuda", generator=g) * 4
    eps_ncl[0, 3, 5] = float("nan")
    eps_ncl[-1, 7, 9] = float("inf")
    noise = torch.randn(B, 16, L, device="cuda", generator=g)
    x, x_dup, pred = torch.empty(B * L, 16, device="cuda"), torch.empty(B * L, 16, device="cuda"), torch.empty(B * L, 16, device="cuda")
    eps = nlc(eps_ncl)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    d = L_.Ddpm()
    d.x, d.x_dup, d.eps, d.pred_x0, d.noise, d.coef, d.step = _ptr(x), _ptr(x_dup) if cfg else None, _ptr(eps), _ptr(pred), \
        _ptr(noise), _ptr(coef), _ptr(step)
    d.T, d.B, d.C, d.L, d.cfg, d.scale, d.clip = T, B, 16, L, int(cfg), scale, int(clip)
    lib = L_.load()
    stream = torch.cuda.current_stream().cuda_stream
    if cfg:
        e_u, e_c = eps_ncl.chunk(2)
        e = e_u + scale * (e_c - e_u)                                             # ddim.py:175
    else:
        e = eps_ncl
    clamped = 0
    for t in range(T):
        x.copy_(nlc(x_ncl))
        step.fill_(T - 1 - t)
        L_.check(lib.mugd_ddpm_update(C.byref(d), stream), "mugd_ddpm_update")
        tt = torch.full((B,), t, device="cuda", dtype=torch.long)
        x_recon = MugDiffusionB200.predict_start_from_noise(ns, x_ncl, tt, e)      # diffusion.py:261
        if clip:
            clamped += int((x_recon.abs() > 10).sum())
            x_recon.clamp_(-10., 10.)                                             # :266-267
        model_mean, _, model_log_variance = MugDiffusionB200.q_posterior(ns, x_recon, x_ncl, tt)   # :268-273
        nonzero_mask = (1 - (tt == 0).float()).reshape(B, 1, 1)
        want = model_mean + nonzero_mask * (0.5 * model_log_variance).exp() * noise            # :276-277
        got, got_pred = ncl(x, B), ncl(pred, B)
        assert torch.equal(got.isnan(), want.isnan()) and int(want.isnan().sum()) >= 1, t
        assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(want)), t
        assert torch.equal(torch.nan_to_num(got_pred), torch.nan_to_num(x_recon)), t
        if cfg:
            assert torch.equal(x_dup.isnan(), x.isnan()) and torch.equal(torch.nan_to_num(x_dup), torch.nan_to_num(x)), t
    assert not clip or clamped > 0


@pytest.mark.parametrize("name", list(dc.DDPM_CASES))
def test_device_loop_against_the_reference_goldens(name, golden_dir):
    """the golden's own CPU noise in a noise table, run by mugd_sample_ddpm through Session and lib one logged stretch per call"""
    case = dc.DDPM_CASES[name]
    L, B, T, every = case["L"], case["B"], case["T"], case["log_every_t"]
    m, _ = model_for(L, T)
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    x_T, noise = dc.cpu_noise(case["seed"], (B, 16, L), T)
    assert torch.equal(x_T, g["x_T"])
    inp = synth.synthetic_inputs(B, L)
    table = torch.stack(noise).cuda()
    coef = m.ddpm_coef_table()
    pred = torch.empty(B * L, 16, device="cuda")
    with m.engine.lock:
        sess: Session = m.engine.session(B, L, per_sample_t=False)
        sess.set_timestep_table(list(reversed(range(T))))
        sess.set_context(inp["c"].cuda())
        sess.set_audio([w.cuda() for w in inp["w"]])
        sess.load_x(x_T.cuda(), dup=False)
        sess.set_step(0)
        d = sess.ddpm(B, T, False, 1.0, True, _ptr(pred), _ptr(table), coef)
        logged, i = [], 0
        for t_log in dc.logged_steps(T, every):
            j = T - 1 - t_log
            d.noise = _ptr(table[i])
            sess.plan.launch_ddpm(d, i, j - i + 1)
            logged.append(sess.read_rows(sess.xin.r(0, B * L), B, 16, L))
            i = j + 1
        assert i == T
    z = logged[-1]
    logits = m.model.decode(z)
    errs = [rel_err(a, g[f"x_inter_{k}"]) for k, a in enumerate(logged)]
    print(f"{name}: rel err z {rel_err(z, g['z']):.2e} logits {rel_err(logits, g['logits']):.2e} logged x max {max(errs):.2e}")
    assert rel_err(z, g["z"]) < 1e-3
    assert rel_err(logits, g["logits"]) < 1e-3
    assert max(errs) < 1e-3


def test_against_the_oracle_at_the_config2_shape():
    """B = 4, L = 512, CFG 5, T = 50 through DDPMSampler; the oracle is fed the noise the CUDA generator gave the sampler"""
    L, B, T = 512, 4, 50
    m, sd = model_for(L, T)
    inp = synth.synthetic_inputs(B, L)
    torch.cuda.manual_seed(21)
    z, _ = DDPMSampler(m).sample(**request(B, L, True))
    torch.cuda.manual_seed(21)
    noise = [torch.randn(B, 16, L, device="cuda").cpu() for _ in range(T)]
    with torch.no_grad():
        z_ref, _ = ddpm_sample(sd, T, inp["c"], inp["w"], x_T=inp["x_T"], noise_seq=noise, scale=5.0, uc=inp["uc"], log_every_t=T)
    print(f"config2 T=50: rel err z {rel_err(z, z_ref):.2e}")
    assert rel_err(z, z_ref) < 1e-3


def test_device_loop_is_taken_and_checks_its_step_range(monkeypatch):
    """no Session.eval per step: mugd_sample_ddpm calls, DDIM's launches per step (the plan's + 2); a step range outside the request
    is refused before any launch"""
    L, B, T = 96, 2, 50
    m, _ = model_for(L, T)
    calls = []
    orig = Session.eval
    monkeypatch.setattr(Session, "eval", lambda self, graph=True: (calls.append(1), orig(self, graph))[1])
    sampler = DDPMSampler(m)
    kw = request(B, L, True)
    sampler.sample(**kw)
    assert calls == []
    sess = m.engine.session(2 * B, L, per_sample_t=False)
    assert sampler.last_launches_per_step == sess.plan.launches + 2
    sampler.sample(img_callback=lambda p, i: None, **kw)
    assert len(calls) == T
    table = torch.zeros(1, B, 16, L, device="cuda")
    pred = torch.zeros(B * L, 16, device="cuda")
    d = sess.ddpm(B, T, True, 5.0, True, _ptr(pred), _ptr(table), m.ddpm_coef_table())
    before, step0 = sess.read_rows(sess.xin.r(0, B * L), B, 16, L), sess.step.clone()
    for first, n in ((0, T + 1), (T, 1), (-1, 1), (2, -1)):
        with pytest.raises(L_.MugdError, match=f"outside the T={T} steps"):
            sess.plan.launch_ddpm(d, first, n)
    torch.cuda.synchronize()
    assert torch.equal(sess.read_rows(sess.xin.r(0, B * L), B, 16, L), before) and torch.equal(sess.step, step0)
