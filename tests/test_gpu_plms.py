"""PLMSSampler on the GPU.  The device loop (mugd_sample_plms) equals the per-step loop (forced with a callback) bit for bit: z, every
recorded intermediate and the CUDA generator afterwards, with call boundaries inside the Heun step and the history warm-up.  The
combine kernel equals the torch expressions of plms.py bit for bit.  Trajectories match the UNMODIFIED reference (goldens) and the
oracle within DESIGN §2's 10-step tolerance; inpainting through the per-step loop matches the oracle fed the same noise."""
import ctypes as C
import itertools
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

import golden_cases as gc  # noqa: E402
import plms_cases as pc  # noqa: E402
from gpu_util import rel_err  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.runtime import Session  # noqa: E402
from mug_diffusion_b200.sampler import MugDiffusionB200, PLMSSampler  # noqa: E402
from oracle import mug_oracle as orc  # noqa: E402
from plms_oracle import plms_sample  # noqa: E402

_models = {}


def model_for(L):
    if L not in _models:
        _models.clear()
        _models[L] = (MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L), synth.synthetic_state_dict(L))
    return _models[L]


def request(B, L, S, cfg, **kw):
    inp = synth.synthetic_inputs(B, L)
    out = dict(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
               shape=(16, L))
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


# S = 3 is refused (its schedule reaches timestep 1000); S = 6 runs 7 steps
MATRIX = list(itertools.product((1, 2, 4, 6, 10), (False, True), (1, 4), (1, 3, 100)))


@pytest.mark.parametrize("S,cfg,B,log_every_t", MATRIX)
def test_device_loop_equals_the_per_step_loop(S, cfg, B, log_every_t):
    L = 96
    m, _ = model_for(L)
    kw = request(B, L, S, cfg, log_every_t=log_every_t, match_reference_rng=True, noise_dropout=0.25 if B == 4 else 0.0)
    sampler = PLMSSampler(m)
    (z1, i1, g1), (z2, i2, g2) = both_loops(sampler, 11, **kw)
    assert torch.equal(z1, z2)
    total = len(sampler.ddim_timesteps)
    for key in ("x_inter", "pred_x0"):
        assert len(i1[key]) == len(i2[key]) == pc.n_logged(S, log_every_t)
        for a, b in zip(i1[key], i2[key]):
            assert torch.equal(a, b), key
    assert torch.equal(g1, g2)
    # match_reference_rng drew 1 + total step noises (twice at step 0), with the dropout masks
    torch.cuda.manual_seed(11)
    for _ in range(total + 1):
        n = torch.randn(B, 16, L, device="cuda")
        if B == 4:
            torch.nn.functional.dropout(n, p=0.25)
    assert torch.equal(torch.randn(4, device="cuda"), g1)
    assert torch.isfinite(z1).all() and not torch.equal(z1, kw["x_T"])


def _combine(p, step, heun):
    L_.check(L_.load().mugd_plms_combine(C.byref(p), step, heun, torch.cuda.current_stream().cuda_stream), "mugd_plms_combine")


@pytest.mark.parametrize("cfg", [False, True])
def test_combine_kernel_equals_the_torch_expressions(cfg):
    """each Adams-Bashforth order (steps 1, 2, 3 and 4..6 for the ring's wrap), Heun mode, CFG on and off: bit for bit"""
    n, S, scale = 3 * 16 * 257, 8, 5.0
    g = torch.Generator(device="cuda").manual_seed(5)
    work = torch.full((5, n), float("nan"), device="cuda")
    eps = torch.empty((2 if cfg else 1) * n, device="cuda")
    dummy = torch.zeros(n, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    p = L_.Plms()
    u = p.update
    u.x, u.x_dup, u.pred_x0, u.coef, u.step = dummy.data_ptr(), None, None, dummy.data_ptr(), step.data_ptr()
    u.eps, u.noise, u.S, u.n, u.cfg = work[0].data_ptr(), None, S, n, 0
    p.eps, p.e_prime, p.hist, p.x_stash = eps.data_ptr(), work[0].data_ptr(), work[1].data_ptr(), work[4].data_ptr()
    p.cfg, p.scale = int(cfg), scale

    def e_of_eps():
        if not cfg:
            return eps.clone()
        e_u, e_c = eps.view(2, n)
        return e_u + scale * (e_c - e_u)                                         # plms.py:186

    old_eps = []
    for k in range(S):
        eps.copy_(torch.randn(eps.shape, device="cuda", generator=g) * 3)
        e_t = e_of_eps()
        _combine(p, k, 0)
        if len(old_eps) == 0:
            want = e_t                                                           # the Euler half: e' = e_t
        elif len(old_eps) == 1:
            want = (3 * e_t - old_eps[-1]) / 2
        elif len(old_eps) == 2:
            want = (23 * e_t - 16 * old_eps[-1] + 5 * old_eps[-2]) / 12
        else:
            want = (55 * e_t - 59 * old_eps[-1] + 37 * old_eps[-2] - 9 * old_eps[-3]) / 24
        torch.cuda.synchronize()
        assert torch.equal(work[0], want), k
        assert torch.equal(work[1 + k % 3], e_t), k
        if k == 0:
            eps.copy_(torch.randn(eps.shape, device="cuda", generator=g) * 3)
            e_next = e_of_eps()
            _combine(p, 0, 1)
            torch.cuda.synchronize()
            assert torch.equal(work[0], (e_t + e_next) / 2)                      # :223
            assert torch.equal(work[1], e_t)                                     # Heun mode leaves the ring alone
        old_eps.append(e_t)
        if len(old_eps) >= 4:
            old_eps.pop(0)


@pytest.mark.parametrize("name", list(pc.PLMS_CASES))
def test_against_the_reference_goldens(name, golden_dir):
    case = pc.PLMS_CASES[name]
    m, _ = model_for(case["L"])
    kw = request(case["B"], case["L"], case["S"], case["scale"] != 1.0, log_every_t=pc.LOG_EVERY_T)
    z, inter = PLMSSampler(m).sample(**kw)
    logits = m.model.decode(z)
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    assert rel_err(z, g["z"]) < 1e-3
    assert rel_err(logits, g["logits"]) < 1e-3
    for key in ("x_inter", "pred_x0"):
        ref = pc.intermediates(g, key)
        assert len(inter[key]) == len(ref)
        for a, b in zip(inter[key], ref):
            assert rel_err(a, b) < 1e-3, key
    mine, ref = orc.notes_from_logits(logits.cpu()), orc.notes_from_logits(g["logits"])
    flips = mine != ref
    ref8 = torch.cat([g["logits"][:, 0:4], g["logits"][:, 8:12]], dim=1)
    assert bool((ref8[flips].abs() < 1e-3 * ref8.abs().max()).all())


def test_against_the_oracle_at_the_config2_shape():
    L, B, S = 512, 4, 10
    m, sd = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    z, _ = PLMSSampler(m).sample(**request(B, L, S, True))
    with torch.no_grad():
        z_ref, _ = plms_sample(sd, S, inp["c"], inp["w"], inp["x_T"], scale=5.0, uc=inp["uc"])
    assert rel_err(z, z_ref) < 1e-3


def test_inpainting_per_step_loop_against_the_oracle():
    """mask / x0 (plms.py:147-150) run the per-step loop; the oracle is fed the q_sample noise the CUDA generator gave it"""
    L, B, S = 96, 2, 10
    m, sd = model_for(L)
    inp = synth.synthetic_inputs(B, L)
    x0, mask = synth.synthetic_inpainting(B, L)
    sampler = PLMSSampler(m)
    torch.cuda.manual_seed(9)
    z, inter = sampler.sample(**request(B, L, S, True, mask=mask.cuda(), x0=x0.cuda()))
    total = len(sampler.ddim_timesteps)
    torch.cuda.manual_seed(9)
    q = [torch.randn(B, 16, L, device="cuda").cpu() for _ in range(total)]
    with torch.no_grad():
        z_ref, _ = plms_sample(sd, S, inp["c"], inp["w"], inp["x_T"], scale=5.0, uc=inp["uc"], mask=mask, x0=x0, q_noise_seq=q)
        z_plain, _ = plms_sample(sd, S, inp["c"], inp["w"], inp["x_T"], scale=5.0, uc=inp["uc"])
    assert rel_err(z, z_ref) < 2e-4
    assert rel_err(z_plain, z_ref) > 1e-2                                        # the mask steered the trajectory


def test_device_loop_is_taken_and_checks_its_step_range(monkeypatch):
    """no Session.eval per step: one mugd_sample_plms call per stretch, the plan's launches + 3 per step; a step range outside the
    request is refused before any launch"""
    L, B = 96, 2
    m, _ = model_for(L)
    calls = []
    orig = Session.eval
    monkeypatch.setattr(Session, "eval", lambda self, graph=True: (calls.append(1), orig(self, graph))[1])
    sampler = PLMSSampler(m)
    kw = request(B, L, 6, True)
    sampler.sample(**kw)
    assert calls == []
    sess = m.engine.session(2 * B, L, per_sample_t=False)
    assert sampler.last_launches_per_step == sess.plan.launches + 3
    sampler.sample(callback=lambda i: None, **kw)
    assert len(calls) == 8                                                      # 7 steps, step 0 evaluates twice
    work = torch.zeros(5, B * L * 16, device="cuda")
    pred = torch.zeros(B * L * 16, device="cuda")
    p = sess.plms(B, 7, True, 5.0, pred.data_ptr(), work)
    before, step0 = sess.read_rows(sess.xin.r(0, B * L), B, 16, L), sess.step.clone()
    for first, n in ((0, 8), (7, 1), (-1, 1), (2, -1)):
        with pytest.raises(L_.MugdError, match="outside the S=7 steps"):
            sess.plan.launch_plms(p, first, n)
    torch.cuda.synchronize()
    assert torch.equal(sess.read_rows(sess.xin.r(0, B * L), B, 16, L), before) and torch.equal(sess.step, step0)
