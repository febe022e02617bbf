"""Per-chart guidance scales on the GPU: the MUGD_OP_CFG_SCALES kernel against torch's eager expression; the guided-scales path at one
shared scale bit-identical to today's path for every sampler and flow; each chart of a mixed-scale request against the chart requested
alone at its scale (bit for bit with batch_invariant=True); device loop against per-step loop, graph reuse and ragged requests."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import sampler as sampler_mod  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.config import ModelConfig  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402
from mug_diffusion_b200.sampler import (DDIMSampler, DDPMSampler, DPMSolverSampler, MugDiffusionB200, PLMSSampler,  # noqa: E402
                                        UniPCSampler)

from gpu_util import OpRunner, rel_err  # noqa: E402

NAN = float("nan")
SCALES = [1.0, 3.0, 5.0, 7.5]
# chart b of a mixed-scale request vs the chart alone: the relative max-abs error bound of ragged requests (DESIGN §6b N17)
PIN = 2e-5


# ---- 1. the kernel ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def R():
    return OpRunner()


def _guided_ref(eu, ec, scales, L):
    """torch's eager eu + s * (ec - eu) per chart, ec where s == 1"""
    out = torch.empty_like(ec)
    for b, s in enumerate(scales):
        r = slice(b * L, (b + 1) * L)
        out[r] = ec[r] if s == 1.0 else eu[r] + torch.tensor(s, dtype=torch.float32, device="cuda") * (ec[r] - eu[r])
    return out


def _same(a, b):
    """equal bit for bit, NaN where NaN"""
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(0.0), b.nan_to_num(0.0))


# (B, L, C, ld, float offset of the rows): the plans' shapes (C = 16, dense), a padded ld, a C that is no multiple of 4 and rows off
# the 16-byte alignment (both on the one-element path)
KERNEL_SHAPES = [(1, 96, 16, 16, 0), (4, 96, 16, 16, 0), (4, 512, 16, 16, 0), (32, 512, 16, 16, 0), (3, 64, 16, 20, 0),
                 (2, 32, 13, 13, 0), (4, 96, 16, 16, 1), (5, 40, 7, 9, 3)]


@pytest.mark.parametrize("shape", KERNEL_SHAPES, ids=lambda s: "B{}-L{}-C{}-ld{}-off{}".format(*s))
def test_cfg_scales_kernel_is_torch_eager(R, shape):
    B, L, C, ld, off = shape
    torch.manual_seed(B * 31 + L + C)
    rows = B * L
    scales = [(1.0, 3.0, 5.0, 7.5, -2.0, 0.0)[b % 6] for b in range(B)]
    store = torch.randn(off + 2 * rows * ld + 4, device="cuda")
    eps = store[off:off + 2 * rows * ld].view(2 * rows, ld)
    eps[:, C:] = NAN                                                   # columns past C: never read
    eu, ec = eps[:rows, :C], eps[rows:, :C]
    eu[0, 0] = NAN                                                     # chart 0 (s = 1): not read; chart 1: propagates
    if B > 1:
        eu[L, 0] = NAN
        ec[L, 1] = NAN
    guard = 64
    out_buf = torch.full((2 * guard + rows * C + off,), -7777.0, device="cuda")
    out = out_buf[guard + off:guard + off + rows * C].view(rows, C)
    sdev = torch.tensor(scales, dtype=torch.float32, device="cuda")
    d = L_.CfgScales()
    d.eps, d.ld, d.out, d.scales, d.B, d.L, d.C = eps.data_ptr(), ld, out.data_ptr(), sdev.data_ptr(), B, L, C
    ops = OpList()
    ops.add(L_.OP_CFG_SCALES, d)
    R.run(ops)
    ref = _guided_ref(eu.contiguous(), ec.contiguous(), scales, L)
    assert _same(out, ref)
    assert torch.equal(out[:L], ec[:L]) and not torch.isnan(out[0, 0])           # s = 1: exactly e_c
    if B > 1:
        assert torch.isnan(out[L, 0]) and torch.isnan(out[L, 1])
    assert torch.all(out_buf[:guard + off] == -7777.0) and torch.all(out_buf[guard + off + rows * C:] == -7777.0)


def test_cfg_scales_refusals_on_the_device(R):
    eps = torch.zeros(2 * 96, 16, device="cuda")
    sdev = torch.ones(1, device="cuda")
    out = torch.empty(96, 16, device="cuda")
    for kw, msg in ((dict(ld=8), "bad shape"), (dict(out=eps.data_ptr() + 4 * 16), "overlaps"), (dict(scales=None), "must be given")):
        d = L_.CfgScales()
        d.eps, d.ld, d.out, d.scales, d.B, d.L, d.C = eps.data_ptr(), 16, out.data_ptr(), sdev.data_ptr(), 1, 96, 16
        for k, v in kw.items():
            setattr(d, k, v)
        op = L_.make_op(L_.OP_CFG_SCALES, d)
        assert R.lib.mugd_op_run(R.handle, C.byref(op), torch.cuda.current_stream().cuda_stream) == 1
        assert msg in R.lib.mugd_last_error().decode()


# ---- requests ---------------------------------------------------------------------------------------------------------------------
_models = {}


def model_for(L, T=1000, invariant=False):
    key = (L, T, invariant)
    if key not in _models:
        if len(_models) > 3:
            _models.clear()
        _models[key] = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), cfg=ModelConfig(timesteps=T), z_length=L,
                                                        batch_invariant=invariant)
    return _models[key]


def request(B, L, seed=77):
    inp = synth.synthetic_inputs(B, L, seed=seed)
    return dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, shape=(16, L), verbose=False,
                unconditional_conditioning=inp["uc"].cuda())


def one_chart(kw, b):
    out = dict(kw, c=kw["c"][b:b + 1], w=[w[b:b + 1] for w in kw["w"]], batch_size=1,
               unconditional_conditioning=kw["unconditional_conditioning"][b:b + 1])
    for k in ("mask", "x0", "x_T"):
        if k in kw:
            out[k] = kw[k][b:b + 1] if kw[k].shape[0] > 1 else kw[k]
    return out


def _cond(kw):
    return {k: v for k, v in kw.items() if k not in ("batch_size", "shape", "verbose")}


def _guided_key(m):
    return [k for k in m.engine.sessions if "guided" in k]


# ---- 2. the guided-scales path at one shared scale is today's path, bit for bit -----------------------------------------------------
def _inpaint_kw(B, L):
    g = torch.Generator(device="cuda").manual_seed(5)
    x0 = torch.randn(B, 16, L, device="cuda", generator=g)
    mask = torch.ones(B, 1, L, device="cuda")
    mask[:, :, L // 3:2 * L // 3] = 0.
    return dict(mask=mask, x0=x0)


def _ddim_decode(m, kw):
    s = DDIMSampler(m)
    s.make_schedule(10, verbose=False)
    xl = s.stochastic_encode(kw["x_T"], torch.tensor([9, 5, 2, 7]), seeds=40)
    return s.decode(xl, kw["c"], kw["w"], [9, 5, 2, 7], unconditional_guidance_scale=kw["unconditional_guidance_scale"],
                    unconditional_conditioning=kw["unconditional_conditioning"]), None


def _dpm_decode(m, kw):
    s = DPMSolverSampler(m)
    sched = s.make_dpm_schedule(8)
    xl = s.stochastic_encode(kw["x_T"], [8, 3, 6, 1], sched, seeds=41)
    return s.decode(xl, kw["c"], kw["w"], [8, 3, 6, 1], sched, unconditional_guidance_scale=kw["unconditional_guidance_scale"],
                    unconditional_conditioning=kw["unconditional_conditioning"]), None


def _dpm_invert(m, kw):
    s = DPMSolverSampler(m)
    z = s.invert(kw["x_T"], kw["c"], kw["w"], [6, 2, 4, 6], s.make_dpm_schedule(6), unconditional_guidance_scale=kw["unconditional_guidance_scale"],
                 unconditional_conditioning=kw["unconditional_conditioning"], verbose=False, log_every_t=2)
    return z, s.last_intermediates


def _unipc_invert(m, kw):
    s = UniPCSampler(m)
    z = s.invert(kw["x_T"], kw["c"], kw["w"], [5, 5, 2, 3], s.make_unipc_schedule(5), unconditional_guidance_scale=kw["unconditional_guidance_scale"],
                 unconditional_conditioning=kw["unconditional_conditioning"], verbose=False)
    return z, s.last_intermediates


PIN_RUNS = {
    "ddim_eta0": lambda m, kw: DDIMSampler(m).sample(S=10, log_every_t=3, **kw),
    "ddim_eta1": lambda m, kw: DDIMSampler(m).sample(S=10, eta=1.0, seeds=3, log_every_t=3, **kw),
    "plms": lambda m, kw: PLMSSampler(m).sample(S=10, log_every_t=3, **kw),
    "ddpm_T50": lambda m, kw: DDPMSampler(m).sample(seeds=4, log_every_t=10, **kw),
    "dpm2": lambda m, kw: DPMSolverSampler(m).sample(S=10, order=2, log_every_t=3, **kw),
    "unipc_bh2": lambda m, kw: UniPCSampler(m).sample(S=6, variant="bh2", log_every_t=2, **kw),
    "ddim_inpaint": lambda m, kw: DDIMSampler(m).sample(S=10, seeds=6, **_inpaint_kw(4, 96), **kw),
    "dpm_inpaint": lambda m, kw: DPMSolverSampler(m).inpaint(S=8, seeds=6, **_inpaint_kw(4, 96), **kw),
    "unipc_inpaint": lambda m, kw: UniPCSampler(m).inpaint(S=6, seeds=6, **_inpaint_kw(4, 96), **kw),
    "ddim_remix": _ddim_decode,
    "dpm_remix": _dpm_decode,
    "dpm_invert": _dpm_invert,
    "unipc_invert": _unipc_invert,
    "ddim_ragged": lambda m, kw: DDIMSampler(m).sample(S=10, seeds=8, z_lengths=[96, 64, 32, 96], **dict(kw, x_T=None)),
}


@pytest.mark.parametrize("name", sorted(PIN_RUNS))
def test_guided_path_at_one_scale_is_todays_path(monkeypatch, name):
    m = model_for(96, 50 if name == "ddpm_T50" else 1000)
    kw = dict(request(4, 96), unconditional_guidance_scale=5.0, x_T=torch.randn(4, 16, 96, device="cuda",
                                                                              generator=torch.Generator(device="cuda").manual_seed(9)))
    if name.endswith(("remix", "invert")):
        kw = _cond(kw)
    for k in _guided_key(m):
        del m.engine.sessions[k]
    z0, i0 = PIN_RUNS[name](m, kw)
    assert not _guided_key(m)
    monkeypatch.setattr(sampler_mod._DeviceLoopSampler, "force_per_chart_scales", True)
    z1, i1 = PIN_RUNS[name](m, kw)
    assert _guided_key(m), "the forced request ran on the guided session"
    assert torch.equal(z0, z1), name
    if i0 is not None:
        for k in ("x_inter", "pred_x0"):
            assert len(i0[k]) == len(i1[k]) and all(torch.equal(a, b) for a, b in zip(i0[k], i1[k])), k
    lens = [96, 64, 32, 96] if name == "ddim_ragged" else None
    assert torch.equal(m.model.decode(z0, z_lengths=lens), m.model.decode(z1, z_lengths=lens))


# ---- 3. mixed scales: each chart against the chart requested alone at its scale -------------------------------------------------
MIX_RUNS = {
    "ddim": lambda m, **a: DDIMSampler(m).sample(S=10, **a)[0],
    "ddim_eta1": lambda m, **a: DDIMSampler(m).sample(S=10, eta=1.0, **a)[0],
    "plms": lambda m, **a: PLMSSampler(m).sample(S=10, **a)[0],
    "ddpm_T50": lambda m, **a: DDPMSampler(m).sample(**a)[0],
    "dpm2": lambda m, **a: DPMSolverSampler(m).sample(S=10, order=2, **a)[0],
    "unipc_bh2": lambda m, **a: UniPCSampler(m).sample(S=6, variant="bh2", **a)[0],
}


def _mix_vs_alone(name, L, invariant):
    seed = 900
    m = model_for(L, 50 if name == "ddpm_T50" else 1000, invariant)
    kw = request(4, L)
    z = MIX_RUNS[name](m, seeds=seed, unconditional_guidance_scale=SCALES, **kw)
    assert _guided_key(m)
    logits = m.model.decode(z)
    notes = m.model.decode_to_hit_objects(z, 10.0)
    worst_z = worst_l = 0.0
    flips = []
    for b, s in enumerate(SCALES):
        zb = MIX_RUNS[name](m, seeds=[seed + b], unconditional_guidance_scale=s, **one_chart(kw, b))
        lb = m.model.decode(zb)
        if invariant and s != 1.0:
            assert torch.equal(z[b], zb[0]) and torch.equal(logits[b], lb[0]), (name, b)
        worst_z = max(worst_z, rel_err(z[b], zb[0]))
        worst_l = max(worst_l, rel_err(logits[b], lb[0]))
        alone = m.model.decode_to_hit_objects(zb, 10.0)[0]
        if L == 96 or invariant and s != 1.0:
            assert notes[b] == alone, (name, b)
        else:
            # 8 * 512 frames of logits that match to GEMM rounding: a logit within that rounding of 0 may turn a note or its tail on
            # or off (bit-identical notes are what batch_invariant=True gives); at most a handful of a chart's thousands of lines
            flips.append(len(set(notes[b]) ^ set(alone)))
            assert flips[-1] <= max(4, len(alone) // 1000), (name, b, flips[-1], len(alone))
    print(f"{name} L={L} invariant={invariant}: chart vs alone, max rel err z {worst_z:.2e} logits {worst_l:.2e}, "
          f"hit-object lines that differ {flips}")
    assert worst_z <= PIN and worst_l <= PIN, (worst_z, worst_l)


@pytest.mark.parametrize("L", [96, 512])
@pytest.mark.parametrize("name", sorted(MIX_RUNS))
def test_mixed_scale_chart_equals_the_chart_requested_alone(name, L):
    _mix_vs_alone(name, L, False)


@pytest.mark.parametrize("L", [96, 512])
@pytest.mark.parametrize("name", sorted(MIX_RUNS))
def test_mixed_scale_chart_is_bit_identical_alone_when_batch_invariant(name, L):
    _mix_vs_alone(name, L, True)


# ---- 4. loops and sessions -----------------------------------------------------------------------------------------------------
def test_device_loop_equals_per_step_loop():
    m = model_for(96, 50)
    kw = dict(request(4, 96), unconditional_guidance_scale=SCALES)
    runs = (lambda **a: DDIMSampler(m).sample(S=10, eta=1.0, log_every_t=4, **a), lambda **a: PLMSSampler(m).sample(S=8, **a),
            lambda **a: DPMSolverSampler(m).sample(S=8, **a), lambda **a: UniPCSampler(m).sample(S=6, **a),
            lambda **a: DDPMSampler(m).sample(log_every_t=20, **a),
            lambda **a: DDIMSampler(m).sample(S=10, **_inpaint_kw(4, 96), **a))
    for run in runs:
        z, inter = run(seeds=3, **kw)
        zs, inter_s = run(seeds=3, callback=lambda i: None, **kw)
        assert torch.equal(z, zs)
        for a, b in zip(inter["pred_x0"] + inter["x_inter"], inter_s["pred_x0"] + inter_s["x_inter"]):
            assert torch.equal(a, b)


def test_second_scale_mix_reuses_the_session_and_graph():
    m = model_for(96)
    kw = request(4, 96)
    s = DDIMSampler(m)
    s.sample(S=10, seeds=11, unconditional_guidance_scale=SCALES, **kw)
    key = (8, 96, False, "guided")
    sess = m.engine.sessions[key]
    plan = sess.plan
    assert plan.captured and s.last_launches_per_step == plan.launches + 2
    mix = [9.0, 1.0, 2.0, 4.0]
    z = s.sample(S=10, seeds=11, unconditional_guidance_scale=mix, **kw)[0]
    assert m.engine.sessions[key] is sess and sess.plan is plan and sess.scales.tolist() == mix
    for b, sc in enumerate(mix):
        zb = s.sample(S=10, seeds=[11 + b], unconditional_guidance_scale=sc, **one_chart(kw, b))[0]
        assert rel_err(z[b], zb[0]) <= PIN


def test_with_lengths_padded_tails_stay_zero_and_nan_tails_change_no_bit():
    lens = [96, 64, 32, 96]
    m = model_for(96)
    kw = dict(request(4, 96), unconditional_guidance_scale=SCALES)
    x_T = torch.randn(4, 16, 96, device="cuda")
    clean_x, nan_x = x_T.clone(), x_T.clone()
    clean_w, nan_w = [w.clone() for w in kw["w"]], [w.clone() for w in kw["w"]]
    for b, Lb in enumerate(lens):
        clean_x[b, :, Lb:] = 0.
        nan_x[b, :, Lb:] = NAN
        for w0, w1 in zip(clean_w, nan_w):
            k = w0.shape[-1] * Lb // 96
            w0[b, :, k:] = 0.
            w1[b, :, k:] = NAN
    for run in (lambda **a: DDIMSampler(m).sample(S=6, **a)[0], lambda **a: UniPCSampler(m).sample(S=5, **a)[0]):
        a = run(x_T=clean_x, z_lengths=lens, **dict(kw, w=clean_w))
        b = run(x_T=nan_x, z_lengths=lens, **dict(kw, w=nan_w))
        assert torch.isfinite(b).all() and torch.equal(a, b)
        for c, Lb in enumerate(lens):
            assert torch.all(a[c, :, Lb:] == 0)
    assert (8, 96, False, "ragged", "guided") in m.engine.sessions
