"""Section prompts on the GPU (DESIGN §6b N20): MUGD_OP_ATTENTION_SEC against the float64 attention formula row by row, and requests
with sections against today's path, against the same chart requested alone, across the device and per-step loops, and composed with
ragged lengths, per-chart guidance scales and DPM-Solver++ inpainting."""
import os

import pytest
import torch

import attention_cases as ac
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.engine import OpList, View
from mug_diffusion_b200.sampler import DDIMSampler, DPMSolverSampler, MugDiffusionB200, UniPCSampler

from gpu_util import OpRunner, ptr, rel_err, view

pytestmark = pytest.mark.gpu

SENT = -7777.0
TOL = 2e-5               # the attention tests' bound on attention_cases.row_error
PIN = 2e-5               # chart in a batch vs the chart alone (the ragged and guidance-scale requests' bound)


@pytest.fixture(scope="module")
def R():
    return OpRunner()


def _table(layouts, Lq, level):
    """[B, 8] starts at Lq rows per sample for per-sample layouts in latent frames"""
    rows = []
    for st in layouts:
        rows.append([0] + [v >> level for v in st] + [Lq] * (L_.SECTIONS - 1 - len(st)))
    return torch.tensor(rows, dtype=torch.int32)


# (L, level) -> the cross-attention's rows Lq = L >> level; layouts in latent frames (multiples of 8 below L)
def _layouts(L, B):
    coarse = L >> 3
    every = [8 * r for r in range(1, min(coarse, L_.SECTIONS))]              # a change on every coarse row (up to 7)
    one_row = [8, 16] if L > 16 else [8]                                     # a one-row section at the coarsest level
    base = [every, one_row, [], [L - 8], [8 * (coarse // 2)]]
    return [base[b % len(base)] for b in range(B)]


KERNEL_CASES = [(L, lvl, B, D, T, impl) for L, lvl, B, D in [(96, 0, 2, 32), (96, 1, 3, 48), (96, 3, 8, 64), (512, 0, 1, 32),
                                                           (512, 2, 4, 64), (512, 3, 2, 64), (2048, 0, 2, 32), (2048, 1, 1, 48),
                                                           (2048, 3, 8, 64)]
                for T in (21, 32) for impl in (1, 0)]


@pytest.mark.parametrize("L,lvl,B,D,T,impl", KERNEL_CASES)
def test_attention_sec_against_fp64(R, L, lvl, B, D, T, impl):
    """every row against the float64 formula over its own section's keys; memory around the output keeps its sentinel"""
    H = 8
    Cc, Lq = H * D, L >> lvl
    g = torch.Generator().manual_seed(L * 131 + lvl * 17 + B * 7 + D + T + impl)
    q = torch.randn(B, Lq, Cc, generator=g)
    k = torch.randn(B * L_.SECTIONS, T, Cc, generator=g)
    v = torch.randn(B * L_.SECTIONS, T, Cc, generator=g)
    rel = torch.randn(129, H, generator=g)
    cg = 1 + 0.25 * torch.randn(129, H, generator=g)
    lay = _layouts(L, B)
    starts = _table(lay, Lq, lvl)
    qc = q.reshape(-1, Cc).cuda()
    kv = torch.cat([k.reshape(-1, Cc), v.reshape(-1, Cc)], 1).cuda()
    out = torch.full((B * Lq + 64, Cc + 64), SENT).cuda()
    relc, cgc, st = rel.cuda(), cg.cuda(), starts.cuda()
    ops = OpList()
    ops.attention(view(qc), view(kv, 0, Cc), view(kv, Cc, 2 * Cc), View(out.data_ptr() + 4 * 32, out.shape[1], B * Lq, Cc),
                  ptr(relc), ptr(cgc), B, H, Lq, T, 64, starts=ptr(st), sec_stride=T)
    assert ops.ops[0].kind == L_.OP_ATTENTION_SEC
    L_.check(R.lib.mugd_set_attention_impl(R.handle, impl), "attention_impl")
    try:
        R.run(ops)
    finally:
        L_.check(R.lib.mugd_set_attention_impl(R.handle, 1), "attention_impl")
    res = out.cpu()
    o = res[:B * Lq, 32:32 + Cc].reshape(B, Lq, Cc)
    rows = torch.arange(Lq)
    err = 0.0
    for b in range(B):
        sec = (starts[b, 1:][None, :] <= rows[:, None]).sum(1)
        for s in sec.unique().tolist():
            ref, mag = ac.ref_attention(q[b:b + 1], k[L_.SECTIONS * b + s][None], v[L_.SECTIONS * b + s][None], rel, cg, H, 64,
                                        D ** -0.5)
            sel = sec == s
            err = max(err, ac.row_error(o[b:b + 1, sel], ref[:, sel], mag[:, sel], H))
    print(f"attention_sec impl={impl} L={L} level={lvl} B={B} D={D} T={T} row_err={err:.3e}")
    assert err < TOL
    outside = res.clone()
    outside[:B * Lq, 32:32 + Cc] = SENT
    assert bool((outside == SENT).all())


# ---- requests -------------------------------------------------------------------------------------------------------------------
_models = {}


def model_for(L, invariant=False):
    key = (L, invariant)
    if key not in _models:
        if len(_models) > 2:
            _models.clear()
        _models[key] = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), cfg=ModelConfig(), z_length=L,
                                                        batch_invariant=invariant)
    return _models[key]


def request(B, L, seed=77):
    inp = synth.synthetic_inputs(B, L, seed=seed)
    return dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, shape=(16, L), verbose=False,
                unconditional_conditioning=inp["uc"].cuda(), unconditional_guidance_scale=5.0)


def prompts(kw, n, seed=5):
    """n prompts shaped like c[0], different from every c[b]"""
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(tuple(kw["c"].shape[1:]), generator=g).cuda() for _ in range(n)]


def layouts(kw, L):
    p = prompts(kw, 4)
    B = kw["batch_size"]
    base = [[(32, p[0]), (64, p[1])], [(8, p[2])], [], [(16, p[3]), (24, p[0]), (L - 8, p[1])]]
    return [base[b % 4] for b in range(B)]


def one_chart(kw, b, sections=None):
    out = dict(kw, c=kw["c"][b:b + 1], w=[w[b:b + 1] for w in kw["w"]], batch_size=1,
               unconditional_conditioning=kw["unconditional_conditioning"][b:b + 1])
    for k in ("mask", "x0"):
        if k in kw:
            out[k] = kw[k][b:b + 1]
    if isinstance(kw.get("unconditional_guidance_scale"), list):
        out["unconditional_guidance_scale"] = kw["unconditional_guidance_scale"][b]
    if sections is not None:
        out["sections"] = [sections[b]]
    return out


RUNS = {"ddim": lambda m, **a: DDIMSampler(m).sample(S=10, **a),
        "dpm": lambda m, **a: DPMSolverSampler(m).sample(S=8, **a),
        "unipc": lambda m, **a: UniPCSampler(m).sample(S=6, **a)}


def test_no_sections_is_todays_path():
    m = model_for(96)
    kw = request(2, 96)
    z0 = RUNS["ddim"](m, seeds=3, **kw)[0]
    for sec in (None, [[], []]):
        z = RUNS["ddim"](m, seeds=3, sections=sec, **kw)[0]
        assert torch.equal(z, z0)
    assert not [k for k in m.engine.sessions if "sectioned" in k]


def test_every_section_at_c_is_todays_chart():
    m = model_for(96)
    kw = request(2, 96)
    z0 = RUNS["ddim"](m, seeds=3, **kw)[0]
    sec = [[(8, kw["c"][b]), (48, kw["c"][b])] for b in range(2)]
    z = RUNS["ddim"](m, seeds=3, sections=sec, **kw)[0]
    assert [k for k in m.engine.sessions if "sectioned" in k]
    assert rel_err(z, z0) <= 2e-5
    assert m.model.decode_to_hit_objects(z, 10.0) == m.model.decode_to_hit_objects(z0, 10.0)


def test_a_section_prompt_changes_the_chart():
    """a section prompt changes the chart (the U-Net's receptive field spreads it before its start too)"""
    m = model_for(96)
    kw = request(2, 96)
    z0 = RUNS["ddim"](m, seeds=3, **kw)[0]
    z = RUNS["ddim"](m, seeds=3, sections=layouts(kw, 96)[:2], **kw)[0]
    assert not torch.equal(z, z0) and bool(torch.isfinite(z).all())


@pytest.mark.parametrize("name", list(RUNS))
@pytest.mark.parametrize("invariant", [False, True], ids=["default", "invariant"])
def test_chart_in_a_batch_equals_the_chart_alone(name, invariant):
    m = model_for(96, invariant)
    kw = request(4, 96)
    sec = layouts(kw, 96)
    z = RUNS[name](m, seeds=11, sections=sec, **kw)[0]
    for b in range(4):
        zb = RUNS[name](m, seeds=[11 + b], **one_chart(kw, b, sec))[0]
        if invariant and sec[b]:
            assert torch.equal(z[b], zb[0]), (name, b)
        elif invariant:
            # a chart without sections requested alone takes today's plan, whose head-dim-32 cross-attentions run on another kernel
            assert rel_err(z[b], zb[0]) <= PIN, (name, b, rel_err(z[b], zb[0]))
        else:
            assert rel_err(z[b], zb[0]) <= PIN, (name, b, rel_err(z[b], zb[0]))


def test_device_loop_equals_per_step_loop_and_a_second_layout_reuses_the_graph():
    m = model_for(96)
    kw = request(4, 96)
    sec = layouts(kw, 96)
    for name in RUNS:
        z = RUNS[name](m, seeds=3, sections=sec, **kw)[0]
        zs = RUNS[name](m, seeds=3, sections=sec, callback=lambda i: None, **kw)[0]
        assert torch.equal(z, zs), name
    key = (8, 96, False, "sectioned")
    sess = m.engine.sessions[key]
    plan = sess.plan
    p = prompts(kw, 2, seed=9)
    RUNS["ddim"](m, seeds=3, sections=[[(40, p[0])], [(88, p[1])], [], [(8, p[0]), (16, p[1])]], **kw)
    assert m.engine.sessions[key] is sess and sess.plan is plan and plan.captured


def test_with_lengths_scales_and_inpainting():
    m = model_for(96)
    kw = request(4, 96)
    p = prompts(kw, 3)
    # ragged: starts below each chart's own length
    sec = [[(8, p[0])], [(32, p[1])], [], [(56, p[2])]]
    lens = [32, 64, 96, 64]
    z = RUNS["ddim"](m, seeds=5, sections=sec, z_lengths=lens, **kw)[0]
    for b in range(4):
        kb = one_chart(dict(kw, shape=(16, lens[b])), b, sec)
        kb["w"] = [w[b:b + 1, :, :w.shape[2] * lens[b] // 96] for w in kw["w"]]
        zb = DDIMSampler(model_for(96)).sample(S=10, seeds=[5 + b], **kb)[0]
        assert rel_err(z[b, :, :lens[b]], zb[0]) <= PIN, b
    # per-chart guidance scales
    kws = dict(kw, unconditional_guidance_scale=[1.0, 3.0, 5.0, 7.5])
    sec = layouts(kw, 96)
    z = RUNS["ddim"](m, seeds=7, sections=sec, **kws)[0]
    for b in range(4):
        zb = RUNS["ddim"](m, seeds=[7 + b], **one_chart(kws, b, sec))[0]
        assert rel_err(z[b], zb[0]) <= PIN, b
    # DPM-Solver++ inpainting
    x0 = torch.randn(4, 16, 96, generator=torch.Generator().manual_seed(2)).cuda()
    mask = torch.ones(4, 16, 96).cuda()
    mask[:, :, 40:72] = 0
    kwi = dict(kw, x0=x0, mask=mask)
    z = DPMSolverSampler(m).inpaint(S=8, seeds=9, sections=sec, **kwi)[0]
    for b in range(4):
        zb = DPMSolverSampler(m).inpaint(S=8, seeds=[9 + b], **one_chart(kwi, b, sec))[0]
        assert rel_err(z[b], zb[0]) <= PIN, b


# ---- against the reference with its CrossAttention.forward run once per section (tools/make_section_goldens.py) ------------------
def _golden_request():
    import section_cases as sc
    inp = synth.synthetic_inputs(sc.B, sc.L)
    lay = [[(s, ctx.cuda()) for s, ctx in chart] for chart in sc.layouts()]
    return sc, inp, lay


@pytest.mark.parametrize("impl", ["auto", "simt"])
def test_unet_evaluation_against_the_reference_golden(impl, golden_dir):
    import golden_cases as gc
    sc, inp, lay = _golden_request()
    m = model_for(sc.L)
    if impl == "simt":
        m = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(sc.L), cfg=ModelConfig(), z_length=sc.L, gemm_impl="simt")
    w = synth.wave_list([torch.cat([wi, wi]).cuda() for wi in inp["w"]])
    eps = m.model.forward(torch.cat([inp["x_T"]] * 2).cuda(), torch.tensor(sc.T_EVAL * 2).cuda(),
                          torch.cat([inp["uc"], inp["c"]]).cuda(), w, sections=[[]] * sc.B + lay)
    g = gc.load_golden(os.path.join(golden_dir, sc.EVAL_NAME + ".npz"))["eps"]
    assert rel_err(eps, g) < 1e-4


def test_ddim_trajectory_and_logits_against_the_reference_golden(golden_dir):
    import golden_cases as gc
    sc, inp, lay = _golden_request()
    m = model_for(sc.L)
    z, _ = DDIMSampler(m).sample(S=sc.S, c=inp["c"].cuda(), w=synth.wave_list([w.cuda() for w in inp["w"]]), batch_size=sc.B,
                                 shape=None, verbose=False, x_T=inp["x_T"].cuda(), eta=0.0, unconditional_guidance_scale=sc.SCALE,
                                 unconditional_conditioning=inp["uc"].cuda(), sections=lay)
    logits = m.model.decode(z)
    g = gc.load_golden(os.path.join(golden_dir, sc.DDIM_NAME + ".npz"))
    assert rel_err(z, g["z"]) < 1e-3 and rel_err(logits, g["logits"]) < 1e-3


# ---- decode and invert ---------------------------------------------------------------------------------------------------------
def _x_latent(B, L, seed=4):
    return torch.randn(B, 16, L, generator=torch.Generator().manual_seed(seed)).cuda()


STARTS = {"ddim": [6, 3, 9, 6], "dpm": [5, 2, 8, 5], "unipc": [4, 2, 6, 4]}      # t_start / t_enc per chart


@pytest.mark.parametrize("flow", ["decode", "invert"])
@pytest.mark.parametrize("name", list(RUNS))
def test_decode_and_invert_take_sections(flow, name):
    """with sections, each chart equals the chart alone (its own start or stop, its own sections); all-empty lists are today's call"""
    m = model_for(96)
    kw = request(4, 96)
    cond = dict(c=kw["c"], w=kw["w"], unconditional_guidance_scale=5.0, unconditional_conditioning=kw["unconditional_conditioning"])
    x = _x_latent(4, 96)
    sec = layouts(kw, 96)
    z = _one(flow, name, m, x, STARTS[name], dict(cond, sections=sec))
    plain = _one(flow, name, m, x, STARTS[name], cond)
    assert torch.equal(_one(flow, name, m, x, STARTS[name], dict(cond, sections=[[]] * 4)), plain)
    assert not torch.equal(z, plain)
    for b in range(4):
        one = dict(c=cond["c"][b:b + 1], w=[w[b:b + 1] for w in cond["w"]], unconditional_guidance_scale=5.0,
                   unconditional_conditioning=cond["unconditional_conditioning"][b:b + 1], sections=[sec[b]])
        zb = _one(flow, name, m, x[b:b + 1], STARTS[name][b], one)
        assert rel_err(z[b], zb[0]) <= PIN, (flow, name, b)


def _one(flow, name, m, x, start, kw):
    if name == "ddim":
        s = DDIMSampler(m)
        s.make_schedule(10, verbose=False)
        return s.decode(x, t_start=start, **kw) if flow == "decode" else s.invert(x, t_enc=start, verbose=False, **kw)
    if name == "dpm":
        s = DPMSolverSampler(m)
        sch = s.make_dpm_schedule(8)
    else:
        s = UniPCSampler(m)
        sch = s.make_unipc_schedule(6)
    return s.decode(x, t_start=start, sched=sch, **kw) if flow == "decode" else s.invert(x, t_enc=start, sched=sch, verbose=False, **kw)
