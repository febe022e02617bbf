"""Ragged requests on the GPU.

* Kernels against float64: the ragged GroupNorm(+SiLU) (every register variant and the two-pass form, every shape the ragged U-Net and
  decoder plans launch) and ragged self-attention (the wgmma, FFMA and lane-per-key kernels, each at every shape the plans launch
  that the dispatch gives it), with the padded input rows filled with NaN.  The row-mask op is exact.
* Two ragged DDIM steps (lengths 96, 64 padded to 96, CFG 5) against the CPU oracle evaluated at L = 64, under the U-Net bound 1e-4.
* The main pin: each chart of a seeded ragged request (lengths 96, 64, 32, 96) equals the same seed requested alone at its own
  z_length, for DDIM (CFG 5, and eta = 1), DPM-Solver++ 2M, UniPC bh2 and DDPM T = 50; the decoded logits and notes as well.
* The device loop equals the per-step loop bit for bit; NaN in the padded tails of x_T and of the audio features changes no bit;
  a second length mix reuses the captured graph; all lengths = Lmax is bit-identical to a request without lengths."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from gpu_util import OpRunner, rel_err  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import packer, synth  # noqa: E402
from mug_diffusion_b200.config import ModelConfig  # noqa: E402
from mug_diffusion_b200.engine import Arena, DecoderCompiler, OpList, UNetCompiler, View  # noqa: E402
from mug_diffusion_b200.sampler import (DDIMSampler, DDPMSampler, DPMSolverSampler, MugDiffusionB200,  # noqa: E402
                                        UniPCSampler)

NAN = float("nan")
LENS = [96, 64, 32, 96]
# chart b of a ragged request vs the chart alone: relative max-abs error bound (measured maximum in DESIGN §6b N17)
PIN = 2e-5


@pytest.fixture(scope="module")
def R():
    return OpRunner()


def _valid_dev(vals):
    return torch.tensor(vals, dtype=torch.int32, device="cuda")


def _plan_shapes():
    """(B, L, C, G, silu) of every GroupNorm and (B, H, D, L) of every self-attention in the ragged plans at Lmax 96 and 512"""
    cfg = ModelConfig()
    blob = packer.pack_model(synth.synthetic_state_dict(96), cfg.unet, cfg.decoder)
    comp = UNetCompiler(cfg.unet, blob, 1 << 30)
    gn, at = {}, {}
    for Beff, Lz in ((8, 96), (8, 512)):
        blocks = list(comp.lay.blocks())
        ext = dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21,
                   ctx_kv=[View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin)
                           for i, b in enumerate(x for x in blocks if x.kind == "attn")],
                   s4_kt={b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin)
                          for i, b in enumerate(x for x in blocks if x.kind == "s4")})
        ops = comp.compile(Arena(1 << 32), Beff, Lz, ext, False, None, [1 << 43] * 4)["ops"].ops
        ops += DecoderCompiler(cfg.decoder, blob, 1 << 30).compile(Arena(1 << 32), Beff // 2, Lz, {m: 1 << 43 for m in (1, 2, 4, 8)})["ops"].ops
        for o in ops:
            if o.kind == L_.OP_GROUPNORM_VAR:
                d = o.u.gnv.gn
                gn.setdefault((d.B, d.L, d.C, d.G, d.silu), None)
            elif o.kind == L_.OP_ATTENTION_VAR:
                a = o.u.attnv.attn
                at.setdefault((a.B, a.H, a.D, a.Lq), None)
    return list(gn), list(at)


GN_PLAN, ATTN_PLAN = _plan_shapes()
# register-kernel boundaries (float4 per thread 2 / 4 / 8 / 16 / 32) and the two-pass form, beside the plan shapes
GN_EDGES = [(3, 96, 64, 16, 1), (2, 512, 256, 32, 0), (2, 1024, 256, 32, 1), (2, 2048, 256, 32, 1), (2, 4096, 256, 32, 0),
            (2, 4096, 512, 32, 1)]


def _gn_variant(B, L, C, G):
    pt = (L * (C // G // 4) + 255) // 256
    return next((f"reg{n}" for n in (2, 4, 8, 16, 32) if pt <= n), "two")


def _lengths(B, L):
    base = [L, max(1, (L * 2) // 3), 1, 0, L - 1, L // 2]
    return [base[b % len(base)] for b in range(B)]


@pytest.mark.parametrize("shape", GN_PLAN + GN_EDGES, ids=lambda s: "B{}-L{}-C{}-G{}-s{}".format(*s))
def test_groupnorm_var_against_fp64(R, shape):
    B, L, C, G, silu = shape
    torch.manual_seed(B * 7 + L + C)
    lens = _lengths(B, L)
    x = torch.randn(B, L, C, device="cuda") * 2 + 0.5
    for b, Lv in enumerate(lens):
        x[b, Lv:] = NAN                                          # padding: never read
    gamma, beta = torch.randn(C, device="cuda"), torch.randn(C, device="cuda")
    y = torch.full((B * L, C), -7777.0, device="cuda")
    valid = _valid_dev(lens)
    ops = OpList(valid={L: valid.data_ptr()})
    ops.groupnorm(View(x.data_ptr(), C, B * L, C), View(y.data_ptr(), C, B * L, C), gamma.data_ptr(), beta.data_ptr(), B, L, G, bool(silu))
    assert ops.ops[0].kind == L_.OP_GROUPNORM_VAR
    R.run(ops)
    y = y.view(B, L, C).double()
    worst = 0.0
    for b, Lv in enumerate(lens):
        assert torch.all(y[b, Lv:] == 0), (b, Lv)               # exact zeros, by a store
        if Lv == 0:
            continue
        xv = x[b, :Lv].double().view(Lv, G, C // G)
        m = xv.mean(dim=(0, 2), keepdim=True)
        r = 1.0 / torch.sqrt(xv.var(dim=(0, 2), unbiased=False, keepdim=True) + 1e-6)
        g64, b64 = gamma.double().view(G, C // G), beta.double().view(G, C // G)
        ref = (xv - m) * r * g64 + b64
        A = (xv.abs() + m.abs()) * r * g64.abs() + b64.abs()
        if silu:
            ref = ref * torch.sigmoid(ref)
            A = A * 1.1
        err = (y[b, :Lv].view(Lv, G, C // G) - ref).abs() / (2.0 ** -24 * (A + ref.abs()))
        worst = max(worst, float(err.max()))
    print(f"groupnorm_var {shape} ({_gn_variant(B, L, C, G)}): max err / 2^-24 (A + |ref|) = {worst:.2f}")
    assert worst <= 16, worst


class _Impl:
    def __init__(self, R, impl):
        self.R, self.impl = R, impl

    def __enter__(self):
        L_.check(self.R.lib.mugd_set_attention_impl(self.R.handle, self.impl), "attention_impl")

    def __exit__(self, *a):
        L_.check(self.R.lib.mugd_set_attention_impl(self.R.handle, 1), "attention_impl")


def _kernel_of(impl, L, D):
    if impl == 0:
        return "ffma"
    return "lane" if L <= 32 and D >= 48 else "wgmma"


# the plans' self-attention shapes, each on every kernel the dispatch gives it (impl 1: wgmma or lane-per-key; impl 0: FFMA), plus
# bounds at tile edges: the wgmma kernel's 128-key and the FFMA kernel's 64-key tiles, partial last tiles, and 32 keys or fewer
ATTN_CASES = [(s, impl) for s in ATTN_PLAN for impl in (1, 0)] + [((13, 4, D, L), impl) for D in (32, 48, 64)
                                                                 for L in (300, 256) for impl in (1, 0)]


@pytest.mark.parametrize("shape,impl", ATTN_CASES, ids=lambda v: "B{}-H{}-D{}-L{}".format(*v) if isinstance(v, tuple) else str(v))
def test_attention_var_against_fp64(R, shape, impl):
    B, H, D, L = shape
    P = 64
    torch.manual_seed(L * 3 + D + B)
    Cc = H * D
    cand = [L, 1, 0, 20, 32, 33, 64, 65, 127, 128, 129, 200, L - 1]
    lens = [v for v in cand if v <= L]
    lens = [lens[b % len(lens)] for b in range(max(B, 2))][:B]
    qkv = torch.randn(B, L, 3 * Cc, device="cuda")
    for b, Lv in enumerate(lens):
        qkv[b, Lv:] = NAN
    rel, cg = torch.randn(2 * P + 1, H, device="cuda") * 0.5, torch.rand(2 * P + 1, H, device="cuda") + 0.5
    o = torch.full((B * L, Cc), -7777.0, device="cuda")
    valid = _valid_dev(lens)
    base = qkv.data_ptr()
    ops = OpList(valid={L: valid.data_ptr()})
    ops.attention(View(base, 3 * Cc, B * L, Cc), View(base + 4 * Cc, 3 * Cc, B * L, Cc), View(base + 8 * Cc, 3 * Cc, B * L, Cc),
                  View(o.data_ptr(), Cc, B * L, Cc), rel.data_ptr(), cg.data_ptr(), B, H, L, L, P, self_attn=True)
    assert ops.ops[0].kind == L_.OP_ATTENTION_VAR
    with _Impl(R, impl):
        R.run(ops)
    o = o.view(B, L, H, D).double()
    q, k, v = (qkv[..., i * Cc:(i + 1) * Cc].double().view(B, L, H, D) for i in range(3))
    worst = 0.0
    for b, Lv in enumerate(lens):
        assert torch.all(o[b, Lv:] == 0), (b, Lv)
        if Lv == 0:
            continue
        idx = (torch.arange(Lv, device="cuda")[None, :] - torch.arange(Lv, device="cuda")[:, None]).clamp(-P, P) + P
        s = torch.einsum("ihd,jhd->hij", q[b, :Lv], k[b, :Lv]) + rel.double()[idx].permute(2, 0, 1)
        p = torch.softmax(s * D ** -0.5, dim=-1) * cg.double()[idx].permute(2, 0, 1)
        ref = torch.einsum("hij,jhd->ihd", p, v[b, :Lv])
        worst = max(worst, float((o[b, :Lv] - ref).abs().max() / ref.abs().max()))
    print(f"attention_var {shape} {_kernel_of(impl, L, D)}: lengths {lens}, max rel err {worst:.2e}")
    assert worst <= 2e-5, worst


def test_row_mask_is_exact(R):
    B, L, ld, c0, cols = 5, 96, 40, 4, 29
    torch.manual_seed(0)
    x = torch.randn(B * L, ld, device="cuda")
    x[::7] = NAN
    lens = [96, 0, 1, 50, 95]
    before = x.clone()
    ops = OpList(valid={L: _valid_dev(lens).data_ptr()})
    ops.row_mask(View(x.data_ptr() + 4 * c0, ld, B * L, cols), B, L)
    R.run(ops)
    want = before.clone().view(B, L, ld)
    for b, Lv in enumerate(lens):
        want[b, Lv:, c0:c0 + cols] = 0.
    assert torch.equal(x.view(B, L, ld).nan_to_num(1e30), want.nan_to_num(1e30))


# ---- requests ---------------------------------------------------------------------------------------------------------------------
_models = {}


def model_for(L, T=1000):
    if (L, T) not in _models:
        _models.clear()
        _models[(L, T)] = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), cfg=ModelConfig(timesteps=T), z_length=L)
    return _models[(L, T)]


def request(B, L, cfg=True):
    inp = synth.synthetic_inputs(B, L, seed=99)
    kw = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, shape=(16, L), verbose=False)
    if cfg:
        kw.update(unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    return kw


def alone(kw, b, Lb):
    """the B = 1 request of chart b at its own length Lb: the first Lb positions of every per-position input"""
    out = dict(kw, c=kw["c"][b:b + 1], batch_size=1, shape=(16, Lb),
               w=[w[b:b + 1, :, :w.shape[-1] * Lb // kw["shape"][1]].contiguous() for w in kw["w"]])
    if "unconditional_conditioning" in kw:
        out["unconditional_conditioning"] = kw["unconditional_conditioning"][b:b + 1]
    return out


RUNS = {
    "ddim_cfg5": lambda m, **a: DDIMSampler(m).sample(S=10, **a)[0],
    "ddim_eta1": lambda m, **a: DDIMSampler(m).sample(S=10, eta=1.0, **a)[0],
    "dpm2": lambda m, **a: DPMSolverSampler(m).sample(S=10, order=2, **a)[0],
    "unipc_bh2": lambda m, **a: UniPCSampler(m).sample(S=6, variant="bh2", **a)[0],
    "ddpm_T50": lambda m, **a: DDPMSampler(m).sample(**a)[0],
}


@pytest.mark.parametrize("name", sorted(RUNS))
def test_ragged_chart_equals_the_chart_requested_alone(name):
    Lmax, seed = 96, 500
    m = model_for(Lmax, 50 if name == "ddpm_T50" else 1000)
    kw = request(len(LENS), Lmax)
    z = RUNS[name](m, seeds=seed, z_lengths=LENS, **kw)            # the longest length runs first (S4 kernels at L_int)
    logits = m.model.decode(z, z_lengths=LENS)
    notes = m.model.decode_to_hit_objects(z, 10.0, z_lengths=LENS)
    worst_z = worst_l = 0.0
    for b, Lb in enumerate(LENS):
        assert torch.all(z[b, :, Lb:] == 0) and torch.all(logits[b, :, 8 * Lb:] == 0)
        zb = RUNS[name](m, seeds=[seed + b], **alone(kw, b, Lb))
        lb = m.model.decode(zb)
        worst_z = max(worst_z, rel_err(z[b, :, :Lb], zb[0]))
        worst_l = max(worst_l, rel_err(logits[b, :, :8 * Lb], lb[0]))
        assert notes[b] == m.model.decode_to_hit_objects(zb, 10.0)[0], b
    print(f"{name}: chart vs alone, max rel err z {worst_z:.2e} logits {worst_l:.2e}")
    assert worst_z <= PIN and worst_l <= PIN, (worst_z, worst_l)


def test_ragged_unet_evaluations_against_the_oracle():
    from oracle import mug_oracle as orc
    L = 96
    m = model_for(L)
    sd = synth.synthetic_state_dict(L)
    inp = synth.synthetic_inputs(2, L, seed=7)
    kw = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=2, shape=(16, L), verbose=False, x_T=inp["x_T"].cuda(),
              unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    # S = 2 (timesteps 1 and 501): the second evaluation's eps carries a sizeable weight in z
    z = DDIMSampler(m).sample(S=2, z_lengths=[96, 64], **kw)[0]
    w64 = [w[1:2, :, :w.shape[-1] * 2 // 3] for w in inp["w"]]
    with torch.no_grad():
        ref = orc.ddim_sample(sd, 2, inp["c"][1:2], w64, inp["x_T"][1:2, :, :64], scale=5.0, uc=inp["uc"][1:2])
    err = rel_err(z[1, :, :64], ref[0])
    print(f"ragged chart (64 of 96) vs the oracle at L = 64: {err:.2e}")
    assert err <= 1e-4 and torch.all(z[1, :, 64:] == 0)


def test_ragged_device_loop_equals_per_step_loop():
    m = model_for(96)
    kw = request(len(LENS), 96)
    for run in (lambda **a: DDIMSampler(m).sample(S=10, eta=1.0, **a), lambda **a: UniPCSampler(m).sample(S=6, **a),
                lambda **a: DPMSolverSampler(m).sample(S=8, **a)):
        z, inter = run(seeds=3, z_lengths=LENS, **kw)
        zs, inter_s = run(seeds=3, z_lengths=LENS, callback=lambda i: None, **kw)
        assert torch.equal(z, zs)
        for a, b in zip(inter["pred_x0"] + inter["x_inter"], inter_s["pred_x0"] + inter_s["x_inter"]):
            assert torch.equal(a, b)
            for c, Lb in enumerate(LENS):
                assert torch.all(a[c, :, Lb:] == 0)


def test_nan_in_padded_tails_changes_no_bit():
    m = model_for(96)
    kw = request(len(LENS), 96)
    x_T = torch.randn(len(LENS), 16, 96, device="cuda")
    clean_x, nan_x = x_T.clone(), x_T.clone()
    clean_w, nan_w = [w.clone() for w in kw["w"]], [w.clone() for w in kw["w"]]
    for b, Lb in enumerate(LENS):
        clean_x[b, :, Lb:] = 0.
        nan_x[b, :, Lb:] = NAN
        for w0, w1 in zip(clean_w, nan_w):
            k = w0.shape[-1] * Lb // 96
            w0[b, :, k:] = 0.
            w1[b, :, k:] = NAN
    for run in (lambda **a: DDIMSampler(m).sample(S=6, **a)[0], lambda **a: UniPCSampler(m).sample(S=5, **a)[0]):
        a = run(x_T=clean_x, z_lengths=LENS, **dict(kw, w=clean_w))
        b = run(x_T=nan_x, z_lengths=LENS, **dict(kw, w=nan_w))
        assert torch.isfinite(b).all() and torch.equal(a, b)
    z = DDIMSampler(m).sample(S=6, x_T=clean_x, z_lengths=LENS, **dict(kw, w=clean_w))[0]
    znan = z.clone()
    for b, Lb in enumerate(LENS):
        znan[b, :, Lb:] = NAN
    assert torch.equal(m.model.decode(z, z_lengths=LENS), m.model.decode(znan, z_lengths=LENS))


def test_second_length_mix_reuses_the_captured_graph():
    m = model_for(96)
    kw = request(len(LENS), 96)
    s = DDIMSampler(m)
    s.sample(S=10, seeds=11, z_lengths=LENS, **kw)
    key = (8, 96, False, "ragged")
    sess = m.engine.sessions[key]
    plan = sess.plan
    assert plan.captured
    mix = [64, 96, 96, 32]
    z = s.sample(S=10, seeds=11, z_lengths=mix, **kw)[0]
    assert m.engine.sessions[key] is sess and sess.plan is plan and sess.lens == mix * 2
    for b, Lb in enumerate(mix):
        zb = s.sample(S=10, seeds=[11 + b], **alone(kw, b, Lb))[0]
        assert rel_err(z[b, :, :Lb], zb[0]) <= PIN and torch.all(z[b, :, Lb:] == 0)


def test_lengths_all_lmax_are_bit_identical_to_no_lengths():
    m = model_for(96)
    kw = request(len(LENS), 96)
    for run in (lambda **a: DDIMSampler(m).sample(S=6, **a)[0], lambda **a: DPMSolverSampler(m).sample(S=6, **a)[0]):
        assert torch.equal(run(seeds=21, z_lengths=[96] * 4, **kw), run(seeds=21, **kw))
