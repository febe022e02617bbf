"""The chart encoder: hit-object lines -> note array (host), Encoder.forward (launch plan) and the posterior (MUGD_OP_POSTERIOR).

CPU: parameter surface, config recovery, the oracle and the host convertor against the reference's recorded outputs, and the plan
compiler's bookkeeping (including the decoder plan, which shares the compiler and must not change).
GPU: the encoder against the reference golden and the live oracle, the posterior kernel against torch, and inpainting from an
encoded chart end to end.

Tolerances (max-abs error relative to the tensor's max magnitude): encoder outputs <= 1e-4 on the GPU (as the audio encoder),
<= 2e-5 for the oracle against the reference; the masked 6-step trajectory <= 1e-3 (DESIGN §2).
"""
import ctypes as C
import gzip
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import encoder_cases as ec
import encoder_oracle as eo
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import engine, netspec, packer, synth
from mug_diffusion_b200.config import EncoderConfig, ModelConfig
from mug_diffusion_b200.engine import Arena, DecoderCompiler, EncoderCompiler
from mug_diffusion_b200.postprocess import objects_to_array
from oracle import mug_oracle as orc

ENC = "model.first_stage_model.encoder."


def _rel(a, b) -> float:
    a, b = torch.as_tensor(a).detach().float().cpu(), torch.as_tensor(b).detach().float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _golden(golden_dir):
    g = np.load(os.path.join(golden_dir, f"encoder_L{ec.ENCODER_L}_B{ec.ENCODER_B}.npz"))
    return {k: torch.from_numpy(g[k]) for k in g.files}


def _golden_notes() -> torch.Tensor:
    """the two inputs of the encoder golden: the golden chart's note array and a dense uniform array, [2, 16, 768]"""
    frames = 8 * ec.ENCODER_L
    chart, _ = objects_to_array(ec.encoder_chart_lines(), 4, ec.golden_charts()["frame_ms"], frames)
    return torch.from_numpy(np.stack([chart, ec.dense_notes(frames)]))


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------
def _surface(golden_dir):
    with gzip.open(os.path.join(golden_dir, "ddpm_surface.json.gz"), "rt") as f:
        return json.load(f)


def test_encoder_param_specs_match_reference_state_dict(golden_dir):
    ref = {k: v for k, v in _surface(golden_dir)["state_dict"].items() if k.startswith(ENC)}
    mine = netspec.encoder_param_specs(EncoderConfig())
    assert len(ref) == 64 and set(mine) == set(ref)
    assert all(list(shape) == ref[k] for k, (shape, _) in mine.items())


def test_config_from_reference_recovers_encoder(golden_dir):
    from types import SimpleNamespace

    from test_from_reference import _standin_ddpm
    from mug_diffusion_b200.sampler import MugDiffusionB200

    ddpm = _standin_ddpm(_surface(golden_dir))
    _, cfg = MugDiffusionB200.config_from_reference(ddpm)
    assert cfg.encoder == EncoderConfig() and cfg.decoder == ModelConfig().decoder
    # the group count comes from the live encoder when the module has one
    ddpm.model.first_stage_model.encoder = SimpleNamespace(norm_out=SimpleNamespace(num_groups=4))
    assert MugDiffusionB200.config_from_reference(ddpm)[1].encoder.num_groups == 4
    # AutoencoderKL(constant_var=...) is refused, not half-supported
    ddpm.model.first_stage_model.log_var = torch.zeros(1)
    with pytest.raises(L_.MugdError, match="constant_var"):
        MugDiffusionB200.config_from_reference(ddpm)


def test_oracle_encoder_and_posterior_match_reference_golden(golden_dir):
    g = _golden(golden_dir)
    p = synth.synthetic_encoder_state_dict(seed=ec.ENCODER_SEED)
    with torch.no_grad():
        params = eo.encoder_forward(p, _golden_notes())
    torch.manual_seed(ec.SAMPLE_SEED)
    post = eo.posterior(params, 1.0, torch.randn(g["mean"].shape))
    assert _rel(params, g["parameters"]) <= 2e-5
    for k in ("mean", "logvar", "std", "sample"):
        assert _rel(post[k], g[k]) <= 2e-5, k
    assert torch.equal(g["mode"], g["mean"] * 1.0)


def test_objects_to_array_is_bit_identical_to_reference(golden_dir):
    with gzip.open(os.path.join(golden_dir, "objects_to_array.json.gz"), "rt") as f:
        gold = json.load(f)
    cases = ec.objects_cases()
    assert {c["name"] for c in cases} == set(gold)
    args = ("lines", "key_count", "frame_ms", "max_frame", "rate", "offset_ms")
    for c in cases:
        want = np.asarray(gold[c["name"]]["array"], dtype=np.float32)
        want_valid = np.asarray(gold[c["name"]]["valid_flag"])
        for fn in (objects_to_array, eo.objects_to_array):
            arr, valid = fn(*(c[a] for a in args))
            assert arr.dtype == np.float32 and arr.shape == (4 * c["key_count"], c["max_frame"]), c["name"]
            assert np.array_equal(arr, want), c["name"]
            assert np.array_equal(valid, want_valid), c["name"]


@pytest.fixture(scope="module")
def blobs():
    cfg = ModelConfig()
    sd = synth.synthetic_state_dict(96)
    plain = packer.pack_model(sd, cfg.unet, cfg.decoder)
    with_enc = packer.pack_model({**sd, **synth.synthetic_encoder_state_dict()}, cfg.unet, cfg.decoder)
    return cfg, plain, with_enc


def test_decoder_plan_and_plain_blob_are_unchanged(blobs):
    """the encoder shares the decoder's compiler and packer: the decoder plan and a blob without encoder weights must come out
    exactly as before the encoder existed (hashes recorded from the earlier compiler)"""
    cfg, plain, _ = blobs
    res = DecoderCompiler(cfg.decoder, plain, 1 << 30).compile(Arena(1 << 32), 4, 512)
    assert len(res["ops"].ops) == 49
    assert hashlib.sha256(bytes(res["ops"].array())).hexdigest() == "9ea4b1a1de279ffe670f8da2a37b59afdb2c4917952c856a170bd915de2ab8c4"
    assert hashlib.sha256(plain.data.numpy().tobytes()).hexdigest() == "c3fd5d58e682cc1a294bfc0c254aa489561795df4ec6eaa35440e4d0271c7258"
    assert "encoder_cfg" not in plain.meta and not any(k.startswith(ENC) for k in plain.entries)


def test_packer_folds_encoder_nin_shortcut(blobs):
    _, plain, blob = blobs
    assert blob.meta["encoder_cfg"] == EncoderConfig()
    assert torch.equal(blob.data[:plain.numel], plain.data[:plain.numel])      # the encoder is appended behind the decoder
    esd = synth.synthetic_encoder_state_dict()
    p = ENC + "down.1.block.0."
    w = blob.view(p + "out_skip.weight")
    assert w.shape == (128, 3 * 128 + 64)
    assert torch.equal(w[:, 384:], esd[p + "nin_shortcut.weight"][:, :, 0])
    assert torch.equal(blob.view(p + "out_skip.bias"), esd[p + "conv2.bias"] + esd[p + "nin_shortcut.bias"])
    assert torch.equal(blob.view(ENC + "down.0.downsample.conv.weight").view(64, 3, 64)[:, 2], esd[ENC + "down.0.downsample.conv.weight"][:, :, 2])


def _ranges(op):
    """(start, end) byte ranges an op reads and writes"""
    out = []
    if op.kind == L_.OP_GEMM:
        g = op.u.gemm
        rows_in = g.M // g.Lout * g.Lin
        out.append((g.A, g.A + 4 * ((rows_in - 1) * g.lda + g.K)))
        if g.A2:
            out.append((g.A2, g.A2 + 4 * ((g.M - 1) * g.lda2 + g.K2)))
        if g.residual:
            out.append((g.residual, g.residual + 4 * ((g.M - 1) * g.ldr + g.N)))
        out.append((g.C, g.C + 4 * ((g.M - 1) * g.ldc + g.N)))
    elif op.kind == L_.OP_GROUPNORM:
        d = op.u.gn
        out.append((d.x, d.x + 4 * ((d.B * d.L - 1) * d.ldx + d.C)))
        out.append((d.y, d.y + 4 * ((d.B * d.L - 1) * d.ldy + d.C)))
    return out


class _TrackingArena(Arena):
    """records every allocation with the op index at which it was made and released"""

    def __init__(self, base, clock):
        super().__init__(base)
        self.clock, self.allocs = clock, []

    def alloc(self, rows, cols):
        v = super().alloc(rows, cols)
        self.allocs.append([v.ptr, v.ptr + 4 * rows * cols, self.clock(), None])
        return v

    def release(self, mark):
        for a in self.allocs:
            if a[3] is None and a[0] >= self.base + mark:
                a[3] = self.clock()
        super().release(mark)


@pytest.mark.parametrize("B,Lz", [(2, 96), (4, 512), (8, 992)])
def test_encoder_plan_compiles(blobs, B, Lz, monkeypatch):
    _, _, blob = blobs
    lib = L_.load()
    comp = EncoderCompiler(EncoderConfig(), blob, 1 << 30)
    n_ops = [0]
    add = engine.OpList.add

    def counting_add(self, *a, **k):
        n_ops[0] += 1
        return add(self, *a, **k)

    monkeypatch.setattr(engine.OpList, "add", counting_add)
    arena = _TrackingArena(1 << 32, lambda: n_ops[0])
    res = comp.compile(arena, B, Lz)
    ops = res["ops"].ops
    kinds = [o.kind for o in ops]
    gemms = [o.u.gemm for o in ops if o.kind == L_.OP_GEMM]
    assert kinds.count(L_.OP_GROUPNORM) == 13 and set(kinds) == {L_.OP_GEMM, L_.OP_GROUPNORM}
    down = [g for g in gemms if g.conv_mode == L_.CONV_DOWN]
    assert [(g.Lin, g.Lout) for g in down] == [(8 * Lz, 4 * Lz), (4 * Lz, 2 * Lz), (2 * Lz, Lz)]
    assert (res["inp"].rows, res["inp"].cols) == (B * 8 * Lz, 16) and (res["out"].rows, res["out"].cols) == (B * Lz, 32)
    assert res["Lout"] == Lz and gemms[0].M == B * 8 * Lz and gemms[-1].M == B * Lz
    # every GEMM but conv_in (K = 16 per tap) is taken by the tensor-core kernel
    for i, g in enumerate(gemms):
        ok = C.c_int32()
        assert lib.mugd_gemm_tc_query(None, C.byref(g), 132, C.byref(ok), None, None, None) == 0
        assert bool(ok.value) == (i != 0), (i, g.M, g.N, g.K)
    # ~2.8 GFLOP per chart at L = 512, scaling with L (the three folded nin_shortcut 1x1 terms ride as K2 columns)
    flops = sum(2.0 * g.M * g.N * (g.K * g.taps + g.K2) for g in gemms)
    assert abs(flops / B / 1e9 - 2.8 * Lz / 512) < 0.1 * Lz / 512
    # no two arena buffers that are live at the same time share a byte: a buffer lives from its allocation to its release, and
    # longer if an op still reads or writes it (a use after release would collide with the buffer that reuses its bytes)
    live = [list(a) for a in arena.allocs]
    for k, op in enumerate(ops):
        for lo, hi in _ranges(op):
            owner = [a for a in live if a[0] <= lo and hi <= a[1] and a[2] <= k]
            assert owner, (k, op.kind)
            a = max(owner, key=lambda a: a[2])                    # the latest allocation made before op k that holds the range
            a[3] = max(a[3] if a[3] is not None else len(ops), k + 1)
    for i, a in enumerate(live):
        for b in live[i + 1:]:
            t_overlap = a[2] < (b[3] if b[3] is not None else len(ops)) and b[2] < (a[3] if a[3] is not None else len(ops))
            assert not (t_overlap and a[0] < b[1] and b[0] < a[1]), (a, b)


def test_library_abi_has_posterior():
    lib = L_.load()
    sizes = (C.c_int32 * 13)()
    assert lib.mugd_abi_sizes(sizes, 13) == 0 and sizes[12] == C.sizeof(L_.Posterior) == 64
    assert lib.mugd_abi_sizes(sizes, 12) != 0
    assert L_.ABI_VERSION == 13 and L_.OP_POSTERIOR == 13 and sizes[0] == C.sizeof(L_.Op)


# ---------------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------------
_model = {}


def _encoder_model(L=96, impl="auto"):
    from mug_diffusion_b200.sampler import MugDiffusionB200

    if (L, impl) not in _model:
        _model.clear()
        sd = {**synth.synthetic_state_dict(L), **synth.synthetic_encoder_state_dict(seed=ec.ENCODER_SEED)}
        _model[L, impl] = MugDiffusionB200.from_state_dict(sd, z_length=L, gemm_impl=impl)
    return _model[L, impl]


@pytest.mark.gpu
def test_encode_matches_reference_golden(golden_dir):
    _encode_vs_golden(golden_dir, "auto")


@pytest.mark.gpu
def test_encode_simt_matches_reference_golden(golden_dir):
    """the chart encoder with every GEMM on the exact-fp32 FFMA kernel: same tolerance"""
    _encode_vs_golden(golden_dir, "simt")


def _encode_vs_golden(golden_dir, impl):
    g = _golden(golden_dir)
    m = _encoder_model(impl=impl)
    post = m.model.encode({"note": _golden_notes().cuda()})
    for k in ("parameters", "mean", "logvar", "std"):
        got = getattr(post, k)
        assert got.is_cuda and got.shape == g[k].shape, k
        print(f"encode {impl} {k} rel_err={_rel(got, g[k]):.2e}")
        assert _rel(got, g[k]) <= 1e-4, (k, _rel(got, g[k]))
    assert torch.equal(post.mode(), post.mean * 1.0)
    assert torch.equal(post.var, torch.exp(post.logvar))
    torch.manual_seed(ec.SAMPLE_SEED)
    s = post.sample()
    assert s.is_cuda and _rel(s, g["sample"]) <= 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("B,L", [(4, 512), (2, 992)])
def test_encode_vs_live_oracle(B, L):
    m = _encoder_model()
    frames = 8 * L
    g = ec.golden_charts()
    charts = (g["ddim_L512_B1_S50_cfg5"] + g["synthetic"])[:B - 1]
    notes = torch.cat([eo.chart_arrays(charts, g["frame_ms"], frames), torch.from_numpy(ec.dense_notes(frames, seed=L))[None]])
    post = m.model.encode({"note": notes.cuda()})
    with torch.no_grad():
        params = eo.encoder_forward(synth.synthetic_encoder_state_dict(seed=ec.ENCODER_SEED), notes)
    ref = eo.posterior(params)
    assert _rel(post.parameters, params) <= 1e-4
    for k in ("mean", "logvar", "std"):
        assert _rel(getattr(post, k), ref[k]) <= 1e-4, k


def _ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    ia, ib = a.contiguous().view(torch.int32).long(), b.contiguous().view(torch.int32).long()
    assert torch.equal(a.sign(), b.sign())
    return int((ia - ib).abs().max())


@pytest.mark.gpu
def test_posterior_op_vs_torch():
    from gpu_util import OpRunner
    from mug_diffusion_b200.engine import OpList

    B, Z, L, scale = 3, 16, 200, 0.7
    gen = torch.Generator().manual_seed(11)
    params = (torch.randn(B, 2 * Z, L, generator=gen) * 12.0).cuda()           # logvar well past both clamp bounds
    params[:, Z:, :8] = torch.tensor([-1e4, -10.0, -9.99, 19.99, 20.0, 20.01, 3e4, 0.0]).cuda()
    noise = torch.randn(B, Z, L, generator=gen).cuda()
    lv_raw = params[:, Z:]
    assert (lv_raw < -10).any() and (lv_raw > 20).any()
    run = OpRunner()
    outs = {n: torch.full((B, Z, L), float("nan"), device="cuda") for n in ("mean", "logvar", "std", "z", "zs")}

    def op(noise_t, **o):
        d = L_.Posterior()
        d.params, d.noise = params.data_ptr(), noise_t.data_ptr() if noise_t is not None else None
        for k, t in o.items():
            setattr(d, k, t.data_ptr())
        d.scale, d.B, d.Z, d.L = scale, B, Z, L
        ops = OpList()
        ops.add(L_.OP_POSTERIOR, d)
        run.run(ops)

    op(None, mean=outs["mean"], logvar=outs["logvar"], std=outs["std"], z=outs["z"])
    op(noise, z=outs["zs"])
    mean, logvar = torch.chunk(params, 2, dim=1)
    logvar = torch.clamp(logvar, -10.0, 20.0)
    std = torch.exp(0.5 * logvar)
    assert torch.equal(outs["mean"], mean) and torch.equal(outs["logvar"], logvar)
    assert torch.equal(outs["z"], mean * scale)
    assert _ulps(outs["std"], std) <= 2
    assert _ulps(outs["zs"], (mean + std * noise) * scale) <= 2


@pytest.mark.gpu
def test_inpainting_from_an_encoded_chart_vs_oracle():
    """keep the first half of a real chart, regenerate the rest: hit-object lines -> encode_hit_objects -> mode() = x0, then the
    masked sampler.  The sampler's only RNG call per step at eta = 0 is q_sample's randn_like(x0) on the CUDA generator, so re-seeding
    and repeating the draws hands the oracle the very same noise."""
    from mug_diffusion_b200.sampler import DDIMSampler

    L, B, S = 96, 2, 6
    m = _encoder_model(L)
    g = ec.golden_charts()
    charts = g["ddim_L96_B2_S10_cfg5"]
    x0 = m.model.encode_hit_objects(charts, g["frame_ms"]).mode()
    assert x0.shape == (B, 16, L)
    mask = torch.zeros(B, 16, L)
    mask[:, :, :L // 2] = 1.0                                        # latent frame j covers note frames 8j .. 8j+7
    inp = synth.synthetic_inputs(B, L)
    sampler = DDIMSampler(m)
    kw = dict(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), eta=0.0,
              shape=(16, L), unconditional_guidance_scale=3.0, unconditional_conditioning=inp["uc"].cuda())
    torch.cuda.manual_seed(77)
    z, _ = sampler.sample(mask=mask.cuda(), x0=x0, **kw)
    z_plain, _ = sampler.sample(**kw)
    torch.cuda.manual_seed(77)
    n_steps = len(range(0, 1000, 1000 // S))
    qseq = [torch.randn((B, 16, L), device="cuda").cpu() for _ in range(n_steps)]
    sd = synth.synthetic_state_dict(L)
    with torch.no_grad():
        x0_ref = eo.posterior(eo.encoder_forward(synth.synthetic_encoder_state_dict(seed=ec.ENCODER_SEED),
                                                 eo.chart_arrays(charts, g["frame_ms"], 8 * L)))["mode"]
        ref = orc.ddim_sample(sd, S, inp["c"], inp["w"], inp["x_T"], scale=3.0, uc=inp["uc"], mask=mask, x0=x0_ref, q_noise_seq=qseq)
    assert _rel(x0, x0_ref) <= 1e-4
    assert _rel(z, ref) <= 1e-3
    assert _rel(z_plain, z) > 1e-2                                   # the kept half really steered the trajectory


@pytest.mark.gpu
def test_encoder_and_decoder_sessions_share_the_lru():
    m = _encoder_model()
    notes = _golden_notes().cuda()
    p1 = m.model.encode({"note": notes}).parameters
    z = torch.randn(2, 16, 96, generator=torch.Generator().manual_seed(3)).cuda()
    l1 = m.model.decode(z)
    other = m.model.encode({"note": notes[:1, :, :384]}).parameters            # B = 1, L = 48: a second encoder plan
    assert other.shape == (1, 32, 48)
    assert torch.equal(m.model.encode({"note": notes}).parameters, p1)
    assert torch.equal(m.model.decode(z), l1)
    keys = set(m.engine.dec_sessions)
    assert {("enc", 2, 96), ("enc", 1, 48), (2, 96)} <= keys


@pytest.mark.gpu
def test_engine_without_encoder_refuses_encode():
    from mug_diffusion_b200.sampler import MugDiffusionB200

    _model.clear()
    m = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(96), z_length=96)
    with pytest.raises(L_.MugdError, match="encoder"):
        m.model.encode({"note": torch.zeros(1, 16, 768, device="cuda")})
    with pytest.raises(L_.MugdError, match="encoder"):
        m.engine.encoder_session(1, 96)
