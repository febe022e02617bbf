"""Ragged requests on the CPU: the ragged U-Net and decoder plans (every op that mixes rows is masked), the C ABI of the three new
op kinds, the refusals of the flows a ragged request cannot take, and audio.pad_features."""
import ctypes as C
import hashlib
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from mug_diffusion_b200 import audio, packer, synth
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200.config import ModelConfig
from mug_diffusion_b200.engine import Arena, DecoderCompiler, UNetCompiler, View
from mug_diffusion_b200.sampler import (DDIMSampler, DDPMSampler, DPMSolverSampler, PLMSSampler, UniPCSampler, ragged_lengths,
                                        register_schedule)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VALID = 1 << 43                                   # fake device address of the valid-length arrays


@pytest.fixture(scope="module")
def blob():
    cfg = ModelConfig()
    return cfg, packer.pack_model(synth.synthetic_state_dict(96), cfg.unet, cfg.decoder)


def _ext(comp, Beff, Lz):
    blocks = list(comp.lay.blocks())
    ctx_kv = [View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin) for i, b in enumerate(x for x in blocks if x.kind == "attn")]
    s4 = {b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin) for i, b in enumerate(x for x in blocks if x.kind == "s4")}
    return dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21, ctx_kv=ctx_kv, s4_kt=s4)


def _rect(arena, ptr, ld, rows, cols):
    """the byte intervals [start, end) of a strided view's rows, sorted"""
    s = ptr + 4 * ld * np.arange(rows, dtype=np.int64)
    return s, s + 4 * cols


def _overlap(a, b) -> bool:
    j = np.searchsorted(b[1], a[0], side="right")           # first interval of b that ends after each interval of a starts
    ok = j < len(b[0])
    return bool(np.any(b[0][j[ok]] < a[1][ok]))


def _writes(op, arena):
    k = op.kind
    if k == L_.OP_GEMM:
        g = op.u.gemm
        return _rect(arena, g.C, g.ldc, g.M, g.N // 2 if g.gate else g.N)
    if k in (L_.OP_GROUPNORM, L_.OP_GROUPNORM_VAR):
        d = op.u.gn if k == L_.OP_GROUPNORM else op.u.gnv.gn
        return _rect(arena, d.y, d.ldy, d.B * d.L, d.C)
    if k == L_.OP_LAYERNORM:
        return _rect(arena, op.u.ln.y, op.u.ln.ldy, op.u.ln.rows, op.u.ln.C)
    if k in (L_.OP_ATTENTION, L_.OP_ATTENTION_VAR):
        a = op.u.attn if k == L_.OP_ATTENTION else op.u.attnv.attn
        return _rect(arena, a.o, a.ldo, a.B * a.Lq, a.H * a.D)
    if k == L_.OP_S4CONV:
        return _rect(arena, op.u.s4.y, op.u.s4.ldy, op.u.s4.B * op.u.s4.L, op.u.s4.H)
    if k == L_.OP_COPY2D:
        return _rect(arena, op.u.cp.dst, op.u.cp.ldd, op.u.cp.rows, op.u.cp.cols)
    if k == L_.OP_ROW_MASK:
        return _rect(arena, op.u.mask.x, op.u.mask.ld, op.u.mask.B * op.u.mask.L, op.u.mask.cols)
    raise AssertionError(f"op kind {k} in a ragged plan")


def _check_masked_convs(ops, arena):
    """every GEMM with taps > 1 reads A rows whose last writer is a GROUPNORM_VAR or a ROW_MASK; returns their count"""
    writes = [_writes(o, arena) for o in ops]
    n = 0
    for i, op in enumerate(ops):
        if op.kind != L_.OP_GEMM or op.u.gemm.taps == 1:
            continue
        g = op.u.gemm
        a = _rect(arena, g.A, g.lda, g.M // g.Lout * g.Lin, g.K)
        last = next((j for j in range(i - 1, -1, -1) if _overlap(writes[j], a)), None)
        assert last is not None, f"GEMM {i} reads rows no op of the plan wrote"
        assert ops[last].kind in (L_.OP_GROUPNORM_VAR, L_.OP_ROW_MASK), (i, last, ops[last].kind)
        n += 1
    return n


@pytest.mark.parametrize("Beff,Lz", [(8, 512), (4, 96)])
def test_ragged_unet_plan_masks_every_op_that_mixes_rows(blob, Beff, Lz):
    cfg, b = blob
    comp = UNetCompiler(cfg.unet, b, 1 << 30)
    arena = Arena(1 << 32)
    valid = [VALID + 256 * l for l in range(cfg.unet.levels)]
    res = comp.compile(arena, Beff, Lz, _ext(comp, Beff, Lz), False, None, valid)
    ops = res["ops"].ops
    lens = [Lz >> l for l in range(cfg.unet.levels)]
    kinds = [o.kind for o in ops]
    assert L_.OP_GROUPNORM not in kinds and kinds.count(L_.OP_GROUPNORM_VAR) == 77
    for o in ops:
        if o.kind == L_.OP_GROUPNORM_VAR:
            d = o.u.gnv
            assert d.valid == valid[lens.index(d.gn.L)] and d.gn.B == Beff
        elif o.kind == L_.OP_ATTENTION_VAR:                       # self-attention: bounded keys
            a = o.u.attnv
            assert a.attn.Lq == a.attn.Lk and a.valid == valid[lens.index(a.attn.Lq)]
        elif o.kind == L_.OP_ATTENTION:                           # cross-attention to the prompt tokens: unchanged
            assert o.u.attn.Lk == 21 and o.u.attn.Lq != 21
        elif o.kind == L_.OP_ROW_MASK:
            assert o.u.mask.valid == valid[lens.index(o.u.mask.L)] and o.u.mask.B == Beff
    assert kinds.count(L_.OP_ATTENTION_VAR) == 16 and kinds.count(L_.OP_ATTENTION) == 16
    # x, the 8 audio slots, 3 Downsample and 3 Upsample inputs and the 16 S4 out_layer inputs
    assert kinds.count(L_.OP_ROW_MASK) == 31
    first = [o.u.mask.x for o in ops[:12] if o.kind == L_.OP_ROW_MASK]
    assert first[0] == res["xin"].ptr and sorted(first[1:]) == sorted(v.ptr for _, v in res["audio_slots"])
    assert _check_masked_convs(ops, arena) == sum(1 for o in ops if o.kind == L_.OP_GEMM and o.u.gemm.taps > 1) > 40


def test_ragged_decoder_plan_masks_every_op_that_mixes_rows(blob):
    cfg, b = blob
    arena = Arena(1 << 32)
    valid = {m: VALID + 256 * k for k, m in enumerate((1, 2, 4, 8))}
    res = DecoderCompiler(cfg.decoder, b, 1 << 30).compile(arena, 4, 96, valid)
    ops = res["ops"].ops
    kinds = [o.kind for o in ops]
    assert L_.OP_GROUPNORM not in kinds and kinds.count(L_.OP_GROUPNORM_VAR) == 21
    # z (conv_in), the three Upsample inputs and the logits
    assert kinds.count(L_.OP_ROW_MASK) == 5 and ops[-1].kind == L_.OP_ROW_MASK and ops[-1].u.mask.x == res["out"].ptr
    assert ops[-1].u.mask.L == 8 * 96 and ops[-1].u.mask.valid == valid[8]
    assert ops[0].kind == L_.OP_ROW_MASK and ops[0].u.mask.x == res["inp"].ptr
    assert _check_masked_convs(ops, arena) > 10


def test_plans_without_lengths_are_unchanged(blob):
    """valid=None emits today's op lists, field for field (hashes of the plans compiled before ragged plans existed)"""
    cfg, b = blob
    comp = UNetCompiler(cfg.unet, b, 1 << 30)
    want = {(8, 512): "7ca81e628501890132bbf980e5645f86545e4c3eeb48aae468995a5eea4816cd",
            (2, 96): "ec77cfd9f7afb8773494f2c4ec05d6ac29ad014b3e95f5c39e72c6380890c619"}
    for (Beff, Lz), h in want.items():
        res = comp.compile(Arena(1 << 32), Beff, Lz, _ext(comp, Beff, Lz), False, None, None)
        assert len(res["ops"].ops) == 329
        assert hashlib.sha256(bytes(res["ops"].array())).hexdigest() == h
    res = DecoderCompiler(cfg.decoder, b, 1 << 30).compile(Arena(1 << 32), 4, 512, None)
    assert hashlib.sha256(bytes(res["ops"].array())).hexdigest() == "9ea4b1a1de279ffe670f8da2a37b59afdb2c4917952c856a170bd915de2ab8c4"


# ---- C ABI ---------------------------------------------------------------------------------------------------------------------
def test_abi_new_op_kinds_layout(tmp_path):
    assert L_.ABI_VERSION == 13 and C.sizeof(L_.Op) == 256
    assert (L_.OP_GROUPNORM_VAR, L_.OP_ATTENTION_VAR, L_.OP_ROW_MASK) == (14, 15, 16)
    structs = {"mugd_groupnorm_var": L_.GroupNormVar, "mugd_attention_var": L_.AttentionVar, "mugd_row_mask": L_.RowMask}
    src = tmp_path / "layout.c"
    body = "".join(f'  printf("%zu", sizeof({n}));\n' + "".join(f'  printf(" %zu", offsetof({n}, {f}));\n' for f, _ in t._fields_)
                   + '  printf("\\n");\n' for n, t in structs.items())
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "mugd.h"\nint main(void) {\n'
                   '  printf("%zu %d %d %d\\n", sizeof(mugd_op), MUGD_OP_GROUPNORM_VAR, MUGD_OP_ATTENTION_VAR, MUGD_OP_ROW_MASK);\n'
                   + body + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src), "-I" + os.path.join(ROOT, "include")], check=True)
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert lines[0].split() == ["256", "14", "15", "16"]
    for line, t in zip(lines[1:], structs.values()):
        assert [int(v) for v in line.split()] == [C.sizeof(t)] + [getattr(t, f).offset for f, _ in t._fields_]


def test_abi_sizes_accepts_13_and_reports_the_new_descriptors():
    lib = L_.load()
    assert lib.mugd_abi_version() == 13
    sizes = (C.c_int32 * 16)(*([-1] * 16))
    assert lib.mugd_abi_sizes(sizes, 13) == 0 and sizes[0] == 256 and list(sizes[13:]) == [-1, -1, -1]
    assert lib.mugd_abi_sizes(sizes, 12) != 0
    assert lib.mugd_abi_sizes(sizes, 16) == 0
    assert list(sizes[13:]) == [C.sizeof(L_.GroupNormVar), C.sizeof(L_.AttentionVar), C.sizeof(L_.RowMask)] == [80, 120, 40]


# ---- refusals before any GPU work ------------------------------------------------------------------------------------------------
class _NoGpu:
    def __getattr__(self, name):
        raise AssertionError(f"engine.{name} used before the refusal")


def _cpu(cls):
    s = object.__new__(cls)
    s.model = types.SimpleNamespace(engine=_NoGpu(), z_channels=16, z_length=96, num_timesteps=1000, cfg=ModelConfig(),
                                    clip_denoised=True, **register_schedule())
    s.ddpm_num_timesteps, s.device, s.last_launches_per_step = 1000, torch.device("cpu"), 0
    return s


def _req(**kw):
    inp = synth.synthetic_inputs(2, 96)
    out = dict(c=inp["c"], w=inp["w"], batch_size=2, shape=(16, 96), verbose=False, unconditional_guidance_scale=5.0,
               unconditional_conditioning=inp["uc"])
    out.update(kw)
    return out


X0 = torch.zeros(2, 16, 96)
MASK = torch.ones(2, 1, 96)
SAMPLE = {
    "ddim": lambda **kw: _cpu(DDIMSampler).sample(S=10, **_req(**kw)),
    "plms": lambda **kw: _cpu(PLMSSampler).sample(S=10, **_req(**kw)),
    "ddpm": lambda **kw: _cpu(DDPMSampler).sample(**_req(**kw)),
    "dpm": lambda **kw: _cpu(DPMSolverSampler).sample(S=10, **_req(**kw)),
    "unipc": lambda **kw: _cpu(UniPCSampler).sample(S=10, **_req(**kw)),
}
BAD_LENGTHS = [([64, 80], "multiple of 32"), ([64, 128], r"\[32, 96\]"), ([0, 64], r"\[32, 96\]"), ([64], "1 entries for 2 charts"),
               ([64, 64, 64], "3 entries"), (64, "one length per chart"), ([64.0, 64], "multiple of 32"), ([True, 64], "multiple of 32")]


@pytest.mark.parametrize("which", sorted(SAMPLE))
@pytest.mark.parametrize("lens,msg", BAD_LENGTHS, ids=[f"bad{i}" for i in range(len(BAD_LENGTHS))])
def test_samplers_refuse_bad_lengths_before_any_gpu_work(which, lens, msg):
    with pytest.raises(L_.MugdError, match=msg):
        SAMPLE[which](z_lengths=lens)


@pytest.mark.parametrize("which,kw,msg", [
    ("ddim", dict(mask=MASK, x0=X0), "inpainting"), ("plms", dict(mask=MASK, x0=X0), "inpainting"),
    ("ddim", dict(noise_dropout=0.1), "noise_dropout"), ("plms", dict(noise_dropout=0.1), "noise_dropout"),
    ("ddim", dict(match_reference_rng=True), "match_reference_rng"), ("plms", dict(match_reference_rng=True), "match_reference_rng")])
def test_samplers_refuse_flows_a_ragged_request_cannot_take(which, kw, msg):
    with pytest.raises(L_.MugdError, match=msg):
        SAMPLE[which](z_lengths=[64, 96], **kw)


def test_flows_from_an_existing_chart_refuse_lengths():
    from mug_diffusion_b200 import dist, dpm_solver, unipc
    from mug_diffusion_b200.sampler import alphas_cumprod_f64
    acp = alphas_cumprod_f64(ModelConfig())
    ddim = _cpu(DDIMSampler)
    ddim.make_schedule(10, verbose=False)
    dsch, usch = dpm_solver.multistep_schedule(acp, 10, 2), unipc.multistep_schedule(acp, 10, 2)
    dpm, uni = _cpu(DPMSolverSampler), _cpu(UniPCSampler)
    inp = synth.synthetic_inputs(2, 96)
    c, w = inp["c"], inp["w"]
    calls = [lambda: ddim.stochastic_encode(X0, torch.tensor([1, 2]), z_lengths=[64, 96]),
             lambda: dpm.stochastic_encode(X0, 3, dsch, z_lengths=[64, 96]),
             lambda: uni.stochastic_encode(X0, 3, usch, z_lengths=[64, 96]),
             lambda: ddim.decode(X0, c, w, 3, z_lengths=[64, 96]),
             lambda: dpm.decode(X0, c, w, 3, dsch, z_lengths=[64, 96]),
             lambda: uni.decode(X0, c, w, 3, usch, z_lengths=[64, 96]),
             lambda: ddim.invert(X0, c, w, 3, z_lengths=[64, 96]),
             lambda: dpm.invert(X0, c, w, 3, dsch, z_lengths=[64, 96]),
             lambda: uni.invert(X0, c, w, 3, usch, z_lengths=[64, 96]),
             lambda: dist.sample_sharded(None, None, {}, torch.device("cpu"), z_lengths=[64, 96])]
    for call in calls:
        with pytest.raises(L_.MugdError, match="z_lengths"):
            call()


def test_lengths_that_are_all_lmax_take_todays_path():
    assert ragged_lengths(None, 2, 96) is None and ragged_lengths([96, 96], 2, 96) is None
    assert ragged_lengths(torch.tensor([64, 96]), 2, 96) == [64, 96]
    # valid lengths pass every check: the request then needs the engine (here: the stand-in raises)
    for which in SAMPLE:
        with pytest.raises(AssertionError, match="engine"):
            SAMPLE[which](z_lengths=[32, 96], seeds=[5, 6])


# ---- pad_features --------------------------------------------------------------------------------------------------------------
def test_pad_features_shapes_and_zero_tails():
    songs = []
    for L, b in ((64, 1), (96, 2), (32, 1)):
        f = [None] * 6 + [torch.randn(b, ch, L >> l) + 1.0 for l, ch in enumerate((16, 32, 64, 128))]
        songs.append(f)
    w, lens = audio.pad_features(songs)
    assert lens == [64, 96, 96, 32]
    assert w[:6] == [None] * 6
    for l, ch in enumerate((16, 32, 64, 128)):
        t = w[6 + l]
        assert t.shape == (4, ch, 96 >> l)
        assert torch.equal(t[0, :, :64 >> l], songs[0][6 + l][0]) and torch.all(t[0, :, 64 >> l:] == 0)
        assert torch.equal(t[1:3], songs[1][6 + l])
        assert torch.equal(t[3, :, :32 >> l], songs[2][6 + l][0]) and torch.all(t[3, :, 32 >> l:] == 0)
    with pytest.raises(ValueError):
        audio.pad_features([songs[0], songs[1][:-1]])
    with pytest.raises(ValueError):
        audio.pad_features([])
