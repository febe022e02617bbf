"""Audio encoder (SURVEY §8f N1): oracle vs the reference's outputs (CPU), plan bookkeeping (CPU), GPU encoder vs golden
and the whole request path mel -> encoder -> DDIM -> decode -> notes on the GPU."""
import os

import pytest
import torch

import golden_cases as gc
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth, wave
from oracle import wave_oracle as worc


def rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / b.abs().max())


@pytest.fixture(scope="module")
def gold(golden_dir):
    return gc.load_golden(os.path.join(golden_dir, "wave_T6144_B2.npz"))


def test_wave_param_names_and_count():
    specs = wave.wave_param_specs(wave.WaveConfig())
    assert len(specs) == 364                                    # reference state_dict entries under model.wave_model.
    n = 0
    for shape, _ in specs.values():
        k = 1
        for s in shape:
            k *= s
        n += k
    assert n == 49392192                                        # 49.4 M parameters (SURVEY §2)


def test_wave_oracle_vs_reference(gold):
    sd = wave.synthetic_wave_state_dict()
    with torch.no_grad():
        hs = worc.wave_forward(sd, wave.synthetic_mel(2, 64 * 96))
    assert [tuple(h.shape[1:]) for h in hs[6:]] == [(256, 96), (512, 48), (512, 24), (512, 12)]
    for i in range(6, 10):
        assert gold[f"h{i}"].abs().max() > 0.1
        assert rel(hs[i], gold[f"h{i}"]) < 2e-5


def test_wave_plan_compiles():
    from mug_diffusion_b200.engine import Arena
    from mug_diffusion_b200.packer import WeightBlob
    cfg = wave.WaveConfig()
    blob = WeightBlob()
    wave.pack_wave(blob, wave.synthetic_wave_state_dict(cfg), cfg)
    blob.finalize()
    res = wave.WaveCompiler(cfg, blob, 1 << 30).compile(Arena(1 << 32), 2, 6144)
    kinds = [o.kind for o in res["ops"].ops]
    assert kinds.count(L_.OP_ATTENTION) == 12 and kinds.count(L_.OP_GROUPNORM) == 40 + 6
    assert [(c, l) for _, c, l in res["outs"]][6:] == [(256, 96), (512, 48), (512, 24), (512, 12)]
    dil = sorted({o.u.gemm.tap_dilation for o in res["ops"].ops if o.kind == L_.OP_GEMM and o.u.gemm.conv_mode == L_.CONV_TAPS})
    assert dil == [1, 2, 4, 8]


def _wave_vs_reference(gold, impl):
    from mug_diffusion_b200.sampler import MugDiffusionB200
    sd = {**synth.synthetic_state_dict(96), **wave.synthetic_wave_state_dict()}
    m = MugDiffusionB200.from_state_dict(sd, z_length=96, gemm_impl=impl)
    hs = m.model.wave_model(wave.synthetic_mel(2, 64 * 96).cuda())
    assert len(hs) == 10 and all(h is None for h in hs[:6])
    for i in range(6, 10):
        e = rel(hs[i], gold[f"h{i}"])
        print(f"audio encoder {impl} h{i} rel_err={e:.2e}")
        assert e < 1e-4


@pytest.mark.gpu
def test_gpu_wave_encoder_vs_reference(gold):
    _wave_vs_reference(gold, "auto")


@pytest.mark.gpu
def test_gpu_wave_encoder_simt_vs_reference(gold):
    """every GEMM of the audio encoder on the exact-fp32 FFMA kernel (dilated taps, Downsample, residuals): same tolerance"""
    _wave_vs_reference(gold, "simt")


@pytest.mark.gpu
def test_gpu_request_path_mel_to_hit_objects():
    """webui.startMapping's tensor path (webui.py:360-390) with every stage on the GPU: mel -> wave encoder -> DDIM
    sampler (CFG) -> decoder -> note extraction, compared with the CPU oracle chain on the same inputs"""
    from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200
    from oracle import mug_oracle as orc
    L, B, S = 96, 1, 4
    sd = {**synth.synthetic_state_dict(L), **wave.synthetic_wave_state_dict()}
    inp = synth.synthetic_inputs(B, L)
    mel = wave.synthetic_mel(B, 64 * L, seed=77)
    m = MugDiffusionB200.from_state_dict(sd, z_length=L)
    w = m.model.wave_model(mel.cuda())
    z, _ = DDIMSampler(m).sample(S=S, c=inp["c"].cuda(), w=w, batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
                                 unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    lines = m.model.decode_to_hit_objects(z, 46.439909297052154)
    with torch.no_grad():
        w_ref = worc.wave_forward(sd, mel)[-4:]
        z_ref = orc.ddim_sample(sd, S, inp["c"], w_ref, inp["x_T"], scale=5.0, uc=inp["uc"])
        lg_ref = orc.decoder_forward(sd, z_ref)
    assert rel(z, z_ref) < 1e-3
    ref_lines = orc.array_to_objects(lg_ref[0].numpy(), 4, 46.439909297052154)
    assert len(set(lines[0]) & set(ref_lines)) >= 0.97 * len(ref_lines)


@pytest.mark.gpu
def test_gpu_wave_encoder_three_minute_audio_vs_live_oracle():
    """the 3-minute shape the sampler's headline config runs on (T = 64 * 512 = 32768 mel frames -> w[-4:] at 512/256/128/64),
    against the live CPU oracle (itself pinned to the reference at T = 6144)"""
    from mug_diffusion_b200.sampler import MugDiffusionB200
    T = 64 * 512
    sd = {**synth.synthetic_state_dict(512), **wave.synthetic_wave_state_dict()}
    mel = wave.synthetic_mel(1, T, seed=5)
    m = MugDiffusionB200.from_state_dict(sd, z_length=512)
    hs = m.model.wave_model(mel.cuda())
    with torch.no_grad():
        ref = worc.wave_forward(sd, mel)
    assert [tuple(h.shape) for h in hs[6:]] == [(1, 256, 512), (1, 512, 256), (1, 512, 128), (1, 512, 64)]
    for i in range(6, 10):
        assert rel(hs[i], ref[i]) < 1e-4
