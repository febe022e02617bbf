"""Long songs on the CPU: the oracle against the reference's outputs past z_length 1568 (tests/golden/, made by
tools/make_long_goldens.py), webui's z_length rule at the boundaries that matter, and the z_length ceiling, which is refused on
the host before any GPU work."""
import os

import pytest
import torch

import golden_cases as gc
import long_cases as lc
from mug_diffusion_b200 import audio, s4_setup, synth
from mug_diffusion_b200 import lib as L_
from oracle import mug_oracle as orc


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def persisted_state_dict(L_persisted: int, L_request: int):
    """the synthetic weights persisted at L_persisted, with every S4 layer's C~ lengthened for L_request as the reference does on its
    first forward (s4.py:557-584)"""
    sd = dict(synth.synthetic_state_dict(L_persisted, decoder=False))
    for key in [k for k in sd if k.endswith("kernel.kernel.L")]:
        pre = key[:-1]
        ds = L_persisted // int(sd[key])
        params = {n: sd[pre + n] for n in ("C", "log_dt", "P", "inv_w_real", "w_imag")}
        sd[pre + "C"], L_new = s4_setup.lengthen(params, int(sd[key]), L_request // ds)
        sd[key] = torch.tensor(L_new)
    return sd


@pytest.mark.parametrize("name", list(lc.LONG_UNET_CASES))
def test_unet_eval_vs_reference(name, golden_dir):
    case = lc.LONG_UNET_CASES[name]
    L = case["L"]
    sd = persisted_state_dict(case["persisted"], L) if case["persisted"] else synth.synthetic_state_dict(L, decoder=False)
    if case["persisted"]:
        assert int(sd["model.unet_model.input_blocks.2.1.s4_model.kernel.kernel.L"]) == L    # 512 doubled twice
    inp = synth.synthetic_inputs(case["B"], L)
    with torch.no_grad():
        eps = orc.unet_forward(sd, inp["x_T"], torch.tensor(case["t"]), inp["c"], inp["w"])
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))["eps"]
    assert eps.shape == g.shape and g.abs().max() > 0.1
    assert rel_err(eps, g) < 1e-4


def test_ddim_vs_reference(golden_dir):
    name = "ddim_L1600_B1_S4_cfg5"
    case = lc.LONG_DDIM_CASES[name]
    sd = synth.synthetic_state_dict(case["L"])
    inp = synth.synthetic_inputs(case["B"], case["L"])
    with torch.no_grad():
        z = orc.ddim_sample(sd, case["S"], inp["c"], inp["w"], inp["x_T"], scale=case["scale"], uc=inp["uc"])
        logits = orc.decoder_forward(sd, z)
    g = gc.load_golden(os.path.join(golden_dir, name + ".npz"))
    assert rel_err(z, g["z"]) < 1e-3
    assert rel_err(logits, g["logits"]) < 1e-3
    mine, ref = orc.notes_from_logits(logits), orc.notes_from_logits(g["logits"])
    flips = mine != ref
    ref8 = torch.cat([g["logits"][:, 0:4], g["logits"][:, 8:12]], dim=1)
    assert bool((ref8[flips].abs() < 1e-3 * ref8.abs().max()).all())


@pytest.mark.parametrize("samples,z_length", [(12_844_927, 1568), (12_844_928, 1600), (67_108_735, 8192), (67_108_736, 8224)])
def test_z_length_for_at_the_boundaries(samples, z_length):
    """samples at 22,050 Hz -> webui's z_length: 1568 is the longest the resident S4 kernel takes, 8192 the supported maximum"""
    assert audio.z_length_for(audio.n_frames(samples, audio.MelConfig().hop_length)) == z_length


def test_max_samples_is_the_last_audio_within_the_ceiling():
    n = audio.max_samples()
    assert n == 67_108_735
    hop = audio.MelConfig().hop_length
    assert audio.z_length_for(audio.n_frames(n, hop)) == audio.MAX_Z_LENGTH
    assert audio.z_length_for(audio.n_frames(n + 1, hop)) > audio.MAX_Z_LENGTH


def test_z_length_ceiling_is_refused_without_a_device():
    for ok in (32, 1568, 1600, 8192):
        audio.check_z_length(ok)
    with pytest.raises(L_.MugdError, match=r"z_length 8224 .* maximum 8192.*67,108,735 samples at 22,050 Hz \(3043\.5 s"):
        audio.check_z_length(8224)
