"""Note extraction (SURVEY §8f N2): oracle restatement vs the reference's own hit-object lines (CPU), and the GPU kernel
through decode_to_hit_objects / the C ABI vs the oracle (gpu)."""
import json
import os

import numpy as np
import pytest
import torch

import golden_cases as gc
from oracle import mug_oracle as orc


@pytest.fixture(scope="module")
def gold(golden_dir):
    return json.load(open(os.path.join(golden_dir, "hit_objects.json")))


@pytest.mark.parametrize("name", ["ddim_L512_B1_S50_cfg5", "ddim_L96_B2_S10_cfg5"])
def test_oracle_hit_objects_equal_reference(name, gold, golden_dir):
    lg = gc.load_golden(os.path.join(golden_dir, name + ".npz"))["logits"].numpy()
    for b in range(lg.shape[0]):
        assert orc.array_to_objects(lg[b], 4, gold["frame_ms"]) == gold[name][b]
        assert len(gold[name][b]) > 50


def test_oracle_hit_objects_corner_cases(gold):
    syn = gc.synthetic_note_logits().numpy()
    for b in range(syn.shape[0]):
        assert orc.array_to_objects(syn[b], 4, gold["frame_ms"]) == gold["synthetic"][b]
    assert any(",128,0," in l for l in gold["synthetic"][1])      # long notes present


@pytest.mark.gpu
def test_gpu_note_kernel_equals_reference(gold):
    import ctypes as C
    from mug_diffusion_b200 import lib as L_
    from mug_diffusion_b200.engine import OpList
    from mug_diffusion_b200.runtime import hit_object_lines
    from gpu_util import OpRunner, nlc
    R = OpRunner()
    syn = gc.synthetic_note_logits()
    B, _, T = syn.shape
    lg = nlc(syn).cuda()
    cnt = torch.zeros(B, 4, dtype=torch.int32).cuda()
    st = torch.full((B, 4, T), -1, dtype=torch.int32).cuda()
    en = torch.full((B, 4, T), -1, dtype=torch.int32).cuda()
    d = L_.Notes()
    d.logits, d.ld, d.count, d.start_ms, d.end_ms = lg.data_ptr(), 16, cnt.data_ptr(), st.data_ptr(), en.data_ptr()
    d.frame_ms, d.B, d.T, d.K = gold["frame_ms"], B, T, 4
    ops = OpList()
    ops.add(L_.OP_NOTES, d)
    R.run(ops)
    lines = hit_object_lines(cnt.cpu(), st.cpu(), en.cpu(), 4)
    for b in range(B):
        assert lines[b] == gold["synthetic"][b]


@pytest.mark.gpu
def test_decode_to_hit_objects_end_to_end(gold, golden_dir):
    """z (reference golden latent) -> CUDA decoder -> GPU note extraction == reference decoder + reference convertor,
    except for notes whose deciding logit is within the logit tolerance of 0"""
    from mug_diffusion_b200 import synth
    from mug_diffusion_b200.sampler import MugDiffusionB200
    g = gc.load_golden(os.path.join(golden_dir, "ddim_L96_B2_S10_cfg5.npz"))
    m = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(96), z_length=96)
    mine = m.model.decode_to_hit_objects(g["z"].cuda(), gold["frame_ms"])
    ref = gold["ddim_L96_B2_S10_cfg5"]
    for b in range(2):
        same = len(set(mine[b]) & set(ref[b]))
        assert same >= 0.98 * len(ref[b]) and abs(len(mine[b]) - len(ref[b])) <= 0.02 * len(ref[b]) + 1
