"""The section-prompt golden cases shared by tools/make_section_goldens.py (which runs the UNMODIFIED reference with its
CrossAttention.forward applied once per section, tests/section_oracle.py's rule) and the tests that replay them.  Inputs come from
the seeds of mug_diffusion_b200.synth; only reference outputs are stored."""
import torch

from mug_diffusion_b200 import synth

L, B = 96, 2
T_EVAL = [981, 1]                    # the U-Net evaluation's timestep of each chart (both CFG halves)
S, SCALE = 10, 5.0                   # the DDIM trajectory


def section_prompts():
    """three prompts drawn like c (synthetic_inputs of another seed), [context_dim, T] each"""
    return list(synth.synthetic_inputs(3, L, seed=20)["c"])


def layouts():
    """chart 0 changes prompt at latent frames 32 and 64, chart 1 at 8: [(start, context)] per chart"""
    p = section_prompts()
    return [[(32, p[0]), (64, p[1])], [(8, p[2])]]


EVAL_NAME = "sections_unet_L96_B2_cfg"
DDIM_NAME = "sections_ddim_L96_B2_S10_cfg5"
