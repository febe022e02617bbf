"""Generate tests/golden/sections_*.npz by running the UNMODIFIED reference (/root/reference, CPU fp32, via tools/ref_shim.py) on the
seeded synthetic weights and inputs of mug_diffusion_b200.synth, with section prompts (DESIGN §6b N20): while a case runs, the
reference's own CrossAttention.forward (mug/model/attention.py:91-126) is called once per section slot with that slot's context and
the slot's rows are kept (tests/section_oracle.section_rule); every other module runs unchanged.  Self-attention (context None) is
untouched.

Cases (tests/section_cases.py): one CFG U-Net evaluation at L = 96, B = 2 (batch [uc half, c half], chart 0 changing prompt at
latent frames 32 and 64, chart 1 at 8), and the DDIM S = 10, CFG 5 trajectory of the same request with its decoded logits.

Run in the build container only (the GPU box has no /root/reference):
    python tools/make_section_goldens.py [out_dir]
"""
import contextlib
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import make_goldens as mg  # noqa: E402
import section_cases as sc  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from section_oracle import section_rule  # noqa: E402


@contextlib.contextmanager
def reference_sections(layouts):
    """the reference's CrossAttention.forward with the section rule for batches of 2B samples (uc half without sections)"""
    from mug.model.attention import CrossAttention
    orig = CrossAttention.forward
    lay = [[]] * len(layouts) + list(layouts)

    def forward(self, x, context=None, mask=None):
        if context is None or x.shape[0] != len(lay):
            return orig(self, x, context, mask)
        return section_rule(lambda xx, cc: orig(self, xx, cc, mask), x, context, lay, sc.L)

    CrossAttention.forward = forward
    try:
        yield
    finally:
        CrossAttention.forward = orig


@torch.no_grad()
def make(out_dir):
    mg.GOLD = out_dir
    inp = synth.synthetic_inputs(sc.B, sc.L)
    w = synth.wave_list(inp["w"])
    lay = sc.layouts()
    model, _ = mg.fresh_model(sc.L)
    from mug.diffusion.ddim import DDIMSampler          # importable once ref_shim has put the reference on the path
    t = torch.tensor(sc.T_EVAL * 2, dtype=torch.long)
    with reference_sections(lay):
        eps = model.model.forward(torch.cat([inp["x_T"]] * 2), t, torch.cat([inp["uc"], inp["c"]]),
                                  [torch.cat([wi, wi]) if wi.numel() else wi for wi in w])
    mg.save(sc.EVAL_NAME, eps=eps.numpy())
    model, _ = mg.fresh_model(sc.L)
    model.z_length = sc.L
    t0 = time.time()
    with reference_sections(lay):
        z, _ = DDIMSampler(model).sample(S=sc.S, c=inp["c"], w=w, batch_size=sc.B, shape=None, verbose=False, x_T=inp["x_T"],
                                         eta=0.0, unconditional_guidance_scale=sc.SCALE, unconditional_conditioning=inp["uc"])
    logits = model.model.decode(z)
    print(sc.DDIM_NAME, "ref sample+decode %.2fs" % (time.time() - t0))
    mg.save(sc.DDIM_NAME, z=z.numpy(), logits=logits.numpy())


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    out = sys.argv[1] if len(sys.argv) > 1 else mg.GOLD
    os.makedirs(out, exist_ok=True)
    make(out)
