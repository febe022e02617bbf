"""Generate tests/golden/plms_*.npz by running the UNMODIFIED reference PLMS sampler (/root/reference/mug/diffusion/plms.py, CPU
fp32, via tools/ref_shim.py) on the seeded synthetic weights and inputs of mug_diffusion_b200.synth.

plms.py is dead code in the reference for three mechanical reasons; this script bridges them without touching its arithmetic:
  1. it imports ``ldm.modules.diffusionmodules.util``, which does not exist: aliased to ``mug.diffusion.utils`` (the same three
     functions with the same signatures);
  2. ``PLMSSampler.register_buffer`` moves every tensor to CUDA: patched to keep them where they are (CPU);
  3. it calls ``model.apply_model(x, t, c)``, which has no audio argument: ``Adapter`` passes the audio the way ddim.py:170-174 does
     (``[cat(wi, wi)]`` when x carries both CFG halves) to ``model.model.forward``.
``sample()`` unpacks an image shape ``C, H, W``, so make_schedule and plms_sampling are called directly.

The reference's coefficients are ``[b, 1, 1, 1]`` tensors (plms.py:201-204): from the first update on, x is ``[B, B, C, L]`` with B
equal copies of the ``[B, C, L]`` latent (row k of the CFG batch ``cat([x] * 2)`` holds it at ``[k, k mod B]``).  The adapter hands
the U-Net that latent; the stored x_inter / pred_x0 / z are copy 0.

Run in the build container only (the GPU box has no /root/reference):
    python tools/make_plms_goldens.py
"""
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import plms_cases as pc  # noqa: E402
from make_goldens import GOLD, fresh_model, save  # noqa: E402
import ref_shim  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402


def import_reference_plms():
    ref_shim.install_shims()
    import mug.diffusion.utils as mug_utils
    for name in ("ldm", "ldm.modules", "ldm.modules.diffusionmodules"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["ldm.modules.diffusionmodules.util"] = mug_utils
    from mug.diffusion import plms
    plms.PLMSSampler.register_buffer = lambda self, name, attr: setattr(self, name, attr)
    return plms.PLMSSampler


def latent(x: torch.Tensor) -> torch.Tensor:
    """the [B, C, L] latent of the reference's x ([B, B, C, L] after the first update, its B copies equal)"""
    if x.dim() == 3:
        return x
    assert all(torch.equal(x[0], x[k]) for k in range(x.shape[0]))
    return x[0]


class Adapter:
    """The model object plms.py expects, over a reference DDPM and the request's audio features."""

    def __init__(self, ddpm, w):
        self.ddpm, self.w = ddpm, w
        self.num_timesteps = ddpm.num_timesteps
        self.betas, self.alphas_cumprod, self.alphas_cumprod_prev = ddpm.betas, ddpm.alphas_cumprod, ddpm.alphas_cumprod_prev
        self.device = torch.device("cpu")

    def q_sample(self, x_start, t, noise=None):
        return self.ddpm.q_sample(x_start, t, noise)

    def apply_model(self, x, t, c):
        if x.dim() == 4:
            k = torch.arange(x.shape[0])
            x = x[k, k % x.shape[1]]
        B = self.w[-1].shape[0]
        w_in = self.w if x.shape[0] == B else [torch.cat([wi, wi]) if wi.numel() else wi for wi in self.w]
        return self.ddpm.model.forward(x, t, c, w_in)


@torch.no_grad()
def make_plms():
    PLMSSampler = import_reference_plms()
    for name, case in pc.PLMS_CASES.items():
        model, _ = fresh_model(case["L"])
        model.z_length = case["L"]
        inp = synth.synthetic_inputs(case["B"], case["L"])
        sampler = PLMSSampler(Adapter(model, synth.wave_list(inp["w"])))
        sampler.make_schedule(ddim_num_steps=case["S"], ddim_eta=0.0, verbose=False)
        t0 = time.time()
        z, inter = sampler.plms_sampling(inp["c"], (case["B"], 16, case["L"]), x_T=inp["x_T"], log_every_t=pc.LOG_EVERY_T,
                                         unconditional_guidance_scale=case["scale"], unconditional_conditioning=inp["uc"])
        z = latent(z)
        logits = model.model.decode(z)
        print(name, "ref sample+decode %.2fs" % (time.time() - t0))
        out = dict(z=z.numpy(), logits=logits.numpy())
        for key in ("x_inter", "pred_x0"):
            for k, v in enumerate(inter[key]):
                out[f"{key}_{k}"] = latent(v).numpy()
        save(name, **out)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    make_plms()
