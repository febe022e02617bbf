"""Generate tests/golden/remix_*.npz by running the UNMODIFIED reference samplers with ``timesteps=k`` (the truncated schedule of
/root/reference/mug/diffusion/ddim.py:123-131 and plms.py:128-136, CPU fp32, via tools/ref_shim.py) on the seeded synthetic weights and
inputs of mug_diffusion_b200.synth.  The cases are tests/remix_cases.py's.  PLMS runs through make_plms_goldens.py's shims (an aliased
import, CPU buffers and an adapter that hands the U-Net the audio); DDIM runs as it is.

Run in the build container only (the GPU box has no /root/reference):
    python tools/make_remix_goldens.py
"""
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import remix_cases as rc  # noqa: E402
from make_goldens import GOLD, fresh_model, save  # noqa: E402
from make_plms_goldens import Adapter, import_reference_plms, latent  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402


class _Quiet:
    """tqdm_class stand-in: iterates without printing"""

    def __init__(self, it, **kw):
        self.it = it

    def __iter__(self):
        return iter(self.it)


@torch.no_grad()
def make_remix():
    PLMSSampler = import_reference_plms()                   # installs ref_shim's shims too
    from mug.diffusion.ddim import DDIMSampler
    for name, case in rc.REMIX_CASES.items():
        model, _ = fresh_model(case["L"])
        model.z_length = case["L"]
        inp = synth.synthetic_inputs(case["B"], case["L"])
        w = synth.wave_list(inp["w"])
        shape = (case["B"], 16, case["L"])
        t0 = time.time()
        if case["sampler"] == "ddim":
            sampler = DDIMSampler(model)
            sampler.make_schedule(ddim_num_steps=case["S"], ddim_eta=0.0, verbose=False)
            z, inter = sampler.ddim_sampling(w, inp["c"], shape, x_T=inp["x_T"], timesteps=case["k"], log_every_t=rc.LOG_EVERY_T,
                                             unconditional_guidance_scale=case["scale"], unconditional_conditioning=inp["uc"],
                                             tqdm_class=_Quiet)
        else:
            sampler = PLMSSampler(Adapter(model, w))
            sampler.make_schedule(ddim_num_steps=case["S"], ddim_eta=0.0, verbose=False)
            z, inter = sampler.plms_sampling(inp["c"], shape, x_T=inp["x_T"], timesteps=case["k"], log_every_t=rc.LOG_EVERY_T,
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
    make_remix()
