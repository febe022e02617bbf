"""Generate the long-song goldens of tests/long_cases.py (tests/golden/unet_L2048_*.npz, ddim_L1600_B1_S4_cfg5.npz) by running the
UNMODIFIED reference on the CPU in fp32 through tools/ref_shim.py, on the seeded synthetic weights and inputs of
mug_diffusion_b200.synth -- the recipe of tools/make_goldens.py (`unet`, `ddim`, and `s4len` for the persisted-length case).

Needs a reference checkout (MUG_REFERENCE_ROOT):
    python tools/make_long_goldens.py [--only unet|ddim]
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import long_cases as lc  # noqa: E402
from make_goldens import fresh_model, save  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402


@torch.no_grad()
def make_unet():
    for name, case in lc.LONG_UNET_CASES.items():
        model, _ = fresh_model(case["persisted"] or case["L"])
        inp = synth.synthetic_inputs(case["B"], case["L"])
        t0 = time.time()
        eps = model.model.forward(inp["x_T"], torch.tensor(case["t"], dtype=torch.long), inp["c"], synth.wave_list(inp["w"]))
        print(name, "ref eval %.1fs" % (time.time() - t0))
        save(name, eps=eps.numpy())


@torch.no_grad()
def make_ddim():
    from mug.diffusion.ddim import DDIMSampler

    for name, case in lc.LONG_DDIM_CASES.items():
        model, _ = fresh_model(case["L"])
        model.z_length = case["L"]
        inp = synth.synthetic_inputs(case["B"], case["L"])
        sampler = DDIMSampler(model)
        pred = []
        t0 = time.time()
        z, _ = sampler.sample(S=case["S"], c=inp["c"], w=synth.wave_list(inp["w"]), batch_size=case["B"], shape=None, verbose=False,
                              x_T=inp["x_T"], eta=0.0, unconditional_guidance_scale=case["scale"], unconditional_conditioning=inp["uc"],
                              img_callback=lambda p, i: pred.append(p.clone()))
        logits = model.model.decode(z)
        print(name, "ref sample+decode %.1fs" % (time.time() - t0))
        save(name, z=z.numpy(), logits=logits.numpy(), pred_x0_first=pred[0].numpy(), pred_x0_last=pred[-1].numpy())


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["unet", "ddim"])
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    if a.only in (None, "unet"):
        make_unet()
    if a.only in (None, "ddim"):
        make_ddim()
