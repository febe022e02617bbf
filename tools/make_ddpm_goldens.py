"""Generate tests/golden/ddpm_*.npz by running the UNMODIFIED reference DDPM sampler, ``DDPM.log_beatmap``
(mug/diffusion/diffusion.py:227-282, CPU fp32, via tools/ref_shim.py), on the seeded synthetic weights and inputs of
mug_diffusion_b200.synth.

log_beatmap is the reference's validation hook.  It runs with these wrappers only; its loop is not touched:
  * instance attributes ``model.model.wave_output`` / ``cond_output`` return the synthetic audio features ``w`` / prompt ``c``;
  * ``model.model.decode`` is wrapped to record each logged ``x`` (and return zeros, so nothing is decoded per log);
  * ``count=0``, so no chart file is written; ``log_index=1``, so the call samples (log_index % 5 == 2 after its increment);
  * ``torch.manual_seed(seed)`` before the call: x_T and the per-step noise are the CPU generator's draws.
``ddpm_L96_B2_T50`` first calls the reference's own ``register_schedule(timesteps=50)`` on the fresh model.

Each golden stores z (the x of i = 0), the logged x's in order, x_T, the decoder logits of z and the reference's float32 schedule
buffers.  The T = 1000 case takes about two minutes of CPU.

Run in the build container only (the GPU box has no reference checkout):
    python tools/make_ddpm_goldens.py
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ddpm_cases as dc  # noqa: E402
from make_goldens import GOLD, fresh_model, save  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402


@torch.no_grad()
def make_ddpm():
    for name, case in dc.DDPM_CASES.items():
        L, B, T = case["L"], case["B"], case["T"]
        model, _ = fresh_model(L)
        model.z_length = L
        if T != model.num_timesteps:
            model.register_schedule(timesteps=T)
        assert model.num_timesteps == T and model.parameterization == "eps" and model.clip_denoised
        model.log_every_t = case["log_every_t"]
        model.log_index = 1
        inp = synth.synthetic_inputs(B, L)
        w, c = synth.wave_list(inp["w"]), inp["c"]
        model.model.wave_output = lambda batch: w
        model.model.cond_output = lambda batch: c
        decode = model.model.decode
        logged = []

        def record(x):
            logged.append(x.clone())
            return torch.zeros(x.shape[0], 1, 1)

        model.model.decode = record
        batch = {"note": torch.zeros(B, 16, 8 * L), "valid_flag": torch.ones(B, 8 * L)}
        torch.manual_seed(case["seed"])
        t0 = time.time()
        model.log_beatmap(batch, count=0)
        z = logged[-1]
        logits = decode(z)
        print(name, "ref sample+decode %.1fs" % (time.time() - t0), len(logged), "logged")
        assert len(logged) == len(dc.logged_steps(T, case["log_every_t"]))
        x_T, _ = dc.cpu_noise(case["seed"], (B, 16, L), 0)
        out = dict(z=z.numpy(), x_T=x_T.numpy(), logits=logits.numpy())
        for k, v in enumerate(logged):
            out[f"x_inter_{k}"] = v.numpy()
        for key in dc.SCHEDULE_KEYS:
            out[f"sched_{key}"] = getattr(model, key).numpy()
        save(name, **out)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    os.makedirs(GOLD, exist_ok=True)
    make_ddpm()
