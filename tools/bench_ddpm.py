"""DDPM (all T = 1000 ancestral steps) vs DDIM (S = 50) steps per second at the headline shape (L = 512, B = 4, CFG 5), both from
their one-call device loops.

    python tools/bench_ddpm.py [--reps 3] [--warmup 1] [--S 50]

First, outputs: the DDPM device loop's latent must equal the per-step loop's (forced with a callback) bit for bit from the same seed.
Then ``--warmup`` untimed requests of each sampler, a sustain phase of at least 1 s, then ``--reps`` timed requests of each, the two
samplers alternating; each is timed with CUDA events around one sampler.sample call.  A step is one iteration of the sampler's loop
(one batched U-Net evaluation).  The host time spent in draw_step_noise (enqueueing the step noise on the device's generator) is
summed per DDPM request.  Prints one JSON line: the median steps/s and request time of each, the launches per step, the noise time, and
the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_staged import card  # noqa: E402
from mug_diffusion_b200 import sampler as sampler_mod  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, DDPMSampler, MugDiffusionB200  # noqa: E402

noise_host_s = [0.0]
_draw = sampler_mod.draw_step_noise


def timed_draw(*a, **k):
    t0 = time.perf_counter()
    _draw(*a, **k)
    noise_host_s[0] += time.perf_counter() - t0


sampler_mod.draw_step_noise = timed_draw


def timed(sample, kw):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    noise_host_s[0] = 0.0
    e0.record()
    z, _ = sample(**kw)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 1000.0, z, noise_host_s[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--S", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ddpm needs a CUDA device")
    info = card()
    L, B, scale = 512, 4, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    kw = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), shape=(16, L),
              unconditional_guidance_scale=scale, unconditional_conditioning=inp["uc"].cuda())
    ddpm, ddim = DDPMSampler(model), DDIMSampler(model)
    samplers = {"ddpm": (ddpm.sample, kw), "ddim": (ddim.sample, dict(kw, S=a.S))}

    zs = []
    for cb in (None, lambda i: None):
        torch.cuda.manual_seed(1)
        zs.append(ddpm.sample(callback=cb, **kw)[0])
    same = torch.equal(zs[0], zs[1])
    if not same:
        raise SystemExit("DDPM: the device loop and the per-step loop disagree")

    for _ in range(a.warmup):
        for fn, k in samplers.values():
            timed(fn, k)
    t_end = time.perf_counter() + 1.0                                           # sustain phase
    while time.perf_counter() < t_end:
        for fn, k in samplers.values():
            timed(fn, k)
    times = {n: [] for n in samplers}
    noise_s = []
    for _ in range(a.reps):
        for n, (fn, k) in samplers.items():
            if n == "ddpm":
                torch.cuda.manual_seed(1)
            t, z, ns = timed(fn, k)
            times[n].append(t)
            if n == "ddpm":
                noise_s.append(ns)
                if not torch.equal(z, zs[0]):
                    raise SystemExit("DDPM: a timed request changed its result")
    steps = {"ddpm": model.num_timesteps, "ddim": len(ddim.ddim_timesteps)}
    row = dict(L=L, B=B, cfg=scale, T=model.num_timesteps, S=a.S, reps=a.reps, outputs_equal=same, **info)
    for n, s in (("ddpm", ddpm), ("ddim", ddim)):
        row[f"{n}_steps_per_s"] = round(steps[n] / statistics.median(times[n]), 2)
        row[f"{n}_request_ms"] = round(1000 * statistics.median(times[n]), 2)
        row[f"{n}_launches_per_step"] = s.last_launches_per_step
    row["ddpm_over_ddim_per_step"] = round(row["ddpm_steps_per_s"] / row["ddim_steps_per_s"], 4)
    row["ddpm_noise_host_ms_per_request"] = round(1000 * statistics.median(noise_s), 2)
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
