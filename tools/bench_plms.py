"""PLMS vs DDIM steps per second at the headline shape (L = 512, B = 4, CFG 5, S = 50), both from their one-call device loops.

    python tools/bench_plms.py [--reps 5] [--warmup 3] [--S 50]

First, outputs: the PLMS device loop's latent must equal the per-step loop's (forced with a callback) bit for bit from the same seed.
Then bench.py's protocol: ``--warmup`` untimed requests of each sampler, a sustain phase of at least 1 s, then ``--reps`` timed requests
of each, the two samplers alternating; each is timed with CUDA events around one sampler.sample call.  A step is one iteration of the
sampler's loop (one batched U-Net evaluation; PLMS evaluates twice at its first step).  Prints one JSON line: the median steps/s of
each, the launches per step, and the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
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
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200, PLMSSampler  # noqa: E402


def timed(sampler, kw):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    z, _ = sampler.sample(**kw)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 1000.0, z


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--S", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_plms needs a CUDA device")
    info = card()
    L, B, scale = 512, 4, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    kw = dict(S=a.S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
              shape=(16, L), unconditional_guidance_scale=scale, unconditional_conditioning=inp["uc"].cuda())
    samplers = {"plms": PLMSSampler(model), "ddim": DDIMSampler(model)}

    zs = []
    for cb in (None, lambda i: None):
        torch.cuda.manual_seed(1)
        zs.append(samplers["plms"].sample(callback=cb, **kw)[0])
    same = torch.equal(zs[0], zs[1])
    if not same:
        raise SystemExit("PLMS: the device loop and the per-step loop disagree")

    for _ in range(a.warmup):
        for s in samplers.values():
            timed(s, kw)
    t_end = time.perf_counter() + 1.0                                           # sustain phase
    while time.perf_counter() < t_end:
        for s in samplers.values():
            timed(s, kw)
    times = {n: [] for n in samplers}
    for _ in range(a.reps):
        for n, s in samplers.items():
            t, z = timed(s, kw)
            times[n].append(t)
            if n == "plms" and not torch.equal(z, zs[0]):
                raise SystemExit("PLMS: a timed request changed its result")
    steps = len(samplers["plms"].ddim_timesteps)
    row = dict(L=L, B=B, cfg=scale, S=a.S, steps=steps, reps=a.reps, outputs_equal=same, **info)
    for n, s in samplers.items():
        row[f"{n}_steps_per_s"] = round(steps / statistics.median(times[n]), 2)
        row[f"{n}_request_ms"] = round(1000 * statistics.median(times[n]), 2)
        row[f"{n}_launches_per_step"] = s.last_launches_per_step
    row["plms_over_ddim"] = round(row["plms_steps_per_s"] / row["ddim_steps_per_s"], 4)
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
