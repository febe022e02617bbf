"""Time an inpainting + eta = 1 request through the per-step loop (forced with a callback) and through the device loop
(mugd_sample_staged), at two shapes: L=96, B=1 without guidance, and L=512, B=4 with CFG 5; S = 50 each.

    python tools/bench_staged.py [--reps 3]

Both loops are first checked to give the same z bit for bit from the same seed.  Then, best of ``--reps``: wall time of one
sampler.sample call ending in a device synchronise, as DDIM steps per second, and the host CPU time (process time) per step.  Prints
one JSON line per shape with the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + [None] * 3)[:3] if q.returncode == 0 else (torch.cuda.get_device_name(), None, None)
    return dict(gpu=name, power_limit_w=float(power) if power else None, sm_max_mhz=int(clock) if clock else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--S", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_staged needs a CUDA device")
    info = card()
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(512), z_length=512)
    sampler = DDIMSampler(model)
    for L, B, scale in ((96, 1, 1.0), (512, 4, 5.0)):
        inp = synth.synthetic_inputs(B, L)
        x0, mask = synth.synthetic_inpainting(B, L)
        kw = dict(S=a.S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), eta=1.0,
                  shape=(16, L), mask=mask.cuda(), x0=x0.cuda())
        if scale != 1.0:
            kw.update(unconditional_guidance_scale=scale, unconditional_conditioning=inp["uc"].cuda())
        paths = {"per_step": lambda i: None, "device_loop": None}
        zs = {}
        for name, cb in paths.items():
            torch.cuda.manual_seed(1)
            zs[name], _ = sampler.sample(callback=cb, **kw)               # also the warm-up of this shape
        same = torch.equal(zs["per_step"], zs["device_loop"])
        if not same:
            raise SystemExit(f"L={L} B={B}: the two loops disagree")
        steps = len(sampler.ddim_timesteps)
        best = {n: (float("inf"), float("inf")) for n in paths}
        for _ in range(a.reps):
            for name, cb in paths.items():                               # alternate the two loops
                torch.cuda.synchronize()
                t0, c0 = time.perf_counter(), time.process_time()
                sampler.sample(callback=cb, **kw)
                torch.cuda.synchronize()
                t, c = time.perf_counter() - t0, time.process_time() - c0
                best[name] = min(best[name], (t, c))
        row = dict(L=L, B=B, cfg=scale, S=a.S, steps=steps, eta=1.0, inpainting=True, outputs_equal=same, **info)
        for name, (t, c) in best.items():
            row[f"{name}_steps_per_s"] = round(steps / t, 2)
            row[f"{name}_host_cpu_ms_per_step"] = round(1000 * c / steps, 3)
        row["speedup"] = round(best["per_step"][0] / best["device_loop"][0], 3)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
