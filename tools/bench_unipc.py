"""UniPC against DPM-Solver++ 2M and DDIM at the headline shape (L = 512, B = 4, CFG 5), each from its one-call device loop.

    python tools/bench_unipc.py [--reps 3] [--warmup 2]
    python tools/bench_unipc.py --convergence

Timing rows: UniPC-2 (bh2) at S = 5, 8, 10, 15; DPM++ 2M at S = 10, 15, 20; DDIM at S = 50.  First, outputs: the UniPC device loop's
latent must equal its per-step loop's (forced with a callback) bit for bit.  Then ``--warmup`` untimed requests of every row, a sustain
phase of at least 1 s, then ``--reps`` timed rounds with the rows alternating, each request timed with CUDA events around one
sampler.sample call; the median is reported.  Prints one JSON line: per row the request time, the time per step and the launches per
step, and the card's name, power limit and max SM clock read in the same run.

``--convergence``: solver accuracy on the synthetic (untrained) network, NOT chart quality: the max-abs distance of the final latent
from DDIM through all 1000 timesteps of the same request, for UniPC orders 2 and 3 (bh1 and bh2) and DPM++ 2M at S = 5, 8, 10, 15, 20.
One JSON line.  Needs a CUDA device.
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
from mug_diffusion_b200.dpm_solver import NoiseScheduleVP  # noqa: E402
from mug_diffusion_b200.sampler import (DDIMSampler, DPMSolverSampler, MugDiffusionB200, UniPCSampler, alphas_cumprod_f64,  # noqa: E402
                                        ddim_timesteps_uniform)


def timed(sampler, kw):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    z, _ = sampler.sample(**kw)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), z


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--convergence", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_unipc needs a CUDA device")
    info = card()
    L, B, scale = 512, 4, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    base = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(),
                shape=(16, L), unconditional_guidance_scale=scale, unconditional_conditioning=inp["uc"].cuda())
    uni, dpm, ddim = UniPCSampler(model), DPMSolverSampler(model), DDIMSampler(model)

    if a.convergence:
        # DDIM through every one of the 1000 timesteps: order 1 on the grid of all nodes (999 steps from t = 1 to 1/N) is DDIM's update
        # (tests/test_dpm_solver.py); DDIMSampler itself cannot take S = 1000, whose uniform schedule reaches timestep 1000
        fine = dpm.make_dpm_schedule(999, 1, t_grid=NoiseScheduleVP(alphas_cumprod_f64(model.cfg)).t_array[::-1])
        z_ref, _ = dpm.dpm_sampling(base["w"], base["c"], (B, 16, L), fine, x_T=base["x_T"], unconditional_guidance_scale=scale,
                                    unconditional_conditioning=base["unconditional_conditioning"], progress=False)
        row = dict(L=L, B=B, cfg=scale, reference="ddim_all_1000_timesteps", weights="synthetic (untrained)", **info)
        for S in (5, 8, 10, 15, 20):
            for order in (2, 3):
                for variant in ("bh1", "bh2"):
                    z = uni.sample(S=S, order=order, variant=variant, **base)[0]
                    row[f"unipc{order}_{variant}_S{S}"] = float((z - z_ref).abs().max())
            row[f"dpm2m_S{S}"] = float((dpm.sample(S=S, order=2, **base)[0] - z_ref).abs().max())
        print(json.dumps(row), flush=True)
        return

    zs = [uni.sample(S=10, callback=cb, **base)[0] for cb in (None, lambda i: None)]
    if not torch.equal(zs[0], zs[1]):
        raise SystemExit("UniPC: the device loop and the per-step loop disagree")

    rows = {f"unipc2_bh2_S{S}": (uni, dict(S=S, order=2, variant="bh2", **base), S) for S in (5, 8, 10, 15)}
    rows.update({f"dpm2m_S{S}": (dpm, dict(S=S, order=2, **base), S) for S in (10, 15, 20)})
    rows["ddim_S50"] = (ddim, dict(S=50, **base), 50)
    for _ in range(a.warmup):
        for s, kw, _ in rows.values():
            timed(s, kw)
    t_end = time.perf_counter() + 1.0                                           # sustain phase
    while time.perf_counter() < t_end:
        for s, kw, _ in rows.values():
            timed(s, kw)
    times = {n: [] for n in rows}
    launches = {}
    for _ in range(a.reps):
        for n, (s, kw, _) in rows.items():
            t, z = timed(s, kw)
            times[n].append(t)
            launches[n] = s.last_launches_per_step
            if n == "unipc2_bh2_S10" and not torch.equal(z, zs[0]):
                raise SystemExit("UniPC: a timed request changed its result")
    out = dict(L=L, B=B, cfg=scale, reps=a.reps, outputs_equal=True, **info)
    for n, (s, kw, S) in rows.items():
        ms = statistics.median(times[n])
        steps = S if s is not ddim else len(ddim_timesteps_uniform(S, 1000))    # DDIM runs len(range(0, 1000, 1000 // S)) steps
        out[n] = dict(request_ms=round(ms, 2), steps=steps, ms_per_step=round(ms / steps, 3), launches_per_step=launches[n])
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
