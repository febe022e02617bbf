"""DPM-Solver++ inpainting and remix against DDIM's at the headline shape (L = 512, B = 4, CFG 5), each from its one-call device loop.

    python tools/bench_dpm_remix.py [--reps 3] [--warmup 2]

Rows: DPM++ 2M inpainting at S = 15, 20, 25 and DDIM inpainting at S = 50 (the same mask and x0); DPM++ 2M ``decode`` at S = 20 with
t_start = S and with mixed strengths [1/4, 1/2, 3/4, 1] * S, and DDIM ``decode`` at S = 50 with t_start = 50 and the same mixed
fractions.  First, outputs: the DPM++ inpainting device loop's latent must equal its per-step loop's (forced with a callback) bit for
bit, and the mixed decode must equal its per-step referee.  Then ``--warmup`` untimed requests of every row, a sustain phase of at least
1 s, then ``--reps`` timed rounds with the rows alternating, each request timed with CUDA events around one sampler call; the median
is reported.  Prints one JSON line: per row the request time, the U-Net steps of the request (a mixed decode runs max(t_start)), the
time per step and the launches per step, and the card's name, power limit and max SM clock read in the same run.
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
from mug_diffusion_b200.sampler import DDIMSampler, DPMSolverSampler, MugDiffusionB200, ddim_timesteps_uniform  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dpm_remix needs a CUDA device")
    info = card()
    L, B, scale = 512, 4, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    x0, mask = (t.cuda() for t in synth.synthetic_inpainting(B, L))
    c, w, uc = inp["c"].cuda(), [t.cuda() for t in inp["w"]], inp["uc"].cuda()
    base = dict(c=c, w=w, batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), shape=(16, L), unconditional_guidance_scale=scale,
                unconditional_conditioning=uc)
    dpm, ddim = DPMSolverSampler(model), DDIMSampler(model)
    z_lat = inp["x_T"].cuda() * 0.5                                             # stands for an encoded chart: decode's input latent

    zs = []
    for cb in (None, lambda i: None):
        torch.cuda.manual_seed(5)
        zs.append(dpm.inpaint(20, mask=mask, x0=x0, order=2, callback=cb, **base)[0])
    if not torch.equal(zs[0], zs[1]):
        raise SystemExit("DPM-Solver++ inpainting: the device loop and the per-step loop disagree")
    sched20 = dpm.make_dpm_schedule(20, 2)
    mixed20 = [5, 10, 15, 20]
    z_mixed = dpm.decode(z_lat, c, w, mixed20, sched20, scale, uc)
    if not torch.equal(z_mixed, dpm.dpm_decoding(w, c, z_lat, mixed20, sched20, scale, uc, per_step=True)):
        raise SystemExit("DPM-Solver++ decode: the device loop and the per-step loop disagree")

    ddim.make_schedule(50, verbose=False)
    n50 = len(ddim.ddim_timesteps)
    mixed50 = [n50 // 4, n50 // 2, 3 * n50 // 4, n50]
    rows = {}
    for S in (15, 20, 25):
        rows[f"dpm2m_inpaint_S{S}"] = (dpm, lambda S=S: dpm.inpaint(S, mask=mask, x0=x0, order=2, **base), S)
    rows["ddim_inpaint_S50"] = (ddim, lambda: ddim.sample(50, mask=mask, x0=x0, **base), n50)
    rows["dpm2m_decode_S20_full"] = (dpm, lambda: dpm.decode(z_lat, c, w, 20, sched20, scale, uc), 20)
    rows["dpm2m_decode_S20_mixed"] = (dpm, lambda: dpm.decode(z_lat, c, w, mixed20, sched20, scale, uc), 20)

    def ddim_decode(starts):
        ddim.make_schedule(50, verbose=False)
        return ddim.decode(z_lat, c, w, starts, scale, uc)

    rows["ddim_decode_S50_full"] = (ddim, lambda: ddim_decode(n50), n50)
    rows["ddim_decode_S50_mixed"] = (ddim, lambda: ddim_decode(mixed50), n50)
    for _ in range(a.warmup):
        for _, fn, _ in rows.values():
            timed(fn)
    t_end = time.perf_counter() + 1.0                                           # sustain phase
    while time.perf_counter() < t_end:
        for _, fn, _ in rows.values():
            timed(fn)
    times = {n: [] for n in rows}
    launches = {}
    for _ in range(a.reps):
        for n, (s, fn, _) in rows.items():
            t, out = timed(fn)
            times[n].append(t)
            launches[n] = s.last_launches_per_step
            if n == "dpm2m_decode_S20_mixed" and not torch.equal(out, z_mixed):
                raise SystemExit("DPM-Solver++ decode: a timed request changed its result")
    out = dict(L=L, B=B, cfg=scale, reps=a.reps, outputs_equal=True, mixed_t_start=dict(dpm_S20=mixed20, ddim_S50=mixed50),
               ddim_steps_S50=len(ddim_timesteps_uniform(50, 1000)), **info)
    for n, (s, fn, steps) in rows.items():
        ms = statistics.median(times[n])
        out[n] = dict(request_ms=round(ms, 2), steps=steps, ms_per_step=round(ms / steps, 3), launches_per_step=launches[n])
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
