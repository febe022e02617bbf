"""UniPC inpainting, remix and edit (invert + decode) against DPM-Solver++ 2M and DDIM at the headline shape (L = 512, B = 4, CFG 5),
each from its one-call device loop.

    python tools/bench_unipc_edit.py [--reps 3] [--warmup 2]

Rows: UniPC-2 (bh1 and bh2) inpainting, remix (``stochastic_encode`` + ``decode`` over all S steps) and edit (``invert`` without
guidance, then ``decode`` with CFG 5, both over all S steps) at S = 8 and 10, against DPM++ 2M at S = 20 and DDIM at S = 50 (DDIM's
edit uses its own ``invert``).  First, outputs: every UniPC inpainting, decode and inversion latent must equal its per-step loop
(forced with a callback, or ``per_step``) bit for bit.  Then ``--warmup`` untimed requests of every row, a sustain phase of at least
1 s, then ``--reps`` timed rounds with the rows alternating, each request timed with CUDA events around its sampler calls; the median
is reported.  Prints one JSON line: per row the request time, the U-Net steps, the time per step and the launches per step, and the
card's name, power limit and max SM clock read in the same run.
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

from bench_dpm_remix import timed  # noqa: E402
from bench_staged import card  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, DPMSolverSampler, MugDiffusionB200, UniPCSampler  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_unipc_edit needs a CUDA device")
    info = card()
    L, B, scale = 512, 4, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    c, w, uc = inp["c"].cuda(), [t.cuda() for t in inp["w"]], inp["uc"].cuda()
    x0m, mask = (t.cuda() for t in synth.synthetic_inpainting(B, L))
    x0 = inp["x_T"].cuda() * 0.5                                                # stands for an encoded chart
    x_T = inp["x_T"].cuda()
    guided = dict(unconditional_guidance_scale=scale, unconditional_conditioning=uc)
    uni, dpm, ddim = UniPCSampler(model), DPMSolverSampler(model), DDIMSampler(model)

    for variant in ("bh1", "bh2"):
        sched = uni.make_unipc_schedule(10, 2, variant=variant)
        outs = []
        for cb in (None, lambda i: None):
            torch.cuda.manual_seed(1)
            outs.append(uni.inpaint(10, c, w, B, mask=mask, x0=x0m, shape=(16, L), x_T=x_T, variant=variant, callback=cb,
                                    verbose=False, **guided)[0])
        outs += [uni.decode(x0, c, w, [10, 7, 4, 1], sched, scale, uc),
                 uni.unipc_decoding(w, c, x0, [10, 7, 4, 1], sched, scale, uc, per_step=True)]
        outs += [uni.invert(x0, c, w, 10, sched, callback=cb, verbose=False) for cb in (None, lambda i: None)]
        if not all(torch.equal(outs[k], outs[k + 1]) for k in (0, 2, 4)):
            raise SystemExit(f"UniPC-2 {variant}: a device loop and its per-step loop disagree")

    rows = {}
    for S in (8, 10):
        for variant in ("bh1", "bh2"):
            sched = uni.make_unipc_schedule(S, 2, variant=variant)
            tag = f"unipc2_{variant}_S{S}"
            rows[f"{tag}_inpaint"] = (uni, lambda S=S, v=variant: uni.inpaint(S, c, w, B, mask=mask, x0=x0m, shape=(16, L), x_T=x_T,
                                                                               variant=v, verbose=False, **guided), S)
            rows[f"{tag}_remix"] = (uni, lambda S=S, s=sched: uni.decode(uni.stochastic_encode(x0, S, s), c, w, S, s, scale, uc), S)
            rows[f"{tag}_edit"] = (uni, lambda S=S, s=sched: uni.decode(uni.invert(x0, c, w, S, s, verbose=False), c, w, S, s, scale,
                                                                        uc), 2 * S)
    sd = dpm.make_dpm_schedule(20, 2)
    rows["dpm2m_S20_inpaint"] = (dpm, lambda: dpm.inpaint(20, c, w, B, mask=mask, x0=x0m, shape=(16, L), x_T=x_T, verbose=False,
                                                          **guided), 20)
    rows["dpm2m_S20_remix"] = (dpm, lambda: dpm.decode(dpm.stochastic_encode(x0, 20, sd), c, w, 20, sd, scale, uc), 20)
    rows["dpm2m_S20_edit"] = (dpm, lambda: dpm.decode(dpm.invert(x0, c, w, 20, sd, verbose=False), c, w, 20, sd, scale, uc), 40)
    ddim.make_schedule(50, verbose=False)
    rows["ddim_S50_inpaint"] = (ddim, lambda: ddim.sample(50, c, w, B, shape=(16, L), mask=mask, x0=x0m, x_T=x_T, verbose=False,
                                                          **guided), 50)
    rows["ddim_S50_remix"] = (ddim, lambda: ddim.decode(ddim.stochastic_encode(x0, torch.full((B,), 49, device="cuda")), c, w, 50,
                                                        scale, uc), 50)
    rows["ddim_S50_edit"] = (ddim, lambda: ddim.decode(ddim.invert(x0, c, w, 50, verbose=False), c, w, 50, scale, uc), 100)

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
        for n, (smp, fn, _) in rows.items():
            t, _ = timed(fn)
            times[n].append(t)
            launches[n] = smp.last_launches_per_step
    out = dict(L=L, B=B, reps=a.reps, outputs_equal=True, **info)
    for n, (_, fn, steps) in rows.items():
        ms = statistics.median(times[n])
        out[n] = dict(request_ms=round(ms, 2), steps=steps, ms_per_step=round(ms / steps, 3), launches_per_step=launches[n])
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
