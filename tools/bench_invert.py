"""DPM-Solver++ inversion against sampling and remix at the headline shape (L = 512, B = 4), each from its one-call device loop.

    python tools/bench_invert.py [--reps 3] [--warmup 2]

Rows: DPM++ 2M ``invert`` over all S = 20 steps without guidance and with CFG 5, DPM++ 2M ``sample`` at S = 20 with CFG 5, a full edit
(``invert`` without guidance, then ``decode`` with CFG 5, both over all 20 steps) and a 20-step remix (``stochastic_encode``, then
``decode`` with CFG 5).  First, outputs: each inversion's device loop must equal its per-step loop (forced with a callback) bit for bit.
Then ``--warmup`` untimed requests of every row, a sustain phase of at least 1 s, then ``--reps`` timed rounds with the rows
alternating, each request timed with CUDA events around its sampler calls; the median is reported.  Prints one JSON line: per row the
request time, the U-Net steps, the time per step and the launches per step, and the card's name, power limit and max SM clock read in
the same run.
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
from mug_diffusion_b200.sampler import DPMSolverSampler, MugDiffusionB200  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_invert needs a CUDA device")
    info = card()
    L, B, S, scale = 512, 4, 20, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    c, w, uc = inp["c"].cuda(), [t.cuda() for t in inp["w"]], inp["uc"].cuda()
    dpm = DPMSolverSampler(model)
    sched = dpm.make_dpm_schedule(S, 2)
    x0 = inp["x_T"].cuda() * 0.5                                                # stands for an encoded chart
    guided = dict(unconditional_guidance_scale=scale, unconditional_conditioning=uc)

    for kw in ({}, guided):
        zs = [dpm.invert(x0, c, w, S, sched, callback=cb, verbose=False, **kw) for cb in (None, lambda i: None)]
        if not torch.equal(zs[0], zs[1]):
            raise SystemExit("DPM-Solver++ inversion: the device loop and the per-step loop disagree")

    def edit():
        return dpm.decode(dpm.invert(x0, c, w, S, sched, verbose=False), c, w, S, sched, scale, uc)

    def remix():
        return dpm.decode(dpm.stochastic_encode(x0, S, sched), c, w, S, sched, scale, uc)

    rows = {
        "dpm2m_invert_S20_nocfg": (lambda: dpm.invert(x0, c, w, S, sched, verbose=False), S),
        "dpm2m_invert_S20_cfg5": (lambda: dpm.invert(x0, c, w, S, sched, verbose=False, **guided), S),
        "dpm2m_sample_S20_cfg5": (lambda: dpm.sample(S, c, w, B, shape=(16, L), x_T=inp["x_T"].cuda(), order=2, verbose=False,
                                                     **guided), S),
        "edit_S20_invert_nocfg_decode_cfg5": (edit, 2 * S),
        "remix_S20_encode_decode_cfg5": (remix, S),
    }
    for _ in range(a.warmup):
        for fn, _ in rows.values():
            timed(fn)
    t_end = time.perf_counter() + 1.0                                           # sustain phase
    while time.perf_counter() < t_end:
        for fn, _ in rows.values():
            timed(fn)
    times = {n: [] for n in rows}
    launches = {}
    for _ in range(a.reps):
        for n, (fn, _) in rows.items():
            t, _ = timed(fn)
            times[n].append(t)
            launches[n] = dpm.last_launches_per_step
    out = dict(L=L, B=B, S=S, reps=a.reps, outputs_equal=True, **info)
    for n, (fn, steps) in rows.items():
        ms = statistics.median(times[n])
        out[n] = dict(request_ms=round(ms, 2), steps=steps, ms_per_step=round(ms / steps, 3), launches_per_step=launches[n])
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
