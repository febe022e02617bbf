"""What per-chart guidance scales save and cost: a guidance sweep of one chart at scales 3 / 5 / 7 / 9 (one seed, z_length 512) as one
request of four charts against four sequential one-chart requests, and a uniform-scale request of four charts (CFG 5) on today's
path against the same request forced onto the guided-scales session.

    python tools/bench_guidance.py [--reps 3] [--warmup 1]

Flows: DDIM S = 50 and UniPC bh2 S = 10, seeded, from their one-call device loops.  After ``--warmup`` untimed rounds (which compile
and capture every session), ``--reps`` timed rounds alternate the variants; each is timed with CUDA events around its sampler.sample
calls and the median is reported, with the launches per step of each variant.  Prints one JSON line with the card's name, power limit
and max SM clock read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_staged import card  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200, UniPCSampler  # noqa: E402

SWEEP = [3.0, 5.0, 7.0, 9.0]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_guidance needs a CUDA device")
    info = card()
    L, B = 512, len(SWEEP)
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    c, uc, w = inp["c"].cuda(), inp["uc"].cuda(), [t.cuda() for t in inp["w"]]
    # the sweep: one chart (prompt, audio and seed of chart 0) at four scales
    c1, uc1, w1 = c[:1], uc[:1], [t[:1] for t in w]
    c4, uc4, w4 = c1.expand(B, -1, -1).contiguous(), uc1.expand(B, -1, -1).contiguous(), [t.expand(B, -1, -1).contiguous() for t in w1]
    common = dict(verbose=False, shape=(16, L))
    samplers = {"ddim_S50": (DDIMSampler(model), dict(S=50)), "unipc_bh2_S10": (UniPCSampler(model), dict(S=10, variant="bh2"))}
    launches = {}

    def run(name, s, fn):
        fn()
        launches[name] = s.last_launches_per_step

    def sequential(s, kw):
        for sc in SWEEP:
            s.sample(c=c1, w=w1, batch_size=1, unconditional_conditioning=uc1, unconditional_guidance_scale=sc, seeds=[7], **kw, **common)

    def sweep(s, kw):
        s.sample(c=c4, w=w4, batch_size=B, unconditional_conditioning=uc4, unconditional_guidance_scale=SWEEP, seeds=[7] * B, **kw,
                 **common)

    def uniform(s, kw, forced):
        s.force_per_chart_scales = forced
        try:
            s.sample(c=c, w=w, batch_size=B, unconditional_conditioning=uc, unconditional_guidance_scale=5.0, seeds=7, **kw, **common)
        finally:
            s.force_per_chart_scales = False

    variants = {"sequential": sequential, "sweep": sweep, "uniform_today": lambda s, kw: uniform(s, kw, False),
                "uniform_guided": lambda s, kw: uniform(s, kw, True)}
    for _ in range(a.warmup):
        for n, (s, kw) in samplers.items():
            for v, f in variants.items():
                run(f"{n}_{v}", s, lambda: f(s, kw))
    ms = {(n, v): [] for n in samplers for v in variants}
    for _ in range(a.reps):
        for n, (s, kw) in samplers.items():
            for v, f in variants.items():
                ms[(n, v)].append(timed(lambda: f(s, kw)))
    row = dict(scales=SWEEP, z_length=L, reps=a.reps, **info)
    for (n, v), t in ms.items():
        row[f"{n}_{v}_ms"] = round(statistics.median(t), 2)
    for n, (s, kw) in samplers.items():
        row[f"{n}_sweep_speedup"] = round(row[f"{n}_sequential_ms"] / row[f"{n}_sweep_ms"], 3)
        row[f"{n}_guided_over_today"] = round(row[f"{n}_uniform_guided_ms"] / row[f"{n}_uniform_today_ms"], 4)
        steps = kw["S"]
        row[f"{n}_guided_minus_today_ms_per_step"] = round((row[f"{n}_uniform_guided_ms"] - row[f"{n}_uniform_today_ms"]) / steps, 4)
        for v in ("uniform_today", "uniform_guided", "sweep"):
            row[f"{n}_{v}_launches_per_step"] = launches.get(f"{n}_{v}")
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
