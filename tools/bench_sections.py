"""What section prompts cost: the headline request (z_length 512, 4 charts, CFG 5, DDIM S = 50, seeded) with four sections per chart
(prompt changes at latent frames 128, 256 and 384) against the same request without sections.

    python tools/bench_sections.py [--reps 3] [--warmup 1]

Reported per variant: the whole request (sampler.sample, its one-call device loop), the U-Net graph replay per step (CUDA events
around 50 replays of the captured evaluation), the launches per step, and the once-per-request context projection (the prompt
transposes and the 16 K|V GEMMs of Session.set_context; 8 context slots per sample with sections).  After ``--warmup`` untimed rounds
(which compile and capture both sessions), ``--reps`` timed rounds alternate the variants and the median is reported.  Prints one
JSON line with the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
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

from bench_guidance import timed  # noqa: E402
from bench_staged import card  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200, section_contexts, section_prompts  # noqa: E402

L, B, S, SCALE = 512, 4, 50, 5.0
STARTS = (128, 256, 384)
REPLAYS = 50


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    m = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    c, uc = inp["c"].cuda(), inp["uc"].cuda()
    w = synth.wave_list([x.cuda() for x in inp["w"]])
    extra = synth.synthetic_inputs(len(STARTS), L, seed=21)["c"].cuda()
    sections = [[(s, extra[(k + b) % len(STARTS)]) for k, s in enumerate(STARTS)] for b in range(B)]
    kw = dict(S=S, c=c, w=w, batch_size=B, shape=(16, L), verbose=False, seeds=1, unconditional_guidance_scale=SCALE,
              unconditional_conditioning=uc)
    sampler = DDIMSampler(m)
    variants = {"plain": {}, "sections": dict(sections=sections)}
    checked = section_prompts(sections, c, B, L)
    ctx = {"plain": [uc, c], "sections": section_contexts(c, uc, checked)}
    keys = {"plain": (2 * B, L, False), "sections": (2 * B, L, False, "sectioned")}
    res = {v: dict(request_ms=[], replay_ms_per_step=[], context_ms=[]) for v in variants}
    launches = {}
    for r in range(args.warmup + args.reps):
        for v, extra_kw in variants.items():
            t_req = timed(lambda: sampler.sample(**kw, **extra_kw))
            launches[v] = sampler.last_launches_per_step
            sess = m.engine.sessions[keys[v]]
            t_rep = timed(lambda: sess.plan.replay(REPLAYS)) / REPLAYS
            t_ctx = timed(lambda: sess.set_context(ctx[v]))
            if r >= args.warmup:
                res[v]["request_ms"].append(t_req)
                res[v]["replay_ms_per_step"].append(t_rep)
                res[v]["context_ms"].append(t_ctx)
    out = dict(workload=f"L{L}_B{B}_cfg{SCALE:g}_S{S}", sections_per_chart=len(STARTS) + 1, card=card())
    for v in variants:
        out[v] = {k: round(statistics.median(x), 4) for k, x in res[v].items()}
        out[v]["launches_per_step"] = launches[v]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
