"""What per-chart seeds cost: seeded (mugd_randn, one launch per noise table) against unseeded (torch's generator, one randn per step
per table) requests at the headline shape (L = 512, B = 4, CFG 5), and mugd_randn alone.

    python tools/bench_seeds.py [--reps 3] [--warmup 1]

Flows: DDPM (all T = 1000 steps) and DDIM S = 50 at eta = 1 with inpainting (two noise tables per call), both from their one-call
device loops.  After ``--warmup`` untimed requests of each variant, ``--reps`` timed requests of each, seeded and unseeded
alternating; each is timed with CUDA events around one sampler.sample call, and the median is reported.  The generator alone fills a
64 MiB table (``[n][4, 16, 512]``): the median of 20 launches, and its write rate against the 3.35 TB/s HBM3 bound of an H100 SXM.
Prints one JSON line with the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_staged import card  # noqa: E402
from mug_diffusion_b200 import seeding, synth  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, DDPMSampler, MugDiffusionB200  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


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
        raise SystemExit("bench_seeds needs a CUDA device")
    info = card()
    L, B, scale = 512, 4, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    x0, mask = synth.synthetic_inpainting(B, L)
    kw = dict(c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, shape=(16, L),
              unconditional_guidance_scale=scale, unconditional_conditioning=inp["uc"].cuda())
    ddpm, ddim = DDPMSampler(model), DDIMSampler(model)
    flows = {
        "ddpm": lambda **s: ddpm.sample(**kw, **s),
        "ddim_eta1_inpaint": lambda **s: ddim.sample(S=50, eta=1.0, mask=mask.cuda(), x0=x0.cuda(), **kw, **s),
    }
    variants = {"unseeded": {}, "seeded": dict(seeds=1000)}
    for _ in range(a.warmup):
        for f in flows.values():
            for v in variants.values():
                timed(lambda: f(**v))
    ms = {(n, v): [] for n in flows for v in variants}
    for _ in range(a.reps):
        for n, f in flows.items():
            for v, extra in variants.items():
                torch.cuda.manual_seed(1)
                ms[(n, v)].append(timed(lambda: f(**extra)))
    row = dict(L=L, B=B, cfg=scale, reps=a.reps, **info)
    for (n, v), t in ms.items():
        row[f"{n}_{v}_ms"] = round(statistics.median(t), 2)
    for n in flows:
        row[f"{n}_seeded_over_unseeded"] = round(row[f"{n}_seeded_ms"] / row[f"{n}_unseeded_ms"], 4)

    # mugd_randn alone on a 64 MiB table
    n_draws = (64 << 20) // (4 * B * 16 * L)
    out = torch.empty(n_draws, B, 16 * L, device="cuda")
    sd = torch.from_numpy(seeding.seed_array(seeding.chart_seeds(1000, B)).view(np.int64)).cuda()
    fill = lambda: seeding.randn(out, sd, seeding.STEP, 0, n_draws)  # noqa: E731
    for _ in range(3):
        fill()
    kernel_ms = statistics.median(timed(fill) for _ in range(20))
    nbytes = out.numel() * 4
    row.update(randn_table_mib=nbytes >> 20, randn_kernel_us=round(1000 * kernel_ms, 2),
               randn_tb_per_s=round(nbytes / (kernel_ms / 1000) / 1e12, 3),
               randn_of_write_bound=round(nbytes / (kernel_ms / 1000) / HBM_BYTES_PER_S, 3))
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
