"""What batch-invariant plans cost: DDIM S = 50, CFG 5, seeded, on a default engine and a batch_invariant engine over the same weights,
at z_length 512 for B = 1, 4, 8, 32 and at z_length 992 for B = 8.

    python tools/bench_batch_invariant.py [--reps 3] [--warmup 1]

After ``--warmup`` untimed requests per (engine, shape), which compile and capture every session, the two engines run alternately
``--reps`` times; each request is timed with CUDA events around ``DDIMSampler.sample`` and the median is reported, with the largest
difference between the two engines' latents (bit-identity with the charts requested alone is what tests/test_gpu_batch_invariant.py
checks).  Prints one JSON line with the card's name, power limit and max SM
clock read in the same run.  Needs a CUDA device.
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
from mug_diffusion_b200 import packer, synth  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200.config import ModelConfig  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200  # noqa: E402

CASES = [(512, 1), (512, 4), (512, 8), (512, 32), (992, 8)]


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
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batch_invariant needs a CUDA device")
    info = card()
    cfg = ModelConfig()
    results = []
    for L in sorted({L for L, _ in CASES}):
        sd = synth.synthetic_state_dict(L)
        blob = packer.pack_model(sd, cfg.unet, cfg.decoder)
        models = {"default": MugDiffusionB200(sd, cfg, z_length=L, blob=blob),
                  "invariant": MugDiffusionB200(sd, cfg, z_length=L, blob=blob, batch_invariant=True)}
        for L_case, B in CASES:
            if L_case != L:
                continue
            inp = synth.synthetic_inputs(B, L)
            kw = dict(S=50, eta=0.0, c=inp["c"].cuda(), w=[t.cuda() for t in inp["w"]], batch_size=B, shape=(16, L), verbose=False,
                      unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda(), seeds=100)
            run = {k: (lambda m=m: DDIMSampler(m).sample(**kw)[0]) for k, m in models.items()}
            for _ in range(a.warmup):
                for f in run.values():
                    f()
            times = {k: [] for k in run}
            outs = {}
            for _ in range(a.reps):
                for k, f in run.items():
                    ms, outs[k] = timed(f)
                    times[k].append(ms)
            sess = models["invariant"].engine.session(2 * B, L, unit=2)
            kinds = [op.kind for op in sess.plan._arr]
            med = {k: statistics.median(v) for k, v in times.items()}
            results.append(dict(L=L, B=B, default_ms=round(med["default"], 2), invariant_ms=round(med["invariant"], 2),
                                ratio=round(med["invariant"] / med["default"], 4),
                                serial_gemms=kinds.count(L_.OP_GEMM_SERIAL),
                                forced_split_gemms=sum(1 for op in sess.plan._arr if op.kind == L_.OP_GEMM and op.u.gemm.split_k),
                                max_abs_diff=float((outs["invariant"] - outs["default"]).abs().max())))
            print(json.dumps(results[-1]), file=sys.stderr)
        del models
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=info, reps=a.reps, results=results)))


if __name__ == "__main__":
    main()
