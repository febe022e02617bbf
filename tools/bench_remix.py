"""Remix (DDIMSampler.decode) cost at the headline shape (L = 512, B = 4, CFG 5, S = 50), against a full DDIM request.

    python tools/bench_remix.py [--reps 3] [--warmup 2] [--S 50]

Rows: decode at a uniform t_start of 12, 25 and 50 (the plain mugd_sample loop), decode at the mixed t_start = [12, 25, 37, 50] (the
mugd_sample_join loop, 50 iterations) and a full sampler.sample.  bench.py's protocol: ``--warmup`` untimed runs of every row, a
sustain phase of at least 1 s, then ``--reps`` timed runs, the rows alternating; each is timed with CUDA events around one call, and
the median is reported.  Before timing, the mixed decode is checked against the same charts decoded one start at a time (each within
1e-5).  Prints one JSON line per row (milliseconds per request, iterations, ms per iteration, launches per iteration) and one with
the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
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
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200  # noqa: E402


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
    ap.add_argument("--S", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_remix needs a CUDA device")
    info = card()
    L, B, scale = 512, 4, 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    inp = synth.synthetic_inputs(B, L)
    c, w, uc = inp["c"].cuda(), [wi.cuda() for wi in inp["w"]], inp["uc"].cuda()
    full_kw = dict(S=a.S, c=c, w=w, batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), shape=(16, L),
                   unconditional_guidance_scale=scale, unconditional_conditioning=uc)
    sampler = DDIMSampler(model)
    sampler.make_schedule(a.S, verbose=False)
    n = len(sampler.ddim_timesteps)
    torch.cuda.manual_seed(2)
    z_enc = sampler.stochastic_encode(inp["x_T"].cuda(), torch.full((B,), n // 2, device="cuda"))
    mixed = [min(v, n) for v in (12, 25, 37, 50)]

    def decode(t_start):
        return lambda: sampler.decode(z_enc, c, w, t_start, scale, uc, tqdm_class=_Quiet)

    z_mixed = decode(mixed)()
    worst = 0.0
    for b, s in enumerate(mixed):
        one = sampler.decode(z_enc[b:b + 1], c[b:b + 1], [wi[b:b + 1] for wi in w], s, scale, uc[b:b + 1], tqdm_class=_Quiet)
        worst = max(worst, float((z_mixed[b] - one[0]).abs().max() / one[0].abs().max()))
    if worst > 1e-5:
        raise SystemExit(f"the mixed decode is {worst:.2e} away from the per-chart runs")

    rows = {f"decode t_start={s}": (decode(min(s, n)), min(s, n)) for s in (12, 25, 50)}
    rows[f"decode t_start={mixed}"] = (decode(mixed), max(mixed))
    rows[f"sample S={a.S}"] = (lambda: sampler.sample(tqdm_class=_Quiet, **full_kw), None)
    launches = {}

    def run_all(record=None):
        for name, (fn, _) in rows.items():
            ms, _ = timed(fn)
            launches[name] = sampler.last_launches_per_step
            if record is not None:
                record[name].append(ms)

    for _ in range(a.warmup):
        run_all()
    t_end = time.perf_counter() + 1.0                                           # sustain phase
    while time.perf_counter() < t_end:
        run_all()
    times = {name: [] for name in rows}
    for _ in range(a.reps):
        run_all(times)
    for name, (_, iters) in rows.items():
        iters = iters if iters is not None else len(sampler.ddim_timesteps)
        ms = statistics.median(times[name])
        print(json.dumps(dict(row=name, L=L, B=B, cfg=scale, S=a.S, iterations=iters, request_ms=round(ms, 2),
                              ms_per_iteration=round(ms / iters, 3), launches_per_iteration=launches[name], reps=a.reps)), flush=True)
    print(json.dumps(dict(mixed_vs_per_chart_max_rel_err=worst, **info)), flush=True)


class _Quiet:
    """tqdm_class stand-in: iterates without printing"""

    def __init__(self, it, **kw):
        self.it = it

    def __iter__(self):
        return iter(self.it)


if __name__ == "__main__":
    main()
