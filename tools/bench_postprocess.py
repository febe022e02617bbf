"""Time webui's chart post-processing on the host (postprocess.py) against the device path (chartpost.py).

    python tools/bench_postprocess.py [--reps 3]

Workloads (tools/make_postprocess_goldens.chart, seeded): 4 and 32 charts of about 2,000 notes and 4 of about 8,000, with 15 %
long notes and jack_ratio 0.3; one rice chart (no long notes) of about 2,500 and one of about 9,600 notes with jack_ratio 0.3, where
the host's held_at walks back to the start of the chart on every jack.  Both paths are first checked to give equal outputs.  Then,
best of ``--reps``, wall time ending in a device synchronise of:
  snap:        [postprocess.snap_lines(c, bpm, offset) ...]   vs  chartpost.Lines + chartpost.snap_charts (parse, kernel, format)
  mini-jacks:  [postprocess.remove_intractable_mania_mini_jacks(c, verbose=False) ...]  vs  model.model.remove_mini_jacks
  custom_gridify: the host composition of webui.py:401-407 per chart  vs  model.model.postprocess_charts,
with the CUDA-event time of the snap and mini-jack kernels and, for postprocess_charts, where the wall time goes: the timing search
(scans and refits), the two kernel calls with their copies, and the rest (parsing and formatting the lines).  Prints one JSON line per
workload with the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_postprocess_goldens import chart  # noqa: E402
from mug_diffusion_b200 import chartpost as cp  # noqa: E402
from mug_diffusion_b200 import postprocess as pp  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import MugDiffusionB200  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + [None] * 3)[:3] if q.returncode == 0 else (torch.cuda.get_device_name(), None, None)
    return dict(gpu=name, power_limit_w=float(power) if power else None, sm_max_mhz=int(clock) if clock else None)


def mixed(count: int, slots: int, seed: int):
    """``count`` charts; ``slots`` grid slots give about 1.5 notes each (chords), 15 % long notes, jack_ratio 0.3"""
    return [chart(seed=seed + i, bpm=150 + 37.3 * i % 150, offset=200 + 97 * i, n=slots, div=4 if i % 2 else 8, jitter=2.0,
                  ln_ratio=0.15, jack_ratio=0.3) for i in range(count)]


def rice(slots: int, seed: int):
    return [chart(seed=seed, bpm=200.0, offset=300, n=slots, div=4, jitter=2.0, ln_ratio=0.0, jack_ratio=0.3)]


def custom_gridify(lines, auto_snap=True, jack_interval=90):
    """webui.py:401-407"""
    new, bpm, off = pp.gridify(lines, verbose=False)
    if auto_snap:
        lines = new
    return bpm, off, pp.remove_intractable_mania_mini_jacks(lines, verbose=False, jack_interval=jack_interval)


def same_timed(a, b) -> bool:
    return len(a) == len(b) and all(x[2] == y[2] and type(x[0]) is type(y[0]) and x[0] == y[0] and type(x[1]) is type(y[1])
                                    and x[1] == y[1] for x, y in zip(a, b))


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_postprocess needs a CUDA device")
    info = card()
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(96), z_length=96)
    scanner, post = model.grid_scanner, model.chart_post
    spent = {"search": 0.0, "snap": 0.0, "jacks": 0.0}

    def timed(key, fn):
        def run(*args, **kw):
            t = time.perf_counter()
            r = fn(*args, **kw)
            torch.cuda.synchronize()
            spent[key] += time.perf_counter() - t
            return r
        return run

    scanner.search = timed("search", scanner.search)
    post.snap = timed("snap", post.snap)
    post.mini_jacks = timed("jacks", post.mini_jacks)
    warm = mixed(1, 100, 1)
    custom_gridify(warm[0])                                           # imports scikit-learn
    model.model.postprocess_charts(warm)
    model.model.remove_mini_jacks(warm)
    for name, cs in (("4x2000", mixed(4, 1070, 2000)), ("32x2000", mixed(32, 1070, 3000)), ("4x8000", mixed(4, 4250, 4000)),
                     ("rice2500", rice(1310, 5000)), ("rice9600", rice(5050, 5001))):
        notes = [len(c) for c in cs]
        host_pp = [custom_gridify(c) for c in cs]
        dev_pp = model.model.postprocess_charts(cs)
        if not same_timed(host_pp, dev_pp):
            raise SystemExit(f"{name}: postprocess_charts differs from custom_gridify")
        timing = [(bpm, off) for bpm, off, _ in dev_pp]
        host_snap = [pp.snap_lines(c, bpm, off) for c, (bpm, off) in zip(cs, timing)]
        if cp.snap_charts(post, cp.Lines(cs), timing) != host_snap:
            raise SystemExit(f"{name}: snap_charts differs from snap_lines")
        host_jacks = [pp.remove_intractable_mania_mini_jacks(c, verbose=False) for c in cs]
        if model.model.remove_mini_jacks(cs) != host_jacks:
            raise SystemExit(f"{name}: remove_mini_jacks differs from the host function")
        best = {}

        def keep(key, seconds, extra=None):
            if key not in best or seconds < best[key][0]:
                best[key] = (seconds, extra)

        for _ in range(a.reps):
            keep("host_snap", wall(lambda: [pp.snap_lines(c, bpm, off) for c, (bpm, off) in zip(cs, timing)])[0])
            keep("host_jacks", wall(lambda: [pp.remove_intractable_mania_mini_jacks(c, verbose=False) for c in cs])[0])
            keep("host_pp", wall(lambda: [custom_gridify(c) for c in cs])[0])
            post.kernel_ms = []
            keep("dev_snap", wall(lambda: cp.snap_charts(post, cp.Lines(cs), timing))[0], post.kernel_ms)
            post.kernel_ms = []
            keep("dev_jacks", wall(lambda: model.model.remove_mini_jacks(cs))[0], post.kernel_ms)
            post.kernel_ms = None
            for k in spent:
                spent[k] = 0.0
            keep("dev_pp", wall(lambda: model.model.postprocess_charts(cs))[0], dict(spent))
        ms = {k: round(v[0] * 1e3, 2) for k, v in best.items()}
        split = best["dev_pp"][1]
        print(json.dumps(dict(
            workload=name, charts=len(cs), notes_mean=round(sum(notes) / len(cs)), notes_max=max(notes),
            snap_host_ms=ms["host_snap"], snap_dev_ms=ms["dev_snap"], snap_kernel_ms=round(sum(best["dev_snap"][1]), 3),
            jacks_host_ms=ms["host_jacks"], jacks_dev_ms=ms["dev_jacks"], jacks_kernel_ms=round(sum(best["dev_jacks"][1]), 3),
            custom_gridify_host_ms=ms["host_pp"], postprocess_charts_ms=ms["dev_pp"],
            pp_search_ms=round(split["search"] * 1e3, 2), pp_kernel_calls_ms=round((split["snap"] + split["jacks"]) * 1e3, 2),
            pp_parse_format_ms=round((best["dev_pp"][0] - sum(split.values())) * 1e3, 2), **info)), flush=True)


if __name__ == "__main__":
    main()
