"""Time gridify's timing search on the CPU (postprocess.gridify) against model.model.gridify (scans on the GPU).

    python tools/bench_gridify.py [--reps 3]

Workloads: 4 and 32 charts of about 2,000 notes and 4 charts of about 8,000 notes (tools/make_postprocess_goldens.chart, seeded,
bpm 150 .. 300 with 1/4 and 1/8 divisions).  Both paths are first checked to give equal outputs (lines, and bpm / offset equal in
value and numpy type).  Then, best of ``--reps``: the wall time of the CPU loop ``[postprocess.gridify(c, verbose=False) ...]`` and of
the batched ``model.model.gridify(charts)`` (each scan ends in a device synchronise, so the call's wall time covers the device
work), with, for the GPU call, the number of scans, the summed CUDA-event time of the scan calls and the host time spent in refits
(fit_grid with refit), and the host time of the snapping (snap_lines) alone.  scikit-learn is imported before anything is timed.  Prints one JSON line per workload with the card's
name, power limit and max SM clock read in the same run.  Needs a CUDA device.
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
from mug_diffusion_b200 import postprocess as pp  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.sampler import MugDiffusionB200  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + [None] * 3)[:3] if q.returncode == 0 else (torch.cuda.get_device_name(), None, None)
    return dict(gpu=name, power_limit_w=float(power) if power else None, sm_max_mhz=int(clock) if clock else None)


def charts(count: int, slots: int, seed: int):
    """``count`` charts; ``slots`` grid slots give about 1.5 notes each (chords)"""
    return [chart(seed=seed + i, bpm=150 + 37.3 * i % 150, offset=200 + 97 * i, n=slots, div=4 if i % 2 else 8, jitter=2.0,
                  ln_ratio=0.15, jack_ratio=0.0) for i in range(count)]


def same(a, b) -> bool:
    return len(a) == len(b) and all(x[0] == y[0] and type(x[1]) is type(y[1]) and x[1] == y[1] and type(x[2]) is type(y[2])
                                    and x[2] == y[2] for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gridify needs a CUDA device")
    info = card()
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(96), z_length=96)
    scanner = model.grid_scanner
    fit_grid = pp.fit_grid
    refit_s = [0.0]

    def timed_fit_grid(*args):
        t = time.perf_counter()
        r = fit_grid(*args)
        if args[4]:
            refit_s[0] += time.perf_counter() - t
        return r

    pp.fit_grid = timed_fit_grid                                    # search_timing's refits, timed
    first = charts(1, 100, 1)[0]
    pp.gridify(first, verbose=False)                                # imports scikit-learn
    model.model.gridify([first])
    for name, count, slots in (("4x2000", 4, 1300), ("32x2000", 32, 1300), ("4x8000", 4, 5000)):
        cs = charts(count, slots, 1000 + count + slots)
        notes = [len(c) for c in cs]
        cpu = [pp.gridify(c, verbose=False) for c in cs]
        gpu = model.model.gridify(cs)
        if not same(cpu, gpu):
            raise SystemExit(f"{name}: model.model.gridify differs from postprocess.gridify")
        cpu_s, gpu_s, best = [], [], None
        for _ in range(a.reps):
            t = time.perf_counter()
            [pp.gridify(c, verbose=False) for c in cs]
            cpu_s.append(time.perf_counter() - t)
            scanner.kernel_ms, scanner.scan_s, refit_s[0] = [], 0.0, 0.0
            torch.cuda.synchronize()
            t = time.perf_counter()
            model.model.gridify(cs)
            torch.cuda.synchronize()
            gpu_s.append(time.perf_counter() - t)
            if best is None or gpu_s[-1] <= min(gpu_s):
                best = dict(scans=len(scanner.kernel_ms), kernel_ms=round(sum(scanner.kernel_ms), 3),
                            scan_call_ms=round(scanner.scan_s * 1e3, 3), refit_ms=round(refit_s[0] * 1e3, 3))
        t = time.perf_counter()
        [pp.snap_lines(c, bpm, off) for c, (_, bpm, off) in zip(cs, gpu)]
        best["snap_ms"] = round((time.perf_counter() - t) * 1e3, 2)
        scanner.kernel_ms = None
        print(json.dumps(dict(workload=name, charts=count, notes_mean=round(sum(notes) / count), notes_max=max(notes),
                              cpu_loop_ms=round(min(cpu_s) * 1e3, 2), gpu_call_ms=round(min(gpu_s) * 1e3, 2),
                              speedup=round(min(cpu_s) / min(gpu_s), 2), **best, **info)), flush=True)


if __name__ == "__main__":
    main()
