"""Time the chart encoder (model.model.encode: Encoder.forward plan + posterior) on the GPU.

    python tools/bench_encode.py [--iters 200] [--warmup 20]

For each shape (B=4, L=512 and B=8, L=992; the note arrays have 8L frames) the encoder plan is captured once, warmed up, and then
replayed ``--iters`` times between two CUDA events.  The work is counted from the plan's GEMM shapes (2 M N (taps K + K2) per GEMM;
GroupNorms are not counted).  Prints one JSON line per shape with the card's name and power limit read in the same run.  Needs a
CUDA device: there is no CPU measurement.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.engine import Arena, EncoderCompiler  # noqa: E402
from mug_diffusion_b200.sampler import MugDiffusionB200  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power, clock = (q.stdout.strip().split(", ") + [None] * 3)[:3] if q.returncode == 0 else (torch.cuda.get_device_name(), None, None)
    return dict(gpu=name, power_limit_w=float(power) if power else None, sm_max_mhz=int(clock) if clock else None)


def plan_gflop(model, B: int, Lz: int) -> float:
    eng = model.engine
    res = EncoderCompiler(eng.encoder_cfg, eng.blob, 0, {}).compile(Arena(0), B, Lz)
    return sum(2.0 * o.u.gemm.M * o.u.gemm.N * (o.u.gemm.K * o.u.gemm.taps + o.u.gemm.K2)
               for o in res["ops"].ops if o.kind == L_.OP_GEMM) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode needs a CUDA device")
    sd = {**synth.synthetic_state_dict(512), **synth.synthetic_encoder_state_dict()}
    model = MugDiffusionB200.from_state_dict(sd, z_length=512)
    info = card()
    for B, L in ((4, 512), (8, 992)):
        notes = synth._gauss(synth._rng(7, "bench_notes"), (B, 16, 8 * L)).clamp(0, 1).cuda()
        s = model.engine.encoder_session(B, L)
        post = s.encode(notes)                                   # captures the plan's CUDA graph
        torch.cuda.synchronize()
        s.plan.replay(a.warmup)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        s.plan.replay(a.iters)
        t1.record()
        t1.synchronize()
        ms_plan = t0.elapsed_time(t1) / a.iters
        # the whole call as a user makes it (transpose in, graph, transpose out, posterior op, allocation of the outputs)
        for _ in range(a.warmup):
            s.encode(notes)
        t0.record()
        for _ in range(a.iters):
            post = s.encode(notes)
        t1.record()
        t1.synchronize()
        ms_call = t0.elapsed_time(t1) / a.iters
        gf = plan_gflop(model, B, L)
        print(json.dumps(dict(B=B, L=L, frames=8 * L, ms_graph=round(ms_plan, 4), ms_encode=round(ms_call, 4), gflop=round(gf, 3),
                              tflops_graph=round(gf / ms_plan, 2), finite=bool(torch.isfinite(post.mean).all()), **info)))


if __name__ == "__main__":
    main()
