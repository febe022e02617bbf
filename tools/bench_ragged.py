"""What a ragged request saves: four songs of different lengths (z_length 384, 448, 480, 512; one chart each, CFG 5) charted as four
sequential requests against one ragged request of four charts padded to Lmax = 512, and the masking overhead of the ragged plan.

    python tools/bench_ragged.py [--reps 3] [--warmup 1]

Flows: DDIM S = 50 and UniPC bh2 S = 10, seeded, from their one-call device loops.  After ``--warmup`` untimed rounds (which compile
and capture every session), ``--reps`` timed rounds; each variant is timed with CUDA events around its sampler.sample calls and the
median is reported.  The per-evaluation cost of the ragged U-Net plan against the plain plan at the same (Beff = 8, Lmax = 512) is
the median of 50 graph replays of each: the difference is what the masks and the ragged GroupNorm / attention cost.  Prints one JSON
line with the card's name, power limit and max SM clock read in the same run.  Needs a CUDA device.
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

LENS = [384, 448, 480, 512]


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
        raise SystemExit("bench_ragged needs a CUDA device")
    info = card()
    Lmax, B, scale = max(LENS), len(LENS), 5.0
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(Lmax), z_length=Lmax)
    inp = synth.synthetic_inputs(B, Lmax)
    c, uc, w = inp["c"].cuda(), inp["uc"].cuda(), [t.cuda() for t in inp["w"]]
    songs = []                                # one song per chart at its own length: the features a song of that length gives
    for b, Lb in enumerate(LENS):
        songs.append([t[b:b + 1, :, :t.shape[-1] * Lb // Lmax].contiguous() for t in w])
    from mug_diffusion_b200.audio import pad_features
    w_pad, lens = pad_features(songs)
    assert lens == LENS
    common = dict(verbose=False, unconditional_guidance_scale=scale)
    samplers = {"ddim_S50": (DDIMSampler(model), dict(S=50)), "unipc_bh2_S10": (UniPCSampler(model), dict(S=10, variant="bh2"))}

    def sequential(s, kw):
        for b, Lb in enumerate(LENS):
            s.sample(c=c[b:b + 1], w=songs[b], batch_size=1, shape=(16, Lb), unconditional_conditioning=uc[b:b + 1], seeds=[7 + b],
                     **kw, **common)

    def ragged(s, kw):
        s.sample(c=c, w=w_pad, batch_size=B, shape=(16, Lmax), unconditional_conditioning=uc, seeds=7, z_lengths=LENS, **kw, **common)

    variants = {"sequential": sequential, "ragged": ragged}
    for _ in range(a.warmup):
        for s, kw in samplers.values():
            for f in variants.values():
                f(s, kw)
    ms = {(n, v): [] for n in samplers for v in variants}
    for _ in range(a.reps):
        for n, (s, kw) in samplers.items():
            for v, f in variants.items():
                ms[(n, v)].append(timed(lambda: f(s, kw)))
    row = dict(lengths=LENS, Lmax=Lmax, cfg=scale, reps=a.reps, **info)
    for (n, v), t in ms.items():
        row[f"{n}_{v}_ms"] = round(statistics.median(t), 2)
    for n in samplers:
        row[f"{n}_speedup"] = round(row[f"{n}_sequential_ms"] / row[f"{n}_ragged_ms"], 3)

    # per-evaluation cost of the ragged plan against the plain plan at the same (Beff, Lmax): graph replays of the captured plans
    eng = model.engine
    plain = eng.session(2 * B, Lmax)
    rag = eng.session(2 * B, Lmax, ragged=True)
    rag.set_lengths(LENS * 2)
    for sess in (plain, rag):
        sess.plan.ensure_captured()
        sess.plan.replay(5)
    per_eval = {}
    for name, sess in (("plain", plain), ("ragged", rag)):
        per_eval[name] = statistics.median(timed(lambda: sess.plan.replay(10)) / 10 for _ in range(5))
    row.update(eval_plain_ms=round(per_eval["plain"], 3), eval_ragged_ms=round(per_eval["ragged"], 3),
               eval_ragged_over_plain=round(per_eval["ragged"] / per_eval["plain"], 4),
               launches_plain=plain.plan.launches, launches_ragged=rag.plan.launches)
    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
