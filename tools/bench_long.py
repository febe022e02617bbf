"""Long songs: what a DDIM step costs as z_length grows past the resident S4 kernel's limit (1568) to the supported maximum (8192).

    python tools/bench_long.py [--lengths 512,992,1568,1600,2048,4096,8192] [--S 50] [--B 4]

Per z_length, at B = 4 with CFG 5 (8 U-Net rows per step):
* ms per step: one untimed request, then one DDIM request of S steps timed with CUDA events around sampler.sample;
* in-graph time per op family (gemm / attention / s4conv / groupnorm / other): every op of the U-Net plan timed in its own
  captured graph (tools/profile_ops.py's method, REPS copies back to back), summed per family;
* FLOPs per step counted from the plan's shapes (GEMM 2MN(K*taps + K2), attention 4*B*H*Lq*Lk*D, S4 B*H*L*(L+1) for the causal
  direct form) and the U-Net session's arena bytes.
Then the resident and the streamed S4 kernels at the level-0 shape (B = 8, H = 128) of z_length 512, 992 and 1568: CUDA events
around graphs of 20 launches, the two alternating.  Prints the card's name, power limit and max SM clock, and one JSON line.
"""
import argparse
import collections
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_staged import card  # noqa: E402
from profile_ops import NAMES  # noqa: E402
from mug_diffusion_b200 import lib as L_, synth  # noqa: E402
from mug_diffusion_b200.engine import OpList, View  # noqa: E402
from mug_diffusion_b200.runtime import Plan  # noqa: E402
from mug_diffusion_b200.sampler import DDIMSampler, MugDiffusionB200  # noqa: E402

REPS = 5


def graph_ms(eng, ops, replays=5):
    pl = Plan(eng, ops)
    pl.run()
    pl.capture()
    pl.replay(2)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    pl.replay(replays)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / replays


def flops(op) -> float:
    k = op.kind
    if k == L_.OP_GEMM:
        g = op.u.gemm
        return 2.0 * g.M * g.N * (g.K * g.taps + g.K2)
    if k == L_.OP_ATTENTION:
        a = op.u.attn
        return 4.0 * a.B * a.H * a.Lq * a.Lk * a.D
    if k == L_.OP_S4CONV:
        s = op.u.s4
        return float(s.B) * s.H * s.L * (s.L + 1)
    return 0.0


def family(op) -> str:
    f = NAMES.get(op.kind, "other")
    return f if f in ("gemm", "attention", "s4conv", "groupnorm") else "other"


def per_length(L, B, S):
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(L), z_length=L)
    eng = model.engine
    inp = synth.synthetic_inputs(B, L)
    kw = dict(S=S, c=inp["c"].cuda(), w=[w.cuda() for w in inp["w"]], batch_size=B, verbose=False, x_T=inp["x_T"].cuda(), eta=0.0,
              shape=(16, L), unconditional_guidance_scale=5.0, unconditional_conditioning=inp["uc"].cuda())
    sampler = DDIMSampler(model)
    sampler.sample(**kw)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    sampler.sample(**kw)
    e1.record()
    e1.synchronize()
    ms_step = e0.elapsed_time(e1) / S
    sess = eng.session(2 * B, L)
    arr, n = sess.plan._arr, sess.plan.n_ops
    sigs = collections.OrderedDict()
    for i in range(n):
        sigs.setdefault(bytes(arr[i]), []).append(i)
    fam_ms = collections.Counter()
    fam_gflop = collections.Counter()
    for idx in sigs.values():
        op = arr[idx[0]]
        sub = OpList()
        sub.ops.extend([op] * REPS)
        eng.attach_workspace(sub)
        fam_ms[family(op)] += graph_ms(eng, sub) / REPS * len(idx)
        fam_gflop[family(op)] += flops(op) * len(idx) / 1e9
    row = dict(z_length=L, ms_per_step=round(ms_step, 3), family_ms={k: round(v, 3) for k, v in fam_ms.items()},
               family_gflop={k: round(v, 1) for k, v in fam_gflop.items() if v}, arena_bytes=int(sess.arena_t.numel() * 4))
    print(json.dumps(row), flush=True)
    del sampler, sess, model, eng
    torch.cuda.empty_cache()
    return row


def resident_vs_streamed(lengths, B=8, H=128, launches=20, rounds=5):
    model = MugDiffusionB200.from_state_dict(synth.synthetic_state_dict(96), z_length=96)
    eng = model.engine
    out = {}
    for L in lengths:
        u = torch.randn(B * L, H, device="cuda")
        kt = torch.randn(L, H, device="cuda") * torch.exp(-torch.arange(L, device="cuda") / 1000.0)[:, None]
        d = torch.randn(H, device="cuda")
        ys = {impl: torch.empty(B * L, H, device="cuda") for impl in (1, 2)}
        plans = {}
        for impl in (1, 2):
            ops = OpList()
            for _ in range(launches):
                ops.s4conv(View(u.data_ptr(), H, B * L, H), kt.data_ptr(), d.data_ptr(), View(ys[impl].data_ptr(), H, B * L, H), B, L)
            L_.check(eng.lib.mugd_set_s4conv_impl(eng.handle, impl), "s4conv_impl")
            pl = Plan(eng, ops)
            pl.run()
            pl.capture()                                        # the graph keeps the kernel chosen at capture
            plans[impl] = pl
        L_.check(eng.lib.mugd_set_s4conv_impl(eng.handle, 0), "s4conv_impl")
        torch.cuda.synchronize()
        assert torch.equal(ys[1], ys[2]), L
        times = {1: [], 2: []}
        for _ in range(rounds):
            for impl in (1, 2):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                plans[impl].replay(5)
                e1.record()
                e1.synchronize()
                times[impl].append(e0.elapsed_time(e1) * 1000 / (5 * launches))
        gflop = B * H * L * (L + 1) / 1e9
        out[L] = {name: dict(us=round(statistics.median(times[impl]), 2), tflops=round(gflop / statistics.median(times[impl]) * 1e3, 2))
                  for name, impl in (("resident", 1), ("streamed", 2))}
        print(json.dumps({"s4conv": dict(L=L, B=B, H=H, **out[L])}), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", default="512,992,1568,1600,2048,4096,8192")
    ap.add_argument("--S", type=int, default=50)
    ap.add_argument("--B", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_long needs a CUDA device")
    info = card()
    print(json.dumps(info), flush=True)
    rows = [per_length(int(L), a.B, a.S) for L in a.lengths.split(",")]
    s4 = resident_vs_streamed([512, 992, 1568])
    print(json.dumps(dict(info, B=a.B, S=a.S, cfg=5.0, lengths=rows, s4conv=s4)))


if __name__ == "__main__":
    main()
