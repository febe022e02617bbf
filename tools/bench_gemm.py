"""Micro-benchmark of single GEMM ops through the C ABI (tensor-core vs FFMA), back-to-back launches.
usage (on the GPU box): python tools/bench_gemm.py [--reps 20]"""
import argparse
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_util import OpRunner, ptr, view  # noqa: E402
from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402
from mug_diffusion_b200.packer import tf32_split  # noqa: E402

# (label, B, L, Cin, Cout, taps)
SHAPES = [
    ("l0 conv3 384->128", 8, 512, 384, 128, 3), ("l0 conv3 128->128", 8, 512, 128, 128, 3), ("l0 1x1 384->128", 8, 512, 384, 128, 1),
    ("l1 conv3 640->256", 8, 256, 640, 256, 3), ("l1 qkv 256->768", 8, 256, 256, 768, 1), ("l1 ff1 256->2048", 8, 256, 256, 2048, 1),
    ("l1 ff2 1024->256", 8, 256, 1024, 256, 1), ("l2 conv3 1408->384", 8, 128, 1408, 384, 3), ("l2 ff1 384->3072", 8, 128, 384, 3072, 1),
    ("l3 conv3 1536->512", 8, 64, 1536, 512, 3), ("l3 conv3 512->512", 8, 64, 512, 512, 3), ("l3 1x1 512->512", 8, 64, 512, 512, 1),
    ("l3 ff1 512->4096", 8, 64, 512, 4096, 1), ("big conv3 640->256 B64", 64, 256, 640, 256, 3), ("tiny 1x1 128->128 k4", 8, 512, 128, 128, 1),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--split", type=int, default=0)
    a = ap.parse_args()
    R = OpRunner()
    print(f"{'shape':28s} {'M':>6s} {'N':>5s} {'Ktot':>5s} | {'tc us':>8s} {'tc TF/s':>8s} | {'simt us':>8s} {'simt TF/s':>9s} | splits")
    for label, B, L, Cin, Cout, taps in SHAPES:
        M = B * L
        x = torch.randn(M, Cin, device="cuda")
        w = torch.randn(Cout, taps * Cin) / math.sqrt(taps * Cin)
        hi, lo = tf32_split(w)
        wc, hc, lc = w.cuda(), hi.cuda(), lo.cuda()
        out = torch.zeros(M, Cout, device="cuda")
        res = {}
        import ctypes as C
        stamps = None
        for impl in (L_.GEMM_TC, L_.GEMM_SIMT):
            ops = OpList()
            for _ in range(a.reps):
                ops.gemm(view(x), ptr(wc), Cout, Cin, view(out), W_hi=ptr(hc), W_lo=ptr(lc), taps=taps,
                         mode=L_.CONV_SAME if taps == 3 else L_.CONV_NONE, Lin=L, Lout=L, impl=impl, split_k=a.split)
            R.run(ops)                      # warm (also attaches workspace)
            arr = ops.array()
            plan = C.c_void_p()
            L_.check(R.lib.mugd_plan_create(R.handle, arr, len(ops.ops), C.byref(plan)), "plan")
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                L_.check(R.lib.mugd_plan_capture(plan, side.cuda_stream), "capture")
            torch.cuda.synchronize()
            st = torch.cuda.current_stream().cuda_stream
            L_.check(R.lib.mugd_plan_replay(plan, 1, st), "replay")
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            L_.check(R.lib.mugd_plan_replay(plan, 3, st), "replay")
            e1.record()
            torch.cuda.synchronize()
            res[impl] = e0.elapsed_time(e1) * 1000 / (3 * a.reps)
            R.lib.mugd_plan_destroy(plan)
            if impl == L_.GEMM_TC:
                buf = torch.zeros(8, dtype=torch.int64, device="cuda")
                R.lib.mugd_debug_set_tc_timing(buf.data_ptr())
                L_.check(R.lib.mugd_op_run(R.handle, C.byref(ops.ops[0]), st), "op")
                torch.cuda.synchronize()
                R.lib.mugd_debug_set_tc_timing(None)
                t = buf.cpu().tolist()
                stamps = [(t[1] - t[0]) / 1e3, (t[2] - t[1]) / 1e3, (t[3] - t[2]) / 1e3, (t[4] - t[3]) / 1e3]
        flops = 2.0 * M * Cout * Cin * taps
        sp = C.c_int32()
        g = ops.ops[0].u.gemm
        R.lib.mugd_gemm_tc_query(R.handle, C.byref(g), 132, None, C.byref(sp), None, None)
        print(f"{label:28s} {M:6d} {Cout:5d} {taps*Cin:5d} | {res[L_.GEMM_TC]:8.1f} {flops/res[L_.GEMM_TC]/1e6:8.1f} | "
              f"{res[L_.GEMM_SIMT]:8.1f} {flops/res[L_.GEMM_SIMT]/1e6:9.1f} | {sp.value}  cta0 setup/main/stage/epi us = "
              f"{stamps[0]:.1f}/{stamps[1]:.1f}/{stamps[2]:.1f}/{stamps[3]:.1f}")


if __name__ == "__main__":
    main()
