"""A launch plan hands every tensor-core GEMM the next tensor-core GEMM of the plan, whose weights it prefetches into L2.
The prefetch must not change a single output bit: a chain of GEMMs run as a plan (prefetching) must equal the same ops run one by
one (no prefetch), including split-K GEMMs, an FFMA GEMM between two tensor-core ones and serial-split GEMMs (MUGD_OP_GEMM_SERIAL),
both prefetching and prefetched."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.engine import OpList  # noqa: E402
from mug_diffusion_b200.packer import tf32_split  # noqa: E402

from gpu_util import OpRunner, ptr, view  # noqa: E402


def test_plan_prefetch_keeps_outputs_bit_identical():
    R = OpRunner()
    R.set_impl("tc")
    M = 1024
    # (K, N, serial split): 384->1536 splits K, 1536->384 fills the grid, 48->64 (K % 32 != 0) runs on the FFMA kernel;
    # 384->384 prefetches the weights of a serial split; 384->320 (serial, 3 x 8 CTAs) prefetches 320->160's 204800 bytes, which its
    # 24 CTAs do not divide evenly, and 320->160 (serial) prefetches a plain tensor-core GEMM's
    chain = [(384, 1536, 0), (1536, 384, 0), (384, 48, 0), (48, 384, 0), (384, 384, 0), (384, 320, 5), (320, 160, 2), (160, 384, 0)]
    keep = []
    x = synth._gauss(synth._rng(3, "x"), (M, chain[0][0])).cuda()
    bufs = [x] + [torch.zeros(M, n, device="cuda") for _, n, _ in chain]
    ops = OpList()
    for i, (K, N, serial) in enumerate(chain):
        w = synth._gauss(synth._rng(3, f"w{i}"), (N, K)) / math.sqrt(K)
        hi, lo = tf32_split(w)
        wc, hc, lc = w.cuda(), hi.cuda(), lo.cuda()
        keep += [wc, hc, lc]
        tc = K % 32 == 0
        j = ops.gemm(view(bufs[i]), ptr(wc), N, K, view(bufs[i + 1]), W_hi=ptr(hc) if tc else 0, W_lo=ptr(lc) if tc else 0,
                     impl=L_.GEMM_TC if tc else L_.GEMM_SIMT, split_k=serial)
        if serial:
            ops.ops[j].kind = L_.OP_GEMM_SERIAL
    assert 204800 % 24 != 0 and 320 * 160 * 4 == 204800
    R.run(ops)
    eager = [b.clone() for b in bufs[1:]]
    for b in bufs[1:]:
        b.zero_()
    plan = C.c_void_p()
    L_.check(R.lib.mugd_plan_create(R.handle, ops.array(), len(ops.ops), C.byref(plan)), "plan")
    try:
        L_.check(R.lib.mugd_plan_run(plan, C.c_void_p(torch.cuda.current_stream().cuda_stream)), "plan_run")
        torch.cuda.synchronize()
    finally:
        R.lib.mugd_plan_destroy(plan)
    for i, (a, b) in enumerate(zip(eager, bufs[1:])):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b), f"GEMM {i} of the chain differs when run in a plan"
