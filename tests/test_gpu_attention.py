"""The three attention kernels -- the wgmma kernel (attention_tc.cu, 3xTF32), the lane-per-key kernel for <= 32 keys and the exact-fp32
FFMA referee (attention.cu) -- against the float64 statement of mugd_attention in attention_cases.py:

* every attention signature of the real U-Net and wave-encoder plans, with q / k / v laid out as the plans lay them out (column
  windows of one fused qkv or kv buffer), through the plan's kernel and through the referee;
* hand-picked edges of each kernel: key and query tile boundaries, j - i beyond +-pos_max, pos_max 0 .. 1024, one head of dim 48,
  windows at column offsets that are not multiples of 32, and four data regimes (attention_cases.make_inputs);
* PDL ordering inside a captured plan: GEMM -> attention -> GEMM replayed from a graph equals the same ops run one by one.

Error metric: for every (sample, query row, head), max_c |o - ref| / max_c M with M = sum_j p_ij |cgain_ij| |v_jc|
(attention_cases.row_error): a wrong row or head cannot hide behind the largest value of the whole output.  The float64 reference
covers samples 0, B/2 and B-1; every sample is checked for stores outside the output window, untouched inputs and bit-identical
reruns.

Tolerances are about 3x the largest error observed on an H100, per kernel and data regime (TOL below, with the observed values).
They are tight enough to fail on a dropped hi/lo MMA of either wgmma product, a wrong V^T key order, or a lane-per-key kernel that
lets lanes without a key into the softmax."""
import ctypes as C
import math
import os

import pytest
import torch

import attention_cases as ac
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200.engine import OpList, View
from mug_diffusion_b200.packer import tf32_split

from gpu_util import OpRunner, ptr, view

SENT = -7777.0           # pre-fill of the output buffer: every element outside the output window must keep it
SENT_ROWS = 64           # sentinel rows below the last sample's rows
NAN = float("nan")       # fill of the input buffers' columns outside the q / k / v windows: never read

# (kernel, data regime) -> bound on attention_cases.row_error, about 3x the largest error over all cases of this file on an H100 80GB
# HBM3 (700 W power limit):
#            randn     peaked    gain      offset
#   tc       4.5e-6    6.2e-6    3.5e-6    5.5e-6     (3xTF32; one TF32 pass in either product gives 1e-4 .. 5e-4)
#   lane     7.5e-7    1.5e-6    9.3e-7    4.4e-7     (exact fp32)
#   ffma     7.5e-7    3.6e-6    9.3e-7    1.3e-6     (exact fp32)
TOL = {
    ("tc", "randn"): 1.4e-5, ("tc", "peaked"): 2e-5, ("tc", "gain"): 1.1e-5, ("tc", "offset"): 1.7e-5,
    ("lane", "randn"): 2.5e-6, ("lane", "peaked"): 4.5e-6, ("lane", "gain"): 3e-6, ("lane", "offset"): 1.4e-6,
    ("ffma", "randn"): 2.5e-6, ("ffma", "peaked"): 1.1e-5, ("ffma", "gain"): 3e-6, ("ffma", "offset"): 4e-6,
}


@pytest.fixture(scope="module")
def R():
    return OpRunner()


class attention_impl:
    """mugd_set_attention_impl for a block (per handle: always back to the default, 1)"""

    def __init__(self, R, impl):
        self.R, self.impl = R, impl

    def __enter__(self):
        L_.check(self.R.lib.mugd_set_attention_impl(self.R.handle, self.impl), "attention_impl")

    def __exit__(self, *exc):
        L_.check(self.R.lib.mugd_set_attention_impl(self.R.handle, 1), "attention_impl")


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.detach().cpu().contiguous().view(torch.int32)


class Device:
    """a case's operands on the GPU, laid out like the plan: q / k / v windows of fused buffers whose other columns hold NaN, and
    the output a column window of a wider buffer pre-filled with SENT, with SENT_ROWS more rows below it"""

    def __init__(self, c: ac.Case, q, k, v, rel, cg):
        self.c = c
        Cc = c.C
        if c.fused == "qkv":
            buf = torch.full((c.B * c.Lq, c.ldq), NAN)
            for col, t in ((c.cq, q), (c.ck, k), (c.cv, v)):
                buf[:, col:col + Cc] = t.reshape(-1, Cc)
            self.host = [buf]
            qb = kb = vb = 0
        else:
            assert c.fused == "kv" and c.ldk == c.ldv
            bq = torch.full((c.B * c.Lq, c.ldq), NAN)
            bq[:, c.cq:c.cq + Cc] = q.reshape(-1, Cc)
            bkv = torch.full((c.B * c.Lk, c.ldk), NAN)
            bkv[:, c.ck:c.ck + Cc] = k.reshape(-1, Cc)
            bkv[:, c.cv:c.cv + Cc] = v.reshape(-1, Cc)
            self.host = [bq, bkv]
            qb, kb, vb = 0, 1, 1
        self.bufs = [b.cuda() for b in self.host]
        self.rel, self.cg = rel.cuda(), cg.cuda()
        self.o0 = 32 + c.cq                                      # the output window: columns o0 .. o0+C
        self.out = torch.full((c.B * c.Lq + SENT_ROWS, Cc + 96), SENT).cuda()
        self.ops = OpList()
        self.ops.attention(view(self.bufs[qb], c.cq, c.cq + Cc), view(self.bufs[kb], c.ck, c.ck + Cc), view(self.bufs[vb], c.cv, c.cv + Cc),
                           View(self.out.data_ptr() + 4 * self.o0, self.out.shape[1], c.B * c.Lq, Cc), ptr(self.rel), ptr(self.cg),
                           c.B, c.H, c.Lq, c.Lk, c.pos_max)

    def output(self):
        """the output window [B, Lq, C] (host), and whether every element outside it still holds SENT"""
        c, o = self.c, self.out.cpu()
        n = c.B * c.Lq
        win = o[:n, self.o0:self.o0 + c.C].reshape(c.B, c.Lq, c.C).clone()
        o[:n, self.o0:self.o0 + c.C] = SENT
        return win, bool((o == SENT).all())

    def inputs_unchanged(self) -> bool:
        return all(torch.equal(_bits(d), _bits(h)) for d, h in zip(self.bufs, self.host))


def check_case(R, c: ac.Case, impl: int, tol=None, salt: str = "") -> float:
    kern = ac.kernel_for(c, impl)
    q, k, v, rel, cg = ac.make_inputs(c, salt)
    d = Device(c, q, k, v, rel, cg)
    with attention_impl(R, impl):
        R.run(d.ops)
        out, kept = d.output()
        first = d.out.clone()
        R.run(d.ops)
    assert kept, "a store left the output window"
    assert d.inputs_unchanged(), "q / k / v changed"
    assert torch.equal(_bits(first), _bits(d.out)), "two runs differ"
    err = 0.0
    for b in sorted({0, c.B // 2, c.B - 1}):
        ref, mag = ac.ref_attention(q[b:b + 1], k[b:b + 1], v[b:b + 1], rel, cg, c.H, c.pos_max, c.scale)
        err = max(err, ac.row_error(out[b:b + 1], ref, mag, c.H))
    tol = TOL[(kern, c.regime)] if tol is None else tol
    print(f"attention {kern} {c.regime} {c.id} row_err={err:.3e} tol={tol:.1e}")
    assert err < tol, (kern, c.regime, err)
    return err


# ---- the plans' attention signatures -------------------------------------------------------------------------------------------
def test_plan_signatures():
    """(no GPU) the attention ops of real plans: every U-Net plan has 16 self-attentions (Lk = Lq, q / k / v windows 0, C, 2C of one
    3C buffer) and 16 cross-attentions to the 21 prompt tokens (k / v windows 0, C of one 2C buffer), every wave-encoder plan 12
    self-attentions; together they reach head dims 32 / 48 / 64 and both the wgmma and the lane-per-key kernel.  PLAN_CASES, which
    the GPU tests run, is exactly their set of distinct signatures: a change of the plans has to bring the case list along."""
    ops = ac.plan_attention_ops()
    for (kind, B, L), cases in ops.items():
        if kind == "unet":
            assert len(cases) == 32
            self_ = [c for c in cases if c.fused == "qkv"]
            cross = [c for c in cases if c.fused == "kv"]
            assert len(self_) == 16 and len(cross) == 16
            for c in self_:
                assert c.Lk == c.Lq and c.ldq == c.ldk == c.ldv == 3 * c.C and (c.cq, c.ck, c.cv) == (0, c.C, 2 * c.C)
            for c in cross:
                assert c.Lk == 21 and c.ldk == c.ldv == 2 * c.C and (c.ck, c.cv) == (0, c.C)
        else:
            assert kind == "wave" and len(cases) == 12
            for c in cases:
                assert c.fused == "qkv" and c.Lk == c.Lq and (c.cq, c.ck, c.cv) == (0, c.C, 2 * c.C)
        for c in cases:
            assert c.B == B and c.pos_max == 64 and (c.ldo, c.co) == (c.C, 0)
    sig = ac.plan_signatures()
    assert len(sig) == len(ac.PLAN_CASES) and set(sig) == set(ac.PLAN_CASES)
    assert {c.D for c in sig} == {32, 48, 64}
    assert {ac.kernel_for(c, 1) for c in sig} == {"tc", "lane"}


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["plan", "ffma"])
@pytest.mark.parametrize("case", ac.PLAN_CASES, ids=[c.id for c in ac.PLAN_CASES])
def test_plan_case(R, case, impl):
    check_case(R, case, impl)


# ---- edges of each kernel ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["plan", "ffma"])
@pytest.mark.parametrize("name", list(ac.EDGE_CASES))
def test_edge_case(R, name, impl):
    """names carry the kernel the case is meant for with impl 1 ("-tc-" or "-lane-"); impl 0 runs it through the FFMA referee"""
    c = ac.EDGE_CASES[name]
    assert ac.kernel_for(c, 1) == ("tc" if "-tc-" in name else "lane"), name
    check_case(R, c, impl)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["plan", "ffma"])
@pytest.mark.parametrize("Lk", [21, 150])
def test_rejects_misaligned_window(R, Lk, impl):
    """windows must start on 16 bytes (a multiple of 4 columns): a window 2 columns in is refused, not read misaligned"""
    c = ac.layout(1, 8, 48, 40, Lk, fused="kv", pad=2)
    d = Device(c, *ac.make_inputs(c))
    with attention_impl(R, impl), pytest.raises(L_.MugdError, match="alignment"):
        R.run(d.ops)
    assert d.output()[1]


# ---- ordering inside a captured plan ---------------------------------------------------------------------------------------------
def make_plan(R, ops: OpList):
    for op in ops.ops:
        if op.kind == L_.OP_GEMM:
            gm = op.u.gemm
            gm.workspace, gm.workspace_bytes = R.ws.data_ptr(), R.ws.numel() * 4
            gm.counters, gm.n_counters = R.counters.data_ptr(), R.counters.numel()
    arr = ops.array()
    plan = C.c_void_p()
    L_.check(R.lib.mugd_plan_create(R.handle, arr, len(ops.ops), C.byref(plan)), "plan_create")
    return plan


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 32])
def test_captured_plan_orders_attention_between_gemms(R, D):
    """[wgmma GEMM -> qkv ; attention over the qkv windows -> ao ; wgmma GEMM over ao] captured on a side stream with programmatic
    launch edges (PDL, the default) and replayed once over qkv / ao / out filled with NaN: bit-identical to the ops run one by one.
    An attention that read qkv before the first GEMM finished, or a GEMM that read ao early, would leave NaN or different bits."""
    B, L, H, K = 8, 512, 8, 256
    Cc = H * D
    g = torch.Generator().manual_seed(11 + D)
    x = torch.randn(B * L, K, generator=g)
    w1, w2 = torch.randn(3 * Cc, K, generator=g) / math.sqrt(K), torch.randn(Cc, Cc, generator=g) / math.sqrt(Cc)
    rel, cg = torch.randn(129, H, generator=g), 1 + 0.25 * torch.randn(129, H, generator=g)
    dev = [t.cuda() for t in (x, w1, *tf32_split(w1), w2, *tf32_split(w2), rel, cg)]
    xc, w1c, w1h, w1l, w2c, w2h, w2l, relc, cgc = dev
    qkv, ao, out = (torch.full((B * L, n), NAN).cuda() for n in (3 * Cc, Cc, Cc))
    ops = OpList()
    ops.gemm(view(xc), ptr(w1c), 3 * Cc, K, view(qkv), W_hi=ptr(w1h), W_lo=ptr(w1l), impl=L_.GEMM_TC)
    ops.attention(view(qkv, 0, Cc), view(qkv, Cc, 2 * Cc), view(qkv, 2 * Cc, 3 * Cc), view(ao), ptr(relc), ptr(cgc), B, H, L, L, 64)
    ops.gemm(view(ao), ptr(w2c), Cc, Cc, view(out), W_hi=ptr(w2h), W_lo=ptr(w2l), impl=L_.GEMM_TC)
    plan = make_plan(R, ops)
    st = torch.cuda.Stream()
    try:
        L_.check(R.lib.mugd_set_pdl(1), "pdl")
        R.run(ops)                                                # eager, one op at a time
        eager = [t.clone() for t in (qkv, ao, out)]
        assert all(bool(torch.isfinite(t).all()) for t in eager)
        for t in (qkv, ao, out):
            t.fill_(NAN)
        torch.cuda.synchronize()
        L_.check(R.lib.mugd_plan_capture(plan, C.c_void_p(st.cuda_stream)), "capture")
        assert bool(torch.isnan(out).all())                       # capturing runs nothing
        L_.check(R.lib.mugd_plan_replay(plan, 1, C.c_void_p(st.cuda_stream)), "replay")
        st.synchronize()
        for name, e, t in zip(("qkv", "ao", "out"), eager, (qkv, ao, out)):
            assert torch.equal(_bits(e), _bits(t)), name
    finally:
        R.lib.mugd_set_pdl(int(os.environ.get("MUGD_PDL", "1") != "0"))
        R.lib.mugd_plan_destroy(plan)


# ---- small shapes of every kernel (moved from test_gpu_ops.py) -----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("impl", [1, 0], ids=["wgmma", "ffma"])
@pytest.mark.parametrize("B,H,D,Lq,Lk", [(2, 8, 32, 48, 48), (2, 8, 48, 24, 21), (1, 8, 64, 200, 200), (2, 8, 32, 256, 256),
                                         (1, 8, 64, 124, 124), (3, 8, 48, 130, 21), (1, 8, 32, 496, 496), (1, 8, 48, 300, 300),
                                         (2, 8, 64, 12, 12), (1, 4, 64, 129, 257), (8, 8, 64, 64, 21), (8, 8, 32, 256, 21), (2, 8, 48, 128, 32),
                                         (1, 8, 32, 70, 1), (2, 8, 64, 33, 33)])
def test_attention(R, B, H, D, Lq, Lk, impl):
    """the attention kernels (tensor-core 3xTF32, lane-per-key for <= 32 keys, and the exact FFMA referee) against the fp64 formula;
    covers several key tiles, ragged last tiles (Lk % 16 != 0), Lq < one tile, the 21-token prompt context, 1 / 32 / 33 keys.
    q is the first window of a 3C-wide buffer, k and v are contiguous; every sample against the reference."""
    Cc = H * D
    c = ac.Case(B, H, D, Lq, Lk, 64, 3 * Cc, 0, Cc, 0, Cc, 0, Cc, 0, "kv")
    q, k, v, rel, cg = ac.make_inputs(c)
    qkv = torch.zeros(B * Lq, 3 * Cc)
    qkv[:, :Cc] = q.reshape(-1, Cc)
    qkv, kc, vc = qkv.cuda(), k.reshape(-1, Cc).cuda(), v.reshape(-1, Cc).cuda()
    out = torch.zeros(B * Lq, Cc).cuda()
    relc, cgc = rel.cuda(), cg.cuda()
    ops = OpList()
    ops.attention(view(qkv, 0, Cc), view(kc), view(vc), view(out), ptr(relc), ptr(cgc), B, H, Lq, Lk, 64)
    with attention_impl(R, impl):
        R.run(ops)
    ref, mag = ac.ref_attention(q, k, v, rel, cg, H, 64, c.scale)
    err = ac.row_error(out.cpu().view(B, Lq, Cc), ref, mag, H)
    print(f"attention {ac.kernel_for(c, impl)} randn {c.id} row_err={err:.3e}")
    assert err < TOL[(ac.kernel_for(c, impl), "randn")]
