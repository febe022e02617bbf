"""The GroupNorm(+SiLU) kernels -- groupnorm_silu_reg_kernel<2|4|8|16|32> (the slab of a group in registers) and the two-pass
groupnorm_silu_kernel -- and layernorm_kernel (csrc/norm.cu) against the float64 statement of the ops in norm_cases.py:

* every norm signature of the real U-Net, decoder, encoder and wave-encoder plans, with x and y laid out as the plans lay them out
  (column windows of concat buffers), in the randn and offset regimes;
* hand-picked edges: both sides of every register-kernel boundary, one-row groups, LayerNorm widths 4 .. 1024 at 1, 7, 8, 9 rows,
  windows with ldx != ldy, and five data regimes (norm_cases.make_inputs) on every kernel;
* PDL ordering inside a captured plan: GEMM -> GroupNorm(+SiLU) -> GEMM replayed from a graph equals the same ops run one by one;
* the launchers' refusals of malformed descriptors (mugd_op_run is public ABI).

Error bound, element by element:  |y - ref| <= K 2^-24 (A + |ref|),  A = ((|x| + |m|) r |gamma| + |beta|) (x 1.1 with SiLU), with m
and r = 1 / sqrt(var + eps) the float64 moments of the group or row.  The fp32 rounding of the mean alone moves x - m by 2^-24 |m|,
so A grows with the conditioning |m| / spread, and the bound stays tight on well-conditioned data.  K per (kernel, regime) is in TOL.
The bound is checked for samples 0, B/2 and B-1; every sample is checked for stores outside the output window, untouched inputs
and bit-identical reruns."""
import ctypes as C
import math
import os
from dataclasses import replace

import pytest
import torch

import norm_cases as nc
from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200.engine import OpList, View
from mug_diffusion_b200.packer import tf32_split

from gpu_util import OpRunner, ptr, view

SENT = -7777.0           # pre-fill of the output buffer: every element outside the output window must keep it
SPARE = 8                # spare rows above and below each window, NaN (input) or SENT (output)
NAN = float("nan")       # fill of the input buffer outside the x window: a stray read poisons the moments

# (kernel, data regime) -> K, about 3x the largest ratio |y - ref| / (2^-24 (A + |ref|)) over all cases of this file on an H100
# 80GB HBM3 (700 W power limit):
#            randn   offset  flat    tiny    wide
#   reg2     2.58    0.74    2.05    1.05    2.04
#   reg4     2.79    0.79    2.37    1.33    2.18
#   reg8     2.96    0.69    2.48    1.24    1.79
#   reg16    2.77    0.93    2.48    1.16    1.52
#   reg32    2.65    0.52    2.45    1.40    1.43
#   two      2.84    0.53    2.39    1.19    1.25
#   ln       21.50   1.70    4.08    1.43    43.79
# GroupNorm forms its moments in fp64, so its mean is off by the fp32 rounding of m alone.  layernorm_kernel sums in fp32: its mean
# is off by a few 2^-24 sum|x| / C, which exceeds 2^-24 |m| where the row mean is small next to the row's entries (randn: |m| ~
# C^-1/2) or one entry dominates the sum (wide), hence its larger K there.  With the moments in fp32 (E[x^2] - m^2) either kernel
# lands at 1e3 .. 1e4 in the offset regime (test_bound_separates_fp64_from_fp32_moments).
TOL = {
    ("reg2", "randn"): 8, ("reg2", "offset"): 2.5, ("reg2", "flat"): 6.5, ("reg2", "tiny"): 3.5, ("reg2", "wide"): 6.5,
    ("reg4", "randn"): 8.5, ("reg4", "offset"): 2.5, ("reg4", "flat"): 7.5, ("reg4", "tiny"): 4, ("reg4", "wide"): 7,
    ("reg8", "randn"): 9, ("reg8", "offset"): 2.5, ("reg8", "flat"): 7.5, ("reg8", "tiny"): 4, ("reg8", "wide"): 5.5,
    ("reg16", "randn"): 8.5, ("reg16", "offset"): 3, ("reg16", "flat"): 7.5, ("reg16", "tiny"): 3.5, ("reg16", "wide"): 5,
    ("reg32", "randn"): 8, ("reg32", "offset"): 2, ("reg32", "flat"): 7.5, ("reg32", "tiny"): 4.5, ("reg32", "wide"): 4.5,
    ("two", "randn"): 9, ("two", "offset"): 2, ("two", "flat"): 7.5, ("two", "tiny"): 4, ("two", "wide"): 4,
    ("ln", "randn"): 64.5, ("ln", "offset"): 5.5, ("ln", "flat"): 12.5, ("ln", "tiny"): 4.5, ("ln", "wide"): 131.5,
}


@pytest.fixture(scope="module")
def R():
    return OpRunner()


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().view(torch.int32)


class Device:
    """a case's operands on the GPU: x the window (rows SPARE.., columns cx..) of an ldx-wide buffer whose other elements are NaN, y the
    window (rows SPARE.., columns cy..) of an ldy-wide buffer pre-filled with SENT"""

    def __init__(self, c: nc.Case, x, gamma, beta):
        self.c = c
        n = c.B * c.L
        self.xbuf = torch.full((n + 2 * SPARE, c.ldx), NAN, device="cuda")
        self.xbuf[SPARE:SPARE + n, c.cx:c.cx + c.C] = x
        self.ybuf = torch.full((n + 2 * SPARE, c.ldy), SENT, device="cuda")
        self.gamma, self.beta = gamma.cuda(), beta.cuda()
        self.saved = [t.clone() for t in (self.xbuf, self.gamma, self.beta)]
        xv = View(self.xbuf.data_ptr() + 4 * (SPARE * c.ldx + c.cx), c.ldx, n, c.C)
        yv = View(self.ybuf.data_ptr() + 4 * (SPARE * c.ldy + c.cy), c.ldy, n, c.C)
        self.ops = OpList()
        if c.is_ln:
            self.ops.layernorm(xv, yv, ptr(self.gamma), ptr(self.beta))
        else:
            self.ops.groupnorm(xv, yv, ptr(self.gamma), ptr(self.beta), c.B, c.L, c.G, bool(c.silu))

    def window(self, buf=None) -> torch.Tensor:
        c = self.c
        buf = self.ybuf if buf is None else buf
        return buf[SPARE:SPARE + c.B * c.L, c.cy:c.cy + c.C]

    def outside_kept(self) -> bool:
        o = self.ybuf.clone()
        self.window(o).fill_(SENT)
        return bool((o == SENT).all())

    def inputs_unchanged(self) -> bool:
        return all(torch.equal(_bits(a), _bits(b)) for a, b in zip((self.xbuf, self.gamma, self.beta), self.saved))


def check_case(R, c: nc.Case) -> float:
    kern = nc.kernel_for(c)
    x, gamma, beta = nc.make_inputs(c, "cuda")
    d = Device(c, x, gamma, beta)
    R.run(d.ops)
    first = d.ybuf.clone()
    R.run(d.ops)
    assert d.outside_kept(), "a store left the output window"
    assert d.inputs_unchanged(), "x / gamma / beta changed"
    assert torch.equal(_bits(first), _bits(d.ybuf)), "two runs differ"
    y = d.window()
    if c.regime == "flat" and not c.silu and not c.is_ln:
        # the fp64 moments give the float mean of a constant group exactly, so x - mean is 0 whatever r is: the output is beta bit
        # for bit (the LayerNorm's fp32 mean of a constant row is rounded; it is held to the bound only)
        yg, bg = nc._grouped(y, c), nc._grouped(d.beta.expand(y.shape), c)
        mask = nc.flat_groups(c).cuda().expand(yg.shape)
        assert torch.equal(_bits(yg[mask]), _bits(bg[mask])), "a constant group is not mapped to beta"
    rows = c.L if c.is_ln else c.B * c.L
    samples = [slice(0, rows)] if c.is_ln else [slice(b * c.L, (b + 1) * c.L) for b in sorted({0, c.B // 2, c.B - 1})]
    ratio = 0.0
    for s in samples:
        sub = nc.ln(c.L, c.C) if c.is_ln else nc.gn(1, c.L, c.C, c.G, c.silu)
        ref, A = nc.reference(x[s], gamma, beta, sub)
        ratio = max(ratio, nc.bound_ratio(y[s], ref, A))
    tol = TOL[(kern, c.regime)]
    print(f"norm {kern} {c.regime} {c.id} ratio={ratio:.3f} K={tol}")
    assert ratio <= tol, (kern, c.regime, ratio)
    return ratio


# ---- the plans' norm signatures ------------------------------------------------------------------------------------------------
def test_plan_signatures():
    """(no GPU) the norm ops of real plans: 77 GroupNorms per U-Net evaluation, and 48 LayerNorms where the fold is off
    (Beff * Lz >= 8192); 21 GroupNorms per decoder plan and 13 per encoder plan (G = 8); 46 GroupNorms and 18 LayerNorms per
    wave-encoder plan.  PLAN_CASES, which the GPU tests run, is exactly their set of distinct signatures."""
    ops = nc.plan_norm_ops()
    for (kind, B, L), cases in ops.items():
        ngn = sum(not c.is_ln for c in cases)
        nln = sum(c.is_ln for c in cases)
        if kind == "unet":
            assert (ngn, nln) == (77, 48 if B * L >= 8192 else 0), (kind, B, L)
        else:
            assert (ngn, nln) == {"decoder": (21, 0), "encoder": (13, 0), "wave": (46, 18)}[kind], (kind, B, L)
        for c in cases:
            assert c.is_ln or (c.B == B and c.G == (32 if kind in ("unet", "wave") else 8))
            assert (c.ldy, c.cy) == (c.C, 0)
            assert (c.ldx, c.cx) in ((c.C, 0), (2 * c.C, c.C), (3 * c.C, 2 * c.C)) and (c.ldx == c.C or kind == "unet")
    sig = nc.plan_signatures()
    assert len(sig) == len(nc.PLAN_CASES) and set(sig) == set(nc.PLAN_CASES)


def test_cases_reach_every_kernel():
    """(no GPU) the plan signatures alone run all six GroupNorm kernels and the LayerNorm kernel; the boundary cases of every group
    width sit on both sides of each register-kernel boundary (so they too reach all six); the regime shapes sit on the kernels
    their names carry"""
    assert {nc.kernel_for(c) for c in nc.PLAN_CASES} == set(nc.GN_KERNELS) | {"ln"}
    for cg in (4, 12, 20, 44, 48):
        slabs = [c for name, c in nc.EDGE_CASES.items() if name.startswith("slab") and name.endswith(f"-cg{cg}")]
        assert len(slabs) == 10 and {nc.kernel_for(c) for c in slabs} == set(nc.GN_KERNELS), cg
    for kern, shape in nc.REGIME_SHAPES.items():
        assert nc.kernel_for(nc.gn(*shape, 0)) == kern


def _bound_cases():
    """small cases of every regime for the host emulation, GroupNorm with and without SiLU and LayerNorm"""
    for regime in nc.REGIMES:
        for c in (nc.gn(3, 64, 128, 32, 0, regime=regime), nc.gn(3, 200, 256, 8, 1, regime=regime), nc.gn(3, 1, 1536, 32, 1, regime=regime)):
            yield c
        for C in (256, 1024):
            yield nc.ln(50, C, regime=regime)


def test_bound_separates_fp64_from_fp32_moments():
    """(no GPU) the kernels' arithmetic emulated on the host meets the bound with the smallest K of its regime; the same arithmetic
    with the moments in fp32 (E[x^2] - m^2 cancels) breaks the largest K of the offset regime by far.  Loosening TOL until a kernel
    with fp32 moments passes breaks this test."""
    for c in _bound_cases():
        x, gamma, beta = nc.make_inputs(c)
        ref, A = nc.reference(x, gamma, beta, c)
        if c.is_ln:
            good, bad = nc.emulate_layernorm(x, gamma, beta), nc.emulate_layernorm(x, gamma, beta, "raw")
            kernels = ["ln"]
        else:
            good, bad = nc.emulate_groupnorm(x, gamma, beta, c), nc.emulate_groupnorm(x, gamma, beta, c, "fp32")
            kernels = list(nc.GN_KERNELS)
        r_good, r_bad = nc.bound_ratio(good, ref, A), nc.bound_ratio(bad, ref, A)
        print(f"emulated {c.id}: ratio {r_good:.3f} (fp32 moments {r_bad:.3g})")
        assert r_good <= min(TOL[(k, c.regime)] for k in kernels), (c.id, r_good)
        if c.regime == "offset":
            assert r_bad > 10 * max(TOL[(k, c.regime)] for k in kernels), (c.id, r_bad)


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["randn", "offset"])
@pytest.mark.parametrize("case", nc.PLAN_CASES, ids=[c.id for c in nc.PLAN_CASES])
def test_plan_case(R, case, regime):
    check_case(R, replace(case, regime=regime))


# ---- edges of each kernel ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(nc.EDGE_CASES))
def test_edge_case(R, name):
    check_case(R, nc.EDGE_CASES[name])


# ---- refusals --------------------------------------------------------------------------------------------------------------------
def _refused(R, x: View, y: View, ybuf, match, G=None, B=1):
    g = torch.ones(2048, device="cuda")
    ops = OpList()
    if G is None:
        ops.layernorm(x, y, ptr(g), ptr(g))
    else:
        ops.groupnorm(x, y, ptr(g), ptr(g), B, x.rows // B if B else 0, G, True)
    with pytest.raises(L_.MugdError, match=match):
        R.run(ops)
    assert bool((ybuf == SENT).all()), "a refused op wrote its output"


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["groupnorm", "layernorm"])
@pytest.mark.parametrize("what", ["misaligned", "ld_lt_C", "empty"])
def test_rejects_bad_views(R, op, what):
    """a window 2 columns in (not 16-byte aligned), a leading dimension smaller than C, and an empty shape are refused"""
    G = 8 if op == "groupnorm" else None
    x, y = torch.zeros(64, 136, device="cuda"), torch.full((64, 136), SENT, device="cuda")
    Cc = 128
    if what == "misaligned":
        xv, yv, match = view(x, 2, 2 + Cc), view(y, 0, Cc), "16-byte aligned"
    elif what == "ld_lt_C":
        xv, yv, match = View(x.data_ptr(), Cc - 4, 64, Cc), view(y, 0, Cc), "leading dimension smaller than C"
    else:
        xv, yv, match = View(x.data_ptr(), 136, 0, Cc), View(y.data_ptr(), 136, 0, Cc), "empty shape"
    _refused(R, xv, yv, y, f"{op}: .*{match}" if what != "empty" else f"{op}: empty shape", G=G, B=0 if what == "empty" else 1)


@pytest.mark.gpu
@pytest.mark.parametrize("C,G", [(96, 32), (40, 20), (100, 32)])
def test_groupnorm_rejects_group_width(R, C, G):
    """C/G must be a multiple of 4 (every float4 belongs to one group)"""
    x, y = torch.zeros(16, C, device="cuda"), torch.full((16, C), SENT, device="cuda")
    _refused(R, view(x), view(y), y, r"groupnorm: C/G must be a multiple of 4", G=G, B=2)


@pytest.mark.gpu
@pytest.mark.parametrize("Cc", [1028, 6])
def test_layernorm_rejects_width(R, Cc):
    """one warp holds a row in 8 float4 per lane: C a multiple of 4 up to 1024"""
    x, y = torch.zeros(16, 1032, device="cuda"), torch.full((16, 1032), SENT, device="cuda")
    _refused(R, view(x, 0, Cc), view(y, 0, Cc), y, r"layernorm: C=%d must be a multiple of 4 and <= 1024" % Cc)


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
@pytest.mark.parametrize("B,L,Cc,G", [(8, 512, 256, 32), (2, 2048, 256, 8)], ids=["reg4", "two"])
def test_captured_plan_orders_groupnorm_between_gemms(R, B, L, Cc, G):
    """[wgmma GEMM -> h ; GroupNorm+SiLU h -> n ; wgmma GEMM over n] captured on a side stream with programmatic launch edges (PDL,
    the default) and replayed once over h / n / out filled with NaN: bit-identical to the ops run one by one.  A GroupNorm that read h
    before the first GEMM finished, or a GEMM that read n early, would leave NaN or different bits."""
    K = 256
    assert nc.kernel_for(nc.gn(B, L, Cc, G, 1)) == ("two" if G == 8 else "reg4")
    g = torch.Generator().manual_seed(L + G)
    x = torch.randn(B * L, K, generator=g)
    w1, w2 = torch.randn(Cc, K, generator=g) / math.sqrt(K), torch.randn(Cc, Cc, generator=g) / math.sqrt(Cc)
    gamma, beta = 1 + 0.5 * torch.randn(Cc, generator=g), 0.5 * torch.randn(Cc, generator=g)
    dev = [t.cuda() for t in (x, w1, *tf32_split(w1), w2, *tf32_split(w2), gamma, beta)]
    xc, w1c, w1h, w1l, w2c, w2h, w2l, gc, bc = dev
    h, n, out = (torch.full((B * L, Cc), NAN).cuda() for _ in range(3))
    ops = OpList()
    ops.gemm(view(xc), ptr(w1c), Cc, K, view(h), W_hi=ptr(w1h), W_lo=ptr(w1l), impl=L_.GEMM_TC)
    ops.groupnorm(view(h), view(n), ptr(gc), ptr(bc), B, L, G, True)
    ops.gemm(view(n), ptr(w2c), Cc, Cc, view(out), W_hi=ptr(w2h), W_lo=ptr(w2l), impl=L_.GEMM_TC)
    plan = make_plan(R, ops)
    st = torch.cuda.Stream()
    try:
        L_.check(R.lib.mugd_set_pdl(1), "pdl")
        R.run(ops)                                                # eager, one op at a time
        eager = [t.clone() for t in (h, n, out)]
        assert all(bool(torch.isfinite(t).all()) for t in eager)
        for t in (h, n, out):
            t.fill_(NAN)
        torch.cuda.synchronize()
        L_.check(R.lib.mugd_plan_capture(plan, C.c_void_p(st.cuda_stream)), "capture")
        assert bool(torch.isnan(out).all())                       # capturing runs nothing
        L_.check(R.lib.mugd_plan_replay(plan, 1, C.c_void_p(st.cuda_stream)), "replay")
        st.synchronize()
        for name, e, t in zip(("h", "n", "out"), eager, (h, n, out)):
            assert torch.equal(_bits(e), _bits(t)), name
    finally:
        R.lib.mugd_set_pdl(int(os.environ.get("MUGD_PDL", "1") != "0"))
        R.lib.mugd_plan_destroy(plan)
