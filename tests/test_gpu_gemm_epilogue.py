"""Fused epilogues of the wgmma GEMM (gemm_tc.cuh) on both of its store paths -- the direct tile store (tc_store_tile, split_k = 1)
and the split-K second pass (tc_reduce), which finishes most output tiles of a small-batch U-Net evaluation -- against ONE fp64
statement of mugd_gemm (ref_gemm below), with every operand each epilogue takes: bias, the time-embedding row (per sample and
chosen by the device step counter), A / residual / output column windows, the second source, the row-moment sink and the folded
LayerNorm.  Also the step counter under CUDA-graph replay and the opt-in single-pass TF32 mode.

Tolerances are those of test_gpu_gemm_tc.py / test_gpu_fusion.py: 1e-5 of max |ref| (2e-5 with the folded LayerNorm)."""
import ctypes as C
import math
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from mug_diffusion_b200 import lib as L_  # noqa: E402
from mug_diffusion_b200 import synth  # noqa: E402
from mug_diffusion_b200.engine import OpList, View  # noqa: E402
from mug_diffusion_b200.packer import tf32_split  # noqa: E402

from gpu_util import OpRunner, ptr, rel_err, view  # noqa: E402

TOL, TOL_LN = 1e-5, 2e-5
SENT = 7777.0            # pre-fill of output buffers: every element outside the output window must keep it
STEPS, STEP = 5, 3       # rows of the step-indexed time-embedding table, value of the device step counter
LN_EPS = 1e-5


def ref_gemm(A, W, *, B, Lin, Lout, K, taps=1, mode=L_.CONV_NONE, tap_shift=0, dilation=1, A2=None, bias=None, rowvec=None,
             rowvec_b_stride=0, rowvec_step_stride=0, step=0, act=L_.ACT_NONE, gate=L_.GATE_NONE, residual=None, ln=None):
    """mugd_gemm (include/mugd.h) in float64 on the operands as the kernel reads them.
    A [B*Lin, K], A2 [B*Lout, K2], W [N, taps*K + K2] (tap-major K blocks, then the K2 columns of the second source).
    Output row l of sample b reads source row  l (NONE), l+t-1 (SAME), 2l+t (DOWN: stride 2, right pad), l+(t+tap_shift)*dilation
    (TAPS); rows outside [0, Lin) are zero.  Then the folded LayerNorm  (acc - mean*colsum) * rstd  with mean / rstd from the row
    moments ln = (stats [M, 2] = {sum, sum of squares} over K, colsum [N], eps); + bias[n];
    + rowvec[step*rowvec_step_stride + b*rowvec_b_stride + n]; act; gate on the interleaved accumulator columns (2j, 2j+1) =
    (value_j, gate_j), the weight-row order packer._interleave_halves produces, -> N/2 columns; + residual."""
    N = W.shape[0]
    a = A.double().reshape(B, Lin, K)
    w = W.double()
    lo = torch.arange(Lout)
    y = torch.zeros(B, Lout, N, dtype=torch.float64)
    for t in range(taps):
        if mode == L_.CONV_NONE:
            assert taps == 1 and Lin == Lout
            src = lo
        elif mode == L_.CONV_SAME:
            src = lo + t - 1
        elif mode == L_.CONV_DOWN:
            src = 2 * lo + t
        elif mode == L_.CONV_TAPS:
            src = lo + (t + tap_shift) * max(dilation, 1)
        else:
            raise ValueError(mode)
        ok = (src >= 0) & (src < Lin)
        xs = torch.zeros(B, Lout, K, dtype=torch.float64)
        xs[:, ok] = a[:, src[ok]]
        y += xs @ w[:, t * K:(t + 1) * K].T
    if A2 is not None:
        y += A2.double().reshape(B, Lout, -1) @ w[:, taps * K:].T
    y = y.reshape(B * Lout, N)
    if ln is not None:
        stats, colsum, eps = ln
        mean = stats[:, 0] / K
        var = stats[:, 1] / K - mean ** 2
        y = (y - mean[:, None] * colsum.double()[None]) / torch.sqrt(var + eps)[:, None]
    if bias is not None:
        y = y + bias.double()
    if rowvec is not None:
        b = torch.arange(B * Lout) // Lout
        y = y + rowvec.double().reshape(-1)[step * rowvec_step_stride + b[:, None] * rowvec_b_stride + torch.arange(N)[None]]
    if act == L_.ACT_SILU:
        y = F.silu(y)
    elif act == L_.ACT_GELU:
        y = F.gelu(y)
    if gate != L_.GATE_NONE:
        v, gt = y[:, 0::2], y[:, 1::2]
        y = v * (F.gelu(gt) if gate == L_.GATE_GEGLU else torch.sigmoid(gt))
    if residual is not None:
        y = y + residual.double()
    return y


@dataclass(frozen=True)
class Case:
    B: int
    Lin: int
    Lout: int
    K: int
    N: int                      # weight rows = accumulator columns (output columns: N/2 when gated)
    taps: int = 1
    mode: int = L_.CONV_NONE
    shift: int = 0
    dilation: int = 1
    K2: int = 0
    act: int = L_.ACT_NONE
    gate: int = L_.GATE_NONE
    sink: bool = False
    ln: bool = False
    bias: bool = True
    rowvec: str = "both"        # time-embedding row: "both" = per sample AND by step, rowvec[step*B*N + b*N + n] of a [STEPS, B, N]
                                # table; "step" = by step only, [STEPS, N] (the U-Net's DDIM plan); "" = none
    residual: bool = True       # read from a column window
    parity: int = -1            # >= 0: output row m is buffer row 2m+parity (the parity-split Upsample); else a column window

    @property
    def M(self):
        return self.B * self.Lout

    @property
    def nout(self):
        return self.N // 2 if self.gate else self.N

    @property
    def ksteps(self):
        return (self.taps * self.K + self.K2) // 32

    @property
    def rowvec_strides(self):
        """(rowvec_b_stride, rowvec_step_stride)"""
        return (self.N, self.B * self.N) if self.rowvec == "both" else (0, self.N)


def g(name, shape, seed=31):
    return synth._gauss(synth._rng(seed, name), shape)


class Operands:
    """host tensors of one case (seeded by its name) and their fp64 result"""

    def __init__(self, c: Case, name: str):
        self.c = c
        kt = c.taps * c.K + c.K2
        self.A = g(name + ".A", (c.B * c.Lin, c.K))
        self.A2 = g(name + ".A2", (c.M, c.K2)) if c.K2 else None
        self.W = g(name + ".W", (c.N, kt)) / math.sqrt(kt)
        self.bias = 0.1 * g(name + ".b", (c.N,)) if c.bias else None
        self.table = None
        if c.rowvec:
            self.table = g(name + ".e", (STEPS, c.B, c.N) if c.rowvec == "both" else (STEPS, c.N))
        self.res = g(name + ".r", (c.M, c.nout + 32)) if c.residual else None      # the residual is columns 16 .. 16+nout
        self.ln = None
        if c.ln:
            a = self.A.double()
            stats = torch.stack([a.sum(1), (a * a).sum(1)], dim=1)
            self.ln = (stats, self.W.double().sum(1).float(), LN_EPS)

    def ref(self, step=STEP):
        c = self.c
        bs, ss = c.rowvec_strides
        return ref_gemm(self.A, self.W, B=c.B, Lin=c.Lin, Lout=c.Lout, K=c.K, taps=c.taps, mode=c.mode, tap_shift=c.shift,
                        dilation=c.dilation, A2=self.A2, bias=self.bias, rowvec=self.table, rowvec_b_stride=bs, rowvec_step_stride=ss,
                        step=step, act=c.act, gate=c.gate, residual=None if self.res is None else self.res[:, 16:16 + c.nout],
                        ln=self.ln)


class Device:
    """the operands of a case on the GPU, an output buffer pre-filled with SENT and the op list of the GEMM"""

    def __init__(self, o: Operands, split: int):
        c = o.c
        self.c = c
        a = torch.zeros(c.B * c.Lin, c.K + 64)                       # A is columns 32 .. 32+K of a wider buffer
        a[:, 32:32 + c.K] = o.A
        self.a = a.cuda()
        if c.K2:
            a2 = torch.zeros(c.M, c.K2 + 64)
            a2[:, 32:32 + c.K2] = o.A2
            self.a2 = a2.cuda()
        hi, lo = tf32_split(o.W)
        self.w, self.w_hi, self.w_lo = o.W.cuda(), hi.cuda(), lo.cuda()
        self.step = torch.tensor([STEP], dtype=torch.int32).cuda()
        kw = {}
        if c.bias:
            self.bias = o.bias.cuda()
            kw["bias"] = ptr(self.bias)
        if c.rowvec:
            self.table = o.table.cuda()
            bs, ss = c.rowvec_strides
            kw.update(rowvec=ptr(self.table), rowvec_b_stride=bs, rowvec_step_stride=ss, step=ptr(self.step))
        if c.residual:
            self.res = o.res.cuda()
        if c.parity >= 0:
            self.out = torch.full((2 * c.M, c.nout), SENT).cuda()
            dst = View(self.out.data_ptr() + 4 * c.parity * c.nout, 2 * c.nout, c.M, c.nout)
        else:
            self.out = torch.full((c.M, c.nout + 64), SENT).cuda()   # the output is columns 32 .. 32+nout
            dst = view(self.out, 32, 32 + c.nout)
        if c.ln:
            self.stats, self.colsum = o.ln[0].cuda(), o.ln[1].cuda()
            kw["ln"] = (self.stats.data_ptr(), ptr(self.colsum), LN_EPS)
        self.ops = OpList()
        self.i = self.ops.gemm(view(self.a, 32, 32 + c.K), ptr(self.w), c.N, c.K, dst, W_hi=ptr(self.w_hi), W_lo=ptr(self.w_lo),
                               taps=c.taps, mode=c.mode, Lin=c.Lin, Lout=c.Lout, act=c.act, gate=c.gate,
                               residual=view(self.res, 16, 16 + c.nout) if c.residual else None,
                               A2=view(self.a2, 32, 32 + c.K2) if c.K2 else None, tap_shift=c.shift, dilation=c.dilation,
                               impl=L_.GEMM_TC, split_k=split, **kw)
        self.moments = None
        if c.sink:
            self.moments = torch.zeros(c.M, 2, dtype=torch.float64).cuda()
            self.ops.ops[self.i].u.gemm.row_moments = self.moments.data_ptr()

    @property
    def gemm(self):
        return self.ops.ops[self.i].u.gemm

    def output(self):
        """the output window (host), and whether every element outside it still holds SENT"""
        c, o = self.c, self.out.cpu()
        if c.parity >= 0:
            win, rest = o[c.parity::2], o[1 - c.parity::2]
        else:
            win, rest = o[:, 32:32 + c.nout], torch.cat([o[:, :32], o[:, 32 + c.nout:]], dim=1)
        return win.clone(), bool((rest == SENT).all())


def sm_count(R):
    n = C.c_int32()
    L_.check(R.lib.mugd_device_info(R.handle, C.byref(n), None, None), "device_info")
    return n.value


def planned(R, gm):
    """(K splits, tile width) the planner picks for this GEMM on this device"""
    sp, bn = C.c_int32(), C.c_int32()
    L_.check(R.lib.mugd_gemm_tc_query(None, C.byref(gm), sm_count(R), None, C.byref(sp), None, None), "tc_query")
    L_.check(R.lib.mugd_gemm_tc_variant(C.byref(gm), sm_count(R), C.byref(bn), None, None), "tc_variant")
    return sp.value, bn.value


class tile_width:
    """mugd_debug_set_tc_tile_n for a block (process-wide: always reset to the cost model)"""

    def __init__(self, R, bn):
        self.R, self.bn = R, bn

    def __enter__(self):
        L_.check(self.R.lib.mugd_debug_set_tc_tile_n(self.bn), "tile_n")

    def __exit__(self, *exc):
        L_.check(self.R.lib.mugd_debug_set_tc_tile_n(0), "tile_n")


@pytest.fixture(scope="module")
def R():
    return OpRunner()


# ---- the epilogue x path x tile-width matrix ---------------------------------------------------------------------------------
EPIS = {
    "none": {}, "silu": dict(act=L_.ACT_SILU), "gelu": dict(act=L_.ACT_GELU), "geglu": dict(gate=L_.GATE_GEGLU),
    "glu": dict(gate=L_.GATE_GLU), "sink": dict(sink=True), "ln": dict(ln=True), "ln_geglu": dict(ln=True, gate=L_.GATE_GEGLU),
}
# L = 48: several samples share a 128-row tile, short last tile;  L = 200: a sample spans two tiles, ragged last tile
SHAPES = {"B3xL48": (3, 48), "B2xL200": (2, 200)}
SPLIT = 3                                            # the reduce path; every shape below has a k-step count that 3 does not divide


def matrix_case(epi, conv, shape):
    B, L = SHAPES[shape]
    e = dict(EPIS[epi])
    if e.get("ln"):              # the folded LayerNorm takes a single-source Linear without time-embedding row
        return Case(B, L, L, 224, 192, rowvec="", **e)
    if conv == "linear":         # + the second source: the transformer's ff_out GEMM (A2 + residual)
        return Case(B, L, L, 224, 192, K2=32, **e)
    return Case(B, L, L, 64, 192, taps=3, mode=L_.CONV_SAME, K2=32, **e)


MATRIX = [(e, c, s) for e in EPIS for c in ("linear", "conv3") for s in SHAPES if not (e.startswith("ln") and c == "conv3")]


def check_case(R, c: Case, name: str, split: int, bn: int, tol: float):
    o = Operands(c, name)
    ref = o.ref()
    force = bn if (bn == 64 and c.N >= 128) else 0
    with tile_width(R, force):
        d = Device(o, split)
        assert planned(R, d.gemm) == (split, bn)                   # the path under test is the one that runs
        R.run(d.ops)
        out, kept = d.output()
        d2 = Device(o, split)
        R.run(d2.ops)
        out2, _ = d2.output()
        if split > 1:
            dd = Device(o, 1)
            assert planned(R, dd.gemm) == (1, bn)
            R.run(dd.ops)
            direct, _ = dd.output()
    e = rel_err(out, ref)
    print(f"{name} split={split} bn={bn} rel_err={e:.2e}")
    assert e < tol
    assert kept, "a store left the output window"
    assert torch.equal(out, out2), "two runs differ"
    if split > 1:
        assert float((out - direct).abs().max()) < tol * float(ref.abs().max())
    if c.sink:
        s = out.double()
        exp = torch.stack([s.sum(1), (s * s).sum(1)], dim=1)
        assert float((d.moments.cpu() - exp).abs().max() / exp.abs().max()) < 1e-6


@pytest.mark.parametrize("bn", [128, 64])
@pytest.mark.parametrize("split", [1, SPLIT], ids=["direct", "reduce"])
@pytest.mark.parametrize("epi,conv,shape", MATRIX, ids=["-".join(m) for m in MATRIX])
def test_epilogue_matrix(R, epi, conv, shape, split, bn):
    c = matrix_case(epi, conv, shape)
    assert c.ksteps % SPLIT != 0                                   # the last split owns fewer k-steps (it_rem != 0)
    check_case(R, c, f"{epi}-{conv}-{shape}", split, bn, TOL_LN if c.ln else TOL)


# ---- strided / tap addressing and narrow outputs, on both paths (tile width: the cost model's) ----------------------------------
EXTRA = {
    # Downsample (stride-2 conv, right pad) into a column window
    "down": (Case(3, 96, 48, 96, 128, taps=3, mode=L_.CONV_DOWN), 2, 128),
    # one parity half of the Upsample: 2 taps, output rows 2m+1 of a buffer whose even rows stay untouched
    "taps_upsample": (Case(2, 100, 100, 96, 128, taps=2, mode=L_.CONV_TAPS, shift=-1, parity=1), 4, 128),
    # dilated taps (wave.py), 64-wide tile from N < 128
    "taps_dilated": (Case(2, 70, 70, 64, 64, taps=3, mode=L_.CONV_TAPS, shift=-1, dilation=2), 4, 64),
    # the U-Net's 16-channel output conv: a 64-wide tile of which 16 columns exist
    "conv3_n16": (Case(2, 200, 200, 128, 16, taps=3, mode=L_.CONV_SAME), 5, 64),
    # gated, N < 128: the 64-wide tile is not filled (40 output columns)
    "glu_n80": (Case(3, 48, 48, 96, 80, gate=L_.GATE_GLU), 2, 64),
}


@pytest.mark.parametrize("path", ["direct", "reduce"])
@pytest.mark.parametrize("name", list(EXTRA))
def test_addressing_modes(R, name, path):
    c, split, bn = EXTRA[name]
    assert c.ksteps % split != 0
    check_case(R, c, name, 1 if path == "direct" else split, bn, TOL)


# ---- one captured graph serves every DDIM step --------------------------------------------------------------------------------
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


@pytest.mark.parametrize("split", [1, 4], ids=["direct", "reduce"])
def test_step_counter_under_graph_replay(R, split):
    """[ResBlock conv3 + time-embedding row of the current step ; STEP_ADVANCE] captured once, replayed once per step: replay i
    adds table row i (mugd.h: step-dependent rows are selected on the device, so one graph serves all steps)"""
    c = Case(2, 200, 200, 64, 192, taps=3, mode=L_.CONV_SAME, rowvec="step", residual=False)
    assert c.ksteps % 4 != 0
    o = Operands(c, "graph")
    d = Device(o, split)
    d.step.zero_()
    assert planned(R, d.gemm)[0] == split
    adv = L_.StepAdvance()
    adv.step = ptr(d.step)
    d.ops.add(L_.OP_STEP_ADVANCE, adv)
    plan = make_plan(R, d.ops)
    st = torch.cuda.Stream()
    try:
        torch.cuda.synchronize()
        L_.check(R.lib.mugd_plan_capture(plan, C.c_void_p(st.cuda_stream)), "capture")
        assert int(d.step.item()) == 0                             # capturing runs nothing
        for i in range(STEPS):
            d.out.fill_(SENT)
            torch.cuda.synchronize()
            L_.check(R.lib.mugd_plan_replay(plan, 1, C.c_void_p(st.cuda_stream)), "replay")
            st.synchronize()
            out, kept = d.output()
            assert rel_err(out, o.ref(step=i)) < TOL, i
            assert kept
        assert int(d.step.item()) == STEPS
    finally:
        R.lib.mugd_plan_destroy(plan)


# ---- opt-in single-pass TF32 ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def R1():
    """a second handle: the single-pass switch is per handle"""
    r = OpRunner()
    yield r
    r.lib.mugd_set_tc_single_pass_tf32(r.handle, 0)
    r.lib.mugd_destroy(r.handle)


@pytest.mark.parametrize("split", [1, SPLIT], ids=["direct", "reduce"])
def test_single_pass_tf32(R, R1, split):
    """plain TF32 products: each element within 2^-9 (|A| |W|^T) of fp64 (two round-to-nearest TF32 operands: <= 2^-10 per product,
    the rest is headroom for fp32 accumulation) and clearly worse than 3xTF32, so the mode is in effect.  The mode is read at every
    launch: a graph captured with it keeps it, eager runs take the current one."""
    c = Case(2, 200, 200, 64, 192, taps=3, mode=L_.CONV_SAME, K2=32, bias=False, rowvec="", residual=False)
    o = Operands(c, "tf32")
    ref = o.ref()
    bound = 2.0 ** -9 * ref_gemm(o.A.abs(), o.W.abs(), B=c.B, Lin=c.Lin, Lout=c.Lout, K=c.K, taps=3, mode=L_.CONV_SAME, A2=o.A2.abs())
    d0 = Device(o, split)                                          # on a handle that never switched
    assert planned(R, d0.gemm)[0] == split
    R.run(d0.ops)
    exact, _ = d0.output()
    lib, h = R1.lib, R1.handle
    plan = None
    try:
        L_.check(lib.mugd_set_tc_single_pass_tf32(h, 1), "single_pass")
        d = Device(o, split)
        R1.run(d.ops)
        sp, kept = d.output()
        assert kept
        err = (sp.double() - ref).abs()
        assert bool((err <= bound).all()), float((err / bound).max())
        e = rel_err(sp, ref)
        print(f"single-pass TF32 split={split} rel_err={e:.2e} (3xTF32: {rel_err(exact, ref):.2e})")
        assert e > TOL
        # a graph captured in single-pass mode keeps it after the switch goes off
        dg = Device(o, split)
        plan = make_plan(R1, dg.ops)
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        L_.check(lib.mugd_plan_capture(plan, C.c_void_p(st.cuda_stream)), "capture")
        L_.check(lib.mugd_set_tc_single_pass_tf32(h, 0), "single_pass")
        L_.check(lib.mugd_plan_replay(plan, 1, C.c_void_p(st.cuda_stream)), "replay")
        st.synchronize()
        assert torch.equal(dg.output()[0], sp)
        # eager runs take the mode current at run time: the same plan run eagerly, and a single op, are 3xTF32 again
        dg.out.fill_(SENT)
        torch.cuda.synchronize()
        L_.check(lib.mugd_plan_run(plan, C.c_void_p(st.cuda_stream)), "plan_run")
        st.synchronize()
        assert torch.equal(dg.output()[0], exact)
        d1 = Device(o, split)
        R1.run(d1.ops)
        assert torch.equal(d1.output()[0], exact)
    finally:
        lib.mugd_set_tc_single_pass_tf32(h, 0)
        if plan is not None:
            lib.mugd_plan_destroy(plan)
