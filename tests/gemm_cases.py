"""Cases of the wgmma GEMM tests (test_gpu_gemm_epilogue.py) and their fp64 statement, importable without a GPU: ONE float64
statement of mugd_gemm (ref_gemm), the case descriptor and its seeded operands, the epilogue x path x tile-width matrix, the
addressing-mode cases, the serial-split cases (one per class of serial op the batch-invariant plans contain, and the K-range
layouts), and the class of a serial op (serial_class) with the classes the invariant plans produce at 132 SMs (plan_serial_classes).
For the exact-fp32 FFMA kernel (gemm_simt.cu): its tile rule (ffma_tile), a per-element error bound (ffma_bound), its factor cases
(FFMA), one case per class of FFMA op the plans contain (ffma_class, plan_ffma_classes, PLAN_FFMA).
test_gemm_cases.py checks ref_gemm against torch's float64 conv / linear / layer_norm and the cases against the planner."""
import ctypes as C
import math
from dataclasses import dataclass, replace

import torch
import torch.nn.functional as F

from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth
from mug_diffusion_b200.engine import OpList, View

TOL, TOL_LN = 1e-5, 2e-5
SENT = 7777.0            # pre-fill of output buffers: every element outside the output window must keep it
STEPS, STEP = 5, 3       # rows of the step-indexed time-embedding table, value of the device step counter
LN_EPS = 1e-5


def src_rows(mode, t, lo, Lin, Lout, tap_shift=0, dilation=1):
    """source row of output rows ``lo`` at tap t, -1 where the tap reads the zero padding: l (NONE), l+t-1 (SAME), 2l+t (DOWN: stride
    2, right pad), l+(t+tap_shift)*dilation (TAPS), (l+t-1) >> 1 for 0 <= l+t-1 < Lout (UP: nearest x2, then a conv3 on the
    upsampled axis)"""
    if mode == L_.CONV_NONE:
        src = lo
    elif mode == L_.CONV_SAME:
        src = lo + t - 1
    elif mode == L_.CONV_DOWN:
        src = 2 * lo + t
    elif mode == L_.CONV_TAPS:
        src = lo + (t + tap_shift) * max(dilation, 1)
    elif mode == L_.CONV_UP:
        r = lo + t - 1
        src = torch.where((r >= 0) & (r < Lout), r // 2, torch.full_like(r, -1))
    else:
        raise ValueError(mode)
    return torch.where((src >= 0) & (src < Lin), src, torch.full_like(src, -1))


def ref_gemm(A, W, *, B, Lin, Lout, K, taps=1, mode=L_.CONV_NONE, tap_shift=0, dilation=1, A2=None, bias=None, rowvec=None,
             rowvec_b_stride=0, rowvec_step_stride=0, step=0, act=L_.ACT_NONE, gate=L_.GATE_NONE, residual=None, ln=None,
             rows=src_rows, pre=False):
    """mugd_gemm (include/mugd.h) in float64 on the operands as the kernel reads them.
    A [B*Lin, K], A2 [B*Lout, K2], W [N, taps*K + K2] (tap-major K blocks, then the K2 columns of the second source).
    Output row l of sample b reads source row rows(mode, t, l, ...) of its sample at tap t (src_rows; -1 = zero).  Then the folded
    LayerNorm  (acc - mean*colsum) * rstd  with mean / rstd from the row moments ln = (stats [M, 2] = {sum, sum of squares} over K,
    colsum [N], eps); + bias[n]; + rowvec[step*rowvec_step_stride + b*rowvec_b_stride + n] -- the pre-activation value, returned
    as it is with ``pre`` -- then ref_finish: act, gate, residual."""
    N = W.shape[0]
    a = A.double().reshape(B, Lin, K)
    w = W.double()
    lo = torch.arange(Lout)
    assert mode != L_.CONV_NONE or (taps == 1 and Lin == Lout)
    y = torch.zeros(B, Lout, N, dtype=torch.float64)
    for t in range(taps):
        src = rows(mode, t, lo, Lin, Lout, tap_shift, dilation)
        ok = src >= 0
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
        y = y + rowvec_rows(rowvec, B, Lout, N, rowvec_b_stride, rowvec_step_stride, step)
    return y if pre else ref_finish(y, act, gate, residual)


def rowvec_rows(rowvec, B, Lout, N, b_stride, step_stride, step):
    """the time-embedding row each output element adds, [B*Lout, N] in float64"""
    b = torch.arange(B * Lout) // Lout
    return rowvec.double().reshape(-1)[step * step_stride + b[:, None] * b_stride + torch.arange(N)[None]]


def ref_finish(z, act=L_.ACT_NONE, gate=L_.GATE_NONE, residual=None):
    """act; gate on the interleaved accumulator columns (2j, 2j+1) = (value_j, gate_j), the weight-row order
    packer._interleave_halves produces, -> N/2 columns; + residual"""
    y = z
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
                                # table; "step" = by step only, [STEPS, N] (the U-Net's DDIM plan); "batch" = per sample only,
                                # [B, N] without a step counter (the per-sample-t plan); "" = none
    residual: bool = True       # read from a column window
    parity: int = -1            # >= 0: output row m is buffer row 2m+parity (the parity-split Upsample); else a column window
    dense: bool = False         # the output is a whole [M, nout] buffer (ldc = nout) instead of a column window

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
        return {"both": (self.N, self.B * self.N), "batch": (self.N, 0)}.get(self.rowvec, (0, self.N))


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
            self.table = g(name + ".e", {"both": (STEPS, c.B, c.N), "batch": (c.B, c.N)}.get(c.rowvec, (STEPS, c.N)))
        self.res = g(name + ".r", (c.M, c.nout + 32)) if c.residual else None      # the residual is columns 16 .. 16+nout
        self.ln = None
        if c.ln:
            a = self.A.double()
            stats = torch.stack([a.sum(1), (a * a).sum(1)], dim=1)
            self.ln = (stats, self.W.double().sum(1).float(), LN_EPS)

    @property
    def residual(self):
        return None if self.res is None else self.res[:, 16:16 + self.c.nout]

    def kwargs(self, step=STEP):
        """ref_gemm's arguments for these operands"""
        c = self.c
        bs, ss = c.rowvec_strides
        return dict(B=c.B, Lin=c.Lin, Lout=c.Lout, K=c.K, taps=c.taps, mode=c.mode, tap_shift=c.shift, dilation=c.dilation, A2=self.A2,
                    bias=self.bias, rowvec=self.table, rowvec_b_stride=bs, rowvec_step_stride=ss, step=step, act=c.act, gate=c.gate,
                    residual=self.residual, ln=self.ln)

    def ref(self, step=STEP, **over):
        """the fp64 result; ``over`` replaces ref_gemm arguments (the mutations of test_gemm_cases.py)"""
        kw = {**self.kwargs(step), **over}
        return ref_gemm(kw.pop("A", self.A), kw.pop("W", self.W), **kw)

    def sample(self, b: int) -> "Operands":
        """the operands of sample b alone: a B = 1 case on the same rows, table entries and residual"""
        c, one = self.c, object.__new__(Operands)
        one.c = replace(c, B=1)
        one.A = self.A[b * c.Lin:(b + 1) * c.Lin]
        one.A2 = None if self.A2 is None else self.A2[b * c.Lout:(b + 1) * c.Lout]
        one.W, one.bias, one.ln = self.W, self.bias, None
        one.table = {"both": lambda t: t[:, b:b + 1].contiguous(), "batch": lambda t: t[b:b + 1]}.get(c.rowvec, lambda t: t)(self.table) \
            if c.rowvec else None
        one.res = None if self.res is None else self.res[b * c.Lout:(b + 1) * c.Lout]
        assert not c.ln
        return one


def case_gemm(ops: OpList, c: Case, split: int, *, a, w, w_hi, w_lo, out, a2=0, res=0, bias=0, table=0, step=0, stats=0, colsum=0,
              moments=0, impl=L_.GEMM_TC, a_off=32) -> int:
    """append the GEMM of case ``c`` at K split ``split`` (``impl``: the kernel it is forced to) to ``ops`` and return its index.
    The arguments are the addresses of the buffers test_gpu_gemm_epilogue.Device lays out: A = columns a_off .. a_off+K of a
    [B*Lin, K+64] buffer, A2 = columns 32 .. 32+K2 of [M, K2+64], the residual columns 16 .. 16+nout of [M, nout+32], the output
    columns 32 .. 32+nout of [M, nout+64] or, with a parity, rows 2m+parity of [2M, nout], or all of [M, nout] when dense."""
    kw = {}
    if c.bias:
        kw["bias"] = bias
    if c.rowvec:
        bs, ss = c.rowvec_strides
        kw.update(rowvec=table, rowvec_b_stride=bs, rowvec_step_stride=ss, step=step if c.rowvec != "batch" else 0)
    if c.ln:
        kw["ln"] = (stats, colsum, LN_EPS)
    if c.parity >= 0:
        dst = View(out + 4 * c.parity * c.nout, 2 * c.nout, c.M, c.nout)
    elif c.dense:
        dst = View(out, c.nout, c.M, c.nout)
    else:
        dst = View(out + 4 * 32, c.nout + 64, c.M, c.nout)
    i = ops.gemm(View(a + 4 * a_off, c.K + 64, c.B * c.Lin, c.K), w, c.N, c.K, dst, W_hi=w_hi, W_lo=w_lo, taps=c.taps, mode=c.mode,
                 Lin=c.Lin, Lout=c.Lout, act=c.act, gate=c.gate,
                 residual=View(res + 4 * 16, c.nout + 32, c.M, c.nout) if c.residual else None,
                 A2=View(a2 + 4 * 32, c.K2 + 64, c.M, c.K2) if c.K2 else None, tap_shift=c.shift, dilation=c.dilation,
                 impl=impl, split_k=split, **kw)
    if c.sink:
        ops.ops[i].u.gemm.row_moments = moments
    return i


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


# ---- the serial split (MUGD_OP_GEMM_SERIAL) --------------------------------------------------------------------------------------
def _lin(B, L, K, N, **kw):
    return Case(B, L, L, K, N, **{"rowvec": "", "residual": False, **kw})


def _conv3(B, L, K, N, **kw):
    return Case(B, L, L, K, N, taps=3, mode=L_.CONV_SAME, **{"rowvec": "", "residual": False, **kw})


def _taps(B, L, K, N, **kw):
    return Case(B, L, L, K, N, taps=2, mode=L_.CONV_TAPS, **{"rowvec": "", "residual": False, **kw})


# One case per class of serial op the invariant plans contain (plan_serial_classes; the plans' time-embedding row is the by-step
# one): name -> (case, split, tile width, whether the last K-range is short).  B3 x L48: Lrows < 128, several samples per tile;
# B2 x L200 (conv) / M = 200 (linear): Lrows >= 128.  Conv3 of K = 64: 6 k-steps (split 2 even, 4 uneven); conv3 of K = 96 + K2 = 32:
# 10 k-steps (2 even, 3 uneven); linear of K = 128, or K = 96 + K2 = 32: 4 k-steps (2 even, 3 uneven).
SERIAL = {
    "glu": (_lin(2, 100, 128, 256, gate=L_.GATE_GLU), 2, 128, False),
    "ln": (_lin(2, 100, 128, 192, ln=True), 2, 128, False),
    "ln_geglu": (_lin(2, 100, 128, 256, ln=True, gate=L_.GATE_GEGLU), 2, 128, False),
    "sink": (_lin(2, 100, 128, 192, sink=True), 2, 128, False),
    "sink_res": (_lin(2, 100, 128, 192, sink=True, residual=True), 2, 128, False),
    "ff_out": (_lin(2, 100, 96, 192, K2=32, residual=True), 2, 128, False),
    "ff_out_uneven": (_lin(2, 100, 96, 192, K2=32, residual=True), 3, 128, True),
    "conv3": (_conv3(2, 200, 64, 192), 2, 128, False),
    "conv3_short": (_conv3(3, 48, 64, 192), 2, 128, False),
    "conv3_res": (_conv3(2, 200, 64, 192, residual=True), 2, 128, False),
    "conv3_res_uneven": (_conv3(2, 200, 64, 192, residual=True), 4, 128, True),
    "conv3_res_short": (_conv3(3, 48, 64, 192, residual=True), 2, 128, False),
    "conv3_temb": (_conv3(2, 200, 64, 192, rowvec="step"), 2, 128, False),
    "conv3_temb_uneven": (_conv3(2, 200, 64, 192, rowvec="step"), 4, 128, True),
    "conv3_temb_short": (_conv3(3, 48, 64, 192, rowvec="step"), 2, 128, False),
    "conv3_temb_short_uneven": (_conv3(3, 48, 64, 192, rowvec="step"), 4, 128, True),
    "conv3_k2": (_conv3(2, 200, 96, 192, K2=32), 2, 128, False),
    "conv3_k2_uneven": (_conv3(2, 200, 96, 192, K2=32), 3, 128, True),
    "conv3_k2_short": (_conv3(3, 48, 96, 192, K2=32), 2, 128, False),
    "conv3_k2_short_uneven": (_conv3(3, 48, 96, 192, K2=32), 3, 128, True),
    "conv3_n64": (_conv3(2, 200, 64, 64), 2, 64, False),
    "conv3_n64_short": (_conv3(3, 48, 64, 64), 2, 64, False),
    "down": (Case(2, 400, 200, 64, 192, taps=3, mode=L_.CONV_DOWN, rowvec="", residual=False), 2, 128, False),
    "down_short": (Case(3, 96, 48, 64, 192, taps=3, mode=L_.CONV_DOWN, rowvec="", residual=False), 2, 128, False),
    "upsample_even": (_taps(2, 200, 96, 192, shift=-1, parity=0), 2, 128, False),
    "upsample_odd_uneven": (_taps(2, 200, 96, 192, shift=0, parity=1), 4, 128, True),
    "upsample_short": (_taps(3, 48, 96, 192, shift=-1, parity=0), 2, 128, False),
}

# K-range layouts of the serial kernel: one range (the direct path's single pass), an even split (it_rem = 0), three ranges with a
# short last one, k-steps - 1 ranges, and one k-step per range (wgmma_wait<0> at every step) -- on a Linear + second source (8 k-steps)
# and a conv3 + second source (10 k-steps).  name -> (split of a case of `ks` k-steps, whether the last K-range is short)
LAYOUT_BASES = {
    "linear": Case(2, 100, 100, 224, 192, K2=32),
    "conv3": Case(2, 200, 200, 96, 192, taps=3, mode=L_.CONV_SAME, K2=32),
}
LAYOUTS = {
    "one": (lambda ks: 1, False),
    "even": (lambda ks: 2, False),
    "three": (lambda ks: 3, True),
    "ksteps-1": (lambda ks: ks - 1, True),
    "ksteps": (lambda ks: ks, False),
}


def layout_split(base: str, layout: str) -> int:
    return LAYOUTS[layout][0](LAYOUT_BASES[base].ksteps)


# ---- classes of serial ops --------------------------------------------------------------------------------------------------------
def epilogue_of(gm) -> str:
    """the kernel instantiation's epilogue (gemm_tc.cuh tc_epi_of)"""
    if gm.ln_stats:
        return "ln_geglu" if gm.gate == L_.GATE_GEGLU else "ln"
    if gm.row_moments:
        return "sink"
    if gm.gate:
        return "geglu" if gm.gate == L_.GATE_GEGLU else "glu"
    return {L_.ACT_SILU: "silu", L_.ACT_GELU: "gelu"}.get(gm.act, "none")


def serial_class(gm, sm_count: int) -> tuple:
    """(epilogue, tile width, conv mode, second source, time-embedding row, residual, Lrows < 128, last K-range short) of a
    tensor-core GEMM at its forced split, as the planner lays it out at ``sm_count`` SMs (mugd_gemm_tc_variant / _query)"""
    lib = L_.load()
    bn, sp = C.c_int32(), C.c_int32()
    L_.check(lib.mugd_gemm_tc_variant(C.byref(gm), sm_count, C.byref(bn), None, None), "tc_variant")
    L_.check(lib.mugd_gemm_tc_query(None, C.byref(gm), sm_count, None, C.byref(sp), None, None), "tc_query")
    lrows = gm.M if gm.conv_mode == L_.CONV_NONE else gm.Lout
    total = (gm.taps * gm.K + gm.K2) // 32
    return (epilogue_of(gm), bn.value, gm.conv_mode, bool(gm.K2), bool(gm.rowvec), bool(gm.residual), lrows < 128,
            total % sp.value != 0)


PLAN_SMS = 132
PLAN_LENGTHS = (96, 512, 992, 2048)
PLAN_BATCHES = (2, 3, 4, 8, 32)


def plan_serial_classes() -> dict:
    """class -> (plan, batch) of its first serial op, over the batch-invariant plans at 132 SMs: the U-Net plain and per-sample-t
    (CFG on and off), decoder and chart encoder, at every z_length of PLAN_LENGTHS and batch of PLAN_BATCHES"""
    from mug_diffusion_b200 import packer
    from mug_diffusion_b200.config import EncoderConfig, ModelConfig
    from mug_diffusion_b200.engine import Arena, DecoderCompiler, EncoderCompiler, UNetCompiler, tc_weight_map, unit_batch_splits

    wbase = 1 << 30
    cfg = ModelConfig()
    sd = {**synth.synthetic_state_dict(96), **synth.synthetic_encoder_state_dict()}
    blob = packer.pack_model(sd, cfg.unet, cfg.decoder, encoder_cfg=cfg.encoder)
    tc = tc_weight_map(blob, wbase)

    def ext(comp, Beff, Lz):              # per-request buffers of the U-Net plan at fake addresses (test_batch_invariant._ext)
        blocks = list(comp.lay.blocks())
        ctx_kv = [View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin) for i, b in enumerate(x for x in blocks if x.kind == "attn")]
        s4 = {b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin) for i, b in enumerate(x for x in blocks if x.kind == "s4")}
        return dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21, ctx_kv=ctx_kv, s4_kt=s4)

    found = {}

    def scan(ops, B, unit, what):
        for op in unit_batch_splits(ops, B, unit, PLAN_SMS).ops:
            if op.kind == L_.OP_GEMM_SERIAL:
                found.setdefault(serial_class(op.u.gemm, PLAN_SMS), what)

    for L in PLAN_LENGTHS:
        for B in PLAN_BATCHES:
            for unit in (2, 1):                                  # CFG on / off
                for per_sample_t in (False, True):
                    comp = UNetCompiler(cfg.unet, blob, wbase, tc)
                    Beff = B * unit
                    ops = comp.compile(Arena(1 << 36), Beff, L, ext(comp, Beff, L), per_sample_t, unit * L < 8192, None)["ops"]
                    scan(ops, Beff, unit, f"unet{'_t' if per_sample_t else ''} cfg={unit == 2} L={L} B={B}")
            scan(DecoderCompiler(cfg.decoder, blob, wbase, tc).compile(Arena(1 << 36), B, L)["ops"], B, 1, f"decoder L={L} B={B}")
            scan(EncoderCompiler(EncoderConfig(), blob, wbase, tc).compile(Arena(1 << 36), B, L)["ops"], B, 1, f"encoder L={L} B={B}")
    return found


# ---- the FFMA kernel (gemm_simt.cu) -------------------------------------------------------------------------------------------
U = 2.0 ** -24                                       # unit roundoff of fp32
FFMA_C = 14.0                                         # about 4x the worst ratio measured on an H100 (DESIGN §2)


def ffma_tile(M: int, N: int, sm_count: int) -> int:
    """launch_gemm's tile rule: 128 x 128 tiles while they still give every SM two, else 64 x 64"""
    return 128 if ((M + 127) // 128) * ((N + 127) // 128) >= 2 * sm_count else 64


def _act(z, act):
    """(f(z), |f'(z)|, e) of an activation, e the error of evaluating it in fp32 beyond the product's rounding (gemm_simt.cu: SiLU
    x / (1 + exp(-x)), sigmoid, and GELU's 0.5 x (1 + erf(x / sqrt 2)), whose 1 + erf loses its relative accuracy where erf is near
    -1: an absolute u |x|)"""
    if act == L_.ACT_SILU:
        s = torch.sigmoid(z)
        f = z * s
        return f, (s * (1 + z * (1 - s))).abs(), U * f.abs()
    if act == L_.ACT_GELU:
        cdf = 0.5 * (1 + torch.erf(z / math.sqrt(2)))
        f = z * cdf
        return f, (cdf + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)).abs(), U * (f.abs() + z.abs())
    if act == "sigmoid":
        s = torch.sigmoid(z)
        return s, s * (1 - s), U * s
    return z, torch.ones_like(z), torch.zeros_like(z)


def ffma_bound(o: "Operands", step=STEP):
    """per-element error bound E (float64, [M, nout]) of a GEMM that forms each product exactly and rounds once per addition
    (fma) and once per epilogue operation, without its constant:  S = sum |a| |w| over the element's products, z the fp64
    pre-activation value,  E_z = u (S + |bias| + |rowvec| + |z|);  through the activation  E = |f'(z)| E_z + u |f(z)| + e_f;  a
    gate y = v h(g):  |h(g)| E_v + |v h'(g)| E_g + |v| e_h + u |y|;  a residual adds u (|y| + |r|).  e_f, e_h: what evaluating
    f / h costs beyond one rounding (_act; u |z| for GELU's 1 + erf form).  S, not sqrt(n) S: the latter admits A rounded to TF32
    at the simt plans' longest K."""
    c = o.c
    kw = o.kwargs(step)
    act, gate, res = kw.pop("act"), kw.pop("gate"), kw.pop("residual")
    assert kw["ln"] is None
    z = ref_gemm(o.A, o.W, **kw, pre=True)
    kw.update(A2=None if o.A2 is None else o.A2.abs(), bias=None, rowvec=None)
    S = ref_gemm(o.A.abs(), o.W.abs(), **kw, pre=True)
    if o.bias is not None:
        S = S + o.bias.double().abs()
    if o.table is not None:
        S = S + rowvec_rows(o.table, c.B, c.Lout, c.N, *c.rowvec_strides, step).abs()
    f, fd, ef = _act(z, act)
    E = fd * (U * (S + z.abs())) + U * f.abs() + ef
    y = f
    if gate != L_.GATE_NONE:
        v, g_, Ev, Eg = f[:, 0::2], f[:, 1::2], E[:, 0::2], E[:, 1::2]
        h, hd, eh = _act(g_, L_.ACT_GELU if gate == L_.GATE_GEGLU else "sigmoid")
        y = v * h
        E = h.abs() * Ev + (v * hd).abs() * Eg + v.abs() * eh + U * y.abs()
    if res is not None:
        E = E + U * (y.abs() + res.double().abs())
    return E


# ---- classes of FFMA ops ------------------------------------------------------------------------------------------------------
def rowvec_kind(gm) -> str:
    """which time-embedding row the GEMM adds: none, by device step only, per sample only, or both"""
    if not gm.rowvec:
        return "none"
    by_step, by_sample = bool(gm.step) and gm.rowvec_step_stride != 0, gm.rowvec_b_stride != 0
    return {(True, True): "both", (True, False): "step", (False, True): "batch", (False, False): "const"}[(by_step, by_sample)]


def ffma_class(gm, sm_count: int = 132) -> tuple:
    """(conv mode, taps, dilation > 1, tap shift, second source, act, gate, bias, time-embedding row, residual, output strided or
    parity, K % 32 != 0, N < 64, tile) of a GEMM on the FFMA kernel, the tile as launch_gemm picks it at ``sm_count`` SMs"""
    nout = gm.N // 2 if gm.gate else gm.N
    return (gm.conv_mode, gm.taps, gm.tap_dilation > 1, gm.tap_shift, gm.K2 > 0, gm.act, gm.gate, bool(gm.bias), rowvec_kind(gm),
            bool(gm.residual), gm.ldc != nout, (gm.K % 32 or gm.K2 % 32) != 0, gm.N < 64, ffma_tile(gm.M, gm.N, sm_count))


FFMA_T = (6144, 32768)                               # audio encoder frames: the 30 s golden and a 3-minute song


def plan_ffma_classes() -> dict:
    """class -> where it first occurs, over the GEMMs of every plan that run on the FFMA kernel at 132 SMs: the U-Net (plain,
    per-sample-t, ragged, guided-scale; CFG on and off), its timestep and context-K/V ops, decoder and chart encoder at every z_length
    of PLAN_LENGTHS and batch of PLAN_BATCHES, and the audio encoder at FFMA_T frames.  Walked twice: with the default TF32 weight
    map (the GEMMs gemm_runs_tc rejects) and with an empty one (every GEMM of the `simt` engine)."""
    import types

    from mug_diffusion_b200 import packer, wave
    from mug_diffusion_b200.config import EncoderConfig, ModelConfig
    from mug_diffusion_b200.engine import (Arena, DecoderCompiler, EncoderCompiler, UNetCompiler, gemm_runs_tc, guided_scales_ops,
                                           tc_weight_map)
    from mug_diffusion_b200.runtime import Session

    wbase = 1 << 30
    cfg = ModelConfig()
    wcfg = wave.WaveConfig()
    sd = {**synth.synthetic_state_dict(96), **synth.synthetic_encoder_state_dict(), **wave.synthetic_wave_state_dict(wcfg)}
    blob = packer.pack_model(sd, cfg.unet, cfg.decoder, encoder_cfg=cfg.encoder, wave_cfg=wcfg)       # as MugEngine packs it
    found = {}

    def ext(comp, Beff, Lz):
        blocks = list(comp.lay.blocks())
        ctx_kv = [View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin) for i, b in enumerate(x for x in blocks if x.kind == "attn")]
        s4 = {b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin) for i, b in enumerate(x for x in blocks if x.kind == "s4")}
        return dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21, ctx_kv=ctx_kv, s4_kt=s4)

    for simt in (False, True):
        tc = {} if simt else tc_weight_map(blob, wbase)

        def scan(ops, what):
            for op in ops.ops:
                if op.kind == L_.OP_GEMM and (simt or not gemm_runs_tc(op.u.gemm, PLAN_SMS)):
                    found.setdefault(ffma_class(op.u.gemm, PLAN_SMS), f"{'simt' if simt else 'auto'} {what}")

        comp = UNetCompiler(cfg.unet, blob, wbase, tc)
        # the per-request ops of a U-Net session (runtime.Session.timestep_ops / context_ops) on stand-in buffers
        eng = types.SimpleNamespace(cfg=cfg, tc_map=tc, batch_ops=lambda ops, B, unit: ops)
        for L in PLAN_LENGTHS:
            for B in PLAN_BATCHES:
                for unit in (2, 1):                                  # CFG on / off
                    Beff = B * unit
                    for per_sample_t in (False, True):
                        res = comp.compile(Arena(1 << 36), Beff, L, ext(comp, Beff, L), per_sample_t, False if simt else None)
                        scan(res["ops"], f"unet{'_t' if per_sample_t else ''} cfg={unit == 2} L={L} B={B}")
                    valid = [(1 << 43) + 256 * lvl for lvl in range(cfg.unet.levels)]
                    scan(comp.compile(Arena(1 << 36), Beff, L, ext(comp, Beff, L), False, False if simt else None, valid)["ops"],
                         f"unet ragged cfg={unit == 2} L={L} B={B}")
                    if unit == 2:
                        res = comp.compile(Arena(1 << 36), Beff, L, ext(comp, Beff, L), False, False if simt else None)
                        scan(guided_scales_ops(res["ops"], res["xin"], res["eps"], B, L, 1 << 44, 1 << 45), f"unet guided L={L} B={B}")
                    if L == PLAN_LENGTHS[0]:
                        emb_total = blob.meta["emb_total"]
                        for R, per_sample_t in ((Beff, True), (10, False), (1000, False)):
                            s = types.SimpleNamespace(engine=eng, comp=comp, Beff=Beff, unit=unit, per_sample_t=per_sample_t,
                                                      temb=torch.empty(1, cfg.unet.model_channels), emb_h1=torch.empty(1, cfg.unet.time_embed_dim),
                                                      emb_h2=torch.empty(1, cfg.unet.time_embed_dim), emb_table=torch.empty(1, emb_total),
                                                      ctx=torch.empty(1, cfg.unet.context_dim),
                                                      ctx_kv=[torch.empty(1, 2 * b.cin) for b in comp.lay.blocks() if b.kind == "attn"])
                            scan(Session.timestep_ops(s, R), f"timestep R={R}")
                            scan(Session.context_ops(s, [(1 << 44, Beff)], 21), f"context B={Beff}")
            for B in PLAN_BATCHES:
                scan(DecoderCompiler(cfg.decoder, blob, wbase, tc).compile(Arena(1 << 36), B, L)["ops"], f"decoder L={L} B={B}")
                scan(EncoderCompiler(EncoderConfig(), blob, wbase, tc).compile(Arena(1 << 36), B, L)["ops"], f"encoder L={L} B={B}")
        for T in FFMA_T:
            for B in (1, 2, 4):
                scan(wave.WaveCompiler(wcfg, blob, wbase, tc).compile(Arena(1 << 36), B, T)["ops"], f"audio T={T} B={B}")
    return found


# ---- FFMA cases ---------------------------------------------------------------------------------------------------------------
FFMA_SMS = (132, 114)                                # H100 SXM and H100 PCIe: every case takes the tile it claims on both


def fill(L: int, N: int) -> int:
    """the fewest samples of L rows whose M x N output takes the 128 x 128 tiles at both SM counts, with 10 % margin"""
    need = math.ceil(1.1 * 2 * max(FFMA_SMS) / ((N + 127) // 128))
    return -(-need * 128 // L)


def _sm(B, L, K, N, **kw):                           # a conv3 of the factor cases' base shape
    return Case(B, L, L, K, N, taps=3, mode=L_.CONV_SAME, **kw)


GEGLU, GLU, SILU, GELU = dict(gate=L_.GATE_GEGLU), dict(gate=L_.GATE_GLU), dict(act=L_.ACT_SILU), dict(act=L_.ACT_GELU)
TAPS = L_.CONV_TAPS

# Factors of the FFMA kernel around one base (conv3, K = 48: three k-steps per tap, none a multiple of 32; N = 68: a partial
# column tile; 3 x 65 rows: a partial row tile, samples that straddle 16-row thread groups; bias, the both-kinds time-embedding
# row, residual; A, residual and output as column windows): name -> (case, tile).  Every 64-tile case is one at both SM counts.
FFMA = {
    "base": (_sm(3, 65, 48, 68), 64),
    # addressing
    "none": (Case(3, 65, 65, 48, 68), 64),
    "down": (Case(3, 130, 65, 48, 68, taps=3, mode=L_.CONV_DOWN), 64),
    "down_odd": (Case(3, 130, 65, 48, 68, taps=3, mode=L_.CONV_DOWN, rowvec="step"), 64),
    "up": (Case(3, 33, 66, 48, 68, taps=3, mode=L_.CONV_UP), 64),
    "taps_m1_d1": (Case(3, 65, 65, 48, 68, taps=3, mode=TAPS, shift=-1), 64),
    "taps_0_d1": (Case(3, 65, 65, 48, 68, taps=2, mode=TAPS, shift=0), 64),
    "taps_m1_d1_2": (Case(3, 65, 65, 48, 68, taps=2, mode=TAPS, shift=-1), 64),
    "taps_m1_d2": (Case(3, 65, 65, 48, 68, taps=3, mode=TAPS, shift=-1, dilation=2), 64),
    "taps_m1_d3": (Case(3, 65, 65, 48, 68, taps=3, mode=TAPS, shift=-1, dilation=3), 64),
    "taps_0_d2": (Case(3, 65, 65, 48, 68, taps=3, mode=TAPS, shift=0, dilation=2), 64),
    "taps_0_d3": (Case(3, 65, 65, 48, 68, taps=3, mode=TAPS, shift=0, dilation=3), 64),
    # the second source
    "none_k2": (Case(3, 65, 65, 48, 68, K2=16), 64),
    "same_k2": (_sm(3, 65, 48, 68, K2=48), 64),
    "same_k2_k16": (_sm(3, 65, 16, 68, K2=16), 64),
    "taps_k2": (Case(3, 65, 65, 48, 68, taps=3, mode=TAPS, shift=-1, dilation=2, K2=16), 64),
    "taps_k2_shift0": (Case(3, 65, 65, 16, 68, taps=2, mode=TAPS, shift=0, K2=48), 64),
    # K: one k-step per tap, five, a single k-step in all
    "k16": (_sm(3, 65, 16, 68), 64),
    "k80": (_sm(3, 65, 80, 68), 64),
    "k16_none": (Case(3, 65, 65, 16, 68), 64),
    # N: inside one float4 column group, partial 16-column thread groups, N < 64, a second column tile
    "n4": (_sm(3, 65, 48, 4), 64),
    "n12": (_sm(3, 65, 48, 12), 64),
    "n16": (_sm(3, 65, 48, 16), 64),
    "n20": (_sm(3, 65, 48, 20), 64),
    "n132": (_sm(3, 65, 48, 132), 64),
    "n4_glu": (Case(3, 65, 65, 48, 8, **GLU), 64),
    # rows per sample: many samples in a tile, each row its own halo; one sample over two tiles
    "l1": (_sm(40, 1, 48, 68), 64),
    "l2": (_sm(30, 2, 48, 68), 64),
    "l3": (_sm(25, 3, 48, 68), 64),
    "l63": (_sm(3, 63, 48, 68), 64),
    "l129": (_sm(2, 129, 48, 68), 64),
    "l1_none": (Case(40, 1, 1, 48, 68), 64),
    "l1_down": (Case(40, 2, 1, 48, 68, taps=3, mode=L_.CONV_DOWN), 64),
    "l1_up": (Case(40, 1, 2, 48, 68, taps=3, mode=L_.CONV_UP), 64),
    "l1_taps_d3": (Case(40, 1, 1, 48, 68, taps=3, mode=TAPS, shift=-1, dilation=3), 64),
    "l2_taps_d2": (Case(30, 2, 2, 48, 68, taps=3, mode=TAPS, shift=-1, dilation=2), 64),
    "l3_up": (Case(25, 3, 6, 48, 68, taps=3, mode=L_.CONV_UP), 64),
    "l63_k2": (_sm(3, 63, 48, 68, K2=16), 64),
    # every epilogue
    "no_bias": (_sm(3, 65, 48, 68, bias=False), 64),
    "rowvec_step": (_sm(3, 65, 48, 68, rowvec="step"), 64),
    "rowvec_batch": (_sm(3, 65, 48, 68, rowvec="batch"), 64),
    "rowvec_none": (_sm(3, 65, 48, 68, rowvec=""), 64),
    "plain": (_sm(3, 65, 48, 68, bias=False, rowvec="", residual=False), 64),
    "silu": (_sm(3, 65, 48, 68, **SILU), 64),
    "gelu": (_sm(3, 65, 48, 68, **GELU), 64),
    "silu_nores": (_sm(3, 65, 48, 68, residual=False, **SILU), 64),
    "gelu_nores": (_sm(3, 65, 48, 68, residual=False, **GELU), 64),
    "geglu": (Case(3, 65, 65, 48, 136, **GEGLU), 64),
    "glu": (Case(3, 65, 65, 48, 136, **GLU), 64),
    "geglu_nores": (Case(3, 65, 65, 48, 136, residual=False, **GEGLU), 64),
    "glu_nores": (Case(3, 65, 65, 48, 136, residual=False, **GLU), 64),
    "glu_same_k2": (_sm(3, 65, 48, 136, K2=16, **GLU), 64),
    "geglu_rowvec_batch": (Case(3, 65, 65, 48, 136, rowvec="batch", **GEGLU), 64),
    "dense": (_sm(3, 65, 48, 68, dense=True), 64),
    "parity": (Case(3, 65, 65, 48, 68, taps=2, mode=TAPS, shift=-1, parity=1), 64),
    # the 128 x 128 tiles: partial row and column tiles, every addressing mode, second source, gate
    "big_none": (Case(fill(129, 132), 129, 129, 48, 132), 128),
    "big_same": (_sm(fill(129, 132), 129, 48, 132), 128),
    "big_down": (Case(fill(65, 132), 130, 65, 48, 132, taps=3, mode=L_.CONV_DOWN), 128),
    "big_up": (Case(fill(130, 132), 65, 130, 16, 132, taps=3, mode=L_.CONV_UP), 128),
    "big_taps_d2": (Case(fill(129, 132), 129, 129, 16, 132, taps=3, mode=TAPS, shift=-1, dilation=2), 128),
    "big_k2": (_sm(fill(129, 132), 129, 16, 132, K2=16), 128),
    "big_n20": (_sm(fill(129, 20), 129, 16, 20, rowvec="step"), 128),
    "big_glu": (Case(fill(65, 264), 65, 65, 48, 264, **GLU), 128),
    "big_l1": (_sm(fill(1, 132), 1, 16, 132), 128),
}


def _plan(mode, K, N, *, taps=1, tiles=(64, 128), **kw):
    """a plan-class case at each tile: A 3 x 65 rows on 64-tiles, fill() on 128-tiles; no bias, time-embedding row or residual, a
    dense output unless given"""
    L = 65
    base = dict(bias=False, rowvec="", residual=False, dense="parity" not in kw, taps=taps, mode=mode)
    base.update(kw)
    out = {}
    for t in tiles:
        B = 3 if t == 64 else fill(L, N)
        Lin = 2 * L if mode == L_.CONV_DOWN else L
        out[t] = (Case(B, Lin, L, K, N, **base), t)
    return out


# One case per class of FFMA op in the plans (plan_ffma_classes; test_gemm_cases.py fails naming any class not covered here):
# name -> {tile: (case, tile)}.
_NONE, _SAME, _DOWN = L_.CONV_NONE, L_.CONV_SAME, L_.CONV_DOWN
PLAN_FFMA_SHAPES = {
    "lin": _plan(_NONE, 32, 68),
    "lin_bias": _plan(_NONE, 32, 68, bias=True),
    "lin_bias_res": _plan(_NONE, 32, 68, bias=True, residual=True),
    "lin_geglu": _plan(_NONE, 32, 136, bias=True, **GEGLU),
    "lin_glu": _plan(_NONE, 32, 136, bias=True, **GLU),
    "lin_silu": _plan(_NONE, 32, 68, bias=True, tiles=(64,), **SILU),
    "lin_k2_res": _plan(_NONE, 32, 68, bias=True, residual=True, K2=32),
    "conv3": _plan(_SAME, 32, 68, taps=3, bias=True),
    "conv3_temb_batch": _plan(_SAME, 32, 68, taps=3, bias=True, rowvec="batch"),
    "conv3_temb_step": _plan(_SAME, 32, 68, taps=3, bias=True, rowvec="step"),
    "conv3_n16": _plan(_SAME, 32, 16, taps=3, bias=True),
    "conv3_k16": _plan(_SAME, 16, 68, taps=3, bias=True),
    "conv3_k16_window": _plan(_SAME, 16, 68, taps=3, bias=True, dense=False),
    "conv3_res": _plan(_SAME, 32, 68, taps=3, bias=True, residual=True),
    "conv3_res_window": _plan(_SAME, 32, 68, taps=3, bias=True, residual=True, dense=False),
    "conv3_k2": _plan(_SAME, 32, 68, taps=3, bias=True, K2=32),
    "down": _plan(_DOWN, 32, 68, taps=3, bias=True),
    "down_window": _plan(_DOWN, 32, 68, taps=3, bias=True, dense=False),
    "upsample_even": _plan(TAPS, 32, 68, taps=2, shift=-1, bias=True, parity=0),
    "upsample_odd": _plan(TAPS, 32, 68, taps=2, shift=0, bias=True, parity=1),
    "taps3": _plan(TAPS, 32, 68, taps=3, shift=-1, bias=True),
    "taps3_dilated": _plan(TAPS, 32, 68, taps=3, shift=-1, dilation=2, bias=True),
    "taps3_dilated_res": _plan(TAPS, 32, 68, taps=3, shift=-1, dilation=4, bias=True, residual=True),
}
PLAN_FFMA = {f"{name}_{t}": v for name, per in PLAN_FFMA_SHAPES.items() for t, v in per.items()}


def ffma_gpu_cases() -> dict:
    """every case the FFMA tests of test_gpu_gemm_epilogue.py run with the bound: name -> (case, tile)"""
    return {**{f"ffma_{k}": v for k, v in FFMA.items()}, **{f"plan_{k}": v for k, v in PLAN_FFMA.items()}}
