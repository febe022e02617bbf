"""Cases of the wgmma GEMM tests (test_gpu_gemm_epilogue.py) and their fp64 statement, importable without a GPU: ONE float64
statement of mugd_gemm (ref_gemm), the case descriptor and its seeded operands, the epilogue x path x tile-width matrix, the
addressing-mode cases, the serial-split cases (one per class of serial op the batch-invariant plans contain, and the K-range
layouts), and the class of a serial op (serial_class) with the classes the invariant plans produce at 132 SMs (plan_serial_classes).
test_gemm_cases.py checks ref_gemm against torch's float64 conv / linear / layer_norm and the cases against the planner."""
import ctypes as C
import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from mug_diffusion_b200 import lib as L_
from mug_diffusion_b200 import synth
from mug_diffusion_b200.engine import OpList, View

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


def case_gemm(ops: OpList, c: Case, split: int, *, a, w, w_hi, w_lo, out, a2=0, res=0, bias=0, table=0, step=0, stats=0, colsum=0,
              moments=0) -> int:
    """append the GEMM of case ``c`` at K split ``split`` to ``ops`` and return its index.  The arguments are the addresses of the
    buffers test_gpu_gemm_epilogue.Device lays out: A = columns 32 .. 32+K of a [B*Lin, K+64] buffer, A2 = columns 32 .. 32+K2 of
    [M, K2+64], the residual columns 16 .. 16+nout of [M, nout+32], the output columns 32 .. 32+nout of [M, nout+64] or, with a
    parity, rows 2m+parity of [2M, nout]."""
    kw = {}
    if c.bias:
        kw["bias"] = bias
    if c.rowvec:
        bs, ss = c.rowvec_strides
        kw.update(rowvec=table, rowvec_b_stride=bs, rowvec_step_stride=ss, step=step)
    if c.ln:
        kw["ln"] = (stats, colsum, LN_EPS)
    if c.parity >= 0:
        dst = View(out + 4 * c.parity * c.nout, 2 * c.nout, c.M, c.nout)
    else:
        dst = View(out + 4 * 32, c.nout + 64, c.M, c.nout)
    i = ops.gemm(View(a + 4 * 32, c.K + 64, c.B * c.Lin, c.K), w, c.N, c.K, dst, W_hi=w_hi, W_lo=w_lo, taps=c.taps, mode=c.mode,
                 Lin=c.Lin, Lout=c.Lout, act=c.act, gate=c.gate,
                 residual=View(res + 4 * 16, c.nout + 32, c.M, c.nout) if c.residual else None,
                 A2=View(a2 + 4 * 32, c.K2 + 64, c.M, c.K2) if c.K2 else None, tap_shift=c.shift, dilation=c.dilation,
                 impl=L_.GEMM_TC, split_k=split, **kw)
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
