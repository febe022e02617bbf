"""GroupNorm(+SiLU) and LayerNorm cases shared by tests/test_gpu_norm.py (importable without a GPU):

* ``ref_groupnorm`` / ``ref_layernorm`` -- the two ops (csrc/norm.cu) in float64, with the per-element magnitude ``A`` the error
  bound is measured against (``bound_ratio``);
* ``emulate_groupnorm`` / ``emulate_layernorm`` -- the kernels' arithmetic on the host, in fp32 where the kernels use fp32, to show
  that the bound holds for that arithmetic and fails for a cheaper one (fp32 moments);
* ``plan_signatures`` -- every OP_GROUPNORM / OP_LAYERNORM of real U-Net, decoder, encoder and wave-encoder plans, compiled on the
  host with fake addresses and reduced to a ``Case`` (shape, leading dimension and column offset of x and y in their buffers);
* ``PLAN_CASES``     -- those signatures written out, so the GPU tests need no plan compile (a CPU test keeps the two equal);
* ``kernel_for``     -- which kernel launch_groupnorm / launch_layernorm runs for a case;
* ``EDGE_CASES``     -- hand-picked shapes, windows and data regimes at the edges of the six GroupNorm kernels and the LayerNorm.
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
from typing import Dict, List

import torch

from attention_cases import _Buffers, _fake_ext, _recording_arena

GN_EPS = 1e-6          # Normalize (models.py): GroupNorm(32, C, eps=1e-6)
LN_EPS = 1e-5          # nn.LayerNorm default
U = 2.0 ** -24         # unit roundoff of fp32
SILU_SLOPE = 1.1       # bounds |silu'(h)| = |sigmoid(h) (1 + h (1 - sigmoid(h)))| <= 1.0998


@dataclass(frozen=True)
class Case:
    """GroupNorm over B samples of L rows and C channels in G groups; G = 0 is a LayerNorm over L rows (B = 1, silu = 0).
    x is a column window at column cx of a buffer with leading dimension ldx, y likewise at cy of ldy."""
    B: int
    L: int
    C: int
    G: int
    silu: int
    ldx: int
    cx: int
    ldy: int
    cy: int
    regime: str = "randn"       # input data, see make_inputs

    @property
    def is_ln(self) -> bool:
        return self.G == 0

    @property
    def eps(self) -> float:
        return LN_EPS if self.is_ln else GN_EPS

    @property
    def id(self) -> str:
        s = f"ln-r{self.L}-C{self.C}" if self.is_ln else f"gn-B{self.B}-L{self.L}-C{self.C}-G{self.G}" + ("-silu" if self.silu else "")
        if (self.ldx, self.cx, self.ldy, self.cy) != (self.C, 0, self.C, 0):
            s += f"-x{self.cx}.{self.ldx}-y{self.cy}.{self.ldy}"
        return s + ("" if self.regime == "randn" else "-" + self.regime)


def gn(B, L, C, G, silu, ldx=0, cx=0, ldy=0, cy=0, regime="randn") -> Case:
    return Case(B, L, C, G, int(silu), ldx or C, cx, ldy or C, cy, regime)


def ln(rows, C, ldx=0, cx=0, ldy=0, cy=0, regime="randn") -> Case:
    return Case(1, rows, C, 0, 0, ldx or C, cx, ldy or C, cy, regime)


GN_THREADS, GN_MAXV = 256, 32          # csrc/norm.cu


def kernel_for(c: Case) -> str:
    """the kernel csrc/norm.cu runs: "ln" (layernorm_kernel), "reg2" .. "reg32" (groupnorm_silu_reg_kernel<NV>: the slab of a group
    in registers, NV float4 per thread) or "two" (groupnorm_silu_kernel, two passes) when a slab exceeds 32 float4 per thread"""
    if c.is_ln:
        return "ln"
    per_thread = (c.L * (c.C // c.G // 4) + GN_THREADS - 1) // GN_THREADS
    for nv in (2, 4, 8, 16, GN_MAXV):
        if per_thread <= nv:
            return f"reg{nv}"
    return "two"


GN_KERNELS = ("reg2", "reg4", "reg8", "reg16", "reg32", "two")


# ---- fp64 reference and the error bound ----------------------------------------------------------------------------------------
def _grouped(x: torch.Tensor, c: Case) -> torch.Tensor:
    """x [B*L, C] viewed as [samples, rows, groups, channels per group]: the moments are taken over dims 1 and 3"""
    return x.view(c.L, 1, 1, c.C) if c.is_ln else x.view(c.B, c.L, c.G, c.C // c.G)


def _ref(x, gamma, beta, c: Case, eps: float):
    xd = _grouped(x.double(), c)
    m = xd.mean((1, 3), keepdim=True)
    var = (xd - m).square().mean((1, 3), keepdim=True)                 # biased, as torch's GroupNorm / LayerNorm
    r = (var + eps).rsqrt()                                            # eps added to the variance
    g = _grouped(gamma.double().expand(x.shape), c)
    b = _grouped(beta.double().expand(x.shape), c)
    h = (xd - m) * r * g + b
    A = (xd.abs() + m.abs()) * r * g.abs() + b.abs()
    if c.silu:
        h = h * torch.sigmoid(h)
        A = A * SILU_SLOPE
    return h.reshape(x.shape), A.reshape(x.shape)


def ref_groupnorm(x, gamma, beta, G: int, eps: float = GN_EPS, silu: bool = False):
    """x [B, L, C] -> (y, A) in float64: y = silu?((x - m) r gamma + beta), m and r = 1 / sqrt(var + eps) from the biased moments
    of each (sample, group) slab; A = ((|x| + |m|) r |gamma| + |beta|) (x 1.1 with SiLU) is the size of the terms an fp32
    evaluation rounds, so an error of y is measured against A + |y| element by element"""
    B, L, C = x.shape
    y, A = _ref(x.reshape(B * L, C), gamma, beta, gn(B, L, C, G, silu), eps)
    return y.view(B, L, C), A.view(B, L, C)


def ref_layernorm(x, gamma, beta, eps: float = LN_EPS):
    """x [rows, C] -> (y, A) in float64, as ref_groupnorm with one group per row (nn.LayerNorm)"""
    return _ref(x, gamma, beta, ln(*x.shape), eps)


def reference(x, gamma, beta, c: Case):
    """(y, A) of case c for x [B*L, C] (any device; float64)"""
    return _ref(x, gamma, beta, c, c.eps)


def bound_ratio(y, ref, A) -> float:
    """max over elements of |y - ref| / (2^-24 (A + |ref|)); the bound holds when this is <= K.  NaN / inf in y give inf."""
    if not bool(torch.isfinite(y).all()):
        return math.inf
    return float(((y.double() - ref).abs() / (U * (A + ref.abs()))).max())


# ---- host emulation of the kernels' arithmetic ---------------------------------------------------------------------------------
def emulate_groupnorm(x, gamma, beta, c: Case, moments: str = "fp64"):
    """groupnorm_silu_*_kernel on the host: moments sum(x), sum(x^2) in fp64 (moments="fp32": in fp32), var = E[x^2] - m^2, the
    float mean, v = float(var) + eps, r = rsqrtf(v) with one Newton step, then (x - mean) * r * gamma + beta and SiLU in fp32"""
    xg = _grouped(x.float(), c)
    n = xg.shape[1] * xg.shape[3]
    acc = xg.double() if moments == "fp64" else xg
    assert moments in ("fp64", "fp32"), moments
    m = acc.sum((1, 3), keepdim=True) / n
    var = acc.square().sum((1, 3), keepdim=True) / n - m * m
    v = var.float().clamp_min(0) + torch.tensor(c.eps, dtype=torch.float32)
    r = v.rsqrt()
    r = r * (1.5 - 0.5 * v * r * r)
    g, b = _grouped(gamma.float().expand(x.shape), c), _grouped(beta.float().expand(x.shape), c)
    h = (xg - m.float()) * r * g + b
    if c.silu:
        h = h / (1 + torch.exp(-h))
    return h.reshape(x.shape)


def emulate_layernorm(x, gamma, beta, variance: str = "centered"):
    """layernorm_kernel on the host, all fp32 in the kernel's order: lane l of a warp sums float4 l, l + 32, ... as (x + y) + (z + w),
    a butterfly of shuffles adds the lanes, mean = sum / C; the variance the same over centered values (variance="raw": E[x^2] -
    mean^2 from a sum of squares), rstd = rsqrtf(var + eps), y = (x - mean) * rstd * gamma + beta"""
    rows, C = x.shape
    nq = C // 4
    lanes = torch.zeros(rows, 8 * 32, 4)
    lanes[:, :nq] = x.float().view(rows, nq, 4)
    lanes = lanes.view(rows, 8, 32, 4)
    valid = (torch.arange(8 * 32) < nq).view(1, 8, 32, 1)

    def warp_sum(v):                                       # v [rows, 8, 32, 4] -> [rows, 1]
        s = torch.zeros(rows, 32)
        for i in range(8):
            q = v[:, i]
            s = s + ((q[..., 0] + q[..., 1]) + (q[..., 2] + q[..., 3]))
        idx = torch.arange(32)
        for o in (16, 8, 4, 2, 1):
            s = s + s[:, idx ^ o]
        return s[:, :1]

    mean = warp_sum(lanes) / C
    if variance == "centered":
        d = torch.where(valid, lanes - mean[:, :, None, None], torch.zeros(()))
        var = warp_sum(d * d) / C
    else:
        assert variance == "raw", variance
        var = warp_sum(lanes * lanes) / C - mean * mean
    rstd = (var + torch.tensor(LN_EPS, dtype=torch.float32)).rsqrt()
    return (x.float() - mean) * rstd * gamma.float() + beta.float()


# ---- inputs ----------------------------------------------------------------------------------------------------------------------
REGIMES = ("randn", "offset", "flat", "tiny", "wide")
FLAT_VALUE = 0.1                       # stored as 0.1f: not a power of two, so a rounded mean would show


def flat_groups(c: Case) -> torch.Tensor:
    """bool [samples, 1, groups, 1] (see _grouped): the exactly constant groups of the "flat" regime -- group b % G of sample b, or
    every seventh row of a LayerNorm"""
    if c.is_ln:
        return (torch.arange(c.L) % 7 == 0).view(c.L, 1, 1, 1)
    return (torch.arange(c.G)[None, :] == (torch.arange(c.B) % c.G)[:, None]).view(c.B, 1, c.G, 1)


def make_inputs(c: Case, device="cpu"):
    """x [B*L, C], gamma [C], beta [C] (float32 on device), seeded by the case.  Regimes (per group, or per row of a LayerNorm):
    randn  -- unit normal x;
    offset -- x = mean + s z with |mean| / s drawn log-uniformly from [100, 1000], s from [1/4, 4], the sign of mean random: the
              moments E[x^2] - m^2 cancel to 4 .. 6 digits, which fp32 sums cannot resolve;
    flat   -- unit normal, but the groups of flat_groups exactly 0.1f: zero variance, eps alone keeps r finite;
    tiny   -- x = 1e-4 u + 1e-5 z: spread far below sqrt(eps), so eps decides the output;
    wide   -- unit normal with every 997th element +-1e4, and |gamma| up to 4: normalised outliers reach +-100 ahead of SiLU."""
    g = torch.Generator(device=device).manual_seed(zlib.crc32(c.id.encode()))
    shape = (c.B * c.L, c.C)
    x = torch.randn(shape, generator=g, device=device)
    gamma = 1 + 0.5 * torch.randn(c.C, generator=g, device=device)
    beta = 0.5 * torch.randn(c.C, generator=g, device=device)
    xg = _grouped(x, c)
    per_group = (xg.shape[0], 1, xg.shape[2], 1)
    if c.regime == "offset":
        ratio = 10 ** (2 + torch.rand(per_group, generator=g, device=device))
        spread = 4 ** (2 * torch.rand(per_group, generator=g, device=device) - 1)
        sign = torch.where(torch.rand(per_group, generator=g, device=device) < 0.5, -1.0, 1.0)
        xg.mul_(spread).add_(sign * ratio * spread)
    elif c.regime == "flat":
        xg.masked_fill_(flat_groups(c).to(device), FLAT_VALUE)
    elif c.regime == "tiny":
        xg.mul_(1e-5).add_(1e-4 * torch.randn(per_group, generator=g, device=device))
    elif c.regime == "wide":
        n = x.view(-1)[::997].numel()
        x.view(-1)[::997] = 1e4 * torch.where(torch.arange(n, device=device) % 2 == 0, 1.0, -1.0)
        sign = torch.where(torch.rand(c.C, generator=g, device=device) < 0.5, -1.0, 1.0)
        gamma = sign * (1 + 3 * torch.rand(c.C, generator=g, device=device))
    else:
        assert c.regime == "randn", c.regime
    return x, gamma, beta


# ---- signatures of real plans ----------------------------------------------------------------------------------------------------
UNET_PLANS = [(2, 96), (8, 512), (64, 512), (16, 992), (2, 2048), (1, 8192)]      # (Beff, Lz)
DECODER_PLANS = [(1, 96), (4, 512), (1, 8192)]                                     # (B, Lz); the encoder runs at the same lengths
WAVE_PLANS = [(2, 6144), (2, 32768), (1, 524288)]                                  # (B, T)


def _signature(o, bufs: _Buffers) -> Case:
    from mug_diffusion_b200 import lib as L_
    if o.kind == L_.OP_GROUPNORM:
        d = o.u.gn
        (_, cx), (_, cy) = bufs.locate(d.x, d.ldx), bufs.locate(d.y, d.ldy)
        assert abs(d.eps - GN_EPS) < 1e-12
        return Case(d.B, d.L, d.C, d.G, d.silu, d.ldx, cx, d.ldy, cy)
    d = o.u.ln
    (_, cx), (_, cy) = bufs.locate(d.x, d.ldx), bufs.locate(d.y, d.ldy)
    assert abs(d.eps - LN_EPS) < 1e-11
    return ln(d.rows, d.C, d.ldx, cx, d.ldy, cy)


def plan_norm_ops():
    """{(plan kind, B, L): [Case of each OP_GROUPNORM / OP_LAYERNORM, in plan order]} from plans compiled on the host, kinds "unet"
    (Beff, Lz; default LayerNorm fold), "decoder" and "encoder" (B, Lz), "wave" (B, T)"""
    from mug_diffusion_b200 import lib as L_
    from mug_diffusion_b200 import packer, synth, wave
    from mug_diffusion_b200.config import EncoderConfig, ModelConfig
    from mug_diffusion_b200.engine import DecoderCompiler, EncoderCompiler, UNetCompiler

    def norms(res, bufs):
        return [_signature(o, bufs) for o in res["ops"].ops if o.kind in (L_.OP_GROUPNORM, L_.OP_LAYERNORM)]

    out = {}
    cfg = ModelConfig()
    blob = packer.pack_model({**synth.synthetic_state_dict(96), **synth.synthetic_encoder_state_dict()}, cfg.unet, cfg.decoder)
    comp = UNetCompiler(cfg.unet, blob, 1 << 30)
    for Beff, Lz in UNET_PLANS:
        bufs = _Buffers()
        out[("unet", Beff, Lz)] = norms(comp.compile(_recording_arena(bufs, 1 << 32), Beff, Lz, _fake_ext(comp, Beff, Lz, bufs), False), bufs)
    for kind, comp in (("decoder", DecoderCompiler(cfg.decoder, blob, 1 << 30)), ("encoder", EncoderCompiler(EncoderConfig(), blob, 1 << 30))):
        for B, Lz in DECODER_PLANS:
            bufs = _Buffers()
            out[(kind, B, Lz)] = norms(comp.compile(_recording_arena(bufs, 1 << 32), B, Lz), bufs)
    wcfg = wave.WaveConfig()
    wblob = packer.WeightBlob()
    wave.pack_wave(wblob, wave.synthetic_wave_state_dict(wcfg), wcfg)
    wblob.finalize()
    wcomp = wave.WaveCompiler(wcfg, wblob, 1 << 30)
    for B, T in WAVE_PLANS:
        bufs = _Buffers()
        out[("wave", B, T)] = norms(wcomp.compile(_recording_arena(bufs, 1 << 32), B, T), bufs)
    return out


def plan_signatures() -> List[Case]:
    """the distinct norm signatures of every plan in UNET_PLANS, DECODER_PLANS (decoder and encoder) and WAVE_PLANS, first-seen order"""
    seen = {}
    for cases in plan_norm_ops().values():
        for c in cases:
            seen.setdefault(c, None)
    return list(seen)


# plan_signatures(), written out (tests/test_gpu_norm.py::test_plan_signatures keeps them equal).  GroupNorm: (B, L, C, G, silu, ldx,
# cx, ldy, cy) -- U-Net G = 32 (x a column window of a 2C / 3C concat buffer where a block reads its skip home), decoder / encoder
# G = 8, wave encoder G = 32 up to 524288 rows; LayerNorm: (rows, C, ldx, cx, ldy, cy), the U-Net plans without the LayerNorm fold
# (Beff * Lz >= 8192) and the wave encoder.
_GN_PLAN = [
    (2,96,384,32,1,384,0,384,0), (2,96,128,32,1,128,0,128,0), (2,96,128,32,0,128,0,128,0), (2,96,128,32,1,256,128,128,0),
    (2,48,640,32,1,640,0,640,0), (2,48,256,32,1,256,0,256,0), (2,48,256,32,0,256,0,256,0), (2,48,256,32,1,512,256,256,0),
    (2,24,768,32,1,768,0,768,0), (2,24,384,32,1,384,0,384,0), (2,24,384,32,0,384,0,384,0), (2,24,384,32,1,768,384,384,0),
    (2,12,896,32,1,896,0,896,0), (2,12,512,32,1,512,0,512,0), (2,12,512,32,0,512,0,512,0), (2,12,512,32,1,1024,512,512,0),
    (2,12,512,32,1,1536,1024,512,0), (2,12,1536,32,1,1536,0,1536,0), (2,12,1024,32,1,1024,0,1024,0), (2,24,1408,32,1,1408,0,1408,0),
    (2,24,640,32,1,640,0,640,0), (2,48,1152,32,1,1152,0,1152,0), (2,48,512,32,1,512,0,512,0), (2,48,384,32,1,384,0,384,0),
    (2,96,640,32,1,640,0,640,0), (2,96,256,32,1,256,0,256,0), (8,512,384,32,1,384,0,384,0), (8,512,128,32,1,128,0,128,0),
    (8,512,128,32,0,128,0,128,0), (8,512,128,32,1,256,128,128,0), (8,256,640,32,1,640,0,640,0), (8,256,256,32,1,256,0,256,0),
    (8,256,256,32,0,256,0,256,0), (8,256,256,32,1,512,256,256,0), (8,128,768,32,1,768,0,768,0), (8,128,384,32,1,384,0,384,0),
    (8,128,384,32,0,384,0,384,0), (8,128,384,32,1,768,384,384,0), (8,64,896,32,1,896,0,896,0), (8,64,512,32,1,512,0,512,0),
    (8,64,512,32,0,512,0,512,0), (8,64,512,32,1,1024,512,512,0), (8,64,512,32,1,1536,1024,512,0), (8,64,1536,32,1,1536,0,1536,0),
    (8,64,1024,32,1,1024,0,1024,0), (8,128,1408,32,1,1408,0,1408,0), (8,128,640,32,1,640,0,640,0), (8,256,1152,32,1,1152,0,1152,0),
    (8,256,512,32,1,512,0,512,0), (8,256,384,32,1,384,0,384,0), (8,512,640,32,1,640,0,640,0), (8,512,256,32,1,256,0,256,0),
    (64,512,384,32,1,384,0,384,0), (64,512,128,32,1,128,0,128,0), (64,512,128,32,0,128,0,128,0), (64,512,128,32,1,256,128,128,0),
    (64,256,640,32,1,640,0,640,0), (64,256,256,32,1,256,0,256,0), (64,256,256,32,0,256,0,256,0), (64,256,256,32,1,512,256,256,0),
    (64,128,768,32,1,768,0,768,0), (64,128,384,32,1,384,0,384,0), (64,128,384,32,0,384,0,384,0), (64,128,384,32,1,768,384,384,0),
    (64,64,896,32,1,896,0,896,0), (64,64,512,32,1,512,0,512,0), (64,64,512,32,0,512,0,512,0), (64,64,512,32,1,1024,512,512,0),
    (64,64,512,32,1,1536,1024,512,0), (64,64,1536,32,1,1536,0,1536,0), (64,64,1024,32,1,1024,0,1024,0), (64,128,1408,32,1,1408,0,1408,0),
    (64,128,640,32,1,640,0,640,0), (64,256,1152,32,1,1152,0,1152,0), (64,256,512,32,1,512,0,512,0), (64,256,384,32,1,384,0,384,0),
    (64,512,640,32,1,640,0,640,0), (64,512,256,32,1,256,0,256,0), (16,992,384,32,1,384,0,384,0), (16,992,128,32,1,128,0,128,0),
    (16,992,128,32,0,128,0,128,0), (16,992,128,32,1,256,128,128,0), (16,496,640,32,1,640,0,640,0), (16,496,256,32,1,256,0,256,0),
    (16,496,256,32,0,256,0,256,0), (16,496,256,32,1,512,256,256,0), (16,248,768,32,1,768,0,768,0), (16,248,384,32,1,384,0,384,0),
    (16,248,384,32,0,384,0,384,0), (16,248,384,32,1,768,384,384,0), (16,124,896,32,1,896,0,896,0), (16,124,512,32,1,512,0,512,0),
    (16,124,512,32,0,512,0,512,0), (16,124,512,32,1,1024,512,512,0), (16,124,512,32,1,1536,1024,512,0), (16,124,1536,32,1,1536,0,1536,0),
    (16,124,1024,32,1,1024,0,1024,0), (16,248,1408,32,1,1408,0,1408,0), (16,248,640,32,1,640,0,640,0), (16,496,1152,32,1,1152,0,1152,0),
    (16,496,512,32,1,512,0,512,0), (16,496,384,32,1,384,0,384,0), (16,992,640,32,1,640,0,640,0), (16,992,256,32,1,256,0,256,0),
    (2,2048,384,32,1,384,0,384,0), (2,2048,128,32,1,128,0,128,0), (2,2048,128,32,0,128,0,128,0), (2,2048,128,32,1,256,128,128,0),
    (2,1024,640,32,1,640,0,640,0), (2,1024,256,32,1,256,0,256,0), (2,1024,256,32,0,256,0,256,0), (2,1024,256,32,1,512,256,256,0),
    (2,512,768,32,1,768,0,768,0), (2,512,384,32,1,384,0,384,0), (2,512,384,32,0,384,0,384,0), (2,512,384,32,1,768,384,384,0),
    (2,256,896,32,1,896,0,896,0), (2,256,512,32,1,512,0,512,0), (2,256,512,32,0,512,0,512,0), (2,256,512,32,1,1024,512,512,0),
    (2,256,512,32,1,1536,1024,512,0), (2,256,1536,32,1,1536,0,1536,0), (2,256,1024,32,1,1024,0,1024,0), (2,512,1408,32,1,1408,0,1408,0),
    (2,512,640,32,1,640,0,640,0), (2,1024,1152,32,1,1152,0,1152,0), (2,1024,512,32,1,512,0,512,0), (2,1024,384,32,1,384,0,384,0),
    (2,2048,640,32,1,640,0,640,0), (2,2048,256,32,1,256,0,256,0), (1,8192,384,32,1,384,0,384,0), (1,8192,128,32,1,128,0,128,0),
    (1,8192,128,32,0,128,0,128,0), (1,8192,128,32,1,256,128,128,0), (1,4096,640,32,1,640,0,640,0), (1,4096,256,32,1,256,0,256,0),
    (1,4096,256,32,0,256,0,256,0), (1,4096,256,32,1,512,256,256,0), (1,2048,768,32,1,768,0,768,0), (1,2048,384,32,1,384,0,384,0),
    (1,2048,384,32,0,384,0,384,0), (1,2048,384,32,1,768,384,384,0), (1,1024,896,32,1,896,0,896,0), (1,1024,512,32,1,512,0,512,0),
    (1,1024,512,32,0,512,0,512,0), (1,1024,512,32,1,1024,512,512,0), (1,1024,512,32,1,1536,1024,512,0), (1,1024,1536,32,1,1536,0,1536,0),
    (1,1024,1024,32,1,1024,0,1024,0), (1,2048,1408,32,1,1408,0,1408,0), (1,2048,640,32,1,640,0,640,0), (1,4096,1152,32,1,1152,0,1152,0),
    (1,4096,512,32,1,512,0,512,0), (1,4096,384,32,1,384,0,384,0), (1,8192,640,32,1,640,0,640,0), (1,8192,256,32,1,256,0,256,0),
    (1,96,256,8,1,256,0,256,0), (1,192,256,8,1,256,0,256,0), (1,384,256,8,1,256,0,256,0), (1,384,128,8,1,128,0,128,0),
    (1,768,128,8,1,128,0,128,0), (1,768,64,8,1,64,0,64,0), (4,512,256,8,1,256,0,256,0), (4,1024,256,8,1,256,0,256,0),
    (4,2048,256,8,1,256,0,256,0), (4,2048,128,8,1,128,0,128,0), (4,4096,128,8,1,128,0,128,0), (4,4096,64,8,1,64,0,64,0),
    (1,8192,256,8,1,256,0,256,0), (1,16384,256,8,1,256,0,256,0), (1,32768,256,8,1,256,0,256,0), (1,32768,128,8,1,128,0,128,0),
    (1,65536,128,8,1,128,0,128,0), (1,65536,64,8,1,64,0,64,0), (1,384,64,8,1,64,0,64,0), (1,192,128,8,1,128,0,128,0),
    (4,2048,64,8,1,64,0,64,0), (4,1024,128,8,1,128,0,128,0), (1,32768,64,8,1,64,0,64,0), (1,16384,128,8,1,128,0,128,0),
    (2,6144,128,32,1,128,0,128,0), (2,3072,128,32,1,128,0,128,0), (2,1536,128,32,1,128,0,128,0), (2,768,128,32,1,128,0,128,0),
    (2,384,128,32,1,128,0,128,0), (2,384,256,32,1,256,0,256,0), (2,192,256,32,1,256,0,256,0), (2,48,512,32,0,512,0,512,0),
    (2,24,512,32,1,512,0,512,0), (2,24,512,32,0,512,0,512,0), (2,32768,128,32,1,128,0,128,0), (2,16384,128,32,1,128,0,128,0),
    (2,8192,128,32,1,128,0,128,0), (2,4096,128,32,1,128,0,128,0), (2,512,256,32,1,256,0,256,0), (2,256,256,32,1,256,0,256,0),
    (2,128,512,32,1,512,0,512,0), (2,128,512,32,0,512,0,512,0), (2,64,512,32,1,512,0,512,0), (2,64,512,32,0,512,0,512,0),
    (1,524288,128,32,1,128,0,128,0), (1,262144,128,32,1,128,0,128,0), (1,131072,128,32,1,128,0,128,0), (1,65536,128,32,1,128,0,128,0),
    (1,32768,128,32,1,128,0,128,0), (1,32768,256,32,1,256,0,256,0), (1,16384,256,32,1,256,0,256,0), (1,4096,512,32,0,512,0,512,0),
    (1,2048,512,32,1,512,0,512,0), (1,2048,512,32,0,512,0,512,0),
]
_LN_PLAN = [
    (16384,256,256,0,256,0), (8192,384,384,0,384,0), (4096,512,512,0,512,0), (7936,256,256,0,256,0), (3968,384,384,0,384,0),
    (1984,512,512,0,512,0), (4096,256,256,0,256,0), (2048,384,384,0,384,0), (1024,512,512,0,512,0), (96,512,512,0,512,0),
    (48,512,512,0,512,0), (24,512,512,0,512,0), (512,512,512,0,512,0), (256,512,512,0,512,0), (128,512,512,0,512,0),
    (2048,512,512,0,512,0),
]

PLAN_CASES: List[Case] = [Case(*t) for t in _GN_PLAN] + [ln(*t) for t in _LN_PLAN]


# ---- edge cases ------------------------------------------------------------------------------------------------------------------
# one shape per kernel for the data regimes: x the second C columns of a 2C-wide buffer (as a U-Net block reading its skip home)
REGIME_SHAPES = {"reg2": (3, 96, 384, 32), "reg4": (3, 400, 256, 32), "reg8": (3, 992, 256, 32), "reg16": (3, 1024, 512, 32),
                 "reg32": (3, 2048, 384, 32), "two": (3, 4096, 128, 8)}


def _edge_cases() -> Dict[str, Case]:
    e: Dict[str, Case] = {}

    def add(name, c):
        assert name not in e, name
        e[name] = c

    # the launcher's variant boundaries, both sides: float4 per slab L * (C/G) / 4 at or below 512 .. 8192, and one row more
    for bound in (512, 1024, 2048, 4096, 8192):
        for cg in (4, 12, 20, 44, 48):
            q = cg // 4
            for L in (bound // q, bound // q + 1):
                C = 8 * cg
                add(f"slab{L * q}-cg{cg}", gn(2, L, C, 8, (L + cg) % 2, ldx=C + 8, cx=4))
    # one row per group
    for C, G in ((256, 8), (128, 32), (1536, 32)):
        add(f"rows1-C{C}-G{G}", gn(64, 1, C, G, True))
    # windows with ldx != ldy, at column offsets that are multiples of 4 but not of 32
    add("window-reg2", gn(3, 100, 256, 32, True, ldx=768, cx=260, ldy=384, cy=68))
    add("window-reg16", gn(2, 700, 640, 32, False, ldx=1288, cx=4, ldy=704, cy=36))
    add("window-two", gn(2, 3000, 192, 8, True, ldx=200, cx=8, ldy=452, cy=260))
    add("window-ln", ln(77, 384, ldx=1028, cx=516, ldy=392, cy=4))
    # LayerNorm: C from one float4 to the kernel's 1024; rows around the 8 warps of a CTA
    for C in (4, 128, 1020, 1024):
        for rows in (1, 7, 8, 9):
            add(f"ln-C{C}-r{rows}", ln(rows, C))
    # the data regimes on every kernel, with and without SiLU
    for regime in REGIMES:
        for kern, (B, L, C, G) in REGIME_SHAPES.items():
            for silu in (0, 1):
                add(f"{regime}-{kern}" + ("-silu" if silu else ""), gn(B, L, C, G, silu, ldx=2 * C, cx=C, regime=regime))
        for rows, C in ((300, 256), (100, 512), (40, 1024)):
            add(f"{regime}-ln-C{C}", ln(rows, C, ldx=2 * C, cx=C, regime=regime))
    # the parameter sets of the earlier test_groupnorm / test_layernorm (a symmetric pad: ldx = ldy = C + pad, window at pad / 2)
    for B, L, C, G, silu, pad in [(2, 96, 384, 32, True, 0), (3, 12, 1536, 32, True, 64), (2, 768, 64, 8, True, 0),
                                  (1, 24, 896, 32, False, 32), (2, 124, 512, 32, False, 0), (8, 512, 128, 32, True, 0),
                                  (2, 992, 256, 32, True, 0), (2, 512, 640, 32, True, 128), (2, 10, 128, 32, False, 0),
                                  (1, 5, 256, 32, True, 0), (2, 992, 640, 32, True, 0), (3, 62, 1408, 32, True, 0)]:
        add(f"ops-B{B}-L{L}-C{C}-G{G}-pad{pad}", gn(B, L, C, G, silu, ldx=C + pad, cx=pad // 2, ldy=C + pad, cy=pad // 2))
    for rows, C in [(100, 256), (37, 384), (64, 512), (5, 1024)]:
        add(f"ops-ln-r{rows}-C{C}", ln(rows, C))
    return e


EDGE_CASES: Dict[str, Case] = _edge_cases()
