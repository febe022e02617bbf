"""Attention cases shared by tests/test_gpu_attention.py (importable without a GPU):

* ``ref_attention``  -- mugd_attention (include/mugd.h, header of csrc/attention.cu) in float64;
* ``plan_signatures`` -- every OP_ATTENTION descriptor of real U-Net and wave-encoder launch plans, compiled on the host with fake
  addresses and reduced to a ``Case`` (shape, pos_max, leading dimension and column offset of each operand in its buffer);
* ``PLAN_CASES``     -- those signatures written out, so the GPU tests need no plan compile (a CPU test keeps the two equal);
* ``kernel_for``     -- which kernel launch_attention picks for a case;
* ``EDGE_CASES``     -- hand-picked shapes, operand layouts and data regimes at the edges of the three kernels.
"""
from __future__ import annotations

import bisect
import zlib
from dataclasses import dataclass
from typing import Dict, List, Tuple

import torch


@dataclass(frozen=True)
class Case:
    B: int
    H: int
    D: int
    Lq: int
    Lk: int
    pos_max: int
    ldq: int
    cq: int                     # column offset of q in its buffer
    ldk: int
    ck: int
    ldv: int
    cv: int
    ldo: int
    co: int
    fused: str                  # "qkv": q, k, v are windows of one [B*Lq, ldq] buffer; "kv": k, v of one [B*Lk, ldk] buffer
    regime: str = "randn"       # input data, see make_inputs

    @property
    def C(self) -> int:
        return self.H * self.D

    @property
    def scale(self) -> float:
        return float(self.D) ** -0.5

    @property
    def id(self) -> str:
        s = f"B{self.B}-H{self.H}-D{self.D}-q{self.Lq}-k{self.Lk}-P{self.pos_max}-{self.fused}"
        if self.cq or self.ck != (self.C if self.fused == "qkv" else 0):
            s += f"-off{self.cq}.{self.ck}.{self.cv}"
        return s + ("" if self.regime == "randn" else "-" + self.regime)


def layout(B: int, H: int, D: int, Lq: int, Lk: int, pos_max: int = 64, fused: str = "", pad: int = 0,
           regime: str = "randn") -> Case:
    """a case laid out like the plans: "qkv" (self-attention, default when Lq == Lk) = q | k | v of one 3C-wide buffer, "kv" =
    q alone, k | v of one 2C-wide buffer.  pad > 0 moves every window pad columns right inside a buffer 2*pad columns wider."""
    C = H * D
    fused = fused or ("qkv" if Lq == Lk else "kv")
    if fused == "qkv":
        ld = 3 * C + 2 * pad
        return Case(B, H, D, Lq, Lk, pos_max, ld, pad, ld, pad + C, ld, pad + 2 * C, C, 0, fused, regime)
    ldq, ldkv = C + 2 * pad, 2 * C + 2 * pad
    return Case(B, H, D, Lq, Lk, pos_max, ldq, pad, ldkv, pad, ldkv, pad + C, C, 0, fused, regime)


def kernel_for(c: Case, impl: int) -> str:
    """the kernel launch_attention (csrc/attention.cu) runs: impl 1 (default) = lane-per-key for <= 32 keys at head dim 48 / 64,
    else the wgmma kernel; impl 0 = the FFMA referee for everything"""
    if impl == 0:
        return "ffma"
    return "lane" if (c.Lk <= 32 and c.D >= 48) else "tc"


# ---- fp64 reference ------------------------------------------------------------------------------------------------------------
def ref_attention(q, k, v, relpos, cgain, H: int, pos_max: int, scale: float):
    """q [B, Lq, H*D], k / v [B, Lk, H*D], relpos / cgain [2P+1, H]; in float64:
        idx_ij = clamp(j - i, -P, P) + P,  s_ij = (q_i . k_j + relpos[idx_ij]) * scale  (the bias inside the scale),
        p = softmax_j(s),  o_i = sum_j p_ij * cgain[idx_ij] * v_j  (the gain on the numerator only).
    Returns o [B, Lq, H*D] and the magnitude M [B, Lq, H, D] = sum_j p_ij |cgain[idx_ij]| |v_jc|, the scale an error of o is
    measured against (row by row: a row whose terms are small or cancel is not hidden behind the largest row)."""
    B, Lq, C = q.shape
    Lk, D = k.shape[1], C // H
    qh, kh, vh = (t.double().reshape(B, -1, H, D).permute(0, 2, 1, 3) for t in (q, k, v))
    idx = (torch.arange(Lk)[None, :] - torch.arange(Lq)[:, None]).clamp(-pos_max, pos_max) + pos_max
    rel = relpos.double()[idx].permute(2, 0, 1)[None]              # [1, H, Lq, Lk]
    cg = cgain.double()[idx].permute(2, 0, 1)[None]
    p = ((qh @ kh.transpose(-1, -2) + rel) * scale).softmax(-1)
    o = (p * cg) @ vh
    mag = (p * cg.abs()) @ vh.abs()
    return o.permute(0, 2, 1, 3).reshape(B, Lq, C), mag.permute(0, 2, 1, 3)


def row_error(o, ref, mag, H: int) -> float:
    """max over (sample, query row, head) of  max_c |o - ref| / max_c M"""
    B, Lq, C = ref.shape
    err = (o.double() - ref).abs().reshape(B, Lq, H, C // H).amax(-1)
    return float((err / mag.amax(-1).clamp_min(1e-300)).max())


# ---- inputs ----------------------------------------------------------------------------------------------------------------------
REGIMES = ("randn", "peaked", "gain", "offset")


def make_inputs(c: Case, salt: str = ""):
    """q [B, Lq, C], k / v [B, Lk, C], relpos / cgain [2P+1, H], seeded by the case.  Regimes:
    randn  -- unit normal q / k / v, relpos N(0, 1), cgain 1 + N(0, 0.25^2);
    peaked -- q x 4 (logits of standard deviation 4) and a relpos ramp that adds (j - i) / 8 to the scaled logit (-8 .. +8 at
              pos_max 64): with pos_max >= Lk the bias climbs 16 per 128 keys, nearly every row peaks in the last key tile and
              the online-softmax rescale of each earlier tile is large;
    gain   -- cgain N(0, 1) with every fifth entry exactly 0: negative and zero gains;
    offset -- v + 100: a large common value offset on top of unit-normal spread."""
    g = torch.Generator().manual_seed(zlib.crc32((c.id + salt).encode()))
    C, NT = c.C, 2 * c.pos_max + 1
    q = torch.randn(c.B, c.Lq, C, generator=g)
    k = torch.randn(c.B, c.Lk, C, generator=g)
    v = torch.randn(c.B, c.Lk, C, generator=g)
    rel = torch.randn(NT, c.H, generator=g)
    cg = 1 + 0.25 * torch.randn(NT, c.H, generator=g)
    if c.regime == "peaked":
        q = q * 4
        rel = ((torch.arange(NT, dtype=torch.float32) - c.pos_max) / 8 / c.scale)[:, None].repeat(1, c.H)
    elif c.regime == "gain":
        cg = torch.randn(NT, c.H, generator=g)
        cg.view(-1)[::5] = 0.0
    elif c.regime == "offset":
        v = v + 100.0
    else:
        assert c.regime == "randn", c.regime
    return q, k, v, rel, cg


# ---- signatures of real plans ----------------------------------------------------------------------------------------------------
UNET_PLANS = [(2, 32), (2, 96), (8, 512), (64, 512), (16, 992)]        # (Beff, Lz)
WAVE_PLANS = [(2, 6144), (2, 32768)]                                    # (B, T)


class _Buffers:
    """start address and width of every buffer a compile hands out, to map an operand address back to (buffer, column)"""

    def __init__(self):
        self.starts: List[int] = []
        self.cols: Dict[int, set] = {}

    def add(self, start: int, cols: int):
        if start not in self.cols:
            bisect.insort(self.starts, start)
            self.cols[start] = set()
        self.cols[start].add(cols)

    def locate(self, ptr: int, ld: int) -> Tuple[int, int]:
        """(buffer start, column offset) of a column window at ptr with leading dimension ld: the nearest buffer of width ld that
        starts at most one row before ptr"""
        i = bisect.bisect_right(self.starts, ptr)
        while i > 0:
            i -= 1
            s = self.starts[i]
            if ptr - s >= 4 * ld:
                break
            if ld in self.cols[s]:
                return s, (ptr - s) // 4
        raise AssertionError(f"no buffer of width {ld} holds address {ptr:#x}")


def _recording_arena(bufs: _Buffers, base: int):
    from mug_diffusion_b200.engine import Arena

    class RecordingArena(Arena):
        def alloc(self, rows, cols):
            v = super().alloc(rows, cols)
            bufs.add(v.ptr, cols)
            return v

    return RecordingArena(base)


def _fake_ext(comp, Beff: int, Lz: int, bufs: _Buffers):
    """the engine's per-session inputs of a U-Net plan (time-embedding table, step counter, context K/V, S4 kernels) at fake
    addresses"""
    from mug_diffusion_b200.engine import View
    blocks = list(comp.lay.blocks())
    ctx_kv = [View((1 << 41) + i * (1 << 24), 2 * b.cin, Beff * 21, 2 * b.cin) for i, b in enumerate(x for x in blocks if x.kind == "attn")]
    for kv in ctx_kv:
        bufs.add(kv.ptr, kv.ld)
    return dict(emb_table=1 << 40, step=(1 << 40) + 4096, ctx_tokens=21, ctx_kv=ctx_kv,
                s4_kt={b.prefix: View((1 << 42) + i * (1 << 24), b.cin, Lz // b.ds, b.cin)
                       for i, b in enumerate(x for x in blocks if x.kind == "s4")})


def _signature(d, bufs: _Buffers) -> Case:
    (bq, cq), (bk, ck), (bv, cv), (_, co) = (bufs.locate(p, ld) for p, ld in ((d.q, d.ldq), (d.k, d.ldk), (d.v, d.ldv), (d.o, d.ldo)))
    if bq == bk == bv:
        fused = "qkv"
    else:
        assert bk == bv and bq != bk, "k and v must share a buffer"
        fused = "kv"
    assert abs(d.scale - float(d.D) ** -0.5) < 1e-7
    return Case(d.B, d.H, d.D, d.Lq, d.Lk, d.pos_max, d.ldq, cq, d.ldk, ck, d.ldv, cv, d.ldo, co, fused)


def plan_attention_ops():
    """{("unet", Beff, Lz) | ("wave", B, T): [Case of each OP_ATTENTION, in plan order]}, from plans compiled on the host"""
    from mug_diffusion_b200 import lib as L_
    from mug_diffusion_b200 import packer, synth, wave
    from mug_diffusion_b200.config import ModelConfig
    from mug_diffusion_b200.engine import UNetCompiler

    out = {}
    cfg = ModelConfig()
    blob = packer.pack_model(synth.synthetic_state_dict(96), cfg.unet, cfg.decoder)
    comp = UNetCompiler(cfg.unet, blob, 1 << 30)
    for Beff, Lz in UNET_PLANS:
        bufs = _Buffers()
        res = comp.compile(_recording_arena(bufs, 1 << 32), Beff, Lz, _fake_ext(comp, Beff, Lz, bufs), False)
        out[("unet", Beff, Lz)] = [_signature(o.u.attn, bufs) for o in res["ops"].ops if o.kind == L_.OP_ATTENTION]
    wcfg = wave.WaveConfig()
    wblob = packer.WeightBlob()
    wave.pack_wave(wblob, wave.synthetic_wave_state_dict(wcfg), wcfg)
    wblob.finalize()
    wcomp = wave.WaveCompiler(wcfg, wblob, 1 << 30)
    for B, T in WAVE_PLANS:
        bufs = _Buffers()
        res = wcomp.compile(_recording_arena(bufs, 1 << 32), B, T)
        out[("wave", B, T)] = [_signature(o.u.attn, bufs) for o in res["ops"].ops if o.kind == L_.OP_ATTENTION]
    return out


def plan_signatures() -> List[Case]:
    """the distinct attention signatures of every plan in UNET_PLANS and WAVE_PLANS, in first-seen order"""
    seen = {}
    for cases in plan_attention_ops().values():
        for c in cases:
            seen.setdefault(c, None)
    return list(seen)


def _qkv(B, H, D, L):
    C = H * D
    return Case(B, H, D, L, L, 64, 3 * C, 0, 3 * C, C, 3 * C, 2 * C, C, 0, "qkv")


def _ctx(B, H, D, L):
    C = H * D
    return Case(B, H, D, L, 21, 64, C, 0, 2 * C, 0, 2 * C, C, C, 0, "kv")


# plan_signatures(), written out (tests/test_gpu_attention.py::test_plan_signatures keeps them equal): U-Net levels 1-3 carry
# attention at head dims 32 / 48 / 64 (self-attention over Lz/2, Lz/4, Lz/8 rows, cross-attention to the 21 prompt tokens); the
# wave encoder's three coarsest levels run two self-attentions each at head dim 64 over T/128, T/256, T/512 frames
PLAN_CASES: List[Case] = list(dict.fromkeys(
    [f(Beff, 8, D, Lz >> lvl) for Beff, Lz in UNET_PLANS for lvl, D in ((1, 32), (2, 48), (3, 64)) for f in (_qkv, _ctx)] +
    [_qkv(B, 8, 64, T >> s) for B, T in WAVE_PLANS for s in (7, 8, 9)]))


# ---- edge cases ------------------------------------------------------------------------------------------------------------------
def _edge_cases() -> Dict[str, Case]:
    e: Dict[str, Case] = {}

    def add(name, c):
        assert name not in e, name
        e[name] = c

    # lane-per-key kernel: 1 .. 32 keys; 33 crosses over to the wgmma kernel
    for D in (48, 64):
        for Lk in (1, 2, 21, 31, 32, 33):
            add(f"keys-{'lane' if Lk <= 32 else 'tc'}-D{D}-k{Lk}", layout(2, 8, D, 77, Lk))
    # key-tile edges: the FFMA kernel's 64-key tile and the wgmma kernel's 128-key tile; 3 tiles at D 32 / 48 reuse a pipeline stage
    for D in (32, 48, 64):
        for Lk in (63, 64, 65, 127, 128, 129, 255, 256, 257):
            add(f"ktile-tc-D{D}-k{Lk}", layout(1, 2, D, 70, Lk, fused="kv"))
    # query-tile edges: ASK_ROWS = 32 (lane-per-key), AT_BQ = 64 (FFMA), BQ = 128 (wgmma) all end in a partial tile
    for Lq in (1, 31, 32, 33, 127, 128, 129):
        add(f"qtile-lane-q{Lq}", layout(2, 8, 64, Lq, 21))
        add(f"qtile-tc-q{Lq}", layout(2, 4, 48, Lq, 150, fused="kv"))
    # j - i beyond +-pos_max on both sides: the clamped ends of the relpos / cgain tables
    add("clamp-tc-D32-q300-k40", layout(2, 4, 32, 300, 40, pos_max=16))
    add("clamp-tc-D32-q40-k300", layout(2, 4, 32, 40, 300, pos_max=16))
    add("clamp-tc-D64-q333-k333", layout(1, 4, 64, 333, 333, pos_max=64))
    add("clamp-lane-D64-q200-k21", layout(2, 8, 64, 200, 21))
    add("clamp-lane-D48-q150-k32", layout(2, 8, 48, 150, 32, pos_max=8))
    # pos_max 0, 1, 64 and the launcher's maximum 1024 (wgmma D 64: ~177 KB of shared memory)
    for P in (0, 1, 64, 1024):
        add(f"posmax{P}-tc-D64", layout(1, 2, 64, 1100 if P == 1024 else 150, 1100 if P == 1024 else 150, pos_max=P))
        add(f"posmax{P}-tc-D32", layout(1, 2, 32, 150, 150, pos_max=P))
        add(f"posmax{P}-lane-D48", layout(2, 8, 48, 40, 21, pos_max=P))
    # one head of dim 48: the second 32-channel TMA slab runs past the tensor's last column and must arrive as zeros
    add("h1-tc-D48", layout(2, 1, 48, 200, 200))
    add("h1-lane-D48", layout(2, 1, 48, 50, 21))
    # windows at column offsets that are multiples of 4 but not of 32
    add("off4-tc-D32", layout(2, 8, 32, 140, 140, pad=4))
    add("off12-tc-D48", layout(2, 3, 48, 200, 200, pad=12))
    add("off4-tc-D64-kv", layout(2, 8, 64, 130, 150, fused="kv", pad=4))
    add("off20-lane-D64", layout(2, 8, 64, 70, 21, pad=20))
    # data regimes, on each kernel (peaked: pos_max >= Lk, so the bias ramp runs over the whole row)
    for regime in REGIMES[1:]:
        P = 300 if regime == "peaked" else 64
        add(f"{regime}-tc-D32", layout(2, 8, 32, 300, 300, pos_max=P, regime=regime))
        add(f"{regime}-tc-D64", layout(2, 8, 64, 300, 300, pos_max=P, regime=regime))
        add(f"{regime}-tc-D32-ctx", layout(2, 8, 32, 100, 21, regime=regime))
        add(f"{regime}-lane-D48", layout(2, 8, 48, 100, 21, regime=regime))
    add("peaked-tc-D48-P64", layout(2, 8, 48, 300, 300, regime="peaked"))
    # the batch of BASELINE configs 3 and 4
    add("beff64-tc-D32-peaked", layout(64, 8, 32, 256, 256, pos_max=256, regime="peaked"))
    return e


EDGE_CASES: Dict[str, Case] = _edge_cases()
