"""Audio (mel-spectrogram) encoder on the GPU -- SURVEY §8f row N1, the step immediately before the DDIM loop.

Reference: ``MelspectrogramScaleEncoder1D`` (mug/cond/wave.py:398-473, shipped config mug_diffusion.yaml:75-87): conv3
128->128, then 10 levels [Downsample (from level 1) ; 2 x (ResnetBlock with dilated k=3 convs (1,2) / (4,8), GroupNorm 32,
no time embedding) ; ContextualTransformer without context at the 3 coarsest levels]; returns the 10 level outputs, of which
the U-Net consumes the last four (unet.py:527-543).  49.8 GFLOP per sample at T = 32768 frames, run once per request.

Everything here reuses the hot-path kernels (wgmma GEMM with dilated-tap TMA addressing, GroupNorm+SiLU, LayerNorm,
attention) through launch plans; no new kernel was needed except the tap dilation in the GEMM addressing.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import lib as L_
from .engine import Arena, GN_EPS, OpList, TAG_ATTN, TAG_IO, TAG_RES, TAG_UPDOWN, View, tc_weight_map
from .packer import WeightBlob, _conv1, _conv3, _interleave_halves

WAVE_PREFIX = "model.wave_model."


@dataclass(frozen=True)
class WaveConfig:
    n_freq: int = 128
    middle_channels: int = 128
    attention_resolutions: Tuple[int, ...] = (128, 256, 512)
    num_res_blocks: int = 2
    num_heads: int = 8
    num_groups: int = 32
    channel_mult: Tuple[int, ...] = (1, 1, 1, 1, 2, 2, 2, 4, 4, 4)
    pos_max: int = 64


@dataclass
class WBlock:
    kind: str                 # conv_in | down | res | attn
    prefix: str
    cin: int
    cout: int
    level: int
    dil: Tuple[int, int] = (1, 1)


def wave_layout(cfg: WaveConfig, prefix: str = WAVE_PREFIX) -> List[WBlock]:
    """Execution order of MelspectrogramScaleEncoder1D.forward (wave.py:453-467)."""
    mc = cfg.middle_channels
    seq = [WBlock("conv_in", prefix + "conv_in.", cfg.n_freq, mc, 0)]
    inm = (1,) + tuple(cfg.channel_mult)
    ds = 1
    for lvl in range(len(cfg.channel_mult)):
        cin, cout = mc * inm[lvl], mc * cfg.channel_mult[lvl]
        if lvl != 0:
            seq.append(WBlock("down", f"{prefix}down.{lvl}.downsample.", cin, cin, lvl))
            ds *= 2
        for j in range(cfg.num_res_blocks):
            seq.append(WBlock("res", f"{prefix}down.{lvl}.block.{j}.", cin, cout, lvl, (1, 2) if j % 2 == 0 else (4, 8)))
            if ds in cfg.attention_resolutions:
                seq.append(WBlock("attn", f"{prefix}down.{lvl}.attn.{j}.", cout, cout, lvl))
            cin = cout
    return seq


def wave_param_specs(cfg: WaveConfig, prefix: str = WAVE_PREFIX) -> Dict[str, Tuple[Tuple[int, ...], str]]:
    out: Dict[str, Tuple[Tuple[int, ...], str]] = {}

    def conv(p, ci, co, k):
        out[p + "weight"] = ((co, ci, k), "w")
        out[p + "bias"] = ((co,), "b")

    def lin(p, ci, co, bias=True):
        out[p + "weight"] = ((co, ci), "w")
        if bias:
            out[p + "bias"] = ((co,), "b")

    def norm(p, c):
        out[p + "weight"] = ((c,), "gamma")
        out[p + "bias"] = ((c,), "beta")

    for b in wave_layout(cfg, prefix):
        p = b.prefix
        if b.kind == "conv_in":
            conv(p, b.cin, b.cout, 3)
        elif b.kind == "down":
            conv(p + "conv.", b.cin, b.cout, 3)
        elif b.kind == "res":
            norm(p + "norm1.", b.cin)
            conv(p + "conv1.", b.cin, b.cout, 3)
            norm(p + "norm2.", b.cout)
            conv(p + "conv2.", b.cout, b.cout, 3)
            if b.cin != b.cout:
                conv(p + "nin_shortcut.", b.cin, b.cout, 1)
        elif b.kind == "attn":
            c = b.cin
            norm(p + "norm.", c)
            conv(p + "proj_in.", c, c, 1)
            t = p + "transformer_blocks.0."
            for a in ("attn1.", "attn2."):
                out[t + a + "relative_position_embedding"] = ((2 * cfg.pos_max + 1, cfg.num_heads), "relpos")
                out[t + a + "C_embedding"] = ((2 * cfg.pos_max + 1, cfg.num_heads), "cemb")
                lin(t + a + "to_q.", c, c, bias=False)
                lin(t + a + "to_k.", c, c, bias=False)
                lin(t + a + "to_v.", c, c, bias=False)
                lin(t + a + "to_out.0.", c, c)
            lin(t + "ff.net.0.proj.", c, 8 * c)
            lin(t + "ff.net.2.", 4 * c, c)
            for n in ("norm1.", "norm2.", "norm3."):
                norm(t + n, c)
            conv(p + "proj_out.", c, c, 1)
    return out


def synthetic_wave_state_dict(cfg: Optional[WaveConfig] = None, seed: int = 0) -> Dict[str, torch.Tensor]:
    from . import synth
    cfg = cfg or WaveConfig()
    return {name: synth._init(name, shape, role, seed) for name, (shape, role) in wave_param_specs(cfg).items()}


def synthetic_mel(B: int, T: int, seed: int = 4321) -> torch.Tensor:
    """log1p-mel-like input: uniform [0,4) rounded through fp16 like the reference loader (mug/util.py:143)."""
    from . import synth
    import numpy as np
    u = synth._rng(seed, "mel").random(size=(B, 128, T), dtype=np.float32) * 4.0
    return torch.from_numpy(u).to(torch.float16).to(torch.float32)


def pack_wave(blob: WeightBlob, sd: Dict[str, torch.Tensor], cfg: WaveConfig, prefix: str = WAVE_PREFIX):
    for b in wave_layout(cfg, prefix):
        p = b.prefix
        if b.kind == "conv_in":
            blob.add_shaped(p + "weight", _conv3(sd[p + "weight"]))
            blob.add_shaped(p + "bias", sd[p + "bias"])
        elif b.kind == "down":
            blob.add_shaped(p + "conv.weight", _conv3(sd[p + "conv.weight"]))
            blob.add_shaped(p + "conv.bias", sd[p + "conv.bias"])
        elif b.kind == "res":
            for n in ("norm1.", "norm2."):
                blob.add_shaped(p + n + "weight", sd[p + n + "weight"])
                blob.add_shaped(p + n + "bias", sd[p + n + "bias"])
            for n in ("conv1.", "conv2."):
                blob.add_shaped(p + n + "weight", _conv3(sd[p + n + "weight"]))
                blob.add_shaped(p + n + "bias", sd[p + n + "bias"])
            if b.cin != b.cout:
                blob.add_shaped(p + "nin_shortcut.weight", _conv1(sd[p + "nin_shortcut.weight"]))
                blob.add_shaped(p + "nin_shortcut.bias", sd[p + "nin_shortcut.bias"])
        elif b.kind == "attn":
            blob.add_shaped(p + "norm.weight", sd[p + "norm.weight"])
            blob.add_shaped(p + "norm.bias", sd[p + "norm.bias"])
            for n in ("proj_in.", "proj_out."):
                blob.add_shaped(p + n + "weight", _conv1(sd[p + n + "weight"]))
                blob.add_shaped(p + n + "bias", sd[p + n + "bias"])
            t = p + "transformer_blocks.0."
            for a in ("attn1.", "attn2."):        # no context: both are self-attention with their own weights
                blob.add_shaped(t + a + "qkv.weight", torch.cat([sd[t + a + "to_q.weight"], sd[t + a + "to_k.weight"],
                                                                 sd[t + a + "to_v.weight"]], dim=0))
                blob.add_shaped(t + a + "to_out.0.weight", sd[t + a + "to_out.0.weight"])
                blob.add_shaped(t + a + "to_out.0.bias", sd[t + a + "to_out.0.bias"])
                blob.add_shaped(t + a + "relative_position_embedding", sd[t + a + "relative_position_embedding"])
                blob.add_shaped(t + a + "C_embedding", sd[t + a + "C_embedding"])
            blob.add_shaped(t + "ff.net.0.proj.weight", _interleave_halves(sd[t + "ff.net.0.proj.weight"]))
            blob.add_shaped(t + "ff.net.0.proj.bias", _interleave_halves(sd[t + "ff.net.0.proj.bias"]))
            blob.add_shaped(t + "ff.net.2.weight", sd[t + "ff.net.2.weight"])
            blob.add_shaped(t + "ff.net.2.bias", sd[t + "ff.net.2.bias"])
            for n in ("norm1.", "norm2.", "norm3."):
                blob.add_shaped(t + n + "weight", sd[t + n + "weight"])
                blob.add_shaped(t + n + "bias", sd[t + n + "bias"])
    blob.meta["wave_cfg"] = cfg


class WaveCompiler:
    """Launch plan of one encoder pass for B spectrograms of T frames (T divisible by 2**9)."""

    def __init__(self, cfg: WaveConfig, blob: WeightBlob, wbase: int, tc_map: Optional[Dict[int, Tuple[int, int]]] = None,
                 prefix: str = WAVE_PREFIX):
        self.cfg, self.blob, self.wbase, self.prefix = cfg, blob, wbase, prefix
        self.tc_map = tc_weight_map(blob, wbase) if tc_map is None else tc_map
        self.seq = wave_layout(cfg, prefix)

    def w(self, name: str) -> int:
        return self.wbase + 4 * self.blob.offset(name)

    def compile(self, arena: Arena, B: int, T: int) -> dict:
        cfg = self.cfg
        nlev = len(cfg.channel_mult)
        assert T % (1 << (nlev - 1)) == 0, "mel length must be a multiple of 512 frames"
        ops = OpList(self.tc_map)
        G, H = cfg.num_groups, cfg.num_heads
        mel = arena.alloc(B * T, cfg.n_freq)
        cur = mel
        Lr = T
        outs: List[Tuple[View, int, int]] = []          # (view, channels, length) per level
        w = self.w

        def dconv(x: View, name: str, cout: int, cin: int, out: View, dil: int, residual: Optional[View] = None):
            ops.gemm(x, w(name + "weight"), cout, cin, out, bias=w(name + "bias"), taps=3, mode=L_.CONV_TAPS, Lin=Lr, Lout=Lr,
                     tap_shift=-1, dilation=dil, residual=residual, tag=TAG_RES)

        level_of_last = {}
        for idx, b in enumerate(self.seq):
            level_of_last[b.level] = idx
        for idx, b in enumerate(self.seq):
            p = b.prefix
            if b.kind == "conv_in":
                o = arena.alloc(B * Lr, b.cout)
                ops.gemm(cur, w(p + "weight"), b.cout, b.cin, o, bias=w(p + "bias"), taps=3, mode=L_.CONV_SAME, Lin=Lr, Lout=Lr, tag=TAG_IO)
                cur = o
            elif b.kind == "down":
                o = arena.alloc(B * Lr // 2, b.cout)
                ops.gemm(cur, w(p + "conv.weight"), b.cout, b.cin, o, bias=w(p + "conv.bias"), taps=3, mode=L_.CONV_DOWN, Lin=Lr,
                         Lout=Lr // 2, tag=TAG_UPDOWN)
                Lr //= 2
                cur = o
            elif b.kind == "res":
                o = arena.alloc(B * Lr, b.cout)
                m = arena.mark()
                t1 = arena.alloc(B * Lr, b.cin)
                ops.groupnorm(cur, t1, w(p + "norm1.weight"), w(p + "norm1.bias"), B, Lr, G, True, TAG_RES)
                t2 = arena.alloc(B * Lr, b.cout)
                dconv(t1, p + "conv1.", b.cout, b.cin, t2, b.dil[0])
                t3 = arena.alloc(B * Lr, b.cout)
                ops.groupnorm(t2, t3, w(p + "norm2.weight"), w(p + "norm2.bias"), B, Lr, G, True, TAG_RES)
                res = cur
                if b.cin != b.cout:
                    t4 = arena.alloc(B * Lr, b.cout)
                    ops.gemm(cur, w(p + "nin_shortcut.weight"), b.cout, b.cin, t4, bias=w(p + "nin_shortcut.bias"), Lout=Lr, tag=TAG_RES)
                    res = t4
                dconv(t3, p + "conv2.", b.cout, b.cout, o, b.dil[1], residual=res)
                arena.release(m)
                cur = o
            elif b.kind == "attn":
                o = arena.alloc(B * Lr, b.cout)
                self._emit_attn(ops, arena, b, cur, o, B, Lr, H, G)
                cur = o
            if level_of_last[b.level] == idx:
                outs.append((cur, b.cout, Lr))
        return dict(ops=ops, mel=mel, outs=outs)

    def _emit_attn(self, ops: OpList, arena: Arena, b: WBlock, x: View, out: View, B: int, Lr: int, H: int, G: int):
        """ContextualTransformer with context=None (attention.py:186-199, 147-151): attn2 is a second self-attention."""
        cfg, w = self.cfg, self.w
        Cc = b.cin
        m = arena.mark()
        p = b.prefix
        t = p + "transformer_blocks.0."
        g = arena.alloc(x.rows, Cc)
        ops.groupnorm(x, g, w(p + "norm.weight"), w(p + "norm.bias"), B, Lr, G, False, TAG_ATTN)
        h0 = arena.alloc(x.rows, Cc)
        ops.gemm(g, w(p + "proj_in.weight"), Cc, Cc, h0, bias=w(p + "proj_in.bias"), Lout=Lr, tag=TAG_ATTN)
        n1 = arena.alloc(x.rows, Cc)
        qkv = arena.alloc(x.rows, 3 * Cc)
        ao = arena.alloc(x.rows, Cc)
        h1 = arena.alloc(x.rows, Cc)
        cur, nxt = h0, h1
        for a, nrm in (("attn1.", "norm1."), ("attn2.", "norm2.")):
            ops.layernorm(cur, n1, w(t + nrm + "weight"), w(t + nrm + "bias"), TAG_ATTN)
            ops.gemm(n1, w(t + a + "qkv.weight"), 3 * Cc, Cc, qkv, Lout=Lr, tag=TAG_ATTN)
            ops.attention(qkv.c(0, Cc), qkv.c(Cc, 2 * Cc), qkv.c(2 * Cc, 3 * Cc), ao, w(t + a + "relative_position_embedding"),
                          w(t + a + "C_embedding"), B, H, Lr, Lr, cfg.pos_max, TAG_ATTN)
            ops.gemm(ao, w(t + a + "to_out.0.weight"), Cc, Cc, nxt, bias=w(t + a + "to_out.0.bias"), residual=cur, Lout=Lr, tag=TAG_ATTN)
            cur, nxt = nxt, cur
        # cur = h after attn2 (lives in h0's buffer), nxt = the other buffer (free)
        ops.layernorm(cur, n1, w(t + "norm3.weight"), w(t + "norm3.bias"), TAG_ATTN)
        ff = arena.alloc(x.rows, 4 * Cc)
        ops.gemm(n1, w(t + "ff.net.0.proj.weight"), 8 * Cc, Cc, ff, bias=w(t + "ff.net.0.proj.bias"), gate=L_.GATE_GEGLU, Lout=Lr, tag=TAG_ATTN)
        ops.gemm(ff, w(t + "ff.net.2.weight"), Cc, 4 * Cc, nxt, bias=w(t + "ff.net.2.bias"), residual=cur, Lout=Lr, tag=TAG_ATTN)
        ops.gemm(nxt, w(p + "proj_out.weight"), Cc, Cc, out, bias=w(p + "proj_out.bias"), residual=x, Lout=Lr, tag=TAG_ATTN)
        arena.release(m)


class WaveSession:
    """Compiled encoder for (B, T).  ``encode`` returns the reference's 10-entry list; the first 6 entries (never read by
    the U-Net, unet.py:527-543) are ``None`` unless ``all_levels`` is set."""

    def __init__(self, engine, B: int, T: int):
        from .runtime import compile_sized
        self.engine, self.B, self.T = engine, B, T
        cfg = engine.blob.meta["wave_cfg"]
        comp = WaveCompiler(cfg, engine.blob, engine.wbase, engine.tc_map)
        self.arena_t, res, self.plan = compile_sized(engine, lambda arena: comp.compile(arena, B, T), batch=(B, 1))
        self.mel, self.outs = res["mel"], res["outs"]
        self.cfg = cfg

    def encode(self, mel: torch.Tensor, all_levels: bool = False) -> List[Optional[torch.Tensor]]:
        self.load(mel)
        return self.run(all_levels)

    def load(self, mel: torch.Tensor):
        """NCL mel [B, n_freq, T] -> the plan's channels-last input rows ``self.mel``"""
        eng = self.engine
        mel = mel.to(eng.device, torch.float32).contiguous()
        assert mel.shape == (self.B, self.cfg.n_freq, self.T), mel.shape
        eng.ncl_to_rows(mel, self.mel)
        self._keep = mel

    def run(self, all_levels: bool = False) -> List[Optional[torch.Tensor]]:
        """One encoder pass over whatever the input rows hold (``load``, or the mel kernel writing them directly)."""
        eng = self.engine
        self.plan.run()
        nlev = len(self.outs)
        return [eng.rows_to_ncl(view, self.B, ch, Lr) if all_levels or i >= nlev - 4 else None
                for i, (view, ch, Lr) in enumerate(self.outs)]
