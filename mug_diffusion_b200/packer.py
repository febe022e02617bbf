"""Weight packer: reference ``state_dict`` -> one contiguous fp32 blob in kernel-friendly layouts.

Layouts (all row-major fp32, every tensor 256-byte aligned inside the blob):
  conv k=3   [Cout][Cin][3]  ->  [Cout][3][Cin]      (K-major per tap: the A operand is channels-last)
  conv k=1   [Cout][Cin][1]  ->  [Cout][Cin]
  self-attn  to_q|to_k|to_v  ->  one [3C][C] matrix  (attention.py:77-79: one GEMM instead of three)
  cross-attn to_k|to_v       ->  one [2C][ctx] matrix (runs once per request: context is step-invariant)
  GEGLU / S4 output_linear   ->  rows interleaved (value_j, gate_j) so the gate is applied in the epilogue
  emb_layers of all ResBlocks->  one [sum Cout][512] matrix (evaluated once per request for all S steps)
  ResBlock conv2 + skip 1x1  ->  one [Cout][3*Cout + Cin] matrix: the skip_connection runs as extra k-steps of the second
                                 conv's GEMM on a second activation source (unet.py:187-193,237-239; decoder nin_shortcut too)
  ff.net.2 then proj_out     ->  one [C][4C + C] matrix  [Wp Wf | Wp]:  proj_out(ff.net.2(f) + h) = (Wp Wf) f + Wp h + (Wp bf + bp)
                                 (attention.py:57-65,194-199; the product is formed in fp64 at pack time)
The blob is what rank 0 broadcasts over NCCL for multi-GPU runs (one collective, SURVEY §8e).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from .config import DecoderConfig, EncoderConfig, UNetConfig
from .netspec import RES_LAYERS, Block, decoder_layout, encoder_layout, unet_layout

ALIGN = 64  # floats (256 B)


@dataclass
class Entry:
    offset: int           # in floats
    shape: Tuple[int, ...]


class WeightBlob:
    def __init__(self):
        self.entries: Dict[str, Entry] = {}
        self._chunks: List[torch.Tensor] = []
        self._size = 0
        self.meta: Dict[str, object] = {}
        self.data: torch.Tensor | None = None      # finalized flat tensor (CPU, then moved)
        self.tc: List[Tuple[str, int, int, int]] = []   # tensor-core weights: (entry, blob offset, elements, offset in the lo buffer)
        self.tc_lo_numel = 0

    def add(self, name: str, t: torch.Tensor):
        assert name not in self.entries, name
        t = t.detach().to(torch.float32).contiguous().reshape(-1).cpu()
        pad = (-self._size) % ALIGN
        if pad:
            self._chunks.append(torch.zeros(pad))
            self._size += pad
        self.entries[name] = Entry(self._size, tuple(t.shape))
        self._chunks.append(t)
        self._size += t.numel()

    def add_shaped(self, name: str, t: torch.Tensor):
        shape = tuple(t.shape)
        self.add(name, t)
        self.entries[name].shape = shape

    def finalize(self) -> torch.Tensor:
        pad = (-self._size) % ALIGN
        if pad:
            self._chunks.append(torch.zeros(pad))
            self._size += pad
        self.data = torch.cat(self._chunks)
        self._chunks = []
        return self.data

    @property
    def numel(self) -> int:
        return self._size

    def offset(self, name: str) -> int:
        return self.entries[name].offset

    def view(self, name: str) -> torch.Tensor:
        e = self.entries[name]
        n = 1
        for s in e.shape:
            n *= s
        return self.data[e.offset:e.offset + n].view(e.shape)


def tf32_rna(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> nearest TF32 value (10-bit mantissa, ties away from zero) = PTX cvt.rna.tf32.f32, as fp32."""
    u = x.contiguous().view(torch.int32)
    return ((u + 0x1000) & ~0x1FFF).view(torch.float32)


def tf32_split(w: torch.Tensor):
    """w ~= hi + lo with both parts exactly representable in TF32 (the B operand of the 3xTF32 tensor-core GEMM)."""
    hi = tf32_rna(w)
    lo = tf32_rna(w - hi)
    return hi, lo


def _conv3(w: torch.Tensor) -> torch.Tensor:
    return w.permute(0, 2, 1).contiguous().reshape(w.shape[0], -1)


def _conv1(w: torch.Tensor) -> torch.Tensor:
    return w.reshape(w.shape[0], w.shape[1])


def _interleave_halves(w: torch.Tensor) -> torch.Tensor:
    """rows [a_0..a_{h-1}, g_0..g_{h-1}] -> [a_0, g_0, a_1, g_1, ...] (works for weight and bias)."""
    h = w.shape[0] // 2
    return torch.stack([w[:h], w[h:]], dim=1).reshape(w.shape)


def _pack_block(blob: WeightBlob, sd: Dict[str, torch.Tensor], b: Block):
    p = b.prefix
    if b.kind in ("conv_in", "dec_conv_in"):
        blob.add_shaped(p + "weight", _conv3(sd[p + "weight"]))
        blob.add_shaped(p + "bias", sd[p + "bias"])
    elif b.kind in RES_LAYERS:
        norm1, conv1, norm2, conv2, skip = RES_LAYERS[b.kind]
        for n in (norm1, norm2):
            blob.add_shaped(p + n + "weight", sd[p + n + "weight"])
            blob.add_shaped(p + n + "bias", sd[p + n + "bias"])
        for n in (conv1,) + (() if b.has_skip_conv else (conv2,)):
            blob.add_shaped(p + n + "weight", _conv3(sd[p + n + "weight"]))
            blob.add_shaped(p + n + "bias", sd[p + n + "bias"])
        if b.has_skip_conv:
            blob.add_shaped(p + "out_skip.weight", torch.cat([_conv3(sd[p + conv2 + "weight"]), _conv1(sd[p + skip + "weight"])], dim=1))
            blob.add_shaped(p + "out_skip.bias", sd[p + conv2 + "bias"] + sd[p + skip + "bias"])
    elif b.kind == "attn":
        blob.add_shaped(p + "norm.weight", sd[p + "norm.weight"])
        blob.add_shaped(p + "norm.bias", sd[p + "norm.bias"])
        blob.add_shaped(p + "proj_in.weight", _conv1(sd[p + "proj_in.weight"]))
        blob.add_shaped(p + "proj_in.bias", sd[p + "proj_in.bias"])
        t = p + "transformer_blocks.0."
        wp, wf = _conv1(sd[p + "proj_out.weight"]).double(), sd[t + "ff.net.2.weight"].double()
        blob.add_shaped(p + "ff_out.weight", torch.cat([wp @ wf, wp], dim=1).float())
        blob.add_shaped(p + "ff_out.bias", (wp @ sd[t + "ff.net.2.bias"].double() + sd[p + "proj_out.bias"].double()).float())
        blob.add_shaped(t + "attn1.qkv.weight", torch.cat([sd[t + "attn1.to_q.weight"], sd[t + "attn1.to_k.weight"],
                                                           sd[t + "attn1.to_v.weight"]], dim=0))
        blob.add_shaped(t + "attn2.to_q.weight", sd[t + "attn2.to_q.weight"])
        blob.add_shaped(t + "attn2.kv.weight", torch.cat([sd[t + "attn2.to_k.weight"], sd[t + "attn2.to_v.weight"]], dim=0))
        for a in ("attn1.", "attn2."):
            blob.add_shaped(t + a + "to_out.0.weight", sd[t + a + "to_out.0.weight"])
            blob.add_shaped(t + a + "to_out.0.bias", sd[t + a + "to_out.0.bias"])
            blob.add_shaped(t + a + "relative_position_embedding", sd[t + a + "relative_position_embedding"])
            blob.add_shaped(t + a + "C_embedding", sd[t + a + "C_embedding"])
        blob.add_shaped(t + "ff.net.0.proj.weight", _interleave_halves(sd[t + "ff.net.0.proj.weight"]))
        blob.add_shaped(t + "ff.net.0.proj.bias", _interleave_halves(sd[t + "ff.net.0.proj.bias"]))
        for n in ("norm1.", "norm2.", "norm3."):
            blob.add_shaped(t + n + "weight", sd[t + n + "weight"])
            blob.add_shaped(t + n + "bias", sd[t + n + "bias"])
        # LayerNorm folded into the Linear behind it (attention.py:147-151):  W LN(h) + b = rstd (W' h - mean colsum) + b'  with
        # W' = W diag(gamma), colsum = W' 1, b' = W beta + b  -- formed in fp64
        for norm, lin, wkey, bkey in (("norm1.", "attn1.qkv", t + "attn1.qkv.weight", None),
                                      ("norm2.", "attn2.to_q", t + "attn2.to_q.weight", None),
                                      ("norm3.", "ff.net.0.proj", t + "ff.net.0.proj.weight", t + "ff.net.0.proj.bias")):
            w = blob_tensor(blob, wkey).double()
            gam, bet = sd[t + norm + "weight"].double(), sd[t + norm + "bias"].double()
            wg = (w * gam[None, :]).float()
            blob.add_shaped(t + lin + "_ln.weight", wg)
            blob.add_shaped(t + lin + "_ln.colsum", wg.double().sum(dim=1).float())
            bias = w @ bet + (blob_tensor(blob, bkey).double() if bkey else 0.0)
            blob.add_shaped(t + lin + "_ln.bias", bias.float())
    elif b.kind == "s4":
        blob.add_shaped(p + "norm.weight", sd[p + "norm.weight"])
        blob.add_shaped(p + "norm.bias", sd[p + "norm.bias"])
        s = p + "s4_model."
        blob.add_shaped(s + "D", sd[s + "D"].reshape(-1))
        k = s + "kernel.kernel."
        for n in ("C", "log_dt", "B", "P", "inv_w_real", "w_imag"):
            blob.add_shaped(k + n, sd[k + n])
        blob.meta[k + "L"] = int(sd[k + "L"].item())
        blob.add_shaped(s + "output_linear.0.weight", _interleave_halves(_conv1(sd[s + "output_linear.0.weight"])))
        blob.add_shaped(s + "output_linear.0.bias", _interleave_halves(sd[s + "output_linear.0.bias"]))
        blob.add_shaped(p + "out_layer.weight", _conv3(sd[p + "out_layer.weight"]))
        blob.add_shaped(p + "out_layer.bias", sd[p + "out_layer.bias"])
    elif b.kind in ("down", "up"):
        w = sd[p + "conv.weight"]
        blob.add_shaped(p + "conv.weight", _conv3(w))
        blob.add_shaped(p + "conv.bias", sd[p + "conv.bias"])
        if b.kind == "up":
            # nearest-x2 upsample followed by conv3 == two 2-tap convs on the un-upsampled rows (models.py:66-70):
            #   y[2j]   = W0 x[j-1] + (W1+W2) x[j]        y[2j+1] = (W0+W1) x[j] + W2 x[j+1]
            w0, w1, w2 = w[:, :, 0], w[:, :, 1], w[:, :, 2]
            blob.add_shaped(p + "conv.up_even.weight", torch.cat([w0, w1 + w2], dim=1).contiguous())
            blob.add_shaped(p + "conv.up_odd.weight", torch.cat([w0 + w1, w2], dim=1).contiguous())
    elif b.kind == "out":
        blob.add_shaped(p + "0.weight", sd[p + "0.weight"])
        blob.add_shaped(p + "0.bias", sd[p + "0.bias"])
        blob.add_shaped(p + "2.weight", _conv3(sd[p + "2.weight"]))
        blob.add_shaped(p + "2.bias", sd[p + "2.bias"])
    elif b.kind == "dec_out":
        blob.add_shaped(p + "norm_out.weight", sd[p + "norm_out.weight"])
        blob.add_shaped(p + "norm_out.bias", sd[p + "norm_out.bias"])
        blob.add_shaped(p + "conv_out.weight", _conv3(sd[p + "conv_out.weight"]))
        blob.add_shaped(p + "conv_out.bias", sd[p + "conv_out.bias"])
    else:
        raise ValueError(b.kind)


def pack_model(sd: Dict[str, torch.Tensor], ucfg: UNetConfig, dcfg: DecoderConfig,
               unet_prefix: str = "model.unet_model.", dec_prefix: str = "model.first_stage_model.decoder.",
               tensor_core_split: bool = True, wave_cfg=None, encoder_cfg: Optional[EncoderConfig] = None,
               enc_prefix: str = "model.first_stage_model.encoder.") -> WeightBlob:
    blob = WeightBlob()
    up = unet_prefix
    for n in ("time_embed.0.", "time_embed.2."):
        blob.add_shaped(up + n + "weight", sd[up + n + "weight"])
        blob.add_shaped(up + n + "bias", sd[up + n + "bias"])
    blocks = list(unet_layout(ucfg, up).blocks())
    # fused emb_layers: one [sum Cout, 512] matrix, per-ResBlock column offsets recorded in meta
    res = [b for b in blocks if b.kind == "res"]
    blob.add_shaped(up + "emb_all.weight", torch.cat([sd[b.prefix + "emb_layers.1.weight"] for b in res], dim=0))
    blob.add_shaped(up + "emb_all.bias", torch.cat([sd[b.prefix + "emb_layers.1.bias"] for b in res], dim=0))
    off = 0
    emb_off = {}
    for b in res:
        emb_off[b.prefix] = off
        off += b.cout
    blob.meta["emb_offsets"] = emb_off
    blob.meta["emb_total"] = off
    for b in blocks:
        _pack_block(blob, sd, b)
    for b in decoder_layout(dcfg, dec_prefix):
        _pack_block(blob, sd, b)
    if any(k.startswith(enc_prefix) for k in sd):
        # the chart encoder (autoencoder.py:185-265), only when its weights are given: blobs without it are unchanged
        ecfg = encoder_cfg or EncoderConfig()
        for b in encoder_layout(ecfg, enc_prefix):
            _pack_block(blob, sd, b)
        blob.meta["encoder_cfg"] = ecfg
    if wave_cfg is not None or any(k.startswith("model.wave_model.") for k in sd):
        from .wave import WaveConfig, pack_wave            # SURVEY §8f N1: the audio encoder, once per request
        pack_wave(blob, sd, wave_cfg or WaveConfig())
    # Tensor-core weights (K per tap % 32 == 0, N >= 16) get their TF32 hi / lo operands ON THE DEVICE, after the blob has been
    # uploaded or broadcast (MUGD_OP_TF32_SPLIT: hi over the plain weight, lo in a second buffer).  The host blob -- what is packed,
    # stored and broadcast -- holds every weight once (0.56 GB, instead of W + W_hi + W_lo = 1.66 GB).
    blob.tc = []
    lo = 0
    for name in list(blob.entries):
        e = blob.entries[name]
        if tensor_core_split and name.endswith("weight") and len(e.shape) == 2 and e.shape[0] >= 16 and e.shape[1] % 32 == 0:
            n = e.shape[0] * e.shape[1]
            blob.tc.append((name, e.offset, n, lo))          # (entry, offset in the blob, elements, offset in the lo buffer)
            lo += (n + ALIGN - 1) // ALIGN * ALIGN
    blob.tc_lo_numel = lo
    blob.finalize()
    return blob


def blob_tensor(blob: WeightBlob, name: str) -> torch.Tensor:
    """an entry that was added earlier (in the packed layout, before finalize)"""
    return _chunk_of(blob, name).view(blob.entries[name].shape)


def _chunk_of(blob: WeightBlob, name: str) -> torch.Tensor:
    """the (not yet concatenated) flat tensor of an entry"""
    off = 0
    target = blob.entries[name].offset
    for c in blob._chunks:
        if off == target and c.numel() == int(torch.tensor(blob.entries[name].shape).prod()):
            return c
        off += c.numel()
    raise KeyError(name)
