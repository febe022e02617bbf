"""Structural walk of the reference networks: which blocks exist, in which order, with which
state_dict key prefixes, channel counts and sequence-length divisors.

This is the single source the weight packer, the launch-plan compiler and the synthetic-weight
generator share.  It mirrors the *constructors* of the reference (mug/diffusion/unet.py:341-493 for the
U-Net, mug/firststage/autoencoder.py:268-327 for the decoder, :185-242 for the encoder) so that key names equal the reference's
``state_dict()`` keys exactly (checked in tests/test_netspec.py against tests/golden/ref_keys.json).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, Iterator, List, Optional, Tuple

from .config import DecoderConfig, EncoderConfig, UNetConfig


@dataclass
class Block:
    kind: str                 # conv_in | res | attn | s4 | down | up | out | dec_res | dec_conv_in | dec_out
    prefix: str               # state_dict prefix, ends with '.'
    cin: int
    cout: int
    ds: int                   # sequence-length divisor relative to z_length (1,2,4,8); first stage: <1 via mul
    mul: int = 1              # decoder / encoder only: length multiplier (1,2,4,8) of the block's input
    heads: int = 0
    has_skip_conv: bool = False


@dataclass
class UNetLayout:
    """input_blocks / middle / output_blocks as the reference orders them.  Each entry of ``input`` and
    ``output`` is either the marker ("audio", level) or a list of Block."""
    input: List[object] = field(default_factory=list)
    middle: List[Block] = field(default_factory=list)
    output: List[object] = field(default_factory=list)
    out: Optional[Block] = None
    skip_channels: List[int] = field(default_factory=list)   # channels of every hs entry, push order

    def blocks(self) -> Iterator[Block]:
        """every Block in execution order: input, middle and output blocks (not the audio markers), then ``out``"""
        for entry in self.input + [self.middle] + self.output:
            if not isinstance(entry, tuple):
                yield from entry
        yield self.out


# sub-layer names (norm1, conv1, norm2, conv2, 1x1 skip) of the U-Net's TimestepResBlock (unet.py:121) and the decoder's ResnetBlock
# (models.py:94): the two compute the same thing, except that the U-Net adds a time-embedding row after conv1
RES_LAYERS = {"res": ("in_layers.0.", "in_layers.2.", "out_layers.0.", "out_layers.3.", "skip_connection."),
              "dec_res": ("norm1.", "conv1.", "norm2.", "conv2.", "nin_shortcut.")}


def unet_layout(cfg: UNetConfig, prefix: str = "model.unet_model.") -> UNetLayout:
    mc = cfg.model_channels
    lay = UNetLayout()
    lay.input.append([Block("conv_in", f"{prefix}input_blocks.0.0.", cfg.in_channels, mc, 1)])
    chans = [mc]
    ch, ds, idx = mc, 1, 1
    for level, mult in enumerate(cfg.channel_mult):
        lay.input.append(("audio", level))
        idx += 1
        ch += cfg.audio_channels[level]
        for _ in range(cfg.num_res_blocks):
            cout = mult * mc
            p = f"{prefix}input_blocks.{idx}."
            blocks = [Block("res", p + "0.", ch, cout, ds, has_skip_conv=(ch != cout))]
            ch = cout
            j = 1
            if ds in cfg.attention_resolutions:
                blocks.append(Block("attn", f"{p}{j}.", ch, ch, ds, heads=cfg.num_heads))
                j += 1
            if cfg.s4_layer:
                blocks.append(Block("s4", f"{p}{j}.", ch, ch, ds))
            lay.input.append(blocks)
            chans.append(ch)
            idx += 1
        if level != cfg.levels - 1:
            lay.input.append([Block("down", f"{prefix}input_blocks.{idx}.0.", ch, ch, ds)])
            chans.append(ch)
            idx += 1
            ds *= 2
    lay.skip_channels = list(chans)
    mp = f"{prefix}middle_block."
    lay.middle = [
        Block("res", mp + "0.", ch, ch, ds),
        Block("attn", mp + "1.", ch, ch, ds, heads=cfg.num_heads),
        Block("res", mp + "2.", ch, ch, ds),
    ]
    idx = 0
    for level in reversed(range(cfg.levels)):
        mult = cfg.channel_mult[level]
        lay.output.append(("audio", level))
        idx += 1
        ch += cfg.audio_channels[level]
        for i in range(cfg.num_res_blocks + 1):
            ich = chans.pop()
            cout = mc * mult
            p = f"{prefix}output_blocks.{idx}."
            blocks = [Block("res", p + "0.", ch + ich, cout, ds, has_skip_conv=(ch + ich != cout))]
            ch = cout
            j = 1
            if ds in cfg.attention_resolutions:
                blocks.append(Block("attn", f"{p}{j}.", ch, ch, ds, heads=cfg.num_heads))
                j += 1
            if cfg.s4_layer and i != cfg.num_res_blocks:
                blocks.append(Block("s4", f"{p}{j}.", ch, ch, ds))
                j += 1
            if level and i == cfg.num_res_blocks:
                blocks.append(Block("up", f"{p}{j}.", ch, ch, ds))
                ds //= 2
            lay.output.append(blocks)
            idx += 1
    lay.out = Block("out", f"{prefix}out.", mc, cfg.out_channels, 1)
    return lay


def decoder_layout(cfg: DecoderConfig, prefix: str = "model.first_stage_model.decoder.") -> List[Block]:
    """Execution order of Decoder.forward (autoencoder.py:329-354)."""
    nres = len(cfg.channel_mult)
    block_in = cfg.middle_channels * cfg.channel_mult[-1]
    seq = [Block("dec_conv_in", prefix + "conv_in.", cfg.z_channels, block_in, 1, mul=1)]
    seq.append(Block("dec_res", prefix + "mid.block_1.", block_in, block_in, 1, mul=1))
    seq.append(Block("dec_res", prefix + "mid.block_2.", block_in, block_in, 1, mul=1))
    mul = 1
    for lvl in reversed(range(nres)):
        block_out = cfg.middle_channels * cfg.channel_mult[lvl]
        for b in range(cfg.num_res_blocks + 1):
            seq.append(Block("dec_res", f"{prefix}up.{lvl}.block.{b}.", block_in, block_out, 1, mul=mul,
                             has_skip_conv=(block_in != block_out)))
            block_in = block_out
        if lvl != 0:
            seq.append(Block("up", f"{prefix}up.{lvl}.upsample.", block_in, block_in, 1, mul=mul))
            mul *= 2
    seq.append(Block("dec_out", prefix, block_in, cfg.x_channels, 1, mul=mul))
    return seq


def encoder_layout(cfg: EncoderConfig, prefix: str = "model.first_stage_model.encoder.") -> List[Block]:
    """Execution order of Encoder.forward (autoencoder.py:244-265): conv_in, per level the ResnetBlocks and (all but the last level)
    a stride-2 Downsample, two mid ResnetBlocks, norm_out + SiLU + conv_out to 2 * z_channels moments.  The decoder's block kinds
    describe every layer; ``mul`` runs 2^(levels-1) .. 1."""
    nres = len(cfg.channel_mult)
    mc = cfg.middle_channels
    mul = 1 << (nres - 1)
    seq = [Block("dec_conv_in", prefix + "conv_in.", cfg.x_channels, mc, 1, mul=mul)]
    block_in = mc                                     # inchannel_mult = (1,) + channel_mult (:199)
    for lvl in range(nres):
        block_out = mc * cfg.channel_mult[lvl]
        for b in range(cfg.num_res_blocks):
            seq.append(Block("dec_res", f"{prefix}down.{lvl}.block.{b}.", block_in, block_out, 1, mul=mul,
                             has_skip_conv=(block_in != block_out)))
            block_in = block_out
        if lvl != nres - 1:
            seq.append(Block("down", f"{prefix}down.{lvl}.downsample.", block_in, block_in, 1, mul=mul))
            mul //= 2
    seq.append(Block("dec_res", prefix + "mid.block_1.", block_in, block_in, 1, mul=mul))
    seq.append(Block("dec_res", prefix + "mid.block_2.", block_in, block_in, 1, mul=mul))
    seq.append(Block("dec_out", prefix, block_in, 2 * cfg.z_channels, 1, mul=mul))
    return seq


# --------------------------------------------------------------------------------------------------
# parameter manifest:  name -> (shape, role)
# roles drive the synthetic initialiser only: w (fan-in scaled), b, gamma, beta, relpos, cemb, s4_*
# --------------------------------------------------------------------------------------------------
Spec = Tuple[Tuple[int, ...], str]


def _conv(out: Dict[str, Spec], pre: str, cin: int, cout: int, k: int):
    out[pre + "weight"] = ((cout, cin, k), "w")
    out[pre + "bias"] = ((cout,), "b")


def _lin(out: Dict[str, Spec], pre: str, cin: int, cout: int, bias: bool = True):
    out[pre + "weight"] = ((cout, cin), "w")
    if bias:
        out[pre + "bias"] = ((cout,), "b")


def _norm(out: Dict[str, Spec], pre: str, c: int):
    out[pre + "weight"] = ((c,), "gamma")
    out[pre + "bias"] = ((c,), "beta")


def _block_params(out: Dict[str, Spec], b: Block, cfg: UNetConfig):
    p = b.prefix
    if b.kind == "conv_in":
        _conv(out, p, b.cin, b.cout, 3)
    elif b.kind == "res":
        _norm(out, p + "in_layers.0.", b.cin)
        _conv(out, p + "in_layers.2.", b.cin, b.cout, 3)
        _lin(out, p + "emb_layers.1.", cfg.time_embed_dim, b.cout)
        _norm(out, p + "out_layers.0.", b.cout)
        _conv(out, p + "out_layers.3.", b.cout, b.cout, 3)
        if b.has_skip_conv:
            _conv(out, p + "skip_connection.", b.cin, b.cout, 1)
    elif b.kind == "attn":
        c = b.cin
        _norm(out, p + "norm.", c)
        _conv(out, p + "proj_in.", c, c, 1)
        t = p + "transformer_blocks.0."
        for name, ctx in (("attn1.", c), ("attn2.", cfg.context_dim)):
            a = t + name
            out[a + "relative_position_embedding"] = ((2 * cfg.pos_max + 1, b.heads), "relpos")
            out[a + "C_embedding"] = ((2 * cfg.pos_max + 1, b.heads), "cemb")
            _lin(out, a + "to_q.", c, c, bias=False)
            _lin(out, a + "to_k.", ctx, c, bias=False)
            _lin(out, a + "to_v.", ctx, c, bias=False)
            _lin(out, a + "to_out.0.", c, c)
        _lin(out, t + "ff.net.0.proj.", c, 8 * c)
        _lin(out, t + "ff.net.2.", 4 * c, c)
        for n in ("norm1.", "norm2.", "norm3."):
            _norm(out, t + n, c)
        _conv(out, p + "proj_out.", c, c, 1)
    elif b.kind == "s4":
        h, n = b.cin, cfg.s4_state // 2
        _norm(out, p + "norm.", h)
        s = p + "s4_model."
        out[s + "D"] = ((1, h), "s4_D")
        k = s + "kernel.kernel."
        out[k + "C"] = ((1, h, n, 2), "s4_C")
        out[k + "log_dt"] = ((h,), "s4_log_dt")
        out[k + "B"] = ((1, h, n, 2), "s4_B")
        out[k + "P"] = ((1, h, n, 2), "s4_P")
        out[k + "inv_w_real"] = ((h, n), "s4_inv_w_real")
        out[k + "w_imag"] = ((h, n), "s4_w_imag")
        out[k + "L"] = ((), "s4_L")
        _conv(out, s + "output_linear.0.", h, 2 * h, 1)
        _conv(out, p + "out_layer.", h, h, 3)
    elif b.kind in ("down", "up"):
        _conv(out, p + "conv.", b.cin, b.cout, 3)
    elif b.kind == "out":
        _norm(out, p + "0.", b.cin)
        _conv(out, p + "2.", b.cin, b.cout, 3)
    else:
        raise ValueError(b.kind)


def unet_param_specs(cfg: UNetConfig, prefix: str = "model.unet_model.") -> Dict[str, Spec]:
    out: Dict[str, Spec] = {}
    _lin(out, prefix + "time_embed.0.", cfg.model_channels, cfg.time_embed_dim)
    _lin(out, prefix + "time_embed.2.", cfg.time_embed_dim, cfg.time_embed_dim)
    for b in unet_layout(cfg, prefix).blocks():
        _block_params(out, b, cfg)
    return out


def _first_stage_params(seq: List[Block]) -> Dict[str, Spec]:
    out: Dict[str, Spec] = {}
    for b in seq:
        p = b.prefix
        if b.kind == "dec_conv_in":
            _conv(out, p, b.cin, b.cout, 3)
        elif b.kind == "dec_res":
            _norm(out, p + "norm1.", b.cin)
            _conv(out, p + "conv1.", b.cin, b.cout, 3)
            _norm(out, p + "norm2.", b.cout)
            _conv(out, p + "conv2.", b.cout, b.cout, 3)
            if b.has_skip_conv:
                _conv(out, p + "nin_shortcut.", b.cin, b.cout, 1)
        elif b.kind in ("up", "down"):
            _conv(out, p + "conv.", b.cin, b.cout, 3)
        elif b.kind == "dec_out":
            _norm(out, p + "norm_out.", b.cin)
            _conv(out, p + "conv_out.", b.cin, b.cout, 3)
    return out


def decoder_param_specs(cfg: DecoderConfig, prefix: str = "model.first_stage_model.decoder.") -> Dict[str, Spec]:
    return _first_stage_params(decoder_layout(cfg, prefix))


def encoder_param_specs(cfg: EncoderConfig, prefix: str = "model.first_stage_model.encoder.") -> Dict[str, Spec]:
    return _first_stage_params(encoder_layout(cfg, prefix))
